#!/usr/bin/env python3
"""Time of loading a snarkjs Groth16 .zkey and a .wtns onto the GPU against the ark route, one run.

For each --log-n: builds a DummyCircuit-shaped R1CS (every row z[2] z[3] = z[1]) and a circom key with
b2s_groth16_setup_qap on --curve, writes them as a zkey with the test-side writer (tests/zkey_oracle.py) and times, with
the host clock around synchronising calls (after one warm-up of every step at 2^12):
  - b2s_zkey_load with validate 0 and 1;
  - the ark route to the same handles: b2s_pk_deserialize_qap of the key's compressed ark bytes (validate 0 and 1) plus
    b2s_r1cs_upload of A and B (host-side coefficient interning);
  - b2s_wtns_read into device memory + b2s_groth16_prove_resident, against b2s_groth16_prove with host z.
It checks that the loaded key equals the original (every b2s_pk_query vector), that the loaded matrices give the same circom
witness map as the uploaded ones and that both proofs are equal.  The h-query window table is switched off
(B2S_PK_PRECOMP=0) so that a load time is the loading.  Prints one JSON line with the card name and power limit read in the
same run.  The synthetic circuit leaves most of a, b_g1 and b_g2 at infinity, which costs no curve arithmetic.
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, round(time.perf_counter() - t0, 4)


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--curve", choices=["bls12_381", "bn254"], default="bls12_381")
    a = ap.parse_args()
    os.environ["B2S_PK_PRECOMP"] = "0"
    import torch

    from oracle.params import BLS12_381, BN254
    from snark_b200 import Backend
    from snark_b200.lib import QAP_CIRCOM
    from tests import zkey_oracle as zo
    from tests.test_gpu_circom import dummy_2k
    from tests.util import pack_fr

    curve_id = 0 if a.curve == "bls12_381" else 1
    curve = BLS12_381 if curve_id == 0 else BN254
    be = Backend(curve=curve_id)
    rng = random.Random(7)

    def run(log_n):
        csr, n_rows, n_inst, n_wit, z_inst, z_wit = dummy_2k(curve, log_n)
        n_vars = n_inst + n_wit
        empty = (np.zeros(n_rows + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32))
        m0 = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
        domain = be.domain_size(m0)
        pk0, vk = be.groth16_setup(m0, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst, qap=QAP_CIRCOM)
        key = zo.key_arrays_device(be, pk0, vk, n_inst, n_wit, domain)
        zkey = zo.write_zkey(curve, key, csr[0], csr[1], n_inst - 1, domain)
        vkb = be.vk_bytes(vk["alpha_g1"], vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"], vk["gamma_abc_g1"][: n_inst * be.g1_bytes // 4], n_inst)
        ark = be.pk_bytes(pk0, vkb, True)
        z = np.concatenate([z_inst, z_wit])
        wtns = zo.write_wtns(curve, z)
        res = {"log_n": log_n, "zkey_bytes": len(zkey), "ark_pk_bytes": len(ark), "wtns_bytes": len(wtns)}
        counts = [n_vars, n_vars, n_vars, domain, n_wit, 3, 2]
        for validate in (0, 1):
            (pk, m, _), dt = timed(lambda: be.zkey_load(zkey, validate=bool(validate)))
            res[f"zkey_load_v{validate}_s"] = dt
            if validate:
                res["key_equal"] = all(np.array_equal(be.pk_query(pk, w, n), be.pk_query(pk0, w, n)) for w, n in enumerate(counts))
                res["witness_map_equal"] = bool(np.array_equal(be.witness_map(m, z, qap=QAP_CIRCOM), be.witness_map(m0, z, qap=QAP_CIRCOM)))
                zt = torch.zeros(n_vars * 8, dtype=torch.int32, device="cuda")
                r, s = pack_fr(curve, [rng.randrange(curve.r)]), pack_fr(curve, [rng.randrange(curve.r)])

                def zkey_prove():
                    be.wtns_read(wtns, n_vars, out=zt)
                    return be.groth16_prove_resident(pk, m, zt, r, s)

                p1, res["wtns_read_prove_resident_s"] = timed(zkey_prove)
                p0, res["prove_host_z_s"] = timed(lambda: be.groth16_prove(pk0, m0, z_inst, z_wit, r, s))
                res["proofs_equal"] = all(np.array_equal(x, y) for x, y in zip(p0, p1))
                _, res["wtns_read_s"] = timed(lambda: (be.wtns_read(wtns, n_vars, out=zt), be.sync()))
            be.pk_free(pk)
            be.r1cs_free(m)
            pka, dt = timed(lambda: be.pk_from_bytes(ark, True, bool(validate), qap=QAP_CIRCOM))
            res[f"ark_pk_deserialize_v{validate}_s"] = dt
            be.pk_free(pka)
        mu, res["ark_r1cs_upload_s"] = timed(lambda: be.r1cs_upload(n_rows, n_inst, n_wit, [csr[0], csr[1], empty]))
        be.r1cs_free(mu)
        for v in (0, 1):
            res[f"speedup_v{v}"] = round((res[f"ark_pk_deserialize_v{v}_s"] + res["ark_r1cs_upload_s"]) / res[f"zkey_load_v{v}_s"], 2)
        be.pk_free(pk0)
        be.r1cs_free(m0)
        return res

    run(12)   # warm-up: kernels, pinned buffers, NTT plans
    cases = [run(n) for n in a.log_n]
    name, power = card()
    print(json.dumps({"tool": "zkey_probe", "curve": a.curve, "gpu": name, "power_limit": power, "cases": cases}))
    be.close()


if __name__ == "__main__":
    main()
