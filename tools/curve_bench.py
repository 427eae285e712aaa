#!/usr/bin/env python3
"""BLS12-377 next to BLS12-381 in one process, the two curves alternated in every round.

    python tools/curve_bench.py --log-prove 24 --log-msm 22 --log-ntt 24 --log-verify 16 --log-pk 20 --reps 3

Per curve and round (median over --reps rounds):
  prove    b2s_groth16_prove_resident of a 2^log_prove DummyCircuit-shaped R1CS, key from b2s_groth16_setup, z on the device
  msm      one G1 MSM of 2^log_msm uniform scalars over device bases (k_i G from the fixed-base kernel)
  ntt      one forward NTT of 2^log_ntt elements in device memory
  verify   proofs/s of groth16_verify_batch and groth16_verify_all (RLC) over 2^log_verify host proofs (8 distinct, tiled)
  pk       a validated, compressed b2s_pk_deserialize of a 2^log_pk key (the ark ProvingKey bytes of a GPU setup)
Host clocks around calls that end in a device synchronise.  Prints one JSON line with the card and its power limit and SM
clock, the per-curve medians and the BLS12-377 / BLS12-381 ratios.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

R = {0: 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
     2: 0x12AB655E9A2CA55660B44D1E5C37B00159AA76FED00000010A11800000000001}
NAMES = {0: "bls12_381", 2: "bls12_377"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def mont(curve, xs):
    return np.frombuffer(b"".join((x * (1 << 256) % R[curve]).to_bytes(32, "little") for x in xs), dtype=np.uint32).copy()


def rand_scalars(rng, n):
    a = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
    a[:, 7] &= np.uint32((1 << 28) - 1)        # < 2^252, below both scalar moduli
    return a.reshape(-1)


def dummy(curve, log_n, seed):
    """DummyCircuit shape: rows x2 * x3 = x1 with x2 = a, x3 = b; n_rows + n_inst fills the domain 2^log_n"""
    N = 1 << log_n
    n_rows, n_inst, n_wit = N - 2, 2, N - 3
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    coeff = np.tile(mont(curve, [1]), nnz)
    csr = [(row_ptr, np.full(nnz, col, dtype=np.uint32), coeff) for col in (2, 3, 1)]
    rng = np.random.default_rng(seed)
    a, b = (int.from_bytes(rng.bytes(32), "little") % R[curve] for _ in range(2))
    z = np.concatenate([mont(curve, [1, a * b % R[curve]]), np.tile(mont(curve, [a]), n_wit)])
    z[8 * 3: 8 * 4] = mont(curve, [b])
    return csr, n_rows, n_inst, n_wit, z


def timed(fn, sync):
    sync()
    t = time.perf_counter()
    fn()
    sync()
    return time.perf_counter() - t


class Case:
    """one curve's resident inputs"""

    def __init__(self, curve, args, torch):
        from snark_b200 import Backend

        self.curve, self.torch = curve, torch
        self.be = be = Backend(curve=curve)
        dev = torch.device("cuda", 0)
        rng = np.random.default_rng(curve + 1)

        def tr(a):   # to the device, finished before the library's stream reads it
            t = torch.from_numpy(a.view(np.int32)).to(dev)
            torch.cuda.synchronize()
            return t

        td = mont(curve, [int(x) + 2 for x in rng.integers(1, 1 << 62, size=5)])
        # prove
        csr, n_rows, n_inst, n_wit, z = dummy(curve, args.log_prove, 7)
        self.m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
        self.pk, _ = be.groth16_setup(self.m, td, n_inst)
        self.z = tr(z)
        self.r, self.s = mont(curve, [3]), mont(curve, [5])
        # msm / ntt
        n = 1 << args.log_msm
        self.msm_n = n
        k = tr(rand_scalars(rng, n))
        self.bases = torch.zeros(n * be.g1_bytes // 4, dtype=torch.int32, device=dev)
        be.fixed_base(1, k, n, mont=False, out=self.bases)
        self.sc = tr(rand_scalars(rng, n))
        self.log_ntt = args.log_ntt
        self.ntt_data = tr(rand_scalars(rng, 1 << args.log_ntt))
        # verify: 8 proofs of a small circuit, tiled
        vcsr, vr, vi, vw, vz = dummy(curve, 10, 9)
        vm = be.r1cs_upload(vr, vi, vw, vcsr)
        vpk, vk = be.groth16_setup(vm, td, vi)
        prf = [be.groth16_prove(vpk, vm, vz[: 8 * vi], vz[8 * vi:], mont(curve, [i + 1]), mont(curve, [i + 2])) for i in range(8)]
        nv = 1 << args.log_verify
        self.nv = nv
        self.va, self.vb, self.vc = (np.tile(np.concatenate([p[j] for p in prf]), nv // 8) for j in range(3))
        self.vin = np.tile(vz[8: 16], nv)
        self.pvk = be.vk_prepare(vk)
        be.pk_free(vpk)
        be.r1cs_free(vm)
        # pk bytes
        pcsr, pr_, pi, pw, _ = dummy(curve, args.log_pk, 11)
        pm = be.r1cs_upload(pr_, pi, pw, pcsr)
        ppk, pvk = be.groth16_setup(pm, td, pi)
        vkb = be.vk_bytes(pvk["alpha_g1"], pvk["beta_g2"], pvk["gamma_g2"], pvk["delta_g2"], pvk["gamma_abc_g1"], pi)
        self.pk_bytes = be.pk_bytes(ppk, vkb)
        be.pk_free(ppk)
        be.r1cs_free(pm)

    def sync(self):
        self.torch.cuda.synchronize()
        self.be.sync()

    def round(self):
        be = self.be
        out = {}
        out["prove_ms"] = 1e3 * timed(lambda: be.groth16_prove_resident(self.pk, self.m, self.z, self.r, self.s), self.sync)
        out["msm_g1_ms"] = 1e3 * timed(lambda: be.msm_g1(self.bases, self.sc, self.msm_n, mont=False), self.sync)
        out["ntt_ms"] = 1e3 * timed(lambda: be.ntt(self.ntt_data, self.log_ntt), self.sync)
        ok = []
        t = timed(lambda: ok.append(be.groth16_verify_batch(self.pvk, self.vin, 1, self.va, self.vb, self.vc)), self.sync)
        assert ok[0].all()
        out["verify_batch_per_s"] = self.nv / t
        t = timed(lambda: ok.append(be.groth16_verify_all(self.pvk, self.vin, 1, self.va, self.vb, self.vc)), self.sync)
        assert ok[1]
        out["verify_rlc_per_s"] = self.nv / t

        def load():
            be.pk_free(be.pk_from_bytes(self.pk_bytes, compressed=True, validate=True))

        out["pk_deserialize_ms"] = 1e3 * timed(load, self.sync)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-prove", type=int, default=24)
    ap.add_argument("--log-msm", type=int, default=22)
    ap.add_argument("--log-ntt", type=int, default=24)
    ap.add_argument("--log-verify", type=int, default=16)
    ap.add_argument("--log-pk", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("curve_bench: no GPU")
    cases = [Case(c, args, torch) for c in (0, 2)]
    for c in cases:                  # warm-up round, not recorded
        c.round()
    runs = {c.curve: [] for c in cases}
    for _ in range(args.reps):
        for c in cases:
            runs[c.curve].append(c.round())
    med = {NAMES[c]: {k: float(np.median([r[k] for r in rs])) for k in rs[0]} for c, rs in runs.items()}
    ratio = {k: med["bls12_377"][k] / med["bls12_381"][k] for k in med["bls12_381"]}
    print(json.dumps({"card": card(), "args": vars(args), "median": med, "ratio_377_over_381": ratio,
                      "runs": {NAMES[c]: rs for c, rs in runs.items()}}))


if __name__ == "__main__":
    main()
