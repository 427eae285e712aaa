#!/usr/bin/env python3
"""Time of loading an ark-groth16 ProvingKey onto the GPU (b2s_pk_deserialize), one run.

Builds a synthetic key with b2s_groth16_setup at domain 2^--log-n on --curve, serializes it with b2s_pk_serialize in both
forms, then times b2s_pk_deserialize for compressed / uncompressed with validate 0 and 1 (host clock around the
synchronising call, after one warm-up at 2^12; the h-query window table is switched off, B2S_PK_PRECOMP=0, so that the
time is the decoding) and checks every b2s_pk_query vector of the loaded key against the original.
Prints one JSON line with the card name and power limit read in the same run.

The Fq multiplication count per point is taken from the algorithm (csrc/deserialize.cuh), counting a squaring as a
multiplication and an Fq2 multiplication as three: a square root in Fq is one exponentiation by (p-3)/4
(bits - 1 squarings + popcount - 1 multiplications) plus 3; an Fq2 root is three such exponentiations plus about 12;
a double-and-add step of XYZZ costs about 10 (doubling) and 14 (addition) multiplications of the coordinate field.
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

BLS_P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
BN_P = 21888242871839275222246405745257275088696311157297823662689037894645226208583
FQ_MUL_CEILING = {0: 2.6e10}   # Fq(381-bit) mul/s on an H100 at 400 W (tools/microbench.cu, DESIGN §4)


def fq_muls_per_point(curve, group, compressed, validate):
    p = BLS_P if curve == 0 else BN_P
    e = (p - 3) // 4
    exp = e.bit_length() - 1 + bin(e).count("1") - 1
    ext = 1 if group == 1 else 3                       # Fq muls per coordinate-field mul
    n = 2 * group + 1                                  # to Montgomery
    if compressed:
        n += (exp + 3) if group == 1 else (3 * exp + 12)
        n += 2 * group                                 # sign choice (from Montgomery)
    elif validate:
        n += 3 * ext                                   # curve equation
    if validate:
        if curve == 0 and group == 1:                  # 2 x [|x|], |x| = 64 bits, weight 6
            n += 2 * (63 * 10 + 5 * 14) + 3
        elif curve == 0:                               # [|x|] + psi
            n += (63 * 10 + 5 * 14) * ext + 4 * ext
        elif group == 2:                               # [6 x^2], 127 bits
            k = 6 * 4965661367192848881 ** 2
            n += ((k.bit_length() - 1) * 10 + (bin(k).count("1") - 1) * 14) * ext + 4 * ext
    return n


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return "unknown", "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--log-n", type=int, default=24)
    ap.add_argument("--curve", choices=["bls12_381", "bn254"], default="bls12_381")
    a = ap.parse_args()
    os.environ["B2S_PK_PRECOMP"] = "0"
    from snark_b200 import Backend
    from tests.test_gpu_fullsize import dummy_csr
    from tests.util import pack_fr

    curve_id = 0 if a.curve == "bls12_381" else 1
    be = Backend(curve=curve_id)
    from oracle.params import BLS12_381, BN254
    curve = BLS12_381 if curve_id == 0 else BN254
    rng = random.Random(5)

    def make_key(log_n):
        n_rows, n_wit = (1 << log_n) - 8, (1 << log_n) - 16     # |a| = |b| ~ the domain, as in the benchmarked key
        csr, _, _ = dummy_csr(curve, n_rows, 3, 5, n_wit)
        m = be.r1cs_upload(n_rows, 2, n_wit, csr)
        pk, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), 2)
        return m, pk, vk, 2 + n_wit, n_wit, be.domain_size(m)

    def key_bytes(pk, vk, compressed):
        vkb = be.vk_bytes(vk["alpha_g1"], vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"], vk["gamma_abc_g1"], 2, compressed)
        return be.pk_bytes(pk, vkb, compressed)

    # warm-up at a small size: contexts, kernels, pinned allocations
    m, pk, vk, *_ = make_key(12)
    be.pk_free(be.pk_from_bytes(key_bytes(pk, vk, True), True, True))
    be.pk_free(pk)
    be.r1cs_free(m)

    m, pk, vk, n_vars, n_wit, domain = make_key(a.log_n)
    counts = [n_vars, n_vars, n_vars, domain - 1, n_wit, 3, 2]
    orig = [be.pk_query(pk, w, n) for w, n in enumerate(counts)]
    g1_pts = 3 * n_vars + domain - 1 + n_wit + 2 + 3 + 2     # a, b_g1, h, l, gamma_abc, alpha / beta / delta
    g2_pts = n_vars + 3
    # the point at infinity is decoded from its flags alone: only finite points cost field arithmetic (the synthetic
    # circuit leaves most of a, b_g1, b_g2 at infinity)
    finite = lambda arr, words: int(np.count_nonzero(arr.reshape(-1, words).any(axis=1)))
    w1, w2 = be.g1_bytes // 4, be.g2_bytes // 4
    g1_fin = sum(finite(orig[w], w1) for w in (0, 1, 3, 4, 5)) + 2   # + gamma_abc_g1
    g2_fin = sum(finite(orig[w], w2) for w in (2, 6)) + 1             # + gamma_g2
    cases = []
    for compressed in (True, False):
        blob = key_bytes(pk, vk, compressed)
        for validate in (False, True):
            t0 = time.perf_counter()
            loaded = be.pk_from_bytes(blob, compressed, validate)
            dt = time.perf_counter() - t0
            equal = all(np.array_equal(be.pk_query(loaded, w, n), o) for (w, n), o in zip(enumerate(counts), orig))
            be.pk_free(loaded)
            muls = (g1_fin * fq_muls_per_point(curve_id, 1, compressed, validate)
                    + g2_fin * fq_muls_per_point(curve_id, 2, compressed, validate))
            case = {"compressed": compressed, "validate": validate, "seconds": round(dt, 4), "bytes": len(blob),
                    "points_per_s": round((g1_pts + g2_pts) / dt), "input_GB_per_s": round(len(blob) / dt / 1e9, 3),
                    "finite_points_per_s": round((g1_fin + g2_fin) / dt), "fq_mul_per_s_est": float("%.3g" % (muls / dt)), "equal_to_original": equal}
            if curve_id in FQ_MUL_CEILING:
                case["fraction_of_fq_mul_ceiling"] = round(muls / dt / FQ_MUL_CEILING[curve_id], 3)
            cases.append(case)
        del blob
    name, power = card()
    print(json.dumps({"tool": "pk_load_probe", "curve": a.curve, "log_n": a.log_n, "g1_points": g1_pts, "g2_points": g2_pts,
                      "g1_finite": g1_fin, "g2_finite": g2_fin,
                      "gpu": name, "power_limit": power, "cases": cases}))
    be.pk_free(pk)
    be.r1cs_free(m)
    be.close()


if __name__ == "__main__":
    main()
