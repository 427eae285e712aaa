"""Proofs per second of b2s_groth16_prove_batch against a loop of b2s_groth16_prove_resident over the same z, r, s.

DummyCircuit-shaped R1CS at domain 2^log_n (every row z[2] * z[3] = z[1]) with a key from the GPU setup.  Two witness
shapes: uniform random scalars, and all-equal (DummyCircuit) witnesses, where the single-proof loop keeps the
multiplicity-aware MSM front end and the batch does not.  The two paths alternate, z / r / s stay on the device for both.
Also reports launches per proof, checks a sample of the batch proofs against the loop's, and with --profile prints the
per-kernel time (b2s_profile_*) of one batch call in a separate run.

  python tools/prove_batch_bench.py [--curves 0 1] [--logs 12 16 20] [--ks 1 16 64 256] [--reps 3] [--profile 16:64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

R = {0: 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
     1: 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001}


def mont(curve, x):
    v = x * (1 << 256) % R[curve]
    return np.array([(v >> (32 * i)) & 0xFFFFFFFF for i in range(8)], dtype=np.uint32)


def instance(curve, log_n):
    N = 1 << log_n
    n_rows, n_inst, n_wit = N - 2, 2, N - 3
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    coeff = np.tile(mont(curve, 1), nnz)
    return [(row_ptr, np.full(nnz, col, dtype=np.uint32), coeff) for col in (2, 3, 1)], n_rows, n_inst, n_wit


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def witnesses(torch, curve, K, n_vars, shape, seed):
    """K rows of n_vars Montgomery scalars on the device, z[0] = 1, z[1] = z[2] z[3] (satisfying)"""
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    rng = np.random.default_rng(seed)
    if shape == "uniform":
        z = torch.randint(-(1 << 31), (1 << 31) - 1, (K, n_vars, 8), dtype=torch.int32, device="cuda", generator=g)
        z[:, :, 7] &= 0x0FFFFFFF                # < 2^252 < r: valid Montgomery representations
    else:
        z = torch.empty((K, n_vars, 8), dtype=torch.int32, device="cuda")
    for k in range(K):
        a, b = (int.from_bytes(rng.bytes(32), "little") % R[curve] for _ in range(2))
        if shape != "uniform":
            z[k, 1:] = torch.from_numpy(mont(curve, a).view(np.int32)).cuda()
        for j, v in ((0, 1), (1, a * b % R[curve]), (2, a), (3, b)):
            z[k, j] = torch.from_numpy(mont(curve, v).view(np.int32)).cuda()
    rs = [np.concatenate([mont(curve, int.from_bytes(rng.bytes(32), "little") % R[curve]) for _ in range(K)]) for _ in range(2)]
    return z.reshape(K, -1).contiguous(), rs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", type=int, nargs="+", default=[0, 1])
    ap.add_argument("--logs", type=int, nargs="+", default=[12, 16, 20])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 16, 64, 256])
    ap.add_argument("--shapes", nargs="+", default=["uniform", "all_equal"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", default="", help="LOG:K -- per-kernel profile of one batch call (separate run)")
    args = ap.parse_args()
    import torch

    from snark_b200 import Backend

    if not torch.cuda.is_available():
        sys.exit("prove_batch_bench: no GPU")
    print(json.dumps({"card": card()}), flush=True)
    for curve in args.curves:
        be = Backend(curve=curve)
        fr = be.fr_bytes // 4
        for log_n in args.logs:
            csr, n_rows, n_inst, n_wit = instance(curve, log_n)
            m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
            td = np.concatenate([mont(curve, 1000003 + 17 * i) for i in range(5)])
            pk, _vk = be.groth16_setup(m, td, n_inst)
            n_vars = n_inst + n_wit
            for shape in args.shapes:
                z, (r, s) = witnesses(torch, curve, max(args.ks), n_vars, shape, 7 + log_n)
                rd = torch.from_numpy(r.view(np.int32)).cuda()
                sd = torch.from_numpy(s.view(np.int32)).cuda()
                for K in args.ks:
                    def batch():
                        return be.groth16_prove_batch(pk, m, z[:K], rd[:K * fr], sd[:K * fr])

                    def loop():
                        return [be.groth16_prove_resident(pk, m, z[k], r[k * fr:(k + 1) * fr], s[k * fr:(k + 1) * fr]) for k in range(K)]

                    out_b, out_l = batch(), loop()      # warm-up of both, and the outputs compared below
                    sample = sorted({0, K // 2, K - 1})
                    same = all(np.array_equal(out_b[j][k].cpu().numpy().view(np.uint32), out_l[k][j]) for k in sample for j in range(3))
                    tb, tl = [], []
                    for _ in range(args.reps):
                        t0 = time.perf_counter(); batch(); tb.append(time.perf_counter() - t0)
                        t0 = time.perf_counter(); loop(); tl.append(time.perf_counter() - t0)
                    n0 = be.launches; batch(); lb = be.launches - n0
                    n0 = be.launches; loop(); ll = be.launches - n0
                    b_ps, l_ps = K / float(np.median(tb)), K / float(np.median(tl))
                    print(json.dumps({"curve": ["bls12_381", "bn254"][curve], "log_n": log_n, "shape": shape, "K": K,
                                      "batch_proofs_per_s": round(b_ps, 2), "loop_proofs_per_s": round(l_ps, 2),
                                      "speedup": round(b_ps / l_ps, 3), "batch_ms": [round(1e3 * t, 2) for t in tb],
                                      "loop_ms": [round(1e3 * t, 2) for t in tl], "launches_per_proof_batch": round(lb / K, 2),
                                      "launches_per_proof_loop": round(ll / K, 2), "sample_identical": same}), flush=True)
                    assert same, "batch proofs differ from the single-proof loop"
                del z, rd, sd
                torch.cuda.empty_cache()
            if args.profile and int(args.profile.split(":")[0]) == log_n:
                K = int(args.profile.split(":")[1])
                z, (r, s) = witnesses(torch, curve, K, n_vars, "uniform", 99)
                rd, sd = torch.from_numpy(r.view(np.int32)).cuda(), torch.from_numpy(s.view(np.int32)).cuda()
                be.groth16_prove_batch(pk, m, z, rd, sd)
                be.profile(True)
                be.profile_report()
                t0 = time.perf_counter()
                be.groth16_prove_batch(pk, m, z, rd, sd)
                wall = time.perf_counter() - t0
                rep = be.profile_report()
                be.profile(False)
                tot = sum(ms for _, ms in rep.values())
                top = sorted(rep.items(), key=lambda kv: -kv[1][1])[:16]
                print(json.dumps({"profile": {"curve": curve, "log_n": log_n, "K": K, "wall_ms": round(1e3 * wall, 2),
                                              "kernel_ms": round(tot, 2), "launches": sum(c for c, _ in rep.values()),
                                              "top": {k: [c, round(ms, 3)] for k, (c, ms) in top}}}), flush=True)
                del z, rd, sd
            be.pk_free(pk)
            be.r1cs_free(m)
        be.close()


if __name__ == "__main__":
    main()
