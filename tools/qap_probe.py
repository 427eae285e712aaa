"""Libsnark- vs circom-reduction Groth16 proofs on one GPU: time, witness-map kernels and bit equality.

DummyCircuit-shaped R1CS at domain 2^log_n (every row z[2] * z[3] = z[1]) with a satisfying assignment resident on the
device.  Per curve and size, one trapdoor gives a B2S_QAP_LIBSNARK and a B2S_QAP_CIRCOM key from the GPU setup; only one key
is resident at a time (at 2^24 each holds the ~20 GiB h-query table), so every round sets up the libsnark key, proves, frees
it, then does the same with the circom key.  In each residency one warm-up proof is followed by --reps timed
b2s_groth16_prove_resident calls (wall clock; the call synchronises).  The medians, the witness-map kernels of one profiled
proof per reduction (b2s_profile_report) and a bit comparison of the two proofs are printed as one JSON line per case, then
b2s_groth16_prove_batch at 2^12 and 2^16 with K = 64 under each reduction (both keys resident, alternated).

  python tools/qap_probe.py [--curves 0 1] [--logs 16 20 24] [--rounds 3] [--reps 2] [--batch-logs 12 16] [--k 64]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

R = {0: 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
     1: 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001}
QAP = {"libsnark": 0, "circom": 1}
WM_KERNELS = ("spmv", "copy_instance", "qap_", "ntt_pass")


def mont(curve, xs):
    out = np.zeros((len(xs), 8), dtype=np.uint32)
    for i, x in enumerate(xs):
        v = x * (1 << 256) % R[curve]
        out[i] = [(v >> (32 * j)) & 0xFFFFFFFF for j in range(8)]
    return out.reshape(-1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def instance(curve, log_n, seed):
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


def wm_kernels(rep):
    return {k: round(v[1], 3) for k, v in sorted(rep.items()) if k.startswith(WM_KERNELS)}


def single(be, torch, curve, log_n, rounds, reps):
    rng = np.random.default_rng(log_n * 7 + curve)
    csr, n_rows, n_inst, n_wit, z = instance(curve, log_n, log_n)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    z_dev = torch.from_numpy(z.view(np.int32)).cuda()
    td = mont(curve, [int.from_bytes(rng.bytes(32), "little") % R[curve] or 1 for _ in range(5)])
    r, s = (mont(curve, [int.from_bytes(rng.bytes(32), "little") % R[curve]]) for _ in range(2))
    times = {q: [] for q in QAP}
    proofs, kernels = {}, {}
    for rnd in range(rounds):
        for name, qap in QAP.items():
            pk, _vk = be.groth16_setup(m, td, n_inst, qap=qap)
            be.groth16_prove_resident(pk, m, z_dev, r, s)             # warm-up
            for _ in range(reps):
                t0 = time.perf_counter()
                proofs[name] = be.groth16_prove_resident(pk, m, z_dev, r, s)
                times[name].append((time.perf_counter() - t0) * 1e3)
            if rnd == rounds - 1:
                be.profile(True)
                be.groth16_prove_resident(pk, m, z_dev, r, s)
                kernels[name] = wm_kernels(be.profile_report())
                be.profile(False)
            be.pk_free(pk)
    identical = all(np.array_equal(x, y) for x, y in zip(proofs["libsnark"], proofs["circom"]))
    be.r1cs_free(m)
    return {"ms_median": {q: round(statistics.median(v), 2) for q, v in times.items()},
            "ms_all": {q: [round(t, 2) for t in v] for q, v in times.items()}, "bit_identical": identical, "wm_kernels_ms": kernels}


def batch(be, torch, curve, log_n, K, reps):
    rng = np.random.default_rng(log_n * 11 + curve)
    csr, n_rows, n_inst, n_wit, z = instance(curve, log_n, log_n + 1)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    td = mont(curve, [int.from_bytes(rng.bytes(32), "little") % R[curve] or 1 for _ in range(5)])
    zs = torch.from_numpy(np.tile(z, (K, 1)).view(np.int32)).cuda()
    r = torch.from_numpy(mont(curve, [int.from_bytes(rng.bytes(32), "little") % R[curve] for _ in range(K)]).view(np.int32)).cuda()
    s = torch.from_numpy(mont(curve, [int.from_bytes(rng.bytes(32), "little") % R[curve] for _ in range(K)]).view(np.int32)).cuda()
    keys = {q: be.groth16_setup(m, td, n_inst, qap=v)[0] for q, v in QAP.items()}
    for pk in keys.values():
        be.groth16_prove_batch(pk, m, zs, r, s)                        # warm-up
    times, outs = {q: [] for q in QAP}, {}
    for _ in range(reps):
        for q, pk in keys.items():
            t0 = time.perf_counter()
            outs[q] = be.groth16_prove_batch(pk, m, zs, r, s)
            times[q].append(time.perf_counter() - t0)
    identical = all(torch.equal(x, y) for x, y in zip(outs["libsnark"], outs["circom"]))
    for pk in keys.values():
        be.pk_free(pk)
    be.r1cs_free(m)
    return {"proofs_per_s": {q: round(K / statistics.median(v), 1) for q, v in times.items()}, "bit_identical": identical}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", type=int, nargs="+", default=[0, 1])
    ap.add_argument("--logs", type=int, nargs="+", default=[16, 20, 24])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--batch-logs", type=int, nargs="+", default=[12, 16])
    ap.add_argument("--k", type=int, default=64)
    args = ap.parse_args()
    import torch

    from snark_b200 import Backend

    gpu = card()
    print(json.dumps({"gpu": gpu}), flush=True)
    for curve in args.curves:
        be = Backend(curve=curve)
        cname = ["bls12_381", "bn254"][curve]
        for log_n in args.logs:
            res = single(be, torch, curve, log_n, args.rounds, args.reps)
            print(json.dumps({"curve": cname, "log_n": log_n, "kind": "single", **res}), flush=True)
        for log_n in args.batch_logs:
            res = batch(be, torch, curve, log_n, args.k, args.rounds)
            print(json.dumps({"curve": cname, "log_n": log_n, "kind": "batch", "K": args.k, **res}), flush=True)
        be.close()


if __name__ == "__main__":
    main()
