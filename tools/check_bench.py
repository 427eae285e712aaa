"""Constraint-satisfaction check on the GPU: b2s_r1cs_check / b2s_gr1cs_check against the SpMV that reads the same CSR and the
proof it would guard.  Needs an H100.

Per curve:
  - b2s_r1cs_check on a DummyCircuit-shaped handle (every row z[2] * z[3] = z[1], one term per row) at 2^20 and 2^24 rows and on
    a BenchCircuit-shaped one (tools/spmv_probe.py) at 2^20, z resident on the device, alternated in the same process with
    b2s_spmv on the same handle; then b2s_groth16_prove_resident at the DummyCircuit sizes under a key from the GPU setup;
  - b2s_gr1cs_check of K = 16 / 64 / 256 resident assignments on a 2^16-row DummyCircuit-shaped R1CS predicate.
Each figure is the median over --reps calls of the kernel time (b2s_profile_report) and of the wall time of the call.  Bytes
are what the kernel must move: 4 B column + 4 B coefficient id + 32 B of z per nonzero, plus the row pointers (8 B per row and
argument); SpMV also writes 32 B per row and matrix.  GB/s and the share of the H100's 3.35 TB/s follow from the kernel time.
The card and its power limit are read in the same run.  No CPU is_satisfied baseline exists at these sizes, so no speed-up
over the CPU is claimed.  One JSON line per case.

  python tools/check_bench.py [--curves 0 1] [--logs 20 24] [--bench-log 20] [--reps 5] [--no-prove]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from spmv_probe import bench_shaped_csr  # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM5 80 GB HBM3
R = {0: 0x73EDA753299D7D483339D80809A1D80553BDA402FFFE5BFEFFFFFFFF00000001,
     1: 0x30644E72E131A029B85045B68181585D2833E84879B9709143E1F593F0000001}


def mont(curve, xs):
    out = np.zeros((len(xs), 8), dtype=np.uint32)
    for i, x in enumerate(xs):
        v = x * (1 << 256) % R[curve]
        out[i] = [(v >> (32 * j)) & 0xFFFFFFFF for j in range(8)]
    return out.reshape(-1)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def dummy(curve, n_rows):
    """DummyCircuit-shaped CSR (z[2] z[3] = z[1] on every row but the last, which is empty) and a satisfying z"""
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    ones = np.tile(mont(curve, [1]), nnz)
    csr = [(row_ptr, np.full(nnz, c, dtype=np.uint32), ones) for c in (2, 3, 1)]
    n_inst, n_wit = 2, n_rows - 1
    a, b = 0x1234567 % R[curve], 0x7654321 % R[curve]
    z = np.concatenate([mont(curve, [1, a * b % R[curve], a, b]), np.tile(mont(curve, [a]), n_inst + n_wit - 4)])
    return csr, n_inst, n_wit, z


def bench_shape(curve, n_rows):
    mats, n_wit = bench_shaped_csr(n_rows)
    one = mont(curve, [1])
    csr = [(rp, col, np.tile(one, len(col))) for rp, col in mats]
    z = np.random.default_rng(1).integers(0, 1 << 30, (1 + n_wit) * 8, dtype=np.int64).astype(np.uint32)   # canonical-range limbs
    return csr, 1, n_wit, z


def check_bytes(csr, n_rows, n_args):
    return 40 * sum(len(c[1]) for c in csr) + 8 * (n_rows + 1) * n_args


def kernel_ms(be, prefix):
    rep = be.profile_report()
    return sum(ms for k, (cnt, ms) in rep.items() if k.startswith(prefix))


def timed(be, fn, prefix):
    """(kernel ms, wall ms) of one call"""
    be.profile(True)
    t0 = time.perf_counter()
    fn()
    be.sync()
    wall = (time.perf_counter() - t0) * 1e3
    be.profile(False)
    return kernel_ms(be, prefix), wall


def med(xs):
    return round(statistics.median(xs), 4)


def bw(nbytes, ms):
    gbs = nbytes / (ms * 1e-3) / 1e9
    return round(gbs, 1), round(gbs * 1e9 / HBM_PEAK, 3)


def r1cs_case(be, torch, curve, shape, log_n, reps, prove, gpu):
    n_rows = (1 << log_n) - 2
    csr, n_inst, n_wit, z = (dummy if shape == "dummy" else bench_shape)(curve, n_rows)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    nb = check_bytes(csr, n_rows, 3)
    zd = torch.from_numpy(z.view(np.int32)).cuda()
    first = torch.zeros(2, dtype=torch.int64, device="cuda")
    outs = torch.empty((3, n_rows, 8), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    check = lambda: be._ck(be.lib.b2s_r1cs_check(be.h, m, 1, zd.data_ptr(), 1, first.data_ptr(), first.data_ptr() + 8))
    spmv = lambda: be._ck(be.lib.b2s_spmv(be.h, m, zd.data_ptr(), 1, *[outs[k].data_ptr() for k in range(3)]))
    check()
    spmv()
    ck, sp = [], []
    for _ in range(reps):   # alternated
        ck.append(timed(be, check, "gr1cs_check_kernel"))
        sp.append(timed(be, spmv, "spmv_kernel"))
    res = {"case": "r1cs_check", "curve": curve, "shape": shape, "log_n": log_n, "rows": n_rows,
           "nnz": sum(len(c[1]) for c in csr), "n_unsat": int(first[1].item()), "card": gpu,
           "check_kernel_ms": med([k for k, _ in ck]), "check_call_ms": med([w for _, w in ck]),
           "spmv_kernel_ms": med([k for k, _ in sp]), "spmv_call_ms": med([w for _, w in sp]), "check_bytes": nb,
           "spmv_bytes": nb + 3 * 32 * n_rows}
    res["check_GBps"], res["check_hbm_share"] = bw(nb, res["check_kernel_ms"])
    res["spmv_GBps"], res["spmv_hbm_share"] = bw(res["spmv_bytes"], res["spmv_kernel_ms"])
    del outs
    if prove and shape == "dummy":
        rng = np.random.default_rng(log_n)
        td = mont(curve, [int(x) for x in rng.integers(1, 1 << 62, 5)])
        pkh, _vk = be.groth16_setup(m, td, n_inst)
        r, s = mont(curve, [5]), mont(curve, [7])
        be.groth16_prove_resident(pkh, m, zd, r, s)
        pw = []
        for _ in range(reps):
            t0 = time.perf_counter()
            be.groth16_prove_resident(pkh, m, zd, r, s)
            pw.append((time.perf_counter() - t0) * 1e3)
        res["prove_ms"] = med(pw)
        res["check_share_of_proof"] = round(res["check_call_ms"] / res["prove_ms"], 4)
        be.pk_free(pkh)
    be.r1cs_free(m)
    return res


def gr1cs_case(be, torch, curve, log_n, K, reps, gpu):
    from snark_b200.lib import PredicateDesc

    n_rows = (1 << log_n) - 2
    csr, n_inst, n_wit, z = dummy(curve, n_rows)
    d = PredicateDesc()
    co = mont(curve, [1, R[curve] - 1])
    arrs = [co, np.array([0, 2, 3], dtype=np.uint32), np.array([0, 1, 2], dtype=np.uint32), np.ones(3, dtype=np.uint32)]
    d.arity, d.n_terms, d.n_rows = 3, 2, n_rows
    d.term_coeffs, d.term_offsets, d.factor_var, d.factor_pow = (a.ctypes.data for a in arrs)
    for j in range(3):
        d.row_ptr[j], d.col[j], d.coeff[j] = (a.ctypes.data for a in csr[j])
    import ctypes

    h = ctypes.c_void_p()
    be._ck(be.lib.b2s_gr1cs_upload(be.h, n_inst, n_wit, 1, ctypes.byref(d), ctypes.byref(h)))
    zd = torch.from_numpy(np.tile(z, K).view(np.int32)).cuda()
    out = torch.zeros((2, K), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    call = lambda: be._ck(be.lib.b2s_gr1cs_check(be.h, h, K, zd.data_ptr(), 1, out[0].data_ptr(), out[1].data_ptr()))
    call()
    runs = [timed(be, call, "gr1cs_check_kernel") for _ in range(reps)]
    nb = K * check_bytes(csr, n_rows, 3)
    res = {"case": "gr1cs_check", "curve": curve, "log_n": log_n, "K": K, "rows": n_rows, "n_unsat": int(out[1].sum().item()),
           "card": gpu, "kernel_ms": med([k for k, _ in runs]), "call_ms": med([w for _, w in runs]), "bytes": nb}
    res["GBps"], res["hbm_share"] = bw(nb, res["kernel_ms"])
    res["assignments_per_s"] = round(K / (res["call_ms"] * 1e-3))
    be.lib.b2s_gr1cs_free(be.h, h)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", type=int, nargs="+", default=[0, 1])
    ap.add_argument("--logs", type=int, nargs="+", default=[20, 24])
    ap.add_argument("--bench-log", type=int, default=20)
    ap.add_argument("--gr1cs-log", type=int, default=16)
    ap.add_argument("--k", type=int, nargs="+", default=[16, 64, 256])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--no-prove", action="store_true")
    args = ap.parse_args()
    import torch

    from snark_b200 import Backend

    gpu = card()
    for curve in args.curves:
        be = Backend(curve=curve)
        for log_n in args.logs:
            print(json.dumps(r1cs_case(be, torch, curve, "dummy", log_n, args.reps, not args.no_prove, gpu)), flush=True)
        if args.bench_log:
            print(json.dumps(r1cs_case(be, torch, curve, "bench", args.bench_log, args.reps, False, gpu)), flush=True)
        for K in args.k:
            print(json.dumps(gr1cs_case(be, torch, curve, args.gr1cs_log, K, args.reps, gpu)), flush=True)
        be.close()


if __name__ == "__main__":
    main()
