"""Time the R1CS -> square R1CS conversion on the GPU, in one process, on BLS12-381:
  b2s_r1cs_to_sr1cs       host clock around the call (it synchronises before it returns)
  b2s_sr1cs_assignment    1 and 64 assignments resident on the device, CUDA events on the library's stream
  b2s_gr1cs_check         on the result, next to b2s_r1cs_check and b2s_spmv on the source (1 resident assignment, events)
for DummyCircuit-shaped systems (a*b = c, one empty row) of 2^20 and 2^24 rows and a BenchCircuit-shaped one of 2^20 rows
(tools/spmv_probe.bench_shaped_csr).  One warm-up call per path and size, then the median of --reps.
Byte model of the assignment kernel (its HBM share): per term of L row 2i+1 (A_i' - B_i') 12 B of column, coefficient id
and orig plus a 32 B gather of z; per new variable 4 B of orig and 32 B written, plus the 32 B read of each copied value.
For context only, --mirror times the C++ mirror's Sr1csAdapter::r1cs_to_sr1cs_with_assignment on the host at 2^16 and 2^20
(tests/native/host_sr1cs_dump, built by tests/test_sr1cs_oracle.py); that is the mirror's time, not ark's.
usage: python tools/sr1cs_probe.py [--reps 5] [--mirror]"""
import argparse
import ctypes
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.params import BLS12_381  # noqa: E402
from tools.spmv_probe import bench_shaped_csr  # noqa: E402
from tests.util import pack_fr  # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def dummy_csr(n):
    rp = np.arange(n + 1, dtype=np.uint64)
    rp[-1] = n - 1
    return [(rp, np.full(n - 1, c, dtype=np.uint32)) for c in (2, 3, 1)], 6, 2


def bench_csr(n):
    mats, n_vars = bench_shaped_csr(n, seed=1)
    return mats, n_vars, 1


def assign_bytes(info, m, nab):
    n_vars = info["n_instance"] + info["n_witness"]
    return nab * (12 + 32) + n_vars * (4 + 32) + (n_vars - m) * 32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mirror", action="store_true")
    a = ap.parse_args()
    if a.mirror:
        return mirror(a.reps)
    import torch

    from snark_b200 import Backend

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    curve = BLS12_381
    be = Backend(curve=0)
    lib = be.lib
    one = pack_fr(curve, [1])
    stream = ctypes.c_void_p(be.stream)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def events(fn, reps):
        fn()
        be.sync()
        ts = []
        for _ in range(reps):
            ev[0].record(torch.cuda.ExternalStream(stream.value))
            fn()
            ev[1].record(torch.cuda.ExternalStream(stream.value))
            ev[1].synchronize()
            ts.append(ev[0].elapsed_time(ev[1]) / 1e3)
        return float(np.median(ts))

    for name, log_n, make in (("dummy", 20, dummy_csr), ("dummy", 24, dummy_csr), ("bench", 20, bench_csr)):
        n = 1 << log_n
        mats, n_vars, n_inst = make(n)
        csr = [(rp, col, np.tile(one, len(col))) for rp, col in mats]
        m = be.r1cs_upload(n, n_inst, n_vars - n_inst, csr)
        nab = int(mats[0][0][-1]) + int(mats[1][0][-1])
        g = be.r1cs_to_sr1cs(m)
        be.gr1cs_free(g)
        ts = []
        for _ in range(a.reps):
            t0 = time.perf_counter()
            g = be.r1cs_to_sr1cs(m)
            ts.append(time.perf_counter() - t0)
            be.gr1cs_free(g)
        t_conv = float(np.median(ts))
        g = be.r1cs_to_sr1cs(m)
        info = be.gr1cs_info(g)
        nv2 = g.n_vars
        row = {"shape": f"{name} 2^{log_n}", "to_sr1cs_ms": 1e3 * t_conv}
        rng = np.random.default_rng(log_n)
        for k in (1, 64):
            z = rng.integers(0, 1 << 32, size=(k, n_vars, 8), dtype=np.uint32)
            z[:, :, 7] &= 0x0FFFFFFF
            zt = torch.from_numpy(z.reshape(k, -1).view(np.int32)).cuda()
            out = torch.zeros((k, 8 * nv2), dtype=torch.int32, device="cuda")
            torch.cuda.synchronize()
            t = events(lambda: lib.b2s_sr1cs_assignment(be.h, g.h, k, zt.data_ptr(), 1, out.data_ptr()), a.reps)
            byts = k * assign_bytes(info, n, nab)
            row[f"assign{k}_ms"] = 1e3 * t
            row[f"assign{k}_hbm_share"] = byts / t / HBM_PEAK
            if k == 1:
                z1, z2 = zt, out
            else:
                del zt, out
        first = torch.zeros(2, dtype=torch.int64, device="cuda")
        cnt = torch.zeros(2, dtype=torch.int64, device="cuda")
        vec = torch.zeros((3, 8 * n), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        row["gr1cs_check_ms"] = 1e3 * events(lambda: lib.b2s_gr1cs_check(be.h, g.h, 1, z2.data_ptr(), 1, first.data_ptr(), cnt.data_ptr()), a.reps)
        row["r1cs_check_ms"] = 1e3 * events(lambda: lib.b2s_r1cs_check(be.h, m, 1, z1.data_ptr(), 1, first.data_ptr(), cnt.data_ptr()), a.reps)
        row["spmv_ms"] = 1e3 * events(lambda: lib.b2s_spmv(be.h, m, z1.data_ptr(), 1, vec[0].data_ptr(), vec[1].data_ptr(), vec[2].data_ptr()), a.reps)
        print(row, flush=True)
        del z1, z2, vec
        be.gr1cs_free(g)
        be.r1cs_free(m)
        torch.cuda.empty_cache()
    be.close()


def mirror(reps):
    """the C++ mirror's conversion of a DummyCircuit-shaped R1CS, timed inside the harness"""
    from tests.test_sr1cs_oracle import build

    exe = build()
    one = " ".join(f"{int(w):08x}" for w in pack_fr(BLS12_381, [1]))
    for log_n in (16, 20):
        n = 1 << log_n
        with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
            f.write(f"2 4 {n}\n" + "\n".join([one] * 5) + "\n")
            row = lambda c: f"1 {c} {one}"
            f.write((row(2) + "\n" + row(3) + "\n" + row(1) + "\n") * (n - 1) + "0\n0\n0\n")
        ts = []
        for _ in range(reps):
            out = subprocess.run([exe, "0", f.name, "time"], capture_output=True, text=True, check=True).stdout
            ts.append(float(out.split()[1]))
        os.unlink(f.name)
        print({"mirror_2^%d_s" % log_n: float(np.median(ts))}, flush=True)


if __name__ == "__main__":
    main()
