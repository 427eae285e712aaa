"""Time instance outlining on the GPU, in one process, on BLS12-381:
  ingest      b2s_r1cs_upload_lcmap_outline against b2s_r1cs_upload_lcmap of the same LcMap (DummyCircuit-like, 2^20, 2^22
              and 2^24 outlined domain, tests/test_gpu_outline.dummy_lcmap), and b2s_gr1cs_upload_lcmap(_outline) of a planted
              GR1CS (tests/gr1cs_lcmap_gen.planted, 2^20 and 2^22 rows in each of two predicates); host clock around each call
              (both synchronise before they return), the two alternating, median of --reps after one warm-up each
  assignment  b2s_gr1cs_outline_assignment of 1 and 64 resident assignments of 2^22 variables, CUDA events on the library's
              stream, median of --reps.  Byte model: per assignment n_src * 32 B read and (n_src + n_instance) * 32 B written.
For context only, --mirror times the C++ mirror's finalize() with outline_r1cs on the host at 2^20 rows of the same shape
(tests/native/host_outline_dump, built by tests/test_outline_oracle.py); that is the mirror's time, not ark's.
usage: python tools/outline_probe.py [--reps 5] [--mirror]"""
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
from tests import outline_oracle as oo  # noqa: E402
from tests.gr1cs_lcmap_gen import planted  # noqa: E402
from tests.test_gpu_outline import dummy_lcmap, r1cs_handle  # noqa: E402
from tests.util import pack_fr  # noqa: E402

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def alternate(reps, calls, free):
    """median seconds of each call in `calls` (each returns a handle for free()): one warm-up each, then alternating"""
    ts = [[] for _ in calls]
    for i in range(reps + 1):
        for k, fn in enumerate(calls):
            t0 = time.perf_counter()
            h = fn()
            t = time.perf_counter() - t0
            free(h)
            if i:
                ts[k].append(t)
    return [float(np.median(t)) for t in ts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--mirror", action="store_true")
    a = ap.parse_args()
    if a.mirror:
        return mirror()
    import torch

    from snark_b200 import Backend

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    curve = BLS12_381
    r = curve.r
    be = Backend(curve=0)
    n_inst, n_wit = 3, 4
    for log_n in (20, 22, 24):
        lm, _ = dummy_lcmap(curve, (1 << log_n) - 2 * n_inst)
        tp, to = alternate(a.reps, [lambda ol=ol: r1cs_handle(be, curve, lm, n_inst, n_wit, outline=ol) for ol in (False, True)], be.r1cs_free)
        print({"ingest": f"r1cs dummy 2^{log_n}", "plain_ms": 1e3 * tp, "outlined_ms": 1e3 * to, "ratio": to / tp}, flush=True)
    for log_n in (20, 22):
        preds, lm = planted(r, {"P2": (2, 1 << log_n), "P3": (3, 1 << log_n)}, 5, 1 << 12, seed=log_n)
        preds["R1CS"] = (3, oo.r1cs_terms(r))
        lm["args"]["R1CS"] = [np.zeros(0, np.uint64)] * 3
        tp, to = alternate(a.reps, [lambda ol=ol: be.gr1cs_upload_lcmap(5, 1 << 12, preds, lm, outline=ol)
                                    for ol in (None, (oo.OUTLINE_R1CS, "R1CS"))], be.gr1cs_free)
        print({"ingest": f"gr1cs planted 2x2^{log_n}", "plain_ms": 1e3 * tp, "outlined_ms": 1e3 * to, "ratio": to / tp}, flush=True)

    # the assignment conversion: 2^22 variables, an outlined GR1CS handle of a tiny planted system over them
    n_src = 1 << 22
    preds, lm = planted(r, {"P2": (2, 1 << 10)}, 8, n_src - 8, seed=1)
    g = be.gr1cs_upload_lcmap(8, n_src - 8, preds, lm, outline=(oo.OUTLINE_SR1CS, "P2"))
    stream = torch.cuda.ExternalStream(ctypes.c_void_p(be.stream).value)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for k in (1, 64):
        z = torch.randint(0, 1 << 28, (k, 8 * n_src), dtype=torch.int32, device="cuda")
        out = torch.zeros((k, 8 * g.n_vars), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        call = lambda: be.lib.b2s_gr1cs_outline_assignment(be.h, g.h, k, z.data_ptr(), 1, out.data_ptr())
        call()
        be.sync()
        ts = []
        for _ in range(a.reps):
            ev[0].record(stream)
            call()
            ev[1].record(stream)
            ev[1].synchronize()
            ts.append(ev[0].elapsed_time(ev[1]) / 1e3)
        t = float(np.median(ts))
        byts = k * (n_src + g.n_vars) * 32
        print({"assign": f"x{k}, 2^22 variables", "ms": 1e3 * t, "hbm_share": byts / t / HBM_PEAK}, flush=True)
        del z, out
        torch.cuda.empty_cache()
    be.gr1cs_free(g)
    be.close()


def mirror():
    """the C++ mirror's finalize() with outline_r1cs on a 2^20-row system of dummy_lcmap's shape, timed inside the harness"""
    from tests.test_outline_oracle import build

    exe = build()
    curve = BLS12_381
    w = lambda v: " ".join(f"{int(x):08x}" for x in pack_fr(curve, [v]))
    one, two, m1 = w(1), w(2), w(curve.r - 1)
    n = 1 << 20
    even = f"R\n2 2 1 {one} 1 0 {two}\n1 3 1 {one}\n3 3 2 {one} 2 2 {one} 2 2 {m1}\n"
    odd = f"R\n1 3 0 {one}\n1 2 2 {one}\n2 3 3 {two} 3 3 {m1}\n"
    with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
        f.write(f"1 3 4 {n}\n" + "\n".join(w(v) for v in (7, 9, 3, 5, 45, 27)) + "\n")
        f.write((even + odd) * (n // 2))
    out = subprocess.run([exe, "0", f.name, "time"], capture_output=True, text=True, timeout=3600)
    os.unlink(f.name)
    print(f"mirror finalize() with outline_r1cs, 2^20 rows: {out.stdout.strip()}", flush=True)


if __name__ == "__main__":
    main()
