"""Time the two LcMap ingests against the uploads of the equivalent prebuilt CSR (what to_matrices() exports), on the GPU:
  b2s_gr1cs_upload_lcmap  vs  b2s_gr1cs_upload   three predicates of arity 2, 3 and 5 (1/2, 1/4, 1/4 of the constraints)
  b2s_r1cs_upload_lcmap   vs  b2s_r1cs_upload    one R1CS of the same number of constraints
The systems are generated in numpy (tests/gr1cs_lcmap_gen.py: Zero, bare-variable and shared-LC arguments, argument 1 a fresh
LC of split coefficients), and both handles of each pair are checked to give the same first_unsat / n_unsat.  Each call is
timed with a host clock; every call synchronises before it returns.  One warm-up call per path and size, then the median of
--reps.  The host cost of the reference's to_matrices() (Rust) is not measured here.
usage: python tools/gr1cs_lcmap_probe.py [--log-n 20 22 24] [--reps 3]"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.params import BLS12_381  # noqa: E402
from snark_b200 import Backend  # noqa: E402
from snark_b200 import lib as L  # noqa: E402
from tests.gr1cs_lcmap_gen import csr_of, planted, random_z  # noqa: E402
from tests.util import pack_fr  # noqa: E402

N_INST = 5


def timed(fn, free, reps):
    fn_h = fn()
    free(fn_h)                       # warm-up
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        h = fn()
        ts.append(time.perf_counter() - t0)
        if _ < reps - 1:
            free(h)
    return float(np.median(ts)), h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, nargs="+", default=[20, 22, 24])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}", flush=True)
    curve = BLS12_381
    be = Backend(curve=0)
    ok = True
    for log_n in a.log_n:
        N = 1 << log_n
        n_wit = N // 4
        # ---- GR1CS: three predicates
        shape = {"p2": (2, N // 2), "p3": (3, N // 4), "p5": (5, N // 4)}
        t0 = time.perf_counter()
        preds, lm = planted(curve.r, shape, N_INST, n_wit, seed=log_n, bad={"p3": [N // 8]})
        pool = pack_fr(curve, lm["pool"]).reshape(-1, 8)
        keep = []
        lc_descs = (L.PredicateLcmapDesc * 3)()
        m_descs = (L.PredicateDesc * 3)()
        nnz = 0
        for dl, dm, label in zip(lc_descs, m_descs, sorted(shape)):
            arity, terms = preds[label]
            co = pack_fr(curve, [c for c, _ in terms])
            offs = np.arange(len(terms) + 1, dtype=np.uint32)
            fv = np.array([m[0][0] for _, m in terms], dtype=np.uint32)
            fp = np.ones(len(terms), dtype=np.uint32)
            keep += [co, offs, fv, fp]
            for d in (dl, dm):
                d.arity, d.n_terms, d.n_rows = arity, len(terms), shape[label][1]
                d.term_coeffs, d.term_offsets, d.factor_var, d.factor_pow = co.ctypes.data, offs.ctypes.data, fv.ctypes.data, fp.ctypes.data
            for j, arg in enumerate(lm["args"][label]):
                rp, col, ids = csr_of(lm, N_INST, arg)
                limbs = np.ascontiguousarray(pool[ids])
                nnz += len(col)
                keep += [arg, rp, col, limbs]
                dl.args[j] = arg.ctypes.data
                dm.row_ptr[j], dm.col[j], dm.coeff[j] = rp.ctypes.data, col.ctypes.data, limbs.ctypes.data
        pool_flat = pool.reshape(-1)
        n_lcs = len(lm["offsets"]) - 1
        gen_s = time.perf_counter() - t0

        def up_lc():
            h = ctypes.c_void_p()
            be._ck(be.lib.b2s_gr1cs_upload_lcmap(be.h, N_INST, n_wit, 3, lc_descs, n_lcs, lm["offsets"].ctypes.data, lm["vars"].ctypes.data,
                                                 lm["coeffs"].ctypes.data, pool_flat.ctypes.data, len(pool), ctypes.byref(h)))
            return h

        def up_m():
            h = ctypes.c_void_p()
            be._ck(be.lib.b2s_gr1cs_upload(be.h, N_INST, n_wit, 3, m_descs, ctypes.byref(h)))
            return h

        free_g = lambda h: be.lib.b2s_gr1cs_free(be.h, h)
        t_lc, g_lc = timed(up_lc, free_g, a.reps)
        t_m, g_m = timed(up_m, free_g, a.reps)
        z = random_z(1, N_INST + n_wit, seed=1)
        r_lc = be.gr1cs_check(L.Gr1cs(g_lc, sorted(shape), N_INST + n_wit), z)
        r_m = be.gr1cs_check(L.Gr1cs(g_m, sorted(shape), N_INST + n_wit), z)
        same = all(np.array_equal(x, y) for x, y in zip(r_lc, r_m)) and r_lc[0][0].tolist() == [L.NOT_FOUND, N // 8, L.NOT_FOUND]
        ok &= same
        free_g(g_lc)
        free_g(g_m)
        print(f"gr1cs 2^{log_n} constraints (arity 2/3/5), {len(lm['vars'])} LcMap terms, {nnz} nonzeros: "
              f"upload_lcmap {t_lc * 1e3:.1f} ms, upload of the CSR {t_m * 1e3:.1f} ms, ratio {t_m / t_lc:.2f}x, "
              f"same verdicts {same} (numpy generation {gen_s:.1f} s)", flush=True)
        del keep, lm, lc_descs, m_descs

        # ---- R1CS: one predicate of N constraints
        t0 = time.perf_counter()
        _, lm = planted(curve.r, {"r": (3, N)}, N_INST, n_wit, seed=100 + log_n)
        args = lm["args"]["r"]
        csr = []
        for arg in args:
            rp, col, ids = csr_of(lm, N_INST, arg)
            csr.append((rp, col, np.ascontiguousarray(pool[ids])))
        nnz = sum(len(c[1]) for c in csr)
        pool_flat = pack_fr(curve, lm["pool"])
        gen_s = time.perf_counter() - t0
        up_lc = lambda: be.r1cs_upload_lcmap(N, N_INST, n_wit, args, lm["offsets"], lm["vars"], lm["coeffs"], pool_flat)
        up_m = lambda: be.r1cs_upload(N, N_INST, n_wit, csr)
        t_lc, m_lc = timed(up_lc, be.r1cs_free, a.reps)
        t_m, m_m = timed(up_m, be.r1cs_free, a.reps)
        z = random_z(1, N_INST + n_wit, seed=2)
        same = all(np.array_equal(x, y) for x, y in zip(be.r1cs_check(m_lc, z), be.r1cs_check(m_m, z)))
        ok &= same
        be.r1cs_free(m_lc)
        be.r1cs_free(m_m)
        print(f"r1cs  2^{log_n} constraints, {len(lm['vars'])} LcMap terms, {nnz} nonzeros: upload_lcmap {t_lc * 1e3:.1f} ms, "
              f"upload of the CSR {t_m * 1e3:.1f} ms, ratio {t_m / t_lc:.2f}x, same verdicts {same} (numpy generation {gen_s:.1f} s)",
              flush=True)
        del csr, lm, args
    be.close()
    print("GR1CS LCMAP PROBE", "OK" if ok else "FAILED")
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
