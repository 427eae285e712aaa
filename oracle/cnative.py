"""ctypes wrapper of the C++ oracle (oracle/c/oracle.cpp).  TEST INFRASTRUCTURE ONLY (checker for
mid-size parity tests; CPU baseline of bench.py).  Buffers use the C-ABI layout of include/b200snark.h."""
import ctypes
import os
import subprocess
from ctypes import POINTER, c_int, c_uint64, c_void_p

import numpy as np

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "c")
_lib = None


def load(build=True):
    global _lib
    if _lib is None:
        so = os.path.join(_DIR, "liboracle.so")
        src = os.path.join(_DIR, "oracle.cpp")
        if build and (not os.path.exists(so) or os.path.getmtime(src) > os.path.getmtime(so)):
            subprocess.check_call(["make", "-s", "-C", _DIR])
        lib = ctypes.CDLL(so)
        lib.orc_threads_default.restype = c_int
        lib.orc_msm.argtypes = [c_int, c_int, c_void_p, c_void_p, c_uint64, c_int, c_int, c_void_p]
        lib.orc_ntt.argtypes = [c_int, c_void_p, c_int, c_int, c_int, c_int]
        lib.orc_spmv.argtypes = [c_int, c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p, c_int]
        lib.orc_groth16_prove.argtypes = [c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), c_uint64, c_uint64,
                                          c_uint64, POINTER(c_void_p)] + [c_void_p] * 8 + [c_int]
        lib.orc_witness_map.argtypes = [c_int, POINTER(c_void_p), POINTER(c_void_p), POINTER(c_void_p), c_uint64, c_uint64, c_void_p, c_int,
                                        c_void_p, c_int]
        lib.orc_witness_map_circom.argtypes = lib.orc_witness_map.argtypes
        lib.orc_multiples.argtypes = [c_int, c_int, c_void_p, c_uint64, c_uint64, c_void_p, c_int]
        lib.orc_fr_dot.argtypes = [c_int, c_void_p, c_void_p, c_uint64, c_void_p]
        _lib = lib
    return _lib


def threads_default():
    """Host threads the CPU baseline may actually use: min(visible CPUs, scheduler affinity, cgroup CPU quota).
    (The GPU boxes show 128 CPUs but cap the container at 16 via cpu.max; oversubscribing is slower.)"""
    n = min(load().orc_threads_default(), len(os.sched_getaffinity(0)))
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = max(1, min(n, int(quota) // int(period)))
    except (OSError, ValueError):
        pass
    return n


def _p(a):
    return a.ctypes.data if a is not None else None


FQ_WORDS = {0: 12, 1: 8, 2: 12}   # 32-bit words of one Fq element: BLS12-381, BN254, BLS12-377


def msm(curve_id, group, bases, scalars, n, mont=True, threads=None):
    fq = FQ_WORDS[curve_id]
    out = np.zeros(2 * group * fq, dtype=np.uint32)
    rc = load().orc_msm(curve_id, group, _p(bases), _p(scalars), n, int(mont), threads or threads_default(), _p(out))
    assert rc == 0
    return out


def ntt(curve_id, data, log_n, inverse=False, coset=False, threads=None):
    rc = load().orc_ntt(curve_id, _p(data), log_n, int(inverse), int(coset), threads or threads_default())
    assert rc == 0
    return data


def spmv(curve_id, csr, z, n_rows, threads=None):
    out = np.zeros(n_rows * 8, dtype=np.uint32)
    rc = load().orc_spmv(curve_id, _p(csr[0]), _p(csr[1]), _p(csr[2]), n_rows, _p(z), _p(out), threads or threads_default())
    assert rc == 0
    return out


def groth16_prove(curve_id, csr3, n_rows, n_inst, n_wit, pk_arrays, z_inst, z_wit, r, s, want_h=False, threads=None):
    """pk_arrays: [alpha_g1, beta_g1, delta_g1, beta_g2, delta_g2, a_query, b_g1_query, b_g2_query, h_query, l_query]."""
    fq = FQ_WORDS[curve_id]
    rp = (c_void_p * 3)(*[_p(m[0]) for m in csr3])
    col = (c_void_p * 3)(*[_p(m[1]) for m in csr3])
    co = (c_void_p * 3)(*[_p(m[2]) for m in csr3])
    pk = (c_void_p * 10)(*[_p(a) for a in pk_arrays])
    a = np.zeros(2 * fq, dtype=np.uint32)
    b = np.zeros(4 * fq, dtype=np.uint32)
    c = np.zeros(2 * fq, dtype=np.uint32)
    need = n_rows + n_inst
    dom = 1 << max((need - 1).bit_length(), 0)
    h = np.zeros(dom * 8, dtype=np.uint32) if want_h else None
    rc = load().orc_groth16_prove(curve_id, rp, col, co, n_rows, n_inst, n_wit, pk, _p(z_inst), _p(z_wit), _p(r), _p(s),
                                  _p(a), _p(b), _p(c), _p(h), threads or threads_default())
    assert rc == 0
    return a, b, c, h


def _witness_map(fn, curve_id, csr3, n_rows, n_inst, z, threads):
    rp = (c_void_p * 3)(*[_p(m[0]) for m in csr3])
    col = (c_void_p * 3)(*[_p(m[1]) for m in csr3])
    co = (c_void_p * 3)(*[_p(m[2]) for m in csr3])
    log_dom = max((n_rows + n_inst - 1).bit_length(), 0)
    h = np.zeros((1 << log_dom) * 8, dtype=np.uint32)
    rc = fn(curve_id, rp, col, co, n_rows, n_inst, _p(z), log_dom, _p(h), threads or threads_default())
    assert rc == 0
    return h


def witness_map(curve_id, csr3, n_rows, n_inst, z, threads=None):
    """h of the LibsnarkReduction (SURVEY App. A.2) for z = instance || witness; domain = next_pow2(n_rows + n_inst)."""
    return _witness_map(load().orc_witness_map, curve_id, csr3, n_rows, n_inst, z, threads)


def witness_map_circom(curve_id, csr3, n_rows, n_inst, z, threads=None):
    """h of the CircomReduction (DESIGN.md §3.6): N evaluations on the odd coset w2 H, same arguments and domain."""
    return _witness_map(load().orc_witness_map_circom, curve_id, csr3, n_rows, n_inst, z, threads)


def multiples(curve_id, group, gen, start, n, threads=None):
    fq = FQ_WORDS[curve_id]
    out = np.zeros(n * 2 * group * fq, dtype=np.uint32)
    rc = load().orc_multiples(curve_id, group, _p(gen), start, n, _p(out), threads or threads_default())
    assert rc == 0
    return out


def fr_dot(curve_id, a, b, n):
    out = np.zeros(8, dtype=np.uint32)
    assert load().orc_fr_dot(curve_id, _p(a), _p(b), n, _p(out)) == 0
    return out
