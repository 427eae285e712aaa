"""Fp::inverse (divsteps, snark_b200/csrc/ff.cuh) compiled for the host through the field harnesses
(tests/native/host_ff.cpp for BLS12-381 and BN254, tests/native/host_bls377.cpp for BLS12-377), on all six fields:
random elements and the edge values of the limb and Montgomery representations against Python's pow(x, -1, p).
Runs without a GPU; tests/test_gpu_inverse.py runs the same checks on the device."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle.params import BLS12_381 as BLS, BN254 as BN
from tests import bls377_oracle as b7
from tests.util import pack_u32, ptr, unpack_u32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (name, p, 32-bit limbs, harness, field id in that harness)
FIELDS = [
    ("bls12_381_fq", BLS.p, 12, "ff", 0), ("bls12_381_fr", BLS.r, 8, "ff", 1),
    ("bn254_fq", BN.p, 8, "ff", 2), ("bn254_fr", BN.r, 8, "ff", 3),
    ("bls12_377_fq", b7.P, 12, "377", 0), ("bls12_377_fr", b7.R, 8, "377", 1),
]


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    d = tmp_path_factory.mktemp("hostinv")
    out = {}
    for key, src in (("ff", "host_ff.cpp"), ("377", "host_bls377.cpp")):
        so = str(d / ("lib%s.so" % key))
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                               os.path.join(ROOT, "tests", "native", src)])
        out[key] = ctypes.CDLL(so)
    return out


def edge_values(p, n):
    """0, 1, 2, p - 1, p - 2, (p - 1) / 2, R, R^2 (mod p), every power of two below p, and values just below p"""
    R = 1 << (32 * n)
    e = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R % p, R * R % p, R * R * R % p]
    e += [1 << k for k in range(p.bit_length())]
    e += [p - k for k in range(3, 40)] + [p - (1 << k) for k in range(1, p.bit_length() - 1)]
    e += [(1 << (32 * k)) - 1 for k in range(1, n) if (1 << (32 * k)) - 1 < p]
    e += [(1 << (30 * k)) % p for k in range(1, 14)] + [((1 << (30 * k)) - 1) % p for k in range(1, 14)]
    return e


def inverse(lib, harness, field, xs, n):
    a = pack_u32(xs, n)
    out = np.zeros_like(a)
    fn = lib.ht_field_op if harness == "ff" else lib.ht377_field_op
    fn(field, 3, ptr(a), ptr(a), ptr(out), len(xs))
    return unpack_u32(out, n)


@pytest.mark.parametrize("f", range(len(FIELDS)), ids=[x[0] for x in FIELDS])
def test_inverse_matches_bigint(libs, f):
    name, p, n, harness, field = FIELDS[f]
    R = 1 << (32 * n)
    Rinv = pow(R, -1, p)
    rng = random.Random(7000 + f)
    xs = edge_values(p, n) + [rng.randrange(p) for _ in range(20000)]
    got = inverse(libs[harness], harness, field, xs, n)
    # Montgomery form in and out: x R -> x^-1 R, and 0 -> 0
    exp = [pow(x * Rinv % p, -1, p) * R % p if x else 0 for x in xs]
    bad = [i for i in range(len(xs)) if got[i] != exp[i]]
    assert not bad, (name, len(bad), hex(xs[bad[0]]))
