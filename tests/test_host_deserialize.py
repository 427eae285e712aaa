"""The point decoder of the load path (snark_b200/csrc/deserialize.cuh), compiled for the host, against the oracle's
CanonicalDeserialize (tests/wire_oracle.py): valid encodings, every rejection class, and above all the subgroup verdict
on points outside the prime-order subgroup, where the decoder's endomorphism criteria must agree with r * P = O."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from tests import wire_oracle as oser
from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests.util import pack_points, unpack_points

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = [BLS12_381, BN254]
STATUS = {0: None, 1: oser.REASON_FLAGS, 2: oser.REASON_NONCANONICAL, 3: oser.REASON_NOT_ON_CURVE, 4: oser.REASON_NOT_IN_SUBGROUP}


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostdec") / "libhostdec.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "host_deserialize.cpp")])
    return ctypes.CDLL(so)


def decode(lib, curve, group, blobs, compressed, validate):
    """-> list of (point or None, oracle-style reason or None) per encoding"""
    fq = 48 if curve is BLS12_381 else 32
    data = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
    out = np.zeros(len(blobs) * 2 * group * fq // 4, dtype=np.uint32)
    st = np.zeros(len(blobs), dtype=np.uint32)
    lib.ht_point_decode(curve.curve_id, group, data.ctypes.data_as(ctypes.c_void_p), int(compressed), int(validate),
                        out.ctypes.data_as(ctypes.c_void_p), st.ctypes.data_as(ctypes.c_void_p), len(blobs))
    pts = unpack_points(curve, group, out)
    return [(pts[i] if st[i] == 0 else None, STATUS[int(st[i])]) for i in range(len(blobs))]


def oracle(curve, group, blob, compressed, validate):
    try:
        return oser.point_deserialize(curve, group, blob, compressed, validate), None
    except ValueError as e:
        return None, str(e)


def encode(curve, group, P, compressed):
    return (oser.point_compressed if compressed else oser.point_uncompressed)(curve, group, P)


def agree(lib, curve, group, blobs, compressed, validate):
    got = decode(lib, curve, group, blobs, compressed, validate)
    exp = [oracle(curve, group, b, compressed, validate) for b in blobs]
    for i, (g, e) in enumerate(zip(got, exp)):
        assert g == e, (curve.name, group, compressed, validate, i, blobs[i].hex())
    return got


PARAMS = [(c, g, comp) for c in (0, 1) for g in (1, 2) for comp in (True, False)]
IDS = [f"{CURVES[c].name}-g{g}-{'c' if comp else 'u'}" for c, g, comp in PARAMS]


@pytest.mark.parametrize("ci,group,compressed", PARAMS, ids=IDS)
def test_valid_encodings(lib, ci, group, compressed):
    curve = CURVES[ci]
    G = groups(curve)[group - 1]
    rng = random.Random(100 + 4 * ci + 2 * group + compressed)
    pts = [G.gen, G.neg(G.gen), None] + [G.mul(G.gen, rng.randrange(1, curve.r)) for _ in range(200 if group == 1 else 60)]
    blobs = [encode(curve, group, P, compressed) for P in pts]
    for validate in (True, False):
        got = agree(lib, curve, group, blobs, compressed, validate)
        assert [g[0] for g in got] == pts


def flip(blob, at, bits):
    b = bytearray(blob)
    b[at] ^= bits
    return bytes(b)


def malformed(curve, group, compressed, rng):
    """one encoding of each rejection class the decoder must agree on"""
    G = groups(curve)[group - 1]
    fq = 48 if curve is BLS12_381 else 32
    P = G.mul(G.gen, rng.randrange(1, curve.r))
    good, inf = encode(curve, group, P, compressed), encode(curve, group, None, compressed)
    n = len(good)
    out = []
    if curve is BLS12_381:
        out += [flip(good, 0, 0x80), flip(inf, 0, 0x80), flip(inf, 0, 0x20), flip(inf, n - 1, 0x01), flip(good, 0, 0x40)]
        if not compressed:
            out += [flip(good, 0, 0x20)]
        first = lambda v: v.to_bytes(fq, "big")   # x, or x.c1 for G2, written first
        over = bytes([good[0] & 0xE0 | first(curve.p)[0]]) + first(curve.p)[1:] + good[fq:]
        out += [over]
        if group == 2:   # x.c0 >= p (second component)
            out += [good[:fq] + curve.p.to_bytes(fq, "big") + good[2 * fq:]]
    else:
        fl = n - 1
        out += [bytes(good[:fl]) + bytes([good[fl] | 0xC0]), flip(inf, 0, 0x01), bytes(inf[:fl]) + bytes([0xC0])]
        out += [curve.p.to_bytes(fq, "little") + good[fq:]]
        if group == 2:
            c1 = curve.p.to_bytes(fq, "little")
            out += [good[:fq] + c1[:-1] + bytes([c1[-1] | (good[2 * fq - 1] & 0xC0 if compressed else 0)]) + good[2 * fq:]]
    # x not on the curve: a compressed x without a root; an uncompressed y off the curve
    while True:
        x = rng.randrange(curve.p) if group == 1 else (rng.randrange(curve.p), rng.randrange(curve.p))
        f = G.f
        rhs = f.add(f.mul(f.sqr(x), x), G.b)
        if (oser._sqrt_fq(curve.p, rhs) if group == 1 else oser._sqrt_fq2(curve.p, rhs)) is None:
            break
    y = P[1]
    bad = encode(curve, group, (x, y), compressed)
    out += [bad]
    if not compressed:
        out += [encode(curve, group, (P[0], f.add(P[1], f.one)), False)]
    return out


@pytest.mark.parametrize("ci,group,compressed", PARAMS, ids=IDS)
def test_rejections(lib, ci, group, compressed):
    curve = CURVES[ci]
    rng = random.Random(200 + 4 * ci + 2 * group + compressed)
    blobs = malformed(curve, group, compressed, rng)
    for validate in (True, False):
        got = agree(lib, curve, group, blobs, compressed, validate)
        if validate or compressed:
            assert all(r is not None for _, r in got), got
    # reason classes are all exercised
    reasons = {r for _, r in decode(lib, curve, group, blobs, compressed, True)}
    assert {oser.REASON_FLAGS, oser.REASON_NONCANONICAL, oser.REASON_NOT_ON_CURVE} <= reasons


@pytest.mark.parametrize("ci,group,compressed", PARAMS, ids=IDS)
def test_subgroup_verdict_matches_definition(lib, ci, group, compressed):
    """Random-x points, P + T torsion points (rejected with validate, accepted without) and cofactor-cleared points
    (accepted): the endomorphism criterion gives the verdict of r * P = O."""
    curve = CURVES[ci]
    G = groups(curve)[group - 1]
    rng = random.Random(300 + 4 * ci + 2 * group + compressed)
    off = oser.points_outside_subgroup(curve, group, rng, 24)
    h = oser.cofactor(curve, group)
    cleared = [oser.mul_unreduced(G, oser.random_curve_point(curve, group, rng), h) for _ in range(8)]
    pts = off + cleared
    blobs = [encode(curve, group, P, compressed) for P in pts]
    got = agree(lib, curve, group, blobs, compressed, True)
    assert [r for _, r in got] == [oser.REASON_NOT_IN_SUBGROUP] * len(off) + [None] * len(cleared)
    got = agree(lib, curve, group, blobs, compressed, False)
    assert [g[0] for g in got] == pts
    if h == 1:
        assert off == []
