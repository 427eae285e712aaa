"""Known answers of the test-side snarkjs writers (tests/zkey_oracle.py), on the CPU: the framing, the R^2 scaling of the
coefficients, the Montgomery form of the points, the input rows and the section sizes that follow from the dimensions."""
import struct

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests import zkey_oracle as zo
from tests.util import csr_from_rows, pack_fr, pack_points

CURVES = [BLS12_381, BN254]


def sections(data, magic, version):
    """parse the binfile framing back: {type: [bytes, ...]} in file order"""
    assert data[:4] == magic
    ver, n = struct.unpack_from("<II", data, 4)
    assert ver == version
    at, out = 12, {}
    for _ in range(n):
        t, size = struct.unpack_from("<IQ", data, at)
        at += 12
        out.setdefault(t, []).append(data[at : at + size])
        at += size
    assert at == len(data)
    return out


def toy_key(curve, n_public, n_vars, domain):
    """a key of the right shape: G1 / G2 generator multiples are not needed for the framing, any limbs do"""
    from oracle.ec import groups

    G1, G2 = groups(curve)
    g1 = lambda k: pack_points(curve, 1, [G1.mul(G1.gen, i + 1) for i in range(k)])
    g2 = lambda k: pack_points(curve, 2, [G2.mul(G2.gen, i + 1) for i in range(k)])
    return {"alpha_g1": g1(1), "beta_g1": g1(1), "delta_g1": g1(1), "beta_g2": g2(1), "gamma_g2": g2(1), "delta_g2": g2(1),
            "gamma_abc_g1": g1(n_public + 1), "a": g1(n_vars), "b_g1": g1(n_vars), "b_g2": g2(n_vars), "h": g1(domain),
            "l": g1(n_vars - n_public - 1)}


@pytest.mark.parametrize("curve", CURVES, ids=["bls12_381", "bn254"])
def test_zkey_known_answers(curve):
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    A, B, _ = cs.to_matrices()
    n_inst, n_wit = len(cs.instance_assignment), len(cs.witness_assignment)
    n_public, n_vars = n_inst - 1, n_inst + n_wit
    domain = 1
    while domain < len(A) + n_inst:
        domain *= 2
    key = toy_key(curve, n_public, n_vars, domain)
    data = zo.write_zkey(curve, key, csr_from_rows(curve, A), csr_from_rows(curve, B), n_public, domain)
    sec = sections(data, b"zkey", 1)
    assert sorted(sec) == list(range(1, 10)) and all(len(v) == 1 for v in sec.values())
    assert struct.unpack("<I", sec[1][0]) == (1,)
    n8q = 8 * curve.fq_limbs64
    g1, g2 = 2 * n8q, 4 * n8q
    h = sec[2][0]
    assert struct.unpack_from("<I", h, 0) == (n8q,) and int.from_bytes(h[4 : 4 + n8q], "little") == curve.p
    assert struct.unpack_from("<I", h, 4 + n8q) == (32,) and int.from_bytes(h[8 + n8q : 40 + n8q], "little") == curve.r
    assert struct.unpack_from("<III", h, 40 + n8q) == (n_vars, n_public, domain)
    assert len(h) == 52 + n8q + 3 * g1 + 3 * g2
    # a point is x R mod q, y R mod q, little-endian: alpha1 is the generator
    from oracle.ec import groups

    G1 = groups(curve)[0]
    x = int.from_bytes(h[52 + n8q : 52 + 2 * n8q], "little")
    assert x == G1.gen[0] * (1 << (8 * n8q)) % curve.p
    # section sizes from the dimensions
    assert [len(sec[t][0]) for t in (3, 5, 6, 7, 8, 9)] == [(n_public + 1) * g1, n_vars * g1, n_vars * g1, n_vars * g2,
                                                            (n_vars - n_public - 1) * g1, domain * g1]
    # coefficients: count, then (matrix, constraint, signal, c R^2 mod r); the input rows close the section
    co = sec[4][0]
    (count,) = struct.unpack_from("<I", co, 0)
    nnz = sum(len(r) for r in A) + sum(len(r) for r in B)
    assert count == nnz + n_public + 1 and len(co) == 4 + 44 * count
    recs = [struct.unpack_from("<III", co, 4 + 44 * i) + (int.from_bytes(co[16 + 44 * i : 48 + 44 * i], "little"),) for i in range(count)]
    R2 = (1 << 512) % curve.r
    want = sorted([(0, i, col, c * R2 % curve.r) for i, row in enumerate(A) for c, col in row]
                  + [(1, i, col, c * R2 % curve.r) for i, row in enumerate(B) for c, col in row], key=lambda t: (t[1], t[0]))
    assert recs[:nnz] == want
    assert recs[nnz:] == [(0, len(A) + s, s, R2) for s in range(n_public + 1)]   # the value 1 is stored as R^2 mod r


@pytest.mark.parametrize("curve", CURVES, ids=["bls12_381", "bn254"])
def test_zkey_shuffled_holds_the_same_sections(curve):
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    A, B, _ = cs.to_matrices()
    n_inst, n_wit = len(cs.instance_assignment), len(cs.witness_assignment)
    key = toy_key(curve, n_inst - 1, n_inst + n_wit, 8)
    args = (curve, key, csr_from_rows(curve, A), csr_from_rows(curve, B), n_inst - 1, 8)
    plain = sections(zo.write_zkey(*args), b"zkey", 1)
    shuf_bytes = zo.write_zkey(*args, order="shuffled", seed=3)
    shuf = sections(shuf_bytes, b"zkey", 1)
    assert sorted(shuf) == list(range(1, 11)) + [77]
    for t in range(1, 10):
        if t != 4:
            assert shuf[t] == plain[t]
    rec = lambda b: sorted(b[4 + 44 * i : 48 + 44 * i] for i in range(struct.unpack_from("<I", b)[0]))
    assert rec(shuf[4][0]) == rec(plain[4][0]) and shuf[4][0] != plain[4][0]


@pytest.mark.parametrize("curve", CURVES, ids=["bls12_381", "bn254"])
def test_wtns_known_answers(curve):
    z = [1, 5, curve.r - 1, 0]
    for data in (zo.write_wtns(curve, z), zo.write_wtns(curve, pack_fr(curve, z)), zo.write_wtns(curve, pack_fr(curve, z, mont=False), mont=False)):
        sec = sections(data, b"wtns", 2)
        assert sorted(sec) == [1, 2]
        h = sec[1][0]
        assert struct.unpack_from("<I", h) == (32,) and int.from_bytes(h[4:36], "little") == curve.r
        assert struct.unpack_from("<I", h, 36) == (len(z),)
        d = sec[2][0]
        assert [int.from_bytes(d[32 * i : 32 * i + 32], "little") for i in range(len(z))] == z   # canonical, not Montgomery


def test_fr_rescale_once_per_distinct_value():
    curve = BN254
    vals = [3, 3, 7, 3, 0]
    got = zo.fr_rescale(curve, pack_fr(curve, vals, mont=False), 11)
    assert np.array_equal(got, pack_fr(curve, [v * 11 for v in vals], mont=False))
