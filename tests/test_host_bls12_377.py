"""BLS12-377's instantiation of the kernel templates, compiled for the host (tests/native/host_bls377.cpp), against the
BLS12-377 oracle (tests/bls377_oracle.py): Fq / Fr / Fq2 arithmetic, the group law, Tonelli-Shanks square roots, point
decoding on every flag and rejection case, the subgroup criteria against [r]P = O, the pairing against oracle^k with k
re-derived here, and the Groth16 and random-linear-combination verdicts."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import groth16 as og
from oracle import r1cs as orc
from tests import bls377_oracle as b7
from tests.bls377_oracle import BLS12_377 as CURVE
from tests.util import pack_fr, pack_points, pack_u32, unpack_points, unpack_u32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P, R = b7.P, b7.R
RQ = 1 << 384
RR = 1 << 256


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("host377") / "libhost377.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "host_bls377.cpp")])
    return ctypes.CDLL(so)


def vp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def fq_pack(xs):
    return pack_u32([x * RQ % P for x in xs], 12)


def fq_unpack(a):
    ri = pow(RQ, -1, P)
    return [v * ri % P for v in unpack_u32(a, 12)]


def fq2_pack(xs):
    return fq_pack([c for x in xs for c in x])


def fq2_unpack(a):
    v = fq_unpack(a)
    return [(v[i], v[i + 1]) for i in range(0, len(v), 2)]


def test_constants(lib):
    """the header's moduli, Montgomery constants, Fr generator and root of unity against values derived from x"""
    out = np.zeros(12, dtype=np.uint32)
    for which, want in [(0, P), (1, RQ % P), (2, RQ * RQ % P)]:
        lib.ht377_field_const(0, which, vp(out))
        assert unpack_u32(out, 12)[0] == want
    out = np.zeros(8, dtype=np.uint32)
    root = pow(22, (R - 1) >> 47, R)
    for which, want in [(0, R), (1, RR % R), (2, RR * RR % R), (3, 22 * RR % R), (4, root * RR % R)]:
        lib.ht377_field_const(1, which, vp(out))
        assert unpack_u32(out, 8)[0] == want
    assert pow(root, 1 << 46, R) == R - 1


@pytest.mark.parametrize("field", [0, 1], ids=["fq", "fr"])
def test_field_ops(lib, field):
    rng = random.Random(0x377 + field)
    m, n, Rm = (P, 12, RQ) if field == 0 else (R, 8, RR)
    xs = [0, 1, m - 1, m - 2, (m - 1) // 2] + [rng.randrange(m) for _ in range(27)]
    ys = [rng.randrange(m) for _ in xs[:-1]] + [0]
    a, b = pack_u32([x * Rm % m for x in xs], n), pack_u32([y * Rm % m for y in ys], n)
    ri = pow(Rm, -1, m)
    for op, f in [(0, lambda x, y: x * y), (1, lambda x, y: x + y), (2, lambda x, y: x - y),
                  (3, lambda x, y: pow(x, -1, m) if x else 0), (4, lambda x, y: -x), (7, lambda x, y: x * x)]:
        out = np.zeros_like(a)
        lib.ht377_field_op(field, op, vp(a), vp(b), vp(out), len(xs))
        assert [v * ri % m for v in unpack_u32(out, n)] == [f(x, y) % m for x, y in zip(xs, ys)], op


def test_fq2_ops(lib):
    """u^2 = -5: products, squares, inverses and the multiplication by xi = u, including the non-residue itself"""
    rng = random.Random(0xF2)
    F = b7.Fld5(P, 2)
    xs = [(0, 1), (1, 0), (0, P - 1), (P - 5, 0), (5, 0), (P - 1, P - 1)] + [(rng.randrange(P), rng.randrange(P)) for _ in range(10)]
    ys = [(0, 1), (0, 1), (0, 1), (0, 1), (3, 7), (P - 1, 1)] + [(rng.randrange(P), rng.randrange(P)) for _ in range(10)]
    assert F.mul((0, 1), (0, 1)) == (P - 5, 0)
    a, b = fq2_pack(xs), fq2_pack(ys)
    ok = np.zeros(len(xs), dtype=np.uint8)

    def run(op):
        out = np.zeros_like(a)
        lib.ht377_fq2_op(op, vp(a), vp(b), vp(out), vp(ok), len(xs))
        return fq2_unpack(out)

    assert run(0) == [F.mul(x, y) for x, y in zip(xs, ys)]
    assert run(1) == [F.sqr(x) for x in xs]
    assert run(2) == [F.inv(x) for x in xs]
    assert run(3) == [F.mul(x, (0, 1)) for x in xs]
    assert run(5) == [F.add(x, y) for x, y in zip(xs, ys)]
    assert run(6) == [F.sub(x, y) for x, y in zip(xs, ys)]


def test_sqrt_tonelli_shanks(lib):
    """Fq and Fq2 square roots: existence agrees with the oracle (Euler's criterion / the norm), a returned root squares
    back; the oracle's Tonelli-Shanks agrees with brute force on small primes with high two-adicity"""
    for q in (97, 193, 257, 7681, 12289, 65537):           # p - 1 divisible by 2^5 .. 2^16
        roots = {x * x % q for x in range(q)}
        for a in range(q):
            s = b7.sqrt_fq(a, q)
            assert (s is not None) == (a in roots) and (s is None or s * s % q == a), (q, a)
    rng = random.Random(0x5027)
    F = b7.Fld5(P, 2)
    xs = [0, 1, P - 1, 5, P - 5, 4] + [rng.randrange(P) for _ in range(20)]
    ok = np.zeros(len(xs), dtype=np.uint8)
    out = np.zeros(len(xs) * 12, dtype=np.uint32)
    lib.ht377_fq_sqrt(vp(fq_pack(xs)), vp(out), vp(ok), len(xs))
    for x, s, k in zip(xs, fq_unpack(out), ok):
        assert bool(k) == (pow(x, (P - 1) // 2, P) in (0, 1)), x
        if k:
            assert s * s % P == x
    ys = [(0, 0), (1, 0), (P - 1, 0), (P - 5, 0), (5, 0), (0, 1)] + [(rng.randrange(P), rng.randrange(P)) for _ in range(10)]
    ys += [F.sqr((rng.randrange(P), rng.randrange(P))) for _ in range(10)] + [F.sqr((rng.randrange(P), 0)) for _ in range(2)]
    ys += [F.sqr((0, rng.randrange(P))) for _ in range(2)]
    ok = np.zeros(len(ys), dtype=np.uint8)
    out = np.zeros(len(ys) * 24, dtype=np.uint32)
    lib.ht377_fq2_op(4, vp(fq2_pack(ys)), vp(fq2_pack(ys)), vp(out), vp(ok), len(ys))
    for y, s, k in zip(ys, fq2_unpack(out), ok):
        norm = (y[0] * y[0] + 5 * y[1] * y[1]) % P
        assert bool(k) == (pow(norm, (P - 1) // 2, P) in (0, 1)) == (b7.sqrt_fq2(y) is not None), y
        if k:
            assert F.sqr(s) == y


@pytest.mark.parametrize("group", [1, 2])
def test_group_law(lib, group):
    rng = random.Random(0xEC + group)
    G = b7.groups()[group - 1]
    gen = np.zeros(4 * 12 * group // 2, dtype=np.uint32)
    lib.ht377_generator(group, vp(gen))
    assert unpack_points(CURVE, group, gen) == [G.gen]
    A = [G.mul(G.gen, rng.randrange(1, R)) for _ in range(4)]
    B = [G.mul(G.gen, rng.randrange(1, R)) for _ in range(4)]
    ks = [rng.randrange(R) for _ in range(4)]
    a, b, k = pack_points(CURVE, group, A), pack_points(CURVE, group, B), pack_u32(ks, 8)
    out = np.zeros_like(a)
    lib.ht377_ec_op(group, 0, vp(a), vp(b), vp(k), 8, vp(out), 4)
    assert unpack_points(CURVE, group, out) == [G.add(x, y) for x, y in zip(A, B)]
    lib.ht377_ec_op(group, 1, vp(a), vp(b), vp(k), 8, vp(out), 4)
    assert unpack_points(CURVE, group, out) == [G.dbl(x) for x in A]
    lib.ht377_ec_op(group, 2, vp(a), vp(b), vp(k), 8, vp(out), 4)
    assert unpack_points(CURVE, group, out) == [G.mul(x, kk) for x, kk in zip(A, ks)]


def decode(lib, group, blobs, compressed, validate):
    out = np.zeros(len(blobs) * 12 * 2 * group, dtype=np.uint32)
    st = np.zeros(len(blobs), dtype=np.uint32)
    buf = np.frombuffer(b"".join(blobs), dtype=np.uint8).copy()
    lib.ht377_point_decode(group, vp(buf), int(compressed), int(validate), vp(out), vp(st), len(blobs))
    return st.tolist(), unpack_points(CURVE, group, out)


def outside_points(group, rng):
    """on the curve, outside the prime-order subgroup: random points, cofactor torsion, and subgroup + torsion"""
    G = b7.groups()[group - 1]
    pts = [b7.random_curve_point(group, rng) for _ in range(3)]
    pts.append(b7.mul_unreduced(G, b7.random_curve_point(group, rng), R))            # [r] of a random point
    if group == 1:
        for q in b7.small_primes(b7.H1, 1000):
            T = b7.torsion_point(1, q, rng)
            pts += [T, G.add(G.mul(G.gen, rng.randrange(1, R)), T)]
    else:
        pts.append(G.add(G.mul(G.gen, rng.randrange(1, R)), pts[-1]))
    assert all(p is not None and G.on_curve(p) and not b7.in_subgroup(group, p) for p in pts)
    return pts


@pytest.mark.parametrize("group", [1, 2])
def test_subgroup_criterion(lib, group):
    """phi(P) = -[x^2]P (G1) and psi(P) = [x]P (G2) against [r]P = O: subgroup points in, every outside point out"""
    rng = random.Random(0x5B + group)
    G = b7.groups()[group - 1]
    inside = [G.gen] + [G.mul(G.gen, rng.randrange(1, R)) for _ in range(3)]
    outside = outside_points(group, rng)
    ok = np.zeros(len(inside) + len(outside), dtype=np.uint8)
    lib.ht377_in_subgroup(group, vp(pack_points(CURVE, group, inside + outside)), vp(ok), len(ok))
    assert ok.tolist() == [1] * len(inside) + [0] * len(outside)


@pytest.mark.parametrize("group", [1, 2])
def test_decode_point(lib, group):
    """SWFlags encodings of the oracle: every point round-trips, and every flag / canonicity / curve / subgroup rejection
    gives the oracle's status, compressed and uncompressed"""
    rng = random.Random(0xDE + group)
    G = b7.groups()[group - 1]
    pts = [None, G.gen, G.neg(G.gen)] + [G.mul(G.gen, rng.randrange(1, R)) for _ in range(4)]
    out_pt = outside_points(group, rng)[:2]
    for compressed in (True, False):
        L = 48 * group * (1 if compressed else 2)
        blobs = [b7.encode_point(group, p, compressed) for p in pts]
        for validate in (True, False):
            st, got = decode(lib, group, blobs, compressed, validate)
            assert st == [0] * len(pts) and got == pts
        bad = []
        e = bytearray(blobs[1]); e[-1] |= 0xC0; bad.append(bytes(e))                       # both flags
        e = bytearray(L); e[-1] = 0x40; e[0] = 1; bad.append(bytes(e))                       # infinity with a nonzero byte
        e = bytearray(L); e[-1] = 0xC0; bad.append(bytes(e))                                 # infinity and "larger"
        pm = bytearray((P + 1).to_bytes(48, "little")) + bytearray(L - 48)
        bad.append(bytes(pm))                                                                # x = p + 1 (c0)
        for bit in range(377, 382):     # stray bits between bit 376 and the flags of the last element: non-canonical
            e = bytearray(blobs[1]); e[-1] |= 1 << (bit - 376); bad.append(bytes(e))
        if not compressed:
            e = bytearray(blobs[1]); e[48 * group] ^= 1; bad.append(bytes(e))             # y changed: off the curve
        # an x with no point above it (compressed) / a point off the subgroup (both modes)
        while compressed:
            x = rng.randrange(P) if group == 1 else (rng.randrange(P), rng.randrange(P))
            rhs = G.f.add(G.f.mul(G.f.sqr(x), x), G.b)
            if (b7.sqrt_fq(rhs) if group == 1 else b7.sqrt_fq2(rhs)) is None:
                e = bytearray(b7.encode_point(group, (x, G.f.one if group == 2 else 1), True))
                e[-1] &= 0x3F
                bad.append(bytes(e))
                break
        bad += [b7.encode_point(group, p, compressed) for p in out_pt]
        want = [b7.decode_point(group, blob, compressed, True)[0] for blob in bad]
        assert set(want) >= {1, 2, 4} and (3 in want)
        st, _ = decode(lib, group, bad, compressed, True)
        assert st == want
        st, got = decode(lib, group, bad[-2:], compressed, False)                             # Validate::No keeps them
        assert st == [0, 0] and got == out_pt


def test_pairing(lib):
    """e = oracle^k, with k = 3 re-derived: T = t - 1 = x > 0 is the kernels' Miller loop, so the Miller functions agree,
    and the hard part computes f^(3 h) by 3 h = (x - 1)^2 (x + p)(x^2 + p^2 - 1) + 3"""
    x, p, r = b7.X, P, R
    h = (p ** 4 - p ** 2 + 1) // r
    assert (x - 1) ** 2 * (x + p) * (x * x + p * p - 1) + 3 == 3 * h and 3 * h % r != 0
    assert (x + 1) - 1 == b7.engine().loop                      # trace t = x + 1
    k = 3
    assert b7.K == k
    rng = random.Random(0xE7)
    G1, G2 = b7.groups()
    E = b7.engine()
    Ps = [G1.mul(G1.gen, rng.randrange(1, R)) for _ in range(2)] + [G1.gen, None, G1.gen]
    Qs = [G2.mul(G2.gen, rng.randrange(1, R)) for _ in range(2)] + [G2.gen, G2.gen, None]
    out = np.zeros(len(Ps) * 144, dtype=np.uint32)
    lib.ht377_pairing(0, vp(pack_points(CURVE, 1, Ps)), vp(pack_points(CURVE, 2, Qs)), vp(out), len(Ps))
    got = b7.gt_to_oracle(out)
    for i in range(3):
        assert got[i] == E.pairing(Ps[i], Qs[i]).pow(k), i
    one = E.Fq12.one()
    assert got[3] == one and got[4] == one and got[2] != one and got[2].pow(R) == one
    m1, m2 = np.zeros_like(out), np.zeros_like(out)
    lib.ht377_pairing(1, vp(pack_points(CURVE, 1, Ps)), vp(pack_points(CURVE, 2, Qs)), vp(m1), len(Ps))
    lib.ht377_pairing(2, vp(pack_points(CURVE, 1, Ps)), vp(pack_points(CURVE, 2, Qs)), vp(m2), len(Ps))
    assert m1.tolist() == m2.tolist()
    assert lib.ht377_prepared_lines() == 63 + bin(x).count("1") - 1


def test_tower(lib):
    """Fq12 products, inverses and Frobenius powers against the oracle's Fq[w]/(w^12 + 5)"""
    rng = random.Random(0x12)
    E = b7.engine()
    A = [E.Fq12([rng.randrange(P) for _ in range(12)]) for _ in range(3)]
    B = [E.Fq12([rng.randrange(P) for _ in range(12)]) for _ in range(3)]
    a, b = b7.gt_from_oracle(A), b7.gt_from_oracle(B)
    assert b7.gt_to_oracle(a) == A

    def op(o, x, y=None):
        out = np.zeros_like(x)
        lib.ht377_fp12_op(o, vp(x), vp(y if y is not None else x), vp(out), len(x) // 144)
        return out

    assert b7.gt_to_oracle(op(0, a, b)) == [x * y for x, y in zip(A, B)]
    assert b7.gt_to_oracle(op(1, a)) == [x * x for x in A]
    assert b7.gt_to_oracle(op(2, a)) == [x.inv() for x in A]
    for j in (1, 2, 3):
        assert b7.gt_to_oracle(op(2 + j, a)) == [x.pow(P ** j) for x in A], j
    c = b7.gt_from_oracle([x.pow(P ** 6 - 1).pow(P ** 2 + 1) for x in A])
    assert op(6, c).tolist() == op(1, c).tolist()


def oracle_proofs(rng):
    cs = orc.circuit2(CURVE, 1, 1, 2)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    pk = og.setup(CURVE, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, R) for _ in range(5)]))
    proofs = [og.prove(pk, mats, inst, wit, rng.randrange(R), rng.randrange(R))[:3] for _ in range(3)]
    vk = dict(alpha_g1=pk.alpha_g1, beta_g2=pk.beta_g2, gamma_g2=pk.gamma_g2, delta_g2=pk.delta_g2, gamma_abc_g1=pk.gamma_abc_g1)
    return vk, list(inst[1:]), proofs


def ic_of(vk, x):
    G1 = b7.groups()[0]
    ic = vk["gamma_abc_g1"][0]
    for xi, base in zip(x, vk["gamma_abc_g1"][1:]):
        ic = G1.add(ic, G1.mul(base, xi))
    return ic


def vk_pack(vk):
    return np.concatenate([pack_points(CURVE, 1, [vk["alpha_g1"]]), pack_points(CURVE, 2, [vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"]])])


def test_groth16_and_rlc_verdicts(lib):
    """the per-proof verdict and the RLC batch verdict on oracle proofs, valid and tampered"""
    rng = random.Random(0x6B7)
    G1 = b7.groups()[0]
    vk, x, proofs = oracle_proofs(rng)
    (A, B, C), (A2, B2, C2), _ = proofs
    x_bad = [(x[0] + 1) % R] + x[1:]
    cases = [(x, (A, B, C)), (x, (A2, B2, C2)), (x, (G1.add(A, G1.gen), B, C)), (x, (A, B2, C)), (x, (A, B, G1.neg(C))),
             (x_bad, (A, B, C)), (x, (None, B, C))]
    ok = np.zeros(len(cases), dtype=np.uint8)
    lib.ht377_groth16_verdict(vp(vk_pack(vk)), vp(pack_points(CURVE, 1, [ic_of(vk, xs) for xs, _ in cases])),
                              vp(pack_points(CURVE, 1, [pr[0] for _, pr in cases])), vp(pack_points(CURVE, 2, [pr[1] for _, pr in cases])),
                              vp(pack_points(CURVE, 1, [pr[2] for _, pr in cases])), vp(ok), len(cases))
    assert ok.tolist() == [1, 1, 0, 0, 0, 0, 0]
    assert b7.engine().groth16_verify(vk, x, (A, B, C)) and not b7.engine().groth16_verify(vk, x_bad, (A, B, C))

    def rlc(prs, xs):
        rho = pack_u32([rng.randrange(1, 1 << 128) for _ in prs], 4)
        return lib.ht377_rlc_verdict(vp(vk_pack(vk)), vp(pack_points(CURVE, 1, vk["gamma_abc_g1"])),
                                     vp(pack_fr(CURVE, [v for xx in xs for v in xx])), len(x),
                                     vp(pack_points(CURVE, 1, [p[0] for p in prs])), vp(pack_points(CURVE, 2, [p[1] for p in prs])),
                                     vp(pack_points(CURVE, 1, [p[2] for p in prs])), vp(rho), len(prs))

    assert rlc(proofs, [x] * 3) == 1
    assert rlc(proofs, [x, x_bad, x]) == 0
    assert rlc([proofs[0], (A, B, G1.neg(C)), proofs[2]], [x] * 3) == 0
