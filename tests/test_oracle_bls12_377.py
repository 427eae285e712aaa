"""The BLS12-377 oracle (tests/bls377_oracle.py) checked on its own terms: the parameters from the seed x, generators on
their curves and of order r, two-adicities, the cofactors, the textbook pairing's bilinearity and non-degeneracy, Groth16
setup / prove / verify with real pairings, the SWFlags wire form, and Tonelli-Shanks against brute force."""
import random

import pytest

from oracle import groth16 as og
from oracle import ntt as ontt
from oracle import r1cs as orc
from tests import bls377_oracle as b7
from tests.bls377_oracle import BLS12_377 as CURVE

P, R, X = b7.P, b7.R, b7.X


def test_parameters():
    assert X == 0x8508C00000000001
    assert R == X ** 4 - X ** 2 + 1 and R.bit_length() == 253
    assert P == (X - 1) ** 2 * R // 3 + X and (X - 1) ** 2 * R % 3 == 0 and P.bit_length() == 377
    assert P == 0x01AE3A4617C510EAC63B05C06CA1493B1A22D9F300F5138F1EF3622FBA094800170B5D44300000008508C00000000001
    assert R == 0x12AB655E9A2CA55660B44D1E5C37B00159AA76FED00000010A11800000000001
    assert b7.two_adicity(P - 1) == 46 and b7.two_adicity(R - 1) == 47 == CURVE.fr_two_adicity
    assert pow(CURVE.fr_generator, (R - 1) // 2, R) == R - 1                    # 22 is a quadratic non-residue
    w = CURVE.fr_root_of_unity
    assert pow(w, 1 << 47, R) == 1 and pow(w, 1 << 46, R) == R - 1
    assert pow(P - 5, (P - 1) // 2, P) == P - 1                                  # u^2 = -5 is irreducible
    assert (P ** 12 - 1) % R == 0 and (P ** 6 - 1) % R != 0                      # embedding degree 12
    # #E(Fq) = p + 1 - t with t = x + 1, and the G2 cofactor formula
    assert (P + 1 - (X + 1)) == b7.H1 * R
    assert b7.H2 * 9 == X ** 8 - 4 * X ** 7 + 5 * X ** 6 - 4 * X ** 4 + 6 * X ** 3 - 4 * X ** 2 - 4 * X + 13


def test_generators_and_cofactors():
    G1, G2 = b7.groups()
    assert G1.on_curve(G1.gen) and G2.on_curve(G2.gen)
    assert b7.mul_unreduced(G1, G1.gen, R) is None and b7.mul_unreduced(G2, G2.gen, R) is None
    F2 = G2.f
    assert F2.mul(b7.B2, (0, 1)) == (1, 0)                                       # b' = 1 / u (D-type twist of b = 1)
    rng = random.Random(7)
    for g, h in ((1, b7.H1), (2, b7.H2)):
        G = b7.groups()[g - 1]
        Q = b7.random_curve_point(g, rng)
        assert G.on_curve(Q) and b7.mul_unreduced(G, Q, h * R) is None
        assert b7.mul_unreduced(G, b7.mul_unreduced(G, Q, h), R) is None         # cofactor clearing lands in the subgroup
    assert b7.small_primes(b7.H1, 1000) == [2, 3, 7, 13, 499]


def test_tonelli_shanks_brute_force():
    for q in (17, 97, 193, 257, 7681, 12289, 40961):
        squares = {x * x % q for x in range(q)}
        for a in range(q):
            s = b7.sqrt_fq(a, q)
            assert (s is not None) == (a in squares) and (s is None or s * s % q == a)
    rng = random.Random(3)
    F = b7.Fld5(P, 2)
    for _ in range(10):
        a = rng.randrange(P)
        s = b7.sqrt_fq(a * a % P)
        assert s in (a, P - a)
        y = (rng.randrange(P), rng.randrange(P))
        assert F.sqr(b7.sqrt_fq2(F.sqr(y))) == F.sqr(y)
    assert b7.sqrt_fq2((P - 5, 0)) is not None and F.sqr(b7.sqrt_fq2((P - 5, 0))) == (P - 5, 0)


def test_pairing_bilinear_nondegenerate():
    G1, G2 = b7.groups()
    E = b7.engine()
    rng = random.Random(11)
    a, b = rng.randrange(2, R), rng.randrange(2, R)
    e = E.pairing(G1.gen, G2.gen)
    one = E.Fq12.one()
    assert e != one and e.pow(R) == one
    assert E.pairing(G1.mul(G1.gen, a), G2.gen) == e.pow(a)
    assert E.pairing(G1.gen, G2.mul(G2.gen, b)) == e.pow(b)
    assert E.pairing(G1.mul(G1.gen, a), G2.mul(G2.gen, b)) == e.pow(a * b % R)


def test_groth16_real_pairings():
    """setup under a known trapdoor, prove, and verify with pairings; a changed input or proof is rejected"""
    rng = random.Random(0x67)
    cs = orc.circuit2(CURVE, 1, 1, 2)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    td = og.Trapdoor(*[rng.randrange(1, R) for _ in range(5)])
    pk = og.setup(CURVE, mats, len(inst), len(wit), td)
    A, B, C = og.prove(pk, mats, inst, wit, rng.randrange(R), rng.randrange(R))[:3]
    vk = dict(alpha_g1=pk.alpha_g1, beta_g2=pk.beta_g2, gamma_g2=pk.gamma_g2, delta_g2=pk.delta_g2, gamma_abc_g1=pk.gamma_abc_g1)
    E = b7.engine()
    x = list(inst[1:])
    assert E.groth16_verify(vk, x, (A, B, C))
    assert not E.groth16_verify(vk, [(x[0] + 1) % R] + x[1:], (A, B, C))
    assert not E.groth16_verify(vk, x, (A, B, b7.groups()[0].neg(C)))


def test_ntt_matches_dft():
    rng = random.Random(5)
    xs = [rng.randrange(R) for _ in range(16)]
    w = CURVE.omega(4)
    assert ontt.ntt(CURVE, xs) == [sum(x * pow(w, i * j, R) for j, x in enumerate(xs)) % R for i in range(16)]


@pytest.mark.parametrize("group", [1, 2])
def test_wire_round_trip(group):
    rng = random.Random(0x51 + group)
    G = b7.groups()[group - 1]
    pts = [None, G.gen, G.neg(G.gen)] + [G.mul(G.gen, rng.randrange(1, R)) for _ in range(4)]
    for compressed in (True, False):
        for Pt in pts:
            blob = b7.encode_point(group, Pt, compressed)
            assert len(blob) == 48 * group * (1 if compressed else 2)
            assert b7.decode_point(group, blob, compressed) == (0, Pt)
        Q = b7.random_curve_point(group, rng)
        assert b7.decode_point(group, b7.encode_point(group, Q, compressed), compressed, True)[0] == 4
        assert b7.decode_point(group, b7.encode_point(group, Q, compressed), compressed, False) == (0, Q)
