"""The pairing of the verify path (snark_b200/csrc/pairing.cuh), compiled for the host, against the oracle's Fq12 and
pairing (oracle/pairing.py): tower arithmetic, the Miller loop with on-the-fly and prepared lines, the final
exponentiation, e = oracle^k with the k stated in pairing.cuh, and the per-proof Groth16 verdict on oracle proofs."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import groth16 as og
from oracle import r1cs as orc
from oracle.ec import groups
from oracle.pairing import engine
from oracle.params import BLS12_381, BN254
from tests.pairing_oracle import K_STATED, gt_from_oracle, gt_to_oracle, pairing_k, random_gt_raw
from tests.util import fq_limbs, pack_points, pack_u32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = [BLS12_381, BN254]
IDS = ["bls12_381", "bn254"]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostpair") / "libhostpair.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "host_pairing.cpp")])
    return ctypes.CDLL(so)


def vp(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def fp12_op(lib, curve, op, a, b=None):
    count = len(a) // (12 * fq_limbs(curve))
    out = np.zeros_like(a)
    lib.ht_fp12_op(curve.curve_id, op, vp(a), vp(b) if b is not None else None, vp(out), count)
    return out


def host_pairing(lib, curve, mode, P, Q):
    p, q = pack_points(curve, 1, P), pack_points(curve, 2, Q)
    out = np.zeros(len(P) * 12 * fq_limbs(curve), dtype=np.uint32)
    lib.ht_pairing(curve.curve_id, mode, vp(p), vp(q), vp(out), len(P))
    return out


def rand_points(curve, rng, n):
    G1, G2 = groups(curve)
    return ([G1.mul(G1.gen, rng.randrange(1, curve.r)) for _ in range(n)],
            [G2.mul(G2.gen, rng.randrange(1, curve.r)) for _ in range(n)])


def in_cyclotomic(curve, lib, raw):
    """f^((p^6 - 1)(p^2 + 1)) for random f: the first half of the final exponentiation, in the oracle"""
    E = engine(curve)
    p = curve.p
    return gt_from_oracle(curve, [f.pow(p ** 6 - 1).pow(p ** 2 + 1) for f in gt_to_oracle(curve, raw)])


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_tower_arithmetic(lib, curve):
    rng = random.Random(0xF12 + curve.curve_id)
    p = curve.p
    a, b = random_gt_raw(curve, rng, 4), random_gt_raw(curve, rng, 4)
    A, B = gt_to_oracle(curve, a), gt_to_oracle(curve, b)
    assert gt_from_oracle(curve, A).tolist() == a.tolist()           # the basis map round-trips
    assert gt_to_oracle(curve, fp12_op(lib, curve, 0, a, b)) == [x * y for x, y in zip(A, B)]
    assert gt_to_oracle(curve, fp12_op(lib, curve, 1, a)) == [x * x for x in A]
    assert gt_to_oracle(curve, fp12_op(lib, curve, 2, a)) == [x.inv() for x in A]
    for j in (1, 2, 3):
        assert gt_to_oracle(curve, fp12_op(lib, curve, 2 + j, a)) == [x.pow(p ** j) for x in A], j


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_cyclotomic_square(lib, curve):
    rng = random.Random(0xC7C + curve.curve_id)
    c = in_cyclotomic(curve, lib, random_gt_raw(curve, rng, 3))
    assert fp12_op(lib, curve, 6, c).tolist() == fp12_op(lib, curve, 1, c).tolist()


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_sparse_line_multiplication(lib, curve):
    rng = random.Random(0x11E + curve.curve_id)
    n, p = fq_limbs(curve), curve.p
    R = 1 << (32 * n)
    f = random_gt_raw(curve, rng, 3)
    lines = [[rng.randrange(p) for _ in range(6)] for _ in range(3)]
    # the same line as a full Fq12 element: coefficients (l0, l1, l2) at w^(0, 2, 3) (M-type) or w^(0, 1, 3) (D-type)
    slots = [0, 1, 4] if curve is BLS12_381 else [0, 3, 4]      # ark layout positions of those powers
    full = []
    for l in lines:
        co = [0] * 12
        for s, (x0, x1) in zip(slots, [(l[0], l[1]), (l[2], l[3]), (l[4], l[5])]):
            co[2 * s], co[2 * s + 1] = x0, x1
        full += co
    full = pack_u32([v * R % p for v in full], n)
    lb = pack_u32([v * R % p for l in lines for v in l], n)
    assert fp12_op(lib, curve, 7, f, lb).tolist() == fp12_op(lib, curve, 0, f, full).tolist()


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_pairing_against_oracle(lib, curve):
    """e = oracle^k on random pairs, with k recomputed from pairing.cuh's derivation; prepared lines give the same Miller
    value as lines on the fly."""
    assert pairing_k(curve) == K_STATED[curve.name]
    rng = random.Random(0xE0 + curve.curve_id)
    E = engine(curve)
    P, Q = rand_points(curve, rng, 2)
    got = gt_to_oracle(curve, host_pairing(lib, curve, 0, P, Q))
    k = pairing_k(curve)
    for i in range(2):
        assert got[i] == E.pairing(P[i], Q[i]).pow(k), i
    assert host_pairing(lib, curve, 1, P, Q).tolist() == host_pairing(lib, curve, 2, P, Q).tolist()


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_pairing_properties(lib, curve):
    rng = random.Random(0xB1 + curve.curve_id)
    G1, G2 = groups(curve)
    r = curve.r
    one = gt_to_oracle(curve, gt_from_oracle(curve, [engine(curve).Fq12.one()]))[0]
    a, b = rng.randrange(2, r), rng.randrange(2, r)
    P, Q = G1.gen, G2.gen
    e = gt_to_oracle(curve, host_pairing(lib, curve, 0, [P, G1.mul(P, a), P, None, P], [Q, Q, G2.mul(Q, b), Q, None]))
    assert e[0] != one                                   # non-degenerate
    assert e[0].pow(r) == one                            # of order r
    assert e[1] == e[0].pow(a)                           # bilinear in P
    assert e[2] == e[0].pow(b)                           # bilinear in Q
    assert e[3] == one and e[4] == one                   # infinity on either side
    m1 = host_pairing(lib, curve, 1, [None, P], [Q, None])
    assert all(x == one for x in gt_to_oracle(curve, m1))        # the Miller loop skips such pairs altogether
    assert host_pairing(lib, curve, 2, [None, P], [Q, None]).tolist() == m1.tolist()


def oracle_proofs(curve, rng):
    """vk, public inputs and proofs of a small circuit from the oracle prover"""
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    pk = og.setup(curve, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)]))
    proofs = [og.prove(pk, mats, inst, wit, rng.randrange(curve.r), rng.randrange(curve.r))[:3] for _ in range(2)]
    vk = dict(alpha_g1=pk.alpha_g1, beta_g2=pk.beta_g2, gamma_g2=pk.gamma_g2, delta_g2=pk.delta_g2, gamma_abc_g1=pk.gamma_abc_g1)
    return vk, list(inst[1:]), proofs


def ic_of(curve, vk, x):
    G1 = groups(curve)[0]
    ic = vk["gamma_abc_g1"][0]
    for xi, base in zip(x, vk["gamma_abc_g1"][1:]):
        ic = G1.add(ic, G1.mul(base, xi))
    return ic


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_groth16_verdict(lib, curve):
    """The verdict function of the verify kernels against oracle.pairing.groth16_verify, on valid and tampered proofs."""
    rng = random.Random(0x6B + curve.curve_id)
    G1 = groups(curve)[0]
    vk, x, proofs = oracle_proofs(curve, rng)
    (A, B, C), (A2, B2, C2) = proofs
    x_bad = [(x[0] + 1) % curve.r] + x[1:]
    cases = [  # (inputs, proof)
        (x, (A, B, C)), (x, (A2, B2, C2)),
        (x, (G1.add(A, G1.gen), B, C)),          # A + G1
        (x, (A, B2, C)),                         # another proof's B
        (x, (A, B, G1.neg(C))),                  # C negated
        (x_bad, (A, B, C)),                      # a public input changed
        (x, (None, B, C)),                       # A at infinity
    ]
    vkb = np.concatenate([pack_points(curve, 1, [vk["alpha_g1"]]),
                          pack_points(curve, 2, [vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"]])])
    ic = pack_points(curve, 1, [ic_of(curve, vk, xs) for xs, _ in cases])
    a = pack_points(curve, 1, [pr[0] for _, pr in cases])
    b = pack_points(curve, 2, [pr[1] for _, pr in cases])
    c = pack_points(curve, 1, [pr[2] for _, pr in cases])
    ok = np.zeros(len(cases), dtype=np.uint8)
    lib.ht_groth16_verdict(curve.curve_id, vp(vkb), vp(ic), vp(a), vp(b), vp(c), vp(ok), len(cases))
    want = [1, 1, 0, 0, 0, 0, 0]
    assert ok.tolist() == want
    for i in (0, 2, 5):   # the oracle's verifier agrees (a sample: each check costs a full oracle pairing product)
        xs, pr = cases[i]
        assert engine(curve).groth16_verify(vk, xs, pr) == bool(want[i]), i
