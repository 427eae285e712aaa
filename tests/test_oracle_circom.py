"""The CircomReduction oracle (tests/circom_oracle.py) against the LibsnarkReduction oracle (oracle/groth16.py), on both
curves: the h identity on the odd coset, proofs that satisfy the verification equation in the exponent and, on BN254, with
real pairings; unsatisfying assignments change h and fail the equation."""
import random

import pytest

from oracle import groth16 as og
from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests import circom_oracle as oc

CURVES = [BLS12_381, BN254]


def small_circuits(curve):
    cs2 = orc.circuit2(curve, 1, 1, 2)
    cs2.finalize()
    yield "circuit2", cs2.to_matrices(), cs2.instance_assignment, cs2.witness_assignment
    rng = random.Random(3)
    mats, inst, wit = orc.dummy_circuit_direct(curve, rng.randrange(curve.r), rng.randrange(curve.r), 12, 11)
    yield "dummy_direct", mats, inst, wit


def spoil(curve, wit):
    """every witness value + 1: breaks the constraints of these circuits"""
    return [(v + 1) % curve.r for v in wit]


@pytest.mark.parametrize("curve", CURVES, ids=["bls12_381", "bn254"])
def test_circom_h_is_minus_two_libsnark_h_on_the_odd_coset(curve):
    r = curve.r
    for name, mats, inst, wit in small_circuits(curve):
        z = inst + wit
        az, bz, cz = (orc.mat_vec_mul(r, M, z) for M in mats)
        assert all(x * y % r == w for x, y, w in zip(az, bz, cz)), name
        h_lib = og.witness_map(curve, mats, z, len(inst))
        h_cir = oc.witness_map_circom(curve, mats, z, len(inst))
        assert len(h_cir) == len(h_lib) == og.domain_size(len(mats[0]), len(inst))
        assert h_cir == [(-2 * v) % r for v in oc.odd_coset_eval(curve, h_lib)], name
        # an unsatisfying assignment: the two maps part ways
        zb = inst + spoil(curve, wit)
        az, bz, cz = (orc.mat_vec_mul(r, M, zb) for M in mats)
        assert not all(x * y % r == w for x, y, w in zip(az, bz, cz)), name
        hb_cir = oc.witness_map_circom(curve, mats, zb, len(inst))
        hb_lib = og.witness_map(curve, mats, zb, len(inst))
        assert hb_cir != [(-2 * v) % r for v in oc.odd_coset_eval(curve, hb_lib)], name


@pytest.mark.parametrize("curve", CURVES, ids=["bls12_381", "bn254"])
def test_circom_proofs_equal_libsnark_proofs_and_verify_in_the_exponent(curve):
    rng = random.Random(0xC1C0)
    for name, mats, inst, wit in small_circuits(curve):
        td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
        pk_l = og.setup(curve, mats, len(inst), len(wit), td)
        pk_c = oc.setup_circom(curve, mats, len(inst), len(wit), td)
        assert len(pk_c.h_query) == pk_c.domain and len(pk_l.h_query) == pk_l.domain - 1
        rr, ss = rng.randrange(curve.r), rng.randrange(curve.r)
        A, B, C, h = oc.prove_circom(pk_c, mats, inst, wit, rr, ss)
        assert oc.check_in_exponent(pk_c, (A, B, C), inst, wit, h, rr, ss), name
        assert og.verify_equation_in_exponent(pk_c, inst, *oc.expected_proof_exponents(pk_c, inst, wit, h, rr, ss)), name
        assert (A, B, C) == og.prove(pk_l, mats, inst, wit, rr, ss)[:3], name
        # unsatisfying: the proof is made, and fails the equation
        bad = spoil(curve, wit)
        Ab, Bb, Cb, hb = oc.prove_circom(pk_c, mats, inst, bad, rr, ss)
        assert oc.check_in_exponent(pk_c, (Ab, Bb, Cb), inst, bad, hb, rr, ss)
        assert not og.verify_equation_in_exponent(pk_c, inst, *oc.expected_proof_exponents(pk_c, inst, bad, hb, rr, ss)), name


def test_circom_proof_verifies_with_pairings_bn254():
    from oracle import pairing

    curve = BN254
    rng = random.Random(77)
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
    pk = oc.setup_circom(curve, mats, len(inst), len(wit), td)
    vk = {"alpha_g1": pk.alpha_g1, "beta_g2": pk.beta_g2, "gamma_g2": pk.gamma_g2, "delta_g2": pk.delta_g2,
          "gamma_abc_g1": pk.gamma_abc_g1}
    rr, ss = rng.randrange(curve.r), rng.randrange(curve.r)
    A, B, C, _ = oc.prove_circom(pk, mats, inst, wit, rr, ss)
    assert pairing.groth16_verify(vk, list(inst[1:]), (A, B, C), curve)
    A, B, C, _ = oc.prove_circom(pk, mats, inst, spoil(curve, wit), rr, ss)
    assert not pairing.groth16_verify(vk, list(inst[1:]), (A, B, C), curve)
