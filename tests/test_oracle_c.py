"""The C++ oracle (oracle/c/oracle.cpp: checker at mid sizes, CPU baseline) against the pure-Python
oracle, which is itself pinned by the definitions in tests/test_oracle_py.py."""
import random

import numpy as np
import pytest

from oracle import cnative
from oracle import groth16 as og
from oracle import msm as omsm
from oracle import ntt as ontt
from oracle import r1cs as orc
from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests import circom_oracle as oc
from tests.bls377_oracle import BLS12_377
from tests.util import csr_from_rows, pack_fr, pack_points, unpack_fr, unpack_points

CURVES = [BLS12_381, BN254, BLS12_377]


@pytest.mark.parametrize("cid", [0, 1, 2])
def test_c_ntt(cid):
    curve = CURVES[cid]
    rng = random.Random(cid)
    for log_n in (0, 1, 2, 5, 9):
        x = [rng.randrange(curve.r) for _ in range(1 << log_n)]
        assert unpack_fr(curve, cnative.ntt(cid, pack_fr(curve, x), log_n)) == ontt.ntt(curve, x)
        assert unpack_fr(curve, cnative.ntt(cid, pack_fr(curve, x), log_n, inverse=True)) == ontt.ntt(curve, x, inverse=True)
        assert unpack_fr(curve, cnative.ntt(cid, pack_fr(curve, x), log_n, coset=True)) == ontt.coset_ntt(curve, x)
        assert unpack_fr(curve, cnative.ntt(cid, pack_fr(curve, x), log_n, inverse=True, coset=True)) == ontt.coset_intt(curve, x)


@pytest.mark.parametrize("cid,group", [(0, 1), (0, 2), (1, 1), (1, 2), (2, 1), (2, 2)])
def test_c_msm(cid, group):
    curve = CURVES[cid]
    G = groups(curve)[group - 1]
    rng = random.Random(10 * cid + group)
    pts = [G.mul(G.gen, rng.randrange(1, curve.r)) for _ in range(12)]
    for n in (1, 5, 40, 700):
        bases = [pts[rng.randrange(12)] if rng.random() > 0.05 else None for _ in range(n)]
        scalars = [rng.choice([0, 1, curve.r - 1, rng.randrange(curve.r)]) for _ in range(n)]
        exp = omsm.msm_pippenger(G, bases, scalars)
        got = cnative.msm(cid, group, pack_points(curve, group, bases), pack_fr(curve, scalars), n, threads=3)
        assert unpack_points(curve, group, got)[0] == exp
        got = cnative.msm(cid, group, pack_points(curve, group, bases), pack_fr(curve, scalars, mont=False), n, mont=False, threads=1)
        assert unpack_points(curve, group, got)[0] == exp
    gen = pack_points(curve, group, [G.gen])
    mult = unpack_points(curve, group, cnative.multiples(cid, group, gen, 5, 9, threads=2))
    assert mult == [G.mul(G.gen, 5 + i) for i in range(9)]


@pytest.mark.parametrize("cid", [0, 1, 2])
def test_c_groth16(cid):
    curve = CURVES[cid]
    rng = random.Random(99 + cid)
    bc = orc.bench_circuit(curve, 12, seed=2)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    csr = [csr_from_rows(curve, m) for m in mats]
    z = inst + wit
    for k in range(3):
        assert unpack_fr(curve, cnative.spmv(cid, csr[k], pack_fr(curve, z), len(mats[k]), threads=2)) == orc.mat_vec_mul(curve.r, mats[k], z)
    td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
    pk = og.setup(curve, mats, len(inst), len(wit), td)
    rr, ss = rng.randrange(curve.r), rng.randrange(curve.r)
    A, B, C, h = og.prove(pk, mats, inst, wit, rr, ss)
    assert og.check_in_exponent(pk, (A, B, C), inst, wit, h, rr, ss)
    P1 = lambda pts: pack_points(curve, 1, pts)
    P2 = lambda pts: pack_points(curve, 2, pts)
    arrays = [P1([pk.alpha_g1]), P1([pk.beta_g1]), P1([pk.delta_g1]), P2([pk.beta_g2]), P2([pk.delta_g2]),
              P1(pk.a_query), P1(pk.b_g1_query), P2(pk.b_g2_query), P1(pk.h_query), P1(pk.l_query)]
    a, b, c, hh = cnative.groth16_prove(cid, csr, len(mats[0]), len(inst), len(wit), arrays, pack_fr(curve, inst),
                                        pack_fr(curve, wit), pack_fr(curve, [rr]), pack_fr(curve, [ss]), want_h=True, threads=4)
    assert unpack_fr(curve, hh) == h
    assert np.array_equal(cnative.witness_map(cid, csr, len(mats[0]), len(inst), pack_fr(curve, z), threads=3), hh)   # stand-alone export
    assert (unpack_points(curve, 1, a)[0], unpack_points(curve, 2, b)[0], unpack_points(curve, 1, c)[0]) == (A, B, C)
    x = [rng.randrange(curve.r) for _ in range(50)]
    y = [rng.randrange(curve.r) for _ in range(50)]
    assert unpack_fr(curve, cnative.fr_dot(cid, pack_fr(curve, x), pack_fr(curve, y), 50))[0] == sum(p * q for p, q in zip(x, y)) % curve.r


@pytest.mark.parametrize("cid", [0, 1, 2])
def test_c_witness_map_circom(cid):
    """orc_witness_map_circom against tests/circom_oracle.py, satisfying and spoiled assignments, unit and random
    coefficients, a full domain and one that has just doubled"""
    curve = CURVES[cid]
    rng = random.Random(0xC1 + cid)
    bc = orc.bench_circuit(curve, 12, seed=3)
    bc.finalize()
    cases = [(bc.to_matrices(), bc.instance_assignment, bc.witness_assignment)]
    for n_rows, n_inst, n_vars in ((29, 3, 40), (14, 3, 20)):      # 29 + 3 = 2^5; 14 + 3 = 2^4 + 1
        mats = [[[(rng.choice([1, 2, curve.r - 1, rng.randrange(curve.r)]), rng.randrange(n_vars))
                  for _ in range(rng.randrange(5))] for _ in range(n_rows)] for _ in range(3)]
        z = [1] + [rng.choice([0, 1, curve.r - 1, rng.randrange(curve.r)]) for _ in range(n_vars - 1)]
        cases.append((mats, z[:n_inst], z[n_inst:]))
    for mats, inst, wit in cases:
        csr = [csr_from_rows(curve, m) for m in mats]
        for w in (wit, [(v + 1) % curve.r for v in wit]):
            z = list(inst) + list(w)
            got = cnative.witness_map_circom(cid, csr, len(mats[0]), len(inst), pack_fr(curve, z), threads=3)
            assert unpack_fr(curve, got) == oc.witness_map_circom(curve, mats, z, len(inst)), len(mats[0])
