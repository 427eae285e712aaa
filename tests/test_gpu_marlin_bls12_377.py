"""The universal-setup (Marlin-style) path on BLS12-377: the element-wise polynomial kernels against big-int arithmetic,
the SRS against double-and-add, and small GPU proofs bit-equal to the big-int prover's and accepted by the oracle
verifier, once with real pairings (tests/bls377_oracle.py registers the curve with the oracle)."""
import random

import numpy as np
import pytest

from tests import bls377_oracle as b7
from tests.bls377_oracle import BLS12_377 as CURVE

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def backends():
    from oracle import marlin as om
    from snark_b200.marlin_gpu import GpuBackend

    gb = GpuBackend(curve=CURVE.curve_id, device=0)
    assert gb.r == CURVE.r and gb.p == CURVE.p and gb.coset_gen == CURVE.fr_generator
    assert gb.omega(10) == CURVE.omega(10)
    yield gb, om.IntBackend(CURVE)
    gb.close()


@pytest.mark.parametrize("n", [1, 17, 1000])
def test_poly_kernels_match_bigint(backends, n):
    gb, ib = backends
    rng = random.Random(377 + n)
    r = CURVE.r
    a = [0 if i % 5 == 0 else rng.randrange(r) for i in range(n)]
    b = [rng.randrange(r) for _ in range(n)]
    s = rng.randrange(r)
    da, db = gb.from_ints(a), gb.from_ints(b)
    assert gb.to_ints(da) == a
    assert gb.to_ints(gb.mul(da, db)) == ib.mul(a, b)
    assert gb.to_ints(gb.add(da, db)) == ib.add(a, b)
    assert gb.to_ints(gb.sub(da, db)) == ib.sub(a, b)
    assert gb.to_ints(gb.scale(da, s)) == ib.scale(a, s)
    assert gb.to_ints(gb.add_scalar(da, s)) == ib.add_scalar(a, s)
    assert gb.to_ints(gb.inv0(da)) == ib.inv0(a)
    assert gb.to_ints(gb.geom(n, s, b[0])) == ib.geom(n, s, b[0])
    assert gb.eval(db, s) == ib.eval(b, s)


def test_srs_is_the_powers_of_tau(backends):
    gb, ib = backends
    G1 = b7.groups()[0]
    tau, size = 0x377377, 300
    srs = gb.setup(size, tau)
    gb.be.sync()
    host = srs.cpu().numpy().astype(np.uint32)
    for i in (0, 1, 2, 157, 299):
        assert gb._point(host[i]) == G1.mul(G1.gen, pow(tau, i, CURVE.r))
    coeffs = [random.Random(3).randrange(CURVE.r) for _ in range(200)]
    assert gb.commit(srs, gb.from_ints(coeffs)) == ib.commit(ib.setup(size, tau), coeffs)


def test_gpu_prover_equals_bigint_prover_and_verifies(backends):
    from oracle import marlin as om
    from oracle import r1cs as orc
    from snark_b200 import marlin as M

    gb, ib = backends
    rng = random.Random(0x3770005)
    css = [orc.circuit2(CURVE, 1, 1, 2), orc.dummy_circuit(CURVE, 3, 5, 8, 8), orc.bench_circuit(CURVE, 9, seed=2)]
    for k, cs in enumerate(css):
        cs.finalize()
        mats, x, w = cs.to_matrices(), list(cs.instance_assignment), list(cs.witness_assignment)
        info = M.index_shape(mats, len(x), len(x) + len(w))
        tau = rng.randrange(2, CURVE.r)
        srs_g, srs_i = gb.setup(info.D + 1, tau), ib.setup(info.D + 1, tau)
        pk_g, vk_g = M.index(gb, srs_g, mats, len(x), len(x) + len(w))
        pk_i, vk_i = M.index(ib, srs_i, mats, len(x), len(x) + len(w))
        assert vk_g.index_comms == vk_i.index_comms and vk_g.info == vk_i.info
        pg = M.prove(gb, pk_g, x, w, check=True)
        pi = M.prove(ib, pk_i, x, w, check=True)
        assert pg.comms == pi.comms and pg.evals1 == pi.evals1 and pg.evals2 == pi.evals2 and pg.openings == pi.openings
        assert om.verify(CURVE, vk_g, x, pg, tau=tau)
        if k == 0:   # the opening check with real pairings: e(P, H) = e(W, tau H)
            G2 = b7.groups()[1]
            assert om.verify(CURVE, vk_g, x, pg, tau_g2=G2.mul(G2.gen, tau), engine=b7.engine())
        if len(x) > 1:
            bad = x[:-1] + [(x[-1] + 1) % CURVE.r]
            assert not om.verify(CURVE, vk_g, bad, pg, tau=tau)
