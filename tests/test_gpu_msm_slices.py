"""Batched-affine rounds in slices of the bucket range (csrc/msm.cu, `bucket_sums_t`): when the rounds' scratch for all
buckets does not fit, they run once per slice of whole buckets.  B2S_MSM_ROUND_BUDGET (bytes) stands in for the free
device memory so that small problems slice; every result must be bit-identical to the rounds in one piece."""
import random

import numpy as np
import pytest

from oracle import msm as omsm
from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests.test_gpu_prove_batch import assert_same, gpu_key, random_z, rs_with_zeros, singles
from tests.test_gpu_groth16 import circuits
from tests.util import limbs_to_ints, pack_fr, pack_points, random_fr_limbs, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
# from many slices of a few buckets each down to a budget under the largest skewed bucket (the rounds then switch off)
BUDGETS = ["40000000", "8000000", "1000000", "100000"]


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def scalars_of(curve, kind, n, seed):
    rng = np.random.default_rng(seed)
    raw = random_fr_limbs(rng, n, bits=curve.r.bit_length() - 1)
    if kind == "skewed":
        # a third of the scalars share one value and a third another: a few buckets per window hold most entries
        raw = raw.reshape(n, 8)
        raw[0::3] = raw[0]
        raw[1::3] = raw[1]
        raw = raw.reshape(-1)
    return raw


@pytest.mark.parametrize("group,log_n", [(1, 12), (1, 15), (2, 12)])
@pytest.mark.parametrize("kind", ["uniform", "skewed"])
def test_sliced_rounds_match_one_piece(be, monkeypatch, group, log_n, kind):
    import torch

    monkeypatch.setenv("B2S_MSM_AFFINE_ROUNDS", "3")
    monkeypatch.setenv("B2S_MSM_DEDUP", "0")           # skewed scalars reach the bucket structure as they are
    curve = CURVES[be.curve]
    n = 1 << log_n
    ks = np.zeros((n, 8), dtype=np.uint32)
    ks[:, 0] = np.arange(1, n + 1, dtype=np.uint32)
    pt_bytes = be.g1_bytes if group == 1 else be.g2_bytes
    bases = torch.empty(n * pt_bytes // 4, dtype=torch.int32, device="cuda")
    ks_t = torch.from_numpy(ks.view(np.int32)).cuda()
    be.fixed_base(group, ks_t, n, mont=False, out=bases)
    # the library reads ks_t on its own stream: done before the tensor's memory can go to the scalars below
    be.sync()
    del ks_t
    raw = scalars_of(curve, kind, n, 0x5A1 + log_n)
    s_t = torch.from_numpy(raw.view(np.int32)).cuda()
    fn = be.msm_g1 if group == 1 else be.msm_g2
    l0 = be.launches
    ref = fn(bases, s_t, n, mont=True)
    one_piece = be.launches - l0
    # bases (i+1) G: the MSM is (sum_i s_i (i+1)) G
    G = groups(curve)[group - 1]
    Rinv = pow(1 << 256, -1, curve.r)
    total = sum(s * (i + 1) for i, s in enumerate(limbs_to_ints(raw))) * Rinv % curve.r
    assert unpack_points(curve, group, ref)[0] == G.mul(G.gen, total)
    sliced = 0
    for budget in BUDGETS:
        monkeypatch.setenv("B2S_MSM_ROUND_BUDGET", budget)
        l0 = be.launches
        got = fn(bases, s_t, n, mont=True)
        sliced += be.launches - l0 > one_piece       # every slice runs its own rounds
        assert np.array_equal(got, ref), budget
    assert sliced >= 2


@pytest.mark.parametrize("group", [1, 2])
def test_sliced_heavy_lists(be, monkeypatch, group):
    """The heavy lists of the multiplicity-aware front end (eight buckets at most) through sliced rounds."""
    monkeypatch.setenv("B2S_MSM_DEDUP_MIN", "1")
    monkeypatch.setenv("B2S_MSM_AFFINE_ROUNDS", "2")
    curve = CURVES[be.curve]
    G = groups(curve)[group - 1]
    rng = random.Random(0x4EA + group)
    pool = [G.mul(G.gen, rng.randrange(1, curve.r)) for _ in range(16)]
    n = 200
    bases = [pool[rng.randrange(len(pool))] for _ in range(n)]
    vals = [rng.randrange(curve.r) for _ in range(4)]
    scalars = [vals[i % 4] if i % 10 < 8 else rng.randrange(curve.r) for i in range(n)]
    exp = omsm.msm_pippenger(G, bases, scalars)
    B, S = pack_points(curve, group, bases), pack_fr(curve, scalars)
    fn = be.msm_g1 if group == 1 else be.msm_g2
    for budget in ("20000", "5000"):
        monkeypatch.setenv("B2S_MSM_ROUND_BUDGET", budget)
        assert unpack_points(curve, group, fn(B, S, n))[0] == exp, budget


@pytest.mark.parametrize("table", [False, True], ids=["plain", "h_query_table"])
def test_sliced_rounds_in_batched_proofs(be, monkeypatch, table):
    """msm_run_batch (K scalar vectors as one bucket structure) and single proofs with sliced rounds give the proofs of
    unsliced ones, with and without the h-query table."""
    monkeypatch.setenv("B2S_MSM_AFFINE_ROUNDS", "2")
    if table:
        monkeypatch.setenv("B2S_PK_PRECOMP_MIN", "1")
        monkeypatch.setenv("B2S_MSM_PRE_C", "7")
    curve = CURVES[be.curve]
    rng = random.Random(0x511CE + be.curve)
    _, mats, inst, wit = list(circuits(curve))[-1]
    m, pkh, _vk, _keep = gpu_key(be, curve, mats, len(inst), len(wit), rng.randrange(1 << 30))
    K = 4
    z = random_z(curve, rng, K, len(inst) + len(wit))
    r, s = rs_with_zeros(curve, rng, K)
    ref = be.groth16_prove_batch(pkh, m, z, r, s)
    assert_same(ref, singles(be, pkh, m, len(inst), z, r, s, range(K)), range(K))
    for budget in ("200000", "20000"):
        monkeypatch.setenv("B2S_MSM_ROUND_BUDGET", budget)
        assert_same(be.groth16_prove_batch(pkh, m, z, r, s), singles(be, pkh, m, len(inst), z, r, s, range(K)), range(K))
        got = be.groth16_prove_batch(pkh, m, z, r, s)
        assert all(np.array_equal(x, y) for x, y in zip(got, ref)), budget
    be.pk_free(pkh)
    be.r1cs_free(m)
