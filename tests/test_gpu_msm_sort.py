"""The two-pass digit sort of the MSM (csrc/msm.cu: msm_partition_kernel, msm_place_kernel) on the distributions that reach
its boundaries: coarse bins of several place chunks, bins split over several CTAs, windows left empty, and the fine-key
width F at 0, at small values and at the flagship value.  Bases are (i+1)*G, so MSM(bases, s) == (sum_i s_i (i+1) mod r) * G."""
import numpy as np
import pytest

from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests.util import random_fr_limbs, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


_bases = {}


def known_bases(be, group, n):
    """(i+1)*G for i < n, built on the GPU by the fixed-base kernel (cached per backend, group and size)."""
    import torch

    key = (id(be), group, n)
    if key not in _bases:
        _bases.clear()
        ks = np.zeros((n, 8), dtype=np.uint32)
        ks[:, 0] = np.arange(1, n + 1, dtype=np.uint32)
        pt_bytes = be.g1_bytes if group == 1 else be.g2_bytes
        out = torch.empty(n * pt_bytes // 4, dtype=torch.int32, device="cuda")
        be.fixed_base(group, torch.from_numpy(ks.view(np.int32)).cuda(), n, mont=False, out=out)
        be.sync()
        _bases[key] = out
    return _bases[key]


def weighted_sum(raw, r):
    """sum_i s_i (i+1) mod r for canonical scalars raw (uint32[n*8]), exact in uint64 on 16-bit half-limbs."""
    a = np.asarray(raw, dtype=np.uint32).reshape(-1, 8)
    w = np.arange(1, a.shape[0] + 1, dtype=np.uint64)
    total = 0
    for j in range(8):
        for h in range(2):
            col = ((a[:, j] >> np.uint32(16 * h)) & np.uint32(0xFFFF)).astype(np.uint64)
            total += int(np.dot(col, w)) << (32 * j + 16 * h)
    return total % r


def check(be, group, raw):
    import torch

    curve = CURVES[be.curve]
    G = groups(curve)[group - 1]
    n = raw.size // 8
    fn = be.msm_g1 if group == 1 else be.msm_g2
    s_t = torch.from_numpy(np.ascontiguousarray(raw).view(np.int32)).cuda()
    got = unpack_points(curve, group, fn(known_bases(be, group, n), s_t, n, mont=False))[0]
    assert got == G.mul(G.gen, weighted_sum(raw, curve.r))


@pytest.mark.parametrize("log_n", [20, 22])
def test_sort_uniform_g1(be, log_n):
    check(be, 1, random_fr_limbs(np.random.default_rng(log_n), 1 << log_n, bits=CURVES[be.curve].r.bit_length() - 1))


def test_sort_uniform_g2(be):
    check(be, 2, random_fr_limbs(np.random.default_rng(18), 1 << 18, bits=CURVES[be.curve].r.bit_length() - 1))


@pytest.mark.parametrize("pool", [100, 4])
def test_sort_value_pool(be, pool, monkeypatch):
    """2^22 scalars drawn from a small pool with the multiplicity-aware front end off: buckets of ~42 k entries (several
    place chunks per coarse bin) with 100 values, ~1 M (coarse bins split over several CTAs) with 4."""
    if be.curve != 0:
        pytest.skip("one curve is enough for the bucket structure")
    monkeypatch.setenv("B2S_MSM_DEDUP", "0")
    rng = np.random.default_rng(1000 + pool)
    values = random_fr_limbs(rng, pool, bits=254).reshape(pool, 8)
    check(be, 1, values[rng.integers(0, pool, size=1 << 22)].reshape(-1))


def test_sort_low_window_only(be, monkeypatch):
    """Scalars below 2^c: window 0 takes every entry, window 1 only digit 1 (from the recoding carry of the top half), every
    other window and coarse bin stays empty."""
    if be.curve != 0:
        pytest.skip("one curve is enough for the bucket structure")
    c = 16
    monkeypatch.setenv("B2S_MSM_C", str(c))
    n = 1 << 20
    raw = np.zeros((n, 8), dtype=np.uint32)
    raw[:, 0] = np.random.default_rng(16).integers(0, 1 << c, size=n, dtype=np.uint32)
    check(be, 1, raw.reshape(-1))


@pytest.mark.parametrize("c", [9, 12, 20])
def test_sort_window_sizes(be, c, monkeypatch):
    """c = 9 gives F = 0 (a coarse bin is one bucket), c = 12 a few fine bits, c = 20 the flagship F = 11."""
    if be.curve != 0:
        pytest.skip("one curve is enough for the bucket structure")
    monkeypatch.setenv("B2S_MSM_C", str(c))
    check(be, 1, random_fr_limbs(np.random.default_rng(c), 1 << 20, bits=254))
