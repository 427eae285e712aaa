"""b2s_groth16_prove_batch: n proofs under one key in one call.  The reference for every case is the single-proof path
(b2s_groth16_prove on the same z_i, r_i, s_i), compared bit for bit.  The witness map gives the same field elements for any
assignment, satisfying or not, so random z with z[0] = 1 is a valid input."""
import random

import numpy as np
import pytest

from oracle import groth16 as og
from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests.test_gpu_groth16 import circuits, upload
from tests.util import make_pk_desc, pack_fr, random_fr_limbs, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
CHUNK_CAP = 256       # PROVE_BATCH_CAP in csrc/groth16.cu


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def gpu_key(be, curve, mats, n_inst, n_wit, seed):
    m, keep = upload(be, curve, mats, n_inst, n_wit)
    rng = random.Random(seed)
    pkh, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst)
    return m, pkh, vk, keep


def random_z(curve, rng, K, n_vars):
    """K rows of n_vars Montgomery scalars, z[0] = 1"""
    z = random_fr_limbs(np.random.default_rng(rng.randrange(1 << 30)), K * n_vars, bits=253).reshape(K, n_vars, 8)
    z[:, 0] = pack_fr(curve, [1])
    return z.reshape(K, n_vars * 8)


def singles(be, pkh, m, n_inst, z, r, s, idx):
    out = []
    for i in idx:
        row = z[i]
        a, b, c = be.groth16_prove(pkh, m, np.ascontiguousarray(row[: 8 * n_inst]), np.ascontiguousarray(row[8 * n_inst:]),
                                   np.ascontiguousarray(r[8 * i: 8 * i + 8]), np.ascontiguousarray(s[8 * i: 8 * i + 8]))
        out.append((a, b, c))
    return out


def assert_same(batch, ref, idx):
    a, b, c = batch
    for i, (ra, rb, rc) in zip(idx, ref):
        assert np.array_equal(a[i], ra) and np.array_equal(b[i], rb) and np.array_equal(c[i], rc), i


def rs_with_zeros(curve, rng, K):
    r = [rng.randrange(curve.r) for _ in range(K)]
    s = [rng.randrange(curve.r) for _ in range(K)]
    for i in range(0, K, 3):     # every third proof deterministic (r = s = 0)
        r[i] = s[i] = 0
    return pack_fr(curve, r), pack_fr(curve, s)


def test_random_assignments_match_single_proofs(be):
    curve = CURVES[be.curve]
    rng = random.Random(0xBA7C + be.curve)
    for name, mats, inst, wit in circuits(curve):
        n_inst, n_wit = len(inst), len(wit)
        m, pkh, _vk, _keep = gpu_key(be, curve, mats, n_inst, n_wit, rng.randrange(1 << 30))
        for K in (1, 2, 7, 33):
            z = random_z(curve, rng, K, n_inst + n_wit)
            r, s = rs_with_zeros(curve, rng, K)
            got = be.groth16_prove_batch(pkh, m, z, r, s)
            assert_same(got, singles(be, pkh, m, n_inst, z, r, s, range(K)), range(K))
        be.pk_free(pkh)
        be.r1cs_free(m)


def test_satisfying_assignments_match_the_oracle(be):
    """The circuits' own assignments under an oracle key: the batch gives the oracle's proofs, which pass its check in the
    exponent."""
    curve = CURVES[be.curve]
    rng = random.Random(0x5A7 + be.curve)
    for name, mats, inst, wit in circuits(curve):
        td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
        pk = og.setup(curve, mats, len(inst), len(wit), td)
        m, _keep = upload(be, curve, mats, len(inst), len(wit))
        keep = []
        pkh = be.pk_upload(make_pk_desc(curve, pk, keep))
        K = 3
        rr = [rng.randrange(curve.r) for _ in range(K)]
        ss = [rng.randrange(curve.r) for _ in range(K)]
        z = np.tile(pack_fr(curve, list(inst) + list(wit)), (K, 1))
        a, b, c = be.groth16_prove_batch(pkh, m, z, pack_fr(curve, rr), pack_fr(curve, ss))
        for i in range(K):
            A, B, C, h = og.prove(pk, mats, inst, wit, rr[i], ss[i])
            assert og.check_in_exponent(pk, (A, B, C), inst, wit, h, rr[i], ss[i])
            got = (unpack_points(curve, 1, a[i])[0], unpack_points(curve, 2, b[i])[0], unpack_points(curve, 1, c[i])[0])
            assert got == (A, B, C), (name, i)
        be.pk_free(pkh)
        be.r1cs_free(m)


def dummy_2k(curve, log_n):
    """DummyCircuit-shaped R1CS at domain 2^log_n (every row z[2] * z[3] = z[1]): any witness with z[1] = z[2] z[3] satisfies it."""
    N = 1 << log_n
    n_rows, n_inst, n_wit = N - 2, 2, N - 3
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    coeff = np.tile(pack_fr(curve, [1]), nnz)
    csr = [(row_ptr, np.full(nnz, col, dtype=np.uint32), coeff) for col in (2, 3, 1)]
    return csr, n_rows, n_inst, n_wit


def test_domain_2_16_batch_verifies(be):
    """64 satisfying random witnesses at domain 2^16 under a GPU-generated key: every proof equals its single proof and
    b2s_groth16_verify_batch accepts them all."""
    curve = CURVES[be.curve]
    rng = random.Random(0x216 + be.curve)
    csr, n_rows, n_inst, n_wit = dummy_2k(curve, 16)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    pkh, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst)
    K = 64
    z = random_z(curve, rng, K, n_inst + n_wit).reshape(K, -1, 8)
    xs = []
    for k in range(K):
        a_, b_ = rng.randrange(curve.r), rng.randrange(curve.r)
        z[k, 1], z[k, 2], z[k, 3] = pack_fr(curve, [a_ * b_ % curve.r]), pack_fr(curve, [a_]), pack_fr(curve, [b_])
        xs.append(a_ * b_ % curve.r)
    z = z.reshape(K, -1)
    r, s = rs_with_zeros(curve, rng, K)
    a, b, c = be.groth16_prove_batch(pkh, m, z, r, s)
    idx = [0, 1, 31, 63]
    assert_same((a, b, c), singles(be, pkh, m, n_inst, z, r, s, idx), idx)
    pvk = be.vk_prepare(vk)
    assert be.groth16_verify_batch(pvk, pack_fr(curve, xs), 1, a.reshape(-1), b.reshape(-1), c.reshape(-1)).all()
    # a proof of another statement is rejected
    wrong = pack_fr(curve, [(xs[0] + 1) % curve.r] + xs[1:])
    assert be.groth16_verify_batch(pvk, wrong, 1, a.reshape(-1), b.reshape(-1), c.reshape(-1)).tolist() == [False] + [True] * (K - 1)
    be.pvk_free(pvk)
    be.pk_free(pkh)
    be.r1cs_free(m)


def test_host_and_device_buffers_agree(be):
    import torch

    curve = CURVES[be.curve]
    rng = random.Random(0xDE7 + be.curve)
    _, mats, inst, wit = list(circuits(curve))[3]
    m, pkh, _vk, _keep = gpu_key(be, curve, mats, len(inst), len(wit), 5)
    K = 9
    z = random_z(curve, rng, K, len(inst) + len(wit))
    r, s = rs_with_zeros(curve, rng, K)
    host = be.groth16_prove_batch(pkh, m, z, r, s)
    t = [torch.from_numpy(x.view(np.int32)).cuda() for x in (z, r, s)]
    dev = be.groth16_prove_batch(pkh, m, *t)
    for h, d in zip(host, dev):
        assert np.array_equal(h, d.cpu().numpy().view(np.uint32))
    be.pk_free(pkh)
    be.r1cs_free(m)


@pytest.mark.parametrize("shape", ["same_z", "all_equal", "all_zero"])
def test_skewed_scalars(be, shape):
    """Repeated scalar vectors (the same buckets K times), all-equal witnesses (heavy buckets and the affine rounds of the
    bucket sums at domain 2^14) and all-zero witnesses."""
    curve = CURVES[be.curve]
    rng = random.Random(len(shape) + 7 * be.curve)
    csr, n_rows, n_inst, n_wit = dummy_2k(curve, 14)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    pkh, _vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst)
    K = 12
    n_vars = n_inst + n_wit
    if shape == "same_z":
        z = np.tile(random_z(curve, rng, 1, n_vars), (K, 1))
    else:
        z = np.zeros((K, n_vars, 8), dtype=np.uint32)
        z[:, 0] = pack_fr(curve, [1])
        if shape == "all_equal":
            for k in range(K):
                z[k, 1:] = pack_fr(curve, [rng.randrange(curve.r)])
        z = z.reshape(K, -1)
    r, s = rs_with_zeros(curve, rng, K)
    got = be.groth16_prove_batch(pkh, m, z, r, s)
    idx = [0, 1, 5, K - 1]
    assert_same(got, singles(be, pkh, m, n_inst, z, r, s, idx), idx)
    be.pk_free(pkh)
    be.r1cs_free(m)


@pytest.mark.parametrize("rounds", [None, "2"])
def test_h_query_table(be, monkeypatch, rounds):
    """The fixed-base table of the h query forced on for small keys (K super-windows of one bucket set each), with and
    without the batched-affine rounds."""
    monkeypatch.setenv("B2S_PK_PRECOMP_MIN", "1")
    monkeypatch.setenv("B2S_MSM_PRE_C", "7")
    if rounds:
        monkeypatch.setenv("B2S_MSM_AFFINE_ROUNDS", rounds)
    curve = CURVES[be.curve]
    rng = random.Random(0x7AB + be.curve)
    for name, mats, inst, wit in list(circuits(curve))[1:]:
        m, pkh, _vk, _keep = gpu_key(be, curve, mats, len(inst), len(wit), rng.randrange(1 << 30))
        K = 5
        z = random_z(curve, rng, K, len(inst) + len(wit))
        r, s = rs_with_zeros(curve, rng, K)
        got = be.groth16_prove_batch(pkh, m, z, r, s)
        assert_same(got, singles(be, pkh, m, len(inst), z, r, s, range(K)), range(K))
        be.pk_free(pkh)
        be.r1cs_free(m)


def test_chunk_boundaries(be):
    """More proofs than two chunks hold, at a tiny domain: the first and last proof of every chunk."""
    curve = CURVES[be.curve]
    rng = random.Random(0xC4 + be.curve)
    _, mats, inst, wit = list(circuits(curve))[0]
    m, pkh, _vk, _keep = gpu_key(be, curve, mats, len(inst), len(wit), 9)
    K = 2 * CHUNK_CAP + 7
    z = random_z(curve, rng, K, len(inst) + len(wit))
    r, s = rs_with_zeros(curve, rng, K)
    got = be.groth16_prove_batch(pkh, m, z, r, s)
    idx = sorted({0, CHUNK_CAP - 1, CHUNK_CAP, 2 * CHUNK_CAP - 1, 2 * CHUNK_CAP, K - 1})
    assert_same(got, singles(be, pkh, m, len(inst), z, r, s, idx), idx)
    be.pk_free(pkh)
    be.r1cs_free(m)


def test_launches_do_not_grow_with_the_batch(be):
    curve = CURVES[be.curve]
    rng = random.Random(0x1A + be.curve)
    _, mats, inst, wit = list(circuits(curve))[3]
    m, pkh, _vk, _keep = gpu_key(be, curve, mats, len(inst), len(wit), 3)
    counts = []
    for K in (2, 33, 2):
        z = random_z(curve, rng, K, len(inst) + len(wit))
        r, s = rs_with_zeros(curve, rng, K)
        n0 = be.launches
        be.groth16_prove_batch(pkh, m, z, r, s)
        counts.append(be.launches - n0)
    assert counts[0] == counts[1] == counts[2], counts
    be.pk_free(pkh)
    be.r1cs_free(m)


def test_errors(be):
    import ctypes

    from snark_b200 import B2SError
    from snark_b200.lib import MEM_HOST, PkDesc

    curve = CURVES[be.curve]
    rng = random.Random(0xE4)
    _, mats, inst, wit = list(circuits(curve))[0]
    n_inst, n_wit = len(inst), len(wit)
    m, pkh, _vk, _keep = gpu_key(be, curve, mats, n_inst, n_wit, 4)
    K = 2
    z = random_z(curve, rng, K, n_inst + n_wit)
    r, s = rs_with_zeros(curve, rng, K)
    outs = [np.zeros(K * w, dtype=np.uint32) for w in (be.g1_bytes // 4, be.g2_bytes // 4, be.g1_bytes // 4)]
    P = [o.ctypes.data for o in outs]

    def call(pk=pkh, mm=m, n=K, zz=z.ctypes.data, rr=r.ctypes.data, ss=s.ctypes.data, o=P):
        return be.lib.b2s_groth16_prove_batch(be.h, pk, mm, n, zz, rr, ss, MEM_HOST, *o)

    assert call(pk=None) == 1 and call(mm=None) == 1                       # MissingCs
    assert call(zz=None) == 2 and call(rr=None) == 2 and call(ss=None) == 2  # AssignmentMissing
    for j in range(3):
        o = list(P)
        o[j] = None
        assert call(o=o) == 16                                                 # InvalidArg
    # a shard key: the first half of every query
    keep = []
    d = PkDesc()
    full = {}
    for q, w in (("a_query", 1), ("b_g1_query", 1), ("b_g2_query", 2), ("h_query", 1), ("l_query", 1)):
        full[q] = be.pk_query(pkh, {"a_query": 0, "b_g1_query": 1, "b_g2_query": 2, "h_query": 3, "l_query": 4}[q],
                              {"a_query": n_inst + n_wit, "b_g1_query": n_inst + n_wit, "b_g2_query": n_inst + n_wit,
                               "h_query": be.domain_size(m) - 1, "l_query": n_wit}[q])
    c1, c2 = be.pk_query(pkh, 5, 3), be.pk_query(pkh, 6, 2)
    keep += [c1, c2] + list(full.values())
    d.n_instance, d.n_witness, d.domain_size = n_inst, n_wit, be.domain_size(m)
    d.alpha_g1, d.beta_g1, d.delta_g1 = c1.ctypes.data, c1.ctypes.data + be.g1_bytes, c1.ctypes.data + 2 * be.g1_bytes
    d.beta_g2, d.delta_g2 = c2.ctypes.data, c2.ctypes.data + be.g2_bytes
    for q, off, ln in (("a_query", "a_off", "a_len"), ("b_g1_query", "b1_off", "b1_len"), ("b_g2_query", "b2_off", "b2_len"),
                       ("h_query", "h_off", "h_len"), ("l_query", "l_off", "l_len")):
        per = be.g2_bytes if q == "b_g2_query" else be.g1_bytes
        total = full[q].nbytes // per
        setattr(d, q, full[q].ctypes.data)
        setattr(d, off, 0)
        setattr(d, ln, max(total // 2, 1))
    shard = be.pk_upload(d)
    assert call(pk=shard) == 7                                                  # MalformedVk
    be.pk_free(shard)
    # key and matrices of different dimensions
    _, mats2, inst2, wit2 = list(circuits(curve))[3]
    m2, _k2 = upload(be, curve, mats2, len(inst2), len(wit2))
    assert call(mm=m2) == 2
    be.r1cs_free(m2)
    # n_proofs == 0: OK, nothing written
    for o in outs:
        o[:] = 0xA5A5A5A5
    assert call(n=0) == 0
    assert all((o == 0xA5A5A5A5).all() for o in outs)
    be.pk_free(pkh)
    be.r1cs_free(m)
