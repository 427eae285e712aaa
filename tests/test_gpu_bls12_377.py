"""BLS12-377 (curve id 2) end to end on the GPU, against the BLS12-377 oracle (tests/bls377_oracle.py): field and group
operations, NTT, MSM, Groth16 setup / prove under both QAP reductions, serialization, decoding and its rejections, the
pairing, the three verifiers, the constraint checks, and a 2^24 DummyCircuit proof checked with the oracle's pairing."""
import random

import numpy as np
import pytest

from oracle import groth16 as og
from oracle import msm as omsm
from oracle import ntt as ontt
from oracle import r1cs as orc
from tests import bls377_oracle as b7
from tests.bls377_oracle import BLS12_377 as CURVE
from tests.circom_oracle import witness_map_circom
from tests.util import csr_from_rows, limbs_to_ints, pack_fr, pack_points, pack_u32, random_fr_limbs, unpack_fr, unpack_points

pytestmark = pytest.mark.gpu
P, R = b7.P, b7.R


@pytest.fixture(scope="module")
def be():
    from snark_b200 import Backend

    b = Backend(curve=2)
    yield b
    b.close()


def test_sizes_and_ids(be):
    from snark_b200 import lib as L

    assert L.BLS12_377 == 2 and L.FR_MODULUS[2] == R
    assert (be.fr_bytes, be.fq_bytes, be.g1_bytes, be.g2_bytes) == (32, 48, 96, 192)


def test_field_and_group_ops(be):
    rng = random.Random(0xF1)
    for field, m, n in ((0, P, 12), (1, R, 8)):
        Rm = 1 << (32 * n)
        xs = [0, 1, m - 1] + [rng.randrange(m) for _ in range(61)]
        ys = [rng.randrange(m) for _ in xs]
        a, b = pack_u32([x * Rm % m for x in xs], n), pack_u32([y * Rm % m for y in ys], n)
        ri = pow(Rm, -1, m)
        for op, f in [(0, lambda x, y: x * y), (1, lambda x, y: x + y), (2, lambda x, y: x - y),
                      (3, lambda x, y: pow(x, -1, m) if x else 0), (7, lambda x, y: x * x)]:
            got = [v * ri % m for v in limbs_to_ints(be.field_op(field, op, a, b), n)]
            assert got == [f(x, y) % m for x, y in zip(xs, ys)], (field, op)
    for group in (1, 2):
        G = b7.groups()[group - 1]
        A = [G.mul(G.gen, rng.randrange(1, R)) for _ in range(8)]
        B = [G.mul(G.gen, rng.randrange(1, R)) for _ in range(8)]
        ks = [rng.randrange(R) for _ in A]
        a, b, k = pack_points(CURVE, group, A), pack_points(CURVE, group, B), pack_u32(ks, 8)
        assert unpack_points(CURVE, group, be.group_op(group, 0, a, b, k)) == [G.add(x, y) for x, y in zip(A, B)]
        assert unpack_points(CURVE, group, be.group_op(group, 2, a, b, k)) == [G.dbl(x) for x in A]
        assert unpack_points(CURVE, group, be.group_op(group, 3, a, b, k)) == [G.mul(x, kk) for x, kk in zip(A, ks)]


def test_ntt(be):
    rng = random.Random(0x17)
    xs = [rng.randrange(R) for _ in range(64)]
    w = CURVE.omega(6)
    assert unpack_fr(CURVE, be.ntt(pack_fr(CURVE, xs), 6)) == [sum(x * pow(w, i * j, R) for j, x in enumerate(xs)) % R
                                                              for i in range(64)]
    assert unpack_fr(CURVE, be.ntt(pack_fr(CURVE, xs), 6, coset=True)) == ontt.coset_ntt(CURVE, xs)
    nrng = np.random.default_rng(5)
    for log_n in (12, 24):
        a = random_fr_limbs(nrng, 1 << log_n, bits=252)
        f = be.ntt(a.copy(), log_n)
        assert not np.array_equal(f, a)
        assert np.array_equal(be.ntt(f, log_n, inverse=True), a), log_n


def test_msm_small(be):
    rng = random.Random(0x35)
    for group in (1, 2):
        G = b7.groups()[group - 1]
        bases = [G.mul(G.gen, rng.randrange(1, R)) for _ in range(48)] + [None]
        sc = [rng.randrange(R) for _ in range(47)] + [0, R - 1]
        fn = be.msm_g1 if group == 1 else be.msm_g2
        assert unpack_points(CURVE, group, fn(pack_points(CURVE, group, bases), pack_fr(CURVE, sc), len(sc)))[0] == \
            omsm.msm_naive(G, bases, sc), group


@pytest.mark.parametrize("log_n", [20, 22])
def test_msm_known_logs(be, log_n):
    """bases k_i G from the fixed-base kernel; MSM = (sum k_i s_i) G for uniform, all-equal and few-heavy-value scalars"""
    n = 1 << log_n
    nrng = np.random.default_rng(log_n)
    k = random_fr_limbs(nrng, n, bits=252)
    kv = limbs_to_ints(k)
    G1 = b7.groups()[0]
    bases = be.fixed_base(1, k, n, mont=False)
    uni = random_fr_limbs(nrng, n, bits=252)
    eq = np.tile(uni[:8], n)
    heavy = uni.reshape(n, 8)[nrng.integers(0, 5, size=n)].reshape(-1).copy()
    for name, s in (("uniform", uni), ("all-equal", eq), ("few-heavy", heavy)):
        sv = limbs_to_ints(s)
        want = G1.mul(G1.gen, sum(a * b for a, b in zip(kv, sv)) % R)
        assert unpack_points(CURVE, 1, be.msm_g1(bases, s, n, mont=False))[0] == want, name


def circuits():
    cs2 = orc.circuit2(CURVE, 1, 1, 2)
    cs2.finalize()
    yield "circuit2", cs2.to_matrices(), cs2.instance_assignment, cs2.witness_assignment
    d = orc.dummy_circuit(CURVE, 3, 5, 16, 16)
    yield "dummy16", d.to_matrices(), d.instance_assignment, d.witness_assignment
    bc = orc.bench_circuit(CURVE, 25, seed=5)
    bc.finalize()
    assert bc.is_satisfied()
    yield "bench25", bc.to_matrices(), bc.instance_assignment, bc.witness_assignment


def setup_key(be, rng, mats, inst, wit, qap=0):
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(CURVE, mt) for mt in mats])
    td = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = be.groth16_setup(m, pack_fr(CURVE, td), len(inst), qap=qap)
    return m, pk, vk, td


def vk_points(vk, n_inst):
    return dict(alpha_g1=unpack_points(CURVE, 1, vk["alpha_g1"])[0], beta_g2=unpack_points(CURVE, 2, vk["beta_g2"])[0],
                gamma_g2=unpack_points(CURVE, 2, vk["gamma_g2"])[0], delta_g2=unpack_points(CURVE, 2, vk["delta_g2"])[0],
                gamma_abc_g1=unpack_points(CURVE, 1, vk["gamma_abc_g1"])[:n_inst])


def proof_points(a, b, c):
    return unpack_points(CURVE, 1, a)[0], unpack_points(CURVE, 2, b)[0], unpack_points(CURVE, 1, c)[0]


def test_witness_maps(be):
    for name, mats, inst, wit in circuits():
        m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(CURVE, mt) for mt in mats])
        z = list(inst) + list(wit)
        assert unpack_fr(CURVE, be.witness_map(m, pack_fr(CURVE, z))) == og.witness_map(CURVE, mats, z, len(inst)), name
        assert unpack_fr(CURVE, be.witness_map(m, pack_fr(CURVE, z), qap=1)) == witness_map_circom(CURVE, mats, z, len(inst)), name
        be.r1cs_free(m)
    # the distributed schedule with G = 2 and 4 virtual ranks on this GPU, on a domain of 2^10
    mats, inst, wit = orc.dummy_circuit_direct(CURVE, 3, 5, 1000, 999)
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(CURVE, mt) for mt in mats])
    assert be.domain_size(m) == 1024
    z = pack_fr(CURVE, list(inst) + list(wit))
    for log_ranks in (1, 2):
        assert np.array_equal(be.witness_map_sim(m, z, log_ranks), be.witness_map(m, z)), log_ranks
    be.r1cs_free(m)


def test_witness_map_2p20_identity(be):
    """h of a 2^20-domain DummyCircuit-shaped R1CS: h(tau) Z(tau) = a(tau) b(tau) - c(tau) at a random tau, with a, b, c
    the interpolants of the rows (plus the instance rows of a) that the big-int oracle would build"""
    n = (1 << 20) - 2
    a_, b_ = 3, 5
    csr, zi, zw = dummy_csr(n, a_, b_, n - 1)
    m = be.r1cs_upload(n, 2, n - 1, csr)
    N = og.domain_size(n, 2)
    assert N == 1 << 20 and be.domain_size(m) == N
    h = limbs_to_ints(be.witness_map(m, np.concatenate([zi, zw])))
    rinv = pow(1 << 256, -1, R)
    tau = random.Random(0x2020).randrange(R)
    acc = 0
    for c in reversed(h):
        acc = (acc * tau + c * rinv) % R
    u = og.lagrange_at_tau(CURVE, N, tau)
    su = sum(u[: n - 1]) % R                   # rows 0 .. n-2: x2 * x3 = x1; row n-1 is empty
    at = (a_ * su + u[n] * 1 + u[n + 1] * (a_ * b_)) % R
    bt, ct = b_ * su % R, a_ * b_ * su % R
    assert acc * (pow(tau, N, R) - 1) % R == (at * bt - ct) % R
    be.r1cs_free(m)


@pytest.mark.parametrize("qap", [0, 1], ids=["libsnark", "circom"])
def test_setup_prove_verify(be, qap):
    """GPU setup and proofs: accepted by the oracle's pairing, equal to the oracle prover's under the same trapdoor and
    randomness (libsnark reduction); prove_resident and prove_batch give the same bits as prove"""
    import torch

    rng = random.Random(0x9A + qap)
    E = b7.engine()
    for name, mats, inst, wit in circuits():
        m, pk, vk, td = setup_key(be, rng, mats, inst, wit, qap)
        rr, ss = rng.randrange(R), rng.randrange(R)
        zi, zw = pack_fr(CURVE, inst), pack_fr(CURVE, wit)
        a, b, c = be.groth16_prove(pk, m, zi, zw, pack_fr(CURVE, [rr]), pack_fr(CURVE, [ss]))
        vkp = vk_points(vk, len(inst))
        prf = proof_points(a, b, c)
        assert E.groth16_verify(vkp, list(inst[1:]), prf), name
        if qap == 0:
            opk = og.setup(CURVE, mats, len(inst), len(wit), og.Trapdoor(*td))
            assert og.prove(opk, mats, inst, wit, rr, ss)[:3] == prf, name
        z_dev = torch.from_numpy(np.concatenate([zi, zw]).view(np.int32)).cuda()
        ra, rb, rc = be.groth16_prove_resident(pk, m, z_dev, pack_fr(CURVE, [rr]), pack_fr(CURVE, [ss]))
        assert np.array_equal(ra, a) and np.array_equal(rb, b) and np.array_equal(rc, c), name
        K = 3
        rs = [rng.randrange(R) for _ in range(2 * K)]
        zb = np.tile(np.concatenate([zi, zw]), K)
        ba, bb, bc = be.groth16_prove_batch(pk, m, zb, pack_fr(CURVE, rs[:K]), pack_fr(CURVE, rs[K:]))
        for i in range(K):
            sa, sb, sc = be.groth16_prove(pk, m, zi, zw, pack_fr(CURVE, [rs[i]]), pack_fr(CURVE, [rs[K + i]]))
            assert np.array_equal(ba[i], sa) and np.array_equal(bb[i], sb) and np.array_equal(bc[i], sc), (name, i)
        be.pk_free(pk)
        be.r1cs_free(m)


def test_shard_finish(be):
    """two base-range shards + b2s_groth16_finish give the oracle's proof"""
    from snark_b200.lib import PkDesc
    from tests.util import make_pk_desc

    rng = random.Random(0x5D)
    mats, inst, wit = orc.dummy_circuit_direct(CURVE, rng.randrange(R), rng.randrange(R), 20, 20)
    opk = og.setup(CURVE, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, R) for _ in range(5)]))
    rr, ss = rng.randrange(R), rng.randrange(R)
    want = og.prove(opk, mats, inst, wit, rr, ss)[:3]
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(CURVE, mt) for mt in mats])
    keep = []
    full = make_pk_desc(CURVE, opk, keep)
    handles, p1, p2 = [], [], []
    for idx in range(2):
        d = PkDesc()
        for f in ("n_instance", "n_witness", "domain_size", "alpha_g1", "beta_g1", "delta_g1", "beta_g2", "delta_g2"):
            setattr(d, f, getattr(full, f))
        for q, off, ln, sz in (("a_query", "a_off", "a_len", be.g1_bytes), ("b_g1_query", "b1_off", "b1_len", be.g1_bytes),
                               ("b_g2_query", "b2_off", "b2_len", be.g2_bytes), ("h_query", "h_off", "h_len", be.g1_bytes),
                               ("l_query", "l_off", "l_len", be.g1_bytes)):
            total = getattr(full, ln)
            lo, hi = total * idx // 2, total * (idx + 1) // 2
            setattr(d, q, getattr(full, q) + lo * sz)
            setattr(d, off, lo)
            setattr(d, ln, hi - lo)
        handles.append(be.pk_upload(d))
        g1, g2 = be.groth16_prove_shard(handles[-1], m, pack_fr(CURVE, inst), pack_fr(CURVE, wit), pack_fr(CURVE, [rr]),
                                        pack_fr(CURVE, [ss]))
        p1.append(g1)
        p2.append(g2)
    a, b, c = be.groth16_finish(handles[0], np.concatenate(p1), np.concatenate(p2), 2, pack_fr(CURVE, [rr]), pack_fr(CURVE, [ss]))
    assert proof_points(a, b, c) == want
    for h in handles:
        be.pk_free(h)
    be.r1cs_free(m)


def test_serialization_round_trips(be):
    """points, proofs, vk and pk in both modes and both validate settings, against the oracle's SWFlags bytes"""
    rng = random.Random(0x5E)
    for group in (1, 2):
        G = b7.groups()[group - 1]
        pts = [None, G.gen] + [G.mul(G.gen, rng.randrange(1, R)) for _ in range(30)]
        arr = pack_points(CURVE, group, pts)
        for compressed in (True, False):
            blob = be.serialize_points(group, arr, len(pts), compressed)
            assert blob == b"".join(b7.encode_point(group, p, compressed) for p in pts), (group, compressed)
            for validate in (True, False):
                assert np.array_equal(be.deserialize_points(group, blob, compressed=compressed, validate=validate), arr)
    bc = orc.bench_circuit(CURVE, 20, seed=2)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    m, pk, vk, _ = setup_key(be, rng, mats, inst, wit)
    a, b, c = be.groth16_prove(pk, m, pack_fr(CURVE, inst), pack_fr(CURVE, wit), pack_fr(CURVE, [5]), pack_fr(CURVE, [7]))
    prf = proof_points(a, b, c)
    vkp = vk_points(vk, len(inst))
    for compressed in (True, False):
        pb = be.proof_bytes(a, b, c, compressed)
        assert pb == b"".join(b7.encode_point(g, p, compressed) for g, p in zip((1, 2, 1), prf))
        for validate in (True, False):
            assert proof_points(*be.proof_from_bytes(pb, compressed, validate)) == prf
        vb = be.vk_bytes(vk["alpha_g1"], vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"], vk["gamma_abc_g1"], len(inst), compressed)
        want = b"".join([b7.encode_point(1, vkp["alpha_g1"], compressed)] +
                        [b7.encode_point(2, vkp[k], compressed) for k in ("beta_g2", "gamma_g2", "delta_g2")] +
                        [len(inst).to_bytes(8, "little")] + [b7.encode_point(1, p, compressed) for p in vkp["gamma_abc_g1"]])
        assert vb == want
        vk2, used = be.vk_from_bytes(vb, compressed)
        assert used == len(vb) and all(np.array_equal(vk2[k], vk[k]) for k in vk)
        kb = be.pk_bytes(pk, vb, compressed)
        for validate in (True, False):
            pk2 = be.pk_from_bytes(kb, compressed, validate)
            assert be.pk_bytes(pk2, vb, compressed) == kb
            a2, b2, c2 = be.groth16_prove(pk2, m, pack_fr(CURVE, inst), pack_fr(CURVE, wit), pack_fr(CURVE, [5]), pack_fr(CURVE, [7]))
            assert np.array_equal(a2, a) and np.array_equal(b2, b) and np.array_equal(c2, c)
            be.pk_free(pk2)
    be.pk_free(pk)
    be.r1cs_free(m)


def test_malformed_encodings_rejected(be):
    """every rejection class through deserialize_points (an error) and verify_batch_bytes (the reason code)"""
    from snark_b200.lib import B2SError

    rng = random.Random(0xBAD)
    G1, G2 = b7.groups()
    off1 = b7.torsion_point(1, 13, rng)
    off2 = b7.mul_unreduced(G2, b7.random_curve_point(2, rng), R)
    for group, off in ((1, off1), (2, off2)):
        G = b7.groups()[group - 1]
        for compressed in (True, False):
            good = b7.encode_point(group, G.gen, compressed)
            bad = []
            e = bytearray(good); e[-1] |= 0xC0; bad.append(bytes(e))
            e = bytearray(good); e[-1] |= 0x04; bad.append(bytes(e))                    # bit 378: non-canonical
            bad.append(b7.encode_point(group, off, compressed))
            for blob in bad:
                with pytest.raises(B2SError):
                    be.deserialize_points(group, blob, compressed=compressed, validate=True)
            assert unpack_points(CURVE, group, be.deserialize_points(group, bad[-1], compressed=compressed, validate=False)) == [off]
    # through the bytes verifier: proof 1's C off the subgroup (reason 16 * 3 + 4), proof 2's A non-canonical (16 + 2)
    bc = orc.circuit2(CURVE, 1, 1, 2)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    m, pk, vk, _ = setup_key(be, rng, mats, inst, wit)
    pvk = be.vk_prepare(vk)
    proofs = [be.groth16_prove(pk, m, pack_fr(CURVE, inst), pack_fr(CURVE, wit), pack_fr(CURVE, [rng.randrange(R)]),
                               pack_fr(CURVE, [rng.randrange(R)])) for _ in range(3)]
    for compressed in (True, False):
        blobs = [bytearray(be.proof_bytes(*p, compressed)) for p in proofs]
        g1 = 48 * (1 if compressed else 2)
        blobs[1][-g1:] = b7.encode_point(1, off1, compressed)
        blobs[2][g1 - 1] |= 0x08
        inputs = pack_fr(CURVE, list(inst[1:]) * 3)
        ok, reason = be.groth16_verify_batch_bytes(pvk, inputs, len(inst) - 1, b"".join(blobs), compressed)
        assert ok.tolist() == [True, False, False] and reason.tolist() == [0, 16 * 3 + 4, 16 + 2]
    be.pvk_free(pvk)
    be.pk_free(pk)
    be.r1cs_free(m)


def test_pairing(be):
    rng = random.Random(0xE2)
    G1, G2 = b7.groups()
    Ps = [G1.gen, G1.mul(G1.gen, rng.randrange(R)), None, G1.gen]
    Qs = [G2.gen, G2.mul(G2.gen, rng.randrange(R)), G2.gen, None]
    got = b7.gt_to_oracle(be.pairing(pack_points(CURVE, 1, Ps), pack_points(CURVE, 2, Qs)))
    E = b7.engine()
    for i in range(2):
        assert got[i] == E.pairing(Ps[i], Qs[i]).pow(b7.K), i
    assert got[2] == E.Fq12.one() and got[3] == E.Fq12.one()


def test_verifiers(be):
    """verify_batch, the RLC check and both byte forms: a valid batch is accepted, a broken proof caught"""
    rng = random.Random(0x7E)
    d = orc.dummy_circuit(CURVE, 3, 5, 16, 16)
    mats, inst, wit = d.to_matrices(), d.instance_assignment, d.witness_assignment
    m, pk, vk, _ = setup_key(be, rng, mats, inst, wit)
    pvk = be.vk_prepare(vk)
    n = 6
    prf = [be.groth16_prove(pk, m, pack_fr(CURVE, inst), pack_fr(CURVE, wit), pack_fr(CURVE, [rng.randrange(R)]),
                            pack_fr(CURVE, [rng.randrange(R)])) for _ in range(n)]
    a, b, c = (np.concatenate([p[i] for p in prf]) for i in range(3))
    ni = len(inst) - 1
    inputs = pack_fr(CURVE, list(inst[1:]) * n)
    assert be.groth16_verify_batch(pvk, inputs, ni, a, b, c).all()
    assert be.groth16_verify_all(pvk, inputs, ni, a, b, c)
    blob = b"".join(be.proof_bytes(*p) for p in prf)
    ok, reason = be.groth16_verify_batch_bytes(pvk, inputs, ni, blob)
    assert ok.all() and not reason.any()
    assert be.groth16_verify_all_bytes(pvk, inputs, ni, blob)[0]
    bad = inputs.copy()
    bad[3 * ni * 8] ^= 1                                           # proof 3's first input changed
    assert be.groth16_verify_batch(pvk, bad, ni, a, b, c).tolist() == [True] * 3 + [False] + [True] * 2
    assert not be.groth16_verify_all(pvk, bad, ni, a, b, c)
    ok, reason = be.groth16_verify_batch_bytes(pvk, bad, ni, blob)
    assert ok.tolist() == [True] * 3 + [False] + [True] * 2 and not reason.any()
    assert not be.groth16_verify_all_bytes(pvk, bad, ni, blob)[0]
    be.pvk_free(pvk)
    be.pk_free(pk)
    be.r1cs_free(m)


def test_constraint_checks(be):
    """r1cs_check and gr1cs_check verdicts: a satisfying assignment, and one with a witness of A changed"""
    bc = orc.bench_circuit(CURVE, 30, seed=6)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(CURVE, mt) for mt in mats])
    z = list(inst) + list(wit)
    k = max(col for row in mats[0] for _, col in row)            # a witness that A reads
    zb = z[:k] + [(z[k] + 1) % R] + z[k + 1:]
    ev = lambda k, i, zz: orc.evaluate_constraint(R, mats[k][i], zz)
    bad_rows = [i for i in range(len(mats[0])) if ev(0, i, zb) * ev(1, i, zb) % R != ev(2, i, zb)]
    assert bad_rows
    zz = np.stack([pack_fr(CURVE, z), pack_fr(CURVE, zb)])
    first, count = be.r1cs_check(m, zz)
    assert first[:, 0].tolist() == [0xFFFFFFFFFFFFFFFF, bad_rows[0]] and count[:, 0].tolist() == [0, len(bad_rows)]
    g = be.gr1cs_upload(len(inst), len(wit), {"r1cs": (3, [(1, [(0, 1), (1, 1)]), (R - 1, [(2, 1)])], mats)})
    assert be.which_is_unsatisfied(g, pack_fr(CURVE, z)) is None
    assert be.which_is_unsatisfied(g, pack_fr(CURVE, zb)) == ("r1cs", bad_rows[0])
    be.gr1cs_free(g)
    be.r1cs_free(m)


def dummy_csr(n_rows, a, b, n_wit):
    """the DummyCircuit shape of tests/test_gpu_fullsize.py: rows (x2) * (x3) = (x1) with x2 = a, x3 = b"""
    one = pack_fr(CURVE, [1])
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    coeff = np.tile(one, nnz)
    csr = [(row_ptr, np.full(nnz, col, dtype=np.uint32), coeff) for col in (2, 3, 1)]
    z_inst = pack_fr(CURVE, [1, a * b % R])
    z_wit = np.tile(pack_fr(CURVE, [a]), n_wit)
    z_wit[8:16] = pack_fr(CURVE, [b])
    return csr, z_inst, z_wit


def test_dummy_2p24_proof(be):
    """a 2^24 DummyCircuit proof with a GPU-made key: accepted by the oracle's pairing and by the GPU verifier, and a proof
    with a changed public input rejected by both"""
    rng = random.Random(0x24)
    n = 1 << 24
    a_, b_ = 3, 5
    csr, zi, zw = dummy_csr(n, a_, b_, n - 1)
    m = be.r1cs_upload(n, 2, n - 1, csr)
    td = [rng.randrange(1, R) for _ in range(5)]
    pk, vk = be.groth16_setup(m, pack_fr(CURVE, td), 2)
    a, b, c = be.groth16_prove(pk, m, zi, zw, pack_fr(CURVE, [rng.randrange(R)]), pack_fr(CURVE, [rng.randrange(R)]))
    E = b7.engine()
    vkp = vk_points(vk, 2)
    assert E.groth16_verify(vkp, [a_ * b_ % R], proof_points(a, b, c))
    assert not E.groth16_verify(vkp, [a_ * b_ % R + 1], proof_points(a, b, c))
    pvk = be.vk_prepare(vk)
    assert be.groth16_verify_batch(pvk, pack_fr(CURVE, [a_ * b_ % R, a_ * b_ + 1]), 1, np.tile(a, 2), np.tile(b, 2),
                                   np.tile(c, 2)).tolist() == [True, False]
    be.pvk_free(pvk)
    be.pk_free(pk)
    be.r1cs_free(m)
