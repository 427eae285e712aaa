"""Groth16 under ark-circom's CircomReduction (B2S_QAP_CIRCOM) on the GPU: the circom witness map and h query against the
CPU oracle (tests/circom_oracle.py), proofs bit-identical to libsnark-key proofs under the same trapdoor, every prove entry
point, the verifiers, serialization and the error codes."""
import random

import numpy as np
import pytest

from oracle import cnative
from oracle import groth16 as og
from oracle import r1cs as orc
from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests import circom_oracle as oc
from tests.util import csr_from_rows, make_pk_desc, pack_fr, random_fr_limbs, unpack_fr, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
LIB, CIRCOM = 0, 1
CHUNK_CAP = 256


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def circuits(curve):
    cs2 = orc.circuit2(curve, 1, 1, 2)
    cs2.finalize()
    yield "circuit2", cs2.to_matrices(), cs2.instance_assignment, cs2.witness_assignment
    d = orc.dummy_circuit(curve, 3, 5, 16, 16)
    yield "dummy16", d.to_matrices(), d.instance_assignment, d.witness_assignment
    rng = random.Random(17)
    mats, inst, wit = orc.dummy_circuit_direct(curve, rng.randrange(curve.r), rng.randrange(curve.r), 40, 37)
    yield "dummy_direct", mats, inst, wit
    bc = orc.bench_circuit(curve, 25, seed=5)
    bc.finalize()
    yield "bench25", bc.to_matrices(), bc.instance_assignment, bc.witness_assignment


def upload(be, curve, mats, n_inst, n_wit, empty_c=False):
    csr = [csr_from_rows(curve, M) for M in mats]
    if empty_c:   # what a snarkjs key carries: A and B only
        csr[2] = (np.zeros(len(mats[0]) + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32))
    return be.r1cs_upload(len(mats[0]), n_inst, n_wit, csr)


def spoil(curve, wit):
    return [(v + 1) % curve.r for v in wit]


def proof_points(curve, abc):
    a, b, c = abc
    return unpack_points(curve, 1, a)[0], unpack_points(curve, 2, b)[0], unpack_points(curve, 1, c)[0]


def same(p, q):
    return all(np.array_equal(x, y) for x, y in zip(p, q))


def dummy_2k(curve, log_n):
    """DummyCircuit-shaped R1CS at domain 2^log_n (every row z[2] z[3] = z[1]) and a satisfying assignment."""
    N = 1 << log_n
    n_rows, n_inst, n_wit = N - 2, 2, N - 3
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    coeff = np.tile(pack_fr(curve, [1]), nnz)
    csr = [(row_ptr, np.full(nnz, col, dtype=np.uint32), coeff) for col in (2, 3, 1)]
    rng = random.Random(log_n)
    a, b = rng.randrange(curve.r), rng.randrange(curve.r)
    z_inst = pack_fr(curve, [1, a * b % curve.r])
    z_wit = np.tile(pack_fr(curve, [a]), n_wit)
    z_wit[8:16] = pack_fr(curve, [b])
    return csr, n_rows, n_inst, n_wit, z_inst, z_wit


def test_witness_map_matches_oracle(be, monkeypatch):
    """b2s_witness_map_qap(CIRCOM) = the oracle's circom map, satisfying or not, with the full-size NTT tables and (fresh ctx)
    with the composed two-level ones; a handle whose C is empty gives the same h."""
    from snark_b200 import Backend

    curve = CURVES[be.curve]
    fresh = None
    for full in (True, False):
        if not full:
            monkeypatch.setenv("B2S_NTT_FULL", "0")
            fresh = Backend(curve=be.curve)
        b = be if full else fresh
        for name, mats, inst, wit in circuits(curve):
            m = upload(b, curve, mats, len(inst), len(wit))
            m_noc = upload(b, curve, mats, len(inst), len(wit), empty_c=True)
            for w in (wit, spoil(curve, wit)):
                z = list(inst) + list(w)
                want = oc.witness_map_circom(curve, mats, z, len(inst))
                got = b.witness_map(m, pack_fr(curve, z), qap=CIRCOM)
                assert unpack_fr(curve, got) == want, (name, full)
                assert np.array_equal(b.witness_map(m_noc, pack_fr(curve, z), qap=CIRCOM), got), (name, full)
            b.r1cs_free(m)
            b.r1cs_free(m_noc)
    fresh.close()


def test_setup_matches_oracle(be):
    curve = CURVES[be.curve]
    rng = random.Random(0xC5E7 + be.curve)
    for name, mats, inst, wit in list(circuits(curve))[:3]:
        td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
        pk = oc.setup_circom(curve, mats, len(inst), len(wit), td)
        m = upload(be, curve, mats, len(inst), len(wit))
        pkh, vk = be.groth16_setup(m, pack_fr(curve, [td.tau, td.alpha, td.beta, td.gamma, td.delta]), len(inst), qap=CIRCOM)
        n_vars = len(inst) + len(wit)
        assert unpack_points(curve, 1, be.pk_query(pkh, 0, n_vars)) == pk.a_query, name
        assert unpack_points(curve, 1, be.pk_query(pkh, 1, n_vars)) == pk.b_g1_query, name
        assert unpack_points(curve, 2, be.pk_query(pkh, 2, n_vars)) == pk.b_g2_query, name
        assert unpack_points(curve, 1, be.pk_query(pkh, 3, pk.domain)) == pk.h_query, name
        assert unpack_points(curve, 1, be.pk_query(pkh, 4, len(wit))) == pk.l_query, name
        assert unpack_points(curve, 1, be.pk_query(pkh, 5, 3)) == [pk.alpha_g1, pk.beta_g1, pk.delta_g1]
        assert unpack_points(curve, 2, be.pk_query(pkh, 6, 2)) == [pk.beta_g2, pk.delta_g2]
        assert unpack_points(curve, 1, vk["alpha_g1"]) == [pk.alpha_g1]
        assert unpack_points(curve, 2, vk["beta_g2"]) == [pk.beta_g2]
        assert unpack_points(curve, 2, vk["gamma_g2"]) == [pk.gamma_g2]
        assert unpack_points(curve, 2, vk["delta_g2"]) == [pk.delta_g2]
        assert unpack_points(curve, 1, vk["gamma_abc_g1"]) == pk.gamma_abc_g1
        # the oracle's circom proof, which passes its check in the exponent
        rr, ss = rng.randrange(curve.r), rng.randrange(curve.r)
        A, B, C, h = oc.prove_circom(pk, mats, inst, wit, rr, ss)
        assert oc.check_in_exponent(pk, (A, B, C), inst, wit, h, rr, ss)
        got = be.groth16_prove(pkh, m, pack_fr(curve, inst), pack_fr(curve, wit), pack_fr(curve, [rr]), pack_fr(curve, [ss]))
        assert proof_points(curve, got) == (A, B, C), name
        be.pk_free(pkh)
        be.r1cs_free(m)


@pytest.mark.parametrize("log_n", [12, 16, 20])
def test_proofs_bit_identical_to_libsnark(be, monkeypatch, log_n):
    """Same trapdoor, same satisfying z, r, s: the libsnark and the circom key give the same proof bytes, through
    b2s_groth16_prove, _resident and (2^12, 2^16 forced; 2^20 by default) the h-query table.  One key resident at a time."""
    import torch

    curve = CURVES[be.curve]
    rng = random.Random(0xB17 + log_n)
    csr, n_rows, n_inst, n_wit, z_inst, z_wit = dummy_2k(curve, log_n)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    td = pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)])
    R, S = pack_fr(curve, [rng.randrange(curve.r)]), pack_fr(curve, [rng.randrange(curve.r)])
    z_dev = torch.from_numpy(np.concatenate([z_inst, z_wit]).view(np.int32)).cuda()
    tables = [False] if log_n == 20 else [False, True]

    def proofs(qap):
        out = []
        for table in tables:
            if table:
                monkeypatch.setenv("B2S_PK_PRECOMP_MIN", "1")
                monkeypatch.setenv("B2S_MSM_PRE_C", "7")
            pkh, _vk = be.groth16_setup(m, td, n_inst, qap=qap)
            out.append(be.groth16_prove(pkh, m, z_inst, z_wit, R, S))
            out.append(be.groth16_prove_resident(pkh, m, z_dev, R, S))
            be.pk_free(pkh)
            monkeypatch.delenv("B2S_PK_PRECOMP_MIN", raising=False)
            monkeypatch.delenv("B2S_MSM_PRE_C", raising=False)
        return out

    lib, cir = proofs(LIB), proofs(CIRCOM)
    for i, (p, q) in enumerate(zip(lib, cir)):
        assert same(p, q), (log_n, i)
        assert same(p, lib[0]), (log_n, i)
    be.r1cs_free(m)


def test_full_size_bls12_381_known_discrete_logs():
    """Synthetic circom key k_j G at domain 2^24: A, B, C are the multiples of G predicted from z, h and the k_j; h equals
    -2 times the libsnark h evaluated on the odd coset, computed with b2s_witness_map, b2s_poly_geom, b2s_poly_op and
    b2s_ntt."""
    import torch

    from snark_b200 import Backend
    from snark_b200.lib import MEM_DEVICE, MEM_HOST, PkDesc

    curve, cid, log_n = BLS12_381, 0, 24
    r = curve.r
    N = 1 << log_n
    rng = random.Random(0x24C)
    csr, n_rows, n_inst, n_wit, z_inst, z_wit = dummy_2k(curve, log_n)
    n_vars = n_inst + n_wit
    rr, ss = rng.randrange(r), rng.randrange(r)
    be = Backend(curve=cid)
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(4321)

    def query(group, n):
        k = torch.randint(-(1 << 31), (1 << 31) - 1, (n, 8), dtype=torch.int32, device=dev, generator=gen)
        k[:, 7] &= 0x1FFFFFFF
        out = torch.empty(n * (be.g1_bytes if group == 1 else be.g2_bytes) // 4, dtype=torch.int32, device=dev)
        be.fixed_base(group, k, n, mont=False, out=out)
        be.sync()
        return out, k.cpu().numpy().view(np.uint32).reshape(-1)

    consts = [rng.randrange(1, r) for _ in range(3)]
    c1 = be.fixed_base(1, pack_fr(curve, consts, mont=False), 3, mont=False)
    c2 = be.fixed_base(2, pack_fr(curve, consts[1:], mont=False), 2, mont=False)
    g1w, g2w = be.g1_bytes // 4, be.g2_bytes // 4
    c1t = torch.from_numpy(c1.view(np.int32)).to(dev)
    c2t = torch.from_numpy(c2.view(np.int32)).to(dev)
    d = PkDesc()
    d.n_instance, d.n_witness, d.domain_size = n_inst, n_wit, N
    d.alpha_g1, d.beta_g1, d.delta_g1 = c1t.data_ptr(), c1t.data_ptr() + 4 * g1w, c1t.data_ptr() + 8 * g1w
    d.beta_g2, d.delta_g2 = c2t.data_ptr(), c2t.data_ptr() + 4 * g2w
    keep, dl = [], {}
    for name, ln, group, total in (("a_query", "a_len", 1, n_vars), ("b_g1_query", "b1_len", 1, n_vars), ("b_g2_query", "b2_len", 2, n_vars),
                                   ("h_query", "h_len", 1, N), ("l_query", "l_len", 1, n_wit)):
        t, k = query(group, total)
        keep.append(t)
        dl[name] = k
        setattr(d, name, t.data_ptr())
        setattr(d, ln, total)
    pk = be.pk_upload(d, mem=MEM_DEVICE, qap=CIRCOM)
    keep.clear()
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    z_all = np.concatenate([z_inst, z_wit])
    ga, gb, gc = be.groth16_prove(pk, m, z_inst, z_wit, pack_fr(curve, [rr]), pack_fr(curve, [ss]))
    be.pk_free(pk)
    h = be.witness_map(m, z_all, qap=CIRCOM)
    # reference h: -2 * (libsnark h scaled by w2^j, forward transform) with existing entry points only
    hl = be.witness_map(m, z_all)
    w2 = oc.omega2(curve, N)
    pw = np.zeros(N * 8, dtype=np.uint32)
    lib = be.lib
    assert lib.b2s_poly_geom(be.h, pack_fr(curve, [1]).ctypes.data, pack_fr(curve, [w2]).ctypes.data, N, MEM_HOST, pw.ctypes.data) == 0
    one, minus_two = pack_fr(curve, [1]), pack_fr(curve, [r - 2])
    assert lib.b2s_poly_op(be.h, 0, hl.ctypes.data, pw.ctypes.data, one.ctypes.data, hl.ctypes.data, N, MEM_HOST) == 0
    be.ntt(hl, log_n)
    assert lib.b2s_poly_op(be.h, 3, hl.ctypes.data, hl.ctypes.data, minus_two.ctypes.data, hl.ctypes.data, N, MEM_HOST) == 0
    be.sync()
    assert np.array_equal(h, hl), "circom h != -2 * libsnark h on the odd coset"

    def dot(k_canon, scal_mont, n):
        return unpack_fr(curve, cnative.fr_dot(cid, k_canon, scal_mont, n), mont=False)[0]

    za = dot(dl["a_query"], z_all, n_vars)
    zb1 = dot(dl["b_g1_query"], z_all, n_vars)
    zb2 = dot(dl["b_g2_query"], z_all, n_vars)
    wl = dot(dl["l_query"], z_wit, n_wit)
    hh = dot(dl["h_query"], h, N)
    alpha, beta, delta = consts
    a_star = (alpha + za + rr * delta) % r
    b1_star = (beta + zb1 + ss * delta) % r
    b2_star = (beta + zb2 + ss * delta) % r
    c_star = (ss * a_star + rr * b1_star - rr * ss % r * delta + wl + hh) % r
    G1, G2 = groups(curve)
    assert unpack_points(curve, 1, ga)[0] == G1.mul(G1.gen, a_star)
    assert unpack_points(curve, 2, gb)[0] == G2.mul(G2.gen, b2_star)
    assert unpack_points(curve, 1, gc)[0] == G1.mul(G1.gen, c_star)
    be.r1cs_free(m)
    be.close()


def test_verifiers_accept_circom_proofs(be):
    """Proofs under a GPU-generated circom key pass b2s_groth16_verify_batch and _rlc; the proof of an unsatisfying
    assignment is rejected."""
    curve = CURVES[be.curve]
    rng = random.Random(0x7E + be.curve)
    a_all, b_all, c_all, xs, expect = [], [], [], [], []
    for name, mats, inst, wit in list(circuits(curve))[1:3]:
        m = upload(be, curve, mats, len(inst), len(wit))
        pkh, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), len(inst), qap=CIRCOM)
        pvk = be.vk_prepare(vk)
        proofs, ins = [], []
        for w, ok in ((wit, True), (spoil(curve, wit), False), (wit, True)):
            R, S = pack_fr(curve, [rng.randrange(curve.r)]), pack_fr(curve, [rng.randrange(curve.r)])
            proofs.append(be.groth16_prove(pkh, m, pack_fr(curve, inst), pack_fr(curve, w), R, S))
            ins.append(pack_fr(curve, inst[1:]))
            expect.append(ok)
        a, b, c = (np.concatenate([p[i] for p in proofs]) for i in range(3))
        x = np.concatenate(ins)
        got = be.groth16_verify_batch(pvk, x, len(inst) - 1, a, b, c)
        assert got.tolist() == [True, False, True], name
        good = [0, 2]
        ag, bg, cg = (np.concatenate([proofs[i][j] for i in good]) for j in range(3))
        assert be.groth16_verify_all(pvk, np.concatenate([ins[i] for i in good]), len(inst) - 1, ag, bg, cg)
        assert not be.groth16_verify_all(pvk, x, len(inst) - 1, a, b, c)
        be.pvk_free(pvk)
        be.pk_free(pkh)
        be.r1cs_free(m)


def random_z(curve, rng, K, n_vars):
    z = random_fr_limbs(np.random.default_rng(rng.randrange(1 << 30)), K * n_vars, bits=253).reshape(K, n_vars, 8)
    z[:, 0] = pack_fr(curve, [1])
    return z.reshape(K, n_vars * 8)


def singles(be, pkh, m, n_inst, z, r, s, idx):
    out = []
    for i in idx:
        row = z[i]
        out.append(be.groth16_prove(pkh, m, np.ascontiguousarray(row[: 8 * n_inst]), np.ascontiguousarray(row[8 * n_inst:]),
                                    np.ascontiguousarray(r[8 * i: 8 * i + 8]), np.ascontiguousarray(s[8 * i: 8 * i + 8])))
    return out


def test_prove_batch_equals_single_proofs(be):
    """b2s_groth16_prove_batch with a circom key: K = 1, 7, 33 and two chunk boundaries equal single circom proofs, host and
    device buffers."""
    import torch

    curve = CURVES[be.curve]
    rng = random.Random(0xBA + be.curve)
    for name, mats, inst, wit in list(circuits(curve))[:2]:
        n_inst, n_wit = len(inst), len(wit)
        m = upload(be, curve, mats, n_inst, n_wit)
        pkh, _vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst, qap=CIRCOM)
        for K in (1, 7, 33, 2 * CHUNK_CAP + 3):
            z = random_z(curve, rng, K, n_inst + n_wit)
            if K == 7:
                z[3] = pack_fr(curve, list(inst) + list(wit))       # one satisfying row
            r = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
            s = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
            got = be.groth16_prove_batch(pkh, m, z, r, s)
            idx = list(range(K)) if K < 64 else sorted({0, CHUNK_CAP - 1, CHUNK_CAP, 2 * CHUNK_CAP - 1, 2 * CHUNK_CAP, K - 1})
            for i, ref in zip(idx, singles(be, pkh, m, n_inst, z, r, s, idx)):
                assert same((got[0][i], got[1][i], got[2][i]), ref), (name, K, i)
            if K == 33:
                t = [torch.from_numpy(x.view(np.int32)).cuda() for x in (z, r, s)]
                dev = be.groth16_prove_batch(pkh, m, *t)
                for h_, d_ in zip(got, dev):
                    assert np.array_equal(h_, d_.cpu().numpy().view(np.uint32)), name
        be.pk_free(pkh)
        be.r1cs_free(m)


def test_shards_join(be):
    """Two base-range shards of a circom key (the h range a slice of the evaluations) + b2s_groth16_finish = the single
    circom proof."""
    from snark_b200.lib import PkDesc

    curve = CURVES[be.curve]
    rng = random.Random(0x5A + be.curve)
    mats, inst, wit = orc.dummy_circuit_direct(curve, rng.randrange(curve.r), rng.randrange(curve.r), 20, 20)
    td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
    pk = oc.setup_circom(curve, mats, len(inst), len(wit), td)
    rr, ss = rng.randrange(curve.r), rng.randrange(curve.r)
    A, B, C, _ = oc.prove_circom(pk, mats, inst, wit, rr, ss)
    m = upload(be, curve, mats, len(inst), len(wit))
    keep = []
    full = make_pk_desc(curve, pk, keep)
    R, S = pack_fr(curve, [rr]), pack_fr(curve, [ss])
    pkh = be.pk_upload(full, qap=CIRCOM)
    assert proof_points(curve, be.groth16_prove(pkh, m, pack_fr(curve, inst), pack_fr(curve, wit), R, S)) == (A, B, C)
    be.pk_free(pkh)
    g1b, g2b = be.g1_bytes, be.g2_bytes
    parts1, parts2, handles = [], [], []
    for idx in range(2):
        d = PkDesc()
        for f in ("n_instance", "n_witness", "domain_size", "alpha_g1", "beta_g1", "delta_g1", "beta_g2", "delta_g2"):
            setattr(d, f, getattr(full, f))
        for q, off, ln, sz in (("a_query", "a_off", "a_len", g1b), ("b_g1_query", "b1_off", "b1_len", g1b),
                               ("b_g2_query", "b2_off", "b2_len", g2b), ("h_query", "h_off", "h_len", g1b),
                               ("l_query", "l_off", "l_len", g1b)):
            total = getattr(full, ln)
            lo, hi = total * idx // 2, total * (idx + 1) // 2
            setattr(d, q, getattr(full, q) + lo * sz)
            setattr(d, off, lo)
            setattr(d, ln, hi - lo)
        h = be.pk_upload(d, qap=CIRCOM)
        handles.append(h)
        g1, g2 = be.groth16_prove_shard(h, m, pack_fr(curve, inst), pack_fr(curve, wit), R, S)
        parts1.append(g1)
        parts2.append(g2)
    got = be.groth16_finish(handles[0], np.concatenate(parts1), np.concatenate(parts2), 2, R, S)
    assert proof_points(curve, got) == (A, B, C)
    for h in handles:
        be.pk_free(h)
    be.r1cs_free(m)


def test_serialized_key_round_trip(be):
    """circom key -> b2s_pk_serialize -> b2s_pk_deserialize_qap(CIRCOM), compressed and uncompressed, validated: the same
    proofs.  Circom bytes through the libsnark reader and libsnark bytes through the circom reader are malformed."""
    from snark_b200 import B2SError

    curve = CURVES[be.curve]
    rng = random.Random(0x5E + be.curve)
    _, mats, inst, wit = list(circuits(curve))[2]
    m = upload(be, curve, mats, len(inst), len(wit))
    td = pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)])
    R, S = pack_fr(curve, [rng.randrange(curve.r)]), pack_fr(curve, [rng.randrange(curve.r)])
    zi, zw = pack_fr(curve, inst), pack_fr(curve, wit)
    keys = {}
    for qap in (LIB, CIRCOM):
        pkh, vk = be.groth16_setup(m, td, len(inst), qap=qap)
        ref = be.groth16_prove(pkh, m, zi, zw, R, S)
        n_abc = len(vk["gamma_abc_g1"]) * 4 // be.g1_bytes
        for compressed in (True, False):
            vkb = be.vk_bytes(vk["alpha_g1"], vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"], vk["gamma_abc_g1"], n_abc, compressed)
            keys[(qap, compressed)] = be.pk_bytes(pkh, vkb, compressed)
        be.pk_free(pkh)
        if qap == CIRCOM:
            for compressed in (True, False):
                back = be.pk_from_bytes(keys[(CIRCOM, compressed)], compressed=compressed, validate=True, qap=CIRCOM)
                assert same(be.groth16_prove(back, m, zi, zw, R, S), ref), compressed
                be.pk_free(back)
    for data, qap in ((keys[(CIRCOM, True)], LIB), (keys[(LIB, True)], CIRCOM)):
        with pytest.raises(B2SError) as e:
            be.pk_from_bytes(data, qap=qap)
        assert e.value.code == 7 and "dimensions" in str(e.value)
    be.r1cs_free(m)


def test_errors(be):
    from snark_b200 import B2SError

    curve = CURVES[be.curve]
    rng = random.Random(0xE + be.curve)
    _, mats, inst, wit = list(circuits(curve))[2]
    m = upload(be, curve, mats, len(inst), len(wit))
    td = pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)])
    z = pack_fr(curve, list(inst) + list(wit))
    lib = be.lib

    def code(fn):
        with pytest.raises(B2SError) as e:
            fn()
        assert str(e.value).split(": ", 1)[1].strip(), "no message"
        return e.value.code

    # a qap value other than 0 / 1
    assert code(lambda: be.witness_map(m, z, qap=2)) == 16
    assert code(lambda: be.groth16_setup(m, td, len(inst), qap=-1)) == 16
    pk_l = og.setup(curve, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)]))
    keep = []
    d = make_pk_desc(curve, pk_l, keep)
    assert code(lambda: be.pk_upload(d, qap=7)) == 16
    assert code(lambda: be.pk_from_bytes(b"\0" * 64, qap=3)) == 16
    # h_len == N - 1 under circom
    assert code(lambda: be.pk_upload(d, qap=CIRCOM)) == 7
    # tau with tau^(2N) = 1 (tau = w2, a 2N-th root outside H)
    N = be.domain_size(m)
    bad_td = pack_fr(curve, [oc.omega2(curve, N)] + [rng.randrange(1, curve.r) for _ in range(4)])
    assert code(lambda: be.groth16_setup(m, bad_td, len(inst), qap=CIRCOM)) == 3
    # a circom key in the group prover (world 1)
    pkh, _vk = be.groth16_setup(m, td, len(inst), qap=CIRCOM)
    grp = be.group_create(None, 0, 1)
    R = pack_fr(curve, [1])
    assert code(lambda: be.groth16_prove_group(grp, pkh, m, pack_fr(curve, inst), pack_fr(curve, wit), R, R)) == 16
    be.group_destroy(grp)
    # a libsnark key stays a libsnark key: the default entry points are unchanged
    assert lib.b2s_witness_map_qap(be.h, m, z.ctypes.data, 0, LIB, np.zeros(N * 8, dtype=np.uint32).ctypes.data) == 0
    be.pk_free(pkh)
    be.r1cs_free(m)
