"""b2s_r1cs_to_sr1cs / b2s_sr1cs_assignment (Sr1csAdapter::r1cs_to_sr1cs[_with_assignment], relations/src/sr1cs/mod.rs) and
the read-back of GR1CS handles (b2s_gr1cs_info / b2s_gr1cs_export), on all three curves.  The converted handle's export must
equal the numpy restatement (tests/sr1cs_oracle.py, itself pinned to the C++ mirror) in canonical form, for handles from
b2s_r1cs_upload, b2s_r1cs_upload_lcmap and b2s_r1cs_file_load, from the reference's small circuits up to a DummyCircuit
shape of 2^24 rows; the converted assignments must equal the oracle's; b2s_gr1cs_check on the result must agree with
b2s_r1cs_check on the source (row 2i for row i)."""
import ctypes
import random

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests import r1cs_file_oracle as ro
from tests import sr1cs_oracle as so
from tests.bls377_oracle import BLS12_377
from tests.test_sr1cs_oracle import random_r1cs
from tests.util import csr_from_rows, pack_fr

CURVES = [BLS12_381, BN254, BLS12_377]
NOT_FOUND = (1 << 64) - 1
INVALID_ARG = 16
gpu = pytest.mark.gpu


@pytest.fixture(scope="module", params=[0, 1, 2], ids=["bls12_381", "bn254", "bls12_377"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def curve_of(be):
    return CURVES[be.curve]


def assert_structure(be, g, o):
    info = be.gr1cs_info(g)
    assert (info["n_instance"], info["n_witness"]) == (o.n_instance, o.n_witness)
    assert len(info["predicates"]) == 1 and info["predicates"][0][:2] == (2, o.n_rows)
    want = o.matrices()
    for j in range(2):
        got = so.canonical_csr(o.r, *be.gr1cs_export(g, 0, j, info))
        for a, b in zip(got, want[j]):
            assert np.array_equal(a, b), j


def random_z(curve, n, n_vars, seed):
    rng = np.random.default_rng(seed)
    z = rng.integers(0, 1 << 32, size=(n, n_vars, 8), dtype=np.uint32)
    z[:, :, 7] &= (1 << (curve.r.bit_length() - 225)) - 1   # below r
    z[:, 0, :] = pack_fr(curve, [1])
    return z.reshape(n, -1)


def small_cases(curve):
    """(name, csr, n_instance, n_witness, z ints): circuit2, DummyCircuit, random R1CS, BenchCircuit 2^10"""
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    yield "circuit2", cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    mats, inst, wit = orc.dummy_circuit_direct(curve, 3, 5, 12, 9)
    yield "dummy", mats, inst, wit
    for seed in range(4):
        mats, n_inst, z = random_r1cs(curve, 100 + seed)
        yield f"random{seed}", mats, z[:n_inst], z[n_inst:]
    cs = orc.bench_circuit(curve, 1 << 10, seed=3)
    cs.finalize()
    yield "bench1024", cs.to_matrices(), cs.instance_assignment, cs.witness_assignment


def check_assignment_all(be, g, o, z, mem):
    """every element of sr1cs_assignment(z) equals the oracle's"""
    want = o.assignment(z)
    if mem == "device":
        import torch

        zt = torch.from_numpy(z.view(np.int32)).cuda()
        got = be.sr1cs_assignment(g, zt)
        be.sync()
        got = got.cpu().numpy().view(np.uint32)
    else:
        got = be.sr1cs_assignment(g, z)
    assert np.array_equal(got, want)
    return got


def check_verdicts(be, m, g, z, z2):
    """gr1cs_check(g, z2) against r1cs_check(m, z): first' = 2 first, same count"""
    f, n = be.r1cs_check(m, z)
    f2, n2 = be.gr1cs_check(g, z2)
    for a in range(z.shape[0]):
        assert int(f2[a, 0]) == (NOT_FOUND if int(f[a, 0]) == NOT_FOUND else 2 * int(f[a, 0]))
        assert int(n2[a, 0]) == int(n[a, 0])


@gpu
def test_small_circuits_upload(be):
    curve = curve_of(be)
    r = curve.r
    for name, mats, inst, wit in small_cases(curve):
        csr = [csr_from_rows(curve, mm) for mm in mats]
        m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), csr)
        g = be.r1cs_to_sr1cs(m)
        o = so.Sr1cs(r, csr, len(inst))
        assert_structure(be, g, o)
        zs = pack_fr(curve, list(inst) + list(wit)).reshape(1, -1)
        bad = zs.copy()
        bad[0, -8] ^= 1                                     # the last witness changed
        batch = np.concatenate([zs, bad, random_z(curve, 1, zs.shape[1] // 8, 7)])
        for mem in ("host", "device"):
            z2 = check_assignment_all(be, g, o, batch, mem)
        check_verdicts(be, m, g, batch, z2)
        # a z' that did not come from the conversion gets the verdicts the oracle computes on the exported matrices
        if name != "bench1024":
            zr = random_z(curve, 1, g.n_vars, 11)
            f, n = be.gr1cs_check(g, zr)
            info = be.gr1cs_info(g)
            bad_rows = so.check(r, [be.gr1cs_export(g, 0, j, info) for j in range(2)], so.limbs_to_ints(zr[0]))
            assert int(n[0, 0]) == len(bad_rows) and int(f[0, 0]) == (bad_rows[0] if bad_rows else NOT_FOUND), name
        be.gr1cs_free(g)
        be.r1cs_free(m)


@gpu
def test_batches_host_and_device(be):
    curve = curve_of(be)
    cs = orc.bench_circuit(curve, 1 << 10, seed=4)
    cs.finalize()
    mats, inst = cs.to_matrices(), cs.instance_assignment
    csr = [csr_from_rows(curve, mm) for mm in mats]
    n_vars = len(inst) + len(cs.witness_assignment)
    m = be.r1cs_upload(len(mats[0]), len(inst), len(cs.witness_assignment), csr)
    g = be.r1cs_to_sr1cs(m)
    o = so.Sr1cs(curve.r, csr, len(inst))
    for n in (1, 3, 64):
        z = random_z(curve, n, n_vars, n)
        for mem in ("host", "device"):
            check_assignment_all(be, g, o, z, mem)
    assert be.sr1cs_assignment(g, np.zeros((0, 8 * n_vars), dtype=np.uint32)).shape == (0, 8 * g.n_vars)
    be.gr1cs_free(g)
    be.r1cs_free(m)


@gpu
def test_lcmap_and_file_handles(be, tmp_path):
    curve = curve_of(be)
    r = curve.r
    # b2s_r1cs_upload_lcmap of the reference's circuits: the handle holds to_matrices() up to term order
    for cs in (orc.circuit2(curve, 1, 1, 2), orc.dummy_circuit(curve, 3, 5, 10, 7)):
        cs.finalize()
        lm = cs.to_lcmap()
        args = [np.array(a, dtype=np.uint64) for a in lm["args"]]
        pool = pack_fr(curve, lm["pool"])
        m = be.r1cs_upload_lcmap(len(args[0]), cs.num_instance_variables, cs.num_witness_variables, args,
                                 np.array(lm["offsets"], dtype=np.uint64), np.array(lm["vars"], dtype=np.uint64),
                                 np.array(lm["coeffs"], dtype=np.uint32), pool)
        g = be.r1cs_to_sr1cs(m)
        # the source as the handle holds it (its term order decides the numbering)
        info = be.gr1cs_info(g)
        o = so.Sr1cs(r, [csr_from_rows(curve, mm) for mm in cs.to_matrices()], cs.num_instance_variables)
        assert (info["n_instance"], info["n_witness"]) == (o.n_instance, o.n_witness)
        assert_structure(be, g, o)
        z = pack_fr(curve, cs.instance_assignment + cs.witness_assignment).reshape(1, -1)
        z2 = check_assignment_all(be, g, o, z, "host")
        check_verdicts(be, m, g, z, z2)
        be.gr1cs_free(g)
        be.r1cs_free(m)
    # b2s_r1cs_file_load: circom rows hold each wire once, in increasing order
    mats, n_inst, zi = random_r1cs(curve, 7)
    rows = [[[(sum(c for c, k in row if k == col) % r, col) for col in sorted({k for _, k in row})] for row in mm] for mm in mats]
    rows = [[[t for t in row if t[0]] for row in mm] for mm in rows]
    csr = [csr_from_rows(curve, mm) for mm in rows]
    n_vars = len(zi)
    data = ro.write_r1cs(curve, csr, 0, n_inst - 1, 0, n_wires=n_vars)
    m = be.r1cs_file_load(data)
    g = be.r1cs_to_sr1cs(m)
    o = so.Sr1cs(r, csr, n_inst)
    assert_structure(be, g, o)
    z = pack_fr(curve, zi).reshape(1, -1)
    z2 = check_assignment_all(be, g, o, z, "device")
    check_verdicts(be, m, g, z, z2)
    be.gr1cs_free(g)
    be.r1cs_free(m)


def unit_csr(curve, row_ptr, col):
    one = pack_fr(curve, [1])
    return row_ptr, col, np.tile(one, len(col))


def spmv_squares(be, m, z_row, n_rows, curve):
    """s_i = (<A_i, z> - <B_i, z>)^2 from b2s_spmv (z[0] = 1), as Montgomery limbs"""
    a, b, _ = be.spmv(m, z_row, n_rows)
    R, r = 1 << 256, curve.r
    Rinv = pow(R, -1, r)
    ai, bi = so.limbs_to_ints(a), so.limbs_to_ints(b)
    return so.ints_to_limbs([((x - y) * Rinv % r) ** 2 % r * R % r for x, y in zip(ai, bi)]).reshape(-1, 8)


@gpu
def test_bench_shaped_2p20(be):
    """BenchCircuit-shaped 2^20 rows: structure, and every element of 3 host assignments (more than one chunk each: a row
    of z is ~100 MB) against the oracle's copies and spmv's squares"""
    from tools.spmv_probe import bench_shaped_csr

    curve = curve_of(be)
    n = 1 << 20
    (A, B, C), n_vars = bench_shaped_csr(n, seed=2)
    csr = [unit_csr(curve, *x) for x in (A, B, C)]
    m = be.r1cs_upload(n, 1, n_vars - 1, csr)
    g = be.r1cs_to_sr1cs(m)
    o = so.Sr1cs(curve.r, csr, 1)
    assert_structure(be, g, o)
    print(f"bench-shaped 2^20 {curve.name}: structure equal", flush=True)   # progress of a long test
    z = random_z(curve, 3, n_vars, 5)
    got = be.sr1cs_assignment(g, z).reshape(3, -1, 8)
    cols, vals = o.copied(z)
    assert np.array_equal(got[:, cols, :], vals)
    for a in range(3):
        assert np.array_equal(got[a, o.sq_col, :], spmv_squares(be, m, z[a], n, curve))
    check_verdicts(be, m, g, z[:1], got[:1].reshape(1, -1))
    be.gr1cs_free(g)
    be.r1cs_free(m)


@gpu
def test_dummy_shaped_2p24(be):
    """DummyCircuit-shaped 2^24 rows (a*b = c, the last row empty): structure, every copied element, s_i on the first, last
    and 4096 random rows, and the verdicts for a satisfying and an unsatisfying z"""
    curve = curve_of(be)
    r = curve.r
    n = 1 << 24
    rp = np.arange(n + 1, dtype=np.uint64)
    rp[-1] = n - 1
    csr = [unit_csr(curve, rp, np.full(n - 1, c, dtype=np.uint32)) for c in (2, 3, 1)]
    n_vars = 6                                        # ONE, c, a, b, two unused witnesses
    m = be.r1cs_upload(n, 2, n_vars - 2, csr)
    g = be.r1cs_to_sr1cs(m)
    o = so.Sr1cs(r, csr, 2)
    assert (o.n_instance, o.n_witness) == (2, 3 + n)
    assert_structure(be, g, o)
    print(f"dummy-shaped 2^24 {curve.name}: structure equal", flush=True)   # progress of a long test
    z = pack_fr(curve, [1, 15, 3, 5, 7, 9] + [1, 14, 3, 5, 7, 9]).reshape(2, -1)
    got = be.sr1cs_assignment(g, z).reshape(2, -1, 8)
    cols, vals = o.copied(z)
    assert np.array_equal(got[:, cols, :], vals)
    rows = sorted({0, n - 1} | set(random.Random(1).sample(range(n), 4096)))
    for a in range(2):
        assert np.array_equal(got[a, o.sq_col[rows], :], so.ints_to_limbs(o.squares(z[a], rows)).reshape(-1, 8))
    check_verdicts(be, m, g, z, got.reshape(2, -1))
    be.gr1cs_free(g)
    be.r1cs_free(m)


@gpu
def test_export_round_trip_and_lifetime(be):
    curve = curve_of(be)
    r = curve.r
    rng = random.Random(5)
    mats = [[[(rng.choice([1, r - 1, rng.randrange(r)]), rng.randrange(9)) for _ in range(rng.randint(0, 4))] for _ in range(6)]
            for _ in range(3)]
    g = be.gr1cs_upload(2, 7, {"P": (3, [(1, [(0, 1), (1, 1)]), (r - 1, [(2, 1)])], mats)})
    info = be.gr1cs_info(g)
    assert (info["n_instance"], info["n_witness"]) == (2, 7)
    assert info["predicates"] == [(3, 6, [sum(len(row) for row in mm) for mm in mats])]
    for j in range(3):
        for a, b in zip(be.gr1cs_export(g, 0, j, info), csr_from_rows(curve, mats[j])):
            assert np.array_equal(a, b)
    be.gr1cs_free(g)
    # the converted handle outlives its source
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    csr = [csr_from_rows(curve, mm) for mm in cs.to_matrices()]
    m = be.r1cs_upload(3, len(cs.instance_assignment), len(cs.witness_assignment), csr)
    g = be.r1cs_to_sr1cs(m)
    be.r1cs_free(m)
    o = so.Sr1cs(r, csr, 2)
    assert_structure(be, g, o)
    z = pack_fr(curve, cs.instance_assignment + cs.witness_assignment).reshape(1, -1)
    z2 = check_assignment_all(be, g, o, z, "host")
    f, n = be.gr1cs_check(g, z2)
    assert int(f[0, 0]) == NOT_FOUND and int(n[0, 0]) == 0
    be.gr1cs_free(g)


@gpu
def test_rejections(be):
    from snark_b200 import Backend

    curve = curve_of(be)
    lib, h = be.lib, be.h
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    csr = [csr_from_rows(curve, mm) for mm in cs.to_matrices()]
    m = be.r1cs_upload(3, len(cs.instance_assignment), len(cs.witness_assignment), csr)
    g = be.r1cs_to_sr1cs(m)
    out = ctypes.c_void_p()
    z = pack_fr(curve, cs.instance_assignment + cs.witness_assignment)
    z2 = np.zeros(8 * g.n_vars, dtype=np.uint32)
    nv, npred = (ctypes.c_uint64 * 2)(), ctypes.c_uint32()
    buf = np.zeros(1 << 12, dtype=np.uint64)
    assert lib.b2s_r1cs_to_sr1cs(h, None, ctypes.byref(out)) == INVALID_ARG
    assert lib.b2s_r1cs_to_sr1cs(h, m, None) == INVALID_ARG
    assert lib.b2s_sr1cs_assignment(h, None, 1, z.ctypes.data, 0, z2.ctypes.data) == INVALID_ARG
    assert lib.b2s_sr1cs_assignment(h, g.h, 1, None, 0, z2.ctypes.data) == INVALID_ARG
    assert lib.b2s_sr1cs_assignment(h, g.h, 1, z.ctypes.data, 0, None) == INVALID_ARG
    assert lib.b2s_sr1cs_assignment(h, g.h, 0, None, 0, None) == 0
    assert lib.b2s_gr1cs_info(h, None, nv, ctypes.byref(npred), None, 0) == INVALID_ARG
    assert lib.b2s_gr1cs_info(h, g.h, None, ctypes.byref(npred), None, 0) == INVALID_ARG
    assert lib.b2s_gr1cs_export(h, g.h, 0, 0, None, 0, None, 0, None, 0) == INVALID_ARG
    # out of range predicate / argument, and buffers too small
    assert lib.b2s_gr1cs_export(h, g.h, 1, 0, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes) == INVALID_ARG
    assert lib.b2s_gr1cs_export(h, g.h, 0, 2, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes) == INVALID_ARG
    assert lib.b2s_gr1cs_export(h, g.h, 0, 0, buf.ctypes.data, 8, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes) == INVALID_ARG
    assert lib.b2s_gr1cs_export(h, g.h, 0, 0, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes, buf.ctypes.data, 32) == INVALID_ARG
    # a plain GR1CS handle has no variable map
    r = curve.r
    plain = be.gr1cs_upload(2, 2, {"R1CS": (3, [(1, [(0, 1), (1, 1)]), (r - 1, [(2, 1)])], cs.to_matrices())})
    assert lib.b2s_sr1cs_assignment(h, plain.h, 1, z.ctypes.data, 0, z2.ctypes.data) == INVALID_ARG
    # a handle from another curve's ctx
    other = Backend(curve=(be.curve + 1) % 3)
    try:
        assert other.lib.b2s_sr1cs_assignment(other.h, g.h, 1, z.ctypes.data, 0, z2.ctypes.data) == INVALID_ARG
        assert other.lib.b2s_gr1cs_info(other.h, g.h, nv, ctypes.byref(npred), None, 0) == INVALID_ARG
        assert other.lib.b2s_gr1cs_export(other.h, plain.h, 0, 0, buf.ctypes.data, buf.nbytes, buf.ctypes.data, buf.nbytes,
                                          buf.ctypes.data, buf.nbytes) == INVALID_ARG
    finally:
        other.close()
    be.gr1cs_free(plain)
    be.gr1cs_free(g)
    be.r1cs_free(m)
