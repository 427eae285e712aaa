"""Instance outlining on the GPU: b2s_gr1cs_upload_lcmap_outline / b2s_r1cs_upload_lcmap_outline and the outlined assignments,
against the oracle's finalize() with an InstanceOutliner and the numpy restatement of tests/outline_oracle.py, on all three
curves: the reference's circuits row for row in term order, random systems under both strategies with bare One / Instance /
Witness arguments mixed in, planted systems whose outlined assignments satisfy every row and whose corrupted copies fail
exactly the predicted rows, Groth16 end to end up to 2^20 (bit-identical to the host-outlined upload), a DummyCircuit shape
whose outlined domain is 2^24, and every rejection."""
import ctypes
import random

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests import outline_oracle as oo
from tests.bls377_oracle import BLS12_377
from tests.gr1cs_lcmap_gen import TAG_INSTANCE, TAG_LC, TAG_ONE, TAG_WITNESS, csr_of, planted, random_z, raw, to_lcmap_all
from tests.test_gpu_gr1cs import expected
from tests.test_outline_oracle import oracle_cs, random_system, set_outliner
from tests.util import pack_fr

CURVES = [BLS12_381, BN254, BLS12_377]
NOT_FOUND = (1 << 64) - 1
INVALID_ARG, DEGREE = 16, 5
gpu = pytest.mark.gpu
LABEL = {oo.OUTLINE_R1CS: "R1CS", oo.OUTLINE_SR1CS: "SR1CS"}


@pytest.fixture(scope="module", params=[0, 1, 2], ids=["bls12_381", "bn254", "bls12_377"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def preds_of(cs):
    """{label: (arity, terms)} of an oracle ConstraintSystem, R1CS included"""
    out = {"R1CS": (3, oo.r1cs_terms(cs.r))}
    out.update({label: (p["arity"], p["terms"]) for label, p in cs.predicates.items()})
    return out


def rows_limbs(curve, rows):
    """rows of (coeff int, col) -> (row_ptr, col, coeff limbs) as b2s_gr1cs_export returns them"""
    rp = np.zeros(len(rows) + 1, dtype=np.uint64)
    rp[1:] = np.cumsum([len(x) for x in rows])
    col = np.array([c for x in rows for _, c in x], dtype=np.uint32)
    co = pack_fr(curve, [v for x in rows for v, _ in x]) if rp[-1] else np.zeros(0, np.uint32)
    return rp, col, co


def assert_export_rows(be, g, curve, mats):
    """every argument of every predicate of g equals mats {label: [rows per argument]} (label order = upload order)"""
    info = be.gr1cs_info(g)
    for p, label in enumerate(sorted(mats)):
        for k, rows in enumerate(mats[label]):
            got = be.gr1cs_export(g, p, k, info)
            want = rows_limbs(curve, rows)
            for a, b in zip(got, want):
                assert np.array_equal(a, b), (label, k)


def assert_export_lcmap(be, g, curve, lm, n_instance):
    """the export of g equals csr_of over the (numpy-outlined) LcMap lm, pool ids resolved"""
    pool = pack_fr(curve, lm["pool"]).reshape(-1, 8)
    info = be.gr1cs_info(g)
    for p, label in enumerate(sorted(lm["args"])):
        for k, arg in enumerate(lm["args"][label]):
            rp, col, cid = csr_of(lm, n_instance, arg)
            got = be.gr1cs_export(g, p, k, info)
            assert np.array_equal(got[0], rp) and np.array_equal(got[1], col), (label, k)
            assert np.array_equal(got[2], pool[cid].reshape(-1)), (label, k)


# ---- the reference's circuits and random systems through the oracle builder --------------------------------------------
@gpu
def test_reference_circuits(be):
    """circuit1 (gr1cs/tests/mod.rs:105-133: exactly n_instance more witnesses) and circuit2, each outlined by outline_r1cs and,
    with an SR1CS predicate registered, by outline_sr1cs: export = to_matrices() after finalize(), assignment = z after it"""
    curve = CURVES[be.curve]
    systems = [lambda: orc.circuit1(curve, *orc.CIRCUIT1_SAT), lambda: orc.circuit2(curve, 3, 4, 12)]
    for make in systems:
        for strategy in (oo.OUTLINE_R1CS, oo.OUTLINE_SR1CS):
            cs = make()
            if strategy == oo.OUTLINE_SR1CS:
                oo.register_sr1cs(cs)
            cs.inline_all_lcs()
            n_inst, n_wit, z = cs.num_instance_variables, cs.num_witness_variables, cs.z()
            g = be.gr1cs_upload_lcmap(n_inst, n_wit, preds_of(cs), to_lcmap_all(cs), outline=(strategy, LABEL[strategy]))
            info = be.gr1cs_info(g)
            assert (info["n_instance"], info["n_witness"]) == (n_inst, n_wit + n_inst)
            set_outliner(cs, strategy)
            cs.finalize()
            assert cs.num_witness_variables == n_wit + n_inst
            assert_export_rows(be, g, curve, cs.to_matrices_all())
            got = be.outline_assignment(g, pack_fr(curve, z).reshape(1, -1))
            assert np.array_equal(got[0], pack_fr(curve, cs.z()))
            first, _ = be.gr1cs_check(g, got)
            assert all(int(f) == NOT_FOUND for f in first[0]) == cs.is_satisfied()
            be.gr1cs_free(g)


@gpu
def test_random_oracle_systems(be):
    """random systems with both predicates, bare arguments, Instance(0), Zero terms and zero coefficients"""
    curve = CURVES[be.curve]
    for seed in range(12):
        for strategy in (oo.OUTLINE_R1CS, oo.OUTLINE_SR1CS):
            system = random_system(curve, 7000 + 10 * seed + strategy, n_cons=random.Random(seed).randint(1, 40))
            cs = oracle_cs(curve, system)
            cs.inline_all_lcs()
            n_inst, n_wit, z = cs.num_instance_variables, cs.num_witness_variables, cs.z()
            g = be.gr1cs_upload_lcmap(n_inst, n_wit, preds_of(cs), to_lcmap_all(cs), outline=(strategy, LABEL[strategy]))
            set_outliner(cs, strategy)
            cs.finalize()
            assert_export_rows(be, g, curve, cs.to_matrices_all())
            got = be.outline_assignment(g, pack_fr(curve, z).reshape(1, -1))
            assert np.array_equal(got[0], pack_fr(curve, cs.z()))
            be.gr1cs_free(g)


# ---- planted systems ----------------------------------------------------------------------------------------------------
def planted_outline(curve, strategy, n, seed, n_inst=4, n_wit=64):
    """a planted GR1CS (every row holds for every z, tests/gr1cs_lcmap_gen.py) of predicates "P2" and "P3" with bare One,
    Instance and Witness arguments, plus an empty "R1CS" (x0 x1 - x2) and "SR1CS" (x0^2 - x1) that receive the tie rows.
    -> (preds, lcmap before outlining, lcmap the numpy restatement outlined)"""
    r = curve.r
    preds, lm = planted(r, {"P2": (2, n), "P3": (3, n)}, n_inst, n_wit, seed, n_shared=64)
    preds["R1CS"] = (3, oo.r1cs_terms(r))
    preds["SR1CS"] = (2, oo.sr1cs_terms(r))
    lm["args"]["R1CS"] = [np.zeros(0, np.uint64)] * 3
    lm["args"]["SR1CS"] = [np.zeros(0, np.uint64)] * 2
    lm["args"] = dict(sorted(lm["args"].items()))
    return preds, lm, oo.outline_lcmap(lm, n_inst, n_wit, strategy, LABEL[strategy])


def limbs_to_ints(curve, z):
    from tests.util import unpack_fr

    return unpack_fr(curve, np.ascontiguousarray(z).reshape(-1))


@gpu
@pytest.mark.parametrize("strategy", [oo.OUTLINE_R1CS, oo.OUTLINE_SR1CS])
def test_planted_small_with_corrupted_copies(be, strategy):
    """export = the numpy restatement; the outlined assignments satisfy every row; a wrong copy of instance i fails exactly the
    rows the restatement predicts (tie row i of the target among them)"""
    curve = CURVES[be.curve]
    n_inst, n_wit = 4, 64
    preds, lm, out = planted_outline(curve, strategy, 300, seed=11 + strategy, n_inst=n_inst, n_wit=n_wit)
    g = be.gr1cs_upload_lcmap(n_inst, n_wit, preds, lm, outline=(strategy, LABEL[strategy]))
    assert_export_lcmap(be, g, curve, out, n_inst)
    z = random_z(2, n_inst + n_wit, seed=3)
    z[:, :8] = pack_fr(curve, [1])
    zo = be.outline_assignment(g, z)
    first, count = be.gr1cs_check(g, zo)
    assert (first == NOT_FOUND).all() and (count == 0).all()
    # the restatement's rows, evaluated in Python ints
    pool = lm["pool"]
    mats = {}
    for label, args in out["args"].items():
        rows = []
        for a in args:
            rp, col, cid = csr_of(out, n_inst, a)
            rows.append([[(pool[cid[e]], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)])
        mats[label] = (preds[label][0], preds[label][1], rows)
    for i in range(n_inst):
        zi = limbs_to_ints(curve, zo[0])
        zi[n_inst + n_wit + i] = (zi[n_inst + n_wit + i] + 1) % curve.r
        want_first, want_count = expected(curve, mats, zi)
        first, count = be.gr1cs_check(g, pack_fr(curve, zi).reshape(1, -1))
        assert [int(x) for x in first[0]] == want_first and [int(x) for x in count[0]] == want_count, i
        assert int(first[0][sorted(preds).index(LABEL[strategy])]) == i   # the target has no rows of its own: tie row i
    be.gr1cs_free(g)


@gpu
@pytest.mark.parametrize("strategy", [oo.OUTLINE_R1CS, oo.OUTLINE_SR1CS])
def test_planted_2p20(be, strategy):
    """2^20 rows per predicate: export = the numpy restatement, every row satisfied by outlined assignments in host and
    device memory, x1 and x3"""
    import torch

    curve = CURVES[be.curve]
    n_inst, n_wit = 5, 1 << 12
    preds, lm, out = planted_outline(curve, strategy, 1 << 20, seed=21 + strategy, n_inst=n_inst, n_wit=n_wit)
    g = be.gr1cs_upload_lcmap(n_inst, n_wit, preds, lm, outline=(strategy, LABEL[strategy]))
    assert_export_lcmap(be, g, curve, out, n_inst)
    z = random_z(3, n_inst + n_wit, seed=4)
    z[:, :8] = pack_fr(curve, [1])
    want = np.concatenate([z, z[:, :8], z[:, 8:8 * n_inst]], axis=1)
    for k in (1, 3):
        host = be.outline_assignment(g, z[:k])
        assert np.array_equal(host, want[:k])
        dev = be.outline_assignment(g, torch.from_numpy(z[:k].view(np.int32)).cuda())
        be.sync()
        assert np.array_equal(dev.cpu().numpy().view(np.uint32), want[:k])
        first, count = be.gr1cs_check(g, host)
        assert (first == NOT_FOUND).all() and (count == 0).all()
    be.gr1cs_free(g)


# ---- the Groth16 matrix handle -------------------------------------------------------------------------------------------
def dummy_lcmap(curve, n_rows, x=(7, 9), ab=(3, 5)):
    """A satisfied DummyCircuit-like R1CS in LcMap form, n_instance = 3 (One, x1, x2), witnesses a, b, c1, c2:
    even rows (x1 + 2) * b = LC[c1 + x2 - x2], odd rows a * x2 = LC[2 c2 - c2]; the bare arguments b, a and x2 stay under
    outlining, the LCs' One and x read the copies.  -> (args, lcmap, z ints)"""
    r = curve.r
    x1, x2 = x
    a, b = ab
    z = [1, x1, x2, a, b, (x1 + 2) * b % r, a * x2 % r]
    off = np.array([0, 0, 2, 5, 7], np.uint64)          # LC 0 empty, LC1, LC2, LC3
    vars_ = np.array([raw(TAG_INSTANCE, 1), raw(TAG_ONE, 0), raw(TAG_WITNESS, 2), raw(TAG_INSTANCE, 2), raw(TAG_INSTANCE, 2),
                      raw(TAG_WITNESS, 3), raw(TAG_WITNESS, 3)], np.uint64)
    coeffs = np.array([0, 2, 0, 0, 1, 2, 1], np.uint32)
    even = np.arange(n_rows) % 2 == 0
    A = np.where(even, raw(TAG_LC, 1), raw(TAG_WITNESS, 0)).astype(np.uint64)
    B = np.where(even, raw(TAG_WITNESS, 1), raw(TAG_INSTANCE, 2)).astype(np.uint64)
    C = np.where(even, raw(TAG_LC, 2), raw(TAG_LC, 3)).astype(np.uint64)
    lm = {"offsets": off, "vars": vars_, "coeffs": coeffs, "pool": [1, r - 1, 2], "args": {"R1CS": [A, B, C]}}
    return lm, z


def r1cs_handle(be, curve, lm, n_inst, n_wit, outline):
    args = lm["args"]["R1CS"]
    from snark_b200.lib import _mont_limbs

    return be.r1cs_upload_lcmap(len(args[0]), n_inst, n_wit, [np.ascontiguousarray(a) for a in args], np.ascontiguousarray(lm["offsets"]),
                                np.ascontiguousarray(lm["vars"]), np.ascontiguousarray(lm["coeffs"]), _mont_limbs(curve.r, lm["pool"]),
                                outline=outline)


@gpu
@pytest.mark.parametrize("log_n", [10, 20])
def test_groth16_end_to_end(be, log_n):
    """setup and prove on the outlined handle: the proof verifies with the original public inputs, fails with one changed, and
    is bit-identical to the proof for the handle of the host-outlined LcMap under the same trapdoor, r and s"""
    curve = CURVES[be.curve]
    r = curve.r
    rng = random.Random(0x07 + log_n + be.curve)
    n_inst, n_wit = 3, 4
    lm, z = dummy_lcmap(curve, (1 << log_n) - 2 * n_inst)
    m = r1cs_handle(be, curve, lm, n_inst, n_wit, outline=True)
    assert be.domain_size(m) == 1 << log_n
    host = oo.outline_lcmap(lm, n_inst, n_wit, oo.OUTLINE_R1CS, "R1CS")
    m2 = r1cs_handle(be, curve, host, n_inst, n_wit + n_inst, outline=False)
    zo = be.outline_assignment(m, pack_fr(curve, z).reshape(1, -1))
    assert np.array_equal(zo[0], pack_fr(curve, oo.outline_z(z, n_inst)))
    first, _ = be.r1cs_check(m, zo)
    assert int(first[0][0]) == NOT_FOUND
    trap = pack_fr(curve, [rng.randrange(1, r) for _ in range(5)])
    pk, vk = be.groth16_setup(m, trap, n_inst)
    pk2, vk2 = be.groth16_setup(m2, trap, n_inst)
    assert all(np.array_equal(vk[k], vk2[k]) for k in vk)
    rr, ss = pack_fr(curve, [rng.randrange(r)]), pack_fr(curve, [rng.randrange(r)])
    zi, zw = zo[0][:8 * n_inst], zo[0][8 * n_inst:]
    proof = be.groth16_prove(pk, m, zi, zw, rr, ss)
    proof2 = be.groth16_prove(pk2, m2, zi, zw, rr, ss)
    assert all(np.array_equal(a, b) for a, b in zip(proof, proof2))
    pvk = be.vk_prepare(vk)
    x = pack_fr(curve, z[1:n_inst])
    assert be.groth16_verify_batch(pvk, x, n_inst - 1, *proof).tolist() == [True]
    bad = pack_fr(curve, [z[1] + 1] + z[2:n_inst])
    assert be.groth16_verify_batch(pvk, bad, n_inst - 1, *proof).tolist() == [False]
    be.pvk_free(pvk)
    for h in (pk, pk2):
        be.pk_free(h)
    be.r1cs_free(m)
    be.r1cs_free(m2)


@gpu
def test_dummy_shaped_2p24(be):
    """a DummyCircuit shape whose outlined domain is 2^24: export = the numpy restatement, assignments x1, x3, x64 in host and
    device memory, and check verdicts equal to the host-outlined upload's for a satisfying and a corrupted z"""
    import torch

    curve = CURVES[be.curve]
    n_inst, n_wit = 3, 4
    lm, z = dummy_lcmap(curve, (1 << 24) - 2 * n_inst)
    m = r1cs_handle(be, curve, lm, n_inst, n_wit, outline=True)
    assert be.domain_size(m) == 1 << 24
    host = oo.outline_lcmap(lm, n_inst, n_wit, oo.OUTLINE_R1CS, "R1CS")
    m2 = r1cs_handle(be, curve, host, n_inst, n_wit + n_inst, outline=False)
    # the export of the R1CS handle through b2s_r1cs_to_sr1cs is not the point here: compare through a GR1CS upload of the
    # same LcMap, whose export reads the very matrices lcmap_build made
    g = be.gr1cs_upload_lcmap(n_inst, n_wit, {"R1CS": (3, oo.r1cs_terms(curve.r))}, lm, outline=(oo.OUTLINE_R1CS, "R1CS"))
    assert_export_lcmap(be, g, curve, host, n_inst)
    print(f"dummy-shaped 2^24 {curve.name}: export equal", flush=True)   # progress of a long test
    zs = np.stack([pack_fr(curve, [1, 7 + k, 9 + 2 * k, 3, 5, (9 + k) * 5 % curve.r, 3 * (9 + 2 * k) % curve.r]) for k in range(64)])
    want = np.concatenate([zs, zs[:, :8], zs[:, 8:8 * n_inst]], axis=1)
    for k in (1, 3, 64):
        assert np.array_equal(be.outline_assignment(m, zs[:k]), want[:k])
        assert np.array_equal(be.outline_assignment(g, zs[:k]), want[:k])
        dev = be.outline_assignment(m, torch.from_numpy(zs[:k].view(np.int32)).cuda())
        be.sync()
        assert np.array_equal(dev.cpu().numpy().view(np.uint32), want[:k])
    zo = want[:2].copy()
    zo[1, 8 * (n_inst + n_wit + 2):8 * (n_inst + n_wit + 3)] = pack_fr(curve, [4])   # a wrong copy of x2
    got, got2 = be.r1cs_check(m, zo), be.r1cs_check(m2, zo)
    assert all(np.array_equal(a, b) for a, b in zip(got, got2))
    assert int(got[0][0][0]) == NOT_FOUND and int(got[0][1][0]) != NOT_FOUND
    be.gr1cs_free(g)
    be.r1cs_free(m)
    be.r1cs_free(m2)


# ---- rejections ----------------------------------------------------------------------------------------------------------
@gpu
def test_rejections(be):
    from snark_b200 import B2SError
    from snark_b200.lib import Outline, _mont_limbs

    curve = CURVES[be.curve]
    r = curve.r
    preds, lm, _ = planted_outline(curve, oo.OUTLINE_R1CS, 16, seed=5)

    def gr(outline, pool=None, n_inst=4, n_wit=64, p=preds):
        l2 = dict(lm, pool=pool or lm["pool"])
        return be.gr1cs_upload_lcmap(n_inst, n_wit, p, l2, outline=outline)

    def rejects(code, words, fn, *a, **k):
        with pytest.raises(B2SError) as e:
            fn(*a, **k)
        assert e.value.code == code, str(e.value)
        assert any(w in str(e.value) for w in words), str(e.value)

    rejects(INVALID_ARG, ["unknown outlining strategy"], gr, (0, "R1CS"))
    rejects(INVALID_ARG, ["unknown outlining strategy"], gr, (3, "R1CS"))
    rejects(INVALID_ARG, ["out of range"], gr, (oo.OUTLINE_R1CS, "nope"))
    rejects(INVALID_ARG, ["arity 2"], gr, (oo.OUTLINE_R1CS, "SR1CS"))
    rejects(INVALID_ARG, ["arity 3"], gr, (oo.OUTLINE_SR1CS, "R1CS"))
    bad_pool = [1, 5] + lm["pool"][2:]
    rejects(INVALID_ARG, ["pool[1] is not -ONE"], gr, (oo.OUTLINE_SR1CS, "SR1CS"), pool=bad_pool)
    be.gr1cs_free(gr((oo.OUTLINE_R1CS, "R1CS"), pool=bad_pool))      # outline_r1cs never reads pool[1]
    # the limits, counted with the copies and the tie rows (nothing is read past the descriptors)
    rejects(DEGREE, ["variables"], gr, (oo.OUTLINE_R1CS, "R1CS"), n_inst=1 << 31, n_wit=1)
    rejects(DEGREE, ["rows"], gr, (oo.OUTLINE_R1CS, "R1CS"), n_inst=(1 << 31) - 1, n_wit=1)
    # the Groth16 handle: outline_r1cs on predicate 0 only, and its domain
    one = np.zeros(1, np.uint64)
    pool = _mont_limbs(r, [1, r - 1])
    off = np.zeros(2, np.uint64)
    h = ctypes.c_void_p()
    call = lambda n_rows, n_inst, args, ol: be.lib.b2s_r1cs_upload_lcmap_outline(
        be.h, n_rows, n_inst, 1, (ctypes.c_void_p * 3)(*[a.ctypes.data for a in args]), 1, off.ctypes.data, one.ctypes.data,
        one.ctypes.data, pool.ctypes.data, 2, ctypes.byref(ol) if ol is not None else None, ctypes.byref(h))
    args = [one] * 3
    for ol, code, word in ((Outline(oo.OUTLINE_SR1CS, 0), INVALID_ARG, b"B2S_OUTLINE_R1CS only"),
                           (Outline(7, 0), INVALID_ARG, b"unknown outlining strategy"),
                           (Outline(oo.OUTLINE_R1CS, 1), INVALID_ARG, b"out of range"),
                           (None, INVALID_ARG, b"null argument")):
        assert call(1, 1, args, ol) == code
        assert word in be.lib.b2s_last_error(be.h)
    big = np.zeros(1 << 26, np.uint64)
    assert call(1 << 26, (1 << 25) + 1, [big] * 3, Outline(oo.OUTLINE_R1CS, 0)) == DEGREE
    assert b"domain" in be.lib.b2s_last_error(be.h)
    # outline_assignment of handles no outlining upload made
    lm0, z = dummy_lcmap(curve, 10)
    m = r1cs_handle(be, curve, lm0, 3, 4, outline=False)
    out = np.zeros(8 * 10, np.uint32)
    zz = pack_fr(curve, z)
    assert be.lib.b2s_r1cs_outline_assignment(be.h, m, 1, zz.ctypes.data, 0, out.ctypes.data) == INVALID_ARG
    assert b"not made by b2s_r1cs_upload_lcmap_outline" in be.lib.b2s_last_error(be.h)
    g = be.gr1cs_upload_lcmap(3, 4, {"R1CS": (3, oo.r1cs_terms(r))}, lm0)
    assert be.lib.b2s_gr1cs_outline_assignment(be.h, g.h, 1, zz.ctypes.data, 0, out.ctypes.data) == INVALID_ARG
    assert b"not made by b2s_gr1cs_upload_lcmap_outline" in be.lib.b2s_last_error(be.h)
    be.gr1cs_free(g)
    be.r1cs_free(m)
