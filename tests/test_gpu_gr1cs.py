"""b2s_gr1cs_check / b2s_r1cs_check: ConstraintSystem::which_is_unsatisfied (constraint_system.rs:652-687, predicate/mod.rs:185-204)
on the GPU, against the oracle (oracle/r1cs.py) on the reference's satisfaction vectors, random GR1CS with up to five polynomial
predicates, Groth16 matrix handles up to 2^24 rows, batches across chunk boundaries and the verdicts of prove + verify."""
import random

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests.util import csr_from_rows, pack_fr

CURVES = [BLS12_381, BN254]
NOT_FOUND = (1 << 64) - 1
CHECK_SCRATCH_BYTES = 64 << 20   # per-chunk device scratch of csrc/gr1cs.cu: z rows of host assignments, and outputs
CHECK_MAX_ASSIGN = 65535          # assignments per launch (gridDim.y)
gpu = pytest.mark.gpu


def r1cs_terms(r):
    return [(1, [(0, 1), (1, 1)]), (r - 1, [(2, 1)])]


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


# ---- the oracle side --------------------------------------------------------------------------------------------------
def predicates_of(cs):
    """{label: (arity, terms, matrices)} of an oracle ConstraintSystem, R1CS included"""
    out = {}
    for label, mats in cs.to_matrices_all().items():
        if label == "R1CS":
            out[label] = (3, r1cs_terms(cs.r), mats)
        else:
            p = cs.predicates[label]
            out[label] = (p["arity"], p["terms"], mats)
    return out


def unsat_rows(r, arity, terms, mats, z):
    """every row of one predicate whose polynomial is nonzero at the row products (what first_unsat / n_unsat summarise)"""
    bad = []
    for i in range(len(mats[0]) if mats else 0):
        x = [sum(c * z[col] for c, col in mats[j][i]) % r for j in range(arity)]
        acc = 0
        for coeff, mono in terms:
            t = coeff
            for v, e in mono:
                t = t * pow(x[v], e, r)
            acc += t
        if acc % r:
            bad.append(i)
    return bad


def random_gr1cs(curve, seed):
    """A random GR1CS with a satisfying assignment: 1-5 predicates of arity 1-8; each polynomial is Q(x_0..x_{a-2}) - x_{a-1}
    with 0-5 terms of degree <= 6 in Q (or, for some predicates, the zero polynomial), so the last argument is a linear output:
    its row is a fresh witness (plus, sometimes, a second term) solved for Q.  Coefficients include ONE, -ONE and zero, rows
    have duplicate and unsorted columns or none at all, and some predicates have no constraints.
    Returns (predicates, n_instance, z, outputs) with outputs[label] = [(row, column of its output witness)]."""
    r = curve.r
    rng = random.Random(seed)
    n_inst = rng.randint(1, 4)
    z = [1] + [rng.randrange(r) for _ in range(n_inst - 1 + rng.randint(1, 10))]
    coeff = lambda: rng.choice([1, r - 1, 0, rng.randrange(r), rng.randrange(r)])
    preds, outputs = {}, {}
    for label in rng.sample([f"pred-{i}" for i in range(10)], rng.randint(1, 5)):
        arity = rng.randint(1, 8)
        zero_poly = rng.random() < 0.15
        terms = []
        if not zero_poly:
            for _ in range(rng.randint(0, 5)):
                mono, d = [], rng.randint(0, 6)
                while d > 0 and arity > 1:
                    e = rng.randint(1, d)
                    mono.append((rng.randrange(arity - 1), e))
                    d -= e
                if arity > 1 and rng.random() < 0.2:
                    mono.append((rng.randrange(arity - 1), 0))   # x^0 = 1
                rng.shuffle(mono)
                terms.append((coeff(), mono))
            terms.append((r - 1, [(arity - 1, 1)]))
            rng.shuffle(terms)
        n_rows = rng.choice([0, 1, rng.randint(2, 40), rng.randint(2, 40)])
        mats = [[] for _ in range(arity)]
        outs = []
        for i in range(n_rows):
            last = arity if zero_poly else arity - 1
            for j in range(last):
                mats[j].append([(coeff(), rng.randrange(len(z))) for _ in range(rng.choice([0, 1, 1, 2, 3, 4]))])
            if zero_poly:
                continue
            x = [sum(c * z[col] for c, col in mats[j][i]) % r for j in range(arity - 1)] + [0]
            q = sum(c * np.prod([pow(x[v], e, r) for v, e in mono] or [1], dtype=object) for c, mono in terms if mono != [(arity - 1, 1)])
            c0 = rng.choice([1, r - 1, rng.randrange(1, r)])
            row = [(c0, len(z))]
            if rng.random() < 0.3:
                row.append((coeff(), rng.randrange(len(z))))
                rng.shuffle(row)
            rest = sum(c * z[col] for c, col in row if col != len(z))
            outs.append((i, len(z)))
            z.append((q - rest) * pow(c0, -1, r) % r)
            mats[arity - 1].append(row)
        preds[label] = (arity, terms, mats)
        outputs[label] = outs
    return preds, n_inst, z, outputs


CORRUPT = ("none", "first", "last", "middle", "every")


def corrupted(z, outputs, how):
    """z with the output witnesses of the chosen rows of every predicate changed (each such row then fails)"""
    z = list(z)
    for outs in outputs.values():
        if not outs or how == "none":
            continue
        pick = {"first": outs[:1], "last": outs[-1:], "middle": [outs[len(outs) // 2]], "every": outs}[how]
        for _, col in pick:
            z[col] += 1
    return z


def oracle_cs(curve, preds, n_inst, z):
    """The same system through the oracle's ConstraintSystem builder (register_predicate / enforce_constraint)"""
    r = curve.r
    cs = orc.ConstraintSystem(curve)
    cs.instance_assignment, cs.witness_assignment = list(z[:n_inst]), list(z[n_inst:])
    cs.num_instance_variables, cs.num_witness_variables = n_inst, len(z) - n_inst
    var = lambda col: orc.V_ONE if col == 0 else (orc.instance(col) if col < n_inst else orc.witness(col - n_inst))
    for label, (arity, terms, mats) in preds.items():
        cs.register_predicate(label, arity, terms)
        for i in range(len(mats[0])):
            cs.enforce_constraint(label, [orc.LinearCombination(r, [(c, var(col)) for c, col in mats[j][i]]) for j in range(arity)])
    return cs


def expected(curve, preds, z):
    """(first, count) in label order, from unsat_rows"""
    first, count = [], []
    for label in sorted(preds):
        bad = unsat_rows(curve.r, *preds[label], z)
        first.append(bad[0] if bad else NOT_FOUND)
        count.append(len(bad))
    return first, count


def test_random_gr1cs_generator_against_the_oracle():
    """CPU: the generator's assignments satisfy every predicate, each corruption fails where it should, and the first failure
    of unsat_rows in label order is the oracle's which_is_unsatisfied"""
    for curve in CURVES:
        for seed in range(40):
            preds, n_inst, z, outputs = random_gr1cs(curve, seed)
            for how in CORRUPT:
                zc = corrupted(z, outputs, how)
                first, count = expected(curve, preds, zc)
                if how == "none":
                    assert count == [0] * len(preds)
                elif any(outputs.values()):
                    # the earliest corrupted output witness breaks its own row (every other change reads only later columns)
                    assert sum(count) >= 1
                want = next(((label, f) for label, f in zip(sorted(preds), first) if f != NOT_FOUND), None)
                assert oracle_cs(curve, preds, n_inst, zc).which_is_unsatisfied() == want, (seed, how)


# ---- 1. the reference's vectors --------------------------------------------------------------------------------------
def reference_systems(curve):
    for name, (x, w) in (("sat", orc.CIRCUIT1_SAT), ("unsat", orc.CIRCUIT1_UNSAT)):
        for mode in ("raw", "finalized", "outlined"):
            cs = orc.circuit1(curve, x, w)
            if mode == "outlined":
                cs.set_instance_outliner("R1CS", orc.outline_r1cs)
            if mode != "raw":
                cs.finalize()
            yield f"circuit1-{name}-{mode}", cs
    for vals in ((1, 1, 2), (2, 1, 4), (1, 3, 5)):   # circuit2's own values, then a changed a (fails row 1) and a changed c (row 0)
        for mode in ("finalized", "outlined"):
            cs = orc.circuit2(curve, *vals)
            if mode == "outlined":
                cs.set_instance_outliner("R1CS", orc.outline_r1cs)
            cs.finalize()
            yield f"circuit2-{vals}-{mode}", cs


@gpu
def test_reference_vectors(be):
    curve = CURVES[be.curve]
    seen = set()
    for name, cs in reference_systems(curve):
        if name == "circuit1-sat-raw":
            assert cs.to_matrices_all() == orc.CIRCUIT1_GOLDEN
        if name.startswith("circuit2-(1, 1, 2)-f"):
            assert cs.to_matrices() == orc.CIRCUIT2_GOLDEN
        g = be.gr1cs_upload(cs.num_instance_variables, cs.num_witness_variables, predicates_of(cs))
        want = cs.which_is_unsatisfied()
        assert be.which_is_unsatisfied(g, pack_fr(curve, cs.z())) == want, name
        seen.add(want)
        be.gr1cs_free(g)
    assert None in seen and ("poly-predicate-A", 0) in seen and ("R1CS", 0) in seen and ("R1CS", 1) in seen


# ---- 2. random GR1CS ------------------------------------------------------------------------------------------------
@gpu
def test_random_gr1cs_matches_the_oracle_lists(be):
    curve = CURVES[be.curve]
    for seed in range(24):
        preds, n_inst, z, outputs = random_gr1cs(curve, 1000 * be.curve + seed)
        g = be.gr1cs_upload(n_inst, len(z) - n_inst, preds)
        zs = [corrupted(z, outputs, how) for how in CORRUPT]
        first, count = be.gr1cs_check(g, pack_fr(curve, [v for zz in zs for v in zz]).reshape(len(zs), -1))
        for i, zz in enumerate(zs):
            f, n = expected(curve, preds, zz)
            assert first[i].tolist() == f and count[i].tolist() == n, (seed, CORRUPT[i])
        be.gr1cs_free(g)


# ---- 3. wrap-around ---------------------------------------------------------------------------------------------------
@gpu
def test_sums_that_vanish_only_mod_r_are_satisfied(be):
    curve = CURVES[be.curve]
    r = curve.r
    v = r - 5
    z = [1, v, v, 3]
    preds = {
        # (r - 1) x0 + x1 with x0 = x1: the integer sum is a multiple of r
        "cancel-terms": (2, [(r - 1, [(0, 1)]), (1, [(1, 1)])], [[[(1, 1)], [(1, 2)]], [[(1, 2)], [(1, 1)]]]),
        # coefficients r - 1 and 1 on equal values inside one row product, then x0 = 0
        "cancel-row": (1, [(1, [(0, 1)])], [[[(r - 1, 1), (1, 2)], [(1, 1), (r - 1, 1)]]]),
        # (r - 1) x0^2 + x1 x1 with x0 = x1 = r - 5: products wrap as well
        "cancel-products": (2, [(r - 1, [(0, 2)]), (1, [(1, 1), (1, 1)])], [[[(1, 1)]], [[(1, 2)]]]),
        "control": (1, [(1, [(0, 1)])], [[[(r - 1, 1), (1, 3)]]]),
    }
    g = be.gr1cs_upload(1, 3, preds)
    first, count = be.gr1cs_check(g, pack_fr(curve, z).reshape(1, -1))
    assert first[0].tolist() == [NOT_FOUND, NOT_FOUND, NOT_FOUND, 0] and count[0].tolist() == [0, 0, 0, 1]
    be.gr1cs_free(g)


# ---- 4. R1CS handles -------------------------------------------------------------------------------------------------
def dummy_rows(curve, log_n, spread):
    """DummyCircuit-shaped R1CS at domain 2^log_n: row i reads a * b = c with a taken from copy i mod `spread` of a (z[4..]),
    b = z[3], c = z[1]; the last row is empty.  Returns (csr, n_rows, n_inst, n_wit, z) with a satisfying z."""
    N = 1 << log_n
    n_rows, n_inst, n_wit = N - 2, 2, N - 3
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    ones = np.tile(pack_fr(curve, [1]), nnz)
    a_col = (4 + np.arange(nnz, dtype=np.uint64) % spread).astype(np.uint32)
    csr = [(row_ptr, a_col, ones), (row_ptr, np.full(nnz, 3, dtype=np.uint32), ones), (row_ptr, np.full(nnz, 1, dtype=np.uint32), ones)]
    rng = random.Random(log_n)
    a, b = rng.randrange(curve.r), rng.randrange(curve.r)
    z = np.tile(pack_fr(curve, [a]), n_inst + n_wit).reshape(-1, 8)
    z[0], z[1], z[3] = pack_fr(curve, [1]), pack_fr(curve, [a * b % curve.r]), pack_fr(curve, [b])
    return csr, n_rows, n_inst, n_wit, z.reshape(-1)


@gpu
def test_r1cs_check_on_the_groth16_test_circuits(be):
    from tests.test_gpu_groth16 import circuits, upload

    curve = CURVES[be.curve]
    for name, mats, inst, wit in circuits(curve):
        m, _keep = upload(be, curve, mats, len(inst), len(wit))
        z = list(inst) + list(wit)
        bad = list(z)
        bad[-1] = (bad[-1] + 1) % curve.r
        first, count = be.r1cs_check(m, pack_fr(curve, z + bad).reshape(2, -1))
        for i, zz in enumerate((z, bad)):
            rows = unsat_rows(curve.r, 3, r1cs_terms(curve.r), mats, zz)
            assert first[i, 0] == (rows[0] if rows else NOT_FOUND) and count[i, 0] == len(rows), (name, i)
        be.r1cs_free(m)


@gpu
@pytest.mark.parametrize("log_n", [12, 16, 20, 24])
def test_r1cs_check_dummy_circuit(be, log_n):
    """satisfied as built; with copy t of a changed, exactly the rows i = t mod spread fail"""
    curve = CURVES[be.curve]
    spread = (1 << (log_n - 2)) + 3
    csr, n_rows, n_inst, n_wit, z = dummy_rows(curve, log_n, spread)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    t = 12345 % spread
    zs = np.tile(z, (2, 1))
    zs[1, 8 * (4 + t): 8 * (5 + t)] = pack_fr(curve, [7])
    del z, csr
    first, count = be.r1cs_check(m, zs)
    n_fail = len(range(t, n_rows - 1, spread))
    assert first[:, 0].tolist() == [NOT_FOUND, t] and count[:, 0].tolist() == [0, n_fail]
    be.r1cs_free(m)


@gpu
def test_upload_and_lcmap_handles_agree(be):
    from tests.test_zz_gpu_lcmap import upload_lcmap

    curve = CURVES[be.curve]
    for cs in (orc.bench_circuit(curve, 40, seed=3), orc.circuit2(curve, 2, 1, 4), orc.dummy_circuit(curve, 3, 5, 16, 16)):
        cs.finalize()
        z = cs.z()
        bad = list(z)
        bad[-1] += 1
        zz = pack_fr(curve, z + bad).reshape(2, -1)
        m1 = be.r1cs_upload(len(cs.constraints), cs.num_instance_variables, cs.num_witness_variables,
                            [csr_from_rows(curve, mm) for mm in cs.to_matrices()])
        m2 = upload_lcmap(be, curve, cs)
        f1, c1 = be.r1cs_check(m1, zz)
        f2, c2 = be.r1cs_check(m2, zz)
        assert np.array_equal(f1, f2) and np.array_equal(c1, c2)
        want = cs.which_is_unsatisfied()
        assert (None if f1[0, 0] == NOT_FOUND else ("R1CS", int(f1[0, 0]))) == want
        be.r1cs_free(m1)
        be.r1cs_free(m2)


@gpu
def test_circom_empty_c_handle_checks_a_times_b_is_zero(be):
    """a handle whose C is empty (as for the circom reduction) checks a * b = 0"""
    curve = CURVES[be.curve]
    r = curve.r
    A = [[(1, 1)], [(1, 2)], [], [(1, 1), (r - 1, 2)]]
    B = [[(1, 2)], [(1, 0)], [(1, 1)], [(1, 3)]]
    csr = [csr_from_rows(curve, mm) for mm in (A, B, [[] for _ in A])]
    m = be.r1cs_upload(len(A), 2, 2, csr)
    z = [1, 5, 0, 9]   # rows: 5 * 0, 0 * 1, 0 * 5, 5 * 9
    first, count = be.r1cs_check(m, pack_fr(curve, z).reshape(1, -1))
    assert first[0, 0] == 3 and count[0, 0] == 1
    be.r1cs_free(m)


# ---- 5. batches -----------------------------------------------------------------------------------------------------
def batch_system(curve):
    preds, n_inst, z, outputs = random_gr1cs(curve, 77)
    while not any(outputs.values()):
        preds, n_inst, z, outputs = random_gr1cs(curve, len(z) + 78)
    return preds, n_inst, z, outputs


@gpu
@pytest.mark.parametrize("n_assign", [0, 1, 7, 33])
def test_batch_rows_equal_single_calls(be, n_assign):
    import torch

    curve = CURVES[be.curve]
    preds, n_inst, z, outputs = batch_system(curve)
    g = be.gr1cs_upload(n_inst, len(z) - n_inst, preds)
    zs = np.stack([pack_fr(curve, corrupted(z, outputs, CORRUPT[i % 5])) for i in range(n_assign)]) if n_assign else \
        np.zeros((0, 8 * len(z)), dtype=np.uint32)
    first, count = be.gr1cs_check(g, zs)
    assert first.shape == count.shape == (n_assign, len(preds))
    for i in range(n_assign):
        f1, c1 = be.gr1cs_check(g, zs[i: i + 1])
        assert np.array_equal(first[i], f1[0]) and np.array_equal(count[i], c1[0])
        assert (first[i].tolist(), count[i].tolist()) == expected(curve, preds, corrupted(z, outputs, CORRUPT[i % 5]))
    f_nc, c_nc = be.gr1cs_check(g, zs, counts=False)
    assert c_nc is None and np.array_equal(f_nc, first)
    zd = torch.from_numpy(zs.view(np.int32)).cuda()
    for counts in (True, False):
        fd, cd = be.gr1cs_check(g, zd, counts=counts)
        assert np.array_equal(fd, first) and (cd is None if not counts else np.array_equal(cd, count))
    be.gr1cs_free(g)


@gpu
def test_batches_across_chunk_boundaries(be):
    """host chunks bounded by scratch (2^16-variable rows: 32 per chunk) and by gridDim.y (65 535 assignments), host and device"""
    import torch

    curve = CURVES[be.curve]
    csr, n_rows, n_inst, n_wit, z = dummy_rows(curve, 16, 1000)
    n_vars = n_inst + n_wit
    per_chunk = CHECK_SCRATCH_BYTES // (32 * n_vars)
    assert per_chunk == 32
    K = per_chunk + 3
    zs = np.tile(z, (K, 1)).reshape(K, n_vars, 8)
    bad = [0, per_chunk - 1, per_chunk, K - 1]
    for k in bad:
        zs[k, 4 + (k * 37) % 1000] = pack_fr(curve, [k + 2])
    zs = zs.reshape(K, -1)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    for zz in (zs, torch.from_numpy(zs.view(np.int32)).cuda()):
        first, count = be.r1cs_check(m, zz)
        want = [((k * 37) % 1000 if k in bad else NOT_FOUND) for k in range(K)]
        assert first[:, 0].tolist() == want
        assert count[:, 0].tolist() == [len(range((k * 37) % 1000, n_rows - 1, 1000)) if k in bad else 0 for k in range(K)]
    be.r1cs_free(m)
    # more assignments than one launch takes: circuit2, every 997th assignment with c changed (fails row 0)
    cs = orc.circuit2(curve, 2, 1, 4)
    cs.finalize()
    cs2 = orc.circuit2(curve, 1, 1, 2)
    cs2.finalize()
    m = be.r1cs_upload(3, cs2.num_instance_variables, cs2.num_witness_variables, [csr_from_rows(curve, mm) for mm in cs2.to_matrices()])
    K = CHECK_MAX_ASSIGN + 100
    zs = np.tile(pack_fr(curve, cs2.z()), (K, 1))
    broken = np.arange(0, K, 997)
    zs[broken] = pack_fr(curve, cs.z())   # a = 2 (with c = 2ab): a (a + b) = a + b fails, row 1
    for zz in (zs, torch.from_numpy(zs.view(np.int32)).cuda()):
        first, count = be.r1cs_check(m, zz)
        want = np.full(K, NOT_FOUND, dtype=np.uint64)
        rows = unsat_rows(curve.r, 3, r1cs_terms(curve.r), cs2.to_matrices(), cs.z())
        want[broken] = rows[0]
        assert np.array_equal(first[:, 0], want)
        assert int(count[:, 0].sum()) == len(broken) * len(rows)
    be.r1cs_free(m)


# ---- 6. agreement with proving ----------------------------------------------------------------------------------------
@gpu
def test_check_agrees_with_prove_and_verify(be):
    """K assignments, some unsatisfying: the check's verdicts are those of b2s_groth16_prove_batch + b2s_groth16_verify_batch"""
    curve = CURVES[be.curve]
    rng = random.Random(0xC4EC + be.curve)
    csr, n_rows, n_inst, n_wit, z = dummy_rows(curve, 10, 50)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    pkh, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst)
    K = 12
    zs = np.tile(z, (K, 1)).reshape(K, -1, 8)
    for k in (1, 4, 5, 11):
        zs[k, 4 + rng.randrange(50)] = pack_fr(curve, [rng.randrange(curve.r)])
    zs = zs.reshape(K, -1)
    first, _ = be.r1cs_check(m, zs)
    sat = first[:, 0] == NOT_FOUND
    assert sat.tolist() == [k not in (1, 4, 5, 11) for k in range(K)]
    r = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
    s = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
    a, b, c = be.groth16_prove_batch(pkh, m, zs, r, s)
    inputs = np.ascontiguousarray(zs.reshape(K, -1, 8)[:, 1:n_inst].reshape(-1))
    pvk = be.vk_prepare(vk)
    ok = be.groth16_verify_batch(pvk, inputs, n_inst - 1, a.reshape(-1), b.reshape(-1), c.reshape(-1))
    assert ok.tolist() == sat.tolist()
    be.pvk_free(pvk)
    be.pk_free(pkh)
    be.r1cs_free(m)


# ---- 7. errors --------------------------------------------------------------------------------------------------------
def raw_upload(be, n_instance, n_witness, descs, keep):
    """b2s_gr1cs_upload on hand-made descriptors -> (status, b2s_last_error)"""
    import ctypes

    from snark_b200.lib import PredicateDesc

    arr = (PredicateDesc * max(len(descs), 1))(*descs)
    h = ctypes.c_void_p()
    st = be.lib.b2s_gr1cs_upload(be.h, n_instance, n_witness, len(descs), arr, ctypes.byref(h))
    if st == 0:
        be.lib.b2s_gr1cs_free(be.h, h)
    return st, be.lib.b2s_last_error(be.h).decode()


def good_desc(curve, keep, arity=2, rows=None, terms=None):
    """one predicate x0 * x1 (or `terms`) over `rows` (default: two rows reading columns 1 and 2)"""
    from snark_b200.lib import PredicateDesc

    rows = rows if rows is not None else [[[(1, 1)], [(1, 2)]] for _ in range(arity)]
    terms = terms if terms is not None else [(1, [(j, 1) for j in range(arity)])]
    d = PredicateDesc()
    co = pack_fr(curve, [c for c, _ in terms])
    offs = np.array([0] + list(np.cumsum([len(t) for _, t in terms])), dtype=np.uint32)
    fv = np.array([v for _, t in terms for v, _ in t] or [0], dtype=np.uint32)
    fp = np.array([e for _, t in terms for _, e in t] or [0], dtype=np.uint32)
    keep += [co, offs, fv, fp]
    d.arity, d.n_terms, d.n_rows = arity, len(terms), len(rows[0])
    d.term_coeffs, d.term_offsets, d.factor_var, d.factor_pow = co.ctypes.data, offs.ctypes.data, fv.ctypes.data, fp.ctypes.data
    for j in range(min(arity, 8)):
        csr = csr_from_rows(curve, rows[j])
        keep += csr
        d.row_ptr[j], d.col[j], d.coeff[j] = (a.ctypes.data for a in csr)
    return d


@gpu
def test_errors(be):
    from snark_b200 import B2SError, Backend

    curve = CURVES[be.curve]
    keep = []
    st, msg = raw_upload(be, 1, 2, [good_desc(curve, keep), good_desc(curve, keep, arity=8)], keep)
    assert st == 0, msg
    cases = []
    d = good_desc(curve, keep)
    d.arity = 0
    cases.append(([good_desc(curve, keep), d], 16, "predicate 1: arity 0"))
    d = good_desc(curve, keep, arity=8)
    d.arity = 9
    cases.append(([d], 16, "predicate 0: arity 9"))
    d = good_desc(curve, keep, terms=[(1, [(0, 1)]), (1, [(1, 2), (2, 1)])])
    cases.append(([d], 16, "predicate 0: factor_var[2] = 2 >= arity 2"))
    d = good_desc(curve, keep, terms=[(1, [(0, 1)]), (1, [(1, 2)])])
    offs = np.array([0, 2, 1], dtype=np.uint32)
    keep.append(offs)
    d.term_offsets = offs.ctypes.data
    cases.append(([d], 16, "term_offsets not monotone at term 1"))
    d = good_desc(curve, keep)
    d.term_coeffs = None
    cases.append(([d], 16, "predicate 0: null term arrays"))
    d = good_desc(curve, keep)
    d.row_ptr[1] = None
    cases.append(([good_desc(curve, keep), d], 16, "predicate 1: null CSR array for argument 1"))
    d = good_desc(curve, keep)
    rp = np.array([0, 1, 0], dtype=np.uint64)
    keep.append(rp)
    d.row_ptr[1] = rp.ctypes.data
    cases.append(([d], 16, "gr1cs: predicate 0: row_ptr[1] not monotone"))
    d = good_desc(curve, keep, rows=[[[(1, 1)], [(1, 3)]], [[(1, 2)], [(1, 2)]]])
    cases.append(([d], 2, "gr1cs: predicate 0: column 3 >= 3 variables"))
    for descs, code, text in cases:
        st, msg = raw_upload(be, 1, 2, descs, keep)
        assert st == code and text in msg, (code, text, st, msg)
    st, msg = raw_upload(be, 1, 1 << 32, [good_desc(curve, keep)], keep)
    assert st == 5 and "columns are u32" in msg
    st, msg = raw_upload(be, 0, 3, [good_desc(curve, keep)], keep)
    assert st == 16 and "n_instance" in msg
    # a handle of the other curve's ctx
    other = Backend(curve=1 - be.curve)
    try:
        g = other.gr1cs_upload(1, 2, {"p": (2, [(1, [(0, 1), (1, 1)])], [[[(1, 1)]], [[(1, 2)]]])})
        with pytest.raises(B2SError) as e:
            be.gr1cs_check(g, pack_fr(curve, [1, 2, 3]).reshape(1, -1))
        assert e.value.code == 16 and f"uploaded on a ctx of curve {1 - be.curve}" in str(e.value)
        other.gr1cs_free(g)
    finally:
        other.close()
    # null buffers
    g = be.gr1cs_upload(1, 2, {"p": (2, [(1, [(0, 1), (1, 1)])], [[[(1, 1)]], [[(1, 2)]]])})
    with pytest.raises(B2SError) as e:
        be._ck(be.lib.b2s_gr1cs_check(be.h, g.h, 1, None, 0, None, None))
    assert e.value.code == 16 and "null buffer" in str(e.value)
    assert be.lib.b2s_gr1cs_check(be.h, g.h, 0, None, 0, None, None) == 0   # n_assign == 0: nothing read or written
    be.gr1cs_free(g)
    with pytest.raises(B2SError) as e:
        be._ck(be.lib.b2s_r1cs_check(be.h, None, 1, None, 0, None, None))
    assert e.value.code == 1


@gpu
def test_many_predicates_bound_the_output_scratch(be):
    """4096 one-row predicates x0 - p: the outputs of a chunk (16 B per predicate and assignment) are bounded like z, so 1030
    assignments take two chunks; host and device buffers, with and without counts"""
    import torch

    curve = CURVES[be.curve]
    r = curve.r
    P, K = 4096, 1030
    assert CHECK_SCRATCH_BYTES // (16 * P) == 1024
    preds = {f"p{p:05d}": (1, [(1, [(0, 1)]), (r - p, [])], [[[(1, 1)]]]) for p in range(P)}
    g = be.gr1cs_upload(1, 1, preds)
    vals = [(7 * i) % P for i in range(K)]
    zs = pack_fr(curve, [v for x in vals for v in (1, x)]).reshape(K, -1)
    want_first = np.zeros((K, P), dtype=np.uint64)
    want_first[np.arange(K), vals] = NOT_FOUND
    for zz in (zs, torch.from_numpy(zs.view(np.int32)).cuda()):
        for counts in (True, False):
            first, count = be.gr1cs_check(g, zz, counts=counts)
            assert np.array_equal(first, want_first)
            if counts:
                assert np.array_equal(count, (want_first == 0).astype(np.uint64))
    be.gr1cs_free(g)


@gpu
def test_assignment_width_is_checked(be):
    """z rows narrower or wider than n_vars, or not 32-bit limbs, never reach the library"""
    import torch

    curve = CURVES[be.curve]
    g = be.gr1cs_upload(1, 2, {"p": (2, [(1, [(0, 1), (1, 1)])], [[[(1, 1)]], [[(1, 2)]]])})
    m = be.r1cs_upload(1, 1, 2, [csr_from_rows(curve, mm) for mm in ([[(1, 1)]], [[(1, 2)]], [[]])])
    good = pack_fr(curve, [1, 2, 0]).reshape(1, -1)
    for bad in (good[:, :-8], np.hstack([good, good[:, :8]]), good.reshape(-1), good.view(np.uint64),
                torch.from_numpy(good[:, :-8].copy().view(np.int32)).cuda()):
        with pytest.raises(ValueError):
            be.gr1cs_check(g, bad)
        with pytest.raises(ValueError):
            be.r1cs_check(m, bad)
    with pytest.raises(ValueError):
        be.which_is_unsatisfied(g, good[0, :-8])
    assert be.which_is_unsatisfied(g, good[0]) is None
    assert be.r1cs_check(m, good)[0][0, 0] == NOT_FOUND
    be.r1cs_free(m)
    with pytest.raises(ValueError):
        be.r1cs_check(m, good)
    be.gr1cs_free(g)
