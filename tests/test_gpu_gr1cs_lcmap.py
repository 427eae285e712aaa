"""b2s_gr1cs_upload_lcmap: the GR1CS handle built on the device from the constraint system's LcMap (every predicate's
argument_lcs, one shared LcMap and interner pool) must check exactly as the b2s_gr1cs_upload handle of to_matrices() does,
and as the oracle's which_is_unsatisfied: the reference's circuits, random GR1CS through the oracle builder, batches across
the check's chunk bounds, about 2^22 constraints generated in numpy with planted failures, and every rejected input."""
import ctypes
import random

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests.bls377_oracle import BLS12_377
from tests.gr1cs_lcmap_gen import csr_of, planted, random_z, to_lcmap_all
from tests.test_gpu_gr1cs import expected, predicates_of, r1cs_terms, reference_systems
from tests.util import pack_fr

CURVES = [BLS12_381, BN254, BLS12_377]
NOT_FOUND = (1 << 64) - 1
INVALID_ARG, ASSIGNMENT_MISSING, DEGREE = 16, 2, 5
CHECK_SCRATCH_BYTES = 64 << 20   # per-chunk device scratch of csrc/gr1cs.cu for host assignments
CHECK_MAX_ASSIGN = 65535          # assignments per launch (gridDim.y)
gpu = pytest.mark.gpu


@pytest.fixture(scope="module", params=[0, 1, 2], ids=["bls12_381", "bn254", "bls12_377"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


# ---- systems through the oracle builder -------------------------------------------------------------------------------
def random_system(curve, seed, bump=frozenset()):
    """A random GR1CS with a satisfying assignment, built with the oracle's ConstraintSystem: "R1CS" and 1-6 predicates of
    arity 1-8, some with no constraints.  Arguments are the Zero variable, One, instance and witness variables, LCs shared
    by all predicates, fresh LCs and the empty LC 0; LCs repeat variables and hold zero coefficients and Zero terms.  Each
    polynomial is Q(x_0..x_{a-2}) - x_{a-1} (or zero), and the last argument of each constraint reads a fresh output witness
    solved for Q.  bump: (label, row) pairs whose output witness gets + 1 (the same rng draws, so the same structure).
    Returns (cs, outputs) with outputs[label] the rows that have an output witness."""
    r = curve.r
    rng = random.Random(seed)
    cs = orc.ConstraintSystem(curve)
    for _ in range(rng.randint(0, 3)):
        cs.new_input_variable(lambda v=rng.randrange(r): v)
    for _ in range(rng.randint(1, 8)):
        cs.new_witness_variable(lambda v=rng.randrange(r): v)
    coeff = lambda: rng.choice([1, r - 1, 0, rng.randrange(r)])

    def var():
        k = rng.randrange(3)
        if k == 0:
            return orc.V_ONE
        if k == 1:
            return orc.instance(rng.randrange(cs.num_instance_variables))
        return orc.witness(rng.randrange(cs.num_witness_variables))

    def messy_lc():
        t = [(coeff(), var()) for _ in range(rng.randint(1, 4))]
        if rng.random() < 0.4:
            t.append((coeff(), t[0][1]))           # a repeated variable
        if rng.random() < 0.3:
            t.append((coeff(), orc.V_ZERO))
        return orc.LinearCombination(r, t)

    shared = [cs.new_lc(messy_lc()) for _ in range(rng.randint(1, 6))]

    def arg():
        k = rng.randrange(6)
        if k == 0:
            return orc.V_ZERO
        if k == 1:
            return var()
        if k in (2, 3):
            return rng.choice(shared)
        if k == 4:
            return cs.new_lc(messy_lc())
        return orc.symbolic_lc(0)

    labels = rng.sample([f"pred-{i}" for i in range(10)], rng.randint(1, 6))
    outputs = {}
    for label in ["R1CS"] + labels:
        if label == "R1CS":
            arity, terms, zero_poly = 3, r1cs_terms(r), False
        else:
            arity = rng.randint(1, 8)
            zero_poly = rng.random() < 0.15
            terms = []
            if not zero_poly:
                for _ in range(rng.randint(0, 4)):
                    mono, d = [], rng.randint(0, 5)
                    while d > 0 and arity > 1:
                        e = rng.randint(1, d)
                        mono.append((rng.randrange(arity - 1), e))
                        d -= e
                    terms.append((coeff(), mono))
                terms.append((r - 1, [(arity - 1, 1)]))
            cs.register_predicate(label, arity, terms)
        outputs[label] = []
        for i in range(rng.choice([0, 1, rng.randint(2, 25), rng.randint(2, 25)])):
            args = [arg() for _ in range(arity if zero_poly else arity - 1)]
            if not zero_poly:
                x = [cs._lc_value(v) for v in args]
                q = 0
                for c, mono in terms[:-1]:
                    t = c
                    for v, e in mono:
                        t = t * pow(x[v], e, r)
                    q += t
                c0 = rng.choice([1, r - 1, rng.randrange(1, r)])
                extra = [(coeff(), var())] if rng.random() < 0.3 else []
                rest = sum(c * cs._lc_value(v) for c, v in extra)
                val = (q - rest) * pow(c0, -1, r) + (1 if (label, i) in bump else 0)
                w = cs.new_witness_variable(lambda: val)
                t = [(c0, w)] + extra
                rng.shuffle(t)
                args.append(cs.new_lc(orc.LinearCombination(r, t)))
                outputs[label].append(i)
            if label == "R1CS":
                cs.constraints.append(tuple(args))
            else:
                cs.predicates[label]["constraints"].append(tuple(args))
    return cs, outputs


def bumps(outputs, how):
    pick = {"first": lambda o: o[:1], "last": lambda o: o[-1:], "every": lambda o: o}[how]
    return frozenset((label, i) for label, o in outputs.items() for i in pick(o))


def polys_of(cs):
    """{label: (arity, terms)}: predicates_of without the matrices"""
    return {label: (arity, terms) for label, (arity, terms, _) in predicates_of(cs).items()}


def upload_lcmap(be, cs):
    return be.gr1cs_upload_lcmap(cs.num_instance_variables, cs.num_witness_variables, polys_of(cs), to_lcmap_all(cs))


def first_in_label_order(labels, first):
    return next(((label, int(f)) for label, f in zip(labels, first) if f != NOT_FOUND), None)


# ---- CPU: the LcMap export against to_matrices_all --------------------------------------------------------------------
def expand_lcmap(lm, n_instance):
    """get_lc + make_row (constraint_system.rs:777-804) over the flat arrays of to_lcmap_all: {label: matrices}"""
    off, vs, cs_, pool = lm["offsets"], lm["vars"], lm["coeffs"], lm["pool"]

    def row(a):
        tag, idx = a >> 61, a & ((1 << 61) - 1)
        terms = [] if tag == orc.ZERO else [(pool[cs_[e]], vs[e]) for e in range(off[idx], off[idx + 1])] if tag == orc.LC else [(1, a)]
        out = []
        for c, v in terms:
            vt, vi = v >> 61, v & ((1 << 61) - 1)
            if c != 0 and vt != orc.ZERO:
                out.append((c, orc.variable_index((vt, vi), n_instance)))
        return out

    return {label: [[row(a) for a in arg] for arg in args] for label, args in lm["args"].items()}


def cpu_systems(curve):
    for name, cs in reference_systems(curve):
        yield name, cs
    for seed in range(30):
        yield f"random-{seed}", random_system(curve, seed)[0]


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
def test_lcmap_export_expands_to_to_matrices_all(curve):
    for name, cs in cpu_systems(curve):
        lm = to_lcmap_all(cs)
        assert list(lm["args"]) == sorted(["R1CS"] + list(cs.predicates)), name
        assert lm["pool"][:2] == [1, curve.r - 1] and lm["offsets"][:2] == [0, 0], name
        assert expand_lcmap(lm, cs.num_instance_variables) == cs.to_matrices_all(), name


def test_random_systems_against_the_oracle():
    """the generator's assignments satisfy every predicate, and each bump breaks the system"""
    for curve in CURVES:
        for seed in range(30):
            cs, outputs = random_system(curve, seed)
            assert cs.is_satisfied(), seed
            if any(outputs.values()):
                bad, _ = random_system(curve, seed, bumps(outputs, "first"))
                assert bad.to_matrices_all() == cs.to_matrices_all() and not bad.is_satisfied(), seed
                first = expected(curve, predicates_of(bad), bad.z())[0]
                assert first_in_label_order(sorted(to_lcmap_all(bad)["args"]), first) == bad.which_is_unsatisfied(), seed


def test_planted_generator_csr_matches_make_row():
    """the numpy CSR of the planted systems is make_row(get_lc(.)) of the same arrays, and only the planted rows fail"""
    curve = BN254
    r = curve.r
    bad = {"a": [0, 5], "b": [], "c": [39]}
    preds, lm = planted(r, {"a": (2, 40), "b": (3, 30), "c": (5, 40)}, 3, 20, seed=7, bad=bad, n_shared=16)
    ref = expand_lcmap({**lm, "offsets": lm["offsets"].tolist(), "vars": lm["vars"].tolist(), "coeffs": lm["coeffs"].tolist(),
                        "args": {k: [a.tolist() for a in v] for k, v in lm["args"].items()}}, 3)
    z = [1] + [random.Random(3).randrange(r) for _ in range(22)]
    for label, (arity, terms) in preds.items():
        mats = []
        for j, a in enumerate(lm["args"][label]):
            rp, col, ids = csr_of(lm, 3, a)
            mats.append([[(lm["pool"][int(ids[e])], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(a))])
        assert mats == ref[label], label
        x = [[sum(c * z[col] for c, col in m[i]) % r for m in mats] for i in range(len(mats[0]))]
        fails = [i for i, xi in enumerate(x) if (sum(xi[j] for j in range(arity) if j != 1) - xi[1]) % r]
        assert fails == bad[label], label


# ---- 1. parity on small systems ---------------------------------------------------------------------------------------
@gpu
def test_reference_circuits(be):
    curve = CURVES[be.curve]
    seen = set()
    for name, cs in reference_systems(curve):
        g_lc, g_m = upload_lcmap(be, cs), be.gr1cs_upload(cs.num_instance_variables, cs.num_witness_variables, predicates_of(cs))
        assert g_lc.labels == g_m.labels
        z = pack_fr(curve, cs.z()).reshape(1, -1)
        f1, c1 = be.gr1cs_check(g_lc, z)
        f2, c2 = be.gr1cs_check(g_m, z)
        assert np.array_equal(f1, f2) and np.array_equal(c1, c2), name
        want = cs.which_is_unsatisfied()
        assert be.which_is_unsatisfied(g_lc, z[0]) == want, name
        seen.add(want)
        be.gr1cs_free(g_lc)
        be.gr1cs_free(g_m)
    assert None in seen and ("poly-predicate-A", 0) in seen and ("R1CS", 0) in seen and ("R1CS", 1) in seen


@gpu
def test_random_systems(be):
    curve = CURVES[be.curve]
    for seed in range(24):
        seed += 1000 * be.curve
        cs, outputs = random_system(curve, seed)
        systems = [cs] + [random_system(curve, seed, bumps(outputs, how))[0] for how in ("first", "last", "every") if any(outputs.values())]
        g_lc, g_m = upload_lcmap(be, cs), be.gr1cs_upload(cs.num_instance_variables, cs.num_witness_variables, predicates_of(cs))
        z = pack_fr(curve, [v for s in systems for v in s.z()]).reshape(len(systems), -1)
        f1, c1 = be.gr1cs_check(g_lc, z)
        f2, c2 = be.gr1cs_check(g_m, z)
        assert np.array_equal(f1, f2) and np.array_equal(c1, c2), seed
        for i, s in enumerate(systems):
            assert (f1[i].tolist(), c1[i].tolist()) == expected(curve, predicates_of(s), s.z()), (seed, i)
            assert first_in_label_order(g_lc.labels, f1[i]) == s.which_is_unsatisfied(), (seed, i)
        be.gr1cs_free(g_lc)
        be.gr1cs_free(g_m)


# ---- the planted systems: the matrix handle from the same arrays ------------------------------------------------------
def csr_handle(be, curve, n_instance, n_witness, preds, lm):
    """b2s_gr1cs_upload of the to_matrices() export of a planted system (csr_of), from the same arrays"""
    from snark_b200 import lib as L

    labels = sorted(preds)
    pool = pack_fr(curve, lm["pool"]).reshape(-1, 8)
    descs = (L.PredicateDesc * len(labels))()
    keep = []
    for d, label in zip(descs, labels):
        arity, terms = preds[label]
        co = pack_fr(curve, [c for c, _ in terms])
        offs = np.arange(len(terms) + 1, dtype=np.uint32)
        fv = np.array([m[0][0] for _, m in terms], dtype=np.uint32)
        fp = np.ones(len(terms), dtype=np.uint32)
        keep += [co, offs, fv, fp]
        d.arity, d.n_terms, d.n_rows = arity, len(terms), len(lm["args"][label][0])
        d.term_coeffs, d.term_offsets, d.factor_var, d.factor_pow = co.ctypes.data, offs.ctypes.data, fv.ctypes.data, fp.ctypes.data
        for j, a in enumerate(lm["args"][label]):
            rp, col, ids = csr_of(lm, n_instance, a)
            limbs = np.ascontiguousarray(pool[ids])
            keep += [rp, col, limbs]
            d.row_ptr[j], d.col[j], d.coeff[j] = rp.ctypes.data, col.ctypes.data, limbs.ctypes.data
    h = ctypes.c_void_p()
    be._ck(be.lib.b2s_gr1cs_upload(be.h, n_instance, n_witness, len(labels), descs, ctypes.byref(h)))
    return L.Gr1cs(h, labels, n_instance + n_witness)


def planted_expected(shape, bad):
    labels = sorted(shape)
    return ([min(bad[label]) if bad[label] else NOT_FOUND for label in labels], [len(set(bad[label])) for label in labels])


# ---- 2. batches -------------------------------------------------------------------------------------------------------
@gpu
def test_batches_across_chunk_boundaries(be):
    """host chunks bounded by scratch (2^16-variable rows: 32 per chunk), host and device; then more assignments than one
    launch takes (65 535), on circuit2 with every 997th assignment failing row 1"""
    import torch

    curve = CURVES[be.curve]
    n_inst, n_wit = 3, (1 << 16) - 3
    per_chunk = CHECK_SCRATCH_BYTES // (32 * (n_inst + n_wit))
    assert per_chunk == 32
    shape = {"a": (2, 3000), "b": (3, 2000), "c": (5, 1000)}
    bad = {"a": [7, 2999], "b": [], "c": [0, 1, 500]}
    preds, lm = planted(curve.r, shape, n_inst, n_wit, seed=11 + be.curve, bad=bad, n_shared=256)
    g_lc = be.gr1cs_upload_lcmap(n_inst, n_wit, preds, lm)
    g_m = csr_handle(be, curve, n_inst, n_wit, preds, lm)
    K = per_chunk + 3
    zs = random_z(K, n_inst + n_wit, seed=5)
    want_first, want_count = planted_expected(shape, bad)
    for zz in (zs, torch.from_numpy(zs.view(np.int32)).cuda()):
        f1, c1 = be.gr1cs_check(g_lc, zz)
        f2, c2 = be.gr1cs_check(g_m, zz)
        assert np.array_equal(f1, f2) and np.array_equal(c1, c2)
        assert f1.tolist() == [want_first] * K and c1.tolist() == [want_count] * K
    be.gr1cs_free(g_lc)
    be.gr1cs_free(g_m)

    good, broken = orc.circuit2(curve, 1, 1, 2), orc.circuit2(curve, 2, 1, 4)
    for cs in (good, broken):
        cs.finalize()
    g = upload_lcmap(be, good)
    K = CHECK_MAX_ASSIGN + 100
    zs = np.tile(pack_fr(curve, good.z()), (K, 1))
    rows = np.arange(0, K, 997)
    zs[rows] = pack_fr(curve, broken.z())
    want = np.full(K, NOT_FOUND, dtype=np.uint64)
    want[rows] = broken.which_is_unsatisfied()[1]
    for zz in (zs, torch.from_numpy(zs.view(np.int32)).cuda()):
        first, count = be.gr1cs_check(g, zz)
        assert np.array_equal(first[:, 0], want)
        assert int(count[:, 0].sum()) == len(rows) * expected(curve, predicates_of(broken), broken.z())[1][0]
    be.gr1cs_free(g)


# ---- 3. at scale ------------------------------------------------------------------------------------------------------
@gpu
def test_planted_system_at_2_22_constraints(be):
    """2^22 constraints over predicates of arity 2, 3 and 5, generated in numpy: both handles report exactly the planted rows"""
    curve = CURVES[be.curve]
    n_inst, n_wit = 5, (1 << 20) - 5
    shape = {"p2": (2, 1 << 21), "p3": (3, 1 << 20), "p5": (5, 1 << 20)}
    rng = np.random.default_rng(be.curve)
    bad = {"p2": sorted({0, (1 << 21) - 1, *rng.integers(0, 1 << 21, 100).tolist()}),
           "p3": sorted(rng.integers(1000, 1 << 20, 37).tolist()),
           "p5": [(1 << 20) - 1]}
    preds, lm = planted(curve.r, shape, n_inst, n_wit, seed=be.curve, bad=bad)
    g_lc = be.gr1cs_upload_lcmap(n_inst, n_wit, preds, lm)
    g_m = csr_handle(be, curve, n_inst, n_wit, preds, lm)
    del lm
    zs = random_z(2, n_inst + n_wit, seed=9)
    f1, c1 = be.gr1cs_check(g_lc, zs)
    f2, c2 = be.gr1cs_check(g_m, zs)
    want_first, want_count = planted_expected(shape, bad)
    assert f1.tolist() == [want_first] * 2 and c1.tolist() == [want_count] * 2
    assert np.array_equal(f1, f2) and np.array_equal(c1, c2)
    be.gr1cs_free(g_lc)
    be.gr1cs_free(g_m)


# ---- 4. errors --------------------------------------------------------------------------------------------------------
def raw_upload_lcmap(be, n_instance, n_witness, descs, lm, pool=None, n_lcs=None):
    """b2s_gr1cs_upload_lcmap on hand-made descriptors and LcMap arrays -> (status, b2s_last_error)"""
    from snark_b200.lib import PredicateLcmapDesc

    arr = (PredicateLcmapDesc * max(len(descs), 1))(*descs)
    off = np.asarray(lm["offsets"], dtype=np.uint64)
    vs = np.asarray(lm["vars"] or [0], dtype=np.uint64)
    co = np.asarray(lm["coeffs"] or [0], dtype=np.uint32)
    pool = pool if pool is not None else pack_fr(CURVES[be.curve], lm["pool"])
    h = ctypes.c_void_p()
    st = be.lib.b2s_gr1cs_upload_lcmap(be.h, n_instance, n_witness, len(descs), arr, len(off) - 1 if n_lcs is None else n_lcs,
                                       off.ctypes.data, vs.ctypes.data, co.ctypes.data, pool.ctypes.data, len(pool) // 8, ctypes.byref(h))
    if st == 0:
        be.lib.b2s_gr1cs_free(be.h, h)
    return st, be.lib.b2s_last_error(be.h).decode()


def good_desc(curve, keep, args, terms=None):
    """one predicate over `args` (lists of raw Variables, one per argument), polynomial x0 * x1 * ... or `terms`"""
    from snark_b200.lib import PredicateLcmapDesc

    arity = len(args)
    terms = terms if terms is not None else [(1, [(j, 1) for j in range(arity)])]
    d = PredicateLcmapDesc()
    co = pack_fr(curve, [c for c, _ in terms])
    offs = np.array([0] + list(np.cumsum([len(t) for _, t in terms])), dtype=np.uint32)
    fv = np.array([v for _, t in terms for v, _ in t] or [0], dtype=np.uint32)
    fp = np.array([e for _, t in terms for _, e in t] or [0], dtype=np.uint32)
    keep += [co, offs, fv, fp]
    d.arity, d.n_terms, d.n_rows = arity, len(terms), len(args[0])
    d.term_coeffs, d.term_offsets, d.factor_var, d.factor_pow = co.ctypes.data, offs.ctypes.data, fv.ctypes.data, fp.ctypes.data
    for j, a in enumerate(args[:8]):
        a = np.asarray(a, dtype=np.uint64)
        keep.append(a)
        d.args[j] = a.ctypes.data
    return d


@gpu
def test_errors(be):
    from snark_b200 import B2SError, Backend

    curve = CURVES[be.curve]
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    lm = to_lcmap_all(cs)
    n_inst, n_wit = cs.num_instance_variables, cs.num_witness_variables
    W = lambda i: (3 << 61) | i
    LC = lambda i: (4 << 61) | i
    keep = []
    ok = lambda: good_desc(curve, keep, [[W(0), LC(1)], [W(1), 0]])
    st, msg = raw_upload_lcmap(be, n_inst, n_wit, [ok(), good_desc(curve, keep, [[W(0)]] * 8)], lm)
    assert st == 0, msg
    cases = []   # (descs, n_instance, n_witness, lm, status, text)
    d = ok()
    d.arity = 0
    cases.append(([ok(), d], n_inst, n_wit, lm, INVALID_ARG, "predicate 1: arity 0"))
    d = good_desc(curve, keep, [[W(0)]] * 8)
    d.arity = 9
    cases.append(([d], n_inst, n_wit, lm, INVALID_ARG, "predicate 0: arity 9"))
    cases.append(([good_desc(curve, keep, [[W(0)], [W(1)]], terms=[(1, [(0, 1)]), (1, [(1, 2), (2, 1)])])], n_inst, n_wit, lm,
                  INVALID_ARG, "predicate 0: factor_var[2] = 2 >= arity 2"))
    d = good_desc(curve, keep, [[W(0)], [W(1)]], terms=[(1, [(0, 1)]), (1, [(1, 2)])])
    offs = np.array([0, 2, 1], dtype=np.uint32)
    keep.append(offs)
    d.term_offsets = offs.ctypes.data
    cases.append(([d], n_inst, n_wit, lm, INVALID_ARG, "term_offsets not monotone at term 1"))
    d = ok()
    offs = np.array([1, 1, 2], dtype=np.uint32)
    keep.append(offs)
    d.term_offsets = offs.ctypes.data
    cases.append(([d], n_inst, n_wit, lm, INVALID_ARG, "predicate 0: term_offsets[0] != 0"))
    d = ok()
    d.n_rows = 1 << 32
    cases.append(([d], n_inst, n_wit, lm, DEGREE, "predicate 0: 4294967296 constraints"))
    d = ok()
    d.term_coeffs = None
    cases.append(([d], n_inst, n_wit, lm, INVALID_ARG, "predicate 0: null term arrays"))
    d = ok()
    d.args[1] = None
    cases.append(([ok(), d], n_inst, n_wit, lm, INVALID_ARG, "predicate 1: null argument array 1"))
    cases.append(([ok()], 0, n_wit + 1, lm, INVALID_ARG, "n_instance"))
    cases.append(([ok()], 1, 1 << 32, lm, DEGREE, "columns are u32"))
    # the LcMap
    cases.append(([ok()], n_inst, n_wit, dict(lm, offsets=[1] + lm["offsets"][1:]), INVALID_ARG, "offsets must start with 0"))
    bad_off = list(lm["offsets"])
    bad_off[2] = bad_off[3] + 1
    cases.append(([ok()], n_inst, n_wit, dict(lm, offsets=bad_off), INVALID_ARG, "offsets not monotone at 2"))
    cases.append(([ok()], n_inst, n_wit, dict(lm, pool=lm["pool"][:1]), INVALID_ARG, "at least ONE and -ONE"))
    cases.append(([ok()], n_inst, n_wit, dict(lm, pool=[2] + lm["pool"][1:]), INVALID_ARG, "pool[0] is not ONE"))
    nested = to_lcmap_all(orc.circuit2(curve, 1, 1, 2))                 # not finalized: LC e = d + d refers to LC d
    cases.append(([good_desc(curve, keep, [[LC(i) for i in range(1, len(nested["offsets"]) - 1)]])], n_inst, n_wit, nested,
                  INVALID_ARG, "call finalize()"))
    cases.append(([ok(), good_desc(curve, keep, [[W(0)], [W(1)], [W(0), LC(99)][1:]])], n_inst, n_wit, lm, INVALID_ARG,
                  "predicate 1, argument 2, constraint 0: lcmap: malformed input (error bits 0x2"))
    cases.append(([good_desc(curve, keep, [[W(0), W(1), (5 << 61) | 1]])], n_inst, n_wit, lm, INVALID_ARG,
                  "predicate 0, argument 0, constraint 2: lcmap: malformed input (error bits 0x1"))
    cases.append(([ok()], n_inst, n_wit, dict(lm, coeffs=[len(lm["pool"])] + lm["coeffs"][1:]), INVALID_ARG, "error bits 0x10"))
    cases.append(([ok(), good_desc(curve, keep, [[W(1)], [W(50)]])], n_inst, n_wit, lm, ASSIGNMENT_MISSING,
                  "predicate 1, argument 1, constraint 0: lcmap: a variable index is outside the"))
    cases.append(([good_desc(curve, keep, [[(2 << 61) | n_inst]])], n_inst, n_wit, lm, ASSIGNMENT_MISSING, "outside the"))
    d = good_desc(curve, keep, [[W(0)], [W(1)]])
    d.n_rows = 1 << 31                                                   # 2^32 (argument, row) slots; nothing is read
    cases.append(([d], n_inst, n_wit, lm, DEGREE, "lcmap: too many rows"))
    # 2^16 + 1 rows of one LC with 2^16 terms: more nonzeros than the 32-bit scan holds (rejected before the fill)
    big = {"offsets": [0, 0, 1 << 16], "vars": [1 << 61] * (1 << 16), "coeffs": [0] * (1 << 16), "pool": lm["pool"]}
    cases.append(([good_desc(curve, keep, [[LC(1)] * ((1 << 16) + 1)])], n_inst, n_wit, big, DEGREE,
                  "4295032832 nonzeros in the arguments of all predicates"))
    for descs, ni, nw, lmap, code, text in cases:
        st, msg = raw_upload_lcmap(be, ni, nw, descs, lmap)
        assert st == code and text in msg, (code, text, st, msg)
    # null pointers
    st, msg = raw_upload_lcmap(be, n_inst, n_wit, [ok()], lm, pool=np.zeros(0, dtype=np.uint32))
    assert st == INVALID_ARG and msg
    assert be.lib.b2s_gr1cs_upload_lcmap(be.h, 1, 1, 1, None, 1, None, None, None, None, 2, None) == INVALID_ARG
    # zero predicates: a valid handle that checks nothing
    g = be.gr1cs_upload_lcmap(n_inst, n_wit, {}, dict(lm, args={}))
    assert be.gr1cs_check(g, pack_fr(curve, cs.z()).reshape(1, -1))[0].shape == (1, 0)
    be.gr1cs_free(g)
    # a handle of the other curve's ctx
    other = Backend(curve=(be.curve + 1) % 3)
    try:
        g = other.gr1cs_upload_lcmap(n_inst, n_wit, polys_of(cs), lm)
        with pytest.raises(B2SError) as e:
            be.gr1cs_check(g, pack_fr(curve, cs.z()).reshape(1, -1))
        assert e.value.code == INVALID_ARG and f"uploaded on a ctx of curve {(be.curve + 1) % 3}" in str(e.value)
        other.gr1cs_free(g)
    finally:
        other.close()
