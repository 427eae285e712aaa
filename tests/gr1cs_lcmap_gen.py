"""GR1CS systems generated straight in the LcMap layout with numpy (no oracle object model), at any size, and the CSR of the
same system as to_matrices() would export it; and to_lcmap_all, the same layout of an oracle ConstraintSystem.  Used by
tests/test_gpu_gr1cs_lcmap.py and tools/gr1cs_lcmap_probe.py.

Every predicate of arity a >= 2 has the polynomial  sum_{j != 1} x_j - x_1,  and argument 1 of each constraint is a fresh LC
that restates the other arguments: each of their terms with its coefficient split in two (c = s + (c - s), so the column
repeats), in shuffled order, padded with a zero-coefficient term and a Zero-variable term.  The other arguments are Zero,
a bare variable (One, Instance or Witness) or a SymbolicLc shared by all predicates.  So every constraint holds for every z,
except the rows named in `bad`, whose argument 1 carries one more term (ONE, One): they fail for every z."""
import numpy as np

TAG_ZERO, TAG_ONE, TAG_INSTANCE, TAG_WITNESS, TAG_LC = 0, 1, 2, 3, 4
SHIFT = np.uint64(61)
N_BASE = 6           # pooled coefficients the shared LCs use: ONE, -ONE, 0 and three random values
SHARED_WIDTH = 2     # terms of a shared LC


def to_lcmap_all(cs):
    """The flat storage to_matrices_all() reads, of an oracle ConstraintSystem: cs.to_lcmap()'s offsets, vars, coeffs and
    pool, with args {label: argument_lcs} for every predicate in label order, "R1CS" (arity 3) included; one list of raw
    Variables (tag << 61 | index) per argument."""
    rawv = lambda v: (v[0] << 61) | v[1]
    out = cs.to_lcmap()
    args = {"R1CS": out["args"]}
    for label, pred in cs.predicates.items():
        args[label] = [[rawv(cons[k]) for cons in pred["constraints"]] for k in range(pred["arity"])]
    out["args"] = dict(sorted(args.items()))
    return out


def raw(tag, idx):
    return (np.uint64(tag) << SHIFT) | np.asarray(idx, dtype=np.uint64)


def planted(r, shape, n_instance, n_witness, seed, bad=None, n_shared=1 << 12):
    """shape: {label: (arity >= 2, n_rows)}; bad: {label: row indices}.  Returns (predicates {label: (arity, terms)},
    lcmap in the layout of to_lcmap_all, with numpy arrays and the pool as Python ints)."""
    rng = np.random.default_rng(seed)
    bad = bad or {}
    # the pool: base ids 0..N_BASE-1, then for every base id b a split (split_a[b], split_b[b]) with values summing to it
    base = [1, r - 1, 0] + [int(x) for x in rng.integers(2, 1 << 62, N_BASE - 3)]
    pool = list(base)
    split_a, split_b = np.zeros(N_BASE, np.uint32), np.zeros(N_BASE, np.uint32)
    for b, v in enumerate(base):
        s = int(rng.integers(1, 1 << 62))
        split_a[b], split_b[b] = len(pool), len(pool) + 1
        pool += [s, (v - s) % r]
    ZERO_ID = 2

    def rand_var(n):
        """n random One / Instance / Witness variables"""
        kind = rng.integers(0, 3, n)
        return np.where(kind == 0, raw(TAG_ONE, 0),
                        np.where(kind == 1, raw(TAG_INSTANCE, rng.integers(0, n_instance, n)), raw(TAG_WITNESS, rng.integers(0, n_witness, n))))

    # LC 0 is the empty LC; LCs 1..n_shared have SHARED_WIDTH terms each (some with coefficient 0 or the Zero variable)
    sh_vars = rand_var(n_shared * SHARED_WIDTH).reshape(n_shared, SHARED_WIDTH)
    sh_vars[rng.random(sh_vars.shape) < 0.1] = raw(TAG_ZERO, 0)
    sh_coeffs = rng.integers(0, N_BASE, (n_shared, SHARED_WIDTH)).astype(np.uint32)
    vars_, coeffs = [sh_vars.reshape(-1)], [sh_coeffs.reshape(-1)]
    lens = [np.zeros(1, np.int64), np.full(n_shared, SHARED_WIDTH, np.int64)]
    n_lcs = 1 + n_shared
    preds, args = {}, {}
    for label in sorted(shape):
        arity, n = shape[label]
        assert arity >= 2
        preds[label] = (arity, [(1, [(j, 1)]) for j in range(arity) if j != 1] + [(r - 1, [(1, 1)])])
        cols = []     # argument 1's terms: (var, coeff id) slots of every other argument, then padding
        a = []
        for j in range(arity):
            if j == 1:
                a.append(None)
                continue
            kind = rng.choice(3, n, p=[0.1, 0.4, 0.5])            # Zero, bare variable, shared LC
            lc = rng.integers(0, n_shared + 1, n)                  # LC 0 (empty) now and then
            bare = rand_var(n)
            aj = np.where(kind == 0, raw(TAG_ZERO, 0), np.where(kind == 1, bare, raw(TAG_LC, lc)))
            a.append(aj)
            v = np.zeros((n, 2 * SHARED_WIDTH), np.uint64)        # Zero variable: the slot is dropped
            c = rng.integers(0, len(pool), (n, 2 * SHARED_WIDTH)).astype(np.uint32)
            isb, islc = kind == 1, (kind == 2) & (lc > 0)
            v[isb, 0], v[isb, 1], c[isb, 0], c[isb, 1] = bare[isb], bare[isb], split_a[0], split_b[0]
            k = lc[islc] - 1
            for t in range(SHARED_WIDTH):
                v[islc, 2 * t], v[islc, 2 * t + 1] = sh_vars[k, t], sh_vars[k, t]
                c[islc, 2 * t], c[islc, 2 * t + 1] = split_a[sh_coeffs[k, t]], split_b[sh_coeffs[k, t]]
            cols.append((v, c))
        pad_v = np.stack([rand_var(n), np.zeros(n, np.uint64), np.zeros(n, np.uint64)], axis=1)
        pad_c = np.stack([np.full(n, ZERO_ID, np.uint32), rng.integers(0, len(pool), n).astype(np.uint32), np.zeros(n, np.uint32)], axis=1)
        rows = np.asarray(bad.get(label, []), dtype=np.int64)
        pad_v[rows, 2] = raw(TAG_ONE, 0)                           # the planted failure: + ONE * One
        v = np.concatenate([x for x, _ in cols] + [pad_v], axis=1)
        c = np.concatenate([y for _, y in cols] + [pad_c], axis=1)
        perm = np.argsort(rng.random(v.shape), axis=1)
        v, c = np.take_along_axis(v, perm, axis=1), np.take_along_axis(c, perm, axis=1)
        a[1] = raw(TAG_LC, n_lcs + np.arange(n))
        n_lcs += n
        vars_.append(v.reshape(-1))
        coeffs.append(c.reshape(-1))
        lens.append(np.full(n, v.shape[1], np.int64))
        args[label] = a
    offsets = np.zeros(n_lcs + 1, np.uint64)
    offsets[1:] = np.cumsum(np.concatenate(lens))
    lcmap = {"offsets": offsets, "vars": np.concatenate(vars_), "coeffs": np.concatenate(coeffs), "pool": pool, "args": args}
    return preds, lcmap


def csr_of(lcmap, n_instance, arg):
    """make_row(get_lc(arg[i])) for every i, from the LcMap arrays: (row_ptr u64, col u32, coefficient ids u32)"""
    arg = np.asarray(arg, dtype=np.uint64)
    off, lc_vars, lc_coeffs = lcmap["offsets"], lcmap["vars"], lcmap["coeffs"]
    tag, idx = (arg >> SHIFT).astype(np.int64), (arg & np.uint64((1 << 61) - 1)).astype(np.int64)
    n, n_terms = len(arg), len(lc_vars)
    # a bare variable is the one-term LC (ONE, v): appended after the LcMap's own terms
    is_lc, is_bare = tag == TAG_LC, (tag != TAG_LC) & (tag != TAG_ZERO)
    start = np.where(is_lc, off[np.where(is_lc, idx, 0)].astype(np.int64), n_terms + np.cumsum(is_bare) - 1)
    count = np.where(is_lc, (off[np.where(is_lc, idx + 1, 1)] - off[np.where(is_lc, idx, 0)]).astype(np.int64), is_bare.astype(np.int64))
    ext_vars = np.concatenate([lc_vars, arg[is_bare]])
    ext_coeffs = np.concatenate([lc_coeffs, np.zeros(int(is_bare.sum()), np.uint32)])
    total = int(count.sum())
    row = np.repeat(np.arange(n), count)
    first = np.cumsum(count) - count
    at = np.repeat(start - first, count) + np.arange(total)
    v, c = ext_vars[at], ext_coeffs[at]
    zero_coeff = np.array([x == 0 for x in lcmap["pool"]], dtype=bool)
    vt, vi = (v >> SHIFT).astype(np.int64), (v & np.uint64((1 << 61) - 1)).astype(np.int64)
    keep = (vt != TAG_ZERO) & ~zero_coeff[c]
    col = np.where(vt == TAG_ONE, 0, np.where(vt == TAG_INSTANCE, vi, vi + n_instance))[keep].astype(np.uint32)
    row_ptr = np.zeros(n + 1, np.uint64)
    row_ptr[1:] = np.cumsum(np.bincount(row[keep], minlength=n))
    return row_ptr, col, c[keep]


def random_z(n_assign, n_vars, seed):
    """n_assign rows of n_vars field elements as Montgomery limbs (any value below 2^252 is a reduced element of every
    curve's Fr), z[0] = ONE is not needed: the planted identities hold for every z"""
    rng = np.random.default_rng(seed)
    z = rng.integers(0, 1 << 32, (n_assign, n_vars, 8), dtype=np.uint64).astype(np.uint32)
    z[:, :, 7] &= 0x0FFFFFFF
    return z.reshape(n_assign, -1)
