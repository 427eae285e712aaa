"""Instance outlining (ConstraintSystem::finalize with an InstanceOutliner, relations/src/gr1cs/constraint_system.rs:826-863,
instance_outliner.rs:40-80) for the tests, in two forms:

  * the square-R1CS pieces the Python oracle's ConstraintSystem lacks: the "SR1CS" predicate x0^2 - x1
    (predicate/mod.rs:124-129), lc_diff! (linear_combination.rs:32-38) and the outline_sr1cs strategy, to use with its
    set_instance_outliner / finalize next to oracle.r1cs.outline_r1cs;
  * outline_lcmap, the same rewrite restated in numpy on the flat LcMap layout of tests/gr1cs_lcmap_gen.py, so that
    csr_of of its result is to_matrices() of the outlined system at any size.

Pinned against the C++ mirror's outline_r1cs / outline_sr1cs (snark_b200/host/ark_relations.hpp) by tests/test_outline_oracle.py."""
import numpy as np

from oracle import r1cs as orc
from tests.gr1cs_lcmap_gen import SHIFT, TAG_INSTANCE, TAG_LC, TAG_ONE, TAG_WITNESS, raw

OUTLINE_R1CS, OUTLINE_SR1CS = 1, 2
MASK = np.uint64((1 << 61) - 1)


def r1cs_terms(r):
    """x0 * x1 - x2 (predicate/mod.rs:116-121) as register_predicate terms"""
    return [(1, [(0, 1), (1, 1)]), (r - 1, [(2, 1)])]


def sr1cs_terms(r):
    """x0^2 - x1 (predicate/mod.rs:124-129)"""
    return [(1, [(0, 2)]), (r - 1, [(1, 1)])]


def register_sr1cs(cs):
    cs.register_predicate("SR1CS", 2, sr1cs_terms(cs.r))


def lc_diff(r, a, b):
    """lc_diff!(a, b) = LinearCombination::diff_vars: [(ONE, a), (-ONE, b)], not compactified; empty when a == b"""
    return orc.LinearCombination(r, [] if a == b else [(1, a), (r - 1, b)])


def enforce_sr1cs_constraint(cs, a, b):
    cs.enforce_constraint("SR1CS", [a, b])


def outline_sr1cs(cs, instance_witness_map):
    """instance_outliner.rs:63-80: (x_i - w_i)^2 = 0 for every instance variable, the constant (Instance(0)) included"""
    for i, w in enumerate(instance_witness_map):
        enforce_sr1cs_constraint(cs, lc_diff(cs.r, orc.instance(i), w), orc.LinearCombination(cs.r))


def outline_lcmap(lcmap, n_instance, n_witness, strategy, label):
    """The LcMap (layout of gr1cs_lcmap_gen.to_lcmap_all / planted) after perform_instance_outlining with `strategy`, whose tie
    rows go to predicate `label`: One and Instance(i) in every stored LC become the witness copies W and W + i (W = n_witness),
    bare arguments stay, and the strategy's tie rows (and for outline_sr1cs their LCs) are appended.  Returns a new dict;
    its variables count n_instance + n_witness + n_instance."""
    v = np.asarray(lcmap["vars"], dtype=np.uint64)
    tag, idx = v >> SHIFT, v & MASK
    W = n_witness
    v = np.where(tag == TAG_ONE, raw(TAG_WITNESS, W), np.where(tag == TAG_INSTANCE, raw(TAG_WITNESS, W + idx), v))
    off = np.asarray(lcmap["offsets"], dtype=np.uint64)
    coeffs = np.asarray(lcmap["coeffs"], dtype=np.uint32)
    args = {k: [np.asarray(a, dtype=np.uint64) for a in a_list] for k, a_list in lcmap["args"].items()}
    i = np.arange(n_instance, dtype=np.uint64)
    tie = args[label]
    if strategy == OUTLINE_R1CS:
        assert len(tie) == 3
        c = np.where(i == 0, raw(TAG_ONE, 0), raw(TAG_INSTANCE, i))
        add = [np.full(n_instance, raw(TAG_WITNESS, W), np.uint64), raw(TAG_WITNESS, W + i), c]
    else:
        assert strategy == OUTLINE_SR1CS and len(tie) == 2
        n_lcs, total = len(off) - 1, int(off[-1])
        v = np.concatenate([v, np.stack([raw(TAG_INSTANCE, i), raw(TAG_WITNESS, W + i)], axis=1).reshape(-1)])
        coeffs = np.concatenate([coeffs, np.tile(np.array([0, 1], np.uint32), n_instance)])
        off = np.concatenate([off, total + 2 * (i + 1)])
        add = [raw(TAG_LC, n_lcs + i), np.full(n_instance, raw(TAG_LC, 0), np.uint64)]
    args[label] = [np.concatenate([a, b]) for a, b in zip(tie, add)]
    return {"offsets": off, "vars": v, "coeffs": coeffs, "pool": lcmap["pool"], "args": args}


def outline_z(z, n_instance):
    """the outlined assignment: z || (ONE, z[1], ..., z[n_instance - 1]) (z[0] = ONE); rows of ints or of limb arrays"""
    return list(z) + [z[0]] + list(z[1:n_instance])
