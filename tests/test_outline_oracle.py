"""Instance outlining in the test oracles, on the CPU: the Python oracle with outline_r1cs / outline_sr1cs
(tests/outline_oracle.py) against the C++ mirror's (snark_b200/host/ark_relations.hpp, through
tests/native/host_outline_dump.cpp), row for row in term order with every assignment element; and the numpy restatement
outline_lcmap against the Python oracle's to_matrices() after finalize().  Random systems mix bare One / Instance / Witness
arguments (which outlining leaves alone) with stored LCs over the same variables, Instance(0), Zero terms and zero
coefficients, in both predicates."""
import os
import random
import subprocess

import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests import outline_oracle as oo
from tests.gr1cs_lcmap_gen import csr_of, to_lcmap_all
from tests.util import pack_fr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "native", "host_outline_dump")
SRC = os.path.join(ROOT, "tests", "native", "host_outline_dump.cpp")
CURVES = [BLS12_381, BN254]
KIND = {0: lambda i: orc.V_ZERO, 1: lambda i: orc.V_ONE, 2: orc.instance, 3: orc.witness}


def build():
    deps = [SRC] + [os.path.join(ROOT, "snark_b200", "host", f) for f in ("ark_relations.hpp", "ark_snark.hpp")]
    if not os.path.exists(EXE) or any(os.path.getmtime(d) > os.path.getmtime(EXE) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", EXE, SRC, "-L", os.path.join(ROOT, "snark_b200"), "-lb200snark",
                               "-Wl,-rpath," + os.path.join(ROOT, "snark_b200")])
    return EXE


def random_system(curve, seed, n_cons=None):
    """(n_inst, n_wit, z, constraints): z the assignment ints (z[0] = 1), constraints [(label "R" / "S", [terms per argument])]
    with terms (kind, index, coeff); an argument is empty, one bare (ONE, v), one scaled term, or 2-5 terms"""
    r = curve.r
    rng = random.Random(seed)
    n_inst, n_wit = rng.randint(1, 5), rng.randint(1, 8)
    z = [1] + [rng.randrange(r) for _ in range(n_inst + n_wit - 1)]

    def var():
        k = rng.choice([0, 1, 2, 2, 3, 3, 3])
        return (k, 0 if k < 2 else rng.randrange(n_inst if k == 2 else n_wit))

    def coeff():
        return rng.choice([1, 1, r - 1, 0, rng.randrange(r)])

    cons = []
    for _ in range(n_cons or rng.randint(1, 12)):
        label = rng.choice("RS")
        args = []
        for _ in range(3 if label == "R" else 2):
            shape = rng.randrange(4)
            if shape == 0:
                args.append([])
            elif shape == 1:
                k, i = var()
                args.append([(k or 1, i, 1)])          # bare: stays as it is under outlining
            elif shape == 2:
                k, i = var()
                args.append([(k, i, rng.randrange(2, r))])
            else:
                args.append([(*var(), coeff()) for _ in range(rng.randint(2, 5))])
        cons.append((label, args))
    return n_inst, n_wit, z, cons


def oracle_cs(curve, system):
    r = curve.r
    n_inst, n_wit, z, cons = system
    cs = orc.ConstraintSystem(curve)
    oo.register_sr1cs(cs)
    for v in z[1:n_inst]:
        cs.new_input_variable(lambda v=v: v)
    for v in z[n_inst:]:
        cs.new_witness_variable(lambda v=v: v)
    for label, args in cons:
        lcs = [orc.LinearCombination(r, [(c, KIND[k](i)) for k, i, c in a]) for a in args]
        cs.enforce_constraint("R1CS" if label == "R" else "SR1CS", lcs)
    return cs


def set_outliner(cs, strategy):
    if strategy == oo.OUTLINE_R1CS:
        cs.set_instance_outliner("R1CS", orc.outline_r1cs)
    elif strategy == oo.OUTLINE_SR1CS:
        cs.set_instance_outliner("SR1CS", oo.outline_sr1cs)


def words(curve, v):
    return " ".join(f"{int(w):08x}" for w in pack_fr(curve, [v]))


def run_mirror(curve, system, strategy, tmp_path):
    """-> ((n_instance, n_witness), {label: [[row of (col, coeff limbs)] per argument]}, z limbs)"""
    n_inst, n_wit, z, cons = system
    lines = [f"{strategy} {n_inst} {n_wit} {len(cons)}"] + [words(curve, v) for v in z[1:]]
    for label, args in cons:
        lines.append(label)
        for a in args:
            lines.append(" ".join([str(len(a))] + [f"{k} {i} {words(curve, c)}" for k, i, c in a]))
    f = tmp_path / f"cs_{curve.name}_{strategy}.txt"
    f.write_text("\n".join(lines) + "\n")
    out = subprocess.run([build(), "0" if curve is BLS12_381 else "1", str(f)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    N, mats, zs = None, {}, []
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        if tag == "N":
            N = (int(rest[0]), int(rest[1]))
        elif tag == "Z":
            zs.append([int(w, 16) for w in rest])
        else:
            label, k, i, terms = rest[0], int(rest[1]), int(rest[2]), rest[3:]
            row = [(int(terms[j]), [int(w, 16) for w in terms[j + 1:j + 9]]) for j in range(0, len(terms), 9)]
            mats.setdefault(label, {}).setdefault(k, {})[i] = row
    return N, mats, zs


def as_limb_rows(curve, mats):
    """to_matrices_all() rows (coeff int, col) -> (col, limbs), as the mirror prints them"""
    return {label: {k: {i: [(col, [int(w) for w in pack_fr(curve, [c])]) for c, col in row] for i, row in enumerate(m)}
                    for k, m in enumerate(ms)} for label, ms in mats.items()}


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("strategy", [0, oo.OUTLINE_R1CS, oo.OUTLINE_SR1CS])
@pytest.mark.parametrize("seed", range(6))
def test_python_oracle_matches_cpp_mirror(curve, strategy, seed, tmp_path):
    system = random_system(curve, 100 * seed + strategy)
    cs = oracle_cs(curve, system)
    n_wit = cs.num_witness_variables
    set_outliner(cs, strategy)
    cs.finalize()
    assert cs.num_witness_variables == n_wit + (cs.num_instance_variables if strategy else 0)
    N, mats, zs = run_mirror(curve, system, strategy, tmp_path)
    assert N == (cs.num_instance_variables, cs.num_witness_variables)
    want = as_limb_rows(curve, cs.to_matrices_all())
    for label in want:   # empty predicates print no rows
        for k in want[label]:
            assert mats.get(label, {}).get(k, {}) == {i: row for i, row in want[label][k].items()}, (label, k)
    assert zs == [[int(w) for w in pack_fr(curve, [v])] for v in cs.z()]
    assert cs.is_satisfied() == (cs.which_is_unsatisfied() is None)


def csr_rows(lcmap, n_instance, arg):
    """csr_of as rows of (coeff int, col)"""
    rp, col, cid = csr_of(lcmap, n_instance, arg)
    pool = lcmap["pool"]
    return [[(pool[cid[e]], int(col[e])) for e in range(int(rp[i]), int(rp[i + 1]))] for i in range(len(rp) - 1)]


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
@pytest.mark.parametrize("strategy", [oo.OUTLINE_R1CS, oo.OUTLINE_SR1CS])
@pytest.mark.parametrize("seed", range(8))
def test_numpy_restatement_matches_oracle(curve, strategy, seed):
    system = random_system(curve, 1000 + 10 * seed + strategy, n_cons=20)
    before = oracle_cs(curve, system)
    before.inline_all_lcs()
    lm = to_lcmap_all(before)
    cs = oracle_cs(curve, system)
    set_outliner(cs, strategy)
    cs.finalize()
    label = "R1CS" if strategy == oo.OUTLINE_R1CS else "SR1CS"
    out = oo.outline_lcmap(lm, before.num_instance_variables, before.num_witness_variables, strategy, label)
    want = cs.to_matrices_all()
    for lab, mats in want.items():
        for k, m in enumerate(mats):
            got = csr_rows(out, cs.num_instance_variables, out["args"][lab][k])
            assert got == [[(c % curve.r, col) for c, col in row] for row in m], (lab, k)
    assert oo.outline_z(before.z(), before.num_instance_variables) == cs.z()


def test_circuit1_instance_outlined():
    """gr1cs/tests/mod.rs:105-133: outlining adds exactly num_instance witnesses"""
    cs = orc.circuit1(BLS12_381, (0,) * 5, (0,) * 8)
    n_inst, n_wit = cs.num_instance_variables, cs.num_witness_variables
    cs.set_instance_outliner("R1CS", orc.outline_r1cs)
    cs.finalize()
    assert cs.num_witness_variables - n_wit == n_inst
