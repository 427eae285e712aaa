"""The numpy restatement of Sr1csAdapter (tests/sr1cs_oracle.py) against the C++ mirror's
`Sr1csAdapter::r1cs_to_sr1cs_with_assignment` (snark_b200/host/ark_relations.hpp), which restates
relations/src/sr1cs/mod.rs:191-265: the variable counts, both arguments in canonical form and every element of the
converted assignment, on the reference's circuit2 and DummyCircuit and on random R1CS with repeated columns, ONE terms,
unused public inputs and empty rows."""
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests import sr1cs_oracle as so
from tests.util import pack_fr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "native", "host_sr1cs_dump")
SRC = os.path.join(ROOT, "tests", "native", "host_sr1cs_dump.cpp")
CURVES = [BLS12_381, BN254]


def build():
    deps = [SRC] + [os.path.join(ROOT, "snark_b200", "host", f) for f in ("ark_relations.hpp", "ark_snark.hpp")]
    if not os.path.exists(EXE) or any(os.path.getmtime(d) > os.path.getmtime(EXE) for d in deps):
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-o", EXE, SRC, "-L", os.path.join(ROOT, "snark_b200"), "-lb200snark",
                               "-Wl,-rpath," + os.path.join(ROOT, "snark_b200")])
    return EXE


def words(curve, v):
    return " ".join(f"{int(w):08x}" for w in pack_fr(curve, [v]))


def run_mirror(curve, mats, n_inst, z, tmp_path):
    """mats: [A, B, C] as rows of (coeff, col); z: n_inst + n_wit ints (z[0] = 1).  -> (source csr, N, dest csr, z')"""
    n_rows = len(mats[0])
    lines = [f"{n_inst} {len(z) - n_inst} {n_rows}"] + [words(curve, v) for v in z[1:]]
    for i in range(n_rows):
        for k in range(3):
            lines.append(" ".join([str(len(mats[k][i]))] + [f"{col} {words(curve, c)}" for c, col in mats[k][i]]))
    f = tmp_path / f"r1cs_{curve.name}.txt"
    f.write_text("\n".join(lines) + "\n")
    out = subprocess.run([build(), "0" if curve is BLS12_381 else "1", str(f)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    srows = [[[] for _ in range(n_rows)] for _ in range(3)]
    N, zs, drows = None, [], {}
    for line in out.stdout.splitlines():
        tag, *rest = line.split()
        if tag == "N":
            N = (int(rest[0]), int(rest[1]))
        elif tag == "Z":
            zs.append(np.array([int(w, 16) for w in rest], dtype=np.uint32))
        else:
            k, i, terms = int(rest[0]), int(rest[1]), rest[2:]
            row = [(int(terms[j]), np.array([int(w, 16) for w in terms[j + 1:j + 9]], dtype=np.uint32)) for j in range(0, len(terms), 9)]
            if tag == "S":
                srows[k][i] = row
            else:
                drows.setdefault(k, {})[i] = row

    def csr(rowlist):
        rp = np.zeros(len(rowlist) + 1, dtype=np.uint64)
        rp[1:] = np.cumsum([len(r) for r in rowlist])
        col = np.array([c for r in rowlist for c, _ in r], dtype=np.uint32)
        co = np.concatenate([w for r in rowlist for _, w in r]) if rp[-1] else np.zeros(0, dtype=np.uint32)
        return rp, col, co
    src = [csr(srows[k]) for k in range(3)]
    n_dst = 2 * n_rows + N[0] - 1
    dst = [csr([drows.get(j, {}).get(i, []) for i in range(n_dst)]) for j in range(2)]
    return src, N, dst, np.concatenate(zs)


def random_r1cs(curve, seed):
    """rows of 0-6 terms over ONE, public and private columns, repeats within a row and across A/B/C, some empty rows,
    public columns that may never occur, coefficients 1, -1, 0-free random values"""
    r = curve.r
    rng = random.Random(seed)
    n_inst, n_wit = rng.randint(1, 6), rng.randint(1, 10)
    n_vars = n_inst + n_wit
    pool = [1, r - 1, 2, rng.randrange(1, r), rng.randrange(1, r)]
    used_pub = rng.sample(range(n_inst), rng.randint(0, n_inst))   # the public columns this system may use
    cols = [c for c in range(n_vars) if c >= n_inst or c in used_pub]
    mats = [[], [], []]
    shared = rng.choice(cols)
    for _ in range(rng.randint(1, 12)):
        empty = rng.random() < 0.15
        for k in range(3):
            row = [] if empty else [(rng.choice(pool), rng.choice(cols)) for _ in range(rng.randint(0, 6))]
            if row and rng.random() < 0.4:
                row.append((rng.choice(pool), row[0][1]))          # repeated in the row
            if not empty and rng.random() < 0.3:
                row.append((rng.choice(pool), shared))             # across A, B, C
            mats[k].append(row)
    z = [1] + [rng.randrange(r) for _ in range(n_vars - 1)]
    return mats, n_inst, z


def cases(curve):
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    yield "circuit2", cs.to_matrices(), len(cs.instance_assignment), list(cs.instance_assignment) + list(cs.witness_assignment)
    mats, inst, wit = orc.dummy_circuit_direct(curve, 3, 5, 12, 9)
    yield "dummy", mats, len(inst), inst + wit
    for seed in range(12):
        mats, n_inst, z = random_r1cs(curve, seed)
        yield f"random{seed}", mats, n_inst, z


@pytest.mark.parametrize("curve", CURVES, ids=lambda c: c.name)
def test_numpy_oracle_matches_cpp_mirror(curve, tmp_path):
    r = curve.r
    for name, mats, n_inst, z in cases(curve):
        src, N, dst, z_dst = run_mirror(curve, mats, n_inst, z, tmp_path)
        o = so.Sr1cs(r, src, n_inst)
        assert (o.n_instance, o.n_witness) == N, name
        got = o.matrices()
        for j in range(2):
            want = so.canonical_csr(r, *dst[j])
            assert len(got[j][0]) == len(want[0]), (name, j)
            for a, b in zip(got[j], want):
                assert np.array_equal(a, b), (name, j)
        zm = pack_fr(curve, z).reshape(1, -1)
        assert np.array_equal(o.assignment(zm)[0], z_dst), name
        # the converted system is satisfied exactly when the source is (first failing row 2i for row i)
        bad_src = [i for i in range(len(mats[0])) if
                   sum(c * z[col] for c, col in mats[0][i]) * sum(c * z[col] for c, col in mats[1][i]) % r
                   != sum(c * z[col] for c, col in mats[2][i]) % r]
        bad = so.check(r, got, so.limbs_to_ints(z_dst))
        assert (bad[:1] == [2 * bad_src[0]]) if bad_src else bad == [], name


def test_oracle_index_work_is_vectorised():
    """A DummyCircuit-shaped R1CS of 2^18 rows converts without field products beyond one per distinct value."""
    import time

    curve = BLS12_381
    m = 1 << 18
    one = pack_fr(curve, [1])
    rp = np.arange(m + 1, dtype=np.uint64)
    rp[-1] = m - 1
    csr = [(rp, np.full(m - 1, c, dtype=np.uint32), np.tile(one, m - 1)) for c in (2, 3, 1)]
    t = time.time()
    o = so.Sr1cs(curve.r, csr, 2)
    L, Rm = o.matrices()
    assert time.time() - t < 60
    assert (o.n_instance, o.n_witness, o.n_rows) == (2, 3 + m, 2 * m + 1)
    assert L[0][-1] == 4 * (m - 1) + 2 and Rm[0][-1] == (m - 1) + 2 * m
