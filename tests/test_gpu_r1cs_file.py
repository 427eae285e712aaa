"""circom .r1cs files loaded on the GPU (b2s_r1cs_file_load, b2s_r1cs_file_read_info): the loaded handle is the one
b2s_r1cs_upload builds from the same A, B, C (SpMV, witness maps, setup and proofs bit-identical), b2s_r1cs_check on it
is the circuit's own satisfaction, it proves under the key of the circuit's .zkey, and every malformed input gets its error
code.  The files come from the test-side writer (tests/r1cs_file_oracle.py), which restates circom's format; parity with
bytes written by circom itself is not pinned."""
import ctypes
import random
import struct

import numpy as np
import pytest

from oracle.params import BLS12_381, BN254
from tests import r1cs_file_oracle as ro
from tests import zkey_oracle as zo
from tests.bls377_oracle import BLS12_377
from tests.test_gpu_gr1cs import oracle_cs, r1cs_terms, unsat_rows
from tests.test_gpu_zkey import small_cases
from tests.util import csr_from_rows, pack_fr

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254, BLS12_377]
LIBSNARK, CIRCOM = 0, 1
INVALID_DATA, INVALID_ARG, DEGREE = 21, 16, 5
NOT_FOUND = (1 << 64) - 1
CHUNK = 1 << 18   # entries per staging chunk (Stager::CH)


@pytest.fixture(scope="module", params=[0, 1, 2], ids=["bls12_381", "bn254", "bls12_377"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def expect(code, text, fn, *args):
    from snark_b200 import B2SError

    with pytest.raises(B2SError) as e:
        fn(*args)
    assert e.value.code == code, str(e.value)
    assert text in str(e.value), str(e.value)


def domain_of(n):
    d = 1
    while d < n:
        d *= 2
    return d


# ---- circuits ------------------------------------------------------------------------------------------------------------
class Circuit:
    """rows-of-(coeff, wire) matrices over z = One, public outputs, public inputs, private inputs, internal wires"""

    def __init__(self, curve, mats, n_out, n_in, n_prv, n_wires):
        self.curve, self.mats = curve, mats
        self.n_out, self.n_in, self.n_prv, self.n_wires = n_out, n_in, n_prv, n_wires
        self.n_rows, self.n_inst = len(mats[0]), 1 + n_out + n_in
        self.csr = [csr_from_rows(curve, M) for M in mats]

    def file(self, **kw):
        return ro.write_r1cs(self.curve, self.csr, self.n_out, self.n_in, self.n_prv, n_wires=self.n_wires, **kw)

    def upload(self, be):
        return be.r1cs_upload(self.n_rows, self.n_inst, self.n_wires - self.n_inst, self.csr)


def random_circuit(curve, rng, n_out, n_in, n_prv, n_internal, n_rows, satisfied=False):
    """Random rows with empty combinations, duplicate wires and coefficients 1, r - 1, 0 and random.  satisfied: constraint i
    defines internal wire i through C (the rows only read earlier wires), and the satisfying z is returned with it."""
    r = curve.r
    n_wires = 1 + n_out + n_in + n_prv + n_internal
    coeff = lambda: rng.choice([1, r - 1, 0, rng.randrange(r), rng.randrange(r)])
    first_internal = 1 + n_out + n_in + n_prv
    z = [1] + [rng.randrange(r) for _ in range(n_wires - 1)]
    mats = [[], [], []]
    for i in range(n_rows):
        known = first_internal + i if satisfied else n_wires
        for k in range(2 if satisfied else 3):
            row = [(coeff(), rng.randrange(known)) for _ in range(rng.choice([0, 1, 1, 2, 3, 5]))]
            if row and rng.random() < 0.3:
                row.append((coeff(), row[0][1]))   # the same wire twice
            mats[k].append(row)
        if satisfied:
            out = first_internal + i
            c0 = rng.choice([1, r - 1, rng.randrange(1, r)])
            row = [(c0, out)] + [(coeff(), rng.randrange(known)) for _ in range(rng.choice([0, 0, 1, 2]))]
            rng.shuffle(row)
            a = sum(c * z[w] for c, w in mats[0][i]) % r
            b = sum(c * z[w] for c, w in mats[1][i]) % r
            rest = sum(c * z[w] for c, w in row if w != out)
            z[out] = (a * b - rest) * pow(c0, -1, r) % r
            mats[2].append(row)
    return Circuit(curve, mats, n_out, n_in, n_prv, n_wires), z


def random_circuits(curve, seed):
    rng = random.Random(seed)
    shapes = [(0, 0, 0, 5, 12), (2, 3, 1, 10, 30), (1, 0, 2, 4, 1), (0, 2, 0, 0, 7), (3, 2, 4, 40, 100), (0, 0, 0, 1, 0)]
    for n_out, n_in, n_prv, n_int, n_rows in shapes:
        yield random_circuit(curve, rng, n_out, n_in, n_prv, n_int, n_rows)[0]


def numpy_csr(be, curve, rng, n_rows, n_wires, max_count, big_row=None):
    """A large random CSR triple per matrix, coefficients from a small table (ONE, -ONE, zero and random values)"""
    table = pack_fr(curve, [1, curve.r - 1, 0] + [int(rng.integers(1, 1 << 62)) * 0x9E3779B97F4A7C15 % curve.r for _ in range(5)]).reshape(-1, 8)
    csr = []
    for k in range(3):
        counts = rng.integers(0, max_count + 1, size=n_rows)
        if big_row is not None and k == 0:
            counts[big_row] = CHUNK + 12345
        row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
        row_ptr[1:] = np.cumsum(counts)
        nnz = int(row_ptr[-1])
        col = rng.integers(0, n_wires, size=nnz).astype(np.uint32)
        pick = rng.choice(len(table), size=nnz, p=[0.6, 0.1, 0.05] + [0.05] * 5)
        csr.append((row_ptr, col, np.ascontiguousarray(table[pick]).reshape(-1)))
    return csr


def random_z(curve, rng, n):
    return pack_fr(curve, [1] + [rng.randrange(curve.r) for _ in range(n - 1)])


def assert_same_handle(be, curve, m_file, m_up, n_rows, n_wires, rng, n_z=3):
    assert be.domain_size(m_file) == be.domain_size(m_up)
    for _ in range(n_z):
        z = random_z(curve, rng, n_wires)
        for x, y in zip(be.spmv(m_file, z, n_rows), be.spmv(m_up, z, n_rows)):
            assert np.array_equal(x, y)
        for qap in (LIBSNARK, CIRCOM) if n_rows else ():
            assert np.array_equal(be.witness_map(m_file, z, qap=qap), be.witness_map(m_up, z, qap=qap)), qap


# ---- 1, 2: the handle and the header -------------------------------------------------------------------------------------
def test_loaded_handle_equals_upload(be):
    """SpMV a, b, c, the domain size and both witness maps of the loaded handle equal a b2s_r1cs_upload handle of the same
    CSR, for random circuits (0 public signals, outputs and inputs, empty and duplicate-wire rows, coefficients 1, r - 1, 0),
    sections in circom's order and shuffled, with and without the wire map"""
    curve = CURVES[be.curve]
    rng = random.Random(0x71 + be.curve)
    for i, circ in enumerate(random_circuits(curve, 0x100 + be.curve)):
        m_up = circ.upload(be)
        for order, wire_map in (("circom", True), ("shuffled", True), ("circom", False)):
            m = be.r1cs_file_load(circ.file(order=order, wire_map=wire_map))
            assert_same_handle(be, curve, m, m_up, circ.n_rows, circ.n_wires, rng)
            be.r1cs_free(m)
        be.r1cs_free(m_up)


def test_witness_map_sim_on_loaded_handle(be):
    """b2s_witness_map_sim (the distributed schedule) of a loaded handle with an even log-domain equals b2s_witness_map"""
    curve = CURVES[be.curve]
    rng = random.Random(0x5E + be.curve)
    circ, _ = random_circuit(curve, rng, 2, 1, 3, 400, 1000)
    m = be.r1cs_file_load(circ.file())
    assert be.domain_size(m) == 1024
    z = random_z(curve, rng, circ.n_wires)
    for log_ranks in (1, 2):
        assert np.array_equal(be.witness_map_sim(m, z, log_ranks), be.witness_map(m, z)), log_ranks
    be.r1cs_free(m)


def test_read_info(be):
    curve = CURVES[be.curve]
    circ, _ = random_circuit(curve, random.Random(3), 2, 3, 4, 20, 57)
    info = be.r1cs_file_info(circ.file(n_labels=1234))
    assert info == {"n_wires": circ.n_wires, "n_pub_out": 2, "n_pub_in": 3, "n_prv_in": 4, "n_labels": 1234, "n_constraints": 57,
                    "domain_size": domain_of(57 + 6)}


# ---- 3: staging chunks ---------------------------------------------------------------------------------------------------
def test_spans_across_chunks(be, tmp_path):
    """a constraint section of several staging chunks (memory-mapped from a file), and one constraint of more than a chunk
    of entries, both load equal to the upload"""
    curve = CURVES[be.curve]
    rng = np.random.default_rng(0xC4 + be.curve)
    prng = random.Random(0xC5 + be.curve)
    for n_rows, n_wires, max_count, big_row in ((1 << 17, 5000, 6, None), (5, 300, 3, 2)):
        csr = numpy_csr(be, curve, rng, n_rows, n_wires, max_count, big_row)
        total = sum(int(m[0][-1]) for m in csr)
        assert total > 3 * CHUNK or big_row is not None
        path = ro.write_r1cs(curve, csr, 1, 2, 0, n_wires=n_wires, path=tmp_path / "big.r1cs")
        m = be.r1cs_file_load(np.memmap(path, dtype=np.uint8, mode="r"))
        m_up = be.r1cs_upload(n_rows, 4, n_wires - 4, csr)
        assert_same_handle(be, curve, m, m_up, n_rows, n_wires, prng, n_z=2)
        be.r1cs_free(m)
        be.r1cs_free(m_up)


# ---- 4: satisfaction -----------------------------------------------------------------------------------------------------
def test_check_is_the_circuits_satisfaction(be):
    """b2s_r1cs_check on the loaded handle, for a batch of assignments with 1-3 tampered values each (and the satisfying one),
    matches the big-int oracle's which_is_unsatisfied and its count of failing rows, for host and device buffers"""
    import torch

    curve = CURVES[be.curve]
    rng = random.Random(0xC3 + be.curve)
    for shape in ((0, 0, 0, 60), (2, 3, 2, 80), (1, 1, 0, 200)):
        circ, z = random_circuit(curve, rng, *shape[:3], shape[3], shape[3], satisfied=True)
        m = be.r1cs_file_load(circ.file())
        zs = [z]
        for _ in range(12):
            t = list(z)
            for w in rng.sample(range(1, circ.n_wires), rng.randint(1, 3)):
                t[w] = (t[w] + rng.randrange(1, curve.r)) % curve.r
            zs.append(t)
        want_first, want_count = [], []
        for t in zs:
            bad = oracle_cs(curve, {"r1cs": (3, r1cs_terms(curve.r), circ.mats)}, circ.n_inst, t).which_is_unsatisfied()
            rows = unsat_rows(curve.r, 3, r1cs_terms(curve.r), circ.mats, t)
            assert (bad is None) == (not rows) and (bad is None or bad[1] == rows[0])
            want_first.append(NOT_FOUND if bad is None else bad[1])
            want_count.append(len(rows))
        assert want_first[0] == NOT_FOUND and any(f != NOT_FOUND for f in want_first)
        packed = pack_fr(curve, [v for t in zs for v in t]).reshape(len(zs), -1)
        for zz in (packed, torch.from_numpy(packed.view(np.int32)).cuda()):
            first, count = be.r1cs_check(m, zz)
            assert first[:, 0].tolist() == want_first and count[:, 0].tolist() == want_count
        be.r1cs_free(m)


# ---- 5, 6: circom end to end, setup from the file ------------------------------------------------------------------------
def test_circom_route_r1cs_zkey_wtns(be):
    """One circuit as .r1cs, .zkey and .wtns: load -> b2s_r1cs_check -> prove -> verify.  Proofs under the zkey's key are
    bit-identical with the r1cs handle and the zkey handle (prove_resident and prove_batch), and the verifier accepts them"""
    import torch

    curve = CURVES[be.curve]
    rng = random.Random(0xE2E + be.curve)
    for case in small_cases(be, curve, rng, ("dummy16", "bench25")):
        n_pub = case.n_inst - 1
        circ_file = ro.write_r1cs(curve, case.csr, n_pub // 2, n_pub - n_pub // 2, 1, n_wires=case.n_vars)
        m_r1cs = be.r1cs_file_load(circ_file)
        pk, m_zkey, vk = be.zkey_load(case.zkey(curve))
        wtns = zo.write_wtns(curve, case.z)
        z = be.wtns_read(wtns, case.n_vars)
        first, _ = be.r1cs_check(m_r1cs, z.reshape(1, -1), counts=False)
        assert first[0, 0] == NOT_FOUND, case.name
        K = 3
        zt = torch.zeros((K, case.n_vars * 8), dtype=torch.int32, device="cuda")
        for i in range(K):
            be.wtns_read(wtns, case.n_vars, out=zt[i])
        be.sync()
        r = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
        s = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
        proofs = []
        for i in range(K):
            ri, si = r[8 * i: 8 * i + 8], s[8 * i: 8 * i + 8]
            got = be.groth16_prove_resident(pk, m_r1cs, zt[i], ri, si)
            ref = be.groth16_prove_resident(pk, m_zkey, zt[i], ri, si)
            assert all(np.array_equal(x, y) for x, y in zip(got, ref)), (case.name, i)
            proofs.append(got)
        rt, st = (torch.from_numpy(x.view(np.int32)).cuda() for x in (r, s))
        batch_r1cs = be.groth16_prove_batch(pk, m_r1cs, zt, rt, st)
        batch_zkey = be.groth16_prove_batch(pk, m_zkey, zt, rt, st)
        for j in range(3):
            assert torch.equal(batch_r1cs[j], batch_zkey[j]), (case.name, j)
            for i in range(K):
                assert np.array_equal(batch_r1cs[j][i].cpu().numpy().view(np.uint32), proofs[i][j]), (case.name, i, j)
        pvk = be.vk_prepare(vk)
        inputs = np.concatenate([z[8: 8 * case.n_inst]] * K) if n_pub else None
        a, b, c = (np.concatenate([p[j] for p in proofs]) for j in range(3))
        assert be.groth16_verify_batch(pvk, inputs, n_pub, a, b, c).tolist() == [True] * K, case.name
        be.pvk_free(pvk)
        be.pk_free(pk)
        be.r1cs_free(m_zkey)
        be.r1cs_free(m_r1cs)
        case.free(be)


def test_setup_from_the_file(be):
    """b2s_groth16_setup_qap on the loaded handle gives, under both reductions and a fixed trapdoor, the b2s_pk_query bytes
    and verifying key of setup on the uploaded handle; a libsnark proof from it verifies"""
    curve = CURVES[be.curve]
    rng = random.Random(0x5E7 + be.curve)
    circ, z = random_circuit(curve, rng, 1, 2, 2, 70, 70, satisfied=True)
    m = be.r1cs_file_load(circ.file())
    m_up = circ.upload(be)
    td = pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)])
    n_vars, n_wit, domain = circ.n_wires, circ.n_wires - circ.n_inst, be.domain_size(m)
    counts = {LIBSNARK: {0: n_vars, 1: n_vars, 2: n_vars, 3: domain - 1, 4: n_wit, 5: 3, 6: 2},
              CIRCOM: {0: n_vars, 1: n_vars, 2: n_vars, 3: domain, 4: n_wit, 5: 3, 6: 2}}
    for qap in (LIBSNARK, CIRCOM):
        pk, vk = be.groth16_setup(m, td, circ.n_inst, qap=qap)
        pk_up, vk_up = be.groth16_setup(m_up, td, circ.n_inst, qap=qap)
        for w, n in counts[qap].items():
            assert np.array_equal(be.pk_query(pk, w, n), be.pk_query(pk_up, w, n)), (qap, w)
        for k in vk:
            assert np.array_equal(vk[k], vk_up[k]), (qap, k)
        if qap == LIBSNARK:
            zp = pack_fr(curve, z)
            proof = be.groth16_prove(pk, m, zp[: 8 * circ.n_inst], zp[8 * circ.n_inst:], pack_fr(curve, [rng.randrange(curve.r)]),
                                     pack_fr(curve, [rng.randrange(curve.r)]))
            pvk = be.vk_prepare(vk)
            assert be.groth16_verify_batch(pvk, zp[8: 8 * circ.n_inst], circ.n_inst - 1, *proof).tolist() == [True]
            be.pvk_free(pvk)
        be.pk_free(pk)
        be.pk_free(pk_up)
    be.r1cs_free(m)
    be.r1cs_free(m_up)


# ---- 7: malformed input --------------------------------------------------------------------------------------------------
def entry_word(circ, i, k, j):
    """the word index, in section 2, of the wire of entry j of matrix k in constraint i (its coefficient follows)"""
    rps = [c[0].astype(np.int64) for c in circ.csr]
    at = 3 * i + ro.ENTRY_WORDS * sum(int(rp[i]) for rp in rps)
    for q in range(k):
        at += 1 + ro.ENTRY_WORDS * int(rps[q][i + 1] - rps[q][i])
    return at + 1 + ro.ENTRY_WORDS * j


def test_malformed_inputs(be):
    """One case per check, each with its error code and the section, or constraint, matrix and entry, b2s_last_error names;
    of several bad entries the lowest in file order is reported"""
    curve = CURVES[be.curve]
    other = CURVES[(be.curve + 1) % 3]
    rng = random.Random(0xBAD + be.curve)
    while True:
        circ, _ = random_circuit(curve, rng, 2, 1, 1, 20, 30)
        rows = [len(circ.mats[2][17]), len(circ.mats[0][5]), len(circ.mats[1][5]), len(circ.mats[0][20])]
        if rows[0] >= 3 and min(rows[1:]) >= 2:
            break
    secs = ro.r1cs_sections(curve, circ.csr, 2, 1, 1, n_wires=circ.n_wires)
    S = dict(secs)
    W = np.frombuffer(S[2], dtype=np.uint32)
    load, info = be.r1cs_file_load, be.r1cs_file_info

    def file_of(**repl):
        out = [(t, repl.get(f"s{t}", body)) for t, body in secs]
        return zo.binfile(b"r1cs", 1, [(t, b) for t, b in out if b is not None])

    def body_with(edits):
        w = W.copy()
        for at, v in edits:
            w[at] = v
        return w.tobytes()

    good = file_of()
    be.r1cs_free(load(good))
    n = circ.n_wires
    r_limbs = lambda: [(curve.r >> (32 * q)) & 0xFFFFFFFF for q in range(8)]
    # entries: a wire out of range, a coefficient >= r, and the lowest of several
    at = entry_word(circ, 17, 2, 2)
    expect(INVALID_DATA, f"r1cs constraint 17 C[2]: wire {n + 5} not below nWires {n}", load, file_of(s2=body_with([(at, n + 5)])))
    at = entry_word(circ, 5, 1, 1)
    expect(INVALID_DATA, "r1cs constraint 5 B[1]: coefficient not below r", load,
           file_of(s2=body_with([(at + 1 + q, v) for q, v in enumerate(r_limbs())])))
    bad = [(entry_word(circ, 20, 0, 0), n), (entry_word(circ, 5, 1, 1), 0xFFFFFFFF), (entry_word(circ, 5, 0, 1), n + 1),
           (entry_word(circ, 17, 2, 0) + 8, 0xFFFFFFFF)]
    expect(INVALID_DATA, f"r1cs constraint 5 A[1]: wire {n + 1}", load, file_of(s2=body_with(bad)))
    expect(INVALID_DATA, "r1cs constraint 5 B[1]: wire 4294967295", load, file_of(s2=body_with(bad[:2] + bad[3:])))
    # the count words: one that overruns the section, a truncated section, a section longer than mConstraints constraints
    expect(INVALID_DATA, "r1cs constraint 3 B: 1000000 entries overrun section 2", load,
           file_of(s2=body_with([(entry_word(circ, 3, 1, 0) - 1, 1000000)])))
    expect(INVALID_DATA, "overrun section 2", load, file_of(s2=S[2][:-4]))
    expect(INVALID_DATA, "r1cs: section 2 holds 12 bytes after its 30 constraints", load, file_of(s2=S[2] + bytes(12)))
    # header: dimensions, size, the other curve's prime, custom gates, the wire map, a domain past the limits
    hdr = lambda **kw: ro.header_section(curve, kw.get("n_wires", n), 2, 1, kw.get("n_prv", 1), n, kw.get("m", 30), kw.get("prime"))
    assert hdr() == S[1]
    expect(INVALID_DATA, "nWires", load, file_of(s1=hdr(n_prv=n - 3)))
    expect(INVALID_DATA, "r1cs: header section holds", load, file_of(s1=S[1] + b"\0\0\0\0"))
    for fn in (load, info):
        expect(INVALID_ARG, "r1cs: the prime", fn, file_of(s1=hdr(prime=other.r)))
        expect(DEGREE, "domain 2^28", fn, file_of(s1=hdr(m=(1 << 28) - 4)))
    expect(INVALID_DATA, "section 3 (wire map)", load, file_of(s3=S[3][:-8]))
    for t in (4, 5):
        expect(INVALID_DATA, f"section {t} (PLONK custom gates)", load, zo.binfile(b"r1cs", 1, secs + [(t, b"\0" * 8)]))
    # framing
    expect(INVALID_DATA, "bad magic", load, b"zkey" + good[4:])
    expect(INVALID_DATA, "version", load, good[:4] + struct.pack("<I", 2) + good[8:])
    expect(INVALID_DATA, "truncated in the header of section 0", load, good[:20])
    expect(INVALID_DATA, "remain", load, good[:-5])
    expect(INVALID_DATA, "trailing bytes", load, good + b"\0")
    expect(INVALID_DATA, "section 2 missing", load, file_of(s2=None))
    expect(INVALID_DATA, "section 1 missing", info, file_of(s1=None))
    for t in (1, 2, 3):
        expect(INVALID_DATA, f"section {t} appears twice", load, zo.binfile(b"r1cs", 1, secs + [(t, S[t])]))
    # null pointers
    h, inf = ctypes.c_void_p(), ro_info()
    buf = np.frombuffer(good, dtype=np.uint8)
    assert be.lib.b2s_r1cs_file_load(be.h, None, len(good), ctypes.byref(h)) == INVALID_ARG
    assert be.lib.b2s_r1cs_file_load(be.h, buf.ctypes.data, len(good), None) == INVALID_ARG
    assert be.lib.b2s_r1cs_file_read_info(be.h, None, len(good), ctypes.byref(inf)) == INVALID_ARG
    assert be.lib.b2s_r1cs_file_read_info(be.h, buf.ctypes.data, len(good), None) == INVALID_ARG
    # still usable after every failure
    m = load(good)
    m_up = circ.upload(be)
    assert_same_handle(be, curve, m, m_up, circ.n_rows, circ.n_wires, rng, n_z=1)
    be.r1cs_free(m)
    be.r1cs_free(m_up)


def ro_info():
    from snark_b200.lib import R1csFileInfo

    return R1csFileInfo()
