"""snarkjs .zkey and circom .wtns files loaded on the GPU (b2s_zkey_load, b2s_wtns_read): the loaded key and matrices equal
their source, proofs from zkey + wtns are bit-identical to proofs from the uploaded key and are accepted by the verifiers,
and every malformed input gets its error code.  The files come from the test-side writers (tests/zkey_oracle.py), which
restate snarkjs's format; parity with bytes written by snarkjs itself is not pinned."""
import random
import struct

import numpy as np
import pytest

from oracle import groth16 as og
from oracle.params import BLS12_381, BN254
from tests import circom_oracle as oc
from tests import zkey_oracle as zo
from tests.test_gpu_circom import circuits, dummy_2k, spoil
from tests.util import csr_from_rows, pack_fr, pack_points, unpack_fr
from tests.wire_oracle import random_curve_point

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
CIRCOM = 1
INVALID_DATA, INVALID_ARG, MALFORMED_VK, DEGREE, ASSIGNMENT = 21, 16, 7, 5, 2


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def domain_of(n_rows, n_inst):
    d = 1
    while d < n_rows + n_inst:
        d *= 2
    return d


def rows_of_csr(csr):
    row_ptr, col, _ = csr   # dummy_2k: every coefficient is 1
    return [[(1, int(col[e])) for e in range(int(row_ptr[i]), int(row_ptr[i + 1]))] for i in range(len(row_ptr) - 1)]


class Case:
    """one circuit with a circom key from b2s_groth16_setup_qap: the source handles, the key arrays and a satisfying z"""

    def __init__(self, be, curve, name, csr, n_rows, n_inst, n_wit, z, rng):
        self.name, self.csr, self.n_rows, self.n_inst, self.n_wit, self.z = name, csr, n_rows, n_inst, n_wit, z
        self.n_vars, self.domain = n_inst + n_wit, domain_of(n_rows, n_inst)
        self.m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
        self.pkh, self.vk = be.groth16_setup(self.m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), n_inst, qap=CIRCOM)
        self.key = zo.key_arrays_device(be, self.pkh, self.vk, n_inst, n_wit, self.domain)

    def zkey(self, curve, order="snarkjs", seed=0):
        return zo.write_zkey(curve, self.key, self.csr[0], self.csr[1], self.n_inst - 1, self.domain, order=order, seed=seed)

    def free(self, be):
        be.pk_free(self.pkh)
        be.r1cs_free(self.m)


def small_cases(be, curve, rng, names=None):
    for name, mats, inst, wit in circuits(curve):
        if names is not None and name not in names:
            continue
        csr = [csr_from_rows(curve, M) for M in mats]
        yield Case(be, curve, name, csr, len(mats[0]), len(inst), len(wit), pack_fr(curve, list(inst) + list(wit)), rng)


def dummy_case(be, curve, log_n, rng):
    csr, n_rows, n_inst, n_wit, z_inst, z_wit = dummy_2k(curve, log_n)
    return Case(be, curve, f"dummy_2^{log_n}", csr, n_rows, n_inst, n_wit, np.concatenate([z_inst, z_wit]), rng)


def assert_key_equal(be, pk, vk, key, n_vars, n_wit, domain, label):
    want = {0: key["a"], 1: key["b_g1"], 2: key["b_g2"], 3: key["h"], 4: key["l"],
            5: np.concatenate([key["alpha_g1"], key["beta_g1"], key["delta_g1"]]), 6: np.concatenate([key["beta_g2"], key["delta_g2"]])}
    counts = {0: n_vars, 1: n_vars, 2: n_vars, 3: domain, 4: n_wit, 5: 3, 6: 2}
    for w in range(7):
        assert np.array_equal(be.pk_query(pk, w, counts[w]), want[w]), (label, w)
    for k in ("alpha_g1", "beta_g2", "gamma_g2", "delta_g2", "gamma_abc_g1"):
        assert np.array_equal(vk[k], key[k]), (label, k)


def test_loaded_key_equals_source(be):
    """Every b2s_pk_query vector and the vk points of the loaded key equal the source, for keys from the oracle's circom
    setup and from b2s_groth16_setup_qap, validate 0 and 1, sections and records in snarkjs order and shuffled."""
    curve = CURVES[be.curve]
    rng = random.Random(0x2E1 + be.curve)
    for i, (name, mats, inst, wit) in enumerate(circuits(curve)):
        n_inst, n_wit = len(inst), len(wit)
        csr = [csr_from_rows(curve, M) for M in mats]
        domain = domain_of(len(mats[0]), n_inst)
        sources = []
        if i < 3:
            td = og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)])
            sources.append(("oracle", zo.key_arrays(curve, oc.setup_circom(curve, mats, n_inst, n_wit, td))))
        case = Case(be, curve, name, csr, len(mats[0]), n_inst, n_wit, None, rng)
        sources.append(("setup_qap", case.key))
        for src, key in sources:
            for order in ("snarkjs", "shuffled"):
                data = zo.write_zkey(curve, key, csr[0], csr[1], n_inst - 1, domain, order=order, seed=i)
                info = be.zkey_info(data)
                assert (info["n_vars"], info["n_public"], info["domain_size"]) == (n_inst + n_wit, n_inst - 1, domain)
                for validate in (False, True):
                    pk, m, vk = be.zkey_load(data, validate=validate)
                    assert be.domain_size(m) == domain
                    assert_key_equal(be, pk, vk, key, n_inst + n_wit, n_wit, domain, (name, src, order, validate))
                    be.pk_free(pk)
                    be.r1cs_free(m)
        case.free(be)


def test_matrices_match_upload(be):
    """b2s_witness_map_qap(CIRCOM) of the loaded matrix handle equals that of a b2s_r1cs_upload handle of the same A, B
    (satisfying and spoiled z, snarkjs order and shuffled records), and at 2^12 the oracle's circom witness map."""
    curve = CURVES[be.curve]
    rng = random.Random(0x3A7 + be.curve)
    cases = list(small_cases(be, curve, rng)) + [dummy_case(be, curve, 12, rng), dummy_case(be, curve, 16, rng)]
    for case in cases:
        m_up = upload_empty_c(be, case)
        z_bad = case.z.copy()
        z_bad[8 * case.n_inst:] = pack_fr(curve, spoil(curve, unpack_fr(curve, case.z[8 * case.n_inst:])))
        for order in ("snarkjs", "shuffled"):
            pk, m, _vk = be.zkey_load(case.zkey(curve, order, seed=5), validate=False)
            for z in (case.z, z_bad):
                got = be.witness_map(m, z, qap=CIRCOM)
                assert np.array_equal(got, be.witness_map(m_up, z, qap=CIRCOM)), (case.name, order)
                if case.name == "dummy_2^12" and order == "snarkjs":
                    mats = [rows_of_csr(case.csr[k]) for k in range(3)]
                    assert unpack_fr(curve, got) == oc.witness_map_circom(curve, mats, unpack_fr(curve, z), case.n_inst)
            first, _ = be.r1cs_check(m, case.z.reshape(1, -1), counts=False)
            first_up, _ = be.r1cs_check(m_up, case.z.reshape(1, -1), counts=False)
            assert np.array_equal(first, first_up), case.name
            be.pk_free(pk)
            be.r1cs_free(m)
        be.r1cs_free(m_up)
        case.free(be)


def upload_empty_c(be, case):
    csr = list(case.csr[:2]) + [(np.zeros(case.n_rows + 1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32))]
    return be.r1cs_upload(case.n_rows, case.n_inst, case.n_wit, csr)


def test_prove_from_zkey_and_wtns(be, tmp_path):
    """zkey (memory-mapped from a file) + wtns through b2s_groth16_prove_resident and _prove_batch (rows from b2s_wtns_read
    into device memory): every proof is bit-identical to b2s_groth16_prove on the uploaded key and matrices with the same
    r, s and is accepted by both verifiers under the zkey's vk; a wtns with a spoiled witness gives a rejected proof."""
    import torch

    curve = CURVES[be.curve]
    rng = random.Random(0x9E0 + be.curve)
    cases = list(small_cases(be, curve, rng, ("dummy16", "bench25"))) + [dummy_case(be, curve, 12, rng)]
    for case in cases:
        path = tmp_path / f"{case.name}.zkey"
        path.write_bytes(case.zkey(curve, "shuffled", seed=1))
        pk, m, vk = be.zkey_load(np.memmap(path, dtype=np.uint8, mode="r"))
        z_bad = case.z.copy()
        z_bad[8 * case.n_inst:] = pack_fr(curve, spoil(curve, unpack_fr(curve, case.z[8 * case.n_inst:])))
        files = [zo.write_wtns(curve, case.z), zo.write_wtns(curve, z_bad), zo.write_wtns(curve, case.z)]
        assert np.array_equal(be.wtns_read(files[0], case.n_vars), case.z)
        K = len(files)
        zt = torch.zeros((K, case.n_vars * 8), dtype=torch.int32, device="cuda")
        for i, f in enumerate(files):
            be.wtns_read(f, case.n_vars, out=zt[i])
        be.sync()
        z_host = zt.cpu().numpy().view(np.uint32)
        r = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
        s = pack_fr(curve, [rng.randrange(curve.r) for _ in range(K)])
        refs = []
        for i in range(K):
            row = z_host[i]
            ri, si = r[8 * i: 8 * i + 8], s[8 * i: 8 * i + 8]
            ref = be.groth16_prove(case.pkh, case.m, np.ascontiguousarray(row[: 8 * case.n_inst]), np.ascontiguousarray(row[8 * case.n_inst:]), ri, si)
            got = be.groth16_prove_resident(pk, m, zt[i], ri, si)
            assert all(np.array_equal(x, y) for x, y in zip(got, ref)), (case.name, i)
            refs.append(ref)
        batch = be.groth16_prove_batch(pk, m, zt, torch.from_numpy(r.view(np.int32)).cuda(), torch.from_numpy(s.view(np.int32)).cuda())
        for i in range(K):
            for j in range(3):
                assert np.array_equal(batch[j][i].cpu().numpy().view(np.uint32), refs[i][j]), (case.name, i, j)
        pvk = be.vk_prepare(vk)
        a, b, c = (np.concatenate([p[j] for p in refs]) for j in range(3))
        inputs = lambda idx: np.concatenate([z_host[i][8: 8 * case.n_inst] for i in idx]) if case.n_inst > 1 else None
        x = inputs(range(K))
        assert be.groth16_verify_batch(pvk, x, case.n_inst - 1, a, b, c).tolist() == [True, False, True], case.name
        good = [0, 2]
        assert be.groth16_verify_all(pvk, inputs(good), case.n_inst - 1, *(np.concatenate([refs[i][j] for i in good]) for j in range(3)))
        assert not be.groth16_verify_all(pvk, x, case.n_inst - 1, a, b, c)
        be.pvk_free(pvk)
        be.pk_free(pk)
        be.r1cs_free(m)
        case.free(be)


# ---- malformed input -------------------------------------------------------------------------------------------------
def expect(be, code, text, fn, *args, **kw):
    from snark_b200 import B2SError

    with pytest.raises(B2SError) as e:
        fn(*args, **kw)
    assert e.value.code == code, str(e.value)
    assert text in str(e.value), str(e.value)


def rebuild(secs, **repl):
    """the zkey of sections `secs` (snarkjs order) with sections replaced (s<type>=bytes) or dropped (s<type>=None)"""
    out = []
    for t, body in secs:
        body = repl.get(f"s{t}", body)
        if body is not None:
            out.append((t, body))
    return zo.binfile(b"zkey", 1, out)


def test_malformed_inputs(be):
    """One case per check, each with its error code and the section / index b2s_last_error names."""
    curve = CURVES[be.curve]
    other = CURVES[1 - be.curve]
    rng = random.Random(0xBAD + be.curve)
    (case,) = small_cases(be, curve, rng, ("dummy16",))
    n_public, D = case.n_inst - 1, case.domain
    rec = zo.coeff_records(curve, case.csr[0], case.csr[1], n_public)
    secs = zo.zkey_sections(curve, case.key, rec, n_public, D)
    S = dict(secs)
    n8q = 8 * curve.fq_limbs64
    g1, g2 = 2 * n8q, 4 * n8q
    good = rebuild(secs)
    pk, m, _ = be.zkey_load(good)
    be.pk_free(pk)
    be.r1cs_free(m)

    def with_point(sec, i, pt_bytes):
        b = bytearray(S[sec])
        b[i * len(pt_bytes): (i + 1) * len(pt_bytes)] = pt_bytes
        return bytes(b)

    def coeffs(r):
        return struct.pack("<I", len(r)) + np.ascontiguousarray(r, dtype=np.uint32).tobytes()

    # points: a coordinate >= q (both modes), an off-curve G1 point (validate = 1 only), a twist point outside the subgroup
    a1 = bytearray(S[5][g1: 2 * g1])
    a1[:n8q] = curve.p.to_bytes(n8q, "little")
    for v in (False, True):
        expect(be, INVALID_DATA, "zkey A[1]: coordinate not below p", be.zkey_load, rebuild(secs, s5=with_point(5, 1, bytes(a1))), validate=v)
    a2 = bytearray(S[5][2 * g1: 3 * g1])
    a2[n8q] ^= 1
    off = rebuild(secs, s5=with_point(5, 2, bytes(a2)))
    pk, m, _ = be.zkey_load(off, validate=False)
    be.pk_free(pk)
    be.r1cs_free(m)
    expect(be, INVALID_DATA, "zkey A[2]: not on the curve", be.zkey_load, off, validate=True)
    tw = pack_points(curve, 2, [random_curve_point(curve, 2, random.Random(5))]).tobytes()
    expect(be, INVALID_DATA, "zkey B2[3]: not in the prime-order subgroup", be.zkey_load, rebuild(secs, s7=with_point(7, 3, tw)))
    # coefficient fields
    bad = rec.copy()
    bad[4, 3:] = [(curve.r >> (32 * j)) & 0xFFFFFFFF for j in range(8)]
    expect(be, INVALID_DATA, "zkey coefficients[4]: value not below r", be.zkey_load, rebuild(secs, s4=coeffs(bad)))
    bad = rec.copy()
    bad[6, 0] = 2
    expect(be, INVALID_DATA, "zkey coefficients[6]: matrix", be.zkey_load, rebuild(secs, s4=coeffs(bad)))
    bad = rec.copy()
    bad[7, 2] = case.n_vars
    expect(be, INVALID_DATA, "zkey coefficients[7]: signal", be.zkey_load, rebuild(secs, s4=coeffs(bad)))
    bad = rec.copy()
    bad[8, 1] = D
    expect(be, INVALID_DATA, "zkey coefficients[8]: constraint", be.zkey_load, rebuild(secs, s4=coeffs(bad)))
    # input rows: the row of z[0] missing; a B entry in an input row; an altered input entry
    n_in = len(rec) - (n_public + 1)
    expect(be, MALFORMED_VK, "input row 0", be.zkey_load, rebuild(secs, s4=coeffs(np.delete(rec, n_in, axis=0))))
    extra = rec[n_in + 1: n_in + 2].copy()
    extra[0, 0] = 1
    expect(be, MALFORMED_VK, f"zkey coefficients[{len(rec)}]: a B entry in an input row", be.zkey_load,
           rebuild(secs, s4=coeffs(np.concatenate([rec, extra]))))
    bad = rec.copy()
    bad[n_in + 1, 2] = 0
    expect(be, MALFORMED_VK, f"zkey coefficients[{n_in + 1}]: an input row entry", be.zkey_load, rebuild(secs, s4=coeffs(bad)))
    # header: domainSize != next_pow2 (sections consistent with it), a domain past the limits, PLONK, the other curve
    hdr_at = lambda d: S[2][:4 + n8q + 4 + 32] + struct.pack("<III", case.n_vars, n_public, d) + S[2][4 + n8q + 4 + 32 + 12:]
    assert hdr_at(D) == S[2]
    expect(be, MALFORMED_VK, "domainSize", be.zkey_load, rebuild(secs, s2=hdr_at(2 * D), s9=S[9] + S[9]))
    expect(be, DEGREE, "domain 2^28", be.zkey_load, rebuild(secs, s2=hdr_at(1 << 28)))
    expect(be, INVALID_DATA, "protocol 2", be.zkey_load, rebuild(secs, s1=struct.pack("<I", 2)))
    on8 = 8 * other.fq_limbs64
    foreign = struct.pack("<I", on8) + other.p.to_bytes(on8, "little") + struct.pack("<I", 32) + other.r.to_bytes(32, "little") + S[2][4 + n8q + 36:]
    expect(be, INVALID_ARG, "not the fields", be.zkey_load, rebuild(secs, s2=foreign))
    expect(be, INVALID_ARG, "not the fields", be.zkey_info, rebuild(secs, s2=foreign))
    # section sizes against the dimensions, and the framing
    expect(be, MALFORMED_VK, "section 5 (A)", be.zkey_load, rebuild(secs, s5=S[5][:-g1]))
    expect(be, MALFORMED_VK, "section 7 (B2)", be.zkey_load, rebuild(secs, s7=S[7] + S[7][:g2]))
    expect(be, INVALID_DATA, "truncated in the header of section 0", be.zkey_load, good[:20])
    expect(be, INVALID_DATA, "remain", be.zkey_load, good[:-5])
    expect(be, INVALID_DATA, "bad magic", be.zkey_load, b"wtns" + good[4:])
    expect(be, INVALID_DATA, "version", be.zkey_load, good[:4] + struct.pack("<I", 2) + good[8:])
    expect(be, INVALID_DATA, "section 9 missing", be.zkey_load, rebuild(secs, s9=None))
    expect(be, INVALID_DATA, "section 3 appears twice", be.zkey_load, zo.binfile(b"zkey", 1, secs + [(3, S[3])]))
    # wtns: wrong length, a value >= r, z[0] != 1, the other curve's prime
    expect(be, ASSIGNMENT, "wtns", be.wtns_read, zo.write_wtns(curve, case.z), case.n_vars + 1)
    w = bytearray(zo.write_wtns(curve, case.z))
    data_at = len(w) - 32 * case.n_vars
    w[data_at + 3 * 32: data_at + 4 * 32] = curve.r.to_bytes(32, "little")
    expect(be, INVALID_DATA, "wtns[3]: value not below r", be.wtns_read, bytes(w), case.n_vars)
    w = bytearray(zo.write_wtns(curve, case.z))
    w[data_at] = 2
    expect(be, INVALID_DATA, "wtns[0]: z[0] is not 1", be.wtns_read, bytes(w), case.n_vars)
    w = bytearray(zo.write_wtns(curve, case.z))
    w[28:60] = other.r.to_bytes(32, "little")   # magic, version, count, section header, n8
    expect(be, INVALID_ARG, "wtns: the prime", be.wtns_read, bytes(w), case.n_vars)
    case.free(be)
