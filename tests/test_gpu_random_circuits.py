"""Random circuits at full size on all three curves, element by element against the C++ oracle (oracle/c/oracle.cpp).

The other full-size tests run the DummyCircuit: unit coefficients, three columns, a witness of two values.  Here the rows
have 0 to 6 terms with duplicate columns, half the coefficients are random values from a pool of 2^16 + 3 (so the
interned coefficient ids run past 2^16), the columns are uniform over every variable, and z is uniform with 0, 1 and r - 1
scattered in.  Two shapes per size: n_rows + n_instance = N (every row of the domain used) and N / 2 + 1 (the domain has
just doubled and is mostly padding).  Checked, with curve ids 0, 1 and 2:

* b2s_witness_map and b2s_witness_map_qap(CIRCOM) at 2^17, 2^20 and 2^24 against orc_witness_map / orc_witness_map_circom,
  at 2^20 also with the composed twiddles (B2S_NTT_FULL=0, a fresh context);
* b2s_ntt forward, inverse, coset and coset-inverse at the same sizes against orc_ntt;
* b2s_groth16_prove and b2s_groth16_prove_batch (3 assignments) under both reductions at 2^20, and b2s_groth16_prove at
  2^24 (libsnark on BN254 and BLS12-377, circom on BN254: the benchmarked shape of those curves, h-query table by the
  default rule), against the proof predicted from a key of known discrete logs and the oracle's h.

The 2^24 cases run when 24 is in B2S_FULLSIZE_LOG, as in test_gpu_fullsize.py.
"""
import functools
import random

import numpy as np
import pytest

from oracle import cnative
from oracle.params import BLS12_381, BN254
from tests.bls377_oracle import BLS12_377
from tests.test_gpu_fullsize import FULLSIZE_LOGS
from tests.util import known_log_key, known_log_proof, pack_fr, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254, BLS12_377]
CIDS = [0, 1, 2]
LIB, CIRCOM = 0, 1
SIZES = [17, 20] + ([24] if 24 in FULLSIZE_LOGS else [])
N_INST = 3
ROW_LEN_P = [0.22, 0.40, 0.20, 0.08, 0.05, 0.03, 0.02]     # terms per row 0..6, mean 1.51
POOL = 1 << 16


@functools.lru_cache(maxsize=None)
def coeff_pool(cid):
    """(POOL + 3) x 8 Montgomery limbs: 1, 2, r - 1, then POOL random values"""
    curve = CURVES[cid]
    rng = random.Random(0x9001 + cid)
    return pack_fr(curve, [1, 2, curve.r - 1] + [rng.randrange(3, curve.r - 1) for _ in range(POOL)]).reshape(-1, 8)


def random_fr(curve, nrng, n):
    """n x 8 limbs of field elements below r, close to uniform, with 0, 1 and r - 1 each at about n / 4096 places"""
    a = nrng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint32)
    bits = curve.r.bit_length()
    a[:, 7] &= np.uint32((1 << (bits - 224)) - 1)
    over = a[:, 7] >= np.uint32(curve.r >> 224)             # possibly >= r: drop the top bit
    a[over, 7] &= np.uint32((1 << (bits - 225)) - 1)
    special = pack_fr(curve, [0, 1, curve.r - 1]).reshape(3, 8)
    k = max(1, n >> 12)
    for i in range(3):
        a[nrng.integers(0, n, size=k)] = special[i]
    return a


def random_matrix(cid, nrng, n_rows, n_vars):
    """CSR (row_ptr u64, col u32, coeff u32 limbs) of a random matrix: row lengths from ROW_LEN_P, columns uniform with about
    one in eight terms after the first of its row repeating the column before it, half the coefficients ONE and the rest
    uniform over the pool"""
    lens = nrng.choice(len(ROW_LEN_P), size=n_rows, p=ROW_LEN_P).astype(np.uint64)
    row_ptr = np.zeros(n_rows + 1, dtype=np.uint64)
    np.cumsum(lens, out=row_ptr[1:])
    nnz = int(row_ptr[-1])
    col = nrng.integers(0, n_vars, size=nnz, dtype=np.uint32)
    first = np.zeros(nnz, dtype=bool)
    first[row_ptr[:-1][lens > 0].astype(np.int64)] = True
    dup = np.flatnonzero(~first & (nrng.integers(0, 8, size=nnz, dtype=np.uint8) == 0))
    col[dup] = col[dup - 1]
    pool = coeff_pool(cid)
    cid_ = nrng.integers(0, len(pool), size=nnz, dtype=np.uint32)
    cid_[nrng.integers(0, 2, size=nnz, dtype=np.uint8) == 0] = 0
    return row_ptr, col, pool[cid_].reshape(-1)


def random_circuit(cid, log_n, shape, seed):
    """(csr3, n_rows, n_wit, z) with n_rows + N_INST = N ("full") or N / 2 + 1 ("half"), n_vars = n_rows + N_INST, z[0] = 1"""
    N = 1 << log_n
    n_rows = (N if shape == "full" else N // 2 + 1) - N_INST
    n_vars = n_rows + N_INST
    nrng = np.random.default_rng([seed, cid, log_n, int(shape == "full")])
    csr = [random_matrix(cid, nrng, n_rows, n_vars) for _ in range(3)]
    z = random_fr(CURVES[cid], nrng, n_vars)
    z[0] = pack_fr(CURVES[cid], [1])
    return csr, n_rows, n_vars - N_INST, z.reshape(-1)


@pytest.mark.parametrize("log_n", SIZES)
@pytest.mark.parametrize("cid", CIDS)
def test_witness_maps(cid, log_n, monkeypatch):
    """both witness maps, every element, both shapes; at 2^20 also with the composed twiddles (B2S_NTT_FULL=0)"""
    from snark_b200 import Backend

    backends = [Backend(curve=cid)]
    for shape in ("full", "half"):
        csr, n_rows, n_wit, z = random_circuit(cid, log_n, shape, seed=1)
        want = {LIB: cnative.witness_map(cid, csr, n_rows, N_INST, z),
                CIRCOM: cnative.witness_map_circom(cid, csr, n_rows, N_INST, z)}
        for i in range(2 if log_n == 20 else 1):
            if i == len(backends):      # only once the first context has built its tables for this size
                monkeypatch.setenv("B2S_NTT_FULL", "0")
                backends.append(Backend(curve=cid))
            be = backends[i]
            m = be.r1cs_upload(n_rows, N_INST, n_wit, csr)
            assert be.domain_size(m) == 1 << log_n
            for qap in (LIB, CIRCOM):
                assert np.array_equal(be.witness_map(m, z, qap=qap), want[qap]), (shape, qap, "composed" if i else "full")
            be.r1cs_free(m)
    for be in backends:
        be.close()


@pytest.mark.parametrize("log_n", SIZES)
@pytest.mark.parametrize("cid", CIDS)
def test_ntt(cid, log_n):
    """b2s_ntt in its four modes, every element"""
    from snark_b200 import Backend

    be = Backend(curve=cid)
    x = random_fr(CURVES[cid], np.random.default_rng([2, cid, log_n]), 1 << log_n).reshape(-1)
    for inverse in (False, True):
        for coset in (False, True):
            want = cnative.ntt(cid, x.copy(), log_n, inverse=inverse, coset=coset)
            got = be.ntt(x.copy(), log_n, inverse=inverse, coset=coset)
            assert np.array_equal(got, want), (inverse, coset)
    be.close()


def check_proofs(cid, qap, log_n, n_proofs, batch):
    """Proofs of n_proofs random assignments of a full-shape random circuit under a known-log key, one by one and (batch)
    in one b2s_groth16_prove_batch call, against the proofs predicted from the oracle's h"""
    from snark_b200 import Backend

    curve = CURVES[cid]
    r = curve.r
    N = 1 << log_n
    rng = random.Random(0x5EED + 8 * cid + 2 * log_n + qap)
    csr, n_rows, n_wit, z0 = random_circuit(cid, log_n, "full", seed=3)
    n_vars = N_INST + n_wit
    nrng = np.random.default_rng([4, cid, log_n])
    zs = [z0] + [random_fr(curve, nrng, n_vars).reshape(-1) for _ in range(n_proofs - 1)]
    for z in zs[1:]:
        z[:8] = pack_fr(curve, [1])
    rs = [rng.randrange(r) for _ in zs]
    ss = [rng.randrange(r) for _ in zs]
    wmap = cnative.witness_map_circom if qap == CIRCOM else cnative.witness_map
    be = Backend(curve=cid)
    m = be.r1cs_upload(n_rows, N_INST, n_wit, csr)
    consts = [rng.randrange(1, r) for _ in range(3)]
    pk, dl = known_log_key(be, curve, consts, N_INST, n_wit, N, seed=rng.randrange(1 << 30), qap=qap)
    want = []
    for z, rr, sv in zip(zs, rs, ss):
        h = wmap(cid, csr, n_rows, N_INST, z)
        want.append(known_log_proof(be, curve, consts, dl, z[: 8 * N_INST], z[8 * N_INST:], h, rr, sv))
    for i, z in enumerate(zs):
        got = be.groth16_prove(pk, m, z[: 8 * N_INST], z[8 * N_INST:], pack_fr(curve, [rs[i]]), pack_fr(curve, [ss[i]]))
        assert (unpack_points(curve, 1, got[0])[0], unpack_points(curve, 2, got[1])[0], unpack_points(curve, 1, got[2])[0]) == want[i], i
    if batch:
        a, b, c = be.groth16_prove_batch(pk, m, np.stack(zs), pack_fr(curve, rs), pack_fr(curve, ss))
        got = list(zip(unpack_points(curve, 1, a), unpack_points(curve, 2, b), unpack_points(curve, 1, c)))
        assert got == want
    be.pk_free(pk)
    be.r1cs_free(m)
    be.close()


@pytest.mark.parametrize("qap", [LIB, CIRCOM], ids=["libsnark", "circom"])
@pytest.mark.parametrize("cid", CIDS)
def test_proofs_2p20(cid, qap):
    check_proofs(cid, qap, 20, n_proofs=3, batch=True)


@pytest.mark.skipif(24 not in FULLSIZE_LOGS, reason="B2S_FULLSIZE_LOG without 24")
@pytest.mark.parametrize("cid,qap", [(1, LIB), (2, LIB), (1, CIRCOM)], ids=["bn254-libsnark", "bls12_377-libsnark", "bn254-circom"])
def test_proof_2p24(cid, qap):
    check_proofs(cid, qap, 24, n_proofs=1, batch=False)
