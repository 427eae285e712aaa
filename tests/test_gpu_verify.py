"""Batched Groth16 verification and element-wise pairings on the GPU (b2s_vk_prepare, b2s_groth16_verify_batch, b2s_pairing):
against the host build of the same pairing code (tests/native/host_pairing.cpp), the oracle's pairing, simulated proofs
with known discrete logs (valid ones and every tampering class), and proofs from the GPU prover."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.ec import groups
from oracle.pairing import engine
from oracle.params import BLS12_381, BN254
from tests.pairing_oracle import gt_to_oracle, pairing_k
from tests.util import csr_from_rows, pack_fr, pack_points, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hostpair") / "libhostpair.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "native", "host_pairing.cpp")])
    return ctypes.CDLL(so)


def fr_words(curve, xs):
    """ints -> Montgomery Fr limbs (uint32), vectorised through bytes"""
    R = 1 << 256
    return np.frombuffer(b"".join((x * R % curve.r).to_bytes(32, "little") for x in xs), dtype=np.uint32).copy()


def fixed_base(be, group, scalars):
    curve = CURVES[be.curve]
    return be.fixed_base(group, fr_words(curve, scalars), len(scalars))


class Sim:
    """A verifying key with known logs (alpha, beta, gamma, delta, g_j) and proofs made without a prover:
    for random a, b:  c = (a b - alpha beta - gamma (g_0 + sum_j x_j g_j)) / delta,  A = aG1, B = bG2, C = cG1."""

    def __init__(self, be, rng, ni, zero_abc0=False):
        self.be, self.curve, self.ni = be, CURVES[be.curve], ni
        r = self.curve.r
        self.al, self.bt, self.gm, self.dl = [rng.randrange(1, r) for _ in range(4)]
        self.g = [0 if zero_abc0 else rng.randrange(1, r)] + [rng.randrange(1, r) for _ in range(ni)]
        g2 = fixed_base(be, 2, [self.bt, self.gm, self.dl])
        w2 = be.g2_bytes // 4
        self.vk = {"alpha_g1": fixed_base(be, 1, [self.al]), "beta_g2": g2[:w2].copy(), "gamma_g2": g2[w2:2 * w2].copy(),
                   "delta_g2": g2[2 * w2:].copy(), "gamma_abc_g1": fixed_base(be, 1, self.g)}
        self.pvk = be.vk_prepare(self.vk)

    def scalars(self, rng, n):
        r = self.curve.r
        x = [[rng.randrange(r) for _ in range(self.ni)] for _ in range(n)]
        a = [rng.randrange(1, r) for _ in range(n)]
        b = [rng.randrange(1, r) for _ in range(n)]
        return x, a, b

    def c_of(self, x, a, b):
        r = self.curve.r
        dinv = pow(self.dl, -1, r)
        ab = self.al * self.bt
        out = []
        for xi, ai, bi in zip(x, a, b):
            ic = self.g[0] + sum(v * gj for v, gj in zip(xi, self.g[1:]))
            out.append((ai * bi - ab - self.gm * ic) * dinv % r)
        return out

    def arrays(self, x, a, b, c):
        be = self.be
        inputs = fr_words(self.curve, [v for row in x for v in row]) if self.ni else None
        return inputs, fixed_base(be, 1, a), fixed_base(be, 2, b), fixed_base(be, 1, c)

    def verify(self, inputs, A, B, C):
        return self.be.groth16_verify_batch(self.pvk, inputs, self.ni, A, B, C)


def tamper(sim, rng, x, a, b, c, n):
    """Apply each tampering class at its own indices; -> (x, a, b, c, zero_a indices, bad indices)"""
    x, a, b, c = [list(r) for r in x], list(a), list(b), list(c)
    r = sim.curve.r
    idx = rng.sample(range(n), min(n, 8))
    bad, zero_a = set(), []
    k = iter(idx)
    i = next(k, None)
    if i is not None:
        a[i] = (a[i] + 1) % r; bad.add(i)                       # A + G1
    i = next(k, None)
    if i is not None:
        b[i] = b[(i + 1) % n] if n > 1 else (b[i] + 1) % r; bad.add(i)   # another proof's B
    i = next(k, None)
    if i is not None:
        c[i] = (-c[i]) % r; bad.add(i)                          # C negated
    if sim.ni:
        i = next(k, None)
        if i is not None:
            x[i][rng.randrange(sim.ni)] += 1; bad.add(i)          # one public input changed
        i, j = next(k, None), next(k, None)
        if j is not None:
            x[i], x[j] = x[j], x[i]; bad.update((i, j))           # two proofs' inputs swapped
    i = next(k, None)
    if i is not None:
        zero_a.append(i); bad.add(i)                            # A at infinity
    return x, a, b, c, zero_a, bad


def check_batch(sim, rng, x, a, b, c, n):
    c_ok = sim.c_of(x, a, b)
    assert sim.verify(*sim.arrays(x, a, b, c_ok)).all()
    tx, ta, tb, tc, zero_a, bad = tamper(sim, rng, x, a, b, c_ok, n)
    inputs, A, B, C = sim.arrays(tx, ta, tb, tc)
    w1 = sim.be.g1_bytes // 4
    for i in zero_a:
        A[i * w1:(i + 1) * w1] = 0
    ok = sim.verify(inputs, A, B, C)
    assert set(np.flatnonzero(~ok).tolist()) == bad


@pytest.mark.parametrize("ni", [0, 1, 16, 100])
def test_simulated_batches(be, ni):
    rng = random.Random(0x5E1 + 7 * ni + be.curve)
    sim = Sim(be, rng, ni)
    n_max = 1 << 16
    x, a, b = sim.scalars(rng, n_max)
    for n in (1, 31, 4097, n_max):
        check_batch(sim, rng, x[:n], a[:n], b[:n], None, n)
    be.pvk_free(sim.pvk)


def test_pairing_matches_host_and_oracle(be, host):
    curve = CURVES[be.curve]
    rng = random.Random(0x9A1 + be.curve)
    n = 200
    P = fixed_base(be, 1, [rng.randrange(1, curve.r) for _ in range(n)])
    Q = fixed_base(be, 2, [rng.randrange(1, curve.r) for _ in range(n)])
    w1, w2 = be.g1_bytes // 4, be.g2_bytes // 4
    for i in (3, 50, 51, 199):
        P[i * w1:(i + 1) * w1] = 0
    for i in (7, 51, 120):
        Q[i * w2:(i + 1) * w2] = 0
    got = be.pairing(P, Q)
    want = np.zeros_like(got)
    host.ht_pairing(be.curve, 0, P.ctypes.data_as(ctypes.c_void_p), Q.ctypes.data_as(ctypes.c_void_p),
                    want.ctypes.data_as(ctypes.c_void_p), n)
    assert np.array_equal(got, want)
    gts = gt_to_oracle(curve, got)
    one = engine(curve).Fq12.one()
    assert all(gts[i] == one for i in (3, 7, 50, 51, 120, 199))
    Pp, Qp = unpack_points(curve, 1, P), unpack_points(curve, 2, Q)
    k = pairing_k(curve)
    for i in (0, 1):
        assert gts[i] == engine(curve).pairing(Pp[i], Qp[i]).pow(k), i
    # device buffers give the same values
    import torch

    dev = torch.device("cuda")
    out = torch.zeros(got.size, dtype=torch.int32, device=dev)
    be.pairing(torch.from_numpy(P.view(np.int32)).to(dev), torch.from_numpy(Q.view(np.int32)).to(dev), n=n, out=out)
    be.sync()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), got)


def test_prepared_alpha_beta_is_the_pairing(be):
    """With gamma_abc = [infinity] and no inputs, the proof (alpha, beta, infinity) is accepted exactly when the kernels'
    e(alpha, beta) equals the one b2s_vk_prepare stored."""
    rng = random.Random(0xAB + be.curve)
    sim = Sim(be, rng, 0, zero_abc0=True)
    A, B = sim.vk["alpha_g1"], sim.vk["beta_g2"]
    C = np.zeros_like(A)
    assert sim.verify(None, A, B, C).tolist() == [True]
    assert sim.verify(None, A, B, sim.vk["alpha_g1"]).tolist() == [False]
    be.pvk_free(sim.pvk)


def test_gpu_prover_proofs(be):
    curve = CURVES[be.curve]
    rng = random.Random(0x9F + be.curve)
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(curve, M) for M in mats])
    pkh, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), len(inst))
    proofs = [be.groth16_prove(pkh, m, pack_fr(curve, inst), pack_fr(curve, wit), pack_fr(curve, [rng.randrange(curve.r)]),
                               pack_fr(curve, [rng.randrange(curve.r)])) for _ in range(3)]
    x = list(inst[1:])
    ni = len(x)
    cat = lambda k: np.concatenate([p[k] for p in proofs])
    inputs = np.tile(pack_fr(curve, x), len(proofs))
    pvk = be.vk_prepare(vk)
    assert be.groth16_verify_batch(pvk, inputs, ni, cat(0), cat(1), cat(2)).all()
    # after a round trip through ark-serialize bytes, with validation
    rt = [be.proof_from_bytes(be.proof_bytes(*p), validate=True) for p in proofs]
    assert be.groth16_verify_batch(pvk, inputs, ni, *[np.concatenate([p[k] for p in rt]) for k in range(3)]).all()
    vk2, _ = be.vk_from_bytes(be.vk_bytes(vk["alpha_g1"], vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"], vk["gamma_abc_g1"], len(inst)))
    pvk2 = be.vk_prepare(vk2)
    assert be.groth16_verify_batch(pvk2, inputs, ni, cat(0), cat(1), cat(2)).all()
    wrong = pack_fr(curve, [(x[0] + 1) % curve.r] + x[1:])
    assert be.groth16_verify_batch(pvk, wrong, ni, *proofs[0]).tolist() == [False]
    be.pvk_free(pvk); be.pvk_free(pvk2); be.pk_free(pkh); be.r1cs_free(m)


def test_device_buffers_and_chunks(be):
    """Device buffers give the host verdicts; a 2^20 host batch crosses several 2^18 chunks with invalid proofs next to
    the chunk boundaries."""
    import torch

    rng = random.Random(0xD1 + be.curve)
    sim = Sim(be, rng, 1)
    n = 1 << 20
    # 2^20 distinct proofs would take minutes of Python: tile 4096 valid ones, then break some near each boundary
    base = 4096
    x, a, b = sim.scalars(rng, base)
    inputs, A, B, C = sim.arrays(x, a, b, sim.c_of(x, a, b))
    reps = n // base
    inputs, A, B, C = np.tile(inputs, reps), np.tile(A, reps), np.tile(B, reps), np.tile(C, reps)
    w1, fr = be.g1_bytes // 4, 8
    bad = sorted({k * (1 << 18) + d for k in range(1, 4) for d in (-1, 0)} | {0, n - 1})
    for i in bad:
        inputs[i * fr] ^= 1              # the public input changes (its Montgomery form is no longer the valid one)
    ok = sim.verify(inputs, A, B, C)
    assert np.flatnonzero(~ok).tolist() == bad
    dev = torch.device("cuda")
    m = 1 << 16
    t = lambda arr: torch.from_numpy(arr.view(np.int32)).to(dev)
    okd = torch.zeros(m, dtype=torch.uint8, device=dev)
    be.groth16_verify_batch(sim.pvk, t(inputs[:m * fr]), 1, t(A[:m * w1]), t(B[:m * 2 * w1]), t(C[:m * w1]), n_proofs=m, ok=okd)
    be.sync()
    assert np.array_equal(okd.cpu().numpy().astype(bool), ok[:m])
    be.pvk_free(sim.pvk)


def test_errors(be):
    from snark_b200 import B2SError

    rng = random.Random(0xE7 + be.curve)
    sim = Sim(be, rng, 2)
    x, a, b = sim.scalars(rng, 1)
    inputs, A, B, C = sim.arrays(x, a, b, sim.c_of(x, a, b))
    with pytest.raises(B2SError) as e:
        be.groth16_verify_batch(sim.pvk, inputs, 1, A, B, C)
    assert e.value.code == 7
    lib = be.lib
    assert lib.b2s_groth16_verify_batch(be.h, None, 1, inputs.ctypes.data, 2, A.ctypes.data, B.ctypes.data, C.ctypes.data, 0, None) == 16
    assert lib.b2s_groth16_verify_batch(be.h, sim.pvk, 1, None, 2, A.ctypes.data, B.ctypes.data, C.ctypes.data, 0, None) == 16
    assert lib.b2s_groth16_verify_batch(be.h, sim.pvk, 0, None, 2, None, None, None, 0, None) == 0
    assert lib.b2s_pairing(be.h, None, None, 1, 0, None) == 16
    assert lib.b2s_pairing(be.h, None, None, 0, 0, None) == 0
    h = ctypes.c_void_p()
    assert lib.b2s_vk_prepare(be.h, sim.vk["alpha_g1"].ctypes.data, sim.vk["beta_g2"].ctypes.data, sim.vk["gamma_g2"].ctypes.data,
                              sim.vk["delta_g2"].ctypes.data, None, 0, ctypes.byref(h)) == 7
    be.pvk_free(sim.pvk)
