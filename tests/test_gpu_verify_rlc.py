"""One verdict for a batch of Groth16 proofs by a random linear combination (b2s_groth16_verify_batch_rlc,
Backend.groth16_verify_all): valid batches, every tampering class, random mixtures against the per-proof verdicts of
b2s_groth16_verify_batch, the randomness actually separating proofs, points at infinity, chunked host batches and device
buffers, proofs from the GPU prover, and the error codes."""
import ctypes
import random

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests.test_gpu_verify import Sim, fixed_base, fr_words, tamper
from tests.util import csr_from_rows, pack_fr, pack_u32

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def verify_all(sim, inputs, A, B, C, rho=None):
    return sim.be.groth16_verify_all(sim.pvk, inputs, sim.ni, A, B, C, rho=rho)


def rows(sim, arrs, n):
    """the first n proofs of (inputs, A, B, C)"""
    inputs, A, B, C = arrs
    w1, w2 = sim.be.g1_bytes // 4, sim.be.g2_bytes // 4
    return (inputs[:n * sim.ni * 8].copy() if sim.ni else None, A[:n * w1].copy(), B[:n * w2].copy(), C[:n * w1].copy())


def tamper_one(sim, kind, i, x, a, b, c, arrs):
    """arrs with one tampering class applied to proof i alone (the classes of test_gpu_verify.tamper)"""
    inputs, A, B, C = [v.copy() if v is not None else None for v in arrs]
    be, r, n = sim.be, sim.curve.r, len(a)
    w1, w2 = be.g1_bytes // 4, be.g2_bytes // 4
    if kind == "a":        # A + G1
        A[i * w1:(i + 1) * w1] = fixed_base(be, 1, [(a[i] + 1) % r])
    elif kind == "b":      # another proof's B
        B[i * w2:(i + 1) * w2] = fixed_base(be, 2, [b[(i + 1) % n] if n > 1 else (b[i] + 1) % r])
    elif kind == "c":      # C negated
        C[i * w1:(i + 1) * w1] = fixed_base(be, 1, [(-c[i]) % r])
    elif kind == "x":      # one public input changed
        inputs[i * sim.ni * 8:i * sim.ni * 8 + 8] = fr_words(sim.curve, [(x[i][0] + 1) % r])
    elif kind == "swap":   # two proofs' inputs swapped
        j = (i + 1) % n
        ri, rj = inputs[i * sim.ni * 8:(i + 1) * sim.ni * 8].copy(), inputs[j * sim.ni * 8:(j + 1) * sim.ni * 8].copy()
        inputs[i * sim.ni * 8:(i + 1) * sim.ni * 8], inputs[j * sim.ni * 8:(j + 1) * sim.ni * 8] = rj, ri
    elif kind == "a_inf":  # A at infinity
        A[i * w1:(i + 1) * w1] = 0
    return inputs, A, B, C


@pytest.mark.parametrize("ni", [0, 1, 16, 100])
def test_valid_tampered_and_mixed(be, ni):
    rng = random.Random(0x7C1 + 5 * ni + be.curve)
    sim = Sim(be, rng, ni)
    n_max = 1 << 16
    x, a, b = sim.scalars(rng, n_max)
    c = sim.c_of(x, a, b)
    full = sim.arrays(x, a, b, c)
    for n in (1, 2, 31, 4097, n_max):
        assert verify_all(sim, *rows(sim, full, n)), n
    n = 31
    base = rows(sim, full, n)
    kinds = ["a", "b", "c", "a_inf"] + (["x", "swap"] if ni else [])
    for kind in kinds:
        for i in (0, n // 2, n - 1):
            arrs = tamper_one(sim, kind, i, x[:n], a[:n], b[:n], c[:n], base)
            assert not sim.verify(*arrs).all(), (kind, i)   # the per-proof path agrees that the batch is broken
            assert not verify_all(sim, *arrs), (kind, i)
    # random mixtures: the batch verdict is the AND of the per-proof verdicts
    for _ in range(5):
        m = rng.randrange(1, 65)
        xs, as_, bs = sim.scalars(rng, m)
        cs = sim.c_of(xs, as_, bs)
        if rng.random() < 0.3:
            arrs = sim.arrays(xs, as_, bs, cs)
        else:
            tx, ta, tb, tc, zero_a, _ = tamper(sim, rng, xs, as_, bs, cs, m)
            arrs = sim.arrays(tx, ta, tb, tc)
            for i in zero_a:
                arrs[1][i * (be.g1_bytes // 4):(i + 1) * (be.g1_bytes // 4)] = 0
        assert verify_all(sim, *arrs) == bool(sim.verify(*arrs).all()), m
    be.pvk_free(sim.pvk)


def test_rho_is_used(be):
    """C_1 + D and C_2 - D: invalid proofs whose errors cancel under equal weights"""
    rng = random.Random(0x2D0 + be.curve)
    sim = Sim(be, rng, 1)
    x, a, b = sim.scalars(rng, 2)
    c = sim.c_of(x, a, b)
    d = rng.randrange(1, sim.curve.r)
    c = [(c[0] + d) % sim.curve.r, (c[1] - d) % sim.curve.r]
    arrs = sim.arrays(x, a, b, c)
    assert sim.verify(*arrs).tolist() == [False, False]
    assert verify_all(sim, *arrs, rho=pack_u32([1, 1], 4))
    assert not verify_all(sim, *arrs, rho=pack_u32([rng.randrange(2, 1 << 128) for _ in range(2)], 4))
    assert not verify_all(sim, *arrs)
    be.pvk_free(sim.pvk)


def test_points_at_infinity(be):
    rng = random.Random(0x1F0 + be.curve)
    sim = Sim(be, rng, 2)
    r = sim.curve.r
    x, a, b = sim.scalars(rng, 5)
    # proof 2 has C = infinity: b chosen so that a b = alpha beta + gamma IC
    ic = sim.g[0] + sum(v * g for v, g in zip(x[2], sim.g[1:]))
    b[2] = (sim.al * sim.bt + sim.gm * ic) * pow(a[2], -1, r) % r
    c = sim.c_of(x, a, b)
    assert c[2] == 0
    inputs, A, B, C = sim.arrays(x, a, b, c)
    w1, w2 = be.g1_bytes // 4, be.g2_bytes // 4
    assert not C[2 * w1:3 * w1].any()
    assert sim.verify(inputs, A, B, C).all()
    assert verify_all(sim, inputs, A, B, C)
    A0 = A.copy()
    A0[3 * w1:4 * w1] = 0
    assert not verify_all(sim, inputs, A0, B, C)
    B0 = B.copy()
    B0[w2:2 * w2] = 0
    assert not verify_all(sim, inputs, A, B0, C)
    be.pvk_free(sim.pvk)


def test_chunks_and_device_buffers(be):
    """2^18 + 3 proofs from host memory cross the 2^18 chunk boundary; device buffers give the same verdicts"""
    import torch

    from snark_b200.lib import random_rho

    rng = random.Random(0xC4 + be.curve)
    sim = Sim(be, rng, 1)
    base = 4096
    x, a, b = sim.scalars(rng, base)
    inputs, A, B, C = sim.arrays(x, a, b, sim.c_of(x, a, b))
    n = (1 << 18) + 3
    reps = -(-n // base)
    w1, w2 = be.g1_bytes // 4, be.g2_bytes // 4
    inputs, A, B, C = np.tile(inputs, reps)[:n * 8], np.tile(A, reps)[:n * w1], np.tile(B, reps)[:n * w2], np.tile(C, reps)[:n * w1]
    bad = inputs.copy()
    i = (1 << 18) + 1                    # in the second chunk
    bad[i * 8] ^= 1
    rho = random_rho(n)
    assert verify_all(sim, inputs, A, B, C, rho=rho)
    assert not verify_all(sim, bad, A, B, C, rho=rho)
    dev = torch.device("cuda")
    t = lambda arr: torch.from_numpy(arr.view(np.int32)).to(dev)
    assert be.groth16_verify_all(sim.pvk, t(inputs), 1, t(A), t(B), t(C), rho=t(rho), n_proofs=n)
    assert not be.groth16_verify_all(sim.pvk, t(bad), 1, t(A), t(B), t(C), rho=t(rho), n_proofs=n)
    assert be.groth16_verify_all(sim.pvk, t(inputs), 1, t(A), t(B), t(C), n_proofs=n)   # rho drawn for device buffers
    be.pvk_free(sim.pvk)


def test_gpu_prover_proofs(be):
    curve = CURVES[be.curve]
    rng = random.Random(0x9E + be.curve)
    cs = orc.circuit2(curve, 1, 1, 2)
    cs.finalize()
    mats, inst, wit = cs.to_matrices(), cs.instance_assignment, cs.witness_assignment
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(curve, M) for M in mats])
    pkh, vk = be.groth16_setup(m, pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)]), len(inst))
    proofs = [be.groth16_prove(pkh, m, pack_fr(curve, inst), pack_fr(curve, wit), pack_fr(curve, [rng.randrange(curve.r)]),
                               pack_fr(curve, [rng.randrange(curve.r)])) for _ in range(3)]
    x = list(inst[1:])
    ni = len(x)
    inputs = np.tile(pack_fr(curve, x), len(proofs))
    pvk = be.vk_prepare(vk)
    assert be.groth16_verify_all(pvk, inputs, ni, *[np.concatenate([p[k] for p in proofs]) for k in range(3)])
    rt = [be.proof_from_bytes(be.proof_bytes(*p), validate=True) for p in proofs]
    assert be.groth16_verify_all(pvk, inputs, ni, *[np.concatenate([p[k] for p in rt]) for k in range(3)])
    wrong = pack_fr(curve, [(x[0] + 1) % curve.r] + x[1:])
    assert not be.groth16_verify_all(pvk, wrong, ni, *proofs[0])
    be.pvk_free(pvk); be.pk_free(pkh); be.r1cs_free(m)


def test_errors(be):
    from snark_b200 import B2SError, Backend
    from snark_b200.lib import random_rho

    rng = random.Random(0xE8 + be.curve)
    sim = Sim(be, rng, 2)
    n = 40
    x, a, b = sim.scalars(rng, n)
    inputs, A, B, C = sim.arrays(x, a, b, sim.c_of(x, a, b))
    rho = random_rho(n)
    rho[17 * 4:18 * 4] = 0
    rho[30 * 4:31 * 4] = 0
    with pytest.raises(B2SError) as e:
        verify_all(sim, inputs, A, B, C, rho=rho)
    assert e.value.code == 16 and "rho[17] is zero" in str(e.value)
    with pytest.raises(B2SError) as e:
        be.groth16_verify_all(sim.pvk, inputs, 1, A, B, C)
    assert e.value.code == 7
    other = Backend(curve=1 - be.curve)
    try:
        osim = Sim(other, random.Random(1), 2)
        with pytest.raises(B2SError) as e:
            be.groth16_verify_all(osim.pvk, inputs, 2, A, B, C)
        assert e.value.code == 16
        other.pvk_free(osim.pvk)
    finally:
        other.close()
    lib, ok = be.lib, ctypes.c_uint8(7)
    rp = random_rho(n)
    args = lambda **kw: [kw.get(k, v) for k, v in [("x", inputs.ctypes.data), ("a", A.ctypes.data), ("b", B.ctypes.data),
                                                     ("c", C.ctypes.data), ("rho", rp.ctypes.data)]]
    for k in ("x", "a", "b", "c", "rho"):
        xi, ai, bi, ci, ri = args(**{k: None})
        assert lib.b2s_groth16_verify_batch_rlc(be.h, sim.pvk, n, xi, 2, ai, bi, ci, ri, 0, ctypes.byref(ok)) == 16, k
    assert lib.b2s_groth16_verify_batch_rlc(be.h, sim.pvk, n, *args()[:1], 2, *args()[1:], 0, None) == 16
    assert lib.b2s_groth16_verify_batch_rlc(be.h, None, n, *args()[:1], 2, *args()[1:], 0, ctypes.byref(ok)) == 16
    ok.value = 7
    assert lib.b2s_groth16_verify_batch_rlc(be.h, sim.pvk, 0, None, 2, None, None, None, None, 0, ctypes.byref(ok)) == 0
    assert ok.value == 1
    assert be.groth16_verify_all(sim.pvk, None, 2, A[:0], B[:0], C[:0])
    be.pvk_free(sim.pvk)
