"""Groth16 verification of ark-serialized proofs (b2s_groth16_verify_batch_bytes, b2s_groth16_verify_batch_rlc_bytes):
valid and algebraically tampered batches against b2s_groth16_verify_batch on the same points, every decode failure on each
of A, B and C at the first, a middle and the last proof and across the 2^18 chunk boundary with the exact reason code the
oracle's rejection implies, the batch verdict, device buffers, proofs from the GPU prover, and the error codes."""
import ctypes
import random

import numpy as np
import pytest

from oracle import r1cs as orc
from oracle.params import BLS12_381, BN254
from tests.test_gpu_verify import Sim, tamper
from tests.util import csr_from_rows, pack_fr
from tests.wire_oracle import (REASON_FLAGS, REASON_NONCANONICAL, REASON_NOT_IN_SUBGROUP, REASON_NOT_ON_CURVE, _sqrt_fq,
                               _sqrt_fq2, point_compressed, point_deserialize, point_uncompressed, points_outside_subgroup)

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
CODE = {REASON_FLAGS: 1, REASON_NONCANONICAL: 2, REASON_NOT_ON_CURVE: 3, REASON_NOT_IN_SUBGROUP: 4}
GROUP = (1, 2, 1)   # the group of a, b, c
CH = 1 << 18


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


@pytest.fixture(scope="module")
def off_subgroup(be):
    """per group, a few on-curve points outside the prime-order subgroup (none for BN254 G1: cofactor 1)"""
    rng = random.Random(0x0FF + be.curve)
    return {g: points_outside_subgroup(CURVES[be.curve], g, rng, 3) for g in (1, 2)}


def encode(be, A, B, C, compressed):
    """affine arrays of n proofs -> n serialized proofs a || b || c, back to back (numpy uint8)"""
    n = len(A) * 4 // be.g1_bytes
    parts = [np.frombuffer(be.serialize_points(g, arr, n, compressed), dtype=np.uint8).reshape(n, -1)
             for g, arr in zip(GROUP, (A, B, C))]
    return np.ascontiguousarray(np.concatenate(parts, axis=1)).reshape(-1)


def elem_span(be, e, compressed):
    """byte range of element e inside one serialized proof, and the proof's size"""
    g1 = be.fq_bytes * (1 if compressed else 2)
    off = (0, g1, 3 * g1)[e]
    return off, off + g1 * GROUP[e], 4 * g1


def malformed(be, kind, group, data, compressed, rng, off_sub):
    """one encoded point (bytes) -> a malformed encoding of the given kind, or None where the kind does not apply"""
    curve = CURVES[be.curve]
    bls = curve is BLS12_381
    fq = be.fq_bytes
    coord = fq * group
    d = bytearray(data)
    flag_at = 0 if bls else (coord - 1 if compressed else 2 * coord - 1)
    if kind == "flags":                   # the compressed-form bit (BLS12-381) / the infinity bit (BN254) flipped
        d[flag_at] ^= 0x80 if bls else 0x40
        return bytes(d)
    if kind == "noncanonical":            # x (its c0 for G2) = p, the flag bits kept
        order = "big" if bls else "little"
        at = fq if (group == 2 and bls) else 0     # c0 is the second element on BLS12-381, the first on BN254
        keep = d[flag_at] & (0xE0 if bls else 0xC0)
        d[at:at + fq] = curve.p.to_bytes(fq, order)
        d[flag_at] = (d[flag_at] & (0x1F if bls else 0x3F)) | keep
        return bytes(d)
    if kind == "noroot":                  # compressed x whose x^3 + b has no square root
        if not compressed:
            return None
        from oracle.ec import groups
        G = groups(curve)[group - 1]
        f = G.f
        while True:
            x = rng.randrange(curve.p) if group == 1 else (rng.randrange(curve.p), rng.randrange(curve.p))
            rhs = f.add(f.mul(f.sqr(x), x), G.b)
            if (_sqrt_fq(curve.p, rhs) if group == 1 else _sqrt_fq2(curve.p, rhs)) is None:
                break
        y = G.gen[1]   # any y: only its sign bit is written
        return point_compressed(curve, group, (x, y))
    if kind == "offcurve":                # uncompressed (x, y + 1)
        if compressed:
            return None
        P = point_deserialize(curve, group, bytes(d), False, True)
        y = (P[1] + 1) % curve.p if group == 1 else ((P[1][0] + 1) % curve.p, P[1][1])
        return point_uncompressed(curve, group, (P[0], y))
    if kind == "subgroup":                # on the curve, outside the prime-order subgroup
        pts = off_sub[group]
        if not pts:
            return None
        enc = point_compressed if compressed else point_uncompressed
        return enc(curve, group, pts[rng.randrange(len(pts))])
    raise ValueError(kind)


KINDS = ("flags", "noncanonical", "noroot", "offcurve", "subgroup")


def expected_code(be, e, group, enc, compressed):
    """the reason code the oracle's rejection of `enc` implies"""
    with pytest.raises(ValueError) as exc:
        point_deserialize(CURVES[be.curve], group, enc, compressed, True)
    return 16 * (1 + e) + CODE[str(exc.value)]


def verify_bytes(sim, inputs, blob, compressed, n=None):
    return sim.be.groth16_verify_batch_bytes(sim.pvk, inputs, sim.ni, blob, compressed=compressed, n_proofs=n)


def valid_batch(sim, rng, n):
    x, a, b = sim.scalars(rng, n)
    return (x, a, b, sim.c_of(x, a, b)), sim.arrays(x, a, b, sim.c_of(x, a, b))


@pytest.mark.parametrize("ni", [0, 1, 16])
def test_valid_and_tampered(be, ni):
    """decoded proofs get the verdicts of the points path; every reason is 0 (A at infinity is a valid encoding)"""
    rng = random.Random(0xB7E + 3 * ni + be.curve)
    sim = Sim(be, rng, ni)
    n = 67
    (x, a, b, c), arrs = valid_batch(sim, rng, n)
    tx, ta, tb, tc, zero_a, bad = tamper(sim, rng, x, a, b, c, n)
    t_arrs = list(sim.arrays(tx, ta, tb, tc))
    w1 = be.g1_bytes // 4
    for i in zero_a:
        t_arrs[1][i * w1:(i + 1) * w1] = 0
    for compressed in (True, False):
        for inputs, A, B, C in (arrs, t_arrs):
            want = sim.verify(inputs, A, B, C)
            ok, reason = verify_bytes(sim, inputs, encode(be, A, B, C, compressed), compressed)
            assert np.array_equal(ok, want), compressed
            assert not reason.any()
        assert set(np.flatnonzero(~ok).tolist()) == bad
        for i in zero_a:
            assert not ok[i] and reason[i] == 0
    be.pvk_free(sim.pvk)


def test_decode_failures(be, off_subgroup):
    """each malformed encoding on A, B and C at the first, a middle and the last proof: ok = 0 and the oracle's reason there,
    every other verdict unchanged; a proof with two bad elements is named by the first; the batch verdict is 0"""
    rng = random.Random(0xDEC + be.curve)
    sim = Sim(be, rng, 1)
    n = 33
    (x, a, b, c), arrs = valid_batch(sim, rng, n)
    arrs = list(arrs)
    inputs = arrs[0].copy()
    inputs[5 * 8] ^= 1                    # proof 5 is algebraically invalid: its verdict stays 0, its reason 0
    base_ok = sim.verify(inputs, *arrs[1:])
    assert np.flatnonzero(~base_ok).tolist() == [5]
    for compressed in (True, False):
        blob = encode(be, *arrs[1:], compressed).reshape(n, -1)
        checked = 0
        for e in range(3):
            lo, hi, _ = elem_span(be, e, compressed)
            for kind in KINDS:
                bad = blob.copy()
                codes = {}
                for i in (0, n // 2, n - 1):
                    enc = malformed(be, kind, GROUP[e], bytes(bad[i, lo:hi]), compressed, rng, off_subgroup)
                    if enc is None:
                        break
                    bad[i, lo:hi] = np.frombuffer(enc, dtype=np.uint8)
                    codes[i] = expected_code(be, e, GROUP[e], enc, compressed)
                if not codes:
                    continue
                checked += 1
                ok, reason = verify_bytes(sim, inputs, bad.reshape(-1), compressed)
                want_ok, want_reason = base_ok.copy(), np.zeros(n, dtype=np.uint8)
                for i, code in codes.items():
                    want_ok[i], want_reason[i] = False, code
                assert np.array_equal(ok, want_ok), (compressed, e, kind)
                assert reason.tolist() == want_reason.tolist(), (compressed, e, kind)
                verdict, rs = be.groth16_verify_all_bytes(sim.pvk, arrs[0], 1, bad.reshape(-1), compressed=compressed)
                assert not verdict and rs.tolist() == want_reason.tolist(), (compressed, e, kind)
        assert checked >= 9
        # two bad elements in one proof: the first one is reported
        bad = blob.copy()
        for e, kind in ((2, "noncanonical"), (1, "flags")):
            lo, hi, _ = elem_span(be, e, compressed)
            bad[3, lo:hi] = np.frombuffer(malformed(be, kind, GROUP[e], bytes(bad[3, lo:hi]), compressed, rng, off_subgroup), dtype=np.uint8)
        ok, reason = verify_bytes(sim, inputs, bad.reshape(-1), compressed)
        assert not ok[3] and reason[3] == 32 + 1 and np.count_nonzero(reason) == 1
    be.pvk_free(sim.pvk)


def test_rlc(be):
    """one verdict: 1 for a valid batch, 0 with the reason for a malformed proof, 0 with all reasons 0 for an algebraically
    bad one; equal to groth16_verify_all on the decoded points with the same rho"""
    from snark_b200.lib import random_rho

    rng = random.Random(0x71C + be.curve)
    for ni in (0, 1, 16):
        sim = Sim(be, rng, ni)
        n = 40
        (x, a, b, c), (inputs, A, B, C) = valid_batch(sim, rng, n)
        rho = random_rho(n)
        for compressed in (True, False):
            blob = encode(be, A, B, C, compressed)
            verdict, reason = be.groth16_verify_all_bytes(sim.pvk, inputs, ni, blob, compressed=compressed, rho=rho)
            assert verdict and not reason.any()
            assert verdict == be.groth16_verify_all(sim.pvk, inputs, ni, A, B, C, rho=rho)
            # one malformed proof (B's flags)
            bad = blob.reshape(n, -1).copy()
            lo = elem_span(be, 1, compressed)[0]
            bad[17, lo + (0 if be.curve == 0 else (be.fq_bytes * 2 * (1 if compressed else 2) - 1))] ^= 0x80 if be.curve == 0 else 0x40
            verdict, reason = be.groth16_verify_all_bytes(sim.pvk, inputs, ni, bad.reshape(-1), compressed=compressed, rho=rho)
            assert not verdict and reason.tolist() == [0] * 17 + [32 + 1] + [0] * (n - 18)
            # one algebraically bad proof (C negated)
            c2 = list(c)
            c2[9] = (-c2[9]) % sim.curve.r
            _, A2, B2, C2 = sim.arrays(x, a, b, c2)
            verdict, reason = be.groth16_verify_all_bytes(sim.pvk, inputs, ni, encode(be, A2, B2, C2, compressed), compressed=compressed,
                                                          rho=rho)
            assert not verdict and not reason.any()
            assert verdict == be.groth16_verify_all(sim.pvk, inputs, ni, A2, B2, C2, rho=rho)
        be.pvk_free(sim.pvk)


def test_chunk_boundary(be, off_subgroup):
    """2^18 + 16 proofs: decode failures next to the chunk boundary, in both paths, from host and from device memory"""
    import torch

    rng = random.Random(0xC8 + be.curve)
    sim = Sim(be, rng, 1)
    base = 256
    (x, a, b, c), (inputs, A, B, C) = valid_batch(sim, rng, base)
    n = CH + 16
    reps = -(-n // base)
    inputs = np.tile(inputs, reps)[:n * 8]
    dev = torch.device("cuda")
    for compressed in (True, False):
        blob = np.tile(encode(be, A, B, C, compressed).reshape(base, -1), (reps, 1))[:n].copy()
        plan = [(CH - 1, 0, "flags"), (CH, 1, "subgroup" if off_subgroup[2] else "noncanonical"), (CH + 1, 2, "noncanonical"),
                (n - 1, 1, "noroot" if compressed else "offcurve")]
        want_reason = np.zeros(n, dtype=np.uint8)
        for i, e, kind in plan:
            lo, hi, _ = elem_span(be, e, compressed)
            enc = malformed(be, kind, GROUP[e], bytes(blob[i, lo:hi]), compressed, rng, off_subgroup)
            blob[i, lo:hi] = np.frombuffer(enc, dtype=np.uint8)
            want_reason[i] = expected_code(be, e, GROUP[e], enc, compressed)
        flat = blob.reshape(-1)
        ok, reason = verify_bytes(sim, inputs, flat, compressed)
        assert np.flatnonzero(~ok).tolist() == [i for i, _, _ in plan]
        assert np.array_equal(reason, want_reason)
        verdict, rs = be.groth16_verify_all_bytes(sim.pvk, inputs, 1, flat, compressed=compressed)
        assert not verdict and np.array_equal(rs, want_reason)
        # device memory: the same verdicts and reasons
        t_in = torch.from_numpy(inputs.view(np.int32)).to(dev)
        t_blob = torch.from_numpy(flat).to(dev)
        okd, rsd = torch.zeros(n, dtype=torch.uint8, device=dev), torch.full((n,), 0xEE, dtype=torch.uint8, device=dev)
        be.groth16_verify_batch_bytes(sim.pvk, t_in, 1, t_blob, compressed=compressed, ok=okd, reason=rsd)
        be.sync()
        assert np.array_equal(okd.cpu().numpy().astype(bool), ok) and np.array_equal(rsd.cpu().numpy(), reason)
        rsd.fill_(0xEE)
        verdict, _ = be.groth16_verify_all_bytes(sim.pvk, t_in, 1, t_blob, compressed=compressed, reason=rsd)
        be.sync()
        assert not verdict and np.array_equal(rsd.cpu().numpy(), want_reason)
        good = torch.from_numpy(np.tile(encode(be, A, B, C, compressed), reps)[:flat.size].copy()).to(dev)
        verdict, _ = be.groth16_verify_all_bytes(sim.pvk, t_in, 1, good, compressed=compressed)
        assert verdict
    be.pvk_free(sim.pvk)


def test_gpu_prover_proofs(be):
    curve = CURVES[be.curve]
    rng = random.Random(0x9D + be.curve)
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
    for compressed in (True, False):
        blob = b"".join(be.proof_bytes(*p, compressed=compressed) for p in proofs)
        ok, reason = be.groth16_verify_batch_bytes(pvk, inputs, ni, blob, compressed=compressed)
        assert ok.all() and not reason.any()
        verdict, reason = be.groth16_verify_all_bytes(pvk, inputs, ni, blob, compressed=compressed)
        assert verdict and not reason.any()
    wrong = pack_fr(curve, [(x[0] + 1) % curve.r] + x[1:])
    ok, reason = be.groth16_verify_batch_bytes(pvk, wrong, ni, be.proof_bytes(*proofs[0]))
    assert ok.tolist() == [False] and reason.tolist() == [0]
    be.pvk_free(pvk); be.pk_free(pkh); be.r1cs_free(m)


def test_errors(be):
    from snark_b200 import B2SError, Backend
    from snark_b200.lib import random_rho

    rng = random.Random(0xE9 + be.curve)
    sim = Sim(be, rng, 2)
    n = 40
    (x, a, b, c), (inputs, A, B, C) = valid_batch(sim, rng, n)
    blob = encode(be, A, B, C, True)
    rho = random_rho(n)
    rho[17 * 4:18 * 4] = 0
    rho[30 * 4:31 * 4] = 0
    with pytest.raises(B2SError) as e:
        be.groth16_verify_all_bytes(sim.pvk, inputs, 2, blob, rho=rho)
    assert e.value.code == 16 and "rho[17] is zero" in str(e.value)
    for fn in (be.groth16_verify_batch_bytes, be.groth16_verify_all_bytes):
        with pytest.raises(B2SError) as e:
            fn(sim.pvk, inputs, 1, blob)
        assert e.value.code == 7
        # a wrong length: one byte short, one byte over, the uncompressed size
        for bad_len in (blob[:-1], np.concatenate([blob, blob[:1]])):
            with pytest.raises(B2SError) as e:
                fn(sim.pvk, inputs, 2, bad_len, n_proofs=n)
            assert e.value.code == 21 and "proofs of" in str(e.value)
        with pytest.raises(B2SError) as e:
            fn(sim.pvk, inputs, 2, blob, compressed=False, n_proofs=n)
        assert e.value.code == 21
    other = Backend(curve=1 - be.curve)
    try:
        osim = Sim(other, random.Random(1), 2)
        for fn in (be.groth16_verify_batch_bytes, be.groth16_verify_all_bytes):
            with pytest.raises(B2SError) as e:
                fn(osim.pvk, inputs, 2, blob)
            assert e.value.code == 16
        other.pvk_free(osim.pvk)
    finally:
        other.close()
    lib = be.lib
    okb, rs = np.zeros(n, dtype=np.uint8), np.zeros(n, dtype=np.uint8)
    x_, p_ = inputs.ctypes.data, blob.ctypes.data
    L = len(blob)
    assert lib.b2s_groth16_verify_batch_bytes(be.h, None, n, x_, 2, p_, L, 1, 0, okb.ctypes.data, None) == 16
    assert lib.b2s_groth16_verify_batch_bytes(be.h, sim.pvk, n, None, 2, p_, L, 1, 0, okb.ctypes.data, None) == 16
    assert lib.b2s_groth16_verify_batch_bytes(be.h, sim.pvk, n, x_, 2, None, L, 1, 0, okb.ctypes.data, None) == 16
    assert lib.b2s_groth16_verify_batch_bytes(be.h, sim.pvk, n, x_, 2, p_, L, 1, 0, None, None) == 16
    assert lib.b2s_groth16_verify_batch_bytes(be.h, sim.pvk, n, x_, 2, p_, L, 1, 0, okb.ctypes.data, None) == 0   # reason optional
    assert okb.all()
    assert lib.b2s_groth16_verify_batch_bytes(be.h, sim.pvk, 0, None, 2, None, 0, 1, 0, None, None) == 0
    ok = ctypes.c_uint8(7)
    rp = random_rho(n)
    r_ = rp.ctypes.data
    assert lib.b2s_groth16_verify_batch_rlc_bytes(be.h, None, n, x_, 2, p_, L, 1, r_, 0, ctypes.byref(ok), None) == 16
    for args in ((None, p_, r_), (x_, None, r_), (x_, p_, None)):
        ok.value = 7
        assert lib.b2s_groth16_verify_batch_rlc_bytes(be.h, sim.pvk, n, args[0], 2, args[1], L, 1, args[2], 0, ctypes.byref(ok), None) == 16
        assert ok.value == 0
    assert lib.b2s_groth16_verify_batch_rlc_bytes(be.h, sim.pvk, n, x_, 2, p_, L, 1, r_, 0, None, None) == 16
    ok.value = 7
    assert lib.b2s_groth16_verify_batch_rlc_bytes(be.h, sim.pvk, n, x_, 2, p_, L - 1, 1, r_, 0, ctypes.byref(ok), None) == 21
    assert ok.value == 0
    ok.value = 7
    assert lib.b2s_groth16_verify_batch_rlc_bytes(be.h, sim.pvk, 0, None, 2, None, 0, 1, None, 0, ctypes.byref(ok), None) == 0
    assert ok.value == 1
    assert lib.b2s_groth16_verify_batch_rlc_bytes(be.h, sim.pvk, n, x_, 2, p_, L, 1, r_, 0, ctypes.byref(ok), rs.ctypes.data) == 0
    assert ok.value == 1 and not rs.any()
    # n = 0 through the bindings
    ok_, reason = be.groth16_verify_batch_bytes(sim.pvk, None, 2, b"")
    assert ok_.size == 0 and reason.size == 0
    assert be.groth16_verify_all_bytes(sim.pvk, None, 2, b"")[0]
    be.pvk_free(sim.pvk)
