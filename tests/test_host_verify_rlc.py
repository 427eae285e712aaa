"""The random-linear-combination batch check of the verify path (snark_b200/csrc/pairing.cuh: cyclotomic_exp, rlc_miller,
rlc_verdict), compiled for the host, against the oracle's GT powers, the per-pair Miller loop of tests/native/host_pairing.cpp
and the per-proof verdict: one verdict for a batch must be the AND of the per-proof verdicts."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from oracle.ec import groups
from oracle.pairing import engine
from oracle.params import BLS12_381, BN254
from tests.pairing_oracle import gt_bytes, gt_to_oracle, pairing_k, random_gt_raw
from tests.util import pack_fr, pack_points, pack_u32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = [BLS12_381, BN254]
IDS = ["bls12_381", "bn254"]


def _compile(tmp_path_factory, name):
    so = str(tmp_path_factory.mktemp(name) / f"lib{name}.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "native", f"{name}.cpp")])
    return ctypes.CDLL(so)


@pytest.fixture(scope="module")
def rlc(tmp_path_factory):
    return _compile(tmp_path_factory, "host_verify_rlc")


@pytest.fixture(scope="module")
def pair(tmp_path_factory):
    return _compile(tmp_path_factory, "host_pairing")


def vp(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def rho_words(rhos):
    return pack_u32(rhos, 4)


def gt_random(pair, curve, rng, count):
    """`count` elements of GT: final exponentiations of random Fq12 elements"""
    f = random_gt_raw(curve, rng, count)
    out = np.zeros_like(f)
    pair.ht_fp12_op(curve.curve_id, 8, vp(f), None, vp(out), count)
    return out


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_cyclotomic_exp(rlc, pair, curve):
    rng = random.Random(0xC5E + curve.curve_id)
    r = curve.r
    exps = [0, 1, 2, r - 1, (1 << 128) - 1, rng.randrange(r), rng.randrange(1 << 256)]
    f = gt_random(pair, curve, rng, 1)
    fs = np.tile(f, len(exps))
    out = np.zeros_like(fs)
    rlc.ht_cyclotomic_exp(curve.curve_id, vp(fs), vp(pack_u32(exps, 8)), 8, vp(out), len(exps))
    F = gt_to_oracle(curve, f)[0]
    got = gt_to_oracle(curve, out)
    for e, g in zip(exps, got):
        assert g == F.pow(e), e
    # fewer words: the exponent's top words are simply absent
    out4 = np.zeros_like(f)
    rlc.ht_cyclotomic_exp(curve.curve_id, vp(f), vp(pack_u32([exps[4]], 4)), 4, vp(out4), 1)
    assert out4.tolist() == out[4 * len(f):5 * len(f)].tolist()


def host_miller(pair, curve, P, Q):
    out = np.zeros(len(P) * gt_bytes(curve) // 4, dtype=np.uint32)
    pair.ht_pairing(curve.curve_id, 1, vp(pack_points(curve, 1, P)), vp(pack_points(curve, 2, Q)), vp(out), len(P))
    return out


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_rlc_miller(rlc, pair, curve):
    """rho A and the Miller loop per thread, NF = 1, 2, 4 with a padded last group: the product of the per-pair Miller
    values of (rho_i A_i, B_i), rho_i A_i computed by the oracle; and after the final exponentiation, the oracle's pairings."""
    rng = random.Random(0x3F1 + curve.curve_id)
    G1, G2 = groups(curve)
    n = 7
    A = [G1.mul(G1.gen, rng.randrange(1, curve.r)) for _ in range(n)]
    B = [G2.mul(G2.gen, rng.randrange(1, curve.r)) for _ in range(n)]
    A[3], B[5] = None, None                                   # a pair at infinity on either side contributes 1
    rho = [rng.randrange(1, 1 << 128) for _ in range(n)]
    rho[1] = 1
    rho[2] = (1 << 128) - 1
    rA = [G1.mul(a, k) if a is not None else None for a, k in zip(A, rho)]
    per_pair = host_miller(pair, curve, rA, B)
    w = gt_bytes(curve) // 4
    for nf in (1, 2, 4):
        groups_ = -(-n // nf)
        out = np.zeros(groups_ * w, dtype=np.uint32)
        rlc.ht_rlc_miller(curve.curve_id, nf, vp(pack_points(curve, 1, A)), vp(pack_points(curve, 2, B)), vp(rho_words(rho)), vp(out), n)
        for g in range(groups_):
            want = per_pair[g * nf * w:(g * nf + 1) * w].copy()
            for i in range(g * nf + 1, min(n, (g + 1) * nf)):
                nxt = np.zeros_like(want)
                pair.ht_fp12_op(curve.curve_id, 0, vp(want), vp(per_pair[i * w:(i + 1) * w].copy()), vp(nxt), 1)
                want = nxt
            assert out[g * w:(g + 1) * w].tolist() == want.tolist(), (nf, g)
        if nf == 2:   # one group against the oracle: e(rho_0 A_0, B_0) e(rho_1 A_1, B_1) = o(.)^k o(.)^k
            fe = np.zeros(w, dtype=np.uint32)
            pair.ht_fp12_op(curve.curve_id, 8, vp(out[:w].copy()), None, vp(fe), 1)
            E, k = engine(curve), pairing_k(curve)
            assert gt_to_oracle(curve, fe)[0] == (E.pairing(rA[0], B[0]) * E.pairing(rA[1], B[1])).pow(k)


class SimKey:
    """A verifying key with known logs and proofs made without a prover, on the CPU (as tests/test_gpu_verify.py's Sim):
    c = (a b - alpha beta - gamma (g_0 + sum_j x_j g_j)) / delta."""

    def __init__(self, curve, rng, ni):
        self.curve, self.ni = curve, ni
        r = curve.r
        self.G1, self.G2 = groups(curve)
        self.al, self.bt, self.gm, self.dl = [rng.randrange(1, r) for _ in range(4)]
        self.g = [rng.randrange(1, r) for _ in range(ni + 1)]
        G1, G2 = self.G1, self.G2
        self.vk = np.concatenate([pack_points(curve, 1, [G1.mul(G1.gen, self.al)]),
                                  pack_points(curve, 2, [G2.mul(G2.gen, k) for k in (self.bt, self.gm, self.dl)])])
        self.abc = pack_points(curve, 1, [G1.mul(G1.gen, k) for k in self.g])

    def ic(self, x):
        return (self.g[0] + sum(v * gj for v, gj in zip(x, self.g[1:]))) % self.curve.r

    def proof(self, rng, x):
        r = self.curve.r
        a, b = rng.randrange(1, r), rng.randrange(1, r)
        return [a, b, (a * b - self.al * self.bt - self.gm * self.ic(x)) * pow(self.dl, -1, r) % r]


def per_proof_and(pair, sim, xs, logs):
    """AND of the per-proof verdicts (ht_groth16_verdict), from the discrete logs of A, B, C"""
    c, G1, G2 = sim.curve, sim.G1, sim.G2
    pt = lambda G, k: G.mul(G.gen, k) if k else None
    ic = pack_points(c, 1, [pt(G1, sim.ic(x)) for x in xs])
    a = pack_points(c, 1, [pt(G1, l[0]) for l in logs])
    b = pack_points(c, 2, [pt(G2, l[1]) for l in logs])
    cc = pack_points(c, 1, [pt(G1, l[2]) for l in logs])
    ok = np.zeros(len(logs), dtype=np.uint8)
    pair.ht_groth16_verdict(c.curve_id, vp(sim.vk), vp(ic), vp(a), vp(b), vp(cc), vp(ok), len(logs))
    return bool(ok.all()), (a, b, cc)


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_rlc_verdict(rlc, pair, curve):
    """Simulated batches of 1 to 8 proofs, valid and with one tampered proof: the RLC verdict equals the AND of the
    per-proof verdicts."""
    rng = random.Random(0x5B7 + curve.curve_id)
    r = curve.r
    seen = set()
    for case, (n, ni, nf) in enumerate([(1, 0, 1), (2, 1, 2), (3, 2, 4), (5, 0, 2), (8, 1, 2), (8, 3, 4)]):
        sim = SimKey(curve, rng, ni)
        xs = [[rng.randrange(r) for _ in range(ni)] for _ in range(n)]
        logs = [sim.proof(rng, x) for x in xs]
        for tamper in (None, "a", "b", "c", "x", "a_inf"):
            if tamper == "x" and ni == 0:
                continue
            tx, tl = [list(x) for x in xs], [list(l) for l in logs]
            i = rng.randrange(n)
            if tamper == "a":
                tl[i][0] = (tl[i][0] + 1) % r
            elif tamper == "b":
                tl[i][1] = (tl[i][1] + 1) % r
            elif tamper == "c":
                tl[i][2] = (-tl[i][2]) % r
            elif tamper == "x":
                tx[i][0] = (tx[i][0] + 1) % r
            elif tamper == "a_inf":
                tl[i][0] = 0
            want, (a, b, c) = per_proof_and(pair, sim, tx, tl)
            assert want == (tamper is None), (case, tamper)
            rho = [rng.randrange(1, 1 << 128) for _ in range(n)]
            inputs = pack_fr(curve, [v for x in tx for v in x]) if ni else None
            got = rlc.ht_rlc_verdict(curve.curve_id, nf, vp(sim.vk), vp(sim.abc), vp(inputs), ni, vp(a), vp(b), vp(c),
                                     vp(rho_words(rho)), n)
            assert bool(got) == want, (case, n, ni, nf, tamper)
            seen.add(want)
    assert seen == {True, False}


@pytest.mark.parametrize("curve", CURVES, ids=IDS)
def test_rlc_uses_rho(rlc, curve):
    """C_1 + D and C_2 - D cancel in the sum of the C terms only when rho_1 = rho_2: all-ones rho accepts the pair of
    invalid proofs, random rho rejects it."""
    rng = random.Random(0xD0 + curve.curve_id)
    r = curve.r
    sim = SimKey(curve, rng, 1)
    xs = [[rng.randrange(r)] for _ in range(2)]
    logs = [sim.proof(rng, x) for x in xs]
    d = rng.randrange(1, r)
    logs[0][2], logs[1][2] = (logs[0][2] + d) % r, (logs[1][2] - d) % r
    G1, G2 = sim.G1, sim.G2
    a = pack_points(curve, 1, [G1.mul(G1.gen, l[0]) for l in logs])
    b = pack_points(curve, 2, [G2.mul(G2.gen, l[1]) for l in logs])
    c = pack_points(curve, 1, [G1.mul(G1.gen, l[2]) for l in logs])
    inputs = pack_fr(curve, [v for x in xs for v in x])
    run = lambda rho: rlc.ht_rlc_verdict(curve.curve_id, 2, vp(sim.vk), vp(sim.abc), vp(inputs), 1, vp(a), vp(b), vp(c),
                                         vp(rho_words(rho)), 2)
    assert run([1, 1]) == 1
    assert run([rng.randrange(2, 1 << 128), rng.randrange(2, 1 << 128)]) == 0
