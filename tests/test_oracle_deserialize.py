"""The oracle's CanonicalDeserialize (tests/wire_oracle.py): round trips of points, proofs, verifying and proving keys in
both forms and both validate modes, and every rejection class the GPU decoder is held to."""
import random

import pytest

from oracle import groth16 as og
from oracle import r1cs as orc
from tests import wire_oracle as oser
from oracle.ec import groups
from oracle.params import BLS12_381, BN254

CURVES = [BLS12_381, BN254]
IDS = ["bls12_381", "bn254"]


def enc(curve, group, P, compressed):
    return (oser.point_compressed if compressed else oser.point_uncompressed)(curve, group, P)


@pytest.fixture(scope="module", params=[0, 1], ids=IDS)
def curve(request):
    return CURVES[request.param]


@pytest.fixture(scope="module")
def small_pk(curve):
    rng = random.Random(71)
    bc = orc.bench_circuit(curve, 12, seed=4)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    return og.setup(curve, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)]))


@pytest.mark.parametrize("compressed", [True, False])
@pytest.mark.parametrize("validate", [True, False])
def test_point_round_trips(curve, compressed, validate):
    rng = random.Random(73)
    for group in (1, 2):
        G = groups(curve)[group - 1]
        P = G.mul(G.gen, rng.randrange(1, curve.r))
        for Q in (G.gen, P, G.neg(P), None):
            assert oser.point_deserialize(curve, group, enc(curve, group, Q, compressed), compressed, validate) == Q


@pytest.mark.parametrize("compressed", [True, False])
@pytest.mark.parametrize("validate", [True, False])
def test_proof_vk_pk_round_trips(curve, small_pk, compressed, validate):
    G1, G2 = groups(curve)
    A, B, C = G1.mul(G1.gen, 9), G2.mul(G2.gen, 10), None
    blob = enc(curve, 1, A, compressed) + enc(curve, 2, B, compressed) + enc(curve, 1, C, compressed)
    assert oser.proof_from_bytes(curve, blob, compressed, validate) == (A, B, C)
    pk = small_pk
    vk = {"alpha_g1": pk.alpha_g1, "beta_g2": pk.beta_g2, "gamma_g2": pk.gamma_g2, "delta_g2": pk.delta_g2, "gamma_abc_g1": pk.gamma_abc_g1}
    assert oser.verifying_key_from_bytes(curve, oser.verifying_key_bytes(curve, vk, compressed), compressed, validate) == vk
    got = oser.proving_key_from_bytes(curve, oser.proving_key_bytes(curve, pk, compressed), compressed, validate)
    for f in ("alpha_g1", "beta_g1", "beta_g2", "delta_g1", "delta_g2", "gamma_g2", "gamma_abc_g1", "a_query", "b_g1_query",
              "b_g2_query", "h_query", "l_query", "domain", "num_instance"):
        assert getattr(got, f) == getattr(pk, f), f


def test_rejections(curve):
    rng = random.Random(79)
    fq = 48 if curve is BLS12_381 else 32
    bls = curve is BLS12_381
    for group in (1, 2):
        G = groups(curve)[group - 1]
        P = G.mul(G.gen, rng.randrange(1, curve.r))
        for compressed in (True, False):
            good, inf = enc(curve, group, P, compressed), enc(curve, group, None, compressed)
            n = len(good)

            def rejects(blob, reason, validate=True):
                with pytest.raises(ValueError) as e:
                    oser.point_deserialize(curve, group, blob, compressed, validate)
                assert str(e.value).startswith(reason), (str(e.value), reason)

            flag_at = 0 if bls else n - 1
            bad_flags = [inf[:n - 1] + bytes([inf[-1] | 1])]
            if bls:
                bad_flags += [bytes([good[0] ^ 0x80]) + good[1:], bytes([inf[0] | 0x20]) + inf[1:], bytes([good[0] | 0x40]) + good[1:]]
                if not compressed:
                    bad_flags += [bytes([good[0] | 0x20]) + good[1:]]
            else:
                bad_flags += [good[:flag_at] + bytes([good[flag_at] | 0xC0]) + good[flag_at + 1:]]
            for b in bad_flags:
                rejects(b, oser.REASON_FLAGS)
            # x >= p in either Fq2 component
            pb = curve.p.to_bytes(fq, "big" if bls else "little")
            for comp in range(group):
                b = bytearray(good)
                b[comp * fq:(comp + 1) * fq] = pb
                if bls and comp == 0:
                    b[0] |= good[0] & 0xE0
                if not bls and compressed and comp == group - 1:
                    b[(comp + 1) * fq - 1] |= good[(comp + 1) * fq - 1] & 0xC0
                rejects(bytes(b), oser.REASON_NONCANONICAL)
            # not on the curve
            if not compressed:
                f = G.f
                rejects(enc(curve, group, (P[0], f.add(P[1], f.one)), False), oser.REASON_NOT_ON_CURVE)
                assert oser.point_deserialize(curve, group, enc(curve, group, (P[0], f.add(P[1], f.one)), False), False, False)
            else:
                while True:
                    x = rng.randrange(curve.p) if group == 1 else (rng.randrange(curve.p), rng.randrange(curve.p))
                    try:
                        oser.point_deserialize(curve, group, enc(curve, group, (x, P[1]), True), True, False)
                    except ValueError as e:
                        assert str(e) == oser.REASON_NOT_ON_CURVE
                        break
            # short / long
            for blob in (good[:-1], good + b"\0", b""):
                rejects(blob, "length")


def test_off_subgroup_points(curve):
    rng = random.Random(83)
    for group in (1, 2):
        off = oser.points_outside_subgroup(curve, group, rng, 6)
        assert (off == []) == (curve is BN254 and group == 1)
        for P in off:
            assert groups(curve)[group - 1].on_curve(P)
            for compressed in (True, False):
                blob = enc(curve, group, P, compressed)
                assert oser.point_deserialize(curve, group, blob, compressed, False) == P
                with pytest.raises(ValueError, match=oser.REASON_NOT_IN_SUBGROUP):
                    oser.point_deserialize(curve, group, blob, compressed, True)


def test_key_framing_rejections(curve, small_pk):
    pk = small_pk
    blob = oser.proving_key_bytes(curve, pk, True)
    g1 = len(oser.point_compressed(curve, 1, None))
    for bad in (blob[:-1], blob + b"\0", blob[:len(blob) // 2]):
        with pytest.raises(ValueError, match="length"):
            oser.proving_key_from_bytes(curve, bad, True)
    at = len(blob) - 8 - g1 * len(pk.l_query)
    huge = blob[:at] + (2 ** 64 - 1).to_bytes(8, "little") + blob[at + 8:]
    with pytest.raises(ValueError, match="Vec prefix"):
        oser.proving_key_from_bytes(curve, huge, True)
    import copy
    short = copy.copy(pk)
    short.l_query = pk.l_query[:-1]
    with pytest.raises(ValueError, match="dimensions"):
        oser.proving_key_from_bytes(curve, oser.proving_key_bytes(curve, short, True), True)
    short = copy.copy(pk)
    short.h_query = pk.h_query[:-1]
    with pytest.raises(ValueError, match="dimensions"):
        oser.proving_key_from_bytes(curve, oser.proving_key_bytes(curve, short, True), True)
