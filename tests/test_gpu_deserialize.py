"""CanonicalDeserialize on the GPU (b2s_deserialize_g1/g2, b2s_proof_deserialize, b2s_vk_deserialize, b2s_pk_deserialize)
against the oracle (tests/wire_oracle.py) and against the library's own serializers, on both curves."""
import random

import numpy as np
import pytest

from oracle import groth16 as og
from oracle import r1cs as orc
from tests import wire_oracle as oser
from oracle.ec import groups
from oracle.params import BLS12_381, BN254
from tests.util import csr_from_rows, make_pk_desc, pack_fr, pack_points, unpack_points

pytestmark = pytest.mark.gpu
CURVES = [BLS12_381, BN254]
CH = 1 << 18   # points per streamed chunk (csrc/deserialize.cu)


@pytest.fixture(scope="module", params=[0, 1], ids=["bls12_381", "bn254"])
def be(request):
    from snark_b200 import Backend

    b = Backend(curve=request.param)
    yield b
    b.close()


def invalid_data(be, fn, *args, **kw):
    from snark_b200 import B2SError

    with pytest.raises(B2SError) as e:
        fn(*args, **kw)
    assert e.value.code == 21, str(e.value)   # B2S_ERR_INVALID_DATA
    return str(e.value)


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
def test_points_across_chunks(be, compressed):
    """More than one chunk of points made on the GPU: decoding inverts the serializer bit for bit, a sample agrees with
    the oracle, and one bad point in the second chunk is reported by its index."""
    curve = CURVES[be.curve]
    rng = np.random.default_rng(7)
    for group in (1, 2):
        n = CH + 1000 if group == 1 else CH + 16
        scalars = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
        scalars[:, 7] &= 0x0FFFFFFF
        pts = be.fixed_base(group, scalars.reshape(-1), n, mont=False)
        per_pt = len(pts) // n
        pts[:per_pt] = 0                        # infinity at index 0
        blob = be.serialize_points(group, pts, n, compressed)
        got = be.deserialize_points(group, blob, n, compressed, validate=True)
        assert np.array_equal(got, pts)
        per = len(blob) // n
        for i in [0, 1, CH - 1, CH, n - 1] + [int(x) for x in rng.integers(0, n, 40)]:
            exp = oser.point_deserialize(curve, group, blob[i * per:(i + 1) * per], compressed, True)
            assert unpack_points(curve, group, got[i * per_pt:(i + 1) * per_pt])[0] == exp, (group, i)
        bad_at = CH + 7
        bad = bytearray(blob)
        bad[bad_at * per + (0 if curve is BLS12_381 else per - 1)] ^= 0x80 if curve is BLS12_381 else 0xC0
        bad[(bad_at + 3) * per + (0 if curve is BLS12_381 else per - 1)] ^= 0x80 if curve is BLS12_381 else 0xC0
        msg = invalid_data(be, be.deserialize_points, group, bytes(bad), n, compressed, True)
        assert f"g{group}[{bad_at}]: bad flags" in msg or f"g{group}[{bad_at}]" in msg, msg
        # exact lengths
        invalid_data(be, be.deserialize_points, group, blob[:-1], n, compressed, True)
        invalid_data(be, be.deserialize_points, group, blob + b"\0", n, compressed, True)


def test_validate_switch(be):
    """On-curve points outside the prime-order subgroup: accepted with validate = 0, rejected with validate = 1."""
    curve = CURVES[be.curve]
    rng = random.Random(41)
    for group in (1, 2):
        off = oser.points_outside_subgroup(curve, group, rng, 12)
        if not off:
            continue
        for compressed in (True, False):
            enc = oser.point_compressed if compressed else oser.point_uncompressed
            blob = b"".join(enc(curve, group, P) for P in off)
            got = be.deserialize_points(group, blob, len(off), compressed, validate=False)
            assert unpack_points(curve, group, got) == off
            msg = invalid_data(be, be.deserialize_points, group, blob, len(off), compressed, True)
            assert f"g{group}[0]: not in the prime-order subgroup" in msg, msg


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
def test_proof_and_vk_invert_the_serializers(be, compressed):
    curve = CURVES[be.curve]
    G1, G2 = groups(curve)
    rng = random.Random(43)
    A, B, C = G1.mul(G1.gen, 5), G2.mul(G2.gen, rng.randrange(curve.r)), None
    blob = be.proof_bytes(pack_points(curve, 1, [A]), pack_points(curve, 2, [B]), pack_points(curve, 1, [C]), compressed)
    a, b, c = be.proof_from_bytes(blob, compressed)
    assert (unpack_points(curve, 1, a)[0], unpack_points(curve, 2, b)[0], unpack_points(curve, 1, c)[0]) == (A, B, C)
    invalid_data(be, be.proof_from_bytes, blob[:-1], compressed)
    vk = {"alpha_g1": G1.mul(G1.gen, 3), "beta_g2": G2.mul(G2.gen, 4), "gamma_g2": G2.mul(G2.gen, 5), "delta_g2": G2.neg(G2.gen),
          "gamma_abc_g1": [G1.mul(G1.gen, rng.randrange(curve.r)) for _ in range(5)] + [None]}
    vkb = oser.verifying_key_bytes(curve, vk, compressed)
    got, used = be.vk_from_bytes(vkb + b"trailing pk bytes", compressed)
    assert used == len(vkb)
    assert {k: unpack_points(curve, 1 if k.endswith("g1") else 2, v) for k, v in got.items()} == {
        k: (v if isinstance(v, list) else [v]) for k, v in vk.items()}
    huge = bytearray(vkb)
    at = len(vkb) - 8 - 6 * len(oser.point_compressed(curve, 1, None)) * (1 if compressed else 2)
    huge[at:at + 8] = (2 ** 64 - 1).to_bytes(8, "little")
    assert "gamma_abc_g1" in invalid_data(be, be.vk_from_bytes, bytes(huge), compressed)


def gpu_key(be, curve, n_rows, n_wit, rng):
    """a key from b2s_groth16_setup over a dummy circuit: (m handle, pk handle, vk dict, z_inst, z_wit, csr)"""
    from tests.test_gpu_fullsize import dummy_csr

    a, b = rng.randrange(1, curve.r), rng.randrange(1, curve.r)
    csr, z_inst, z_wit = dummy_csr(curve, n_rows, a, b, n_wit)
    m = be.r1cs_upload(n_rows, 2, n_wit, csr)
    td = pack_fr(curve, [rng.randrange(1, curve.r) for _ in range(5)])
    pk, vk = be.groth16_setup(m, td, 2)
    return m, pk, vk, z_inst, z_wit, csr


def key_bytes(be, pk, vk, n_inst, compressed):
    vkb = be.vk_bytes(vk["alpha_g1"], vk["beta_g2"], vk["gamma_g2"], vk["delta_g2"], vk["gamma_abc_g1"], n_inst, compressed)
    return be.pk_bytes(pk, vkb, compressed)


def same_key(be, pk0, pk1, n_vars, n_wit, domain):
    counts = [n_vars, n_vars, n_vars, domain - 1, n_wit, 3, 2]
    for which, n in enumerate(counts):
        assert np.array_equal(be.pk_query(pk0, which, n), be.pk_query(pk1, which, n)), which


@pytest.mark.parametrize("compressed", [True, False], ids=["compressed", "uncompressed"])
def test_gpu_key_round_trip_and_proof(be, compressed, monkeypatch):
    """Key from b2s_groth16_setup -> b2s_pk_serialize -> b2s_pk_deserialize: all seven vectors identical (with the appended
    delta pairs) and the same proof for the same z, r, s; once more with the h-query table forced on."""
    curve = CURVES[be.curve]
    rng = random.Random(47)
    n_rows, n_wit = 1000, 40
    m, pk, vk, z_inst, z_wit, _ = gpu_key(be, curve, n_rows, n_wit, rng)
    domain = be.domain_size(m)
    blob = key_bytes(be, pk, vk, 2, compressed)
    r, s = pack_fr(curve, [rng.randrange(curve.r)]), pack_fr(curve, [rng.randrange(curve.r)])
    for precomp in (False, True):
        if precomp:
            monkeypatch.setenv("B2S_PK_PRECOMP_MIN", "1")
            monkeypatch.setenv("B2S_MSM_PRE_C", "7")
        loaded = be.pk_from_bytes(blob, compressed, validate=True)
        same_key(be, pk, loaded, 2 + n_wit, n_wit, domain)
        p0 = be.groth16_prove(pk, m, z_inst, z_wit, r, s)
        p1 = be.groth16_prove(loaded, m, z_inst, z_wit, r, s)
        assert all(np.array_equal(x, y) for x, y in zip(p0, p1)), precomp
        be.pk_free(loaded)
    # validate = 0 loads the same key
    loaded = be.pk_from_bytes(blob, compressed, validate=False)
    same_key(be, pk, loaded, 2 + n_wit, n_wit, domain)
    be.pk_free(loaded)
    be.pk_free(pk)
    be.r1cs_free(m)


def test_oracle_key_loads_and_proves(be):
    curve = CURVES[be.curve]
    rng = random.Random(53)
    bc = orc.bench_circuit(curve, 25, seed=5)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    pk = og.setup(curve, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)]))
    m = be.r1cs_upload(len(mats[0]), len(inst), len(wit), [csr_from_rows(curve, M) for M in mats])
    for compressed in (True, False):
        pkh = be.pk_from_bytes(oser.proving_key_bytes(curve, pk, compressed), compressed)
        keep = []
        ref = be.pk_upload(make_pk_desc(curve, pk, keep))
        same_key(be, ref, pkh, len(inst) + len(wit), len(wit), pk.domain)
        rr, ss = rng.randrange(curve.r), rng.randrange(curve.r)
        a, b, c = be.groth16_prove(pkh, m, pack_fr(curve, inst), pack_fr(curve, wit), pack_fr(curve, [rr]), pack_fr(curve, [ss]))
        proof = (unpack_points(curve, 1, a)[0], unpack_points(curve, 2, b)[0], unpack_points(curve, 1, c)[0])
        h = og.witness_map(curve, mats, list(inst) + list(wit), len(inst))
        assert og.check_in_exponent(pk, proof, inst, wit, h, rr, ss)
        be.pk_free(pkh)
        be.pk_free(ref)
    be.r1cs_free(m)


def test_rejected_keys(be):
    """An off-subgroup h_query point is named by its index; an oversized Vec prefix fails before any allocation; bad
    dimensions are MALFORMED_VK."""
    from snark_b200 import B2SError

    curve = CURVES[be.curve]
    rng = random.Random(59)
    bc = orc.bench_circuit(curve, 25, seed=5)
    bc.finalize()
    mats, inst, wit = bc.to_matrices(), bc.instance_assignment, bc.witness_assignment
    pk = og.setup(curve, mats, len(inst), len(wit), og.Trapdoor(*[rng.randrange(1, curve.r) for _ in range(5)]))
    off = oser.points_outside_subgroup(curve, 1, rng, 1)
    if off:
        i = len(pk.h_query) // 2
        pk.h_query[i] = off[0]
        blob = oser.proving_key_bytes(curve, pk, True)
        msg = invalid_data(be, be.pk_from_bytes, blob, True, True)
        assert f"h_query[{i}]: not in the prime-order subgroup" in msg, msg
        be.pk_free(be.pk_from_bytes(blob, True, False))   # accepted without validation
        pk.h_query[i] = groups(curve)[0].gen
    blob = oser.proving_key_bytes(curve, pk, True)
    g1 = len(oser.point_compressed(curve, 1, None))
    at = len(blob) - 8 - g1 * len(pk.l_query)            # the l_query prefix
    huge = bytearray(blob)
    huge[at:at + 8] = (2 ** 64 - 1).to_bytes(8, "little")
    assert "l_query: length" in invalid_data(be, be.pk_from_bytes, bytes(huge), True)
    invalid_data(be, be.pk_from_bytes, blob[:-1], True)
    invalid_data(be, be.pk_from_bytes, blob + b"\0", True)
    pk.l_query = pk.l_query[:-1]                         # |a| != n_instance + n_witness
    with pytest.raises(B2SError) as e:
        be.pk_from_bytes(oser.proving_key_bytes(curve, pk, True), True)
    assert e.value.code == 7


def test_round_trip_2p20(be):
    """One key at domain 2^20 through both forms."""
    rng = random.Random(61)
    curve = CURVES[be.curve]
    n_rows, n_wit = (1 << 20) - 8, 64
    m, pk, vk, _, _, _ = gpu_key(be, curve, n_rows, n_wit, rng)
    domain = be.domain_size(m)
    assert domain == 1 << 20
    for compressed in (True, False):
        loaded = be.pk_from_bytes(key_bytes(be, pk, vk, 2, compressed), compressed)
        same_key(be, pk, loaded, 2 + n_wit, n_wit, domain)
        be.pk_free(loaded)
    be.pk_free(pk)
    be.r1cs_free(m)
