"""CanonicalDeserialize for the CPU oracle: points, Proof, VerifyingKey and ProvingKey in both forms, with and without
validation -- the inverse of the encoders in oracle/serialize.py, against which the GPU decoder
(snark_b200/csrc/deserialize.cuh) is checked.  TEST INFRASTRUCTURE ONLY.

The decoding rules (flag combinations, canonicity, validation) are recalled from ark-serialize / ark-ec /
ark-bls12-381 / ark-bn254 (crates not in the reference tree) and unpinned against bytes written by a Rust build; they
are stated above `point_deserialize`.  The subgroup check is the definition r * P = O, independent of the endomorphism
criteria the GPU uses.  The encoders are re-exported so that tests can use one module for both directions.
"""
from oracle.params import Curve
from oracle.serialize import (_larger, _sqrt_fq, _sqrt_fq2, point_compressed, point_uncompressed,  # noqa: F401
                              proof_compressed, proving_key_bytes, vec_framed, verifying_key_bytes)


# ---------------------------------------------------------------------------------------------
# CanonicalDeserialize: both forms, with or without validation
# ---------------------------------------------------------------------------------------------
# Encoding rules (recalled, not pinned against bytes written by a Rust build; snark_b200/csrc/deserialize.cuh states the same):
#   BLS12-381, byte 0 of the encoding: 0x80 compressed, 0x40 infinity, 0x20 y is the larger root.  Compressed: 0x80 set.
#     Uncompressed: 0x80 and 0x20 clear.  Infinity: 0x20 clear and every other bit and byte zero.
#   BN254, last byte (of x when compressed, of y when not): 0x80 y is the larger root, 0x40 infinity; 0xC0 is rejected.
#     Infinity: every other bit and byte zero.  Uncompressed points ignore the sign bit.
#   Every coordinate must be below p.  A compressed x without a square root x^3 + b is invalid in both validate modes;
#   with validate (ark's Validate::Yes) an uncompressed point must satisfy the curve equation, and every point must lie
#   in the prime-order subgroup, here tested by the definition r * P = O.
REASON_FLAGS, REASON_NONCANONICAL, REASON_NOT_ON_CURVE, REASON_NOT_IN_SUBGROUP = (
    "bad flags", "coordinate not below p", "not on the curve", "not in the prime-order subgroup")


def _groups(curve: Curve):
    from oracle.ec import groups
    return groups(curve)


def mul_unreduced(G, P, k: int):
    """k * P without reducing k modulo the group order (Group.mul reduces it), so that r * P is O only in the subgroup."""
    acc = G.to_jac(None)
    J = G.to_jac(P)
    for bit in bin(k)[2:] if k > 0 else "":
        acc = G.jdbl(acc)
        if bit == "1":
            acc = G.jadd(acc, J)
    return G.to_affine(acc)


def in_prime_subgroup(curve: Curve, group: int, P) -> bool:
    G = _groups(curve)[group - 1]
    return mul_unreduced(G, P, curve.r) is None


def point_deserialize(curve: Curve, group: int, data: bytes, compressed=True, validate=True):
    """Inverse of `point_compressed` / `point_uncompressed`.  Raises ValueError with one of the REASON_* texts (or
    "length")."""
    p = curve.p
    fq = 48 if curve.name == "bls12_381" else 32
    coord = fq * group
    if len(data) != coord * (1 if compressed else 2):
        raise ValueError("length")
    data = bytearray(data)
    if curve.name == "bls12_381":
        flags = data[0] & 0xE0
        data[0] &= 0x1F
        if bool(flags & 0x80) != compressed or (not compressed and flags & 0x20):
            raise ValueError(REASON_FLAGS)
        if flags & 0x40:
            if flags & 0x20 or any(data):
                raise ValueError(REASON_FLAGS)
            return None
        larger = bool(flags & 0x20)
        order = "big"
    else:
        at = coord - 1 if compressed else 2 * coord - 1
        flags = data[at] & 0xC0
        data[at] &= 0x3F
        if flags == 0xC0:
            raise ValueError(REASON_FLAGS)
        if flags & 0x40:
            if any(data):
                raise ValueError(REASON_FLAGS)
            return None
        larger = bool(flags & 0x80)
        order = "little"

    def coordinate(body):
        if group == 1:
            return (int.from_bytes(body, order),)
        lo, hi = int.from_bytes(body[:fq], order), int.from_bytes(body[fq:], order)
        return (hi, lo) if curve.name == "bls12_381" else (lo, hi)   # (c0, c1)

    def canonical(v):
        if any(c >= p for c in v):
            raise ValueError(REASON_NONCANONICAL)
        return v[0] if group == 1 else v

    x = canonical(coordinate(bytes(data[:coord])))
    G = _groups(curve)[group - 1]
    f = G.f
    rhs = f.add(f.mul(f.sqr(x), x), G.b)
    if compressed:
        y = _sqrt_fq(p, rhs) if group == 1 else _sqrt_fq2(p, rhs)
        if y is None:
            raise ValueError(REASON_NOT_ON_CURVE)
        if _larger(curve, y) != larger:
            y = f.neg(y)
    else:
        y = canonical(coordinate(bytes(data[coord:])))
        if validate and f.sqr(y) != rhs:
            raise ValueError(REASON_NOT_ON_CURVE)
    P = (x, y)
    if validate and not in_prime_subgroup(curve, group, P):
        raise ValueError(REASON_NOT_IN_SUBGROUP)
    return P


def _point_len(curve: Curve, group: int, compressed: bool) -> int:
    return (48 if curve.name == "bls12_381" else 32) * group * (1 if compressed else 2)


class _Reader:
    """Walks a byte string; every Vec length prefix is checked against the bytes that remain before any element is read."""

    def __init__(self, curve, data, compressed, validate):
        self.curve, self.data, self.compressed, self.validate, self.at = curve, bytes(data), compressed, validate, 0

    def point(self, group):
        n = _point_len(self.curve, group, self.compressed)
        if self.at + n > len(self.data):
            raise ValueError("length")
        P = point_deserialize(self.curve, group, self.data[self.at:self.at + n], self.compressed, self.validate)
        self.at += n
        return P

    def vec(self, group):
        if self.at + 8 > len(self.data):
            raise ValueError("length")
        n = int.from_bytes(self.data[self.at:self.at + 8], "little")
        self.at += 8
        if n > (len(self.data) - self.at) // _point_len(self.curve, group, self.compressed):
            raise ValueError("length: Vec prefix exceeds the remaining bytes")
        return [self.point(group) for _ in range(n)]

    def vk(self):
        return {"alpha_g1": self.point(1), "beta_g2": self.point(2), "gamma_g2": self.point(2), "delta_g2": self.point(2),
                "gamma_abc_g1": self.vec(1)}

    def end(self):
        if self.at != len(self.data):
            raise ValueError("length: trailing bytes")


def verifying_key_from_bytes(curve: Curve, data: bytes, compressed=True, validate=True):
    """Inverse of `verifying_key_bytes` (the whole of `data`)."""
    rd = _Reader(curve, data, compressed, validate)
    vk = rd.vk()
    rd.end()
    return vk


def proof_from_bytes(curve: Curve, data: bytes, compressed=True, validate=True):
    rd = _Reader(curve, data, compressed, validate)
    out = (rd.point(1), rd.point(2), rd.point(1))
    rd.end()
    return out


def proving_key_from_bytes(curve: Curve, data: bytes, compressed=True, validate=True):
    """Inverse of `proving_key_bytes` -> oracle.groth16.ProvingKey (no trapdoor).  The dimensions follow from the bytes:
    n_instance = |gamma_abc_g1|, n_witness = |l_query|, domain = |h_query| + 1 (a power of two), and
    |a_query| = |b_g1_query| = |b_g2_query| = n_instance + n_witness; anything else raises ValueError("dimensions")."""
    from oracle.groth16 import ProvingKey

    rd = _Reader(curve, data, compressed, validate)
    vk = rd.vk()
    beta_g1, delta_g1 = rd.point(1), rd.point(1)
    a, b1, b2, h, l_q = rd.vec(1), rd.vec(1), rd.vec(2), rd.vec(1), rd.vec(1)
    rd.end()
    n_inst, n_vars, domain = len(vk["gamma_abc_g1"]), len(vk["gamma_abc_g1"]) + len(l_q), len(h) + 1
    if len(a) != n_vars or len(b1) != n_vars or len(b2) != n_vars or domain & (domain - 1):
        raise ValueError("dimensions")
    return ProvingKey(curve=curve, alpha_g1=vk["alpha_g1"], beta_g1=beta_g1, beta_g2=vk["beta_g2"], delta_g1=delta_g1,
                      delta_g2=vk["delta_g2"], gamma_g2=vk["gamma_g2"], gamma_abc_g1=vk["gamma_abc_g1"], a_query=a,
                      b_g1_query=b1, b_g2_query=b2, h_query=h, l_query=l_q, domain=domain, num_instance=n_inst)


# ---- test helper: points on the curve outside the prime-order subgroup ----------------------------------------------
def cofactor(curve: Curve, group: int) -> int:
    """#E / r for G1 (E(Fq)) and G2 (the twist over Fq2)."""
    if curve.name == "bls12_381":
        x = -0xd201000000010000
        if group == 1:
            return (x - 1) ** 2 // 3
        return (x ** 8 - 4 * x ** 7 + 5 * x ** 6 - 4 * x ** 4 + 6 * x ** 3 - 4 * x ** 2 - 4 * x + 13) // 9
    return 1 if group == 1 else 2 * curve.p - curve.r


SMALL_TORSION = {("bls12_381", 1): (3, 11), ("bls12_381", 2): (13, 23)}   # small primes dividing the cofactor


def random_curve_point(curve: Curve, group: int, rng):
    """A uniformly random point of the whole curve group (random x until x^3 + b is a square)."""
    G = _groups(curve)[group - 1]
    f = G.f
    while True:
        x = rng.randrange(curve.p) if group == 1 else (rng.randrange(curve.p), rng.randrange(curve.p))
        rhs = f.add(f.mul(f.sqr(x), x), G.b)
        y = _sqrt_fq(curve.p, rhs) if group == 1 else _sqrt_fq2(curve.p, rhs)
        if y is not None:
            return (x, y if rng.randrange(2) else f.neg(y))


def points_outside_subgroup(curve: Curve, group: int, rng, count: int):
    """`count` on-curve points outside the prime-order subgroup: random-x points and, where the cofactor has small prime
    factors, P + T with P in the subgroup and T of small prime order l (from [r h / l^v] Q, l^v the power of l in h,
    multiplied by l while that leaves it non-zero).  Empty for a cofactor of 1."""
    h = cofactor(curve, group)
    if h == 1:
        return []
    G = _groups(curve)[group - 1]
    small = SMALL_TORSION.get((curve.name, group), ())
    out = []
    while len(out) < count:
        k = len(out) % (len(small) + 1)
        if k == 0:
            P = random_curve_point(curve, group, rng)
        else:
            ell, rest = small[k - 1], h
            while rest % ell == 0:
                rest //= ell
            T = mul_unreduced(G, random_curve_point(curve, group, rng), curve.r * rest)   # in the l-power torsion
            while T is not None and mul_unreduced(G, T, ell) is not None:
                T = mul_unreduced(G, T, ell)
            if T is None:
                continue
            P = G.add(G.mul(G.gen, rng.randrange(1, curve.r)), T)
        if P is not None and not in_prime_subgroup(curve, group, P):
            out.append(P)
    return out
