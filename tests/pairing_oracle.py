"""Helpers shared by the pairing tests: GT elements between the kernels' tower layout and the oracle's Fq12
(oracle/pairing.py), and the exponent k with e(P, Q) = oracle(P, Q)^k, recomputed from the formulas stated in
snark_b200/csrc/pairing.cuh."""
import numpy as np

from oracle.pairing import engine
from oracle.params import BLS12_381, BN254
from tests.util import fq_limbs, pack_u32, unpack_u32

BLS_X = -0xD201000000010000
BN_X = 4965661367192848881
XI0 = {BLS12_381.name: 1, BN254.name: 9}
# coefficient of w^k at position k of the ark layout (c0.c0, c0.c1, c0.c2, c1.c0, c1.c1, c1.c2)
W_POWERS = [0, 2, 4, 1, 3, 5]


def gt_to_oracle(curve, arr):
    """uint32 limbs of `count` Fq12 elements (ark layout, Montgomery) -> list of oracle Fq12.  Each Fq2 coefficient a + bu
    of w^k sits in the oracle's basis as (a - xi0 b) w^k + b w^(k+6), because w^6 = xi0 + u."""
    n, p, c = fq_limbs(curve), curve.p, XI0[curve.name]
    rinv = pow(1 << (32 * n), -1, p)
    vals = [v * rinv % p for v in unpack_u32(arr, n)]
    E = engine(curve)
    out = []
    for e in range(len(vals) // 12):
        v = vals[12 * e: 12 * e + 12]
        co = [0] * 12
        for slot, k in enumerate(W_POWERS):
            a, b = v[2 * slot], v[2 * slot + 1]
            co[k] = (co[k] + a - c * b) % p
            co[k + 6] = (co[k + 6] + b) % p
        out.append(E.Fq12(co))
    return out


def gt_from_oracle(curve, elems):
    """oracle Fq12 elements -> uint32 limbs in the ark layout (Montgomery)"""
    n, p, c = fq_limbs(curve), curve.p, XI0[curve.name]
    R = 1 << (32 * n)
    flat = []
    for e in elems:
        for k in W_POWERS:
            b = e.c[k + 6]
            a = (e.c[k] + c * b) % p
            flat += [a * R % p, b * R % p]
    return pack_u32(flat, n)


def pairing_k(curve):
    """k with e = oracle^k mod r, from the derivation in pairing.cuh"""
    r, p = curve.r, curve.p
    if curve is BLS12_381:
        return (-3) % r                                  # conjugated |x| loop, hard part times 3
    x = BN_X
    T = 6 * x * x
    assert p - T == r
    n = (6 * x + 2 + p - p * p + p ** 3) // r
    M = (T ** 12 - 1) // r
    c = sum(T ** (11 - j) * p ** j for j in range(12))
    t = c * pow(M, -1, r) % r                            # [f_{r,Q}(P)] = o^t
    ap = (1 + t) % r                                     # [f_{p,Q}(P)] = o^ap
    e_opt = (t * n - ap * (1 - 2 * p + 3 * p * p)) % r
    return e_opt * 2 * x * (6 * x * x + 3 * x + 1) % r


K_STATED = {BLS12_381.name: BLS12_381.r - 3, BN254.name: 147946756881789319005730692170996259610}


def random_gt_raw(curve, rng, count):
    """`count` uniformly random Fq12 elements (not in GT) as limbs"""
    n, p = fq_limbs(curve), curve.p
    R = 1 << (32 * n)
    return pack_u32([rng.randrange(p) * R % p for _ in range(12 * count)], n)


def gt_bytes(curve):
    return 12 * fq_limbs(curve) * 4


def as_u32(a):
    return np.ascontiguousarray(a, dtype=np.uint32)
