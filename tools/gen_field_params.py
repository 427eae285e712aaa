#!/usr/bin/env python3
"""Generate snark_b200/csrc/field_params.h (Montgomery constants for the four prime fields and
the curve constants the kernels need).  Developer tool: run once, commit the header.

The numbers are the standard BLS12-381 / BN254 parameters (SURVEY.md Appendix B); the header is
cross-checked against the oracle's independent copy in tests/test_host_ff.py.
"""
import os

BLS_P = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
BLS_R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001
BN_P = 21888242871839275222246405745257275088696311157297823662689037894645226208583
BN_R = 21888242871839275222246405745257275088548364400416034343698204186575808495617

BLS_G1 = (
    0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
    0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1,
)
BLS_G2 = (
    0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
    0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e,
    0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
    0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be,
)
BN_G1 = (1, 2)
BN_G2 = (
    10857046999023057135944570762232829481370756359578518086990519993285655852781,
    11559732032986387107991004021392285783925812861821192530917403151452391805634,
    8495653923123431417604973247489272438418190587263600148770280649306958101930,
    4082367875863433681332203403145435568316851327593401208105741076214120093531,
)


def limbs(x, n):
    return [(x >> (32 * i)) & 0xFFFFFFFF for i in range(n)]


def arr(x, n):
    return "{" + ", ".join("0x%08xu" % w for w in limbs(x, n)) + "}"


def field_struct(name, p, n, extra=""):
    R = 1 << (32 * n)
    ninv = (-pow(p, -1, 1 << 32)) % (1 << 32)
    spare = 32 * n - p.bit_length()
    fn = lambda nm, val: (
        "    B2S_HD static constexpr uint32_t %s(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n"
        % (nm, n, arr(val, n))
    )
    s = "struct %s {\n" % name
    s += "    static constexpr int N = %d;\n" % n
    s += "    static constexpr int BITS = %d;\n" % p.bit_length()
    s += "    static constexpr int SPARE_BITS = %d;\n" % spare
    s += "    static constexpr uint32_t NINV = 0x%08xu;\n" % ninv
    special = (p & ((1 << 64) - 1)) == (1 << 64) - (1 << 32) + 1
    s += "    static constexpr bool LOW64_IS_2_64_MINUS_2_32_PLUS_1 = %s;\n" % ("true" if special else "false")
    s += fn("mod", p)
    s += fn("r1", R % p)
    s += fn("r2", R * R % p)
    s += extra
    s += "};\n\n"
    return s


def fr_extra(r, n, gen, two_adicity):
    R = 1 << (32 * n)
    root = pow(gen, (r - 1) >> two_adicity, r)
    m = lambda x: arr(x * R % r, n)
    fn = lambda nm, val: (
        "    B2S_HD static constexpr uint32_t %s(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n"
        % (nm, n, m(val))
    )
    s = "    static constexpr int TWO_ADICITY = %d;\n" % two_adicity
    s += "    // Montgomery forms of: multiplicative generator g, g^-1, 2^S-th root of unity and its inverse, 2^-1\n"
    s += fn("gen", gen) + fn("gen_inv", pow(gen, -1, r))
    s += fn("root", root) + fn("root_inv", pow(root, -1, r))
    s += fn("half", pow(2, -1, r))
    return s


def curve_extra(p, n, g1, g2, b, b2):
    R = 1 << (32 * n)
    fn = lambda nm, val: (
        "    B2S_HD static constexpr uint32_t %s(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n"
        % (nm, n, arr(val * R % p, n))
    )
    s = "    // Montgomery forms of the standard generators and curve coefficients\n"
    s += fn("g1x", g1[0]) + fn("g1y", g1[1])
    s += fn("g2x0", g2[0]) + fn("g2x1", g2[1]) + fn("g2y0", g2[2]) + fn("g2y1", g2[3])
    s += fn("b1", b) + fn("b2c0", b2[0]) + fn("b2c1", b2[1])
    return s


# ---- point decoding constants (snark_b200/csrc/deserialize.cuh) ----------------------------------------------------
# Subgroup criteria: BLS12-381 G1 phi(P) = -[x^2]P with phi(x, y) = (beta x, y); BLS12-381 G2 psi(P) = [x]P; BN254 G2
# psi(P) = [6 x^2]P, where psi(x, y) = (conj(x) cx, conj(y) cy) is the untwist-Frobenius-twist map.  beta and the psi
# coefficients are chosen here so that the curve's generator satisfies its criterion, so the header cannot carry the
# wrong cube root of unity or the inverse coefficients.
BLS_X_ABS = 0xd201000000010000     # BLS12-381 x = -0xd201000000010000
BN_X = 4965661367192848881          # BN254 x (p = 36x^4 + 36x^3 + 24x^2 + 6x + 1)


def f2_mul(p, a, b):
    return ((a[0] * b[0] - a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)


def f2_pow(p, a, e):
    r = (1, 0)
    for bit in bin(e)[2:]:
        r = f2_mul(p, r, r)
        if bit == "1":
            r = f2_mul(p, r, a)
    return r


def f2_inv(p, a):
    n = pow(a[0] * a[0] + a[1] * a[1], -1, p)
    return (a[0] * n % p, (-a[1]) * n % p)


def ec_mul(p, ext, P, k):
    """k * P on y^2 = x^3 + b (affine, a = 0) over Fq (ext False) or Fq2 (ext True); None = infinity."""
    mul = (lambda a, b: f2_mul(p, a, b)) if ext else (lambda a, b: a * b % p)
    inv = (lambda a: f2_inv(p, a)) if ext else (lambda a: pow(a, -1, p))
    sub = (lambda a, b: ((a[0] - b[0]) % p, (a[1] - b[1]) % p)) if ext else (lambda a, b: (a - b) % p)
    three = (3, 0) if ext else 3
    two = (2, 0) if ext else 2

    def add(A, B):
        if A is None:
            return B
        if B is None:
            return A
        if A[0] == B[0]:
            if A[1] != B[1]:
                return None
            lam = mul(mul(three, mul(A[0], A[0])), inv(mul(two, A[1])))
        else:
            lam = mul(sub(B[1], A[1]), inv(sub(B[0], A[0])))
        x3 = sub(sub(mul(lam, lam), A[0]), B[0])
        return (x3, sub(mul(lam, sub(A[0], x3)), A[1]))

    acc = None
    for bit in bin(k)[2:]:
        acc = add(acc, acc)
        if bit == "1":
            acc = add(acc, P)
    return acc


def bls_beta():
    p, r = BLS_P, BLS_R
    for g in range(2, 100):
        w = pow(g, (p - 1) // 3, p)
        if w != 1:
            break
    lam = (-BLS_X_ABS * BLS_X_ABS) % r
    target = ec_mul(p, False, BLS_G1, lam)
    hits = [b for b in (w, w * w % p) if (b * BLS_G1[0] % p, BLS_G1[1]) == target]
    assert len(hits) == 1
    return hits[0]


def psi_coeffs(p, r, xi, gen, lam):
    """(cx, cy) with psi(gen) = [lam] gen for cx = xi^(e (p-1)/3), cy = xi^(e (p-1)/2), e = +1 or -1."""
    x, y = (gen[0], gen[1]), (gen[2], gen[3])
    target = ec_mul(p, True, (x, y), lam % r)
    hits = []
    for e in (1, -1):
        base = xi if e == 1 else f2_inv(p, xi)
        cx, cy = f2_pow(p, base, (p - 1) // 3), f2_pow(p, base, (p - 1) // 2)
        if (f2_mul(p, (x[0], -x[1] % p), cx), f2_mul(p, (y[0], -y[1] % p), cy)) == target:
            hits.append((cx, cy))
    assert len(hits) == 1
    return hits[0]


def words(x, n):
    return "{" + ", ".join("0x%08xu" % w for w in limbs(x, n)) + "}"


def decode_extra(p, n, beta, psi, endo_scalar, endo_words):
    """Constants of deserialize.cuh: sqrt exponent, 1/2, beta, psi coefficients (Montgomery) and the subgroup scalar (plain)."""
    R = 1 << (32 * n)
    fn = lambda nm, val: (
        "    B2S_HD static constexpr uint32_t %s(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n"
        % (nm, n, arr(val * R % p, n))
    )
    s = "    // point decoding (deserialize.cuh): (p - 3) / 4 in plain words; Montgomery forms of 1/2, the cube root of unity\n"
    s += "    // beta of the G1 endomorphism (1 when unused) and the psi coefficients cx, cy of G2; the subgroup-test scalar in\n"
    s += "    // plain words (BLS12-381: |x|; BN254: 6 x^2)\n"
    s += "    B2S_HD static constexpr uint32_t sqrt_exp(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (n, words((p - 3) // 4, n))
    s += fn("fq_half", pow(2, -1, p)) + fn("beta", beta)
    s += fn("psi_x0", psi[0][0]) + fn("psi_x1", psi[0][1]) + fn("psi_y0", psi[1][0]) + fn("psi_y1", psi[1][1])
    s += "    static constexpr int ENDO_WORDS = %d;\n" % endo_words
    s += "    B2S_HD static constexpr uint32_t endo_scalar(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (
        endo_words, words(endo_scalar, endo_words))
    return s


# ---- pairing constants (snark_b200/csrc/pairing.cuh) ---------------------------------------------------------------
# Fq12 = Fq2[w] / (w^6 - xi) as Fq6 = Fq2[v] / (v^3 - xi), Fq12 = Fq6[w] / (w^2 - v).  The p^j-power Frobenius sends the
# coefficient a_k of w^k to conj^j(a_k) * xi^(k (p^j - 1) / 6).  Each table is checked against a plain polynomial Fq12
# raised to p^j, and the p^1 coefficients of w^2 and w^3 against the psi coefficients (psi is the Frobenius read through
# the twist, so the p^1 coefficients equal them for BN254's D-type twist and are their inverses for BLS12-381's M-type).
def f12_mul(p, xi, a, b):
    """a * b for a, b lists of six Fq2 coefficients of w^0..w^5, w^6 = xi"""
    t = [(0, 0)] * 11
    for i in range(6):
        for j in range(6):
            m = f2_mul(p, a[i], b[j])
            t[i + j] = ((t[i + j][0] + m[0]) % p, (t[i + j][1] + m[1]) % p)
    for k in range(10, 5, -1):
        m = f2_mul(p, t[k], xi)
        t[k - 6] = ((t[k - 6][0] + m[0]) % p, (t[k - 6][1] + m[1]) % p)
    return t[:6]


def f12_pow(p, xi, a, e):
    r = [(1, 0)] + [(0, 0)] * 5
    for bit in bin(e)[2:]:
        r = f12_mul(p, xi, r, r)
        if bit == "1":
            r = f12_mul(p, xi, r, a)
    return r


def frobenius_coeffs(p, xi, psi, m_type):
    """{j: [xi^(k (p^j - 1) / 6) for k = 0..5]} for j = 1, 2, 3, checked as described above"""
    import random
    rng = random.Random(12)
    g = {j: [f2_pow(p, xi, k * (p ** j - 1) // 6) for k in range(6)] for j in (1, 2, 3)}
    a = [(rng.randrange(p), rng.randrange(p)) for _ in range(6)]
    ap = a
    for j in (1, 2, 3):
        ap = f12_pow(p, xi, ap, p)
        conj = [(c[0], (-c[1]) % p) if j % 2 else c for c in a]
        assert [f2_mul(p, conj[k], g[j][k]) for k in range(6)] == ap, j
        assert all(c[1] == 0 for c in g[2])                   # p^2 coefficients lie in Fq
    cx, cy = (f2_inv(p, g[1][2]), f2_inv(p, g[1][3])) if m_type else (g[1][2], g[1][3])
    assert (cx, cy) == psi
    return g


def naf(n):
    """signed binary digits of n, most significant first (the first digit is 1)"""
    d = []
    while n:
        z = (2 - n % 4) if n & 1 else 0
        n = (n - z) // 2
        d.append(z)
    return d[::-1]


def pairing_extra(p, n, r, xi, frob, x, loop, signed):
    """Constants of pairing.cuh: xi, the Frobenius coefficients, the Miller loop's digits (non-adjacent form when `signed`,
    which saves additions for BN254's 6x + 2 but not for BLS12-381's sparse |x|) and |x| (plain words)."""
    R = 1 << (32 * n)
    digits = naf(loop) if signed else [int(b) for b in bin(loop)[2:]]
    assert sum(d << (len(digits) - 1 - i) for i, d in enumerate(digits)) == loop and digits[0] == 1
    pos = sum(1 << (len(digits) - 1 - i) for i, d in enumerate(digits) if d == 1)
    neg = sum(1 << (len(digits) - 1 - i) for i, d in enumerate(digits) if d == -1)
    lw = (len(digits) + 31) // 32
    rows = [frob[j][k][c] for j in (1, 2, 3) for k in range(1, 6) for c in (0, 1)]
    s = "    // pairing (pairing.cuh): xi = XI0 + u; frob(2 (5 (j - 1) + k - 1) + c, i) = component c of xi^(k (p^j - 1) / 6),\n"
    s += "    // Montgomery, j = 1..3, k = 1..5; the Miller loop's signed digits (+1 in ate_pos, -1 in ate_neg, ATE_BITS digits,\n"
    s += "    // the top one 1); |x| of the curve family in plain words and its sign\n"
    s += "    static constexpr int XI0 = %d;\n" % xi[0]
    s += "    B2S_HD static constexpr uint32_t frob(int j, int i) { constexpr uint32_t t[30][%d] = {%s}; return t[j][i]; }\n" % (
        n, ", ".join(arr(v * R % p, n) for v in rows))
    s += "    static constexpr int ATE_BITS = %d;\n" % len(digits)
    s += "    static constexpr int ATE_WORDS = %d;\n" % lw
    s += "    B2S_HD static constexpr uint32_t ate_pos(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (lw, words(pos, lw))
    s += "    B2S_HD static constexpr uint32_t ate_neg(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (lw, words(neg, lw))
    s += "    static constexpr bool X_NEG = %s;\n" % ("true" if x < 0 else "false")
    s += "    B2S_HD static constexpr uint32_t x_abs(int i) { constexpr uint32_t t[2] = %s; return t[i]; }\n" % words(abs(x), 2)
    return s


def check_pairing_params():
    """The loop lengths and the hard-part chains of pairing.cuh, as identities in the curve parameters."""
    x, p, r = -BLS_X_ABS, BLS_P, BLS_R
    h = (p ** 4 - p ** 2 + 1) // r
    assert (x - 1) ** 2 * (x + p) * (x * x + p * p - 1) + 3 == 3 * h           # BLS12-381 hard part: f^(3 h)
    x, p, r = BN_X, BN_P, BN_R
    assert (6 * x + 2 + p - p * p + p ** 3) % r == 0                           # BN254 optimal ate loop
    h = (p ** 4 - p ** 2 + 1) // r
    lam = [1 + 6 * x + 12 * x * x + 12 * x ** 3, 4 * x + 6 * x * x + 12 * x ** 3, 6 * x + 6 * x * x + 12 * x ** 3,
           -1 + 4 * x + 6 * x * x + 12 * x ** 3]
    assert sum(l * p ** i for i, l in enumerate(lam)) == 2 * x * (6 * x * x + 3 * x + 1) * h   # BN254 hard part


def main():
    out = "// GENERATED by tools/gen_field_params.py -- do not edit.\n"
    out += "// Montgomery constants (R = 2^(32 N)) for BLS12-381 / BN254 base and scalar fields.\n"
    out += "#pragma once\n#include <cstdint>\n#include \"ff.cuh\"\n\nnamespace b2s {\n\n"
    inv82 = pow(82, -1, BN_P)
    bn_b2 = (27 * inv82 % BN_P, (-3 * inv82) % BN_P)
    bls_psi = psi_coeffs(BLS_P, BLS_R, (1, 1), BLS_G2, -BLS_X_ABS)
    bn_psi = psi_coeffs(BN_P, BN_R, (9, 1), BN_G2, 6 * BN_X * BN_X)
    check_pairing_params()
    bls_frob = frobenius_coeffs(BLS_P, (1, 1), bls_psi, True)
    bn_frob = frobenius_coeffs(BN_P, (9, 1), bn_psi, False)
    out += field_struct("BlsFqP", BLS_P, 12, curve_extra(BLS_P, 12, BLS_G1, BLS_G2, 4, (4, 4))
                        + decode_extra(BLS_P, 12, bls_beta(), bls_psi, BLS_X_ABS, 2)
                        + pairing_extra(BLS_P, 12, BLS_R, (1, 1), bls_frob, -BLS_X_ABS, BLS_X_ABS, False))
    out += field_struct("BlsFrP", BLS_R, 8, fr_extra(BLS_R, 8, 7, 32))
    out += field_struct("BnFqP", BN_P, 8, curve_extra(BN_P, 8, BN_G1, BN_G2, 3, bn_b2)
                        + decode_extra(BN_P, 8, 1, bn_psi, 6 * BN_X * BN_X, 4)
                        + pairing_extra(BN_P, 8, BN_R, (9, 1), bn_frob, BN_X, 6 * BN_X + 2, True))
    out += field_struct("BnFrP", BN_R, 8, fr_extra(BN_R, 8, 5, 28))
    out += "}  // namespace b2s\n"
    path = os.path.join(os.path.dirname(__file__), "..", "snark_b200", "csrc", "field_params.h")
    with open(path, "w") as f:
        f.write(out)
    print("wrote", os.path.normpath(path))


if __name__ == "__main__":
    main()
