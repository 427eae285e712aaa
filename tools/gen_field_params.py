#!/usr/bin/env python3
"""Generate snark_b200/csrc/field_params.h (Montgomery constants for the four prime fields and
the curve constants the kernels need).  Developer tool: run once, commit the header.

The numbers are the standard BLS12-381 / BN254 parameters (SURVEY.md Appendix B) and BLS12-377's, derived here from
its seed x; the header is cross-checked against the oracles' independent copies in tests/test_host_ff.py and
tests/test_host_bls12_377.py.
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
# BLS12-377 (ark-bls12-377): everything follows from the seed x, which check_bls377_params asserts
BLS377_X = 0x8508c00000000001
BLS377_P = 0x01ae3a4617c510eac63b05c06ca1493b1a22d9f300f5138f1ef3622fba094800170b5d44300000008508c00000000001
BLS377_R = 0x12ab655e9a2ca55660b44d1e5c37b00159aa76fed00000010a11800000000001
BLS377_G1 = (
    81937999373150964239938255573465948239988671502647976594219695644855304257327692006745978603320413799295628339695,
    241266749859715473739788878240585681733927191168601896383759122102112907357779751001206799952863815012735208165030,
)
BLS377_G2 = (
    233578398248691099356572568220835526895379068987715365179118596935057653620464273615301663571204657964920925606294,
    140913150380207355837477652521042157274541796891053068589147167627541651775299824604154852141315666357241556069118,
    63160294768292073209381361943935198908131692476676907196754037919244929611450776219210369229519898517858833747423,
    149157405641012693445398062341192467754805999074082136895788947234480009303640899064710353187729182149407503257491,
)
BLS377_B2 = (0, (-pow(5, -1, BLS377_P)) % BLS377_P)     # 1 / u with u^2 = -5
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
    # inversion by divsteps (ff.cuh, Fp::inverse): p in signed 30-bit limbs, with room for the (-2p, p) range of the
    # Bezout coefficients; p^-1 mod 2^30; R^3 mod p, which one Montgomery product turns the plain inverse of a
    # Montgomery-form input into the Montgomery form of the inverse
    il = (p.bit_length() + 2 + 29) // 30
    s += "    static constexpr int INV_LIMBS = %d;\n" % il
    s += "    static constexpr uint32_t INV_PINV30 = 0x%08xu;\n" % pow(p, -1, 1 << 30)
    s += "    B2S_HD static constexpr int32_t inv_mod30(int i) { constexpr int32_t t[%d] = {%s}; return t[i]; }\n" % (
        il, ", ".join("0x%08x" % ((p >> (30 * i)) & ((1 << 30) - 1)) for i in range(il)))
    assert p >> (30 * il) == 0
    s += fn("inv_final", R ** 3 % p)
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


# Fq2 = Fq[u] / (u^2 - nr): nr = -1 for BLS12-381 and BN254, -5 for BLS12-377
def f2_mul(p, a, b, nr=-1):
    return ((a[0] * b[0] + nr * a[1] * b[1]) % p, (a[0] * b[1] + a[1] * b[0]) % p)


def f2_pow(p, a, e, nr=-1):
    r = (1, 0)
    for bit in bin(e)[2:]:
        r = f2_mul(p, r, r, nr)
        if bit == "1":
            r = f2_mul(p, r, a, nr)
    return r


def f2_inv(p, a, nr=-1):
    n = pow(a[0] * a[0] - nr * a[1] * a[1], -1, p)
    return (a[0] * n % p, (-a[1]) * n % p)


def ec_mul(p, ext, P, k, nr=-1):
    """k * P on y^2 = x^3 + b (affine, a = 0) over Fq (ext False) or Fq2 (ext True); None = infinity."""
    mul = (lambda a, b: f2_mul(p, a, b, nr)) if ext else (lambda a, b: a * b % p)
    inv = (lambda a: f2_inv(p, a, nr)) if ext else (lambda a: pow(a, -1, p))
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


def bls_beta(p=BLS_P, r=BLS_R, g1=BLS_G1, x=-BLS_X_ABS):
    """the cube root of unity beta with phi(G1) = -[x^2] G1 for a BLS12 curve"""
    for g in range(2, 100):
        w = pow(g, (p - 1) // 3, p)
        if w != 1:
            break
    lam = (-x * x) % r
    target = ec_mul(p, False, g1, lam)
    hits = [b for b in (w, w * w % p) if (b * g1[0] % p, g1[1]) == target]
    assert len(hits) == 1
    return hits[0]


def psi_coeffs(p, r, xi, gen, lam, nr=-1):
    """(cx, cy) with psi(gen) = [lam] gen for cx = xi^(e (p-1)/3), cy = xi^(e (p-1)/2), e = +1 or -1."""
    x, y = (gen[0], gen[1]), (gen[2], gen[3])
    target = ec_mul(p, True, (x, y), lam % r, nr)
    hits = []
    for e in (1, -1):
        base = xi if e == 1 else f2_inv(p, xi, nr)
        cx, cy = f2_pow(p, base, (p - 1) // 3, nr), f2_pow(p, base, (p - 1) // 2, nr)
        if (f2_mul(p, (x[0], -x[1] % p), cx, nr), f2_mul(p, (y[0], -y[1] % p), cy, nr)) == target:
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
    if p % 4 == 3:
        s = "    // point decoding (deserialize.cuh): (p - 3) / 4 in plain words; Montgomery forms of 1/2, the cube root of unity\n"
    else:
        s = "    // point decoding (deserialize.cuh; square roots by Tonelli-Shanks, see the traits below): Montgomery forms of 1/2, the cube root of unity\n"
    s += "    // beta of the G1 endomorphism (1 when unused) and the psi coefficients cx, cy of G2; the subgroup-test scalar in\n"
    s += "    // plain words (BLS12-381: |x|; BN254: 6 x^2)\n"
    if p % 4 == 3:
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
def f12_mul(p, xi, a, b, nr=-1):
    """a * b for a, b lists of six Fq2 coefficients of w^0..w^5, w^6 = xi"""
    t = [(0, 0)] * 11
    for i in range(6):
        for j in range(6):
            m = f2_mul(p, a[i], b[j], nr)
            t[i + j] = ((t[i + j][0] + m[0]) % p, (t[i + j][1] + m[1]) % p)
    for k in range(10, 5, -1):
        m = f2_mul(p, t[k], xi, nr)
        t[k - 6] = ((t[k - 6][0] + m[0]) % p, (t[k - 6][1] + m[1]) % p)
    return t[:6]


def f12_pow(p, xi, a, e, nr=-1):
    r = [(1, 0)] + [(0, 0)] * 5
    for bit in bin(e)[2:]:
        r = f12_mul(p, xi, r, r, nr)
        if bit == "1":
            r = f12_mul(p, xi, r, a, nr)
    return r


def frobenius_coeffs(p, xi, psi, m_type, nr=-1):
    """{j: [xi^(k (p^j - 1) / 6) for k = 0..5]} for j = 1, 2, 3, checked as described above"""
    import random
    rng = random.Random(12)
    g = {j: [f2_pow(p, xi, k * (p ** j - 1) // 6, nr) for k in range(6)] for j in (1, 2, 3)}
    a = [(rng.randrange(p), rng.randrange(p)) for _ in range(6)]
    ap = a
    for j in (1, 2, 3):
        ap = f12_pow(p, xi, ap, p, nr)
        conj = [(c[0], (-c[1]) % p) if j % 2 else c for c in a]
        assert [f2_mul(p, conj[k], g[j][k], nr) for k in range(6)] == ap, j
        assert all(c[1] == 0 for c in g[2])                   # p^2 coefficients lie in Fq
    cx, cy = (f2_inv(p, g[1][2], nr), f2_inv(p, g[1][3], nr)) if m_type else (g[1][2], g[1][3])
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


def traits_extra(p, n, nr, bls12, m_twist, zcash):
    """Named traits that select code paths per curve, and the Tonelli-Shanks constants when p = 1 mod 4."""
    R = 1 << (32 * n)
    s = "    // traits: u^2 = FQ2_NR in Fq2; the BLS12 family (Miller loop over x, no Frobenius lines, BLS12 hard part) or BN;\n"
    s += "    // M- or D-type twist; zcash / IETF serialization (else ark-ec SWFlags); square roots by Tonelli-Shanks\n"
    s += "    static constexpr int FQ2_NR = %d;\n" % nr
    s += "    static constexpr bool BLS12_FAMILY = %s;\n" % ("true" if bls12 else "false")
    s += "    static constexpr bool M_TWIST = %s;\n" % ("true" if m_twist else "false")
    s += "    static constexpr bool ZCASH_SERIAL = %s;\n" % ("true" if zcash else "false")
    s += "    static constexpr bool SQRT_TS = %s;\n" % ("false" if p % 4 == 3 else "true")
    if nr != -1:
        s += "    // Montgomery form of 1 / FQ2_NR (sqrt of a0 in Fq2 with a0 a non-square: sqrt(a0 / FQ2_NR) u)\n"
        s += "    B2S_HD static constexpr uint32_t fq2_nr_inv(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (
            n, arr(pow(nr, -1, p) * R % p, n))
    if p % 4 == 1:
        S, Q = 0, p - 1
        while Q % 2 == 0:
            S, Q = S + 1, Q // 2
        z = next(g for g in range(2, 1000) if pow(g, (p - 1) // 2, p) == p - 1)
        c = pow(z, Q, p)
        assert pow(c, 1 << (S - 1), p) == p - 1                          # a primitive 2^S-th root of unity
        s += "    // Tonelli-Shanks: p - 1 = 2^TS_S q; (q - 1) / 2 in plain words; z^q (Montgomery) for the non-residue z = %d\n" % z
        s += "    static constexpr int TS_S = %d;\n" % S
        s += "    B2S_HD static constexpr uint32_t ts_exp(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (n, words((Q - 1) // 2, n))
        s += "    B2S_HD static constexpr uint32_t ts_root(int i) { constexpr uint32_t t[%d] = %s; return t[i]; }\n" % (n, arr(c * R % p, n))
    return s


def two_adicity(n):
    k = 0
    while n % 2 == 0:
        n, k = n // 2, k + 1
    return k


def check_bls377_params():
    """BLS12-377 from its seed x alone, and the published constants against it."""
    x = BLS377_X
    r = x ** 4 - x ** 2 + 1
    assert (x - 1) ** 2 * r % 3 == 0
    p = (x - 1) ** 2 * r // 3 + x
    assert (p, r) == (BLS377_P, BLS377_R) and p.bit_length() == 377 and r.bit_length() == 253
    assert two_adicity(p - 1) == 46 and two_adicity(r - 1) == 47
    assert pow(22, (r - 1) // 2, r) == r - 1                          # ark's Fr GENERATOR 22 is a non-residue
    assert pow(p - 5, (p - 1) // 2, p) == p - 1                       # u^2 = -5 is irreducible
    g1, g2 = BLS377_G1, BLS377_G2
    assert (g1[1] ** 2 - g1[0] ** 3 - 1) % p == 0 and ec_mul(p, False, g1, r) is None
    gx, gy = (g2[0], g2[1]), (g2[2], g2[3])
    rhs = f2_mul(p, f2_mul(p, gx, gx, -5), gx, -5)
    assert f2_mul(p, gy, gy, -5) == ((rhs[0] + BLS377_B2[0]) % p, (rhs[1] + BLS377_B2[1]) % p)
    assert f2_mul(p, BLS377_B2, (0, 1), -5) == (1, 0)                  # b' = 1 / u: the D-type twist of y^2 = x^3 + 1
    assert ec_mul(p, True, (gx, gy), r, -5) is None


def check_pairing_params():
    """The loop lengths and the hard-part chains of pairing.cuh, as identities in the curve parameters."""
    x, p, r = -BLS_X_ABS, BLS_P, BLS_R
    h = (p ** 4 - p ** 2 + 1) // r
    assert (x - 1) ** 2 * (x + p) * (x * x + p * p - 1) + 3 == 3 * h           # BLS12-381 hard part: f^(3 h)
    x, p, r = BLS377_X, BLS377_P, BLS377_R
    h = (p ** 4 - p ** 2 + 1) // r
    assert (x - 1) ** 2 * (x + p) * (x * x + p * p - 1) + 3 == 3 * h           # BLS12-377 hard part (the same chain, x > 0)
    x, p, r = BN_X, BN_P, BN_R
    assert (6 * x + 2 + p - p * p + p ** 3) % r == 0                           # BN254 optimal ate loop
    h = (p ** 4 - p ** 2 + 1) // r
    lam = [1 + 6 * x + 12 * x * x + 12 * x ** 3, 4 * x + 6 * x * x + 12 * x ** 3, 6 * x + 6 * x * x + 12 * x ** 3,
           -1 + 4 * x + 6 * x * x + 12 * x ** 3]
    assert sum(l * p ** i for i, l in enumerate(lam)) == 2 * x * (6 * x * x + 3 * x + 1) * h   # BN254 hard part


def main():
    out = "// GENERATED by tools/gen_field_params.py -- do not edit.\n"
    out += "// Montgomery constants (R = 2^(32 N)) for BLS12-381 / BN254 / BLS12-377 base and scalar fields.\n"
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
                        + pairing_extra(BLS_P, 12, BLS_R, (1, 1), bls_frob, -BLS_X_ABS, BLS_X_ABS, False)
                        + traits_extra(BLS_P, 12, -1, True, True, True))
    out += field_struct("BlsFrP", BLS_R, 8, fr_extra(BLS_R, 8, 7, 32))
    out += field_struct("BnFqP", BN_P, 8, curve_extra(BN_P, 8, BN_G1, BN_G2, 3, bn_b2)
                        + decode_extra(BN_P, 8, 1, bn_psi, 6 * BN_X * BN_X, 4)
                        + pairing_extra(BN_P, 8, BN_R, (9, 1), bn_frob, BN_X, 6 * BN_X + 2, True)
                        + traits_extra(BN_P, 8, -1, False, False, False))
    out += field_struct("BnFrP", BN_R, 8, fr_extra(BN_R, 8, 5, 28))
    check_bls377_params()
    p7, r7, x7 = BLS377_P, BLS377_R, BLS377_X
    b377_psi = psi_coeffs(p7, r7, (0, 1), BLS377_G2, x7, -5)
    b377_frob = frobenius_coeffs(p7, (0, 1), b377_psi, False, -5)
    out += field_struct("Bls377FqP", p7, 12, curve_extra(p7, 12, BLS377_G1, BLS377_G2, 1, BLS377_B2)
                        + decode_extra(p7, 12, bls_beta(p7, r7, BLS377_G1, x7), b377_psi, x7, 2)
                        + pairing_extra(p7, 12, r7, (0, 1), b377_frob, x7, x7, False)
                        + traits_extra(p7, 12, -5, True, False, False))
    out += field_struct("Bls377FrP", r7, 8, fr_extra(r7, 8, 22, 47))
    out += "}  // namespace b2s\n"
    path = os.path.join(os.path.dirname(__file__), "..", "snark_b200", "csrc", "field_params.h")
    with open(path, "w") as f:
        f.write(out)
    print("wrote", os.path.normpath(path))


if __name__ == "__main__":
    main()
