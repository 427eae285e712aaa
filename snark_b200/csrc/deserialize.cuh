// CanonicalDeserialize of one group element: the per-point half of loading proofs and keys (deserialize.cu), written
// B2S_HD so that tests/native/host_deserialize.cpp compiles the same code for the CPU and checks it against the oracle.
//
// Encodings (ark-serialize as instantiated by ark-bls12-381 / ark-bn254; recalled, crates not in the reference tree, and
// not pinned against bytes written by a Rust build -- the oracle, tests/wire_oracle.py, restates the same rules):
//
//   |              | BLS12-381 (zcash / IETF, big-endian, G2 as c1 || c0)  | BN254 (ark-ec SWFlags, little-endian, G2 c0 || c1) |
//   | flags        | byte 0: 0x80 compressed, 0x40 infinity, 0x20 larger   | last byte: 0x80 larger root, 0x40 infinity;        |
//   |              |                                                       | 0xC0 is rejected                                   |
//   | compressed   | 0x80 must be set                                      | (no mode bit)                                      |
//   | uncompressed | 0x80 and 0x20 must be clear                           | flags in the last byte of y; the sign is not used  |
//   | infinity     | every other bit and byte zero; 0x20 clear             | every other bit and byte zero                      |
//   BLS12-377 uses the SWFlags form of the right-hand column (ark-bls12-377 keeps ark-ec's default); its Fq has 7 spare
//   bits, so any bit between bit 376 and the two flag bits leaves the coordinate >= p: DEC_NONCANONICAL.
//
// Every coordinate must be canonical (< p).  Compressed points take y = sqrt(x^3 + b) (a^((p+1)/4) for p = 3 mod 4,
// Tonelli-Shanks for BLS12-377's p = 1 mod 2^46), the root chosen by the
// "lexicographically larger" bit (y_is_larger, shared with the serializer); no root means the encoding is invalid whatever
// `validate` says.  With validate (ark's Validate::Yes) uncompressed points must satisfy the curve equation and every point
// must lie in the prime-order subgroup, tested by endomorphism criteria instead of r * P = O:
//   BLS12-381 G1  phi(P) = -[x^2]P, phi(x, y) = (beta x, y)       BLS12-381 G2  psi(P) = [x]P, x = -0xd201000000010000
//   BN254 G1      cofactor 1: on the curve is enough               BN254 G2      psi(P) = [6 x^2]P
//   BLS12-377 G1  phi(P) = -[x^2]P                                 BLS12-377 G2  psi(P) = [x]P, x = 0x8508c00000000001
// with psi(x, y) = (conj(x) cx, conj(y) cy).  beta, cx, cy and the scalars are generated (tools/gen_field_params.py, which
// checks each criterion on the generator); tests/test_host_deserialize.py checks the verdicts against r * P = O on points
// outside the subgroup.  Comparisons are projective: no inversion per point.
#pragma once
#include "curves.cuh"

// The exponentiations and scalar multiplications below are kept out of line on the device: inlined into one kernel body
// they leave ptxas with hundreds of live limbs and the kernel spills most of them to local memory.
#if defined(__CUDACC__)
#define B2S_DEC_NOINLINE __host__ __device__ __noinline__
#else
#define B2S_DEC_NOINLINE inline
#endif

namespace b2s {

// reason a point is rejected (0 = accepted); also the low 3 bits of the packed error word of deserialize.cu
enum DecodeStatus : uint32_t { DEC_OK = 0, DEC_BAD_FLAGS = 1, DEC_NONCANONICAL = 2, DEC_NOT_ON_CURVE = 3, DEC_NOT_IN_SUBGROUP = 4 };

template <class B>
B2S_HD int cmp_canon(const B& a, const B& b) {   // canonical (non-Montgomery) values
    for (int i = B::N - 1; i >= 0; i--) {
        if (a.v[i] != b.v[i]) return a.v[i] > b.v[i] ? 1 : -1;
    }
    return 0;
}
// the sign bit of both encodings: y is the larger of y and -y as canonical integers (Fq2: c1 first, then c0)
template <class P>
B2S_HD bool y_is_larger(const Fp<P>& y) {
    const Fp<P> a = y.from_mont(), b = y.neg().from_mont();
    return cmp_canon(a, b) > 0;
}
template <class P>
B2S_HD bool y_is_larger(const Fp2<P>& y) {
    const Fp2<P> n = y.neg();
    const int c1 = cmp_canon(y.c1.from_mont(), n.c1.from_mont());
    if (c1 != 0) return c1 > 0;
    return cmp_canon(y.c0.from_mont(), n.c0.from_mont()) > 0;
}

namespace dec {

// raw limbs of one base-field element from its 4N bytes
template <class P>
B2S_HD void load_fq(const uint8_t* b, bool big_endian, Fp<P>& x) {
    constexpr int NB = 4 * Fp<P>::N;
    for (int i = 0; i < Fp<P>::N; i++) {
        uint32_t w = 0;
        for (int k = 0; k < 4; k++) w |= (uint32_t)b[big_endian ? NB - 1 - (4 * i + k) : 4 * i + k] << (8 * k);
        x.v[i] = w;
    }
}
template <class P>
B2S_HD void load_coord(const uint8_t* b, bool bls, Fp<P>& x) { load_fq(b, bls, x); }
template <class P>
B2S_HD void load_coord(const uint8_t* b, bool bls, Fp2<P>& x) {
    constexpr int NB = 4 * Fp<P>::N;
    if (bls) { load_fq(b, true, x.c1); load_fq(b + NB, true, x.c0); }
    else { load_fq(b, false, x.c0); load_fq(b + NB, false, x.c1); }
}
// the element whose top byte carries the flags: BLS12-381 writes it first, BN254 last; for Fq2 that is c1 in both
template <class P>
B2S_HD Fp<P>& top_elem(Fp<P>& x) { return x; }
template <class P>
B2S_HD Fp<P>& top_elem(Fp2<P>& x) { return x.c1; }

// raw limbs below the modulus (of either field: P is FqP or FrP)
template <class P>
B2S_HD bool below_p(const Fp<P>& a) {
    int c = 0;
    for (int i = Fp<P>::N - 1; i >= 0 && c == 0; i--) c = a.v[i] < P::mod(i) ? -1 : a.v[i] > P::mod(i) ? 1 : 0;
    return c < 0;
}
template <class P>
B2S_HD bool below_p(const Fp2<P>& a) { return below_p(a.c0) && below_p(a.c1); }
// raw limbs -> Montgomery form; false if the value is not below p
template <class P>
B2S_HD bool to_field(Fp<P>& a) {
    if (!below_p(a)) return false;
    a = a.to_mont();
    return true;
}
template <class P>
B2S_HD bool to_field(Fp2<P>& a) { return to_field(a.c0) && to_field(a.c1); }

template <class P>
B2S_HD Fp<P> curve_b(const Fp<P>*) {
    Fp<P> b;
    for (int i = 0; i < Fp<P>::N; i++) b.v[i] = P::b1(i);
    return b;
}
template <class P>
B2S_HD Fp2<P> curve_b(const Fp2<P>*) {
    Fp2<P> b;
    for (int i = 0; i < Fp<P>::N; i++) { b.c0.v[i] = P::b2c0(i); b.c1.v[i] = P::b2c1(i); }
    return b;
}

// a^((p-3)/4): for p = 3 mod 4, r = a^((p+1)/4) = (this) * a is the square root when one exists, and (this) = 1 / r
template <class P>
B2S_DEC_NOINLINE Fp<P> pow_sqrt_exp(const Fp<P>& a) {
    uint32_t e[Fp<P>::N];
    for (int i = 0; i < Fp<P>::N; i++) e[i] = P::sqrt_exp(i);
    return a.pow_words(e, Fp<P>::N);
}
// Tonelli-Shanks for p - 1 = 2^S q (BLS12-377: S = 46): x = a^((q+1)/2) is a root up to the 2^S-th root of unity
// b = a^q; each round finds the order 2^k of b and multiplies x by a power of the precomputed root z^q
template <class P>
B2S_DEC_NOINLINE bool sqrt_ts(const Fp<P>& a, Fp<P>& r) {
    using B = Fp<P>;
    if (a.is_zero()) { r = a; return true; }
    uint32_t e[B::N];
    B z;
    for (int i = 0; i < B::N; i++) { e[i] = P::ts_exp(i); z.v[i] = P::ts_root(i); }
    const B w = a.pow_words(e, B::N);   // a^((q-1)/2)
    B x = a * w, b = x * w;             // a^((q+1)/2), a^q
    int v = P::TS_S;
    while (b != B::one()) {
        int k = 0;
        for (B t = b; t != B::one(); t = t.sqr())
            if (++k == v) return false;   // b has order 2^v: a is not a square
        B g = z;
        for (int i = 0; i < v - k - 1; i++) g = g.sqr();
        z = g.sqr();
        b = b * z;
        x = x * g;
        v = k;
    }
    r = x;
    return true;
}
template <class P>
B2S_DEC_NOINLINE bool sqrt(const Fp<P>& a, Fp<P>& r) {
    if constexpr (P::SQRT_TS) {
        return sqrt_ts(a, r);
    } else {
        r = pow_sqrt_exp(a) * a;
        return r.sqr() == a;
    }
}
// Fq2 = Fq[u]/(u^2 + 5) by the norm method with square roots by sqrt(): alpha = sqrt(a0^2 + 5 a1^2), delta =
// (a0 +- alpha) / 2, x0 = sqrt(delta), x1 = a1 / (2 x0); for a1 = 0 either sqrt(a0) or sqrt(-a0 / 5) u
template <class P>
B2S_DEC_NOINLINE bool sqrt_nr5(const Fp2<P>& a, Fp2<P>& r) {
    using B = Fp<P>;
    if (a.c1.is_zero()) {
        B s;
        if (sqrt(a.c0, s)) { r = {s, B::zero()}; return true; }
        B nr_inv;
        for (int i = 0; i < B::N; i++) nr_inv.v[i] = P::fq2_nr_inv(i);
        if (sqrt(a.c0 * nr_inv, s)) { r = {B::zero(), s}; return true; }   // (s u)^2 = -5 s^2 = a0
        return false;
    }
    B alpha;
    if (!sqrt(a.c0.sqr() + Fp2<P>::times5(a.c1.sqr()), alpha)) return false;
    B half;
    for (int i = 0; i < B::N; i++) half.v[i] = P::fq_half(i);
    B x0;
    if (!sqrt((a.c0 + alpha) * half, x0) && !sqrt((a.c0 - alpha) * half, x0)) return false;
    r = {x0, a.c1 * x0.dbl().inverse()};
    return r.sqr() == a;
}
// Fq2 = Fq[u]/(u^2 + 1) by the norm method: with alpha = sqrt(a0^2 + a1^2) one of (a0 +- alpha) / 2 is a square delta;
// x0 = sqrt(delta), x1 = a1 / (2 x0), where t = delta^((p-3)/4) gives both x0 = t delta and 1 / x0 = t
template <class P>
B2S_DEC_NOINLINE bool sqrt(const Fp2<P>& a, Fp2<P>& r) {
    using B = Fp<P>;
    if constexpr (P::FQ2_NR == -5) {
        return sqrt_nr5(a, r);
    } else {
        if (a.c1.is_zero()) {
            B s;
            if (sqrt(a.c0, s)) { r = {s, B::zero()}; return true; }
            if (sqrt(a.c0.neg(), s)) { r = {B::zero(), s}; return true; }   // sqrt(-a0) u
            return false;
        }
        B alpha;
        if (!sqrt(a.c0.sqr() + a.c1.sqr(), alpha)) return false;
        B half;
        for (int i = 0; i < B::N; i++) half.v[i] = P::fq_half(i);
        B delta = (a.c0 + alpha) * half;
        B t = pow_sqrt_exp(delta);
        if (t.sqr() * delta != B::one()) {
            delta = (a.c0 - alpha) * half;
            t = pow_sqrt_exp(delta);
        }
        r = {t * delta, a.c1 * t * half};
        return r.sqr() == a;
    }
}

// q == a for q projective (XYZZ), a affine, without an inversion
template <class F>
B2S_HD bool eq_affine(const XYZZ<F>& q, const Affine<F>& a) {
    if (q.is_identity()) return a.is_inf();
    return q.x == a.x * q.zz && q.y == a.y * q.zzz;
}

template <class P, class F>
B2S_DEC_NOINLINE XYZZ<F> mul_endo_scalar(const XYZZ<F>& q) {
    uint32_t k[P::ENDO_WORDS];
    for (int i = 0; i < P::ENDO_WORDS; i++) k[i] = P::endo_scalar(i);
    return scalar_mul_words(q, k, P::ENDO_WORDS);
}

// prime-order subgroup membership of an affine point already on the curve
template <class Curve>
B2S_DEC_NOINLINE bool in_subgroup(const Affine<typename Curve::Fq>& p) {
    using P = typename Curve::FqP;
    using F = typename Curve::Fq;
    if (!P::BLS12_FAMILY || p.is_inf()) return true;   // BN254: cofactor 1
    // -[x^2]P == (beta x, y)  <=>  [|x|]([|x|]P) == (beta x, -y)
    F beta;
    for (int i = 0; i < F::N; i++) beta.v[i] = P::beta(i);
    const XYZZ<F> q = mul_endo_scalar<P>(mul_endo_scalar<P>(XYZZ<F>::from_affine(p)));
    return eq_affine(q, Affine<F>{beta * p.x, p.y.neg()});
}
template <class Curve>
B2S_DEC_NOINLINE bool in_subgroup(const Affine<typename Curve::Fq2>& p) {
    using P = typename Curve::FqP;
    using F = typename Curve::Fq2;
    if (p.is_inf()) return true;
    F cx, cy;
    for (int i = 0; i < Fp<P>::N; i++) {
        cx.c0.v[i] = P::psi_x0(i); cx.c1.v[i] = P::psi_x1(i);
        cy.c0.v[i] = P::psi_y0(i); cy.c1.v[i] = P::psi_y1(i);
    }
    const F xc{p.x.c0, p.x.c1.neg()}, yc{p.y.c0, p.y.c1.neg()};
    Affine<F> psi{xc * cx, yc * cy};
    // BLS12-381: psi(P) == [x]P = -[|x|]P;  BLS12-377: psi(P) == [x]P;  BN254: psi(P) == [6 x^2]P
    if (P::X_NEG) psi = psi.neg();
    return eq_affine(mul_endo_scalar<P>(XYZZ<F>::from_affine(p)), psi);
}

}  // namespace dec

// One encoded point of the curve's G1 (F = Fq) or G2 (F = Fq2) -> affine Montgomery (infinity = all-zero limbs).
// Returns a DecodeStatus; `out` is meaningful only for DEC_OK.
template <class Curve, class F>
B2S_HD uint32_t decode_point(const uint8_t* in, bool compressed, bool validate, Affine<F>& out) {
    using P = typename Curve::FqP;
    constexpr bool bls = P::ZCASH_SERIAL;
    constexpr int CB = (int)(sizeof(F) / sizeof(Fp<P>)) * 4 * Fp<P>::N;   // bytes of one coordinate
    constexpr int TOP = Fp<P>::N - 1;
    F x, y = F::zero();
    dec::load_coord(in, bls, x);
    if (!compressed) dec::load_coord(in + CB, bls, y);
    uint32_t& top = dec::top_elem(bls || compressed ? x : y).v[TOP];
    const uint32_t flags = (top >> 24) & (bls ? 0xE0u : 0xC0u);
    top &= bls ? 0x1FFFFFFFu : 0x3FFFFFFFu;
    bool larger = false;
    if (bls) {
        if (compressed != ((flags & 0x80) != 0)) return DEC_BAD_FLAGS;
        if (!compressed && (flags & 0x20)) return DEC_BAD_FLAGS;
        if (flags & 0x40) {
            if ((flags & 0x20) || !x.is_zero() || !y.is_zero()) return DEC_BAD_FLAGS;
            out = Affine<F>::inf();
            return DEC_OK;
        }
        larger = (flags & 0x20) != 0;
    } else {
        if (flags == 0xC0) return DEC_BAD_FLAGS;
        if (flags & 0x40) {
            if (!x.is_zero() || !y.is_zero()) return DEC_BAD_FLAGS;
            out = Affine<F>::inf();
            return DEC_OK;
        }
        larger = (flags & 0x80) != 0;
    }
    if (!dec::to_field(x)) return DEC_NONCANONICAL;
    const F rhs = x.sqr() * x + dec::curve_b((const F*)nullptr);
    if (compressed) {
        if (!dec::sqrt(rhs, y)) return DEC_NOT_ON_CURVE;
        if (y_is_larger(y) != larger) y = y.neg();
    } else {
        if (!dec::to_field(y)) return DEC_NONCANONICAL;
        if (validate && y.sqr() != rhs) return DEC_NOT_ON_CURVE;
    }
    out = Affine<F>{x, y};
    if (validate && !dec::in_subgroup<Curve>(out)) return DEC_NOT_IN_SUBGROUP;
    return DEC_OK;
}

// One point as a snarkjs .zkey stores it (zkey.cu): x || y as Montgomery little-endian limbs, G2 coordinates c0 || c1 --
// already this library's affine layout -- with infinity all-zero.  No flags and no square root: every coordinate must be
// below p; with validate the point must satisfy the curve equation and the subgroup criterion of decode_point.
template <class Curve, class F>
B2S_HD uint32_t decode_point_mont(const uint8_t* in, bool validate, Affine<F>& out) {
    using P = typename Curve::FqP;
    constexpr int CB = (int)(sizeof(F) / sizeof(Fp<P>)) * 4 * Fp<P>::N;
    F x, y;
    dec::load_coord(in, false, x);
    dec::load_coord(in + CB, false, y);
    if (x.is_zero() && y.is_zero()) {
        out = Affine<F>::inf();
        return DEC_OK;
    }
    if (!dec::below_p(x) || !dec::below_p(y)) return DEC_NONCANONICAL;
    if (validate && y.sqr() != x.sqr() * x + dec::curve_b((const F*)nullptr)) return DEC_NOT_ON_CURVE;
    out = Affine<F>{x, y};
    if (validate && !dec::in_subgroup<Curve>(out)) return DEC_NOT_IN_SUBGROUP;
    return DEC_OK;
}

}  // namespace b2s
