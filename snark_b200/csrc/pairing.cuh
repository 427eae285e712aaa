// Optimal ate pairing on BLS12-381, BN254 and BLS12-377: the Fq6 / Fq12 tower, the Miller loop (on-the-fly or prepared lines, several
// pairs sharing one squaring per step), the final exponentiation, and the Groth16 verdict.  Written B2S_HD like
// deserialize.cuh, so tests/native/host_pairing.cpp compiles the same code for the CPU and checks it against the oracle.
//
// Tower (ark-ff's Fp6 / Fp12 layout, so a GT element is bit-identical to ark's Fp12 in memory):
//   Fq6 = Fq2[v] / (v^3 - xi),  Fq12 = Fq6[w] / (w^2 - v),  xi = 1 + u (BLS12-381) or 9 + u (BN254); so w^6 = xi and the
//   coefficient of w^k is  k = 0: c0.c0, 1: c1.c0, 2: c0.c1, 3: c1.c1, 4: c0.c2, 5: c1.c2.
//
// Miller loop, in homogeneous projective coordinates on the twist (ark-ec's G2Prepared formulas, derived again below):
//   BLS12-381 (M-type twist y^2 = x^3 + 4 xi, untwist (x / w^2, y / w^3)): over the bits of |x|, then f is conjugated
//     because x < 0.  A line through T evaluated at P, times w^3 and an Fq2 factor, is  l0 + l1 xP w^2 + l2 yP w^3.
//   BN254 (D-type twist y^2 = x^3 + 3 / xi, untwist (x w^2, y w^3)): over the signed digits of 6x + 2, then the lines
//     through pi(Q) and -pi^2(Q).  A line, times an Fq2 factor, is  l0 yP + l1 xP w + l2 w^3.
//   BLS12-377 (D-type twist y^2 = x^3 + 1 / u, xi = u with u^2 = -5): over the bits of x > 0, no conjugation and no
//     Frobenius lines; the lines have BN254's shape.  The twist type (M_TWIST) and the family (BLS12_FAMILY) are traits.
//   The dropped factors (w^3, Fq2 scalars) and the vertical lines lie in proper subfields of Fq12 that the easy part
//   of the final exponentiation maps to 1.  A pair with P or Q at infinity (all-zero) contributes 1.
//
// Final exponentiation: the easy part (p^6 - 1)(p^2 + 1), then a hard part that computes f^(m h), h = (p^4 - p^2 + 1) / r:
//   BLS12      m = 3:  3 h = (x - 1)^2 (x + p)(x^2 + p^2 - 1) + 3                 (Hayashida, Hayasaka, Teruya 2020)
//              (both BLS12 curves; cyclotomic_exp_x takes the sign of x into account)
//   BN254      m = 2x (6x^2 + 3x + 1):  m h = l0 + l1 p + l2 p^2 + l3 p^3 with      (Fuentes-Castaneda, Knapp,
//              l0 = 1 + 6x + 12x^2 + 12x^3, l1 = 4x + 6x^2 + 12x^3,                    Rodriguez-Henriquez 2011)
//              l2 = 6x + 6x^2 + 12x^3, l3 = -1 + 4x + 6x^2 + 12x^3
//   (tools/gen_field_params.py asserts both identities.)
//
// Relation to the oracle (oracle/pairing.py), which computes o(P, Q) = f_{T,Q}(P)^((p^12 - 1) / r) with the plain ate loop
// T = |t - 1| and no correction:  e(P, Q) = o(P, Q)^k with
//   BLS12-381  k = -3 mod r.  T = |x|, the same Miller function; the conjugation inverts it after the easy part, and the
//              hard part raises to m = 3.
//   BN254      k = 147946756881789319005730692170996259610.  Write [g] = g^((p^12 - 1) / r), Q in G2 = ker(pi - p),
//              T = 6x^2 = p - r.  From f_{ab,Q} = f_{a,Q}^b f_{b,[a]Q} and f_{a,pi(Q)}(P) = f_{a,Q}(P)^p:
//                t := [f_{r,Q}(P)] = o^(c / M), M = (T^12 - 1) / r, c = sum_{j<12} T^(11-j) p^j   (f_{T^12} = f_T^c = f_r^M)
//                a_p := [f_{p,Q}(P)] = o t   (p = T + r),    [f_{p^i,Q}(P)] = a_p^(i p^(i-1))
//                6x + 2 + p - p^2 + p^3 = n r, and the optimal ate value (Vercauteren 2010) is
//                e_opt = [f_{nr,Q}(P)] / a_p^(1 - 2p + 3p^2) = t^n / a_p^(1 - 2p + 3p^2)
//              so e = e_opt^m with m the hard-part multiplier above; k is that exponent reduced mod r.
//   BLS12-377  k = 3.  T = x > 0, the same Miller function and no conjugation; the hard part raises to m = 3.
//   Every k is coprime to r, so e is bilinear and non-degenerate; tests/test_host_pairing.py recomputes k from these
//   formulas and checks e = o^k on random pairs.
#pragma once
#include "curves.cuh"

// The tower operations are kept out of line on the device: inlined into one kernel body they leave ptxas with several
// hundred live limbs (one Fq12 alone is 144 registers on BLS12-381) and the kernel spills most of them.
#if defined(__CUDACC__)
#define B2S_PAIR_NOINLINE __host__ __device__ __noinline__
#else
#define B2S_PAIR_NOINLINE inline
#endif

namespace b2s {

// ---- Fq2 helpers ---------------------------------------------------------------------------------------------------
template <class P>
B2S_HD Fp2<P> conj(const Fp2<P>& a) { return {a.c0, a.c1.neg()}; }
template <class P>
B2S_HD Fp2<P> scale(const Fp2<P>& a, const Fp<P>& s) { return {a.c0 * s, a.c1 * s}; }
// a * xi, xi = XI0 + u:  (XI0 a0 - a1) + (a0 + XI0 a1) u for u^2 = -1;  a * u = -5 a1 + a0 u for xi = u, u^2 = -5
template <class P>
B2S_HD Fp2<P> mul_xi(const Fp2<P>& a) {
    static_assert((P::FQ2_NR == -1 && (P::XI0 == 1 || P::XI0 == 9)) || (P::FQ2_NR == -5 && P::XI0 == 0),
                  "xi = 1 + u or 9 + u with u^2 = -1, or xi = u with u^2 = -5");
    if constexpr (P::XI0 == 0) {
        return {Fp2<P>::times5(a.c1).neg(), a.c0};
    } else {
        if (P::XI0 == 1) return {a.c0 - a.c1, a.c0 + a.c1};
        const Fp<P> n0 = a.c0.dbl().dbl().dbl() + a.c0, n1 = a.c1.dbl().dbl().dbl() + a.c1;
        return {n0 - a.c1, a.c0 + n1};
    }
}
template <class P>
B2S_HD Fp2<P> frob_coeff(int j, int k) {   // xi^(k (p^j - 1) / 6), j = 1..3, k = 1..5
    Fp2<P> g;
    const int row = 2 * (5 * (j - 1) + k - 1);
    for (int i = 0; i < Fp<P>::N; i++) { g.c0.v[i] = P::frob(row, i); g.c1.v[i] = P::frob(row + 1, i); }
    return g;
}

// ---- Fq6 -----------------------------------------------------------------------------------------------------------
template <class P>
struct Fp6 {
    using F2 = Fp2<P>;
    F2 c0, c1, c2;
    B2S_HD static Fp6 zero() { return {F2::zero(), F2::zero(), F2::zero()}; }
    B2S_HD static Fp6 one() { return {F2::one(), F2::zero(), F2::zero()}; }
    B2S_HD bool operator==(const Fp6& o) const { return c0 == o.c0 && c1 == o.c1 && c2 == o.c2; }
    B2S_HD friend Fp6 operator+(const Fp6& a, const Fp6& b) { return {a.c0 + b.c0, a.c1 + b.c1, a.c2 + b.c2}; }
    B2S_HD friend Fp6 operator-(const Fp6& a, const Fp6& b) { return {a.c0 - b.c0, a.c1 - b.c1, a.c2 - b.c2}; }
    B2S_HD Fp6 neg() const { return {c0.neg(), c1.neg(), c2.neg()}; }
    B2S_HD Fp6 mul_v() const { return {mul_xi(c2), c0, c1}; }   // * v, v^3 = xi
};

// Karatsuba over the three coefficients: 6 Fq2 multiplications
template <class P>
B2S_PAIR_NOINLINE Fp6<P> fp6_mul(const Fp6<P>& a, const Fp6<P>& b) {
    const Fp2<P> t0 = a.c0 * b.c0, t1 = a.c1 * b.c1, t2 = a.c2 * b.c2;
    const Fp2<P> r0 = t0 + mul_xi((a.c1 + a.c2) * (b.c1 + b.c2) - t1 - t2);
    const Fp2<P> r1 = (a.c0 + a.c1) * (b.c0 + b.c1) - t0 - t1 + mul_xi(t2);
    const Fp2<P> r2 = (a.c0 + a.c2) * (b.c0 + b.c2) - t0 - t2 + t1;
    return {r0, r1, r2};
}
// a * (b0 + b1 v): 5 Fq2 multiplications
template <class P>
B2S_PAIR_NOINLINE Fp6<P> fp6_mul_by_01(const Fp6<P>& a, const Fp2<P>& b0, const Fp2<P>& b1) {
    const Fp2<P> t0 = a.c0 * b0, t1 = a.c1 * b1;
    const Fp2<P> r0 = t0 + mul_xi(a.c2 * b1);
    const Fp2<P> r1 = (a.c0 + a.c1) * (b0 + b1) - t0 - t1;
    const Fp2<P> r2 = a.c2 * b0 + t1;
    return {r0, r1, r2};
}
// a * (b1 v)
template <class P>
B2S_HD Fp6<P> fp6_mul_by_1(const Fp6<P>& a, const Fp2<P>& b1) { return {mul_xi(a.c2 * b1), a.c0 * b1, a.c1 * b1}; }
template <class P>
B2S_PAIR_NOINLINE Fp6<P> fp6_inverse(const Fp6<P>& a) {
    const Fp2<P> t0 = a.c0.sqr() - mul_xi(a.c1 * a.c2);
    const Fp2<P> t1 = mul_xi(a.c2.sqr()) - a.c0 * a.c1;
    const Fp2<P> t2 = a.c1.sqr() - a.c0 * a.c2;
    const Fp2<P> n = (a.c0 * t0 + mul_xi(a.c2 * t1 + a.c1 * t2)).inverse();
    return {t0 * n, t1 * n, t2 * n};
}

// ---- Fq12 ----------------------------------------------------------------------------------------------------------
template <class P>
struct Fp12 {
    Fp6<P> c0, c1;
    B2S_HD static Fp12 one() { return {Fp6<P>::one(), Fp6<P>::zero()}; }
    // GT equality: every limb is fully reduced Montgomery form, so equal elements have equal limbs
    B2S_HD bool operator==(const Fp12& o) const { return c0 == o.c0 && c1 == o.c1; }
    B2S_HD bool operator!=(const Fp12& o) const { return !(*this == o); }
    B2S_HD Fp12 conj() const { return {c0, c1.neg()}; }   // f^(p^6); the inverse on the cyclotomic subgroup
};

template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_mul(const Fp12<P>& a, const Fp12<P>& b) {
    const Fp6<P> t0 = fp6_mul(a.c0, b.c0), t1 = fp6_mul(a.c1, b.c1);
    const Fp6<P> r1 = fp6_mul(a.c0 + a.c1, b.c0 + b.c1) - t0 - t1;
    return {t0 + t1.mul_v(), r1};
}
// complex squaring: (a0 + a1 w)^2 = (a0 + a1)(a0 + v a1) - (1 + v) a0 a1 + 2 a0 a1 w
template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_sqr(const Fp12<P>& a) {
    const Fp6<P> ab = fp6_mul(a.c0, a.c1);
    const Fp6<P> s = fp6_mul(a.c0 + a.c1, a.c0 + a.c1.mul_v()) - ab - ab.mul_v();
    return {s, ab + ab};
}
template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_inverse(const Fp12<P>& a) {   // 1 / (a0 + a1 w) = (a0 - a1 w) / (a0^2 - v a1^2); 0 -> 0
    const Fp6<P> n = fp6_inverse(fp6_mul(a.c0, a.c0) - fp6_mul(a.c1, a.c1).mul_v());
    return {fp6_mul(a.c0, n), fp6_mul(a.c1, n).neg()};
}
// f * (l0 + l1 w^2 + l4 w^3): the line of an M-type twist (ark's mul_by_014)
template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_mul_by_014(const Fp12<P>& f, const Fp2<P>& l0, const Fp2<P>& l1, const Fp2<P>& l4) {
    const Fp6<P> t0 = fp6_mul_by_01(f.c0, l0, l1), t1 = fp6_mul_by_1(f.c1, l4);
    const Fp6<P> r1 = fp6_mul_by_01(f.c0 + f.c1, l0, l1 + l4) - t0 - t1;
    return {t0 + t1.mul_v(), r1};
}
// f * (l0 + l3 w + l4 w^3): the line of a D-type twist (ark's mul_by_034)
template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_mul_by_034(const Fp12<P>& f, const Fp2<P>& l0, const Fp2<P>& l3, const Fp2<P>& l4) {
    const Fp6<P> t0 = {f.c0.c0 * l0, f.c0.c1 * l0, f.c0.c2 * l0};
    const Fp6<P> t1 = fp6_mul_by_01(f.c1, l3, l4);
    const Fp6<P> r1 = fp6_mul_by_01(f.c0 + f.c1, l0 + l3, l4) - t0 - t1;
    return {t0 + t1.mul_v(), r1};
}
// f^(p^j), j = 1, 2, 3: the coefficient of w^k becomes conj^j(a_k) xi^(k (p^j - 1) / 6)
template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_frobenius(const Fp12<P>& f, int j) {
    auto m = [&](const Fp2<P>& a, int k) -> Fp2<P> {
        const Fp2<P> g = frob_coeff<P>(j, k);
        if (j == 2) return scale(a, g.c0);   // the p^2 coefficients lie in Fq
        return conj(a) * g;
    };
    const Fp2<P> a0 = (j & 1) ? conj(f.c0.c0) : f.c0.c0;
    return {{a0, m(f.c0.c1, 2), m(f.c0.c2, 4)}, {m(f.c1.c0, 1), m(f.c1.c1, 3), m(f.c1.c2, 5)}};
}
// Squaring in the cyclotomic subgroup (Granger, Scott 2010): three Fq4 squarings over the pairs (w^0, w^3), (w^1, w^4),
// (w^2, w^5); valid only for f with f^(p^6 + 1) = 1 (after the easy part of the final exponentiation).
template <class P>
B2S_HD void fp4_sqr(const Fp2<P>& a, const Fp2<P>& b, Fp2<P>& r0, Fp2<P>& r1) {   // (a + b y)^2, y^2 = xi
    const Fp2<P> a2 = a.sqr(), b2 = b.sqr();
    r0 = mul_xi(b2) + a2;
    r1 = (a + b).sqr() - a2 - b2;
}
template <class P>
B2S_PAIR_NOINLINE Fp12<P> fp12_cyclotomic_sqr(const Fp12<P>& f) {
    using F2 = Fp2<P>;
    F2 t0, t1, t2, t3, t4, t5;
    fp4_sqr(f.c0.c0, f.c1.c1, t0, t1);
    fp4_sqr(f.c1.c0, f.c0.c2, t2, t3);
    fp4_sqr(f.c0.c1, f.c1.c2, t4, t5);
    Fp12<P> r;
    r.c0.c0 = (t0 - f.c0.c0).dbl() + t0;     // 3 t0 - 2 z0
    r.c1.c1 = (t1 + f.c1.c1).dbl() + t1;     // 3 t1 + 2 z1
    const F2 t = mul_xi(t5);
    r.c1.c0 = (t + f.c1.c0).dbl() + t;       // 3 xi t5 + 2 z2
    r.c0.c2 = (t4 - f.c0.c2).dbl() + t4;     // 3 t4 - 2 z3
    r.c0.c1 = (t2 - f.c0.c1).dbl() + t2;     // 3 t2 - 2 z4
    r.c1.c2 = (t3 + f.c1.c2).dbl() + t3;     // 3 t3 + 2 z5
    return r;
}
// f^|x| in the cyclotomic subgroup, and f^x (conjugated when x < 0)
template <class P>
B2S_PAIR_NOINLINE Fp12<P> cyclotomic_exp_x(const Fp12<P>& f) {
    Fp12<P> acc = f;
    bool started = false;
    for (int w = 1; w >= 0; w--) {
        for (int b = 31; b >= 0; b--) {
            if (started) acc = fp12_cyclotomic_sqr(acc);
            if ((P::x_abs(w) >> b) & 1) {
                if (started) acc = fp12_mul(acc, f);
                started = true;
            }
        }
    }
    return P::X_NEG ? acc.conj() : acc;
}
// f^e in the cyclotomic subgroup, e = sum_i words[i] 2^(32 i) (little-endian, not Montgomery); e = 0 gives 1
template <class P>
B2S_PAIR_NOINLINE Fp12<P> cyclotomic_exp(const Fp12<P>& f, const uint32_t* words, int nwords) {
    Fp12<P> acc = Fp12<P>::one();
    bool started = false;
    for (int w = nwords - 1; w >= 0; w--) {
        for (int b = 31; b >= 0; b--) {
            if (started) acc = fp12_cyclotomic_sqr(acc);
            if ((words[w] >> b) & 1) {
                acc = started ? fp12_mul(acc, f) : f;
                started = true;
            }
        }
    }
    return acc;
}

// ---- lines ---------------------------------------------------------------------------------------------------------
template <class P>
struct Line { Fp2<P> c0, c1, c2; };   // ark's EllCoeff order (see the header comment for where P enters)
template <class P>
struct G2Proj { Fp2<P> x, y, z; };     // (X : Y : Z) = (X/Z, Y/Z) on the twist

template <class Curve>
struct PairingShape {
    using P = typename Curve::FqP;
    static constexpr bool M_TWIST = P::M_TWIST;   // BLS12-381: M-type; BN254, BLS12-377: D-type
    static constexpr int digits_nonzero() {
        int n = 0;
        for (int i = 0; i < P::ATE_WORDS; i++) {
            uint32_t v = P::ate_pos(i) | P::ate_neg(i);
            for (; v; v &= v - 1) n++;
        }
        return n;
    }
    // doublings + additions (the top digit starts T = Q) + the two Frobenius lines of BN254
    static constexpr int LINES = (P::ATE_BITS - 1) + (digits_nonzero() - 1) + (P::BLS12_FAMILY ? 0 : 2);
};

// ark's G2Prepared for one fixed Q: the lines in the order the Miller loop consumes them; inf = Q at infinity
template <class Curve>
struct G2Prepared {
    uint32_t inf;
    uint32_t pad[3];
    Line<typename Curve::FqP> ell[PairingShape<Curve>::LINES];
};

template <class P>
B2S_HD Fp2<P> twist_b() {
    Fp2<P> b;
    for (int i = 0; i < Fp<P>::N; i++) { b.c0.v[i] = P::b2c0(i); b.c1.v[i] = P::b2c1(i); }
    return b;
}

// T = 2T and the tangent line at T (Costello, Lange, Naehrig 2010, a = 0).  With the curve equation Y^2 Z = X^3 + b' Z^3
// the tangent, scaled by an Fq2 factor (and w^3 for the M-type twist), is
//   (3 b' Z^2 - Y^2) + 3 X^2 xP [w^2 | w] - 2 Y Z yP [w^3 | 1]   (M | D twist)
template <class Curve>
B2S_PAIR_NOINLINE Line<typename Curve::FqP> dbl_step(G2Proj<typename Curve::FqP>& t) {
    using P = typename Curve::FqP;
    using F2 = Fp2<P>;
    Fp<P> half;
    for (int i = 0; i < Fp<P>::N; i++) half.v[i] = P::fq_half(i);
    const F2 a = scale(t.x * t.y, half);
    const F2 b = t.y.sqr(), c = t.z.sqr();
    const F2 e = twist_b<P>() * (c.dbl() + c);
    const F2 f = e.dbl() + e;
    const F2 g = scale(b + f, half);
    const F2 h = (t.y + t.z).sqr() - (b + c);
    const F2 i = e - b;
    const F2 j = t.x.sqr();
    const F2 e2 = e.sqr();
    t.x = a * (b - f);
    t.y = g.sqr() - (e2.dbl() + e2);
    t.z = b * h;
    if (PairingShape<Curve>::M_TWIST) return {i, j.dbl() + j, h.neg()};
    return {h.neg(), j.dbl() + j, i};
}
// T = T + Q (Q affine) and the line through them: theta = Y - yQ Z, lambda = X - xQ Z give
//   (theta xQ - lambda yQ) - theta xP [w^2 | w] + lambda yP [w^3 | 1]
template <class Curve>
B2S_PAIR_NOINLINE Line<typename Curve::FqP> add_step(G2Proj<typename Curve::FqP>& t, const Affine<Fp2<typename Curve::FqP>>& q) {
    using F2 = Fp2<typename Curve::FqP>;
    const F2 theta = t.y - q.y * t.z, lambda = t.x - q.x * t.z;
    const F2 c = theta.sqr(), d = lambda.sqr();
    const F2 e = lambda * d, f = t.z * c, g = t.x * d;
    const F2 h = e + f - g.dbl();
    t.x = lambda * h;
    t.y = theta * (g - h) - e * t.y;
    t.z = t.z * e;
    const F2 j = theta * q.x - lambda * q.y;
    if (PairingShape<Curve>::M_TWIST) return {j, theta.neg(), lambda};
    return {lambda, theta.neg(), j};
}
// f * (line evaluated at P)
template <class Curve>
B2S_HD Fp12<typename Curve::FqP> ell(const Fp12<typename Curve::FqP>& f, const Line<typename Curve::FqP>& l,
                                     const Affine<Fp<typename Curve::FqP>>& p) {
    if (PairingShape<Curve>::M_TWIST) return fp12_mul_by_014(f, l.c0, scale(l.c1, p.x), scale(l.c2, p.y));
    return fp12_mul_by_034(f, scale(l.c0, p.y), scale(l.c1, p.x), l.c2);
}
// pi(Q) on the twist: (conj(x) cx, conj(y) cy); the psi coefficients of deserialize.cuh are these for BN254 (the
// generator asserts that they equal the p^1 Frobenius coefficients of w^2 and w^3)
template <class P>
B2S_HD Affine<Fp2<P>> twist_frobenius(const Affine<Fp2<P>>& q) {
    Fp2<P> cx, cy;
    for (int i = 0; i < Fp<P>::N; i++) {
        cx.c0.v[i] = P::psi_x0(i); cx.c1.v[i] = P::psi_x1(i);
        cy.c0.v[i] = P::psi_y0(i); cy.c1.v[i] = P::psi_y1(i);
    }
    return {conj(q.x) * cx, conj(q.y) * cy};
}
template <class P>
B2S_HD int ate_digit(int b) {   // digit b of the Miller loop (b = 0 least significant): -1, 0 or 1
    if ((P::ate_pos(b >> 5) >> (b & 31)) & 1) return 1;
    if ((P::ate_neg(b >> 5) >> (b & 31)) & 1) return -1;
    return 0;
}

// Walks the line schedule of one Q: calls emit(line) in the order the Miller loop consumes lines.
template <class Curve, class Emit>
B2S_HD void line_schedule(const Affine<Fp2<typename Curve::FqP>>& q, Emit&& emit) {
    using P = typename Curve::FqP;
    G2Proj<P> t{q.x, q.y, Fp2<P>::one()};
    const Affine<Fp2<P>> qn = q.neg();
    for (int b = P::ATE_BITS - 2; b >= 0; b--) {
        emit(dbl_step<Curve>(t));
        const int d = ate_digit<P>(b);
        if (d) emit(add_step<Curve>(t, d > 0 ? q : qn));
    }
    if (!P::BLS12_FAMILY) {
        const Affine<Fp2<P>> q1 = twist_frobenius(q);
        emit(add_step<Curve>(t, q1));
        emit(add_step<Curve>(t, twist_frobenius(q1).neg()));
    }
}

template <class Curve>
B2S_HD void g2_prepare(const Affine<Fp2<typename Curve::FqP>>& q, G2Prepared<Curve>& out) {
    out.inf = q.is_inf() ? 1u : 0u;
    int n = 0;
    if (q.is_inf()) return;
    line_schedule<Curve>(q, [&](const Line<typename Curve::FqP>& l) { out.ell[n++] = l; });
}

// prod_i f_i(P_i): NF pairs with lines computed on the fly (pf[i], qf[i]) and NP pairs with prepared lines (pp[i], prep[i]);
// one Fq12 squaring per step for all of them.  Not yet final-exponentiated.
template <class Curve, int NF, int NP>
B2S_PAIR_NOINLINE Fp12<typename Curve::FqP> multi_miller_loop(const Affine<Fp<typename Curve::FqP>>* pf,
                                                             const Affine<Fp2<typename Curve::FqP>>* qf,
                                                             const Affine<Fp<typename Curve::FqP>>* pp,
                                                             const G2Prepared<Curve>* const* prep) {
    using P = typename Curve::FqP;
    Fp12<P> f = Fp12<P>::one();
    G2Proj<P> t[NF > 0 ? NF : 1];
    bool live_f[NF > 0 ? NF : 1], live_p[NP > 0 ? NP : 1];
    for (int i = 0; i < NF; i++) {
        t[i] = {qf[i].x, qf[i].y, Fp2<P>::one()};
        live_f[i] = !pf[i].is_inf() && !qf[i].is_inf();
    }
    for (int i = 0; i < NP; i++) live_p[i] = !pp[i].is_inf() && !prep[i]->inf;
    int li = 0;
    auto prepared = [&]() {
        for (int i = 0; i < NP; i++)
            if (live_p[i]) f = ell<Curve>(f, prep[i]->ell[li], pp[i]);
        li++;
    };
    for (int b = P::ATE_BITS - 2; b >= 0; b--) {
        if (b != P::ATE_BITS - 2) f = fp12_sqr(f);
        for (int i = 0; i < NF; i++) {
            const Line<P> l = dbl_step<Curve>(t[i]);
            if (live_f[i]) f = ell<Curve>(f, l, pf[i]);
        }
        prepared();
        const int d = ate_digit<P>(b);
        if (d) {
            for (int i = 0; i < NF; i++) {
                const Line<P> l = add_step<Curve>(t[i], d > 0 ? qf[i] : qf[i].neg());
                if (live_f[i]) f = ell<Curve>(f, l, pf[i]);
            }
            prepared();
        }
    }
    if (!P::BLS12_FAMILY) {
        for (int i = 0; i < NF; i++) {
            const Affine<Fp2<P>> q1 = twist_frobenius(qf[i]);
            const Line<P> l1 = add_step<Curve>(t[i], q1);
            const Line<P> l2 = add_step<Curve>(t[i], twist_frobenius(q1).neg());
            if (live_f[i]) f = ell<Curve>(ell<Curve>(f, l1, pf[i]), l2, pf[i]);
        }
        prepared();
        prepared();
    }
    return P::X_NEG ? f.conj() : f;
}

template <class P>
B2S_PAIR_NOINLINE Fp12<P> final_exponentiation(const Fp12<P>& f) {
    // easy part: f^((p^6 - 1)(p^2 + 1)); afterwards f lies in the cyclotomic subgroup
    Fp12<P> e = fp12_mul(f.conj(), fp12_inverse(f));
    e = fp12_mul(fp12_frobenius(e, 2), e);
    if (P::BLS12_FAMILY) {   // BLS12-381, BLS12-377: e^((x - 1)^2 (x + p)(x^2 + p^2 - 1) + 3)
        Fp12<P> t = fp12_mul(cyclotomic_exp_x(e), e.conj());        // e^(x - 1)
        t = fp12_mul(cyclotomic_exp_x(t), t.conj());                  // e^((x - 1)^2)
        t = fp12_mul(cyclotomic_exp_x(t), fp12_frobenius(t, 1));      // ^(x + p)
        t = fp12_mul(fp12_mul(cyclotomic_exp_x(cyclotomic_exp_x(t)), fp12_frobenius(t, 2)), t.conj());   // ^(x^2 + p^2 - 1)
        return fp12_mul(t, fp12_mul(fp12_cyclotomic_sqr(e), e));      // * e^3
    }
    // BN254: e^(l0 + l1 p + l2 p^2 + l3 p^3)
    const Fp12<P> fx = cyclotomic_exp_x(e);
    const Fp12<P> f2x = fp12_cyclotomic_sqr(fx);
    const Fp12<P> f6x = fp12_mul(fp12_cyclotomic_sqr(f2x), f2x);
    const Fp12<P> f6x2 = cyclotomic_exp_x(f6x);
    const Fp12<P> f12x3 = cyclotomic_exp_x(fp12_cyclotomic_sqr(f6x2));
    const Fp12<P> a = fp12_mul(fp12_mul(f12x3, f6x2), f6x);      // l2 = 12x^3 + 6x^2 + 6x
    const Fp12<P> b = fp12_mul(a, f2x.conj());                      // l1 = 12x^3 + 6x^2 + 4x
    Fp12<P> r = fp12_mul(fp12_mul(a, f6x2), e);                     // l0 = l2 + 6x^2 + 1
    r = fp12_mul(r, fp12_frobenius(b, 1));
    r = fp12_mul(r, fp12_frobenius(a, 2));
    return fp12_mul(r, fp12_frobenius(fp12_mul(b, e.conj()), 3));   // l3 = l1 - 1
}

template <class Curve>
B2S_HD Fp12<typename Curve::FqP> pairing(const Affine<Fp<typename Curve::FqP>>& p, const Affine<Fp2<typename Curve::FqP>>& q) {
    return final_exponentiation(multi_miller_loop<Curve, 1, 0>(&p, &q, nullptr, nullptr));
}

// The Groth16 verdict of one proof, in two halves (the verify kernels keep f in memory between them):
//   e(A, B) * e(IC, -gamma) * e(C, -delta) == e(alpha, beta), with -gamma and -delta prepared.
template <class Curve>
B2S_HD Fp12<typename Curve::FqP> groth16_miller(const Affine<Fp<typename Curve::FqP>>& a, const Affine<Fp2<typename Curve::FqP>>& b,
                                                const Affine<Fp<typename Curve::FqP>>& ic, const Affine<Fp<typename Curve::FqP>>& c,
                                                const G2Prepared<Curve>* neg_gamma, const G2Prepared<Curve>* neg_delta) {
    const Affine<Fp<typename Curve::FqP>> pp[2] = {ic, c};
    const G2Prepared<Curve>* prep[2] = {neg_gamma, neg_delta};
    return multi_miller_loop<Curve, 1, 2>(&a, &b, pp, prep);
}
template <class Curve>
B2S_HD bool groth16_verdict(const Affine<Fp<typename Curve::FqP>>& a, const Affine<Fp2<typename Curve::FqP>>& b,
                            const Affine<Fp<typename Curve::FqP>>& ic, const Affine<Fp<typename Curve::FqP>>& c,
                            const G2Prepared<Curve>* neg_gamma, const G2Prepared<Curve>* neg_delta,
                            const Fp12<typename Curve::FqP>& alpha_beta) {
    return final_exponentiation(groth16_miller<Curve>(a, b, ic, c, neg_gamma, neg_delta)) == alpha_beta;
}

// The random-linear-combination check of many proofs under one key (verify_rlc.cu), with caller-drawn nonzero 128-bit
// rho_i:
//   prod_i e(rho_i A_i, B_i) * e(IC*, -gamma) * e(C*, -delta) == e(alpha, beta)^S,
//   S = sum_i rho_i,  C* = sum_i rho_i C_i,  IC* = S gamma_abc[0] + sum_j (sum_i rho_i x_ij) gamma_abc[j+1]  (mod r).
// It holds for valid proofs because every factor goes through the same final exponentiation.  If a proof is invalid, at
// most one rho_i < 2^128 < r (the others fixed) passes, since GT has prime order r.
//
// One thread's share of the left side: prod_j f_{rho_j A_j, B_j}, NF proofs, rho as 4 little-endian words per proof.
// rho_j A_j is made affine with one Fq inversion.  Pairs with A or B at infinity (the padding of a last partial group)
// contribute 1.  Not yet final-exponentiated.
template <class Curve, int NF>
B2S_PAIR_NOINLINE Fp12<typename Curve::FqP> rlc_miller(const Affine<Fp<typename Curve::FqP>>* a,
                                                      const Affine<Fp2<typename Curve::FqP>>* b, const uint32_t* rho) {
    Affine<Fp<typename Curve::FqP>> p[NF];
    for (int i = 0; i < NF; i++) p[i] = scalar_mul_words(Curve::G1::from_affine(a[i]), rho + 4 * i, 4).to_affine();
    return multi_miller_loop<Curve, NF, 0>(p, b, nullptr, nullptr);
}
// The verdict: f = the product of every rlc_miller value, ic = IC*, c = C* (affine), s = S (8 canonical words)
template <class Curve>
B2S_PAIR_NOINLINE bool rlc_verdict(const Fp12<typename Curve::FqP>& f, const Affine<Fp<typename Curve::FqP>>& ic,
                                   const Affine<Fp<typename Curve::FqP>>& c, const G2Prepared<Curve>* neg_gamma,
                                   const G2Prepared<Curve>* neg_delta, const Fp12<typename Curve::FqP>& alpha_beta, const uint32_t* s) {
    const Affine<Fp<typename Curve::FqP>> pp[2] = {ic, c};
    const G2Prepared<Curve>* prep[2] = {neg_gamma, neg_delta};
    const Fp12<typename Curve::FqP> g = fp12_mul(f, multi_miller_loop<Curve, 0, 2>(nullptr, nullptr, pp, prep));
    return final_exponentiation(g) == cyclotomic_exp(alpha_beta, s, 8);
}

}  // namespace b2s
