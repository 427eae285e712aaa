// Prime-field arithmetic on 32-bit limbs for sm_90a.
//
// Replaces (on the GPU) what ark-ff's `Fp<MontBackend<_, N>>` does on the CPU for the prover hot
// path (upstream crate, not in /root/reference; call sites: relations/src/utils/matrix.rs:31,
// relations/src/sr1cs/mod.rs:42-46, relations/src/gr1cs/assignment.rs:48).  Elements are kept in
// Montgomery form with R = 2^(32*N) -- bit-identical to ark-ff's in-memory little-endian u64 limbs
// (R = 2^(64*N/2)) -- and always fully reduced to [0, p).
//
// Multiplication is word-serial Montgomery (CIOS) with the partial products split over two
// accumulators: products a_j*b_i with even j land on limb pairs (j, j+1) of `E`, products with odd
// j on limb pairs of `O`, which carries one limb more weight.  Each of the two accumulations is a
// single carry chain of mad.lo.cc / madc.hi.cc pairs; ptxas fuses every pair into ONE
// `IMAD.WIDE.U32.X Rd, P0, Ra, Rb, Rc, P0` (checked with cuobjdump), so a row costs N wide IMADs
// for a*b_i and N for m*p.  The one-limb right shift of CIOS is free: `O` becomes the next `E`.
//
// Everything here is __host__ __device__: on the host the PTX carry flag is emulated, so the same
// limb schedule is exercised by the CPU unit tests (tests/test_host_ff.py) before it ever reaches a
// GPU.  The host path exists for tests and tiny host-side constants only; no product entry point
// computes on the CPU.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define B2S_HD __host__ __device__ __forceinline__
#define B2S_D __device__ __forceinline__
// Montgomery multiplication is ~300 (8 limbs) / ~650 (12 limbs) instructions.  Inlining it at every use
// is right for the hot kernels (bucket accumulation, NTT butterflies) but makes the cold ones -- scalar
// multiplications, G2 tails, test kernels -- take tens of minutes to compile, so a translation unit
// opts in with B2S_INLINE_MUL; elsewhere the multiplication is one out-of-line function per field.
#if defined(B2S_INLINE_MUL)
#define B2S_MUL_ATTR __host__ __device__ __forceinline__
#else
#define B2S_MUL_ATTR __host__ __device__ __noinline__
#endif
#else
#define B2S_HD inline
#define B2S_D inline
#define B2S_MUL_ATTR inline
#endif

namespace b2s {

// ------------------------------------------------------------------------------------------
// carry-chain primitives
// ------------------------------------------------------------------------------------------
namespace cc {
#if defined(__CUDA_ARCH__)
B2S_D uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2S_D uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2S_D uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2S_D uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2S_D uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2S_D uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0,%1,%2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
B2S_D uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2S_D uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2S_D uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2S_D uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0,%1,%2,%3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
B2S_D uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
B2S_D uint32_t mul_hi(uint32_t a, uint32_t b) { return __umulhi(a, b); }
// x, through an identity byte permutation that ptxas does not see through (see redc_row)
B2S_D uint32_t opaque(uint32_t x) { uint32_t r; asm volatile("prmt.b32 %0,%1,0,0x3210;" : "=r"(r) : "r"(x)); return r; }
#else
// Host emulation of the PTX condition-code register (tests only).
inline uint32_t& cf() { static thread_local uint32_t f = 0; return f; }
inline uint32_t add3_(uint32_t a, uint32_t b, uint32_t cin, bool set) {
    uint64_t s = (uint64_t)a + b + cin;
    if (set) cf() = (uint32_t)(s >> 32);
    return (uint32_t)s;
}
inline uint32_t sub3_(uint32_t a, uint32_t b, uint32_t bin, bool set) {
    uint64_t s = (uint64_t)a - b - bin;
    if (set) cf() = (uint32_t)((s >> 32) & 1);  // borrow
    return (uint32_t)s;
}
inline uint32_t add_cc(uint32_t a, uint32_t b) { return add3_(a, b, 0, true); }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { return add3_(a, b, cf(), true); }
inline uint32_t addc(uint32_t a, uint32_t b) { return add3_(a, b, cf(), false); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { return sub3_(a, b, 0, true); }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { return sub3_(a, b, cf(), true); }
inline uint32_t subc(uint32_t a, uint32_t b) { return sub3_(a, b, cf(), false); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return (uint32_t)((uint64_t)a * b); }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return add3_(mul_lo(a, b), c, 0, true); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return add3_(mul_lo(a, b), c, cf(), true); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return add3_(mul_hi(a, b), c, cf(), true); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return add3_(mul_hi(a, b), c, cf(), false); }
inline uint32_t opaque(uint32_t x) { return x; }
#endif
}  // namespace cc

// ------------------------------------------------------------------------------------------
// Field element.  `P` supplies: N (even), and constexpr functions mod(i), r1(i) [R mod p],
// r2(i) [R^2 mod p], and NINV = -p^-1 mod 2^32  (generated: field_params.h).
// ------------------------------------------------------------------------------------------
template <class P>
struct Fp {
    static constexpr int N = P::N;
    uint32_t v[N];

    B2S_HD static Fp zero() {
        Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = 0;
        return r;
    }
    B2S_HD static Fp one() {  // Montgomery form of 1
        Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = P::r1(i);
        return r;
    }
    B2S_HD static Fp r2() {
        Fp r;
#pragma unroll
        for (int i = 0; i < N; i++) r.v[i] = P::r2(i);
        return r;
    }
    B2S_HD bool is_zero() const {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= v[i];
        return t == 0;
    }
    B2S_HD bool operator==(const Fp& o) const {
        uint32_t t = 0;
#pragma unroll
        for (int i = 0; i < N; i++) t |= v[i] ^ o.v[i];
        return t == 0;
    }
    B2S_HD bool operator!=(const Fp& o) const { return !(*this == o); }

    // r = (x >= p) ? x - p : x, where x = (carry:t) may exceed 2^(32N) by the carry bit.
    B2S_HD static void cond_sub_p(uint32_t t[N], uint32_t carry) {
        uint32_t d[N];
        d[0] = cc::sub_cc(t[0], P::mod(0));
#pragma unroll
        for (int i = 1; i < N; i++) d[i] = cc::subc_cc(t[i], P::mod(i));
        uint32_t borrow = cc::subc(0, 0);  // 0 or 0xffffffff
        // keep t iff the subtraction borrowed and there was no carry limb to absorb it
        bool keep = (borrow != 0) && (carry == 0);
#pragma unroll
        for (int i = 0; i < N; i++) t[i] = keep ? t[i] : d[i];
    }

    B2S_HD friend Fp operator+(const Fp& a, const Fp& b) {
        Fp r;
        r.v[0] = cc::add_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < N; i++) r.v[i] = cc::addc_cc(a.v[i], b.v[i]);
        uint32_t carry = P::SPARE_BITS > 0 ? 0u : cc::addc(0, 0);
        cond_sub_p(r.v, carry);
        return r;
    }
    B2S_HD friend Fp operator-(const Fp& a, const Fp& b) {
        Fp r;
        r.v[0] = cc::sub_cc(a.v[0], b.v[0]);
#pragma unroll
        for (int i = 1; i < N; i++) r.v[i] = cc::subc_cc(a.v[i], b.v[i]);
        uint32_t borrow = cc::subc(0, 0);  // 0 or all-ones
        // add p back under the borrow mask
        r.v[0] = cc::add_cc(r.v[0], P::mod(0) & borrow);
#pragma unroll
        for (int i = 1; i < N - 1; i++) r.v[i] = cc::addc_cc(r.v[i], P::mod(i) & borrow);
        r.v[N - 1] = cc::addc(r.v[N - 1], P::mod(N - 1) & borrow);
        return r;
    }
    B2S_HD Fp neg() const {
        if (is_zero()) return *this;
        Fp r;
        r.v[0] = cc::sub_cc(P::mod(0), v[0]);
#pragma unroll
        for (int i = 1; i < N - 1; i++) r.v[i] = cc::subc_cc(P::mod(i), v[i]);
        r.v[N - 1] = cc::subc(P::mod(N - 1), v[N - 1]);
        return r;
    }
    B2S_HD Fp dbl() const { return *this + *this; }

    // ---- Montgomery multiplication ----------------------------------------------------
    // The last limb of each carry chain is written after its loop, not selected inside it: a choice between two volatile
    // asm statements in the loop body keeps the sm_90a compiler from unrolling the loop, and E / O then live in local memory.
    // One reduction step on (E, O): add m*p with m = E[0] * NINV so that E[0] becomes 0.
    B2S_HD static void redc_row(uint32_t E[N], uint32_t O[N]) {
        if (P::LOW64_IS_2_64_MINUS_2_32_PLUS_1) {
            // p = ... 0xffffffff 0x00000001 (BLS12-381 Fr): NINV = -1, so m = -E[0]; m*p_0 = m and
            // m*p_1 = (m << 32) - m.  Doing these two limbs with plain adds keeps ptxas from
            // strength-reducing the immediates (which un-fuses the whole IMAD.WIDE chain) and moves
            // them from the fma pipe to the otherwise idle alu pipe.
            const uint32_t e0 = E[0];
            const uint32_t m = 0u - e0;
            const uint32_t nz = (e0 != 0u) ? 1u : 0u;
            // odd chain: limb 1 product is (lo = e0, hi = m - nz)
            O[0] = cc::add_cc(O[0], e0);
            O[1] = cc::addc_cc(O[1], m - nz);
#pragma unroll
            for (int j = 3; j < N - 1; j += 2) {
                O[j - 1] = cc::madc_lo_cc(P::mod(j), m, O[j - 1]);
                O[j] = cc::madc_hi_cc(P::mod(j), m, O[j]);
            }
            O[N - 2] = cc::madc_lo_cc(P::mod(N - 1), m, O[N - 2]);
            O[N - 1] = cc::madc_hi(P::mod(N - 1), m, O[N - 1]);
            // even chain: limb 0 product is (lo = m, hi = 0); e0 + m == 0 mod 2^32 with carry nz
            E[0] = 0u;
            E[1] = cc::add_cc(E[1], nz);
#pragma unroll
            for (int j = 2; j < N; j += 2) {
                E[j] = cc::madc_lo_cc(P::mod(j), m, E[j]);
                E[j + 1] = cc::madc_hi_cc(P::mod(j), m, E[j + 1]);
            }
            O[N - 1] = cc::addc(O[N - 1], 0);
            return;
        }
        // NINV = -1 (p = 1 mod 2^32: BLS12-377 Fq and Fr): m = -E[0].  Seen as a negation, that m makes ptxas split every
        // fused IMAD.WIDE.U32.X of the chains below into IMAD.HI.U32.X + IMAD.X (an inlined 12-limb product: 952 instead of
        // 832 instructions), so the negation goes through cc::opaque.
        const uint32_t m = P::NINV == 0xffffffffu ? cc::opaque(0u - E[0]) : cc::mul_lo(E[0], P::NINV);
        // odd limbs of p -> O
        O[0] = cc::mad_lo_cc(P::mod(1), m, O[0]);
        O[1] = cc::madc_hi_cc(P::mod(1), m, O[1]);
#pragma unroll
        for (int j = 3; j < N - 1; j += 2) {
            O[j - 1] = cc::madc_lo_cc(P::mod(j), m, O[j - 1]);
            O[j] = cc::madc_hi_cc(P::mod(j), m, O[j]);
        }
        O[N - 2] = cc::madc_lo_cc(P::mod(N - 1), m, O[N - 2]);
        O[N - 1] = cc::madc_hi(P::mod(N - 1), m, O[N - 1]);
        // even limbs of p -> E, carry out lands on O[N-1]
        E[0] = cc::mad_lo_cc(P::mod(0), m, E[0]);
        E[1] = cc::madc_hi_cc(P::mod(0), m, E[1]);
#pragma unroll
        for (int j = 2; j < N; j += 2) {
            E[j] = cc::madc_lo_cc(P::mod(j), m, E[j]);
            E[j + 1] = cc::madc_hi_cc(P::mod(j), m, E[j + 1]);
        }
        O[N - 1] = cc::addc(O[N - 1], 0);
    }

    B2S_MUL_ATTR friend Fp operator*(const Fp& a, const Fp& b) {
        uint32_t E[N], O[N];
        // row 0: plain products
        {
            const uint32_t bi = b.v[0];
#pragma unroll
            for (int j = 0; j < N; j += 2) {
                E[j] = cc::mul_lo(a.v[j], bi);
                E[j + 1] = cc::mul_hi(a.v[j], bi);
                O[j] = cc::mul_lo(a.v[j + 1], bi);
                O[j + 1] = cc::mul_hi(a.v[j + 1], bi);
            }
            redc_row(E, O);
        }
#pragma unroll
        for (int i = 1; i < N; i++) {
            const uint32_t bi = b.v[i];
            uint32_t E2[N], O2[N];
            // drop the (now zero) limb E[0]: the old O is the new even-aligned accumulator, the
            // old E[2..] the new odd-aligned one; E[1] is folded in with its carry feeding O2.
            E2[0] = cc::add_cc(O[0], E[1]);
#pragma unroll
            for (int j = 1; j < N - 1; j += 2) {
                O2[j - 1] = cc::madc_lo_cc(a.v[j], bi, E[j + 1]);
                O2[j] = cc::madc_hi_cc(a.v[j], bi, E[j + 2]);
            }
            O2[N - 2] = cc::madc_lo_cc(a.v[N - 1], bi, 0u);
            O2[N - 1] = cc::madc_hi(a.v[N - 1], bi, 0u);
            E2[0] = cc::mad_lo_cc(a.v[0], bi, E2[0]);
            E2[1] = cc::madc_hi_cc(a.v[0], bi, O[1]);
#pragma unroll
            for (int j = 2; j < N; j += 2) {
                E2[j] = cc::madc_lo_cc(a.v[j], bi, O[j]);
                E2[j + 1] = cc::madc_hi_cc(a.v[j], bi, O[j + 1]);
            }
            O2[N - 1] = cc::addc(O2[N - 1], 0);
            redc_row(E2, O2);
#pragma unroll
            for (int k = 0; k < N; k++) {
                E[k] = E2[k];
                O[k] = O2[k];
            }
        }
        // merge: result = O + (E >> 32)
        Fp r;
        r.v[0] = cc::add_cc(O[0], E[1]);
#pragma unroll
        for (int k = 1; k < N - 1; k++) r.v[k] = cc::addc_cc(O[k], E[k + 1]);
        r.v[N - 1] = cc::addc(O[N - 1], 0);
        cond_sub_p(r.v, 0);
        return r;
    }
    B2S_HD Fp sqr() const { return (*this) * (*this); }

    B2S_HD Fp& operator+=(const Fp& o) { *this = *this + o; return *this; }
    B2S_HD Fp& operator-=(const Fp& o) { *this = *this - o; return *this; }
    B2S_HD Fp& operator*=(const Fp& o) { *this = *this * o; return *this; }

    // Montgomery <-> canonical
    B2S_HD Fp to_mont() const { return (*this) * r2(); }
    B2S_HD Fp from_mont() const {
        Fp o = zero();
        o.v[0] = 1;
        return (*this) * o;
    }

    // x^e for a small exponent array (little-endian 32-bit words), square-and-multiply.
    B2S_HD Fp pow_words(const uint32_t* e, int nwords) const {
        Fp acc = one();
        bool started = false;
        for (int w = nwords - 1; w >= 0; w--) {
            for (int b = 31; b >= 0; b--) {
                if (started) acc = acc.sqr();
                if ((e[w] >> b) & 1) {
                    acc = started ? acc * (*this) : (*this);
                    started = true;
                }
            }
        }
        return acc;
    }
    B2S_HD Fp pow_u64(uint64_t e) const {
        uint32_t w[2] = {(uint32_t)e, (uint32_t)(e >> 32)};
        return pow_words(w, 2);
    }
    // ---- inversion by divsteps ---------------------------------------------------------
    // Bernstein and Yang, "Fast constant-time gcd computation and modular inversion" (TCHES 2019).  With delta = 1,
    // f = p (odd), g = x, one divstep is
    //     (delta, f, g) -> (1 - delta, g, (g - f) / 2)             if delta > 0 and g is odd,
    //                      (1 + delta, f, (g + (g mod 2) f) / 2)   otherwise,
    // and by their Theorem 11.2 g reaches 0, with f = +-gcd(p, x) = +-1, within floor((49 d + 57) / 17) divsteps for
    // p < 2^d, d >= 46: 1101 / 738 / 735 for d = 381 / 255 / 254.  The count is fixed, and every step is the same
    // masked instruction sequence, so the time does not depend on x (the setup inverts secrets) and the lanes of a
    // warp never diverge.
    //   The steps run in batches of 30 on the low limb of f and g alone (step i needs bit i of the inputs only); a
    // batch yields the integer matrix T with 2^30 (f', g') = T (f, g), |u| + |v|, |q| + |r| <= 2^30, which is then
    // applied to the full f, g and to the Bezout coefficients d, e (d x = f mod p), dividing by 2^30 exactly mod p.
    // All of them live in signed 30-bit limbs so that the 32 x 32 -> 64-bit products of T with a limb never overflow.
    // At the end d = +-x^-1; for a Montgomery input x = a R that is a^-1 R^-1, and one product with R^3 mod p gives
    // the Montgomery form a^-1 R.  0 -> 0 (g starts at 0, d stays 0).
    static constexpr int IL = P::INV_LIMBS;
    static constexpr int32_t M30 = (1 << 30) - 1;
    static constexpr int DIVSTEPS = (49 * P::BITS + 57) / 17;
    static_assert(P::BITS >= 46, "the divstep bound used here holds for d >= 46");

    // 30 divsteps on the low limbs f0, g0; returns delta, T = (u, v, q, r) in t
    B2S_HD static int32_t divsteps30(int32_t delta, uint32_t f, uint32_t g, int32_t t[4]) {
        uint32_t u = 1, v = 0, q = 0, r = 1;  // 2^i (f_i, g_i) = (u f + v g, q f + r g), two's complement
#pragma unroll
        for (int i = 0; i < 30; i++) {
            // m = all ones iff delta > 0 and g odd: then (delta, f, g) -> (-delta, g, -f), and the rows of T alike
            const uint32_t m = (uint32_t)((-delta) >> 31) & (0u - (g & 1u));
            uint32_t x = (f ^ g) & m;
            f ^= x; g ^= x; g = (g ^ m) - m;
            x = (u ^ q) & m;
            u ^= x; q ^= x; q = (q ^ m) - m;
            x = (v ^ r) & m;
            v ^= x; r ^= x; r = (r ^ m) - m;
            delta = (int32_t)(((uint32_t)delta ^ m) - m) + 1;
            // g odd (always so after a swap): g += f; then g /= 2, which the f row pays for by doubling
            const uint32_t odd = 0u - (g & 1u);
            g += f & odd; q += u & odd; r += v & odd;
            g >>= 1; u <<= 1; v <<= 1;
        }
        t[0] = (int32_t)u; t[1] = (int32_t)v; t[2] = (int32_t)q; t[3] = (int32_t)r;
        return delta;
    }

    // (f, g) <- T (f, g) / 2^30, exact; limbs 0..IL-2 end in [0, 2^30), the top limb carries the sign
    B2S_HD static void inv_update_fg(int32_t f[IL], int32_t g[IL], const int32_t t[4]) {
        const int32_t u = t[0], v = t[1], q = t[2], r = t[3];
        int64_t cf = (int64_t)u * f[0] + (int64_t)v * g[0], cg = (int64_t)q * f[0] + (int64_t)r * g[0];
        cf >>= 30; cg >>= 30;
#pragma unroll
        for (int i = 1; i < IL; i++) {
            cf += (int64_t)u * f[i] + (int64_t)v * g[i];
            cg += (int64_t)q * f[i] + (int64_t)r * g[i];
            f[i - 1] = (int32_t)cf & M30; g[i - 1] = (int32_t)cg & M30;
            cf >>= 30; cg >>= 30;
        }
        f[IL - 1] = (int32_t)cf; g[IL - 1] = (int32_t)cg;
    }

    // (d, e) <- (T (d, e) + (md, me) p) / 2^30, with md, me chosen so the division is exact; d, e stay in (-2p, p):
    // a negative input first gets p added through the matrix ((u & sd) + (v & se) multiples of p), which puts T (d, e)
    // in (-2^30 p, 2^30 p), and the exactness term subtracts less than 2^30 p
    B2S_HD static void inv_update_de(int32_t d[IL], int32_t e[IL], const int32_t t[4]) {
        const int32_t u = t[0], v = t[1], q = t[2], r = t[3];
        const int32_t sd = d[IL - 1] >> 31, se = e[IL - 1] >> 31;
        int32_t md = (u & sd) + (v & se), me = (q & sd) + (r & se);
        int64_t cd = (int64_t)u * d[0] + (int64_t)v * e[0], ce = (int64_t)q * d[0] + (int64_t)r * e[0];
        md -= (int32_t)((P::INV_PINV30 * (uint32_t)cd + (uint32_t)md) & (uint32_t)M30);
        me -= (int32_t)((P::INV_PINV30 * (uint32_t)ce + (uint32_t)me) & (uint32_t)M30);
        cd += (int64_t)P::inv_mod30(0) * md; ce += (int64_t)P::inv_mod30(0) * me;
        cd >>= 30; ce >>= 30;
#pragma unroll
        for (int i = 1; i < IL; i++) {
            cd += (int64_t)u * d[i] + (int64_t)v * e[i] + (int64_t)P::inv_mod30(i) * md;
            ce += (int64_t)q * d[i] + (int64_t)r * e[i] + (int64_t)P::inv_mod30(i) * me;
            d[i - 1] = (int32_t)cd & M30; e[i - 1] = (int32_t)ce & M30;
            cd >>= 30; ce >>= 30;
        }
        d[IL - 1] = (int32_t)cd; e[IL - 1] = (int32_t)ce;
    }

    // carries of a signed-30 number: limbs 0..IL-2 into [0, 2^30), the sign into the top limb
    B2S_HD static void carry30(int32_t d[IL]) {
        int32_t c = 0;
#pragma unroll
        for (int i = 0; i < IL - 1; i++) {
            c += d[i];
            d[i] = c & M30;
            c >>= 30;
        }
        d[IL - 1] += c;
    }
    // d + (p & mask), carried
    B2S_HD static void add_p30(int32_t d[IL], int32_t mask) {
#pragma unroll
        for (int i = 0; i < IL; i++) d[i] += P::inv_mod30(i) & mask;
        carry30(d);
    }

    B2S_HD Fp inverse() const {
        int32_t f[IL], g[IL], d[IL], e[IL];
#pragma unroll
        for (int i = 0; i < IL; i++) {
            const int b = 30 * i, w = b / 32, o = b % 32;
            uint32_t x = w < N ? v[w] >> o : 0u;
            if (o > 2 && w + 1 < N) x |= v[w + 1] << (32 - o);
            f[i] = P::inv_mod30(i);
            g[i] = (int32_t)(x & (uint32_t)M30);
            d[i] = 0;
            e[i] = i == 0;
        }
        int32_t delta = 1;
#pragma unroll 1
        for (int s = 0; s < DIVSTEPS; s += 30) {
            int32_t t[4];
            delta = divsteps30(delta, (uint32_t)f[0], (uint32_t)g[0], t);
            inv_update_de(d, e, t);
            inv_update_fg(f, g, t);
        }
        // f = +-1: d = +-x^-1 in (-2p, p); take the sign of f, then bring d into [0, p)
        const int32_t sf = f[IL - 1] >> 31;
#pragma unroll
        for (int i = 0; i < IL; i++) d[i] = (d[i] ^ sf) - sf;
        carry30(d);
        add_p30(d, d[IL - 1] >> 31);
        add_p30(d, d[IL - 1] >> 31);
        int32_t t[IL];
#pragma unroll
        for (int i = 0; i < IL; i++) t[i] = d[i] - P::inv_mod30(i);
        carry30(t);
        const int32_t keep = t[IL - 1] >> 31;  // d < p
#pragma unroll
        for (int i = 0; i < IL; i++) d[i] = (d[i] & keep) | (t[i] & ~keep);
        Fp r, c;
        uint64_t acc = 0;
        int bits = 0, w = 0;
#pragma unroll
        for (int i = 0; i < IL; i++) {
            acc |= (uint64_t)(uint32_t)d[i] << bits;
            bits += 30;
            if (bits >= 32 && w < N) {
                r.v[w++] = (uint32_t)acc;
                acc >>= 32;
                bits -= 32;
            }
        }
#pragma unroll
        for (int i = 0; i < N; i++) c.v[i] = P::inv_final(i);
        return r * c;
    }
};

// ------------------------------------------------------------------------------------------
// Quadratic extension Fq2 = Fq[u]/(u^2 - P::FQ2_NR): -1 for BLS12-381 and BN254, -5 for BLS12-377.
// ------------------------------------------------------------------------------------------
template <class P>
struct Fp2 {
    using B = Fp<P>;
    static_assert(P::FQ2_NR == -1 || P::FQ2_NR == -5, "u^2 = -1 or -5");
    B c0, c1;
    B2S_HD static Fp2 zero() { return {B::zero(), B::zero()}; }
    B2S_HD static Fp2 one() { return {B::one(), B::zero()}; }
    B2S_HD bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    B2S_HD bool operator==(const Fp2& o) const { return c0 == o.c0 && c1 == o.c1; }
    B2S_HD bool operator!=(const Fp2& o) const { return !(*this == o); }
    B2S_HD friend Fp2 operator+(const Fp2& a, const Fp2& b) { return {a.c0 + b.c0, a.c1 + b.c1}; }
    B2S_HD friend Fp2 operator-(const Fp2& a, const Fp2& b) { return {a.c0 - b.c0, a.c1 - b.c1}; }
    B2S_HD Fp2 neg() const { return {c0.neg(), c1.neg()}; }
    B2S_HD Fp2 dbl() const { return {c0.dbl(), c1.dbl()}; }
    // 5 a: two doublings and an add (u^2 = -5)
    B2S_HD static B times5(const B& a) { return a.dbl().dbl() + a; }
    // Karatsuba: 3 base multiplications; c0 = t0 + FQ2_NR t1
    B2S_HD friend Fp2 operator*(const Fp2& a, const Fp2& b) {
        B t0 = a.c0 * b.c0;
        B t1 = a.c1 * b.c1;
        B t2 = (a.c0 + a.c1) * (b.c0 + b.c1);
        if constexpr (P::FQ2_NR == -1) return {t0 - t1, t2 - t0 - t1};
        else return {t0 - times5(t1), t2 - t0 - t1};
    }
    // u^2 = -1: (c0 + c1 u)^2 = (c0 + c1)(c0 - c1) + 2 c0 c1 u
    // u^2 = -5: c0^2 - 5 c1^2 = (c0 + c1)(c0 - 5 c1) + 4 c0 c1
    B2S_HD Fp2 sqr() const {
        if constexpr (P::FQ2_NR == -1) {
            B s = (c0 + c1) * (c0 - c1);
            B t = c0 * c1;
            return {s, t.dbl()};
        } else {
            B t = c0 * c1;
            B t2 = t.dbl();
            B s = (c0 + c1) * (c0 - times5(c1)) + t2.dbl();
            return {s, t2};
        }
    }
    B2S_HD Fp2& operator+=(const Fp2& o) { *this = *this + o; return *this; }
    B2S_HD Fp2& operator-=(const Fp2& o) { *this = *this - o; return *this; }
    B2S_HD Fp2& operator*=(const Fp2& o) { *this = *this * o; return *this; }
    // 1 / (c0 + c1 u) = (c0 - c1 u) / (c0^2 - FQ2_NR c1^2)
    B2S_HD Fp2 inverse() const {
        B n;
        if constexpr (P::FQ2_NR == -1) n = (c0.sqr() + c1.sqr()).inverse();
        else n = (c0.sqr() + times5(c1.sqr())).inverse();
        return {c0 * n, (c1 * n).neg()};
    }
};

}  // namespace b2s
