// Host-side harness for BLS12-377: the SAME field, Fq2, group-law, point-decoding and pairing templates the kernels
// instantiate for curve id 2, compiled for the CPU with the PTX carry flag emulated and exposed to ctypes for
// tests/test_host_bls12_377.py.  Test infrastructure only.  Buffers are Montgomery limbs in the C-ABI layouts, except
// scalars, exponents and rho, which are canonical little-endian words.
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../snark_b200/csrc/deserialize.cuh"
#include "../../snark_b200/csrc/pairing.cuh"

using namespace b2s;
using C = Bls12_377;
using P = C::FqP;
using Fq = C::Fq;
using Fr = C::Fr;
using Fq2 = C::Fq2;
using G1A = Affine<Fq>;
using G2A = Affine<Fq2>;

template <class T>
static T ld(const uint32_t* p, size_t i) {
    T t;
    memcpy(&t, p + i * (sizeof(T) / 4), sizeof(T));
    return t;
}
template <class T>
static void st(uint32_t* p, size_t i, const T& t) { memcpy(p + i * (sizeof(T) / 4), &t, sizeof(T)); }

// field 0 = Fq, 1 = Fr; ops as in host_ff.cpp: 0 a*b 1 a+b 2 a-b 3 1/a 4 -a 5 to_mont 6 from_mont 7 a^2
template <class F>
static F field_binop(int op, const F& x, const F& y) {
    switch (op) {
        case 0: return x * y;
        case 1: return x + y;
        case 2: return x - y;
        case 3: return x.inverse();
        case 4: return x.neg();
        case 5: return x.to_mont();
        case 6: return x.from_mont();
        case 7: return x.sqr();
    }
    return F::zero();
}
extern "C" void ht377_field_op(int field, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, int count) {
    for (int i = 0; i < count; i++) {
        if (field == 0) st(out, i, field_binop(op, ld<Fq>(a, i), ld<Fq>(b, i)));
        else st(out, i, field_binop(op, ld<Fr>(a, i), ld<Fr>(b, i)));
    }
}
// which: 0 mod, 1 R mod p, 2 R^2 mod p, 3 Fr generator, 4 Fr 2^47-th root of unity (field 1 only)
extern "C" void ht377_field_const(int field, int which, uint32_t* out) {
    const int n = field == 0 ? 12 : 8;
    for (int i = 0; i < n; i++) {
        if (field == 0) out[i] = which == 0 ? P::mod(i) : which == 1 ? P::r1(i) : P::r2(i);
        else out[i] = which == 0 ? Bls377FrP::mod(i) : which == 1 ? Bls377FrP::r1(i) : which == 2 ? Bls377FrP::r2(i)
                    : which == 3 ? Bls377FrP::gen(i) : Bls377FrP::root(i);
    }
}

// Fq2: 0 a*b 1 a^2 2 1/a 3 a*xi 4 sqrt (ok[i] = 1 if a root exists) 5 a+b 6 a-b
extern "C" void ht377_fq2_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, uint8_t* ok, int count) {
    for (int i = 0; i < count; i++) {
        const Fq2 x = ld<Fq2>(a, i), y = ld<Fq2>(b, i);
        Fq2 r = Fq2::zero();
        switch (op) {
            case 0: r = x * y; break;
            case 1: r = x.sqr(); break;
            case 2: r = x.inverse(); break;
            case 3: r = mul_xi(x); break;
            case 4: ok[i] = dec::sqrt(x, r) ? 1 : 0; break;
            case 5: r = x + y; break;
            case 6: r = x - y; break;
        }
        st(out, i, r);
    }
}
// Fq square root (Tonelli-Shanks): ok[i] = 1 and out[i] a root, or ok[i] = 0
extern "C" void ht377_fq_sqrt(const uint32_t* a, uint32_t* out, uint8_t* ok, int count) {
    for (int i = 0; i < count; i++) {
        Fq r = Fq::zero();
        ok[i] = dec::sqrt(ld<Fq>(a, i), r) ? 1 : 0;
        st(out, i, r);
    }
}

// group law: 0 a + b (mixed), 1 2a, 2 [k] a (kwords canonical words per point)
template <class F>
static void ec_run(int op, const uint32_t* a, const uint32_t* b, const uint32_t* k, int kwords, uint32_t* out, int count) {
    for (int i = 0; i < count; i++) {
        const Affine<F> pa = ld<Affine<F>>(a, i);
        XYZZ<F> r = XYZZ<F>::from_affine(pa);
        if (op == 0) r.add_affine(ld<Affine<F>>(b, i));
        if (op == 1) r = r.dbl();
        if (op == 2) r = scalar_mul_words(r, k + (size_t)i * kwords, kwords);
        st(out, i, r.to_affine());
    }
}
extern "C" void ht377_ec_op(int group, int op, const uint32_t* a, const uint32_t* b, const uint32_t* k, int kwords, uint32_t* out,
                            int count) {
    if (group == 1) ec_run<Fq>(op, a, b, k, kwords, out, count);
    else ec_run<Fq2>(op, a, b, k, kwords, out, count);
}
extern "C" void ht377_generator(int group, uint32_t* out) {
    if (group == 1) st(out, 0, C::g1_generator());
    else st(out, 0, C::g2_generator());
}

// decode_point on `count` encodings back to back -> affine Montgomery limbs and a DecodeStatus per point
extern "C" void ht377_point_decode(int group, const uint8_t* in, int compressed, int validate, uint32_t* out, uint32_t* status,
                                   int count) {
    const int pb = 48 * group * (compressed ? 1 : 2);
    for (int i = 0; i < count; i++) {
        if (group == 1) {
            G1A p = G1A::inf();
            status[i] = decode_point<C, Fq>(in + (size_t)i * pb, compressed != 0, validate != 0, p);
            st(out, i, p);
        } else {
            G2A p = G2A::inf();
            status[i] = decode_point<C, Fq2>(in + (size_t)i * pb, compressed != 0, validate != 0, p);
            st(out, i, p);
        }
    }
}
// the endomorphism subgroup criterion on affine points already on the curve
extern "C" void ht377_in_subgroup(int group, const uint32_t* pts, uint8_t* ok, int count) {
    for (int i = 0; i < count; i++)
        ok[i] = group == 1 ? dec::in_subgroup<C>(ld<G1A>(pts, i)) : dec::in_subgroup<C>(ld<G2A>(pts, i));
}

// tower: 0 a*b 1 a^2 2 1/a 3..5 a^(p^1..3) 6 cyclotomic a^2 7 a * D-type line (l0 + l1 w + l2 w^3) 8 final exponentiation
extern "C" void ht377_fp12_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, int count) {
    using F12 = Fp12<P>;
    for (int i = 0; i < count; i++) {
        const F12 x = ld<F12>(a, i);
        F12 r = x;
        switch (op) {
            case 0: r = fp12_mul(x, ld<F12>(b, i)); break;
            case 1: r = fp12_sqr(x); break;
            case 2: r = fp12_inverse(x); break;
            case 3: case 4: case 5: r = fp12_frobenius(x, op - 2); break;
            case 6: r = fp12_cyclotomic_sqr(x); break;
            case 7: {
                const Line<P> l = ld<Line<P>>(b, i);
                r = fp12_mul_by_034(x, l.c0, l.c1, l.c2);
                break;
            }
            case 8: r = final_exponentiation(x); break;
        }
        st(out, i, r);
    }
}
// mode 0: e(P_i, Q_i); 1: the Miller loop alone, lines on the fly; 2: the Miller loop alone, Q prepared first
extern "C" void ht377_pairing(int mode, const uint32_t* p, const uint32_t* q, uint32_t* out, int count) {
    std::vector<G2Prepared<C>> prep(1);
    for (int i = 0; i < count; i++) {
        const G1A pi = ld<G1A>(p, i);
        const G2A qi = ld<G2A>(q, i);
        Fp12<P> r;
        if (mode == 0) r = pairing<C>(pi, qi);
        if (mode == 1) r = multi_miller_loop<C, 1, 0>(&pi, &qi, nullptr, nullptr);
        if (mode == 2) {
            g2_prepare<C>(qi, prep[0]);
            const G2Prepared<C>* pp = &prep[0];
            r = multi_miller_loop<C, 0, 1>(nullptr, nullptr, &pi, &pp);
        }
        st(out, i, r);
    }
}
extern "C" int ht377_prepared_lines() { return PairingShape<C>::LINES; }

// the per-proof verdict of the verify kernels (vk: alpha, beta, gamma, delta back to back; ic: the public-input sum)
extern "C" void ht377_groth16_verdict(const uint32_t* vk, const uint32_t* ic, const uint32_t* a, const uint32_t* b, const uint32_t* c,
                                      uint8_t* ok, int count) {
    const G1A alpha = ld<G1A>(vk, 0);
    const uint32_t* g2 = vk + sizeof(G1A) / 4;
    const G2A beta = ld<G2A>(g2, 0), gamma = ld<G2A>(g2, 1), delta = ld<G2A>(g2, 2);
    std::vector<G2Prepared<C>> prep(2);
    g2_prepare<C>(gamma.neg(), prep[0]);
    g2_prepare<C>(delta.neg(), prep[1]);
    const Fp12<P> ab = pairing<C>(alpha, beta);
    for (int i = 0; i < count; i++)
        ok[i] = groth16_verdict<C>(ld<G1A>(a, i), ld<G2A>(b, i), ld<G1A>(ic, i), ld<G1A>(c, i), &prep[0], &prep[1], ab) ? 1 : 0;
}

// The random-linear-combination batch verdict as verify_rlc.cu forms it (sums on the CPU), Miller grouping NF = 2:
// abc: n_inputs + 1 gamma_abc points; inputs: count x ni Montgomery Fr; rho: 4 words per proof.  Returns 0 / 1.
extern "C" int ht377_rlc_verdict(const uint32_t* vk, const uint32_t* abc, const uint32_t* inputs, int ni, const uint32_t* a,
                                 const uint32_t* b, const uint32_t* c, const uint32_t* rho, int count) {
    constexpr int NF = 2;
    const G1A alpha = ld<G1A>(vk, 0);
    const uint32_t* g2 = vk + sizeof(G1A) / 4;
    const G2A beta = ld<G2A>(g2, 0), gamma = ld<G2A>(g2, 1), delta = ld<G2A>(g2, 2);
    std::vector<G2Prepared<C>> prep(2);
    g2_prepare<C>(gamma.neg(), prep[0]);
    g2_prepare<C>(delta.neg(), prep[1]);
    const Fp12<P> ab = pairing<C>(alpha, beta);
    Fp12<P> f = Fp12<P>::one();
    for (int g = 0; g * NF < count; g++) {
        G1A pa[NF];
        G2A pb[NF];
        uint32_t k[4 * NF];
        for (int j = 0; j < NF; j++) {
            const int i = g * NF + j;
            pa[j] = i < count ? ld<G1A>(a, i) : G1A::inf();
            pb[j] = i < count ? ld<G2A>(b, i) : G2A::inf();
            for (int w = 0; w < 4; w++) k[4 * j + w] = i < count ? rho[4 * i + w] : 0;
        }
        f = fp12_mul(f, rlc_miller<C, NF>(pa, pb, k));
    }
    std::vector<Fr> t(ni + 1, Fr::zero());
    C::G1 cs = C::G1::identity();
    for (int i = 0; i < count; i++) {
        Fr r = Fr::zero();
        for (int w = 0; w < 4; w++) r.v[w] = rho[4 * i + w];
        t[0] += r;
        for (int j = 0; j < ni; j++) t[j + 1] += ld<Fr>(inputs, (size_t)i * ni + j) * r;
        cs.add(scalar_mul_words(C::G1::from_affine(ld<G1A>(c, i)), rho + 4 * i, 4));
    }
    C::G1 ic = C::G1::identity();
    for (int j = 0; j <= ni; j++) ic.add(scalar_mul_words(C::G1::from_affine(ld<G1A>(abc, j)), t[j].v, 8));
    return rlc_verdict<C>(f, ic.to_affine(), cs.to_affine(), &prep[0], &prep[1], ab, t[0].v) ? 1 : 0;
}
