// Host-side harness for the pairing (snark_b200/csrc/pairing.cuh): the SAME tower, Miller loop, final exponentiation and
// Groth16 verdict the verify kernels run, compiled for the CPU with the PTX carry flag emulated and exposed to ctypes for
// tests/test_host_pairing.py.  Test infrastructure only.  Buffers are Montgomery limbs in the C-ABI layouts; a GT element
// is ark's Fp12 (c0 = Fp6 {c0, c1, c2 : Fp2}, c1).
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../snark_b200/csrc/pairing.cuh"

using namespace b2s;

template <class T>
static T ld(const uint32_t* p, size_t i) {
    T t;
    memcpy(&t, p + i * (sizeof(T) / 4), sizeof(T));
    return t;
}
template <class T>
static void st(uint32_t* p, size_t i, const T& t) { memcpy(p + i * (sizeof(T) / 4), &t, sizeof(T)); }

// tower operations, element-wise over `count` Fq12 elements:
//   0 a*b  1 a^2  2 1/a  3..5 a^(p^1..3)  6 cyclotomic a^2  7 a * line, b = three Fq2 (l0, l1, l2) per element:
//   014 form (l0 + l1 w^2 + l2 w^3) for curve 0, 034 form (l0 + l1 w + l2 w^3) for curve 1  8 final exponentiation
template <class Curve>
static void fp12_op(int op, const uint32_t* a, const uint32_t* b, uint32_t* out, int count) {
    using P = typename Curve::FqP;
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
                r = PairingShape<Curve>::M_TWIST ? fp12_mul_by_014(x, l.c0, l.c1, l.c2) : fp12_mul_by_034(x, l.c0, l.c1, l.c2);
                break;
            }
            case 8: r = final_exponentiation(x); break;
        }
        st(out, i, r);
    }
}
extern "C" void ht_fp12_op(int curve, int op, const uint32_t* a, const uint32_t* b, uint32_t* out, int count) {
    if (curve == 0) fp12_op<Bls12_381>(op, a, b, out, count);
    else fp12_op<Bn254>(op, a, b, out, count);
}

// mode 0: e(P_i, Q_i); 1: the Miller loop alone, lines on the fly; 2: the Miller loop alone, Q prepared first
template <class Curve>
static void pairing_run(int mode, const uint32_t* p, const uint32_t* q, uint32_t* out, int count) {
    using P = typename Curve::FqP;
    std::vector<G2Prepared<Curve>> prep(1);
    for (int i = 0; i < count; i++) {
        const auto pi = ld<Affine<Fp<P>>>(p, i);
        const auto qi = ld<Affine<Fp2<P>>>(q, i);
        Fp12<P> r;
        if (mode == 0) r = pairing<Curve>(pi, qi);
        if (mode == 1) r = multi_miller_loop<Curve, 1, 0>(&pi, &qi, nullptr, nullptr);
        if (mode == 2) {
            g2_prepare<Curve>(qi, prep[0]);
            const G2Prepared<Curve>* pp = &prep[0];
            r = multi_miller_loop<Curve, 0, 1>(nullptr, nullptr, &pi, &pp);
        }
        st(out, i, r);
    }
}
extern "C" void ht_pairing(int curve, int mode, const uint32_t* p, const uint32_t* q, uint32_t* out, int count) {
    if (curve == 0) pairing_run<Bls12_381>(mode, p, q, out, count);
    else pairing_run<Bn254>(mode, p, q, out, count);
}

// The per-proof verdict of the verify kernels.  vk: alpha (G1), beta, gamma, delta (G2) packed back to back; abc: IC per
// proof (the public-input sum, computed by the caller); a, b, c: the proofs.  ok[i] = 0 / 1.
template <class Curve>
static void verdict_run(const uint32_t* vk, const uint32_t* ic, const uint32_t* a, const uint32_t* b, const uint32_t* c, uint8_t* ok,
                        int count) {
    using P = typename Curve::FqP;
    using G1 = Affine<Fp<P>>;
    using G2 = Affine<Fp2<P>>;
    const G1 alpha = ld<G1>(vk, 0);
    const uint32_t* g2 = vk + sizeof(G1) / 4;
    const G2 beta = ld<G2>(g2, 0), gamma = ld<G2>(g2, 1), delta = ld<G2>(g2, 2);
    std::vector<G2Prepared<Curve>> prep(2);
    g2_prepare<Curve>(gamma.neg(), prep[0]);
    g2_prepare<Curve>(delta.neg(), prep[1]);
    const Fp12<P> ab = pairing<Curve>(alpha, beta);
    for (int i = 0; i < count; i++)
        ok[i] = groth16_verdict<Curve>(ld<G1>(a, i), ld<G2>(b, i), ld<G1>(ic, i), ld<G1>(c, i), &prep[0], &prep[1], ab) ? 1 : 0;
}
extern "C" void ht_groth16_verdict(int curve, const uint32_t* vk, const uint32_t* ic, const uint32_t* a, const uint32_t* b,
                                   const uint32_t* c, uint8_t* ok, int count) {
    if (curve == 0) verdict_run<Bls12_381>(vk, ic, a, b, c, ok, count);
    else verdict_run<Bn254>(vk, ic, a, b, c, ok, count);
}

extern "C" int ht_prepared_lines(int curve) {
    return curve == 0 ? PairingShape<Bls12_381>::LINES : PairingShape<Bn254>::LINES;
}
