// Host-side harness for the random-linear-combination batch check (snark_b200/csrc/pairing.cuh: cyclotomic_exp,
// rlc_miller, rlc_verdict): the SAME per-thread code verify_rlc.cu runs, compiled for the CPU and exposed to ctypes for
// tests/test_host_verify_rlc.py.  Test infrastructure only.  Buffers are Montgomery limbs in the C-ABI layouts, except
// exponents and rho, which are canonical little-endian words.
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

// out[i] = f[i]^e[i], e[i] = nwords canonical words
template <class Curve>
static void cyc_exp_run(const uint32_t* f, const uint32_t* e, int nwords, uint32_t* out, int count) {
    using F12 = Fp12<typename Curve::FqP>;
    for (int i = 0; i < count; i++) st(out, i, cyclotomic_exp(ld<F12>(f, i), e + (size_t)i * nwords, nwords));
}
extern "C" void ht_cyclotomic_exp(int curve, const uint32_t* f, const uint32_t* e, int nwords, uint32_t* out, int count) {
    if (curve == 0) cyc_exp_run<Bls12_381>(f, e, nwords, out, count);
    else cyc_exp_run<Bn254>(f, e, nwords, out, count);
}

// The Miller values verify_rlc_miller writes: out[g] = rlc_miller over proofs [g nf, (g + 1) nf), the last group padded
// with pairs at infinity; rho: 4 words per proof.
template <class Curve, int NF>
static void rlc_miller_nf(const uint32_t* a, const uint32_t* b, const uint32_t* rho, uint32_t* out, int count) {
    using P = typename Curve::FqP;
    for (int g = 0; g * NF < count; g++) {
        Affine<Fp<P>> pa[NF];
        Affine<Fp2<P>> pb[NF];
        uint32_t k[4 * NF];
        for (int j = 0; j < NF; j++) {
            const int i = g * NF + j;
            pa[j] = i < count ? ld<Affine<Fp<P>>>(a, i) : Affine<Fp<P>>::inf();
            pb[j] = i < count ? ld<Affine<Fp2<P>>>(b, i) : Affine<Fp2<P>>::inf();
            for (int w = 0; w < 4; w++) k[4 * j + w] = i < count ? rho[4 * i + w] : 0;
        }
        st(out, g, rlc_miller<Curve, NF>(pa, pb, k));
    }
}
template <class Curve>
static void rlc_miller_run(int nf, const uint32_t* a, const uint32_t* b, const uint32_t* rho, uint32_t* out, int count) {
    if (nf == 1) rlc_miller_nf<Curve, 1>(a, b, rho, out, count);
    if (nf == 2) rlc_miller_nf<Curve, 2>(a, b, rho, out, count);
    if (nf == 4) rlc_miller_nf<Curve, 4>(a, b, rho, out, count);
}
extern "C" void ht_rlc_miller(int curve, int nf, const uint32_t* a, const uint32_t* b, const uint32_t* rho, uint32_t* out, int count) {
    if (curve == 0) rlc_miller_run<Bls12_381>(nf, a, b, rho, out, count);
    else rlc_miller_run<Bn254>(nf, a, b, rho, out, count);
}

// The whole batch verdict as verify_rlc.cu forms it, with the sums done directly on the CPU.  vk: alpha (G1), beta,
// gamma, delta (G2) back to back; abc: the n_inputs + 1 gamma_abc points; inputs: count x n_inputs Montgomery Fr;
// a, b, c: the proofs; rho: 4 words per proof.  nf: the Miller grouping.  Returns 0 / 1.
template <class Curve, int NF>
static int rlc_batch(const uint32_t* vk, const uint32_t* abc, const uint32_t* inputs, int ni, const uint32_t* a, const uint32_t* b,
                     const uint32_t* c, const uint32_t* rho, int count) {
    using P = typename Curve::FqP;
    using Fr = typename Curve::Fr;
    using G1A = Affine<Fp<P>>;
    using G2A = Affine<Fp2<P>>;
    const G1A alpha = ld<G1A>(vk, 0);
    const uint32_t* g2 = vk + sizeof(G1A) / 4;
    const G2A beta = ld<G2A>(g2, 0), gamma = ld<G2A>(g2, 1), delta = ld<G2A>(g2, 2);
    std::vector<G2Prepared<Curve>> prep(2);
    g2_prepare<Curve>(gamma.neg(), prep[0]);
    g2_prepare<Curve>(delta.neg(), prep[1]);
    const Fp12<P> ab = pairing<Curve>(alpha, beta);
    std::vector<uint32_t> fv((size_t)(count + NF - 1) / NF * sizeof(Fp12<P>) / 4);
    rlc_miller_nf<Curve, NF>(a, b, rho, fv.data(), count);
    Fp12<P> f = Fp12<P>::one();
    for (int g = 0; g * NF < count; g++) f = fp12_mul(f, ld<Fp12<P>>(fv.data(), g));
    std::vector<Fr> t(ni + 1, Fr::zero());   // S, t_j: canonical, as verify_rlc_inputs sums them
    typename Curve::G1 cs = Curve::G1::identity();
    for (int i = 0; i < count; i++) {
        Fr r = Fr::zero();
        for (int w = 0; w < 4; w++) r.v[w] = rho[4 * i + w];
        t[0] += r;
        for (int j = 0; j < ni; j++) t[j + 1] += ld<Fr>(inputs, (size_t)i * ni + j) * r;
        cs.add(scalar_mul_words(Curve::G1::from_affine(ld<G1A>(c, i)), rho + 4 * i, 4));
    }
    typename Curve::G1 ic = Curve::G1::identity();
    for (int j = 0; j <= ni; j++) ic.add(scalar_mul_words(Curve::G1::from_affine(ld<G1A>(abc, j)), t[j].v, 8));
    return rlc_verdict<Curve>(f, ic.to_affine(), cs.to_affine(), &prep[0], &prep[1], ab, t[0].v) ? 1 : 0;
}
template <class Curve>
static int rlc_batch_nf(int nf, const uint32_t* vk, const uint32_t* abc, const uint32_t* inputs, int ni, const uint32_t* a,
                        const uint32_t* b, const uint32_t* c, const uint32_t* rho, int count) {
    if (nf == 1) return rlc_batch<Curve, 1>(vk, abc, inputs, ni, a, b, c, rho, count);
    if (nf == 2) return rlc_batch<Curve, 2>(vk, abc, inputs, ni, a, b, c, rho, count);
    return rlc_batch<Curve, 4>(vk, abc, inputs, ni, a, b, c, rho, count);
}
extern "C" int ht_rlc_verdict(int curve, int nf, const uint32_t* vk, const uint32_t* abc, const uint32_t* inputs, int ni,
                              const uint32_t* a, const uint32_t* b, const uint32_t* c, const uint32_t* rho, int count) {
    if (curve == 0) return rlc_batch_nf<Bls12_381>(nf, vk, abc, inputs, ni, a, b, c, rho, count);
    return rlc_batch_nf<Bn254>(nf, vk, abc, inputs, ni, a, b, c, rho, count);
}
