// Groth16 verification of many proofs under one verifying key, and element-wise pairings (pairing.cuh).  One thread per
// proof; three kernels per chunk, so that no kernel holds the public-input sum, the Miller loop and the final
// exponentiation live at once:
//   verify_ic         IC = gamma_abc[0] + sum_j x_j gamma_abc[j+1] from fixed-base window tables (affine result)
//   verify_miller     f = ML(A, B) ML(IC, -gamma) ML(C, -delta): B's lines on the fly, -gamma / -delta prepared (every
//                     thread of a warp reads the same line at the same time)
//   verify_final_exp  f^((p^12 - 1) / r ...) == e(alpha, beta) -> one byte per proof
// f goes through device memory between the last two (576 B per proof on BLS12-381, 384 B on BN254).  Host batches are
// processed in chunks through bounded device scratch, so n_proofs is not limited by device memory.
#include <algorithm>

#include "common.cuh"
#include "pairing.cuh"
#include "verify.cuh"

namespace b2s {

template <class Curve>
__global__ void vk_prepare_kernel(const typename Curve::G1Affine* alpha, const typename Curve::G2Affine* g2 /* beta, gamma, delta */,
                                  G2Prepared<Curve>* prep, Fp12<typename Curve::FqP>* ab) {
    if (blockIdx.x | threadIdx.x) return;
    g2_prepare<Curve>(g2[1].neg(), prep[0]);
    g2_prepare<Curve>(g2[2].neg(), prep[1]);
    *ab = pairing<Curve>(*alpha, g2[0]);
}

template <class Curve>
__global__ void ic_table_kernel(const typename Curve::G1Affine* bases, uint64_t n_entries, typename Curve::G1Affine* table) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_entries) return;
    const uint64_t j = t / (IC_WINDOWS * IC_DIGITS);
    const uint32_t w = (uint32_t)(t / IC_DIGITS % IC_WINDOWS), d = (uint32_t)(t % IC_DIGITS) + 1;
    uint32_t k[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    k[(IC_WBITS * w) / 32] = d << ((IC_WBITS * w) % 32);
    table[t] = scalar_mul_words(Curve::G1::from_affine(bases[j]), k, 8).to_affine();
}

template <class Curve>
__global__ void verify_ic_kernel(const typename Curve::Fr* inputs, uint32_t n, uint32_t ni, const typename Curve::G1Affine* abc0,
                                 const typename Curve::G1Affine* table, typename Curve::G1Affine* ic) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    typename Curve::G1 acc = Curve::G1::from_affine(*abc0);
    for (uint32_t j = 0; j < ni; j++) {
        const typename Curve::Fr s = inputs[(uint64_t)i * ni + j].from_mont();
        const typename Curve::G1Affine* tj = table + (uint64_t)j * IC_WINDOWS * IC_DIGITS;
        for (int w = 0; w < IC_WINDOWS; w++) {
            const uint32_t d = (s.v[w / 4] >> (8 * (w % 4))) & 0xFF;
            if (d) acc.add_affine(tj[w * IC_DIGITS + d - 1]);
        }
    }
    ic[i] = acc.to_affine();
}

template <class Curve>
__global__ void verify_miller_kernel(const typename Curve::G1Affine* a, const typename Curve::G2Affine* b, const typename Curve::G1Affine* ic,
                                     const typename Curve::G1Affine* c, const G2Prepared<Curve>* prep, uint32_t n,
                                     Fp12<typename Curve::FqP>* f) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f[i] = groth16_miller<Curve>(a[i], b[i], ic[i], c[i], &prep[0], &prep[1]);
}

template <class Curve>
__global__ void pairing_miller_kernel(const typename Curve::G1Affine* p, const typename Curve::G2Affine* q, uint32_t n,
                                      Fp12<typename Curve::FqP>* f) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    f[i] = multi_miller_loop<Curve, 1, 0>(&p[i], &q[i], nullptr, nullptr);
}

// ok == nullptr: out[i] = the final exponentiation of f[i]; otherwise ok[i] = [final exponentiation of f[i] == *target]
template <class Curve>
__global__ void final_exp_kernel(const Fp12<typename Curve::FqP>* f, uint32_t n, const Fp12<typename Curve::FqP>* target, uint8_t* ok,
                                 Fp12<typename Curve::FqP>* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fp12<typename Curve::FqP> r = final_exponentiation(f[i]);
    if (ok) ok[i] = r == *target ? 1 : 0;
    else out[i] = r;
}

int32_t vk_prepare(Ctx* c, const void* alpha, const void* beta, const void* gamma, const void* delta, const void* abc, uint64_t n_abc,
                   b2s_pvk** out) {
    if (n_abc == 0) return fail(c, B2S_ERR_MALFORMED_VK, "vk_prepare: gamma_abc_g1 is empty");
    const Sizes s = sizes(c);
    b2s_pvk* pvk = new b2s_pvk();
    pvk->curve = c->curve;
    pvk->n_abc = n_abc;
    auto body = [&]() -> int32_t {
        DevBuf pts;   // alpha, beta, gamma, delta, gamma_abc
        B2S_TRY(pts.alloc(c, s.g1 + 3 * s.g2 + n_abc * s.g1));
        char* d = pts.as<char>();
        B2S_CUDA(c, cudaMemcpyAsync(d, alpha, s.g1, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(d + s.g1, beta, s.g2, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(d + s.g1 + s.g2, gamma, s.g2, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(d + s.g1 + 2 * s.g2, delta, s.g2, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(d + s.g1 + 3 * s.g2, abc, n_abc * s.g1, cudaMemcpyHostToDevice, c->stream));
        const char* abc_dev = d + s.g1 + 3 * s.g2;
        return dispatch_curve(c, [&](auto curve) -> int32_t {
            using C = decltype(curve);
            using G1A = typename C::G1Affine;
            B2S_TRY(pvk->prep.alloc(c, 2 * sizeof(G2Prepared<C>)));
            B2S_TRY(pvk->ab.alloc(c, sizeof(Fp12<typename C::FqP>)));
            B2S_TRY(pvk->abc0.alloc(c, s.g1));
            B2S_CUDA(c, cudaMemcpyAsync(pvk->abc0.p, abc_dev, s.g1, cudaMemcpyDeviceToDevice, c->stream));
            B2S_LAUNCH_N(c, "vk_prepare", vk_prepare_kernel<C>, 1, 1, 0, reinterpret_cast<const G1A*>(d),
                         reinterpret_cast<const typename C::G2Affine*>(d + s.g1), pvk->prep.as<G2Prepared<C>>(),
                         pvk->ab.as<Fp12<typename C::FqP>>());
            const uint64_t entries = (n_abc - 1) * IC_WINDOWS * IC_DIGITS;
            if (entries) {
                B2S_TRY(pvk->table.alloc(c, entries * s.g1));
                B2S_LAUNCH_N(c, "vk_ic_table", ic_table_kernel<C>, cdiv(entries, VERIFY_THREADS), VERIFY_THREADS, 0,
                             reinterpret_cast<const G1A*>(abc_dev + s.g1), entries, pvk->table.as<G1A>());
            }
            B2S_CUDA(c, cudaStreamSynchronize(c->stream));
            return (int32_t)B2S_OK;
        });
    };
    const int32_t st = body();
    if (st != B2S_OK) { delete pvk; return st; }
    *out = pvk;
    return B2S_OK;
}

int32_t groth16_verify_batch(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const void* a, const void* b,
                             const void* cc, int32_t mem, uint8_t* ok) {
    if (pvk->curve != c->curve) return fail(c, B2S_ERR_INVALID_ARG, "verify_batch: the prepared key belongs to another curve");
    if (ni + 1 != pvk->n_abc)
        return fail(c, B2S_ERR_MALFORMED_VK, "verify_batch: %llu public inputs, the key expects %llu", (unsigned long long)ni,
                    (unsigned long long)(pvk->n_abc - 1));
    if (n == 0) return B2S_OK;
    if (!a || !b || !cc || !ok || (ni && !inputs)) return fail(c, B2S_ERR_INVALID_ARG, "verify_batch: null buffer");
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        using C = decltype(curve);
        using F12 = Fp12<typename C::FqP>;
        using G1A = typename C::G1Affine;
        const size_t g1 = sizeof(G1A), g2 = sizeof(typename C::G2Affine), f12 = sizeof(F12);
        RowStager io(c, mem, {col_in(inputs, ni * sizeof(typename C::Fr)), col_in(a, g1), col_in(b, g2), col_in(cc, g1), col_out(ok, 1)});
        const uint64_t ch = chunk_size(n, g1 + f12 + io.row_bytes());
        DevBuf scratch;
        B2S_TRY(scratch.alloc(c, ch * (g1 + f12)));
        auto* ic = scratch.as<G1A>();
        auto* f = reinterpret_cast<F12*>(scratch.as<char>() + ch * g1);
        B2S_TRY(io.alloc(ch));
        for (uint64_t base = 0; base < n; base += ch) {
            const uint32_t m = (uint32_t)std::min<uint64_t>(ch, n - base);
            B2S_TRY(io.load(base, m));
            const unsigned grid = cdiv(m, VERIFY_THREADS);
            B2S_LAUNCH_N(c, "verify_ic", verify_ic_kernel<C>, grid, VERIFY_THREADS, 0, io.ptr<const typename C::Fr>(0), m,
                         (uint32_t)ni, pvk->abc0.as<G1A>(), pvk->table.as<G1A>(), ic);
            B2S_LAUNCH_N(c, "verify_miller", verify_miller_kernel<C>, grid, VERIFY_THREADS, 0, io.ptr<const G1A>(1),
                         io.ptr<const typename C::G2Affine>(2), ic, io.ptr<const G1A>(3), pvk->prep.as<G2Prepared<C>>(), m, f);
            B2S_LAUNCH_N(c, "verify_final_exp", final_exp_kernel<C>, grid, VERIFY_THREADS, 0, f, m, pvk->ab.as<F12>(), io.ptr<uint8_t>(4),
                         (F12*)nullptr);
            B2S_TRY(io.store());
        }
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        return (int32_t)B2S_OK;
    });
}

int32_t pairing_batch(Ctx* c, const void* p, const void* q, uint64_t n, int32_t mem, void* out) {
    if (n == 0) return B2S_OK;
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        using C = decltype(curve);
        using F12 = Fp12<typename C::FqP>;
        const size_t f12 = sizeof(F12);
        RowStager io(c, mem, {col_in(p, sizeof(typename C::G1Affine)), col_in(q, sizeof(typename C::G2Affine)), col_out(out, f12)});
        const uint64_t ch = chunk_size(n, f12 + io.row_bytes());
        DevBuf f;
        B2S_TRY(f.alloc(c, ch * f12));
        B2S_TRY(io.alloc(ch));
        for (uint64_t base = 0; base < n; base += ch) {
            const uint32_t m = (uint32_t)std::min<uint64_t>(ch, n - base);
            B2S_TRY(io.load(base, m));
            const unsigned grid = cdiv(m, VERIFY_THREADS);
            B2S_LAUNCH_N(c, "pairing_miller", pairing_miller_kernel<C>, grid, VERIFY_THREADS, 0, io.ptr<const typename C::G1Affine>(0),
                         io.ptr<const typename C::G2Affine>(1), m, f.as<F12>());
            B2S_LAUNCH_N(c, "pairing_final_exp", final_exp_kernel<C>, grid, VERIFY_THREADS, 0, f.as<F12>(), m, (const F12*)nullptr,
                         (uint8_t*)nullptr, io.ptr<F12>(2));
            B2S_TRY(io.store());
        }
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        return (int32_t)B2S_OK;
    });
}


void pvk_free(b2s_pvk* pvk) { delete pvk; }

}  // namespace b2s
