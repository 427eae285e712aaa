// G2 bucket accumulation (Fq2 = 3 Fq multiplications per product) and the G2 Horner tail, compiled
// with the multiplication inlined: 255 registers on sm_90a (the XYZZ accumulation spills a few bytes), two CTAs of
// 128 threads per SM.  tools/microbench.cu on an H100 80GB HBM3 at a 400 W limit sustains the same XYZZ addition rate
// with two CTAs of 128 threads per SM as with four (2.57e9 vs 2.58e9 G1 additions/s), so two keep the fmaheavy pipe full.
#define B2S_INLINE_MUL 1
#include "msm_affine.cuh"

namespace b2s {

int32_t msm_accumulate_g2(Ctx* c, const void* bases, const uint32_t* sorted, const uint32_t* offsets,
                          const uint32_t* task_off, const uint32_t* perm, MsmShape sh, void* bucket_acc, void* partials) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq2;
        B2S_LAUNCH_N(c, "msm_accumulate_g2", msm_accumulate_kernel<F>, cdiv(sh.max_tasks, MSM_ACC_THREADS), MSM_ACC_THREADS, 0,
                     reinterpret_cast<const Affine<F>*>(bases), sorted, offsets, task_off, perm, sh,
                     reinterpret_cast<XYZZ<F>*>(bucket_acc), reinterpret_cast<XYZZ<F>*>(partials));
        return (int32_t)B2S_OK;
    });
}

int32_t msm_horner_g2(Ctx* c, cudaStream_t st, const void* wins, MsmShape sh, uint32_t K, void* out) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq2;
        B2S_LAUNCH_SN(c, st, "msm_horner_g2", msm_horner_kernel<F>, cdiv(K, 8), 32, 0, reinterpret_cast<const XYZZ<F>*>(wins), sh, K,
                      reinterpret_cast<XYZZ<F>*>(out));
        return (int32_t)B2S_OK;
    });
}

int32_t msm_ba_round_g2(Ctx* c, const BaRoundArgs& a) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq2;
        return msm_ba_round_launch<F>(c, "msm_ba_p1_g2", "msm_ba_inv_g2", "msm_ba_p2_g2", a);
    });
}

}  // namespace b2s
