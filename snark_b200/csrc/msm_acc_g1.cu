// The hot kernel of the prover: G1 bucket accumulation with the Fq multiplication inlined (see
// msm_acc.cuh / msm.cu for the algorithm).  Kept in its own translation unit so that only this
// kernel pays the compile time of full inlining.
#define B2S_INLINE_MUL 1
#include "msm_affine.cuh"

namespace b2s {

int32_t msm_accumulate_g1(Ctx* c, const void* bases, const uint32_t* sorted, const uint32_t* offsets,
                          const uint32_t* task_off, const uint32_t* perm, MsmShape sh, void* bucket_acc, void* partials) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq;
        B2S_LAUNCH_N(c, "msm_accumulate_g1", msm_accumulate_kernel<F>, cdiv(sh.max_tasks, MSM_ACC_THREADS), MSM_ACC_THREADS, 0,
                   reinterpret_cast<const Affine<F>*>(bases), sorted, offsets, task_off, perm, sh,
                   reinterpret_cast<XYZZ<F>*>(bucket_acc), reinterpret_cast<XYZZ<F>*>(partials));
        return (int32_t)B2S_OK;
    });
}

int32_t msm_horner_g1(Ctx* c, cudaStream_t st, const void* wins, MsmShape sh, uint32_t K, void* out) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq;
        B2S_LAUNCH_SN(c, st, "msm_horner_g1", msm_horner_kernel<F>, cdiv(K, 8), 32, 0, reinterpret_cast<const XYZZ<F>*>(wins), sh, K,
                      reinterpret_cast<XYZZ<F>*>(out));
        return (int32_t)B2S_OK;
    });
}

int32_t msm_ba_round_g1(Ctx* c, const BaRoundArgs& a) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq;
        return msm_ba_round_launch<F>(c, "msm_ba_p1_g1", "msm_ba_inv_g1", "msm_ba_p2_g1", a);
    });
}

int32_t msm_bucket_reduce_g1(Ctx* c, const void* bucket_acc, MsmShape sh, uint32_t seg, void* segs, uint32_t segs_per_win, void* wins) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq;
        return msm_bucket_reduce_launch<F>(c, "msm_bucket_segments_g1", "msm_window_sum_g1", bucket_acc, sh, seg, segs, segs_per_win, wins);
    });
}

}  // namespace b2s
