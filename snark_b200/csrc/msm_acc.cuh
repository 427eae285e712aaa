// Bucket accumulation (step 4 of the MSM pipeline in msm.cu), shared between the translation unit that
// compiles it with the field multiplication inlined (msm_acc_g1.cu: G1, the hot kernel of the whole
// prover) and msm.cu (G2, out-of-line multiplication).
#pragma once
#include "common.cuh"
#include "ec_team.cuh"

namespace b2s {

static constexpr int MSM_ACC_THREADS = 128;
static constexpr int MSM_RED_THREADS = 128;

struct MsmShape {
    uint32_t c;        // window bits
    uint32_t nwin;     // number of windows
    uint32_t B;        // buckets per window = 2^(c-1)
    uint32_t G;        // nwin * B
    uint32_t L;        // max points per task
    uint64_t max_tasks;
    // fixed-base precomputation (resident key): the bases array also holds 2^(c w) P_i at [w * pre_stride + i], so every
    // window's digits go to ONE bucket set (G = B) and the per-window reduction / Horner tail disappear.  0 = off.
    uint32_t pre_stride;
};

// ---- vector loads of whole structs ---------------------------------------------------------------
template <class T>
__device__ __forceinline__ T ld_struct(const T* p) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiples only");
    T r;
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&r);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) d[i] = __ldg(s + i);
    return r;
}
template <class T>
__device__ __forceinline__ void st_struct(T* p, const T& v) {
    uint4* d = reinterpret_cast<uint4*>(p);
    const uint4* s = reinterpret_cast<const uint4*>(&v);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) d[i] = s[i];
}

// rare paths of the mixed addition (P + P, P - P), kept out of line so the hot loop stays small.  By value on
// purpose: passing the accumulator by reference would force it into local memory for the whole loop.
template <class F>
__device__ __noinline__ XYZZ<F> madd_rare(Affine<F> q, bool r_is_zero) {
    if (r_is_zero) return XYZZ<F>::dbl_affine(q);
    return XYZZ<F>::identity();
}
// G2 (Fq2) variant: with 96 accumulator registers the by-value form spills; by reference ptxas keeps the
// accumulator in (L1-resident) local memory and the kernel stays at 252 registers without spills.
template <class F>
__device__ __noinline__ void madd_rare_ref(XYZZ<F>& acc, const Affine<F>& q, bool r_is_zero) {
    if (r_is_zero) acc = XYZZ<F>::dbl_affine(q);
    else acc = XYZZ<F>::identity();
}

template <class F>
__device__ __forceinline__ void madd(XYZZ<F>& acc, const Affine<F>& q) {
    if (q.is_inf()) return;
    if (acc.is_identity()) {
        acc.x = q.x; acc.y = q.y; acc.zz = F::one(); acc.zzz = F::one();
        return;
    }
    F p = q.x * acc.zz - acc.x;
    F r = q.y * acc.zzz - acc.y;
    if (p.is_zero()) {
        if (sizeof(F) > 64) madd_rare_ref(acc, q, r.is_zero());
        else acc = madd_rare<F>(q, r.is_zero());
        return;
    }
    F pp = p.sqr();
    F ppp = p * pp;
    F qv = acc.x * pp;
    F x3 = r.sqr() - ppp - qv.dbl();
    acc.y = r * (qv - x3) - acc.y * ppp;
    acc.x = x3;
    acc.zz = acc.zz * pp;
    acc.zzz = acc.zzz * ppp;
}

// One thread per task.  Task t belongs to bucket g = upper_bound(task_off, t) - 1.
template <class F>
__global__ void __launch_bounds__(MSM_ACC_THREADS, 1)
msm_accumulate_kernel(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ sorted,
                      const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ task_off,
                      const uint32_t* __restrict__ perm, MsmShape sh, XYZZ<F>* __restrict__ bucket_acc,
                      XYZZ<F>* __restrict__ partials) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t total = task_off[sh.G];
    if (t >= total) return;
    // binary search: largest g with task_off[g] <= t  (empty buckets have task_off[g] == task_off[g+1])
    uint32_t lo = 0, hi = sh.G;   // invariant: task_off[lo] <= t < task_off[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (task_off[mid] <= t) lo = mid; else hi = mid;
    }
    // task_off is indexed by rank; with `perm` the ranks list the buckets by decreasing size so that the
    // threads of a warp get tasks of (nearly) equal length
    const uint32_t g = perm ? perm[lo] : lo;
    const uint32_t k = t - task_off[lo];
    const uint32_t ntasks = task_off[lo + 1] - task_off[lo];
    const uint32_t beg = offsets[g] + k * sh.L;
    const uint32_t end = min(beg + sh.L, offsets[g + 1]);

    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t pos = beg; pos < end; pos++) {
        // sorted == nullptr: the bases are already in bucket order (output of the batched-affine rounds), no sign bit
        const uint32_t e = sorted ? sorted[pos] : 0u;
        Affine<F> q = ld_struct(bases + (sorted ? (e & 0x7fffffffu) : pos));
        if (e >> 31) q.y = q.y.neg();
        madd(acc, q);
    }
    if (ntasks == 1) st_struct(bucket_acc + g, acc);
    else st_struct(partials + t, acc);
}


// result = sum_w 2^(c w) S_w  (Horner from the top window): ~250 dependent doublings, the longest serial chain of an MSM.
// The four-lane teams of ec_team.cuh cut a doubling from 9 multiplication latencies to 3.  A batch of K MSMs has
// sh.nwin = K * (windows per MSM); team k of the grid (eight per warp) folds MSM k's windows into out[k].
template <class F>
__global__ void __launch_bounds__(32) msm_horner_kernel(const XYZZ<F>* __restrict__ win, MsmShape sh, uint32_t K, XYZZ<F>* __restrict__ out) {
    const uint32_t k = (blockIdx.x * blockDim.x + threadIdx.x) >> 2;
    if (k >= K) return;
    const uint32_t nw = sh.nwin / K;
    win += (size_t)k * nw;
    XYZZ<F> acc = ld_struct(win + (nw - 1));
    for (uint32_t w = nw - 1; w-- > 0;) {
        for (uint32_t i = 0; i < sh.c; i++) team_dbl(acc);
        XYZZ<F> v = ld_struct(win + w);
        team_add(acc, v);
    }
    if ((threadIdx.x & 3) == 0) st_struct(out + k, acc);
}

// Sum `count` XYZZ points with one CTA; result in out[0] (also used by the join of shard partials).
template <class F>
__device__ __forceinline__ XYZZ<F> cta_sum(const XYZZ<F>* __restrict__ pts, uint32_t count, XYZZ<F>* smem) {
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t i = threadIdx.x; i < count; i += blockDim.x) {
        XYZZ<F> v = ld_struct(pts + i);
        acc.add(v);
    }
    smem[threadIdx.x] = acc;
    __syncthreads();
    for (uint32_t d = blockDim.x >> 1; d > 0; d >>= 1) {
        if (threadIdx.x < d) {
            XYZZ<F> a = smem[threadIdx.x];
            a.add(smem[threadIdx.x + d]);
            smem[threadIdx.x] = a;
        }
        __syncthreads();
    }
    return smem[0];
}

// k * p for a small non-negative integer k (double-and-add, most significant bit first)
template <class F>
__device__ __forceinline__ XYZZ<F> mul_small(const XYZZ<F>& p, uint32_t k) {
    XYZZ<F> acc = XYZZ<F>::identity();
    if (k == 0 || p.is_identity()) return acc;
    for (int b = 31 - __clz(k); b >= 0; b--) {
        acc = acc.dbl();
        if ((k >> b) & 1) acc.add(p);
    }
    return acc;
}

// Segment sums: thread handles buckets [s0, s0 + MSM_SEG) of one window (MSM_SEG chosen by the host) (bucket index b is 0-based,
// weight b + 1):  sum (b+1) B_b = sum_{local} (j+1) B_{s0+j} + s0 * sum B_{s0+j}.
template <class F>
__global__ void __launch_bounds__(128)
msm_bucket_segments_kernel(const XYZZ<F>* __restrict__ bucket_acc, MsmShape sh, uint32_t MSM_SEG, XYZZ<F>* __restrict__ seg_out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t segs_per_win = (sh.B + MSM_SEG - 1) / MSM_SEG;
    if (t >= segs_per_win * sh.nwin) return;
    const uint32_t w = t / segs_per_win, sg = t % segs_per_win;
    const uint32_t s0 = sg * MSM_SEG, s1 = min(s0 + MSM_SEG, sh.B);
    const XYZZ<F>* bk = bucket_acc + (size_t)w * sh.B;
    XYZZ<F> run = XYZZ<F>::identity(), acc = XYZZ<F>::identity();
    for (uint32_t j = s1; j-- > s0;) {
        XYZZ<F> v = ld_struct(bk + j);
        run.add(v);
        acc.add(run);
    }
    if (s0 != 0) {
        XYZZ<F> m = mul_small(run, s0);
        acc.add(m);
    }
    st_struct(seg_out + t, acc);
}

// One CTA per window: S_w = sum of its segment results.
template <class F>
__global__ void __launch_bounds__(MSM_RED_THREADS)
msm_window_sum_kernel(const XYZZ<F>* __restrict__ seg, uint32_t segs_per_win, XYZZ<F>* __restrict__ win_out) {
    extern __shared__ uint4 smem_raw[];
    XYZZ<F>* smem = reinterpret_cast<XYZZ<F>*>(smem_raw);
    XYZZ<F> s = cta_sum(seg + (size_t)blockIdx.x * segs_per_win, segs_per_win, smem);
    if (threadIdx.x == 0) st_struct(win_out + blockIdx.x, s);
}

template <class F>
static int32_t msm_bucket_reduce_launch(Ctx* c, const char* l_seg, const char* l_win, const void* bucket_acc, MsmShape sh, uint32_t seg, void* segs,
                                        uint32_t segs_per_win, void* wins) {
    using Pt = XYZZ<F>;
    const size_t red_smem = (size_t)MSM_RED_THREADS * sizeof(Pt);
    B2S_SMEM_ATTR(c, msm_window_sum_kernel<F>, red_smem);
    B2S_LAUNCH_N(c, l_seg, msm_bucket_segments_kernel<F>, cdiv((uint64_t)segs_per_win * sh.nwin, 128), 128, 0, reinterpret_cast<const Pt*>(bucket_acc), sh, seg,
                 reinterpret_cast<Pt*>(segs));
    B2S_LAUNCH_N(c, l_win, msm_window_sum_kernel<F>, sh.nwin, MSM_RED_THREADS, red_smem, reinterpret_cast<const Pt*>(segs), segs_per_win, reinterpret_cast<Pt*>(wins));
    return B2S_OK;
}
int32_t msm_bucket_reduce_g1(Ctx* c, const void* bucket_acc, MsmShape sh, uint32_t seg, void* segs, uint32_t segs_per_win, void* wins);
int32_t msm_bucket_reduce_g2(Ctx* c, const void* bucket_acc, MsmShape sh, uint32_t seg, void* segs, uint32_t segs_per_win, void* wins);

// launches compiled with the multiplication inlined: msm_acc_g1.cu (G1) and msm_acc_g2.cu (G2)
int32_t msm_accumulate_g2(Ctx* c, const void* bases, const uint32_t* sorted, const uint32_t* offsets,
                          const uint32_t* task_off, const uint32_t* perm, MsmShape sh, void* bucket_acc, void* partials);
int32_t msm_horner_g1(Ctx* c, cudaStream_t st, const void* wins, MsmShape sh, uint32_t K, void* out);
int32_t msm_horner_g2(Ctx* c, cudaStream_t st, const void* wins, MsmShape sh, uint32_t K, void* out);
inline int32_t msm_horner(Ctx* c, cudaStream_t st, int group, const void* wins, MsmShape sh, uint32_t K, void* out) {
    return group == 1 ? msm_horner_g1(c, st, wins, sh, K, out) : msm_horner_g2(c, st, wins, sh, K, out);
}
// G1 accumulate for the ctx's curve (msm_acc_g1.cu)
int32_t msm_accumulate_g1(Ctx* c, const void* bases, const uint32_t* sorted, const uint32_t* offsets,
                          const uint32_t* task_off, const uint32_t* perm, MsmShape sh, void* bucket_acc, void* partials);

}  // namespace b2s
