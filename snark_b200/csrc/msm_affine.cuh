// Batched-affine pairwise reduction rounds in front of the XYZZ bucket accumulation (step 3b of msm.cu).
//
// A round halves every bucket: the points of a bucket (contiguous in the bucket-sorted order) are added in
// adjacent pairs IN AFFINE coordinates,  lambda = (y2 - y1) / (x2 - x1),  x3 = lambda^2 - x1 - x2,
// y3 = lambda (x1 - x3) - y1.  All pairs of a round are independent, so the divisions share inversions
// (Montgomery's trick): 6 multiplications per addition instead of the 10 of an XYZZ mixed addition (Fq2: 17 base
// multiplications instead of 28).  After R rounds every bucket holds ceil(n / 2^R) points and the XYZZ kernel
// (msm_acc.cuh) finishes.  All special cases keep the result an exact group element: missing partner /
// infinity -> copy, P + P -> tangent, P + (-P) -> infinity.
//
// Work decomposition (this is what makes the round ALU-bound instead of latency-bound):
//   * outputs of a round are numbered 0 .. T_out-1 in bucket order; 32 consecutive outputs form a ROW, lane l of
//     a warp owns output 32 q + l of row q, K consecutive rows form a UNIT (one warp, one inversion chain per
//     lane).  Work per unit is the same whatever the bucket sizes, so all-equal witnesses (one bucket per window
//     holding every point, relations/src/sr1cs/mod.rs:306-309) and uniform scalars run at the same rate.
//   * where an output's inputs sit follows from one bit per output: `single` = last output of a bucket with an
//     odd count (it has no partner).  inputs of output o = positions 2 o - rank(o) and +1, rank(o) = number of
//     single outputs before o = wrank[q] + popc(bitmap[q] & lanes below).  No per-thread bucket walk.
//   * pass 1 (msm_ba_p1_kernel): per lane, prefix products of the denominators d = x2 - x1 down its K rows
//     (x coordinates only), prefix to HBM (coalesced), lane total to tot[].
//   * inversion (msm_ba_inv_kernel): the lane totals are inverted with the same trick one level up, K2 totals
//     per inversion -- one inversion per 32 K K2 / 32 additions instead of one per K.
//   * pass 2 (msm_ba_p2_kernel): backwards down the rows: 1/d from the running inverse and the stored prefix,
//     then the addition itself; results to HBM (coalesced, bucket order).
//   * operands never wait in registers: each lane stages its own points / x's / prefix for the next rows in a
//     private shared-memory slot ring with cp.async (LDGSTS, 16 B granules, L1 bypass), descriptors (bitmap word,
//     sorted indices) one and two rows further ahead in registers.  A lane only ever reads its own slot, so no
//     barrier is needed -- cp.async.wait_group orders a lane's copies before its reads.
//     Slot stride = odd multiple of 16 B: conflict-free for the 16-byte shared-memory accesses used throughout.
#pragma once
#include <algorithm>

#include "msm_acc.cuh"

namespace b2s {

enum : uint32_t { BA_COPY1 = 0, BA_COPY2 = 1, BA_ADD = 2, BA_DBL = 3, BA_INF = 4 };
enum : uint32_t { BA_F_VALID = 1u, BA_F_SINGLE = 2u };

static constexpr uint32_t BA_KMIN = 16, BA_KMAX = 256;   // rows per unit (chosen on the device from the round's size)
// lane totals per inversion.  The kernel is a few warps per SM, so its time is one thread's chain: K2 products, one
// divsteps inversion (~1100 divsteps) and 2 K2 products back.  32 made the 96 dependent products the longest part once
// the inversion stopped being a 608-product Fermat chain; 16 halves them and still keeps the ~17 k inversions of a
// 2^24 round few enough that their instruction count does not make the kernel issue-bound.
static constexpr uint32_t BA_K2 = 16;
static constexpr uint32_t BA_P1_STAGES = 3, BA_P2_STAGES = 2;

__host__ __device__ constexpr uint32_t ba_slot_bytes(uint32_t n) { return ((((n + 15u) / 16u) | 1u)) * 16u; }

template <class F>
struct BaGeom {
    static constexpr uint32_t FE = sizeof(F), PT = sizeof(Affine<F>);
    static constexpr uint32_t THREADS_ = sizeof(F) > 64 ? 64 : 128;
    static constexpr uint32_t P1_META = 2 * FE, P1_SLOT = ba_slot_bytes(2 * FE + 16);
    // pass 2 stages the two points only; the prefix product travels through registers (one row ahead) so that the slot
    // ring of 16 warps fits an SM: occupancy is what hides the dependent-issue latency of the carry chains
    static constexpr uint32_t P2_META = 2 * PT, P2_SLOT = ba_slot_bytes(2 * PT + 16);
    // threads per CTA: the G2 slots are twice as big, so half the threads keep three CTAs per SM
    static constexpr uint32_t THREADS = THREADS_;
    // streaming rounds: one bulk copy (TMA engine) per warp row brings the row's 64 - #singles input points, which are
    // contiguous in the previous round's output; stage = [64 points][32 x 16 B of per-lane meta][mbarrier]
    static constexpr uint32_t P2B_META = 64 * PT, P2B_MBAR = 64 * PT + 32 * 16, P2B_STAGE = 64 * PT + 32 * 16 + 16;
    static constexpr uint32_t P2B_SMEM = (THREADS_ / 32) * BA_P2_STAGES * P2B_STAGE;
    static constexpr uint32_t P2_MIN_CTAS = 4;      // register cap of pass 2: 65536 / (THREADS * 4) = 128 (G1) / 256 (G2)
    static constexpr uint32_t P1_SMEM = THREADS * BA_P1_STAGES * P1_SLOT, P2_SMEM = THREADS * BA_P2_STAGES * P2_SLOT;
};

// rows per unit for a round with n_rows rows: enough units to fill the machine, chains as long as that allows
__host__ __device__ inline uint32_t ba_rows_per_unit(uint32_t n_rows, uint32_t target_units) {
    uint32_t k = (n_rows + target_units - 1) / target_units;
    return k < BA_KMIN ? BA_KMIN : (k > BA_KMAX ? BA_KMAX : k);
}

// ---- cp.async (LDGSTS) ---------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t smem_addr, const void* gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_addr), "l"(gsrc) : "memory");
}
template <uint32_t BYTES>
__device__ __forceinline__ void cp_async_bytes(uint32_t smem_addr, const void* gsrc) {
    static_assert(BYTES % 16 == 0, "16-byte granules");
#pragma unroll
    for (uint32_t i = 0; i < BYTES; i += 16) cp_async16(smem_addr + i, reinterpret_cast<const char*>(gsrc) + i);
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// ---- bulk asynchronous copies (TMA engine, cp.async.bulk) completing on an mbarrier ----------------------------------
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t smem_dst, const void* gsrc, uint32_t bytes, uint32_t mbar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst), "l"(gsrc), "r"(bytes), "r"(mbar)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(mbar), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <class T>
__device__ __forceinline__ T lds_struct(uint32_t smem_addr) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiples only");
    T r;
    uint4* d = reinterpret_cast<uint4*>(&r);
#pragma unroll
    for (uint32_t i = 0; i < sizeof(T) / 16; i++)
        asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(d[i].x), "=r"(d[i].y), "=r"(d[i].z), "=r"(d[i].w) : "r"(smem_addr + 16 * i));
    return r;
}
__device__ __forceinline__ uint4 lds16(uint32_t smem_addr) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_addr));
    return v;
}
__device__ __forceinline__ void sts16(uint32_t smem_addr, uint4 v) {
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(smem_addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// coherent vector load (for buffers the same kernel also writes)
template <class T>
__device__ __forceinline__ T ld_plain(const T* p) {
    static_assert(sizeof(T) % 16 == 0, "16-byte multiples only");
    T r;
    const uint4* s = reinterpret_cast<const uint4*>(p);
    uint4* d = reinterpret_cast<uint4*>(&r);
#pragma unroll
    for (int i = 0; i < (int)(sizeof(T) / 16); i++) d[i] = s[i];
    return r;
}

// ---- pair classification (identical in both passes: the denominators must agree) ---------------------
template <class F>
__device__ __forceinline__ uint32_t ba_classify(const Affine<F>& p1, const Affine<F>& p2, bool single) {
    if (single || p2.is_inf()) return BA_COPY1;
    if (p1.is_inf()) return BA_COPY2;
    if (p1.x == p2.x) return (p1.y == p2.y && !p1.y.is_zero()) ? BA_DBL : BA_INF;
    return BA_ADD;
}
template <class F>
__device__ __forceinline__ F ba_denominator(uint32_t kind, const Affine<F>& p1, const Affine<F>& p2) {
    if (kind == BA_ADD) return p2.x - p1.x;
    if (kind == BA_DBL) return p1.y.dbl();
    return F::one();
}

// units are handed out dynamically (one atomic per unit): warps that draw shorter rows or faster memory simply take more
__device__ __forceinline__ uint32_t ba_next_unit(uint32_t* ctr, uint32_t lane) {
    uint32_t u = 0;
    if (lane == 0) u = atomicAdd(ctr, 1u);
    return __shfl_sync(0xffffffffu, u, 0);
}

// One output of pass 2: 1 / d from the running inverse and the stored prefix (2 multiplications), then the affine addition
// (3 more); `inv` moves on to the previous output of the lane's chain.
template <class F>
__device__ __forceinline__ Affine<F> ba_output(const Affine<F>& p1, const Affine<F>& p2, bool single, F& inv, const F& pre) {
    const uint32_t kind = ba_classify(p1, p2, single);
    const F d = ba_denominator(kind, p1, p2);
    const F dinv = inv * pre;
    inv = inv * d;
    Affine<F> res;
    if (kind == BA_ADD || kind == BA_DBL) {
        F num;
        if (kind == BA_ADD) num = p2.y - p1.y;
        else { F xx = p1.x.sqr(); num = xx.dbl() + xx; }
        const F lam = num * dinv;
        const F x3 = lam.sqr() - p1.x - p2.x;   // DBL: p2 == p1, so this is lambda^2 - 2 x1
        res.x = x3;
        res.y = lam * (p1.x - x3) - p1.y;
    } else if (kind == BA_COPY1) res = p1;
    else if (kind == BA_COPY2) res = p2;
    else res = Affine<F>::inf();
    return res;
}

// descriptor of (row q, this lane): where its inputs are
struct BaDesc { uint32_t in0, flags; };
__device__ __forceinline__ BaDesc ba_desc(uint32_t word, uint32_t wr, uint32_t q, uint32_t lane, uint32_t t_out) {
    const uint32_t o = q * 32u + lane;
    BaDesc d;
    d.flags = (o < t_out ? BA_F_VALID : 0u) | (((word >> lane) & 1u) ? BA_F_SINGLE : 0u);
    d.in0 = 2u * o - (wr + __popc(word & ((1u << lane) - 1u)));
    return d;
}

// rare path of pass 1: the pair is not a plain addition (or might not be): fetch the y's and classify exactly
template <class F, bool FIRST>
__device__ __noinline__ F ba_slow_denominator(const Affine<F>* __restrict__ bases, const Affine<F>* __restrict__ prev, uint32_t e1,
                                              uint32_t e2, uint32_t in0, bool single) {
    Affine<F> p1, p2;
    if (FIRST) {
        p1 = ld_struct(bases + (e1 & 0x7fffffffu));
        if (e1 >> 31) p1.y = p1.y.neg();
        if (!single) {
            p2 = ld_struct(bases + (e2 & 0x7fffffffu));
            if (e2 >> 31) p2.y = p2.y.neg();
        }
    } else {
        p1 = ld_struct(prev + in0);
        if (!single) p2 = ld_struct(prev + in0 + 1);
    }
    if (single) p2 = Affine<F>::inf();
    return ba_denominator(ba_classify(p1, p2, single), p1, p2);
}

// ---- pass 1 -------------------------------------------------------------------------------------------
// Software pipeline per lane, time step t:  consume row t-S | issue the copies of row t into the slot just freed |
// descriptor + sorted indices of row t+1 | bitmap word of row t+2.  A row's operands are in flight during the S-1
// row computations before its own.
template <class F, bool FIRST>
__global__ void __launch_bounds__(BaGeom<F>::THREADS)
msm_ba_p1_kernel(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ sorted, const Affine<F>* __restrict__ prev,
                 const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ wrank, const uint32_t* __restrict__ t_out_p,
                 uint32_t target_units, uint32_t* __restrict__ unit_ctr, F* __restrict__ prefix, F* __restrict__ tot) {
    using Gm = BaGeom<F>;
    constexpr uint32_t S = BA_P1_STAGES, FE = Gm::FE, SLOT = Gm::P1_SLOT, META = Gm::P1_META;
    extern __shared__ uint4 ba_smem[];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(ba_smem) + (warp * S * 32u + lane) * SLOT;
    const uint32_t t_out = *t_out_p;
    const uint32_t n_rows = (t_out + 31u) >> 5;
    const uint32_t K = ba_rows_per_unit(n_rows, target_units);
    const uint32_t n_units = (n_rows + K - 1) / K;
    for (uint32_t u = ba_next_unit(unit_ctr, lane); u < n_units; u = ba_next_unit(unit_ctr, lane)) {
        const uint32_t q0 = u * K, nr = min(K, n_rows - q0);
        F prod = F::one();
        uint32_t a_word = 0, a_wr = 0;                 // stage A -> B
        uint32_t b_e1 = 0, b_e2 = 0;                   // stage B -> C
        BaDesc b_d{0, 0};
        for (int32_t t = -2; t < (int32_t)(nr + S); t++) {
            // -- consume row t - S
            if (t >= (int32_t)S) {
                cp_async_wait<(int)S - 1>();
                const uint32_t i = (uint32_t)t - S;
                const uint32_t slot = smem0 + (i % S) * 32u * SLOT;
                const uint4 meta = lds16(slot + META);   // e1, e2, in0, flags
                if (meta.w & BA_F_VALID) {
                    const bool single = (meta.w & BA_F_SINGLE) != 0;
                    const uint32_t o = (q0 + i) * 32u + lane;
                    F d = F::one();                              // no partner: the output is a copy
                    if (!single) {
                        const F x1 = lds_struct<F>(slot), x2 = lds_struct<F>(slot + FE);
                        // x = 0 may be the (0,0) encoding of infinity, equal x means doubling or cancellation
                        if (!x1.is_zero() && !x2.is_zero() && x1 != x2) d = x2 - x1;
                        else d = ba_slow_denominator<F, FIRST>(bases, prev, meta.x, meta.y, meta.z, false);
                    }
                    st_struct(prefix + o, prod);
                    prod = prod * d;
                }
            }
            // -- issue the copies of row t (descriptor from the previous step); its slot was freed just above
            if (t >= 0 && (uint32_t)t < nr) {
                const uint32_t slot = smem0 + ((uint32_t)t % S) * 32u * SLOT;
                if (b_d.flags & BA_F_VALID) {
                    const F* px1 = FIRST ? &bases[b_e1 & 0x7fffffffu].x : &prev[b_d.in0].x;
                    cp_async_bytes<FE>(slot, px1);
                    if (!(b_d.flags & BA_F_SINGLE)) {
                        const F* px2 = FIRST ? &bases[b_e2 & 0x7fffffffu].x : &prev[b_d.in0 + 1].x;
                        cp_async_bytes<FE>(slot + FE, px2);
                    }
                }
                sts16(slot + META, make_uint4(b_e1, b_e2, b_d.in0, b_d.flags));
            }
            cp_async_commit();
            // -- descriptor of row t + 1, its sorted indices
            if (t + 1 >= 0 && (uint32_t)(t + 1) < nr) {
                b_d = ba_desc(a_word, a_wr, q0 + (uint32_t)(t + 1), lane, t_out);
                if (FIRST && (b_d.flags & BA_F_VALID)) {
                    b_e1 = sorted[b_d.in0];
                    b_e2 = (b_d.flags & BA_F_SINGLE) ? 0u : sorted[b_d.in0 + 1];
                }
            }
            // -- bitmap word of row t + 2
            if ((uint32_t)(t + 2) < nr) {
                a_word = bitmap[q0 + (uint32_t)(t + 2)];
                a_wr = wrank[q0 + (uint32_t)(t + 2)];
            }
        }
        st_struct(tot + (size_t)u * 32u + lane, prod);
    }
}

// ---- inversion of the lane totals, in place ------------------------------------------------------------
template <class F>
__global__ void __launch_bounds__(128)
msm_ba_inv_kernel(F* __restrict__ tot, const uint32_t* __restrict__ t_out_p, uint32_t target_units, F* __restrict__ scratch) {
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t t_out = *t_out_p;
    const uint32_t n_rows = (t_out + 31u) >> 5;
    const uint32_t K = ba_rows_per_unit(n_rows, target_units);
    const uint32_t n_tot = ((n_rows + K - 1) / K) * 32u;
    const uint32_t n_units = (n_tot + 32u * BA_K2 - 1) / (32u * BA_K2);
    const uint32_t warps_total = gridDim.x * (blockDim.x >> 5);
    for (uint32_t v = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); v < n_units; v += warps_total) {
        const uint32_t e0 = v * 32u * BA_K2 + lane;
        F prod = F::one();
        for (uint32_t j = 0; j < BA_K2; j++) {
            const uint32_t e = e0 + 32u * j;
            if (e < n_tot) {
                F t = ld_plain(tot + e);
                st_struct(scratch + e, prod);
                prod = prod * t;
            }
        }
        F inv = prod.inverse();
        for (uint32_t j = BA_K2; j-- > 0;) {
            const uint32_t e = e0 + 32u * j;
            if (e < n_tot) {
                F t = ld_plain(tot + e);
                F p = ld_plain(scratch + e);
                st_struct(tot + e, inv * p);
                inv = inv * t;
            }
        }
    }
}

// ---- pass 2 -------------------------------------------------------------------------------------------
// Same pipeline as pass 1, rows in descending order (the running inverse walks the chain backwards).
template <class F, bool FIRST>
__global__ void __launch_bounds__(BaGeom<F>::THREADS, BaGeom<F>::P2_MIN_CTAS)
msm_ba_p2_kernel(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ sorted, const Affine<F>* __restrict__ prev,
                 const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ wrank, const uint32_t* __restrict__ t_out_p,
                 uint32_t target_units, uint32_t* __restrict__ unit_ctr, const F* __restrict__ prefix, const F* __restrict__ tot_inv,
                 Affine<F>* __restrict__ out) {
    using Gm = BaGeom<F>;
    constexpr uint32_t S = BA_P2_STAGES, PT = Gm::PT;
    extern __shared__ uint4 ba_smem[];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t smem0 = (uint32_t)__cvta_generic_to_shared(ba_smem) + (warp * S * 32u + lane) * Gm::P2_SLOT;
    const uint32_t t_out = *t_out_p;
    const uint32_t n_rows = (t_out + 31u) >> 5;
    const uint32_t K = ba_rows_per_unit(n_rows, target_units);
    const uint32_t n_units = (n_rows + K - 1) / K;
    for (uint32_t u = ba_next_unit(unit_ctr, lane); u < n_units; u = ba_next_unit(unit_ctr, lane)) {
        const uint32_t q0 = u * K, nr = min(K, n_rows - q0);
        F inv = ld_struct(tot_inv + (size_t)u * 32u + lane);
        uint32_t a_word = 0, a_wr = 0, b_e1 = 0, b_e2 = 0;
        BaDesc b_d{0, 0};
        F pre_next = F::one();    // prefix product of the row consumed next (fetched while the current row computes)
        {
            const uint32_t o0 = (q0 + nr - 1) * 32u + lane;
            if (o0 < t_out) pre_next = ld_struct(prefix + o0);
        }
        // step index i counts rows from the last one down: row q = q0 + nr - 1 - i
        for (int32_t t = -2; t < (int32_t)(nr + S); t++) {
            if (t >= (int32_t)S) {
                cp_async_wait<(int)S - 1>();
                const uint32_t i = (uint32_t)t - S;
                const uint32_t slot = smem0 + (i % S) * 32u * Gm::P2_SLOT;
                const uint4 meta = lds16(slot + Gm::P2_META);   // neg1, neg2, in0, flags
                const F pre_cur = pre_next;
                // the next row's prefix: requested now, used one row of arithmetic later
                if (i + 1 < nr) {
                    const uint32_t on = (q0 + nr - 2 - i) * 32u + lane;
                    if (on < t_out) pre_next = ld_struct(prefix + on);
                }
                if (meta.w & BA_F_VALID) {
                    const bool single = (meta.w & BA_F_SINGLE) != 0;
                    const uint32_t o = (q0 + nr - 1 - i) * 32u + lane;
                    Affine<F> p1 = lds_struct<Affine<F>>(slot), p2;
                    if (FIRST && meta.x) p1.y = p1.y.neg();
                    if (!single) {
                        p2 = lds_struct<Affine<F>>(slot + PT);
                        if (FIRST && meta.y) p2.y = p2.y.neg();
                    } else {
                        p2 = Affine<F>::inf();
                    }
                    st_struct(out + o, ba_output(p1, p2, single, inv, pre_cur));
                }
            }
            if (t >= 0 && (uint32_t)t < nr) {
                const uint32_t slot = smem0 + ((uint32_t)t % S) * 32u * Gm::P2_SLOT;
                if (b_d.flags & BA_F_VALID) {
                    const Affine<F>* a1 = FIRST ? bases + (b_e1 & 0x7fffffffu) : prev + b_d.in0;
                    cp_async_bytes<PT>(slot, a1);
                    if (!(b_d.flags & BA_F_SINGLE)) {
                        const Affine<F>* a2 = FIRST ? bases + (b_e2 & 0x7fffffffu) : prev + b_d.in0 + 1;
                        cp_async_bytes<PT>(slot + PT, a2);
                    }
                }
                sts16(slot + Gm::P2_META, make_uint4(b_e1 >> 31, b_e2 >> 31, b_d.in0, b_d.flags));
            }
            cp_async_commit();
            if (t + 1 >= 0 && (uint32_t)(t + 1) < nr) {
                b_d = ba_desc(a_word, a_wr, q0 + nr - 1 - (uint32_t)(t + 1), lane, t_out);
                if (FIRST && (b_d.flags & BA_F_VALID)) {
                    b_e1 = sorted[b_d.in0];
                    b_e2 = (b_d.flags & BA_F_SINGLE) ? 0u : sorted[b_d.in0 + 1];
                }
            }
            if ((uint32_t)(t + 2) < nr) {
                a_word = bitmap[q0 + nr - 1 - (uint32_t)(t + 2)];
                a_wr = wrank[q0 + nr - 1 - (uint32_t)(t + 2)];
            }
        }
    }
}

// ---- pass 2 of the streaming rounds: operands by bulk copy --------------------------------------------------------------
// In every round but the first the inputs of a warp row -- 64 points minus one per single output -- are CONTIGUOUS in the
// previous round's output.  One lane arms an mbarrier with the byte count and issues ONE cp.async.bulk (TMA engine) for
// the whole row, two rows ahead of its use; the 32 lanes wait on the barrier's phase and read their points at
// (in0 - in0 of lane 0) * sizeof(point).  Replaces 12-24 LDGSTS per lane and row by one instruction per warp and row.
template <class F>
__global__ void __launch_bounds__(BaGeom<F>::THREADS, BaGeom<F>::P2_MIN_CTAS)
msm_ba_p2_bulk_kernel(const Affine<F>* __restrict__ prev, const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ wrank,
                      const uint32_t* __restrict__ t_out_p, uint32_t target_units, uint32_t* __restrict__ unit_ctr, const F* __restrict__ prefix,
                      const F* __restrict__ tot_inv, Affine<F>* __restrict__ out) {
    using Gm = BaGeom<F>;
    constexpr uint32_t S = BA_P2_STAGES, PT = Gm::PT;
    static_assert(S == 2, "parity bookkeeping below is written for two stages");
    extern __shared__ uint4 ba_smem[];
    const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    const uint32_t stage0 = (uint32_t)__cvta_generic_to_shared(ba_smem) + warp * S * Gm::P2B_STAGE;
    if (lane == 0) {
        mbar_init(stage0 + Gm::P2B_MBAR, 1);
        mbar_init(stage0 + Gm::P2B_STAGE + Gm::P2B_MBAR, 1);
        mbar_fence_init();
    }
    __syncwarp();
    uint32_t uses0 = 0, uses1 = 0;     // completed phases of the two stage barriers (warp-uniform)
    const uint32_t t_out = *t_out_p;
    const uint32_t n_rows = (t_out + 31u) >> 5;
    const uint32_t K = ba_rows_per_unit(n_rows, target_units);
    const uint32_t n_units = (n_rows + K - 1) / K;
    for (uint32_t u = ba_next_unit(unit_ctr, lane); u < n_units; u = ba_next_unit(unit_ctr, lane)) {
        const uint32_t q0 = u * K, nr = min(K, n_rows - q0);
        F inv = ld_struct(tot_inv + (size_t)u * 32u + lane);
        uint32_t a_word = 0, a_wr = 0;
        BaDesc b_d{0, 0};
        F pre_next = F::one();
        {
            const uint32_t o0 = (q0 + nr - 1) * 32u + lane;
            if (o0 < t_out) pre_next = ld_struct(prefix + o0);
        }
        for (int32_t t = -2; t < (int32_t)(nr + S); t++) {
            if (t >= (int32_t)S) {
                const uint32_t i = (uint32_t)t - S;
                const uint32_t st = stage0 + (i & 1u) * Gm::P2B_STAGE;
                mbar_wait(st + Gm::P2B_MBAR, (i & 1u) ? (uses1 & 1u) : (uses0 & 1u));
                if (i & 1u) uses1++; else uses0++;
                const uint4 meta = lds16(st + Gm::P2B_META + lane * 16u);   // point offset in the stage, -, -, flags
                const F pre_cur = pre_next;
                if (i + 1 < nr) {
                    const uint32_t on = (q0 + nr - 2 - i) * 32u + lane;
                    if (on < t_out) pre_next = ld_struct(prefix + on);
                }
                if (meta.w & BA_F_VALID) {
                    const bool single = (meta.w & BA_F_SINGLE) != 0;
                    const uint32_t o = (q0 + nr - 1 - i) * 32u + lane;
                    const Affine<F> p1 = lds_struct<Affine<F>>(st + meta.x * PT);
                    const Affine<F> p2 = single ? Affine<F>::inf() : lds_struct<Affine<F>>(st + (meta.x + 1u) * PT);
                    st_struct(out + o, ba_output(p1, p2, single, inv, pre_cur));
                }
                __syncwarp();      // every lane is done reading this stage before it is refilled below
            }
            if (t >= 0 && (uint32_t)t < nr) {
                const uint32_t st = stage0 + ((uint32_t)t & 1u) * Gm::P2B_STAGE;
                // the row's inputs: from lane 0's first point to the last valid lane's last point
                const uint32_t valid = __ballot_sync(0xffffffffu, (b_d.flags & BA_F_VALID) != 0);
                const uint32_t last = 31u - (uint32_t)__clz((int)valid);          // lane 0 of a row is always valid
                const uint32_t first_in = __shfl_sync(0xffffffffu, b_d.in0, 0);
                const uint32_t end_in = __shfl_sync(0xffffffffu, b_d.in0 + ((b_d.flags & BA_F_SINGLE) ? 1u : 2u), (int)last);
                sts16(st + Gm::P2B_META + lane * 16u, make_uint4(b_d.in0 - first_in, 0u, 0u, b_d.flags));
                if (lane == 0) {
                    const uint32_t bytes = (end_in - first_in) * PT;
                    fence_proxy_async();                                            // generic reads of the stage before the async write
                    mbar_expect_tx(st + Gm::P2B_MBAR, bytes);
                    bulk_g2s(st, prev + first_in, bytes, st + Gm::P2B_MBAR);
                }
            }
            if (t + 1 >= 0 && (uint32_t)(t + 1) < nr) b_d = ba_desc(a_word, a_wr, q0 + nr - 1 - (uint32_t)(t + 1), lane, t_out);
            if ((uint32_t)(t + 2) < nr) {
                a_word = bitmap[q0 + nr - 1 - (uint32_t)(t + 2)];
                a_wr = wrank[q0 + nr - 1 - (uint32_t)(t + 2)];
            }
        }
    }
}

// ---- round bookkeeping (tiny kernels, msm.cu) ---------------------------------------------------------
// counts_next[g] = ceil(counts[g] / 2)
static __global__ void msm_ba_halve_kernel(const uint32_t* __restrict__ counts, uint32_t G, uint32_t* __restrict__ next) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g < G) next[g] = (counts[g] + 1) >> 1;
}
// one bit per output of the round: set for the last output of a bucket whose input count is odd
static __global__ void msm_ba_singles_kernel(const uint32_t* __restrict__ counts_in, const uint32_t* __restrict__ off_out, uint32_t G,
                                             uint32_t* __restrict__ bitmap) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const uint32_t c = counts_in[g];
    if (c & 1u) {
        const uint32_t last = off_out[g] + ((c + 1u) >> 1) - 1u;
        atomicOr(&bitmap[last >> 5], 1u << (last & 31u));
    }
}
// wrank[w] = number of set bits in bitmap[0 .. w)   (three kernels: tile sums, spine, apply)
static constexpr uint32_t BA_SCAN_THREADS = 256, BA_SCAN_PER = 8, BA_SCAN_TILE = BA_SCAN_THREADS * BA_SCAN_PER;
__device__ __forceinline__ uint32_t ba_block_scan_incl(uint32_t v, uint32_t* total) {
    __shared__ uint32_t wsum[32];
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= (uint32_t)d) v += o;
    }
    if (lane == 31) wsum[wid] = v;
    __syncthreads();
    const uint32_t nw = (blockDim.x + 31u) >> 5;
    if (wid == 0) {
        uint32_t w = lane < nw ? wsum[lane] : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= (uint32_t)d) w += o;
        }
        wsum[lane] = w;
    }
    __syncthreads();
    if (wid > 0) v += wsum[wid - 1];
    *total = wsum[nw - 1];
    __syncthreads();
    return v;
}
static __global__ void __launch_bounds__(BA_SCAN_THREADS)
msm_ba_rank_tiles_kernel(const uint32_t* __restrict__ bitmap, uint32_t n_words, uint32_t* __restrict__ tile_sums) {
    const uint32_t base = blockIdx.x * BA_SCAN_TILE + threadIdx.x * BA_SCAN_PER;
    uint32_t v = 0;
#pragma unroll
    for (uint32_t k = 0; k < BA_SCAN_PER; k++)
        if (base + k < n_words) v += __popc(bitmap[base + k]);
    uint32_t total;
    ba_block_scan_incl(v, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
static __global__ void __launch_bounds__(1024) msm_ba_rank_spine_kernel(uint32_t* __restrict__ tile_sums, uint32_t n_tiles) {
    const uint32_t per = (n_tiles + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(threadIdx.x * per, n_tiles), hi = min(lo + per, n_tiles);
    uint32_t v = 0;
    for (uint32_t i = lo; i < hi; i++) v += tile_sums[i];
    uint32_t total;
    uint32_t run = ba_block_scan_incl(v, &total) - v;
    for (uint32_t i = lo; i < hi; i++) {
        const uint32_t t = tile_sums[i];
        tile_sums[i] = run;
        run += t;
    }
}
static __global__ void __launch_bounds__(BA_SCAN_THREADS)
msm_ba_rank_apply_kernel(const uint32_t* __restrict__ bitmap, uint32_t n_words, const uint32_t* __restrict__ tile_sums,
                         uint32_t* __restrict__ wrank) {
    const uint32_t base = blockIdx.x * BA_SCAN_TILE + threadIdx.x * BA_SCAN_PER;
    uint32_t c[BA_SCAN_PER], v = 0;
#pragma unroll
    for (uint32_t k = 0; k < BA_SCAN_PER; k++) {
        c[k] = base + k < n_words ? __popc(bitmap[base + k]) : 0u;
        v += c[k];
    }
    uint32_t total;
    uint32_t run = tile_sums[blockIdx.x] + ba_block_scan_incl(v, &total) - v;
#pragma unroll
    for (uint32_t k = 0; k < BA_SCAN_PER; k++) {
        if (base + k < n_words) wrank[base + k] = run;
        run += c[k];
    }
}

// One round's three arithmetic kernels; implemented in msm_acc_g1.cu / msm_acc_g2.cu (multiplication inlined).
struct BaRoundArgs {
    bool first;
    const void* bases;            // first round: the MSM's bases, gathered through `sorted`
    const uint32_t* sorted;
    const void* prev;             // later rounds: the previous round's output (bucket order)
    const uint32_t* bitmap;
    const uint32_t* wrank;
    const uint32_t* t_out;        // device: number of outputs of this round
    uint32_t target_units;
    uint32_t* unit_ctr;           // two zeroed counters (pass 1, pass 2)
    void* prefix;                 // F[t_out bound]
    void* tot;                    // F[lane totals bound]
    void* inv_scratch;            // F[lane totals bound]
    void* out;                    // Affine<F>[t_out bound]
};
int32_t msm_ba_round_g1(Ctx* c, const BaRoundArgs& a);
int32_t msm_ba_round_g2(Ctx* c, const BaRoundArgs& a);

template <class F>
static int32_t msm_ba_round_launch(Ctx* c, const char* l1, const char* li, const char* l2, const BaRoundArgs& a) {
    using Gm = BaGeom<F>;
    const Affine<F>* bases = reinterpret_cast<const Affine<F>*>(a.bases);
    const Affine<F>* prev = reinterpret_cast<const Affine<F>*>(a.prev);
    F* prefix = reinterpret_cast<F*>(a.prefix);
    F* tot = reinterpret_cast<F*>(a.tot);
    // persistent grids: four CTAs per SM for pass 2 (16 warps; register- and shared-memory-bound there), up to five for pass 1
    const unsigned ctas = 4u * (unsigned)c->sm_count;
    auto fit = [&](uint32_t smem) { return (unsigned)c->sm_count * std::max(1u, std::min(5u, (224u * 1024u) / (smem + 1024u))); };
    Affine<F>* out = reinterpret_cast<Affine<F>*>(a.out);
    if (a.first) {
        B2S_SMEM_ATTR(c, (msm_ba_p1_kernel<F, true>), Gm::P1_SMEM);
        B2S_LAUNCH_N(c, l1, (msm_ba_p1_kernel<F, true>), fit(Gm::P1_SMEM), Gm::THREADS, Gm::P1_SMEM, bases, a.sorted, prev, a.bitmap, a.wrank,
                     a.t_out, a.target_units, a.unit_ctr, prefix, tot);
    } else {
        B2S_SMEM_ATTR(c, (msm_ba_p1_kernel<F, false>), Gm::P1_SMEM);
        B2S_LAUNCH_N(c, l1, (msm_ba_p1_kernel<F, false>), fit(Gm::P1_SMEM), Gm::THREADS, Gm::P1_SMEM, bases, a.sorted, prev, a.bitmap, a.wrank,
                     a.t_out, a.target_units, a.unit_ctr, prefix, tot);
    }
    B2S_LAUNCH_N(c, li, msm_ba_inv_kernel<F>, 4 * c->sm_count, 128, 0, tot, a.t_out, a.target_units, reinterpret_cast<F*>(a.inv_scratch));
    if (a.first) {
        B2S_SMEM_ATTR(c, (msm_ba_p2_kernel<F, true>), Gm::P2_SMEM);
        B2S_LAUNCH_N(c, l2, (msm_ba_p2_kernel<F, true>), ctas, Gm::THREADS, Gm::P2_SMEM, bases, a.sorted, prev, a.bitmap, a.wrank, a.t_out,
                     a.target_units, a.unit_ctr + 1, (const F*)prefix, (const F*)tot, out);
    } else if (sizeof(F) <= 64) {
        // later rounds read the previous round's output, where a row's inputs are contiguous: bulk copies for G1, the per-lane
        // cp.async ring for G2 (pass 2, 2^24 uniform points, H100 80GB HBM3 at 400 W: G1 67.0 vs 69.8 ms, G2 215.6 vs 217.0 ms)
        B2S_SMEM_ATTR(c, msm_ba_p2_bulk_kernel<F>, Gm::P2B_SMEM);
        B2S_LAUNCH_N(c, l2, msm_ba_p2_bulk_kernel<F>, ctas, Gm::THREADS, Gm::P2B_SMEM, prev, a.bitmap, a.wrank, a.t_out, a.target_units, a.unit_ctr + 1,
                     (const F*)prefix, (const F*)tot, out);
    } else {
        B2S_SMEM_ATTR(c, (msm_ba_p2_kernel<F, false>), Gm::P2_SMEM);
        B2S_LAUNCH_N(c, l2, (msm_ba_p2_kernel<F, false>), ctas, Gm::THREADS, Gm::P2_SMEM, bases, a.sorted, prev, a.bitmap, a.wrank, a.t_out,
                     a.target_units, a.unit_ctr + 1, (const F*)prefix, (const F*)tot, out);
    }
    return B2S_OK;
}

}  // namespace b2s
