// K4: variable-base multi-scalar multiplication (Pippenger, signed radix-2^c windows) for G1 and G2.
//
// GPU counterpart of ark-ec `VariableBaseMSM::msm` / `msm_bigint` (upstream crate, not in
// /root/reference; SURVEY.md Appendix A.4; callers: ark-groth16 `create_proof_with_assignment`,
// Appendix A.1).  The output is a group element, so after normalisation it is bit-identical to any
// other correct MSM regardless of window size or summation order.
//
// Pipeline (no host synchronisation inside; everything on the ctx stream except the Horner tail, which can run on
// the ctx's aux stream so that it overlaps the next MSM of a proof):
//   1 count     one thread per scalar: Montgomery -> canonical, signed digits, histogram of
//               (window, |digit|) bucket sizes (warp-aggregated global atomics, 4 B each)
//   2 scan      exclusive prefix sums (tile sums, spine, apply): bucket offsets in the sorted index array, and task offsets
//               (a bucket of s points is cut into ceil(s / L) tasks so that no thread ever owns more
//               than L points -- this is what keeps degenerate scalar distributions, e.g. the all-equal
//               witness of the reference's DummyCircuit (relations/src/sr1cs/mod.rs:306-309), balanced)
//   3 sort      the point indices (sign in bit 31) by bucket, in two passes that write whole runs instead of one entry per
//               atomic: partition (per tile of 4096 scalars and per window, a shared-memory counting sort by coarse bin
//               key >> F, one global atomic per non-empty coarse bin) and place (per coarse bin, a shared-memory counting
//               sort by fine key into the exact bucket offsets); 6 B of scratch per entry
//   3a rank     buckets are ranked by decreasing size (second counting sort) and task numbers follow the ranks, so
//               the 32 tasks a warp runs in lockstep have equal length (uniform scalars give Poisson bucket sizes)
//   3b for big problems (windows * n >= 2^27; B2S_MSM_AFFINE_ROUNDS overrides) three batched-affine halving rounds,
//               msm_affine.cuh, instead of 3a
//   4 accumulate one thread per task: XYZZ accumulator += affine base, 8M+2S per point; bases are
//               gathered from HBM (96 B / 192 B per point), everything else stays in registers
//   5 reduce    buckets that were split: CTAs sum the task partials of a bucket (two stages, shared-memory tree)
//   6 bucket sum per window sum_b b*B_b by segments: running sums over 16-32 buckets per thread, then
//               seg_start * (segment total) by double-and-add; one CTA per window adds the segments
//   7 horner    sum_w 2^(c w) S_w, one thread (255 doublings; multiplication inlined for ILP, msm_acc_g*.cu)
//
// Roofline: per (point, scalar) the algorithmic HBM traffic is 96+32 B (G1 BLS12-381), but each point
// costs ceil(255/c) mixed additions of ~10 Fq multiplications = ~3000 wide IMADs; the kernel is
// bound by the fma pipe by two orders of magnitude over HBM (DESIGN.md has the numbers).
#include <algorithm>
#include <array>
#include <cstring>

#include "msm_affine.cuh"

namespace b2s {

// ---- signed-digit recoding -------------------------------------------------------------------------
// Digits of a canonical 256-bit scalar, least significant window first.  Windows other than the
// last are recoded into [-2^(c-1), 2^(c-1)); the last keeps the carry (shape guarantees it fits B).
// v holds the scalar words around window w (bit w * c sits at bit `off` of v); carry is the recoding state between windows
__device__ __forceinline__ int32_t recode_digit(uint64_t v, uint32_t off, uint32_t& carry, uint32_t w, uint32_t c, uint32_t nwin) {
    uint32_t d = (uint32_t)((v >> off) & ((1u << c) - 1u)) + carry;
    carry = 0;
    if (w != nwin - 1 && d >= (1u << (c - 1))) {
        carry = 1;
        return (int32_t)d - (int32_t)(1u << c);
    }
    return (int32_t)d;
}

struct DigitIter {
    uint32_t k[8];
    uint32_t carry;
    __device__ __forceinline__ int32_t next(uint32_t w, uint32_t c, uint32_t nwin) {
        const uint32_t bit = w * c;
        const uint32_t word = bit >> 5, off = bit & 31;
        uint64_t v = 0;
        if (word < 8) v = k[word];
        if (word + 1 < 8) v |= (uint64_t)k[word + 1] << 32;
        return recode_digit(v, off, carry, w, c, nwin);
    }
};

template <class Fr>
__device__ __forceinline__ void load_scalar(DigitIter& it, const Fr* scalars, uint64_t i, bool mont) {
    Fr s = ld_struct(scalars + i);
    // canonical input may be any 256-bit value (the ABI does not promise < r): to_mont / from_mont leaves s mod r, so a
    // top-window digit can never index past the bucket arrays
    if (!mont) s = s.to_mont();
    s = s.from_mont();
#pragma unroll
    for (int j = 0; j < 8; j++) it.k[j] = s.v[j];
    it.carry = 0;
}

// Histogram of (window, |digit|).  Lanes of a warp that hit the same bucket are combined with
// match.any so that skewed scalar distributions (all-equal witnesses, many 0/1 values) issue one
// atomic per distinct bucket per warp instead of 32 to the same address.
// Batch: blockIdx.y is the scalar vector k (at scalars + k * stride); its windows are the super-windows k * nwin + w
// (k alone with a precomputed table) of B buckets each.
template <class Fr>
__global__ void msm_count_kernel(const Fr* __restrict__ scalars, uint64_t n, uint64_t stride, bool mont, MsmShape sh,
                                 uint32_t* __restrict__ counts) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned active = __activemask();
    const unsigned lane = threadIdx.x & 31;
    const uint32_t win0 = blockIdx.y * (sh.pre_stride ? 1u : sh.nwin);
    DigitIter it;
    load_scalar(it, scalars + blockIdx.y * stride, i, mont);
    for (uint32_t w = 0; w < sh.nwin; w++) {
        const int32_t d = it.next(w, sh.c, sh.nwin);
        const uint32_t key = d != 0 ? (sh.pre_stride ? win0 : win0 + w) * sh.B + (uint32_t)(d < 0 ? -d : d) - 1 : 0xffffffffu;
        const unsigned peers = __match_any_sync(active, key);
        if (key != 0xffffffffu && lane == (unsigned)(__ffs(peers) - 1)) atomicAdd(&counts[key], (uint32_t)__popc(peers));
    }
}

// Buckets ordered by decreasing size (counting sort on min(count, SIZE_BINS - 1)): task ranks follow this order,
// so the 32 tasks a warp executes in lockstep have (nearly) the same length.  With uniformly random scalars the
// bucket sizes are Poisson; in natural order a warp waits for its longest bucket (+37 % at a mean of 32 points).
static constexpr uint32_t SIZE_BINS = 4096;

__global__ void msm_size_hist_kernel(const uint32_t* __restrict__ counts, uint32_t G, uint32_t* __restrict__ hist) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const unsigned active = __activemask();
    const uint32_t key = SIZE_BINS - 1 - min(counts[g], SIZE_BINS - 1);
    const unsigned peers = __match_any_sync(active, key);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&hist[key], (uint32_t)__popc(peers));
}
// hist -> exclusive offsets in place in `binoff`; clears hist for reuse as the scatter cursor
__global__ void msm_size_scan_kernel(uint32_t* __restrict__ hist, uint32_t* __restrict__ binoff) {
    __shared__ uint32_t part[1024];
    const uint32_t per = SIZE_BINS / 1024;
    uint32_t local[per], sum = 0;
    for (uint32_t k = 0; k < per; k++) { local[k] = hist[threadIdx.x * per + k]; sum += local[k]; }
    part[threadIdx.x] = sum;
    __syncthreads();
    for (uint32_t d = 1; d < 1024; d <<= 1) {
        uint32_t a = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
        __syncthreads();
        part[threadIdx.x] += a;
        __syncthreads();
    }
    uint32_t run = part[threadIdx.x] - sum;
    for (uint32_t k = 0; k < per; k++) { binoff[threadIdx.x * per + k] = run; run += local[k]; hist[threadIdx.x * per + k] = 0; }
}
__global__ void msm_size_scatter_kernel(const uint32_t* __restrict__ counts, uint32_t G, const uint32_t* __restrict__ binoff,
                                        uint32_t* __restrict__ cursor, uint32_t* __restrict__ perm) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    const unsigned active = __activemask();
    const unsigned lane = threadIdx.x & 31;
    const uint32_t key = SIZE_BINS - 1 - min(counts[g], SIZE_BINS - 1);
    const unsigned peers = __match_any_sync(active, key);
    const unsigned leader = (unsigned)(__ffs(peers) - 1);
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(&cursor[key], (uint32_t)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    perm[binoff[key] + base + __popc(peers & ((1u << lane) - 1u))] = g;
}

// Exclusive scans over the G bucket counts, in three kernels (tile sums -> scan of tile sums -> apply):
//   offsets[g]  = number of points in buckets < g        (position in the sorted index array)
//   task_off[g] = number of tasks in buckets < g         (a bucket of s points has ceil(s / L) tasks)
//   heavy[1..]  = buckets that were split (more than one task), heavy[0] = how many
static constexpr int SCAN_THREADS = 256;
static constexpr int SCAN_PER_THREAD = 8;
static constexpr int SCAN_TILE = SCAN_THREADS * SCAN_PER_THREAD;

struct Scan3 { uint32_t pts, tsk, hvy; };
__device__ __forceinline__ Scan3 operator+(const Scan3& a, const Scan3& b) { return {a.pts + b.pts, a.tsk + b.tsk, a.hvy + b.hvy}; }

// inclusive block scan of one Scan3 per thread; returns the inclusive prefix, total in *total
__device__ __forceinline__ Scan3 block_scan(Scan3 v, Scan3* total) {
    __shared__ Scan3 warp_tot[32];
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        Scan3 o = {__shfl_up_sync(0xffffffffu, v.pts, d), __shfl_up_sync(0xffffffffu, v.tsk, d), __shfl_up_sync(0xffffffffu, v.hvy, d)};
        if (lane >= (unsigned)d) v = v + o;
    }
    if (lane == 31) warp_tot[wid] = v;
    __syncthreads();
    const unsigned nw = (blockDim.x + 31) >> 5;
    if (wid == 0) {
        Scan3 w = lane < nw ? warp_tot[lane] : Scan3{0, 0, 0};
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            Scan3 o = {__shfl_up_sync(0xffffffffu, w.pts, d), __shfl_up_sync(0xffffffffu, w.tsk, d), __shfl_up_sync(0xffffffffu, w.hvy, d)};
            if (lane >= (unsigned)d) w = w + o;
        }
        warp_tot[lane] = w;
    }
    __syncthreads();
    if (wid > 0) v = v + warp_tot[wid - 1];
    *total = warp_tot[nw - 1];
    __syncthreads();
    return v;
}

__global__ void __launch_bounds__(SCAN_THREADS)
msm_scan_tiles_kernel(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ perm, MsmShape sh,
                      Scan3* __restrict__ tile_sums) {
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER_THREAD;
    Scan3 v{0, 0, 0};
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) {
        const uint32_t g = base + k;
        if (g < sh.G) {
            const uint32_t s = counts[perm ? perm[g] : g], t = (s + sh.L - 1) / sh.L;
            v = v + Scan3{s, t, t > 1 ? 1u : 0u};
        }
    }
    Scan3 total;
    block_scan(v, &total);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}

// one CTA: exclusive scan of the tile sums in place; totals to offsets[G], task_off[G], heavy[0]
__global__ void __launch_bounds__(1024)
msm_scan_spine_kernel(Scan3* __restrict__ tile_sums, uint32_t ntiles, MsmShape sh, uint32_t* __restrict__ offsets,
                      uint32_t* __restrict__ task_off, uint32_t* __restrict__ heavy) {
    const uint32_t per = (ntiles + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(threadIdx.x * per, ntiles), hi = min(lo + per, ntiles);
    Scan3 v{0, 0, 0};
    for (uint32_t i = lo; i < hi; i++) v = v + tile_sums[i];
    Scan3 total;
    Scan3 incl = block_scan(v, &total);
    Scan3 run = {incl.pts - v.pts, incl.tsk - v.tsk, incl.hvy - v.hvy};
    for (uint32_t i = lo; i < hi; i++) {
        Scan3 t = tile_sums[i];
        tile_sums[i] = run;
        run = run + t;
    }
    if (threadIdx.x == 0) {
        if (offsets) offsets[sh.G] = total.pts;
        task_off[sh.G] = total.tsk;
        heavy[0] = total.hvy;
    }
}

__global__ void __launch_bounds__(SCAN_THREADS)
msm_scan_apply_kernel(const uint32_t* __restrict__ counts, const uint32_t* __restrict__ perm, MsmShape sh,
                      const Scan3* __restrict__ tile_sums,
                      uint32_t* __restrict__ offsets, uint32_t* __restrict__ task_off, uint32_t* __restrict__ heavy) {
    const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_PER_THREAD;
    uint32_t s[SCAN_PER_THREAD], t[SCAN_PER_THREAD];
    Scan3 v{0, 0, 0};
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) {
        const uint32_t g = base + k;
        s[k] = g < sh.G ? counts[perm ? perm[g] : g] : 0u;
        t[k] = (s[k] + sh.L - 1) / sh.L;
        v = v + Scan3{s[k], t[k], t[k] > 1 ? 1u : 0u};
    }
    Scan3 total;
    Scan3 incl = block_scan(v, &total);
    const Scan3 tb = tile_sums[blockIdx.x];
    Scan3 run = {tb.pts + incl.pts - v.pts, tb.tsk + incl.tsk - v.tsk, tb.hvy + incl.hvy - v.hvy};
#pragma unroll
    for (int k = 0; k < SCAN_PER_THREAD; k++) {
        const uint32_t g = base + k;
        if (g < sh.G) {
            if (offsets) offsets[g] = run.pts;
            task_off[g] = run.tsk;
            if (t[k] > 1) heavy[1 + run.hvy] = g;
            run = run + Scan3{s[k], t[k], t[k] > 1 ? 1u : 0u};
        }
    }
}

// ---- sort of the digits by bucket, in two passes ----------------------------------------------------------------------
// The entries of bucket g go to sorted[offsets[g] .. offsets[g+1]).  Scattering them one by one costs a returning global
// atomic and a lone 4 B store per entry (uniform scalars almost never share a bucket within a warp).  Instead:
//   partition  per CTA of SORT_TILE scalars and per window, a counting sort in shared memory by coarse bin (key >> F);
//              one global atomic per non-empty (CTA, coarse bin) reserves a run inside the bin's region, which starts at
//              offsets[bin << F] because offsets are exact.  Runs leave as u32 entries plus the u16 fine key key & (2^F - 1).
//   place      per coarse bin, chunks of SORT_CHUNK entries are counting-sorted by fine key in shared memory and written
//              to offsets[key] + (shared-memory cursor).  A bin above SORT_SPLIT entries (skewed scalars: a window whose
//              digits all agree) is cut into parts for the split CTAs, which reserve per (part, fine bucket) on cursor[key].
// F is chosen so that uniform scalars give ~16 entries per (CTA, window, coarse bin): 64 B runs instead of 4 B stores.
static constexpr uint32_t SORT_THREADS = 1024;
static constexpr uint32_t SORT_TILE = 4096;           // scalars per partition CTA
static constexpr uint32_t SORT_PER = SORT_TILE / SORT_THREADS;
static constexpr uint32_t SORT_CHUNK = 16384;         // entries per place chunk
static constexpr uint32_t SORT_CHUNK_PER = SORT_CHUNK / SORT_THREADS;
static constexpr uint32_t SORT_SPLIT = 8 * SORT_CHUNK;
static constexpr uint32_t SORT_MAX_F = 11;            // fine keys fit in u16, fine-bucket arrays of one place CTA in 24 KiB

// coarse bins per window = SORT_TILE / 16 = 256 where the window has that many buckets, with at most 2^SORT_MAX_F buckets each
static uint32_t sort_fine_bits(uint32_t c) { return std::min<uint32_t>(SORT_MAX_F, c > 9 ? c - 9 : 0); }
static size_t partition_smem(uint32_t nbw) { return ((size_t)10 * SORT_TILE + 3 * (size_t)nbw + 1) * sizeof(uint32_t); }
static size_t place_smem(uint32_t F) {
    return (size_t)SORT_CHUNK * (sizeof(uint32_t) + sizeof(uint16_t)) + ((size_t)3 * (1u << F) + 1 + SORT_THREADS + 1) * sizeof(uint32_t);
}

// in[0..n) -> out[0..n]: exclusive prefix sums, out[n] = total.  Called by every thread of the CTA; ends with a barrier.
__device__ void block_excl_scan(const uint32_t* in, uint32_t* out, uint32_t n) {
    __shared__ uint32_t wsum[32];
    const uint32_t per = (n + blockDim.x - 1) / blockDim.x;
    const uint32_t lo = min(threadIdx.x * per, n), hi = min(lo + per, n);
    uint32_t s = 0;
    for (uint32_t i = lo; i < hi; i++) s += in[i];
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t incl = s;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= (unsigned)d) incl += o;
    }
    if (lane == 31) wsum[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint32_t w = lane < (blockDim.x >> 5) ? wsum[lane] : 0u;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t o = __shfl_up_sync(0xffffffffu, w, d);
            if (lane >= (unsigned)d) w += o;
        }
        wsum[lane] = w;
    }
    __syncthreads();
    uint32_t run = incl - s + (wid ? wsum[wid - 1] : 0u);
    for (uint32_t i = lo; i < hi; i++) { out[i] = run; run += in[i]; }
    if (threadIdx.x == 0) out[n] = wsum[31];
    __syncthreads();
}

// Pass 1.  Scalars are kept canonical in shared memory, word-major, so that each window reads its two words without bank
// conflicts and the recoding carry walks the windows in order.  Batch: blockIdx.y is the scalar vector k, as in the count
// kernel; a tile never straddles two vectors, and its entries keep the base index because the vectors share the bases.
template <class Fr>
__global__ void __launch_bounds__(SORT_THREADS, 1)
msm_partition_kernel(const Fr* __restrict__ scalars, const uint32_t* __restrict__ index_map, uint64_t n, uint64_t stride, bool mont, MsmShape sh,
                     uint32_t F, const uint32_t* __restrict__ offsets, uint32_t* __restrict__ bin_cursor, uint32_t* __restrict__ part_val,
                     uint16_t* __restrict__ part_fine) {
    extern __shared__ uint4 sort_smem[];
    const uint32_t nbw = sh.B >> F;                          // coarse bins per window
    uint32_t* sc = reinterpret_cast<uint32_t*>(sort_smem);   // [8][SORT_TILE] scalar words
    uint32_t* sv = sc + 8 * SORT_TILE;                       // staged entries of one window, ordered by coarse bin
    uint32_t* sk = sv + SORT_TILE;                           // their window-local bucket |digit| - 1
    uint32_t* hist = sk + SORT_TILE;                         // [nbw]
    uint32_t* start = hist + nbw;                            // [nbw + 1]
    uint32_t* dest = start + nbw + 1;                        // [nbw] staged entry i of bin b goes to dest[b] + i
    const uint64_t tile = (uint64_t)blockIdx.x * SORT_TILE;
    const uint32_t cnt = (uint32_t)min((uint64_t)SORT_TILE, n - tile);
    uint32_t base[SORT_PER];
#pragma unroll
    for (uint32_t j = 0; j < SORT_PER; j++) {
        const uint32_t s = threadIdx.x + j * SORT_THREADS;
        if (s < cnt) {
            DigitIter it;
            load_scalar(it, scalars + blockIdx.y * stride, tile + s, mont);
#pragma unroll
            for (int q = 0; q < 8; q++) sc[q * SORT_TILE + s] = it.k[q];
            base[j] = index_map ? index_map[tile + s] : (uint32_t)(tile + s);
        }
    }
    for (uint32_t b = threadIdx.x; b < nbw; b += SORT_THREADS) hist[b] = 0;
    uint32_t carry = 0;                                      // bit j: recoding carry of scalar j
    __syncthreads();
    for (uint32_t w = 0; w < sh.nwin; w++) {
        const uint32_t bit = w * sh.c, word = bit >> 5, off = bit & 31;
        uint32_t ent[SORT_PER], rank[SORT_PER];              // ent: bucket | sign << 31, or ~0u for a zero digit
#pragma unroll
        for (uint32_t j = 0; j < SORT_PER; j++) {
            const uint32_t s = threadIdx.x + j * SORT_THREADS;
            ent[j] = ~0u;
            if (s < cnt) {
                uint64_t v = 0;
                if (word < 8) v = sc[word * SORT_TILE + s];
                if (word + 1 < 8) v |= (uint64_t)sc[(word + 1) * SORT_TILE + s] << 32;
                uint32_t cy = (carry >> j) & 1u;
                const int32_t d = recode_digit(v, off, cy, w, sh.c, sh.nwin);
                carry = (carry & ~(1u << j)) | (cy << j);
                if (d != 0) {
                    const uint32_t lk = (uint32_t)(d < 0 ? -d : d) - 1;
                    ent[j] = lk | (d < 0 ? 0x80000000u : 0u);
                    rank[j] = atomicAdd(&hist[lk >> F], 1u);
                }
            }
        }
        __syncthreads();
        block_excl_scan(hist, start, nbw);
        const uint32_t bin0 = (sh.pre_stride ? blockIdx.y : blockIdx.y * sh.nwin + w) * nbw;
        for (uint32_t b = threadIdx.x; b < nbw; b += SORT_THREADS) {
            const uint32_t k = hist[b];
            if (k) dest[b] = offsets[(bin0 + b) << F] + atomicAdd(&bin_cursor[bin0 + b], k) - start[b];
            hist[b] = 0;
        }
#pragma unroll
        for (uint32_t j = 0; j < SORT_PER; j++) {
            if (ent[j] != ~0u) {
                const uint32_t lk = ent[j] & 0x7fffffffu;
                const uint32_t p = start[lk >> F] + rank[j];
                sv[p] = (base[j] + w * sh.pre_stride) | (ent[j] & 0x80000000u);
                sk[p] = lk;
            }
        }
        __syncthreads();
        const uint32_t total = start[nbw];
        for (uint32_t i = threadIdx.x; i < total; i += SORT_THREADS) {
            const uint32_t lk = sk[i];
            const uint32_t o = dest[lk >> F] + i;
            part_val[o] = sv[i];
            part_fine[o] = (uint16_t)(lk & ((1u << F) - 1u));
        }
        __syncthreads();
    }
}

// One chunk of a coarse bin: entries [c0, c0 + len) sorted by fine key; cur[f] is where the next entry of fine bucket f goes
// and is advanced past this chunk's entries.
__device__ __forceinline__ void place_chunk(uint32_t c0, uint32_t len, uint32_t nf, const uint32_t* __restrict__ part_val,
                                            const uint16_t* __restrict__ part_fine, uint32_t* __restrict__ sorted, uint32_t* sv, uint16_t* sf,
                                            uint32_t* hist, uint32_t* start, uint32_t* cur) {
    uint32_t fr[SORT_CHUNK_PER];                             // fine key | rank << 16, or ~0u past the end
#pragma unroll
    for (uint32_t j = 0; j < SORT_CHUNK_PER; j++) {
        const uint32_t i = threadIdx.x + j * SORT_THREADS;
        fr[j] = ~0u;
        if (i < len) {
            const uint32_t f = part_fine[c0 + i];
            fr[j] = f | atomicAdd(&hist[f], 1u) << 16;
        }
    }
    __syncthreads();
    block_excl_scan(hist, start, nf);
#pragma unroll
    for (uint32_t j = 0; j < SORT_CHUNK_PER; j++) {
        if (fr[j] != ~0u) {
            const uint32_t f = fr[j] & 0xffffu;
            const uint32_t p = start[f] + (fr[j] >> 16);
            sv[p] = part_val[c0 + threadIdx.x + j * SORT_THREADS];
            sf[p] = (uint16_t)f;
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < len; i += SORT_THREADS) {
        const uint32_t f = sf[i];
        sorted[cur[f] + i - start[f]] = sv[i];
    }
    __syncthreads();
    for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) {
        cur[f] += hist[f];
        hist[f] = 0;
    }
    __syncthreads();
}

// Pass 2.  CTA b < nbins places coarse bin b when it holds at most SORT_SPLIT entries, with its cursors in shared memory.
// The CTAs after them share the larger bins, in parts of SORT_SPLIT entries dealt round-robin: a part counts its fine keys
// first and reserves one run per non-empty fine bucket with an atomic on cursor[key] (zeroed by the caller).
__global__ void __launch_bounds__(SORT_THREADS, 1)
msm_place_kernel(const uint32_t* __restrict__ offsets, uint32_t nbins, uint32_t F, const uint32_t* __restrict__ part_val,
                 const uint16_t* __restrict__ part_fine, uint32_t* __restrict__ cursor, uint32_t* __restrict__ sorted) {
    extern __shared__ uint4 sort_smem[];
    const uint32_t nf = 1u << F;
    uint32_t* sv = reinterpret_cast<uint32_t*>(sort_smem);  // [SORT_CHUNK]
    uint16_t* sf = reinterpret_cast<uint16_t*>(sv + SORT_CHUNK);
    uint32_t* hist = reinterpret_cast<uint32_t*>(sf + SORT_CHUNK);   // [nf]
    uint32_t* start = hist + nf;                             // [nf + 1]
    uint32_t* cur = start + nf + 1;                          // [nf]
    uint32_t* big = cur + nf;                                // [SORT_THREADS] bins to split, then their number
    uint32_t* nbig = big + SORT_THREADS;
    for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) hist[f] = 0;
    if (blockIdx.x < nbins) {
        const uint32_t k0 = blockIdx.x << F;
        const uint32_t lo = offsets[k0], hi = offsets[k0 + nf];
        if (hi == lo || hi - lo > SORT_SPLIT) return;
        for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) cur[f] = offsets[k0 + f];
        __syncthreads();
        for (uint32_t c0 = lo; c0 < hi; c0 += SORT_CHUNK) place_chunk(c0, min(SORT_CHUNK, hi - c0), nf, part_val, part_fine, sorted, sv, sf, hist, start, cur);
        return;
    }
    const uint32_t s = blockIdx.x - nbins, S = gridDim.x - nbins;
    for (uint32_t b0 = 0; b0 < nbins; b0 += SORT_THREADS) {
        const uint32_t b = b0 + threadIdx.x;
        const bool is_big = b < nbins && offsets[(b + 1) << F] - offsets[b << F] > SORT_SPLIT;
        if (threadIdx.x == 0) *nbig = 0;
        if (!__syncthreads_or(is_big)) continue;
        if (is_big) big[atomicAdd(nbig, 1u)] = b;
        __syncthreads();
        const uint32_t m = *nbig;
        for (uint32_t q = 0; q < m; q++) {
            const uint32_t bb = big[q], k0 = bb << F;
            const uint32_t lo = offsets[k0], hi = offsets[k0 + nf];
            const uint32_t parts = (hi - lo + SORT_SPLIT - 1) / SORT_SPLIT;
            for (uint32_t p = (s + S - bb % S) % S; p < parts; p += S) {
                const uint32_t p0 = lo + p * SORT_SPLIT, p1 = min(hi, p0 + SORT_SPLIT);
                for (uint32_t i = p0 + threadIdx.x; i < p1; i += SORT_THREADS) atomicAdd(&hist[part_fine[i]], 1u);
                __syncthreads();
                for (uint32_t f = threadIdx.x; f < nf; f += SORT_THREADS) {
                    const uint32_t k = hist[f];
                    if (k) cur[f] = offsets[k0 + f] + atomicAdd(&cursor[k0 + f], k);
                    hist[f] = 0;
                }
                __syncthreads();
                for (uint32_t c0 = p0; c0 < p1; c0 += SORT_CHUNK) place_chunk(c0, min(SORT_CHUNK, p1 - c0), nf, part_val, part_fine, sorted, sv, sf, hist, start, cur);
            }
        }
        __syncthreads();
    }
}

// Buckets that were split into tasks: sum their task partials.  Big ones (>= `big` partials, e.g. the
// one-bucket-per-window case of an all-equal witness) first get `split` CTAs each, which leave their slice sums in tmp;
// then one CTA per bucket finishes.  Slot of (heavy bucket h, slice j):
//   many buckets (the Pippenger bucket array): tmp[t0 / split + j], t0 = first task of the bucket; slots of different big
//     buckets cannot overlap because each owns >= big = split^2 consecutive tasks (split = 16);
//   few buckets (the <= 8 heavy lists of the multiplicity-aware front end): tmp[h * split + j] with split = 256, so that one
//     list's hundreds of thousands of partials are summed by 256 CTAs instead of 16.
struct HeavyPlan { uint32_t split, big, by_ordinal; };
static HeavyPlan heavy_plan(uint32_t G) { return G <= 64 ? HeavyPlan{256u, 512u, 1u} : HeavyPlan{16u, 256u, 0u}; }
static size_t heavy_tmp_slots(const HeavyPlan& hp, uint32_t G, uint64_t max_tasks) {
    return hp.by_ordinal ? (size_t)G * hp.split + 1 : (size_t)(max_tasks / hp.split) + hp.split + 1;
}

template <class F>
__global__ void __launch_bounds__(MSM_RED_THREADS)
msm_reduce_heavy_stage1_kernel(const uint32_t* __restrict__ heavy, const uint32_t* __restrict__ task_off, HeavyPlan hp,
                               const XYZZ<F>* __restrict__ partials, XYZZ<F>* __restrict__ tmp) {   // heavy[] holds ranks
    extern __shared__ uint4 smem_raw[];
    XYZZ<F>* smem = reinterpret_cast<XYZZ<F>*>(smem_raw);
    const uint32_t nitems = heavy[0] * hp.split;
    for (uint32_t it = blockIdx.x; it < nitems; it += gridDim.x) {
        const uint32_t h = it / hp.split, j = it % hp.split;
        const uint32_t g = heavy[1 + h];
        const uint32_t t0 = task_off[g], cnt = task_off[g + 1] - t0;
        if (cnt < hp.big) continue;
        const uint32_t lo = (uint32_t)((uint64_t)cnt * j / hp.split), hi = (uint32_t)((uint64_t)cnt * (j + 1) / hp.split);
        XYZZ<F> s = cta_sum(partials + t0 + lo, hi - lo, smem);
        if (threadIdx.x == 0) st_struct(tmp + (hp.by_ordinal ? h * hp.split : t0 / hp.split) + j, s);
        __syncthreads();
    }
}

template <class F>
__global__ void __launch_bounds__(MSM_RED_THREADS)
msm_reduce_heavy_kernel(const uint32_t* __restrict__ heavy, const uint32_t* __restrict__ task_off, const uint32_t* __restrict__ perm, HeavyPlan hp,
                        const XYZZ<F>* __restrict__ partials, const XYZZ<F>* __restrict__ tmp, XYZZ<F>* __restrict__ bucket_acc) {
    extern __shared__ uint4 smem_raw[];
    XYZZ<F>* smem = reinterpret_cast<XYZZ<F>*>(smem_raw);
    const uint32_t nheavy = heavy[0];
    for (uint32_t h = blockIdx.x; h < nheavy; h += gridDim.x) {
        const uint32_t rk = heavy[1 + h];
        const uint32_t g = perm ? perm[rk] : rk;
        const uint32_t t0 = task_off[rk], cnt = task_off[rk + 1] - t0;
        XYZZ<F> s = cnt < hp.big ? cta_sum(partials + t0, cnt, smem) : cta_sum(tmp + (hp.by_ordinal ? h * hp.split : t0 / hp.split), hp.split, smem);
        if (threadIdx.x == 0) st_struct(bucket_acc + g, s);
        __syncthreads();
    }
}

// sum of `count` XYZZ points -> affine (join of multi-GPU shard partials; final normalisation)
template <class F>
__global__ void __launch_bounds__(MSM_RED_THREADS)
group_sum_affine_kernel(const XYZZ<F>* __restrict__ pts, uint32_t count, Affine<F>* __restrict__ out) {
    extern __shared__ uint4 smem_raw[];
    XYZZ<F>* smem = reinterpret_cast<XYZZ<F>*>(smem_raw);
    XYZZ<F> s = cta_sum(pts, count, smem);
    if (threadIdx.x == 0) {
        Affine<F> a = s.to_affine();
        st_struct(out, a);
    }
}

// G2 bucket reduction stays in this unit (out-of-line multiplication): inlining 42 base multiplications per general
// addition into its kernels costs a quarter of an hour of ptxas for a ~5 % kernel
int32_t msm_bucket_reduce_g2(Ctx* c, const void* bucket_acc, MsmShape sh, uint32_t seg, void* segs, uint32_t segs_per_win, void* wins) {
    return dispatch_curve(c, [&](auto curve) {
        using F = typename decltype(curve)::Fq2;
        return msm_bucket_reduce_launch<F>(c, "msm_bucket_segments_g2", "msm_window_sum_g2", bucket_acc, sh, seg, segs, segs_per_win, wins);
    });
}

// ---------------------------------------------------------------------------------------------------
static uint32_t env_u32(const char* name, uint32_t dflt) {
    const char* v = getenv(name);
    return v ? (uint32_t)strtoul(v, nullptr, 10) : dflt;
}

uint64_t pool_idle_bytes(Ctx* c) {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, c->device) != cudaSuccess) return 0;
    uint64_t reserved = 0, used = 0;
    cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved);
    cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used);
    return reserved > used ? reserved - used : 0;
}

// Window size: minimise  n * nwin  (bucket accumulation, mixed additions)  +  nwin * 2^(c-1) * 4.7
// (bucket reduction: two general additions per bucket at ~1.4x the cost of a mixed one, plus the
// per-segment double-and-add), subject to the bucket array staying under 4 GiB.  A batch of K scalar vectors keeps the
// window size of one (the cost per vector is the same) and has K times the buckets and entries.
static MsmShape msm_shape(uint64_t n, uint32_t scalar_bits, size_t point_bytes, const MsmPre* pre = nullptr, uint32_t K = 1) {
    MsmShape sh{};
    if (pre) {      // the table fixes c; all windows share one bucket set
        sh.c = pre->c; sh.nwin = pre->nwin; sh.B = 1u << (pre->c - 1); sh.G = K * sh.B; sh.pre_stride = pre->stride;
        const uint64_t t_upper = (uint64_t)K * sh.nwin * n;
        sh.L = (uint32_t)std::max<uint64_t>(64, t_upper >> 18);
        sh.max_tasks = t_upper / sh.L + sh.G + 1;
        return sh;
    }
    auto nwin_of = [&](uint32_t c) {
        uint32_t nw = (scalar_bits + c - 1) / c;
        // the last window keeps the recoding carry: it must fit in 2^(c-1) buckets
        if (scalar_bits - (nw - 1) * c >= c) nw += 1;
        return nw;
    };
    uint32_t best_c = 5;
    double best = 1e300;
    for (uint32_t c = 5; c <= 20; c++) {
        const uint32_t nw = nwin_of(c);
        const double buckets = (double)nw * (double)(1u << (c - 1));
        if (buckets * (double)point_bytes > 4.0 * 1024 * 1024 * 1024) break;
        const double cost = (double)n * nw + buckets * 4.7;
        if (cost < best) { best = cost; best_c = c; }
    }
    uint32_t c = env_u32("B2S_MSM_C", best_c);
    if (c < 2) c = 2;
    if (c > 24) c = 24;
    sh.c = c;
    sh.nwin = nwin_of(c);
    sh.B = 1u << (c - 1);
    sh.G = K * sh.nwin * sh.B;
    const uint64_t t_upper = (uint64_t)K * sh.nwin * n;
    uint64_t L = t_upper >> 18;
    if (L < 64) L = 64;
    L = env_u32("B2S_MSM_L", (uint32_t)L);
    sh.L = (uint32_t)L;
    sh.max_tasks = t_upper / sh.L + sh.G + 1;
    return sh;
}

// ---- bucket sums of an arbitrary bucket structure ---------------------------------------------------------------
// How many batched-affine rounds pay for T entries in G buckets, in how many slices of the bucket range they run, and the
// XYZZ task length after them.  slice_entries: the most entries one slice may hold (T when the rounds run in one piece).
struct RoundPlan { uint32_t rounds, L; uint64_t max_tasks; uint64_t slice_entries; uint32_t L_plain; };

// device bytes that the rounds and the XYZZ partials of T entries in G buckets hold at once: the two output buffers, the
// prefix products and the lane totals (bounded by the first round), and one partial per bucket and per task (plan_tasks
// cuts what is left after the rounds into tasks of at least 16 entries, and at most about 2^18 of them)
static uint64_t round_scratch_bytes(uint64_t T, uint64_t G, size_t aff, size_t xyzz) {
    const uint64_t t0 = std::min<uint64_t>(T, (T + G) / 2 + 1);
    return t0 * (aff * 3 / 2 + aff / 2) + t0 / 4 + (G + std::min<uint64_t>(t0 / 16 + 1, 1u << 18)) * xyzz;
}

// task length and task bound of the XYZZ kernel for T entries in G buckets after rp.rounds rounds
static void plan_tasks(RoundPlan& rp, uint64_t T, uint32_t G) {
    rp.L = rp.L_plain;
    rp.max_tasks = T / rp.L + G + 1;
    if (rp.rounds && !getenv("B2S_MSM_L")) {
        // what the XYZZ kernel sees after the rounds is 2^-R of the input: cut its tasks accordingly, otherwise the heavy
        // buckets of skewed scalars (a few thousand tasks of ~1000 points) leave most of the machine idle
        uint64_t t_after = T;
        for (uint32_t r = 0; r < rp.rounds; r++) t_after = std::min<uint64_t>(t_after, (t_after + G) / 2 + 1);
        rp.L = (uint32_t)std::max<uint64_t>(16, t_after >> 18);
        rp.max_tasks = t_after / rp.L + G + 1;
    }
}

// held: bytes the caller allocates after this call and keeps while the rounds run (sorted indices, bucket sums)
template <class F>
static RoundPlan plan_rounds(Ctx* c, uint64_t T, uint32_t G, bool is_g1, uint32_t L_default, uint64_t held = 0) {
    RoundPlan rp{0, L_default, 0, T, L_default};
    uint32_t ba_auto = 0;
    const uint64_t per_bucket = G ? T / G : 0;
    while ((1ull << ba_auto) < per_bucket) ba_auto++;
    // a round has a fixed price -- one latency-bound inversion level plus a dozen small launches -- and
    // saves 4 (G1) / 11 (G2) base multiplications on each of its T / 2^(r+1) additions: keep the rounds that pay.  Sliced
    // rounds pay the fixed price once per slice, so a slice of t entries keeps the rounds that pay for t.  With Fermat
    // inversions the level alone took 0.72 ms (G1), ~0.8-0.9 ms with the small launches (halve, singles, 3 scan and 3 rank
    // kernels, memset: ~0.08 ms), which at 2.6e10 Fq products/s is 6e6 G1 (2.5e6 G2) additions' saving.  Divsteps
    // inversions and BA_K2 = 16 bring the G1 level to <= 0.19 ms (2.70 ms over the >= 14 levels of a 2^24 proof on an H100),
    // so ~0.27 ms a round with the launches, ~1.7e6 additions' saving; G2 (three Fq products per Fq2 product in the chain)
    // is priced at ~0.3 ms.  1.5e6 / 0.75e6 give a 2^24 heavy list 3 (G1) / 4 (G2) rounds run in one piece, DESIGN.md 3.1 and 4.
    const double min_adds = is_g1 ? 1.5e6 : 0.75e6;
    auto pays = [&](uint64_t t) {
        uint32_t p = 0;
        while (p < 16 && (double)(t >> (p + 1)) > min_adds) p++;
        return std::min(ba_auto, p);
    };
    const bool forced = getenv("B2S_MSM_AFFINE_ROUNDS") != nullptr;
    rp.rounds = forced ? env_u32("B2S_MSM_AFFINE_ROUNDS", 0) : pays(T);
    // B2S_MSM_ROUND_BUDGET (bytes) replaces the free-memory budget, so that small problems can be made to slice
    const char* budget_env = getenv("B2S_MSM_ROUND_BUDGET");
    if (rp.rounds && (budget_env || !forced)) {
        const uint64_t need = round_scratch_bytes(T, G, sizeof(Affine<F>), sizeof(XYZZ<F>));
        uint64_t budget = 0;
        if (budget_env) {
            budget = strtoull(budget_env, nullptr, 10);
        } else {
            // free-memory queries only when the scratch is a large part of the device (they cost milliseconds of host time with
            // a multi-GiB pool, and this runs once per MSM): anything under a third of the device is simply allocated
            size_t free_b = (size_t)c->total_mem, total_b = 0;
            uint64_t pool_held = 0;
            if ((need + held) * 3 > c->total_mem) {
                cudaMemGetInfo(&free_b, &total_b);
                pool_held = pool_idle_bytes(c);
            }
            const uint64_t avail = (uint64_t)free_b + pool_held, reserve = held + ((uint64_t)2 << 30);
            budget = avail > reserve ? avail - reserve : 0;
        }
        if (need > budget) {
            // slices of the bucket range: the scratch grows with the entries, and the buckets of a slice in proportion
            rp.slice_entries = (uint64_t)((double)T * ((double)budget / (double)need));
            if (!forced && rp.slice_entries) rp.rounds = pays(T / ((T + rp.slice_entries - 1) / rp.slice_entries));
            // a slice holds whole buckets: one that cannot hold the average bucket twice over is no slice
            if (rp.slice_entries < 2 * std::max<uint64_t>(per_bucket, 1)) rp.rounds = 0;
            if (!rp.rounds) rp.slice_entries = T;
        }
    }
    plan_tasks(rp, T, G);
    return rp;
}

// One slice of bucket_sums_t (or all of it): G buckets holding T entries, sorted / counts / offsets / bucket_acc already
// advanced to the slice's first bucket.  Without rounds the caller's offsets are rewritten from its counts (same values).
template <class Curve, class F>
static int32_t bucket_slice_t(Ctx* c, const Affine<F>* bases, const uint32_t* sorted, uint32_t* counts, uint32_t* offsets, uint64_t T, uint32_t G,
                              const RoundPlan& rp, XYZZ<F>* bucket_acc) {
    using Pt = XYZZ<F>;
    constexpr bool is_g1 = sizeof(F) == sizeof(typename Curve::Fq);
    MsmShape sh{};
    sh.G = G; sh.L = rp.L; sh.max_tasks = rp.max_tasks;
    const uint32_t ntiles = (G + SCAN_TILE - 1) / SCAN_TILE;
    const uint32_t* no_perm = nullptr;
    DevBuf tiles, tbuf, partials, heavy_tmp;
    B2S_TRY(tiles.alloc(c, (size_t)ntiles * sizeof(Scan3)));
    B2S_TRY(tbuf.alloc(c, ((size_t)2 * G + 3) * sizeof(uint32_t)));       // task_off[G+1] heavy[G+1]
    uint32_t* task_off = tbuf.as<uint32_t>();
    uint32_t* heavy = task_off + G + 1;
    B2S_TRY(partials.alloc(c, (size_t)sh.max_tasks * sizeof(Pt)));
    const HeavyPlan hp = heavy_plan(G);
    B2S_TRY(heavy_tmp.alloc(c, heavy_tmp_slots(hp, G, sh.max_tasks) * sizeof(Pt)));
    const void* acc_bases = bases;
    const uint32_t* acc_sorted = sorted;
    const uint32_t* acc_offsets = offsets;
    const uint32_t* acc_counts = counts;
    DevBuf ba_ints, ba_out[2], ba_prefix, ba_tot, ba_bits;
    if (rp.rounds) {
        // two internal (counts, offsets) pairs: the caller's arrays are only READ (round 0), so a bucket structure can be
        // shared by several calls (the heavy lists of a, b_g1, b_g2 of one proof)
        B2S_TRY(ba_ints.alloc(c, ((size_t)4 * G + 2) * sizeof(uint32_t)));
        uint32_t* pp_cnt[2] = {ba_ints.as<uint32_t>(), ba_ints.as<uint32_t>() + 2 * G + 1};
        uint32_t* pp_off[2] = {pp_cnt[0] + G, pp_cnt[1] + G};
        const uint32_t* cnt_in = counts;
        uint64_t t_in = T;
        // outputs of a round: every bucket keeps ceil(count / 2) points -- at most (t_in + G) / 2 and never more than t_in
        auto round_bound = [&](uint64_t tin) { return std::min<uint64_t>(tin, (tin + G) / 2 + 1); };
        const uint64_t out_bound0 = round_bound(t_in);
        const uint64_t words_bound0 = out_bound0 / 32 + 2;
        const uint64_t tot_bound = (words_bound0 / BA_KMIN + 2) * 32;
        const uint32_t rank_tiles0 = cdiv(words_bound0, BA_SCAN_TILE);
        // bitmap | wrank | rank tile sums
        B2S_TRY(ba_bits.alloc(c, (2 * words_bound0 + rank_tiles0 + 1) * sizeof(uint32_t)));
        uint32_t* bitmap = ba_bits.as<uint32_t>();
        uint32_t* wrank = bitmap + words_bound0;
        uint32_t* rtiles = wrank + words_bound0;
        B2S_TRY(ba_prefix.alloc(c, out_bound0 * sizeof(F)));
        B2S_TRY(ba_tot.alloc(c, 2 * tot_bound * sizeof(F)));
        const uint32_t target_units = 4u * 16u * (uint32_t)c->sm_count;   // ~4 units per resident warp, handed out dynamically
        DevBuf ba_ctr;
        B2S_TRY(ba_ctr.alloc(c, (size_t)2 * rp.rounds * sizeof(uint32_t)));
        B2S_CUDA(c, cudaMemsetAsync(ba_ctr.p, 0, (size_t)2 * rp.rounds * sizeof(uint32_t), c->stream));
        // the two ping-pong output buffers, sized for the rounds that use them (even rounds write [1], odd rounds [0])
        B2S_TRY(ba_out[1].alloc(c, out_bound0 * sizeof(Affine<F>)));
        if (rp.rounds > 1) B2S_TRY(ba_out[0].alloc(c, round_bound(out_bound0) * sizeof(Affine<F>)));
        const void* prev = nullptr;
        for (uint32_t r = 0; r < rp.rounds; r++) {
            const int nxt = (int)(r & 1u);
            uint32_t* cnt_out = pp_cnt[nxt];
            uint32_t* off_out = pp_off[nxt];
            const uint64_t out_bound = round_bound(t_in);
            const uint32_t n_words = (uint32_t)(out_bound / 32 + 2);
            const uint32_t rank_tiles = cdiv(n_words, BA_SCAN_TILE);
            B2S_LAUNCH(c, msm_ba_halve_kernel, cdiv(G, 256), 256, 0, cnt_in, G, cnt_out);
            B2S_LAUNCH(c, msm_scan_tiles_kernel, ntiles, SCAN_THREADS, 0, (const uint32_t*)cnt_out, no_perm, sh, tiles.as<Scan3>());
            B2S_LAUNCH(c, msm_scan_spine_kernel, 1, 1024, 0, tiles.as<Scan3>(), ntiles, sh, off_out, task_off, heavy);
            B2S_LAUNCH(c, msm_scan_apply_kernel, ntiles, SCAN_THREADS, 0, (const uint32_t*)cnt_out, no_perm, sh, tiles.as<Scan3>(), off_out, task_off, heavy);
            B2S_CUDA(c, cudaMemsetAsync(bitmap, 0, (size_t)n_words * sizeof(uint32_t), c->stream));
            B2S_LAUNCH(c, msm_ba_singles_kernel, cdiv(G, 256), 256, 0, cnt_in, (const uint32_t*)off_out, G, bitmap);
            B2S_LAUNCH(c, msm_ba_rank_tiles_kernel, rank_tiles, BA_SCAN_THREADS, 0, bitmap, n_words, rtiles);
            B2S_LAUNCH(c, msm_ba_rank_spine_kernel, 1, 1024, 0, rtiles, rank_tiles);
            B2S_LAUNCH(c, msm_ba_rank_apply_kernel, rank_tiles, BA_SCAN_THREADS, 0, bitmap, n_words, rtiles, wrank);
            BaRoundArgs ra{};
            ra.first = r == 0;
            ra.bases = bases; ra.sorted = sorted; ra.prev = prev;
            ra.bitmap = bitmap; ra.wrank = wrank; ra.t_out = off_out + G;
            ra.target_units = target_units;
            ra.unit_ctr = ba_ctr.as<uint32_t>() + 2 * r;
            ra.prefix = ba_prefix.p; ra.tot = ba_tot.p; ra.inv_scratch = ba_tot.as<F>() + tot_bound; ra.out = ba_out[nxt ^ 1].p;   // even rounds write [1], odd rounds [0]
            if (is_g1) B2S_TRY(msm_ba_round_g1(c, ra));
            else B2S_TRY(msm_ba_round_g2(c, ra));
            prev = ba_out[nxt ^ 1].p;
            t_in = out_bound;
            cnt_in = cnt_out;
        }
        acc_bases = prev;
        acc_sorted = nullptr;
        acc_offsets = pp_off[(rp.rounds - 1) & 1u];
        acc_counts = pp_cnt[(rp.rounds - 1) & 1u];
    } else {
        // task offsets for the caller's counts (the rounds leave them behind as a by-product of their last scan)
        B2S_LAUNCH(c, msm_scan_tiles_kernel, ntiles, SCAN_THREADS, 0, counts, no_perm, sh, tiles.as<Scan3>());
        B2S_LAUNCH(c, msm_scan_spine_kernel, 1, 1024, 0, tiles.as<Scan3>(), ntiles, sh, offsets, task_off, heavy);
        B2S_LAUNCH(c, msm_scan_apply_kernel, ntiles, SCAN_THREADS, 0, counts, no_perm, sh, tiles.as<Scan3>(), offsets, task_off, heavy);
    }
    // task ranks by decreasing bucket size (skipped after affine rounds, which leave the natural order)
    const uint32_t* perm = nullptr;
    DevBuf perm_buf;
    if (!rp.rounds && G >= 1024) {
        B2S_TRY(perm_buf.alloc(c, ((size_t)G + 2 * SIZE_BINS) * sizeof(uint32_t)));
        uint32_t* pm = perm_buf.as<uint32_t>();
        uint32_t* hist = pm + G;
        uint32_t* binoff = hist + SIZE_BINS;
        uint32_t* none = nullptr;
        B2S_CUDA(c, cudaMemsetAsync(hist, 0, SIZE_BINS * sizeof(uint32_t), c->stream));
        B2S_LAUNCH(c, msm_size_hist_kernel, cdiv(G, 256), 256, 0, acc_counts, G, hist);
        B2S_LAUNCH(c, msm_size_scan_kernel, 1, 1024, 0, hist, binoff);
        B2S_LAUNCH(c, msm_size_scatter_kernel, cdiv(G, 256), 256, 0, acc_counts, G, binoff, hist, pm);
        B2S_LAUNCH(c, msm_scan_tiles_kernel, ntiles, SCAN_THREADS, 0, acc_counts, (const uint32_t*)pm, sh, tiles.as<Scan3>());
        B2S_LAUNCH(c, msm_scan_spine_kernel, 1, 1024, 0, tiles.as<Scan3>(), ntiles, sh, none, task_off, heavy);
        B2S_LAUNCH(c, msm_scan_apply_kernel, ntiles, SCAN_THREADS, 0, acc_counts, (const uint32_t*)pm, sh, tiles.as<Scan3>(), none, task_off, heavy);
        perm = pm;
    }
    if (is_g1) B2S_TRY(msm_accumulate_g1(c, acc_bases, acc_sorted, acc_offsets, task_off, perm, sh, bucket_acc, partials.p));
    else B2S_TRY(msm_accumulate_g2(c, acc_bases, acc_sorted, acc_offsets, task_off, perm, sh, bucket_acc, partials.p));
    const size_t red_smem = (size_t)MSM_RED_THREADS * sizeof(Pt);
    B2S_SMEM_ATTR(c, msm_reduce_heavy_kernel<F>, red_smem);
    B2S_SMEM_ATTR(c, msm_reduce_heavy_stage1_kernel<F>, red_smem);
    B2S_LAUNCH(c, msm_reduce_heavy_stage1_kernel<F>, 4 * c->sm_count, MSM_RED_THREADS, red_smem, heavy, task_off, hp,
               partials.as<Pt>(), heavy_tmp.as<Pt>());
    B2S_LAUNCH(c, msm_reduce_heavy_kernel<F>, 2 * c->sm_count, MSM_RED_THREADS, red_smem, heavy, task_off, perm, hp,
               partials.as<Pt>(), heavy_tmp.as<Pt>(), bucket_acc);
    return B2S_OK;
}

// bounds[k] = (g_k, offsets[g_k]) with g_k the first bucket whose entries start at or after k * T / S, k = 0 .. S
__global__ void msm_slice_bounds_kernel(const uint32_t* __restrict__ offsets, uint32_t G, uint64_t T, uint32_t S, uint2* __restrict__ bounds) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k > S) return;
    const uint64_t e = T * k / S;
    uint32_t lo = 0, hi = G;          // offsets[G] = T >= e
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (offsets[mid] < e) lo = mid + 1; else hi = mid;
    }
    bounds[k] = make_uint2(lo, offsets[lo]);
}

// bucket_acc[g] = sum of the points bases[sorted[offsets[g] .. offsets[g+1])] (sign in bit 31), for G buckets holding T
// entries in all.  counts / offsets are the caller's (device); bucket_acc must be zeroed.  Rounds of batched-affine
// halving first (msm_affine.cuh), then the XYZZ kernel, then the buckets that were cut into several tasks are joined.
// When the rounds' scratch for all G buckets does not fit (rp.slice_entries < T), all of that runs once per slice of
// whole buckets [g0, g1): buckets are independent and their entries contiguous in `sorted`, so a slice is a smaller
// problem of the same kind.  The S + 1 bounds are read back once.
template <class Curve, class F>
static int32_t bucket_sums_t(Ctx* c, const Affine<F>* bases, const uint32_t* sorted, uint32_t* counts, uint32_t* offsets, uint64_t T, uint32_t G,
                             const RoundPlan& rp, XYZZ<F>* bucket_acc) {
    if (!rp.rounds || rp.slice_entries >= T) return bucket_slice_t<Curve, F>(c, bases, sorted, counts, offsets, T, G, rp, bucket_acc);
    // even entry targets give slices of at most T / S entries plus the bucket that straddles a target; with skewed scalars
    // that bucket may be large, so S doubles until every slice fits (or one bucket alone is over the budget)
    std::vector<uint2> hb;
    uint32_t S = (uint32_t)std::min<uint64_t>(G, (T + rp.slice_entries - 1) / rp.slice_entries);
    for (int tries = 0;; tries++) {
        DevBuf db;
        B2S_TRY(db.alloc(c, ((size_t)S + 1) * sizeof(uint2)));
        B2S_LAUNCH(c, msm_slice_bounds_kernel, cdiv(S + 1, 256), 256, 0, (const uint32_t*)offsets, G, T, S, db.as<uint2>());
        hb.resize((size_t)S + 1);
        B2S_CUDA(c, cudaMemcpyAsync(hb.data(), db.p, hb.size() * sizeof(uint2), cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        uint64_t largest = 0;
        for (uint32_t k = 0; k < S; k++) largest = std::max<uint64_t>(largest, hb[k + 1].y - hb[k].y);
        if (largest <= rp.slice_entries) break;
        if (tries == 3 || S >= G) {
            // a bucket on its own exceeds the budget: no rounds at all (the XYZZ kernel needs no scratch per entry)
            RoundPlan plain = rp;
            plain.rounds = 0;
            plain.slice_entries = T;
            plan_tasks(plain, T, G);
            return bucket_slice_t<Curve, F>(c, bases, sorted, counts, offsets, T, G, plain, bucket_acc);
        }
        S = std::min<uint32_t>(G, 2 * S);
    }
    for (uint32_t k = 0; k < S; k++) {
        const uint32_t g0 = hb[k].x, g1 = hb[k + 1].x, e0 = hb[k].y, e1 = hb[k + 1].y;
        if (e1 == e0) continue;       // empty buckets keep their zeroed sums
        RoundPlan sp = rp;
        plan_tasks(sp, e1 - e0, g1 - g0);
        B2S_TRY((bucket_slice_t<Curve, F>(c, bases, sorted + e0, counts + g0, offsets + g0, e1 - e0, g1 - g0, sp, bucket_acc + g0)));
    }
    return B2S_OK;
}

// ---- the Pippenger pipeline proper ---------------------------------------------------------------------------------
// index_map (optional): scalar i belongs to base index_map[i] (the multiplicity-aware front end hands over a compacted
// scalar array); nullptr: base i.
// K > 1: K scalar vectors (vector k at scalars + k * stride) over the same n bases, out[k] = MSM of vector k.  They run as one
// Pippenger problem whose bucket key is (vector, window, digit): K * nwin super-windows of B buckets (K with a table).
template <class Curve, class F>
static int32_t msm_core_t(Ctx* c, const Affine<F>* bases, const typename Curve::Fr* scalars, const uint32_t* index_map, uint64_t n, bool mont,
                          XYZZ<F>* out, void* wins_ext, bool* used_aux = nullptr, const MsmPre* pre = nullptr, uint32_t K = 1, uint64_t stride = 0) {
    using Fr = typename Curve::Fr;
    using Pt = XYZZ<F>;
    constexpr bool is_g1 = sizeof(F) == sizeof(typename Curve::Fq);
    if (n == 0) {
        B2S_CUDA(c, cudaMemsetAsync(out, 0, K * sizeof(Pt), c->stream));
        return B2S_OK;
    }
    MsmShape sh = msm_shape(n, Curve::FrP::BITS, sizeof(Pt), pre, K);
    if ((uint64_t)K * sh.nwin * n >= (1ull << 32) || (uint64_t)K * sh.nwin * sh.B >= (1ull << 32))
        return fail(c, B2S_ERR_INVALID_ARG, "msm: vectors * n * windows exceeds 2^32");
    if (pre && (uint64_t)pre->nwin * pre->stride >= (1ull << 31)) return fail(c, B2S_ERR_INVALID_ARG, "msm: precomputed table exceeds 2^31 points");
    const uint32_t MSM_SEG = sh.B >= (1u << 16) ? 32u : 16u;
    // what stays allocated beside the rounds: the u32 arrays, the sorted indices, the bucket sums and the segment sums
    const uint64_t held = (uint64_t)sh.G * (5 * sizeof(uint32_t) + sizeof(Pt)) + (uint64_t)K * sh.nwin * n * sizeof(uint32_t) +
                          (uint64_t)K * (pre ? 1u : sh.nwin) * ((sh.B + MSM_SEG - 1) / MSM_SEG) * sizeof(Pt);
    const RoundPlan rp = plan_rounds<F>(c, (uint64_t)K * sh.nwin * n, sh.G, is_g1, sh.L, held);
    sh.L = rp.L; sh.max_tasks = rp.max_tasks;
    const uint32_t ntiles = (sh.G + SCAN_TILE - 1) / SCAN_TILE;
    DevBuf ibuf, sorted, bucket_acc, segs, wins, tiles;
    B2S_TRY(tiles.alloc(c, (size_t)ntiles * sizeof(Scan3)));
    // u32 arrays: counts[G] cursor[G] offsets[G+1] task_off[G+1] heavy[G+1]
    const size_t ints = (size_t)5 * sh.G + 3;
    B2S_TRY(ibuf.alloc(c, ints * sizeof(uint32_t)));
    uint32_t* counts = ibuf.as<uint32_t>();
    uint32_t* cursor = counts + sh.G;
    uint32_t* offsets = cursor + sh.G;
    uint32_t* task_off = offsets + sh.G + 1;
    uint32_t* heavy = task_off + sh.G + 1;
    B2S_CUDA(c, cudaMemsetAsync(counts, 0, (size_t)2 * sh.G * sizeof(uint32_t), c->stream));
    const uint64_t T = (uint64_t)K * sh.nwin * n;
    B2S_TRY(sorted.alloc(c, (size_t)T * sizeof(uint32_t)));
    B2S_TRY(bucket_acc.alloc(c, (size_t)sh.G * sizeof(Pt)));
    B2S_CUDA(c, cudaMemsetAsync(bucket_acc.p, 0, (size_t)sh.G * sizeof(Pt), c->stream));  // identity = zeros
    const uint32_t segs_per_win = (sh.B + MSM_SEG - 1) / MSM_SEG;
    // what the bucket reduction and the Horner tail see: K * nwin windows of B buckets, or K with a precomputed table
    MsmShape sh_red = sh;
    sh_red.nwin = K * (pre ? 1u : sh.nwin);
    B2S_TRY(segs.alloc(c, (size_t)segs_per_win * sh_red.nwin * sizeof(Pt)));
    if (sh.nwin > 64 || K > 1) wins_ext = nullptr;   // caller scratch holds 64 window sums; tiny windows take the in-stream path
    if (!wins_ext) B2S_TRY(wins.alloc(c, (size_t)std::max(sh.nwin, sh_red.nwin) * sizeof(Pt)));
    Pt* wins_p = wins_ext ? reinterpret_cast<Pt*>(wins_ext) : wins.as<Pt>();

    B2S_LAUNCH(c, msm_count_kernel<Fr>, dim3(cdiv(n, 256), K), 256, 0, scalars, n, stride, mont, sh, counts);
    const uint32_t* no_perm = nullptr;
    B2S_LAUNCH(c, msm_scan_tiles_kernel, ntiles, SCAN_THREADS, 0, counts, no_perm, sh, tiles.as<Scan3>());
    B2S_LAUNCH(c, msm_scan_spine_kernel, 1, 1024, 0, tiles.as<Scan3>(), ntiles, sh, offsets, task_off, heavy);
    B2S_LAUNCH(c, msm_scan_apply_kernel, ntiles, SCAN_THREADS, 0, counts, no_perm, sh, tiles.as<Scan3>(), offsets, task_off, heavy);
    {
        // the partitioned entries (u32 value + u16 fine key) go back to the pool before bucket_sums_t allocates its rounds
        const uint32_t fine_bits = sort_fine_bits(sh.c), nbins = sh.G >> fine_bits, nbw = sh.B >> fine_bits;
        DevBuf part;
        B2S_TRY(part.alloc(c, (size_t)T * (sizeof(uint32_t) + sizeof(uint16_t)) + (size_t)nbins * sizeof(uint32_t)));
        uint32_t* part_val = part.as<uint32_t>();
        uint32_t* bin_cursor = part_val + T;
        uint16_t* part_fine = reinterpret_cast<uint16_t*>(bin_cursor + nbins);
        B2S_CUDA(c, cudaMemsetAsync(bin_cursor, 0, (size_t)nbins * sizeof(uint32_t), c->stream));
        B2S_SMEM_ATTR(c, msm_partition_kernel<Fr>, partition_smem(nbw));
        B2S_SMEM_ATTR(c, msm_place_kernel, place_smem(fine_bits));
        B2S_LAUNCH(c, msm_partition_kernel<Fr>, dim3(cdiv(n, SORT_TILE), K), SORT_THREADS, partition_smem(nbw), scalars, index_map, n, stride, mont, sh,
                   fine_bits, (const uint32_t*)offsets, bin_cursor, part_val, part_fine);
        B2S_LAUNCH(c, msm_place_kernel, nbins + c->sm_count, SORT_THREADS, place_smem(fine_bits), (const uint32_t*)offsets, nbins, fine_bits,
                   (const uint32_t*)part_val, (const uint16_t*)part_fine, cursor, sorted.as<uint32_t>());
    }
    B2S_TRY((bucket_sums_t<Curve, F>(c, bases, sorted.as<uint32_t>(), counts, offsets, T, sh.G, rp, bucket_acc.as<Pt>())));
    // bucket reduction: compiled with the multiplication inlined (msm_acc_g1.cu), 2 general additions per bucket
    if (is_g1) B2S_TRY(msm_bucket_reduce_g1(c, bucket_acc.p, sh_red, MSM_SEG, segs.p, segs_per_win, wins_p));
    else B2S_TRY(msm_bucket_reduce_g2(c, bucket_acc.p, sh_red, MSM_SEG, segs.p, segs_per_win, wins_p));
    if (!wins_ext) {
        B2S_TRY(msm_horner(c, c->stream, is_g1 ? 1 : 2, wins_p, sh_red, K, out));
    } else {
        // tail on the aux stream: it only needs the window sums, the main stream goes on with the next MSM
        B2S_CUDA(c, cudaEventRecord(c->ev_tail, c->stream));
        B2S_CUDA(c, cudaStreamWaitEvent(c->aux, c->ev_tail, 0));
        B2S_TRY(msm_horner(c, c->aux, is_g1 ? 1 : 2, wins_p, sh_red, K, out));
        c->aux_pending = true;
        if (used_aux) *used_aux = true;
    }
    return B2S_OK;
}

// ---- multiplicity-aware front end -----------------------------------------------------------------------------------
// Witness vectors repeat values: the reference's own synthetic circuits assign ONE value to every witness
// (relations/src/sr1cs/mod.rs:306-309), real circuits are full of 0, 1 and a handful of constants.  Pippenger spends
// ceil(255 / c) additions on every (point, scalar) pair regardless; but  sum_{i : s_i = v} s_i P_i = v * sum_{i : s_i = v} P_i,
// ONE addition per point plus one scalar multiplication per distinct heavy value.  So, per MSM:
//   1 sample   1024 scalars to the host; values seen in >= 3 % of the sample become candidates (at most 8; zero scalars are
//              simply dropped).  Candidates are hints only -- membership is decided by full 256-bit comparison, so the
//              result is exact whatever the sample looked like;
//   2 classify every scalar: candidate j -> heavy list j (a bucket structure of <= 8 buckets), anything else -> the REST;
//   3 heavy    bucket sums of the heavy lists with the same batched-affine rounds + XYZZ kernels (bucket_sums_t);
//   4 rest     the ordinary pipeline (msm_core_t) over the compacted rest, bases addressed through the index list;
//   5 finish   out = rest + sum_j v_j * S_j  (four-lane team scalar multiplications, one warp per candidate).
// Uniform scalars never get past step 1 (one 32 KiB copy and a stream synchronisation).
static constexpr uint32_t DEDUP_SAMPLES = 1024, DEDUP_MAX = 8;
struct DedupCand { uint32_t v[DEDUP_MAX][8]; uint32_t k; };   // candidate values in the caller's representation (Montgomery or canonical)

template <class Fr>
__global__ void msm_sample_kernel(const Fr* __restrict__ scalars, uint64_t n, uint64_t stride, Fr* __restrict__ out) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= DEDUP_SAMPLES) return;
    const uint64_t i = (uint64_t)t * stride;
    if (i < n) st_struct(out + t, ld_struct(scalars + i));
}
// gid: 0..k-1 heavy list, DEDUP_MAX = rest, DEDUP_MAX + 1 = zero (dropped)
template <class Fr>
__device__ __forceinline__ uint32_t dedup_gid(const Fr& s, const DedupCand& cd) {
    uint32_t nz = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) nz |= s.v[j];
    if (nz == 0) return DEDUP_MAX + 1;
    for (uint32_t k = 0; k < cd.k; k++) {
        uint32_t d = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) d |= s.v[j] ^ cd.v[k][j];
        if (d == 0) return k;
    }
    return DEDUP_MAX;
}
// pass 0: counts[gid]++;  pass 1: lists (heavy: index into sorted at off[gid] + cursor, rest: compacted index + scalar copy)
template <class Fr, int PASS>
__global__ void msm_classify_kernel(const Fr* __restrict__ scalars, uint64_t n, DedupCand cd, uint32_t* __restrict__ counts /*DEDUP_MAX + 1*/,
                                    const uint32_t* __restrict__ off, uint32_t* __restrict__ cursor, uint32_t* __restrict__ heavy_sorted,
                                    uint32_t* __restrict__ rest_idx, Fr* __restrict__ rest_scalars) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31;
    Fr s = Fr::zero();
    uint32_t gid = DEDUP_MAX + 1;
    if (i < n) { s = ld_struct(scalars + i); gid = dedup_gid(s, cd); }
    const unsigned peers = __match_any_sync(0xffffffffu, gid);
    if (gid > DEDUP_MAX) return;
    const unsigned leader = (unsigned)(__ffs(peers) - 1);
    const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
    if (PASS == 0) {
        if (lane == leader) atomicAdd(&counts[gid], (uint32_t)__popc(peers));
    } else {
        uint32_t base = 0;
        if (lane == leader) base = atomicAdd(&cursor[gid], (uint32_t)__popc(peers));
        base = __shfl_sync(peers, base, leader);
        if (gid < DEDUP_MAX) heavy_sorted[off[gid] + base + rank] = (uint32_t)i;
        else { rest_idx[base + rank] = (uint32_t)i; st_struct(rest_scalars + base + rank, s); }
    }
}
// out += sum_j v_j * S_j   (one warp per candidate)
template <class Curve, class F>
__global__ void __launch_bounds__(32 * DEDUP_MAX)
msm_heavy_finish_kernel(const XYZZ<F>* __restrict__ sums, DedupCand cd, bool mont, XYZZ<F>* __restrict__ out) {
    using Fr = typename Curve::Fr;
    extern __shared__ uint4 fin_smem[];
    XYZZ<F>* table = reinterpret_cast<XYZZ<F>*>(fin_smem);            // [k][16]
    XYZZ<F>* res = table + (size_t)DEDUP_MAX * 16;                      // [k]
    const uint32_t w = threadIdx.x >> 5;
    if (w < cd.k) {
        Fr v;
#pragma unroll
        for (int j = 0; j < 8; j++) v.v[j] = cd.v[w][j];
        if (mont) v = v.from_mont();
        else { v = v.to_mont(); v = v.from_mont(); }                    // canonical input may exceed r: reduce
        XYZZ<F> r = team_scalar_mul(ld_struct(sums + w), v.v, Fr::N, table + (size_t)w * 16);
        if ((threadIdx.x & 31) == 0) res[w] = r;
    }
    __syncthreads();
    if (w == 0) {
        XYZZ<F> acc = ld_plain(out);
        for (uint32_t j = 0; j < cd.k; j++) team_add(acc, res[j]);
        if (threadIdx.x == 0) st_struct(out, acc);
    }
}

// A rest of a handful of points (the DummyCircuit witness leaves ~10) does not deserve the Pippenger pipeline -- two dozen
// launches and a 255-doubling Horner tail for nothing: one warp per (point, scalar) product, then one warp sums.
static constexpr uint32_t TINY_REST = 24;
template <class Curve, class F>
__global__ void __launch_bounds__(32)
msm_tiny_products_kernel(const Affine<F>* __restrict__ bases, const uint32_t* __restrict__ rest_idx, const typename Curve::Fr* __restrict__ rest_scal, uint32_t n_rest,
                         const XYZZ<F>* __restrict__ heavy_sums, DedupCand cd, bool mont, XYZZ<F>* __restrict__ prods) {
    using Fr = typename Curve::Fr;
    const uint32_t j = blockIdx.x;      // j < n_rest: rest element j;  else heavy list j - n_rest
    Fr v;
    XYZZ<F> p;
    if (j < n_rest) {
        v = ld_struct(rest_scal + j);
        p = XYZZ<F>::from_affine(ld_struct(bases + rest_idx[j]));
    } else {
#pragma unroll
        for (int t = 0; t < 8; t++) v.v[t] = cd.v[j - n_rest][t];
        p = ld_struct(heavy_sums + (j - n_rest));
    }
    if (mont) v = v.from_mont();
    else { v = v.to_mont(); v = v.from_mont(); }
    __shared__ XYZZ<F> table[16];
    const XYZZ<F> r = team_scalar_mul(p, v.v, Fr::N, table);
    if (threadIdx.x == 0) st_struct(prods + j, r);
}
template <class F>
__global__ void __launch_bounds__(32) msm_tiny_sum_kernel(const XYZZ<F>* __restrict__ prods, uint32_t count, XYZZ<F>* __restrict__ out) {
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t j = 0; j < count; j++) team_add(acc, ld_struct(prods + j));
    if (threadIdx.x == 0) st_struct(out, acc);
}

}  // namespace b2s
struct b2s::MsmDedupCache {
    bool valid = false;
    const void* scalars = nullptr;
    uint64_t n = 0, n_heavy = 0, n_rest = 0;
    bool mont = false;
    DedupCand cd{};
    DevBuf ints, heavy_sorted, rest_idx, rest_scal;
};
namespace b2s {
void msm_dedup_scope_begin(Ctx* c) {
    if (!c->dedup_cache) c->dedup_cache = new MsmDedupCache();
}
void msm_dedup_scope_end(Ctx* c) {
    delete c->dedup_cache;      // DevBufs go back to the pool in stream order
    c->dedup_cache = nullptr;
}

template <class Curve, class F>
static int32_t msm_run_t(Ctx* c, const void* bases_dev, const void* scalars_dev, uint64_t n, bool mont, void* out_dev, void* wins_ext,
                         const MsmPre* pre) {
    using Fr = typename Curve::Fr;
    using Pt = XYZZ<F>;
    constexpr bool is_g1 = sizeof(F) == sizeof(typename Curve::Fq);
    if (n >= (1ull << 31)) return fail(c, B2S_ERR_INVALID_ARG, "msm: n = %llu exceeds 2^31 - 1", (unsigned long long)n);
    const Fr* scalars = reinterpret_cast<const Fr*>(scalars_dev);
    const Affine<F>* bases = reinterpret_cast<const Affine<F>*>(bases_dev);
    Pt* out = reinterpret_cast<Pt*>(out_dev);
    // classification of this scalar vector: from the proof's cache when an earlier MSM of the same proof used the same one
    MsmDedupCache local;
    MsmDedupCache* dc = c->dedup_cache ? c->dedup_cache : &local;
    const bool hit = dc->valid && dc->scalars == scalars_dev && dc->n == n && dc->mont == mont;
    if (!hit) {
        if (dc->valid && c->aux_pending) {
            // the lists about to be replaced may still be read by tiny-rest kernels of earlier MSMs on the aux stream
            B2S_CUDA(c, cudaEventRecord(c->ev_done, c->aux));
            B2S_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_done, 0));
        }
        dc->valid = false;
        dc->cd = DedupCand{};
        if (n >= env_u32("B2S_MSM_DEDUP_MIN", 1u << 16) && env_u32("B2S_MSM_DEDUP", 1)) {
            // step 1: sample
            DevBuf sm;
            B2S_TRY(sm.alloc(c, DEDUP_SAMPLES * sizeof(Fr)));
            const uint64_t stride = std::max<uint64_t>(1, n / DEDUP_SAMPLES);
            B2S_LAUNCH(c, msm_sample_kernel<Fr>, cdiv(DEDUP_SAMPLES, 256), 256, 0, scalars, n, stride, sm.as<Fr>());
            std::vector<uint32_t> hs((size_t)DEDUP_SAMPLES * 8);
            B2S_CUDA(c, cudaMemcpyAsync(hs.data(), sm.p, hs.size() * 4, cudaMemcpyDeviceToHost, c->stream));
            B2S_CUDA(c, cudaStreamSynchronize(c->stream));
            std::map<std::array<uint32_t, 8>, uint32_t> freq;
            const uint32_t taken = (uint32_t)std::min<uint64_t>(DEDUP_SAMPLES, (n + stride - 1) / stride);
            for (uint32_t t = 0; t < taken; t++) {
                std::array<uint32_t, 8> key;
                memcpy(key.data(), hs.data() + (size_t)t * 8, 32);
                freq[key]++;
            }
            std::vector<std::pair<uint32_t, std::array<uint32_t, 8>>> top;
            for (auto& kv : freq) {
                bool zero = true;
                for (uint32_t w : kv.first) zero = zero && w == 0;
                if (!zero && kv.second * 100 >= taken * 3) top.push_back({kv.second, kv.first});
            }
            std::sort(top.begin(), top.end(), [](auto& a, auto& b) { return a.first > b.first; });
            for (size_t j = 0; j < top.size() && j < DEDUP_MAX; j++) memcpy(dc->cd.v[dc->cd.k++], top[j].second.data(), 32);
        }
        dc->scalars = scalars_dev; dc->n = n; dc->mont = mont;
        dc->n_heavy = dc->n_rest = 0;
        if (dc->cd.k != 0) {
            // step 2: classify (count, then lists)
            B2S_TRY(dc->ints.alloc(c, (3 * (DEDUP_MAX + 2)) * sizeof(uint32_t)));          // counts | offsets | cursor
            uint32_t* counts = dc->ints.as<uint32_t>();
            uint32_t* offs = counts + DEDUP_MAX + 2;
            uint32_t* cursor = offs + DEDUP_MAX + 2;
            B2S_CUDA(c, cudaMemsetAsync(dc->ints.p, 0, dc->ints.bytes, c->stream));
            B2S_LAUNCH_N(c, "msm_classify_count", (msm_classify_kernel<Fr, 0>), cdiv(n, 256), 256, 0, scalars, n, dc->cd, counts, (const uint32_t*)offs, cursor,
                         (uint32_t*)nullptr, (uint32_t*)nullptr, (Fr*)nullptr);
            uint32_t hcounts[DEDUP_MAX + 1];
            B2S_CUDA(c, cudaMemcpyAsync(hcounts, counts, sizeof(hcounts), cudaMemcpyDeviceToHost, c->stream));
            B2S_CUDA(c, cudaStreamSynchronize(c->stream));
            uint64_t n_heavy = 0;
            uint32_t hoffs[DEDUP_MAX + 2] = {0};
            for (uint32_t j = 0; j < DEDUP_MAX; j++) { hoffs[j] = (uint32_t)n_heavy; n_heavy += hcounts[j]; }
            hoffs[DEDUP_MAX] = (uint32_t)n_heavy;
            dc->n_heavy = n_heavy;
            dc->n_rest = hcounts[DEDUP_MAX];
            if (n_heavy * 8 < n) {
                dc->cd.k = 0;       // the sample misled: not worth it
            } else {
                B2S_CUDA(c, cudaMemcpyAsync(offs, hoffs, sizeof(hoffs), cudaMemcpyHostToDevice, c->stream));
                B2S_CUDA(c, cudaStreamSynchronize(c->stream));      // hoffs lives on this stack frame
                B2S_TRY(dc->heavy_sorted.alloc(c, std::max<uint64_t>(n_heavy, 1) * sizeof(uint32_t)));
                B2S_TRY(dc->rest_idx.alloc(c, std::max<uint64_t>(dc->n_rest, 1) * sizeof(uint32_t)));
                B2S_TRY(dc->rest_scal.alloc(c, std::max<uint64_t>(dc->n_rest, 1) * sizeof(Fr)));
                B2S_LAUNCH_N(c, "msm_classify_lists", (msm_classify_kernel<Fr, 1>), cdiv(n, 256), 256, 0, scalars, n, dc->cd, counts, (const uint32_t*)offs,
                             cursor, dc->heavy_sorted.as<uint32_t>(), dc->rest_idx.as<uint32_t>(), dc->rest_scal.as<Fr>());
            }
        }
        dc->valid = true;
    }
    if (dc->cd.k == 0) return msm_core_t<Curve, F>(c, bases, scalars, nullptr, n, mont, out, wins_ext, nullptr, pre);
    const DedupCand cd = dc->cd;
    const uint64_t n_heavy = dc->n_heavy, n_rest = dc->n_rest;
    uint32_t* counts = dc->ints.as<uint32_t>();
    uint32_t* offs = counts + DEDUP_MAX + 2;
    DevBuf& heavy_sorted = dc->heavy_sorted;
    DevBuf& rest_idx = dc->rest_idx;
    DevBuf& rest_scal = dc->rest_scal;
    // heavy-list sums and (tiny rest) products: read by aux-stream kernels, so they live in the ctx's persistent slot ring
    static_assert((DEDUP_MAX + TINY_REST + DEDUP_MAX) * sizeof(XYZZ<F>) <= Ctx::AUX_SLOT_BYTES, "aux slot too small");
    Pt* const hsums = reinterpret_cast<Pt*>(c->aux_slot());
    Pt* const prods_ring = hsums + DEDUP_MAX;
    // step 3: heavy bucket sums (<= DEDUP_MAX buckets)
    B2S_CUDA(c, cudaMemsetAsync(hsums, 0, DEDUP_MAX * sizeof(Pt), c->stream));
    {
        const RoundPlan rp = plan_rounds<F>(c, n_heavy, DEDUP_MAX, is_g1, (uint32_t)std::max<uint64_t>(64, n_heavy >> 18));
        B2S_TRY((bucket_sums_t<Curve, F>(c, bases, heavy_sorted.as<uint32_t>(), counts, offs, n_heavy, DEDUP_MAX, rp, hsums)));
    }
    if (n_rest <= TINY_REST) {
        // steps 4 + 5 for a tiny rest: every product v * P (rest) and v_j * S_j (heavy) in its own warp, then one sum
        const uint32_t count = (uint32_t)n_rest + cd.k;
        Pt* const prods = prods_ring;
        // latency-bound (255 dependent doublings): inside a proof it goes to the aux stream, under the next MSM
        const bool on_aux = wins_ext != nullptr;
        cudaStream_t ts = on_aux ? c->aux : c->stream;
        if (on_aux) {
            B2S_CUDA(c, cudaEventRecord(c->ev_tail, c->stream));
            B2S_CUDA(c, cudaStreamWaitEvent(c->aux, c->ev_tail, 0));
        }
        B2S_LAUNCH_SN(c, ts, is_g1 ? "msm_tiny_products_g1" : "msm_tiny_products_g2", (msm_tiny_products_kernel<Curve, F>), count, 32, 0, bases,
                      (const uint32_t*)rest_idx.as<uint32_t>(), (const Fr*)rest_scal.as<Fr>(), (uint32_t)n_rest, (const Pt*)hsums, cd, mont, prods);
        B2S_LAUNCH_SN(c, ts, is_g1 ? "msm_tiny_sum_g1" : "msm_tiny_sum_g2", msm_tiny_sum_kernel<F>, 1, 32, 0, (const Pt*)prods, count, out);
        if (on_aux) c->aux_pending = true;
        return B2S_OK;
    }
    // step 4: the rest through the ordinary pipeline
    bool used_aux = false;
    B2S_TRY((msm_core_t<Curve, F>(c, bases, rest_scal.as<Fr>(), rest_idx.as<uint32_t>(), n_rest, mont, out, wins_ext, &used_aux, pre)));
    // step 5: on the stream that writes `out` (the aux stream when the Horner tail went there; the heavy sums were finished on
    // the main stream before the event the aux stream waits for)
    cudaStream_t fs = used_aux ? c->aux : c->stream;
    const size_t fin_smem = ((size_t)DEDUP_MAX * 16 + DEDUP_MAX) * sizeof(Pt);
    B2S_SMEM_ATTR(c, (msm_heavy_finish_kernel<Curve, F>), fin_smem);
    B2S_LAUNCH_SN(c, fs, is_g1 ? "msm_heavy_finish_g1" : "msm_heavy_finish_g2", (msm_heavy_finish_kernel<Curve, F>), 1, 32 * DEDUP_MAX, fin_smem,
                  (const Pt*)hsums, cd, mont, out);
    return B2S_OK;
}

// Generic use of the scan kernels (setup_groth16.cu: column-sorted matrices): offsets[i] = sum_{j<i} counts[j],
// task_off[i] = sum_{j<i} ceil(counts[j] / L); both arrays have n + 1 entries.
int32_t scan_counts(Ctx* c, const uint32_t* counts, uint32_t n, uint32_t L, uint32_t* offsets, uint32_t* task_off) {
    MsmShape sh{};
    sh.G = n;
    sh.L = L;
    const uint32_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    DevBuf tiles, heavy;
    B2S_TRY(tiles.alloc(c, (size_t)ntiles * sizeof(Scan3)));
    B2S_TRY(heavy.alloc(c, ((size_t)n + 1) * sizeof(uint32_t)));
    const uint32_t* no_perm = nullptr;
    B2S_LAUNCH(c, msm_scan_tiles_kernel, ntiles, SCAN_THREADS, 0, counts, no_perm, sh, tiles.as<Scan3>());
    B2S_LAUNCH(c, msm_scan_spine_kernel, 1, 1024, 0, tiles.as<Scan3>(), ntiles, sh, offsets, task_off, heavy.as<uint32_t>());
    B2S_LAUNCH(c, msm_scan_apply_kernel, ntiles, SCAN_THREADS, 0, counts, no_perm, sh, tiles.as<Scan3>(), offsets, task_off, heavy.as<uint32_t>());
    return B2S_OK;
}

int32_t msm_join_tails(Ctx* c) {
    if (!c->aux_pending) return B2S_OK;
    B2S_CUDA(c, cudaEventRecord(c->ev_done, c->aux));
    B2S_CUDA(c, cudaStreamWaitEvent(c->stream, c->ev_done, 0));
    c->aux_pending = false;
    return B2S_OK;
}

int32_t msm_run(Ctx* c, int group, const void* bases_dev, const void* scalars_dev, uint64_t n, bool scalars_mont,
                void* out_xyzz_dev, void* wins_ext, const MsmPre* pre) {
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        if (group == 1) return msm_run_t<C, typename C::Fq>(c, bases_dev, scalars_dev, n, scalars_mont, out_xyzz_dev, wins_ext, pre);
        return msm_run_t<C, typename C::Fq2>(c, bases_dev, scalars_dev, n, scalars_mont, out_xyzz_dev, wins_ext, pre);
    });
}

int32_t msm_run_batch(Ctx* c, int group, const void* bases_dev, const void* scalars_dev, uint64_t n, uint64_t stride, uint32_t K,
                      bool scalars_mont, void* out_xyzz_dev, const MsmPre* pre) {
    if (n >= (1ull << 31)) return fail(c, B2S_ERR_INVALID_ARG, "msm: n = %llu exceeds 2^31 - 1", (unsigned long long)n);
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        const auto* s = reinterpret_cast<const typename C::Fr*>(scalars_dev);
        if (group == 1) {
            using F = typename C::Fq;
            return msm_core_t<C, F>(c, reinterpret_cast<const Affine<F>*>(bases_dev), s, nullptr, n, scalars_mont, reinterpret_cast<XYZZ<F>*>(out_xyzz_dev),
                                    nullptr, nullptr, pre, K, stride);
        }
        using F = typename C::Fq2;
        return msm_core_t<C, F>(c, reinterpret_cast<const Affine<F>*>(bases_dev), s, nullptr, n, scalars_mont, reinterpret_cast<XYZZ<F>*>(out_xyzz_dev),
                                nullptr, nullptr, pre, K, stride);
    });
}

// bits of the ctx curve's scalar field: 255 (BLS12-381), 254 (BN254), 253 (BLS12-377)
static uint32_t fr_bits(Ctx* c) {
    uint32_t bits = 0;
    dispatch_curve(c, [&](auto curve) { bits = decltype(curve)::FrP::BITS; return (int32_t)B2S_OK; });
    return bits;
}

// Per vector of a batch: device bytes of an MSM over n points, and how many vectors the u32 entry and bucket indices allow.
uint64_t msm_batch_bytes(Ctx* c, int group, uint64_t n, const MsmPre* pre, uint64_t* max_k) {
    const Sizes z = sizes(c);
    const uint32_t bits = fr_bits(c);
    const size_t pt = z.xyzz(group);
    const MsmShape sh = msm_shape(std::max<uint64_t>(n, 1), bits, pt, pre);
    const uint64_t T = (uint64_t)sh.nwin * n, G = sh.G;
    *max_k = std::max<uint64_t>(1, std::min(((1ull << 32) - 1) / std::max<uint64_t>(T, 1), ((1ull << 32) - 1) / G));
    // buckets with their five u32 arrays and segment sums; per entry the sorted index, the partitioned entry, the task
    // partials, and the scratch of the batched-affine rounds (half the entries: 1.5 affine points and one field element each)
    const uint64_t fe = z.aff(group) / 2;
    return G * (pt + 5 * sizeof(uint32_t)) + T * (sizeof(uint32_t) * 2 + sizeof(uint16_t)) + (T / 16 + G) * pt + T * (3 * fe + fe) / 2;
}

// Device bytes of one msm_run over n points beside its inputs: *sort_bytes while it sorts (u32 arrays, sorted and partitioned
// entries, bucket and segment sums), *round_bytes more while its batched-affine rounds run in one piece.
void msm_working_set(Ctx* c, int group, uint64_t n, const MsmPre* pre, uint64_t* sort_bytes, uint64_t* round_bytes) {
    const Sizes z = sizes(c);
    const size_t pt = z.xyzz(group);
    const MsmShape sh = msm_shape(std::max<uint64_t>(n, 1), fr_bits(c), pt, pre);
    const uint64_t T = (uint64_t)sh.nwin * n, G = sh.G;
    const uint64_t segs = (uint64_t)(pre ? 1u : sh.nwin) * (sh.B / 16 + 1);
    *sort_bytes = G * (5 * sizeof(uint32_t) + pt) + segs * pt + T * (2 * sizeof(uint32_t) + sizeof(uint16_t));
    *round_bytes = round_scratch_bytes(T, G, z.aff(group), pt);
}

// ---- fixed-base window precomputation for a resident key ----------------------------------------------------------------
// table[w * n + i] = 2^(c w) * P_i, normalised to affine: c doublings per window step, one inversion per output (a one-off at
// key upload).  With it the digits of ALL windows of an MSM over these bases share one set of 2^(c-1) buckets: nwin times
// fewer buckets to reduce, no per-window sums, no Horner tail, and a shard of the key keeps the window size of the full key.
template <class F>
__global__ void __launch_bounds__(128) msm_precompute_kernel(const Affine<F>* __restrict__ bases, uint64_t n, uint32_t c, uint32_t nwin, Affine<F>* __restrict__ table) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Affine<F> p = ld_struct(bases + i);
    st_struct(table + i, p);
    XYZZ<F> acc = XYZZ<F>::from_affine(p);
    for (uint32_t w = 1; w < nwin; w++) {
        for (uint32_t k = 0; k < c; k++) acc = acc.dbl();
        const Affine<F> q = acc.to_affine();
        st_struct(table + (uint64_t)w * n + i, q);
        acc = XYZZ<F>::from_affine(q);          // keep the chain in the cheaper mixed form
    }
}

uint32_t msm_precompute_windows(Ctx* c, uint64_t n, uint32_t* c_out) {
    // one bucket set whatever the number of windows: c = 20 balances n * nwin additions against 2^(c-1) buckets from 2^18
    // points up, and beat c = 22 at 2^24 (DESIGN.md section 4)
    (void)n;
    const uint32_t bits = fr_bits(c);
    const uint32_t cc = env_u32("B2S_MSM_PRE_C", 20);
    uint32_t nw = (bits + cc - 1) / cc;
    if (bits - (nw - 1) * cc >= cc) nw += 1;
    if (c_out) *c_out = cc;
    return nw;
}

int32_t msm_precompute(Ctx* c, int group, const void* bases_dev, uint64_t n, void* table_dev, MsmPre* pre) {
    uint32_t cc = 0;
    const uint32_t nw = msm_precompute_windows(c, n, &cc);
    if ((uint64_t)nw * n >= (1ull << 31)) return fail(c, B2S_ERR_INVALID_ARG, "msm_precompute: table of %u x %llu points exceeds 2^31", nw, (unsigned long long)n);
    pre->c = cc; pre->nwin = nw; pre->stride = (uint32_t)n;
    if (n == 0) return B2S_OK;
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        if (group == 1)
            B2S_LAUNCH_N(c, "msm_precompute_g1", msm_precompute_kernel<typename C::Fq>, cdiv(n, 128), 128, 0, reinterpret_cast<const Affine<typename C::Fq>*>(bases_dev), n,
                         cc, nw, reinterpret_cast<Affine<typename C::Fq>*>(table_dev));
        else
            B2S_LAUNCH_N(c, "msm_precompute_g2", msm_precompute_kernel<typename C::Fq2>, cdiv(n, 128), 128, 0, reinterpret_cast<const Affine<typename C::Fq2>*>(bases_dev),
                         n, cc, nw, reinterpret_cast<Affine<typename C::Fq2>*>(table_dev));
        return (int32_t)B2S_OK;
    });
}

template <class Curve, class F>
static int32_t group_sum_t(Ctx* c, const void* xyzz_dev, uint32_t count, void* out_affine_dev) {
    const size_t red_smem = (size_t)MSM_RED_THREADS * sizeof(XYZZ<F>);
    B2S_CUDA(c, cudaFuncSetAttribute(group_sum_affine_kernel<F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)red_smem));
    B2S_LAUNCH(c, group_sum_affine_kernel<F>, 1, MSM_RED_THREADS, red_smem, reinterpret_cast<const XYZZ<F>*>(xyzz_dev),
               count, reinterpret_cast<Affine<F>*>(out_affine_dev));
    return B2S_OK;
}

int32_t group_sum_to_affine(Ctx* c, int group, const void* xyzz_dev, uint32_t count, void* out_affine_dev) {
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        if (group == 1) return group_sum_t<C, typename C::Fq>(c, xyzz_dev, count, out_affine_dev);
        return group_sum_t<C, typename C::Fq2>(c, xyzz_dev, count, out_affine_dev);
    });
}

}  // namespace b2s
