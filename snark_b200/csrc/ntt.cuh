// Pieces of the NTT shared by the single-GPU schedule (ntt.cu) and the distributed four-step schedule (dntt.cu):
// power tables, vector loads, the shared-memory tile and its radix-2 DIF butterflies.
#pragma once
#include "common.cuh"

namespace b2s {

static constexpr int NTT_TILE_LOG = 10;   // elements per CTA tile (32 KiB of shared memory)
static constexpr int NTT_THREADS = 256;
static constexpr int NTT_MAX_RADIX_LOG = 10;

struct PowTab {
    const void* lo = nullptr;   // lo[i] = base^i,            i < 2^a
    const void* hi = nullptr;   // hi[i] = c * base^(i 2^a),  i < 2^(log_n - a)   (c = optional constant)
    uint32_t a = 0;
};

// Full-size factor tables of a plan (ntt.cu, built on the first single-GPU transform of that size).  The passes are bound by the
// integer-multiply pipe while DRAM sits at ~7 %: reading a precomputed factor (32 B per element, streamed like the data) is
// free, composing it from two small tables costs a multiplication per element.
struct NttFull {
    DevBuf buf;
    const void* bnd[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};   // [inverse][pass]: inter-pass twiddles, entry k * 2^log_m + m
    const void* wr[2][3] = {{nullptr, nullptr, nullptr}, {nullptr, nullptr, nullptr}};   // [inverse][pass]: butterfly twiddles w_R^e, e < R/2
    // witness-map scalings (r1cs.cu): input g^j / N for the coset NTT behind an UNSCALED inverse transform, output
    // g^-j * Zinv / N for the closing coset inverse transform
    const void* wm_pre = nullptr;
    const void* wm_post = nullptr;
    const void* wm_beta = nullptr;   // one element: Zinv / N
    // circom witness map (NTT_M_ODD): input w2^j / N, built on the first odd-coset transform of the size (N entries)
    DevBuf odd_buf;
    const void* odd_pre = nullptr;
};

struct NttPlan {
    uint32_t log_n = 0;
    int npass = 0;
    uint32_t radix[3] = {0, 0, 0};
    DevBuf tables;     // all pow tables, contiguous
    PowTab fwd, inv, coset_in, coset_out_scaled;
    const void* n_inv = nullptr;   // one element: N^-1 (plain iNTT output scaling)
    const void* zinv = nullptr;    // one element: (g^N - 1)^-1, the vanishing polynomial's inverse on the coset g H
    const void* one = nullptr;     // one element: 1
    bool full_tried = false;
    NttFull* full = nullptr;       // nullptr: factors are composed from the two-level tables
    // NTT_M_ODD input scaling w2^j / N (w2 = primitive 2N-th root), two-level form; built on the first odd-coset transform
    DevBuf odd_tables;
    PowTab odd_in;
    ~NttPlan() { delete full; }
};

template <class Fr>
__device__ __forceinline__ Fr gld(const Fr* p) {
    static_assert(Fr::N == 8, "scalar fields are 8 x 32-bit limbs");
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = q[0], b = q[1];
    Fr r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
template <class Fr>
__device__ __forceinline__ void gst(Fr* p, const Fr& r) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
    q[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

template <class Fr>
__device__ __forceinline__ Fr pow_lookup(const PowTab& t, uint64_t e) {
    const Fr* lo = reinterpret_cast<const Fr*>(t.lo);
    const Fr* hi = reinterpret_cast<const Fr*>(t.hi);
    Fr l = gld<Fr>(lo + (e & ((1ull << t.a) - 1)));
    return l * gld<Fr>(hi + (e >> t.a));
}

// out[i] = c * base^(i * stride)
template <class Fr>
__global__ void pow_table_kernel(Fr* out, uint32_t count, Fr base, uint64_t stride, Fr c) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    out[i] = c * base.pow_u64((uint64_t)i * stride);
}

// ---- shared-memory tile: element (row j, column c) as two uint4 at pitch (2C+1) -----------------
template <class Fr>
__device__ __forceinline__ Fr tile_ld(const uint4* sm, uint32_t j, uint32_t c, uint32_t pitch) {
    static_assert(Fr::N == 8, "scalar fields are 8 x 32-bit limbs");
    const uint4* p = sm + j * pitch + 2 * c;
    uint4 a = p[0], b = p[1];
    Fr r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
template <class Fr>
__device__ __forceinline__ void tile_st(uint4* sm, uint32_t j, uint32_t c, uint32_t pitch, const Fr& r) {
    uint4* p = sm + j * pitch + 2 * c;
    p[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
    p[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}
// R-point DIF NTT on every column of the tile; result row rho holds output bitrev(rho).
template <class Fr>
__device__ __forceinline__ void tile_dif(uint4* sm, const Fr* wtab, uint32_t log_r, uint32_t log_c, uint32_t pitch) {
    const uint32_t C = 1u << log_c;
    const uint32_t nbf = (1u << (log_r - 1)) << log_c;  // butterflies per stage
    for (uint32_t s = 0; s < log_r; s++) {
        const uint32_t lh = log_r - 1 - s;  // log2(half)
        const uint32_t half = 1u << lh;
        for (uint32_t b = threadIdx.x; b < nbf; b += blockDim.x) {
            const uint32_t c = b & (C - 1);
            const uint32_t t = b >> log_c;
            const uint32_t pos = t & (half - 1);
            const uint32_t j0 = ((t >> lh) << (lh + 1)) | pos;
            const uint32_t j1 = j0 + half;
            Fr x = tile_ld<Fr>(sm, j0, c, pitch);
            Fr y = tile_ld<Fr>(sm, j1, c, pitch);
            Fr d = x - y;
            if (lh != 0) d = d * gld<Fr>(wtab + (pos << s));   // last stage: all twiddles are 1
            tile_st<Fr>(sm, j0, c, pitch, x + y);
            tile_st<Fr>(sm, j1, c, pitch, d);
        }
        __syncthreads();
    }
}

__device__ __forceinline__ uint32_t bitrev(uint32_t x, uint32_t bits) { return bits ? (__brev(x) >> (32 - bits)) : 0; }

// plan (tables) for 2^log_n on this ctx, built on first use (ntt.cu)
int32_t ntt_get_plan(Ctx* c, uint32_t log_n, NttPlan** out);
// Transform modes.  INVERSE / COSET are ark-poly's four transforms (ifft scales by 1/N, the coset forms scale by g^j on the
// way in / g^-j on the way out).  WM marks the three variants witness_map chains together (they need plan->full):
//   WM | INVERSE           inverse transform WITHOUT the 1/N scaling
//   WM | COSET             forward coset transform whose input scaling is g^j / N   (makes up for the line above)
//   WM | INVERSE | COSET   inverse coset transform whose output scaling is g^-j * Zinv / N
// ODD marks the two variants of the circom witness map (odd coset w2 H, w2 a primitive 2N-th root; full tables optional):
//   ODD | INVERSE          inverse transform WITHOUT the 1/N scaling
//   ODD                    forward transform on the odd coset whose input scaling is w2^j / N (makes up for the line above)
enum : uint32_t { NTT_M_INVERSE = 1, NTT_M_COSET = 2, NTT_M_WM = 4, NTT_M_ODD = 8 };
// K > 1: K transforms of the vectors data_dev + k * 2^log_n, one launch per pass for all of them
int32_t ntt_run_mode(Ctx* c, void* data_dev, uint32_t log_n, uint32_t mode, uint32_t K = 1);
// plan with full-size tables, or *out = nullptr when they are switched off (B2S_NTT_FULL=0) or would not fit
int32_t ntt_get_full(Ctx* c, uint32_t log_n, NttPlan** out);
// dynamic shared memory of one pass CTA (tile of 1024 elements at pitch 2C+1, butterfly twiddles behind it)
inline size_t ntt_pass_smem_bytes() {
    return ((size_t)(1u << NTT_TILE_LOG) * 2 + (1u << NTT_MAX_RADIX_LOG) + 2) * sizeof(uint4) + (size_t)(1u << (NTT_MAX_RADIX_LOG - 1)) * 32;
}

}  // namespace b2s
