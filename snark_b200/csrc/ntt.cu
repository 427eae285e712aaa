// K2: radix-2 NTT / iNTT / coset variants over the scalar field, natural order in and out.
//
// GPU counterpart of ark-poly `Radix2EvaluationDomain::{fft,ifft}_in_place` and `get_coset`
// (upstream crate, not in /root/reference; SURVEY.md Appendix A.3; consumer: ark-groth16
// `witness_map`, Appendix A.2).  Exact field arithmetic, so any schedule gives identical bits.
//
// Schedule.  N = 2^log_n is factored N = R1 * R2 * R3 (up to three passes, R_i <= 2^10).  Viewing the
// data as [P][R][M'] (P = product of earlier radices, M' = product of later ones), pass i runs, for every
// (p, m), an R-point decimation-in-frequency NTT over the middle index in shared memory, multiplies
// output k by the inter-pass twiddle w_N^(P*m*k) and stores it at [p][k][m].  After the last pass the
// element at [k1][k2][k3] is X[k1 + R1*k2 + R1*R2*k3]; the last pass writes it straight to that index
// (a tile holds chunks with consecutive k1, so those writes are contiguous runs), which removes the
// separate bit-reversal pass.  Pass 1 streams data -> scratch, the middle pass works in place in
// scratch, the last pass streams scratch -> data: 3 reads + 3 writes of N*32 B in total.
//
// Per element and transform: 32 B read + 32 B written once is the algorithmic traffic (SURVEY 8d);
// the arithmetic is log_n/2 butterfly multiplications + 2 twiddle multiplications per extra pass --
// the kernel is bound by the integer-multiply (fma) pipe, not by HBM (see DESIGN.md).
//
// Factors.  The compact form composes w^e = lo[e mod 2^a] * hi[e >> a] from two 2^(log_n/2)-entry tables (256 KiB at
// 2^24, L2/L1 resident) -- one extra multiplication per use.  The passes are bound by the integer-multiply pipe with
// DRAM at ~7 % of its bandwidth, so the single-GPU schedule trades memory for multiplications: the inter-pass twiddles
// (N entries for the first boundary, N / R1 for the second) and the butterfly twiddles are precomputed per plan
// (NttFull, 1 GiB per direction at 2^24) and streamed next to the data.  Multiplications per element at 2^24:
// 10.5 in the butterflies (the last stage of a pass has twiddle 1) + 2 at the boundaries = 12.5, against 14.9 composed.
// Coset scaling (g^j on the way in, g^-j * N^-1 on the way out) is fused into the first / last pass, and so is the odd-coset
// scaling w2^j / N of the circom witness map (NTT_M_ODD).
#define B2S_INLINE_MUL 1   // Fr butterflies: the multiplication is the kernel
#include <cassert>
#include <memory>

#include "ntt.cuh"

namespace b2s {

struct PassArgs {
    uint32_t log_n, log_r, log_m, log_p, log_c;
    // final pass only
    uint32_t log_r1, log_pp;
    PowTab tw;        // w_N (or w_N^-1) powers
    PowTab pre;       // input scaling by base^index (lo == nullptr: none)
    PowTab post;      // output scaling by base^index * const (lo == nullptr: none)
    const void* post_const;  // else: output scaling by one constant (nullptr: none)
    // precomputed factors (NttFull); nullptr: composed from the two-level tables above
    const void* wr;          // butterfly twiddles w_R^e, e < R/2
    const void* bnd;         // strided pass: inter-pass twiddle of output (k, m) at entry k * 2^log_m + m
    const void* pre_full;    // input scaling, entry = global input index (takes the place of pre)
    const void* post_full;   // final pass: output scaling, entry = output index (takes the place of post / post_const)
    uint64_t bstride;        // batch: transform blockIdx.y works on src / dst + blockIdx.y * bstride (the factors are shared)
};

// Non-final pass: sub-NTTs over a strided middle index, in-place positions.
template <class Fr>
__global__ void __launch_bounds__(NTT_THREADS) ntt_pass_strided(const Fr* __restrict__ src, Fr* __restrict__ dst, PassArgs a) {
    extern __shared__ uint4 smem[];
    const uint32_t R = 1u << a.log_r, C = 1u << a.log_c;
    const uint32_t pitch = 2 * C + 1;
    uint4* tile = smem;
    src += blockIdx.y * a.bstride;
    dst += blockIdx.y * a.bstride;
    Fr* wtab = reinterpret_cast<Fr*>(smem + (size_t)R * pitch + 1);   // twiddles w_R^e behind the tile (16-byte aligned)
    const uint32_t tiles_per_p = 1u << (a.log_m - a.log_c);
    const uint64_t p = blockIdx.x / tiles_per_p;
    const uint64_t m0 = (uint64_t)(blockIdx.x % tiles_per_p) << a.log_c;
    const Fr* wr = reinterpret_cast<const Fr*>(a.wr);
    const Fr* bnd = reinterpret_cast<const Fr*>(a.bnd);
    const Fr* pre_full = reinterpret_cast<const Fr*>(a.pre_full);

    for (uint32_t e = threadIdx.x; e < R / 2; e += blockDim.x)
        gst<Fr>(wtab + e, wr ? gld<Fr>(wr + e) : pow_lookup<Fr>(a.tw, (uint64_t)e << (a.log_n - a.log_r)));
    for (uint32_t idx = threadIdx.x; idx < R * C; idx += blockDim.x) {
        const uint32_t c = idx & (C - 1), j = idx >> a.log_c;
        const uint64_t g = (((p << a.log_r) + j) << a.log_m) + m0 + c;
        Fr v = gld<Fr>(src + g);
        if (pre_full) v = v * gld<Fr>(pre_full + g);
        else if (a.pre.lo) v = v * pow_lookup<Fr>(a.pre, g);
        tile_st<Fr>(tile, j, c, pitch, v);
    }
    __syncthreads();
    tile_dif<Fr>(tile, wtab, a.log_r, a.log_c, pitch);
    for (uint32_t idx = threadIdx.x; idx < R * C; idx += blockDim.x) {
        const uint32_t c = idx & (C - 1), rho = idx >> a.log_c;
        const uint32_t k = bitrev(rho, a.log_r);
        const uint64_t m = m0 + c;
        Fr v = tile_ld<Fr>(tile, rho, c, pitch);
        const uint64_t e = (m * k) << a.log_p;
        if (e) v = v * (bnd ? gld<Fr>(bnd + (((uint64_t)k << a.log_m) + m)) : pow_lookup<Fr>(a.tw, e));
        gst<Fr>(dst + ((((p << a.log_r) + k) << a.log_m) + m), v);
    }
}

// Final pass: contiguous R-point chunks; writes each result to its natural-order index.
template <class Fr>
__global__ void __launch_bounds__(NTT_THREADS) ntt_pass_final(const Fr* __restrict__ src, Fr* __restrict__ dst, PassArgs a) {
    extern __shared__ uint4 smem[];
    const uint32_t R = 1u << a.log_r, C = 1u << a.log_c;
    const uint32_t pitch = 2 * C + 1;
    uint4* tile = smem;
    src += blockIdx.y * a.bstride;
    dst += blockIdx.y * a.bstride;
    Fr* wtab = reinterpret_cast<Fr*>(smem + (size_t)R * pitch + 1);
    const uint64_t PP = 1ull << a.log_pp;
    const uint64_t pp = blockIdx.x & (PP - 1);
    const uint64_t k1_0 = (uint64_t)(blockIdx.x >> a.log_pp) << a.log_c;
    const Fr* wr = reinterpret_cast<const Fr*>(a.wr);
    const Fr* pre_full = reinterpret_cast<const Fr*>(a.pre_full);
    const Fr* post_full = reinterpret_cast<const Fr*>(a.post_full);

    for (uint32_t e = threadIdx.x; e < R / 2; e += blockDim.x)
        gst<Fr>(wtab + e, wr ? gld<Fr>(wr + e) : pow_lookup<Fr>(a.tw, (uint64_t)e << (a.log_n - a.log_r)));
    for (uint32_t idx = threadIdx.x; idx < R * C; idx += blockDim.x) {
        const uint32_t j = idx & (R - 1), cc = idx >> a.log_r;
        const uint64_t chunk = ((k1_0 + cc) << a.log_pp) + pp;
        const uint64_t g = (chunk << a.log_r) + j;
        Fr v = gld<Fr>(src + g);
        if (pre_full) v = v * gld<Fr>(pre_full + g);
        else if (a.pre.lo) v = v * pow_lookup<Fr>(a.pre, g);
        tile_st<Fr>(tile, j, cc, pitch, v);
    }
    __syncthreads();
    tile_dif<Fr>(tile, wtab, a.log_r, a.log_c, pitch);
    for (uint32_t idx = threadIdx.x; idx < R * C; idx += blockDim.x) {
        const uint32_t cc = idx & (C - 1), rho = idx >> a.log_c;
        const uint64_t k = bitrev(rho, a.log_r);
        const uint64_t out = (k1_0 + cc) + ((pp + (k << a.log_pp)) << a.log_r1);
        Fr v = tile_ld<Fr>(tile, rho, cc, pitch);
        if (post_full) v = v * gld<Fr>(post_full + out);
        else if (a.post.lo) v = v * pow_lookup<Fr>(a.post, out);
        else if (a.post_const) v = v * gld<Fr>(reinterpret_cast<const Fr*>(a.post_const));
        gst<Fr>(dst + out, v);
    }
}

// ---- full-size factor tables (NttFull) ---------------------------------------------------------
// inter-pass twiddles of a strided pass: out[k * 2^log_m + m] = w^((m k) << log_p)
template <class Fr>
__global__ void ntt_bnd_table_kernel(Fr* __restrict__ out, PowTab tw, uint32_t log_m, uint32_t log_p, uint64_t count) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const uint64_t k = i >> log_m, m = i & ((1ull << log_m) - 1);
    gst<Fr>(out + i, pow_lookup<Fr>(tw, (m * k) << log_p));
}
// butterfly twiddles of an R-point sub-transform: out[e] = w^(e << shift), e < R/2
template <class Fr>
__global__ void ntt_wr_table_kernel(Fr* __restrict__ out, PowTab tw, uint32_t shift, uint32_t count) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < count) gst<Fr>(out + e, pow_lookup<Fr>(tw, (uint64_t)e << shift));
}
// out[j] = cst * base^j (base^j from the two-level table)
template <class Fr>
__global__ void ntt_scale_table_kernel(Fr* __restrict__ out, PowTab tab, const Fr* __restrict__ cst, uint64_t count) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j < count) gst<Fr>(out + j, gld<Fr>(cst) * pow_lookup<Fr>(tab, j));
}
// consts[0] = (g^N - 1)^-1, consts[1] = 1, consts[2] = Zinv / N      (n_inv: one element, N^-1)
template <class Fr, class FrP>
__global__ void ntt_consts_kernel(Fr* consts, const Fr* n_inv, uint64_t domain) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    Fr g;
    for (int i = 0; i < Fr::N; i++) g.v[i] = FrP::gen(i);
    const Fr zinv = (g.pow_u64(domain) - Fr::one()).inverse();
    consts[0] = zinv;
    consts[1] = Fr::one();
    consts[2] = zinv * n_inv[0];
}

// -------------------------------------------------------------------------------------------
#define B2S_FR_CONST(name, fn)          \
    Fr name;                            \
    for (int i_ = 0; i_ < Fr::N; i_++) name.v[i_] = FrP::fn(i_);

template <class Curve>
static int32_t build_plan(Ctx* c, uint32_t log_n, NttPlan** out) {
    using Fr = typename Curve::Fr;
    using FrP = typename Curve::FrP;
    if (log_n > (uint32_t)FrP::TWO_ADICITY || log_n > 3 * NTT_MAX_RADIX_LOG - 3)
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "NTT size 2^%u unsupported", log_n);
    NttPlan* pl = new NttPlan();
    pl->log_n = log_n;
    pl->npass = log_n <= NTT_MAX_RADIX_LOG ? 1 : (log_n <= 18 ? 2 : 3);
    for (int i = 0; i < pl->npass; i++) pl->radix[i] = log_n / pl->npass + ((uint32_t)i < log_n % pl->npass ? 1 : 0);
    const uint32_t a = (log_n + 1) / 2, b = log_n - a;
    const uint32_t nlo = 1u << a, nhi = 1u << b;
    // tables: fwd(lo,hi) inv(lo,hi) coset_in(lo,hi) coset_out(lo,hi) n_inv[1] zinv[1] one[1] zinv_n[1]
    const size_t total = 4 * (size_t)(nlo + nhi) + 4;
    int32_t st = pl->tables.alloc(c, total * sizeof(Fr));
    if (st != B2S_OK) { delete pl; return st; }
    Fr* base = pl->tables.as<Fr>();
    // host-side constants (tiny host use of the field templates: a handful of multiplications)
    B2S_FR_CONST(root, root) B2S_FR_CONST(root_inv, root_inv)
    B2S_FR_CONST(g, gen) B2S_FR_CONST(g_inv, gen_inv) B2S_FR_CONST(half, half)
    Fr w = root, wi = root_inv;
    for (uint32_t i = log_n; i < (uint32_t)FrP::TWO_ADICITY; i++) { w = w.sqr(); wi = wi.sqr(); }
    Fr n_inv = Fr::one();
    for (uint32_t i = 0; i < log_n; i++) n_inv = n_inv * half;
    const Fr one = Fr::one();
    struct Spec { Fr bse; Fr c; PowTab* dst; } specs[4] = {
        {w, one, &pl->fwd}, {wi, one, &pl->inv}, {g, one, &pl->coset_in}, {g_inv, n_inv, &pl->coset_out_scaled}};
    Fr* cur = base;
    for (auto& sp : specs) {
        sp.dst->lo = cur; sp.dst->hi = cur + nlo; sp.dst->a = a;
        pow_table_kernel<Fr><<<cdiv(nlo, 256), 256, 0, c->stream>>>(cur, nlo, sp.bse, 1, one);
        pow_table_kernel<Fr><<<cdiv(nhi, 256), 256, 0, c->stream>>>(cur + nlo, nhi, sp.bse, 1ull << a, sp.c);
        c->launches += 2;
        cur += nlo + nhi;
    }
    pl->n_inv = cur;
    pow_table_kernel<Fr><<<1, 32, 0, c->stream>>>(cur, 1, one, 0, n_inv);
    pl->zinv = cur + 1; pl->one = cur + 2;      // cur + 3: Zinv / N (NttFull::wm_beta)
    ntt_consts_kernel<Fr, FrP><<<1, 32, 0, c->stream>>>(cur + 1, cur, 1ull << log_n);
    c->launches += 2;
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { delete pl; return fail(c, B2S_ERR_CUDA, "ntt table build: %s", cudaGetErrorString(e)); }
    *out = pl;
    return B2S_OK;
}

int32_t ntt_get_plan(Ctx* c, uint32_t log_n, NttPlan** out) {
    auto it = c->ntt_plans.find(log_n);
    if (it != c->ntt_plans.end()) { *out = it->second; return B2S_OK; }
    NttPlan* pl = nullptr;
    B2S_TRY(dispatch_curve(c, [&](auto curve) { return build_plan<decltype(curve)>(c, log_n, &pl); }));
    c->ntt_plans[log_n] = pl;
    *out = pl;
    return B2S_OK;
}

// Full-size factor tables for this plan: built once, on the first single-GPU transform of the size (the distributed schedule,
// dntt.cu, only uses the two-level tables, so a rank of a group never pays for these).
template <class Curve>
static int32_t build_full(Ctx* c, NttPlan* pl) {
    using Fr = typename Curve::Fr;
    pl->full_tried = true;
    const char* env = getenv("B2S_NTT_FULL");
    if (env && atoi(env) == 0) return B2S_OK;
    const uint32_t log_n = pl->log_n;
    if (log_n == 0) return B2S_OK;
    const uint64_t N = 1ull << log_n;
    // entries: per direction, every non-final pass N >> log_p inter-pass twiddles and every pass R/2 butterfly twiddles;
    // two witness-map scalings of N entries
    uint64_t per_dir = 0;
    {
        uint32_t log_p = 0;
        for (int i = 0; i < pl->npass; i++) {
            if (i != pl->npass - 1) per_dir += N >> log_p;
            per_dir += 1ull << (pl->radix[i] - 1);
            log_p += pl->radix[i];
        }
    }
    const uint64_t total = 2 * per_dir + 2 * N;
    if (total * sizeof(Fr) > c->total_mem / 8) return B2S_OK;       // 2^26: 6 GiB, fine; beyond that the composed factors do
    std::unique_ptr<NttFull> fu(new NttFull());
    if (fu->buf.alloc(c, total * sizeof(Fr)) != B2S_OK) {           // no room: not an error, the composed factors do
        c->err.clear();
        cudaGetLastError();
        return B2S_OK;
    }
    Fr* cur = fu->buf.as<Fr>();
    for (int inv = 0; inv < 2; inv++) {
        const PowTab tw = inv ? pl->inv : pl->fwd;
        uint32_t log_p = 0;
        for (int i = 0; i < pl->npass; i++) {
            const uint32_t log_r = pl->radix[i], log_m = log_n - log_p - log_r;
            if (i != pl->npass - 1) {
                const uint64_t cnt = N >> log_p;
                B2S_LAUNCH(c, ntt_bnd_table_kernel<Fr>, cdiv(cnt, 256), 256, 0, cur, tw, log_m, log_p, cnt);
                fu->bnd[inv][i] = cur;
                cur += cnt;
            }
            const uint32_t half = 1u << (log_r - 1);
            B2S_LAUNCH(c, ntt_wr_table_kernel<Fr>, cdiv(half, 256), 256, 0, cur, tw, log_n - log_r, half);
            fu->wr[inv][i] = cur;
            cur += half;
            log_p += log_r;
        }
    }
    const Fr* n_inv = reinterpret_cast<const Fr*>(pl->n_inv);
    const Fr* zinv = reinterpret_cast<const Fr*>(pl->zinv);
    // g^j / N   and   (g^-j / N) * Zinv   (coset_out_scaled already carries the 1/N)
    B2S_LAUNCH(c, ntt_scale_table_kernel<Fr>, cdiv(N, 256), 256, 0, cur, pl->coset_in, n_inv, N);
    fu->wm_pre = cur;
    cur += N;
    B2S_LAUNCH(c, ntt_scale_table_kernel<Fr>, cdiv(N, 256), 256, 0, cur, pl->coset_out_scaled, zinv, N);
    fu->wm_post = cur;
    fu->wm_beta = zinv + 2;
    pl->full = fu.release();
    return B2S_OK;
}

// Factors of the odd-coset forward transform (NTT_M_ODD): w2^j / N with w2 the primitive 2N-th root, w2^2 = w.  Built on the
// first such transform of the size, so that a process that never runs the circom witness map allocates nothing for them: the
// two-level table (2^ceil(log_n/2) + 2^floor(log_n/2) entries) always, the full N-entry table when the plan has full tables.
template <class Curve>
static int32_t build_odd(Ctx* c, NttPlan* pl) {
    using Fr = typename Curve::Fr;
    using FrP = typename Curve::FrP;
    const uint32_t log_n = pl->log_n;
    // domains stop at 2^27 (r1cs upload, b2s_ntt) and the two-adicity is 28 (BN254) / 32 (BLS12-381): w2 always exists
    assert(log_n < (uint32_t)FrP::TWO_ADICITY);
    const uint32_t a = (log_n + 1) / 2, b = log_n - a;
    const uint32_t nlo = 1u << a, nhi = 1u << b;
    B2S_TRY(pl->odd_tables.alloc(c, (size_t)(nlo + nhi) * sizeof(Fr)));
    B2S_FR_CONST(w2, root) B2S_FR_CONST(half, half)
    for (uint32_t i = log_n + 1; i < (uint32_t)FrP::TWO_ADICITY; i++) w2 = w2.sqr();
    Fr n_inv = Fr::one();
    for (uint32_t i = 0; i < log_n; i++) n_inv = n_inv * half;
    Fr* lo = pl->odd_tables.as<Fr>();
    B2S_LAUNCH(c, pow_table_kernel<Fr>, cdiv(nlo, 256), 256, 0, lo, nlo, w2, (uint64_t)1, Fr::one());
    B2S_LAUNCH(c, pow_table_kernel<Fr>, cdiv(nhi, 256), 256, 0, lo + nlo, nhi, w2, 1ull << a, n_inv);
    pl->odd_in.lo = lo; pl->odd_in.hi = lo + nlo; pl->odd_in.a = a;
    NttFull* fu = pl->full;
    if (!fu) return B2S_OK;
    const uint64_t N = 1ull << log_n;
    if (fu->odd_buf.alloc(c, N * sizeof(Fr)) != B2S_OK) {   // no room: not an error, the two-level table does
        c->err.clear();
        cudaGetLastError();
        return B2S_OK;
    }
    B2S_LAUNCH(c, ntt_scale_table_kernel<Fr>, cdiv(N, 256), 256, 0, fu->odd_buf.as<Fr>(), pl->odd_in, reinterpret_cast<const Fr*>(pl->one), N);
    fu->odd_pre = fu->odd_buf.p;
    return B2S_OK;
}

int32_t ntt_get_full(Ctx* c, uint32_t log_n, NttPlan** out) {
    NttPlan* pl = nullptr;
    *out = nullptr;
    B2S_TRY(ntt_get_plan(c, log_n, &pl));
    if (!pl->full_tried) B2S_TRY(dispatch_curve(c, [&](auto curve) { return build_full<decltype(curve)>(c, pl); }));
    if (pl->full) *out = pl;
    return B2S_OK;
}

template <class Curve>
static int32_t ntt_run_t(Ctx* c, void* data_dev, uint32_t log_n, uint32_t mode, uint32_t K) {
    using Fr = typename Curve::Fr;
    const bool inverse = (mode & NTT_M_INVERSE) != 0, coset = (mode & NTT_M_COSET) != 0, wm = (mode & NTT_M_WM) != 0;
    const bool odd = (mode & NTT_M_ODD) != 0;
    if (log_n == 0 && !wm) return B2S_OK;  // size-1 transform is the identity (coset scaling g^0 = 1, 1/N = 1, w2^0 / N = 1)
    NttPlan* pl = nullptr;
    B2S_TRY(ntt_get_plan(c, log_n, &pl));
    if (!pl->full_tried) B2S_TRY(build_full<Curve>(c, pl));
    const NttFull* fu = pl->full;
    if (wm && !fu) return fail(c, B2S_ERR_INVALID_ARG, "ntt: witness-map transform modes need the full-size tables");
    if (odd && !inverse && !pl->odd_in.lo) B2S_TRY(build_odd<Curve>(c, pl));
    Fr* data = reinterpret_cast<Fr*>(data_dev);
    DevBuf scratch;
    if (pl->npass > 1) B2S_TRY(scratch.alloc(c, (sizeof(Fr) << log_n) * K));
    Fr* tmp = scratch.as<Fr>();

    PowTab none;
    const PowTab tw = inverse ? pl->inv : pl->fwd;
    const void* odd_full = (odd && !inverse && fu) ? fu->odd_pre : nullptr;
    const PowTab pre = (coset && !inverse && !wm) ? pl->coset_in : ((odd && !inverse && !odd_full) ? pl->odd_in : none);
    const PowTab post = (inverse && coset && !wm) ? pl->coset_out_scaled : none;
    const void* post_const = (inverse && !coset && !wm && !odd) ? pl->n_inv : nullptr;
    const void* pre_full = (wm && coset && !inverse) ? fu->wm_pre : odd_full;
    const void* post_full = (wm && coset && inverse) ? fu->wm_post : nullptr;

    const size_t smem_bytes = ((size_t)(1u << NTT_TILE_LOG) * 2 + (1u << NTT_MAX_RADIX_LOG) + 2) * sizeof(uint4) +
                              (size_t)(1u << (NTT_MAX_RADIX_LOG - 1)) * sizeof(Fr);
    B2S_SMEM_ATTR(c, ntt_pass_strided<Fr>, smem_bytes);
    B2S_SMEM_ATTR(c, ntt_pass_final<Fr>, smem_bytes);

    uint32_t log_p = 0;
    const Fr* src = data;
    for (int i = 0; i < pl->npass; i++) {
        const uint32_t log_r = pl->radix[i];
        const bool last = (i == pl->npass - 1);
        PassArgs a{};
        a.log_n = log_n; a.log_r = log_r; a.log_p = log_p; a.log_m = log_n - log_p - log_r;
        a.tw = tw;
        a.pre = (i == 0) ? pre : none;
        a.pre_full = (i == 0) ? pre_full : nullptr;
        a.post = none;
        a.post_const = nullptr;
        a.post_full = nullptr;
        a.wr = fu ? fu->wr[inverse ? 1 : 0][i] : nullptr;
        a.bnd = nullptr;
        a.bstride = 1ull << log_n;
        if (!last) {
            a.log_c = min((uint32_t)NTT_TILE_LOG - log_r, a.log_m);
            a.bnd = fu ? fu->bnd[inverse ? 1 : 0][i] : nullptr;
            Fr* dst = tmp;
            const unsigned grid = 1u << (log_n - log_r - a.log_c);
            B2S_LAUNCH(c, ntt_pass_strided<Fr>, dim3(grid, K), NTT_THREADS, smem_bytes, src, dst, a);
            src = tmp;
        } else {
            a.log_r1 = (pl->npass == 1) ? 0 : pl->radix[0];
            a.log_pp = log_p - a.log_r1;
            a.log_c = min((uint32_t)NTT_TILE_LOG - min(log_r, (uint32_t)NTT_TILE_LOG), a.log_r1);
            a.post = post;
            a.post_const = post_const;
            a.post_full = post_full;
            const unsigned grid = 1u << (log_n - log_r - a.log_c);
            B2S_LAUNCH(c, ntt_pass_final<Fr>, dim3(grid, K), NTT_THREADS, smem_bytes, src, data, a);
        }
        log_p += log_r;
    }
    return B2S_OK;
}

int32_t ntt_run_mode(Ctx* c, void* data_dev, uint32_t log_n, uint32_t mode, uint32_t K) {
    return dispatch_curve(c, [&](auto curve) { return ntt_run_t<decltype(curve)>(c, data_dev, log_n, mode, K); });
}

int32_t ntt_run(Ctx* c, void* data_dev, uint32_t log_n, bool inverse, bool coset) {
    return ntt_run_mode(c, data_dev, log_n, (inverse ? NTT_M_INVERSE : 0u) | (coset ? NTT_M_COSET : 0u));
}

void ntt_free_plans(Ctx* c) {
    for (auto& kv : c->ntt_plans) delete kv.second;
    c->ntt_plans.clear();
}

}  // namespace b2s
