// R1CS -> square R1CS on the GPU: Sr1csAdapter::r1cs_to_sr1cs and r1cs_to_sr1cs_with_assignment.
//
// Replaces, on the GPU:
//   Sr1csAdapter::r1cs_to_sr1cs                    /root/reference/relations/src/sr1cs/mod.rs:124-183
//   Sr1csAdapter::r1cs_to_sr1cs_with_assignment    /root/reference/relations/src/sr1cs/mod.rs:191-265
// Row i of a*b = c becomes (a+b)^2 = 4c + s_i (row 2i) and (a-b)^2 = s_i (row 2i+1), predicate x0^2 - x1.  The reference walks
// the rows in order and gives a column its new witness the first time it meets it (A_i, then B_i, then C_i, then s_i), so
// the numbering is a function of each column's first position in that scan.  Here every term has a scan key (its position
// in the concatenation of all rows' A, B, C terms and square slots); one atomicMin per term finds each column's first key,
// a flag per key plus one scan numbers the witnesses, and a fill writes both arguments renamed.  Row pointers are closed
// forms of the source's.  Everything is index work over the source CSR and runs once per circuit.
#define B2S_INLINE_MUL 1   // Fr only in this unit
#include <algorithm>
#include <cstddef>

#include "r1cs.cuh"

namespace b2s {
namespace {

constexpr uint64_t NONE = ~0ull;
// gridDim.y carries the assignment, and host batches go through this much device scratch per chunk (as gr1cs_check)
constexpr uint64_t ASSIGN_MAX_PER_LAUNCH = 65535;
constexpr uint64_t ASSIGN_SCRATCH_BYTES = 64ull << 20;

// the source A, B, C (device pointers)
struct Src {
    const uint64_t* rp[3];
    const uint32_t* col[3];
    const uint32_t* cid[3];
    uint64_t m;
};

// the row holding entry e of matrix k: the largest i with rp[i] <= e
__device__ __forceinline__ uint64_t row_of(const uint64_t* __restrict__ rp, uint64_t m, uint64_t e) {
    uint64_t lo = 0, hi = m;
    while (hi - lo > 1) {
        const uint64_t mid = (lo + hi) / 2;
        if (__ldg(rp + mid) <= e) lo = mid; else hi = mid;
    }
    return lo;
}

// where row i starts in the scan: every term and square slot of the rows before it
__device__ __forceinline__ uint64_t row_key(const Src& s, uint64_t i) { return s.rp[0][i] + s.rp[1][i] + s.rp[2][i] + i; }

// scan key of entry e of matrix K (row i): its row's start, the terms of the matrices before K in that row, its offset
template <int K>
__device__ __forceinline__ uint64_t entry_key(const Src& s, uint64_t i, uint64_t e) {
    uint64_t k = row_key(s, i) + (e - s.rp[K][i]);
    if (K >= 1) k += s.rp[0][i + 1] - s.rp[0][i];
    if (K >= 2) k += s.rp[1][i + 1] - s.rp[1][i];
    return k;
}

// one thread per entry of matrix K: first[col] = the smallest scan key of col (col 0, ONE, is never renamed)
template <int K>
__global__ void sr1cs_first_kernel(Src s, uint64_t nnz, unsigned long long* __restrict__ first) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const uint32_t col = s.col[K][e];
    if (col == 0) return;
    atomicMin(first + col, (unsigned long long)entry_key<K>(s, row_of(s.rp[K], s.m, e), e));
}

// one thread per entry of matrix K: flag[key] = 1 where a column is first met
template <int K>
__global__ void sr1cs_flag_kernel(Src s, uint64_t nnz, const unsigned long long* __restrict__ first, uint32_t* __restrict__ flag) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const uint32_t col = s.col[K][e];
    if (col == 0) return;
    const uint64_t key = entry_key<K>(s, row_of(s.rp[K], s.m, e), e);
    if (first[col] == key) flag[key] = 1;
}

// one thread per source column c < n_src: pub_flag[c] = 1 for a used public column (1 <= c < n_inst); threads c < m flag
// the square slot of row c, the last key of its row
__global__ void sr1cs_mark_kernel(Src s, uint64_t n_src, uint64_t n_inst, const unsigned long long* __restrict__ first,
                                  uint32_t* __restrict__ pub_flag, uint32_t* __restrict__ flag) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_inst) pub_flag[t] = t >= 1 && first[t] != NONE;
    if (t < s.m) flag[row_key(s, t + 1) - 1] = 1;
    (void)n_src;
}

// one thread per source column: ren[c] = its column in the result (1 + P + witness number; ONE stays 0; unused: 0), and
// orig[new column] = c for every used column; orig[1 + k] = p_k for the k-th used public column.  orig of a square stays 0.
__global__ void sr1cs_rename_kernel(uint64_t n_src, uint64_t n_inst, const unsigned long long* __restrict__ first,
                                    const uint32_t* __restrict__ wid, const uint32_t* __restrict__ pub_at, uint32_t P,
                                    uint32_t* __restrict__ ren, uint32_t* __restrict__ orig) {
    const uint64_t c = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n_src) return;
    uint32_t r = 0;
    if (c != 0 && first[c] != NONE) {
        r = 1 + P + wid[first[c]];
        orig[r] = (uint32_t)c;
        if (c < n_inst) orig[1 + pub_at[c]] = (uint32_t)c;
    }
    ren[c] = r;
}

// the result's two arguments, L (x0) and R (x1), in CSR
struct Dst {
    uint64_t* rp[2];
    uint32_t* col[2];
    uint32_t* cid[2];
};

// one thread per entry of matrix K, written renamed where the conversion puts it:
//   A: L row 2i and L row 2i+1, same id;  B: after A in both, id in row 2i and id + S (-coeff) in row 2i+1;
//   C: R row 2i, id + 2S (4 coeff)
// L row 2i starts at 2 (rpA[i] + rpB[i]) and row 2i+1 right after it; R row 2i at rpC[i] + 2i.
template <int K>
__global__ void sr1cs_fill_kernel(Src s, uint64_t nnz, const uint32_t* __restrict__ ren, uint32_t S, Dst d) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const uint64_t i = row_of(s.rp[K], s.m, e);
    const uint32_t col = ren[s.col[K][e]], id = s.cid[K][e];
    const uint64_t off = e - s.rp[K][i];
    if (K == 2) {
        const uint64_t at = s.rp[2][i] + 2 * i + off;
        d.col[1][at] = col;
        d.cid[1][at] = id + 2 * S;
        return;
    }
    const uint64_t a0 = s.rp[0][i], a1 = s.rp[0][i + 1], b0 = s.rp[1][i], b1 = s.rp[1][i + 1];
    const uint64_t row2i = 2 * (a0 + b0), len = (a1 - a0) + (b1 - b0);
    const uint64_t at = row2i + (K == 1 ? a1 - a0 : 0) + off;
    d.col[0][at] = col;
    d.cid[0][at] = id;
    d.col[0][at + len] = col;
    d.cid[0][at + len] = K == 1 ? id + S : id;
}

// one thread per result row r < 2m + P, and one more for the closing row pointers.  Rows 2i / 2i+1 write their row
// pointers and the square term of R; tie rows 2m + k write L = w(p_k) - x_k (ids 0 and S, i.e. ONE and -ONE).
__global__ void sr1cs_rows_kernel(Src s, uint32_t P, uint32_t S, const uint32_t* __restrict__ wid, const uint32_t* __restrict__ ren,
                                  const uint32_t* __restrict__ orig, Dst d) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t m = s.m, n_rows = 2 * m + P;
    const uint64_t nab = s.rp[0][m] + s.rp[1][m], nc = s.rp[2][m];
    if (r > n_rows) return;
    if (r == n_rows) {
        d.rp[0][r] = 2 * nab + 2 * (uint64_t)P;
        d.rp[1][r] = nc + 2 * m;
        return;
    }
    if (r >= 2 * m) {
        const uint64_t k = r - 2 * m, at = 2 * nab + 2 * k;
        d.rp[0][r] = at;
        d.rp[1][r] = nc + 2 * m;
        d.col[0][at] = ren[orig[1 + k]];
        d.cid[0][at] = 0;
        d.col[0][at + 1] = (uint32_t)(1 + k);
        d.cid[0][at + 1] = S;
        return;
    }
    const uint64_t i = r >> 1;
    const uint64_t a0 = s.rp[0][i], a1 = s.rp[0][i + 1], b0 = s.rp[1][i], b1 = s.rp[1][i + 1];
    const uint32_t sq = 1 + P + wid[row_key(s, i + 1) - 1];
    if ((r & 1) == 0) {
        d.rp[0][r] = 2 * (a0 + b0);
        d.rp[1][r] = s.rp[2][i] + 2 * i;
        const uint64_t at = s.rp[2][i + 1] + 2 * i;   // the slot after C_i's terms
        d.col[1][at] = sq;
        d.cid[1][at] = 0;
    } else {
        d.rp[0][r] = 2 * (a0 + b0) + (a1 - a0) + (b1 - b0);
        const uint64_t at = s.rp[2][i + 1] + 2 * i + 1;
        d.rp[1][r] = at;
        d.col[1][at] = sq;
        d.cid[1][at] = 0;
    }
}

// the pool [pool | -pool | 4 pool]
template <class Fr>
__global__ void sr1cs_pool_kernel(const Fr* __restrict__ src, uint32_t S, Fr* __restrict__ dst) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= S) return;
    const Fr v = src[j];
    dst[j] = v;
    dst[S + j] = Fr::zero() - v;
    dst[2 * (uint64_t)S + j] = v.dbl().dbl();
}

// one thread per (t, assignment blockIdx.y), t < n_vars + m.  t < n_vars: variable t of the result, a gather through orig
// (ONE for t = 0; squares, orig 0, are left to the row threads).  t = n_vars + i: s_i = (<A_i, z> - <B_i, z>)^2, read as
// L row 2i+1 = A_i' - B_i' (no square in it) through orig straight from z, written at the square's column, R row 2i+1's
// only term.
template <class Fr>
__global__ void __launch_bounds__(256)
sr1cs_assign_kernel(const uint64_t* __restrict__ l_rp, const uint32_t* __restrict__ l_col, const uint32_t* __restrict__ l_cid,
                    const uint64_t* __restrict__ r_rp, const uint32_t* __restrict__ r_col, const uint32_t* __restrict__ orig,
                    const Fr* __restrict__ pool, uint64_t n_vars, uint64_t m, const Fr* __restrict__ z, uint64_t z_stride,
                    Fr* __restrict__ out, uint64_t out_stride) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    z += blockIdx.y * z_stride;
    out += blockIdx.y * out_stride;
    if (t < n_vars) {
        if (t == 0) { out[0] = Fr::one(); return; }
        const uint32_t o = __ldg(orig + t);
        if (o != 0) out[t] = z[o];
        return;
    }
    const uint64_t i = t - n_vars;
    if (i >= m) return;
    const uint64_t beg = __ldg(l_rp + 2 * i + 1), end = __ldg(l_rp + 2 * i + 2);
    Fr acc = Fr::zero();
    for (uint64_t e = beg; e < end; e++) {
        const uint32_t c = __ldg(l_col + e), id = __ldg(l_cid + e);
        Fr v = c == 0 ? Fr::one() : z[__ldg(orig + c)];
        if (id != 0) v = v * pool[id];
        acc = acc + v;
    }
    out[__ldg(r_col + __ldg(r_rp + 2 * i + 1))] = acc.sqr();
}

// the gather of export: coefficient values of ids
template <class Fr>
__global__ void gr1cs_coeff_kernel(const uint32_t* __restrict__ cid, uint64_t n, const Fr* __restrict__ pool, Fr* __restrict__ out) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n) out[e] = pool[cid[e]];
}

// the SR1CS polynomial x0^2 - x1: terms (ONE, x0^2) and (-ONE, x1^1)
template <class FrP>
void sr1cs_poly(uint32_t coeff[2][8], uint32_t off[3], uint32_t var[2], uint32_t pow[2]) {
    uint64_t borrow = 0;
    for (int i = 0; i < 8; i++) {
        coeff[0][i] = FrP::r1(i);
        const uint64_t d = (uint64_t)FrP::mod(i) - FrP::r1(i) - borrow;   // r - ONE
        coeff[1][i] = (uint32_t)d;
        borrow = (d >> 63) & 1;
    }
    off[0] = 0, off[1] = 1, off[2] = 2;
    var[0] = 0, pow[0] = 2;
    var[1] = 1, pow[1] = 1;
}

template <class Curve>
int32_t to_sr1cs_t(Ctx* c, const b2s_r1cs* src, b2s_gr1cs** out) {
    using Fr = typename Curve::Fr;
    using FrP = typename Curve::FrP;
    const uint64_t m = src->n_rows, n_inst = src->n_instance, n_src = src->n_instance + src->n_witness;
    const uint64_t nnz[3] = {src->nnz[0], src->nnz[1], src->nnz[2]};
    const uint64_t n_keys = nnz[0] + nnz[1] + nnz[2] + m;
    if (2 * m >= (1ull << 32))
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs_to_sr1cs: %llu rows give 2^32 or more constraints", (unsigned long long)m);
    if (n_keys >= (1ull << 32) || n_src >= (1ull << 32))
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs_to_sr1cs: %llu nonzeros and rows, %llu variables; the limit is 2^32 - 1",
                    (unsigned long long)n_keys, (unsigned long long)n_src);
    const uint64_t S = src->pool_size;
    if (3 * S >= (1ull << 32)) return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs_to_sr1cs: pool of %llu coefficients", (unsigned long long)S);

    // a zkey handle leaves C unallocated: an empty matrix with zeroed row pointers
    Src s{};
    for (int k = 0; k < 3; k++) {
        s.rp[k] = src->row_ptr[k].as<uint64_t>();
        s.col[k] = src->col[k].as<uint32_t>();
        s.cid[k] = src->coeff_id[k].as<uint32_t>();
    }
    s.m = m;

    DevBuf first, flag, wid, wtask, pub_flag, pub_at, pub_task, ren;
    B2S_TRY(first.alloc(c, n_src * 8));
    B2S_TRY(flag.alloc(c, n_keys * 4 + 4));
    B2S_TRY(wid.alloc(c, (n_keys + 1) * 4));
    B2S_TRY(wtask.alloc(c, (n_keys + 1) * 4));
    B2S_TRY(pub_flag.alloc(c, n_inst * 4));
    B2S_TRY(pub_at.alloc(c, (n_inst + 1) * 4));
    B2S_TRY(pub_task.alloc(c, (n_inst + 1) * 4));
    B2S_TRY(ren.alloc(c, n_src * 4));
    B2S_CUDA(c, cudaMemsetAsync(first.p, 0xFF, n_src * 8, c->stream));
    B2S_CUDA(c, cudaMemsetAsync(flag.p, 0, n_keys * 4 + 4, c->stream));
    auto* fst = first.as<unsigned long long>();
    if (nnz[0]) B2S_LAUNCH(c, sr1cs_first_kernel<0>, cdiv(nnz[0], 256), 256, 0, s, nnz[0], fst);
    if (nnz[1]) B2S_LAUNCH(c, sr1cs_first_kernel<1>, cdiv(nnz[1], 256), 256, 0, s, nnz[1], fst);
    if (nnz[2]) B2S_LAUNCH(c, sr1cs_first_kernel<2>, cdiv(nnz[2], 256), 256, 0, s, nnz[2], fst);
    if (nnz[0]) B2S_LAUNCH(c, sr1cs_flag_kernel<0>, cdiv(nnz[0], 256), 256, 0, s, nnz[0], fst, flag.as<uint32_t>());
    if (nnz[1]) B2S_LAUNCH(c, sr1cs_flag_kernel<1>, cdiv(nnz[1], 256), 256, 0, s, nnz[1], fst, flag.as<uint32_t>());
    if (nnz[2]) B2S_LAUNCH(c, sr1cs_flag_kernel<2>, cdiv(nnz[2], 256), 256, 0, s, nnz[2], fst, flag.as<uint32_t>());
    const uint64_t n_mark = std::max(n_inst, m);
    B2S_LAUNCH(c, sr1cs_mark_kernel, cdiv(n_mark, 256), 256, 0, s, n_src, n_inst, (const unsigned long long*)fst, pub_flag.as<uint32_t>(),
               flag.as<uint32_t>());
    if (n_keys) B2S_TRY(scan_counts(c, flag.as<uint32_t>(), (uint32_t)n_keys, 1u, wid.as<uint32_t>(), wtask.as<uint32_t>()));
    else B2S_CUDA(c, cudaMemsetAsync(wid.p, 0, 4, c->stream));
    B2S_TRY(scan_counts(c, pub_flag.as<uint32_t>(), (uint32_t)n_inst, 1u, pub_at.as<uint32_t>(), pub_task.as<uint32_t>()));
    uint32_t n_w = 0, P = 0;   // U + m witnesses, P used public columns
    B2S_CUDA(c, cudaMemcpyAsync(&n_w, wid.as<uint32_t>() + n_keys, 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&P, pub_at.as<uint32_t>() + n_inst, 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    const uint64_t n_vars = 1 + (uint64_t)P + n_w, n_rows = 2 * m + P;
    if (n_vars >= (1ull << 32) || n_rows >= (1ull << 32))
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs_to_sr1cs: the result has %llu variables and %llu constraints; the limit is 2^32 - 1",
                    (unsigned long long)n_vars, (unsigned long long)n_rows);

    std::unique_ptr<b2s_gr1cs> g(new b2s_gr1cs());
    g->curve = c->curve;
    g->n_instance = 1 + P;
    g->n_witness = n_w;
    g->sr1cs_src_vars = n_src;
    g->sr1cs_rows = m;
    B2S_TRY(g->sr1cs_orig.alloc(c, n_vars * 4));
    B2S_CUDA(c, cudaMemsetAsync(g->sr1cs_orig.p, 0, n_vars * 4, c->stream));
    B2S_LAUNCH(c, sr1cs_rename_kernel, cdiv(n_src, 256), 256, 0, n_src, n_inst, (const unsigned long long*)fst, (const uint32_t*)wid.as<uint32_t>(),
               (const uint32_t*)pub_at.as<uint32_t>(), P, ren.as<uint32_t>(), g->sr1cs_orig.as<uint32_t>());

    std::unique_ptr<Gr1csPredicate> pr(new Gr1csPredicate());
    pr->arity = 2;
    pr->n_terms = 2;
    pr->n_rows = n_rows;
    pr->nnz[0] = 2 * (nnz[0] + nnz[1]) + 2 * (uint64_t)P;
    pr->nnz[1] = nnz[2] + 2 * m;
    Dst d{};
    for (int j = 0; j < 2; j++) {
        B2S_TRY(pr->row_ptr[j].alloc(c, (n_rows + 1) * 8));
        B2S_TRY(pr->col[j].alloc(c, pr->nnz[j] * 4));
        B2S_TRY(pr->coeff_id[j].alloc(c, pr->nnz[j] * 4));
        d.rp[j] = pr->row_ptr[j].as<uint64_t>();
        d.col[j] = pr->col[j].as<uint32_t>();
        d.cid[j] = pr->coeff_id[j].as<uint32_t>();
    }
    const uint32_t* rn = ren.as<uint32_t>();
    if (nnz[0]) B2S_LAUNCH(c, sr1cs_fill_kernel<0>, cdiv(nnz[0], 256), 256, 0, s, nnz[0], rn, (uint32_t)S, d);
    if (nnz[1]) B2S_LAUNCH(c, sr1cs_fill_kernel<1>, cdiv(nnz[1], 256), 256, 0, s, nnz[1], rn, (uint32_t)S, d);
    if (nnz[2]) B2S_LAUNCH(c, sr1cs_fill_kernel<2>, cdiv(nnz[2], 256), 256, 0, s, nnz[2], rn, (uint32_t)S, d);
    B2S_LAUNCH(c, sr1cs_rows_kernel, cdiv(n_rows + 1, 256), 256, 0, s, P, (uint32_t)S, (const uint32_t*)wid.as<uint32_t>(), rn,
               (const uint32_t*)g->sr1cs_orig.as<uint32_t>(), d);

    // the polynomial x0^2 - x1
    struct { uint32_t coeff[2][8]; uint32_t off[3], var[2], pow[2]; } poly;
    sr1cs_poly<FrP>(poly.coeff, poly.off, poly.var, poly.pow);
    B2S_TRY(pr->term_coeff.alloc(c, sizeof(poly.coeff)));
    B2S_TRY(pr->term_off.alloc(c, sizeof(poly.off)));
    B2S_TRY(pr->factor_var.alloc(c, sizeof(poly.var)));
    B2S_TRY(pr->factor_pow.alloc(c, sizeof(poly.pow)));
    B2S_CUDA(c, cudaMemcpyAsync(pr->term_coeff.p, poly.coeff, sizeof(poly.coeff), cudaMemcpyHostToDevice, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(pr->term_off.p, poly.off, sizeof(poly.off), cudaMemcpyHostToDevice, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(pr->factor_var.p, poly.var, sizeof(poly.var), cudaMemcpyHostToDevice, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(pr->factor_pow.p, poly.pow, sizeof(poly.pow), cudaMemcpyHostToDevice, c->stream));

    g->pool_size = (uint32_t)(3 * S);
    B2S_TRY(g->pool.alloc(c, 3 * S * sizeof(Fr)));
    if (S) B2S_LAUNCH(c, sr1cs_pool_kernel<Fr>, cdiv(S, 256), 256, 0, src->pool.as<Fr>(), (uint32_t)S, g->pool.as<Fr>());
    g->preds.push_back(std::move(pr));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));   // the host-side poly above, and the scratch freed with it
    *out = g.release();
    return B2S_OK;
}

template <class Curve>
int32_t assign_t(Ctx* c, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z) {
    using Fr = typename Curve::Fr;
    const uint64_t n_src = g->sr1cs_src_vars, n_vars = g->n_instance + g->n_witness, m = g->sr1cs_rows;
    const uint64_t in_row = n_src * sizeof(Fr), out_row = n_vars * sizeof(Fr);
    const Gr1csPredicate& pr = *g->preds[0];
    RowStager io(c, mem, {col_in(z, in_row), col_out(out_z, out_row)});
    uint64_t ch = std::min(ASSIGN_MAX_PER_LAUNCH, n_assign);
    if (io.staged) ch = std::min(ch, std::max<uint64_t>(1, ASSIGN_SCRATCH_BYTES / (in_row + out_row)));
    B2S_TRY(io.alloc(ch));
    for (uint64_t a0 = 0; a0 < n_assign; a0 += ch) {
        const uint64_t K = std::min(ch, n_assign - a0);
        B2S_TRY(io.load(a0, (uint32_t)K));
        B2S_LAUNCH(c, sr1cs_assign_kernel<Fr>, dim3(cdiv(n_vars + m, 256), (unsigned)K), 256, 0, pr.row_ptr[0].as<uint64_t>(),
                   pr.col[0].as<uint32_t>(), pr.coeff_id[0].as<uint32_t>(), pr.row_ptr[1].as<uint64_t>(), pr.col[1].as<uint32_t>(),
                   g->sr1cs_orig.as<uint32_t>(), g->pool.as<Fr>(), n_vars, m, io.ptr<const Fr>(0), n_src, io.ptr<Fr>(1), n_vars);
        B2S_TRY(io.store());
    }
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

int32_t same_curve(Ctx* c, const b2s_gr1cs* g, const char* who) {
    if (g->curve != c->curve)
        return fail(c, B2S_ERR_INVALID_ARG, "%s: the handle was made on a ctx of curve %d, this ctx is curve %d", who, g->curve, c->curve);
    return B2S_OK;
}

}  // namespace

int32_t r1cs_to_sr1cs(Ctx* c, const b2s_r1cs* m, b2s_gr1cs** out) {
    return dispatch_curve(c, [&](auto curve) { return to_sr1cs_t<decltype(curve)>(c, m, out); });
}

int32_t sr1cs_assignment(Ctx* c, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z) {
    B2S_TRY(same_curve(c, g, "sr1cs_assignment"));
    if (!g->sr1cs_orig.p)
        return fail(c, B2S_ERR_INVALID_ARG, "sr1cs_assignment: the handle was not made by b2s_r1cs_to_sr1cs");
    if (n_assign == 0) return B2S_OK;
    return dispatch_curve(c, [&](auto curve) { return assign_t<decltype(curve)>(c, g, n_assign, z, mem, out_z); });
}

int32_t gr1cs_info(Ctx* c, const b2s_gr1cs* g, uint64_t* n_vars, uint32_t* n_predicates, b2s_gr1cs_pred_info* preds, uint32_t cap) {
    B2S_TRY(same_curve(c, g, "gr1cs_info"));
    n_vars[0] = g->n_instance;
    n_vars[1] = g->n_witness;
    *n_predicates = (uint32_t)g->preds.size();
    for (uint32_t p = 0; p < std::min<uint32_t>(cap, (uint32_t)g->preds.size()); p++) {
        const Gr1csPredicate& pr = *g->preds[p];
        b2s_gr1cs_pred_info& o = preds[p];
        o = b2s_gr1cs_pred_info{};
        o.arity = pr.arity;
        o.n_rows = pr.n_rows;
        for (uint32_t j = 0; j < pr.arity; j++) o.nnz[j] = pr.nnz[j];
    }
    return B2S_OK;
}

int32_t gr1cs_export(Ctx* c, const b2s_gr1cs* g, uint32_t pred, uint32_t arg, uint64_t* row_ptr, uint64_t cap_row_ptr, uint32_t* col,
                     uint64_t cap_col, void* coeff, uint64_t cap_coeff) {
    B2S_TRY(same_curve(c, g, "gr1cs_export"));
    if (pred >= g->preds.size())
        return fail(c, B2S_ERR_INVALID_ARG, "gr1cs_export: predicate %u of %zu", pred, g->preds.size());
    const Gr1csPredicate& pr = *g->preds[pred];
    if (arg >= pr.arity) return fail(c, B2S_ERR_INVALID_ARG, "gr1cs_export: argument %u of arity %u", arg, pr.arity);
    const uint64_t nnz = pr.nnz[arg], rp_bytes = (pr.n_rows + 1) * 8;
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        using Fr = typename decltype(curve)::Fr;
        if (rp_bytes > cap_row_ptr || nnz * 4 > cap_col || nnz * sizeof(Fr) > cap_coeff)
            return fail(c, B2S_ERR_INVALID_ARG, "gr1cs_export: buffer too small (row_ptr %llu, col %llu, coeff %llu bytes needed)",
                        (unsigned long long)rp_bytes, (unsigned long long)(nnz * 4), (unsigned long long)(nnz * sizeof(Fr)));
        B2S_CUDA(c, cudaMemcpyAsync(row_ptr, pr.row_ptr[arg].p, rp_bytes, cudaMemcpyDeviceToHost, c->stream));
        DevBuf vals;
        if (nnz) {
            B2S_TRY(vals.alloc(c, nnz * sizeof(Fr)));
            B2S_LAUNCH(c, gr1cs_coeff_kernel<Fr>, cdiv(nnz, 256), 256, 0, pr.coeff_id[arg].as<uint32_t>(), nnz, g->pool.as<Fr>(), vals.as<Fr>());
            B2S_CUDA(c, cudaMemcpyAsync(col, pr.col[arg].p, nnz * 4, cudaMemcpyDeviceToHost, c->stream));
            B2S_CUDA(c, cudaMemcpyAsync(coeff, vals.p, nnz * sizeof(Fr), cudaMemcpyDeviceToHost, c->stream));
        }
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        return B2S_OK;
    });
}

}  // namespace b2s
