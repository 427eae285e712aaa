// K1: R1CS matrices x assignment (CSR SpMV), K3: the pointwise QAP quotient, and their composition
// into `witness_map`, under either QAP reduction (LibsnarkReduction, or ark-circom's CircomReduction).
//
// Replaces, on the GPU:
//   mat_vec_mul                         /root/reference/relations/src/utils/matrix.rs:26-36
//   Sr1csAdapter::evaluate_constraint   /root/reference/relations/src/sr1cs/mod.rs:24-56
//   (out of tree) ark-groth16 LibsnarkReduction::witness_map_from_matrices, SURVEY.md Appendix A.2
// The matrices are those exported by ConstraintSystem::to_matrices()
// (/root/reference/relations/src/gr1cs/constraint_system.rs:768-804): rows may hold duplicate or unsorted
// columns; the product simply sums.  Column c reads z[c] with z = instance || witness.
//
// SpMV is the one HBM-bound kernel of the path: per nonzero 4 B column + 4 B coefficient id + a 32 B
// gather from z (40 B/nnz), plus 8 B row_ptr and a 32 B result per row (SURVEY 8d).  Coefficients are
// interned like the reference's FieldInterner (relations/src/gr1cs/field_interner.rs:13-35, id 0 = ONE)
// so real circuits -- whose coefficients are almost all 1 -- skip the multiplication entirely.
#define B2S_INLINE_MUL 1   // Fr only in this unit
#include <unordered_map>

#include "ntt.cuh"
#include "r1cs.cuh"

namespace b2s {

template <class Fr>
__device__ __forceinline__ Fr fr_ld(const Fr* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = __ldg(q), b = __ldg(q + 1);
    Fr r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
template <class Fr>
__device__ __forceinline__ void fr_st(Fr* p, const Fr& r) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
    q[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

struct SpmvMat {
    const uint64_t* row_ptr;
    const uint32_t* col;
    const uint32_t* cid;
    void* out;
};

// One thread per (matrix, row) of the first NM matrices: 3 = A, B, C; 2 = A and B only (the circom witness map never reads
// C).  Batch: blockIdx.y is the assignment k, read at z + k * z_stride, its rows written at out + k * out_stride.
template <class Fr, int NM>
__global__ void __launch_bounds__(256)
spmv_kernel(SpmvMat m0, SpmvMat m1, SpmvMat m2, const Fr* __restrict__ pool, const Fr* __restrict__ z, uint64_t n_rows, uint64_t z_stride,
            uint64_t out_stride) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= NM * n_rows) return;
    z += blockIdx.y * z_stride;
    const uint32_t k = (uint32_t)(t / n_rows);
    const uint64_t row = t - (uint64_t)k * n_rows;
    const SpmvMat m = k == 0 ? m0 : (k == 1 || NM == 2 ? m1 : m2);
    const uint64_t beg = m.row_ptr[row], end = m.row_ptr[row + 1];
    Fr acc = Fr::zero();
    for (uint64_t e = beg; e < end; e++) {
        const uint32_t cid = m.cid[e];
        Fr v = fr_ld(z + m.col[e]);
        if (cid != 0) v = v * fr_ld(pool + cid);
        acc = acc + v;
    }
    fr_st(reinterpret_cast<Fr*>(m.out) + blockIdx.y * out_stride + row, acc);
}

// a[n_rows + i] = z[i], i < n_instance   (input-consistency rows of the LibsnarkReduction); blockIdx.y: assignment, as in spmv
template <class Fr>
__global__ void copy_instance_kernel(Fr* a, const Fr* z, uint64_t n_rows, uint64_t n_instance, uint64_t z_stride, uint64_t a_stride) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_instance) fr_st(a + blockIdx.y * a_stride + n_rows + i, fr_ld(z + blockIdx.y * z_stride + i));
}

// K3, first half: a[i] *= b[i]   (evaluations of A B on the coset g H)
template <class Fr>
__global__ void __launch_bounds__(256) qap_mul_kernel(Fr* a, const Fr* b, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fr_st(a + i, fr_ld(a + i) * fr_ld(b + i));
}
// K3, second half, on COEFFICIENTS: h[j] = q[j] * alpha - c[j] * beta   (in place over q; alpha, beta one element each)
template <class Fr>
__global__ void __launch_bounds__(256) qap_quotient_kernel(Fr* q, const Fr* c, const Fr* alpha, const Fr* beta, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fr_st(q + i, fr_ld(q + i) * fr_ld(alpha) - fr_ld(c + i) * fr_ld(beta));
}

// circom witness map, after the padding / instance rows: c[i] = a[i] * b[i]   (A z o B z on H; C is never read)
template <class Fr>
__global__ void __launch_bounds__(256) qap_prod_kernel(Fr* __restrict__ c, const Fr* __restrict__ a, const Fr* __restrict__ b, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fr_st(c + i, fr_ld(a + i) * fr_ld(b + i));
}
// circom witness map, last step, on odd-coset EVALUATIONS: h[j] = a[j] * b[j] - c[j]   (in place over a)
template <class Fr>
__global__ void __launch_bounds__(256) qap_circom_h_kernel(Fr* a, const Fr* __restrict__ b, const Fr* __restrict__ c, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    fr_st(a + i, fr_ld(a + i) * fr_ld(b + i) - fr_ld(c + i));
}

// -------------------------------------------------------------------------------------------
int32_t csr_intern_upload(Ctx* c, CoeffInterner& in, const char* who, int k, uint64_t n_rows, uint64_t n_vars, const uint64_t* row_ptr,
                          const uint32_t* col, const void* coeff, DevBuf& d_row_ptr, DevBuf& d_col, DevBuf& d_cid, uint64_t* nnz_out) {
    if (row_ptr[0] != 0) return fail(c, B2S_ERR_INVALID_ARG, "%s: row_ptr[%d][0] != 0", who, k);
    const uint64_t nnz = row_ptr[n_rows];
    *nnz_out = nnz;
    std::vector<uint32_t> cid(nnz);
    const Key32* vals = reinterpret_cast<const Key32*>(coeff);
    for (uint64_t e = 0; e < nnz; e++) {
        if (col[e] >= n_vars) return fail(c, B2S_ERR_ASSIGNMENT_MISSING, "%s: column %u >= %llu variables", who, col[e], (unsigned long long)n_vars);
        Key32 v;
        memcpy(&v, vals + e, 32);
        if (v == in.one) { cid[e] = 0; continue; }
        auto it = in.ids.find(v);
        if (it == in.ids.end()) {
            it = in.ids.emplace(v, (uint32_t)in.pool.size()).first;
            in.pool.push_back(v);
        }
        cid[e] = it->second;
    }
    for (uint64_t r = 0; r < n_rows; r++)
        if (row_ptr[r + 1] < row_ptr[r]) return fail(c, B2S_ERR_INVALID_ARG, "%s: row_ptr[%d] not monotone", who, k);
    B2S_TRY(d_row_ptr.alloc(c, (n_rows + 1) * 8));
    B2S_TRY(d_col.alloc(c, nnz * 4));
    B2S_TRY(d_cid.alloc(c, nnz * 4));
    cudaError_t ce = cudaMemcpyAsync(d_row_ptr.p, row_ptr, (n_rows + 1) * 8, cudaMemcpyHostToDevice, c->stream);
    if (ce == cudaSuccess && nnz) ce = cudaMemcpyAsync(d_col.p, col, nnz * 4, cudaMemcpyHostToDevice, c->stream);
    if (ce == cudaSuccess && nnz) ce = cudaMemcpyAsync(d_cid.p, cid.data(), nnz * 4, cudaMemcpyHostToDevice, c->stream);
    const cudaError_t se = cudaStreamSynchronize(c->stream);  // cid goes out of scope
    if (ce == cudaSuccess) ce = se;
    if (ce != cudaSuccess) return fail(c, B2S_ERR_CUDA, "%s upload of matrix %d failed: %s", who, k, cudaGetErrorString(ce));
    return B2S_OK;
}

int32_t coeff_pool_upload(Ctx* c, const CoeffInterner& in, const char* who, DevBuf& pool, uint32_t* pool_size) {
    *pool_size = (uint32_t)in.pool.size();
    B2S_TRY(pool.alloc(c, in.pool.size() * 32));
    cudaMemcpyAsync(pool.p, in.pool.data(), in.pool.size() * 32, cudaMemcpyHostToDevice, c->stream);
    if (cudaStreamSynchronize(c->stream) != cudaSuccess) return fail(c, B2S_ERR_CUDA, "%s upload failed", who);
    return B2S_OK;
}

template <class Curve>
static int32_t r1cs_upload_t(Ctx* c, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                             const uint64_t* const row_ptr[3], const uint32_t* const col[3], const void* const coeff[3],
                             b2s_r1cs** out) {
    using Fr = typename Curve::Fr;
    using FrP = typename Curve::FrP;
    const uint64_t n_vars = n_instance + n_witness;
    if (n_instance == 0) return fail(c, B2S_ERR_INVALID_ARG, "r1cs: n_instance counts the constant One and must be >= 1");
    uint64_t need = n_rows + n_instance;
    uint32_t logd = 0;
    while ((1ull << logd) < need) logd++;
    if (logd > (uint32_t)FrP::TWO_ADICITY || logd > 27)
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs: domain 2^%u unsupported", logd);
    b2s_r1cs* m = new b2s_r1cs();
    m->n_rows = n_rows; m->n_instance = n_instance; m->n_witness = n_witness; m->log_domain = logd;
    CoeffInterner in(fr_one_key<FrP>());
    int32_t st = B2S_OK;
    for (int k = 0; k < 3 && st == B2S_OK; k++)
        st = csr_intern_upload(c, in, "r1cs", k, n_rows, n_vars, row_ptr[k], col[k], coeff[k], m->row_ptr[k], m->col[k], m->coeff_id[k], &m->nnz[k]);
    if (st == B2S_OK) st = coeff_pool_upload(c, in, "r1cs", m->pool, &m->pool_size);
    if (st != B2S_OK) { delete m; return st; }
    *out = m;
    return B2S_OK;
}

int32_t r1cs_upload(Ctx* c, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness, const uint64_t* const row_ptr[3],
                    const uint32_t* const col[3], const void* const coeff[3], b2s_r1cs** out) {
    return dispatch_curve(c, [&](auto curve) {
        return r1cs_upload_t<decltype(curve)>(c, n_rows, n_instance, n_witness, row_ptr, col, coeff, out);
    });
}

// oc == nullptr: A and B only
template <class Curve>
static int32_t spmv_t(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* oa, void* ob, void* oc, uint32_t K = 1, uint64_t z_stride = 0,
                      uint64_t out_stride = 0) {
    using Fr = typename Curve::Fr;
    if (m->n_rows == 0) return B2S_OK;
    SpmvMat mm[3];
    void* outs[3] = {oa, ob, oc};
    const int nm = oc ? 3 : 2;
    for (int k = 0; k < 3; k++)
        mm[k] = k < nm ? SpmvMat{m->row_ptr[k].as<uint64_t>(), m->col[k].as<uint32_t>(), m->coeff_id[k].as<uint32_t>(), outs[k]} : SpmvMat{};
    auto* const spmv3 = spmv_kernel<Fr, 3>;
    auto* const spmv2 = spmv_kernel<Fr, 2>;
    if (nm == 3)
        B2S_LAUNCH_N(c, "spmv_kernel<Fr>", spmv3, dim3(cdiv(3 * m->n_rows, 256), K), 256, 0, mm[0], mm[1], mm[2], m->pool.as<Fr>(),
                   reinterpret_cast<const Fr*>(z_dev), m->n_rows, z_stride, out_stride);
    else
        B2S_LAUNCH_N(c, "spmv_kernel<Fr> A,B", spmv2, dim3(cdiv(2 * m->n_rows, 256), K), 256, 0, mm[0], mm[1], mm[2], m->pool.as<Fr>(),
                   reinterpret_cast<const Fr*>(z_dev), m->n_rows, z_stride, out_stride);
    return B2S_OK;
}

int32_t spmv_run(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* oa, void* ob, void* oc) {
    return dispatch_curve(c, [&](auto curve) { return spmv_t<decltype(curve)>(c, m, z_dev, oa, ob, oc); });
}

// h = coefficients of (A B - C) / Z.  ark-groth16 (SURVEY.md Appendix A.2) evaluates a, b AND c on the coset g H, forms
// (a b - c) / Z there and interpolates: 7 transforms.  Z is the constant g^N - 1 on that coset and C has degree < N, so the
// interpolation of the c term gives back C's own coefficients: h = (cosetiNTT(a_coset * b_coset) - iNTT(c)) * Zinv, exactly,
// for every assignment (satisfying or not) -- 6 transforms, the same field elements.  With the plan's full-size tables the
// scalings are merged as well: the three inverse transforms run unscaled, the 1/N goes into the coset input scaling of a and
// b (g^j / N), Zinv into the output scaling of the closing transform, and c's 1/N * Zinv into the (HBM-bound) last kernel.
// A batch of K assignments (z_dev + k * z_stride) gives h_dev + k * N with the same launches: every kernel takes the
// assignment from blockIdx.y, and the pointwise ones simply run over K * N elements.
template <class Curve>
static int32_t witness_map_t(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* h_dev, uint32_t K, uint64_t z_stride) {
    using Fr = typename Curve::Fr;
    const uint64_t N = 1ull << m->log_domain;
    Fr* a = reinterpret_cast<Fr*>(h_dev);
    DevBuf bb, cb;
    B2S_TRY(bb.alloc(c, K * N * sizeof(Fr)));
    B2S_TRY(cb.alloc(c, K * N * sizeof(Fr)));
    Fr* b = bb.as<Fr>();
    Fr* cc = cb.as<Fr>();
    // zero the padding [n_rows, N) of every vector
    const size_t pitch = N * sizeof(Fr), pad = (N - m->n_rows) * sizeof(Fr);
    B2S_CUDA(c, cudaMemset2DAsync(a + m->n_rows, pitch, 0, pad, K, c->stream));
    B2S_CUDA(c, cudaMemset2DAsync(b + m->n_rows, pitch, 0, pad, K, c->stream));
    B2S_CUDA(c, cudaMemset2DAsync(cc + m->n_rows, pitch, 0, pad, K, c->stream));
    B2S_TRY(spmv_t<Curve>(c, m, z_dev, a, b, cc, K, z_stride, N));
    B2S_LAUNCH(c, copy_instance_kernel<Fr>, dim3(cdiv(m->n_instance, 256), K), 256, 0, a, reinterpret_cast<const Fr*>(z_dev),
               m->n_rows, m->n_instance, z_stride, N);
    NttPlan* pl = nullptr;
    B2S_TRY(ntt_get_full(c, m->log_domain, &pl));
    const uint32_t wm = pl ? NTT_M_WM : 0u;
    if (!pl) B2S_TRY(ntt_get_plan(c, m->log_domain, &pl));
    Fr* bufs[3] = {a, b, cc};
    for (Fr* v : bufs) B2S_TRY(ntt_run_mode(c, v, m->log_domain, NTT_M_INVERSE | wm, K));
    B2S_TRY(ntt_run_mode(c, a, m->log_domain, NTT_M_COSET | wm, K));
    B2S_TRY(ntt_run_mode(c, b, m->log_domain, NTT_M_COSET | wm, K));
    B2S_LAUNCH(c, qap_mul_kernel<Fr>, cdiv(K * N, 256), 256, 0, a, (const Fr*)b, K * N);
    B2S_TRY(ntt_run_mode(c, a, m->log_domain, NTT_M_INVERSE | NTT_M_COSET | wm, K));
    // composed scalings: q and c both still lack Zinv;  merged: q is finished, c lacks Zinv / N
    const Fr* alpha = reinterpret_cast<const Fr*>(wm ? pl->one : pl->zinv);
    const Fr* beta = reinterpret_cast<const Fr*>(wm ? pl->full->wm_beta : pl->zinv);
    B2S_LAUNCH(c, qap_quotient_kernel<Fr>, cdiv(K * N, 256), 256, 0, a, (const Fr*)cc, alpha, beta, K * N);
    return B2S_OK;
}

// h = ark-circom CircomReduction::witness_map: the N evaluations of A B - C' on the odd coset w2 H (w2 a primitive 2N-th root,
// w2^2 = w), where C' interpolates (A z) o (B z) on H.  C is never read, and nothing is divided by Z (it is the constant
// w2^N - 1 = -2 there; the circom h query, the odd-indexed Lagrange basis of the size-2N domain, absorbs it).  a and b are
// A z and B z with the instance rows in a, c = a o b pointwise on H, then each of a, b, c goes to the odd coset by an
// unscaled inverse transform and a forward transform whose input scaling is w2^j / N: six transforms, none of them a closing
// inverse.  The batch layout is that of witness_map_t.
template <class Curve>
static int32_t witness_map_circom_t(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* h_dev, uint32_t K, uint64_t z_stride) {
    using Fr = typename Curve::Fr;
    const uint64_t N = 1ull << m->log_domain;
    Fr* a = reinterpret_cast<Fr*>(h_dev);
    DevBuf bb, cb;
    B2S_TRY(bb.alloc(c, K * N * sizeof(Fr)));
    B2S_TRY(cb.alloc(c, K * N * sizeof(Fr)));
    Fr* b = bb.as<Fr>();
    Fr* cc = cb.as<Fr>();
    const size_t pitch = N * sizeof(Fr), pad = (N - m->n_rows) * sizeof(Fr);
    B2S_CUDA(c, cudaMemset2DAsync(a + m->n_rows, pitch, 0, pad, K, c->stream));
    B2S_CUDA(c, cudaMemset2DAsync(b + m->n_rows, pitch, 0, pad, K, c->stream));
    B2S_TRY(spmv_t<Curve>(c, m, z_dev, a, b, nullptr, K, z_stride, N));
    B2S_LAUNCH(c, copy_instance_kernel<Fr>, dim3(cdiv(m->n_instance, 256), K), 256, 0, a, reinterpret_cast<const Fr*>(z_dev),
               m->n_rows, m->n_instance, z_stride, N);
    B2S_LAUNCH(c, qap_prod_kernel<Fr>, cdiv(K * N, 256), 256, 0, cc, (const Fr*)a, (const Fr*)b, K * N);
    Fr* bufs[3] = {a, b, cc};
    for (Fr* v : bufs) B2S_TRY(ntt_run_mode(c, v, m->log_domain, NTT_M_INVERSE | NTT_M_ODD, K));
    for (Fr* v : bufs) B2S_TRY(ntt_run_mode(c, v, m->log_domain, NTT_M_ODD, K));
    B2S_LAUNCH(c, qap_circom_h_kernel<Fr>, cdiv(K * N, 256), 256, 0, a, (const Fr*)b, (const Fr*)cc, K * N);
    return B2S_OK;
}

int32_t witness_map_run(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* h_dev, int32_t qap, uint32_t K, uint64_t z_stride) {
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        return qap == B2S_QAP_CIRCOM ? witness_map_circom_t<C>(c, m, z_dev, h_dev, K, z_stride)
                                     : witness_map_t<C>(c, m, z_dev, h_dev, K, z_stride);
    });
}

}  // namespace b2s
