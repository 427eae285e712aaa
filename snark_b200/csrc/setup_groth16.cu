// Groth16 key generation on the GPU (SURVEY.md 8(f) row 2): `CircuitSpecificSetupSNARK::setup` /
// `SNARK::circuit_specific_setup` (/root/reference/snark/src/lib.rs:43-46, 84-93) for the R1CS matrices
// exported by `to_matrices()`; algebra of ark-groth16's generator with the LibsnarkReduction instance map
// (upstream crate, not in /root/reference; SURVEY.md Appendix A.5).  The trapdoor (tau, alpha, beta, gamma,
// delta) is drawn by the caller from its rng, as upstream does, and passed in.
//
//   u_i    = L_i(tau) = Z(tau) w^i / (N (tau - w^i))                     one thread per row of the domain
//   A_j(tau) = sum_i u_i A[i][j] (+ u_{n+j} for instance j), B_j, C_j     column sums: the CSR matrices are
//            counting-sorted by column on the device; a column of s entries is cut into ceil(s / 4096) tasks
//            so that the one-variable-in-every-row columns of synthetic circuits do not serialise
//   a_query[j] = A_j(tau) G1, b_g1/g2_query[j] = B_j(tau) G1/G2, h_query[i] = tau^i Z(tau)/delta G1,
//   l_query[j] = (beta A_j + alpha B_j + C_j)/delta G1 (witness j), gamma_abc_g1[j] = (...)/gamma G1 (instance j)
//            all through the fixed-base kernel (setup.cu)
// Under ark-circom's CircomReduction (snarkjs keys) only the h query differs: h_query[j] = L^(2N)_{2j+1}(tau)/delta G1, j < N,
// the odd-indexed Lagrange basis of the size-2N domain at tau (w2 = primitive 2N-th root):
//   L^(2N)_{2j+1}(tau) = (tau^2N - 1) w2^(2j+1) / (2N (tau - w2^(2j+1)))
#define B2S_INLINE_MUL 1   // Fr only
#include <cassert>

#include "r1cs.cuh"

namespace b2s {

static constexpr uint32_t COL_TASK = 4096;

template <class Fr>
struct SetupConsts { Fr tau, alpha, beta, gamma, delta, w, zt_over_n, zt_dinv, dinv, ginv; };

template <class Fr>
__global__ void lagrange_kernel(SetupConsts<Fr> k, uint64_t N, Fr* __restrict__ u) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N) return;
    const Fr wi = k.w.pow_u64(i);
    u[i] = k.zt_over_n * wi * (k.tau - wi).inverse();
}

__global__ void col_count_kernel(const uint32_t* __restrict__ col, uint64_t nnz, uint32_t* __restrict__ counts) {
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nnz) return;
    const unsigned active = __activemask();
    const uint32_t key = col[e];
    const unsigned peers = __match_any_sync(active, key);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&counts[key], (uint32_t)__popc(peers));
}

// one thread per row: scatter its entries (row, coefficient id) to their column segments
__global__ void col_scatter_kernel(const uint64_t* __restrict__ row_ptr, const uint32_t* __restrict__ col, const uint32_t* __restrict__ cid,
                                   uint64_t n_rows, const uint32_t* __restrict__ offsets, uint32_t* __restrict__ cursor,
                                   uint32_t* __restrict__ t_row, uint32_t* __restrict__ t_cid) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_rows) return;
    for (uint64_t e = row_ptr[r]; e < row_ptr[r + 1]; e++) {
        const uint32_t j = col[e];
        const uint32_t pos = offsets[j] + atomicAdd(&cursor[j], 1u);
        t_row[pos] = (uint32_t)r;
        t_cid[pos] = cid[e];
    }
}

// task t of column j: partial[t] = sum over <= COL_TASK entries of u[row] * coeff
template <class Fr>
__global__ void col_partial_kernel(const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ task_off, uint32_t n_vars,
                                   const uint32_t* __restrict__ t_row, const uint32_t* __restrict__ t_cid, const Fr* __restrict__ pool,
                                   const Fr* __restrict__ u, Fr* __restrict__ partial) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= task_off[n_vars]) return;
    uint32_t lo = 0, hi = n_vars;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (task_off[mid] <= t) lo = mid; else hi = mid;
    }
    const uint32_t beg = offsets[lo] + (t - task_off[lo]) * COL_TASK;
    const uint32_t end = min(beg + COL_TASK, offsets[lo + 1]);
    Fr acc = Fr::zero();
    for (uint32_t e = beg; e < end; e++) {
        Fr v = u[t_row[e]];
        const uint32_t c = t_cid[e];
        if (c != 0) v = v * pool[c];
        acc = acc + v;
    }
    partial[t] = acc;
}

template <class Fr>
__global__ void col_sum_kernel(const uint32_t* __restrict__ task_off, uint32_t n_vars, const Fr* __restrict__ partial, Fr* __restrict__ out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_vars) return;
    Fr acc = Fr::zero();
    for (uint32_t t = task_off[j]; t < task_off[j + 1]; t++) acc = acc + partial[t];
    out[j] = acc;
}

// per-variable query scalars from A_j, B_j, C_j (a is updated in place with the input-consistency rows)
template <class Fr>
__global__ void query_scalars_kernel(SetupConsts<Fr> k, uint64_t n_rows, uint64_t n_inst, uint64_t n_vars, const Fr* __restrict__ u,
                                     Fr* __restrict__ a, const Fr* __restrict__ b, const Fr* __restrict__ c, Fr* __restrict__ lq,
                                     Fr* __restrict__ abc) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_vars) return;
    Fr aj = a[j];
    if (j < n_inst) { aj = aj + u[n_rows + j]; a[j] = aj; }
    const Fr v = k.beta * aj + k.alpha * b[j] + c[j];
    if (j < n_inst) abc[j] = v * k.ginv;
    else lq[j - n_inst] = v * k.dinv;
}

template <class Fr>
__global__ void h_scalars_kernel(SetupConsts<Fr> k, uint64_t count, Fr* __restrict__ hq) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    hq[i] = k.zt_dinv * k.tau.pow_u64(i);
}

// circom h query scalars, one thread per j < N: scale * x / (tau - x), x = w2^(2j+1), scale = (tau^2N - 1) / (2N delta)
template <class Fr>
__global__ void h_scalars_circom_kernel(Fr tau, Fr w2, Fr scale, uint64_t N, Fr* __restrict__ hq) {
    const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= N) return;
    const Fr x = w2.pow_u64(2 * j + 1);
    hq[j] = scale * x * (tau - x).inverse();
}

template <class Curve>
static int32_t setup_t(Ctx* c, const b2s_r1cs* m, const void* trapdoor_host, int32_t qap, b2s_pk** out_pk, void* o_alpha_g1, void* o_beta_g2,
                       void* o_gamma_g2, void* o_delta_g2, void* o_gamma_abc) {
    using Fr = typename Curve::Fr;
    using FrP = typename Curve::FrP;
    const uint64_t N = 1ull << m->log_domain, n_rows = m->n_rows, ell = m->n_instance, mw = m->n_witness, n_vars = ell + mw;
    if (n_vars >= (1ull << 32) || m->nnz[0] >= (1ull << 32) || m->nnz[1] >= (1ull << 32) || m->nnz[2] >= (1ull << 32))
        return fail(c, B2S_ERR_INVALID_ARG, "setup: more than 2^32 variables or nonzeros");
    // host: a handful of field operations on the trapdoor (constants of the kernels)
    SetupConsts<Fr> k;
    HostWipe wipe_k{&k, sizeof(k)};   // the trapdoor copy on this stack frame does not outlive the call
    const Fr* td = reinterpret_cast<const Fr*>(trapdoor_host);
    k.tau = td[0]; k.alpha = td[1]; k.beta = td[2]; k.gamma = td[3]; k.delta = td[4];
    if (k.gamma.is_zero() || k.delta.is_zero()) return fail(c, B2S_ERR_DIVISION_BY_ZERO, "setup: gamma or delta is zero");
    Fr w;
    for (int i = 0; i < Fr::N; i++) w.v[i] = FrP::root(i);
    for (uint32_t i = m->log_domain; i < (uint32_t)FrP::TWO_ADICITY; i++) w = w.sqr();
    k.w = w;
    const Fr zt = k.tau.pow_u64(N) - Fr::one();
    if (zt.is_zero()) return fail(c, B2S_ERR_DIVISION_BY_ZERO, "setup: tau lies in the evaluation domain");
    Fr half, n_inv = Fr::one();
    for (int i = 0; i < Fr::N; i++) half.v[i] = FrP::half(i);
    for (uint32_t i = 0; i < m->log_domain; i++) n_inv = n_inv * half;
    k.dinv = k.delta.inverse(); k.ginv = k.gamma.inverse();
    k.zt_over_n = zt * n_inv; k.zt_dinv = zt * k.dinv;
    // circom: w2 (w2^2 = w; domains stop at 2^27 below both two-adicities) and (tau^2N - 1) / (2N delta)
    Fr w2, circom_scale;
    HostWipe wipe_cs{&circom_scale, sizeof(circom_scale)};
    if (qap == B2S_QAP_CIRCOM) {
        assert(m->log_domain < (uint32_t)FrP::TWO_ADICITY);
        for (int i = 0; i < Fr::N; i++) w2.v[i] = FrP::root(i);
        for (uint32_t i = m->log_domain + 1; i < (uint32_t)FrP::TWO_ADICITY; i++) w2 = w2.sqr();
        const Fr zt2 = (zt + Fr::one()).sqr() - Fr::one();   // tau^2N - 1
        if (zt2.is_zero()) return fail(c, B2S_ERR_DIVISION_BY_ZERO, "setup: tau^(2N) = 1 (circom h query)");
        circom_scale = zt2 * n_inv * half * k.dinv;
    }

    DevBuf u, abc3, lq, gabc, hq;
    u.secret = abc3.secret = lq.secret = gabc.secret = hq.secret = true;   // powers of tau, delta^-1, ...
    B2S_TRY(u.alloc(c, N * sizeof(Fr)));
    B2S_LAUNCH(c, lagrange_kernel<Fr>, cdiv(N, 128), 128, 0, k, N, u.as<Fr>());
    B2S_TRY(abc3.alloc(c, 3 * n_vars * sizeof(Fr)));
    for (int mat = 0; mat < 3; mat++) {
        const uint64_t nnz = m->nnz[mat];
        Fr* out = abc3.as<Fr>() + mat * n_vars;
        DevBuf ints, trow, tcid, partial;
        B2S_TRY(ints.alloc(c, (4 * n_vars + 2) * sizeof(uint32_t)));
        uint32_t* counts = ints.as<uint32_t>();
        uint32_t* cursor = counts + n_vars;
        uint32_t* offsets = cursor + n_vars;
        uint32_t* task_off = offsets + n_vars + 1;
        B2S_CUDA(c, cudaMemsetAsync(counts, 0, 2 * n_vars * sizeof(uint32_t), c->stream));
        if (nnz) B2S_LAUNCH(c, col_count_kernel, cdiv(nnz, 256), 256, 0, m->col[mat].as<uint32_t>(), nnz, counts);
        B2S_TRY(scan_counts(c, counts, (uint32_t)n_vars, COL_TASK, offsets, task_off));
        B2S_TRY(trow.alloc(c, nnz * 4));
        B2S_TRY(tcid.alloc(c, nnz * 4));
        if (n_rows) B2S_LAUNCH(c, col_scatter_kernel, cdiv(n_rows, 256), 256, 0, m->row_ptr[mat].as<uint64_t>(), m->col[mat].as<uint32_t>(),
                               m->coeff_id[mat].as<uint32_t>(), n_rows, offsets, cursor, trow.as<uint32_t>(), tcid.as<uint32_t>());
        const uint64_t max_tasks = nnz / COL_TASK + n_vars + 1;
        B2S_TRY(partial.alloc(c, max_tasks * sizeof(Fr)));
        B2S_LAUNCH(c, col_partial_kernel<Fr>, cdiv(max_tasks, 128), 128, 0, offsets, task_off, (uint32_t)n_vars, trow.as<uint32_t>(),
                   tcid.as<uint32_t>(), m->pool.as<Fr>(), u.as<Fr>(), partial.as<Fr>());
        B2S_LAUNCH(c, col_sum_kernel<Fr>, cdiv(n_vars, 128), 128, 0, task_off, (uint32_t)n_vars, partial.as<Fr>(), out);
    }
    Fr* a = abc3.as<Fr>();
    Fr* b = a + n_vars;
    Fr* cc = b + n_vars;
    B2S_TRY(lq.alloc(c, (mw + 1) * sizeof(Fr)));
    B2S_TRY(gabc.alloc(c, ell * sizeof(Fr)));
    B2S_TRY(hq.alloc(c, N * sizeof(Fr)));
    B2S_LAUNCH(c, query_scalars_kernel<Fr>, cdiv(n_vars, 128), 128, 0, k, n_rows, ell, n_vars, u.as<Fr>(), a, b, cc, lq.as<Fr>(), gabc.as<Fr>());
    const uint64_t h_len = pk_full_h_len(qap, N);
    if (qap == B2S_QAP_CIRCOM) B2S_LAUNCH(c, h_scalars_circom_kernel<Fr>, cdiv(N, 128), 128, 0, k.tau, w2, circom_scale, N, hq.as<Fr>());
    else B2S_LAUNCH(c, h_scalars_kernel<Fr>, cdiv(N - 1, 128), 128, 0, k, N - 1, hq.as<Fr>());
    // group part
    const size_t g1 = sizeof(typename Curve::G1Affine), g2 = sizeof(typename Curve::G2Affine);
    DevBuf qa, qb1, qb2, qh, ql, qabc, k1, k2, ks;
    ks.secret = true;
    B2S_TRY(qa.alloc(c, n_vars * g1)); B2S_TRY(qb1.alloc(c, n_vars * g1)); B2S_TRY(qb2.alloc(c, n_vars * g2));
    B2S_TRY(qh.alloc(c, N * g1)); B2S_TRY(ql.alloc(c, (mw + 1) * g1)); B2S_TRY(qabc.alloc(c, ell * g1));
    B2S_TRY(fixed_base_run(c, 1, a, n_vars, true, qa.p));
    B2S_TRY(fixed_base_run(c, 1, b, n_vars, true, qb1.p));
    B2S_TRY(fixed_base_run(c, 2, b, n_vars, true, qb2.p));
    B2S_TRY(fixed_base_run(c, 1, hq.p, h_len, true, qh.p));
    B2S_TRY(fixed_base_run(c, 1, lq.p, mw, true, ql.p));
    B2S_TRY(fixed_base_run(c, 1, gabc.p, ell, true, qabc.p));
    // constants: G1 [alpha, beta, delta], G2 [beta, gamma, delta]
    B2S_TRY(ks.alloc(c, 6 * sizeof(Fr)));
    const Fr s1[3] = {k.alpha, k.beta, k.delta}, s2[3] = {k.beta, k.gamma, k.delta};
    B2S_CUDA(c, cudaMemcpyAsync(ks.p, s1, sizeof(s1), cudaMemcpyHostToDevice, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(ks.as<Fr>() + 3, s2, sizeof(s2), cudaMemcpyHostToDevice, c->stream));
    B2S_TRY(k1.alloc(c, 3 * g1)); B2S_TRY(k2.alloc(c, 3 * g2));
    B2S_TRY(fixed_base_run(c, 1, ks.p, 3, true, k1.p));
    B2S_TRY(fixed_base_run(c, 2, ks.as<Fr>() + 3, 3, true, k2.p));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));   // s1/s2 live on this stack frame
    // verifying key elements to the host
    char* p1 = k1.as<char>();
    char* p2 = k2.as<char>();
    B2S_CUDA(c, cudaMemcpyAsync(o_alpha_g1, p1, g1, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(o_beta_g2, p2, g2, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(o_gamma_g2, p2 + g2, g2, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(o_delta_g2, p2 + 2 * g2, g2, cudaMemcpyDeviceToHost, c->stream));
    if (ell) B2S_CUDA(c, cudaMemcpyAsync(o_gamma_abc, qabc.p, ell * g1, cudaMemcpyDeviceToHost, c->stream));
    // proving key handle (device-to-device copies inside pk_upload add the delta pairs of the prover)
    b2s_pk_desc d{};
    d.n_instance = ell; d.n_witness = mw; d.domain_size = N;
    d.alpha_g1 = p1; d.beta_g1 = p1 + g1; d.delta_g1 = p1 + 2 * g1; d.beta_g2 = p2; d.delta_g2 = p2 + 2 * g2;
    d.a_query = qa.p; d.a_len = n_vars; d.b_g1_query = qb1.p; d.b1_len = n_vars; d.b_g2_query = qb2.p; d.b2_len = n_vars;
    d.h_query = qh.p; d.h_len = h_len; d.l_query = ql.p; d.l_len = mw;
    return pk_upload(c, &d, B2S_MEM_DEVICE, qap, out_pk);
}

int32_t groth16_setup(Ctx* c, const b2s_r1cs* m, const void* trapdoor_host, int32_t qap, b2s_pk** out_pk, void* o_alpha_g1, void* o_beta_g2,
                      void* o_gamma_g2, void* o_delta_g2, void* o_gamma_abc) {
    return dispatch_curve(c, [&](auto curve) {
        return setup_t<decltype(curve)>(c, m, trapdoor_host, qap, out_pk, o_alpha_g1, o_beta_g2, o_gamma_g2, o_delta_g2, o_gamma_abc);
    });
}

// copy one query vector of a device-resident key to the host (which: 0 a, 1 b_g1, 2 b_g2, 3 h, 4 l, 5 [alpha,beta,delta]_g1, 6 [beta,delta]_g2)
int32_t pk_query_download(Ctx* c, const b2s_pk* pk, int which, void* out_host, uint64_t cap_bytes) {
    const Sizes z = sizes(c);
    const DevBuf* src = nullptr;
    size_t bytes = 0;
    if (which >= 0 && which < PK_QUERIES) { src = &pk->q[which].pts; bytes = pk->q[which].len * z.aff(PK_QUERY[which].group); }
    else if (which == 5) { src = &pk->consts_g1; bytes = 3 * z.g1; }
    else if (which == 6) { src = &pk->consts_g2; bytes = 2 * z.g2; }
    else return fail(c, B2S_ERR_INVALID_ARG, "pk_query: unknown vector %d", which);
    if (bytes > cap_bytes) return fail(c, B2S_ERR_INVALID_ARG, "pk_query: buffer too small (%zu > %llu)", bytes, (unsigned long long)cap_bytes);
    if (bytes) B2S_CUDA(c, cudaMemcpyAsync(out_host, src->p, bytes, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

}  // namespace b2s
