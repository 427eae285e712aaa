// Element-wise polynomial kernels of the universal-setup (Marlin-style) path, SURVEY.md 8(f) row 4 / BASELINE config 5.
//
// The reference tree only declares the interface of such a scheme (trait UniversalSetupSNARK,
// /root/reference/snark/src/lib.rs:107-133); the implementations (ark-marlin over ark-poly's `Evaluations` / `DensePolynomial`
// arithmetic and ark-poly-commit's KZG10) are out of tree.  What those crates do between their FFTs and MSMs is element-wise
// work over vectors of |H| ... 4|K| field elements: products and sums of evaluation vectors, batched inversion
// (ark-ff `batch_inversion`), geometric sequences (domain elements, coset points), Horner evaluation.  These kernels are that
// layer; the transforms and commitments go through b2s_ntt / b2s_msm_g1 / b2s_fixed_base_g1, the matrix products through
// b2s_spmv.  All HBM-bound streaming kernels (32 B per element per operand) except the batched inversion (3 multiplications
// per element and one divsteps inversion per 16 elements) and the geometric sequence (~7 per element).
#define B2S_INLINE_MUL 1   // Fr only in this unit
#include "common.cuh"

namespace b2s {

namespace {

template <class Fr>
__device__ __forceinline__ Fr pld(const Fr* p) {
    static_assert(Fr::N == 8, "scalar fields are 8 x 32-bit limbs");
    const uint4* q = reinterpret_cast<const uint4*>(p);
    uint4 a = q[0], b = q[1];
    Fr r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}
template <class Fr>
__device__ __forceinline__ void pst(Fr* p, const Fr& r) {
    uint4* q = reinterpret_cast<uint4*>(p);
    q[0] = make_uint4(r.v[0], r.v[1], r.v[2], r.v[3]);
    q[1] = make_uint4(r.v[4], r.v[5], r.v[6], r.v[7]);
}

// op: 0 a*b  1 a+b  2 a-b  3 a*s  4 a+s
template <class Fr>
__global__ void __launch_bounds__(256) poly_op_kernel(int op, const Fr* __restrict__ a, const Fr* __restrict__ b, Fr s, Fr* __restrict__ out, uint64_t n) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const Fr x = pld(a + i);
    Fr r;
    switch (op) {
        case 0: r = x * pld(b + i); break;
        case 1: r = x + pld(b + i); break;
        case 2: r = x - pld(b + i); break;
        case 3: r = x * s; break;
        default: r = x + s; break;
    }
    pst(out + i, r);
}

// out[i] = 1 / a[i], and 0 where a[i] = 0 (ark-ff batch_inversion semantics): Montgomery's trick over runs of INV_RUN
// elements per thread, zeros left out of the running product.
static constexpr int INV_RUN = 16;
template <class Fr>
__global__ void __launch_bounds__(128) poly_inv0_kernel(const Fr* __restrict__ a, Fr* __restrict__ out, uint64_t n) {
    const uint64_t base = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * INV_RUN;
    if (base >= n) return;
    const int cnt = (int)min((uint64_t)INV_RUN, n - base);
    Fr acc = Fr::one();
    // first sweep: prefix products into `out` (the product of the non-zero elements BEFORE position j)
    for (int j = 0; j < cnt; j++) {
        const Fr v = pld(a + base + j);
        pst(out + base + j, acc);
        if (!v.is_zero()) acc = acc * v;
    }
    Fr inv = acc.inverse();
    for (int j = cnt - 1; j >= 0; j--) {
        const Fr v = pld(a + base + j);
        if (v.is_zero()) {
            pst(out + base + j, Fr::zero());
        } else {
            const Fr pre = pld(out + base + j);
            pst(out + base + j, inv * pre);
            inv = inv * v;
        }
    }
}

// out[i] = c * s^i : a run of GEOM_RUN elements per thread, its first element by square-and-multiply
static constexpr int GEOM_RUN = 16;
template <class Fr>
__global__ void __launch_bounds__(128) poly_geom_kernel(Fr c, Fr s, Fr* __restrict__ out, uint64_t n) {
    const uint64_t base = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * GEOM_RUN;
    if (base >= n) return;
    const int cnt = (int)min((uint64_t)GEOM_RUN, n - base);
    Fr t = c * s.pow_u64(base);
    for (int j = 0; j < cnt; j++) {
        pst(out + base + j, t);
        t = t * s;
    }
}

// partial[block] = sum over the block's coefficients of c_i z^i : Horner over a run per thread, z^(run start) by
// square-and-multiply, shared-memory tree.
static constexpr int EVAL_RUN = 16, EVAL_THREADS = 256;
template <class Fr>
__device__ __forceinline__ Fr block_sum(Fr v, Fr* sm) {
    sm[threadIdx.x] = v;
    __syncthreads();
    for (int d = EVAL_THREADS / 2; d > 0; d >>= 1) {
        if ((int)threadIdx.x < d) sm[threadIdx.x] = sm[threadIdx.x] + sm[threadIdx.x + d];
        __syncthreads();
    }
    return sm[0];
}
template <class Fr>
__global__ void __launch_bounds__(EVAL_THREADS) poly_eval_kernel(const Fr* __restrict__ coeffs, uint64_t n, Fr z, Fr* __restrict__ partial) {
    __shared__ Fr sm[EVAL_THREADS];
    const uint64_t base = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * EVAL_RUN;
    Fr acc = Fr::zero();
    if (base < n) {
        const int cnt = (int)min((uint64_t)EVAL_RUN, n - base);
        for (int j = cnt - 1; j >= 0; j--) acc = acc * z + pld(coeffs + base + j);
        acc = acc * z.pow_u64(base);
    }
    const Fr tot = block_sum(acc, sm);
    if (threadIdx.x == 0) pst(partial + blockIdx.x, tot);
}
template <class Fr>
__global__ void __launch_bounds__(EVAL_THREADS) poly_sum_kernel(const Fr* __restrict__ partial, uint32_t count, Fr* __restrict__ out) {
    __shared__ Fr sm[EVAL_THREADS];
    Fr acc = Fr::zero();
    for (uint32_t i = threadIdx.x; i < count; i += EVAL_THREADS) acc = acc + pld(partial + i);
    const Fr tot = block_sum(acc, sm);
    if (threadIdx.x == 0) pst(out, tot);
}

template <class Fr>
Fr host_scalar(const void* p) {
    Fr s = Fr::zero();
    if (p) memcpy(s.v, p, sizeof(s.v));
    return s;
}

}  // namespace

template <class Curve>
static int32_t poly_op_t(Ctx* c, int op, const void* a, const void* b, const void* s_host, void* out, uint64_t n, int32_t mem) {
    using Fr = typename Curve::Fr;
    if (n == 0) return B2S_OK;
    const bool two = op <= 2, scalar = op == 3 || op == 4;
    if (!a || !out || (two && !b) || (scalar && !s_host)) return fail(c, B2S_ERR_INVALID_ARG, "poly_op: null argument for op %d", op);
    InBuf A, B;
    B2S_TRY(A.bind(c, a, n * sizeof(Fr), mem));
    if (two) B2S_TRY(B.bind(c, b, n * sizeof(Fr), mem));
    OutBuf O;
    B2S_TRY(O.bind(c, out, n * sizeof(Fr), mem));
    Fr* o = O.as<Fr>();
    if (op == 5) {
        if (o == A.as<Fr>()) return fail(c, B2S_ERR_INVALID_ARG, "poly_op: the batched inversion does not run in place");
        B2S_LAUNCH(c, poly_inv0_kernel<Fr>, cdiv(cdiv(n, INV_RUN), 128), 128, 0, A.as<Fr>(), o, n);
    } else {
        B2S_LAUNCH(c, poly_op_kernel<Fr>, cdiv(n, 256), 256, 0, op, A.as<Fr>(), two ? B.as<Fr>() : A.as<Fr>(), host_scalar<Fr>(s_host), o, n);
    }
    return O.finish(c);
}

int32_t poly_op_run(Ctx* c, int op, const void* a, const void* b, const void* s_host, void* out, uint64_t n, int32_t mem) {
    if (op < 0 || op > 5) return fail(c, B2S_ERR_INVALID_ARG, "poly_op: unknown op %d", op);
    return dispatch_curve(c, [&](auto curve) { return poly_op_t<decltype(curve)>(c, op, a, b, s_host, out, n, mem); });
}

template <class Curve>
static int32_t poly_geom_t(Ctx* c, const void* c_host, const void* s_host, uint64_t n, int32_t mem, void* out) {
    using Fr = typename Curve::Fr;
    if (n == 0) return B2S_OK;
    if (!c_host || !s_host || !out) return fail(c, B2S_ERR_INVALID_ARG, "poly_geom: null argument");
    OutBuf O;
    B2S_TRY(O.bind(c, out, n * sizeof(Fr), mem));
    B2S_LAUNCH(c, poly_geom_kernel<Fr>, cdiv(cdiv(n, GEOM_RUN), 128), 128, 0, host_scalar<Fr>(c_host), host_scalar<Fr>(s_host), O.as<Fr>(), n);
    return O.finish(c);
}

int32_t poly_geom_run(Ctx* c, const void* c_host, const void* s_host, uint64_t n, int32_t mem, void* out) {
    return dispatch_curve(c, [&](auto curve) { return poly_geom_t<decltype(curve)>(c, c_host, s_host, n, mem, out); });
}

template <class Curve>
static int32_t poly_eval_t(Ctx* c, const void* coeffs, uint64_t n, const void* z_host, int32_t mem, void* out_host) {
    using Fr = typename Curve::Fr;
    if (!out_host || !z_host || (n && !coeffs)) return fail(c, B2S_ERR_INVALID_ARG, "poly_eval: null argument");
    if (n == 0) { memset(out_host, 0, sizeof(Fr)); return B2S_OK; }
    InBuf A;
    B2S_TRY(A.bind(c, coeffs, n * sizeof(Fr), mem));
    const uint32_t blocks = cdiv(cdiv(n, EVAL_RUN), EVAL_THREADS);
    DevBuf part;
    B2S_TRY(part.alloc(c, ((size_t)blocks + 1) * sizeof(Fr)));
    B2S_LAUNCH(c, poly_eval_kernel<Fr>, blocks, EVAL_THREADS, 0, A.as<Fr>(), n, host_scalar<Fr>(z_host), part.as<Fr>());
    B2S_LAUNCH(c, poly_sum_kernel<Fr>, 1, EVAL_THREADS, 0, (const Fr*)part.as<Fr>(), blocks, part.as<Fr>() + blocks);
    B2S_CUDA(c, cudaMemcpyAsync(out_host, part.as<Fr>() + blocks, sizeof(Fr), cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

int32_t poly_eval_run(Ctx* c, const void* coeffs, uint64_t n, const void* z_host, int32_t mem, void* out_host) {
    return dispatch_curve(c, [&](auto curve) { return poly_eval_t<decltype(curve)>(c, coeffs, n, z_host, mem, out_host); });
}

}  // namespace b2s
