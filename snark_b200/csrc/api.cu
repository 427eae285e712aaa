// extern "C" surface of libb200snark.so (include/b200snark.h): argument checking, host<->device
// staging and locking.  No arithmetic happens on the host here; every entry point launches the
// sm_90a kernels in the sibling translation units and fails with B2S_ERR_NO_DEVICE without a GPU.
#include <cstdlib>
#include <cstring>

#include "common.cuh"
#include "dntt.cuh"
#include "r1cs.cuh"

using namespace b2s;

struct b2s_ctx : public b2s::Ctx {};

namespace b2s {
int32_t field_op_run(Ctx* c, int field, int op, const void* a, const void* b, void* out, uint64_t count);
int32_t group_op_run(Ctx* c, int group, int op, const void* a, const void* b, const void* k, void* out, uint64_t count);
// poly.cu
int32_t poly_op_run(Ctx* c, int op, const void* a, const void* b, const void* s_host, void* out, uint64_t n, int32_t mem);
int32_t poly_geom_run(Ctx* c, const void* c_host, const void* s_host, uint64_t n, int32_t mem, void* out);
int32_t poly_eval_run(Ctx* c, const void* coeffs, uint64_t n, const void* z_host, int32_t mem, void* out_host);
int32_t fixed_base_run(Ctx* c, int group, const void* scalars_dev, uint64_t n, bool mont, void* out_dev);
void fixed_base_free(Ctx* c);
int32_t serialize_points_ex(Ctx* c, int group, const void* affine, int32_t mem, uint64_t count, bool compressed, uint8_t* out, uint64_t cap);
int32_t proof_serialize(Ctx* c, const void* a_g1, const void* b_g2, const void* c_g1, bool compressed, uint8_t* out, uint64_t cap);
uint64_t vk_serialized_size(Ctx* c, uint64_t n_gamma_abc, bool compressed);
int32_t vk_serialize(Ctx* c, const void* alpha_g1, const void* beta_g2, const void* gamma_g2, const void* delta_g2, const void* gamma_abc,
                     uint64_t n_gamma_abc, bool compressed, uint8_t* out, uint64_t cap);
uint64_t pk_serialized_size(Ctx* c, const b2s_pk* pk, uint64_t vk_len, bool compressed);
int32_t pk_serialize(Ctx* c, const b2s_pk* pk, const uint8_t* vk_bytes, uint64_t vk_len, bool compressed, uint8_t* out, uint64_t cap);
// deserialize.cu
int32_t deserialize_points(Ctx* c, int group, const uint8_t* in, uint64_t len, uint64_t count, bool compressed, bool validate, void* out_host);
int32_t proof_deserialize(Ctx* c, const uint8_t* in, uint64_t len, bool compressed, bool validate, void* a, void* b, void* cc);
int32_t vk_deserialize(Ctx* c, const uint8_t* in, uint64_t len, bool compressed, bool validate, void* alpha, void* beta, void* gamma,
                       void* delta, void* abc, uint64_t cap_abc, uint64_t* n_abc, uint64_t* consumed);
int32_t pk_deserialize(Ctx* c, const uint8_t* in, uint64_t len, bool compressed, bool validate, int32_t qap, b2s_pk** out);
// zkey.cu
int32_t zkey_read_info(Ctx* c, const uint8_t* in, uint64_t len, b2s_zkey_info* out);
int32_t zkey_load(Ctx* c, const uint8_t* in, uint64_t len, bool validate, b2s_pk** out_pk, b2s_r1cs** out_m, void* alpha_g1,
                  void* beta_g2, void* gamma_g2, void* delta_g2, void* gamma_abc, uint64_t cap_abc);
int32_t wtns_read(Ctx* c, const uint8_t* in, uint64_t len, uint64_t n_vars, int32_t mem, void* out_z);
int32_t r1cs_file_read_info(Ctx* c, const uint8_t* in, uint64_t len, b2s_r1cs_file_info* out);
int32_t r1cs_file_load(Ctx* c, const uint8_t* in, uint64_t len, b2s_r1cs** out);
// verify.cu
int32_t vk_prepare(Ctx* c, const void* alpha, const void* beta, const void* gamma, const void* delta, const void* abc, uint64_t n_abc,
                   b2s_pvk** out);
void pvk_free(b2s_pvk* pvk);
int32_t groth16_verify_batch(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const void* a, const void* b,
                             const void* cc, int32_t mem, uint8_t* ok);
int32_t pairing_batch(Ctx* c, const void* p, const void* q, uint64_t n, int32_t mem, void* out);
// verify_rlc.cu
int32_t groth16_verify_batch_rlc(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const void* a, const void* b,
                                 const void* cc, const void* rho, int32_t mem, uint8_t* ok);
// verify_bytes.cu
int32_t groth16_verify_batch_bytes(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const uint8_t* proofs,
                                   uint64_t len, bool compressed, int32_t mem, uint8_t* ok, uint8_t* reason);
int32_t groth16_verify_batch_rlc_bytes(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const uint8_t* proofs,
                                       uint64_t len, bool compressed, const void* rho, int32_t mem, uint8_t* ok, uint8_t* reason);
}  // namespace b2s

#define LOCK(ctx)                                      \
    if (!(ctx)) return B2S_ERR_INVALID_ARG;            \
    std::lock_guard<std::mutex> guard__((ctx)->mu);    \
    if (cudaSetDevice((ctx)->device) != cudaSuccess) return fail(ctx, B2S_ERR_NO_DEVICE, "cudaSetDevice(%d) failed", (ctx)->device)

extern "C" {

const char* b2s_version(void) { return "b200snark 0.1 (sm_90a)"; }

int32_t b2s_ctx_create(int32_t curve_id, int32_t device_ordinal, b2s_ctx** out) {
    if (!out) return B2S_ERR_INVALID_ARG;
    *out = nullptr;
    if (curve_id != B2S_CURVE_BLS12_381 && curve_id != B2S_CURVE_BN254 && curve_id != B2S_CURVE_BLS12_377) return B2S_ERR_INVALID_ARG;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return B2S_ERR_NO_DEVICE;
    if (device_ordinal < 0 || device_ordinal >= ndev) return B2S_ERR_NO_DEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device_ordinal) != cudaSuccess) return B2S_ERR_NO_DEVICE;
    if (prop.major != 9 || prop.minor != 0) return B2S_ERR_NO_DEVICE;  // the kernels are built for sm_90a only
    if (cudaSetDevice(device_ordinal) != cudaSuccess) return B2S_ERR_NO_DEVICE;
    b2s_ctx* c = new b2s_ctx();
    c->curve = curve_id;
    c->device = device_ordinal;
    c->sm_count = prop.multiProcessorCount;
    c->total_mem = (uint64_t)prop.totalGlobalMem;
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->aux, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_tail, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ev_done, cudaEventDisableTiming) != cudaSuccess) {
        delete c;
        return B2S_ERR_CUDA;
    }
    if (cudaMalloc(&c->aux_ring, b2s::Ctx::AUX_SLOT_BYTES * b2s::Ctx::AUX_SLOTS) != cudaSuccess) {
        delete c;
        return B2S_ERR_OOM;
    }
    // keep freed blocks in the stream-ordered pool: proofs reuse the same multi-GiB scratch every call
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device_ordinal) == cudaSuccess) {
        uint64_t thr = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    *out = c;
    return B2S_OK;
}

void b2s_ctx_destroy(b2s_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    ntt_free_plans(ctx);
    fixed_base_free(ctx);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->aux);
    cudaStreamSynchronize(ctx->side);
    if (ctx->aux_ring) cudaFree(ctx->aux_ring);
    cudaStreamDestroy(ctx->side);
    cudaEventDestroy(ctx->ev_tail);
    cudaEventDestroy(ctx->ev_done);
    cudaStreamDestroy(ctx->aux);
    cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* b2s_last_error(const b2s_ctx* ctx) { return ctx ? ctx->err.c_str() : "null ctx"; }

int32_t b2s_sizes(const b2s_ctx* ctx, uint32_t out[6]) {
    if (!ctx || !out) return B2S_ERR_INVALID_ARG;
    const Sizes z = sizes(ctx);
    out[0] = z.fr; out[1] = z.fq; out[2] = z.g1; out[3] = z.g2; out[4] = z.g1x; out[5] = z.g2x;
    return B2S_OK;
}

uint64_t b2s_launch_count(const b2s_ctx* ctx) { return ctx ? ctx->launches : 0; }

int32_t b2s_sync(b2s_ctx* ctx) {
    LOCK(ctx);
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2S_OK;
}

void* b2s_stream(b2s_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

// ---- NTT ----------------------------------------------------------------------------------------
int32_t b2s_ntt(b2s_ctx* ctx, void* data, uint32_t log_n, int32_t inverse, int32_t coset, int32_t mem) {
    LOCK(ctx);
    if (!data) return fail(ctx, B2S_ERR_INVALID_ARG, "ntt: null data");
    if (log_n > 27) return fail(ctx, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "ntt: 2^%u exceeds the backend limit 2^27", log_n);
    OutBuf d;
    B2S_TRY(d.bind(ctx, data, (size_t)32 << log_n, mem, true));
    B2S_TRY(ntt_run(ctx, d.dptr, log_n, inverse != 0, coset != 0));
    return d.finish(ctx);
}

// ---- MSM ----------------------------------------------------------------------------------------
static int32_t msm_common(b2s_ctx* ctx, int group, const void* bases, const void* scalars, uint64_t n, int32_t mont,
                          int32_t mem, void* out, bool affine) {
    if ((!bases || !scalars) && n) return fail(ctx, B2S_ERR_INVALID_ARG, "msm: null input");
    if (!out) return fail(ctx, B2S_ERR_INVALID_ARG, "msm: null output");
    const Sizes z = sizes(ctx);
    const size_t pt = z.aff(group), xyzz = z.xyzz(group);
    InBuf b, s;
    B2S_TRY(b.bind(ctx, bases, n * pt, mem));
    B2S_TRY(s.bind(ctx, scalars, n * 32, mem));
    OutBuf o;   // the result goes to the host whatever `mem` says
    DevBuf res;
    B2S_TRY(o.bind(ctx, out, affine ? pt : xyzz, B2S_MEM_HOST));
    if (affine) B2S_TRY(res.alloc(ctx, xyzz));
    B2S_TRY(msm_run(ctx, group, b.dptr, s.dptr, n, mont != 0, affine ? res.p : o.dptr));
    if (affine) B2S_TRY(group_sum_to_affine(ctx, group, res.p, 1, o.dptr));
    return o.finish(ctx);
}

int32_t b2s_msm_g1(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont, int32_t mem,
                   void* out_affine) {
    LOCK(ctx);
    return msm_common(ctx, 1, bases, scalars, n, scalars_mont, mem, out_affine, true);
}
int32_t b2s_msm_g2(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont, int32_t mem,
                   void* out_affine) {
    LOCK(ctx);
    return msm_common(ctx, 2, bases, scalars, n, scalars_mont, mem, out_affine, true);
}
int32_t b2s_msm_g1_partial(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont,
                           int32_t mem, void* out_xyzz) {
    LOCK(ctx);
    return msm_common(ctx, 1, bases, scalars, n, scalars_mont, mem, out_xyzz, false);
}
int32_t b2s_msm_g2_partial(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont,
                           int32_t mem, void* out_xyzz) {
    LOCK(ctx);
    return msm_common(ctx, 2, bases, scalars, n, scalars_mont, mem, out_xyzz, false);
}

static int32_t sum_common(b2s_ctx* ctx, int group, const void* xyzz, uint32_t count, void* out_affine) {
    if (!xyzz || !out_affine || count == 0) return fail(ctx, B2S_ERR_INVALID_ARG, "group sum: bad arguments");
    const Sizes z = sizes(ctx);
    InBuf in;
    OutBuf aff;
    B2S_TRY(in.bind(ctx, xyzz, (size_t)count * z.xyzz(group), B2S_MEM_HOST));
    B2S_TRY(aff.bind(ctx, out_affine, z.aff(group), B2S_MEM_HOST));
    B2S_TRY(group_sum_to_affine(ctx, group, in.dptr, count, aff.dptr));
    return aff.finish(ctx);
}
int32_t b2s_g1_sum(b2s_ctx* ctx, const void* xyzz, uint32_t count, void* out_affine) {
    LOCK(ctx);
    return sum_common(ctx, 1, xyzz, count, out_affine);
}
int32_t b2s_g2_sum(b2s_ctx* ctx, const void* xyzz, uint32_t count, void* out_affine) {
    LOCK(ctx);
    return sum_common(ctx, 2, xyzz, count, out_affine);
}

// ---- element-wise polynomial kernels (universal-setup path) ----------------------------------------
int32_t b2s_poly_op(b2s_ctx* ctx, int32_t op, const void* a, const void* b, const void* s, void* out, uint64_t n, int32_t mem) {
    LOCK(ctx);
    return poly_op_run(ctx, op, a, b, s, out, n, mem);
}
int32_t b2s_poly_geom(b2s_ctx* ctx, const void* c, const void* s, uint64_t n, int32_t mem, void* out) {
    LOCK(ctx);
    return poly_geom_run(ctx, c, s, n, mem, out);
}
int32_t b2s_poly_eval(b2s_ctx* ctx, const void* coeffs, uint64_t n, const void* z, int32_t mem, void* out) {
    LOCK(ctx);
    return poly_eval_run(ctx, coeffs, n, z, mem, out);
}

// ---- element-wise test kernels ------------------------------------------------------------------
int32_t b2s_field_op(b2s_ctx* ctx, int32_t field, int32_t op, const void* a, const void* b, void* out, uint64_t count) {
    LOCK(ctx);
    if (!a || !b || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "field_op: null buffer");
    return field_op_run(ctx, field, op, a, b, out, count);
}
int32_t b2s_group_op(b2s_ctx* ctx, int32_t group, int32_t op, const void* a, const void* b, const void* k, void* out,
                     uint64_t count) {
    LOCK(ctx);
    if (!a || !b || !k || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "group_op: null buffer");
    if (group != 1 && group != 2) return fail(ctx, B2S_ERR_INVALID_ARG, "group_op: group must be 1 or 2");
    return group_op_run(ctx, group, op, a, b, k, out, count);
}

// ---- fixed-base batch multiplication -----------------------------------------------------------
static int32_t fixed_base_common(b2s_ctx* ctx, int group, const void* scalars, uint64_t n, int32_t mont, int32_t mem, void* out) {
    if ((!scalars || !out) && n) return fail(ctx, B2S_ERR_INVALID_ARG, "fixed_base: null buffer");
    const size_t pt = sizes(ctx).aff(group);
    InBuf s;
    OutBuf o;
    B2S_TRY(s.bind(ctx, scalars, n * 32, mem));
    B2S_TRY(o.bind(ctx, out, n * pt, mem));
    B2S_TRY(fixed_base_run(ctx, group, s.dptr, n, mont != 0, o.dptr));
    return o.finish(ctx);
}
int32_t b2s_fixed_base_g1(b2s_ctx* ctx, const void* scalars, uint64_t n, int32_t scalars_mont, int32_t mem, void* out) {
    LOCK(ctx);
    return fixed_base_common(ctx, 1, scalars, n, scalars_mont, mem, out);
}
int32_t b2s_fixed_base_g2(b2s_ctx* ctx, const void* scalars, uint64_t n, int32_t scalars_mont, int32_t mem, void* out) {
    LOCK(ctx);
    return fixed_base_common(ctx, 2, scalars, n, scalars_mont, mem, out);
}

}  // extern "C"

// ---- R1CS / witness map / Groth16 --------------------------------------------------------------
// The prove entry points take z as two host pieces (z_dev == nullptr) or as one device array.
static bool z_missing(const b2s_r1cs* m, const void* z_inst, const void* z_wit, const void* z_dev) {
    return !z_dev && (!z_inst || (!z_wit && m->n_witness));
}

// the `qap` argument of the *_qap entry points
static int32_t check_qap(b2s_ctx* ctx, int32_t qap, const char* who) {
    if (qap != B2S_QAP_LIBSNARK && qap != B2S_QAP_CIRCOM)
        return fail(ctx, B2S_ERR_INVALID_ARG, "%s: unknown QAP reduction %d (B2S_QAP_LIBSNARK = 0, B2S_QAP_CIRCOM = 1)", who, (int)qap);
    return B2S_OK;
}

// one proof on one GPU with a full key
static int32_t prove_full(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_inst, const void* z_wit, const void* z_dev,
                          const void* r, const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    if (!pk || !m) return fail(ctx, B2S_ERR_MISSING_CS, "prove: null key or matrices");
    if (z_missing(m, z_inst, z_wit, z_dev) || !r || !s) return fail(ctx, B2S_ERR_ASSIGNMENT_MISSING, "prove: null assignment");
    if (!out_a_g1 || !out_b_g2 || !out_c_g1) return fail(ctx, B2S_ERR_INVALID_ARG, "prove: null output");
    if (!pk_is_full(pk)) return fail(ctx, B2S_ERR_MALFORMED_VK, "prove: needs a full (unsharded) proving key");
    const Sizes z = sizes(ctx);
    DevBuf g1, g2;
    B2S_TRY(g1.alloc(ctx, 4 * z.g1x));
    B2S_TRY(g2.alloc(ctx, z.g2x));
    B2S_TRY(groth16_shard(ctx, pk, m, z_inst, z_wit, z_dev, r, s, g1.p, g2.p));
    return groth16_finish(ctx, pk, g1.p, g2.p, 1, r, s, out_a_g1, out_b_g2, out_c_g1);
}

// one shard's partial sums, to the host
static int32_t prove_partial(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_inst, const void* z_wit, const void* z_dev,
                             const void* r, const void* s, void* out_g1_partials, void* out_g2_partial) {
    if (!pk || !m) return fail(ctx, B2S_ERR_MISSING_CS, "prove_shard: null key or matrices");
    if (z_missing(m, z_inst, z_wit, z_dev) || !r || !s || !out_g1_partials || !out_g2_partial)
        return fail(ctx, B2S_ERR_ASSIGNMENT_MISSING, "prove_shard: null assignment or output");
    const Sizes z = sizes(ctx);
    DevBuf g1, g2;
    B2S_TRY(g1.alloc(ctx, 4 * z.g1x));
    B2S_TRY(g2.alloc(ctx, z.g2x));
    B2S_TRY(groth16_shard(ctx, pk, m, z_inst, z_wit, z_dev, r, s, g1.p, g2.p));
    B2S_CUDA(ctx, cudaMemcpyAsync(out_g1_partials, g1.p, 4 * z.g1x, cudaMemcpyDeviceToHost, ctx->stream));
    B2S_CUDA(ctx, cudaMemcpyAsync(out_g2_partial, g2.p, z.g2x, cudaMemcpyDeviceToHost, ctx->stream));
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return B2S_OK;
}
extern "C" {

int32_t b2s_r1cs_upload(b2s_ctx* ctx, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                        const uint64_t* const row_ptr[3], const uint32_t* const col[3], const void* const coeff[3],
                        b2s_r1cs** out) {
    LOCK(ctx);
    if (!out || !row_ptr || !col || !coeff) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload: null argument");
    for (int k = 0; k < 3; k++)
        if (!row_ptr[k] || ((!col[k] || !coeff[k]) && row_ptr[k][n_rows] != 0))
            return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload: null CSR array for matrix %d", k);
    *out = nullptr;
    return r1cs_upload(ctx, n_rows, n_instance, n_witness, row_ptr, col, coeff, out);
}

int32_t b2s_r1cs_upload_lcmap(b2s_ctx* ctx, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                              const uint64_t* const args[3], uint64_t n_lcs, const uint64_t* lc_offsets,
                              const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len,
                              b2s_r1cs** out) {
    LOCK(ctx);
    if (!out || !args || !lc_offsets || !pool) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap: null argument");
    for (int k = 0; k < 3; k++)
        if (!args[k] && n_rows) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap: null argument array %d", k);
    if (n_lcs && lc_offsets[n_lcs] != 0 && (!lc_vars || !lc_coeffs)) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap: null LC arrays");
    *out = nullptr;
    return r1cs_upload_lcmap(ctx, n_rows, n_instance, n_witness, args, n_lcs, lc_offsets, lc_vars, lc_coeffs, pool, pool_len, nullptr, out);
}

int32_t b2s_r1cs_upload_lcmap_outline(b2s_ctx* ctx, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                                      const uint64_t* const args[3], uint64_t n_lcs, const uint64_t* lc_offsets,
                                      const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len,
                                      const b2s_outline* outline, b2s_r1cs** out) {
    LOCK(ctx);
    if (!out || !args || !lc_offsets || !pool || !outline) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap_outline: null argument");
    for (int k = 0; k < 3; k++)
        if (!args[k] && n_rows) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap_outline: null argument array %d", k);
    if (n_lcs && lc_offsets[n_lcs] != 0 && (!lc_vars || !lc_coeffs))
        return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap_outline: null LC arrays");
    *out = nullptr;
    return r1cs_upload_lcmap(ctx, n_rows, n_instance, n_witness, args, n_lcs, lc_offsets, lc_vars, lc_coeffs, pool, pool_len, outline, out);
}

int32_t b2s_r1cs_outline_assignment(b2s_ctx* ctx, const b2s_r1cs* m, uint64_t n_assign, const void* z, int32_t mem, void* out_z) {
    LOCK(ctx);
    if (!m || (n_assign && (!z || !out_z))) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_outline_assignment: null argument");
    if (!m->outline_copies)
        return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_outline_assignment: the handle was not made by b2s_r1cs_upload_lcmap_outline");
    const uint64_t n_src = m->n_instance + m->n_witness - m->outline_copies;
    return outline_assignment(ctx, n_src, m->outline_copies, n_assign, z, mem, out_z);
}

void b2s_r1cs_free(b2s_ctx* ctx, b2s_r1cs* m) {
    if (!ctx || !m) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->device);
    delete m;
}

uint64_t b2s_r1cs_domain_size(const b2s_r1cs* m) { return m ? (1ull << m->log_domain) : 0; }

int32_t b2s_spmv(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, void* out_a, void* out_b, void* out_c) {
    LOCK(ctx);
    if (!m) return fail(ctx, B2S_ERR_MISSING_CS, "spmv: null matrices");
    if (!z || !out_a || !out_b || !out_c) return fail(ctx, B2S_ERR_INVALID_ARG, "spmv: null buffer");
    const size_t nz = (m->n_instance + m->n_witness) * 32, no = m->n_rows * 32;
    InBuf zi;
    OutBuf a, b, c;
    B2S_TRY(zi.bind(ctx, z, nz, mem));
    B2S_TRY(a.bind(ctx, out_a, no, mem));
    B2S_TRY(b.bind(ctx, out_b, no, mem));
    B2S_TRY(c.bind(ctx, out_c, no, mem));
    B2S_TRY(spmv_run(ctx, m, zi.dptr, a.dptr, b.dptr, c.dptr));
    B2S_TRY(a.copy_back(ctx));
    B2S_TRY(b.copy_back(ctx));
    return c.finish(ctx);
}

static int32_t witness_map_common(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, int32_t qap, void* out_h) {
    if (!m) return fail(ctx, B2S_ERR_MISSING_CS, "witness_map: null matrices");
    if (!z || !out_h) return fail(ctx, B2S_ERR_INVALID_ARG, "witness_map: null buffer");
    B2S_TRY(check_qap(ctx, qap, "witness_map"));
    const size_t nz = (m->n_instance + m->n_witness) * 32, nh = (size_t)32 << m->log_domain;
    InBuf zi;
    OutBuf h;
    B2S_TRY(zi.bind(ctx, z, nz, mem));
    B2S_TRY(h.bind(ctx, out_h, nh, mem));
    B2S_TRY(witness_map_run(ctx, m, zi.dptr, h.dptr, qap));
    return h.finish(ctx);
}

int32_t b2s_witness_map(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, void* out_h) {
    LOCK(ctx);
    return witness_map_common(ctx, m, z, mem, B2S_QAP_LIBSNARK, out_h);
}

int32_t b2s_witness_map_qap(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, int32_t qap, void* out_h) {
    LOCK(ctx);
    return witness_map_common(ctx, m, z, mem, qap, out_h);
}

int32_t b2s_witness_map_sim(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, uint32_t log_ranks, void* out_h) {
    LOCK(ctx);
    if (!m) return fail(ctx, B2S_ERR_MISSING_CS, "witness_map_sim: null matrices");
    if (!z || !out_h) return fail(ctx, B2S_ERR_INVALID_ARG, "witness_map_sim: null buffer");
    if (!dist_supported(m->log_domain, log_ranks))
        return fail(ctx, B2S_ERR_INVALID_ARG, "witness_map_sim: domain 2^%u cannot be cut over 2^%u ranks", m->log_domain, log_ranks);
    const size_t nz = (m->n_instance + m->n_witness) * 32, nh = (size_t)32 << m->log_domain;
    InBuf zi;
    OutBuf h;
    B2S_TRY(zi.bind(ctx, z, nz, mem));
    B2S_TRY(h.bind(ctx, out_h, nh, mem));
    B2S_TRY(witness_map_sim(ctx, m, zi.dptr, log_ranks, h.dptr));
    return h.finish(ctx);
}

int32_t b2s_gr1cs_upload(b2s_ctx* ctx, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates, const b2s_predicate_desc* preds,
                         b2s_gr1cs** out) {
    LOCK(ctx);
    if (!out || (!preds && n_predicates)) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_upload: null argument");
    *out = nullptr;
    return gr1cs_upload(ctx, n_instance, n_witness, n_predicates, preds, out);
}

int32_t b2s_gr1cs_upload_lcmap(b2s_ctx* ctx, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates,
                               const b2s_predicate_lcmap_desc* preds, uint64_t n_lcs, const uint64_t* lc_offsets, const uint64_t* lc_vars,
                               const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len, b2s_gr1cs** out) {
    LOCK(ctx);
    if (!out || (!preds && n_predicates) || !lc_offsets || !pool) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_upload_lcmap: null argument");
    if (n_lcs && lc_offsets[n_lcs] != 0 && (!lc_vars || !lc_coeffs)) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_upload_lcmap: null LC arrays");
    *out = nullptr;
    return gr1cs_upload_lcmap(ctx, n_instance, n_witness, n_predicates, preds, LcMapHost{n_lcs, lc_offsets, lc_vars, lc_coeffs, pool, pool_len},
                              nullptr, out);
}

int32_t b2s_gr1cs_upload_lcmap_outline(b2s_ctx* ctx, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates,
                                       const b2s_predicate_lcmap_desc* preds, uint64_t n_lcs, const uint64_t* lc_offsets,
                                       const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len,
                                       const b2s_outline* outline, b2s_gr1cs** out) {
    LOCK(ctx);
    if (!out || (!preds && n_predicates) || !lc_offsets || !pool || !outline)
        return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_upload_lcmap_outline: null argument");
    if (n_lcs && lc_offsets[n_lcs] != 0 && (!lc_vars || !lc_coeffs))
        return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_upload_lcmap_outline: null LC arrays");
    *out = nullptr;
    return gr1cs_upload_lcmap(ctx, n_instance, n_witness, n_predicates, preds, LcMapHost{n_lcs, lc_offsets, lc_vars, lc_coeffs, pool, pool_len},
                              outline, out);
}

int32_t b2s_gr1cs_outline_assignment(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z) {
    LOCK(ctx);
    if (!g || (n_assign && (!z || !out_z))) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_outline_assignment: null argument");
    if (g->curve != ctx->curve)
        return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_outline_assignment: the handle was made on a ctx of curve %d, this ctx is curve %d",
                    g->curve, ctx->curve);
    if (!g->outline_copies)
        return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_outline_assignment: the handle was not made by b2s_gr1cs_upload_lcmap_outline");
    const uint64_t n_src = g->n_instance + g->n_witness - g->outline_copies;
    return outline_assignment(ctx, n_src, g->outline_copies, n_assign, z, mem, out_z);
}

void b2s_gr1cs_free(b2s_ctx* ctx, b2s_gr1cs* g) {
    if (!ctx || !g) return;
    std::lock_guard<std::mutex> guard(ctx->mu);
    cudaSetDevice(ctx->device);
    delete g;
}

int32_t b2s_gr1cs_check(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, uint64_t* first_unsat,
                        uint64_t* n_unsat) {
    LOCK(ctx);
    if (!g) return fail(ctx, B2S_ERR_MISSING_CS, "gr1cs_check: null constraint system");
    if (n_assign && (!z || !first_unsat)) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_check: null buffer");
    return gr1cs_check(ctx, g, n_assign, z, mem, first_unsat, n_unsat);
}

int32_t b2s_r1cs_check(b2s_ctx* ctx, const b2s_r1cs* m, uint64_t n_assign, const void* z, int32_t mem, uint64_t* first_unsat,
                       uint64_t* n_unsat) {
    LOCK(ctx);
    if (!m) return fail(ctx, B2S_ERR_MISSING_CS, "r1cs_check: null matrices");
    if (n_assign && (!z || !first_unsat)) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_check: null buffer");
    return r1cs_check(ctx, m, n_assign, z, mem, first_unsat, n_unsat);
}

int32_t b2s_r1cs_to_sr1cs(b2s_ctx* ctx, const b2s_r1cs* m, b2s_gr1cs** out) {
    LOCK(ctx);
    if (!m || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_to_sr1cs: null argument");
    *out = nullptr;
    return r1cs_to_sr1cs(ctx, m, out);
}

int32_t b2s_sr1cs_assignment(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z) {
    LOCK(ctx);
    if (!g || (n_assign && (!z || !out_z))) return fail(ctx, B2S_ERR_INVALID_ARG, "sr1cs_assignment: null argument");
    return sr1cs_assignment(ctx, g, n_assign, z, mem, out_z);
}

int32_t b2s_gr1cs_info(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_vars[2], uint32_t* n_predicates, b2s_gr1cs_pred_info* preds,
                       uint32_t cap) {
    LOCK(ctx);
    if (!g || !n_vars || !n_predicates || (cap && !preds)) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_info: null argument");
    return gr1cs_info(ctx, g, n_vars, n_predicates, preds, cap);
}

int32_t b2s_gr1cs_export(b2s_ctx* ctx, const b2s_gr1cs* g, uint32_t pred, uint32_t arg, uint64_t* row_ptr, uint64_t cap_row_ptr,
                         uint32_t* col, uint64_t cap_col, void* coeff, uint64_t cap_coeff) {
    LOCK(ctx);
    if (!g || !row_ptr || (cap_col && !col) || (cap_coeff && !coeff)) return fail(ctx, B2S_ERR_INVALID_ARG, "gr1cs_export: null argument");
    return gr1cs_export(ctx, g, pred, arg, row_ptr, cap_row_ptr, col, cap_col, coeff, cap_coeff);
}

int32_t b2s_pk_upload(b2s_ctx* ctx, const b2s_pk_desc* desc, int32_t mem, b2s_pk** out) {
    LOCK(ctx);
    if (!desc || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "pk_upload: null argument");
    *out = nullptr;
    return pk_upload(ctx, desc, mem, B2S_QAP_LIBSNARK, out);
}

int32_t b2s_pk_upload_qap(b2s_ctx* ctx, const b2s_pk_desc* desc, int32_t mem, int32_t qap, b2s_pk** out) {
    LOCK(ctx);
    if (!desc || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "pk_upload: null argument");
    *out = nullptr;
    B2S_TRY(check_qap(ctx, qap, "pk_upload"));
    return pk_upload(ctx, desc, mem, qap, out);
}

void b2s_pk_free(b2s_ctx* ctx, b2s_pk* pk) {
    if (!ctx || !pk) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->device);
    delete pk;
}

int32_t b2s_groth16_prove_shard(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_instance,
                                const void* z_witness, const void* r, const void* s, void* out_g1_partials,
                                void* out_g2_partial) {
    LOCK(ctx);
    return prove_partial(ctx, pk, m, z_instance, z_witness, nullptr, r, s, out_g1_partials, out_g2_partial);
}

int32_t b2s_groth16_finish(b2s_ctx* ctx, const b2s_pk* pk, const void* g1_partials, const void* g2_partials,
                           uint32_t n_shards, const void* r, const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    LOCK(ctx);
    if (!pk) return fail(ctx, B2S_ERR_MISSING_CS, "finish: null key");
    if (!g1_partials || !g2_partials || !n_shards || !r || !s || !out_a_g1 || !out_b_g2 || !out_c_g1)
        return fail(ctx, B2S_ERR_INVALID_ARG, "finish: null argument");
    const Sizes z = sizes(ctx);
    InBuf p1, p2;
    B2S_TRY(p1.bind(ctx, g1_partials, (size_t)n_shards * 4 * z.g1x, B2S_MEM_HOST));
    B2S_TRY(p2.bind(ctx, g2_partials, (size_t)n_shards * z.g2x, B2S_MEM_HOST));
    return groth16_finish(ctx, pk, p1.dptr, p2.dptr, n_shards, r, s, out_a_g1, out_b_g2, out_c_g1);
}

int32_t b2s_groth16_prove(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_instance, const void* z_witness,
                          const void* r, const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    LOCK(ctx);
    return prove_full(ctx, pk, m, z_instance, z_witness, nullptr, r, s, out_a_g1, out_b_g2, out_c_g1);
}

int32_t b2s_groth16_prove_resident(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void* r,
                                   const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    LOCK(ctx);
    return prove_full(ctx, pk, m, nullptr, nullptr, z_dev, r, s, out_a_g1, out_b_g2, out_c_g1);
}

int32_t b2s_groth16_prove_batch(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, uint64_t n_proofs, const void* z, const void* r,
                                const void* s, int32_t mem, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    LOCK(ctx);
    if (!pk || !m) return fail(ctx, B2S_ERR_MISSING_CS, "prove_batch: null key or matrices");
    if (!z || !r || !s) return fail(ctx, B2S_ERR_ASSIGNMENT_MISSING, "prove_batch: null assignment");
    if (!out_a_g1 || !out_b_g2 || !out_c_g1) return fail(ctx, B2S_ERR_INVALID_ARG, "prove_batch: null output");
    if (!pk_is_full(pk)) return fail(ctx, B2S_ERR_MALFORMED_VK, "prove_batch: needs a full (unsharded) proving key");
    return groth16_prove_batch(ctx, pk, m, n_proofs, z, r, s, mem, out_a_g1, out_b_g2, out_c_g1);
}

int32_t b2s_groth16_prove_shard_resident(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void* r,
                                         const void* s, void* out_g1_partials, void* out_g2_partial) {
    LOCK(ctx);
    return prove_partial(ctx, pk, m, nullptr, nullptr, z_dev, r, s, out_g1_partials, out_g2_partial);
}

int32_t b2s_profile_enable(b2s_ctx* ctx, int32_t on) {
    LOCK(ctx);
    ctx->profiling = on != 0;
    return B2S_OK;
}

int32_t b2s_profile_report(b2s_ctx* ctx, char* buf, uint64_t cap) {
    LOCK(ctx);
    if (!buf || cap == 0) return fail(ctx, B2S_ERR_INVALID_ARG, "profile_report: null buffer");
    B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    std::map<std::string, std::pair<uint64_t, double>> agg;
    const bool verbose = getenv("B2S_PROFILE_VERBOSE") != nullptr;
    cudaEvent_t prev_end = nullptr;
    for (auto& r : ctx->prof) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, r.e0, r.e1);
        if (verbose) {
            // idle time between the end of the previous recorded launch and the start of this one (launch order; kernels of the
            // aux stream overlap the main stream, so a negative or tiny gap there means "ran concurrently")
            float gap = 0.f;
            if (prev_end) cudaEventElapsedTime(&gap, prev_end, r.e0);
            fprintf(stderr, "[b2s-profile] %-40s %.3f ms  gap %.3f ms\n", r.name, ms, gap);
            prev_end = r.e1;
        }
        auto& a = agg[r.name];
        a.first++;
        a.second += ms;
    }
    for (auto& r : ctx->prof) {
        cudaEventDestroy(r.e0);
        cudaEventDestroy(r.e1);
    }
    ctx->prof.clear();
    std::string out;
    char line[256];
    for (auto& kv : agg) {
        snprintf(line, sizeof(line), "%s\t%llu\t%.6f\n", kv.first.c_str(), (unsigned long long)kv.second.first, kv.second.second);
        out += line;
    }
    const size_t nn = out.size() < cap - 1 ? out.size() : (size_t)cap - 1;
    memcpy(buf, out.data(), nn);
    buf[nn] = 0;
    return B2S_OK;
}


static int32_t setup_common(b2s_ctx* ctx, const b2s_r1cs* m, const void* trapdoor, int32_t qap, b2s_pk** out_pk, void* out_alpha_g1,
                            void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1) {
    if (!m) return fail(ctx, B2S_ERR_MISSING_CS, "setup: null matrices");
    if (!trapdoor || !out_pk || !out_alpha_g1 || !out_beta_g2 || !out_gamma_g2 || !out_delta_g2 || !out_gamma_abc_g1)
        return fail(ctx, B2S_ERR_INVALID_ARG, "setup: null argument");
    *out_pk = nullptr;
    B2S_TRY(check_qap(ctx, qap, "setup"));
    return groth16_setup(ctx, m, trapdoor, qap, out_pk, out_alpha_g1, out_beta_g2, out_gamma_g2, out_delta_g2, out_gamma_abc_g1);
}

int32_t b2s_groth16_setup(b2s_ctx* ctx, const b2s_r1cs* m, const void* trapdoor, b2s_pk** out_pk, void* out_alpha_g1,
                          void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1) {
    LOCK(ctx);
    return setup_common(ctx, m, trapdoor, B2S_QAP_LIBSNARK, out_pk, out_alpha_g1, out_beta_g2, out_gamma_g2, out_delta_g2, out_gamma_abc_g1);
}

int32_t b2s_groth16_setup_qap(b2s_ctx* ctx, const b2s_r1cs* m, const void* trapdoor, int32_t qap, b2s_pk** out_pk, void* out_alpha_g1,
                              void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1) {
    LOCK(ctx);
    return setup_common(ctx, m, trapdoor, qap, out_pk, out_alpha_g1, out_beta_g2, out_gamma_g2, out_delta_g2, out_gamma_abc_g1);
}

int32_t b2s_pk_query(b2s_ctx* ctx, const b2s_pk* pk, int32_t which, void* out, uint64_t cap_bytes) {
    LOCK(ctx);
    if (!pk || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "pk_query: null argument");
    return pk_query_download(ctx, pk, which, out, cap_bytes);
}


int32_t b2s_serialize_g1_compressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap) {
    LOCK(ctx);
    if ((!affine || !out) && count) return fail(ctx, B2S_ERR_INVALID_ARG, "serialize: null buffer");
    return serialize_points_ex(ctx, 1, affine, B2S_MEM_HOST, count, true, out, cap);
}
int32_t b2s_serialize_g2_compressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap) {
    LOCK(ctx);
    if ((!affine || !out) && count) return fail(ctx, B2S_ERR_INVALID_ARG, "serialize: null buffer");
    return serialize_points_ex(ctx, 2, affine, B2S_MEM_HOST, count, true, out, cap);
}
int32_t b2s_serialize_g1_uncompressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap) {
    LOCK(ctx);
    if ((!affine || !out) && count) return fail(ctx, B2S_ERR_INVALID_ARG, "serialize: null buffer");
    return serialize_points_ex(ctx, 1, affine, B2S_MEM_HOST, count, false, out, cap);
}
int32_t b2s_serialize_g2_uncompressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap) {
    LOCK(ctx);
    if ((!affine || !out) && count) return fail(ctx, B2S_ERR_INVALID_ARG, "serialize: null buffer");
    return serialize_points_ex(ctx, 2, affine, B2S_MEM_HOST, count, false, out, cap);
}
int32_t b2s_proof_serialize_uncompressed(b2s_ctx* ctx, const void* a_g1, const void* b_g2, const void* c_g1, uint8_t* out, uint64_t cap) {
    LOCK(ctx);
    if (!a_g1 || !b_g2 || !c_g1 || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "proof_serialize: null buffer");
    return proof_serialize(ctx, a_g1, b_g2, c_g1, false, out, cap);
}
uint64_t b2s_vk_serialized_size(const b2s_ctx* ctx, uint64_t n_gamma_abc, int32_t compressed) {
    return ctx ? vk_serialized_size(const_cast<b2s_ctx*>(ctx), n_gamma_abc, compressed != 0) : 0;
}
int32_t b2s_vk_serialize(b2s_ctx* ctx, const void* alpha_g1, const void* beta_g2, const void* gamma_g2, const void* delta_g2,
                         const void* gamma_abc_g1, uint64_t n_gamma_abc, int32_t compressed, uint8_t* out, uint64_t cap) {
    LOCK(ctx);
    if (!alpha_g1 || !beta_g2 || !gamma_g2 || !delta_g2 || (!gamma_abc_g1 && n_gamma_abc) || !out)
        return fail(ctx, B2S_ERR_INVALID_ARG, "vk_serialize: null buffer");
    return vk_serialize(ctx, alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1, n_gamma_abc, compressed != 0, out, cap);
}
uint64_t b2s_pk_serialized_size(const b2s_ctx* ctx, const b2s_pk* pk, uint64_t vk_len, int32_t compressed) {
    return (ctx && pk) ? pk_serialized_size(const_cast<b2s_ctx*>(ctx), pk, vk_len, compressed != 0) : 0;
}
int32_t b2s_pk_serialize(b2s_ctx* ctx, const b2s_pk* pk, const uint8_t* vk_bytes, uint64_t vk_len, int32_t compressed, uint8_t* out,
                         uint64_t cap) {
    LOCK(ctx);
    if (!pk || (!vk_bytes && vk_len) || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "pk_serialize: null argument");
    return pk_serialize(ctx, pk, vk_bytes, vk_len, compressed != 0, out, cap);
}

int32_t b2s_proof_serialize_compressed(b2s_ctx* ctx, const void* a_g1, const void* b_g2, const void* c_g1, uint8_t* out,
                                       uint64_t cap) {
    LOCK(ctx);
    if (!a_g1 || !b_g2 || !c_g1 || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "proof_serialize: null buffer");
    return proof_serialize(ctx, a_g1, b_g2, c_g1, true, out, cap);
}

int32_t b2s_deserialize_g1(b2s_ctx* ctx, const uint8_t* in, uint64_t len, uint64_t count, int32_t compressed, int32_t validate,
                           void* out_affine) {
    LOCK(ctx);
    if ((!in && len) || (!out_affine && count)) return fail(ctx, B2S_ERR_INVALID_ARG, "deserialize: null buffer");
    return deserialize_points(ctx, 1, in, len, count, compressed != 0, validate != 0, out_affine);
}
int32_t b2s_deserialize_g2(b2s_ctx* ctx, const uint8_t* in, uint64_t len, uint64_t count, int32_t compressed, int32_t validate,
                           void* out_affine) {
    LOCK(ctx);
    if ((!in && len) || (!out_affine && count)) return fail(ctx, B2S_ERR_INVALID_ARG, "deserialize: null buffer");
    return deserialize_points(ctx, 2, in, len, count, compressed != 0, validate != 0, out_affine);
}
int32_t b2s_proof_deserialize(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, void* out_a_g1,
                              void* out_b_g2, void* out_c_g1) {
    LOCK(ctx);
    if (!in || !out_a_g1 || !out_b_g2 || !out_c_g1) return fail(ctx, B2S_ERR_INVALID_ARG, "proof_deserialize: null buffer");
    return proof_deserialize(ctx, in, len, compressed != 0, validate != 0, out_a_g1, out_b_g2, out_c_g1);
}
int32_t b2s_vk_deserialize(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, void* out_alpha_g1,
                           void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1, uint64_t cap_gamma_abc,
                           uint64_t* n_gamma_abc, uint64_t* consumed) {
    LOCK(ctx);
    if (!in || (out_gamma_abc_g1 && (!out_alpha_g1 || !out_beta_g2 || !out_gamma_g2 || !out_delta_g2)))
        return fail(ctx, B2S_ERR_INVALID_ARG, "vk_deserialize: null buffer");
    return vk_deserialize(ctx, in, len, compressed != 0, validate != 0, out_alpha_g1, out_beta_g2, out_gamma_g2, out_delta_g2,
                          out_gamma_abc_g1, cap_gamma_abc, n_gamma_abc, consumed);
}
int32_t b2s_pk_deserialize(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, b2s_pk** out) {
    LOCK(ctx);
    if (!in || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "pk_deserialize: null argument");
    *out = nullptr;
    return pk_deserialize(ctx, in, len, compressed != 0, validate != 0, B2S_QAP_LIBSNARK, out);
}
int32_t b2s_pk_deserialize_qap(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, int32_t qap,
                               b2s_pk** out) {
    LOCK(ctx);
    if (!in || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "pk_deserialize: null argument");
    *out = nullptr;
    B2S_TRY(check_qap(ctx, qap, "pk_deserialize"));
    return pk_deserialize(ctx, in, len, compressed != 0, validate != 0, qap, out);
}

int32_t b2s_zkey_read_info(b2s_ctx* ctx, const uint8_t* in, uint64_t len, b2s_zkey_info* out) {
    LOCK(ctx);
    if (!in || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "zkey_read_info: null argument");
    return zkey_read_info(ctx, in, len, out);
}
int32_t b2s_zkey_load(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t validate, b2s_pk** out_pk, b2s_r1cs** out_m,
                      void* out_alpha_g1, void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1,
                      uint64_t cap_gamma_abc) {
    LOCK(ctx);
    if (!in || !out_pk || !out_m || !out_alpha_g1 || !out_beta_g2 || !out_gamma_g2 || !out_delta_g2 || !out_gamma_abc_g1)
        return fail(ctx, B2S_ERR_INVALID_ARG, "zkey_load: null argument");
    *out_pk = nullptr;
    *out_m = nullptr;
    return zkey_load(ctx, in, len, validate != 0, out_pk, out_m, out_alpha_g1, out_beta_g2, out_gamma_g2, out_delta_g2,
                     out_gamma_abc_g1, cap_gamma_abc);
}
int32_t b2s_wtns_read(b2s_ctx* ctx, const uint8_t* in, uint64_t len, uint64_t n_vars, int32_t mem, void* out_z) {
    LOCK(ctx);
    if (!in || !out_z) return fail(ctx, B2S_ERR_INVALID_ARG, "wtns_read: null argument");
    return wtns_read(ctx, in, len, n_vars, mem, out_z);
}
int32_t b2s_r1cs_file_read_info(b2s_ctx* ctx, const uint8_t* in, uint64_t len, b2s_r1cs_file_info* out) {
    LOCK(ctx);
    if (!in || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_file_read_info: null argument");
    return r1cs_file_read_info(ctx, in, len, out);
}
int32_t b2s_r1cs_file_load(b2s_ctx* ctx, const uint8_t* in, uint64_t len, b2s_r1cs** out) {
    LOCK(ctx);
    if (!in || !out) return fail(ctx, B2S_ERR_INVALID_ARG, "r1cs_file_load: null argument");
    *out = nullptr;
    return r1cs_file_load(ctx, in, len, out);
}

int32_t b2s_vk_prepare(b2s_ctx* ctx, const void* alpha_g1, const void* beta_g2, const void* gamma_g2, const void* delta_g2,
                       const void* gamma_abc_g1, uint64_t n_gamma_abc, b2s_pvk** out) {
    LOCK(ctx);
    if (!out || !alpha_g1 || !beta_g2 || !gamma_g2 || !delta_g2 || (!gamma_abc_g1 && n_gamma_abc))
        return fail(ctx, B2S_ERR_INVALID_ARG, "vk_prepare: null argument");
    *out = nullptr;
    return vk_prepare(ctx, alpha_g1, beta_g2, gamma_g2, delta_g2, gamma_abc_g1, n_gamma_abc, out);
}
void b2s_pvk_free(b2s_ctx* ctx, b2s_pvk* pvk) {
    if (!ctx || !pvk) return;
    std::lock_guard<std::mutex> g(ctx->mu);
    cudaSetDevice(ctx->device);
    pvk_free(pvk);
}
int32_t b2s_groth16_verify_batch(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                 const void* a_g1, const void* b_g2, const void* c_g1, int32_t mem, uint8_t* ok) {
    LOCK(ctx);
    if (!pvk) return fail(ctx, B2S_ERR_INVALID_ARG, "verify_batch: null prepared key");
    return groth16_verify_batch(ctx, pvk, n_proofs, inputs, n_inputs, a_g1, b_g2, c_g1, mem, ok);
}
int32_t b2s_groth16_verify_batch_rlc(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                     const void* a_g1, const void* b_g2, const void* c_g1, const void* rho, int32_t mem, uint8_t* ok) {
    LOCK(ctx);
    if (!pvk) return fail(ctx, B2S_ERR_INVALID_ARG, "verify_batch_rlc: null prepared key");
    return groth16_verify_batch_rlc(ctx, pvk, n_proofs, inputs, n_inputs, a_g1, b_g2, c_g1, rho, mem, ok);
}
int32_t b2s_groth16_verify_batch_bytes(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                       const uint8_t* proofs, uint64_t len, int32_t compressed, int32_t mem, uint8_t* ok,
                                       uint8_t* reason) {
    LOCK(ctx);
    if (!pvk) return fail(ctx, B2S_ERR_INVALID_ARG, "verify_batch_bytes: null prepared key");
    return groth16_verify_batch_bytes(ctx, pvk, n_proofs, inputs, n_inputs, proofs, len, compressed != 0, mem, ok, reason);
}
int32_t b2s_groth16_verify_batch_rlc_bytes(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                           const uint8_t* proofs, uint64_t len, int32_t compressed, const void* rho, int32_t mem,
                                           uint8_t* ok, uint8_t* reason) {
    LOCK(ctx);
    if (!pvk) return fail(ctx, B2S_ERR_INVALID_ARG, "verify_batch_rlc_bytes: null prepared key");
    return groth16_verify_batch_rlc_bytes(ctx, pvk, n_proofs, inputs, n_inputs, proofs, len, compressed != 0, rho, mem, ok, reason);
}
int32_t b2s_pairing(b2s_ctx* ctx, const void* p_g1, const void* q_g2, uint64_t n, int32_t mem, void* out_gt) {
    LOCK(ctx);
    if (n && (!p_g1 || !q_g2 || !out_gt)) return fail(ctx, B2S_ERR_INVALID_ARG, "pairing: null buffer");
    return pairing_batch(ctx, p_g1, q_g2, n, mem, out_gt);
}

}  // extern "C"
