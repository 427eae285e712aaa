// Groth16 verification of ark-serialized proofs: bytes in, verdicts out, the decoded points never leave the device.
// Every point is decoded with validation (flags, canonical coordinates, curve equation, prime-order subgroup) by
// decode_point (deserialize.cuh), and a proof that fails to decode is rejected on its own, with its reason, instead of
// failing the call.  Per chunk of proofs:
//   verify_decode_g1   two threads per proof, one for A and one for C
//   verify_decode_g2   one thread per proof, for B (the Fq2 square root and the psi criterion do not set the register
//                      budget of the G1 decode)
// Both read the interleaved a || b || c bytes in place and write the affine point into chunk scratch (infinity when the
// point is rejected) and one status byte per (proof, element).  Then
//   per proof   groth16_verify_batch (verify.cu) in device mode on the scratch points, and verify_bytes_fold ANDs the
//               decode status into ok[i] and writes reason[i];
//   RLC         the steps of RlcRun (verify_rlc.cu) on the scratch points; verify_bytes_fold raises one device flag for
//               any decode failure, and verify_bytes_veto clears the verdict with it before the one read-back.
// Host batches are processed in chunks through bounded device scratch, as in verify.cu, so n_proofs is not limited by
// device memory.
#include <algorithm>

#include "common.cuh"
#include "deserialize.cuh"
#include "verify.cuh"

namespace b2s {

int32_t groth16_verify_batch(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const void* a, const void* b,
                             const void* cc, int32_t mem, uint8_t* ok);   // verify.cu

// status[3 i + e]: the DecodeStatus of element e (0 = A, 1 = B, 2 = C) of proof i
template <class Curve>
__global__ void verify_decode_g1_kernel(const uint8_t* in, uint32_t m, int compressed, typename Curve::G1Affine* a,
                                        typename Curve::G1Affine* c, uint8_t* status) {
    using F = typename Curve::Fq;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2 * m) return;
    const uint32_t i = t >> 1, e = t & 1;   // e = 0: A, 1: C
    const size_t g1 = sizeof(F) * (compressed ? 1 : 2), proof = 4 * g1;
    Affine<F> p = Affine<F>::inf();
    const uint32_t st = decode_point<Curve, F>(in + i * proof + (e ? 3 * g1 : 0), compressed != 0, true, p);
    if (st != DEC_OK) p = Affine<F>::inf();
    (e ? c : a)[i] = p;
    status[3 * i + 2 * e] = (uint8_t)st;
}

template <class Curve>
__global__ void verify_decode_g2_kernel(const uint8_t* in, uint32_t m, int compressed, typename Curve::G2Affine* b, uint8_t* status) {
    using F = typename Curve::Fq2;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const size_t g1 = sizeof(typename Curve::Fq) * (compressed ? 1 : 2), proof = 4 * g1;
    Affine<F> p = Affine<F>::inf();
    const uint32_t st = decode_point<Curve, F>(in + i * proof + g1, compressed != 0, true, p);
    if (st != DEC_OK) p = Affine<F>::inf();
    b[i] = p;
    status[3 * i + 1] = (uint8_t)st;
}

// reason[i] = 0 when all three elements decoded, else 16 (1 + e) + status of the first failing element e; ok[i] is
// cleared for such a proof, and *bad is set.  Each of ok, reason and bad may be null.
__global__ void verify_bytes_fold_kernel(const uint8_t* status, uint32_t m, uint8_t* ok, uint8_t* reason, uint8_t* bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    uint8_t r = 0;
    for (int e = 2; e >= 0; e--) {
        const uint8_t s = status[3 * i + e];
        if (s) r = (uint8_t)(16 * (1 + e) + s);
    }
    if (reason) reason[i] = r;
    if (r && ok) ok[i] = 0;
    if (r && bad) *bad = 1;
}

__global__ void verify_bytes_veto_kernel(const uint8_t* bad, uint8_t* ok) {
    if (blockIdx.x | threadIdx.x) return;
    if (*bad) *ok = 0;
}

namespace {

// The chunk scratch both paths share: the decoded points and the status bytes.
struct Decoded {
    DevBuf buf;
    void *a = nullptr, *b = nullptr, *c = nullptr;
    uint8_t* status = nullptr;
    static size_t per_proof(Ctx* ctx) {
        const Sizes z = sizes(ctx);
        return 2 * z.g1 + z.g2 + 3;
    }
    int32_t alloc(Ctx* ctx, uint64_t ch) {
        const Sizes z = sizes(ctx);
        B2S_TRY(buf.alloc(ctx, ch * per_proof(ctx)));
        char* q = buf.as<char>();
        a = q; q += ch * z.g1;
        b = q; q += ch * z.g2;
        c = q; q += ch * z.g1;
        status = reinterpret_cast<uint8_t*>(q);
        return B2S_OK;
    }
    // the proof bytes of a chunk of m proofs, on the device -> a, b, c, status
    int32_t decode(Ctx* ctx, const uint8_t* in, uint32_t m, bool compressed) {
        return dispatch_curve(ctx, [&](auto curve) -> int32_t {
            using C = decltype(curve);
            B2S_LAUNCH_N(ctx, "verify_decode_g1", verify_decode_g1_kernel<C>, cdiv(2ull * m, VERIFY_THREADS), VERIFY_THREADS, 0, in, m,
                         (int)compressed, static_cast<typename C::G1Affine*>(a), static_cast<typename C::G1Affine*>(c), status);
            B2S_LAUNCH_N(ctx, "verify_decode_g2", verify_decode_g2_kernel<C>, cdiv(m, VERIFY_THREADS), VERIFY_THREADS, 0, in, m,
                         (int)compressed, static_cast<typename C::G2Affine*>(b), status);
            return (int32_t)B2S_OK;
        });
    }
};

// bytes of one serialized proof
size_t proof_bytes(Ctx* c, bool compressed) {
    const Sizes z = sizes(c);
    return 2 * z.enc(1, compressed) + z.enc(2, compressed);
}

// the checks both entry points share, in the order of the points entry points; then the length of `proofs`
int32_t check_args(Ctx* c, const char* name, const b2s_pvk* pvk, uint64_t n, uint64_t ni, uint64_t len, bool compressed) {
    if (pvk->curve != c->curve) return fail(c, B2S_ERR_INVALID_ARG, "%s: the prepared key belongs to another curve", name);
    if (ni + 1 != pvk->n_abc)
        return fail(c, B2S_ERR_MALFORMED_VK, "%s: %llu public inputs, the key expects %llu", name, (unsigned long long)ni,
                    (unsigned long long)(pvk->n_abc - 1));
    const size_t pb = proof_bytes(c, compressed);
    if (n > len / pb || n * pb != len)
        return fail(c, B2S_ERR_INVALID_DATA, "%s: %llu bytes are not %llu proofs of %zu bytes", name, (unsigned long long)len,
                    (unsigned long long)n, pb);
    return B2S_OK;
}

}  // namespace

int32_t groth16_verify_batch_bytes(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const uint8_t* proofs,
                                   uint64_t len, bool compressed, int32_t mem, uint8_t* ok, uint8_t* reason) {
    const char* name = "verify_batch_bytes";
    B2S_TRY(check_args(c, name, pvk, n, ni, len, compressed));
    if (n == 0) return B2S_OK;
    if (!proofs || !ok || (ni && !inputs)) return fail(c, B2S_ERR_INVALID_ARG, "%s: null buffer", name);
    RowStager io(c, mem, {col_in(inputs, ni * sizes(c).fr), col_in(proofs, proof_bytes(c, compressed)), col_out(ok, 1), col_out(reason, 1)});
    const uint64_t ch = chunk_size(n, Decoded::per_proof(c) + io.row_bytes());
    Decoded d;
    B2S_TRY(d.alloc(c, ch));
    B2S_TRY(io.alloc(ch));
    for (uint64_t base = 0; base < n; base += ch) {
        const uint32_t m = (uint32_t)std::min<uint64_t>(ch, n - base);
        B2S_TRY(io.load(base, m));
        uint8_t *oki = io.ptr<uint8_t>(2), *rsi = io.ptr<uint8_t>(3);
        B2S_TRY(d.decode(c, io.ptr<uint8_t>(1), m, compressed));
        B2S_TRY(groth16_verify_batch(c, pvk, m, io.ptr(0), ni, d.a, d.b, d.c, B2S_MEM_DEVICE, oki));
        B2S_LAUNCH_N(c, "verify_bytes_fold", verify_bytes_fold_kernel, cdiv(m, VERIFY_THREADS), VERIFY_THREADS, 0, d.status, m, oki, rsi,
                     (uint8_t*)nullptr);
        B2S_TRY(io.store());
    }
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

int32_t groth16_verify_batch_rlc_bytes(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const uint8_t* proofs,
                                       uint64_t len, bool compressed, const void* rho, int32_t mem, uint8_t* ok, uint8_t* reason) {
    const char* name = "verify_batch_rlc_bytes";
    if (!ok) return fail(c, B2S_ERR_INVALID_ARG, "%s: null buffer", name);
    *ok = 0;
    B2S_TRY(check_args(c, name, pvk, n, ni, len, compressed));
    if (n == 0) { *ok = 1; return B2S_OK; }
    if (!proofs || !rho || (ni && !inputs)) return fail(c, B2S_ERR_INVALID_ARG, "%s: null buffer", name);
    RowStager io(c, mem, {col_in(inputs, ni * sizes(c).fr), col_in(proofs, proof_bytes(c, compressed)), col_in(rho, RLC_RHO),
                          col_out(reason, 1)});
    const uint64_t ch = chunk_size(n, rlc_per_proof(c) + Decoded::per_proof(c) + io.row_bytes());
    RlcRun r;
    B2S_TRY(rlc_begin(c, pvk, ni, ch, name, r));
    Decoded d;
    B2S_TRY(d.alloc(c, ch));
    B2S_TRY(io.alloc(ch));
    DevBuf bad;   // the decode-failure flag
    B2S_TRY(bad.alloc(c, 1));
    B2S_CUDA(c, cudaMemsetAsync(bad.p, 0, 1, c->stream));
    for (uint64_t base = 0; base < n; base += ch) {
        const uint32_t m = (uint32_t)std::min<uint64_t>(ch, n - base);
        B2S_TRY(io.load(base, m));
        B2S_TRY(d.decode(c, io.ptr<uint8_t>(1), m, compressed));
        B2S_LAUNCH_N(c, "verify_bytes_fold", verify_bytes_fold_kernel, cdiv(m, VERIFY_THREADS), VERIFY_THREADS, 0, d.status, m,
                     (uint8_t*)nullptr, io.ptr<uint8_t>(3), bad.as<uint8_t>());
        B2S_TRY(rlc_chunk(r, io.ptr(0), d.a, d.b, d.c, io.ptr(2), m, base, base + m == n));
        B2S_TRY(io.store());
    }
    B2S_LAUNCH_N(c, "verify_bytes_veto", verify_bytes_veto_kernel, 1, 1, 0, bad.as<const uint8_t>(), r.ok_dev);
    return rlc_read(r, ok);
}

}  // namespace b2s
