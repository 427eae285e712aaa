// Wire format of group elements, proofs and keys (SURVEY.md 8(f) row 3): what
// `CanonicalSerialize::serialize_compressed` / `serialize_uncompressed` give for the associated types of `SNARK`
// (/root/reference/snark/src/lib.rs:25-36 bounds; encodings of ark-serialize / ark-bls12-381 / ark-bn254, not in
// /root/reference, SURVEY.md Appendix A.7):
//   BLS12-381 (zcash / IETF form): x big-endian; top bits of byte 0: 0x80 compressed, 0x40 infinity, 0x20 y is the
//                                  lexicographically larger root; G2 writes x.c1 || x.c0
//   BN254, BLS12-377 (ark-ec SWFlags): x little-endian; top bits of the LAST byte: 0x80 y > -y, 0x40 infinity; G2 writes
//                                  x.c0 || x.c1
//   "larger" compares canonical integers; for Fq2, c1 first then c0.   Proof = A || B || C.
//   Uncompressed: x || y in the same byte / component order; BLS12-381 keeps only the infinity bit (0x40) in byte 0, BN254
//   keeps both SWFlags in the last byte of y.   Vec<T> = u64 little-endian length, then the elements.
//   VerifyingKey = alpha_g1 || beta_g2 || gamma_g2 || delta_g2 || Vec(gamma_abc_g1);
//   ProvingKey   = vk || beta_g1 || delta_g1 || Vec(a_query) || Vec(b_g1_query) || Vec(b_g2_query) || Vec(h_query) || Vec(l_query)
//   (ark-groth16 derive order, recalled; the oracle restates the same in oracle/serialize.py).
// The GPU turns Montgomery limbs into canonical ones and decides the sign bit (field arithmetic stays on the
// device); the host only orders bytes.  Known answers: the standard compressed BLS12-381 generators
// (tests/test_gpu_serialize.py).
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "deserialize.cuh"   // y_is_larger

namespace b2s {

struct CanonPoint { uint32_t x[24]; uint32_t y[24]; uint32_t flags; uint32_t pad[3]; };   // up to 2 x 12 limbs each; flags: 1 = inf, 2 = y larger

template <class P>
__device__ __forceinline__ void put_canon(uint32_t* o, const Fp<P>& x) {
    const Fp<P> c = x.from_mont();
    for (int i = 0; i < Fp<P>::N; i++) o[i] = c.v[i];
}
template <class P>
__device__ __forceinline__ void put_canon(uint32_t* o, const Fp2<P>& x) {
    const Fp<P> c0 = x.c0.from_mont(), c1 = x.c1.from_mont();
    for (int i = 0; i < Fp<P>::N; i++) { o[i] = c0.v[i]; o[Fp<P>::N + i] = c1.v[i]; }
}

template <class F>
__global__ void canon_points_kernel(const Affine<F>* pts, uint32_t count, CanonPoint* out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const Affine<F> p = pts[i];
    CanonPoint o;
    for (int k = 0; k < 24; k++) { o.x[k] = 0; o.y[k] = 0; }
    o.pad[0] = o.pad[1] = o.pad[2] = 0;
    if (p.is_inf()) o.flags = 1;
    else { put_canon(o.x, p.x); put_canon(o.y, p.y); o.flags = y_is_larger(p.y) ? 2u : 0u; }
    out[i] = o;
}

// byte order on the host: one canonical point -> its encoding
static void encode_point(bool bls, int group, bool compressed, size_t fq, const CanonPoint& p, uint8_t* o) {
    const size_t words = fq / 4, coord = (group == 1 ? 1 : 2) * fq, out_bytes = (compressed ? 1 : 2) * coord;
    auto put = [&](uint8_t* dst, const uint32_t* limbs) {   // one coordinate (Fq or Fq2) in the curve's byte / component order
        const uint8_t* le0 = reinterpret_cast<const uint8_t*>(limbs);
        const uint8_t* le1 = reinterpret_cast<const uint8_t*>(limbs + words);
        if (bls) {
            if (group == 1) for (size_t b = 0; b < fq; b++) dst[b] = le0[fq - 1 - b];
            else for (size_t b = 0; b < fq; b++) { dst[b] = le1[fq - 1 - b]; dst[fq + b] = le0[fq - 1 - b]; }
        } else {
            memcpy(dst, le0, fq);
            if (group == 2) memcpy(dst + fq, le1, fq);
        }
    };
    memset(o, 0, out_bytes);
    const bool inf = p.flags & 1, larger = p.flags & 2;
    if (!inf) {
        put(o, p.x);
        if (!compressed) put(o + coord, p.y);
    }
    if (bls) {
        if (compressed) o[0] |= 0x80;
        if (inf) o[0] |= 0x40;
        if (compressed && larger && !inf) o[0] |= 0x20;
    } else {
        if (inf) o[out_bytes - 1] |= 0x40;
        else if (larger) o[out_bytes - 1] |= 0x80;
    }
}

// `count` affine Montgomery points (HOST or DEVICE) -> encoded bytes on the host; chunked so that keys of any size stream through
int32_t serialize_points_ex(Ctx* c, int group, const void* affine, int32_t mem, uint64_t count, bool compressed, uint8_t* out, uint64_t cap) {
    bool bls = false;   // zcash / IETF form (BLS12-381); otherwise ark-ec SWFlags (BN254, BLS12-377)
    B2S_TRY(dispatch_curve(c, [&](auto curve) { bls = decltype(curve)::FqP::ZCASH_SERIAL; return (int32_t)B2S_OK; }));
    const Sizes z = sizes(c);
    const size_t in_bytes = z.aff(group), out_bytes = z.enc(group, compressed);
    if (count * out_bytes > cap) return fail(c, B2S_ERR_INVALID_ARG, "serialize: output buffer too small");
    const uint64_t CH = 1u << 18;
    DevBuf d;
    RowStager io(c, mem, {col_in(affine, in_bytes)});
    B2S_TRY(d.alloc(c, (size_t)std::min<uint64_t>(count, CH) * sizeof(CanonPoint)));
    B2S_TRY(io.alloc(std::min<uint64_t>(count, CH)));
    std::vector<CanonPoint> h((size_t)std::min<uint64_t>(count, CH));
    for (uint64_t base = 0; base < count; base += CH) {
        const uint32_t n = (uint32_t)std::min<uint64_t>(CH, count - base);
        B2S_TRY(io.load(base, n));
        const char* src = io.ptr(0);
        int32_t st = dispatch_curve(c, [&](auto curve) {
            using C = decltype(curve);
            if (group == 1) B2S_LAUNCH(c, canon_points_kernel<typename C::Fq>, cdiv(n, 64), 64, 0, reinterpret_cast<const Affine<typename C::Fq>*>(src), n, d.as<CanonPoint>());
            else B2S_LAUNCH(c, canon_points_kernel<typename C::Fq2>, cdiv(n, 64), 64, 0, reinterpret_cast<const Affine<typename C::Fq2>*>(src), n, d.as<CanonPoint>());
            return (int32_t)B2S_OK;
        });
        B2S_TRY(st);
        B2S_CUDA(c, cudaMemcpyAsync(h.data(), d.p, (size_t)n * sizeof(CanonPoint), cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        for (uint32_t i = 0; i < n; i++) encode_point(bls, group, compressed, z.fq, h[i], out + (base + i) * out_bytes);
    }
    return B2S_OK;
}

static void put_u64(uint8_t* o, uint64_t v) { for (int i = 0; i < 8; i++) o[i] = (uint8_t)(v >> (8 * i)); }

// A || B || C; HOST affine Montgomery
int32_t proof_serialize(Ctx* c, const void* a_g1, const void* b_g2, const void* c_g1, bool compressed, uint8_t* out, uint64_t cap) {
    const Sizes z = sizes(c);
    const size_t g1 = z.enc(1, compressed), g2 = z.enc(2, compressed);
    if (cap < 2 * g1 + g2) return fail(c, B2S_ERR_INVALID_ARG, "proof_serialize: output buffer too small");
    B2S_TRY(serialize_points_ex(c, 1, a_g1, B2S_MEM_HOST, 1, compressed, out, g1));
    B2S_TRY(serialize_points_ex(c, 2, b_g2, B2S_MEM_HOST, 1, compressed, out + g1, g2));
    return serialize_points_ex(c, 1, c_g1, B2S_MEM_HOST, 1, compressed, out + g1 + g2, g1);
}

uint64_t vk_serialized_size(Ctx* c, uint64_t n_gamma_abc, bool compressed) {
    return sizes(c).enc(1, compressed) * (1 + n_gamma_abc) + 3 * sizes(c).enc(2, compressed) + 8;
}
// alpha_g1, beta_g2, gamma_g2, delta_g2, Vec(gamma_abc_g1); all HOST affine Montgomery
int32_t vk_serialize(Ctx* c, const void* alpha_g1, const void* beta_g2, const void* gamma_g2, const void* delta_g2, const void* gamma_abc,
                     uint64_t n_gamma_abc, bool compressed, uint8_t* out, uint64_t cap) {
    if (vk_serialized_size(c, n_gamma_abc, compressed) > cap) return fail(c, B2S_ERR_INVALID_ARG, "vk_serialize: output buffer too small");
    const size_t g1 = sizes(c).enc(1, compressed), g2 = sizes(c).enc(2, compressed);
    uint8_t* o = out;
    B2S_TRY(serialize_points_ex(c, 1, alpha_g1, B2S_MEM_HOST, 1, compressed, o, g1)); o += g1;
    B2S_TRY(serialize_points_ex(c, 2, beta_g2, B2S_MEM_HOST, 1, compressed, o, g2)); o += g2;
    B2S_TRY(serialize_points_ex(c, 2, gamma_g2, B2S_MEM_HOST, 1, compressed, o, g2)); o += g2;
    B2S_TRY(serialize_points_ex(c, 2, delta_g2, B2S_MEM_HOST, 1, compressed, o, g2)); o += g2;
    put_u64(o, n_gamma_abc); o += 8;
    return serialize_points_ex(c, 1, gamma_abc, B2S_MEM_HOST, n_gamma_abc, compressed, o, g1 * n_gamma_abc);
}

}  // namespace b2s

#include "r1cs.cuh"
namespace b2s {

uint64_t pk_serialized_size(Ctx* c, const b2s_pk* pk, uint64_t vk_len, bool compressed) {
    const Sizes z = sizes(c);
    uint64_t n = vk_len + 2 * z.enc(1, compressed) + PK_QUERIES * 8;
    for (int w = 0; w < PK_QUERIES; w++) n += z.enc(PK_QUERY[w].group, compressed) * pk->q[w].len;
    return n;
}
// vk bytes (from vk_serialize) || beta_g1 || delta_g1 || the five query vectors of the device-resident FULL key
int32_t pk_serialize(Ctx* c, const b2s_pk* pk, const uint8_t* vk_bytes, uint64_t vk_len, bool compressed, uint8_t* out, uint64_t cap) {
    if (pk_serialized_size(c, pk, vk_len, compressed) > cap) return fail(c, B2S_ERR_INVALID_ARG, "pk_serialize: output buffer too small");
    if (!pk_is_full(pk)) return fail(c, B2S_ERR_MALFORMED_VK, "pk_serialize: needs a full (unsharded) proving key");
    const Sizes z = sizes(c);
    const size_t g1 = z.enc(1, compressed);
    uint8_t* o = out;
    memcpy(o, vk_bytes, vk_len); o += vk_len;
    const char* k1 = pk->consts_g1.as<char>();   // alpha, beta, delta
    B2S_TRY(serialize_points_ex(c, 1, k1 + z.g1, B2S_MEM_DEVICE, 1, compressed, o, g1)); o += g1;
    B2S_TRY(serialize_points_ex(c, 1, k1 + 2 * z.g1, B2S_MEM_DEVICE, 1, compressed, o, g1)); o += g1;
    for (int w = 0; w < PK_QUERIES; w++) {
        const PkQuery& q = pk->q[w];
        const int group = PK_QUERY[w].group;
        const size_t pb = z.enc(group, compressed);
        put_u64(o, q.len); o += 8;
        B2S_TRY(serialize_points_ex(c, group, q.pts.p, B2S_MEM_DEVICE, q.len, compressed, o, pb * q.len));
        o += pb * q.len;
    }
    return B2S_OK;
}

}  // namespace b2s
