// CanonicalDeserialize of points, Proof, VerifyingKey and ProvingKey (the inverse of serialize.cu).  The raw bytes go to
// the device unchanged: flags, byte order, the canonicity check, the Montgomery conversion, the square root and the
// curve / subgroup checks all run in the decode kernel (deserialize.cuh).  The host reads only the Vec length prefixes and
// checks the bounds.  Input streams in chunks through two pinned staging buffers: the copy of chunk k + 1 (side stream)
// overlaps the decoding of chunk k (ctx stream), and points land directly in their final device arrays -- for a proving
// key the b2s_pk query buffers.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>

#include "common.cuh"
#include "deserialize.cuh"
#include "r1cs.cuh"
#include "stager.cuh"

namespace b2s {

int32_t pk_finish(Ctx* c, b2s_pk* pk);   // groth16.cu

int32_t deserialize_points(Ctx* c, int group, const uint8_t* in, uint64_t len, uint64_t count, bool compressed, bool validate,
                           void* out_host) {
    const size_t pb = sizes(c).enc(group, compressed);
    if (count > len / pb || count * pb != len)
        return fail(c, B2S_ERR_INVALID_DATA, "deserialize: %llu bytes are not %llu points of %zu bytes", (unsigned long long)len,
                    (unsigned long long)count, pb);
    Stager st(c);
    return st.decode_host(group, in, count, compressed, validate, out_host, group == 1 ? "g1" : "g2");
}

int32_t proof_deserialize(Ctx* c, const uint8_t* in, uint64_t len, bool compressed, bool validate, void* a, void* b, void* cc) {
    const size_t g1 = sizes(c).enc(1, compressed), g2 = sizes(c).enc(2, compressed);
    if (len != 2 * g1 + g2) return fail(c, B2S_ERR_INVALID_DATA, "proof: %llu bytes, expected %zu", (unsigned long long)len, 2 * g1 + g2);
    Stager st(c);
    B2S_TRY(st.decode_host(1, in, 1, compressed, validate, a, "proof.a"));
    B2S_TRY(st.decode_host(2, in + g1, 1, compressed, validate, b, "proof.b"));
    return st.decode_host(1, in + g1 + g2, 1, compressed, validate, cc, "proof.c");
}

// Walks the framing of a serialized key: every Vec prefix is checked against the bytes that remain before anything is
// allocated or decoded.
struct Frame {
    Ctx* c;
    const uint8_t* in;
    uint64_t len, at = 0;
    bool compressed;
    int32_t point(int group, uint64_t* off) {
        const size_t pb = sizes(c).enc(group, compressed);
        if (len - at < pb) return fail(c, B2S_ERR_INVALID_DATA, "key: truncated at byte %llu", (unsigned long long)at);
        *off = at;
        at += pb;
        return B2S_OK;
    }
    int32_t vec(int group, const char* name, uint64_t* off, uint64_t* n) {
        if (len - at < 8) return fail(c, B2S_ERR_INVALID_DATA, "key: truncated before the length of %s", name);
        uint64_t v = 0;
        for (int i = 0; i < 8; i++) v |= (uint64_t)in[at + i] << (8 * i);
        at += 8;
        const size_t pb = sizes(c).enc(group, compressed);
        if (v > (len - at) / pb)
            return fail(c, B2S_ERR_INVALID_DATA, "%s: length %llu exceeds the %llu bytes that remain", name, (unsigned long long)v,
                        (unsigned long long)(len - at));
        *off = at;
        *n = v;
        at += v * pb;
        return B2S_OK;
    }
};
struct VkFrame { uint64_t alpha, beta, gamma, delta, abc, n_abc; };
static int32_t frame_vk(Frame& f, VkFrame& v) {
    B2S_TRY(f.point(1, &v.alpha));
    B2S_TRY(f.point(2, &v.beta));
    B2S_TRY(f.point(2, &v.gamma));
    B2S_TRY(f.point(2, &v.delta));
    return f.vec(1, "gamma_abc_g1", &v.abc, &v.n_abc);
}

int32_t vk_deserialize(Ctx* c, const uint8_t* in, uint64_t len, bool compressed, bool validate, void* alpha, void* beta, void* gamma,
                       void* delta, void* abc, uint64_t cap_abc, uint64_t* n_abc, uint64_t* consumed) {
    Frame f{c, in, len, 0, compressed};
    VkFrame v;
    B2S_TRY(frame_vk(f, v));
    if (n_abc) *n_abc = v.n_abc;
    if (consumed) *consumed = f.at;
    if (!abc) return B2S_OK;
    if (cap_abc < v.n_abc) return fail(c, B2S_ERR_INVALID_ARG, "vk_deserialize: gamma_abc_g1 has %llu points, room for %llu",
                                       (unsigned long long)v.n_abc, (unsigned long long)cap_abc);
    Stager st(c);
    B2S_TRY(st.decode_host(1, in + v.alpha, 1, compressed, validate, alpha, "alpha_g1"));
    B2S_TRY(st.decode_host(2, in + v.beta, 1, compressed, validate, beta, "beta_g2"));
    B2S_TRY(st.decode_host(2, in + v.gamma, 1, compressed, validate, gamma, "gamma_g2"));
    B2S_TRY(st.decode_host(2, in + v.delta, 1, compressed, validate, delta, "delta_g2"));
    return st.decode_host(1, in + v.abc, v.n_abc, compressed, validate, abc, "gamma_abc_g1");
}

int32_t pk_deserialize(Ctx* c, const uint8_t* in, uint64_t len, bool compressed, bool validate, int32_t qap, b2s_pk** out) {
    Frame f{c, in, len, 0, compressed};
    VkFrame v;
    uint64_t beta1, delta1, at[PK_QUERIES], n[PK_QUERIES];
    B2S_TRY(frame_vk(f, v));
    B2S_TRY(f.point(1, &beta1));
    B2S_TRY(f.point(1, &delta1));
    for (int w = 0; w < PK_QUERIES; w++) B2S_TRY(f.vec(PK_QUERY[w].group, PK_QUERY[w].name, &at[w], &n[w]));
    if (f.at != len) return fail(c, B2S_ERR_INVALID_DATA, "pk: %llu trailing bytes", (unsigned long long)(len - f.at));
    // |h_query| = domain - 1 (libsnark) or domain (circom), the domain a power of two
    const uint64_t n_instance = v.n_abc, n_witness = n[Q_L], n_vars = n_instance + n_witness;
    const uint64_t domain = qap == B2S_QAP_CIRCOM ? n[Q_H] : n[Q_H] + 1;
    if (n[Q_A] != n_vars || n[Q_B_G1] != n_vars || n[Q_B_G2] != n_vars || domain == 0 || (domain & (domain - 1)))
        return fail(c, B2S_ERR_MALFORMED_VK, "pk: inconsistent dimensions (instance %llu, witness %llu, a %llu, b_g1 %llu, b_g2 %llu, h %llu)",
                    (unsigned long long)n_instance, (unsigned long long)n_witness, (unsigned long long)n[Q_A], (unsigned long long)n[Q_B_G1],
                    (unsigned long long)n[Q_B_G2], (unsigned long long)n[Q_H]);
    const size_t g1 = sizes(c).g1, g2 = sizes(c).g2;
    b2s_pk* pk = new b2s_pk();
    pk->n_instance = n_instance; pk->n_witness = n_witness; pk->domain_size = domain; pk->qap = qap;
    for (int w = 0; w < PK_QUERIES; w++) pk->q[w].len = n[w];   // a full key: every range starts at 0
    auto body = [&]() -> int32_t {
        Stager st(c);
        DevBuf scratch;   // gamma_g2 and gamma_abc_g1: validated, not kept by the prover
        B2S_TRY(scratch.alloc(c, std::max<size_t>(g2, std::max<uint64_t>(v.n_abc, 1) * g1)));
        B2S_TRY(pk->consts_g1.alloc(c, 3 * g1));
        B2S_TRY(pk->consts_g2.alloc(c, 2 * g2));
        char* k1 = pk->consts_g1.as<char>();
        char* k2 = pk->consts_g2.as<char>();
        B2S_TRY(st.decode(1, in + v.alpha, 1, compressed, validate, k1, "alpha_g1"));
        B2S_TRY(st.decode(2, in + v.beta, 1, compressed, validate, k2, "beta_g2"));
        B2S_TRY(st.decode(2, in + v.gamma, 1, compressed, validate, scratch.p, "gamma_g2"));
        B2S_TRY(st.decode(2, in + v.delta, 1, compressed, validate, k2 + g2, "delta_g2"));
        B2S_TRY(st.decode(1, in + v.abc, v.n_abc, compressed, validate, scratch.p, "gamma_abc_g1"));
        B2S_TRY(st.decode(1, in + beta1, 1, compressed, validate, k1 + g1, "beta_g1"));
        B2S_TRY(st.decode(1, in + delta1, 1, compressed, validate, k1 + 2 * g1, "delta_g1"));
        for (int w = 0; w < PK_QUERIES; w++) {   // room for the two extra points pk_finish appends
            const PkQueryInfo& info = PK_QUERY[w];
            DevBuf& b = pk->q[w].pts;
            B2S_TRY(b.alloc(c, (n[w] + 2) * sizes(c).aff(info.group)));
            B2S_TRY(st.decode(info.group, in + at[w], n[w], compressed, validate, b.p, info.name));
        }
        return pk_finish(c, pk);
    };
    const int32_t s = body();
    if (s != B2S_OK) { delete pk; return s; }
    *out = pk;
    return B2S_OK;
}

}  // namespace b2s
