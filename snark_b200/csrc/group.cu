// Multi-GPU behind the C ABI: a `b2s_group` owns one NCCL communicator per rank (one process per GPU, or one host
// thread per GPU), so that a single call -- the backend of one `SNARK::prove`
// (/root/reference/snark/src/lib.rs:50-54) -- runs a proof over all the GPUs of a box (SURVEY.md 8(b), 8(e)).
//
// What is exchanged: the five MSMs of a proof are cut by base range, every rank holds a shard of the proving key
// and produces five partial sums (4 G1 + 1 G2 in XYZZ form, 1.2 KiB).  EC addition is not an NCCL reduction
// operator, so the join is ONE ncclAllGather of those device buffers on the ctx stream followed by a tiny
// summation kernel and the r/s epilogue on rank 0 -- no host bounce, no Python in the data plane.
//
// NCCL is bound at run time (dlopen of libnccl.so.2, the library the host program -- torch, or a Rust caller's
// own -- already has in the process): libb200snark.so keeps no link-time dependency on it, and single-GPU users never
// need it.
#include <dlfcn.h>
#include <nccl.h>

#include "dntt.cuh"
#include "r1cs.cuh"

using namespace b2s;

struct b2s_ctx : public b2s::Ctx {};

namespace {

struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    std::string err;
};

NcclApi* nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = {getenv("B2S_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* n : names) {
            if (!n) continue;
            api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (!api.handle) { api.err = "libnccl.so.2 not found (set B2S_NCCL_LIB)"; return; }
        auto sym = [&](const char* s) {
            void* p = dlsym(api.handle, s);
            if (!p && api.err.empty()) api.err = std::string("NCCL symbol missing: ") + s;
            return p;
        };
        api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
        api.Send = (decltype(api.Send))sym("ncclSend");
        api.Recv = (decltype(api.Recv))sym("ncclRecv");
        api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
        api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
        api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    });
    return &api;
}

}  // namespace

struct b2s_group {
    b2s_ctx* ctx = nullptr;
    ncclComm_t comm = nullptr;
    int rank = 0, world = 1;
    // whether every rank's (key shard, matrices) pair allows the distributed witness map; agreed once per pair
    const b2s_pk* agreed_pk = nullptr;
    const b2s_r1cs* agreed_m = nullptr;
    bool agreed_dist = false;
};

#define B2S_NCCL(ctx, expr)                                                                                   \
    do {                                                                                                      \
        ncclResult_t r__ = (expr);                                                                            \
        if (r__ != ncclSuccess)                                                                               \
            return ::b2s::fail(ctx, B2S_ERR_NCCL, "%s:%d %s: %s", __FILE__, __LINE__, #expr, nccl_api()->GetErrorString(r__)); \
    } while (0)

// all-to-all of the distributed witness map: NCCL point-to-point pairs fused into one group per batch of vectors
struct NcclExchange : DistExchange {
    b2s_group* g;
    bool open = false;
    explicit NcclExchange(b2s_group* grp) : g(grp) {}
    int32_t all_to_all(Ctx* c, const void* const* send, void* const* recv, size_t blk, bool flush) override {
        NcclApi* api = nccl_api();
        const char* s = reinterpret_cast<const char*>(send[0]);
        char* d = reinterpret_cast<char*>(recv[0]);
        if (!open) { B2S_NCCL(c, api->GroupStart()); open = true; }
        for (int peer = 0; peer < g->world; peer++) {
            if (peer == g->rank) {
                B2S_CUDA(c, cudaMemcpyAsync(d + (size_t)peer * blk, s + (size_t)peer * blk, blk, cudaMemcpyDeviceToDevice, c->stream));
            } else {
                B2S_NCCL(c, api->Send(s + (size_t)peer * blk, blk, ncclChar, peer, g->comm, c->stream));
                B2S_NCCL(c, api->Recv(d + (size_t)peer * blk, blk, ncclChar, peer, g->comm, c->stream));
            }
        }
        if (flush) { open = false; B2S_NCCL(c, api->GroupEnd()); }
        return B2S_OK;
    }
};

// h of this rank's coefficient slab, computed by all ranks together (dntt.cu)
struct DistributedH : HSource {
    b2s_group* g;
    uint32_t lg;
    DevBuf slab;
    DistributedH(b2s_group* grp, uint32_t lg_) : g(grp), lg(lg_) {}
    int32_t get(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void** h_for_shard) override {
        B2S_TRY(slab.alloc(c, (size_t)32 << (m->log_domain - lg)));
        NcclExchange x(g);
        std::vector<uint32_t> ranks{(uint32_t)g->rank};
        void* out[1] = {slab.p};
        B2S_TRY(witness_map_dist(c, m, z_dev, lg, ranks, &x, out));
        (void)pk;
        *h_for_shard = slab.p;    // the shard is the slab (checked by slab_aligned below)
        return B2S_OK;
    }
};

static bool slab_aligned(const b2s_pk* pk, const b2s_r1cs* m, int rank, int world) {
    const uint64_t N = 1ull << m->log_domain, per = N / (uint64_t)world, off = per * (uint64_t)rank;
    const uint64_t len = std::min<uint64_t>(per, N - 1 - off);
    return pk->q[Q_H].off == off && pk->q[Q_H].len == len;
}

namespace b2s {
// groth16.cu
int32_t groth16_finish_strided(Ctx* c, const b2s_pk* pk, const void* packed_dev, uint32_t n_shards, const void* r_host, const void* s_host,
                               void* out_a, void* out_b, void* out_c);
}  // namespace b2s

static int32_t prove_group(b2s_group* g, const b2s_pk* pk, const b2s_r1cs* m, const void* z_inst, const void* z_wit, const void* z_dev,
                           const void* r, const void* s, void* out_a, void* out_b, void* out_c) {
    b2s_ctx* ctx = g->ctx;
    if (!pk || !m) return fail(ctx, B2S_ERR_MISSING_CS, "prove_group: null key or matrices");
    if ((!z_dev && (!z_inst || (!z_wit && m->n_witness))) || !r || !s) return fail(ctx, B2S_ERR_ASSIGNMENT_MISSING, "prove_group: null assignment");
    if (g->rank == 0 && (!out_a || !out_b || !out_c)) return fail(ctx, B2S_ERR_INVALID_ARG, "prove_group: rank 0 needs the proof buffers");
    if (pk->qap != B2S_QAP_LIBSNARK)
        return fail(ctx, B2S_ERR_INVALID_ARG, "prove_group: circom keys have no distributed witness map; prove with b2s_groth16_prove_shard "
                                              "on each rank and join with b2s_groth16_finish");
    const Sizes z = sizes(ctx);
    const size_t p1 = z.g1x, p2 = z.g2x, per = 4 * p1 + p2;   // XYZZ sizes; one rank's packet
    DevBuf mine, all;
    B2S_TRY(mine.alloc(ctx, per));
    B2S_TRY(all.alloc(ctx, per * (size_t)g->world));
    // distributed witness map when every rank can (power-of-two group, even log2 of the domain, h-query shards = slabs);
    // the ranks agree once per (key shard, matrices) pair with a 4-byte all-gather
    uint32_t lg = 0;
    while ((1 << lg) < g->world) lg++;
    if (g->world > 1 && (g->agreed_pk != pk || g->agreed_m != m)) {
        const int32_t mine_ok = ((1 << lg) == g->world && dist_supported(m->log_domain, lg) && slab_aligned(pk, m, g->rank, g->world)) ? 1 : 0;
        DevBuf flags;
        B2S_TRY(flags.alloc(ctx, sizeof(int32_t) * (size_t)(g->world + 1)));
        int32_t* fd = flags.as<int32_t>();
        B2S_CUDA(ctx, cudaMemcpyAsync(fd + g->world, &mine_ok, sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
        B2S_NCCL(ctx, nccl_api()->AllGather(fd + g->world, fd, sizeof(int32_t), ncclChar, g->comm, ctx->stream));
        std::vector<int32_t> all_ok((size_t)g->world);
        B2S_CUDA(ctx, cudaMemcpyAsync(all_ok.data(), fd, sizeof(int32_t) * (size_t)g->world, cudaMemcpyDeviceToHost, ctx->stream));
        B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        g->agreed_dist = std::all_of(all_ok.begin(), all_ok.end(), [](int32_t v) { return v == 1; });
        g->agreed_pk = pk;
        g->agreed_m = m;
    }
    DistributedH dist_h(g, lg);
    HSource* hs = (g->world > 1 && g->agreed_dist) ? &dist_h : nullptr;
    B2S_TRY(groth16_shard(ctx, pk, m, z_inst, z_wit, z_dev, r, s, mine.p, mine.as<char>() + 4 * p1, hs));
    if (g->world > 1) {
        B2S_NCCL(ctx, nccl_api()->AllGather(mine.p, all.p, per, ncclChar, g->comm, ctx->stream));
    } else {
        B2S_CUDA(ctx, cudaMemcpyAsync(all.p, mine.p, per, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    if (g->rank != 0) {
        B2S_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        return B2S_OK;
    }
    return groth16_finish_strided(ctx, pk, all.p, (uint32_t)g->world, r, s, out_a, out_b, out_c);
}

extern "C" {

int32_t b2s_group_unique_id(uint8_t out[B2S_GROUP_ID_BYTES]) {
    static_assert(sizeof(ncclUniqueId) == B2S_GROUP_ID_BYTES, "ncclUniqueId is 128 bytes");
    if (!out) return B2S_ERR_INVALID_ARG;
    NcclApi* api = nccl_api();
    if (!api->err.empty()) return B2S_ERR_NCCL;
    ncclUniqueId id;
    if (api->GetUniqueId(&id) != ncclSuccess) return B2S_ERR_NCCL;
    memcpy(out, &id, sizeof(id));
    return B2S_OK;
}

int32_t b2s_group_create(b2s_ctx* ctx, const uint8_t id[B2S_GROUP_ID_BYTES], int32_t rank, int32_t world, b2s_group** out) {
    if (!ctx || !out) return B2S_ERR_INVALID_ARG;
    *out = nullptr;
    std::lock_guard<std::mutex> guard(ctx->mu);
    if (world < 1 || rank < 0 || rank >= world) return fail(ctx, B2S_ERR_INVALID_ARG, "group: rank %d of %d", rank, world);
    if (cudaSetDevice(ctx->device) != cudaSuccess) return fail(ctx, B2S_ERR_NO_DEVICE, "cudaSetDevice(%d) failed", ctx->device);
    b2s_group* g = new b2s_group();
    g->ctx = ctx; g->rank = rank; g->world = world;
    if (world > 1) {
        NcclApi* api = nccl_api();
        if (!api->err.empty()) { delete g; return fail(ctx, B2S_ERR_NCCL, "%s", api->err.c_str()); }
        if (!id) { delete g; return fail(ctx, B2S_ERR_INVALID_ARG, "group: null id"); }
        ncclUniqueId uid;
        memcpy(&uid, id, sizeof(uid));
        ncclResult_t r = api->CommInitRank(&g->comm, world, uid, rank);
        if (r != ncclSuccess) { delete g; return fail(ctx, B2S_ERR_NCCL, "ncclCommInitRank: %s", api->GetErrorString(r)); }
    }
    *out = g;
    return B2S_OK;
}

void b2s_group_destroy(b2s_group* g) {
    if (!g) return;
    if (g->comm) {
        cudaSetDevice(g->ctx->device);
        cudaStreamSynchronize(g->ctx->stream);
        nccl_api()->CommDestroy(g->comm);
    }
    delete g;
}

int32_t b2s_groth16_prove_group(b2s_group* g, const b2s_pk* pk_shard, const b2s_r1cs* m, const void* z_instance, const void* z_witness,
                                const void* r, const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    if (!g) return B2S_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> guard(g->ctx->mu);
    if (cudaSetDevice(g->ctx->device) != cudaSuccess) return fail(g->ctx, B2S_ERR_NO_DEVICE, "cudaSetDevice(%d) failed", g->ctx->device);
    return prove_group(g, pk_shard, m, z_instance, z_witness, nullptr, r, s, out_a_g1, out_b_g2, out_c_g1);
}

int32_t b2s_groth16_prove_group_resident(b2s_group* g, const b2s_pk* pk_shard, const b2s_r1cs* m, const void* z_dev, const void* r,
                                         const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1) {
    if (!g) return B2S_ERR_INVALID_ARG;
    std::lock_guard<std::mutex> guard(g->ctx->mu);
    if (cudaSetDevice(g->ctx->device) != cudaSuccess) return fail(g->ctx, B2S_ERR_NO_DEVICE, "cudaSetDevice(%d) failed", g->ctx->device);
    return prove_group(g, pk_shard, m, nullptr, nullptr, z_dev, r, s, out_a_g1, out_b_g2, out_c_g1);
}

}  // extern "C"
