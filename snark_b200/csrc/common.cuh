// Library-internal plumbing shared by the .cu translation units: the context object behind
// `b2s_ctx` (include/b200snark.h), error handling that never unwinds across the C ABI, stream-ordered
// device buffers and the kernel-launch counter that bench.py reports as `gpu_launches`.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/b200snark.h"
#include "curves.cuh"

namespace b2s {

struct NttPlan;  // ntt.cu
struct MsmDedupCache;  // msm.cu: classification of a scalar vector, shared by the MSMs of one proof that use the same scalars

struct Ctx {
    int curve = 0;
    int device = 0;
    cudaStream_t stream = nullptr;
    // second stream for latency-bound MSM tails (Horner) so they overlap the next MSM's bucket work
    cudaStream_t aux = nullptr;
    cudaEvent_t ev_tail = nullptr, ev_done = nullptr;
    // third stream: host-to-device copies of the point loader (deserialize.cu) overlap the decoding of the previous chunk
    cudaStream_t side = nullptr;
    bool aux_pending = false;
    std::mutex mu;
    std::string err;
    uint64_t launches = 0;
    int sm_count = 132;
    uint64_t total_mem = 0;     // device memory, queried once (cudaMemGetInfo costs milliseconds with a multi-GiB pool: not per MSM)
    std::map<uint32_t, NttPlan*> ntt_plans;   // keyed by log_n
    // optional per-kernel timing (b2s_profile_*): CUDA events around every launch on `stream`
    bool profiling = false;
    struct ProfRec { const char* name; cudaEvent_t e0, e1; };
    std::vector<ProfRec> prof;
    void* fixed_base_tables[2] = {nullptr, nullptr};  // G1 / G2 window tables (setup.cu)
    MsmDedupCache* dedup_cache = nullptr;             // non-null between msm_dedup_scope_begin / _end (one proof)
    // small buffers read by aux-stream kernels (heavy-list sums, tiny-rest products): a ring of persistent slots instead of
    // stream-ordered allocations freed on the other stream -- cross-stream frees make the pool insert dependencies between
    // the streams, and the main stream then stalls on the aux stream's work
    static constexpr size_t AUX_SLOT_BYTES = 16384, AUX_SLOTS = 16;
    void* aux_ring = nullptr;
    uint32_t aux_ring_next = 0;
    void* aux_slot() {
        void* p = static_cast<char*>(aux_ring) + (size_t)(aux_ring_next % AUX_SLOTS) * AUX_SLOT_BYTES;
        aux_ring_next++;
        return p;
    }
};

inline int32_t fail(Ctx* c, int32_t code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (c) c->err = buf;
    return code;
}

#define B2S_CUDA(ctx, expr)                                                                         \
    do {                                                                                            \
        cudaError_t e__ = (expr);                                                                   \
        if (e__ != cudaSuccess)                                                                     \
            return ::b2s::fail(ctx, e__ == cudaErrorMemoryAllocation ? B2S_ERR_OOM : B2S_ERR_CUDA, \
                               "%s:%d %s: %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e__)); \
    } while (0)

#define B2S_TRY(expr)                 \
    do {                              \
        int32_t s__ = (expr);         \
        if (s__ != B2S_OK) return s__; \
    } while (0)

// Launch + count + check.  Usage: B2S_LAUNCH(ctx, kernel<T>, grid, block, smem, args...)
#define B2S_LAUNCH(ctx, kern, grid, block, smem, ...) B2S_LAUNCH_N(ctx, #kern, kern, grid, block, smem, __VA_ARGS__)
#define B2S_LAUNCH_N(ctx, label, kern, grid, block, smem, ...) \
    B2S_LAUNCH_SN(ctx, (ctx)->stream, label, kern, grid, block, smem, __VA_ARGS__)
#define B2S_LAUNCH_SN(ctx, strm, label, kern, grid, block, smem, ...)                   \
    do {                                                                                \
        ::b2s::Ctx::ProfRec pr__{label, nullptr, nullptr};                              \
        if ((ctx)->profiling) {                                                         \
            cudaEventCreate(&pr__.e0);                                                  \
            cudaEventCreate(&pr__.e1);                                                  \
            cudaEventRecord(pr__.e0, (strm));                                    \
        }                                                                               \
        kern<<<(grid), (block), (smem), (strm)>>>(__VA_ARGS__);                  \
        (ctx)->launches++;                                                              \
        if ((ctx)->profiling) {                                                         \
            cudaEventRecord(pr__.e1, (strm));                                    \
            (ctx)->prof.push_back(pr__);                                                \
        }                                                                               \
        B2S_CUDA(ctx, cudaGetLastError());                                              \
    } while (0)

// Stream-ordered device allocation (cudaMallocAsync pool; freed on the same stream).
struct DevBuf {
    Ctx* ctx = nullptr;
    void* p = nullptr;
    size_t bytes = 0;
    bool secret = false;   // holds trapdoor-derived scalars: cleared before the block returns to the pool
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
    int32_t alloc(Ctx* c, size_t n) {
        release();
        ctx = c;
        bytes = n;
        if (n == 0) return B2S_OK;
        cudaError_t e = cudaMallocAsync(&p, n, c->stream);
        if (e != cudaSuccess) {
            p = nullptr;
            return fail(c, e == cudaErrorMemoryAllocation ? B2S_ERR_OOM : B2S_ERR_CUDA, "cudaMallocAsync(%zu): %s", n,
                        cudaGetErrorString(e));
        }
        return B2S_OK;
    }
    void release() {
        if (p && secret) cudaMemsetAsync(p, 0, bytes, ctx->stream);
        if (p) cudaFreeAsync(p, ctx->stream);
        p = nullptr;
        bytes = 0;
    }
    template <class T>
    T* as() const { return reinterpret_cast<T*>(p); }
};

// Where a caller buffer lives (`mem` of the C ABI): B2S_MEM_DEVICE is the ctx's GPU, any other value the host.
inline bool on_host(int32_t mem) { return mem != B2S_MEM_DEVICE; }
// the copy kind that brings a caller buffer in `mem` to the device
inline cudaMemcpyKind to_device(int32_t mem) { return on_host(mem) ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice; }

// Bring a caller buffer onto the device (copy if it lives on the host, alias if already there).
struct InBuf {
    DevBuf own;
    const void* dptr = nullptr;
    int32_t bind(Ctx* c, const void* src, size_t bytes, int32_t mem) {
        if (!on_host(mem)) { dptr = src; return B2S_OK; }
        B2S_TRY(own.alloc(c, bytes));
        if (bytes) B2S_CUDA(c, cudaMemcpyAsync(own.p, src, bytes, cudaMemcpyHostToDevice, c->stream));
        dptr = own.p;
        return B2S_OK;
    }
    template <class T>
    const T* as() const { return reinterpret_cast<const T*>(dptr); }
};

// A caller buffer the call writes, or with `in` reads and rewrites in place.  Device: dptr is the caller's pointer and
// finish() does nothing.  Host: dptr is stream-ordered scratch (with `in`, filled from the caller); finish() copies it to
// the caller and synchronises the stream, and copy_back() only queues the copy.
struct OutBuf {
    DevBuf own;
    void* dst = nullptr;
    void* dptr = nullptr;
    bool host = false;
    int32_t bind(Ctx* c, void* out, size_t bytes, int32_t mem, bool in = false) {
        dst = dptr = out;
        host = on_host(mem);
        if (!host) return B2S_OK;
        B2S_TRY(own.alloc(c, bytes));
        if (in && bytes) B2S_CUDA(c, cudaMemcpyAsync(own.p, out, bytes, cudaMemcpyHostToDevice, c->stream));
        dptr = own.p;
        return B2S_OK;
    }
    int32_t copy_back(Ctx* c) {
        if (host && own.bytes) B2S_CUDA(c, cudaMemcpyAsync(dst, own.p, own.bytes, cudaMemcpyDeviceToHost, c->stream));
        return B2S_OK;
    }
    int32_t finish(Ctx* c) {
        B2S_TRY(copy_back(c));
        if (host) B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        return B2S_OK;
    }
    template <class T>
    T* as() const { return reinterpret_cast<T*>(dptr); }
};

// One caller column of a batch: `bytes` per row, read by the work (`in`) or written by it (`out`).  A column with a null
// pointer or no bytes is absent: its device pointer is null and it takes no scratch.
struct Col {
    const void* in;
    void* out;
    size_t bytes;
};
inline Col col_in(const void* p, size_t bytes) { return {p, nullptr, bytes}; }
inline Col col_out(void* p, size_t bytes) { return {nullptr, p, bytes}; }

// The caller columns of a batch of rows, brought to the device one chunk at a time; the caller picks the chunk size.
// Device (staged == false): the pointers of chunk [base, base + m) are the caller's, `base` rows in, and row_bytes() is 0.
// Host: alloc(ch) takes one scratch allocation of ch * row_bytes() for chunks of up to ch rows, load(base, m) copies the
// chunk's rows of every input column into it, store() copies the output columns' rows back to the caller, one copy per
// column.  Copies are queued on the ctx stream; nothing synchronises.  Per-row scratch that is not a caller column is the
// caller's own.
struct RowStager {
    static constexpr int MAX_COLS = 5;
    Ctx* c;
    const bool staged;
    int n = 0;
    Col col[MAX_COLS];
    char* dev[MAX_COLS] = {};
    DevBuf scratch;
    uint64_t ch = 0, base = 0;
    uint32_t m = 0;
    RowStager(Ctx* ctx, int32_t mem, std::initializer_list<Col> cols) : c(ctx), staged(on_host(mem)) {
        for (const Col& k : cols) col[n++] = k;
    }
    static bool present(const Col& k) { return (k.in || k.out) && k.bytes; }
    size_t row_bytes() const {
        size_t r = 0;
        for (int k = 0; k < n; k++)
            if (staged && present(col[k])) r += col[k].bytes;
        return r;
    }
    int32_t alloc(uint64_t rows) {
        ch = rows;
        return scratch.alloc(c, ch * row_bytes());
    }
    int32_t load(uint64_t b, uint32_t rows) {
        base = b;
        m = rows;
        char* s = scratch.as<char>();
        for (int k = 0; k < n; k++) {
            const Col& q = col[k];
            if (!present(q)) { dev[k] = nullptr; continue; }
            const char* caller = static_cast<const char*>(q.in ? q.in : q.out) + base * q.bytes;
            if (!staged) { dev[k] = const_cast<char*>(caller); continue; }
            dev[k] = s;
            s += ch * q.bytes;
            if (q.in) B2S_CUDA(c, cudaMemcpyAsync(dev[k], caller, m * q.bytes, cudaMemcpyHostToDevice, c->stream));
        }
        return B2S_OK;
    }
    int32_t store() {
        for (int k = 0; k < n; k++)
            if (staged && present(col[k]) && col[k].out)
                B2S_CUDA(c, cudaMemcpyAsync(static_cast<char*>(col[k].out) + base * col[k].bytes, dev[k], m * col[k].bytes,
                                            cudaMemcpyDeviceToHost, c->stream));
        return B2S_OK;
    }
    template <class T = char>
    T* ptr(int k) const { return reinterpret_cast<T*>(dev[k]); }
};

// Kernels that need more than 48 KiB of dynamic shared memory: the attribute is per device, so it is (re)applied
// on every launch path rather than cached in a process-wide flag (a second ctx on another GPU needs it too).
#define B2S_SMEM_ATTR(ctx, kern, bytes) \
    B2S_CUDA(ctx, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes)))

// clears a host object holding secrets when the scope ends, whichever way it ends
struct HostWipe {
    void* p;
    size_t n;
    ~HostWipe() {
        volatile unsigned char* q = reinterpret_cast<volatile unsigned char*>(p);
        for (size_t i = 0; i < n; i++) q[i] = 0;
    }
};

inline unsigned cdiv(uint64_t a, uint64_t b) { return (unsigned)((a + b - 1) / b); }

// Per-curve dispatch helper: F is a generic lambda taking a curve tag.
template <class F>
inline int32_t dispatch_curve(Ctx* c, F&& f) {
    switch (c->curve) {
        case B2S_CURVE_BLS12_381: return f(Bls12_381{});
        case B2S_CURVE_BN254: return f(Bn254{});
        case B2S_CURVE_BLS12_377: return f(Bls12_377{});
    }
    return fail(c, B2S_ERR_INVALID_ARG, "unknown curve id %d", c->curve);
}

// Byte sizes of the ctx curve's elements as the kernels lay them out, in the order of b2s_sizes' out[6].
struct Sizes {
    size_t fr, fq, g1, g2, g1x, g2x;   // Fr, Fq, affine G1 / G2, XYZZ G1 / G2
    size_t aff(int group) const { return group == 1 ? g1 : g2; }
    size_t xyzz(int group) const { return group == 1 ? g1x : g2x; }
    // ark-serialize encoding of one point: x only when compressed, x || y otherwise
    size_t enc(int group, bool compressed) const { return compressed ? aff(group) / 2 : aff(group); }
};
inline Sizes sizes(const Ctx* c) {
    Sizes s{};
    // fail() writes the ctx only for an unknown curve, which b2s_ctx_create rejects
    dispatch_curve(const_cast<Ctx*>(c), [&](auto curve) {
        using C = decltype(curve);
        using Fq = typename C::Fq;
        static_assert(sizeof(typename C::G1Affine) == 2 * sizeof(Fq) && sizeof(typename C::G2Affine) == 4 * sizeof(Fq) &&
                          sizeof(typename C::G1) == 4 * sizeof(Fq) && sizeof(typename C::G2) == 8 * sizeof(Fq),
                      "the ABI points are packed coordinates: 2, 4, 4 and 8 Fq");
        s = {sizeof(typename C::Fr), sizeof(Fq), sizeof(typename C::G1Affine), sizeof(typename C::G2Affine), sizeof(typename C::G1),
             sizeof(typename C::G2)};
        return (int32_t)B2S_OK;
    });
    return s;
}

// ---- entry points implemented per translation unit (all take the ctx lock in api.cu) -----------
int32_t ntt_run(Ctx* c, void* data_dev, uint32_t log_n, bool inverse, bool coset);
void ntt_free_plans(Ctx* c);
// wins_ext == nullptr: the whole MSM runs on c->stream.  Otherwise wins_ext is caller-owned scratch for the
// window sums (>= 64 XYZZ points, alive until msm_join_tails): the Horner tail is queued on c->aux and the
// caller must call msm_join_tails(c) before reading out_xyzz_dev on c->stream.
// pre (optional): bases_dev is a precomputed table [pre->nwin][pre->stride] with row w = 2^(pre->c w) * (row 0), see msm_precompute
struct MsmPre { uint32_t c, nwin; uint32_t stride; };
int32_t msm_run(Ctx* c, int group, const void* bases_dev, const void* scalars_dev, uint64_t n, bool scalars_mont,
                void* out_xyzz_dev, void* wins_ext = nullptr, const MsmPre* pre = nullptr);
// K scalar vectors over the same n bases (vector k at scalars_dev + k * stride scalars): out_xyzz_dev[k] = MSM of vector k.
// One Pippenger problem on c->stream, so the launches do not grow with K; no multiplicity-aware front end.
int32_t msm_run_batch(Ctx* c, int group, const void* bases_dev, const void* scalars_dev, uint64_t n, uint64_t stride, uint32_t K,
                      bool scalars_mont, void* out_xyzz_dev, const MsmPre* pre = nullptr);
// device bytes per vector of msm_run_batch over n points; *max_k = the most vectors its u32 indices allow
uint64_t msm_batch_bytes(Ctx* c, int group, uint64_t n, const MsmPre* pre, uint64_t* max_k);
// device bytes of one msm_run over n points while it sorts, and what its batched-affine rounds add when they run in one piece
void msm_working_set(Ctx* c, int group, uint64_t n, const MsmPre* pre, uint64_t* sort_bytes, uint64_t* round_bytes);
// bytes the stream-ordered pool holds but no allocation uses (free for the next allocation, not counted by cudaMemGetInfo)
uint64_t pool_idle_bytes(Ctx* c);
// table[w * n + i] = 2^(c w) bases[i] (affine), w < nwin; picks c / nwin for n points itself and reports them in *pre
int32_t msm_precompute(Ctx* c, int group, const void* bases_dev, uint64_t n, void* table_dev, MsmPre* pre);
uint32_t msm_precompute_windows(Ctx* c, uint64_t n, uint32_t* c_out);
int32_t msm_join_tails(Ctx* c);
// a, b_g1 and b_g2 of a proof are MSMs over the SAME scalar vector: inside a scope the multiplicity-aware front end
// classifies a (pointer, length) pair once and the following MSMs reuse the lists (no second sample / count round trip)
void msm_dedup_scope_begin(Ctx* c);
void msm_dedup_scope_end(Ctx* c);
int32_t scan_counts(Ctx* c, const uint32_t* counts, uint32_t n, uint32_t L, uint32_t* offsets, uint32_t* task_off);
int32_t fixed_base_run(Ctx* c, int group, const void* scalars_dev, uint64_t n, bool mont, void* out_dev);
int32_t group_sum_to_affine(Ctx* c, int group, const void* xyzz_dev, uint32_t count, void* out_affine_dev);

}  // namespace b2s
