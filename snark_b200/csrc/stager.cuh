// Host-to-device streaming of large host inputs (serialized keys, snarkjs files) in chunks through two pinned staging
// buffers: the copy of chunk k + 1 (side stream) overlaps the kernel that consumes chunk k (ctx stream).  Shared by the
// ark-serialize readers (deserialize.cu) and the snarkjs readers (zkey.cu).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <utility>

#include "common.cuh"
#include "deserialize.cuh"

namespace b2s {

// MONT = false: ark-serialize encodings (decode_point); true: snarkjs Montgomery limbs (decode_point_mont)
template <class Curve, class F, bool MONT>
__global__ void decode_points_kernel(const uint8_t* in, uint32_t n, uint32_t pb, int compressed, int validate, uint64_t base,
                                     Affine<F>* out, unsigned long long* err) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    Affine<F> p = Affine<F>::inf();
    const uint32_t st = MONT ? decode_point_mont<Curve, F>(in + (size_t)i * pb, validate != 0, p)
                             : decode_point<Curve, F>(in + (size_t)i * pb, compressed != 0, validate != 0, p);
    if (st != DEC_OK) {
        atomicMin(err, (unsigned long long)((base + i) << 3 | st));   // lowest failing index, with its reason
        p = Affine<F>::inf();
    }
    out[i] = p;
}

inline const char* reason_text(uint32_t st) {
    switch (st) {
        case DEC_BAD_FLAGS: return "bad flags";
        case DEC_NONCANONICAL: return "coordinate not below p";
        case DEC_NOT_ON_CURVE: return "not on the curve";
        case DEC_NOT_IN_SUBGROUP: return "not in the prime-order subgroup";
    }
    return "invalid";
}

// Two pinned host buffers and two device buffers, reused by every vector of one call.
struct Stager {
    static constexpr uint64_t CH = 1u << 18;   // items per chunk
    Ctx* c;
    size_t cap = 0;
    uint8_t* pinned[2] = {nullptr, nullptr};
    DevBuf dev[2], err;
    cudaEvent_t copied[2] = {nullptr, nullptr}, consumed[2] = {nullptr, nullptr};
    explicit Stager(Ctx* ctx) : c(ctx) {}
    ~Stager() {
        cudaStreamSynchronize(c->side);
        cudaStreamSynchronize(c->stream);
        for (int s = 0; s < 2; s++) {
            if (pinned[s]) cudaFreeHost(pinned[s]);
            if (copied[s]) cudaEventDestroy(copied[s]);
            if (consumed[s]) cudaEventDestroy(consumed[s]);
        }
    }
    int32_t reserve(size_t bytes) {
        if (!err.p) {
            B2S_TRY(err.alloc(c, sizeof(unsigned long long)));
            for (int s = 0; s < 2; s++) {
                B2S_CUDA(c, cudaEventCreateWithFlags(&copied[s], cudaEventDisableTiming));
                B2S_CUDA(c, cudaEventCreateWithFlags(&consumed[s], cudaEventDisableTiming));
            }
        }
        if (bytes <= cap) return B2S_OK;
        B2S_CUDA(c, cudaStreamSynchronize(c->side));
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        for (int s = 0; s < 2; s++) {
            if (pinned[s]) cudaFreeHost(pinned[s]);
            pinned[s] = nullptr;
            B2S_CUDA(c, cudaMallocHost(&pinned[s], bytes));
            B2S_TRY(dev[s].alloc(c, bytes));
        }
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));   // the side stream copies into dev[] allocated on the ctx stream
        cap = bytes;
        return B2S_OK;
    }

    // `count` items of `pb` bytes from the HOST, CH at a time: launch(src_dev, n, base) queues on the ctx stream the kernel
    // that consumes items [base, base + n), staged at src_dev.  The error word `err` is set to ~0 first.
    template <class Launch>
    int32_t chunks(const uint8_t* in, uint64_t count, size_t pb, Launch&& launch) {
        B2S_TRY(reserve((size_t)std::min<uint64_t>(count, CH) * pb));
        return copy_loop<true>(in, (count + CH - 1) / CH, pb,
                               [&](uint64_t k) { return std::make_pair(k * CH * pb, std::min<uint64_t>(CH, count - k * CH) * pb); }, launch);
    }
    // Variable-length items from the HOST: span j is bytes [cut[j], cut[j + 1]) of `in`, j < n_spans, chosen by the caller
    // (runs of whole items, about a chunk's worth each).  The buffers are reserved for the longest span, so one item longer
    // than a chunk still goes in one piece.  launch(src_dev, j) queues the kernel that consumes span j, staged at src_dev.
    // The error word `err` is set to ~0 first.
    template <class Launch>
    int32_t spans(const uint8_t* in, const uint64_t* cut, uint64_t n_spans, Launch&& launch) {
        uint64_t longest = 0;
        for (uint64_t j = 0; j < n_spans; j++) longest = std::max(longest, cut[j + 1] - cut[j]);
        B2S_TRY(reserve((size_t)longest));
        return copy_loop<false>(in, n_spans, 0, [&](uint64_t j) { return std::make_pair(cut[j], cut[j + 1] - cut[j]); }, launch);
    }
    // the copy / launch pipeline of chunks and spans: piece k is span(k) = (offset, bytes) of `in`, at most cap bytes, consumed
    // by launch(src_dev, items, first item) of pb-byte items (ITEMS) or by launch(src_dev, k)
    template <bool ITEMS, class Span, class Launch>
    int32_t copy_loop(const uint8_t* in, uint64_t n_pieces, size_t pb, Span&& span, Launch&& launch) {
        B2S_CUDA(c, cudaMemsetAsync(err.p, 0xFF, sizeof(unsigned long long), c->stream));
        for (uint64_t k = 0; k < n_pieces; k++) {
            const int s = (int)(k & 1);
            const auto [off, n] = span(k);
            if (k >= 2) B2S_CUDA(c, cudaEventSynchronize(copied[s]));   // pinned[s] is free again
            memcpy(pinned[s], in + off, (size_t)n);
            if (k >= 2) B2S_CUDA(c, cudaStreamWaitEvent(c->side, consumed[s], 0));   // dev[s] has been consumed
            B2S_CUDA(c, cudaMemcpyAsync(dev[s].p, pinned[s], (size_t)n, cudaMemcpyHostToDevice, c->side));
            B2S_CUDA(c, cudaEventRecord(copied[s], c->side));
            B2S_CUDA(c, cudaStreamWaitEvent(c->stream, copied[s], 0));
            if constexpr (ITEMS) B2S_TRY(launch(dev[s].as<const uint8_t>(), (uint32_t)(n / pb), off / pb));
            else B2S_TRY(launch(dev[s].as<const uint8_t>(), k));
            B2S_CUDA(c, cudaEventRecord(consumed[s], c->stream));
        }
        return B2S_OK;
    }
    // the error word after the last chunk (~0 = none)
    int32_t read_err(unsigned long long* word) {
        B2S_CUDA(c, cudaMemcpyAsync(word, err.p, sizeof(*word), cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        return B2S_OK;
    }

    // `count` encodings from the HOST -> affine Montgomery points at out_dev; `name` labels the error message.  MONT: the
    // snarkjs form (decode_point_mont), `compressed` ignored
    template <bool MONT = false>
    int32_t decode(int group, const uint8_t* in, uint64_t count, bool compressed, bool validate, void* out_dev, const char* name) {
        if (!count) return B2S_OK;
        const size_t pb = MONT ? sizes(c).aff(group) : sizes(c).enc(group, compressed), ab = sizes(c).aff(group);
        B2S_TRY(chunks(in, count, pb, [&](const uint8_t* src, uint32_t n, uint64_t base) {
            unsigned long long* e = err.as<unsigned long long>();
            char* dst = static_cast<char*>(out_dev) + base * ab;
            return dispatch_curve(c, [&](auto curve) {
                using C = decltype(curve);
                if (group == 1) {
                    auto kern = decode_points_kernel<C, typename C::Fq, MONT>;
                    B2S_LAUNCH_N(c, "decode_points_g1", kern, cdiv(n, 128), 128, 0, src, n, (uint32_t)pb, (int)compressed, (int)validate,
                                 base, reinterpret_cast<Affine<typename C::Fq>*>(dst), e);
                } else {
                    auto kern = decode_points_kernel<C, typename C::Fq2, MONT>;
                    B2S_LAUNCH_N(c, "decode_points_g2", kern, cdiv(n, 128), 128, 0, src, n, (uint32_t)pb, (int)compressed, (int)validate,
                                 base, reinterpret_cast<Affine<typename C::Fq2>*>(dst), e);
                }
                return (int32_t)B2S_OK;
            });
        }));
        unsigned long long word = 0;
        B2S_TRY(read_err(&word));
        if (word != ~0ull)
            return fail(c, B2S_ERR_INVALID_DATA, "%s[%llu]: %s", name, (unsigned long long)(word >> 3), reason_text((uint32_t)(word & 7)));
        return B2S_OK;
    }
    // the same into HOST memory
    template <bool MONT = false>
    int32_t decode_host(int group, const uint8_t* in, uint64_t count, bool compressed, bool validate, void* out_host, const char* name) {
        if (!count) return B2S_OK;
        DevBuf out;
        B2S_TRY(out.alloc(c, count * sizes(c).aff(group)));
        B2S_TRY(decode<MONT>(group, in, count, compressed, validate, out.p, name));
        B2S_CUDA(c, cudaMemcpyAsync(out_host, out.p, count * sizes(c).aff(group), cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
        return B2S_OK;
    }
};

}  // namespace b2s
