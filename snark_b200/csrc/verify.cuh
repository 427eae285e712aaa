// The device-resident prepared verifying key and the chunking rule shared by the verify paths (verify.cu: one verdict per
// proof; verify_rlc.cu: one verdict per batch; verify_bytes.cu: both, from serialized proofs).
#pragma once
#include <algorithm>

#include "common.cuh"

namespace b2s {

// Public-input sum: per base g_j a table of [d 2^(8 w)] g_j, d = 1..255, w < 32 (affine), so a scalar costs at most 32
// mixed additions.  Memory per public input: 32 * 255 affine G1 points = 765 KiB (BLS12-381) / 510 KiB (BN254).
constexpr int IC_WBITS = 8, IC_WINDOWS = 32, IC_DIGITS = (1 << IC_WBITS) - 1;

constexpr int VERIFY_THREADS = 128;

// Device scratch for one chunk: host buffers are copied in, device buffers are used in place.
inline uint64_t chunk_size(uint64_t n, size_t per_proof) {
    constexpr uint64_t MAX_CHUNK = 1u << 18, SCRATCH = 1ull << 30;
    return std::max<uint64_t>(1, std::min<uint64_t>({n, MAX_CHUNK, SCRATCH / per_proof}));
}

// Bytes of one rho_i of the random-linear-combination check: a little-endian 128-bit integer.
constexpr size_t RLC_RHO = 16;

// The random-linear-combination check of verify_rlc.cu in steps, so that callers with their own staging (host points,
// decoded bytes) share it: rlc_begin, then rlc_chunk for each chunk of at most `ch` proofs with every buffer on the
// device (the last one also queues the verdict into *ok_dev), then rlc_read, the one read-back of the call.
struct RlcRun {
    Ctx* c = nullptr;
    const b2s_pvk* pvk = nullptr;
    const char* name = nullptr;   // prefix of the zero-rho error
    uint64_t ni = 0, ch = 0;
    DevBuf scratch, state;
    void *f = nullptr, *rho_fr = nullptr, *part = nullptr;                                 // per chunk
    void *prod = nullptr, *c_acc = nullptr, *c_chunk = nullptr, *st = nullptr;             // running values
    unsigned long long* zero_at = nullptr;
    uint8_t* ok_dev = nullptr;
};
size_t rlc_per_proof(Ctx* c);   // device bytes per proof of the chunk scratch rlc_begin allocates
int32_t rlc_begin(Ctx* c, const b2s_pvk* pvk, uint64_t ni, uint64_t ch, const char* name, RlcRun& r);
int32_t rlc_chunk(RlcRun& r, const void* x, const void* a, const void* b, const void* cc, const void* rho, uint32_t m, uint64_t base,
                  bool last);
int32_t rlc_read(RlcRun& r, uint8_t* ok);

}  // namespace b2s

struct b2s_pvk {
    int curve = 0;
    uint64_t n_abc = 0;
    b2s::DevBuf prep;    // G2Prepared[2]: -gamma, -delta
    b2s::DevBuf ab;      // e(alpha, beta) in GT
    b2s::DevBuf abc0;    // gamma_abc[0]
    b2s::DevBuf table;   // (n_abc - 1) x IC_WINDOWS x IC_DIGITS affine G1
};
