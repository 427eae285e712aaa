// The device-resident prepared verifying key and the chunking rule shared by the verify paths (verify.cu: one verdict per
// proof; verify_rlc.cu: one verdict per batch).
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

}  // namespace b2s

struct b2s_pvk {
    int curve = 0;
    uint64_t n_abc = 0;
    b2s::DevBuf prep;    // G2Prepared[2]: -gamma, -delta
    b2s::DevBuf ab;      // e(alpha, beta) in GT
    b2s::DevBuf abc0;    // gamma_abc[0]
    b2s::DevBuf table;   // (n_abc - 1) x IC_WINDOWS x IC_DIGITS affine G1
};
