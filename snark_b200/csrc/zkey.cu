// Readers of the three files a circom user has: the Groth16 .zkey written by `snarkjs groth16 setup` / `zkey contribute`,
// the .wtns written by circom's witness generator and the circuit's .r1cs written by the circom compiler.  They stand in for
// ark-circom's `read_zkey` / `R1CSFile` and snarkjs's `zkey_utils.js` / `wtns_utils.js`, and give the handles
// b2s_pk_upload_qap(.., B2S_QAP_CIRCOM, ..) and b2s_r1cs_upload would build from the same points and matrices.
//
// The formats, restated from snarkjs, ark-circom and the iden3 r1cs binfile spec (none is in the reference tree, and no file
// written by snarkjs or circom is available here, so byte parity with them is NOT pinned -- tests/zkey_oracle.py and
// tests/r1cs_file_oracle.py restate the same writers):
//   binfile framing (all three files): 4-byte magic "zkey" / "wtns" / "r1cs", u32 LE version (zkey 1, wtns 2, r1cs 1), u32 LE
//     section count, then per section a u32 type, a u64 size and `size` bytes.  Sections may come in any order and are indexed
//     by type; unknown types and zkey section 10 (contributions) are skipped; a section this reader indexes that appears twice
//     is malformed.
//   zkey  1  u32 protocol: 1 = Groth16 (2 PLONK and 10 FFLONK are rejected)
//         2  n8q, q (n8q bytes LE), n8r, r, nVars, nPublic, domainSize (u32 each), then alpha1 (G1), beta1 (G1), beta2 (G2),
//            gamma2 (G2), delta1 (G1), delta2 (G2)
//         3  IC: nPublic + 1 G1 points (the verifying key's gamma_abc_g1)
//         4  coefficients: u32 count, then per entry u32 matrix (0 = A, 1 = B), u32 constraint, u32 signal and an n8r-byte value
//         5 / 6 / 7  A / B1 / B2: nVars points each (G1 / G1 / G2)
//         8  C: nVars - nPublic - 1 G1 points (ark's l_query)
//         9  H: domainSize G1 points, snarkjs's odd-coset Lagrange form -- exactly the B2S_QAP_CIRCOM h_query
//   points: toRprLEM, x then y (G2: x.c0, x.c1, y.c0, y.c1), each a Montgomery little-endian field element; infinity is all
//     zero bytes.  That is this library's affine layout (R = 2^(8 n8q) for every curve here): no byte swap, no square root.
//   coefficient values: c R^2 mod r in plain LE (for snarkjs's wasm prover); one Montgomery reduction gives the Montgomery
//     limbs of c, as ark-circom's deserialize_field_fr does with Fr::new_unchecked(Fr::new_unchecked(x).into_bigint()).
//   input rows: snarkjs appends the nPublic + 1 rows A[nConstraints + s] = 1 * z[s] (s = 0..nPublic) to the coefficients.  The
//     circom witness map copies z[s] into those rows itself (copy_instance_kernel), so the loader takes n_constraints =
//     (largest A row + 1) - (nPublic + 1), checks that the last nPublic + 1 A rows hold exactly (s, ONE) and that B has no
//     entry there, keeps rows [0, n_constraints) and requires domainSize = next_pow2(n_constraints + nPublic + 1).
//   wtns  1  n8, prime (n8 bytes LE), u32 nWitness
//         2  nWitness values, canonical LE (not Montgomery); nWitness = nVars and z[0] = 1
//   r1cs  1  header, exactly n8 + 32 bytes: u32 n8, the prime (n8 bytes LE), u32 nWires, nPubOut, nPubIn, nPrvIn, u64 nLabels,
//            u32 mConstraints
//         2  constraints: per constraint, for A, then B, then C, a u32 count and `count` x (u32 wire, n8-byte coefficient);
//            coefficients canonical LE (not Montgomery), each below r.  Constraint i: <A_i, z> <B_i, z> - <C_i, z> = 0 with z
//            in wire order (One, public outputs, public inputs, private inputs, internal wires).  Duplicate wires in one
//            linear combination are summed; empty combinations are allowed.
//         3  wire -> label map (optional): nWires u64, not read
//         4 / 5  PLONK custom gates: rejected
//     The handle: n_rows = mConstraints, n_instance = 1 + nPubOut + nPubIn, n_witness = nWires - n_instance, A, B, C filled.
//
// The host reads the file headers and section offsets only (for an .r1cs also the 3 m count words, the one sequential
// dependency of the file: they give each constraint's offset).  Points are checked in place by the decode kernel (stager.cuh,
// decode_point_mont); coefficient records are parsed, range-checked and reduced by one kernel per chunk, then sorted into CSR
// by row counts, a scan and a placement pass, which also checks the input rows.  Non-ONE coefficients get one pool entry each,
// compacted by a scan (no host-side interning: the sums are exact, whatever the order and the duplication).  An .r1cs is
// already in CSR order: its row pointers come from a scan of the walk's counts, and one kernel per run of whole constraints
// decodes, checks and places every entry.
#include <cuda_runtime.h>

#include <cstring>
#include <vector>

#include "common.cuh"
#include "deserialize.cuh"
#include "r1cs.cuh"
#include "stager.cuh"

namespace b2s {

int32_t pk_finish(Ctx* c, b2s_pk* pk);   // groth16.cu

namespace {

constexpr uint32_t FR_BYTES = 32;                  // n8r of every curve here
constexpr uint32_t ZKEY_REC = 12 + FR_BYTES;       // one coefficient record
enum ZkeySection { Z_PROTOCOL = 1, Z_HEADER, Z_IC, Z_COEFFS, Z_A, Z_B1, Z_B2, Z_C, Z_H, Z_SECTIONS = Z_H };
enum CoeffReason : uint32_t { CO_MATRIX = 1, CO_CONSTRAINT, CO_SIGNAL, CO_VALUE, CO_B_INPUT_ROW, CO_INPUT_ENTRY };

uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
uint64_t rd64(const uint8_t* p) { return (uint64_t)rd32(p) | (uint64_t)rd32(p + 4) << 32; }

struct Section { uint64_t off = 0, size = 0; bool seen = false; };

// Indexes a binfile: sections 1..n_types kept in sec[type] (each at most once), any other type skipped; sections
// 1..n_required must be present (n_required < 0: all n_types).  Every section must lie inside the `len` bytes and the last one
// must end there.
int32_t bin_sections(Ctx* c, const char* magic, const uint8_t* in, uint64_t len, uint32_t version, int n_types, Section* sec,
                     int n_required = -1) {
    if (len < 12 || memcmp(in, magic, 4) != 0) return fail(c, B2S_ERR_INVALID_DATA, "%s: bad magic (not a .%s file)", magic, magic);
    const uint32_t ver = rd32(in + 4), n = rd32(in + 8);
    if (ver != version) return fail(c, B2S_ERR_INVALID_DATA, "%s: version %u, expected %u", magic, ver, version);
    uint64_t at = 12;
    for (uint32_t k = 0; k < n; k++) {
        if (len - at < 12) return fail(c, B2S_ERR_INVALID_DATA, "%s: truncated in the header of section %u of %u", magic, k, n);
        const uint32_t type = rd32(in + at);
        const uint64_t size = rd64(in + at + 4);
        at += 12;
        if (size > len - at)
            return fail(c, B2S_ERR_INVALID_DATA, "%s: section %u holds %llu bytes, %llu remain", magic, type, (unsigned long long)size,
                        (unsigned long long)(len - at));
        if (type >= 1 && type <= (uint32_t)n_types) {
            if (sec[type].seen) return fail(c, B2S_ERR_INVALID_DATA, "%s: section %u appears twice", magic, type);
            sec[type] = {at, size, true};
        }
        at += size;
    }
    if (at != len) return fail(c, B2S_ERR_INVALID_DATA, "%s: %llu trailing bytes after the last section", magic, (unsigned long long)(len - at));
    for (int t = 1; t <= (n_required < 0 ? n_types : n_required); t++)
        if (!sec[t].seen) return fail(c, B2S_ERR_INVALID_DATA, "%s: section %d missing", magic, t);
    return B2S_OK;
}

// n8 bytes at b are the modulus of P
template <class P>
bool is_modulus(const uint8_t* b, uint32_t n8) {
    if (n8 != 4 * Fp<P>::N) return false;
    for (int i = 0; i < Fp<P>::N; i++)
        if (rd32(b + 4 * i) != P::mod(i)) return false;
    return true;
}

struct Zkey {
    Section s[Z_SECTIONS + 1];
    uint64_t n_vars = 0, n_public = 0, domain = 0, n_coeffs = 0;
    uint64_t coeffs = 0;   // offset of the first coefficient record
    uint64_t pt[6] = {};   // offsets of alpha1, beta1, beta2, gamma2, delta1, delta2
};

// framing, protocol, curve and dimensions: every check that needs no per-entry data
int32_t zkey_parse(Ctx* c, const uint8_t* in, uint64_t len, Zkey& z) {
    B2S_TRY(bin_sections(c, "zkey", in, len, 1, Z_SECTIONS, z.s));
    const Section& p = z.s[Z_PROTOCOL];
    if (p.size != 4) return fail(c, B2S_ERR_INVALID_DATA, "zkey: protocol section holds %llu bytes, expected 4", (unsigned long long)p.size);
    const uint32_t protocol = rd32(in + p.off);
    if (protocol != 1) return fail(c, B2S_ERR_INVALID_DATA, "zkey: protocol %u is not Groth16 (1)", protocol);
    const Section& h = z.s[Z_HEADER];
    const uint8_t* b = in + h.off;
    const uint32_t n8q = h.size >= 4 ? rd32(b) : 0;
    if (n8q == 0 || n8q > 64 || h.size < 8ull + n8q) return fail(c, B2S_ERR_INVALID_DATA, "zkey: truncated header section");
    const uint32_t n8r = rd32(b + 4 + n8q);
    if (n8r == 0 || n8r > 64 || h.size < 8ull + n8q + n8r) return fail(c, B2S_ERR_INVALID_DATA, "zkey: truncated header section");
    const bool same_curve = dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        return (int32_t)(is_modulus<typename C::FqP>(b + 4, n8q) && is_modulus<typename C::FrP>(b + 8 + n8q, n8r));
    }) == 1;
    if (!same_curve) return fail(c, B2S_ERR_INVALID_ARG, "zkey: q / r (%u / %u bytes) are not the fields of the ctx's curve", n8q, n8r);
    const Sizes sz = sizes(c);
    const uint64_t dims = 8ull + n8q + n8r;
    if (h.size != dims + 12 + 3 * sz.g1 + 3 * sz.g2)
        return fail(c, B2S_ERR_INVALID_DATA, "zkey: header section holds %llu bytes, expected %llu", (unsigned long long)h.size,
                    (unsigned long long)(dims + 12 + 3 * sz.g1 + 3 * sz.g2));
    z.n_vars = rd32(b + dims);
    z.n_public = rd32(b + dims + 4);
    z.domain = rd32(b + dims + 8);
    const size_t psz[6] = {sz.g1, sz.g1, sz.g2, sz.g2, sz.g1, sz.g2};
    uint64_t at = h.off + dims + 12;
    for (int i = 0; i < 6; i++) { z.pt[i] = at; at += psz[i]; }
    const Section& co = z.s[Z_COEFFS];
    if (co.size < 4) return fail(c, B2S_ERR_INVALID_DATA, "zkey: truncated coefficient section");
    z.n_coeffs = rd32(in + co.off);
    z.coeffs = co.off + 4;
    if (co.size != 4 + z.n_coeffs * ZKEY_REC)
        return fail(c, B2S_ERR_INVALID_DATA, "zkey: coefficient section holds %llu bytes, %llu entries need %llu", (unsigned long long)co.size,
                    (unsigned long long)z.n_coeffs, (unsigned long long)(4 + z.n_coeffs * ZKEY_REC));
    if (z.n_vars < z.n_public + 1)
        return fail(c, B2S_ERR_MALFORMED_VK, "zkey: nVars %llu < nPublic %llu + 1", (unsigned long long)z.n_vars, (unsigned long long)z.n_public);
    if (z.domain == 0 || (z.domain & (z.domain - 1)))
        return fail(c, B2S_ERR_MALFORMED_VK, "zkey: domainSize %llu is not a power of two", (unsigned long long)z.domain);
    uint32_t logd = 0;
    while ((1ull << logd) < z.domain) logd++;
    const uint32_t two_adicity = (uint32_t)dispatch_curve(c, [](auto curve) { return (int32_t)decltype(curve)::FrP::TWO_ADICITY; });
    if (logd > two_adicity || logd > 27)   // the limits of b2s_r1cs_upload
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "zkey: domain 2^%u unsupported", logd);
    const struct { int sec; const char* name; uint64_t want; } dim[] = {
        {Z_IC, "IC", (z.n_public + 1) * sz.g1}, {Z_A, "A", z.n_vars * sz.g1}, {Z_B1, "B1", z.n_vars * sz.g1},
        {Z_B2, "B2", z.n_vars * sz.g2}, {Z_C, "C", (z.n_vars - z.n_public - 1) * sz.g1}, {Z_H, "H", z.domain * sz.g1}};
    for (const auto& d : dim)
        if (z.s[d.sec].size != d.want)
            return fail(c, B2S_ERR_MALFORMED_VK, "zkey: section %d (%s) holds %llu bytes, nVars %llu / nPublic %llu / domainSize %llu need %llu",
                        d.sec, d.name, (unsigned long long)z.s[d.sec].size, (unsigned long long)z.n_vars, (unsigned long long)z.n_public,
                        (unsigned long long)z.domain, (unsigned long long)d.want);
    return B2S_OK;
}

// One thread per coefficient record of a chunk: range checks (lowest bad record index into err, with its CoeffReason), the
// Montgomery reduction c R^2 -> c R, and the per-(matrix, row) counts.  max_a1 = 1 + the largest A row.
template <class Curve>
__global__ void zkey_coeff_kernel(const uint8_t* __restrict__ src, uint32_t n, uint64_t base, uint32_t n_vars, uint32_t D,
                                  uint32_t* __restrict__ key, uint32_t* __restrict__ colv, typename Curve::Fr* __restrict__ val,
                                  uint32_t* __restrict__ nonone, uint32_t* __restrict__ counts, uint32_t* max_a1, unsigned long long* err) {
    using Fr = typename Curve::Fr;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(src + (size_t)i * ZKEY_REC);
    const uint32_t m = w[0], row = w[1], col = w[2];
    Fr v;
#pragma unroll
    for (int j = 0; j < Fr::N; j++) v.v[j] = w[3 + j];
    const uint64_t e = base + i;
    const uint32_t bad = m > 1 ? CO_MATRIX : row >= D ? CO_CONSTRAINT : col >= n_vars ? CO_SIGNAL : !dec::below_p(v) ? CO_VALUE : 0;
    if (bad) {
        atomicMin(err, (unsigned long long)(e << 3 | bad));
    } else {
        v = v.from_mont();
        key[e] = m << 31 | row;
        colv[e] = col;
        val[e] = v;
        nonone[e] = v != Fr::one();
        atomicAdd(&counts[(uint64_t)m * D + row], 1u);
    }
    const unsigned act = __activemask();
    const uint32_t mx = __reduce_max_sync(act, (!bad && m == 0) ? row + 1 : 0u);
    if ((threadIdx.x & 31) == (uint32_t)(__ffs(act) - 1) && mx) atomicMax(max_a1, mx);
}

struct CsrOut { uint64_t* row_ptr[2]; uint32_t* col[2]; uint32_t* cid[2]; };

// row_ptr of A and B over rows [0, n_c] from the scanned counts (matrix m's rows start at offsets[m D]), pool[0] = ONE, and
// the count of every input row (A row n_c + s must hold one entry): the lowest bad s into row_err
template <class Fr>
__global__ void zkey_rows_kernel(const uint32_t* __restrict__ offsets, uint32_t D, uint32_t n_c, uint32_t n_inst, CsrOut o, Fr* pool,
                                 uint32_t* row_err) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t rows = (uint64_t)n_c + 1;
    if (t < 2 * rows) {
        const uint32_t m = (uint32_t)(t / rows);
        const uint64_t r = t - m * rows;
        o.row_ptr[m][r] = (uint64_t)(offsets[(uint64_t)m * D + r] - offsets[(uint64_t)m * D]);
    }
    if (t < n_inst && offsets[n_c + t + 1] - offsets[n_c + t] != 1) atomicMin(row_err, (uint32_t)t);
    if (t == 0) pool[0] = Fr::one();
}

// One thread per record: rows below n_c go to their CSR slot (cursor: a copy of offsets, advanced atomically; the order
// within a row does not matter), with coefficient id 0 for ONE and 1 + pool_off[e] otherwise.  Records in the input rows
// are checked instead: B must have none, A only (s, ONE) in row n_c + s.
template <class Fr>
__global__ void zkey_place_kernel(uint32_t N, const uint32_t* __restrict__ key, const uint32_t* __restrict__ colv, const Fr* __restrict__ val,
                                  const uint32_t* __restrict__ nonone, const uint32_t* __restrict__ pool_off, uint32_t* cursor,
                                  const uint32_t* __restrict__ offsets, uint32_t D, uint32_t n_c, CsrOut o, Fr* pool, unsigned long long* err) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= N) return;
    const uint32_t k = key[e], m = k >> 31, row = k & 0x7FFFFFFFu;
    if (row >= n_c) {
        if (m == 1) atomicMin(err, (unsigned long long)e << 3 | CO_B_INPUT_ROW);
        else if (colv[e] != row - n_c || nonone[e]) atomicMin(err, (unsigned long long)e << 3 | CO_INPUT_ENTRY);
        return;
    }
    const uint64_t mb = (uint64_t)m * D;
    const uint32_t at = atomicAdd(&cursor[mb + row], 1u) - offsets[mb];
    o.col[m][at] = colv[e];
    uint32_t id = 0;
    if (nonone[e]) {
        id = 1 + pool_off[e];
        pool[id] = val[e];
    }
    o.cid[m][at] = id;
}

const char* coeff_reason(uint32_t r) {
    switch (r) {
        case CO_MATRIX: return "matrix is neither 0 (A) nor 1 (B)";
        case CO_CONSTRAINT: return "constraint not below domainSize";
        case CO_SIGNAL: return "signal not below nVars";
        case CO_VALUE: return "value not below r";
        case CO_B_INPUT_ROW: return "a B entry in an input row";
        case CO_INPUT_ENTRY: return "an input row entry other than (s, 1)";
    }
    return "invalid";
}

// The matrix handle from the coefficient section: A and B in CSR over rows [0, n_c), C empty (the circom witness map never
// reads it).
template <class Curve>
int32_t zkey_matrices(Ctx* c, Stager& st, const uint8_t* in, const Zkey& z, b2s_r1cs* m) {
    using Fr = typename Curve::Fr;
    const uint32_t N = (uint32_t)z.n_coeffs, D = (uint32_t)z.domain;
    const uint64_t n_inst = z.n_public + 1, D2 = 2ull * D;
    DevBuf key, colv, val, nonone, counts, offsets, task, cursor, pool_off, task2, words;
    B2S_TRY(key.alloc(c, (size_t)N * 4));
    B2S_TRY(colv.alloc(c, (size_t)N * 4));
    B2S_TRY(val.alloc(c, (size_t)N * sizeof(Fr)));
    B2S_TRY(nonone.alloc(c, (size_t)N * 4));
    B2S_TRY(counts.alloc(c, D2 * 4));
    B2S_TRY(words.alloc(c, 16));   // [0, 8) placement error word, [8, 12) max_a1, [12, 16) lowest bad input row
    B2S_CUDA(c, cudaMemsetAsync(counts.p, 0, D2 * 4, c->stream));
    B2S_CUDA(c, cudaMemsetAsync(words.p, 0xFF, 16, c->stream));
    B2S_CUDA(c, cudaMemsetAsync(words.as<char>() + 8, 0, 4, c->stream));
    unsigned long long* place_err = words.as<unsigned long long>();
    uint32_t* max_a1 = words.as<uint32_t>() + 2;
    uint32_t* row_err = words.as<uint32_t>() + 3;
    B2S_TRY(st.chunks(in + z.coeffs, N, ZKEY_REC, [&](const uint8_t* src, uint32_t n, uint64_t base) -> int32_t {
        B2S_LAUNCH(c, zkey_coeff_kernel<Curve>, cdiv(n, 256), 256, 0, src, n, base, (uint32_t)z.n_vars, D, key.as<uint32_t>(),
                   colv.as<uint32_t>(), val.as<Fr>(), nonone.as<uint32_t>(), counts.as<uint32_t>(), max_a1, st.err.as<unsigned long long>());
        return B2S_OK;
    }));
    unsigned long long word = ~0ull;
    uint32_t h_max_a1 = 0;
    if (N) B2S_TRY(st.read_err(&word));
    B2S_CUDA(c, cudaMemcpyAsync(&h_max_a1, max_a1, 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    if (word != ~0ull) return fail(c, B2S_ERR_INVALID_DATA, "zkey coefficients[%llu]: %s", word >> 3, coeff_reason((uint32_t)(word & 7)));
    if (h_max_a1 < n_inst)
        return fail(c, B2S_ERR_MALFORMED_VK, "zkey coefficients: A has %u rows, fewer than the %llu input rows", h_max_a1, (unsigned long long)n_inst);
    const uint32_t n_c = (uint32_t)(h_max_a1 - n_inst);
    uint64_t need = 1;
    while (need < h_max_a1) need <<= 1;
    if (need != D)
        return fail(c, B2S_ERR_MALFORMED_VK, "zkey: domainSize %u, but %u constraints and %llu input rows need %llu", D, n_c,
                    (unsigned long long)n_inst, (unsigned long long)need);
    // CSR offsets of both matrices in one scan; pool slots of the non-ONE records in another
    B2S_TRY(offsets.alloc(c, (D2 + 1) * 4));
    B2S_TRY(task.alloc(c, (D2 + 1) * 4));
    B2S_TRY(cursor.alloc(c, D2 * 4));
    B2S_TRY(pool_off.alloc(c, ((size_t)N + 1) * 4));
    B2S_TRY(task2.alloc(c, ((size_t)N + 1) * 4));
    B2S_TRY(scan_counts(c, counts.as<uint32_t>(), (uint32_t)D2, 1u, offsets.as<uint32_t>(), task.as<uint32_t>()));
    B2S_TRY(scan_counts(c, nonone.as<uint32_t>(), N, 1u, pool_off.as<uint32_t>(), task2.as<uint32_t>()));
    B2S_CUDA(c, cudaMemcpyAsync(cursor.p, offsets.p, D2 * 4, cudaMemcpyDeviceToDevice, c->stream));
    uint32_t h_off[3] = {0, 0, 0}, n_pool = 0;   // offsets[n_c], [D], [D + n_c]
    const uint64_t at[3] = {n_c, D, (uint64_t)D + n_c};
    for (int i = 0; i < 3; i++)
        B2S_CUDA(c, cudaMemcpyAsync(&h_off[i], offsets.as<uint32_t>() + at[i], 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&n_pool, pool_off.as<uint32_t>() + N, 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    if (n_pool == UINT32_MAX) return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "zkey: more than 2^32 - 2 coefficients other than 1");
    m->n_rows = n_c;
    m->n_instance = n_inst;
    m->n_witness = z.n_vars - n_inst;
    m->log_domain = (uint32_t)__builtin_ctz(D);
    m->nnz[0] = h_off[0];
    m->nnz[1] = h_off[2] - h_off[1];
    m->pool_size = n_pool + 1;
    CsrOut o{};
    for (int k = 0; k < 3; k++) B2S_TRY(m->row_ptr[k].alloc(c, ((size_t)n_c + 1) * 8));
    for (int k = 0; k < 2; k++) {
        B2S_TRY(m->col[k].alloc(c, m->nnz[k] * 4));
        B2S_TRY(m->coeff_id[k].alloc(c, m->nnz[k] * 4));
        o.row_ptr[k] = m->row_ptr[k].as<uint64_t>();
        o.col[k] = m->col[k].as<uint32_t>();
        o.cid[k] = m->coeff_id[k].as<uint32_t>();
    }
    B2S_CUDA(c, cudaMemsetAsync(m->row_ptr[2].p, 0, ((size_t)n_c + 1) * 8, c->stream));
    B2S_TRY(m->pool.alloc(c, (size_t)m->pool_size * sizeof(Fr)));
    const uint64_t nt = std::max<uint64_t>(2ull * (n_c + 1), n_inst);
    B2S_LAUNCH(c, zkey_rows_kernel<Fr>, cdiv(nt, 256), 256, 0, (const uint32_t*)offsets.as<uint32_t>(), D, n_c, (uint32_t)n_inst, o,
               m->pool.as<Fr>(), row_err);
    B2S_LAUNCH(c, zkey_place_kernel<Fr>, cdiv(N, 256), 256, 0, N, (const uint32_t*)key.as<uint32_t>(), (const uint32_t*)colv.as<uint32_t>(),
               (const Fr*)val.as<Fr>(), (const uint32_t*)nonone.as<uint32_t>(), (const uint32_t*)pool_off.as<uint32_t>(), cursor.as<uint32_t>(),
               (const uint32_t*)offsets.as<uint32_t>(), D, n_c, o, m->pool.as<Fr>(), place_err);
    unsigned long long h_err = 0;
    uint32_t h_row = 0;
    B2S_CUDA(c, cudaMemcpyAsync(&h_err, place_err, 8, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&h_row, row_err, 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    if (h_err != ~0ull) return fail(c, B2S_ERR_MALFORMED_VK, "zkey coefficients[%llu]: %s", h_err >> 3, coeff_reason((uint32_t)(h_err & 7)));
    if (h_row != UINT32_MAX)
        return fail(c, B2S_ERR_MALFORMED_VK, "zkey coefficients: input row %u (A row %llu) does not hold exactly one entry", h_row,
                    (unsigned long long)n_c + h_row);
    return B2S_OK;
}

// canonical LE -> Montgomery, each value below r, z[0] = 1 (reasons 1 and 2 in err)
template <class Curve>
__global__ void wtns_kernel(const uint8_t* __restrict__ src, uint32_t n, uint64_t base, typename Curve::Fr* __restrict__ out,
                            unsigned long long* err) {
    using Fr = typename Curve::Fr;
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(src + (size_t)i * FR_BYTES);
    Fr v, one = Fr::zero();
    one.v[0] = 1;
#pragma unroll
    for (int j = 0; j < Fr::N; j++) v.v[j] = w[j];
    const uint64_t e = base + i;
    if (!dec::below_p(v)) atomicMin(err, (unsigned long long)(e << 3 | 1));
    else if (e == 0 && v != one) atomicMin(err, 2ull);
    out[e] = v.to_mont();
}

// ---- circom .r1cs ----------------------------------------------------------------------------------------------------
constexpr uint32_t R1CS_ENTRY = 4 + FR_BYTES;   // u32 wire, then the coefficient
enum R1csSection { R_HEADER = 1, R_CONSTRAINTS, R_WIRE_MAP, R_GATES_USED, R_GATES_APPLIED, R_SECTIONS = R_GATES_APPLIED };
enum EntryReason : uint32_t { EN_WIRE = 1, EN_VALUE };
const char MATRIX_NAME[3] = {'A', 'B', 'C'};

struct R1csFile {
    Section s[R_SECTIONS + 1];
    b2s_r1cs_file_info info{};
    uint64_t n_instance = 0;
    uint32_t log_domain = 0;
};

// framing, curve and dimensions, the domain limits included: every check that needs no per-constraint data
int32_t r1cs_parse(Ctx* c, const uint8_t* in, uint64_t len, R1csFile& f) {
    B2S_TRY(bin_sections(c, "r1cs", in, len, 1, R_SECTIONS, f.s, R_CONSTRAINTS));
    for (int t : {R_GATES_USED, R_GATES_APPLIED})
        if (f.s[t].seen) return fail(c, B2S_ERR_INVALID_DATA, "r1cs: section %d (PLONK custom gates) is not supported", t);
    const Section& h = f.s[R_HEADER];
    const uint8_t* b = in + h.off;
    const uint32_t n8 = h.size >= 4 ? rd32(b) : 0;
    if (h.size < 4 || h.size != 32ull + n8)
        return fail(c, B2S_ERR_INVALID_DATA, "r1cs: header section holds %llu bytes, n8 = %u needs %llu", (unsigned long long)h.size, n8,
                    32ull + n8);
    const bool same_field = dispatch_curve(c, [&](auto curve) { return (int32_t)is_modulus<typename decltype(curve)::FrP>(b + 4, n8); }) == 1;
    if (!same_field) return fail(c, B2S_ERR_INVALID_ARG, "r1cs: the prime (%u bytes) is not the scalar field of the ctx's curve", n8);
    const uint8_t* d = b + 4 + n8;
    b2s_r1cs_file_info& i = f.info;
    i.n_wires = rd32(d);
    i.n_pub_out = rd32(d + 4);
    i.n_pub_in = rd32(d + 8);
    i.n_prv_in = rd32(d + 12);
    i.n_labels = rd64(d + 16);
    i.n_constraints = rd32(d + 24);
    if (i.n_wires < 1 + i.n_pub_out + i.n_pub_in + i.n_prv_in)
        return fail(c, B2S_ERR_INVALID_DATA, "r1cs: nWires %llu < 1 + nPubOut %llu + nPubIn %llu + nPrvIn %llu", (unsigned long long)i.n_wires,
                    (unsigned long long)i.n_pub_out, (unsigned long long)i.n_pub_in, (unsigned long long)i.n_prv_in);
    const Section& wm = f.s[R_WIRE_MAP];
    if (wm.seen && wm.size != 8 * i.n_wires)
        return fail(c, B2S_ERR_INVALID_DATA, "r1cs: section 3 (wire map) holds %llu bytes, nWires %llu need %llu", (unsigned long long)wm.size,
                    (unsigned long long)i.n_wires, (unsigned long long)(8 * i.n_wires));
    f.n_instance = 1 + i.n_pub_out + i.n_pub_in;
    uint32_t logd = 0;
    while ((1ull << logd) < i.n_constraints + f.n_instance) logd++;
    const uint32_t two_adicity = (uint32_t)dispatch_curve(c, [](auto curve) { return (int32_t)decltype(curve)::FrP::TWO_ADICITY; });
    if (logd > two_adicity || logd > 27)   // the limits of b2s_r1cs_upload
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs: %llu constraints and %llu instance variables need domain 2^%u, unsupported",
                    (unsigned long long)i.n_constraints, (unsigned long long)f.n_instance, logd);
    f.log_domain = logd;
    i.domain_size = 1ull << logd;
    return B2S_OK;
}

// The host's part of the constraint section: its 3 m count words, each checked against the bytes that remain (64-bit), and
// the walk must end at the section's end.  counts[k m + i] = the entries of matrix k in constraint i.  The section is cut
// into spans of whole constraints of at most a chunk's bytes (one longer constraint makes a span of its own): span j holds
// constraints [row[j], row[j + 1]), bytes [cut[j], cut[j + 1]) of the section, and matrix k's entries from first[3 j + k].
struct R1csWalk {
    std::vector<uint32_t> counts;
    uint64_t nnz[3] = {0, 0, 0};
    std::vector<uint64_t> cut, row, first;
};

int32_t r1cs_walk(Ctx* c, const uint8_t* p, uint64_t size, uint64_t m, R1csWalk& w) {
    const uint64_t span_max = Stager::CH * R1CS_ENTRY;
    w.counts.resize(3 * m);
    auto close_span = [&](uint64_t at, uint64_t i) {
        w.cut.push_back(at);
        w.row.push_back(i);
        w.first.insert(w.first.end(), w.nnz, w.nnz + 3);
    };
    close_span(0, 0);
    uint64_t at = 0;
    for (uint64_t i = 0; i < m; i++) {
        const uint64_t start = at;
        for (int k = 0; k < 3; k++) {
            if (size - at < 4)
                return fail(c, B2S_ERR_INVALID_DATA, "r1cs constraint %llu %c: the count word overruns section 2 (%llu bytes)", (unsigned long long)i,
                            MATRIX_NAME[k], (unsigned long long)size);
            const uint64_t n = rd32(p + at);
            at += 4;
            if (n > (size - at) / R1CS_ENTRY)
                return fail(c, B2S_ERR_INVALID_DATA, "r1cs constraint %llu %c: %llu entries overrun section 2 (%llu bytes remain)",
                            (unsigned long long)i, MATRIX_NAME[k], (unsigned long long)n, (unsigned long long)(size - at));
            at += n * R1CS_ENTRY;
            w.counts[k * m + i] = (uint32_t)n;
        }
        if (start > w.cut.back() && at - w.cut.back() > span_max) close_span(start, i);
        for (int k = 0; k < 3; k++) w.nnz[k] += w.counts[k * m + i];
    }
    if (at != size)
        return fail(c, B2S_ERR_INVALID_DATA, "r1cs: section 2 holds %llu bytes after its %llu constraints", (unsigned long long)(size - at),
                    (unsigned long long)m);
    if (m) close_span(at, m);
    for (int k = 0; k < 3; k++)
        if (w.nnz[k] >= (1ull << 32))
            return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs: matrix %c has %llu nonzeros, 2^32 or more", MATRIX_NAME[k],
                        (unsigned long long)w.nnz[k]);
    return B2S_OK;
}

struct R1csMats {
    uint64_t* row_ptr[3];
    uint32_t* col[3];
    uint32_t* cid[3];
    uint64_t base[3];   // matrix k's entries start at base[k] in the arrays of all entries (val, nonone, pool_off)
};
// member k of three, without indexing a kernel parameter by a runtime k (which would copy it to local memory)
template <class T>
__device__ __forceinline__ T pick3(const T (&a)[3], uint32_t k) { return k == 0 ? a[0] : k == 1 ? a[1] : a[2]; }
struct R1csSpan {
    uint64_t row0, row1, byte0;   // constraints [row0, row1), staged from section byte byte0 on
    uint64_t first[3];            // the span's first entry of each matrix
    uint32_t n[3];                // and its entries of each matrix
};

// row_ptr[k][r] = offsets[k (M + 1) + r] (the three per-matrix scans of the counts, widened)
__global__ void r1cs_rows_kernel(const uint32_t* __restrict__ offsets, uint64_t M, R1csMats o) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 3 * (M + 1)) return;
    const uint32_t k = (uint32_t)(t / (M + 1));
    pick3(o.row_ptr, k)[t - k * (M + 1)] = offsets[t];
}

// One thread per entry of a span, A's entries first, then B's, then C's.  Entry e of matrix k lies in the row i whose range
// [row_ptr[k][i], row_ptr[k][i + 1]) holds it (binary search over the span's rows), at section byte
// 12 i + 4 (k + 1) + R1CS_ENTRY (e + sum_{k' < k} row_ptr[k'][i + 1] + sum_{k' > k} row_ptr[k'][i]).  Range checks (the
// lowest bad entry, in file order, into err with its EntryReason), then the wire into col and the Montgomery value with its
// ONE flag at base[k] + e.
template <class Curve>
__global__ void __launch_bounds__(256) r1cs_entry_kernel(const uint8_t* __restrict__ src, R1csSpan sp, R1csMats o, uint32_t n_wires,
                                                         typename Curve::Fr* __restrict__ val, uint32_t* __restrict__ nonone,
                                                         unsigned long long* err) {
    using Fr = typename Curve::Fr;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= sp.n[0] + sp.n[1] + sp.n[2]) return;
    const uint32_t k = t < sp.n[0] ? 0 : t < sp.n[0] + sp.n[1] ? 1 : 2;
    const uint64_t e = pick3(sp.first, k) + t - (k > 0 ? sp.n[0] : 0) - (k > 1 ? sp.n[1] : 0);
    const uint64_t* rp = pick3(o.row_ptr, k);
    uint64_t lo = sp.row0, hi = sp.row1 - 1;   // the last row i of the span with rp[i] <= e
    while (lo < hi) {
        const uint64_t mid = (lo + hi + 1) >> 1;
        if (rp[mid] <= e) lo = mid;
        else hi = mid - 1;
    }
    const uint64_t i = lo;
    uint64_t before = e;
#pragma unroll
    for (uint32_t q = 0; q < 3; q++)
        if (q != k) before += o.row_ptr[q][q < k ? i + 1 : i];   // q unrolled: no runtime index into o
    const uint64_t at = 12 * i + 4 * (k + 1) + (uint64_t)R1CS_ENTRY * before - sp.byte0;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(src + at);
    const uint32_t wire = w[0];
    Fr v;
#pragma unroll
    for (int j = 0; j < Fr::N; j++) v.v[j] = w[1 + j];
    const uint32_t bad = wire >= n_wires ? EN_WIRE : !dec::below_p(v) ? EN_VALUE : 0;
    if (bad) {   // (3 i + k) < 2^29 and the index in the row < 2^32: the key sorts in file order
        atomicMin(err, ((3 * i + k) << 32 | (e - rp[i])) << 2 | bad);
        return;
    }
    v = v.to_mont();
    const uint64_t g = pick3(o.base, k) + e;
    pick3(o.col, k)[e] = wire;
    val[g] = v;
    nonone[g] = v != Fr::one();
}

// coefficient ids over all N entries: 0 for ONE, 1 + pool_off otherwise (that pool slot receives the value); pool[0] = ONE
template <class Fr>
__global__ void r1cs_place_kernel(uint64_t N, R1csMats o, const Fr* __restrict__ val, const uint32_t* __restrict__ nonone,
                                  const uint32_t* __restrict__ pool_off, Fr* pool) {
    const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (g == 0) pool[0] = Fr::one();
    if (g >= N) return;
    const uint32_t k = g >= o.base[2] ? 2 : g >= o.base[1] ? 1 : 0;
    uint32_t id = 0;
    if (nonone[g]) {
        id = 1 + pool_off[g];
        pool[id] = val[g];
    }
    pick3(o.cid, k)[g - pick3(o.base, k)] = id;
}

template <class Curve>
int32_t r1cs_matrices(Ctx* c, const uint8_t* sec, const R1csFile& f, const R1csWalk& w, b2s_r1cs* m) {
    using Fr = typename Curve::Fr;
    const uint64_t M = f.info.n_constraints, N = w.nnz[0] + w.nnz[1] + w.nnz[2];
    if (N >= UINT32_MAX)
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs: %llu nonzeros in all, more than the coefficient pool's 2^32 - 2",
                    (unsigned long long)N);
    m->n_rows = M;
    m->n_instance = f.n_instance;
    m->n_witness = f.info.n_wires - f.n_instance;
    m->log_domain = f.log_domain;
    R1csMats o{};
    for (int k = 0; k < 3; k++) {
        m->nnz[k] = w.nnz[k];
        B2S_TRY(m->row_ptr[k].alloc(c, (M + 1) * 8));
        B2S_TRY(m->col[k].alloc(c, w.nnz[k] * 4));
        B2S_TRY(m->coeff_id[k].alloc(c, w.nnz[k] * 4));
        o.row_ptr[k] = m->row_ptr[k].as<uint64_t>();
        o.col[k] = m->col[k].as<uint32_t>();
        o.cid[k] = m->coeff_id[k].as<uint32_t>();
        o.base[k] = k == 0 ? 0 : o.base[k - 1] + w.nnz[k - 1];
    }
    // row pointers: the counts of each matrix scanned on the device
    DevBuf counts, offsets, task, val, nonone, pool_off, task2;
    if (M) {
        B2S_TRY(counts.alloc(c, 3 * M * 4));
        B2S_TRY(offsets.alloc(c, 3 * (M + 1) * 4));
        B2S_TRY(task.alloc(c, 3 * (M + 1) * 4));
        B2S_CUDA(c, cudaMemcpyAsync(counts.p, w.counts.data(), 3 * M * 4, cudaMemcpyHostToDevice, c->stream));
        for (uint64_t k = 0; k < 3; k++)
            B2S_TRY(scan_counts(c, counts.as<uint32_t>() + k * M, (uint32_t)M, 1u, offsets.as<uint32_t>() + k * (M + 1),
                                task.as<uint32_t>() + k * (M + 1)));
        B2S_LAUNCH(c, r1cs_rows_kernel, cdiv(3 * (M + 1), 256), 256, 0, (const uint32_t*)offsets.as<uint32_t>(), M, o);
    } else {
        for (int k = 0; k < 3; k++) B2S_CUDA(c, cudaMemsetAsync(m->row_ptr[k].p, 0, 8, c->stream));
    }
    // every entry decoded, checked and placed, one span of whole constraints at a time
    B2S_TRY(val.alloc(c, N * sizeof(Fr)));
    B2S_TRY(nonone.alloc(c, N * 4));
    Stager st(c);
    const uint64_t n_spans = w.cut.size() - 1;
    B2S_TRY(st.spans(sec, w.cut.data(), n_spans, [&](const uint8_t* src, uint64_t j) -> int32_t {
        R1csSpan sp{w.row[j], w.row[j + 1], w.cut[j], {}, {}};
        for (int k = 0; k < 3; k++) {
            sp.first[k] = w.first[3 * j + k];
            sp.n[k] = (uint32_t)(w.first[3 * (j + 1) + k] - sp.first[k]);
        }
        const uint64_t n = (uint64_t)sp.n[0] + sp.n[1] + sp.n[2];
        if (n)
            B2S_LAUNCH(c, r1cs_entry_kernel<Curve>, cdiv(n, 256), 256, 0, src, sp, o, (uint32_t)f.info.n_wires, val.as<Fr>(),
                       nonone.as<uint32_t>(), st.err.as<unsigned long long>());
        return B2S_OK;
    }));
    unsigned long long word = ~0ull;
    B2S_TRY(st.read_err(&word));
    if (word != ~0ull) {
        const uint64_t i = (word >> 34) / 3, j = (word >> 2) & 0xFFFFFFFFull;
        const uint32_t k = (uint32_t)((word >> 34) % 3);
        if ((word & 3) == EN_VALUE)
            return fail(c, B2S_ERR_INVALID_DATA, "r1cs constraint %llu %c[%llu]: coefficient not below r", (unsigned long long)i, MATRIX_NAME[k],
                        (unsigned long long)j);
        uint64_t at = 0;   // the entry's byte in the section, for the wire in the message
        for (uint64_t q = 0; q < i; q++) at += 12 + (uint64_t)R1CS_ENTRY * (w.counts[q] + w.counts[M + q] + w.counts[2 * M + q]);
        for (uint32_t q = 0; q < k; q++) at += 4 + (uint64_t)R1CS_ENTRY * w.counts[q * M + i];
        at += 4 + (uint64_t)R1CS_ENTRY * j;
        return fail(c, B2S_ERR_INVALID_DATA, "r1cs constraint %llu %c[%llu]: wire %u not below nWires %llu", (unsigned long long)i, MATRIX_NAME[k],
                    (unsigned long long)j, rd32(sec + at), (unsigned long long)f.info.n_wires);
    }
    // pool slots of the entries other than ONE, compacted by a scan
    uint32_t n_pool = 0;
    if (N) {
        B2S_TRY(pool_off.alloc(c, (N + 1) * 4));
        B2S_TRY(task2.alloc(c, (N + 1) * 4));
        B2S_TRY(scan_counts(c, nonone.as<uint32_t>(), (uint32_t)N, 1u, pool_off.as<uint32_t>(), task2.as<uint32_t>()));
        B2S_CUDA(c, cudaMemcpyAsync(&n_pool, pool_off.as<uint32_t>() + N, 4, cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    m->pool_size = n_pool + 1;
    B2S_TRY(m->pool.alloc(c, (size_t)m->pool_size * sizeof(Fr)));
    B2S_LAUNCH(c, r1cs_place_kernel<Fr>, cdiv(std::max<uint64_t>(N, 1), 256), 256, 0, N, o, (const Fr*)val.as<Fr>(),
               (const uint32_t*)nonone.as<uint32_t>(), (const uint32_t*)pool_off.as<uint32_t>(), m->pool.as<Fr>());
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

}  // namespace

int32_t zkey_read_info(Ctx* c, const uint8_t* in, uint64_t len, b2s_zkey_info* out) {
    Zkey z;
    B2S_TRY(zkey_parse(c, in, len, z));
    *out = b2s_zkey_info{z.n_vars, z.n_public, z.domain, z.n_coeffs};
    return B2S_OK;
}

int32_t zkey_load(Ctx* c, const uint8_t* in, uint64_t len, bool validate, b2s_pk** out_pk, b2s_r1cs** out_m, void* alpha_g1,
                  void* beta_g2, void* gamma_g2, void* delta_g2, void* gamma_abc, uint64_t cap_abc) {
    Zkey z;
    B2S_TRY(zkey_parse(c, in, len, z));
    const uint64_t n_inst = z.n_public + 1;
    if (cap_abc < n_inst)
        return fail(c, B2S_ERR_INVALID_ARG, "zkey_load: IC has %llu points, room for %llu", (unsigned long long)n_inst, (unsigned long long)cap_abc);
    const Sizes sz = sizes(c);
    b2s_pk* pk = new b2s_pk();
    b2s_r1cs* m = new b2s_r1cs();
    pk->n_instance = n_inst;
    pk->n_witness = z.n_vars - n_inst;
    pk->domain_size = z.domain;
    pk->qap = B2S_QAP_CIRCOM;
    // in the order of PkQueryId: a, b_g1, b_g2, h, l
    const int sec[PK_QUERIES] = {Z_A, Z_B1, Z_B2, Z_H, Z_C};
    static const char* const name[PK_QUERIES] = {"zkey A", "zkey B1", "zkey B2", "zkey H", "zkey C"};
    auto body = [&]() -> int32_t {
        Stager st(c);
        B2S_TRY(pk->consts_g1.alloc(c, 3 * sz.g1));
        B2S_TRY(pk->consts_g2.alloc(c, 2 * sz.g2));
        char* k1 = pk->consts_g1.as<char>();
        char* k2 = pk->consts_g2.as<char>();
        B2S_TRY(st.decode<true>(1, in + z.pt[0], 1, false, validate, k1, "zkey alpha1"));
        B2S_TRY(st.decode<true>(1, in + z.pt[1], 1, false, validate, k1 + sz.g1, "zkey beta1"));
        B2S_TRY(st.decode<true>(2, in + z.pt[2], 1, false, validate, k2, "zkey beta2"));
        B2S_TRY(st.decode_host<true>(2, in + z.pt[3], 1, false, validate, gamma_g2, "zkey gamma2"));
        B2S_TRY(st.decode<true>(1, in + z.pt[4], 1, false, validate, k1 + 2 * sz.g1, "zkey delta1"));
        B2S_TRY(st.decode<true>(2, in + z.pt[5], 1, false, validate, k2 + sz.g2, "zkey delta2"));
        B2S_TRY(st.decode_host<true>(1, in + z.s[Z_IC].off, n_inst, false, validate, gamma_abc, "zkey IC"));
        for (int w = 0; w < PK_QUERIES; w++) {   // room for the two extra points pk_finish appends
            const int g = PK_QUERY[w].group;
            PkQuery& q = pk->q[w];
            q.len = z.s[sec[w]].size / sz.aff(g);
            B2S_TRY(q.pts.alloc(c, (q.len + 2) * sz.aff(g)));
            B2S_TRY(st.decode<true>(g, in + z.s[sec[w]].off, q.len, false, validate, q.pts.p, name[w]));
        }
        B2S_CUDA(c, cudaMemcpyAsync(alpha_g1, k1, sz.g1, cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(beta_g2, k2, sz.g2, cudaMemcpyDeviceToHost, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(delta_g2, k2 + sz.g2, sz.g2, cudaMemcpyDeviceToHost, c->stream));
        B2S_TRY(dispatch_curve(c, [&](auto curve) { return zkey_matrices<decltype(curve)>(c, st, in, z, m); }));
        return pk_finish(c, pk);   // synchronises
    };
    const int32_t s = body();
    if (s != B2S_OK) {
        delete pk;
        delete m;
        return s;
    }
    *out_pk = pk;
    *out_m = m;
    return B2S_OK;
}

int32_t wtns_read(Ctx* c, const uint8_t* in, uint64_t len, uint64_t n_vars, int32_t mem, void* out_z) {
    Section s[3];
    B2S_TRY(bin_sections(c, "wtns", in, len, 2, 2, s));
    const uint8_t* h = in + s[1].off;
    const uint32_t n8 = s[1].size >= 4 ? rd32(h) : 0;
    if (n8 == 0 || n8 > 64 || s[1].size != 8ull + n8) return fail(c, B2S_ERR_INVALID_DATA, "wtns: header section holds %llu bytes", (unsigned long long)s[1].size);
    const bool same_field = dispatch_curve(c, [&](auto curve) { return (int32_t)is_modulus<typename decltype(curve)::FrP>(h + 4, n8); }) == 1;
    if (!same_field) return fail(c, B2S_ERR_INVALID_ARG, "wtns: the prime (%u bytes) is not the scalar field of the ctx's curve", n8);
    const uint64_t n_wit = rd32(h + 4 + n8);
    if (n_wit != n_vars)   // snarkjs: "Invalid witness length"
        return fail(c, B2S_ERR_ASSIGNMENT_MISSING, "wtns: %llu values, the key has %llu variables", (unsigned long long)n_wit, (unsigned long long)n_vars);
    if (s[2].size != n_wit * FR_BYTES)
        return fail(c, B2S_ERR_INVALID_DATA, "wtns: data section holds %llu bytes, %llu values need %llu", (unsigned long long)s[2].size,
                    (unsigned long long)n_wit, (unsigned long long)(n_wit * FR_BYTES));
    if (n_wit == 0) return fail(c, B2S_ERR_INVALID_DATA, "wtns: no values (z[0] = 1 is required)");
    OutBuf z;
    B2S_TRY(z.bind(c, out_z, n_wit * FR_BYTES, mem));
    Stager st(c);
    B2S_TRY(st.chunks(in + s[2].off, n_wit, FR_BYTES, [&](const uint8_t* src, uint32_t n, uint64_t base) {
        return dispatch_curve(c, [&](auto curve) {
            using C = decltype(curve);
            B2S_LAUNCH(c, wtns_kernel<C>, cdiv(n, 256), 256, 0, src, n, base, z.as<typename C::Fr>(),
                       st.err.as<unsigned long long>());
            return (int32_t)B2S_OK;
        });
    }));
    unsigned long long word = 0;
    B2S_TRY(st.read_err(&word));
    if (word != ~0ull)
        return fail(c, B2S_ERR_INVALID_DATA, "wtns[%llu]: %s", word >> 3, (word & 7) == 1 ? "value not below r" : "z[0] is not 1");
    return z.finish(c);
}

int32_t r1cs_file_read_info(Ctx* c, const uint8_t* in, uint64_t len, b2s_r1cs_file_info* out) {
    R1csFile f;
    B2S_TRY(r1cs_parse(c, in, len, f));
    *out = f.info;
    return B2S_OK;
}

int32_t r1cs_file_load(Ctx* c, const uint8_t* in, uint64_t len, b2s_r1cs** out) {
    R1csFile f;
    B2S_TRY(r1cs_parse(c, in, len, f));
    R1csWalk w;
    const Section& sec = f.s[R_CONSTRAINTS];
    B2S_TRY(r1cs_walk(c, in + sec.off, sec.size, f.info.n_constraints, w));
    b2s_r1cs* m = new b2s_r1cs();
    const int32_t s = dispatch_curve(c, [&](auto curve) { return r1cs_matrices<decltype(curve)>(c, in + sec.off, f, w, m); });
    if (s != B2S_OK) {
        delete m;
        return s;
    }
    *out = m;
    return B2S_OK;
}

}  // namespace b2s
