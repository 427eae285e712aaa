// Argument matrices built on the device from the constraint system's flat LcMap (lcmap.cuh has the reference citations and
// the per-row logic): A, B, C for b2s_r1cs_upload_lcmap, every argument of every predicate for b2s_gr1cs_upload_lcmap.
// The matrices are one flat list of (matrix, row) slots, so any number of them takes the same launches: count, scan
// (msm.cu's scan kernels), bounds, fill; everything is HBM-bound index work and runs once per circuit.
// Instance outlining rides on the same launches: a tie kernel writes the tie rows' arguments (and, for outline_sr1cs, their
// 2-term LCs after the caller's) into the device copies before the count, and the View's remap rewrites the stored LCs' One
// and Instance terms as the count and the fill read them.
#include <algorithm>
#include <cstring>
#include <vector>

#include "common.cuh"
#include "lcmap.cuh"
#include "r1cs.cuh"

namespace b2s {

using lcmap::View;

// where matrix m's CSR goes (device pointers)
struct LcOut { uint64_t* row_ptr; uint32_t* col; uint32_t* coeff_id; };

// the matrix that holds slot t: the largest m with row0[m] <= t (row0[0] = 0; empty matrices share their row0 with the next)
__device__ __forceinline__ uint32_t matrix_of(const uint64_t* __restrict__ row0, uint32_t n_mats, uint64_t t) {
    uint32_t lo = 0, hi = n_mats;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (row0[mid] <= t) lo = mid; else hi = mid;
    }
    return lo;
}

// one thread per slot: counts[t] = nonzeros make_row keeps for argument args[t]
// total64: the same sum in 64 bits (one atomic per warp) -- the scan below is 32-bit and must not wrap unnoticed
// err_at: the lowest slot whose argument was rejected, so that the message can name it
__global__ void lcmap_count_kernel(View v, const uint64_t* __restrict__ args, uint64_t n_slots, uint32_t* __restrict__ counts,
                                   uint32_t* __restrict__ err, unsigned long long* __restrict__ total64,
                                   unsigned long long* __restrict__ err_at) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_slots) return;
    uint32_t e = 0;
    const uint32_t n = lcmap::count_row(v, args[t], &e);
    counts[t] = n;
    if (e) {
        atomicOr(err, e);
        atomicMin(err_at, (unsigned long long)t);
    }
    atomicAdd(total64, (unsigned long long)n);
}

// bounds[m] = offsets[row0[m]], m <= n_mats: where matrix m's nonzeros start in the one scan over all slots
__global__ void lcmap_bounds_kernel(const uint32_t* __restrict__ offsets, const uint64_t* __restrict__ row0, uint32_t n_mats,
                                    uint32_t* __restrict__ bounds) {
    const uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (m <= n_mats) bounds[m] = offsets[row0[m]];
}

// offsets: exclusive scan of counts over all n_slots slots.  Threads past the slots write the closing row_ptr entry of
// matrix t - n_slots.
__global__ void lcmap_fill_kernel(View v, const uint64_t* __restrict__ args, const uint64_t* __restrict__ row0, uint32_t n_mats,
                                  uint64_t n_slots, const uint32_t* __restrict__ offsets, const LcOut* __restrict__ out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_slots + n_mats) return;
    if (t >= n_slots) {
        const uint32_t m = (uint32_t)(t - n_slots);
        out[m].row_ptr[row0[m + 1] - row0[m]] = (uint64_t)(offsets[row0[m + 1]] - offsets[row0[m]]);
        return;
    }
    const uint32_t m = matrix_of(row0, n_mats, t);
    const uint32_t at = offsets[t] - offsets[row0[m]];
    const LcOut o = out[m];
    o.row_ptr[t - row0[m]] = at;
    lcmap::fill_row(v, args[t], o.col + at, o.coeff_id + at);
}

// Raw Variable (utils/variable.rs:4-14)
__device__ __forceinline__ uint64_t raw_var(uint32_t tag, uint64_t idx) { return (uint64_t)tag << lcmap::TAG_SHIFT | idx; }

// Where the tie rows of instance outlining go: argument j's first tie slot, and the LcMap's extent before them
struct TieSpec {
    int32_t strategy;
    uint64_t slot[3];
    uint64_t n_inst, w0, n_lcs, total;   // w0 = W, the witness that copies One
};

// one thread per instance variable i < n_inst: the arguments of tie row i (instance_outliner.rs:40-80), and for
// outline_sr1cs LC n_lcs + i = [(ONE, Instance(i)), (-ONE, w_{W+i})] (ids 0 and 1) with its closing offset
__global__ void lcmap_tie_kernel(TieSpec t, uint64_t* __restrict__ args, uint64_t* __restrict__ off, uint64_t* __restrict__ vars,
                                 uint32_t* __restrict__ coeffs) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= t.n_inst) return;
    using namespace lcmap;
    if (t.strategy == B2S_OUTLINE_R1CS) {   // w_W * w_W = One, w_W * w_{W+i} = Instance(i)
        args[t.slot[0] + i] = raw_var(TAG_WITNESS, t.w0);
        args[t.slot[1] + i] = raw_var(TAG_WITNESS, t.w0 + i);
        args[t.slot[2] + i] = i == 0 ? raw_var(TAG_ONE, 0) : raw_var(TAG_INSTANCE, i);
        return;
    }
    args[t.slot[0] + i] = raw_var(TAG_LC, t.n_lcs + i);   // (Instance(i) - w_{W+i})^2 = SymbolicLc(0)
    args[t.slot[1] + i] = raw_var(TAG_LC, 0);
    const uint64_t e = t.total + 2 * i;
    vars[e] = raw_var(TAG_INSTANCE, i);
    coeffs[e] = 0;
    vars[e + 1] = raw_var(TAG_WITNESS, t.w0 + i);
    coeffs[e + 1] = 1;
    off[t.n_lcs + 1 + i] = e + 2;
}

// one thread per (element t of an outlined row, assignment blockIdx.y): z' = z || (ONE, z[1], ..., z[n_copies - 1]).
// Elements move as two 16-byte words; nothing is computed, so one kernel serves every curve.
struct Words32 { uint4 lo, hi; };
__global__ void __launch_bounds__(256)
outline_assign_kernel(const uint4* __restrict__ z, uint64_t n_src, uint64_t n_copies, Words32 one, uint4* __restrict__ out) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t n_out = n_src + n_copies;
    if (t >= n_out) return;
    z += 2 * (uint64_t)blockIdx.y * n_src;
    out += 2 * ((uint64_t)blockIdx.y * n_out + t);
    const uint64_t from = t < n_src ? t : t - n_src;   // the copy of variable k reads z[k]; k = 0 is ONE
    if (t == n_src) {
        out[0] = one.lo;
        out[1] = one.hi;
        return;
    }
    out[0] = __ldg(z + 2 * from);
    out[1] = __ldg(z + 2 * from + 1);
}

int32_t lcmap_validate(Ctx* c, const LcMapHost& lm, uint64_t n_slots) {
    if (lm.n_lcs == 0 || !lm.offsets || lm.offsets[0] != 0)
        return fail(c, B2S_ERR_INVALID_ARG, "lcmap: offsets must start with 0 (LC 0 is the empty LC)");
    if (lm.pool_len < 2 || !lm.pool) return fail(c, B2S_ERR_INVALID_ARG, "lcmap: the interner pool holds at least ONE and -ONE");
    if (n_slots >= (1ull << 32)) return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "lcmap: too many rows");
    for (uint64_t j = 0; j < lm.n_lcs; j++)
        if (lm.offsets[j + 1] < lm.offsets[j]) return fail(c, B2S_ERR_INVALID_ARG, "lcmap: offsets not monotone at %llu", (unsigned long long)j);
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        // pool[0] must be ONE: the SpMV and check kernels skip the multiplication for id 0 (sr1cs/mod.rs:42-46)
        using FrP = typename decltype(curve)::FrP;
        uint32_t one[8];
        for (int i = 0; i < 8; i++) one[i] = FrP::r1(i);
        if (memcmp(lm.pool, one, 32) != 0) return fail(c, B2S_ERR_INVALID_ARG, "lcmap: pool[0] is not ONE (Montgomery form)");
        return B2S_OK;
    });
}

int32_t outline_validate(Ctx* c, const char* who, const b2s_outline& ol, uint32_t n_predicates, uint32_t target_arity, const LcMapHost& lm) {
    if (ol.strategy != B2S_OUTLINE_R1CS && ol.strategy != B2S_OUTLINE_SR1CS)
        return fail(c, B2S_ERR_INVALID_ARG, "%s: unknown outlining strategy %d (B2S_OUTLINE_R1CS 1, B2S_OUTLINE_SR1CS 2)", who, ol.strategy);
    if (ol.pred >= n_predicates)
        return fail(c, B2S_ERR_INVALID_ARG, "%s: outlining predicate %u out of range (%u predicates)", who, ol.pred, n_predicates);
    const uint32_t want = ol.strategy == B2S_OUTLINE_R1CS ? 3 : 2;
    if (target_arity != want)
        return fail(c, B2S_ERR_INVALID_ARG, "%s: outlining predicate %u has arity %u; %s ties need arity %u", who, ol.pred, target_arity,
                    ol.strategy == B2S_OUTLINE_R1CS ? "outline_r1cs" : "outline_sr1cs", want);
    if (ol.strategy != B2S_OUTLINE_SR1CS) return B2S_OK;
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        // the tie LCs name -ONE by id 1, as the interner assigns it (field_interner.rs:32-33)
        using FrP = typename decltype(curve)::FrP;
        uint32_t minus_one[8];
        uint64_t borrow = 0;
        for (int i = 0; i < 8; i++) {
            const uint64_t d = (uint64_t)FrP::mod(i) - FrP::r1(i) - borrow;
            minus_one[i] = (uint32_t)d;
            borrow = (d >> 63) & 1;
        }
        if (lm.pool_len < 2 || memcmp(static_cast<const uint8_t*>(lm.pool) + 32, minus_one, 32) != 0)
            return fail(c, B2S_ERR_INVALID_ARG, "%s: pool[1] is not -ONE (Montgomery form); the outline_sr1cs ties use it", who);
        return B2S_OK;
    });
}

int32_t lcmap_build(Ctx* c, const LcMapHost& lm, uint64_t n_instance, uint64_t n_vars, const std::vector<LcMatrix>& mats,
                    const char* what, const std::function<std::string(size_t, uint64_t)>& where, DevBuf& pool, uint32_t* pool_size,
                    const LcOutline* ol) {
    constexpr size_t FR_BYTES = 32;
    const uint32_t M = (uint32_t)mats.size();
    std::vector<uint64_t> row0(M + 1, 0);
    for (uint32_t m = 0; m < M; m++) row0[m + 1] = row0[m] + mats[m].n_rows + mats[m].n_tie;
    const uint64_t T = row0[M];                      // < 2^32: lcmap_validate
    const uint64_t total = lm.offsets[lm.n_lcs];
    // outline_sr1cs appends one 2-term LC per instance variable
    const uint64_t n_tie_lcs = ol && ol->strategy == B2S_OUTLINE_SR1CS ? n_instance : 0;
    const uint64_t n_lcs = lm.n_lcs + n_tie_lcs, n_terms = total + 2 * n_tie_lcs;

    // zero flags of the pool (byte comparison on the host; the pool is one entry per DISTINCT coefficient)
    std::vector<uint8_t> is_zero(lm.pool_len);
    {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(lm.pool);
        static const uint8_t zeros[FR_BYTES] = {0};
        for (uint32_t i = 0; i < lm.pool_len; i++) is_zero[i] = memcmp(p + (size_t)i * FR_BYTES, zeros, FR_BYTES) == 0;
    }
    B2S_TRY(pool.alloc(c, (size_t)lm.pool_len * FR_BYTES));
    B2S_CUDA(c, cudaMemcpyAsync(pool.p, lm.pool, (size_t)lm.pool_len * FR_BYTES, cudaMemcpyHostToDevice, c->stream));
    *pool_size = lm.pool_len;
    if (M == 0) return B2S_OK;

    DevBuf d_off, d_vars, d_coeffs, d_zero, d_args, d_row0, d_counts, d_offsets, d_task, d_err, d_bounds, d_out;
    B2S_TRY(d_off.alloc(c, (n_lcs + 1) * 8));
    B2S_CUDA(c, cudaMemcpyAsync(d_off.p, lm.offsets, (lm.n_lcs + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    B2S_TRY(d_vars.alloc(c, n_terms * 8));
    B2S_TRY(d_coeffs.alloc(c, n_terms * 4));
    if (total) {
        B2S_CUDA(c, cudaMemcpyAsync(d_vars.p, lm.vars, total * 8, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(d_coeffs.p, lm.coeffs, total * 4, cudaMemcpyHostToDevice, c->stream));
    }
    B2S_TRY(d_zero.alloc(c, lm.pool_len));
    B2S_CUDA(c, cudaMemcpyAsync(d_zero.p, is_zero.data(), lm.pool_len, cudaMemcpyHostToDevice, c->stream));
    B2S_TRY(d_args.alloc(c, T * 8));
    for (uint32_t m = 0; m < M; m++)
        if (mats[m].n_rows)
            B2S_CUDA(c, cudaMemcpyAsync(d_args.as<uint64_t>() + row0[m], mats[m].args, mats[m].n_rows * 8, cudaMemcpyHostToDevice, c->stream));
    for (uint32_t m = 0; m < M; m++) B2S_TRY(mats[m].row_ptr->alloc(c, (mats[m].n_rows + mats[m].n_tie + 1) * 8));
    B2S_TRY(d_row0.alloc(c, (M + 1) * 8));
    B2S_CUDA(c, cudaMemcpyAsync(d_row0.p, row0.data(), (M + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    View v{d_off.as<uint64_t>(), d_vars.as<uint64_t>(), d_coeffs.as<uint32_t>(), d_zero.as<uint8_t>(), n_lcs, lm.pool_len, n_instance, n_vars};
    if (ol) {
        TieSpec t{ol->strategy, {0, 0, 0}, n_instance, ol->n_witness, lm.n_lcs, total};
        const uint32_t arity = ol->strategy == B2S_OUTLINE_R1CS ? 3 : 2;
        for (uint32_t j = 0; j < arity; j++) t.slot[j] = row0[ol->first_mat + j] + mats[ol->first_mat + j].n_rows;
        B2S_LAUNCH(c, lcmap_tie_kernel, cdiv(n_instance, 256), 256, 0, t, d_args.as<uint64_t>(), d_off.as<uint64_t>(), d_vars.as<uint64_t>(),
                   d_coeffs.as<uint32_t>());
        v.remap_lcs = lm.n_lcs;                      // the tie LCs stay as they are
        v.copy0 = n_instance + ol->n_witness;
    }

    B2S_TRY(d_err.alloc(c, 24));         // [0..3] error bits, [8..15] 64-bit nonzero total, [16..23] first rejected slot
    B2S_CUDA(c, cudaMemsetAsync(d_err.p, 0, 16, c->stream));
    B2S_CUDA(c, cudaMemsetAsync(d_err.as<uint8_t>() + 16, 0xFF, 8, c->stream));
    unsigned long long* d_total64 = reinterpret_cast<unsigned long long*>(d_err.as<uint8_t>() + 8);
    unsigned long long* d_err_at = reinterpret_cast<unsigned long long*>(d_err.as<uint8_t>() + 16);
    B2S_TRY(d_offsets.alloc(c, (T + 1) * 4));
    if (T) {
        B2S_TRY(d_counts.alloc(c, T * 4));
        B2S_TRY(d_task.alloc(c, (T + 1) * 4));
        B2S_LAUNCH(c, lcmap_count_kernel, cdiv(T, 256), 256, 0, v, (const uint64_t*)d_args.as<uint64_t>(), T, d_counts.as<uint32_t>(),
                   d_err.as<uint32_t>(), d_total64, d_err_at);
        B2S_TRY(scan_counts(c, d_counts.as<uint32_t>(), (uint32_t)T, 1u, d_offsets.as<uint32_t>(), d_task.as<uint32_t>()));
    } else {
        B2S_CUDA(c, cudaMemsetAsync(d_offsets.p, 0, 4, c->stream));
    }
    B2S_TRY(d_bounds.alloc(c, (M + 1) * 4));
    B2S_LAUNCH(c, lcmap_bounds_kernel, cdiv(M + 1, 256), 256, 0, (const uint32_t*)d_offsets.as<uint32_t>(),
               (const uint64_t*)d_row0.as<uint64_t>(), M, d_bounds.as<uint32_t>());
    std::vector<uint32_t> bounds(M + 1);
    uint32_t h_err = 0;
    unsigned long long h_total64 = 0, h_err_at = 0;
    B2S_CUDA(c, cudaMemcpyAsync(bounds.data(), d_bounds.p, (M + 1) * 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&h_err, d_err.p, 4, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&h_total64, d_total64, 8, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&h_err_at, d_err_at, 8, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    if (h_err) {
        const size_t m = (size_t)(std::upper_bound(row0.begin(), row0.end(), (uint64_t)h_err_at) - row0.begin()) - 1;
        const std::string at = where ? where(m, h_err_at - row0[m]) : std::string();
        if (h_err & lcmap::ERR_NESTED_LC)
            return fail(c, B2S_ERR_INVALID_ARG, "%slcmap: a linear combination refers to another one -- call finalize() (inline_all_lcs) first",
                        at.c_str());
        if (h_err & lcmap::ERR_COLUMN)
            return fail(c, B2S_ERR_ASSIGNMENT_MISSING, "%slcmap: a variable index is outside the %llu variables", at.c_str(),
                        (unsigned long long)n_vars);
        return fail(c, B2S_ERR_INVALID_ARG, "%slcmap: malformed input (error bits 0x%x: 1 tag, 2 lc index, 16 coefficient id)", at.c_str(), h_err);
    }
    if (h_total64 >> 32)
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "lcmap: %llu nonzeros in %s together; the limit is 2^32 - 1", h_total64, what);
    std::vector<LcOut> lo(M);
    for (uint32_t m = 0; m < M; m++) {
        *mats[m].nnz = (uint64_t)(bounds[m + 1] - bounds[m]);
        B2S_TRY(mats[m].col->alloc(c, *mats[m].nnz * 4));
        B2S_TRY(mats[m].coeff_id->alloc(c, *mats[m].nnz * 4));
        lo[m] = {mats[m].row_ptr->as<uint64_t>(), mats[m].col->as<uint32_t>(), mats[m].coeff_id->as<uint32_t>()};
    }
    B2S_TRY(d_out.alloc(c, M * sizeof(LcOut)));
    B2S_CUDA(c, cudaMemcpyAsync(d_out.p, lo.data(), M * sizeof(LcOut), cudaMemcpyHostToDevice, c->stream));
    B2S_LAUNCH(c, lcmap_fill_kernel, cdiv(T + M, 256), 256, 0, v, (const uint64_t*)d_args.as<uint64_t>(), (const uint64_t*)d_row0.as<uint64_t>(),
               M, T, (const uint32_t*)d_offsets.as<uint32_t>(), (const LcOut*)d_out.as<LcOut>());
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));   // host inputs may be released by the caller after return
    return B2S_OK;
}

int32_t r1cs_upload_lcmap(Ctx* c, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness, const uint64_t* const args[3],
                          uint64_t n_lcs, const uint64_t* lc_offsets, const uint64_t* lc_vars, const uint32_t* lc_coeffs,
                          const void* pool, uint32_t pool_len, const b2s_outline* ol, b2s_r1cs** out) {
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        using FrP = typename decltype(curve)::FrP;
        if (n_instance == 0) return fail(c, B2S_ERR_INVALID_ARG, "r1cs: n_instance counts the constant One and must be >= 1");
        const LcMapHost lm{n_lcs, lc_offsets, lc_vars, lc_coeffs, pool, pool_len};
        // outlining: n_instance tie rows and n_instance copies (witnesses n_witness ..)
        const uint64_t n_tie = ol ? n_instance : 0, rows = n_rows + n_tie, n_vars = n_instance + n_witness + n_tie;
        if (ol) {
            if (ol->strategy == B2S_OUTLINE_SR1CS)
                return fail(c, B2S_ERR_INVALID_ARG, "r1cs_upload_lcmap_outline: the Groth16 matrix handle takes B2S_OUTLINE_R1CS only");
            B2S_TRY(outline_validate(c, "r1cs_upload_lcmap_outline", *ol, 1, 3, lm));
            if (n_vars > (1ull << 32))
                return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs: %llu variables after outlining; columns are u32, the limit is 2^32",
                            (unsigned long long)n_vars);
        }
        B2S_TRY(lcmap_validate(c, lm, 3 * rows));
        uint32_t logd = 0;
        while ((1ull << logd) < rows + n_instance) logd++;
        if (logd > (uint32_t)FrP::TWO_ADICITY || logd > 27) return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "r1cs: domain 2^%u unsupported", logd);

        std::unique_ptr<b2s_r1cs> m(new b2s_r1cs());
        m->n_rows = rows; m->n_instance = n_instance; m->n_witness = n_witness + n_tie; m->log_domain = logd;
        m->outline_copies = n_tie;
        std::vector<LcMatrix> mats;
        for (int k = 0; k < 3; k++) mats.push_back({args[k], n_rows, &m->row_ptr[k], &m->col[k], &m->coeff_id[k], &m->nnz[k], n_tie});
        const LcOutline lo{B2S_OUTLINE_R1CS, n_witness, 0};
        B2S_TRY(lcmap_build(c, lm, n_instance, n_vars, mats, "A, B, C", nullptr, m->pool, &m->pool_size, ol ? &lo : nullptr));
        *out = m.release();
        return B2S_OK;
    });
}

int32_t outline_assignment(Ctx* c, uint64_t n_src, uint64_t n_copies, uint64_t n_assign, const void* z, int32_t mem, void* out_z) {
    // gridDim.y carries the assignment; host batches go through this much device scratch per chunk (as sr1cs_assignment)
    constexpr uint64_t MAX_PER_LAUNCH = 65535, SCRATCH_BYTES = 64ull << 20;
    if (n_assign == 0) return B2S_OK;
    Words32 one;
    B2S_TRY(dispatch_curve(c, [&](auto curve) -> int32_t {
        using FrP = typename decltype(curve)::FrP;
        uint32_t w[8];
        for (int i = 0; i < 8; i++) w[i] = FrP::r1(i);
        memcpy(&one, w, 32);
        return B2S_OK;
    }));
    const uint64_t n_out = n_src + n_copies, in_row = n_src * 32, out_row = n_out * 32;
    RowStager io(c, mem, {col_in(z, in_row), col_out(out_z, out_row)});
    uint64_t ch = std::min(MAX_PER_LAUNCH, n_assign);
    if (io.staged) ch = std::min(ch, std::max<uint64_t>(1, SCRATCH_BYTES / (in_row + out_row)));
    B2S_TRY(io.alloc(ch));
    for (uint64_t a0 = 0; a0 < n_assign; a0 += ch) {
        const uint64_t K = std::min(ch, n_assign - a0);
        B2S_TRY(io.load(a0, (uint32_t)K));
        B2S_LAUNCH(c, outline_assign_kernel, dim3(cdiv(n_out, 256), (unsigned)K), 256, 0, io.ptr<const uint4>(0), n_src, n_copies, one,
                   io.ptr<uint4>(1));
        B2S_TRY(io.store());
    }
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

}  // namespace b2s
