// Device-side CSR ingest straight from the constraint system's flat LcMap (SURVEY.md 8(f) row 1).
//
// The reference exports matrices through `to_matrices()` -> `get_lc` + `make_row`
// (/root/reference/relations/src/gr1cs/constraint_system.rs:768-804): 40 B per nonzero and one heap allocation per
// row, on the host.  The data it reads is already flat:
//   LcMap            { vars: Vec<Variable>, coeffs: Vec<InternedField>, offsets: Vec<usize> }   gr1cs/lc_map.rs:51-56
//   FieldInterner    { vec: Vec<F> }, vec[0] = ONE, vec[1] = -ONE, ids index vec              gr1cs/field_interner.rs:13-45
//   Variable         tag (top 3 bits: Zero 0, One 1, Instance 2, Witness 3, SymbolicLc 4) | 61-bit index
//                                                                                               utils/variable.rs:4-14,177-183
//   argument_lcs[k][i]   the k-th argument of the i-th constraint, a Variable                   gr1cs/predicate/mod.rs:81-94
// The interner's convention (id 0 = ONE) is the one the SpMV kernel already uses, so `coeffs` and the pool go to the
// device unchanged; what is left is, per (matrix k, row i):
//   get_lc      Zero -> no terms; SymbolicLc(j) -> the j-th LC; any other variable v -> the single term (ONE, v)
//   make_row    drop terms with a zero coefficient or the Zero variable; column = get_variable_index(num_instance):
//               One -> 0, Instance(i) -> i, Witness(i) -> i + num_instance                     utils/variable.rs:105-113
// done by a counting kernel, an exclusive scan (row_ptr) and a fill kernel.  The per-row logic lives in the
// host/device functions below so that tests can run exactly the kernels' code on the CPU
// (tests/native/host_ff.cpp: ht_lcmap_*, tests/test_host_lcmap.py).
//
// Instance outlining (ConstraintSystem::perform_instance_outlining, constraint_system.rs:826-863) is folded into the same
// walk: with remap_lcs > 0, every term of an LC j < remap_lcs that is One or Instance(i) reads as the witness copy of
// variable 0 or i, at column copy0 (+ i).  Bare arguments and the LCs at or past remap_lcs (the tie LCs the outlining
// strategy appends after the rewrite) keep their columns, as upstream.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define B2S_LC_HD __host__ __device__ __forceinline__
#else
#define B2S_LC_HD inline
#endif

namespace b2s {
namespace lcmap {

constexpr int TAG_SHIFT = 61;
constexpr uint64_t PAYLOAD_MASK = (uint64_t(1) << TAG_SHIFT) - 1;
enum : uint32_t { TAG_ZERO = 0, TAG_ONE = 1, TAG_INSTANCE = 2, TAG_WITNESS = 3, TAG_LC = 4 };

// Why an input was rejected (OR-ed into one device word; reported as B2S_ERR_INVALID_ARG / ASSIGNMENT_MISSING).
enum : uint32_t {
    ERR_BAD_TAG = 1,        // tag > 4
    ERR_LC_INDEX = 2,       // SymbolicLc(j) with j >= number of LCs
    ERR_NESTED_LC = 4,      // an LC term that is itself a SymbolicLc: finalize() / inline_all_lcs() has not run (make_row would panic)
    ERR_COLUMN = 8,         // column >= number of variables
    ERR_COEFF = 16,         // coefficient id outside the pool
};

struct View {
    const uint64_t* lc_offsets;   // n_lcs + 1
    const uint64_t* lc_vars;      // Variable, raw
    const uint32_t* lc_coeffs;    // InternedField
    const uint8_t* pool_is_zero;  // pool_len flags: the pooled value is 0 (make_row drops such terms)
    uint64_t n_lcs;
    uint32_t pool_len;
    uint64_t n_instance, n_vars;
    uint64_t remap_lcs = 0;       // outlining: LCs below this index are rewritten (0: none is)
    uint64_t copy0 = 0;           // outlining: the column of the copy of variable 0 (One / Instance(0))
};

B2S_LC_HD uint32_t tag_of(uint64_t var) { return (uint32_t)(var >> TAG_SHIFT); }
B2S_LC_HD uint64_t payload_of(uint64_t var) { return var & PAYLOAD_MASK; }

// Visits the terms `make_row(get_lc(arg))` keeps, in order, as f(column, coeff_id); returns the error bits met.
// Erroneous terms are skipped, so a caller that only counts and a caller that fills always agree.
template <class Fn>
B2S_LC_HD uint32_t for_each_kept_term(const View& v, uint64_t arg, Fn&& f) {
    uint32_t err = 0;
    auto plain = [&](uint64_t var, uint32_t coeff_id, bool remap) {
        const uint32_t tag = tag_of(var);
        if (tag == TAG_ZERO) return;
        if (tag == TAG_LC) { err |= ERR_NESTED_LC; return; }
        if (tag > TAG_LC) { err |= ERR_BAD_TAG; return; }
        if (coeff_id >= v.pool_len) { err |= ERR_COEFF; return; }
        if (v.pool_is_zero[coeff_id]) return;
        const uint64_t col = tag == TAG_ONE ? 0 : tag == TAG_INSTANCE ? payload_of(var) : payload_of(var) + v.n_instance;
        if (col >= v.n_vars || (tag == TAG_INSTANCE && col >= v.n_instance)) { err |= ERR_COLUMN; return; }
        f((uint32_t)(remap && tag != TAG_WITNESS ? v.copy0 + col : col), coeff_id);
    };
    const uint32_t tag = tag_of(arg);
    if (tag == TAG_ZERO) return 0;
    if (tag > TAG_LC) return ERR_BAD_TAG;
    if (tag != TAG_LC) { plain(arg, 0u, false); return err; }   // LinearCombination::from(var): coefficient ONE = id 0
    const uint64_t j = payload_of(arg);
    if (j >= v.n_lcs) return ERR_LC_INDEX;
    const bool remap = j < v.remap_lcs;
    for (uint64_t e = v.lc_offsets[j]; e < v.lc_offsets[j + 1]; e++) plain(v.lc_vars[e], v.lc_coeffs[e], remap);
    return err;
}

B2S_LC_HD uint32_t count_row(const View& v, uint64_t arg, uint32_t* err) {
    uint32_t n = 0;
    *err |= for_each_kept_term(v, arg, [&](uint32_t, uint32_t) { n++; });
    return n;
}

B2S_LC_HD void fill_row(const View& v, uint64_t arg, uint32_t* col_out, uint32_t* coeff_out) {
    uint32_t n = 0;
    for_each_kept_term(v, arg, [&](uint32_t col, uint32_t id) { col_out[n] = col; coeff_out[n] = id; n++; });
}

}  // namespace lcmap
}  // namespace b2s
