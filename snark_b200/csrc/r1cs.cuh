// Device-resident R1CS matrices, GR1CS predicates and Groth16 proving key (the handles behind b2s_r1cs / b2s_gr1cs / b2s_pk).
#pragma once
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.cuh"

struct b2s_r1cs {
    uint64_t n_rows = 0, n_instance = 0, n_witness = 0;
    uint32_t log_domain = 0;          // domain = next_pow2(n_rows + n_instance)
    uint64_t nnz[3] = {0, 0, 0};
    // CSR per matrix; coefficients interned: id 0 == ONE (multiplication skipped, as
    // relations/src/sr1cs/mod.rs:42-46 does), other ids index `pool`.
    b2s::DevBuf row_ptr[3];           // uint64[n_rows + 1]
    b2s::DevBuf col[3];               // uint32[nnz]
    b2s::DevBuf coeff_id[3];          // uint32[nnz]
    b2s::DevBuf pool;                 // Fr[pool_size]
    uint32_t pool_size = 0;
    // set by b2s_r1cs_upload_lcmap_outline only: the instance variables copied into witnesses (b2s_r1cs_outline_assignment)
    uint64_t outline_copies = 0;
};

namespace b2s {
// One polynomial predicate of a GR1CS (predicate/mod.rs, polynomial_constraint.rs): argument j's matrix in CSR, coefficients
// interned into the handle's pool, and the polynomial as flattened terms (term t = coeff[t] * prod over factors
// [term_off[t], term_off[t+1]) of x[factor_var]^factor_pow).
struct Gr1csPredicate {
    uint32_t arity = 0, n_terms = 0;
    uint64_t n_rows = 0;
    uint64_t nnz[B2S_GR1CS_MAX_ARITY] = {};
    DevBuf row_ptr[B2S_GR1CS_MAX_ARITY];   // uint64[n_rows + 1], j < arity
    DevBuf col[B2S_GR1CS_MAX_ARITY];       // uint32[nnz]
    DevBuf coeff_id[B2S_GR1CS_MAX_ARITY];  // uint32[nnz]
    DevBuf term_coeff;                     // Fr[n_terms]
    DevBuf term_off;                       // uint32[n_terms + 1]
    DevBuf factor_var, factor_pow;         // uint32[term_off[n_terms]]
};
}  // namespace b2s

struct b2s_gr1cs {
    int curve = 0;                        // of the ctx that uploaded it
    uint64_t n_instance = 0, n_witness = 0;
    b2s::DevBuf pool;                     // Fr[pool_size], shared by every predicate; id 0 == ONE
    uint32_t pool_size = 0;
    std::vector<std::unique_ptr<b2s::Gr1csPredicate>> preds;   // upload order
    // set by b2s_r1cs_to_sr1cs only: orig[new column] = the source column it copies (ONE and squares: 0), the source's
    // n_instance + n_witness and rows; what b2s_sr1cs_assignment needs besides the predicate itself
    b2s::DevBuf sr1cs_orig;               // uint32[n_instance + n_witness]
    uint64_t sr1cs_src_vars = 0, sr1cs_rows = 0;
    // set by b2s_gr1cs_upload_lcmap_outline only: the instance variables copied into witnesses (b2s_gr1cs_outline_assignment)
    uint64_t outline_copies = 0;
};

namespace b2s {
// Coefficient interning of the matrix uploads (host, once per circuit; byte comparisons only -- no field arithmetic), like the
// reference's FieldInterner (relations/src/gr1cs/field_interner.rs:13-35): id 0 is ONE, whose multiplication the kernels
// skip; every other value gets the next id on first use.
struct Key32 {
    uint64_t w[4];
    bool operator==(const Key32& o) const { return w[0] == o.w[0] && w[1] == o.w[1] && w[2] == o.w[2] && w[3] == o.w[3]; }
};
struct Key32Hash {
    size_t operator()(const Key32& k) const {
        uint64_t h = k.w[0] * 0x9E3779B97F4A7C15ull;
        h ^= (k.w[1] + 0x7F4A7C15ull) * 0xC2B2AE3D27D4EB4Full;
        h ^= (k.w[2] + 0x165667B1ull) * 0x9E3779B97F4A7C15ull;
        h ^= (k.w[3] + 0x27D4EB2Full) * 0xC2B2AE3D27D4EB4Full;
        return (size_t)(h ^ (h >> 29));
    }
};
struct CoeffInterner {
    Key32 one;
    std::unordered_map<Key32, uint32_t, Key32Hash> ids;
    std::vector<Key32> pool;
    explicit CoeffInterner(const Key32& one_mont) : one(one_mont) {
        pool.push_back(one);
        ids.emplace(one, 0u);
    }
};
// Montgomery ONE of a field's parameters as an interning key
template <class P>
inline Key32 fr_one_key() {
    uint32_t o[8];
    for (int i = 0; i < 8; i++) o[i] = P::r1(i);
    Key32 k;
    memcpy(k.w, o, 32);
    return k;
}
// Checks one CSR matrix (row_ptr[0] == 0, columns < n_vars, row_ptr monotone), interns its coefficients and copies row_ptr,
// col and the coefficient ids to the device.  Failure messages read "<who>: row_ptr[<k>] ...".  Shared by b2s_r1cs_upload
// (k = matrix) and b2s_gr1cs_upload (k = argument).
int32_t csr_intern_upload(Ctx* c, CoeffInterner& in, const char* who, int k, uint64_t n_rows, uint64_t n_vars, const uint64_t* row_ptr,
                          const uint32_t* col, const void* coeff, DevBuf& d_row_ptr, DevBuf& d_col, DevBuf& d_cid, uint64_t* nnz);
// the interned values to the device: *pool_size = in.pool.size()
int32_t coeff_pool_upload(Ctx* c, const CoeffInterner& in, const char* who, DevBuf& pool, uint32_t* pool_size);

// gr1cs.cu
int32_t gr1cs_upload(Ctx* c, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates, const b2s_predicate_desc* preds,
                     b2s_gr1cs** out);
// the same handle from the constraint system's LcMap: the argument matrices by lcmap_build, the pool kept as the caller's
struct LcMapHost;
// ol: instance outlining as finalize() does it with an InstanceOutliner (lcmap.cuh), or null for none
int32_t gr1cs_upload_lcmap(Ctx* c, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates, const b2s_predicate_lcmap_desc* preds,
                           const LcMapHost& lm, const b2s_outline* ol, b2s_gr1cs** out);
// first_unsat / n_unsat (n_unsat may be null): n_assign x n_predicates, in `mem` like z
int32_t gr1cs_check(Ctx* c, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, uint64_t* first_unsat, uint64_t* n_unsat);
int32_t r1cs_check(Ctx* c, const b2s_r1cs* m, uint64_t n_assign, const void* z, int32_t mem, uint64_t* first_unsat, uint64_t* n_unsat);
// sr1cs.cu: the square R1CS of an R1CS handle, its assignments, and the read-back of any GR1CS handle
int32_t r1cs_to_sr1cs(Ctx* c, const b2s_r1cs* m, b2s_gr1cs** out);
int32_t sr1cs_assignment(Ctx* c, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z);
int32_t gr1cs_info(Ctx* c, const b2s_gr1cs* g, uint64_t* n_vars, uint32_t* n_predicates, b2s_gr1cs_pred_info* preds, uint32_t cap);
int32_t gr1cs_export(Ctx* c, const b2s_gr1cs* g, uint32_t pred, uint32_t arg, uint64_t* row_ptr, uint64_t cap_row_ptr, uint32_t* col,
                     uint64_t cap_col, void* coeff, uint64_t cap_coeff);
// The five query vectors of a proving key, in the order of b2s_pk_query's `which`.
enum PkQueryId { Q_A, Q_B_G1, Q_B_G2, Q_H, Q_L, PK_QUERIES };
// Where the scalars of a query's MSM start: z + off, z + n_instance + off (the witness), or the h shard (HSource).
enum PkScalars { FROM_Z, FROM_WITNESS, FROM_H };
// What is fixed per query.  The shard that owns the end of an a / b range also owns two extra (base, scalar) pairs with
// scalars (r, s): a appends [delta, O], b_g1 and b_g2 append [O, delta] (delta of the query's group).  h and l append
// [O, O] and never use them.
struct PkQueryInfo {
    const char* name;       // in error messages
    int group;
    int delta_at;           // which extra pair holds delta: 0, 1, or -1 for none (no extra pairs)
    PkScalars scalars;
};
inline constexpr PkQueryInfo PK_QUERY[PK_QUERIES] = {{"a_query", 1, 0, FROM_Z},
                                                     {"b_g1_query", 1, 1, FROM_Z},
                                                     {"b_g2_query", 2, 1, FROM_Z},
                                                     {"h_query", 1, -1, FROM_H},
                                                     {"l_query", 1, -1, FROM_WITNESS}};
struct PkQuery {
    DevBuf pts;                       // affine points [len + 2]: the two extra points follow the range
    uint64_t off = 0, len = 0;        // indices into the full vector held by this shard
    uint32_t ext = 0;                 // 2 when the extra pairs belong to the MSM (this shard owns the end of the range)
};
}  // namespace b2s

struct b2s_pk {
    uint64_t n_instance = 0, n_witness = 0, domain_size = 0;
    // the QAP reduction the key was made for (B2S_QAP_LIBSNARK / B2S_QAP_CIRCOM), fixed when the handle is created: it selects
    // the witness map of every proof under the key and the length of a full key's h query
    int32_t qap = B2S_QAP_LIBSNARK;
    b2s::DevBuf consts_g1;            // alpha_g1, beta_g1, delta_g1 (affine)
    b2s::DevBuf consts_g2;            // beta_g2, delta_g2 (affine)
    b2s::PkQuery q[b2s::PK_QUERIES];  // indexed by PkQueryId
    // fixed-base window table of h_query (msm_precompute): [h_pre.nwin][q[Q_H].len] affine points; empty when switched off / too big
    b2s::DevBuf h_table;
    b2s::MsmPre h_pre{0, 0, 0};
};

namespace b2s {
// length of a full key's h query: tau^i Z(tau) / delta for i < domain_size - 1 (libsnark), or the domain_size odd-indexed
// Lagrange points of the size-2N domain (circom)
inline uint64_t pk_full_h_len(int32_t qap, uint64_t domain_size) { return qap == B2S_QAP_CIRCOM ? domain_size : domain_size - 1; }
// a full (unsharded) key: every query covers its whole vector
inline bool pk_is_full(const b2s_pk* pk) {
    const uint64_t n_vars = pk->n_instance + pk->n_witness;
    const PkQuery* q = pk->q;
    return q[Q_A].len == n_vars && q[Q_B_G1].len == n_vars && q[Q_B_G2].len == n_vars && q[Q_L].len == pk->n_witness &&
           q[Q_H].len == pk_full_h_len(pk->qap, pk->domain_size);
}

int32_t r1cs_upload(Ctx* c, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness, const uint64_t* const row_ptr[3],
                    const uint32_t* const col[3], const void* const coeff[3], b2s_r1cs** out);
// lcmap.cu: argument matrices built on the device from the constraint system's flat LcMap (lcmap.cuh), shared by
// b2s_r1cs_upload_lcmap (A, B, C) and b2s_gr1cs_upload_lcmap (every argument of every predicate)
struct LcMapHost {               // host pointers, as the caller holds them
    uint64_t n_lcs;
    const uint64_t* offsets;     // n_lcs + 1
    const uint64_t* vars;        // offsets[n_lcs] raw Variables
    const uint32_t* coeffs;      // offsets[n_lcs] ids into pool
    const void* pool;            // pool_len Montgomery Fr, pool[0] = ONE
    uint32_t pool_len;
};
// one argument matrix: n_rows raw Variables in (host), a CSR whose coefficient ids index the caller's pool out.  n_tie
// more rows follow the caller's: the tie rows of instance outlining, whose arguments lcmap_build makes on the device.
struct LcMatrix {
    const uint64_t* args;
    uint64_t n_rows;
    DevBuf* row_ptr;             // uint64[n_rows + n_tie + 1]
    DevBuf* col;                 // uint32[nnz]
    DevBuf* coeff_id;            // uint32[nnz]
    uint64_t* nnz;
    uint64_t n_tie = 0;
};
// Instance outlining in lcmap_build: W = the witnesses before outlining, n_instance copies follow them; the tie rows go
// to the matrices mats[first_mat + j], j < arity of the strategy (3 for B2S_OUTLINE_R1CS, 2 for B2S_OUTLINE_SR1CS)
struct LcOutline {
    int32_t strategy;
    uint64_t n_witness;
    size_t first_mat;
};
// The checks of the LcMap itself, made before anything is allocated; n_slots: the rows of all matrices together.
int32_t lcmap_validate(Ctx* c, const LcMapHost& lm, uint64_t n_slots);
// The checks of an outlining descriptor against the target predicate's arity and the pool (B2S_OUTLINE_SR1CS reads
// pool[1] as -ONE), made before anything is allocated; `who` prefixes the messages.
int32_t outline_validate(Ctx* c, const char* who, const b2s_outline& ol, uint32_t n_predicates, uint32_t target_arity, const LcMapHost& lm);
// Builds every matrix of `mats` with one count, scan and fill over all their rows and copies the pool as it is to `pool`.
// where(m, row), when set, prefixes the message of a rejected argument; `what` names the matrices in the nonzero limit's.
// ol, when set, outlines the instance variables (n_vars then counts the copies).
int32_t lcmap_build(Ctx* c, const LcMapHost& lm, uint64_t n_instance, uint64_t n_vars, const std::vector<LcMatrix>& mats,
                    const char* what, const std::function<std::string(size_t, uint64_t)>& where, DevBuf& pool, uint32_t* pool_size,
                    const LcOutline* ol = nullptr);
// the same handle as r1cs_upload from the constraint system's LcMap; ol: instance outlining (B2S_OUTLINE_R1CS), or null
int32_t r1cs_upload_lcmap(Ctx* c, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness, const uint64_t* const args[3],
                          uint64_t n_lcs, const uint64_t* lc_offsets, const uint64_t* lc_vars, const uint32_t* lc_coeffs,
                          const void* pool, uint32_t pool_len, const b2s_outline* ol, b2s_r1cs** out);
// z' = z || (ONE, z[1], ..., z[n_copies - 1]) for n_assign rows of n_src elements, in `mem` like z
int32_t outline_assignment(Ctx* c, uint64_t n_src, uint64_t n_copies, uint64_t n_assign, const void* z, int32_t mem, void* out_z);
// out_k: device arrays with at least n_rows elements each
int32_t spmv_run(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* out_a, void* out_b, void* out_c);
// h_dev: device array of domain elements (output); z_dev: n_instance + n_witness elements; qap: the reduction (libsnark: h's
// coefficients, circom: its odd-coset evaluations).  K > 1: K assignments at z_dev + k * z_stride (elements) give K vectors
// h_dev + k * domain, with the launches of one
int32_t witness_map_run(Ctx* c, const b2s_r1cs* m, const void* z_dev, void* h_dev, int32_t qap, uint32_t K = 1, uint64_t z_stride = 0);
int32_t pk_upload(Ctx* c, const b2s_pk_desc* d, int32_t mem, int32_t qap, b2s_pk** out);
int32_t groth16_setup(Ctx* c, const b2s_r1cs* m, const void* trapdoor_host, int32_t qap, b2s_pk** out_pk, void* o_alpha_g1, void* o_beta_g2,
                      void* o_gamma_g2, void* o_delta_g2, void* o_gamma_abc);
int32_t pk_query_download(Ctx* c, const b2s_pk* pk, int which, void* out_host, uint64_t cap_bytes);
// Where the h-query MSM of a shard takes its scalars from: the default computes the whole h on this GPU (replicated
// witness_map); the multi-GPU group computes it distributed and hands back this rank's coefficient slab (group.cu).
struct HSource {
    // z_dev: the full assignment on the device.  On return *h_for_shard points at the scalars matching pk->q[Q_H]
    // (its len elements starting at coefficient off); the memory stays valid until the HSource is destroyed.
    virtual int32_t get(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void** h_for_shard) = 0;
    virtual ~HSource() = default;
};
// z either as two host pieces (z_dev == nullptr) or as one device array; hs == nullptr: replicated witness_map
int32_t groth16_shard(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, const void* z_inst_host, const void* z_wit_host,
                      const void* z_dev, const void* r_host, const void* s_host, void* g1_partials_dev /*4 xyzz*/,
                      void* g2_partial_dev /*1 xyzz*/, HSource* hs = nullptr);
// n_proofs proofs under one full key: z holds n_proofs rows of n_instance + n_witness scalars, r and s one scalar per proof,
// out_a / out_b / out_c n_proofs affine points; all in host memory, or all on the device (mem == B2S_MEM_DEVICE)
int32_t groth16_prove_batch(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, uint64_t n_proofs, const void* z, const void* r, const void* s,
                            int32_t mem, void* out_a, void* out_b, void* out_c);
int32_t groth16_finish(Ctx* c, const b2s_pk* pk, const void* g1_partials_dev, const void* g2_partials_dev, uint32_t n_shards,
                       const void* r_host, const void* s_host, void* out_a, void* out_b, void* out_c);
}  // namespace b2s
