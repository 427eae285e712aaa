/*
 * b200snark.h -- C ABI of libb200snark.so, the H100 (sm_90a) backend for the Groth16 prover hot path.
 *
 * The reference (arkworks-rs/snark) has NO FFI: its seam is trait-level.  Each entry point below
 * names the reference interface it sits behind (paths relative to the arkworks-rs/snark tree):
 *
 *   SNARK::prove / CircuitSpecificSetupSNARK::setup      snark/src/lib.rs:43-54, 84-93
 *   ConstraintSystem::to_matrices()                      relations/src/gr1cs/constraint_system.rs:768-774
 *   instance_assignment() / witness_assignment()         relations/src/gr1cs/constraint_system.rs:193-206
 *   Matrix<F>, mat_vec_mul                               relations/src/utils/matrix.rs:4,26-36
 *   Sr1csAdapter::evaluate_constraint                    relations/src/sr1cs/mod.rs:24-56
 *   ConstraintSystem::is_satisfied / which_is_unsatisfied relations/src/gr1cs/constraint_system.rs:652-687
 *   SynthesisError (status codes)                        relations/src/utils/error.rs:5-21
 *   (out of tree, SURVEY.md App. A)  ark-poly Radix2EvaluationDomain::{fft,ifft}, get_coset;
 *                                    ark-ec VariableBaseMSM::msm; ark-groth16 prover / generator
 *
 * DATA CONVENTIONS (what a Rust caller already has in memory):
 *   - Field element: little-endian limbs, MONTGOMERY form with R = 2^(64*N64), N64 = 4 for both
 *     scalar fields and BN254 Fq, 6 for BLS12-381 and BLS12-377 Fq.  Identical to ark-ff `Fp<MontBackend>`'s in-memory
 *     `BigInt<N>` -- `&[F]` can be passed as is.  "canonical" scalars (ark `into_bigint()`) are accepted
 *     where a `scalars_mont` flag says so.
 *   - G1 affine point: x || y (2 field elements, packed, no padding).  G2 affine: x.c0 || x.c1 || y.c0 ||
 *     y.c1.  The point at infinity is ALL-ZERO bytes ((0,0) is on none of the curves).  ark-ec's `Affine`
 *     carries a separate `infinity: bool`; the adapter writes zeros for such points (INTEGRATION.md).
 *   - Matrices: CSR per matrix (row_ptr[n_rows+1] u64, col[nnz] u32, coeff[nnz] field elements) built
 *     from `to_matrices()` rows in order; duplicate / unsorted columns are allowed and are summed
 *     (constraint_system.rs:792-804 only filters zeros).  Column 0 is the constant One, columns
 *     1..n_inst-1 the instance variables, n_inst.. the witnesses (relations/src/utils/variable.rs:105-113).
 *   - z = instance_assignment || witness_assignment, z[0] == 1 (relations/src/sr1cs/mod.rs:199-200).
 *
 * OWNERSHIP: caller-owned buffers are only read/written during the call.  `mem` says where a buffer
 * lives: B2S_MEM_HOST (any host pointer, pageable or pinned; copied to and from device scratch with stream-ordered copies,
 * and batches in bounded chunks) or B2S_MEM_DEVICE (a device pointer on the ctx's GPU, e.g. torch tensor storage, used
 * in place).  Any `mem` other than B2S_MEM_DEVICE means the host.  Handles are freed by b2s_*_free.
 *
 * THREADING: one in-flight call per ctx (calls on one ctx are serialised by an internal mutex).
 * ERRORS: never unwinds (reference builds with panic=abort for FFI, Cargo.toml:33); int32 status.
 * NO CPU FALLBACK: every entry point fails with B2S_ERR_NO_DEVICE when no sm_90 GPU is usable.
 */
#ifndef B200SNARK_H
#define B200SNARK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2S_CURVE_BLS12_381 0
#define B2S_CURVE_BN254 1
#define B2S_CURVE_BLS12_377 2   /* ark-bls12-377: Fq 377 bits (N64 = 6), Fr 253 bits (N64 = 4), SWFlags serialization */

#define B2S_MEM_HOST 0
#define B2S_MEM_DEVICE 1

/* QAP reduction of a Groth16 key (ark-groth16's R1CSToQAP): fixed when the device-resident key is created, it selects the
 * witness map of every proof under the key and the form of its h query.
 *   B2S_QAP_LIBSNARK  ark-groth16's LibsnarkReduction (Groth16<E>): h = coefficients of (A B - C) / Z, |h_query| = N - 1,
 *                     h_query[i] = tau^i Z(tau) / delta.  What every entry point without a `qap` argument uses.
 *   B2S_QAP_CIRCOM    ark-circom's CircomReduction (Groth16<E, CircomReduction>, snarkjs keys): with w2 a primitive 2N-th
 *                     root (w2^2 = w) and x_j = w2 w^j the odd coset, h_j = a_j b_j - c_j where a, b are A z and B z (instance
 *                     rows in a) and c = (A z) o (B z) on H, all three moved to x_j; C is never read.  |h_query| = N,
 *                     h_query[j] = L^(2N)_{2j+1}(tau) / delta (the odd-indexed Lagrange basis of the size-2N domain, as snarkjs
 *                     writes it).  The rest of the key and the proof are unchanged; the verifiers below take circom proofs as
 *                     they are.  Not provided: the distributed witness map (b2s_groth16_prove_group* refuse circom keys with
 *                     B2S_ERR_INVALID_ARG; b2s_groth16_prove_shard + b2s_groth16_finish work).  snarkjs .zkey and circom
 *                     .wtns and .r1cs files load directly: b2s_zkey_load / b2s_wtns_read / b2s_r1cs_file_load below.
 * Any other value is B2S_ERR_INVALID_ARG. */
#define B2S_QAP_LIBSNARK 0
#define B2S_QAP_CIRCOM 1

/* status codes; 1..7 mirror SynthesisError (relations/src/utils/error.rs:5-21) */
#define B2S_OK 0
#define B2S_ERR_MISSING_CS 1
#define B2S_ERR_ASSIGNMENT_MISSING 2        /* z / scalar length does not match the uploaded matrices / key */
#define B2S_ERR_DIVISION_BY_ZERO 3
#define B2S_ERR_UNSATISFIABLE 4
#define B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE 5 /* domain larger than 2^two_adicity or than the backend limit */
#define B2S_ERR_UNEXPECTED_IDENTITY 6
#define B2S_ERR_MALFORMED_VK 7
#define B2S_ERR_INVALID_ARG 16
#define B2S_ERR_NO_DEVICE 17
#define B2S_ERR_CUDA 18
#define B2S_ERR_OOM 19
#define B2S_ERR_NCCL 20
#define B2S_ERR_INVALID_DATA 21             /* SerializationError::InvalidData: bad flags or length, coordinate >= p, not on
                                               the curve, not in the prime-order subgroup */

typedef struct b2s_ctx b2s_ctx;
typedef struct b2s_r1cs b2s_r1cs;   /* device-resident A/B/C in CSR (witness independent; upload once per circuit) */
typedef struct b2s_pk b2s_pk;       /* device-resident Groth16 proving key (or one base-range shard of it) */
typedef struct b2s_pvk b2s_pvk;     /* device-resident PreparedVerifyingKey (b2s_vk_prepare) */

/* ---- context ------------------------------------------------------------------------------ */
int32_t b2s_ctx_create(int32_t curve_id, int32_t device_ordinal, b2s_ctx** out);
void b2s_ctx_destroy(b2s_ctx* ctx);
const char* b2s_last_error(const b2s_ctx* ctx);      /* text of the last failure on this ctx */
const char* b2s_version(void);
/* sizes in bytes for the ctx's curve: [0]=Fr, [1]=Fq, [2]=G1 affine, [3]=G2 affine, [4]=G1 xyzz, [5]=G2 xyzz */
int32_t b2s_sizes(const b2s_ctx* ctx, uint32_t out[6]);
/* kernel launches issued by this ctx since creation (bench.py's gpu_launches) */
uint64_t b2s_launch_count(const b2s_ctx* ctx);
/* block until all work queued by this ctx is done */
int32_t b2s_sync(b2s_ctx* ctx);
/* the CUDA stream (cudaStream_t) the ctx launches on, for CUDA-event timing by the harness */
void* b2s_stream(b2s_ctx* ctx);

/* Per-kernel device timing: when enabled, every kernel launch of this ctx is bracketed by CUDA events on
 * the ctx stream.  b2s_profile_report synchronises, writes one line per kernel name
 * ("<name>\t<launches>\t<total_ms>\n", NUL terminated, truncated to cap) and clears the records. */
int32_t b2s_profile_enable(b2s_ctx* ctx, int32_t on);
int32_t b2s_profile_report(b2s_ctx* ctx, char* buf, uint64_t cap);

/* ---- K2: radix-2 NTT over Fr (ark-poly Radix2EvaluationDomain::{fft,ifft}_in_place, get_coset) ----
 * In place on 2^log_n Montgomery-form elements, natural order in and out.
 *   inverse = 0: X[i] = sum_j x[j] (c w^i)^j            inverse = 1: the inverse map (includes 1/N)
 *   coset   = 0: c = 1                                  coset = 1: c = Fr::GENERATOR (7 / 5)          */
int32_t b2s_ntt(b2s_ctx* ctx, void* data, uint32_t log_n, int32_t inverse, int32_t coset, int32_t mem);

/* ---- K4: variable-base MSM (ark-ec VariableBaseMSM::msm / msm_bigint) --------------------------
 * out = sum_i scalars[i] * bases[i], i < n.  Result written to HOST memory as one affine point.
 * scalars_mont = 1: scalars are Montgomery-form Fr (`&[Fr]`); 0: canonical integers (`into_bigint()`). */
int32_t b2s_msm_g1(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont,
                   int32_t mem, void* out_affine);
int32_t b2s_msm_g2(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont,
                   int32_t mem, void* out_affine);
/* Shard form for multi-GPU: same sum, returned un-normalised (X,Y,ZZ,ZZZ) to HOST so that ranks can
 * exchange partials (all-gather) and finish with b2s_g{1,2}_sum. */
int32_t b2s_msm_g1_partial(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont,
                           int32_t mem, void* out_xyzz);
int32_t b2s_msm_g2_partial(b2s_ctx* ctx, const void* bases, const void* scalars, uint64_t n, int32_t scalars_mont,
                           int32_t mem, void* out_xyzz);
/* out_affine = sum of `count` XYZZ points (HOST in, HOST out). */
int32_t b2s_g1_sum(b2s_ctx* ctx, const void* xyzz, uint32_t count, void* out_affine);
int32_t b2s_g2_sum(b2s_ctx* ctx, const void* xyzz, uint32_t count, void* out_affine);

/* ---- K1: R1CS matrices x assignment (Matrix<F>, mat_vec_mul, evaluate_constraint) --------------
 * Upload A, B, C once per circuit.  row_ptr[k] has n_rows+1 entries, col[k]/coeff[k] have row_ptr[k][n_rows]. */
int32_t b2s_r1cs_upload(b2s_ctx* ctx, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                        const uint64_t* const row_ptr[3], const uint32_t* const col[3],
                        const void* const coeff[3], b2s_r1cs** out);
/* The same handle built ON THE DEVICE from the constraint system's flat storage, bypassing to_matrices()
 * (SURVEY 8(f) row 1; constraint_system.rs:768-804 get_lc + make_row done by kernels):
 *   args[k]      n_rows Variables: the k-th argument of every R1CS constraint (predicate/mod.rs:81-94 argument_lcs[k]);
 *                a Variable is the raw u64 of utils/variable.rs:4-14 (tag << 61 | index; Zero 0, One 1, Instance 2,
 *                Witness 3, SymbolicLc 4)
 *   lc_offsets   n_lcs + 1 entries, lc_vars / lc_coeffs lc_offsets[n_lcs] entries  (gr1cs/lc_map.rs:51-56)
 *   pool         the interner's `vec` (gr1cs/field_interner.rs:19-22): pool_len Montgomery field elements,
 *                pool[0] = ONE, pool[1] = -ONE; lc_coeffs index it
 * The system must be finalized (no LC may refer to another LC), otherwise B2S_ERR_INVALID_ARG.  HOST pointers. */
int32_t b2s_r1cs_upload_lcmap(b2s_ctx* ctx, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                              const uint64_t* const args[3], uint64_t n_lcs, const uint64_t* lc_offsets,
                              const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool,
                              uint32_t pool_len, b2s_r1cs** out);
void b2s_r1cs_free(b2s_ctx* ctx, b2s_r1cs* m);
/* out_k[i] = <M_k row i, z>, i < n_rows; z has n_instance + n_witness elements.  All buffers share `mem`. */
int32_t b2s_spmv(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, void* out_a, void* out_b, void* out_c);
/* h = LibsnarkReduction::witness_map (SURVEY App. A.2: SpMV -> 3 iNTT -> 3 coset NTT -> (ab-c)/Z -> coset iNTT), computed with
 * six transforms: Z is constant on the coset and deg C < N, so h = (cosetiNTT(a_coset b_coset) - iNTT(c)) / Z(g) -- the same
 * field elements for every assignment.
 * out_h receives domain_size elements (the top one is 0); domain_size = next_pow2(n_rows + n_instance). */
int32_t b2s_witness_map(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, void* out_h);
/* The witness map of either reduction (B2S_QAP_*): B2S_QAP_LIBSNARK is b2s_witness_map; B2S_QAP_CIRCOM writes the domain_size
 * odd-coset evaluations h_j = a_j b_j - c_j (CircomReduction::witness_map_from_matrices), six transforms, C not read.
 * out_h receives domain_size elements under either reduction. */
int32_t b2s_witness_map_qap(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, int32_t qap, void* out_h);
uint64_t b2s_r1cs_domain_size(const b2s_r1cs* m);
/* The same (libsnark) h computed by the DISTRIBUTED schedule of b2s_groth16_prove_group (four-step transforms, SpMV and quotient on
 * column slabs, SURVEY 8(e)) with 2^log_ranks virtual ranks on this one GPU, the all-to-all replaced by device copies.
 * Exists so that the index algebra of the multi-GPU path is checked bit for bit on a one-GPU box; B2S_ERR_INVALID_ARG
 * when the domain cannot be cut that way (log2(domain) odd, or too few rows per rank). */
int32_t b2s_witness_map_sim(b2s_ctx* ctx, const b2s_r1cs* m, const void* z, int32_t mem, uint32_t log_ranks, void* out_h);

/* ---- constraint satisfaction (ConstraintSystem::is_satisfied / which_is_unsatisfied) ------------------------------------
 * The check of relations/src/gr1cs/constraint_system.rs:652-687 (-> predicate/mod.rs:185-204 -> polynomial_constraint.rs:46-48)
 * on the GPU, for one assignment or a batch: constraint i of a polynomial predicate is satisfied when its polynomial, evaluated
 * at the arity row products <M_j row i, z>, is 0 mod r.  One thread per (constraint, assignment); the CSR reads are those of
 * b2s_spmv.  A prover computes a proof for any z (the witness map is defined for every assignment), so a service can run this
 * first and keep bad witnesses out of b2s_groth16_prove_batch.
 *   b2s_gr1cs_upload  the predicates of a GR1CS as to_matrices() (BTreeMap<Label, Vec<Matrix>>, one matrix per argument) and
 *                     get_all_predicate_types() (Predicate::Polynomial: terms, num_vars) return them; pass them in label order
 *                     to get the reference's order.  Coefficients of all matrices share one interned pool.  Errors as for
 *                     b2s_r1cs_upload: B2S_ERR_INVALID_ARG for an arity of 0 or above B2S_GR1CS_MAX_ARITY (rejected, never
 *                     truncated: the arguments live in registers), factor_var >= arity, term_offsets or row_ptr not monotone or
 *                     not starting at 0, null pointers (b2s_last_error names the predicate and the index);
 *                     B2S_ERR_ASSIGNMENT_MISSING for a column >= n_instance + n_witness; B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE for
 *                     more than 2^32 variables (columns are u32) or 2^32 or more constraints in one predicate.  HOST pointers.
 *   b2s_gr1cs_check   which_is_unsatisfied for n_assign assignments (below).  A handle from another curve's ctx is
 *                     B2S_ERR_INVALID_ARG.
 *   b2s_r1cs_check    the same on a Groth16 handle, with the R1CS predicate x0 * x1 - x2 over its A, B, C (n_predicates = 1).
 *                     A handle whose C was left empty for the circom reduction checks a * b = 0.
 * z: n_assign rows of n_instance + n_witness Montgomery Fr (z[0] = 1, as for b2s_groth16_prove_batch).
 * first_unsat[i * n_predicates + p] = the index of the first constraint of predicate p (upload order) that assignment i does not
 * satisfy, or UINT64_MAX; n_unsat (may be NULL) the number of such constraints, same layout.  z and the outputs share `mem`; host
 * batches go through bounded device scratch in chunks.  n_assign == 0 -> B2S_OK, nothing written.  An unsatisfied assignment is
 * a result, not an error. */
#define B2S_GR1CS_MAX_ARITY 8
typedef struct b2s_gr1cs b2s_gr1cs;        /* device-resident predicates of a GR1CS (to_matrices() + get_all_predicate_types()) */
typedef struct b2s_predicate_desc {
    uint32_t arity;                        /* 1..B2S_GR1CS_MAX_ARITY (PolynomialPredicate::arity = num_vars) */
    uint32_t n_terms;                      /* 0 = the zero polynomial: every constraint satisfied */
    const void* term_coeffs;               /* n_terms Montgomery Fr */
    const uint32_t* term_offsets;          /* n_terms + 1; term t = coeff_t * prod over [off_t, off_t+1) of x[var]^pow */
    const uint32_t* factor_var;            /* < arity */
    const uint32_t* factor_pow;            /* any u32; x^0 = 1 (ark-poly SparseTerm) */
    uint64_t n_rows;                       /* this predicate's num_constraints */
    const uint64_t* row_ptr[B2S_GR1CS_MAX_ARITY];   /* argument j's matrix, CSR exactly as b2s_r1cs_upload, j < arity */
    const uint32_t* col[B2S_GR1CS_MAX_ARITY];
    const void* coeff[B2S_GR1CS_MAX_ARITY];
} b2s_predicate_desc;
int32_t b2s_gr1cs_upload(b2s_ctx* ctx, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates,
                         const b2s_predicate_desc* preds, b2s_gr1cs** out);
/* The same handle built ON THE DEVICE from the constraint system's flat storage, bypassing to_matrices() for every predicate,
 * as b2s_r1cs_upload_lcmap does for the R1CS one: one descriptor per entry of predicate_constraint_systems (pass them in label
 * order), each with its polynomial as in b2s_predicate_desc and, for argument j < arity, get_constraints()[j]: n_rows raw
 * Variables.  All predicates share one LcMap and one interner pool, laid out as for b2s_r1cs_upload_lcmap; the pool is kept
 * as it is, not re-interned.  Row i of argument j is make_row(get_lc(args[j][i])): Zero gives no terms, SymbolicLc(k) the
 * terms of LC k, any other variable the single term (ONE, v); terms with a zero coefficient or the Zero variable are dropped,
 * repeated columns stay.  For every z b2s_gr1cs_check then gives what it gives on the b2s_gr1cs_upload handle of
 * to_matrices().  Rejected, with the status codes of b2s_gr1cs_upload: a descriptor it rejects (args[j] null with
 * n_rows > 0 included), checked before anything is allocated; and with those of b2s_r1cs_upload_lcmap: an LcMap it rejects
 * (B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE also for 2^32 or more (argument, row) slots or nonzeros over all predicates).
 * b2s_last_error names the predicate (upload index) and, for a rejected argument, the argument and the constraint.
 * HOST pointers; the call returns after the last copy, so the caller may free them. */
typedef struct b2s_predicate_lcmap_desc {
    uint32_t arity;                        /* as b2s_predicate_desc */
    uint32_t n_terms;
    const void* term_coeffs;
    const uint32_t* term_offsets;
    const uint32_t* factor_var;
    const uint32_t* factor_pow;
    uint64_t n_rows;                       /* this predicate's num_constraints */
    const uint64_t* args[B2S_GR1CS_MAX_ARITY];   /* get_constraints()[j]: n_rows raw Variables, j < arity */
} b2s_predicate_lcmap_desc;
int32_t b2s_gr1cs_upload_lcmap(b2s_ctx* ctx, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates,
                               const b2s_predicate_lcmap_desc* preds, uint64_t n_lcs, const uint64_t* lc_offsets,
                               const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len,
                               b2s_gr1cs** out);
void b2s_gr1cs_free(b2s_ctx* ctx, b2s_gr1cs* g);
int32_t b2s_gr1cs_check(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem,
                        uint64_t* first_unsat, uint64_t* n_unsat);
int32_t b2s_r1cs_check(b2s_ctx* ctx, const b2s_r1cs* m, uint64_t n_assign, const void* z, int32_t mem,
                       uint64_t* first_unsat, uint64_t* n_unsat);

/* ---- R1CS -> square R1CS (Sr1csAdapter, relations/src/sr1cs/mod.rs:18-265) ----------------------------------------------
 *   b2s_r1cs_to_sr1cs     Sr1csAdapter::r1cs_to_sr1cs (sr1cs/mod.rs:124-183), built on the device.  Row i of a * b = c becomes
 *                         (a + b)^2 = 4c + s_i (row 2i) and (a - b)^2 = s_i (row 2i + 1), one new witness s_i per row.  Scanning
 *                         the rows in order (A_i, B_i, C_i as stored, then s_i), every column other than ONE gets the next
 *                         witness the first time it occurs, public and private alike; unused columns are dropped.  Each used
 *                         public column p_k (increasing p) gets the input 1 + k and the row 2m + k: w(p_k) - x_k = 0 squared.
 *                         Result: one predicate "SR1CS" of arity 2, polynomial x0^2 - x1, 2m + P rows; n_instance = 1 + P,
 *                         n_witness = (used columns other than ONE) + m; witness w at column 1 + P + w.  Repeated columns
 *                         stay and the order of terms within a row may differ from the reference's; row sums are exactly its.
 *                         The pool becomes [pool | -pool | 4 pool].  The handle records what b2s_sr1cs_assignment needs and
 *                         holds no pointer to m, which may be freed.  A handle whose C was left empty for the circom
 *                         reduction (b2s_zkey_load) converts a * b = 0.  B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE for 2^32 or
 *                         more variables or constraints in the result, or for 2^32 or more nonzeros plus rows in m.
 *   b2s_sr1cs_assignment  with the call above, Sr1csAdapter::r1cs_to_sr1cs_with_assignment (sr1cs/mod.rs:191-265): z holds
 *                         n_assign rows of m's n_instance + n_witness Montgomery Fr, out_z receives n_assign rows of the
 *                         result's n_instance + n_witness: z'[0] = 1, z'[1 + k] = z[p_k], a column's witness z[col], and
 *                         s_i = (<A_i, z> - <B_i, z>)^2 (ONE terms read 1).  z and out_z share `mem`; host batches go through
 *                         bounded device scratch in chunks.  n_assign == 0 -> B2S_OK.  B2S_ERR_INVALID_ARG for a handle
 *                         that b2s_r1cs_to_sr1cs did not make.
 *   b2s_gr1cs_info        the shape of any b2s_gr1cs handle: n_vars[0] = n_instance, n_vars[1] = n_witness, *n_predicates, and
 *                         for the first min(cap, n_predicates) predicates (upload order) their arity, rows and nonzeros.
 *   b2s_gr1cs_export      argument `arg` of predicate `pred` as to_matrices() holds it, in CSR to HOST buffers of the given
 *                         byte capacities: row_ptr (n_rows + 1 u64), col (nnz u32), coeff (nnz Montgomery Fr, pool ids
 *                         resolved).  B2S_ERR_INVALID_ARG for a buffer too small or an index out of range.
 * A handle from another curve's ctx, or a null pointer, is B2S_ERR_INVALID_ARG. */
typedef struct b2s_gr1cs_pred_info {
    uint32_t arity;
    uint32_t reserved;
    uint64_t n_rows;
    uint64_t nnz[B2S_GR1CS_MAX_ARITY];     /* argument j < arity */
} b2s_gr1cs_pred_info;
int32_t b2s_r1cs_to_sr1cs(b2s_ctx* ctx, const b2s_r1cs* m, b2s_gr1cs** out);
int32_t b2s_sr1cs_assignment(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z);
int32_t b2s_gr1cs_info(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_vars[2], uint32_t* n_predicates, b2s_gr1cs_pred_info* preds,
                       uint32_t cap);
int32_t b2s_gr1cs_export(b2s_ctx* ctx, const b2s_gr1cs* g, uint32_t pred, uint32_t arg, uint64_t* row_ptr, uint64_t cap_row_ptr,
                         uint32_t* col, uint64_t cap_col, void* coeff, uint64_t cap_coeff);

/* ---- instance outlining (ConstraintSystem::finalize with an InstanceOutliner, constraint_system.rs:689-707, 826-863;
 *      instance_outliner.rs:40-80) -----------------------------------------------------------------------------------------
 * The LcMap uploads above, with the instance variables outlined on the device as finalize() does when an outliner is set.
 * The caller runs inline_all_lcs() (not finalize() with an outliner) and passes the LcMap and arguments as they stand then;
 * n_instance and n_witness are the counts before outlining (W = n_witness).  The result is the handle of the outlined system:
 *   - n_instance more witnesses: witness W copies One, witness W + i copies Instance(i), i >= 1; the copy of variable i is at
 *     column n_instance + W + i.
 *   - every term of every stored LC that is One or Instance(i) reads as the copy of 0 or i (Instance(0) as One).  A bare
 *     argument (a single (ONE, v), which the system never stores as an LC) keeps its column, so instances may still occur
 *     outside the tie rows, as they do upstream.
 *   - n_instance tie rows appended to predicate `pred` (upload index; the predicate the outliner's label names), not rewritten:
 *       B2S_OUTLINE_R1CS  (outline_r1cs, arity 3)   row 0: w_W * w_W = One;  row i: w_W * w_{W+i} = Instance(i); bare arguments
 *       B2S_OUTLINE_SR1CS (outline_sr1cs, arity 2)  row i: argument 0 the LC [(ONE, Instance(i)), (-ONE, w_{W+i})] (appended to
 *                                                   the LcMap; Instance(0) is column 0), argument 1 SymbolicLc(0), the empty LC
 * Rows and the order of terms within them are exactly those of to_matrices() on the host-outlined system.  Variables of the
 * LcMap are checked against the outlined system's n_instance + W + n_instance.  Rejected before anything is allocated, with
 * B2S_ERR_INVALID_ARG and b2s_last_error naming the cause: a null descriptor, an unknown strategy, pred out of range, a target
 * arity other than the strategy's, and for B2S_OUTLINE_SR1CS a pool whose pool[1] is not -ONE (field_interner.rs:32-33);
 * B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE for the 2^32 limits on slots, nonzeros and variables counted with the tie rows and the
 * copies; otherwise as the upload without outlining.
 *   b2s_gr1cs_upload_lcmap_outline  b2s_gr1cs_upload_lcmap, outlined.
 *   b2s_r1cs_upload_lcmap_outline   b2s_r1cs_upload_lcmap, outlined: B2S_OUTLINE_R1CS with pred 0 only.  The result is an
 *                                   ordinary b2s_r1cs of n_rows + n_instance rows and n_witness + n_instance witnesses (domain
 *                                   next_pow2(n_rows + 2 n_instance), B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE above the curve's
 *                                   limit): setup, proving, checks and b2s_r1cs_to_sr1cs take it as any other.
 *   b2s_gr1cs_outline_assignment /
 *   b2s_r1cs_outline_assignment     the assignment of the outlined system, as outlining appends to witness_assignment in prove
 *                                   mode: z holds n_assign rows of n_instance + W Montgomery Fr (z[0] = ONE), out_z receives
 *                                   n_assign rows of n_instance + W + n_instance: z || (ONE, z[1], ..., z[n_instance - 1]).  z and
 *                                   out_z share `mem`; host batches go through bounded device scratch in chunks.  n_assign == 0
 *                                   -> B2S_OK.  B2S_ERR_INVALID_ARG for a handle no outlining upload made. */
#define B2S_OUTLINE_R1CS 1
#define B2S_OUTLINE_SR1CS 2
typedef struct b2s_outline {
    int32_t strategy;                      /* B2S_OUTLINE_R1CS or B2S_OUTLINE_SR1CS */
    uint32_t pred;                         /* upload index of the predicate that receives the tie rows */
} b2s_outline;
int32_t b2s_gr1cs_upload_lcmap_outline(b2s_ctx* ctx, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates,
                                       const b2s_predicate_lcmap_desc* preds, uint64_t n_lcs, const uint64_t* lc_offsets,
                                       const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len,
                                       const b2s_outline* outline, b2s_gr1cs** out);
int32_t b2s_r1cs_upload_lcmap_outline(b2s_ctx* ctx, uint64_t n_rows, uint64_t n_instance, uint64_t n_witness,
                                      const uint64_t* const args[3], uint64_t n_lcs, const uint64_t* lc_offsets,
                                      const uint64_t* lc_vars, const uint32_t* lc_coeffs, const void* pool, uint32_t pool_len,
                                      const b2s_outline* outline, b2s_r1cs** out);
int32_t b2s_gr1cs_outline_assignment(b2s_ctx* ctx, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, void* out_z);
int32_t b2s_r1cs_outline_assignment(b2s_ctx* ctx, const b2s_r1cs* m, uint64_t n_assign, const void* z, int32_t mem, void* out_z);

/* ---- Groth16 (ark-groth16 ProvingKey / create_proof_with_reduction, SURVEY App. A.1) ------------
 * Query vectors are affine point arrays in HOST or DEVICE memory (`mem`); they are copied to the GPU.
 *   a_query, b_g1_query, b_g2_query: n_vars = n_instance + n_witness points
 *   h_query: domain_size - 1 points (B2S_QAP_LIBSNARK) or domain_size points (B2S_QAP_CIRCOM);  l_query: n_witness points
 * For a base-range shard (multi-GPU) pass the sub-ranges and their offsets; a full key has offsets 0.  Every h range lies in
 * [0, domain_size); a shard of a circom key holds a slice of the odd-coset points.
 */
typedef struct b2s_pk_desc {
    uint64_t n_instance, n_witness, domain_size;
    const void* alpha_g1;   /* 1 G1 affine */
    const void* beta_g1;
    const void* delta_g1;
    const void* beta_g2;    /* 1 G2 affine */
    const void* delta_g2;
    const void* a_query;    uint64_t a_off, a_len;     /* indices into the full vector held by this shard */
    const void* b_g1_query; uint64_t b1_off, b1_len;
    const void* b_g2_query; uint64_t b2_off, b2_len;
    const void* h_query;    uint64_t h_off, h_len;
    const void* l_query;    uint64_t l_off, l_len;
} b2s_pk_desc;
int32_t b2s_pk_upload(b2s_ctx* ctx, const b2s_pk_desc* desc, int32_t mem, b2s_pk** out);
/* The same for a key of either reduction; b2s_pk_upload is the B2S_QAP_LIBSNARK case.  Under B2S_QAP_CIRCOM a full key has
 * h_len == domain_size; a full-looking key with h_len == domain_size - 1 is B2S_ERR_MALFORMED_VK. */
int32_t b2s_pk_upload_qap(b2s_ctx* ctx, const b2s_pk_desc* desc, int32_t mem, int32_t qap, b2s_pk** out);
void b2s_pk_free(b2s_ctx* ctx, b2s_pk* pk);

/* CircuitSpecificSetupSNARK::setup (snark/src/lib.rs:84-93) on the GPU for uploaded matrices.  `trapdoor` = 5 Montgomery
 * Fr on the HOST: tau, alpha, beta, gamma, delta, drawn by the caller from its rng (as ark-groth16's generator does).
 * Returns the device-resident proving key and writes the verifying-key elements to the HOST: alpha_g1 (G1),
 * beta_g2, gamma_g2, delta_g2 (G2), gamma_abc_g1 (n_instance G1 points). */
int32_t b2s_groth16_setup(b2s_ctx* ctx, const b2s_r1cs* m, const void* trapdoor, b2s_pk** out_pk, void* out_alpha_g1,
                          void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1);
/* The same for either reduction; b2s_groth16_setup is the B2S_QAP_LIBSNARK case.  B2S_QAP_CIRCOM builds the N-point circom
 * h query (see B2S_QAP_CIRCOM) and rejects tau with tau^(2N) = 1 (B2S_ERR_DIVISION_BY_ZERO).  Every other element of the key
 * and the verifying key is the same as under libsnark for the same trapdoor, and so are the proofs of a satisfying
 * assignment with the same r, s. */
int32_t b2s_groth16_setup_qap(b2s_ctx* ctx, const b2s_r1cs* m, const void* trapdoor, int32_t qap, b2s_pk** out_pk,
                              void* out_alpha_g1, void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2,
                              void* out_gamma_abc_g1);
/* Copy one vector of a device-resident key to the HOST (to serialise a ProvingKey):
 * which = 0 a_query, 1 b_g1_query, 2 b_g2_query, 3 h_query, 4 l_query, 5 [alpha,beta,delta]_g1, 6 [beta,delta]_g2. */
int32_t b2s_pk_query(b2s_ctx* ctx, const b2s_pk* pk, int32_t which, void* out, uint64_t cap_bytes);

/* One proof on one GPU (full key).  z_instance (n_instance, z[0] = 1), z_witness, r, s: Montgomery Fr, HOST.
 * Outputs (HOST): A (G1 affine), B (G2 affine), C (G1 affine) -- `Proof { a, b, c }`.
 * This and every prove / shard / serialize entry point below run under the key's own reduction (B2S_QAP_*). */
int32_t b2s_groth16_prove(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_instance,
                          const void* z_witness, const void* r, const void* s, void* out_a_g1, void* out_b_g2,
                          void* out_c_g1);
/* Same, with z = instance || witness already resident on the GPU (n_instance + n_witness elements). */
int32_t b2s_groth16_prove_resident(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void* r,
                                   const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1);
/* n_proofs proofs under one full key in one call.  z: n_proofs rows of n_instance + n_witness Montgomery Fr, row i =
 * proof i's instance || witness with z[0] = 1 (as b2s_groth16_prove_resident takes one); r, s: n_proofs Montgomery Fr each.
 * Outputs: n_proofs affine A (G1), B (G2) and C (G1).  Every buffer is in `mem` (B2S_MEM_HOST or B2S_MEM_DEVICE).
 * Proof i is bit-identical to b2s_groth16_prove on (z_i, r_i, s_i).  Errors as b2s_groth16_prove; n_proofs == 0 returns
 * B2S_OK and writes nothing.  Host batches go through bounded device scratch in chunks, so n_proofs is not limited by device
 * memory.  Within a chunk the witness maps and each of the five MSMs run batched, with the launches of one proof.  The batch
 * MSMs do not use the multiplicity-aware front end of the single-proof path (repeated witness values, e.g. 0 / 1 heavy
 * witnesses, cost the batch full Pippenger price).
 * When to use which (H100 80GB HBM3, 400 W, DESIGN.md section 4): for 16 or more proofs at domains up to 2^16 the batch
 * wins, 2.9x to 25x over a loop of b2s_groth16_prove_resident; at 2^20 it wins 1.1x (BLS12-381) / 1.5x (BN254) on uniform
 * witnesses and LOSES (0.5x to 0.7x) on witnesses made of a few repeated values, where the loop's front end pays off; a
 * single proof (n_proofs == 1) is 7 % to 17 % slower than b2s_groth16_prove_resident.  Large single proofs (2^20 and up with
 * repeated witness values, 2^24) belong to the single-proof entry points. */
int32_t b2s_groth16_prove_batch(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, uint64_t n_proofs, const void* z,
                                const void* r, const void* s, int32_t mem, void* out_a_g1, void* out_b_g2, void* out_c_g1);
/* Shard step for multi-GPU: computes this shard's five MSM partial sums
 *   out_partials = [ h_acc, l_acc, a_acc, b1_acc ] (4 G1 XYZZ) and out_b2_partial (1 G2 XYZZ), HOST.
 * r, s are needed here too: the shard that owns the end of a query range folds r*delta / s*delta into its MSMs. */
int32_t b2s_groth16_prove_shard(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_instance,
                                const void* z_witness, const void* r, const void* s, void* out_g1_partials,
                                void* out_g2_partial);
/* Same with z resident on the GPU. */
int32_t b2s_groth16_prove_shard_resident(b2s_ctx* ctx, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void* r,
                                         const void* s, void* out_g1_partials, void* out_g2_partial);
/* Join: sums the per-shard partials (n_shards x 4 G1 XYZZ, n_shards G2 XYZZ) and applies the r/s epilogue. */
int32_t b2s_groth16_finish(b2s_ctx* ctx, const b2s_pk* pk, const void* g1_partials, const void* g2_partials,
                           uint32_t n_shards, const void* r, const void* s, void* out_a_g1, void* out_b_g2,
                           void* out_c_g1);

/* ---- multi-GPU group (SURVEY 8(b) `b2s_ctx_create(curve, n_gpus)` / 8(e)): one rank per GPU, NCCL inside -------------
 * So that ONE `SNARK::prove` (snark/src/lib.rs:50-54) drives every GPU of a box: each rank (process, or host thread with
 * its own ctx) holds a base-range SHARD of the proving key (b2s_pk_upload with offsets), the same matrices and the same z;
 * the call computes the rank's five MSM partial sums, all-gathers them with NCCL on the ctx stream (device buffers, 1.2 KiB
 * per rank -- EC addition is not an NCCL reduction) and rank 0 joins them and applies the r/s epilogue.
 * NCCL (libnccl.so.2) is bound at run time; B2S_ERR_NCCL if it is missing or fails.  world == 1 needs no NCCL.
 *   b2s_group_unique_id   rank 0 draws the NCCL id (128 bytes) and hands it to the other ranks by the host program's
 *                         own channel (torch.distributed / MPI / a file);
 *   b2s_group_create      collective over all ranks;
 *   b2s_groth16_prove_group[_resident]   collective; the proof is written on rank 0 (outputs may be NULL elsewhere). */
typedef struct b2s_group b2s_group;
#define B2S_GROUP_ID_BYTES 128
int32_t b2s_group_unique_id(uint8_t out[B2S_GROUP_ID_BYTES]);
int32_t b2s_group_create(b2s_ctx* ctx, const uint8_t id[B2S_GROUP_ID_BYTES], int32_t rank, int32_t world, b2s_group** out);
void b2s_group_destroy(b2s_group* group);
int32_t b2s_groth16_prove_group(b2s_group* group, const b2s_pk* pk_shard, const b2s_r1cs* m, const void* z_instance,
                                const void* z_witness, const void* r, const void* s, void* out_a_g1, void* out_b_g2,
                                void* out_c_g1);
int32_t b2s_groth16_prove_group_resident(b2s_group* group, const b2s_pk* pk_shard, const b2s_r1cs* m, const void* z_dev,
                                         const void* r, const void* s, void* out_a_g1, void* out_b_g2, void* out_c_g1);

/* ---- wire format (SURVEY 8(f) row 3): CanonicalSerialize::serialize_compressed of group elements / Proof --------
 * (snark/src/lib.rs:25-36 bounds).  BLS12-381: zcash/IETF big-endian form, 48 B (G1) / 96 B (G2); BN254: ark-ec
 * SWFlags little-endian form, 32 B / 64 B; BLS12-377: the same SWFlags form, 48 B / 96 B.  HOST affine Montgomery points in, bytes out; `cap` = size of `out`. */
int32_t b2s_serialize_g1_compressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap);
int32_t b2s_serialize_g2_compressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap);
/* Proof { a, b, c } -> a || b || c (192 B on BLS12-381 and BLS12-377, 128 B on BN254). */
int32_t b2s_proof_serialize_compressed(b2s_ctx* ctx, const void* a_g1, const void* b_g2, const void* c_g1, uint8_t* out,
                                       uint64_t cap);

/* serialize_uncompressed of the same types: x || y in the curve's byte / component order (96 / 192 B on BLS12-381 with only
 * the infinity bit in byte 0; 64 / 128 B on BN254 and 96 / 192 B on BLS12-377 with both SWFlags in the last byte). */
int32_t b2s_serialize_g1_uncompressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap);
int32_t b2s_serialize_g2_uncompressed(b2s_ctx* ctx, const void* affine, uint32_t count, uint8_t* out, uint64_t cap);
int32_t b2s_proof_serialize_uncompressed(b2s_ctx* ctx, const void* a_g1, const void* b_g2, const void* c_g1, uint8_t* out,
                                         uint64_t cap);
/* ark-groth16 key framing (snark/src/lib.rs:25-36: ProvingKey / VerifyingKey are CanonicalSerialize):
 *   VerifyingKey = alpha_g1 || beta_g2 || gamma_g2 || delta_g2 || Vec(gamma_abc_g1)       (Vec = u64 LE length + elements)
 *   ProvingKey   = VerifyingKey || beta_g1 || delta_g1 || Vec(a_query) || Vec(b_g1_query) || Vec(b_g2_query) ||
 *                  Vec(h_query) || Vec(l_query)
 * The vk elements are HOST affine points (what b2s_groth16_setup wrote); the proving key is the device-resident FULL key,
 * streamed through the GPU in chunks (canonical form and sign bits on the device, byte order on the host).
 * compressed = 1 / 0 selects serialize_compressed / serialize_uncompressed.  The *_size functions give the exact length. */
uint64_t b2s_vk_serialized_size(const b2s_ctx* ctx, uint64_t n_gamma_abc, int32_t compressed);
int32_t b2s_vk_serialize(b2s_ctx* ctx, const void* alpha_g1, const void* beta_g2, const void* gamma_g2, const void* delta_g2,
                         const void* gamma_abc_g1, uint64_t n_gamma_abc, int32_t compressed, uint8_t* out, uint64_t cap);
uint64_t b2s_pk_serialized_size(const b2s_ctx* ctx, const b2s_pk* pk, uint64_t vk_len, int32_t compressed);
int32_t b2s_pk_serialize(b2s_ctx* ctx, const b2s_pk* pk, const uint8_t* vk_bytes, uint64_t vk_len, int32_t compressed,
                         uint8_t* out, uint64_t cap);

/* ---- CanonicalDeserialize of the same types (the inverse of the serializers above) --------------------------------------
 * Bytes on the HOST, in the encodings above.  The raw bytes are copied to the device in chunks; flags, byte order, the
 * canonicity check (every coordinate < p), the Montgomery conversion, the square root of compressed points and the checks
 * run in CUDA kernels.  compressed = 1 / 0 as for the serializers; validate = 1 is ark's Validate::Yes (uncompressed points
 * satisfy the curve equation, every point lies in the prime-order subgroup), 0 is Validate::No.  A compressed x without a
 * square root is rejected in both modes.  Failures return B2S_ERR_INVALID_DATA and b2s_last_error names the vector, the
 * lowest failing index and the reason, e.g. "h_query[1234]: not in the prime-order subgroup".
 *   b2s_deserialize_g1/g2  `count` points from exactly `len` bytes -> HOST affine Montgomery (infinity = all-zero)
 *   b2s_proof_deserialize  Proof { a, b, c } from exactly `len` bytes
 *   b2s_vk_deserialize     VerifyingKey from the start of `in` (a ProvingKey starts with its VerifyingKey, so this reads the vk
 *                          out of pk bytes): *n_gamma_abc = |gamma_abc_g1|, *consumed = the vk's byte length; with
 *                          out_gamma_abc_g1 = NULL only those two are filled in, nothing is decoded
 *   b2s_pk_deserialize     a whole ark-groth16 ProvingKey (exactly `len` bytes) -> the device-resident full key, the same
 *                          handle b2s_pk_upload returns for the same points.  The dimensions follow from the bytes:
 *                          n_instance = |gamma_abc_g1|, n_witness = |l_query|, domain_size = |h_query| + 1 (a power of two),
 *                          |a_query| = |b_g1_query| = |b_g2_query| = n_instance + n_witness, else B2S_ERR_MALFORMED_VK.
 *   b2s_pk_deserialize_qap the same for either reduction (b2s_pk_deserialize is B2S_QAP_LIBSNARK); under B2S_QAP_CIRCOM
 *                          domain_size = |h_query| (a power of two): the bytes of a Groth16<Bn254, CircomReduction> key
 * Every Vec length prefix is checked against the bytes that remain before anything is allocated. */
int32_t b2s_deserialize_g1(b2s_ctx* ctx, const uint8_t* in, uint64_t len, uint64_t count, int32_t compressed, int32_t validate,
                           void* out_affine);
int32_t b2s_deserialize_g2(b2s_ctx* ctx, const uint8_t* in, uint64_t len, uint64_t count, int32_t compressed, int32_t validate,
                           void* out_affine);
int32_t b2s_proof_deserialize(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, void* out_a_g1,
                              void* out_b_g2, void* out_c_g1);
int32_t b2s_vk_deserialize(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, void* out_alpha_g1,
                           void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1, uint64_t cap_gamma_abc,
                           uint64_t* n_gamma_abc, uint64_t* consumed);
int32_t b2s_pk_deserialize(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, b2s_pk** out);
int32_t b2s_pk_deserialize_qap(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t compressed, int32_t validate, int32_t qap,
                               b2s_pk** out);

/* ---- snarkjs files: Groth16 .zkey and circom .wtns (ark-circom read_zkey, snarkjs zkey_utils.js / wtns_utils.js) ---------
 * The formats are restated from snarkjs / ark-circom in snark_b200/csrc/zkey.cu; they are NOT pinned against bytes written
 * by snarkjs.  Bytes on the HOST; the host reads headers and section offsets only, and every framing and size check runs
 * before anything is allocated.  Points (Montgomery little-endian limbs in the file, this library's own layout) are checked
 * on the device: every coordinate < q always; with validate = 1 also the curve equation and the prime-order subgroup.
 * Coefficient and witness values must always be < r.
 *   b2s_zkey_read_info  the framing and the header: nVars, nPublic, domainSize and the number of coefficient entries.
 *   b2s_zkey_load       a Groth16 zkey -> the handles b2s_pk_upload_qap(.., B2S_QAP_CIRCOM, ..) and b2s_r1cs_upload would
 *                       build from the same points and matrices: a full circom key (n_instance = nPublic + 1, the h query
 *                       table built as by b2s_pk_deserialize) and a matrix handle of A and B over the circuit's constraints
 *                       with an EMPTY C (snarkjs's trailing input rows are checked and left to the witness map).  On such a
 *                       handle b2s_r1cs_check checks A z o B z = 0, which is not the circuit's satisfaction: load the
 *                       circuit's .r1cs with b2s_r1cs_file_load for that (its handle proves under this key too).  The verifying key
 *                       goes to the HOST in the form b2s_vk_prepare takes: alpha_g1, beta_g2, gamma_g2, delta_g2 and
 *                       nPublic + 1 gamma_abc_g1 points (cap_gamma_abc = room in out_gamma_abc_g1).
 *   b2s_wtns_read       a .wtns -> z = instance || witness, n_vars Montgomery Fr in `mem` (HOST or DEVICE), for
 *                       b2s_groth16_prove_resident / _prove_batch (one call per row of a batch, at a row offset).
 * Errors (b2s_last_error names the section or vector, the lowest failing index and the reason, e.g.
 * "zkey B2[17]: not in the prime-order subgroup"):
 *   B2S_ERR_INVALID_DATA    bad magic, version, framing, truncation or protocol (only Groth16 = 1); a matrix, constraint or
 *                           signal field out of range; a non-canonical, off-curve or non-subgroup value; wtns z[0] != 1
 *   B2S_ERR_INVALID_ARG     q / r of another curve than the ctx's; a null buffer; cap_gamma_abc too small
 *   B2S_ERR_MALFORMED_VK    section sizes that disagree with nVars / nPublic / domainSize; missing or altered input rows;
 *                           domainSize != next_pow2(constraints + nPublic + 1)
 *   B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE  a domain past the limits of b2s_r1cs_upload
 *   B2S_ERR_ASSIGNMENT_MISSING           nWitness != n_vars (snarkjs's "Invalid witness length") */
typedef struct b2s_zkey_info { uint64_t n_vars, n_public, domain_size, n_coeffs; } b2s_zkey_info;
int32_t b2s_zkey_read_info(b2s_ctx* ctx, const uint8_t* in, uint64_t len, b2s_zkey_info* out);
int32_t b2s_zkey_load(b2s_ctx* ctx, const uint8_t* in, uint64_t len, int32_t validate, b2s_pk** out_pk, b2s_r1cs** out_m,
                      void* out_alpha_g1, void* out_beta_g2, void* out_gamma_g2, void* out_delta_g2, void* out_gamma_abc_g1,
                      uint64_t cap_gamma_abc);
int32_t b2s_wtns_read(b2s_ctx* ctx, const uint8_t* in, uint64_t len, uint64_t n_vars, int32_t mem, void* out_z);

/* ---- circom .r1cs files (ark-circom R1CSFile + to_matrices + b2s_r1cs_upload, in one call) -------------------------------
 * The format (iden3 r1cs binfile, version 1) is restated in snark_b200/csrc/zkey.cu; it is NOT pinned against bytes written
 * by circom.  Bytes on the HOST.  The host walks the 3 mConstraints count words only; every entry is decoded and checked on
 * the device.  There is no validate flag: every check is always on.
 *   b2s_r1cs_file_read_info  the framing and the header (section 1) only; allocates nothing.  domain_size =
 *                            next_pow2(nConstraints + 1 + nPubOut + nPubIn).
 *   b2s_r1cs_file_load       the circuit -> the handle b2s_r1cs_upload builds from the same matrices: n_rows = mConstraints,
 *                            n_instance = 1 + nPubOut + nPubIn, n_witness = nWires - n_instance, A, B and C filled (duplicate
 *                            wires in one linear combination are summed).  Every entry point that takes a b2s_r1cs works on
 *                            it: b2s_r1cs_check checks the circuit's own constraints, b2s_groth16_setup[_qap] makes keys under
 *                            either reduction, and it proves under the key of b2s_zkey_load (the circom witness map reads
 *                            A and B only; snarkjs's input rows stay implicit, as for the zkey's handle).
 * Errors (b2s_last_error names the section, or the constraint, matrix and entry, with the reason, e.g.
 * "r1cs constraint 17 C[2]: wire 900 not below nWires 512"):
 *   B2S_ERR_INVALID_DATA    bad magic, version or framing; truncation; a duplicate, missing or wrongly sized section; PLONK
 *                           custom-gate sections (4, 5); nWires < 1 + nPubOut + nPubIn + nPrvIn; a count that overruns
 *                           section 2, or bytes after its mConstraints constraints; a wire >= nWires; a coefficient >= r
 *   B2S_ERR_INVALID_ARG     a prime other than the ctx curve's r; a null pointer
 *   B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE  a domain past the limits of b2s_r1cs_upload (decided from the header, before the walk
 *                           or any allocation); 2^32 or more nonzeros in one matrix */
typedef struct b2s_r1cs_file_info {
    uint64_t n_wires, n_pub_out, n_pub_in, n_prv_in, n_labels, n_constraints, domain_size;
} b2s_r1cs_file_info;
int32_t b2s_r1cs_file_read_info(b2s_ctx* ctx, const uint8_t* in, uint64_t len, b2s_r1cs_file_info* out);
int32_t b2s_r1cs_file_load(b2s_ctx* ctx, const uint8_t* in, uint64_t len, b2s_r1cs** out);

/* ---- verification: pairings and batched Groth16 verify ----------------------------------------------------------------
 * The optimal ate pairing in CUDA (snark_b200/csrc/pairing.cuh): BLS12-381 loops over |x| and conjugates, BN254 over the
 * signed digits of 6x + 2 with the two Frobenius lines, BLS12-377 over the bits of x > 0 with neither.  GT is ark's Fp12 in memory (c0 = Fp6 {c0, c1, c2 : Fp2}, c1),
 * Montgomery limbs, fully reduced.  The value is a fixed power of the textbook reduced ate pairing
 * o(P, Q) = f_{|t-1|,Q}(P)^((p^12 - 1) / r):  e = o^k with k = -3 mod r (BLS12-381),
 * k = 147946756881789319005730692170996259610 (BN254) and k = 3 (BLS12-377), all coprime to r (pairing.cuh derives them).
 *   b2s_vk_prepare   SNARK::process_vk (snark/src/lib.rs:68-71): HOST affine points, as returned by b2s_groth16_setup /
 *                    b2s_vk_deserialize.  Computes e(alpha_g1, beta_g2) in GT, the line coefficients of -gamma_g2 and
 *                    -delta_g2 (ark's G2Prepared), and per gamma_abc base j >= 1 a fixed-base table of 32 x 255 affine
 *                    points for the public-input sum: 765 KiB (BLS12-381) / 510 KiB (BN254) of device memory per public
 *                    input.  B2S_ERR_MALFORMED_VK if n_gamma_abc == 0.
 *   b2s_groth16_verify_batch  SNARK::verify_with_processed_vk (lib.rs:76-80) for n_proofs proofs at once, one verdict each:
 *                    ok[i] = [ e(A_i, B_i) * e(IC_i, -gamma) * e(C_i, -delta) == e(alpha, beta) ],
 *                    IC_i = gamma_abc[0] + sum_j x_ij gamma_abc[j+1].  inputs: n_proofs x n_inputs Montgomery Fr, row-major
 *                    (NULL when n_inputs == 0); a, b, c: affine arrays; ok: n_proofs bytes (1 = accepted).  All buffers
 *                    share `mem`; host batches go through bounded device scratch in chunks, so n_proofs is not limited by
 *                    device memory.  n_inputs + 1 != n_gamma_abc -> B2S_ERR_MALFORMED_VK (ark's prepare_inputs error);
 *                    n_proofs == 0 -> B2S_OK.  Points are assumed valid, as in ark: untrusted bytes go to the _bytes form below.
 *   b2s_groth16_verify_batch_rlc  one verdict for the whole batch (bellman's groth16::batch, Zcash's batch verifier): with
 *                    caller-drawn 128-bit rho_i,
 *                      prod_i e(rho_i A_i, B_i) * e(IC*, -gamma) * e(C*, -delta) == e(alpha, beta)^S,
 *                    S = sum_i rho_i, C* = sum_i rho_i C_i, IC* = S gamma_abc[0] + sum_j (sum_i rho_i x_ij) gamma_abc[j+1]
 *                    (mod r).  One Miller loop over one pair per proof, one G1 MSM for the C terms and one final
 *                    exponentiation for the batch.  *ok = 1 when every proof is accepted.  If a proof is invalid, the batch
 *                    is accepted with probability <= 2^-128, provided (1) the rho_i are unpredictable to whoever made the
 *                    proofs: draw them from a CSPRNG for each call, and (2) every point lies in its prime-order subgroup:
 *                    decode untrusted bytes with validate = 1.  rho: n_proofs x 16 bytes, little-endian 128-bit integers,
 *                    in `mem` like inputs, a, b, c (same layouts as b2s_groth16_verify_batch); ok: one byte, always HOST,
 *                    always written.  A zero rho_i would leave proof i unchecked: B2S_ERR_INVALID_ARG, b2s_last_error names
 *                    the lowest such index.  Another curve's key or a null buffer -> B2S_ERR_INVALID_ARG;
 *                    n_inputs + 1 != n_gamma_abc -> B2S_ERR_MALFORMED_VK; n_proofs == 0 -> B2S_OK with *ok = 1.  To learn
 *                    which proofs of a rejected batch failed, run b2s_groth16_verify_batch on it.
 *   b2s_groth16_verify_batch_bytes / b2s_groth16_verify_batch_rlc_bytes  the same two checks on ark-serialized proofs as
 *                    received from untrusted parties: `proofs` is n_proofs Proofs back to back (a || b || c, as
 *                    b2s_proof_serialize_* writes them, 192 / 128 B compressed on BLS12-381 / BN254), exactly `len` bytes,
 *                    else B2S_ERR_INVALID_DATA.  compressed = 1 / 0 as for the deserializers.  Every point is decoded ON THE
 *                    DEVICE with validation always on (flags, canonical coordinates, curve equation, prime-order subgroup),
 *                    so the RLC bound above holds without a separate decoding step; the decoded points never leave the
 *                    device.  A proof that fails to decode is rejected on its own: the call does not fail for it.
 *                      ok[i]      (per proof) 1 = proof i decoded and satisfies the verification equation, else 0
 *                      *ok        (RLC, HOST, always written) 1 = every proof decoded and the combination holds
 *                      reason[i]  may be NULL; 0 = proof i decoded, else 16 * (1 + e) + r with e = 0 / 1 / 2 for a / b / c (the
 *                                 first failing element) and r the decode reason: 1 bad flags, 2 coordinate >= p, 3 not on
 *                                 the curve (or no square root), 4 not in the prime-order subgroup
 *                    `mem` covers inputs, proofs, rho, the per-proof ok and reason.  Argument errors are those of the points
 *                    entry points above; n_proofs == 0 (with len == 0) -> B2S_OK, RLC *ok = 1.
 *   b2s_pairing     Pairing::pairing, element-wise: out[i] = e(P_i, Q_i), i < n; a pair with P or Q at infinity (all-zero)
 *                    gives 1.  All buffers share `mem`. */
int32_t b2s_vk_prepare(b2s_ctx* ctx, const void* alpha_g1, const void* beta_g2, const void* gamma_g2, const void* delta_g2,
                       const void* gamma_abc_g1, uint64_t n_gamma_abc, b2s_pvk** out);
void b2s_pvk_free(b2s_ctx* ctx, b2s_pvk* pvk);
int32_t b2s_groth16_verify_batch(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                 const void* a_g1, const void* b_g2, const void* c_g1, int32_t mem, uint8_t* ok);
int32_t b2s_groth16_verify_batch_rlc(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                     const void* a_g1, const void* b_g2, const void* c_g1, const void* rho, int32_t mem,
                                     uint8_t* ok);
int32_t b2s_groth16_verify_batch_bytes(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                       const uint8_t* proofs, uint64_t len, int32_t compressed, int32_t mem, uint8_t* ok,
                                       uint8_t* reason);
int32_t b2s_groth16_verify_batch_rlc_bytes(b2s_ctx* ctx, const b2s_pvk* pvk, uint64_t n_proofs, const void* inputs, uint64_t n_inputs,
                                           const uint8_t* proofs, uint64_t len, int32_t compressed, const void* rho, int32_t mem,
                                           uint8_t* ok, uint8_t* reason);
int32_t b2s_pairing(b2s_ctx* ctx, const void* p_g1, const void* q_g2, uint64_t n, int32_t mem, void* out_gt);

/* ---- setup helper (SURVEY 8(f) row 2): fixed-base batch multiplication -------------------------
 * out[i] = scalars[i] * G (the curve's standard generator), affine, i < n.  Used to build proving keys
 * (a_query[j] = A_j(tau) G1, ...) and synthetic bases on the GPU.  scalars: Fr; all buffers share `mem`. */
int32_t b2s_fixed_base_g1(b2s_ctx* ctx, const void* scalars, uint64_t n, int32_t scalars_mont, int32_t mem, void* out);
int32_t b2s_fixed_base_g2(b2s_ctx* ctx, const void* scalars, uint64_t n, int32_t scalars_mont, int32_t mem, void* out);

/* ---- element-wise polynomial kernels: universal-setup (Marlin-style) path, SURVEY 8(f) row 4 -----
 * The reference declares that path as a trait only (UniversalSetupSNARK, snark/src/lib.rs:107-133: universal_setup / index,
 * then SNARK::prove, lib.rs:50-54); ark-marlin's AHP is generic over ark-poly-commit's `PolynomialCommitment` and ark-poly's
 * `EvaluationDomain`.  A binding accelerates those two seams: commit / open = b2s_msm_g1 over the SRS (itself
 * b2s_fixed_base_g1 of the powers of tau), every fft / ifft / coset form = b2s_ntt, matrix products = b2s_spmv, and the
 * element-wise arithmetic in between (ark-poly `Evaluations` / `DensePolynomial` operators, ark-ff `batch_inversion`) = the
 * three entry points below.  Vectors: Fr in Montgomery form, `n` elements, all in `mem`; scalars (s, c, z): ONE Montgomery Fr
 * on the HOST.  Device-memory calls are queued on the ctx stream and return without synchronising (b2s_poly_eval
 * synchronises: it returns a value).
 *   b2s_poly_op   op 0: out = a * b   1: a + b   2: a - b   3: a * s   4: a + s   5: 1 / a with 0 -> 0 (batched inversion;
 *                 not in place).  b is ignored for ops 3-5, s for ops 0-2 and 5.  out may alias a or b for ops 0-4.
 *   b2s_poly_geom out[i] = c * s^i                      (domain elements, coset points, shifted powers)
 *   b2s_poly_eval *out = sum_i coeffs[i] z^i            (out: one Montgomery Fr on the HOST) */
int32_t b2s_poly_op(b2s_ctx* ctx, int32_t op, const void* a, const void* b, const void* s, void* out, uint64_t n, int32_t mem);
int32_t b2s_poly_geom(b2s_ctx* ctx, const void* c, const void* s, uint64_t n, int32_t mem, void* out);
int32_t b2s_poly_eval(b2s_ctx* ctx, const void* coeffs, uint64_t n, const void* z, int32_t mem, void* out);

/* ---- element-wise field kernels (unit tests of the device arithmetic; K3 building blocks) -------
 * op: 0 mul, 1 add, 2 sub, 3 inverse(a), 4 neg(a), 5 to_mont(a), 6 from_mont(a), 7 sqr(a).
 * field: 0 = Fq, 1 = Fr of the ctx's curve.  HOST buffers of `count` elements. */
int32_t b2s_field_op(b2s_ctx* ctx, int32_t field, int32_t op, const void* a, const void* b, void* out, uint64_t count);
/* group: 1 or 2.  op: 0 mixed add a+b, 1 general add, 2 double a, 3 k*a (k: one canonical Fr per point).
 * HOST affine in / HOST affine out, `count` points. */
int32_t b2s_group_op(b2s_ctx* ctx, int32_t group, int32_t op, const void* a, const void* b, const void* k, void* out,
                     uint64_t count);

#ifdef __cplusplus
}
#endif
#endif /* B200SNARK_H */
