//! `Groth16B200`: ark-snark's `SNARK` trait over the H100 backend (include/b200snark.h).
//! SOURCE ONLY -- never compiled here (no Rust toolchain in the build image).  See INTEGRATION.md.
use std::os::raw::c_void;

use ark_ec::{pairing::Pairing, AffineRepr};
use ark_groth16::{Groth16, PreparedVerifyingKey, Proof, ProvingKey, VerifyingKey};
use ark_ff::PrimeField;
use ark_relations::utils::variable::{VarKind, Variable};
use ark_relations::gr1cs::{
    predicate::{polynomial_constraint::{PolynomialPredicate, SR1CS_PREDICATE_LABEL}, Predicate}, ConstraintSynthesizer, ConstraintSystem, Label, Matrix, OptimizationGoal, SynthesisError,
    R1CS_PREDICATE_LABEL,
};
use ark_snark::{CircuitSpecificSetupSNARK, SNARK};
use ark_std::{rand::{CryptoRng, RngCore}, UniformRand};

#[repr(C)] pub struct B2sCtx { _p: [u8; 0] }
#[repr(C)] pub struct B2sR1cs { _p: [u8; 0] }
#[repr(C)] pub struct B2sPk { _p: [u8; 0] }
#[repr(C)] pub struct B2sPvk { _p: [u8; 0] }
#[repr(C)] pub struct B2sGr1cs { _p: [u8; 0] }

/// Widest predicate the satisfaction check takes (its arguments live in registers); wider ones are rejected.
pub const B2S_GR1CS_MAX_ARITY: usize = 8;
#[repr(C)]
pub struct B2sPredicateDesc {
    pub arity: u32, pub n_terms: u32,
    pub term_coeffs: *const c_void, pub term_offsets: *const u32, pub factor_var: *const u32, pub factor_pow: *const u32,
    pub n_rows: u64,
    pub row_ptr: [*const u64; B2S_GR1CS_MAX_ARITY], pub col: [*const u32; B2S_GR1CS_MAX_ARITY],
    pub coeff: [*const c_void; B2S_GR1CS_MAX_ARITY],
}
/// `b2s_predicate_lcmap_desc`: a predicate's polynomial as in `B2sPredicateDesc`, and for argument j < arity
/// `get_constraints()[j]` as raw Variables (tag << 61 | index)
#[repr(C)]
pub struct B2sPredicateLcmapDesc {
    pub arity: u32, pub n_terms: u32,
    pub term_coeffs: *const c_void, pub term_offsets: *const u32, pub factor_var: *const u32, pub factor_pow: *const u32,
    pub n_rows: u64,
    pub args: [*const u64; B2S_GR1CS_MAX_ARITY],
}

/// `b2s_outline`: the outlining strategy and the upload index (label order) of the predicate that receives the tie rows
#[repr(C)]
pub struct B2sOutline {
    pub strategy: i32,
    pub pred: u32,
}

/// Which `InstanceOutliner` function the upload stands in for.  An `InstanceOutliner` holds its strategy as an opaque
/// `Rc<dyn Fn>`, so the caller names it here instead of setting it on the cs: `Outliner::R1cs` is `outline_r1cs` and
/// `Outliner::Sr1cs` is `outline_sr1cs` (instance_outliner.rs:40-80); `pred_label` is the outliner's label.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Outliner {
    R1cs = 1,
    Sr1cs = 2,
}

#[repr(C)]
#[derive(Default)]
pub struct B2sZkeyInfo { pub n_vars: u64, pub n_public: u64, pub domain_size: u64, pub n_coeffs: u64 }

#[repr(C)]
#[derive(Default)]
pub struct B2sR1csFileInfo {
    pub n_wires: u64, pub n_pub_out: u64, pub n_pub_in: u64, pub n_prv_in: u64, pub n_labels: u64, pub n_constraints: u64,
    pub domain_size: u64,
}

#[repr(C)]
pub struct B2sPkDesc {
    pub n_instance: u64, pub n_witness: u64, pub domain_size: u64,
    pub alpha_g1: *const c_void, pub beta_g1: *const c_void, pub delta_g1: *const c_void,
    pub beta_g2: *const c_void, pub delta_g2: *const c_void,
    pub a_query: *const c_void, pub a_off: u64, pub a_len: u64,
    pub b_g1_query: *const c_void, pub b1_off: u64, pub b1_len: u64,
    pub b_g2_query: *const c_void, pub b2_off: u64, pub b2_len: u64,
    pub h_query: *const c_void, pub h_off: u64, pub h_len: u64,
    pub l_query: *const c_void, pub l_off: u64, pub l_len: u64,
}

extern "C" {
    pub fn b2s_ctx_create(curve_id: i32, device: i32, out: *mut *mut B2sCtx) -> i32;
    pub fn b2s_ctx_destroy(ctx: *mut B2sCtx);
    pub fn b2s_last_error(ctx: *const B2sCtx) -> *const std::os::raw::c_char;
    pub fn b2s_r1cs_upload(ctx: *mut B2sCtx, n_rows: u64, n_inst: u64, n_wit: u64, row_ptr: *const *const u64,
                           col: *const *const u32, coeff: *const *const c_void, out: *mut *mut B2sR1cs) -> i32;
    pub fn b2s_r1cs_free(ctx: *mut B2sCtx, m: *mut B2sR1cs);
    pub fn b2s_pk_upload(ctx: *mut B2sCtx, desc: *const B2sPkDesc, mem: i32, out: *mut *mut B2sPk) -> i32;
    pub fn b2s_pk_free(ctx: *mut B2sCtx, pk: *mut B2sPk);
    pub fn b2s_groth16_prove(ctx: *mut B2sCtx, pk: *const B2sPk, m: *const B2sR1cs, z_inst: *const c_void,
                             z_wit: *const c_void, r: *const c_void, s: *const c_void, out_a: *mut c_void,
                             out_b: *mut c_void, out_c: *mut c_void) -> i32;
    // multi-GPU group (one rank per GPU, NCCL communicator inside the library; INTEGRATION.md section 7)
    pub fn b2s_group_unique_id(out: *mut u8) -> i32; // 128 bytes
    pub fn b2s_group_create(ctx: *mut B2sCtx, id: *const u8, rank: i32, world: i32, out: *mut *mut B2sGroup) -> i32;
    pub fn b2s_group_destroy(group: *mut B2sGroup);
    pub fn b2s_groth16_prove_group(group: *mut B2sGroup, pk_shard: *const B2sPk, m: *const B2sR1cs, z_inst: *const c_void,
                                   z_wit: *const c_void, r: *const c_void, s: *const c_void, out_a: *mut c_void,
                                   out_b: *mut c_void, out_c: *mut c_void) -> i32;
    pub fn b2s_groth16_prove_batch(ctx: *mut B2sCtx, pk: *const B2sPk, m: *const B2sR1cs, n_proofs: u64, z: *const c_void,
                                   r: *const c_void, s: *const c_void, mem: i32, out_a: *mut c_void, out_b: *mut c_void,
                                   out_c: *mut c_void) -> i32;
    // CanonicalSerialize of the key types (snark/src/lib.rs:25-31)
    pub fn b2s_vk_serialized_size(ctx: *const B2sCtx, n_gamma_abc: u64, compressed: i32) -> u64;
    pub fn b2s_vk_serialize(ctx: *mut B2sCtx, alpha_g1: *const c_void, beta_g2: *const c_void, gamma_g2: *const c_void,
                            delta_g2: *const c_void, gamma_abc_g1: *const c_void, n_gamma_abc: u64, compressed: i32,
                            out: *mut u8, cap: u64) -> i32;
    pub fn b2s_pk_serialized_size(ctx: *const B2sCtx, pk: *const B2sPk, vk_len: u64, compressed: i32) -> u64;
    pub fn b2s_pk_serialize(ctx: *mut B2sCtx, pk: *const B2sPk, vk_bytes: *const u8, vk_len: u64, compressed: i32,
                            out: *mut u8, cap: u64) -> i32;
    // CanonicalDeserialize of the same types, decoded and validated on the GPU (validate = 1: Validate::Yes)
    pub fn b2s_deserialize_g1(ctx: *mut B2sCtx, inp: *const u8, len: u64, count: u64, compressed: i32, validate: i32,
                              out_affine: *mut c_void) -> i32;
    pub fn b2s_deserialize_g2(ctx: *mut B2sCtx, inp: *const u8, len: u64, count: u64, compressed: i32, validate: i32,
                              out_affine: *mut c_void) -> i32;
    pub fn b2s_proof_deserialize(ctx: *mut B2sCtx, inp: *const u8, len: u64, compressed: i32, validate: i32, out_a_g1: *mut c_void,
                                 out_b_g2: *mut c_void, out_c_g1: *mut c_void) -> i32;
    pub fn b2s_vk_deserialize(ctx: *mut B2sCtx, inp: *const u8, len: u64, compressed: i32, validate: i32, out_alpha_g1: *mut c_void,
                              out_beta_g2: *mut c_void, out_gamma_g2: *mut c_void, out_delta_g2: *mut c_void,
                              out_gamma_abc_g1: *mut c_void, cap_gamma_abc: u64, n_gamma_abc: *mut u64, consumed: *mut u64) -> i32;
    pub fn b2s_pk_deserialize(ctx: *mut B2sCtx, inp: *const u8, len: u64, compressed: i32, validate: i32, out: *mut *mut B2sPk) -> i32;
    // the QAP reduction of a key (B2S_QAP_LIBSNARK = 0, B2S_QAP_CIRCOM = 1): see QAP_LIBSNARK / QAP_CIRCOM below
    pub fn b2s_pk_deserialize_qap(ctx: *mut B2sCtx, inp: *const u8, len: u64, compressed: i32, validate: i32, qap: i32,
                                  out: *mut *mut B2sPk) -> i32;
    pub fn b2s_pk_upload_qap(ctx: *mut B2sCtx, desc: *const B2sPkDesc, mem: i32, qap: i32, out: *mut *mut B2sPk) -> i32;
    // snarkjs files (ark-circom read_zkey, snarkjs zkey_utils.js / wtns_utils.js), read and checked on the GPU
    pub fn b2s_zkey_read_info(ctx: *mut B2sCtx, inp: *const u8, len: u64, out: *mut B2sZkeyInfo) -> i32;
    pub fn b2s_zkey_load(ctx: *mut B2sCtx, inp: *const u8, len: u64, validate: i32, out_pk: *mut *mut B2sPk, out_m: *mut *mut B2sR1cs,
                         out_alpha_g1: *mut c_void, out_beta_g2: *mut c_void, out_gamma_g2: *mut c_void, out_delta_g2: *mut c_void,
                         out_gamma_abc_g1: *mut c_void, cap_gamma_abc: u64) -> i32;
    pub fn b2s_wtns_read(ctx: *mut B2sCtx, inp: *const u8, len: u64, n_vars: u64, mem: i32, out_z: *mut c_void) -> i32;
    // circom .r1cs files (ark-circom R1CSFile + to_matrices + b2s_r1cs_upload), walked on the host and decoded on the GPU
    pub fn b2s_r1cs_file_read_info(ctx: *mut B2sCtx, inp: *const u8, len: u64, out: *mut B2sR1csFileInfo) -> i32;
    pub fn b2s_r1cs_file_load(ctx: *mut B2sCtx, inp: *const u8, len: u64, out: *mut *mut B2sR1cs) -> i32;
    pub fn b2s_groth16_setup_qap(ctx: *mut B2sCtx, m: *const B2sR1cs, trapdoor: *const c_void, qap: i32, out_pk: *mut *mut B2sPk,
                                 out_alpha_g1: *mut c_void, out_beta_g2: *mut c_void, out_gamma_g2: *mut c_void,
                                 out_delta_g2: *mut c_void, out_gamma_abc_g1: *mut c_void) -> i32;
    pub fn b2s_witness_map_qap(ctx: *mut B2sCtx, m: *const B2sR1cs, z: *const c_void, mem: i32, qap: i32, out_h: *mut c_void) -> i32;
    // verification (SNARK::process_vk / verify_with_processed_vk for many proofs; pairings in CUDA)
    pub fn b2s_vk_prepare(ctx: *mut B2sCtx, alpha_g1: *const c_void, beta_g2: *const c_void, gamma_g2: *const c_void,
                          delta_g2: *const c_void, gamma_abc_g1: *const c_void, n_gamma_abc: u64, out: *mut *mut B2sPvk) -> i32;
    pub fn b2s_pvk_free(ctx: *mut B2sCtx, pvk: *mut B2sPvk);
    pub fn b2s_groth16_verify_batch(ctx: *mut B2sCtx, pvk: *const B2sPvk, n_proofs: u64, inputs: *const c_void, n_inputs: u64,
                                    a_g1: *const c_void, b_g2: *const c_void, c_g1: *const c_void, mem: i32, ok: *mut u8) -> i32;
    pub fn b2s_groth16_verify_batch_rlc(ctx: *mut B2sCtx, pvk: *const B2sPvk, n_proofs: u64, inputs: *const c_void, n_inputs: u64,
                                        a_g1: *const c_void, b_g2: *const c_void, c_g1: *const c_void, rho: *const c_void, mem: i32,
                                        ok: *mut u8) -> i32;
    pub fn b2s_groth16_verify_batch_bytes(ctx: *mut B2sCtx, pvk: *const B2sPvk, n_proofs: u64, inputs: *const c_void, n_inputs: u64,
                                          proofs: *const u8, len: u64, compressed: i32, mem: i32, ok: *mut u8, reason: *mut u8) -> i32;
    pub fn b2s_groth16_verify_batch_rlc_bytes(ctx: *mut B2sCtx, pvk: *const B2sPvk, n_proofs: u64, inputs: *const c_void,
                                              n_inputs: u64, proofs: *const u8, len: u64, compressed: i32, rho: *const c_void,
                                              mem: i32, ok: *mut u8, reason: *mut u8) -> i32;
    pub fn b2s_pairing(ctx: *mut B2sCtx, p_g1: *const c_void, q_g2: *const c_void, n: u64, mem: i32, out_gt: *mut c_void) -> i32;
    // universal-setup schemes (UniversalSetupSNARK, snark/src/lib.rs:107-133): the seams a polynomial-commitment /
    // evaluation-domain backend binds (INTEGRATION.md section 8).  mem: 0 host, 1 device; s, c, z: one Montgomery Fr on the host
    pub fn b2s_ntt(ctx: *mut B2sCtx, data: *mut c_void, log_n: u32, inverse: i32, coset: i32, mem: i32) -> i32;
    pub fn b2s_msm_g1(ctx: *mut B2sCtx, bases: *const c_void, scalars: *const c_void, n: u64, scalars_mont: i32, mem: i32,
                      out_affine: *mut c_void) -> i32;
    pub fn b2s_fixed_base_g1(ctx: *mut B2sCtx, scalars: *const c_void, n: u64, scalars_mont: i32, mem: i32, out: *mut c_void) -> i32;
    pub fn b2s_poly_op(ctx: *mut B2sCtx, op: i32, a: *const c_void, b: *const c_void, s: *const c_void, out: *mut c_void,
                       n: u64, mem: i32) -> i32;
    pub fn b2s_poly_geom(ctx: *mut B2sCtx, c: *const c_void, s: *const c_void, n: u64, mem: i32, out: *mut c_void) -> i32;
    pub fn b2s_poly_eval(ctx: *mut B2sCtx, coeffs: *const c_void, n: u64, z: *const c_void, mem: i32, out: *mut c_void) -> i32;
    pub fn b2s_gr1cs_upload(ctx: *mut B2sCtx, n_instance: u64, n_witness: u64, n_predicates: u32, preds: *const B2sPredicateDesc,
                            out: *mut *mut B2sGr1cs) -> i32;
    pub fn b2s_gr1cs_upload_lcmap(ctx: *mut B2sCtx, n_instance: u64, n_witness: u64, n_predicates: u32,
                                  preds: *const B2sPredicateLcmapDesc, n_lcs: u64, lc_offsets: *const u64, lc_vars: *const u64,
                                  lc_coeffs: *const u32, pool: *const c_void, pool_len: u32, out: *mut *mut B2sGr1cs) -> i32;
    /// b2s_gr1cs_upload_lcmap with instance outlining (ConstraintSystem::finalize with an InstanceOutliner)
    pub fn b2s_gr1cs_upload_lcmap_outline(ctx: *mut B2sCtx, n_instance: u64, n_witness: u64, n_predicates: u32,
                                          preds: *const B2sPredicateLcmapDesc, n_lcs: u64, lc_offsets: *const u64, lc_vars: *const u64,
                                          lc_coeffs: *const u32, pool: *const c_void, pool_len: u32, outline: *const B2sOutline,
                                          out: *mut *mut B2sGr1cs) -> i32;
    /// z || (ONE, z[1], ..., z[n_instance - 1]): what outlining appends to witness_assignment in prove mode
    pub fn b2s_gr1cs_outline_assignment(ctx: *mut B2sCtx, g: *const B2sGr1cs, n_assign: u64, z: *const c_void, mem: i32,
                                        out_z: *mut c_void) -> i32;
    pub fn b2s_gr1cs_free(ctx: *mut B2sCtx, g: *mut B2sGr1cs);
    pub fn b2s_gr1cs_check(ctx: *mut B2sCtx, g: *const B2sGr1cs, n_assign: u64, z: *const c_void, mem: i32, first_unsat: *mut u64,
                           n_unsat: *mut u64) -> i32;
    pub fn b2s_r1cs_check(ctx: *mut B2sCtx, m: *const B2sR1cs, n_assign: u64, z: *const c_void, mem: i32, first_unsat: *mut u64,
                          n_unsat: *mut u64) -> i32;
    /// Sr1csAdapter::r1cs_to_sr1cs (relations/src/sr1cs/mod.rs:124-183)
    pub fn b2s_r1cs_to_sr1cs(ctx: *mut B2sCtx, m: *const B2sR1cs, out: *mut *mut B2sGr1cs) -> i32;
    /// with b2s_r1cs_to_sr1cs: Sr1csAdapter::r1cs_to_sr1cs_with_assignment (sr1cs/mod.rs:191-265)
    pub fn b2s_sr1cs_assignment(ctx: *mut B2sCtx, g: *const B2sGr1cs, n_assign: u64, z: *const c_void, mem: i32,
                                out_z: *mut c_void) -> i32;
    pub fn b2s_gr1cs_info(ctx: *mut B2sCtx, g: *const B2sGr1cs, n_vars: *mut u64, n_predicates: *mut u32,
                          preds: *mut B2sGr1csPredInfo, cap: u32) -> i32;
    pub fn b2s_gr1cs_export(ctx: *mut B2sCtx, g: *const B2sGr1cs, pred: u32, arg: u32, row_ptr: *mut u64, cap_row_ptr: u64,
                            col: *mut u32, cap_col: u64, coeff: *mut c_void, cap_coeff: u64) -> i32;
}
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct B2sGr1csPredInfo {
    pub arity: u32,
    pub reserved: u32,
    pub n_rows: u64,
    pub nnz: [u64; B2S_GR1CS_MAX_ARITY],
}
#[repr(C)]
pub struct B2sGroup {
    _p: [u8; 0],
}

#[derive(Debug)]
pub enum B200Error { Synthesis(SynthesisError), Backend(i32) }
impl From<SynthesisError> for B200Error { fn from(e: SynthesisError) -> Self { B200Error::Synthesis(e) } }
impl core::fmt::Display for B200Error {
    fn fmt(&self, f: &mut core::fmt::Formatter<'_>) -> core::fmt::Result { write!(f, "{self:?}") }
}
impl ark_std::error::Error for B200Error {}
impl B200Error {
    /// status codes 1..7 mirror SynthesisError (relations/src/utils/error.rs:5-21)
    pub fn from_status(st: i32) -> Self {
        match st {
            1 => SynthesisError::MissingCS.into(),
            2 => SynthesisError::AssignmentMissing.into(),
            3 => SynthesisError::DivisionByZero.into(),
            4 => SynthesisError::Unsatisfiable.into(),
            5 => SynthesisError::PolynomialDegreeTooLarge.into(),
            6 => SynthesisError::UnexpectedIdentity.into(),
            7 => SynthesisError::MalformedVerifyingKey.into(),
            s => B200Error::Backend(s),
        }
    }
}

/// `Matrix<F>` (relations/src/utils/matrix.rs:4) -> CSR, once per circuit.
pub fn to_csr<F: Copy>(m: &Matrix<F>) -> (Vec<u64>, Vec<u32>, Vec<F>) {
    let mut rp = Vec::with_capacity(m.len() + 1);
    let (mut col, mut co) = (Vec::new(), Vec::new());
    rp.push(0u64);
    for row in m {
        for (c, j) in row { col.push(*j as u32); co.push(*c); }
        rp.push(col.len() as u64);
    }
    (rp, col, co)
}

/// The in-memory bytes of a field element.  ark-ff's `Fp<MontBackend<_, N>>` is `BigInt<N>` (N little-endian u64
/// limbs, Montgomery form) plus a zero-sized marker, and `Fp2` is `{ c0, c1 }` of those -- exactly the C-ABI layout.
fn raw<T>(t: &T) -> &[u8] { unsafe { core::slice::from_raw_parts((t as *const T).cast::<u8>(), core::mem::size_of::<T>()) } }

/// `Affine {{ x, y, infinity }}` -> x || y, all-zero bytes for the point at infinity (include/b200snark.h, "Layouts").
pub fn pack_points<G: AffineRepr>(pts: &[G]) -> Vec<u8> {
    let w = core::mem::size_of::<G::BaseField>();
    let mut out = vec![0u8; 2 * w * pts.len()];
    for (i, p) in pts.iter().enumerate() {
        if let Some((x, y)) = p.xy() {
            out[2 * w * i..2 * w * i + w].copy_from_slice(raw(&x));
            out[2 * w * i + w..2 * w * (i + 1)].copy_from_slice(raw(&y));
        }
    }
    out
}

/// x || y (Montgomery limbs; zeros = infinity) -> `Affine`.  The coordinates come from the prover, so they are on the
/// curve by construction: `new_unchecked`.
pub fn unpack_point<G: AffineRepr>(bytes: &[u8]) -> G where G::BaseField: Copy {
    let w = core::mem::size_of::<G::BaseField>();
    if bytes.iter().all(|b| *b == 0) { return G::zero(); }
    let read = |b: &[u8]| -> G::BaseField { unsafe { core::ptr::read_unaligned(b.as_ptr().cast::<G::BaseField>()) } };
    G::new_unchecked(read(&bytes[..w]), read(&bytes[w..2 * w]))
}

fn check(ctx: *mut B2sCtx, st: i32) -> Result<(), B200Error> {
    let _ = ctx;   // b2s_last_error(ctx) carries the message for logs
    if st == 0 { Ok(()) } else { Err(B200Error::from_status(st)) }
}

pub struct Groth16B200<E: Pairing>(core::marker::PhantomData<E>);

/// ark-groth16's `LibsnarkReduction` (`Groth16<E>`): |h_query| = domain - 1.
pub const QAP_LIBSNARK: i32 = 0;
/// ark-circom's `CircomReduction` (`Groth16<Bn254, CircomReduction>`, keys converted from snarkjs zkeys): |h_query| = domain.
pub const QAP_CIRCOM: i32 = 1;

/// Device handles for one (proving key, circuit shape): matrices and key are witness independent.
pub struct Resident { pub ctx: *mut B2sCtx, pub pk: *mut B2sPk, pub mat: *mut B2sR1cs }

impl<E: Pairing + B200Curve> Groth16B200<E> {
    fn ctx_and_matrices(curve_id: i32, mats: &[Matrix<E::ScalarField>], n_inst: usize, n_wit: usize)
        -> Result<(*mut B2sCtx, *mut B2sR1cs), B200Error> {
        // the id passed in must be E's: a BLS12-377 key on a BLS12-381 ctx would be read as the wrong curve's points
        if curve_id != E::CURVE_ID { return Err(B200Error::Backend(ERR_INVALID_ARG)); }
        let mut ctx: *mut B2sCtx = core::ptr::null_mut();
        check(ctx, unsafe { b2s_ctx_create(curve_id, 0, &mut ctx) })?;
        let csr: Vec<_> = mats.iter().map(to_csr).collect();
        let rp: Vec<*const u64> = csr.iter().map(|m| m.0.as_ptr()).collect();
        let col: Vec<*const u32> = csr.iter().map(|m| m.1.as_ptr()).collect();
        let co: Vec<*const c_void> = csr.iter().map(|m| m.2.as_ptr().cast()).collect();
        let mut mat: *mut B2sR1cs = core::ptr::null_mut();
        check(ctx, unsafe { b2s_r1cs_upload(ctx, mats[0].len() as u64, n_inst as u64, n_wit as u64, rp.as_ptr(), col.as_ptr(), co.as_ptr(), &mut mat) })?;
        Ok((ctx, mat))
    }

    /// Upload the matrices and the key once per (key, circuit shape).  `curve_id` must be `E::CURVE_ID` (0 = BLS12-381,
    /// 1 = BN254, 2 = BLS12-377); another id is `B2S_ERR_INVALID_ARG`.
    pub fn make_resident(curve_id: i32, pk: &ProvingKey<E>, mats: &[Matrix<E::ScalarField>], n_inst: usize, n_wit: usize)
        -> Result<Resident, B200Error> {
        let (ctx, mat) = Self::ctx_and_matrices(curve_id, mats, n_inst, n_wit)?;
        let n = (mats[0].len() + n_inst).next_power_of_two() as u64;          // the QAP domain (LibsnarkReduction)
        let (alpha, beta1, delta1) = (pack_points(&[pk.vk.alpha_g1]), pack_points(&[pk.beta_g1]), pack_points(&[pk.delta_g1]));
        let (beta2, delta2) = (pack_points(&[pk.vk.beta_g2]), pack_points(&[pk.vk.delta_g2]));
        let (a, b1, b2, h, l) = (pack_points(&pk.a_query), pack_points(&pk.b_g1_query), pack_points(&pk.b_g2_query),
                                 pack_points(&pk.h_query), pack_points(&pk.l_query));
        let d = B2sPkDesc {
            n_instance: n_inst as u64, n_witness: n_wit as u64, domain_size: n,
            alpha_g1: alpha.as_ptr().cast(), beta_g1: beta1.as_ptr().cast(), delta_g1: delta1.as_ptr().cast(),
            beta_g2: beta2.as_ptr().cast(), delta_g2: delta2.as_ptr().cast(),
            a_query: a.as_ptr().cast(), a_off: 0, a_len: pk.a_query.len() as u64,
            b_g1_query: b1.as_ptr().cast(), b1_off: 0, b1_len: pk.b_g1_query.len() as u64,
            b_g2_query: b2.as_ptr().cast(), b2_off: 0, b2_len: pk.b_g2_query.len() as u64,
            h_query: h.as_ptr().cast(), h_off: 0, h_len: pk.h_query.len() as u64,
            l_query: l.as_ptr().cast(), l_off: 0, l_len: pk.l_query.len() as u64,
        };
        let mut pkh: *mut B2sPk = core::ptr::null_mut();
        check(ctx, unsafe { b2s_pk_upload(ctx, &d, 0 /* B2S_MEM_HOST */, &mut pkh) })?;
        Ok(Resident { ctx, pk: pkh, mat })
    }

    /// The same handle from the bytes of a serialized `ProvingKey` (what `serialize_compressed` / `serialize_uncompressed`
    /// wrote after setup), without building the key on the CPU: framing is read on the host, every point is decoded and,
    /// with `validate`, checked (curve equation, prime-order subgroup) on the GPU, straight into the resident key.
    pub fn make_resident_from_bytes(curve_id: i32, pk_bytes: &[u8], compressed: bool, validate: bool, mats: &[Matrix<E::ScalarField>],
                                    n_inst: usize, n_wit: usize) -> Result<Resident, B200Error> {
        Self::make_resident_from_bytes_qap(curve_id, pk_bytes, compressed, validate, QAP_LIBSNARK, mats, n_inst, n_wit)
    }

    /// The same for a key of either QAP reduction.  With `QAP_CIRCOM` the bytes are those of a
    /// `ProvingKey<Bn254>` for `Groth16<Bn254, CircomReduction>` (what ark-circom's zkey reader returns, serialized), and
    /// `mats` the circuit's A, B, C (C may have no entries: the circom witness map never reads it).  Every proof under the
    /// resident key then runs the circom witness map and verifies with the key's ordinary `VerifyingKey`.
    pub fn make_resident_from_bytes_qap(curve_id: i32, pk_bytes: &[u8], compressed: bool, validate: bool, qap: i32,
                                        mats: &[Matrix<E::ScalarField>], n_inst: usize, n_wit: usize) -> Result<Resident, B200Error> {
        let (ctx, mat) = Self::ctx_and_matrices(curve_id, mats, n_inst, n_wit)?;
        let mut pkh: *mut B2sPk = core::ptr::null_mut();
        check(ctx, unsafe {
            b2s_pk_deserialize_qap(ctx, pk_bytes.as_ptr(), pk_bytes.len() as u64, compressed as i32, validate as i32, qap, &mut pkh)
        })?;
        Ok(Resident { ctx, pk: pkh, mat })
    }

    /// The resident circom key, its matrices and its `VerifyingKey` straight from the bytes of a snarkjs Groth16 `.zkey`,
    /// without ark-circom: the file is parsed and checked on the GPU (b2s_zkey_load; with `validate`, the curve equation
    /// and the prime-order subgroup of every point).  The matrix handle holds A and B; C is empty, as the circom witness map
    /// never reads it.  z for its proofs comes from the witness generator's `.wtns` via `b2s_wtns_read`.  The format is
    /// restated from snarkjs, not pinned against its bytes.
    pub fn make_resident_from_zkey(curve_id: i32, zkey: &[u8], validate: bool) -> Result<(Resident, VerifyingKey<E>), B200Error>
    where <E::G1Affine as AffineRepr>::BaseField: Copy, <E::G2Affine as AffineRepr>::BaseField: Copy {
        if curve_id != E::CURVE_ID { return Err(B200Error::Backend(ERR_INVALID_ARG)); }
        let mut ctx: *mut B2sCtx = core::ptr::null_mut();
        check(ctx, unsafe { b2s_ctx_create(curve_id, 0, &mut ctx) })?;
        let fail = |ctx: *mut B2sCtx, st: i32| -> B200Error { unsafe { b2s_ctx_destroy(ctx) }; B200Error::from_status(st) };
        let mut info = B2sZkeyInfo::default();
        let st = unsafe { b2s_zkey_read_info(ctx, zkey.as_ptr(), zkey.len() as u64, &mut info) };
        if st != 0 { return Err(fail(ctx, st)); }
        let g1 = 2 * core::mem::size_of::<<E::G1Affine as AffineRepr>::BaseField>();
        let n_abc = info.n_public as usize + 1;
        let (mut alpha, mut beta, mut gamma, mut delta, mut abc) = (vec![0u8; g1], vec![0u8; 2 * g1], vec![0u8; 2 * g1], vec![0u8; 2 * g1],
                                                                    vec![0u8; n_abc * g1]);
        let (mut pk, mut mat): (*mut B2sPk, *mut B2sR1cs) = (core::ptr::null_mut(), core::ptr::null_mut());
        let st = unsafe {
            b2s_zkey_load(ctx, zkey.as_ptr(), zkey.len() as u64, validate as i32, &mut pk, &mut mat, alpha.as_mut_ptr().cast(),
                          beta.as_mut_ptr().cast(), gamma.as_mut_ptr().cast(), delta.as_mut_ptr().cast(), abc.as_mut_ptr().cast(), n_abc as u64)
        };
        if st != 0 { return Err(fail(ctx, st)); }
        let vk = VerifyingKey {
            alpha_g1: unpack_point(&alpha), beta_g2: unpack_point(&beta), gamma_g2: unpack_point(&gamma), delta_g2: unpack_point(&delta),
            gamma_abc_g1: abc.chunks(g1).map(unpack_point::<E::G1Affine>).collect(),
        };
        Ok((Resident { ctx, pk, mat }, vk))
    }

    /// The circuit's A, B and C from the bytes of its circom `.r1cs`, loaded into `res`'s context (b2s_r1cs_file_load: the
    /// count words are walked on the host, every entry is decoded and range-checked on the GPU).  Unlike the zkey's matrix
    /// handle it has C, so b2s_r1cs_check on it checks the circuit's own constraints, and it proves under `res.pk` with the
    /// same proofs.  The caller frees it with `b2s_r1cs_free(res.ctx, m)` before `res` is dropped.  The format is restated
    /// from the iden3 r1cs spec, not pinned against bytes circom wrote.
    pub fn load_r1cs(res: &Resident, r1cs: &[u8]) -> Result<*mut B2sR1cs, B200Error> {
        let mut mat: *mut B2sR1cs = core::ptr::null_mut();
        check(res.ctx, unsafe { b2s_r1cs_file_load(res.ctx, r1cs.as_ptr(), r1cs.len() as u64, &mut mat) })?;
        Ok(mat)
    }

    /// `prove` for many circuits of one shape under one resident key, in one GPU call (b2s_groth16_prove_batch): each
    /// circuit is synthesised on the host, r and s are drawn per proof in ark's order (r, then s, then synthesis), and
    /// the witness maps and MSMs of the whole batch run batched on the GPU.  Proof i is the proof `prove` would give
    /// with the same r and s.  Every circuit must have the matrices `res` was made for.
    pub fn prove_batch<C: ConstraintSynthesizer<E::ScalarField>, R: RngCore + CryptoRng>(res: &Resident, circuits: Vec<C>, rng: &mut R)
        -> Result<Vec<Proof<E>>, B200Error> {
        let n = circuits.len();
        let (mut z, mut r, mut s) = (Vec::new(), Vec::with_capacity(n), Vec::with_capacity(n));
        let mut row = None;
        for circuit in circuits {
            r.push(E::ScalarField::rand(rng));
            s.push(E::ScalarField::rand(rng));
            let cs = ConstraintSystem::new_ref();
            cs.set_optimization_goal(OptimizationGoal::Constraints);
            circuit.generate_constraints(cs.clone())?;
            cs.finalize();
            let (zi, zw) = (cs.instance_assignment()?, cs.witness_assignment()?);
            if *row.get_or_insert(zi.len() + zw.len()) != zi.len() + zw.len() { return Err(SynthesisError::AssignmentMissing.into()); }
            z.extend_from_slice(&zi);
            z.extend_from_slice(&zw);
        }
        let g1 = 2 * core::mem::size_of::<<E::G1Affine as AffineRepr>::BaseField>();
        let (mut a, mut b, mut c) = (vec![0u8; n * g1], vec![0u8; n * 2 * g1], vec![0u8; n * g1]);
        check(res.ctx, unsafe {
            b2s_groth16_prove_batch(res.ctx, res.pk, res.mat, n as u64, z.as_ptr().cast(), r.as_ptr().cast(), s.as_ptr().cast(),
                                    0 /* B2S_MEM_HOST */, a.as_mut_ptr().cast(), b.as_mut_ptr().cast(), c.as_mut_ptr().cast())
        })?;
        Ok((0..n).map(|i| Proof { a: unpack_point::<E::G1Affine>(&a[i * g1..(i + 1) * g1]), b: unpack_point::<E::G2Affine>(&b[i * 2 * g1..(i + 1) * 2 * g1]),
                                  c: unpack_point::<E::G1Affine>(&c[i * g1..(i + 1) * g1]) }).collect())
    }

    /// `verify_with_processed_vk` for many proofs under one key, one verdict per proof (`inputs[i]` belongs to
    /// `proofs[i]`).  The key is prepared on the GPU (e(alpha, beta), the lines of -gamma and -delta, window tables for the
    /// public-input sum) and every proof runs its Miller loop and final exponentiation in CUDA; host memory streams through
    /// bounded device scratch.  A wrong input count is `MalformedVerifyingKey`, as in ark.  The points are used as given,
    /// as in ark: proofs from untrusted bytes are decoded with validation first.
    pub fn verify_batch(vk: &VerifyingKey<E>, inputs: &[Vec<E::ScalarField>], proofs: &[Proof<E>]) -> Result<Vec<bool>, B200Error> {
        if inputs.len() != proofs.len() { return Err(SynthesisError::AssignmentMissing.into()); }
        let (ni, x) = Self::flat_inputs(vk, inputs)?;
        Self::with_prepared(vk, |ctx, pvk| {
            let a = pack_points(&proofs.iter().map(|p| p.a).collect::<Vec<_>>());
            let b = pack_points(&proofs.iter().map(|p| p.b).collect::<Vec<_>>());
            let c = pack_points(&proofs.iter().map(|p| p.c).collect::<Vec<_>>());
            let mut ok = vec![0u8; proofs.len()];
            check(ctx, unsafe { b2s_groth16_verify_batch(ctx, pvk, proofs.len() as u64,
                                                         if ni == 0 { core::ptr::null() } else { x.as_ptr().cast() }, ni as u64,
                                                         a.as_ptr().cast(), b.as_ptr().cast(), c.as_ptr().cast(), 0 /* B2S_MEM_HOST */,
                                                         ok.as_mut_ptr()) })?;
            Ok(ok.into_iter().map(|v| v != 0).collect())
        })
    }

    /// One verdict for the whole batch: `true` when every proof is accepted, by a random linear combination of the
    /// proofs with nonzero 128-bit weights drawn from `rng` (bellman's `batch::Verifier::verify(rng, ..)`).  One Miller
    /// loop over one pair per proof, one MSM for the C terms and one final exponentiation for the batch.  A batch with an
    /// invalid proof passes with probability at most 2^-128 if `rng` is unpredictable to whoever made the proofs and
    /// every point lies in its prime-order subgroup (decode untrusted proofs with validation).  On `false`,
    /// `verify_batch` tells which proofs failed.
    pub fn verify_all<R: RngCore + CryptoRng>(vk: &VerifyingKey<E>, inputs: &[Vec<E::ScalarField>], proofs: &[Proof<E>], rng: &mut R)
        -> Result<bool, B200Error> {
        if inputs.len() != proofs.len() { return Err(SynthesisError::AssignmentMissing.into()); }
        let (ni, x) = Self::flat_inputs(vk, inputs)?;
        let rho = Self::draw_rho(proofs.len(), rng);
        Self::with_prepared(vk, |ctx, pvk| {
            let a = pack_points(&proofs.iter().map(|p| p.a).collect::<Vec<_>>());
            let b = pack_points(&proofs.iter().map(|p| p.b).collect::<Vec<_>>());
            let c = pack_points(&proofs.iter().map(|p| p.c).collect::<Vec<_>>());
            let mut ok = 0u8;
            check(ctx, unsafe { b2s_groth16_verify_batch_rlc(ctx, pvk, proofs.len() as u64,
                                                             if ni == 0 { core::ptr::null() } else { x.as_ptr().cast() }, ni as u64,
                                                             a.as_ptr().cast(), b.as_ptr().cast(), c.as_ptr().cast(), rho.as_ptr().cast(),
                                                             0 /* B2S_MEM_HOST */, &mut ok) })?;
            Ok(ok != 0)
        })
    }

    /// `verify_batch` on serialized proofs as received from untrusted parties: `proofs` is `inputs.len()` ark `Proof`s
    /// back to back (`serialize_compressed` / `serialize_uncompressed` of each, a || b || c).  Every point is decoded and
    /// validated (curve equation, prime-order subgroup) on the GPU, where it stays.  A proof that fails to decode is
    /// rejected on its own: the verdict is `false` and `reasons[i]` is 16 * (1 + e) + r for its first bad element e
    /// (0 a, 1 b, 2 c) and decode reason r (1 flags, 2 coordinate >= p, 3 not on the curve, 4 not in the subgroup);
    /// 0 when the proof decoded.  A wrong byte length is `InvalidData`.
    pub fn verify_batch_bytes(vk: &VerifyingKey<E>, inputs: &[Vec<E::ScalarField>], proofs: &[u8], compressed: bool)
        -> Result<(Vec<bool>, Vec<u8>), B200Error> {
        let (ni, x) = Self::flat_inputs(vk, inputs)?;
        Self::with_prepared(vk, |ctx, pvk| {
            let (mut ok, mut reason) = (vec![0u8; inputs.len()], vec![0u8; inputs.len()]);
            check(ctx, unsafe { b2s_groth16_verify_batch_bytes(ctx, pvk, inputs.len() as u64,
                                                               if ni == 0 { core::ptr::null() } else { x.as_ptr().cast() }, ni as u64,
                                                               proofs.as_ptr(), proofs.len() as u64, compressed as i32,
                                                               0 /* B2S_MEM_HOST */, ok.as_mut_ptr(), reason.as_mut_ptr()) })?;
            Ok((ok.into_iter().map(|v| v != 0).collect(), reason))
        })
    }

    /// `verify_all` on serialized proofs (layout and reasons as for `verify_batch_bytes`): `true` only when every proof
    /// decodes and the random linear combination holds.  Validation is always on, so the 2^-128 bound of `verify_all`
    /// needs no separate decoding step.
    pub fn verify_all_bytes<R: RngCore + CryptoRng>(vk: &VerifyingKey<E>, inputs: &[Vec<E::ScalarField>], proofs: &[u8],
                                                   compressed: bool, rng: &mut R) -> Result<(bool, Vec<u8>), B200Error> {
        let (ni, x) = Self::flat_inputs(vk, inputs)?;
        let rho = Self::draw_rho(inputs.len(), rng);
        Self::with_prepared(vk, |ctx, pvk| {
            let (mut ok, mut reason) = (0u8, vec![0u8; inputs.len()]);
            check(ctx, unsafe { b2s_groth16_verify_batch_rlc_bytes(ctx, pvk, inputs.len() as u64,
                                                                   if ni == 0 { core::ptr::null() } else { x.as_ptr().cast() },
                                                                   ni as u64, proofs.as_ptr(), proofs.len() as u64, compressed as i32,
                                                                   rho.as_ptr().cast(), 0 /* B2S_MEM_HOST */, &mut ok,
                                                                   reason.as_mut_ptr()) })?;
            Ok((ok != 0, reason))
        })
    }

    /// n nonzero 128-bit weights from `rng`, 16 little-endian bytes each
    fn draw_rho<R: RngCore + CryptoRng>(n: usize, rng: &mut R) -> Vec<u8> {
        let mut rho = vec![0u8; 16 * n];
        for w in rho.chunks_mut(16) {
            while w.iter().all(|b| *b == 0) { rng.fill_bytes(w); }
        }
        rho
    }

    /// the public inputs row-major, after the input-count check (`MalformedVerifyingKey`, as in ark)
    fn flat_inputs(vk: &VerifyingKey<E>, inputs: &[Vec<E::ScalarField>]) -> Result<(usize, Vec<E::ScalarField>), B200Error> {
        let ni = vk.gamma_abc_g1.len().saturating_sub(1);
        if inputs.iter().any(|x| x.len() != ni) { return Err(SynthesisError::MalformedVerifyingKey.into()); }
        Ok((ni, inputs.iter().flat_map(|v| v.iter().copied()).collect()))
    }

    /// runs `f` with a ctx and the key prepared on it, and frees both whatever `f` returns
    fn with_prepared<T>(vk: &VerifyingKey<E>, f: impl FnOnce(*mut B2sCtx, *mut B2sPvk) -> Result<T, B200Error>) -> Result<T, B200Error> {
        // the curve from E's B200Curve impl: the base field width cannot tell BLS12-381 from BLS12-377 (both 48 bytes)
        let curve_id = E::CURVE_ID;
        let mut ctx: *mut B2sCtx = core::ptr::null_mut();
        check(ctx, unsafe { b2s_ctx_create(curve_id, 0, &mut ctx) })?;
        let run = || -> Result<T, B200Error> {
            let (alpha, beta, gamma, delta) = (pack_points(&[vk.alpha_g1]), pack_points(&[vk.beta_g2]), pack_points(&[vk.gamma_g2]),
                                               pack_points(&[vk.delta_g2]));
            let abc = pack_points(&vk.gamma_abc_g1);
            let mut pvk: *mut B2sPvk = core::ptr::null_mut();
            check(ctx, unsafe { b2s_vk_prepare(ctx, alpha.as_ptr().cast(), beta.as_ptr().cast(), gamma.as_ptr().cast(),
                                               delta.as_ptr().cast(), abc.as_ptr().cast(), vk.gamma_abc_g1.len() as u64, &mut pvk) })?;
            let out = f(ctx, pvk);
            unsafe { b2s_pvk_free(ctx, pvk) };
            out
        };
        let out = run();
        unsafe { b2s_ctx_destroy(ctx) };
        out
    }
}

impl Drop for Resident {
    fn drop(&mut self) { unsafe { b2s_pk_free(self.ctx, self.pk); b2s_r1cs_free(self.ctx, self.mat); b2s_ctx_destroy(self.ctx); } }
}

/// Which curve id the backend should use for `E`: 0 = BLS12-381, 1 = BN254, 2 = BLS12-377.
pub trait B200Curve { const CURVE_ID: i32; }

impl<E: Pairing + B200Curve> SNARK<E::ScalarField> for Groth16B200<E> {
    type ProvingKey = ProvingKey<E>;
    type VerifyingKey = VerifyingKey<E>;
    type Proof = Proof<E>;
    type ProcessedVerifyingKey = PreparedVerifyingKey<E>;
    type Error = B200Error;

    fn circuit_specific_setup<C: ConstraintSynthesizer<E::ScalarField>, R: RngCore + CryptoRng>(
        circuit: C, rng: &mut R,
    ) -> Result<(Self::ProvingKey, Self::VerifyingKey), Self::Error> {
        Groth16::<E>::circuit_specific_setup(circuit, rng).map_err(B200Error::from)
    }

    fn prove<C: ConstraintSynthesizer<E::ScalarField>, R: RngCore + CryptoRng>(
        pk: &Self::ProvingKey, circuit: C, rng: &mut R,
    ) -> Result<Self::Proof, Self::Error> {
        let r = E::ScalarField::rand(rng);
        let s = E::ScalarField::rand(rng);
        let cs = ConstraintSystem::new_ref();
        cs.set_optimization_goal(OptimizationGoal::Constraints);
        circuit.generate_constraints(cs.clone())?;
        cs.finalize();
        let mats = cs.to_matrices()?.remove(R1CS_PREDICATE_LABEL).ok_or(SynthesisError::MissingCS)?;
        let (zi, zw) = (cs.instance_assignment()?, cs.witness_assignment()?);
        let h = Self::make_resident(E::CURVE_ID, pk, &mats, zi.len(), zw.len())?;   // cache per (key, circuit) in a long-lived prover
        let g1 = 2 * core::mem::size_of::<<E::G1Affine as AffineRepr>::BaseField>();
        let (mut a, mut b, mut c) = (vec![0u8; g1], vec![0u8; 2 * g1], vec![0u8; g1]);
        let st = unsafe {
            b2s_groth16_prove(h.ctx, h.pk, h.mat, zi.as_ptr().cast(), zw.as_ptr().cast(), (&r as *const E::ScalarField).cast(),
                              (&s as *const E::ScalarField).cast(), a.as_mut_ptr().cast(), b.as_mut_ptr().cast(), c.as_mut_ptr().cast())
        };
        if st != 0 { return Err(B200Error::from_status(st)); }
        Ok(Proof { a: unpack_point::<E::G1Affine>(&a), b: unpack_point::<E::G2Affine>(&b), c: unpack_point::<E::G1Affine>(&c) })
    }

    fn process_vk(vk: &Self::VerifyingKey) -> Result<Self::ProcessedVerifyingKey, Self::Error> {
        Ok(ark_groth16::prepare_verifying_key(vk))
    }

    // One proof stays on ark: its verification is a short, latency-bound chain (three Miller loops and one final
    // exponentiation) that a GPU launch would only slow down.  Many proofs under one key: Groth16B200::verify_batch.
    fn verify_with_processed_vk(
        pvk: &Self::ProcessedVerifyingKey, x: &[E::ScalarField], proof: &Self::Proof,
    ) -> Result<bool, Self::Error> {
        Groth16::<E>::verify_with_processed_vk(pvk, x, proof).map_err(B200Error::from)
    }
}

impl<E: Pairing + B200Curve> CircuitSpecificSetupSNARK<E::ScalarField> for Groth16B200<E> {}

// e.g. in the application:  impl B200Curve for ark_bls12_381::Bls12_381 { const CURVE_ID: i32 = 0; }
//                           impl B200Curve for ark_bn254::Bn254 { const CURVE_ID: i32 = 1; }
//                           impl B200Curve for ark_bls12_377::Bls12_377 { const CURVE_ID: i32 = 2; }

/// `ConstraintSystem::is_satisfied` / `which_is_unsatisfied` (relations/src/gr1cs/constraint_system.rs:652-687) on the GPU:
/// the predicates of a finalized constraint system, uploaded once per circuit shape, checked against any assignment of the
/// same shape.  `F` is fixed at upload, so an assignment of another field does not type-check.
pub struct Gr1csB200<F: PrimeField> {
    pub ctx: *mut B2sCtx,
    pub g: *mut B2sGr1cs,
    pub labels: Vec<Label>,
    /// n_instance + n_witness: the length of every assignment
    pub n_vars: usize,
    /// of an outlined upload: n_instance + n_witness before outlining, the length `outline_assignment` takes (0 otherwise)
    pub src_vars: usize,
    _f: core::marker::PhantomData<F>,
}

/// `B2S_ERR_INVALID_ARG`
const ERR_INVALID_ARG: i32 = 16;

impl<F: PrimeField> Gr1csB200<F> {
    /// Uploads `cs.to_matrices()` (one matrix per argument) and `cs.get_all_predicate_types()` (the polynomial of each
    /// predicate), in the BTreeMap's label order.  `curve_id`: 0 = BLS12-381, 1 = BN254, 2 = BLS12-377; it must be
    /// `F`'s curve (checked by the modulus size: 255 / 254 / 253 bits).  A predicate that is not polynomial (`Predicate` is `#[non_exhaustive]`,
    /// predicate/mod.rs:19-25) is `B200Error::Backend(B2S_ERR_INVALID_ARG)`.
    pub fn upload(curve_id: i32, cs: &ConstraintSystem<F>) -> Result<Self, B200Error> {
        Self::check_curve(curve_id)?;
        let mats = cs.to_matrices()?;
        let types = cs.get_all_predicate_types();
        // per predicate: (arity, coefficients, term offsets, factor variables, factor powers) and its CSR matrices
        let mut terms = Vec::new();
        let mut csrs = Vec::new();
        let mut labels = Vec::new();
        for (label, ms) in &mats {
            let p = match types.get(label) {
                Some(Predicate::Polynomial(p)) => p,
                _ => return Err(B200Error::Backend(ERR_INVALID_ARG)),
            };
            terms.push(poly_terms(p));
            csrs.push(ms.iter().map(to_csr).collect::<Vec<_>>());
            labels.push(label.clone());
        }
        let descs: Vec<B2sPredicateDesc> = terms.iter().zip(&csrs).map(|((arity, co, off, var, pow), csr)| {
            let mut d = B2sPredicateDesc {
                arity: *arity, n_terms: co.len() as u32, term_coeffs: co.as_ptr().cast(), term_offsets: off.as_ptr(),
                factor_var: var.as_ptr(), factor_pow: pow.as_ptr(), n_rows: csr.first().map_or(0, |m| m.0.len() as u64 - 1),
                row_ptr: [core::ptr::null(); B2S_GR1CS_MAX_ARITY], col: [core::ptr::null(); B2S_GR1CS_MAX_ARITY],
                coeff: [core::ptr::null(); B2S_GR1CS_MAX_ARITY],
            };
            for (j, m) in csr.iter().take(B2S_GR1CS_MAX_ARITY).enumerate() {
                d.row_ptr[j] = m.0.as_ptr();
                d.col[j] = m.1.as_ptr();
                d.coeff[j] = m.2.as_ptr().cast();
            }
            d
        }).collect();
        Self::create(curve_id, cs, labels, |ctx, g| unsafe {
            b2s_gr1cs_upload(ctx, cs.num_instance_variables() as u64, cs.num_witness_variables() as u64, descs.len() as u32,
                             descs.as_ptr(), g)
        })
    }

    /// The same handle built on the GPU from the constraint system's own storage, without `to_matrices()`: every entry of
    /// `cs.predicate_constraint_systems` (its `get_constraints()` and `get_predicate()`, in label order) over the one
    /// `cs.lc_map` (`#[doc(hidden)] pub`).  `cs` must be finalized (nested LCs are `B200Error::Backend(B2S_ERR_INVALID_ARG)`).
    /// The interner is private upstream (`constraint_system.rs:88`, `gr1cs/mod.rs:9`), so its two facts come from the
    /// caller until it has a one-line accessor: `pool` is its `vec` (pool[0] = ONE, pool[1] = -ONE) and `coeff_ids` the
    /// index each `InternedField` of the LcMap names in it, flat in the order of `cs.lc_map.iter()`.
    pub fn upload_lcmap(curve_id: i32, cs: &ConstraintSystem<F>, pool: &[F], coeff_ids: &[u32]) -> Result<Self, B200Error> {
        Self::lcmap_upload(curve_id, cs, pool, coeff_ids, None)
    }

    /// `upload_lcmap` of the system `cs.finalize()` would give with an `InstanceOutliner { pred_label, func }` set, the
    /// outlining done on the GPU.  Recipe: run `cs.inline_all_lcs()` (public) instead of `finalize()`, set no outliner on
    /// the cs, and pass the outliner's strategy and label here.  The handle has `cs.num_instance_variables()` more witnesses
    /// (the copies of One and of every instance) and as many tie rows in `pred_label`'s predicate; prove-mode assignments
    /// of the outlined system come from `outline_assignment`.  A label the cs has no predicate for is
    /// `B200Error::Backend(B2S_ERR_INVALID_ARG)` (upstream `finalize()` skips outlining then).
    pub fn upload_lcmap_outlined(curve_id: i32, cs: &ConstraintSystem<F>, pool: &[F], coeff_ids: &[u32], outliner: Outliner,
                                 pred_label: &str) -> Result<Self, B200Error> {
        Self::lcmap_upload(curve_id, cs, pool, coeff_ids, Some((outliner, pred_label)))
    }

    /// z = instance || witness of the system before outlining -> the outlined system's z (z || copies), on the GPU
    pub fn outline_assignment(&self, z: &[F]) -> Result<Vec<F>, B200Error> {
        if self.src_vars == 0 { return Err(B200Error::Backend(ERR_INVALID_ARG)); }
        if z.len() != self.src_vars { return Err(B200Error::Synthesis(SynthesisError::AssignmentMissing)); }
        let mut out = vec![F::zero(); self.n_vars];
        check(self.ctx, unsafe {
            b2s_gr1cs_outline_assignment(self.ctx, self.g, 1, z.as_ptr().cast(), 0 /* B2S_MEM_HOST */, out.as_mut_ptr().cast())
        })?;
        Ok(out)
    }

    fn lcmap_upload(curve_id: i32, cs: &ConstraintSystem<F>, pool: &[F], coeff_ids: &[u32], outline: Option<(Outliner, &str)>)
        -> Result<Self, B200Error> {
        Self::check_curve(curve_id)?;
        let raw = |v: &Variable| -> u64 {
            ((v.kind() as u64) << 61) | v.index().unwrap_or(0) as u64
        };
        // the LcMap's variables, flat: LC i's terms at offsets[i]..offsets[i + 1]
        let (mut offsets, mut vars) = (vec![0u64], Vec::new());
        for lc in cs.lc_map.iter() {
            vars.extend(lc.map(|(_, v)| raw(v)));
            offsets.push(vars.len() as u64);
        }
        if coeff_ids.len() != vars.len() { return Err(B200Error::Backend(ERR_INVALID_ARG)); }
        let mut terms = Vec::new();
        let mut args: Vec<Vec<Vec<u64>>> = Vec::new();
        let mut labels = Vec::new();
        for (label, pcs) in &cs.predicate_constraint_systems {
            let p = match pcs.get_predicate() {
                Predicate::Polynomial(p) => p,
                _ => return Err(B200Error::Backend(ERR_INVALID_ARG)),
            };
            terms.push(poly_terms(p));
            args.push(pcs.get_constraints().iter().map(|a| a.iter().map(raw).collect()).collect());
            labels.push(label.clone());
        }
        let descs: Vec<B2sPredicateLcmapDesc> = terms.iter().zip(&args).zip(&cs.predicate_constraint_systems)
            .map(|(((arity, co, off, var, pow), a), (_, pcs))| {
                let mut d = B2sPredicateLcmapDesc {
                    arity: *arity, n_terms: co.len() as u32, term_coeffs: co.as_ptr().cast(), term_offsets: off.as_ptr(),
                    factor_var: var.as_ptr(), factor_pow: pow.as_ptr(), n_rows: pcs.num_constraints() as u64,
                    args: [core::ptr::null(); B2S_GR1CS_MAX_ARITY],
                };
                for (j, col) in a.iter().take(B2S_GR1CS_MAX_ARITY).enumerate() { d.args[j] = col.as_ptr(); }
                d
            }).collect();
        let ol = match outline {
            None => None,
            Some((o, label)) => {
                let pred = labels.iter().position(|l| l.as_str() == label).ok_or(B200Error::Backend(ERR_INVALID_ARG))?;
                Some(B2sOutline { strategy: o as i32, pred: pred as u32 })
            }
        };
        let mut h = Self::create(curve_id, cs, labels, |ctx, g| unsafe {
            let (n_inst, n_wit, n_pred) = (cs.num_instance_variables() as u64, cs.num_witness_variables() as u64, descs.len() as u32);
            let (n_lcs, pool_len) = ((offsets.len() - 1) as u64, pool.len() as u32);
            match &ol {
                None => b2s_gr1cs_upload_lcmap(ctx, n_inst, n_wit, n_pred, descs.as_ptr(), n_lcs, offsets.as_ptr(), vars.as_ptr(),
                                               coeff_ids.as_ptr(), pool.as_ptr().cast(), pool_len, g),
                Some(o) => b2s_gr1cs_upload_lcmap_outline(ctx, n_inst, n_wit, n_pred, descs.as_ptr(), n_lcs, offsets.as_ptr(),
                                                          vars.as_ptr(), coeff_ids.as_ptr(), pool.as_ptr().cast(), pool_len, o, g),
            }
        })?;
        if ol.is_some() {
            h.src_vars = h.n_vars;
            h.n_vars += cs.num_instance_variables();
        }
        Ok(h)
    }

    fn check_curve(curve_id: i32) -> Result<(), B200Error> {
        let bits = match curve_id { 0 => 255, 1 => 254, 2 => 253, _ => return Err(B200Error::Backend(ERR_INVALID_ARG)) };
        if F::MODULUS_BIT_SIZE != bits || core::mem::size_of::<F>() != 32 { return Err(B200Error::Backend(ERR_INVALID_ARG)); }
        Ok(())
    }

    /// a ctx on `curve_id` and the handle `upload` makes on it; the ctx is destroyed again if the upload fails
    fn create(curve_id: i32, cs: &ConstraintSystem<F>, labels: Vec<Label>, upload: impl FnOnce(*mut B2sCtx, *mut *mut B2sGr1cs) -> i32)
        -> Result<Self, B200Error> {
        let n_vars = cs.num_instance_variables() + cs.num_witness_variables();
        let mut ctx: *mut B2sCtx = core::ptr::null_mut();
        check(ctx, unsafe { b2s_ctx_create(curve_id, 0, &mut ctx) })?;
        let mut g: *mut B2sGr1cs = core::ptr::null_mut();
        let st = upload(ctx, &mut g);
        if st != 0 { unsafe { b2s_ctx_destroy(ctx) }; }
        check(ctx, st)?;
        Ok(Gr1csB200 { ctx, g, labels, n_vars, src_vars: 0, _f: core::marker::PhantomData })
    }

    /// The reference's answer without a `ConstraintLayer`: `Some("{label} - {index}")` for the first unsatisfied constraint
    /// in label order, `None` when z = instance || witness (z[0] = 1) satisfies every predicate.  A z whose length is not
    /// n_vars is `SynthesisError::AssignmentMissing`; nothing is read from it.
    pub fn which_is_unsatisfied(&self, z: &[F]) -> Result<Option<String>, B200Error> {
        if z.len() != self.n_vars { return Err(SynthesisError::AssignmentMissing.into()); }
        let mut first = vec![u64::MAX; self.labels.len()];
        check(self.ctx, unsafe {
            b2s_gr1cs_check(self.ctx, self.g, 1, z.as_ptr().cast(), 0, first.as_mut_ptr(), core::ptr::null_mut())
        })?;
        Ok(self.labels.iter().zip(&first).find(|(_, f)| **f != u64::MAX).map(|(l, f)| format!("{l} - {f}")))
    }

    pub fn is_satisfied(&self, z: &[F]) -> Result<bool, B200Error> { Ok(self.which_is_unsatisfied(z)?.is_none()) }

    /// instance_assignment || witness_assignment of `cs` (constraint_system.rs:193-206), the z the checks take
    pub fn assignment(cs: &ConstraintSystem<F>) -> Result<Vec<F>, B200Error> {
        Ok([cs.instance_assignment()?, cs.witness_assignment()?].concat())
    }
}

/// A polynomial predicate as the C ABI takes it: (arity, coefficients, term offsets, factor variables, factor powers)
fn poly_terms<F: PrimeField>(p: &PolynomialPredicate<F>) -> (u32, Vec<F>, Vec<u32>, Vec<u32>, Vec<u32>) {
    let (mut co, mut off, mut var, mut pow) = (Vec::new(), vec![0u32], Vec::new(), Vec::new());
    for (c, term) in &p.polynomial.terms {
        co.push(*c);
        for (v, e) in term.iter() { var.push(*v as u32); pow.push(*e as u32); }
        off.push(var.len() as u32);
    }
    (p.polynomial.num_vars as u32, co, off, var, pow)
}

impl<F: PrimeField> Drop for Gr1csB200<F> {
    fn drop(&mut self) { unsafe { b2s_gr1cs_free(self.ctx, self.g); b2s_ctx_destroy(self.ctx); } }
}

impl<F: PrimeField> Gr1csB200<F> {
    /// `to_matrices()` of one argument of one predicate (upload order), read back from the device: (row_ptr, col, coeff)
    pub fn export(&self, pred: u32, arg: u32) -> Result<(Vec<u64>, Vec<u32>, Vec<F>), B200Error> {
        let (mut nv, mut np) = ([0u64; 2], 0u32);
        check(self.ctx, unsafe { b2s_gr1cs_info(self.ctx, self.g, nv.as_mut_ptr(), &mut np, core::ptr::null_mut(), 0) })?;
        let mut info = vec![B2sGr1csPredInfo::default(); np as usize];
        check(self.ctx, unsafe { b2s_gr1cs_info(self.ctx, self.g, nv.as_mut_ptr(), &mut np, info.as_mut_ptr(), np) })?;
        let p = info.get(pred as usize).ok_or(B200Error::Backend(ERR_INVALID_ARG))?;
        if arg >= p.arity { return Err(B200Error::Backend(ERR_INVALID_ARG)); }
        let nnz = p.nnz[arg as usize] as usize;
        let (mut rp, mut col, mut co) = (vec![0u64; p.n_rows as usize + 1], vec![0u32; nnz], vec![F::zero(); nnz]);
        check(self.ctx, unsafe {
            b2s_gr1cs_export(self.ctx, self.g, pred, arg, rp.as_mut_ptr(), (rp.len() * 8) as u64, col.as_mut_ptr(), (nnz * 4) as u64,
                             co.as_mut_ptr().cast(), (nnz * core::mem::size_of::<F>()) as u64)
        })?;
        Ok((rp, col, co))
    }
}

/// `Sr1csAdapter` (relations/src/sr1cs/mod.rs:18-265) on the GPU: the square R1CS of `cs`'s R1CS predicate, built on the
/// device, and the conversion of assignments.  `gr1cs` is the converted system (predicate "SR1CS", x0^2 - x1), checked and
/// exported like any other.
pub struct Sr1csB200<F: PrimeField> {
    pub gr1cs: Gr1csB200<F>,
    /// n_instance + n_witness of the source: the length of every assignment `assignment` takes
    pub src_vars: usize,
}

impl<F: PrimeField> Sr1csB200<F> {
    /// `r1cs_to_sr1cs(cs)`: uploads the R1CS predicate of `cs.to_matrices()`, converts it and frees the upload
    pub fn r1cs_to_sr1cs(curve_id: i32, cs: &ConstraintSystem<F>) -> Result<Self, B200Error> {
        Gr1csB200::<F>::check_curve(curve_id)?;
        let mats = cs.to_matrices()?;
        let r1cs = mats.get(R1CS_PREDICATE_LABEL).ok_or(B200Error::Backend(ERR_INVALID_ARG))?;
        let csr: Vec<_> = r1cs.iter().map(to_csr).collect();
        let src_vars = cs.num_instance_variables() + cs.num_witness_variables();
        let mut ctx: *mut B2sCtx = core::ptr::null_mut();
        check(ctx, unsafe { b2s_ctx_create(curve_id, 0, &mut ctx) })?;
        let rp: Vec<*const u64> = csr.iter().map(|m| m.0.as_ptr()).collect();
        let col: Vec<*const u32> = csr.iter().map(|m| m.1.as_ptr()).collect();
        let co: Vec<*const c_void> = csr.iter().map(|m| m.2.as_ptr().cast()).collect();
        let mut m: *mut B2sR1cs = core::ptr::null_mut();
        let mut g: *mut B2sGr1cs = core::ptr::null_mut();
        let mut st = unsafe {
            b2s_r1cs_upload(ctx, csr[0].0.len() as u64 - 1, cs.num_instance_variables() as u64, cs.num_witness_variables() as u64,
                            rp.as_ptr(), col.as_ptr(), co.as_ptr(), &mut m)
        };
        if st == 0 {
            st = unsafe { b2s_r1cs_to_sr1cs(ctx, m, &mut g) };
            unsafe { b2s_r1cs_free(ctx, m) };
        }
        let mut nv = [0u64; 2];
        let mut np = 0u32;
        if st == 0 { st = unsafe { b2s_gr1cs_info(ctx, g, nv.as_mut_ptr(), &mut np, core::ptr::null_mut(), 0) }; }
        if let Err(e) = check(ctx, st) {
            unsafe { b2s_gr1cs_free(ctx, g); b2s_ctx_destroy(ctx) };
            return Err(e);
        }
        let gr1cs = Gr1csB200 { ctx, g, labels: vec![SR1CS_PREDICATE_LABEL.to_string()], n_vars: (nv[0] + nv[1]) as usize,
                                src_vars: 0, _f: core::marker::PhantomData };
        Ok(Sr1csB200 { gr1cs, src_vars })
    }

    /// the assignment `r1cs_to_sr1cs_with_assignment` gives the converted system for the source's z = instance || witness:
    /// instance' || witness'.  A z whose length is not `src_vars` is `SynthesisError::AssignmentMissing`.
    pub fn assignment(&self, z: &[F]) -> Result<Vec<F>, B200Error> {
        if z.len() != self.src_vars { return Err(SynthesisError::AssignmentMissing.into()); }
        let mut out = vec![F::zero(); self.gr1cs.n_vars];
        check(self.gr1cs.ctx, unsafe {
            b2s_sr1cs_assignment(self.gr1cs.ctx, self.gr1cs.g, 1, z.as_ptr().cast(), 0, out.as_mut_ptr().cast())
        })?;
        Ok(out)
    }
}
