// Constraint satisfaction on the GPU: ConstraintSystem::is_satisfied / which_is_unsatisfied for every polynomial predicate of a
// GR1CS, for one assignment or a batch.
//
// Replaces, on the GPU:
//   ConstraintSystem::which_is_unsatisfied   /root/reference/relations/src/gr1cs/constraint_system.rs:652-687
//   Predicate::which_is_unsatisfied          /root/reference/relations/src/gr1cs/predicate/mod.rs:185-204
//   PolynomialPredicate::is_satisfied        /root/reference/relations/src/gr1cs/predicate/polynomial_constraint.rs:46-48
// The reference walks the constraints one at a time on the CPU and looks every argument's LC up in the LcMap.  Here the
// arguments come from to_matrices() (one CSR matrix per argument, coefficients interned as for b2s_r1cs_upload) and one thread
// handles one (constraint, assignment): the arity row products go into registers, the polynomial is evaluated from the term
// arrays, and the first failing index / the failure count go out by one atomicMin / atomicAdd per warp.
#define B2S_INLINE_MUL 1   // Fr only in this unit
#include <algorithm>
#include <cstddef>
#include <type_traits>

#include "r1cs.cuh"

namespace b2s {
namespace {

constexpr int MAXA = B2S_GR1CS_MAX_ARITY;
// gridDim.y carries the assignment: at most 65 535 per launch
constexpr uint64_t CHECK_MAX_ASSIGN = 65535;
// device scratch per chunk: as many whole z rows (host-memory assignments) as fit in this, and as many assignments' outputs
// (first and count, 16 B per predicate), at least one assignment
constexpr uint64_t CHECK_SCRATCH_BYTES = 64ull << 20;

// What the kernel reads of one predicate (device pointers; argument j < arity)
struct PredView {
    const uint64_t* row_ptr[MAXA];
    const uint32_t* col[MAXA];
    const uint32_t* cid[MAXA];
    const void* term_coeff;      // Fr[n_terms]
    const uint32_t* term_off;    // [n_terms + 1]
    const uint32_t* factor_var;
    const uint32_t* factor_pow;
    uint64_t n_rows;
    uint32_t arity, n_terms;
};

template <class Fr>
__device__ __forceinline__ Fr ld_fr(const Fr* p) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = __ldg(q), b = __ldg(q + 1);
    Fr r;
    r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w;
    r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w;
    return r;
}

// b^e by square-and-multiply from the top bit; b^0 = 1 for every b (ark-poly SparseTerm::evaluate)
template <class Fr>
__device__ __forceinline__ Fr pow_u32(const Fr& b, uint32_t e) {
    if (e == 0) return Fr::one();
    Fr r = b;
    for (int i = 30 - __clz(e); i >= 0; i--) {
        r = r.sqr();
        if ((e >> i) & 1) r = r * b;
    }
    return r;
}

// One thread per (row of predicate p, assignment blockIdx.y); z row at z + blockIdx.y * z_stride as in spmv_kernel.
// first[blockIdx.y * out_stride] = min failing row (atomicMin), count[...] += failing rows (one add per warp).
template <class Fr>
__global__ void __launch_bounds__(256)
gr1cs_check_kernel(PredView p, const Fr* __restrict__ pool, const Fr* __restrict__ z, uint64_t z_stride, unsigned long long* first,
                   unsigned long long* count, uint32_t out_stride) {
    const uint64_t row = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    z += blockIdx.y * z_stride;
    bool bad = false;
    if (row < p.n_rows) {
        // the arguments: x[j] = <M_j row, z>; the argument index is compile-time everywhere, so x stays in registers
        Fr x[MAXA];
#pragma unroll
        for (int j = 0; j < MAXA; j++) {
            x[j] = Fr::zero();
            if (j < (int)p.arity) {
                const uint64_t beg = p.row_ptr[j][row], end = p.row_ptr[j][row + 1];
                for (uint64_t e = beg; e < end; e++) {
                    const uint32_t cid = p.cid[j][e];
                    Fr v = ld_fr(z + p.col[j][e]);
                    if (cid != 0) v = v * ld_fr(pool + cid);
                    x[j] = x[j] + v;
                }
            }
        }
        // the polynomial: every thread walks the same terms (warp-uniform loads)
        const Fr* tc = reinterpret_cast<const Fr*>(p.term_coeff);
        Fr acc = Fr::zero();
        for (uint32_t t = 0; t < p.n_terms; t++) {
            Fr term = ld_fr(tc + t);
            const uint32_t f1 = __ldg(p.term_off + t + 1);
            for (uint32_t f = __ldg(p.term_off + t); f < f1; f++) {
                const uint32_t var = __ldg(p.factor_var + f);
                Fr b = x[0];
#pragma unroll
                for (int j = 1; j < MAXA; j++)
                    if (var == (uint32_t)j) b = x[j];
                term = term * pow_u32(b, __ldg(p.factor_pow + f));
            }
            acc = acc + term;
        }
        bad = !acc.is_zero();   // ff.cuh keeps elements fully reduced: 0 mod r is the all-zero limb vector
    }
    const unsigned m = __ballot_sync(0xffffffffu, bad);
    if (m && (int)(threadIdx.x & 31) == __ffs(m) - 1) {   // the lowest failing lane holds the warp's lowest failing row
        atomicMin(first + (uint64_t)blockIdx.y * out_stride, (unsigned long long)row);
        atomicAdd(count + (uint64_t)blockIdx.y * out_stride, (unsigned long long)__popc(m));
    }
}

// which_is_unsatisfied of n_assign assignments (rows of n_vars scalars in `mem`) over the predicates `views`
template <class Curve>
int32_t check_t(Ctx* c, const std::vector<PredView>& views, const void* pool, uint64_t n_vars, uint64_t n_assign, const void* z,
                int32_t mem, uint64_t* first, uint64_t* count) {
    using Fr = typename Curve::Fr;
    if (n_assign == 0) return B2S_OK;
    const uint64_t P = views.size(), row_bytes = n_vars * sizeof(Fr);
    if (P == 0) return B2S_OK;
    const size_t out_row = P * sizeof(uint64_t);
    RowStager io(c, mem, {col_in(z, row_bytes), col_out(first, out_row), col_out(count, out_row)});
    // host: the z rows and the outputs of a chunk each within the scratch bound; scratch stands in for a null count
    uint64_t ch = std::min(CHECK_MAX_ASSIGN, n_assign);
    if (io.staged) ch = std::min(ch, std::max<uint64_t>(1, CHECK_SCRATCH_BYTES / row_bytes));
    if (io.staged || !count) ch = std::min(ch, std::max<uint64_t>(1, CHECK_SCRATCH_BYTES / (2 * out_row)));
    B2S_TRY(io.alloc(ch));
    DevBuf ob;
    if (!count) B2S_TRY(ob.alloc(c, ch * out_row));
    for (uint64_t a0 = 0; a0 < n_assign; a0 += ch) {
        const uint64_t K = std::min(ch, n_assign - a0), n_out = K * P;
        B2S_TRY(io.load(a0, (uint32_t)K));
        const Fr* zc = io.ptr<const Fr>(0);
        uint64_t* fo = io.ptr<uint64_t>(1);
        uint64_t* co = count ? io.ptr<uint64_t>(2) : ob.as<uint64_t>();
        B2S_CUDA(c, cudaMemsetAsync(fo, 0xFF, n_out * sizeof(uint64_t), c->stream));
        B2S_CUDA(c, cudaMemsetAsync(co, 0, n_out * sizeof(uint64_t), c->stream));
        for (uint64_t p = 0; p < P; p++) {
            if (views[p].n_rows == 0) continue;
            B2S_LAUNCH(c, gr1cs_check_kernel<Fr>, dim3(cdiv(views[p].n_rows, 256), (unsigned)K), 256, 0, views[p],
                       reinterpret_cast<const Fr*>(pool), zc, n_vars, reinterpret_cast<unsigned long long*>(fo + p),
                       reinterpret_cast<unsigned long long*>(co + p), (uint32_t)P);
        }
        B2S_TRY(io.store());
    }
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

// The checks shared by both uploads: the variable count, and of one descriptor the arity, the row count and the polynomial
int32_t check_vars(Ctx* c, uint64_t n_instance, uint64_t n_witness) {
    const uint64_t n_vars = n_instance + n_witness;
    if (n_instance == 0) return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: n_instance counts the constant One and must be >= 1");
    if (n_vars > (1ull << 32))
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "gr1cs: %llu variables; columns are u32, the limit is 2^32", (unsigned long long)n_vars);
    return B2S_OK;
}

template <class Desc>
int32_t check_poly(Ctx* c, uint32_t p, const Desc& d) {
    if (d.arity == 0 || d.arity > MAXA)
        return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: arity %u outside 1..%d", p, d.arity, MAXA);
    if (d.n_rows >= (1ull << 32))
        return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "gr1cs: predicate %u: %llu constraints; the limit is 2^32 - 1", p,
                    (unsigned long long)d.n_rows);
    if (d.n_terms) {
        if (!d.term_coeffs || !d.term_offsets) return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: null term arrays", p);
        if (d.term_offsets[0] != 0) return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: term_offsets[0] != 0", p);
        for (uint32_t t = 0; t < d.n_terms; t++)
            if (d.term_offsets[t + 1] < d.term_offsets[t])
                return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: term_offsets not monotone at term %u", p, t);
        const uint32_t nf = d.term_offsets[d.n_terms];
        if (nf && (!d.factor_var || !d.factor_pow)) return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: null factor arrays", p);
        for (uint32_t f = 0; f < nf; f++)
            if (d.factor_var[f] >= d.arity)
                return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: factor_var[%u] = %u >= arity %u", p, f, d.factor_var[f], d.arity);
    }
    return B2S_OK;
}

// a new predicate with the shape and the polynomial (term arrays on the device) of a checked descriptor
template <class Desc>
int32_t upload_poly(Ctx* c, const Desc& d, std::unique_ptr<Gr1csPredicate>& out) {
    std::unique_ptr<Gr1csPredicate> pr(new Gr1csPredicate());
    pr->arity = d.arity;
    pr->n_terms = d.n_terms;
    pr->n_rows = d.n_rows;
    if (d.n_terms) {
        const uint64_t nf = d.term_offsets[d.n_terms];
        B2S_TRY(pr->term_coeff.alloc(c, (uint64_t)d.n_terms * 32));
        B2S_TRY(pr->term_off.alloc(c, ((uint64_t)d.n_terms + 1) * 4));
        B2S_TRY(pr->factor_var.alloc(c, nf * 4));
        B2S_TRY(pr->factor_pow.alloc(c, nf * 4));
        B2S_CUDA(c, cudaMemcpyAsync(pr->term_coeff.p, d.term_coeffs, (uint64_t)d.n_terms * 32, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(pr->term_off.p, d.term_offsets, ((uint64_t)d.n_terms + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        if (nf) {
            B2S_CUDA(c, cudaMemcpyAsync(pr->factor_var.p, d.factor_var, nf * 4, cudaMemcpyHostToDevice, c->stream));
            B2S_CUDA(c, cudaMemcpyAsync(pr->factor_pow.p, d.factor_pow, nf * 4, cudaMemcpyHostToDevice, c->stream));
        }
        B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    }
    out = std::move(pr);
    return B2S_OK;
}

template <class Curve>
int32_t gr1cs_upload_t(Ctx* c, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates, const b2s_predicate_desc* preds,
                       b2s_gr1cs** out) {
    using FrP = typename Curve::FrP;
    const uint64_t n_vars = n_instance + n_witness;
    B2S_TRY(check_vars(c, n_instance, n_witness));
    // the descriptors first: nothing is interned or allocated for a malformed one
    for (uint32_t p = 0; p < n_predicates; p++) {
        const b2s_predicate_desc& d = preds[p];
        B2S_TRY(check_poly(c, p, d));
        for (uint32_t j = 0; j < d.arity; j++)
            if (!d.row_ptr[j] || ((!d.col[j] || !d.coeff[j]) && d.row_ptr[j][d.n_rows] != 0))
                return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: null CSR array for argument %u", p, j);
    }
    std::unique_ptr<b2s_gr1cs> g(new b2s_gr1cs());
    g->curve = c->curve;
    g->n_instance = n_instance;
    g->n_witness = n_witness;
    CoeffInterner in(fr_one_key<FrP>());
    for (uint32_t p = 0; p < n_predicates; p++) {
        const b2s_predicate_desc& d = preds[p];
        std::unique_ptr<Gr1csPredicate> pr;
        B2S_TRY(upload_poly(c, d, pr));
        char who[48];
        snprintf(who, sizeof(who), "gr1cs: predicate %u", p);
        for (uint32_t j = 0; j < d.arity; j++)
            B2S_TRY(csr_intern_upload(c, in, who, (int)j, d.n_rows, n_vars, d.row_ptr[j], d.col[j], d.coeff[j], pr->row_ptr[j], pr->col[j],
                                      pr->coeff_id[j], &pr->nnz[j]));
        g->preds.push_back(std::move(pr));
    }
    B2S_TRY(coeff_pool_upload(c, in, "gr1cs", g->pool, &g->pool_size));
    *out = g.release();
    return B2S_OK;
}

PredView view_of(const Gr1csPredicate& pr) {
    PredView v{};
    for (uint32_t j = 0; j < pr.arity; j++) {
        v.row_ptr[j] = pr.row_ptr[j].as<uint64_t>();
        v.col[j] = pr.col[j].as<uint32_t>();
        v.cid[j] = pr.coeff_id[j].as<uint32_t>();
    }
    v.term_coeff = pr.term_coeff.p;
    v.term_off = pr.term_off.as<uint32_t>();
    v.factor_var = pr.factor_var.as<uint32_t>();
    v.factor_pow = pr.factor_pow.as<uint32_t>();
    v.n_rows = pr.n_rows;
    v.arity = pr.arity;
    v.n_terms = pr.n_terms;
    return v;
}

// The R1CS predicate x0 * x1 - x2 as term arrays: terms (ONE, x0^1 x1^1) and (-ONE, x2^1).  Built at compile time and held in
// device memory once per curve, so b2s_r1cs_check allocates and uploads nothing for it.
struct R1csPoly {
    uint32_t coeff[2][8];
    uint32_t off[3];
    uint32_t var[3];
    uint32_t pow[3];
};
template <class FrP>
constexpr R1csPoly r1cs_poly() {
    R1csPoly p{};
    uint64_t borrow = 0;
    for (int i = 0; i < 8; i++) {
        p.coeff[0][i] = FrP::r1(i);
        const uint64_t d = (uint64_t)FrP::mod(i) - FrP::r1(i) - borrow;   // r - ONE: ONE is reduced, so no final borrow
        p.coeff[1][i] = (uint32_t)d;
        borrow = (d >> 63) & 1;
    }
    for (int f = 0; f < 3; f++) {
        p.var[f] = f;
        p.pow[f] = 1;
    }
    p.off[0] = 0, p.off[1] = 2, p.off[2] = 3;
    return p;
}
__device__ R1csPoly r1cs_poly_bls = r1cs_poly<BlsFrP>();
__device__ R1csPoly r1cs_poly_bn = r1cs_poly<BnFrP>();
__device__ R1csPoly r1cs_poly_bls377 = r1cs_poly<Bls377FrP>();

}  // namespace

int32_t gr1cs_upload(Ctx* c, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates, const b2s_predicate_desc* preds,
                     b2s_gr1cs** out) {
    return dispatch_curve(c, [&](auto curve) {
        return gr1cs_upload_t<decltype(curve)>(c, n_instance, n_witness, n_predicates, preds, out);
    });
}

int32_t gr1cs_upload_lcmap(Ctx* c, uint64_t n_instance, uint64_t n_witness, uint32_t n_predicates, const b2s_predicate_lcmap_desc* preds,
                           const LcMapHost& lm, const b2s_outline* ol, b2s_gr1cs** out) {
    B2S_TRY(check_vars(c, n_instance, n_witness));
    // outlining: n_instance copies (witnesses n_witness ..) and n_instance tie rows in predicate ol->pred
    const uint64_t n_tie = ol ? n_instance : 0;
    if (ol) {
        const uint32_t target_arity = ol->pred < n_predicates ? preds[ol->pred].arity : 0;
        B2S_TRY(outline_validate(c, "gr1cs_upload_lcmap_outline", *ol, n_predicates, target_arity, lm));
        B2S_TRY(check_vars(c, n_instance, n_witness + n_tie));
    }
    uint64_t n_slots = 0;   // (argument, row) slots of all predicates, saturated at 2^32 (lcmap_validate rejects that)
    for (uint32_t p = 0; p < n_predicates; p++) {
        const b2s_predicate_lcmap_desc& d = preds[p];
        B2S_TRY(check_poly(c, p, d));
        for (uint32_t j = 0; j < d.arity; j++)
            if (!d.args[j] && d.n_rows) return fail(c, B2S_ERR_INVALID_ARG, "gr1cs: predicate %u: null argument array %u", p, j);
        const uint64_t rows = d.n_rows + (ol && p == ol->pred ? n_tie : 0);
        if (rows >= (1ull << 32))
            return fail(c, B2S_ERR_POLYNOMIAL_DEGREE_TOO_LARGE, "gr1cs: predicate %u: %llu constraints with the tie rows; the limit is 2^32 - 1", p,
                        (unsigned long long)rows);
        n_slots = std::min<uint64_t>(n_slots + d.arity * rows, 1ull << 32);
    }
    B2S_TRY(lcmap_validate(c, lm, n_slots));
    std::unique_ptr<b2s_gr1cs> g(new b2s_gr1cs());
    g->curve = c->curve;
    g->n_instance = n_instance;
    g->n_witness = n_witness + n_tie;
    g->outline_copies = n_tie;
    std::vector<LcMatrix> mats;
    std::vector<std::pair<uint32_t, uint32_t>> arg_of;   // (predicate, argument) of each matrix, for messages
    LcOutline lo{ol ? ol->strategy : 0, n_witness, 0};
    for (uint32_t p = 0; p < n_predicates; p++) {
        const b2s_predicate_lcmap_desc& d = preds[p];
        std::unique_ptr<Gr1csPredicate> pr;
        B2S_TRY(upload_poly(c, d, pr));
        const uint64_t tie = ol && p == ol->pred ? n_tie : 0;
        if (tie) lo.first_mat = mats.size();
        pr->n_rows = d.n_rows + tie;
        for (uint32_t j = 0; j < d.arity; j++) {
            mats.push_back({d.args[j], d.n_rows, &pr->row_ptr[j], &pr->col[j], &pr->coeff_id[j], &pr->nnz[j], tie});
            arg_of.emplace_back(p, j);
        }
        g->preds.push_back(std::move(pr));
    }
    const auto where = [&](size_t m, uint64_t row) {
        char buf[96];
        snprintf(buf, sizeof(buf), "gr1cs: predicate %u, argument %u, constraint %llu: ", arg_of[m].first, arg_of[m].second,
                 (unsigned long long)row);
        return std::string(buf);
    };
    B2S_TRY(lcmap_build(c, lm, n_instance, n_instance + n_witness + n_tie, mats, "the arguments of all predicates", where, g->pool,
                        &g->pool_size, ol ? &lo : nullptr));
    *out = g.release();
    return B2S_OK;
}

int32_t gr1cs_check(Ctx* c, const b2s_gr1cs* g, uint64_t n_assign, const void* z, int32_t mem, uint64_t* first_unsat, uint64_t* n_unsat) {
    if (g->curve != c->curve)
        return fail(c, B2S_ERR_INVALID_ARG, "gr1cs_check: the handle was uploaded on a ctx of curve %d, this ctx is curve %d", g->curve, c->curve);
    std::vector<PredView> views;
    for (const auto& pr : g->preds) views.push_back(view_of(*pr));
    return dispatch_curve(c, [&](auto curve) {
        return check_t<decltype(curve)>(c, views, g->pool.p, g->n_instance + g->n_witness, n_assign, z, mem, first_unsat, n_unsat);
    });
}

int32_t r1cs_check(Ctx* c, const b2s_r1cs* m, uint64_t n_assign, const void* z, int32_t mem, uint64_t* first_unsat, uint64_t* n_unsat) {
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        using FrP = typename C::FrP;
        static_assert(std::is_same<FrP, BlsFrP>::value || std::is_same<FrP, BnFrP>::value || std::is_same<FrP, Bls377FrP>::value,
                      "one R1CS polynomial per curve");
        void* poly = nullptr;
        B2S_CUDA(c, cudaGetSymbolAddress(&poly, std::is_same<FrP, BlsFrP>::value  ? r1cs_poly_bls
                                                : std::is_same<FrP, BnFrP>::value ? r1cs_poly_bn
                                                                                  : r1cs_poly_bls377));
        const char* d = static_cast<const char*>(poly);
        PredView v{};
        for (int j = 0; j < 3; j++) {
            v.row_ptr[j] = m->row_ptr[j].as<uint64_t>();
            v.col[j] = m->col[j].as<uint32_t>();
            v.cid[j] = m->coeff_id[j].as<uint32_t>();
        }
        v.term_coeff = d + offsetof(R1csPoly, coeff);
        v.term_off = reinterpret_cast<const uint32_t*>(d + offsetof(R1csPoly, off));
        v.factor_var = reinterpret_cast<const uint32_t*>(d + offsetof(R1csPoly, var));
        v.factor_pow = reinterpret_cast<const uint32_t*>(d + offsetof(R1csPoly, pow));
        v.n_rows = m->n_rows;
        v.arity = 3;
        v.n_terms = 2;
        return check_t<C>(c, std::vector<PredView>{v}, m->pool.p, m->n_instance + m->n_witness, n_assign, z, mem, first_unsat, n_unsat);
    });
}

}  // namespace b2s
