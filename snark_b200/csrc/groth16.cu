// Groth16 prover composition on the GPU: witness_map -> five MSMs -> r/s epilogue.
//
// GPU counterpart of ark-groth16 `create_proof_with_reduction` / `create_proof_with_assignment`
// (upstream crate, not in /root/reference; SURVEY.md Appendix A.1), behind the trait method
// `SNARK::prove` (/root/reference/snark/src/lib.rs:50-54).
//
//   h      = witness_map(A, B, C, z)                                        (r1cs.cu)
//   h_acc  = MSM(h_query, h[0 .. N-1))          l_acc = MSM(l_query, z_witness)
//   a_acc  = MSM(a_query ++ [delta_1, O], z ++ [r, s])      = sum z_j a_j + r delta_1
//   b1_acc = MSM(b_g1_query ++ [O, delta_1], z ++ [r, s])   = sum z_j b_j + s delta_1
//   b2_acc = MSM(b_g2_query ++ [O, delta_2], z ++ [r, s])   = sum z_j b_j + s delta_2      (G2)
//   A = alpha_1 + a_acc      B1 = beta_1 + b1_acc      B2 = beta_2 + b2_acc
//   C = s A + r B1 - (r s) delta_1 + l_acc + h_acc
// ark adds query[0] and r*delta / s*delta separately (z[0] = 1, fresh r, s); putting them into the MSMs as
// two extra (base, scalar) pairs is the same group element and removes three 255-bit scalar multiplications
// (one of them in G2) from the latency-bound tail.  What remains serial is s*A, r*B1, (rs)*delta_1, run
// side by side in three warps.
//
// Multi-GPU: the five MSMs are cut by base range; each rank holds a shard of the key and returns five XYZZ
// partial sums; the rank that owns the END of a query range also owns its two extra pairs.  The join adds
// the partials (EC addition is not an NCCL reduction, so the exchange is an all-gather of 5 small points)
// and applies the epilogue.
#include "ec_team.cuh"
#include "r1cs.cuh"

namespace b2s {

// Warps 0, 1, 2 run the three remaining scalar multiplications side by side (4-bit windows, four-lane teams of
// ec_team.cuh: a doubling costs 3 multiplication latencies instead of 9); warp 3 normalises A meanwhile.
// One CTA per proof k = blockIdx.x: its sums are sums[j * gridDim.x + k] (j = h, l, a, b1), its r and s rs[k * rs_stride + 0 / 1].
template <class Curve>
__global__ void __launch_bounds__(128)
groth16_epilogue_g1_kernel(const Affine<typename Curve::Fq>* consts /*alpha,beta,delta*/, const XYZZ<typename Curve::Fq>* sums /*h,l,a,b1*/,
                           const typename Curve::Fr* rs, uint64_t rs_stride, Affine<typename Curve::Fq>* out_a, Affine<typename Curve::Fq>* out_c) {
    using Fq = typename Curve::Fq;
    using Fr = typename Curve::Fr;
    using P = XYZZ<Fq>;
    __shared__ P sh[3];
    __shared__ P table[3][16];
    const int role = threadIdx.x >> 5;
    const bool lead = (threadIdx.x & 31) == 0;
    sums += blockIdx.x;
    const uint32_t K = gridDim.x;
    rs += blockIdx.x * rs_stride;
    out_a += blockIdx.x;
    out_c += blockIdx.x;
    if (role == 0) {   // s * A,  A = alpha + a_acc
        P a = sums[2 * K];
        a.add_affine(consts[0]);
        Fr s = rs[1].from_mont();
        P v = team_scalar_mul(a, s.v, Fr::N, table[0]);
        if (lead) sh[0] = v;
    } else if (role == 1) {   // r * B1,  B1 = beta + b1_acc
        P b = sums[3 * K];
        b.add_affine(consts[1]);
        Fr r = rs[0].from_mont();
        P v = team_scalar_mul(b, r.v, Fr::N, table[1]);
        if (lead) sh[1] = v;
    } else if (role == 2) {   // (r s) * delta
        Fr rsp = (rs[0] * rs[1]).from_mont();
        P v = team_scalar_mul(P::from_affine(consts[2]), rsp.v, Fr::N, table[2]);
        if (lead) sh[2] = v;
    } else {   // A itself, normalised (one inversion) while the others multiply
        P a = sums[2 * K];
        a.add_affine(consts[0]);
        if (lead) *out_a = a.to_affine();
    }
    __syncthreads();
    if (role == 0) {
        P c = sh[0];
        team_add(c, sh[1]);
        team_add(c, sh[2].neg());
        team_add(c, sums[K]);
        team_add(c, sums[0]);
        if (lead) *out_c = c.to_affine();
    }
}

// one thread per proof: B = beta_2 + b2_acc[k], k = blockIdx.x
template <class Curve>
__global__ void groth16_epilogue_g2_kernel(const Affine<typename Curve::Fq2>* consts /*beta,delta*/,
                                           const XYZZ<typename Curve::Fq2>* b2_sum, Affine<typename Curve::Fq2>* out_b) {
    if (threadIdx.x != 0) return;
    XYZZ<typename Curve::Fq2> acc = b2_sum[blockIdx.x];
    acc.add_affine(consts[0]);
    out_b[blockIdx.x] = acc.to_affine();
}

// sums[j] = sum over shards of partials[shard * stride + j], j < count
template <class F>
__global__ void sum_shards_kernel(const XYZZ<F>* partials, uint32_t n_shards, uint32_t stride, uint32_t count, XYZZ<F>* sums) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= count) return;
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t sidx = 0; sidx < n_shards; sidx++) acc.add(partials[sidx * stride + j]);
    sums[j] = acc;
}

// What a key handle holds beyond its points, shared by pk_upload and pk_deserialize.  The constants and the query points
// are on the device, each query buffer with room for two more points; this appends the extra (base, scalar) pairs of the
// shard that owns the end of a range and builds the h-query table when it fits.  Synchronises the ctx stream.
int32_t pk_finish(Ctx* c, b2s_pk* pk) {
    const Sizes z = sizes(c);
    const uint64_t n_vars = pk->n_instance + pk->n_witness;
    const char* delta[3] = {nullptr, pk->consts_g1.as<char>() + 2 * z.g1, pk->consts_g2.as<char>() + z.g2};   // by group
    for (int w = 0; w < PK_QUERIES; w++) {
        PkQuery& q = pk->q[w];
        const PkQueryInfo& info = PK_QUERY[w];
        const size_t pt = z.aff(info.group);
        q.ext = (info.delta_at >= 0 && q.off + q.len == n_vars) ? 2 : 0;
        char* d = q.pts.as<char>() + q.len * pt;
        B2S_CUDA(c, cudaMemsetAsync(d, 0, 2 * pt, c->stream));   // O = all-zero bytes
        if (q.ext) B2S_CUDA(c, cudaMemcpyAsync(d + info.delta_at * pt, delta[info.group], pt, cudaMemcpyDeviceToDevice, c->stream));
    }
    const PkQuery& h = pk->q[Q_H];
    // Fixed-base window table for the h query: its scalars (the quotient polynomial) are never repeated values, so this is
    // the MSM that always pays the full Pippenger price; the other queries run over the witness, where the multiplicity-aware
    // front end usually leaves little.  13 x the query (20.9 GB at 2^24), built when it fits next to the proof's peak working
    // set with a 2 GiB margin: the witness map (a, b, c, h and the NTT factor tables, 7 scalars per domain element), the sort
    // scratch of the largest MSM, and the batched-affine rounds of the h MSM over the table in one piece.  The rounds of the
    // other MSMs need no room here: when they do not fit beside the table they run in slices of the bucket range (msm.cu).
    {
        const char* env = getenv("B2S_PK_PRECOMP");
        const uint64_t min_n = getenv("B2S_PK_PRECOMP_MIN") ? strtoull(getenv("B2S_PK_PRECOMP_MIN"), nullptr, 10) : (1ull << 18);
        uint32_t cc = 0;
        const uint32_t nw = msm_precompute_windows(c, h.len, &cc);
        const uint64_t need = (uint64_t)nw * h.len * z.g1;
        if (!(env && env[0] == '0') && h.len >= min_n && (uint64_t)nw * h.len < (1ull << 31)) {
            const MsmPre h_shape{cc, nw, (uint32_t)h.len};
            uint64_t sort_max = 0, rounds_h = 0;
            for (int w = 0; w < PK_QUERIES; w++) {
                uint64_t sort_b = 0, round_b = 0;
                msm_working_set(c, PK_QUERY[w].group, pk->q[w].len + pk->q[w].ext, w == Q_H ? &h_shape : nullptr, &sort_b, &round_b);
                sort_max = std::max(sort_max, sort_b);
                if (w == Q_H) rounds_h = round_b;
            }
            const uint64_t working = 7 * pk->domain_size * z.fr + sort_max + rounds_h + ((uint64_t)2 << 30);
            size_t free_b = 0, total_b = 0;
            cudaMemGetInfo(&free_b, &total_b);
            if (need + working <= (uint64_t)free_b + pool_idle_bytes(c)) {
                B2S_TRY(pk->h_table.alloc(c, need));
                B2S_TRY(msm_precompute(c, 1, h.pts.p, h.len, pk->h_table.p, &pk->h_pre));
            }
        }
    }
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

int32_t pk_upload(Ctx* c, const b2s_pk_desc* d, int32_t mem, int32_t qap, b2s_pk** out) {
    const Sizes z = sizes(c);
    const uint64_t n_vars = d->n_instance + d->n_witness;
    // [off, off + len) must lie in [0, bound).  h is held to domain_size under either reduction (a full libsnark key's h is
    // domain_size - 1 long, a full circom key's domain_size)
    struct { const void* pts; uint64_t off, len, bound; } src[PK_QUERIES] = {
        {d->a_query, d->a_off, d->a_len, n_vars},
        {d->b_g1_query, d->b1_off, d->b1_len, n_vars},
        {d->b_g2_query, d->b2_off, d->b2_len, n_vars},
        {d->h_query, d->h_off, d->h_len, d->domain_size},
        {d->l_query, d->l_off, d->l_len, d->n_witness}};
    for (const auto& s : src)
        if (s.off + s.len > s.bound) return fail(c, B2S_ERR_MALFORMED_VK, "pk: a query range exceeds the key dimensions");
    if (!d->alpha_g1 || !d->beta_g1 || !d->delta_g1 || !d->beta_g2 || !d->delta_g2)
        return fail(c, B2S_ERR_MALFORMED_VK, "pk: missing group constants");
    if (qap == B2S_QAP_CIRCOM && d->h_off == 0 && d->h_len + 1 == d->domain_size && d->a_len == n_vars && d->b1_len == n_vars &&
        d->b2_len == n_vars && d->l_len == d->n_witness)
        return fail(c, B2S_ERR_MALFORMED_VK, "pk: a full circom key has domain_size = %llu h_query points, not %llu (a libsnark key?)",
                    (unsigned long long)d->domain_size, (unsigned long long)d->h_len);
    b2s_pk* pk = new b2s_pk();
    pk->n_instance = d->n_instance; pk->n_witness = d->n_witness; pk->domain_size = d->domain_size; pk->qap = qap;
    for (int w = 0; w < PK_QUERIES; w++) { pk->q[w].off = src[w].off; pk->q[w].len = src[w].len; }
    const cudaMemcpyKind kind = to_device(mem);
    auto body = [&]() -> int32_t {
        const size_t g1 = z.g1, g2 = z.g2;
        B2S_TRY(pk->consts_g1.alloc(c, 3 * g1));
        B2S_TRY(pk->consts_g2.alloc(c, 2 * g2));
        char* p1 = pk->consts_g1.as<char>();
        char* p2 = pk->consts_g2.as<char>();
        B2S_CUDA(c, cudaMemcpyAsync(p1, d->alpha_g1, g1, kind, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(p1 + g1, d->beta_g1, g1, kind, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(p1 + 2 * g1, d->delta_g1, g1, kind, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(p2, d->beta_g2, g2, kind, c->stream));
        B2S_CUDA(c, cudaMemcpyAsync(p2 + g2, d->delta_g2, g2, kind, c->stream));
        for (int w = 0; w < PK_QUERIES; w++) {   // with room for the two extra points pk_finish appends
            const size_t pt = z.aff(PK_QUERY[w].group);
            B2S_TRY(pk->q[w].pts.alloc(c, (src[w].len + 2) * pt));
            if (src[w].len) B2S_CUDA(c, cudaMemcpyAsync(pk->q[w].pts.p, src[w].pts, src[w].len * pt, kind, c->stream));
        }
        return pk_finish(c, pk);
    };
    const int32_t st = body();
    if (st != B2S_OK) { delete pk; return st; }
    *out = pk;
    return B2S_OK;
}

// the whole h on this GPU, under the key's reduction (a shard's h range is a slice of the coefficients or of the evaluations)
struct ReplicatedH : HSource {
    DevBuf h;
    int32_t get(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, const void* z_dev, const void** h_for_shard) override {
        B2S_TRY(h.alloc(c, (size_t)32 << m->log_domain));
        B2S_TRY(witness_map_run(c, m, z_dev, h.p, pk->qap));
        *h_for_shard = h.as<char>() + pk->q[Q_H].off * 32;
        return B2S_OK;
    }
};

static int32_t pk_matches(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m) {
    const uint64_t N = 1ull << m->log_domain;
    if (pk->n_instance != m->n_instance || pk->n_witness != m->n_witness || pk->domain_size != N)
        return fail(c, B2S_ERR_ASSIGNMENT_MISSING, "prove: key (%llu,%llu,%llu) does not match matrices (%llu,%llu,%llu)",
                    (unsigned long long)pk->n_instance, (unsigned long long)pk->n_witness, (unsigned long long)pk->domain_size,
                    (unsigned long long)m->n_instance, (unsigned long long)m->n_witness, (unsigned long long)N);
    return B2S_OK;
}

template <class Curve>
static int32_t shard_t(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, const void* z_inst, const void* z_wit, const void* z_dev,
                       const void* r_host, const void* s_host, void* g1_out, void* g2_out, HSource* hs) {
    using Fr = typename Curve::Fr;
    using P1 = XYZZ<typename Curve::Fq>;
    using P2 = XYZZ<typename Curve::Fq2>;
    B2S_TRY(pk_matches(c, pk, m));
    const uint64_t n_vars = m->n_instance + m->n_witness;
    // z_ext = z ++ [r, s]
    DevBuf z, tails;
    ReplicatedH replicated;
    if (!hs) hs = &replicated;
    B2S_TRY(z.alloc(c, (n_vars + 2) * sizeof(Fr)));
    B2S_TRY(tails.alloc(c, 4 * 64 * sizeof(P1) + 64 * sizeof(P2)));
    // Horner tails run on c->aux and read `tails` / write the outputs: whatever way this function is left, the aux
    // stream must be done before the buffers above (and the caller's outputs) go back to the pool
    struct AuxGuard {
        Ctx* c;
        ~AuxGuard() {
            if (c->aux_pending) {
                cudaStreamSynchronize(c->aux);
                c->aux_pending = false;
            }
        }
    } aux_guard{c};
    Fr* zd = z.as<Fr>();
    if (z_dev) {
        B2S_CUDA(c, cudaMemcpyAsync(zd, z_dev, n_vars * sizeof(Fr), cudaMemcpyDeviceToDevice, c->stream));
    } else {
        B2S_CUDA(c, cudaMemcpyAsync(zd, z_inst, m->n_instance * sizeof(Fr), cudaMemcpyHostToDevice, c->stream));
        if (m->n_witness)
            B2S_CUDA(c, cudaMemcpyAsync(zd + m->n_instance, z_wit, m->n_witness * sizeof(Fr), cudaMemcpyHostToDevice, c->stream));
    }
    B2S_CUDA(c, cudaMemcpyAsync(zd + n_vars, r_host, sizeof(Fr), cudaMemcpyHostToDevice, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(zd + n_vars + 1, s_host, sizeof(Fr), cudaMemcpyHostToDevice, c->stream));
    P1* g1 = reinterpret_cast<P1*>(g1_out);
    P1* w1 = tails.as<P1>();
    void* w2 = w1 + 4 * 64;
    const void* h_shard = nullptr;
    // the MSMs that only need z (their Horner tails run on the aux stream under the following work); G2 first because its
    // tail is the longest
    // a, b_g1, b_g2 (and l, when its range coincides) run over the same scalars: classify them once (msm.cu)
    struct DedupScope {
        Ctx* c;
        explicit DedupScope(Ctx* ctx) : c(ctx) { msm_dedup_scope_begin(c); }
        ~DedupScope() { msm_dedup_scope_end(c); }
    } dedup_scope(c);
    // the MSM of query w over its points (or `bases`, the h-query table) and the scalars PK_QUERY[w] names
    auto msm = [&](int w, void* out, void* wins, const void* bases = nullptr, const MsmPre* pre = nullptr) {
        const PkQuery& q = pk->q[w];
        const PkScalars from = PK_QUERY[w].scalars;
        const void* scalars = from == FROM_H ? h_shard : zd + (from == FROM_WITNESS ? m->n_instance : 0) + q.off;
        return msm_run(c, PK_QUERY[w].group, bases ? bases : q.pts.p, scalars, q.len + q.ext, true, out, wins, pre);
    };
    B2S_TRY(msm(Q_B_G2, g2_out, w2));
    B2S_TRY(msm(Q_A, g1 + 2, w1 + 2 * 64));
    B2S_TRY(msm(Q_B_G1, g1 + 3, w1 + 3 * 64));
    B2S_TRY(msm(Q_L, g1 + 1, w1 + 1 * 64));
    // the witness map (SpMV, six transforms, quotient -- or its distributed form) runs after those MSMs, not beside them on a
    // side stream: both are fmaheavy-bound (domain 2^24, H100 80GB HBM3 at 400 W: 342 vs 260 ms per proof with z resident)
    B2S_TRY(hs->get(c, pk, m, zd, &h_shard));
    if (pk->h_table.p) B2S_TRY(msm(Q_H, g1 + 0, w1 + 0 * 64, pk->h_table.p, &pk->h_pre));
    else B2S_TRY(msm(Q_H, g1 + 0, w1 + 0 * 64));
    B2S_TRY(msm_join_tails(c));
    return B2S_OK;
}

int32_t groth16_shard(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, const void* z_inst, const void* z_wit, const void* z_dev,
                      const void* r_host, const void* s_host, void* g1_out, void* g2_out, HSource* hs) {
    return dispatch_curve(c, [&](auto curve) {
        return shard_t<decltype(curve)>(c, pk, m, z_inst, z_wit, z_dev, r_host, s_host, g1_out, g2_out, hs);
    });
}

// ---- many proofs under one key -----------------------------------------------------------------------------------------
// Proofs per chunk at most (DESIGN.md section 4): at domain 2^12 proofs/s still grow from 64 to 256 proofs (799 -> 991 on
// BLS12-381), at 2^16 they are flat from 16 on.  Free memory and the u32 entry limits of the MSM lower it at larger domains.
static constexpr uint64_t PROVE_BATCH_CAP = 256;

// The chunk's K assignments sit on the device as rows z_k ++ [r_k, s_k] of n_vars + 2 scalars, so that each MSM of shard_t
// becomes one batched MSM over the same bases (scalar stride n_vars + 2; h at stride N), the witness map runs once for all K,
// and the epilogue runs one CTA per proof.  No multiplicity-aware front end: the batched MSMs see every scalar.
template <class Curve>
static int32_t prove_batch_t(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, uint64_t n_proofs, const void* z, const void* r, const void* s,
                             int32_t mem, void* out_a, void* out_b, void* out_c) {
    using Fr = typename Curve::Fr;
    using Fq = typename Curve::Fq;
    using Fq2 = typename Curve::Fq2;
    using P1 = XYZZ<Fq>;
    using P2 = XYZZ<Fq2>;
    using A1 = Affine<Fq>;
    using A2 = Affine<Fq2>;
    B2S_TRY(pk_matches(c, pk, m));
    if (n_proofs == 0) return B2S_OK;
    const uint64_t N = 1ull << m->log_domain;
    const uint64_t n_vars = m->n_instance + m->n_witness, row = n_vars + 2;
    const MsmPre* h_pre = pk->h_table.p ? &pk->h_pre : nullptr;
    // per proof: its row, the witness map (h, two more vectors, transform scratch), sums and outputs, the largest MSM
    uint64_t max_k = PROVE_BATCH_CAP, msm_bytes = 0;
    for (int w = 0; w < PK_QUERIES; w++) {
        uint64_t mk = 0;
        msm_bytes = std::max(msm_bytes, msm_batch_bytes(c, PK_QUERY[w].group, pk->q[w].len + pk->q[w].ext, w == Q_H ? h_pre : nullptr, &mk));
        max_k = std::min(max_k, mk);
    }
    const uint64_t per_proof = row * sizeof(Fr) + 4 * N * sizeof(Fr) + msm_bytes + 4 * sizeof(P1) + sizeof(P2) + 2 * sizeof(A1) + sizeof(A2);
    size_t free_b = 0, total_b = 0;
    B2S_CUDA(c, cudaMemGetInfo(&free_b, &total_b));
    max_k = std::max<uint64_t>(1, std::min<uint64_t>(max_k, free_b / 2 / per_proof));
    const uint32_t ch = (uint32_t)std::min<uint64_t>(max_k, n_proofs);
    const cudaMemcpyKind kind = to_device(mem);
    DevBuf zb, h, sums1, sums2;
    B2S_TRY(zb.alloc(c, (size_t)ch * row * sizeof(Fr)));
    B2S_TRY(sums1.alloc(c, (size_t)4 * ch * sizeof(P1)));
    B2S_TRY(sums2.alloc(c, (size_t)ch * sizeof(P2)));
    RowStager outs(c, mem, {col_out(out_a, sizeof(A1)), col_out(out_b, sizeof(A2)), col_out(out_c, sizeof(A1))});
    B2S_TRY(outs.alloc(ch));
    Fr* zd = zb.as<Fr>();
    const size_t fr = sizeof(Fr);
    for (uint64_t p0 = 0; p0 < n_proofs; p0 += ch) {
        const uint32_t K = (uint32_t)std::min<uint64_t>(ch, n_proofs - p0);
        B2S_CUDA(c, cudaMemcpy2DAsync(zd, row * fr, static_cast<const char*>(z) + p0 * n_vars * fr, n_vars * fr, n_vars * fr, K, kind, c->stream));
        B2S_CUDA(c, cudaMemcpy2DAsync(zd + n_vars, row * fr, static_cast<const char*>(r) + p0 * fr, fr, fr, K, kind, c->stream));
        B2S_CUDA(c, cudaMemcpy2DAsync(zd + n_vars + 1, row * fr, static_cast<const char*>(s) + p0 * fr, fr, fr, K, kind, c->stream));
        P1* g1 = sums1.as<P1>();   // [h | l | a | b1] x K, the layout the epilogue reads
        auto msm = [&](int w, void* out, const void* scalars, uint64_t stride, const void* bases = nullptr, const MsmPre* pre = nullptr) {
            const PkQuery& q = pk->q[w];
            return msm_run_batch(c, PK_QUERY[w].group, bases ? bases : q.pts.p, scalars, q.len + q.ext, stride, K, true, out, pre);
        };
        auto from_z = [&](int w) { return zd + (PK_QUERY[w].scalars == FROM_WITNESS ? m->n_instance : 0) + pk->q[w].off; };
        B2S_TRY(msm(Q_B_G2, sums2.p, from_z(Q_B_G2), row));
        B2S_TRY(msm(Q_A, g1 + 2 * K, from_z(Q_A), row));
        B2S_TRY(msm(Q_B_G1, g1 + 3 * K, from_z(Q_B_G1), row));
        B2S_TRY(msm(Q_L, g1 + 1 * K, from_z(Q_L), row));
        {
            B2S_TRY(h.alloc(c, (size_t)K * N * fr));
            B2S_TRY(witness_map_run(c, m, zd, h.p, pk->qap, K, row));
            const Fr* hs = h.as<Fr>() + pk->q[Q_H].off;
            if (h_pre) B2S_TRY(msm(Q_H, g1, hs, N, pk->h_table.p, h_pre));
            else B2S_TRY(msm(Q_H, g1, hs, N));
            h.release();
        }
        B2S_TRY(outs.load(p0, K));
        B2S_LAUNCH(c, groth16_epilogue_g1_kernel<Curve>, K, 128, 0, pk->consts_g1.as<A1>(), (const P1*)g1, (const Fr*)(zd + n_vars), row,
                   outs.ptr<A1>(0), outs.ptr<A1>(2));
        B2S_LAUNCH(c, groth16_epilogue_g2_kernel<Curve>, K, 32, 0, pk->consts_g2.as<A2>(), sums2.as<P2>(), outs.ptr<A2>(1));
        B2S_TRY(outs.store());
    }
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

int32_t groth16_prove_batch(Ctx* c, const b2s_pk* pk, const b2s_r1cs* m, uint64_t n_proofs, const void* z, const void* r, const void* s,
                            int32_t mem, void* out_a, void* out_b, void* out_c) {
    return dispatch_curve(c, [&](auto curve) {
        return prove_batch_t<decltype(curve)>(c, pk, m, n_proofs, z, r, s, mem, out_a, out_b, out_c);
    });
}

// g1_partials: shard i's four G1 sums start at element i * g1_stride (XYZZ<Fq> units); g2_partials likewise (XYZZ<Fq2>)
template <class Curve>
static int32_t finish_t(Ctx* c, const b2s_pk* pk, const void* g1_partials, uint32_t g1_stride, const void* g2_partials, uint32_t g2_stride,
                        uint32_t n_shards, const void* r_host, const void* s_host, void* out_a, void* out_b, void* out_c) {
    using Fr = typename Curve::Fr;
    using Fq = typename Curve::Fq;
    using Fq2 = typename Curve::Fq2;
    DevBuf rs, sums1, sums2, outs;
    B2S_TRY(rs.alloc(c, 2 * sizeof(Fr)));
    B2S_CUDA(c, cudaMemcpyAsync(rs.p, r_host, sizeof(Fr), cudaMemcpyHostToDevice, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(rs.as<Fr>() + 1, s_host, sizeof(Fr), cudaMemcpyHostToDevice, c->stream));
    B2S_TRY(sums1.alloc(c, 4 * sizeof(XYZZ<Fq>)));
    B2S_TRY(sums2.alloc(c, sizeof(XYZZ<Fq2>)));
    B2S_LAUNCH(c, sum_shards_kernel<Fq>, 1, 32, 0, reinterpret_cast<const XYZZ<Fq>*>(g1_partials), n_shards, g1_stride, 4u, sums1.as<XYZZ<Fq>>());
    B2S_LAUNCH(c, sum_shards_kernel<Fq2>, 1, 32, 0, reinterpret_cast<const XYZZ<Fq2>*>(g2_partials), n_shards, g2_stride, 1u, sums2.as<XYZZ<Fq2>>());
    const size_t g1 = sizeof(Affine<Fq>), g2 = sizeof(Affine<Fq2>);
    B2S_TRY(outs.alloc(c, 2 * g1 + g2));
    char* o = outs.as<char>();
    B2S_LAUNCH(c, groth16_epilogue_g1_kernel<Curve>, 1, 128, 0, pk->consts_g1.as<Affine<Fq>>(), sums1.as<XYZZ<Fq>>(), rs.as<Fr>(), (uint64_t)2,
               reinterpret_cast<Affine<Fq>*>(o), reinterpret_cast<Affine<Fq>*>(o + g1));
    B2S_LAUNCH(c, groth16_epilogue_g2_kernel<Curve>, 1, 32, 0, pk->consts_g2.as<Affine<Fq2>>(), sums2.as<XYZZ<Fq2>>(),
               reinterpret_cast<Affine<Fq2>*>(o + 2 * g1));
    B2S_CUDA(c, cudaMemcpyAsync(out_a, o, g1, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(out_c, o + g1, g1, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(out_b, o + 2 * g1, g2, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    return B2S_OK;
}

int32_t groth16_finish(Ctx* c, const b2s_pk* pk, const void* g1_partials_dev, const void* g2_partials_dev, uint32_t n_shards,
                       const void* r_host, const void* s_host, void* out_a, void* out_b, void* out_c) {
    return dispatch_curve(c, [&](auto curve) {
        return finish_t<decltype(curve)>(c, pk, g1_partials_dev, 4u, g2_partials_dev, 1u, n_shards, r_host, s_host, out_a, out_b, out_c);
    });
}

// The all-gathered layout of group.cu: rank i's packet = [4 G1 XYZZ | 1 G2 XYZZ] at byte i * (4 |P1| + |P2|); |P2| = 2 |P1|,
// so the G1 sums sit at stride 6 (P1 units) and the G2 sum at element 2 + 3 i (P2 units).
int32_t groth16_finish_strided(Ctx* c, const b2s_pk* pk, const void* packed_dev, uint32_t n_shards, const void* r_host, const void* s_host,
                               void* out_a, void* out_b, void* out_c) {
    return dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        static_assert(sizeof(XYZZ<typename C::Fq2>) == 2 * sizeof(XYZZ<typename C::Fq>), "packet layout");
        const char* base = reinterpret_cast<const char*>(packed_dev);
        return finish_t<C>(c, pk, base, 6u, base + 4 * sizeof(XYZZ<typename C::Fq>), 3u, n_shards, r_host, s_host, out_a, out_b, out_c);
    });
}

}  // namespace b2s
