// Groth16 verification of a whole batch under one key with one verdict: the random-linear-combination check stated in
// pairing.cuh above rlc_miller.  Instead of a three-pair Miller loop and a final exponentiation per proof, every proof
// costs a 128-bit G1 scalar multiplication and a one-pair Miller loop; the C terms go through one MSM and the whole batch
// through one final exponentiation.
//
// Host batches are processed in chunks through bounded scratch, as in verify.cu.  Across chunks four running values stay
// on the device: the Fq12 Miller product, C* (XYZZ), S and t_j = sum_i rho_i x_ij (canonical Fr).  The host side is cut
// into the steps of RlcRun (verify.cuh), which verify_bytes.cu shares.  Per chunk (rlc_chunk):
//   verify_rlc_miller   one thread per RLC_NF proofs: rho_i A_i, then the Miller loop with B_i's lines on the fly; also
//                       widens rho to Fr words for the MSM and records the lowest zero rho
//   verify_rlc_product  the chunk's Fq12 values multiplied together, in place, into the running product
//   msm_*               C*_chunk = sum_i rho_i C_i (canonical scalars)
//   verify_rlc_inputs   S and t_j: per-block partial sums, then one block adds them and C*_chunk to the running values
// and after the last chunk verify_rlc_final (one thread): IC* from S gamma_abc[0] and the public-input window tables applied to
// t_j, C* affine, the two prepared pairs, the final exponentiation, and the comparison with e(alpha, beta)^S.
#include <algorithm>

#include "common.cuh"
#include "pairing.cuh"
#include "verify.cuh"

namespace b2s {

// Proofs per thread of verify_rlc_miller: they share the Fq12 squarings of the Miller loop.  Measured on 2^20 proofs (H100
// 80GB HBM3, 400 W limit): verify_rlc_miller took 1235 / 988 / 952 ms (BLS12-381) and 702 / 598 / 551 ms (BN254) for
// NF = 1 / 2 / 4.
constexpr int RLC_NF = 4;
// Fq12 values one thread of verify_rlc_product multiplies per pass.  The narrow last passes are latency-bound chains, so
// the chain per pass is kept short: with 32 the kernel took 42 ms per 2^20 proofs on BLS12-381.
constexpr uint32_t RLC_PER = 4;
// Rows per block of the first verify_rlc_inputs stage.
constexpr uint32_t RLC_ROWS = 256;

template <class Curve, int NF>
__global__ void verify_rlc_miller_kernel(const typename Curve::G1Affine* a, const typename Curve::G2Affine* b, const uint32_t* rho,
                                         uint32_t m, uint64_t base, typename Curve::Fr* rho_fr, unsigned long long* zero_at,
                                         Fp12<typename Curve::FqP>* f) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if ((uint64_t)t * NF >= m) return;
    typename Curve::G1Affine pa[NF];
    typename Curve::G2Affine pb[NF];
    uint32_t k[4 * NF];
    for (int j = 0; j < NF; j++) {
        const uint32_t i = t * NF + j;
        uint32_t nz = 0;
        for (int w = 0; w < 4; w++) k[4 * j + w] = i < m ? rho[4 * (uint64_t)i + w] : 0;
        if (i < m) {
            pa[j] = a[i];
            pb[j] = b[i];
            typename Curve::Fr s = Curve::Fr::zero();
            for (int w = 0; w < 4; w++) { s.v[w] = k[4 * j + w]; nz |= k[4 * j + w]; }
            rho_fr[i] = s;
            if (!nz) atomicMin(zero_at, (unsigned long long)(base + i));
        } else {   // padding: a pair at infinity contributes 1
            pa[j] = Curve::G1Affine::inf();
            pb[j] = Curve::G2Affine::inf();
        }
    }
    f[t] = rlc_miller<Curve, NF>(pa, pb, k);
}

// f[t] = prod_{i = t mod stride} f[i], t < stride, in place (element t < stride is read only by thread t, before it writes);
// with acc (one thread, stride 1): *acc *= the product of all n
template <class P>
__global__ void verify_rlc_product_kernel(Fp12<P>* f, uint32_t n, uint32_t stride, Fp12<P>* acc) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= stride) return;
    Fp12<P> p = f[t];
    for (uint64_t i = t + (uint64_t)stride; i < n; i += stride) p = fp12_mul(p, f[i]);
    if (acc) *acc = fp12_mul(*acc, p);
    else f[t] = p;
}

// Block b sums rows [b RLC_ROWS, (b + 1) RLC_ROWS): column 0 is sum rho_i, column j + 1 is sum rho_i x_ij.  x is
// Montgomery and rho canonical (< 2^128 < r), so the Montgomery product x rho R^-1 is the canonical x_ij rho_i: every sum
// is canonical, which is what the window tables and the GT exponent read.
template <class Fr>
__global__ void verify_rlc_inputs_kernel(const Fr* x, const uint32_t* rho, uint32_t m, uint32_t ni, Fr* part) {
    const uint32_t r0 = blockIdx.x * RLC_ROWS, r1 = min(m, r0 + RLC_ROWS);
    for (uint32_t j = threadIdx.x; j <= ni; j += blockDim.x) {
        Fr acc = Fr::zero();
        for (uint32_t i = r0; i < r1; i++) {
            Fr r = Fr::zero();
            for (int w = 0; w < 4; w++) r.v[w] = rho[4 * (uint64_t)i + w];
            acc += j ? x[(uint64_t)i * ni + j - 1] * r : r;
        }
        part[(uint64_t)blockIdx.x * (ni + 1) + j] = acc;
    }
}
// One block: the running S / t_j += the partial sums of `blocks` blocks, and the running C* += this chunk's C*
template <class Curve>
__global__ void verify_rlc_fold_kernel(const typename Curve::Fr* part, uint32_t blocks, uint32_t ni, typename Curve::Fr* st,
                                       const typename Curve::G1* c_chunk, typename Curve::G1* c_acc) {
    for (uint32_t j = threadIdx.x; j <= ni; j += blockDim.x) {
        typename Curve::Fr acc = st[j];
        for (uint32_t b = 0; b < blocks; b++) acc += part[(uint64_t)b * (ni + 1) + j];
        st[j] = acc;
    }
    if (threadIdx.x == 0) {
        typename Curve::G1 s = *c_acc;
        s.add(*c_chunk);
        *c_acc = s;
    }
}

template <class Curve>
__global__ void verify_rlc_final_kernel(const Fp12<typename Curve::FqP>* f, const typename Curve::Fr* st, uint32_t ni,
                                        const typename Curve::G1Affine* abc0, const typename Curve::G1Affine* table,
                                        const typename Curve::G1* c_acc, const G2Prepared<Curve>* prep,
                                        const Fp12<typename Curve::FqP>* ab, uint8_t* ok) {
    if (blockIdx.x | threadIdx.x) return;
    const typename Curve::Fr s = st[0];
    typename Curve::G1 ic = scalar_mul_words(Curve::G1::from_affine(*abc0), s.v, 8);
    for (uint32_t j = 0; j < ni; j++) {   // the digits of t_j through the tables verify_ic uses
        const typename Curve::Fr t = st[1 + j];
        const typename Curve::G1Affine* tj = table + (uint64_t)j * IC_WINDOWS * IC_DIGITS;
        for (int w = 0; w < IC_WINDOWS; w++) {
            const uint32_t d = (t.v[w / 4] >> (8 * (w % 4))) & 0xFF;
            if (d) ic.add_affine(tj[w * IC_DIGITS + d - 1]);
        }
    }
    *ok = rlc_verdict<Curve>(*f, ic.to_affine(), c_acc->to_affine(), &prep[0], &prep[1], *ab, s.v) ? 1 : 0;
}

size_t rlc_per_proof(Ctx* c) {
    size_t out = 0;
    dispatch_curve(c, [&](auto curve) {
        using C = decltype(curve);
        out = sizeof(Fp12<typename C::FqP>) / RLC_NF + sizeof(typename C::Fr);   // its share of the Miller values, rho widened
        return (int32_t)B2S_OK;
    });
    return out;
}

int32_t rlc_begin(Ctx* c, const b2s_pvk* pvk, uint64_t ni, uint64_t ch, const char* name, RlcRun& r) {
    r.c = c; r.pvk = pvk; r.name = name; r.ni = ni; r.ch = ch;
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        using C = decltype(curve);
        using F12 = Fp12<typename C::FqP>;
        using Fr = typename C::Fr;
        const size_t fr = sizeof(Fr), f12 = sizeof(F12);
        const uint64_t groups = cdiv(ch, RLC_NF), blocks = cdiv(ch, RLC_ROWS);
        B2S_TRY(r.scratch.alloc(c, groups * f12 + ch * fr + blocks * (ni + 1) * fr));
        char* sp = r.scratch.as<char>();
        r.f = sp;
        r.rho_fr = sp + groups * f12;
        r.part = sp + groups * f12 + ch * fr;
        // running values: the Miller product, C*, this chunk's C*, S and t_j, the lowest zero rho, the verdict
        const size_t xyzz = sizeof(typename C::G1);
        B2S_TRY(r.state.alloc(c, f12 + 2 * xyzz + (ni + 1) * fr + 8 + 8));
        char* q = r.state.as<char>();
        r.prod = q;
        r.c_acc = q + f12;
        r.c_chunk = q + f12 + xyzz;
        r.st = q + f12 + 2 * xyzz;
        r.zero_at = reinterpret_cast<unsigned long long*>(q + f12 + 2 * xyzz + (ni + 1) * fr);
        r.ok_dev = reinterpret_cast<uint8_t*>(r.zero_at + 1);
        const F12 one = F12::one();
        B2S_CUDA(c, cudaMemcpyAsync(r.prod, &one, f12, cudaMemcpyHostToDevice, c->stream));
        B2S_CUDA(c, cudaMemsetAsync(r.c_acc, 0, xyzz + xyzz + (ni + 1) * fr, c->stream));   // identity, zeros
        B2S_CUDA(c, cudaMemsetAsync(r.zero_at, 0xFF, 8, c->stream));
        return (int32_t)B2S_OK;
    });
}

int32_t rlc_chunk(RlcRun& r, const void* xi, const void* ai, const void* bi, const void* ci, const void* ri, uint32_t m, uint64_t base,
                  bool last) {
    Ctx* c = r.c;
    const uint64_t ni = r.ni;
    return dispatch_curve(c, [&](auto curve) -> int32_t {
        using C = decltype(curve);
        using P = typename C::FqP;
        using F12 = Fp12<P>;
        using Fr = typename C::Fr;
        using G1A = typename C::G1Affine;
        auto* f = static_cast<F12*>(r.f);
        auto* rho_fr = static_cast<Fr*>(r.rho_fr);
        auto* part = static_cast<Fr*>(r.part);
        auto* c_chunk = static_cast<typename C::G1*>(r.c_chunk);
        const uint32_t* rw = static_cast<const uint32_t*>(ri);
        const uint32_t g = cdiv(m, RLC_NF);
        B2S_LAUNCH_N(c, "verify_rlc_miller", (verify_rlc_miller_kernel<C, RLC_NF>), cdiv(g, VERIFY_THREADS), VERIFY_THREADS, 0,
                     static_cast<const G1A*>(ai), static_cast<const typename C::G2Affine*>(bi), rw, m, base, rho_fr, r.zero_at, f);
        uint32_t cnt = g;
        while (cnt > RLC_PER) {
            const uint32_t stride = cdiv(cnt, RLC_PER);
            B2S_LAUNCH_N(c, "verify_rlc_product", verify_rlc_product_kernel<P>, cdiv(stride, VERIFY_THREADS), VERIFY_THREADS, 0, f,
                         cnt, stride, (F12*)nullptr);
            cnt = stride;
        }
        B2S_LAUNCH_N(c, "verify_rlc_product", verify_rlc_product_kernel<P>, 1, 1, 0, f, cnt, 1u, static_cast<F12*>(r.prod));
        B2S_TRY(msm_run(c, 1, ci, rho_fr, m, false, c_chunk));
        const uint32_t nb = cdiv(m, RLC_ROWS);
        const unsigned cols = (unsigned)std::min<uint64_t>(VERIFY_THREADS, 32 * cdiv(ni + 1, 32));
        B2S_LAUNCH_N(c, "verify_rlc_inputs", verify_rlc_inputs_kernel<Fr>, nb, cols, 0, static_cast<const Fr*>(xi), rw, m,
                     (uint32_t)ni, part);
        B2S_LAUNCH_N(c, "verify_rlc_inputs", verify_rlc_fold_kernel<C>, 1, cols, 0, (const Fr*)part, nb, (uint32_t)ni,
                     static_cast<Fr*>(r.st), (const typename C::G1*)c_chunk, static_cast<typename C::G1*>(r.c_acc));
        if (last)
            B2S_LAUNCH_N(c, "verify_rlc_final", verify_rlc_final_kernel<C>, 1, 1, 0, static_cast<const F12*>(r.prod),
                         static_cast<const Fr*>(r.st), (uint32_t)ni, r.pvk->abc0.as<G1A>(), r.pvk->table.as<G1A>(),
                         static_cast<const typename C::G1*>(r.c_acc), r.pvk->prep.as<G2Prepared<C>>(), r.pvk->ab.as<F12>(), r.ok_dev);
        return (int32_t)B2S_OK;
    });
}

int32_t rlc_read(RlcRun& r, uint8_t* ok) {
    Ctx* c = r.c;
    unsigned long long zero_host = 0;
    uint8_t ok_host = 0;
    B2S_CUDA(c, cudaMemcpyAsync(&zero_host, r.zero_at, 8, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaMemcpyAsync(&ok_host, r.ok_dev, 1, cudaMemcpyDeviceToHost, c->stream));
    B2S_CUDA(c, cudaStreamSynchronize(c->stream));
    if (zero_host != ~0ull) return fail(c, B2S_ERR_INVALID_ARG, "%s: rho[%llu] is zero", r.name, zero_host);
    *ok = ok_host;
    return B2S_OK;
}

int32_t groth16_verify_batch_rlc(Ctx* c, const b2s_pvk* pvk, uint64_t n, const void* inputs, uint64_t ni, const void* a, const void* b,
                                 const void* cc, const void* rho, int32_t mem, uint8_t* ok) {
    if (pvk->curve != c->curve) return fail(c, B2S_ERR_INVALID_ARG, "verify_batch_rlc: the prepared key belongs to another curve");
    if (ni + 1 != pvk->n_abc)
        return fail(c, B2S_ERR_MALFORMED_VK, "verify_batch_rlc: %llu public inputs, the key expects %llu", (unsigned long long)ni,
                    (unsigned long long)(pvk->n_abc - 1));
    if (!ok) return fail(c, B2S_ERR_INVALID_ARG, "verify_batch_rlc: null buffer");
    *ok = 0;
    if (n == 0) { *ok = 1; return B2S_OK; }
    if (!a || !b || !cc || !rho || (ni && !inputs)) return fail(c, B2S_ERR_INVALID_ARG, "verify_batch_rlc: null buffer");
    const Sizes z = sizes(c);
    RowStager io(c, mem, {col_in(inputs, ni * z.fr), col_in(a, z.g1), col_in(b, z.g2), col_in(cc, z.g1), col_in(rho, RLC_RHO)});
    const uint64_t ch = chunk_size(n, rlc_per_proof(c) + io.row_bytes());
    RlcRun r;
    B2S_TRY(rlc_begin(c, pvk, ni, ch, "verify_batch_rlc", r));
    B2S_TRY(io.alloc(ch));
    for (uint64_t base = 0; base < n; base += ch) {
        const uint32_t m = (uint32_t)std::min<uint64_t>(ch, n - base);
        B2S_TRY(io.load(base, m));
        B2S_TRY(rlc_chunk(r, io.ptr(0), io.ptr(1), io.ptr(2), io.ptr(3), io.ptr(4), m, base, base + m == n));
    }
    return rlc_read(r, ok);
}

}  // namespace b2s
