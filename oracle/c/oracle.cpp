// CPU restatement (C++17, unsigned __int128 Montgomery, std::thread) of the prover hot path.
// TEST INFRASTRUCTURE ONLY: the checker for mid-size parity tests and the `cpu_baseline` /
// `--impl reference` leg of bench.py.  Nothing under snark_b200/ links or calls this file.
//
// PARITY UNPINNED for MSM / NTT / proofs (see oracle/params.py): the reference tree holds none of this
// arithmetic; the algorithms below restate the un-vendored crates as recalled in SURVEY.md App. A:
//   Fp            ark-ff  Fp<MontBackend<_, N>>            (Montgomery, R = 2^(64 N))
//   Jacobian ops  ark-ec  short_weierstrass::Projective    (add-2007-bl / madd-2007-bl / dbl-2009-l, a = 0)
//   msm           ark-ec  VariableBaseMSM::msm_bigint_wnaf (window rule, signed digits, running sums) A.4
//   ntt           ark-poly Radix2EvaluationDomain::{fft,ifft}_in_place, coset                        A.3
//   spmv          relations/src/utils/matrix.rs:26-36 (mat_vec_mul), sr1cs/mod.rs:24-56 (skip coeff == 1)
//   witness_map   ark-groth16 LibsnarkReduction                                                       A.2
//   witness_map_circom  ark-circom CircomReduction (odd-coset evaluations)                      DESIGN.md §3.6
//   prove         ark-groth16 create_proof_with_assignment                                            A.1
// It is validated against the pure-Python oracle (tests/test_oracle_c.py) which in turn is pinned by
// the definitions (naive DFT, double-and-add) and the known-trapdoor Groth16 check.
//
// Data layout = the C ABI of include/b200snark.h (little-endian Montgomery limbs, affine (x, y) with
// (0, 0) = infinity), so the same buffers feed both sides.  The group formulas are deliberately NOT the
// XYZZ ones the GPU uses, and the limbs are 64-bit rather than 32-bit: an independent implementation.
//
// Threading: ark-ec parallelises an MSM over its <= 17 windows with rayon; here the points are also cut
// into one chunk per thread so that all host cores work (a stronger baseline than the reference's own).
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <functional>
#include <cstring>
#include <thread>
#include <vector>

typedef unsigned __int128 u128;
typedef uint64_t u64;

// ------------------------------------------------------------------------------------------------
template <int N>
struct Params {
    u64 p[N];
    u64 ninv;      // -p^-1 mod 2^64
    u64 r1[N];     // R mod p
    u64 r2[N];     // R^2 mod p
};

template <int N>
static inline bool geq(const u64* a, const u64* b) {
    for (int i = N - 1; i >= 0; i--) {
        if (a[i] != b[i]) return a[i] > b[i];
    }
    return true;
}
template <int N>
static inline u64 add_n(u64* r, const u64* a, const u64* b) {
    u128 c = 0;
    for (int i = 0; i < N; i++) { c += (u128)a[i] + b[i]; r[i] = (u64)c; c >>= 64; }
    return (u64)c;
}
template <int N>
static inline u64 sub_n(u64* r, const u64* a, const u64* b) {
    u64 borrow = 0;
    for (int i = 0; i < N; i++) {
        u128 d = (u128)a[i] - b[i] - borrow;
        r[i] = (u64)d;
        borrow = (u64)(d >> 64) & 1;
    }
    return borrow;
}

template <int N, int ID>
struct Fp {
    u64 v[N];
    static Params<N> P;

    static Fp zero() { Fp r; memset(r.v, 0, sizeof(r.v)); return r; }
    static Fp one() { Fp r; memcpy(r.v, P.r1, sizeof(r.v)); return r; }
    bool is_zero() const { u64 t = 0; for (int i = 0; i < N; i++) t |= v[i]; return t == 0; }
    bool operator==(const Fp& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
    bool operator!=(const Fp& o) const { return !(*this == o); }

    Fp operator+(const Fp& o) const {
        Fp r;
        u64 c = add_n<N>(r.v, v, o.v);
        if (c || geq<N>(r.v, P.p)) sub_n<N>(r.v, r.v, P.p);
        return r;
    }
    Fp operator-(const Fp& o) const {
        Fp r;
        if (sub_n<N>(r.v, v, o.v)) add_n<N>(r.v, r.v, P.p);
        return r;
    }
    Fp neg() const { return is_zero() ? *this : (zero() - *this); }
    Fp dbl() const { return *this + *this; }
    // CIOS Montgomery product
    Fp operator*(const Fp& o) const {
        u64 t[N + 2];
        memset(t, 0, sizeof(t));
        for (int i = 0; i < N; i++) {
            u128 c = 0;
            for (int j = 0; j < N; j++) { c += (u128)v[j] * o.v[i] + t[j]; t[j] = (u64)c; c >>= 64; }
            c += t[N]; t[N] = (u64)c; t[N + 1] = (u64)(c >> 64);
            u64 m = t[0] * P.ninv;
            c = (u128)m * P.p[0] + t[0];
            c >>= 64;
            for (int j = 1; j < N; j++) { c += (u128)m * P.p[j] + t[j]; t[j - 1] = (u64)c; c >>= 64; }
            c += t[N]; t[N - 1] = (u64)c;
            t[N] = t[N + 1] + (u64)(c >> 64);
        }
        Fp r;
        memcpy(r.v, t, sizeof(r.v));
        if (t[N] || geq<N>(r.v, P.p)) sub_n<N>(r.v, r.v, P.p);
        return r;
    }
    Fp sqr() const { return *this * *this; }
    Fp from_mont() const { Fp o = zero(); o.v[0] = 1; return *this * o; }
    Fp to_mont() const { Fp o; memcpy(o.v, P.r2, sizeof(o.v)); return *this * o; }
    Fp pow(const u64* e, int words) const {
        Fp acc = one();
        for (int w = words - 1; w >= 0; w--)
            for (int b = 63; b >= 0; b--) { acc = acc.sqr(); if ((e[w] >> b) & 1) acc = acc * *this; }
        return acc;
    }
    Fp pow64(u64 e) const { return pow(&e, 1); }
    Fp inverse() const {
        u64 e[N];
        u64 two[N] = {2};
        sub_n<N>(e, P.p, two);
        return pow(e, N);
    }
    static Fp from_u64(u64 x) { Fp r = zero(); r.v[0] = x; return r.to_mont(); }
};
template <int N, int ID> Params<N> Fp<N, ID>::P;

template <int N>
static void init_params(Params<N>& P, const u64* modulus) {
    memcpy(P.p, modulus, sizeof(P.p));
    u64 inv = 1;  // Newton: inv = p^-1 mod 2^64
    for (int i = 0; i < 6; i++) inv *= 2 - modulus[0] * inv;
    P.ninv = (u64)0 - inv;
    // R mod p by doubling 1 exactly 64 N times; R^2 by doubling R another 64 N times
    u64 x[N];
    memset(x, 0, sizeof(x));
    x[0] = 1;
    for (int pass = 0; pass < 2; pass++) {
        for (int i = 0; i < 64 * N; i++) {
            u64 c = add_n<N>(x, x, x);
            if (c || geq<N>(x, P.p)) sub_n<N>(x, x, P.p);
        }
        memcpy(pass == 0 ? P.r1 : P.r2, x, sizeof(x));
    }
}

// Fp2 = B[u] / (u^2 + K): u^2 = -1 (K = 1) for BLS12-381 and BN254, u^2 = -5 (K = 5) for BLS12-377.  Schoolbook product.
template <class B, int K = 1>
struct Fp2 {
    B c0, c1;
    static B times_k(const B& x) { B r = x; for (int i = 1; i < K; i++) r = r + x; return r; }
    static Fp2 zero() { return {B::zero(), B::zero()}; }
    static Fp2 one() { return {B::one(), B::zero()}; }
    bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
    bool operator==(const Fp2& o) const { return c0 == o.c0 && c1 == o.c1; }
    bool operator!=(const Fp2& o) const { return !(*this == o); }
    Fp2 operator+(const Fp2& o) const { return {c0 + o.c0, c1 + o.c1}; }
    Fp2 operator-(const Fp2& o) const { return {c0 - o.c0, c1 - o.c1}; }
    Fp2 operator*(const Fp2& o) const { return {c0 * o.c0 - times_k(c1 * o.c1), c0 * o.c1 + c1 * o.c0}; }
    Fp2 sqr() const { return *this * *this; }
    Fp2 neg() const { return {c0.neg(), c1.neg()}; }
    Fp2 dbl() const { return {c0.dbl(), c1.dbl()}; }
    Fp2 inverse() const { B n = (c0.sqr() + times_k(c1.sqr())).inverse(); return {c0 * n, (c1 * n).neg()}; }
};

// ------------------------------------------------------------------------------------------------
template <class F> struct Aff { F x, y; bool inf() const { return x.is_zero() && y.is_zero(); } };

template <class F>
struct Jac {
    F x, y, z;
    static Jac identity() { return {F::one(), F::one(), F::zero()}; }
    bool is_identity() const { return z.is_zero(); }
    static Jac from_affine(const Aff<F>& a) { return a.inf() ? identity() : Jac{a.x, a.y, F::one()}; }
    Jac neg() const { return {x, y.neg(), z}; }
    Jac dbl() const {  // dbl-2009-l (a = 0)
        if (is_identity() || y.is_zero()) return identity();
        F A = x.sqr(), B = y.sqr(), C = B.sqr();
        F D = ((x + B).sqr() - A - C).dbl();
        F E = A.dbl() + A, Fq = E.sqr();
        F x3 = Fq - D.dbl();
        F y3 = E * (D - x3) - C.dbl().dbl().dbl();
        F z3 = (y * z).dbl();
        return {x3, y3, z3};
    }
    Jac add(const Jac& o) const {  // add-2007-bl
        if (is_identity()) return o;
        if (o.is_identity()) return *this;
        F z1z1 = z.sqr(), z2z2 = o.z.sqr();
        F u1 = x * z2z2, u2 = o.x * z1z1;
        F s1 = y * o.z * z2z2, s2 = o.y * z * z1z1;
        if (u1 == u2) return s1 == s2 ? dbl() : identity();
        F h = u2 - u1, i = h.dbl().sqr(), j = h * i, rr = (s2 - s1).dbl(), v = u1 * i;
        F x3 = rr.sqr() - j - v.dbl();
        F y3 = rr * (v - x3) - (s1 * j).dbl();
        F z3 = ((z + o.z).sqr() - z1z1 - z2z2) * h;
        return {x3, y3, z3};
    }
    Jac add_affine(const Aff<F>& o) const {  // madd-2007-bl
        if (o.inf()) return *this;
        if (is_identity()) return from_affine(o);
        F z1z1 = z.sqr();
        F u2 = o.x * z1z1, s2 = o.y * z * z1z1;
        if (x == u2) return y == s2 ? dbl() : identity();
        F h = u2 - x, hh = h.sqr(), i = hh.dbl().dbl(), j = h * i, rr = (s2 - y).dbl(), v = x * i;
        F x3 = rr.sqr() - j - v.dbl();
        F y3 = rr * (v - x3) - (y * j).dbl();
        F z3 = (z + h).sqr() - z1z1 - hh;
        return {x3, y3, z3};
    }
    Aff<F> to_affine() const {
        if (is_identity()) return {F::zero(), F::zero()};
        F zi = z.inverse(), zi2 = zi.sqr();
        return {x * zi2, y * zi2 * zi};
    }
    Jac mul(const u64* k, int words) const {
        Jac acc = identity();
        for (int w = words - 1; w >= 0; w--)
            for (int b = 63; b >= 0; b--) { acc = acc.dbl(); if ((k[w] >> b) & 1) acc = acc.add(*this); }
        return acc;
    }
};

// ------------------------------------------------------------------------------------------------
static void run_parallel(int threads, int jobs, const std::function<void(int)>& fn);

static int ark_window_bits(size_t n) {  // ark-ec: 3 if n < 32 else ln_without_floats(n) + 2
    if (n < 32) return 3;
    int lg = 0;
    while (((size_t)1 << lg) < n) lg++;
    return lg * 69 / 100 + 2;
}

// Signed-digit Pippenger over one contiguous chunk (ark-ec msm_bigint_wnaf), scalars canonical 4 x u64.
template <class F>
static Jac<F> msm_chunk(const Aff<F>* bases, const u64* scalars, size_t n, int num_bits) {
    if (n == 0) return Jac<F>::identity();
    const int c = ark_window_bits(n);
    const int nwin = (num_bits + c - 1) / c;
    std::vector<int32_t> digits(n * (size_t)nwin);
    const int64_t radix = (int64_t)1 << c, half = radix >> 1;
    for (size_t i = 0; i < n; i++) {
        const u64* k = scalars + 4 * i;
        int64_t carry = 0;
        for (int w = 0; w < nwin; w++) {
            const int bit = w * c, word = bit >> 6, off = bit & 63;
            u64 v = word < 4 ? k[word] >> off : 0;
            if (off && word + 1 < 4) v |= k[word + 1] << (64 - off);
            int64_t d = (int64_t)(v & (u64)(radix - 1)) + carry;
            carry = 0;
            if (w != nwin - 1 && d >= half) { d -= radix; carry = 1; }
            digits[i * nwin + w] = (int32_t)d;
        }
    }
    Jac<F> total = Jac<F>::identity();
    std::vector<Jac<F>> buckets;
    for (int w = nwin - 1; w >= 0; w--) {
        // the top window keeps its carry, so it may need up to 2^c buckets
        const size_t nb = (w == nwin - 1) ? ((size_t)1 << c) : ((size_t)1 << (c - 1));
        buckets.assign(nb + 1, Jac<F>::identity());
        for (size_t i = 0; i < n; i++) {
            const int32_t d = digits[i * nwin + w];
            if (d > 0) buckets[d] = buckets[d].add_affine(bases[i]);
            else if (d < 0) { Aff<F> nb_ = {bases[i].x, bases[i].y.neg()}; buckets[-d] = buckets[-d].add_affine(nb_); }
        }
        Jac<F> run = Jac<F>::identity(), sum = Jac<F>::identity();
        for (size_t b = nb; b >= 1; b--) { run = run.add(buckets[b]); sum = sum.add(run); }
        for (int i = 0; i < c; i++) total = total.dbl();
        total = total.add(sum);
    }
    return total;
}

template <class F, class Fr>
static Jac<F> msm(const Aff<F>* bases, const Fr* scalars, size_t n, bool mont, int threads, int num_bits) {
    if (n == 0) return Jac<F>::identity();
    std::vector<u64> canon(4 * n);
    const int T = (int)std::max<size_t>(1, std::min<size_t>(threads, (n + 255) / 256));
    run_parallel(T, T, [&](int t) {
        size_t lo = n * t / T, hi = n * (t + 1) / T;
        for (size_t i = lo; i < hi; i++) {
            Fr s = mont ? scalars[i].from_mont() : scalars[i];
            memcpy(&canon[4 * i], s.v, 32);
        }
    });
    std::vector<Jac<F>> part(T);
    run_parallel(T, T, [&](int t) {
        size_t lo = n * t / T, hi = n * (t + 1) / T;
        part[t] = msm_chunk<F>(bases + lo, canon.data() + 4 * lo, hi - lo, num_bits);
    });
    Jac<F> acc = Jac<F>::identity();
    for (auto& p : part) acc = acc.add(p);
    return acc;
}

// ------------------------------------------------------------------------------------------------
template <class Fr>
struct FrConsts { Fr gen, root; int two_adicity; };

template <class Fr>
static void ntt_inplace(Fr* a, int log_n, const Fr& w_n, int threads) {
    const size_t n = (size_t)1 << log_n;
    const int TP = (int)std::max<size_t>(1, std::min<size_t>(threads, n / 4096 + 1));
    // bit reversal (pairs (i, rev i) are disjoint, so ranges of i can run concurrently)
    run_parallel(TP, TP, [&](int t) {
        for (size_t i = n * t / TP; i < n * (t + 1) / TP; i++) {
            size_t j = 0;
            for (int b = 0; b < log_n; b++) j |= ((i >> b) & 1) << (log_n - 1 - b);
            if (i < j) std::swap(a[i], a[j]);
        }
    });
    // twiddle table w^i, i < n/2
    const size_t nt = std::max<size_t>(1, n / 2);
    std::vector<Fr> tw(nt);
    run_parallel(TP, TP, [&](int t) {
        size_t lo = nt * t / TP, hi = nt * (t + 1) / TP;
        if (lo >= hi) return;
        tw[lo] = w_n.pow64(lo);
        for (size_t i = lo + 1; i < hi; i++) tw[i] = tw[i - 1] * w_n;
    });
    for (int s = 1; s <= log_n; s++) {
        const size_t m = (size_t)1 << s, half = m >> 1, stride = n / m;
        const size_t nbf = n / 2;
        const int T = (int)std::max<size_t>(1, std::min<size_t>(threads, nbf / 4096 + 1));
        run_parallel(T, T, [&](int t) {
            size_t lo = nbf * t / T, hi = nbf * (t + 1) / T;
            for (size_t b = lo; b < hi; b++) {
                const size_t grp = b / half, j = b % half, k = grp * m + j;
                Fr tt = a[k + half] * tw[j * stride];
                Fr u = a[k];
                a[k] = u + tt;
                a[k + half] = u - tt;
            }
        });
    }
}

// a[i] *= c0 * base^i, i < n
template <class Fr>
static void scale_pow(Fr* a, size_t n, const Fr& base, const Fr& c0, int threads) {
    const int T = (int)std::max<size_t>(1, std::min<size_t>(threads, n / 4096 + 1));
    run_parallel(T, T, [&](int t) {
        size_t lo = n * t / T, hi = n * (t + 1) / T;
        Fr cur = c0 * base.pow64(lo);
        for (size_t i = lo; i < hi; i++) { a[i] = a[i] * cur; cur = cur * base; }
    });
}

// primitive 2^log_n-th root of unity
template <class Fr>
static Fr root_of_unity(const FrConsts<Fr>& K, int log_n) {
    Fr w = K.root;
    for (int i = log_n; i < K.two_adicity; i++) w = w.sqr();
    return w;
}

template <class Fr>
static void ntt_full(Fr* a, int log_n, bool inverse, bool coset, const FrConsts<Fr>& K, int threads) {
    const size_t n = (size_t)1 << log_n;
    const Fr w = root_of_unity(K, log_n);
    if (!inverse) {
        if (coset) scale_pow(a, n, K.gen, Fr::one(), threads);
        ntt_inplace(a, log_n, w, threads);
    } else {
        ntt_inplace(a, log_n, w.inverse(), threads);
        Fr ninv = Fr::from_u64(n).inverse();
        scale_pow(a, n, coset ? K.gen.inverse() : Fr::one(), ninv, threads);
    }
}

struct Csr { const u64* row_ptr; const uint32_t* col; const void* coeff; };

template <class Fr>
static void spmv(const Csr& m, const Fr* z, Fr* out, size_t n_rows, int threads) {
    const Fr one = Fr::one();
    const Fr* co = reinterpret_cast<const Fr*>(m.coeff);
    const int T = (int)std::max<size_t>(1, std::min<size_t>(threads, n_rows / 1024 + 1));
    run_parallel(T, T, [&](int t) {
        size_t lo = n_rows * t / T, hi = n_rows * (t + 1) / T;
        for (size_t r = lo; r < hi; r++) {
            Fr acc = Fr::zero();
            for (u64 e = m.row_ptr[r]; e < m.row_ptr[r + 1]; e++) {
                const Fr& zz = z[m.col[e]];
                acc = acc + (co[e] == one ? zz : zz * co[e]);   // sr1cs/mod.rs:42-46
            }
            out[r] = acc;
        }
    });
}

template <class Fr>
static void witness_map(const Csr mats[3], size_t n_rows, size_t n_inst, const Fr* z, int log_dom, Fr* h,
                        const FrConsts<Fr>& K, int threads) {
    const size_t N = (size_t)1 << log_dom;
    std::vector<Fr> b(N, Fr::zero()), c(N, Fr::zero());
    for (size_t i = 0; i < N; i++) h[i] = Fr::zero();
    spmv(mats[0], z, h, n_rows, threads);
    spmv(mats[1], z, b.data(), n_rows, threads);
    spmv(mats[2], z, c.data(), n_rows, threads);
    for (size_t i = 0; i < n_inst; i++) h[n_rows + i] = z[i];
    Fr* v[3] = {h, b.data(), c.data()};
    for (auto p : v) ntt_full(p, log_dom, true, false, K, threads);
    for (auto p : v) ntt_full(p, log_dom, false, true, K, threads);
    u64 e = N;
    Fr zinv = (K.gen.pow(&e, 1) - Fr::one()).inverse();
    for (size_t i = 0; i < N; i++) h[i] = (h[i] * b[i] - c[i]) * zinv;
    ntt_full(h, log_dom, true, true, K, threads);
}

// ark-circom CircomReduction::witness_map_from_matrices (DESIGN.md §3.6): a = A z with the instance rows copied in, b = B z,
// c = a o b on H; each of a, b, c interpolated, its k-th coefficient multiplied by w2^k (w2 the primitive 2N-th root, so
// that the next transform evaluates at x_j = w2 w^j, the odd coset) and transformed; h = a b - c there.  C is not read.
template <class Fr>
static void witness_map_circom(const Csr mats[3], size_t n_rows, size_t n_inst, const Fr* z, int log_dom, Fr* h,
                               const FrConsts<Fr>& K, int threads) {
    const size_t N = (size_t)1 << log_dom;
    std::vector<Fr> b(N, Fr::zero()), c(N);
    for (size_t i = 0; i < N; i++) h[i] = Fr::zero();
    spmv(mats[0], z, h, n_rows, threads);
    spmv(mats[1], z, b.data(), n_rows, threads);
    for (size_t i = 0; i < n_inst; i++) h[n_rows + i] = z[i];
    for (size_t i = 0; i < N; i++) c[i] = h[i] * b[i];
    const Fr w2 = root_of_unity(K, log_dom + 1);
    for (Fr* p : {h, b.data(), c.data()}) {
        ntt_full(p, log_dom, true, false, K, threads);
        scale_pow(p, N, w2, Fr::one(), threads);
        ntt_full(p, log_dom, false, false, K, threads);
    }
    for (size_t i = 0; i < N; i++) h[i] = h[i] * b[i] - c[i];
}

// ------------------------------------------------------------------------------------------------
static void run_parallel(int threads, int jobs, const std::function<void(int)>& fn) {
    if (threads <= 1 || jobs <= 1) { for (int j = 0; j < jobs; j++) fn(j); return; }
    std::vector<std::thread> th;
    for (int j = 0; j < jobs; j++) th.emplace_back(fn, j);
    for (auto& t : th) t.join();
}

// optional phase timing on stderr (ORC_TIMING=1)
struct PhaseTimer {
    std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
    bool on = getenv("ORC_TIMING") != nullptr;
    void lap(const char* what) {
        if (!on) return;
        auto t1 = std::chrono::steady_clock::now();
        fprintf(stderr, "[oracle] %-12s %.3f s\n", what, std::chrono::duration<double>(t1 - t0).count());
        t0 = t1;
    }
};

// ---- curve instantiation -----------------------------------------------------------------------
typedef Fp<6, 0> BlsFq;
typedef Fp<4, 1> BlsFr;
typedef Fp<4, 2> BnFq;
typedef Fp<4, 3> BnFr;
typedef Fp<6, 4> Bls377Fq;
typedef Fp<4, 5> Bls377Fr;
static FrConsts<BlsFr> g_bls_fr;
static FrConsts<BnFr> g_bn_fr;
static FrConsts<Bls377Fr> g_bls377_fr;
static bool g_init = false;

// K.root = gen^((r-1)/2^S), S the two-adicity of r - 1 (S < 64)
template <class Fr>
static void init_fr_consts(FrConsts<Fr>& K, const u64* r, u64 gen, int S) {
    K.gen = Fr::from_u64(gen);
    K.two_adicity = S;
    u64 e[4], one[4] = {1, 0, 0, 0};
    sub_n<4>(e, r, one);
    for (int i = 0; i < 4; i++) e[i] = (e[i] >> S) | (i + 1 < 4 ? e[i + 1] << (64 - S) : 0);
    K.root = K.gen.pow(e, 4);
}

static void init_all() {
    if (g_init) return;
    const u64 bls_p[6] = {0xb9feffffffffaaabull, 0x1eabfffeb153ffffull, 0x6730d2a0f6b0f624ull, 0x64774b84f38512bfull, 0x4b1ba7b6434bacd7ull, 0x1a0111ea397fe69aull};
    const u64 bls_r[4] = {0xffffffff00000001ull, 0x53bda402fffe5bfeull, 0x3339d80809a1d805ull, 0x73eda753299d7d48ull};
    const u64 bn_p[4] = {0x3c208c16d87cfd47ull, 0x97816a916871ca8dull, 0xb85045b68181585dull, 0x30644e72e131a029ull};
    const u64 bn_r[4] = {0x43e1f593f0000001ull, 0x2833e84879b97091ull, 0xb85045b68181585dull, 0x30644e72e131a029ull};
    // BLS12-377: the published moduli, p = (x - 1)^2 r / 3 + x and r = x^4 - x^2 + 1 for x = 0x8508c00000000001
    const u64 bls377_p[6] = {0x8508c00000000001ull, 0x170b5d4430000000ull, 0x1ef3622fba094800ull, 0x1a22d9f300f5138full, 0xc63b05c06ca1493bull, 0x01ae3a4617c510eaull};
    const u64 bls377_r[4] = {0x0a11800000000001ull, 0x59aa76fed0000001ull, 0x60b44d1e5c37b001ull, 0x12ab655e9a2ca556ull};
    init_params<6>(BlsFq::P, bls_p);
    init_params<4>(BlsFr::P, bls_r);
    init_params<4>(BnFq::P, bn_p);
    init_params<4>(BnFr::P, bn_r);
    init_params<6>(Bls377Fq::P, bls377_p);
    init_params<4>(Bls377Fr::P, bls377_r);
    init_fr_consts(g_bls_fr, bls_r, 7, 32);
    init_fr_consts(g_bn_fr, bn_r, 5, 28);
    init_fr_consts(g_bls377_fr, bls377_r, 22, 47);
    g_init = true;
}

// One struct per curve id, for the dispatch of the exported functions
struct Bls12_381 { typedef BlsFq Fq; typedef Fp2<BlsFq> Fq2; typedef BlsFr Fr; static constexpr int bits = 255; static const FrConsts<Fr>& K() { return g_bls_fr; } };
struct Bn254 { typedef BnFq Fq; typedef Fp2<BnFq> Fq2; typedef BnFr Fr; static constexpr int bits = 254; static const FrConsts<Fr>& K() { return g_bn_fr; } };
struct Bls12_377 { typedef Bls377Fq Fq; typedef Fp2<Bls377Fq, 5> Fq2; typedef Bls377Fr Fr; static constexpr int bits = 253; static const FrConsts<Fr>& K() { return g_bls377_fr; } };

// fn(curve struct) for curve id 0 / 1 / 2 -> 0, or 1 for an unknown id
template <class Fn>
static int with_curve(int curve, Fn&& fn) {
    init_all();
    switch (curve) {
        case 0: fn(Bls12_381()); return 0;
        case 1: fn(Bn254()); return 0;
        case 2: fn(Bls12_377()); return 0;
        default: return 1;
    }
}

template <class C>
static void prove_t(const Csr mats[3], size_t n_rows, size_t n_inst, size_t n_wit, const void* const* pk,
                    const typename C::Fr* z_inst, const typename C::Fr* z_wit, const typename C::Fr* r, const typename C::Fr* s,
                    void* out_a, void* out_b, void* out_c, void* out_h, int threads) {
    typedef typename C::Fq Fq; typedef typename C::Fq2 Fq2; typedef typename C::Fr Fr;
    const FrConsts<Fr>& K = C::K();
    const int num_bits = C::bits;
    typedef Aff<Fq> A1; typedef Aff<Fq2> A2; typedef Jac<Fq> J1; typedef Jac<Fq2> J2;
    // pk pointers: alpha_g1, beta_g1, delta_g1, beta_g2, delta_g2, a_query, b_g1_query, b_g2_query, h_query, l_query
    const A1 *alpha = (const A1*)pk[0], *beta1 = (const A1*)pk[1], *delta1 = (const A1*)pk[2];
    const A2 *beta2 = (const A2*)pk[3], *delta2 = (const A2*)pk[4];
    const A1 *aq = (const A1*)pk[5], *b1q = (const A1*)pk[6], *hq = (const A1*)pk[8], *lq = (const A1*)pk[9];
    const A2* b2q = (const A2*)pk[7];
    const size_t n_vars = n_inst + n_wit;
    size_t need = n_rows + n_inst;
    int log_dom = 0;
    while (((size_t)1 << log_dom) < need) log_dom++;
    const size_t N = (size_t)1 << log_dom;
    std::vector<Fr> z(n_vars), h(N);
    memcpy(z.data(), z_inst, n_inst * sizeof(Fr));
    memcpy(z.data() + n_inst, z_wit, n_wit * sizeof(Fr));
    PhaseTimer pt;
    witness_map(mats, n_rows, n_inst, z.data(), log_dom, h.data(), K, threads);
    pt.lap("witness_map");
    if (out_h) memcpy(out_h, h.data(), N * sizeof(Fr));
    J1 h_acc = msm<Fq, Fr>(hq, h.data(), N - 1, true, threads, num_bits);
    pt.lap("msm h");
    J1 l_acc = msm<Fq, Fr>(lq, z.data() + n_inst, n_wit, true, threads, num_bits);
    pt.lap("msm l");
    Fr rc = r->from_mont(), sc = s->from_mont(), rsc = (*r * *s).from_mont();
    // calculate_coeff: r * delta + query[0] + msm(query[1..], z[1..]) + vk_param
    J1 g_a = J1::from_affine(*delta1).mul(rc.v, 4).add_affine(aq[0]).add(msm<Fq, Fr>(aq + 1, z.data() + 1, n_vars - 1, true, threads, num_bits)).add_affine(*alpha);
    J1 g1_b = J1::from_affine(*delta1).mul(sc.v, 4).add_affine(b1q[0]).add(msm<Fq, Fr>(b1q + 1, z.data() + 1, n_vars - 1, true, threads, num_bits)).add_affine(*beta1);
    J2 g2_b = J2::from_affine(*delta2).mul(sc.v, 4).add_affine(b2q[0]).add(msm<Fq2, Fr>(b2q + 1, z.data() + 1, n_vars - 1, true, threads, num_bits)).add_affine(*beta2);
    pt.lap("msm a,b1,b2");
    J1 g_c = g_a.mul(sc.v, 4).add(g1_b.mul(rc.v, 4)).add(J1::from_affine(*delta1).mul(rsc.v, 4).neg()).add(l_acc).add(h_acc);
    A1 oa = g_a.to_affine(), oc = g_c.to_affine();
    A2 ob = g2_b.to_affine();
    memcpy(out_a, &oa, sizeof(oa)); memcpy(out_b, &ob, sizeof(ob)); memcpy(out_c, &oc, sizeof(oc));
}

// out[i] = (start + i) * G for the standard generator given in affine Montgomery form (input generation for
// CPU-side MSM samples): running additions, normalised one by one.
template <class F>
static void multiples_t(const Aff<F>* gen, u64 start, size_t n, Aff<F>* out, int threads) {
    const int T = (int)std::max<size_t>(1, std::min<size_t>(threads, n / 64 + 1));
    run_parallel(T, T, [&](int t) {
        size_t lo = n * t / T, hi = n * (t + 1) / T;
        if (lo >= hi) return;
        u64 k = start + lo;
        Jac<F> cur = Jac<F>::from_affine(*gen).mul(&k, 1);
        for (size_t i = lo; i < hi; i++) { out[i] = cur.to_affine(); cur = cur.add_affine(*gen); }
    });
}

extern "C" {

int orc_threads_default() { unsigned h = std::thread::hardware_concurrency(); return h ? (int)h : 1; }

// group: 1 / 2; scalars Montgomery (mont = 1) or canonical; out: one affine point
int orc_msm(int curve, int group, const void* bases, const void* scalars, uint64_t n, int mont, int threads, void* out) {
    if (group != 1 && group != 2) return 1;
    return with_curve(curve, [&](auto c) {
        typedef decltype(c) C;
        typedef typename C::Fr Fr;
        if (group == 1) { auto r = msm<typename C::Fq, Fr>((const Aff<typename C::Fq>*)bases, (const Fr*)scalars, n, mont, threads, C::bits).to_affine(); memcpy(out, &r, sizeof(r)); }
        else { auto r = msm<typename C::Fq2, Fr>((const Aff<typename C::Fq2>*)bases, (const Fr*)scalars, n, mont, threads, C::bits).to_affine(); memcpy(out, &r, sizeof(r)); }
    });
}

int orc_ntt(int curve, void* data, int log_n, int inverse, int coset, int threads) {
    return with_curve(curve, [&](auto c) {
        typedef decltype(c) C;
        ntt_full((typename C::Fr*)data, log_n, inverse, coset, C::K(), threads);
    });
}

int orc_spmv(int curve, const uint64_t* row_ptr, const uint32_t* col, const void* coeff, uint64_t n_rows, const void* z,
             void* out, int threads) {
    Csr m{row_ptr, col, coeff};
    return with_curve(curve, [&](auto c) {
        typedef typename decltype(c)::Fr Fr;
        spmv(m, (const Fr*)z, (Fr*)out, n_rows, threads);
    });
}

// pk: 10 pointers (see prove_t).  out_h may be null.
int orc_groth16_prove(int curve, const uint64_t* const row_ptr[3], const uint32_t* const col[3], const void* const coeff[3],
                      uint64_t n_rows, uint64_t n_inst, uint64_t n_wit, const void* const* pk, const void* z_inst,
                      const void* z_wit, const void* r, const void* s, void* out_a, void* out_b, void* out_c, void* out_h,
                      int threads) {
    Csr mats[3];
    for (int k = 0; k < 3; k++) mats[k] = Csr{row_ptr[k], col[k], coeff[k]};
    return with_curve(curve, [&](auto c) {
        typedef decltype(c) C;
        typedef typename C::Fr Fr;
        prove_t<C>(mats, n_rows, n_inst, n_wit, pk, (const Fr*)z_inst, (const Fr*)z_wit, (const Fr*)r, (const Fr*)s, out_a, out_b,
                   out_c, out_h, threads);
    });
}

// h = witness_map(A, B, C, z) alone (SpMV + 7 transforms + quotient), z = instance || witness: the full-size parity
// tests compare the GPU's h with it element by element (2^24 / 2^25 domains take seconds on the host cores)
int orc_witness_map(int curve, const uint64_t* const row_ptr[3], const uint32_t* const col[3], const void* const coeff[3],
                    uint64_t n_rows, uint64_t n_inst, const void* z, int log_dom, void* out_h, int threads) {
    Csr mats[3];
    for (int k = 0; k < 3; k++) mats[k] = Csr{row_ptr[k], col[k], coeff[k]};
    return with_curve(curve, [&](auto c) {
        typedef decltype(c) C;
        typedef typename C::Fr Fr;
        witness_map(mats, n_rows, n_inst, (const Fr*)z, log_dom, (Fr*)out_h, C::K(), threads);
    });
}

// the CircomReduction's h (N odd-coset evaluations, see witness_map_circom) for the same arguments; C is not read
int orc_witness_map_circom(int curve, const uint64_t* const row_ptr[3], const uint32_t* const col[3], const void* const coeff[3],
                           uint64_t n_rows, uint64_t n_inst, const void* z, int log_dom, void* out_h, int threads) {
    Csr mats[3];
    for (int k = 0; k < 3; k++) mats[k] = Csr{row_ptr[k], col[k], coeff[k]};
    return with_curve(curve, [&](auto c) {
        typedef decltype(c) C;
        typedef typename C::Fr Fr;
        witness_map_circom(mats, n_rows, n_inst, (const Fr*)z, log_dom, (Fr*)out_h, C::K(), threads);
    });
}

// out[i] = (start + i) * gen, affine
int orc_multiples(int curve, int group, const void* gen, uint64_t start, uint64_t n, void* out, int threads) {
    if (group != 1 && group != 2) return 1;
    return with_curve(curve, [&](auto c) {
        typedef decltype(c) C;
        typedef typename C::Fq Fq; typedef typename C::Fq2 Fq2;
        if (group == 1) multiples_t((const Aff<Fq>*)gen, start, n, (Aff<Fq>*)out, threads);
        else multiples_t((const Aff<Fq2>*)gen, start, n, (Aff<Fq2>*)out, threads);
    });
}

// sum_i a[i] * b[i] over Fr (Montgomery in, Montgomery out): used by full-size parity checks
int orc_fr_dot(int curve, const void* a, const void* b, uint64_t n, void* out) {
    return with_curve(curve, [&](auto c) {
        typedef typename decltype(c)::Fr Fr;
        Fr acc = Fr::zero();
        const Fr *x = (const Fr*)a, *y = (const Fr*)b;
        for (uint64_t i = 0; i < n; i++) acc = acc + x[i] * y[i];
        memcpy(out, &acc, 32);
    });
}

}  // extern "C"
