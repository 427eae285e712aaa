// Micro-benchmarks that set the ALU roofline for the field arithmetic: how many Montgomery
// multiplications / mixed additions per second the chip sustains when nothing else is in the way, and the latency
// and throughput of the field inversion against the Fermat chain it replaced (`microbench inv` runs only that case).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -DB2S_INLINE_MUL -I snark_b200/csrc -o build/microbench tools/microbench.cu
#define B2S_INLINE_MUL 1
#include <cstdio>
#include <string>
#include <cuda_runtime.h>
#include "curves.cuh"
using namespace b2s;

template <class F, int ILP>
__global__ void mul_chain(F* out, const F* in, int iters) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    F x[ILP], y = in[i];
#pragma unroll
    for (int k = 0; k < ILP; k++) x[k] = in[i + k + 1];
    for (int it = 0; it < iters; it++) {
#pragma unroll
        for (int k = 0; k < ILP; k++) x[k] = x[k] * y;
    }
    F acc = x[0];
#pragma unroll
    for (int k = 1; k < ILP; k++) acc = acc + x[k];
    out[i] = acc;
}

template <class F>
__global__ void madd_chain(XYZZ<F>* out, const Affine<F>* in, int iters) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    XYZZ<F> acc = XYZZ<F>::from_affine(in[i]);
    Affine<F> q = in[i + 1];
    for (int it = 0; it < iters; it++) {
        acc.add_affine(q);
        q.x = q.x + acc.zz;  // keep the operand changing (not a curve point; the formulas do not care)
    }
    out[i] = acc;
}

// inversion: each thread runs `iters` dependent steps of one kind -- 0: inverse() (divsteps), 1: the Fermat chain
// pow_words(p - 2), 2: one Montgomery product
struct Words { uint32_t w[12]; };

template <class F, int OP>
__global__ void inv_chain(F* out, const F* in, int iters, Words pm2) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    F x = in[i], y = in[i + 1];
    for (int it = 0; it < iters; it++) {
        if (OP == 0) x = x.inverse();
        if (OP == 1) x = x.pow_words(pm2.w, F::N);
        if (OP == 2) x = x * y;
    }
    out[i] = x;
}

template <class P>
Words p_minus_2(const Fp<P>*) {
    Words e{};
    uint64_t borrow = 2;
    for (int i = 0; i < P::N; i++) {
        const uint64_t d = (uint64_t)P::mod(i) - borrow;
        e.w[i] = (uint32_t)d;
        borrow = (d >> 63) & 1;
    }
    return e;
}

template <class K, class... A>
float time_kernel(K k, dim3 g, dim3 b, A... args) {
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    k<<<g, b>>>(args...);
    cudaDeviceSynchronize();
    cudaEventRecord(e0);
    k<<<g, b>>>(args...);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    return ms;
}

template <class F, int ILP>
void bench_mul(const char* name, int threads, int blocks_per_sm) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int blocks = sms * blocks_per_sm, iters = 2000;
    size_t n = (size_t)blocks * threads + ILP + 2;
    F *in, *out; cudaMalloc(&in, n * sizeof(F)); cudaMalloc(&out, n * sizeof(F));
    cudaMemset(in, 0x5a, n * sizeof(F));
    float ms = time_kernel(mul_chain<F, ILP>, dim3(blocks), dim3(threads), out, in, iters);
    double muls = (double)blocks * threads * iters * ILP;
    printf("%-10s ilp=%d thr=%d blk/sm=%d : %.3f ms  %.3e mul/s\n", name, ILP, threads, blocks_per_sm, ms, muls / ms * 1e3);
    cudaFree(in); cudaFree(out);
}

template <class F>
void bench_madd(const char* name, int threads, int blocks_per_sm) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    int blocks = sms * blocks_per_sm, iters = 500;
    size_t n = (size_t)blocks * threads + 2;
    Affine<F>* in; XYZZ<F>* out; cudaMalloc(&in, n * sizeof(Affine<F>)); cudaMalloc(&out, n * sizeof(XYZZ<F>));
    cudaMemset(in, 0x3c, n * sizeof(Affine<F>));
    float ms = time_kernel(madd_chain<F>, dim3(blocks), dim3(threads), out, in, iters);
    double adds = (double)blocks * threads * iters;
    printf("%-10s madd thr=%d blk/sm=%d : %.3f ms  %.3e add/s\n", name, threads, blocks_per_sm, ms, adds / ms * 1e3);
    cudaFree(in); cudaFree(out);
}

// latency: one warp, each lane a chain of dependent operations; throughput: 4 CTAs of 128 threads per SM
template <class F, int OP>
double bench_inv_one(bool latency, int iters) {
    int sms; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    const int blocks = latency ? 1 : sms * 4, threads = latency ? 32 : 128;
    size_t n = (size_t)blocks * threads + 2;
    F *in, *out; cudaMalloc(&in, n * sizeof(F)); cudaMalloc(&out, n * sizeof(F));
    cudaMemset(in, 0x11, n * sizeof(F));   // 0x11.. words: below p for every field here
    float ms = time_kernel(inv_chain<F, OP>, dim3(blocks), dim3(threads), out, in, iters, p_minus_2((const F*)nullptr));
    cudaFree(in); cudaFree(out);
    const double ops = (double)blocks * threads * iters;
    return latency ? ms * 1e3 / iters : ops / ms * 1e3;   // us per operation, or operations per second
}

template <class F>
void bench_inv(const char* name) {
    const double li = bench_inv_one<F, 0>(true, 200), lp = bench_inv_one<F, 1>(true, 10), lm = bench_inv_one<F, 2>(true, 20000);
    printf("%-10s latency  : inverse %.2f us  pow(p-2) %.2f us  mul %.4f us  (pow / inverse = %.1fx, inverse = %.0f muls)\n",
           name, li, lp, lm, lp / li, li / lm);
    const double ti = bench_inv_one<F, 0>(false, 8), tp = bench_inv_one<F, 1>(false, 1), tm = bench_inv_one<F, 2>(false, 4000);
    printf("%-10s throughput: inverse %.3e/s  pow(p-2) %.3e/s  mul %.3e/s  (inverse / pow = %.1fx)\n", name, ti, tp, tm, ti / tp);
}

int main(int argc, char** argv) {
    using BF = Bls12_381::Fq; using BR = Bls12_381::Fr; using NF = Bn254::Fq;
    bench_inv<BF>("bls_fq");
    bench_inv<BR>("bls_fr");
    if (argc > 1 && std::string(argv[1]) == "inv") {
        cudaError_t e = cudaDeviceSynchronize();
        printf("status: %s\n", cudaGetErrorString(e));
        return e != cudaSuccess;
    }
    for (int bps : {1, 2, 4}) {
        bench_mul<BF, 1>("bls_fq", 128, bps);
        bench_mul<BF, 2>("bls_fq", 128, bps);
    }
    bench_mul<BF, 1>("bls_fq", 256, 2);
    bench_mul<BF, 1>("bls_fq", 256, 4);
    for (int bps : {2, 4, 8}) { bench_mul<BR, 1>("bls_fr", 128, bps); bench_mul<BR, 2>("bls_fr", 128, bps); }
    for (int bps : {2, 4, 8}) { bench_mul<NF, 1>("bn_fq", 128, bps); bench_mul<NF, 2>("bn_fq", 128, bps); }
    for (int bps : {1, 2, 3, 4}) bench_madd<BF>("bls_g1", 128, bps);
    for (int bps : {2, 4}) bench_madd<NF>("bn_g1", 128, bps);
    cudaError_t e = cudaDeviceSynchronize();
    printf("status: %s\n", cudaGetErrorString(e));
    return e != cudaSuccess;
}
