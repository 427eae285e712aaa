// Latency-bound group arithmetic for the serial tails of a proof (Horner over the window sums: ~250 dependent doublings;
// the r/s scalar multiplications of the epilogue: 255 doublings each).  A lone thread pays 9 field multiplications per
// XYZZ doubling one after the other; here a TEAM of four adjacent lanes holds identical copies of the operands, each
// lane computes ONE of the independent products of a dependency level and the results are exchanged with warp shuffles:
// a doubling is 3 multiplication latencies deep instead of 9, a general addition 4 instead of 14.  Same formulas as
// ec.cuh (EFD xyzz dbl-2008-s-1 / add-2008-s, a = 0), same special cases, bit-identical results.
//
// Teams are lanes {4k .. 4k+3}.  Every lane of a team must call these functions with the SAME operands (team-uniform
// branches, shuffles masked to the team), so the eight teams of a warp may work on eight different points (the batched
// Horner tail) or all compute the same thing.  team_scalar_mul fills its table from lane 0: there all teams of the warp agree.
#pragma once
#include "ec.cuh"

namespace b2s {

template <class F>
__device__ __forceinline__ F team_bcast(const F& v, uint32_t src) {
    static_assert(sizeof(F) % 4 == 0, "32-bit limbs");
    F r;
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
    uint32_t* d = reinterpret_cast<uint32_t*>(&r);
    const uint32_t first = threadIdx.x & 31u & ~3u;
    const unsigned team = 0xfu << first;
#pragma unroll
    for (uint32_t i = 0; i < sizeof(F) / 4; i++) d[i] = __shfl_sync(team, s[i], (int)(first | src));
    return r;
}
template <class F>
__device__ __forceinline__ F team_sel(uint32_t t, const F& a0, const F& a1, const F& a2, const F& a3) {
    return t == 0 ? a0 : (t == 1 ? a1 : (t == 2 ? a2 : a3));
}

// p = 2 p
template <class F>
__device__ __forceinline__ void team_dbl(XYZZ<F>& p) {
    const uint32_t t = threadIdx.x & 3u;
    if (p.is_identity() || p.y.is_zero()) { p = XYZZ<F>::identity(); return; }   // uniform across the team
    const F u = p.y.dbl();
    F a = t == 0 ? u : p.x;
    F r1 = a * a;                                   // t0: V = U^2      t1: XX = X^2
    const F v = team_bcast(r1, 0), xx = team_bcast(r1, 1);
    const F m = xx.dbl() + xx;
    a = team_sel(t, u, p.x, m, m);
    F b = t == 2 ? m : v;
    F r2 = a * b;                                   // t0: W = U V      t1: S = X V      t2: M^2
    const F w = team_bcast(r2, 0), s = team_bcast(r2, 1), mm = team_bcast(r2, 2);
    const F x3 = mm - s.dbl();
    a = team_sel(t, m, w, v, w);
    b = team_sel(t, s - x3, p.y, p.zz, p.zzz);
    F r3 = a * b;                                   // t0: M (S - X3)   t1: W Y   t2: V ZZ   t3: W ZZZ
    const F ya = team_bcast(r3, 0), yb = team_bcast(r3, 1);
    p.zz = team_bcast(r3, 2);
    p.zzz = team_bcast(r3, 3);
    p.x = x3;
    p.y = ya - yb;
}

// p += q   (general XYZZ addition)
template <class F>
__device__ __forceinline__ void team_add(XYZZ<F>& p, const XYZZ<F>& q) {
    const uint32_t t = threadIdx.x & 3u;
    if (q.is_identity()) return;
    if (p.is_identity()) { p = q; return; }
    F a = team_sel(t, p.x, q.x, p.y, q.y);
    F b = team_sel(t, q.zz, p.zz, q.zzz, p.zzz);
    F r1 = a * b;                                   // U1 = X1 ZZ2   U2 = X2 ZZ1   S1 = Y1 ZZZ2   S2 = Y2 ZZZ1
    const F u1 = team_bcast(r1, 0), u2 = team_bcast(r1, 1), s1 = team_bcast(r1, 2), s2 = team_bcast(r1, 3);
    const F pp_ = u2 - u1, rr_ = s2 - s1;
    if (pp_.is_zero()) {                            // same x: doubling or cancellation (uniform across the team)
        if (rr_.is_zero()) team_dbl(p);
        else p = XYZZ<F>::identity();
        return;
    }
    a = team_sel(t, pp_, rr_, p.zz, p.zzz);
    b = team_sel(t, pp_, rr_, q.zz, q.zzz);
    F r2 = a * b;                                   // PP = P^2   RR = R^2   ZZ1 ZZ2   ZZZ1 ZZZ2
    const F pp = team_bcast(r2, 0), rr = team_bcast(r2, 1), za = team_bcast(r2, 2), zb = team_bcast(r2, 3);
    a = team_sel(t, pp_, u1, za, za);
    F r3 = a * pp;                                  // PPP = P PP   Q = U1 PP   ZZ3 = ZZ1 ZZ2 PP
    const F ppp = team_bcast(r3, 0), qv = team_bcast(r3, 1);
    p.zz = team_bcast(r3, 2);
    const F x3 = rr - ppp - qv.dbl();
    a = team_sel(t, rr_, s1, zb, zb);
    b = team_sel(t, qv - x3, ppp, ppp, ppp);
    F r4 = a * b;                                   // R (Q - X3)   S1 PPP   ZZZ3 = ZZZ1 ZZZ2 PPP
    const F ya = team_bcast(r4, 0), yb = team_bcast(r4, 1);
    p.zzz = team_bcast(r4, 2);
    p.x = x3;
    p.y = ya - yb;
}

// k * p, k little-endian 32-bit words (NOT Montgomery), fixed 4-bit windows; `table` = 16 XYZZ points of scratch owned by
// the team (shared memory).
template <class F>
__device__ __forceinline__ XYZZ<F> team_scalar_mul(const XYZZ<F>& p, const uint32_t* k, int nwords, XYZZ<F>* table) {
    const bool writer = (threadIdx.x & 31u) == 0;   // every team of the warp holds the same data: one lane fills the table
    XYZZ<F> acc = p;
    if (writer) { table[0] = XYZZ<F>::identity(); table[1] = p; }
    for (int i = 2; i < 16; i++) {
        team_add(acc, p);                           // acc = i p
        if (writer) table[i] = acc;
    }
    __syncwarp();
    acc = XYZZ<F>::identity();
    for (int w = nwords * 8 - 1; w >= 0; w--) {
        if (w != nwords * 8 - 1)
            for (int d = 0; d < 4; d++) team_dbl(acc);
        const uint32_t dig = (k[w >> 3] >> ((w & 7) * 4)) & 15u;
        if (dig) team_add(acc, table[dig]);         // digit is the same in every lane of the team
    }
    return acc;
}

// k * p without a table (double-and-add, most significant bit first): for one-off products where 16 table entries of shared
// memory per product are not worth having
template <class F>
__device__ __forceinline__ XYZZ<F> team_scalar_mul_plain(const XYZZ<F>& p, const uint32_t* k, int nwords) {
    XYZZ<F> acc = XYZZ<F>::identity();
    bool started = false;
    for (int w = nwords - 1; w >= 0; w--) {
        for (int b = 31; b >= 0; b--) {
            if (started) team_dbl(acc);
            if ((k[w] >> b) & 1u) {        // the scalar is the same in every lane of the warp
                team_add(acc, p);
                started = true;
            }
        }
    }
    return acc;
}

}  // namespace b2s