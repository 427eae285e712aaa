// Curve bundles: the field / group types and generators for the three supported pairing curves.
// curve ids match B2S_CURVE_* in include/b200snark.h.
#pragma once
#include "ec.cuh"
#include "field_params.h"

namespace b2s {

template <class FqP_, class FrP_, int ID>
struct CurveT {
    static constexpr int id = ID;
    using FqP = FqP_;
    using FrP = FrP_;
    using Fq = Fp<FqP_>;
    using Fr = Fp<FrP_>;
    using Fq2 = Fp2<FqP_>;
    using G1Affine = Affine<Fq>;
    using G2Affine = Affine<Fq2>;
    using G1 = XYZZ<Fq>;
    using G2 = XYZZ<Fq2>;

    B2S_HD static G1Affine g1_generator() {
        G1Affine g;
#pragma unroll
        for (int i = 0; i < Fq::N; i++) { g.x.v[i] = FqP::g1x(i); g.y.v[i] = FqP::g1y(i); }
        return g;
    }
    B2S_HD static G2Affine g2_generator() {
        G2Affine g;
#pragma unroll
        for (int i = 0; i < Fq::N; i++) {
            g.x.c0.v[i] = FqP::g2x0(i); g.x.c1.v[i] = FqP::g2x1(i);
            g.y.c0.v[i] = FqP::g2y0(i); g.y.c1.v[i] = FqP::g2y1(i);
        }
        return g;
    }
};

using Bls12_381 = CurveT<BlsFqP, BlsFrP, 0>;
using Bn254 = CurveT<BnFqP, BnFrP, 1>;
using Bls12_377 = CurveT<Bls377FqP, Bls377FrP, 2>;

}  // namespace b2s
