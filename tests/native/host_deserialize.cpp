// Host-side harness for the point decoder (snark_b200/csrc/deserialize.cuh): the SAME code the decode kernels run,
// compiled for the CPU with the PTX carry flag emulated, exposed to ctypes so that tests/test_host_deserialize.py can
// check it against the oracle without a GPU.  Test infrastructure only.
#include <cstdint>
#include <cstring>

#include "../../snark_b200/csrc/deserialize.cuh"

using namespace b2s;

template <class Curve, class F>
static uint32_t decode(const uint8_t* in, int compressed, int validate, uint32_t* out) {
    Affine<F> p = Affine<F>::inf();
    const uint32_t st = decode_point<Curve, F>(in, compressed != 0, validate != 0, p);
    memcpy(out, &p, sizeof(p));
    return st;
}

// curve: 0 bls12-381, 1 bn254; group 1 or 2.  `count` encodings back to back -> affine Montgomery limbs and a DecodeStatus
// per point.
extern "C" void ht_point_decode(int curve, int group, const uint8_t* in, int compressed, int validate, uint32_t* out,
                                uint32_t* status, int count) {
    const int fq = curve == 0 ? 48 : 32;
    const int pb = fq * group * (compressed ? 1 : 2), ob = 2 * fq * group / 4;
    for (int i = 0; i < count; i++) {
        const uint8_t* b = in + (size_t)i * pb;
        uint32_t* o = out + (size_t)i * ob;
        if (curve == 0 && group == 1) status[i] = decode<Bls12_381, Bls12_381::Fq>(b, compressed, validate, o);
        if (curve == 0 && group == 2) status[i] = decode<Bls12_381, Bls12_381::Fq2>(b, compressed, validate, o);
        if (curve == 1 && group == 1) status[i] = decode<Bn254, Bn254::Fq>(b, compressed, validate, o);
        if (curve == 1 && group == 2) status[i] = decode<Bn254, Bn254::Fq2>(b, compressed, validate, o);
    }
}
