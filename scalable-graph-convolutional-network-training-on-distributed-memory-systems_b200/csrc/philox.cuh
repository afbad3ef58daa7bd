// Philox4x32-10, the counter-based generator of Salmon et al., "Parallel random numbers: as easy as 1, 2, 3" (SC 2011),
// with the Random123 constants. A pure function of a 128-bit counter and a 64-bit key, so a device thread draws the
// words of any counter without state, and a host (tests/dropout_oracle.py) reproduces them bit for bit.
//
// Known answers (Random123 kat_vectors):
//   counter 0, key 0                                            -> 6627e8d5 e169c58d bc57ac4c 9b00dbd8
//   counter ffffffff x4, key ffffffff x2                        -> 408f276d 41c83b0e a20bc7c6 6d5451fd
//   counter 243f6a88 85a308d3 13198a2e 03707344, key a4093822 299f31d0
//                                                               -> d16cfe09 94fdcceb 5001e420 24126ea1
#pragma once

#include <cstdint>

namespace pgcn {

constexpr uint32_t kPhiloxM0 = 0xD2511F53u, kPhiloxM1 = 0xCD9E8D57u;
constexpr uint32_t kPhiloxW0 = 0x9E3779B9u, kPhiloxW1 = 0xBB67AE85u;

__host__ __device__ __forceinline__ void philox_mulhilo(uint32_t a, uint32_t b, uint32_t& hi, uint32_t& lo)
{
#ifdef __CUDA_ARCH__
    lo = a * b;
    hi = __umulhi(a, b);
#else
    const uint64_t p = (uint64_t)a * b;
    lo = (uint32_t)p;
    hi = (uint32_t)(p >> 32);
#endif
}

// The four words of counter (c0, c1, c2, c3) under key (k0, k1), written to w[0..3].
__host__ __device__ __forceinline__ void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                                       uint32_t k1, uint32_t w[4])
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) {
            k0 += kPhiloxW0;
            k1 += kPhiloxW1;
        }
        uint32_t hi0, lo0, hi1, lo1;
        philox_mulhilo(kPhiloxM0, c0, hi0, lo0);
        philox_mulhilo(kPhiloxM1, c2, hi1, lo1);
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
    }
    w[0] = c0; w[1] = c1; w[2] = c2; w[3] = c3;
}

}  // namespace pgcn
