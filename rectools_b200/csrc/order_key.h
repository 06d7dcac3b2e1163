// Order key of an fp32 score for the radix selection of large_k_select.cuh: an unsigned 32-bit integer whose order is the
// order of the scores the selection keeps.  Plain C++ (no CUDA header needed), so that tests/test_large_k_select_cpu.py
// compiles it with g++ and pins it.
//
//  - -0.0 and +0.0 get the same key: the streaming passes compare scores with == / >, so the two zeros tie and are
//    ordered by object id.
//  - -inf and every NaN get key 0, which no kept score has: the passes keep only scores > -inf, so these never rank.
//  - every other score s maps to a key >= 0x00800000 (-FLT_MAX) and <= 0xFF800000 (+inf), strictly increasing in s.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define B200_KEY_FN __host__ __device__ __forceinline__
#else
#define B200_KEY_FN inline
#endif

namespace b200 {

constexpr uint32_t ORDER_KEY_INVALID = 0u;

B200_KEY_FN uint32_t order_key(float s) {
    if (!(s > -__builtin_huge_valf())) return ORDER_KEY_INVALID;  // -inf, NaN
    if (s == 0.0f) return 0x80000000u;                            // -0.0 == +0.0
    uint32_t b;
    memcpy(&b, &s, sizeof(b));
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

}  // namespace b200
