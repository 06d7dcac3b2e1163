// Shared device helpers for the b200_rank kernels (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>
#include <stdint.h>

#define B200_FULL_MASK 0xffffffffu
#define B200_PAD_ID 0x7fffffff

namespace b200 {

// Object factors are read in their stored type (fp32, or fp16 / bf16 kept at 16 bits) and widened on load: every 16-bit
// value is exact in fp32, so a kernel sees the operand a widened fp32 copy would have given it.
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }

// The same from the raw 16 bits of one element (elements unpacked from a vector load).
template <typename T>
__device__ __forceinline__ float bits_to_f32(unsigned bits);
template <>
__device__ __forceinline__ float bits_to_f32<__half>(unsigned bits) {
    return __half2float(__ushort_as_half((unsigned short)bits));
}
template <>
__device__ __forceinline__ float bits_to_f32<__nv_bfloat16>(unsigned bits) {
    return __bfloat162float(__ushort_as_bfloat16((unsigned short)bits));
}

// "a ranks before b": higher score first, ties by smaller object id (the order fixed by the oracle).
__device__ __forceinline__ bool ranks_before(float as, int ai, float bs, int bi) {
    return as > bs || (as == bs && ai < bi);
}

// Bitonic sort of one (score, id) pair per lane; lane 0 ends up with the best pair.
__device__ __forceinline__ void warp_sort32(float& s, int& id, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const float os = __shfl_xor_sync(B200_FULL_MASK, s, j);
            const int oi = __shfl_xor_sync(B200_FULL_MASK, id, j);
            const bool lower = (lane & j) == 0;
            const bool dir = (lane & k) == 0;  // k == 32: always true -> best-first overall
            const bool keep_better = (lower == dir);
            const bool take = keep_better ? ranks_before(os, oi, s, id) : ranks_before(s, id, os, oi);
            if (take) {
                s = os;
                id = oi;
            }
        }
    }
}

// run (sorted best-first) <- best 32 of run U fresh (fresh sorted best-first).
__device__ __forceinline__ void warp_merge_top32(float& run_s, int& run_i, float fresh_s, int fresh_i, int lane) {
    const float rs = __shfl_sync(B200_FULL_MASK, fresh_s, 31 - lane);
    const int ri = __shfl_sync(B200_FULL_MASK, fresh_i, 31 - lane);
    if (ranks_before(rs, ri, run_s, run_i)) {
        run_s = rs;
        run_i = ri;
    }
    // (run, reversed fresh) element-wise best is bitonic and holds the best 32: one bitonic merge finishes the job
#pragma unroll
    for (int j = 16; j > 0; j >>= 1) {
        const float os = __shfl_xor_sync(B200_FULL_MASK, run_s, j);
        const int oi = __shfl_xor_sync(B200_FULL_MASK, run_i, j);
        const bool lower = (lane & j) == 0;
        const bool take = lower ? ranks_before(os, oi, run_s, run_i) : ranks_before(run_s, run_i, os, oi);
        if (take) {
            run_s = os;
            run_i = oi;
        }
    }
}

// Is `item` among the sorted column ids indices[lo, hi)?  (filter_pairs_csr structure lookup)
__device__ __forceinline__ bool csr_contains(const int32_t* __restrict__ indices, int64_t lo, int64_t hi, int item) {
    const int64_t end = hi;
    while (lo < hi) {  // lower_bound
        const int64_t mid = (lo + hi) >> 1;
        const int v = __ldg(indices + mid);
        if (v < item)
            lo = mid + 1;
        else
            hi = mid;
    }
    return lo < end && __ldg(indices + lo) == item;
}

}  // namespace b200
