// Path 6 (b200_rank_topk_pairs): the k best rows of each group of scored pairs, by (order key descending, input position
// ascending).  Kernels of pairs.cu; nothing else includes this header.
//
//  1. pairs_count_kernel     rows per group (-1: dropped row), and a flag for codes outside [-1, n_groups)
//  2. pairs_group_kernel     kept[g] = min(k, count[g]) and the rows of each size class; two exclusive scans (CUB) then
//                            give the segment offsets and the output offsets
//  3. pairs_classify_kernel  the groups of each size class, in any order
//  4. pairs_scatter_kernel   each row's (order key, position) into its group's segment, in any order within the segment
//  5. per class, one launch each: a warp per segment of <= 32 rows, a CTA bitonic sort in shared memory up to
//     PAIRS_SMEM_MAX rows, and above that a radix select of the min(k, len) best (key, ~position) composites in global
//     memory, whose survivors the host sorts with two CUB segmented sorts (position, then key, stable).
// Every comparison is the total order (key desc, position asc), so the result does not depend on the launch shape or on
// the order in which the scatter filled a segment.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200_rank.h"

#define B200_PAIRS_FULL_MASK 0xffffffffu

namespace b200 {

constexpr int PAIRS_WARP_MAX = 32;     // segments of up to this many rows: one warp each
constexpr int PAIRS_SMEM_MAX = 8192;   // segments of up to this many rows sort in shared memory (16 B per row: 128 KiB)
constexpr int PAIRS_N_CLASSES = 5;     // warp, CTA <= 256, CTA <= 2048, CTA <= PAIRS_SMEM_MAX, radix select
constexpr int PAIRS_SELECT_THREADS = 1024;

__host__ __device__ __forceinline__ int pairs_class(int64_t len) {
    return len <= PAIRS_WARP_MAX ? 0 : len <= 256 ? 1 : len <= 2048 ? 2 : len <= PAIRS_SMEM_MAX ? 3 : 4;
}

// Descending order key of a score: a larger key ranks first.  Floats: -0 is +0, every NaN gets 0 (below -inf's
// 0x000FFFFFFFFFFFFF), then the IEEE order-preserving bit map.  fp32 is widened to fp64 first, which is exact.  Ints:
// the sign bit flipped.
__device__ __forceinline__ uint64_t pairs_f64_key(double v) {
    if (v != v) return 0ull;
    if (v == 0.0) v = 0.0;
    const uint64_t b = (uint64_t)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}

__device__ __forceinline__ uint64_t pairs_key(const void* __restrict__ scores, int type, int64_t i) {
    switch (type) {
        case B200_PAIRS_F64: return pairs_f64_key(__ldg(reinterpret_cast<const double*>(scores) + i));
        case B200_PAIRS_F32: return pairs_f64_key((double)__ldg(reinterpret_cast<const float*>(scores) + i));
        case B200_PAIRS_I64:
            return (uint64_t)__ldg(reinterpret_cast<const long long*>(scores) + i) ^ 0x8000000000000000ull;
        default: return (uint64_t)(int64_t)__ldg(reinterpret_cast<const int*>(scores) + i) ^ 0x8000000000000000ull;
    }
}

// "row (ka, pa) ranks before row (kb, pb)"
__device__ __forceinline__ bool pairs_before(uint64_t ka, int64_t pa, uint64_t kb, int64_t pb) {
    return ka > kb || (ka == kb && pa < pb);
}

// Adds `v` to counter[g] once per distinct g of the warp's active lanes; returns the lane's slot among the lanes that
// share its g, plus the counter's old value.
__device__ __forceinline__ unsigned long long pairs_warp_add(unsigned long long* counter, int64_t g) {
    const unsigned active = __activemask();
    const unsigned peers = __match_any_sync(active, (unsigned long long)g);
    const int lane = threadIdx.x & 31, leader = __ffs(peers) - 1;
    unsigned long long base = 0;
    if (lane == leader) base = atomicAdd(counter + g, (unsigned long long)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    return base + __popc(peers & ((1u << lane) - 1u));
}

__global__ void __launch_bounds__(256) pairs_count_kernel(int64_t n, const int64_t* __restrict__ codes, int64_t n_groups,
                                                          unsigned long long* __restrict__ count, int* __restrict__ bad) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = __ldg(codes + i);
        if (g < -1 || g >= n_groups) {
            atomicOr(bad, 1);
        } else if (g >= 0) {
            pairs_warp_add(count, g);
        }
    }
}

// kept[g] = min(k, count[g]); class_count[c] += groups of class c (empty groups have none).
__global__ void __launch_bounds__(256) pairs_group_kernel(int64_t n_groups, int32_t k, const unsigned long long* __restrict__ count,
                                                          int64_t* __restrict__ kept, unsigned long long* __restrict__ class_count) {
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t len = (int64_t)count[g];
        kept[g] = len < k ? len : k;
        if (len > 0) pairs_warp_add(class_count, pairs_class(len));
    }
}

// class_list[class_off[c] + j] = the j-th group of class c found (any order)
__global__ void __launch_bounds__(256) pairs_classify_kernel(int64_t n_groups, const int64_t* __restrict__ seg_off,
                                                             const int64_t* __restrict__ class_off,
                                                             unsigned long long* __restrict__ class_cursor, int64_t* __restrict__ class_list) {
    for (int64_t g = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; g < n_groups; g += (int64_t)gridDim.x * blockDim.x) {
        const int64_t len = seg_off[g + 1] - seg_off[g];
        if (len == 0) continue;
        const int c = pairs_class(len);
        class_list[class_off[c] + (int64_t)pairs_warp_add(class_cursor, c)] = g;
    }
}

__global__ void __launch_bounds__(256) pairs_scatter_kernel(int64_t n, const int64_t* __restrict__ codes, const void* __restrict__ scores,
                                                            int type, const int64_t* __restrict__ seg_off,
                                                            unsigned long long* __restrict__ cursor, uint64_t* __restrict__ seg_key,
                                                            int64_t* __restrict__ seg_pos) {
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t g = __ldg(codes + i);
        if (g < 0) continue;
        const int64_t dst = seg_off[g] + (int64_t)pairs_warp_add(cursor, g);
        seg_key[dst] = pairs_key(scores, type, i);
        seg_pos[dst] = i;
    }
}

// Segments of <= 32 rows, one warp each: a lane's rank is the number of rows that rank before it.
__global__ void __launch_bounds__(256) pairs_warp_kernel(int64_t n_seg, const int64_t* __restrict__ list, const int64_t* __restrict__ seg_off,
                                                         const int64_t* __restrict__ out_off, const uint64_t* __restrict__ seg_key,
                                                         const int64_t* __restrict__ seg_pos, int64_t* __restrict__ out_pos) {
    const int64_t s = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (s >= n_seg) return;
    const int lane = threadIdx.x & 31;
    const int64_t g = list[s], lo = seg_off[g], len = seg_off[g + 1] - lo, o = out_off[g], kept = out_off[g + 1] - o;
    const bool valid = lane < len;
    const uint64_t key = valid ? seg_key[lo + lane] : 0ull;
    const int64_t pos = valid ? seg_pos[lo + lane] : INT64_MAX;
    int rank = 0;
#pragma unroll
    for (int j = 0; j < 32; ++j) {
        const uint64_t kj = __shfl_sync(B200_PAIRS_FULL_MASK, key, j);
        const int64_t pj = __shfl_sync(B200_PAIRS_FULL_MASK, pos, j);
        rank += pairs_before(kj, pj, key, pos);
    }
    if (valid && rank < kept) out_pos[o + rank] = pos;
}

// Segments of (256, 2048 or PAIRS_SMEM_MAX] rows (class by CAP), one CTA each: a bitonic sort of the segment, padded to
// a power of two with rows that rank last, in dynamic shared memory (CAP x 16 B), then the first min(k, len) positions.
template <int CAP, int THREADS>
__global__ void __launch_bounds__(THREADS) pairs_cta_kernel(const int64_t* __restrict__ list, const int64_t* __restrict__ seg_off,
                                                            const int64_t* __restrict__ out_off, const uint64_t* __restrict__ seg_key,
                                                            const int64_t* __restrict__ seg_pos, int64_t* __restrict__ out_pos) {
    extern __shared__ uint64_t pairs_smem[];
    uint64_t* sk = pairs_smem;
    int64_t* sp = reinterpret_cast<int64_t*>(pairs_smem + CAP);
    const int tid = threadIdx.x;
    const int64_t g = list[blockIdx.x], lo = seg_off[g], o = out_off[g];
    const int len = (int)(seg_off[g + 1] - lo), kept = (int)(out_off[g + 1] - o);
    int N = 2;
    while (N < len) N <<= 1;
    for (int i = tid; i < N; i += THREADS) {
        sk[i] = i < len ? seg_key[lo + i] : 0ull;
        sp[i] = i < len ? seg_pos[lo + i] : INT64_MAX;
    }
    __syncthreads();
    for (int size = 2; size <= N; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = tid; t < (N >> 1); t += THREADS) {
                const int i = 2 * t - (t & (stride - 1)), j = i + stride;
                const uint64_t ki = sk[i], kj = sk[j];
                const int64_t pi = sp[i], pj = sp[j];
                const bool first = (i & size) == 0;  // this run ends up best-first
                if (first ? pairs_before(kj, pj, ki, pi) : pairs_before(ki, pi, kj, pj)) {
                    sk[i] = kj;
                    sk[j] = ki;
                    sp[i] = pj;
                    sp[j] = pi;
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < kept; i += THREADS) out_pos[o + i] = sp[i];
}

// Segments of more than PAIRS_SMEM_MAX rows, one CTA each: radix select, 8 bits at a time from the top, of the
// min(k, len) largest composites (key, ~position) -- unique, so the select ends at a prefix whose bucket is taken whole --
// and every row at or above that prefix copied to surv_* at out_off[g], in any order.  Block s also writes its segment's
// bounds in surv_* to seg_begin[s] / seg_end[s] for the sorts that follow.
__global__ void __launch_bounds__(PAIRS_SELECT_THREADS) pairs_select_kernel(const int64_t* __restrict__ list, const int64_t* __restrict__ seg_off,
                                                                            const int64_t* __restrict__ out_off, const uint64_t* __restrict__ seg_key,
                                                                            const int64_t* __restrict__ seg_pos, uint64_t* __restrict__ surv_key,
                                                                            int64_t* __restrict__ surv_pos, int64_t* __restrict__ seg_begin,
                                                                            int64_t* __restrict__ seg_end) {
    __shared__ unsigned long long hist[256];
    __shared__ unsigned long long s_need, s_fill;
    __shared__ int s_digit, s_done;
    const int tid = threadIdx.x;
    const int64_t g = list[blockIdx.x], lo = seg_off[g], len = seg_off[g + 1] - lo, o = out_off[g], kept = out_off[g + 1] - o;
    const uint64_t* key = seg_key + lo;
    const int64_t* pos = seg_pos + lo;
    uint64_t pre_hi = 0, pre_lo = 0, mask_hi = 0, mask_lo = 0;  // the composite's top bytes chosen so far
    if (tid == 0) {
        s_need = (unsigned long long)kept;
        s_fill = 0;
        seg_begin[blockIdx.x] = o;
        seg_end[blockIdx.x] = o + kept;
    }
    __syncthreads();
    bool all = kept == len;  // every row survives: no select
    for (int d = 0; d < 16 && !all; ++d) {
        for (int b = tid; b < 256; b += PAIRS_SELECT_THREADS) hist[b] = 0;
        __syncthreads();
        const int shift = 56 - 8 * (d & 7);
        for (int64_t i = tid; i < len; i += PAIRS_SELECT_THREADS) {
            const uint64_t hi = key[i];
            if ((hi & mask_hi) != pre_hi) continue;
            const uint64_t lw = ~(uint64_t)pos[i];
            if ((lw & mask_lo) != pre_lo) continue;
            pairs_warp_add(hist, (int64_t)(((d < 8 ? hi : lw) >> shift) & 255u));
        }
        __syncthreads();
        if (tid == 0) {  // the bucket holding the need-th largest of the rows that match the prefix
            unsigned long long need = s_need, cum = 0;
            int b = 255;
            for (; b > 0 && cum + hist[b] < need; --b) cum += hist[b];
            s_digit = b;
            s_need = need - cum;
            s_done = hist[b] == need - cum;
        }
        __syncthreads();
        const uint64_t dg = (uint64_t)s_digit << shift, dm = 255ull << shift;
        if (d < 8) {
            pre_hi |= dg;
            mask_hi |= dm;
        } else {
            pre_lo |= dg;
            mask_lo |= dm;
        }
        const bool done = s_done;
        __syncthreads();
        if (done) break;
    }
    for (int64_t base = 0; base < len; base += PAIRS_SELECT_THREADS) {
        const int64_t i = base + tid;
        bool take = false;
        uint64_t hi = 0;
        int64_t p = 0;
        if (i < len) {
            hi = key[i];
            p = pos[i];
            const uint64_t mh = hi & mask_hi, ml = ~(uint64_t)p & mask_lo;
            take = all || mh > pre_hi || (mh == pre_hi && ml >= pre_lo);
        }
        const unsigned ballot = __ballot_sync(B200_PAIRS_FULL_MASK, take);
        const int lane = tid & 31;
        unsigned long long base_slot = 0;
        if (lane == 0 && ballot) base_slot = atomicAdd(&s_fill, (unsigned long long)__popc(ballot));
        base_slot = __shfl_sync(B200_PAIRS_FULL_MASK, base_slot, 0);
        if (take) {
            const int64_t dst = o + (int64_t)base_slot + __popc(ballot & ((1u << lane) - 1u));
            surv_key[dst] = hi;
            surv_pos[dst] = p;
        }
    }
}

// The sorted survivors of each radix-select segment into the output.
__global__ void __launch_bounds__(256) pairs_copy_kernel(const int64_t* __restrict__ list, const int64_t* __restrict__ out_off,
                                                         const int64_t* __restrict__ src, int64_t* __restrict__ out_pos) {
    const int64_t g = list[blockIdx.x], lo = out_off[g], hi = out_off[g + 1];
    for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) out_pos[i] = src[i];
}

}  // namespace b200
