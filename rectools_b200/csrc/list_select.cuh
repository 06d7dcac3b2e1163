// Path 7 (b200_rank_topk_list): the first k positions of one shared, ordered list whose id is not among a row's viewed ids
// -- the per-user step of `PopularModel._recommend_u2i` (rectools/models/popular.py:229-277).  Kernels of list.cu;
// nothing else includes this header.
//
// Row r scans the list positions [0, min(n_list, k + m_r)), m_r = its viewed count, as the reference's window does
// (popular.py:264-275): with distinct list ids that window holds at least k unviewed positions whenever the list does, so
// the result is also the first k unviewed positions of the whole list.  The scan goes in steps of 32 x W consecutive
// positions: every lane binary-searches its position's id in the row's sorted viewed ids, a ballot (and, for W > 1, the
// warps' counts in shared memory) gives each kept position its output slot, and the row stops once k are kept.
//   W = 1: one warp per row, eight rows per CTA (k_out <= LIST_WARP_K);
//   W = 8: one CTA of 256 threads per row, for long scans.
// The list is read by every row, so it stays in L2 (4 MB at 10^6 entries).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "common.cuh"

namespace b200 {

constexpr int LIST_THREADS = 256;
constexpr int LIST_WARP_K = 256;  // k_out up to this: a warp per row

struct ListRows {
    const int32_t* list;    // [n_list] ids, in list order
    int64_t n_list;
    const int64_t* indptr;  // [n_rows + 1] row pointers of this chunk, absolute (minus `base`); NULL: nothing viewed
    int64_t base;           // indptr value of the chunk's first row
    const int32_t* indices; // the chunk's viewed ids, sorted ascending within a row
    int64_t n_rows;
    int k;
    int k_out;
    int32_t* out_pos;       // [n_rows, k_out]
    int32_t* out_counts;    // [n_rows]
};

template <int W>
__global__ void __launch_bounds__(LIST_THREADS) list_select_kernel(ListRows a) {
    static_assert(W == 1 || W == LIST_THREADS / 32, "a row is one warp or one CTA");
    constexpr int ROWS = LIST_THREADS / 32 / W;  // rows per CTA
    __shared__ int warp_kept[LIST_THREADS / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int sub = warp % W;  // warp within the row
    const int64_t r = (int64_t)blockIdx.x * ROWS + warp / W;
    if (r >= a.n_rows) return;  // (W > 1: the whole CTA)
    int64_t lo = 0, hi = 0;
    if (a.indptr) {
        lo = a.indptr[r] - a.base;
        hi = a.indptr[r + 1] - a.base;
    }
    const int64_t limit = min(a.n_list, (int64_t)a.k + (hi - lo));
    int32_t* out = a.out_pos + r * a.k_out;
    const unsigned below = (1u << lane) - 1u;
    int kept = 0;  // the same in every thread of the row
    for (int64_t p0 = 0; p0 < limit && kept < a.k; p0 += 32 * W) {
        const int64_t p = p0 + sub * 32 + lane;
        bool keep = false;
        if (p < limit) keep = !(hi > lo && csr_contains(a.indices, lo, hi, __ldg(a.list + p)));
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        int before = 0, total = __popc(ballot);
        if constexpr (W > 1) {
            if (lane == 0) warp_kept[warp] = total;
            __syncthreads();
            total = 0;
            for (int w = 0; w < W; ++w) {
                const int c = warp_kept[w];
                if (w < sub) before += c;
                total += c;
            }
            __syncthreads();  // warp_kept is rewritten by the next step
        }
        const int slot = kept + before + __popc(ballot & below);
        if (keep && slot < a.k) out[slot] = (int32_t)p;
        kept += total;
    }
    kept = min(kept, a.k);
    for (int j = kept + sub * 32 + lane; j < a.k_out; j += 32 * W) out[j] = -1;
    if (sub == 0 && lane == 0) a.out_counts[r] = kept;
}

}  // namespace b200
