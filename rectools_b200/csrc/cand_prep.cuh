// Path 5 from device memory (b200_rank_topk_candidates_device): raw per-row candidate lists -- int32 ids in any order,
// repeats allowed, ids outside [0, n_objects) meaning "no candidate" -- turned into the strictly ascending lists that
// cand_score_kernel and cand_select_kernel (cand_select.cuh) take, on the device, one row chunk at a time.
//
//  1. cand_prep_kernel, one CTA per row: the row's valid ids are compacted in position order (block-wide scans), sorted
//     ascending by lk_sort_desc on the key ~id (large_k_select.cuh; in shared memory up to smem_pairs entries, above that
//     in 16 B per raw entry of global scratch, which holds the chunk's long rows only, each at its sort_off entry), and
//     written once each, ascending, at the row's chunk-local raw offset of `ids`; the kept count goes to kept[r].
//  2. an in-place exclusive scan of the kept counts (cub::DeviceScan) gives the chunk-local, 0-based row pointers.
//  3. cand_compact_kernel moves each row's prepared ids from its raw offset to its place in that ragged layout.
// The ranking kernels then run unchanged, so a pair's score bits and a row's result are those of the host route on the
// same lists normalised on the host.
#pragma once
#include "large_k_select.cuh"

namespace b200 {

struct CandPrepParams {
    const int64_t* raw_indptr;   // [n_rows + 1]: the chunk's rows, absolute offsets into raw_indices
    const int32_t* raw_indices;
    int64_t raw_base = 0;        // raw_indptr[0]: row r starts at chunk-local raw offset raw_indptr[r] - raw_base
    int64_t n_rows = 0;
    int64_t n_objects = 0;
    int32_t smem_pairs = 0;      // rows of at most this many raw entries sort in dynamic shared memory (16 B per entry)
    uint32_t* scratch;           // [4 x raw entries of the chunk's rows longer than smem_pairs] words, or nullptr
    const int64_t* sort_off;     // [n_rows]: a row longer than smem_pairs sorts at scratch + 4 x sort_off[r] (else unread)
    int32_t* ids;                // [raw entries]: row r's prepared ids at its chunk-local raw offset
    int64_t* kept;               // [n_rows + 1]: kept[r] = row r's prepared count
};

// One CTA of LK_THREADS threads per row; dynamic shared memory 16 x smem_pairs bytes.
__global__ void __launch_bounds__(LK_THREADS) cand_prep_kernel(const CandPrepParams p) {
    extern __shared__ uint32_t lk_smem[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t wcnt[LK_WARPS][256];
    __shared__ uint32_t s_warp[LK_WARPS];
    const int tid = threadIdx.x;
    const int64_t r = blockIdx.x;
    const int64_t lo = __ldg(p.raw_indptr + r), n = __ldg(p.raw_indptr + r + 1) - lo;
    const int64_t off = lo - p.raw_base;
    const int32_t* src = p.raw_indices + lo;
    constexpr int64_t TILE = (int64_t)LK_THREADS * LK_ITEMS;

    uint32_t *ka, *pa, *kb, *pb;
    if (n <= p.smem_pairs) {
        ka = lk_smem;
        pa = ka + p.smem_pairs;
        kb = pa + p.smem_pairs;
        pb = kb + p.smem_pairs;
    } else {
        ka = p.scratch + 4 * __ldg(p.sort_off + r);
        pa = ka + n;
        kb = pa + n;
        pb = kb + n;
    }

    // a. the valid ids in position order: key ~id (descending key = ascending id), the id itself as the value
    uint32_t m = 0;
    for (int64_t base = 0; base < n; base += TILE) {
        const int64_t p0 = base + (int64_t)tid * LK_ITEMS;
        int32_t v[LK_ITEMS];
        uint32_t cnt = 0;
#pragma unroll
        for (int j = 0; j < LK_ITEMS; ++j) {
            v[j] = p0 + j < n ? __ldg(src + p0 + j) : -1;
            if (v[j] >= 0 && (int64_t)v[j] < p.n_objects) ++cnt;
            else v[j] = -1;
        }
        uint32_t total;
        uint32_t dst = m + lk_block_scan(cnt, s_warp, total);
#pragma unroll
        for (int j = 0; j < LK_ITEMS; ++j) {
            if (v[j] < 0) continue;
            ka[dst] = ~(uint32_t)v[j];
            pa[dst] = (uint32_t)v[j];
            ++dst;
        }
        m += total;
    }
    __syncthreads();

    // b. ascending ids (stable sort by key descending)
    const uint32_t* sorted = lk_sort_desc(ka, pa, kb, pb, m, hist, wcnt) ? pb : pa;
    __syncthreads();

    // c. each id once, ascending, at the row's raw offset
    int32_t* out = p.ids + off;
    uint32_t kept = 0;
    for (int64_t base = 0; base < (int64_t)m; base += TILE) {
        const int64_t p0 = base + (int64_t)tid * LK_ITEMS;
        int32_t v[LK_ITEMS];
        uint32_t cnt = 0;
#pragma unroll
        for (int j = 0; j < LK_ITEMS; ++j) {
            const int64_t i = p0 + j;
            v[j] = -1;
            if (i < (int64_t)m && (i == 0 || sorted[i] != sorted[i - 1])) {
                v[j] = (int32_t)sorted[i];
                ++cnt;
            }
        }
        uint32_t total;
        uint32_t dst = kept + lk_block_scan(cnt, s_warp, total);
#pragma unroll
        for (int j = 0; j < LK_ITEMS; ++j)
            if (v[j] >= 0) out[dst++] = v[j];
        kept += total;
    }
    if (tid == 0) p.kept[r] = kept;
}

// grid (n_rows, segments of CS_SEG entries), 256 threads: row r's prepared ids from its raw offset to c_indptr[r].
__global__ void __launch_bounds__(256) cand_compact_kernel(const int64_t* __restrict__ raw_indptr, int64_t raw_base,
                                                           const int32_t* __restrict__ ids, const int64_t* __restrict__ c_indptr,
                                                           int32_t* __restrict__ c_indices, int64_t seg) {
    const int64_t r = blockIdx.x;
    const int64_t lo = c_indptr[r], n = c_indptr[r + 1] - lo;
    const int32_t* src = ids + (__ldg(raw_indptr + r) - raw_base);
    const int64_t stride = (int64_t)gridDim.y * seg;
    for (int64_t base = (int64_t)blockIdx.y * seg; base < n; base += stride)
        for (int64_t e = base + threadIdx.x; e < min(n, base + seg); e += 256) c_indices[lo + e] = src[e];
}

}  // namespace b200
