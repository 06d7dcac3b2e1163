// Top-k_out selection of materialised fp32 score rows for large k (paths 2 and 3 with k_out > 1024, k = None): a constant
// number of reads of each score row plus one sort of the k_out survivors, where the streaming passes of
// scores_topk_kernel (sparse.cuh) read every row ceil(k_out / 32) times.  Results are bit-identical to those passes:
// order (score desc, object id asc), only scores > -inf kept (-inf and NaN never rank, a real -FLT_MAX does), objects
// listed in the row's filter_pairs_csr slice never returned, ids LOCAL (the caller adds the id offset), unfilled slots
// -1 / -FLT_MAX and out_counts = min(k_out, kept scores).
//
//  1. filter_mask_kernel: one warp per row writes -inf over the row's filtered positions.
//  2. large_k_select_kernel, one CTA per row:
//     a. radix select on order_key (order_key.h), MSD 8-bit digits with shared-memory histograms, at most 4 reads of the
//        row, stopping once the bucket holding the k_out-th key is taken whole: the selected keys are those whose resolved
//        high bits are above the bucket's (n_gt of them) plus the first `take` in position order of those inside it;
//     b. stable compaction of the survivors in position order (block-wide scans; a fifth read of the row at most);
//     c. stable LSD radix sort of the survivors by key, descending: in shared memory up to LK_SMEM_PAIRS survivors,
//        above that in global scratch (4 x k_out words per row), still one CTA per row.  Position order is id order (the
//        whitelist is sorted, the id offset constant), so stability gives id ascending among equal scores;
//     d. write-out of ids (pos2obj) and the rows' own score bits, padding and the count.
#pragma once
#include "common.cuh"
#include "order_key.h"
#include "sizes.h"

namespace b200 {

constexpr int LK_THREADS = 1024;
constexpr int LK_WARPS = LK_THREADS / 32;
constexpr int LK_ITEMS = 4;  // consecutive positions per thread of a compaction tile
constexpr size_t lk_smem_bytes(int k_out) { return (size_t)16 * (size_t)(k_out < LK_SMEM_PAIRS ? k_out : LK_SMEM_PAIRS); }

// One warp per score row: -inf at every position whose object the row's filter slice lists.  Filter ids are global:
// local = id - id_off; ids outside [0, n_obj) (or not in the whitelist) match no position and are ignored.
__global__ void __launch_bounds__(256) filter_mask_kernel(float* __restrict__ scores, const int32_t* __restrict__ rows, int64_t n_rows,
                                                          int64_t n_pos, const int32_t* __restrict__ pos2obj,
                                                          const int64_t* __restrict__ f_indptr, const int32_t* __restrict__ f_indices,
                                                          int32_t id_off) {
    const int lane = threadIdx.x & 31;
    const int64_t sr = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (sr >= n_rows) return;
    const int64_t row = rows ? (int64_t)rows[sr] : sr;
    const int64_t hi = f_indptr[row + 1];
    float* srow = scores + sr * n_pos;
    for (int64_t e = f_indptr[row] + lane; e < hi; e += 32) {
        const int64_t local = (int64_t)__ldg(f_indices + e) - id_off;
        if (local < 0) continue;
        int64_t pos = -1;
        if (pos2obj) {  // sorted unique whitelist: lower_bound
            int64_t lo = 0, up = n_pos;
            while (lo < up) {
                const int64_t mid = (lo + up) >> 1;
                if ((int64_t)__ldg(pos2obj + mid) < local)
                    lo = mid + 1;
                else
                    up = mid;
            }
            if (lo < n_pos && (int64_t)__ldg(pos2obj + lo) == local) pos = lo;
        } else if (local < n_pos) {
            pos = local;
        }
        if (pos >= 0) srow[pos] = -INFINITY;
    }
}

struct LargeKParams {
    const float* scores;   // [n_rows, n_pos] score rows, filter already masked
    const int32_t* rows;   // nullable: score row r belongs to logical row rows[r] (outputs)
    int64_t n_rows = 0, n_pos = 0;
    const int32_t* pos2obj;  // whitelist (local ids) or nullptr
    int32_t k_out = 0;
    int32_t smem_pairs = 0;  // survivors the dynamic shared buffer holds: min(k_out, LK_SMEM_PAIRS)
    uint32_t* scratch;       // [n_rows][4][k_out] words; used by rows with more than smem_pairs survivors
    int32_t* out_ids;
    float* out_scores;
    int32_t* out_counts;
};

// hist[digit] += 1 for every active lane, one shared atomic per distinct digit of the warp: tie blocks would otherwise
// serialise 32 lanes on one bin.  Every lane of the warp calls it.
__device__ __forceinline__ void lk_hist_add(uint32_t* hist, uint32_t digit, bool active) {
    const unsigned act = __ballot_sync(B200_FULL_MASK, active);
    if (!active) return;
    const unsigned peers = __match_any_sync(act, digit);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(hist + digit, (uint32_t)__popc(peers));
}

// Warp 0: the bin holding the need-th largest counted key, scanning bins from 255 down.  out = {bin, keys in higher
// bins, keys in the bin, all counted keys}; the first three only when need <= all counted keys.
__device__ __forceinline__ void lk_find_bin(const uint32_t* hist, uint32_t need, uint32_t* out) {
    const int lane = threadIdx.x & 31;
    uint32_t h[8], sum = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        h[j] = hist[255 - 8 * lane - j];
        sum += h[j];
    }
    uint32_t incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(B200_FULL_MASK, incl, o);
        if (lane >= o) incl += t;
    }
    uint32_t cum = incl - sum;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (cum < need && need <= cum + h[j]) {
            out[0] = 255 - 8 * lane - j;
            out[1] = cum;
            out[2] = h[j];
        }
        cum += h[j];
    }
    if (lane == 31) out[3] = incl;
}

// Exclusive block-wide sum (LK_THREADS threads); `total` = the sum over the block.
__device__ __forceinline__ uint32_t lk_block_scan(uint32_t v, uint32_t* s_warp, uint32_t& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(B200_FULL_MASK, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = s_warp[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(B200_FULL_MASK, w, o);
            if (lane >= o) w += t;
        }
        s_warp[lane] = w;
    }
    __syncthreads();
    const uint32_t excl = incl - v + (warp ? s_warp[warp - 1] : 0u);
    total = s_warp[LK_WARPS - 1];
    __syncthreads();
    return excl;
}

// Stable LSD radix sort of n (key, position) pairs by key, descending, 8-bit digits; (ka, pa) holds the input and
// (kb, pb) is the other buffer, in shared or global memory.  A digit every key shares moves nothing and is skipped.
// Returns true when the result is in (kb, pb).
__device__ bool lk_sort_desc(uint32_t* ka, uint32_t* pa, uint32_t* kb, uint32_t* pb, uint32_t n, uint32_t* hist,
                             uint32_t (*wcnt)[256]) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    bool in_b = false;
    for (int shift = 0; shift < 32; shift += 8) {
        const uint32_t* sk = in_b ? kb : ka;
        const uint32_t* sp = in_b ? pb : pa;
        uint32_t* dk = in_b ? ka : kb;
        uint32_t* dp = in_b ? pa : pb;
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
        for (uint32_t b = 0; b < n; b += LK_THREADS) {
            const uint32_t i = b + tid;
            const bool v = i < n;
            lk_hist_add(hist, v ? (~sk[i] >> shift) & 255u : 0u, v);
        }
        __syncthreads();
        if (__syncthreads_or(tid < 256 && hist[tid] == n)) continue;
        if (warp == 0) {  // exclusive scan over the bins (ascending digit of ~key: descending key)
            uint32_t h[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                h[j] = hist[8 * lane + j];
                sum += h[j];
            }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(B200_FULL_MASK, incl, o);
                if (lane >= o) incl += t;
            }
            uint32_t run = incl - sum;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                hist[8 * lane + j] = run;
                run += h[j];
            }
        }
        for (uint32_t b = 0; b < n; b += LK_THREADS) {
            for (int e = tid; e < LK_WARPS * 256; e += LK_THREADS) (&wcnt[0][0])[e] = 0;
            __syncthreads();
            const uint32_t i = b + tid;
            const bool v = i < n;
            const uint32_t key = v ? sk[i] : 0u, pos = v ? sp[i] : 0u;
            const uint32_t dg = v ? (~key >> shift) & 255u : 256u;
            const unsigned peers = __match_any_sync(B200_FULL_MASK, dg);
            const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
            if (v && rank == 0) wcnt[warp][dg] = __popc(peers);
            __syncthreads();
            if (tid < 256) {  // this tile's start of digit `tid` for every warp, in warp order
                uint32_t r = hist[tid];
                for (int w = 0; w < LK_WARPS; ++w) {
                    const uint32_t c = wcnt[w][tid];
                    wcnt[w][tid] = r;
                    r += c;
                }
                hist[tid] = r;
            }
            __syncthreads();
            if (v) {
                const uint32_t dst = wcnt[warp][dg] + rank;
                dk[dst] = key;
                dp[dst] = pos;
            }
            __syncthreads();
        }
        in_b = !in_b;
    }
    return in_b;
}

// One CTA per score row; dynamic shared memory lk_smem_bytes(k_out).
__global__ void __launch_bounds__(LK_THREADS) large_k_select_kernel(const LargeKParams p) {
    extern __shared__ uint32_t lk_smem[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t wcnt[LK_WARPS][256];
    __shared__ uint32_t s_warp[LK_WARPS];
    __shared__ uint32_t s_bin[4];
    const int tid = threadIdx.x;
    const int64_t sr = blockIdx.x;
    const int64_t row = p.rows ? (int64_t)p.rows[sr] : sr;
    const int64_t n_pos = p.n_pos;
    const float* srow = p.scores + sr * n_pos;
    constexpr int64_t TILE = (int64_t)LK_THREADS * LK_ITEMS;

    // a. the selected keys: (key & mask) > prefix, or (key & mask) == prefix among the first `need` in position order
    uint32_t mask = 0, prefix = 0, need = (uint32_t)p.k_out, n_gt = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        if (tid < 256) hist[tid] = 0;
        __syncthreads();
        for (int64_t base = 0; base < n_pos; base += TILE) {
#pragma unroll
            for (int j = 0; j < LK_ITEMS; ++j) {
                const int64_t pos = base + (int64_t)j * LK_THREADS + tid;
                const uint32_t key = pos < n_pos ? order_key(__ldg(srow + pos)) : ORDER_KEY_INVALID;
                lk_hist_add(hist, (key >> shift) & 255u, key != ORDER_KEY_INVALID && (key & mask) == prefix);
            }
        }
        __syncthreads();
        if (tid < 32) lk_find_bin(hist, need, s_bin);
        __syncthreads();
        if (shift == 24 && s_bin[3] <= need) {  // at most k_out kept scores: all of them
            need = s_bin[3];
            break;
        }
        const uint32_t b = s_bin[0], above = s_bin[1], in_bin = s_bin[2];
        n_gt += above;
        need -= above;
        prefix |= b << shift;
        mask |= 255u << shift;
        __syncthreads();
        if (in_bin == need) break;  // the bucket is taken whole
    }
    const uint32_t take = need, m = n_gt + take;

    // b. survivors (key, position) in position order
    const int64_t k_out = p.k_out;
    uint32_t *ka, *pa, *kb, *pb;
    if (m <= (uint32_t)p.smem_pairs) {
        ka = lk_smem;
        pa = ka + p.smem_pairs;
        kb = pa + p.smem_pairs;
        pb = kb + p.smem_pairs;
    } else {
        ka = p.scratch + sr * 4 * k_out;
        pa = ka + k_out;
        kb = pa + k_out;
        pb = kb + k_out;
    }
    uint32_t gt_base = 0, eq_base = 0;
    for (int64_t base = 0; base < n_pos && gt_base + min(eq_base, take) < m; base += TILE) {
        const int64_t p0 = base + (int64_t)tid * LK_ITEMS;
        uint32_t keys[LK_ITEMS];
        uint32_t cnt = 0;  // (above << 16) | inside: at most TILE = 4096 each per tile
#pragma unroll
        for (int j = 0; j < LK_ITEMS; ++j) {
            keys[j] = p0 + j < n_pos ? order_key(__ldg(srow + p0 + j)) : ORDER_KEY_INVALID;
            const uint32_t kk = keys[j] & mask;
            if (keys[j] != ORDER_KEY_INVALID) cnt += kk > prefix ? (1u << 16) : kk == prefix ? 1u : 0u;
        }
        uint32_t total;
        const uint32_t excl = lk_block_scan(cnt, s_warp, total);
        uint32_t gt_before = gt_base + (excl >> 16), eq_before = eq_base + (excl & 0xFFFFu);
#pragma unroll
        for (int j = 0; j < LK_ITEMS; ++j) {
            if (keys[j] == ORDER_KEY_INVALID) continue;
            const uint32_t kk = keys[j] & mask;
            if (kk > prefix) {
                const uint32_t dst = gt_before + min(eq_before, take);
                ka[dst] = keys[j];
                pa[dst] = (uint32_t)(p0 + j);
                ++gt_before;
            } else if (kk == prefix) {
                if (eq_before < take) {
                    const uint32_t dst = gt_before + eq_before;
                    ka[dst] = keys[j];
                    pa[dst] = (uint32_t)(p0 + j);
                }
                ++eq_before;
            }
        }
        gt_base += total >> 16;
        eq_base += total & 0xFFFFu;
    }
    __syncthreads();

    // c. stable sort by key, descending
    const uint32_t* fp = lk_sort_desc(ka, pa, kb, pb, m, hist, wcnt) ? pb : pa;

    // d. write-out
    int32_t* oi = p.out_ids + row * k_out;
    float* os = p.out_scores + row * k_out;
    for (int64_t i = tid; i < k_out; i += LK_THREADS) {
        int32_t id = -1;
        float s = -FLT_MAX;
        if (i < (int64_t)m) {
            const uint32_t pos = fp[i];
            id = p.pos2obj ? __ldg(p.pos2obj + pos) : (int32_t)pos;
            s = __ldg(srow + pos);
        }
        oi[i] = id;
        os[i] = s;
    }
    if (tid == 0) p.out_counts[row] = (int32_t)m;
}

}  // namespace b200
