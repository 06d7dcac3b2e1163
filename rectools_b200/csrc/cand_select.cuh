// Path 5, candidate sets (b200_rank_topk_candidates): batch row r is ranked against its own object ids
// c_indices[c_indptr[r] .. c_indptr[r+1]), strictly ascending, minus the ids its filter_pairs_csr slice lists.
//
//  1. cand_score_kernel<TO>: one CTA per row (and row segment) stages the subject row in shared memory, as the re-score
//     does, and every thread scores candidates with exact_score<TO> -- the result definition itself, so a pair's score
//     bits are those of path 1's re-score.  A candidate the row's sorted filter slice lists (binary search) gets NaN, whose
//     order key is never kept.  The scores form one ragged fp32 buffer addressed by the chunk-rebased c_indptr.
//  2. cand_select_kernel: large_k_select_kernel (large_k_select.cuh) over that ragged row, built from the same pieces:
//     radix select on order_key, stable compaction in position order, stable LSD sort by key descending, write-out.
//     Positions are in id order (the lists are ascending), so stability orders equal scores by id: (score desc, id asc),
//     -inf and NaN never returned, +-0 equal keys, unfilled slots -1 / -FLT_MAX, out_counts = min(k_out, kept scores).
//     Position -> id goes through the row's own candidate ids.  One launch per row chunk for every k_out.
// These kernels stand beside those of paths 1-4 and share no template with them, so their code is left as it was.
#pragma once
#include "large_k_select.cuh"
#include "row_select.cuh"
#include "select.cuh"

namespace b200 {

constexpr int CS_THREADS = 256;  // threads of cand_score_kernel
constexpr int CS_SEG = CS_THREADS * 4;  // candidates one CTA of cand_score_kernel takes per row segment

struct CandParams {
    SelectParams sp;           // exact_score's inputs: objects, d, obj_norms (COSINE) -- nothing else is read
    const float* subjects;     // subject row of batch row r: subjects + (row_map ? row_map[r] : r) * d
    const int64_t* row_map;    // nullable
    const int64_t* c_indptr;   // [n_rows + 1], c_indptr[0] == 0: row r's candidates and scores
    const int32_t* c_indices;  // object ids, strictly ascending within a row
    const int64_t* f_indptr;   // [n_rows + 1] or nullptr: the filter slice of row r in f_indices
    const int32_t* f_indices;
    float* scores;             // [c_indptr[n_rows]]
    int64_t n_rows = 0;
    int32_t k_out = 0;
    int32_t smem_pairs = 0;    // min(k_out, LK_SMEM_PAIRS)
    uint32_t* scratch;         // [4 * c_indptr[n_rows]] words: row r sorts at 4 * c_indptr[r], when it keeps > smem_pairs
    int32_t* out_ids;          // [n_rows, k_out]
    float* out_scores;
    int32_t* out_counts;
};

// grid (n_rows, segments), CS_THREADS threads, dynamic shared memory d floats.
template <typename TO>
__global__ void __launch_bounds__(CS_THREADS) cand_score_kernel(const CandParams p) {
    extern __shared__ __align__(16) float cs_sub[];
    const int64_t r = blockIdx.x;
    const int64_t lo = __ldg(p.c_indptr + r), hi = __ldg(p.c_indptr + r + 1);
    const int64_t first = lo + (int64_t)blockIdx.y * CS_SEG;
    if (first >= hi) return;  // the whole CTA: the row has no candidate in this segment
    const int d = p.sp.d;
    const int64_t sr = p.row_map ? __ldg(p.row_map + r) : r;
    for (int j = threadIdx.x; j < d; j += CS_THREADS) cs_sub[j] = __ldg(p.subjects + sr * d + j);
    __syncthreads();
    const int64_t f_lo = p.f_indptr ? __ldg(p.f_indptr + r) : 0, f_hi = p.f_indptr ? __ldg(p.f_indptr + r + 1) : 0;
    const int64_t stride = (int64_t)gridDim.y * CS_SEG;
    for (int64_t base = first; base < hi; base += stride) {
        for (int64_t e = base + threadIdx.x; e < min(hi, base + CS_SEG); e += CS_THREADS) {
            const int32_t id = __ldg(p.c_indices + e);
            const bool filtered = f_lo < f_hi && rs_listed(p.f_indices, f_lo, f_hi, id);
            p.scores[e] = filtered ? __int_as_float(0x7fc00000) : exact_score<TO>(p.sp, cs_sub, id);
        }
    }
}

// One CTA per batch row; dynamic shared memory lk_smem_bytes(k_out).
__global__ void __launch_bounds__(LK_THREADS) cand_select_kernel(const CandParams p) {
    extern __shared__ uint32_t lk_smem[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t wcnt[LK_WARPS][256];
    __shared__ uint32_t s_warp[LK_WARPS];
    __shared__ uint32_t s_bin[4];
    const int tid = threadIdx.x;
    const int64_t r = blockIdx.x;
    const int64_t off = __ldg(p.c_indptr + r);
    const int64_t n_pos = __ldg(p.c_indptr + r + 1) - off;
    const float* srow = p.scores + off;
    const int32_t* ids = p.c_indices + off;
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

    // b. survivors (key, position) in position order; a row keeps at most n_pos of them
    uint32_t *ka, *pa, *kb, *pb;
    if (m <= (uint32_t)p.smem_pairs) {
        ka = lk_smem;
        pa = ka + p.smem_pairs;
        kb = pa + p.smem_pairs;
        pb = kb + p.smem_pairs;
    } else {
        ka = p.scratch + 4 * off;
        pa = ka + n_pos;
        kb = pa + n_pos;
        pb = kb + n_pos;
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

    // d. write-out: ids through the row's candidate list, the scores' own bits
    const int64_t k_out = p.k_out;
    int32_t* oi = p.out_ids + r * k_out;
    float* os = p.out_scores + r * k_out;
    for (int64_t i = tid; i < k_out; i += LK_THREADS) {
        int32_t id = -1;
        float s = -FLT_MAX;
        if (i < (int64_t)m) {
            const uint32_t pos = fp[i];
            id = __ldg(ids + pos);
            s = __ldg(srow + pos);
        }
        oi[i] = id;
        os[i] = s;
    }
    if (tid == 0) p.out_counts[r] = (int32_t)m;
}

}  // namespace b200
