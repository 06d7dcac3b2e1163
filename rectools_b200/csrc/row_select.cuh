// Top-k_out selection of rows the engine already holds (path 4, b200_rank_query.object_rows): batch row r is scored as
// score(r, j) = obj[object_rows[r], j], the master row itself, widened to fp32 when it is kept at 16 bits (EASE item-to-item: row t of the weight matrix is
// target t's score row).  One CTA per row reads the stored row where it lies and writes nothing into it, so the filter is
// applied on the fly instead of by filter_mask_kernel.  Otherwise this is large_k_select_kernel (large_k_select.cuh) with
// a different row source, built from the same pieces: radix select on order_key, stable compaction of the survivors in
// position order, stable LSD sort by key descending, write-out -- so the results are bit-identical to it and to the
// streaming passes of paths 2 and 3: order (score desc, object id asc), -inf and NaN never returned, +-0 equal keys,
// filtered objects never returned, unfilled slots -1 / -FLT_MAX, out_counts = min(k_out, kept scores).  One launch for
// every k_out, k <= 1024 included.
//
// The filter of row r is its sorted slice of filter_pairs_csr (global object ids; the engine refuses an id offset, so
// they are object ids of this engine):
//  - histograms: after each pass over the row, every listed object that is a position of the call (ids outside
//    [0, n_obj) or outside the whitelist match nothing; repeated ids count once) takes its key's digit back out, so the
//    bucket search sees only the kept scores;
//  - compaction: a position whose key could survive is looked up in the slice (binary search); only those pay.
#pragma once
#include "large_k_select.cuh"

namespace b200 {

struct RowSelectParams {
    const void* objects;        // [n_obj, d] stored objects in the kernel's type TO (fp32, fp16 or bf16), d == n_obj
    int64_t n_obj = 0, d = 0;
    const int64_t* object_rows;  // [n_rows] stored row of each batch row (in range: checked on the host for host inputs)
    int64_t n_rows = 0, n_pos = 0;
    const int32_t* pos2obj;       // whitelist or nullptr
    const int64_t* f_indptr;      // [n_rows + 1] (batch rows) or nullptr
    const int32_t* f_indices;
    int32_t k_out = 0;
    int32_t smem_pairs = 0;  // min(k_out, LK_SMEM_PAIRS)
    uint32_t* scratch;       // [n_rows][4][k_out] words; used by rows with more than smem_pairs survivors
    int32_t* out_ids;
    float* out_scores;
    int32_t* out_counts;
};

// Position of object `id` among the call's positions, or -1.
__device__ __forceinline__ int64_t rs_position(int64_t id, int64_t n_obj, const int32_t* __restrict__ pos2obj, int64_t n_pos) {
    if (id < 0 || id >= n_obj) return -1;
    if (!pos2obj) return id;
    int64_t lo = 0, up = n_pos;
    while (lo < up) {
        const int64_t mid = (lo + up) >> 1;
        if ((int64_t)__ldg(pos2obj + mid) < id)
            lo = mid + 1;
        else
            up = mid;
    }
    return lo < n_pos && (int64_t)__ldg(pos2obj + lo) == id ? lo : -1;
}

// Is object `id` in the sorted slice [lo, hi)?
__device__ __forceinline__ bool rs_listed(const int32_t* __restrict__ f, int64_t lo, const int64_t end, int32_t id) {
    int64_t up = end;
    while (lo < up) {
        const int64_t mid = (lo + up) >> 1;
        if (__ldg(f + mid) < id)
            lo = mid + 1;
        else
            up = mid;
    }
    return lo < end && __ldg(f + lo) == id;
}

// One CTA per batch row; dynamic shared memory lk_smem_bytes(k_out).  A 16-bit stored row is widened to fp32 before the
// order key is taken, so its keys and returned scores are those of its widened fp32 copy.
template <typename TO>
__global__ void __launch_bounds__(LK_THREADS) row_select_kernel(const RowSelectParams p) {
    extern __shared__ uint32_t lk_smem[];
    __shared__ uint32_t hist[256];
    __shared__ uint32_t wcnt[LK_WARPS][256];
    __shared__ uint32_t s_warp[LK_WARPS];
    __shared__ uint32_t s_bin[4];
    const int tid = threadIdx.x;
    const int64_t r = blockIdx.x;
    const int64_t n_pos = p.n_pos;
    const TO* srow = static_cast<const TO*>(p.objects) + __ldg(p.object_rows + r) * p.d;
    const int32_t* wl = p.pos2obj;
    auto score = [&](int64_t pos) { return to_f32(__ldg(srow + (wl ? (int64_t)__ldg(wl + pos) : pos))); };
    const int64_t f_lo = p.f_indptr ? __ldg(p.f_indptr + r) : 0, f_hi = p.f_indptr ? __ldg(p.f_indptr + r + 1) : 0;
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
                const uint32_t key = pos < n_pos ? order_key(score(pos)) : ORDER_KEY_INVALID;
                lk_hist_add(hist, (key >> shift) & 255u, key != ORDER_KEY_INVALID && (key & mask) == prefix);
            }
        }
        __syncthreads();
        // the filtered positions leave the histogram (each counted once above when its key is kept and matches)
        for (int64_t e = f_lo + tid; e < f_hi; e += LK_THREADS) {
            const int32_t id = __ldg(p.f_indices + e);
            if (e > f_lo && __ldg(p.f_indices + e - 1) == id) continue;  // a repeated id: its first entry stands for it
            const int64_t pos = rs_position(id, p.n_obj, wl, n_pos);
            if (pos < 0) continue;
            const uint32_t key = order_key(score(pos));
            if (key != ORDER_KEY_INVALID && (key & mask) == prefix) atomicSub(hist + ((key >> shift) & 255u), 1u);
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

    // b. survivors (key, position) in position order; a filtered position is no key at all
    const int64_t k_out = p.k_out;
    uint32_t *ka, *pa, *kb, *pb;
    if (m <= (uint32_t)p.smem_pairs) {
        ka = lk_smem;
        pa = ka + p.smem_pairs;
        kb = pa + p.smem_pairs;
        pb = kb + p.smem_pairs;
    } else {
        ka = p.scratch + r * 4 * k_out;
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
            keys[j] = p0 + j < n_pos ? order_key(score(p0 + j)) : ORDER_KEY_INVALID;
            if (keys[j] != ORDER_KEY_INVALID && (keys[j] & mask) >= prefix && f_lo < f_hi &&
                rs_listed(p.f_indices, f_lo, f_hi, wl ? __ldg(wl + p0 + j) : (int32_t)(p0 + j)))
                keys[j] = ORDER_KEY_INVALID;
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

    // d. write-out: ids through the whitelist, the stored row's own score bits
    int32_t* oi = p.out_ids + r * k_out;
    float* os = p.out_scores + r * k_out;
    for (int64_t i = tid; i < k_out; i += LK_THREADS) {
        int32_t id = -1;
        float s = -FLT_MAX;
        if (i < (int64_t)m) {
            const uint32_t pos = fp[i];
            id = wl ? __ldg(wl + pos) : (int32_t)pos;
            s = score(pos);
        }
        oi[i] = id;
        os[i] = s;
    }
    if (tid == 0) p.out_counts[r] = (int32_t)m;
}

}  // namespace b200
