// Path 9 kernels (knn.cu): the ItemKNN score of every touched item of a user row, summed in the row's entry order, and
// its candidates handed to path 6's segmented selection as (row, fp64 score) pairs in ascending item id.
//
// Row u has entries (j_e, w_e) in CSR order; item i's score is s_u(i) = (((0 + p_1) + p_2) + ...) over the entries whose
// S row holds i, p = fl64(S[j_e, i] * (double)w_e): a rounded product, then a rounded add, never a fused multiply-add.
// One CTA walks the entries in order with a barrier between two of them; its threads cover the entries of S[j_e], and an
// item occurs once per S row, so no two threads add to one item between two barriers.
#pragma once
#include <cuda_runtime.h>

#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

#include <cstdint>

namespace b200 {

constexpr int KNN_THREADS = 256;
constexpr int KNN_ITEMS = 16;                          // table slots per thread
constexpr int KNN_TABLE = KNN_THREADS * KNN_ITEMS;     // 4096: KNN_TABLE_BOUND (knn_plan.h) fills it to 3/4 at most

struct KnnRows {
    int64_t n_items;
    const int64_t* s_indptr;
    const int32_t* s_indices;
    const double* s_data;
    const int64_t* u_indptr;  // the chunk's rows, rebased: entries u_indptr[r] - u_base ...
    int64_t u_base;
    const int32_t* u_indices;
    const float* u_data;
    const int64_t* f_indptr;  // nullable
    int64_t f_base;
    const int32_t* f_indices;
    const int32_t* whitelist;  // nullable
    int64_t n_whitelist;
    const int64_t* slot;       // the chunk's slot offsets, rebased to 0
    int64_t* pair_code;        // [slots]: the row, or -1 (pre-set) for an unused slot
    double* pair_score;
    int32_t* pair_id;
};

__device__ __forceinline__ bool knn_sorted_has(const int32_t* a, int64_t n, int32_t x) {
    int64_t lo = 0, hi = n;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && a[lo] == x;
}

// Whether item i is a candidate of row r: not in the row's filter slice, and in the whitelist when there is one.
__device__ __forceinline__ bool knn_keep(const KnnRows& a, int64_t r, int32_t i) {
    if (a.f_indptr) {
        const int64_t f0 = a.f_indptr[r] - a.f_base;
        if (knn_sorted_has(a.f_indices + f0, a.f_indptr[r + 1] - a.f_indptr[r], i)) return false;
    }
    return !a.whitelist || knn_sorted_has(a.whitelist, a.n_whitelist, i);
}

// The entry loop of row r: add(i, p) for every item of S[j_e], entry by entry, with a barrier after each.
template <class Add>
__device__ __forceinline__ void knn_walk(const KnnRows& a, int64_t r, Add add) {
    const int64_t e0 = a.u_indptr[r] - a.u_base, e1 = a.u_indptr[r + 1] - a.u_base;
    for (int64_t e = e0; e < e1; ++e) {
        const int32_t j = a.u_indices[e];
        const double w = (double)a.u_data[e];
        const int64_t s0 = a.s_indptr[j], s1 = a.s_indptr[j + 1];
        for (int64_t t = s0 + threadIdx.x; t < s1; t += blockDim.x) add(a.s_indices[t], __dmul_rn(a.s_data[t], w));
        __syncthreads();
    }
}

union KnnTableSmem {
    struct {
        int32_t key[KNN_TABLE];
        double val[KNN_TABLE];
    } table;
    typename cub::BlockRadixSort<int32_t, KNN_THREADS, KNN_ITEMS, double>::TempStorage sort;
    typename cub::BlockScan<int32_t, KNN_THREADS>::TempStorage scan;
};

// One CTA per listed row whose bound fits the table: open addressing (linear probing, keys claimed with atomicCAS,
// empty = n_items), then the table sorted by item id and the candidates written in that order.
__global__ void __launch_bounds__(KNN_THREADS) knn_table_kernel(KnnRows a, const int32_t* __restrict__ rows, int key_bits) {
    extern __shared__ __align__(16) unsigned char knn_smem[];
    KnnTableSmem& sm = *reinterpret_cast<KnnTableSmem*>(knn_smem);
    const int64_t r = rows[blockIdx.x];
    const int32_t empty = (int32_t)a.n_items;
    for (int s = threadIdx.x; s < KNN_TABLE; s += KNN_THREADS) {
        sm.table.key[s] = empty;
        sm.table.val[s] = 0.0;
    }
    __syncthreads();
    knn_walk(a, r, [&](int32_t i, double p) {
        uint32_t s = ((uint32_t)i * 2654435761u) & (KNN_TABLE - 1);
        for (;;) {
            const int32_t old = atomicCAS(&sm.table.key[s], empty, i);
            if (old == empty || old == i) break;
            s = (s + 1) & (KNN_TABLE - 1);
        }
        sm.table.val[s] = __dadd_rn(sm.table.val[s], p);
    });
    int32_t key[KNN_ITEMS];
    double val[KNN_ITEMS];
#pragma unroll
    for (int q = 0; q < KNN_ITEMS; ++q) {
        key[q] = sm.table.key[threadIdx.x * KNN_ITEMS + q];
        val[q] = sm.table.val[threadIdx.x * KNN_ITEMS + q];
    }
    __syncthreads();
    cub::BlockRadixSort<int32_t, KNN_THREADS, KNN_ITEMS, double>(sm.sort).Sort(key, val, 0, key_bits);
    int32_t keep[KNN_ITEMS], n_keep = 0;
#pragma unroll
    for (int q = 0; q < KNN_ITEMS; ++q) {
        keep[q] = key[q] != empty && knn_keep(a, r, key[q]);
        n_keep += keep[q];
    }
    __syncthreads();
    int32_t at = 0;
    cub::BlockScan<int32_t, KNN_THREADS>(sm.scan).ExclusiveSum(n_keep, at);
    const int64_t base = a.slot[r];
#pragma unroll
    for (int q = 0; q < KNN_ITEMS; ++q)
        if (keep[q]) {
            a.pair_code[base + at] = r;
            a.pair_score[base + at] = val[q];
            a.pair_id[base + at] = key[q];
            ++at;
        }
}

// The rows above the table's bound: CTA b takes rows[b], rows[b + gridDim.x], ..., each in its own dense fp64 row of
// n_items (acc) with a touched flag per item (touched, zero on entry and left zero), then writes the candidates in one
// ascending sweep over the items.
__global__ void __launch_bounds__(KNN_THREADS) knn_dense_kernel(KnnRows a, const int32_t* __restrict__ rows, int64_t n_rows,
                                                                double* __restrict__ acc_all, uint8_t* __restrict__ touched_all) {
    __shared__ typename cub::BlockScan<int32_t, KNN_THREADS>::TempStorage scan;
    __shared__ int32_t carry;
    double* acc = acc_all + (int64_t)blockIdx.x * a.n_items;
    uint8_t* touched = touched_all + (int64_t)blockIdx.x * a.n_items;
    for (int64_t q = blockIdx.x; q < n_rows; q += gridDim.x) {
        const int64_t r = rows[q];
        knn_walk(a, r, [&](int32_t i, double p) {
            acc[i] = __dadd_rn(touched[i] ? acc[i] : 0.0, p);
            touched[i] = 1;
        });
        if (threadIdx.x == 0) carry = 0;
        __syncthreads();
        const int64_t base = a.slot[r];
        for (int64_t i0 = 0; i0 < a.n_items; i0 += KNN_THREADS) {
            const int64_t i = i0 + threadIdx.x;
            int32_t keep = 0;
            if (i < a.n_items && touched[i]) {
                touched[i] = 0;
                keep = knn_keep(a, r, (int32_t)i);
            }
            int32_t at = 0, total = 0;
            cub::BlockScan<int32_t, KNN_THREADS>(scan).ExclusiveSum(keep, at, total);
            if (keep) {
                a.pair_code[base + carry + at] = r;
                a.pair_score[base + carry + at] = acc[i];
                a.pair_id[base + carry + at] = (int32_t)i;
            }
            __syncthreads();
            if (threadIdx.x == 0) carry += total;
            __syncthreads();
        }
    }
}

// Path 6's positions back to ids and scores: row r's kept positions pos[off[r] .. off[r+1]) fill out_ids / out_scores
// [r, 0 .. k), unfilled slots id -1 and score 0; out_counts[r] the kept count.
__global__ void __launch_bounds__(256) knn_gather_kernel(int64_t n_rows, int32_t k, const int64_t* __restrict__ off,
                                                         const int64_t* __restrict__ pos, const int32_t* __restrict__ pair_id,
                                                         const double* __restrict__ pair_score, int32_t* __restrict__ out_ids,
                                                         double* __restrict__ out_scores, int32_t* __restrict__ out_counts) {
    const int64_t total = n_rows * (int64_t)k;
    for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = t / k, c = t % k, n = off[r + 1] - off[r];
        if (c < n) {
            const int64_t p = pos[off[r] + c];
            out_ids[t] = pair_id[p];
            out_scores[t] = pair_score[p];
        } else {
            out_ids[t] = -1;
            out_scores[t] = 0.0;
        }
        if (c == 0) out_counts[r] = (int32_t)n;
    }
}

}  // namespace b200
