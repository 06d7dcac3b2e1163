// Path 8 (b200_rank_topk_list_mix): per-category ordered lists, each minus a row's viewed ids, mixed into one list per
// row -- the per-user step of `PopularInCategoryModel._recommend_u2i` (rectools/models/popular_in_category.py:289-373).
// Kernel of list_mix.cu; nothing else includes this header.
//
// One CTA per row, in one pass:
//   1. a warp per category takes the category's first k unviewed positions within path 7's window (list_select.cuh),
//      entry (c, j) of rank j going to slot slots[c] + j, so slot order is (category asc, rank asc);
//   2. the entries are sorted on (id, fallback flag, slot): the first of each id in the sequence "main entries (rank <
//      quota[c]) in (c, j) order, then fallback entries in (c, j) order" survives -- the reference's drop_duplicates;
//   3. when main and fallback survivors exceed k, the fallback survivors are sorted on (rank, category) and the first
//      k - #main are kept (the main ones always are: at most sum(quota) <= k of them);
//   4. a warp per category numbers its kept entries r' in rank order, and each kept entry writes itself to its output
//      slot: group = (c, j) order, rotate = (r', c) order.
// The sorts are bitonic over the row's scratch (list_mix_plan.h: mix_row_scratch), which is dynamic shared memory when it
// fits, or a global slice per row of the chunk otherwise (SMEM = false); the code is the same.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "../../include/b200_rank.h"
#include "common.cuh"

namespace b200 {

constexpr int MIX_THREADS = 256;

struct MixRows {
    const int32_t* list;     // [n_total] ids of every list, concatenated in priority order
    const int64_t* offsets;  // [n_lists + 1] list c = list[offsets[c] .. offsets[c + 1])
    const int64_t* slots;    // [n_lists + 1] entry slots of list c = [slots[c], slots[c + 1]), min(k, n_c) of them
    const int32_t* quota;    // [n_lists]
    int32_t n_lists;
    int32_t mixing;          // B200_MIX_ROTATE / B200_MIX_GROUP
    const int64_t* indptr;   // [n_rows + 1] row pointers of this chunk, absolute (minus `base`); NULL: nothing viewed
    int64_t base;
    const int32_t* indices;  // the chunk's viewed ids, sorted ascending within a row
    int64_t n_rows;
    int k;
    int k_out;
    int64_t n_slots;         // slots[n_lists]
    int64_t keys_cap;        // next_pow2(n_slots): the sort keys of a row
    unsigned char* scratch;  // SMEM = false: row r's scratch at scratch + r * row_scratch
    int64_t row_scratch;
    int32_t* out_pos;        // [n_rows, k_out]
    int32_t* out_counts;     // [n_rows]
};

// Ascending bitonic sort of keys[0, n) by the whole CTA, padded with ~0 up to a power of two (keys has room for it).
// Every key sorted here is below ~0.  Ends with a barrier.
__device__ __forceinline__ void mix_block_sort(uint64_t* keys, int n) {
    int P = 1;
    while (P < n) P <<= 1;
    for (int i = n + threadIdx.x; i < P; i += MIX_THREADS) keys[i] = ~0ull;
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = threadIdx.x; i < (P >> 1); i += MIX_THREADS) {
                const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                const uint64_t x = keys[lo], y = keys[hi];
                if ((x > y) == ((lo & size) == 0)) {
                    keys[lo] = y;
                    keys[hi] = x;
                }
            }
            __syncthreads();
        }
    }
}

template <bool SMEM>
__global__ void __launch_bounds__(MIX_THREADS, 1) list_mix_kernel(MixRows a) {
    extern __shared__ __align__(16) unsigned char mix_smem[];
    __shared__ int n_main, n_fallback, n_sel;  // main / fallback survivors; fallback survivors gathered for step 3
    constexpr int WARPS = MIX_THREADS / 32;
    const int64_t r = blockIdx.x;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const unsigned below = (1u << lane) - 1u;
    unsigned char* base = SMEM ? mix_smem : a.scratch + r * a.row_scratch;
    uint64_t* keys = reinterpret_cast<uint64_t*>(base);
    int32_t* pos = reinterpret_cast<int32_t*>(keys + a.keys_cap);  // [n_slots] list position of each entry
    int32_t* state = pos + a.n_slots;                              // [n_slots] -1 dropped, else kept (step 4: r')
    int32_t* cnt = state + a.n_slots;                              // [n_lists] entries of each list
    int32_t* pre = cnt + a.n_lists;                                // [n_lists + 1] prefix of cnt, then of the kept counts
    int64_t lo = 0, hi = 0;
    if (a.indptr) {
        lo = a.indptr[r] - a.base;
        hi = a.indptr[r + 1] - a.base;
    }
    if (tid == 0) n_main = n_fallback = n_sel = 0;

    // 1. each list's first min(k, n_c) unviewed positions within [0, min(n_c, k + m_r)), as path 7 takes them
    for (int c = warp; c < a.n_lists; c += WARPS) {
        const int64_t off = a.offsets[c], n_c = a.offsets[c + 1] - off, s0 = a.slots[c];
        const int kc = (int)(a.slots[c + 1] - s0);
        const int64_t limit = min(n_c, (int64_t)a.k + (hi - lo));
        int kept = 0;
        for (int64_t p0 = 0; p0 < limit && kept < kc; p0 += 32) {
            const int64_t p = p0 + lane;
            bool keep = false;
            if (p < limit) keep = !(hi > lo && csr_contains(a.indices, lo, hi, __ldg(a.list + off + p)));
            const unsigned ballot = __ballot_sync(0xffffffffu, keep);
            const int slot = kept + __popc(ballot & below);
            if (keep && slot < kc) pos[s0 + slot] = (int32_t)(off + p);
            kept += __popc(ballot);
        }
        if (lane == 0) cnt[c] = min(kept, kc);
    }
    __syncthreads();
    if (tid == 0) {
        int s = 0;
        for (int c = 0; c < a.n_lists; ++c) {
            pre[c] = s;
            s += cnt[c];
        }
        pre[a.n_lists] = s;
    }
    __syncthreads();
    const int n_entries = pre[a.n_lists];

    // 2. first occurrences: key = id << 32 | fallback << 31 | slot
    for (int c = warp; c < a.n_lists; c += WARPS) {
        const int n = cnt[c], q = a.quota[c], d0 = pre[c];
        const int64_t s0 = a.slots[c];
        for (int j = lane; j < n; j += 32) {
            const int64_t e = s0 + j;
            keys[d0 + j] = ((uint64_t)(uint32_t)__ldg(a.list + pos[e]) << 32) | ((uint64_t)(j >= q) << 31) | (uint64_t)e;
        }
    }
    mix_block_sort(keys, n_entries);
    int nm = 0, nf = 0;
    for (int i = tid; i < n_entries; i += MIX_THREADS) {
        const uint64_t key = keys[i];
        const bool first = i == 0 || (keys[i - 1] >> 32) != (key >> 32);
        state[key & 0x7fffffffu] = first ? 0 : -1;
        if (first) (key >> 31 & 1u) ? ++nf : ++nm;
    }
    if (nm) atomicAdd(&n_main, nm);
    if (nf) atomicAdd(&n_fallback, nf);
    __syncthreads();

    // 3. too many survivors: keep the k - n_main fallback survivors first in (rank, category) order
    const int NM = n_main, NF = n_fallback;
    if (NM + NF > a.k) {
        const int need = a.k - NM;
        for (int c = warp; c < a.n_lists; c += WARPS) {
            const int n = cnt[c], q = a.quota[c];
            const int64_t s0 = a.slots[c];
            for (int j = q + lane; j < n; j += 32) {
                if (state[s0 + j] != 0) continue;
                state[s0 + j] = -1;
                if (need > 0) keys[atomicAdd(&n_sel, 1)] = (uint64_t)j << 32 | (uint32_t)c;
            }
        }
        if (need > 0) {
            mix_block_sort(keys, NF);  // (its first barrier publishes the gathered keys and states)
            for (int i = tid; i < need; i += MIX_THREADS) {
                const uint64_t key = keys[i];
                state[a.slots[(uint32_t)key] + (int64_t)(key >> 32)] = 0;
            }
        }
        __syncthreads();
    }

    // 4. r' = a kept entry's index among the kept entries of its list, in rank order; pre = kept counts, then their prefix
    for (int c = warp; c < a.n_lists; c += WARPS) {
        const int n = cnt[c];
        const int64_t s0 = a.slots[c];
        int kept = 0;
        for (int j0 = 0; j0 < n; j0 += 32) {
            const int j = j0 + lane;
            const bool kp = j < n && state[s0 + j] >= 0;
            const unsigned ballot = __ballot_sync(0xffffffffu, kp);
            if (kp) state[s0 + j] = kept + __popc(ballot & below);
            kept += __popc(ballot);
        }
        if (lane == 0) pre[c] = kept;
    }
    __syncthreads();
    if (tid == 0) {
        int s = 0;
        for (int c = 0; c < a.n_lists; ++c) {
            const int kc = pre[c];
            pre[c] = s;
            s += kc;
        }
        pre[a.n_lists] = s;
    }
    __syncthreads();
    const int total = pre[a.n_lists];
    int32_t* out = a.out_pos + r * a.k_out;
    for (int c = warp; c < a.n_lists; c += WARPS) {
        const int n = cnt[c];
        const int64_t s0 = a.slots[c];
        for (int j = lane; j < n; j += 32) {
            const int rr = state[s0 + j];
            if (rr < 0) continue;
            int slot;
            if (a.mixing == B200_MIX_GROUP) {
                slot = pre[c] + rr;
            } else {  // kept entries of any list with r' < rr, then those with r' = rr of the lists before c
                slot = 0;
                for (int c2 = 0; c2 < a.n_lists; ++c2) {
                    const int k2 = pre[c2 + 1] - pre[c2];
                    slot += min(k2, rr) + (c2 < c && k2 > rr);
                }
            }
            out[slot] = pos[s0 + j];
        }
    }
    for (int j = total + tid; j < a.k_out; j += MIX_THREADS) out[j] = -1;
    if (tid == 0) a.out_counts[r] = total;
}

}  // namespace b200
