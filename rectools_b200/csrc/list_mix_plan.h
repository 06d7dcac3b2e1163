// The argument checks, scratch layout and row chunks of one b200_rank_topk_list_mix call (path 8: per-category lists,
// each minus a row's viewed ids, mixed as `PopularInCategoryModel._recommend_u2i` mixes them).  Pure C++17 on host arrays
// (no CUDA header), so that tests/list_mix_plan_driver.cpp compiles it with g++ alone and pins it.
#pragma once
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/b200_rank.h"
#include "list_plan.h"

namespace b200 {

// Largest per-row scratch kept in shared memory (one CTA per row); above it every row of the call works in a chunk-owned
// slice of global memory.  B200_LIST_MIX_SMEM=n lowers the limit to n bytes (0 or unset: this default).
constexpr int64_t MIX_SMEM_BYTES = 200 * 1024;

inline int64_t list_mix_smem_hook() {
    const char* v = std::getenv("B200_LIST_MIX_SMEM");
    return v ? std::max<long long>(0, std::atoll(v)) : 0;
}

inline int64_t next_pow2(int64_t n) {
    int64_t p = 1;
    while (p < n) p <<= 1;
    return p;
}

// Per-row scratch of the kernel (list_mix.cuh), in this order: sort keys (8 B x next_pow2(U)), entry list positions and
// entry states (4 B x U each), per-category counts and prefixes (4 B x (2 n_lists + 1)), rounded up to 16 B.  U = the
// entry slots of a row, sum over categories of min(k, n_c).
inline int64_t mix_row_scratch(int64_t U, int64_t n_lists) {
    const int64_t b = 8 * next_pow2(std::max<int64_t>(U, 1)) + 8 * U + 4 * (2 * n_lists + 1);
    return (b + 15) / 16 * 16;
}

struct ListMixArgs {
    int64_t n_lists = 0;
    const int64_t* offsets = nullptr;  // [n_lists + 1]
    const int32_t* list_ids = nullptr;  // [offsets[n_lists]]
    const int32_t* quota = nullptr;     // [n_lists]
    int64_t mixing = B200_MIX_ROTATE;
    int64_t n_rows = 0;
    const int64_t* indptr = nullptr;  // nullable: nothing viewed
    const int32_t* indices = nullptr;
    int64_t k = 0;
    bool out_pos = false;
    bool out_counts = false;
};

struct ListMixPlan {
    int k_out = 0;                 // min(k, total list length)
    int64_t n_total = 0;           // total list length
    std::vector<int64_t> slots;    // [n_lists + 1]: entry slot c starts at slots[c] (prefix of min(k, n_c))
    int64_t row_scratch = 0;       // bytes of one row's scratch
    bool smem = false;             // scratch in shared memory (else a global slice per row of the chunk)
    std::vector<int64_t> bounds;   // chunk c = rows [bounds[c], bounds[c + 1])
    int64_t max_chunk_rows = 0;
    int64_t max_chunk_nnz = 0;
    int error = B200_OK;
    std::string message;
    int64_t n_chunks() const { return bounds.empty() ? 0 : (int64_t)bounds.size() - 1; }
};

// Device memory of one row in a chunk: its row pointer, viewed ids, output positions and count (list_row_bytes), plus its
// scratch when that is global.
inline int64_t list_mix_row_bytes(int64_t m, int64_t k_out, int64_t global_scratch) {
    return list_row_bytes(m, k_out) + global_scratch;
}

// Every refusal of the call, then its layout and row chunks.  Chunks take whole rows, in order, while list_mix_row_bytes of
// their rows stays within `budget` and their rows within `max_rows` (0: no cap); a row that alone exceeds the budget is
// refused with B200_E_NOMEM.  A call with no row, no list or only empty lists has no chunk.
inline ListMixPlan plan_list_mix(const ListMixArgs& a, int64_t max_rows, int64_t smem_cap = 0,
                                 int64_t budget = LIST_CHUNK_BYTES) {
    ListMixPlan p;
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_topk_list_mix: " + why;
        p.bounds.clear();
        p.slots.clear();
        return p;
    };
    if (a.n_lists < 0 || a.n_rows < 0) return refuse(B200_E_INVALID, "n_lists and n_rows must be >= 0");
    if (a.k < 1) return refuse(B200_E_INVALID, "k must be >= 1");
    if (a.mixing != B200_MIX_ROTATE && a.mixing != B200_MIX_GROUP)
        return refuse(B200_E_INVALID, "unknown mixing " + std::to_string(a.mixing));
    if (a.n_lists > 0 && !a.offsets) return refuse(B200_E_INVALID, "list_offsets is NULL");
    if (a.n_lists > 0 && !a.quota) return refuse(B200_E_INVALID, "quota is NULL");
    if (a.n_lists > 0) {
        if (a.offsets[0] != 0) return refuse(B200_E_INVALID, "list_offsets[0] = " + std::to_string(a.offsets[0]) + ", not 0");
        for (int64_t c = 0; c < a.n_lists; ++c)
            if (a.offsets[c + 1] < a.offsets[c]) return refuse(B200_E_INVALID, "list_offsets is not monotone at list " + std::to_string(c));
        p.n_total = a.offsets[a.n_lists];
    }
    if (p.n_total > INT_MAX) return refuse(B200_E_INVALID, "the lists hold more than 2^31 - 1 ids (positions are int32)");
    if (p.n_total > 0 && !a.list_ids) return refuse(B200_E_INVALID, "list_ids is NULL");
    for (int64_t i = 0; i < p.n_total; ++i)
        if (a.list_ids[i] < 0) return refuse(B200_E_INVALID, "list_ids[" + std::to_string(i) + "] = " + std::to_string(a.list_ids[i]) + " is negative");
    int64_t quota_sum = 0;
    for (int64_t c = 0; c < a.n_lists; ++c) {
        if (a.quota[c] < 0) return refuse(B200_E_INVALID, "quota[" + std::to_string(c) + "] = " + std::to_string(a.quota[c]) + " is negative");
        quota_sum += a.quota[c];
    }
    if (quota_sum > a.k) return refuse(B200_E_INVALID, "the quotas sum to " + std::to_string(quota_sum) + ", more than k");
    p.k_out = (int)std::min<int64_t>(a.k, p.n_total);
    if (a.n_rows > 0 && !a.out_counts) return refuse(B200_E_INVALID, "out_counts is NULL");
    if (a.n_rows > 0 && p.k_out > 0 && !a.out_pos) return refuse(B200_E_INVALID, "out_pos is NULL");
    const int64_t* ip = a.indptr;
    if (ip) {
        // the CSR checks of b200_rank_topk_list
        if (ip[0] != 0) return refuse(B200_E_INVALID, "csr_indptr[0] = " + std::to_string(ip[0]) + ", not 0");
        for (int64_t r = 0; r < a.n_rows; ++r)
            if (ip[r + 1] < ip[r]) return refuse(B200_E_INVALID, "csr_indptr is not monotone at row " + std::to_string(r));
        if (ip[a.n_rows] > 0 && !a.indices) return refuse(B200_E_INVALID, "csr_indices is NULL");
        for (int64_t r = 0; r < a.n_rows; ++r)
            for (int64_t e = ip[r] + 1; e < ip[r + 1]; ++e)
                if (a.indices[e] < a.indices[e - 1])
                    return refuse(B200_E_INVALID, "row " + std::to_string(r) + ": viewed ids are not ascending");
    }
    if (a.n_rows == 0 || p.k_out == 0) return p;
    p.slots.assign(a.n_lists + 1, 0);
    for (int64_t c = 0; c < a.n_lists; ++c)
        p.slots[c + 1] = p.slots[c] + std::min<int64_t>(a.k, a.offsets[c + 1] - a.offsets[c]);
    p.row_scratch = mix_row_scratch(p.slots[a.n_lists], a.n_lists);
    p.smem = p.row_scratch <= (smem_cap > 0 ? std::min(smem_cap, MIX_SMEM_BYTES) : MIX_SMEM_BYTES);
    const int64_t global_scratch = p.smem ? 0 : p.row_scratch;
    p.bounds.push_back(0);
    int64_t bytes = 0, nnz = 0, rows = 0;
    for (int64_t r = 0; r < a.n_rows; ++r) {
        const int64_t m = ip ? ip[r + 1] - ip[r] : 0, b = list_mix_row_bytes(m, p.k_out, global_scratch);
        if (b > budget)
            return refuse(B200_E_NOMEM, "row " + std::to_string(r) + " (" + std::to_string(m) + " viewed ids, " +
                                            std::to_string(p.slots[a.n_lists]) + " entry slots) needs " + std::to_string(b) +
                                            " bytes, more than a chunk's " + std::to_string(budget));
        if (rows > 0 && (bytes + b > budget || rows == max_rows)) {
            p.bounds.push_back(r);
            p.max_chunk_rows = std::max(p.max_chunk_rows, rows);
            p.max_chunk_nnz = std::max(p.max_chunk_nnz, nnz);
            bytes = nnz = rows = 0;
        }
        bytes += b;
        nnz += m;
        ++rows;
    }
    p.bounds.push_back(a.n_rows);
    p.max_chunk_rows = std::max(p.max_chunk_rows, rows);
    p.max_chunk_nnz = std::max(p.max_chunk_nnz, nnz);
    return p;
}

}  // namespace b200
