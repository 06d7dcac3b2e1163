// The argument checks and row chunks of one b200_rank_topk_list call (path 7: the first k of one shared, ordered list,
// minus each row's viewed ids).  Pure C++17 on host arrays (no CUDA header), so that tests/list_plan_driver.cpp compiles
// it with g++ alone and pins it.
#pragma once
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/b200_rank.h"

namespace b200 {

// Device memory of one row chunk: the chunk's row pointers (8 B per row), viewed ids (4 B each), output positions
// (4 B x k_out per row) and counts (4 B per row).  The shared list (4 B per entry) is uploaded once, outside the budget.
constexpr int64_t LIST_CHUNK_BYTES = (int64_t)1 << 30;

inline int64_t list_row_bytes(int64_t m, int64_t k_out) { return 8 + 4 * m + 4 * k_out + 4; }

// B200_LIST_CHUNK_ROWS=n caps the rows of a chunk (0 or unset: no cap beyond the byte budget).
inline int64_t list_chunk_rows_hook() {
    const char* v = std::getenv("B200_LIST_CHUNK_ROWS");
    return v ? std::max<long long>(0, std::atoll(v)) : 0;
}

struct ListArgs {
    int64_t n_list = 0;
    const int32_t* list_ids = nullptr;
    int64_t n_rows = 0;
    const int64_t* indptr = nullptr;  // nullable: nothing viewed
    const int32_t* indices = nullptr;
    int64_t k = 0;
    bool out_pos = false;     // out_pos given
    bool out_counts = false;  // out_counts given
};

struct ListPlan {
    int k_out = 0;
    std::vector<int64_t> bounds;  // chunk c = rows [bounds[c], bounds[c + 1])
    int64_t max_chunk_rows = 0;
    int64_t max_chunk_nnz = 0;    // viewed ids of the largest chunk
    int error = B200_OK;
    std::string message;
    int64_t n_chunks() const { return bounds.empty() ? 0 : (int64_t)bounds.size() - 1; }
};

// Every refusal of the call, then its row chunks.  Chunks take whole rows, in order, while list_row_bytes of their rows
// stays within `budget` and their rows within `max_rows` (0: no cap); a row that alone exceeds the budget is refused with
// B200_E_NOMEM.  A call with no row or k_out = 0 (an empty list) has no chunk.
inline ListPlan plan_list(const ListArgs& a, int64_t max_rows, int64_t budget = LIST_CHUNK_BYTES) {
    ListPlan p;
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_topk_list: " + why;
        p.bounds.clear();
        return p;
    };
    if (a.n_list < 0 || a.n_rows < 0) return refuse(B200_E_INVALID, "n_list and n_rows must be >= 0");
    if (a.k < 1) return refuse(B200_E_INVALID, "k must be >= 1");
    if (a.n_list > INT_MAX) return refuse(B200_E_INVALID, "n_list exceeds 2^31 - 1 (positions are int32)");
    p.k_out = (int)std::min<int64_t>(a.k, a.n_list);
    if (a.n_list > 0 && !a.list_ids) return refuse(B200_E_INVALID, "list_ids is NULL");
    if (a.n_rows > 0 && !a.out_counts) return refuse(B200_E_INVALID, "out_counts is NULL");
    if (a.n_rows > 0 && p.k_out > 0 && !a.out_pos) return refuse(B200_E_INVALID, "out_pos is NULL");
    for (int64_t i = 0; i < a.n_list; ++i)
        if (a.list_ids[i] < 0) return refuse(B200_E_INVALID, "list_ids[" + std::to_string(i) + "] = " + std::to_string(a.list_ids[i]) + " is negative");
    const int64_t* ip = a.indptr;
    if (ip) {
        // the checks b200_rank_topk makes of a host filter CSR, with the row pointers starting at 0
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
    p.bounds.push_back(0);
    int64_t bytes = 0, nnz = 0, rows = 0;
    for (int64_t r = 0; r < a.n_rows; ++r) {
        const int64_t m = ip ? ip[r + 1] - ip[r] : 0, b = list_row_bytes(m, p.k_out);
        if (b > budget)
            return refuse(B200_E_NOMEM, "row " + std::to_string(r) + " (" + std::to_string(m) + " viewed ids, k_out = " +
                                            std::to_string(p.k_out) + ") needs " + std::to_string(b) + " bytes, more than a chunk's " +
                                            std::to_string(budget));
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
