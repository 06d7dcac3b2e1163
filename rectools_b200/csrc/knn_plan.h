// The argument checks and row chunks of one b200_rank_topk_knn call (path 9: ItemKNN user scores accumulated from the
// neighbour matrix S).  Pure C++17 on host arrays (no CUDA header), so that tests/knn_plan_driver.cpp compiles it with
// g++ alone and pins it.
#pragma once
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../include/b200_rank.h"

namespace b200 {

// Device memory of one row chunk, as for the other host-buffer paths.  S and the whitelist are uploaded once, outside the
// budget, and so is the dense route's scratch.
constexpr int64_t KNN_CHUNK_BYTES = (int64_t)1 << 30;

// A row whose bound B_u = sum_e |S[j_e]| is at most this accumulates in the shared-memory table of knn.cuh (4096 slots,
// at most 3/4 full); a larger one in a dense fp64 row of n_items in global scratch.
constexpr int64_t KNN_TABLE_BOUND = 3072;

// Bytes of a row with m weighted entries, f filter ids, `slots` candidate slots and k output columns: its row pointers
// (2 x 8 B), entries (4 B id + 4 B weight), filter ids (4 B), per slot the pair code, score and id of the hand-off plus
// path 6's order key and position (8 + 8 + 4 + 8 + 8 B), and per output column the ids, scores, path 6's positions and
// its sort buffers (4 + 8 + 8 + 32 B), plus the row's count and route entry.
inline int64_t knn_row_bytes(int64_t m, int64_t f, int64_t slots, int64_t k) { return 16 + 8 * m + 4 * f + 36 * slots + 52 * k + 8; }

// B200_KNN_CHUNK_ROWS=n caps the rows of a chunk (0 or unset: no cap beyond the byte budget).
inline int64_t knn_chunk_rows_hook() {
    const char* v = std::getenv("B200_KNN_CHUNK_ROWS");
    return v ? std::max<long long>(0, std::atoll(v)) : 0;
}

struct KnnArgs {
    int64_t n_items = 0;
    const int64_t* s_indptr = nullptr;  // [n_items + 1]
    const int32_t* s_indices = nullptr;
    const double* s_data = nullptr;
    int64_t n_rows = 0;
    const int64_t* u_indptr = nullptr;  // [n_rows + 1]
    const int32_t* u_indices = nullptr;
    const float* u_data = nullptr;
    const int64_t* f_indptr = nullptr;  // nullable: no filter
    const int32_t* f_indices = nullptr;
    const int32_t* whitelist = nullptr;
    int64_t n_whitelist = -1;  // < 0: no whitelist
    int64_t k = 0;
    bool outputs = false;  // out_ids, out_scores and out_counts given
};

struct KnnPlan {
    std::vector<int64_t> bounds;  // chunk c = rows [bounds[c], bounds[c + 1])
    std::vector<int64_t> bound;   // B_u of every row
    std::vector<int64_t> slot;    // slot offsets of every row (n_rows + 1): row r's candidates go to [slot[r], slot[r + 1])
    int64_t max_chunk_rows = 0;
    int64_t max_chunk_u = 0;      // weighted entries of the largest chunk
    int64_t max_chunk_f = 0;      // filter ids of the largest chunk
    int64_t max_chunk_slots = 0;
    int64_t max_chunk_dense = 0;  // rows above KNN_TABLE_BOUND in one chunk
    int error = B200_OK;
    std::string message;
    int64_t n_chunks() const { return bounds.empty() ? 0 : (int64_t)bounds.size() - 1; }
};

// Every refusal of the call, then its row chunks.  Chunks take whole rows, in order, while knn_row_bytes of their rows
// stays within `budget` and their rows within `max_rows` (0: no cap); a row that alone exceeds the budget is refused with
// B200_E_NOMEM.  A call with no row has no chunk.
inline KnnPlan plan_knn(const KnnArgs& a, int64_t max_rows, int64_t budget = KNN_CHUNK_BYTES) {
    KnnPlan p;
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_topk_knn: " + why;
        p.bounds.clear();
        p.bound.clear();
        p.slot.clear();
        return p;
    };
    auto csr = [&](const char* name, const int64_t* ip, int64_t rows, const void* idx, int64_t& nnz) -> std::string {
        if (!ip) return std::string(name) + "_indptr is NULL";
        if (ip[0] != 0) return std::string(name) + "_indptr[0] = " + std::to_string(ip[0]) + ", not 0";
        for (int64_t r = 0; r < rows; ++r)
            if (ip[r + 1] < ip[r]) return std::string(name) + "_indptr is not monotone at row " + std::to_string(r);
        nnz = ip[rows];
        if (nnz > 0 && !idx) return std::string(name) + "_indices is NULL";
        return "";
    };
    if (a.n_items < 0 || a.n_rows < 0) return refuse(B200_E_INVALID, "n_items and n_rows must be >= 0");
    if (a.n_items > INT_MAX) return refuse(B200_E_INVALID, "n_items exceeds 2^31 - 1 (ids are int32)");
    if (a.k < 1) return refuse(B200_E_INVALID, "k must be >= 1");
    if (a.n_rows > 0 && !a.outputs) return refuse(B200_E_INVALID, "out_ids / out_scores / out_counts are NULL");
    int64_t s_nnz = 0, u_nnz = 0, f_nnz = 0;
    std::string why = csr("s", a.s_indptr, a.n_items, a.s_indices, s_nnz);
    if (why.empty() && s_nnz > 0 && !a.s_data) why = "s_data is NULL";
    if (why.empty()) why = csr("u", a.u_indptr, a.n_rows, a.u_indices, u_nnz);
    if (why.empty() && u_nnz > 0 && !a.u_data) why = "u_data is NULL";
    if (why.empty() && a.f_indptr) why = csr("f", a.f_indptr, a.n_rows, a.f_indices, f_nnz);
    if (!why.empty()) return refuse(B200_E_INVALID, why);
    {
        std::vector<int64_t> seen((size_t)a.n_items, -1);  // an item occurs once per S row: the kernel adds without atomics
        for (int64_t i = 0; i < a.n_items; ++i)
            for (int64_t e = a.s_indptr[i]; e < a.s_indptr[i + 1]; ++e) {
                const int32_t j = a.s_indices[e];
                if (j < 0 || j >= a.n_items)
                    return refuse(B200_E_INVALID, "s_indices[" + std::to_string(e) + "] = " + std::to_string(j) + " lies outside [0, n_items)");
                if (seen[j] == i) return refuse(B200_E_INVALID, "S row " + std::to_string(i) + " holds item " + std::to_string(j) + " twice");
                seen[j] = i;
                if (!std::isfinite(a.s_data[e])) return refuse(B200_E_INVALID, "s_data[" + std::to_string(e) + "] is not finite");
            }
    }
    for (int64_t e = 0; e < u_nnz; ++e) {
        if (a.u_indices[e] < 0 || a.u_indices[e] >= a.n_items)
            return refuse(B200_E_INVALID, "u_indices[" + std::to_string(e) + "] = " + std::to_string(a.u_indices[e]) + " lies outside [0, n_items)");
        if (!std::isfinite(a.u_data[e])) return refuse(B200_E_INVALID, "u_data[" + std::to_string(e) + "] is not finite");
    }
    if (a.f_indptr)
        for (int64_t r = 0; r < a.n_rows; ++r)
            for (int64_t e = a.f_indptr[r] + 1; e < a.f_indptr[r + 1]; ++e)
                if (a.f_indices[e] < a.f_indices[e - 1])
                    return refuse(B200_E_INVALID, "row " + std::to_string(r) + ": filter ids are not ascending");
    const bool wl = a.n_whitelist >= 0;
    if (wl && a.n_whitelist > 0 && !a.whitelist) return refuse(B200_E_INVALID, "whitelist is NULL");
    for (int64_t i = 0; wl && i < a.n_whitelist; ++i) {
        if (a.whitelist[i] < 0 || a.whitelist[i] >= a.n_items)
            return refuse(B200_E_INVALID, "whitelist[" + std::to_string(i) + "] = " + std::to_string(a.whitelist[i]) + " lies outside [0, n_items)");
        if (i > 0 && a.whitelist[i] <= a.whitelist[i - 1]) return refuse(B200_E_INVALID, "the whitelist is not strictly ascending");
    }
    if (a.n_rows == 0) return p;
    // a row's candidates are touched items, so no more than B_u, n_items and the whitelist's length
    const int64_t n_cand = wl ? a.n_whitelist : a.n_items;
    p.bound.resize(a.n_rows);
    p.slot.resize(a.n_rows + 1);
    p.slot[0] = 0;
    for (int64_t r = 0; r < a.n_rows; ++r) {
        int64_t b = 0;
        for (int64_t e = a.u_indptr[r]; e < a.u_indptr[r + 1]; ++e) {
            const int32_t j = a.u_indices[e];
            b += a.s_indptr[j + 1] - a.s_indptr[j];
        }
        p.bound[r] = b;
        p.slot[r + 1] = p.slot[r] + std::min(b, n_cand);
    }
    p.bounds.push_back(0);
    int64_t bytes = 0, u = 0, f = 0, slots = 0, dense = 0, rows = 0;
    auto close = [&]() {
        p.max_chunk_rows = std::max(p.max_chunk_rows, rows);
        p.max_chunk_u = std::max(p.max_chunk_u, u);
        p.max_chunk_f = std::max(p.max_chunk_f, f);
        p.max_chunk_slots = std::max(p.max_chunk_slots, slots);
        p.max_chunk_dense = std::max(p.max_chunk_dense, dense);
    };
    for (int64_t r = 0; r < a.n_rows; ++r) {
        const int64_t m = a.u_indptr[r + 1] - a.u_indptr[r], fr = a.f_indptr ? a.f_indptr[r + 1] - a.f_indptr[r] : 0;
        const int64_t s = p.slot[r + 1] - p.slot[r], b = knn_row_bytes(m, fr, s, a.k);
        if (b > budget)
            return refuse(B200_E_NOMEM, "row " + std::to_string(r) + " (" + std::to_string(m) + " entries, " + std::to_string(s) +
                                            " candidate slots, k = " + std::to_string(a.k) + ") needs " + std::to_string(b) +
                                            " bytes, more than a chunk's " + std::to_string(budget));
        if (rows > 0 && (bytes + b > budget || rows == max_rows)) {
            p.bounds.push_back(r);
            close();
            bytes = u = f = slots = dense = rows = 0;
        }
        bytes += b;
        u += m;
        f += fr;
        slots += s;
        dense += p.bound[r] > KNN_TABLE_BOUND;
        ++rows;
    }
    p.bounds.push_back(a.n_rows);
    close();
    return p;
}

}  // namespace b200
