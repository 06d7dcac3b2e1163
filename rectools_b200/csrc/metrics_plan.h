// The argument checks and device bytes of one b200_rank_metrics call (path 10: RecTools' classification and ranking
// metrics from one join of the test interactions with the reco table).  Pure C++17 on host arrays (no CUDA header), so that
// tests/metrics_plan_driver.cpp compiles it with g++ alone and pins it.
#pragma once
#include <climits>
#include <cstdint>
#include <string>

#include "../../include/b200_rank.h"

namespace b200 {

struct MetricsArgs {
    int64_t n_inter = 0;
    bool inter = false;  // inter_users and inter_items given
    int64_t n_reco = 0;
    bool reco = false;   // reco_users, reco_items and reco_ranks given
    int32_t n_k = 0;
    const int64_t* ks = nullptr;
    int32_t n_ndcg = 0;
    const int64_t* ndcg_offsets = nullptr;  // [n_ndcg + 1]
    bool ndcg_terms = false;
    bool outputs = false;  // out_n_users, out_users, out_first_order, out_liked, out_min_rank and out_flags given
    bool out_tp = false;
    bool out_ndcg = false;
};

struct MetricsPlan {
    int64_t slots = 0;      // hash-table slots: the smallest power of two >= 2 x n_reco, at least 16
    int64_t k_max = 0;      // the largest k (0: none)
    int64_t n_terms = 0;    // NDCG term-table entries in all
    int64_t device_bytes = 0;  // every buffer of the call but CUB's scratch
    int error = B200_OK;
    std::string message;
};

// Bits needed to write x >= 0 (0 for 0).
inline int metrics_bits(uint64_t x) {
    int b = 0;
    while (b < 64 && (x >> b) != 0) ++b;
    return b;
}

// Device bytes of a call with n interaction rows, m reco rows, `slots` table slots, n_k k values, n_terms NDCG term
// entries in n_ndcg tables, with or without the MAP stage.  Per interaction row: users and items (16 B), its matched rank
// (8 B), the sort by user (8 B key + 2 x 4 B row index), and with MAP the hit keys (2 x 8 B) and precisions (8 B).  Per
// test user, at most n of them: the user, its row count and segment offset (3 x 8 B), the first-row sort (2 x 4 B keys,
// 2 x 8 B segment ids), the smallest matched rank (8 B), TP per k (8 B), the NDCG sums (8 B per table) and, with MAP,
// the hit count and offset (2 x 8 B) and the precision sums (8 B per k).  Per reco row: users, items and ranks (24 B);
// per slot 4 B.  Plus the k values, the NDCG tables, the flags and the user count; an empty buffer still takes 16 B.
inline int64_t metrics_device_bytes(int64_t n, int64_t m, int64_t slots, int64_t n_k, int64_t n_ndcg, int64_t n_terms, bool map) {
    const int64_t per_row = 16 + 8 + 16 + (map ? 24 : 0);
    const int64_t per_user = 24 + 24 + 8 + 8 * n_k + 8 * n_ndcg + (map ? 16 + 8 * n_k : 0);
    return n * (per_row + per_user) + 24 * m + 4 * slots + 8 * n_k + 8 * (n_ndcg + 1) + 8 * n_terms + 4 + 8;
}

// Every refusal of the call, then its table size and device bytes.  `map`: the MAP stage runs (out_map given).
inline MetricsPlan plan_metrics(const MetricsArgs& a, bool map) {
    MetricsPlan p;
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_metrics: " + why;
        return p;
    };
    if (a.n_inter < 0 || a.n_reco < 0) return refuse(B200_E_INVALID, "n_inter and n_reco must be >= 0");
    if (a.n_inter > INT_MAX || a.n_reco > INT_MAX) return refuse(B200_E_INVALID, "n_inter and n_reco must be <= 2^31 - 1 (rows are int32)");
    if (a.n_k < 0 || a.n_ndcg < 0) return refuse(B200_E_INVALID, "n_k and n_ndcg must be >= 0");
    if (a.n_inter > 0 && !a.inter) return refuse(B200_E_INVALID, "inter_users / inter_items are NULL");
    if (a.n_reco > 0 && !a.reco) return refuse(B200_E_INVALID, "reco_users / reco_items / reco_ranks are NULL");
    if (a.n_k > 0 && !a.ks) return refuse(B200_E_INVALID, "ks is NULL");
    for (int32_t q = 0; q < a.n_k; ++q) {
        if (a.ks[q] < 1 || a.ks[q] > INT_MAX) return refuse(B200_E_INVALID, "ks[" + std::to_string(q) + "] = " + std::to_string(a.ks[q]) + " lies outside [1, 2^31 - 1]");
        if (q > 0 && a.ks[q] <= a.ks[q - 1]) return refuse(B200_E_INVALID, "ks are not strictly ascending");
    }
    if (map && a.n_k == 0) return refuse(B200_E_INVALID, "out_map is given without a k");
    if (a.n_ndcg > 0 && !a.ndcg_offsets) return refuse(B200_E_INVALID, "ndcg_offsets is NULL");
    if (a.n_ndcg > 0) {
        if (a.ndcg_offsets[0] != 0) return refuse(B200_E_INVALID, "ndcg_offsets[0] = " + std::to_string(a.ndcg_offsets[0]) + ", not 0");
        for (int32_t s = 0; s < a.n_ndcg; ++s) {
            const int64_t len = a.ndcg_offsets[s + 1] - a.ndcg_offsets[s];
            if (len < 1 || len > INT_MAX) return refuse(B200_E_INVALID, "NDCG table " + std::to_string(s) + " has " + std::to_string(len) + " terms, not [1, 2^31 - 1]");
        }
        p.n_terms = a.ndcg_offsets[a.n_ndcg];
        if (!a.ndcg_terms) return refuse(B200_E_INVALID, "ndcg_terms is NULL");
    }
    if (a.n_inter > 0 && !a.outputs) return refuse(B200_E_INVALID, "out_n_users / out_users / out_first_order / out_liked / out_min_rank / out_flags are NULL");
    if (a.n_inter > 0 && a.n_k > 0 && !a.out_tp) return refuse(B200_E_INVALID, "out_tp is NULL");
    if (a.n_inter > 0 && a.n_ndcg > 0 && !a.out_ndcg) return refuse(B200_E_INVALID, "out_ndcg is NULL");
    p.k_max = a.n_k > 0 ? a.ks[a.n_k - 1] : 0;
    p.slots = 16;
    while (p.slots < 2 * a.n_reco) p.slots *= 2;
    p.device_bytes = metrics_device_bytes(a.n_inter, a.n_reco, p.slots, a.n_k, a.n_ndcg, p.n_terms, map);
    return p;
}

}  // namespace b200
