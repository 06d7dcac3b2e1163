// The decision of one b200_rank_topk call: which path ranks it, with which tensor-core mode and list size K', in how
// many row chunks -- or which refusal it gets.  Pure arithmetic on the query shape, the engine's properties and the
// B200_* environment hooks, in plain C++17 (no CUDA header), so that tests/test_call_plan_cpu.py compiles it with g++
// alone and pins it.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <optional>
#include <string>
#include <vector>

#include "../../include/b200_rank.h"
#include "sizes.h"

namespace b200 {

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// Tuning, measurement and test variables, read once per call (tests set them between calls, never during one).
struct Hooks {
    int wide = 1;               // B200_WIDE: 0 keeps 24 < k <= 1024 off the wide mode (multi-pass route / path 3)
    std::optional<int> wide_t;  // B200_WIDE_T: the wide mode's expected candidate count T
    int tc_kcand = 0;           // B200_TC_KCAND: K' of the main pass (4 .. 32)
    int tc_splits = 0;          // B200_TC_SPLITS: object splits of a fused-kernel launch (1 .. its maximum)
    int tc_carousel = 1;        // B200_TC_CAROUSEL: 0 starts every work item at its first object tile
    int tc_debug = 0;           // B200_TC_DEBUG: fused-kernel measurement modes (TcParams::debug_mode; results are invalid)
    int64_t chunk_rows = 0;     // B200_CHUNK_ROWS: row chunk of host-input calls and of path 4 (0: 8 waves; at least 256)
    int wide_budget_mb = 2048;  // B200_WIDE_BUDGET_MB: device memory for the append lists of k > 128
    int tc_snapshot = 0;        // B200_TC_SNAPSHOT: the fused-kernel launch whose state is kept (0: none)
    int select = 1;             // B200_SELECT: paths 2 / 3 select with 0 the streaming passes for every k, 2 the radix
                                // selection for every k (cross-checks); 1 the radix selection for k > 1024 only
};

inline Hooks read_hooks() {
    auto get = [](const char* name, int dflt) {
        const char* v = std::getenv(name);
        return v ? std::atoi(v) : dflt;
    };
    Hooks h;
    h.wide = get("B200_WIDE", h.wide);
    if (const char* v = std::getenv("B200_WIDE_T")) h.wide_t = std::atoi(v);
    h.tc_kcand = get("B200_TC_KCAND", h.tc_kcand);
    h.tc_splits = get("B200_TC_SPLITS", h.tc_splits);
    h.tc_carousel = get("B200_TC_CAROUSEL", h.tc_carousel);
    h.tc_debug = get("B200_TC_DEBUG", h.tc_debug);
    if (const char* v = std::getenv("B200_CHUNK_ROWS")) h.chunk_rows = std::max<int64_t>(256, std::atoll(v));
    h.wide_budget_mb = get("B200_WIDE_BUDGET_MB", h.wide_budget_mb);
    h.tc_snapshot = get("B200_TC_SNAPSHOT", h.tc_snapshot);
    h.select = get("B200_SELECT", h.select);
    return h;
}

// Wide mode: T = the candidates a row is expected to collect, and the slots of each of its two append lists.  The
// threshold frozen after a fraction q of the stream is about the (lists x K' - 6)-th best of that fraction, i.e. rank
// ~ (lists x K' - 6) / q overall, so q follows from T.  k <= 128: T = 1.35 k + 40 (K' = 24), at most WIDE_MAX slots per row.
// k > 128: T = 1.6 k + 64 (K' = 32), at most WIDE_MAX_L slots per row -- the frozen threshold is an order statistic of
// ~58 samples, and this margin keeps the rows with fewer than k candidates (or an overflowing list) near 0.3 % (DESIGN 3.4).
struct WideGeom {
    double T = 0;
    int cand_stride = 0;
};

inline WideGeom wide_geom(int kp, const Hooks& h) {
    WideGeom g;
    g.T = h.wide_t.value_or(kp <= 128 ? (int)(1.35 * kp + 40) : (int)(1.6 * kp + 64));
    g.cand_stride = std::min((int)round_up((int64_t)(g.T / 2 * 1.5 + 32), 8), (kp <= 128 ? WIDE_MAX : WIDE_MAX_L) / 2);
    return g;
}

// Object splits of a fused-kernel launch: fill the machine when there are few row tiles, even out the last wave
// otherwise (`n_units` CTA pairs work concurrently).  `forced` (B200_TC_SPLITS) wins when it is in range.
// At most MAX_SPLITS, so a row has at most 2 x 16 = 32 lists: rescore_select_kernel keeps one list per lane.
constexpr int MAX_SPLITS = 16;
static_assert(2 * MAX_SPLITS <= 32, "rescore_select_kernel holds one candidate list per lane of a warp");

inline int choose_splits(int n_row_tiles, int n_obj_tiles, int n_units, bool wide, int forced) {
    int best_splits = 1;
    double best_eff = -1.0;
    const int max_splits = wide ? 1 : std::max(1, std::min(MAX_SPLITS, n_obj_tiles * 2 / 32));
    for (int s = 1; s <= max_splits; ++s) {
        const double work = (double)n_row_tiles * s;
        const double waves = std::ceil(work / n_units);
        const double eff = work / (waves * n_units) - 0.01 * (s - 1);
        if (eff > best_eff + 1e-9) {
            best_eff = eff;
            best_splits = s;
        }
    }
    if (forced >= 1 && forced <= max_splits) best_splits = forced;
    return best_splits;
}

// What a call ranks and what the engine knows about itself.
struct CallShape {
    int64_t n_rows = 0;
    int64_t n_pos = 0;  // object positions: the whitelist, else the catalogue
    int64_t k = 0;      // requested k
    int d = 0, d_pad = 0;
    int sm_count = 0;
    int tc_dtype = B200_TC_OFF;  // the engine's resolved tensor-core type
    int n_peers = 0;             // ranks the engine shares thresholds with
    int32_t flags = 0;           // B200_Q_*
    bool sparse = false;         // sparse subject rows
    bool rows = false;           // stored rows as score rows (b200_rank_query.object_rows)
    int64_t n_objects = 0;       // the engine's objects (path 4: the length of a stored row must be d)
    bool cosine = false;         // the engine is a COSINE engine
    bool id_offset = false;      // the engine has a non-zero id offset
};

enum class Path { EXACT = 0, TC = 1, SPARSE = 2, DENSE_LARGE_K = 3, ROWS = 4, CANDIDATES = 5 };  // = b200_rank_stats::path

// How the tensor-core path ranks the rows of the main pass.
enum class TcMode {
    NARROW,      // k <= 24: adaptive lists of K' slots
    WIDE,        // 24 < k <= 128: one pass, frozen threshold + append lists
    WIDE_L,      // 128 < k <= 1024: the same with longer append lists and the large re-score
    MULTI_PASS,  // 24 < k without the wide mode: certified passes of 20 results for every row
};

// How paths 2 and 3 select from their materialised score rows.
enum class Select {
    PASSES,  // ceil(k_out / 32) streaming passes of scores_topk_kernel over every row
    RADIX,   // large_k_select_kernel: radix select + one sort of the k_out survivors (k_out > 1024);
             // path 4: row_select_kernel, the same selection over the stored rows, for every k_out
};

// Bytes per row of a path-2 / path-3 row chunk: the fp32 score row and, when the radix selection sorts more survivors than
// its shared memory holds, the sort's global scratch (4 words per entry).  Chunks keep within 1 GiB of these.
inline int64_t select_row_bytes(int64_t n_pos, int64_t k_out, Select sel) {
    return 4 * n_pos + (sel == Select::RADIX && k_out > LK_SMEM_PAIRS ? 16 * k_out : 0);
}
constexpr int64_t SELECT_CHUNK_BYTES = (int64_t)1 << 30;

// Path 4 reads the stored rows in place: a row chunk holds no score row, only the sort scratch above LK_SMEM_PAIRS.
inline int64_t rows_row_bytes(int64_t k_out) { return k_out > LK_SMEM_PAIRS ? 16 * k_out : 0; }

struct CallPlan {
    int k_out = 0;
    Path path = Path::EXACT;
    Select select = Select::PASSES;  // paths SPARSE / DENSE_LARGE_K (the re-rank of rows a wide pass rejects: PASSES); ROWS: RADIX
    TcMode mode = TcMode::NARROW;  // path TC only
    bool bf16 = false;             // operand type of the tensor-core passes
    static constexpr int nw = 8;   // epilogue warps of the fused kernel: one geometry (b200_rank_stats::epi_warps)
    int k_cand = 0;                // K' of the main pass
    bool peers = false;            // the main pass shares thresholds (B200_Q_SHARED_THRESHOLDS)
    WideGeom geom;                 // WIDE / WIDE_L
    int64_t chunk = 0, n_chunks = 0;  // row chunks of the main pass
    int error = B200_OK;           // otherwise the call is refused with this code and message
    std::string message;

    bool tc() const { return path == Path::TC; }
    bool wide() const { return tc() && (mode == TcMode::WIDE || mode == TcMode::WIDE_L); }
};

// Path 4: batch row r is the engine's stored row object_rows[r], ranked by row_select_kernel in one launch per row chunk,
// whatever k is.  Row chunks: 8 waves of CTA pairs (or B200_CHUNK_ROWS) when the call has at least two of them, so that
// the copies of one chunk overlap the ranking of another, and within SELECT_CHUNK_BYTES of sort scratch.
inline CallPlan plan_rows(const CallShape& s, const Hooks& h) {
    CallPlan p;
    const int k = p.k_out = (int)std::min<int64_t>(s.k, s.n_pos);
    if (s.n_rows == 0 || k <= 0) return p;  // nothing to rank
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_topk: object_rows: " + why;
        return p;
    };
    if (s.d != s.n_objects)
        return refuse(B200_E_INVALID, "a stored row is a score row only when d == n_objects (d=" + std::to_string(s.d) +
                                          ", n_objects=" + std::to_string(s.n_objects) + ")");
    if (s.cosine) return refuse(B200_E_UNSUPPORTED, "COSINE engines score through the object norms, not the stored rows");
    if (s.id_offset) return refuse(B200_E_UNSUPPORTED, "engines with an id offset hold one shard of the catalogue");
    if (s.flags & B200_Q_SHARED_THRESHOLDS) return refuse(B200_E_UNSUPPORTED, "B200_Q_SHARED_THRESHOLDS has no thresholds to share here");
    if (s.flags & B200_Q_FORCE_TC) return refuse(B200_E_UNSUPPORTED, "no tensor-core pass ranks stored rows (B200_Q_FORCE_TC)");
    p.path = Path::ROWS;
    p.select = Select::RADIX;
    p.chunk = s.n_rows;
    const int64_t want = h.chunk_rows > 0 ? h.chunk_rows : 8 * (int64_t)(s.sm_count / 2) * 256;
    if (s.n_rows >= 2 * want) p.chunk = want;
    if (const int64_t bytes = rows_row_bytes(k)) p.chunk = std::min(p.chunk, std::max<int64_t>(1, SELECT_CHUNK_BYTES / bytes));
    p.n_chunks = (s.n_rows + p.chunk - 1) / p.chunk;
    return p;
}

inline CallPlan plan_call(const CallShape& s, const Hooks& h) {
    if (s.rows) return plan_rows(s, h);
    CallPlan p;
    const int k = p.k_out = (int)std::min<int64_t>(s.k, s.n_pos);
    if (s.n_rows == 0 || k <= 0) return p;  // nothing to rank
    p.bf16 = s.tc_dtype == B200_TC_BF16;
    const bool shared = s.flags & B200_Q_SHARED_THRESHOLDS;
    const bool wide = k > 24 && k <= 128 && h.wide != 0;
    // 128 < k <= 1024: the same single wide pass with longer append lists and a large-k re-score, when the expected
    // candidate count stays well inside the catalogue (k = None and near-catalogue requests keep path 3).  Item-sharded
    // calls that share thresholds need k <= 24 and keep path 3 here as well.
    const bool wide_l = k > 128 && k <= 1024 && h.wide != 0 && !s.sparse && !shared && wide_geom(k, h).T <= 0.5 * (double)s.n_pos;

    // Candidates kept per list by the tensor-core pass (K' >= k / lists; the surplus is the certificate's safety margin).
    // A row has two lists, one per column group of the tile stream, so a small surplus per list already gives ~2k
    // candidates; rows where (nearly) all of the top-k fall into one column group fail the certificate and take the
    // second-chance pass.  Inserts, the dominant epilogue cost, scale with K'.
    int k_cand = 0;
    if (k <= 24) {
        const int surplus = p.bf16 ? std::max(6, k / 2) : std::max(2, k / 4);
        k_cand = std::min(32, k + surplus);
    } else if (k <= 128) {
        k_cand = wide ? 24 : (p.bf16 ? 30 : 25);  // wide: adaptive lists of phase 1;  else passes of 20
    } else if (wide_l) {
        k_cand = 32;  // the full 32 slots: the frozen threshold samples ~58 ranks instead of ~42
    }
    if (shared && s.n_peers > 0 && k <= 24) {
        // Shared thresholds: the pruning bound of a row is the MAXIMUM over all L = ranks x lists list minima, i.e. the
        // largest K'-th best of L samples of N/L objects -- about global rank L K' - c_L L sqrt(K') (c_L = expected maximum
        // of L standard normals).  The certificate needs that rank to stay above k plus a margin; everything beyond is
        // wasted insertions (K' = 12 on 8 ranks sits near rank 100, K' = 6 near rank 27).
        const int L = (s.n_peers + 1) * 2;
        const double cL = L <= 2 ? 0.56 : L <= 4 ? 1.03 : L <= 8 ? 1.42 : L <= 16 ? 1.77 : L <= 32 ? 2.07 : 2.33;
        const double target = k + std::max(12.0, 0.6 * k) + (p.bf16 ? 20.0 : 0.0);
        int kc = 4;
        while (kc < 32 && L * kc - cL * L * std::sqrt((double)kc) < target) ++kc;
        k_cand = kc;
    }
    const int forced = h.tc_kcand;
    if (forced >= 4 && forced <= 32 && (forced >= k || wide || wide_l || shared)) k_cand = forced;

    bool use_tc = !s.sparse && s.tc_dtype != B200_TC_OFF && k_cand > 0 && !(s.flags & B200_Q_FORCE_EXACT) &&
                  s.n_pos >= (int64_t)k_cand * 4;
    // tiny problems are cheaper (and exercised) on the exhaustive kernel
    if (use_tc && !(s.flags & B200_Q_FORCE_TC) && (double)s.n_rows * (double)s.n_pos < 4.0e6) use_tc = false;
    auto refuse = [&](const std::string& why) {
        p.error = B200_E_UNSUPPORTED;
        p.message = "b200_rank_topk: " + why;
        return p;
    };
    if (use_tc && (size_t)SEL_WARPS * s.d * sizeof(float) > 64 * 1024) return refuse("d too large for the re-score kernel");
    if ((s.flags & B200_Q_FORCE_TC) && !use_tc)
        return refuse("tensor-core path unavailable (tc_dtype=" + std::to_string(s.tc_dtype) + ", k=" + std::to_string(k) +
                      ", d_pad=" + std::to_string(s.d_pad) + ", n_pos=" + std::to_string(s.n_pos) + ")");
    if (shared && use_tc && k > 24) return refuse("B200_Q_SHARED_THRESHOLDS needs k <= 24");

    p.path = s.sparse ? Path::SPARSE : use_tc ? Path::TC : k > 128 ? Path::DENSE_LARGE_K : Path::EXACT;
    if ((p.path == Path::SPARSE || p.path == Path::DENSE_LARGE_K) && (h.select == 2 || (h.select != 0 && k > 1024)))
        p.select = Select::RADIX;
    p.chunk = s.n_rows;
    if (p.tc()) {
        p.mode = wide ? TcMode::WIDE : wide_l ? TcMode::WIDE_L : k > 24 ? TcMode::MULTI_PASS : TcMode::NARROW;
        p.peers = shared;  // (zero peers: the same protocol, nothing to adopt)
        // every route above keeps K' within a list: the kernel's lists have no room for more
        if (k_cand > LIST_SLOTS) return refuse("K' = " + std::to_string(k_cand) + " exceeds the candidate-list capacity");
        p.k_cand = k_cand;
        if (p.wide()) p.geom = wide_geom(k, h);
        const int64_t wave = (int64_t)(s.sm_count / 2) * 256;  // subject rows one wave of CTA pairs works on
        if (!(s.flags & B200_Q_INPUTS_ON_DEVICE) && p.mode != TcMode::MULTI_PASS) {
            // host inputs: row chunks let the copies of one chunk overlap the ranking of another
            const int64_t want = h.chunk_rows > 0 ? h.chunk_rows : 8 * wave;
            if (s.n_rows >= 2 * want) p.chunk = want;
        }
        if (p.mode == TcMode::WIDE_L) {
            // the append lists take lists x cand_stride x 8 B per row (~21 GB for 1M rows at k = 1000): row chunks keep them
            // within the budget, for device inputs too.  Whole waves of CTA pairs where the budget allows.
            const int64_t per_row = (int64_t)2 * p.geom.cand_stride * 8;
            const int64_t budget = (int64_t)h.wide_budget_mb << 20;
            int64_t fit = std::max<int64_t>(256, budget / per_row / 256 * 256);
            if (fit >= wave) fit = fit / wave * wave;
            p.chunk = std::min(p.chunk, fit);
        }
    }
    p.n_chunks = (s.n_rows + p.chunk - 1) / p.chunk;
    return p;
}

// ---- path 5: candidate sets (b200_rank_topk_candidates).  Row r is scored against its own ascending object ids
// cand_indices[cand_indptr[r] .. cand_indptr[r+1]): cand_score_kernel writes one fp32 score per candidate into a ragged
// buffer, cand_select_kernel selects from it.  A row chunk holds, per row, its 4 B scores, 16 B of sort scratch per
// candidate when k_out > LK_SMEM_PAIRS (a row sorts at most |C_r| survivors; the scratch is addressed by candidate) and its
// 8 B x k_out of device outputs -- within SELECT_CHUNK_BYTES, the 1 GiB rule of paths 2-4.
struct CandShape {
    int64_t n_rows = 0;
    int64_t n_objects = 0;
    int64_t k = 0;           // requested k
    int d = 0;
    int32_t flags = 0;       // B200_Q_*
    bool whitelist = false;  // query.whitelist given
    bool sparse = false;     // query.sub_* given
    bool rows = false;       // query.object_rows given
    bool res_device = false; // the batch reads resident subjects that live in device memory
    bool id_offset = false;  // the engine has a non-zero id offset
};

// Largest subject row cand_score_kernel stages in shared memory (fp32 elements).
constexpr int64_t CAND_MAX_D = 48 * 1024;

inline int64_t cand_row_bytes(int64_t len, int64_t k_out) {
    return 4 * len + (k_out > LK_SMEM_PAIRS ? 16 * len : 0) + 8 * k_out;
}

struct CandPlan {
    int k_out = 0;
    std::vector<int64_t> bounds;  // chunk c = rows [bounds[c], bounds[c + 1])
    int64_t max_chunk_cands = 0;  // candidates of the largest chunk (score buffer, sort scratch)
    int64_t max_chunk_rows = 0;
    int error = B200_OK;
    std::string message;
    int64_t n_chunks() const { return bounds.empty() ? 0 : (int64_t)bounds.size() - 1; }
};

// The candidate-row-pointer checks and the row chunks of a call that passed its refusals (`p` holds its k_out).  Chunks
// take whole rows, in order, while the bytes `row_bytes(len)` of their rows stay within `budget` and their rows within
// B200_CHUNK_ROWS when it is set; a row that alone exceeds the budget is refused with B200_E_NOMEM.  `who` prefixes the
// messages.
template <typename RowBytes>
inline CandPlan cand_chunks(CandPlan p, int64_t n_rows, const int64_t* indptr, const Hooks& h, int64_t budget, const std::string& who,
                            RowBytes row_bytes) {
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = who + why;
        return p;
    };
    if (!indptr) return refuse(B200_E_INVALID, "cand_indptr is NULL");
    if (indptr[0] < 0) return refuse(B200_E_INVALID, "cand_indptr[0] < 0");
    for (int64_t r = 0; r < n_rows; ++r)
        if (indptr[r + 1] < indptr[r])
            return refuse(B200_E_INVALID, "cand_indptr is not monotone at row " + std::to_string(r));
    const int64_t max_rows = h.chunk_rows > 0 ? h.chunk_rows : n_rows;
    p.bounds.push_back(0);
    int64_t bytes = 0, cands = 0, rows = 0;
    for (int64_t r = 0; r < n_rows; ++r) {
        const int64_t len = indptr[r + 1] - indptr[r], b = row_bytes(len);
        if (b > budget)
            return refuse(B200_E_NOMEM, "row " + std::to_string(r) + " (" + std::to_string(len) + " candidates, k_out = " +
                                            std::to_string(p.k_out) + ") needs " + std::to_string(b) + " bytes, more than a chunk's " +
                                            std::to_string(budget));
        if (rows > 0 && (bytes + b > budget || rows == max_rows)) {
            p.bounds.push_back(r);
            p.max_chunk_cands = std::max(p.max_chunk_cands, cands);
            p.max_chunk_rows = std::max(p.max_chunk_rows, rows);
            bytes = cands = rows = 0;
        }
        bytes += b;
        cands += len;
        ++rows;
    }
    p.bounds.push_back(n_rows);
    p.max_chunk_cands = std::max(p.max_chunk_cands, cands);
    p.max_chunk_rows = std::max(p.max_chunk_rows, rows);
    return p;
}

// The refusals, the candidate-row-pointer check and the row chunks of one call.  `indptr` (host, [n_rows + 1]) is read
// only after the refusals.  Chunks take whole rows, in order, while their bytes stay within `budget` and their rows within
// B200_CHUNK_ROWS when it is set; a row that alone exceeds the budget is refused with B200_E_NOMEM.
inline CandPlan plan_candidates(const CandShape& s, const int64_t* indptr, const Hooks& h, int64_t budget = SELECT_CHUNK_BYTES) {
    CandPlan p;
    p.k_out = (int)std::min<int64_t>(s.k, s.n_objects);
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_topk_candidates: " + why;
        return p;
    };
    if (s.flags & (B200_Q_INPUTS_ON_DEVICE | B200_Q_OUTPUTS_ON_DEVICE))
        return refuse(B200_E_UNSUPPORTED, "candidate sets take host inputs and outputs only");
    if (s.res_device) return refuse(B200_E_UNSUPPORTED, "resident subjects in device memory are not read here");
    if (s.sparse) return refuse(B200_E_UNSUPPORTED, "sparse subjects (sub_*) are not ranked against candidate sets");
    if (s.rows) return refuse(B200_E_UNSUPPORTED, "stored rows (object_rows) are not ranked against candidate sets");
    if (s.whitelist) return refuse(B200_E_UNSUPPORTED, "a global whitelist is not taken: intersect it into the candidate lists");
    if (s.flags & B200_Q_SHARED_THRESHOLDS) return refuse(B200_E_UNSUPPORTED, "B200_Q_SHARED_THRESHOLDS has no thresholds to share here");
    if (s.flags & B200_Q_FORCE_TC) return refuse(B200_E_UNSUPPORTED, "no tensor-core pass scores candidate sets (B200_Q_FORCE_TC)");
    if (s.id_offset) return refuse(B200_E_UNSUPPORTED, "engines with an id offset hold one shard of the catalogue");
    if (s.d > CAND_MAX_D) return refuse(B200_E_UNSUPPORTED, "d = " + std::to_string(s.d) + " exceeds the staged subject row's limit");
    if (s.n_rows == 0 || p.k_out <= 0) return p;  // nothing to rank
    return cand_chunks(p, s.n_rows, indptr, h, budget, "b200_rank_topk_candidates: ",
                       [&](int64_t len) { return cand_row_bytes(len, p.k_out); });
}

// ---- path 5 from device memory (b200_rank_topk_candidates_device).  The raw lists are any int32 ids in any order: a
// preparation pass sorts each row, drops ids outside [0, n_objects) and repeats, and the kernels above rank what is left.
// Chunks are planned on the raw lengths, which bound the prepared ones from above.  Per raw entry: 4 B of prepared ids and
// 4 B of scores, 16 B of preparation scratch when the row is longer than LK_SMEM_PAIRS (it sorts in global memory), 16 B
// of selection scratch when k_out > LK_SMEM_PAIRS; plus 8 B x k_out per row of staged outputs when they go to the host.
inline int64_t cand_device_row_bytes(int64_t len, int64_t k_out, bool host_out) {
    return 8 * len + (len > LK_SMEM_PAIRS ? 16 * len : 0) + (k_out > LK_SMEM_PAIRS ? 16 * len : 0) + (host_out ? 8 * k_out : 0);
}

// The refusals of a device call that need no array (B200_OK: none); s.res_device is no refusal here.
inline CandPlan refuse_candidates_device(const CandShape& s) {
    CandPlan p;
    p.k_out = (int)std::min<int64_t>(s.k, s.n_objects);
    auto refuse = [&](int code, const std::string& why) {
        p.error = code;
        p.message = "b200_rank_topk_candidates_device: " + why;
        return p;
    };
    if (!(s.flags & B200_Q_INPUTS_ON_DEVICE))
        return refuse(B200_E_INVALID, "needs B200_Q_INPUTS_ON_DEVICE: host candidate lists go to b200_rank_topk_candidates");
    if (s.sparse) return refuse(B200_E_UNSUPPORTED, "sparse subjects (sub_*) are not ranked against candidate sets");
    if (s.rows) return refuse(B200_E_UNSUPPORTED, "stored rows (object_rows) are not ranked against candidate sets");
    if (s.whitelist) return refuse(B200_E_UNSUPPORTED, "a global whitelist is not taken: mask it into the candidate lists");
    if (s.flags & B200_Q_SHARED_THRESHOLDS) return refuse(B200_E_UNSUPPORTED, "B200_Q_SHARED_THRESHOLDS has no thresholds to share here");
    if (s.flags & B200_Q_FORCE_TC) return refuse(B200_E_UNSUPPORTED, "no tensor-core pass scores candidate sets (B200_Q_FORCE_TC)");
    if (s.id_offset) return refuse(B200_E_UNSUPPORTED, "engines with an id offset hold one shard of the catalogue");
    if (s.d > CAND_MAX_D) return refuse(B200_E_UNSUPPORTED, "d = " + std::to_string(s.d) + " exceeds the staged subject row's limit");
    return p;
}

// The refusals, the row-pointer checks and the row chunks of one device call.  `indptr` is the host copy of the device
// cand_indptr ([n_rows + 1], any base), read only after the refusals.
inline CandPlan plan_candidates_device(const CandShape& s, const int64_t* indptr, const Hooks& h, int64_t budget = SELECT_CHUNK_BYTES) {
    const CandPlan p = refuse_candidates_device(s);
    if (p.error != B200_OK || s.n_rows == 0 || p.k_out <= 0) return p;  // refused, or nothing to rank
    const bool host_out = !(s.flags & B200_Q_OUTPUTS_ON_DEVICE);
    return cand_chunks(p, s.n_rows, indptr, h, budget, "b200_rank_topk_candidates_device: ",
                       [&](int64_t len) { return cand_device_row_bytes(len, p.k_out, host_out); });
}

// The candidate ids of rows [0, n_rows): in [0, n_objects) and strictly ascending within a row.  B200_OK, or
// B200_E_INVALID with the first offending row in `message`.
inline int check_candidate_ids(const int64_t* indptr, const int32_t* indices, int64_t n_rows, int64_t n_objects, std::string& message) {
    if (indptr[n_rows] > indptr[0] && !indices) {
        message = "b200_rank_topk_candidates: cand_indices is NULL";
        return B200_E_INVALID;
    }
    for (int64_t r = 0; r < n_rows; ++r) {
        for (int64_t e = indptr[r]; e < indptr[r + 1]; ++e) {
            const int32_t id = indices[e];
            if (id < 0 || id >= n_objects) {
                message = "b200_rank_topk_candidates: row " + std::to_string(r) + ": candidate " + std::to_string(id) +
                          " is not an object of this engine (n_objects = " + std::to_string(n_objects) + ")";
                return B200_E_INVALID;
            }
            if (e > indptr[r] && id <= indices[e - 1]) {
                message = "b200_rank_topk_candidates: row " + std::to_string(r) + ": candidate ids are not strictly ascending";
                return B200_E_INVALID;
            }
        }
    }
    return B200_OK;
}

}  // namespace b200
