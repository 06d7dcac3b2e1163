// The row split of an engine-group call (b200_rank_group_topk): which contiguous row slices the members pull, and how a
// host CSR array is cut to one slice.  Plain C++17 without CUDA headers, so that tests/test_engine_group_cpu.py compiles
// it with g++ alone and pins it.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdlib>

namespace b200 {

// A slice of a group call takes at least this many rows (unless the call has fewer): a member call has a fixed cost
// (staging, a synchronisation, the copy-back), and a slice this size still fills a wave of CTA pairs on an H100.
constexpr int64_t GROUP_MIN_SLICE = 32768;
// Slices per member: the members pull slices from one counter, so rows whose certificate fails (and that go to the
// re-rank passes) on one member are evened out by the others taking more slices.
constexpr int64_t GROUP_SLICES_PER_MEMBER = 4;

// B200_GROUP_SLICE_ROWS: forced slice size (tests: many small slices), read once per call; 0 = the default below.
inline int64_t read_group_slice_hook() {
    const char* v = std::getenv("B200_GROUP_SLICE_ROWS");
    return v ? std::max<int64_t>(0, std::atoll(v)) : 0;
}

// Rows per slice of a call of `n_rows` rows over `n_members` members.  A group of one ranks the whole batch in one call.
inline int64_t group_slice_rows(int64_t n_rows, int n_members, int64_t forced) {
    if (n_rows <= 0) return 1;
    if (forced > 0) return forced;
    if (n_members <= 1) return n_rows;
    const int64_t parts = GROUP_SLICES_PER_MEMBER * n_members;
    return std::max((n_rows + parts - 1) / parts, std::min(n_rows, GROUP_MIN_SLICE));
}

inline int64_t group_n_slices(int64_t n_rows, int64_t slice_rows) { return n_rows <= 0 ? 0 : (n_rows + slice_rows - 1) / slice_rows; }

struct GroupSlice {
    int64_t r0 = 0, r1 = 0;  // rows [r0, r1) of the call
};

inline GroupSlice group_slice(int64_t n_rows, int64_t slice_rows, int64_t i) {
    GroupSlice s;
    s.r0 = std::min(n_rows, i * slice_rows);
    s.r1 = std::min(n_rows, s.r0 + slice_rows);
    return s;
}

// A host CSR array cut to rows [r0, r1): `out` [r1 - r0 + 1] gets indptr[r0 .. r1] minus indptr[r0], and the returned
// base indptr[r0] is the offset of the slice's first entry in the indices / data arrays.  The engine stages a host CSR
// array from entry 0 up to indptr[n_rows], so a slice handed over without rebasing would copy every row before it.
inline int64_t rebase_indptr(const int64_t* indptr, int64_t r0, int64_t r1, int64_t* out) {
    const int64_t base = indptr[r0];
    for (int64_t r = r0; r <= r1; ++r) out[r - r0] = indptr[r] - base;
    return base;
}

}  // namespace b200
