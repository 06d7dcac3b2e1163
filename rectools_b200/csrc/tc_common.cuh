// sm_90a building blocks of the fused scoring + candidate-selection kernel (fused_topk.cuh): wgmma / TMA / mbarrier
// PTX wrappers, the kernel parameter block, and the per-row selection state of the epilogue
// (candidate lists in shared memory, filter_pairs_csr merge cursor, exclusion cursor, register-chunk helpers).
//
// The code built from these pieces replaces `scores = query @ items.T` + mask + select of implicit's top-k (call site
// rectools/models/rank/rank_implicit.py:264-272, :175-182) and `TorchRanker.rank`'s batched matmul / masked_fill /
// torch.topk (rectools/models/rank/rank_torch.py:133-152) as a CANDIDATE generator; exact scores, the final order and
// the certificate come from select.cuh.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace b200 {
namespace tc {

constexpr int TILE_M = 128;                // subject rows per CTA
constexpr int TILE_N = 256;                // objects per tile (scored in four quarters of QUART_N)
constexpr int QUART_N = 64;                // objects per MMA pass, object block and accumulator staging
constexpr int HALF_N = 128;                // object rows the resident 16-bit copy is padded to
constexpr int KBLK = 64;                   // 16-bit elements per shared-memory block row (128 B, one swizzle atom)
constexpr int BLK_BYTES = 128 * KBLK * 2;  // 16 KiB: [128 subject rows][128 B]
constexpr int OBJ_BLK_BYTES = QUART_N * KBLK * 2;  // 8 KiB: [64 object rows][128 B], one ring stage
constexpr int STG_STRIDE = QUART_N + 4;    // floats per staged accumulator row (+4: conflict-free 16-byte row reads)
constexpr int STG_BYTES = TILE_M * STG_STRIDE * 4;
constexpr int MAX_STAGES = 16;
constexpr int SMEM_LIMIT = 232448;  // 227 KiB
constexpr int MAX_PEERS = 8;        // ranks sharing pruning thresholds over NVLink peer memory (multi-GPU item sharding)

struct TcParams {
    int32_t kblocks;          // d_pad / 64
    int32_t n_stages;         // object ring depth (blocks of 8 KiB)
    int32_t k_cand;           // K': slots used per candidate list (<= the kernel's list capacity)
    int64_t n_rows;           // valid subject rows
    int64_t n_pos;            // valid object positions
    int32_t n_row_tiles;      // tiles of 256 subject rows (one per CTA pair)
    int32_t n_splits;
    int32_t n_obj_tiles;
    int32_t tiles_per_split;
    const int32_t* pos2obj;   // nullable whitelist map
    const int64_t* indptr;    // nullable CSR filter by subject row
    const int32_t* indices;
    const int32_t* row_ids;   // nullable: batch row -> row of the CSR filter (re-ranked subsets)
    const int32_t* excl;      // nullable: [rows][excl_stride] ids already returned by earlier passes, sorted ascending
    int32_t excl_stride;
    int32_t excl_n;           // ids per row in `excl` (rows with fewer results are padded with B200_PAD_ID)
    int32_t id_off;           // global id = local object id + id_off (CSR column ids are global)
    float* cand_scores;       // [n_lists][rows_pad][cand_stride]   (n_lists = n_splits * lists per row)
    int32_t* cand_ids;
    int32_t* cand_counts;     // [n_lists][rows_pad]: entries produced (may exceed cand_stride in append mode: overflow)
    float* cand_thr;          // [n_lists][rows_pad]: the list's final pruning threshold (bounds every discarded score)
    int64_t rows_pad;
    int32_t cand_stride;      // slots per list in the global arrays (32, or the append capacity)
    // wide mode (k > 24): the first `phase1_tiles` tiles of a work item keep adaptive K'-slot lists; then the threshold is
    // frozen and every later score above it is appended to the global list (no more list maintenance)
    int32_t phase1_tiles;     // >= tiles of a work item: never switch (plain adaptive lists)
    int32_t debug_mode;       // 0 = normal; 1 = no candidates (fast path only); 2 = epilogue skips the staged-accumulator reads (measurement hooks)
    // carousel: a work item starts streaming the objects where the other CTA pairs currently are, so that all pairs keep
    // reading the same few MB of the object matrix and the L2 serves most reads (nullptr: start at t0)
    int32_t* front;           // [n_splits] object tile most recently issued by the reference pair
    int32_t* starts;          // [n_pairs][starts_stride] start tile chosen for each work item (-1: not decided yet)
    int32_t starts_stride;
    // pruning thresholds shared between the ranks of an item-sharded catalogue (NVLink peer memory): every rank publishes,
    // per subject row of the call, (epoch, threshold in units of 2^row_exp) and adopts the maximum of its peers' values --
    // any rank's K'-th best score is a lower bound of the global one
    int32_t n_peers;                         // 0: off
    uint32_t peer_epoch;                     // tag of this call (same on every rank)
    int32_t peer_exp;                        // this engine's object exponent: published = thr * 2^-peer_exp
    int64_t peer_row0;                       // absolute row of batch row 0 inside the published arrays
    unsigned long long* peer_pub;            // this rank's array [rows of the call]
    const unsigned long long* peer_in[MAX_PEERS];  // the other ranks' arrays (peer-mapped)
};

// ------------------------------------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Wait for the phase with the given parity to complete.  A watchdog turns a protocol bug into a trap, not a hang
// (a failed try_wait already suspends the thread for a few hundred cycles, so 2^24 failures are seconds).
__device__ __forceinline__ uint32_t mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    return done;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity))
        if (++spins > (1u << 24)) __trap();
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1)
        : "memory");
}

// Shared-memory matrix descriptor of a K-major operand block: 128-byte rows, SWIZZLE_128B, 8-row groups 1024 B apart.
//   lo: bits [0,14) start address >> 4, bits [16,30) leading byte offset >> 4 (ignored for swizzled K-major: 1)
//   hi: bits [0,14) stride byte offset >> 4 (1024 >> 4), bits [30,32) layout 1 (128-byte swizzle)
__device__ __forceinline__ uint32_t smem_desc_lo(uint32_t saddr) { return ((saddr & 0x3FFFF) >> 4) | (1u << 16); }
constexpr uint32_t SMEM_DESC_HI = (1024u >> 4) | (1u << 30);

// Hand registers of this warp group back to the CTA / take them (all four warps execute it together).
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// Pin the accumulator registers at this point of the instruction stream (before wgmma.fence, after wgmma.wait_group:
// never while a wgmma that writes them is in flight, or ptxas drains the pipe there).  The accumulators are b32
// registers from the wgmma to the staging store, so no type conversion ever copies one.
template <int N>
__device__ __forceinline__ void fence_acc(uint32_t (&r)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x 64] (+)= A[64 x 16] * B[64 x 16]^T, both operands K-major in shared memory, fp32 accumulators in registers
// (warp w of the warp group, lane l holds rows 16 w + l / 4 (+ 8) and columns 8 j + 2 (l % 4) (+ 1) of D).  The fp32
// accumulators are bound as b32 registers ("+r"), the type the staging store reads them in.
#define B200_F8(a, n) "+r"(a[n]), "+r"(a[n + 1]), "+r"(a[n + 2]), "+r"(a[n + 3]), "+r"(a[n + 4]), "+r"(a[n + 5]), "+r"(a[n + 6]), "+r"(a[n + 7])
#define B200_WGMMA_64x64(TYPE)                                                                                              \
    asm volatile(                                                                                                           \
        "{\n\t.reg .pred p;\n\t.reg .b64 da, db;\n\t"                                                                       \
        "mov.b64 da, {%32, %34};\n\t"                                                                                       \
        "mov.b64 db, {%33, %34};\n\t"                                                                                       \
        "setp.ne.b32 p, %35, 0;\n\t"                                                                                        \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPE "." TYPE " "                                                     \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "                                           \
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, da, db, p, 1, 1, 0, 0;\n\t}"     \
        : B200_F8(d, 0), B200_F8(d, 8), B200_F8(d, 16), B200_F8(d, 24)                                                      \
        : "r"(a_lo), "r"(b_lo), "r"(SMEM_DESC_HI), "r"(accum))
// (the operand type is a template parameter: a run-time branch around each wgmma makes ptxas serialise the pipeline)
template <bool BF16>
__device__ __forceinline__ void wgmma_64x64(uint32_t (&d)[32], uint32_t a_lo, uint32_t b_lo, uint32_t accum) {
    if constexpr (BF16)
        B200_WGMMA_64x64("bf16");
    else
        B200_WGMMA_64x64("f16");
}
#undef B200_WGMMA_64x64
#undef B200_F8

// One epilogue thread's row of a staged accumulator quarter: 64 fp32 columns, 16-byte loads.
__device__ __forceinline__ void stage_ld(uint32_t a, uint32_t (&r)[64]) {
#pragma unroll
    for (int j = 0; j < 16; ++j)
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                     : "=r"(r[4 * j]), "=r"(r[4 * j + 1]), "=r"(r[4 * j + 2]), "=r"(r[4 * j + 3])
                     : "r"(a + 16 * j)
                     : "memory");
}

__device__ __forceinline__ float max3(float a, float b, float c) { return fmaxf(fmaxf(a, b), c); }
__device__ __forceinline__ float fu(uint32_t x) { return __uint_as_float(x); }

// Pin a loop-invariant value in a register: without this the compiler re-derives shared-memory / TMEM addresses from
// %tid, the shared window base and the kernel parameters in every tile iteration (~45 instructions per tile measured)
// instead of spending a register on them.
__device__ __forceinline__ uint32_t pin(uint32_t x) {
    uint32_t y;
    asm volatile("mov.u32 %0, %1;" : "=r"(y) : "r"(x));
    return y;
}

// ------------------------------------------------------------------------------------------------ shared-memory accessors
__device__ __forceinline__ float lds_f32(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ int lds_s32(uint32_t a) {
    int v;
    asm volatile("ld.shared.s32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_s32(uint32_t a, int v) { asm volatile("st.shared.s32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_v2(uint32_t a, float x, uint32_t y) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(__float_as_uint(x)), "r"(y) : "memory");
}
__device__ __forceinline__ void sts_v2(uint32_t a, uint32_t x, uint32_t y) {
    asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void lds_v2(uint32_t a, float& x, uint32_t& y) {
    uint32_t xb;
    asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(xb), "=r"(y) : "r"(a) : "memory");
    x = __uint_as_float(xb);
}
// (work-item tag, threshold) pairs exchanged between the threads that scan the column groups of one row
__device__ __forceinline__ void sts_thr(uint32_t a, uint32_t tag, float thr) {
    asm volatile("{\n\t.reg .b64 t;\n\tmov.b64 t, {%1, %2};\n\tst.volatile.shared.b64 [%0], t;\n\t}"
                 ::"r"(a), "r"(__float_as_uint(thr)), "r"(tag)
                 : "memory");
}
__device__ __forceinline__ void lds_thr(uint32_t a, uint32_t& tag, float& thr) {
    uint32_t tb;
    asm volatile("{\n\t.reg .b64 t;\n\tld.volatile.shared.b64 t, [%2];\n\tmov.b64 {%0, %1}, t;\n\t}"
                 : "=r"(tb), "=r"(tag)
                 : "r"(a)
                 : "memory");
    thr = __uint_as_float(tb);
}
// (epoch, threshold) pairs published to / read from the other ranks: system scope, never cached in L1
__device__ __forceinline__ void stg_peer(unsigned long long* a, uint32_t epoch, float thr) {
    const unsigned long long v = ((unsigned long long)epoch << 32) | (unsigned long long)__float_as_uint(thr);
    asm volatile("st.relaxed.sys.global.b64 [%0], %1;" ::"l"(a), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ldg_peer(const unsigned long long* a) {
    unsigned long long v;
    asm volatile("ld.relaxed.sys.global.b64 %0, [%1];" : "=l"(v) : "l"(a) : "memory");
    return v;
}

// ------------------------------------------------------------------------------------------------ per-row selection state
// Registers of the thread that owns a (row, column group) of the tile stream.
struct RowState {
    float thr;    // pruning threshold: smallest entry of the full list, or a bound adopted from the row's other lists / ranks
    int cnt;      // entries produced (<= K' while the list is adaptive; keeps counting in append mode)
    int minpos;   // slot of the smallest entry once the list is full
    int nv;       // next viewed global object id >= the stream position (B200_PAD_ID when the CSR row is exhausted)
    int64_t cur;  // index of `nv` in csr indices
    int64_t fhi;  // end of the row's CSR slice
    // multi-pass ranking: objects returned by earlier passes are excluded the same way
    const int32_t* xrow;  // this row's sorted exclusion list (nullptr: none)
    int xcur, xnv;        // cursor / next excluded global object id
};

// Candidate lists live in shared memory as [slot][lane]: the thread that owns a row reads and writes only its own
// column (bank = lane, conflict-free), so all 32 rows of a warp can take candidates at the same time.
// Keep the K' best (score, id) pairs of a row: append while the list is short, afterwards overwrite the current
// minimum and re-scan for the new one (K' independent shared-memory loads; runs for all rows of the warp in parallel).
// ls / li = shared addresses of slot 0 of this thread's column in the score / id arrays.
__device__ __forceinline__ void list_insert(uint32_t ls, uint32_t li, int kc, RowState& rs, float val, int obj) {
    const int slot = rs.cnt < kc ? rs.cnt : rs.minpos;
    sts_f32(ls + slot * 128, val);
    sts_s32(li + slot * 128, obj);
    if (rs.cnt < kc && ++rs.cnt < kc) return;
    float mn = INFINITY;
    int mp = 0;
#pragma unroll 8
    for (int e = 0; e < kc; ++e) {
        const float x = lds_f32(ls + e * 128);
        if (x < mn) {
            mn = x;
            mp = e;
        }
    }
    rs.minpos = mp;
    rs.thr = fmaxf(rs.thr, mn);  // never loosen a bound borrowed from the row's other lists
}

// Merge cursor over the (short, <= k entries) sorted list of objects already returned by earlier passes.
__device__ __forceinline__ bool is_excluded(RowState& rs, int n, int g) {
    while (rs.xnv < g) {
        ++rs.xcur;
        rs.xnv = rs.xcur < n ? __ldg(rs.xrow + rs.xcur) : B200_PAD_ID;
    }
    return rs.xnv == g;
}

// Position the two cursors of a row at the first object (global id g_first) of a stream segment.
__device__ __forceinline__ void row_cursors_init(const TcParams& p, RowState& rs, int64_t frow, int g_first) {
    rs.nv = B200_PAD_ID;
    rs.cur = 0;
    rs.fhi = 0;
    rs.xrow = nullptr;
    rs.xcur = 0;
    rs.xnv = B200_PAD_ID;
    if (frow < 0) return;
    if (p.indptr) {
        int64_t lo = p.indptr[frow];
        rs.fhi = p.indptr[frow + 1];
        int64_t hi = rs.fhi;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (__ldg(p.indices + mid) < g_first)
                lo = mid + 1;
            else
                hi = mid;
        }
        rs.cur = lo;
        rs.nv = lo < rs.fhi ? __ldg(p.indices + lo) : B200_PAD_ID;
    }
    if (p.excl) {
        rs.xrow = p.excl + frow * p.excl_stride;
        int lo = 0, hi = p.excl_n;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (__ldg(rs.xrow + mid) < g_first)
                lo = mid + 1;
            else
                hi = mid;
        }
        rs.xcur = lo;
        rs.xnv = lo < p.excl_n ? __ldg(rs.xrow + lo) : B200_PAD_ID;
    }
}

// Per-thread view of the row's filter_pairs_csr slice: a window of four consecutive viewed ids starting at index `cur`
// (B200_PAD_ID past the end of the slice).  Candidates arrive in ascending id order, so a window is only ever moved
// forward; its loads are issued when a candidate turns out to lie beyond it and are consumed one step later
// (fifo_step), i.e. their latency is off the critical path.
struct CsrWindow {
    int64_t cur, fhi;
    int w0, w1, w2, w3;
    int streak;  // consecutive moves for the same candidate (long slices: switch to a binary search)
};

__device__ __forceinline__ void window_load(const int32_t* __restrict__ indices, CsrWindow& cw) {
    cw.w0 = cw.cur + 0 < cw.fhi ? __ldg(indices + cw.cur + 0) : B200_PAD_ID;
    cw.w1 = cw.cur + 1 < cw.fhi ? __ldg(indices + cw.cur + 1) : B200_PAD_ID;
    cw.w2 = cw.cur + 2 < cw.fhi ? __ldg(indices + cw.cur + 2) : B200_PAD_ID;
    cw.w3 = cw.cur + 3 < cw.fhi ? __ldg(indices + cw.cur + 3) : B200_PAD_ID;
}

// ------------------------------------------------------------------------------------------------ register-chunk helpers
// Maximum of the 32 staged scores r[OFF .. OFF+32) (11 three-input maxima + 1).
template <int OFF, int NR>
__device__ __forceinline__ float chunk_max(const uint32_t (&r)[NR]) {
    const float g0 = max3(max3(fu(r[OFF + 0]), fu(r[OFF + 1]), fu(r[OFF + 2])), max3(fu(r[OFF + 3]), fu(r[OFF + 4]), fu(r[OFF + 5])),
                          max3(fu(r[OFF + 6]), fu(r[OFF + 7]), fu(r[OFF + 8])));
    const float g1 = max3(max3(fu(r[OFF + 9]), fu(r[OFF + 10]), fu(r[OFF + 11])), max3(fu(r[OFF + 12]), fu(r[OFF + 13]), fu(r[OFF + 14])),
                          max3(fu(r[OFF + 15]), fu(r[OFF + 16]), fu(r[OFF + 17])));
    const float g2 = max3(max3(fu(r[OFF + 18]), fu(r[OFF + 19]), fu(r[OFF + 20])), max3(fu(r[OFF + 21]), fu(r[OFF + 22]), fu(r[OFF + 23])),
                          max3(fu(r[OFF + 24]), fu(r[OFF + 25]), fu(r[OFF + 26])));
    const float g3 = max3(max3(fu(r[OFF + 27]), fu(r[OFF + 28]), fu(r[OFF + 29])), fu(r[OFF + 30]), fu(r[OFF + 31]));
    return fmaxf(max3(g0, g1, g2), g3);
}

template <int OFF, int J0, int J1, int NR>
__device__ __forceinline__ unsigned group_mask(const uint32_t (&r)[NR], float thr) {
    unsigned m = 0;
#pragma unroll
    for (int j = J0; j < J1; ++j) m |= (fu(r[OFF + j]) > thr) ? (1u << j) : 0u;
    return m;
}

// Per-lane bit mask of the columns of chunk OFF above the row threshold; the mask of a 9-column group is built only
// when the group's maximum shows a hit somewhere in the warp.
template <int OFF, int NR>
__device__ __forceinline__ unsigned chunk_hits(const uint32_t (&r)[NR], float thr) {
    const float g0 = max3(max3(fu(r[OFF + 0]), fu(r[OFF + 1]), fu(r[OFF + 2])), max3(fu(r[OFF + 3]), fu(r[OFF + 4]), fu(r[OFF + 5])),
                          max3(fu(r[OFF + 6]), fu(r[OFF + 7]), fu(r[OFF + 8])));
    const float g1 = max3(max3(fu(r[OFF + 9]), fu(r[OFF + 10]), fu(r[OFF + 11])), max3(fu(r[OFF + 12]), fu(r[OFF + 13]), fu(r[OFF + 14])),
                          max3(fu(r[OFF + 15]), fu(r[OFF + 16]), fu(r[OFF + 17])));
    const float g2 = max3(max3(fu(r[OFF + 18]), fu(r[OFF + 19]), fu(r[OFF + 20])), max3(fu(r[OFF + 21]), fu(r[OFF + 22]), fu(r[OFF + 23])),
                          max3(fu(r[OFF + 24]), fu(r[OFF + 25]), fu(r[OFF + 26])));
    const float g3 = max3(max3(fu(r[OFF + 27]), fu(r[OFF + 28]), fu(r[OFF + 29])), fu(r[OFF + 30]), fu(r[OFF + 31]));
    unsigned hits = 0;
    if (__any_sync(B200_FULL_MASK, g0 > thr)) hits |= group_mask<OFF, 0, 9>(r, thr);
    if (__any_sync(B200_FULL_MASK, g1 > thr)) hits |= group_mask<OFF, 9, 18>(r, thr);
    if (__any_sync(B200_FULL_MASK, g2 > thr)) hits |= group_mask<OFF, 18, 27>(r, thr);
    if (__any_sync(B200_FULL_MASK, g3 > thr)) hits |= group_mask<OFF, 27, 32>(r, thr);
    return hits;
}

// r[OFF + j] for a run-time j without local memory: 5-level select tree (31 SEL).
template <int OFF, int NR>
__device__ __forceinline__ float chunk_select(const uint32_t (&r)[NR], int j) {
    uint32_t a[16], b[8], c[4], d[2];
    const bool b0 = j & 1, b1 = j & 2, b2 = j & 4, b3 = j & 8, b4 = j & 16;
#pragma unroll
    for (int i = 0; i < 16; ++i) a[i] = b0 ? r[OFF + 2 * i + 1] : r[OFF + 2 * i];
#pragma unroll
    for (int i = 0; i < 8; ++i) b[i] = b1 ? a[2 * i + 1] : a[2 * i];
#pragma unroll
    for (int i = 0; i < 4; ++i) c[i] = b2 ? b[2 * i + 1] : b[2 * i];
#pragma unroll
    for (int i = 0; i < 2; ++i) d[i] = b3 ? c[2 * i + 1] : c[2 * i];
    return fu(b4 ? d[1] : d[0]);
}

// Start tile of a work item: decided once by the even CTA's load-issuing thread (the current front of its object split),
// published through global memory, read by every other role of both CTAs of the pair.
__device__ __forceinline__ int carousel_start(const TcParams& p, int pair, uint32_t work_it, int split, int t0, int t1, bool decide) {
    if (p.front == nullptr) return t0;
    volatile int32_t* slot = p.starts + (size_t)pair * p.starts_stride + work_it;
    if (decide) {
        int s = *reinterpret_cast<volatile int32_t*>(p.front + split);
        s = min(max(s, t0), t1 - 1);
        *slot = s;
        __threadfence();
        return s;
    }
    int s;
    for (uint32_t spins = 0; (s = *slot) < 0; ++spins)
        if (spins > (1u << 26)) __trap();
    return s;
}

}  // namespace tc
}  // namespace b200
