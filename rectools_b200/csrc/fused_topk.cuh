// The fused scoring + candidate-selection kernel: one persistent CTA per SM, two CTAs (a "pair") per 256 subject rows.
//
//   TMA (own 128 subject rows once per work item; every 256-object tile as four quarters of 64 objects, streamed through a
//   ring of 8 KiB blocks) -> wgmma 64 x 64 x 16 (fp16 / bf16 -> fp32) into the registers of the MMA warp group
//   -> each finished quarter [128 rows x 64 columns] is staged in shared memory, one m-half of 64 rows at a time, and
//   read back by the epilogue warps, one row per thread; a staged half is handed back as soon as its rows are in registers.
//   Only the 16-row slices (one MMA warp's) with a score above their row's threshold are stored: a flag per slice tells
//   the epilogue which rows of the buffer hold the current quarter (store_half)
//   -> threshold scan (3-input max tree), hits extracted into per-thread ring FIFOs in shared memory
//   -> deferred, bounded steps: filter_pairs_csr lookup through a prefetched 4-entry window, candidate-list insertion.
// Score rows never reach HBM: only the K' best (score, id) pairs per row and column group are written.
//
// Warps 0-3: the MMA warp group; warps 4-11: the eight epilogue warps; warp 12: the producer (one thread issues every TMA
// load, and a ring slot returns to it through its `empty` barrier); with PEERS two more warps poll the other ranks' published thresholds over NVLink and publish this rank's.  Epilogue warp w reads
// the row quarter w & 3 of column group w >> 2: group g of a tile is made of its quarters g and g + 2 (128 columns), and
// each group has its own candidate list per row (two lists of 32 slots).
// The two CTAs of a pair work on the same object tiles in the same order; the odd CTA waits for the start tile the even
// one publishes through global memory, so the pair is launched as a cluster of two (co-scheduled by the hardware).
//
// Three selection modes share the epilogue:
//   * adaptive lists (k <= 24): replace-minimum lists of K' slots, the list minimum is the running threshold;
//   * wide mode (24 < k <= 1024): adaptive lists for the first `phase1_tiles` tiles of the stream, then the threshold is
//     FROZEN and every later score above it is appended to a global list -- ~1.5 k candidates per row in ONE pass with
//     ~3x fewer hits than adaptive lists of that size would take;
//   * shared thresholds (item-sharded multi-GPU): the row's threshold is the maximum over all ranks' thresholds.
// In every mode a list's final threshold bounds every score the list ever discarded: the certificate of select.cuh.
//
// Replaces the same reference code as named in tc_common.cuh (rank_implicit.py:264-272 / rank_torch.py:133-152).
#pragma once
#include "sizes.h"
#include "tc_common.cuh"

namespace b200 {
namespace tc {

constexpr uint32_t TAG_NONE = 0xffffffffu, TAG_DONE = 0xfffffffeu;  // exchange-slot tags no work item carries

struct FusedCfg {
    static constexpr int EPI0 = 4;                    // first epilogue warp; (warp & 3) is its row quarter
    static constexpr int EPILOGUE_WARPS = 8;          // epilogue warps
    static constexpr int PRODUCER = EPI0 + EPILOGUE_WARPS;  // the TMA warp
    static constexpr int HELPERS = 2;                 // peer-threshold warps behind the producer (PEERS kernels only)
    __host__ __device__ static constexpr int threads(bool peers) { return (PRODUCER + 1 + (peers ? HELPERS : 0)) * 32; }
    // Registers per thread.  The register file is split over the SM's four sub-partitions (warp w runs on w mod 4); with
    // 13-15 warps one of them holds four, so a thread gets 128 at launch.  setmaxnreg moves them within the CTA's
    // allocation: the MMA warp group drops to 96, the two epilogue warp groups rise to 144 (96 + 2 x 144 + 128 = 4 x 128
    // on the sub-partition with the producer); the producer and helper warps, no whole warp group, keep 128.
    static constexpr int REGS_LAUNCH = 128, REGS_MMA = 96, REGS_EPILOGUE = 144;
    static_assert(REGS_MMA + 2 * REGS_EPILOGUE + REGS_LAUNCH <= 4 * REGS_LAUNCH, "register plan of DESIGN section 5");
    static constexpr int COLS = 128;                  // accumulator columns per epilogue thread and tile
    static constexpr int NLIST = 2;                   // column groups = candidate lists per row
    static constexpr int NQ = COLS / QUART_N;         // staged quarters per epilogue thread and tile
    static constexpr int SLOTS = LIST_SLOTS;          // list capacity (K' <= SLOTS)
    static constexpr int Q = 8;                       // deferred hits per thread (ring FIFO)
    static constexpr int QSTRIDE = EPILOGUE_WARPS * 32 * 8;  // bytes between FIFO slots: [slot][epilogue thread] x (score, position)
    static constexpr int QBYTES = Q * QSTRIDE;
    static constexpr int BACKLOG = 4;                 // a row with this many pending hits gets a step at once
    static constexpr int PERIOD = 16;                 // otherwise deferred work runs every PERIOD-th tile (power of two)
    static constexpr int LIST_BYTES = NLIST * TILE_M * SLOTS * 4;  // one of the two arrays (scores / ids): 32 KiB
    static constexpr int THR_BYTES = (NLIST + 1) * TILE_M * 8;     // (tag, threshold) per list + one slot for the peers' maximum
    static constexpr int FIXED_BYTES = STG_BYTES + 2 * LIST_BYTES + QBYTES + THR_BYTES + 1024 /*alignment slack*/ + 512 /*barriers*/;
};

#ifdef B200_FUSED_PROFILE
// Measurement build only: clock64() cycles summed over the CTAs of every launch (b200_rank_fused_profile reads and
// clears them).  Thread 0 of the MMA warp group measures its waits on `full` (TMA / L2), on `qempty` (the hand-off), in
// wgmma.wait_group (the tensor pipe), and the pass (its first to its last instruction); the producer its waits on
// `empty` and `aempty` (ring slots and subject blocks still in use); lane 0 of each epilogue warp its waits on `qfull`.
enum { PROF_FULL, PROF_HANDOFF, PROF_PIPE, PROF_EMPTY, PROF_QFULL, PROF_PASS, PROF_N };
static __device__ unsigned long long fused_prof[PROF_N];
#define B200_PROF_ADD(i, v) atomicAdd(&fused_prof[i], (unsigned long long)(v))
#define B200_TIMED(cyc, stmt)            \
    do {                                 \
        const long long t_ = clock64();  \
        stmt;                            \
        (cyc) += clock64() - t_;         \
    } while (0)
#else
#define B200_PROF_ADD(i, v) (void)0
#define B200_TIMED(cyc, stmt) \
    do {                      \
        stmt;                 \
        (void)(cyc);          \
    } while (0)
#endif

// Move this thread's pending hits of chunk OFF (ascending column order) into its FIFO (a ring of QN slots).  Returns
// true when some lane still has hits but no free slot: the caller runs a fifo_step and calls again with the remaining mask.
template <int OFF, int QN, int QS, int NR>
__device__ __forceinline__ bool chunk_push(const uint32_t (&r)[NR], unsigned& hits, uint32_t pos0, float thr, uint32_t n_pos,
                                           uint32_t qaddr, int head, int& tail) {
    while (__any_sync(B200_FULL_MASK, hits != 0)) {
        if (hits && tail - head < QN) {
            const int j = __ffs(hits) - 1;
            hits &= hits - 1;
            // (taking the chunk maximum when it is the only score above the threshold, instead of the select tree, measured
            // slower: the extra branch costs more than the 31 selects it saves)
            const float val = chunk_select<OFF>(r, j);
            const uint32_t pos = pos0 + (uint32_t)(OFF + j);
            if (val > thr && pos < n_pos) {
                sts_v2(qaddr + (uint32_t)(tail & (QN - 1)) * QS, val, pos);
                ++tail;
            }
        }
        if (__any_sync(B200_FULL_MASK, hits != 0 && tail - head == QN)) return true;
    }
    return false;
}

// Where accepted candidates go: the row's replace-minimum list in shared memory (adaptive) or, once the threshold is
// frozen, the next free slot of its global list.
struct Sink {
    float* gs;      // this thread's global list (scores / ids), `cap` slots
    int32_t* gi;
    int cap;
    bool appending;
};

// One step of the deferred work, for all 32 rows of the warp at once (no warp-collective inside: lanes may diverge):
// look at the oldest pending hit of the row; drop it if the threshold has passed it; if it lies beyond the CSR window,
// move the window (loads issued, not waited for) and leave the hit for the next step; otherwise test it against the
// window / the exclusion list and hand it to the sink.
template <int QN, int QS, bool WIDE>
__device__ __forceinline__ void fifo_step(const TcParams& p, RowState& rs, CsrWindow& cw, uint32_t qaddr, int& head, int tail,
                                          uint32_t ls, uint32_t li, int kc, const Sink& sink) {
    if (head == tail) return;
    float val;
    uint32_t pos;
    lds_v2(qaddr + (uint32_t)(head & (QN - 1)) * QS, val, pos);
    if (!(val > rs.thr)) {
        ++head;
        return;
    }
    const int obj = p.pos2obj ? __ldg(p.pos2obj + pos) : (int)pos;
    const int g = obj + p.id_off;
    if (g > cw.w3) {  // every id of the window is smaller (w3 == PAD_ID once the slice is exhausted: never taken then)
        cw.cur += 4;
        if (++cw.streak >= 2) {  // long slice: lower_bound of g in the rest
            int64_t lo = cw.cur, hi = cw.fhi;
            while (lo < hi) {
                const int64_t mid = (lo + hi) >> 1;
                if (__ldg(p.indices + mid) < g)
                    lo = mid + 1;
                else
                    hi = mid;
            }
            cw.cur = lo;
        }
        window_load(p.indices, cw);
        return;
    }
    cw.streak = 0;
    ++head;
    const bool viewed = (g == cw.w0) | (g == cw.w1) | (g == cw.w2) | (g == cw.w3);
    if (!viewed && !(rs.xrow && is_excluded(rs, p.excl_n, g))) {
        if (WIDE && sink.appending) {
            if (rs.cnt < sink.cap) {
                sink.gs[rs.cnt] = val;
                sink.gi[rs.cnt] = obj;
            }
            ++rs.cnt;  // beyond the capacity: counted, not stored -- the row fails its certificate and is re-ranked
        } else {
            list_insert(ls, li, kc, rs, val, obj);
        }
    }
}

// One m-half of a quarter (64 subject rows x 64 objects, all KB k blocks) as one wgmma commit group, straight-line code
// (ptxas serialises a group whose wgmmas are spread over a loop or a barrier wait): the object blocks sit in ring slots
// s, s + 1, ... (mod NS) and have landed.  Every accumulator sums its k steps in the same order as ever: kb, then k.
template <bool BF16, int KB>
__device__ __forceinline__ void mma_half(uint32_t (&d)[32], uint32_t a_lo, uint32_t b_lo0, int NS, uint32_t s) {
    constexpr uint32_t BLK16 = BLK_BYTES >> 4, OBJ16 = OBJ_BLK_BYTES >> 4;
    fence_acc(d);
    wgmma_fence();
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
        const uint32_t b_lo = b_lo0 + s * OBJ16;
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_64x64<BF16>(d, a_lo + kb * BLK16 + 2 * k, b_lo + 2 * k, (kb | k) != 0);
        if (++s == (uint32_t)NS) s = 0;
    }
    wgmma_commit();
}

// Wait until the KB object blocks of a quarter (ring slots s, s + 1, ... from phase ph) have landed.
template <int KB>
__device__ __forceinline__ void blocks_landed(uint32_t bar_full, int NS, uint32_t s, uint32_t ph) {
#pragma unroll
    for (int kb = 0; kb < KB; ++kb) {
        mbar_wait(bar_full + 8 * s, ph);
        if (++s == (uint32_t)NS) {
            s = 0;
            ph ^= 1;
        }
    }
}

// Hand one m-half of a finished quarter to the epilogue: wait until its two readers have taken the previous one, store
// this thread's 32 accumulators of it, arrive on the half's `full` barrier.
// The threshold gate: the warp's 16 rows of the half are staged only if one of their 64 scores lies above that row's
// threshold.  `thr` is the row's exchange slot of the list this quarter feeds (its column group): the list's own rs.thr
// at some earlier tile of the same work item (the tag says which work item), hence never above the threshold the
// epilogue scans this quarter with -- a gated row could not have produced a hit.  No other slot may be used: the other
// list's or the peers' value can lie above anything this list ever adopts (after its last tile, say), and the list's
// final threshold must bound every score it discarded.  A slot of another work item counts as -inf (stage).  The
// decision is per warp (one vote over its 32 threads, 16 columns of 2 rows each); the warp's flag tells the epilogue
// whether its rows of the buffer are this quarter's or still an earlier one's.  Gated or not, the barrier protocol is
// the same: only the data stores are skipped.
__device__ __forceinline__ void store_half(const uint32_t (&d)[32], uint32_t stg, uint32_t qempty, uint32_t parity, uint32_t qfull,
                                           uint32_t thr, uint32_t tag, uint32_t flag, long long& wait_cycles) {
    float m0 = fmaxf(fu(d[0]), fu(d[1])), m1 = fmaxf(fu(d[2]), fu(d[3]));  // this thread's columns of its two rows
#pragma unroll
    for (int j = 1; j < 8; ++j) {
        m0 = max3(m0, fu(d[4 * j]), fu(d[4 * j + 1]));
        m1 = max3(m1, fu(d[4 * j + 2]), fu(d[4 * j + 3]));
    }
    uint32_t tg0, tg1;
    float t0, t1;
    lds_thr(thr, tg0, t0);
    lds_thr(thr + 8 * 8, tg1, t1);  // the row 8 below
    const bool hit = (m0 > (tg0 == tag ? t0 : -INFINITY)) | (m1 > (tg1 == tag ? t1 : -INFINITY));
    const bool staged = __any_sync(B200_FULL_MASK, hit);
    B200_TIMED(wait_cycles, mbar_wait(qempty, parity));
    if (staged) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const uint32_t a = stg + (uint32_t)(8 * j * 4);
            sts_v2(a, d[4 * j], d[4 * j + 1]);
            sts_v2(a + 8 * STG_STRIDE * 4, d[4 * j + 2], d[4 * j + 3]);
        }
    }
    if ((threadIdx.x & 31) == 0) sts_s32(flag, staged ? 1 : 0);
    mbar_arrive(qfull);
}

// The staging flags of two MMA warps, read after the half's `full` barrier (ordered after it like the staged data).
__device__ __forceinline__ void lds_flags2(uint32_t a, uint32_t& f0, uint32_t& f1) {
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(f0), "=r"(f1) : "r"(a) : "memory");
}

// Shared-memory map (dynamic, 1 KiB aligned): [KB] subject blocks (16 KiB each) | [NS] object blocks (8 KiB each: 64
// objects of a tile quarter) | accumulator staging [128 rows][STG_STRIDE] fp32 | candidate lists [NLIST][128 rows][SLOTS]
// scores + ids | FIFOs | thresholds [NLIST + 1][128] | barriers, staging flags.
// WIDE / PEERS compile the wide mode (threshold freeze + global append) and the peer-threshold exchange in; the plain
// instantiation carries neither in its tile loop.  BF16 selects the MMA operand type.
template <bool WIDE, bool PEERS, bool BF16>
__global__ void __cluster_dims__(2, 1, 1) __maxnreg__(FusedCfg::REGS_LAUNCH)
fused_topk_kernel(const __grid_constant__ CUtensorMap tm_sub, const __grid_constant__ CUtensorMap tm_obj, const TcParams p) {
    using Cfg = FusedCfg;
    constexpr int NLIST = Cfg::NLIST, SLOTS = Cfg::SLOTS, NQ = Cfg::NQ, QN = Cfg::Q, QS = Cfg::QSTRIDE;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);

    const int KB = p.kblocks, NS = p.n_stages;
    uint8_t* sA = smem;
    uint8_t* sB = sA + (size_t)KB * BLK_BYTES;
    uint8_t* sStg = sB + (size_t)NS * OBJ_BLK_BYTES;
    uint8_t* sLs = sStg + STG_BYTES;  // per warp [slot][lane] arrays
    uint8_t* sLi = sLs + Cfg::LIST_BYTES;
    uint8_t* sQ = sLi + Cfg::LIST_BYTES;
    unsigned long long* sThr = reinterpret_cast<unsigned long long*>(sQ + Cfg::QBYTES);  // [NLIST + 1][128]
    uint64_t* bars = reinterpret_cast<uint64_t*>(sThr + (NLIST + 1) * TILE_M);
    const uint32_t bar_full = smem_u32(bars);                     // [NS] object block landed
    const uint32_t bar_afull = smem_u32(bars + MAX_STAGES);       // subject blocks landed
    // the staging buffer's two m-halves (rows 0-63 / 64-127) are handed over separately
    const uint32_t bar_qfull = smem_u32(bars + MAX_STAGES + 1);   // [4][2] half h of quarter q of the current tile staged
    const uint32_t bar_qempty = smem_u32(bars + MAX_STAGES + 9);  // [2] staged half read by its two epilogue warps
    // staging flags, u32 [2 halves][4 MMA warps] in the unused tail of the barrier area: 1 = the warp's 16 rows of the half
    // hold the current quarter, 0 = the threshold gate skipped them (store_half)
    const uint32_t stg_flags = smem_u32(bars + MAX_STAGES + 11);
    const uint32_t bar_empty = smem_u32(bars + MAX_STAGES + 15);       // [NS] object block read by the MMA warp group
    const uint32_t bar_aempty = smem_u32(bars + 2 * MAX_STAGES + 15);  // subject blocks no longer read

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int rank = blockIdx.x & 1;  // which 128 rows of the pair's 256 (== the CTA's rank in its cluster)
    const int n_pairs = gridDim.x >> 1, pair = blockIdx.x >> 1;

    if (threadIdx.x == 0) {
        for (int i = 0; i < NS; ++i) {
            mbar_init(bar_full + 8 * i, 1);
            mbar_init(bar_empty + 8 * i, 4);  // lane 0 of each MMA warp
        }
        mbar_init(bar_afull, 1);
        mbar_init(bar_aempty, 4);
        for (int i = 0; i < 8; ++i) mbar_init(bar_qfull + 8 * i, 128);  // every thread of the MMA warp group
        for (int h = 0; h < 2; ++h) mbar_init(bar_qempty + 8 * h, 2);
        fence_barrier_init();
        tma_prefetch_desc(&tm_sub);
        tma_prefetch_desc(&tm_obj);
    }
    for (int i = threadIdx.x; i < (NLIST + 1) * TILE_M; i += blockDim.x) sts_thr(smem_u32(sThr + i), TAG_NONE, INFINITY);
    __syncthreads();

    const int n_work = p.n_row_tiles * p.n_splits;
    constexpr uint32_t BLK16 = BLK_BYTES >> 4, OBJ16 = OBJ_BLK_BYTES >> 4;  // blocks in descriptor address units

    if (warp < Cfg::EPI0) {
        // ===================================================================== MMA warp group
        setmaxnreg_dec<Cfg::REGS_MMA>();
#ifdef B200_FUSED_PROFILE
        const bool issuer = threadIdx.x == 0;  // the thread that measures
        const long long t_start = clock64();
#endif
        long long full_cycles = 0, handoff_cycles = 0, pipe_cycles = 0;
        const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
        // A ring slot goes back to the producer once the wgmmas that read it have retired in every warp of the warp group
        // (wgmma.wait_group waits for the executing thread's groups only): lane 0 of each warp arrives on its `empty`
        // barrier after its own wait.  Slots are released in the order they were filled.
        uint32_t rel = 0;
        auto release = [&](int n) {
            for (int i = 0; i < n; ++i) {
                if (lane == 0) mbar_arrive(bar_empty + 8 * rel);
                if (++rel == (uint32_t)NS) rel = 0;
            }
        };

        // this thread's accumulator rows / columns in the staging buffer (m-half 1: + 64 rows; second row of a fragment: + 8)
        const uint32_t stg_w = smem_u32(sStg) + (uint32_t)(((warp * 16 + (lane >> 2)) * STG_STRIDE + 2 * (lane & 3)) * 4);
        const uint32_t stg_w1 = stg_w + (uint32_t)(64 * STG_STRIDE * 4);
        // the exchange slot of this thread's first row in list 0 (m-half 1: + 64 rows; list 1: + 128 rows), its warp's flags
        const uint32_t thr_w = smem_u32(sThr + warp * 16 + (lane >> 2));
        const uint32_t flag_w = stg_flags + (uint32_t)warp * 4, flag_w1 = flag_w + 16;
        const uint32_t a_lo0 = smem_desc_lo(sA_u), b_lo0 = smem_desc_lo(sB_u);
        // fp32 accumulators of the two m-halves, as bit patterns
        uint32_t acc[2][32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[0][i] = acc[1][i] = 0u;
        uint32_t stage = 0, ph = 0, work_it = 0, n_store = 0;
        // d_pad = 128 (two k blocks; the ring holds two quarters' object blocks): each m-half is its own commit group and
        // the hand-off of one half overlaps the MMAs of the other --
        //   G0(q), G1(q) | wait<1>, store half 0 of q, G0(q + 1) | wait<1>, release q's blocks, store half 1 of q,
        //   G1(q + 1) | ...
        // The ring slots of quarter q are refilled once G1(q), their second reader, has retired.
        constexpr int PKB = 2;
        const bool pipelined = KB == PKB && 2 * PKB <= NS;
        auto advance = [&]() {  // ring position of the next quarter's first block
            stage += (uint32_t)PKB;
            if (stage >= (uint32_t)NS) {
                stage -= (uint32_t)NS;
                ph ^= 1;
            }
        };
        for (int w = pair; w < n_work; w += n_pairs, ++work_it) {
            const int split = w / p.n_row_tiles;
            const int t0 = split * p.tiles_per_split;
            const int t1 = min(t0 + p.tiles_per_split, p.n_obj_tiles);
            mbar_wait(bar_afull, work_it & 1);
            const int nq = 4 * (t1 - t0);  // quarters of the work item, in stream order
            // (rows 64-127 of the subject block start 8 KiB = +512 descriptor units further)
            if (pipelined) {
                B200_TIMED(full_cycles, blocks_landed<PKB>(bar_full, NS, stage, ph));
                mma_half<BF16, PKB>(acc[0], a_lo0, b_lo0, NS, stage);
                mma_half<BF16, PKB>(acc[1], a_lo0 + 512, b_lo0, NS, stage);
                advance();
                for (int qi = 0; qi + 1 < nq; ++qi, ++n_store) {
                    const uint32_t qf = bar_qfull + 16 * (qi & 3), par = (n_store & 1) ^ 1;
                    const uint32_t thr_q = thr_w + (uint32_t)(qi & 1) * (TILE_M * 8);  // quarter qi feeds list qi & 1
                    B200_TIMED(pipe_cycles, wgmma_wait<1>());  // G0(qi)
                    fence_acc(acc[0]);
                    store_half(acc[0], stg_w, bar_qempty, par, qf, thr_q, work_it, flag_w, handoff_cycles);
                    B200_TIMED(full_cycles, blocks_landed<PKB>(bar_full, NS, stage, ph));
                    mma_half<BF16, PKB>(acc[0], a_lo0, b_lo0, NS, stage);
                    B200_TIMED(pipe_cycles, wgmma_wait<1>());  // G1(qi): quarter qi's object blocks are free
                    fence_acc(acc[1]);
                    release(PKB);
                    store_half(acc[1], stg_w1, bar_qempty + 8, par, qf + 8, thr_q + 64 * 8, work_it, flag_w1, handoff_cycles);
                    mma_half<BF16, PKB>(acc[1], a_lo0 + 512, b_lo0, NS, stage);
                    advance();
                }
                const uint32_t qf = bar_qfull + 16 * ((nq - 1) & 3), par = (n_store & 1) ^ 1;
                const uint32_t thr_q = thr_w + (uint32_t)((nq - 1) & 1) * (TILE_M * 8);
                B200_TIMED(pipe_cycles, wgmma_wait<1>());
                fence_acc(acc[0]);
                store_half(acc[0], stg_w, bar_qempty, par, qf, thr_q, work_it, flag_w, handoff_cycles);
                B200_TIMED(pipe_cycles, wgmma_wait<0>());  // the work item's last MMAs (the next one reloads the subject blocks)
                fence_acc(acc[1]);
                release(PKB);
                store_half(acc[1], stg_w1, bar_qempty + 8, par, qf + 8, thr_q + 64 * 8, work_it, flag_w1, handoff_cycles);
                ++n_store;
            } else {
                // deeper d: one commit group per k block (both m-halves), its ring slot refilled as soon as the next
                // block's group has been issued and the block's own group has retired
                for (int qi = 0; qi < nq; ++qi, ++n_store) {
                    uint32_t a_lo = a_lo0;
                    fence_acc(acc[0]);
                    fence_acc(acc[1]);
                    for (int kb = 0; kb < KB; ++kb, a_lo += BLK16) {
                        B200_TIMED(full_cycles, mbar_wait(bar_full + 8 * stage, ph));
                        wgmma_fence();
                        const uint32_t b_lo = b_lo0 + stage * OBJ16;
                        // +32 B per K = 16 step inside the 128 B swizzle atom = +2 in descriptor address units
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint32_t accum = (kb | k) != 0;
                            wgmma_64x64<BF16>(acc[0], a_lo + 2 * k, b_lo + 2 * k, accum);
                            wgmma_64x64<BF16>(acc[1], a_lo + 512 + 2 * k, b_lo + 2 * k, accum);
                        }
                        wgmma_commit();
                        if (++stage == (uint32_t)NS) {
                            stage = 0;
                            ph ^= 1;
                        }
                        if (kb > 0) {
                            B200_TIMED(pipe_cycles, wgmma_wait<1>());  // the previous k block's MMAs have read their ring slot
                            release(1);
                        }
                    }
                    B200_TIMED(pipe_cycles, wgmma_wait<0>());
                    fence_acc(acc[0]);
                    fence_acc(acc[1]);
                    release(1);
                    const uint32_t qf = bar_qfull + 16 * (qi & 3), par = (n_store & 1) ^ 1;
                    const uint32_t thr_q = thr_w + (uint32_t)(qi & 1) * (TILE_M * 8);
                    store_half(acc[0], stg_w, bar_qempty, par, qf, thr_q, work_it, flag_w, handoff_cycles);
                    store_half(acc[1], stg_w1, bar_qempty + 8, par, qf + 8, thr_q + 64 * 8, work_it, flag_w1, handoff_cycles);
                }
            }
            // every work item ends in wgmma.wait_group 0: the subject blocks may be reloaded
            if (lane == 0) mbar_arrive(bar_aempty);
        }
#ifdef B200_FUSED_PROFILE
        if (issuer) {
            B200_PROF_ADD(PROF_FULL, full_cycles);
            B200_PROF_ADD(PROF_HANDOFF, handoff_cycles);
            B200_PROF_ADD(PROF_PIPE, pipe_cycles);
            B200_PROF_ADD(PROF_PASS, clock64() - t_start);
        }
#endif
    } else if (warp < Cfg::PRODUCER) {
        // ===================================================================== epilogue: select candidates
        setmaxnreg_inc<Cfg::REGS_EPILOGUE>();
        long long qfull_cycles = 0;
        const int ew = warp - Cfg::EPI0;
        const int colg = ew >> 2, quarter = warp & 3;  // column group of the tile / row quarter of the CTA's 128 rows
        const int wrow0 = quarter * 32;                // first CTA-local subject row of this warp
        // [slot][lane] arrays of this warp: SLOTS x 32 lanes x 4 B, slot stride 128 B (as list_insert expects)
        const uint32_t ls = pin(smem_u32(sLs) + (uint32_t)((colg * TILE_M + wrow0) * SLOTS * 4) + lane * 4);
        const uint32_t li = pin(smem_u32(sLi) + (uint32_t)((colg * TILE_M + wrow0) * SLOTS * 4) + lane * 4);
        const uint32_t qaddr = pin(smem_u32(sQ) + (uint32_t)(ew * 32 + lane) * 8);
        const uint32_t thr_row = pin(smem_u32(sThr + wrow0 + lane));  // + l * 128 * 8: the threads of this row, [NLIST]: peers
        const uint32_t my_thr = pin(thr_row + (uint32_t)colg * (TILE_M * 8));
        const uint32_t stg_r = pin(smem_u32(sStg) + (uint32_t)((wrow0 + lane) * STG_STRIDE * 4));
        // the m-half of the staging buffer that holds this warp's rows: quarters 0, 1 -> half 0; 2, 3 -> half 1
        const uint32_t half = (uint32_t)quarter >> 1;
        const uint32_t qfull0 = pin(bar_qfull + (uint32_t)colg * 16 + half * 8), qempty = pin(bar_qempty + half * 8);
        // the flags of the two MMA warps that staged this warp's rows: lanes 0-15 / 16-31 are the rows of MMA warps
        // 2 (quarter & 1) and 2 (quarter & 1) + 1 of the half (not pinned: one register less in the tile loop)
        const uint32_t flags2 = stg_flags + (half * 4 + 2 * ((uint32_t)quarter & 1)) * 4;
        const bool lane0 = pin((uint32_t)lane) == 0;
        const uint32_t n_pos = (uint32_t)p.n_pos;
        const int kc = p.k_cand;  // (<= SLOTS, guaranteed by the host; a visible bound makes the compiler unroll the list scans fully and spill)
        const bool dbg_skip = p.debug_mode == 2;
        const bool peers = PEERS && p.n_peers > 0;
        const uint32_t other_thr = pin(thr_row + (uint32_t)(colg ^ 1) * (TILE_M * 8));  // the other list of the row
        uint32_t tpar = 0, work_tag = 0;  // parity of the quarter barriers (one phase per tile)
        for (int w = pair; w < n_work; w += n_pairs, ++work_tag) {
            const int split = w / p.n_row_tiles, rt = w - split * p.n_row_tiles;
            const int t0 = split * p.tiles_per_split;
            const int t1 = min(t0 + p.tiles_per_split, p.n_obj_tiles);
            const int64_t grow = ((int64_t)rt * 2 + rank) * TILE_M + wrow0 + lane;
            const bool row_ok = grow < p.n_rows;
            RowState rs;
            rs.thr = (row_ok && p.debug_mode == 0) ? -INFINITY : INFINITY;  // padded rows never produce candidates
            rs.cnt = 0;
            rs.minpos = 0;
            int head = 0, tail = 0;
            CsrWindow cw;
            sts_thr(my_thr, work_tag, rs.thr);
            const int nt = t1 - t0;
            int ts = 0;
            if (lane == 0) ts = carousel_start(p, pair, work_tag, split, t0, t1, false);
            ts = __shfl_sync(B200_FULL_MASK, ts, 0);
            const int64_t frow = row_ok ? (p.row_ids ? (int64_t)p.row_ids[grow] : grow) : -1;
            const int64_t lrow = (int64_t)(split * NLIST + colg) * p.rows_pad + (row_ok ? grow : 0);  // this thread's global list
            Sink sink;
            sink.gs = p.cand_scores + lrow * p.cand_stride;
            sink.gi = p.cand_ids + lrow * p.cand_stride;
            sink.cap = p.cand_stride;
            sink.appending = false;
            auto cursors_at = [&](int tile) {  // (re)position the CSR / exclusion cursors at the first object of `tile`
                const int64_t pos_first = (int64_t)tile * TILE_N + colg * QUART_N;
                const bool live = frow >= 0 && pos_first < p.n_pos;
                const int g_first = live ? (p.pos2obj ? __ldg(p.pos2obj + pos_first) : (int)pos_first) + p.id_off : 0;
                row_cursors_init(p, rs, live ? frow : -1, g_first);
                cw.cur = rs.cur;
                cw.fhi = rs.fhi;
                cw.streak = 0;
                window_load(p.indices, cw);
            };
            // (a macro, not a lambda: an outlined lambda would force every captured variable into local memory)
#define B200_STEP() fifo_step<QN, QS, WIDE>(p, rs, cw, qaddr, head, tail, ls, li, kc, sink)
            cursors_at(ts);
            int t = ts;
            uint32_t pos_t = (uint32_t)ts * TILE_N + (uint32_t)(colg * QUART_N);
            for (int it = 0; it < nt; ++it) {
                // exchange thresholds with the thread that owns the other column group of this row and with the other
                // ranks (monotone, racy by design: a stale value is only a weaker bound; the tag keeps a value of the
                // previous work item out)
                {
                    sts_thr(my_thr, work_tag, rs.thr);
                    {
                        uint32_t ptag;
                        float pthr;
                        lds_thr(other_thr, ptag, pthr);
                        if (ptag == work_tag) rs.thr = fmaxf(rs.thr, pthr);
                    }
                    if constexpr (PEERS) {
                        if (peers) {
                            uint32_t ptag;
                            float pthr;
                            lds_thr(thr_row + (uint32_t)NLIST * (TILE_M * 8), ptag, pthr);
                            if (ptag == work_tag) rs.thr = fmaxf(rs.thr, pthr);
                        }
                    }
                }
                if (WIDE && it == p.phase1_tiles) {
                    // wide mode: freeze the threshold.  Everything pending goes through the adaptive list first; then the
                    // list moves to the front of the row's global list and later candidates are appended behind it.
                    while (__any_sync(B200_FULL_MASK, head != tail)) B200_STEP();
                    if (row_ok) {
                        const int n = min(rs.cnt, kc);
                        for (int e = 0; e < n; ++e) {
                            sink.gs[e] = lds_f32(ls + e * 128);
                            sink.gi[e] = lds_s32(li + e * 128);
                        }
                    }
                    sink.appending = true;
                }
                // the last tile before the stream wraps around / of the work item: every pending hit must be handled
                // before the cursors are repositioned or the list is written
                const bool force = (t + 1 == t1);
                const bool last = (it + 1 == nt);
#pragma unroll
                for (int s = 0; s < NQ; ++s) {
                    B200_TIMED(qfull_cycles, mbar_wait(qfull0 + (uint32_t)(s * NLIST * 16), tpar));
                    // rows the threshold gate left unstaged cannot hit (store_half); a warp with none staged reads nothing
                    uint32_t f0, f1;
                    lds_flags2(flags2, f0, f1);
                    const bool staged = (lane < 16 ? f0 : f1) != 0;
                    const bool scan = !dbg_skip && (f0 | f1) != 0;
                    uint32_t r[QUART_N];
                    if (scan) stage_ld(stg_r, r);
                    __syncwarp();
                    if (lane0) mbar_arrive(qempty);  // staging buffer free again
                    if (scan) {
                        const uint32_t pos_q = pos_t + (uint32_t)(s * NLIST * QUART_N);
                        const float m0 = chunk_max<0>(r), m1 = chunk_max<32>(r);
                        const float mx = fmaxf(m0, m1);
                        // an unstaged row's part of the buffer is an earlier quarter: no hits for its lane
                        const float thr = staged ? rs.thr : INFINITY;
                        if (__any_sync(B200_FULL_MASK, mx > thr)) {
                            unsigned h0 = 0, h1 = 0;
                            if (__any_sync(B200_FULL_MASK, m0 > thr)) h0 = chunk_hits<0>(r, thr);
                            if (__any_sync(B200_FULL_MASK, m1 > thr)) h1 = chunk_hits<32>(r, thr);
                            for (;;) {
                                bool stuck = chunk_push<0, QN, QS>(r, h0, pos_q, rs.thr, n_pos, qaddr, head, tail);
                                if (!stuck) stuck = chunk_push<32, QN, QS>(r, h1, pos_q, rs.thr, n_pos, qaddr, head, tail);
                                if (!stuck) break;
                                B200_STEP();  // dense phase: make room, then go on
                            }
                        }
                    }
                }
                if (!dbg_skip) {
                    // deferred work: at most one step per tile (bounded latency in front of the next quarter), by default
                    // every PERIOD-th tile or as soon as some row has BACKLOG hits waiting, except where everything pending
                    // has to be finished
                    const bool due = (tail - head >= Cfg::BACKLOG) ||
                                     (head != tail && ((it & (Cfg::PERIOD - 1)) == Cfg::PERIOD - 1 || force || last));
                    if (__any_sync(B200_FULL_MASK, due)) {
                        B200_STEP();
                        if (force || last)
                            while (__any_sync(B200_FULL_MASK, head != tail)) B200_STEP();
                    }
                }
                tpar ^= 1;
                ++t;
                pos_t += TILE_N;
                if (t == t1 && !last) {  // wrapped around: objects ascend again from the split's first tile
                    t = t0;
                    pos_t = (uint32_t)t0 * TILE_N + (uint32_t)(colg * QUART_N);
                    cursors_at(t0);
                }
            }
            // ---- this thread's candidate list (unsorted), its length and its final threshold
            if (row_ok) {
                if (!(WIDE && sink.appending)) {
                    const int n = min(rs.cnt, kc);
                    for (int e = 0; e < n; ++e) {
                        sink.gs[e] = lds_f32(ls + e * 128);
                        sink.gi[e] = lds_s32(li + e * 128);
                    }
                }
                p.cand_counts[lrow] = rs.cnt;
                p.cand_thr[lrow] = rs.thr;
            }
            // last work item of this CTA: lets the helper warps leave their polling loop
            if (PEERS && peers && w + n_pairs >= n_work) sts_thr(my_thr, TAG_DONE, INFINITY);
        }
#undef B200_STEP
        if (lane == 0) B200_PROF_ADD(PROF_QFULL, qfull_cycles);
    } else if (warp == Cfg::PRODUCER) {
        // ===================================================================== producer: every TMA load of the CTA
        // Object blocks in consumption order (work item, tile, quarter, k block), up to NS blocks ahead of the MMAs; a
        // slot is refilled once its `empty` barrier says every MMA warp has retired the wgmmas that read it.
        if (lane == 0) {
            const uint32_t sA_u = smem_u32(sA), sB_u = smem_u32(sB);
            long long empty_cycles = 0;
            uint32_t stage = 0, ph = 0, work_it = 0;
            for (int w = pair; w < n_work; w += n_pairs, ++work_it) {
                const int split = w / p.n_row_tiles, rt = w - split * p.n_row_tiles;
                const int t0 = split * p.tiles_per_split;
                const int t1 = min(t0 + p.tiles_per_split, p.n_obj_tiles);
                const int nt = t1 - t0;
                // the subject blocks are reloaded once the previous work item's MMAs have all retired
                if (work_it > 0) B200_TIMED(empty_cycles, mbar_wait(bar_aempty, (work_it - 1) & 1));
                mbar_arrive_expect_tx(bar_afull, (uint32_t)(KB * BLK_BYTES));
                for (int kb = 0; kb < KB; ++kb)
                    tma_load_2d(sA_u + (uint32_t)kb * BLK_BYTES, &tm_sub, bar_afull, kb * KBLK, (rt * 2 + rank) * TILE_M);
                const int ts = carousel_start(p, pair, work_it, split, t0, t1, rank == 0);
                for (int i = 0; i < nt; ++i) {
                    const int t = ts + i < t1 ? ts + i : ts + i - nt;
                    // the front is the position of the reference pair (pair 0 of each split's work items)
                    if (rank == 0 && p.front && pair == 0 && (i & 15) == 0) *reinterpret_cast<volatile int32_t*>(p.front + split) = t;
                    for (int q = 0; q < 4; ++q)
                        for (int kb = 0; kb < KB; ++kb) {
                            // (a fresh barrier passes the wait for parity 1: the first round finds every slot free)
                            B200_TIMED(empty_cycles, mbar_wait(bar_empty + 8 * stage, ph ^ 1));
                            mbar_arrive_expect_tx(bar_full + 8 * stage, OBJ_BLK_BYTES);
                            tma_load_2d(sB_u + stage * OBJ_BLK_BYTES, &tm_obj, bar_full + 8 * stage, kb * KBLK, t * TILE_N + q * QUART_N);
                            if (++stage == (uint32_t)NS) {
                                stage = 0;
                                ph ^= 1;
                            }
                        }
                }
            }
            B200_PROF_ADD(PROF_EMPTY, empty_cycles);
        }
    } else if (PEERS && p.n_peers > 0) {
        // ===================================================================== peer-threshold helpers (two warps)
        // Thread h serves CTA-local rows h and h + 64.  Per round and row: read the row's own thresholds from the exchange
        // slots, publish their maximum to this rank's global array, read the other ranks' published values (NVLink peer
        // loads, latency irrelevant here), leave their maximum in the row's extra exchange slot.  All values are monotone
        // lower bounds of the row's final threshold: a stale one is only weaker, never wrong.
        const int h = (warp - Cfg::PRODUCER - 1) * 32 + lane;
        float published[2] = {-INFINITY, -INFINITY};
        uint32_t pub_tag[2] = {0xffffffffu, 0xffffffffu};
        bool done[2] = {false, false};
        while (!(done[0] && done[1])) {
#pragma unroll
            for (int s = 0; s < 2; ++s) {
                const int r = h + 64 * s;
                uint32_t tag;
                float own;
                lds_thr(smem_u32(sThr + r), tag, own);
                done[s] = tag == TAG_DONE;  // the row's first column group has finished its last work item
                if (tag >= TAG_DONE) continue;
#pragma unroll
                for (int l = 1; l < NLIST; ++l) {
                    uint32_t tl;
                    float vl;
                    lds_thr(smem_u32(sThr + l * TILE_M + r), tl, vl);
                    if (tl == tag) own = fmaxf(own, vl);
                }
                const int w = pair + (int)tag * n_pairs;
                if (w >= n_work) continue;
                const int rt = w % p.n_row_tiles;
                const int64_t grow = ((int64_t)rt * 2 + rank) * TILE_M + r;
                if (grow >= p.n_rows) continue;
                if (pub_tag[s] != tag) {
                    pub_tag[s] = tag;
                    published[s] = -INFINITY;
                }
                if (own > published[s] && own < INFINITY) {
                    published[s] = own;
                    stg_peer(p.peer_pub + p.peer_row0 + grow, p.peer_epoch, ldexpf(own, -p.peer_exp));
                }
                // all peer loads in flight at once: one NVLink round trip per row and round
                unsigned long long v[MAX_PEERS];
#pragma unroll
                for (int q = 0; q < MAX_PEERS; ++q) v[q] = q < p.n_peers ? ldg_peer(p.peer_in[q] + p.peer_row0 + grow) : 0ull;
                float best = -INFINITY;
#pragma unroll
                for (int q = 0; q < MAX_PEERS; ++q)
                    if (q < p.n_peers && (uint32_t)(v[q] >> 32) == p.peer_epoch) best = fmaxf(best, __uint_as_float((uint32_t)v[q]));
                if (best > -INFINITY) sts_thr(smem_u32(sThr + NLIST * TILE_M + r), tag, ldexpf(best, p.peer_exp));
            }
            __nanosleep(200);
        }
    }
}

}  // namespace tc
}  // namespace b200
