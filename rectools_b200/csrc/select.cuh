// Exhaustive fp64 scoring kernel + warp-level list selection / re-scoring kernels.
//
// Replaces, for the rows it is given, the arithmetic of `implicit.cpu.topk.topk` as called at
// rectools/models/rank/rank_implicit.py:264-272 (score, /item_norms, CSR mask, per-row top-k), with the result
// definition of include/b200_rank.h (fp64-accumulated dot rounded once to fp32; order = score desc, id asc).
#pragma once
#include <type_traits>

#include "common.cuh"
#include "sizes.h"

namespace b200 {

constexpr int LIST_LEN = 32;  // every partial list is one warp wide

// ---------------------------------------------------------------------------------------------------------------
// Exhaustive kernel: 32 subjects per block (4 per warp), object positions streamed 32 at a time (lane = object).
// ---------------------------------------------------------------------------------------------------------------
constexpr int EX_THREADS = 256;
constexpr int EX_ROWS = 32;
constexpr int EX_ROWS_PER_WARP = 4;
constexpr int EX_DK = 64;

struct ExactParams {
    const float* subjects;   // fp32 [*, d]
    const int64_t* row_map;  // nullable: logical row -> physical row of `subjects`
    const int32_t* rows;     // nullable: compact index -> logical row (re-rank subset)
    const int32_t* n_sel_dev;  // nullable: device-side count overriding n_sel (early exit for unused blocks)
    int64_t n_sel;           // number of compact indices
    const void* objects;     // [n_objects, d] in the kernel's object type TO (fp32, fp16 or bf16)
    const int32_t* pos2obj;  // nullable whitelist: position -> object id (sorted ascending)
    int64_t n_pos;
    int32_t d;
    const float* obj_norms;  // nullable (COSINE): fp32 norm per object id, zero already replaced by 1e-10
    const int64_t* indptr;   // nullable CSR filter, by logical row
    const int32_t* indices;
    int32_t id_off;          // CSR column ids are global: global id = local object id + id_off
    int32_t k_out;           // row stride of out_*
    int32_t k0;              // this pass selects entries [k0, k0 + kp)
    int32_t kp;              // <= 32
    const int32_t* out_ids;  // previous passes (bound), [n_rows, k_out]
    const float* out_scores;
    const int32_t* out_counts;
    float* part_scores;  // [n_splits][part_stride_rows][32]
    int32_t* part_ids;
    int64_t part_stride_rows;  // >= n_sel
};

template <typename TO>
__global__ void __launch_bounds__(EX_THREADS) exact_topk_kernel(const ExactParams p) {
    const TO* objects = static_cast<const TO*>(p.objects);
    __shared__ float s_obj[32][EX_DK + 1];
    __shared__ float s_sub[EX_ROWS][EX_DK];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t n_sel = p.n_sel_dev ? (int64_t)*p.n_sel_dev : p.n_sel;
    const int64_t sel0 = (int64_t)blockIdx.x * EX_ROWS;
    if (sel0 >= n_sel) return;

    const int n_splits = gridDim.y, split = blockIdx.y;
    const int64_t tiles_total = (p.n_pos + 31) >> 5;
    const int64_t tiles_per = (tiles_total + n_splits - 1) / n_splits;
    const int64_t t0 = split * tiles_per;
    const int64_t t1 = min(t0 + tiles_per, tiles_total);

    // per-warp subjects
    int64_t lrow[EX_ROWS_PER_WARP], flo[EX_ROWS_PER_WARP], fhi[EX_ROWS_PER_WARP];
    bool active[EX_ROWS_PER_WARP];
    float thr[EX_ROWS_PER_WARP], ls[EX_ROWS_PER_WARP], bs[EX_ROWS_PER_WARP];
    int li[EX_ROWS_PER_WARP], bi[EX_ROWS_PER_WARP];
#pragma unroll
    for (int q = 0; q < EX_ROWS_PER_WARP; ++q) {
        const int64_t sel = sel0 + warp * EX_ROWS_PER_WARP + q;
        active[q] = sel < n_sel;
        lrow[q] = active[q] ? (p.rows ? (int64_t)p.rows[sel] : sel) : 0;
        thr[q] = -INFINITY;
        ls[q] = -INFINITY;
        li[q] = B200_PAD_ID;
        bs[q] = INFINITY;
        bi[q] = -1;
        flo[q] = fhi[q] = 0;
        if (active[q]) {
            if (p.indptr) {
                flo[q] = p.indptr[lrow[q]];
                fhi[q] = p.indptr[lrow[q] + 1];
            }
            if (p.k0 > 0) {
                if (p.out_counts[lrow[q]] < p.k0) {
                    active[q] = false;  // row exhausted by earlier passes
                } else {
                    bs[q] = p.out_scores[lrow[q] * p.k_out + p.k0 - 1];
                    bi[q] = p.out_ids[lrow[q] * p.k_out + p.k0 - 1];
                }
            }
        }
    }

    for (int64_t t = t0; t < t1; ++t) {
        double acc[EX_ROWS_PER_WARP];
#pragma unroll
        for (int q = 0; q < EX_ROWS_PER_WARP; ++q) acc[q] = 0.0;

        for (int dk0 = 0; dk0 < p.d; dk0 += EX_DK) {
            __syncthreads();
            for (int e = tid; e < 32 * EX_DK; e += EX_THREADS) {
                const int it = e >> 6, j = e & (EX_DK - 1);
                const int64_t pos = t * 32 + it;
                float v = 0.f;
                if (pos < p.n_pos && dk0 + j < p.d) {
                    const int64_t obj = p.pos2obj ? (int64_t)p.pos2obj[pos] : pos;
                    v = to_f32(__ldg(objects + obj * p.d + dk0 + j));
                }
                s_obj[it][j] = v;
            }
            for (int e = tid; e < EX_ROWS * EX_DK; e += EX_THREADS) {
                const int r = e >> 6, j = e & (EX_DK - 1);
                const int64_t sel = sel0 + r;
                float v = 0.f;
                if (sel < n_sel && dk0 + j < p.d) {
                    const int64_t lr = p.rows ? (int64_t)p.rows[sel] : sel;
                    const int64_t pr = p.row_map ? p.row_map[lr] : lr;
                    v = __ldg(p.subjects + pr * p.d + dk0 + j);
                }
                s_sub[r][j] = v;
            }
            __syncthreads();
            const int jn = min(EX_DK, p.d - dk0);
            for (int j = 0; j < jn; ++j) {
                const double ov = (double)s_obj[lane][j];
#pragma unroll
                for (int q = 0; q < EX_ROWS_PER_WARP; ++q)
                    acc[q] = fma(ov, (double)s_sub[warp * EX_ROWS_PER_WARP + q][j], acc[q]);
            }
        }

        const int64_t pos = t * 32 + lane;
        const bool valid = pos < p.n_pos;
        const int obj = valid ? (p.pos2obj ? p.pos2obj[pos] : (int)pos) : B200_PAD_ID;
        const double inv_div = (valid && p.obj_norms) ? (double)__ldg(p.obj_norms + obj) : 1.0;
#pragma unroll
        for (int q = 0; q < EX_ROWS_PER_WARP; ++q) {
            if (!active[q]) continue;  // warp-uniform
            const float s = p.obj_norms ? (float)(acc[q] / inv_div) : (float)acc[q];
            bool c = valid && s > thr[q] && (s < bs[q] || (s == bs[q] && obj > bi[q]));
            if (c && p.indptr) c = !csr_contains(p.indices, flo[q], fhi[q], obj + p.id_off);
            unsigned m = __ballot_sync(B200_FULL_MASK, c);
            while (m) {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                const float cs = __shfl_sync(B200_FULL_MASK, s, src);
                const int ci = __shfl_sync(B200_FULL_MASK, obj, src);
                if (!(cs > thr[q])) continue;  // threshold rose while draining this ballot
                const int ins = __popc(__ballot_sync(B200_FULL_MASK, ls[q] >= cs));
                const float us = __shfl_up_sync(B200_FULL_MASK, ls[q], 1);
                const int ui = __shfl_up_sync(B200_FULL_MASK, li[q], 1);
                if (lane == ins) {
                    ls[q] = cs;
                    li[q] = ci;
                } else if (lane > ins) {
                    ls[q] = us;
                    li[q] = ui;
                }
                thr[q] = __shfl_sync(B200_FULL_MASK, ls[q], p.kp - 1);
            }
        }
    }

#pragma unroll
    for (int q = 0; q < EX_ROWS_PER_WARP; ++q) {
        const int64_t sel = sel0 + warp * EX_ROWS_PER_WARP + q;
        if (sel >= n_sel) continue;
        const int64_t o = ((int64_t)split * p.part_stride_rows + sel) * LIST_LEN + lane;
        const bool keep = active[q] && lane < p.kp;
        p.part_scores[o] = keep ? ls[q] : -INFINITY;
        p.part_ids[o] = keep ? li[q] : B200_PAD_ID;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Selection kernels: one warp (or block) per row turns candidate lists into the next `kp` output entries.
//   merge_select_kernel   : lists carry final scores (exhaustive-kernel partial lists, per-shard results of an
//                           item-sharded catalogue); optional certificate over per-list bounds.
//   rescore_select_kernel : lists carry approximate (tensor-core) scores; every candidate is re-scored in fp64 from the
//                           master copies (objects: fp32, or fp16 / bf16 widened on load) and the row is certified or
//                           queued for a re-rank (kp <= 32).
//   rescore_wide_kernel   : the same for the wide mode (kp <= 128, up to 512 candidates per row), one block per row;
//   rescore_wide_large_kernel : the wide mode for 128 < kp <= 1024 (up to 4096 candidates per row), one block per row.
// Certificate: every list reports the final pruning threshold `thr` of its stream -- no discarded object had an
// approximate score above it.  With eps = eps_rel * |u|_2 * max_i |i|_2 bounding |approx - exact|, a row whose kp-th exact
// score exceeds max(thr) + eps cannot have lost a top-kp object.
// ---------------------------------------------------------------------------------------------------------------
struct SelectParams {
    const float* in_scores;    // [n_lists][list_stride_rows][L]
    const int32_t* in_ids;     // pad entries: id == B200_PAD_ID (or beyond in_counts)
    const int32_t* in_counts;  // nullable [n_lists][list_stride_rows]
    const float* in_thr;       // rescore: [n_lists][list_stride_rows] final thresholds (approximate-score units)
    int32_t n_lists;
    int32_t L;                 // slots per list
    int64_t n_sel;
    int64_t list_stride_rows;  // rows between consecutive lists (>= n_sel)
    int64_t list_stride_elems; // merge only: elements between the lists of in_scores / in_ids / in_counts / in_bounds when they
                               // live in one packed buffer per list (0: dense [n_lists][rows][L] arrays)
    const int32_t* rows;       // nullable: compact index -> logical row
    int32_t k_out, k0, kp;
    int32_t* out_ids;
    float* out_scores;
    int32_t* out_counts;
    // re-scoring inputs
    const float* subjects;
    const int64_t* row_map;
    const void* objects;       // [n_objects, d] in the re-score kernel's object type TO (fp32, fp16 or bf16)
    const float* obj_norms;
    int32_t d;
    // certificate
    const int32_t* row_exp;   // per batch row: power-of-two exponent applied to the subject before rounding
    int32_t obj_exp;          // exponent applied to the objects
    float eps_rel;            // bound on |approx - exact| / (|u|_2 * max_i |i|_2), see DESIGN.md
    float max_obj_norm;       // max_i |i|_2 (1 for pre-normalised COSINE objects)
    int32_t* fb_count;        // device counter of rows that failed the certificate
    int32_t* fb_rows;         // their logical rows (+ fb_row0)
    int64_t fb_row0;
    // shared-threshold mode (item-sharded multi-GPU): no local verdict; the bound on this shard's discarded scores goes
    // out with the results and the merge certifies the global top-k
    float* out_bounds;        // rescore: nullable [rows] (exact-score units, already includes eps);  merge: unused
    const float* in_bounds;   // merge: nullable [n_lists][rows]
};

// the smallest fp32 that is >= x (bounds are compared against fp32 scores)
__device__ __forceinline__ float round_up_f32(double x) {
    float f = (float)x;
    if ((double)f < x) f = nextafterf(f, INFINITY);
    return f;
}

__global__ void __launch_bounds__(SEL_WARPS * 32) merge_select_kernel(const SelectParams p) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t sel = (int64_t)blockIdx.x * SEL_WARPS + warp;
    if (sel >= p.n_sel) return;
    const int64_t lrow = p.rows ? (int64_t)p.rows[sel] : sel;

    float bs = INFINITY;
    int bi = -1;
    if (p.k0 > 0) {
        if (p.out_counts[lrow] < p.k0) return;
        bs = p.out_scores[lrow * p.k_out + p.k0 - 1];
        bi = p.out_ids[lrow * p.k_out + p.k0 - 1];
    }
    float run_s = -INFINITY;
    int run_i = B200_PAD_ID;
    int n_valid = 0;
    const int total = p.n_lists * p.L;
    for (int base = 0; base < total; base += 32) {
        const int c = base + lane;
        const int list = c / p.L, e = c - list * p.L;
        bool valid = c < total;
        const int64_t lbase = p.list_stride_elems ? (int64_t)list * p.list_stride_elems : (int64_t)list * p.list_stride_rows * p.L;
        const int64_t cbase = p.list_stride_elems ? (int64_t)list * p.list_stride_elems : (int64_t)list * p.list_stride_rows;
        int id = B200_PAD_ID;
        float s = -INFINITY;
        if (valid) {
            const int cnt = p.in_counts ? p.in_counts[cbase + sel] : p.L;
            valid = e < cnt;
            if (valid) {
                id = p.in_ids[lbase + sel * p.L + e];
                s = p.in_scores[lbase + sel * p.L + e];
            }
            valid = valid && id != B200_PAD_ID && id >= 0;
        }
        valid = valid && (s < bs || (s == bs && id > bi));
        if (!valid) {
            s = -INFINITY;
            id = B200_PAD_ID;
        }
        n_valid += __popc(__ballot_sync(B200_FULL_MASK, valid));
        warp_sort32(s, id, lane);
        warp_merge_top32(run_s, run_i, s, id, lane);
    }
    const int n_out = min(n_valid, p.kp);
    if (lane < p.kp) {
        const bool w = lane < n_out;
        p.out_ids[lrow * p.k_out + p.k0 + lane] = w ? run_i : -1;
        p.out_scores[lrow * p.k_out + p.k0 + lane] = w ? run_s : -FLT_MAX;
    }
    if (lane == 0) p.out_counts[lrow] = p.k0 + n_out;
    if (p.in_bounds) {  // global certificate of an item-sharded, threshold-sharing pass
        float b = -INFINITY;
        for (int l = lane; l < p.n_lists; l += 32) {
            const int64_t cbase = p.list_stride_elems ? (int64_t)l * p.list_stride_elems : (int64_t)l * p.list_stride_rows;
            b = fmaxf(b, p.in_bounds[cbase + sel]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) b = fmaxf(b, __shfl_xor_sync(B200_FULL_MASK, b, o));
        const float e_k = __shfl_sync(B200_FULL_MASK, run_s, p.kp - 1);
        const bool ok = !(b > -INFINITY) || (n_valid >= p.kp && e_k > b);
        if (!ok && lane == 0) {
            const int slot = atomicAdd(p.fb_count, 1);
            p.fb_rows[slot] = (int32_t)(lrow + p.fb_row0);
        }
    }
}

// fp64-accumulated dot of the staged subject row with object `id` (the result definition of include/b200_rank.h).  The
// elements are summed in index order whatever the load width, so a 16-bit row gives the sum of its widened fp32 copy.
template <typename TO>
__device__ __forceinline__ float exact_score(const SelectParams& p, const float* sub, int id) {
    double acc = 0.0;
    const TO* orow = static_cast<const TO*>(p.objects) + (int64_t)id * p.d;
    if constexpr (std::is_same<TO, float>::value) {
        // 4 elements per load only where the row starts on a 16-byte boundary: a borrowed matrix (a tensor view, a
        // C-ABI pointer) need only be element-aligned
        if ((p.d & 3) == 0 && (reinterpret_cast<uintptr_t>(orow) & 15) == 0) {
            const float4* o4 = reinterpret_cast<const float4*>(orow);
            const float4* s4 = reinterpret_cast<const float4*>(sub);
            for (int j = 0; j < (p.d >> 2); ++j) {
                const float4 ov = __ldg(o4 + j);
                const float4 sv = s4[j];
                acc = fma((double)ov.x, (double)sv.x, acc);
                acc = fma((double)ov.y, (double)sv.y, acc);
                acc = fma((double)ov.z, (double)sv.z, acc);
                acc = fma((double)ov.w, (double)sv.w, acc);
            }
        } else {
            for (int j = 0; j < p.d; ++j) acc = fma((double)__ldg(orow + j), (double)sub[j], acc);
        }
    } else if ((p.d & 7) == 0 && (reinterpret_cast<uintptr_t>(orow) & 15) == 0) {
        // 16-bit rows that start on a 16-byte boundary (d % 8 == 0, aligned matrix): 8 elements per load
        const uint4* o8 = reinterpret_cast<const uint4*>(orow);
        const float4* s4 = reinterpret_cast<const float4*>(sub);
        for (int j = 0; j < (p.d >> 3); ++j) {
            const uint4 ov = __ldg(o8 + j);
            const float4 sa = s4[2 * j], sb = s4[2 * j + 1];
            acc = fma((double)bits_to_f32<TO>(ov.x), (double)sa.x, acc);
            acc = fma((double)bits_to_f32<TO>(ov.x >> 16), (double)sa.y, acc);
            acc = fma((double)bits_to_f32<TO>(ov.y), (double)sa.z, acc);
            acc = fma((double)bits_to_f32<TO>(ov.y >> 16), (double)sa.w, acc);
            acc = fma((double)bits_to_f32<TO>(ov.z), (double)sb.x, acc);
            acc = fma((double)bits_to_f32<TO>(ov.z >> 16), (double)sb.y, acc);
            acc = fma((double)bits_to_f32<TO>(ov.w), (double)sb.z, acc);
            acc = fma((double)bits_to_f32<TO>(ov.w >> 16), (double)sb.w, acc);
        }
    } else {  // any other 16-bit row: element by element (no head / tail to align)
        for (int j = 0; j < p.d; ++j) acc = fma((double)to_f32(__ldg(orow + j)), (double)sub[j], acc);
    }
    return p.obj_norms ? (float)(acc / (double)__ldg(p.obj_norms + id)) : (float)acc;
}

template <typename TO>
__global__ void __launch_bounds__(SEL_WARPS * 32) rescore_select_kernel(const SelectParams p) {
    extern __shared__ float s_sub[];  // [SEL_WARPS][d] subject rows
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t sel = (int64_t)blockIdx.x * SEL_WARPS + warp;
    if (sel >= p.n_sel) return;
    const int64_t lrow = p.rows ? (int64_t)p.rows[sel] : sel;

    float bs = INFINITY;
    int bi = -1;
    if (p.k0 > 0) {
        if (p.out_counts[lrow] < p.k0) return;
        bs = p.out_scores[lrow * p.k_out + p.k0 - 1];
        bi = p.out_ids[lrow * p.k_out + p.k0 - 1];
    }
    float* sub = s_sub + (size_t)warp * p.d;
    double unorm2 = 0.0;
    {
        const int64_t pr = p.row_map ? p.row_map[lrow] : lrow;
        for (int j = lane; j < p.d; j += 32) {
            const float v = __ldg(p.subjects + pr * p.d + j);
            sub[j] = v;
            unorm2 = fma((double)v, (double)v, unorm2);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) unorm2 += __shfl_xor_sync(B200_FULL_MASK, unorm2, o);
        __syncwarp();
    }
    // list lengths and thresholds: lane l holds list l (at most 16 object splits x two lists: n_lists <= 32)
    int cnt = 0;
    float thr_max = -INFINITY;
    bool overflow = false;
    if (lane < p.n_lists) {
        const int64_t o = (int64_t)lane * p.list_stride_rows + sel;
        const int c = p.in_counts[o];
        overflow = c > p.L;
        cnt = min(c, p.L);
        thr_max = fmaxf(thr_max, p.in_thr[o]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) thr_max = fmaxf(thr_max, __shfl_xor_sync(B200_FULL_MASK, thr_max, o));
    overflow = __any_sync(B200_FULL_MASK, overflow);
    int total = cnt;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(B200_FULL_MASK, total, o);

    // approximate scores are in units scaled by 2^(row_exp + obj_exp); row_exp is indexed by batch row
    const int ex = (p.row_exp ? p.row_exp[sel] : 0) + p.obj_exp;
    const double eps = (double)p.eps_rel * sqrt(unorm2) * (double)p.max_obj_norm;
    const double eps_scaled = ldexp(eps, ex);
    float run_s = -INFINITY;
    int run_i = B200_PAD_ID;
    int n_valid = 0;
    for (int base = 0; base < total; base += 32) {
        // compact index -> (list, entry): the lists are short, so 32 candidates usually cover all of them in one round
        const int ci = base + lane;
        int list = -1, e = 0, acc = 0;
        for (int l = 0; l < p.n_lists; ++l) {
            const int c = __shfl_sync(B200_FULL_MASK, cnt, l);
            if (list < 0 && ci < acc + c) {
                list = l;
                e = ci - acc;
            }
            acc += c;
        }
        bool valid = list >= 0;
        int id = B200_PAD_ID;
        float approx = -INFINITY;
        if (valid) {
            const int64_t o = ((int64_t)list * p.list_stride_rows + sel) * p.L + e;
            id = p.in_ids[o];
            valid = id != B200_PAD_ID && id >= 0;
            if (valid) approx = p.in_scores[o];
        }
        // Candidates that provably cannot reach the top-kp are not re-scored (their 512-byte rows are not gathered): with
        // |approx - exact| <= eps for every candidate, one whose approximate score lies more than 2 eps below the kp-th best
        // approximate score ranks below kp others.  (Single-round rows of a first pass only.)
        bool skip = false;
        if (p.k0 == 0 && total <= 32) {
            float sa = approx;
            int si = lane;
            warp_sort32(sa, si, lane);
            const float a_k = __shfl_sync(B200_FULL_MASK, sa, p.kp - 1);  // -inf with fewer than kp candidates: nothing is skipped
            skip = valid && (double)approx < (double)a_k - 2.0 * eps_scaled * (1.0 + 1e-6);
        }
        float s = -INFINITY;
        if (valid && !skip) s = exact_score<TO>(p, sub, id);
        valid = valid && !skip && (s < bs || (s == bs && id > bi));
        n_valid += __popc(__ballot_sync(B200_FULL_MASK, skip));  // still candidates of the row (the certificate counts them)
        if (!valid) {
            s = -INFINITY;
            id = B200_PAD_ID;
        }
        n_valid += __popc(__ballot_sync(B200_FULL_MASK, valid));
        warp_sort32(s, id, lane);
        warp_merge_top32(run_s, run_i, s, id, lane);
    }

    const int n_out = min(n_valid, p.kp);
    if (lane < p.kp) {
        const bool w = lane < n_out;
        p.out_ids[lrow * p.k_out + p.k0 + lane] = w ? run_i : -1;
        p.out_scores[lrow * p.k_out + p.k0 + lane] = w ? run_s : -FLT_MAX;
    }
    if (lane == 0) p.out_counts[lrow] = p.k0 + n_out;

    const double thr = ldexp((double)thr_max, -ex);
    if (p.out_bounds) {
        // one fp32 ulp of slack: a discarded object whose exact score rounds up to e_k could tie with a smaller id.  The
        // slack is relative to |thr + eps|: a factor (1 + 2.4e-7) would move a negative bound DOWN, below thr + eps.
        if (lane == 0) {
            const double b = thr + eps;
            p.out_bounds[lrow] = overflow ? INFINITY : (thr_max > -INFINITY ? round_up_f32(b + 2.4e-7 * fabs(b) + 1e-37) : -INFINITY);
        }
        return;
    }
    if (thr_max > -INFINITY || overflow) {
        const float e_k = __shfl_sync(B200_FULL_MASK, run_s, p.kp - 1);
        const bool ok = !overflow && n_valid >= p.kp && (double)e_k > thr + eps + 1.2e-7 * fabs((double)e_k);
        if (!ok && lane == 0) {
            const int slot = atomicAdd(p.fb_count, 1);
            p.fb_rows[slot] = (int32_t)(lrow + p.fb_row0);
        }
    }
}

// Wide mode: one block per row.  Two stages: the candidates are sorted by their APPROXIMATE scores first; only those within
// 2 eps of the kp-th best approximate score can reach the exact top-kp (everything below ranks under kp others, see
// rescore_select_kernel) and are re-scored (thread = candidate) -- ~110 of ~180 gathered rows at k = 100 -- then sorted by
// (exact score desc, id asc) with the same bitonic network in shared memory.
//   rescore_wide_kernel       : kp <= 128, up to WIDE_MAX candidates per row, 128 threads, static shared arrays;
//   rescore_wide_large_kernel : 128 < kp <= 1024, up to WIDE_MAX_L candidates per row, 256 threads, the arrays in dynamic
//                               shared memory behind the subject row (32 KiB of score / id pairs at full capacity).
// (WIDE_MAX / WIDE_MAX_L: sizes.h, the host sizes the append lists by them)
constexpr int WIDE_THREADS = 128;
constexpr int WIDE_THREADS_L = 256;

// best-first bitonic sort of s_sc / s_id [0, n), n a power of two (all threads of the block)
template <int THREADS>
__device__ __forceinline__ void block_bitonic_sort(float* s_sc, int* s_id, int n, int tid) {
    for (int k = 2; k <= n; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = tid; i < n; i += THREADS) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const float a = s_sc[i], b = s_sc[ixj];
                    const int ai = s_id[i], bi2 = s_id[ixj];
                    const bool up = (i & k) == 0;  // this pair sorts best-first
                    const bool swap = up ? ranks_before(b, bi2, a, ai) : ranks_before(a, ai, b, bi2);
                    if (swap) {
                        s_sc[i] = b;
                        s_sc[ixj] = a;
                        s_id[i] = bi2;
                        s_id[ixj] = ai;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// sum over the warps of the block (s_part: one slot per warp, written by lane 0 before the barrier that precedes the call)
template <int THREADS, typename T>
__device__ __forceinline__ T warp_slots_sum(const T* s_part) {
    T v = s_part[0];
#pragma unroll
    for (int w = 1; w < THREADS / 32; ++w) v += s_part[w];
    return v;
}

// The body shared by both wide re-score kernels: s_dyn = subject row [d], s_sc / s_id = MAX candidate slots.
template <int THREADS, int MAX, typename TO>
__device__ __forceinline__ void rescore_wide_row(const SelectParams& p, float* s_dyn, float* s_sc, int* s_id) {
    __shared__ int s_off[65];
    __shared__ double s_red[THREADS / 32];
    __shared__ int s_cnt[THREADS / 32];
    __shared__ float s_thr;
    __shared__ int s_flag;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t sel = blockIdx.x;
    const int64_t lrow = p.rows ? (int64_t)p.rows[sel] : sel;

    float bs = INFINITY;
    int bi = -1;
    if (p.k0 > 0) {
        if (p.out_counts[lrow] < p.k0) return;  // block-uniform
        bs = p.out_scores[lrow * p.k_out + p.k0 - 1];
        bi = p.out_ids[lrow * p.k_out + p.k0 - 1];
    }
    double un = 0.0;
    {
        const int64_t pr = p.row_map ? p.row_map[lrow] : lrow;
        for (int j = tid; j < p.d; j += THREADS) {
            const float v = __ldg(p.subjects + pr * p.d + j);
            s_dyn[j] = v;
            un = fma((double)v, (double)v, un);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) un += __shfl_xor_sync(B200_FULL_MASK, un, o);
        if (lane == 0) s_red[warp] = un;
    }
    if (tid == 0) {
        int acc = 0, ovf = 0;
        float tm = -INFINITY;
        for (int l = 0; l < p.n_lists; ++l) {
            const int64_t o = (int64_t)l * p.list_stride_rows + sel;
            const int c = p.in_counts[o];
            ovf |= c > p.L;
            s_off[l] = acc;
            acc += min(c, p.L);
            tm = fmaxf(tm, p.in_thr[o]);
        }
        if (acc > MAX) {  // (cannot happen when the engine keeps n_lists * L <= MAX)
            ovf = 1;
            acc = MAX;
        }
        s_off[p.n_lists] = acc;
        s_thr = tm;
        s_flag = ovf;
    }
    __syncthreads();
    const int total = s_off[p.n_lists];
    const double unorm2 = warp_slots_sum<THREADS>(s_red);
    const int ex = (p.row_exp ? p.row_exp[sel] : 0) + p.obj_exp;
    const double eps = (double)p.eps_rel * sqrt(unorm2) * (double)p.max_obj_norm;
    int n = 2;
    while (n < total) n <<= 1;
    // ---- stage 1: candidates with their approximate scores, best first
    int n_valid = 0;
    for (int c = tid; c < n; c += THREADS) {
        float s = -INFINITY;
        int id = B200_PAD_ID;
        if (c < total) {
            int list = 0;
            while (c >= s_off[list + 1]) ++list;
            const int64_t o = ((int64_t)list * p.list_stride_rows + sel) * p.L + (c - s_off[list]);
            id = p.in_ids[o];
            if (id != B200_PAD_ID && id >= 0) {
                s = p.in_scores[o];
                ++n_valid;
            } else {
                id = B200_PAD_ID;
            }
        }
        s_sc[c] = s;
        s_id[c] = id;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n_valid += __shfl_xor_sync(B200_FULL_MASK, n_valid, o);
    if (lane == 0) s_cnt[warp] = n_valid;
    __syncthreads();
    n_valid = warp_slots_sum<THREADS>(s_cnt);
    block_bitonic_sort<THREADS>(s_sc, s_id, n, tid);
    // ---- the band: [0, m) = candidates that may still reach the exact top-kp (first pass only; later passes re-score all)
    int m = n_valid;
    if (p.k0 == 0 && n_valid > p.kp) {
        const double cut = (double)s_sc[p.kp - 1] - 2.0 * ldexp(eps, ex) * (1.0 + 1e-6);
        int below = 0;  // sorted: the candidates under the cut form a suffix of [0, n_valid)
        for (int c = tid; c < n_valid; c += THREADS) below += (double)s_sc[c] < cut ? 1 : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) below += __shfl_xor_sync(B200_FULL_MASK, below, o);
        __syncthreads();  // (s_cnt is read above by every thread before it is rewritten)
        if (lane == 0) s_cnt[warp] = below;
        __syncthreads();
        m = n_valid - warp_slots_sum<THREADS>(s_cnt);
    }
    __syncthreads();
    // ---- stage 2: exact scores of the band, everything else leaves the ranking
    int n2 = 2;
    while (n2 < m) n2 <<= 1;
    for (int c = tid; c < n; c += THREADS) {
        float s = -INFINITY;
        int id = B200_PAD_ID;
        if (c < m) {
            id = s_id[c];
            s = exact_score<TO>(p, s_dyn, id);
            if (!(s < bs || (s == bs && id > bi))) {  // (later passes: at or above the previous pass's last entry)
                s = -INFINITY;
                id = B200_PAD_ID;
            }
        }
        s_sc[c] = s;
        s_id[c] = id;
    }
    __syncthreads();
    block_bitonic_sort<THREADS>(s_sc, s_id, n2, tid);
    int n_rank = 0;  // candidates still in the ranking (valid ones sort before the (-inf, PAD) fillers)
    for (int i = tid; i < n2; i += THREADS) n_rank += s_id[i] != B200_PAD_ID ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) n_rank += __shfl_xor_sync(B200_FULL_MASK, n_rank, o);
    __syncthreads();
    if (lane == 0) s_cnt[warp] = n_rank;
    __syncthreads();
    n_rank = warp_slots_sum<THREADS>(s_cnt);
    if (p.k0 > 0) n_valid = n_rank;  // later passes: only what survived the bound counts
    const int n_out = min(n_rank, p.kp);
    for (int i = tid; i < p.kp; i += THREADS) {
        const bool w = i < n_out;
        p.out_ids[lrow * p.k_out + p.k0 + i] = w ? s_id[i] : -1;
        p.out_scores[lrow * p.k_out + p.k0 + i] = w ? s_sc[i] : -FLT_MAX;
    }
    if (tid == 0) {
        p.out_counts[lrow] = p.k0 + n_out;
        const bool overflow = s_flag != 0;
        if (s_thr > -INFINITY || overflow) {
            const double thr = ldexp((double)s_thr, -ex);
            const float e_k = n_rank >= p.kp ? s_sc[p.kp - 1] : -INFINITY;
            const bool ok = !overflow && n_valid >= p.kp && n_rank >= p.kp && (double)e_k > thr + eps + 1.2e-7 * fabs((double)e_k);
            if (!ok) {
                const int slot = atomicAdd(p.fb_count, 1);
                p.fb_rows[slot] = (int32_t)(lrow + p.fb_row0);
            }
        }
    }
}

template <typename TO>
__global__ void __launch_bounds__(WIDE_THREADS) rescore_wide_kernel(const SelectParams p) {
    extern __shared__ float s_dyn[];  // [d] subject row
    __shared__ float s_sc[WIDE_MAX];
    __shared__ int s_id[WIDE_MAX];
    rescore_wide_row<WIDE_THREADS, WIDE_MAX, TO>(p, s_dyn, s_sc, s_id);
}

// dynamic shared memory: [d] subject row (rounded up to 4 floats), [WIDE_MAX_L] scores, [WIDE_MAX_L] ids
__host__ __device__ constexpr size_t wide_large_smem(int d) { return ((size_t)(d + 3) / 4 * 4 + 2 * WIDE_MAX_L) * 4; }

template <typename TO>
__global__ void __launch_bounds__(WIDE_THREADS_L) rescore_wide_large_kernel(const SelectParams p) {
    extern __shared__ float s_dyn[];
    float* s_sc = s_dyn + (p.d + 3) / 4 * 4;
    int* s_id = reinterpret_cast<int*>(s_sc + WIDE_MAX_L);
    rescore_wide_row<WIDE_THREADS_L, WIDE_MAX_L, TO>(p, s_dyn, s_sc, s_id);
}

// Multi-pass ranking: the ids a row has received so far, sorted ascending, become the row's exclusion list for the next
// pass (one warp per row, rank counting; unfilled slots sort last as B200_PAD_ID).  rows: nullable subset.
__global__ void build_exclusion_kernel(const int32_t* __restrict__ out_ids, const int32_t* __restrict__ rows, int64_t n_sel, int32_t k_out,
                                       int32_t k0, int32_t id_off, int32_t* __restrict__ excl) {
    const int lane = threadIdx.x & 31;
    const int64_t sel = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (sel >= n_sel) return;
    const int64_t row = rows ? (int64_t)rows[sel] : sel;
    const int32_t* src = out_ids + row * k_out;
    for (int i = lane; i < k0; i += 32) {
        const int32_t raw = src[i];
        const int32_t key = raw < 0 ? B200_PAD_ID : raw + id_off;  // the kernels compare GLOBAL ids
        int rank = 0;
        for (int j = 0; j < k0; ++j) {
            const int32_t rj = src[j];
            const int32_t kj = rj < 0 ? B200_PAD_ID : rj + id_off;
            rank += (kj < key || (kj == key && j < i)) ? 1 : 0;
        }
        excl[row * k_out + rank] = key;
    }
}

// Local object ids -> global ids of an item-sharded catalogue (unfilled slots stay -1).
__global__ void add_offset_kernel(int32_t* ids, int64_t n, int32_t off) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && ids[i] >= 0) ids[i] += off;
}
// The same for a subset of rows (rows re-ranked after the main pass).
__global__ void add_offset_rows_kernel(int32_t* ids, const int32_t* __restrict__ rows, int64_t n_sel, int32_t k_out, int32_t off) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_sel * k_out) return;
    const int64_t o = (int64_t)rows[i / k_out] * k_out + i % k_out;
    if (ids[o] >= 0) ids[o] += off;
}

// Initialise the output arrays: ids = -1, scores = -FLT_MAX, counts = 0.
__global__ void init_outputs_kernel(int32_t* ids, float* scores, int32_t* counts, int64_t n_rows, int32_t k_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_rows * k_out) {
        ids[i] = -1;
        scores[i] = -FLT_MAX;
    }
    if (i < n_rows) counts[i] = 0;
}
// The same for a subset of rows.
__global__ void init_rows_kernel(int32_t* ids, float* scores, int32_t* counts, const int32_t* __restrict__ rows, int64_t n_sel,
                                 int32_t k_out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_sel * k_out) return;
    const int64_t r = rows[i / k_out];
    ids[r * k_out + i % k_out] = -1;
    scores[r * k_out + i % k_out] = -FLT_MAX;
    if (i % k_out == 0) counts[r] = 0;
}

// Rows re-ranked after their chunk was copied back: packed copies [n_sel][k_out] (+ counts) for one more small transfer.
__global__ void gather_rows_kernel(const int32_t* __restrict__ ids, const float* __restrict__ scores, const int32_t* __restrict__ counts,
                                   const int32_t* __restrict__ rows, int64_t n_sel, int32_t k_out, int32_t* __restrict__ g_ids,
                                   float* __restrict__ g_scores, int32_t* __restrict__ g_counts) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_sel * k_out) return;
    const int64_t r = rows[i / k_out];
    g_ids[i] = ids[r * k_out + i % k_out];
    g_scores[i] = scores[r * k_out + i % k_out];
    if (i % k_out == 0) g_counts[i / k_out] = counts[r];
}

// Start positions of the carousel: front[s] = first tile of split s, every work item's start slot undecided (-1).
__global__ void carousel_init_kernel(int32_t* buf, int32_t n_splits, int32_t tiles_per_split, int64_t n_ints) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_ints) buf[i] = i < n_splits ? (int32_t)i * tiles_per_split : -1;
}

}  // namespace b200
