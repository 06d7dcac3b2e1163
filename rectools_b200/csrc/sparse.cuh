// Sparse-subject scorer: `EASEModel` hands the ranker the user x item interaction CSR as SUBJECT factors and the dense
// item x item weight matrix as object factors (rectools/models/ease.py:134-161; `ImplicitRanker` accepts CSR subjects
// for Distance.DOT only, rank_implicit.py:66-67, and densifies the requested rows, :236 / :157-159).  Here the rows stay
// sparse:  score(u, i) = sum_{j in row u} x_uj * O[i, j]  is a gather of nnz(u) rows of the TRANSPOSED object matrix
// O^T [d, n_objects] -- an HBM / L2 bound SpMM, not a GEMM -- accumulated in fp64 and rounded once to fp32 (the result
// definition of include/b200_rank.h), followed by a streaming warp-per-row top-k over the materialised score rows of a
// bounded row chunk.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int SP_THREADS = 256;
constexpr int SP_COLS = 4;                      // positions per thread
constexpr int SP_BLOCK_COLS = SP_THREADS * SP_COLS;

// grid (rows, column blocks): rows vary fastest, so the blocks running together read the same column panel of O^T
// (d x 4 KiB = 80 MB at d = 20 K: L2 resident) for different sparse rows.
__global__ void __launch_bounds__(SP_THREADS) sparse_scores_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                                                                   const float* __restrict__ data, const float* __restrict__ objT,
                                                                   int64_t n_obj, int32_t d, const int32_t* __restrict__ pos2obj,
                                                                   int64_t n_pos, float* __restrict__ scores) {
    __shared__ int32_t s_j[SP_THREADS];
    __shared__ float s_x[SP_THREADS];
    const int64_t row = blockIdx.x;
    const int64_t pos0 = (int64_t)blockIdx.y * SP_BLOCK_COLS + (int64_t)threadIdx.x * SP_COLS;
    const int64_t lo = indptr[row], hi = indptr[row + 1];
    double acc[SP_COLS] = {0.0, 0.0, 0.0, 0.0};
    int64_t obj[SP_COLS];
    bool contiguous = pos2obj == nullptr && pos0 + SP_COLS <= n_pos && (n_obj & 3) == 0;
#pragma unroll
    for (int c = 0; c < SP_COLS; ++c) {
        const int64_t pos = pos0 + c;
        obj[c] = pos < n_pos ? (pos2obj ? (int64_t)pos2obj[pos] : pos) : -1;
    }
    for (int64_t base = lo; base < hi; base += SP_THREADS) {
        __syncthreads();
        const int64_t e = base + threadIdx.x;
        if (e < hi) {
            const int32_t j = indices[e];
            s_j[threadIdx.x] = (j >= 0 && j < d) ? j : -1;  // columns beyond the factor dimension contribute nothing
            s_x[threadIdx.x] = data[e];
        }
        __syncthreads();
        const int n = (int)((hi - base) < (int64_t)SP_THREADS ? (hi - base) : (int64_t)SP_THREADS);
        for (int t = 0; t < n; ++t) {
            const int32_t j = s_j[t];
            if (j < 0) continue;
            const double x = (double)s_x[t];
            const float* w = objT + (int64_t)j * n_obj;
            if (contiguous) {
                const float4 v = __ldg(reinterpret_cast<const float4*>(w + pos0));
                acc[0] = fma(x, (double)v.x, acc[0]);
                acc[1] = fma(x, (double)v.y, acc[1]);
                acc[2] = fma(x, (double)v.z, acc[2]);
                acc[3] = fma(x, (double)v.w, acc[3]);
            } else {
#pragma unroll
                for (int c = 0; c < SP_COLS; ++c)
                    if (obj[c] >= 0) acc[c] = fma(x, (double)__ldg(w + obj[c]), acc[c]);
            }
        }
    }
#pragma unroll
    for (int c = 0; c < SP_COLS; ++c)
        if (obj[c] >= 0) scores[row * n_pos + pos0 + c] = (float)acc[c];
}

// Dense subjects, k > 128 (k = None: "all objects", rank_implicit.py:233-234): score rows are materialised ONCE with the
// exhaustive kernel's arithmetic (fp64-accumulated dot, / norm for COSINE, rounded to fp32) and the k / 32 selection passes
// stream 4-byte scores instead of repeating 2 d fp64 FLOP per object and pass.
// Block = 32 subjects x 32 positions per step (lane = position), grid (row blocks, position splits).
// `rows` (nullable): entry r of the batch is logical row rows[r] (the rows a wide pass could not certify); score row r of
// the output stays compact.
// TO: the stored object type (fp32, fp16 or bf16), widened on load.
constexpr int DS_DK = 64;

template <typename TO>
__global__ void __launch_bounds__(256) dense_scores_kernel(const float* __restrict__ subjects, const int64_t* __restrict__ row_map,
                                                           const int32_t* __restrict__ rows, int64_t n_rows, const TO* __restrict__ objects,
                                                           const int32_t* __restrict__ pos2obj, int64_t n_pos, int32_t d,
                                                           const float* __restrict__ obj_norms, float* __restrict__ scores) {
    __shared__ float s_obj[32][DS_DK + 1];
    __shared__ float s_sub[32][DS_DK];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int64_t row0 = (int64_t)blockIdx.x * 32;
    const int64_t tiles_total = (n_pos + 31) >> 5;
    const int64_t tiles_per = (tiles_total + gridDim.y - 1) / gridDim.y;
    const int64_t t0 = blockIdx.y * tiles_per, t1 = min(t0 + tiles_per, tiles_total);
    for (int64_t t = t0; t < t1; ++t) {
        double acc[4] = {0.0, 0.0, 0.0, 0.0};
        for (int dk0 = 0; dk0 < d; dk0 += DS_DK) {
            __syncthreads();
            for (int e = tid; e < 32 * DS_DK; e += 256) {
                const int it = e >> 6, j = e & (DS_DK - 1);
                const int64_t pos = t * 32 + it;
                float v = 0.f;
                if (pos < n_pos && dk0 + j < d) {
                    const int64_t obj = pos2obj ? (int64_t)pos2obj[pos] : pos;
                    v = to_f32(__ldg(objects + obj * d + dk0 + j));
                }
                s_obj[it][j] = v;
                const int64_t r = row0 + it;
                float u = 0.f;
                if (r < n_rows && dk0 + j < d) {
                    const int64_t lr = rows ? (int64_t)rows[r] : r;
                    u = __ldg(subjects + (row_map ? row_map[lr] : lr) * d + dk0 + j);
                }
                s_sub[it][j] = u;
            }
            __syncthreads();
            const int jn = min(DS_DK, d - dk0);
            for (int j = 0; j < jn; ++j) {
                const double ov = (double)s_obj[lane][j];
#pragma unroll
                for (int q = 0; q < 4; ++q) acc[q] = fma(ov, (double)s_sub[warp * 4 + q][j], acc[q]);
            }
        }
        const int64_t pos = t * 32 + lane;
        if (pos < n_pos) {
            const int obj = pos2obj ? pos2obj[pos] : (int)pos;
            const double nrm = obj_norms ? (double)__ldg(obj_norms + obj) : 1.0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int64_t r = row0 + warp * 4 + q;
                if (r < n_rows) scores[r * n_pos + pos] = obj_norms ? (float)(acc[q] / nrm) : (float)acc[q];
            }
        }
    }
}

// One warp per row: streaming top-kp (kp <= 32) over a materialised score row, order (score desc, id asc), objects listed
// in the row's filter_pairs_csr slice never returned; entries [k0, k0 + kp) of a k > 32 query are bounded by the previous
// pass's last entry exactly as in exact_topk_kernel.  `rows` (nullable): score row r belongs to logical row rows[r], which
// indexes the filter and the outputs.
__global__ void __launch_bounds__(256) scores_topk_kernel(const float* __restrict__ scores, const int32_t* __restrict__ rows, int64_t n_rows,
                                                          int64_t n_pos,
                                                          const int32_t* __restrict__ pos2obj, const int64_t* __restrict__ f_indptr,
                                                          const int32_t* __restrict__ f_indices, int32_t id_off, int32_t k_out, int32_t k0,
                                                          int32_t kp, int32_t* __restrict__ out_ids, float* __restrict__ out_scores,
                                                          int32_t* __restrict__ out_counts) {
    const int lane = threadIdx.x & 31;
    const int64_t sr = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (sr >= n_rows) return;
    const int64_t row = rows ? (int64_t)rows[sr] : sr;
    float bs = INFINITY;
    int bi = -1;
    if (k0 > 0) {
        if (out_counts[row] < k0) return;
        bs = out_scores[row * k_out + k0 - 1];
        bi = out_ids[row * k_out + k0 - 1];
    }
    int64_t flo = 0, fhi = 0;
    if (f_indptr) {
        flo = f_indptr[row];
        fhi = f_indptr[row + 1];
    }
    float thr = -INFINITY, ls = -INFINITY;
    int li = B200_PAD_ID;
    const float* srow = scores + sr * n_pos;
    for (int64_t p0 = 0; p0 < n_pos; p0 += 32) {
        const int64_t pos = p0 + lane;
        const bool valid = pos < n_pos;
        const float s = valid ? __ldg(srow + pos) : -INFINITY;
        const int obj = valid ? (pos2obj ? pos2obj[pos] : (int)pos) : B200_PAD_ID;
        bool c = valid && s > thr && (s < bs || (s == bs && obj > bi));
        if (c && f_indptr) c = !csr_contains(f_indices, flo, fhi, obj + id_off);
        unsigned m = __ballot_sync(B200_FULL_MASK, c);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const float cs = __shfl_sync(B200_FULL_MASK, s, src);
            const int ci = __shfl_sync(B200_FULL_MASK, obj, src);
            if (!(cs > thr)) continue;  // threshold rose while draining this ballot
            const int ins = __popc(__ballot_sync(B200_FULL_MASK, ls >= cs));
            const float us = __shfl_up_sync(B200_FULL_MASK, ls, 1);
            const int ui = __shfl_up_sync(B200_FULL_MASK, li, 1);
            if (lane == ins) {
                ls = cs;
                li = ci;
            } else if (lane > ins) {
                ls = us;
                li = ui;
            }
            thr = __shfl_sync(B200_FULL_MASK, ls, kp - 1);
        }
    }
    const int n_out = __popc(__ballot_sync(B200_FULL_MASK, lane < kp && li != B200_PAD_ID));
    if (lane < kp) {
        const bool w = lane < n_out;
        out_ids[row * k_out + k0 + lane] = w ? li : -1;
        out_scores[row * k_out + k0 + lane] = w ? ls : -FLT_MAX;
    }
    if (lane == 0) out_counts[row] = k0 + n_out;
}

}  // namespace b200
