// libb200rank.so -- ItemKNN user scores (path 9, b200_rank_topk_knn): `ImplicitItemKNNWrapperModel._recommend_u2i`
// (rectools/models/implicit_knn.py:152-211), which calls implicit's `recommend` once per user, without the per-user loop.
// No engine: S is uploaded once per call and the call owns its stream and scratch.  Every refusal is decided on the host
// by plan_knn (knn_plan.h) before the device is touched.  Per chunk of rows, the kernels of knn.cuh accumulate each row's
// scores and write its candidates as (row, fp64 score) pairs in ascending item id; b200_rank_topk_pairs (path 6) selects
// each row's k best on the device, which orders them by (score desc, position asc) = (score desc, id asc).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
#include "engine_internal.h"
#include "knn.cuh"
#include "knn_plan.h"

namespace {

// Dense-route scratch: at most this many bytes of fp64 rows and flags, and no more CTAs than two per SM.
constexpr int64_t KNN_DENSE_BYTES = (int64_t)1 << 28;

}  // namespace

extern "C" int b200_rank_topk_knn(int32_t device, int64_t n_items, const int64_t* s_indptr, const int32_t* s_indices,
                                  const double* s_data, int64_t n_rows, const int64_t* u_indptr, const int32_t* u_indices,
                                  const float* u_data, const int64_t* f_indptr, const int32_t* f_indices, const int32_t* whitelist,
                                  int64_t n_whitelist, int32_t k, int32_t* out_ids, double* out_scores, int32_t* out_counts,
                                  b200_rank_stats* stats) {
    using namespace b200;
    KnnArgs args;
    args.n_items = n_items;
    args.s_indptr = s_indptr;
    args.s_indices = s_indices;
    args.s_data = s_data;
    args.n_rows = n_rows;
    args.u_indptr = u_indptr;
    args.u_indices = u_indices;
    args.u_data = u_data;
    args.f_indptr = f_indptr;
    args.f_indices = f_indices;
    args.whitelist = whitelist;
    args.n_whitelist = n_whitelist;
    args.k = k;
    args.outputs = out_ids && out_scores && out_counts;
    const KnnPlan P = plan_knn(args, knn_chunk_rows_hook());
    if (P.error != B200_OK) return b200_set_error(P.error, P.message.c_str());
    b200_rank_stats S{};
    S.path = 9;
    S.k_out = k;
    if (P.n_chunks() == 0) {
        if (stats) *stats = S;
        return B200_OK;
    }
    const int64_t s_nnz = s_indptr[n_items];
    const bool wl = n_whitelist >= 0;
    try {
        CK(cudaSetDevice(device));
        int sms = 0;
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        CallScratch<6> R;
        cudaStream_t st = R.st;
        // every allocation before the first output write: a failed one leaves the outputs untouched
        const int64_t mr = P.max_chunk_rows;
        int64_t* d_s_indptr = R.get<int64_t>(n_items + 1);
        int32_t* d_s_indices = R.get<int32_t>(s_nnz);
        double* d_s_data = R.get<double>(s_nnz);
        int32_t* d_wl = wl ? R.get<int32_t>(n_whitelist) : nullptr;
        int64_t* d_u_indptr = R.get<int64_t>(mr + 1);
        int32_t* d_u_indices = R.get<int32_t>(P.max_chunk_u);
        float* d_u_data = R.get<float>(P.max_chunk_u);
        int64_t* d_f_indptr = f_indptr ? R.get<int64_t>(mr + 1) : nullptr;
        int32_t* d_f_indices = f_indptr ? R.get<int32_t>(P.max_chunk_f) : nullptr;
        int64_t* d_slot = R.get<int64_t>(mr + 1);
        int32_t* d_route = R.get<int32_t>(mr);
        int64_t* d_code = R.get<int64_t>(P.max_chunk_slots);
        double* d_score = R.get<double>(P.max_chunk_slots);
        int32_t* d_id = R.get<int32_t>(P.max_chunk_slots);
        int64_t* d_pos = R.get<int64_t>(std::min<int64_t>(P.max_chunk_slots, mr * k));
        int64_t* d_off = R.get<int64_t>(mr + 1);
        int32_t* d_ids = R.get<int32_t>(mr * k);
        double* d_scores = R.get<double>(mr * k);
        int32_t* d_counts = R.get<int32_t>(mr);
        int64_t dense_ctas = 0;
        double* d_acc = nullptr;
        uint8_t* d_touched = nullptr;
        if (P.max_chunk_dense > 0) {
            dense_ctas = std::max<int64_t>(1, std::min<int64_t>({P.max_chunk_dense, 2 * (int64_t)sms, KNN_DENSE_BYTES / (9 * std::max<int64_t>(n_items, 1))}));
            d_acc = R.get<double>(dense_ctas * n_items);
            d_touched = R.get<uint8_t>(dense_ctas * n_items);
            CK(cudaMemsetAsync(d_touched, 0, dense_ctas * n_items, st));
        }
        const int smem = (int)sizeof(KnnTableSmem);
        CK(cudaFuncSetAttribute(knn_table_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        int key_bits = 1;
        while (key_bits < 31 && ((int64_t)1 << key_bits) <= n_items) ++key_bits;  // n_items (the empty key) fits

        CK(cudaEventRecord(R.ev[0], st));
        CK(cudaMemcpyAsync(d_s_indptr, s_indptr, sizeof(int64_t) * (n_items + 1), cudaMemcpyHostToDevice, st));
        if (s_nnz > 0) {
            CK(cudaMemcpyAsync(d_s_indices, s_indices, sizeof(int32_t) * s_nnz, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_s_data, s_data, sizeof(double) * s_nnz, cudaMemcpyHostToDevice, st));
        }
        if (wl && n_whitelist > 0) CK(cudaMemcpyAsync(d_wl, whitelist, sizeof(int32_t) * n_whitelist, cudaMemcpyHostToDevice, st));
        S.h2d_bytes += (int64_t)(sizeof(int64_t) * (n_items + 1) + 12 * s_nnz + (wl ? 4 * n_whitelist : 0));

        std::vector<int64_t> slot(mr + 1);
        std::vector<int32_t> route(mr);
        for (int64_t c = 0; c < P.n_chunks(); ++c) {
            const int64_t r0 = P.bounds[c], r1 = P.bounds[c + 1], nr = r1 - r0;
            if (c > 0) CK(cudaEventRecord(R.ev[0], st));
            // rows whose bound fits the table first, then the dense ones
            int64_t n_table = 0;
            for (int64_t r = r0; r < r1; ++r)
                if (P.bound[r] <= KNN_TABLE_BOUND) route[n_table++] = (int32_t)(r - r0);
            int64_t n_dense = 0;
            for (int64_t r = r0; r < r1; ++r)
                if (P.bound[r] > KNN_TABLE_BOUND) route[n_table + n_dense++] = (int32_t)(r - r0);
            for (int64_t r = r0; r <= r1; ++r) slot[r - r0] = P.slot[r] - P.slot[r0];
            const int64_t n_slots = slot[nr];
            const int64_t u0 = u_indptr[r0], nu = u_indptr[r1] - u0;
            CK(cudaMemcpyAsync(d_u_indptr, u_indptr + r0, sizeof(int64_t) * (nr + 1), cudaMemcpyHostToDevice, st));
            if (nu > 0) {
                CK(cudaMemcpyAsync(d_u_indices, u_indices + u0, sizeof(int32_t) * nu, cudaMemcpyHostToDevice, st));
                CK(cudaMemcpyAsync(d_u_data, u_data + u0, sizeof(float) * nu, cudaMemcpyHostToDevice, st));
            }
            int64_t f0 = 0, nf = 0;
            if (f_indptr) {
                f0 = f_indptr[r0];
                nf = f_indptr[r1] - f0;
                CK(cudaMemcpyAsync(d_f_indptr, f_indptr + r0, sizeof(int64_t) * (nr + 1), cudaMemcpyHostToDevice, st));
                if (nf > 0) CK(cudaMemcpyAsync(d_f_indices, f_indices + f0, sizeof(int32_t) * nf, cudaMemcpyHostToDevice, st));
            }
            CK(cudaMemcpyAsync(d_slot, slot.data(), sizeof(int64_t) * (nr + 1), cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_route, route.data(), sizeof(int32_t) * nr, cudaMemcpyHostToDevice, st));
            S.h2d_bytes += (int64_t)(24 * (nr + 1) + 8 * nu + 4 * nf + 4 * nr);
            CK(cudaEventRecord(R.ev[1], st));

            // ---- scores, and each row's candidates in ascending id
            const KnnRows a{n_items, d_s_indptr, d_s_indices, d_s_data, d_u_indptr, u0, d_u_indices, d_u_data,
                            f_indptr ? d_f_indptr : nullptr, f0, d_f_indices, d_wl, wl ? n_whitelist : 0, d_slot, d_code, d_score, d_id};
            if (n_slots > 0) CK(cudaMemsetAsync(d_code, 0xff, sizeof(int64_t) * n_slots, st));  // -1: an unused slot
            if (n_table > 0) {
                knn_table_kernel<<<(unsigned)n_table, KNN_THREADS, smem, st>>>(a, d_route, key_bits);
                CK(cudaGetLastError());
                ++S.n_launches;
            }
            if (n_dense > 0) {
                knn_dense_kernel<<<(unsigned)std::min(n_dense, dense_ctas), KNN_THREADS, 0, st>>>(a, d_route + n_table, n_dense, d_acc,
                                                                                                 d_touched);
                CK(cudaGetLastError());
                ++S.n_launches;
            }
            CK(cudaEventRecord(R.ev[2], st));

            // ---- each row's k best (path 6 on the device buffers), then positions back to ids and scores
            b200_rank_stats ps{};
            const int rc = b200_rank_topk_pairs(device, st, n_slots, d_code, d_score, B200_PAIRS_F64, nr, k,
                                                B200_Q_INPUTS_ON_DEVICE | B200_Q_OUTPUTS_ON_DEVICE, d_pos, d_off, &ps);
            if (rc != B200_OK) return rc;  // its message stands
            S.n_launches += ps.n_launches;
            const int64_t cells = nr * (int64_t)k;
            knn_gather_kernel<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>((cells + 255) / 256, 16 * (int64_t)sms)), 256, 0, st>>>(
                nr, k, d_off, d_pos, d_id, d_score, d_ids, d_scores, d_counts);
            CK(cudaGetLastError());
            ++S.n_launches;
            CK(cudaEventRecord(R.ev[3], st));
            CK(cudaMemcpyAsync(out_ids + r0 * (int64_t)k, d_ids, sizeof(int32_t) * cells, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(out_scores + r0 * (int64_t)k, d_scores, sizeof(double) * cells, cudaMemcpyDeviceToHost, st));
            CK(cudaMemcpyAsync(out_counts + r0, d_counts, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost, st));
            S.d2h_bytes += (int64_t)(12 * cells + 4 * nr);
            CK(cudaEventRecord(R.ev[4], st));
            CK(cudaStreamSynchronize(st));  // the chunk's device buffers are reused by the next one
            S.ms_h2d += R.ms(0, 1);
            S.ms_main += R.ms(1, 2);
            S.ms_select += R.ms(2, 3);
            S.ms_d2h += R.ms(3, 4);
        }
        S.ms_total = S.ms_h2d + S.ms_main + S.ms_select + S.ms_d2h;
        S.n_chunks = (int32_t)P.n_chunks();
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk_knn", ce);
    }
    if (stats) *stats = S;
    return B200_OK;
}
