// libb200rank.so -- RecTools' classification and ranking metrics (path 10, b200_rank_metrics): the join of
// `merge_reco` (rectools/metrics/base.py:81-103) and the per-user groupbys of `calc_confusions`, `NDCG`, `MRR` and
// `MAP.fit` (rectools/metrics/classification.py:503-538, ranking.py:173-234, 422-572) on the device.  No engine: the call
// owns its scratch and runs on the caller's stream (or its own).  Every refusal is decided on the host by plan_metrics
// (metrics_plan.h) before the device is touched.  The kernels are in metrics.cuh; the means and the metric formulas stay
// with the caller, which feeds these per-user arrays to the stock pandas code.
#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <cstdint>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
#include "engine_internal.h"
#include "metrics.cuh"
#include "metrics_plan.h"

extern "C" int b200_rank_metrics(int32_t device, void* stream, int64_t n_inter, const int64_t* inter_users,
                                 const int64_t* inter_items, int64_t n_reco, const int64_t* reco_users, const int64_t* reco_items,
                                 const int64_t* reco_ranks, int32_t n_k, const int64_t* ks, int32_t n_ndcg,
                                 const int64_t* ndcg_offsets, const double* ndcg_terms, int64_t* out_n_users, int64_t* out_users,
                                 int64_t* out_first_order, int64_t* out_liked, int64_t* out_min_rank, int64_t* out_tp,
                                 double* out_map, double* out_ndcg, int32_t* out_flags, b200_rank_stats* stats) {
    using namespace b200;
    MetricsArgs args;
    args.n_inter = n_inter;
    args.inter = inter_users && inter_items;
    args.n_reco = n_reco;
    args.reco = reco_users && reco_items && reco_ranks;
    args.n_k = n_k;
    args.ks = ks;
    args.n_ndcg = n_ndcg;
    args.ndcg_offsets = ndcg_offsets;
    args.ndcg_terms = ndcg_terms != nullptr;
    args.outputs = out_n_users && out_users && out_first_order && out_liked && out_min_rank && out_flags;
    args.out_tp = out_tp != nullptr;
    args.out_ndcg = out_ndcg != nullptr;
    const bool map = out_map != nullptr;
    const MetricsPlan P = plan_metrics(args, map);
    if (P.error != B200_OK) return b200_set_error(P.error, P.message.c_str());
    b200_rank_stats S{};
    S.path = 10;
    if (n_inter == 0) {
        if (out_n_users) *out_n_users = 0;
        if (out_flags) *out_flags = 0;
        if (stats) *stats = S;
        return B200_OK;
    }
    const int64_t n = n_inter, m = n_reco;
    try {
        CK(cudaSetDevice(device));
        int sms = 0;
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        CallScratch<5> R(static_cast<cudaStream_t>(stream));
        cudaStream_t st = R.st;
        // every allocation before the first output write: a failed one leaves the outputs untouched
        int64_t* d_iu = R.get<int64_t>(n);
        int64_t* d_ii = R.get<int64_t>(n);
        int64_t* d_ru = R.get<int64_t>(m);
        int64_t* d_ri = R.get<int64_t>(m);
        int64_t* d_rr = R.get<int64_t>(m);
        int32_t* d_slot = R.get<int32_t>(P.slots);
        int64_t* d_ks = R.get<int64_t>(n_k);
        int64_t* d_toff = R.get<int64_t>(n_ndcg + 1);
        double* d_terms = R.get<double>(P.n_terms);
        uint32_t* d_flags = R.get<uint32_t>(1);
        int64_t* d_nruns = R.get<int64_t>(1);
        int64_t* d_hit = R.get<int64_t>(n);
        int32_t* d_row = R.get<int32_t>(n);
        int64_t* d_su = R.get<int64_t>(n);
        int32_t* d_srow = R.get<int32_t>(n);
        int64_t* d_users = R.get<int64_t>(n);
        int64_t* d_cnt = R.get<int64_t>(n);
        int64_t* d_off = R.get<int64_t>(n);
        int32_t* d_first = R.get<int32_t>(n);
        int64_t* d_seg = R.get<int64_t>(n);
        int32_t* d_first_s = R.get<int32_t>(n);
        int64_t* d_order = R.get<int64_t>(n);
        int64_t* d_min = R.get<int64_t>(n);
        int64_t* d_tp = R.get<int64_t>(n * n_k);
        double* d_ndcg = R.get<double>(n * n_ndcg);
        uint64_t *d_keys = nullptr, *d_keys_s = nullptr;
        int64_t *d_hcount = nullptr, *d_hoff = nullptr;
        double *d_prec = nullptr, *d_map = nullptr;
        if (map) {
            d_keys = R.get<uint64_t>(n);
            d_keys_s = R.get<uint64_t>(n);
            d_prec = R.get<double>(n);
            d_hcount = R.get<int64_t>(n);
            d_hoff = R.get<int64_t>(n);
            d_map = R.get<double>(n * n_k);
        }
        // CUB scratch: the largest of the call's device-wide primitives, at their largest sizes
        size_t tmp_bytes = 0, b = 0;
        CK(cub::DeviceRadixSort::SortPairs(nullptr, b, d_iu, d_su, d_row, d_srow, (int)n, 0, 64, st));
        tmp_bytes = std::max(tmp_bytes, b);
        CK(cub::DeviceRunLengthEncode::Encode(nullptr, b, d_su, d_users, d_cnt, d_nruns, (int)n, st));
        tmp_bytes = std::max(tmp_bytes, b);
        CK(cub::DeviceScan::ExclusiveSum(nullptr, b, d_cnt, d_off, (int)n, st));
        tmp_bytes = std::max(tmp_bytes, b);
        CK(cub::DeviceRadixSort::SortPairs(nullptr, b, d_first, d_first_s, d_seg, d_order, (int)n, 0, 32, st));
        tmp_bytes = std::max(tmp_bytes, b);
        if (map) {
            CK(cub::DeviceRadixSort::SortKeys(nullptr, b, d_keys, d_keys_s, (int)n, 0, 64, st));
            tmp_bytes = std::max(tmp_bytes, b);
        }
        void* d_tmp = R.get<uint8_t>(tmp_bytes);

        CK(cudaEventRecord(R.ev[0], st));
        CK(cudaMemcpyAsync(d_iu, inter_users, sizeof(int64_t) * n, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(d_ii, inter_items, sizeof(int64_t) * n, cudaMemcpyHostToDevice, st));
        if (m > 0) {
            CK(cudaMemcpyAsync(d_ru, reco_users, sizeof(int64_t) * m, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_ri, reco_items, sizeof(int64_t) * m, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_rr, reco_ranks, sizeof(int64_t) * m, cudaMemcpyHostToDevice, st));
        }
        if (n_k > 0) CK(cudaMemcpyAsync(d_ks, ks, sizeof(int64_t) * n_k, cudaMemcpyHostToDevice, st));
        if (n_ndcg > 0) {
            CK(cudaMemcpyAsync(d_toff, ndcg_offsets, sizeof(int64_t) * (n_ndcg + 1), cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_terms, ndcg_terms, sizeof(double) * P.n_terms, cudaMemcpyHostToDevice, st));
        }
        S.h2d_bytes = 16 * n + 24 * m + 8 * n_k + (n_ndcg > 0 ? 8 * (n_ndcg + 1) + 8 * P.n_terms : 0);
        CK(cudaEventRecord(R.ev[1], st));

        // ---- the join: every reco pair into the table, then each interaction row's rank
        const auto grid = [&](int64_t work) {
            return (unsigned)std::max<int64_t>(1, std::min<int64_t>((work + METRICS_THREADS - 1) / METRICS_THREADS, 32 * (int64_t)sms));
        };
        CK(cudaMemsetAsync(d_slot, 0xff, sizeof(int32_t) * P.slots, st));
        CK(cudaMemsetAsync(d_flags, 0, sizeof(uint32_t), st));
        if (m > 0) {
            metrics_insert_kernel<<<grid(m), METRICS_THREADS, 0, st>>>(m, d_ru, d_ri, d_rr, d_slot, (uint64_t)(P.slots - 1), d_flags);
            CK(cudaGetLastError());
            ++S.n_launches;
        }
        uint32_t flags = 0;
        CK(cudaMemcpyAsync(&flags, d_flags, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (flags != 0) {  // the caller's stock path takes the call: nothing else is computed
            CK(cudaEventRecord(R.ev[2], st));
            CK(cudaEventSynchronize(R.ev[2]));
            S.ms_h2d = R.ms(0, 1);
            S.ms_main = R.ms(1, 2);
            S.ms_total = S.ms_h2d + S.ms_main;
            *out_flags = (int32_t)flags;
            *out_n_users = 0;
            if (stats) *stats = S;
            return B200_OK;
        }
        metrics_probe_kernel<<<grid(n), METRICS_THREADS, 0, st>>>(n, d_iu, d_ii, d_ru, d_ri, d_rr, d_slot, (uint64_t)(P.slots - 1),
                                                                   d_hit, d_row);
        CK(cudaGetLastError());
        ++S.n_launches;

        // ---- user segments: a stable sort of the row indices by user (rows stay in interaction order within a user)
        CK(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_iu, d_su, d_row, d_srow, (int)n, 0, 64, st));
        CK(cub::DeviceRunLengthEncode::Encode(d_tmp, tmp_bytes, d_su, d_users, d_cnt, d_nruns, (int)n, st));
        S.n_launches += 2;
        int64_t U = 0;
        CK(cudaMemcpyAsync(&U, d_nruns, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        CK(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_cnt, d_off, (int)U, st));
        // first-appearance order: the segments sorted by their first row
        metrics_first_kernel<<<grid(U), METRICS_THREADS, 0, st>>>(U, d_off, d_srow, d_first, d_seg);
        CK(cudaGetLastError());
        CK(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_first, d_first_s, d_seg, d_order, (int)U, 0, 32, st));
        S.n_launches += 3;

        // ---- per-user reductions
        const int rbits = map ? std::max(1, metrics_bits((uint64_t)P.k_max)) : 0;
        const int key_bits = map ? std::max(1, metrics_bits((uint64_t)U)) + rbits : 0;
        MetricsUsers a{U, n, d_off, d_cnt, d_srow, d_hit, n_k, d_ks, d_tp, d_min, n_ndcg, d_toff, d_terms, d_ndcg,
                       P.k_max, rbits, map ? (((uint64_t)1 << key_bits) - 1) : 0, d_keys, d_hcount};
        metrics_user_kernel<<<grid(U), METRICS_THREADS, 0, st>>>(a);
        CK(cudaGetLastError());
        ++S.n_launches;
        if (map) {
            CK(cub::DeviceRadixSort::SortKeys(d_tmp, tmp_bytes, d_keys, d_keys_s, (int)n, 0, key_bits, st));
            CK(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_hcount, d_hoff, (int)U, st));
            metrics_map_kernel<<<grid(U), METRICS_THREADS, 0, st>>>(U, n, d_hoff, d_hcount, d_keys_s, rbits, n_k, d_ks, d_prec, d_map);
            CK(cudaGetLastError());
            S.n_launches += 3;
        }
        CK(cudaEventRecord(R.ev[2], st));

        // ---- outputs: the per-k and per-table rows at stride n_inter
        CK(cudaMemcpyAsync(out_users, d_users, sizeof(int64_t) * U, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out_liked, d_cnt, sizeof(int64_t) * U, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out_min_rank, d_min, sizeof(int64_t) * U, cudaMemcpyDeviceToHost, st));
        if (n_k > 0) CK(cudaMemcpy2DAsync(out_tp, sizeof(int64_t) * n, d_tp, sizeof(int64_t) * n, sizeof(int64_t) * U, n_k, cudaMemcpyDeviceToHost, st));
        if (n_ndcg > 0)
            CK(cudaMemcpy2DAsync(out_ndcg, sizeof(double) * n, d_ndcg, sizeof(double) * n, sizeof(double) * U, n_ndcg, cudaMemcpyDeviceToHost, st));
        if (map) CK(cudaMemcpy2DAsync(out_map, sizeof(double) * n, d_map, sizeof(double) * n, sizeof(double) * U, n_k, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out_first_order, d_order, sizeof(int64_t) * U, cudaMemcpyDeviceToHost, st));
        S.d2h_bytes = U * (8 * 4 + 8 * n_k + 8 * n_ndcg + (map ? 8 * n_k : 0));
        CK(cudaEventRecord(R.ev[3], st));
        CK(cudaStreamSynchronize(st));
        *out_n_users = U;
        *out_flags = 0;
        S.ms_h2d = R.ms(0, 1);
        S.ms_main = R.ms(1, 2);
        S.ms_d2h = R.ms(2, 3);
        S.ms_total = S.ms_h2d + S.ms_main + S.ms_d2h;
        S.n_chunks = 1;
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_metrics", ce);
    }
    if (stats) *stats = S;
    return B200_OK;
}
