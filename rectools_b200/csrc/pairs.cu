// libb200rank.so -- scored pairs (path 6, b200_rank_topk_pairs): the per-group top-k of `Reranker.recommend`
// (rectools/models/ranking/candidate_ranking.py:203-236), which keeps the k best pairs of each user of a two-stage model's
// scored candidates.  No engine and no catalogue: the call owns its scratch and frees it before it returns.  The kernels
// are in pairs_select.cuh; everything runs on the caller's stream, so the hand-over of device buffers is stream order.
#include <cuda_runtime.h>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include <algorithm>
#include <climits>
#include <cstdint>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
#include "engine_internal.h"
#include "pairs_select.cuh"

namespace {

size_t score_bytes(int32_t type) { return type == B200_PAIRS_F64 || type == B200_PAIRS_I64 ? 8 : 4; }

unsigned grid_stride(int64_t n, int sms) {
    const int64_t want = (n + 255) / 256;
    return (unsigned)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sms * 16));
}

}  // namespace

extern "C" int b200_rank_topk_pairs(int32_t device, void* stream, int64_t n, const int64_t* group_codes, const void* scores,
                                    int32_t score_type, int64_t n_groups, int32_t k, int32_t flags, int64_t* out_pos,
                                    int64_t* out_offsets, b200_rank_stats* stats) {
    using namespace b200;
    if (n < 0 || n_groups < 0) return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: n and n_groups must be >= 0");
    if (k < 1) return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: k must be >= 1");
    if (score_type < B200_PAIRS_F64 || score_type > B200_PAIRS_I32)
        return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: unknown score type");
    if (flags & ~(B200_Q_INPUTS_ON_DEVICE | B200_Q_OUTPUTS_ON_DEVICE))
        return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: only B200_Q_INPUTS_ON_DEVICE / B200_Q_OUTPUTS_ON_DEVICE are accepted");
    if (!out_offsets) return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: out_offsets is NULL");
    if (n > 0 && (!group_codes || !scores)) return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: group_codes / scores are NULL");
    if (n > 0 && n_groups > 0 && !out_pos) return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: out_pos is NULL");
    const bool in_dev = flags & B200_Q_INPUTS_ON_DEVICE, out_dev = flags & B200_Q_OUTPUTS_ON_DEVICE;
    const int64_t G = n_groups;
    b200_rank_stats S{};
    S.path = 6;
    S.k_out = k;
    S.n_chunks = 1;
    try {
        CK(cudaSetDevice(device));
        int sms = 0;
        CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
        cudaStream_t st = stream ? reinterpret_cast<cudaStream_t>(stream) : cudaStreamLegacy;
        CallScratch<7> mem(st);
        int launches = 0;

        // ---- order keys and grouping
        CK(cudaEventRecord(mem.ev[0], st));
        const int64_t* codes = group_codes;
        const void* sc = scores;
        if (!in_dev && n > 0) {
            int64_t* d_codes = mem.get<int64_t>(n);
            void* d_sc = mem.get<uint8_t>(score_bytes(score_type) * n);
            CK(cudaMemcpyAsync(d_codes, group_codes, sizeof(int64_t) * n, cudaMemcpyHostToDevice, st));
            CK(cudaMemcpyAsync(d_sc, scores, score_bytes(score_type) * n, cudaMemcpyHostToDevice, st));
            S.h2d_bytes = (int64_t)((sizeof(int64_t) + score_bytes(score_type)) * n);
            codes = d_codes;
            sc = d_sc;
        }
        CK(cudaEventRecord(mem.ev[1], st));
        int64_t* count = mem.get<int64_t>(G + 1);  // rows per group, then the scatter's cursors
        int64_t* seg_off = mem.get<int64_t>(G + 1);
        int64_t* kept = mem.get<int64_t>(G + 1);
        int64_t* out_off = mem.get<int64_t>(G + 1);
        int64_t* small = mem.get<int64_t>(3 * PAIRS_N_CLASSES + 1);  // class counts, offsets, cursors; the bad-code flag
        int64_t* class_count = small;
        int64_t* class_off = small + PAIRS_N_CLASSES;
        int64_t* class_cursor = small + 2 * PAIRS_N_CLASSES;
        int* bad = reinterpret_cast<int*>(small + 3 * PAIRS_N_CLASSES);
        CK(cudaMemsetAsync(count, 0, sizeof(int64_t) * (G + 1), st));
        CK(cudaMemsetAsync(kept, 0, sizeof(int64_t) * (G + 1), st));
        CK(cudaMemsetAsync(small, 0, sizeof(int64_t) * (3 * PAIRS_N_CLASSES + 1), st));
        if (n > 0) {
            pairs_count_kernel<<<grid_stride(n, sms), 256, 0, st>>>(n, codes, G, reinterpret_cast<unsigned long long*>(count), bad);
            CK(cudaGetLastError());
            ++launches;
        }
        if (G > 0) {
            pairs_group_kernel<<<grid_stride(G, sms), 256, 0, st>>>(G, k, reinterpret_cast<const unsigned long long*>(count), kept,
                                                                    reinterpret_cast<unsigned long long*>(class_count));
            CK(cudaGetLastError());
            ++launches;
        }
        size_t scan_bytes = 0;
        CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, count, seg_off, G + 1, st));
        void* scan_tmp = mem.get<uint8_t>(scan_bytes);
        CK(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, count, seg_off, G + 1, st));
        CK(cub::DeviceScan::ExclusiveSum(scan_tmp, scan_bytes, kept, out_off, G + 1, st));
        launches += 2;
        int64_t h_small[PAIRS_N_CLASSES + 1] = {};
        int h_bad = 0;
        int64_t total_out = 0;
        CK(cudaMemcpyAsync(h_small, class_count, sizeof(int64_t) * PAIRS_N_CLASSES, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(&h_bad, bad, sizeof(int), cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(&total_out, out_off + G, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
        CK(cudaEventRecord(mem.ev[2], st));
        CK(cudaStreamSynchronize(st));
        if (h_bad) return b200_set_error(B200_E_INVALID, "b200_rank_topk_pairs: a group code lies outside [-1, n_groups)");
        const int64_t n_large = h_small[PAIRS_N_CLASSES - 1];
        if (n_large > 0 && total_out > INT_MAX)
            return b200_set_error(B200_E_NOMEM, "b200_rank_topk_pairs: more than 2^31 - 1 output rows with groups beyond shared memory");
        int64_t h_class_off[PAIRS_N_CLASSES];
        for (int64_t c = 0, run = 0; c < PAIRS_N_CLASSES; run += h_small[c++]) h_class_off[c] = run;
        // every allocation before the first output write: a refusal leaves the outputs untouched
        int64_t* class_list = mem.get<int64_t>(G);
        uint64_t* seg_key = mem.get<uint64_t>(n);
        int64_t* seg_pos = mem.get<int64_t>(n);
        int64_t* dpos = out_dev ? out_pos : mem.get<int64_t>(total_out);
        uint64_t *sk0 = nullptr, *sk1 = nullptr;
        int64_t *sp0 = nullptr, *sp1 = nullptr, *lbeg = nullptr, *lend = nullptr;
        void* sort_tmp = nullptr;
        size_t sort_bytes = 0;
        if (n_large > 0) {
            sk0 = mem.get<uint64_t>(total_out);
            sk1 = mem.get<uint64_t>(total_out);
            sp0 = mem.get<int64_t>(total_out);
            sp1 = mem.get<int64_t>(total_out);
            lbeg = mem.get<int64_t>(n_large);
            lend = mem.get<int64_t>(n_large);
            size_t a = 0, b = 0;
            CK(cub::DeviceSegmentedSort::SortPairs(nullptr, a, sp0, sp1, sk0, sk1, (int)total_out, (int)n_large, lbeg, lend, st));
            CK(cub::DeviceSegmentedSort::StableSortPairsDescending(nullptr, b, sk1, sk0, sp1, sp0, (int)total_out, (int)n_large, lbeg, lend, st));
            sort_bytes = std::max(a, b);
            sort_tmp = mem.get<uint8_t>(sort_bytes);
        }

        CK(cudaEventRecord(mem.ev[3], st));
        CK(cudaMemcpyAsync(class_off, h_class_off, sizeof(h_class_off), cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(count, 0, sizeof(int64_t) * (G + 1), st));
        if (G > 0) {
            pairs_classify_kernel<<<grid_stride(G, sms), 256, 0, st>>>(G, seg_off, class_off, reinterpret_cast<unsigned long long*>(class_cursor),
                                                                       class_list);
            CK(cudaGetLastError());
            ++launches;
        }
        if (n > 0) {
            pairs_scatter_kernel<<<grid_stride(n, sms), 256, 0, st>>>(n, codes, sc, score_type, seg_off,
                                                                      reinterpret_cast<unsigned long long*>(count), seg_key, seg_pos);
            CK(cudaGetLastError());
            ++launches;
        }
        CK(cudaEventRecord(mem.ev[4], st));

        // ---- per-group selection, one launch per size class
        if (h_small[0] > 0) {
            pairs_warp_kernel<<<(unsigned)((h_small[0] + 7) / 8), 256, 0, st>>>(h_small[0], class_list + h_class_off[0], seg_off, out_off,
                                                                                seg_key, seg_pos, dpos);
            CK(cudaGetLastError());
            ++launches;
        }
        auto cta = [&](int c, auto kernel, int cap, int threads) {
            if (h_small[c] == 0) return;
            const int smem = cap * 16;
            CK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
            kernel<<<(unsigned)h_small[c], threads, smem, st>>>(class_list + h_class_off[c], seg_off, out_off, seg_key, seg_pos, dpos);
            CK(cudaGetLastError());
            ++launches;
        };
        cta(1, pairs_cta_kernel<256, 128>, 256, 128);
        cta(2, pairs_cta_kernel<2048, 512>, 2048, 512);
        cta(3, pairs_cta_kernel<PAIRS_SMEM_MAX, 1024>, PAIRS_SMEM_MAX, 1024);
        if (n_large > 0) {
            const int64_t* list = class_list + h_class_off[4];
            pairs_select_kernel<<<(unsigned)n_large, PAIRS_SELECT_THREADS, 0, st>>>(list, seg_off, out_off, seg_key, seg_pos, sk0, sp0,
                                                                                    lbeg, lend);
            CK(cudaGetLastError());
            // position ascending (positions are unique), then key descending, stable: (key desc, position asc)
            CK(cub::DeviceSegmentedSort::SortPairs(sort_tmp, sort_bytes, sp0, sp1, sk0, sk1, (int)total_out, (int)n_large, lbeg, lend, st));
            CK(cub::DeviceSegmentedSort::StableSortPairsDescending(sort_tmp, sort_bytes, sk1, sk0, sp1, sp0, (int)total_out, (int)n_large,
                                                                   lbeg, lend, st));
            pairs_copy_kernel<<<(unsigned)n_large, 256, 0, st>>>(list, out_off, sp0, dpos);
            CK(cudaGetLastError());
            launches += 4;
        }
        CK(cudaEventRecord(mem.ev[5], st));

        // ---- outputs
        if (out_dev) {
            CK(cudaMemcpyAsync(out_offsets, out_off, sizeof(int64_t) * (G + 1), cudaMemcpyDeviceToDevice, st));
        } else {
            CK(cudaMemcpyAsync(out_offsets, out_off, sizeof(int64_t) * (G + 1), cudaMemcpyDeviceToHost, st));
            if (total_out > 0) CK(cudaMemcpyAsync(out_pos, dpos, sizeof(int64_t) * total_out, cudaMemcpyDeviceToHost, st));
            S.d2h_bytes = (int64_t)sizeof(int64_t) * (G + 1 + total_out);
        }
        CK(cudaEventRecord(mem.ev[6], st));
        CK(cudaStreamSynchronize(st));
        S.ms_h2d = mem.ms(0, 1);
        S.ms_main = mem.ms(1, 2) + mem.ms(3, 4);
        S.ms_select = mem.ms(4, 5);
        S.ms_d2h = out_dev ? 0.f : mem.ms(5, 6);
        S.ms_total = mem.ms(0, 6);
        S.n_launches = launches;
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk_pairs", ce);
    }
    if (stats) *stats = S;
    return B200_OK;
}
