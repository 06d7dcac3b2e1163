// libb200rank.so -- per-category lists minus viewed ids, mixed (path 8, b200_rank_topk_list_mix): the per-user step of
// `PopularInCategoryModel._recommend_u2i` (rectools/models/popular_in_category.py:333-373), which asks each category's
// `PopularModel` for its list and mixes the lists in pandas.  No engine and no catalogue: the call owns its stream and
// scratch and frees them before it returns.  Every refusal is decided on the host by plan_list_mix (list_mix_plan.h)
// before the device is touched; the kernel is in list_mix.cuh.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/b200_rank.h"
#include "engine_internal.h"
#include "list_call.h"
#include "list_mix.cuh"
#include "list_mix_plan.h"

extern "C" int b200_rank_topk_list_mix(int32_t device, int32_t n_lists, const int64_t* list_offsets, const int32_t* list_ids,
                                       const int32_t* quota, int32_t mixing, int64_t n_rows, const int64_t* csr_indptr,
                                       const int32_t* csr_indices, int32_t k, int32_t* out_pos, int32_t* out_counts,
                                       b200_rank_stats* stats) {
    using namespace b200;
    ListMixArgs args;
    args.n_lists = n_lists;
    args.offsets = list_offsets;
    args.list_ids = list_ids;
    args.quota = quota;
    args.mixing = mixing;
    args.n_rows = n_rows;
    args.indptr = csr_indptr;
    args.indices = csr_indices;
    args.k = k;
    args.out_pos = out_pos != nullptr;
    args.out_counts = out_counts != nullptr;
    const ListMixPlan P = plan_list_mix(args, list_chunk_rows_hook(), list_mix_smem_hook());
    if (P.error != B200_OK) return b200_set_error(P.error, P.message.c_str());
    b200_rank_stats S{};
    S.path = 8;
    S.k_out = P.k_out;
    if (P.n_chunks() == 0) {  // no row, or no list entry: every row keeps nothing
        std::fill(out_counts, out_counts + n_rows, 0);
        if (stats) *stats = S;
        return B200_OK;
    }
    const int64_t k_out = P.k_out, n_total = P.n_total;
    try {
        LCK(cudaSetDevice(device));
        CallResources R;
        cudaStream_t st = R.st;
        // every allocation before the first output write: a failed one leaves the outputs untouched
        int32_t* d_list = R.get<int32_t>(n_total);
        int64_t* d_offsets = R.get<int64_t>(n_lists + 1);
        int64_t* d_slots = R.get<int64_t>(n_lists + 1);
        int32_t* d_quota = R.get<int32_t>(n_lists);
        int64_t* d_indptr = csr_indptr ? R.get<int64_t>(P.max_chunk_rows + 1) : nullptr;
        int32_t* d_indices = csr_indptr ? R.get<int32_t>(P.max_chunk_nnz) : nullptr;
        int32_t* d_pos = R.get<int32_t>(P.max_chunk_rows * k_out);
        int32_t* d_counts = R.get<int32_t>(P.max_chunk_rows);
        unsigned char* d_scratch = P.smem ? nullptr : R.get<unsigned char>(P.max_chunk_rows * P.row_scratch);
        // always the same value, so concurrent calls from several host threads cannot undo each other's setting
        if (P.smem)
            LCK(cudaFuncSetAttribute(list_mix_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MIX_SMEM_BYTES));
        LCK(cudaEventRecord(R.ev[0], st));
        LCK(cudaMemcpyAsync(d_list, list_ids, sizeof(int32_t) * n_total, cudaMemcpyHostToDevice, st));
        LCK(cudaMemcpyAsync(d_offsets, list_offsets, sizeof(int64_t) * (n_lists + 1), cudaMemcpyHostToDevice, st));
        LCK(cudaMemcpyAsync(d_slots, P.slots.data(), sizeof(int64_t) * (n_lists + 1), cudaMemcpyHostToDevice, st));
        LCK(cudaMemcpyAsync(d_quota, quota, sizeof(int32_t) * n_lists, cudaMemcpyHostToDevice, st));
        S.h2d_bytes += (int64_t)(sizeof(int32_t) * (n_total + n_lists) + 2 * sizeof(int64_t) * (n_lists + 1));
        float ms_h2d = 0.f, ms_main = 0.f, ms_d2h = 0.f;
        for (int64_t c = 0; c < P.n_chunks(); ++c) {
            const int64_t r0 = P.bounds[c], r1 = P.bounds[c + 1], nr = r1 - r0;
            MixRows a{d_list, d_offsets, d_slots, d_quota, n_lists, mixing, nullptr, 0, nullptr, nr, k, (int)k_out,
                      P.slots[n_lists], next_pow2(std::max<int64_t>(P.slots[n_lists], 1)), d_scratch, P.row_scratch,
                      d_pos, d_counts};
            if (c > 0) LCK(cudaEventRecord(R.ev[0], st));
            if (csr_indptr) {
                const int64_t e0 = csr_indptr[r0], ne = csr_indptr[r1] - e0;
                LCK(cudaMemcpyAsync(d_indptr, csr_indptr + r0, sizeof(int64_t) * (nr + 1), cudaMemcpyHostToDevice, st));
                if (ne > 0) LCK(cudaMemcpyAsync(d_indices, csr_indices + e0, sizeof(int32_t) * ne, cudaMemcpyHostToDevice, st));
                S.h2d_bytes += (int64_t)(sizeof(int64_t) * (nr + 1) + sizeof(int32_t) * ne);
                a.indptr = d_indptr;
                a.base = e0;
                a.indices = d_indices;
            }
            LCK(cudaEventRecord(R.ev[1], st));
            if (P.smem)
                list_mix_kernel<true><<<(unsigned)nr, MIX_THREADS, (size_t)P.row_scratch, st>>>(a);
            else
                list_mix_kernel<false><<<(unsigned)nr, MIX_THREADS, 0, st>>>(a);
            LCK(cudaGetLastError());
            ++S.n_launches;
            LCK(cudaEventRecord(R.ev[2], st));
            LCK(cudaMemcpyAsync(out_pos + r0 * k_out, d_pos, sizeof(int32_t) * nr * k_out, cudaMemcpyDeviceToHost, st));
            LCK(cudaMemcpyAsync(out_counts + r0, d_counts, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost, st));
            S.d2h_bytes += (int64_t)sizeof(int32_t) * nr * (k_out + 1);
            LCK(cudaEventRecord(R.ev[3], st));
            LCK(cudaStreamSynchronize(st));  // the chunk's device buffers are reused by the next one
            ms_h2d += R.ms(0, 1);
            ms_main += R.ms(1, 2);
            ms_d2h += R.ms(2, 3);
        }
        S.ms_h2d = ms_h2d;
        S.ms_main = ms_main;
        S.ms_d2h = ms_d2h;
        S.ms_total = ms_h2d + ms_main + ms_d2h;
        S.n_chunks = (int32_t)P.n_chunks();
    } catch (const ListError& le) {
        cudaGetLastError();  // a failed allocation must not surface in a later call
        char msg[512];
        snprintf(msg, sizeof(msg), "b200_rank_topk_list_mix: %s failed at line %d: %s", le.what, le.line,
                 cudaGetErrorString(le.e));
        return b200_set_error(le.e == cudaErrorMemoryAllocation ? B200_E_NOMEM : B200_E_CUDA, msg);
    }
    if (stats) *stats = S;
    return B200_OK;
}
