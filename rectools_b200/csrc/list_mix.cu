// libb200rank.so -- per-category lists minus viewed ids, mixed (path 8, b200_rank_topk_list_mix): the per-user step of
// `PopularInCategoryModel._recommend_u2i` (rectools/models/popular_in_category.py:333-373), which asks each category's
// `PopularModel` for its list and mixes the lists in pandas.  No engine and no catalogue: the call owns its stream and
// scratch and frees them before it returns.  Every refusal is decided on the host by plan_list_mix (list_mix_plan.h)
// before the device is touched; the kernel is in list_mix.cuh.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
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
        CK(cudaSetDevice(device));
        CallScratch<4> R;
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
            CK(cudaFuncSetAttribute(list_mix_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MIX_SMEM_BYTES));
        const std::initializer_list<HostCopy> lists = {{d_list, list_ids, sizeof(int32_t) * n_total},
                                                       {d_offsets, list_offsets, sizeof(int64_t) * (n_lists + 1)},
                                                       {d_slots, P.slots.data(), sizeof(int64_t) * (n_lists + 1)},
                                                       {d_quota, quota, sizeof(int32_t) * n_lists}};
        run_list_chunks(R, lists, P.bounds, csr_indptr, csr_indices, d_indptr, d_indices, k_out, d_pos, d_counts, out_pos, out_counts, S,
                        [&](int64_t nr, const int64_t* indptr, int64_t base, const int32_t* indices) {
                            const MixRows a{d_list, d_offsets, d_slots, d_quota, n_lists, mixing, indptr, base, indices, nr, k, (int)k_out,
                                            P.slots[n_lists], next_pow2(std::max<int64_t>(P.slots[n_lists], 1)), d_scratch,
                                            P.row_scratch, d_pos, d_counts};
                            if (P.smem)
                                list_mix_kernel<true><<<(unsigned)nr, MIX_THREADS, (size_t)P.row_scratch, R.st>>>(a);
                            else
                                list_mix_kernel<false><<<(unsigned)nr, MIX_THREADS, 0, R.st>>>(a);
                        });
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk_list_mix", ce);
    }
    if (stats) *stats = S;
    return B200_OK;
}
