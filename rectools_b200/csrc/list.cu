// libb200rank.so -- shared list minus viewed ids (path 7, b200_rank_topk_list): the per-user step of
// `PopularModel._recommend_u2i` (rectools/models/popular.py:229-277), which takes the first k entries of one ordered
// popularity list that a user has not viewed.  No engine and no catalogue: the call owns its stream and scratch and frees
// them before it returns.  Every refusal is decided on the host by plan_list (list_plan.h) before the device is touched;
// the kernel is in list_select.cuh.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"
#include "engine_internal.h"
#include "list_call.h"
#include "list_plan.h"
#include "list_select.cuh"

extern "C" int b200_rank_topk_list(int32_t device, int64_t n_list, const int32_t* list_ids, int64_t n_rows,
                                   const int64_t* csr_indptr, const int32_t* csr_indices, int32_t k, int32_t* out_pos,
                                   int32_t* out_counts, b200_rank_stats* stats) {
    using namespace b200;
    ListArgs args;
    args.n_list = n_list;
    args.list_ids = list_ids;
    args.n_rows = n_rows;
    args.indptr = csr_indptr;
    args.indices = csr_indices;
    args.k = k;
    args.out_pos = out_pos != nullptr;
    args.out_counts = out_counts != nullptr;
    const ListPlan P = plan_list(args, list_chunk_rows_hook());
    if (P.error != B200_OK) return b200_set_error(P.error, P.message.c_str());
    b200_rank_stats S{};
    S.path = 7;
    S.k_out = P.k_out;
    if (P.n_chunks() == 0) {  // no row, or an empty list: every row keeps nothing
        std::fill(out_counts, out_counts + n_rows, 0);
        if (stats) *stats = S;
        return B200_OK;
    }
    const int64_t k_out = P.k_out;
    try {
        CK(cudaSetDevice(device));
        CallScratch<4> R;
        // every allocation before the first output write: a failed one leaves the outputs untouched
        int32_t* d_list = R.get<int32_t>(n_list);
        int64_t* d_indptr = csr_indptr ? R.get<int64_t>(P.max_chunk_rows + 1) : nullptr;
        int32_t* d_indices = csr_indptr ? R.get<int32_t>(P.max_chunk_nnz) : nullptr;
        int32_t* d_pos = R.get<int32_t>(P.max_chunk_rows * k_out);
        int32_t* d_counts = R.get<int32_t>(P.max_chunk_rows);
        run_list_chunks(R, {{d_list, list_ids, sizeof(int32_t) * n_list}}, P.bounds, csr_indptr, csr_indices, d_indptr, d_indices,
                        k_out, d_pos, d_counts, out_pos, out_counts, S,
                        [&](int64_t nr, const int64_t* indptr, int64_t base, const int32_t* indices) {
                            const ListRows a{d_list, n_list, indptr, base, indices, nr, k, (int)k_out, d_pos, d_counts};
                            if (k_out <= LIST_WARP_K) {
                                constexpr int rows_per_cta = LIST_THREADS / 32;
                                list_select_kernel<1><<<(unsigned)((nr + rows_per_cta - 1) / rows_per_cta), LIST_THREADS, 0, R.st>>>(a);
                            } else {
                                list_select_kernel<LIST_THREADS / 32><<<(unsigned)nr, LIST_THREADS, 0, R.st>>>(a);
                            }
                        });
    } catch (const CudaError& ce) {
        return cuda_fail("b200_rank_topk_list", ce);
    }
    if (stats) *stats = S;
    return B200_OK;
}
