// libb200rank.so -- shared list minus viewed ids (path 7, b200_rank_topk_list): the per-user step of
// `PopularModel._recommend_u2i` (rectools/models/popular.py:229-277), which takes the first k entries of one ordered
// popularity list that a user has not viewed.  No engine and no catalogue: the call owns its stream and scratch and frees
// them before it returns.  Every refusal is decided on the host by plan_list (list_plan.h) before the device is touched;
// the kernel is in list_select.cuh.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../include/b200_rank.h"
#include "engine_internal.h"
#include "list_plan.h"
#include "list_select.cuh"

namespace {

struct ListError {
    cudaError_t e;
    const char* what;
    int line;
};

#define LCK(call)                                                    \
    do {                                                             \
        cudaError_t e__ = (call);                                    \
        if (e__ != cudaSuccess) throw ListError{e__, #call, __LINE__}; \
    } while (0)

// the stream, events and device allocations of one call, released when it returns
struct CallResources {
    cudaStream_t st = nullptr;
    cudaEvent_t ev[4] = {};
    std::vector<void*> bufs;
    CallResources() {
        try {
            LCK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
            for (auto& e : ev) LCK(cudaEventCreate(&e));
        } catch (...) {
            release();
            throw;
        }
    }
    template <typename T>
    T* get(size_t count) {
        void* p = nullptr;
        LCK(cudaMalloc(&p, std::max<size_t>(count * sizeof(T), 16)));
        bufs.push_back(p);
        return static_cast<T*>(p);
    }
    float ms(int a, int b) const {
        float t = 0.f;
        LCK(cudaEventElapsedTime(&t, ev[a], ev[b]));
        return t;
    }
    ~CallResources() { release(); }
    void release() {
        if (st) cudaStreamSynchronize(st);
        for (void* p : bufs) cudaFree(p);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (st) cudaStreamDestroy(st);
    }
};

}  // namespace

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
        LCK(cudaSetDevice(device));
        CallResources R;
        cudaStream_t st = R.st;
        // every allocation before the first output write: a failed one leaves the outputs untouched
        int32_t* d_list = R.get<int32_t>(n_list);
        int64_t* d_indptr = csr_indptr ? R.get<int64_t>(P.max_chunk_rows + 1) : nullptr;
        int32_t* d_indices = csr_indptr ? R.get<int32_t>(P.max_chunk_nnz) : nullptr;
        int32_t* d_pos = R.get<int32_t>(P.max_chunk_rows * k_out);
        int32_t* d_counts = R.get<int32_t>(P.max_chunk_rows);
        LCK(cudaEventRecord(R.ev[0], st));
        LCK(cudaMemcpyAsync(d_list, list_ids, sizeof(int32_t) * n_list, cudaMemcpyHostToDevice, st));
        S.h2d_bytes += (int64_t)sizeof(int32_t) * n_list;
        float ms_h2d = 0.f, ms_main = 0.f, ms_d2h = 0.f;
        for (int64_t c = 0; c < P.n_chunks(); ++c) {
            const int64_t r0 = P.bounds[c], r1 = P.bounds[c + 1], nr = r1 - r0;
            ListRows a{d_list, n_list, nullptr, 0, nullptr, nr, k, (int)k_out, d_pos, d_counts};
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
            if (k_out <= LIST_WARP_K) {
                constexpr int rows_per_cta = LIST_THREADS / 32;
                list_select_kernel<1><<<(unsigned)((nr + rows_per_cta - 1) / rows_per_cta), LIST_THREADS, 0, st>>>(a);
            } else {
                list_select_kernel<LIST_THREADS / 32><<<(unsigned)nr, LIST_THREADS, 0, st>>>(a);
            }
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
        snprintf(msg, sizeof(msg), "b200_rank_topk_list: %s failed at line %d: %s", le.what, le.line, cudaGetErrorString(le.e));
        return b200_set_error(le.e == cudaErrorMemoryAllocation ? B200_E_NOMEM : B200_E_CUDA, msg);
    }
    if (stats) *stats = S;
    return B200_OK;
}
