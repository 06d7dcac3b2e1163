// The chunk loop of a host-buffer list call (paths 7 and 8: list.cu, list_mix.cu).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <initializer_list>
#include <vector>

#include "../../include/b200_rank.h"
#include "cuda_call.h"

namespace {

struct HostCopy {
    void* dst;
    const void* src;
    size_t bytes;
};

// One list call on R's stream: the `lists` uploads once, then per chunk of rows [bounds[c], bounds[c + 1]) the chunk's
// rows of the host CSR filter (if any) into d_indptr / d_indices, `launch(nr, d_indptr, base, d_indices)`, and the
// chunk's positions and counts back into the outputs.  Every chunk is synchronised before the next reuses the device
// buffers.  Adds the bytes, launches, chunks and the h2d / main / d2h times to S.
template <class Launch>
void run_list_chunks(CallScratch<4>& R, std::initializer_list<HostCopy> lists, const std::vector<int64_t>& bounds,
                     const int64_t* csr_indptr, const int32_t* csr_indices, int64_t* d_indptr, int32_t* d_indices, int64_t k_out,
                     const int32_t* d_pos, const int32_t* d_counts, int32_t* out_pos, int32_t* out_counts, b200_rank_stats& S,
                     Launch launch) {
    cudaStream_t st = R.st;
    CK(cudaEventRecord(R.ev[0], st));
    for (const HostCopy& h : lists) {
        CK(cudaMemcpyAsync(h.dst, h.src, h.bytes, cudaMemcpyHostToDevice, st));
        S.h2d_bytes += (int64_t)h.bytes;
    }
    const int64_t n_chunks = (int64_t)bounds.size() - 1;
    for (int64_t c = 0; c < n_chunks; ++c) {
        const int64_t r0 = bounds[c], r1 = bounds[c + 1], nr = r1 - r0;
        int64_t base = 0;
        if (c > 0) CK(cudaEventRecord(R.ev[0], st));
        if (csr_indptr) {
            base = csr_indptr[r0];
            const int64_t ne = csr_indptr[r1] - base;
            CK(cudaMemcpyAsync(d_indptr, csr_indptr + r0, sizeof(int64_t) * (nr + 1), cudaMemcpyHostToDevice, st));
            if (ne > 0) CK(cudaMemcpyAsync(d_indices, csr_indices + base, sizeof(int32_t) * ne, cudaMemcpyHostToDevice, st));
            S.h2d_bytes += (int64_t)(sizeof(int64_t) * (nr + 1) + sizeof(int32_t) * ne);
        }
        CK(cudaEventRecord(R.ev[1], st));
        launch(nr, d_indptr, base, d_indices);
        CK(cudaGetLastError());
        ++S.n_launches;
        CK(cudaEventRecord(R.ev[2], st));
        CK(cudaMemcpyAsync(out_pos + r0 * k_out, d_pos, sizeof(int32_t) * nr * k_out, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out_counts + r0, d_counts, sizeof(int32_t) * nr, cudaMemcpyDeviceToHost, st));
        S.d2h_bytes += (int64_t)sizeof(int32_t) * nr * (k_out + 1);
        CK(cudaEventRecord(R.ev[3], st));
        CK(cudaStreamSynchronize(st));  // the chunk's device buffers are reused by the next one
        S.ms_h2d += R.ms(0, 1);
        S.ms_main += R.ms(1, 2);
        S.ms_d2h += R.ms(2, 3);
    }
    S.ms_total = S.ms_h2d + S.ms_main + S.ms_d2h;
    S.n_chunks = (int32_t)n_chunks;
}

}  // namespace
