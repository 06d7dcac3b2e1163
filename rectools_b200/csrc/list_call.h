// The stream, events and device allocations of one host-buffer list call (paths 7 and 8: list.cu, list_mix.cu), released
// when the call returns, and the error that carries a failed CUDA call out of it.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <vector>

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
