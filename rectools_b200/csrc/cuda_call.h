// Host-side CUDA plumbing of every libb200rank.so entry point: the error a failed CUDA call throws, how it becomes a
// return code and a b200_rank_last_error() message, grow-only device buffers, and the scratch of one call.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/b200_rank.h"
#include "engine_internal.h"

namespace {

struct CudaError {
    cudaError_t e;
    const char* what;
    int line;
};

#define CK(call)                                                       \
    do {                                                               \
        cudaError_t e__ = (call);                                      \
        if (e__ != cudaSuccess) throw CudaError{e__, #call, __LINE__}; \
    } while (0)

// The return code of a failed CUDA call (B200_E_NOMEM for a refused allocation, else B200_E_CUDA) and its message,
// "<call> failed at line <n>: <error>".  Clears the thread's last CUDA error: a refused cudaMalloc leaves it set, and the
// thread's next call would otherwise fail at its first cudaGetLastError().
inline int cuda_failure(const CudaError& ce, std::string& message) {
    cudaGetLastError();
    char buf[512];
    snprintf(buf, sizeof(buf), "%s failed at line %d: %s", ce.what, ce.line, cudaGetErrorString(ce.e));
    message = buf;
    return ce.e == cudaErrorMemoryAllocation ? B200_E_NOMEM : B200_E_CUDA;
}

// The same, reported by entry point `who` on the calling thread; returns the code.
inline int cuda_fail(const char* who, const CudaError& ce) {
    std::string message;
    const int code = cuda_failure(ce, message);
    return b200_set_error(code, (std::string(who) + ": " + message).c_str());
}

// Device memory that only grows: ensure() with slack (the per-call buffers), ensure_exact() at the size asked.
struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    void ensure(size_t bytes) {
        if (bytes <= cap) return;
        if (p) CK(cudaFree(p));
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 8 + 256;
        CK(cudaMalloc(&p, want));
        cap = want;
    }
    void* ensure_exact(size_t bytes) {  // no slack: the resident objects, and the engine group's copies and staging
        if (bytes > cap) {
            release();
            CK(cudaMalloc(&p, bytes));
            cap = bytes;
        }
        return p;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T>
    T* as() const {
        return reinterpret_cast<T*>(p);
    }
};

// The device allocations and N timing events of one call, freed when it returns, and its stream: the caller's, or with
// NULL one of its own, which is synchronised before anything is freed.
template <int N>
struct CallScratch {
    cudaStream_t st;
    bool own;
    cudaEvent_t ev[N] = {};
    std::vector<void*> bufs;
    explicit CallScratch(cudaStream_t caller = nullptr) : st(caller), own(!caller) {
        try {
            if (own) CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
            for (auto& e : ev) CK(cudaEventCreate(&e));
        } catch (...) {
            release();
            throw;
        }
    }
    ~CallScratch() { release(); }
    template <typename T>
    T* get(size_t count) {
        void* p = nullptr;
        CK(cudaMalloc(&p, std::max<size_t>(count * sizeof(T), 16)));
        bufs.push_back(p);
        return static_cast<T*>(p);
    }
    float ms(int a, int b) const {
        float t = 0.f;
        CK(cudaEventElapsedTime(&t, ev[a], ev[b]));
        return t;
    }
    void release() {
        if (own && st) cudaStreamSynchronize(st);
        for (void* p : bufs) cudaFree(p);
        for (auto& e : ev)
            if (e) cudaEventDestroy(e);
        if (own && st) cudaStreamDestroy(st);
    }
};

}  // namespace
