// cuda_runtime.h — a host-only stand-in for the CUDA runtime calls of bifromq_b200/csrc/cuda_buf.h, so that
// tests/native/cuda_buf_harness.cc checks the buffer's allocation rules with g++ and no GPU. "Device" and pinned memory are
// both plain malloc; every call is appended to a log, allocations and frees are counted per allocator, and the next
// allocation can be made to fail.
#pragma once
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0, cudaErrorMemoryAllocation = 2;
typedef struct CUstream_st* cudaStream_t;
enum cudaMemcpyKind { cudaMemcpyDeviceToDevice = 3 };

namespace fake_cuda {
struct State {
    long device_allocs = 0, device_frees = 0, pinned_allocs = 0, pinned_frees = 0;
    bool fail_next_alloc = false;
    std::vector<std::string> log;   // "malloc <bytes>", "free", "malloc_host <bytes>", "free_host", "memcpy <bytes>", "sync"
};
inline State& state() {
    static State s;
    return s;
}
inline cudaError_t alloc(void** p, size_t bytes, const char* what, long* count) {
    State& s = state();
    if (s.fail_next_alloc) {
        s.fail_next_alloc = false;
        return cudaErrorMemoryAllocation;
    }
    *p = malloc(bytes ? bytes : 1);
    (*count)++;
    s.log.push_back(std::string(what) + " " + std::to_string(bytes));
    return cudaSuccess;
}
}  // namespace fake_cuda

inline cudaError_t cudaMalloc(void** p, size_t bytes) { return fake_cuda::alloc(p, bytes, "malloc", &fake_cuda::state().device_allocs); }
inline cudaError_t cudaMallocHost(void** p, size_t bytes) {
    return fake_cuda::alloc(p, bytes, "malloc_host", &fake_cuda::state().pinned_allocs);
}
inline cudaError_t cudaFree(void* p) {
    free(p);
    fake_cuda::state().device_frees++;
    fake_cuda::state().log.push_back("free");
    return cudaSuccess;
}
inline cudaError_t cudaFreeHost(void* p) {
    free(p);
    fake_cuda::state().pinned_frees++;
    fake_cuda::state().log.push_back("free_host");
    return cudaSuccess;
}
inline cudaError_t cudaMemcpyAsync(void* dst, const void* src, size_t bytes, cudaMemcpyKind, cudaStream_t) {
    memcpy(dst, src, bytes);
    fake_cuda::state().log.push_back("memcpy " + std::to_string(bytes));
    return cudaSuccess;
}
inline cudaError_t cudaStreamSynchronize(cudaStream_t) {
    fake_cuda::state().log.push_back("sync");
    return cudaSuccess;
}
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaErrorMemoryAllocation ? "out of memory" : "unknown error"; }
