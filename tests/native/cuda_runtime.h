// cuda_runtime.h — a host-only stand-in for the CUDA runtime calls of bifromq_b200/csrc/cuda_buf.h and lease.h, so that
// tests/native/cuda_buf_harness.cc and lease_harness.cc check the buffer's allocation rules and the workspace pool with g++
// and no GPU. "Device" and pinned memory are both plain malloc; streams and events are numbered handles. Every call is
// appended to a log, allocations, frees, creations and destructions are counted, and the next allocation, stream creation
// or event creation can be made to fail.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

typedef int cudaError_t;
constexpr cudaError_t cudaSuccess = 0, cudaErrorMemoryAllocation = 2;
typedef struct CUstream_st* cudaStream_t;
typedef struct CUevent_st* cudaEvent_t;
enum cudaMemcpyKind { cudaMemcpyDeviceToDevice = 3 };
constexpr unsigned cudaStreamNonBlocking = 1, cudaEventDisableTiming = 2;

namespace fake_cuda {
struct State {
    long device_allocs = 0, device_frees = 0, pinned_allocs = 0, pinned_frees = 0;
    long streams_created = 0, streams_destroyed = 0, events_created = 0, events_destroyed = 0;
    uintptr_t next_handle = 0;   // streams and events are numbered 1, 2, ... in one sequence
    bool fail_next_alloc = false, fail_next_stream = false, fail_next_event = false;
    // "malloc <bytes>", "free", "malloc_host <bytes>", "free_host", "memcpy <bytes>", "sync", "stream_create s<k>",
    // "stream_destroy s<k>", "event_create e<k>", "event_destroy e<k>", "event_record e<k> s<k>", "event_sync e<k>",
    // "set_device <d>"
    std::vector<std::string> log;
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
namespace fake_cuda {
inline std::string name(const void* handle, const char* prefix) { return prefix + std::to_string((uintptr_t) handle); }
template <typename H>
cudaError_t create(H* out, bool* fail, long* count, const char* what, const char* prefix) {
    State& s = state();
    if (*fail) {
        *fail = false;
        return cudaErrorMemoryAllocation;
    }
    *out = reinterpret_cast<H>(++s.next_handle);
    (*count)++;
    s.log.push_back(std::string(what) + " " + name(*out, prefix));
    return cudaSuccess;
}
}  // namespace fake_cuda

inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned) {
    auto& st = fake_cuda::state();
    return fake_cuda::create(s, &st.fail_next_stream, &st.streams_created, "stream_create", "s");
}
inline cudaError_t cudaStreamDestroy(cudaStream_t s) {
    fake_cuda::state().streams_destroyed++;
    fake_cuda::state().log.push_back("stream_destroy " + fake_cuda::name(s, "s"));
    return cudaSuccess;
}
inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned) {
    auto& st = fake_cuda::state();
    return fake_cuda::create(e, &st.fail_next_event, &st.events_created, "event_create", "e");
}
inline cudaError_t cudaEventDestroy(cudaEvent_t e) {
    fake_cuda::state().events_destroyed++;
    fake_cuda::state().log.push_back("event_destroy " + fake_cuda::name(e, "e"));
    return cudaSuccess;
}
inline cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s) {
    fake_cuda::state().log.push_back("event_record " + fake_cuda::name(e, "e") + " " + fake_cuda::name(s, "s"));
    return cudaSuccess;
}
inline cudaError_t cudaEventSynchronize(cudaEvent_t e) {
    fake_cuda::state().log.push_back("event_sync " + fake_cuda::name(e, "e"));
    return cudaSuccess;
}
inline cudaError_t cudaSetDevice(int d) {
    fake_cuda::state().log.push_back("set_device " + std::to_string(d));
    return cudaSuccess;
}
inline const char* cudaGetErrorString(cudaError_t e) { return e == cudaErrorMemoryAllocation ? "out of memory" : "unknown error"; }
