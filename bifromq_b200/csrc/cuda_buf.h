// cuda_buf.h — the owning device / pinned-host buffer and the CUDA error path of every host-side source.
//
// Every cudaMalloc / cudaMallocHost of the library goes through CudaBuf, so device memory is freed by whoever owns the buffer
// (a destructor, a move, an early return) and never by a hand-kept list. The sizes are part of the statistics callers see
// (bfq_index_stats / bfq_rindex_stats report device_bytes = the sum of bytes()), so reserve and grow keep exact rules.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstddef>
#include <string>

#include "../../include/bfq_gpumatch.h"
#include "codec.h"

namespace bfq {

template <typename T, bool Pinned>
struct CudaBuf {
    T* p = nullptr;
    size_t cap = 0;   // elements asked for by the last reserve / grow that allocated

    CudaBuf() = default;
    CudaBuf(const CudaBuf&) = delete;
    CudaBuf& operator=(const CudaBuf&) = delete;
    CudaBuf(CudaBuf&& o) noexcept : p(o.p), cap(o.cap) {
        o.p = nullptr;
        o.cap = 0;
    }
    CudaBuf& operator=(CudaBuf&& o) noexcept {
        if (this != &o) {
            release();
            p = o.p;
            cap = o.cap;
            o.p = nullptr;
            o.cap = 0;
        }
        return *this;
    }
    ~CudaBuf() { release(); }

    size_t bytes() const { return cap * sizeof(T); }
    void release() {
        if (p && Pinned) cudaFreeHost(p);
        else if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    // Room for exactly n elements, contents not kept. The old buffer is freed before the new one is allocated (peak memory
    // stays one buffer). reserve(0) never allocates: an empty buffer keeps p == nullptr.
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        release();
        T* q = nullptr;
        const cudaError_t e = alloc(&q, n);
        if (e != cudaSuccess) return e;
        p = q;
        cap = n;
        return cudaSuccess;
    }
    // Like reserve, but keeps the first `keep` elements (device-to-device copy on st, synchronised before the old buffer is
    // freed) and grows by at least half the capacity.
    cudaError_t grow(size_t n, size_t keep, cudaStream_t st) {
        static_assert(!Pinned, "grow copies device to device");
        if (n <= cap) return cudaSuccess;
        const size_t want = std::max(n, cap + cap / 2);
        T* q = nullptr;
        cudaError_t e = alloc(&q, want);
        if (e != cudaSuccess) return e;
        if (keep) e = cudaMemcpyAsync(q, p, keep * sizeof(T), cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            cudaFree(q);
            return e;
        }
        release();
        p = q;
        cap = want;
        return cudaSuccess;
    }

  private:
    static cudaError_t alloc(T** q, size_t n) {
        if (Pinned) return cudaMallocHost((void**) q, n * sizeof(T));
        return cudaMalloc((void**) q, n * sizeof(T));
    }
};

template <typename T>
using DeviceBuf = CudaBuf<T, false>;
template <typename T>
using PinnedBuf = CudaBuf<T, true>;

inline int32_t fail(int32_t code, const std::string& msg) { return set_error(code, msg); }

// Typed arrays placed one after another in one block, each at a 256-byte boundary. With base == nullptr it only counts the
// bytes; with base set it hands out the pointers.
struct Carve {
    uint8_t* base = nullptr;
    size_t bytes = 0;
    template <typename T>
    T* take(size_t n) {
        bytes = (bytes + 255) & ~(size_t) 255;
        T* p = base ? reinterpret_cast<T*>(base + bytes) : nullptr;
        bytes += n * sizeof(T);
        return p;
    }
};

// A layout written once (layout(Carve&) takes every array of a call) and run twice: to size `arena` (contents not kept), then
// to hand out the arrays in it. `what` names the arena in the error message.
template <typename Layout>
int32_t carve(DeviceBuf<uint8_t>& arena, const char* what, Layout&& layout) {
    Carve count;
    layout(count);
    const cudaError_t e = arena.reserve(count.bytes);
    if (e != cudaSuccess) return fail(BFQ_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
    Carve place{arena.p};
    layout(place);
    return BFQ_OK;
}

}  // namespace bfq

// returns BFQ_E_CUDA from the enclosing function, with the failed expression and CUDA's message in bfq_last_error()
#define BFQ_CUDA_TRY(expr)                                                                             \
    do {                                                                                               \
        const cudaError_t _e = (expr);                                                                 \
        if (_e != cudaSuccess) return bfq::fail(BFQ_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)
