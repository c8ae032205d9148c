// lease.h — the workspace pool of both indexes (forward: index_state.h Workspace, inverse: rmatch_kernels.cu RWorkspace), the
// lease of one call, and what a call that enqueues work on a device result's leased workspace owes the result's release.
//
// A match runs on a workspace leased from its handle's pool, and a result whose arrays live there keeps it until it is freed.
// Calls on a completed device result (expand, budget, fan-out, delivery, exchange gather, retain key gather) enqueue kernels
// that read and write that workspace, and some return before those kernels run. Release hands the workspace back to the
// pool, where the next match on the handle can take it, so it first waits for everything such calls enqueued: each call
// records an event of the result on its stream when it returns, one event per stream the result was used on.
//
// No kernel is included here. A workspace type W brings `cudaError_t init(int device)`, `cudaError_t drain()` (waits for the
// workspace's own streams) and `UseEvents use_events`.
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "cuda_buf.h"

namespace bfq {

constexpr size_t POOL_KEEP = 4;   // idle workspaces a pool keeps for reuse; more are freed when they come back

// The workspaces of one handle. Shared (std::shared_ptr) with every result in flight: a result freed after its handle (a
// garbage-collected host language decides the order) still has a place to return its workspace to.
template <typename W>
struct Pool {
    std::mutex mu;
    std::vector<W*> idle;   // LIFO: the workspace given back last is handed out first
    std::vector<W*> live;   // every workspace made and not freed, idle or leased (bfq_rindex_stats slots 11-12)
    int device = 0;
    bool closed = false;    // the handle is gone: workspaces still leased are freed when they come back

    ~Pool() { close(); }

    int32_t acquire(W** out) {
        {
            std::lock_guard<std::mutex> g(mu);
            if (!idle.empty()) {
                *out = idle.back();
                idle.pop_back();
                return BFQ_OK;
            }
        }
        auto* w = new W();
        const cudaError_t e = w->init(device);
        if (e != cudaSuccess) {
            delete w;
            return fail(BFQ_E_CUDA, std::string("workspace: ") + cudaGetErrorString(e));
        }
        std::lock_guard<std::mutex> g(mu);
        live.push_back(w);
        *out = w;
        return BFQ_OK;
    }
    // The caller has waited for everything enqueued on w.
    void give_back(W* w) {
        {
            std::lock_guard<std::mutex> g(mu);
            if (!closed && idle.size() < POOL_KEEP) {
                idle.push_back(w);
                return;
            }
            live.erase(std::remove(live.begin(), live.end(), w), live.end());
        }
        cudaSetDevice(device);   // the workspace's buffers are freed on this device
        delete w;
    }
    // At handle destroy: frees the idle workspaces now, and each leased one when it comes back.
    void close() {
        std::vector<W*> gone;
        {
            std::lock_guard<std::mutex> g(mu);
            closed = true;
            gone.swap(idle);
            for (W* w : gone) live.erase(std::remove(live.begin(), live.end(), w), live.end());
        }
        if (gone.empty()) return;
        cudaSetDevice(device);
        for (W* w : gone) delete w;
    }
};

// A workspace leased for the length of one call: on every return it is drained and goes back to the pool, unless a result
// has taken it over (take()).
template <typename W>
struct CallLease {
    Pool<W>& pool;
    W* w = nullptr;
    explicit CallLease(Pool<W>& p) : pool(p) {}
    CallLease(const CallLease&) = delete;
    CallLease& operator=(const CallLease&) = delete;
    ~CallLease() {
        if (!w) return;
        w->drain();
        pool.give_back(w);
    }
    W* take() {
        W* t = w;
        w = nullptr;
        return t;
    }
};

// The use events a workspace owns: created on demand and kept from one lease to the next.
struct UseEvents {
    std::vector<cudaEvent_t> ev;
    ~UseEvents() {
        for (cudaEvent_t e : ev) cudaEventDestroy(e);
    }
};

// The streams one lease of a device result was used on, in order of first use: the last use on streams[i] is recorded on
// the workspace's event i. One event per stream: re-recording covers that stream's earlier uses, but not another stream's.
struct StreamUses {
    std::mutex mu;
    std::vector<cudaStream_t> streams;

    // the event to record a use on `stream` on: this lease's event for it, or the workspace's next one (created if it has
    // none yet)
    cudaError_t event_for(UseEvents& events, cudaStream_t stream, cudaEvent_t* ev) {
        std::lock_guard<std::mutex> g(mu);
        size_t i = 0;
        while (i < streams.size() && streams[i] != stream) i++;
        if (i == streams.size()) {
            if (events.ev.size() == i) {
                cudaEvent_t e = nullptr;
                const cudaError_t err = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
                if (err != cudaSuccess) return err;
                events.ev.push_back(e);
            }
            streams.push_back(stream);
        }
        *ev = events.ev[i];
        return cudaSuccess;
    }
    // waits for the last use on every stream of this lease
    void wait(const UseEvents& events) {
        std::lock_guard<std::mutex> g(mu);
        for (size_t i = 0; i < streams.size(); i++) cudaEventSynchronize(events.ev[i]);
    }
};

// Checks that res is a completed forward device match: BFQ_E_INVALID without a lease, BFQ_E_STATE before a successful
// bfq_device_result_wait ("<who> needs a completed match"). Selects the result's device and returns in *ev the result's
// event for `stream`, which the caller records after its last launch (RecordOnExit).
int32_t lease_use(const bfq_device_result* res, cudaStream_t stream, const char* who, cudaEvent_t* ev);

// Records the event on every return path of the call, error returns after a launch included. If the record itself fails,
// the stream is synchronised instead, so release never hands back a workspace with unrecorded work on it.
struct RecordOnExit {
    cudaEvent_t ev;
    cudaStream_t stream;
    RecordOnExit(cudaEvent_t e, cudaStream_t s) : ev(e), stream(s) {}
    RecordOnExit(const RecordOnExit&) = delete;
    RecordOnExit& operator=(const RecordOnExit&) = delete;
    ~RecordOnExit() {
        if (cudaEventRecord(ev, stream) != cudaSuccess) cudaStreamSynchronize(stream);
    }
};

}  // namespace bfq
