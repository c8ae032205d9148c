// lease.h — what a call that enqueues work on a device result's leased workspace owes bfq_device_result_release.
//
// A device result's arrays live in a workspace leased from the handle's pool. Calls on a completed result (expand, budget,
// fan-out, delivery, exchange gather) enqueue kernels that read and write that workspace, and some of them return before
// those kernels run. bfq_device_result_release hands the workspace back to the pool, where the next match on the handle can
// take it, so it first waits for everything such calls enqueued: each call records an event of the result on its stream
// when it returns, one event per stream the result was used on.
#pragma once
#include <cuda_runtime.h>

#include "../../include/bfq_gpumatch.h"

namespace bfq {

// Checks that res is a completed device match: BFQ_E_INVALID without a lease, BFQ_E_STATE before a successful
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
