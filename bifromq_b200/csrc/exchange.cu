// exchange.cu — the ONE exchange step of the tenant-sharded path (SURVEY.md §8e; include/bfq_gpumatch.h "multi-GPU").
//
// Tenants are independent key ranges (DWS/KVSchemaUtil.java:91-94), so N GPUs match their own tenants' topics with no
// data-path collective. What has to travel is the reply: the dist-server reassembles the per-worker BatchDistReply messages
// into one answer per batch (bifromq-dist/bifromq-dist-server/.../scheduler/BatchDistServerCall.java:186-205,245-271). Here
// every rank contributes the device result of its own match — per topic the matched-route count and the number of matched
// ranges, plus the dense array of {first rank, count} ranges — and every rank ends with all ranks' results, in rank order:
//   1. local compaction of the sparse result (counts -> exclusive scan -> total), all on the caller's stream;
//   2. ncclAllGather of {n_topics, n_ranges} per rank (16 bytes) -> the ONE host synchronisation of the exchange: NCCL
//      needs the receive counts on the host;
//   3. the compaction's gather kernel writes this rank's dense ranges straight into its slice of the reassembly buffer (slices
//      have one padded stride, the largest rank's size);
//   4. one NCCL group of in-place ncclAllGather calls fills the other slices over NVLink / NVSwitch.
// No torch, no host-side copies, no per-element host work. NCCL is resolved at run time from the process (dlopen of
// libnccl.so.2: a Java host links the system library, a PyTorch host already carries its own copy).
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nccl.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "cuda_buf.h"
#include "lease.h"
#include "match_kernels.cuh"

using namespace bfq;

namespace {

struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
    std::string err;
};

NcclApi& nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        // the copy already in the process first (a PyTorch host has loaded its own), then the system library
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) {
            api.err = std::string("libnccl.so.2 not found: ") + (dlerror() ? dlerror() : "");
            return;
        }
        bool all = true;
        auto sym = [&](const char* name) {
            void* p = dlsym(h, name);
            if (!p) {
                all = false;
                api.err = std::string("NCCL symbol missing: ") + name;
            }
            return p;
        };
        api.GetUniqueId = (decltype(api.GetUniqueId)) sym("ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank)) sym("ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy)) sym("ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather)) sym("ncclAllGather");
        api.Broadcast = (decltype(api.Broadcast)) sym("ncclBroadcast");
        api.GroupStart = (decltype(api.GroupStart)) sym("ncclGroupStart");
        api.GroupEnd = (decltype(api.GroupEnd)) sym("ncclGroupEnd");
        api.GetErrorString = (decltype(api.GetErrorString)) sym("ncclGetErrorString");
        api.ok = all;
    });
    return api;
}
#define X_NCCL(expr)                                                                                \
    do {                                                                                            \
        ncclResult_t _r = (expr);                                                                   \
        if (_r != ncclSuccess) return fail(BFQ_E_CUDA, std::string(#expr) + ": " + nccl().GetErrorString(_r)); \
    } while (0)

// room for n elements, with headroom: the sizes move a little from batch to batch
template <typename T>
cudaError_t reserve_headroom(DeviceBuf<T>& b, size_t n) {
    return n <= b.cap ? cudaSuccess : b.reserve(std::max<size_t>(n + n / 4, 1024));
}

__global__ void exchange_meta_kernel(long long* meta, long long n_topics, const uint32_t* new_begin, const uint32_t* counts) {
    meta[0] = n_topics;
    meta[1] = n_topics > 0 ? (long long) new_begin[n_topics - 1] + counts[n_topics - 1] : 0;
}

}  // namespace

struct bfq_exchange {
    int device = 0, rank = 0, world = 1;
    ncclComm_t comm = nullptr;
    DeviceBuf<uint32_t> d_cnt, d_begin, d_final_begin, d_final_count;   // local compaction scratch
    DeviceBuf<uint8_t> d_scan_tmp;
    DeviceBuf<long long> d_meta;                 // {n_topics, n_ranges} x world
    PinnedBuf<long long> h_meta;                 // pinned copy
    DeviceBuf<uint32_t> g_route_count, g_span_count;
    DeviceBuf<uint2> g_ranges;
    std::vector<int64_t> topic_base, range_base, topic_count, range_count;
    ~bfq_exchange() {
        cudaSetDevice(device);   // the buffers are freed after this body, on this device
        if (comm && nccl().ok) nccl().CommDestroy(comm);
    }
};

extern "C" {

int32_t bfq_exchange_unique_id(uint8_t* id_out, int32_t cap) {
    if (!id_out || cap < (int32_t) sizeof(ncclUniqueId)) return fail(BFQ_E_INVALID, "id buffer must hold BFQ_EXCHANGE_ID_BYTES bytes");
    if (!nccl().ok) return fail(BFQ_E_STATE, nccl().err);
    ncclUniqueId id;
    X_NCCL(nccl().GetUniqueId(&id));
    memcpy(id_out, &id, sizeof(id));
    return BFQ_OK;
}

int32_t bfq_exchange_create(int32_t device_ordinal, int32_t rank, int32_t world, const uint8_t* id, bfq_exchange** out) {
    if (!out || !id || world < 1 || rank < 0 || rank >= world) return fail(BFQ_E_INVALID, "bad argument");
    if (!nccl().ok) return fail(BFQ_E_STATE, nccl().err);
    BFQ_CUDA_TRY(cudaSetDevice(device_ordinal));
    auto* x = new bfq_exchange();
    x->device = device_ordinal;
    x->rank = rank;
    x->world = world;
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof(uid));
    ncclResult_t r = nccl().CommInitRank(&x->comm, world, uid, rank);
    if (r != ncclSuccess) {
        x->comm = nullptr;
        delete x;
        return fail(BFQ_E_CUDA, std::string("ncclCommInitRank: ") + nccl().GetErrorString(r));
    }
    cudaError_t e = reserve_headroom(x->d_meta, (size_t) 2 * world);
    if (e == cudaSuccess) e = x->h_meta.reserve((size_t) 2 * world);
    if (e != cudaSuccess) {
        delete x;
        return fail(BFQ_E_CUDA, cudaGetErrorString(e));
    }
    x->topic_base.assign((size_t) world + 1, 0);
    x->range_base.assign((size_t) world + 1, 0);
    x->topic_count.assign((size_t) world, 0);
    x->range_count.assign((size_t) world, 0);
    *out = x;
    return BFQ_OK;
}

void bfq_exchange_destroy(bfq_exchange* x) { delete x; }

int32_t bfq_exchange_gather(bfq_exchange* x, const bfq_device_result* res, int32_t what, void* stream, bfq_gathered* out) {
    if (!x || !res || !out) return fail(BFQ_E_INVALID, "bad argument");
    if (what != BFQ_EXCHANGE_COUNTS && what != BFQ_EXCHANGE_RANGES) return fail(BFQ_E_INVALID, "what: BFQ_EXCHANGE_COUNTS or BFQ_EXCHANGE_RANGES");
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    const int32_t rc = lease_use(res, st, "bfq_exchange_gather", &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);   // the compaction's phase 2 reads the result's ranges after the call's one synchronisation
    BFQ_CUDA_TRY(cudaSetDevice(x->device));
    const int64_t n = res->n_topics;
    const int W = x->world;
    const bool with_ranges = what == BFQ_EXCHANGE_RANGES;
    // ---- 1. local compaction, phase 1 (counts, exclusive scan); the total goes into this rank's meta slot on the device
    BFQ_CUDA_TRY(reserve_headroom(x->d_cnt, (size_t) std::max<int64_t>(n, 1)));
    BFQ_CUDA_TRY(reserve_headroom(x->d_begin, (size_t) std::max<int64_t>(n, 1)));
    BFQ_CUDA_TRY(reserve_headroom(x->d_final_begin, (size_t) std::max<int64_t>(n, 1)));
    BFQ_CUDA_TRY(reserve_headroom(x->d_final_count, (size_t) std::max<int64_t>(n, 1)));
    CompactParams cp{};
    cp.n_topics = n;
    cp.span_begin = res->d_span_begin;
    cp.span_count = res->d_span_count;
    cp.ranges = reinterpret_cast<const uint2*>(res->d_ranges);
    cp.leader = nullptr;            // peers get every topic's ranges in full: a slice must be self-contained
    cp.counts = x->d_cnt.p;
    cp.new_begin = x->d_begin.p;
    cp.final_begin = x->d_final_begin.p;
    cp.final_count = x->d_final_count.p;
    cp.total_out = reinterpret_cast<unsigned long long*>(x->d_meta.p + 2 * x->rank + 1);
    size_t tmp_bytes = 0;
    {
        CompactParams q = cp;
        q.n_topics = std::max<int64_t>(n, 1);
        BFQ_CUDA_TRY(launch_compact(q, nullptr, &tmp_bytes, st, 1));
        BFQ_CUDA_TRY(reserve_headroom(x->d_scan_tmp, tmp_bytes + 256));
    }
    if (n > 0) BFQ_CUDA_TRY(launch_compact(cp, x->d_scan_tmp.p, &tmp_bytes, st, 1));
    exchange_meta_kernel<<<1, 1, 0, st>>>(x->d_meta.p + 2 * x->rank, (long long) n, x->d_begin.p, x->d_cnt.p);
    BFQ_CUDA_TRY(cudaGetLastError());
    // ---- 2. sizes of every rank (the receive counts NCCL needs on the host): the exchange's one host synchronisation
    X_NCCL(nccl().AllGather(x->d_meta.p + 2 * x->rank, x->d_meta.p, 2, ncclInt64, x->comm, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(x->h_meta.p, x->d_meta.p, (size_t) 2 * W * sizeof(long long), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    // every rank's slice has the same (padded) stride, so the payload travels as plain ncclAllGather calls — the ring / NVLS
    // algorithms at full NVLink rate, where per-root broadcasts of exactly-sized slices would serialise the roots
    int64_t max_t = 1, max_r = 1;
    for (int r = 0; r < W; r++) {
        max_t = std::max<int64_t>(max_t, x->h_meta.p[2 * r]);
        max_r = std::max<int64_t>(max_r, x->h_meta.p[2 * r + 1]);
    }
    max_t = (max_t + 31) / 32 * 32;   // keep every slice 128-byte aligned
    max_r = (max_r + 15) / 16 * 16;
    int64_t nt_all = 0, nr_all = 0;
    for (int r = 0; r < W; r++) {
        x->topic_base[(size_t) r] = (int64_t) r * max_t;
        x->range_base[(size_t) r] = (int64_t) r * max_r;
        x->topic_count[(size_t) r] = x->h_meta.p[2 * r];
        x->range_count[(size_t) r] = x->h_meta.p[2 * r + 1];
        nt_all += x->h_meta.p[2 * r];
        nr_all += x->h_meta.p[2 * r + 1];
    }
    x->topic_base[(size_t) W] = (int64_t) W * max_t;
    x->range_base[(size_t) W] = (int64_t) W * max_r;
    if ((int64_t) W * max_r >= (int64_t) 0xFFFFFFF0ll) return fail(BFQ_E_RANGE, "more than 2^32 ranges in one exchanged batch; split the batch");
    BFQ_CUDA_TRY(reserve_headroom(x->g_route_count, (size_t) (W * max_t)));
    if (with_ranges) {
        BFQ_CUDA_TRY(reserve_headroom(x->g_span_count, (size_t) (W * max_t)));
        BFQ_CUDA_TRY(reserve_headroom(x->g_ranges, (size_t) (W * max_r)));
    }
    // ---- 3. this rank's slice, written in place
    const int64_t tb = x->topic_base[(size_t) x->rank], rb = x->range_base[(size_t) x->rank];
    if (n > 0) {
        BFQ_CUDA_TRY(cudaMemcpyAsync(x->g_route_count.p + tb, res->d_route_count, (size_t) n * 4, cudaMemcpyDeviceToDevice, st));
        if (with_ranges) {
            BFQ_CUDA_TRY(cudaMemcpyAsync(x->g_span_count.p + tb, x->d_cnt.p, (size_t) n * 4, cudaMemcpyDeviceToDevice, st));
            cp.ranges_out = x->g_ranges.p + rb;
            cp.ranges_out_cap = (uint64_t) x->h_meta.p[2 * x->rank + 1];
            cp.out_base = 0;
            BFQ_CUDA_TRY(launch_compact(cp, x->d_scan_tmp.p, &tmp_bytes, st, 2));
        }
    }
    // ---- 4. every rank's slice to every rank: in-place all-gathers over the padded slices, one NCCL group
    if (W > 1) {
        X_NCCL(nccl().GroupStart());
        X_NCCL(nccl().AllGather(x->g_route_count.p + tb, x->g_route_count.p, (size_t) max_t, ncclUint32, x->comm, st));
        if (with_ranges) {
            X_NCCL(nccl().AllGather(x->g_span_count.p + tb, x->g_span_count.p, (size_t) max_t, ncclUint32, x->comm, st));
            X_NCCL(nccl().AllGather(x->g_ranges.p + rb, x->g_ranges.p, (size_t) max_r * 2, ncclUint32, x->comm, st));
        }
        X_NCCL(nccl().GroupEnd());
    }
    out->d_route_count = x->g_route_count.p;
    out->d_span_count = with_ranges ? x->g_span_count.p : nullptr;
    out->d_ranges = with_ranges ? reinterpret_cast<const bfq_range*>(x->g_ranges.p) : nullptr;
    out->topic_base = x->topic_base.data();
    out->range_base = x->range_base.data();
    out->topic_count = x->topic_count.data();
    out->range_count = x->range_count.data();
    out->n_topics_total = nt_all;
    out->n_ranges_total = nr_all;
    out->world = W;
    out->bytes_received = (nt_all - n) * (with_ranges ? 8 : 4) + (with_ranges ? (nr_all - x->h_meta.p[2 * x->rank + 1]) * 8 : 0);
    return BFQ_OK;
}

}  // extern "C"
