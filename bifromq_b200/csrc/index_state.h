// index_state.h — the state behind a forward index handle, shared by capi.cu (index, commits, match) and result_calls.cu (the
// calls on a completed device result): snapshots, workspaces and their pool, the handle, and a device match in flight.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <memory>
#include <mutex>
#include <thread>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "cuda_buf.h"
#include "fanout.h"
#include "index_builder.h"
#include "match_kernels.cuh"

namespace bfq {

// ------------------------------------------------------------------------------------------------ snapshots
// One committed state of the index: device arrays + the host-side tables results are resolved against (segment table,
// route kinds, raw KV). Immutable once published and reference counted: every match pins the snapshot it ran on, so a
// result's ranks always resolve against the KV order they were produced from, whatever is committed meanwhile.
struct Snapshot {
    int device = 0;
    uint64_t generation = 0;
    DeviceBuf<Slot> d_slots, d_roots;
    DeviceBuf<uint32_t> d_segs, d_pfxP, d_pfxG;
    DeviceBuf<uint8_t> d_rkind, d_tags;
    FlatIndex flat;          // host copy (segs / tenant map / tenant table / statistics; the uploaded arrays are dropped)
    // per tenant, aligned with flat.tenants (key order): the committed KV (route lookups; shared with the staging area and
    // with the neighbouring snapshots, a delta commit replaces only the touched tenants') and the route kinds
    struct TenantHost {
        std::shared_ptr<const KVBlob> kv;
        std::shared_ptr<const std::vector<uint8_t>> rkind;
        std::shared_ptr<const TenantFan> fan;   // routes -> deliverer ids, built on the first fan-out that sees this blob
        std::shared_ptr<const TenantWire> wire; // routes -> MatchInfo bytes, built on the first encode that sees this blob
    };
    // fan-out tables of the whole snapshot (device), assembled from the tenants' on first use
    struct FanTable {
        DeviceBuf<uint32_t> d_rdeliv, d_gmem_off, d_gmem_deliv;
        DeviceBuf<uint8_t> d_gordered;
        uint32_t n_deliverers = 0;   // incl. the reserved last id (ordered shared subscriptions)
    };
    // receiverUrls of the ordered groups' members (device), for the $oshare pick: built on the first ordered delivery call
    struct UrlTable {
        DeviceBuf<unsigned long long> d_words;   // member m: its url at byte 4 of words d_word[m] .., zero-padded
        DeviceBuf<long long> d_word;             // [members of the fan table]
        DeviceBuf<uint32_t> d_len;
        uint32_t member_bits = 1;                // bits of the largest ordered group's size
    };
    // every route's MatchInfo bytes (device), for bfq_delivery_encode: built on the first encode call
    struct WireTable {
        DeviceBuf<uint32_t> d_first;             // per rank: its first entry
        DeviceBuf<unsigned long long> d_off;     // [entries + 1]
        DeviceBuf<uint8_t> d_bytes;
        size_t n_entries = 0;
        int64_t bytes() const { return (int64_t) (d_first.bytes() + d_off.bytes() + d_bytes.bytes()); }
    };
    std::mutex fan_mu;
    std::shared_ptr<FanTable> fan;
    std::shared_ptr<UrlTable> urls;
    std::shared_ptr<WireTable> wire;
    std::shared_ptr<DeviceBuf<uint32_t>> mi_hash;   // per MatchInfo table entry, for bfq_delivery_reply: built on its first call
    std::atomic<int64_t> wire_bytes{0};      // wire->bytes() once built (bfq_index_stats reads it without fan_mu)
    std::vector<TenantHost> th;
    uint64_t garbage_slots = 0;   // slots of regions that delta commits replaced (reclaimed by the next full build)
    int64_t delta_commits = 0;    // delta commits since the last full build
    size_t l2_window_bytes = 0;
    // rank -> (index into flat.tenants, rank inside the tenant); false if out of range
    bool locate(int64_t rank, size_t* ti, int64_t* local) const {
        if (rank < 0 || rank >= flat.n_routes || flat.tenants.empty()) return false;
        size_t lo = 0, hi = flat.tenants.size();
        while (hi - lo > 1) {
            const size_t mid = (lo + hi) / 2;
            if (flat.tenants[mid].lo <= rank) lo = mid;
            else hi = mid;
        }
        *ti = lo;
        *local = rank - flat.tenants[lo].lo;
        return *local < flat.tenants[lo].n_routes;
    }
    int64_t device_bytes() const {
        return (int64_t) (d_slots.bytes() + d_tags.bytes() + d_roots.bytes() + d_segs.bytes() + d_rkind.bytes() + d_pfxP.bytes() + d_pfxG.bytes());
    }
    ~Snapshot() { cudaSetDevice(device); }   // runs before the members are destroyed: the buffers are freed on this device
};

constexpr int MAX_CHUNKS = 8;

// Everything ONE match in flight needs: streams, device scratch, pinned result buffers. A workspace is leased from the
// index's pool for the duration of a call AND of the result it produced (the result's arrays live in it), so concurrent
// matches on one handle never share a buffer. Returned to the pool by bfq_result_free / bfq_device_result_release.
struct Workspace {
    int device = 0;
    cudaStream_t stream = nullptr, copy_stream = nullptr, work_stream[2] = {nullptr, nullptr};
    cudaEvent_t ev[2] = {nullptr, nullptr};
    cudaEvent_t ev_h2d[MAX_CHUNKS] = {};
    cudaEvent_t evk[2] = {nullptr, nullptr};
    cudaEvent_t ev_done = nullptr;   // device path: recorded behind the last thing a match enqueued (what wait() waits for)
    std::vector<cudaEvent_t> ev_use; // device path: one per stream the result was used on after the match (lease.h), created on demand
    // resolved tenant table of the previous call on this workspace (reused when the same list comes again)
    uint64_t tab_generation = ~0ull;
    std::vector<uint8_t> tab_blob;
    std::vector<int64_t> tab_off;
    std::vector<int32_t> tab_caps;
    int32_t tab_n = -1;
    bool any_cap = true;
    DeviceBuf<int32_t> d_tenant_tab;   // root | maxP | maxG, 3 x n_tenants
    PinnedBuf<int32_t> h_tenant_tab;
    // per-call device buffers
    DeviceBuf<uint8_t> d_topics;
    DeviceBuf<int64_t> d_topic_off;
    DeviceBuf<int32_t> d_topic_tenant;
    DeviceBuf<uint32_t> d_span_begin, d_span_count, d_route_count, d_overflow, d_flagged, d_kept, d_defer;
    DeviceBuf<uint2> d_ranges, d_scratch, d_ranges_c;
    DeviceBuf<uint8_t> d_scan_tmp;
    DeviceBuf<uint32_t> d_cnt, d_new_begin, d_final_begin, d_final_count;
    // locality order + dedup (launch_order): per compute-stream slot (two sub-batches can be in flight)
    DeviceBuf<uint32_t> d_ord_keys, d_leader, d_order;
    DeviceBuf<SpanRecord> d_pos_rec;            // tier 0's span record per work-order position (MatchParams::pos_rec)
    DeviceBuf<unsigned long long> d_hash_tab;   // 2 x hash_stride
    DeviceBuf<uint32_t> d_hist;                 // 2 x hist_stride (launch_order's scratch)
    size_t hash_stride = 0, hist_stride = 0;
    DeviceBuf<uint3> d_throttled;
    DeviceBuf<unsigned long long> d_counters;
    PinnedBuf<unsigned long long> h_counters;
    DeviceBuf<unsigned long long> d_exp_counts;
    // calls on a completed device result (result_calls.cu): one arena per call family, laid out by its call (carve), and the cub
    // scratch of the families that do not use d_scan_tmp. A family's outputs stay valid until its next call on this workspace.
    DeviceBuf<uint8_t> d_bud;                  // bfq_expand_device_budget
    DeviceBuf<uint8_t> d_fo, d_fo_tmp;         // bfq_fanout_device
    DeviceBuf<uint8_t> d_os, d_dl, d_dl_tmp;   // delivery: $oshare phase 1 (read by phase 2), and the nesting
    DeviceBuf<uint8_t> d_wr, d_wr_tmp;         // bfq_delivery_encode
    DeviceBuf<uint8_t> d_rp, d_rp_tmp;         // bfq_delivery_reply
    PinnedBuf<unsigned long long> h_rp_ctr;
    // the nesting the last delivery call left in d_dl (n_packs < 0: none, or a call that failed): its counts and the pointers
    // it returned, which encode and reply compare a nesting against
    int64_t dl_n_pairs = -1, dl_n_packages = -1, dl_n_packs = -1;
    bool dl_ordered = false;
    const int64_t *dl_package_off = nullptr, *dl_match_off = nullptr, *dl_pack_pub_off = nullptr;
    // pinned result buffers
    PinnedBuf<uint32_t> h_span_begin, h_span_count, h_route_count;
    PinnedBuf<uint2> h_ranges;
    PinnedBuf<uint3> h_throttled;

    cudaError_t init(int dev) {
        device = dev;
        cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking);
        for (auto& w : work_stream)
            if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&w, cudaStreamNonBlocking);
        for (auto& x : ev)
            if (e == cudaSuccess) e = cudaEventCreate(&x);
        for (auto& x : evk)
            if (e == cudaSuccess) e = cudaEventCreate(&x);
        for (auto& x : ev_h2d)
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&x, cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_done, cudaEventDisableTiming);
        return e;
    }
    ~Workspace() {
        cudaSetDevice(device);   // the buffers are freed after this body, on this device
        for (auto& e : ev) if (e) cudaEventDestroy(e);
        for (auto& e : evk) if (e) cudaEventDestroy(e);
        for (auto& e : ev_h2d) if (e) cudaEventDestroy(e);
        if (ev_done) cudaEventDestroy(ev_done);
        for (auto& e : ev_use) cudaEventDestroy(e);
        if (copy_stream) cudaStreamDestroy(copy_stream);
        for (auto& w : work_stream) if (w) cudaStreamDestroy(w);
        if (stream) cudaStreamDestroy(stream);
    }
};

// idle workspaces of one index. Shared with every result / lease in flight, so that freeing a result after its index was
// destroyed (a garbage-collected host language decides the order) still has a valid place to return its workspace to.
struct Pool {
    std::mutex mu;
    std::vector<Workspace*> idle;
    int device = 0;
    bool closed = false;
    ~Pool() {
        cudaSetDevice(device);
        for (Workspace* w : idle) delete w;
    }
};

struct CoreOut {
    int64_t n_ranges = 0, n_throttled = 0, n_overflow = 0, n_flagged = 0, n_launches = 0, n_deferred = 0, n_leaders = 0;
    uint64_t want_dyn = 0, want_thr = 0;
    int64_t chunk_throttled[MAX_CHUNKS] = {};
};

struct CoreCtx {
    bfq_index* h;
    Workspace* w;
    const Snapshot* s;
    const uint8_t* d_topics;
    const int64_t* d_topic_off;
    const int32_t* d_topic_tenant;
    int32_t n_tenants;
    cudaStream_t stream;
};

// A device-side match in flight (bfq_match_device_async .. bfq_device_result_wait .. bfq_device_result_release)
struct DeviceLease {
    bfq_index* h = nullptr;
    std::shared_ptr<Pool> pool;
    std::shared_ptr<Snapshot> snap;
    Workspace* ws = nullptr;
    CoreCtx ctx{};
    int64_t n = 0;
    bool done = false;
    int32_t rc = BFQ_OK;
    CoreOut co;
    double tier0_ms = 0;
    // streams the result was used on after the match; stream i's last use is recorded on ws->ev_use[i] (lease.h). One event
    // per stream: re-recording covers that stream's earlier uses, but not another stream's.
    std::mutex use_mu;
    std::vector<cudaStream_t> used_on;
};

}  // namespace bfq

// the handle (global: the C-ABI names it)
struct bfq_index {
    int device = 0;
    std::mutex mu;         // current snapshot pointer, workspace pool, statistics
    std::mutex stage_mu;   // staging area: reset / load / apply and the (long) host-side rebuild of commit
    bfq::Staging staging;
    std::shared_ptr<bfq::Snapshot> snap;
    uint64_t next_generation = 1;
    std::shared_ptr<bfq::Pool> pool = std::make_shared<bfq::Pool>();   // idle workspaces
    std::shared_ptr<bfq::DelivererTable> deliverers = std::make_shared<bfq::DelivererTable>();   // (subBrokerId, delivererKey) -> id, append-only
    int64_t order_min = 32768;           // batches smaller than this are matched in arrival order (BFQ_ORDER=0: never order)
    bool dedup = true;                   // BFQ_DEDUP=0: match duplicates of a (tenant, topic) pair separately
    int32_t tier0_ctas_per_sm = 0;       // bfq_index_set_option("tier0_ctas_per_sm"): 0 = as many as fit
    int32_t dedup_hash_bits = 64;        // bfq_index_set_option("dedup_hash_bits"): test knob, < 64 forces de-dup hash collisions
    bool fanout_global = false;          // bfq_index_set_option("fanout_global"): test knob, every fan-out takes the global pass
    double last_kernel_ms = 0;
    int64_t launches = 0, overflow_topics = 0, flagged_topics = 0, deferred_topics = 0, duplicate_topics = 0, buffer_retries = 0;
    int64_t global_fanouts = 0;
    int64_t full_commits = 0, delta_commits = 0;
    int64_t rebuilt_tenants = 0;         // tenants the last commit built (bfq_index_stats slot 21)
    // Releases the host image of a full build (2.3 GB of records at 10M filters: 0.4 s of page freeing) off the committing
    // thread. Touched under stage_mu only (commits are serialised); joined before the next one starts and at destroy.
    std::thread janitor;

    ~bfq_index() {
        if (janitor.joinable()) janitor.join();
        cudaSetDevice(device);
        std::vector<bfq::Workspace*> idle;
        {
            std::lock_guard<std::mutex> g(pool->mu);
            pool->closed = true;   // workspaces still leased are freed when they come back
            idle.swap(pool->idle);
        }
        for (bfq::Workspace* w : idle) delete w;
    }
};
