// capi.cu — implementation of the C-ABI declared in include/bfq_gpumatch.h (forward index + match).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>
#include <string>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "codec.h"
#include "cuda_buf.h"
#include "index_builder.h"
#include "fanout.h"
#include "lease.h"
#include "match_kernels.cuh"

using namespace bfq;

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
    // delivery budgets (bfq_expand_device_budget)
    DeviceBuf<long long> d_bud_bytes;
    DeviceBuf<uint8_t> d_bud_bw, d_bud_flags;
    DeviceBuf<uint32_t> d_bud_dp, d_bud_list;
    DeviceBuf<unsigned long long> d_bud_ctr;
    // fan-out expansion (fanout.cu)
    DeviceBuf<uint32_t> d_fo_counts, d_fo_base, d_pack_topic, d_pack_rank, d_pack_member;
    DeviceBuf<long long> d_pack_offsets;
    DeviceBuf<uint8_t> d_fo_tmp;
    // delivery nesting (fanout.cu: launch_delivery): scratch per topic (6 words each + 2) and per pair (10 words each + 2), the outputs
    DeviceBuf<uint32_t> d_dl_topic_tmp, d_dl_pair_tmp, d_dl_pcount, d_package_tenant, d_dl_pack_topic, d_match_rank, d_match_member;
    DeviceBuf<unsigned long long> d_dl_totals;
    DeviceBuf<long long> d_package_off, d_dl_pack_off, d_match_off;
    DeviceBuf<uint8_t> d_dl_tmp;
    // $oshare resolution (bfq_delivery_device_ordered): per CSR pair flags and item counts, the check words, the sort keys of
    // pairs and items, the per-item / per-emit-position words, and the publisher outputs
    DeviceBuf<uint32_t> d_os_flag, d_os_u32, d_pack_pub;
    DeviceBuf<unsigned long long> d_os_items, d_os_check, d_os_key;
    DeviceBuf<long long> d_pack_pub_off;
    // the nesting the last delivery call left in the buffers above (n_packs < 0: none, or a call that failed)
    int64_t dl_n_pairs = -1, dl_n_packages = -1, dl_n_packs = -1;
    bool dl_ordered = false;
    // DeliveryRequest encoding (bfq_delivery_encode): the size scans (pairs, packs, packages), the checks, the offsets
    DeviceBuf<unsigned long long> d_wr_pos, d_wr_check;
    DeviceBuf<long long> d_req_off, d_wr_tenant_off;
    DeviceBuf<uint8_t> d_wr_tenants, d_wr_tmp;
    // DeliveryReply join (bfq_delivery_reply): per deliverer, per map entry slot (one per package), per chunk, the key table,
    // per pair, the stale lists, and the outputs
    DeviceBuf<unsigned long long> d_rp_ctr, d_rp_chunk_base, d_rp_slot_key, d_rp_slot_rpos, d_rp_pkg_stale;
    DeviceBuf<uint8_t> d_rp_dl_fail, d_rp_ent_bad, d_rp_tmp, d_rp_pair_code, d_rp_status, d_rp_tenants;
    DeviceBuf<int32_t> d_rp_dl_code;
    DeviceBuf<uint32_t> d_rp_u32;
    DeviceBuf<long long> d_rp_ent, d_rp_chunks, d_rp_tenant_off;
    DeviceBuf<bfq_stale_match> d_rp_stale;
    PinnedBuf<unsigned long long> h_rp_ctr;
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

struct bfq_result {
    bfq_index* owner = nullptr;
    std::shared_ptr<Pool> pool;
    std::shared_ptr<Snapshot> snap;      // the snapshot the match ran on (ranks resolve against it)
    Workspace* ws = nullptr;             // leased: the arrays below live in its pinned buffers
    int64_t n_topics = 0, n_ranges = 0, n_throttled = 0;
    const uint32_t *span_begin = nullptr, *span_count = nullptr, *route_count = nullptr;
    const bfq_range* ranges = nullptr;
    const bfq_throttled* throttled = nullptr;
    double ms[4] = {0, 0, 0, 0};
};

struct bfq_index {
    int device = 0;
    std::mutex mu;         // current snapshot pointer, workspace pool, statistics
    std::mutex stage_mu;   // staging area: reset / load / apply and the (long) host-side rebuild of commit
    Staging staging;
    std::shared_ptr<Snapshot> snap;
    uint64_t next_generation = 1;
    std::shared_ptr<Pool> pool = std::make_shared<Pool>();   // idle workspaces
    std::shared_ptr<DelivererTable> deliverers = std::make_shared<DelivererTable>();   // (subBrokerId, delivererKey) -> id, append-only
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
        std::vector<Workspace*> idle;
        {
            std::lock_guard<std::mutex> g(pool->mu);
            pool->closed = true;   // workspaces still leased are freed when they come back
            idle.swap(pool->idle);
        }
        for (Workspace* w : idle) delete w;
    }
};

namespace {

constexpr size_t POOL_KEEP = 4;   // idle workspaces kept for reuse; more are freed when they come back

int32_t acquire(bfq_index* h, std::shared_ptr<Snapshot>* snap, Workspace** ws, const char* who) {
    Workspace* w = nullptr;
    {
        std::lock_guard<std::mutex> g(h->mu);
        if (!h->snap) return fail(BFQ_E_STATE, std::string(who) + " before the first bfq_index_commit");
        *snap = h->snap;
    }
    {
        std::lock_guard<std::mutex> g(h->pool->mu);
        if (!h->pool->idle.empty()) {
            w = h->pool->idle.back();
            h->pool->idle.pop_back();
        }
    }
    if (!w) {
        w = new Workspace();
        cudaError_t e = w->init(h->device);
        if (e != cudaSuccess) {
            delete w;
            return fail(BFQ_E_CUDA, std::string("workspace: ") + cudaGetErrorString(e));
        }
    }
    w->dl_n_packs = -1;   // a new lease starts without a delivery nesting: one left by the previous lease is not this result's
    *ws = w;
    return BFQ_OK;
}

void give_back(const std::shared_ptr<Pool>& pool, Workspace* w) {
    if (!w) return;
    {
        std::lock_guard<std::mutex> g(pool->mu);
        if (!pool->closed && pool->idle.size() < POOL_KEEP) {
            pool->idle.push_back(w);
            return;
        }
    }
    cudaSetDevice(pool->device);
    delete w;
}

struct CoreOut {
    int64_t n_ranges = 0, n_throttled = 0, n_overflow = 0, n_flagged = 0, n_launches = 0, n_deferred = 0, n_leaders = 0;
    uint64_t want_dyn = 0, want_thr = 0;
    int64_t chunk_throttled[MAX_CHUNKS] = {};
};

// tenant ids -> root ordinals of this snapshot + caps, uploaded to the workspace (skipped when the previous call on this
// workspace carried the same list against the same snapshot: compared byte for byte, not by fingerprint)
int32_t resolve_tenants(Workspace* w, const Snapshot* s, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                        const int32_t* max_p, const int32_t* max_g, cudaStream_t stream) {
    if (n_tenants < 0) return fail(BFQ_E_INVALID, "n_tenants < 0");
    if (n_tenants >= (1 << 30)) return fail(BFQ_E_RANGE, "more than 2^30 tenants in one batch");   // bit 30 of the lane's tenant word is a flag
    const size_t nt = (size_t) std::max(n_tenants, 1);
    const size_t blob_n = n_tenants ? (size_t) (tenant_off[n_tenants] - tenant_off[0]) : 0;
    bool same = w->tab_generation == s->generation && w->tab_n == n_tenants && w->tab_blob.size() == blob_n;
    if (same && n_tenants > 0) {
        same = memcmp(w->tab_blob.data(), tenants + tenant_off[0], blob_n) == 0;
        for (int32_t i = 0; same && i <= n_tenants; i++) same = w->tab_off[i] == tenant_off[i] - tenant_off[0];
        for (int32_t i = 0; same && i < n_tenants; i++)
            same = w->tab_caps[i] == (max_p ? max_p[i] : 0x7FFFFFFF) && w->tab_caps[nt + i] == (max_g ? max_g[i] : 0x7FFFFFFF);
    }
    if (same) return BFQ_OK;
    BFQ_CUDA_TRY(w->h_tenant_tab.reserve(3 * nt));
    BFQ_CUDA_TRY(w->d_tenant_tab.reserve(3 * nt));
    w->tab_blob.assign(tenants ? tenants + (n_tenants ? tenant_off[0] : 0) : nullptr, tenants ? tenants + (n_tenants ? tenant_off[0] : 0) + blob_n : nullptr);
    w->tab_off.resize(nt + 1);
    w->tab_caps.assign(2 * nt, 0x7FFFFFFF);
    bool any_cap = false;
    for (int32_t i = 0; i < n_tenants; i++) {
        std::string t((const char*) tenants + tenant_off[i], (size_t) (tenant_off[i + 1] - tenant_off[i]));
        auto it = s->flat.tenant_ordinal.find(t);
        const int32_t mp = max_p ? max_p[i] : 0x7FFFFFFF, mg = max_g ? max_g[i] : 0x7FFFFFFF;
        w->h_tenant_tab.p[i] = it == s->flat.tenant_ordinal.end() ? -1 : (int32_t) it->second;
        w->h_tenant_tab.p[nt + i] = mp;
        w->h_tenant_tab.p[2 * nt + i] = mg;
        w->tab_off[i] = tenant_off[i] - tenant_off[0];
        w->tab_caps[i] = mp;
        w->tab_caps[nt + i] = mg;
        any_cap = any_cap || mp != 0x7FFFFFFF || mg != 0x7FFFFFFF;
    }
    if (n_tenants > 0) w->tab_off[n_tenants] = tenant_off[n_tenants] - tenant_off[0];
    // the workspace is idle between calls, so nothing reads the pinned staging table while it is rewritten; the streams
    // that read the device table are ordered behind this copy (same stream, or through the H2D events of the host path)
    BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_tenant_tab.p, w->h_tenant_tab.p, 3 * nt * sizeof(int32_t), cudaMemcpyHostToDevice, stream));
    w->tab_generation = s->generation;
    w->tab_n = n_tenants;
    w->any_cap = any_cap;
    return BFQ_OK;
}

// One sub-batch of a match: topics [begin, begin + n) of a batch of n_total. Device buffers are indexed by the position
// in the whole batch, so sub-batches of one call never overlap; each has its own counter block, its own slice of the
// dynamic range region and of the throttled list.
struct SubBatch {
    int64_t begin = 0, n = 0, n_total = 0;
    int chunk = 0;
    uint64_t dyn_off = 0, dyn_cap = 0;     // slice of ranges[n_total * INLINE_RANGES ...) for tiers 1/2
    uint64_t thr_off = 0, thr_cap = 0;     // slice of the throttled list
};
constexpr int32_t BFQ_RETRY_GROW = -100;   // internal: a slice was too small, redo the batch un-chunked with bigger buffers

int32_t prepare_workspace(bfq_index* h, Workspace* w, int64_t n, int n_chunks, int32_t n_tenants) {
    const size_t nn = (size_t) std::max<int64_t>(n, 1);
    if (n >= (int64_t) 0x3FFFFFFF) return fail(BFQ_E_INVALID, "too many topics in one batch");
    BFQ_CUDA_TRY(w->d_span_begin.reserve(nn));
    BFQ_CUDA_TRY(w->d_span_count.reserve(nn));
    BFQ_CUDA_TRY(w->d_route_count.reserve(nn));
    BFQ_CUDA_TRY(w->d_overflow.reserve(nn));
    BFQ_CUDA_TRY(w->d_flagged.reserve(nn));
    BFQ_CUDA_TRY(w->d_kept.reserve(nn));
    BFQ_CUDA_TRY(w->d_defer.reserve(nn));
    BFQ_CUDA_TRY(w->d_counters.reserve(CTR_COUNT * MAX_CHUNKS));
    BFQ_CUDA_TRY(w->h_counters.reserve(CTR_COUNT * MAX_CHUNKS));
    // ranges[0, n * INLINE_RANGES): tier-0 inline slots; the rest: cursor-allocated region of tiers 1 and 2
    const uint64_t dyn_base = (uint64_t) n * INLINE_RANGES;
    if (dyn_base >= 0xF0000000ull) return fail(BFQ_E_RANGE, "batch too large for 32-bit range indices; split the batch");
    const size_t min_dyn = std::max<size_t>((size_t) n_chunks << 18, nn);
    if (w->d_ranges.cap < dyn_base + min_dyn) BFQ_CUDA_TRY(w->d_ranges.reserve((size_t) (dyn_base + std::max<size_t>(1 << 20, min_dyn))));
    const int64_t per_chunk = (n + n_chunks - 1) / n_chunks + 1;
    if (per_chunk >= h->order_min) {
        BFQ_CUDA_TRY(w->d_ord_keys.reserve(nn));
        BFQ_CUDA_TRY(w->d_leader.reserve(nn));
        BFQ_CUDA_TRY(w->d_order.reserve(nn));
        BFQ_CUDA_TRY(w->d_pos_rec.reserve(nn));
        const size_t hist_stride = order_scratch_words(per_chunk, n_tenants);
        const size_t hash_stride = order_hash_entries(per_chunk);
        if (hist_stride > w->hist_stride) {
            BFQ_CUDA_TRY(w->d_hist.reserve(2 * hist_stride));
            w->hist_stride = hist_stride;
        }
        if (hash_stride > w->hash_stride) {
            BFQ_CUDA_TRY(w->d_hash_tab.reserve(2 * hash_stride));
            w->hash_stride = hash_stride;
        }
    }
    if (w->d_throttled.cap < ((size_t) n_chunks << 14)) BFQ_CUDA_TRY(w->d_throttled.reserve(std::max<size_t>(1 << 16, (size_t) n_chunks << 14)));
    return BFQ_OK;
}

SubBatch whole_batch(Workspace* w, int64_t n) {
    SubBatch sb;
    sb.begin = 0;
    sb.n = sb.n_total = n;
    sb.dyn_cap = w->d_ranges.cap - (uint64_t) n * INLINE_RANGES;
    sb.thr_cap = w->d_throttled.cap;
    return sb;
}

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

MatchParams core_params(const CoreCtx& c, const SubBatch& sb) {
    Workspace* w = c.w;
    const size_t nt = (size_t) std::max(c.n_tenants, 1);
    const int64_t b = sb.begin;
    MatchParams p{};
    p.slots = c.s->d_slots.p;
    p.roots = c.s->d_roots.p;
    p.tags = reinterpret_cast<const uint4*>(c.s->d_tags.p);
    p.n_blocks = c.s->flat.n_blocks;
    p.topics = c.d_topics;
    p.topic_off = c.d_topic_off + b;
    p.topic_tenant = c.d_topic_tenant + b;
    p.tenant_root = w->d_tenant_tab.p;
    p.max_pfanout = w->d_tenant_tab.p + nt;
    p.max_gfanout = w->d_tenant_tab.p + 2 * nt;
    p.n_tenants = c.n_tenants;
    p.n_topics = sb.n;
    p.span_begin = w->d_span_begin.p + b;
    p.span_count = w->d_span_count.p + b;
    p.route_count = w->d_route_count.p + b;
    p.overflow_list = w->d_overflow.p + b;
    p.defer_list = w->d_defer.p + b;
    p.flagged_list = w->d_flagged.p + b;
    p.counters = w->d_counters.p + (size_t) sb.chunk * CTR_COUNT;
    // range indices are relative to the sub-batch's first inline slot
    p.ranges = w->d_ranges.p + (uint64_t) b * INLINE_RANGES;
    p.dyn_base = (uint64_t) (sb.n_total - b) * INLINE_RANGES + sb.dyn_off;
    p.ranges_cap = p.dyn_base + sb.dyn_cap;
    p.max_ctas_per_sm = c.h->tier0_ctas_per_sm;
    return p;
}

CapsParams caps_params(const CoreCtx& c, const SubBatch& sb, const MatchParams& p) {
    CapsParams q{};
    q.flagged_list = p.flagged_list;
    q.topic_tenant = p.topic_tenant;
    q.max_pfanout = p.max_pfanout;
    q.max_gfanout = p.max_gfanout;
    q.span_begin = p.span_begin;
    q.span_count = p.span_count;
    q.ranges = p.ranges;
    q.segs = c.s->d_segs.p;
    q.rkind = c.s->d_rkind.p;
    q.pfx_persistent = c.s->d_pfxP.p;
    q.pfx_group = c.s->d_pfxG.p;
    q.kept_count = c.w->d_kept.p + sb.begin;
    q.counters = p.counters;
    q.throttled = c.w->d_throttled.p + sb.thr_off;
    q.throttled_cap = sb.thr_cap;
    q.topic_base = (uint32_t) sb.begin;
    return q;
}

bool wants_order(const CoreCtx& c, const SubBatch& sb) {
    return sb.n >= c.h->order_min && c.w->d_order.cap >= (size_t) (sb.begin + sb.n) &&
           c.w->d_pos_rec.cap >= (size_t) (sb.begin + sb.n) && c.w->hist_stride > 0 &&
           c.w->hist_stride >= order_scratch_words(sb.n, c.n_tenants) && c.w->hash_stride >= order_hash_entries(sb.n);
}

// Enqueues one sub-batch on c.stream WITHOUT synchronising: [dedup + locality order] -> tier 0 -> tier 1 -> [span records
// to topic order, followers] -> [caps], every count read on the device. The host looks at the counters only in finish_core.
int32_t enqueue_core(const CoreCtx& c, const SubBatch& sb, CoreOut* out) {
    Workspace* w = c.w;
    cudaStream_t stream = c.stream;
    const int64_t n = sb.n, b = sb.begin;
    MatchParams p = core_params(c, sb);
    // tier 0's 16-byte sector stores: every inline run and spill block starts on a 32-byte boundary
    if ((reinterpret_cast<uintptr_t>(p.ranges) % (RANGE_SECTOR * sizeof(uint2))) != 0 || p.dyn_base % RANGE_SECTOR != 0)
        return fail(BFQ_E_STATE, "internal error: tier-0 range region not sector-aligned");
    if (c.s->l2_window_bytes > 0) {
        cudaStreamAttrValue attr{};
        attr.accessPolicyWindow.base_ptr = c.s->d_tags.p;
        attr.accessPolicyWindow.num_bytes = c.s->l2_window_bytes;
        attr.accessPolicyWindow.hitRatio = 1.0f;
        attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cudaStreamSetAttribute(stream, cudaStreamAttributeAccessPolicyWindow, &attr);
        cudaGetLastError();
    }
    BFQ_CUDA_TRY(cudaMemsetAsync(p.counters, 0, CTR_COUNT * sizeof(unsigned long long), stream));
    bool ordered = false;
    if (wants_order(c, sb)) {
        // group the topics by tenant and leading levels so that neighbouring lanes walk the same part of the trie, and
        // match every distinct (tenant, topic) pair once
        const int slot = sb.chunk & 1;
        OrderParams q{};
        q.n_topics = n;
        q.topics = c.d_topics;
        q.topic_off = p.topic_off;
        q.topic_tenant = p.topic_tenant;
        q.n_tenants = c.n_tenants;
        q.keys = w->d_ord_keys.p + b;
        q.leader = w->d_leader.p + b;
        q.order = w->d_order.p + b;
        q.hash_tab = w->d_hash_tab.p + (size_t) slot * w->hash_stride;
        q.hash_mask = order_hash_entries(n) - 1;
        q.hist = w->d_hist.p + (size_t) slot * w->hist_stride;
        q.dedup = c.h->dedup ? 1 : 0;
        q.dedup_hash_mask = c.h->dedup_hash_bits >= 64 ? ~0ull : (1ull << c.h->dedup_hash_bits) - 1;
        q.counters = p.counters;
        BFQ_CUDA_TRY(launch_order(q, stream));
        p.order = q.order;
        p.order_count = p.counters + CTR_NLEAD;
        p.pos_rec = w->d_pos_rec.p + b;
        out->n_launches += 3;
        ordered = true;
    }
    if (n > 0) {
        // tier 0 (one lane per topic), then tier 1 (one warp per topic) over whatever tier 0 deferred — its count is read
        // on the device, so both launches go out back to back
        if (sb.chunk == 0) BFQ_CUDA_TRY(cudaEventRecord(w->evk[0], stream));
        launch_match_lanes(p, stream);
        if (sb.chunk == 0) BFQ_CUDA_TRY(cudaEventRecord(w->evk[1], stream));
        p.work_list = p.defer_list;
        p.n_work = -1;
        launch_match(p, false, 0, stream);
        out->n_launches += 2;
        if (ordered) {
            // tier 0 wrote span records by position: gather them to topic order (behind tier 1, whose spans repeats copy)
            FinalizeParams f{};
            f.n_topics = n;
            f.leader = w->d_leader.p + b;
            f.pos = w->d_ord_keys.p + b;
            f.pos_rec = p.pos_rec;
            f.span_begin = p.span_begin;
            f.span_count = p.span_count;
            f.route_count = p.route_count;
            f.flagged_list = p.flagged_list;
            f.counters = p.counters;
            f.second_pass = 0;
            launch_finalize(f, stream);
            out->n_launches += 1;
        }
        if (w->any_cap) {
            CapsParams q = caps_params(c, sb, p);
            q.n_flagged = -1;
            launch_caps(q, stream);
            out->n_launches += 2;
        }
    }
    BFQ_CUDA_TRY(cudaGetLastError());
    return BFQ_OK;
}

int32_t copy_counters(const CoreCtx& c, const SubBatch& sb) {
    BFQ_CUDA_TRY(cudaMemcpyAsync(c.w->h_counters.p + (size_t) sb.chunk * CTR_COUNT, c.w->d_counters.p + (size_t) sb.chunk * CTR_COUNT,
                             CTR_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c.stream));
    return BFQ_OK;
}

// Waits for the sub-batch and handles what the optimistic enqueue could not: topics that need tier 2 (frontier / range
// overflow of tier 1: scratch sized from the index statistics, then the followers and caps passes once more for what
// tier 2 added) and slices that turned out too small (BFQ_RETRY_GROW). *reran = tier 2 changed the spans.
int32_t finish_core(const CoreCtx& c, const SubBatch& sb, CoreOut* out, bool* reran, cudaEvent_t done = nullptr) {
    Workspace* w = c.w;
    cudaStream_t stream = c.stream;
    unsigned long long* hc = w->h_counters.p + (size_t) sb.chunk * CTR_COUNT;
    if (reran) *reran = false;
    // the device path waits for ITS match only (an event behind it): later matches may already be queued on the same stream
    if (done) BFQ_CUDA_TRY(cudaEventSynchronize(done));
    else BFQ_CUDA_TRY(cudaStreamSynchronize(stream));
    out->n_overflow += (int64_t) hc[CTR_OVERFLOW];
    out->n_deferred += (int64_t) hc[CTR_DEFER];
    if (hc[CTR_OVERFLOW] > 0) {
        MatchParams p = core_params(c, sb);
        const uint64_t capF = (uint64_t) c.s->flat.max_nodes_per_depth + 2;
        const uint64_t capR = 2 * ((uint64_t) c.s->flat.max_tenant_nodes + 2) + 2;
        const uint64_t per_warp = 4 * capF + capR;   // uint2 units: two frontier buffers of uint4 entries + ranges
        uint64_t warps = std::min<uint64_t>(hc[CTR_OVERFLOW], std::max<uint64_t>(8, (1ull << 31) / (per_warp * sizeof(uint2))));
        warps = std::min<uint64_t>(warps, (uint64_t) device_sm_count() * 8);
        warps = (warps + 7) / 8 * 8;
        if (w->d_scratch.cap < (size_t) (warps * per_warp)) {
            BFQ_CUDA_TRY(cudaDeviceSynchronize());   // the other compute stream of this workspace may be in tier 2 on the old scratch
            BFQ_CUDA_TRY(w->d_scratch.reserve((size_t) (warps * per_warp)));
        }
        p.scratch = w->d_scratch.p;
        p.scratch_frontier_cap = capF;
        p.scratch_ranges_cap = capR;
        p.work_list = p.overflow_list;
        p.n_work = (int64_t) hc[CTR_OVERFLOW];
        launch_match(p, true, (int) warps, stream);
        out->n_launches++;
        if (w->hist_stride > 0 && c.h->dedup && wants_order(c, sb)) {
            FinalizeParams f{};
            f.n_topics = sb.n;
            f.leader = w->d_leader.p + sb.begin;
            f.span_begin = p.span_begin;
            f.span_count = p.span_count;
            f.route_count = p.route_count;
            f.flagged_list = p.flagged_list;
            f.counters = p.counters;
            f.second_pass = 1;
            launch_finalize(f, stream);
            out->n_launches++;
        }
        if (w->any_cap) {
            CapsParams q = caps_params(c, sb, p);
            q.n_flagged = -1;
            launch_caps(q, stream);
            out->n_launches += 2;
        }
        BFQ_CUDA_TRY(cudaGetLastError());
        int32_t rc = copy_counters(c, sb);
        if (rc != BFQ_OK) return rc;
        BFQ_CUDA_TRY(cudaStreamSynchronize(stream));
        if (hc[CTR_ERROR] != 0) return fail(BFQ_E_STATE, "tier-2 scratch exhausted (index statistics inconsistent)");
        if (reran) *reran = true;
    }
    if (hc[CTR_RANGES] > sb.dyn_cap) {
        out->want_dyn = std::max<uint64_t>(out->want_dyn, hc[CTR_RANGES]);
        return BFQ_RETRY_GROW;
    }
    if (hc[CTR_THROTTLED] > sb.thr_cap) {
        out->want_thr = std::max<uint64_t>(out->want_thr, hc[CTR_THROTTLED]);
        return BFQ_RETRY_GROW;
    }
    out->n_ranges += (int64_t) hc[CTR_RANGES];
    out->n_flagged += (int64_t) hc[CTR_FLAGGED];
    out->n_leaders += wants_order(c, sb) ? (int64_t) hc[CTR_NLEAD] : sb.n;
    out->chunk_throttled[sb.chunk] = (int64_t) hc[CTR_THROTTLED];
    out->n_throttled += (int64_t) hc[CTR_THROTTLED];
    return BFQ_OK;
}

void add_stats(bfq_index* h, const CoreOut& co, int64_t n, double kernel_ms) {
    std::lock_guard<std::mutex> g(h->mu);
    h->launches += co.n_launches;
    h->overflow_topics += co.n_overflow;
    h->deferred_topics += co.n_deferred;
    h->flagged_topics += co.n_flagged;
    h->duplicate_topics += n - co.n_leaders;
    if (kernel_ms >= 0) h->last_kernel_ms = kernel_ms;
}

void count_retry(bfq_index* h) {
    std::lock_guard<std::mutex> g(h->mu);
    h->buffer_retries++;
}

// grows the buffers a retry asked for (the caller has synchronised the device)
int32_t grow_for_retry(Workspace* w, const CoreOut& co, int64_t n, int C) {
    if (co.want_dyn) {
        const size_t want = (size_t) ((uint64_t) n * INLINE_RANGES + (co.want_dyn + co.want_dyn / 4 + 1024) * (uint64_t) C);
        if (want >= 0xFFFFFFF0ull) return fail(BFQ_E_RANGE, "more than 2^32 matched ranges in one batch; split the batch");
        BFQ_CUDA_TRY(w->d_ranges.reserve(want));
    }
    if (co.want_thr) BFQ_CUDA_TRY(w->d_throttled.reserve((size_t) ((co.want_thr + co.want_thr / 4 + 1024) * (uint64_t) C)));
    return BFQ_OK;
}

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

void fill_device_result(const DeviceLease* L, bfq_device_result* out) {
    Workspace* w = L->ws;
    out->d_span_begin = w->d_span_begin.p;
    out->d_span_count = w->d_span_count.p;
    out->d_route_count = w->d_route_count.p;
    out->d_ranges = reinterpret_cast<const bfq_range*>(w->d_ranges.p);
    out->d_throttled = reinterpret_cast<const bfq_throttled*>(w->d_throttled.p);
    out->n_ranges = (int64_t) ((uint64_t) L->n * INLINE_RANGES) + L->co.n_ranges;   // extent of the sparse range array
    out->n_throttled = L->co.n_throttled;
    out->n_routes = -1;
    out->n_overflow_topics = L->co.n_overflow;
    out->n_flagged_topics = L->co.n_flagged;
    out->n_launches = L->co.n_launches;
    out->n_topics = L->n;
    out->n_distinct_topics = L->co.n_leaders;
    out->tier0_ms = L->tier0_ms;
    out->generation = L->snap->generation;
}

int32_t device_enqueue(DeviceLease* L) {
    int32_t rc = prepare_workspace(L->h, L->ws, L->n, 1, L->ctx.n_tenants);
    if (rc != BFQ_OK) return rc;
    L->co = CoreOut();
    const SubBatch sb = whole_batch(L->ws, L->n);
    rc = enqueue_core(L->ctx, sb, &L->co);
    if (rc != BFQ_OK) return rc;
    rc = copy_counters(L->ctx, sb);
    if (rc != BFQ_OK) return rc;
    BFQ_CUDA_TRY(cudaEventRecord(L->ws->ev_done, L->ctx.stream));
    return BFQ_OK;
}

int32_t device_wait(DeviceLease* L) {
    if (L->done) return L->rc;
    L->done = true;
    for (int attempt = 0;; attempt++) {
        if (attempt == 8) return L->rc = fail(BFQ_E_STATE, "buffer sizing did not converge");
        int32_t rc = finish_core(L->ctx, whole_batch(L->ws, L->n), &L->co, nullptr, L->ws->ev_done);
        if (rc == BFQ_OK) break;
        if (rc != BFQ_RETRY_GROW) return L->rc = rc;
        count_retry(L->h);
        if (cudaDeviceSynchronize() != cudaSuccess) return L->rc = fail(BFQ_E_CUDA, "cudaDeviceSynchronize");
        rc = grow_for_retry(L->ws, L->co, L->n, 1);
        if (rc == BFQ_OK) rc = device_enqueue(L);
        if (rc != BFQ_OK) return L->rc = rc;
    }
    if (L->n > 0) {
        float kms = 0;
        cudaEventElapsedTime(&kms, L->ws->evk[0], L->ws->evk[1]);
        L->tier0_ms = kms;
    }
    add_stats(L->h, L->co, L->n, L->n > 0 ? L->tier0_ms : -1.0);
    return L->rc = BFQ_OK;
}

int64_t emit_bytes(const std::string& s, uint8_t* out, int64_t cap) {
    if (out && (int64_t) s.size() <= cap) memcpy(out, s.data(), s.size());
    return (int64_t) s.size();
}

}  // namespace

extern "C" {

int32_t bfq_index_create(int32_t device_ordinal, bfq_index** out) {
    if (!out) return fail(BFQ_E_INVALID, "out is NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(BFQ_E_CUDA, std::string("no usable CUDA device (there is no CPU fallback): ") + cudaGetErrorString(e));
    if (device_ordinal < 0 || device_ordinal >= count) return fail(BFQ_E_INVALID, "device ordinal out of range");
    BFQ_CUDA_TRY(cudaSetDevice(device_ordinal));
    auto* h = new bfq_index();
    h->device = device_ordinal;
    h->pool->device = device_ordinal;
    if (const char* eo = getenv("BFQ_ORDER")) {   // experiment switch: 0 = never order, N > 0 = order batches of >= N topics
        const long long v = atoll(eo);
        h->order_min = v <= 0 ? (int64_t) 1 << 62 : (int64_t) v;
    }
    if (const char* ed = getenv("BFQ_DEDUP")) h->dedup = atoi(ed) != 0;   // experiment switch
    *out = h;
    return BFQ_OK;
}

void bfq_index_destroy(bfq_index* h) { delete h; }

int32_t bfq_index_reset(bfq_index* h) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    std::lock_guard<std::mutex> g(h->stage_mu);
    h->staging.reset();
    return BFQ_OK;
}

int32_t bfq_index_load(bfq_index* h, const uint8_t* keys, const int64_t* key_off, const uint8_t* vals,
                       const int64_t* val_off, int64_t n) {
    if (!h || n < 0 || (n > 0 && (!keys || !key_off || !vals || !val_off))) return fail(BFQ_E_INVALID, "bad argument");
    std::lock_guard<std::mutex> g(h->stage_mu);
    if (n > 0 && h->staging.has_delta())
        return fail(BFQ_E_STATE, "bfq_index_load after bfq_index_apply: commit (or reset) the staged delta first");
    std::string err;
    if (!h->staging.load(keys, key_off, vals, val_off, n, &err)) return fail(BFQ_E_INVALID, err);
    return BFQ_OK;
}

int32_t bfq_index_apply(bfq_index* h, const uint8_t* add_keys, const int64_t* add_key_off, const uint8_t* add_vals,
                        const int64_t* add_val_off, int64_t n_add, const uint8_t* del_keys, const int64_t* del_key_off,
                        int64_t n_del) {
    if (!h || n_add < 0 || n_del < 0) return fail(BFQ_E_INVALID, "bad argument");
    if (n_add > 0 && (!add_keys || !add_key_off || !add_vals || !add_val_off)) return fail(BFQ_E_INVALID, "NULL add set");
    if (n_del > 0 && (!del_keys || !del_key_off)) return fail(BFQ_E_INVALID, "NULL delete set");
    // all or nothing: every add key is decoded before the staging area is touched
    for (int64_t i = 0; i < n_add; i++) {
        if (add_key_off[i + 1] < add_key_off[i] || add_val_off[i + 1] < add_val_off[i]) return fail(BFQ_E_INVALID, "offsets not ascending");
        DecodedKey d;
        if (!decode_route_key(sv((const char*) add_keys + add_key_off[i], (size_t) (add_key_off[i + 1] - add_key_off[i])), &d))
            return fail(BFQ_E_INVALID, "undecodable route key in add set (nothing was staged)");
    }
    for (int64_t i = 0; i < n_del; i++) {
        if (del_key_off[i + 1] < del_key_off[i]) return fail(BFQ_E_INVALID, "offsets not ascending");
        if (tenant_prefix_of(sv((const char*) del_keys + del_key_off[i], (size_t) (del_key_off[i + 1] - del_key_off[i]))).empty())
            return fail(BFQ_E_INVALID, "undecodable route key in delete set (nothing was staged)");
    }
    std::lock_guard<std::mutex> g(h->stage_mu);
    for (int64_t i = 0; i < n_add; i++)
        h->staging.upsert(sv((const char*) add_keys + add_key_off[i], (size_t) (add_key_off[i + 1] - add_key_off[i])),
                          sv((const char*) add_vals + add_val_off[i], (size_t) (add_val_off[i + 1] - add_val_off[i])));
    for (int64_t i = 0; i < n_del; i++)
        h->staging.erase(sv((const char*) del_keys + del_key_off[i], (size_t) (del_key_off[i + 1] - del_key_off[i])));
    return BFQ_OK;
}

namespace {

void set_l2_window(bfq_index* h, Snapshot* sn) {
    // Keep the tag array of the (rare) global tag table resident in L2 (persisting access window). BFQ_L2PERSIST=0 disables.
    const char* e = getenv("BFQ_L2PERSIST");
    if (e && atoi(e) == 0) return;
    int max_persist = 0, max_window = 0;
    cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, h->device);
    cudaDeviceGetAttribute(&max_window, cudaDevAttrMaxAccessPolicyWindowSize, h->device);
    size_t want = std::min<size_t>(sn->d_tags.bytes(), std::min<size_t>((size_t) max_persist, (size_t) max_window));
    if (want > 0 && cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) sn->l2_window_bytes = want;
    cudaGetLastError();
}

void publish(bfq_index* h, std::shared_ptr<Snapshot> sn) {
    std::shared_ptr<Snapshot> old;
    {
        std::lock_guard<std::mutex> g(h->mu);
        sn->generation = h->next_generation++;
        old = std::move(h->snap);
        h->snap = std::move(sn);
    }
    old.reset();   // freed here unless a match or a result still pins it
}

// every tenant rebuilt on all host cores, everything uploaded: bfq_index_load, the first commit, and whenever the delta
// path cannot be used
int32_t commit_full(bfq_index* h) {
    const bool trace = getenv("BFQ_COMMIT_TRACE") != nullptr;
    auto t_prev = std::chrono::steady_clock::now();
    auto lap = [&](const char* what) {
        if (!trace) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[bfq full commit] %-38s %9.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
        t_prev = now;
    };
    h->staging.merge_all();
    lap("merge staged deltas");
    std::vector<const KVBlob*> parts;   // the staged per-tenant blobs themselves: no concatenated copy of the KV
    for (auto& kvp : h->staging.tenants()) parts.push_back(kvp.second.base.get());
    auto sn = std::make_shared<Snapshot>();
    sn->device = h->device;
    FlatIndex& flat = sn->flat;
    std::string err;
    if (!build_flat_index_parts(parts, &flat, &err)) return fail(BFQ_E_INVALID, err);
    lap("build (host, all cores)");
    BFQ_CUDA_TRY(sn->d_slots.reserve(flat.slots.size()));
    BFQ_CUDA_TRY(sn->d_tags.reserve(flat.tags.size()));
    BFQ_CUDA_TRY(sn->d_roots.reserve(std::max<size_t>(flat.roots.size(), 1)));
    BFQ_CUDA_TRY(sn->d_segs.reserve(flat.segs.size()));
    BFQ_CUDA_TRY(sn->d_rkind.reserve(std::max<size_t>(flat.rkind.size(), 1)));
    BFQ_CUDA_TRY(sn->d_pfxP.reserve(flat.pfx_persistent.size()));
    BFQ_CUDA_TRY(sn->d_pfxG.reserve(flat.pfx_group.size()));
    // (one pageable cudaMemcpy: a threaded upload through per-thread pinned bounce buffers pays more for the pinned
    // allocations than the driver's own staging loses)
    BFQ_CUDA_TRY(cudaMemcpy(sn->d_slots.p, flat.slots.data(), flat.slots.size() * sizeof(Slot), cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(sn->d_tags.p, flat.tags.data(), flat.tags.size(), cudaMemcpyHostToDevice));
    if (!flat.roots.empty())
        BFQ_CUDA_TRY(cudaMemcpy(sn->d_roots.p, flat.roots.data(), flat.roots.size() * sizeof(Slot), cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(sn->d_segs.p, flat.segs.data(), flat.segs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    if (!flat.rkind.empty())
        BFQ_CUDA_TRY(cudaMemcpy(sn->d_rkind.p, flat.rkind.data(), flat.rkind.size(), cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(sn->d_pfxP.p, flat.pfx_persistent.data(), flat.pfx_persistent.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(sn->d_pfxG.p, flat.pfx_group.data(), flat.pfx_group.size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
    lap("device allocations + upload");
    // per-tenant host side: the staged blobs are shared (no second copy of the KV), the route kinds are sliced
    sn->th.resize(flat.tenants.size());
    {
        size_t i = 0;
        for (auto& kvp : h->staging.tenants()) {
            if (i >= flat.tenants.size() || kvp.second.base->n() != flat.tenants[i].n_routes)
                return fail(BFQ_E_STATE, "internal error: staged tenants and built tenants disagree");
            sn->th[i].kv = kvp.second.base;
            sn->th[i].rkind = std::make_shared<const std::vector<uint8_t>>(flat.rkind.begin() + flat.tenants[i].lo,
                                                                            flat.rkind.begin() + flat.tenants[i].lo + flat.tenants[i].n_routes);
            i++;
        }
        if (i != flat.tenants.size()) return fail(BFQ_E_STATE, "internal error: staged tenants and built tenants disagree");
    }
    // the host keeps only what it needs after the upload (the tag bytes too, about 2 B per wide edge: delta commits place
    // rebuilt tenants' wide edges into a copy of them); the rest is handed to the janitor thread
    {
        struct Garbage {
            SlotVec slots;
            std::vector<uint8_t> rkind;
            std::vector<Slot> roots;
            std::vector<uint32_t> pfxP, pfxG;
        };
        auto* g = new Garbage();
        g->slots = std::move(flat.slots);
        g->rkind = std::move(flat.rkind);
        g->roots = std::move(flat.roots);
        g->pfxP = std::move(flat.pfx_persistent);
        g->pfxG = std::move(flat.pfx_group);
        flat.slots = SlotVec();
        flat.rkind = std::vector<uint8_t>();
        flat.roots = std::vector<Slot>();
        flat.pfx_persistent = std::vector<uint32_t>();
        flat.pfx_group = std::vector<uint32_t>();
        if (h->janitor.joinable()) h->janitor.join();
        h->janitor = std::thread([g]() { delete g; });
    }
    lap("host bookkeeping (image released in the background)");
    set_l2_window(h, sn.get());
    h->staging.clear_bulk_changed();
    publish(h, std::move(sn));
    lap("publish (drops the old snapshot)");
    return BFQ_OK;
}

constexpr int32_t BFQ_NEED_FULL = -101;   // internal: the delta path does not apply, do a full build

// walks one tenant's slice of the segment table (a sequence of {n_segments, total, (first, count) x n_segments}) and moves
// the ranks in it by `d`
void shift_seg_slice(std::vector<uint32_t>& segs, uint64_t base, uint64_t words, int64_t d) {
    uint64_t w = base;
    while (w + 2 <= base + words) {
        const uint32_t nseg = segs[w];
        for (uint32_t k = 0; k < nseg && w + 2 + 2 * k + 1 < base + words + 1; k++) segs[w + 2 + 2 * k] = (uint32_t) ((int64_t) segs[w + 2 + 2 * k] + d);
        w += 2 + 2 * (uint64_t) nseg;
    }
}

// The delta path (SURVEY.md 8f rank 1; DW/DistWorkerCoProc.java:304-513 applies one batch of SUBs / UNSUBs, of any number of
// tenants, per mutation): only the touched tenants are merged, rebuilt and uploaded. The new snapshot is a device-side copy of
// the previous one (a few milliseconds for gigabytes at HBM speed; the previous snapshot stays untouched for the matches and
// results that pin it) in which
//   * every rebuilt tenant gets a fresh slot region appended behind the existing ones (its old region becomes garbage until
//     the next full build) and a patched root record;
//   * ranks stay dense positions in KV order, so the tenants behind a tenant that grew or shrank have the ranks in their
//     records moved by the difference (one streaming kernel over their regions) and their per-rank arrays copied to the
//     shifted position.
// The host work runs on all cores, so k touched tenants cost about what the largest of them costs plus k times a small
// fixed amount: the tenants are merged in parallel, built in parallel (build_tenant_image: trie, plans, sizes; largest
// first), given their bases in key order by prefix sums, and placed (place_tenant_image) in parallel into one staging
// buffer. The device work is a fixed number of copies and launches whatever k is: one upload of the rebuilt regions (they
// sit back to back at [old n_slots, new n_slots)), one upload of their per-rank arrays packed with a run table, and one
// kernel that assembles the new per-rank arrays from the old ones and the packed ones (assemble_rank_arrays_kernel).
// The shared tag table (the children of wide nodes) is patched in place of being rebuilt. A tag-table slot IS the child's
// record and its id is the child's node id, which its own children carry as their parent key; so a tenant's wide edges are
// placed on the host, into a copy of the snapshot's tag bytes, while the tenant's records are emitted (knowing every node
// id). In this order:
//   1. the tag slots of every replaced or removed tenant are freed (EdgeTable::release): a rebuilt tenant keeps its ordinal,
//      so its root-level edges come back with the same keys, and a stale entry must not be found before the new one;
//   2. the rebuilt tenants with wide edges are placed one after another in key order (the full build's EdgeTable::claim
//      probe order); tenants without wide edges touch no shared state and are placed in parallel before them;
//   3. on the device, their tag-table records are scattered to their slots;
//   4. the records of the untouched tenants whose ranks moved are shifted: their regions, and their listed tag slots;
//   5. the new tag bytes are uploaded and the snapshot is published.
// The tag table cannot grow without a full build (home_block depends on n_blocks), and freed slots leave their blocks'
// overflow bytes set (only a full build clears them); so the commit is a full build instead when, after it,
//   * more than 3/4 of the table's usable slots would be claimed, or
//   * more than 1/4 of its blocks would have their overflow byte set (longer probes for every lookup that lands there).
// The kernels see exactly the layout a full build would have produced, up to the placement of the regions and tag slots.
// *built is set to the number of tenants rebuilt.
int32_t commit_delta(bfq_index* h, const std::shared_ptr<Snapshot>& old, const std::vector<std::string>& dirty, int64_t* built) {
    const FlatIndex& of = old->flat;
    const bool trace = getenv("BFQ_COMMIT_TRACE") != nullptr;
    auto t_prev = std::chrono::steady_clock::now();
    auto lap = [&](const char* what) {
        if (!trace) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[bfq delta commit] %-34s %9.3f ms\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
        t_prev = now;
    };
    if (old->garbage_slots > (uint64_t) of.n_slots / 4 + 4096) return BFQ_NEED_FULL;   // reclaim the replaced regions
    // ---- merge the touched tenants' KV (copy-on-write: the old blobs stay with the old snapshot)
    h->staging.merge_tenants(dirty);
    struct Plan {
        std::string prefix;            // key prefix
        int old_index = -1;            // position in of.tenants, or -1 for a new tenant
        std::shared_ptr<const KVBlob> kv;   // null: the tenant is gone
        uint32_t ordinal = 0;
        int64_t pack_lo = 0;           // its first rank in the packed upload of the rebuilt tenants' per-rank arrays
        TenantImage img;
    };
    std::vector<Plan> plans;
    std::unordered_map<std::string, int> old_pos;   // tenant id -> index in of.tenants
    for (size_t i = 0; i < of.tenants.size(); i++) old_pos.emplace(of.tenants[i].tenant, (int) i);
    for (auto& p : dirty) {
        Plan pl;
        pl.prefix = p;
        const std::string id = p.substr(3);
        auto it = old_pos.find(id);
        pl.old_index = it == old_pos.end() ? -1 : it->second;
        auto st = h->staging.tenants().find(p);
        if (st != h->staging.tenants().end()) pl.kv = st->second.base;
        if (pl.old_index < 0 && !pl.kv) continue;   // created and deleted between two commits
        plans.push_back(std::move(pl));
    }
    if (plans.empty()) return BFQ_OK;   // nothing changed
    for (auto& pl : plans) *built += pl.kv ? 1 : 0;
    lap("merge touched tenants' KV");
    // ---- the tag table: a copy of the snapshot's tag bytes (the snapshot's own stay as they are if this commit fails), with
    // the slots of the replaced and removed tenants freed
    EdgeTable table;
    table.tags = of.tags;
    table.n_blocks = of.n_blocks;
    table.overflowed_blocks = of.overflowed_blocks;
    uint64_t tag_live = of.n_big_edges;
    const uint64_t tag_max = (uint64_t) of.n_blocks * BLOCK_USABLE * 3 / 4;
    if (table.tags.size() != (size_t) of.n_blocks * 16) return BFQ_NEED_FULL;
    for (auto& pl : plans) {
        if (pl.old_index < 0) continue;
        const TenantMeta& om = of.tenants[(size_t) pl.old_index];
        for (uint32_t s : om.tag_slots) table.release(s);
        tag_live -= om.big_edges;
    }
    // ---- the new tenant list in key order: old tenants (untouched or replaced) merged with the new ones
    struct Entry {
        int old_index;   // -1: new tenant
        int plan;        // -1: untouched
    };
    std::vector<Entry> entries;
    {
        std::vector<int> plan_of_old(of.tenants.size(), -1);
        std::vector<std::pair<std::string, int>> fresh;   // (prefix, plan) of new tenants, in key order (dirty is in key order)
        for (size_t k = 0; k < plans.size(); k++) {
            if (plans[k].old_index >= 0) plan_of_old[(size_t) plans[k].old_index] = (int) k;
            else fresh.emplace_back(plans[k].prefix, (int) k);
        }
        size_t f = 0;
        auto prefix_of_old = [&](size_t i) { return make_tenant_begin_key(of.tenants[i].tenant); };
        for (size_t i = 0; i <= of.tenants.size(); i++) {
            const std::string bound = i < of.tenants.size() ? prefix_of_old(i) : std::string();
            while (f < fresh.size() && (i == of.tenants.size() || fresh[f].first < bound)) entries.push_back({-1, fresh[f++].second});
            if (i == of.tenants.size()) break;
            const int pk = plan_of_old[i];
            if (pk >= 0 && !plans[(size_t) pk].kv) continue;   // tenant removed
            entries.push_back({(int) i, pk});
        }
    }
    auto sn = std::make_shared<Snapshot>();
    sn->device = h->device;
    FlatIndex& nf = sn->flat;
    nf.tenant_ordinal = of.tenant_ordinal;
    nf.host_roots = of.host_roots;
    nf.segs = of.segs;
    nf.n_blocks = of.n_blocks;
    nf.max_nodes_per_depth = of.max_nodes_per_depth;
    nf.max_tenant_nodes = of.max_tenant_nodes;
    for (int k = 0; k < 5; k++) nf.child_hist[k] = of.child_hist[k];
    // ---- ordinals and ranks (a tenant's ranks depend only on the sizes of the tenants before it), then the build step of
    // every rebuilt tenant on all host cores, largest first
    std::vector<uint32_t> by_size;
    {
        int64_t rank = 0;
        for (auto& e : entries) {
            if (e.plan < 0) {
                rank += of.tenants[(size_t) e.old_index].n_routes;
                continue;
            }
            Plan& pl = plans[(size_t) e.plan];
            if (pl.old_index >= 0) {
                pl.ordinal = of.tenants[(size_t) pl.old_index].ordinal;
            } else {
                pl.ordinal = (uint32_t) nf.host_roots.size();
                nf.host_roots.emplace_back();
                nf.tenant_ordinal[pl.prefix.substr(3)] = pl.ordinal;
            }
            pl.img.meta.lo = rank;
            rank += pl.kv->n();
            by_size.push_back((uint32_t) e.plan);
        }
        if (rank >= (int64_t) 0x7FFFFFFF) return BFQ_NEED_FULL;
    }
    std::sort(by_size.begin(), by_size.end(), [&](uint32_t a, uint32_t b) { return plans[a].kv->n() > plans[b].kv->n(); });
    std::vector<std::string> errs(plans.size());
    parallel_for_each(by_size, [&](uint32_t k) {
        Plan& pl = plans[k];
        const std::string id = pl.prefix.substr(3);
        build_tenant_image(*pl.kv, sv(id), pl.ordinal, pl.img.meta.lo, &pl.img, &errs[k]);
    });
    for (auto& e : errs)
        if (!e.empty()) return fail(BFQ_E_INVALID, e);
    lap("build touched tenants (host, all cores)");
    // the tag-table fill bound: placing the wide tenants one by one fails at the first that passes 3/4, i.e. exactly when
    // their wide edges together pass it
    {
        uint64_t added = 0;
        for (uint32_t k : by_size) added += plans[k].img.meta.big_edges;
        if (added > 0 && tag_live + added > tag_max) return BFQ_NEED_FULL;
    }
    // ---- bases in key order: dense ranks, appended slot regions / segment slices, running prefix-count bases; the runs of the
    // per-rank arrays (untouched tenants: from the old snapshot, shifted; rebuilt ones: from the packed upload)
    uint64_t slot_cursor = of.n_slots, seg_cursor = of.segs.size();
    int64_t rank = 0, pack_n = 0;
    uint32_t ppb = 0, pgb = 0;
    nf.tenants.reserve(entries.size());
    std::vector<RankRun> runs;
    auto add_run = [&](int64_t new_lo, int64_t len, int64_t src_lo, uint32_t packed, uint32_t dP, uint32_t dG) {
        if (len <= 0) return;
        if (!runs.empty()) {
            RankRun& r = runs.back();
            if (r.packed == packed && (int64_t) r.src_lo + r.len == src_lo && r.dP == dP && r.dG == dG) {
                r.len += (uint32_t) len;
                return;
            }
        }
        runs.push_back(RankRun{(uint32_t) new_lo, (uint32_t) len, (uint32_t) src_lo, packed, dP, dG});
    };
    for (auto& e : entries) {
        if (e.plan < 0) {   // untouched: same region, ranks moved by the growth of the tenants before it
            TenantMeta m = of.tenants[(size_t) e.old_index];
            add_run(rank, m.n_routes, m.lo, 0, ppb - m.pp_base, pgb - m.pg_base);
            m.lo = rank;
            m.pp_base = ppb;
            m.pg_base = pgb;
            rank += m.n_routes;
            ppb += m.pp;
            pgb += m.pg;
            nf.tenants.push_back(std::move(m));
            continue;
        }
        Plan& pl = plans[(size_t) e.plan];
        TenantMeta& m = pl.img.meta;
        m.region_base = slot_cursor;
        m.seg_base = seg_cursor;
        m.pp_base = ppb;
        m.pg_base = pgb;
        pl.pack_lo = pack_n;
        add_run(rank, m.n_routes, pack_n, 1, 0, 0);
        slot_cursor += m.csr_slots;
        seg_cursor += m.seg_words;
        rank += m.n_routes;
        pack_n += m.n_routes;
        ppb += m.pp;
        pgb += m.pg;
        nf.tenants.emplace_back();   // its placed meta, below
    }
    if (slot_cursor >= 0x7FFFFFF0ull) return BFQ_NEED_FULL;
    // ---- the place step, into two staging buffers uploaded with one copy each: the rebuilt regions back to back (uninitialised;
    // first touched by the placing threads), and [rkind | pfxP | pfxG | runs] of the rebuilt tenants. (Pageable: pinning
    // gigabytes when a commit rebuilds most tenants costs more than the driver's staged copy.)
    const uint64_t up_slots = slot_cursor - of.n_slots;
    SlotVec regions_up((size_t) up_slots);
    const size_t off_pfxP = ((size_t) pack_n + 15) & ~(size_t) 15, off_pfxG = off_pfxP + (size_t) pack_n * 4;
    const size_t off_runs = (off_pfxG + (size_t) pack_n * 4 + 15) & ~(size_t) 15, pack_bytes = off_runs + runs.size() * sizeof(RankRun);
    std::vector<uint8_t> pack(pack_bytes);
    memcpy(pack.data() + off_runs, runs.data(), runs.size() * sizeof(RankRun));
    lap("staging allocation");
    auto place = [&](uint32_t k, EdgeTable* tags, uint64_t tag_room) {
        Plan& pl = plans[k];
        TenantImage& img = pl.img;
        const TenantMeta& m = img.meta;
        if (!place_tenant_image(&img, m.region_base, m.seg_base, m.pp_base, m.pg_base, tags, tag_room,
                                regions_up.data() + (m.region_base - of.n_slots), &errs[k]))
            return;
        const size_t n = (size_t) m.n_routes, at = (size_t) pl.pack_lo;
        memcpy(pack.data() + at, img.rkind.data(), n);
        memcpy(pack.data() + off_pfxP + at * 4, img.pfxP.data(), n * 4);
        memcpy(pack.data() + off_pfxG + at * 4, img.pfxG.data(), n * 4);
    };
    std::vector<uint32_t> narrow;
    for (uint32_t k : by_size)
        if (plans[k].img.meta.big_edges == 0) narrow.push_back(k);
    parallel_for_each(narrow, [&](uint32_t k) { place(k, nullptr, 0); });
    for (auto& e : entries) {   // the wide ones: one after another in key order, into the copy of the tag bytes
        if (e.plan < 0 || plans[(size_t) e.plan].img.meta.big_edges == 0) continue;
        place((uint32_t) e.plan, &table, tag_max > tag_live ? tag_max - tag_live : 0);
        if (!errs[(size_t) e.plan].empty()) break;
        if (!plans[(size_t) e.plan].img.placed) return BFQ_NEED_FULL;   // its wide edges would fill the tag table past 3/4
        tag_live += plans[(size_t) e.plan].img.meta.big_edges;
    }
    for (auto& e : errs)
        if (!e.empty()) return fail(BFQ_E_INVALID, e);
    if ((uint64_t) table.overflowed_blocks * 4 > (uint64_t) table.n_blocks) return BFQ_NEED_FULL;   // probes got too long
    lap("place touched tenants (host, all cores)");
    sn->th.reserve(entries.size());
    // the old snapshot's per-tenant fan-out tables may be filled in by a concurrent bfq_fanout_device: copy them under its lock
    std::vector<Snapshot::TenantHost> old_th;
    {
        std::lock_guard<std::mutex> gf(old->fan_mu);
        old_th = old->th;
    }
    for (size_t i = 0; i < entries.size(); i++) {
        const Entry& e = entries[i];
        if (e.plan < 0) {
            sn->th.push_back(old_th[(size_t) e.old_index]);
            continue;
        }
        Plan& pl = plans[(size_t) e.plan];
        nf.host_roots[pl.ordinal] = pl.img.root;
        nf.segs.insert(nf.segs.end(), pl.img.segs.begin(), pl.img.segs.end());
        nf.max_nodes_per_depth = std::max(nf.max_nodes_per_depth, pl.img.meta.max_depth_nodes);
        nf.max_tenant_nodes = std::max(nf.max_tenant_nodes, pl.img.meta.walk_nodes);
        nf.tenants[i] = pl.img.meta;
        Snapshot::TenantHost thh;
        thh.kv = pl.kv;
        thh.rkind = std::make_shared<const std::vector<uint8_t>>(std::move(pl.img.rkind));
        sn->th.push_back(std::move(thh));
    }
    for (auto& pl : plans)
        if (!pl.kv) nf.tenant_ordinal.erase(pl.prefix.substr(3));   // its root record stays behind, unreachable
    nf.tags = std::move(table.tags);
    nf.n_big_edges = tag_live;
    nf.overflowed_blocks = table.overflowed_blocks;
    nf.n_routes = rank;
    nf.n_slots = (uint32_t) slot_cursor;
    nf.n_nodes = 0;
    nf.n_multi = 0;
    nf.n_cont_chunks = 0;
    for (auto& m : nf.tenants) {
        nf.n_nodes += m.tenant_nodes;
        nf.n_multi += m.n_multi;
        nf.n_cont_chunks += m.n_cont;
    }
    sn->garbage_slots = old->garbage_slots;
    for (auto& pl : plans)
        if (pl.old_index >= 0) sn->garbage_slots += of.tenants[(size_t) pl.old_index].csr_slots;
    sn->delta_commits = old->delta_commits + 1;
    lap("host bookkeeping");
    // ---- device: copy, upload, assemble, patch, shift
    cudaStream_t st = nullptr;
    BFQ_CUDA_TRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    // temporaries the enqueued work reads: declared ahead of the guard, so they are freed after it has synchronised the stream
    DeviceBuf<uint8_t> d_pack;   // the packed per-rank arrays and the run table
    DeviceBuf<uint32_t> d_ids;
    DeviceBuf<Slot> d_recs;
    DeviceBuf<RankShiftRegion> d_regions;
    DeviceBuf<RankShiftSlot> d_list;
    struct StreamGuard {
        cudaStream_t s;
        ~StreamGuard() { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
    } guard{st};
    const size_t n_new = (size_t) rank;
    BFQ_CUDA_TRY(sn->d_slots.reserve((size_t) slot_cursor));
    BFQ_CUDA_TRY(sn->d_tags.reserve(std::max<size_t>(nf.tags.size(), 1)));
    BFQ_CUDA_TRY(sn->d_roots.reserve(std::max<size_t>(nf.host_roots.size(), 1)));
    BFQ_CUDA_TRY(sn->d_segs.reserve(std::max<size_t>(nf.segs.size(), 2)));
    BFQ_CUDA_TRY(sn->d_rkind.reserve(std::max<size_t>(n_new, 1)));
    BFQ_CUDA_TRY(sn->d_pfxP.reserve(n_new + 1));
    BFQ_CUDA_TRY(sn->d_pfxG.reserve(n_new + 1));
    BFQ_CUDA_TRY(d_pack.reserve(pack_bytes));
    lap("device allocations");
    BFQ_CUDA_TRY(cudaMemcpyAsync(sn->d_slots.p, old->d_slots.p, (size_t) of.n_slots * sizeof(Slot), cudaMemcpyDeviceToDevice, st));
    if (up_slots) BFQ_CUDA_TRY(cudaMemcpyAsync(sn->d_slots.p + of.n_slots, regions_up.data(), (size_t) up_slots * sizeof(Slot), cudaMemcpyHostToDevice, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(d_pack.p, pack.data(), pack_bytes, cudaMemcpyHostToDevice, st));
    // the whole tag array (16 B per block, ~2 B per wide edge): one small upload
    if (!nf.tags.empty()) BFQ_CUDA_TRY(cudaMemcpyAsync(sn->d_tags.p, nf.tags.data(), nf.tags.size(), cudaMemcpyHostToDevice, st));
    {
        AssembleRankParams ap;
        ap.rkind = sn->d_rkind.p;
        ap.pfxP = sn->d_pfxP.p;
        ap.pfxG = sn->d_pfxG.p;
        ap.old_rkind = old->d_rkind.p;
        ap.old_pfxP = old->d_pfxP.p;
        ap.old_pfxG = old->d_pfxG.p;
        ap.up_rkind = d_pack.p;
        ap.up_pfxP = (const uint32_t*) (d_pack.p + off_pfxP);
        ap.up_pfxG = (const uint32_t*) (d_pack.p + off_pfxG);
        ap.runs = (const RankRun*) (d_pack.p + off_runs);
        ap.n_runs = (int32_t) runs.size();
        ap.n = (int64_t) n_new;
        ap.tailP = ppb;
        ap.tailG = pgb;
        launch_assemble_rank_arrays(ap, st);
    }
    // untouched tenants whose ranks move: slot regions and tag slots; rebuilt tenants: their tag-table records
    std::vector<RankShiftRegion> regions;
    std::vector<RankShiftSlot> shift_slots;
    std::vector<uint32_t> scatter_ids;
    std::vector<Slot> scatter_recs;
    for (size_t i = 0; i < nf.tenants.size(); i++) {
        const Entry& e = entries[i];
        const TenantMeta& m = nf.tenants[i];
        if (e.plan >= 0) {
            const TenantImage& img = plans[(size_t) e.plan].img;
            scatter_ids.insert(scatter_ids.end(), m.tag_slots.begin(), m.tag_slots.end());
            scatter_recs.insert(scatter_recs.end(), img.tag_recs.begin(), img.tag_recs.end());
            continue;
        }
        const TenantMeta& om = of.tenants[(size_t) e.old_index];
        const int64_t d = m.lo - om.lo;
        if (d != 0) {
            if (m.csr_slots) regions.push_back(RankShiftRegion{m.region_base, m.csr_slots, (int32_t) d});
            for (uint32_t s : m.tag_slots) shift_slots.push_back(RankShiftSlot{s, (int32_t) d});
            Slot& r = nf.host_roots[m.ordinal];
            if (r.w[W_OWN_COUNT] > 0 && !(r.w[W_META] & FLAG_OWN_MULTI)) r.w[W_OWN_FIRST] = (uint32_t) ((int64_t) r.w[W_OWN_FIRST] + d);
            if (r.w[W_HASH_COUNT] > 0 && !(r.w[W_META] & FLAG_HASH_MULTI)) r.w[W_HASH_FIRST] = (uint32_t) ((int64_t) r.w[W_HASH_FIRST] + d);
            if (m.seg_words) shift_seg_slice(nf.segs, m.seg_base, m.seg_words, d);
        }
    }
    if (!scatter_ids.empty()) {
        BFQ_CUDA_TRY(d_ids.reserve(scatter_ids.size()));
        BFQ_CUDA_TRY(d_recs.reserve(scatter_recs.size()));
        BFQ_CUDA_TRY(cudaMemcpyAsync(d_ids.p, scatter_ids.data(), scatter_ids.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
        BFQ_CUDA_TRY(cudaMemcpyAsync(d_recs.p, scatter_recs.data(), scatter_recs.size() * sizeof(Slot), cudaMemcpyHostToDevice, st));
        launch_scatter_records(sn->d_slots.p, d_ids.p, d_recs.p, (int64_t) scatter_ids.size(), st);
    }
    if (!regions.empty()) {
        BFQ_CUDA_TRY(d_regions.reserve(regions.size()));
        BFQ_CUDA_TRY(cudaMemcpyAsync(d_regions.p, regions.data(), regions.size() * sizeof(RankShiftRegion), cudaMemcpyHostToDevice, st));
        launch_rank_shift(sn->d_slots.p, d_regions.p, (int) regions.size(), st);
    }
    if (!shift_slots.empty()) {
        BFQ_CUDA_TRY(d_list.reserve(shift_slots.size()));
        BFQ_CUDA_TRY(cudaMemcpyAsync(d_list.p, shift_slots.data(), shift_slots.size() * sizeof(RankShiftSlot), cudaMemcpyHostToDevice, st));
        launch_rank_shift_listed(sn->d_slots.p, d_list.p, (int64_t) shift_slots.size(), st);
    }
    BFQ_CUDA_TRY(cudaMemcpyAsync(sn->d_roots.p, nf.host_roots.data(), nf.host_roots.size() * sizeof(Slot), cudaMemcpyHostToDevice, st));
    if (!nf.segs.empty()) BFQ_CUDA_TRY(cudaMemcpyAsync(sn->d_segs.p, nf.segs.data(), nf.segs.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    BFQ_CUDA_TRY(cudaGetLastError());
    lap("device copy + patch + rank shift");
    set_l2_window(h, sn.get());
    publish(h, std::move(sn));
    lap("publish (drops the old snapshot)");
    return BFQ_OK;
}

}  // namespace

int32_t bfq_index_commit(bfq_index* h) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    // The rebuild runs under the staging lock only: matches keep running on the previous snapshot meanwhile; the new one
    // is published by swapping one shared pointer. Matches and results in flight keep the old snapshot alive.
    std::lock_guard<std::mutex> gs(h->stage_mu);
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    std::shared_ptr<Snapshot> old;
    {
        std::lock_guard<std::mutex> g(h->mu);
        old = h->snap;
    }
    static const bool delta_enabled = [] {
        const char* e = getenv("BFQ_DELTA_COMMIT");   // experiment switch: 0 = every commit is a full build
        return !e || atoi(e) != 0;
    }();
    if (old && delta_enabled && !h->staging.bulk_changed()) {
        const std::vector<std::string> dirty = h->staging.dirty_tenants();
        if (dirty.empty()) {   // nothing staged since the last commit
            std::lock_guard<std::mutex> g(h->mu);
            h->rebuilt_tenants = 0;
            return BFQ_OK;
        }
        int64_t built = 0;
        const int32_t rc = commit_delta(h, old, dirty, &built);
        if (rc != BFQ_NEED_FULL) {
            if (rc == BFQ_OK) {
                std::lock_guard<std::mutex> g(h->mu);
                h->delta_commits++;
                h->rebuilt_tenants = built;
            }
            return rc;
        }
    }
    const int32_t rc = commit_full(h);
    if (rc == BFQ_OK) {
        std::lock_guard<std::mutex> g(h->mu);
        h->full_commits++;
        h->rebuilt_tenants = (int64_t) h->snap->flat.tenants.size();
    }
    return rc;
}

int32_t bfq_index_set_option(bfq_index* h, const char* name, int64_t value) {
    if (!h || !name) return fail(BFQ_E_INVALID, "bad argument");
    std::lock_guard<std::mutex> g(h->mu);
    const std::string n(name);
    if (n == "tier0_ctas_per_sm") h->tier0_ctas_per_sm = (int32_t) std::max<int64_t>(0, std::min<int64_t>(value, 32));
    else if (n == "order_min_topics") h->order_min = value <= 0 ? (int64_t) 1 << 62 : value;
    else if (n == "dedup") h->dedup = value != 0;
    else if (n == "dedup_hash_bits") {
        if (value < 0 || value > 64) return fail(BFQ_E_INVALID, "dedup_hash_bits must be in [0, 64]");
        h->dedup_hash_bits = (int32_t) value;
    } else if (n == "fanout_global") h->fanout_global = value != 0;
    else return fail(BFQ_E_INVALID, "unknown option: " + n);
    return BFQ_OK;
}

int32_t bfq_index_generation(bfq_index* h, uint64_t* generation) {
    if (!h || !generation) return fail(BFQ_E_INVALID, "bad argument");
    std::lock_guard<std::mutex> g(h->mu);
    *generation = h->snap ? h->snap->generation : 0;
    return BFQ_OK;
}

int32_t bfq_index_stats(bfq_index* h, int64_t* stats, int32_t n) {
    if (!h || !stats) return fail(BFQ_E_INVALID, "bad argument");
    std::lock_guard<std::mutex> g(h->mu);
    static const FlatIndex empty;
    const FlatIndex& f = h->snap ? h->snap->flat : empty;
    const int64_t wire_bytes = h->snap ? h->snap->wire_bytes.load() : 0;
    const int64_t v[23] = {f.n_routes, (int64_t) f.tenant_ordinal.size(), f.n_nodes, (int64_t) f.n_slots,
                           h->snap ? h->snap->device_bytes() : 0, f.max_nodes_per_depth, h->launches, h->overflow_topics,
                           h->flagged_topics, f.n_multi, f.n_cont_chunks, h->deferred_topics, h->duplicate_topics,
                           h->full_commits, h->delta_commits, h->snap ? (int64_t) h->snap->garbage_slots : 0,
                           h->buffer_retries, h->global_fanouts,
                           h->snap ? (int64_t) f.n_blocks * BLOCK_USABLE : 0, (int64_t) f.n_big_edges, f.overflowed_blocks,
                           h->rebuilt_tenants, wire_bytes};
    for (int32_t i = 0; i < n && i < 23; i++) stats[i] = v[i];
    return BFQ_OK;
}

int32_t bfq_host_build_stats(const uint8_t* keys, const int64_t* key_off, const uint8_t* vals, const int64_t* val_off,
                             int64_t n, int64_t* stats, int32_t n_stats) {
    if (n < 0 || !stats) return fail(BFQ_E_INVALID, "bad argument");
    Staging st;
    std::string err;
    const auto t0 = std::chrono::steady_clock::now();
    if (!st.load(keys, key_off, vals, val_off, n, &err)) return fail(BFQ_E_INVALID, err);
    const auto t1 = std::chrono::steady_clock::now();
    // the production path: straight from the staged per-tenant blobs
    std::vector<const KVBlob*> parts;
    for (auto& kvp : st.tenants()) parts.push_back(kvp.second.base.get());
    FlatIndex flat;
    if (!build_flat_index_parts(parts, &flat, &err)) return fail(BFQ_E_INVALID, err);
    const auto t2 = std::chrono::steady_clock::now();
    // stats[16]: a checksum of everything the build hands to the device (records, tags, roots, segments, per-rank arrays):
    // two builds of the same KV are the same image (tests compare the sorted-order and the hash-table trie construction);
    // stats[17]: 1 if the build from ONE concatenated blob (boundary scan) gives the same image as the per-tenant one
    auto image_sum_of = [](const FlatIndex& f) {
        uint64_t image_sum = 0;
        auto fold = [&](const void* p, size_t bytes) {
            const uint8_t* b = (const uint8_t*) p;
            uint64_t h[4] = {0x9E3779B97F4A7C15ull, 0xC2B2AE3D27D4EB4Full, 0x165667B19E3779F9ull, 0x27D4EB2F165667C5ull};
            size_t i = 0;
            for (; i + 32 <= bytes; i += 32)
                for (int k = 0; k < 4; k++) {
                    uint64_t w;
                    memcpy(&w, b + i + 8 * k, 8);
                    h[k] = (h[k] ^ w) * 0x100000001B3ull + (h[k] >> 29);
                }
            for (; i < bytes; i++) h[0] = (h[0] ^ b[i]) * 0x100000001B3ull;
            image_sum = fmix64(image_sum ^ fmix64(h[0] ^ fmix64(h[1] ^ fmix64(h[2] ^ fmix64(h[3] ^ bytes)))));
        };
        fold(f.slots.data(), (size_t) f.n_slots * sizeof(Slot));
        fold(f.tags.data(), f.tags.size());
        fold(f.roots.data(), f.roots.size() * sizeof(Slot));
        fold(f.segs.data(), f.segs.size() * sizeof(uint32_t));
        fold(f.rkind.data(), f.rkind.size());
        fold(f.pfx_persistent.data(), f.pfx_persistent.size() * sizeof(uint32_t));
        fold(f.pfx_group.data(), f.pfx_group.size() * sizeof(uint32_t));
        return image_sum;
    };
    uint64_t image_sum = 0;
    int64_t same_as_concat = -1;
    if (n_stats > 16) image_sum = image_sum_of(flat);
    if (n_stats > 17) {
        const KVBlob snapshot = st.concat();
        FlatIndex flat2;
        if (!build_flat_index(snapshot, &flat2, &err)) return fail(BFQ_E_INVALID, err);
        same_as_concat = image_sum_of(flat2) == image_sum && flat2.n_nodes == flat.n_nodes && flat2.tenants.size() == flat.tenants.size();
    }
    // stats[18]: tenants whose stand-alone image (build_tenant_image + place_tenant_image with the full build's bases — what a
    // delta commit uploads for a touched tenant) equals their part of the full image byte for byte; -1 - index of the first
    // that differs
    int64_t tenant_images_equal = 0;
    if (n_stats > 18) {
        size_t ti = 0;
        for (auto& kvp : st.tenants()) {
            if (ti >= flat.tenants.size()) break;
            const TenantMeta& m = flat.tenants[ti];
            TenantImage img;
            if (!build_tenant_image(*kvp.second.base, sv(m.tenant), m.ordinal, m.lo, m.region_base, m.seg_base, m.pp_base, m.pg_base, &img, &err))
                return fail(BFQ_E_INVALID, err);
            bool same = img.meta.big_edges == m.big_edges && img.meta.n_routes == m.n_routes;
            if (same && m.big_edges == 0) {
                same = img.meta.csr_slots == m.csr_slots && img.meta.seg_words == m.seg_words && img.meta.pp == m.pp && img.meta.pg == m.pg &&
                       img.meta.tenant_nodes == m.tenant_nodes && img.meta.n_multi == m.n_multi &&
                       memcmp(img.slots.data(), flat.slots.data() + m.region_base, (size_t) m.csr_slots * sizeof(Slot)) == 0 &&
                       memcmp(&img.root, &flat.roots[m.ordinal], sizeof(Slot)) == 0 &&
                       (m.seg_words == 0 || memcmp(img.segs.data(), flat.segs.data() + m.seg_base, (size_t) m.seg_words * 4) == 0) &&
                       (m.n_routes == 0 || (memcmp(img.rkind.data(), flat.rkind.data() + m.lo, (size_t) m.n_routes) == 0 &&
                                            memcmp(img.pfxP.data(), flat.pfx_persistent.data() + m.lo, (size_t) m.n_routes * 4) == 0 &&
                                            memcmp(img.pfxG.data(), flat.pfx_group.data() + m.lo, (size_t) m.n_routes * 4) == 0));
            }
            if (!same) {
                tenant_images_equal = -1 - (int64_t) ti;
                break;
            }
            tenant_images_equal++;
            ti++;
        }
    }
    // The lookup rules of the kernels, on the host: is the node record `sl` at slot s found again from its parent's record
    // `pr`? (nullptr = yes, else what is wrong). Wide nodes' children through the tag table `t`, the rest through the CSR rules.
    auto lookup_error = [](const Slot& sl, uint32_t s, const Slot& pr, const EdgeTable& t) -> const char* {
        if (sl.w[W_LEN] == LEN_PLUS) return pr.w[W_PLUS] == s ? nullptr : "'+' child is not linked from its parent";
        const uint32_t meta = pr.w[W_META];
        if (!(meta & FLAG_HAS_EXACT)) return "parent of an exact child lacks HAS_EXACT";
        uint32_t found;
        if (meta & FLAG_BIG) {
            found = t.find(sl.w[W_PARENT], sl.w[W_LEN], &sl.w[W_TOK]);
        } else {
            const uint32_t lg = meta_log2size(meta), sd = meta >> 16, t32 = fold32(token_hash(sl.w[W_LEN], &sl.w[W_TOK]));
            if (lg == 0 && (t32 & 0xFFFFu) != sd) return "single-child fingerprint mismatch";
            found = pr.w[W_CHILD_BASE] + (lg ? child_index(t32, sd, lg) : 0u);
        }
        return found == s ? nullptr : "child lookup does not find a placed node";
    };
    // stats[19]: tenants with wide edges whose delta rebuild, simulated here, is found again node for node by those rules.
    // The simulation is what bfq_index_commit's delta path does to the tenant: its tag slots are freed in a copy of the
    // image's tag table, it is rebuilt into a fresh region behind the image and its wide edges are placed into that table
    // (with the same key for its root-level edges: it keeps its ordinal), then its new tag-table records are written.
    int64_t wide_rebuilds_found = 0;
    if (n_stats > 19) {
        const size_t tag_region = (size_t) flat.n_blocks * BLOCK_SLOTS;
        size_t ti = 0;
        for (auto& kvp : st.tenants()) {
            if (ti >= flat.tenants.size()) break;
            const TenantMeta& m = flat.tenants[ti++];
            if (m.big_edges == 0) continue;
            EdgeTable sim;
            sim.n_blocks = flat.n_blocks;
            sim.tags = flat.tags;
            sim.overflowed_blocks = flat.overflowed_blocks;
            sim.slots.assign(flat.slots.begin(), flat.slots.begin() + (ptrdiff_t) tag_region);
            for (uint32_t s : m.tag_slots) sim.release(s);
            const uint64_t base = flat.n_slots;
            TenantImage img;
            if (!build_tenant_image(*kvp.second.base, sv(m.tenant), m.ordinal, m.lo, &img, &err) ||
                !place_tenant_image(&img, base, flat.segs.size(), m.pp_base, m.pg_base, &sim, ~0ull, nullptr, &err))
                return fail(BFQ_E_INVALID, err);
            if (!img.placed || img.meta.tag_slots.size() != m.big_edges) continue;
            for (size_t k = 0; k < img.tag_recs.size(); k++) sim.slots[img.meta.tag_slots[k]] = img.tag_recs[k];
            auto record_of = [&](uint32_t id) -> const Slot* {
                if (id >= ROOT_BASE) return id == ROOT_BASE + m.ordinal ? &img.root : nullptr;
                if (id < tag_region) return &sim.slots[id];
                return id >= base && id - base < img.slots.size() ? &img.slots[id - base] : nullptr;
            };
            int64_t found = 0;
            bool ok = true;
            auto check = [&](uint32_t s, const Slot& sl) {
                const Slot* pr = record_of(sl.w[W_PARENT]);
                ok = ok && pr && lookup_error(sl, s, *pr, sim) == nullptr;
                found++;
            };
            for (size_t i = 0; i < img.slots.size(); i++)
                if (img.slots[i].w[W_PARENT] != EMPTY_PARENT) check((uint32_t) (base + i), img.slots[i]);
            for (uint32_t s : img.meta.tag_slots) check(s, sim.slots[s]);
            if (ok && found + 1 == img.meta.tenant_nodes) wide_rebuilds_found++;
        }
    }
    // self-check: every placed node is found again from its parent's record the way the kernels look it up
    {
        EdgeTable t;
        t.slots = std::move(flat.slots);
        t.tags = std::move(flat.tags);
        t.n_blocks = flat.n_blocks;
        int64_t used = 0;
        for (uint32_t s = 0; s < flat.n_slots; s++) {
            const Slot& sl = t.slots[s];
            if (sl.w[W_PARENT] == EMPTY_PARENT) continue;
            used++;
            const uint32_t pid = sl.w[W_PARENT];
            const Slot& pr = pid >= ROOT_BASE ? flat.roots[pid - ROOT_BASE] : t.slots[pid];
            if (const char* e = lookup_error(sl, s, pr, t)) return fail(BFQ_E_STATE, e);
        }
        if (used + (int64_t) flat.roots.size() != flat.n_nodes) return fail(BFQ_E_STATE, "node count mismatch");
    }
    const int64_t v[8] = {flat.n_routes, (int64_t) flat.tenant_ordinal.size(), flat.n_nodes, (int64_t) flat.n_slots,
                          flat.max_nodes_per_depth, flat.max_tenant_nodes, flat.n_multi, flat.n_cont_chunks};
    for (int32_t i = 0; i < n_stats && i < 8; i++) stats[i] = v[i];
    if (n_stats > 8) stats[8] = flat.overflowed_blocks;
    for (int32_t i = 9; i < n_stats && i < 9 + 5; i++) stats[i] = flat.child_hist[i - 9];
    if (n_stats > 14) stats[14] = std::chrono::duration_cast<std::chrono::microseconds>(t1 - t0).count();   // staging
    if (n_stats > 15) stats[15] = std::chrono::duration_cast<std::chrono::microseconds>(t2 - t1).count();   // flatten
    if (n_stats > 16) stats[16] = (int64_t) image_sum;
    if (n_stats > 17) stats[17] = same_as_concat;
    if (n_stats > 18) stats[18] = tenant_images_equal;
    if (n_stats > 19) stats[19] = wide_rebuilds_found;
    return BFQ_OK;
}

int32_t bfq_index_last_kernel_ms(bfq_index* h, double* ms) {
    if (!h || !ms) return fail(BFQ_E_INVALID, "bad argument");
    std::lock_guard<std::mutex> g(h->mu);
    *ms = h->last_kernel_ms;
    return BFQ_OK;
}

namespace {
int32_t lookup_in(const Snapshot* s, int64_t rank, uint8_t* key_out, int64_t key_cap, int64_t* key_len, uint8_t* val_out,
                  int64_t val_cap, int64_t* val_len) {
    size_t ti = 0;
    int64_t local = 0;
    if (!s->locate(rank, &ti, &local)) return fail(BFQ_E_RANGE, "rank out of range");
    sv k = s->th[ti].kv->key(local), v = s->th[ti].kv->val(local);
    if (key_len) *key_len = (int64_t) k.size();
    if (val_len) *val_len = (int64_t) v.size();
    if (key_out && (int64_t) k.size() <= key_cap) memcpy(key_out, k.data(), k.size());
    if (val_out && (int64_t) v.size() <= val_cap) memcpy(val_out, v.data(), v.size());
    return BFQ_OK;
}
int32_t kinds_in(const Snapshot* s, const int64_t* ranks, int64_t n, uint8_t* kinds_out) {
    for (int64_t i = 0; i < n; i++) {
        size_t ti = 0;
        int64_t local = 0;
        if (!s->locate(ranks[i], &ti, &local)) return fail(BFQ_E_RANGE, "rank out of range");
        kinds_out[i] = (*s->th[ti].rkind)[(size_t) local];
    }
    return BFQ_OK;
}
std::shared_ptr<Snapshot> current(bfq_index* h) {
    std::lock_guard<std::mutex> g(h->mu);
    return h->snap;
}
}  // namespace

int32_t bfq_route_lookup(bfq_index* h, int64_t rank, uint8_t* key_out, int64_t key_cap, int64_t* key_len,
                         uint8_t* val_out, int64_t val_cap, int64_t* val_len) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    auto s = current(h);
    if (!s) return fail(BFQ_E_STATE, "no committed snapshot");
    return lookup_in(s.get(), rank, key_out, key_cap, key_len, val_out, val_cap, val_len);
}

int32_t bfq_route_kind(bfq_index* h, int64_t rank, int32_t* kind) {
    if (!h || !kind) return fail(BFQ_E_INVALID, "bad argument");
    auto s = current(h);
    if (!s) return fail(BFQ_E_STATE, "no committed snapshot");
    uint8_t k = 0;
    int32_t rc = kinds_in(s.get(), &rank, 1, &k);
    if (rc == BFQ_OK) *kind = k;
    return rc;
}

int32_t bfq_route_kinds(bfq_index* h, const int64_t* ranks, int64_t n, uint8_t* kinds_out) {
    if (!h || n < 0 || (n > 0 && (!ranks || !kinds_out))) return fail(BFQ_E_INVALID, "bad argument");
    auto s = current(h);
    if (!s) return fail(BFQ_E_STATE, "no committed snapshot");
    return kinds_in(s.get(), ranks, n, kinds_out);
}

int32_t bfq_result_route_lookup(const bfq_result* r, int64_t rank, uint8_t* key_out, int64_t key_cap, int64_t* key_len,
                                uint8_t* val_out, int64_t val_cap, int64_t* val_len) {
    if (!r || !r->snap) return fail(BFQ_E_INVALID, "result is NULL");
    return lookup_in(r->snap.get(), rank, key_out, key_cap, key_len, val_out, val_cap, val_len);
}
int32_t bfq_result_route_kinds(const bfq_result* r, const int64_t* ranks, int64_t n, uint8_t* kinds_out) {
    if (!r || !r->snap || n < 0 || (n > 0 && (!ranks || !kinds_out))) return fail(BFQ_E_INVALID, "bad argument");
    return kinds_in(r->snap.get(), ranks, n, kinds_out);
}
uint64_t bfq_result_generation(const bfq_result* r) { return r && r->snap ? r->snap->generation : 0; }

int32_t bfq_match(bfq_index* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                  const uint8_t* topics, const int64_t* topic_off, const int32_t* topic_tenant, int64_t n,
                  const int32_t* max_pfanout, const int32_t* max_gfanout, bfq_result** out) {
    if (!h || !out || n < 0 || n_tenants < 0) return fail(BFQ_E_INVALID, "bad argument");
    if (n > 0 && (!topics || !topic_off || !topic_tenant || !tenants || !tenant_off)) return fail(BFQ_E_INVALID, "NULL input");
    if (n_tenants > 0 && (!tenants || !tenant_off)) return fail(BFQ_E_INVALID, "NULL tenant list");
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    std::shared_ptr<Snapshot> snap;
    Workspace* w = nullptr;
    int32_t rc = acquire(h, &snap, &w, "bfq_match");
    if (rc != BFQ_OK) return rc;
    // the workspace goes back to the pool on every error path; on success the result keeps it
    struct Lease {
        bfq_index* h;
        Workspace* w;
        ~Lease() { if (w) { cudaSetDevice(h->device); cudaDeviceSynchronize(); give_back(h->pool, w); } }
    } lease{h, w};
    // topic_tenant[i] is range-checked on the device (an index outside [0, n_tenants) yields an empty result)
    auto t0 = std::chrono::steady_clock::now();
    const size_t nn = (size_t) std::max<int64_t>(n, 1);
    const int64_t blob_e = n ? topic_off[n] : 0;
    BFQ_CUDA_TRY(w->d_topics.reserve((size_t) std::max<int64_t>(blob_e, 1) + 64));
    BFQ_CUDA_TRY(w->d_topic_off.reserve(nn + 1));
    BFQ_CUDA_TRY(w->d_topic_tenant.reserve(nn));
    BFQ_CUDA_TRY(w->d_cnt.reserve(nn));
    BFQ_CUDA_TRY(w->d_new_begin.reserve(nn));
    BFQ_CUDA_TRY(w->d_final_begin.reserve(nn));
    BFQ_CUDA_TRY(w->d_final_count.reserve(nn));
    BFQ_CUDA_TRY(w->h_span_begin.reserve(nn));
    BFQ_CUDA_TRY(w->h_span_count.reserve(nn));
    BFQ_CUDA_TRY(w->h_route_count.reserve(nn));

    // Large batches are cut into sub-batches that flow through three streams: all H2D copies on one, the kernels +
    // compaction + D2H of consecutive sub-batches alternating on two others, so the copy of sub-batch c+1 and the
    // result read-back of c-1 overlap the kernels of c (PCIe is full duplex; the copies dominate the host path).
    // four sub-batches, not eight: a 125k-topic sub-batch is less than one wave of tier-0 lanes, its kernel takes as long as
    // a 250k one
    int C = n >= (1 << 17) ? 4 : 1;
    {
        static const int forced = [] {   // experiment switch BFQ_SUBBATCHES
            const char* e = getenv("BFQ_SUBBATCHES");
            return e ? std::min(std::max(atoi(e), 1), (int) MAX_CHUNKS) : 0;
        }();
        if (forced > 0 && n >= (1 << 17)) C = forced;
    }
    CoreOut co;
    int64_t rbase = 0, tbase = 0;
    double kernel_ms = -1;
    for (int attempt = 0;; attempt++) {
        if (attempt == 8) return fail(BFQ_E_STATE, "buffer sizing did not converge");
        rc = prepare_workspace(h, w, n, C, n_tenants);
        if (rc != BFQ_OK) return rc;
        BFQ_CUDA_TRY(w->d_ranges_c.reserve(w->d_ranges.cap));
        const uint64_t dyn_total = w->d_ranges.cap - (uint64_t) n * INLINE_RANGES;
        // whole spill blocks per slice: tier 0 writes a spill block in 32-byte sectors, so it must start on one
        const uint64_t dyn_slice = dyn_total / (uint64_t) C / SPILL_RANGES * SPILL_RANGES, thr_slice = w->d_throttled.cap / (uint64_t) C;
        size_t tmp_bytes = 0;
        {
            CompactParams q{};
            q.n_topics = (n + C - 1) / C + 1;
            q.counts = w->d_cnt.p;
            q.new_begin = w->d_new_begin.p;
            BFQ_CUDA_TRY(launch_compact(q, nullptr, &tmp_bytes, w->stream, 1));
            BFQ_CUDA_TRY(w->d_scan_tmp.reserve(tmp_bytes * 2 + 512));   // one scratch per compute stream
        }
        co = CoreOut();
        rbase = tbase = 0;
        // ---- H2D of every sub-batch, back to back on the copy stream
        BFQ_CUDA_TRY(cudaEventRecord(w->ev[0], w->copy_stream));
        // the kernels read whole aligned 16-byte granules: define the bytes behind the blob's end (masked out, but read)
        BFQ_CUDA_TRY(cudaMemsetAsync(w->d_topics.p + blob_e, 0, 64, w->copy_stream));
        rc = resolve_tenants(w, snap.get(), tenants, tenant_off, n_tenants, max_pfanout, max_gfanout, w->copy_stream);
        if (rc != BFQ_OK) return rc;
        int64_t bounds[MAX_CHUNKS + 1];
        for (int c = 0; c <= C; c++) bounds[c] = n * c / C;
        for (int c = 0; c < C && n > 0; c++) {
            const int64_t b = bounds[c], e = bounds[c + 1];
            const int64_t ob = topic_off[b], oe = topic_off[e];
            BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_topic_off.p + b, topic_off + b, (size_t) (e - b + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, w->copy_stream));
            BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_topic_tenant.p + b, topic_tenant + b, (size_t) (e - b) * sizeof(int32_t), cudaMemcpyHostToDevice, w->copy_stream));
            BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_topics.p + ob, topics + ob, (size_t) (oe - ob), cudaMemcpyHostToDevice, w->copy_stream));
            BFQ_CUDA_TRY(cudaEventRecord(w->ev_h2d[c], w->copy_stream));
        }
        BFQ_CUDA_TRY(cudaEventRecord(w->ev[1], w->copy_stream));
        if (n == 0) BFQ_CUDA_TRY(cudaStreamSynchronize(w->copy_stream));
        bool retry = false;
        for (int c = 0; c < C && n > 0; c++) {
            cudaStream_t st = C == 1 ? w->stream : w->work_stream[c & 1];
            BFQ_CUDA_TRY(cudaStreamWaitEvent(st, w->ev_h2d[c], 0));
            SubBatch sb;
            sb.begin = bounds[c];
            sb.n = bounds[c + 1] - bounds[c];
            sb.n_total = n;
            sb.chunk = c;
            sb.dyn_off = (uint64_t) c * dyn_slice;
            sb.dyn_cap = dyn_slice;
            sb.thr_off = (uint64_t) c * thr_slice;
            sb.thr_cap = thr_slice;
            CoreCtx ctx{h, w, snap.get(), w->d_topics.p, w->d_topic_off.p, w->d_topic_tenant.p, n_tenants, st};
            rc = enqueue_core(ctx, sb, &co);
            if (rc != BFQ_OK) return rc;
            // ---- compaction of this sub-batch: counts + scan + total (enqueued optimistically behind the match kernels),
            // then, once the total is known on the host, the gather into the dense result position
            unsigned long long* hc = w->h_counters.p + (size_t) c * CTR_COUNT;
            const uint64_t region = (uint64_t) sb.begin * INLINE_RANGES + sb.dyn_off;   // this sub-batch's private slice of d_ranges_c
            CompactParams cp{};
            cp.n_topics = sb.n;
            cp.span_begin = w->d_span_begin.p + sb.begin;
            cp.span_count = w->d_span_count.p + sb.begin;
            cp.ranges = w->d_ranges.p + (uint64_t) sb.begin * INLINE_RANGES;
            cp.leader = (wants_order(ctx, sb) && h->dedup) ? w->d_leader.p + sb.begin : nullptr;   // repeats share their leader's dense span
            cp.counts = w->d_cnt.p + sb.begin;
            cp.new_begin = w->d_new_begin.p + sb.begin;
            cp.final_begin = w->d_final_begin.p + sb.begin;
            cp.final_count = w->d_final_count.p + sb.begin;
            cp.ranges_out = w->d_ranges_c.p + region;
            cp.ranges_out_cap = (uint64_t) sb.n * INLINE_RANGES + sb.dyn_cap;
            cp.total_out = w->d_counters.p + (size_t) c * CTR_COUNT + CTR_ROUTES;
            uint8_t* scan_tmp = w->d_scan_tmp.p + (size_t) (c & 1) * ((tmp_bytes + 256) / 256 * 256);
            BFQ_CUDA_TRY(launch_compact(cp, scan_tmp, &tmp_bytes, st, 1));
            rc = copy_counters(ctx, sb);
            if (rc != BFQ_OK) return rc;
            bool reran = false;
            rc = finish_core(ctx, sb, &co, &reran);
            if (rc == BFQ_RETRY_GROW) {
                retry = true;
                break;
            }
            if (rc != BFQ_OK) return rc;
            if (reran) {   // tier 2 changed spans: redo the counting pass
                BFQ_CUDA_TRY(launch_compact(cp, scan_tmp, &tmp_bytes, st, 1));
                rc = copy_counters(ctx, sb);
                if (rc != BFQ_OK) return rc;
                BFQ_CUDA_TRY(cudaStreamSynchronize(st));
                co.n_launches += 3;
            }
            if (c == 0) {
                float kms = 0;
                cudaEventElapsedTime(&kms, w->evk[0], w->evk[1]);
                kernel_ms = kms;
            }
            const int64_t total_c = (int64_t) hc[CTR_ROUTES], thr_c = co.chunk_throttled[c];
            // host result buffers grow by reallocation: wait for the copies in flight before moving them
            if ((size_t) (rbase + total_c) > w->h_ranges.cap || (size_t) (tbase + thr_c) > w->h_throttled.cap) {
                BFQ_CUDA_TRY(cudaDeviceSynchronize());
                if ((size_t) (rbase + total_c) > w->h_ranges.cap) {
                    PinnedBuf<uint2> nb;
                    BFQ_CUDA_TRY(nb.reserve((size_t) ((rbase + total_c) * (C - c > 1 ? 2 : 1) + (1 << 16))));
                    if (rbase) memcpy(nb.p, w->h_ranges.p, (size_t) rbase * sizeof(uint2));
                    w->h_ranges = std::move(nb);
                }
                if ((size_t) (tbase + thr_c) > w->h_throttled.cap) {
                    PinnedBuf<uint3> nb;
                    BFQ_CUDA_TRY(nb.reserve((size_t) ((tbase + thr_c) * 2 + 1024)));
                    if (tbase) memcpy(nb.p, w->h_throttled.p, (size_t) tbase * sizeof(uint3));
                    w->h_throttled = std::move(nb);
                }
            }
            cp.out_base = (uint32_t) rbase;
            BFQ_CUDA_TRY(launch_compact(cp, scan_tmp, &tmp_bytes, st, 2));
            co.n_launches += 4;
            BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_span_begin.p + sb.begin, w->d_final_begin.p + sb.begin, (size_t) sb.n * 4, cudaMemcpyDeviceToHost, st));
            BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_span_count.p + sb.begin, w->d_final_count.p + sb.begin, (size_t) sb.n * 4, cudaMemcpyDeviceToHost, st));
            BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_route_count.p + sb.begin, w->d_route_count.p + sb.begin, (size_t) sb.n * 4, cudaMemcpyDeviceToHost, st));
            if (total_c > 0)
                BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_ranges.p + rbase, w->d_ranges_c.p + region, (size_t) total_c * sizeof(uint2), cudaMemcpyDeviceToHost, st));
            if (thr_c > 0)
                BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_throttled.p + tbase, w->d_throttled.p + sb.thr_off, (size_t) thr_c * sizeof(uint3), cudaMemcpyDeviceToHost, st));
            rbase += total_c;
            tbase += thr_c;
        }
        if (!retry) break;
        // a slice of the range / throttled buffers was too small: grow them and redo the batch un-chunked
        count_retry(h);
        BFQ_CUDA_TRY(cudaDeviceSynchronize());
        rc = grow_for_retry(w, co, n, C);
        if (rc != BFQ_OK) return rc;
        C = 1;
    }
    BFQ_CUDA_TRY(cudaStreamSynchronize(w->work_stream[0]));
    BFQ_CUDA_TRY(cudaStreamSynchronize(w->work_stream[1]));
    BFQ_CUDA_TRY(cudaStreamSynchronize(w->stream));
    BFQ_CUDA_TRY(cudaStreamSynchronize(w->copy_stream));
    add_stats(h, co, n, kernel_ms);
    co.n_ranges = rbase;
    co.n_throttled = tbase;
    if (co.n_throttled > 1) {
        uint3* th = w->h_throttled.p;
        std::sort(th, th + co.n_throttled, [](const uint3& a, const uint3& b) { return a.x != b.x ? a.x < b.x : a.y < b.y; });
    }
    auto* r = new bfq_result();
    r->owner = h;
    r->pool = h->pool;
    r->snap = std::move(snap);
    r->ws = w;
    lease.w = nullptr;   // the result holds the workspace from here on
    r->n_topics = n;
    r->n_ranges = co.n_ranges;
    r->n_throttled = co.n_throttled;
    r->span_begin = w->h_span_begin.p;
    r->span_count = w->h_span_count.p;
    r->route_count = w->h_route_count.p;
    r->ranges = reinterpret_cast<const bfq_range*>(w->h_ranges.p);
    r->throttled = reinterpret_cast<const bfq_throttled*>(w->h_throttled.p);
    float a = 0;
    cudaEventElapsedTime(&a, w->ev[0], w->ev[1]);
    r->ms[0] = a;                       // H2D stream busy time (overlapped with the kernels of earlier sub-batches)
    r->ms[1] = kernel_ms < 0 ? 0 : kernel_ms;   // tier-0 kernel of the first sub-batch
    r->ms[2] = (double) C;              // number of sub-batches
    r->ms[3] = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    *out = r;
    return BFQ_OK;
}

int64_t bfq_result_num_topics(const bfq_result* r) { return r ? r->n_topics : 0; }
const uint32_t* bfq_result_span_begin(const bfq_result* r) { return r->span_begin; }
const uint32_t* bfq_result_span_count(const bfq_result* r) { return r->span_count; }
const uint32_t* bfq_result_route_count(const bfq_result* r) { return r->route_count; }
const bfq_range* bfq_result_ranges(const bfq_result* r, int64_t* n_ranges) {
    if (n_ranges) *n_ranges = r->n_ranges;
    return r->ranges;
}
const bfq_throttled* bfq_result_throttled(const bfq_result* r, int64_t* n_throttled) {
    if (n_throttled) *n_throttled = r->n_throttled;
    return r->throttled;
}

int64_t bfq_result_expand(const bfq_result* r, int64_t* offsets, int64_t* ranks, int64_t rank_cap) {
    if (!r || !offsets) return BFQ_E_INVALID;
    const std::vector<uint32_t>& segs = r->snap->flat.segs;   // the snapshot the ranges were produced from
    const int64_t n = r->n_topics;
    // throttled[] is sorted by (topic, rank): first entry of every topic
    std::vector<int64_t> thr_begin((size_t) n + 1, r->n_throttled);
    {
        int64_t ti = 0;
        for (int64_t t = 0; t <= n; t++) {
            while (ti < r->n_throttled && (int64_t) r->throttled[ti].topic < t) ti++;
            thr_begin[(size_t) t] = ti;
        }
    }
    // pass 1: survivors per topic -> offsets (route_count counts every matched route, a multi-segment range included)
    int64_t total = 0;
    for (int64_t t = 0; t < n; t++) {
        offsets[t] = total;
        total += (int64_t) r->route_count[t] - (thr_begin[(size_t) t + 1] - thr_begin[(size_t) t]);
    }
    offsets[n] = total;
    if (!ranks || total > rank_cap) return total;
    // pass 2: topics are independent -> all host threads
    auto fill = [&](int64_t t_lo, int64_t t_hi) {
        std::vector<int64_t> tmp;
        for (int64_t t = t_lo; t < t_hi; t++) {
            tmp.clear();
            const uint32_t b = r->span_begin[t], c = r->span_count[t];
            for (uint32_t j = 0; j < c; j++) {
                const bfq_range rg = r->ranges[b + j];
                if (rg.count & RANGE_MULTI) {
                    const uint32_t nseg = segs[2 * (size_t) rg.first];
                    for (uint32_t s = 0; s < nseg; s++) {
                        const uint32_t f = segs[2 * ((size_t) rg.first + 1 + s)], m = segs[2 * ((size_t) rg.first + 1 + s) + 1];
                        for (uint32_t x = 0; x < m; x++) tmp.push_back((int64_t) f + x);
                    }
                } else {
                    for (uint32_t x = 0; x < rg.count; x++) tmp.push_back((int64_t) rg.first + x);
                }
            }
            if (c > 1) std::sort(tmp.begin(), tmp.end());
            int64_t ti = thr_begin[(size_t) t], te = thr_begin[(size_t) t + 1], o = offsets[t];
            for (int64_t x : tmp) {
                while (ti < te && (int64_t) r->throttled[ti].rank < x) ti++;
                if (ti < te && (int64_t) r->throttled[ti].rank == x) continue;
                ranks[o++] = x;
            }
        }
    };
    const int64_t workers = std::max<int64_t>(1, std::min<int64_t>((int64_t) std::thread::hardware_concurrency(), std::min<int64_t>(64, total / 65536)));
    if (workers <= 1) {
        fill(0, n);
    } else {
        std::vector<std::thread> th;
        for (int64_t k = 0; k < workers; k++) th.emplace_back(fill, n * k / workers, n * (k + 1) / workers);
        for (auto& x : th) x.join();
    }
    return total;
}

int32_t bfq_result_timings(const bfq_result* r, double* ms, int32_t n) {
    if (!r || !ms) return fail(BFQ_E_INVALID, "bad argument");
    for (int32_t i = 0; i < n && i < 4; i++) ms[i] = r->ms[i];
    return BFQ_OK;
}
void bfq_result_free(bfq_result* r) {
    if (!r) return;
    give_back(r->pool, r->ws);
    delete r;
}

int32_t bfq_match_device_async(bfq_index* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                               const uint8_t* d_topics, const int64_t* d_topic_off, const int32_t* d_topic_tenant, int64_t n,
                               const int32_t* max_pfanout, const int32_t* max_gfanout, void* stream, bfq_device_result* out) {
    if (!h || !out || n < 0 || n_tenants < 0) return fail(BFQ_E_INVALID, "bad argument");
    if (n_tenants > 0 && (!tenants || !tenant_off)) return fail(BFQ_E_INVALID, "NULL tenant list");
    memset(out, 0, sizeof(*out));
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    auto* L = new DeviceLease();
    L->h = h;
    L->pool = h->pool;
    int32_t rc = acquire(h, &L->snap, &L->ws, "bfq_match_device");
    if (rc != BFQ_OK) {
        delete L;
        return rc;
    }
    cudaStream_t st = (cudaStream_t) stream;
    L->n = n;
    L->ctx = CoreCtx{h, L->ws, L->snap.get(), d_topics, d_topic_off, d_topic_tenant, n_tenants, st};
    rc = resolve_tenants(L->ws, L->snap.get(), tenants, tenant_off, n_tenants, max_pfanout, max_gfanout, st);
    if (rc == BFQ_OK) rc = device_enqueue(L);
    if (rc != BFQ_OK) {
        cudaStreamSynchronize(st);
        give_back(h->pool, L->ws);
        delete L;
        return rc;
    }
    fill_device_result(L, out);
    out->lease = L;
    return BFQ_OK;
}

int32_t bfq_device_result_wait(bfq_device_result* out) {
    if (!out || !out->lease) return fail(BFQ_E_INVALID, "no match in flight behind this result");
    auto* L = static_cast<DeviceLease*>(out->lease);
    if (cudaSetDevice(L->h->device) != cudaSuccess) return fail(BFQ_E_CUDA, "cudaSetDevice");
    const int32_t rc = device_wait(L);
    if (rc == BFQ_OK) fill_device_result(L, out);
    return rc;
}

void bfq_device_result_release(bfq_device_result* out) {
    if (!out || !out->lease) return;
    auto* L = static_cast<DeviceLease*>(out->lease);
    cudaSetDevice(L->pool->device);
    // never hand a busy workspace back: the match, and every call that used the result since, on each of its streams
    cudaEventSynchronize(L->ws->ev_done);
    for (size_t i = 0; i < L->used_on.size(); i++) cudaEventSynchronize(L->ws->ev_use[i]);
    give_back(L->pool, L->ws);
    delete L;
    out->lease = nullptr;
}

int32_t bfq_match_device(bfq_index* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                         const uint8_t* d_topics, const int64_t* d_topic_off, const int32_t* d_topic_tenant, int64_t n,
                         const int32_t* max_pfanout, const int32_t* max_gfanout, void* stream, bfq_device_result* out) {
    int32_t rc = bfq_match_device_async(h, tenants, tenant_off, n_tenants, d_topics, d_topic_off, d_topic_tenant, n, max_pfanout,
                                        max_gfanout, stream, out);
    if (rc != BFQ_OK) return rc;
    rc = bfq_device_result_wait(out);
    if (rc != BFQ_OK) bfq_device_result_release(out);
    return rc;
}

}  // extern "C"

int32_t bfq::lease_use(const bfq_device_result* res, cudaStream_t stream, const char* who, cudaEvent_t* ev) {
    if (!res || !res->lease) return fail(BFQ_E_INVALID, std::string(who) + ": no match in flight behind this result");
    auto* L = static_cast<DeviceLease*>(res->lease);
    if (!L->done || L->rc != BFQ_OK) return fail(BFQ_E_STATE, std::string(who) + " needs a completed match (bfq_device_result_wait)");
    BFQ_CUDA_TRY(cudaSetDevice(L->h->device));
    std::lock_guard<std::mutex> g(L->use_mu);
    size_t i = 0;
    while (i < L->used_on.size() && L->used_on[i] != stream) i++;
    if (i == L->used_on.size()) {
        Workspace* w = L->ws;
        if (w->ev_use.size() == i) {
            cudaEvent_t e = nullptr;
            BFQ_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            w->ev_use.push_back(e);
        }
        L->used_on.push_back(stream);
    }
    *ev = L->ws->ev_use[i];
    return BFQ_OK;
}

namespace {
// the expand's inputs for a completed device match (its workspace, snapshot and caps) and the caller's CSR outputs
ExpandParams expand_params(const DeviceLease* L, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap) {
    const Workspace* w = L->ws;
    const Snapshot* s = L->snap.get();
    const size_t nt = (size_t) std::max(L->ctx.n_tenants, 1);
    ExpandParams p{};
    p.n_topics = L->n;
    p.span_begin = w->d_span_begin.p;
    p.span_count = w->d_span_count.p;
    p.route_count = w->d_route_count.p;
    p.kept_count = w->d_kept.p;
    p.ranges = w->d_ranges.p;
    p.segs = s->d_segs.p;
    p.counts = w->d_exp_counts.p;
    p.offsets = d_offsets;
    p.ranks = d_ranks;
    p.rank_cap = d_ranks ? rank_cap : 0;
    p.flagged_list = w->d_flagged.p;
    p.n_flagged = L->co.n_flagged;
    p.topic_tenant = L->ctx.d_topic_tenant;
    p.max_pfanout = w->d_tenant_tab.p + nt;
    p.max_gfanout = w->d_tenant_tab.p + 2 * nt;
    p.rkind = s->d_rkind.p;
    p.pfx_persistent = s->d_pfxP.p;
    p.pfx_group = s->d_pfxG.p;
    return p;
}
}  // namespace

extern "C" {

int32_t bfq_expand_device(const bfq_device_result* res, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap, void* stream,
                          int64_t* n_ranks) {
    if (!res || !res->lease || !d_offsets) return fail(BFQ_E_INVALID, "bad argument");
    auto* L = static_cast<DeviceLease*>(res->lease);
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    const int32_t rc = lease_use(res, st, "bfq_expand_device", &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);   // phase 2 is still running when the call returns
    bfq_index* h = L->h;
    Workspace* w = L->ws;
    const int64_t n_topics = L->n;
    BFQ_CUDA_TRY(w->d_exp_counts.reserve((size_t) n_topics + 1));
    const ExpandParams p = expand_params(L, d_offsets, d_ranks, rank_cap);
    size_t tmp_bytes = 0;
    BFQ_CUDA_TRY(launch_expand(p, nullptr, &tmp_bytes, st, 1));
    BFQ_CUDA_TRY(w->d_scan_tmp.reserve(tmp_bytes + 256));
    BFQ_CUDA_TRY(launch_expand(p, w->d_scan_tmp.p, &tmp_bytes, st, 1));
    long long total = 0;
    BFQ_CUDA_TRY(cudaMemcpyAsync(&total, d_offsets + n_topics, sizeof(long long), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    if (n_ranks) *n_ranks = (int64_t) total;
    int64_t launches = 2;
    if (d_ranks && total <= rank_cap) {
        BFQ_CUDA_TRY(launch_expand(p, w->d_scan_tmp.p, &tmp_bytes, st, 2));
        launches += 2;
    }
    std::lock_guard<std::mutex> g(h->mu);
    h->launches += launches;
    return BFQ_OK;
}

int32_t bfq_expand_device_budget(const bfq_device_result* res, const int32_t* d_msg_bytes, const int64_t* max_pfanout_bytes,
                                 const uint8_t* tenant_bandwidth, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap,
                                 void* stream, bfq_budget_result* out) {
    if (!res || !res->lease || !d_offsets || !out) return fail(BFQ_E_INVALID, "bad argument");
    auto* L = static_cast<DeviceLease*>(res->lease);
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    const int32_t rc = lease_use(res, st, "bfq_expand_device_budget", &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);   // phase 2 is still running when the call returns
    const int64_t n_topics = L->n;
    const int32_t n_tenants = L->ctx.n_tenants;
    if (n_topics > 0 && !d_msg_bytes) return fail(BFQ_E_INVALID, "NULL d_msg_bytes");
    if (n_tenants > 0 && (!max_pfanout_bytes || !tenant_bandwidth)) return fail(BFQ_E_INVALID, "NULL per-tenant budget table");
    for (int32_t i = 0; i < n_tenants; i++)
        if (max_pfanout_bytes[i] <= 0)
            return fail(BFQ_E_INVALID, "max_pfanout_bytes[" + std::to_string(i) + "] = " + std::to_string(max_pfanout_bytes[i]) +
                                           ": MaxPersistentFanoutBytes must be > 0");
    bfq_index* h = L->h;
    Workspace* w = L->ws;
    const size_t nn = (size_t) std::max<int64_t>(n_topics, 1), nt = (size_t) std::max(n_tenants, 1);
    BFQ_CUDA_TRY(w->d_exp_counts.reserve(nn + 1));
    BFQ_CUDA_TRY(w->d_bud_bytes.reserve(nt));
    BFQ_CUDA_TRY(w->d_bud_bw.reserve(nt));
    BFQ_CUDA_TRY(w->d_bud_flags.reserve(nn));
    BFQ_CUDA_TRY(w->d_bud_dp.reserve(nn));
    BFQ_CUDA_TRY(w->d_bud_list.reserve(nn));
    BFQ_CUDA_TRY(w->d_bud_ctr.reserve(BUD_CTR_COUNT));
    if (n_tenants > 0) {
        BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_bud_bytes.p, max_pfanout_bytes, (size_t) n_tenants * sizeof(long long), cudaMemcpyHostToDevice, st));
        BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_bud_bw.p, tenant_bandwidth, (size_t) n_tenants, cudaMemcpyHostToDevice, st));
    }
    BFQ_CUDA_TRY(cudaMemsetAsync(w->d_bud_ctr.p, 0, BUD_CTR_COUNT * sizeof(unsigned long long), st));
    BudgetParams q{};
    q.e = expand_params(L, d_offsets, d_ranks, rank_cap);
    q.n_tenants = n_tenants;
    q.msg_bytes = d_msg_bytes;
    q.max_bytes = w->d_bud_bytes.p;
    q.bandwidth = w->d_bud_bw.p;
    q.delivered_p = w->d_bud_dp.p;
    q.flags = w->d_bud_flags.p;
    q.list = w->d_bud_list.p;
    q.ctr = w->d_bud_ctr.p;
    size_t tmp_bytes = 0;
    BFQ_CUDA_TRY(launch_budget(q, nullptr, &tmp_bytes, st, 1));
    BFQ_CUDA_TRY(w->d_scan_tmp.reserve(tmp_bytes + 256));
    BFQ_CUDA_TRY(launch_budget(q, w->d_scan_tmp.p, &tmp_bytes, st, 1));
    long long total = 0;
    unsigned long long ctr[BUD_CTR_COUNT];
    BFQ_CUDA_TRY(cudaMemcpyAsync(&total, d_offsets + n_topics, sizeof(long long), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(ctr, w->d_bud_ctr.p, sizeof(ctr), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    int64_t launches = 2;
    const bool ok = ctr[BUD_BAD_SIZE] == 0;
    if (ok && d_ranks && total <= rank_cap) {
        q.n_listed = (int64_t) ctr[BUD_LISTED];
        BFQ_CUDA_TRY(launch_budget(q, w->d_scan_tmp.p, &tmp_bytes, st, 2));
        launches += 2;
    }
    {
        std::lock_guard<std::mutex> g(h->mu);
        h->launches += launches;
    }
    if (!ok) return fail(BFQ_E_INVALID, std::to_string(ctr[BUD_BAD_SIZE]) + " negative d_msg_bytes entries");
    out->d_delivered_persistent = w->d_bud_dp.p;
    out->d_topic_flags = w->d_bud_flags.p;
    out->n_delivered = (int64_t) total;
    out->n_dropped_bytes = (int64_t) ctr[BUD_DROP_BYTES];
    out->n_dropped_persistent_bandwidth = (int64_t) ctr[BUD_DROP_PBW];
    out->n_dropped_transient_bandwidth = (int64_t) ctr[BUD_DROP_TBW];
    return BFQ_OK;
}

// ---------------------------------------------------------------- fan-out expansion (fanout.cu)
namespace {
// the snapshot's fan-out tables: every tenant's routes resolved to deliverer ids (cached per tenant blob: a delta commit
// re-resolves only the tenants it rebuilt), concatenated in rank order and uploaded once per snapshot
int32_t ensure_fan_table(bfq_index* h, Snapshot* s, std::shared_ptr<Snapshot::FanTable>* out) {
    std::lock_guard<std::mutex> g(s->fan_mu);
    if (s->fan) {
        *out = s->fan;
        return BFQ_OK;
    }
    const size_t T = s->th.size();
    std::vector<std::string> errs(T);
    {
        std::atomic<size_t> cursor{0};
        auto worker = [&]() {
            while (true) {
                const size_t i = cursor.fetch_add(1);
                if (i >= T) break;
                if (s->th[i].fan) continue;
                auto tf = std::make_shared<TenantFan>();
                if (build_tenant_fan(*s->th[i].kv, h->deliverers.get(), tf.get(), &errs[i])) s->th[i].fan = std::move(tf);
            }
        };
        const unsigned nt = (unsigned) std::max<size_t>(1, std::min<size_t>(std::min<size_t>(std::thread::hardware_concurrency(), 64), T));
        std::vector<std::thread> th;
        for (unsigned t = 1; t < nt; t++) th.emplace_back(worker);
        worker();
        for (auto& x : th) x.join();
    }
    for (size_t i = 0; i < T; i++)
        if (!s->th[i].fan) return fail(BFQ_E_INVALID, "fan-out tables: " + errs[i]);
    std::vector<uint32_t> rdeliv((size_t) std::max<int64_t>(s->flat.n_routes, 1), 0), gmem_off(1, 0), gmem_deliv;
    std::vector<uint8_t> gordered;
    for (size_t i = 0; i < T; i++) {
        const TenantFan& tf = *s->th[i].fan;
        const uint32_t gbase = (uint32_t) gordered.size(), mbase = (uint32_t) gmem_deliv.size();
        const int64_t lo = s->flat.tenants[i].lo;
        for (size_t r = 0; r < tf.rdeliv.size(); r++)
            rdeliv[(size_t) lo + r] = (tf.rdeliv[r] & FO_GROUP_BIT) ? (FO_GROUP_BIT | ((tf.rdeliv[r] & ~FO_GROUP_BIT) + gbase)) : tf.rdeliv[r];
        for (size_t k = 1; k < tf.gmem_off.size(); k++) gmem_off.push_back(tf.gmem_off[k] + mbase);
        gmem_deliv.insert(gmem_deliv.end(), tf.gmem_deliv.begin(), tf.gmem_deliv.end());
        gordered.insert(gordered.end(), tf.gordered.begin(), tf.gordered.end());
    }
    auto ft = std::make_shared<Snapshot::FanTable>();
    {
        std::lock_guard<std::mutex> gd(h->deliverers->mu);
        ft->n_deliverers = (uint32_t) h->deliverers->list.size() + 1;
    }
    // ids share rdeliv[] with FO_GROUP_BIT, and n_deliverers and the global pass's n_deliverers + 1 counts are int32
    if (ft->n_deliverers > 0x7FFFFFFEu) return fail(BFQ_E_RANGE, "more than 2^31 - 3 distinct (subBrokerId, delivererKey) pairs on one handle");
    BFQ_CUDA_TRY(ft->d_rdeliv.reserve(rdeliv.size()));
    BFQ_CUDA_TRY(ft->d_gmem_off.reserve(gmem_off.size()));
    BFQ_CUDA_TRY(ft->d_gmem_deliv.reserve(std::max<size_t>(gmem_deliv.size(), 1)));
    BFQ_CUDA_TRY(ft->d_gordered.reserve(std::max<size_t>(gordered.size(), 1)));
    BFQ_CUDA_TRY(cudaMemcpy(ft->d_rdeliv.p, rdeliv.data(), rdeliv.size() * 4, cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(ft->d_gmem_off.p, gmem_off.data(), gmem_off.size() * 4, cudaMemcpyHostToDevice));
    if (!gmem_deliv.empty()) BFQ_CUDA_TRY(cudaMemcpy(ft->d_gmem_deliv.p, gmem_deliv.data(), gmem_deliv.size() * 4, cudaMemcpyHostToDevice));
    if (!gordered.empty()) BFQ_CUDA_TRY(cudaMemcpy(ft->d_gordered.p, gordered.data(), gordered.size(), cudaMemcpyHostToDevice));
    s->fan = ft;
    *out = ft;
    return BFQ_OK;
}

// the snapshot's ordered-group member urls, from the tenants' fan-out tables (call after ensure_fan_table), in the fan table's
// member order: each url at byte 4 of its own run of 8-byte words, so the pick reads LE32(hash) ‖ url as whole words
int32_t ensure_url_table(Snapshot* s, std::shared_ptr<Snapshot::UrlTable>* out) {
    std::lock_guard<std::mutex> g(s->fan_mu);
    if (s->urls) {
        *out = s->urls;
        return BFQ_OK;
    }
    std::vector<unsigned long long> words;
    std::vector<long long> word;
    std::vector<uint32_t> len;
    uint32_t largest = 0;
    for (const auto& th : s->th) {
        const TenantFan& tf = *th.fan;
        for (size_t m = 0; m + 1 < tf.ourl_off.size(); m++) {
            const uint32_t a = tf.ourl_off[m], n = tf.ourl_off[m + 1] - a;
            word.push_back((long long) words.size());
            len.push_back(n);
            if (n == 0) continue;
            const size_t w0 = words.size();
            words.resize(w0 + (4 + (size_t) n + 7) / 8, 0);
            memcpy(reinterpret_cast<uint8_t*>(words.data() + w0) + 4, tf.ourl.data() + a, n);
        }
        for (size_t k = 0; k < tf.gordered.size(); k++)
            if (tf.gordered[k]) largest = std::max(largest, tf.gmem_off[k + 1] - tf.gmem_off[k]);
    }
    auto ut = std::make_shared<Snapshot::UrlTable>();
    ut->member_bits = largest ? 32u - (uint32_t) __builtin_clz(largest) : 1u;
    BFQ_CUDA_TRY(ut->d_words.reserve(std::max<size_t>(words.size(), 1)));
    BFQ_CUDA_TRY(ut->d_word.reserve(std::max<size_t>(word.size(), 1)));
    BFQ_CUDA_TRY(ut->d_len.reserve(std::max<size_t>(len.size(), 1)));
    if (!words.empty()) BFQ_CUDA_TRY(cudaMemcpy(ut->d_words.p, words.data(), words.size() * 8, cudaMemcpyHostToDevice));
    if (!word.empty()) BFQ_CUDA_TRY(cudaMemcpy(ut->d_word.p, word.data(), word.size() * 8, cudaMemcpyHostToDevice));
    if (!len.empty()) BFQ_CUDA_TRY(cudaMemcpy(ut->d_len.p, len.data(), len.size() * 4, cudaMemcpyHostToDevice));
    s->urls = ut;
    *out = ut;
    return BFQ_OK;
}
}  // namespace

int32_t bfq_fanout_device(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs, void* stream,
                          bfq_fanout_result* out) {
    if (!res || !res->lease || !out || !d_offsets || n_pairs < 0 || (n_pairs > 0 && !d_ranks)) return fail(BFQ_E_INVALID, "bad argument");
    auto* L = static_cast<DeviceLease*>(res->lease);
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    int32_t rc = lease_use(res, st, "bfq_fanout_device", &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);   // the call never synchronises: every pass is still queued when it returns
    if (n_pairs >= (int64_t) 0xFFFFFFF0ll) return fail(BFQ_E_RANGE, "more than 2^32 (topic, route) pairs in one batch; split the batch");
    bfq_index* h = L->h;
    Workspace* w = L->ws;
    std::shared_ptr<Snapshot::FanTable> ft;
    rc = ensure_fan_table(h, L->snap.get(), &ft);
    if (rc != BFQ_OK) return rc;
    bool force_global;
    {
        std::lock_guard<std::mutex> g(h->mu);
        force_global = h->fanout_global;
    }
    const bool tiled = !force_global && fanout_tiled(ft->n_deliverers, n_pairs);
    const size_t words = fanout_scratch_words(ft->n_deliverers, n_pairs, tiled);
    BFQ_CUDA_TRY(w->d_fo_counts.reserve(words));
    BFQ_CUDA_TRY(w->d_fo_base.reserve(words));
    BFQ_CUDA_TRY(w->d_pack_offsets.reserve((size_t) ft->n_deliverers + 1));
    BFQ_CUDA_TRY(w->d_pack_topic.reserve((size_t) std::max<int64_t>(n_pairs, 1)));
    BFQ_CUDA_TRY(w->d_pack_rank.reserve((size_t) std::max<int64_t>(n_pairs, 1)));
    BFQ_CUDA_TRY(w->d_pack_member.reserve((size_t) std::max<int64_t>(n_pairs, 1)));
    FanoutParams p{};
    p.n_topics = L->n;
    p.offsets = d_offsets;
    p.n_pairs = n_pairs;
    p.ranks = d_ranks;
    p.rdeliv = ft->d_rdeliv.p;
    p.gmem_off = ft->d_gmem_off.p;
    p.gmem_deliv = ft->d_gmem_deliv.p;
    p.gordered = ft->d_gordered.p;
    p.n_deliverers = ft->n_deliverers;
    p.counts = w->d_fo_counts.p;
    p.base = w->d_fo_base.p;
    p.pack_offsets = w->d_pack_offsets.p;
    p.pack_topic = w->d_pack_topic.p;
    p.pack_rank = w->d_pack_rank.p;
    p.pack_member = w->d_pack_member.p;
    size_t tmp_bytes = 0;
    BFQ_CUDA_TRY(launch_fanout(p, tiled, nullptr, &tmp_bytes, st));
    BFQ_CUDA_TRY(w->d_fo_tmp.reserve(tmp_bytes + 256));
    BFQ_CUDA_TRY(launch_fanout(p, tiled, w->d_fo_tmp.p, &tmp_bytes, st));
    out->d_pack_offsets = (const int64_t*) w->d_pack_offsets.p;
    out->d_pack_topic = w->d_pack_topic.p;
    out->d_pack_rank = w->d_pack_rank.p;
    out->d_pack_member = w->d_pack_member.p;
    out->n_pairs = n_pairs;
    out->n_deliverers = (int32_t) ft->n_deliverers;
    out->ordered_share_id = (int32_t) ft->n_deliverers - 1;
    out->generation = L->snap->generation;
    std::lock_guard<std::mutex> g(h->mu);
    h->launches += 5;
    if (!tiled) h->global_fanouts++;
    return BFQ_OK;
}

namespace {
struct PublisherPacks {   // bfq_delivery_device_ordered's publisher arrays
    const int64_t* pub_off;
    const int32_t* pub_hash;
    int64_t n_pubs;
};

// bfq_delivery_device (pubs == nullptr) and bfq_delivery_device_ordered (pubs and oout set)
int32_t run_delivery_call(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs,
                          const int32_t* d_topic_tenant, void* stream, const char* who, const PublisherPacks* pubs,
                          bfq_delivery_result* out, bfq_delivery_ordered_result* oout) {
    auto* L = static_cast<DeviceLease*>(res->lease);
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    int32_t rc = lease_use(res, st, who, &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);   // the call synchronises after its last launch, but an error return may come before that
    if (L->n > 0 && !d_topic_tenant) return fail(BFQ_E_INVALID, "NULL d_topic_tenant");
    if (pubs && !pubs->pub_off) return fail(BFQ_E_INVALID, "NULL d_pub_off");
    if (pubs && (pubs->n_pubs < 0 || (pubs->n_pubs > 0 && !pubs->pub_hash))) return fail(BFQ_E_INVALID, "bad d_pub_hash / n_pubs");
    if (n_pairs >= (int64_t) 0xFFFFFFF0ll) return fail(BFQ_E_RANGE, "more than 2^32 (topic, route) pairs in one batch; split the batch");
    bfq_index* h = L->h;
    Workspace* w = L->ws;
    w->dl_n_packs = -1;   // the buffers below are about to change
    std::shared_ptr<Snapshot::FanTable> ft;
    rc = ensure_fan_table(h, L->snap.get(), &ft);
    if (rc != BFQ_OK) return rc;
    std::shared_ptr<Snapshot::UrlTable> ut;
    if (pubs && (rc = ensure_url_table(L->snap.get(), &ut)) != BFQ_OK) return rc;
    const int64_t T = L->n;
    DeliveryParams q{};
    q.f.n_topics = T;
    q.f.offsets = d_offsets;
    q.f.n_pairs = n_pairs;
    q.f.ranks = d_ranks;
    q.f.rdeliv = ft->d_rdeliv.p;
    q.f.gmem_off = ft->d_gmem_off.p;
    q.f.gmem_deliv = ft->d_gmem_deliv.p;
    q.f.gordered = ft->d_gordered.p;
    q.f.n_deliverers = ft->n_deliverers;
    q.topic_tenant = d_topic_tenant;
    q.n_tenants = L->ctx.n_tenants;
    int64_t n_items = 0;
    if (pubs) {
        // phase 1: which pairs are $oshare pairs to resolve, how many (pair, publisher) items, and the d_pub_off check
        q.oshare = true;
        q.o.pub_off = pubs->pub_off;
        q.o.pub_hash = pubs->pub_hash;
        q.o.n_pubs = pubs->n_pubs;
        q.o.url_words = ut->d_words.p;
        q.o.url_word = ut->d_word.p;
        q.o.url_len = ut->d_len.p;
        q.o.member_bits = ut->member_bits;
        BFQ_CUDA_TRY(w->d_os_flag.reserve((size_t) n_pairs + 1));
        BFQ_CUDA_TRY(w->d_os_items.reserve((size_t) n_pairs + 1));
        BFQ_CUDA_TRY(w->d_os_check.reserve(4));
        q.o.oflag = w->d_os_flag.p;
        q.o.oitems = w->d_os_items.p;
        q.o.check = w->d_os_check.p;
        size_t tmp_bytes = 0;
        BFQ_CUDA_TRY(launch_oshare_count(q, nullptr, &tmp_bytes, st));
        BFQ_CUDA_TRY(w->d_dl_tmp.reserve(tmp_bytes + 256));
        BFQ_CUDA_TRY(launch_oshare_count(q, w->d_dl_tmp.p, &tmp_bytes, st));
        unsigned long long chk[4];
        BFQ_CUDA_TRY(cudaMemcpyAsync(chk, w->d_os_check.p, sizeof(chk), cudaMemcpyDeviceToHost, st));
        BFQ_CUDA_TRY(cudaStreamSynchronize(st));
        if ((int64_t) chk[3] != n_pairs)
            return fail(BFQ_E_INVALID, "n_pairs = " + std::to_string(n_pairs) + " but d_offsets[n_topics] = " + std::to_string((int64_t) chk[3]));
        if (chk[2]) return fail(BFQ_E_INVALID, "d_pub_off must run from 0 to n_pubs = " + std::to_string(pubs->n_pubs) + " without decreasing");
        if (chk[1] >= 0xFFFFFFF0ull || (uint64_t) n_pairs + chk[1] >= 0xFFFFFFF0ull)
            return fail(BFQ_E_RANGE, "more than 2^32 pairs and ($oshare pair, publisher) items in one batch; split the batch");
        q.o.n_opairs = (int64_t) chk[0];
        n_items = (int64_t) chk[1];
        q.o.n_items = n_items;
    }
    const size_t np = (size_t) std::max<int64_t>(n_pairs + n_items, 1);
    BFQ_CUDA_TRY(w->d_dl_topic_tmp.reserve(6 * (size_t) T + 2));
    BFQ_CUDA_TRY(w->d_dl_pair_tmp.reserve(10 * np + 2));
    BFQ_CUDA_TRY(w->d_dl_pcount.reserve((size_t) ft->n_deliverers + 1));
    BFQ_CUDA_TRY(w->d_dl_totals.reserve(5));
    BFQ_CUDA_TRY(w->d_package_off.reserve((size_t) ft->n_deliverers + 1));
    BFQ_CUDA_TRY(w->d_package_tenant.reserve(np));
    BFQ_CUDA_TRY(w->d_dl_pack_off.reserve(np + 1));
    BFQ_CUDA_TRY(w->d_dl_pack_topic.reserve(np));
    BFQ_CUDA_TRY(w->d_match_off.reserve(np + 1));
    BFQ_CUDA_TRY(w->d_match_rank.reserve(np));
    BFQ_CUDA_TRY(w->d_match_member.reserve(np));
    uint32_t* tt = w->d_dl_topic_tmp.p;
    q.tkey[0] = tt;
    q.tkey[1] = tt + T;
    q.tval[0] = tt + 2 * T;
    q.tval[1] = tt + 3 * T;
    q.tcount = tt + 4 * T;
    q.tstart = tt + 5 * T + 1;
    uint32_t* pt = w->d_dl_pair_tmp.p;
    q.key[0] = pt;
    q.key[1] = pt + np;
    q.val[0] = pt + 2 * np;
    q.val[1] = pt + 3 * np;
    q.e_topic = pt + 4 * np;
    q.e_rank = pt + 5 * np;
    q.e_member = pt + 6 * np;
    q.s_topic = pt + 7 * np;
    q.package_head = pt + 8 * np;
    q.pack_head = pt + 9 * np + 1;
    q.pcount = w->d_dl_pcount.p;
    q.totals = w->d_dl_totals.p;
    q.package_off = w->d_package_off.p;
    q.package_tenant = w->d_package_tenant.p;
    q.pack_off = w->d_dl_pack_off.p;
    q.pack_topic = w->d_dl_pack_topic.p;
    q.match_off = w->d_match_off.p;
    q.match_rank = w->d_match_rank.p;
    q.match_member = w->d_match_member.p;
    if (pubs) {
        const size_t O = (size_t) q.o.n_opairs, I = (size_t) n_items;
        BFQ_CUDA_TRY(w->d_os_key.reserve(std::max<size_t>(2 * O + 2 * I, 1)));
        BFQ_CUDA_TRY(w->d_os_u32.reserve((O + 1) + 2 * I + 2 * (I + 1) + I + 3 * np + 1));
        BFQ_CUDA_TRY(w->d_pack_pub.reserve(std::max<size_t>(I, 1)));
        BFQ_CUDA_TRY(w->d_pack_pub_off.reserve(np + 1));
        unsigned long long* kp = w->d_os_key.p;
        q.o.okey[0] = kp;
        q.o.okey[1] = kp + O;
        q.o.ikey[0] = kp + 2 * O;
        q.o.ikey[1] = kp + 2 * O + I;
        uint32_t* up = w->d_os_u32.p;
        q.o.istart = up;
        up += O + 1;
        q.o.ival[0] = up;
        q.o.ival[1] = up + I;
        up += 2 * I;
        q.o.ihead = up;
        up += I + 1;
        q.o.sub_start = up;
        up += I + 1;
        q.o.sub_pack = up;
        up += I;
        q.o.e_sub = up;
        q.o.s_sub = up + np;
        q.o.pub_count = up + 2 * np;
        q.o.pack_pub_off = w->d_pack_pub_off.p;
        q.o.pack_pub = w->d_pack_pub.p;
    }
    size_t tmp_bytes = 0;
    BFQ_CUDA_TRY(launch_delivery(q, nullptr, &tmp_bytes, st));
    BFQ_CUDA_TRY(w->d_dl_tmp.reserve(tmp_bytes + 256));
    BFQ_CUDA_TRY(launch_delivery(q, w->d_dl_tmp.p, &tmp_bytes, st));
    unsigned long long tot[5] = {0, 0, 0, 0, 0};
    BFQ_CUDA_TRY(cudaMemcpyAsync(tot, w->d_dl_totals.p, (pubs ? 5 : 4) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    {
        std::lock_guard<std::mutex> g(h->mu);
        h->launches += pubs ? 25 : 11;
    }
    if ((int64_t) tot[3] != n_pairs)
        return fail(BFQ_E_INVALID, "n_pairs = " + std::to_string(n_pairs) + " but d_offsets[n_topics] = " + std::to_string((int64_t) tot[3]));
    out->d_package_off = (const int64_t*) w->d_package_off.p;
    out->d_package_tenant = w->d_package_tenant.p;
    out->d_pack_off = (const int64_t*) w->d_dl_pack_off.p;
    out->d_pack_topic = w->d_dl_pack_topic.p;
    out->d_match_off = (const int64_t*) w->d_match_off.p;
    out->d_match_rank = w->d_match_rank.p;
    out->d_match_member = w->d_match_member.p;
    out->n_pairs = (int64_t) tot[0];
    out->n_packages = (int64_t) tot[1];
    out->n_packs = (int64_t) tot[2];
    out->n_deliverers = (int32_t) ft->n_deliverers;
    out->ordered_share_id = (int32_t) ft->n_deliverers - 1;
    out->generation = L->snap->generation;
    w->dl_n_pairs = out->n_pairs;
    w->dl_n_packages = out->n_packages;
    w->dl_n_packs = out->n_packs;
    w->dl_ordered = pubs != nullptr;
    if (oout) {
        oout->d_pack_pub_off = (const int64_t*) w->d_pack_pub_off.p;
        oout->d_pack_pub = w->d_pack_pub.p;
        oout->n_pack_pubs = n_items;
        oout->n_ordered_packs = (int64_t) tot[4];
    }
    return BFQ_OK;
}
}  // namespace

int32_t bfq_delivery_device(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs,
                            const int32_t* d_topic_tenant, void* stream, bfq_delivery_result* out) {
    if (!res || !res->lease || !out || !d_offsets || n_pairs < 0 || (n_pairs > 0 && !d_ranks)) return fail(BFQ_E_INVALID, "bad argument");
    return run_delivery_call(res, d_offsets, d_ranks, n_pairs, d_topic_tenant, stream, "bfq_delivery_device", nullptr, out, nullptr);
}

int32_t bfq_delivery_device_ordered(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs,
                                    const int32_t* d_topic_tenant, const int64_t* d_pub_off, const int32_t* d_pub_hash, int64_t n_pubs,
                                    void* stream, bfq_delivery_ordered_result* out) {
    if (!res || !res->lease || !out || !d_offsets || n_pairs < 0 || (n_pairs > 0 && !d_ranks)) return fail(BFQ_E_INVALID, "bad argument");
    const PublisherPacks pubs{d_pub_off, d_pub_hash, n_pubs};
    return run_delivery_call(res, d_offsets, d_ranks, n_pairs, d_topic_tenant, stream, "bfq_delivery_device_ordered", &pubs, &out->d,
                             out);
}

namespace {
// the snapshot's MatchInfo table: every tenant's entries (cached per tenant blob, so a delta commit re-encodes only the tenants it
// rebuilt), concatenated in rank order and uploaded once per snapshot
int32_t ensure_wire_table(Snapshot* s, std::shared_ptr<Snapshot::WireTable>* out) {
    std::lock_guard<std::mutex> g(s->fan_mu);
    if (s->wire) {
        *out = s->wire;
        return BFQ_OK;
    }
    const size_t T = s->th.size();
    std::vector<std::string> errs(T);
    {
        std::atomic<size_t> cursor{0};
        auto worker = [&]() {
            while (true) {
                const size_t i = cursor.fetch_add(1);
                if (i >= T) break;
                if (s->th[i].wire) continue;
                auto tw = std::make_shared<TenantWire>();
                if (build_tenant_wire(*s->th[i].kv, tw.get(), &errs[i])) s->th[i].wire = std::move(tw);
            }
        };
        const unsigned nt = (unsigned) std::max<size_t>(1, std::min<size_t>(std::min<size_t>(std::thread::hardware_concurrency(), 64), T));
        std::vector<std::thread> th;
        for (unsigned t = 1; t < nt; t++) th.emplace_back(worker);
        worker();
        for (auto& x : th) x.join();
    }
    size_t entries = 0, bytes = 0;
    for (size_t i = 0; i < T; i++) {
        if (!s->th[i].wire) return fail(BFQ_E_INVALID, "MatchInfo table: " + errs[i]);
        entries += s->th[i].wire->off.size() - 1;
        bytes += s->th[i].wire->bytes.size();
    }
    if (entries >= 0xFFFFFFFFull) return fail(BFQ_E_RANGE, "2^32 or more MatchInfos in one snapshot");
    std::vector<uint32_t> first((size_t) std::max<int64_t>(s->flat.n_routes, 1), 0);
    std::vector<unsigned long long> off(1, 0);
    off.reserve(entries + 1);
    std::vector<uint8_t> blob;
    blob.reserve(bytes);
    for (size_t i = 0; i < T; i++) {
        const TenantWire& tw = *s->th[i].wire;
        const uint32_t ebase = (uint32_t) (off.size() - 1);
        const unsigned long long bbase = blob.size();
        const int64_t lo = s->flat.tenants[i].lo;
        for (size_t r = 0; r < tw.first.size(); r++) first[(size_t) lo + r] = tw.first[r] + ebase;
        for (size_t e = 1; e < tw.off.size(); e++) off.push_back(tw.off[e] + bbase);
        blob.insert(blob.end(), tw.bytes.begin(), tw.bytes.end());
    }
    auto wt = std::make_shared<Snapshot::WireTable>();
    BFQ_CUDA_TRY(wt->d_first.reserve(first.size()));
    BFQ_CUDA_TRY(wt->d_off.reserve(off.size()));
    BFQ_CUDA_TRY(wt->d_bytes.reserve(std::max<size_t>(blob.size(), 1)));
    BFQ_CUDA_TRY(cudaMemcpy(wt->d_first.p, first.data(), first.size() * 4, cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(wt->d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice));
    if (!blob.empty()) BFQ_CUDA_TRY(cudaMemcpy(wt->d_bytes.p, blob.data(), blob.size(), cudaMemcpyHostToDevice));
    wt->n_entries = entries;
    s->wire = wt;
    s->wire_bytes = wt->bytes();
    *out = wt;
    return BFQ_OK;
}

// the nesting is the one the last delivery call on this result left in its workspace (plain or ordered)
bool latest_nesting(const DeviceLease* L, const bfq_delivery_result* nest) {
    const Workspace* w = L->ws;
    return nest->generation == L->snap->generation && nest->d_package_off == (const int64_t*) w->d_package_off.p &&
           nest->d_match_off == (const int64_t*) w->d_match_off.p && w->dl_n_packs >= 0 && nest->n_packs == w->dl_n_packs &&
           nest->n_packages == w->dl_n_packages && nest->n_pairs == w->dl_n_pairs;
}

// bfq_delivery_encode (oout == nullptr) and bfq_delivery_encode_ordered: nest is the nesting's plain part either way
int32_t run_encode(const bfq_device_result* res, const bfq_delivery_result* nest, const bfq_delivery_ordered_result* onest,
                   const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_topics,
                   const int64_t* d_topic_off, const int64_t* d_pub_off, const uint8_t* d_pubpack_bytes,
                   const int64_t* d_pubpack_off, uint8_t* d_out, int64_t out_cap, void* stream, const char* who,
                   bfq_delivery_wire_result* out) {
    if (!res || !res->lease || !nest || !out || out_cap < 0) return fail(BFQ_E_INVALID, "bad argument");
    auto* L = static_cast<DeviceLease*>(res->lease);
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    int32_t rc = lease_use(res, st, who, &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);   // the write pass is still running when the call returns
    if (!d_topics || !d_topic_off || !d_pub_off || !d_pubpack_bytes || !d_pubpack_off)
        return fail(BFQ_E_INVALID, std::string(who) + ": NULL topic or publisher pack array");
    if (n_tenants != L->ctx.n_tenants || (n_tenants > 0 && (!tenants || !tenant_off)))
        return fail(BFQ_E_INVALID, std::string(who) + ": the tenant list must be the match's (" + std::to_string(L->ctx.n_tenants) + " tenants)");
    Workspace* w = L->ws;
    if (!latest_nesting(L, nest) || w->dl_ordered != (onest != nullptr) ||
        (onest && onest->d_pack_pub_off != (const int64_t*) w->d_pack_pub_off.p))
        return fail(BFQ_E_RANGE, std::string(who) + ": the nesting is not the latest " +
                                     (onest ? "bfq_delivery_device_ordered" : "bfq_delivery_device") + " result of this device result");
    bfq_index* h = L->h;
    std::shared_ptr<Snapshot::WireTable> wt;
    if ((rc = ensure_wire_table(L->snap.get(), &wt)) != BFQ_OK) return rc;
    const int64_t np = nest->n_pairs, nk = nest->n_packs, ng = nest->n_packages;
    const uint32_t D = (uint32_t) nest->n_deliverers;
    BFQ_CUDA_TRY(w->d_wr_pos.reserve((size_t) (np + 1 + nk + 1 + ng + 1)));
    BFQ_CUDA_TRY(w->d_wr_check.reserve(4));
    BFQ_CUDA_TRY(w->d_req_off.reserve((size_t) D + 1));
    BFQ_CUDA_TRY(w->d_wr_tenant_off.reserve((size_t) n_tenants + 1));
    const int64_t tbytes = n_tenants > 0 ? tenant_off[n_tenants] : 0;
    BFQ_CUDA_TRY(w->d_wr_tenants.reserve((size_t) std::max<int64_t>(tbytes, 1)));
    if (n_tenants > 0) {
        BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_wr_tenant_off.p, tenant_off, ((size_t) n_tenants + 1) * 8, cudaMemcpyHostToDevice, st));
        if (tbytes > 0) BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_wr_tenants.p, tenants, (size_t) tbytes, cudaMemcpyHostToDevice, st));
    }
    WireParams p{};
    p.n_packages = ng;
    p.n_packs = nk;
    p.n_pairs = np;
    p.n_deliverers = D;
    p.package_off = (const long long*) nest->d_package_off;
    p.package_tenant = nest->d_package_tenant;
    p.pack_off = (const long long*) nest->d_pack_off;
    p.pack_topic = nest->d_pack_topic;
    p.match_off = (const long long*) nest->d_match_off;
    p.match_rank = nest->d_match_rank;
    p.match_member = nest->d_match_member;
    p.pack_pub_off = onest ? (const long long*) onest->d_pack_pub_off : nullptr;
    p.pack_pub = onest ? onest->d_pack_pub : nullptr;
    p.tenants = w->d_wr_tenants.p;
    p.tenant_off = w->d_wr_tenant_off.p;
    p.topics = d_topics;
    p.topic_off = (const long long*) d_topic_off;
    p.n_topics = L->n;
    p.pub_off = (const long long*) d_pub_off;
    p.pubpack = d_pubpack_bytes;
    p.pubpack_off = (const long long*) d_pubpack_off;
    p.mi_first = wt->d_first.p;
    p.mi_off = wt->d_off.p;
    p.mi_bytes = wt->d_bytes.p;
    p.pair_pos = w->d_wr_pos.p;
    p.pack_pos = p.pair_pos + np + 1;
    p.package_pos = p.pack_pos + nk + 1;
    p.check = w->d_wr_check.p;
    p.req_off = w->d_req_off.p;
    p.out = d_out;
    size_t tmp_bytes = 0;
    BFQ_CUDA_TRY(launch_wire_size(p, nullptr, &tmp_bytes, st));
    BFQ_CUDA_TRY(w->d_wr_tmp.reserve(tmp_bytes + 256));
    BFQ_CUDA_TRY(launch_wire_size(p, w->d_wr_tmp.p, &tmp_bytes, st));
    unsigned long long chk[4];
    BFQ_CUDA_TRY(cudaMemcpyAsync(chk, w->d_wr_check.p, sizeof(chk), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    if (chk[0]) return fail(BFQ_E_INVALID, std::string(who) + ": d_pub_off / d_pubpack_off must start at 0 and never decrease, and "
                                                               "every publisher of the nesting must be below d_pub_off[n_topics]");
    const bool write = d_out && (int64_t) chk[1] <= out_cap;
    if (write) BFQ_CUDA_TRY(launch_wire_write(p, st));
    {
        std::lock_guard<std::mutex> g(h->mu);
        h->launches += write ? 10 : 8;
    }
    out->d_req_off = (const int64_t*) w->d_req_off.p;
    out->n_bytes = (int64_t) chk[1];
    out->n_match_infos = (int64_t) chk[2];
    out->n_skipped = np - (int64_t) chk[2];
    out->n_deliverers = (int32_t) D;
    out->ordered_share_id = (int32_t) D - 1;
    out->generation = L->snap->generation;
    return BFQ_OK;
}
}  // namespace

int32_t bfq_delivery_encode(const bfq_device_result* res, const bfq_delivery_result* nesting, const uint8_t* tenants,
                            const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_topics, const int64_t* d_topic_off,
                            const int64_t* d_pub_off, const uint8_t* d_pubpack_bytes, const int64_t* d_pubpack_off, uint8_t* d_out,
                            int64_t out_cap, void* stream, bfq_delivery_wire_result* out) {
    return run_encode(res, nesting, nullptr, tenants, tenant_off, n_tenants, d_topics, d_topic_off, d_pub_off, d_pubpack_bytes,
                      d_pubpack_off, d_out, out_cap, stream, "bfq_delivery_encode", out);
}

int32_t bfq_delivery_encode_ordered(const bfq_device_result* res, const bfq_delivery_ordered_result* nesting, const uint8_t* tenants,
                                    const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_topics, const int64_t* d_topic_off,
                                    const int64_t* d_pub_off, const uint8_t* d_pubpack_bytes, const int64_t* d_pubpack_off,
                                    uint8_t* d_out, int64_t out_cap, void* stream, bfq_delivery_wire_result* out) {
    return run_encode(res, nesting ? &nesting->d : nullptr, nesting, tenants, tenant_off, n_tenants, d_topics, d_topic_off, d_pub_off,
                      d_pubpack_bytes, d_pubpack_off, d_out, out_cap, stream, "bfq_delivery_encode_ordered", out);
}

namespace {
// the hash of every MatchInfo in the snapshot's table (bfq_delivery_reply's join key), built once per snapshot on `st`
int32_t ensure_mi_hash(Snapshot* s, const Snapshot::WireTable& wt, cudaStream_t st, std::shared_ptr<DeviceBuf<uint32_t>>* out) {
    std::lock_guard<std::mutex> g(s->fan_mu);
    if (!s->mi_hash) {
        auto hb = std::make_shared<DeviceBuf<uint32_t>>();
        BFQ_CUDA_TRY(hb->reserve(std::max<size_t>(wt.n_entries, 1)));
        BFQ_CUDA_TRY(launch_mi_hash(wt.d_bytes.p, wt.d_off.p, (int64_t) wt.n_entries, hb->p, st));
        BFQ_CUDA_TRY(cudaStreamSynchronize(st));   // other streams read it from now on
        s->mi_hash = hb;
    }
    *out = s->mi_hash;
    return BFQ_OK;
}
}  // namespace

int32_t bfq_delivery_reply(const bfq_device_result* res, const bfq_delivery_result* nest, const uint8_t* tenants,
                           const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_reply, const int64_t* d_reply_off,
                           void* stream, bfq_delivery_reply_result* out) {
    const char* who = "bfq_delivery_reply";
    if (!res || !res->lease || !nest || !out) return fail(BFQ_E_INVALID, "bad argument");
    auto* L = static_cast<DeviceLease*>(res->lease);
    cudaStream_t st = (cudaStream_t) stream;
    cudaEvent_t ev = nullptr;
    int32_t rc = lease_use(res, st, who, &ev);
    if (rc != BFQ_OK) return rc;
    RecordOnExit rec(ev, st);
    if (!d_reply || !d_reply_off) return fail(BFQ_E_INVALID, std::string(who) + ": NULL reply array");
    if (n_tenants != L->ctx.n_tenants || (n_tenants > 0 && (!tenants || !tenant_off)))
        return fail(BFQ_E_INVALID, std::string(who) + ": the tenant list must be the match's (" + std::to_string(L->ctx.n_tenants) + " tenants)");
    if (!latest_nesting(L, nest))
        return fail(BFQ_E_RANGE, std::string(who) + ": the nesting is not the latest delivery nesting of this device result");
    bfq_index* h = L->h;
    Workspace* w = L->ws;
    std::shared_ptr<Snapshot::WireTable> wt;
    if ((rc = ensure_wire_table(L->snap.get(), &wt)) != BFQ_OK) return rc;
    std::shared_ptr<DeviceBuf<uint32_t>> mh;
    if ((rc = ensure_mi_hash(L->snap.get(), *wt, st, &mh)) != BFQ_OK) return rc;
    const int64_t np = nest->n_pairs, nk = nest->n_packs, ng = nest->n_packages;
    const uint32_t D = (uint32_t) nest->n_deliverers;
    if (np >= (int64_t) 1 << 31) return fail(BFQ_E_RANGE, std::string(who) + ": 2^31 or more pairs in one nesting");
    uint64_t T = 2;
    while (T < 2 * (uint64_t) np) T <<= 1;
    const int64_t cap = std::max<int64_t>(np, 1), G = std::max<int64_t>(ng, 1);
    const uint64_t nch = RP_MAX_CHUNKS + (uint64_t) ng;
    BFQ_CUDA_TRY(w->d_rp_ctr.reserve(RP_CTR_N));
    BFQ_CUDA_TRY(w->h_rp_ctr.reserve(RP_CTR_N));
    BFQ_CUDA_TRY(w->d_rp_chunk_base.reserve((size_t) ng + 1));
    BFQ_CUDA_TRY(w->d_rp_slot_key.reserve(T));
    BFQ_CUDA_TRY(w->d_rp_slot_rpos.reserve(T));
    BFQ_CUDA_TRY(w->d_rp_pkg_stale.reserve(2 * ((size_t) ng + 1)));
    BFQ_CUDA_TRY(w->d_rp_dl_fail.reserve(D));
    BFQ_CUDA_TRY(w->d_rp_ent_bad.reserve((size_t) G));
    BFQ_CUDA_TRY(w->d_rp_pair_code.reserve((size_t) cap));
    BFQ_CUDA_TRY(w->d_rp_status.reserve(D));
    BFQ_CUDA_TRY(w->d_rp_dl_code.reserve(D));
    BFQ_CUDA_TRY(w->d_rp_u32.reserve((size_t) D + 2 * (size_t) G + 3 * T + (size_t) cap * 6));
    BFQ_CUDA_TRY(w->d_rp_ent.reserve(4 * (size_t) G));
    BFQ_CUDA_TRY(w->d_rp_chunks.reserve(3 * nch));
    BFQ_CUDA_TRY(w->d_rp_stale.reserve((size_t) cap));
    BFQ_CUDA_TRY(w->d_rp_tenant_off.reserve((size_t) n_tenants + 1));
    const int64_t tbytes = n_tenants > 0 ? tenant_off[n_tenants] : 0;
    BFQ_CUDA_TRY(w->d_rp_tenants.reserve((size_t) std::max<int64_t>(tbytes, 1)));
    if (n_tenants > 0) {
        BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_rp_tenant_off.p, tenant_off, ((size_t) n_tenants + 1) * 8, cudaMemcpyHostToDevice, st));
        if (tbytes > 0) BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_rp_tenants.p, tenants, (size_t) tbytes, cudaMemcpyHostToDevice, st));
    }
    ReplyParams p{};
    p.n_packages = ng;
    p.n_packs = nk;
    p.n_pairs = np;
    p.n_deliverers = D;
    p.package_off = (const long long*) nest->d_package_off;
    p.package_tenant = nest->d_package_tenant;
    p.pack_off = (const long long*) nest->d_pack_off;
    p.match_off = (const long long*) nest->d_match_off;
    p.match_rank = nest->d_match_rank;
    p.match_member = nest->d_match_member;
    p.tenants = w->d_rp_tenants.p;
    p.tenant_off = w->d_rp_tenant_off.p;
    p.mi_first = wt->d_first.p;
    p.mi_off = wt->d_off.p;
    p.mi_bytes = wt->d_bytes.p;
    p.mi_hash = mh->p;
    p.reply = d_reply;
    p.reply_off = (const long long*) d_reply_off;
    p.ctr = w->d_rp_ctr.p;
    p.dl_fail = w->d_rp_dl_fail.p;
    p.dl_code = w->d_rp_dl_code.p;
    uint32_t* u = w->d_rp_u32.p;
    p.dl_entries = u;
    u += D;
    p.ent_pkg = u;
    u += G;
    p.pkg_claimed = u;
    u += G;
    p.slot_pair = u;
    u += T;
    p.slot_code = u;
    u += T;
    p.slot_rlen = u;
    u += T;
    p.pair_slot = u;
    u += cap;
    p.stale_list = u;
    u += cap;
    p.sort_key_in = u;
    u += cap;
    p.sort_key_out = u;
    u += cap;
    p.sort_val_in = u;
    u += cap;
    p.sort_val_out = u;
    p.ent_s = w->d_rp_ent.p;
    p.ent_e = p.ent_s + G;
    p.ent_vs = p.ent_e + G;
    p.ent_ve = p.ent_vs + G;
    p.ent_bad = w->d_rp_ent_bad.p;
    p.chunk_base = w->d_rp_chunk_base.p;
    p.ch_guess = w->d_rp_chunks.p;
    p.ch_exit = p.ch_guess + nch;
    p.ch_start = p.ch_exit + nch;
    p.slot_key = w->d_rp_slot_key.p;
    p.slot_rpos = w->d_rp_slot_rpos.p;
    p.table_mask = T - 1;
    p.pkg_stale = w->d_rp_pkg_stale.p;
    p.pkg_cursor = p.pkg_stale + ng + 1;
    p.stale_cap = cap;
    p.pair_code = w->d_rp_pair_code.p;
    p.status = w->d_rp_status.p;
    p.stale = w->d_rp_stale.p;
    size_t tmp_bytes = 0;
    BFQ_CUDA_TRY(launch_reply(p, nullptr, &tmp_bytes, st));
    BFQ_CUDA_TRY(w->d_rp_tmp.reserve(tmp_bytes + 256));
    BFQ_CUDA_TRY(launch_reply(p, w->d_rp_tmp.p, &tmp_bytes, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_rp_ctr.p, w->d_rp_ctr.p, RP_CTR_N * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    {
        std::lock_guard<std::mutex> g(h->mu);
        h->launches += 17;
    }
    const unsigned long long* c = w->h_rp_ctr.p;
    if (c[RP_BAD_OFF]) return fail(BFQ_E_INVALID, std::string(who) + ": d_reply_off must never decrease");
    out->d_pair_code = w->d_rp_pair_code.p;
    out->d_status = w->d_rp_status.p;
    out->d_stale = w->d_rp_stale.p;
    for (int i = 0; i < 8; i++) out->n_code[i] = (int64_t) c[RP_N_CODE + i];
    out->n_pairs = np;
    out->n_stale = (int64_t) c[RP_N_STALE];
    out->n_fallback = (int32_t) c[RP_N_FALLBACK];
    out->n_deliverers = (int32_t) D;
    out->ordered_share_id = (int32_t) D - 1;
    out->generation = L->snap->generation;
    return BFQ_OK;
}

int32_t bfq_fanout_deliverer(bfq_index* h, int32_t id, int32_t* sub_broker_id, uint8_t* key_out, int64_t key_cap, int64_t* key_len) {
    if (!h || id < 0) return fail(BFQ_E_INVALID, "bad argument");
    std::lock_guard<std::mutex> g(h->deliverers->mu);
    if ((size_t) id >= h->deliverers->list.size()) return fail(BFQ_E_RANGE, "deliverer id out of range (the last id of a fan-out result is the ordered-share marker)");
    const auto& e = h->deliverers->list[(size_t) id];
    if (sub_broker_id) *sub_broker_id = e.first;
    if (key_len) *key_len = (int64_t) e.second.size();
    if (key_out && (int64_t) e.second.size() <= key_cap) memcpy(key_out, e.second.data(), e.second.size());
    return BFQ_OK;
}

// ---------------------------------------------------------------- codec exports
int64_t bfq_receiver_url(int32_t sub_broker_id, const uint8_t* receiver_id, int64_t rn, const uint8_t* deliverer_key,
                         int64_t dn, uint8_t* out, int64_t cap) {
    return emit_bytes(make_receiver_url(sub_broker_id, sv((const char*) receiver_id, (size_t) rn), sv((const char*) deliverer_key, (size_t) dn)), out, cap);
}
int64_t bfq_route_key(const uint8_t* tenant, int64_t tn, const uint8_t* tf, int64_t fn, const uint8_t* url, int64_t un,
                      uint8_t* out, int64_t cap) {
    return emit_bytes(make_route_key(sv((const char*) tenant, (size_t) tn), sv((const char*) tf, (size_t) fn), sv((const char*) url, (size_t) un)), out, cap);
}
int64_t bfq_retain_key(const uint8_t* tenant, int64_t tn, const uint8_t* topic, int64_t n, uint8_t* out, int64_t cap) {
    return emit_bytes(make_retain_key(sv((const char*) tenant, (size_t) tn), sv((const char*) topic, (size_t) n)), out, cap);
}
int64_t bfq_retain_key_prefix(const uint8_t* tenant, int64_t tn, const uint8_t* tf, int64_t fn, uint8_t* out, int64_t cap) {
    return emit_bytes(make_retain_key_prefix(sv((const char*) tenant, (size_t) tn), sv((const char*) tf, (size_t) fn)), out, cap);
}
int64_t bfq_tenant_begin_key(const uint8_t* tenant, int64_t tn, uint8_t* out, int64_t cap) {
    return emit_bytes(make_tenant_begin_key(sv((const char*) tenant, (size_t) tn)), out, cap);
}
int32_t bfq_is_valid_topic(const uint8_t* topic, int64_t n, int32_t a, int32_t b, int32_t c) {
    return is_valid_topic(sv((const char*) topic, (size_t) n), a, b, c) ? 1 : 0;
}
int32_t bfq_is_valid_topic_filter(const uint8_t* tf, int64_t n, int32_t a, int32_t b, int32_t c) {
    return is_valid_topic_filter(sv((const char*) tf, (size_t) n), a, b, c) ? 1 : 0;
}

}  // extern "C"
