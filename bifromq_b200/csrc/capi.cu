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
#include "index_state.h"
#include "fanout.h"
#include "match_kernels.cuh"

using namespace bfq;

struct bfq_result {
    bfq_index* owner = nullptr;
    std::shared_ptr<Pool<Workspace>> pool;
    std::shared_ptr<Snapshot> snap;      // the snapshot the match ran on (ranks resolve against it)
    Workspace* ws = nullptr;             // leased: the arrays below live in its pinned buffers
    int64_t n_topics = 0, n_ranges = 0, n_throttled = 0;
    const uint32_t *span_begin = nullptr, *span_count = nullptr, *route_count = nullptr;
    const bfq_range* ranges = nullptr;
    const bfq_throttled* throttled = nullptr;
    double ms[4] = {0, 0, 0, 0};
};

namespace {

int32_t acquire(bfq_index* h, std::shared_ptr<Snapshot>* snap, Workspace** ws, const char* who) {
    {
        std::lock_guard<std::mutex> g(h->mu);
        if (!h->snap) return fail(BFQ_E_STATE, std::string(who) + " before the first bfq_index_commit");
        *snap = h->snap;
    }
    const int32_t rc = h->pool->acquire(ws);
    if (rc != BFQ_OK) return rc;
    (*ws)->dl_n_packs = -1;   // a new lease starts without a delivery nesting: one left by the previous lease is not this result's
    return BFQ_OK;
}


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
            // the old scratch is freed: tier 2 may still run on it on the workspace's other work stream, or on the device
            // path, on the caller's stream the match runs on
            BFQ_CUDA_TRY(w->drain());
            if (done) BFQ_CUDA_TRY(cudaStreamSynchronize(stream));
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

// grows the buffers a retry asked for (the caller has waited for every stream that writes them)
int32_t grow_for_retry(Workspace* w, const CoreOut& co, int64_t n, int C) {
    if (co.want_dyn) {
        const size_t want = (size_t) ((uint64_t) n * INLINE_RANGES + (co.want_dyn + co.want_dyn / 4 + 1024) * (uint64_t) C);
        if (want >= 0xFFFFFFF0ull) return fail(BFQ_E_RANGE, "more than 2^32 matched ranges in one batch; split the batch");
        BFQ_CUDA_TRY(w->d_ranges.reserve(want));
    }
    if (co.want_thr) BFQ_CUDA_TRY(w->d_throttled.reserve((size_t) ((co.want_thr + co.want_thr / 4 + 1024) * (uint64_t) C)));
    return BFQ_OK;
}


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
        // the buffers that grow are written by the match alone, on the caller's stream
        if (cudaStreamSynchronize(L->ctx.stream) != cudaSuccess) return L->rc = fail(BFQ_E_CUDA, "cudaStreamSynchronize");
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
    CallLease<Workspace> lease(*h->pool);   // the workspace goes back to the pool on every error path; on success the result keeps it
    int32_t rc = acquire(h, &snap, &lease.w, "bfq_match");
    if (rc != BFQ_OK) return rc;
    Workspace* w = lease.w;
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
                BFQ_CUDA_TRY(w->drain());
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
        BFQ_CUDA_TRY(w->drain());
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
    r->ws = lease.take();   // the result holds the workspace from here on
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
    r->pool->give_back(r->ws);
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
        h->pool->give_back(L->ws);
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
    L->uses.wait(L->ws->use_events);
    L->pool->give_back(L->ws);
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
