// result_calls.cu — the calls on a completed device result (include/bfq_gpumatch.h): the expand and its delivery budgets, the
// fan-out, the delivery nesting (plain and $oshare), its DeliveryRequest bytes, the DeliveryReply join, and the per-snapshot
// tables they build on first use. Each call family lays its scratch and outputs out in one arena of the leased workspace.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <numeric>
#include <optional>
#include <string>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "cuda_buf.h"
#include "fanout.h"
#include "index_builder.h"
#include "index_state.h"
#include "lease.h"
#include "match_kernels.cuh"

using namespace bfq;

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

// The start of every call here (res and res->lease already checked): the lease, its handle and workspace, the call's stream,
// and lease_use's verdict in rc. Once lease_use accepts the result, the result's event for the stream is recorded on every
// return (RecordOnExit), so that release waits for whatever the call leaves queued.
struct ResultCall {
    DeviceLease* L;
    bfq_index* h;
    Workspace* w;
    cudaStream_t st;
    int32_t rc;
    std::optional<RecordOnExit> rec;
    ResultCall(const bfq_device_result* res, void* stream, const char* who)
        : L(static_cast<DeviceLease*>(res->lease)), h(L->h), w(L->ws), st((cudaStream_t) stream) {
        cudaEvent_t ev = nullptr;
        rc = lease_use(res, st, who, &ev);
        if (rc == BFQ_OK) rec.emplace(ev, st);
    }
};

void add_launches(bfq_index* h, int64_t n, int64_t global_fanouts = 0) {
    std::lock_guard<std::mutex> g(h->mu);
    h->launches += n;
    h->global_fanouts += global_fanouts;
}

// A launch that takes cub scratch: launch(tmp, &tmp_bytes) once with tmp == nullptr to ask the size, then on `tmp` grown to fit
template <typename Launch>
int32_t launch_with_temp(DeviceBuf<uint8_t>& tmp, size_t& tmp_bytes, const char* what, Launch&& launch) {
    tmp_bytes = 0;
    cudaError_t e = launch(nullptr, &tmp_bytes);
    if (e == cudaSuccess) e = tmp.reserve(tmp_bytes + 256);
    if (e == cudaSuccess) e = launch(tmp.p, &tmp_bytes);
    return e == cudaSuccess ? BFQ_OK : fail(BFQ_E_CUDA, std::string(what) + ": " + cudaGetErrorString(e));
}

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

// the fan-out's inputs: the caller's CSR of a completed device match and the snapshot's fan-out tables
FanoutParams fanout_inputs(const DeviceLease* L, const Snapshot::FanTable& ft, const int64_t* d_offsets, const int64_t* d_ranks,
                           int64_t n_pairs) {
    FanoutParams p{};
    p.n_topics = L->n;
    p.offsets = d_offsets;
    p.n_pairs = n_pairs;
    p.ranks = d_ranks;
    p.rdeliv = ft.d_rdeliv.p;
    p.gmem_off = ft.d_gmem_off.p;
    p.gmem_deliv = ft.d_gmem_deliv.p;
    p.gordered = ft.d_gordered.p;
    p.n_deliverers = ft.n_deliverers;
    return p;
}

// ---------------------------------------------------------------- per-snapshot tables
// The snapshot's table in `slot`, built by build(T&) on the first call that needs it. fan_mu is held throughout, so concurrent
// first calls build it once.
template <typename T, typename Build>
int32_t cached(Snapshot* s, std::shared_ptr<T>& slot, std::shared_ptr<T>* out, Build&& build) {
    std::lock_guard<std::mutex> g(s->fan_mu);
    if (!slot) {
        auto t = std::make_shared<T>();
        const int32_t rc = build(*t);
        if (rc != BFQ_OK) return rc;
        slot = std::move(t);
    }
    *out = slot;
    return BFQ_OK;
}

// a host table's device copy (one element at least, so that an empty table still has an address)
template <typename T>
int32_t upload(DeviceBuf<T>& d, const std::vector<T>& v) {
    BFQ_CUDA_TRY(d.reserve(std::max<size_t>(v.size(), 1)));
    if (!v.empty()) BFQ_CUDA_TRY(cudaMemcpy(d.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return BFQ_OK;
}

// f(i) for every tenant of the snapshot, on all host cores
void for_each_tenant(const Snapshot* s, const std::function<void(uint32_t)>& f) {
    std::vector<uint32_t> all(s->th.size());
    std::iota(all.begin(), all.end(), 0u);
    parallel_for_each(all, f);
}

// the snapshot's fan-out tables: every tenant's routes resolved to deliverer ids (cached per tenant blob: a delta commit
// re-resolves only the tenants it rebuilt), concatenated in rank order and uploaded once per snapshot
int32_t ensure_fan_table(bfq_index* h, Snapshot* s, std::shared_ptr<Snapshot::FanTable>* out) {
    return cached(s, s->fan, out, [&](Snapshot::FanTable& ft) -> int32_t {
        const size_t T = s->th.size();
        std::vector<std::string> errs(T);
        for_each_tenant(s, [&](uint32_t i) {
            if (s->th[i].fan) return;
            auto tf = std::make_shared<TenantFan>();
            if (build_tenant_fan(*s->th[i].kv, h->deliverers.get(), tf.get(), &errs[i])) s->th[i].fan = std::move(tf);
        });
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
        {
            std::lock_guard<std::mutex> gd(h->deliverers->mu);
            ft.n_deliverers = (uint32_t) h->deliverers->list.size() + 1;
        }
        // ids share rdeliv[] with FO_GROUP_BIT, and n_deliverers and the global pass's n_deliverers + 1 counts are int32
        if (ft.n_deliverers > 0x7FFFFFFEu) return fail(BFQ_E_RANGE, "more than 2^31 - 3 distinct (subBrokerId, delivererKey) pairs on one handle");
        int32_t rc = upload(ft.d_rdeliv, rdeliv);
        if (rc == BFQ_OK) rc = upload(ft.d_gmem_off, gmem_off);
        if (rc == BFQ_OK) rc = upload(ft.d_gmem_deliv, gmem_deliv);
        if (rc == BFQ_OK) rc = upload(ft.d_gordered, gordered);
        return rc;
    });
}

// the snapshot's ordered-group member urls, from the tenants' fan-out tables (call after ensure_fan_table), in the fan table's
// member order: each url at byte 4 of its own run of 8-byte words, so the pick reads LE32(hash) ‖ url as whole words
int32_t ensure_url_table(Snapshot* s, std::shared_ptr<Snapshot::UrlTable>* out) {
    return cached(s, s->urls, out, [&](Snapshot::UrlTable& ut) -> int32_t {
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
        ut.member_bits = largest ? 32u - (uint32_t) __builtin_clz(largest) : 1u;
        int32_t rc = upload(ut.d_words, words);
        if (rc == BFQ_OK) rc = upload(ut.d_word, word);
        if (rc == BFQ_OK) rc = upload(ut.d_len, len);
        return rc;
    });
}

// the snapshot's MatchInfo table: every tenant's entries (cached per tenant blob, so a delta commit re-encodes only the tenants it
// rebuilt), concatenated in rank order and uploaded once per snapshot
int32_t ensure_wire_table(Snapshot* s, std::shared_ptr<Snapshot::WireTable>* out) {
    return cached(s, s->wire, out, [&](Snapshot::WireTable& wt) -> int32_t {
        const size_t T = s->th.size();
        std::vector<std::string> errs(T);
        for_each_tenant(s, [&](uint32_t i) {
            if (s->th[i].wire) return;
            auto tw = std::make_shared<TenantWire>();
            if (build_tenant_wire(*s->th[i].kv, tw.get(), &errs[i])) s->th[i].wire = std::move(tw);
        });
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
        int32_t rc = upload(wt.d_first, first);
        if (rc == BFQ_OK) rc = upload(wt.d_off, off);
        if (rc == BFQ_OK) rc = upload(wt.d_bytes, blob);
        if (rc != BFQ_OK) return rc;
        wt.n_entries = entries;
        s->wire_bytes = wt.bytes();
        return BFQ_OK;
    });
}

// the hash of every MatchInfo in the snapshot's table (bfq_delivery_reply's join key), built once per snapshot on `st`
int32_t ensure_mi_hash(Snapshot* s, const Snapshot::WireTable& wt, cudaStream_t st, std::shared_ptr<DeviceBuf<uint32_t>>* out) {
    return cached(s, s->mi_hash, out, [&](DeviceBuf<uint32_t>& hb) -> int32_t {
        BFQ_CUDA_TRY(hb.reserve(std::max<size_t>(wt.n_entries, 1)));
        BFQ_CUDA_TRY(launch_mi_hash(wt.d_bytes.p, wt.d_off.p, (int64_t) wt.n_entries, hb.p, st));
        BFQ_CUDA_TRY(cudaStreamSynchronize(st));   // other streams read it from now on
        return BFQ_OK;
    });
}

}  // namespace

extern "C" {

int32_t bfq_expand_device(const bfq_device_result* res, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap, void* stream,
                          int64_t* n_ranks) {
    if (!res || !res->lease || !d_offsets) return fail(BFQ_E_INVALID, "bad argument");
    ResultCall c(res, stream, "bfq_expand_device");
    if (c.rc != BFQ_OK) return c.rc;
    const int64_t n_topics = c.L->n;
    BFQ_CUDA_TRY(c.w->d_exp_counts.reserve((size_t) n_topics + 1));
    const ExpandParams p = expand_params(c.L, d_offsets, d_ranks, rank_cap);
    size_t tmp_bytes = 0;
    const int32_t rc = launch_with_temp(c.w->d_scan_tmp, tmp_bytes, "launch_expand",
                                        [&](void* t, size_t* b) { return launch_expand(p, t, b, c.st, 1); });
    if (rc != BFQ_OK) return rc;
    long long total = 0;
    BFQ_CUDA_TRY(cudaMemcpyAsync(&total, d_offsets + n_topics, sizeof(long long), cudaMemcpyDeviceToHost, c.st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(c.st));
    if (n_ranks) *n_ranks = (int64_t) total;
    int64_t launches = 2;
    if (d_ranks && total <= rank_cap) {
        BFQ_CUDA_TRY(launch_expand(p, c.w->d_scan_tmp.p, &tmp_bytes, c.st, 2));
        launches += 2;
    }
    add_launches(c.h, launches);
    return BFQ_OK;
}

int32_t bfq_expand_device_budget(const bfq_device_result* res, const int32_t* d_msg_bytes, const int64_t* max_pfanout_bytes,
                                 const uint8_t* tenant_bandwidth, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap,
                                 void* stream, bfq_budget_result* out) {
    if (!res || !res->lease || !d_offsets || !out) return fail(BFQ_E_INVALID, "bad argument");
    ResultCall c(res, stream, "bfq_expand_device_budget");
    if (c.rc != BFQ_OK) return c.rc;
    const int64_t n_topics = c.L->n;
    const int32_t n_tenants = c.L->ctx.n_tenants;
    if (n_topics > 0 && !d_msg_bytes) return fail(BFQ_E_INVALID, "NULL d_msg_bytes");
    if (n_tenants > 0 && (!max_pfanout_bytes || !tenant_bandwidth)) return fail(BFQ_E_INVALID, "NULL per-tenant budget table");
    for (int32_t i = 0; i < n_tenants; i++)
        if (max_pfanout_bytes[i] <= 0)
            return fail(BFQ_E_INVALID, "max_pfanout_bytes[" + std::to_string(i) + "] = " + std::to_string(max_pfanout_bytes[i]) +
                                           ": MaxPersistentFanoutBytes must be > 0");
    const size_t nn = (size_t) std::max<int64_t>(n_topics, 1), nt = (size_t) std::max(n_tenants, 1);
    BFQ_CUDA_TRY(c.w->d_exp_counts.reserve(nn + 1));
    BudgetParams q{};
    long long* max_bytes = nullptr;
    uint8_t* bandwidth = nullptr;
    int32_t rc = carve(c.w->d_bud, "budget arena", [&](Carve& a) {
        q.max_bytes = max_bytes = a.take<long long>(nt);
        q.bandwidth = bandwidth = a.take<uint8_t>(nt);
        q.flags = a.take<uint8_t>(nn);
        q.delivered_p = a.take<uint32_t>(nn);
        q.list = a.take<uint32_t>(nn);
        q.ctr = a.take<unsigned long long>(BUD_CTR_COUNT);
    });
    if (rc != BFQ_OK) return rc;
    if (n_tenants > 0) {
        BFQ_CUDA_TRY(cudaMemcpyAsync(max_bytes, max_pfanout_bytes, (size_t) n_tenants * sizeof(long long), cudaMemcpyHostToDevice, c.st));
        BFQ_CUDA_TRY(cudaMemcpyAsync(bandwidth, tenant_bandwidth, (size_t) n_tenants, cudaMemcpyHostToDevice, c.st));
    }
    BFQ_CUDA_TRY(cudaMemsetAsync(q.ctr, 0, BUD_CTR_COUNT * sizeof(unsigned long long), c.st));
    q.e = expand_params(c.L, d_offsets, d_ranks, rank_cap);
    q.n_tenants = n_tenants;
    q.msg_bytes = d_msg_bytes;
    size_t tmp_bytes = 0;
    rc = launch_with_temp(c.w->d_scan_tmp, tmp_bytes, "launch_budget", [&](void* t, size_t* b) { return launch_budget(q, t, b, c.st, 1); });
    if (rc != BFQ_OK) return rc;
    long long total = 0;
    unsigned long long ctr[BUD_CTR_COUNT];
    BFQ_CUDA_TRY(cudaMemcpyAsync(&total, d_offsets + n_topics, sizeof(long long), cudaMemcpyDeviceToHost, c.st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(ctr, q.ctr, sizeof(ctr), cudaMemcpyDeviceToHost, c.st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(c.st));
    int64_t launches = 2;
    const bool ok = ctr[BUD_BAD_SIZE] == 0;
    if (ok && d_ranks && total <= rank_cap) {
        q.n_listed = (int64_t) ctr[BUD_LISTED];
        BFQ_CUDA_TRY(launch_budget(q, c.w->d_scan_tmp.p, &tmp_bytes, c.st, 2));
        launches += 2;
    }
    add_launches(c.h, launches);
    if (!ok) return fail(BFQ_E_INVALID, std::to_string(ctr[BUD_BAD_SIZE]) + " negative d_msg_bytes entries");
    out->d_delivered_persistent = q.delivered_p;
    out->d_topic_flags = q.flags;
    out->n_delivered = (int64_t) total;
    out->n_dropped_bytes = (int64_t) ctr[BUD_DROP_BYTES];
    out->n_dropped_persistent_bandwidth = (int64_t) ctr[BUD_DROP_PBW];
    out->n_dropped_transient_bandwidth = (int64_t) ctr[BUD_DROP_TBW];
    return BFQ_OK;
}

int32_t bfq_fanout_device(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs, void* stream,
                          bfq_fanout_result* out) {
    if (!res || !res->lease || !out || !d_offsets || n_pairs < 0 || (n_pairs > 0 && !d_ranks)) return fail(BFQ_E_INVALID, "bad argument");
    ResultCall c(res, stream, "bfq_fanout_device");
    if (c.rc != BFQ_OK) return c.rc;
    if (n_pairs >= (int64_t) 0xFFFFFFF0ll) return fail(BFQ_E_RANGE, "more than 2^32 (topic, route) pairs in one batch; split the batch");
    std::shared_ptr<Snapshot::FanTable> ft;
    int32_t rc = ensure_fan_table(c.h, c.L->snap.get(), &ft);
    if (rc != BFQ_OK) return rc;
    bool force_global;
    {
        std::lock_guard<std::mutex> g(c.h->mu);
        force_global = c.h->fanout_global;
    }
    const bool tiled = !force_global && fanout_tiled(ft->n_deliverers, n_pairs);
    const size_t words = fanout_scratch_words(ft->n_deliverers, n_pairs, tiled), np = (size_t) std::max<int64_t>(n_pairs, 1);
    FanoutParams p = fanout_inputs(c.L, *ft, d_offsets, d_ranks, n_pairs);
    rc = carve(c.w->d_fo, "fan-out arena", [&](Carve& a) {
        p.counts = a.take<uint32_t>(words);
        p.base = a.take<uint32_t>(words);
        p.pack_offsets = a.take<long long>((size_t) ft->n_deliverers + 1);
        p.pack_topic = a.take<uint32_t>(np);
        p.pack_rank = a.take<uint32_t>(np);
        p.pack_member = a.take<uint32_t>(np);
    });
    if (rc != BFQ_OK) return rc;
    size_t tmp_bytes = 0;
    rc = launch_with_temp(c.w->d_fo_tmp, tmp_bytes, "launch_fanout", [&](void* t, size_t* b) { return launch_fanout(p, tiled, t, b, c.st); });
    if (rc != BFQ_OK) return rc;
    out->d_pack_offsets = (const int64_t*) p.pack_offsets;
    out->d_pack_topic = p.pack_topic;
    out->d_pack_rank = p.pack_rank;
    out->d_pack_member = p.pack_member;
    out->n_pairs = n_pairs;
    out->n_deliverers = (int32_t) ft->n_deliverers;
    out->ordered_share_id = (int32_t) ft->n_deliverers - 1;
    out->generation = c.L->snap->generation;
    add_launches(c.h, 5, tiled ? 0 : 1);
    return BFQ_OK;
}

}  // extern "C"

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
    ResultCall c(res, stream, who);
    if (c.rc != BFQ_OK) return c.rc;
    if (c.L->n > 0 && !d_topic_tenant) return fail(BFQ_E_INVALID, "NULL d_topic_tenant");
    if (pubs && !pubs->pub_off) return fail(BFQ_E_INVALID, "NULL d_pub_off");
    if (pubs && (pubs->n_pubs < 0 || (pubs->n_pubs > 0 && !pubs->pub_hash))) return fail(BFQ_E_INVALID, "bad d_pub_hash / n_pubs");
    if (n_pairs >= (int64_t) 0xFFFFFFF0ll) return fail(BFQ_E_RANGE, "more than 2^32 (topic, route) pairs in one batch; split the batch");
    Workspace* w = c.w;
    w->dl_n_packs = -1;   // the arena below is about to change
    std::shared_ptr<Snapshot::FanTable> ft;
    int32_t rc = ensure_fan_table(c.h, c.L->snap.get(), &ft);
    if (rc != BFQ_OK) return rc;
    std::shared_ptr<Snapshot::UrlTable> ut;
    if (pubs && (rc = ensure_url_table(c.L->snap.get(), &ut)) != BFQ_OK) return rc;
    const size_t T = (size_t) c.L->n;
    DeliveryParams q{};
    q.f = fanout_inputs(c.L, *ft, d_offsets, d_ranks, n_pairs);
    q.topic_tenant = d_topic_tenant;
    q.n_tenants = c.L->ctx.n_tenants;
    int64_t n_items = 0;
    size_t tmp_bytes = 0;
    if (pubs) {
        // phase 1: which pairs are $oshare pairs to resolve, how many (pair, publisher) items, and the d_pub_off check. Its
        // arena is apart from the nesting's: phase 2 reads it, and is sized from what it counted.
        q.oshare = true;
        q.o.pub_off = pubs->pub_off;
        q.o.pub_hash = pubs->pub_hash;
        q.o.n_pubs = pubs->n_pubs;
        q.o.url_words = ut->d_words.p;
        q.o.url_word = ut->d_word.p;
        q.o.url_len = ut->d_len.p;
        q.o.member_bits = ut->member_bits;
        rc = carve(w->d_os, "$oshare count arena", [&](Carve& a) {
            q.o.oflag = a.take<uint32_t>((size_t) n_pairs + 1);
            q.o.oitems = a.take<unsigned long long>((size_t) n_pairs + 1);
            q.o.check = a.take<unsigned long long>(4);
        });
        if (rc != BFQ_OK) return rc;
        rc = launch_with_temp(w->d_dl_tmp, tmp_bytes, "launch_oshare_count",
                              [&](void* t, size_t* b) { return launch_oshare_count(q, t, b, c.st); });
        if (rc != BFQ_OK) return rc;
        unsigned long long chk[4];
        BFQ_CUDA_TRY(cudaMemcpyAsync(chk, q.o.check, sizeof(chk), cudaMemcpyDeviceToHost, c.st));
        BFQ_CUDA_TRY(cudaStreamSynchronize(c.st));
        if ((int64_t) chk[3] != n_pairs)
            return fail(BFQ_E_INVALID, "n_pairs = " + std::to_string(n_pairs) + " but d_offsets[n_topics] = " + std::to_string((int64_t) chk[3]));
        if (chk[2]) return fail(BFQ_E_INVALID, "d_pub_off must run from 0 to n_pubs = " + std::to_string(pubs->n_pubs) + " without decreasing");
        if (chk[1] >= 0xFFFFFFF0ull || (uint64_t) n_pairs + chk[1] >= 0xFFFFFFF0ull)
            return fail(BFQ_E_RANGE, "more than 2^32 pairs and ($oshare pair, publisher) items in one batch; split the batch");
        q.o.n_opairs = (int64_t) chk[0];
        n_items = (int64_t) chk[1];
        q.o.n_items = n_items;
    }
    const size_t np = (size_t) std::max<int64_t>(n_pairs + n_items, 1), O = (size_t) q.o.n_opairs, I = (size_t) n_items;
    rc = carve(w->d_dl, "delivery arena", [&](Carve& a) {
        // the outputs first: package_off and match_off, which encode and reply check a nesting by, then move only with the arena
        q.package_off = a.take<long long>((size_t) ft->n_deliverers + 1);
        q.match_off = a.take<long long>(np + 1);
        q.package_tenant = a.take<uint32_t>(np);
        q.pack_off = a.take<long long>(np + 1);
        q.pack_topic = a.take<uint32_t>(np);
        q.match_rank = a.take<uint32_t>(np);
        q.match_member = a.take<uint32_t>(np);
        for (auto& x : q.tkey) x = a.take<uint32_t>(T);
        for (auto& x : q.tval) x = a.take<uint32_t>(T);
        q.tcount = a.take<uint32_t>(T + 1);
        q.tstart = a.take<uint32_t>(T + 1);
        for (auto& x : q.key) x = a.take<uint32_t>(np);
        for (auto& x : q.val) x = a.take<uint32_t>(np);
        q.e_topic = a.take<uint32_t>(np);
        q.e_rank = a.take<uint32_t>(np);
        q.e_member = a.take<uint32_t>(np);
        q.s_topic = a.take<uint32_t>(np);
        q.package_head = a.take<uint32_t>(np + 1);
        q.pack_head = a.take<uint32_t>(np + 1);
        q.pcount = a.take<uint32_t>((size_t) ft->n_deliverers + 1);
        q.totals = a.take<unsigned long long>(5);
        if (!pubs) return;
        q.o.pack_pub_off = a.take<long long>(np + 1);
        q.o.pack_pub = a.take<uint32_t>(std::max<size_t>(I, 1));
        for (auto& x : q.o.okey) x = a.take<unsigned long long>(O);
        for (auto& x : q.o.ikey) x = a.take<unsigned long long>(I);
        q.o.istart = a.take<uint32_t>(O + 1);
        for (auto& x : q.o.ival) x = a.take<uint32_t>(I);
        q.o.ihead = a.take<uint32_t>(I + 1);
        q.o.sub_start = a.take<uint32_t>(I + 1);
        q.o.sub_pack = a.take<uint32_t>(I);
        q.o.e_sub = a.take<uint32_t>(np);
        q.o.s_sub = a.take<uint32_t>(np);
        q.o.pub_count = a.take<uint32_t>(np + 1);
    });
    if (rc != BFQ_OK) return rc;
    rc = launch_with_temp(w->d_dl_tmp, tmp_bytes, "launch_delivery", [&](void* t, size_t* b) { return launch_delivery(q, t, b, c.st); });
    if (rc != BFQ_OK) return rc;
    unsigned long long tot[5] = {0, 0, 0, 0, 0};
    BFQ_CUDA_TRY(cudaMemcpyAsync(tot, q.totals, (pubs ? 5 : 4) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c.st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(c.st));
    add_launches(c.h, pubs ? 25 : 11);
    if ((int64_t) tot[3] != n_pairs)
        return fail(BFQ_E_INVALID, "n_pairs = " + std::to_string(n_pairs) + " but d_offsets[n_topics] = " + std::to_string((int64_t) tot[3]));
    out->d_package_off = (const int64_t*) q.package_off;
    out->d_package_tenant = q.package_tenant;
    out->d_pack_off = (const int64_t*) q.pack_off;
    out->d_pack_topic = q.pack_topic;
    out->d_match_off = (const int64_t*) q.match_off;
    out->d_match_rank = q.match_rank;
    out->d_match_member = q.match_member;
    out->n_pairs = (int64_t) tot[0];
    out->n_packages = (int64_t) tot[1];
    out->n_packs = (int64_t) tot[2];
    out->n_deliverers = (int32_t) ft->n_deliverers;
    out->ordered_share_id = (int32_t) ft->n_deliverers - 1;
    out->generation = c.L->snap->generation;
    w->dl_n_pairs = out->n_pairs;
    w->dl_n_packages = out->n_packages;
    w->dl_n_packs = out->n_packs;
    w->dl_ordered = pubs != nullptr;
    w->dl_package_off = out->d_package_off;
    w->dl_match_off = out->d_match_off;
    w->dl_pack_pub_off = pubs ? (const int64_t*) q.o.pack_pub_off : nullptr;
    if (oout) {
        oout->d_pack_pub_off = (const int64_t*) q.o.pack_pub_off;
        oout->d_pack_pub = q.o.pack_pub;
        oout->n_pack_pubs = n_items;
        oout->n_ordered_packs = (int64_t) tot[4];
    }
    return BFQ_OK;
}

// the nesting is the one the last delivery call on this result left in its workspace (plain or ordered)
bool latest_nesting(const DeviceLease* L, const bfq_delivery_result* nest) {
    const Workspace* w = L->ws;
    return nest->generation == L->snap->generation && nest->d_package_off == w->dl_package_off &&
           nest->d_match_off == w->dl_match_off && w->dl_n_packs >= 0 && nest->n_packs == w->dl_n_packs &&
           nest->n_packages == w->dl_n_packages && nest->n_pairs == w->dl_n_pairs;
}

// The match's tenant list, which encode and reply take again (a nesting names tenants by their index in it), and its device
// copy in the calling family's arena
struct TenantList {
    const uint8_t* bytes;
    const int64_t* off;
    int32_t n;
    long long* d_off = nullptr;
    uint8_t* d_bytes = nullptr;
    int32_t check(const DeviceLease* L, const char* who) const {
        if (n != L->ctx.n_tenants || (n > 0 && (!bytes || !off)))
            return fail(BFQ_E_INVALID, std::string(who) + ": the tenant list must be the match's (" + std::to_string(L->ctx.n_tenants) + " tenants)");
        return BFQ_OK;
    }
    int64_t n_bytes() const { return n > 0 ? off[n] : 0; }
    void take(Carve& a) {
        d_off = a.take<long long>((size_t) n + 1);
        d_bytes = a.take<uint8_t>((size_t) std::max<int64_t>(n_bytes(), 1));
    }
    int32_t upload(cudaStream_t st) const {
        if (n > 0) {
            BFQ_CUDA_TRY(cudaMemcpyAsync(d_off, off, ((size_t) n + 1) * 8, cudaMemcpyHostToDevice, st));
            if (n_bytes() > 0) BFQ_CUDA_TRY(cudaMemcpyAsync(d_bytes, bytes, (size_t) n_bytes(), cudaMemcpyHostToDevice, st));
        }
        return BFQ_OK;
    }
};

// what encode and reply both read: the nesting, the device copy of the tenant list and the snapshot's MatchInfo table
template <typename P>
void nesting_inputs(P& p, const bfq_delivery_result* nest, const TenantList& tl, const Snapshot::WireTable& wt) {
    p.n_packages = nest->n_packages;
    p.n_packs = nest->n_packs;
    p.n_pairs = nest->n_pairs;
    p.n_deliverers = (uint32_t) nest->n_deliverers;
    p.package_off = (const long long*) nest->d_package_off;
    p.package_tenant = nest->d_package_tenant;
    p.pack_off = (const long long*) nest->d_pack_off;
    p.match_off = (const long long*) nest->d_match_off;
    p.match_rank = nest->d_match_rank;
    p.match_member = nest->d_match_member;
    p.tenants = tl.d_bytes;
    p.tenant_off = tl.d_off;
    p.mi_first = wt.d_first.p;
    p.mi_off = wt.d_off.p;
    p.mi_bytes = wt.d_bytes.p;
}

// bfq_delivery_encode (oout == nullptr) and bfq_delivery_encode_ordered: nest is the nesting's plain part either way
int32_t run_encode(const bfq_device_result* res, const bfq_delivery_result* nest, const bfq_delivery_ordered_result* onest,
                   const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_topics,
                   const int64_t* d_topic_off, const int64_t* d_pub_off, const uint8_t* d_pubpack_bytes,
                   const int64_t* d_pubpack_off, uint8_t* d_out, int64_t out_cap, void* stream, const char* who,
                   bfq_delivery_wire_result* out) {
    if (!res || !res->lease || !nest || !out || out_cap < 0) return fail(BFQ_E_INVALID, "bad argument");
    ResultCall c(res, stream, who);
    if (c.rc != BFQ_OK) return c.rc;
    if (!d_topics || !d_topic_off || !d_pub_off || !d_pubpack_bytes || !d_pubpack_off)
        return fail(BFQ_E_INVALID, std::string(who) + ": NULL topic or publisher pack array");
    TenantList tl{tenants, tenant_off, n_tenants};
    int32_t rc = tl.check(c.L, who);
    if (rc != BFQ_OK) return rc;
    if (!latest_nesting(c.L, nest) || c.w->dl_ordered != (onest != nullptr) || (onest && onest->d_pack_pub_off != c.w->dl_pack_pub_off))
        return fail(BFQ_E_RANGE, std::string(who) + ": the nesting is not the latest " +
                                     (onest ? "bfq_delivery_device_ordered" : "bfq_delivery_device") + " result of this device result");
    std::shared_ptr<Snapshot::WireTable> wt;
    if ((rc = ensure_wire_table(c.L->snap.get(), &wt)) != BFQ_OK) return rc;
    const int64_t np = nest->n_pairs, nk = nest->n_packs, ng = nest->n_packages;
    const uint32_t D = (uint32_t) nest->n_deliverers;
    WireParams p{};
    rc = carve(c.w->d_wr, "encode arena", [&](Carve& a) {
        p.req_off = a.take<long long>((size_t) D + 1);
        p.pair_pos = a.take<unsigned long long>((size_t) np + 1);
        p.pack_pos = a.take<unsigned long long>((size_t) nk + 1);
        p.package_pos = a.take<unsigned long long>((size_t) ng + 1);
        p.check = a.take<unsigned long long>(4);
        tl.take(a);
    });
    if (rc != BFQ_OK) return rc;
    if ((rc = tl.upload(c.st)) != BFQ_OK) return rc;
    nesting_inputs(p, nest, tl, *wt);
    p.pack_topic = nest->d_pack_topic;
    p.pack_pub_off = onest ? (const long long*) onest->d_pack_pub_off : nullptr;
    p.pack_pub = onest ? onest->d_pack_pub : nullptr;
    p.topics = d_topics;
    p.topic_off = (const long long*) d_topic_off;
    p.n_topics = c.L->n;
    p.pub_off = (const long long*) d_pub_off;
    p.pubpack = d_pubpack_bytes;
    p.pubpack_off = (const long long*) d_pubpack_off;
    p.out = d_out;
    size_t tmp_bytes = 0;
    rc = launch_with_temp(c.w->d_wr_tmp, tmp_bytes, "launch_wire_size", [&](void* t, size_t* b) { return launch_wire_size(p, t, b, c.st); });
    if (rc != BFQ_OK) return rc;
    unsigned long long chk[4];
    BFQ_CUDA_TRY(cudaMemcpyAsync(chk, p.check, sizeof(chk), cudaMemcpyDeviceToHost, c.st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(c.st));
    if (chk[0]) return fail(BFQ_E_INVALID, std::string(who) + ": d_pub_off / d_pubpack_off must start at 0 and never decrease, and "
                                                               "every publisher of the nesting must be below d_pub_off[n_topics]");
    const bool write = d_out && (int64_t) chk[1] <= out_cap;
    if (write) BFQ_CUDA_TRY(launch_wire_write(p, c.st));
    add_launches(c.h, write ? 10 : 8);
    out->d_req_off = (const int64_t*) p.req_off;
    out->n_bytes = (int64_t) chk[1];
    out->n_match_infos = (int64_t) chk[2];
    out->n_skipped = np - (int64_t) chk[2];
    out->n_deliverers = (int32_t) D;
    out->ordered_share_id = (int32_t) D - 1;
    out->generation = c.L->snap->generation;
    return BFQ_OK;
}

}  // namespace

extern "C" {

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

int32_t bfq_delivery_reply(const bfq_device_result* res, const bfq_delivery_result* nest, const uint8_t* tenants,
                           const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_reply, const int64_t* d_reply_off,
                           void* stream, bfq_delivery_reply_result* out) {
    const char* who = "bfq_delivery_reply";
    if (!res || !res->lease || !nest || !out) return fail(BFQ_E_INVALID, "bad argument");
    ResultCall c(res, stream, who);
    if (c.rc != BFQ_OK) return c.rc;
    if (!d_reply || !d_reply_off) return fail(BFQ_E_INVALID, std::string(who) + ": NULL reply array");
    TenantList tl{tenants, tenant_off, n_tenants};
    int32_t rc = tl.check(c.L, who);
    if (rc != BFQ_OK) return rc;
    if (!latest_nesting(c.L, nest))
        return fail(BFQ_E_RANGE, std::string(who) + ": the nesting is not the latest delivery nesting of this device result");
    std::shared_ptr<Snapshot::WireTable> wt;
    if ((rc = ensure_wire_table(c.L->snap.get(), &wt)) != BFQ_OK) return rc;
    std::shared_ptr<DeviceBuf<uint32_t>> mh;
    if ((rc = ensure_mi_hash(c.L->snap.get(), *wt, c.st, &mh)) != BFQ_OK) return rc;
    const int64_t np = nest->n_pairs, ng = nest->n_packages;
    const uint32_t D = (uint32_t) nest->n_deliverers;
    if (np >= (int64_t) 1 << 31) return fail(BFQ_E_RANGE, std::string(who) + ": 2^31 or more pairs in one nesting");
    uint64_t T = 2;
    while (T < 2 * (uint64_t) np) T <<= 1;
    const size_t cap = (size_t) std::max<int64_t>(np, 1), G = (size_t) std::max<int64_t>(ng, 1), nch = RP_MAX_CHUNKS + (size_t) ng;
    BFQ_CUDA_TRY(c.w->h_rp_ctr.reserve(RP_CTR_N));
    ReplyParams p{};
    rc = carve(c.w->d_rp, "reply arena", [&](Carve& a) {
        p.pair_code = a.take<uint8_t>(cap);
        p.status = a.take<uint8_t>(D);
        p.stale = a.take<bfq_stale_match>(cap);
        p.ctr = a.take<unsigned long long>(RP_CTR_N);
        p.dl_fail = a.take<uint8_t>(D);
        p.dl_code = a.take<int32_t>(D);
        p.dl_entries = a.take<uint32_t>(D);
        for (long long** x : {&p.ent_s, &p.ent_e, &p.ent_vs, &p.ent_ve}) *x = a.take<long long>(G);
        p.ent_pkg = a.take<uint32_t>(G);
        p.ent_bad = a.take<uint8_t>(G);
        p.pkg_claimed = a.take<uint32_t>(G);
        p.chunk_base = a.take<unsigned long long>((size_t) ng + 1);
        for (long long** x : {&p.ch_guess, &p.ch_exit, &p.ch_start}) *x = a.take<long long>(nch);
        p.slot_key = a.take<unsigned long long>(T);
        p.slot_rpos = a.take<unsigned long long>(T);
        for (uint32_t** x : {&p.slot_pair, &p.slot_code, &p.slot_rlen}) *x = a.take<uint32_t>(T);
        p.pair_slot = a.take<uint32_t>(cap);
        p.pkg_stale = a.take<unsigned long long>((size_t) ng + 1);
        p.pkg_cursor = a.take<unsigned long long>((size_t) ng + 1);
        for (uint32_t** x : {&p.stale_list, &p.sort_key_in, &p.sort_key_out, &p.sort_val_in, &p.sort_val_out}) *x = a.take<uint32_t>(cap);
        tl.take(a);
    });
    if (rc != BFQ_OK) return rc;
    if ((rc = tl.upload(c.st)) != BFQ_OK) return rc;
    nesting_inputs(p, nest, tl, *wt);
    p.mi_hash = mh->p;
    p.reply = d_reply;
    p.reply_off = (const long long*) d_reply_off;
    p.table_mask = T - 1;
    p.stale_cap = (int64_t) cap;
    size_t tmp_bytes = 0;
    rc = launch_with_temp(c.w->d_rp_tmp, tmp_bytes, "launch_reply", [&](void* t, size_t* b) { return launch_reply(p, t, b, c.st); });
    if (rc != BFQ_OK) return rc;
    BFQ_CUDA_TRY(cudaMemcpyAsync(c.w->h_rp_ctr.p, p.ctr, RP_CTR_N * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c.st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(c.st));
    add_launches(c.h, 17);
    const unsigned long long* n = c.w->h_rp_ctr.p;
    if (n[RP_BAD_OFF]) return fail(BFQ_E_INVALID, std::string(who) + ": d_reply_off must never decrease");
    out->d_pair_code = p.pair_code;
    out->d_status = p.status;
    out->d_stale = p.stale;
    for (int i = 0; i < 8; i++) out->n_code[i] = (int64_t) n[RP_N_CODE + i];
    out->n_pairs = np;
    out->n_stale = (int64_t) n[RP_N_STALE];
    out->n_fallback = (int32_t) n[RP_N_FALLBACK];
    out->n_deliverers = (int32_t) D;
    out->ordered_share_id = (int32_t) D - 1;
    out->generation = c.L->snap->generation;
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

}  // extern "C"
