"""Host-side mirror of the reference interfaces the CUDA matcher sits behind.

* GpuRouteIndex            — one per dist-worker KV range, owns the bfq_index handle; it is fed the way
                             DistWorkerCoProc feeds its caches: reset()/load() on
                             DistWorkerCoProc.reset (DW/DistWorkerCoProc.java:283-291), apply() from the
                             post-persist Supplier of mutate() (:188-209), commit() to publish.
* GpuTenantRouteMatcher    — ITenantRouteMatcher.matchAll(Set<String> topics, int maxPersistentFanoutCount,
                             int maxGroupFanoutCount) -> Map<String, IMatchedRoutes>
                             (DW/cache/ITenantRouteMatcher.java:28-38), same argument meaning, same contract
                             (an entry for every requested topic, caps applied in KV order, throttle events
                             reported to the event collector).
* MatchedRoutes            — the read side of IMatchedRoutes (DW/cache/IMatchedRoutes.java:68-151).
DW/ = bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/ in the reference.

All matching happens in the CUDA library; this module only marshals buffers and re-hydrates results.
"""
import ctypes as C
from collections import namedtuple

import numpy as np

from . import _native as N
from . import schema

INT_MAX = 2 ** 31 - 1
RANGE_MULTI = 0x80000000

PersistentFanoutThrottled = namedtuple("PersistentFanoutThrottled", "tenant_id topic mqtt_topic_filter max_count")
GroupFanoutThrottled = namedtuple("GroupFanoutThrottled", "tenant_id topic mqtt_topic_filter max_count")
PersistentFanoutBytesThrottled = namedtuple("PersistentFanoutBytesThrottled", "tenant_id topic max_bytes")
OutOfTenantResource = namedtuple("OutOfTenantResource", "reason tenant_id topic")
PERSISTENT_BANDWIDTH = "TotalPersistentFanOutBytesPerSeconds"   # TenantResourceType names, the reason OutOfTenantResource carries
TRANSIENT_BANDWIDTH = "TotalTransientFanOutBytesPerSeconds"


def budget_events(tenants, topics, topic_tenant, flags, delivered_persistent, msg_bytes, max_pfanout_bytes):
    """The events and meter values of a bfq_expand_device_budget result, as DeliverExecutorGroup.submit reports them.
    flags / delivered_persistent: the result's per-topic arrays copied to the host; msg_bytes: the sizes passed to the call.
    -> (events, meter): events in topic order, for each topic PersistentFanoutBytesThrottled, then OutOfTenantResource for
    persistent, then for transient bandwidth; meter = [(topic position, MqttPersistentFanOutBytes value)] for every topic
    the reference records it for (zero values included). The reference reports OutOfTenantResource once per publisher of
    the message pack (with its ClientInfo): repeating each one per publisher is the caller's job."""
    events, meter = [], []
    flags = np.asarray(flags)
    for t in np.flatnonzero(flags).tolist():
        f = int(flags[t])
        tenant = int(topic_tenant[t])
        tid = tenants[tenant]
        if f & N.BUDGET_BYTES_THROTTLED:
            events.append(PersistentFanoutBytesThrottled(tid, topics[t], int(max_pfanout_bytes[tenant])))
        if f & N.BUDGET_NO_PERSISTENT_BW:
            events.append(OutOfTenantResource(PERSISTENT_BANDWIDTH, tid, topics[t]))
        if f & N.BUDGET_NO_TRANSIENT_BW:
            events.append(OutOfTenantResource(TRANSIENT_BANDWIDTH, tid, topics[t]))
        if f & N.BUDGET_METERED:
            meter.append((t, int(delivered_persistent[t]) * int(msg_bytes[t])))
    return events, meter


class BatchResult:
    """Numpy views over one bfq_match result. The arrays are private to this result and stay valid until close();
    route()/route_kinds() resolve ranks against the snapshot the match ran on, whatever was committed since."""

    def __init__(self, handle, n, owner=None):
        self._h = handle
        self._owner = owner   # keeps the index alive for as long as this result is
        self.n_topics = n
        lib = N.lib

        def arr(p, count, dtype):
            dtype = np.dtype(dtype)
            if count == 0 or not p:
                return np.zeros(0, dtype)
            return np.frombuffer((C.c_uint8 * (count * dtype.itemsize)).from_address(p), dtype=dtype)
        self.span_begin = arr(lib.bfq_result_span_begin(handle), n, np.uint32)
        self.span_count = arr(lib.bfq_result_span_count(handle), n, np.uint32)
        self.route_count = arr(lib.bfq_result_route_count(handle), n, np.uint32)
        nr, nt = C.c_int64(0), C.c_int64(0)
        pr = lib.bfq_result_ranges(handle, C.byref(nr))
        pt = lib.bfq_result_throttled(handle, C.byref(nt))
        self.ranges = arr(pr, nr.value, np.dtype([("first", np.uint32), ("count", np.uint32)]))
        self.throttled = arr(pt, nt.value, np.dtype([("topic", np.uint32), ("rank", np.uint32), ("kind", np.uint32)]))
        ms = np.zeros(4, np.float64)
        lib.bfq_result_timings(handle, ms.ctypes.data, 4)
        self.timings_ms = dict(zip(["h2d_stream_busy", "tier0_kernel_first_sub_batch", "sub_batches", "total"], ms.tolist()))

    def expand(self):
        """-> (offsets[n+1], ranks) surviving route ranks, ascending per topic"""
        offsets = np.zeros(self.n_topics + 1, np.int64)
        total = N.lib.bfq_result_expand(self._h, offsets.ctypes.data, None, 0)
        ranks = np.zeros(max(total, 1), np.int64)
        N.lib.bfq_result_expand(self._h, offsets.ctypes.data, ranks.ctypes.data, total)
        return offsets, ranks[:total]

    @property
    def generation(self):
        return int(N.lib.bfq_result_generation(self._h))

    def route(self, rank):
        """(key, value) of a route rank of THIS result (bfq_result_route_lookup)"""
        kl, vl = C.c_int64(0), C.c_int64(0)
        N.check(N.lib.bfq_result_route_lookup(self._h, int(rank), None, 0, C.byref(kl), None, 0, C.byref(vl)))
        kb, vb = C.create_string_buffer(max(kl.value, 1)), C.create_string_buffer(max(vl.value, 1))
        N.check(N.lib.bfq_result_route_lookup(self._h, int(rank), C.addressof(kb), kl.value, C.byref(kl), C.addressof(vb), vl.value, C.byref(vl)))
        return kb.raw[:kl.value], vb.raw[:vl.value]

    def route_kinds(self, ranks):
        ranks = np.ascontiguousarray(ranks, dtype=np.int64)
        out = np.zeros(max(len(ranks), 1), np.uint8)
        N.check(N.lib.bfq_result_route_kinds(self._h, ranks.ctypes.data, len(ranks), out.ctypes.data))
        return out[:len(ranks)]

    def close(self):
        if self._h:
            N.lib.bfq_result_free(self._h)
            self._h = None

    def __del__(self):
        self.close()


class DeliveryResult:
    """One bfq_delivery_device result: the raw struct's fields (d_package_off, n_packs, ordered_share_id, ...) plus nesting().
    A bfq_delivery_device_ordered result also carries each pack's publisher positions (`ordered` is its full struct)."""

    def __init__(self, raw, ordered=None):
        self.raw = raw
        self.ordered = ordered

    def __getattr__(self, name):
        if name in ("raw", "ordered"):
            raise AttributeError(name)
        return getattr(self.raw, name)

    def arrays(self, device=None):
        """the seven arrays copied to the host (numpy), after a device synchronise; an ordered result adds pack_pub_off and
        pack_pub"""
        import torch

        from .dist import device_view
        torch.cuda.synchronize(device)
        r = self.raw

        def get(p, n, t):
            return device_view(p, max(n, 1), t, device).cpu().numpy()[:n].astype(np.int64)
        a = {"package_off": get(r.d_package_off, r.n_deliverers + 1, "<i8"),
             "package_tenant": get(r.d_package_tenant, r.n_packages, "<u4"),
             "pack_off": get(r.d_pack_off, r.n_packages + 1, "<i8"),
             "pack_topic": get(r.d_pack_topic, r.n_packs, "<u4"),
             "match_off": get(r.d_match_off, r.n_packs + 1, "<i8"),
             "match_rank": get(r.d_match_rank, r.n_pairs, "<u4"),
             "match_member": get(r.d_match_member, r.n_pairs, "<u4")}
        if self.ordered is not None:
            a["pack_pub_off"] = get(self.ordered.d_pack_pub_off, r.n_packs + 1, "<i8")
            a["pack_pub"] = get(self.ordered.d_pack_pub, self.ordered.n_pack_pubs, "<u4")
        return a

    def nesting(self, device=None):
        """{deliverer id: {tenant index: [(topic position, {(rank, member), ...}), ...]}}: deliverers without pairs are left
        out, packages in ascending tenant order, packs in their order. An ordered result's packs are
        (topic position, {(rank, member)}, (publisher position, ...)), the tuple empty for a whole TopicMessagePack.
        For tests and small batches: the walk is on the host."""
        a = self.arrays(device)
        out = {}
        for d in range(self.raw.n_deliverers):
            p0, p1 = int(a["package_off"][d]), int(a["package_off"][d + 1])
            if p0 == p1:
                continue
            pkgs = out[d] = {}
            for p in range(p0, p1):
                packs = pkgs[int(a["package_tenant"][p])] = []
                for k in range(int(a["pack_off"][p]), int(a["pack_off"][p + 1])):
                    m0, m1 = int(a["match_off"][k]), int(a["match_off"][k + 1])
                    pack = (int(a["pack_topic"][k]), set(zip(a["match_rank"][m0:m1].tolist(), a["match_member"][m0:m1].tolist())))
                    if self.ordered is not None:
                        pack += (tuple(a["pack_pub"][int(a["pack_pub_off"][k]):int(a["pack_pub_off"][k + 1])].tolist()),)
                    packs.append(pack)
        return out


class DeviceResult:
    """One bfq_match_device[_async] result: device pointers + counts; the buffers stay valid until release()."""

    def __init__(self, raw, owner=None):
        self.raw = raw
        self._owner = owner   # keeps the index alive for as long as this result is

    def __getattr__(self, name):   # d_span_begin, n_ranges, tier0_ms, ... straight from the C struct
        if name == "raw":
            raise AttributeError(name)
        return getattr(self.raw, name)

    def wait(self):
        N.check(N.lib.bfq_device_result_wait(C.byref(self.raw)))
        return self

    def expand(self, d_offsets_ptr, d_ranks_ptr, rank_cap, stream=0):
        """device CSR of the surviving routes; returns the total number"""
        total = C.c_int64(0)
        N.check(N.lib.bfq_expand_device(C.byref(self.raw), d_offsets_ptr, d_ranks_ptr, rank_cap, stream, C.byref(total)))
        return total.value

    def expand_budget(self, d_msg_bytes_ptr, max_pfanout_bytes, tenant_bandwidth, d_offsets_ptr, d_ranks_ptr, rank_cap, stream=0):
        """bfq_expand_device_budget: device CSR of the routes DeliverExecutorGroup.submit delivers. d_msg_bytes_ptr: int32
        message size per topic position (device); max_pfanout_bytes (MaxPersistentFanoutBytes) and tenant_bandwidth (bit 0
        persistent, bit 1 transient bandwidth) per tenant of the match's tenant list. -> BfqBudgetResult; its per-topic
        device arrays stay valid until release() or the next budget call on this result"""
        mb = np.ascontiguousarray(max_pfanout_bytes, dtype=np.int64)
        bw = np.ascontiguousarray(tenant_bandwidth, dtype=np.uint8)
        out = N.BfqBudgetResult()
        N.check(N.lib.bfq_expand_device_budget(C.byref(self.raw), d_msg_bytes_ptr, N.ptr(mb) if mb.size else None,
                                               N.ptr(bw) if bw.size else None, d_offsets_ptr, d_ranks_ptr, rank_cap, stream,
                                               C.byref(out)))
        return out

    def fanout(self, d_offsets_ptr, d_ranks_ptr, n_pairs, stream=0):
        """bfq_fanout_device: the (topic, route) pairs of this result's device CSR grouped by deliverer id -> BfqFanoutResult
        (device pointers into this result's workspace)"""
        out = N.BfqFanoutResult()
        N.check(N.lib.bfq_fanout_device(C.byref(self.raw), d_offsets_ptr, d_ranks_ptr, n_pairs, stream, C.byref(out)))
        return out

    def delivery(self, d_offsets_ptr, d_ranks_ptr, n_pairs, d_topic_tenant_ptr, stream=0):
        """bfq_delivery_device: the same pairs nested per deliverer, tenant and topic position, as BatchDeliveryCall sends
        them -> DeliveryResult (device pointers into this result's workspace)"""
        out = N.BfqDeliveryResult()
        N.check(N.lib.bfq_delivery_device(C.byref(self.raw), d_offsets_ptr, d_ranks_ptr, n_pairs, d_topic_tenant_ptr, stream,
                                          C.byref(out)))
        return DeliveryResult(out)

    def delivery_ordered(self, d_offsets_ptr, d_ranks_ptr, n_pairs, d_topic_tenant_ptr, d_pub_off_ptr, d_pub_hash_ptr, n_pubs,
                         stream=0):
        """bfq_delivery_device_ordered: delivery() with every $oshare pair resolved per publisher. d_pub_off_ptr: int64
        [n_topics + 1] publisher packs per topic position, d_pub_hash_ptr: int32 [n_pubs] each publisher's
        ClientInfo.hashCode() (device). -> DeliveryResult whose nesting() also gives each pack's publisher positions"""
        out = N.BfqDeliveryOrderedResult()
        N.check(N.lib.bfq_delivery_device_ordered(C.byref(self.raw), d_offsets_ptr, d_ranks_ptr, n_pairs, d_topic_tenant_ptr,
                                                  d_pub_off_ptr, d_pub_hash_ptr, n_pubs, stream, C.byref(out)))
        return DeliveryResult(out.d, out)

    def delivery_wire(self, nesting, tenants, d_topics_ptr, d_topic_off_ptr, d_pub_off_ptr, d_pubpack_ptr, d_pubpack_off_ptr,
                      d_out_ptr, out_cap, stream=0):
        """bfq_delivery_encode[_ordered]: `nesting` (the latest delivery() or delivery_ordered() of this result) as one
        serialized DeliveryRequest per deliverer. tenants: the match's tenant list (or tenant_blob(...)); topics as the match
        took them; d_pub_off_ptr: int64 [n_topics + 1] publisher packs per topic position, d_pubpack_ptr / d_pubpack_off_ptr
        (int64 [n_pubs + 1]) their serialized TopicMessagePack.PublisherPack bytes (device). Bytes go to d_out_ptr only if they
        fit out_cap (d_out_ptr = None only sizes). -> BfqDeliveryWireResult: deliverer d's request is
        out[d_req_off[d] .. d_req_off[d + 1])"""
        tb, toff, nt = GpuRouteIndex._tenants(tenants)
        out = N.BfqDeliveryWireResult()
        args = (N.ptr(tb), N.ptr(toff), nt, d_topics_ptr, d_topic_off_ptr, d_pub_off_ptr, d_pubpack_ptr, d_pubpack_off_ptr,
                d_out_ptr, out_cap, stream, C.byref(out))
        if nesting.ordered is not None:
            N.check(N.lib.bfq_delivery_encode_ordered(C.byref(self.raw), C.byref(nesting.ordered), *args))
        else:
            N.check(N.lib.bfq_delivery_encode(C.byref(self.raw), C.byref(nesting.raw), *args))
        return out

    def delivery_reply(self, nesting, tenants, d_reply_ptr, d_reply_off_ptr, stream=0):
        """bfq_delivery_reply: every deliverer's serialized DeliveryReply (device bytes; deliverer d's is
        reply[reply_off[d] .. reply_off[d + 1]), int64 offsets) joined back to the pairs of `nesting` (the latest delivery() or
        delivery_ordered() of this result, the one its requests were encoded from). tenants: the match's tenant list.
        -> BfqDeliveryReplyResult: d_pair_code per pair, d_status per deliverer, d_stale (BfqStaleMatch) per stale MatchInfo"""
        tb, toff, nt = GpuRouteIndex._tenants(tenants)
        out = N.BfqDeliveryReplyResult()
        N.check(N.lib.bfq_delivery_reply(C.byref(self.raw), C.byref(nesting.raw), N.ptr(tb), N.ptr(toff), nt, d_reply_ptr,
                                         d_reply_off_ptr, stream, C.byref(out)))
        return out

    def release(self):
        if getattr(self, "raw", None) is not None and self.raw.lease:
            N.lib.bfq_device_result_release(C.byref(self.raw))

    close = release

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class GpuRouteIndex:
    def __init__(self, device=0):
        h = C.c_void_p()
        N.check(N.lib.bfq_index_create(device, C.byref(h)))
        self._h = h
        self.device = device

    def close(self):
        if getattr(self, "_h", None):
            N.lib.bfq_index_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    # ---- feed
    def reset(self):
        N.check(N.lib.bfq_index_reset(self._h))

    def load(self, keys, key_off, vals, val_off):
        """bulk stage sorted raw KV pairs given as (uint8 blob, int64 offsets) or raw pointers"""
        n = len(key_off) - 1
        N.check(N.lib.bfq_index_load(self._h, N.ptr(keys), N.ptr(key_off), N.ptr(vals), N.ptr(val_off), n))

    def load_ptrs(self, keys_ptr, key_off_ptr, vals_ptr, val_off_ptr, n):
        N.check(N.lib.bfq_index_load(self._h, keys_ptr, key_off_ptr, vals_ptr, val_off_ptr, n))

    def load_pairs(self, pairs):
        pairs = sorted(pairs)
        k, ko = N.as_blob([p[0] for p in pairs])
        v, vo = N.as_blob([p[1] for p in pairs])
        self.load(k, ko, v, vo)

    def apply(self, adds=(), dels=()):
        adds, dels = list(adds), list(dels)
        ak, ako = N.as_blob([a[0] for a in adds])
        av, avo = N.as_blob([a[1] for a in adds])
        dk, dko = N.as_blob(dels)
        N.check(N.lib.bfq_index_apply(self._h, N.ptr(ak), N.ptr(ako), N.ptr(av), N.ptr(avo), len(adds), N.ptr(dk), N.ptr(dko), len(dels)))

    def commit(self):
        N.check(N.lib.bfq_index_commit(self._h))

    def stats(self):
        s = np.zeros(23, np.int64)
        N.check(N.lib.bfq_index_stats(self._h, s.ctypes.data, len(s)))
        names = ["routes", "tenants", "nodes", "slots", "device_bytes", "max_nodes_per_depth", "launches",
                 "overflow_topics", "flagged_topics", "multi_segment_filters", "long_token_chunks", "deferred_topics",
                 "duplicate_topics", "full_commits", "delta_commits", "garbage_slots", "buffer_retries", "global_fanouts",
                 "tag_usable_slots", "tag_used_slots", "tag_overflowed_blocks", "rebuilt_tenants", "wire_table_bytes"]
        return dict(zip(names, s.tolist()))

    def deliverer(self, deliverer_id):
        """(subBrokerId, delivererKey bytes) of a fan-out deliverer id"""
        broker, kl = C.c_int32(0), C.c_int64(0)
        N.check(N.lib.bfq_fanout_deliverer(self._h, int(deliverer_id), C.byref(broker), None, 0, C.byref(kl)))
        kb = C.create_string_buffer(max(kl.value, 1))
        N.check(N.lib.bfq_fanout_deliverer(self._h, int(deliverer_id), C.byref(broker), C.addressof(kb), kl.value, C.byref(kl)))
        return broker.value, kb.raw[:kl.value]

    def set_option(self, name, value):
        N.check(N.lib.bfq_index_set_option(self._h, name.encode(), int(value)))

    def generation(self):
        g = C.c_uint64(0)
        N.check(N.lib.bfq_index_generation(self._h, C.byref(g)))
        return g.value

    def last_kernel_ms(self):
        ms = C.c_double(0)
        N.check(N.lib.bfq_index_last_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    # ---- lookups
    def route(self, rank):
        kl, vl = C.c_int64(0), C.c_int64(0)
        N.check(N.lib.bfq_route_lookup(self._h, int(rank), None, 0, C.byref(kl), None, 0, C.byref(vl)))
        kb, vb = C.create_string_buffer(max(kl.value, 1)), C.create_string_buffer(max(vl.value, 1))
        N.check(N.lib.bfq_route_lookup(self._h, int(rank), C.addressof(kb), kl.value, C.byref(kl), C.addressof(vb), vl.value, C.byref(vl)))
        return kb.raw[:kl.value], vb.raw[:vl.value]

    def route_kinds(self, ranks):
        ranks = np.ascontiguousarray(ranks, dtype=np.int64)
        out = np.zeros(max(len(ranks), 1), np.uint8)
        N.check(N.lib.bfq_route_kinds(self._h, ranks.ctypes.data, len(ranks), out.ctypes.data))
        return out[:len(ranks)]

    # ---- match
    @staticmethod
    def tenant_blob(tenants):
        """pre-marshal a tenant list once when the same list is used for many batches"""
        tb, toff = N.as_blob(tenants)
        return ("blob", tb, toff, len(tenants))

    @staticmethod
    def _tenants(tenants):
        if isinstance(tenants, tuple) and tenants and tenants[0] == "blob":
            return tenants[1], tenants[2], tenants[3]
        tb, toff = N.as_blob(tenants)
        return tb, toff, len(tenants)

    def match(self, tenants, topics_blob, topic_off, topic_tenant, max_pfanout=None, max_gfanout=None):
        """tenants: list[str] (or tenant_blob(...)); topics as (uint8 blob, int64 offsets[n+1]); topic_tenant int32[n];
        caps per tenant."""
        tb, toff, nt = self._tenants(tenants)
        n = len(topic_off) - 1
        mp = np.full(max(nt, 1), INT_MAX, np.int32) if max_pfanout is None else np.ascontiguousarray(max_pfanout, dtype=np.int32)
        mg = np.full(max(nt, 1), INT_MAX, np.int32) if max_gfanout is None else np.ascontiguousarray(max_gfanout, dtype=np.int32)
        tt = np.ascontiguousarray(topic_tenant, dtype=np.int32)
        r = C.c_void_p()
        N.check(N.lib.bfq_match(self._h, N.ptr(tb), N.ptr(toff), nt, N.ptr(topics_blob), N.ptr(topic_off), N.ptr(tt), n,
                                N.ptr(mp), N.ptr(mg), C.byref(r)))
        return BatchResult(r, n, self)

    def match_topics(self, tenants, topics, topic_tenant=None, max_pfanout=None, max_gfanout=None):
        blob, off = N.as_blob(topics)
        tt = np.zeros(max(len(topics), 1), np.int32) if topic_tenant is None else topic_tenant
        return self.match(tenants, blob, off, tt, max_pfanout, max_gfanout)

    def match_device(self, tenants, d_topics_ptr, d_topic_off_ptr, d_topic_tenant_ptr, n, max_pfanout=None,
                     max_gfanout=None, stream=0, wait=True):
        """batch resident in device memory, result left there. wait=False only enqueues (bfq_match_device_async): call
        .wait() on the returned DeviceResult before reading its counts; .release() hands the buffers back."""
        tb, toff, nt = self._tenants(tenants)
        mp = np.full(max(nt, 1), INT_MAX, np.int32) if max_pfanout is None else np.ascontiguousarray(max_pfanout, dtype=np.int32)
        mg = np.full(max(nt, 1), INT_MAX, np.int32) if max_gfanout is None else np.ascontiguousarray(max_gfanout, dtype=np.int32)
        out = N.BfqDeviceResult()
        fn = N.lib.bfq_match_device if wait else N.lib.bfq_match_device_async
        N.check(fn(self._h, N.ptr(tb), N.ptr(toff), nt, d_topics_ptr, d_topic_off_ptr, d_topic_tenant_ptr,
                   n, N.ptr(mp), N.ptr(mg), stream, C.byref(out)))
        return DeviceResult(out, self)


class MatchedRoutes:
    """Read side of IMatchedRoutes for one (tenant, topic)."""

    def __init__(self, tenant_id, topic, max_persistent_fanout, max_group_fanout, routes, persistent_fanout, group_fanout):
        self.tenant_id, self.topic = tenant_id, topic
        self._max_p, self._max_g = max_persistent_fanout, max_group_fanout
        self._routes, self._pf, self._gf = routes, persistent_fanout, group_fanout

    def max_persistent_fanout(self):
        return self._max_p

    def max_group_fanout(self):
        return self._max_g

    def persistent_fanout(self):
        return self._pf

    def group_fanout(self):
        return self._gf

    def routes(self):
        return self._routes


class GpuTenantRouteMatcher:
    def __init__(self, tenant_id, index, event_collector=None):
        self.tenant_id = tenant_id
        self.index = index
        self.event_collector = event_collector  # callable(event) or object with .report(event)

    def _report(self, ev):
        if self.event_collector is None:
            return
        if callable(self.event_collector):
            self.event_collector(ev)
        else:
            self.event_collector.report(ev)

    def match_all(self, topics, max_persistent_fanout_count, max_group_fanout_count):
        topics = list(topics)
        res = self.index.match_topics([self.tenant_id], topics, None, [max_persistent_fanout_count], [max_group_fanout_count])
        offsets, ranks = res.expand()
        kinds = res.route_kinds(ranks)   # resolved against the snapshot the match ran on
        out = {}
        cache = {}

        def matching(rank):
            m = cache.get(rank)
            if m is None:
                m = cache[rank] = schema.build_match_route(*res.route(rank))
            return m
        for i, topic in enumerate(topics):
            rk = ranks[offsets[i]:offsets[i + 1]]
            kd = kinds[offsets[i]:offsets[i + 1]]
            out[topic] = MatchedRoutes(self.tenant_id, topic, max_persistent_fanout_count, max_group_fanout_count,
                                       {matching(int(r)) for r in rk}, int((kd == 1).sum()), int((kd == 2).sum()))
        for t, rank, kind in res.throttled.tolist():
            m = matching(int(rank))
            cls = PersistentFanoutThrottled if kind == 1 else GroupFanoutThrottled
            self._report(cls(self.tenant_id, topics[t], m.mqtt_topic_filter,
                             max_persistent_fanout_count if kind == 1 else max_group_fanout_count))
        res.close()
        return out
