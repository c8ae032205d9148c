"""Host-side mirror of the reference's inverse-match indexes, backed by the CUDA library (bfq_rindex):

* GpuRetainTopicIndex — IRetainTopicIndex{add, remove, match, findAll}
  (bifromq-retain/bifromq-retain-store/src/main/java/org/apache/bifromq/retain/store/index/IRetainTopicIndex.java:27-35,
   implementation replaced: RetainTopicIndex.java:35-144). Mutations are staged; commit() publishes a device snapshot
  (the reference rebuilds its index the same way in RetainStoreCoProc.load, RetainStoreCoProc.java:279-296).
* GpuTopicIndex — TopicIndex<V>{add, remove, get, match}
  (bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/TopicIndex.java:39-156), values kept host-side.
"""
import ctypes as C

import numpy as np

from . import _native as N


class RMatchResult:
    def __init__(self, handle, index_handle=None, with_retain_keys=False):
        lib = N.lib
        n = lib.bfq_rresult_num_filters(handle)
        self.n_filters = n

        def arr(p, count):
            if count == 0 or not p:
                return np.zeros(0, np.int64)
            return np.frombuffer((C.c_uint8 * (count * 8)).from_address(p), dtype=np.int64).copy()
        self.offsets = arr(lib.bfq_rresult_offsets(handle), n + 1) if n else np.zeros(1, np.int64)
        nid = C.c_int64(0)
        p = lib.bfq_rresult_ids(handle, C.byref(nid))
        self.ids = arr(p, nid.value)
        self.totals = arr(lib.bfq_rresult_total_matches(handle), n)
        ms = np.zeros(8, np.float64)
        lib.bfq_rresult_timings(handle, ms.ctypes.data, 8)
        self.timings_ms = dict(zip(["h2d", "kernels", "d2h", "total", "device_all_kernels", "device_rmatch_kernel"], ms[:6].tolist()))
        self.n_ranges, self.n_overflow_filters = int(ms[6]), int(ms[7])
        self.generation = int(lib.bfq_rresult_generation(handle))
        self.retain_keys = None
        if with_retain_keys and index_handle is not None:
            # the keys of RetainStoreCoProc.match's follow-up reader.get calls, as one batch (bfq_rresult_retain_keys)
            koff = np.zeros(len(self.ids) + 1, np.int64)
            total = lib.bfq_rresult_retain_keys(index_handle, handle, None, 0, koff.ctypes.data)
            if total < 0:
                lib.bfq_rresult_free(handle)
                raise N.NativeError("bfq_rresult_retain_keys: %d" % total)
            blob = np.zeros(max(total, 1), np.uint8)
            lib.bfq_rresult_retain_keys(index_handle, handle, blob.ctypes.data, total, koff.ctypes.data)
            self.retain_keys = (blob[:total], koff)
        lib.bfq_rresult_free(handle)

    def matches(self, i):
        return self.ids[self.offsets[i]:self.offsets[i + 1]]


class RDeviceResult:
    """One bfq_rmatch_device result: device pointers (d_offsets, d_ids, d_total) + counts; the arrays stay valid until
    release()."""

    def __init__(self, raw, owner):
        self.raw = raw
        self._owner = owner   # the index: keeps it alive for as long as this result is

    def __getattr__(self, name):   # d_ids, n_ids, generation, kernel_ms, ... straight from the C struct
        if name == "raw":
            raise AttributeError(name)
        return getattr(self.raw, name)

    def retain_keys_device(self, d_key_off_ptr, d_keys_ptr, cap, stream=0):
        """bfq_rretain_keys_device: the retainMessageKey of every id, in result order, gathered on the device. d_key_off_ptr:
        int64 [n_ids + 1] (always written); the bytes go to d_keys_ptr only if they fit cap (None only sizes). -> total bytes"""
        n = C.c_int64(0)
        N.check(N.lib.bfq_rretain_keys_device(self._owner._h, C.byref(self.raw), d_key_off_ptr, d_keys_ptr, cap, stream, C.byref(n)))
        return n.value

    def release(self):
        if getattr(self, "raw", None) is not None and self.raw.lease:
            N.lib.bfq_rdevice_result_release(C.byref(self.raw))

    close = release

    def __del__(self):
        try:
            self.release()
        except Exception:
            pass


class GpuTopicMatchIndex:
    """thin wrapper over bfq_rindex_*"""

    def __init__(self, device=0):
        h = C.c_void_p()
        N.check(N.lib.bfq_rindex_create(device, C.byref(h)))
        self._h = h

    def close(self):
        if getattr(self, "_h", None):
            N.lib.bfq_rindex_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()

    def reset(self):
        N.check(N.lib.bfq_rindex_reset(self._h))

    def add_blobs(self, tenants, topics_blob, topic_off, topic_tenant):
        tb, toff = N.as_blob(tenants)
        n = len(topic_off) - 1
        ids = np.zeros(max(n, 1), np.int64)
        tt = np.ascontiguousarray(topic_tenant, dtype=np.int32)
        N.check(N.lib.bfq_rindex_add(self._h, N.ptr(tb), N.ptr(toff), len(tenants), N.ptr(topics_blob), N.ptr(topic_off), N.ptr(tt), n, N.ptr(ids)))
        return ids[:n]

    def add(self, tenant, topics):
        blob, off = N.as_blob(topics)
        return self.add_blobs([tenant], blob, off, np.zeros(max(len(topics), 1), np.int32))

    def remove(self, tenant, topic):
        t = tenant.encode() if isinstance(tenant, str) else tenant
        p = topic.encode() if isinstance(topic, str) else topic
        N.check(N.lib.bfq_rindex_remove(self._h, t, len(t), p, len(p)))

    def commit(self):
        N.check(N.lib.bfq_rindex_commit(self._h))

    STAT_NAMES = ["topics", "tenants", "nodes", "garbage_nodes", "used_slots", "usable_slots", "full_commits", "delta_commits",
                  "rebuilt_tenants", "device_bytes", "overflowed_blocks", "workspaces", "workspace_bytes", "key_table_bytes"]

    def stats(self):
        """bfq_rindex_stats of the committed snapshot, by name"""
        s = np.zeros(len(self.STAT_NAMES), np.int64)
        N.check(N.lib.bfq_rindex_stats(self._h, s.ctypes.data, len(s)))
        return dict(zip(self.STAT_NAMES, s.tolist()))

    def lookup(self, topic_id):
        tl, pl = C.c_int64(0), C.c_int64(0)
        N.check(N.lib.bfq_rindex_lookup(self._h, int(topic_id), None, 0, C.byref(tl), None, 0, C.byref(pl)))
        tb, pb = C.create_string_buffer(max(tl.value, 1)), C.create_string_buffer(max(pl.value, 1))
        N.check(N.lib.bfq_rindex_lookup(self._h, int(topic_id), C.addressof(tb), tl.value, C.byref(tl), C.addressof(pb), pl.value, C.byref(pl)))
        return tb.raw[:tl.value].decode(), pb.raw[:pl.value].decode()

    def load_keys(self, keys_blob, key_off):
        """bfq_rindex_load_keys: the feed of RetainStoreCoProc.load() — raw retain-store KV keys of a range scan -> topic ids
        (-1 for bytes that are not a retain key)"""
        n = len(key_off) - 1
        ids = np.zeros(max(n, 1), np.int64)
        N.check(N.lib.bfq_rindex_load_keys(self._h, N.ptr(keys_blob), N.ptr(np.ascontiguousarray(key_off, dtype=np.int64)), n, ids.ctypes.data))
        return ids[:n]

    def match_blobs(self, tenants, filters_blob, filter_off, filter_tenant, limit=None, with_retain_keys=False):
        tb, toff = N.as_blob(tenants)
        n = len(filter_off) - 1
        ft = np.ascontiguousarray(filter_tenant, dtype=np.int32)
        lim = None if limit is None else np.ascontiguousarray(limit, dtype=np.int64)
        r = C.c_void_p()
        N.check(N.lib.bfq_rmatch(self._h, N.ptr(tb), N.ptr(toff), len(tenants), N.ptr(filters_blob), N.ptr(filter_off), N.ptr(ft), n,
                                 N.ptr(lim) if lim is not None else None, C.byref(r)))
        return RMatchResult(r, self._h, with_retain_keys)

    def match_device(self, tenants, d_filters_ptr, d_filter_off_ptr, d_filter_tenant_ptr, n, d_limit_ptr=None, stream=0):
        """bfq_rmatch_device: n filters already in device memory (uint8 blob, int64 offsets [n + 1], int32 tenant index per
        filter, optional int64 limit per filter; None = unlimited), written on `stream`. -> RDeviceResult, ready when returned"""
        tb, toff = N.as_blob(tenants)
        out = N.BfqRDeviceResult()
        N.check(N.lib.bfq_rmatch_device(self._h, N.ptr(tb), N.ptr(toff), len(tenants), d_filters_ptr, d_filter_off_ptr,
                                        d_filter_tenant_ptr, n, d_limit_ptr, stream, C.byref(out)))
        return RDeviceResult(out, self)

    def match(self, tenant, filters, limit=None):
        blob, off = N.as_blob(filters)
        lim = None if limit is None else np.full(max(len(filters), 1), limit, np.int64)
        return self.match_blobs([tenant], blob, off, np.zeros(max(len(filters), 1), np.int32), lim)


class GpuRetainTopicIndex:
    def __init__(self, device=0):
        self._idx = GpuTopicMatchIndex(device)
        self._info = {}   # topic id -> (tenant, topic, timestamp, expiry_seconds)  == RetainedMsgInfo
        self._dirty = True

    def add(self, tenant_id, topic, timestamp=0, expiry_seconds=0):
        tid = int(self._idx.add(tenant_id, [topic])[0])
        self._info[tid] = (tenant_id, topic, timestamp, expiry_seconds)
        self._dirty = True

    def remove(self, tenant_id, topic):
        self._idx.remove(tenant_id, topic)
        self._dirty = True

    def _sync(self):
        if self._dirty:
            self._idx.commit()
            self._dirty = False

    def match(self, tenant_id, topic_filter, limit=None):
        self._sync()
        r = self._idx.match(tenant_id, [topic_filter], limit)
        return {self._info[int(i)] for i in r.matches(0)}

    def find_all(self):
        """RetainTopicIndex.findAll (RetainTopicIndex.java:141-143): every indexed topic, '$' topics included —
        '#' plus the per-'$'-root filters cover the whole trie."""
        self._sync()
        out = set()
        for tenant in {v[0] for v in self._info.values()}:
            sys_roots = {v[1].split("/")[0] for v in self._info.values() if v[0] == tenant and v[1].startswith("$")}
            filters = ["#"] + [r + "/#" for r in sorted(sys_roots)]
            r = self._idx.match(tenant, filters)
            for i in range(len(filters)):
                out |= {self._info[int(x)] for x in r.matches(i)}
        return out


class GpuTopicIndex:
    """TopicIndex<V>: topic -> set of values, matched by filters (no tenant level: one implicit tenant)."""
    _TENANT = "_"

    def __init__(self, device=0):
        self._idx = GpuTopicMatchIndex(device)
        self._values = {}   # topic -> set(values)
        self._ids = {}      # topic id -> topic
        self._dirty = True

    def add(self, topic, value):
        if topic not in self._values:
            tid = int(self._idx.add(self._TENANT, [topic])[0])
            self._ids[tid] = topic
            self._values[topic] = set()
            self._dirty = True
        self._values[topic].add(value)

    def remove(self, topic, value):
        vs = self._values.get(topic)
        if vs is None:
            return
        vs.discard(value)
        if not vs:
            del self._values[topic]
            self._idx.remove(self._TENANT, topic)
            self._dirty = True

    def get(self, topic):
        return set(self._values.get(topic, ()))

    def match(self, topic_filter):
        if self._dirty:
            self._idx.commit()
            self._dirty = False
        r = self._idx.match(self._TENANT, [topic_filter])
        out = set()
        for i in r.matches(0):
            out |= self._values.get(self._ids[int(i)], set())
        return out
