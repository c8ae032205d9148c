"""The inverse match on device-resident batches (bfq_rmatch_device), the host call over the same core (bfq_rmatch), concurrent
matches on one handle with commits running beside them, the leased workspaces, and retain keys gathered on the device
(bfq_rretain_keys_device).

Both calls run one match (rmatch_kernels.cu: rmatch_core), so every case compares the two with each other (offsets, ids in
order, totals, range and tier-2 counts) and with the CPU oracle. The cases of test_gpu_inverse_edges.py (tier-1 limits, the
level-0 '$' cuts, long filters, tier 2, the range-buffer re-run on a fresh handle) are re-run through the device call.
"""
import random
import threading

import numpy as np
import pytest

import oracle_lib as O
import test_gpu_inverse_edges as E


@pytest.fixture(scope="module")
def R():
    import torch

    import bifromq_b200
    from bifromq_b200 import _native, retain, workload
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.N, ns.retain, ns.workload, ns.torch = _native, retain, workload, torch
    ns.dev = torch.device("cuda", 0)
    return ns


class Batch:
    """a filter batch on the host and on the device"""

    def __init__(self, R, filters, tenants=None, limit=None):
        self.tenants = tenants or E.tenants_of(filters) or ["t"]
        self.filters = filters
        self.blob, self.off = R.N.as_blob([f for _, f in filters])
        self.ft = np.array([self.tenants.index(t) for t, _ in filters] or [0], np.int32)
        self.limit = None if limit is None else np.ascontiguousarray(limit, np.int64)
        t = R.torch
        self.d_blob = t.from_numpy(self.blob).to(R.dev)
        self.d_off = t.from_numpy(self.off).to(R.dev)
        self.d_ft = t.from_numpy(self.ft).to(R.dev)
        self.d_limit = None if self.limit is None else t.from_numpy(self.limit).to(R.dev)
        t.cuda.synchronize()
        self.n = len(filters)

    def host(self, idx, with_keys=False):
        return idx.match_blobs(self.tenants, self.blob, self.off, self.ft, self.limit, with_retain_keys=with_keys)

    def device(self, idx, stream=0):
        return idx.match_device(self.tenants, self.d_blob.data_ptr(), self.d_off.data_ptr(), self.d_ft.data_ptr(), self.n,
                                None if self.d_limit is None else self.d_limit.data_ptr(), stream)


class _DevArray:
    """an int64 device array the library owns, seen by torch through __cuda_array_interface__ (read only here)"""

    def __init__(self, ptr, count):
        self.__cuda_array_interface__ = {"shape": (count,), "typestr": "<i8", "data": (ptr, False), "version": 3, "strides": None}


def fetch(R, dres):
    """a device result's arrays on the host -> (offsets, ids, totals)"""
    t = R.torch

    def arr(p, count):
        if count == 0:
            return []
        return t.as_tensor(_DevArray(p, count), device=R.dev).cpu().tolist()
    return arr(dres.d_offsets, dres.n_filters + 1), arr(dres.d_ids, dres.n_ids), arr(dres.d_total, dres.n_filters)


def same(R, host, dres):
    """the device result equals the host result of the same batch"""
    off, ids, tot = fetch(R, dres)
    assert dres.n_filters == host.n_filters
    assert off == host.offsets.tolist()
    assert ids == host.ids.tolist()
    assert tot == host.totals.tolist()
    assert (dres.n_ranges, dres.n_overflow_filters) == (host.n_ranges, host.n_overflow_filters)
    assert dres.generation == host.generation
    return off, ids, tot


def device_keys(R, idx, dres, stream=0):
    """bfq_rretain_keys_device -> list of keys (bytes)"""
    t = R.torch
    koff = t.zeros(dres.n_ids + 1, dtype=t.int64, device=R.dev)
    total = dres.retain_keys_device(koff.data_ptr(), None, 0, stream)
    keys = t.zeros(max(total, 1), dtype=t.uint8, device=R.dev)
    assert dres.retain_keys_device(koff.data_ptr(), keys.data_ptr(), total, stream) == total
    t.cuda.synchronize()
    o, b = koff.cpu().numpy(), keys.cpu().numpy()
    assert o[-1] == total
    return [bytes(b[o[j]:o[j + 1]]) for j in range(dres.n_ids)]


# ------------------------------------------------------------------ same answers
LIMITS = [None, 0, 1, 10]


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(E.CASES))
def test_cases_device_equals_host_and_oracle(R, case):
    topics, filters = E.CASES[case]()
    idx, entries = E.make_index(R, topics)
    exp = E.Expect(entries)
    for lim in LIMITS:
        b = Batch(R, filters, limit=None if lim is None else [lim] * len(filters))
        host = b.host(idx)
        d = b.device(idx)
        try:
            off, ids, tot = same(R, host, d)
            if lim is None:
                E.check(host, exp, filters)
            else:
                full = Batch(R, filters).host(idx)
                assert tot == full.totals.tolist()
                for i in range(len(filters)):
                    assert host.matches(i).tolist() == full.matches(i).tolist()[:lim]
        finally:
            d.release()


@pytest.mark.gpu
def test_c5_scaled_device_and_host_against_the_oracle(R):
    w = R.workload.Workload("C5", scale=0.1)
    assert w.n_query_filters >= E.ORDER_MIN_FILTERS
    idx = R.retain.GpuTopicMatchIndex(0)
    ids = idx.add_blobs(w.tenants, w.topics, w.topic_off, w.topic_tenant[:w.n_topics])
    idx.commit()
    orc = O.TopicLevelIndex()
    tl = w.topic_list()
    for i in range(w.n_topics):
        orc.add(tl[i], int(ids[i]), w.tenants[w.topic_tenant[i]])
    fl = w.query_filter_list()
    ft = w.filter_tenant[:w.n_query_filters]
    filters = [(w.tenants[ft[i]], fl[i]) for i in range(w.n_query_filters)]
    full = None
    for lim in LIMITS:
        b = Batch(R, filters, tenants=list(w.tenants), limit=None if lim is None else [lim] * len(filters))
        host = b.host(idx)
        d = b.device(idx)
        try:
            same(R, host, d)
        finally:
            d.release()
        if lim is None:
            full = host
            for i in range(0, w.n_query_filters, 7):
                got = host.matches(i).tolist()
                assert sorted(got) == orc.match(fl[i], w.tenants[ft[i]]) and len(set(got)) == len(got)
        else:
            assert host.totals.tolist() == full.totals.tolist()
            for i in range(0, w.n_query_filters, 3):
                assert host.matches(i).tolist() == full.matches(i).tolist()[:lim]


@pytest.mark.gpu
@pytest.mark.parametrize("w", [64, 65])
def test_range_buffer_grows_on_a_fresh_handle_through_the_device_call(R, w):
    topics, filters = E.rerun_case(w)
    b = Batch(R, filters)
    idx, entries = E.make_index(R, topics)
    d = b.device(idx)                       # the first call on the handle: the workspace's range buffer starts small
    try:
        assert d.n_ranges == w * len(filters) and d.n_ranges > E.initial_range_cap(len(filters))
        assert d.n_overflow_filters == (len(filters) if w > 64 else 0)
        host = b.host(idx)
        E.check(host, E.Expect(entries), filters)
        same(R, host, d)
    finally:
        d.release()


# ------------------------------------------------------------------ concurrency
class History:
    """the commit thread's record: per generation, the add / remove ops since the last reset and the live entries"""

    def __init__(self):
        self.ops, self.entries, self.nxt = [], {}, 0
        self.at = {}

    def add(self, idx, R, pairs):
        tenants = E.tenants_of(pairs)
        blob, off = R.N.as_blob([p for _, p in pairs])
        got = idx.add_blobs(tenants, blob, off, np.array([tenants.index(t) for t, _ in pairs], np.int32)).tolist()
        for k, i in zip(pairs, got):
            if k not in self.entries:
                assert i == self.nxt
                self.nxt += 1
            self.entries[k] = i
        self.ops.append(("add", list(pairs)))

    def remove(self, idx, pair):
        idx.remove(*pair)
        self.entries.pop(pair, None)
        self.ops.append(("remove", pair))

    def reset(self, idx):
        idx.reset()
        self.ops, self.entries, self.nxt = [], {}, 0

    def committed(self, gen):
        self.at[gen] = (list(self.ops), dict(self.entries))


def twin_answer(R, ops, batch):
    """a fresh handle given the same add / remove history, committed once, matched serially"""
    twin = R.retain.GpuTopicMatchIndex(0)
    h = History()
    for op, arg in ops:
        if op == "add":
            h.add(twin, R, arg)
        else:
            h.remove(twin, arg)
    twin.commit()
    r = batch.host(twin)
    twin.close()
    return r


@pytest.mark.gpu
def test_eight_matching_threads_and_a_committing_one(R):
    topics, filters = E.dollar_case()
    extra = [("d_mix", "a/c%d" % i) for i in range(40)] + [("d_hi", "z/%d/q" % i) for i in range(40)]
    batches = [Batch(R, filters), Batch(R, filters[::3], limit=[2] * len(filters[::3]))]
    idx = R.retain.GpuTopicMatchIndex(0)
    hist = History()
    hist.add(idx, R, topics)
    idx.commit()
    gen = 1
    hist.committed(gen)
    results = []   # (kind, batch index, generation, offsets, ids, totals, keys)
    errors = []
    stop = threading.Event()
    lock = threading.Lock()

    def matcher(k):
        try:
            s = R.torch.cuda.Stream(R.dev)
            rng = random.Random(k)
            for it in range(12):
                bi = rng.randrange(len(batches))
                b = batches[bi]
                if (k + it) % 2 == 0:
                    r = b.host(idx, with_keys=True)
                    blob, koff = r.retain_keys
                    keys = [bytes(blob[koff[j]:koff[j + 1]]) for j in range(len(r.ids))]
                    rec = ("host", bi, r.generation, r.offsets.tolist(), r.ids.tolist(), r.totals.tolist(), keys)
                else:
                    d = b.device(idx, s.cuda_stream)
                    try:
                        off, ids, tot = fetch(R, d)
                        keys = device_keys(R, idx, d, s.cuda_stream)
                        rec = ("device", bi, d.generation, off, ids, tot, keys)
                    finally:
                        d.release()
                with lock:
                    results.append(rec)
        except Exception as e:   # reported by the main thread
            errors.append(e)

    def committer():
        nonlocal gen
        try:
            rng = random.Random(99)
            cyc = 0
            while not stop.is_set() and cyc < 10:
                cyc += 1
                if cyc % 4 == 0:          # reset and reload: a full build, ids restart at 0
                    live = list(hist.entries)
                    hist.reset(idx)
                    rng.shuffle(live)
                    hist.add(idx, R, live)
                else:                     # a few adds and removes: a delta commit
                    hist.add(idx, R, rng.sample(extra, 6))
                    for p in rng.sample(sorted(hist.entries), 4):
                        hist.remove(idx, p)
                idx.commit()
                gen += 1
                hist.committed(gen)
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=matcher, args=(k,)) for k in range(8)] + [threading.Thread(target=committer)]
    for t in threads:
        t.start()
    for t in threads[:8]:
        t.join()
    stop.set()
    threads[8].join()
    assert not errors, errors
    st = idx.stats()
    assert st["full_commits"] >= 2 and st["delta_commits"] >= 2
    assert len(results) == 8 * 12
    seen_gens = set()
    twins = {}
    for kind, bi, g, off, ids, tot, keys in results:
        ops, entries = hist.at[g]
        seen_gens.add(g)
        if (g, bi) not in twins:
            twins[(g, bi)] = twin_answer(R, ops, batches[bi])
        want = twins[(g, bi)]
        assert off == want.offsets.tolist(), (kind, g)
        assert ids == want.ids.tolist(), (kind, g)
        assert tot == want.totals.tolist(), (kind, g)
        name = {i: k for k, i in entries.items()}
        assert keys == [O.retain_key(*name[i]) for i in ids], (kind, g)
    assert {k for k, *_ in results} == {"host", "device"}
    assert len(seen_gens) >= 1


@pytest.mark.gpu
def test_results_held_across_commits_and_a_reset_keep_their_ids_and_keys(R):
    old = [("t", "old/%d" % i) for i in range(6)] + [("u", "x/é/%d" % i) for i in range(4)]
    new = [("t", "new/%d" % i) for i in range(10)]
    idx = R.retain.GpuTopicMatchIndex(0)
    h = History()
    h.add(idx, R, old)
    idx.commit()
    b = Batch(R, [("t", "#"), ("u", "x/+/#")])
    d1 = b.device(idx)
    try:
        off1, ids1, _ = fetch(R, d1)
        name1 = {i: k for k, i in h.entries.items()}
        want1 = [O.retain_key(*name1[i]) for i in ids1]
        assert sorted(ids1) == list(range(10)) and device_keys(R, idx, d1) == want1
        h.add(idx, R, [("t", "old/x")])          # a delta commit: the result keeps its ids
        idx.commit()
        assert fetch(R, d1)[1] == ids1 and device_keys(R, idx, d1) == want1
        h.reset(idx)                              # reset and reload: every id now names another topic
        h.add(idx, R, new)
        assert idx.stats()["key_table_bytes"] == 0
        idx.commit()
        assert fetch(R, d1)[1] == ids1 and device_keys(R, idx, d1) == want1
        d2 = b.device(idx)
        try:
            _, ids2, _ = fetch(R, d2)
            assert sorted(ids2) == list(range(10))
            assert device_keys(R, idx, d2) == [O.retain_key(*new[i]) for i in ids2]
            assert idx.stats()["key_table_bytes"] > 0
        finally:
            d2.release()
    finally:
        d1.release()


# ------------------------------------------------------------------ workspaces
@pytest.mark.gpu
def test_sequential_calls_reuse_one_workspace_and_held_results_hold_distinct_ones(R):
    topics, filters = E.dollar_case()
    idx, _ = E.make_index(R, topics)
    b = Batch(R, filters)
    assert idx.stats()["workspaces"] == 0
    for _ in range(3):
        b.host(idx)
        b.device(idx).release()
    st = idx.stats()
    assert st["workspaces"] == 1 and st["workspace_bytes"] > 0
    assert st["device_bytes"] >= st["workspace_bytes"] + st["key_table_bytes"]
    held = [b.device(idx) for _ in range(3)]
    try:
        assert idx.stats()["workspaces"] == 3
        assert len({d.d_ids for d in held}) == 3 and len({d.d_offsets for d in held}) == 3
        want = b.host(idx)                     # a fourth workspace while three are leased
        assert idx.stats()["workspaces"] == 4
        for d in held:
            same(R, want, d)
    finally:
        for d in held:
            d.release()
    assert idx.stats()["workspaces"] == 4      # back in the pool


@pytest.mark.gpu
def test_release_waits_for_a_key_gather_on_another_stream(R):
    w = R.workload.Workload("C5", scale=0.1)
    idx = R.retain.GpuTopicMatchIndex(0)
    ids = idx.add_blobs(w.tenants, w.topics, w.topic_off, w.topic_tenant[:w.n_topics])
    idx.commit()
    tl = w.topic_list()
    fl = w.query_filter_list()
    ft = w.filter_tenant[:w.n_query_filters]
    b = Batch(R, [(w.tenants[ft[i]], fl[i]) for i in range(w.n_query_filters)], tenants=list(w.tenants))
    d = b.device(idx)
    t = R.torch
    s = t.cuda.Stream(R.dev)
    koff = t.zeros(d.n_ids + 1, dtype=t.int64, device=R.dev)
    total = d.retain_keys_device(koff.data_ptr(), None, 0, s.cuda_stream)
    keys = t.zeros(total, dtype=t.uint8, device=R.dev)
    _, dids, _ = fetch(R, d)
    assert d.retain_keys_device(koff.data_ptr(), keys.data_ptr(), total, s.cuda_stream) == total
    d.release()                                  # waits for the copy on s
    assert s.query()
    o, kb = koff.cpu().numpy(), keys.cpu().numpy()
    name = {int(ids[i]): (w.tenants[w.topic_tenant[i]], tl[i]) for i in range(w.n_topics)}
    for j in range(0, len(dids), max(1, len(dids) // 5000)):
        assert bytes(kb[o[j]:o[j + 1]]) == O.retain_key(*name[dids[j]])
    assert d.n_ids > 50000


# ------------------------------------------------------------------ keys
KEY_TOPICS = [("t", "é/ü/日本/𝄞"), ("t", "a//b"), ("t", "/"), ("t", ""), ("t", "$SYS/x"), ("t", "$"), ("t", "x" * 255),
              ("t", "/".join(["y"] * 127) + "z"), ("T" * 300, "a/b"), ("é" * 200, "$x/é")]


def host_keys(R, idx, b):
    r = b.host(idx, with_keys=True)
    blob, koff = r.retain_keys
    return r, [bytes(blob[koff[j]:koff[j + 1]]) for j in range(len(r.ids))]


@pytest.mark.gpu
def test_device_keys_are_the_host_keys(R):
    idx = R.retain.GpuTopicMatchIndex(0)
    h = History()
    h.add(idx, R, KEY_TOPICS)
    idx.commit()
    tenants = E.tenants_of(KEY_TOPICS)
    b = Batch(R, [(t, f) for t in tenants for f in ("#", "$SYS/#", "$/#", "$x/#", "+", "+/+")], tenants=tenants)
    r, want = host_keys(R, idx, b)
    d = b.device(idx)
    try:
        assert fetch(R, d)[1] == r.ids.tolist()
        name = {i: k for k, i in h.entries.items()}
        assert want == [O.retain_key(*name[i]) for i in r.ids.tolist()]
        assert device_keys(R, idx, d) == want
        assert set(r.ids.tolist()) == set(range(len(KEY_TOPICS)))
        n_first = len(want)                   # filters overlap ('#' and '+/+' both match '/'): more ids than topics
        assert n_first == 14
        built = idx.stats()["key_table_bytes"]
        assert built > 0
    finally:
        d.release()
    # ids added after the key table was built
    more = [("t", "late/%d/é" % i) for i in range(50)] + [("T" * 300, "late")]
    h.add(idx, R, more)
    idx.commit()
    r, want = host_keys(R, idx, b)
    d = b.device(idx)
    try:
        assert device_keys(R, idx, d) == want
        assert len(want) == n_first + len(more) + 1   # '#' matches each new topic, and '+' the one-level one too
        assert set(r.ids.tolist()) == set(range(len(KEY_TOPICS) + len(more)))
        assert idx.stats()["key_table_bytes"] >= built
    finally:
        d.release()
    # after a reset and reload in another order
    h.reset(idx)
    h.add(idx, R, list(reversed(KEY_TOPICS)))
    idx.commit()
    r, want = host_keys(R, idx, b)
    d = b.device(idx)
    try:
        assert device_keys(R, idx, d) == want
        name = {i: k for k, i in h.entries.items()}
        assert want == [O.retain_key(*name[i]) for i in r.ids.tolist()]
    finally:
        d.release()


@pytest.mark.gpu
def test_key_sizing_and_a_buffer_one_byte_short(R):
    idx = R.retain.GpuTopicMatchIndex(0)
    History().add(idx, R, KEY_TOPICS)
    idx.commit()
    b = Batch(R, [("t", "#")])
    d = b.device(idx)
    t = R.torch
    try:
        koff = t.full((d.n_ids + 1,), -7, dtype=t.int64, device=R.dev)
        total = d.retain_keys_device(koff.data_ptr(), None, 0)
        t.cuda.synchronize()
        o = koff.cpu().tolist()
        assert o[0] == 0 and o[-1] == total and all(x < y for x, y in zip(o, o[1:]))
        buf = t.full((total,), 0xAB, dtype=t.uint8, device=R.dev)
        koff2 = t.zeros(d.n_ids + 1, dtype=t.int64, device=R.dev)
        assert d.retain_keys_device(koff2.data_ptr(), buf.data_ptr(), total - 1) == total
        t.cuda.synchronize()
        assert koff2.cpu().tolist() == o                 # offsets always written
        assert (buf.cpu().numpy() == 0xAB).all()         # bytes only if they fit
        assert d.retain_keys_device(koff2.data_ptr(), buf.data_ptr(), total) == total
        t.cuda.synchronize()
        assert not (buf.cpu().numpy() == 0xAB).all()
    finally:
        d.release()
    empty = Batch(R, [("t", "nothing/here")]).device(idx)
    try:
        koff = t.full((1,), -7, dtype=t.int64, device=R.dev)
        assert empty.n_ids == 0 and empty.retain_keys_device(koff.data_ptr(), None, 0) == 0
        t.cuda.synchronize()
        assert koff.cpu().tolist() == [0]
    finally:
        empty.release()


# ------------------------------------------------------------------ error contract
@pytest.mark.gpu
def test_device_errors(R):
    import ctypes as C
    N, lib = R.N, R.N.lib
    idx = R.retain.GpuTopicMatchIndex(0)
    History().add(idx, R, [("t", "a/b"), ("u", "a/c")])
    b = Batch(R, [("t", "a/+"), ("u", "#")])
    with pytest.raises(N.NativeError, match="bfq error -4"):   # before the first commit
        b.device(idx)
    idx.commit()
    good = b.device(idx)
    good.release()
    # a filter_tenant out of range, found on the device: the whole call fails and leaves the result empty
    t = R.torch
    tb, toff = N.as_blob(b.tenants)
    for bad in ([0, 2], [-1, 0], [1, 99]):
        d_ft = t.tensor(bad, dtype=t.int32, device=R.dev)
        out = N.BfqRDeviceResult()
        out.n_ids = 12345
        rc = lib.bfq_rmatch_device(idx._h, N.ptr(tb), N.ptr(toff), 2, b.d_blob.data_ptr(), b.d_off.data_ptr(), d_ft.data_ptr(), 2,
                                   None, 0, C.byref(out))
        assert rc == -5, bad
        assert not out.lease and out.n_ids == 0 and out.d_ids is None
    # NULL arrays
    args = [b.d_blob.data_ptr(), b.d_off.data_ptr(), b.d_ft.data_ptr()]
    for k in range(3):
        a = list(args)
        a[k] = None
        out = N.BfqRDeviceResult()
        assert lib.bfq_rmatch_device(idx._h, N.ptr(tb), N.ptr(toff), 2, *a, 2, None, 0, C.byref(out)) == -1
    out = N.BfqRDeviceResult()
    assert lib.bfq_rmatch_device(idx._h, None, None, 2, *args, 2, None, 0, C.byref(out)) == -1
    assert lib.bfq_rmatch_device(idx._h, N.ptr(tb), N.ptr(toff), 2, *args, 2, None, 0, None) == -1
    assert lib.bfq_rmatch_device(None, N.ptr(tb), N.ptr(toff), 2, *args, 2, None, 0, C.byref(out)) == -1
    n = C.c_int64(0)
    assert lib.bfq_rretain_keys_device(idx._h, C.byref(out), None, None, 0, None, C.byref(n)) == -1
    # the handle still matches afterwards, and an empty batch gives offsets [0]
    again = b.device(idx)
    try:
        assert fetch(R, again)[0] == b.host(idx).offsets.tolist()
    finally:
        again.release()
    e = Batch(R, [], tenants=["t"]).device(idx)
    try:
        assert e.n_filters == 0 and e.n_ids == 0 and fetch(R, e)[0] == [0]
    finally:
        e.release()
