"""Delivery budgets (bfq_expand_device_budget) against a literal restatement of DeliverExecutorGroup.submit.

submit (bifromq-dist-worker .../DeliverExecutorGroup.java:112-231) sends a message to each of its matched routes unless
MaxPersistentFanoutBytes or a tenant bandwidth throttle stops it, and reports PersistentFanoutBytesThrottled /
OutOfTenantResource and the MqttPersistentFanOutBytes meter. `submit` below restates that loop over the surviving routes
in ascending rank order, so "the first k persistent routes" are the lowest ranks, the order the library fixes. It runs
with the match's caps too and must then report no count event (the match already applied them).

Expectations come from the KV each test builds: oracle_lib decodes each route's kind, the oracle's match (KV.match_batch)
gives the surviving ranks per topic. Nothing is looked up through the library's own route lookup. CPU tests show that
every generator lands on the edge it is named after.
"""
import numpy as np
import pytest

import oracle_lib as O
import test_gpu_edges as E
import test_gpu_fanout as F

INT_MAX, I64_MAX, S_MAX = 2 ** 31 - 1, 2 ** 63 - 1, 2 ** 31 - 1
NORMAL, PERSISTENT, GROUP = 0, 1, 2
HAS_P, HAS_T = 1, 2                                    # tenant_bandwidth bits
BYTES, NO_P, NO_T, METERED = 1, 2, 4, 8                # topic flags
DROPS = BYTES | NO_P | NO_T
P_BW, T_BW = "TotalPersistentFanOutBytesPerSeconds", "TotalTransientFanOutBytesPerSeconds"


# ------------------------------------------------------------------ the reference (plain Python, no GPU)
def kinds_of(pairs):
    """route kind per rank of a sorted pair list, decoded by the oracle"""
    out = np.zeros(len(pairs), np.int8)
    for r, (k, v) in enumerate(pairs):
        m = O.build_match_route(k, v)
        out[r] = GROUP if m["type"] == "Group" else PERSISTENT if m["subBrokerId"] == 1 else NORMAL
    return out


def submit(kinds, ranks, s, max_bytes, bw, max_p=INT_MAX, max_g=INT_MAX):
    """DeliverExecutorGroup.submit over one message's routes, iterated in ascending rank order -> (sent ranks, events,
    meter value or None). Events: ("bytes", maxBytes), ("oor", reason), ("pcount", maxCount), ("gcount", maxCount)."""
    ranks = sorted(int(r) for r in ranks)
    if len(ranks) == 0:
        return [], [], None
    if len(ranks) == 1:
        return ranks, [], (s if kinds[ranks[0]] == PERSISTENT else None)
    has_t, has_p = bool(bw & HAS_T), bool(bw & HAS_P)
    p_thr = t_thr = g_thr = False
    p_count = p_bytes = g_count = 0
    sent, events = [], []
    for r in ranks:
        if kinds[r] == PERSISTENT:
            if p_count < max_p and p_bytes < max_bytes:
                if has_p:
                    p_count += 1
                    p_bytes += s
                    sent.append(r)
                elif not p_thr:
                    p_thr = True
                    events.append(("oor", P_BW))
            elif not p_thr:
                p_thr = True
                if p_count >= max_p:
                    events.append(("pcount", max_p))
                if p_bytes >= max_bytes:
                    events.append(("bytes", max_bytes))
        elif kinds[r] == NORMAL:
            if has_t:
                sent.append(r)
            elif not t_thr:
                t_thr = True
                events.append(("oor", T_BW))
        else:
            if g_count < max_g:
                g_count += 1
                sent.append(r)
            elif not g_thr:
                g_thr = True
                events.append(("gcount", max_g))
        if p_thr and t_thr and g_thr:
            break
    return sent, events, p_bytes


class Case:
    """one batch: sorted pairs, tenant entries (a tenant id may be listed twice with other budgets), topics, topic_tenant,
    per-position message sizes, per-entry MaxPersistentFanoutBytes and bandwidth bits, uniform match caps"""

    def __init__(self, pairs, tenants, topics, tt, sizes, max_bytes, bw, caps=(INT_MAX, INT_MAX)):
        self.pairs, self.tenants, self.topics = pairs, list(tenants), list(topics)
        self.tt = np.asarray(tt, np.int32)
        self.sizes = np.asarray(sizes, np.int64)
        self.max_bytes, self.bw, self.caps = list(max_bytes), list(bw), caps


class Expected:
    pass


def expect(case, kinds=None, kv=None):
    """the reference answer of a case: delivered CSR (ranks ascending per topic), flags, delivered persistent counts, events
    and meter per topic, the survivors of the match and the drop totals"""
    kinds = kinds_of(case.pairs) if kinds is None else kinds
    kv = E.kv_of(case.pairs) if kv is None else kv
    full = E.oracle_match(kv, case.tenants, case.topics, case.tt, INT_MAX, INT_MAX, O.MODE_TRIE)
    capped = E.oracle_match(kv, case.tenants, case.topics, case.tt, case.caps[0], case.caps[1], O.MODE_TRIE)
    n, nt = len(case.topics), len(case.tenants)
    x = Expected()
    x.route_count = np.diff(full.offsets)
    x.survivors = [capped.routes(i) for i in range(n)]
    x.flags, x.dp = np.zeros(n, np.uint8), np.zeros(n, np.int64)
    x.events, x.meter, sent_all = [], [], []
    x.drop = {"bytes": 0, "pbw": 0, "tbw": 0}
    for i in range(n):
        e = int(case.tt[i])
        known = 0 <= e < nt
        surv = x.survivors[i]
        sent, ev, meter = submit(kinds, surv, int(case.sizes[i]), case.max_bytes[e] if known else I64_MAX,
                                 case.bw[e] if known else HAS_P | HAS_T, case.caps[0], case.caps[1])
        assert not [v for v in ev if v[0] in ("pcount", "gcount")], ev     # the match's caps leave submit nothing to count
        sent_all.append(sent)
        f = 0
        for kind, arg in ev:
            f |= BYTES if kind == "bytes" else NO_P if arg == P_BW else NO_T
        if meter is not None:
            f |= METERED
            x.meter.append((i, meter))
        x.flags[i] = f
        x.dp[i] = sum(1 for r in sent if kinds[r] == PERSISTENT)
        sk = [int(kinds[r]) for r in surv]
        P, T = sk.count(PERSISTENT), sk.count(NORMAL)
        if f & BYTES:
            x.drop["bytes"] += P - int(x.dp[i])
        if f & NO_P:
            x.drop["pbw"] += P
        if f & NO_T:
            x.drop["tbw"] += T
        tid = case.tenants[e] if known else None
        for kind, arg in ev:
            x.events.append(("PersistentFanoutBytesThrottled", tid, case.topics[i], arg) if kind == "bytes"
                            else ("OutOfTenantResource", arg, tid, case.topics[i]))
    x.offsets = np.concatenate([[0], np.cumsum([len(s) for s in sent_all])]).astype(np.int64)
    x.ranks = np.array([r for s in sent_all for r in s], np.int64)
    x.sent = sent_all
    return x


# ------------------------------------------------------------------ generators
def entries_case(pairs, entries, topics, caps=(INT_MAX, INT_MAX)):
    """entries: [(tenant, max_bytes, bw, size)]: every topic once per entry, with the entry's size"""
    tenants = [e[0] for e in entries]
    tps, tt, sizes = [], [], []
    for j, e in enumerate(entries):
        for t in topics:
            tps.append(t)
            tt.append(j)
            sizes.append(e[3])
    return Case(pairs, tenants, tps, tt, sizes, [e[1] for e in entries], [e[2] for e in entries], caps)


FT_TOPICS = ["p/x", "t/x", "g/x", "m/x", "one/p", "one/t", "one/g", "none/x"]
FT_ENTRIES = {"bytes": ("ft", 10, HAS_P | HAS_T, 11), "no_p": ("ft", I64_MAX, HAS_T, 100),
              "no_t": ("ft", I64_MAX, HAS_P, 100), "none": ("ft", 1, 0, 100), "all": ("ft", I64_MAX, HAS_P | HAS_T, 100)}


def throttled_case(caps=(INT_MAX, INT_MAX)):
    """FanoutThrottledTest's scenarios as this project's inputs: 3 persistent, 3 transient, 3 group routes, all three mixed,
    and one route of each kind, under a bytes budget of 10 (messages of 11 bytes), no persistent / no transient bandwidth,
    neither (B = 1 < s) and no throttle"""
    r = [("ft", "p/x", "p", 3), ("ft", "t/x", "n", 3), ("ft", "g/x", "g", 3), ("ft", "m/x", "p", 3), ("ft", "m/x", "n", 3),
         ("ft", "m/x", "g", 3), ("ft", "one/p", "p", 1), ("ft", "one/t", "n", 1), ("ft", "one/g", "g", 1)]
    return entries_case(E.make_pairs(r), list(FT_ENTRIES.values()), FT_TOPICS, caps)


BIG_P = 12289
GRID_K = [1, 2, 127, 128, 129, 4095, 4096, 4097]
GRID_S = 1000


def grid_entries():
    """(tenant entry, expected k): B in {k*s - 1, k*s, k*s + 1}, s = 0, B = 1, and the largest B and s"""
    out = []
    for k in GRID_K:
        for d in (-1, 0, 1):
            out.append((("bp", k * GRID_S + d, HAS_P | HAS_T, GRID_S), k + (d > 0)))
    out += [(("bp", 1, HAS_P | HAS_T, 0), BIG_P), (("bp", 1, HAS_P | HAS_T, GRID_S), 1),
            (("bp", I64_MAX, HAS_P | HAS_T, S_MAX), BIG_P), (("bp", 3 * S_MAX, HAS_P | HAS_T, S_MAX), 3),
            (("bp", 3 * S_MAX + 1, HAS_P | HAS_T, S_MAX), 4), (("bp", I64_MAX, HAS_P | HAS_T, 1), BIG_P),
            (("bp", BIG_P, HAS_P | HAS_T, 1), BIG_P), (("bp", BIG_P - 1, HAS_P | HAS_T, 1), BIG_P - 1)]
    return out


def grid_case():
    """one topic with 12289 persistent routes (plus transient and group routes) under every bytes budget of grid_entries"""
    r = [("bp", "bp/#", "p", BIG_P), ("bp", "bp/+", "n", 5), ("bp", "bp/x", "g", 3)]
    return entries_case(E.make_pairs(r), [e for e, _ in grid_entries()], ["bp/x"])


LV = "abcdefg"
RANGE_TENANTS = {"r127": 127, "r128": 128, "r129": 129}


def range_routes():
    """per tenant a 7-level topic matching 127, 128 or 129 filters ('+'/literal combinations, 129 adds "a/#"): each filter
    holds 1-3 persistent routes between transient routes (subBrokerId 0 sorts before 1) and, every other filter, a group;
    and test_gpu_caps' multi-segment construction: the routes of "m" are two rank runs"""
    r = []
    for tenant, n in RANGE_TENANTS.items():
        filters = ["/".join("+" if mask >> i & 1 else LV[i] for i in range(7)) for mask in range(128)]
        filters = filters[128 - min(n, 128):] + (["a/#"] if n == 129 else [])
        for i, f in enumerate(filters):
            r += [(tenant, f, "p", 1 + i % 3), (tenant, f, "n", 1)]
            if i % 2:
                r.append((tenant, f, "g", 1))
    r += [("ms", "m", "p", 40), ("ms", "m", "n", 10), ("ms", "m", "g", 6), ("ms", "m//b", "p", 20), ("ms", "m/#", "p", 2)]
    return E.make_pairs(r)


RANGE_TOPIC = "/".join(LV)


def range_case(caps=(INT_MAX, INT_MAX)):
    """every tenant of range_routes under bytes budgets of k = 1 s, 2 s, 37 s, ... (s = 7): the k-th persistent survivor
    falls in later and later ranges"""
    entries, topics, tt, sizes = [], [], [], []
    for tenant in list(RANGE_TENANTS) + ["ms"]:
        topic = "m" if tenant == "ms" else RANGE_TOPIC
        for k in (1, 2, 37, 41, 100, 199, 255, 400):
            tt.append(len(entries))
            entries.append((tenant, k * 7, HAS_P | HAS_T, 7))
            topics.append(topic)
            sizes.append(7)
    return Case(range_routes(), [e[0] for e in entries], topics, tt, sizes, [e[1] for e in entries],
                [e[2] for e in entries], caps)


BATCH_TENANTS = [("ba", 5000, HAS_P | HAS_T), ("bb", I64_MAX, HAS_P), ("bc", 1, HAS_T), ("bd", 300, 0), ("ba", 700, HAS_P)]
BATCH_TOPICS = ["s/x", "s/y", "s/z", "q/z", "q/w", "none"]


def batch_case(n=40000, seed=5, caps=(INT_MAX, INT_MAX)):
    """> 32768 topics (de-dup and locality order run) of four tenants listed five times with different budgets, 5 % of them
    outside the tenant list, repeated topics with sizes from 0 to 3000 per position"""
    r = []
    for t in ("ba", "bb", "bc", "bd"):
        r += [(t, "s/+", "p", 5), (t, "s/#", "n", 3), (t, "s/x", "g", 2), (t, "s/y", "p", 1), (t, "q/z", "n", 1),
              (t, "q/w", "g", 1), (t, "s/#", "g", 1)]
    rng = np.random.default_rng(seed)
    nt = len(BATCH_TENANTS)
    tt = rng.integers(0, nt, n).astype(np.int32)
    tt[rng.random(n) < 0.05] = nt + 3
    topics = [BATCH_TOPICS[i] for i in rng.integers(0, len(BATCH_TOPICS), n)]
    sizes = rng.integers(0, 3001, n)
    return Case(E.make_pairs(r), [t for t, _, _ in BATCH_TENANTS], topics, tt, sizes, [b for _, b, _ in BATCH_TENANTS],
                [w for _, _, w in BATCH_TENANTS], caps)


def fan_case():
    """test_gpu_fanout's groups case (normal routes of subBrokerIds 0-2, $share groups, $oshare and an empty group) with
    the persistent bytes budget binding in one entry and transient bandwidth off in the other"""
    pairs, tenants, topics, tt = F.groups_case()
    return entries_case(pairs, [("g", 2 * 50, HAS_P, 50), ("g", I64_MAX, HAS_T, 50), ("g", 3, HAS_P | HAS_T, 1)], topics[:12])


def old_start():
    r = [("os", "o/+", "n", 4), ("os", "o/+", "p", 6), ("os", "o/+", "g", 2), ("os", "o/#", "p", 3)]
    return dict(E.make_pairs(r))


def old_delta():
    """remove a transient route of "o/+" and add 5 persistent routes that sort before its others"""
    dels = [O.route_key("os", "o/+", O.receiver_url(0, "r0", "d"))]
    adds = [(O.route_key("os", "o/+", O.receiver_url(1, "a%d" % j, "d")), O.incarnation_bytes(9)) for j in range(5)]
    return adds, dels


def old_case(pairs):
    return entries_case(pairs, [("os", 3 * 10, HAS_P, 10), ("os", 5 * 10, HAS_P | HAS_T, 10)], ["o/x", "o/y"])


# ------------------------------------------------------------------ CPU: the generators land on their edges
def test_reference_single_route_exemption_and_throttled_scenarios():
    c = throttled_case()
    x = expect(c)
    row = {(list(FT_ENTRIES)[int(c.tt[i])], c.topics[i]): i for i in range(len(c.topics))}
    n = lambda e, t: len(x.sent[row[e, t]])
    assert n("bytes", "p/x") == 1 and x.flags[row["bytes", "p/x"]] == BYTES | METERED
    assert n("no_p", "p/x") == 0 and x.flags[row["no_p", "p/x"]] == NO_P | METERED and x.route_count[row["no_p", "p/x"]] == 3
    assert n("no_t", "t/x") == 0 and x.flags[row["no_t", "t/x"]] == NO_T | METERED
    for e in FT_ENTRIES:
        assert n(e, "g/x") == 3 and x.flags[row[e, "g/x"]] == METERED
        for t in ("one/p", "one/t", "one/g"):
            assert n(e, t) == 1
    assert [m for i, m in x.meter if i == row["none", "one/p"]] == [100]
    assert not x.flags[row["none", "one/t"]] and not x.flags[row["none", "one/g"]]
    assert x.flags[row["none", "m/x"]] == NO_P | NO_T | METERED and n("none", "m/x") == 3


def test_grid_case_hits_every_k():
    c = grid_case()
    x = expect(c)
    assert x.route_count[0] == BIG_P + 5 + 3
    for i, (e, k) in enumerate(grid_entries()):
        assert x.dp[i] == min(k, BIG_P)
        assert bool(x.flags[i] & BYTES) == (k < BIG_P)
        if e[3] > 0 and k < BIG_P:
            assert (x.dp[i] - 1) * e[3] < e[1] <= x.dp[i] * e[3]   # the last send saw sent * s < B, the next would not
    assert x.dp[len(GRID_K) * 3] == BIG_P                       # s = 0 with B = 1


@pytest.mark.parametrize("caps", [(INT_MAX, INT_MAX), (40, 7), (300, 2)])
def test_range_case_cuts_in_later_ranges(caps):
    c = range_case(caps)
    x = expect(c)
    kinds = kinds_of(c.pairs)
    full = E.oracle_match(E.kv_of(c.pairs), c.tenants, c.topics, c.tt, INT_MAX, INT_MAX, O.MODE_TRIE)
    kv = E.kv_of(c.pairs)
    n_filters = {len(E.matched_filters(kv, full, i)) for i in range(len(c.topics)) if c.topics[i] == RANGE_TOPIC}
    assert n_filters == {127, 128, 129}
    target = lambda r: O.build_match_route(*c.pairs[r])["mqttTopicFilter"].split("$share/", 1)[-1].split("/", 1)[-1] \
        if kinds[r] == GROUP else O.build_match_route(*c.pairs[r])["mqttTopicFilter"]
    later = 0
    for i in range(len(c.topics)):
        if x.flags[i] & BYTES and c.topics[i] == RANGE_TOPIC:
            last = max(r for r in x.sent[i] if kinds[r] == PERSISTENT)
            # the last persistent route sent lies in the 15th or a later range of the topic, behind transient / group ranks
            if len({target(r) for r in x.survivors[i].tolist() if r <= last}) >= 15:
                later += 1
                assert any(kinds[r] != PERSISTENT for r in x.survivors[i].tolist() if r < last)
    assert later >= 3
    if caps[0] == 40:                                           # both sides of min(maxP, k)
        assert {k for k in x.dp.tolist()} >= {1, 2, 37, 40}
    # the multi-segment filter: "m"'s ranks are several runs and a cut lands behind the first one
    m_rows = [i for i, t in enumerate(c.topics) if t == "m"]
    own = [r for r in full.routes(m_rows[0]).tolist() if O.build_match_route(*c.pairs[r])["mqttTopicFilter"] == "m"]
    runs = np.split(np.array(own), np.where(np.diff(own) != 1)[0] + 1)
    assert len(runs) >= 2
    first_p = sum(1 for r in runs[0] if kinds[r] == PERSISTENT)
    p_m = sum(1 for r in x.survivors[m_rows[0]].tolist() if kinds[r] == PERSISTENT)
    assert any(first_p < k < p_m for k in x.dp[m_rows].tolist())


def test_batch_case_shape():
    c = batch_case()
    x = expect(c)
    assert len(c.topics) > 32768 and (c.tt >= len(c.tenants)).sum() > 1000
    assert len({(b, w) for _, b, w in BATCH_TENANTS}) == len(BATCH_TENANTS) >= 3
    assert len({(int(c.tt[i]), c.topics[i], int(c.sizes[i])) for i in range(len(c.topics))}) > 1000
    for bit in (BYTES, NO_P, NO_T, METERED):
        assert (x.flags & bit).any()
    assert (x.flags[c.tt >= len(c.tenants)] == 0).all()


def test_old_delta_changes_kinds_of_the_matched_filter():
    kv = old_start()
    a = expect(old_case(sorted(kv.items())))
    adds, dels = old_delta()
    for k in dels:
        del kv[k]
    kv.update(adds)
    b = expect(old_case(sorted(kv.items())))
    assert a.ranks.tolist() != b.ranks.tolist() and a.route_count.tolist() != b.route_count.tolist()


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def B():
    import torch

    import bifromq_b200
    from bifromq_b200 import dist
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.pkg, ns.torch, ns.dist = bifromq_b200, torch, dist
    ns.dev = torch.device("cuda", 0)
    ns.stream = torch.cuda.current_stream(ns.dev).cuda_stream
    return ns


def match(B, idx, case, wait=True):
    torch = B.torch
    blob, off = O.blob(case.topics)
    keep = [torch.from_numpy(blob).to(B.dev), torch.from_numpy(off).to(B.dev), torch.from_numpy(case.tt).to(B.dev)]
    nt = len(case.tenants)
    out = idx.match_device(case.tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), len(case.topics),
                           [case.caps[0]] * nt, [case.caps[1]] * nt, B.stream, wait)
    out.keep = keep
    return out


def budget(B, out, case):
    """sizing call + writing call -> dict of host copies, the device CSR and the result struct"""
    torch, n = B.torch, len(case.topics)
    d_msg = torch.from_numpy(case.sizes.astype(np.int32)).to(B.dev)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device=B.dev)
    r0 = out.expand_budget(d_msg.data_ptr(), case.max_bytes, case.bw, d_off.data_ptr(), None, 0, B.stream)
    total = r0.n_delivered
    d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=B.dev)
    r = out.expand_budget(d_msg.data_ptr(), case.max_bytes, case.bw, d_off.data_ptr(), d_ranks.data_ptr(), total, B.stream)
    torch.cuda.synchronize()
    view = lambda p, k, t: B.dist.device_view(p, k, t, B.dev).cpu().numpy()
    return {"r": r, "total": total, "d_off": d_off, "d_ranks": d_ranks, "offsets": d_off.cpu().numpy(),
            "ranks": d_ranks.cpu().numpy()[:total], "flags": view(r.d_topic_flags, n, "|u1"),
            "dp": view(r.d_delivered_persistent, n, "<u4").astype(np.int64)}


def compare(B, got, x, case):
    from bifromq_b200 import budget_events
    assert got["offsets"].tolist() == x.offsets.tolist()
    assert got["r"].n_delivered == got["total"] == int(x.offsets[-1])
    n = len(case.topics)
    topic = np.repeat(np.arange(n, dtype=np.int64), np.diff(got["offsets"]))
    assert np.array_equal(np.sort(F.pair_keys(topic, got["ranks"])), np.sort(F.pair_keys(topic, x.ranks)))
    assert got["flags"].tolist() == x.flags.tolist()
    assert got["dp"].tolist() == x.dp.tolist()
    r = got["r"]
    assert (r.n_dropped_bytes, r.n_dropped_persistent_bandwidth, r.n_dropped_transient_bandwidth) == \
        (x.drop["bytes"], x.drop["pbw"], x.drop["tbw"])
    events, meter = budget_events(case.tenants, case.topics, case.tt, got["flags"], got["dp"], case.sizes, case.max_bytes)
    assert sorted((type(e).__name__,) + tuple(e) for e in events) == sorted(x.events)
    assert meter == x.meter


def run(B, case, idx=None, fan_path=None):
    own = idx is None
    if own:
        idx = F.make_index(B, case.pairs)
    x = expect(case)
    out = match(B, idx, case)
    rc_before = B.dist.device_view(out.d_route_count, len(case.topics), "<u4", B.dev).cpu().numpy().copy()
    thr_before = out.n_throttled
    got = budget(B, out, case)
    compare(B, got, x, case)
    rc = B.dist.device_view(out.d_route_count, len(case.topics), "<u4", B.dev).cpu().numpy()
    assert rc.tolist() == rc_before.tolist() == x.route_count.tolist() and out.n_throttled == thr_before
    if fan_path is not None:
        idx.set_option("fanout_global", 1 if fan_path == "global" else 0)
        fo = F.fanout_once(B, out, got["d_off"], got["d_ranks"], got["total"])
        want = Expected()
        want.offsets, want.ranks = x.offsets, x.ranks
        s = F.check(idx, fo, got["offsets"], got["ranks"], want, case.pairs)
        got["fan"] = s
    out.release()
    if own:
        idx.close()
    return got, x


# ------------------------------------------------------------------ GPU: semantics
@pytest.mark.gpu
@pytest.mark.parametrize("caps", [(INT_MAX, INT_MAX), (2, 1)])
def test_throttled_scenarios_and_single_route_exemption(B, caps):
    got, x = run(B, throttled_case(caps))
    c = throttled_case(caps)
    row = {(list(FT_ENTRIES)[int(c.tt[i])], c.topics[i]): i for i in range(len(c.topics))}
    sizes = np.diff(got["offsets"])
    if caps[0] == INT_MAX:
        assert sizes[row["bytes", "p/x"]] == 1 and got["flags"][row["bytes", "p/x"]] & BYTES
        assert sizes[row["no_p", "p/x"]] == 0 and got["flags"][row["no_p", "p/x"]] & NO_P
        assert x.route_count[row["no_p", "p/x"]] == 3
    assert sizes[row["no_t", "t/x"]] == 0 and got["flags"][row["no_t", "t/x"]] & NO_T
    for t in ("one/p", "one/t", "one/g"):
        assert sizes[row["none", t]] == 1


@pytest.mark.gpu
def test_bytes_arithmetic_grid(B):
    got, x = run(B, grid_case())
    assert got["dp"].tolist() == [min(k, BIG_P) for _, k in grid_entries()]


@pytest.mark.gpu
@pytest.mark.parametrize("caps", [(INT_MAX, INT_MAX), (40, 7), (300, 2)])
def test_kv_order_across_ranges_and_segments(B, caps):
    idx = F.make_index(B, range_case(caps).pairs)
    st = idx.stats()
    got, x = run(B, range_case(caps), idx)
    assert idx.stats()["multi_segment_filters"] >= 1
    if caps[0] != INT_MAX:
        assert idx.stats()["flagged_topics"] > st["flagged_topics"]
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("caps", [(INT_MAX, INT_MAX), (3, 1)])
def test_many_tenants_in_locality_order(B, caps):
    c = batch_case(caps=caps)
    idx = F.make_index(B, c.pairs)
    st = idx.stats()
    run(B, c, idx)
    assert idx.stats()["duplicate_topics"] - st["duplicate_topics"] > 30000
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", F.PATHS)
def test_budgeted_csr_feeds_the_fanout(B, path):
    got, x = run(B, fan_case(), fan_path=path)
    assert got["fan"]["parked"] > 0 and got["fan"]["normal"] > 0 and got["fan"]["share"] > 0
    assert got["r"].n_dropped_bytes > 0 and got["r"].n_dropped_transient_bandwidth > 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["groups", "tier2", "hot"])
def test_budgets_that_never_bind_equal_the_expand(B, name):
    pairs, tenants, topics, tt = {"groups": F.groups_case, "tier2": F.tier2_case, "hot": F.hot_case}[name]()
    caps = (3, 1) if name != "hot" else (INT_MAX, INT_MAX)
    idx = F.make_index(B, pairs)
    c = Case(pairs, tenants, topics, tt, np.full(len(topics), S_MAX), [I64_MAX] * len(tenants), [3] * len(tenants), caps)
    out = match(B, idx, c)
    d_off, d_ranks, total = F.device_csr(B, out, len(topics))
    got = budget(B, out, c)
    assert got["offsets"].tolist() == d_off.cpu().numpy().tolist()
    topic = np.repeat(np.arange(len(topics), dtype=np.int64), np.diff(got["offsets"]))
    assert np.array_equal(np.sort(F.pair_keys(topic, got["ranks"])), np.sort(F.pair_keys(topic, d_ranks.cpu().numpy()[:total])))
    assert not (got["flags"] & DROPS).any()
    compare(B, got, expect(c), c)
    out.release()
    idx.close()


@pytest.mark.gpu
def test_old_result_budgets_against_its_own_snapshot(B):
    kv = old_start()
    old_pairs = sorted(kv.items())
    idx = F.make_index(B, old_pairs)
    c_old = old_case(old_pairs)
    out_old = match(B, idx, c_old)
    adds, dels = old_delta()
    for k in dels:
        del kv[k]
    kv.update(adds)
    idx.apply(adds=adds, dels=dels)
    st = idx.stats()
    idx.commit()
    assert idx.stats()["delta_commits"] == st["delta_commits"] + 1
    compare(B, budget(B, out_old, c_old), expect(c_old), c_old)
    out_old.release()
    c_new = old_case(sorted(kv.items()))
    run(B, c_new, idx)
    idx.close()


# ------------------------------------------------------------------ GPU: errors
@pytest.mark.gpu
def test_budget_argument_and_state_errors(B):
    from bifromq_b200._native import NativeError
    c = throttled_case()
    idx = F.make_index(B, c.pairs)
    torch, n = B.torch, len(c.topics)
    d_off = torch.zeros(n + 1, dtype=torch.int64, device=B.dev)
    d_msg = torch.from_numpy(c.sizes.astype(np.int32)).to(B.dev)
    out = match(B, idx, c, wait=False)
    with pytest.raises(NativeError) as e:
        out.expand_budget(d_msg.data_ptr(), c.max_bytes, c.bw, d_off.data_ptr(), None, 0, B.stream)
    assert F.bfq_code(e.value) == -4                                     # BFQ_E_STATE: not waited yet
    out.wait()
    bad = [(0, c.max_bytes, c.bw), (d_msg.data_ptr(), [], c.bw), (d_msg.data_ptr(), c.max_bytes, []),
           (d_msg.data_ptr(), [0] + c.max_bytes[1:], c.bw), (d_msg.data_ptr(), c.max_bytes[:-1] + [-5], c.bw)]
    for msg, mb, bw in bad:
        with pytest.raises(NativeError) as e:
            out.expand_budget(msg or None, mb, bw, d_off.data_ptr(), None, 0, B.stream)
        assert F.bfq_code(e.value) == -1                                 # BFQ_E_INVALID
    neg = c.sizes.astype(np.int32).copy()
    neg[len(neg) // 2] = -1
    d_neg = torch.from_numpy(neg).to(B.dev)
    d_ranks = torch.zeros(1000, dtype=torch.int64, device=B.dev)
    with pytest.raises(NativeError) as e:
        out.expand_budget(d_neg.data_ptr(), c.max_bytes, c.bw, d_off.data_ptr(), d_ranks.data_ptr(), 1000, B.stream)
    assert F.bfq_code(e.value) == -1 and "negative" in str(e.value)
    compare(B, budget(B, out, c), expect(c), c)                          # the result is still usable
    out.release()
    idx.close()
