"""The forward match at the edges of its bounded tiers, its buffer-growth re-runs and its de-duplication.

The forward path is exact by construction: work that does not fit tier 0's bounded per-lane state is handed, whole, to
tier 1 (warp per topic), and what does not fit tier 1's shared buffers to tier 2 (global scratch); buffers that turn out
too small are grown and the batch is re-run; repeated (tenant, topic) pairs are matched once. Each hand-off is its own code
path, and a slip in one sends a message to the wrong subscribers without any error. Every test here builds its case from
plain routes and topics, checks the whole answer against the CPU oracle (offsets, ranks, throttle events, pre-cap route
counts) and asserts, through idx.stats(), that the path it targets was taken. Where the shape of the input is the point
("this topic matches exactly 64 filters", "this level starts at every offset mod 16") a CPU test checks it on the oracle
side, so a generator cannot drift off its edge unnoticed.

Limits exercised (bifromq_b200/csrc/match_kernels.cu{,h}): tier 0 = 12 levels (L_MAXLV), 24-byte levels (TOKEN_BYTES),
12 inline ranges then one 64-range spill block (INLINE_RANGES / SPILL_RANGES), topics of <= 65535 bytes; tier 1 = 64
frontier nodes, 48 ranges (FR_CAP / RG_CAP).
"""
import itertools
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O

INT_MAX = 2 ** 31 - 1
L_MAXLV, TOKEN_BYTES, INLINE_RANGES, SPILL_RANGES, RG_CAP = 12, 24, 12, 64, 48
# initial buffer sizes of a fresh workspace (capi.cu: prepare_workspace): the cursor-allocated range region holds
# max(2^20, n) ranges, cut into one slice per sub-batch on the host path; the throttle list max(2^16, sub_batches * 2^14)
# events. Batches of >= 2^17 topics take the host path's 4-sub-batch pipeline.
SPILL_REGION, THROTTLE_LIST, PIPELINE_TOPICS, SUB_BATCHES = 1 << 20, 1 << 16, 1 << 17, 4
CAPS = [(INT_MAX, INT_MAX), (5, 2)]
NO_TENANT = "\x7fno such tenant"


# ------------------------------------------------------------------ case building (plain Python data, no GPU)
def make_pairs(routes):
    """routes: iterable of (tenant, filter, kind, n) with kind 'p' persistent (subBrokerId 1), 'n' normal (subBrokerId 0),
    'g' shared group; n routes of the filter (receivers r0..). -> sorted, de-duplicated (key, value) pairs"""
    out = {}
    for tenant, f, kind, n in routes:
        for j in range(n):
            if kind == "g":
                members = {O.receiver_url(0, "m%d" % j, "d"): 1}
                out[O.route_key(tenant, "$share/g%d/%s" % (j, f))] = O.route_group(members)
            else:
                url = O.receiver_url(1 if kind == "p" else 0, "r%d" % j, "d")
                out[O.route_key(tenant, f, url)] = O.incarnation_bytes(j + 1)
    return sorted(out.items())


def one_route_each(tenant, filters):
    """every filter exactly one route (so a topic's route count is its number of matched filters); the kinds cycle through
    persistent / group / normal, so both caps counters move across the inline -> spill move"""
    return [(tenant, f, "pgn"[i % 3], 1) for i, f in enumerate(filters)]


def kv_of(pairs):
    kv = O.KV()
    for k, v in pairs:
        kv.put(k, v)
    kv.freeze()
    return kv


def oracle_match(kv, tenants, topics, tt, max_p, max_g, mode=O.MODE_BRUTE):
    """the oracle's answer; a topic whose tenant index is outside [0, n_tenants) matches nothing (as on the GPU)"""
    tt = np.asarray(tt, np.int64)
    bad = (tt < 0) | (tt >= len(tenants))
    tt_o = np.where(bad, len(tenants), tt).astype(np.int32)
    return kv.match_batch(list(tenants) + [NO_TENANT], topics, tt_o, max_p, max_g, mode, False, 8)


def matched_filters(kv, res, i):
    """the topic filters topic i of an oracle result matched (a group route's "$share/<group>/" prefix removed)"""
    out = set()
    for r in res.routes(i):
        f = O.build_match_route(kv.key(int(r)), kv.value(int(r)))["mqttTopicFilter"]
        out.add(f.split("/", 2)[2] if f.startswith("$share/") else f)
    return out


def route_counts(kv, tenants, topics, tt, mode=O.MODE_BRUTE):
    return np.diff(oracle_match(kv, tenants, topics, tt, INT_MAX, INT_MAX, mode).offsets)


def true_repeats(tenants, topics, tt):
    """repeats of a (tenant, topic bytes) pair; every out-of-range tenant index is one group (as in the de-dup pass)"""
    nt = len(tenants)
    keys = {((t if 0 <= t < nt else -1), O._b(s)) for s, t in zip(topics, np.asarray(tt).tolist())}
    return len(topics) - len(keys)


def levels_case():
    """topics of 11, 12, 13 and 16 levels (16 = the reference's default MaxTopicLevels) against exact filters, '+' at the
    first / last / every level, prefix/# at every depth (incl. the parent-level match of a 12-level topic) and a '+' branch
    parked at level 11, the deepest slot tier 0 has, that the DFS must pop after the exact branch ends. Tenant "lv0" keeps
    every topic at <= 12 matched filters (inline slots only), tenant "lv" spills."""
    L = ["L%d" % i for i in range(16)]
    j = "/".join
    routes = []
    full = set()
    for n in (11, 12, 13, 16):
        full.add(j(L[:n]))
        for i in range(n):
            full.add(j(L[:i] + ["+"] + L[i + 1:n]))
    for k in range(17):
        full.add(j(L[:k] + ["#"]))
    full |= {j(L[:10] + ["+", "L11"]), j(L[:10] + ["+", "+"])}
    routes += one_route_each("lv", sorted(full))
    small = [j(L[:11]), j(L[:12]), j(L[:11] + ["+"]), j(["+"] + L[1:12]), j(L[:11] + ["#"]), j(L[:12] + ["#"]),
             j(L[:10] + ["+", "L11"]), j(L[:10] + ["+", "+"]), j(L[:13])]
    routes += one_route_each("lv0", small)
    topics, tt = [], []
    for n in (11, 12, 13, 16):
        for t in (j(L[:n]), j(L[:n - 1] + ["X"]), j(["Y"] + L[1:n]), j(L[:10] + ["Z"] + L[11:n])):
            topics.append(t)
            tt.append(0)
    for n in (11, 12, 13):
        for t in (j(L[:n]), j(L[:n - 1] + ["X"]), j(L[:10] + ["Z"] + L[11:n])):
            topics.append(t)
            tt.append(1)
    deep = sum(1 for t in topics if t.count("/") + 1 > L_MAXLV)   # each reaches level 11 with a level to go: tier 1
    return make_pairs(routes), ["lv", "lv0"], topics, np.array(tt, np.int32), deep


LEVEL_LENGTHS = [0, 1, 23, 24, 25, 27, 28, 29]


def level_strings():
    out = ["".join(chr(ord("a") + (7 * n + i) % 26) for i in range(n)) for n in LEVEL_LENGTHS]
    out += ["你好" * 4, "é" * 12, "x" + "你好" * 4, "你好" * 4 + "q"]   # multi-byte UTF-8 ending at byte 24 (and 25)
    return out


def alignment_case(a):
    """level lengths 0..29 (and UTF-8 levels ending at byte 24) at level-start offset a (mod 16) in the blob, as the last,
    a middle and the first level and as the whole topic. Every test topic is followed by a filler topic of 'c' bytes that
    continue a stored token ("ab/<s>c" is stored: "ab/<s>" must not match it), and the blob ends with a test topic.
    -> pairs, topics, level starts {byte length: [blob offset of the level]}"""
    S = level_strings()
    filters = {"ab/+", "+/z", "ab/#", "+"}
    for s in S:
        filters |= {"ab/" + s, "ab/" + s + "c", "ab/" + s + "cc", "ab/" + s + "/z", s + "/z", s + "c/z", "+/" + s}
        if s:
            filters |= {s, s + "c", "ab/" + s[:-1]}
    topics, starts, cur = [], {}, 0
    items = [(s, kind) for kind in ("last", "mid", "first", "only") for s in S]
    items.sort(key=lambda x: (x[0] == S[a % len(S)] and x[1] == "last"))   # the blob ends with a test level
    for s, kind in items:
        t = {"last": "ab/" + s, "mid": "ab/" + s + "/z", "first": s + "/z", "only": s}[kind]
        d = 3 if kind in ("last", "mid") else 0
        fill = (a - d - cur) % 16 or 16
        topics.append("c" * fill)
        cur += fill
        starts.setdefault(len(s.encode()), []).append(cur + d)
        topics.append(t)
        cur += len(t.encode())
    return make_pairs(one_route_each("al", sorted(filters))), topics, starts


RANGE_COUNTS = [11, 12, 13, 48, 49, 63, 64, 65]


def ranges_case():
    """one topic per count N that matches exactly N distinct filters, each one route: 7 levels (tier 0: inline, spill,
    > 64 -> tier 1 -> > 48 -> tier 2) and 14 levels (tier 0 defers it for its depth: tier 1's 48 / 49 directly)"""
    routes, topics = [], []
    for deep in (False, True):
        rest = list("abcdefghijklm") if deep else list("abcdef")
        for n in RANGE_COUNTS:
            head = ("d%d" if deep else "r%d") % n
            lv = [head] + rest
            cands = []
            for combo in itertools.product([False, True], repeat=6):
                cands.append("/".join([head] + ["+" if c else x for c, x in zip(combo, rest[:6])] + rest[6:]))
            cands += ["/".join(lv[:k] + ["#"]) for k in range(1, len(lv) + 1)]
            random.Random(n * 7 + deep).shuffle(cands)
            routes += one_route_each("rg", cands[:n])
            topics.append("/".join(lv))
    return make_pairs(routes), ["rg"], topics, np.zeros(len(topics), np.int32)


def random_edge_case(seed, n_topics=40):
    """levels 10-14, level lengths 22-24 or 22-26, 10-14 or 46-66 matched filters per topic (filters derived from the topic: '+' and
    '#' masks), random blob alignment through filler topics"""
    rng = random.Random(seed)
    alpha = "abcdefghij"
    routes, topics, want_n, deferred = [], [], [], 0
    for i in range(n_topics):
        depth = rng.randint(10, 14)
        hi = rng.choice([TOKEN_BYTES, TOKEN_BYTES + 2])   # half the topics keep every level within tier 0's 24 bytes
        lv = ["t%03d" % i + "".join(rng.choice(alpha) for _ in range(rng.randint(18, hi - 4)))]
        lv += ["".join(rng.choice(alpha) for _ in range(rng.randint(22, hi))) for _ in range(depth - 1)]
        n = rng.choice([rng.randint(10, 14), rng.randint(46, 66)])
        fs = {"/".join([lv[0]] + ["+" if k == 1 else x for k, x in enumerate(lv) if k > 0])}   # the walk reaches every level
        while len(fs) < n:
            if rng.random() < 0.15:
                fs.add("/".join(lv[:rng.randint(1, depth)] + ["#"]))
            else:
                fs.add("/".join([lv[0]] + [("+" if rng.random() < 0.3 else x) for x in lv[1:]]))
        routes += one_route_each("rnd", sorted(fs))
        topics.append("c" * rng.randint(0, 15))   # filler: shifts the alignment of what follows
        topics.append("/".join(lv))
        want_n.append(n)
        deferred += depth > L_MAXLV or n > SPILL_RANGES or any(len(x) > TOKEN_BYTES for x in lv)
    return make_pairs(routes), ["rnd"], topics, np.zeros(len(topics), np.int32), want_n, deferred


def spill_filters(tenant, kind="pgn"):
    """a topic "k<i>/a/b/c/d" matches 16 + 2 filters: 18 ranges, a spill block each"""
    fs = ["/".join(["+"] + [("+" if c else x) for c, x in zip(combo, "abcd")]) for combo in itertools.product([0, 1], repeat=4)]
    fs += ["+/#", "#"]
    return [(tenant, f, kind[i % len(kind)], 1) for i, f in enumerate(fs)]


TIER2_FILTERS = ["/".join(c) for c in itertools.product(["a", "+"], repeat=8)] + ["/".join(["a"] * n) + "/#" for n in range(1, 8)]
TIER2_TOPIC = "/".join(["a"] * 8)          # 263 ranges, frontier up to 128: tier 0 -> tier 1 -> tier 2
TIER1_TOPIC = "/".join(["b"] * 14)         # 14 levels, few ranges: tier 0 -> tier 1


def tier2_case(n_other=300, reps2=40, reps1=25, seed=3):
    routes = one_route_each("t", TIER2_FILTERS)
    routes += one_route_each("t", ["b/#", TIER1_TOPIC, "/".join(["b"] * 13 + ["+"]), "b/+", "c/+", "c/d"])
    rng = random.Random(seed)
    topics = [TIER2_TOPIC] * reps2 + [TIER1_TOPIC] * reps1
    topics += [rng.choice(["a/a", "a/b", "c/d", "c/e", "a/a/a", "b/b"]) + "/%d" % rng.randint(0, 40) for _ in range(n_other)]
    topics += ["a/a", "c/d", "b/b"]
    rng.shuffle(topics)
    return routes, ["t"], topics


def dedup_collision_case(seed=17, n_random=3000):
    """adversarial groups for the de-dup compare: same length and tenant, equal in the first 48 bytes (the order-key window)
    and different in one byte at 48, 49, 63, 64 or the last; different only inside the window; lengths 47/48/49 and 63/64/65;
    the same bytes under two tenants; out-of-range tenant indices; "", "/", "//". Each distinct pair appears 1-4 times, in
    shuffled order (so at varied blob alignments), among n_random ordinary distinct topics."""
    rng = random.Random(seed)
    tenants = ["tA", "tB", "tC"]
    base = []
    for n in (47, 48, 49, 63, 64, 65, 80, 100, 200):
        root = "g%03d/" % n + "".join(rng.choice("abcdefgh/") for _ in range(n - 5))
        assert len(root) == n
        base.append(root)
        for p in (0, 5, 46, 47, 48, 49, 63, 64, n - 1):
            if p < n:
                s = list(root)
                s[p] = "Z" if s[p] != "Z" else "Y"
                base.append("".join(s))
    base += ["", "/", "//"]
    entries = []
    for s in base:
        for t in (0, 1, -1, 3, 7):   # two real tenants, and out-of-range indices (one group between them)
            entries.append((s, t))
    for i in range(n_random):
        entries.append(("r/%05d/" % i + "x" * rng.randint(0, 60), rng.randrange(3)))
    batch = []
    for e in entries:
        batch += [e] * rng.choice([1, 1, 2, 4])
    rng.shuffle(batch)
    topics = [s for s, _ in batch]
    tt = np.array([t for _, t in batch], np.int32)
    # exact filters for half the distinct strings (so a wrong merge changes an answer), '#' for tenant tB only
    fs = sorted({s for s, _ in entries if s and rng.random() < 0.5})
    routes = one_route_each("tA", fs) + one_route_each("tC", fs[::3]) + [("tB", "#", "p", 1), ("tB", "+/+", "g", 1)]
    return make_pairs(routes), tenants, topics, tt


# ------------------------------------------------------------------ CPU checks of the generators (oracle side only)
def test_levels_case_shape():
    pairs, tenants, topics, tt, deep = levels_case()
    depth = [t.count("/") + 1 for t in topics]
    assert {11, 12, 13, 16} <= set(depth) and deep > 0
    kv = kv_of(pairs)
    n = route_counts(kv, tenants, topics, tt)
    small = n[tt == 1]
    assert small.max() <= INLINE_RANGES and n[tt == 0].max() > INLINE_RANGES
    L = ["L%d" % i for i in range(16)]
    # a 12-level topic matches its parent-level '#' filter and the '+' branch parked at level 11
    one = oracle_match(kv, ["lv"], ["/".join(L[:12])], [0], INT_MAX, INT_MAX)
    got = matched_filters(kv, one, 0)
    assert {"/".join(L[:12] + ["#"]), "/".join(L[:10] + ["+", "L11"]), "/".join(L[:10] + ["+", "+"])} <= got


@pytest.mark.parametrize("a", [0, 7, 15])
def test_alignment_case_shape(a):
    pairs, topics, starts = alignment_case(a)
    blob = b"".join(O._b(t) for t in topics)
    for n in LEVEL_LENGTHS + [24, 25]:
        assert n in starts and all(s % 16 == a for s in starts[n]), n
    assert blob.endswith(O._b("ab/" + level_strings()[a % len(level_strings())]))
    assert {len(s.encode()) for s in level_strings()} >= set(LEVEL_LENGTHS)
    assert "你好".encode() * 4 == ("你好" * 4).encode() and len(("你好" * 4).encode()) == 24
    # the stored continuation "ab/<s>c" is not matched by "ab/<s>" followed by a 'c' filler
    kv = kv_of(pairs)
    s1 = level_strings()[LEVEL_LENGTHS.index(1)]
    i = topics.index("ab/" + s1)
    assert topics[i + 1].startswith("c")
    res = oracle_match(kv, ["al"], ["ab/" + s1, "ab/" + s1 + "c"], [0, 0], INT_MAX, INT_MAX)
    f0, f1 = matched_filters(kv, res, 0), matched_filters(kv, res, 1)
    assert "ab/" + s1 + "c" not in f0 and "ab/" + s1 in f0 and "ab/" + s1 + "c" in f1


def test_alignment_covers_every_offset():
    for n in LEVEL_LENGTHS:
        assert {a for a in range(16) if n in alignment_case(a)[2]} == set(range(16))


def test_ranges_case_shape():
    pairs, tenants, topics, tt = ranges_case()
    n = route_counts(kv_of(pairs), tenants, topics, tt)
    assert n.tolist() == RANGE_COUNTS + RANGE_COUNTS   # every filter one route: route count == matched filters
    assert [t.count("/") + 1 for t in topics] == [7] * 8 + [14] * 8


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_edge_case_shape(seed):
    pairs, tenants, topics, tt, want_n, deferred = random_edge_case(seed)
    assert 0 < deferred < len(want_n)
    n = route_counts(kv_of(pairs), tenants, topics, tt)
    assert n[1::2].tolist() == want_n
    blob_off = np.cumsum([0] + [len(O._b(t)) for t in topics])
    assert len({int(o) % 16 for o in blob_off[1::2]}) >= 8


def test_spill_and_tier2_case_shape():
    kv = kv_of(make_pairs(spill_filters("t")))
    assert route_counts(kv, ["t"], ["k1/a/b/c/d", "k2/a/b/c/x"], [0, 0]).tolist() == [18, 10]
    routes, tenants, topics = tier2_case()
    kv = kv_of(make_pairs(routes))
    n = route_counts(kv, tenants, [TIER2_TOPIC, TIER1_TOPIC], [0, 0])
    assert n[0] == 256 + 7 and 0 < n[1] <= RG_CAP
    assert topics.count(TIER2_TOPIC) > 10 and topics.count(TIER1_TOPIC) > 10


def test_dedup_case_shape():
    pairs, tenants, topics, tt = dedup_collision_case()
    rep = true_repeats(tenants, topics, tt)
    assert 0 < rep < len(topics)
    lens = {len(O._b(t)) for t in topics}
    assert {0, 1, 2, 47, 48, 49, 63, 64, 65} <= lens
    # same bytes under two real tenants are not repeats, two out-of-range indices are
    assert true_repeats(tenants, ["a", "a"], [0, 1]) == 0 and true_repeats(tenants, ["a", "a"], [-1, 9]) == 1


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def B():
    import bifromq_b200
    bifromq_b200.load_library()
    return bifromq_b200


def make_index(B, pairs):
    idx = B.GpuRouteIndex(0)
    idx.load_pairs(pairs)
    idx.commit()
    return idx


def delta(idx, before):
    after = idx.stats()
    return {k: after[k] - before[k] for k in ("deferred_topics", "overflow_topics", "duplicate_topics", "buffer_retries",
                                              "flagged_topics")}


def events_of(want):
    return sorted((k, t, r) for k, t, r, _ in want.events)


def check_host(idx, kv, tenants, topics, tt, caps, mode=O.MODE_BRUTE):
    """bfq_match vs the oracle, exactly: offsets, ranks, throttle events (kind, topic, rank), pre-cap route counts.
    -> (stats delta, result) — the caller closes the result"""
    before = idx.stats()
    nt = len(tenants)
    tt = np.ascontiguousarray(tt, np.int32)
    res = idx.match_topics(tenants, topics, tt, [caps[0]] * nt, [caps[1]] * nt)
    d = delta(idx, before)
    offsets, ranks = res.expand()
    want = oracle_match(kv, tenants, topics, tt, caps[0], caps[1], mode)
    assert offsets.tolist() == want.offsets.tolist()
    assert ranks.tolist() == want.ranks.tolist()
    assert sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist()) == events_of(want)
    uncapped = oracle_match(kv, tenants, topics, tt, INT_MAX, INT_MAX, mode) if caps != (INT_MAX, INT_MAX) else want
    assert res.route_count.tolist() == np.diff(uncapped.offsets).tolist()
    return d, res


def check_device(idx, kv, tenants, topics, tt, caps, mode=O.MODE_BRUTE):
    """bfq_match_device + bfq_expand_device vs the oracle (ranks are unordered within a topic on the device) -> stats delta"""
    import torch
    from bifromq_b200 import _native as N
    from bifromq_b200 import dist as D
    dev = torch.device("cuda", 0)
    blob, off = N.as_blob(topics)
    n, nt = len(topics), len(tenants)
    tt = np.ascontiguousarray(tt, np.int32)
    d_topics = torch.from_numpy(blob).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    d_tt = torch.from_numpy(tt).to(dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    before = idx.stats()
    out = idx.match_device(tenants, d_topics.data_ptr(), d_off.data_ptr(), d_tt.data_ptr(), n, [caps[0]] * nt, [caps[1]] * nt, stream)
    d = delta(idx, before)
    d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    total = out.expand(d_offsets.data_ptr(), None, 0, stream)
    d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=dev)
    assert out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream) == total
    rc = D.device_view(out.d_route_count, n, "<u4", dev).cpu().numpy().astype(np.int64)
    thr = D.device_view(out.d_throttled, max(3 * out.n_throttled, 1), "<u4", dev).cpu().numpy()[:3 * out.n_throttled].reshape(-1, 3)
    torch.cuda.synchronize()
    offsets = d_offsets.cpu().numpy()
    ranks = d_ranks.cpu().numpy()[:total]
    want = oracle_match(kv, tenants, topics, tt, caps[0], caps[1], mode)
    assert offsets.tolist() == want.offsets.tolist()
    seg = np.repeat(np.arange(n), np.diff(offsets))
    assert ranks[np.lexsort((ranks, seg))].tolist() == want.ranks.tolist()
    assert sorted((int(k), int(t), int(r)) for t, r, k in thr.tolist()) == events_of(want)
    uncapped = oracle_match(kv, tenants, topics, tt, INT_MAX, INT_MAX, mode) if caps != (INT_MAX, INT_MAX) else want
    assert rc.tolist() == np.diff(uncapped.offsets).tolist()
    out.release()
    return d


def both_orders(idx, kv, tenants, topics, tt, caps_list=CAPS, mode=O.MODE_BRUTE):
    """each case in arrival order and in locality order with de-dup (order_min_topics 1) -> {(order, caps): stats delta}"""
    out = {}
    for order in ("arrival", "locality"):
        idx.set_option("order_min_topics", 0 if order == "arrival" else 1)
        for caps in caps_list:
            d, res = check_host(idx, kv, tenants, topics, tt, caps, mode)
            res.close()
            out[(order, caps)] = d
    idx.set_option("order_min_topics", 32768)
    return out


def distinct(tenants, topics, tt):
    return len(topics) - true_repeats(tenants, topics, tt)


# ------------------------------------------------------------------ A. tier-0 / tier-1 limits at the edge
@pytest.mark.gpu
def test_levels_at_the_tier0_depth_limit(B):
    pairs, tenants, topics, tt, deep = levels_case()
    idx = make_index(B, pairs)
    for (order, caps), d in both_orders(idx, kv_of(pairs), tenants, topics, tt).items():
        assert d["deferred_topics"] == deep, (order, caps, d)   # > 12 levels: tier 1; 11 and 12 stay in tier 0
        assert d["overflow_topics"] == 0
        assert d["duplicate_topics"] == 0
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("a", range(16))
def test_level_length_at_every_alignment(B, a):
    pairs, topics, starts = alignment_case(a)
    idx = make_index(B, pairs)
    tt = np.zeros(len(topics), np.int32)
    n_long = sum(1 for t in topics if any(len(x.encode()) > TOKEN_BYTES for x in t.split("/")))
    for (order, caps), d in both_orders(idx, kv_of(pairs), ["al"], topics, tt).items():
        # a level of > 24 bytes is deferred when the walk reaches it; the fillers repeat, so locality order de-dups them
        assert 0 < d["deferred_topics"] <= n_long, (order, d)
        assert d["duplicate_topics"] == (true_repeats(["al"], topics, tt) if order == "locality" else 0)
    idx.close()


@pytest.mark.gpu
def test_matched_filter_counts_across_inline_spill_and_tier_limits(B):
    pairs, tenants, topics, tt = ranges_case()
    idx = make_index(B, pairs)
    for (order, caps), d in both_orders(idx, kv_of(pairs), tenants, topics, tt).items():
        # 7 levels: <= 64 ranges stay in tier 0 (inline or spill), 65 -> tier 1 -> > 48 -> tier 2;
        # 14 levels: all deferred for depth, >= 49 ranges -> tier 2
        assert d["deferred_topics"] == 1 + len(RANGE_COUNTS), (order, caps, d)
        assert d["overflow_topics"] == 1 + sum(1 for n in RANGE_COUNTS if n > RG_CAP), (order, caps, d)
    idx.close()


@pytest.mark.gpu
def test_topic_length_limit(B):
    one_65535, one_65536 = "x" * 65535, "x" * 65536
    many_65535 = ("a/" * 32768)[:65535]
    many_65536 = "a/" * 32767 + "aa"
    topics = [one_65535, one_65536, many_65535, many_65536, "a", "x"]
    assert [len(t) for t in topics[:4]] == [65535, 65536, 65535, 65536]
    # "a/" * 13 + "#": the walk of the many-level topics reaches level 11 with levels to go
    pairs = make_pairs(one_route_each("long", ["#", "+", "+/#", "a/#", "a/a/#", "+/+/+", "x" * 30 + "/#", one_65535, "a/+/#",
                                               "a/" * 13 + "#"]))
    idx = make_index(B, pairs)
    kv = kv_of(pairs)
    for (order, caps), d in both_orders(idx, kv, ["long"], topics, np.zeros(len(topics), np.int32)).items():
        assert d["deferred_topics"] == 4, (order, d)   # > 65535 bytes at once, the others for a long level / their depth
    assert route_counts(kv, ["long"], topics, np.zeros(6, np.int32)).tolist()[:4] == [4, 3, 6, 6]
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_random_edge_batches(B, seed):
    pairs, tenants, topics, tt, want_n, deferred = random_edge_case(seed)
    idx = make_index(B, pairs)
    for (order, caps), d in both_orders(idx, kv_of(pairs), tenants, topics, tt).items():
        # > 12 levels, > 64 matched filters or a level of > 24 bytes (every level is walked): tier 1
        assert d["deferred_topics"] == deferred, (order, caps, d)
        assert d["duplicate_topics"] == (true_repeats(tenants, topics, tt) if order == "locality" else 0)
    idx.close()


# ------------------------------------------------------------------ B. buffer-growth re-runs
def spill_batch(n):
    return ["k%d/a/b/c/d" % i for i in range(n)]


@pytest.mark.gpu
def test_spill_region_exhausted_device_path(B):
    """enough distinct topics take a 64-range spill block to overflow a fresh workspace's range region: the batch is
    re-run with a grown region (device path); a second match on the handle reuses the grown workspace"""
    n = SPILL_REGION // SPILL_RANGES + 2048
    pairs = make_pairs(spill_filters("t"))
    kv = kv_of(pairs)
    topics = spill_batch(n)
    tt = np.zeros(n, np.int32)
    idx = make_index(B, pairs)
    for rep in range(2):
        d = check_device(idx, kv, ["t"], topics, tt, (INT_MAX, INT_MAX))
        assert d["buffer_retries"] == (1 if rep == 0 else 0), d
    d = check_device(idx, kv, ["t"], topics, tt, (6, 5))   # one drop per topic: the throttle list does not fill
    assert d["buffer_retries"] == 0 and d["flagged_topics"] > 0
    idx.close()


def check_dense_spans(res):
    sb, sc = res.span_begin.astype(np.int64), res.span_count.astype(np.int64)
    spans = np.unique(np.stack([sb[sc > 0], sc[sc > 0]], axis=1), axis=0)
    assert spans[0, 0] == 0 and (spans[1:, 0] == spans[:-1, 0] + spans[:-1, 1]).all()
    assert spans[-1, 0] + spans[-1, 1] == len(res.ranges)


@pytest.mark.gpu
def test_spill_region_exhausted_host_path(B):
    """>= 2^17 topics: the 4-sub-batch pipeline, one slice of the range region each; a slice overflows and the batch is
    redone un-chunked with grown buffers"""
    n = max(PIPELINE_TOPICS + 8192, SUB_BATCHES * (SPILL_REGION // SUB_BATCHES // SPILL_RANGES + 2048))
    pairs = make_pairs(spill_filters("t"))
    kv = kv_of(pairs)
    topics = spill_batch(n // 2) * 2   # every topic twice: locality order de-dups them (each sub-batch is ordered)
    random.Random(4).shuffle(topics)
    tt = np.zeros(len(topics), np.int32)
    # the re-run is un-chunked (one de-dup pass over the whole batch); with the grown workspace the next call is pipelined
    # again and each sub-batch is de-duplicated on its own
    n = len(topics)
    bounds = [n * c // SUB_BATCHES for c in range(SUB_BATCHES + 1)]
    per_sub = sum(true_repeats(["t"], topics[b:e], tt[b:e]) for b, e in zip(bounds, bounds[1:]))
    idx = make_index(B, pairs)
    for rep in range(2):
        d, res = check_host(idx, kv, ["t"], topics, tt, (INT_MAX, INT_MAX))
        assert d["buffer_retries"] == (1 if rep == 0 else 0), d
        assert d["duplicate_topics"] == (n // 2 if rep == 0 else per_sub), (rep, d)
        assert int(res.timings_ms["sub_batches"]) == (1 if rep == 0 else SUB_BATCHES)
        check_dense_spans(res)
        res.close()
    idx.close()


def throttle_case(n, per_topic):
    """every topic "k<i>/x" matches one filter of `per_topic` persistent routes: with a persistent cap of 0 each drops
    all of them"""
    pairs = make_pairs([("t", "+/x", "p", per_topic), ("t", "+/y", "n", 2)])
    return pairs, ["k%d/x" % i for i in range(n)]


@pytest.mark.gpu
def test_throttle_list_exhausted_device_path(B):
    per = 10
    n = THROTTLE_LIST // per + 1000
    pairs, topics = throttle_case(n, per)
    kv = kv_of(pairs)
    tt = np.zeros(n, np.int32)
    idx = make_index(B, pairs)
    for rep in range(2):
        d = check_device(idx, kv, ["t"], topics, tt, (0, 0))
        assert d["buffer_retries"] == (1 if rep == 0 else 0), d
    idx.close()


@pytest.mark.gpu
def test_throttle_list_exhausted_host_path(B):
    n = PIPELINE_TOPICS + 8192
    pairs, topics = throttle_case(n, 2)
    topics = topics + ["k%d/y" % i for i in range(64)]
    tt = np.zeros(len(topics), np.int32)
    kv = kv_of(pairs)
    idx = make_index(B, pairs)
    for rep in range(2):
        d, res = check_host(idx, kv, ["t"], topics, tt, (1, 0), O.MODE_TRIE)
        assert len(res.throttled) == n > THROTTLE_LIST
        assert d["buffer_retries"] == (1 if rep == 0 else 0), d
        check_dense_spans(res)
        assert res.throttled["topic"].max() == n - 1
        res.close()
    idx.close()


# ------------------------------------------------------------------ C. tier 2 with de-dup and caps
TIER2_CAPS = [(5, 0), (3, 1), (INT_MAX, INT_MAX)]


@pytest.mark.gpu
def test_repeated_tier2_topic_in_locality_order(B):
    routes, tenants, topics = tier2_case()
    pairs = make_pairs(routes)
    kv = kv_of(pairs)
    tt = np.zeros(len(topics), np.int32)
    idx = make_index(B, pairs)
    idx.set_option("order_min_topics", 1)
    rep = true_repeats(tenants, topics, tt)
    for caps in TIER2_CAPS:
        d, res = check_host(idx, kv, tenants, topics, tt, caps)
        res.close()
        assert d["overflow_topics"] == 1 and d["deferred_topics"] == 2 and d["duplicate_topics"] == rep, (caps, d)
        d = check_device(idx, kv, tenants, topics, tt, caps)
        assert d["overflow_topics"] == 1 and d["deferred_topics"] == 2 and d["duplicate_topics"] == rep, (caps, d)
    idx.close()


@pytest.mark.gpu
def test_repeated_tier2_topic_default_order_threshold(B):
    """>= 32768 topics: de-dup and locality order on the default setting"""
    routes, tenants, topics = tier2_case(n_other=33000, reps2=500, reps1=300, seed=5)
    pairs = make_pairs(routes)
    kv = kv_of(pairs)
    tt = np.zeros(len(topics), np.int32)
    assert len(topics) >= 32768
    idx = make_index(B, pairs)
    rep = true_repeats(tenants, topics, tt)
    for caps in TIER2_CAPS:
        d, res = check_host(idx, kv, tenants, topics, tt, caps, O.MODE_TRIE)
        res.close()
        assert d["overflow_topics"] == 1 and d["deferred_topics"] == 2 and d["duplicate_topics"] == rep, (caps, d)
        d = check_device(idx, kv, tenants, topics, tt, caps, O.MODE_TRIE)
        assert d["overflow_topics"] == 1 and d["deferred_topics"] == 2 and d["duplicate_topics"] == rep, (caps, d)
    idx.close()


@pytest.mark.gpu
def test_tier2_after_delta_commit_widens_the_deepest_level(B):
    """tier-2 scratch is sized from max_nodes_per_depth / max_tenant_nodes, which a delta commit merges: add {a,+}^9
    (512 nodes at depth 9, a frontier of 512 for a^9) to a tenant through the delta path and match a^9 repeatedly"""
    routes, tenants, topics = tier2_case()
    routes = routes + [("other", "x/+", "p", 3)]
    pairs = make_pairs(routes)
    idx = make_index(B, pairs)
    kv = kv_of(pairs)
    wide = one_route_each("t", ["/".join(c) for c in itertools.product(["a", "+"], repeat=9)])
    extra = make_pairs(wide)
    before = idx.stats()
    idx.apply(adds=extra)
    idx.commit()
    for k, v in extra:
        kv.put(k, v)
    kv.freeze()
    st = idx.stats()
    assert st["delta_commits"] == before["delta_commits"] + 1 and st["max_nodes_per_depth"] > before["max_nodes_per_depth"]
    topic9 = "/".join(["a"] * 9)
    topics = topics + [topic9] * 30
    random.Random(9).shuffle(topics)
    tt = np.zeros(len(topics), np.int32)
    idx.set_option("order_min_topics", 1)
    for caps in TIER2_CAPS:
        d, res = check_host(idx, kv, tenants, topics, tt, caps)
        res.close()
        assert d["overflow_topics"] == 2 and d["duplicate_topics"] == true_repeats(tenants, topics, tt), (caps, d)
    assert route_counts(kv, tenants, [topic9], [0]).tolist() == [512 + 7]
    idx.close()


# ------------------------------------------------------------------ D. de-dup under forced hash collisions
@pytest.mark.gpu
@pytest.mark.parametrize("bits", [0, 10])
def test_dedup_with_forced_hash_collisions(B, bits):
    pairs, tenants, topics, tt = dedup_collision_case()
    idx = make_index(B, pairs)
    kv = kv_of(pairs)
    idx.set_option("order_min_topics", 1)
    idx.set_option("dedup_hash_bits", bits)
    rep = true_repeats(tenants, topics, tt)
    for caps in [(INT_MAX, INT_MAX), (0, 1)]:
        d, res = check_host(idx, kv, tenants, topics, tt, caps)
        res.close()
        assert d["duplicate_topics"] == rep, (caps, d)
    d = check_device(idx, kv, tenants, topics, tt, (INT_MAX, INT_MAX))
    assert d["duplicate_topics"] == rep, d
    with pytest.raises(B.NativeError):
        idx.set_option("dedup_hash_bits", 65)
    idx.close()


# ------------------------------------------------------------------ E. tier-0 builds and occupancy
_BUILD_SCRIPT = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import bifromq_b200
d = sys.argv[2]
z = np.load(d + "/case.npz", allow_pickle=False)
tenants = [t.decode() for t in z["tenants"]]
idx = bifromq_b200.GpuRouteIndex(0)
idx.load(z["keys"], z["key_off"], z["vals"], z["val_off"])
idx.commit()
nt = len(tenants)
for order in (0, 1):
    idx.set_option("order_min_topics", 0 if order == 0 else 1)
    res = idx.match(tenants, z["topics"], z["topic_off"], z["tt"], [3] * nt, [1] * nt)
    off, ranks = res.expand()
    np.save(d + "/offsets%d.npy" % order, off)
    np.save(d + "/ranks%d.npy" % order, ranks)
    np.save(d + "/route_count%d.npy" % order, res.route_count.astype(np.int64))
    np.save(d + "/events%d.npy" % order, np.array(sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist()), np.int64).reshape(-1, 3))
    res.close()
st = idx.stats()
np.save(d + "/deferred.npy", np.array([st["deferred_topics"], st["duplicate_topics"]], np.int64))
"""


@pytest.fixture(scope="module")
def build_case(tmp_path_factory):
    """a C3 slice plus the section-A edge topics of an extra tenant, with '$' topics and root '#' / '+' filters"""
    from bifromq_b200 import workload
    w = workload.Workload("C3", scale=0.005)
    keys = [bytes(w.keys[w.key_off[i]:w.key_off[i + 1]]) for i in range(len(w.key_off) - 1)]
    vals = [bytes(w.vals[w.val_off[i]:w.val_off[i + 1]]) for i in range(len(w.val_off) - 1)]
    lv_pairs, _, lv_topics, lv_tt, _ = levels_case()
    rg_pairs, _, rg_topics, _ = ranges_case()
    edge = make_pairs(one_route_each("zzedge", ["#", "+", "+/x", "$sys/+", "$sys/#"]))
    edge_t = ["lv", "lv0", "rg", "zzedge"]
    pairs = dict(zip(keys, vals))
    for k, v in lv_pairs + rg_pairs + edge:
        pairs[k] = v
    pairs = sorted(pairs.items())
    tenants = w.tenants + edge_t
    base = len(w.tenants)
    topics = w.topic_list() + lv_topics + rg_topics + ["$sys/a", "$sys/x/y", "$", "x", "a/x", "/x"]
    tt = np.concatenate([np.asarray(w.topic_tenant[:w.n_topics], np.int32), base + lv_tt, np.full(len(rg_topics), base + 2, np.int32),
                         np.full(6, base + 3, np.int32)]).astype(np.int32)
    d = tmp_path_factory.mktemp("builds")
    kb, ko = O.blob([k for k, _ in pairs])
    vb, vo = O.blob([v for _, v in pairs])
    tb, to = O.blob(topics)
    np.savez(d / "case.npz", keys=kb, key_off=ko, vals=vb, val_off=vo, topics=tb, topic_off=to, tt=tt,
             tenants=np.array([t.encode() for t in tenants]))
    kv = O.KV()
    kv.load(kb, ko, vb, vo)
    kv.freeze()
    want = kv.match_batch(tenants, topics, tt, 3, 1, O.MODE_TRIE, False, 8)
    uncapped = kv.match_batch(tenants, topics, tt, INT_MAX, INT_MAX, O.MODE_TRIE, False, 8)
    return d, want, np.diff(uncapped.offsets)


BUILDS = [dict(BFQ_ROOTSTEP=str(r), BFQ_PREFETCH=str(p), BFQ_NOALLOC=str(a)) for r in (0, 1) for p in (0, 1) for a in (0, 1)]
BUILDS.append(dict(BFQ_CTAS="1"))


@pytest.mark.gpu
@pytest.mark.parametrize("env", BUILDS, ids=lambda e: ",".join("%s=%s" % kv for kv in sorted(e.items())))
def test_tier0_builds(build_case, env, tmp_path):
    """the tier-0 switches are read once per process: each build runs in its own process (ctypes only) and writes its
    results; both orders equal the oracle"""
    d, want, route_count = build_case
    out = tmp_path / "out"
    out.mkdir()
    import shutil
    shutil.copy(d / "case.npz", out / "case.npz")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    e = dict(os.environ)
    for k in ("BFQ_ROOTSTEP", "BFQ_PREFETCH", "BFQ_NOALLOC", "BFQ_CTAS", "BFQ_ORDER", "BFQ_DEDUP"):
        e.pop(k, None)
    e.update(env)
    subprocess.run([sys.executable, "-c", _BUILD_SCRIPT, root, str(out)], env=e, check=True, timeout=600)
    for order in (0, 1):
        assert np.load(out / ("offsets%d.npy" % order)).tolist() == want.offsets.tolist()
        assert np.load(out / ("ranks%d.npy" % order)).tolist() == want.ranks.tolist()
        assert [tuple(x) for x in np.load(out / ("events%d.npy" % order)).tolist()] == events_of(want)
        assert np.load(out / ("route_count%d.npy" % order)).tolist() == route_count.tolist()
    deferred, dups = np.load(out / "deferred.npy").tolist()
    assert deferred > 0


@pytest.mark.gpu
def test_tier0_occupancy_settings_large_device_batch(B):
    """>= 2^17 topics on the device path (at most 4 tier-0 CTAs per SM by default) with tier0_ctas_per_sm unset, 1 and 6"""
    from bifromq_b200 import workload
    w = workload.Workload("C3", scale=0.02)
    idx = B.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    idx.commit()
    kv = O.KV()
    kv.load(w.keys, w.key_off, w.vals, w.val_off)
    kv.freeze()
    reps = (PIPELINE_TOPICS + 4096 + w.n_topics - 1) // w.n_topics
    perm = np.random.RandomState(7).permutation(w.n_topics * reps)
    base = w.topic_list()
    topics = [base[i % w.n_topics] for i in perm]
    tt = np.ascontiguousarray(np.asarray(w.topic_tenant[:w.n_topics], np.int32)[perm % w.n_topics])
    assert len(topics) >= PIPELINE_TOPICS
    for ctas in (None, 1, 6):
        if ctas is not None:
            idx.set_option("tier0_ctas_per_sm", ctas)
        d = check_device(idx, kv, w.tenants, topics, tt, (3, 1), O.MODE_TRIE)
        assert d["duplicate_topics"] == true_repeats(w.tenants, topics, tt), (ctas, d)
    idx.close()
