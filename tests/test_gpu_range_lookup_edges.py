"""bfq_range_lookup at its edges: every row is compared with the oracle's literal restatement of TenantRangeLookupCache.lookup
and, where the topic is shallow enough to enumerate, with the brute force of tests/range_lookup_brute.py.

Depth (topics of up to 2000 levels and one near MaxTopicLength, bounds of up to 200 levels, in batches with shallow topics),
level order around "#" / "+" and in multi-byte text, bounds derived from each topic's own members, the '$' rule, the candidate
loop (stops, missing Facts, empty chains between other rows), ranges cut from a generated route set, many blocks and a topic
blob passed as a slice, and the call's error contract."""
import random
import threading

import numpy as np
import pytest

import oracle_lib as O
import range_lookup_brute as R

pytestmark = pytest.mark.gpu

BFQ_OK, BFQ_E_INVALID, BFQ_E_RANGE = 0, -1, -5


def oracle_rows(rows):
    """the oracle's answer per row; run in a thread with a large stack, since its topic trie is walked recursively and the
    longest topic here has about 40 000 levels"""
    out = [None] * len(rows)

    def run():
        for i, (tenant, topic, chain) in enumerate(rows):
            out[i] = O.range_lookup(tenant, topic, chain)
    old = threading.stack_size(1 << 30)
    try:
        th = threading.Thread(target=run)
        th.start()
        th.join()
    finally:
        threading.stack_size(old)
    assert all(o is not None for o in out)
    return out


def check_rows(rows):
    """rows: (tenant, topic, chain); one tenant entry per row, all in ONE call. Returns the kernel's rows."""
    from bifromq_b200 import dist as D
    got = D.range_lookup([r[0] for r in rows], [r[1] for r in rows], np.arange(len(rows), dtype=np.int32), [r[2] for r in rows])
    want = oracle_rows(rows)
    for i, (tenant, topic, chain) in enumerate(rows):
        assert got[i] == want[i], (i, tenant, topic[:200], len(topic.split("/")), chain[:4], got[i], want[i])
        if topic.count("/") < R.BRUTE_MAX_LEVELS:
            assert want[i] == R.brute_lookup(tenant, topic, chain), (tenant, topic, chain)
    return got


def singles(tenant, topic, pairs):
    """one row per candidate, so no candidate's stop hides the ones behind it"""
    return [(tenant, topic, [p]) for p in pairs]


# ------------------------------------------------------------------ depth
def test_deep_topics_and_bounds_with_shallow_topics_in_one_batch():
    """Topics of 1..2000 levels and one of about 40 000 levels (65 534 bytes of empty and one-byte levels), bounds of the tenant
    plus 33, 34, 35 and 200 levels and of the topic's own depth +-1, next to shallow topics: the whole batch succeeds and every
    row matches the oracle, which takes every depth here."""
    rows = []
    rng = random.Random(5)
    for n in R.DEPTH_TOPIC_LEVELS:
        topic = R.deep_topic(n)
        for k in sorted(set(R.DEPTH_BOUND_LEVELS + [1, max(1, n - 1), n, n + 1])):
            for b in R.depth_bounds(topic, R.TENANT, k):
                rows += singles(R.TENANT, topic, [(b, b), (b, [R.TENANT, "~"]), (b, b[:-1] + ["$"]), ([R.TENANT, "!"], b)])
        rows += singles("tA", topic, [([R.TENANT], [R.TENANT, "~"])])   # a bound of a greater tenant
        rows += singles("tC", topic, [([R.TENANT], [R.TENANT, "~"]), ([R.TENANT], ["tC", "~"])])
        rows.append((R.TENANT, topic, [None, ([R.TENANT, "a"], [R.TENANT, "b"]), None]))
    lt = R.long_topic()
    lv = lt.split("/")
    for k in (1, 34, 35, 1000, len(lv) - 1, len(lv), len(lv) + 1):
        for b in R.depth_bounds(lt, R.TENANT, k):
            rows += singles(R.TENANT, lt, [(b, b), (b, [R.TENANT, "~"])])
    for topic in R.order_topics(rng, 200, 6):   # shallow rows around the deep ones
        rows.append((R.TENANT, topic, [([R.TENANT, "!"], [R.TENANT, "z"]), ([R.TENANT, "a"], [R.TENANT, "a", "#"])]))
    rng.shuffle(rows)
    got = check_rows(rows)
    assert sum(map(len, got)) > len(rows) // 4
    assert any(len(t.split("/")) > 34 and g for (_, t, _), g in zip(rows, got))


def test_deep_bounds_on_shallow_topics():
    """bounds of the tenant plus 33, 34, 35 and 200 levels against topics of 1-6 levels: members run out long before the bound
    does, so the seek falls back from shallow depths"""
    rng = random.Random(9)
    rows = []
    for topic in R.order_topics(rng, 40, 6):
        t = topic.split("/")
        for k in R.DEPTH_BOUND_LEVELS:
            for b in R.depth_bounds(topic, R.TENANT, k) + [[R.TENANT] + ["+"] * k, [R.TENANT] + t + ["#"] * (k - len(t))]:
                rows += singles(R.TENANT, topic, [(b, b), (b, [R.TENANT, "~"]), ([R.TENANT], b), (b[:len(t) + 1], b)])
    got = check_rows(rows)
    assert any(got) and not all(got)


# ------------------------------------------------------------------ level order and derived bounds
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_level_order_bands_with_derived_bounds(seed):
    """levels from every band around "#" / "+" and multi-byte text; bounds from each topic's own members (each member, with a
    level dropped, appended or replaced by a neighbour, under smaller / equal / greater / prefix / extended tenants), paired
    with last <, = and > first"""
    rng = random.Random(seed)
    rows = []
    for topic in R.order_topics(rng, 10, 4):
        rows += singles(R.TENANT, topic, R.bound_pairs(R.derived_bounds(topic)))
    got = check_rows(rows)
    assert 0.05 < sum(map(len, got)) / len(rows) < 0.95


def test_fallback_from_every_depth_of_the_tight_path():
    rng = random.Random(17)
    rows = []
    for topic in R.order_topics(rng, 60, 12):
        for d, b in R.tight_path_bounds(topic):
            rows += singles(R.TENANT, topic, [(b, b), (b, [R.TENANT, "~"]), (b, [R.TENANT]), (b, b[:-1] + ["#"])])
    check_rows(rows)


def test_sys_rule():
    """'$' topics of 1-4 levels (and the topic "$") with bounds through "+" / "#" at level 1 and deeper; a tenant id starting
    with '$' does not trigger the rule"""
    rows = []
    for topic in ["$", "$s", "$s/a", "$s/#x/!", "$s//a/b", "$/+b/ab/中", "$sys/~/é/z"]:
        for tenant in (R.TENANT, "$t", "$"):
            rows += singles(tenant, topic, R.bound_pairs(R.derived_bounds(topic, tenant)))
            t = topic.split("/")
            for d in range(len(t) + 1):
                for w in ("#", "+"):
                    b = [tenant] + t[:d] + [w]
                    rows += singles(tenant, topic, [(b, b), (b, [tenant, "~"])])
    got = check_rows(rows)
    assert any(g for g in got)


# ------------------------------------------------------------------ the candidate loop
def test_candidate_chains_and_empty_chains_between_rows():
    """chains of 0, 1, 2 and 1000 candidates; stops on candidate 0, in the middle and at the end; no-Fact ranges before and
    after a stop; Facts without first, last or both; tenants with empty chains as the first, a middle and the last row"""
    from bifromq_b200 import dist as D
    rng = random.Random(23)
    tenants, chains, topics, tt = [], [], [], []

    def entry(tenant, chain):
        tenants.append(tenant)
        chains.append(chain)
        return len(tenants) - 1
    empty = [entry(R.TENANT, []) for _ in range(3)]
    topics_of = ["a/!/中", "$s/a", "/", "~/+b/é", "a"]
    for topic in topics_of:
        pools = R.candidate_pools(R.TENANT, topic)
        for pattern in R.CHAIN_PATTERNS + ["K" * 2, "".join(rng.choice("KKKDDNFLB") for _ in range(999)) + "S",
                                           "".join(rng.choice("KDN") for _ in range(499)) + "S" + "KN" * 250]:
            e = entry(R.TENANT, R.chain_from_pattern(rng, pools, pattern))
            topics.append(topic)
            tt.append(e)
            if rng.random() < 0.5:            # an empty chain in the middle, several in a row
                for _ in range(rng.randint(1, 3)):
                    topics.append(topic)
                    tt.append(rng.choice(empty))
    topics = [topics_of[0]] + topics + [topics_of[1]]
    tt = [empty[0]] + tt + [empty[2]]
    got = D.range_lookup(tenants, topics, np.asarray(tt, np.int32), chains)
    want = oracle_rows([(tenants[e], topics[i], chains[e]) for i, e in enumerate(tt)])
    for i, e in enumerate(tt):
        assert got[i] == want[i], (i, topics[i], len(chains[e]), got[i], want[i])
        assert want[i] == R.brute_lookup(tenants[e], topics[i], chains[e])
    assert got[0] == [] and got[-1] == []
    assert {len(chains[e]) for e in tt} >= {0, 1, 2, 1000}


# ------------------------------------------------------------------ real route sets
def test_ranges_cut_from_a_route_set_keep_every_range_holding_a_match():
    """per tenant the distinct filters of a generated route set (config C3, reduced), in Java level order, cut into 1, 7 and 64
    contiguous ranges whose Facts are their smallest and largest filter. For every topic of the workload, a range holding a
    filter that matches the topic (the oracle's predicate) is kept, and the kept set equals the oracle's."""
    from bifromq_b200 import dist as D
    from bifromq_b200.workload import Workload
    w = Workload("C3", scale=0.0005)
    per = R.tenant_filters(w)
    tenants = w.tenants
    topics = [w.topic(i).decode() if isinstance(w.topic(i), bytes) else w.topic(i) for i in range(w.n_topics)]
    tti = [int(x) for x in w.topic_tenant[:w.n_topics]]
    matches = {}
    for i, topic in enumerate(topics):
        fs = per[tenants[tti[i]]]
        matches[i] = {j for j, f in enumerate(fs) if O.topic_matches_filter(topic, "/".join(f[1:]))}
    assert sum(map(len, matches.values())) > len(topics)
    for k in (1, 7, 64):
        ents, chains = [], []
        for t in tenants:
            ranges = R.cut_ranges(per[t], k)
            ents.append(t)
            chains.append([(f, l) for f, l, _ in ranges])
        got = D.range_lookup(ents, topics, np.asarray(tti, np.int32), chains)
        want = oracle_rows([(tenants[tti[i]], topics[i], chains[tti[i]]) for i in range(len(topics))])
        for i, topic in enumerate(topics):
            fs = per[tenants[tti[i]]]
            assert got[i] == want[i], (topic, k, got[i], want[i])
            ranges = R.cut_ranges(fs, k)
            pos = 0
            for r, (_, _, part) in enumerate(ranges):
                if any(j in matches[i] for j in range(pos, pos + len(part))):
                    assert r in got[i], (topic, k, r)
                pos += len(part)


# ------------------------------------------------------------------ size
def _pack(tenants, topics_blob, topic_off, tt, chains):
    from bifromq_b200 import _native as N
    tb, toff = N.as_blob(tenants)
    cand_off = np.zeros(len(tenants) + 1, np.int64)
    flags, firsts, lasts = [], [], []
    for t, cl in enumerate(chains):
        cand_off[t + 1] = cand_off[t] + len(cl)
        for c in cl:
            f, l = (None, None) if c is None else c
            flags.append(0 if c is None else 1 | (2 if f is not None else 0) | (4 if l is not None else 0))
            firsts.append("\0".join(f).encode() if f is not None else b"")
            lasts.append("\0".join(l).encode() if l is not None else b"")
    fl = np.asarray(flags + [0], np.uint8)
    fb, foff = N.as_blob(firsts)
    lb, loff = N.as_blob(lasts)
    tt = np.ascontiguousarray(tt, np.int32)
    total = int(sum(cand_off[t + 1] - cand_off[t] for t in tt.tolist() if 0 <= t < len(tenants)))
    keep_off = np.zeros(len(tt) + 1, np.int64)
    keep = np.zeros(max(total, 1), np.uint8)
    args = [0, N.ptr(tb), N.ptr(toff), len(tenants), N.ptr(topics_blob), N.ptr(topic_off), N.ptr(tt), len(tt), N.ptr(cand_off),
            N.ptr(fl), N.ptr(fb), N.ptr(foff), N.ptr(lb), N.ptr(loff), N.ptr(keep_off), N.ptr(keep)]
    return args, (tb, toff, tt, cand_off, fl, fb, foff, lb, loff, topics_blob, topic_off), keep_off, keep


def test_millions_of_pairs_from_a_sliced_topic_blob_and_long_levels():
    """2 million (topic, candidate) pairs over many blocks, the topic blob passed as a slice of a larger one (topic_off[0] > 0),
    levels of 255+ bytes; a repeat call gives identical rows"""
    from bifromq_b200 import _native as N
    from bifromq_b200.workload import Workload
    w = Workload("C3", scale=0.0005)
    per = R.tenant_filters(w)
    tenant = max(per, key=lambda t: len(per[t]))
    fs = per[tenant]
    ranges = R.cut_ranges(fs, 1000)
    assert len(ranges) == 1000
    chain = [(f, l) for f, l, _ in ranges]
    chain[500] = None
    rng = random.Random(29)
    topics = []
    for i in range(2000):
        f = list(rng.choice(fs)[1:])
        lv = [x if x not in ("+", "#") else rng.choice(["a", "", "x" * 300]) for x in f]
        if i % 7 == 0:
            lv[rng.randrange(len(lv))] = rng.choice(["é" * 130, "z" * 255, "!" * 400])
        topics.append("/".join(lv))
    junk = b"junk/prefix/" * 3
    blob = junk + b"".join(t.encode() for t in topics)
    off = np.zeros(len(topics) + 1, np.int64)
    off[0] = len(junk)
    off[1:] = len(junk) + np.cumsum([len(t.encode()) for t in topics])
    blob_np = np.frombuffer(blob, np.uint8).copy()
    args, keep_alive, keep_off, keep = _pack([tenant], blob_np, off, np.zeros(len(topics), np.int32), [chain])
    assert N.lib.bfq_range_lookup(*args) == BFQ_OK
    assert int(keep_off[-1]) == 2_000_000
    first = keep.copy()
    got = [np.nonzero(keep[keep_off[i]:keep_off[i + 1]])[0].tolist() for i in range(len(topics))]
    want = oracle_rows([(tenant, t, chain) for t in topics])
    for i, t in enumerate(topics):
        assert got[i] == want[i], (i, t[:100], got[i][:10], want[i][:10])
    assert sum(map(len, got)) > len(topics)
    keep[:] = 7
    assert N.lib.bfq_range_lookup(*args) == BFQ_OK
    assert np.array_equal(keep, first)


# ------------------------------------------------------------------ errors
def test_error_contract():
    from bifromq_b200 import _native as N
    chain = [([R.TENANT, "a"], [R.TENANT, "b"]), None]
    blob = np.frombuffer(b"a/b", np.uint8).copy()
    off = np.asarray([0, 3], np.int64)
    args, keep_alive, keep_off, keep = _pack([R.TENANT], blob, off, [1], [chain])
    assert N.lib.bfq_range_lookup(*args) == BFQ_E_RANGE            # topic_tenant 1 of 1 tenant
    args, keep_alive, keep_off, keep = _pack([R.TENANT], blob, off, [-1], [chain])
    assert N.lib.bfq_range_lookup(*args) == BFQ_E_RANGE
    args, keep_alive, keep_off, keep = _pack([R.TENANT], blob, off, [0], [chain])
    for i in (1, 2, 4, 5, 6, 8, 14, 15):   # tenants, tenant_off, topics, topic_off, topic_tenant, cand_off, keep_off, keep
        bad = list(args)
        bad[i] = None
        assert N.lib.bfq_range_lookup(*bad) == BFQ_E_INVALID, i
    for i in (9, 11, 13):                  # cand_flags, first_off, last_off, with candidates present
        bad = list(args)
        bad[i] = None
        assert N.lib.bfq_range_lookup(*bad) == BFQ_E_INVALID, i
    assert N.lib.bfq_range_lookup(*args) == BFQ_OK
    assert keep[:2].tolist() == [1, 1] and keep_off.tolist() == [0, 2]
    # no topics; and topics whose chains are all empty: OK, every row empty
    args, keep_alive, keep_off, keep = _pack([R.TENANT], blob, off[:1], [], [chain])
    assert N.lib.bfq_range_lookup(*args) == BFQ_OK and keep_off.tolist() == [0]
    args, keep_alive, keep_off, keep = _pack([R.TENANT, "tC"], np.frombuffer(b"a/ba/b", np.uint8).copy(),
                                             np.asarray([0, 3, 3, 6], np.int64), [0, 1, 0], [[], []])
    keep_off[:] = 9
    assert N.lib.bfq_range_lookup(*args) == BFQ_OK and keep_off.tolist() == [0, 0, 0, 0]


def test_supplementary_plane_text_orders_by_utf8_bytes():
    """Documents a known divergence that stays out of scope (the MQTT edge rejects supplementary-plane text): the kernel
    compares UTF-8 bytes, Java compares UTF-16 code units, and the two disagree between U+1F600 and U+FF5E. For topic "～" and
    the range [😀, ～] Java's seek finds "～" and keeps the range; the kernel finds nothing at or above "😀" and stops."""
    from bifromq_b200 import dist as D
    a, b = "\U0001F600", "～"
    chain = [([R.TENANT, a], [R.TENANT, b]), None]
    assert O.range_lookup(R.TENANT, b, chain) == [0, 1]
    assert D.range_lookup([R.TENANT], [b], np.zeros(1, np.int32), [chain]) == [[]]
    # on BMP text both orders agree
    chain = [([R.TENANT, "中"], [R.TENANT, b]), None]
    assert D.range_lookup([R.TENANT], [b], np.zeros(1, np.int32), [chain]) == [O.range_lookup(R.TENANT, b, chain)] == [[0, 1]]
