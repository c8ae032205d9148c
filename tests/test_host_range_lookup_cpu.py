"""The range lookup's brute force (tests/range_lookup_brute.py) against the oracle's restatement of TenantRangeLookupCache.lookup,
without a GPU, on every case generator the kernel tests use; and the shape of each generator, so a later change to one cannot
silently stop reaching the edge it is there for."""
import random

import pytest

import oracle_lib as O
import range_lookup_brute as R


def agree(tenant, topic, candidates):
    want = O.range_lookup(tenant, topic, candidates)
    assert R.brute_lookup(tenant, topic, candidates) == want, (tenant, topic, candidates, want)
    return want


def test_brute_force_on_hand_checked_cases():
    # tB/a/!: the expansion set in Java order is "#" < "+" < "a" at level 1, and under a: "!" < "#" < "+"; a one-level
    # filter other than "#" does not match a two-level topic
    assert R.expansion_set("tB", "a/!") == [
        ("tB", "#"), ("tB", "+", "!"), ("tB", "+", "!", "#"), ("tB", "+", "#"), ("tB", "+", "+"), ("tB", "+", "+", "#"),
        ("tB", "a", "!"), ("tB", "a", "!", "#"), ("tB", "a", "#"), ("tB", "a", "+"), ("tB", "a", "+", "#")]
    # no wildcard right under the tenant level of a '$' topic, but below it
    assert R.expansion_set("tB", "$s/x") == [("tB", "$s", "#"), ("tB", "$s", "+"), ("tB", "$s", "+", "#"), ("tB", "$s", "x"),
                                             ("tB", "$s", "x", "#")]
    # a '$' in the tenant id is not the '$' rule
    assert ("$t", "#") in R.expansion_set("$t", "a")
    b = R.Brute("tB", "a/!")
    assert b.seek(["tB", "a", " "]) == ("tB", "a", "!")
    assert b.seek(["tB", "a", "\""]) == ("tB", "a", "#")
    assert b.seek(["tB", "a", "+", "$"]) is None
    # no Fact: kept; found <= last: kept; no last: skipped; nothing >= first: stop, so the last no-Fact range is not kept
    assert b.lookup([None, (["tB", "a", "\"x"], ["tB", "a", "#"]), (["tB", "b"], None), (["tB", "b"], ["tB", "z"]), None]) == [0, 1]
    assert b.lookup([(["tC"], ["tC"]), None]) == []


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_derived_bounds_on_order_topics(seed):
    """every band of the level order, bounds from the topic's own members, last <, = and > first"""
    rng = random.Random(seed)
    kept = dropped = 0
    for topic in R.order_topics(rng, 12, 3):
        for first, last in R.bound_pairs(R.derived_bounds(topic)):
            got = agree(R.TENANT, topic, [(first, last)])
            kept += len(got)
            dropped += 1 - len(got)
    assert kept > 1000 and dropped > 1000


def test_tight_path_fallback_from_every_depth():
    rng = random.Random(7)
    for topic in R.order_topics(rng, 40, 12):
        for d, b in R.tight_path_bounds(topic):
            for last in (b, [R.TENANT, "~"], [R.TENANT]):
                agree(R.TENANT, topic, [(b, last)])


def test_depth_cases_within_enumeration():
    for n in [x for x in R.DEPTH_TOPIC_LEVELS if x <= R.BRUTE_MAX_LEVELS] + [R.BRUTE_MAX_LEVELS]:
        topic = R.deep_topic(n)
        for k in range(1, n + 3):
            bounds = R.depth_bounds(topic, R.TENANT, k)
            agree(R.TENANT, topic, [(b, b) for b in bounds])
            agree(R.TENANT, topic, [(b, [R.TENANT, "~"]) for b in bounds])


def test_sys_rule_cases():
    cases = ["$", "$s", "$s/a", "$s/#x/!", "$s//a/b", "$/+b/ab/中"]
    for topic in cases:
        for tenant in ("tB", "$t", "$"):
            for first, last in R.bound_pairs(R.derived_bounds(topic, tenant)):
                agree(tenant, topic, [(first, last)])


def test_candidate_chains():
    rng = random.Random(11)
    for topic in ["a/!/中", "$s/a", "/", "~/+b/é"]:
        pools = R.candidate_pools(R.TENANT, topic)
        for pattern in R.CHAIN_PATTERNS:
            agree(R.TENANT, topic, R.chain_from_pattern(rng, pools, pattern))
        agree(R.TENANT, topic, R.chain_from_pattern(rng, pools, "".join(rng.choice("KKKDDNFLB") for _ in range(999)) + "S"))


def test_real_route_set_ranges():
    """ranges cut from a generated route set; every range that holds a filter matching the topic is kept"""
    from bifromq_b200.workload import Workload
    w = Workload("C3", scale=0.0005)
    per = R.tenant_filters(w)
    tenants = w.tenants
    for i in range(0, w.n_topics, 5):
        tenant = tenants[w.topic_tenant[i]]
        topic = w.topic(i)
        topic = topic.decode() if isinstance(topic, bytes) else topic
        for k in (1, 7, 64):
            ranges = R.cut_ranges(per[tenant], k)
            kept = agree(tenant, topic, [(f, l) for f, l, _ in ranges])
            for r, (_, _, fs) in enumerate(ranges):
                if any(O.topic_matches_filter(topic, "/".join(f[1:])) for f in fs):
                    assert r in kept, (topic, r)


# ------------------------------------------------------------------ shapes of the generators
def test_order_vocab_covers_every_band():
    bands = {
        "below #": lambda v: v == "" or v[0] < "#",
        "#-prefixed": lambda v: v.startswith("#") and v != "#",
        "between # and +": lambda v: v and "#" < v[0] < "+",
        "+-prefixed": lambda v: v.startswith("+") and v != "+",
        "above + in ASCII": lambda v: v and "+" < v[0] <= "~",
        "DEL": lambda v: v == "\x7f",
        "two-byte": lambda v: len(v.encode()) == 2,
        "three-byte": lambda v: len(v.encode()) == 3,
    }
    for name, pred in bands.items():
        assert any(pred(v) for v in R.TOPIC_VOCAB), name
    for name in ["", " ", "!", "\"", "$", "%", "*", ",", "~", "\x7f", "é", "中", "～"]:
        assert name in R.TOPIC_VOCAB, name
    assert "#" not in R.TOPIC_VOCAB and "+" not in R.TOPIC_VOCAB


def test_depth_generators_reach_the_old_limit_and_beyond():
    for n in R.DEPTH_TOPIC_LEVELS:
        assert len(R.deep_topic(n).split("/")) == n
    assert {34, 35, 2000} <= set(R.DEPTH_TOPIC_LEVELS)
    topic = R.deep_topic(2000)
    for k in R.DEPTH_BOUND_LEVELS:
        for b in R.depth_bounds(topic, R.TENANT, k):
            assert len(b) == k + 1
    assert {33, 34, 35} <= set(R.DEPTH_BOUND_LEVELS)   # 34 and 35 levels including the tenant level are both reached
    lt = R.long_topic()
    assert 65000 < len(lt.encode()) <= 65535
    assert set(lt.split("/")) == {"", "a", "b"} and len(lt.split("/")) > 39000
    # the deep topics send the completion through levels below "#" as well as ordinary ones
    assert {"", "!", "a"} <= set(topic.split("/"))


def test_tight_path_bounds_leave_at_every_depth():
    topic = "a/!/中/$"
    t = topic.split("/")
    sides = {}
    for d, bound in R.tight_path_bounds(topic):
        assert len(bound) == d + 2 and bound[:d + 1] == [R.TENANT] + t[:d]
        here = R.java_key([(t + ["#"])[d]])
        assert R.java_key([bound[-1]]) != here
        sides.setdefault(d, set()).add(R.java_key([bound[-1]]) < here)
    # every depth, including one past the last level, is left both below and above the tight path
    assert sides == {d: {True, False} for d in range(len(t) + 1)}


def test_derived_bounds_hit_every_relation():
    topic = "a/!/中"
    bounds = R.derived_bounds(topic)
    members = set(R.expansion_set(R.TENANT, topic))
    assert sum(tuple(b) in members for b in bounds) == len(members)
    assert {b[0] for b in bounds} == set(R.TENANT_VARIANTS)
    tk = R.java_key([R.TENANT])
    rel = {(R.java_key([tv]) > tk) - (R.java_key([tv]) < tk) for tv in R.TENANT_VARIANTS}
    assert rel == {-1, 0, 1}
    pairs = R.bound_pairs(bounds)
    order = {(R.java_key(l) > R.java_key(f)) - (R.java_key(l) < R.java_key(f)) for f, l in pairs}
    assert order == {-1, 0, 1}
    kinds = {R.classify(R.TENANT, topic, f, l) for f, l in pairs}
    assert kinds == {"keep", "drop", "stop"}
    # a bound equal to a member but with last < first: kept only through the "found equals first" rule
    assert any(tuple(f) in members and R.java_key(l) < R.java_key(f) for f, l in pairs)


def test_chain_patterns_reach_their_edges():
    rng = random.Random(3)
    topic = "a/!/中"
    pools = R.candidate_pools(R.TENANT, topic)
    b = R.Brute(R.TENANT, topic)
    for pattern in R.CHAIN_PATTERNS:
        chain = R.chain_from_pattern(rng, pools, pattern)
        assert len(chain) == len(pattern)
        kept = b.lookup(chain)
        stop = pattern.find("S")
        want = [k for k, ch in enumerate(pattern) if (ch in "KN" and (stop < 0 or k < stop))]
        assert kept == want, (pattern, kept)
    assert "SN" in R.CHAIN_PATTERNS and "NS" in R.CHAIN_PATTERNS   # a stop on candidate 0 with no-Fact ranges behind it; and before
    assert any(p.endswith("S") and len(p) > 2 for p in R.CHAIN_PATTERNS)   # a stop on the last candidate
    assert any("S" in p[1:-1] for p in R.CHAIN_PATTERNS)   # a stop in the middle
    assert {"F", "L", "B"} <= set("".join(R.CHAIN_PATTERNS))


def test_real_route_set_filters_have_no_empty_levels():
    """so key order (NUL-joined) and level order agree on the ranges cut from them"""
    from bifromq_b200.workload import Workload
    w = Workload("C3", scale=0.0005)
    per = R.tenant_filters(w)
    assert len(per) >= 4
    for fs in per.values():
        assert all("" not in f for f in fs)
        assert sorted(fs, key=R.java_joined) == fs
        assert len(R.cut_ranges(fs, 64)) == min(64, len(fs))


def test_supplementary_plane_order_differs_between_utf8_and_utf16():
    """Out of scope: the MQTT edge rejects supplementary-plane text. U+1F600 sorts below U+FF5E in Java (surrogate 0xD83D <
    0xFF5E) but above it in UTF-8 bytes, so an order built on bytes and one built on UTF-16 code units part ways there."""
    a, b = "\U0001F600", "～"
    assert R.java_key([a]) < R.java_key([b])
    assert a.encode() > b.encode()
    cands = [(["tB", a], ["tB", b]), None]
    # in Java order seek finds tB/～, which is <= last: both ranges are kept (the oracle and the brute force agree)
    assert agree("tB", b, cands) == [0, 1]
    # in byte order every member of the topic sorts below the bound, so a byte-order walk stops and keeps nothing
    members = R.expansion_set("tB", b)
    assert all(tuple(x.encode() for x in m) < (b"tB", a.encode()) for m in members)
