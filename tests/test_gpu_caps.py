"""The fan-out caps against a per-tenant reference, at their flag, saturation and segment edges, on every match path.

MatchedRoutes (bifromq-dist-worker .../cache/MatchedRoutes.java:87-141) keeps, in KV order, the first maxPersistentFanout
persistent routes and the first maxGroupFanout group routes of a topic and reports every route it drops. The caps decide
who receives a message, so a slip drops or delivers routes without any error. They are per-tenant settings: one batch
carries a caps pair per tenant entry, and the decision is made or carried in several places — the tier-0 flag
(TENANT_CAPPED and finish()), the tier-1/2 pre-check, the followers pass of the de-dup, caps_kernel, expand_flagged_kernel
on the device path, the host merge in bfq_result_expand, and the cached tenant/caps table of a workspace.

`caps_reference` restates addNormalMatching / putGroupMatching literally and applies it, in KV order, to each topic's
uncapped route set (the oracle's brute-force answer at INT_MAX caps) with the caps of the topic's own tenant entry. Every
GPU test compares the whole answer with it: offsets, ranks (ascending per topic on the host path), throttle events and the
pre-cap route count. The tier-0 pre-check sums one saturating byte per matched range (255 = "255 or more"), so a topic is
flagged for the exact caps pass iff one of its caps is finite and either a byte of that kind is 255 or the bytes sum above
the cap; `flag_model` predicts the flagged_topics counter from that rule. CPU tests check the reference against the
oracle's own caps and check, on the oracle side, that every case has the route counts, range counts and levels it claims.
"""
import random
import threading
from collections import Counter

import numpy as np
import pytest

import oracle_lib as O
import test_gpu_edges as E
import test_gpu_fanout as F
import test_gpu_forward as FW

INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
NO_TENANT = E.NO_TENANT
NORMAL, PERSISTENT, GROUP = 0, 1, 2          # route kinds; PERSISTENT / GROUP are also the throttle-event kinds
BUILT_KIND = {"n": NORMAL, "p": PERSISTENT, "g": GROUP}


# ------------------------------------------------------------------ the reference (plain Python, no GPU)
class World:
    """one committed route set: sorted pairs (rank = position), the oracle KV, and per rank the kind the test built the
    route with and its target (the filter without a "$share/<group>/" prefix: one matched range per target)"""

    def __init__(self, pairs, kinds):
        self.pairs = sorted(pairs)
        self.kv = E.kv_of(self.pairs)
        self.kinds = np.array([kinds[k] for k, _ in self.pairs], np.int8)
        self.filters = [O.build_match_route(k, v)["mqttTopicFilter"] for k, v in self.pairs]
        self.targets = [f.split("/", 2)[2] if f.startswith(("$share/", "$oshare/")) else f for f in self.filters]


def build(routes):
    """routes as in test_gpu_edges.make_pairs -> (pairs, {key: kind}) with each route's kind taken from its tuple"""
    pairs, kinds = {}, {}
    for r in routes:
        for k, v in E.make_pairs([r]):
            pairs[k] = v
            kinds[k] = BUILT_KIND[r[2]]
    return sorted(pairs.items()), kinds


def decoded_kinds(pairs):
    """kinds of routes a generator built without recording them (random_pairs): decoded by the oracle's own decoder"""
    out = {}
    for k, v in pairs:
        m = O.build_match_route(k, v)
        out[k] = GROUP if m["type"] == "Group" else PERSISTENT if m["subBrokerId"] == 1 else NORMAL
    return out


def matched_routes(world, ranks, max_p, max_g):
    """MatchedRoutes.addNormalMatching / putGroupMatching over ranks in KV order -> (survivors, events (kind, rank, max),
    persistentFanout, groupFanout)"""
    all_matchings, group_matchings, events = set(), {}, []
    persistent_fanout = 0
    for r in ranks:
        if world.kinds[r] == GROUP:
            f = world.filters[r]
            if f not in group_matchings:
                group_matchings[f] = r
                if len(group_matchings) <= max_g:
                    all_matchings.add(r)
                else:
                    del group_matchings[f]
                    events.append((GROUP, r, max_g))
            else:
                all_matchings.discard(group_matchings[f])
                group_matchings[f] = r
                all_matchings.add(r)
        elif r not in all_matchings:
            all_matchings.add(r)
            if world.kinds[r] == PERSISTENT:
                if persistent_fanout < max_p:
                    persistent_fanout += 1
                else:
                    all_matchings.discard(r)
                    events.append((PERSISTENT, r, max_p))
    return sorted(all_matchings), events, persistent_fanout, len(group_matchings)


def sat8(v):
    return min(v, 255)


def flag_model(world, ranks, max_p, max_g):
    """the pre-check: one byte per matched range (its persistent / group count, 255 = 255 or more); flagged iff a cap is
    finite and a byte of its kind is 255 or the bytes sum above the cap (a negative cap counts as 0)"""
    pc, gc = Counter(), Counter()
    for r in ranks:
        t = world.targets[r]
        pc[t] += world.kinds[r] == PERSISTENT
        gc[t] += world.kinds[r] == GROUP
    flag = False
    for counts, cap in ((pc, max_p), (gc, max_g)):
        b = [sat8(c) for c in counts.values()]
        flag |= cap != INT_MAX and (255 in b or sum(b) > max(cap, 0))
    return flag


class CapsAnswer:
    pass


def caps_reference(world, tenants, topics, tt, max_p, max_g):
    """the reference answer of a batch whose tenant entries carry their own caps. A topic whose tenant index is outside
    [0, len(tenants)) matches nothing. Each distinct (entry, topic) pair is computed once."""
    nt = len(tenants)
    tt = np.asarray(tt, np.int64)
    keys = [(int(t) if 0 <= t < nt else -1, O._b(s)) for s, t in zip(topics, tt.tolist())]
    uniq = {}
    inv = [uniq.setdefault(k, len(uniq)) for k in keys]
    u = list(uniq)
    full = E.oracle_match(world.kv, tenants, [k[1] for k in u], [k[0] for k in u], INT_MAX, INT_MAX)
    per = []
    for j, (e, _) in enumerate(u):
        ranks = full.routes(j).tolist()
        mp, mg = (int(max_p[e]), int(max_g[e])) if e >= 0 else (INT_MAX, INT_MAX)
        surv, ev, pf, gf = matched_routes(world, ranks, mp, mg)
        n_ranges = len({world.targets[r] for r in ranks})
        per.append((surv, ev, pf, gf, len(ranks), flag_model(world, ranks, mp, mg), n_ranges))
    a = CapsAnswer()
    counts = np.array([len(per[j][0]) for j in inv], np.int64)
    a.offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    a.ranks = np.array([r for j in inv for r in per[j][0]], np.int64)
    a.events = sorted((k, i, r, m) for i, j in enumerate(inv) for k, r, m in per[j][1])
    a.persistent_fanout = [per[j][2] for j in inv]
    a.group_fanout = [per[j][3] for j in inv]
    a.route_count = [per[j][4] for j in inv]
    a.flagged = [per[j][5] for j in inv]
    a.n_ranges = [per[j][6] for j in inv]
    a.full = full
    a.inv = inv
    return a


def events3(events):
    return sorted((k, t, r) for k, t, r, _ in events)


# ------------------------------------------------------------------ cases
MIX_TENANTS = ["tA", "tB", "tC", "tD", "tE", "tF", "tG"]
MIX_TOPICS = ["s/x", "s/y", "q/x", "$sys/x", "k1/a/b/c/d", "k2/a/b/c/x", E.TIER2_TOPIC, E.TIER1_TOPIC, "none/z"]


def mix_routes(t):
    """the same filter set for every tenant: small fan-outs at tier 0 (root '#', '$sys/#'), a spill topic, a tier-1 topic
    (14 levels) and a tier-2 topic (263 ranges)"""
    r = [(t, "s/+", "p", 3), (t, "s/+", "n", 2), (t, "s/x", "p", 2), (t, "s/#", "g", 2), (t, "s/#", "p", 1), (t, "+/x", "g", 1),
         (t, "#", "p", 1), (t, "#", "g", 1), (t, "$sys/#", "p", 2), (t, "$sys/+", "g", 1)]
    r += E.spill_filters(t)
    r += E.one_route_each(t, E.TIER2_FILTERS)
    r += E.one_route_each(t, ["b/#", E.TIER1_TOPIC, "/".join(["b"] * 13 + ["+"])])
    return r


def counts_of(world, tenant, topic):
    """(persistent, group) routes the topic matches in the tenant, uncapped"""
    res = E.oracle_match(world.kv, [tenant], [topic], [0], INT_MAX, INT_MAX)
    k = world.kinds[res.routes(0)]
    return int((k == PERSISTENT).sum()), int((k == GROUP).sum())


def mix_entries(world):
    """(tenant, maxP, maxG) entries: uncapped, zero, negative, one cap finite, INT_MAX-1, caps exactly at a topic's
    counts, a tenant listed twice with different caps, an unknown tenant"""
    px, gx = counts_of(world, "tG", "s/x")
    p2, g2 = counts_of(world, "tG", E.TIER2_TOPIC)
    return [("tA", INT_MAX, INT_MAX), ("tB", 0, 0), ("tC", -1, -7), ("tD", 1, INT_MAX), ("tE", INT_MAX, 1),
            ("tF", INT_MAX - 1, INT_MAX - 1), ("tG", px, gx), ("tA", 2, 1), ("tG", p2, g2), ("tB", INT_MIN, 3),
            (NO_TENANT, 0, 0)]


def mix_batch(entries, reps=3):
    """topic i of the batch: entry i % len(entries) (and one out-of-range index), topic (i // n_entries) % len(topics): every
    32-topic chunk and every warp mixes capped and uncapped tenants"""
    ne = len(entries) + 1
    n = reps * ne * len(MIX_TOPICS)
    topics = [MIX_TOPICS[(i // ne) % len(MIX_TOPICS)] for i in range(n)]
    tt = np.array([(i % ne) if i % ne < len(entries) else -1 for i in range(n)], np.int32)
    return topics, tt


def split(entries):
    return [e[0] for e in entries], [e[1] for e in entries], [e[2] for e in entries]


MS_TOPIC = "m"


def boundary_routes():
    """per tier, topics whose caps cut at a range boundary, inside a range, inside the second segment of a multi-segment
    range, across a node's own range and its '#' range and on a tenant-root '#' ($ and non-$ topics)"""
    r = [("bd", "n/x/y", "p", 4), ("bd", "n/x/y", "g", 2), ("bd", "n/x/y", "n", 1), ("bd", "n/x/y/#", "p", 3), ("bd", "n/x/y/#", "g", 2),
         ("bd", "n/+/y", "p", 2), ("bd", "n/+/y", "g", 1), ("bd", "n/#", "p", 2), ("bd", "n/#", "g", 3), ("bd", "#", "p", 3),
         ("bd", "#", "g", 2), ("bd", "+/x/#", "p", 1), ("bd", "$sys/x/y", "p", 2), ("bd", "$sys/x/y", "g", 1), ("bd", "$sys/#", "p", 3),
         ("bd", "$sys/#", "g", 2), ("bd", "$sys/+/y", "n", 2)]
    # test_multi_segment_filter_interleaving's construction: the keys of "m//b" sort inside the bucket range of "m", so the
    # routes of "m" are two rank runs
    r += [("ms", "m", "p", 40), ("ms", "m", "n", 10), ("ms", "m", "g", 6), ("ms", "m//b", "p", 20), ("ms", "m/#", "p", 2)]
    r += [("sp", f, k, n) for f in [x[1] for x in E.spill_filters("sp")] for k, n in (("p", 2), ("g", 1), ("n", 1))]
    # the tier-limit topics of test_gpu_edges.ranges_case, every matched filter given two more persistent and group routes
    pairs, _, topics, _ = E.ranges_case()
    kv = E.kv_of(pairs)
    res = E.oracle_match(kv, ["rg"], topics, np.zeros(len(topics), np.int32), INT_MAX, INT_MAX)
    for i in range(len(topics)):
        for f in sorted(E.matched_filters(kv, res, i)):
            r += [("rg", f, "p", 2), ("rg", f, "g", 2)]
    r += E.one_route_each("rg", sorted({f for i in range(len(topics)) for f in E.matched_filters(kv, res, i)}))
    for n in SAT_COUNTS:
        r += [("sat", "s%d/x" % n, "p", n), ("sat", "g%d/x" % n, "g", n), ("sat", "/".join(["d%d" % n] + ["l"] * 13), "p", n),
              ("sat", "/".join(["d%d" % n] + ["l"] * 13), "g", n)]
    r += [("sat", "w/x", "p", 254), ("sat", "w/+", "p", 1), ("sat", "w/#", "g", 254), ("sat", "w/x/#", "g", 1)]
    return r


SAT_COUNTS = (254, 255, 256)
RG = ["r%d" % n for n in E.RANGE_COUNTS]
DEEP = ["d%d" % n for n in E.RANGE_COUNTS]
RG_TOPIC = {h: "/".join([h] + list("abcdef")) for h in RG}
RG_TOPIC.update({h: "/".join([h] + list("abcdefghijklm")) for h in DEEP})
TIERS = {
    "inline": [("bd", "n/x/y"), ("bd", "$sys/x/y"), ("bd", "q/x"), ("ms", MS_TOPIC), ("rg", RG_TOPIC["r11"]), ("rg", RG_TOPIC["r12"])],
    "spill": [("sp", "k1/a/b/c/d")] + [("rg", RG_TOPIC[h]) for h in ("r13", "r48", "r49", "r63", "r64")],
    "tier1": [("rg", RG_TOPIC[h]) for h in ("d11", "d12", "d13", "d48")],
    "tier2": [("rg", RG_TOPIC[h]) for h in ("d49", "d63", "d64", "d65", "r65")],
    "saturation": [("sat", t) for n in SAT_COUNTS for t in ("s%d/x" % n, "g%d/x" % n, "/".join(["d%d" % n] + ["l"] * 13))]
    + [("sat", "w/x")],
}


def cut_caps(world, ranks, kind):
    """caps that cut a topic's routes of one kind everywhere that matters: every count up to 48, else at and next to each
    change of range along KV order, and at c-1, c, c+1"""
    rk = [r for r in ranks if world.kinds[r] == kind]
    c = len(rk)
    if c <= 48:
        return set(range(-1, c + 2))
    out = {c - 1, c, c + 1, 0}
    for i in range(1, c):
        if world.targets[rk[i]] != world.targets[rk[i - 1]]:
            out |= {i - 1, i, i + 1}
    return out


def boundary_batch(world, tier):
    """one entry per (topic, caps) of the tier: c-1..c+1 x g-1..g+1, the persistent and the group cuts alone, and paired"""
    entries, topics, tt = [], [], []
    for tenant, topic in TIERS[tier]:
        res = E.oracle_match(world.kv, [tenant], [topic], [0], INT_MAX, INT_MAX)
        ranks = res.routes(0).tolist()
        k = world.kinds[ranks]
        c, g = int((k == PERSISTENT).sum()), int((k == GROUP).sum())
        if tier == "saturation":
            combos = {(x, INT_MAX) for x in range(253, 258)} | {(INT_MAX, x) for x in range(253, 258)}
            combos |= {(INT_MAX, INT_MAX), (0, INT_MAX), (INT_MAX - 1, 255)}
        else:
            pc, gcut = sorted(cut_caps(world, ranks, PERSISTENT)), sorted(cut_caps(world, ranks, GROUP))
            combos = {(a, b) for a in (c - 1, c, c + 1) for b in (g - 1, g, g + 1)}
            combos |= {(a, INT_MAX) for a in pc} | {(INT_MAX, b) for b in gcut}
            combos |= set(zip(pc, gcut[::-1]))
        for a, b in sorted(combos):
            topics.append(topic)
            tt.append(len(entries))
            entries.append((tenant, a, b))
    order = list(range(len(topics)))
    random.Random(len(order)).shuffle(order)
    return entries, [topics[i] for i in order], np.array([tt[i] for i in order], np.int32)


def levels(topic):
    return topic.count("/") + 1


def path_model(world, tenants, topics, tt, want):
    """(deferred, overflow) of tier 0 / tier 1 for a batch of known tenants: > 12 levels or > 64 ranges leave tier 0,
    > 48 of those leave tier 1"""
    deferred = overflow = 0
    for s, e, n in zip(topics, tt.tolist(), want.n_ranges):
        if 0 <= e < len(tenants) and n > 0 and (levels(s) > E.L_MAXLV or n > E.SPILL_RANGES):
            deferred += 1
            overflow += n > E.RG_CAP
    return deferred, overflow


# ------------------------------------------------------------------ module-wide route set (plain Python data)
_WORLD = {}


def world():
    if "w" not in _WORLD:
        routes = [r for t in MIX_TENANTS for r in mix_routes(t)] + boundary_routes()
        _WORLD["w"] = World(*build(routes))
    return _WORLD["w"]


# ------------------------------------------------------------------ CPU checks
class _Schema:
    """what test_gpu_forward.random_pairs needs of bifromq_b200.schema, from the oracle's encoders"""
    receiver_url = staticmethod(O.receiver_url)
    route_key = staticmethod(O.route_key)
    incarnation_bytes = staticmethod(O.incarnation_bytes)

    @staticmethod
    def route_group_bytes(members):
        return O.route_group(members)


class _NS:
    schema = _Schema


UNIFORM_CAPS = [INT_MAX, INT_MAX - 1, 256, 255, 1, 0, -1, INT_MIN]


@pytest.mark.parametrize("seed", [1, 2])
@pytest.mark.parametrize("cap", UNIFORM_CAPS)
def test_reference_equals_oracle_at_uniform_caps(seed, cap):
    pairs, tenants, topics, tt = FW.random_pairs(_NS, random.Random(seed), 600, ["a", "b", "c", "dd", "e1"], 5)
    w = World(pairs, decoded_kinds(pairs))
    for mp, mg in ((cap, cap), (cap, 2), (1, cap)):
        want = E.oracle_match(w.kv, tenants, topics, tt, mp, mg)
        got = caps_reference(w, tenants, topics, tt, [mp] * len(tenants), [mg] * len(tenants))
        assert got.offsets.tolist() == want.offsets.tolist()
        assert got.ranks.tolist() == want.ranks.tolist()
        assert got.events == want.events                    # maxCount included
        assert got.persistent_fanout == want.persistent_fanout.tolist() and got.group_fanout == want.group_fanout.tolist()
    assert sum(got.route_count) > 0


def test_built_kinds_match_the_decoded_routes():
    w = world()
    assert w.kinds.tolist() == [decoded_kinds([p])[p[0]] for p in w.pairs]


def test_mix_case_shape():
    w = world()
    entries = mix_entries(w)
    tenants, mp, mg = split(entries)
    topics, tt = mix_batch(entries)
    want = caps_reference(w, tenants, topics, tt, mp, mg)
    capped = [0 <= e < len(entries) and (mp[e] != INT_MAX or mg[e] != INT_MAX) for e in tt.tolist()]
    for c in range(0, len(topics), 32):
        assert 0 < sum(capped[c:c + 32]) < len(capped[c:c + 32])
    assert len(set(tenants)) < len(tenants) and NO_TENANT in tenants and (tt == -1).any()
    # caps exactly at a topic's counts: nothing dropped, yet every route of both kinds kept
    px, gx = counts_of(w, "tG", "s/x")
    assert px > 1 and gx > 1 and ("tG", px, gx) in entries
    assert len(want.events) > 0 and any(want.flagged) and not all(want.flagged)
    n_ranges = Counter()
    for s, n in zip(topics, want.n_ranges):
        n_ranges[s] = max(n_ranges[s], n)
    assert n_ranges[E.TIER2_TOPIC] > E.SPILL_RANGES and E.INLINE_RANGES < n_ranges["k1/a/b/c/d"] <= E.SPILL_RANGES


def test_boundary_cases_shape():
    w = world()
    for tier, items in TIERS.items():
        entries, topics, tt = boundary_batch(w, tier)
        tenants, mp, mg = split(entries)
        want = caps_reference(w, tenants, topics, tt, mp, mg)
        for s, n in zip(topics, want.n_ranges):
            lv = levels(s)
            if tier == "inline":
                assert lv <= E.L_MAXLV and n <= E.INLINE_RANGES, (s, n)
            elif tier == "spill":
                assert lv <= E.L_MAXLV and E.INLINE_RANGES < n <= E.SPILL_RANGES, (s, n)
            elif tier == "tier1":
                assert lv > E.L_MAXLV and n <= E.RG_CAP, (s, n)
            elif tier == "tier2":
                assert n > E.RG_CAP and (lv > E.L_MAXLV or n > E.SPILL_RANGES), (s, n)
        assert len(want.events) > 0 and any(want.flagged) and not all(want.flagged)
    # the ranges_case topics keep their range counts with the routes added to their filters
    tenants, topics, tt, mp, mg = _args(w, "spill")
    got = dict(zip(topics, caps_reference(w, tenants, topics, tt, mp, mg).n_ranges))
    assert got[RG_TOPIC["r64"]] == 64 and got[RG_TOPIC["r13"]] == 13
    # the tenant-root '#' is matched by the non-$ topic only, '$sys/#' by the $ topic
    res = E.oracle_match(w.kv, ["bd"], ["q/x", "$sys/x/y"], [0, 0], INT_MAX, INT_MAX)
    assert "#" in {w.targets[r] for r in res.routes(0)} and "#" not in {w.targets[r] for r in res.routes(1)}
    assert "$sys/#" in {w.targets[r] for r in res.routes(1)}
    # a node's own range and its '#' range are both matched by "n/x/y"
    res = E.oracle_match(w.kv, ["bd"], ["n/x/y"], [0], INT_MAX, INT_MAX)
    assert {"n/x/y", "n/x/y/#"} <= {w.targets[r] for r in res.routes(0)}


def _args(w, tier):
    entries, topics, tt = boundary_batch(w, tier)
    tenants, mp, mg = split(entries)
    return tenants, topics, tt, mp, mg


def test_multi_segment_cut_lands_in_the_second_segment():
    """the routes of "m" are two rank runs, the second with persistent routes: some cap of the inline batch cuts in it"""
    w = world()
    res = E.oracle_match(w.kv, ["ms"], [MS_TOPIC], [0], INT_MAX, INT_MAX)
    own = [r for r in res.routes(0).tolist() if w.targets[r] == "m"]
    runs = np.split(np.array(own), np.where(np.diff(own) != 1)[0] + 1)
    assert len(runs) >= 2
    persistent = [r for r in res.routes(0).tolist() if w.kinds[r] == PERSISTENT]
    first_run_p = sum(1 for r in runs[0] if w.kinds[r] == PERSISTENT)
    second_run_p = sum(1 for r in runs[1] if w.kinds[r] == PERSISTENT)
    assert second_run_p >= 2
    # a cap of first_run_p + 1 keeps one persistent route of the second run and drops the next one
    assert persistent.index(int(next(r for r in runs[1] if w.kinds[r] == PERSISTENT))) >= first_run_p
    caps = {e[1] for e in boundary_batch(w, "inline")[0] if e[0] == "ms"}
    assert first_run_p + 1 in caps


def test_saturation_case_shape():
    w = world()
    for n in SAT_COUNTS:
        assert counts_of(w, "sat", "s%d/x" % n) == (n, 0)
        assert counts_of(w, "sat", "g%d/x" % n) == (0, n)
        assert counts_of(w, "sat", "/".join(["d%d" % n] + ["l"] * 13)) == (n, n)
    assert counts_of(w, "sat", "w/x") == (255, 255)   # bytes 254 + 1: the sum reaches the caps without a saturated byte
    tenants, topics, tt, mp, mg = _args(w, "saturation")
    want = caps_reference(w, tenants, topics, tt, mp, mg)
    # with INT_MAX caps nothing is flagged, saturated bytes or not
    assert not any(f for f, e in zip(want.flagged, tt.tolist()) if (mp[e], mg[e]) == (INT_MAX, INT_MAX))
    assert any(want.flagged) and len(want.events) > 0


def test_flag_model_examples():
    w = world()
    res = E.oracle_match(w.kv, ["sat"], ["s254/x", "s255/x", "w/x"], [0, 0, 0], INT_MAX, INT_MAX)
    r254, r255, rw = (res.routes(i).tolist() for i in range(3))
    assert not flag_model(w, r254, 254, INT_MAX) and flag_model(w, r254, 253, INT_MAX)
    assert flag_model(w, r255, 1000, INT_MAX) and not flag_model(w, r255, INT_MAX, 0)
    assert not flag_model(w, rw, 255, INT_MAX) and flag_model(w, rw, 254, INT_MAX) and flag_model(w, rw, -1, INT_MAX)


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


@pytest.fixture(scope="module")
def IDX(B):
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(world().pairs)
    idx.commit()
    yield idx
    idx.close()


def check_host(idx, w, tenants, topics, tt, mp, mg):
    """bfq_match with per-entry caps vs caps_reference: offsets, ranks (ascending per topic), events, pre-cap route counts
    -> (stats delta, reference)"""
    before = idx.stats()
    res = idx.match_topics(tenants, topics, np.ascontiguousarray(tt, np.int32), mp, mg)
    d = E.delta(idx, before)
    offsets, ranks = res.expand()
    want = caps_reference(w, tenants, topics, tt, mp, mg)
    assert offsets.tolist() == want.offsets.tolist()
    seg = np.repeat(np.arange(len(topics)), np.diff(offsets))
    assert (np.diff(ranks)[seg[1:] == seg[:-1]] > 0).all()      # ascending per topic
    assert ranks.tolist() == want.ranks.tolist()
    assert sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist()) == events3(want.events)
    assert res.route_count.tolist() == want.route_count
    subs = int(res.timings_ms["sub_batches"])
    res.close()
    return d, want, subs


def match_device(B, idx, tenants, topics, tt, mp, mg, wait=True):
    torch = B.torch
    blob, off = O.blob(topics)
    keep = [torch.from_numpy(blob).to(B.dev), torch.from_numpy(off).to(B.dev),
            torch.from_numpy(np.ascontiguousarray(tt, np.int32)).to(B.dev)]
    out = idx.match_device(tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), len(topics), mp, mg, B.stream, wait)
    out.keep = keep
    return out


def read_device(B, out, n, want):
    """bfq_expand_device of a completed device match vs a reference: offsets, per-topic rank sets, events, route counts"""
    d_offsets, d_ranks, total = F.device_csr(B, out, n)
    rc = B.dist.device_view(out.d_route_count, max(n, 1), "<u4", B.dev).cpu().numpy()[:n].astype(np.int64)
    thr = B.dist.device_view(out.d_throttled, max(3 * out.n_throttled, 1), "<u4", B.dev).cpu().numpy()[:3 * out.n_throttled]
    B.torch.cuda.synchronize()
    offsets = d_offsets.cpu().numpy()
    ranks = d_ranks.cpu().numpy()[:total]
    assert offsets.tolist() == want.offsets.tolist()
    seg = np.repeat(np.arange(n), np.diff(offsets))
    assert ranks[np.lexsort((ranks, seg))].tolist() == want.ranks.tolist()
    assert sorted((int(k), int(t), int(r)) for t, r, k in thr.reshape(-1, 3).tolist()) == events3(want.events)
    assert rc.tolist() == want.route_count
    return d_offsets, d_ranks, total


def check_device(B, idx, w, tenants, topics, tt, mp, mg):
    before = idx.stats()
    out = match_device(B, idx, tenants, topics, tt, mp, mg)
    d = E.delta(idx, before)
    want = caps_reference(w, tenants, topics, tt, mp, mg)
    read_device(B, out, len(topics), want)
    out.release()
    return d, want


def set_order(idx, order):
    idx.set_option("order_min_topics", 0 if order == "arrival" else 1)


ORDERS = ["arrival", "locality"]


# ------------------------------------------------------------------ per-tenant caps in one batch
@pytest.mark.gpu
@pytest.mark.parametrize("order", ORDERS)
def test_per_tenant_caps_host_and_device(B, IDX, order):
    w = world()
    entries = mix_entries(w)
    tenants, mp, mg = split(entries)
    topics, tt = mix_batch(entries)
    set_order(IDX, order)
    try:
        d, want, _ = check_host(IDX, w, tenants, topics, tt, mp, mg)
        assert d["flagged_topics"] == sum(want.flagged), d
        assert d["duplicate_topics"] == (E.true_repeats(tenants, topics, tt) if order == "locality" else 0)
        d, want = check_device(B, IDX, w, tenants, topics, tt, mp, mg)
        assert d["flagged_topics"] == sum(want.flagged), d
    finally:
        IDX.set_option("order_min_topics", 32768)


@pytest.mark.gpu
def test_per_tenant_caps_pipelined_host_path(B, IDX):
    """>= 2^17 topics: four sub-batches; throttle events carry global topic indices"""
    w = world()
    entries = mix_entries(w)
    tenants, mp, mg = split(entries)
    per = (len(entries) + 1) * len(MIX_TOPICS)
    topics, tt = mix_batch(entries, reps=(E.PIPELINE_TOPICS + 4096) // per + 1)
    assert len(topics) >= E.PIPELINE_TOPICS
    # a fresh workspace's throttle list is too small for this batch: the first call is redone un-chunked with grown
    # buffers, the second runs the pipeline
    for rep in range(2):
        d, want, subs = check_host(IDX, w, tenants, topics, tt, mp, mg)
        assert d["flagged_topics"] == sum(want.flagged), d
    assert subs == E.SUB_BATCHES
    assert len(want.events) > E.THROTTLE_LIST and max(t for _, t, _, _ in want.events) > 3 * len(topics) // 4


@pytest.mark.gpu
def test_per_tenant_caps_fanout(B, IDX):
    """bfq_fanout_device groups the reference's survivors, and nothing else"""
    w = world()
    entries = mix_entries(w)
    tenants, mp, mg = split(entries)
    topics, tt = mix_batch(entries)
    want = caps_reference(w, tenants, topics, tt, mp, mg)
    out = match_device(B, IDX, tenants, topics, tt, mp, mg)
    read_device(B, out, len(topics), want)
    got, s = F.fan_check(B, IDX, out, topics, want, w.pairs)
    assert got["n_pairs"] == len(want.ranks) and s["normal"] > 0 and s["share"] > 0
    out.release()


# ------------------------------------------------------------------ boundaries in each tier
@pytest.mark.gpu
@pytest.mark.parametrize("tier", list(TIERS))
def test_caps_at_boundaries(B, IDX, tier):
    w = world()
    entries, topics, tt = boundary_batch(w, tier)
    tenants, mp, mg = split(entries)
    try:
        for order in ORDERS:
            set_order(IDX, order)
            d, want, _ = check_host(IDX, w, tenants, topics, tt, mp, mg)
            deferred, overflow = path_model(w, tenants, topics, tt, want)
            assert (d["deferred_topics"], d["overflow_topics"], d["duplicate_topics"]) == (deferred, overflow, 0), (order, d)
            assert d["flagged_topics"] == sum(want.flagged), (order, d)
            d, want = check_device(B, IDX, w, tenants, topics, tt, mp, mg)
            assert (d["deferred_topics"], d["overflow_topics"], d["flagged_topics"]) == (deferred, overflow, sum(want.flagged)), (order, d)
    finally:
        IDX.set_option("order_min_topics", 32768)
    if tier == "saturation":
        assert deferred > 0 and sum(want.flagged) > 0


# ------------------------------------------------------------------ the workspace's cached caps table
@pytest.mark.gpu
def test_caps_table_cache_on_repeated_calls(B, IDX):
    w = world()
    entries = mix_entries(w)
    tenants, mp_a, mg_a = split(entries)
    mp_b, mg_b = mp_a[::-1], mg_a[1:] + mg_a[:1]
    topics, tt = mix_batch(entries)
    # A, B, A, then only the group caps changed, then A again
    for mp, mg in ((mp_a, mg_a), (mp_b, mg_b), (mp_a, mg_a), (mp_a, mg_b), (mp_a, mg_a)):
        check_host(IDX, w, tenants, topics, tt, mp, mg)
        check_device(B, IDX, w, tenants, topics, tt, mp, mg)
    # the same caps, the tenant list permuted (topics follow their tenant)
    perm = list(range(len(entries)))
    random.Random(3).shuffle(perm)
    inv = np.argsort(perm)
    p_entries = [entries[i] for i in perm]
    ptt = np.array([inv[e] if e >= 0 else e for e in tt.tolist()], np.int32)
    pt, pmp, pmg = split(p_entries)
    check_host(IDX, w, pt, topics, ptt, pmp, pmg)
    check_host(IDX, w, tenants, topics, tt, mp_a, mg_a)


@pytest.mark.gpu
def test_caps_table_after_commit_shifting_root_ordinals(B):
    """the same tenant list and caps after a delta commit that adds a tenant sorting first (every root ordinal moves)"""
    routes = [r for t in MIX_TENANTS[:4] for r in mix_routes(t)]
    pairs, kinds = build(routes)
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(pairs)
    idx.commit()
    w = World(pairs, kinds)
    entries = [e for e in mix_entries(w) if e[0] in MIX_TENANTS[:4] + [NO_TENANT]]
    tenants, mp, mg = split(entries)
    topics, tt = mix_batch(entries)
    check_host(idx, w, tenants, topics, tt, mp, mg)
    check_device(B, idx, w, tenants, topics, tt, mp, mg)
    extra, extra_kinds = build(mix_routes("0"))      # tenant "0" sorts before every "tX"
    before = idx.stats()
    idx.apply(adds=extra)
    idx.commit()
    assert idx.stats()["delta_commits"] == before["delta_commits"] + 1
    w2 = World(pairs + extra, {**kinds, **extra_kinds})
    check_host(idx, w2, tenants, topics, tt, mp, mg)
    check_device(B, idx, w2, tenants, topics, tt, mp, mg)
    # and the new tenant in the list, capped, before the others
    entries2 = [("0", 1, 0)] + entries
    t2, mp2, mg2 = split(entries2)
    check_host(idx, w2, t2, topics, np.where(tt >= 0, tt + 1, tt).astype(np.int32), mp2, mg2)
    idx.close()


@pytest.mark.gpu
def test_caps_table_six_threads_share_one_tenant_list(B, IDX):
    w = world()
    entries = mix_entries(w)
    tenants, mp0, mg0 = split(entries)
    topics, tt = mix_batch(entries)
    T = 6
    caps = [([max(-1, p - k) if p < INT_MAX - 1 else p for p in mp0], [g if k % 2 else min(g, k) for g in mg0]) for k in range(T)]
    want = {k: caps_reference(w, tenants, topics, tt, *caps[k]) for k in range(T)}
    got, errs = {}, []
    barrier = threading.Barrier(T)

    def worker(k):
        try:
            for rep in range(3):
                barrier.wait()
                res = IDX.match_topics(tenants, topics, tt, *caps[k])
                barrier.wait()
                offsets, ranks = res.expand()
                ev = sorted((int(kk), int(t), int(r)) for t, r, kk in res.throttled.tolist())
                got[(k, rep)] = (offsets.tolist(), ranks.tolist(), ev)
                res.close()
        except Exception as e:   # pragma: no cover
            errs.append(e)
            barrier.abort()
    th = [threading.Thread(target=worker, args=(k,)) for k in range(T)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs
    assert len(got) == 3 * T
    assert len({tuple(v[1]) for v in got.values()}) > 1
    for (k, rep), (offsets, ranks, ev) in got.items():
        assert offsets == want[k].offsets.tolist() and ranks == want[k].ranks.tolist() and ev == events3(want[k].events), (k, rep)


# ------------------------------------------------------------------ caps across delta commits
@pytest.mark.gpu
def test_caps_across_delta_commits_that_shift_later_tenants(B):
    """adding and removing persistent and group routes of the first tenant shifts every later tenant's ranks and prefix
    counts; the later tenants' caps still cut at the same routes. A device match enqueued before the commit and expanded
    after it answers from the snapshot it started on."""
    routes = [r for t in MIX_TENANTS[:5] for r in mix_routes(t)]
    pairs, kinds = build(routes)
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(pairs)
    idx.commit()
    w = World(pairs, kinds)
    entries = [e for e in mix_entries(w) if e[0] in MIX_TENANTS[:5] + [NO_TENANT]]
    tenants, mp, mg = split(entries)
    topics, tt = mix_batch(entries)
    _, want_old, _ = check_host(idx, w, tenants, topics, tt, mp, mg)
    live = dict(pairs)
    for rnd, (add, drop_kind) in enumerate([([("tA", "s/+", "p", 9), ("tA", "s/#", "g", 7)], None),
                                             ([("tA", "+/x", "g", 5)], PERSISTENT), ([], GROUP)]):
        extra, extra_kinds = build(add)
        kinds.update(extra_kinds)
        cur = World(sorted(live.items()), kinds)
        dels = [k for i, (k, _) in enumerate(cur.pairs) if drop_kind is not None and cur.kinds[i] == drop_kind
                and k.startswith(O.tenant_begin_key("tA")) and i % 3 == 0]
        pending = match_device(B, idx, tenants, topics, tt, mp, mg, wait=False)
        idx.apply(adds=extra, dels=dels)
        idx.commit()
        pending.wait()
        read_device(B, pending, len(topics), caps_reference(cur, tenants, topics, tt, mp, mg))
        pending.release()
        for k, v in extra:
            live[k] = v
        for k in dels:
            del live[k]
        new = World(sorted(live.items()), kinds)
        d, want, _ = check_host(idx, new, tenants, topics, tt, mp, mg)
        check_device(B, idx, new, tenants, topics, tt, mp, mg)
        # the later tenants keep the same routes (by key), at shifted ranks
        first = O.tenant_begin_key("tA")
        for i, e in enumerate(tt.tolist()):
            if e >= 0 and tenants[e] not in ("tA", NO_TENANT):
                a = [w.pairs[r][0] for r in want_old.ranks[want_old.offsets[i]:want_old.offsets[i + 1]]]
                b = [new.pairs[r][0] for r in want.ranks[want.offsets[i]:want.offsets[i + 1]]]
                assert a == b and not any(k.startswith(first) for k in b)
    idx.close()


# ------------------------------------------------------------------ the host mirror
@pytest.mark.gpu
def test_host_mirror_fanouts_and_event_max_count(B, IDX):
    w = world()
    for tenant, mp, mg in mix_entries(w):
        events = []
        m = B.pkg.GpuTenantRouteMatcher(tenant, IDX, events.append)
        got = m.match_all(MIX_TOPICS, mp, mg)
        want = caps_reference(w, [tenant], MIX_TOPICS, np.zeros(len(MIX_TOPICS), np.int32), [mp], [mg])
        for i, topic in enumerate(MIX_TOPICS):
            r = got[topic]
            assert (r.persistent_fanout(), r.group_fanout()) == (want.persistent_fanout[i], want.group_fanout[i]), (tenant, topic)
            assert (r.max_persistent_fanout(), r.max_group_fanout()) == (mp, mg)
            assert len(r.routes()) == want.offsets[i + 1] - want.offsets[i]
        want_ev = sorted((k, MIX_TOPICS[t], w.filters[rank], mx) for k, t, rank, mx in want.events)
        got_ev = sorted((PERSISTENT if isinstance(e, B.pkg.PersistentFanoutThrottled) else GROUP, e.topic, e.mqtt_topic_filter,
                         e.max_count) for e in events)
        assert got_ev == want_ev and all(e.tenant_id == tenant for e in events)
