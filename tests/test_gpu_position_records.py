"""Tier 0's span records by work-order position, gathered back to topic order by finalize_kernel.

In an ordered batch tier 0 writes each topic's {span_begin, span_count, route_count} as one record at the topic's position in
the locality order, and finalize_kernel maps the records back to topic indices: a leader takes its own record, a repeat its
leader's, a topic tier 0 deferred keeps what tier 1 (or tier 2) wrote. A slip in that mapping gives a topic another topic's
routes without any error. Every test here checks the whole answer against the CPU oracle (offsets, ranks, throttle events,
pre-cap route counts) in arrival order, in locality order with de-dup, and in locality order without de-dup, on the device
and the host path (one batch, and the host path's 4-sub-batch pipeline), and asserts through idx.stats() which path ran.

The batch mixes every kind of topic a record can describe: topics that spill past the 12 inline ranges, topics tier 0 defers
to tier 1 and tier 1 to tier 2, topics flagged for the caps, topics of a tenant without routes and of out-of-range tenant
indices, each repeated, in shuffled order.
"""
import random

import numpy as np
import pytest

import oracle_lib as O
from test_gpu_edges import (CAPS, INLINE_RANGES, INT_MAX, PIPELINE_TOPICS, SUB_BATCHES, TIER1_TOPIC, TIER2_TOPIC,
                            check_device, delta, events_of, kv_of, make_index, make_pairs, one_route_each, oracle_match,
                            spill_filters, tier2_case, true_repeats)

TENANTS = ["sp", "t", "empty"]   # spill topics and fillers / tier 1 and tier 2 topics / no routes at all
MODES = ["arrival", "locality", "locality-nodedup"]
SPILL_TOPICS = 48                # "k<i>/a/b/c/d": 18 ranges each in tenant "sp" (a spill block in tier 0)


def mixed_routes():
    routes = spill_filters("sp") + one_route_each("sp", ["+/x", "f/+/z"])
    routes += tier2_case()[0]
    return make_pairs(routes)


def mixed_batch(n_fill=300, seed=23):
    """-> topics, tenant indices. A filler pair appears 1-4 times, every other pair 2-4 times."""
    rng = random.Random(seed)
    fill = [("k%d/x" % i, 0) for i in range(n_fill)]                                # 3 ranges: inline slots only
    fill += [("f/%d/z" % i, 0) for i in range(n_fill // 4)]
    entries = [("k%d/a/b/c/d" % i, 0) for i in range(SPILL_TOPICS)]
    entries += [(TIER2_TOPIC, 1), (TIER1_TOPIC, 1), ("b/b", 1), ("a/a", 1), ("c/d", 1)]
    entries += [(s, t) for s in ("k1/a/b/c/d", TIER2_TOPIC, "k2/x", "", "/") for t in (2, -1, 7)]   # nothing to match
    entries += [("", 0), ("/", 0), ("k3/a/b/c/d", 1)]
    batch = []
    for e in fill:
        batch += [e] * rng.choice([1, 2, 2, 4])
    for e in entries:
        batch += [e] * rng.choice([2, 3, 4])
    rng.shuffle(batch)
    return [s for s, _ in batch], np.array([t for _, t in batch], np.int32)


def deferred_pairs(topics, tt, distinct):
    """topics tier 0 hands to tier 1 (tenant "t": 14 levels, or more than 64 ranges), and of those tier 1 hands to tier 2"""
    d1 = [(s, t) for s, t in zip(topics, tt.tolist()) if t == 1 and s in (TIER1_TOPIC, TIER2_TOPIC)]
    d2 = [p for p in d1 if p[0] == TIER2_TOPIC]
    return (len(set(d1)), len(set(d2))) if distinct else (len(d1), len(d2))


def set_mode(idx, mode):
    idx.set_option("order_min_topics", 0 if mode == "arrival" else 1)
    idx.set_option("dedup", 0 if mode == "locality-nodedup" else 1)


def reset_mode(idx):
    idx.set_option("order_min_topics", 32768)
    idx.set_option("dedup", 1)


def want_of(kv, topics, tt, caps):
    want = oracle_match(kv, TENANTS, topics, tt, caps[0], caps[1], O.MODE_TRIE)
    uncapped = oracle_match(kv, TENANTS, topics, tt, INT_MAX, INT_MAX, O.MODE_TRIE) if caps != (INT_MAX, INT_MAX) else want
    return want, np.diff(uncapped.offsets).tolist()


def check_host(idx, topics, tt, caps, want, want_rc):
    """bfq_match vs the oracle's (precomputed) answer, exactly -> (stats delta, sub-batches)"""
    before = idx.stats()
    res = idx.match_topics(TENANTS, topics, tt, [caps[0]] * len(TENANTS), [caps[1]] * len(TENANTS))
    d = delta(idx, before)
    offsets, ranks = res.expand()
    assert offsets.tolist() == want.offsets.tolist()
    assert ranks.tolist() == want.ranks.tolist()
    assert sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist()) == events_of(want)
    assert res.route_count.tolist() == want_rc
    subs = int(res.timings_ms["sub_batches"])
    res.close()
    return d, subs


def expected_stats(mode, topics, tt, per_sub=None):
    dedup = mode == "locality"
    n1, n2 = deferred_pairs(topics, tt, dedup)
    if dedup and per_sub:   # each sub-batch is ordered and de-duplicated on its own
        n1 = n2 = dup = 0
        for b, e in per_sub:
            a1, a2 = deferred_pairs(topics[b:e], tt[b:e], True)
            n1, n2, dup = n1 + a1, n2 + a2, dup + true_repeats(TENANTS, topics[b:e], tt[b:e])
    else:
        dup = true_repeats(TENANTS, topics, tt) if dedup else 0
    return {"deferred_topics": n1, "overflow_topics": n2, "duplicate_topics": dup, "buffer_retries": 0}


# ------------------------------------------------------------------ CPU check of the batch (oracle side only)
def test_mixed_batch_shape():
    topics, tt = mixed_batch()
    kv = kv_of(mixed_routes())
    n = np.diff(oracle_match(kv, TENANTS, topics, tt, INT_MAX, INT_MAX).offsets)
    nt = len(TENANTS)
    rep = {}
    for s, t, c in zip(topics, tt.tolist(), n.tolist()):
        key = (t if 0 <= t < nt else -1, s)
        rep.setdefault(key, []).append(c)
    # every kind of topic repeats: spill (> 12 ranges), tier 1 and tier 2, no routes, out-of-range tenant
    assert any(len(v) > 1 and v[0] > INLINE_RANGES for (t, s), v in rep.items() if t == 0 and s.endswith("/a/b/c/d"))
    assert len(rep[(1, TIER1_TOPIC)]) > 1 and len(rep[(1, TIER2_TOPIC)]) > 1 and rep[(1, TIER2_TOPIC)][0] == 263
    assert len(rep[(2, TIER2_TOPIC)]) > 1 and rep[(2, TIER2_TOPIC)][0] == 0
    assert len(rep[(-1, TIER2_TOPIC)]) > 1 and rep[(-1, TIER2_TOPIC)][0] == 0
    assert (tt < 0).any() and (tt >= nt).any()
    # the caps flag repeated topics: 6 persistent and 6 group routes of 18 against (5, 2)
    capped = oracle_match(kv, TENANTS, ["k1/a/b/c/d"], [0], 5, 2)
    assert len(capped.events) == 1 + 4


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def B():
    import bifromq_b200
    bifromq_b200.load_library()
    return bifromq_b200


@pytest.mark.gpu
def test_records_one_batch_host_and_device(B):
    pairs = mixed_routes()
    kv = kv_of(pairs)
    topics, tt = mixed_batch()
    idx = make_index(B, pairs)
    flagged = {}
    for caps in CAPS:
        want, want_rc = want_of(kv, topics, tt, caps)
        for mode in MODES:
            set_mode(idx, mode)
            exp = expected_stats(mode, topics, tt)
            d, subs = check_host(idx, topics, tt, caps, want, want_rc)
            assert subs == 1
            flagged[(caps, mode, "host")] = d.pop("flagged_topics")
            assert d == exp, (caps, mode, d, exp)
            d = check_device(idx, kv, TENANTS, topics, tt, caps, O.MODE_TRIE)
            flagged[(caps, mode, "device")] = d.pop("flagged_topics")
            assert d == exp, (caps, mode, d, exp)
        # every flagged topic joins the caps list exactly once, whichever pass put it there
        got = {k: v for k, v in flagged.items() if k[0] == caps}
        assert len(set(got.values())) == 1, got
        assert (next(iter(got.values())) > 0) == (caps != (INT_MAX, INT_MAX)), got
    reset_mode(idx)
    idx.close()


@pytest.mark.gpu
def test_records_host_pipeline_sub_batches(B):
    """>= 2^17 topics: the host path's 4-sub-batch pipeline, each sub-batch ordered on its own (its records and order
    positions are relative to the sub-batch)"""
    pairs = mixed_routes()
    kv = kv_of(pairs)
    topics, tt = mixed_batch(n_fill=PIPELINE_TOPICS // 2, seed=29)
    n = len(topics)
    assert n >= PIPELINE_TOPICS + 8192
    bounds = [n * c // SUB_BATCHES for c in range(SUB_BATCHES + 1)]
    per_sub = list(zip(bounds, bounds[1:]))
    idx = make_index(B, pairs)
    for caps in CAPS:
        want, want_rc = want_of(kv, topics, tt, caps)
        flagged = set()
        for mode in MODES:
            set_mode(idx, mode)
            d, subs = check_host(idx, topics, tt, caps, want, want_rc)
            assert subs == SUB_BATCHES
            flagged.add(d.pop("flagged_topics"))
            exp = expected_stats(mode, topics, tt, per_sub)
            assert d == exp, (caps, mode, d, exp)
        assert len(flagged) == 1, flagged
    reset_mode(idx)
    idx.close()
