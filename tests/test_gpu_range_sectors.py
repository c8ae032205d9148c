"""Tier 0 writes a topic's ranges one whole 32-byte sector (4 ranges) at a time: a lane holds the pending ranges of its current
sector in registers, writes the sector when its fourth range arrives, and writes the last, partial sector whole (padded) when the
topic finishes; a topic with more than 12 ranges moves them to a 64-range spill block. Two things can go wrong with that, and
each has a case here, checked in full against the oracle:

  * a range lost or duplicated at a sector edge, or a padded sector written over a neighbouring position's run: topics that
    match exactly 1, 3, 4, 5, 8, 9, ... ranges (every count at and around the sector edges, inline and in the spill block),
    neighbours in the batch holding different counts, in arrival and locality order, under both caps settings;
  * a spill block that does not start on a sector boundary. On the host path the cursor-allocated range region is cut into
    one slice per sub-batch; a workspace sized by an earlier, larger batch leaves a region whose quarter is not a multiple of 4
    ranges, and the slices are rounded down to whole spill blocks.
"""
import itertools
import random

import numpy as np
import pytest

from test_gpu_edges import (INLINE_RANGES, INT_MAX, PIPELINE_TOPICS, SPILL_RANGES, SPILL_REGION, SUB_BATCHES, both_orders,
                            check_host, kv_of, make_index, make_pairs, one_route_each, route_counts, spill_filters)

# every count from 1 to 20 (the inline sectors, the inline limit, the first two sectors of the spill block) and the spill
# block's last sector
SECTOR_COUNTS = list(range(1, 21)) + [61, 62, 63, 64]


def sector_counts_case(reps=3):
    """topic "s<n>_<k>/a/b/c/d/e/f" matches exactly n filters, each one route (so route count == matched filters), for n in
    SECTOR_COUNTS; `reps` topics per count, shuffled so that neighbouring positions hold different counts"""
    rest = list("abcdef")
    routes, topics = [], []
    for n in SECTOR_COUNTS:
        for k in range(reps):
            head = "s%d_%d" % (n, k)
            cands = ["/".join([head] + ["+" if c else x for c, x in zip(combo, rest)]) for combo in itertools.product([False, True], repeat=6)]
            cands += ["/".join([head] + rest[:j] + ["#"]) for j in range(len(rest) + 1)]
            random.Random(n * 31 + k).shuffle(cands)
            routes += one_route_each("sc", cands[:n])
            topics.append("/".join([head] + rest))
    order = list(range(len(topics)))
    random.Random(5).shuffle(order)
    topics = [topics[i] for i in order]
    return make_pairs(routes), ["sc"], topics, np.zeros(len(topics), np.int32)


def test_sector_counts_case_shape():
    pairs, tenants, topics, tt = sector_counts_case()
    n = route_counts(kv_of(pairs), tenants, topics, tt)
    want = [int(t.split("_")[0][1:]) for t in topics]
    assert n.tolist() == want
    assert max(want) == SPILL_RANGES and INLINE_RANGES + 1 in want
    assert sum(a == b for a, b in zip(want, want[1:])) < len(want) // 4   # mostly different counts side by side


@pytest.mark.gpu
def test_ranges_at_every_sector_edge():
    import bifromq_b200
    bifromq_b200.load_library()
    pairs, tenants, topics, tt = sector_counts_case()
    idx = make_index(bifromq_b200, pairs)
    for (order, caps), d in both_orders(idx, kv_of(pairs), tenants, topics, tt).items():
        assert d["deferred_topics"] == 0 and d["overflow_topics"] == 0, (order, caps, d)   # all in tier 0
    idx.close()


def unrounded_slice_case(n, seed):
    """n topics: every 64th takes a spill block (18 ranges), the others match 2 or 3 filters"""
    rng = random.Random(seed)
    topics = ["k%d/a/b/c/d" % i if i % 64 == 0 else "x%d/%s" % (i, rng.choice("yz")) for i in range(n)]
    rng.shuffle(topics)
    return topics


def test_unrounded_slice_case_shape():
    n1 = PIPELINE_TOPICS + 8193
    # the workspace of the first call holds n1 * 12 inline slots and a region of SPILL_REGION ranges behind them; the second
    # call, one topic shorter, sees 12 more ranges of region: a quarter of SPILL_REGION + 12 is 3 mod 4
    assert n1 < SPILL_REGION and (SPILL_REGION + 12) // SUB_BATCHES % 4 == 3
    topics = unrounded_slice_case(n1 - 1, 2)
    bounds = [(n1 - 1) * c // SUB_BATCHES for c in range(SUB_BATCHES + 1)]
    assert all(any(t.startswith("k") for t in topics[b:e]) for b, e in zip(bounds, bounds[1:]))


@pytest.mark.gpu
def test_spill_blocks_in_unrounded_host_slices():
    import bifromq_b200
    bifromq_b200.load_library()
    pairs = make_pairs(spill_filters("t") + [("t", "+/y", "p", 1)])
    kv = kv_of(pairs)
    idx = make_index(bifromq_b200, pairs)
    n1 = PIPELINE_TOPICS + 8193
    for n in (n1, n1 - 1):
        topics = unrounded_slice_case(n, n)
        tt = np.zeros(n, np.int32)
        for caps in ((INT_MAX, INT_MAX), (5, 2)):
            d, res = check_host(idx, kv, ["t"], topics, tt, caps)
            assert d["buffer_retries"] == 0, (n, caps, d)
            assert int(res.timings_ms["sub_batches"]) == SUB_BATCHES
            res.close()
    idx.close()
