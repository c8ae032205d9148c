"""De-duplication and locality order on batches dominated by a few (tenant, topic) pairs.

A popular topic can make up much of a publish batch: every one of its copies probes the same slot of the de-dup table and
must end up with a leader whose tenant and bytes equal its own. These batches put half of all topics on one pair and
thousands on a few others, next to the same bytes under another tenant and near-twins that differ in one byte, and check
every topic's answer against the CPU oracle on the host and the device path, and the `duplicate_topics` stat against the
true repeat count: with the full hash, with 8 hash bits and with none (every pair then shares one tag, so every leader is
found by the byte compare), and with order_min_topics 1 on a small batch.
"""
import random

import numpy as np
import pytest

from test_gpu_edges import B, INT_MAX, check_device, check_host, kv_of, make_index, make_pairs, one_route_each, true_repeats  # noqa: F401

HOT = "plant/7/line/3/sensor/temperature"


def hot_case(n_topics, seed=5):
    """half the batch one pair (tenant tA, HOT); three pairs of n/12 copies each (one of them HOT under tenant tB, one a
    near-twin of HOT that differs in its last byte); 200 pairs of 1-4 copies; the rest distinct topics. Shuffled."""
    rng = random.Random(seed)
    batch = [(HOT, 0)] * (n_topics // 2)
    twin = HOT[:-1] + "X"
    for s, t in ((HOT, 1), (twin, 0), ("plant/7/line/4/sensor/temperature", 0)):
        batch += [(s, t)] * (n_topics // 12)
    for i in range(200):
        batch += [("plant/%d/line/%d/sensor/p%d" % (i % 9, i, i), rng.randrange(3))] * rng.choice([1, 2, 4])
    i = 0
    while len(batch) < n_topics:
        batch.append(("r/%06d/" % i + "y" * rng.randint(0, 50), rng.randrange(3)))
        i += 1
    rng.shuffle(batch)
    topics = [s for s, _ in batch]
    tt = np.array([t for _, t in batch], np.int32)
    tenants = ["tA", "tB", "tC"]
    fs = [HOT, twin, "plant/+/line/+/sensor/#", "plant/7/#", "r/+/+"]
    routes = (one_route_each("tA", fs) + one_route_each("tB", [HOT, "plant/7/line/+/sensor/temperature"]) +
              [("tC", "#", "p", 2)])
    return make_pairs(routes), tenants, topics, tt


def test_hot_case_shape():
    _, tenants, topics, tt = hot_case(32768)
    assert len(topics) == 32768
    pairs = {}
    for s, t in zip(topics, tt.tolist()):
        pairs[(t, s)] = pairs.get((t, s), 0) + 1
    counts = sorted(pairs.values(), reverse=True)
    assert counts[0] == 16384 and counts[1:4] == [2730] * 3 and counts[4] <= 4
    assert true_repeats(tenants, topics, tt) == len(topics) - len(pairs)


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [64, 8, 0])
def test_hot_pairs_full_batch(B, bits):
    """a 40 000-topic batch: ordered by default (>= 32 768 topics), de-duplicated under the given hash bits"""
    pairs, tenants, topics, tt = hot_case(40000)
    idx = make_index(B, pairs)
    kv = kv_of(pairs)
    idx.set_option("dedup_hash_bits", bits)
    rep = true_repeats(tenants, topics, tt)
    for caps in [(INT_MAX, INT_MAX), (1, 0)]:
        d, res = check_host(idx, kv, tenants, topics, tt, caps)
        res.close()
        assert d["duplicate_topics"] == rep, (caps, d)
    d = check_device(idx, kv, tenants, topics, tt, (INT_MAX, INT_MAX))
    assert d["duplicate_topics"] == rep, d
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [64, 0])
def test_hot_pairs_small_batch_ordered(B, bits):
    """the same shape at 600 topics with order_min_topics 1, so a batch far below the default threshold is ordered"""
    pairs, tenants, topics, tt = hot_case(600, seed=9)
    idx = make_index(B, pairs)
    kv = kv_of(pairs)
    idx.set_option("order_min_topics", 1)
    idx.set_option("dedup_hash_bits", bits)
    rep = true_repeats(tenants, topics, tt)
    d, res = check_host(idx, kv, tenants, topics, tt, (INT_MAX, INT_MAX))
    res.close()
    assert d["duplicate_topics"] == rep, d
    d = check_device(idx, kv, tenants, topics, tt, (2, 1))
    assert d["duplicate_topics"] == rep, d
    idx.close()
