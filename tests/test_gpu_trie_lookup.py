"""The forward trie's child lookups at their hash edges, on the GPU: tier 0's find_child_lanes and tiers 1 and 2's
find_child / probe on keys placed from the model of the tag table (tests/trie_hash.py) — full home blocks, chains of 2 and 3
blocks, a chain that wraps from the last block to block 0, 4 keys with one fingerprint in one block, absent names with a
present key's block and fingerprint, a name with one block and fingerprint under two tenant roots, 24-byte length twins, fold
pairs that make nodes wide below the root, single-child twins. Every answer is checked exactly against the CPU oracle (offsets,
ranks, throttle events, pre-cap counts) on the host and the device path, in arrival and locality order, uncapped and at caps
(5, 2), and each case asserts the stats of the path it targets. The engineered cases are built and pinned to their edges in
test_host_trie_lookup_cpu.py.

BFQ_PERFECT_LOG2_MAX = 1 / 2 sends every node of 3 / 5 or more children to the tag table, so whole workloads (random sets, C3,
C4, a SUB/UNSUB delta stream) take the wide-node lookups at every depth, with tier-0 warps mixing them with small-node lanes. The
switch is read once per process: each setting runs in its own process."""
import os
import pickle
import random
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O
import trie_hash as T
from test_gpu_edges import CAPS, INT_MAX, B, check_device, check_host, events_of, kv_of, make_index, make_pairs, oracle_match, true_repeats  # noqa: F401
from test_host_trie_lookup_cpu import (ENG, LONG, NB, as_arrays, eng_model, forced_big_edges, long_topics, model_table, pairs_of,
                                       random_forced_pairs, root_case, tiered, topics_of)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def case():
    return root_case()


def tier_batches(c):
    """tier -> (batch, its expected stats delta): tier 0 keeps every topic, tier 1 takes each one whole (a > 24-byte level),
    tier 2 each one of eng (a frontier of > 64 nodes below the engineered key)"""
    t0 = topics_of(c)
    t1 = tiered(t0, 1) + long_topics(c)
    t2 = [x for x in tiered(t0, 2) if x[0] == ENG]
    return {0: (t0, 0, 0), 1: (t1, len(t1), 0), 2: (t2, len(t2), len(t2))}


def every_path(idx, kv, batch, deferred, overflow):
    """host and device path, arrival and locality order, both caps; the stats delta of each run"""
    tenants, topics, tt = as_arrays(batch)
    rep = true_repeats(tenants, topics, tt)
    for order in (0, 1):
        idx.set_option("order_min_topics", 0 if order == 0 else 1)
        for caps in CAPS:
            d, res = check_host(idx, kv, tenants, topics, tt, caps)
            res.close()
            d2 = check_device(idx, kv, tenants, topics, tt, caps)
            for dd in (d, d2):
                assert dd["deferred_topics"] == deferred and dd["overflow_topics"] == overflow, (order, caps, dd)
                assert dd["duplicate_topics"] == (rep if order else 0)
    idx.set_option("order_min_topics", 32768)


def tag_stats(idx):
    st = idx.stats()
    return st["tag_usable_slots"], st["tag_used_slots"], st["tag_overflowed_blocks"]


@pytest.mark.gpu
@pytest.mark.parametrize("tier", [0, 1, 2])
def test_engineered_root_every_tier(B, case, tier):  # noqa: F811
    pairs = pairs_of(case)
    tab, _, _ = eng_model(pairs)
    idx = make_index(B, pairs)
    assert tag_stats(idx) == (15 * NB, tab.claimed(), tab.overflowed())
    batch, deferred, overflow = tier_batches(case)[tier]
    assert len(batch) > 40
    every_path(idx, kv_of(pairs), batch, deferred, overflow)
    idx.close()


# ------------------------------------------------------------------ delta commits around a shared, filled home block
def delta_case():
    """da and db: two wide roots (fold pairs) whose keys share home block 5. da's 15 keys there fill it; db's 3 keys, one with
    the fingerprint of a da key in that block, arrive by a delta commit after da is placed, so they sit behind it"""
    pa, pb = T.ROOT_BASE, T.ROOT_BASE + 1
    (a1, b1), (a2, b2) = T.fold_pairs(2, seed=51)
    fill = T.names_homed(pa, NB, 5, 15, seed=52)
    fp = T.edge_place(*T.chunks(fill[7])[-1], pa, NB)[1]
    twins = T.names_homed(pb, NB, 5, 1, fp=fp, seed=53) + T.names_homed(pb, NB, 5, 2, seed=54, exclude=fill)
    da = [("da", f, "pgn"[i % 3], 1 + i % 7) for i, f in enumerate(fill + [n + "/#" for n in fill] + [a1, b1, "+/zz", "zz/#"])]
    db = [("db", f, "pgn"[i % 3], 1 + i % 4) for i, f in enumerate(twins + [n + "/#" for n in twins] + [a2, b2, "+/zz"])]
    return fill, twins, make_pairs(da), make_pairs(db)


def filter_of(k, v):
    return T.inner_filter(O.build_match_route(k, v)["mqttTopicFilter"])


def delta_topics(fill, twins):
    out = [("da", n) for n in fill + twins] + [("db", n) for n in fill[:4] + twins]
    out += [(t, n + "/" + LONG) for t, n in out[:]]
    return ["da", "db"], [n for _, n in out], np.array([0 if t == "da" else 1 for t, _ in out], np.int32)


class DeltaModel:
    """the tag table across commits: a delta commit frees the slots of the tenants it rebuilds and places them again, in the
    builder's order; freed tags are cleared, control bytes stay"""

    def __init__(self, pairs):
        self.tab, self.where, _ = model_table(pairs)
        self.ordinal = {t: o for o, t in enumerate(T.Trie(pairs).tenants)}

    def rebuild(self, pairs, tenant):
        for node in [n for n in self.where if n[0] == tenant]:
            self.tab.release(self.where.pop(node))
        self.ordinal.setdefault(tenant, len(self.ordinal))
        ids = {(tenant,): T.ROOT_BASE + self.ordinal[tenant]}
        prefix = b"\x00" + len(tenant).to_bytes(2, "big") + tenant.encode()
        for node in T.Trie([p for p in pairs if p[0].startswith(prefix)]).big_edges().get(tenant, []):
            ids[node] = self.where[node] = self.tab.claim(ids[node[:-1]], *node[-1])[0]


@pytest.mark.gpu
def test_delta_commits_around_a_shared_filled_block(B):  # noqa: F811
    fill, twins, da, db = delta_case()
    tenants, topics, tt = delta_topics(fill, twins)
    idx = make_index(B, da)
    model = DeltaModel(da)
    live = dict(da)
    twin_keys = [k for k, v in db if filter_of(k, v).split("/")[0] in twins]
    # (what, the tenant the commit rebuilds, adds, deletes, the block db's twins sit in afterwards)
    steps = [("db arrives behind da's full block", "db", list(db), [], 6),
             ("da alone: its slots are freed and placed again", "da", make_pairs([("da", "yy", "p", 1)]), [], 6),
             ("da drops 5 of its block-5 keys", "da", [], [k for k, v in da if filter_of(k, v).split("/")[0] in fill[:5]], 6),
             ("db's twins are unsubscribed", "db", [], twin_keys, None),
             ("and subscribed again: block 5 has room now", "db", [(k, v) for k, v in db if k in twin_keys], [], 5)]
    for what, tenant, adds, dels, at in steps:
        assert adds or dels, what
        before = idx.stats()
        idx.apply(adds=adds, dels=dels)
        idx.commit()
        for k, v in adds:
            live[k] = v
        for k in dels:
            live.pop(k, None)
        pairs = sorted(live.items())
        model.rebuild(pairs, tenant)
        st = idx.stats()
        assert (st["delta_commits"] - before["delta_commits"], st["full_commits"] - before["full_commits"]) == (1, 0), what
        assert tag_stats(idx) == (15 * NB, model.tab.claimed(), model.tab.overflowed()), what
        assert model.tab.tags[5, 15] == 1
        if at is not None:
            assert {model.where[("db", T.chunks(n)[-1])] // 16 for n in twins} == {at}, what
        kv = kv_of(pairs)
        fresh = make_index(B, pairs)
        for h in (idx, fresh):
            for caps in CAPS:
                d, res = check_host(h, kv, tenants, topics, tt, caps)
                res.close()
                assert d["deferred_topics"] > 0
                check_device(h, kv, tenants, topics, tt, caps)
        fresh.close()
    idx.close()


# ------------------------------------------------------------------ forced wide nodes, one process per setting
_FORCED_SCRIPT = r"""
import pickle, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import bifromq_b200
d = sys.argv[2]
spec = pickle.load(open(d + "/spec.pkl", "rb"))
out = {}

def run(idx, tag, tenants, topics, tt):
    nt = len(tenants)
    for order in (0, 1):
        idx.set_option("order_min_topics", 0 if order == 0 else 1)
        for caps in spec["caps"]:
            res = idx.match_topics(tenants, topics, np.asarray(tt, np.int32), [caps[0]] * nt, [caps[1]] * nt)
            off, ranks = res.expand()
            out[tag + (order, caps)] = (off.tolist(), ranks.tolist(),
                                        sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist()),
                                        res.route_count.astype(np.int64).tolist())
            res.close()

for c in spec["cases"]:
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load_pairs(c["pairs"])
    idx.commit()
    out[(c["name"], 0, "stats")] = idx.stats()
    run(idx, (c["name"], 0), c["tenants"], c["topics"], c["tt"])
    for step, (adds, dels, final) in enumerate(c.get("deltas", []), 1):
        idx.apply(adds=adds, dels=dels)
        idx.commit()
        out[(c["name"], step, "stats")] = idx.stats()
        run(idx, (c["name"], step), c["tenants"], c["topics"], c["tt"])
        twin = bifromq_b200.GpuRouteIndex(0)
        twin.load_pairs(final)
        twin.commit()
        run(twin, (c["name"], step, "twin"), c["tenants"], c["topics"], c["tt"])
        twin.close()
    idx.close()
pickle.dump(out, open(d + "/out.pkl", "wb"))
"""


def workload_case(config, scale, n_topics):
    from bifromq_b200 import workload
    w = workload.Workload(config, scale=scale)
    keys = [bytes(w.keys[w.key_off[i]:w.key_off[i + 1]]) for i in range(len(w.key_off) - 1)]
    vals = [bytes(w.vals[w.val_off[i]:w.val_off[i + 1]]) for i in range(len(w.val_off) - 1)]
    n = min(n_topics, w.n_topics)
    return dict(name=config, pairs=list(zip(keys, vals)), tenants=list(w.tenants), topics=w.topic_list()[:n],
                tt=np.asarray(w.topic_tenant[:n], np.int32).tolist())


def random_stream_case():
    """a random small-vocabulary set and 8 rounds of SUB / UNSUB on it, each commit also built in full"""
    pairs, tenants, topics, tt = random_forced_pairs(1)
    pool, _, _, _ = random_forced_pairs(2)
    rng = random.Random(3)
    live = dict(pairs)
    deltas = []
    for _ in range(8):
        adds = [rng.choice(pool) for _ in range(rng.randint(5, 40))]
        dels = [k for k in rng.sample(sorted(live), rng.randint(5, 40)) if k not in dict(adds)]
        for k, v in adds:
            live[k] = v
        for k in dels:
            live.pop(k)
        deltas.append((adds, dels, sorted(live.items())))
    return dict(name="rand", pairs=pairs, tenants=tenants, topics=topics, tt=list(tt), deltas=deltas)


def engineered_case(c):
    tenants, topics, tt = as_arrays(topics_of(c) + tiered(topics_of(c), 1) + long_topics(c))
    return dict(name="eng", pairs=pairs_of(c), tenants=tenants, topics=topics, tt=tt.tolist())


FORCED = [dict(BFQ_PERFECT_LOG2_MAX="1"), dict(BFQ_PERFECT_LOG2_MAX="2"), dict(BFQ_PERFECT_LOG2_MAX="8"),
          dict(BFQ_NOALLOC="1"), dict(BFQ_ROOTSTEP="1")]


@pytest.mark.gpu
@pytest.mark.parametrize("env", FORCED, ids=lambda e: ",".join("%s=%s" % kv for kv in sorted(e.items())))
def test_forced_wide_nodes_and_tier0_switches(case, env, tmp_path):
    m = int(env.get("BFQ_PERFECT_LOG2_MAX", T.PERFECT_LOG2_MAX))
    cases = [engineered_case(case)]
    if "BFQ_PERFECT_LOG2_MAX" in env:
        cases += [random_stream_case(), workload_case("C3", 0.005, 6000), workload_case("C4", 0.005, 6000)]
    caps_list = [(INT_MAX, INT_MAX), (5, 2)]
    pickle.dump(dict(cases=cases, caps=caps_list), open(tmp_path / "spec.pkl", "wb"))
    e = dict(os.environ)
    for k in ("BFQ_PERFECT_LOG2_MAX", "BFQ_ROOTSTEP", "BFQ_PREFETCH", "BFQ_NOALLOC", "BFQ_CTAS", "BFQ_ORDER", "BFQ_DEDUP"):
        e.pop(k, None)
    e.update(env)
    subprocess.run([sys.executable, "-c", _FORCED_SCRIPT, ROOT, str(tmp_path)], env=e, check=True, timeout=900)
    out = pickle.load(open(tmp_path / "out.pkl", "rb"))
    for c in cases:
        states = [(0, c["pairs"])] + [(s, d[2]) for s, d in enumerate(c.get("deltas", []), 1)]
        prev = None
        for step, pairs in states:
            kv = kv_of(sorted(pairs))
            st = out[(c["name"], step, "stats")]
            if m <= 2:
                assert st["tag_used_slots"] == forced_big_edges(pairs, m), (c["name"], step)
            if prev is not None:
                assert st["full_commits"] + st["delta_commits"] == prev["full_commits"] + prev["delta_commits"] + 1
            prev = st
            uncapped = oracle_match(kv, c["tenants"], c["topics"], c["tt"], INT_MAX, INT_MAX, O.MODE_TRIE)
            for caps in caps_list:
                want = oracle_match(kv, c["tenants"], c["topics"], c["tt"], caps[0], caps[1], O.MODE_TRIE)
                for tag in ((c["name"], step), (c["name"], step, "twin")) if step else ((c["name"], step),):
                    for order in (0, 1):
                        off, ranks, events, rc = out[tag + (order, caps)]
                        assert off == want.offsets.tolist(), (tag, order, caps)
                        assert ranks == want.ranks.tolist(), (tag, order, caps)
                        assert events == events_of(want), (tag, order, caps)
                        assert rc == np.diff(uncapped.offsets).tolist(), (tag, order, caps)
        if c.get("deltas"):
            assert prev["delta_commits"] > 0   # the stream took the delta path
