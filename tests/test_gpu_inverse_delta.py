"""Delta commits of the inverse (retain) index: a commit rebuilds only the tenants whose staged topic set changed, appends their
regions behind the existing ones and inserts their exact edges into the live device hash table (rinsert_edges_kernel).

The reference each answer is checked against is the TWIN: a fresh handle given the same add / remove history and committed
once, i.e. a full build. Ids are handed out at add time, so the twin's ids are the same, and "equal to the twin" means identical
offsets, ids (order included), totals, n_ranges and n_overflow_filters. Every answer is also checked against the CPU oracle
(TopicLevelIndex).

The commit path is predicted in plain Python from bfq_rindex_stats before the commit and the shapes of the rebuilt tries (nodes
and exact edges per tenant, long names included), with the bounds include/bfq_gpumatch.h states for bfq_rindex_commit: garbage
nodes <= live / 4 + 4096, occupied slots <= 3/4 of the usable ones. Each commit must take the predicted path and leave the
predicted stats.
"""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_lib as O

GARBAGE_SLACK = 4096
TOKEN_BYTES = 24
BLOCK_USABLE = 15
STAT_NAMES = ["topics", "tenants", "nodes", "garbage_nodes", "used_slots", "usable_slots", "full_commits", "delta_commits",
              "rebuilt_tenants", "device_bytes", "overflowed_blocks"]


# ------------------------------------------------------------------ plain-Python model (no GPU)
def tenant_shape(topics):
    """(node records, exact edges) of one tenant's trie as the per-tenant builder lays it out: a root plus one node per distinct
    level prefix; one edge per node, plus one chunk edge per distinct 24-byte-chunk prefix of a name longer than 24 bytes
    under the same parent"""
    prefixes, virt = set(), set()
    for p in topics:
        lv = p.encode().split(b"/")
        for i in range(len(lv)):
            parent, name = tuple(lv[:i]), lv[i]
            prefixes.add(tuple(lv[:i + 1]))
            for j in range((len(name) - 1) // TOKEN_BYTES if name else 0):
                virt.add((parent, name[:TOKEN_BYTES * (j + 1)]))
    return 1 + len(prefixes), len(prefixes) + len(virt)


def table_usable(n_edges):
    """usable slots of the table a full build sizes for n_edges edges (load 1/2, at least 64 blocks of 15)"""
    return max(64, (2 * n_edges + BLOCK_USABLE - 1) // BLOCK_USABLE) * BLOCK_USABLE


class Model:
    """the staged index as the C-ABI keeps it: ids in add order, the dirty tenants, and each live tenant's region size"""

    def __init__(self):
        self.entries, self.nxt, self.dirty, self.region, self.history = {}, 0, set(), {}, []

    def add(self, pairs):
        self.history.append(("add", list(pairs)))
        for k in pairs:
            if k not in self.entries:
                self.entries[k] = self.nxt
                self.nxt += 1
                self.dirty.add(k[0])

    def remove(self, t, p):
        self.history.append(("del", (t, p)))
        if (t, p) in self.entries:
            del self.entries[(t, p)]
            self.dirty.add(t)

    def topics_of(self, t):
        return [p for (tt, p) in self.entries if tt == t]

    def live_tenants(self):
        return {t for t, _ in self.entries}

    def predict(self, st):
        """the path and stats of the next commit, given the stats before it; self.why names the bound a full build crossed"""
        self.why = None
        if st["full_commits"] == 0:
            return self._full()
        if not self.dirty:
            return "noop", dict(st, rebuilt_tenants=0)
        garbage, nodes, used, rebuilt = st["garbage_nodes"], st["nodes"], st["used_slots"], 0
        region = dict(self.region)
        for t in self.dirty:
            if t in region:
                garbage += region.pop(t)
            tops = self.topics_of(t)
            if tops:
                n, e = tenant_shape(tops)
                nodes, used, rebuilt, region[t] = nodes + n, used + e, rebuilt + 1, n
        if garbage > (nodes - garbage) // 4 + GARBAGE_SLACK:
            self.why = "garbage"
        elif used * 4 > st["usable_slots"] * 3:
            self.why = "table"
        if self.why:
            return self._full()
        want = dict(st, nodes=nodes, garbage_nodes=garbage, used_slots=used, rebuilt_tenants=rebuilt, tenants=len(region),
                    topics=len(self.entries), delta_commits=st["delta_commits"] + 1)
        return "delta", (want, region)

    def _full(self):
        region, nodes, edges, by_tenant = {}, 0, 0, {}
        for t, p in self.entries:
            by_tenant.setdefault(t, []).append(p)
        for t, tops in by_tenant.items():
            n, e = tenant_shape(tops)
            region[t], nodes, edges = n, nodes + n, edges + e
        want = dict(nodes=nodes, garbage_nodes=0, used_slots=edges, usable_slots=table_usable(edges), tenants=len(region),
                    topics=len(self.entries), rebuilt_tenants=len(region))
        return "full", (want, region)


def replay(idx, history, N):
    for op, arg in history:
        if op == "add":
            tenants = list(dict.fromkeys(t for t, _ in arg))
            blob, off = N.as_blob([p for _, p in arg])
            idx.add_blobs(tenants, blob, off, np.array([tenants.index(t) for t, _ in arg], np.int32))
        else:
            idx.remove(*arg)


# ------------------------------------------------------------------ the random stream (plain Python data)
N_TENANTS = 56
ROUNDS = 25
WIDE, VANISH, BURST = "wide", "t07", "t31"
WORDS = ["a", "b", "x", "y", "dev", "sensor", "$sys", "$x", "", "é"]


def long_name(rng):
    """23-73 bytes; one in three shares its first 24 or 48 bytes with other long names"""
    n = rng.randint(23, 73)
    if rng.random() < 0.33:
        return ("L" * 48 + "".join(rng.choice("pqrs") for _ in range(30)))[:n]
    return "".join(rng.choice("abcdefghijklmnopqrstuvwxyz0123456789") for _ in range(n))


def random_topic(rng):
    lv = []
    for i in range(rng.randint(1, 4)):
        r = rng.random()
        if r < 0.1:
            lv.append(long_name(rng))
        elif i == 0 and r < 0.2:
            lv.append(rng.choice(["$sys", "$x", "$"]))
        else:
            lv.append(rng.choice(WORDS))
    return "/".join(lv)


def stream(seed=7):
    """the ops of each round; round 0 is the initial load. An op is ("add", [(t, p), ...]) or ("del", (t, p))"""
    rng = random.Random(seed)
    tenants = ["t%02d" % i for i in range(N_TENANTS)]
    live = {}
    removed = []
    rounds = []
    init = []
    for t in tenants:
        for _ in range(rng.randint(10, 20)):
            init.append((t, random_topic(rng)))
    init += [(WIDE, "w%02d/x" % i) for i in range(40)]
    init += [(BURST, "burst/%d" % i) for i in range(5)]
    rounds.append([("add", init)])
    for k in init:
        live[k] = 1
    for r in range(1, ROUNDS + 1):
        ops = []
        for t in rng.sample(tenants, 3):
            mine = [k for k in live if k[0] == t]
            adds = [(t, random_topic(rng)) for _ in range(rng.randint(1, 4))]
            ops.append(("add", adds))
            for k in adds:
                live[k] = 1
            for k in rng.sample(mine, min(len(mine), rng.randint(0, 2))):
                ops.append(("del", k))
                live.pop(k, None)
                removed.append(k)
        if removed and r % 3 == 0:          # a re-add of a removed topic: a new id
            k = removed.pop(0)
            ops.append(("add", [k]))
            live[k] = 1
        some = rng.choice(sorted(live))      # re-adding a live topic dirties nothing
        ops.append(("add", [some]))
        if r == 5 or r == 17:                # the tenant vanishes ...
            for k in sorted(k for k in live if k[0] == VANISH):
                ops.append(("del", k))
                live.pop(k)
        if r == 9:                           # ... and returns
            back = [(VANISH, "back/%d" % i) for i in range(6)] + [(VANISH, "$sys/back")]
            ops.append(("add", back))
            for k in back:
                live[k] = 1
        if r == 17:                          # vanishes and returns within one round
            ops.append(("add", [(VANISH, "again")]))
            live[(VANISH, "again")] = 1
        if r == 12:                          # widened past 64 level-0 names: '+' on it goes to tier 2
            wide = [(WIDE, "w%02d/x" % i) for i in range(40, 72)]
            ops.append(("add", wide))
            for k in wide:
                live[k] = 1
        if r == 14:
            ops.append(("add", [("newcomer", "n/1"), ("newcomer", "$sys/n")]))
            live[("newcomer", "n/1")] = live[("newcomer", "$sys/n")] = 1
        rounds.append(ops)
    return rounds


GENERIC_FILTERS = ["#", "+", "+/#", "+/+", "+/+/#", "+/+/+", "$sys/#", "$sys/+", "$/#", "/#", "/+", "+/", "", "a/#", "+/x",
                   "a/+/#", "back/+", "w05/+", "+/x/#"]


def filters_for(rng, model, tenants):
    out = []
    for t in sorted(tenants):
        out += [(t, f) for f in GENERIC_FILTERS]
        tops = sorted(model.topics_of(t))
        for p in rng.sample(tops, min(3, len(tops))):
            lv = p.split("/")
            out += [(t, p), (t, lv[0] + "/#"), (t, "/".join(lv[:-1] + ["+"]))]
    return out


# ------------------------------------------------------------------ CPU: the generator's shape
def test_stream_generator_shape():
    rounds = stream()
    assert len(rounds) == ROUNDS + 1
    m = Model()
    present, readded, wide_max, seen_long, seen_dollar, seen_empty = [], 0, 0, set(), False, False
    ever_removed = set()
    for ops in rounds:
        for op, arg in ops:
            if op == "add":
                readded += sum(k in ever_removed and k not in m.entries for k in arg)
                m.add(arg)
            else:
                ever_removed.add(arg)
                m.remove(*arg)
        present.append(bool(m.topics_of(VANISH)))
        wide_max = max(wide_max, len({p.split("/")[0] for p in m.topics_of(WIDE)}))
        for _, p in m.entries:
            for lv in p.split("/"):
                if len(lv.encode()) >= 23:
                    seen_long.add(len(lv.encode()))
            seen_dollar |= p.startswith("$")
            seen_empty |= "" in p.split("/")
    assert len(m.live_tenants()) >= 50
    # the tenant vanishes and returns
    assert present[0] and not all(present) and present[-1]
    assert any(a and not b for a, b in zip(present, present[1:])) and any(b and not a for a, b in zip(present, present[1:]))
    assert min(seen_long) <= 24 and max(seen_long) >= 49 and wide_max > 64 and readded > 0
    assert seen_dollar and seen_empty


def test_tenant_shape_counts_chunk_nodes_once_per_shared_prefix():
    assert tenant_shape(["a/b", "a/c", "a"]) == (4, 3)
    assert tenant_shape([""]) == (2, 1)
    assert tenant_shape(["x" * 24]) == (2, 1)
    assert tenant_shape(["x" * 25]) == (2, 2)
    assert tenant_shape(["x" * 48 + "1", "x" * 48 + "2", "x" * 30]) == (4, 3 + 2)


def test_stats_is_exported_and_a_null_handle_is_invalid():
    import bifromq_b200
    from bifromq_b200 import _native
    bifromq_b200.load_library()
    raw = C.CDLL(_native.LIB_PATH)
    assert hasattr(raw, "bfq_rindex_stats")
    s = np.zeros(len(STAT_NAMES), np.int64)
    assert _native.lib.bfq_rindex_stats(None, s.ctypes.data, len(s)) == -1   # BFQ_E_INVALID


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def R():
    import bifromq_b200
    from bifromq_b200 import _native, retain, workload
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.N, ns.retain, ns.workload = _native, retain, workload
    return ns


def run(R, idx, filters, limit=None):
    tenants = list(dict.fromkeys(t for t, _ in filters)) or ["t"]
    blob, off = R.N.as_blob([f for _, f in filters])
    ft = np.array([tenants.index(t) for t, _ in filters] or [0], np.int32)
    return idx.match_blobs(tenants, blob, off, ft, limit)


def same(a, b):
    assert a.offsets.tolist() == b.offsets.tolist()
    assert a.ids.tolist() == b.ids.tolist()
    assert a.totals.tolist() == b.totals.tolist()
    assert (a.n_ranges, a.n_overflow_filters) == (b.n_ranges, b.n_overflow_filters)


def check_oracle(res, model, filters):
    orc = O.TopicLevelIndex()
    for (t, p), i in model.entries.items():
        orc.add(p, i, t)
    for i, (t, f) in enumerate(filters):
        got = res.matches(i).tolist()
        want = orc.match(f, t)
        assert len(set(got)) == len(got) and sorted(got) == want, (t, f)
        assert int(res.totals[i]) == len(want), (t, f)


def twin_of(R, model):
    twin = R.retain.GpuTopicMatchIndex(0)
    replay(twin, model.history, R.N)
    twin.commit()
    assert twin.stats()["full_commits"] == 1
    return twin


def commit_as_predicted(idx, model):
    """commit, check the path and the stats against the model's prediction -> the path taken"""
    before = idx.stats()
    path, info = model.predict(before)
    idx.commit()
    st = idx.stats()
    if path == "noop":
        assert st == info
        return path
    want, region = info
    for k, v in want.items():
        if k not in ("device_bytes", "overflowed_blocks"):   # inserts may overflow blocks: checked below
            assert st[k] == v, (path, k, st[k], v)
    assert st["full_commits"] == before["full_commits"] + (path == "full")
    assert st["delta_commits"] == before["delta_commits"] + (path == "delta")
    if path == "delta":
        assert st["overflowed_blocks"] >= before["overflowed_blocks"]
    model.region, model.dirty = region, set()
    return path


def apply_ops(idx, model, ops, N):
    for op, arg in ops:
        if op == "add":
            model.add(arg)
            tenants = list(dict.fromkeys(t for t, _ in arg))
            blob, off = N.as_blob([p for _, p in arg])
            ids = idx.add_blobs(tenants, blob, off, np.array([tenants.index(t) for t, _ in arg], np.int32)).tolist()
            assert ids == [model.entries[k] for k in arg]
        else:
            model.remove(*arg)
            idx.remove(*arg)


# ------------------------------------------------------------------ GPU: the random stream
@pytest.mark.gpu
def test_random_stream_matches_oracle_and_twin(R):
    rng = random.Random(3)
    idx = R.retain.GpuTopicMatchIndex(0)
    model = Model()
    paths, tier2 = [], 0
    for r, ops in enumerate(stream()):
        touched_before = set(model.dirty)
        apply_ops(idx, model, ops, R.N)
        dirty = set(model.dirty) | touched_before
        paths.append(commit_as_predicted(idx, model))
        if r > 0 and paths[-1] == "delta":
            assert idx.stats()["rebuilt_tenants"] == len({t for t in dirty if model.topics_of(t)})
        sample = (dirty | set(rng.sample(sorted(model.live_tenants()), 5)) | {WIDE, VANISH, "nobody"})
        filters = filters_for(rng, model, sample)
        res = run(R, idx, filters)
        check_oracle(res, model, filters)
        twin = twin_of(R, model)
        same(res, run(R, twin, filters))
        lim = np.array([rng.choice([-1, 0, 1, 2, 5]) for _ in filters], np.int64)
        got = run(R, idx, filters, lim)
        same(got, run(R, twin, filters, lim))
        for i in range(len(filters)):
            k = int(res.totals[i]) if lim[i] < 0 else min(int(res.totals[i]), int(lim[i]))
            assert got.matches(i).tolist() == res.matches(i).tolist()[:k]
        twin.close()
        tier2 += res.n_overflow_filters
    assert paths[0] == "full"
    assert paths[1:].count("delta") >= 15, paths
    assert tier2 > 0
    # a commit with nothing staged since the last one does no work
    assert commit_as_predicted(idx, model) == "noop"


# ------------------------------------------------------------------ GPU: the bounds
@pytest.mark.gpu
def test_garbage_bound_turns_a_delta_into_a_full_build(R):
    idx = R.retain.GpuTopicMatchIndex(0)
    model = Model()
    base = [("s%03d" % i, "k/%d" % j) for i in range(400) for j in range(100)]
    big = [("big", "b/%d/%d" % (i, j)) for i in range(30) for j in range(60)]
    apply_ops(idx, model, [("add", base + big)], R.N)
    assert commit_as_predicted(idx, model) == "full"
    paths = []
    for r in range(20):
        apply_ops(idx, model, [("add", [("big", "touch/%d" % r)])], R.N)
        paths.append(commit_as_predicted(idx, model))
        if paths[-1] == "full":
            break
    assert paths[-1] == "full" and model.why == "garbage", (paths, model.why)
    assert paths[:-1] == ["delta"] * (len(paths) - 1) and len(paths) >= 3, paths
    st = idx.stats()
    assert st["garbage_nodes"] == 0 and st["rebuilt_tenants"] == 401 and st["full_commits"] == 2
    filters = [("big", f) for f in ("#", "touch/+", "b/7/+", "b/+/59")] + [("s005", "k/+")]
    res = run(R, idx, filters)
    check_oracle(res, model, filters)
    twin = twin_of(R, model)
    same(res, run(R, twin, filters))


@pytest.mark.gpu
def test_table_bound_just_under_is_a_delta_one_over_is_a_full_build(R):
    idx = R.retain.GpuTopicMatchIndex(0)
    model = Model()
    apply_ops(idx, model, [("add", [("t%d" % i, "a/%d" % j) for i in range(20) for j in range(100)])], R.N)
    assert commit_as_predicted(idx, model) == "full"
    st = idx.stats()
    room = st["usable_slots"] * 3 // 4 - st["used_slots"]
    assert room > 100
    fill = [("fill", "%d" % j) for j in range(room)]        # a new tenant: one edge per topic
    assert tenant_shape([p for _, p in fill])[1] == room
    apply_ops(idx, model, [("add", fill)], R.N)
    assert commit_as_predicted(idx, model) == "delta"
    assert idx.stats()["used_slots"] == st["usable_slots"] * 3 // 4
    apply_ops(idx, model, [("add", [("one", "more")])], R.N)
    assert commit_as_predicted(idx, model) == "full" and model.why == "table"
    filters = [("fill", "+"), ("fill", "77"), ("one", "#"), ("t3", "a/+")]
    res = run(R, idx, filters)
    check_oracle(res, model, filters)
    same(res, run(R, twin_of(R, model), filters))


@pytest.mark.gpu
def test_overflow_chains_find_every_inserted_edge(R):
    """a 64-block table filled to its bound by one delta: blocks overflow into their neighbours, and every edge is found"""
    idx = R.retain.GpuTopicMatchIndex(0)
    model = Model()
    apply_ops(idx, model, [("add", [("seed", "s/%d" % j) for j in range(8)])], R.N)
    assert commit_as_predicted(idx, model) == "full"
    st = idx.stats()
    assert st["usable_slots"] == 64 * BLOCK_USABLE and st["overflowed_blocks"] == 0
    n = st["usable_slots"] * 3 // 4 - st["used_slots"] - 1 - 2    # "p" and a long chunk edge under the same root
    many = [("many", "p/%d" % j) for j in range(n)] + [("many", "q" * 40)]
    apply_ops(idx, model, [("add", many)], R.N)
    assert commit_as_predicted(idx, model) == "delta"
    st2 = idx.stats()
    assert st2["overflowed_blocks"] > 0 and st2["used_slots"] == st["usable_slots"] * 3 // 4
    filters = [("many", p) for _, p in many] + [("many", "p/+"), ("many", "#"), ("seed", "s/+"), ("many", "q" * 40 + "/#")]
    res = run(R, idx, filters)
    check_oracle(res, model, filters)
    assert all(int(res.totals[i]) == 1 for i in range(len(many)))
    same(res, run(R, twin_of(R, model), filters))


# ------------------------------------------------------------------ GPU: retain keys across a delta
@pytest.mark.gpu
def test_retain_keys_of_an_older_result_survive_a_delta_commit(R):
    idx = R.retain.GpuTopicMatchIndex(0)
    model = Model()
    apply_ops(idx, model, [("add", [("t", "old/%d" % i) for i in range(6)] + [("u", "x")])], R.N)
    commit_as_predicted(idx, model)
    r1 = idx.match_blobs(["t"], *R.N.as_blob(["old/+"]), np.zeros(1, np.int32), with_retain_keys=True)
    ids1 = r1.ids.tolist()
    apply_ops(idx, model, [("del", ("t", "old/%d" % i)) for i in range(3)] + [("add", [("t", "new/%d" % i) for i in range(6)])],
              R.N)
    assert commit_as_predicted(idx, model) == "delta"
    r2 = idx.match_blobs(["t"], *R.N.as_blob(["old/+", "new/+"]), np.zeros(2, np.int32), with_retain_keys=True)
    blob, koff = r1.retain_keys
    keys1 = [bytes(blob[koff[j]:koff[j + 1]]) for j in range(len(ids1))]
    assert keys1 == [O.retain_key("t", "old/%d" % i) for i in ids1]
    blob2, koff2 = r2.retain_keys
    names = {i: p for (t, p), i in model.entries.items()}
    assert [bytes(blob2[koff2[j]:koff2[j + 1]]) for j in range(len(r2.ids))] == [O.retain_key("t", names[i]) for i in r2.ids]
    assert sorted(names[i] for i in r2.ids) == sorted(["old/3", "old/4", "old/5"] + ["new/%d" % i for i in range(6)])


# ------------------------------------------------------------------ GPU: C5 at 1/20 scale
@pytest.mark.gpu
def test_c5_scaled_one_topic_delta_equals_the_twin(R):
    w = R.workload.Workload("C5", scale=0.05)
    assert w.n_query_filters >= 4096
    tenants = w.tenants
    ft = w.filter_tenant[:w.n_query_filters]
    tt = w.topic_tenant[:w.n_topics]

    def load(idx):
        return idx.add_blobs(tenants, w.topics, w.topic_off, tt)
    idx = R.retain.GpuTopicMatchIndex(0)
    ids = load(idx)
    idx.commit()
    tl = w.topic_list()
    t0 = tenants[int(ft[0])]
    extra = (tl[int(np.nonzero(tt == int(ft[0]))[0][0])].decode() + "/delta")
    idx.add(t0, [extra])
    idx.commit()
    st = idx.stats()
    assert st["full_commits"] == 1 and st["delta_commits"] == 1 and st["rebuilt_tenants"] == 1 and st["garbage_nodes"] > 0
    twin = R.retain.GpuTopicMatchIndex(0)
    assert load(twin).tolist() == ids.tolist()
    extra_id = int(twin.add(t0, [extra])[0])
    twin.commit()
    a = idx.match_blobs(tenants, w.filters, w.filter_off, ft)
    same(a, twin.match_blobs(tenants, w.filters, w.filter_off, ft))
    lim = np.full(w.n_query_filters, 10, np.int64)
    same(idx.match_blobs(tenants, w.filters, w.filter_off, ft, lim), twin.match_blobs(tenants, w.filters, w.filter_off, ft, lim))
    # the touched tenant's answers against the oracle
    orc = O.TopicLevelIndex()
    for i in range(w.n_topics):
        if int(tt[i]) == int(ft[0]):
            orc.add(tl[i], int(ids[i]), t0)
    orc.add(extra, extra_id, t0)
    fl = w.query_filter_list()
    mine = [i for i in range(w.n_query_filters) if int(ft[i]) == int(ft[0])]
    assert mine
    for i in mine:
        assert sorted(a.matches(i).tolist()) == orc.match(fl[i], t0)
