"""Delta commits that touch many tenants at once (one batchAddRoute / batchRemoveRoute batch spanning a range's tenants, as
in a reconnect storm). bfq_index_commit rebuilds every touched tenant on all host cores and assembles the new snapshot's
per-rank arrays on the device in one launch, whatever the number of tenants. Every commit here is asserted to take the path
it should (stats 13/14) and to have rebuilt the tenants it should (stat 21), and its whole answer is compared with the CPU
oracle fed the same mutations (offsets, ranks and throttle events under several caps, route lookups and route kinds), with a
twin handle fully built from the same KV, and with results taken before the commit, which keep resolving against their own
snapshot. At the tag table's fill bound the path of each commit is predicted with the model of the table in
test_host_wide_delta_cpu.py, and stats 18..20 are checked against it."""
import random
import threading

import numpy as np
import pytest

import oracle_lib as O
from test_host_wide_delta_cpu import ROOT_BASE, TagModel, home_block, route

pytestmark = pytest.mark.gpu
INT_MAX = 2 ** 31 - 1
CAPS = [(INT_MAX, 100), (2, 1), (4, 4)]
LONG = "a-level-that-is-longer-than-twenty-four-bytes"
VOCAB = ["a", "b", "c", "dd", "e1", LONG, ""]


@pytest.fixture(scope="module")
def B():
    import torch

    import bifromq_b200
    from bifromq_b200 import dist, schema
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.pkg, ns.schema, ns.torch, ns.dist = bifromq_b200, schema, torch, dist
    ns.dev = torch.device("cuda", 0)
    ns.stream = torch.cuda.current_stream(ns.dev).cuda_stream
    return ns


def random_filter(rng):
    lv = []
    n = rng.randint(1, 4)
    for i in range(n):
        r = rng.random()
        if r < 0.2:
            lv.append("+")
        elif r < 0.3 and i == n - 1:
            lv.append("#")
        else:
            lv.append(rng.choice(VOCAB))
    return "/".join(lv)


def random_topic(rng):
    return "/".join(rng.choice(VOCAB) for _ in range(rng.randint(1, 4)))


def tenant_routes(B, rng, tenant, n):
    """n routes of one tenant: normal routes (several receivers on some filters), $share groups, empty levels (multi-segment
    filters), levels longer than 24 B"""
    out = {}
    while len(out) < n:
        f = random_filter(rng)
        if rng.random() < 0.12:
            members = {B.schema.receiver_url(rng.choice([0, 1]), "m%d" % rng.randint(0, 5), "d"): rng.randint(1, 9)
                       for _ in range(rng.randint(1, 3))}
            out[B.schema.route_key(tenant, "$share/g%d/%s" % (rng.randint(0, 2), f))] = B.schema.route_group_bytes(members)
        else:
            url = B.schema.receiver_url(rng.choice([0, 1, 1, 2]), "r%d" % rng.randint(0, 400), "d%d" % rng.randint(0, 3))
            out[B.schema.route_key(tenant, f, url)] = B.schema.incarnation_bytes(rng.randint(0, 99))
    return out


def tkey(B, tenant):
    return B.schema.tenant_begin_key(tenant)


class Index:
    """a handle plus the KV it should hold (the oracle's input)"""

    def __init__(self, B, pairs):
        self.B = B
        self.live = dict(pairs)
        self.idx = B.pkg.GpuRouteIndex(0)
        self.idx.load_pairs(sorted(self.live.items()))
        self.idx.commit()

    def apply(self, adds=(), dels=()):
        adds = dict(adds)
        dels = [k for k in set(dels) if k in self.live and k not in adds]
        self.idx.apply(adds=list(adds.items()), dels=dels)
        self.live.update(adds)
        for k in dels:
            del self.live[k]

    def tenant_keys(self, tenant):
        p = tkey(self.B, tenant)
        return [k for k in self.live if k.startswith(p)]

    def commit(self):
        """commits; returns (path, tenants rebuilt)"""
        st = self.idx.stats()
        self.idx.commit()
        st2 = self.idx.stats()
        assert st2["full_commits"] + st2["delta_commits"] == st["full_commits"] + st["delta_commits"] + 1
        return ("delta" if st2["delta_commits"] == st["delta_commits"] + 1 else "full"), st2["rebuilt_tenants"]

    def garbage_full_next(self):
        st = self.idx.stats()
        return st["garbage_slots"] > st["slots"] // 4 + 4096

    def answer(self, idx, tenants, topics, tt, caps):
        nt = len(tenants)
        res = idx.match_topics(tenants, topics, tt, [caps[0]] * nt, [caps[1]] * nt)
        offsets, ranks = res.expand()
        ev = sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist())
        res.close()
        return offsets.tolist(), ranks.tolist(), ev

    def check(self, tenants, topics, tt, seed=0):
        """the whole answer against the oracle and a fully built twin, under every cap; route lookups and kinds on sampled
        ranks. Returns the number of routes matched under the first caps."""
        tt = np.asarray(tt, np.int32)
        kv = O.KV()
        for k, v in self.live.items():
            kv.put(k, v)
        kv.freeze()
        twin = self.B.pkg.GpuRouteIndex(0)
        twin.load_pairs(sorted(self.live.items()))
        twin.commit()
        total = None
        for caps in CAPS:
            got = self.answer(self.idx, tenants, topics, tt, caps)
            want = kv.match_batch(tenants, topics, tt, caps[0], caps[1], O.MODE_BRUTE)
            assert got[0] == want.offsets.tolist(), caps
            assert got[1] == want.ranks.tolist(), caps
            assert got[2] == sorted((k, t, r) for k, t, r, _ in want.events), caps
            assert self.answer(twin, tenants, topics, tt, caps) == got, caps
            total = len(got[1]) if total is None else total
        keys = sorted(self.live)
        assert self.idx.stats()["routes"] == len(keys)
        rng = random.Random(seed)
        sample = sorted(set(rng.randrange(len(keys)) for _ in range(300)) | {0, len(keys) - 1})
        for r in sample:
            assert self.idx.route(r) == (keys[r], self.live[keys[r]]), r
        assert self.idx.route_kinds(sample).tolist() == twin.route_kinds(sample).tolist()
        twin.close()
        return total

    def hold(self, tenants, topics, tt):
        """a result taken now, with the routes of its first ranks: it must keep resolving against its own snapshot"""
        res = self.idx.match_topics(tenants, topics, np.asarray(tt, np.int32))
        _, ranks = res.expand()
        ranks = ranks[:60].tolist()
        return res, ranks, [res.route(r) for r in ranks]

    @staticmethod
    def check_held(held):
        res, ranks, routes = held
        assert [res.route(r) for r in ranks] == routes
        res.close()


# ------------------------------------------------------------------ an index of about 300 tenants of mixed shapes
N_NARROW = 296
WIDE = {"t100": "%s", "t400": "site/w/%s"}   # a wide node at the root, one below an exact parent


def mixed_index(B, seed):
    """tenants t000, t002, ... (odd numbers are free: new tenants sort between them), 3..40 routes each; t100 and t400 hold
    a wide node of 1500 children"""
    rng = random.Random(seed)
    names = ["t%03d" % (2 * i) for i in range(N_NARROW)]
    pairs = {}
    for t in names:
        pairs.update(tenant_routes(B, rng, t, rng.randint(3, 40)))
    for t, fmt in WIDE.items():
        pairs.update(route(t, fmt % ("c%05d" % i), i, i % 3) for i in range(1500))
    L = Index(B, pairs.items())
    all_names = names + ["t%03d" % (2 * i + 1) for i in range(N_NARROW)]   # every tenant a test may create
    topics = [random_topic(rng) for _ in range(500)] + ["c00007", "c01499", "c01500", "site/w/c00010", "site/w/c02000"]
    tt = [rng.randrange(len(names)) for _ in range(500)] + [50, 50, 50, 200, 200]   # names[50] = t100, names[200] = t400
    tt += [rng.randrange(len(all_names)) for _ in range(200)]
    topics += [random_topic(rng) for _ in range(200)]
    assert all_names[50] == "t100" and all_names[200] == "t400"
    st = L.idx.stats()
    assert st["tenants"] == N_NARROW and st["tag_used_slots"] >= 3000   # plus t100's random root-level edges
    return L, names, all_names, topics, tt, rng


def one_sub(B, rng, tenant, i):
    url = B.schema.receiver_url(rng.choice([0, 1, 2]), "new%d" % i, "d")
    return B.schema.route_key(tenant, random_filter(rng), url), B.schema.incarnation_bytes(i % 97)


@pytest.mark.parametrize("k", [63, 64, 65, 66, 150, "all-but-one", "all"])
def test_one_sub_into_each_of_k_tenants(B, k):
    """one SUB into each of k tenants (wide ones included), then the whole answer; a commit touching every tenant is a delta,
    and the garbage it leaves makes the next commit a full build"""
    L, names, all_names, topics, tt, rng = mixed_index(B, 7)
    n = {"all-but-one": len(names) - 1, "all": len(names)}.get(k, k)
    touched = sorted(rng.sample(names, n))
    if k not in ("all-but-one", "all"):
        touched = sorted(set(touched[:-2]) | {"t100", "t400"})
        touched += sorted(rng.sample([t for t in names if t not in touched], n - len(touched)))
    assert len(set(touched)) == n
    held = L.hold(all_names, topics, tt)
    L.apply([one_sub(B, rng, t, i) for i, t in enumerate(touched)])
    assert L.commit() == ("delta", n)
    Index.check_held(held)
    assert L.check(all_names, topics, tt, seed=n) > 0
    if k == "all":
        assert L.garbage_full_next()
        L.apply([one_sub(B, rng, names[3], 999)])
        assert L.commit() == ("full", len(names))
        L.check(all_names, topics, tt)
    L.idx.close()


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_tenants_created_removed_grown_and_shrunk_in_one_commit(B, seed):
    """one commit holding new tenants that sort between existing ones, removed tenants, a tenant removed and re-added, a
    tenant created and removed again before the commit, and tenants that grow and shrink: the untouched runs between them
    shift by positive, negative and zero amounts. Three such commits in a row, each a delta."""
    L, names, all_names, topics, tt, rng = mixed_index(B, seed)
    live_names = set(names)
    for rnd in range(3):
        adds, dels = {}, []
        expect = set()
        fresh = rng.sample([t for t in all_names if t not in live_names], 25)
        for t in fresh:   # new tenants between existing ones
            adds.update(tenant_routes(B, rng, t, rng.randint(1, 12)))
            expect.add(t)
        cand = [t for t in sorted(live_names) if t not in WIDE]
        rng.shuffle(cand)
        removed, readded, grow, shrink = cand[:15], cand[15:18], cand[18:58], cand[58:90]
        for t in removed:
            dels += L.tenant_keys(t)
        for t in readded:   # every key deleted, new ones added
            dels += L.tenant_keys(t)
            adds.update(tenant_routes(B, rng, t, rng.randint(1, 20)))
            expect.add(t)
        for t in grow + ["t100"]:
            adds.update(tenant_routes(B, rng, t, rng.randint(1, 6)))
            expect.add(t)
        for t in shrink + ["t400"]:
            ks = L.tenant_keys(t)
            if len(ks) > 1:
                dels += rng.sample(ks, min(len(ks) - 1, rng.randint(1, 5)))
                expect.add(t)
        ghost = "t%03d" % (2 * N_NARROW + 1)   # created and deleted before the commit: nothing to build
        L.idx.apply(adds=[route(ghost, "a/b", 0)])
        L.idx.apply(dels=[route(ghost, "a/b", 0)[0]])
        held = L.hold(all_names, topics, tt)
        L.apply(adds.items(), dels)
        assert L.commit() == ("delta", len(expect)), rnd
        assert len(expect) > 64
        live_names = (live_names - set(removed)) | set(fresh)
        assert L.idx.stats()["tenants"] == len(live_names)
        Index.check_held(held)
        assert L.check(all_names, topics, tt, seed=rnd) > 0
    L.idx.close()


# ------------------------------------------------------------------ the tag table's fill bound, many wide tenants at once
class Tags(TagModel):
    def place_all(self, groups):
        """every wide tenant's root children placed into a table whose slots were all freed (every wide tenant is rebuilt):
        block occupancies and overflow bytes of linear probing do not depend on the order of placement"""
        occ = [0] * self.n_blocks
        for names, ordinal in groups:
            for nm in names:
                b = home_block(nm, ROOT_BASE + ordinal, self.n_blocks)
                while occ[b] == 15:
                    self.overflowed.add(b)
                    b = (b + 1) % self.n_blocks
                occ[b] += 1
        return len(self.overflowed)


def test_many_wide_tenants_at_the_fill_bound(B):
    """four wide tenants and 70 narrow ones, every one of them touched by each commit: the commit that leaves the tag table
    one edge below 3/4 of its usable slots is a delta, the one onto the bound is a delta, the one past it is a full build;
    the path and stats 18..20 follow the model of the table"""
    rng = random.Random(5)
    wide = ["w0", "w1", "w2", "w3"]            # ordinals 0..3: the shorter ids sort first
    narrow = ["n%03d" % i for i in range(70)]
    children = {w: ["d%05d" % i for i in range(1500)] for w in wide}
    pairs = {}
    for w in wide:
        pairs.update(route(w, c, i, i % 3) for i, c in enumerate(children[w]))
    for t in narrow:
        pairs.update(tenant_routes(B, rng, t, rng.randint(3, 10)))
    L = Index(B, pairs.items())
    groups = lambda: [(children[w], o) for o, w in enumerate(wide)]
    model = Tags(6000)
    ovf = model.place_all(groups())
    st = L.idx.stats()
    assert (st["tag_usable_slots"], st["tag_used_slots"], st["tag_overflowed_blocks"]) == (model.usable, 6000, ovf)
    bound = 3 * model.usable // 4
    tenants = wide + narrow
    topics = [c for w in wide for c in children[w][::300]] + ["d09999", "zz"] + [random_topic(rng) for _ in range(100)]
    tt = [o for o in range(4) for _ in children["w0"][::300]] + [0, 1] + [rng.randrange(len(tenants)) for _ in range(100)]
    seen = []
    extra = 0
    for total in (bound - 1, bound, bound + 1):
        adds = {}
        new = total - sum(len(c) for c in children.values())
        for j in range(new):   # the new children, spread over the wide tenants
            w = wide[j % 4]
            nm = "e%05d" % (extra + j)
            children[w].append(nm)
            adds.update([route(w, nm, j, 1)])
        extra += new
        for i, w in enumerate(wide):   # one more receiver on an existing child: the tenant is touched, no new edge
            adds.update([route(w, children[w][0], 5000 + extra + i, 2)])
        for i, t in enumerate(narrow):
            adds.update([one_sub(B, rng, t, extra + i)])
        trial = Tags(0)
        trial.n_blocks, trial.usable, trial.overflowed = model.n_blocks, model.usable, set(model.overflowed)
        want = model.path(total, trial.place_all(groups()))
        if want == "full":
            model = Tags(total)
            ovf = model.place_all(groups())
        else:
            model, ovf = trial, len(trial.overflowed)
        held = L.hold(tenants, topics, tt)
        L.apply(adds.items())
        got = L.commit()
        assert got == (want, len(tenants)), (total, bound)
        seen.append((total, got[0]))
        st = L.idx.stats()
        assert (st["tag_usable_slots"], st["tag_used_slots"], st["tag_overflowed_blocks"]) == (model.usable, total, ovf)
        Index.check_held(held)
        L.check(tenants, topics, tt)
    assert seen == [(bound - 1, "delta"), (bound, "delta"), (bound + 1, "full")]
    L.idx.close()


# ------------------------------------------------------------------ concurrency and the fan-out's deliverer ids
def test_matches_in_flight_while_wide_commits_land(B):
    """four threads match while the main thread commits deltas of 100 tenants each (and the full builds the garbage rule asks
    for in between); every result equals the oracle's answer for the generation it reports"""
    L, names, all_names, topics, tt, rng = mixed_index(B, 21)
    tt = np.asarray(tt, np.int32)
    expected, got, errors = {}, [], []
    deltas = 0
    stop = threading.Event()

    def snapshot_answer():
        kv = O.KV()
        for k, v in L.live.items():
            kv.put(k, v)
        kv.freeze()
        want = kv.match_batch(all_names, topics, tt, 4, 4, O.MODE_BRUTE)
        expected[L.idx.generation()] = (want.offsets.tolist(), want.ranks.tolist())

    def worker():
        try:
            while not stop.is_set():
                res = L.idx.match_topics(all_names, topics, tt, [4] * len(all_names), [4] * len(all_names))
                o, r = res.expand()
                got.append((res.generation, o.tolist(), r.tolist()))
                res.close()
        except Exception as e:   # reported by the main thread
            errors.append(e)
    snapshot_answer()
    threads = [threading.Thread(target=worker) for _ in range(4)]
    for t in threads:
        t.start()
    try:
        for rnd in range(6):
            touched = rng.sample(names, 100)
            dels = [rng.choice(L.tenant_keys(t)) for t in touched[:30] if len(L.tenant_keys(t)) > 1]
            L.apply([one_sub(B, rng, t, 1000 * rnd + i) for i, t in enumerate(touched)], dels)
            # every third commit or so is a full build: the garbage of ~100 replaced tenants per commit adds up
            want = ("full", len(names)) if L.garbage_full_next() else ("delta", 100)
            assert L.commit() == want
            deltas += want[0] == "delta"
            snapshot_answer()
    finally:
        stop.set()
        for t in threads:
            t.join()
    assert not errors, errors
    assert deltas >= 3 and len(got) > 6 and len({g for g, _, _ in got}) > 1
    for gen, o, r in got:
        assert (o, r) == expected[gen], gen
    L.idx.close()


def test_fanout_deliverer_ids_stable_across_many_tenant_commits(B):
    """bfq_fanout_device on results of successive deltas of 80 tenants each: the (subBrokerId, delivererKey) -> id map only
    grows"""
    from test_gpu_fanout import fan_check, match_device, oracle
    rng = random.Random(3)
    names = ["f%03d" % i for i in range(120)]
    pairs = {}
    for t in names:
        for i in range(rng.randint(2, 8)):
            url = B.schema.receiver_url(i % 3, "r%d" % rng.randint(0, 50), "inbox%d" % rng.randint(0, 9))
            pairs[B.schema.route_key(t, rng.choice(["a/+", "a/b", "#", "+/b"]), url)] = B.schema.incarnation_bytes(1)
        members = {B.schema.receiver_url(0, "m%d" % j, "inbox%d" % j): 1 for j in range(3)}
        pairs[B.schema.route_key(t, "$share/g/a/#")] = B.schema.route_group_bytes(members)
    L = Index(B, pairs.items())
    topics = ["a/b", "x/b", "a/c"] * 40
    tt = np.asarray([i // 3 for i in range(120)], np.int32)
    ids = {}
    for rnd in range(4):
        out = match_device(B, L.idx, names, topics, tt)
        want = oracle(sorted(L.live.items()), names, topics, tt)
        _, s = fan_check(B, L.idx, out, topics, want, sorted(L.live.items()))
        out.release()
        for key, d in s["ids"].items():
            assert ids.setdefault(key, d) == d
        touched = rng.sample(names, 80)
        adds = [(B.schema.route_key(t, "a/b", B.schema.receiver_url(1, "new%d" % rnd, "inbox-new%d" % i)), B.schema.incarnation_bytes(1))
                for i, t in enumerate(touched)]
        L.apply(adds)
        assert L.commit() == ("delta", 80)
    L.idx.close()


# ------------------------------------------------------------------ full size
def test_c4_one_sub_into_each_of_65_500_and_1000_tenants(B):
    """C4 at scale 1.0 (1000 tenants, 10M filters): one SUB into each of 65, then 500 tenants, each a delta; the garbage of the
    500 makes the next commit a full build; then one SUB into every tenant, a delta. After each delta a 200k-topic slice of
    the batch equals the oracle fed the same mutations."""
    import os
    from bifromq_b200 import workload
    threads = os.cpu_count() or 8
    w = workload.Workload("C4")
    idx = B.pkg.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    idx.commit()
    kv = O.KV()
    kv.load(w.keys, w.key_off, w.vals, w.val_off)
    names = w.tenants
    assert len(names) == 1000
    tenants = idx.tenant_blob(names)
    tb, toff = O.blob(names)
    tt_all = np.ascontiguousarray(w.topic_tenant[:w.n_topics]).astype(np.int32)
    rng = random.Random(65)

    def commit(touched, tag):
        adds = [(B.schema.route_key(t, rng.choice(["%s/+/x", "#", "%s/a/b"]).replace("%s", tag),
                                    B.schema.receiver_url(i % 3, "storm-%s-%d" % (tag, i), "d")), B.schema.incarnation_bytes(i % 50))
                for i, t in enumerate(touched)]
        idx.apply(adds=adds)
        for k, v in adds:
            kv.put(k, v)
        st = idx.stats()
        idx.commit()
        st2 = idx.stats()
        return ("delta" if st2["delta_commits"] == st["delta_commits"] + 1 else "full"), st2["rebuilt_tenants"]

    def check(lo, hi):
        kv.freeze()
        off = np.ascontiguousarray(w.topic_off[lo:hi + 1])
        nt = len(names)
        r = idx.match(tenants, w.topics, off, tt_all[lo:hi], [INT_MAX] * nt, [100] * nt)
        offsets, ranks = r.expand()
        r.close()
        want = kv.match_blobs(tb, toff, w.topics, off, tt_all[lo:hi], hi - lo, INT_MAX, 100, O.MODE_TRIE, False, threads)
        assert np.array_equal(offsets, want.offsets) and np.array_equal(ranks, want.ranks)
        assert len(ranks) > 0

    assert commit(sorted(rng.sample(names, 65)), "k65") == ("delta", 65)
    check(0, 200_000)
    assert commit(sorted(rng.sample(names, 500)), "k500") == ("delta", 500)
    check(400_000, 600_000)
    assert commit([names[1]], "reclaim") == ("full", 1000)
    assert commit(list(names), "k1000") == ("delta", 1000)
    check(800_000, 1_000_000)
    assert idx.stats()["routes"] == len(kv)
    idx.close()
