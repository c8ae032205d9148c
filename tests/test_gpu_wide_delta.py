"""Delta commits of the forward index with wide nodes (more children than a private perfect-hash array holds: their children
live in the shared tag table). bfq_index_commit rebuilds only the touched tenants: their old tag slots are freed, their new
wide edges are placed into the live table, their tag-table records are scattered on the device, and the tag-table records of
the untouched tenants whose ranks moved are shifted. Every commit here is asserted to take the path it should (stats 13/14),
and every answer is compared with the CPU oracle fed the same mutations (offsets, ranks, throttle events), and with a twin
handle fully built from the same KV. At the tag table's bounds the path of each commit is predicted with the model of the
table in test_host_wide_delta_cpu.py, and stats 18..20 are checked against it."""
import random
import threading

import numpy as np
import pytest

import oracle_lib as O
from test_gpu_forward import random_pairs
from test_host_wide_delta_cpu import TagModel, host_stats, route

pytestmark = pytest.mark.gpu
INT_MAX = 2 ** 31 - 1
CAPS = [(INT_MAX, 100), (4, 4)]


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


class Live:
    """a handle plus the KV it should hold (the oracle's input)"""

    def __init__(self, B, pairs):
        self.B = B
        self.live = dict(pairs)
        self.idx = B.pkg.GpuRouteIndex(0)
        self.idx.load_pairs(sorted(self.live.items()))
        self.idx.commit()

    def apply(self, adds=(), dels=()):
        adds = list(adds)
        dels = [k for k in dels if k in self.live and k not in dict(adds)]
        self.idx.apply(adds=adds, dels=dels)
        for k, v in adds:
            self.live[k] = v
        for k in dels:
            del self.live[k]

    def commit(self):
        """commits and returns the path it took (the garbage bound of the replaced regions is not what these tests are about:
        it must not be the reason for a full build)"""
        st = self.idx.stats()
        assert st["garbage_slots"] <= st["slots"] // 4 + 4096, st
        self.idx.commit()
        st2 = self.idx.stats()
        assert st2["full_commits"] + st2["delta_commits"] == st["full_commits"] + st["delta_commits"] + 1
        return "delta" if st2["delta_commits"] == st["delta_commits"] + 1 else "full"

    def kv(self):
        kv = O.KV()
        for k, v in self.live.items():
            kv.put(k, v)
        kv.freeze()
        return kv

    def answer(self, idx, tenants, topics, tt, caps):
        nt = len(tenants)
        res = idx.match_topics(tenants, topics, tt, [caps[0]] * nt, [caps[1]] * nt)
        offsets, ranks = res.expand()
        ev = sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist())
        res.close()
        return offsets, ranks, ev

    def check(self, tenants, topics, tt=None, twin=False, mode=O.MODE_BRUTE):
        """the whole answer against the oracle under both caps; twin: also against a handle fully built from the same KV"""
        tt = np.zeros(len(topics), np.int32) if tt is None else np.asarray(tt, np.int32)
        kv = self.kv()
        other = None
        if twin:
            other = self.B.pkg.GpuRouteIndex(0)
            other.load_pairs(sorted(self.live.items()))
            other.commit()
        total = 0
        for caps in CAPS:
            offsets, ranks, ev = self.answer(self.idx, tenants, topics, tt, caps)
            want = kv.match_batch(tenants, topics, tt, caps[0], caps[1], mode)
            assert offsets.tolist() == want.offsets.tolist()
            assert ranks.tolist() == want.ranks.tolist()
            assert ev == sorted((k, t, r) for k, t, r, _ in want.events)
            if other is not None:
                o2, r2, e2 = self.answer(other, tenants, topics, tt, caps)
                assert o2.tolist() == offsets.tolist() and r2.tolist() == ranks.tolist() and e2 == ev
            total += len(ranks)
        if other is not None:
            other.close()
        return total


def devices(B, tenant, names, fmt="%s/state", broker=0):
    """one subscriber per name (receiver r<position>); broker None: subBrokerId = position % 3"""
    return [route(tenant, fmt % nm, i, broker if broker is not None else i % 3) for i, nm in enumerate(names)]


# ------------------------------------------------------------------ the random SUB / UNSUB stream
@pytest.mark.parametrize("seed", [31, 32])
def test_random_stream_with_wide_nodes(B, seed):
    """25 rounds of adds, overwrites, deletes, a vanishing and returning tenant, $share groups and persistent routes on an
    index whose tenants have wide nodes at the root, below an exact parent and below a '+'. Every commit is a delta; its
    answers equal the oracle's and a fully built twin's; results taken before a commit still resolve against their snapshot."""
    rng = random.Random(seed)
    pairs, tenants, topics, tt = random_pairs(B, rng, 500, ["a", "b", "c", "dd", "e1"], 5)
    pool, _, _, _ = random_pairs(B, random.Random(seed + 100), 700, ["a", "b", "c", "dd", "e1", "zz"], 5)
    all_pairs = dict(pairs)
    # an untouched tenant of 30k filters (about 3e5 slots): the regions the 25 rounds replace stay below the garbage bound
    all_pairs.update(route("pad", "a%03d/b%03d" % (i // 100, i % 100), i) for i in range(30_000))
    for i in range(1500):   # wide at the root of "tW" (one persistent subscriber per device), below "w" in tA, below '+' in t
        all_pairs.update([route("tW", "d%05d/state" % i, i, 1), route("tA", "site/w/c%05d" % i, i, i % 3), route("t", "+/p%05d" % i, i)])
    for g in range(3):
        members = {B.schema.receiver_url(g % 2, "m%d" % j, "d"): j for j in range(3)}
        all_pairs[B.schema.route_key("tW", "$share/g%d/d%05d/state" % (g, 7 * g))] = B.schema.route_group_bytes(members)
    L = Live(B, all_pairs.items())
    tenants = tenants + ["tW"]
    dev_topics = ["d%05d/state" % i for i in (0, 1, 7, 14, 777, 1499, 1500, 1501, 1600, 9999)]
    wtopics = ["site/w/c%05d" % i for i in (0, 3, 1499, 1500, 1700)] + ["x/p%05d" % i for i in (0, 5, 1499, 1650)]
    topics = list(topics[:120]) + dev_topics + wtopics
    tt = list(tt[:120]) + [3] * len(dev_topics) + [0] * 5 + [2] * 4
    st0 = L.idx.stats()
    assert st0["tag_used_slots"] >= 4500 and st0["full_commits"] == 1
    held = []
    pad = B.schema.tenant_begin_key("pad")
    for rnd in range(25):
        adds, dels = [], []
        mutable = sorted(k for k in L.live if not k.startswith(pad))
        for _ in range(rng.randint(1, 5)):
            r = rng.random()
            if r < 0.3:
                adds.append(rng.choice(pool))
            elif r < 0.5:   # a new device / child in one of the wide nodes
                i = rng.randint(1500, 1700)
                adds.append(rng.choice([route("tW", "d%05d/state" % i, i, 1), route("tA", "site/w/c%05d" % i, i, 0),
                                        route("t", "+/p%05d" % i, i)]))
            elif r < 0.6:   # overwrite the value of a live route
                k = rng.choice(mutable)
                adds.append((k, B.schema.incarnation_bytes(rng.randint(100, 200)) if len(L.live[k]) == 8 else L.live[k]))
            elif r < 0.7:   # a shared subscription joins a wide tenant
                members = {B.schema.receiver_url(rng.randint(0, 1), "m%d" % rng.randint(0, 9), "d"): 1}
                adds.append((B.schema.route_key("tW", "$share/h%d/d%05d/state" % (rnd, rng.randint(0, 1600))),
                             B.schema.route_group_bytes(members)))
            else:
                dels.append(rng.choice(mutable))
        if rnd == 10:   # a tenant vanishes; pool routes may bring it back later
            dels += [k for k in L.live if b"\x00\x02tB" in k[:6]]
        if rnd == 17:   # a wide tenant loses every device of a range, and its whole '+' node shrinks
            dels += [k for k in L.live if b"\x00\x02tW" in k[:6] and b"d010" in k]
        L.apply(adds, dels)
        res_old = L.idx.match_topics(tenants, topics[:60], np.asarray(tt[:60], np.int32))
        o_old, r_old = res_old.expand()
        keys_old = [res_old.route(int(x))[0] for x in r_old[:40]]
        assert L.commit() == "delta", rnd
        assert L.check(tenants, topics, tt, twin=rnd % 5 == 4) > 0
        assert [res_old.route(int(x))[0] for x in r_old[:40]] == keys_old
        held.append(res_old)
        if len(held) > 3:
            held.pop(0).close()
        st = L.idx.stats()
        assert st["routes"] == len(L.live) and st["tag_usable_slots"] == st0["tag_usable_slots"]
    for r in held:
        r.close()
    L.check(tenants, topics, tt, twin=True)
    L.idx.close()


# ------------------------------------------------------------------ rank shifts and the duplicate-key trap
def test_sub_before_a_wide_tenant_shifts_its_tag_table_records(B):
    """a SUB / UNSUB into a tenant that sorts before a wide tenant moves the wide tenant's ranks: its records in the tag table
    (root-level wide edges, and wide edges below an exact parent) must move with them"""
    names = ["d%05d" % i for i in range(2000)]
    pairs = devices(B, "w2", names) + [route("w2", "x/c%05d/y" % i, i, 1) for i in range(1200)] + [route("w2", "+/state", 0, 1)]
    pairs += [route("a", "a/b", i) for i in range(5)]
    L = Live(B, pairs)
    topics = ["%s/state" % n for n in names[::97]] + ["x/c%05d/y" % i for i in (0, 600, 1199, 1200)] + ["d99999/state"]
    tenants, tt = ["a", "w2"], [1] * (len(names[::97]) + 5)
    before = L.check(tenants, topics, tt)
    for adds, dels in (([route("a", "a/%d" % i, i) for i in range(7)], []), ([], [route("a", "a/b", i)[0] for i in range(5)]),
                       ([route("a", "z", 0)], [])):
        L.apply(adds, dels)
        assert L.commit() == "delta"
        assert L.check(tenants, topics, tt) == before   # the same routes, at ranks moved by the growth of "a"


def test_rebuilt_wide_tenant_keeps_its_ordinal_and_no_stale_entry_is_found(B):
    """a rebuilt tenant keeps its ordinal, so its root-level wide edges come back with the very same keys: the stale entries
    of the replaced tenant must not be found. A device that sorts first moves every other device's rank by one, and removed
    devices must match nothing."""
    names = ["d%05d" % i for i in range(1500)]
    L = Live(B, devices(B, "w", names) + [route("s", "q", 0)])
    topics = ["%s/state" % n for n in names[::50]] + ["c00000/state", "d00003/state"]
    tenants, tt = ["w", "s"], [0] * (len(names[::50]) + 2)
    L.apply([route("w", "c00000/state", 0)])
    assert L.commit() == "delta"
    L.check(tenants, topics, tt)
    L.apply([], [route("w", "%s/state" % n, i, 0)[0] for i, n in enumerate(names[:200])])
    assert L.commit() == "delta"
    assert L.check(tenants, topics, tt, twin=True) > 0
    off, ranks, _ = L.answer(L.idx, tenants, ["d00003/state", "d00150/state"], np.zeros(2, np.int32), CAPS[0])
    assert off.tolist() == [0, 0, 0]


def test_node_kind_changes_across_deltas(B):
    """a node grows from a perfect-hash array into the tag table (300 -> 1500 children) and shrinks back, each step a delta;
    the kind is read from bfq_host_build_stats on the same KV (slot 19 counts the tenants with wide edges)"""
    other = devices(B, "other", ["o%05d" % i for i in range(4000)])
    small = [route("t", "a/b/n%05d" % i, i) for i in range(300)] + [route("t", "a/+/x", 0, 1)]
    grow = [route("t", "a/b/n%05d" % i, i) for i in range(300, 1500)]
    L = Live(B, other + small)
    topics = ["a/b/n%05d" % i for i in (0, 299, 300, 1499, 1500)] + ["a/q/x"]
    tenants, tt = ["t", "other"], [0] * 6
    assert host_stats(list(L.live.items()))[19] == 1
    for adds, dels, wide in ((grow, [], 2), ([], [k for k, _ in grow], 1), (grow, [], 2)):
        L.apply(adds, dels)
        assert L.commit() == "delta"
        assert host_stats(list(L.live.items()))[19] == wide
        L.check(tenants, topics, tt, twin=True)


# ------------------------------------------------------------------ the fallback rules at their bounds
def wide_index(B, names):
    """an index whose only wide node is the root of tenant "w" (ordinal 0: the shortest id sorts first)"""
    return Live(B, devices(B, "w", names, fmt="%s") + [route("s1", "a/b", 0), route("s2", "+/x", 1, 1)])


def test_tag_table_fill_bound(B):
    """the commit that leaves exactly 3/4 of the usable tag slots claimed is a delta, the one past it is a full build (which
    sizes a new table at load 0.5); stats 18..20 follow the model of the table after every commit"""
    names = ["d%05d" % i for i in range(1500)]
    L = wide_index(B, names)
    model = TagModel(len(names))
    ovf = model.place(names, 0)
    st = L.idx.stats()
    assert (st["tag_usable_slots"], st["tag_used_slots"], st["tag_overflowed_blocks"]) == (model.usable, 1500, ovf)
    bound = 3 * model.usable // 4
    steps = [bound - 100 - len(names), 99, 1, 1]   # up to one below the bound, onto it, one past it, then one more
    seen = []
    for n in steps:
        new = ["d%05d" % i for i in range(len(names), len(names) + n)]
        names += new
        L.apply(devices(B, "w", new, fmt="%s"))
        trial = TagModel(0)
        trial.n_blocks, trial.usable, trial.overflowed = model.n_blocks, model.usable, set(model.overflowed)
        want = model.path(len(names), trial.place(names, 0))
        if want == "full":
            model = TagModel(len(names))
            ovf = model.place(names, 0)
        else:
            model, ovf = trial, len(trial.overflowed)
        got = L.commit()
        assert got == want, (len(names), bound)
        seen.append((len(names), got))
        st = L.idx.stats()
        assert (st["tag_usable_slots"], st["tag_used_slots"], st["tag_overflowed_blocks"]) == (model.usable, len(names), ovf)
        L.check(["w"], [names[0], names[-1], names[len(names) // 2], "d99999"])
    assert seen[1:] == [(bound - 1, "delta"), (bound, "delta"), (bound + 1, "full")]
    assert L.idx.stats()["tag_usable_slots"] > 15 * 200


def test_tag_table_overflow_bound(B):
    """children whose home blocks are chosen (from the model's hash) to overflow one more block per commit: the commit that
    leaves a quarter of the blocks overflowed is a delta, the next one is a full build, which resets the overflow bytes"""
    names = ["d%05d" % i for i in range(1500)]
    L = wide_index(B, names)
    model = TagModel(len(names))
    model.place(names, 0)
    nb = model.n_blocks
    from test_host_wide_delta_cpu import home_block, ROOT_BASE
    cands = {}
    for i in range(200000):
        nm = "o%05d" % i if i < 100000 else "p%05d" % (i - 100000)
        cands.setdefault(home_block(nm, ROOT_BASE, nb), []).append(nm)
    seen = []
    target = 0
    while True:
        # enough new children homed at the next block that is not overflowed yet to overflow it
        while target in model.overflowed:
            target += 1
        new = cands[target][:16]
        cands[target] = cands[target][16:]
        trial = TagModel(0)
        trial.n_blocks, trial.usable, trial.overflowed = nb, model.usable, set(model.overflowed)
        ovf = trial.place(names + new, 0)
        want = model.path(len(names) + len(new), ovf)
        assert 4 * (len(names) + len(new)) <= 3 * model.usable   # only the overflow rule can trip here
        names += new
        L.apply(devices(B, "w", new, fmt="%s"))
        got = L.commit()
        assert got == want, (ovf, nb)
        seen.append((ovf, got))
        st = L.idx.stats()
        if got == "full":
            fresh = TagModel(len(names))
            assert (st["tag_usable_slots"], st["tag_overflowed_blocks"]) == (fresh.usable, fresh.place(names, 0))
            break
        model = trial
        assert st["tag_overflowed_blocks"] == ovf and st["tag_used_slots"] == len(names)
    L.check(["w"], names[::37] + ["o99999x"])
    deltas = [o for o, p in seen if p == "delta"]
    assert deltas and 4 * deltas[-1] <= nb < 4 * seen[-1][0]


# ------------------------------------------------------------------ concurrency and the fan-out's deliverer ids
def test_matches_in_flight_while_wide_deltas_land(B):
    """several threads match while the main thread commits wide deltas; every result equals the oracle's answer for the
    generation it reports"""
    names = ["d%05d" % i for i in range(2000)]
    L = Live(B, devices(B, "w", names, fmt="%s", broker=None) + [route("a", "q/+", 0, 1)])
    topics = names[::40] + ["d02100", "d02200", "q/z"]
    tenants = ["w", "a"]
    tt = np.array([0] * (len(topics) - 1) + [1], np.int32)
    expected = {}
    got = []
    stop = threading.Event()
    errors = []

    def snapshot_answer():
        kv = L.kv()
        want = kv.match_batch(tenants, topics, tt, 4, 4, O.MODE_BRUTE)
        expected[L.idx.generation()] = (want.offsets.tolist(), want.ranks.tolist())

    def worker():
        try:
            while not stop.is_set():
                res = L.idx.match_topics(tenants, topics, tt, [4, 4], [4, 4])
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
        for rnd in range(12):
            i = 2000 + 10 * rnd
            gone = rnd * 7   # devices() gave it receiver r<gone> and subBrokerId gone % 3
            L.apply(devices(B, "w", ["d%05d" % j for j in range(i, i + 10)], fmt="%s", broker=None),
                    [route("w", names[gone], gone, gone % 3)[0]])
            assert L.commit() == "delta"
            snapshot_answer()
    finally:
        stop.set()
        for t in threads:
            t.join()
    assert not errors, errors
    assert len(got) > 12 and len({g for g, _, _ in got}) > 1
    for gen, o, r in got:
        assert (o, r) == expected[gen], gen


def test_fanout_deliverer_ids_stable_across_wide_deltas(B):
    """bfq_fanout_device on results of successive wide deltas: the (subBrokerId, delivererKey) -> id map only grows"""
    from test_gpu_fanout import fan_check, match_device, oracle
    names = ["d%05d" % i for i in range(1500)]
    pairs = []
    for i, n in enumerate(names):
        url = B.schema.receiver_url(i % 3, "r%d" % i, "inbox%d" % (i % 40))
        pairs.append((B.schema.route_key("w", n, url), B.schema.incarnation_bytes(1)))
    members = {B.schema.receiver_url(0, "m%d" % j, "inbox%d" % j): 1 for j in range(5)}
    pairs.append((B.schema.route_key("w", "$share/g/+"), B.schema.route_group_bytes(members)))
    L = Live(B, pairs)
    topics = names[::11] + ["d01600", "d01601"]
    tenants, tt = ["w"], np.zeros(len(topics), np.int32)
    ids = {}
    for rnd in range(4):
        out = match_device(B, L.idx, tenants, topics, tt)
        want = oracle(sorted(L.live.items()), tenants, topics, tt)
        _, s = fan_check(B, L.idx, out, topics, want, sorted(L.live.items()))
        out.release()
        for k, d in s["ids"].items():
            assert ids.setdefault(k, d) == d
        url = B.schema.receiver_url(1, "new%d" % rnd, "inbox-new%d" % rnd)
        L.apply([(B.schema.route_key("w", "d%05d" % (1600 + rnd), url), B.schema.incarnation_bytes(1))],
                [pairs[rnd * 13][0]])
        assert L.commit() == "delta"


# ------------------------------------------------------------------ full size
def test_full_size_c4_plus_100k_iot_tenant(B):
    """C4 at scale 1.0 plus a tenant of 100 000 devices (dev/<id>/state, dev/+/state, dev/#): delta commits into the IoT
    tenant and into a small C4 tenant, each a delta, each with every topic of a 100k-topic slice equal to the oracle"""
    import os
    from bifromq_b200 import workload
    w = workload.Workload("C4")
    iot = "iot-tenant-with-a-name-longer-than-any-c4-tenant"
    ipairs = devices(B, iot, ["dev/%06d" % i for i in range(100_000)], broker=None)
    ipairs += [route(iot, "dev/+/state", 0, 1), route(iot, "dev/#", 1, 1)]
    ipairs.sort()
    idx = B.pkg.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    from bifromq_b200 import _native as N
    ik, iko = N.as_blob([k for k, _ in ipairs])
    iv, ivo = N.as_blob([v for _, v in ipairs])
    idx.load(ik, iko, iv, ivo)
    idx.commit()
    kv = O.KV()
    kv.load(w.keys, w.key_off, w.vals, w.val_off)
    for k, v in ipairs:
        kv.put(k, v)
    names = w.tenants + [iot]
    st0 = idx.stats()
    assert st0["tag_used_slots"] >= 100_000 and st0["tenants"] == len(names)
    muts = [route(iot, "dev/%06d/state" % 100_001, 7, 1), route(names[len(names) // 3], "delta/+/x", 3),
            route(iot, "dev/000000/extra", 8)]
    for k, v in muts:
        idx.apply(adds=[(k, v)])
        kv.put(k, v)
        before = idx.stats()
        idx.commit()
        after = idx.stats()
        assert after["delta_commits"] == before["delta_commits"] + 1 and after["full_commits"] == before["full_commits"]
    kv.freeze()
    tenants = idx.tenant_blob(names)
    tb, toff = O.blob(names)
    lo, hi = 200_000, 250_000
    itopics = ["dev/%06d/state" % i for i in range(0, 100_002, 2)]
    ctopics = [w.topic(i) for i in range(lo, hi)]
    blob, off = O.blob(ctopics + [t.encode() for t in itopics])
    tt = np.concatenate([w.topic_tenant[lo:hi].astype(np.int32), np.full(len(itopics), len(names) - 1, np.int32)])
    assert len(tt) >= 100_000
    nt = len(names)
    threads = os.cpu_count() or 8
    for caps in CAPS:
        r = idx.match(tenants, blob, off, tt, [caps[0]] * nt, [caps[1]] * nt)
        offsets, ranks = r.expand()
        r.close()
        want = kv.match_blobs(tb, toff, blob, off, tt, len(tt), caps[0], caps[1], O.MODE_TRIE, False, threads)
        assert np.array_equal(offsets, want.offsets) and np.array_equal(ranks, want.ranks)
    idx.close()
