"""Long mixed commit streams for the forward index, generated in plain Python: the generator the GPU stream test
(tests/test_gpu_commit_streams.py) feeds a handle with, and the checks that it is what it claims to be, without a GPU.

A stream is seeded. It keeps the live KV (a dict) and the oracle KV built from it, and every round is one apply + commit of
one kind:
  a  1-4 SUBs / UNSUBs into 1-3 small tenants: normal, $share and $oshare routes, filters with empty levels;
  b  value-only changes: a new incarnation of a normal route or a new member list of a group; one round empties a $share
     group and a later one gives it members back, one adds a member to an $oshare group that wins a fixed publisher;
  c  one SUB into each of k >= 64 small tenants;
  d  the grower tenant "wg" grows past the wide-node threshold (its root children move to the shared tag table), then past
     the tag table's fill bound, then shrinks below the threshold;
  e  a small tenant is removed entirely, and recreated in a later round;
  f  routes through new (subBrokerId, delivererKey) pairs appear, and every route of one deliverer disappears;
  g  reset + reload of the whole live set;
  h  an empty commit.
The generator predicts each round's path (delta, full build, or nothing for the empty commit), the number of tenants it
rebuilds and the tag table's claimed and overflowed slots. The tag table is modelled with trie_hash.TagModel, extended to
several wide tenants: a full build claims every wide tenant's root children in key order into a table of n_blocks_for(edges)
blocks; a delta frees the rebuilt tenants' slots and claims their new edges into a copy of the table, and is a full build
instead when the fill or overflow rule of TagModel.path says so. Root ordinals follow the builder: key order on a full build,
appended for a tenant a delta creates (so a recreated tenant comes back at another ordinal)."""
import copy
import random

import numpy as np
import pytest

import delivery_wire as DW
import oracle_lib as O
import rendezvous_hash as RH
import test_gpu_edges as E
from trie_hash import ROOT_BASE, TAG_CTRL, TagModel, chunks

INT_MAX, I64_MAX = 2 ** 31 - 1, 2 ** 63 - 1
WIDE_MIN, NARROW_MAX = 1100, 400   # a root with >= 1100 exact children is wide, one with <= 400 gets a perfect hash
W0_CHILDREN, WG_START, WG_GROW = 3000, 300, 1150
SMALL = ["s%03d" % i for i in range(70)]
BATCH_SMALL = SMALL[:12]   # the small tenants the fixed batch queries
VOCAB = ["a", "b", "x", "", "lv-longer-than-twenty-four-bytes"]
FIXED_PUBLISHER = 0   # the first publisher of every position hashes to 0 (test_gpu_delivery_oshare.publishers)
SEEDS = [1, 2, 3]
N_ROUNDS = 40
KINDS = "abcdefgh"


# ------------------------------------------------------------------ routes
def normal(tenant, tf, broker, rid, dkey, inc=1):
    return O.route_key(tenant, tf, O.receiver_url(broker, rid, dkey)), O.incarnation_bytes(inc)


def group_key(tenant, tf, name, ordered=False):
    return O.route_key(tenant, ("$oshare/" if ordered else "$share/") + name + "/" + tf)


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


def members(rng, n, tag):
    return {O.receiver_url(rng.choice([0, 1, 2]), "%s%d" % (tag, j), "dm%d" % rng.randint(0, 5)): rng.randint(0, 9)
            for j in range(n)}


def random_route(rng, tenant, tag):
    """a normal route (60 %), a $share group (20 %) or an $oshare group (20 %) on a random filter"""
    f, r = random_filter(rng), rng.random()
    if r < 0.6:
        return normal(tenant, f, rng.choice([0, 1, 1, 2]), "r%s" % tag, "d%d" % rng.randint(0, 5), rng.randint(0, 99))
    ordered = r >= 0.8
    return group_key(tenant, f, "g%d" % rng.randint(0, 3), ordered), O.route_group(members(rng, rng.randint(1, 3), tag))


def wide_names(n):
    return ["c%05d" % i for i in range(n)]


WIDE_KEY_NAME = {}   # route key -> root child name, for the routes of the two tenants that can be wide


def wide_route(tenant, i):
    k, v = normal(tenant, "c%05d" % i, i % 3, "r%d" % i, "d%s%d" % (tenant, i % 5))
    WIDE_KEY_NAME[k] = "c%05d" % i
    return k, v


OG_KEY = ("s001", "x/+", "og")   # an $oshare group whose winner for the fixed publisher a b round changes
EG_KEY = ("s001", "x/#", "eg")   # a $share group a b round empties and a later one fills again
X1_ROUTE = ("s001", "x/1", 0, "x1", "d0")   # a normal route the fixed batch matches, whose incarnation a b round changes


def start_pairs(rng):
    kv = {}
    kv.update(wide_route("w0", i) for i in range(W0_CHILDREN))
    kv.update(wide_route("wg", i) for i in range(WG_START))
    kv.update(normal("pad", "p%03d/q%03d" % (i // 100, i % 100), 0, "z%d" % i, "dp") for i in range(12000))
    kv.update(E.make_pairs(E.one_route_each("tier", E.TIER2_FILTERS + ["b/#", E.TIER1_TOPIC, "b/+"]) + E.spill_filters("tier")))
    for t in SMALL:
        for j in range(rng.randint(3, 8)):
            kv.update([random_route(rng, t, "%s_%d" % (t, j))])
    kv[group_key(*OG_KEY, ordered=True)] = O.route_group({O.receiver_url(j % 3, "o%d" % j, "do%d" % j): 1 for j in range(3)})
    kv[group_key(*EG_KEY)] = O.route_group({O.receiver_url(0, "e0", "d1"): 1, O.receiver_url(1, "e1", "d2"): 2})
    kv.update([normal(*X1_ROUTE)])
    return kv


def _tenant(key):
    """the tenant id of a route key: <version byte><u16 big-endian length><tenant id>..."""
    n = int.from_bytes(key[1:3], "big")
    return key[3:3 + n].decode()


def tenant_order(tenants):
    return sorted(tenants, key=O.tenant_begin_key)


def oracle_of(live):
    """the oracle KV of a live set"""
    pairs = sorted(live.items())
    kv = O.KV()
    k, ko = O.blob([p[0] for p in pairs])
    v, vo = O.blob([p[1] for p in pairs])
    kv.load(k, ko, v, vo)
    kv.freeze()
    return kv


# ------------------------------------------------------------------ the tag table of several wide tenants
class StreamTags(TagModel):
    """TagModel's table holding the root children of several wide tenants, with each tenant's claimed slots"""

    def __init__(self, wide, ordinals):
        """a full build: every wide tenant's children claimed, tenants in key order"""
        super().__init__(sum(len(v) for v in wide.values()))
        self.slots = {}
        for t in tenant_order(wide):
            self.place_tenant(t, wide[t], ordinals[t])

    def place_tenant(self, tenant, names, ordinal):
        self.slots[tenant] = [self.claim(ROOT_BASE + ordinal, *chunks(nm)[0])[0] for nm in sorted(names)]

    def used(self):
        return sum(len(s) for s in self.slots.values())

    def n_overflowed(self):
        return int((self.tags[:, TAG_CTRL] != 0).sum())

    def delta(self, touched, wide, ordinals):
        """the table after a delta commit that rebuilds `touched` (wide: the wide tenants after it), or None where the fill or
        overflow rule makes the commit a full build"""
        t = copy.deepcopy(self)
        for x in touched:
            for s in t.slots.pop(x, []):
                t.release(s)
        for x in tenant_order(touched):
            if x in wide:
                t.place_tenant(x, wide[x], ordinals[x])
        return None if t.path(t.used(), t.n_overflowed()) == "full" else t


# ------------------------------------------------------------------ the stream
class Round:
    def __init__(self, index, kind, label):
        self.index, self.kind, self.label = index, kind, label
        self.adds, self.dels, self.reset = [], [], False
        self.path = self.rebuilt = self.tag_used = self.tag_overflowed = self.tag_usable = None
        self.ordinals = None


def schedule(rng, n):
    kinds = list("ab" * 5 + "a" * 3 + "ccc" + "fff" + "hh" + "g") + ["e-", "e+", "d1", "d2", "d3"]
    kinds += ["a"] * (n - len(kinds))
    rng.shuffle(kinds)
    for group in (["e-", "e+"], ["d1", "d2", "d3"]):   # in order, wherever the shuffle put them
        pos = sorted(i for i, k in enumerate(kinds) if k in group)
        for p, k in zip(pos, group):
            kinds[p] = k
    b = [i for i, k in enumerate(kinds) if k == "b"]
    labels = {b[0]: "b-empty", b[1]: "b-winner", b[2]: "b-refill", b[3]: "b-incarnation"}
    return [labels.get(i, k) for i, k in enumerate(kinds)]


class Stream:
    """one seeded stream: iterate rounds() to get each Round after the live set has moved to its state"""

    def __init__(self, seed, n_rounds=N_ROUNDS):
        self.seed, self.n_rounds = seed, n_rounds
        self.rng = random.Random(seed)
        self.live = start_pairs(self.rng)
        self.labels = schedule(self.rng, n_rounds)
        self.removed = None
        self.new_deliverers = []
        self._full_build()

    # -- the index state the generator predicts
    def tenants(self):
        return {_tenant(k) for k in self.live}

    def wide(self):
        out = {}
        for t in ("w0", "wg"):
            names = {WIDE_KEY_NAME[k] for k in self.live if k in WIDE_KEY_NAME and _tenant(k) == t}
            assert not NARROW_MAX < len(names) < WIDE_MIN, (t, len(names))
            if len(names) >= WIDE_MIN:
                out[t] = sorted(names)
        return out

    def _full_build(self):
        order = tenant_order(self.tenants())
        self.ordinals = {t: i for i, t in enumerate(order)}
        self.n_roots = len(order)
        self.tags = StreamTags(self.wide(), self.ordinals)

    def pairs(self):
        return sorted(self.live.items())

    def oracle(self):
        return oracle_of(self.live)

    # -- rounds
    def rounds(self):
        for i, label in enumerate(self.labels):
            r = Round(i, label[0], label)
            before = self.tenants()
            getattr(self, "_" + label.replace("-", "_").replace("+", "_back"))(r)
            touched = {_tenant(k) for k, _ in r.adds} | {_tenant(k) for k in r.dels}
            for k, v in r.adds:
                self.live[k] = v
            for k in r.dels:
                del self.live[k]
            after = self.tenants()
            if r.kind == "h":
                assert not touched
                r.path, r.rebuilt = "none", 0
            elif r.reset:
                r.path = "full"
            else:
                ords = dict(self.ordinals)
                n_roots = self.n_roots
                for t in after - before:
                    assert t in touched
                for t in tenant_order(after - set(ords)):   # a delta appends the root of every tenant it creates
                    ords[t] = n_roots
                    n_roots += 1
                for t in before - after:
                    del ords[t]
                tags = self.tags.delta(touched, self.wide(), ords)
                if tags is None:
                    r.path = "full"
                else:
                    r.path, r.rebuilt = "delta", len(touched & after)
                    self.tags, self.ordinals, self.n_roots = tags, ords, n_roots
            if r.path == "full":
                self._full_build()
                r.rebuilt = len(after)
            r.tag_used, r.tag_overflowed, r.tag_usable = self.tags.used(), self.tags.n_overflowed(), self.tags.usable
            r.ordinals = dict(self.ordinals)
            yield r

    def _small_alive(self):
        alive = self.tenants()
        return [t for t in SMALL if t in alive]

    def _keys_of(self, tenant):
        return sorted(k for k in self.live if _tenant(k) == tenant)

    def _a(self, r):
        rng = self.rng
        fixed = (group_key(*OG_KEY, ordered=True), group_key(*EG_KEY), normal(*X1_ROUTE)[0])
        for t in rng.sample(self._small_alive(), rng.randint(1, 3)):
            for j in range(rng.randint(1, 2)):
                keys = [k for k in self._keys_of(t) if k not in r.dels and k not in fixed]
                if rng.random() < 0.35 and len(keys) > 1:   # an UNSUB that leaves the tenant alive
                    r.dels.append(rng.choice(keys))
                    continue
                k, v = random_route(rng, t, "a%d_%d" % (r.index, j))
                if k not in self.live:
                    r.adds.append((k, v))
        if not r.adds and not r.dels:
            r.adds.append(normal(SMALL[0] if SMALL[0] in self.tenants() else "s001", "a//b", 1, "ra%d" % r.index, "d3"))

    def _b(self, r):
        """new values for keys that stay: incarnations of normal routes, member lists of groups"""
        rng = self.rng
        for t in rng.sample(self._small_alive(), rng.randint(1, 3)):
            for k in rng.sample(self._keys_of(t), 1):
                if k in (group_key(*OG_KEY, ordered=True), group_key(*EG_KEY)):
                    continue
                v = self.live[k]
                if O.build_match_route(k, v)["type"] == "Normal":
                    r.adds.append((k, O.incarnation_bytes(1000 + r.index)))
                else:
                    r.adds.append((k, O.route_group(members(rng, rng.randint(1, 4), "b%d_" % r.index))))
        if not r.adds:
            k = group_key(*OG_KEY, ordered=True)
            r.adds.append((k, self.live[k]))   # the same list in a fresh value: the tenant is rebuilt all the same

    def _b_empty(self, r):
        r.adds.append((group_key(*EG_KEY), O.route_group({})))

    def _b_refill(self, r):
        r.adds.append((group_key(*EG_KEY), O.route_group({O.receiver_url(2, "e%d" % j, "dE%d" % j): j for j in range(3)})))

    def _b_incarnation(self, r):
        """the same key, a new incarnation: only the route's MatchInfo changes"""
        k = normal(*X1_ROUTE)[0]
        r.adds.append((k, O.incarnation_bytes(500 + r.index)))

    def _b_winner(self, r):
        k = group_key(*OG_KEY, ordered=True)
        urls = O.route_group_members_in_wire_order(self.live[k])
        best = max(RH.score(FIXED_PUBLISHER, u) for u in urls)
        j = 0
        while RH.score(FIXED_PUBLISHER, O.receiver_url(1, "win%d" % j, "dWin")) <= best:
            j += 1
        new = {u: 1 for u in urls}
        new[O.receiver_url(1, "win%d" % j, "dWin")] = 1
        r.adds.append((k, O.route_group(new)))
        r.winner = (urls, list(new))

    def _c(self, r):
        rng = self.rng
        alive = self._small_alive()
        for i, t in enumerate(rng.sample(alive, rng.randint(64, len(alive)))):
            r.adds.append(normal(t, random_filter(rng), rng.choice([0, 1, 2]), "c%d_%d" % (r.index, i), "d%d" % (i % 6), i))

    def _d1(self, r):   # past the wide-node threshold
        have = len(self.wide().get("wg", [])) or WG_START
        r.adds += [wide_route("wg", i) for i in range(have, WG_GROW)]

    def _d2(self, r):   # one edge past the tag table's fill bound
        have = len(self.wide().get("wg", []))
        assert have >= WIDE_MIN
        need = 3 * self.tags.usable // 4 + 1 - self.tags.used()
        r.adds += [wide_route("wg", i) for i in range(have, have + need)]

    def _d3(self, r):   # below the threshold again
        keys = self._keys_of("wg")
        r.dels += keys[WG_START:]

    def _e_(self, r):
        rng = self.rng
        t = rng.choice([x for x in self._small_alive() if x in BATCH_SMALL and x not in ("s000", "s001")])
        self.removed = t
        r.dels += self._keys_of(t)

    def _e_back(self, r):
        t = self.removed
        for j in range(3):
            r.adds.append(random_route(self.rng, t, "e%d_%d" % (r.index, j)))
        r.adds.append(normal(t, "x/1", 1, "back%d" % r.index, "dBack"))

    def _f(self, r):
        rng = self.rng
        fresh = "nx%d" % r.index
        batch_alive = [x for x in self._small_alive() if x in BATCH_SMALL]
        for j in range(rng.randint(2, 4)):
            t = rng.choice(batch_alive)
            r.adds.append(normal(t, rng.choice(["x/1", "x/+", "a/#", "b"]), j % 3, "f%d_%d" % (r.index, j), fresh))
        if self.new_deliverers:
            gone = self.new_deliverers.pop(0)   # only normal routes go through the nx deliverers
            for k, v in self.live.items():
                m = O.build_match_route(k, v)
                if m["type"] == "Normal" and O.deliverer_of_receiver_url(m["receiverUrl"])[1] == gone.encode():
                    r.dels.append(k)
            r.gone = gone
        self.new_deliverers.append(fresh)

    def _g(self, r):
        r.reset = True

    def _h(self, r):
        pass


# ------------------------------------------------------------------ CPU checks of the generator
def summary(seed, n=N_ROUNDS):
    s = Stream(seed, n)
    return [(r.label, r.path, r.rebuilt, r.tag_used, r.tag_overflowed, r.tag_usable, sorted(r.adds), sorted(r.dels))
            for r in s.rounds()], s


@pytest.mark.parametrize("seed", SEEDS)
def test_stream_is_deterministic_per_seed(seed):
    a, sa = summary(seed)
    b, sb = summary(seed)
    assert a == b and sa.live == sb.live
    assert summary(seed + 100)[0] != a


@pytest.mark.parametrize("seed", SEEDS)
def test_every_round_kind_and_path_occurs(seed):
    s = Stream(seed)
    rounds = list(s.rounds())
    assert {r.kind for r in rounds} == set(KINDS)
    assert {"b-empty", "b-winner", "b-refill", "b-incarnation", "e-", "e+", "d1", "d2", "d3"} <= {r.label for r in rounds}
    paths = {p: sum(r.path == p for r in rounds) for p in ("delta", "full", "none")}
    assert paths["delta"] > 25 and paths["full"] >= 2 and paths["none"] == 2
    c = [r for r in rounds if r.kind == "c"]
    assert all(r.rebuilt >= 64 for r in c if r.path == "delta")
    # the removed tenant comes back at another root ordinal than it had
    rm = next(r for r in rounds if r.label == "e-")
    back = next(r for r in rounds if r.label == "e+")
    before = rounds[rm.index - 1].ordinals if rm.index else None
    t = s.removed
    assert t not in rm.ordinals and t in back.ordinals and (before is None or before[t] != back.ordinals[t])
    # the winner round's new member wins the fixed publisher
    w = next(r for r in rounds if r.label == "b-winner")
    old, new = w.winner
    assert RH.rendezvous_pick(FIXED_PUBLISHER, new) == len(new) - 1 != RH.rendezvous_pick(FIXED_PUBLISHER, old)


@pytest.mark.parametrize("seed", SEEDS)
def test_predicted_full_build_is_the_fill_bound_of_tag_model(seed):
    s = Stream(seed)
    prev = None
    for r in s.rounds():
        if r.label == "d2":
            # one edge past 3/4 of the usable slots of the table the previous round left
            assert r.path == "full"
            assert prev_tags.path(prev_tags.used() + len(r.adds), 0) == "full"
            assert 4 * (prev_tags.used() + len(r.adds) - 1) <= 3 * prev_tags.usable
            assert r.tag_used == prev_tags.used() + len(r.adds) and r.tag_usable > prev_tags.usable
        if r.label == "d1":
            assert r.tag_used >= W0_CHILDREN + WG_GROW or r.path == "full"
        if r.label == "d3":
            assert r.tag_used == W0_CHILDREN and r.path == "delta"
        if r.kind not in "dg" and r.path == "delta":
            assert r.tag_used == (prev.tag_used if prev else W0_CHILDREN)
        prev, prev_tags = r, copy.deepcopy(s.tags)


def batch_keys(live, batch):
    """the route keys the fixed batch matches (uncapped) on a live set"""
    keys = sorted(live)
    got = E.oracle_match(oracle_of(live), batch.tenants, batch.topics, batch.tt, INT_MAX, INT_MAX, O.MODE_TRIE)
    return {keys[r] for r in set(got.ranks.tolist())}


@pytest.mark.parametrize("seed", SEEDS)
def test_value_only_removal_and_deliverer_rounds_reach_the_fixed_batch(seed):
    """a new incarnation of a normal route the batch matches (only its MatchInfo changes), the recreated tenant and the
    vanished deliverer's routes are all read by the fixed batch, so every consumer sees them"""
    s = Stream(seed)
    batch = fixed_batch(seed)
    prev = dict(s.live)
    seen = {"incarnation": 0, "recreated": 0, "vanished": 0}
    for r in s.rounds():
        if r.kind == "b":
            changed = [k for k, v in r.adds if k in prev and prev[k] != v and len(v) == 8]   # normal routes: 8-byte value
            if changed and set(changed) & batch_keys(s.live, batch):
                assert all(len(prev[k]) == 8 for k in changed) and not r.dels
                assert all(DW.route_match_infos(k, prev[k]) != DW.route_match_infos(k, self_v)
                           for k, self_v in r.adds if k in changed)   # the MatchInfo bytes change with the value
                seen["incarnation"] += 1
        if r.label == "e+":
            assert s.removed in batch.tenants
            seen["recreated"] += bool({k for k, _ in r.adds} & batch_keys(s.live, batch))
        if getattr(r, "gone", None):
            seen["vanished"] += bool(set(r.dels) & batch_keys(prev, batch))
        prev = dict(s.live)
    assert seen["incarnation"] >= 1 and seen["recreated"] == 1 and seen["vanished"] >= 1, seen


def test_short_stream_references_are_self_consistent():
    """the oracle equals the brute-force predicate, and the restatements agree where they cover the same pairs"""
    import test_gpu_caps as C
    import test_gpu_delivery as D
    import test_gpu_fanout as F
    import test_host_oshare_cpu as H
    s = Stream(7, n_rounds=12)
    batch = fixed_batch(11)
    for r in s.rounds():
        if r.index % 4 != 3:
            continue
        pairs = s.pairs()
        kv = s.oracle()
        world = C.World(pairs, C.decoded_kinds(pairs))
        uncapped = E.oracle_match(kv, batch.tenants, batch.topics, batch.tt, INT_MAX, INT_MAX, O.MODE_TRIE)
        filters = [O.build_match_route(k, v) for k, v in pairs]
        for i in range(0, len(batch.topics), 7):
            e = int(batch.tt[i])
            want = [] if not 0 <= e < len(batch.tenants) else [
                j for j, m in enumerate(filters) if m["tenantId"] == batch.tenants[e]
                and O.topic_matches_filter(batch.topics[i], m["mqttTopicFilter"].split("/", 2)[2]
                                           if m["type"] == "Group" else m["mqttTopicFilter"])]
            assert uncapped.routes(i).tolist() == want, (r.label, batch.topics[i])
        caps = C.caps_reference(world, batch.tenants, batch.topics, batch.tt, batch.max_p, batch.max_g)
        for e in range(len(batch.tenants)):   # one entry's caps applied by the oracle itself
            rows = np.flatnonzero(batch.tt == e)
            got = E.oracle_match(kv, [batch.tenants[e]], [batch.topics[i] for i in rows], np.zeros(len(rows), np.int32),
                                 batch.max_p[e], batch.max_g[e], O.MODE_TRIE)
            assert [got.routes(j).tolist() for j in range(len(rows))] == \
                [caps.ranks[caps.offsets[i]:caps.offsets[i + 1]].tolist() for i in rows]
        route_of = lambda x: F.decode(pairs, x)
        plain = D.batch_delivery(batch.tt, len(batch.tenants), caps.offsets, caps.ranks, route_of, lambda t, x: 0)
        flat = sorted((t, x) for pkgs in plain.values() for packs in pkgs.values() for t, ms in packs for x, _ in ms)
        topic = np.repeat(np.arange(len(batch.topics)), np.diff(caps.offsets))
        ok = (batch.tt[topic] >= 0) & (batch.tt[topic] < len(batch.tenants))
        assert flat == sorted(zip(topic[ok].tolist(), caps.ranks[ok].tolist()))
        no_pubs = np.zeros(len(batch.topics) + 1, np.int64)
        assert H.batch_delivery_ordered(batch.tt, len(batch.tenants), caps.offsets, caps.ranks, route_of, lambda t, x: 0,
                                        no_pubs, np.zeros(0, np.int32)) == \
            {d: {tn: [p + ((),) for p in packs] for tn, packs in pkgs.items()} for d, pkgs in plain.items()}


# ------------------------------------------------------------------ the fixed mixed batch
class Batch:
    pass


NO_TENANT = E.NO_TENANT
# (tenant, maxPersistentFanout, maxGroupFanout, MaxPersistentFanoutBytes, tenant bandwidth bits)
ENTRIES = [("s000", INT_MAX, INT_MAX, I64_MAX, 3), ("s001", 3, 2, 5000, 3), ("s002", INT_MAX, 1, I64_MAX, 1),
           ("s003", 2, INT_MAX, 300, 2), ("s004", 1, 1, 1, 0), ("s005", 4, 3, 2000, 3), ("s006", 0, 0, I64_MAX, 3),
           ("s007", INT_MAX, INT_MAX, 900, 3), ("s008", 5, INT_MAX, I64_MAX, 1), ("s009", INT_MAX, 2, 4000, 3),
           ("s010", 2, 2, I64_MAX, 3), ("s011", INT_MAX, INT_MAX, I64_MAX, 3), ("w0", 5, 5, 10 ** 6, 3),
           ("wg", INT_MAX, 2, 3000, 3), ("pad", 1, 0, I64_MAX, 3), ("tier", 40, 7, 50000, 3),
           ("s001", INT_MAX, INT_MAX, I64_MAX, 3), (NO_TENANT, INT_MAX, INT_MAX, I64_MAX, 3)]
SMALL_TOPICS = ["x/1", "x/2", "a/b", "a//b", "/a", "b", "x/a/b", "$sys/x", "lv-longer-than-twenty-four-bytes/x", "a/b/",
                "x//x", "b/lv-longer-than-twenty-four-bytes"]
TOPICS = {"w0": ["c00007", "c00299", "c01149", "c02999", "c03500", "$c"], "pad": ["p005/q007", "p119/q099", "p120/q000"],
          "tier": [E.TIER2_TOPIC, E.TIER1_TOPIC, "k1/a/b/c/d", "a/a", "b/b"]}
TOPICS["wg"] = TOPICS["w0"] + ["c01500", "c04000"]


def fixed_batch(seed, big=False):
    """every entry's topics, some twice, one position whose tenant index is outside the list; big: 33 000 more positions
    drawn from the light ones (> 32 768 topics: the match de-duplicates and orders them for locality)"""
    rng = np.random.default_rng(seed)
    tt, topics = [], []
    for e, (t, *_) in enumerate(ENTRIES):
        for tp in TOPICS.get(t, SMALL_TOPICS):
            tt.append(e)
            topics.append(tp)
    rep = rng.choice(len(topics), len(topics) // 3, replace=False)
    tt += [tt[i] for i in rep]
    topics += [topics[i] for i in rep]
    tt += [len(ENTRIES) + 2]
    topics.append("x/1")
    if big:
        light = [i for i in range(len(topics)) if topics[i] not in (E.TIER2_TOPIC, E.TIER1_TOPIC)]
        pick = rng.choice(light, 33000)
        tt += [tt[i] for i in pick]
        topics += [topics[i] for i in pick]
    order = rng.permutation(len(topics))
    b = Batch()
    b.tenants = [e[0] for e in ENTRIES]
    b.max_p, b.max_g = [e[1] for e in ENTRIES], [e[2] for e in ENTRIES]
    b.max_bytes, b.bw = [e[3] for e in ENTRIES], [e[4] for e in ENTRIES]
    b.topics = [topics[i] for i in order]
    b.tt = np.asarray([tt[i] for i in order], np.int32)
    b.sizes = rng.integers(0, 3001, len(topics))
    b.pub_counts = rng.integers(0, 4, len(topics)).tolist()
    return b


def test_fixed_batch_shape():
    b = fixed_batch(3)
    big = fixed_batch(3, big=True)
    assert len(big.topics) >= 32768 and len(b.topics) < 1000
    assert len(set(zip(b.tt.tolist(), b.topics))) < len(b.topics)                       # repeats
    assert any(t.startswith("$") for t in b.topics) and (b.tt >= len(b.tenants)).sum() == 1
    assert NO_TENANT in b.tenants and b.tenants.count("s001") == 2 and set(BATCH_SMALL) <= set(b.tenants)
    finite = {(p, g) for p, g in zip(b.max_p, b.max_g) if p != INT_MAX or g != INT_MAX}
    assert len(finite) >= 6
