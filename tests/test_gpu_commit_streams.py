"""Long mixed commit streams end to end: after every commit of a seeded stream (tests/test_host_commit_streams_cpu.py), one
fixed mixed batch runs through every consumer of a match and is checked against the suite's references, results of earlier
generations are re-run and must reproduce what they returned when taken, and a freshly built twin must agree.

Per round:
  * the path the generator predicted, through the stats() deltas: delta / full commits, rebuilt tenants, the tag table's
    usable, claimed and overflowed slots (an empty commit changes none of them and keeps the generation);
  * bfq_match and the device match + expand against caps_reference (per-entry caps), expand_budget with binding budgets
    against test_gpu_fanout_budget.expect, the fan-out on both passes against test_gpu_fanout.check, delivery and
    delivery_ordered against the restatements of test_gpu_delivery / test_gpu_delivery_oshare, both encoders with every slice
    decoded (test_gpu_delivery_wire.encode_check), route / route_kinds of the matched ranks against the KV, and
    Exchange(world=1).gather against the host result;
  * deliverer ids are compared through idx.deliverer(id): an id once seen names the same (subBrokerId, delivererKey) for
    the life of the handle, reset included;
  * the device results of the last four generations re-run the whole downstream chain: same CSR, budget outputs, fan-out
    map, nestings, requests (byte for byte up to the order of a pack's MatchInfos, which the nesting leaves unspecified) and
    route lookups; one round enqueues an async match before its commit;
  * every fifth round and at the end, a handle built from the live set: bfq_match arrays bit for bit, downstream outputs
    key for key (deliverers by (subBrokerId, delivererKey)).
"""
import numpy as np
import pytest

import delivery_wire as DW
import oracle_lib as O
import test_gpu_caps as C
import test_gpu_delivery as D
import test_gpu_delivery_oshare as S
import test_gpu_delivery_wire as W
import test_gpu_fanout as F
import test_gpu_fanout_budget as FB
import test_host_commit_streams_cpu as G

pytestmark = pytest.mark.gpu
HELD = 4
BIG_ROUNDS = (7, 23)        # rounds whose batch has > 32 768 topics
ASYNC_FROM = 5             # the first delta round from here on enqueues a device match before its commit
ORDERED = D.ORDERED


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


# ------------------------------------------------------------------ references of one generation
KIND_CACHE = {}


class World(C.World):
    """caps' World over the stream's live set, route kinds decoded once per key, the oracle KV the stream built"""

    def __init__(self, stream):
        self.pairs = stream.pairs()
        self.kv = stream.oracle()
        for k, v in self.pairs:
            if k not in KIND_CACHE or KIND_CACHE[k][0] != v:
                m = O.build_match_route(k, v)
                kind = C.GROUP if m["type"] == "Group" else C.PERSISTENT if m["subBrokerId"] == 1 else C.NORMAL
                f = m["mqttTopicFilter"]
                KIND_CACHE[k] = (v, kind, f, f.split("/", 2)[2] if f.startswith(("$share/", "$oshare/")) else f)
        self.kinds = np.array([KIND_CACHE[k][1] for k, _ in self.pairs], np.int8)
        self.filters = [KIND_CACHE[k][2] for k, _ in self.pairs]
        self.targets = [KIND_CACHE[k][3] for k, _ in self.pairs]


def budget_expect(world, batch):
    """FB.expect per tenant entry (its own uniform caps), merged back into batch positions"""
    x = FB.Expected()
    n = len(batch.topics)
    per = [None] * n
    x.flags, x.dp = np.zeros(n, np.uint8), np.zeros(n, np.int64)
    x.events, x.meter, x.drop = [], [], {"bytes": 0, "pbw": 0, "tbw": 0}
    nt = len(batch.tenants)
    groups = {}
    for i, e in enumerate(batch.tt.tolist()):
        groups.setdefault(e if 0 <= e < nt else -1, []).append(i)
    for e, rows in groups.items():
        ent = [] if e < 0 else [0]
        case = FB.Case(world.pairs, [batch.tenants[e]] if e >= 0 else [], [batch.topics[i] for i in rows],
                       np.zeros(len(rows), np.int32) if e >= 0 else np.full(len(rows), 5, np.int32),
                       batch.sizes[rows], [batch.max_bytes[e]] * len(ent), [batch.bw[e]] * len(ent),
                       (batch.max_p[e], batch.max_g[e]) if e >= 0 else (G.INT_MAX, G.INT_MAX))
        sub = FB.expect(case, world.kinds, world.kv)
        for j, i in enumerate(rows):
            per[i] = sub.sent[j]
            x.flags[i], x.dp[i] = sub.flags[j], sub.dp[j]
        x.meter += [(rows[j], m) for j, m in sub.meter]
        x.events += sub.events
        for k in x.drop:
            x.drop[k] += sub.drop[k]
    x.meter.sort()
    x.offsets = np.concatenate([[0], np.cumsum([len(s) for s in per])]).astype(np.int64)
    x.ranks = np.array([r for s in per for r in s], np.int64)
    return x


def budget_case(batch):
    return FB.Case(None, batch.tenants, batch.topics, batch.tt, batch.sizes, batch.max_bytes, batch.bw)


# ------------------------------------------------------------------ one batch through every consumer
class Taken:
    """a device result with everything its downstream chain was given, and what it returned"""


def take(B, idx, batch, wait=True):
    t = Taken()
    t.batch = batch
    t.out = C.match_device(B, idx, batch.tenants, batch.topics, batch.tt, batch.max_p, batch.max_g, wait=wait)
    t.res = idx.match_topics(batch.tenants, batch.topics, batch.tt, batch.max_p, batch.max_g)
    t.pub_off, t.pub_hash = S.publishers(batch.pub_counts, 1)
    sizes = [4, 13, 100, 127, 128] if len(batch.topics) > 10000 else None
    t.packs = W.publisher_packs(int(t.pub_off[-1]), 5, sizes)
    return t


def outputs(B, idx, t):
    """every downstream call on a completed result -> host copies (deliverer ids as the handle numbers them)"""
    torch, out, n = B.torch, t.out, len(t.batch.topics)
    d_off, d_ranks, total = F.device_csr(B, out, n)
    got = {"total": total}
    torch.cuda.synchronize()
    off, rk = d_off.cpu().numpy(), d_ranks.cpu().numpy()[:total]
    seg = np.repeat(np.arange(n), np.diff(off))
    got["csr"] = (off.tolist(), rk[np.lexsort((rk, seg))].tolist())
    bud = FB.budget(B, out, budget_case(t.batch))
    r = bud["r"]
    got["budget"] = (bud["offsets"].tolist(), sorted(F.pair_keys(np.repeat(np.arange(n), np.diff(bud["offsets"])),
                                                                  bud["ranks"]).tolist()),
                     bud["flags"].tolist(), bud["dp"].tolist(),
                     (r.n_dropped_bytes, r.n_dropped_persistent_bandwidth, r.n_dropped_transient_bandwidth))
    for path in (0, 1):
        idx.set_option("fanout_global", path)
        got["fan%d" % path] = F.fanout_once(B, out, d_off, d_ranks, total)
    idx.set_option("fanout_global", 0)
    d_tt = out.keep[2].data_ptr()
    blob, poff = O.blob(t.packs)
    d_pub_off, d_pp, d_pp_off = (W.upload(B, t.pub_off, np.int64), W.upload(B, blob, np.uint8), W.upload(B, poff, np.int64))
    d_hash = W.upload(B, t.pub_hash, np.int32)
    enc_args = (t.batch.tenants, out.keep[0].data_ptr(), out.keep[1].data_ptr(), d_pub_off.data_ptr(), d_pp.data_ptr(),
                d_pp_off.data_ptr())

    def encode(nest):
        nb = out.delivery_wire(nest, *enc_args, None, 0, B.stream).n_bytes
        buf = torch.zeros(max(nb, 1), dtype=torch.uint8, device=B.dev)
        wr = out.delivery_wire(nest, *enc_args, buf.data_ptr(), nb, B.stream)
        torch.cuda.synchronize()
        req = B.dist.device_view(wr.d_req_off, wr.n_deliverers + 1, "<i8", B.dev).cpu().numpy()
        data = buf.cpu().numpy().tobytes()[:nb]
        return decoded({d: data[req[d]:req[d + 1]] for d in range(wr.n_deliverers) if req[d + 1] > req[d]})
    dl = out.delivery(d_off.data_ptr(), d_ranks.data_ptr(), total, d_tt, B.stream)
    got["plain"] = dl.nesting(B.dev)
    got["plain_wire"] = encode(dl)
    od = out.delivery_ordered(d_off.data_ptr(), d_ranks.data_ptr(), total, d_tt, d_pub_off.data_ptr(), d_hash.data_ptr(),
                              len(t.pub_hash), B.stream)
    got["ordered"] = od.nesting(B.dev)
    got["ordered_wire"] = encode(od)
    got["ordered_id"] = dl.ordered_share_id
    sample = sorted(set(rk[::max(1, len(rk) // 300)].tolist()) | set(rk[-3:].tolist()))
    got["routes"] = [t.res.route(x) for x in sample]
    got["kinds"] = t.res.route_kinds(sample).tolist()
    got["sample"] = sample
    return got


def fan_map(g, names):
    keys = F.pair_keys(g["topic"], g["rank"]).tolist()
    dl = np.repeat(np.arange(g["D"]), np.diff(g["off"])).tolist()
    return dict(zip(keys, zip([names(d, g["ordered"]) for d in dl], g["member"].tolist())))


def by_name(got, idx):
    """the outputs with every deliverer id replaced by the (subBrokerId, delivererKey) it names"""
    names = {}

    def name(d, od):
        if d not in names:
            names[d] = ORDERED if d == od else idx.deliverer(d)
        return names[d]
    osid = got["ordered_id"]
    out = {k: got[k] for k in ("csr", "budget", "routes", "kinds", "sample")}
    for k in ("plain", "ordered", "plain_wire", "ordered_wire"):
        out[k] = {name(d, osid): v for d, v in got[k].items()}
    for k in ("fan0", "fan1"):
        out[k] = fan_map(got[k], name)
    return out


def same(a, b):
    """two outputs() of one result: equal, fan-out order within a deliverer free"""
    for k in a:
        if k in ("fan0", "fan1"):
            F.same_map(a[k], b[k])
        else:
            assert a[k] == b[k], k


def check(B, idx, world, t, known):
    """every consumer of one completed result of the current generation against the references -> outputs()"""
    batch, out, n = t.batch, t.out, len(t.batch.topics)
    pairs = world.pairs
    want = C.caps_reference(world, batch.tenants, batch.topics, batch.tt, batch.max_p, batch.max_g)
    # bfq_match
    res = t.res
    offsets, ranks = res.expand()
    assert offsets.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    assert sorted((int(k), int(x), int(r)) for x, r, k in res.throttled.tolist()) == C.events3(want.events)
    assert res.route_count.tolist() == want.route_count
    # device match + expand
    d_off, d_ranks, total = C.read_device(B, out, n, want)
    # expand_budget
    bud = FB.budget(B, out, budget_case(batch))
    x = budget_expect(world, batch)
    FB.compare(B, bud, x, budget_case(batch))
    # fan-out, both passes
    B.torch.cuda.synchronize()
    csr_off, csr_ranks = d_off.cpu().numpy(), d_ranks.cpu().numpy()[:total]
    fans = []
    for path in (0, 1):
        idx.set_option("fanout_global", path)
        fans.append(F.fanout_once(B, out, d_off, d_ranks, total))
        s = F.check(idx, fans[-1], csr_off, csr_ranks, want, pairs)
        for p, d in s["ids"].items():
            assert known.setdefault(d, p) == p, d
    idx.set_option("fanout_global", 0)
    F.same_map(*fans)
    # delivery + its encoding, delivery_ordered + its encoding
    dl, _, got = D.nest_check(B, idx, out, batch.tenants, batch.tt, d_off, d_ranks, total, out.keep[2], pairs)
    _, data, req = W.encode_check(B, out, dl, got, pairs, batch.tenants, batch.topics, t.pub_off, packs=t.packs)
    plain_wire = {d: data[req[d]:req[d + 1]] for d in range(len(req) - 1) if req[d + 1] > req[d]}
    od, got_o = S.ordered_check(B, idx, out, batch.tenants, batch.tt, d_off, d_ranks, total, out.keep[2], pairs, t.pub_off,
                                t.pub_hash)
    if got_o is None:
        got_o = od.nesting(B.dev)
    _, data_o, req_o = W.encode_check(B, out, od, got_o, pairs, batch.tenants, batch.topics, t.pub_off, packs=t.packs)
    # route / route_kinds of the matched ranks
    sample = sorted(set(ranks[::7].tolist()))
    assert [res.route(r) for r in sample] == [pairs[r] for r in sample]
    assert res.route_kinds(ranks).tolist() == world.kinds[ranks].tolist()
    if out.generation == idx.generation():
        assert [idx.route(r) for r in sample[::5]] == [pairs[r] for r in sample[::5]]
    # Exchange(world=1).gather
    g = exchange(B).gather(out, ranges=True, stream=B.stream)
    B.torch.cuda.synchronize()
    assert g.topic_count == [n] and g.route_count().cpu().numpy().tolist() == res.route_count.tolist()
    assert g.span_count().cpu().numpy().tolist() == res.span_count.tolist()
    # what outputs() records for the held results is what the references checked
    rec = outputs(B, idx, t)
    assert rec["plain"] == got and rec["ordered"] == got_o and rec["plain_wire"] == decoded(plain_wire)
    assert rec["ordered_wire"] == decoded({d: data_o[req_o[d]:req_o[d + 1]] for d in range(len(req_o) - 1)
                                           if req_o[d + 1] > req_o[d]})
    for d in range(rec["ordered_id"]):
        assert known.setdefault(d, idx.deliverer(d)) == idx.deliverer(d)
    return rec


def exchange(B):
    if getattr(B, "xg", None) is None:
        B.xg = B.dist.Exchange(0, rank=0, world=1)
    return B.xg


def decoded(wire):
    """{deliverer: its DeliveryRequest decoded, each pack's MatchInfos sorted}: the nesting leaves their order inside a pack
    unspecified, and two delivery calls on one result may write them in different orders; everything else is compared
    byte for byte"""
    return {d: [(tn, [(tp, pubs, sorted(ms)) for tp, pubs, ms in packs]) for tn, packs in DW.decode_request(b)]
            for d, b in wire.items()}


def twin_check(B, stream, idx, t, rec):
    """a handle built from the live set: bfq_match arrays bit for bit, downstream outputs key for key"""
    twin = B.pkg.GpuRouteIndex(0)
    twin.load_pairs(stream.pairs())
    twin.commit()
    batch = t.batch
    a = idx.match_topics(batch.tenants, batch.topics, batch.tt, batch.max_p, batch.max_g)
    b = twin.match_topics(batch.tenants, batch.topics, batch.tt, batch.max_p, batch.max_g)
    for x, y in zip(a.expand(), b.expand()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.route_count, b.route_count)
    assert sorted(a.throttled.tolist()) == sorted(b.throttled.tolist())
    a.close()
    b.close()
    tt = take(B, twin, batch)
    theirs = by_name(outputs(B, twin, tt), twin)
    mine = by_name(rec, idx)
    for k in mine:
        assert mine[k] == theirs[k], k
    release(tt)
    twin.close()


def release(t):
    t.out.release()
    t.res.close()


# ------------------------------------------------------------------ the stream
def run_stream(B, seed, n_rounds=G.N_ROUNDS):
    stream = G.Stream(seed, n_rounds)
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(stream.pairs())
    idx.commit()
    small, big = G.fixed_batch(seed), G.fixed_batch(seed, big=True)
    known, held, tally = {}, [], {}
    seen = {"full": 0, "reset": 0, "recreated": 0, "async": 0}
    prev_world, async_done = None, False
    for r in stream.rounds():
        try:
            pending = None
            if not async_done and r.index >= ASYNC_FROM and r.path == "delta":
                pending = take(B, idx, small, wait=False)   # enqueued on the previous generation, consumed after the commit
                async_done = True
            st, gen = idx.stats(), idx.generation()
            if r.reset:
                idx.reset()
                idx.load_pairs(stream.pairs())
            else:
                idx.apply(adds=r.adds, dels=r.dels)
            if r.path == "delta":
                assert st["garbage_slots"] <= st["slots"] // 4 + 4096, (r.label, st)   # not what a stream round is about
            idx.commit()
            st2 = idx.stats()
            took = {(0, 0): "none", (1, 0): "delta", (0, 1): "full"}[(st2["delta_commits"] - st["delta_commits"],
                                                                      st2["full_commits"] - st["full_commits"])]
            assert took == r.path, (seed, r.index, r.label)
            assert (idx.generation() == gen) == (r.path == "none")
            assert st2["rebuilt_tenants"] == r.rebuilt, (r.label, st2["rebuilt_tenants"], r.rebuilt)
            assert (st2["tag_usable_slots"], st2["tag_used_slots"], st2["tag_overflowed_blocks"]) == \
                (r.tag_usable, r.tag_used, r.tag_overflowed), (r.label, st2)
            assert st2["routes"] == len(stream.live) and st2["tenants"] == len(r.ordinals)
            tally[r.label[0]] = tally.get(r.label[0], {})
            tally[r.label[0]][took] = tally[r.label[0]].get(took, 0) + 1
            seen["full"] += took == "full" and not r.reset
            seen["reset"] += r.reset
            seen["recreated"] += r.label == "e+"
            seen["async"] += pending is not None
            world = World(stream)
            if pending is not None:
                pending.out.wait()
                assert pending.out.generation == gen
                check(B, idx, prev_world, pending, known)
                release(pending)
            t = take(B, idx, big if r.index in BIG_ROUNDS else small)
            assert t.out.generation == idx.generation()
            rec = check(B, idx, world, t, known)
            for h in held:   # results of earlier generations reproduce what they returned when taken
                same(h.rec, outputs(B, idx, h))
            t.rec = rec
            if r.index % 5 == 4 or r.index == len(stream.labels) - 1:
                twin_check(B, stream, idx, t, rec)
            if len(t.batch.topics) > 10000:
                release(t)        # the large batch is checked, not held
            else:
                held.append(t)
                if len(held) > HELD:
                    release(held.pop(0))
            for d, p in known.items():
                assert idx.deliverer(d) == p
            prev_world = world
        except Exception as e:   # say where in the stream it failed
            e.add_note("seed %d, round %d (%s)" % (seed, r.index, r.label))
            raise
    for h in held:
        release(h)
    idx.close()
    assert seen["full"] >= 1 and seen["reset"] == 1 and seen["recreated"] == 1 and seen["async"] == 1
    return "seed %d: %s; full-build fallbacks %d, resets %d, tenants recreated %d" % (
        seed, ", ".join("%s %s" % (k, v) for k, v in sorted(tally.items())), seen["full"], seen["reset"], seen["recreated"])


@pytest.mark.parametrize("seed", G.SEEDS)
def test_commit_stream(B, seed, capsys):
    line = run_stream(B, seed)
    with capsys.disabled():   # the rounds per path are part of what the test reports, captured or not
        print("\n" + line)
