"""Leased workspaces: release waits for the work it hands back, and one handle stays exact through many call shapes.

Every match leases a workspace (streams, device scratch, result buffers) from its handle's pool; the pool keeps up to
POOL_KEEP idle workspaces and hands out the one given back last (LIFO). A workspace carries state from one call to the
next: buffer capacities, the order stage's strides, the cached tenant/caps table, the fan-out, delivery and budget scratch.

Part 1 checks the lease contract of bfq_device_result_release: it returns only after everything the library enqueued for
the result has finished, on every stream the result was used on (expand and budget phase 2, the fan-out, the delivery,
the exchange gather's compaction). Each test enqueues such work, releases, and then asks the stream (or an event recorded
right behind the call) whether it is idle. Nothing here reuses a workspace while work is pending on it.

Part 2 drives one forward handle through a fixed call program whose every transition (batch sizes across the order and
sub-batch thresholds, tenant lists across the order key's tenant bits, host and device paths, a buffer-growth re-run,
tier 2, both fan-out passes, delivery, budgets, option changes, commits while results are held) lands on one workspace.
`plan` models acquire / give_back and predicts which workspace each call gets; where two device results share a
workspace whose span buffer did not grow, their d_span_begin pointers must be equal. Every output is compared with the
plain references of the suite: caps_reference (the oracle's brute-force match with per-entry caps), submit, the fan-out
check, batch_delivery and the host path.
"""
import random
import threading

import numpy as np
import pytest

import oracle_lib as O
import test_gpu_caps as C
import test_gpu_delivery as FD
import test_gpu_edges as E
import test_gpu_fanout as F
import test_gpu_fanout_budget as FB
import test_gpu_inverse_edges as IE

INT_MAX, I64_MAX = 2 ** 31 - 1, 2 ** 63 - 1
E_STATE = -4

# ------------------------------------------------------------------ restated thresholds (lease.h, capi.cu, match_kernels.cu)
POOL_KEEP = 4                # idle workspaces a handle keeps (lease.h: POOL_KEEP)
ORDER_MIN = 32768            # default order_min_topics
PIPELINE_TOPICS, SUB_BATCHES = 1 << 17, 4


def sub_batches(n, host):
    """bfq_match cuts a batch of >= 2^17 topics into 4 sub-batches; the device path never does"""
    return SUB_BATCHES if host and n >= PIPELINE_TOPICS else 1


def per_chunk(n, chunks):
    """prepare_workspace reserves the order stage's buffers when this reaches order_min"""
    return (n + chunks - 1) // chunks + 1


def ordered(n, host, order_min=ORDER_MIN):
    """a sub-batch is put in locality order (and de-duplicated) when it has at least order_min topics"""
    c = sub_batches(n, host)
    return n > 0 and min(n * (k + 1) // c - n * k // c for k in range(c)) >= order_min


def tenant_bits(n_tenants):
    b = 0
    while b < 20 and (1 << b) < n_tenants:
        b += 1
    return b


def key_bits(tb):
    return max(min(32, (tb + 12 + 7) // 8 * 8), min(32, tb + 3))


def hist_bits(n, n_tenants):
    nb = 12
    while nb < 22 and (1 << nb) < 4 * n:
        nb += 1
    return max(12, min(nb, key_bits(tenant_bits(n_tenants))))


def hash_entries(n):
    e = 1024
    while e < (1 << 31) and e < 2 * n:
        e <<= 1
    return e


# ------------------------------------------------------------------ the pool model
class PoolModel:
    """acquire pops the idle workspace given back last, or makes a new one; give_back keeps at most POOL_KEEP idle and
    frees the rest. Each workspace's span capacity follows prepare_workspace's exact reserve(max(n, 1))."""

    def __init__(self):
        self.idle, self.span_cap, self.made, self.freed = [], {}, 0, []

    def acquire(self, n):
        """-> (workspace id, whether its span buffers grew for a batch of n)"""
        if self.idle:
            w = self.idle.pop()
        else:
            w = self.made
            self.made += 1
            self.span_cap[w] = 0
        grew = max(n, 1) > self.span_cap[w]
        self.span_cap[w] = max(self.span_cap[w], max(n, 1))
        return w, grew

    def give_back(self, w):
        if len(self.idle) < POOL_KEEP:
            self.idle.append(w)
        else:
            self.freed.append(w)


# ------------------------------------------------------------------ the call program (plain data)
BIG_LIST = (1 << 20) + 1
LIST_SIZES = {"L1": 1, "L4097": 4097, "Lbig": BIG_LIST}
TENANTS = ["tA", "tB", "tC", "tD"]
BASE_TOPICS = ["s/x", "s/y", "q/x", "$sys/x", "k1/a/b/c/d", "k2/a/b/c/x", "none/z"]
TIER0_TOPICS = ["s/x", "s/y", "q/x", "$sys/x", "none/z"]
TIER2_TOPICS = [E.TIER2_TOPIC, E.TIER1_TOPIC] + BASE_TOPICS
# m1 sizes the main workspace's range region: 12 inline slots per topic of its 131072, then 2^20 for tiers 1 and 2 (host path,
# 4 sub-batches). m8's distinct spill topics (a 64-range spill block each) overflow what that region leaves them.
REGION_AFTER_M1 = 131072 * E.INLINE_RANGES + (1 << 20)
SPILL_N = 48000
COLLIDE_AT = [0]             # entries i and i + 2^20 of the big list: one tenant key once masked to 20 bits


def tenant_list(name, caps_seed):
    """a tenant list of LIST_SIZES[name] entries over four tenant ids, with per-entry caps drawn from caps_seed (0: none).
    In the big list, entries i and i + 2^20 name different tenants: their order keys collide once masked to 20 bits."""
    n = LIST_SIZES[name]
    ids = [TENANTS[i % 4] for i in range(n)]
    if name == "Lbig":
        for i in COLLIDE_AT:
            ids[i], ids[i + (1 << 20)] = "tA", "tB"
    if caps_seed == 0:
        return ids, [INT_MAX] * n, [INT_MAX] * n
    rng = random.Random(caps_seed)
    choice = [INT_MAX, INT_MAX, 0, 1, 2, 3, -1]
    return ids, [rng.choice(choice) for _ in range(n)], [rng.choice(choice) for _ in range(n)]


def batch(n, list_name, seed, pool):
    """n topics drawn from `pool` (or the distinct spill topics), tenant entries drawn over the list; the big list's batch
    also carries the colliding entry pairs, under the same topic text"""
    rng = random.Random(seed)
    nt = LIST_SIZES[list_name]
    if pool == "spill":
        topics = E.spill_batch(n)
        return topics, np.array([rng.randrange(nt) for _ in range(n)], np.int32)
    src = {"base": BASE_TOPICS, "tier0": TIER0_TOPICS, "tier2": TIER2_TOPICS}[pool]
    topics = [rng.choice(src) for _ in range(n)]
    tt = [rng.randrange(nt) for _ in range(n)]
    if list_name == "Lbig" and n >= 2 * len(COLLIDE_AT):
        for k, i in enumerate(COLLIDE_AT):
            topics[2 * k] = topics[2 * k + 1] = "s/x"
            tt[2 * k], tt[2 * k + 1] = i, i + (1 << 20)
    return topics, np.array(tt, np.int32)


def program():
    """the single-threaded phase: a list of steps. A match step names its path, batch, tenant list, caps and options, and
    what is done with its result (fan-out pass, delivery, budget, gather) and when it is released (hold: by a later
    "release" step). "commit" steps change the route set while results are held."""
    M = lambda **k: dict(op="match", **k)
    steps = [
        M(name="m1", path="host", n=131072, lst="L1", caps=0, pool="base"),                     # 4 sub-batches, ordered
        M(name="m2", path="device", n=32767, lst="L4097", caps=1, pool="base", fan="auto"),     # arrival order
        dict(op="opt", dedup_hash_bits=10),
        M(name="m3", path="device", n=32768, lst="Lbig", caps=2, pool="base"),                  # ordered, 20 tenant bits
        M(name="m4", path="device", n=1, lst="L4097", caps=3, pool="base"),                     # the list of m2, other caps
        M(name="m5", path="device", n=1, lst="L4097", caps=1, pool="base"),                     # only the caps change
        dict(op="opt", dedup_hash_bits=64, tier0_ctas_per_sm=1),
        M(name="m6", path="host", n=0, lst="L1", caps=0, pool="base"),
        M(name="m7", path="device", n=131073, lst="L4097", caps=1, pool="base"),                # grows every span buffer
        dict(op="opt", tier0_ctas_per_sm=0, order_min_topics=0),
        M(name="m8", path="device", n=SPILL_N, lst="L1", caps=0, pool="spill", retry=True),     # re-run with a grown region
        M(name="m9", path="device", n=100, lst="L1", caps=0, pool="base"),
        dict(op="opt", order_min_topics=ORDER_MIN),
        M(name="m10", path="host", n=131072, lst="L4097", caps=3, pool="base"),                 # 4 sub-batches again
        M(name="m11", path="device", n=3000, lst="L4097", caps=0, pool="tier2", fan="auto"),    # tier 2: grows d_scratch
        M(name="m12", path="device", n=3000, lst="L4097", caps=0, pool="tier0", fan="global"),
        M(name="m13", path="device", n=2000, lst="L4097", caps=0, pool="base", fan="auto", deliver=True, budget="bind"),
        M(name="m14", path="device", n=300, lst="L4097", caps=0, pool="base", deliver=True, budget="free", gather=True),
        # five results in flight: m15 takes the main workspace, m16-m19 new ones; commits while they are held
        M(name="m15", path="device", n=5000, lst="L4097", caps=1, pool="base", hold=True, fan="auto"),
        M(name="m16", path="device", n=700, lst="L1", caps=0, pool="tier2", hold=True),
        dict(op="commit", kind="delta"),
        M(name="m17", path="device", n=900, lst="L4097", caps=2, pool="base", hold=True, fan="auto"),
        dict(op="commit", kind="full"),
        M(name="m18", path="device", n=40000, lst="L4097", caps=0, pool="base", hold=True),
        M(name="m19", path="device", n=64, lst="L1", caps=0, pool="base", hold=True),
        dict(op="release", names=["m16", "m17", "m18", "m15", "m19"]),   # m19's workspace is the fifth: freed
        M(name="m20", path="device", n=131072, lst="L4097", caps=1, pool="base"),               # the main workspace again
    ]
    return steps


def plan(steps):
    """runs the pool model over the program -> {match name: (workspace, span buffers grew)}. A match that is not held
    gives its workspace back before the next step; a gather compares with a host match of the same batch, taken while
    the device result is held."""
    pool = PoolModel()
    out, held = {}, {}
    for s in steps:
        if s["op"] == "match":
            w, grew = pool.acquire(s["n"])
            out[s["name"]] = (w, grew)
            if s.get("gather"):
                hw, _ = pool.acquire(s["n"])
                pool.give_back(hw)
            if s.get("hold"):
                held[s["name"]] = w
            else:
                pool.give_back(w)
        elif s["op"] == "release":
            for nm in s["names"]:
                pool.give_back(held.pop(nm))
    assert not held
    return out, pool


# ------------------------------------------------------------------ route sets of the program (plain Python data)
def routes_of(generation):
    """generation 0: the caps suite's mix for four tenants plus each tenant's spill filters; 1 (a delta commit): tB gains
    routes on s/x and +/x; 2 (a full commit): generation 0 again"""
    r = [x for t in TENANTS for x in C.mix_routes(t)]
    if generation == 1:
        r += [("tB", "s/x", "p", 5), ("tB", "+/x", "g", 2), ("tB", "s/x", "n", 1)]
    return r


_WORLDS = {}


def world_of(generation):
    if generation not in _WORLDS:
        _WORLDS[generation] = C.World(*C.build(routes_of(generation)))
    return _WORLDS[generation]


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def B():
    import torch

    import bifromq_b200
    from bifromq_b200 import dist
    from bifromq_b200._native import NativeError
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.pkg, ns.torch, ns.dist, ns.NativeError = bifromq_b200, torch, dist, NativeError
    ns.dev = torch.device("cuda", 0)
    ns.stream = torch.cuda.current_stream(ns.dev).cuda_stream
    return ns


SLEEP_CYCLES = 40_000_000        # torch.cuda._sleep: about 20 ms at the H100's clock
BIG_TOPICS, BIG_ROUTES = 24576, 12288


def big_csr_case(n_topics=BIG_TOPICS, n_routes=BIG_ROUTES):
    """every topic e/<i> matches one filter of n_routes routes: a device CSR of n_topics * n_routes (302 M) ranks, 2.4 GB
    that the expand's phase 2 writes after the call has returned"""
    kv = {}
    for i in range(n_routes):
        F.nroute(kv, "c", "e/#", i % 3, "r%d" % i, "d%d" % (i % 7))
    return sorted(kv.items()), ["c"], ["e/%d" % k for k in range(n_topics)], np.zeros(n_topics, np.int32)


@pytest.fixture(scope="module")
def BIG(B):
    pairs, tenants, topics, tt = big_csr_case()
    idx = F.make_index(B, pairs)
    yield idx, tenants, topics, tt
    idx.close()


def match_on(B, idx, tenants, topics, tt, S, wait=True):
    """bfq_match_device with its inputs copied and matched on torch stream S (the caller's current stream)"""
    torch = B.torch
    blob, off = O.blob(topics)
    with torch.cuda.stream(S):
        keep = [torch.from_numpy(blob).to(B.dev), torch.from_numpy(off).to(B.dev),
                torch.from_numpy(np.ascontiguousarray(tt, np.int32)).to(B.dev)]
        out = idx.match_device(tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), len(topics),
                               stream=S.cuda_stream, wait=wait)
    out.keep = keep
    return out


def sized_csr(B, out, n, S, fill=False):
    """the CSR arrays of a completed result, allocated on S and sized by a counting expand on S; fill=True also writes the
    ranks and waits for them"""
    torch = B.torch
    with torch.cuda.stream(S):
        d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=B.dev)
        total = out.expand(d_offsets.data_ptr(), None, 0, S.cuda_stream)
        d_ranks = torch.empty(max(total, 1), dtype=torch.int64, device=B.dev)
        if fill:
            assert out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, S.cuda_stream) == total
            S.synchronize()
    return d_offsets, d_ranks, total


def idle_after(B, stream_obj):
    """a torch event recorded on the stream right after a library call returned"""
    ev = B.torch.cuda.Event()
    ev.record(stream_obj)
    return ev


# ------------------------------------------------------------------ part 1: release waits for the work it hands back
@pytest.mark.gpu
def test_release_waits_for_expand_phase2(B, BIG):
    idx, tenants, topics, tt = BIG
    torch = B.torch
    S = torch.cuda.Stream(B.dev)
    out = match_on(B, idx, tenants, topics, tt, S)
    d_offsets, d_ranks, total = sized_csr(B, out, len(topics), S)
    assert total == BIG_TOPICS * BIG_ROUTES
    assert out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, S.cuda_stream) == total
    ev = idle_after(B, S)
    out.release()
    assert ev.query(), "release returned before the expand's phase 2 finished"
    with torch.cuda.stream(S):
        last = d_ranks[total - BIG_ROUTES:total].cpu().numpy()
    assert sorted(last.tolist()) == list(range(BIG_ROUTES))


@pytest.mark.gpu
def test_release_waits_for_budget_phase2(B, BIG):
    idx, tenants, topics, tt = BIG
    torch = B.torch
    S = torch.cuda.Stream(B.dev)
    n = len(topics)
    out = match_on(B, idx, tenants, topics, tt, S)
    with torch.cuda.stream(S):
        d_msg = torch.full((n,), 10, dtype=torch.int32, device=B.dev)
        d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=B.dev)
        total = out.expand_budget(d_msg.data_ptr(), [I64_MAX], [3], d_offsets.data_ptr(), None, 0, S.cuda_stream).n_delivered
        assert total == n * BIG_ROUTES
        d_ranks = torch.empty(total, dtype=torch.int64, device=B.dev)
    r = out.expand_budget(d_msg.data_ptr(), [I64_MAX], [3], d_offsets.data_ptr(), d_ranks.data_ptr(), total, S.cuda_stream)
    ev = idle_after(B, S)
    out.release()
    assert ev.query(), "release returned before the budget's phase 2 finished"
    assert r.n_delivered == total


@pytest.mark.gpu
def test_release_waits_for_fanout(B):
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    torch = B.torch
    S = torch.cuda.Stream(B.dev)
    out = match_on(B, idx, tenants, topics, tt, S)
    d_offsets, d_ranks, total = sized_csr(B, out, len(topics), S, fill=True)
    # the first fan-out of a snapshot builds its tables with synchronous copies; the one under test finds them built
    out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, S.cuda_stream)
    with torch.cuda.stream(S):
        torch.cuda._sleep(SLEEP_CYCLES)
    out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, S.cuda_stream)
    out.release()
    assert S.query(), "release returned while the fan-out was still queued"
    idx.close()


@pytest.mark.gpu
def test_release_waits_for_delivery(B):
    """bfq_delivery_device synchronises its stream itself: pinned here so that stays true"""
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    torch = B.torch
    S = torch.cuda.Stream(B.dev)
    out = match_on(B, idx, tenants, topics, tt, S)
    d_offsets, d_ranks, total = sized_csr(B, out, len(topics), S, fill=True)
    with torch.cuda.stream(S):
        torch.cuda._sleep(SLEEP_CYCLES)
    out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), S.cuda_stream)
    out.release()
    assert S.query()
    idx.close()


@pytest.mark.gpu
def test_release_waits_on_every_stream_the_result_was_used_on(B):
    """the long work is on the stream the result was NOT used on last: a fan-out queued behind a sleep on S1, then an
    expand on S2 that synchronises S2 only. An event re-recorded by each call would cover S2 alone. The two calls share no
    buffer: the fan-out reads CSR A and writes the fan-out arrays, the expand writes the expand scratch and CSR B."""
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    torch = B.torch
    S1, S2 = torch.cuda.Stream(B.dev), torch.cuda.Stream(B.dev)
    out = match_on(B, idx, tenants, topics, tt, S1)
    d_off_a, d_ranks_a, total = sized_csr(B, out, len(topics), S1, fill=True)
    out.fanout(d_off_a.data_ptr(), d_ranks_a.data_ptr(), total, S1.cuda_stream)   # builds the fan-out tables
    S1.synchronize()
    with torch.cuda.stream(S1):
        torch.cuda._sleep(SLEEP_CYCLES)
    out.fanout(d_off_a.data_ptr(), d_ranks_a.data_ptr(), total, S1.cuda_stream)
    d_off_b, d_ranks_b, total_b = sized_csr(B, out, len(topics), S2)
    assert total_b == total
    assert out.expand(d_off_b.data_ptr(), d_ranks_b.data_ptr(), total, S2.cuda_stream) == total
    ev2 = idle_after(B, S2)
    out.release()
    assert S1.query(), "release left the fan-out running on the stream the result was used on first"
    assert ev2.query()
    idx.close()


@pytest.mark.gpu
def test_host_matches_do_not_wait_for_unrelated_work(B):
    """a match waits for its own workspace's streams only: a host match on a fresh handle, whose pinned range buffer must
    grow, and a host inverse match both return while a sleep of seconds on an unrelated stream is still running"""
    from bifromq_b200 import _native, retain
    torch = B.torch
    R = type("R", (), {"N": _native, "retain": retain})
    pairs, tenants, topics, tt = F.groups_case()
    ritopics, filters = IE.dollar_case()
    # every kernel both matches launch is loaded before the sleep is queued (loading a kernel may synchronise the device)
    warm = F.make_index(B, pairs)
    warm.match_topics(tenants, topics, tt).close()
    warm.close()
    rwarm, _ = IE.make_index(R, ritopics)
    IE.run(R, rwarm, filters)
    rwarm.close()
    idx = F.make_index(B, pairs)
    ridx, entries = IE.make_index(R, ritopics)
    S = torch.cuda.Stream(B.dev)
    with torch.cuda.stream(S):
        torch.cuda._sleep(1000)
    S.synchronize()
    ev = torch.cuda.Event()
    with torch.cuda.stream(S):
        torch.cuda._sleep(SLEEP_CYCLES * 250)   # about 5 s
        ev.record(S)
    res = idx.match_topics(tenants, topics, tt)
    forward_waited = ev.query()
    rres = IE.run(R, ridx, filters)
    inverse_waited = ev.query()
    S.synchronize()
    assert not forward_waited, "a host match waited for a sleep on an unrelated stream"
    assert not inverse_waited, "a host inverse match waited for a sleep on an unrelated stream"
    want = F.oracle(pairs, tenants, topics, tt)
    offsets, ranks = res.expand()
    assert len(ranks) > 0
    assert offsets.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    IE.check(rres, IE.Expect(entries), filters)
    res.close()
    idx.close()
    ridx.close()


def gather_world1(B):
    return B.dist.Exchange(0, rank=0, world=1)


@pytest.mark.gpu
def test_release_waits_for_gather_compaction(B):
    """world-1 gather of a batch whose every topic matches 263 ranges (tier 2, de-duplicated by the match): the
    compaction writes every topic's ranges in full, 210 M of them (1.7 GB), after the gather's one synchronisation"""
    routes, tenants, topics = E.tier2_case()
    idx = F.make_index(B, E.make_pairs(routes))
    n = 800000
    topics = [E.TIER2_TOPIC] * n
    tt = np.zeros(n, np.int32)
    torch = B.torch
    S = torch.cuda.Stream(B.dev)
    x = gather_world1(B)
    out = match_on(B, idx, tenants, topics, tt, S)
    g = x.gather(out, ranges=True, stream=S.cuda_stream)
    ev = idle_after(B, S)
    out.release()
    assert ev.query(), "release returned before the gather's compaction finished"
    assert g.n_ranges_total == 263 * n
    x.close()
    idx.close()


@pytest.mark.gpu
def test_gather_needs_a_completed_match(B):
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    x = gather_world1(B)
    out = F.match_device(B, idx, tenants, topics, tt, wait=False)
    with pytest.raises(B.NativeError) as e:
        x.gather(out, ranges=True, stream=B.stream)
    assert F.bfq_code(e.value) == E_STATE
    out.wait()
    g = x.gather(out, ranges=True, stream=B.stream)
    check_gather(B, idx, g, tenants, topics, tt)
    out.release()
    x.close()
    idx.close()


def check_gather(B, idx, g, tenants, topics, tt, mp=None, mg=None):
    """a world-1 gather equals the host path's answer for the same batch: route and span counts, per-topic range sets"""
    n = len(topics)
    route_count = g.route_count().cpu().numpy()
    span_count = g.span_count().cpu().numpy().astype(np.int64)
    got = g.ranges().cpu().numpy()
    res = idx.match_topics(tenants, topics, np.ascontiguousarray(tt, np.int32), mp, mg)
    assert g.world == 1 and g.topic_count == [n] and g.n_topics_total == n
    assert route_count.tolist() == res.route_count.tolist()
    assert span_count.tolist() == res.span_count.tolist()
    gb = np.concatenate([[0], np.cumsum(span_count)])
    want = np.stack([res.ranges["first"], res.ranges["count"]], axis=1)
    sb = res.span_begin
    for i in range(n):
        a, b = int(sb[i]), int(sb[i]) + int(res.span_count[i])
        assert sorted(map(tuple, got[gb[i]:gb[i + 1]].tolist())) == sorted(map(tuple, want[a:b].tolist())), i
    res.close()


# ------------------------------------------------------------------ part 2: the call program
class Runner:
    """executes program() on one handle, checking every output against its reference"""

    def __init__(self, B, idx):
        self.B, self.idx = B, idx
        self.gen = 0
        self.lists = {}
        self.held = {}
        self.span = {}          # match name -> d_span_begin of its device result
        self.fan_paths = []
        self.order_min = ORDER_MIN

    def tenant_list(self, name, caps):
        key = (name, caps)
        if key not in self.lists:
            ids, mp, mg = tenant_list(name, caps)
            self.lists[key] = (self.B.pkg.GpuRouteIndex.tenant_blob(ids), ids, np.array(mp, np.int32), np.array(mg, np.int32))
        return self.lists[key]

    def step(self, s):
        op = s["op"]
        if op == "opt":
            for k, v in s.items():
                if k != "op":
                    self.idx.set_option(k, v)
            if "order_min_topics" in s:
                self.order_min = s["order_min_topics"] if s["order_min_topics"] > 0 else 1 << 62
        elif op == "commit":
            if s["kind"] == "delta":
                adds = sorted(set(world_of(1).pairs) - set(world_of(0).pairs))
                self.idx.apply(adds=adds)
                self.idx.commit()
                self.gen = 1
            else:
                self.idx.reset()
                self.idx.load_pairs(world_of(0).pairs)
                self.idx.commit()
                self.gen = 2
        elif op == "release":
            for nm in s["names"]:
                out, check = self.held.pop(nm)
                check()
                out.release()
        else:
            self.match(s)

    def match(self, s):
        B, idx = self.B, self.idx
        blob, ids, mp, mg = self.tenant_list(s["lst"], s["caps"])
        topics, tt = batch(s["n"], s["lst"], int(s["name"][1:]), s["pool"])
        w = world_of(self.gen)
        if s["path"] == "host":
            before = idx.stats()
            res = idx.match_topics(blob, topics, tt, mp, mg)
            offsets, ranks = res.expand()
            if s["n"] == 0:
                assert offsets.tolist() == [0] and len(ranks) == 0 and len(res.throttled) == 0
                res.close()
                return
            want = C.caps_reference(w, ids, topics, tt, mp, mg)
            assert offsets.tolist() == want.offsets.tolist(), s["name"]
            assert ranks.tolist() == want.ranks.tolist(), s["name"]
            assert sorted((int(k), int(t), int(r)) for t, r, k in res.throttled.tolist()) == C.events3(want.events)
            assert res.route_count.tolist() == want.route_count
            assert int(res.timings_ms["sub_batches"]) == (sub_batches(s["n"], True) if s["n"] else 1)
            if ordered(s["n"], True):
                d = E.delta(idx, before)
                c = sub_batches(s["n"], True)
                bounds = [s["n"] * k // c for k in range(c + 1)]
                assert d["duplicate_topics"] == sum(E.true_repeats(ids, topics[a:b], tt[a:b]) for a, b in zip(bounds, bounds[1:]))
            res.close()
            return
        before = idx.stats()
        out = C.match_device(B, idx, blob, topics, tt, mp, mg)
        d = E.delta(idx, before)
        self.span[s["name"]] = out.d_span_begin
        # m8 must overflow its range region; other calls may re-run once for a throttle list their caps overfill
        assert d["buffer_retries"] == 1 if s.get("retry") else d["buffer_retries"] <= 1, (s["name"], d)
        if ordered(s["n"], False, self.order_min):
            assert d["duplicate_topics"] == E.true_repeats(ids, topics, tt), (s["name"], d)
        else:
            assert d["duplicate_topics"] == 0, (s["name"], d)

        def check(out=out, w=w, topics=topics, tt=tt):
            want = C.caps_reference(w, ids, topics, tt, mp, mg)
            d_offsets, d_ranks, total = C.read_device(B, out, len(topics), want)
            if s.get("fan"):
                self.fanout(s, out, d_offsets, d_ranks, total, want, w)
            if s.get("deliver"):
                FD.nest_check(B, idx, out, ids, tt, d_offsets, d_ranks, total, out.keep[2], w.pairs)
            if s.get("budget"):
                self.budget(s, out, w, ids, topics, tt, mp, mg)
            if s.get("gather"):
                x = gather_world1(B)
                g = x.gather(out, ranges=True, stream=B.stream)
                check_gather(B, idx, g, blob, topics, tt, mp, mg)
                x.close()

        if s.get("hold"):
            self.held[s["name"]] = (out, check)
        else:
            check()
            out.release()

    def fanout(self, s, out, d_offsets, d_ranks, total, want, w):
        B, idx = self.B, self.idx
        idx.set_option("fanout_global", 1 if s["fan"] == "global" else 0)
        before = idx.stats()["global_fanouts"]
        got = F.fanout_once(B, out, d_offsets, d_ranks, total)
        taken = idx.stats()["global_fanouts"] - before
        idx.set_option("fanout_global", 0)
        tiled = s["fan"] == "auto" and F.expect_tiled(got["D"], got["n_pairs"])
        assert taken == (0 if tiled else 1), (s["name"], got["D"], got["n_pairs"])
        self.fan_paths.append("tiled" if tiled else "global")
        B.torch.cuda.synchronize()
        F.check(idx, got, d_offsets.cpu().numpy(), d_ranks.cpu().numpy()[:total], want, w.pairs)

    def budget(self, s, out, w, ids, topics, tt, mp, mg):
        assert (mp == INT_MAX).all() and (mg == INT_MAX).all()   # expect() takes uniform caps
        nt = len(ids)
        rng = random.Random(len(topics))
        sizes = [rng.choice([0, 7, 100, 1000]) for _ in topics]
        if s["budget"] == "bind":
            max_bytes = [rng.choice([1, 7, 150, 2500]) for _ in range(nt)]
            bw = [rng.choice([0, 1, 2, 3, 3]) for _ in range(nt)]
        else:
            max_bytes, bw = [I64_MAX] * nt, [3] * nt
        case = FB.Case(w.pairs, ids, topics, tt, sizes, max_bytes, bw)
        x = FB.expect(case, w.kinds, w.kv)
        got = FB.budget(self.B, out, case)
        FB.compare(self.B, got, x, case)
        if s["budget"] == "bind":
            assert got["r"].n_dropped_bytes + got["r"].n_dropped_persistent_bandwidth + got["r"].n_dropped_transient_bandwidth > 0
        else:
            assert int(got["offsets"][-1]) == len(x.ranks) and not (got["flags"] & FB.DROPS).any()


@pytest.mark.gpu
def test_one_handle_through_the_call_program(B):
    steps = program()
    predicted, pool = plan(steps)
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(world_of(0).pairs)
    idx.commit()
    run = Runner(B, idx)
    for s in steps:
        run.step(s)
    assert not run.held
    # device results the model puts on one workspace, where the span buffers did not grow in between: the same buffer
    device = [s["name"] for s in steps if s["op"] == "match" and s["path"] == "device"]
    same = 0
    for a, b in zip(device, device[1:]):
        (wa, _), (wb, grew) = predicted[a], predicted[b]
        if wa == wb and not grew and not any(predicted[m][1] for m in between(steps, a, b)):
            assert run.span[a] == run.span[b], (a, b)
            same += 1
    assert same >= 8
    assert run.fan_paths[1:4] == ["tiled", "global", "tiled"]
    assert pool.made == 5 and len(pool.freed) == 1
    idx.close()


def between(steps, a, b):
    names = [s["name"] for s in steps if s["op"] == "match"]
    return names[names.index(a) + 1:names.index(b)]


# ------------------------------------------------------------------ part 2, second phase: two threads, two streams
@pytest.mark.gpu
def test_two_threads_release_each_others_results(B):
    torch = B.torch
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(world_of(0).pairs)
    idx.commit()
    w = world_of(0)
    streams = [torch.cuda.Stream(B.dev), torch.cuda.Stream(B.dev)]
    shapes = [(32768, "L4097", 1, "base"), (1, "L1", 0, "base"), (3000, "L4097", 0, "tier2"), (0, "L1", 0, "base"),
              (20000, "L4097", 3, "base"), (5000, "L1", 0, "tier0")]
    lists = {}
    for _, lst, caps, _ in shapes:
        if (lst, caps) not in lists:
            ids, mp, mg = tenant_list(lst, caps)
            lists[(lst, caps)] = (ids, np.array(mp, np.int32), np.array(mg, np.int32))
    handed = [[], []]
    errors = []
    barrier = threading.Barrier(2)

    def worker(me):
        try:
            S = streams[me]
            with torch.cuda.stream(S):
                stream = S.cuda_stream
                for k, (n, lst, caps, pool) in enumerate(shapes[me::2] + shapes[1 - me::2]):
                    ids, mp, mg = lists[(lst, caps)]
                    topics, tt = batch(n, lst, 100 * me + k, pool)
                    blob, off = O.blob(topics)
                    keep = [torch.from_numpy(blob).to(B.dev), torch.from_numpy(off).to(B.dev), torch.from_numpy(tt).to(B.dev)]
                    out = idx.match_device(ids, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), n, mp, mg, stream)
                    out.keep = keep
                    d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=B.dev)
                    total = out.expand(d_offsets.data_ptr(), None, 0, stream)
                    d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=B.dev)
                    out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
                    S.synchronize()
                    offsets = d_offsets.cpu().numpy()
                    ranks = d_ranks.cpu().numpy()[:total]
                    want = C.caps_reference(w, ids, topics, tt, mp, mg) if n else None
                    assert offsets.tolist() == (want.offsets.tolist() if n else [0])
                    seg = np.repeat(np.arange(n), np.diff(offsets))
                    assert ranks[np.lexsort((ranks, seg))].tolist() == (want.ranks.tolist() if n else [])
                    # a fan-out still queued behind a sleep when the result goes to the other thread
                    torch.cuda._sleep(SLEEP_CYCLES // 4)
                    out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
                    handed[1 - me].append((out, S, (d_offsets, d_ranks)))
            barrier.wait()
            mine = handed[me][:]
            random.Random(me).shuffle(mine)
            for out, S_other, _ in mine:
                out.release()
            for out, S_other, _ in mine:
                assert S_other.query()
        except Exception as e:   # noqa: BLE001 - re-raised on the main thread
            errors.append(e)
            try:
                barrier.abort()
            except Exception:
                pass

    th = [threading.Thread(target=worker, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errors:
        raise errors[0]
    idx.close()
