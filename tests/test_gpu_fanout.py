"""The fan-out pass (bfq_fanout_device) against a plain group-by, at its tile, chunk and deliverer limits.

bfq_fanout_device takes the device CSR of a completed match (surviving route ranks per topic) and groups every
(topic, route) pair by the (subBrokerId, delivererKey) it is delivered through, picking one member of a $share group and
parking $oshare pairs (and empty groups) under the result's ordered_share_id. The pass has two forms (csrc/fanout.cu): a
tile pass (4096-pair tiles, 16 consecutive pairs per thread, a shared-memory histogram per tile) for few deliverers, and
a global-count pass for many; the "fanout_global" option forces the global one so small cases check both.

Every expectation here comes from the KV each test builds in Python and from the CPU oracle: the sorted pair list of each
committed generation gives rank -> (key, value); oracle_lib decodes the route and its deliverer; KV.match_batch gives the
surviving ranks per topic. Nothing is looked up through the library's own route lookup. A CPU test per shape proves, from
the oracle alone, that its generator lands on the edge it is named after.
"""
import threading

import numpy as np
import pytest

import oracle_lib as O

INT_MAX = 2 ** 31 - 1
TILE, CHUNK = 4096, 16           # pairs per tile and per thread of both passes (csrc/fanout.cu: FO_TILE, FO_TILE / FO_THREADS)
NO_MEMBER = 0xFFFFFFFF
CAPS = [(INT_MAX, INT_MAX), (3, 1), (INT_MAX, 100), (0, 0)]
PATHS = ["auto", "global"]


def expect_tiled(n_deliverers, n_pairs):
    """fanout_tiled(): the tile pass while its [deliverer][tile] matrix has at most one cell per pair"""
    tiles = max(1, -(-n_pairs // TILE))
    return n_deliverers * tiles <= min(max(n_pairs, TILE), INT_MAX)


# ------------------------------------------------------------------ case building (plain Python data, no GPU)
def nroute(kv, tenant, tf, broker, receiver, dkey, inc=1):
    kv[O.route_key(tenant, tf, O.receiver_url(broker, receiver, dkey))] = O.incarnation_bytes(inc)


def groute(kv, tenant, tf, grp, member_urls, ordered=False):
    """a shared subscription; member_urls in the wire order of the stored RouteGroup"""
    kv[O.route_key(tenant, ("$oshare/" if ordered else "$share/") + grp + "/" + tf)] = O.route_group({u: 1 for u in member_urls})


def mixed_routes(kv, tenant, tf, n, tag="r"):
    """n routes of one filter: normal routes over 5 deliverer keys and subBrokerIds 0-2, 2-member $share and $oshare groups"""
    for i in range(n):
        k = i % 9
        if k < 6:
            nroute(kv, tenant, tf, i % 3, "%s%d" % (tag, i), "d%d" % (i % 5))
        elif k < 8:
            groute(kv, tenant, tf, "%s%d" % (tag, i), [O.receiver_url(0, "m%d" % i, "d1"), O.receiver_url(2, "m%d" % i, "d3")])
        else:
            groute(kv, tenant, tf, "%s%d" % (tag, i), [O.receiver_url(0, "o%d" % i, "d2")], ordered=True)


def count_case(n_routes, n_topics, prefix="e"):
    """n_routes routes on "e/#", topics <prefix>/0 ..: n_routes * n_topics pairs (0 for another prefix)"""
    kv = {}
    mixed_routes(kv, "c", "e/#", n_routes)
    return sorted(kv.items()), ["c"], ["%s/%d" % (prefix, k) for k in range(n_topics)], np.zeros(n_topics, np.int32)


# (n_routes, n_topics, topic prefix) -> n_pairs
COUNT_SHAPES = {0: (5, 1, "f"), 1: (1, 1, "e"), 15: (15, 1, "e"), 16: (16, 1, "e"), 17: (17, 1, "e"),
                4095: (4095, 1, "e"), 4096: (4096, 1, "e"), 4097: (4097, 1, "e"), 8192: (8192, 1, "e"),
                4097 * 512: (4097, 512, "e")}


def hot_case():
    """one hot/# filter with 12289 routes (> 3 tiles per topic), 0-pair topics at the start, the middle and the end"""
    kv = {}
    mixed_routes(kv, "h", "hot/#", 12289)
    topics = ["cold/0", "hot/a", "cold/1", "cold/2", "hot/b", "cold/3"]
    return sorted(kv.items()), ["h"], topics, np.zeros(len(topics), np.int32)


BOUNDARY_COUNTS = [16, 1, 15, 4064, 1, 4095, 1, 0, 4095, 1]   # topic ends at 16, 17, 32, 4096, 4097, 8192, 8193, 8193, 12288, 12289


def boundary_case():
    kv = {}
    for k, c in enumerate(BOUNDARY_COUNTS):
        mixed_routes(kv, "b", "b/%d" % k, c, tag="b%d_" % k)
    topics = ["b/%d" % k for k in range(len(BOUNDARY_COUNTS))]
    return sorted(kv.items()), ["b"], topics, np.zeros(len(topics), np.int32)


def one_bin_case():
    """15000 pairs, every one through the same deliverer (one histogram bin takes every count)"""
    kv = {}
    for i in range(5000):
        nroute(kv, "o", "one/#", 0, "r%d" % i, "hot")
    return sorted(kv.items()), ["o"], ["one/0", "one/1", "one/2"], np.zeros(3, np.int32)


# 4095 ids + the ordered id over 4095 pairs: the tile pass at its bound (4096 cells = 4096); 4096 ids: one cell past it
K_DELIVERERS = [0, 1, 2, 4095, 4096, 8191, 8192, 8193]


def deliverers_case(k):
    """k routes on dl/#, each through its own deliverer; k = 0: only $oshare routes (every pair under the ordered id)"""
    kv = {}
    if k == 0:
        for i in range(20):
            groute(kv, "k", "dl/#", "o%d" % i, [O.receiver_url(0, "m%d" % i, "om")], ordered=True)
    for i in range(k):
        nroute(kv, "k", "dl/#", i % 3, "r%d" % i, "k%06d" % i)
    return sorted(kv.items()), ["k"], ["dl/x"], np.zeros(1, np.int32)


def inbox_case(n_tenants=1000, buckets=100, servers=4):
    """persistent sessions of n_tenants tenants, each spread over `buckets` inbox deliverers "<tenant>_NNNNN" (subBrokerId 1,
    the inbox service's key), plus transient sessions "<server>:<tenant>:<idx>" (subBrokerId 0): about 100k deliverers"""
    kv = {}
    tenants = ["tn%04d" % t for t in range(n_tenants)]
    for t in tenants:
        for b in range(buckets):
            nroute(kv, t, "s/#", 1, "inbox%d" % b, "%s_%05d" % (t, b))
        for s in range(servers):
            nroute(kv, t, "s/+", 0, "c%d" % s, "srv%d:%s:%d" % (s, t, s))
    return sorted(kv.items()), tenants, ["s/x"] * n_tenants, np.arange(n_tenants, dtype=np.int32)


NONASCII = b"\xe4\xbd\xa0\x00\xff"


def groups_case():
    """$share groups of 1, 2, 7 and 200 members next to normal routes that use some of the same deliverers; subBrokerIds 0, 1
    (persistent: capped) and 2; an empty delivererKey and non-ASCII bytes (a NUL and an invalid UTF-8 byte) in keys; an empty
    group; $oshare next to $share of the same group name on the same filter"""
    kv = {}
    dk = [(0, b"dA"), (1, b"dB"), (2, b"dC"), (0, b""), (1, NONASCII)]
    for i in range(12):
        b, d = dk[i % len(dk)]
        nroute(kv, "g", "grp/+", b, "n%d" % i, d)
    for i in range(6):
        nroute(kv, "g", "grp/#", 1, "p%d" % i, "dP")
    for n in (1, 2, 7, 200):
        # the first five members go through the normal routes' deliverers, the rest through their own
        urls = [O.receiver_url(dk[j][0], "s%d_%d" % (n, j), dk[j][1]) if j < len(dk)
                else O.receiver_url(j % 3, "s%d_%d" % (n, j), "m%03d" % j) for j in range(n)]
        groute(kv, "g", "grp/+", "s%d" % n, urls)
    seven = [O.receiver_url(j % 3, "o%d" % j, "m%03d" % j) for j in range(7)]
    groute(kv, "g", "grp/+", "s7", seven, ordered=True)
    groute(kv, "g", "grp/+", "empty", [])
    topics = ["grp/%d" % i for i in range(40)]
    return sorted(kv.items()), ["g"], topics, np.zeros(len(topics), np.int32)


def tier2_case():
    """a 7-level topic matching all 128 '+'/literal filters (> 64 ranges: tier 1, > 48: tier 2) next to topics whose
    persistent and group routes exceed the caps (3, 1)"""
    kv = {}
    lv = list("abcdefg")
    for mask in range(128):
        f = "/".join("+" if mask >> i & 1 else lv[i] for i in range(7))
        nroute(kv, "m", f, mask % 3 if mask % 3 != 1 else 2, "w%d" % mask, "w%d" % (mask % 11))
    for i in range(10):
        nroute(kv, "m", "cap/+", 1, "p%d" % i, "dp%d" % (i % 2))
    for i in range(5):
        groute(kv, "m", "cap/+", "g%d" % i, [O.receiver_url(0, "g%d" % i, "dg"), O.receiver_url(1, "h%d" % i, "dh")])
    topics = ["a/b/c/d/e/f/g", "cap/x", "a/b/c/d/e/f/g", "cap/y", "none"]
    return sorted(kv.items()), ["m"], topics, np.zeros(len(topics), np.int32)


def kv_of(pairs):
    kv = O.KV()
    for k, v in pairs:
        kv.put(k, v)
    kv.freeze()
    return kv


def oracle(pairs, tenants, topics, tt, caps=(INT_MAX, INT_MAX)):
    return kv_of(pairs).match_batch(tenants, topics, tt, caps[0], caps[1], O.MODE_TRIE, False, 8)


def decode(pairs, rank):
    """('N', (subBrokerId, delivererKey)) | ('S', [member deliverers in wire order]) | ('O', None): $oshare or empty group"""
    k, v = pairs[rank]
    m = O.build_match_route(k, v)
    if m["type"] == "Normal":
        return "N", O.deliverer_of_receiver_url(m["receiverUrl"])
    members = O.route_group_members_in_wire_order(v)
    if m["mqttTopicFilter"].startswith("$oshare/") or not members:
        return "O", None
    return "S", [O.deliverer_of_receiver_url(u) for u in members]


def deliverers_of(pairs, ranks):
    out = set()
    for r in set(int(x) for x in ranks):
        kind, d = decode(pairs, r)
        if kind == "N":
            out.add(d)
        elif kind == "S":
            out.update(d)
    return out


# ------------------------------------------------------------------ CPU: the generators land on their edges
@pytest.mark.parametrize("n_pairs", sorted(COUNT_SHAPES))
def test_count_shapes_land_on_their_pair_counts(n_pairs):
    pairs, tenants, topics, tt = count_case(*COUNT_SHAPES[n_pairs])
    want = oracle(pairs, tenants, topics, tt)
    assert int(want.offsets[-1]) == n_pairs
    if n_pairs >= 9:
        assert {decode(pairs, r)[0] for r in set(want.ranks.tolist())} == {"N", "S", "O"}


def test_hot_case_spans_three_tiles_between_empty_topics():
    want = oracle(*hot_case())
    assert np.diff(want.offsets).tolist() == [0, 12289, 0, 0, 12289, 0]
    assert 12289 > 3 * TILE


def test_boundary_case_ends_topics_at_chunk_and_tile_edges():
    want = oracle(*boundary_case())
    ends = set(want.offsets.tolist())
    for e in (CHUNK, CHUNK + 1, TILE, TILE + 1, 2 * TILE, 2 * TILE + 1, 3 * TILE, 3 * TILE + 1):
        assert e in ends
    assert 0 in np.diff(want.offsets).tolist()   # an empty topic between two tiles' worth


def test_one_bin_case_has_one_deliverer():
    pairs, tenants, topics, tt = one_bin_case()
    want = oracle(pairs, tenants, topics, tt)
    assert len(want.ranks) == 15000 and deliverers_of(pairs, want.ranks) == {(0, b"hot")}


@pytest.mark.parametrize("k", K_DELIVERERS)
def test_deliverers_case_has_k_deliverers(k):
    pairs, tenants, topics, tt = deliverers_case(k)
    want = oracle(pairs, tenants, topics, tt)
    kinds = [decode(pairs, int(r))[0] for r in want.ranks]
    assert len(deliverers_of(pairs, want.ranks)) == k and len(want.ranks) == max(k, 20 if k == 0 else k)
    assert k or set(kinds) == {"O"}


def test_inbox_case_has_about_100k_deliverers():
    pairs, tenants, topics, tt = inbox_case()
    want = oracle(pairs, tenants, topics, tt)
    ds = deliverers_of(pairs, want.ranks)
    assert len(ds) == 1000 * 100 + 1000 * 4 and len(want.ranks) == len(ds)
    assert {b for b, _ in ds} == {0, 1}


def test_groups_case_shapes():
    pairs, tenants, topics, tt = groups_case()
    want = oracle(pairs, tenants, topics, tt)
    dec = [decode(pairs, int(r)) for r in sorted(set(want.ranks.tolist()))]
    sizes = sorted(len(d) for k, d in dec if k == "S")
    assert sizes == [1, 2, 7, 200]
    normal = {d for k, d in dec if k == "N"}
    member = {x for k, d in dec if k == "S" for x in d}
    assert normal & member                                   # members share deliverers with normal routes
    assert {b for b, _ in normal} == {0, 1, 2} and (0, b"") in normal and (1, NONASCII) in normal
    assert sum(1 for k, _ in dec if k == "O") == 2            # the $oshare twin of s7 and the empty group
    keys = {O.build_match_route(*pairs[int(r)])["mqttTopicFilter"] for r in want.ranks}
    assert {"$share/s7/grp/+", "$oshare/s7/grp/+", "$share/empty/grp/+"} <= keys
    for caps in CAPS[1:]:
        capped = oracle(pairs, tenants, topics, tt, caps)
        assert len(capped.ranks) < len(want.ranks) or caps == (INT_MAX, 100)


def test_tier2_case_shapes():
    pairs, tenants, topics, tt = tier2_case()
    want = oracle(pairs, tenants, topics, tt, (3, 1))
    full = oracle(pairs, tenants, topics, tt)
    assert np.diff(full.offsets).tolist()[0] == 128 and np.diff(full.offsets).tolist()[1] == 15
    assert len(want.events) > 0 and np.diff(want.offsets).tolist()[1] == 3 + 1


# ------------------------------------------------------------------ GPU harness
@pytest.fixture(scope="module")
def B():
    import torch

    import bifromq_b200
    from bifromq_b200 import dist
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.pkg, ns.torch, ns.dist = bifromq_b200, torch, dist
    ns.dev = torch.device("cuda", 0)
    ns.stream = torch.cuda.current_stream(ns.dev).cuda_stream
    return ns


def make_index(B, pairs, path="auto"):
    idx = B.pkg.GpuRouteIndex(0)
    idx.load_pairs(pairs)
    idx.commit()
    if path == "global":
        idx.set_option("fanout_global", 1)
    return idx


def match_device(B, idx, tenants, topics, tt, caps=(INT_MAX, INT_MAX), wait=True):
    torch = B.torch
    blob, off = O.blob(topics)
    keep = [torch.from_numpy(blob).to(B.dev), torch.from_numpy(off).to(B.dev),
            torch.from_numpy(np.ascontiguousarray(tt, np.int32)).to(B.dev)]
    nt = len(tenants)
    out = idx.match_device(tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), len(topics),
                           [caps[0]] * nt, [caps[1]] * nt, B.stream, wait)
    out.keep = keep
    return out


def device_csr(B, out, n):
    torch = B.torch
    d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=B.dev)
    total = out.expand(d_offsets.data_ptr(), None, 0, B.stream)
    d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=B.dev)
    assert out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, B.stream) == total
    return d_offsets, d_ranks, total


def fanout_once(B, out, d_offsets, d_ranks, total):
    fo = out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, B.stream)
    B.torch.cuda.synchronize()
    D = fo.n_deliverers
    view = lambda p, n, t: B.dist.device_view(p, n, t, B.dev).cpu().numpy()
    n1 = max(total, 1)
    return {"D": D, "ordered": fo.ordered_share_id, "n_pairs": fo.n_pairs, "generation": fo.generation,
            "off": view(fo.d_pack_offsets, D + 1, "<i8"), "topic": view(fo.d_pack_topic, n1, "<u4")[:total].astype(np.int64),
            "rank": view(fo.d_pack_rank, n1, "<u4")[:total].astype(np.int64),
            "member": view(fo.d_pack_member, n1, "<u4")[:total].astype(np.int64)}


def pair_keys(topic, rank):
    return (np.asarray(topic, np.int64) << 32) | np.asarray(rank, np.int64)


def check(idx, got, csr_off, csr_ranks, want, pairs):
    """got: one fan-out call; (csr_off, csr_ranks) the device CSR it was given; want: the oracle's match of the generation
    whose sorted pair list is `pairs`. Returns per-kind pair counts and the (subBrokerId, delivererKey) -> id table the
    pairs were checked against (every id below the result's ordered_share_id)."""
    n = len(csr_off) - 1
    total = int(csr_off[-1])
    # the CSR holds the oracle's surviving ranks per topic (unordered within a topic)
    assert csr_off.tolist() == want.offsets.tolist()
    csr_topic = np.repeat(np.arange(n, dtype=np.int64), np.diff(csr_off))
    csr = np.sort(pair_keys(csr_topic, csr_ranks))
    assert np.array_equal(csr, np.sort(pair_keys(csr_topic, want.ranks)))
    D, od, off = got["D"], got["ordered"], got["off"]
    assert got["n_pairs"] == total and od == D - 1 and len(off) == D + 1
    assert off[0] == 0 and off[-1] == total and (np.diff(off) >= 0).all()
    pt, pr, pm = got["topic"], got["rank"], got["member"]
    assert np.array_equal(np.sort(pair_keys(pt, pr)), csr)
    dl = np.repeat(np.arange(D, dtype=np.int64), np.diff(off))
    # expectations per distinct rank, from the pair list and the oracle's decoders
    uniq = np.unique(pr)
    ids = {}
    for d in range(od):
        ids[idx.deliverer(d)] = d
    assert len(ids) == od                                       # ids are distinct pairs
    kind = np.zeros(len(uniq), np.int64)                        # 0 normal, 1 $share, 2 parked under the ordered id
    nid = np.full(len(uniq), -1, np.int64)
    moff = np.zeros(len(uniq) + 1, np.int64)
    mids = []
    for u, r in enumerate(uniq.tolist()):
        k, d = decode(pairs, r)
        if k == "N":
            nid[u] = ids[d]
        elif k == "S":
            kind[u] = 1
            mids += [ids[x] for x in d]
        else:
            kind[u] = 2
        moff[u + 1] = len(mids)
    mids = np.asarray(mids + [0], np.int64)
    u = np.searchsorted(uniq, pr)
    k = kind[u]
    norm, share, park = k == 0, k == 1, k == 2
    assert (dl[norm] == nid[u[norm]]).all() and (pm[norm] == NO_MEMBER).all()
    assert (dl[park] == od).all() and (pm[park] == NO_MEMBER).all()
    nmem = moff[u + 1] - moff[u]
    assert (pm[share] < nmem[share]).all()
    pick = np.where(share, moff[u] + np.where(pm < nmem, pm, 0), 0)
    assert (dl[share] == mids[pick[share]]).all()
    return {"normal": int(norm.sum()), "share": int(share.sum()), "parked": int(park.sum()), "ids": ids}


def same_map(a, b):
    """two fan-out calls on the same CSR: the same (topic, rank) -> (deliverer, member); order within a deliverer is free"""
    def m(g):
        keys = pair_keys(g["topic"], g["rank"])
        o = np.argsort(keys)
        dl = np.repeat(np.arange(g["D"], dtype=np.int64), np.diff(g["off"]))
        return keys[o], dl[o], g["member"][o]
    for x, y in zip(m(a), m(b)):
        assert np.array_equal(x, y)


def fan_check(B, idx, out, topics, want, pairs):
    """expand + two fan-out calls on one completed match, both checked; returns the first call and check()'s summary"""
    d_offsets, d_ranks, total = device_csr(B, out, len(topics))
    B.torch.cuda.synchronize()
    csr_off = d_offsets.cpu().numpy()
    csr_ranks = d_ranks.cpu().numpy()[:total]
    a = fanout_once(B, out, d_offsets, d_ranks, total)
    b = fanout_once(B, out, d_offsets, d_ranks, total)
    same_map(a, b)
    s = check(idx, a, csr_off, csr_ranks, want, pairs)
    a["csr"] = (d_offsets, d_ranks, total)
    return a, s


def run_case(B, case, path="auto", caps=(INT_MAX, INT_MAX), idx=None):
    pairs, tenants, topics, tt = case
    own = idx is None
    if own:
        idx = make_index(B, pairs, path)
    want = oracle(pairs, tenants, topics, tt, caps)
    before = idx.stats()["global_fanouts"]
    out = match_device(B, idx, tenants, topics, tt, caps)
    got, s = fan_check(B, idx, out, topics, want, pairs)
    taken = idx.stats()["global_fanouts"] - before
    tiled = expect_tiled(got["D"], got["n_pairs"])
    if path == "global":
        assert taken == 2
    else:
        assert taken == (0 if tiled else 2), (got["D"], got["n_pairs"])
    # the other setting of the option on the same CSR: where the auto choice is the tile pass, the two passes must give
    # the same (topic, rank) -> (deliverer, member) map, member picks included
    idx.set_option("fanout_global", 0 if path == "global" else 1)
    before = idx.stats()["global_fanouts"]
    other = fanout_once(B, out, *got["csr"])
    assert idx.stats()["global_fanouts"] - before == (0 if path == "global" and tiled else 1)
    same_map(got, other)
    idx.set_option("fanout_global", 1 if path == "global" else 0)
    out.release()
    if own:
        idx.close()
    return got, s


# ------------------------------------------------------------------ GPU: shapes
@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("n_pairs", sorted(COUNT_SHAPES))
def test_fanout_pair_counts(B, n_pairs, path):
    got, s = run_case(B, count_case(*COUNT_SHAPES[n_pairs]), path)
    assert got["n_pairs"] == n_pairs
    if n_pairs >= 9:
        assert s["normal"] and s["share"] and s["parked"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_fanout_hot_topic_over_three_tiles(B, path):
    got, s = run_case(B, hot_case(), path)
    assert got["n_pairs"] == 2 * 12289 and set(got["topic"].tolist()) == {1, 4}


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_fanout_topic_ends_at_chunk_and_tile_edges(B, path):
    got, s = run_case(B, boundary_case(), path)
    counts = np.bincount(got["topic"], minlength=len(BOUNDARY_COUNTS)).tolist()
    assert counts == BOUNDARY_COUNTS


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_fanout_every_pair_under_one_deliverer(B, path):
    got, s = run_case(B, one_bin_case(), path)
    sizes = np.diff(got["off"])
    assert sizes.max() == 15000 and (sizes > 0).sum() == 1


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("k", K_DELIVERERS)
def test_fanout_distinct_deliverers(B, k, path):
    got, s = run_case(B, deliverers_case(k), path)
    if path == "auto" and k in (4095, 4096):
        assert expect_tiled(k + 1, k) == (k == 4095)
    if k == 0:
        assert s["parked"] == 20 and s["normal"] == 0 and np.diff(got["off"])[got["ordered"]] == 20
    else:
        assert got["D"] == k + 1 and s["normal"] == k and (np.diff(got["off"])[:k] == 1).all()


@pytest.mark.gpu
def test_fanout_inbox_scale_deliverers(B):
    got, s = run_case(B, inbox_case())
    assert got["D"] == 104000 + 1 and s["normal"] == 104000


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("caps", CAPS)
def test_fanout_groups_members_and_caps(B, caps, path):
    got, s = run_case(B, groups_case(), path, caps)
    if caps[1] >= 100:
        assert s["share"] > 0 and s["parked"] > 0
    elif caps[1] == 1:
        assert s["share"] + s["parked"] == 40                              # one group route per topic survives
    if caps == (0, 0):
        assert s["share"] == 0 and s["parked"] == 0 and s["normal"] > 0   # only the uncapped transient routes survive


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_fanout_repeated_topics_in_locality_order(B, path):
    pairs, tenants, topics, tt = groups_case()
    rng = np.random.default_rng(11)
    many = [topics[i] for i in rng.integers(0, 10, 600)]
    idx = make_index(B, pairs, path)
    idx.set_option("order_min_topics", 64)
    before = idx.stats()["duplicate_topics"]
    got, s = run_case(B, (pairs, tenants, many, np.zeros(600, np.int32)), path, (3, 1), idx)
    assert idx.stats()["duplicate_topics"] - before >= 590
    assert set(got["topic"].tolist()) == set(range(600))   # every occurrence has its own pairs under its own position
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_fanout_mixes_tier2_and_capped_topics(B, path):
    pairs, tenants, topics, tt = tier2_case()
    idx = make_index(B, pairs, path)
    st = idx.stats()
    run_case(B, (pairs, tenants, topics, tt), path, (3, 1), idx)
    st2 = idx.stats()
    assert st2["overflow_topics"] - st["overflow_topics"] == 2 and st2["flagged_topics"] - st["flagged_topics"] >= 2
    idx.close()


# ------------------------------------------------------------------ GPU: spread of the $share member pick
def member_counts(got, n):
    m = got["member"][got["member"] != NO_MEMBER]
    return np.bincount(m, minlength=n)


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_share_pick_spreads_over_topics(B, path):
    """one 7-member group matched by 50k distinct topics: the rank is fixed, the topic position varies"""
    from scipy.stats import chisquare
    kv = {}
    groute(kv, "u", "spread/+", "g7", [O.receiver_url(0, "m%d" % j, "d%d" % j) for j in range(7)])
    topics = ["spread/%d" % i for i in range(50000)]
    got, s = run_case(B, (sorted(kv.items()), ["u"], topics, np.zeros(len(topics), np.int32)), path)
    c = member_counts(got, 7)
    assert c.sum() == 50000 and chisquare(c).pvalue > 1e-6, c


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_share_pick_spreads_over_routes(B, path):
    """one topic matching 7000 $share routes with the same 7 members: the topic position is fixed, the rank varies"""
    from scipy.stats import chisquare
    kv = {}
    members = [O.receiver_url(0, "m%d" % j, "d%d" % j) for j in range(7)]
    for g in range(7000):
        groute(kv, "u", "hot", "g%d" % g, members)
    got, s = run_case(B, (sorted(kv.items()), ["u"], ["hot"], np.zeros(1, np.int32)), path)
    c = member_counts(got, 7)
    assert c.sum() == 7000 and chisquare(c).pvalue > 1e-6, c


# ------------------------------------------------------------------ GPU: commits and snapshots
class Gen:
    """the KV a test feeds the handle, and the sorted pair list of every committed generation"""

    def __init__(self, kv):
        self.kv = dict(kv)

    def pairs(self):
        return sorted(self.kv.items())


DELTA_TENANTS = ["t1", "t2", "t25", "t3", "t4", "tz"]


def delta_start():
    kv = {}
    for t in ("t1", "t2", "t3", "t4"):
        mixed_routes(kv, t, "x/#", 20, tag=t)
    nroute(kv, "t2", "x/1", 0, "lonely", "lonely")
    groute(kv, "t2", "x/+", "gg", [O.receiver_url(0, "a", "ga"), O.receiver_url(1, "b", "gb")])
    for i in range(3000):   # no node with more than 60 children: a wide node would make every commit a full build
        nroute(kv, "tz", "big/%d/%d" % (i // 50, i % 50), 0, "z", "dz%d" % (i % 4))
    return kv


def delta_topics():
    topics, tt = [], []
    for i, t in enumerate(DELTA_TENANTS):
        for topic in ("x/1", "x/2", "big/7/3"):
            topics.append(topic)
            tt.append(i)
    return topics, np.array(tt, np.int32)


def check_generation(B, idx, g, known_ids):
    topics, tt = delta_topics()
    pairs = g.pairs()
    want = oracle(pairs, DELTA_TENANTS, topics, tt)
    out = match_device(B, idx, DELTA_TENANTS, topics, tt)
    assert out.generation == idx.generation()
    got, s = fan_check(B, idx, out, topics, want, pairs)
    out.release()
    for p, i in s["ids"].items():
        assert known_ids.setdefault(p, i) == i, p     # a pair seen before keeps its id
    for p, i in known_ids.items():
        assert idx.deliverer(i) == p
    return got, s


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_fanout_after_delta_full_and_reset(B, path):
    g = Gen(delta_start())
    idx = make_index(B, g.pairs(), path)
    known = {}
    check_generation(B, idx, g, known)

    def commit(adds=(), dels=(), expect="delta"):
        st = idx.stats()
        for k, v in adds:
            g.kv[k] = v
        for k in dels:
            del g.kv[k]
        idx.apply(adds=adds, dels=dels)
        idx.commit()
        st2 = idx.stats()
        took = "delta" if st2["delta_commits"] == st["delta_commits"] + 1 else "full"
        assert st2["delta_commits"] + st2["full_commits"] == st["delta_commits"] + st["full_commits"] + 1
        if expect:
            assert took == expect
        got, s = check_generation(B, idx, g, known)
        return took, st, got
    # a SUB with a new deliverer into a middle tenant: the ranks of t3, t4 and tz move by one
    add = {}
    nroute(add, "t2", "x/+", 0, "newcomer", "new1")
    commit(list(add.items()))
    assert (0, b"new1") in known
    # an UNSUB of a deliverer's last route
    lonely = O.route_key("t2", "x/1", O.receiver_url(0, "lonely", "lonely"))
    commit(dels=[lonely])
    # a $share join: the group value is upserted with one more member, through a new deliverer
    add = {}
    groute(add, "t2", "x/+", "gg", [O.receiver_url(0, "a", "ga"), O.receiver_url(1, "b", "gb"), O.receiver_url(2, "c", "gc")])
    commit(list(add.items()))
    assert (2, b"gc") in known
    # a new tenant and a removed tenant in one commit
    add = {}
    mixed_routes(add, "t25", "x/#", 10, tag="n")
    commit(list(add.items()), dels=[k for k in g.kv if O.build_match_route(k, g.kv[k])["tenantId"] == "t4"])
    # the big tenant touched until the garbage bound turns a commit into a full build
    for i in range(20):
        add = {}
        nroute(add, "tz", "big/%d/0" % i, 0, "z%d" % i, "dz%d" % (i % 4))
        took, st, _ = commit(list(add.items()), expect=None)
        bound = st["slots"] // 4 + 4096
        assert took == ("full" if st["garbage_slots"] > bound else "delta"), (i, st)
        if took == "full":
            break
    assert took == "full"
    # reset + reload of the same KV: every id seen so far is kept
    n_ids = len(known)
    idx.reset()
    idx.load_pairs(g.pairs())
    st = idx.stats()
    idx.commit()
    assert idx.stats()["full_commits"] == st["full_commits"] + 1
    check_generation(B, idx, g, known)
    assert len(known) == n_ids
    idx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fan_first", [True, False])
def test_old_result_fans_out_against_its_own_snapshot(B, fan_first):
    """a result taken before a commit resolves its fan-out against its own snapshot: old ranks, the group's old member list,
    and an ordered_share_id that separates its parked pairs even after a newer snapshot interned more deliverers"""
    g = Gen(delta_start())
    old_pairs = g.pairs()
    idx = make_index(B, old_pairs)
    topics, tt = delta_topics()
    want_old = oracle(old_pairs, DELTA_TENANTS, topics, tt)
    out_old = match_device(B, idx, DELTA_TENANTS, topics, tt)
    if fan_first:
        first, _ = fan_check(B, idx, out_old, topics, want_old, old_pairs)
    # a route sorting first in t1 shifts every rank; the group gains a member through a new deliverer; new deliverers appear
    add = {}
    nroute(add, "t1", "!first", 0, "f", "brand-new")
    groute(add, "t2", "x/+", "gg", [O.receiver_url(0, "a", "ga"), O.receiver_url(1, "b", "gb"), O.receiver_url(2, "c", "late")])
    for i in range(5):
        nroute(add, "t3", "x/2", 0, "late%d" % i, "late%d" % i)
    g.kv.update(add)
    idx.apply(adds=list(add.items()))
    idx.commit()
    new_pairs = g.pairs()
    want_new = oracle(new_pairs, DELTA_TENANTS, topics, tt)
    out_new = match_device(B, idx, DELTA_TENANTS, topics, tt)
    new, _ = fan_check(B, idx, out_new, topics, want_new, new_pairs)
    old, s = fan_check(B, idx, out_old, topics, want_old, old_pairs)
    assert s["parked"] > 0 and out_old.generation == new["generation"] - 1 == old["generation"]
    if fan_first:
        assert old["ordered"] == first["ordered"] < new["ordered"]
        assert old["ordered"] < new["D"] - 1           # the old ordered id is a real deliverer of the newer snapshot
    out_old.release()
    out_new.release()
    idx.close()


@pytest.mark.gpu
def test_fanout_on_old_result_while_a_delta_commit_runs(B):
    """the commit copies the old snapshot's per-tenant fan-out tables under their lock while the fan-out fills them in"""
    g = Gen(delta_start())
    old_pairs = g.pairs()
    idx = make_index(B, old_pairs)
    topics, tt = delta_topics()
    want_old = oracle(old_pairs, DELTA_TENANTS, topics, tt)
    out_old = match_device(B, idx, DELTA_TENANTS, topics, tt)
    add = {}
    for t in ("t1", "t2", "t3"):
        nroute(add, t, "x/+", 0, "during", "during-" + t)
    g.kv.update(add)
    idx.apply(adds=list(add.items()))
    st = idx.stats()
    errs = []

    def committer():
        try:
            idx.commit()
        except Exception as e:   # pragma: no cover
            errs.append(e)
    th = threading.Thread(target=committer)
    th.start()
    fan_check(B, idx, out_old, topics, want_old, old_pairs)
    th.join()
    assert not errs, errs
    assert idx.stats()["delta_commits"] == st["delta_commits"] + 1
    out_old.release()
    topics, tt = delta_topics()
    new_pairs = g.pairs()
    out = match_device(B, idx, DELTA_TENANTS, topics, tt)
    fan_check(B, idx, out, topics, oracle(new_pairs, DELTA_TENANTS, topics, tt), new_pairs)
    out.release()
    idx.close()


# ------------------------------------------------------------------ GPU: errors
def bfq_code(e):
    return int(str(e).split("bfq error ")[1].split(":")[0])


@pytest.mark.gpu
def test_fanout_argument_and_state_errors(B):
    from bifromq_b200._native import NativeError
    pairs, tenants, topics, tt = groups_case()
    idx = make_index(B, pairs)
    out = match_device(B, idx, tenants, topics, tt, wait=False)
    d_offsets = B.torch.zeros(len(topics) + 1, dtype=B.torch.int64, device=B.dev)
    d_ranks = B.torch.zeros(1, dtype=B.torch.int64, device=B.dev)
    with pytest.raises(NativeError) as e:
        out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), 0, B.stream)
    assert bfq_code(e.value) == -4                        # BFQ_E_STATE: not waited yet
    out.wait()
    d_offsets, d_ranks, total = device_csr(B, out, len(topics))
    for n_pairs, ranks in ((-1, d_ranks.data_ptr()), (total, None)):
        with pytest.raises(NativeError) as e:
            out.fanout(d_offsets.data_ptr(), ranks, n_pairs, B.stream)
        assert bfq_code(e.value) == -1                    # BFQ_E_INVALID
    got = fanout_once(B, out, d_offsets, d_ranks, total)  # the handle is still usable
    assert got["n_pairs"] == total > 0
    out.release()
    idx.close()


@pytest.mark.gpu
def test_receiver_url_without_deliverer_key_fails_fanout_only(B):
    from bifromq_b200._native import NativeError
    kv = {}
    nroute(kv, "v", "a/+", 0, "ok", "d")
    kv[O.route_key("v", "a/b", b"0\x00no-deliverer-key")] = O.incarnation_bytes(1)   # one NUL: no delivererKey
    pairs = sorted(kv.items())
    idx = make_index(B, pairs)                             # the load accepts the key
    want = oracle(pairs, ["v"], ["a/b"], np.zeros(1, np.int32))
    out = match_device(B, idx, ["v"], ["a/b"], np.zeros(1, np.int32))
    d_offsets, d_ranks, total = device_csr(B, out, 1)
    B.torch.cuda.synchronize()
    assert total == 2 and d_offsets.cpu().numpy().tolist() == want.offsets.tolist()
    with pytest.raises(NativeError) as e:
        out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, B.stream)
    assert bfq_code(e.value) == -1
    out.release()
    res = idx.match_topics(["v"], ["a/b", "a/c"])          # matching on the handle still works
    offsets, ranks = res.expand()
    assert offsets.tolist() == [0, 2, 3]
    res.close()
    idx.close()
