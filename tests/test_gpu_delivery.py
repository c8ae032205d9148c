"""Delivery requests on the device (bfq_delivery_device) against a literal restatement of the deliverer's batcher.

BatchDeliveryCall.add / execute (bifromq-deliverer/.../BatchDeliveryCall.java:58,75-104) nests the calls a deliverer gets as
tenantId -> TopicMessagePackHolder -> Set<MatchInfo> and sends that map as one DeliveryRequest. batch_delivery() below says
the same thing in plain Python: topic positions in batch order, each surviving route of a position mapped to its deliverer
with oracle_lib.deliverer_of_receiver_url ($share members from the fan-out's pick, $oshare and member-less groups under the
ordered-share id), appended to batch[deliverer][tenant][position]. The CPU tests pin that restatement on hand-built cases;
the GPU tests compare the device's nesting with it exactly (package sets per deliverer, pack order, MatchInfo sets) and,
pair for pair as sets, with bfq_fanout_device on the same result.
"""
import functools
import threading

import numpy as np
import pytest

import oracle_lib as O
import test_gpu_fanout as F
import test_gpu_fanout_budget as FB

INT_MAX = 2 ** 31 - 1
NO_MEMBER = 0xFFFFFFFF
ORDERED = "ordered-share"


# ------------------------------------------------------------------ the restatement (no GPU)
def batch_delivery(topic_tenant, n_tenants, offsets, ranks, route_of, pick):
    """route_of(rank) -> ('N', deliverer) | ('S', [member deliverers in wire order]) | ('O', None) ($oshare or no member);
    pick(position, rank) -> the member index a $share route was resolved to.
    -> {deliverer: {tenant index: [(position, {(rank, member), ...}), ...]}}, packs in the order add() saw them"""
    batch = {}
    for t in range(len(offsets) - 1):                      # the request's packs, submitted in order
        tenant = int(topic_tenant[t])
        if not 0 <= tenant < n_tenants:                    # the match gives such a position no routes
            continue
        for r in ranks[int(offsets[t]):int(offsets[t + 1])]:
            r = int(r)
            kind, d = route_of(r)
            member = NO_MEMBER
            if kind == "S":
                member = pick(t, r)
                d = d[member]
            elif kind == "O":
                d = ORDERED
            # add(): tenantId -> TopicMessagePackHolder (one per pack, so per position) -> Set<MatchInfo>
            batch.setdefault(d, {}).setdefault(tenant, {}).setdefault(t, set()).add((r, member))
    return {d: {tn: list(packs.items()) for tn, packs in pkgs.items()} for d, pkgs in batch.items()}


# ranks of a hand-built route table: 0 -> deliverer a, 1 -> a $share over (a, b), 5 -> b, 6 -> $oshare, 7 -> empty group
HAND_ROUTES = {0: ("N", "a"), 1: ("S", ["a", "b"]), 5: ("N", "b"), 6: ("O", None), 7: ("O", None)}


def hand_csr(rows):
    off = np.zeros(len(rows) + 1, np.int64)
    off[1:] = np.cumsum([len(r) for r in rows])
    return off, np.asarray([x for r in rows for x in r], np.int64)


def test_restatement_interleaved_tenants_repeats_groups_and_empty_topic():
    # positions: 0 (tenant 1), 1 (tenant 0), 2 (tenant 1: repeats 0's topic), 3 (tenant 0, no routes), 4 (tenant 0: repeats 1)
    rows = [[5, 6], [0, 1], [5, 7], [], [0, 1]]
    tt = [1, 0, 1, 0, 0]
    off, ranks = hand_csr(rows)
    picks = {(1, 1): 0, (4, 1): 1}                         # the same group resolved to a member on each deliverer
    got = batch_delivery(tt, 2, off, ranks, HAND_ROUTES.__getitem__, lambda t, r: picks[(t, r)])
    assert got == {
        "a": {0: [(1, {(0, NO_MEMBER), (1, 0)}), (4, {(0, NO_MEMBER)})]},
        "b": {1: [(0, {(5, NO_MEMBER)}), (2, {(5, NO_MEMBER)})], 0: [(4, {(1, 1)})]},
        ORDERED: {1: [(0, {(6, NO_MEMBER)}), (2, {(7, NO_MEMBER)})]},
    }
    assert list(got["b"]) == [1, 0]                        # tenants in first-seen order: the batch interleaves them


def test_restatement_drops_positions_outside_the_tenant_list():
    off, ranks = hand_csr([[0], [0], [5]])
    got = batch_delivery([0, 2, -1], 2, off, ranks, HAND_ROUTES.__getitem__, None)
    assert got == {"a": {0: [(0, {(0, NO_MEMBER)})]}}


def test_restatement_of_an_oracle_match_holds_every_pair_once():
    pairs, tenants, topics, tt = F.groups_case()
    want = F.oracle(pairs, tenants, topics, tt)
    got = batch_delivery(tt, 1, want.offsets, want.ranks, functools.partial(F.decode, pairs), lambda t, r: 0)
    flat = [(t, r) for pkgs in got.values() for packs in pkgs.values() for t, ms in packs for r, _ in ms]
    topic = np.repeat(np.arange(len(topics)), np.diff(want.offsets))
    assert sorted(flat) == sorted(zip(topic.tolist(), want.ranks.tolist()))
    assert ORDERED in got and len(got) > 3


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


def read_fanout(B, fo, total):
    view = lambda p, n, t: B.dist.device_view(p, n, t, B.dev).cpu().numpy()
    n1 = max(total, 1)
    D = fo.n_deliverers
    off = view(fo.d_pack_offsets, D + 1, "<i8")
    return {"D": D, "deliverer": np.repeat(np.arange(D, dtype=np.int64), np.diff(off)),
            "topic": view(fo.d_pack_topic, n1, "<u4")[:total].astype(np.int64),
            "rank": view(fo.d_pack_rank, n1, "<u4")[:total].astype(np.int64),
            "member": view(fo.d_pack_member, n1, "<u4")[:total].astype(np.int64)}


def rows(deliverer, topic, rank, member):
    """(deliverer, topic, rank, member) rows, sorted, as one int array per column"""
    a = np.stack([np.asarray(x, np.int64) for x in (deliverer, topic, rank, member)], axis=1)
    return a[np.lexsort(a.T[::-1])] if len(a) else a


def check_structure(a, dl, tt):
    D, P, K, n = dl.n_deliverers, dl.n_packages, dl.n_packs, dl.n_pairs
    po, pt, ko, kt, mo = a["package_off"], a["package_tenant"], a["pack_off"], a["pack_topic"], a["match_off"]
    assert len(po) == D + 1 and po[0] == 0 and po[-1] == P and (np.diff(po) >= 0).all()
    assert len(ko) == P + 1 and ko[0] == 0 and ko[-1] == K and (np.diff(ko) > 0).all()      # no empty package
    assert len(mo) == K + 1 and mo[0] == 0 and mo[-1] == n and (np.diff(mo) > 0).all()      # no empty pack
    pkg_d = np.repeat(np.arange(D), np.diff(po))
    same_d = pkg_d[1:] == pkg_d[:-1]
    assert (pt[1:][same_d] > pt[:-1][same_d]).all()        # each tenant once per deliverer, ascending
    pack_p = np.repeat(np.arange(P), np.diff(ko))
    same_p = pack_p[1:] == pack_p[:-1]
    assert (kt[1:][same_p] > kt[:-1][same_p]).all()        # packs in ascending topic position inside a package
    assert (np.asarray(tt, np.int64)[kt] == pt[pack_p]).all()   # a pack's position belongs to its package's tenant
    key = (np.repeat(np.arange(K), np.diff(mo)) << 32) | a["match_rank"]
    assert len(np.unique(np.stack([key, a["match_member"]]), axis=1)[0]) == n       # no MatchInfo twice in a pack
    return pkg_d, pack_p


def nest_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, d_tt, pairs):
    """fan-out then delivery on one completed match; both compared with each other and with batch_delivery().
    -> (the delivery result, its host arrays, the nesting)"""
    fo = out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, B.stream)
    dl = out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), B.stream)
    fan = read_fanout(B, fo, total)                         # read after the delivery call: its buffers are its own
    a = dl.arrays(B.dev)
    got = dl.nesting(B.dev)
    B.torch.cuda.synchronize()
    csr_off = d_offsets.cpu().numpy()
    csr_ranks = d_ranks.cpu().numpy()[:total]
    assert dl.n_deliverers == fan["D"] and dl.ordered_share_id == fan["D"] - 1 and dl.generation == out.generation
    pkg_d, pack_p = check_structure(a, dl, tt)
    # pair for pair, as sets, the fan-out's (deliverer, topic, rank, member) on the same result and CSR
    pair_pack = np.repeat(np.arange(dl.n_packs), np.diff(a["match_off"]))
    pair_d = pkg_d[pack_p[pair_pack]] if dl.n_pairs else np.zeros(0, np.int64)
    mine = rows(pair_d, a["pack_topic"][pair_pack], a["match_rank"], a["match_member"])
    valid = np.isin(fan["topic"], np.flatnonzero((np.asarray(tt) >= 0) & (np.asarray(tt) < len(tenants))))
    theirs = rows(*(fan[k][valid] for k in ("deliverer", "topic", "rank", "member")))
    assert np.array_equal(mine, theirs)
    # the restatement, with the fan-out's member picks, deliverers decoded from the KV and mapped to the handle's ids
    picks = dict(zip(zip(fan["topic"].tolist(), fan["rank"].tolist()), fan["member"].tolist()))
    ids = {idx.deliverer(d): d for d in range(dl.ordered_share_id)}
    ids[ORDERED] = dl.ordered_share_id
    route_of = functools.lru_cache(maxsize=None)(lambda r: F.decode(pairs, r))
    want = batch_delivery(tt, len(tenants), csr_off, csr_ranks, route_of, lambda t, r: picks[(t, r)])
    want = {ids[d]: pkgs for d, pkgs in want.items()}
    assert got == want
    return dl, a, got


def run_case(B, case, caps=(INT_MAX, INT_MAX), idx=None):
    pairs, tenants, topics, tt = case
    own = idx is None
    if own:
        idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt, caps)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    B.torch.cuda.synchronize()
    # the oracle takes in-range tenant indexes only; a position outside the list has no routes
    tt = np.asarray(tt, np.int32)
    ok = np.flatnonzero((tt >= 0) & (tt < len(tenants)))
    want = F.oracle(pairs, tenants, [topics[i] for i in ok], tt[ok], caps)
    counts = np.zeros(len(topics), np.int64)
    counts[ok] = np.diff(want.offsets)
    assert np.array_equal(np.diff(d_offsets.cpu().numpy()), counts)
    r = nest_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs)
    out.release()
    if own:
        idx.close()
    return r


# ------------------------------------------------------------------ GPU: the fan-out's shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["one_bin", "hot", "boundary", "groups"])
def test_delivery_fanout_shapes(B, name):
    case = {"one_bin": F.one_bin_case, "hot": F.hot_case, "boundary": F.boundary_case, "groups": F.groups_case}[name]()
    dl, a, got = run_case(B, case)
    if name == "one_bin":
        assert len(got) == 1 and dl.n_packages == 1 and dl.n_packs == 3 and dl.n_pairs == 15000
    if name == "hot":
        assert all(len(pkgs) == 1 and {t for t, _ in pkgs[0]} <= {1, 4} for pkgs in got.values())
        assert any([t for t, _ in pkgs[0]] == [1, 4] for pkgs in got.values())


@pytest.mark.gpu
@pytest.mark.parametrize("k", [0, 1, 2, 4096, 8193])
def test_delivery_distinct_deliverers(B, k):
    dl, a, got = run_case(B, F.deliverers_case(k))
    if k == 0:
        assert list(got) == [dl.ordered_share_id] and dl.n_pairs == 20
    else:
        assert len(got) == k and dl.n_packages == k and dl.n_packs == k


@pytest.mark.gpu
def test_delivery_inbox_scale_deliverers(B):
    dl, a, got = run_case(B, F.inbox_case())
    assert dl.n_deliverers == 104000 + 1 and len(got) == 104000 and dl.n_packages == 104000


@pytest.mark.gpu
@pytest.mark.parametrize("caps", F.CAPS)
def test_delivery_groups_members_and_caps(B, caps):
    run_case(B, F.groups_case(), caps)


@pytest.mark.gpu
def test_delivery_tier2_and_capped_topics(B):
    pairs, tenants, topics, tt = F.tier2_case()
    idx = F.make_index(B, pairs)
    st = idx.stats()
    dl, a, got = run_case(B, (pairs, tenants, topics, tt), (3, 1), idx)
    st2 = idx.stats()
    assert st2["overflow_topics"] - st["overflow_topics"] == 2 and st2["flagged_topics"] - st["flagged_topics"] >= 2
    assert any(len(packs) >= 2 for pkgs in got.values() for packs in pkgs.values())   # the repeated tier-2 topic: 2 packs
    idx.close()


# ------------------------------------------------------------------ GPU: interleaved tenants, repeated topics
def interleaved_case(n_tenants=5, n=600, seed=3):
    """tenants whose routes go through the same deliverers, positions of all tenants interleaved, topics repeated, one
    position with a tenant index outside the list and one with no routes"""
    kv = {}
    tenants = ["it%d" % i for i in range(n_tenants)]
    for i, tn in enumerate(tenants):
        for j in range(6):
            F.nroute(kv, tn, "x/+", j % 2, "r%d_%d" % (i, j), "shared%d" % (j % 3))
        F.groute(kv, tn, "x/#", "g", [O.receiver_url(0, "m%d" % i, "shared0"), O.receiver_url(1, "m%d" % i, "own%d" % i)])
        F.groute(kv, tn, "x/1", "g", [O.receiver_url(0, "o%d" % i, "shared1")], ordered=True)
    rng = np.random.default_rng(seed)
    tt = rng.integers(0, n_tenants, n).astype(np.int32)
    topics = ["x/%d" % v for v in rng.integers(0, 4, n)]
    tt[7] = n_tenants + 2
    topics[9] = "y/none"
    return sorted(kv.items()), tenants, topics, tt


@pytest.mark.gpu
def test_delivery_interleaved_tenants_one_package_each(B):
    pairs, tenants, topics, tt = interleaved_case()
    dl, a, got = run_case(B, (pairs, tenants, topics, tt))
    shared = [d for d, pkgs in got.items() if len(pkgs) == len(tenants)]
    assert shared                                          # deliverers that serve every tenant: one package per tenant
    assert all(7 not in [t for packs in pkgs.values() for t, _ in packs] for pkgs in got.values())


@pytest.mark.gpu
def test_delivery_repeated_topics_in_locality_order(B):
    pairs, tenants, topics, tt = interleaved_case(n=40000, seed=8)
    idx = F.make_index(B, pairs)
    before = idx.stats()["duplicate_topics"]
    dl, a, got = run_case(B, (pairs, tenants, topics, tt), idx=idx)
    assert len(topics) >= 32768 and idx.stats()["duplicate_topics"] - before > 30000
    # every occurrence of a repeated (tenant, topic) is a pack of its own
    assert any(len(packs) > len({topics[t] for t, _ in packs}) for pkgs in got.values() for packs in pkgs.values())
    assert dl.n_packs > sum(len({topics[t] for t, _ in packs}) for pkgs in got.values() for packs in pkgs.values())
    idx.close()


# ------------------------------------------------------------------ GPU: the budgeted CSR
@pytest.mark.gpu
def test_delivery_of_a_budgeted_csr(B):
    case = FB.batch_case()
    idx = F.make_index(B, case.pairs)
    out = FB.match(B, idx, case)
    got = FB.budget(B, out, case)
    r = got["r"]
    assert r.n_dropped_bytes > 0 and r.n_dropped_persistent_bandwidth > 0 and r.n_dropped_transient_bandwidth > 0
    dl, a, nest = nest_check(B, idx, out, case.tenants, case.tt, got["d_off"], got["d_ranks"], got["total"], out.keep[2],
                             case.pairs)
    assert dl.n_pairs == got["total"]
    out.release()
    idx.close()


# ------------------------------------------------------------------ GPU: snapshots
@pytest.mark.gpu
def test_delivery_on_old_result_while_a_delta_commit_runs(B):
    g = F.Gen(F.delta_start())
    old_pairs = g.pairs()
    idx = F.make_index(B, old_pairs)
    topics, tt = F.delta_topics()
    out_old = F.match_device(B, idx, F.DELTA_TENANTS, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out_old, len(topics))
    add = {}
    for t in ("t1", "t2", "t3"):
        F.nroute(add, t, "x/+", 0, "during", "during-" + t)
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
    dl, _, _ = nest_check(B, idx, out_old, F.DELTA_TENANTS, tt, d_offsets, d_ranks, total, out_old.keep[2], old_pairs)
    th.join()
    assert not errs, errs
    assert idx.stats()["delta_commits"] == st["delta_commits"] + 1 and dl.generation == out_old.generation
    out_old.release()
    new_pairs = g.pairs()
    out = F.match_device(B, idx, F.DELTA_TENANTS, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    dl, _, got = nest_check(B, idx, out, F.DELTA_TENANTS, tt, d_offsets, d_ranks, total, out.keep[2], new_pairs)
    assert dl.generation == out.generation > out_old.generation
    assert any((0, b"during-t1") == idx.deliverer(d) for d in got)
    out.release()
    idx.close()


# ------------------------------------------------------------------ GPU: errors
@pytest.mark.gpu
def test_delivery_argument_and_state_errors(B):
    from bifromq_b200._native import NativeError
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt, wait=False)
    d_tt = out.keep[2].data_ptr()
    d_offsets = B.torch.zeros(len(topics) + 1, dtype=B.torch.int64, device=B.dev)
    d_ranks = B.torch.zeros(1, dtype=B.torch.int64, device=B.dev)
    with pytest.raises(NativeError) as e:
        out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), 0, d_tt, B.stream)
    assert F.bfq_code(e.value) == -4                      # BFQ_E_STATE: not waited yet
    out.wait()
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    assert total > 0
    bad = [(d_offsets.data_ptr(), d_ranks.data_ptr(), -1, d_tt), (d_offsets.data_ptr(), None, total, d_tt),
           (None, d_ranks.data_ptr(), total, d_tt), (d_offsets.data_ptr(), d_ranks.data_ptr(), total, None),
           (d_offsets.data_ptr(), d_ranks.data_ptr(), total - 1, d_tt), (d_offsets.data_ptr(), d_ranks.data_ptr(), total + 1, d_tt)]
    for args in bad:
        with pytest.raises(NativeError) as e:
            out.delivery(*args, B.stream)
        assert F.bfq_code(e.value) == -1, args            # BFQ_E_INVALID
    with pytest.raises(NativeError) as e:
        out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), 2 ** 32, d_tt, B.stream)
    assert F.bfq_code(e.value) == -5                      # BFQ_E_RANGE
    B.torch.cuda.synchronize()
    nest_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs)   # the result is still usable
    out.release()
    idx.close()


@pytest.mark.gpu
def test_receiver_url_without_deliverer_key_fails_delivery(B):
    from bifromq_b200._native import NativeError
    kv = {}
    F.nroute(kv, "v", "a/+", 0, "ok", "d")
    kv[O.route_key("v", "a/b", b"0\x00no-deliverer-key")] = O.incarnation_bytes(1)
    idx = F.make_index(B, sorted(kv.items()))
    out = F.match_device(B, idx, ["v"], ["a/b"], np.zeros(1, np.int32))
    d_offsets, d_ranks, total = F.device_csr(B, out, 1)
    with pytest.raises(NativeError) as e:
        out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), B.stream)
    assert F.bfq_code(e.value) == -1
    out.release()
    idx.close()
