"""$oshare routes resolved on the device (bfq_delivery_device_ordered) against the restatement in test_host_oshare_cpu.

Every case runs bfq_delivery_device and bfq_delivery_device_ordered on one completed match and checks:
  * the packs whose publisher span is empty equal bfq_delivery_device's, pack for pack, once the $oshare pairs that get
    resolved are taken out of the ordered-share deliverer (member-less groups stay there);
  * the sub-packs (non-empty spans) are exactly the (topic position, $oshare rank, winner) groups of the rendezvous pick over
    the members of the result's own snapshot, each with its publishers in order, on the winner's deliverer;
  * within a package every topic position's whole pack comes first, then its sub-packs by (rank, member);
  * on the smaller cases, the whole nesting equals batch_delivery_ordered() exactly.
Member receiverUrls, deliverers and groups are decoded from the KV each test builds (oracle_lib), never through the library.
"""
import functools
import threading

import numpy as np
import pytest

import oracle_lib as O
import test_gpu_delivery as D
import test_gpu_fanout as F
import test_gpu_fanout_budget as FB
import rendezvous_hash as RH
import test_host_oshare_cpu as H

INT_MAX, INT_MIN = 2 ** 31 - 1, -2 ** 31
NO_MEMBER = 0xFFFFFFFF
FULL_RESTATEMENT_MAX_PAIRS = 200_000


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


# ------------------------------------------------------------------ routes and publishers
def route_of_fn(pairs):
    """rank -> ('N', d) | ('S', [d...]) | ('O', None) (member-less group) | ('R', [(url, d)...]) ($oshare with members)"""
    @functools.lru_cache(maxsize=None)
    def route_of(r):
        kind, d = F.decode(pairs, r)
        if kind == "O":
            members = O.route_group_members_in_wire_order(pairs[r][1])
            if members:
                return "R", [(u, O.deliverer_of_receiver_url(u)) for u in members]
        return kind, d
    return route_of


SPECIAL_HASHES = [0, -1, INT_MIN, INT_MAX]


def publishers(counts, seed):
    """pub_off / pub_hash for per-position publisher counts: the special hashes first, repeats, then random ones"""
    rng = np.random.default_rng(seed)
    pub_off = np.zeros(len(counts) + 1, np.int64)
    pub_off[1:] = np.cumsum(counts)
    hashes = []
    for c in counts:
        h = (SPECIAL_HASHES + [7, 7] + rng.integers(INT_MIN, INT_MAX, max(c, 1), dtype=np.int64, endpoint=True).tolist())[:c]
        hashes += h
    return pub_off, np.asarray(hashes, np.int32)


def utf8_id(k):
    return ("é你" * k)[:k] if k % 3 == 0 else "r" * k


def url_of(j, dkey):
    """member urls whose 4 + length walks through every residue mod 16 and several 16-byte blocks; every third id is
    multi-byte UTF-8"""
    return O.receiver_url(j % 3, "m%d_%s" % (j, utf8_id(j % 53)), dkey)


GROUP_SIZES = [1, 2, 31, 32, 33, 200, 1000]


def edge_case():
    """$oshare groups of 1 .. 1000 members whose members sit on deliverers shared with normal and $share routes of the same
    filter (so several $oshare routes pick members on one deliverer), a member-less $oshare group, and positions with 0, 1,
    5, 37 and 1000 publishers (one position repeated)"""
    kv = {}
    for i in range(4):
        F.nroute(kv, "o", "e/+", i % 3, "n%d" % i, "dA" if i % 2 else "dB")
    F.groute(kv, "o", "e/+", "sh", [O.receiver_url(0, "s0", "dA"), O.receiver_url(1, "s1", "dB")])
    for n in GROUP_SIZES:
        F.groute(kv, "o", "e/+", "g%d" % n, [url_of(j, ("dA", "dB", "dX%d" % (j % 5))[j % 3]) for j in range(n)], ordered=True)
    F.groute(kv, "o", "e/+", "nobody", [], ordered=True)
    topics = ["e/0", "e/1", "e/2", "e/3", "e/1", "e/4", "e/5"]
    counts = [1, 0, 1000, 5, 3, 37, 2]
    return sorted(kv.items()), ["o"], topics, np.zeros(len(topics), np.int32), counts


# ------------------------------------------------------------------ the check
def host_arrays(dl, B):
    a = dl.arrays(B.dev)
    po, ko = a["package_off"], a["pack_off"]
    pkg_d = np.repeat(np.arange(dl.n_deliverers), np.diff(po))
    pack_p = np.repeat(np.arange(dl.n_packages), np.diff(ko))
    a["pack_d"] = pkg_d[pack_p]
    a["pack_tenant"] = a["package_tenant"][pack_p]
    a["pack_p"] = pack_p
    return a


def pack_rows(a, k):
    m0, m1 = int(a["match_off"][k]), int(a["match_off"][k + 1])
    return tuple(sorted(zip(a["match_rank"][m0:m1].tolist(), a["match_member"][m0:m1].tolist())))


def rendezvous_winners(tt, n_tenants, csr_off, csr_ranks, route_of, pub_off, pub_hash):
    """{(position, $oshare rank, publisher): winning member} for every ($oshare pair, publisher) of the nested positions,
    scored in one numpy pass (rendezvous_hash.scores_np, checked against the plain restatement in test_host_oshare_cpu)"""
    items, hs, urls, first = [], [], [], []
    for t in range(len(csr_off) - 1):
        if not 0 <= int(tt[t]) < n_tenants:
            continue
        for r in csr_ranks[csr_off[t]:csr_off[t + 1]].tolist():
            kind, members = route_of(int(r))
            if kind != "R":
                continue
            for p in range(int(pub_off[t]), int(pub_off[t + 1])):
                items.append((t, int(r), p))
                first.append(len(hs))
                hs += [int(pub_hash[p])] * len(members)
                urls += [u for u, _ in members]
    scores = RH.scores_np(hs, urls) if hs else np.zeros(0, np.int64)
    bounds = first + [len(hs)]
    # np.argmax takes the first maximum: a later equal score never wins, as in RendezvousHash.get
    return {it: int(np.argmax(scores[bounds[q]:bounds[q + 1]])) for q, it in enumerate(items)}


def expected_subpacks(tt, winners, route_of, ids):
    """{(deliverer, tenant, position, rank, member): (publishers...)}: the publishers of a pair grouped by their winner"""
    out = {}
    for (t, r, p), w in winners.items():
        out.setdefault((ids[route_of(r)[1][w][1]], int(tt[t]), t, r, w), []).append(p)
    return {k: tuple(v) for k, v in out.items()}


def ordered_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, d_tt, pairs, pub_off, pub_hash, full=None):
    """bfq_delivery_device then bfq_delivery_device_ordered on one result; returns the ordered DeliveryResult and nesting"""
    torch = B.torch
    tt = np.asarray(tt)
    base = out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), B.stream)
    ba = host_arrays(base, B)
    d_pub_off = torch.from_numpy(np.asarray(pub_off, np.int64)).to(B.dev)
    d_pub_hash = torch.from_numpy(np.asarray(pub_hash, np.int32) if len(pub_hash) else np.zeros(1, np.int32)).to(B.dev)
    od = out.delivery_ordered(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), d_pub_off.data_ptr(),
                              d_pub_hash.data_ptr(), len(pub_hash), B.stream)
    oa = host_arrays(od, B)
    torch.cuda.synchronize()
    csr_off, csr_ranks = d_offsets.cpu().numpy(), d_ranks.cpu().numpy()[:total]
    route_of = route_of_fn(pairs)
    assert od.n_deliverers == base.n_deliverers and od.ordered_share_id == base.ordered_share_id
    assert od.generation == out.generation
    OS = od.ordered_share_id
    ids = {idx.deliverer(d): d for d in range(OS)}
    ids[D.ORDERED] = OS
    # structure: no empty package or pack, offsets consistent, spans inside the publisher list
    po, ko, mo, so = oa["package_off"], oa["pack_off"], oa["match_off"], oa["pack_pub_off"]
    assert po[-1] == od.n_packages and ko[-1] == od.n_packs and mo[-1] == od.n_pairs and so[-1] == od.ordered.n_pack_pubs
    assert (np.diff(ko) > 0).all() and (np.diff(mo) > 0).all() and (np.diff(so) >= 0).all()
    span = np.diff(so)
    sub = span > 0
    assert int(sub.sum()) == od.ordered.n_ordered_packs
    assert (np.diff(mo)[sub] == 1).all()                    # a sub-pack carries exactly one MatchInfo
    # order inside a package: position ascending; the whole pack first, then sub-packs by (rank, member)
    okey = [(int(oa["pack_p"][k]), int(oa["pack_topic"][k]), int(sub[k]), *(pack_rows(oa, k)[0] if sub[k] else (0, 0)))
            for k in range(od.n_packs)]
    assert okey == sorted(okey) and len(set(okey)) == len(okey)
    # whole packs == bfq_delivery_device's, pack for pack, less the resolved $oshare pairs
    resolved = lambda r: route_of(int(r))[0] == "R"
    base_packs = []
    for k in range(base.n_packs):
        rows = pack_rows(ba, k)
        if int(ba["pack_d"][k]) == OS:
            rows = tuple(x for x in rows if not resolved(x[0]))
        if rows:
            base_packs.append((int(ba["pack_d"][k]), int(ba["pack_tenant"][k]), int(ba["pack_topic"][k]), rows))
    whole = [(int(oa["pack_d"][k]), int(oa["pack_tenant"][k]), int(oa["pack_topic"][k]), pack_rows(oa, k))
             for k in range(od.n_packs) if not sub[k]]
    assert whole == base_packs
    # sub-packs == the rendezvous pick's groups
    got_subs = {}
    for k in np.flatnonzero(sub).tolist():
        (r, m), = pack_rows(oa, k)
        key = (int(oa["pack_d"][k]), int(oa["pack_tenant"][k]), int(oa["pack_topic"][k]), r, m)
        assert key not in got_subs
        got_subs[key] = tuple(oa["pack_pub"][so[k]:so[k + 1]].tolist())
    winners = rendezvous_winners(tt, len(tenants), csr_off, csr_ranks, route_of, pub_off, pub_hash)
    assert got_subs == expected_subpacks(tt, winners, route_of, ids)
    got = None
    if full if full is not None else total <= FULL_RESTATEMENT_MAX_PAIRS:
        got = od.nesting(B.dev)
        picks = {(int(ba["pack_topic"][k]), r): m for k in range(base.n_packs) for r, m in pack_rows(ba, k)}
        want = H.batch_delivery_ordered(tt, len(tenants), csr_off, csr_ranks, route_of, lambda t, r: picks[(t, r)], pub_off,
                                        pub_hash, lambda t, r, p: winners[(t, r, p)])
        assert got == {ids[d]: pkgs for d, pkgs in want.items()}
    return od, got


def run(B, case, caps=(INT_MAX, INT_MAX), idx=None, seed=1, full=None):
    pairs, tenants, topics, tt, counts = case
    own = idx is None
    if own:
        idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt, caps)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    pub_off, pub_hash = publishers(counts, seed)
    r = ordered_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs, pub_off, pub_hash, full)
    out.release()
    if own:
        idx.close()
    return r


# ------------------------------------------------------------------ GPU: shapes
@pytest.mark.gpu
def test_group_sizes_url_lengths_and_publisher_hashes(B):
    od, got = run(B, edge_case())
    # every group size resolved, two $oshare routes on one deliverer in separate packs, the member-less group still parked
    subs = [p for pkgs in got.values() for packs in pkgs.values() for p in packs if p[2]]
    assert len({next(iter(p[1]))[0] for p in subs}) == len(GROUP_SIZES)
    assert any(len({next(iter(p[1]))[0] for p in packs if p[2] and p[0] == 2}) > 1 for pkgs in got.values()
               for packs in pkgs.values())
    assert od.ordered_share_id in got and all(not p[2] for packs in got[od.ordered_share_id].values() for p in packs)
    assert all(p[0] != 1 or not p[2] for pkgs in got.values() for packs in pkgs.values() for p in packs)   # 0 publishers
    assert od.ordered.n_pack_pubs == len(GROUP_SIZES) * (1 + 1000 + 5 + 3 + 37 + 2)


@pytest.mark.gpu
@pytest.mark.parametrize("caps", [(INT_MAX, 3), (1, 5), (0, 0)])
def test_group_fanout_caps_drop_some_oshare_routes(B, caps):
    od, got = run(B, edge_case(), caps)
    if caps == (0, 0):
        assert od.ordered.n_ordered_packs == 0 and od.ordered.n_pack_pubs == 0   # every group route capped away
    else:
        assert 0 < len({next(iter(p[1]))[0] for pkgs in got.values() for packs in pkgs.values() for p in packs if p[2]}) < len(GROUP_SIZES)


@pytest.mark.gpu
def test_groups_case_and_no_publishers_anywhere(B):
    pairs, tenants, topics, tt = F.groups_case()
    run(B, (pairs, tenants, topics, tt, [3] * len(topics)))
    od, got = run(B, (pairs, tenants, topics, tt, [0] * len(topics)))
    assert od.ordered.n_ordered_packs == 0 and od.ordered.n_pack_pubs == 0


@pytest.mark.gpu
def test_interleaved_tenants_and_repeated_positions(B):
    pairs, tenants, topics, tt = D.interleaved_case()
    counts = np.random.default_rng(4).integers(0, 4, len(topics)).tolist()
    od, got = run(B, (pairs, tenants, topics, tt, counts))
    assert od.ordered.n_ordered_packs > 0


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C3", "C4"])
def test_workload_oshare_groups_in_locality_order(B, config):
    from bifromq_b200.workload import Workload
    w = Workload(config, scale=0.1)
    n, tenants = w.n_topics, w.tenants
    vb, kb = w.vals.tobytes(), w.keys.tobytes()
    pairs = [(kb[w.key_off[i]:w.key_off[i + 1]], vb[w.val_off[i]:w.val_off[i + 1]]) for i in range(w.n_routes)]
    idx = B.pkg.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    idx.commit()
    torch = B.torch
    keep = [torch.from_numpy(np.ascontiguousarray(x)).to(B.dev) for x in (w.topics, w.topic_off, w.topic_tenant[:n])]
    out = idx.match_device(tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), n, [INT_MAX] * len(tenants),
                           [100] * len(tenants), B.stream)
    assert n >= 32768                                       # the match ran in locality order
    d_offsets, d_ranks, total = F.device_csr(B, out, n)
    counts = np.random.default_rng(11).integers(1, 4, n).tolist()
    pub_off, pub_hash = publishers(counts, 12)
    od, got = ordered_check(B, idx, out, tenants, w.topic_tenant[:n], d_offsets, d_ranks, total, keep[2], pairs, pub_off,
                            pub_hash, full=False)
    assert od.ordered.n_ordered_packs > 100
    out.release()
    idx.close()


@pytest.mark.gpu
def test_budgeted_csr(B):
    case = FB.fan_case()
    idx = F.make_index(B, case.pairs)
    out = FB.match(B, idx, case)
    got = FB.budget(B, out, case)
    assert got["r"].n_dropped_bytes > 0
    pub_off, pub_hash = publishers([2] * len(case.topics), 5)
    od, _ = ordered_check(B, idx, out, case.tenants, case.tt, got["d_off"], got["d_ranks"], got["total"], out.keep[2], case.pairs,
                          pub_off, pub_hash)
    assert od.ordered.n_ordered_packs > 0
    out.release()
    idx.close()


# ------------------------------------------------------------------ GPU: snapshots
def snapshot_start():
    kv = {}
    for t in ("s1", "s2"):
        F.mixed_routes(kv, t, "x/#", 18, tag=t)
        F.groute(kv, t, "x/+", "og", [url_of(j, "dq%d" % j) for j in range(5)], ordered=True)
    for i in range(3000):   # a tenant the commits never touch: they stay delta commits
        F.nroute(kv, "tz", "big/%d/%d" % (i // 50, i % 50), 0, "z", "dz%d" % (i % 4))
    return kv


@pytest.mark.gpu
@pytest.mark.parametrize("change", ["add", "remove", "reorder"])
def test_old_result_resolves_against_its_own_snapshot(B, change):
    g = F.Gen(snapshot_start())
    old_pairs = g.pairs()
    idx = F.make_index(B, old_pairs)
    tenants, topics = ["s1", "s2"], ["x/1", "x/2", "x/1"]
    tt = np.array([0, 1, 1], np.int32)
    counts = [6, 4, 9]
    out_old = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out_old, len(topics))
    members = [url_of(j, "dq%d" % j) for j in range(5)]
    new = {"add": members + [url_of(9, "dq9"), url_of(10, "dA")], "remove": members[1:4], "reorder": members[::-1]}[change]
    key = O.route_key("s1", "$oshare/og/x/+")
    g.kv[key] = O.route_group({u: 1 for u in new})
    idx.apply(adds=[(key, g.kv[key])])
    st = idx.stats()
    errs = []

    def committer():
        try:
            idx.commit()
        except Exception as e:   # pragma: no cover
            errs.append(e)
    th = threading.Thread(target=committer)
    th.start()
    pub_off, pub_hash = publishers(counts, 3)
    od, _ = ordered_check(B, idx, out_old, tenants, tt, d_offsets, d_ranks, total, out_old.keep[2], old_pairs, pub_off, pub_hash)
    th.join()
    assert not errs, errs
    assert idx.stats()["delta_commits"] == st["delta_commits"] + 1 and od.generation == out_old.generation
    # once more after the commit: the old snapshot still answers with its own members
    ordered_check(B, idx, out_old, tenants, tt, d_offsets, d_ranks, total, out_old.keep[2], old_pairs, pub_off, pub_hash)
    out_old.release()
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    od, _ = ordered_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], g.pairs(), pub_off, pub_hash)
    assert od.generation > out_old.generation
    out.release()
    idx.close()


# ------------------------------------------------------------------ GPU: errors and release
@pytest.mark.gpu
def test_ordered_argument_and_state_errors(B):
    from bifromq_b200._native import NativeError
    pairs, tenants, topics, tt, counts = edge_case()
    idx = F.make_index(B, pairs)
    torch = B.torch
    out = F.match_device(B, idx, tenants, topics, tt, wait=False)
    d_tt = out.keep[2].data_ptr()
    pub_off, pub_hash = publishers(counts, 2)
    P = lambda a: torch.from_numpy(np.asarray(a)).to(B.dev)
    d_po, d_ph = P(pub_off), P(pub_hash)
    n_pubs = len(pub_hash)
    d_offsets = torch.zeros(len(topics) + 1, dtype=torch.int64, device=B.dev)
    d_ranks = torch.zeros(1, dtype=torch.int64, device=B.dev)
    call = lambda off, rk, n, t, po, ph, np_: out.delivery_ordered(off, rk, n, t, po, ph, np_, B.stream)
    with pytest.raises(NativeError) as e:
        call(d_offsets.data_ptr(), d_ranks.data_ptr(), 0, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs)
    assert F.bfq_code(e.value) == -4                      # BFQ_E_STATE: not waited yet
    out.wait()
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    o, r = d_offsets.data_ptr(), d_ranks.data_ptr()
    not_monotone = pub_off.copy()
    not_monotone[3] = not_monotone[2] - 1
    from_one = pub_off + 1
    short_end = pub_off.copy()
    short_end[-1] -= 1
    bad = [(o, r, -1, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs), (o, None, total, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs),
           (None, r, total, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs), (o, r, total, None, d_po.data_ptr(), d_ph.data_ptr(), n_pubs),
           (o, r, total, d_tt, None, d_ph.data_ptr(), n_pubs), (o, r, total, d_tt, d_po.data_ptr(), None, n_pubs),
           (o, r, total, d_tt, d_po.data_ptr(), d_ph.data_ptr(), -1),
           (o, r, total - 1, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs), (o, r, total + 1, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs),
           (o, r, total, d_tt, P(not_monotone).data_ptr(), d_ph.data_ptr(), n_pubs),
           (o, r, total, d_tt, P(from_one).data_ptr(), d_ph.data_ptr(), n_pubs),
           (o, r, total, d_tt, P(short_end).data_ptr(), d_ph.data_ptr(), n_pubs),
           (o, r, total, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs - 1)]
    for args in bad:
        with pytest.raises(NativeError) as e:
            call(*args)
        assert F.bfq_code(e.value) == -1, args[2:]        # BFQ_E_INVALID
    with pytest.raises(NativeError) as e:
        call(o, r, 2 ** 32, d_tt, d_po.data_ptr(), d_ph.data_ptr(), n_pubs)
    assert F.bfq_code(e.value) == -5                      # BFQ_E_RANGE
    torch.cuda.synchronize()
    ordered_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs, pub_off, pub_hash)   # still usable
    out.release()
    idx.close()


@pytest.mark.gpu
def test_release_waits_for_the_ordered_delivery(B):
    """bfq_delivery_device_ordered synchronises its stream itself: pinned here so that stays true"""
    import test_gpu_workspace_lease as WL
    pairs, tenants, topics, tt, counts = edge_case()
    idx = F.make_index(B, pairs)
    torch = B.torch
    S = torch.cuda.Stream(B.dev)
    out = WL.match_on(B, idx, tenants, topics, tt, S)
    d_offsets, d_ranks, total = WL.sized_csr(B, out, len(topics), S, fill=True)
    pub_off, pub_hash = publishers(counts, 2)
    with torch.cuda.stream(S):
        d_po = torch.from_numpy(pub_off).to(B.dev)
        d_ph = torch.from_numpy(pub_hash).to(B.dev)
        torch.cuda._sleep(WL.SLEEP_CYCLES)
    out.delivery_ordered(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), d_po.data_ptr(),
                         d_ph.data_ptr(), len(pub_hash), S.cuda_stream)
    out.release()
    assert S.query()
    idx.close()
