"""bfq_delivery_encode[_ordered]: every deliverer's DeliveryRequest slice decoded and compared, pack for pack, with the
restatement of tests/delivery_wire.py built from the literal nesting (the nesting itself is checked against
BatchDeliveryCall's restatement by the helpers of test_gpu_delivery.py / test_gpu_delivery_oshare.py, reused here). MatchInfo
order inside a pack is compared as a multiset: the nesting leaves it unspecified."""
import os
import sys

import numpy as np
import pytest

import delivery_wire as W
import oracle_lib as O
import test_gpu_delivery as D
import test_gpu_delivery_oshare as S
import test_gpu_fanout as F

INT_MAX = 2 ** 31 - 1
NO_MEMBER = 0xFFFFFFFF
B = D.B


def exact_pack(length, q):
    """a serialized PublisherPack {publisher = 1: a client id, message = 2: payload} of exactly `length` bytes (>= 4)"""
    for client in range(0, 12):
        body = W.field(1, (b"c%d-" % q + b"x" * client)[:client])
        rest = length - len(body)
        for pad in range(max(rest - 4, 0), max(rest, 0) + 1):
            if 1 + len(W.varint(pad)) + pad == rest:
                return body + W.field(2, bytes((q + i) % 251 for i in range(min(pad, 64))) + b"p" * max(pad - 64, 0))
    raise ValueError(length)


def publisher_packs(n_pubs, seed, sizes=None):
    """n serialized PublisherPacks whose lengths cycle through `sizes`: by default both sides of the 1- / 2- and 2- / 3-byte
    varint boundaries (127, 128, 16383, 16384) and a few others"""
    sizes = sizes or [4, 13, 100, 127, 128, 1000, 16383, 16384]
    return [exact_pack(sizes[(q + seed) % len(sizes)], q) for q in range(n_pubs)]


def upload(B, arr, dtype):
    a = np.asarray(arr, dtype)
    return B.torch.from_numpy(a if a.size else np.zeros(1, dtype)).to(B.dev)


def expected_requests(got, pairs, tenants, topics, packs, pub_off):
    """{deliverer: [(tenant, [(topic, [publisher packs], sorted MatchInfos)])]} from a nesting() dict"""
    infos = {}

    def mi(r, m):
        if r not in infos:
            infos[r] = W.route_match_infos(*pairs[r])
        return infos[r][0 if m == NO_MEMBER else m]
    out = {}
    for d, pkgs in got.items():
        req = []
        for tn, plist in pkgs.items():
            wp = []
            for p in plist:
                t, ms = p[0], p[1]
                pubs = p[2] if len(p) > 2 and p[2] else range(int(pub_off[t]), int(pub_off[t + 1]))
                wp.append((topics[t].encode(), [packs[q] for q in pubs], sorted(mi(r, m) for r, m in ms)))
            req.append((tenants[tn].encode(), wp))
        out[d] = req
    return out


def encode_check(B, out, dl, got, pairs, tenants, topics, pub_off, seed=5, packs=None):
    """size, a write one byte short (nothing written), the write; every slice decoded against expected_requests"""
    torch = B.torch
    packs = publisher_packs(int(pub_off[-1]), seed) if packs is None else packs
    blob, off = O.blob(packs)
    d_pub_off, d_pp, d_pp_off = upload(B, pub_off, np.int64), upload(B, blob, np.uint8), upload(B, off, np.int64)
    topics_d, toff_d = out.keep[0], out.keep[1]
    args = (tenants, topics_d.data_ptr(), toff_d.data_ptr(), d_pub_off.data_ptr(), d_pp.data_ptr(), d_pp_off.data_ptr())
    sized = out.delivery_wire(dl, *args, None, 0, B.stream)
    n = sized.n_bytes
    buf = torch.full((n + 16,), 0xAB, dtype=torch.uint8, device=B.dev)
    short = out.delivery_wire(dl, *args, buf.data_ptr(), n - 1, B.stream)
    assert short.n_bytes == n
    torch.cuda.synchronize()
    assert n == 0 or (buf.cpu().numpy() == 0xAB).all()     # one byte short: nothing written
    wr = out.delivery_wire(dl, *args, buf.data_ptr(), n, B.stream)
    torch.cuda.synchronize()
    assert wr.n_bytes == n and wr.generation == out.generation and wr.ordered_share_id == dl.ordered_share_id
    req_off = B.dist.device_view(wr.d_req_off, wr.n_deliverers + 1, "<i8", B.dev).cpu().numpy()
    data = buf.cpu().numpy().tobytes()
    assert req_off[0] == 0 and req_off[-1] == n and (np.diff(req_off) >= 0).all() and data[n:] == b"\xab" * 16
    osid = dl.ordered_share_id
    skipped = sum(len(p[1]) for plist in got.get(osid, {}).values() for p in plist)
    assert wr.n_skipped == skipped and wr.n_match_infos == dl.n_pairs - skipped
    assert req_off[osid] == req_off[osid + 1]
    want = expected_requests({d: v for d, v in got.items() if d != osid}, pairs, tenants, topics, packs, pub_off)
    for d in range(wr.n_deliverers):
        dec = W.decode_request(data[req_off[d]:req_off[d + 1]])
        dec = [(t, [(tp, pubs, sorted(ms)) for tp, pubs, ms in plist]) for t, plist in dec]
        assert dec == want.get(d, []), "deliverer %d" % d
    return wr, data, req_off


def plain(B, case, counts, idx=None):
    pairs, tenants, topics, tt = case
    own = idx is None
    if own:
        idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    dl, _, got = D.nest_check(B, idx, out, tenants, np.asarray(tt, np.int32), d_offsets, d_ranks, total, out.keep[2], pairs)
    pub_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    r = encode_check(B, out, dl, got, pairs, tenants, topics, pub_off)
    return idx, out, dl, r


def ordered(B, case, counts, idx=None):
    pairs, tenants, topics, tt = case
    own = idx is None
    if own:
        idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    pub_off, pub_hash = S.publishers(counts, 1)
    od, got = S.ordered_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs, pub_off, pub_hash)
    if got is None:   # too many pairs for ordered_check's full restatement: the nesting it checked against the plain one
        got = od.nesting(B.dev)
    r = encode_check(B, out, od, got, pairs, tenants, topics, pub_off)
    return idx, out, od, r


def close(idx, out):
    out.release()
    idx.close()


@pytest.mark.gpu
def test_normal_share_oshare_and_memberless_groups(B):
    case = F.groups_case()
    counts = [i % 4 for i in range(len(case[2]))]
    idx, out, dl, (wr, _, _) = plain(B, case, counts)
    assert wr.n_skipped > 0 and wr.n_match_infos > 0       # $oshare and the empty group parked, the rest encoded
    close(idx, out)
    idx, out, od, (wr, _, _) = ordered(B, case, counts)
    assert od.ordered.n_ordered_packs > 0 and wr.n_skipped > 0   # the member-less group stays parked
    stats = idx.stats()
    assert stats["wire_table_bytes"] > 0
    close(idx, out)


@pytest.mark.gpu
def test_oshare_sub_packs_of_every_group_size_and_publisher_count(B):
    pairs, tenants, topics, tt, counts = S.edge_case()
    idx, out, od, _ = ordered(B, (pairs, tenants, topics, tt), counts)
    close(idx, out)


@pytest.mark.gpu
def test_interleaved_tenants_and_repeated_positions(B):
    case = D.interleaved_case()
    counts = np.random.default_rng(4).integers(0, 4, len(case[2])).tolist()
    close(*plain(B, case, counts)[:2])
    close(*ordered(B, case, counts)[:2])


@pytest.mark.gpu
def test_multibyte_tenants_and_topics_and_no_publishers(B):
    kv = {}
    tenants = ["ténant✓", "t你"]
    for tn in tenants:
        F.nroute(kv, tn, "é/+", 0, "r你", "d0", inc=2 ** 64 - 1)
        F.nroute(kv, tn, "é//+", 1, "", "d1", inc=0)
        # members with incarnation 0 (field omitted in the RouteGroup and in the MatchInfo), 1 and 2^64 - 1
        kv[O.route_key(tn, "$share/g✓/é/#")] = group_value([(O.receiver_url(0, "m✓", "d0"), 0), (O.receiver_url(2, "n", "d2"), 1),
                                                            (O.receiver_url(1, "", "d1"), 2 ** 64 - 1)])
    topics = ["é/ü", "é//x", "é/ü", "é/✓"]
    tt = np.asarray([0, 1, 1, 0], np.int32)
    close(*plain(B, (sorted(kv.items()), tenants, topics, tt), [0, 0, 0, 0])[:2])
    close(*plain(B, (sorted(kv.items()), tenants, topics, tt), [2, 0, 1, 3])[:2])


@pytest.mark.gpu
def test_old_result_encodes_against_its_own_snapshot_after_a_delta_commit(B):
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    counts = [1] * len(topics)
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    dl, _, got = D.nest_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs)
    # a delta commit changes the members of the 7-member $share group
    k7 = next(k for k, v in pairs if b"s7" in k and W.route_detail(k)[1] == W.FLAG_UNORDERED)
    idx.apply(adds=[(k7, D_group([O.receiver_url(0, "new%d" % j, "dNew") for j in range(3)]))])
    idx.commit()
    assert idx.generation() != out.generation
    encode_check(B, out, dl, got, pairs, tenants, topics, np.arange(len(topics) + 1, dtype=np.int64))
    out.release()
    # a new match sees the new members
    new_pairs = dict(pairs)
    new_pairs[k7] = D_group([O.receiver_url(0, "new%d" % j, "dNew") for j in range(3)])
    new_pairs = sorted(new_pairs.items())
    close(*plain(B, (new_pairs, tenants, topics, tt), counts, idx=idx)[:2])


def D_group(urls):
    return group_value([(u, 1) for u in urls])


def group_value(members):
    """RouteGroup {map<string, uint64> members = 1} with the given (receiverUrl, incarnation) entries in wire order"""
    return b"".join(W.field(1, W.field(1, u) + (W.varint(2 << 3) + W.varint(inc) if inc else b"")) for u, inc in members)


@pytest.mark.gpu
def test_argument_state_and_nesting_errors(B):
    pairs, tenants, topics, tt = F.groups_case()
    idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    dl = out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), B.stream)
    pub_off = np.arange(len(topics) + 1, dtype=np.int64)
    packs = publisher_packs(len(topics), 1)
    blob, off = O.blob(packs)
    d_pub_off, d_pp, d_pp_off = upload(B, pub_off, np.int64), upload(B, blob, np.uint8), upload(B, off, np.int64)
    t0, t1 = out.keep[0].data_ptr(), out.keep[1].data_ptr()

    def enc(nest, tn=tenants, po=d_pub_off, ppo=d_pp_off, pp=d_pp, res=out):
        return res.delivery_wire(nest, tn, t0, t1, po.data_ptr() if po is not None else None, pp.data_ptr(),
                                 ppo.data_ptr(), None, 0, B.stream)
    assert enc(dl).n_bytes > 0
    with pytest.raises(RuntimeError, match=r"\(-1\)|NULL"):
        enc(dl, po=None)
    with pytest.raises(RuntimeError, match="tenant list"):
        enc(dl, tn=tenants + ["x"])
    bad = pub_off.copy()
    bad[3], bad[4] = bad[4], bad[3]
    with pytest.raises(RuntimeError, match="never decrease"):
        enc(dl, po=upload(B, bad, np.int64))
    bad_pp = off.copy()
    bad_pp[2] = bad_pp[3] + 1
    with pytest.raises(RuntimeError, match="never decrease"):
        enc(dl, ppo=upload(B, bad_pp, np.int64))
    # an ordered call replaces the nesting: the plain one is stale now
    pub_hash = upload(B, np.zeros(len(topics), np.int32), np.int32)
    od = out.delivery_ordered(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), d_pub_off.data_ptr(),
                              pub_hash.data_ptr(), len(topics), B.stream)
    with pytest.raises(RuntimeError, match="not the latest"):
        enc(dl)
    assert enc(od).n_bytes > 0
    # a nesting of another result
    out2 = F.match_device(B, idx, tenants, topics, tt)
    with pytest.raises(RuntimeError, match="not the latest|needs a completed"):
        enc(od, res=out2)
    out2.release()
    # a match that has not completed
    out3 = F.match_device(B, idx, tenants, topics, tt, wait=False)
    with pytest.raises(RuntimeError, match="needs a completed match"):
        enc(od, res=out3)
    out3.wait()
    out3.release()
    close(idx, out)


@pytest.mark.gpu
def test_release_waits_for_a_long_write_pass(B):
    """one route, one position and one 256 MB publisher pack: the write pass is one warp copying 256 MB, which takes far
    longer than the calls that follow it. release() returns only after it, so the bytes compared right after it, on a stream
    that does not wait for the encode's, equal an encode that was waited for. (Without the wait in release this compare
    sees a partly written buffer.)"""
    torch = B.torch
    kv = {}
    F.nroute(kv, "t", "x", 0, "r", "d0")
    pairs, tenants, topics, tt = sorted(kv.items()), ["t"], ["x"], np.zeros(1, np.int32)
    idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    dl = out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), B.stream)
    big = 256 << 20
    d_pp = torch.arange(big, dtype=torch.int32, device=B.dev).remainder_(251).to(torch.uint8)
    header = b"\x12" + W.varint(big - 5)                    # message = 2 of big - 5 bytes: a valid pack
    d_pp[:5] = torch.frombuffer(bytearray(header), dtype=torch.uint8).to(B.dev)
    d_pp_off, d_pub_off = upload(B, [0, big], np.int64), upload(B, [0, 1], np.int64)
    side = torch.cuda.Stream(B.dev)
    args = (tenants, out.keep[0].data_ptr(), out.keep[1].data_ptr(), d_pub_off.data_ptr(), d_pp.data_ptr(), d_pp_off.data_ptr())
    n = out.delivery_wire(dl, *args, None, 0, side.cuda_stream).n_bytes
    assert n > big
    ref = torch.zeros(n, dtype=torch.uint8, device=B.dev)
    out.delivery_wire(dl, *args, ref.data_ptr(), n, side.cuda_stream)
    side.synchronize()
    info = W.field(3, W.route_match_infos(*pairs[0])[0])      # the request ends with the pack, then its MatchInfo
    assert bytes(ref[-len(info):].cpu().numpy()) == info
    assert bytes(ref[-len(info) - 1000:-len(info)].cpu().numpy()) == bytes(d_pp[-1000:].cpu().numpy())
    buf = torch.zeros(n, dtype=torch.uint8, device=B.dev)
    torch.cuda.synchronize()
    out.delivery_wire(dl, *args, buf.data_ptr(), n, side.cuda_stream)   # returns with the write pass queued on `side`
    out.release()
    done = side.query()                                     # the write pass has finished by the time release() returns
    # on the current stream, which does not wait for `side`: only release() ordered the write pass before this compare
    same = bool(torch.equal(buf, ref))
    side.synchronize()
    assert done and same
    idx.close()


@pytest.mark.gpu
def test_pack_package_and_entry_lengths_on_every_varint_boundary(B):
    """one tenant per publisher-pack length, each with one route and one position: its map entry holds one package with one
    pack, so the message pack, pack, package and entry lengths follow the publisher pack's and, over the sweep, land on
    127, 128, 16383 and 16384 each (pinned below on the restatement)"""
    lengths = [L for b in (128, 16384) for L in range(max(b - 220, 4), b + 4)]
    kv, tenants = {}, ["t%03d" % i for i in range(len(lengths))]
    for tn in tenants:
        F.nroute(kv, tn, "x", 0, "r", "d0", inc=5)
    pairs = sorted(kv.items())
    mi = W.route_match_infos(*pairs[0])[0]
    levels = {"message pack": set(), "pack": set(), "package": set(), "entry": set()}
    for i, L in enumerate(lengths):
        mp = W.topic_message_pack(b"x", [exact_pack(L, i)])
        pack = W.field(2, mp) + W.field(3, mi)
        package = W.field(1, pack)
        entry = W.field(1, tenants[i].encode()) + W.field(2, package)
        for k, v in (("message pack", mp), ("pack", pack), ("package", package), ("entry", entry)):
            levels[k].add(len(v))
    for k, got in levels.items():
        assert {127, 128, 16383, 16384} <= got, k
    topics = ["x"] * len(tenants)
    tt = np.arange(len(tenants), dtype=np.int32)
    idx = F.make_index(B, pairs)
    out = F.match_device(B, idx, tenants, topics, tt)
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    dl, _, got = D.nest_check(B, idx, out, tenants, tt, d_offsets, d_ranks, total, out.keep[2], pairs)
    encode_check(B, out, dl, got, pairs, tenants, topics, np.arange(len(topics) + 1, dtype=np.int64),
                 packs=[exact_pack(L, i) for i, L in enumerate(lengths)])
    close(idx, out)


@pytest.mark.gpu
def test_repeated_positions_in_locality_order(B):
    pairs, tenants, topics, tt = D.interleaved_case(n=40000, seed=8)
    counts = np.random.default_rng(9).integers(0, 3, len(topics)).tolist()
    idx = F.make_index(B, pairs)
    before = idx.stats()["duplicate_topics"]
    _, out, dl, _ = plain(B, (pairs, tenants, topics, tt), counts, idx=idx)
    assert idx.stats()["duplicate_topics"] - before > 30000   # the match ran in locality order and de-duplicated
    out.release()
    _, out, od, _ = ordered(B, (pairs, tenants, topics, tt), counts, idx=idx)
    assert od.ordered.n_ordered_packs > 0
    close(idx, out)


@pytest.mark.gpu
def test_budgeted_csr(B):
    import test_gpu_fanout_budget as FB
    case = FB.batch_case()
    idx = F.make_index(B, case.pairs)
    out = FB.match(B, idx, case)
    bud = FB.budget(B, out, case)
    assert bud["r"].n_dropped_bytes > 0
    dl, _, got = D.nest_check(B, idx, out, case.tenants, case.tt, bud["d_off"], bud["d_ranks"], bud["total"], out.keep[2],
                              case.pairs)
    topics = [t if isinstance(t, str) else t.decode() for t in case.topics]
    encode_check(B, out, dl, got, case.pairs, case.tenants, topics, np.arange(len(topics) + 1, dtype=np.int64))
    close(idx, out)


@pytest.mark.gpu
def test_delta_commit_reuses_untouched_tenants_tables(B):
    """the MatchInfo table is built on one snapshot; a delta commit grows the FIRST tenant, so every other tenant's cached
    entries move to new ranks on the next snapshot"""
    pairs, tenants, topics, tt = D.interleaved_case()
    counts = [1] * len(topics)
    idx = F.make_index(B, pairs)
    close_out = plain(B, (pairs, tenants, topics, tt), counts, idx=idx)[1]
    close_out.release()
    built = idx.stats()["wire_table_bytes"]
    assert built > 0
    kv = dict(pairs)
    for j in range(5):
        F.nroute(kv, tenants[0], "x/+", 0, "added%d" % j, "dAdded", inc=1000 + j)
    new_pairs = sorted(kv.items())
    idx.apply(adds=[(k, v) for k, v in new_pairs if k not in dict(pairs)])
    delta_before = idx.stats()["delta_commits"]
    idx.commit()
    st = idx.stats()
    assert st["delta_commits"] == delta_before + 1 and st["rebuilt_tenants"] == 1 and st["wire_table_bytes"] == 0
    _, out, dl, _ = plain(B, (new_pairs, tenants, topics, tt), counts, idx=idx)
    assert idx.stats()["wire_table_bytes"] > built
    close(idx, out)


def iter_fields(mv, i, end):
    """(field number, payload start, payload end) of the length-delimited fields in mv[i:end], without copying"""
    while i < end:
        tag, i = W.read_varint(mv, i)
        assert tag & 7 == 2
        n, i = W.read_varint(mv, i)
        yield tag >> 3, i, i + n
        i += n
    assert i == end


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C3", "C4"])
@pytest.mark.parametrize("rekey", [0, 10000, 100000])
def test_workload_shapes_sampled(B, config, rekey):
    """the deliverer shapes of tools/delivery_bench.py at scale 0.1 with a 1 000-byte publisher pack per position (tens of GB
    written, offsets past 2^32 where the shape has many packs). Every sampled deliverer's request is walked entry by entry and
    pack by pack against the nesting, and a sample of its packs is decoded in full against the restatement: the heaviest
    deliverer, the lightest non-empty one and three at random."""
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import fanout_bench
    from bifromq_b200 import _native as N
    from bifromq_b200.workload import Workload
    torch = B.torch
    w = Workload(config, scale=0.1)
    n, tenants = w.n_topics, w.tenants
    kb, vb = w.keys.tobytes(), w.vals.tobytes()
    idx = B.pkg.GpuRouteIndex(0)
    if rekey == 0:
        keys = [kb[w.key_off[i]:w.key_off[i + 1]] for i in range(w.n_routes)]
        src = list(range(w.n_routes))
        idx.load(w.keys, w.key_off, w.vals, w.val_off)
    else:
        rk = fanout_bench.rekey(w.keys, w.key_off, rekey)
        keys, src = [k for k, _ in rk], [i for _, i in rk]
        kk, ko = N.as_blob(keys)
        vv, vo = N.as_blob([vb[w.val_off[i]:w.val_off[i + 1]] for i in src])
        idx.load(kk, ko, vv, vo)
    idx.commit()
    keep = [torch.from_numpy(np.ascontiguousarray(x)).to(B.dev) for x in (w.topics, w.topic_off, w.topic_tenant[:n])]
    out = idx.match_device(tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), n, [INT_MAX] * len(tenants),
                           [100] * len(tenants), B.stream)
    d_offsets, d_ranks, total = F.device_csr(B, out, n)
    dl = out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, keep[2].data_ptr(), B.stream)
    payload = bytes(range(256)) * 4
    packs = [W.field(1, b"client-%07d" % t) + W.field(2, payload[:1000]) for t in range(n)]
    blob, off = O.blob(packs)
    d_pub_off, d_pp, d_pp_off = upload(B, np.arange(n + 1), np.int64), upload(B, blob, np.uint8), upload(B, off, np.int64)
    args = (tenants, keep[0].data_ptr(), keep[1].data_ptr(), d_pub_off.data_ptr(), d_pp.data_ptr(), d_pp_off.data_ptr())
    nb = out.delivery_wire(dl, *args, None, 0, B.stream).n_bytes
    buf = torch.empty(nb, dtype=torch.uint8, device=B.dev)
    wr = out.delivery_wire(dl, *args, buf.data_ptr(), nb, B.stream)
    torch.cuda.synchronize()
    if dl.n_packs > 10_000_000:
        assert nb > 2 ** 32
    a = dl.arrays(B.dev)
    req_off = B.dist.device_view(wr.d_req_off, wr.n_deliverers + 1, "<i8", B.dev).cpu().numpy()
    assert req_off[-1] == nb and wr.n_match_infos + wr.n_skipped == dl.n_pairs
    po, ko, mo = a["package_off"], a["pack_off"], a["match_off"]
    sizes = np.diff(req_off)
    nonempty = np.flatnonzero(sizes)
    rng = np.random.default_rng(rekey + len(config))
    sample = {int(np.argmax(sizes)), int(nonempty[np.argmin(sizes[nonempty])])}
    sample |= set(rng.choice(nonempty, min(3, len(nonempty)), replace=False).tolist())
    infos = {}

    def mi(r, m):
        if r not in infos:
            infos[r] = W.route_match_infos(keys[r], vb[w.val_off[src[r]]:w.val_off[src[r] + 1]])
        return infos[r][0 if m == NO_MEMBER else m]
    checked = 0
    for d in sorted(sample):
        assert d != wr.ordered_share_id
        data = buf[int(req_off[d]):int(req_off[d + 1])].cpu().numpy().tobytes()
        mv = memoryview(data)
        entries = list(iter_fields(mv, 0, len(data)))
        assert len(entries) == po[d + 1] - po[d]
        for g, (no, e0, e1) in zip(range(int(po[d]), int(po[d + 1])), entries):
            (k1, t0, t1), (k2, p0, p1) = iter_fields(mv, e0, e1)
            assert (no, k1, k2) == (3, 1, 2) and bytes(mv[t0:t1]) == tenants[int(a["package_tenant"][g])].encode()
            plist = list(iter_fields(mv, p0, p1))
            assert len(plist) == ko[g + 1] - ko[g]
            pick = {0, len(plist) - 1} | set(rng.integers(0, len(plist), 2).tolist())
            for j in pick:
                k = int(ko[g]) + j
                t = int(a["pack_topic"][k])
                _, q0, q1 = plist[j]
                dec = W.decode_request(W.field(3, W.field(1, b"") + W.field(2, W.field(1, bytes(mv[q0:q1])))))[0][1][0]
                want = sorted(mi(int(r), int(m)) for r, m in zip(a["match_rank"][mo[k]:mo[k + 1]], a["match_member"][mo[k]:mo[k + 1]]))
                assert (dec[0], dec[1], sorted(dec[2])) == (bytes(w.topics[w.topic_off[t]:w.topic_off[t + 1]]), [packs[t]], want)
                checked += 1
    assert checked >= 10
    del buf
    out.release()
    idx.close()
    torch.cuda.empty_cache()
