"""bfq_delivery_reply: every deliverer's DeliveryReply joined back to the pairs of the nesting its request was encoded from,
checked deliverer by deliverer against tests/delivery_reply.py's restatement of BatchDeliveryCall.execute: each pair's code,
each deliverer's status and the stale set. A deliverer a case makes FALLBACK only has to be FALLBACK, its pairs UNDECIDED.
The requests are the encoder's own bytes (tests/test_gpu_delivery_wire.py checks them against their restatement)."""
import zlib

import numpy as np
import pytest

import delivery_reply as R
import delivery_wire as W
import oracle_lib as O
import test_gpu_delivery as D
import test_gpu_delivery_wire as WT
import test_gpu_fanout as F

NO_MEMBER = 0xFFFFFFFF
B = D.B
STALE_DT = np.dtype([("deliverer", "<i4"), ("tenant", "<i4"), ("rank", "<u4"), ("member", "<u4"), ("reply_off", "<i8"),
                     ("reply_len", "<i4"), ("code", "<i4")])


def pair_table(B, dl, pairs):
    """per pair of the nesting: deliverer, tenant index, rank, member, and its canonical MatchInfo bytes"""
    a = dl.arrays(B.dev)
    po, ko, mo = a["package_off"], a["pack_off"], a["match_off"]
    pkg_d = np.repeat(np.arange(len(po) - 1), np.diff(po))
    pack_pkg = np.repeat(np.arange(len(ko) - 1), np.diff(ko))
    pair_pkg = pack_pkg[np.repeat(np.arange(len(mo) - 1), np.diff(mo))]
    infos = {}

    def mi(r, m):
        if r not in infos:
            infos[r] = W.route_match_infos(*pairs[r])
        i = 0 if m == NO_MEMBER else m
        return infos[r][i] if i < len(infos[r]) else b""   # a member-less group under ordered_share_id: never sent
    ranks, members = a["match_rank"], a["match_member"]
    return {"d": pkg_d[pair_pkg], "tenant": a["package_tenant"][pair_pkg], "rank": ranks, "member": members,
            "mi": [mi(int(r), int(m)) for r, m in zip(ranks, members)]}


def code_of(seed):
    def f(tenant, mi):
        h = zlib.crc32(tenant.encode() + mi) ^ seed
        return R.NO_SUB if h % 50 == 0 else R.NO_RECEIVER if h % 100 == 1 else R.NO_SUB if h % 7 == 3 else R.OK
    return f


def results_of(request, seed, drop=0, unknown=b"", pad=False, explicit=False, code_first=False):
    """[(tenant bytes, DeliveryResults bytes)] answering every distinct MatchInfo of the request with code_of(seed), `drop`
    of every 8 left out (NO_RESULT), optional unknown fields and per-record padding that shifts every record's offset"""
    cof = code_of(seed)
    out = []
    for tenant, infos in R.request_match_infos(request).items():
        body = b""
        for i, m in enumerate(infos):
            mb = m.SerializeToString()
            if (zlib.crc32(mb) + seed) % 8 < drop:
                continue
            if pad:
                body += W.field(15, b"\x0a" * (i % 41))
            body += R.record(mb, cof(tenant, mb), unknown=unknown if i % 3 == 0 else b"", code_first=code_first and i % 2 == 0,
                             explicit_code=explicit)
        out.append((tenant.encode(), body))
    return out


def resolved(variant, seed=1):
    """(request bytes) -> reply bytes of a deliverer the device must decide"""
    return {
        "local": lambda q: R.local_dist_reply(q, code_of(seed)),
        "pipeline": R.pipeline_no_receiver_reply,
        "dropped": lambda q: R.reply(results_of(q, seed, drop=3)),
        "odd": lambda q: R.reply(results_of(q, seed, unknown=b"".join(R.UNKNOWN), pad=True, explicit=True, code_first=True),
                                 unknown=b"".join(R.UNKNOWN), value_first=True, code_last=True, explicit_code=True),
        "bpr": lambda q: b"\x08\x01",
        "bpr_with_results": lambda q: R.reply(results_of(q, seed), code=1),
        "failed": lambda q: R.FAILED_CALL,
        "code7": lambda q: b"\x08\x07",
        "empty": lambda q: b"",
    }[variant]


def fallback(trigger, seed=1):
    """(request bytes) -> reply bytes the device must leave to the host"""
    def first(q):
        return results_of(q, seed)

    def with_first_result(q, f):
        ents = first(q)
        t, body = ents[0]
        return R.reply([(t, f(body))] + ents[1:])

    def first_mi(q):
        return next(iter(R.request_match_infos(q).values()))[0].SerializeToString()
    return {
        "repeated_code": lambda q: b"\x08\x00" + R.reply(first(q)) + b"\x08\x00",
        "repeated_tenant": lambda q: R.reply(first(q) + first(q)[:1]),
        "absent_tenant": lambda q: R.reply(first(q) + [(b"no-such-tenant", b"")]),
        "invalid_utf8_tenant": lambda q: R.reply(first(q) + [(b"\xc3\x28", b"")]),
        "duplicate_match_info": lambda q: with_first_result(q, lambda b: b + R.record(first_mi(q), 0)),
        "explicit_zero_incarnation": lambda q: R.reply([(next(iter(R.request_match_infos(q))).encode(),
                                                         R.record(first_mi(q) + b"\x18\x00", 1))]),
        "reordered_match_info": lambda q: R.reply([(next(iter(R.request_match_infos(q))).encode(),
                                                    R.record(reorder(first_mi(q)), 1))]),
        "long_length_varint": lambda q: R.reply([(next(iter(R.request_match_infos(q))).encode(),
                                                  R.record(long_matcher_length(first_mi(q)), 1))]),
        "foreign_match_info": lambda q: with_first_result(q, lambda b: b + R.record(W.match_info(W.field(2, b"zz"), b"1\0q\0d", 1), 0)),
        "truncated": lambda q: R.reply(first(q))[:-1] if R.reply(first(q)) else b"\x08",
        "code_as_bytes": lambda q: with_first_result(q, lambda b: W.field(1, W.field(1, first_mi(q)) + W.field(2, b"\x01"))),
        "repeated_match_info_field": lambda q: with_first_result(q, lambda b: W.field(1, W.field(1, first_mi(q)) * 2)),
        "repeated_result_code": lambda q: with_first_result(q, lambda b: W.field(1, W.field(1, first_mi(q)) + b"\x10\x01\x10\x01")),
        "repeated_entry_key": lambda q: W.field(2, W.field(1, first(q)[0][0]) * 2 + W.field(2, first(q)[0][1])),
        "results_as_varint": lambda q: W.field(2, W.field(1, first(q)[0][0]) + W.varint(2 << 3) + b"\x01"),
        "group_wire_type": lambda q: b"\x1b\x1c" + R.reply(first(q)),
    }[trigger]


def long_matcher_length(mi):
    """the MatchInfo with its matcher field's length written as a varint one byte longer than needed"""
    n, i = W.read_varint(mi, 1)
    v = W.varint(n)
    return b"\x0a" + v[:-1] + bytes([v[-1] | 0x80, 0]) + mi[i:]


def reorder(mi):
    f = W.fields(mi)
    return b"".join(W.varint(no << 3 | wt) + (W.varint(len(v)) + v if wt == 2 else W.varint(v)) for no, wt, v in reversed(f))


def check(B, out, dl, table, tenants, req_data, req_off, make, base=0, stream=None, buf=None):
    """replies from make(d, request) -> (bytes, expect_fallback) placed from byte `base` of a device buffer (slices of
    deliverers without a request hold junk the call must not read); bfq_delivery_reply against the restatement"""
    torch = B.torch
    nd = dl.n_deliverers
    osid = nd - 1
    sent = set(int(d) for d in np.unique(table["d"])) - {osid}
    blob, offs, fb = bytearray(), [base], {}
    for d in range(nd):
        if d in sent:
            rep, fb[d] = make(d, req_data[int(req_off[d]):int(req_off[d + 1])])
        else:
            rep = b"\x0a\xff\xff"   # junk: never read
        blob += rep
        offs.append(base + len(blob))
    if buf is None:
        buf = torch.zeros(base + len(blob) + 1, dtype=torch.uint8, device=B.dev)
    if blob:
        buf[base:base + len(blob)] = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(B.dev)
    d_off = WT.upload(B, offs, np.int64)
    st = B.stream if stream is None else stream
    res = out.delivery_reply(dl, tenants, buf.data_ptr(), d_off.data_ptr(), st)
    torch.cuda.synchronize()
    assert res.n_pairs == dl.n_pairs and res.n_deliverers == nd and res.ordered_share_id == osid
    assert res.generation == out.generation
    codes = B.dist.device_view(res.d_pair_code, max(dl.n_pairs, 1), "|u1", B.dev).cpu().numpy()[:dl.n_pairs]
    status = B.dist.device_view(res.d_status, nd, "|u1", B.dev).cpu().numpy()
    stale = np.frombuffer(B.dist.device_view(res.d_stale, max(res.n_stale, 1) * STALE_DT.itemsize, "|u1", B.dev).cpu().numpy()
                          .tobytes(), STALE_DT)[:res.n_stale]
    want_codes = np.full(dl.n_pairs, R.NOT_SENT, np.uint8)
    want_status = np.full(nd, R.NOT_SENT, np.uint8)
    want_stale = []
    cls = R.classes()
    n_fb = 0
    for d in sorted(sent):
        js = np.flatnonzero(table["d"] == d)
        rep = bytes(blob[offs[d] - base:offs[d + 1] - base])
        if fb[d]:
            want_status[d] = want_codes[js] = R.UNDECIDED
            n_fb += 1
            continue
        tasks = [(tenants[int(table["tenant"][j])], table["mi"][j]) for j in js]
        st_, cs, stale_set = R.execute(tasks, rep)
        want_status[d] = st_
        want_codes[js] = cs
        rows = set()
        for j, (t, m) in zip(js, tasks):
            if (t, R.mi_key(cls["MatchInfo"].FromString(m))) in stale_set:
                rows.add((d, int(table["tenant"][j]), int(table["rank"][j]), int(table["member"][j]), int(want_codes[j])))
        want_stale += sorted(rows)
    assert status.tolist() == want_status.tolist()
    assert res.n_fallback == n_fb
    bad = np.flatnonzero(codes != want_codes)
    assert bad.size == 0, "pair %d: got %d, want %d" % (bad[0], codes[bad[0]], want_codes[bad[0]])
    assert list(res.n_code) == np.bincount(want_codes, minlength=8).tolist()
    got_stale = [(int(s["deliverer"]), int(s["tenant"]), int(s["rank"]), int(s["member"]), int(s["code"])) for s in stale]
    assert got_stale == want_stale
    # each stale entry's bytes in d_reply are its MatchInfo
    mis = {(int(table["d"][j]), int(table["tenant"][j]), int(table["rank"][j]), int(table["member"][j])): table["mi"][j]
           for j in range(dl.n_pairs)}
    for s in stale[:2000]:
        o = int(s["reply_off"]) - base
        got = cls["MatchInfo"].FromString(bytes(blob[o:o + int(s["reply_len"])]))
        assert R.mi_key(got) == R.mi_key(cls["MatchInfo"].FromString(mis[tuple(int(s[f]) for f in ("deliverer", "tenant", "rank", "member"))]))
    return res, want_status


def encoded(B, case, ordered=False, counts=None, idx=None):
    pairs = case[0]
    counts = [1] * len(case[2]) if counts is None else counts
    idx, out, dl, (wr, data, req_off) = (WT.ordered if ordered else WT.plain)(B, case, counts, idx=idx)
    return idx, out, dl, pair_table(B, dl, pairs), data, req_off


VARIANTS = ["local", "pipeline", "dropped", "odd", "bpr", "bpr_with_results", "failed", "code7", "empty"]
TRIGGERS = ["repeated_code", "repeated_tenant", "absent_tenant", "invalid_utf8_tenant", "duplicate_match_info",
            "explicit_zero_incarnation", "reordered_match_info", "long_length_varint", "foreign_match_info", "truncated",
            "code_as_bytes", "repeated_match_info_field", "repeated_result_code", "repeated_entry_key", "results_as_varint",
            "group_wire_type"]


@pytest.mark.gpu
@pytest.mark.parametrize("ordered", [False, True])
def test_every_reply_shape_on_share_and_oshare_nestings(B, ordered):
    case = F.groups_case()
    idx, out, dl, table, data, req_off = encoded(B, case, ordered)
    seen = set()
    for rot in range(len(VARIANTS)):
        def make(d, q, rot=rot):
            v = VARIANTS[(d + rot) % len(VARIANTS)]
            return resolved(v, seed=rot + d)(q), False
        _, st = check(B, out, dl, table, case[1], data, req_off, make, base=rot * 13)
        seen |= set(st.tolist())
    assert {0, 3, 4, 6} <= seen
    WT.close(idx, out)


@pytest.mark.gpu
def test_each_fallback_trigger_beside_resolved_deliverers(B):
    case = F.groups_case()
    idx, out, dl, table, data, req_off = encoded(B, case)
    sent = sorted(set(int(d) for d in np.unique(table["d"])) - {dl.n_deliverers - 1})
    assert len(sent) >= 3
    for i, trig in enumerate(TRIGGERS):
        victim = sent[i % len(sent)]

        def make(d, q, trig=trig, victim=victim):
            if d == victim:
                return fallback(trig)(q), True
            return resolved("local", seed=d)(q), False
        res, _ = check(B, out, dl, table, case[1], data, req_off, make)
        assert res.n_fallback == 1, trig
    WT.close(idx, out)


@pytest.mark.gpu
def test_one_match_info_for_many_packs_and_equal_bytes_under_two_tenants_and_deliverers(B):
    kv = {}
    for tn in ("t1", "t2"):
        for dk in ("dA", "dB"):                       # same filter and receiverId on two deliverers: equal MatchInfo bytes
            F.nroute(kv, tn, "a/+", 0, "r", dk, inc=7)
        F.nroute(kv, tn, "a/#", 1, "s", "dA", inc=0)
    pairs = sorted(kv.items())
    tenants, topics = ["t1", "t2"], ["a/x", "a/y", "a/x", "a/x", "a/z", "a/x"]
    tt = np.asarray([0, 1, 0, 1, 0, 0], np.int32)
    idx, out, dl, table, data, req_off = encoded(B, (pairs, tenants, topics, tt))
    assert len(set(table["mi"])) < len(table["mi"])
    res, _ = check(B, out, dl, table, tenants, data, req_off, lambda d, q: (resolved("pipeline")(q), False))
    # every distinct (deliverer, tenant, MatchInfo) is stale once, however many packs and positions carry it
    assert res.n_stale == len({(int(d), int(t), int(r), int(m)) for d, t, r, m in
                               zip(table["d"], table["tenant"], table["rank"], table["member"]) if d != dl.n_deliverers - 1})
    assert res.n_stale < dl.n_pairs
    for seed in range(1, 4):
        check(B, out, dl, table, tenants, data, req_off, lambda d, q, seed=seed: (resolved("local", seed)(q), False))
    WT.close(idx, out)


def receiver_for(mi_len, tenant, tf, inc):
    """a receiverId whose MatchInfo is exactly mi_len bytes"""
    m = W.route_matcher(O.route_key(tenant, tf, O.receiver_url(0, "", "d0")))
    for n in range(mi_len, 0, -1):
        rid = ("\n\x05" * n)[:n]
        if len(W.match_info(m, b"0\0" + rid.encode() + b"\0d0", inc)) == mi_len:
            return rid
    raise ValueError(mi_len)


@pytest.mark.gpu
def test_adversarial_bytes_long_replies_and_chunk_straddles(B):
    """tenant ids, filter levels and receiverIds made of record-header bytes (0a, 12, 08), one deliverer with thousands of
    MatchInfos (a reply spanning many chunks) whose records are shifted by padding of every length, MatchInfos of 127, 128,
    16383 and 16384 bytes, and a reply slice placed past 2^32 bytes. A host model of the chunk guesses shows that wrong guesses
    occur (so the repair path runs) and where chunk boundaries cut records; the results must still equal the restatement"""
    kv = {}
    tenants = ["\n\x0c\n\n", "t\x12\x08"]
    for tn in tenants:
        for i in range(2500):
            # receiverIds holding a whole fake DeliveryResult (0a 04 0a 02 'x' 'y'): chunk guesses land inside MatchInfos
            rid = "\n\x04\n\x02xy%d" % i if i % 2 else "\n\x08\x12%d" % i
            F.nroute(kv, tn, "\n\x0a/+", 0, rid, "d0", inc=i)
        for L in (127, 128, 16383, 16384):
            F.nroute(kv, tn, "\n\x0a/+", 0, receiver_for(L, tn, "\n\x0a/+", 3), "d1", inc=3)
    pairs = sorted(kv.items())
    topics = ["\n\x0a/\n", "\n\x0a/\x0a\x0a"]
    tt = np.asarray([0, 1], np.int32)
    idx, out, dl, table, data, req_off = encoded(B, (pairs, tenants, topics, tt))
    assert {127, 128, 16383, 16384} <= {len(m) for m in table["mi"]}
    heavy = int(np.bincount(table["d"]).argmax())
    q = data[int(req_off[heavy]):int(req_off[heavy + 1])]
    crossed = set()
    for variant in ("odd", "dropped", "local"):
        # the device's guesses, modelled on the heaviest deliverer's reply: some are wrong (the repair path runs)
        guesses, crossings = R.chunk_guesses(resolved(variant, 5)(q))
        assert len(guesses) > 40 and sum(g != t for g, t in guesses) > 10, variant
        crossed |= set(crossings)
        check(B, out, dl, table, tenants, data, req_off, lambda d, q, v=variant: (resolved(v, 5)(q), False))
    # over the three replies, chunk boundaries fall at every offset from 1 to 24 bytes into a field
    assert set(range(1, 25)) <= crossed
    # a reply slice past 2^32 bytes, on a side stream
    torch = B.torch
    base = 2 ** 32 + 7
    big = torch.zeros(base + (4 << 20), dtype=torch.uint8, device=B.dev)
    side = torch.cuda.Stream(B.dev)
    check(B, out, dl, table, tenants, data, req_off, lambda d, q: (resolved("odd", 9)(q), False), base=base,
          stream=side.cuda_stream, buf=big)
    del big
    WT.close(idx, out)
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_old_result_after_a_delta_commit(B):
    pairs, tenants, topics, tt = F.groups_case()
    idx, out, dl, table, data, req_off = encoded(B, (pairs, tenants, topics, tt))
    kv = dict(pairs)
    F.nroute(kv, tenants[0], "x/+", 0, "late", "dLate", inc=9)
    idx.apply(adds=[(k, v) for k, v in sorted(kv.items()) if k not in dict(pairs)])
    idx.commit()
    assert idx.generation() != out.generation
    check(B, out, dl, table, tenants, data, req_off, lambda d, q: (resolved("local", 3)(q), False))
    WT.close(idx, out)


@pytest.mark.gpu
def test_argument_state_and_nesting_errors(B):
    torch = B.torch
    pairs, tenants, topics, tt = F.groups_case()
    idx, out, dl, table, data, req_off = encoded(B, (pairs, tenants, topics, tt))
    res, _ = check(B, out, dl, table, tenants, data, req_off, lambda d, q: (resolved("local", 1)(q), False))
    before = B.dist.device_view(res.d_pair_code, dl.n_pairs, "|u1", B.dev).cpu().numpy()
    buf = torch.zeros(64, dtype=torch.uint8, device=B.dev)
    off = WT.upload(B, [0] * (dl.n_deliverers + 1), np.int64)
    with pytest.raises(RuntimeError, match="NULL"):
        out.delivery_reply(dl, tenants, None, off.data_ptr(), B.stream)
    with pytest.raises(RuntimeError, match="NULL"):
        out.delivery_reply(dl, tenants, buf.data_ptr(), None, B.stream)
    with pytest.raises(RuntimeError, match="tenant list"):
        out.delivery_reply(dl, tenants + ["x"], buf.data_ptr(), off.data_ptr(), B.stream)
    dec = np.zeros(dl.n_deliverers + 1, np.int64)
    dec[1:] = 10
    dec[-1] = 5
    with pytest.raises(RuntimeError, match="never decrease"):
        out.delivery_reply(dl, tenants, buf.data_ptr(), WT.upload(B, dec, np.int64).data_ptr(), B.stream)
    after = B.dist.device_view(res.d_pair_code, dl.n_pairs, "|u1", B.dev).cpu().numpy()
    assert (before == after).all()                       # nothing written
    d_offsets, d_ranks, total = F.device_csr(B, out, len(topics))
    pub_off = WT.upload(B, np.arange(len(topics) + 1), np.int64)
    pub_hash = WT.upload(B, np.zeros(len(topics), np.int32), np.int32)
    od = out.delivery_ordered(d_offsets.data_ptr(), d_ranks.data_ptr(), total, out.keep[2].data_ptr(), pub_off.data_ptr(),
                              pub_hash.data_ptr(), len(topics), B.stream)
    with pytest.raises(RuntimeError, match="not the latest"):
        out.delivery_reply(dl, tenants, buf.data_ptr(), off.data_ptr(), B.stream)
    assert out.delivery_reply(od, tenants, buf.data_ptr(), off.data_ptr(), B.stream).n_pairs == od.n_pairs
    out2 = F.match_device(B, idx, tenants, topics, tt)
    with pytest.raises(RuntimeError, match="not the latest"):
        out2.delivery_reply(od, tenants, buf.data_ptr(), off.data_ptr(), B.stream)
    out2.release()
    out3 = F.match_device(B, idx, tenants, topics, tt, wait=False)
    with pytest.raises(RuntimeError, match="needs a completed match"):
        out3.delivery_reply(od, tenants, buf.data_ptr(), off.data_ptr(), B.stream)
    out3.wait()
    out3.release()
    WT.close(idx, out)


@pytest.mark.gpu
def test_repeated_positions_in_locality_order(B):
    pairs, tenants, topics, tt = D.interleaved_case(n=4000, seed=8)
    for ordered in (False, True):
        idx, out, dl, table, data, req_off = encoded(B, (pairs, tenants, topics, tt), ordered)
        check(B, out, dl, table, tenants, data, req_off,
              lambda d, q: (resolved(VARIANTS[d % 4], d)(q), False))
        WT.close(idx, out)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["C3", "C4"])
@pytest.mark.parametrize("rekey", [0, 10000, 100000])
def test_workload_shapes(B, config, rekey):
    """the deliverer shapes of tools/delivery_bench.py at scale 0.1, every deliverer answered with LocalDistService's reply
    written from the nesting by delivery_reply.nesting_replies (about 2 % NO_SUB, 1 % NO_RECEIVER). Every pair's code and every
    stale row against the codes the replies were written with, the totals, and the heaviest, the lightest and three random
    deliverers pair for pair against the restatement of execute"""
    import os
    import sys
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
        keys, src = [kb[w.key_off[i]:w.key_off[i + 1]] for i in range(w.n_routes)], list(range(w.n_routes))
        idx.load(w.keys, w.key_off, w.vals, w.val_off)
    else:
        rk = fanout_bench.rekey(w.keys, w.key_off, rekey)
        keys, src = [k for k, _ in rk], [i for _, i in rk]
        kk, ko = N.as_blob(keys)
        vv, vo = N.as_blob([vb[w.val_off[i]:w.val_off[i + 1]] for i in src])
        idx.load(kk, ko, vv, vo)
    idx.commit()
    keep = [torch.from_numpy(np.ascontiguousarray(x)).to(B.dev) for x in (w.topics, w.topic_off, w.topic_tenant[:n])]
    out = idx.match_device(tenants, keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), n, [2 ** 31 - 1] * len(tenants),
                           [100] * len(tenants), B.stream)
    d_offsets, d_ranks, total = F.device_csr(B, out, n)
    dl = out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, keep[2].data_ptr(), B.stream)
    a = dl.arrays(B.dev)
    infos = {}

    def mi_of(r, m):
        if r not in infos:
            infos[r] = W.route_match_infos(keys[r], vb[w.val_off[src[r]]:w.val_off[src[r] + 1]])
        return infos[r][0 if m == NO_MEMBER else m]
    rp = R.nesting_replies(a, dl.n_deliverers, tenants, mi_of, np.random.default_rng(rekey + len(config)), 0.02, 0.01)
    blob, off = rp["blob"], rp["off"]
    d_reply = torch.from_numpy(np.frombuffer(blob, np.uint8).copy()).to(B.dev)
    d_off = WT.upload(B, off, np.int64)
    res = out.delivery_reply(dl, tenants, d_reply.data_ptr(), d_off.data_ptr(), B.stream)
    torch.cuda.synchronize()
    nd, osid = dl.n_deliverers, dl.n_deliverers - 1
    codes = B.dist.device_view(res.d_pair_code, dl.n_pairs, "|u1", B.dev).cpu().numpy()
    status = B.dist.device_view(res.d_status, nd, "|u1", B.dev).cpu().numpy()
    stale = np.frombuffer(B.dist.device_view(res.d_stale, max(res.n_stale, 1) * STALE_DT.itemsize, "|u1", B.dev).cpu().numpy()
                          .tobytes(), STALE_DT)[:res.n_stale]
    # every pair and every deliverer against the codes the replies carry
    po, ko, mo = a["package_off"], a["pack_off"], a["match_off"]
    pkg_d = np.repeat(np.arange(nd), np.diff(po))
    pair_pkg = np.repeat(np.arange(dl.n_packages), np.diff(ko))[np.repeat(np.arange(dl.n_packs), np.diff(mo))]
    pair_d = pkg_d[pair_pkg]
    want = np.where(pair_d == osid, R.NOT_SENT, rp["code"][rp["key_of_pair"]]).astype(np.uint8)
    assert res.n_fallback == 0
    want_status = np.where(np.bincount(pair_d, minlength=nd) > 0, R.OK, R.NOT_SENT)
    want_status[osid] = R.NOT_SENT
    assert (status == want_status).all()
    bad = np.flatnonzero(codes != want)
    assert bad.size == 0, "pair %d: got %d, want %d" % (bad[0], codes[bad[0]], want[bad[0]])
    assert list(res.n_code) == np.bincount(want, minlength=8).tolist()
    sel = rp["sent"] & (rp["code"] > 0)
    kp = rp["pkg"][sel]
    want_rows = np.stack([pkg_d[kp], a["package_tenant"][kp], rp["rank"][sel], rp["member"][sel], rp["code"][sel]]).T
    got_rows = np.stack([stale["deliverer"], stale["tenant"], stale["rank"], stale["member"], stale["code"]]).T.astype(np.int64)
    assert res.n_stale == len(want_rows) > 0 and (got_rows == want_rows.astype(np.int64)).all()
    # sampled deliverers pair for pair against the restatement of execute
    sizes = np.bincount(pair_d[pair_d != osid], minlength=nd)
    nonempty = np.flatnonzero(sizes)
    rng = np.random.default_rng(rekey + 7)
    sample = {int(np.argmax(sizes)), int(nonempty[np.argmin(sizes[nonempty])])}
    sample |= set(rng.choice(nonempty, min(3, len(nonempty)), replace=False).tolist())
    cls = R.classes()
    for d in sorted(sample):
        js = np.flatnonzero(pair_d == d)
        tasks = [(tenants[int(a["package_tenant"][pair_pkg[j]])], mi_of(int(a["match_rank"][j]), int(a["match_member"][j])))
                 for j in js]
        st, cs, stale_set = R.execute(tasks, blob[off[d]:off[d + 1]])
        assert status[d] == st and codes[js].tolist() == cs, "deliverer %d" % d
        rows = stale[stale["deliverer"] == d]
        got = {(tenants[int(s["tenant"])], R.mi_key(cls["MatchInfo"].FromString(blob[int(s["reply_off"]):int(s["reply_off"]) + int(s["reply_len"])])))
               for s in rows}
        assert got == stale_set and len(rows) == len(stale_set), "deliverer %d" % d
    del d_reply
    out.release()
    idx.close()
    torch.cuda.empty_cache()
