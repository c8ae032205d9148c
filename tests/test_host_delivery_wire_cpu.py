"""The DeliveryRequest restatement (tests/delivery_wire.py) pinned on hand-built routes, its decoder, and both checked against
protobuf messages built from descriptors restated in that module (skipped where google.protobuf is not importable)."""
import struct

import pytest

import delivery_wire as W
import oracle_lib as O

PB = W.protobuf_classes()


def normal(tenant, tf, rid, inc, broker=0, dkey="d0"):
    url = O.receiver_url(broker, rid, dkey)
    return O.route_key(tenant, tf, url), struct.pack(">Q", inc)


def group_value(members):
    """RouteGroup {map<string, uint64> members = 1}: entries in the given order"""
    return b"".join(W.field(1, W.field(1, url) + (W.varint(2 << 3) + W.varint(inc) if inc else b"")) for url, inc in members)


def group(tenant, tf, members):
    return O.route_key(tenant, tf), group_value(members)


def test_route_matchers_of_normal_share_and_oshare_routes_pinned():
    k, _ = normal("t", "a//b", "r", 1)
    # Normal: no type, three levels (the middle one empty), the filter as written
    assert W.route_matcher(k) == b"\x12\x01a\x12\x00\x12\x01b\x22\x04a//b"
    k, _ = group("t", "$share/g/a/+", [])
    assert W.route_matcher(k) == b"\x08\x01\x12\x01a\x12\x01+\x1a\x01g\x22\x0c$share/g/a/+"
    k, _ = group("t", "$oshare/g/#", [])
    assert W.route_matcher(k) == b"\x08\x02\x12\x01#\x1a\x01g\x22\x0b$oshare/g/#"
    # a filter of one empty level: one empty filterLevel, no mqttTopicFilter (proto3 drops the empty string)
    k, _ = normal("t", "", "r", 1)
    assert W.route_matcher(k) == b"\x12\x00"


def test_match_info_incarnations_and_receiver_ids():
    k, v = normal("t", "x", "rid", 0)
    m = W.route_matcher(k)
    assert W.route_match_infos(k, v) == [W.field(1, m) + b"\x12\x03rid"]                   # incarnation 0 omitted
    k, v = normal("t", "x", "rid", 1)
    assert W.route_match_infos(k, v) == [W.field(1, m) + b"\x12\x03rid\x18\x01"]
    k, v = normal("t", "x", "rid", 2 ** 64 - 1)
    assert W.route_match_infos(k, v) == [W.field(1, m) + b"\x12\x03rid\x18" + b"\xff" * 9 + b"\x01"]
    k, v = normal("t", "x", "", 5)                                                         # empty receiverId omitted
    assert W.route_match_infos(k, v) == [W.field(1, m) + b"\x18\x05"]


def test_share_members_carry_the_group_matcher_in_wire_order():
    urls = [O.receiver_url(1, "m%d" % i, "dk") for i in range(3)]
    k, v = group("t", "$share/g/a", [(urls[2], 7), (urls[0], 0), (urls[1], 2 ** 63)])
    m = W.route_matcher(k)
    assert W.route_match_infos(k, v) == [W.field(1, m) + W.field(2, b"m2") + b"\x18\x07", W.field(1, m) + W.field(2, b"m0"),
                                         W.field(1, m) + W.field(2, b"m1") + b"\x18" + W.varint(2 ** 63)]
    assert W.route_match_infos(*group("t", "$share/g/a", [])) == []


@pytest.mark.parametrize("n", [0, 1, 127, 128, 16383, 16384, 2 ** 21 - 1, 2 ** 21])
def test_length_prefixes_are_minimal_varints_at_their_boundaries(n):
    f = W.field(2, b"x" * n)
    assert len(f) == 1 + (1 if n < 128 else 2 if n < 16384 else 3 if n < 2 ** 21 else 4) + n
    assert W.fields(f) == [(2, 2, b"x" * n)]
    with pytest.raises(AssertionError):
        W.fields(b"\x12\x80\x00")                          # a two-byte zero is not minimal


def sample_request():
    ku, vu = normal("ténant✓", "a/+/é", "rid", 3)
    kg, vg = group("ténant✓", "$share/g/a/#", [(O.receiver_url(0, "m0", "d"), 1), (O.receiver_url(2, "", "d2"), 0)])
    ko, vo = group("other", "$oshare/o/#", [(O.receiver_url(0, "q", "d"), 9)])
    pubs = [W.field(1, b"client-%d" % i) + W.field(2, b"m" * (100 * i)) for i in range(3)]
    packages = [
        ("ténant✓".encode(), [(W.topic_message_pack("a/ü/é".encode(), pubs), W.route_match_infos(ku, vu) + W.route_match_infos(kg, vg)[1:]),
                              (W.topic_message_pack(b"a/x", []), W.route_match_infos(ku, vu))]),   # a pack with no publisher packs
        (b"other", [(W.topic_message_pack(b"a/b", pubs[2:]), W.route_match_infos(ko, vo))]),
    ]
    return packages


def test_restatement_round_trips_through_the_decoder():
    packages = sample_request()
    got = W.decode_request(W.delivery_request(packages))
    want = [(t, [(W.fields(tmp)[0][2] if W.fields(tmp) and W.fields(tmp)[0][0] == 1 else b"",
                  [v for n, _, v in W.fields(tmp) if n == 2], infos) for tmp, infos in packs]) for t, packs in packages]
    assert got == want
    assert got[0][1][1][1] == []                            # the pack without publisher packs keeps its topic and MatchInfo
    assert W.decode_request(b"") == []


def test_map_entries_and_packs_at_varint_boundaries():
    # publisher packs sized so the pack, package and entry lengths cross 127/128 and 16383/16384
    k, v = normal("t", "x", "r", 1)
    mi = W.route_match_infos(k, v)
    for size in range(100, 140):
        for big in (0, 16250):
            pp = W.field(2, b"p" * (size + big))
            req = W.delivery_request([(b"t", [(W.topic_message_pack(b"x", [pp]), mi)])])
            assert W.decode_request(req) == [(b"t", [(b"x", [pp], mi)])]


@pytest.mark.skipif(PB is None, reason="google.protobuf is not importable")
def test_restatement_equals_protobuf_messages_built_from_the_descriptors():
    ku, vu = normal("ténant✓", "a//é", "rid", 2 ** 64 - 1)
    kg, vg = group("ténant✓", "$oshare/g/a/+", [(O.receiver_url(0, "m0", "d"), 0)])
    kn, vn = normal("ténant✓", "", "", 0)
    # each MatchInfo serialized by protobuf from the fields NormalMatching sets
    for (k, v), (typ, levels, grp, tf, rid, inc) in [
            ((ku, vu), (0, ["a", "", "é"], None, "a//é", "rid", 2 ** 64 - 1)),
            ((kg, vg), (2, ["a", "+"], "g", "$oshare/g/a/+", "m0", 0)),
            ((kn, vn), (0, [""], None, "", "", 0))]:
        m = PB["RouteMatcher"](type=typ, filterLevel=levels, mqttTopicFilter=tf)
        if grp is not None:
            m.group = grp
        assert W.route_match_infos(k, v) == [PB["MatchInfo"](matcher=m, receiverId=rid, incarnation=inc).SerializeToString()]
    # the whole request parses, and equals the same request built with the builders
    packages = sample_request()
    req = PB["DeliveryRequest"]()
    for tenant, packs in packages:
        pkg = req.package[tenant.decode()]
        for tmp, infos in packs:
            p = pkg.pack.add()
            p.messagePack.ParseFromString(tmp)
            for mi in infos:
                p.matchInfo.add().ParseFromString(mi)
    parsed = PB["DeliveryRequest"].FromString(W.delivery_request(packages))
    assert parsed == req
    # one map entry re-serialized by protobuf is byte for byte the restatement's
    one = PB["DeliveryRequest"]()
    one.package["other"].CopyFrom(req.package["other"])
    assert one.SerializeToString() == W.delivery_request(packages[1:])
