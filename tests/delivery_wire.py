"""Restatement of the DeliveryRequest bytes a deliverer sends, and a small wire decoder for them.

What BatchDeliveryCall.execute (bifromq-deliverer/.../BatchDeliveryCall.java:91-108) serializes, built here literally:
  DeliveryRequest  { map<string tenantId, DeliveryPackage> package = 3 }   (subbroker/type.proto)
  DeliveryPackage  { repeated DeliveryPack pack = 1 }
  DeliveryPack     { TopicMessagePack messagePack = 2; repeated MatchInfo matchInfo = 3 }
  TopicMessagePack { string topic = 1; repeated PublisherPack message = 2 }          (commontype/TopicMessage.proto)
  MatchInfo        { RouteMatcher matcher = 1; string receiverId = 2; uint64 incarnation = 3 }   (commontype/MatchInfo.proto)
  RouteMatcher     { Type type = 1; repeated string filterLevel = 2; optional string group = 3; string mqttTopicFilter = 4 }
The MatchInfo of a route is NormalMatching's (schema/cache/NormalMatching.java:43-60): the RouteMatcher RouteDetailCache.get
builds from the route key (RouteDetailCache.java:53-109), the receiverUrl's second NUL-separated part (ReceiverCache.java:32-36)
and the incarnation (the normal route's 8-byte big-endian value). A group's members are NormalMatchings over the GROUP's
matcher (GroupMatching.java:41-50): type UnorderedShare / OrderedShare, group set, "$share/<g>/..." or "$oshare/<g>/...".
Proto3: a scalar at its default is not written, a message field that was set is, map entries carry both fields.
"""
import struct


def varint(v):
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def field(no, payload):
    """a length-delimited field: tag (no << 3 | 2), varint length, payload"""
    return varint(no << 3 | 2) + varint(len(payload)) + bytes(payload)


# ------------------------------------------------------------------ route key -> MatchInfo (RouteDetailCache, NormalMatching)
FLAG_NORMAL, FLAG_UNORDERED, FLAG_ORDERED = 1, 2, 3


def route_detail(key):
    """<VER><u16 tenant len><tenant><escaped filter><SEP SEP><bucket><flag><receiver bytes><u16 receiver len>
    -> (tenantId, flag, escaped filter, receiverInfo)"""
    key = bytes(key)
    tl = struct.unpack(">H", key[1:3])[0]
    rl = struct.unpack(">H", key[-2:])[0]
    rs = len(key) - 2 - rl
    flag = key[rs - 1]
    return key[3:3 + tl], flag, key[3 + tl:rs - 1 - 3], key[rs:len(key) - 2]


def route_matcher(key):
    _, flag, escaped, receiver = route_detail(key)
    unescaped = escaped.replace(b"\0", b"/")
    out = b""
    if flag != FLAG_NORMAL:                                  # Type.Normal = 0 is not written
        out += varint(1 << 3) + varint(1 if flag == FLAG_UNORDERED else 2)
    for level in escaped.split(b"\0"):                       # parse(escapedTopicFilter, true): every level, empty ones too
        out += field(2, level)
    if flag == FLAG_NORMAL:
        tf = unescaped
    else:
        out += field(3, receiver)                            # setGroup(receiverInfo): optional, so written even when empty
        tf = (b"$share" if flag == FLAG_UNORDERED else b"$oshare") + b"/" + receiver + b"/" + unescaped
    if tf:
        out += field(4, tf)
    return out


def match_info(matcher, receiver_url, incarnation):
    """MatchInfo.newBuilder().setMatcher(m).setReceiverId(parts[1]).setIncarnation(inc)"""
    out = field(1, matcher)
    rid = bytes(receiver_url).split(b"\0")[1]
    if rid:
        out += field(2, rid)
    if incarnation:
        out += varint(3 << 3) + varint(incarnation)
    return out


def group_members(value):
    """(receiverUrl, incarnation) of a RouteGroup value {map<string, uint64> members = 1}, in wire order"""
    out = []
    for no, wt, v in fields(bytes(value)):
        assert no == 1 and wt == 2
        url, inc = b"", 0
        for no2, wt2, v2 in fields(v):
            if no2 == 1:
                url = v2
            elif no2 == 2:
                inc = v2
        out.append((url, inc))
    return out


def route_match_infos(key, value):
    """the MatchInfos of one route: [one] for a normal route, one per member (wire order) for a group"""
    _, flag, _, receiver = route_detail(key)
    m = route_matcher(key)
    if flag == FLAG_NORMAL:
        return [match_info(m, receiver, struct.unpack(">Q", bytes(value)[:8])[0])]
    return [match_info(m, url, inc) for url, inc in group_members(value)]


# ------------------------------------------------------------------ the request (BatchDeliveryCall.execute)
def topic_message_pack(topic, publisher_packs):
    """TopicMessagePack.newBuilder().setTopic(topic).addMessage(pp)... (DeliverExecutorGroup.java:271-273)"""
    return (field(1, topic) if topic else b"") + b"".join(field(2, pp) for pp in publisher_packs)


def delivery_request(packages):
    """packages: [(tenantId bytes, [(TopicMessagePack bytes, [MatchInfo bytes, ...]), ...]), ...] in map order"""
    out = b""
    for tenant, packs in packages:
        package = b"".join(field(1, field(2, tmp) + b"".join(field(3, mi) for mi in infos)) for tmp, infos in packs)
        out += field(3, field(1, tenant) + field(2, package))
    return out


# ------------------------------------------------------------------ decoder
def read_varint(b, i):
    v = shift = 0
    while True:
        c = b[i]
        i += 1
        v |= (c & 0x7F) << shift
        if not c & 0x80:
            return v, i
        shift += 7


def fields(b, minimal=True):
    """[(field number, wire type, value)]: bytes for length-delimited fields, int for varints. minimal: assert every varint is
    the shortest encoding of its value"""
    out, i = [], 0
    while i < len(b):
        j = i
        tag, i = read_varint(b, i)
        no, wt = tag >> 3, tag & 7
        k = i
        v, i = read_varint(b, i)
        if minimal:
            assert i - k == len(varint(v)) and k - j == len(varint(tag)), "non-minimal varint"
        if wt == 2:
            assert i + v <= len(b), "length past the end"
            out.append((no, wt, bytes(b[i:i + v])))
            i += v
        else:
            assert wt == 0, "unexpected wire type %d" % wt
            out.append((no, wt, v))
    return out


def decode_request(b):
    """DeliveryRequest bytes -> [(tenantId, [(topic, [publisher pack bytes], [MatchInfo bytes]), ...]), ...]"""
    out = []
    for no, _, entry in fields(b):
        assert no == 3
        e = fields(entry)
        assert [f[0] for f in e] == [1, 2], "map entry must carry key then value"
        packs = []
        for no2, _, pack in fields(e[1][2]):
            assert no2 == 1
            p = fields(pack)
            assert p and p[0][0] == 2 and all(f[0] == 3 for f in p[1:]), "messagePack first, then matchInfo"
            tmp = fields(p[0][2])
            topic = tmp[0][2] if tmp and tmp[0][0] == 1 else b""
            pubs = [v for n, _, v in tmp if n == 2]
            assert len(pubs) + (1 if topic else 0) == len(tmp)
            packs.append((topic, pubs, [v for _, _, v in p[1:]]))
        out.append((e[0][2], packs))
    return out


# ------------------------------------------------------------------ protobuf messages from descriptors restated here
def protobuf_classes():
    """{name: message class} built from descriptors restated from the field numbers above, or None without google.protobuf"""
    try:
        from google.protobuf import descriptor_pb2, descriptor_pool, message_factory
    except ImportError:
        return None
    F = descriptor_pb2.FieldDescriptorProto
    fd = descriptor_pb2.FileDescriptorProto(name="bfq_delivery_wire_test.proto", package="bfqwire", syntax="proto3")

    def msg(name, specs, parent=None):
        m = (parent.nested_type if parent else fd.message_type).add(name=name)
        for fname, no, typ, label, tname in specs:
            f = m.field.add(name=fname, number=no, type=typ, label=label)
            if tname:
                f.type_name = tname
        return m
    OPT, REP = F.LABEL_OPTIONAL, F.LABEL_REPEATED
    rm = msg("RouteMatcher", [("type", 1, F.TYPE_ENUM, OPT, ".bfqwire.RouteMatcher.Type"),
                              ("filterLevel", 2, F.TYPE_STRING, REP, None), ("group", 3, F.TYPE_STRING, OPT, None),
                              ("mqttTopicFilter", 4, F.TYPE_STRING, OPT, None)])
    rm.field[2].proto3_optional = True
    rm.field[2].oneof_index = 0
    rm.oneof_decl.add(name="_group")
    e = rm.enum_type.add(name="Type")
    for i, n in enumerate(["Normal", "UnorderedShare", "OrderedShare"]):
        e.value.add(name=n, number=i)
    msg("MatchInfo", [("matcher", 1, F.TYPE_MESSAGE, OPT, ".bfqwire.RouteMatcher"), ("receiverId", 2, F.TYPE_STRING, OPT, None),
                      ("incarnation", 3, F.TYPE_UINT64, OPT, None)])
    # a publisher pack is opaque here: its two fields as bytes keep the wire form
    msg("PublisherPack", [("publisher", 1, F.TYPE_BYTES, OPT, None), ("message", 2, F.TYPE_BYTES, REP, None)])
    msg("TopicMessagePack", [("topic", 1, F.TYPE_STRING, OPT, None), ("message", 2, F.TYPE_MESSAGE, REP, ".bfqwire.PublisherPack")])
    msg("DeliveryPack", [("messagePack", 2, F.TYPE_MESSAGE, OPT, ".bfqwire.TopicMessagePack"),
                         ("matchInfo", 3, F.TYPE_MESSAGE, REP, ".bfqwire.MatchInfo")])
    msg("DeliveryPackage", [("pack", 1, F.TYPE_MESSAGE, REP, ".bfqwire.DeliveryPack")])
    req = msg("DeliveryRequest", [("package", 3, F.TYPE_MESSAGE, REP, ".bfqwire.DeliveryRequest.PackageEntry")])
    ent = msg("PackageEntry", [("key", 1, F.TYPE_STRING, OPT, None), ("value", 2, F.TYPE_MESSAGE, OPT, ".bfqwire.DeliveryPackage")], req)
    ent.options.map_entry = True
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fd)
    names = ["RouteMatcher", "MatchInfo", "PublisherPack", "TopicMessagePack", "DeliveryPack", "DeliveryPackage", "DeliveryRequest"]
    return {n: message_factory.GetMessageClass(pool.FindMessageTypeByName("bfqwire." + n)) for n in names}
