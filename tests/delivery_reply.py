"""Restatements of a deliverer's DeliveryReply and of what BatchDeliveryCall.execute does with it, plus a byte-level reply
writer for the shapes protobuf's own serializer never makes (unknown fields, permuted or repeated fields, non-canonical
MatchInfos).

  DeliveryReply   { Code code = 1 (OK, BACK_PRESSURE_REJECTED, ERROR); map<string tenantId, DeliveryResults> result = 2 }
  DeliveryResults { repeated DeliveryResult result = 1 }
  DeliveryResult  { MatchInfo matchInfo = 1; Code code = 2 (OK, NO_SUB, NO_RECEIVER) }       (subbroker/type.proto:41-63)

The messages are built on the protobuf classes of delivery_wire.protobuf_classes() (MatchInfo is that module's), so what is
equal here is what protobuf says is equal. Java's MatchInfo.equals compares fields and unknown fields; a deterministic
serialization does too, so it stands in for the HashMap key of TypeUtil.toMap.
"""
import numpy as np

import delivery_wire as W

# DeliveryCallResult, and the device's three codes for pairs it does not complete from a result
OK, NO_SUB, NO_RECEIVER, BACK_PRESSURE_REJECTED, ERROR, NO_RESULT, NOT_SENT, UNDECIDED = range(8)
FALLBACK = UNDECIDED


def protobuf_classes():
    """delivery_wire.protobuf_classes() plus DeliveryResult, DeliveryResults and DeliveryReply, or None without protobuf"""
    cls = W.protobuf_classes()
    if cls is None:
        return None
    from google.protobuf import descriptor_pb2, message_factory
    F = descriptor_pb2.FieldDescriptorProto
    pool = cls["MatchInfo"].DESCRIPTOR.file.pool
    fd = descriptor_pb2.FileDescriptorProto(name="bfq_delivery_reply_test.proto", package="bfqwire", syntax="proto3",
                                            dependency=["bfq_delivery_wire_test.proto"])
    OPT, REP = F.LABEL_OPTIONAL, F.LABEL_REPEATED

    def msg(name, specs, parent=None):
        m = (parent.nested_type if parent else fd.message_type).add(name=name)
        for fname, no, typ, label, tname in specs:
            f = m.field.add(name=fname, number=no, type=typ, label=label)
            if tname:
                f.type_name = tname
        return m
    r = msg("DeliveryResult", [("matchInfo", 1, F.TYPE_MESSAGE, OPT, ".bfqwire.MatchInfo"),
                               ("code", 2, F.TYPE_ENUM, OPT, ".bfqwire.DeliveryResult.Code")])
    e = r.enum_type.add(name="Code")
    for i, n in enumerate(["OK", "NO_SUB", "NO_RECEIVER"]):
        e.value.add(name=n, number=i)
    msg("DeliveryResults", [("result", 1, F.TYPE_MESSAGE, REP, ".bfqwire.DeliveryResult")])
    rep = msg("DeliveryReply", [("code", 1, F.TYPE_ENUM, OPT, ".bfqwire.DeliveryReply.Code"),
                                ("result", 2, F.TYPE_MESSAGE, REP, ".bfqwire.DeliveryReply.ResultEntry")])
    e = rep.enum_type.add(name="Code")
    for i, n in enumerate(["OK", "BACK_PRESSURE_REJECTED", "ERROR"]):
        e.value.add(name=n, number=i)
    ent = msg("ResultEntry", [("key", 1, F.TYPE_STRING, OPT, None), ("value", 2, F.TYPE_MESSAGE, OPT, ".bfqwire.DeliveryResults")], rep)
    ent.options.map_entry = True
    pool.Add(fd)
    for n in ["DeliveryResult", "DeliveryResults", "DeliveryReply"]:
        cls[n] = message_factory.GetMessageClass(pool.FindMessageTypeByName("bfqwire." + n))
    return cls


_CLS = None


def classes():
    global _CLS
    if _CLS is None:
        _CLS = protobuf_classes()
    return _CLS


def request_match_infos(request):
    """{tenantId: [distinct MatchInfo messages in request order]} of a serialized DeliveryRequest"""
    c = classes()
    req = c["DeliveryRequest"].FromString(bytes(request))
    out = {}
    for tenant in sorted(req.package):
        seen, infos = set(), []
        for pack in req.package[tenant].pack:
            for mi in pack.matchInfo:
                k = mi.SerializeToString(deterministic=True)
                if k not in seen:
                    seen.add(k)
                    infos.append(mi)
        out[tenant] = infos
    return out


# ------------------------------------------------------------------ what a sub-broker sends
def local_dist_reply(request, code_of):
    """LocalDistService.dist (bifromq-mqtt-server/.../LocalDistService.java:196-205): code OK, per tenant of the request one
    DeliveryResult per distinct MatchInfo, echoing the request's MatchInfo object: the OK ones first, then NO_SUB, then
    NO_RECEIVER. code_of(tenant, MatchInfo bytes) -> 0, 1 or 2."""
    c = classes()
    reply = c["DeliveryReply"]()
    for tenant, infos in request_match_infos(request).items():
        res = reply.result[tenant]
        coded = [(code_of(tenant, mi.SerializeToString()), mi) for mi in infos]
        for want in (OK, NO_SUB, NO_RECEIVER):
            for code, mi in coded:
                if code == want:
                    r = res.result.add(code=code)
                    r.matchInfo.CopyFrom(mi)
    return reply.SerializeToString()


def pipeline_no_receiver_reply(request):
    """DeliveryPipeline.deliver on ServerNotFoundException (bifromq-mqtt-broker-client/.../DeliveryPipeline.java:49-80): code OK
    (not written), every distinct MatchInfo of every tenant NO_RECEIVER"""
    return local_dist_reply(request, lambda tenant, mi: NO_RECEIVER)


FAILED_CALL = b"\x08\x02"   # `.exceptionally`: DeliveryReply.newBuilder().setCode(ERROR).build()


# ------------------------------------------------------------------ execute's reply branch
class DuplicateKey(Exception):
    """Collectors.toMap's IllegalStateException"""


def mi_key(mi):
    return mi.SerializeToString(deterministic=True)


def wire_fields(b):
    """[(field number, wire type, value)] of wire types 0, 1, 2 and 5: an int, or the bytes of the fixed / length-delimited"""
    out, i = [], 0
    while i < len(b):
        tag, i = W.read_varint(b, i)
        no, wt = tag >> 3, tag & 7
        if wt == 0:
            v, i = W.read_varint(b, i)
        elif wt in (1, 5):
            n = 8 if wt == 1 else 4
            v, i = bytes(b[i:i + n]), i + n
        else:
            assert wt == 2, "wire type %d" % wt
            n, i = W.read_varint(b, i)
            v, i = bytes(b[i:i + n]), i + n
        out.append((no, wt, v))
    return out


def result_map(reply_bytes):
    """reply.getResultMap() as protobuf-java parses it: a map entry's unknown fields are skipped (MapEntryLite.parseEntry) and
    a later entry for a key replaces the earlier one. (upb, under Python's protobuf, would instead keep an entry that carries
    unknown fields among the reply's unknown fields, so the entries are read here and only their values parsed by protobuf.)"""
    c = classes()
    out = {}
    for no, wt, v in wire_fields(bytes(reply_bytes)):
        if no != 2 or wt != 2:
            continue
        key, value = b"", b""
        for no2, wt2, v2 in wire_fields(v):
            if no2 == 1 and wt2 == 2:
                key = v2
            elif no2 == 2 and wt2 == 2:
                value = v2
        out[key.decode("utf-8")] = c["DeliveryResults"].FromString(value)
    return out


def to_map(reply_bytes):
    """TypeUtil.toMap (bifromq-plugin-sub-broker/.../TypeUtil.java:27-41): {tenantId: {MatchInfo key: code}}"""
    out = {}
    for tenant, results in result_map(reply_bytes).items():
        inner = out[tenant] = {}
        for r in results.result:
            k = mi_key(r.matchInfo)
            if k in inner:
                raise DuplicateKey((tenant, k))
            inner[k] = r.code
    return out


def execute(tasks, reply_bytes):
    """BatchDeliveryCall.execute's reply handling (BatchDeliveryCall.java:108-172) for one deliverer.
    tasks: [(tenantId, MatchInfo bytes)] one per (tenant, MatchInfo, pack) call; reply_bytes: the serialized DeliveryReply.
    -> (status: OK, BACK_PRESSURE_REJECTED or ERROR; [code per task]; {(tenantId, MatchInfo key)} the stale MatchInfos).
    A task without a result is NO_RESULT (the reference completes it OK and logs "No deliver result")."""
    c = classes()
    reply = c["DeliveryReply"].FromString(bytes(reply_bytes))
    if reply.code == 1:
        return BACK_PRESSURE_REJECTED, [BACK_PRESSURE_REJECTED] * len(tasks), set()
    if reply.code != 0:
        return ERROR, [ERROR] * len(tasks), set()
    result_map = to_map(reply_bytes)
    codes, stale = [], set()
    for tenant, mi in tasks:
        k = mi_key(c["MatchInfo"].FromString(bytes(mi)))
        r = result_map.get(tenant, {}).get(k)
        if r is None:
            codes.append(NO_RESULT)
            continue
        if r in (NO_SUB, NO_RECEIVER):
            stale.add((tenant, k))
        codes.append(r if r in (OK, NO_SUB, NO_RECEIVER) else ERROR)
    return OK, codes, stale


# ------------------------------------------------------------------ byte-level writer
UNKNOWN = [W.varint(9 << 3 | 0) + W.varint(300),                        # varint
           W.varint(10 << 3 | 1) + bytes(range(8)),                    # fixed64
           W.varint(11 << 3 | 2) + W.varint(3) + b"\x0a\x05\x12",      # length-delimited that looks like a record head
           W.varint(12 << 3 | 5) + b"\x0a\x02\x08\x01"]                # fixed32


def varint_field(no, v):
    return W.varint(no << 3) + W.varint(v & (2 ** 64 - 1))              # a negative int32 is its 10-byte two's complement


def record(mi, code, unknown=b"", code_first=False, explicit_code=False):
    """one DeliveryResult field (result = 1 of DeliveryResults)"""
    parts = [W.field(1, mi), varint_field(2, code) if code or explicit_code else b""]
    if code_first:
        parts.reverse()
    return W.field(1, unknown + b"".join(parts))


def reply(entries, code=0, unknown=b"", value_first=False, code_last=False, explicit_code=False):
    """a DeliveryReply: entries [(tenant bytes, DeliveryResults bytes)] as map entries (key, value or value, key)"""
    out = varint_field(1, code) if code or explicit_code else b""
    body = b""
    for tenant, results in entries:
        kv = [W.field(1, tenant), W.field(2, results)]
        if value_first:
            kv.reverse()
        body += W.field(2, unknown + b"".join(kv))
    return unknown + (body + out if code_last else out + body)


# ------------------------------------------------------------------ replies for a whole nesting (large batches)
def nesting_replies(a, n_deliverers, tenants, mi_of, rng, p_no_sub, p_no_receiver):
    """LocalDistService's replies for every deliverer of a nesting, written from its arrays (dl.arrays()): per package one map
    entry, per distinct (rank, member) of the package one DeliveryResult with a seeded code (about p_no_sub NO_SUB and
    p_no_receiver NO_RECEIVER, the rest OK with the code omitted). mi_of(rank, member) -> the pair's MatchInfo bytes.
    ordered_share_id gets an empty slice. -> dict: blob, off [n_deliverers + 1], per distinct key its package, rank, member and
    code, and per pair its key index"""
    po, ko, mo = a["package_off"], a["pack_off"], a["match_off"]
    pack_pkg = np.repeat(np.arange(len(ko) - 1), np.diff(ko))
    pair_pkg = pack_pkg[np.repeat(np.arange(len(mo) - 1), np.diff(mo))]
    keys = np.stack([pair_pkg.astype(np.int64), a["match_rank"].astype(np.int64), a["match_member"].astype(np.int64)])
    order = np.lexsort(keys[::-1])
    k = keys[:, order]
    first = np.ones(k.shape[1], bool)
    first[1:] = (np.diff(k, axis=1) != 0).any(axis=0)
    key_of_pair = np.empty(k.shape[1], np.int64)
    key_of_pair[order] = np.cumsum(first) - 1
    pkg, rank, member = k[:, first]
    u = rng.random(len(pkg))
    code = np.where(u < p_no_sub, NO_SUB, np.where(u < p_no_sub + p_no_receiver, NO_RECEIVER, OK))
    tail = {0: b"", 1: b"\x10\x01", 2: b"\x10\x02"}
    bounds = np.searchsorted(pkg, np.arange(len(ko)))          # each package's first key, and the end
    blob, off = [], [0]
    for d in range(n_deliverers):
        parts = []
        if d < n_deliverers - 1:
            for g in range(int(po[d]), int(po[d + 1])):
                body = b"".join(W.field(1, W.field(1, mi_of(int(rank[i]), int(member[i]))) + tail[int(code[i])])
                                for i in range(int(bounds[g]), int(bounds[g + 1])))
                parts.append(W.field(2, W.field(1, tenants[int(a["package_tenant"][g])].encode()) + W.field(2, body)))
        rep = b"".join(parts)
        blob.append(rep)
        off.append(off[-1] + len(rep))
    return {"blob": b"".join(blob), "off": np.asarray(off, np.int64), "pkg": pkg, "rank": rank, "member": member,
            "code": code, "key_of_pair": key_of_pair, "sent": pkg < po[n_deliverers - 1]}


# ------------------------------------------------------------------ a model of the device's chunk guesses (tests only)
def _varint(b, i, end, max_bytes):
    v = 0
    for k in range(max_bytes):
        if i >= end:
            return None, i
        c = b[i]
        i += 1
        v |= (c & 0x7F) << (7 * k)
        if not c & 0x80:
            return v, i
    return None, i


def _field(b, i, end):
    """(field number, wire type, payload start, payload end or value, next) or None, as the device reads a field"""
    tag, i = _varint(b, i, end, 5)
    if tag is None or tag > 0xFFFFFFFF or tag >> 3 == 0:
        return None
    wt = tag & 7
    if wt == 0:
        v, i = _varint(b, i, end, 10)
        return None if v is None else (tag >> 3, 0, v, v, i)
    if wt in (1, 5):
        i += 8 if wt == 1 else 4
        return None if i > end else (tag >> 3, wt, i, i, i)
    if wt == 2:
        n, i = _varint(b, i, end, 5)
        if n is None or n > end - i:
            return None
        return tag >> 3, 2, i, i + n, i + n
    return None


def _is_result(b, s, e):
    seen_mi = seen_code = False
    while s < e:
        f = _field(b, s, e)
        if f is None:
            return False
        no, wt, _, _, s = f
        if no == 1:
            if wt != 2 or seen_mi:
                return False
            seen_mi = True
        elif no == 2:
            if wt != 0 or seen_code:
                return False
            seen_code = True
    return seen_mi


def chunk_guesses(reply_bytes, chunk=2048):
    """Per map entry of a well-formed reply, its DeliveryResults cut into `chunk`-byte chunks as the device cuts them: for
    every chunk after the first, (the device's guess, or None; the true start: the first field at or past the chunk's start),
    and for every field that crosses a chunk boundary, how far into the field the boundary falls."""
    b = bytes(reply_bytes)
    guesses, crossings = [], []
    for no, wt, v in wire_fields(b):
        if no != 2 or wt != 2:
            continue
        value = b""
        for no2, wt2, v2 in wire_fields(v):
            if no2 == 2 and wt2 == 2:
                value = v2
        starts, i = [], 0
        while i < len(value):
            starts.append(i)
            i = _field(value, i, len(value))[4]
        for c in range(chunk, len(value), chunk):
            guess = None
            for q in range(c, min(c + chunk, len(value))):
                if value[q] != 0x0A:
                    continue
                n, r = _varint(value, q + 1, len(value), 5)
                if n is not None and n <= len(value) - r and _is_result(value, r, r + n):
                    guess = q
                    break
            true = next((x for x in starts if x >= c), len(value))
            guesses.append((guess, true))
        for x, y in zip(starts, starts[1:] + [len(value)]):
            crossings += [c - x for c in range((x // chunk + 1) * chunk, y, chunk)]
    return guesses, crossings
