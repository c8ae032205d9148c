"""The DeliveryReply restatements of tests/delivery_reply.py pinned on hand-written cases, without a GPU."""
import pytest

import delivery_reply as R
import delivery_wire as W

pytestmark = pytest.mark.skipif(R.classes() is None, reason="google.protobuf is not installed")


def mi(filter_, rid, inc=0):
    return W.match_info(W.field(2, filter_) + W.field(4, filter_), b"1\0" + rid + b"\0d", inc)


A, B_, C = mi(b"a", b"r1", 5), mi(b"b", b"r2"), mi(b"c", b"r3", 2 ** 64 - 1)


def request(packages):
    return W.delivery_request([(t, [(W.topic_message_pack(b"x", []), infos) for infos in packs]) for t, packs in packages])


def test_local_dist_reply_echoes_every_distinct_match_info():
    req = request([(b"t1", [[A, B_], [A]]), (b"t2", [[C]])])
    codes = {A: R.NO_SUB, B_: R.OK, C: R.NO_RECEIVER}
    rep = R.local_dist_reply(req, lambda t, m: codes[m])
    tasks = [("t1", A), ("t1", B_), ("t1", A), ("t2", C)]
    status, got, stale = R.execute(tasks, rep)
    assert status == R.OK and got == [R.NO_SUB, R.OK, R.NO_SUB, R.NO_RECEIVER]
    assert {(t, k) for t, k in stale} == {("t1", A), ("t2", C)}
    parsed = R.classes()["DeliveryReply"].FromString(rep)
    assert [r.code for r in parsed.result["t1"].result] == [R.OK, R.NO_SUB]   # OK first, then NO_SUB, each MatchInfo once


def test_pipeline_reply_is_all_no_receiver_and_every_match_info_is_stale():
    req = request([(b"t1", [[A, B_], [B_]])])
    status, got, stale = R.execute([("t1", A), ("t1", B_), ("t1", B_)], R.pipeline_no_receiver_reply(req))
    assert status == R.OK and got == [R.NO_RECEIVER] * 3 and len(stale) == 2


def test_reply_codes_and_a_failed_call():
    tasks = [("t1", A), ("t1", B_)]
    assert R.execute(tasks, b"\x08\x01")[:2] == (R.BACK_PRESSURE_REJECTED, [R.BACK_PRESSURE_REJECTED] * 2)
    assert R.execute(tasks, R.FAILED_CALL)[:2] == (R.ERROR, [R.ERROR] * 2)
    assert R.execute(tasks, b"\x08\x07")[:2] == (R.ERROR, [R.ERROR] * 2)            # UNRECOGNIZED -> default branch
    assert R.execute(tasks, b"") == (R.OK, [R.NO_RESULT] * 2, set())                 # a default reply: no results
    # results are ignored under BACK_PRESSURE_REJECTED: no stale routes
    rep = R.reply([(b"t1", R.record(A, R.NO_SUB))], code=1)
    assert R.execute(tasks, rep) == (R.BACK_PRESSURE_REJECTED, [R.BACK_PRESSURE_REJECTED] * 2, set())


def test_unknown_result_codes_complete_as_error_and_are_not_stale():
    rep = R.reply([(b"t1", R.record(A, 7) + R.record(B_, -1) + R.record(C, R.NO_SUB))])
    status, got, stale = R.execute([("t1", A), ("t1", B_), ("t1", C)], rep)
    assert status == R.OK and got == [R.ERROR, R.ERROR, R.NO_SUB] and stale == {("t1", C)}


def test_duplicates_raise():
    rep = R.reply([(b"t1", R.record(A, 0) + R.record(A, 1))])
    with pytest.raises(R.DuplicateKey):
        R.execute([("t1", A)], rep)
    # a non-canonical encoding of A is still A: a duplicate too
    reordered = W.field(2, b"r1") + W.field(1, W.field(2, b"a") + W.field(4, b"a")) + W.varint(3 << 3) + W.varint(5)
    rep = R.reply([(b"t1", R.record(A, 0) + R.record(reordered, 1))])
    with pytest.raises(R.DuplicateKey):
        R.execute([("t1", A)], rep)
    # the same MatchInfo under two tenants is two keys
    rep = R.reply([(b"t1", R.record(A, 1)), (b"t2", R.record(A, 2))])
    assert R.execute([("t1", A), ("t2", A)], rep)[1] == [R.NO_SUB, R.NO_RECEIVER]


def test_non_canonical_match_infos_still_match():
    reordered = W.field(2, b"r1") + W.field(1, W.field(2, b"a") + W.field(4, b"a")) + W.varint(3 << 3) + W.varint(5)
    explicit_zero = B_ + W.varint(3 << 3) + W.varint(0)
    long_len = W.varint(1 << 3 | 2) + b"\x86\x00" + W.field(2, b"b") + W.field(4, b"b") + W.field(2, b"r2")   # 2-byte length 6
    for enc, want in ((reordered, A), (explicit_zero, B_), (long_len, B_)):
        assert enc != want
        rep = R.reply([(b"t1", R.record(enc, R.NO_SUB))])
        status, got, stale = R.execute([("t1", want)], rep)
        assert got == [R.NO_SUB] and len(stale) == 1


def test_unknown_fields_and_permuted_order_parse_as_the_plain_reply():
    plain = R.reply([(b"t1", R.record(A, R.NO_SUB) + R.record(B_, R.OK))], code=0)
    odd = R.reply([(b"t1", R.UNKNOWN[3] + R.record(A, R.NO_SUB, unknown=b"".join(R.UNKNOWN), code_first=True) + R.UNKNOWN[0] +
                    R.record(B_, R.OK, explicit_code=True))],
                  unknown=b"".join(R.UNKNOWN), value_first=True, code_last=True, explicit_code=True)
    tasks = [("t1", A), ("t1", B_), ("t1", C)]
    assert R.execute(tasks, odd) == R.execute(tasks, plain)
    assert R.execute(tasks, plain)[1] == [R.NO_SUB, R.OK, R.NO_RESULT]


def test_a_result_without_code_is_ok():
    rep = R.reply([(b"t1", W.field(1, W.field(1, A)))])
    assert R.execute([("t1", A)], rep) == (R.OK, [R.OK], set())
