"""Pins the CPU oracle against the golden vectors the reference's own tests carry for this path
(SURVEY.md §8c). Every case names the reference test it transcribes. Paths relative to the reference repository's root.

The reference is Java and cannot run here (no JDK); these vectors are literal constants of its test
sources, re-typed (inputs and expected outputs only).
"""
import random

import numpy as np
import pytest

import oracle_lib as O

# ------------------------------------------------------------------------------------------------
# bifromq-util/src/test/java/org/apache/bifromq/util/TopicUtilsTest.java
# ------------------------------------------------------------------------------------------------


def test_parse_vectors():  # TopicUtilsTest.java:45-62
    def esc(s):
        return s.replace("/", "\0")
    cases = {"": [""], " ": [" "], "/": ["", ""], "//": ["", "", ""], " //": [" ", "", ""], " / / ": [" ", " ", " "],
             "a/": ["a", ""], "a/b": ["a", "b"], "a/b/": ["a", "b", ""]}
    for s, want in cases.items():
        assert O.parse(s, False) == want
        assert O.parse(esc(s), True) == want


def test_is_valid_topic_vectors():  # TopicUtilsTest.java:64-85
    T, F = True, False
    cases = [("/", 40, 16, 255, T), ("//", 40, 16, 255, T), ("", 40, 16, 255, F), (" ", 40, 16, 255, T),
             ("/ ", 40, 16, 255, T), ("/ /", 40, 16, 255, T), ("/\0abc/", 40, 16, 255, F), ("/abc/", 2, 16, 255, F),
             ("abc", 4, 1, 255, T), ("/", 4, 1, 255, F), ("/", 4, 2, 255, T), ("/abcde/fghij", 5, 4, 10, F),
             ("/+/#", 5, 4, 10, F), ("$share/a/", 5, 4, 10, F), ("$share/a//", 5, 4, 10, F),
             ("$share", 10, 4, 20, T), ("$shared/a//", 10, 4, 20, T)]
    for s, a, b, c, want in cases:
        assert O.is_valid_topic(s, a, b, c) == want, s


def test_is_valid_topic_filter_vectors():  # TopicUtilsTest.java:87-150
    T, F = True, False
    cases = [("/", 40, 16, 255, T), ("//", 40, 16, 255, T), ("", 40, 16, 255, F), (" ", 40, 16, 255, T),
             ("/ ", 40, 16, 255, T), ("/ /", 40, 16, 255, T), ("/\0abc/", 40, 16, 255, F), ("/abc/", 2, 16, 255, F),
             ("abc", 4, 1, 255, T), ("/", 4, 1, 255, F), ("/", 4, 2, 255, T), ("/abcde/fghij", 5, 4, 10, F),
             ("#", 40, 16, 255, T), ("a/#", 40, 16, 255, T), ("+", 40, 16, 255, T), ("+/", 40, 16, 255, T),
             ("+/+", 40, 16, 255, T), ("/+/#", 40, 16, 255, T), ("+/a/#", 40, 16, 255, T),
             ("#a", 40, 16, 255, F), ("#/a", 40, 16, 255, F), ("/a#", 40, 16, 255, F), ("/a#a", 40, 16, 255, F),
             ("/a+/", 40, 16, 255, F), ("/+a/", 40, 16, 255, F), ("/a+a/", 40, 16, 255, F), ("a+", 40, 16, 255, F),
             ("+a", 40, 16, 255, F), ("/a/+#", 40, 16, 255, F),
             ("$share/", 5, 4, 10, F), ("$share/a", 5, 4, 10, F), ("$share/\0/", 5, 4, 10, F), ("$share//", 5, 4, 10, F),
             ("$oshare/", 5, 4, 10, F), ("$oshare//", 5, 4, 10, F), ("$oshare/a", 5, 4, 10, F),
             ("$oshare/\0/", 5, 4, 10, F),
             ("$share", 10, 4, 100, T), ("$oshare", 10, 4, 100, T), ("$shared/", 10, 4, 10, T),
             ("$oshared/", 10, 4, 100, T), ("$share/g/", 10, 4, 100, T), ("$share/g//", 10, 4, 100, T),
             ("$share/g/abcdef/", 5, 4, 10, F), ("$share/g/1/2/3/4/5", 5, 4, 255, F), ("$share/g//1/2/3/4", 5, 4, 255, F),
             ("$share/g//1/2/3/", 5, 4, 255, F),
             ("$share/g/+/a", 10, 4, 100, T), ("$share/g/#", 10, 4, 100, T), ("$share/g//#", 10, 4, 100, T),
             ("$share/g//+/a/#", 10, 4, 100, T),
             ("$share/g//a+", 10, 4, 100, F), ("$share/g/+a", 10, 4, 100, F), ("$share/g/#/a", 10, 4, 100, F)]
    for s, a, b, c, want in cases:
        assert O.is_valid_topic_filter(s, a, b, c) == want, s


def test_is_wildcard_topic_filter():  # TopicUtilsTest.java:~38-42
    assert O.is_wildcard_topic_filter("/+")
    assert not O.is_wildcard_topic_filter("/")
    assert O.is_wildcard_topic_filter("#")
    assert O.is_wildcard_topic_filter("a/#")


def test_route_matcher_serde():  # TopicUtilsTest.java:152-194
    m = O.route_matcher_from("a/b/c")
    assert m == {"type": "Normal", "filterLevels": ["a", "b", "c"], "group": "", "mqttTopicFilter": "a/b/c"}
    m = O.route_matcher_from("$share/group/a/b/c")
    assert (m["type"], m["filterLevels"], m["group"]) == ("UnorderedShare", ["a", "b", "c"], "group")
    m = O.route_matcher_from("$share/group//a/b/c")
    assert (m["type"], m["filterLevels"], m["group"]) == ("UnorderedShare", ["", "a", "b", "c"], "group")
    m = O.route_matcher_from("$oshare/group/a/b/c")
    assert (m["type"], m["filterLevels"], m["group"]) == ("OrderedShare", ["a", "b", "c"], "group")
    m = O.route_matcher_from("$oshare/group//a/b/c")
    assert (m["type"], m["filterLevels"], m["group"], m["mqttTopicFilter"]) == \
           ("OrderedShare", ["", "a", "b", "c"], "group", "$oshare/group//a/b/c")


# ------------------------------------------------------------------------------------------------
# JDK String behaviours + the worked key example of SURVEY.md §8a
# ------------------------------------------------------------------------------------------------


def test_java_string_hash_and_bucket():
    assert O.java_hash("hello") == 99162322            # well-known JDK value
    assert O.java_hash("") == 0
    assert O.java_hash("a") == 97
    assert O.java_hash("polygenelubricants") == -2147483648   # well-known Integer.MIN_VALUE hash
    assert O.java_hash("你好") == 0x4f60 * 31 + 0x597d
    assert O.java_hash("😄") == 0xD83D * 31 + 0xDE04           # surrogate pair = two UTF-16 units
    assert O.bucket(b"0\x00inbox1\x00d1") == 0xC0              # SURVEY.md §8a worked example
    assert O.bucket("g1") == 0xAA


def test_java_compare_is_utf16_order():
    assert O.java_compare("a", "b") < 0
    assert O.java_compare("a", "a") == 0
    assert O.java_compare("", "#") < 0 and O.java_compare("#", "+") < 0 and O.java_compare("+", "a") < 0
    # U+FF5E (BMP) vs U+1F604 (supplementary): UTF-8 bytes order them one way, UTF-16 units the other
    assert "～".encode() < "😄".encode()
    assert O.java_compare("～", "😄") > 0


def test_worked_route_keys():  # SURVEY.md §8a (hand-derived from KVSchemaUtil.java:91-130)
    url = O.receiver_url(0, "inbox1", "d1")
    assert url == b"0\x00inbox1\x00d1"
    k = O.route_key("t", "a/+", url)
    assert k == bytes.fromhex("00" "000174" "6100" "2b00" "00" "c0" "01" "3000696e626f7831006431" "000b")
    k = O.route_key("t", "$share/g1/a/#")
    assert k == bytes.fromhex("00" "000174" "6100" "2300" "00" "aa" "02" "6731" "0002")
    assert O.tenant_begin_key("t") == bytes.fromhex("00000174")
    assert O.tenant_route_start_key("t", "a/+") == bytes.fromhex("00000174" "6100" "2b00" "00")
    assert O.upper_bound(bytes.fromhex("00000174")) == bytes.fromhex("00000175")
    assert O.upper_bound(b"\x01\xff\xff") == b"\x02"
    assert O.upper_bound(b"\xff\xff") is None


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-worker-schema/src/test/.../KVSchemaUtilTest.java (codec round trips)
# ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("tf", ["/a/b/c", "a", "a/", "/", "#", "+/+", "$sys/#",
                                "$share/group//a/b/c", "$oshare/group//a/b/c", "$share/g/#", "$oshare/g/+"])
def test_route_key_roundtrip(tf):
    url = O.receiver_url(1, "inbox1", "deliverer1")
    key = O.route_key("tenantA", tf, url)
    shared = tf.startswith("$share/") or tf.startswith("$oshare/")
    val = O.route_group({url: 7}) if shared else O.incarnation_bytes(42)
    m = O.build_match_route(key, val)
    assert m["tenantId"] == "tenantA"
    assert m["mqttTopicFilter"] == tf
    want_levels = O.route_matcher_from(tf)["filterLevels"]
    assert m["filterLevels"] == want_levels
    if shared:
        assert m["type"] == "Group" and m["members"] == {url: 7}
    else:
        assert (m["type"], m["receiverUrl"], m["incarnation"], m["subBrokerId"]) == ("Normal", url, 42, 1)


def test_negative_sub_broker_id():
    url = O.receiver_url(-5, "r", "d")
    m = O.build_match_route(O.route_key("t", "a", url), O.incarnation_bytes(1))
    assert m["subBrokerId"] == -5


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-coproc-proto/src/test/.../trie/Fixtures.java:31-105 (+ TopicFilterIteratorTest)
# ------------------------------------------------------------------------------------------------
GLOBAL_FIXTURES = {
    "tenantA/a": ["tenantA/#", "tenantA/+", "tenantA/+/#", "tenantA/a", "tenantA/a/#"],
    "tenantA/a/b": ["tenantA/#", "tenantA/+/#", "tenantA/+/+", "tenantA/+/+/#", "tenantA/+/b", "tenantA/+/b/#",
                    "tenantA/a/#", "tenantA/a/+", "tenantA/a/+/#", "tenantA/a/b", "tenantA/a/b/#"],
    "tenantA/$sys/a": ["tenantA/$sys/#", "tenantA/$sys/+", "tenantA/$sys/+/#", "tenantA/$sys/a", "tenantA/$sys/a/#"],
    "tenantA//": ["tenantA//", "tenantA///#", "tenantA//#", "tenantA//+", "tenantA//+/#", "tenantA/#", "tenantA/+/",
                  "tenantA/+//#", "tenantA/+/#", "tenantA/+/+", "tenantA/+/+/#"],
}
LOCAL_FIXTURES = {
    "a": ["#", "+", "+/#", "a", "a/#"],
    "$sys/a": ["$sys/#", "$sys/+", "$sys/+/#", "$sys/a", "$sys/a/#"],
    "/": ["/", "//#", "/#", "/+", "/+/#", "#", "+/", "+//#", "+/#", "+/+", "+/+/#"],
}


@pytest.mark.parametrize("is_global,fixtures", [(True, GLOBAL_FIXTURES), (False, LOCAL_FIXTURES)])
def test_expansion_fixtures(is_global, fixtures):  # TopicFilterIteratorTest.expandGlobalTopics/expandLocalTopics :61-68,344-360
    for topic, filters in fixtures.items():
        got = ["/".join(lv) for lv, _ in O.expansion_list([topic], is_global)]
        assert got == filters, topic
    # all topics together: union, still sorted in iterator order (level-wise compareTo)
    topics = list(fixtures)
    got = [lv for lv, _ in O.expansion_list(topics, is_global)]
    want = sorted({tuple(f.split("/")) for fs in fixtures.values() for f in fs})
    assert [tuple(g) for g in got] == want


def test_expansion_associated_values():  # TopicFilterIteratorTest.associatedValues :283-314
    topics = ["a", "a/b", "c"]
    ex = {tuple(lv): sorted(v) for lv, v in O.expansion_list(topics)}
    assert ex[("#",)] == [0, 1, 2]
    assert ex[("+",)] == [0, 2]
    assert ex[("a", "#")] == [0, 1]
    assert ex[("a", "+")] == [1]
    assert ex[("a", "+", "#")] == [1]
    for f in ["#", "+", "a/#", "a/+", "a/+/#"]:
        assert O.expansion_seek(topics, f) == f.split("/")


def test_expansion_sys_topic_rule():  # TopicFilterIteratorTest.localSysTopicMatch/globalSysTopicMatch :317-342
    ex = {tuple(lv): sorted(v) for lv, v in O.expansion_list(["$sys/a", "a/b", "c"])}
    assert ex[("#",)] == [1, 2]
    ex = {tuple(lv): sorted(v) for lv, v in O.expansion_list(["tenant/$sys/a", "tenant/a/b", "tenant/c"], True)}
    assert ex[("tenant", "#")] == [1, 2]


def _random_topic(rng, max_level=6):
    # DCPT/TestUtil.java:54-66 shape (BMP alphabet incl. CJK; '$' prefix and leading '/' with p=0.5)
    syms = "ABCDEFGHIJKLMNOPQRSTUVWXYZ你好abcdefghijklmnopqrstuvwxyz0123456789 !\"$%&'()*,-."
    lv = ["".join(rng.choice(syms) for _ in range(rng.randint(1, 7))) for _ in range(rng.randint(1, max_level))]
    if rng.random() > 0.5:
        lv[0] = "$" + lv[0]
    t = "/".join(lv)
    return "/" + t if rng.random() > 0.5 else t


def _random_filter(rng, max_level=6):
    syms = "ABCabc你好012 $-"
    n = rng.randint(1, max_level)
    lv = []
    for i in range(n):
        if rng.random() > 0.5:
            lv.append("+" if i < n - 1 else "#")
        else:
            lv.append("".join(rng.choice(syms) for _ in range(rng.randint(1, 4))))
    return "/".join(lv)


def test_expansion_seek_then_iterate_random():  # TopicFilterIteratorTest.seekExistAndIteration/randomSeekAndIteration :70-118
    rng = random.Random(7)
    for _ in range(60):
        topics = [_random_topic(rng) for _ in range(3)]
        gen = [lv for lv, _ in O.expansion_list(topics)]
        # sorted, strictly increasing in level-wise String.compareTo order
        for a, b in zip(gen, gen[1:]):
            assert a != b
            cmp = 0
            for x, y in zip(a, b):
                cmp = O.java_compare(x, y)
                if cmp:
                    break
            assert cmp < 0 or (cmp == 0 and len(a) < len(b))
        # every generated filter matches at least one topic under the predicate; seek(existing) == itself
        for lv in gen[:: max(1, len(gen) // 8)]:
            f = "/".join(lv)
            assert any(O.topic_matches_filter(t, f) for t in topics)
            assert O.expansion_seek(topics, f) == lv
        # random seek lands on the least generated filter >= target
        for _ in range(5):
            f = _random_filter(rng)
            got = O.expansion_seek(topics, f)
            target = f.split("/")

            def ge(a):
                for x, y in zip(a, target):
                    c = O.java_compare(x, y)
                    if c:
                        return c > 0
                return len(a) >= len(target)
            want = next((g for g in gen if ge(g)), None)
            assert got == want, (topics, f)


def test_expansion_equals_predicate_exhaustive():
    # the expansion set is exactly {filters over the batch vocabulary that match >= 1 topic}
    topics = ["a", "a/b", "/", "a/", "$s", "$s/a", "b//c"]
    gen = {tuple(lv) for lv, _ in O.expansion_list(topics)}
    vocab = ["", "a", "b", "c", "$s", "+", "#"]
    import itertools
    for n in range(1, 5):
        for combo in itertools.product(vocab, repeat=n):
            if "#" in combo[:-1]:
                continue
            f = "/".join(combo)
            want = any(O.topic_matches_filter(t, f) for t in topics)
            assert (combo in gen) == want, f


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-coproc-proto/src/test/.../TopicMatcherTest.java:55-71
# ------------------------------------------------------------------------------------------------


def test_topic_matcher_kat():
    m = O.topic_matches_filter
    assert m("/", "/") and m("/", "#") and m("/", "+/+") and m("/", "+/#") and m("/", "//#")
    assert not m("/", "+") and not m("/", "a")
    assert m("a", "a") and m("a", "a/#") and m("a", "+") and m("a", "#") and m("a", "+/#")
    assert not m("a", "a/+") and not m("a", "/a") and not m("a", "a/")
    assert m("a/b/c", "a/+/c") and m("a/b/c", "a/#") and m("a/b/c", "a/b/c/#") and m("a/b/c", "+/+/+")
    assert not m("a/b/c", "a/+") and not m("a/b/c", "a/b") and not m("a/b/c", "a/b/c/d")
    assert m("$sys/a", "$sys/#") and m("$sys/a", "$sys/+") and m("$sys/a", "$sys/a")
    assert not m("$sys/a", "#") and not m("$sys/a", "+/a") and not m("$sys/a", "+/#")
    assert m("$sys", "$sys/#") and not m("$sys", "+") and not m("$sys", "#")


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-worker/src/test/.../cache/TenantRouteMatcherTest.java:89-342
# ------------------------------------------------------------------------------------------------
TENANT_ID, OTHER_TENANT = "tenantA", "tenantB"
ALL_MODES = [O.MODE_REFERENCE, O.MODE_BRUTE, O.MODE_TRIE]


def normal(kv, tenant, tf, broker, receiver, deliverer, inc):
    url = O.receiver_url(broker, receiver, deliverer)
    kv.put(O.route_key(tenant, tf, url), O.incarnation_bytes(inc))
    return ("N", tenant, tf, url, inc)


def group(kv, tenant, tf, grp, members, ordered=False):
    full = ("$oshare/" if ordered else "$share/") + grp + "/" + tf
    kv.put(O.route_key(tenant, full), O.route_group(members))
    return ("G", tenant, full, tuple(sorted(members.items())))


def ids(matchings):
    return {O.matching_identity(m) for m in matchings}


@pytest.mark.parametrize("mode", ALL_MODES)
def test_match_all_returns_empty_when_no_tenant_data(mode):  # :89-111
    kv = O.KV()
    normal(kv, OTHER_TENANT, "sensors/+/temp", 1, "receiverX", "delivererX", 1)
    topics = ["sensors/device1/temp", "sensors/device1/humidity"]
    res, out = kv.match_all(TENANT_ID, topics, 10, 10, mode)
    assert set(res) == set(topics)
    assert all(v == [] for v in res.values())
    assert out.persistent_fanout.tolist() == [0, 0] and out.group_fanout.tolist() == [0, 0]
    assert out.events == []


@pytest.mark.parametrize("mode", ALL_MODES)
def test_match_all_across_multiple_topics(mode):  # :113-146
    kv = O.KV()
    temp = normal(kv, TENANT_ID, "sensors/+/temp", 1, "receiverA", "delivererA", 1)
    hum = normal(kv, TENANT_ID, "sensors/+/humidity", 1, "receiverB", "delivererB", 2)
    topics = ["sensors/device1/temp", "sensors/device1/humidity", "sensors/device2/temp"]
    res, out = kv.match_all(TENANT_ID, topics, 10, 10, mode)
    assert ids(res["sensors/device1/temp"]) == {temp}
    assert ids(res["sensors/device2/temp"]) == {temp}
    assert ids(res["sensors/device1/humidity"]) == {hum}
    assert out.persistent_fanout.tolist() == [1, 1, 1]
    assert out.group_fanout.tolist() == [0, 0, 0]
    assert out.events == []


@pytest.mark.parametrize("mode", ALL_MODES)
def test_reuse_cached_filter_matches(mode):  # :148-175
    kv = O.KV()
    first = normal(kv, TENANT_ID, "devices/+/status", 1, "receiverA", "delivererA", 1)
    second = normal(kv, TENANT_ID, "devices/+/status", 2, "receiverB", "delivererB", 1)
    topics = ["devices/a/status", "devices/b/status"]
    res, out = kv.match_all(TENANT_ID, topics, 5, 5, mode)
    for i, t in enumerate(topics):
        assert ids(res[t]) == {first, second}
        assert out.persistent_fanout[i] == 1  # only subBrokerId == 1 counts as persistent
        assert out.group_fanout[i] == 0
    assert out.events == []


@pytest.mark.parametrize("mode", ALL_MODES)
def test_match_all_with_shared_subscription(mode):  # :177-204
    kv = O.KV()
    members = {O.receiver_url(1, "receiverA", "delivererA"): 10, O.receiver_url(2, "receiverB", "delivererB"): 11}
    g = group(kv, TENANT_ID, "alerts/+/+/temperature", "groupAlpha", members)
    topics = ["alerts/site1/device1/temperature", "alerts/site1/device2/temperature"]
    res, out = kv.match_all(TENANT_ID, topics, 10, 10, mode)
    for i, t in enumerate(topics):
        assert ids(res[t]) == {g}
        assert out.persistent_fanout[i] == 0 and out.group_fanout[i] == 1
    assert out.events == []


@pytest.mark.parametrize("mode", ALL_MODES)
def test_skip_non_matching_routes_and_fallback_to_seek(mode):  # :206-236
    kv = O.KV()
    for i in range(21):
        normal(kv, TENANT_ID, "invalid/%d" % i, 1, "noise%d" % i, "deliverer%d" % i, i)
    valid = normal(kv, TENANT_ID, "metrics/+/cpu", 1, "receiverA", "delivererA", 1)
    res, out = kv.match_all(TENANT_ID, ["metrics/server1/cpu"], 10, 10, mode)
    assert ids(res["metrics/server1/cpu"]) == {valid}
    assert out.persistent_fanout.tolist() == [1] and out.group_fanout.tolist() == [0]
    if mode == O.MODE_REFERENCE:
        assert out.stats["seeks"] >= 2   # initial seek + fallback seek
        assert out.stats["nexts"] >= 21  # probed through the noise entries
    assert out.events == []


@pytest.mark.parametrize("mode", ALL_MODES)
def test_isolate_routes_by_tenant(mode):  # :238-268
    kv = O.KV()
    mine = normal(kv, TENANT_ID, "devices/+/signal", 1, "receiverA", "delivererA", 1)
    other = normal(kv, OTHER_TENANT, "devices/+/signal", 1, "receiverB", "delivererB", 1)
    res, _ = kv.match_all(TENANT_ID, ["devices/a/signal"], 10, 10, mode)
    assert ids(res["devices/a/signal"]) == {mine}
    res, _ = kv.match_all(OTHER_TENANT, ["devices/a/signal"], 10, 10, mode)
    assert ids(res["devices/a/signal"]) == {other}


@pytest.mark.parametrize("mode", ALL_MODES)
def test_trigger_persistent_fanout_throttling(mode):  # :270-301
    kv = O.KV()
    normal(kv, TENANT_ID, "alarms/+/critical", 1, "receiverA", "delivererA", 1)
    second = normal(kv, TENANT_ID, "alarms/+/critical", 1, "receiverB", "delivererB", 2)
    res, out = kv.match_all(TENANT_ID, ["alarms/device1/critical"], 1, 10, mode)
    assert out.persistent_fanout.tolist() == [1] and out.group_fanout.tolist() == [0]
    assert len(res["alarms/device1/critical"]) == 1
    assert len(out.events) == 1
    kind, topic_idx, rank, max_count = out.events[0]
    assert (kind, topic_idx, max_count) == (1, 0, 1)
    dropped = O.build_match_route(kv.key(rank), kv.value(rank))
    assert dropped["mqttTopicFilter"] == second[2]


@pytest.mark.parametrize("mode", ALL_MODES)
def test_trigger_group_fanout_throttling(mode):  # :303-342
    kv = O.KV()
    first = group(kv, TENANT_ID, "jobs/+/progress", "groupA", {O.receiver_url(1, "receiverA", "delivererA"): 1})
    group(kv, TENANT_ID, "jobs/+/progress", "groupB", {O.receiver_url(1, "receiverB", "delivererB"): 1})
    res, out = kv.match_all(TENANT_ID, ["jobs/job1/progress"], 10, 1, mode)
    assert out.group_fanout.tolist() == [1]
    assert sum(1 for m in res["jobs/job1/progress"] if m["type"] == "Group") == 1
    assert len(out.events) == 1
    kind, topic_idx, rank, max_count = out.events[0]
    assert (kind, topic_idx, max_count) == (2, 0, 1)
    # "second comes before first in lexicographical order by bucketing key" (:339-340)
    dropped = O.build_match_route(kv.key(rank), kv.value(rank))
    assert dropped["mqttTopicFilter"] == first[2]


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-worker/src/test/.../cache/MatchedRoutesTest.java:59-190 — the cap rules of the accumulator,
# expressed through matchAll (the mutable add/remove/adjust API of IMatchedRoutes stays in Java and is out of scope)
# ------------------------------------------------------------------------------------------------
MR_TOPIC = "sensors/temperature"


@pytest.mark.parametrize("mode", ALL_MODES)
def test_matched_routes_persistent_within_and_over_limit(mode):  # :59-96
    kv = O.KV()
    normal(kv, TENANT_ID, MR_TOPIC, 1, "receiverA", "delivererA", 1)
    res, out = kv.match_all(TENANT_ID, [MR_TOPIC], 2, 2, mode)
    assert len(res[MR_TOPIC]) == 1 and out.persistent_fanout.tolist() == [1] and not out.events
    normal(kv, TENANT_ID, MR_TOPIC, 1, "receiverB", "delivererB", 1)
    res, out = kv.match_all(TENANT_ID, [MR_TOPIC], 1, 2, mode)
    assert len(res[MR_TOPIC]) == 1 and out.persistent_fanout.tolist() == [1]
    assert [(e[0], e[1], e[3]) for e in out.events] == [(1, 0, 1)]       # PersistentFanoutThrottled, maxCount 1


@pytest.mark.parametrize("mode", ALL_MODES)
def test_matched_routes_non_persistent_is_not_capped(mode):  # :97-107
    kv = O.KV()
    for i in range(3):
        normal(kv, TENANT_ID, MR_TOPIC, 0, "receiver%d" % i, "deliverer", 1)     # subBrokerId 0: not persistent
    res, out = kv.match_all(TENANT_ID, [MR_TOPIC], 1, 2, mode)
    assert len(res[MR_TOPIC]) == 3 and out.persistent_fanout.tolist() == [0] and not out.events


@pytest.mark.parametrize("mode", ALL_MODES)
def test_matched_routes_group_within_and_over_limit(mode):  # :152-190
    kv = O.KV()
    group(kv, TENANT_ID, MR_TOPIC, "groupA", {O.receiver_url(1, "receiverA", "delivererA"): 1})
    res, out = kv.match_all(TENANT_ID, [MR_TOPIC], 2, 2, mode)
    assert len(res[MR_TOPIC]) == 1 and out.group_fanout.tolist() == [1] and not out.events
    group(kv, TENANT_ID, MR_TOPIC, "groupB", {O.receiver_url(1, "receiverB", "delivererB"): 1})
    res, out = kv.match_all(TENANT_ID, [MR_TOPIC], 2, 1, mode)
    assert len(res[MR_TOPIC]) == 1 and out.group_fanout.tolist() == [1]
    assert [(e[0], e[1], e[3]) for e in out.events] == [(2, 0, 1)]       # GroupFanoutThrottled, maxCount 1


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-worker/src/test/.../DistQoS0Test.java:82-340,450-561 — the integration tests' SUB sets and the
# fan-out count BatchDistReply reports for the published topic (a shared-subscription group counts once, whatever its
# member count; MqttBroker = 0, InboxService = 1, DistWorkerTest.java:130-131)
# ------------------------------------------------------------------------------------------------
INT_MAX = 2 ** 31 - 1


def _qos0_case(name):
    kv = O.KV()
    A, B = TENANT_ID, OTHER_TENANT
    if name == "case1":          # :83-92
        normal(kv, A, "TopicA/#", 0, "inbox1", "batch1", 1)
        return kv, "TopicB", 0
    if name == "case2":          # :95-149 (BMP and supplementary-plane characters, '#' below an empty first level)
        normal(kv, A, "/你好/hello/😄", 0, "inbox1", "batch1", 1)
        normal(kv, A, "/#", 0, "inbox1", "batch1", 1)
        normal(kv, A, "/#", 1, "inbox2", "batch2", 1)
        return kv, "/你好/hello/😄", 3
    if name == "case3":          # :152-193
        normal(kv, A, "/a/b/c", 0, "inbox1", "batch1", 1)
        normal(kv, A, "/a/b/c", 0, "inbox2", "batch1", 1)
        return kv, "/a/b/c", 2
    if name in ("case4", "case5"):   # :196-243 unordered share, :246-284 ordered share: two members, ONE group
        group(kv, A, "/a/b/c", "group", {O.receiver_url(0, "inbox1", "batch1"): 1, O.receiver_url(0, "inbox2", "batch2"): 1},
              ordered=name == "case5")
        return kv, "/a/b/c", 1
    if name == "case6":          # :287-306 normal + $share + $oshare of the same filter are three routes
        normal(kv, A, "/a/b/c", 0, "inbox6", "batch1", 1)
        group(kv, A, "/a/b/c", "group", {O.receiver_url(0, "inbox7", "batch2"): 1})
        group(kv, A, "/a/b/c", "group", {O.receiver_url(0, "inbox8", "batch3"): 1}, ordered=True)
        return kv, "/a/b/c", 3
    if name == "case7":          # :309-338 another tenant's '#' does not leak
        normal(kv, A, "/a/b/c", 0, "inbox1", "batch1", 1)
        normal(kv, B, "#", 0, "inbox1", "batch1", 1)
        return kv, "/a/b/c", 1
    if name == "wildcard_refresh":   # :450-515 final state: exact + '/#' + '$share/group/#' + '$oshare/group/#'
        normal(kv, A, "/a/b/c", 0, "inbox1", "batch1", 1)
        normal(kv, A, "/#", 0, "inbox2", "batch2", 1)
        group(kv, A, "#", "group", {O.receiver_url(0, "inbox3", "batch3"): 1})
        group(kv, A, "#", "group", {O.receiver_url(0, "inbox3", "batch3"): 1}, ordered=True)
        return kv, "/a/b/c", 4
    if name == "probe_and_seek":     # :518-528 more than 20 routes of "test" sit between the cursor and "test/#"
        normal(kv, A, "test/#", 0, "inbox", "batch1", 1)
        for i in range(21):
            normal(kv, A, "test", 0, "inbox%d" % i, "batch1", 1)
        return kv, "test/r1", 1
    if name == "ordered_share_groups":   # :531-562 two ordered groups on '#'
        group(kv, A, "#", "group1", {O.receiver_url(0, "inbox1", "batch1"): 1}, ordered=True)
        group(kv, A, "#", "group2", {O.receiver_url(0, "inbox1", "batch1"): 1}, ordered=True)
        return kv, "/a/b/c", 2
    raise KeyError(name)


# bifromq-dist/bifromq-dist-worker/src/test/.../FanoutThrottledTest.java:52-70,148-166,240-262 and BatchDistTest.java:78-109
@pytest.mark.parametrize("mode", ALL_MODES)
def test_fanout_throttled_and_batch_dist_counts(mode):
    kv = O.KV()
    for i in (1, 2, 3):          # persistent sessions (InboxService = 1): capped at MaxPersistentFanout = 2
        normal(kv, TENANT_ID, "/fanout/topic", 1, "inbox%d" % i, "batch%d" % i, 1)
    res, out = kv.match_all(TENANT_ID, ["/fanout/topic"], 2, INT_MAX, mode)
    assert len(res["/fanout/topic"]) == 2 and len(out.events) == 1
    kv = O.KV()
    for i in (1, 2, 3):          # three shared groups: capped at MaxGroupFanout = 2
        group(kv, TENANT_ID, "fanout/topic", "group%d" % i, {O.receiver_url(1, "inbox%d" % i, "batch%d" % i): 1})
    res, out = kv.match_all(TENANT_ID, ["fanout/topic"], INT_MAX, 2, mode)
    assert len(res["fanout/topic"]) == 2 and len(out.events) == 1
    kv = O.KV()
    for i in (1, 2, 3):          # transient sessions (MqttBroker = 0) are never capped
        normal(kv, TENANT_ID, "/fanout/topic2", 0, "inbox%d" % i, "batch%d" % i, 1)
    res, out = kv.match_all(TENANT_ID, ["/fanout/topic2"], 2, 2, mode)
    assert len(res["/fanout/topic2"]) == 3 and not out.events
    kv = O.KV()                  # BatchDistTest: one request, four topics
    normal(kv, TENANT_ID, "/a/1", 0, "inbox1", "batch1", 1)
    normal(kv, TENANT_ID, "/a/2", 0, "inbox1", "batch1", 1)
    normal(kv, TENANT_ID, "/a/2", 0, "inbox3", "batch1", 1)
    normal(kv, TENANT_ID, "/a/3", 1, "inbox2", "batch2", 1)
    normal(kv, TENANT_ID, "/a/4", 1, "inbox2", "batch2", 1)
    topics = ["/a/1", "/a/2", "/a/3", "/a/4"]
    res, out = kv.match_all(TENANT_ID, topics, INT_MAX, INT_MAX, mode)
    assert [len(res[t]) for t in topics] == [1, 2, 1, 1]


QOS0_CASES = ["case1", "case2", "case3", "case4", "case5", "case6", "case7", "wildcard_refresh", "probe_and_seek",
              "ordered_share_groups"]


@pytest.mark.parametrize("mode", ALL_MODES)
@pytest.mark.parametrize("name", QOS0_CASES)
def test_dist_qos0_fanout_counts(name, mode):
    kv, topic, fanout = _qos0_case(name)
    res, out = kv.match_all(TENANT_ID, [topic], INT_MAX, INT_MAX, mode)
    assert set(res) == {topic}
    assert len(res[topic]) == fanout
    assert not out.events


# ------------------------------------------------------------------------------------------------
# bifromq-dist/bifromq-dist-worker/src/test/.../KeyLayoutTest.java:47-78 — key byte order == iterator order
# ------------------------------------------------------------------------------------------------


def test_key_layout_order_equals_iterator_order():
    rng = random.Random(11)
    topics = ["$", "b", "a/b", "b/c", "a/b/c", "b/c/d"]
    generated = ["/".join(lv) for lv, _ in O.expansion_list(topics)]
    kv = O.KV()
    for tf in generated:
        for _ in range(10):
            url = O.receiver_url(rng.randint(-2 ** 31, 2 ** 31 - 1), "%032x" % rng.getrandbits(128), "%032x" % rng.getrandbits(128))
            kv.put(O.route_key("t", tf, url), O.incarnation_bytes(rng.getrandbits(40)))
    parsed = []
    for k, v in kv.items():
        f = O.build_match_route(k, v)["mqttTopicFilter"]
        if not parsed or parsed[-1] != f:
            parsed.append(f)
    assert parsed == generated


# ------------------------------------------------------------------------------------------------
# Inverse match: DWT/TopicIndexTest.java:41-73,136-139, RST/index/RetainTopicIndexTest.java:42-75,112-117,
# RST/RetainMatchTest.java:38-111
# ------------------------------------------------------------------------------------------------
INDEXED = ["/", "/a", "/b", "a", "a/", "a/b", "a/b/c", "$a", "$a/", "$a/b"]
INVERSE_CASES = {
    "/": ["/"], "/a": ["/a"], "/b": ["/b"], "a": ["a"], "a/": ["a/"], "a/b": ["a/b"], "a/b/c": ["a/b/c"],
    "$a": ["$a"], "$a/": ["$a/"], "$a/b": ["$a/b"], "": [], "fakeTopic": [],
    "#": ["/", "/a", "/b", "a", "a/", "a/b", "a/b/c"], "+": ["a"],
    "+/#": ["/", "/a", "/b", "a", "a/", "a/b", "a/b/c"], "+/+": ["/", "/a", "/b", "a/", "a/b"],
    "/+": ["/", "/a", "/b"], "/#": ["/", "/a", "/b"], "a/+": ["a/", "a/b"], "a/#": ["a", "a/", "a/b", "a/b/c"],
    "$a/+": ["$a/", "$a/b"], "$a/+/#": ["$a/", "$a/b"], "$a/#": ["$a", "$a/", "$a/b"],
}
TOPIC_INDEX_ONLY = {"+/+/#": ["/", "/a", "/b", "a/", "a/b", "a/b/c"], "/+/#": ["/", "/a", "/b"]}


@pytest.mark.parametrize("tenant", [None, "tenantA"])
def test_inverse_match_vectors(tenant):
    idx = O.TopicLevelIndex()
    for i, t in enumerate(INDEXED):
        idx.add(t, i, tenant)
    cases = dict(INVERSE_CASES)
    cases.update(TOPIC_INDEX_ONLY)
    for f, want in cases.items():
        got = sorted(INDEXED[i] for i in idx.match(f, tenant))
        assert got == sorted(want), f
    if tenant is not None:
        assert idx.match("#", "tenantB") == []
        assert sorted(INDEXED[i] for i in idx.find_all()) == sorted(INDEXED)   # RetainTopicIndexTest.testFindAll
    else:
        for i, t in enumerate(INDEXED):  # TopicIndexTest.testGet
            assert idx.get(t) == [i]


@pytest.mark.parametrize("tenant", [None, "tenantA"])
def test_inverse_remove_and_edge(tenant):  # TopicIndexTest.testRemove/testEdgeCases, RetainTopicIndexTest.testRemove
    idx = O.TopicLevelIndex()
    for i, t in enumerate(INDEXED):
        idx.add(t, i, tenant)
    for i, t in enumerate(INDEXED):
        idx.remove(t, i, tenant)
        assert idx.match(t, tenant) == []
    assert idx.match("#", tenant) == []
    idx2 = O.TopicLevelIndex()
    idx2.add("/", 0, tenant)
    idx2.add("/", 0, tenant)
    assert idx2.match("#", tenant) == [0]


def test_inverse_multi_value():  # TopicIndexTest.testMultiValue :116-132
    idx = O.TopicLevelIndex()
    idx.add("a", 1)
    idx.add("a", 1)
    idx.add("a", 2)
    assert idx.get("a") == [1, 2]
    idx.remove("a", 3)
    assert idx.get("a") == [1, 2]
    idx.remove("a", 2)
    assert idx.get("a") == [1]
    idx.remove("a", 1)
    assert idx.get("a") == []


def test_retain_match_vectors():  # RST/RetainMatchTest.java:38-111
    msgs = ["/a/b/c", "/a/b/", "/c/", "a"]
    idx = O.TopicLevelIndex()
    for i, t in enumerate(msgs):
        idx.add(t, i, "tenantA")
    cases = {"#": [0, 1, 2, 3], "+": [3], "+/#": [0, 1, 2, 3], "+/+/#": [0, 1, 2], "+/+/+": [2], "/#": [0, 1, 2],
             "/c/#": [2], "/a/+": [], "/a/#": [0, 1], "/a/+/+": [0, 1], "/a/+/#": [0, 1], "/+/b/": [1],
             "/+/b/#": [0, 1], "/a/b/c/#": [0], "/a/b/#": [0, 1]}
    for f, want in cases.items():
        assert idx.match(f, "tenantA") == want, f


# ------------------------------------------------------------------------------------------------
# Cross-check of the three forward matchers on random workloads (incl. '$' topics, empty levels, shared
# subscriptions, tight caps): literal reference algorithm == brute-force predicate == trie walk.
# ------------------------------------------------------------------------------------------------


def _mk_workload(rng, n_filters, n_topics, vocab, depth, empty_levels=False):
    def level(i, allow_empty):
        r = rng.random()
        if r < 0.08 and allow_empty:
            return ""
        if r < 0.15 and i == 0:
            return "$" + rng.choice(vocab)
        return rng.choice(vocab)

    def topic():
        return "/".join(level(i, empty_levels) for i in range(rng.randint(1, depth)))

    def filt():
        n = rng.randint(1, depth)
        lv = []
        for i in range(n):
            r = rng.random()
            if r < 0.25:
                lv.append("+")
            elif r < 0.35 and i == n - 1:
                lv.append("#")
            else:
                lv.append(level(i, empty_levels))
        return "/".join(lv)
    kv = O.KV()
    tenants = ["tA", "tB", "t"]
    for _ in range(n_filters):
        tenant = rng.choice(tenants)
        f = filt()
        r = rng.random()
        if r < 0.15:
            members = {O.receiver_url(rng.choice([0, 1]), "m%d" % rng.randint(0, 5), "d"): rng.randint(1, 9)
                       for _ in range(rng.randint(1, 3))}
            full = rng.choice(["$share/", "$oshare/"]) + "g%d" % rng.randint(0, 3) + "/" + f
            kv.put(O.route_key(tenant, full), O.route_group(members))
        else:
            for _ in range(rng.choice([1, 1, 1, 2, 5])):
                url = O.receiver_url(rng.choice([0, 1, 1, 2]), "r%d" % rng.randint(0, 400), "d%d" % rng.randint(0, 3))
                kv.put(O.route_key(tenant, f, url), O.incarnation_bytes(rng.randint(0, 99)))
    topics = [topic() for _ in range(n_topics)]
    tt = np.array([rng.randrange(len(tenants)) for _ in topics], dtype=np.int32)
    return kv, tenants, topics, tt


@pytest.mark.parametrize("seed,caps", [(1, (2 ** 31 - 1, 100)), (2, (2, 1)), (3, (0, 0)), (4, (4, 4))])
def test_three_matchers_agree_random(seed, caps):
    # no empty levels in topics or filters: the literal reference algorithm, the brute-force predicate and the
    # trie walk must agree exactly, caps and throttle events included. (With empty levels the reference's
    # probe/seek loop can skip routes or even seek backwards forever — see the two tests below.)
    rng = random.Random(seed)
    kv, tenants, topics, tt = _mk_workload(rng, 400, 120, ["a", "b", "c", "dd", "e1"], 4)
    outs = [kv.match_batch(tenants, topics, tt, caps[0], caps[1], mode) for mode in ALL_MODES]
    ref = outs[0]
    assert ref.stats["backward_seeks"] == 0
    for o in outs[1:]:
        assert o.route_sets() == ref.route_sets()
        assert o.persistent_fanout.tolist() == ref.persistent_fanout.tolist()
        assert o.group_fanout.tolist() == ref.group_fanout.tolist()
        assert o.events == ref.events
    assert sum(len(r) for r in ref.route_sets()) > 0
    # production shape (one matchAll per topic) gives the same answer
    single = kv.match_batch(tenants, topics, tt, caps[0], caps[1], O.MODE_REFERENCE, singleton=True, nthreads=4)
    assert single.route_sets() == ref.route_sets() and single.events == ref.events


@pytest.mark.parametrize("seed", [5, 6])
def test_semantic_matchers_agree_with_empty_filter_levels(seed):
    # topics and filters WITH empty levels: brute force == trie walk; the literal algorithm may only lose
    # routes (see test_reference_probe_seek_quirk_with_mid_empty_levels)
    rng = random.Random(seed)
    kv, tenants, topics, tt = _mk_workload(rng, 400, 120, ["a", "b", "c"], 4, empty_levels=True)
    brute = kv.match_batch(tenants, topics, tt, mode=O.MODE_BRUTE)
    trie = kv.match_batch(tenants, topics, tt, mode=O.MODE_TRIE)
    ref = kv.match_batch(tenants, topics, tt, mode=O.MODE_REFERENCE)
    assert brute.route_sets() == trie.route_sets()
    for a, b in zip(ref.route_sets(), brute.route_sets()):
        assert set(a) <= set(b)


def test_reference_probe_seek_quirk_with_mid_empty_levels():
    """Documented divergence (DESIGN.md "Known reference quirk"): when a filter contains an EMPTY level
    after a prefix F (e.g. [a,"",b]) its keys sort INSIDE F's bucket range, and after 20 failed probes the
    reference seeks past the rest of F's routes (TenantRouteMatcher.java:127-136), silently dropping matching
    routes. The semantic matchers (brute / trie / the CUDA product) return them."""
    kv = O.KV()
    # routes of filter "a" spread over many buckets, > 20 routes of the non-matching filter "a//b" in between
    for i in range(200):
        url = O.receiver_url(0, "r%d" % i, "d")
        kv.put(O.route_key("t", "a", url), O.incarnation_bytes(1))
    for i in range(40):
        url = O.receiver_url(0, "x%d" % i, "d")
        kv.put(O.route_key("t", "a//b", url), O.incarnation_bytes(1))
    ref = kv.match_batch(["t"], ["a"], None, mode=O.MODE_REFERENCE)
    brute = kv.match_batch(["t"], ["a"], None, mode=O.MODE_BRUTE)
    trie = kv.match_batch(["t"], ["a"], None, mode=O.MODE_TRIE)
    assert brute.route_sets() == trie.route_sets()
    assert len(brute.routes(0)) == 200
    assert set(ref.routes(0).tolist()) <= set(brute.routes(0).tolist())
    # whether the literal algorithm loses routes depends on bucket bytes; with this fixture it does
    assert len(ref.routes(0)) < 200


def test_reference_backward_seek_with_trailing_empty_topic_level():
    """Second documented reference quirk: for topic "dd/" the expansion successor of the stored filter "+" is
    ["+", ""], whose start key `2b 00 00 00` sorts BEFORE every route key of "+" (`2b 00 00 <bucket>`), so
    after 20 probes TenantRouteMatcher.java:134-135 seeks backwards and never terminates. The oracle's literal
    restatement counts and breaks such seeks; the semantic matchers are unaffected."""
    kv = O.KV()
    for i in range(30):
        kv.put(O.route_key("t", "+", O.receiver_url(0, "r%d" % i, "d")), O.incarnation_bytes(1))
    kv.put(O.route_key("t", "dd/", O.receiver_url(0, "x", "d")), O.incarnation_bytes(1))
    ref = kv.match_batch(["t"], ["dd/"], None, mode=O.MODE_REFERENCE)
    assert ref.stats["backward_seeks"] > 0
    brute = kv.match_batch(["t"], ["dd/"], None, mode=O.MODE_BRUTE)
    trie = kv.match_batch(["t"], ["dd/"], None, mode=O.MODE_TRIE)
    assert brute.route_sets() == trie.route_sets() == ref.route_sets()
    assert len(brute.routes(0)) == 1


# ------------------------------------------------------------------ retain store schema
# bifromq-retain/bifromq-retain-store-schema/src/test/java/org/apache/bifromq/retain/store/schema/KVSchemaUtilTest.java:43-74,
# LevelHashTest.java:30-41. The reference's vectors are structural (prefix = tenantNS ++ levels ++ LevelHash.hash(prefix levels));
# LevelHash itself is FNV-1a 32 (offset 0x811c9dc5, prime 0x01000193) over UTF-16 code units, low byte: the published FNV-1a test
# vectors "" -> 0x811c9dc5 and "a" -> 0xe40c292c pin its two constants.
def _levels_u16(n):
    return bytes([(n >> 8) & 0xFF, n & 0xFF])


def test_level_hash_known_answers():
    assert O.level_hash_byte("") == 0xC5 and O.level_hash_byte("a") == 0x2C
    assert O.level_hash_byte("foobar") == 0xBF9CF968 & 0xFF          # FNV-1a 32 published vector
    assert len({O.level_hash_byte(x) for x in ["a", "b", "c"]}) == 3


def test_retain_message_key_prefix_vectors():   # KVSchemaUtilTest.java:43-74
    tenant = "tenantA"
    ns = O.tenant_begin_key(tenant)

    def H(*levels):
        return bytes(O.level_hash_byte(l) for l in levels)
    cases = [("#", 0, H()), ("/#", 1, H("")), ("+", 1, H()), ("+/#", 1, H()), ("a/#", 1, H("a")), ("/a", 2, H("", "a")),
             ("a/+", 2, H("a")), ("a/b", 2, H("a", "b")), ("/a/#", 2, H("", "a")), ("/a/+", 3, H("", "a")),
             ("/a/+/+", 4, H("", "a")), ("/+/b/", 4, H("")), ("/+/b/+/", 5, H(""))]
    for tf, levels, hashes in cases:
        assert O.retain_key_prefix(tenant, tf) == ns + _levels_u16(levels) + hashes, tf


def test_retain_message_key_layout_and_tenant_parse():   # KVSchemaUtilTest.java:96-104 + KVSchemaUtil.java:44-50
    k = O.retain_key("tenantA", "/a/b/c")
    ns = O.tenant_begin_key("tenantA")
    assert k.startswith(ns) and k[len(ns):len(ns) + 2] == _levels_u16(4)
    assert k[len(ns) + 2:len(ns) + 6] == bytes(O.level_hash_byte(l) for l in ["", "a", "b", "c"])
    assert k[len(ns) + 6:] == b"\x00a\x00b\x00c"               # escape(topic): '/' -> NUL
    # a retain key starts with the prefix of every filter that can match its topic by a plain prefix scan
    for tf in ["/a/b/c", "/a/b/+", "/a/+/+", "/+/b/c"]:
        assert k.startswith(O.retain_key_prefix("tenantA", tf))


# ------------------------------------------------------------------ dist-server range pruning
def test_tenant_range_lookup_cache_vectors():
    """TenantRangeLookupCacheTest.java:109-330 through the oracle's literal restatement of TenantRangeLookupCache.lookup"""
    from golden.range_lookup_vectors import T, VECTORS
    for topic, cands, want in VECTORS:
        assert O.range_lookup(T, topic, cands) == want, (topic, cands)
