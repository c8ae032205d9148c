"""The host half of the forward delta commit for tenants with wide nodes, without a GPU. bfq_host_build_stats slot 19 simulates
on the full image what bfq_index_commit's delta path does to every tenant that has wide edges (children in the shared tag
table): its tag slots are freed, it is rebuilt into a fresh region and its wide edges are placed again (root-level ones with the
same keys: the tenant keeps its ordinal). Then every node of the rebuilt tenant must be found again from its parent by the
kernels' lookup rules. The slot must count every wide tenant, on shapes where the wide node sits at the root, below a '+' and
below an exact parent, next to perfect-hashed nodes of 300 children, and on random, adversarial and generated key sets.

Which tenants are wide is decided here from the filters alone: a node with at least 1100 exact children cannot get a
perfect-hash array (2^16 slots hold about 1000 children), one with at most 400 gets one (short of a 32-bit hash collision
among its children, which these fixed key sets do not have)."""
import random

import numpy as np

from test_host_cpu import _route_blobs

WIDE_MIN, NARROW_MAX = 1100, 400


def host_stats(pairs):
    from bifromq_b200 import _native as N
    pairs = sorted(pairs)
    k, ko, v, vo = _route_blobs(pairs)
    st = np.zeros(20, np.int64)
    rc = N.lib.bfq_host_build_stats(k.ctypes.data, ko.ctypes.data, v.ctypes.data, vo.ctypes.data, len(pairs), st.ctypes.data, 20)
    assert rc == 0, N.lib.bfq_last_error()
    return st


def inner_filter(tf):
    for pfx in ("$share/", "$oshare/"):
        if tf.startswith(pfx):
            return tf.split("/", 2)[2]
    return tf


def wide_tenants(pairs):
    """tenant -> its largest exact fan-out, counted on the chunked trie the builder makes (levels longer than 24 bytes are a
    chain of 24-byte chunks; '+' is not an exact child and a trailing '#' is inlined into its parent)"""
    from bifromq_b200 import schema
    children = {}
    for k, v in pairs:
        m = schema.build_match_route(k, v)
        levels = inner_filter(m.mqtt_topic_filter).split("/")
        if levels[-1] == "#":
            levels = levels[:-1]
        node = (m.tenant_id,)
        for lv in levels:
            if lv == "+":
                node = node + ("+",)
                continue
            b = lv.encode()
            chunks = [b[i:i + 24] for i in range(0, len(b), 24)] or [b""]
            for j, c in enumerate(chunks):
                edge = (c, j, j == len(chunks) - 1)
                children.setdefault(node, set()).add(edge)
                node = node + (edge,)
    fan = {}
    for node, cs in children.items():
        fan[node[0]] = max(fan.get(node[0], 0), len(cs))
    assert not [t for t, c in fan.items() if NARROW_MAX < c < WIDE_MIN], "a fan-out between the two kinds: ambiguous"
    return sorted(t for t, c in fan.items() if c >= WIDE_MIN)


# the tag-table model the GPU tests use to predict commit paths lives in tests/trie_hash.py
from trie_hash import ROOT_BASE, TagModel, level_home_block as home_block  # noqa: E402,F401


def route(tenant, tf, i, broker=0):
    from bifromq_b200 import schema
    return (schema.route_key(tenant, tf, schema.receiver_url(broker, "r%d" % i, "d")), schema.incarnation_bytes(1))


def shapes(n_wide):
    """wide at the root, below a '+', below an exact parent; 300 children (perfect hash) in every tenant"""
    pairs = []
    for i in range(n_wide):
        pairs.append(route("root", "dev%05d/state" % i, i))
        pairs.append(route("plus", "+/c%05d" % i, i, 1))
        pairs.append(route("exact", "site/w/c%05d/x" % i, i))
    for t in ("root", "plus", "exact", "narrow"):
        for i in range(300):
            pairs.append(route(t, "p/c%04d" % i, i))
        pairs.append(route(t, "+/state", 0, 1))
        pairs.append(route(t, "#", 1))
    return pairs


def check(pairs):
    pairs = sorted(dict(pairs).items())
    wide = wide_tenants(pairs)
    st = host_stats(pairs)
    assert st[19] == len(wide), (st[19], wide)
    return wide


def test_wide_node_shapes():
    for n in (1500, 3000):
        assert check(shapes(n)) == ["exact", "plus", "root"]
    # the same nodes with 300 children: perfect-hashed, no tenant is wide
    assert check(shapes(300)) == []


def test_node_crossing_between_the_kinds():
    """one node at 300 children (perfect hash), then at 1500 (tag table), next to a tenant that stays wide"""
    base = [route("other", "o%05d" % i, i) for i in range(2000)]
    for n, want in ((300, ["other"]), (1500, ["other", "t"]), (300, ["other"])):
        pairs = base + [route("t", "a/b/n%05d" % i, i) for i in range(n)] + [route("t", "a/+/x", 0)]
        assert check(pairs) == want


def test_random_key_sets():
    rng = random.Random(5)
    vocab = ["a", "b", "c", "dd", "e1", "", "$x"]
    for rnd in range(3):
        pairs = []
        for t in ("tA", "tB", "tC"):
            for _ in range(400):
                lv = [rng.choice(vocab + ["+"]) for _ in range(rng.randint(1, 5))]
                if lv[0] == "":
                    lv[0] = "a"
                if rng.random() < 0.2:
                    lv.append("#")
                tf = "/".join(lv)
                if rng.random() < 0.15:
                    tf = "$share/g%d/%s" % (rng.randint(0, 2), tf)
                    from bifromq_b200 import schema
                    pairs.append((schema.route_key(t, tf), schema.route_group_bytes({schema.receiver_url(0, "m", "d"): 1})))
                else:
                    pairs.append(route(t, tf, rng.randint(0, 50), rng.randint(0, 2)))
        # a wide node somewhere in two of the tenants, at a random depth
        for t in ("tA", "tC")[:1 + rnd % 2]:
            prefix = "/".join(rng.choice(["a", "b", "+"]) for _ in range(rng.randint(0, 2)))
            for i in range(1200 + 400 * rnd):
                tf = (prefix + "/" if prefix else "") + "w%05d" % rng.randint(0, 10 ** 5)
                pairs.append(route(t, tf + rng.choice(["", "/s", "/#"]), i))
        check(pairs)


def test_adversarial_key_sets():
    """wide nodes whose children are levels longer than one 24-byte token (continuation chunks share their first chunk),
    empty and control-byte levels, '$' levels, and a wide node whose children are wide too"""
    pairs = []
    long = "L" * 24
    for i in range(1500):
        pairs.append(route("long", long + "%05d/x" % i, i))          # 1500 chunk chains below one continuation node
        pairs.append(route("long", "k%05d" % i + long + "/y", i))     # 1500 distinct first chunks at the root
        pairs.append(route("ctl", "\x01%05d/\x02" % i, i))
        pairs.append(route("ctl", "/" + "e%05d" % i, i))               # below the empty first level
        pairs.append(route("dollar", "$sys/%05d" % i, i))
    for i in range(1200):
        for j in range(2):
            pairs.append(route("nested", "g%05d/h%d" % (i, j), i * 2 + j))
    for i in range(1200):
        pairs.append(route("nested", "g00000/m%05d" % i, i))
    assert check(pairs) == ["ctl", "dollar", "long", "nested"]


def test_generated_key_sets_plus_iot_tenants():
    """C3 and C4 at 5 % size, each with two IoT tenants (one subscriber per device at dev/<id>/state, plus dev/+/state and
    dev/#) appended behind their tenants"""
    from bifromq_b200 import workload
    for config in ("C3", "C4"):
        w = workload.Workload(config, scale=0.05)
        keys, koff, vals, voff = w.keys.tobytes(), w.key_off, w.vals.tobytes(), w.val_off
        pairs = [(keys[koff[i]:koff[i + 1]], vals[voff[i]:voff[i + 1]]) for i in range(w.n_routes)]
        for name, n in (("iot-tenant-with-a-long-name-%s-1" % config, 5000), ("iot-tenant-with-a-long-name-%s-2" % config, 1500)):
            for i in range(n):
                pairs.append(route(name, "dev/%06d/state" % i, i, i % 3))
            pairs.append(route(name, "dev/+/state", 0, 1))
            pairs.append(route(name, "dev/#", 1, 1))
        wide = check(pairs)
        assert len(wide) >= 2


def test_tag_table_model_agrees_with_the_builder():
    """the model above against the builder's own count of overflowed blocks (host stats slot 8), on loads from 0.5 to the
    3/4 bound: the GPU tests rely on it to place commits on either side of the delta rules' bounds"""
    for n, extra in ((1500, 0), (1500, 750), (3000, 1500), (1200, 200)):
        names = ["d%05d" % i for i in range(n)] + ["o%05d" % i for i in range(extra)]
        pairs = [route("w", nm, i) for i, nm in enumerate(names)] + [route("s1", "a/b", 0), route("s2", "+/x", 1)]
        st = host_stats(pairs)
        model = TagModel(n + extra)
        assert st[8] == model.place(names, 0), (n, extra)
        assert st[19] == 1
