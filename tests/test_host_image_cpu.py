"""The host half of the product against the oracle WITHOUT a GPU: tests/native/image_walk_harness.cc (test infrastructure, never
linked into the product) stages raw route KV the way bfq_index_load / bfq_index_apply do, builds the flat index image with the
product's own builder (bifromq_b200/csrc/index_builder.cc) and walks publish topics through that image on the CPU the way the
kernels look things up. Every topic's matched route ranks must equal the oracle's (no caps here: those are the caps kernel's,
covered by the -m gpu tests). What this pins on the CPU: key decoding, per-tenant staging and delta merge, the sorted-order trie
construction, single-child fingerprints / perfect-hash child arrays / the global tag table, '+' slots, inlined '#' ranges,
continuation chunks of long levels, the segment table of split rank runs, the '$' rule, rank = position in KV order."""
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

import oracle_lib as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MAX = 2 ** 31 - 1


@pytest.fixture(scope="module")
def walker(tmp_path_factory):
    csrc = os.path.join(ROOT, "bifromq_b200", "csrc")
    exe = str(tmp_path_factory.mktemp("image_walk") / "image_walk")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I" + csrc, os.path.join(ROOT, "tests", "native", "image_walk_harness.cc"),
                           os.path.join(csrc, "index_builder.cc"), os.path.join(csrc, "codec.cc"), "-lpthread", "-o", exe])
    return exe


def _blob(items):
    items = [x if isinstance(x, bytes) else x.encode("utf-8") for x in items]
    off = np.zeros(len(items) + 1, np.int64)
    off[1:] = np.cumsum([len(x) for x in items])
    return b"".join(items), off


PIECES = {"BFQ_INSERT_PARALLEL_MIN": "2", "BFQ_INSERT_THREADS": "6"}   # force the several-thread insertion of large tenants


def walk(walker, tmp, pairs, tenants, topics, tt, deltas=(), env=None, dump=False):
    """pairs: the KV handed to load (sorted); deltas: [("put", key, value) | ("del", key)] staged on top, like bfq_index_apply;
    dump: the harness also writes <tmp>/dump.txt (node ids and kinds along every topic, every tag block)"""
    os.makedirs(tmp, exist_ok=True)
    kb, ko = _blob([k for k, _ in pairs])
    vb, vo = _blob([v for _, v in pairs])
    tb, to = _blob(tenants)
    pb, po = _blob(topics)
    for name, data in (("keys", kb), ("vals", vb), ("tenants", tb), ("topics", pb)):
        open(os.path.join(tmp, name + ".bin"), "wb").write(data)
    for name, arr in (("koff", ko), ("voff", vo), ("tenant_off", to), ("topic_off", po)):
        arr.astype(np.int64).tofile(os.path.join(tmp, name + ".bin"))
    np.asarray(tt, np.int32).tofile(os.path.join(tmp, "topic_tenant.bin"))
    with open(os.path.join(tmp, "deltas.bin"), "wb") as f:
        for d in deltas:
            k = d[1]
            v = d[2] if d[0] == "put" else b""
            f.write(struct.pack("<BI", 1 if d[0] == "put" else 2, len(k)) + k + struct.pack("<I", len(v)) + v)
    r = subprocess.run([walker, tmp] + (["dump"] if dump else []), capture_output=True, text=True, timeout=300,
                       env=dict(os.environ, **(env or {})))
    assert r.returncode == 0, r.stdout + r.stderr
    return np.fromfile(os.path.join(tmp, "out_off.bin"), np.int64), np.fromfile(os.path.join(tmp, "out_ranks.bin"), np.int64), r.stdout


def oracle(pairs, tenants, topics, tt):
    kv = O.KV()
    for k, v in pairs:
        kv.put(k, v)
    kv.freeze()
    want = kv.match_batch(tenants, topics, np.asarray(tt, np.int32), INT_MAX, INT_MAX, O.MODE_TRIE)
    brute = kv.match_batch(tenants, topics, np.asarray(tt, np.int32), INT_MAX, INT_MAX, O.MODE_BRUTE)
    assert brute.route_sets() == want.route_sets()
    return want


def random_pairs(schema, rng, n_filters, vocab, depth):
    def level(i):
        r = rng.random()
        if r < 0.08:
            return ""
        if r < 0.15 and i == 0:
            return "$" + rng.choice(vocab)
        return rng.choice(vocab)

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
                lv.append(level(i))
        return "/".join(lv)
    tenants = ["tA", "tB", "t"]
    pairs = {}
    for _ in range(n_filters):
        tenant = rng.choice(tenants)
        f = filt()
        if rng.random() < 0.15:
            members = {schema.receiver_url(rng.choice([0, 1]), "m%d" % rng.randint(0, 5), "d"): rng.randint(1, 9) for _ in range(rng.randint(1, 3))}
            pairs[schema.route_key(tenant, rng.choice(["$share/", "$oshare/"]) + "g%d" % rng.randint(0, 3) + "/" + f)] = schema.route_group_bytes(members)
        else:
            for _ in range(rng.choice([1, 1, 1, 2, 5])):
                url = schema.receiver_url(rng.choice([0, 1, 1, 2]), "r%d" % rng.randint(0, 400), "d%d" % rng.randint(0, 3))
                pairs[schema.route_key(tenant, f, url)] = schema.incarnation_bytes(rng.randint(0, 99))
    topics = ["/".join(level(i) for i in range(rng.randint(1, depth))) for _ in range(400)]
    topics += ["", "/", "//", "$sys", "$sys/a", "a", "a/", "/a"]
    tt = [rng.randrange(len(tenants)) for _ in topics]
    return pairs, tenants, topics, tt


@pytest.mark.parametrize("seed,env", [(1, None), (2, None), (3, None), (4, PIECES), (5, PIECES)])
def test_image_walk_random_small_vocab_equals_oracle(walker, tmp_path, seed, env):
    from bifromq_b200 import schema
    rng = random.Random(seed)
    pairs, tenants, topics, tt = random_pairs(schema, rng, 700, ["a", "b", "c", "dd", "e1"], 5)
    pairs = sorted(pairs.items())
    # a tenant the index has never seen, mixed into the batch
    tenants = tenants + ["nobody"]
    tt = [3 if i % 11 == 0 else t for i, t in enumerate(tt)]
    off, ranks, _ = walk(walker, str(tmp_path), pairs, tenants, topics, tt, env=env)
    want = oracle(pairs, tenants, topics, tt)
    assert off.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    assert len(ranks) > 1000


def test_image_walk_wide_fanouts_long_levels_and_split_runs(walker, tmp_path):
    """every child-array kind (1, 3, 17, 300 perfect-hashed; 1500 / 2500 children: the global tag table), levels longer than one
    24-byte token (shared chunks), and filters whose routes are split rank runs (the empty-level interleaving of DESIGN.md §2)"""
    from bifromq_b200 import schema
    pairs = {}
    widths = {"w1": 1, "w3": 3, "w17": 17, "w300": 300, "w1500": 1500}
    for name, n in widths.items():
        for i in range(n):
            pairs[schema.route_key("t", "%s/c%04d" % (name, i), schema.receiver_url(i % 2, "r%s%d" % (name, i), "d"))] = schema.incarnation_bytes(1)
        pairs[schema.route_key("t", "%s/+" % name, schema.receiver_url(0, "p" + name, "d"))] = schema.incarnation_bytes(1)
        pairs[schema.route_key("t", "%s/#" % name, schema.receiver_url(1, "h" + name, "d"))] = schema.incarnation_bytes(1)
    for i in range(2500):
        pairs[schema.route_key("t2", "dev%05d/state" % i, schema.receiver_url(0, "s%d" % i, "d"))] = schema.incarnation_bytes(1)
    long_a, long_b = "L" * 24 + "p", "L" * 24 + "q"
    for lv in (long_a, long_b, "L" * 24, "L" * 50 + "x", "L" * 50 + "y"):
        pairs[schema.route_key("t", "long/" + lv + "/end", schema.receiver_url(0, "l" + lv[-1], "d"))] = schema.incarnation_bytes(2)
    # one filter, many receivers -> bucket bytes all over the range, and the same prefix continued by an empty level: F's routes
    # interleave with F + [""]'s in KV order
    for i in range(300):
        pairs[schema.route_key("t", "il/x", schema.receiver_url(0, "q%d" % i, "d"))] = schema.incarnation_bytes(1)
        pairs[schema.route_key("t", "il/x/", schema.receiver_url(0, "e%d" % i, "d"))] = schema.incarnation_bytes(1)
        pairs[schema.route_key("t", "il/x//y", schema.receiver_url(0, "f%d" % i, "d"))] = schema.incarnation_bytes(1)
    pairs = sorted(pairs.items())
    tenants = ["t", "t2"]
    topics = ["w1/c0000", "w3/c0002", "w3/nope", "w17/c0016", "w300/c0299", "w300/c0300", "w1500/c1499", "w1500/zzz", "w1500",
              "long/" + long_a + "/end", "long/" + long_b + "/end", "long/" + "L" * 24 + "/end", "long/" + "L" * 50 + "x/end",
              "long/" + "L" * 50 + "z/end", "long/" + "L" * 23 + "/end", "il/x", "il/x/", "il/x//y", "il/x//", "il"]
    tt = [0] * len(topics)
    topics += ["dev00000/state", "dev02499/state", "dev02500/state", "dev00017"]
    tt += [1, 1, 1, 1]
    off, ranks, log = walk(walker, str(tmp_path), pairs, tenants, topics, tt, env=PIECES)
    want = oracle(pairs, tenants, topics, tt)
    assert off.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    assert int(log.split(" tag blocks")[0].split()[-1]) > 64          # the global tag table was really used
    assert (np.diff(off)[15:18] >= 300).all()                          # the interleaved filters each return all their routes


def test_image_walk_after_staged_deltas_equals_oracle_of_the_final_kv(walker, tmp_path):
    """bfq_index_load + bfq_index_apply + commit on the host side: upserts, overwrites, deletes, a tenant that vanishes, one that
    appears — the image built from the merged staging area answers like the oracle fed the final KV"""
    from bifromq_b200 import schema
    rng = random.Random(77)
    pairs, tenants, topics, tt = random_pairs(schema, rng, 500, ["a", "b", "c", "dd"], 4)
    more, _, _, _ = random_pairs(schema, rng, 200, ["a", "b", "c", "zz"], 4)
    base = sorted(pairs.items())
    final = dict(pairs)
    deltas = []
    for k, v in more.items():                       # new routes and overwrites
        deltas.append(("put", k, v))
        final[k] = v
    for k, _ in base[::7]:                          # deletes (some of keys just overwritten: last one wins)
        deltas.append(("del", k))
        final.pop(k, None)
    for k in [k for k in final if k.startswith(b"\x00\x00\x02tB")]:   # tenant tB vanishes
        deltas.append(("del", k))
        final.pop(k)
    newcomer = schema.route_key("zz-new", "#", schema.receiver_url(1, "p", "d"))
    deltas.append(("put", newcomer, schema.incarnation_bytes(5)))
    final[newcomer] = schema.incarnation_bytes(5)
    tenants = tenants + ["zz-new"]
    topics = topics + ["anything/at/all", "$sys/x"]
    tt = tt + [3, 3]
    off, ranks, _ = walk(walker, str(tmp_path), base, tenants, topics, tt, deltas)
    want = oracle(sorted(final.items()), tenants, topics, tt)
    assert off.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    assert np.diff(off)[-2] == 1 and np.diff(off)[-1] == 0            # "#" matches everything but a '$' topic
    assert all(np.diff(off)[i] == 0 for i, t in enumerate(tt) if t == 1)   # nothing left under the vanished tenant


@pytest.mark.parametrize("config,scale", [("C3", 0.02), ("C4", 0.02), ("C2", 0.05)])
def test_image_walk_baseline_workloads_equal_oracle(walker, tmp_path, config, scale):
    """the BASELINE generators (bench.py's own inputs) at a small scale: tens of thousands of filters, the whole topic batch"""
    from bifromq_b200.workload import Workload
    w = Workload(config, scale=scale)
    n = min(w.n_topics, 20000)
    tmp = str(tmp_path)
    np.ascontiguousarray(w.keys).tofile(os.path.join(tmp, "keys.bin"))
    np.ascontiguousarray(w.vals).tofile(os.path.join(tmp, "vals.bin"))
    np.ascontiguousarray(w.key_off, dtype=np.int64).tofile(os.path.join(tmp, "koff.bin"))
    np.ascontiguousarray(w.val_off, dtype=np.int64).tofile(os.path.join(tmp, "voff.bin"))
    tb, toff = O.blob(w.tenants)
    np.ascontiguousarray(tb).tofile(os.path.join(tmp, "tenants.bin"))
    np.ascontiguousarray(toff, dtype=np.int64).tofile(os.path.join(tmp, "tenant_off.bin"))
    poff = np.ascontiguousarray(w.topic_off[:n + 1], dtype=np.int64)
    np.ascontiguousarray(w.topics[:int(poff[-1])]).tofile(os.path.join(tmp, "topics.bin"))
    poff.tofile(os.path.join(tmp, "topic_off.bin"))
    tt = np.ascontiguousarray(w.topic_tenant[:n], dtype=np.int32)
    tt.tofile(os.path.join(tmp, "topic_tenant.bin"))
    r = subprocess.run([walker, tmp], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    off = np.fromfile(os.path.join(tmp, "out_off.bin"), np.int64)
    ranks = np.fromfile(os.path.join(tmp, "out_ranks.bin"), np.int64)
    kv = O.KV()
    kv.load(w.keys, w.key_off, w.vals, w.val_off)
    kv.freeze()
    want = kv.match_blobs(tb, toff, w.topics, poff, tt, n, INT_MAX, INT_MAX, O.MODE_TRIE, False, os.cpu_count() or 1)
    assert np.array_equal(off, want.offsets) and np.array_equal(ranks, want.ranks)
    assert len(ranks) > n // 4
