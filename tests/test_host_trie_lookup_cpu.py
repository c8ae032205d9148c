"""The forward trie's child lookups at their hash edges, without a GPU: the builder's image (read back through
tests/native/image_walk_harness.cc dump) against the model in tests/trie_hash.py, and the engineered cases the GPU tests
(test_gpu_trie_lookup.py) run, each pinned to the edge it exists for.

A child lookup is exact only through details random keys rarely reach: the walk past a full home block (control byte) and
its wrap from the last block to block 0, every tag candidate of a block tried, the parent word compared (the tag table is shared
by every tenant), the length word compared ((24, P) and (LEN_CONT | 0, P) have the same token words), the slot compare behind
a single child's 16-bit fingerprint, and the fold-collision rule that makes a 2-child node wide. The cases below put keys on
each of these on purpose: full blocks, chains of 2 and 3 blocks, a chain that wraps, 4 keys with one fingerprint in one
block, absent names with a present key's block and fingerprint, a name with the same block and fingerprint under two tenant
roots, 24-byte length twins, fold pairs that make nodes wide below the root, single-child twins. BFQ_PERFECT_LOG2_MAX = 1 or 2
sends every node of 3 (5) or more children to the tag table, so whole workloads walk it at every depth."""
import itertools
import os

import numpy as np
import pytest

import trie_hash as T
from test_gpu_edges import make_pairs
from test_host_image_cpu import oracle, walk, walker  # noqa: F401  (walker: the harness fixture)

NB = 64                                   # every engineered case keeps <= 480 wide edges: 64 blocks
LONG = "L" * 30                           # a level of > 24 bytes: tier 0 hands the topic to tier 1
TIER2_TAIL = "/".join(["a"] * 8)          # with the '+/{a,+}^8' filters: a frontier of > 64 nodes, tier 2
# eng's private region opens the slot array right behind the tag table, and its root's '+' child is the region's first slot
ENG_PLUS_ID = 16 * NB
ENG, MIX, ENG2 = "eng", "mix", "eng2"     # tenant ordinals 0, 1, 2 (key order: a route key holds the tenant id behind its length)


def _routes(tenant, filters):
    """one route per filter, except every 5th (7 persistent routes) and every 7th (3 group routes): caps (5, 2) bind"""
    out = []
    for i, f in enumerate(filters):
        out.append((tenant, f, "p", 7) if i % 5 == 0 else (tenant, f, "g", 3) if i % 7 == 0 else (tenant, f, "pgn"[i % 3], 1))
    return out


def _fresh(names, taken):
    out = [n for n in names if n not in taken]
    taken.update(out)
    return out


def root_case():
    """the engineered tenant roots. eng: a wide root whose keys are placed from the model; eng2: a second wide root (a fold pair
    makes it wide) with the cross-parent twins; mix: a perfect-hash root with single-child nodes, for lanes of other kinds in
    the same warps. -> dict of the names per edge, the filters per tenant and the tier-0 topics"""
    p1, p2 = T.ROOT_BASE + 0, T.ROOT_BASE + 2
    taken = set()
    c = {}
    c["full"] = _fresh(T.names_homed(p1, NB, 10, 17, seed=10), taken)                 # 15 fill block 10, 2 chain into 11
    c["chain3"] = _fresh(T.names_homed(p1, NB, 20, 18, seed=11) + T.names_homed(p1, NB, 21, 15, seed=12), taken)
    c["wrap"] = _fresh(T.names_homed(p1, NB, NB - 1, 17, seed=13), taken)             # 2 wrap into block 0
    c["fp"] = _fresh(T.names_homed(p1, NB, 30, 4, fp=77, seed=14), taken)            # one fingerprint 4 times in one block
    c["k1"] = T.cross_parent_twin(p1, p2, NB, seed=15)                                # under eng only
    c["k2"] = T.cross_parent_twin(p1, p2, NB, seed=16)                                # under both roots
    c["p1"] = T.length_twin(p1, NB, seed=17)                                          # filter P1/X1 only
    c["p2"] = T.length_twin(p1, NB, seed=18)                                          # filter P2X2 only
    c["x1"], c["x2"] = T.length_twin_suffix("yy", False, seed=41), T.length_twin_suffix("yy", True, seed=42)
    taken.update([c["k1"], c["k2"], c["p1"], c["p2"]])
    reserved = {9, 10, 11, 12, 19, 20, 21, 22, 23, 29, 30, 31, NB - 2, NB - 1, 0, 1}
    rng = np.random.default_rng(20)
    fill = []
    while len(fill) < 100:
        nm = "f%07d" % rng.integers(0, 10 ** 7)
        if nm not in taken and T.level_home_block(nm, p1, NB) not in reserved:
            taken.add(nm)
            fill.append(nm)
    c["fill"] = fill
    (a, b), (a3, b3), (a2, b2), (a1, b1) = T.fold_pairs(4, seed=21)
    (qa, qb), = T.fold_pairs(1, seed=22, lenw=32)
    c["x_pair"], c["plus_pair"], c["eng2_pair"], c["eng_pair"], c["cont_pair"] = (a, b), (a3, b3), (a2, b2), (a1, b1), (qa, qb)
    c["q"] = "Q" * 24
    c["single"] = [("s1", "c1"), ("d/e/f", "c2"), ("m00", "v")]
    # eng's root has ~200 children, few enough for a perfect hash: the fold pair (a1, b1) makes it wide
    roots = c["full"] + c["chain3"] + c["wrap"] + c["fp"] + fill + [c["k1"], c["k2"]]
    eng = roots + [n + "/#" for n in roots] + [a1, b1, c["p1"] + "/" + c["x1"], c["p1"] + "/yy", c["p2"] + c["x2"], c["p2"] + "yy"]
    eng += ["x/" + a, "x/" + b, "+/" + a3, "+/" + b3, c["q"] + qa, c["q"] + qb, "s1/c1", "d/e/f/c2"]
    eng += ["+/+/+/+/zz"] + ["+/" + "/".join(p) for p in itertools.product(["a", "+"], repeat=8)]
    eng2 = [a2, b2, c["k2"], "+/+/+/+/zz"]
    mix = ["m%02d/v" % i for i in range(20)] + ["m%02d" % i for i in range(20)] + ["+/+/+/+/zz"]
    c["filters"] = {ENG: eng, ENG2: eng2, MIX: mix}
    # absent names with a present key's block and fingerprint, homed where the chains start: they walk each chain to its end
    tab = model_table(pairs_of(c))
    c["absent"] = []
    for blk, members in ((10, c["full"]), (20, c["chain3"]), (NB - 1, c["wrap"])):
        spilled = [nm for nm in members if tab_slot(tab, ENG, nm) // 16 != blk]
        fp = T.edge_place(*T.chunks(spilled[-1])[-1], p1, NB)[1]
        c["absent"] += _fresh(T.names_homed(p1, NB, blk, 2, fp=fp, seed=23 + blk), taken)
    c["absent"] += _fresh(T.names_homed(p1, NB, 30, 2, fp=77, seed=27), taken)
    c["twin_s"] = [T.single_child_twin(ch, seed=30 + i) for i, (_, ch) in enumerate(c["single"])]
    return c


def pairs_of(c):
    routes = []
    for t in (ENG, MIX, ENG2):
        routes += _routes(t, c["filters"][t])
    return make_pairs(routes)


def model_table(pairs, known=None, perfect_max=T.PERFECT_LOG2_MAX):
    """the tag table of a full build, tenants placed in ordinal order -> (TagTable, {(tenant, node path): slot}, Trie).
    A wide node outside the tag table (a '+' node: its id is a slot of the tenant's private region) needs its id in `known`
    (from the harness dump); without it its children are not placed. They are claimed after every root child (breadth-first
    order), so the root's keys do not depend on them."""
    trie = T.Trie(pairs)
    big = trie.big_edges(perfect_max)
    tab = T.TagTable(T.n_blocks_for(sum(len(v) for v in big.values())))
    ids, where = dict(known or {}), {}
    for o, t in enumerate(trie.tenants):
        ids[(t,)] = T.ROOT_BASE + o
    for t in trie.tenants:
        for node in big[t]:
            if node[:-1] in ids:
                ids[node] = where[node] = tab.claim(ids[node[:-1]], *node[-1])[0]
    return tab, where, trie


def eng_model(pairs):
    """model_table of an engineered case: eng's '+' node is wide (a fold pair), its id is ENG_PLUS_ID"""
    return model_table(pairs, {(ENG, "+"): ENG_PLUS_ID})


def tab_slot(model, tenant, level):
    """the slot of a root child of one chunk; model = (table, slots) of model_table"""
    return model[1][(tenant, T.chunks(level)[-1])]


def topics_of(c):
    """(tenant, topic) of the tier-0 batch: every engineered key and its absent twins"""
    eng = [nm for k in ("full", "chain3", "wrap", "fp", "absent") for nm in c[k]] + c["fill"][:30]
    eng += [c["k1"], c["k2"], c["k1"] + "/zz", c["p1"] + "/" + c["x1"], c["p2"] + "/" + c["x2"], "x/" + c["x_pair"][0], "x/" + c["x_pair"][1],
            "x/nope", "q/" + c["plus_pair"][1], "q/" + c["plus_pair"][0] + "x"]
    eng += ["s1/c1", "s1/" + c["twin_s"][0], "d/e/f/c2", "d/e/f/" + c["twin_s"][1]]
    out = [(ENG, t) for t in eng]
    out += [(ENG2, c["k1"]), (ENG2, c["k2"]), (ENG2, c["eng2_pair"][0]), (ENG2, c["eng2_pair"][1]), (ENG2, c["x_pair"][0])]
    out += [(MIX, "m%02d/v" % i) for i in range(0, 20, 3)] + [(MIX, "m00/" + c["twin_s"][2]), (MIX, "m07")]
    # interleave the tenants so that every warp mixes wide-root lanes with perfect-hash and single-child lanes
    rng = np.random.default_rng(40)
    return [out[i] for i in rng.permutation(len(out))]


def long_topics(c):
    """topics that reach a level longer than 24 bytes: the length twins P1X1, P2X2 (tier 1 looks up (LEN_CONT | 0, P))"""
    return [(ENG, c["p1"] + c["x1"]), (ENG, c["p2"] + c["x2"]), (ENG, c["q"] + c["cont_pair"][0]), (ENG, c["q"] + c["cont_pair"][1]),
            (ENG, c["q"] + "nope")]


def tiered(batch, tier):
    """tier 0: as is; tier 1: a level of > 24 bytes appended (tier 0 hands the topic over, tier 1 walks it from the root);
    tier 2: the root-level names, 8 more levels that the '+/{a,+}^8' filters turn into a frontier of > 64 nodes"""
    if tier == 0:
        return batch
    if tier == 1:
        return [(t, s + "/" + LONG) for t, s in batch if s.count("/") < 4]
    return [(t, s + "/" + TIER2_TAIL) for t, s in batch if "/" not in s]


def as_arrays(batch):
    tenants = [ENG, ENG2, MIX]
    return tenants, [s for _, s in batch], np.array([tenants.index(t) for t, _ in batch], np.int32)


# ------------------------------------------------------------------ the harness dump
def read_dump(path):
    nodes, tags, nb = {}, {}, None
    for line in open(path):
        f = line.split()
        if f[0] == "n_blocks":
            nb = int(f[1])
        elif f[0] == "node":
            nodes[(int(f[1]), int(f[2]))] = (None if f[3] == "NONE" else int(f[3]), f[4], int(f[5]), int(f[6]))
        else:
            tags[int(f[1])] = bytes.fromhex(f[2])
    return nb, nodes, np.array([list(tags[b]) for b in range(nb)], np.uint8).reshape(nb, 16)


def dump(walker, tmp, pairs, batch, env=None):  # noqa: F811
    tenants, topics, tt = as_arrays(batch)
    off, ranks, _ = walk(walker, tmp, pairs, tenants, topics, tt, env=env, dump=True)
    return read_dump(os.path.join(tmp, "dump.txt")), (off, ranks), (tenants, topics, tt)


@pytest.fixture(scope="module")
def case():
    return root_case()


def test_engineered_cases_sit_on_their_edges(case):
    c = case
    tab, where, trie = model_table(pairs_of(c))
    assert tab.n_blocks == NB
    p1 = T.ROOT_BASE

    def blk(nm):
        return tab_slot((tab, where), ENG, nm) // 16
    full = (tab.tags[:, :15] != 0).all(axis=1)
    assert full[10] and tab.tags[10, 15] == 1 and tab.tags[11, 15] == 0                # a chain of 2 blocks
    assert 11 in {blk(n) for n in c["full"]}
    assert full[20] and full[21] and tab.tags[20, 15] == tab.tags[21, 15] == 1 and tab.tags[22, 15] == 0
    assert 22 in {blk(n) for n in c["chain3"]}                                          # a chain of 3 blocks
    assert full[NB - 1] and tab.tags[NB - 1, 15] == 1 and tab.tags[0, 15] == 0          # >= 16 at the last block: wrap
    assert 0 in {blk(n) for n in c["wrap"]}
    fp_slots = sorted(tab_slot((tab, where), ENG, n) for n in c["fp"])
    assert [s // 16 for s in fp_slots] == [30] * 4 and (tab.tags[30, :15] == 77).sum() == 4
    pos = []                                                                            # 3 of them are a later candidate
    for n in c["fp"]:
        s, path = tab.probe(p1, *T.chunks(n)[-1])
        assert len(path) == 1
        pos.append(path[0][1].index(s))
    assert sorted(pos) == [0, 1, 2, 3]
    for nm in c["absent"]:                                                               # absent, yet a candidate somewhere
        s, path = tab.probe(p1, *T.chunks(nm)[-1])
        assert s is None and any(cands for _, cands in path), nm
        assert len(path) >= 2 or path[0][0] == 30
    assert max(len(tab.probe(p1, *T.chunks(nm)[-1])[1]) for nm in c["absent"]) == 3       # one walks a 3-block chain
    assert {len(tab.probe(p1, *T.chunks(nm)[-1])[1]) for nm in c["wrap"]} >= {1, 2}
    for k in ("k1", "k2"):
        assert T.edge_place(*T.chunks(c[k])[-1], p1, NB) == T.edge_place(*T.chunks(c[k])[-1], p1 + 2, NB)
    for p, x in (("p1", "x1"), ("p2", "x2")):
        assert len(c[p]) == 24 and T.edge_place(24, c[p].encode(), p1, NB) == T.edge_place(T.LEN_CONT, c[p].encode(), p1, NB)
    # below either twin, X spelled the other way hashes to X's own slot
    pl = trie.plans()
    for node, x, own, other in (((ENG, (24, c["p1"].encode())), c["x1"], 8, 32), ((ENG, (T.LEN_CONT, c["p2"].encode())), c["x2"], 32, 8)):
        kind, lg, sd = pl[node]
        assert kind == "perfect" and len(trie.children[node]) == 2
        assert T.child_index(T.edge_fold(own, x.encode()), sd, lg) == T.child_index(T.edge_fold(other, x.encode()), sd, lg)
    assert pl[(ENG,)][0] == "big" and pl[(ENG2,)][0] == "big" and pl[(MIX,)][0] == "perfect"
    x, plus = (ENG, T.chunks("x")[0]), (ENG, "+")
    cont = (ENG, (T.LEN_CONT, c["q"].encode()))
    for node in (x, plus, cont):                                                         # small nodes made wide by a fold pair
        assert len(trie.children[node]) <= 3 and pl[node][0] == "big", node
    for (parent, child), twin in zip(c["single"], c["twin_s"]):
        assert twin != child and T.edge_fold(*T.chunks(twin)[-1]) & 0xFFFF == T.edge_fold(*T.chunks(child)[-1]) & 0xFFFF
        node = (MIX if parent == "m00" else ENG,) + tuple(T.chunks(lv)[-1] for lv in parent.split("/"))
        assert pl[node][0] == "single", node
    assert sum(len(v) for v in trie.big_edges().values()) <= 480


def test_model_agrees_with_the_builder_on_the_engineered_cases(walker, tmp_path, case):  # noqa: F811
    """slots, tags, control bytes and node kinds of the image equal the model's; the walk equals the oracle"""
    pairs = pairs_of(case)
    batch = topics_of(case) + long_topics(case)
    (_, ids, _), _, _ = dump(walker, str(tmp_path / "ids"), pairs, [(ENG, "+")])
    (nb, nodes, tags), (off, ranks), (tenants, topics, tt) = dump(walker, str(tmp_path / "walk"), pairs, batch)
    assert ids[(0, 1)][0] == ENG_PLUS_ID
    tab, where, trie = eng_model(pairs)
    assert nb == tab.n_blocks == NB and tab.claimed() == sum(len(v) for v in trie.big_edges().values())
    # eng2's keys may take slots in eng's blocks in either order (tenants are placed by concurrent threads): every block's
    # tags as a multiset, every control byte, and the exact slot of every eng key in a block eng2 does not reach
    assert (np.sort(tags[:, :15], axis=1) == np.sort(tab.tags[:, :15], axis=1)).all()
    assert (tags[:, 15] == tab.tags[:, 15]).all()
    eng2_blocks = {s // 16 for n, s in where.items() if n[0] == ENG2}
    pl = trie.plans()
    for i, (t, s) in enumerate(batch):
        node = (t,)
        for d, lv in enumerate(s.split("/")):
            got = nodes.get((i, d))
            assert got is not None
            kind = pl[node][0] if node in pl else "none"
            want_kind = {"single": "single", "perfect": "perfect", "big": "big", "none": "none"}[kind]
            assert got[1] == want_kind, (s, d, got, kind)
            if kind == "perfect":
                assert (got[2], got[3]) == pl[node][1:], (s, d)
            if kind == "single":
                assert got[3] == pl[node][2]
            if node in where and where[node] // 16 not in eng2_blocks:
                assert got[0] == where[node], (s, d)
            node = node + (("+",) if lv == "+" else tuple(T.chunks(lv)))
            if node not in trie.nodes:
                break
    want = oracle(pairs, tenants, topics, tt)
    assert off.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    assert sum(np.diff(off) > 0) > len(batch) // 2


def test_model_agrees_with_host_build_stats(case):
    from test_host_wide_delta_cpu import host_stats
    pairs = pairs_of(case)
    tab, _, _ = eng_model(pairs)
    assert host_stats(pairs)[8] == tab.overflowed() > 0


# ------------------------------------------------------------------ BFQ_PERFECT_LOG2_MAX: wide nodes at every depth
def random_forced_pairs(seed):
    import random
    from test_host_image_cpu import random_pairs
    from bifromq_b200 import schema
    rng = random.Random(seed)
    pairs, tenants, topics, tt = random_pairs(schema, rng, 900, ["a", "b", "c", "dd", "e1", "f", "g"], 5)
    return sorted(pairs.items()), tenants, topics, tt


def forced_big_edges(pairs, m):
    """wide edges the model predicts at BFQ_PERFECT_LOG2_MAX = m"""
    return sum(len(v) for v in T.Trie(pairs).big_edges(m).values())


@pytest.mark.parametrize("m", [1, 2])
@pytest.mark.parametrize("seed", [1, 2])
def test_forced_wide_nodes_walk_and_edge_count(walker, tmp_path, m, seed):  # noqa: F811
    pairs, tenants, topics, tt = random_forced_pairs(seed)
    off, ranks, _ = walk(walker, str(tmp_path), pairs, tenants, topics, tt, env={"BFQ_PERFECT_LOG2_MAX": str(m)}, dump=True)
    want = oracle(pairs, tenants, topics, tt)
    assert off.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    nb, _, tags = read_dump(os.path.join(str(tmp_path), "dump.txt"))
    trie = T.Trie(pairs)
    # the rule restated: c >= 3 (m = 1) or c >= 5 (m = 2) children, or two children with one fold
    folds = {n: [T.edge_fold(*e) for e in cs] for n, cs in trie.children.items()}
    rule = sum(len(f) for f in folds.values() if len(f) >= 2 * m + 1 or len(set(f)) < len(f))
    got = int((tags[:, :15] != 0).sum())
    assert got == forced_big_edges(pairs, m) == rule > 100
    assert nb == T.n_blocks_for(got)


@pytest.mark.parametrize("m", [1, 2])
def test_forced_wide_nodes_on_the_engineered_cases(walker, tmp_path, case, m):  # noqa: F811
    """the engineered keys with most other nodes wide too; the fold-pair nodes stay wide and the walk equals the oracle"""
    pairs = pairs_of(case)
    batch = topics_of(case) + long_topics(case)
    (nb, nodes, tags), (off, ranks), (tenants, topics, tt) = dump(walker, str(tmp_path), pairs, batch, env={"BFQ_PERFECT_LOG2_MAX": str(m)})
    want = oracle(pairs, tenants, topics, tt)
    assert off.tolist() == want.offsets.tolist() and ranks.tolist() == want.ranks.tolist()
    assert int((tags[:, :15] != 0).sum()) == forced_big_edges(pairs, m)
    assert nodes[(batch.index((MIX, "m00/v")), 0)][1] == "big"          # the 20-child root: wide at m = 1 and 2
