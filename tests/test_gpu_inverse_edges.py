"""The inverse match (topic filters -> indexed topics) at the edges of its tiers, its range-buffer re-run, its locality order
and its level-0 '$' cuts.

The inverse path (bifromq_b200/csrc/rmatch_kernels.cu) walks one warp per filter over a BFS-numbered topic trie. A filter whose
frontier or range list does not fit tier 1's shared-memory buffers is handed, whole, to tier 2 (global scratch); a batch whose
ranges do not fit the range buffer grows it and is re-run; batches of >= 4096 filters run in locality order. Each is its own code
path, and a slip in one sends a retained message to the wrong subscriber, or drops one, without any error. Every test here
builds its case from plain topics and filters, checks the whole answer against the CPU oracle (offsets, per-filter id sets,
distinct ids, totals) and asserts, through what the result reports (n_overflow_filters, n_ranges), that the path it targets
was taken.

The numbers the GPU reports are predicted by a plain-Python model of the kernel's bookkeeping (TrieModel below): the tries
as rebuild() lays them out and each filter walked with rmatch_one's rules. The model is itself checked against the oracle's
TopicLevelIndex and the brute-force predicate on every case this file generates, and CPU shape tests pin each generator to its
edge ("this filter has exactly 64 frontier intervals", "this level is 48 bytes and shares its first 24 with a sibling").

Limits exercised (rmatch_kernels.cu): tier 1 holds 64 frontier intervals and 64 ranges per filter (R_FR_CAP / R_RG_CAP, :95;
over either the filter goes to tier 2, :371-384 and :973-994); filters of <= 256 bytes are staged in shared memory, longer ones
are read from global (R_STAGE, :133-138); levels over 24 bytes are chains of virtual nodes shared by names with the same
leading chunks (TOKEN_BYTES, :639-672 and :321-348); the level-0 '$' run is cut out of '#', a final '+', '+/#' and a non-final
'+' (:240-252, :273-295, :307-315); batches of >= 4096 filters run in locality order (:927-958); the range buffer starts at
max(2^18, 8n) ranges and is grown and the batch re-run when too small (:886, :959-1002); rexpand_kernel keeps the first
min(total, limit) ids of each filter (:420-449).
"""
import ctypes as C
import random

import numpy as np
import pytest

import oracle_lib as O

R_FR_CAP, R_RG_CAP = 64, 64
R_STAGE = 256
TOKEN_BYTES = 24
ORDER_MIN_FILTERS = 4096     # batches of at least this many filters run in locality order


def initial_range_cap(n):
    """ranges the range buffer of a fresh handle holds before its first re-run"""
    return max(2 ** 18, 8 * max(n, 1))


DFS, BFS = 0, 1


# ------------------------------------------------------------------ model of the kernel's bookkeeping (plain Python)
class TrieModel:
    """rebuild()'s layout of a set of live topics and rmatch_one's walk over it.

    entries: {(tenant, topic): id}. Children are sorted bytewise; nodes get one global BFS numbering, tenant roots first (in
    bytewise tenant order); topics get a DFS rank per tenant (pre-order, own topic first) and a BFS rank (by the BFS id of
    the node they end at); the children of a node whose names start with '$' form one run."""

    def __init__(self, entries):
        kids, own = [], []

        def new():
            kids.append({})
            own.append(-1)
            return len(kids) - 1
        root_of, roots = {}, []
        for (tenant, topic), tid in sorted((( O._b(t), O._b(p)), i) for (t, p), i in entries.items()):
            if tenant not in root_of:
                root_of[tenant] = new()
                roots.append(root_of[tenant])
            cur = root_of[tenant]
            for lv in topic.split(b"/"):
                if lv not in kids[cur]:
                    kids[cur][lv] = new()
                cur = kids[cur][lv]
            own[cur] = tid
        order = list(roots)
        i = 0
        while i < len(order):
            order += [kids[order[i]][k] for k in sorted(kids[order[i]])]
            i += 1
        bfs = {h: b for b, h in enumerate(order)}
        n = len(order)
        self.child_begin, self.child_count = [0] * (n + 1), [0] * (n + 1)
        self.own_prefix, self.sys_begin, self.sys_count = [0] * (n + 1), [0] * (n + 1), [0] * (n + 1)
        self.sub_begin, self.sub_end = [0] * (n + 1), [0] * (n + 1)
        self.bfs_to_id, self.dfs_to_id = [], []
        self.child = {}        # (parent BFS id, name) -> child BFS id: the exact-edge table
        nxt = len(roots)
        for b, h in enumerate(order):
            names = sorted(kids[h])
            self.child_begin[b], self.child_count[b] = nxt, len(names)
            self.own_prefix[b] = len(self.bfs_to_id)
            if own[h] >= 0:
                self.bfs_to_id.append(own[h])
            sys = [k for k, nm in enumerate(names) if nm[:1] == b"$"]
            if sys:
                self.sys_begin[b], self.sys_count[b] = nxt + sys[0], len(sys)
            for nm in names:
                self.child[(b, nm)] = bfs[kids[h][nm]]
            nxt += len(names)
        self.child_begin[n], self.own_prefix[n] = nxt, len(self.bfs_to_id)
        for r in roots:
            stack = [(r, iter(sorted(kids[r])))]
            self.sub_begin[bfs[r]] = len(self.dfs_to_id)
            while stack:
                h, it = stack[-1]
                nm = next(it, None)
                if nm is None:
                    self.sub_end[bfs[h]] = len(self.dfs_to_id)
                    stack.pop()
                    continue
                c = kids[h][nm]
                self.sub_begin[bfs[c]] = len(self.dfs_to_id)
                if own[c] >= 0:
                    self.dfs_to_id.append(own[c])
                stack.append((c, iter(sorted(kids[c]))))
        self.root = {t: bfs[r] for t, r in root_of.items()}

    def own(self, v):
        return self.own_prefix[v + 1] - self.own_prefix[v]

    def walk(self, tenant, flt):
        """-> (largest frontier in intervals, ranges [(space, first, count)] in emit order, ids in expand order)"""
        root = self.root.get(O._b(tenant))
        if root is None:
            return 0, [], []
        levels = O._b(flt).split(b"/")
        fr, max_fr, rg = [(root, 1)], 1, []
        op = self.own_prefix

        def emit(space, first, count):
            if count > 0:
                rg.append((space, first, count))

        def subtree(v, lo, level):
            # the topics of v's subtree from DFS rank lo; at level 0 without the subtrees of the '$' children
            if level == 0 and self.sys_count[v]:
                s0, s1 = self.sys_begin[v], self.sys_begin[v] + self.sys_count[v] - 1
                emit(DFS, lo, self.sub_begin[s0] - lo)
                emit(DFS, self.sub_end[s1], self.sub_end[v] - self.sub_end[s1])
            else:
                emit(DFS, lo, self.sub_end[v] - lo)
        for level, tok in enumerate(levels):
            last = level == len(levels) - 1
            hash_next = level == len(levels) - 2 and levels[-1] == b"#"
            nodes = [v for a, c in fr for v in range(a, a + c)]
            nxt = []
            if last and tok == b"#":
                for v in nodes:
                    subtree(v, self.sub_begin[v] + self.own(v), level)
                break
            if tok == b"+":
                for a, c in fr:
                    n0, n1 = a, a + c - 1
                    cb, ce = self.child_begin[n0], self.child_begin[n1] + self.child_count[n1]
                    sb, se = self.sys_begin[n0], self.sys_begin[n0] + self.sys_count[n0]
                    parts = [(cb, sb), (se, ce)] if level == 0 and self.sys_count[n0] else [(cb, ce)]
                    for x, y in parts:
                        if last:
                            emit(BFS, op[x], op[y] - op[x])
                        elif not hash_next and y > x:
                            nxt.append((x, y - x))
                if hash_next:
                    for v in nodes:
                        subtree(v, self.sub_begin[v] + self.own(v), level)
                if last or hash_next:
                    break
            else:
                for v in nodes:
                    ch = self.child.get((v, tok))
                    if ch is None:
                        continue
                    if last:
                        emit(BFS, op[ch], self.own(ch))
                    elif hash_next:
                        emit(DFS, self.sub_begin[ch], self.sub_end[ch] - self.sub_begin[ch])
                    else:
                        nxt.append((ch, 1))
                if last or hash_next:
                    break
            max_fr = max(max_fr, len(nxt))
            fr = nxt
            if not fr:
                break
        ids = []
        for space, first, count in rg:
            ids += (self.bfs_to_id if space == BFS else self.dfs_to_id)[first:first + count]
        return max_fr, rg, ids

    def tier2(self, tenant, flt):
        mf, rg, _ = self.walk(tenant, flt)
        return mf > R_FR_CAP or len(rg) > R_RG_CAP


def ids_of(topics):
    """(tenant, topic) pairs in add order -> {pair: id} the way the index hands ids out (insertion order, repeats keep theirs)"""
    out = {}
    for k in topics:
        out.setdefault(k, len(out))
    return out


def oracle_of(entries):
    orc = O.TopicLevelIndex()
    for (t, p), i in entries.items():
        orc.add(p, i, t)
    return orc


def predicate_ids(entries, tenant, flt):
    return sorted(i for (t, p), i in entries.items() if t == tenant and O.topic_matches_filter(p, flt))


# ------------------------------------------------------------------ cases (plain Python data, no GPU)
WIDTHS = (63, 64, 65)
TIER1_FILTERS = ["+/x/y/z", "+/x", "+/x/#", "+/+/#", "+/x/y", "+/+", "+", "#", "+/#", "+/+/+", "+/+/+/#", "a00/x/y",
                 "a00/+/y/z", "+/x/+/z", "$s/+/y", "$s/#"]


def wide_names(w):
    """w level-0 names sorting on both sides of '$' ('!' < '$' < 'a')"""
    return [("!%02d" if i % 2 else "a%02d") % i for i in range(w)]


def wide_tenant(w, sys):
    return "w%d%s" % (w, "s" if sys else "")


def wide_topics(w, sys):
    """w level-0 names, each with <name>/x and <name>/x/y, the first also <name>/x/y/z; with sys a '$s' name with the same
    children, which no wildcard at level 0 may reach"""
    t = wide_tenant(w, sys)
    names = wide_names(w) + (["$s"] if sys else [])
    out = []
    for nm in names:
        out += [(t, nm + "/x"), (t, nm + "/x/y")]
    out += [(t, names[0] + "/x/y/z")]
    if sys:
        out += [(t, "$s/x/y/z"), (t, "$s")]
    return out


def wide_case():
    topics, filters = [], []
    for w in WIDTHS:
        for sys in (False, True):
            topics += wide_topics(w, sys)
            filters += [(wide_tenant(w, sys), f) for f in TIER1_FILTERS]
    return topics, filters


DOLLAR_NAMES = ["", "!", "$", "$$", "$SYS", "$a", "%", "A", "a", "é"]
DOLLAR_TENANTS = {"d_mix": DOLLAR_NAMES, "d_sys": ["$", "$$", "$SYS", "$a"], "d_lo": ["", "!", "!!", '"'],
                  "d_hi": ["%", "A", "a", "é"]}
DOLLAR_FILTERS = ["#", "+", "+/#", "+/+", "+/+/#", "+/x", "$SYS/#", "$SYS/+", "/#", "a/+", "a/+/#", "+/$x", "a/#", "$/#",
                  "$/+", "+/+/+", "$SYS", "", "a/$x", "+/x/y"]


def dollar_case():
    """level-0 names on both sides of the '$' run, only '$' names, only names before / after it; names under a level-1 '$'
    (a '+' there must not cut them). The tenants are neighbours in the BFS numbering and hold topics at the same depths."""
    topics = []
    for t, names in DOLLAR_TENANTS.items():
        for nm in names:
            topics += [(t, nm), (t, nm + "/x"), (t, nm + "/x/y")]
        if "a" in names:
            topics += [(t, "a/$x"), (t, "a/$x/y"), (t, "a/b"), (t, "a/$")]
    filters = [(t, f) for t in DOLLAR_TENANTS for f in DOLLAR_FILTERS]
    return topics, filters


def text(n, seed):
    """n bytes of lower-case letters and digits (no '/', '+', '#')"""
    rng = random.Random(seed)
    return "".join(rng.choice("abcdefghijklmnopqrstuvwxyz0123456789") for _ in range(n))


def path_of_len(n, plen, seed):
    """a topic of levels of <= 20 bytes whose filter (behind a plen-byte prefix) is n bytes long"""
    s, k = "", 0
    while plen + len(s) + 21 < n:
        s += text(19, seed * 100 + k) + "/"
        k += 1
    return s + text(n - plen - len(s), seed * 100 + k)


def path_slash_at(p, plen, seed):
    """a topic whose filter (behind a plen-byte prefix) has a '/' at byte p, then two more levels"""
    s, k = "", 0
    while plen + len(s) + 20 <= p:
        s += text(19, seed * 100 + k) + "/"
        k += 1
    return s + text(p - plen - len(s), seed * 100 + k) + "/" + text(5, seed) + "/q"


FILTER_LENGTHS = [255, 256, 257, 300, 1000]
SLASH_AT = [255, 256, 257]
LEVEL_LENGTHS = [23, 24, 25, 47, 48, 49, 72, 73]
LEVEL_COUNTS = [1, 31, 32, 33, 64, 200]
EMPTY_TOPICS = ["", "/", "//", "e//f", "/e", "e/", "e//", "e"]
EMPTY_FILTERS = ["", "/", "//", "+", "+/+", "/+", "+/", "+//+", "e//f", "e//#", "/#", "e/#", "e/+", "e/+/f", "+/+/+", "e//+"]


def long_parts(plen):
    """(topics, filters) of the long-filter and long-level cases, written for filters behind a plen-byte prefix"""
    topics, filters = [], []
    for n in FILTER_LENGTHS:
        p = path_of_len(n, plen, n)
        lv = p.split("/")
        topics += [p, "/".join(lv[:-1] + ["other"])]
        filters += [p, "/".join(lv[:-1] + ["+"]), "/".join(lv[:len(lv) // 2] + ["#"]), "/".join(["+"] + lv[1:]), p[:-1]]
    for s in SLASH_AT:
        p = path_slash_at(s, plen, s)
        lv = p.split("/")
        topics += [p, "/".join(lv[:-1])]
        filters += [p, "/".join(lv[:-1]), "/".join(lv[:-1] + ["#"]), "/".join(lv[:-2] + ["+", "+"]), "/".join(lv[:-2] + ["+", "q"])]
    for n in LEVEL_LENGTHS:
        s = text(n, 1000 + n)
        topics += ["lv/" + s, "lv/" + s + "/t"]
        filters += ["lv/" + s, "lv/" + s + "/t", "lv/" + s + "/#", "lv/" + s + "/+", "+/" + s, "+/" + s + "/t", "lv/" + s[:-1],
                    "lv/" + s + "x", "lv/" + s[:-1] + "/t"]
    # sibling names sharing their first 24 or 48 bytes (one shared virtual node), a 24-byte name beside a 25-byte one
    a24 = text(24, 7)
    a48 = a24 + text(24, 8)
    sib = [a24, a24 + "b", a24 + text(10, 9), a24 + text(30, 10), a48, a48 + "x", a48 + "y" + text(30, 11), a48[:24] + "Q" * 24]
    for nm in sib:
        topics += ["sh/" + nm, "sh/" + nm + "/k"]
        filters += ["sh/" + nm, "sh/" + nm + "/k", "sh/" + nm + "/#", "+/" + nm + "/k", "sh/" + nm + "/+"]
    filters += ["sh/" + a24 + "c", "sh/" + a24[:23], "sh/" + a48 + "z", "sh/" + a48[:47], "sh/+/k", "sh/+", "sh/#", "sh/+/#",
                "+/+/k", "+/+/t", "lv/+/t", "lv/+/#"]
    for n in LEVEL_COUNTS:
        lv = ["m%d" % i for i in range(n)]
        topics += ["/".join(lv), "/".join(lv[:-1] + ["z"])]
        filters += ["/".join(lv), "/".join(["+"] + lv[1:]), "/".join(lv[:-1] + ["+"]), "/".join(lv[:n // 2] + ["+"] + lv[n // 2 + 1:]),
                    "/".join(["+"] * n), "/".join(lv[:n // 2] + ["#"]), "/".join(lv + ["#"])]
    topics += EMPTY_TOPICS
    filters += EMPTY_FILTERS
    return topics, filters


LONG_TIER2_PREFIX = ("+/x/", "a00/x/")   # the filter prefix and where the topics hang: 65 frontier intervals after "+/x"


def long_case(tier2):
    """tier 1: the long filters and levels on their own tenant; tier 2: the same behind "+/x/" on the 65-name tenant of the
    tier-1 case, the topics under its first name, so every filter reaches 65 frontier intervals and goes to tier 2"""
    fpre, tpre = LONG_TIER2_PREFIX if tier2 else ("", "")
    tenant = wide_tenant(65, False) if tier2 else "long"
    tp, fl = long_parts(len(fpre))
    topics = (wide_topics(65, False) if tier2 else []) + [(tenant, tpre + t) for t in tp]
    return topics, [(tenant, fpre + f) for f in fl]


CASES = {"wide": wide_case, "dollar": dollar_case, "long": lambda: long_case(False), "long_tier2": lambda: long_case(True)}


def rerun_case(w, n=4200):
    """n filters on the w-wide tenants that each emit exactly w ranges and no more than w frontier intervals"""
    fs = ["+/x", "+/x/#", "+/+/#", "+/x/y"]
    topics = wide_topics(w, False) + wide_topics(w, True)
    filters = [(wide_tenant(w, i % 2 == 1), fs[i % len(fs)]) for i in range(n)]
    return topics, filters


# ------------------------------------------------------------------ CPU: the model against the oracle and the predicate
@pytest.mark.parametrize("case", sorted(CASES))
def test_model_agrees_with_oracle_and_predicate(case):
    topics, filters = CASES[case]()
    entries = ids_of(topics)
    model, orc = TrieModel(entries), oracle_of(entries)
    nonempty = 0
    for t, f in filters:
        _, _, ids = model.walk(t, f)
        want = orc.match(f, t)
        assert sorted(ids) == want, (t, f)
        assert want == predicate_ids(entries, t, f), (t, f)
        assert len(set(ids)) == len(ids)
        nonempty += bool(want)
    assert nonempty > len(filters) // 2


def test_model_after_removals_and_unknown_tenants():
    topics, filters = dollar_case()
    entries = ids_of(topics)
    live = {k: i for k, i in entries.items() if i % 4 == 1}
    model, orc = TrieModel(live), oracle_of(live)
    for t, f in filters + [("nobody", "#"), ("d_mix2", "+")]:
        assert sorted(model.walk(t, f)[2]) == orc.match(f, t) == predicate_ids(live, t, f), (t, f)


# ------------------------------------------------------------------ CPU: the shapes the GPU tests rely on
def test_tier1_case_shape():
    topics, _ = wide_case()
    model = TrieModel(ids_of(topics))
    for w in WIDTHS:
        for sys in (False, True):
            t = wide_tenant(w, sys)
            fr0 = 2 if sys else 1                        # the '$s' name splits the level-0 interval in two
            mf, rg, _ = model.walk(t, "+/x/y/z")          # frontier-bound: w single-node intervals, 1 range
            assert mf == w and len(rg) == 1
            for f in ("+/x", "+/x/#", "+/+/#"):           # range-bound, the frontier stays the level-0 interval(s)
                mf, rg, _ = model.walk(t, f)
                assert len(rg) == w and mf <= fr0, (t, f)
            mf, rg, _ = model.walk(t, "+/x/y")            # both at once
            assert mf == w and len(rg) == w
            mf, rg, _ = model.walk(t, "+/+")              # one BFS range per frontier interval whatever the width
            assert len(rg) == fr0 and mf == fr0 and all(s == BFS for s, _, _ in rg)
            assert model.tier2(t, "+/x") == (w > 64) and not model.tier2(t, "+/+")
            names = sorted(O._b(n) for n in wide_names(w) + (["$s"] if sys else []))
            if sys:
                k = names.index(b"$s")
                assert 0 < k < len(names) - 1            # names on both sides of the '$' run
    n_tier2 = sum(model.tier2(t, f) for t, f in wide_case()[1])
    assert 0 < n_tier2 < len(wide_case()[1])


def test_dollar_case_shape():
    names = sorted(O._b(n) for n in DOLLAR_NAMES)
    sys = [i for i, n in enumerate(names) if n[:1] == b"$"]
    assert sys == list(range(sys[0], sys[-1] + 1)) and 0 < sys[0] and sys[-1] < len(names) - 1
    assert names[-1] == "é".encode() and names[0] == b""
    assert all(n.startswith("$") for n in DOLLAR_TENANTS["d_sys"])
    assert all(O._b(n) < b"$" for n in DOLLAR_TENANTS["d_lo"]) and all(O._b(n) > b"$~" for n in DOLLAR_TENANTS["d_hi"])
    topics, filters = dollar_case()
    model = TrieModel(ids_of(topics))
    # the tenants' roots are neighbours in the BFS numbering, and each holds topics at depths 1, 2 and 3
    assert sorted(model.root.values()) == list(range(len(DOLLAR_TENANTS)))
    for t in DOLLAR_TENANTS:
        assert {p.count("/") + 1 for tt, p in topics if tt == t} >= {1, 2, 3}
    # the final '+' at level 0 emits two BFS ranges on d_mix (names before and after the '$' run), one elsewhere
    assert len(model.walk("d_mix", "+")[1]) == 2 and len(model.walk("d_hi", "+")[1]) == 1
    assert len(model.walk("d_mix", "#")[1]) == 2 and model.walk("d_sys", "#")[1] == []
    # a level-1 '$' name under a '+' is matched: the '$' cut is a level-0 rule
    assert any(p == "a/$x" for (t, p), i in ids_of(topics).items() if i in model.walk("d_mix", "a/+")[2])


def test_long_case_shape():
    for tier2 in (False, True):
        topics, filters = long_case(tier2)
        fb = [O._b(f) for _, f in filters]
        lens = {len(f) for f in fb}
        assert set(FILTER_LENGTHS) <= lens, tier2
        assert max(lens) > R_STAGE >= min(lens)
        for p in SLASH_AT:
            assert any(len(f) > p and f[p:p + 1] == b"/" for f in fb), (tier2, p)
        lv_lens = {len(lv) for _, f in filters for lv in O._b(f).split(b"/")}
        assert set(LEVEL_LENGTHS) <= lv_lens
        depths = {f.count(b"/") + 1 for f in fb}
        off = 2 if tier2 else 0
        assert {n + off for n in LEVEL_COUNTS} <= depths
        model = TrieModel(ids_of(topics))
        tier2_n = sum(model.tier2(t, f) for t, f in filters)
        assert tier2_n == (len(filters) if tier2 else 0), tier2
    # names sharing their first 24 / 48 bytes, and a 24-byte name beside a 25-byte one with the same first 24
    tp, _ = long_parts(0)
    sh = [O._b(t)[3:] for t in tp if t.startswith("sh/") and "/k" not in t]
    a24 = [s for s in sh if len(s) == TOKEN_BYTES]
    assert len(a24) == 1 and O._b(a24[0]) + b"b" in sh
    assert sum(1 for s in sh if len(s) > TOKEN_BYTES and s[:24] == a24[0]) >= 4
    assert sum(1 for s in sh if len(s) > 2 * TOKEN_BYTES and s[:48] == next(x for x in sh if len(x) == 48)) >= 2
    assert "" in EMPTY_FILTERS and "/" in EMPTY_FILTERS


def test_rerun_case_shape():
    for w in (64, 65):
        topics, filters = rerun_case(w)
        model = TrieModel(ids_of(topics))
        per = {tf: model.walk(*tf) for tf in set(filters)}
        assert all(len(rg) == w and mf <= w for mf, rg, _ in per.values())
        n_ranges = sum(len(per[tf][1]) for tf in filters)
        assert n_ranges > initial_range_cap(len(filters)) and 8 * len(filters) < 2 ** 18
        assert len(filters) >= ORDER_MIN_FILTERS
        assert sum(model.tier2(t, f) for t, f in set(filters)) == (0 if w == 64 else len(set(filters)))


def test_locality_case_shape():
    shared, padded, pos = locality_batches()
    assert len(shared) == ORDER_MIN_FILTERS - 1 and len(padded) >= ORDER_MIN_FILTERS
    at = set(pos)
    assert [padded[p] for p in pos] == shared and all(t == "pad" for i, (t, _) in enumerate(padded) if i not in at)


def locality_batches():
    """the same 4095 filters of cases 1-3 alone (arrival order), then with filters of tenant "pad" mixed in (locality order)
    -> (shared, padded, position of shared[i] in padded)"""
    rng = random.Random(5)
    pool = []
    for case in ("wide", "dollar", "long"):
        pool += CASES[case]()[1]
    shared = [pool[i % len(pool)] for i in range(ORDER_MIN_FILTERS - 1)]
    rng.shuffle(shared)
    padded, pos = [], []
    for f in shared:
        while rng.random() < 0.05:
            padded.append(("pad", rng.choice(["#", "p/+", "p/1", "+/#"])))
        pos.append(len(padded))
        padded.append(f)
    padded += [("pad", "#")] * 40
    return shared, padded, pos


PAD_TOPICS = [("pad", "p/%d" % i) for i in range(30)]


def all_topics():
    out = []
    for case in ("wide", "dollar", "long"):
        out += CASES[case]()[0]
    return out + PAD_TOPICS


# ------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def R():
    import bifromq_b200
    from bifromq_b200 import _native, retain, workload
    bifromq_b200.load_library()

    class NS:
        pass
    ns = NS()
    ns.N, ns.retain, ns.workload = _native, retain, workload
    return ns


def tenants_of(pairs):
    return list(dict.fromkeys(t for t, _ in pairs))


def make_index(R, topics):
    """a fresh handle with the topics added (ids checked against insertion order) and committed -> (idx, entries)"""
    idx = R.retain.GpuTopicMatchIndex(0)
    entries, _ = add(R, idx, topics, {}, 0)
    idx.commit()
    return idx, entries


def add(R, idx, topics, entries, nxt):
    """add topics to the staged index; a new (tenant, topic) must get id nxt, nxt + 1, ... (removed topics keep their id's
    slot, so nxt is the number of ids handed out since the last reset) -> (entries with the new ids, next id)"""
    tenants = tenants_of(topics)
    blob, off = R.N.as_blob([p for _, p in topics])
    tt = np.array([tenants.index(t) for t, _ in topics], np.int32)
    got = idx.add_blobs(tenants, blob, off, tt).tolist()
    out = dict(entries)
    for k, i in zip(topics, got):
        if k not in out:
            assert i == nxt
            out[k] = nxt
            nxt += 1
        assert out[k] == i
    return out, nxt


def run(R, idx, filters, limit=None, tenants=None):
    tenants = tenants or tenants_of(filters) or ["t"]
    blob, off = R.N.as_blob([f for _, f in filters])
    ft = np.array([tenants.index(t) for t, _ in filters] or [0], np.int32)
    return idx.match_blobs(tenants, blob, off, ft, limit)


class Expect:
    """the oracle's answer and the model's counts for a topic set, per distinct (tenant, filter)"""

    def __init__(self, entries):
        self.entries = entries
        self.tenant_of = {i: t for (t, _), i in entries.items()}
        self.model, self.orc = TrieModel(entries), oracle_of(entries)
        self.memo = {}

    def __call__(self, t, f):
        if (t, f) not in self.memo:
            mf, rg, ids = self.model.walk(t, f)
            want = self.orc.match(f, t)
            assert sorted(ids) == want, (t, f)
            self.memo[(t, f)] = (want, len(rg), mf > R_FR_CAP or len(rg) > R_RG_CAP, rg, ids)
        return self.memo[(t, f)]


def check(res, exp, filters):
    """the whole answer against the oracle, and the path counts against the model -> (tier-2 filters, ranges)"""
    assert res.n_filters == len(filters)
    assert res.offsets[0] == 0 and len(res.offsets) == len(filters) + 1
    n_ovf = n_rg = 0
    for i, (t, f) in enumerate(filters):
        want, nr, ovf, _, _ = exp(t, f)
        got = res.matches(i).tolist()
        assert len(set(got)) == len(got), (t, f)
        assert sorted(got) == want, (t, f)
        assert all(exp.tenant_of[x] == t for x in got), (t, f)   # never a neighbouring tenant's topic
        assert int(res.totals[i]) == len(want), (t, f)
        n_ovf += ovf
        n_rg += nr
    assert res.offsets[-1] == len(res.ids)
    assert res.n_overflow_filters == n_ovf and res.n_ranges == n_rg
    return n_ovf, n_rg


# ------------------------------------------------------------------ GPU: tier-1 limits, '$' at level 0, long filters
@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_case_exact_with_path_counts(R, case):
    topics, filters = CASES[case]()
    idx, entries = make_index(R, topics)
    exp = Expect(entries)
    n_ovf, n_rg = check(run(R, idx, filters), exp, filters)
    if case == "wide":
        assert 0 < n_ovf < len(filters)               # tier 1 and tier 2 side by side in one batch
    elif case == "long_tier2":
        assert n_ovf == len(filters)
    else:
        assert n_ovf == 0
    # every filter alone: the same answer and counts as inside the batch
    for t, f in filters[::7]:
        check(run(R, idx, [(t, f)]), exp, [(t, f)])


@pytest.mark.gpu
def test_tier1_limits_one_filter_per_call(R):
    topics, filters = wide_case()
    idx, entries = make_index(R, topics)
    exp = Expect(entries)
    for w in WIDTHS:
        for sys in (False, True):
            t = wide_tenant(w, sys)
            for f in ("+/x/y/z", "+/x", "+/x/#", "+/+/#", "+/x/y", "+/+"):
                res = run(R, idx, [(t, f)])
                n_ovf, _ = check(res, exp, [(t, f)])
                assert n_ovf == (w > 64 and f != "+/+"), (t, f)


# ------------------------------------------------------------------ GPU: locality order
@pytest.mark.gpu
def test_locality_order_gives_the_arrival_order_answer(R):
    idx, entries = make_index(R, all_topics())
    exp = Expect(entries)
    shared, padded, pos = locality_batches()
    a = run(R, idx, shared)
    b = run(R, idx, padded)
    check(a, exp, shared)
    check(b, exp, padded)
    for i, p in enumerate(pos):
        assert a.matches(i).tolist() == b.matches(p).tolist(), shared[i]


@pytest.mark.gpu
def test_c5_scaled_through_locality_order(R):
    w = R.workload.Workload("C5", scale=0.05)
    assert w.n_query_filters >= ORDER_MIN_FILTERS
    idx = R.retain.GpuTopicMatchIndex(0)
    tenants = w.tenants
    ids = idx.add_blobs(tenants, w.topics, w.topic_off, w.topic_tenant[:w.n_topics])
    idx.commit()
    orc = O.TopicLevelIndex()
    tl = w.topic_list()
    for i in range(w.n_topics):
        orc.add(tl[i], int(ids[i]), tenants[w.topic_tenant[i]])
    ft = w.filter_tenant[:w.n_query_filters]
    res = idx.match_blobs(tenants, w.filters, w.filter_off, ft)
    fl = w.query_filter_list()
    hits = 0
    for i in range(w.n_query_filters):
        want = orc.match(fl[i], tenants[ft[i]])
        got = res.matches(i).tolist()
        assert sorted(got) == want and len(set(got)) == len(got)
        assert int(res.totals[i]) == len(want)
        hits += bool(want)
    assert hits > 0.5 * w.n_query_filters
    lim = np.full(w.n_query_filters, 10, np.int64)
    res10 = idx.match_blobs(tenants, w.filters, w.filter_off, ft, lim)
    assert res10.totals.tolist() == res.totals.tolist()
    for i in range(w.n_query_filters):
        assert res10.matches(i).tolist() == res.matches(i).tolist()[:10]


# ------------------------------------------------------------------ GPU: range-buffer re-run
@pytest.mark.gpu
@pytest.mark.parametrize("w", [64, 65])
def test_range_buffer_rerun(R, w):
    """a fresh handle's range buffer holds max(2^18, 8n) ranges: 4200 filters of w ranges each overflow it; at w = 65 every
    filter goes to tier 2, on the first attempt and on the re-run"""
    topics, filters = rerun_case(w)
    idx, entries = make_index(R, topics)
    exp = Expect(entries)
    res = run(R, idx, filters)
    n_ovf, n_rg = check(res, exp, filters)
    assert n_rg == w * len(filters) and res.n_ranges > initial_range_cap(len(filters))
    assert n_ovf == (len(filters) if w > 64 else 0)
    again = run(R, idx, filters)
    assert again.offsets.tolist() == res.offsets.tolist() and again.ids.tolist() == res.ids.tolist()


# ------------------------------------------------------------------ GPU: limits
LIMIT_KINDS = ["-1", "-2^63", "0", "1", "total-1", "total", "total+1", "2^62", "range0", "range0+1"]


def limits_for(kind, totals, first_range):
    out = []
    for t, r0 in zip(totals, first_range):
        out.append({"-1": -1, "-2^63": -2 ** 63, "0": 0, "1": 1, "total-1": t - 1, "total": t, "total+1": t + 1,
                    "2^62": 2 ** 62, "range0": r0, "range0+1": r0 + 1}[kind])
    return np.array(out, np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(CASES))
def test_limits_keep_a_prefix_of_the_unlimited_answer(R, case):
    """a limit keeps the first min(total, limit) ids of the unlimited answer of the same batch; the totals do not change.
    "range0" cuts at the end of a filter's first range (a range boundary), "range0+1" one id into its second, "1" / "total-1"
    inside a range. A filter's ranges share one rank space (they all come from its last level), so the DFS / BFS change
    happens between filters of the batch."""
    topics, filters = CASES[case]()
    idx, entries = make_index(R, topics)
    exp = Expect(entries)
    full = run(R, idx, filters)
    check(full, exp, filters)
    totals = full.totals.tolist()
    first_range = [exp(t, f)[3][0][2] if exp(t, f)[3] else 0 for t, f in filters]
    multi = 0
    for i, (t, f) in enumerate(filters):
        rg, ids = exp(t, f)[3], exp(t, f)[4]
        if len(rg) > 1:
            # the cut of "range0" lands on the boundary between the first and second range
            assert set(full.matches(i).tolist()[:rg[0][2]]) == set(ids[:rg[0][2]]), (t, f)
            multi += 1
    assert multi > 5
    spaces = [exp(t, f)[3][0][0] for t, f in filters if exp(t, f)[3]]
    assert DFS in spaces and BFS in spaces
    for kind in LIMIT_KINDS:
        lim = limits_for(kind, totals, first_range)
        res = run(R, idx, filters, lim)
        assert res.totals.tolist() == totals, kind
        for i in range(len(filters)):
            k = totals[i] if lim[i] < 0 else min(totals[i], int(lim[i]))
            assert res.matches(i).tolist() == full.matches(i).tolist()[:k], (kind, filters[i])


# ------------------------------------------------------------------ GPU: index lifecycle
@pytest.mark.gpu
def test_index_lifecycle(R):
    topics, filters = dollar_case()
    wt, wf = wide_case()
    topics, filters = topics + wt[:200], filters + wf
    idx = R.retain.GpuTopicMatchIndex(0)
    half = len(topics) // 2
    entries, nxt = add(R, idx, topics[:half], {}, 0)
    idx.commit()
    check(run(R, idx, filters), Expect(entries), filters)
    entries, nxt = add(R, idx, topics[half:], entries, nxt)  # grow
    idx.commit()
    check(run(R, idx, filters), Expect(entries), filters)
    gone = [k for k, i in entries.items() if i % 4 != 1]    # shrink: remove three in four
    for t, p in gone:
        idx.remove(t, p)
    live = {k: i for k, i in entries.items() if i % 4 == 1}
    idx.commit()
    check(run(R, idx, filters), Expect(live), filters)
    back, _ = add(R, idx, gone, live, nxt)                  # re-added topics get new ids
    assert min(back[k] for k in gone) == len(entries)
    idx.commit()
    check(run(R, idx, filters), Expect(back), filters)
    idx.reset()                                             # an empty snapshot: every filter matches nothing
    idx.commit()
    res = run(R, idx, filters)
    assert res.offsets.tolist() == [0] * (len(filters) + 1) and res.totals.tolist() == [0] * len(filters)
    assert len(res.ids) == 0 and res.n_ranges == 0 and res.n_overflow_filters == 0
    entries, _ = add(R, idx, topics, {}, 0)                 # ids restart at 0 after a reset
    assert sorted(entries.values()) == list(range(len(entries)))
    idx.commit()
    exp = Expect(entries)
    # the batch's tenant list in another order than the adds, with a repeated name and tenants the index does not hold
    tenants = ["nobody", "d_sys", "w64s", "d_mix", "d_lo", "d_mix", "", "d_hi", "w63", "w65s", "w64", "w63s", "w65"]
    rng = random.Random(11)
    picks = [(rng.randrange(len(tenants)), f) for _, f in filters]
    res = idx.match_blobs(tenants, *R.N.as_blob([f for _, f in picks]), np.array([t for t, _ in picks], np.int32))
    check(res, exp, [(tenants[t], f) for t, f in picks])
    empty = run(R, idx, [], tenants=["d_mix"])              # an empty batch
    assert empty.n_filters == 0 and empty.offsets.tolist() == [0] and len(empty.ids) == 0


# ------------------------------------------------------------------ GPU: retain keys pin the snapshot's id table
def _raw_match(N, h, tenant, filters):
    tb, toff = N.as_blob([tenant])
    fb, foff = N.as_blob(filters)
    ft = np.zeros(len(filters), np.int32)
    r = C.c_void_p()
    N.check(N.lib.bfq_rmatch(h, N.ptr(tb), N.ptr(toff), 1, N.ptr(fb), N.ptr(foff), N.ptr(ft), len(filters), None, C.byref(r)))
    return r


def _raw_ids(N, r):
    n = C.c_int64(0)
    p = N.lib.bfq_rresult_ids(r, C.byref(n))
    return np.frombuffer((C.c_uint8 * (n.value * 8)).from_address(p), np.int64).tolist() if n.value else []


def _raw_keys(N, h, r):
    n = len(_raw_ids(N, r))
    koff = np.zeros(n + 1, np.int64)
    total = N.lib.bfq_rresult_retain_keys(h, r, None, 0, koff.ctypes.data)
    assert total >= 0, total
    blob = np.zeros(max(total, 1), np.uint8)
    assert N.lib.bfq_rresult_retain_keys(h, r, blob.ctypes.data, total, koff.ctypes.data) == total
    return [bytes(blob[koff[j]:koff[j + 1]]) for j in range(n)]


def _raw_load(N, h, pairs):
    kb, ko = N.as_blob([O.retain_key(t, p) for t, p in pairs])
    ids = np.zeros(len(pairs), np.int64)
    N.check(N.lib.bfq_rindex_load_keys(h, N.ptr(kb), N.ptr(ko), len(pairs), ids.ctypes.data))
    return ids.tolist()


@pytest.mark.gpu
def test_retain_keys_resolve_against_the_snapshot_of_the_result(R):
    """bfq_rindex_reset restarts ids at 0; a reload of as many other topics reuses every id. A result taken before the reset,
    and a match run between the reset and the next commit, still get the retain keys of the topics they matched."""
    N = R.N
    lib = N.lib
    old = [("t", "old/%d" % i) for i in range(6)]
    new = [("t", "new/%d" % i) for i in range(6)]
    h = C.c_void_p()
    N.check(lib.bfq_rindex_create(0, C.byref(h)))
    results = []
    try:
        assert _raw_load(N, h, old) == list(range(6))
        N.check(lib.bfq_rindex_commit(h))
        r1 = _raw_match(N, h, "t", ["#"])
        results.append(r1)
        ids1 = _raw_ids(N, r1)
        assert sorted(ids1) == list(range(6))
        want1 = [O.retain_key(*old[i]) for i in ids1]
        assert _raw_keys(N, h, r1) == want1
        N.check(lib.bfq_rindex_reset(h))
        assert _raw_load(N, h, new) == list(range(6))   # every id now names another topic in staging
        assert _raw_keys(N, h, r1) == want1              # a result taken before the reset
        r2 = _raw_match(N, h, "t", ["old/+", "new/+"])   # between the reset and the commit: the committed snapshot
        results.append(r2)
        ids2 = _raw_ids(N, r2)
        assert sorted(ids2) == list(range(6))
        assert _raw_keys(N, h, r2) == [O.retain_key(*old[i]) for i in ids2]
        # bfq_rindex_lookup resolves against staging
        tl, pl = C.c_int64(0), C.c_int64(0)
        tb, pb = C.create_string_buffer(16), C.create_string_buffer(16)
        N.check(lib.bfq_rindex_lookup(h, 0, C.addressof(tb), 16, C.byref(tl), C.addressof(pb), 16, C.byref(pl)))
        assert pb.raw[:pl.value] == b"new/0"
        N.check(lib.bfq_rindex_commit(h))
        r3 = _raw_match(N, h, "t", ["#", "old/+"])
        results.append(r3)
        ids3 = _raw_ids(N, r3)
        assert sorted(ids3) == list(range(6))
        assert _raw_keys(N, h, r3) == [O.retain_key(*new[i]) for i in ids3]
        assert _raw_keys(N, h, r1) == want1 and _raw_keys(N, h, r2) == [O.retain_key(*old[i]) for i in ids2]
    finally:
        for r in results:
            lib.bfq_rresult_free(r)
        lib.bfq_rindex_destroy(h)
