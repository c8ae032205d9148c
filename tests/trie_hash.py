"""A plain restatement of the forward trie's child lookup hashes (bifromq_b200/csrc/trie_layout.h) and of the builder's choice of
lookup per node (index_builder.cc, build_tenant), with searches for level names that land on the lookups' edges. No GPU, no
native code: the tests compare it with the builder's image (tests/native/image_walk_harness.cc --dump) and then use it to place
keys where a lookup can go wrong.

Edge keys: a level of at most 24 bytes is one edge (length word = its byte length, 6 little-endian token words, zero padded);
a longer level is a chain of 24-byte chunks with length words LEN_CONT | j, then its last chunk with the level's full length.
Every search here is seeded, so a test sees the same names on every run."""
import numpy as np

M64 = (1 << 64) - 1
TOKC = [0x9E3779B97F4A7C15, 0xA24BAED4963EE407, 0x9FB21C651E98DF25, 0xD6E8FEB86659FD93, 0xCA5A826395121157, 0x8CB92BA72F3D8DD7,
        0xE7037ED1A0B428DB]
ROOT_BASE = 0x80000000
LEN_CONT = 0x80000000
TOKEN_BYTES = 24
BLOCK_SLOTS, BLOCK_USABLE, TAG_CTRL = 16, 15, 15
PERFECT_LOG2_MAX = 16
ALPHA = np.frombuffer(b"abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789", np.uint8)

_U = np.uint64


# ------------------------------------------------------------------ the hashes, scalar (Python ints)
def fmix64(k):
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & M64
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & M64
    return k ^ (k >> 33)


def token_words(chunk):
    b = chunk.encode() if isinstance(chunk, str) else bytes(chunk)
    assert len(b) <= TOKEN_BYTES
    return [int(x) for x in np.frombuffer(b.ljust(TOKEN_BYTES, b"\0"), "<u4")]


def token_hash(lenw, words):
    return (lenw * TOKC[0] + sum(w * c for w, c in zip(words, TOKC[1:]))) & M64


def fold32(tokh):
    return (tokh ^ (tokh >> 32)) & 0xFFFFFFFF


def child_index(t32, seed, lg):
    return ((((t32 ^ ((seed * 0x9E3779B9) & 0xFFFFFFFF)) * 0x85EBCA6B) & 0xFFFFFFFF) >> (32 - lg))


def edge_hash(tokh, parent):
    return fmix64((tokh + parent * 0xC2B2AE3D27D4EB4F) & M64)


def home_block(h, n_blocks):
    return ((h >> 32) * n_blocks) >> 32


def fingerprint(h):
    f = h & 0xFF
    return f + 2 if f < 2 else f


def chunks(level):
    """the edges of one level: [(lenw, chunk bytes)], continuation chunks first"""
    b = level.encode() if isinstance(level, str) else bytes(level)
    out = []
    j = 0
    while len(b) - 24 * j > TOKEN_BYTES:
        out.append((LEN_CONT | j, b[24 * j:24 * j + 24]))
        j += 1
    out.append((len(b), b[24 * j:]))
    return out


def edge_tokh(lenw, chunk):
    return token_hash(lenw, token_words(chunk))


def edge_fold(lenw, chunk):
    return fold32(edge_tokh(lenw, chunk))


def edge_place(lenw, chunk, parent, n_blocks):
    """(home block, fingerprint) of the edge in the shared tag table"""
    h = edge_hash(edge_tokh(lenw, chunk), parent)
    return home_block(h, n_blocks), fingerprint(h)


def n_blocks_for(n_edges):
    """blocks of the table a full build makes for n_edges wide edges (load 0.5, at least 64 blocks)"""
    return max(64, (2 * n_edges + BLOCK_USABLE - 1) // BLOCK_USABLE)


# ------------------------------------------------------------------ the node-kind rule
def plan(folds, perfect_max=PERFECT_LOG2_MAX):
    """the builder's lookup for a node whose exact children have these 32-bit folds:
    ("single", 0, fingerprint) | ("perfect", lg, seed) | ("big", 0, 0)"""
    c = len(folds)
    assert c >= 1
    if c == 1:
        return ("single", 0, folds[0] & 0xFFFF)
    if len(set(folds)) < c:
        return ("big", 0, 0)   # two children with one fold: no seed can separate them
    lg = 1
    while (1 << lg) < c:
        lg += 1
    if c > 4:
        lg += 1
    while lg <= perfect_max and (c * c) // 16 > (1 << lg):
        lg += 1
    t32 = np.asarray(folds, np.uint64)
    while lg <= perfect_max:
        # the first seed whose c child indices are distinct, 1024 seeds at a time
        for s0 in range(0, 65536, 1024):
            seeds = np.arange(s0, s0 + 1024, dtype=np.uint64)
            x = (t32[None, :] ^ ((seeds[:, None] * _U(0x9E3779B9)) & _U(0xFFFFFFFF))) * _U(0x85EBCA6B)
            idx = np.sort((x & _U(0xFFFFFFFF)) >> _U(32 - lg), axis=1)
            ok = np.flatnonzero(~(idx[:, 1:] == idx[:, :-1]).any(axis=1))
            if len(ok):
                return ("perfect", lg, s0 + int(ok[0]))
        lg += 1
    return ("big", 0, 0)


# ------------------------------------------------------------------ the trie the builder makes, and its claim order
def inner_filter(tf):
    for pfx in ("$share/", "$oshare/"):
        if tf.startswith(pfx):
            return tf.split("/", 2)[2]
    return tf


class Trie:
    """the chunked filter trie of every tenant, nodes numbered in the order the sorted-order construction creates them (the
    order of the first route key that reaches each node). A node is (tenant, path of edges); an edge is (lenw, chunk) or "+"."""

    def __init__(self, pairs):
        from bifromq_b200 import schema
        self.children = {}      # node -> [exact child edge] in creation order
        self.nodes = set()
        self.tenants = []       # in key order: ordinal = index
        for k, v in sorted(pairs):
            m = schema.build_match_route(k, v)
            if not self.tenants or self.tenants[-1] != m.tenant_id:
                self.tenants.append(m.tenant_id)
            levels = inner_filter(m.mqtt_topic_filter).split("/")
            if levels[-1] == "#":
                levels = levels[:-1]
            node = (m.tenant_id,)
            self.nodes.add(node)
            for lv in levels:
                if lv == "+":
                    node = node + ("+",)
                else:
                    for e in chunks(lv):
                        cs = self.children.setdefault(node, [])
                        if e not in cs:
                            cs.append(e)
                        node = node + (e,)
                self.nodes.add(node)

    def plans(self, perfect_max=PERFECT_LOG2_MAX):
        return {n: plan([edge_fold(*e) for e in cs], perfect_max) for n, cs in self.children.items()}

    def big_edges(self, perfect_max=PERFECT_LOG2_MAX):
        """the wide edges of every tenant in the order its placement claims them: breadth first from the root, a node's '+'
        child queued before its exact children, exact children in creation order -> {tenant: [node path of the child]}"""
        pl = self.plans(perfect_max)
        out = {}
        for t in self.tenants:
            order, qi = [(t,)], 0
            edges = out.setdefault(t, [])
            while qi < len(order):
                n = order[qi]
                qi += 1
                if n + ("+",) in self.nodes:
                    order.append(n + ("+",))
                for e in self.children.get(n, []):
                    if pl[n][0] == "big":
                        edges.append(n + (e,))
                    order.append(n + (e,))
        return out


# ------------------------------------------------------------------ the shared tag table
class TagTable:
    """the tag table of trie_layout.h (EdgeTable.claim / release / find), byte for byte: which slot each key claims, its tag,
    and the control bytes of the blocks it walked past"""

    def __init__(self, n_blocks):
        self.n_blocks = n_blocks
        self.tags = np.zeros((n_blocks, 16), np.uint8)
        self.keys = {}   # slot -> (parent, lenw, chunk)

    def claim(self, parent, lenw, chunk):
        """-> (slot, blocks walked past); every full block on the way gets its control byte"""
        b, fp = edge_place(lenw, chunk, parent, self.n_blocks)
        walked = 0
        while True:
            free = np.flatnonzero(self.tags[b, :BLOCK_USABLE] == 0)
            if len(free):
                s = b * BLOCK_SLOTS + int(free[0])
                self.tags[b, free[0]] = fp
                self.keys[s] = (parent, lenw, bytes(chunk))
                return s, walked
            self.tags[b, TAG_CTRL] = 1
            walked += 1
            b = b + 1 if b + 1 < self.n_blocks else 0

    def release(self, slot):
        self.tags[slot // BLOCK_SLOTS, slot % BLOCK_SLOTS] = 0
        self.keys.pop(slot, None)

    def probe(self, parent, lenw, chunk):
        """the lookup: -> (slot or None, [(block, [candidate slots tried])])"""
        b, fp = edge_place(lenw, chunk, parent, self.n_blocks)
        path = []
        while True:
            cands = [b * BLOCK_SLOTS + int(j) for j in np.flatnonzero(self.tags[b, :BLOCK_USABLE] == fp)]
            path.append((b, cands))
            for s in cands:
                if self.keys.get(s) == (parent, lenw, bytes(chunk)):
                    return s, path
            if self.tags[b, TAG_CTRL] == 0:
                return None, path
            b = b + 1 if b + 1 < self.n_blocks else 0

    def claimed(self):
        return int((self.tags[:, :BLOCK_USABLE] != 0).sum())

    def overflowed(self):
        return int((self.tags[:, TAG_CTRL] != 0).sum())


def level_home_block(level, parent, n_blocks):
    """home block of a level of <= 24 bytes under `parent`"""
    (lenw, chunk), = chunks(level)
    return edge_place(lenw, chunk, parent, n_blocks)[0]


class TagModel(TagTable):
    """the table of an index whose only wide node is one tenant's root: its children claim slots in key order (same-length
    names: key order == sorted order). A delta commit frees all of the tenant's slots first, so it re-places them into an empty
    table whose control bytes stay as they were. The GPU tests predict the path of every commit at the table's bounds from it."""

    def __init__(self, n_edges):
        super().__init__(n_blocks_for(n_edges))
        self.usable = BLOCK_USABLE * self.n_blocks
        self.overflowed = set()

    def place(self, names, ordinal):
        """the tenant's root children, into a table whose slots are all free; -> the overflowed block count (the overflowed blocks
        of earlier placements included)"""
        if self.tags.shape[0] != self.n_blocks:   # a caller may resize the table by setting n_blocks
            self.tags = np.zeros((self.n_blocks, 16), np.uint8)
        self.tags[:, :BLOCK_USABLE] = 0
        self.keys.clear()
        for nm in sorted(names):
            (lenw, chunk), = chunks(nm)
            self.claim(ROOT_BASE + ordinal, lenw, chunk)
        self.overflowed |= set(np.flatnonzero(self.tags[:, TAG_CTRL]).tolist())
        return len(self.overflowed)

    def path(self, n_edges, overflowed):
        """the path the delta rules give a commit that leaves n_edges claimed and `overflowed` blocks overflowed"""
        return "full" if 4 * n_edges > 3 * self.usable or 4 * overflowed > self.n_blocks else "delta"


# ------------------------------------------------------------------ searches (numpy, fixed seeds)
def _random_names(rng, n, length, prefix=b""):
    body = ALPHA[rng.integers(0, len(ALPHA), size=(n, length - len(prefix)))]
    if prefix:
        body = np.concatenate([np.tile(np.frombuffer(prefix, np.uint8), (n, 1)), body], axis=1)
    return body


def _words(names):
    """(n, L <= 24) uint8 -> (n, 6) uint64 token words"""
    n, L = names.shape
    pad = np.zeros((n, TOKEN_BYTES), np.uint8)
    pad[:, :L] = names
    return pad.view("<u4").astype(np.uint64)


def _tokh(lenw, words):
    h = np.full(len(words), (lenw * TOKC[0]) & M64, np.uint64)
    for j in range(6):
        h = h + words[:, j] * _U(TOKC[j + 1])
    return h


def _fmix(k):
    k = k ^ (k >> _U(33))
    k = k * _U(0xff51afd7ed558ccd)
    k = k ^ (k >> _U(33))
    k = k * _U(0xc4ceb9fe1a85ec53)
    return k ^ (k >> _U(33))


def _place(tokh, parent, n_blocks):
    h = _fmix(tokh + _U((parent * 0xC2B2AE3D27D4EB4F) & M64))
    b = ((h >> _U(32)) * _U(n_blocks)) >> _U(32)
    f = h & _U(0xFF)
    return b.astype(np.int64), np.where(f < 2, f + 2, f).astype(np.int64)


def _fold(tokh):
    return ((tokh ^ (tokh >> _U(32))) & _U(0xFFFFFFFF)).astype(np.int64)


def _dec(names):
    return [bytes(r).decode() for r in names]


def fold_pairs(n_pairs=2, length=8, seed=1, lenw=None, batch=1 << 18):
    """pairs of distinct names of `length` bytes whose edges (length word `lenw`, default the name's length: the last chunk of a
    level of lenw bytes) have equal 32-bit folds (birthday search)"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n_pairs:
        names = _random_names(rng, batch, length)
        f = _fold(_tokh(length if lenw is None else lenw, _words(names)))
        order = np.argsort(f, kind="stable")
        fs = f[order]
        for i in np.flatnonzero(fs[1:] == fs[:-1]):
            a, b = _dec(names[order[[i, i + 1]]])
            if a != b and len(out) < n_pairs:
                out.append((a, b))
    return out


def names_homed(parent, n_blocks, block, count, fp=None, length=8, prefix="", seed=2, exclude=(), batch=1 << 17):
    """`count` names (of `length` bytes, starting with `prefix`) whose edge under `parent` has the given home block (and
    fingerprint)"""
    rng = np.random.default_rng(seed)
    out, seen = [], set(exclude)
    while len(out) < count:
        names = _random_names(rng, batch, length, prefix.encode())
        b, f = _place(_tokh(length, _words(names)), parent, n_blocks)
        hit = (b == block) if fp is None else (b == block) & (f == fp)
        for nm in _dec(names[hit]):
            if nm not in seen and len(out) < count:
                seen.add(nm)
                out.append(nm)
    return out


def single_child_twin(child, length=8, seed=3, batch=1 << 18):
    """a name other than `child` (a level of <= 24 bytes) whose fold agrees with the child's in its low 16 bits: the single-child
    fingerprint passes it and only the slot compare can reject it"""
    want = edge_fold(*chunks(child)[-1]) & 0xFFFF
    rng = np.random.default_rng(seed)
    while True:
        names = _random_names(rng, batch, length)
        hit = np.flatnonzero((_fold(_tokh(length, _words(names))) & 0xFFFF) == want)
        for nm in _dec(names[hit]):
            if nm != child:
                return nm


def cross_parent_twin(p1, p2, n_blocks, length=8, seed=4, batch=1 << 17):
    """a name whose edges under parents p1 and p2 have the same home block and fingerprint"""
    rng = np.random.default_rng(seed)
    while True:
        names = _random_names(rng, batch, length)
        t = _tokh(length, _words(names))
        b1, f1 = _place(t, p1, n_blocks)
        b2, f2 = _place(t, p2, n_blocks)
        hit = np.flatnonzero((b1 == b2) & (f1 == f2))
        if len(hit):
            return _dec(names[hit[:1]])[0]


def length_twin_suffix(sibling, cont, seed=6, length=8):
    """a name X for a 2-child node below a length twin P, next to `sibling`: the node is P's level ((24, P): children (len X, X)
    and the sibling) or, with `cont`, P's continuation chunk ((LEN_CONT | 0, P): children (24 + len X, X) and the sibling as last
    chunks). X is chosen so that the perfect hash sends X spelled the other way to X's own slot: a walk that took the wrong one
    of the two twins reaches X's record, and only the length word tells the two spellings apart"""
    rng = np.random.default_rng(seed)
    while True:
        x = _dec(_random_names(rng, 1, length))[0]
        own, other = (TOKEN_BYTES + length, length) if cont else (length, TOKEN_BYTES + length)
        kind, lg, sd = plan([edge_fold(own, x.encode()), edge_fold((TOKEN_BYTES if cont else 0) + len(sibling), sibling.encode())])
        if kind == "perfect" and child_index(edge_fold(own, x.encode()), sd, lg) == child_index(edge_fold(other, x.encode()), sd, lg):
            return x


def length_twin(parent, n_blocks, seed=5, batch=1 << 17, prefix=""):
    """a 24-byte name P whose edges (24, P) and (LEN_CONT | 0, P) under `parent` have the same home block and fingerprint: the
    level P and the first chunk of any longer level starting with P differ in their length word alone"""
    rng = np.random.default_rng(seed)
    while True:
        names = _random_names(rng, batch, TOKEN_BYTES, prefix.encode())
        w = _words(names)
        b1, f1 = _place(_tokh(TOKEN_BYTES, w), parent, n_blocks)
        b2, f2 = _place(_tokh(LEN_CONT, w), parent, n_blocks)
        hit = np.flatnonzero((b1 == b2) & (f1 == f2))
        if len(hit):
            return _dec(names[hit[:1]])[0]
