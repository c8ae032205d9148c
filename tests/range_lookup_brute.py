"""A brute-force TenantRangeLookupCache.lookup in plain Python, and the case generators the range lookup tests share.

The brute force enumerates a topic's whole global expansion set (every filter that matches it, tenant id as level 0), sorts it
level-wise in Java String.compareTo order and answers seek(first) with a bisect. It shares nothing with the oracle's iterator
(oracle/expansion.cc) or with the kernel's walk (bifromq_b200/csrc/range_lookup.cu). The set has about 2^n members for n topic
levels, so it is used up to BRUTE_MAX_LEVELS.

Candidates are what bifromq_b200.dist.range_lookup takes: per range None (no Fact) or (first, last), either of which may be None
(the Fact lacks it); first / last are global filter level lists."""
import bisect

BRUTE_MAX_LEVELS = 13

# one level name from each band of the order around the wildcards "#" (0x23) and "+" (0x2B): below "#", "#"-prefixed, between
# the two, "+"-prefixed, above "+" in ASCII, DEL, and two- and three-byte BMP text (U+FF5E sorts last in UTF-8 and in UTF-16)
ORDER_VOCAB = ["", " ", "!", "\"", "#a", "#", "$", "$s", "%", "&", "'", "(", ")", "*", "+b", "+", ",", "0", "9", "A", "a", "ab",
               "z", "~", "\x7f", "é", "中", "～"]
# what an MQTT topic level can be: no wildcard level
TOPIC_VOCAB = [v for v in ORDER_VOCAB if v not in ("#", "+")]
APPENDED = ["", "!", "#", "+", "~"]
TENANT = "tB"
TENANT_VARIANTS = ["tA", "tB", "tC", "t", "tB!", "tBa"]   # smaller, equal, greater, a prefix of, extended from TENANT


def java_key(levels):
    """level-wise String.compareTo, shorter prefix first: UTF-16 code units compare like big-endian UTF-16 bytes"""
    return tuple(lv.encode("utf-16-be", "surrogatepass") for lv in levels)


def java_joined(levels):
    return "\0".join(levels).encode("utf-16-be", "surrogatepass")


def expansion_set(tenant, topic):
    """every global filter matching `topic`: the tenant level, then per level the topic's level or "+", ending at full length
    or in "#" (which matches the parent level too); no "+" / "#" right under the tenant level when the topic starts with '$'"""
    t = topic.split("/")
    assert len(t) <= BRUTE_MAX_LEVELS, len(t)
    sys_topic = t[0].startswith("$")
    out = set()

    def walk(i, pre):
        wild = not (i == 0 and sys_topic)
        if wild:
            out.add(pre + ("#",))
        if i == len(t):
            out.add(pre)
            return
        walk(i + 1, pre + (t[i],))
        if wild:
            walk(i + 1, pre + ("+",))
    walk(0, (tenant,))
    return sorted(out, key=java_key)


class Brute:
    def __init__(self, tenant, topic):
        self.members = expansion_set(tenant, topic)
        self.keys = [java_key(m) for m in self.members]

    def seek(self, first):
        """least member >= first, or None"""
        i = bisect.bisect_left(self.keys, java_key(first))
        return self.members[i] if i < len(self.members) else None

    def lookup(self, candidates):
        """TenantRangeLookupCache.java:77-103 literally: kept candidate indices"""
        kept = []
        for k, c in enumerate(candidates):
            if c is None:                       # no Fact: kept
                kept.append(k)
                continue
            first, last = c
            if first is None or last is None:   # the range is empty
                continue
            found = self.seek(first)
            if found is None:                   # nothing >= first: later ranges are not looked at
                break
            if list(found) == list(first) or java_joined(found) <= java_joined(last):
                kept.append(k)
        return kept


_BRUTES = {}


def brute(tenant, topic):
    key = (tenant, topic)
    if key not in _BRUTES:
        if len(_BRUTES) > 4096:
            _BRUTES.clear()
        _BRUTES[key] = Brute(tenant, topic)
    return _BRUTES[key]


def brute_lookup(tenant, topic, candidates):
    return brute(tenant, topic).lookup(candidates)


def classify(tenant, topic, first, last):
    """what one candidate (first, last) does on its own: "keep", "drop" or "stop" """
    kept = brute(tenant, topic).lookup([(first, last)])
    if kept:
        return "keep"
    return "stop" if brute(tenant, topic).seek(first) is None else "drop"


# ------------------------------------------------------------------ generators
def order_topics(rng, count, max_levels, sys_share=0.15):
    """topics whose levels mix every band of ORDER_VOCAB; some start with '$'"""
    out = []
    for _ in range(count):
        levels = [rng.choice(TOPIC_VOCAB) for _ in range(rng.randint(1, max_levels))]
        if rng.random() < sys_share:
            levels[0] = rng.choice(["$", "$s", "$sys"])
        out.append("/".join(levels))
    return out


_SORTED_VOCAB = sorted(set(ORDER_VOCAB), key=lambda v: java_key([v]))
_SORTED_KEYS = [java_key([v]) for v in _SORTED_VOCAB]


def neighbours(name):
    """names just below and just above `name` in level order: its vocabulary neighbours, its prefix one character shorter and
    the name with one more (low) byte"""
    k = java_key([name])
    lo, hi = bisect.bisect_left(_SORTED_KEYS, k), bisect.bisect_right(_SORTED_KEYS, k)
    out = {name + "\x01"}
    if lo > 0:
        out.add(_SORTED_VOCAB[lo - 1])
    if hi < len(_SORTED_VOCAB):
        out.add(_SORTED_VOCAB[hi])
    if name:
        out.add(name[:-1])
    out.discard(name)
    return sorted(out, key=lambda v: java_key([v]))


def derived_bounds(topic, tenant=TENANT):
    """bounds built systematically from the topic's own members: every member; each with its last level dropped or one level
    (APPENDED) added; each with one level (tenant level included) replaced by a neighbour; each member under every tenant
    variant. Returned in Java level order, without duplicates."""
    out = set()
    for m in brute(tenant, topic).members:
        m = list(m)
        out.add(tuple(m))
        if len(m) > 1:
            out.add(tuple(m[:-1]))
        for a in APPENDED:
            out.add(tuple(m + [a]))
        for j in range(1, len(m)):
            for nb in neighbours(m[j]):
                out.add(tuple(m[:j] + [nb] + m[j + 1:]))
        for tv in TENANT_VARIANTS:
            out.add(tuple([tv] + m[1:]))
    return [list(b) for b in sorted(out, key=java_key)]


def bound_pairs(bounds):
    """(first, last) with last <, = and > first: each bound paired with itself and its neighbours in level order"""
    pairs = []
    for i, b in enumerate(bounds):
        pairs.append((b, b))
        if i > 0:
            pairs.append((b, bounds[i - 1]))
        if i + 1 < len(bounds):
            pairs.append((b, bounds[i + 1]))
        if i + 5 < len(bounds):
            pairs.append((b, bounds[i + 5]))
    return pairs


def tight_path_bounds(topic, tenant=TENANT):
    """for each depth d: a bound that follows the topic for d levels and then leaves it just below and just above its
    level d + 1 (or, past the last level, just below and above "#"), so the seek falls back from every depth"""
    t = topic.split("/")
    out = []
    for d in range(len(t) + 1):
        here = t[d] if d < len(t) else "#"
        for nb in neighbours(here):
            out.append((d, [tenant] + t[:d] + [nb]))
    return out


# the depths the kernel is driven to: topics of these many levels, and bounds of the tenant level plus these many levels (an
# earlier kernel kept 34 levels per topic and per bound, tenant level included)
DEPTH_TOPIC_LEVELS = [1, 16, 33, 34, 35, 64, 65, 200, 2000]
DEPTH_BOUND_LEVELS = [33, 34, 35, 200]


def deep_topic(n_levels, seed=0):
    """n_levels levels, drawn so the seek meets levels that sort below "#" ("", "!") deep down as well as ordinary ones"""
    import random
    rng = random.Random(seed * 7919 + n_levels)
    return "/".join(rng.choice(["a", "b", "", "!", "zz", "#x"]) for _ in range(n_levels))


def long_topic(max_bytes=65535):
    """one topic near MaxTopicLength made of empty and one-byte levels (about 2 levels per 3 bytes)"""
    levels, size = [], -1
    i = 0
    while True:
        lv = "" if i % 3 == 1 else "ab"[i % 2]
        if size + 1 + len(lv) > max_bytes:
            break
        levels.append(lv)
        size += 1 + len(lv)
        i += 1
    return "/".join(levels)


def depth_bounds(topic, tenant, n_bound_levels):
    """bounds of tenant + n_bound_levels levels around `topic`: its own prefix (or the topic followed by "" levels), that
    prefix ending in "#", and the prefix with its last level raised or lowered"""
    t = topic.split("/")
    body = (t + [""] * n_bound_levels)[:n_bound_levels]
    b = [tenant] + body
    return [b, b[:-1] + ["#"], b[:-1] + [b[-1] + "\x01"], b[:-1] + ["" if b[-1] else "~"], b[:-1] + ["+"]]


POOL_KINDS = ("keep", "drop", "stop")


def candidate_pools(tenant, topic):
    """single candidates sorted by what they do on their own: keep / drop / stop (brute force)"""
    pools = {k: [] for k in POOL_KINDS}
    for first, last in bound_pairs(derived_bounds(topic, tenant)):
        pools[classify(tenant, topic, first, last)].append((first, last))
    return pools


def chain_from_pattern(rng, pools, pattern):
    """K keep, D drop, S stop, N no Fact, F Fact without first, L without last, B without both"""
    out = []
    for ch in pattern:
        if ch == "N":
            out.append(None)
        elif ch in "FLB":
            first, last = rng.choice(pools["keep"])
            out.append((None if ch in "FB" else first, None if ch in "LB" else last))
        else:
            out.append(rng.choice(pools[{"K": "keep", "D": "drop", "S": "stop"}[ch]]))
    return out


CHAIN_PATTERNS = ["", "K", "S", "D", "N", "F", "L", "B", "KD", "SK", "SN", "NS", "NSN", "SNNK", "KKS", "KDKDS",
                  "NFLBKDS", "KNDSKN", "BS", "SS", "DKNFLBNKD"]


# ------------------------------------------------------------------ real route sets
def inner_filter(tf):
    for pfx in ("$share/", "$oshare/"):
        if tf.startswith(pfx):
            return tf.split("/", 2)[2]
    return tf


def tenant_filters(w):
    """tenant -> its distinct global filter level lists (routes of shared subscriptions by their inner filter), in Java level
    order"""
    from bifromq_b200 import schema
    kb, vb = w.keys.tobytes(), w.vals.tobytes()
    per = {}
    for i in range(w.n_routes):
        m = schema.build_match_route(kb[w.key_off[i]:w.key_off[i + 1]], vb[w.val_off[i]:w.val_off[i + 1]])
        per.setdefault(m.tenant_id, set()).add((m.tenant_id,) + tuple(inner_filter(m.mqtt_topic_filter).split("/")))
    return {t: sorted(fs, key=java_key) for t, fs in per.items()}


def cut_ranges(filters, k):
    """k contiguous ranges of a sorted filter list (fewer if there are fewer filters): (first, last, filters in the range)"""
    k = min(k, len(filters))
    out = []
    for r in range(k):
        part = filters[len(filters) * r // k:len(filters) * (r + 1) // k]
        out.append((list(part[0]), list(part[-1]), part))
    return out
