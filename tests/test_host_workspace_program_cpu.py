"""CPU pins of tests/test_gpu_workspace_lease.py: the pool model, the call program's determinism and coverage, and the
thresholds it restates from the library. No GPU."""
import numpy as np

import test_gpu_workspace_lease as T


def test_pool_model_is_lifo_and_keeps_four():
    p = T.PoolModel()
    a, _ = p.acquire(10)
    p.give_back(a)
    assert p.acquire(5) == (a, False)                   # the same workspace, no growth
    assert p.acquire(5)[0] == 1                         # a second one while the first is out
    p.give_back(1)
    p.give_back(a)
    assert p.acquire(11) == (a, True)                   # given back last, handed out first; grew past 10
    ws = [a] + [p.acquire(1)[0] for _ in range(5)]      # idle [1] is taken, then four new ones
    assert ws[1] == 1 and p.made == 6
    for w in ws:
        p.give_back(w)
    assert p.idle == ws[:4] and p.freed == ws[4:]
    assert p.acquire(0) == (ws[3], False)               # an empty batch still reserves one element


def test_program_is_deterministic():
    a, b = T.program(), T.program()
    assert a == b
    for s in a:
        if s["op"] == "match" and 0 < s["n"] <= 5000:
            x = T.batch(s["n"], s["lst"], int(s["name"][1:]), s["pool"])
            y = T.batch(s["n"], s["lst"], int(s["name"][1:]), s["pool"])
            assert x[0] == y[0] and np.array_equal(x[1], y[1])
    assert T.tenant_list("L4097", 3) == T.tenant_list("L4097", 3)


def main_matches():
    steps = T.program()
    plan, pool = T.plan(steps)
    main = {nm for nm, (w, _) in plan.items() if w == 0}
    return steps, plan, pool, main


def test_every_transition_lands_on_the_main_workspace():
    steps, plan, pool, main = main_matches()
    seq = [s for s in steps if s["op"] == "match" and s["name"] in main]
    sizes = [s["n"] for s in seq]
    # batch sizes 131072 -> 32767 -> 32768 -> 1 -> 0 -> 131073, in that order
    want = [131072, 32767, 32768, 1, 0, 131073]
    it = iter(sizes)
    assert all(any(x == w for x in it) for w in want)
    # tenant lists 1 -> 4097 -> 2^20 + 1 -> 4097 with other caps -> 4097 with only the caps changed
    lists = [(s["lst"], s["caps"]) for s in seq]
    i = lists.index(("Lbig", 2))
    assert lists[i - 1][0] == "L4097" and lists[i + 1] == ("L4097", 3) and lists[i + 2] == ("L4097", 1)
    assert lists[i - 1] == ("L4097", 1) and ("L1", 0) in lists[:i]
    # host <-> device, retry then a small call and a 4-sub-batch call, tier 2 then tier 0 only
    paths = [s["path"] for s in seq]
    assert any(a != b for a, b in zip(paths, paths[1:])) and paths.count("host") >= 3
    r = [s.get("retry", False) for s in seq].index(True)
    assert seq[r + 1]["n"] < 1000 and seq[r + 2]["path"] == "host" and T.sub_batches(seq[r + 2]["n"], True) == 4
    t2 = [s["pool"] for s in seq].index("tier2")
    assert seq[t2 + 1]["pool"] == "tier0"
    # fan-out tiled -> global -> tiled, delivery on more then fewer topics, budget binding then not
    fans = [(s["name"], s["fan"]) for s in seq if s.get("fan")]
    kinds = [f for _, f in fans]
    assert "global" in kinds and kinds[kinds.index("global") - 1] == "auto" and kinds[kinds.index("global") + 1] == "auto"
    dl = [s["n"] for s in seq if s.get("deliver")]
    assert len(dl) == 2 and dl[0] > dl[1]
    assert [s["budget"] for s in seq if s.get("budget")] == ["bind", "free"]
    assert [s["name"] for s in seq if s.get("gather")]
    # options change between calls
    opts = {k for s in steps if s["op"] == "opt" for k in s if k != "op"}
    assert {"order_min_topics", "dedup_hash_bits", "tier0_ctas_per_sm"} <= opts


def test_held_results_make_and_free_a_workspace():
    steps, plan, pool, main = main_matches()
    held = [s["name"] for s in steps if s["op"] == "match" and s.get("hold")]
    assert 5 <= len(held) <= 6
    assert len({plan[nm][0] for nm in held}) == len(held)
    assert pool.made == 5 and len(pool.freed) == 1
    ops = [s["op"] for s in steps]
    first, last = ops.index("match", [i for i, s in enumerate(steps) if s.get("hold")][0]), ops.index("release")
    commits = [steps[i]["kind"] for i in range(first, last) if ops[i] == "commit"]
    assert commits == ["delta", "full"]
    # the main workspace comes back after the release and no span buffer grew: the last call reuses it
    assert plan["m20"] == (0, False)


def test_thresholds_hit_their_values():
    steps = {s["name"]: s for s in T.program() if s["op"] == "match"}
    # order: 131072 on the host path is 4 ordered sub-batches of 32768; 32767 on the device path is not ordered, but
    # prepare_workspace's per_chunk (n + 1) reaches order_min and reserves the order buffers; 32768 is ordered
    assert T.sub_batches(steps["m1"]["n"], True) == 4 and T.ordered(steps["m1"]["n"], True)
    assert T.per_chunk(131072, 4) == 32769
    assert not T.ordered(steps["m2"]["n"], False) and T.per_chunk(steps["m2"]["n"], 1) == T.ORDER_MIN
    assert T.ordered(steps["m3"]["n"], False) and not T.ordered(32767, False)
    assert T.sub_batches(steps["m7"]["n"], False) == 1 and T.ordered(steps["m7"]["n"], False)
    assert T.sub_batches(131071, True) == 1
    # tenant, key and histogram bits: 1 -> 0, 4097 -> 13, 2^20 + 1 -> capped at 20
    assert [T.tenant_bits(T.LIST_SIZES[k]) for k in ("L1", "L4097", "Lbig")] == [0, 13, 20]
    assert [T.key_bits(b) for b in (0, 13, 20)] == [16, 32, 32]
    assert T.hist_bits(32768, 1) == 16 and T.hist_bits(32768, 4097) == 17 and T.hist_bits(32768, T.BIG_LIST) == 17
    assert T.hist_bits(131073, 4097) == 20 and T.hist_bits(1, 1) == 12
    assert T.hash_entries(32768) == 65536 and T.hash_entries(32769) == 131072 and T.hash_entries(1) == 1024
    # the colliding entries: same tenant key once masked to 20 bits, different tenant ids, same topic text
    ids, _, _ = T.tenant_list("Lbig", 2)
    topics, tt = T.batch(steps["m3"]["n"], "Lbig", 3, "base")
    for k, i in enumerate(T.COLLIDE_AT):
        j = i + (1 << 20)
        assert j < T.BIG_LIST and (i & ((1 << 20) - 1)) == (j & ((1 << 20) - 1)) and ids[i] != ids[j]
        assert topics[2 * k] == topics[2 * k + 1] and (tt[2 * k], tt[2 * k + 1]) == (i, j)
    # the retry: m8's spill blocks exceed what the region m1 sized leaves after m8's inline slots
    assert T.SPILL_N * T.E.SPILL_RANGES > T.REGION_AFTER_M1 - T.SPILL_N * T.E.INLINE_RANGES
    assert steps["m8"]["n"] == T.SPILL_N and len(set(T.batch(T.SPILL_N, "L1", 8, "spill")[0])) == T.SPILL_N


def test_tier_pools_reach_their_tiers():
    w = T.world_of(0)
    res = T.E.oracle_match(w.kv, ["tA"], [T.E.TIER2_TOPIC, "s/x", "k1/a/b/c/d"], np.zeros(3, np.int32), T.INT_MAX, T.INT_MAX)
    ranges = [len(T.E.matched_filters(w.kv, res, i)) for i in range(3)]
    assert ranges[0] > T.E.RG_CAP and ranges[1] <= T.E.INLINE_RANGES and ranges[2] > T.E.INLINE_RANGES
    assert all(t.count("/") + 1 <= T.E.L_MAXLV for t in T.TIER0_TOPICS)
    delta = sorted(set(T.world_of(1).pairs) - set(w.pairs))
    assert delta and not set(w.pairs) - set(T.world_of(1).pairs)
