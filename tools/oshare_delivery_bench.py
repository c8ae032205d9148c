"""Time bfq_delivery_device_ordered against bfq_delivery_device, and against resolving the $oshare pairs on the host.

Input: the C4 workload (its own $oshare groups) at --scale, matched once (MaxGroupFanout 100), with --pubs seeded publishers
per topic position (ClientInfo hashes drawn from a seeded generator). Per publisher count, rounds alternate `--iters`
bfq_delivery_device calls and `--iters` bfq_delivery_device_ordered calls, each block timed with CUDA events after warm-up
(both calls include their stream synchronisations). The host leg times what a host holding bfq_delivery_device's nesting
has to do instead: the rendezvous pick of every ($oshare pair, publisher) over the group's member receiverUrls, with the
numpy restatement of Guava's murmur3_128 in tests/rendezvous_hash.py, and the grouping of publishers per winner. Its sub-pack count is
checked against the device's. Prints the GPU name and power limit, then one JSON line per publisher count.

    python tools/oshare_delivery_bench.py [--scale 0.1] [--pubs 1,8] [--iters 20] [--rounds 5] [--warmup 5]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import fanout_bench  # noqa: E402  (gpu_info)


def members_in_wire_order(value, schema):
    """receiverUrls of a RouteGroup value in wire order (the order the pick walks; schema.parse_route_group sorts them)"""
    out, p = [], 0
    while p < len(value):
        _, p = schema._varint(value, p)
        ln, p = schema._varint(value, p)
        end = p + ln
        while p < end:
            t, p = schema._varint(value, p)
            if t == 0x0A:
                kl, p = schema._varint(value, p)
                out.append(bytes(value[p:p + kl]))
                p += kl
            else:
                _, p = schema._varint(value, p)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4")
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--pubs", default="1,8", help="publishers per topic position")
    ap.add_argument("--iters", type=int, default=20, help="calls per timed block")
    ap.add_argument("--rounds", type=int, default=5, help="alternating (delivery block, ordered block) rounds")
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch

    import bifromq_b200
    import rendezvous_hash as RH
    from bifromq_b200 import schema
    from bifromq_b200.workload import Workload
    bifromq_b200.load_library()
    name, limit = fanout_bench.gpu_info()
    print("gpu: %s, power limit %s" % (name, limit), flush=True)
    w = Workload(args.config, scale=args.scale)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    n, tenants = w.n_topics, w.tenants
    nt = len(tenants)
    tt_host = np.ascontiguousarray(w.topic_tenant[:n]).astype(np.int64)
    d_topics = torch.from_numpy(np.ascontiguousarray(w.topics)).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(w.topic_off)).to(dev)
    d_tt = torch.from_numpy(np.ascontiguousarray(w.topic_tenant[:n])).to(dev)
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    idx.commit()
    out = idx.match_device(tenants, d_topics.data_ptr(), d_off.data_ptr(), d_tt.data_ptr(), n, [2 ** 31 - 1] * nt, [100] * nt, stream)
    d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    total = out.expand(d_offsets.data_ptr(), None, 0, stream)
    d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=dev)
    out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
    torch.cuda.synchronize()
    csr_off, csr_ranks = d_offsets.cpu().numpy(), d_ranks.cpu().numpy()[:total]
    # the $oshare routes of the CSR and their member urls, decoded from the workload's KV (host leg input)
    kb, vb = w.keys.tobytes(), w.vals.tobytes()
    members = {}
    for r in np.unique(csr_ranks).tolist():
        k, v = kb[w.key_off[r]:w.key_off[r + 1]], vb[w.val_off[r]:w.val_off[r + 1]]
        m = schema.build_match_route(k, v)
        if isinstance(m, schema.GroupMatching) and m.ordered:
            urls = members_in_wire_order(v, schema)
            if urls:
                members[r] = urls
    topic_of = np.repeat(np.arange(n), np.diff(csr_off))
    valid = (tt_host >= 0) & (tt_host < nt)
    oshare = np.flatnonzero(np.isin(csr_ranks, list(members)) & valid[topic_of])
    deliver = lambda: out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), stream)
    for k in [int(x) for x in args.pubs.split(",")]:
        rng = np.random.default_rng(k)
        pub_off = np.arange(n + 1, dtype=np.int64) * k
        pub_hash = rng.integers(-2 ** 31, 2 ** 31, n * k, dtype=np.int64).astype(np.int32)
        d_po = torch.from_numpy(pub_off).to(dev)
        d_ph = torch.from_numpy(pub_hash if len(pub_hash) else np.zeros(1, np.int32)).to(dev)
        ordered = lambda: out.delivery_ordered(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), d_po.data_ptr(),
                                               d_ph.data_ptr(), len(pub_hash), stream)
        for _ in range(args.warmup):
            deliver()
            ordered()
        torch.cuda.synchronize()
        ms = {"delivery": [], "ordered": []}
        for _ in range(args.rounds):
            for leg, fn in (("delivery", deliver), ("ordered", ordered)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    r = fn()
                e1.record()
                torch.cuda.synchronize()
                ms[leg].append(e0.elapsed_time(e1) / args.iters)
                if leg == "ordered":
                    od = r
        # host leg: every ($oshare pair, publisher) scored over its members, publishers grouped per (pair, winner)
        t0 = time.perf_counter()
        hs, urls, first = [], [], []
        for j in oshare.tolist():
            t, r = int(topic_of[j]), int(csr_ranks[j])
            for p in range(int(pub_off[t]), int(pub_off[t + 1])):
                first.append(len(hs))
                hs += [int(pub_hash[p])] * len(members[r])
                urls += members[r]
        scores = RH.scores_np(hs, urls) if hs else np.zeros(0, np.int64)
        bounds = first + [len(hs)]
        subs = set()
        q = 0
        for j in oshare.tolist():
            t = int(topic_of[j])
            for p in range(int(pub_off[t]), int(pub_off[t + 1])):
                subs.add((j, int(np.argmax(scores[bounds[q]:bounds[q + 1]]))))
                q += 1
        host_ms = (time.perf_counter() - t0) * 1e3
        dl_ms, od_ms = float(np.median(ms["delivery"])), float(np.median(ms["ordered"]))
        print(json.dumps({
            "config": args.config, "scale": args.scale, "pubs_per_position": k, "n_topics": n, "n_pairs": total,
            "n_oshare_pairs": int(len(oshare)), "n_items": int(len(first)), "n_ordered_packs": od.ordered.n_ordered_packs,
            "host_sub_packs_equal": len(subs) == od.ordered.n_ordered_packs,
            "delivery_ms": round(dl_ms, 4), "delivery_ms_rounds": [round(x, 4) for x in ms["delivery"]],
            "ordered_ms": round(od_ms, 4), "ordered_ms_rounds": [round(x, 4) for x in ms["ordered"]],
            "host_oshare_ms": round(host_ms, 1), "gpu": name, "power_limit": limit}), flush=True)
    out.release()
    idx.close()


if __name__ == "__main__":
    main()
