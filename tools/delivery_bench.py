"""Time bfq_delivery_device against bfq_fanout_device, and against re-grouping the fan-out's output on the host.

Input: the shapes of tools/fanout_bench.py (the C4 workload's routes as generated, and re-keyed to about 10k and 100k
deliverers). Per shape one completed match and its device CSR are made once; then rounds alternate `--iters` fan-out calls
and `--iters` delivery calls, each block timed with CUDA events after warm-up (a delivery call includes its one stream
synchronise). The host leg copies the fan-out's arrays back once and times a numpy re-grouping of them into the same
nesting (stable sort on (deliverer, tenant, topic position), then segment heads): what a host reading the fan-out has to
do instead of the delivery call. The device nesting is checked against that re-grouping, pack for pack.

Counted bytes per call (the work each call has to do, not what the kernels move): both read the CSR (8 per pair + 8 per
topic) and the deliverer id of each route (4 per pair); the fan-out writes 12 per pair + 8 per deliverer id, the delivery
8 per pair + 12 per pack + 12 per package + 8 per deliverer id. Prints the GPU name and power limit, then one JSON line per
shape.

    python tools/delivery_bench.py [--scale 0.1] [--iters 20] [--rounds 5] [--warmup 5] [--host-reps 3] [--rekey 0,10000,100000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import fanout_bench  # noqa: E402  (gpu_info, rekey)


def host_regroup(deliverer, topic, rank, member, topic_tenant, n_tenants, n_deliverers):
    """the fan-out's pairs -> the delivery arrays, with numpy on the host"""
    tenant = topic_tenant[topic].astype(np.int64)
    keep = (tenant >= 0) & (tenant < n_tenants)
    deliverer, topic, rank, member, tenant = deliverer[keep], topic[keep], rank[keep], member[keep], tenant[keep]
    n_topics = len(topic_tenant)
    key = (deliverer.astype(np.int64) * n_tenants + tenant) * n_topics + topic
    o = np.argsort(key, kind="stable")
    key, deliverer, tenant, topic = key[o], deliverer[o], tenant[o], topic[o]
    pack_head = np.ones(len(key), bool)
    pack_head[1:] = key[1:] != key[:-1]
    dt = deliverer * n_tenants + tenant
    package_head = np.ones(len(key), bool)
    package_head[1:] = dt[1:] != dt[:-1]
    packs = np.flatnonzero(pack_head)
    packages = np.flatnonzero(package_head)
    pack_of_package = np.cumsum(pack_head)[packages] - 1
    return {"package_off": np.concatenate([[0], np.cumsum(np.bincount(deliverer[packages], minlength=n_deliverers))]),
            "package_tenant": tenant[packages], "pack_off": np.concatenate([pack_of_package, [len(packs)]]),
            "pack_topic": topic[packs], "match_off": np.concatenate([packs, [len(key)]]),
            "match_rank": rank[o], "match_member": member[o]}


def same_nesting(dev, host):
    for k in ("package_off", "package_tenant", "pack_off", "pack_topic", "match_off"):
        if not np.array_equal(np.asarray(dev[k], np.int64), np.asarray(host[k], np.int64)):
            return False
    # MatchInfos inside a pack are unordered, and a rank occurs once per pack: compare them sorted by (pack, rank)
    pack = np.repeat(np.arange(len(dev["match_off"]) - 1, dtype=np.int64), np.diff(dev["match_off"]))

    def by_pack_rank(a):
        key = pack << 32 | np.asarray(a["match_rank"], np.int64)
        o = np.argsort(key, kind="stable")
        return key[o], np.asarray(a["match_member"], np.int64)[o]
    (k0, m0), (k1, m1) = by_pack_rank(dev), by_pack_rank(host)
    return np.array_equal(k0, k1) and np.array_equal(m0, m1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4")
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=20, help="calls per timed block")
    ap.add_argument("--rounds", type=int, default=5, help="alternating (fan-out block, delivery block) rounds")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--rekey", default="0,10000,100000", help="0 = the workload's own deliverer keys")
    args = ap.parse_args()
    import torch

    import bifromq_b200
    from bifromq_b200 import _native as N
    from bifromq_b200.dist import device_view
    from bifromq_b200.workload import Workload
    bifromq_b200.load_library()
    name, limit = fanout_bench.gpu_info()
    print("gpu: %s, power limit %s, library %s" % (name, limit, N.LIB_PATH), flush=True)
    w = Workload(args.config, scale=args.scale)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    n, tenants = w.n_topics, w.tenants
    tt_host = np.ascontiguousarray(w.topic_tenant[:n]).astype(np.int64)
    d_topics = torch.from_numpy(np.ascontiguousarray(w.topics)).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(w.topic_off)).to(dev)
    d_tt = torch.from_numpy(np.ascontiguousarray(w.topic_tenant[:n])).to(dev)
    vb = w.vals.tobytes()
    for nd in [int(x) for x in args.rekey.split(",")]:
        idx = bifromq_b200.GpuRouteIndex(0)
        if nd == 0:
            idx.load(w.keys, w.key_off, w.vals, w.val_off)
        else:
            rk = fanout_bench.rekey(w.keys, w.key_off, nd)
            kk, ko = N.as_blob([k for k, _ in rk])
            vv, vo = N.as_blob([vb[w.val_off[i]:w.val_off[i + 1]] for _, i in rk])
            idx.load(kk, ko, vv, vo)
        idx.commit()
        nt = len(tenants)
        out = idx.match_device(tenants, d_topics.data_ptr(), d_off.data_ptr(), d_tt.data_ptr(), n, [2 ** 31 - 1] * nt, [100] * nt, stream)
        d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        total = out.expand(d_offsets.data_ptr(), None, 0, stream)
        d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=dev)
        out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
        fan = lambda: out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
        deliver = lambda: out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), stream)
        for _ in range(args.warmup):
            fan()
            deliver()
        torch.cuda.synchronize()
        ms = {"fanout": [], "delivery": []}
        for _ in range(args.rounds):
            for leg, fn in (("fanout", fan), ("delivery", deliver)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    r = fn()
                e1.record()
                torch.cuda.synchronize()
                ms[leg].append(e0.elapsed_time(e1) / args.iters)
                if leg == "fanout":
                    fo = r
                else:
                    dl = r
        # host leg: the fan-out's output copied back once (timed apart), then re-grouped with numpy
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        D = fo.n_deliverers
        n1 = max(total, 1)
        f_off = device_view(fo.d_pack_offsets, D + 1, "<i8", dev).cpu().numpy()
        f_topic = device_view(fo.d_pack_topic, n1, "<u4", dev).cpu().numpy()[:total].astype(np.int64)
        f_rank = device_view(fo.d_pack_rank, n1, "<u4", dev).cpu().numpy()[:total].astype(np.int64)
        f_member = device_view(fo.d_pack_member, n1, "<u4", dev).cpu().numpy()[:total].astype(np.int64)
        copy_ms = (time.perf_counter() - t0) * 1e3
        f_deliv = np.repeat(np.arange(D, dtype=np.int64), np.diff(f_off))
        host_ms = []
        for _ in range(args.host_reps):
            t0 = time.perf_counter()
            host = host_regroup(f_deliv, f_topic, f_rank, f_member, tt_host, nt, D)
            host_ms.append((time.perf_counter() - t0) * 1e3)
        got = dl.arrays(dev)
        same = same_nesting(got, host)
        fo_ms, dl_ms = float(np.median(ms["fanout"])), float(np.median(ms["delivery"]))
        nb_read = 8 * total + 8 * (n + 1) + 4 * total
        fo_bytes = nb_read + 12 * total + 8 * (D + 1)
        dl_bytes = nb_read + 8 * total + 12 * dl.n_packs + 12 * dl.n_packages + 8 * (D + 1)
        print(json.dumps({
            "config": args.config, "scale": args.scale, "rekey": nd, "n_topics": n, "n_tenants": nt, "n_pairs": total,
            "n_deliverers": D, "n_packages": dl.n_packages, "n_packs": dl.n_packs, "nesting_equal_host": bool(same),
            "fanout_ms": round(fo_ms, 4), "fanout_ms_rounds": [round(x, 4) for x in ms["fanout"]],
            "delivery_ms": round(dl_ms, 4), "delivery_ms_rounds": [round(x, 4) for x in ms["delivery"]],
            "host_regroup_ms": round(float(np.median(host_ms)), 2), "host_copy_ms": round(copy_ms, 2),
            "fanout_counted_GBps": round(fo_bytes / fo_ms / 1e6, 1), "delivery_counted_GBps": round(dl_bytes / dl_ms / 1e6, 1),
            "gpu": name, "power_limit": limit}), flush=True)
        out.release()
        idx.close()


if __name__ == "__main__":
    main()
