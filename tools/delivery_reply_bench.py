"""Time bfq_delivery_reply: every deliverer's DeliveryReply joined back to a delivery nesting, and the same join on the host.

Input: the shapes of tools/delivery_bench.py (the C4 workload's routes as generated, and re-keyed to about 10k and 100k
deliverers), matched once (MaxGroupFanout 100), nested with bfq_delivery_device. The replies are what LocalDistService.dist
sends, written from the nesting itself by tests/delivery_reply.nesting_replies (not by the code under test): per deliverer one map entry per package, one
DeliveryResult per distinct MatchInfo of the package (the MatchInfo restated from the route KV by tests/delivery_wire.py), with
a seeded code: about --no-sub NO_SUB, --no-receiver NO_RECEIVER, the rest OK (code field omitted). Per shape, the replies are
copied to the device once (that copy timed on its own with CUDA events, from pinned memory), then rounds alternate a block of
`--iters` bfq_delivery_device calls and a block of `--iters` bfq_delivery_reply calls (each block timed with CUDA events after
warm-up; every reply call includes its stream synchronisation). Reported per shape: the median per call of each leg, the reply
bytes and records per second, and the host leg: execute's join restated in tests/delivery_reply.py (protobuf parse plus dict
join) on the first --host-deliverers deliverers' replies, with the whole batch at that rate (extrapolated, labelled so).
Prints the GPU name and power limit.

    python tools/delivery_reply_bench.py [--scale 0.1] [--iters 10] [--rounds 5] [--warmup 2]
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

import fanout_bench  # noqa: E402  (gpu_info, rekey)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4")
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=10, help="calls per timed block")
    ap.add_argument("--rounds", type=int, default=5, help="alternating (delivery block, reply block) rounds")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-sub", type=float, default=0.02)
    ap.add_argument("--no-receiver", type=float, default=0.01)
    ap.add_argument("--host-deliverers", type=int, default=3)
    ap.add_argument("--rekey", default="0,10000,100000", help="0 = the workload's own deliverer keys")
    args = ap.parse_args()
    import torch

    import bifromq_b200
    import delivery_reply as R
    from bifromq_b200 import dist
    import delivery_wire as W
    from bifromq_b200 import _native as N
    from bifromq_b200.workload import Workload
    bifromq_b200.load_library()
    name, limit = fanout_bench.gpu_info()
    print("gpu: %s, power limit %s" % (name, limit), flush=True)
    w = Workload(args.config, scale=args.scale)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    n, tenants = w.n_topics, w.tenants
    nt = len(tenants)
    d_topics = torch.from_numpy(np.ascontiguousarray(w.topics)).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(w.topic_off)).to(dev)
    d_tt = torch.from_numpy(np.ascontiguousarray(w.topic_tenant[:n])).to(dev)
    tblob = bifromq_b200.GpuRouteIndex.tenant_blob(tenants)
    kb, vb = w.keys.tobytes(), w.vals.tobytes()
    for nd in [int(x) for x in args.rekey.split(",")]:
        idx = bifromq_b200.GpuRouteIndex(0)
        if nd == 0:
            keys = [kb[w.key_off[i]:w.key_off[i + 1]] for i in range(w.n_routes)]
            vals_of = None
            idx.load(w.keys, w.key_off, w.vals, w.val_off)
        else:
            rk = fanout_bench.rekey(w.keys, w.key_off, nd)
            keys = [k for k, _ in rk]
            kk, ko = N.as_blob(keys)
            vv, vo = N.as_blob([vb[w.val_off[i]:w.val_off[i + 1]] for _, i in rk])
            idx.load(kk, ko, vv, vo)
            vals_of = [i for _, i in rk]
        idx.commit()
        out = idx.match_device(tenants, d_topics.data_ptr(), d_off.data_ptr(), d_tt.data_ptr(), n, [2 ** 31 - 1] * nt, [100] * nt, stream)
        d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        total = out.expand(d_offsets.data_ptr(), None, 0, stream)
        d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=dev)
        out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
        deliver = lambda: out.delivery(d_offsets.data_ptr(), d_ranks.data_ptr(), total, d_tt.data_ptr(), stream)
        dl = deliver()
        a = dl.arrays(dev)
        infos = {}

        def mi_of(r, m):
            if r not in infos:
                v = vals_of[r] if vals_of else r
                infos[r] = W.route_match_infos(keys[r], vb[w.val_off[v]:w.val_off[v + 1]])
            return infos[r][0 if m == 0xFFFFFFFF else m]
        t0 = time.perf_counter()
        rp = R.nesting_replies(a, dl.n_deliverers, tenants, mi_of, np.random.default_rng(nd + 1), args.no_sub, args.no_receiver)
        blob, offs = rp["blob"], rp["off"]
        n_records, n_stale_codes = int(rp["sent"].sum()), int((rp["code"][rp["sent"]] > 0).sum())
        gen_s = time.perf_counter() - t0
        h_reply = torch.from_numpy(np.frombuffer(blob, np.uint8).copy()).pin_memory()
        d_reply = torch.empty(max(len(blob), 1), dtype=torch.uint8, device=dev)
        d_roff = torch.from_numpy(offs).to(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        d_reply[:len(blob)].copy_(h_reply, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        h2d_ms = e0.elapsed_time(e1)

        def reply():
            return out.delivery_reply(dl, tblob, d_reply.data_ptr(), d_roff.data_ptr(), stream)
        for _ in range(args.warmup):
            deliver()
            dl = deliver()
            reply()
        torch.cuda.synchronize()
        ms = {"delivery": [], "reply": []}
        for _ in range(args.rounds):
            for leg, fn in (("delivery", deliver), ("reply", reply)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    r = fn()
                e1.record()
                torch.cuda.synchronize()
                ms[leg].append(e0.elapsed_time(e1) / args.iters)
        res = reply()
        status = dist.device_view(res.d_status, res.n_deliverers, "|u1", dev).cpu().numpy()
        # host leg: execute restated on the first deliverers' replies
        hd = [d for d in range(dl.n_deliverers - 1) if offs[d + 1] > offs[d]][:args.host_deliverers]
        ko, mo = a["pack_off"], a["match_off"]
        t0 = time.perf_counter()
        host_records = 0
        for d in hd:
            tasks = []
            for g in range(int(a["package_off"][d]), int(a["package_off"][d + 1])):
                tn = tenants[int(a["package_tenant"][g])]
                for j in range(int(mo[ko[g]]), int(mo[ko[g + 1]])):
                    tasks.append((tn, mi_of(int(a["match_rank"][j]), int(a["match_member"][j]))))
            rep = blob[offs[d]:offs[d + 1]]
            R.execute(tasks, rep)
            host_records += len(tasks)
        host_s = time.perf_counter() - t0
        reply_ms = float(np.median(ms["reply"]))
        print(json.dumps({
            "config": args.config, "scale": args.scale, "rekey": nd, "n_pairs": total, "n_packs": dl.n_packs,
            "n_packages": dl.n_packages, "n_deliverers": dl.n_deliverers, "reply_bytes": len(blob), "reply_records": n_records,
            "stale_codes": n_stale_codes, "n_stale": res.n_stale, "n_fallback": res.n_fallback, "n_code": list(res.n_code),
            "status_ok": int((status == 0).sum()), "reply_generation_s": round(gen_s, 1),
            "h2d_ms": round(h2d_ms, 3), "h2d_bytes_per_s": round(len(blob) / (h2d_ms * 1e-3), 1) if h2d_ms > 0 else None,
            "delivery_ms": round(float(np.median(ms["delivery"])), 3), "delivery_ms_rounds": [round(x, 3) for x in ms["delivery"]],
            "reply_ms": round(reply_ms, 3), "reply_ms_rounds": [round(x, 3) for x in ms["reply"]],
            "reply_bytes_per_s": round(len(blob) / (reply_ms * 1e-3), 1), "reply_records_per_s": round(n_records / (reply_ms * 1e-3), 1),
            "host_sample_pairs": host_records, "host_sample_s": round(host_s, 3),
            "host_full_batch_s_extrapolated": round(host_s * total / max(host_records, 1), 1),
            "gpu": name, "power_limit": limit}), flush=True)
        out.release()
        idx.close()
        del d_reply
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
