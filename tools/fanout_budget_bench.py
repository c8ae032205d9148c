"""Time the delivery budgets (bfq_expand_device_budget) against the plain expand (bfq_expand_device), both followed by
bfq_fanout_device, with CUDA events around many calls on one completed match, after warm-up.

Input: the C4 workload (a quarter of the routes persistent, up to 10 000 routes per filter), every message 1000 bytes.
Shapes:
  expand           bfq_expand_device (sizing + writing call), then bfq_fanout_device: the path without budgets
  never_binds      bfq_expand_device_budget with MaxPersistentFanoutBytes = 2^63 - 1 and both bandwidths for every tenant
  bytes_4s         MaxPersistentFanoutBytes = 4 s: at most 4 persistent routes of a multi-route topic are delivered
  transient_half   transient bandwidth off for every other tenant of the list
Each shape is timed `--repeats` times over `--iters` calls; the JSON line gives the median and the spread of the per-call
times, separately for the expand step and the fan-out step. The budget outputs are checked against a host restatement of
DeliverExecutorGroup.submit on a sample of topics (kinds from bfq_route_kinds, survivors from the plain expand).

    python tools/fanout_budget_bench.py [--scale 0.1] [--iters 50] [--warmup 5] [--repeats 5]

Set BFQ_LIB to time another build of the library on the same inputs (A/B runs in one session); a build without
bfq_expand_device_budget times the expand shape only.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

I64_MAX, MSG = 2 ** 63 - 1, 1000


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def restate(kinds, ranks, s, max_bytes, bw):
    """DeliverExecutorGroup.submit's sends for one topic, persistent routes in ascending rank order"""
    order = np.argsort(ranks)
    ranks, kinds = ranks[order], kinds[order]
    if len(ranks) <= 1:
        return sorted(ranks.tolist())
    sent, sent_bytes = [], 0
    for r, k in zip(ranks.tolist(), kinds.tolist()):
        if k == 2 or (k == 0 and bw & 2):
            sent.append(r)
        elif k == 1 and bw & 1 and sent_bytes < max_bytes:
            sent.append(r)
            sent_bytes += s
    return sorted(sent)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4")
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--sample", type=int, default=2000, help="topics checked against the host restatement per shape")
    args = ap.parse_args()
    import torch

    from bifromq_b200 import _native as N
    has_budget = hasattr(C.CDLL(N.LIB_PATH), "bfq_expand_device_budget")
    if not has_budget:
        N._SIGNATURES.pop("bfq_expand_device_budget")
    import bifromq_b200
    from bifromq_b200.workload import Workload
    bifromq_b200.load_library()
    name, limit = gpu_info()
    print("gpu: %s, power limit %s, library %s" % (name, limit, N.LIB_PATH), flush=True)
    w = Workload(args.config, scale=args.scale)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    n, tenants = w.n_topics, w.tenants
    nt = len(tenants)
    d_topics = torch.from_numpy(np.ascontiguousarray(w.topics)).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(w.topic_off)).to(dev)
    tt = np.ascontiguousarray(w.topic_tenant[:n])
    d_tt = torch.from_numpy(tt).to(dev)
    d_msg = torch.full((max(n, 1),), MSG, dtype=torch.int32, device=dev)
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    idx.commit()
    out = idx.match_device(tenants, d_topics.data_ptr(), d_off.data_ptr(), d_tt.data_ptr(), n, [2 ** 31 - 1] * nt, [100] * nt, stream)
    d_offsets = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    total = out.expand(d_offsets.data_ptr(), None, 0, stream)
    d_ranks = torch.zeros(max(total, 1), dtype=torch.int64, device=dev)
    cap = max(total, 1)

    def expand():
        t = out.expand(d_offsets.data_ptr(), None, 0, stream)
        out.expand(d_offsets.data_ptr(), d_ranks.data_ptr(), cap, stream)
        return t

    def budgeted(mb, bw):
        def f():
            r = out.expand_budget(d_msg.data_ptr(), mb, bw, d_offsets.data_ptr(), None, 0, stream)
            out.expand_budget(d_msg.data_ptr(), mb, bw, d_offsets.data_ptr(), d_ranks.data_ptr(), cap, stream)
            return r.n_delivered
        return f, mb, bw

    shapes = [("expand", expand, None, None)]
    if has_budget:
        both = np.full(nt, 3, np.uint8)
        half = np.where(np.arange(nt) % 2 == 0, 1, 3).astype(np.uint8)
        shapes += [(s,) + budgeted(mb, bw) for s, mb, bw in (("never_binds", np.full(nt, I64_MAX, np.int64), both),
                                                             ("bytes_4s", np.full(nt, 4 * MSG, np.int64), both),
                                                             ("transient_half", np.full(nt, I64_MAX, np.int64), half))]
    expand()
    torch.cuda.synchronize()
    plain_off = d_offsets.cpu().numpy().copy()
    plain_ranks = d_ranks.cpu().numpy()[:total].copy()
    rng = np.random.default_rng(1)
    sample = rng.choice(n, min(args.sample, n), replace=False)
    heavy = np.argsort(np.diff(plain_off))[-min(args.sample, n) // 20:]   # the heaviest topics, where the budgets bind
    sample = np.unique(np.concatenate([sample, heavy]))
    for shape, fn, mb, bw in shapes:
        n_pairs = fn()
        torch.cuda.synchronize()
        checked = 0
        if mb is not None:
            got_off = d_offsets.cpu().numpy()
            got_ranks = d_ranks.cpu().numpy()[:n_pairs]
            for i in sample.tolist():
                surv = plain_ranks[plain_off[i]:plain_off[i + 1]]
                want = restate(idx.route_kinds(surv), surv, MSG, int(mb[tt[i]]), int(bw[tt[i]]))
                assert sorted(got_ranks[got_off[i]:got_off[i + 1]].tolist()) == want, (shape, i)
                checked += 1
        for _ in range(args.warmup):
            fn()
            out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), n_pairs, stream)
        torch.cuda.synchronize()
        exp_ms, fan_ms = [], []
        for _ in range(args.repeats):
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            for _ in range(args.iters):
                out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), n_pairs, stream)
            e2.record()
            torch.cuda.synchronize()
            exp_ms.append(e0.elapsed_time(e1) / args.iters)
            fan_ms.append(e1.elapsed_time(e2) / args.iters)
        print(json.dumps({"config": args.config, "scale": args.scale, "shape": shape, "n_topics": n, "n_matched": total,
                          "n_delivered": n_pairs, "checked_topics": checked,
                          "expand_ms": round(float(np.median(exp_ms)), 4),
                          "expand_ms_spread": [round(min(exp_ms), 4), round(max(exp_ms), 4)],
                          "fanout_ms": round(float(np.median(fan_ms)), 4),
                          "fanout_ms_spread": [round(min(fan_ms), 4), round(max(fan_ms), 4)],
                          "gpu": name, "power_limit": limit, "library": os.path.basename(N.LIB_PATH)}), flush=True)
    out.release()
    idx.close()


if __name__ == "__main__":
    main()
