"""Time bfq_range_lookup on ranges cut from a generated route set, and A/B builds of the library in one session.

Input (seeded, the same for every build): the distinct filters of config C3's route set (reduced scale), per tenant in Java
level order, cut into --ranges contiguous ranges whose Facts are their smallest and largest filter; a publish batch of --topics
topics of --levels levels each, grown from the tenant's own filters so many of them match. One call answers every
(topic, range) pair of the batch: --topics x --ranges pairs (10^7 by default).

The call copies its inputs to the device, runs range_lookup_kernel, copies the rows back and synchronises, so it is timed with
a host clock (median and min of --iters calls after --warmup). In a separate run of its own, torch.profiler with CUDA activities
gives the kernel's device time. Each build prints the SHA-256 of its keep rows, which must agree between builds.

    python tools/range_lookup_bench.py [--lib name=path ...] [--runs 3] [--topics 10000] [--ranges 1000] [--levels 16]

Without --lib the in-tree library is timed. With several, the builds alternate run by run, each in a fresh process (BFQ_LIB).
"""
import argparse
import hashlib
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORDS = ["a", "b", "c", "dev", "x", "sensor", "07", "room", "~", "é"]


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def make_inputs(args):
    """(argument arrays for bfq_range_lookup, the arrays they point into, keep_off, keep)"""
    import range_lookup_brute as R
    from bifromq_b200 import _native as N
    from bifromq_b200.workload import Workload
    w = Workload("C3", scale=args.scale)
    per = R.tenant_filters(w)
    tenants = sorted(per)
    rng = random.Random(args.seed)
    topics, tt = [], []
    for i in range(args.topics):
        t = rng.randrange(len(tenants))
        f = list(rng.choice(per[tenants[t]])[1:])
        lv = [x if x not in ("+", "#") else rng.choice(WORDS) for x in f]
        lv = (lv + [rng.choice(WORDS) for _ in range(args.levels)])[:args.levels]
        topics.append("/".join(lv))
        tt.append(t)
    cand_off = np.zeros(len(tenants) + 1, np.int64)
    firsts, lasts = [], []
    for t, tenant in enumerate(tenants):
        ranges = R.cut_ranges(per[tenant], args.ranges)
        cand_off[t + 1] = cand_off[t] + len(ranges)
        for f, l, _ in ranges:
            firsts.append("\0".join(f).encode())
            lasts.append("\0".join(l).encode())
    fl = np.full(len(firsts) + 1, 7, np.uint8)
    tb, toff = N.as_blob(tenants)
    pb, poff = N.as_blob(topics)
    fb, foff = N.as_blob(firsts)
    lb, loff = N.as_blob(lasts)
    tt = np.asarray(tt, np.int32)
    n_pairs = int(sum(cand_off[t + 1] - cand_off[t] for t in tt.tolist()))
    keep_off = np.zeros(len(topics) + 1, np.int64)
    keep = np.zeros(max(n_pairs, 1), np.uint8)
    call = [0, N.ptr(tb), N.ptr(toff), len(tenants), N.ptr(pb), N.ptr(poff), N.ptr(tt), len(topics), N.ptr(cand_off), N.ptr(fl),
            N.ptr(fb), N.ptr(foff), N.ptr(lb), N.ptr(loff), N.ptr(keep_off), N.ptr(keep)]
    return call, (tb, toff, pb, poff, tt, cand_off, fl, fb, foff, lb, loff), keep_off, keep, n_pairs


def one_build(args):
    """time (or profile) the library this process loads; print one JSON line"""
    import torch

    import bifromq_b200
    from bifromq_b200 import _native as N
    bifromq_b200.load_library()
    torch.cuda.init()
    call, _alive, keep_off, keep, n_pairs = make_inputs(args)
    for _ in range(args.warmup):
        N.check(N.lib.bfq_range_lookup(*call))
    out = {"lib": args.name, "n_topics": args.topics, "levels": args.levels, "n_pairs": n_pairs,
           "kept": int(np.count_nonzero(keep[:n_pairs])), "keep_sha256": hashlib.sha256(keep[:n_pairs].tobytes()).hexdigest()}
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                N.check(N.lib.bfq_range_lookup(*call))
            torch.cuda.synchronize()
        ks = [e for e in prof.events() if e.device_type.name == "CUDA" and "range_lookup_kernel" in e.name]
        dev = [getattr(e, "device_time", None) or e.cuda_time for e in ks]   # microseconds
        out["kernel_launches"] = len(ks)
        out["kernel_ms_median"] = round(statistics.median(dev) / 1e3, 4) if dev else None
    else:
        ms = []
        for _ in range(args.iters):
            t0 = time.perf_counter()
            N.check(N.lib.bfq_range_lookup(*call))
            ms.append((time.perf_counter() - t0) * 1e3)
        out["call_ms_median"] = round(statistics.median(ms), 3)
        out["call_ms_min"] = round(min(ms), 3)
        out["pairs_per_s"] = round(n_pairs / (statistics.median(ms) / 1e3))
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="name=path of a libbfq_gpumatch.so build (repeatable)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scale", type=float, default=0.002)
    ap.add_argument("--topics", type=int, default=10000)
    ap.add_argument("--ranges", type=int, default=1000)
    ap.add_argument("--levels", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--name", default="in-tree")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child or not args.lib:
        one_build(args)
        return
    name, limit = gpu_info()
    print("gpu: %s, power limit %s" % (name, limit), flush=True)
    libs = [x.split("=", 1) for x in args.lib]
    base = [sys.executable, os.path.abspath(__file__), "--child", "--scale", str(args.scale), "--topics", str(args.topics),
            "--ranges", str(args.ranges), "--levels", str(args.levels), "--iters", str(args.iters), "--warmup", str(args.warmup),
            "--seed", str(args.seed)]
    results = {n: [] for n, _ in libs}
    for mode in ("time", "profile"):
        for run in range(args.runs if mode == "time" else 1):
            for n, path in libs:
                env = dict(os.environ, BFQ_LIB=os.path.abspath(path))
                cmd = base + ["--name", n] + (["--profile"] if mode == "profile" else [])
                line = subprocess.run(cmd, env=env, check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1]
                r = json.loads(line)
                r.update(run=run, mode=mode, gpu=name, power_limit=limit)
                results[n].append(r)
                print(json.dumps(r), flush=True)
    shas = {r["keep_sha256"] for rs in results.values() for r in rs}
    summary = {"identical_keep_rows": len(shas) == 1, "gpu": name, "power_limit": limit}
    for n, rs in results.items():
        t = [r["call_ms_median"] for r in rs if r["mode"] == "time"]
        k = [r["kernel_ms_median"] for r in rs if r["mode"] == "profile"]
        summary[n] = {"call_ms_median_per_run": t, "kernel_ms_median": k[0] if k else None}
    print(json.dumps({"summary": summary}), flush=True)


if __name__ == "__main__":
    main()
