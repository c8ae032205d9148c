#!/usr/bin/env python
"""Times bfq_index_commit on BASELINE C4 (10M filters, 1000 tenants) for commits that touch k tenants: one commit holding one
SUB into each of k tenants, for k in 1, 8, 64, 65, 128, 256, 512, 1000. The time is the wall clock around commit(), which
returns after the device is synchronised; every arm gives the median (and the range) of several commits per k.

A delta commit that rebuilds a large share of the tenants leaves their old regions as garbage, so the next commit may be a
full build (the garbage rule). Such a commit is run untimed before the next timed one, so that every timed commit of the
"delta" arm starts from the same kind of snapshot.

Arms, each in a subprocess of its own:
  * "delta": this build, every k; also the BFQ_COMMIT_TRACE laps of one commit of k = 1 and one of k = 1000;
  * "full": the same with BFQ_DELTA_COMMIT=0 (every commit a full build);
  * "parent" (with --parent-lib, a libbfq_gpumatch.so built from an earlier commit): k <= 64 only, alternated round by round
    with "delta" runs of the same k (--rounds), so the two are compared within the same call.

Prints the GPU name and power limit, then one JSON line per arm run, then a summary table.

    python tools/many_tenant_commit_bench.py [--scale 1.0] [--reps 5] [--parent-lib PATH] [--rounds 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KS = [1, 8, 64, 65, 128, 256, 512, 1000]


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def run_child(ks, reps, trace_ks, scale):
    import random

    import bifromq_b200
    from bifromq_b200 import schema, workload
    w = workload.Workload("C4", scale=scale)
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    t0 = time.perf_counter()
    idx.commit()
    out = {"config": "C4", "scale": scale, "routes": w.n_routes, "tenants": w.n_tenants,
           "first_full_commit_s": round(time.perf_counter() - t0, 3), "ms": {}, "paths": {}}
    names = w.tenants
    rng = random.Random(1)
    serial = [0]

    def storm(k):
        touched = rng.sample(names, min(k, len(names)))
        adds = []
        for t in touched:
            serial[0] += 1
            url = schema.receiver_url(serial[0] % 3, "storm%d" % serial[0], "d")
            adds.append((schema.route_key(t, "storm/%d/+" % (serial[0] % 7), url), schema.incarnation_bytes(1)))
        idx.apply(adds=adds)
        st = idx.stats()
        t0 = time.perf_counter()
        idx.commit()
        dt = time.perf_counter() - t0
        st2 = idx.stats()
        return dt * 1e3, "delta" if st2["delta_commits"] > st["delta_commits"] else "full"

    def reclaim():
        st = idx.stats()
        if st["delta_commits"] > 0 and st["garbage_slots"] > st["slots"] // 4 + 4096:
            storm(1)   # a full build (garbage rule), untimed

    for _ in range(reps):
        for k in ks:
            reclaim()
            ms, path = storm(k)
            out["ms"].setdefault(str(k), []).append(round(ms, 3))
            out["paths"].setdefault(str(k), []).append(path)
            sys.stderr.write("== k=%d %s %.3f ms\n" % (k, path, ms))
    for k in trace_ks:
        reclaim()
        sys.stderr.write("== trace k=%d\n" % k)
        sys.stderr.flush()
        os.environ["BFQ_COMMIT_TRACE"] = "1"
        ms, path = storm(k)
        del os.environ["BFQ_COMMIT_TRACE"]
        sys.stderr.write("== trace end k=%d %s %.3f ms\n" % (k, path, ms))
        sys.stderr.flush()
    idx.close()
    return out


def traces(stderr):
    """the BFQ_COMMIT_TRACE lines between the child's markers, per k"""
    out, cur = {}, None
    for line in stderr.splitlines():
        if line.startswith("== trace k="):
            cur = line.split("=")[-1].strip()
            out[cur] = []
        elif line.startswith("== trace end"):
            out[cur].append(line[3:])
            cur = None
        elif cur is not None and line.startswith("[bfq"):
            out[cur].append(line)
    return out


def arm(name, env_extra, ks, reps, trace_ks, scale):
    env = dict(os.environ)
    env.pop("BFQ_COMMIT_TRACE", None)
    env.update(env_extra)
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--scale", str(scale), "--ks", ",".join(map(str, ks)),
           "--reps", str(reps), "--trace-ks", ",".join(map(str, trace_ks))]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stderr[-4000:])
        raise SystemExit("arm %s failed" % name)
    res = json.loads(r.stdout.strip().splitlines()[-1])
    res["arm"] = name
    res["trace"] = traces(r.stderr)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--full-reps", type=int, default=3)
    ap.add_argument("--ks", default=",".join(map(str, KS)))
    ap.add_argument("--parent-lib", default=None, help="libbfq_gpumatch.so of the commit to compare with (k <= 64)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--trace-ks", default="")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    ks = [int(x) for x in a.ks.split(",") if x]
    if a.child:
        print(json.dumps(run_child(ks, a.reps, [int(x) for x in a.trace_ks.split(",") if x], a.scale)))
        return
    name, limit = gpu_info()
    print("GPU %s, power limit %s" % (name, limit), flush=True)
    runs = []
    small = [k for k in ks if k <= 64]
    if a.parent_lib and small:
        for _ in range(a.rounds):
            runs.append(arm("delta", {"BFQ_DELTA_COMMIT": "1"}, small, a.reps, [], a.scale))
            runs.append(arm("parent", {"BFQ_DELTA_COMMIT": "1", "BFQ_LIB": os.path.abspath(a.parent_lib)}, small, a.reps, [], a.scale))
    runs.append(arm("delta", {"BFQ_DELTA_COMMIT": "1"}, ks, a.reps, [k for k in (1, 1000) if k in ks], a.scale))
    runs.append(arm("full", {"BFQ_DELTA_COMMIT": "0"}, ks, a.full_reps, [], a.scale))
    print("GPU %s, power limit %s: median [min, max] ms of one commit, per arm run" % (name, limit))
    for k in ks:
        cells = []
        for r in runs:
            v = r["ms"].get(str(k))
            if v:
                paths = set(r["paths"][str(k)])
                cells.append("%s %.1f [%.1f, %.1f]%s" % (r["arm"], float(np.median(v)), min(v), max(v),
                                                         "" if paths == {"delta" if r["arm"] != "full" else "full"} else " " + "/".join(sorted(paths))))
        print("k=%4d  %s" % (k, "  |  ".join(cells)))


if __name__ == "__main__":
    main()
