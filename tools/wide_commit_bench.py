#!/usr/bin/env python
"""Times bfq_index_commit on an index with wide nodes: BASELINE C4 (10M filters) plus two IoT tenants of 100 000 and 5 000
devices (one subscriber per device at dev/<id>/state, plus dev/+/state and dev/#): their "dev" nodes hold every device, so
their children live in the shared tag table.

Prints the GPU name and power limit, then one JSON line per arm:
  * "delta": the full commit; one SUB into the 100k tenant; one SUB into a mid-size C4 tenant; one UNSUB; a new tenant; then
    50 SUBs into the 100k tenant, each committed on its own, with the path taken and the tag table's fill (stats 18..20)
    after each; the tier-0 device time of a 1M-topic batch over the IoT tenants before and after the 50 commits;
  * "full" (the same sequence in a subprocess with BFQ_DELTA_COMMIT=0: every commit a full build), the "before" arm.

    python tools/wide_commit_bench.py [--scale 1.0] [--arms delta,full]
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

IOT = [("iot-tenant-with-a-name-longer-than-any-c4-tenant-a", 100_000), ("iot-tenant-with-a-name-longer-than-any-c4-tenant-b", 5_000)]


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def iot_pairs(schema):
    pairs = []
    for tenant, n in IOT:
        for i in range(n):
            url = schema.receiver_url(i % 3, "r%d" % i, "inbox%d" % (i % 100))
            pairs.append((schema.route_key(tenant, "dev/%07d/state" % i, url), schema.incarnation_bytes(1)))
        pairs.append((schema.route_key(tenant, "dev/+/state", schema.receiver_url(1, "all", "d")), schema.incarnation_bytes(1)))
        pairs.append((schema.route_key(tenant, "dev/#", schema.receiver_url(1, "any", "d")), schema.incarnation_bytes(1)))
    return sorted(pairs)


def run_arm(scale):
    import bifromq_b200
    from bifromq_b200 import _native as N, schema, workload
    w = workload.Workload("C4", scale=scale)
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    ip = iot_pairs(schema)
    k, ko = N.as_blob([p[0] for p in ip])
    v, vo = N.as_blob([p[1] for p in ip])
    idx.load(k, ko, v, vo)
    t0 = time.perf_counter()
    idx.commit()
    out = {"delta_commit_env": os.environ.get("BFQ_DELTA_COMMIT", "1"), "config": "C4+IoT", "scale": scale,
           "routes": idx.stats()["routes"], "full_commit_s": round(time.perf_counter() - t0, 3), "commits": []}
    names = w.tenants + [t for t, _ in IOT]
    tenants = idx.tenant_blob(names)
    # 1M topics over the IoT tenants (90 % to the big one), devices that exist and some that do not
    rng = np.random.RandomState(7)
    n_topics = 1_000_000
    big = rng.rand(n_topics) < 0.9
    dev = np.where(big, rng.randint(0, 110_000, n_topics), rng.randint(0, 5_500, n_topics))
    tl = [b"dev/%07d/state" % d for d in dev.tolist()]
    tblob = np.frombuffer(b"".join(tl), np.uint8).copy()
    toff = np.zeros(n_topics + 1, np.int64)
    toff[1:] = np.cumsum([len(x) for x in tl])
    tt = np.where(big, len(names) - 2, len(names) - 1).astype(np.int32)

    def tier0_ms():
        best = []
        for _ in range(6):
            r = idx.match(tenants, tblob, toff, tt)
            r.close()
            best.append(idx.last_kernel_ms())
        return round(float(np.median(best[1:])), 4)

    def commit(label, adds=(), dels=()):
        idx.apply(adds=list(adds), dels=list(dels))
        st = idx.stats()
        t0 = time.perf_counter()
        idx.commit()
        dt = time.perf_counter() - t0
        st2 = idx.stats()
        rec = {"what": label, "ms": round(dt * 1e3, 3), "path": "delta" if st2["delta_commits"] > st["delta_commits"] else "full",
               "tag_usable": st2["tag_usable_slots"], "tag_used": st2["tag_used_slots"], "tag_overflowed_blocks": st2["tag_overflowed_blocks"]}
        out["commits"].append(rec)
        sys.stderr.write("== %s\n" % json.dumps(rec))
    url = schema.receiver_url(0, "newcomer", "d")
    big_t, mid_t = IOT[0][0], names[len(w.tenants) // 2]
    commit("one SUB into the 100k-device tenant", adds=[(schema.route_key(big_t, "dev/%07d/state" % 200_000, url), schema.incarnation_bytes(2))])
    commit("one SUB into a mid-size C4 tenant (%s)" % mid_t, adds=[(schema.route_key(mid_t, "delta/+/x", url), schema.incarnation_bytes(3))])
    commit("one UNSUB (the 100k tenant's new route)", dels=[schema.route_key(big_t, "dev/%07d/state" % 200_000, url)])
    commit("one SUB creating a new tenant", adds=[(schema.route_key("zz-new-tenant", "#", url), schema.incarnation_bytes(1))])
    out["tier0_ms_before_50"] = tier0_ms()
    for i in range(50):
        commit("SUB %d into the 100k-device tenant" % (i + 1),
               adds=[(schema.route_key(big_t, "dev/%07d/state" % (300_000 + 7919 * i), url), schema.incarnation_bytes(4))])
    out["tier0_ms_after_50"] = tier0_ms()
    out["stats"] = idx.stats()
    idx.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--arms", default="delta,full")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        print(json.dumps(run_arm(a.scale)))
        return
    name, limit = gpu_info()
    print("GPU %s, power limit %s" % (name, limit))
    for arm in a.arms.split(","):
        env = dict(os.environ)
        env["BFQ_DELTA_COMMIT"] = "1" if arm == "delta" else "0"
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--scale", str(a.scale)], env=env,
                           capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stderr[-4000:])
            raise SystemExit("arm %s failed" % arm)
        res = json.loads(r.stdout.strip().splitlines()[-1])
        res["arm"] = arm
        print(json.dumps(res))


if __name__ == "__main__":
    main()
