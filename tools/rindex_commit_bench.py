#!/usr/bin/env python
"""Times bfq_rindex_commit at BASELINE C5 size (1M retained topics, 1000 tenants): the load and full commit, delta commits of a
few typical retain-store mutations, and the commit that the garbage bound turns into a full build. Each time is wall time around
commit(), which returns after the device is patched (it ends in a stream synchronise). Prints one JSON line.
Run on a GPU machine:  python tools/rindex_commit_bench.py [scale]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return {"gpu": name, "power_limit": power}
    except Exception as e:   # the numbers are still valid, only unlabelled
        return {"gpu": None, "power_limit": None, "gpu_query_error": str(e)}


def main():
    import bifromq_b200
    from bifromq_b200 import retain, workload
    bifromq_b200.load_library()
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    w = workload.Workload("C5", scale=scale)
    tenants = w.tenants
    tt = w.topic_tenant[:w.n_topics]
    idx = retain.GpuTopicMatchIndex(0)
    t0 = time.perf_counter()
    idx.add_blobs(tenants, w.topics, w.topic_off, tt)
    load_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    idx.commit()
    full_s = time.perf_counter() - t0
    out = {"config": "C5", "scale": scale, "topics": int(w.n_topics), "tenants": len(tenants), "load_s": round(load_s, 3),
           "full_commit_s": round(full_s, 3), "delta_commits": []}
    out.update(gpu_info())

    def timed(label):
        full_before = idx.stats()["full_commits"]
        t0 = time.perf_counter()
        idx.commit()
        dt = time.perf_counter() - t0
        st = idx.stats()
        out["delta_commits"].append({"what": label, "ms": round(dt * 1e3, 3),
                                     "path": "full" if st["full_commits"] > full_before else "delta",
                                     "rebuilt_tenants": st["rebuilt_tenants"]})
        sys.stderr.write("== %s: %.3f ms\n" % (label, dt * 1e3))
        return dt
    sizes = np.bincount(tt, minlength=len(tenants))
    big = tenants[int(np.argmax(sizes))]
    small = [tenants[i] for i in np.argsort(sizes, kind="stable")[:8]]
    idx.add(big, ["delta/one/topic"])
    timed("one topic into the largest tenant (%s, %d topics)" % (big, int(sizes.max())))
    idx.remove(big, "delta/one/topic")
    timed("one remove from the largest tenant")
    idx.add("zz-new-tenant", ["a/b/c"])
    timed("one topic creating a new tenant")
    idx.add_blobs(small, *_blob(["d8/x"] * 8), np.arange(8, dtype=np.int32))
    timed("8 tenants x 1 topic")
    idx.add(small[0], ["bulk/%d/x" % i for i in range(1000)])
    timed("1000 topics into one tenant")
    # touch the largest tenant until the garbage bound turns a commit into a full build
    before = idx.stats()["full_commits"]
    deltas = 0
    for i in range(100000):
        idx.add(big, ["touch/%d" % i])
        t0 = time.perf_counter()
        idx.commit()
        dt = time.perf_counter() - t0
        if idx.stats()["full_commits"] > before:
            out["garbage_bound_full_commit"] = {"ms": round(dt * 1e3, 3), "delta_commits_before": deltas}
            break
        deltas += 1
    out["stats"] = idx.stats()
    print(json.dumps(out))


def _blob(strs):
    from bifromq_b200 import _native as N
    return N.as_blob(strs)


if __name__ == "__main__":
    main()
