#!/usr/bin/env python
"""Times bfq_index_commit's delta path at full BASELINE C4 size (10M filters): one SUB into tenants of different sizes, an UNSUB,
a new tenant; prints one JSON line. Run on a GPU machine:  BFQ_COMMIT_TRACE=1 python tools/commit_bench.py"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import bifromq_b200
    from bifromq_b200 import schema, workload
    scale = float(sys.argv[1]) if len(sys.argv) > 1 else 1.0
    w = workload.Workload("C4", scale=scale)
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    t0 = time.perf_counter()
    idx.commit()
    full_s = time.perf_counter() - t0
    names = w.tenants
    out = {"config": "C4", "scale": scale, "routes": w.n_routes, "tenants": w.n_tenants, "full_commit_s": round(full_s, 3), "delta_commits": []}

    def timed(label, adds=(), dels=()):
        idx.apply(adds=list(adds), dels=list(dels))
        t0 = time.perf_counter()
        idx.commit()
        dt = time.perf_counter() - t0
        out["delta_commits"].append({"what": label, "ms": round(dt * 1e3, 3)})
        sys.stderr.write("== %s: %.3f ms\n" % (label, dt * 1e3))
    url = schema.receiver_url(0, "newcomer", "d")
    for t in ["tenant999", "tenant500", "tenant100", "tenant10", "tenant1", "tenant0"]:
        if t in names:
            timed("one SUB into %s" % t, adds=[(schema.route_key(t, "delta/+/x", url), schema.incarnation_bytes(3))])
    timed("one SUB creating a new tenant", adds=[(schema.route_key("zz-new-tenant", "#", url), schema.incarnation_bytes(1))])
    timed("one UNSUB (tenant999's new route)", dels=[schema.route_key("tenant999", "delta/+/x", url)])
    timed("8 SUBs into 8 small tenants", adds=[(schema.route_key("tenant%d" % (900 + i), "d2/#", url), schema.incarnation_bytes(1)) for i in range(8)])
    out["stats"] = idx.stats()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
