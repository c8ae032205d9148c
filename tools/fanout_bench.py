"""Time bfq_fanout_device alone: CUDA events around many calls on one completed match, after warm-up.

Shapes: the C4 workload's routes as generated (about 33 deliverers: the tile pass), and the same routes with the
delivererKey of every normal route re-keyed to about 10k and 100k deliverers (the global pass). The match and its device
CSR are made once per shape; only the fan-out is timed. Prints the GPU name and power limit, then one JSON line per shape.

    python tools/fanout_bench.py [--scale 0.1] [--iters 200] [--warmup 20] [--rekey 0,10000,100000]

Set BFQ_LIB to time another build of the library on the same inputs (A/B runs in one session).
"""
import argparse
import json
import os
import subprocess
import sys
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def rekey(keys, key_off, n_deliverers):
    """every normal route's delivererKey -> "k<NNNNNN>" chosen by a hash of its receiverId; keys re-sorted (values follow)"""
    out = []
    kb = keys.tobytes()
    for i in range(len(key_off) - 1):
        k = kb[key_off[i]:key_off[i + 1]]
        rlen = int.from_bytes(k[-2:], "big")
        rs = len(k) - 2 - rlen
        if k[rs - 1] != 1:   # group route: members stay as they are
            out.append((k, i))
            continue
        broker, rid, _ = k[rs:len(k) - 2].split(b"\0", 2)
        url = broker + b"\0" + rid + b"\0" + b"k%06d" % (zlib.crc32(rid) % n_deliverers)
        out.append((k[:rs] + url + len(url).to_bytes(2, "big"), i))
    out.sort()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4")
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rekey", default="0,10000,100000", help="0 = the workload's own deliverer keys")
    args = ap.parse_args()
    import torch

    import bifromq_b200
    from bifromq_b200 import _native as N
    from bifromq_b200.workload import Workload
    bifromq_b200.load_library()
    name, limit = gpu_info()
    print("gpu: %s, power limit %s, library %s" % (name, limit, N.LIB_PATH), flush=True)
    w = Workload(args.config, scale=args.scale)
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    n, tenants = w.n_topics, w.tenants
    d_topics = torch.from_numpy(np.ascontiguousarray(w.topics)).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(w.topic_off)).to(dev)
    d_tt = torch.from_numpy(np.ascontiguousarray(w.topic_tenant[:n])).to(dev)
    vb = w.vals.tobytes()
    for nd in [int(x) for x in args.rekey.split(",")]:
        idx = bifromq_b200.GpuRouteIndex(0)
        if nd == 0:
            idx.load(w.keys, w.key_off, w.vals, w.val_off)
        else:
            rk = rekey(w.keys, w.key_off, nd)
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
        for _ in range(args.warmup):
            fo = out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
        torch.cuda.synchronize()
        g0 = idx.stats()["global_fanouts"]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            fo = out.fanout(d_offsets.data_ptr(), d_ranks.data_ptr(), total, stream)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        path = "global" if idx.stats()["global_fanouts"] > g0 else "tile"
        print(json.dumps({"config": args.config, "scale": args.scale, "rekey": nd, "n_topics": n, "n_pairs": total,
                          "n_deliverers": fo.n_deliverers, "path": path, "ms_per_call": round(ms, 4),
                          "pairs_per_s": round(total / (ms / 1e3)) if ms > 0 else None, "gpu": name, "power_limit": limit}),
              flush=True)
        out.release()
        idx.close()


if __name__ == "__main__":
    main()
