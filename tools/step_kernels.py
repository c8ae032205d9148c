"""Per-kernel times of one forward step (bfq_match_device), from torch.profiler with CUDA activities.

bench.py reports tier 0 and the whole step; this shows where the rest of the step goes: the order stage (prep, scan,
scatter), tier 0, tier 1, finalize (span records to topic order, repeats), caps, and the memsets. It builds the index of one
config like bench.py does (same caps: MaxPersistentFanout INT_MAX, MaxGroupFanout 100), runs --warmup untimed steps, then
--steps steps under the profiler, one at a time (each waited for and released). The profile runs in this process only:
take end-to-end numbers from bench.py, not from here.

Writes <out>/step_kernels.json (per kernel and per stage: mean us per step, launches per step; the GPU name and power
limit) and <out>/step_kernels.md (the same as a table), and prints the table. A/B against another build: run it once per
build with BFQ_LIB pointing at that build's libbfq_gpumatch.so.

    python tools/step_kernels.py [--config C4] [--scale 1.0] [--steps 20] [--warmup 5] [--out profiles/step_kernels]
"""
import argparse
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

# stage of a kernel, by the first pattern its profiler name matches (order matters: tier 2 before tier 1)
STAGES = [
    ("order prep", r"order_prep_kernel"),
    ("order scan", r"order_scan_kernel"),
    ("order scatter", r"order_scatter_kernel"),
    ("tier 0", r"match_topics_lane_kernel"),
    ("tier 2", r"match_topics_kernel<true>"),
    ("tier 1", r"match_topics_kernel<false>"),
    ("finalize", r"finalize_kernel"),
    ("caps", r"caps_kernel|caps_advance_kernel"),
    ("memset", r"^Memset"),
]


def stage_of(name):
    for stage, pat in STAGES:
        if re.search(pat, name):
            return stage
    return "other"


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", default="C4", choices=["C1", "C2", "C3", "C4"])
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--max-pfanout", type=int, default=2 ** 31 - 1)
    ap.add_argument("--max-gfanout", type=int, default=100)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "step_kernels"))
    ap.add_argument("--label", default="", help="free text stored with the result (e.g. which build)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    import bifromq_b200
    from bifromq_b200 import _native as N
    from bifromq_b200.workload import Workload
    bifromq_b200.load_library()
    if not torch.cuda.is_available():
        raise SystemExit("step_kernels: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)

    w = Workload(args.config, scale=args.scale)
    idx = bifromq_b200.GpuRouteIndex(0)
    idx.load(w.keys, w.key_off, w.vals, w.val_off)
    idx.commit()
    tenants = idx.tenant_blob(w.tenants)
    n = w.n_topics
    blob_bytes = int(w.topic_off[-1])
    d_topics = torch.from_numpy(np.ascontiguousarray(w.topics[:max(blob_bytes, 1)])).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(w.topic_off)).to(dev)
    d_tt = torch.from_numpy(np.ascontiguousarray(w.topic_tenant[:max(n, 1)])).to(dev)
    nt = len(w.tenants)
    max_p, max_g = [args.max_pfanout] * nt, [args.max_gfanout] * nt
    stream = torch.cuda.current_stream(dev)

    def step():
        res = idx.match_device(tenants, d_topics.data_ptr(), d_off.data_ptr(), d_tt.data_ptr(), n, max_p, max_g,
                               stream=stream.cuda_stream, wait=False)
        res.wait()
        info = (res.n_distinct_topics, res.n_overflow_topics, res.tier0_ms)
        res.release()
        return info

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    tier0_ms = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            n_distinct, n_overflow, t0 = step()
            tier0_ms.append(t0)
        torch.cuda.synchronize()

    per_kernel = defaultdict(lambda: [0.0, 0])   # name -> [device us, launches]
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        per_kernel[e.name][0] += e.device_time
        per_kernel[e.name][1] += 1
    per_stage = defaultdict(lambda: [0.0, 0])
    for name, (us, k) in per_kernel.items():
        s = per_stage[stage_of(name)]
        s[0] += us
        s[1] += k
    steps = args.steps
    stages = [{"stage": s, "us_per_step": per_stage[s][0] / steps, "launches_per_step": per_stage[s][1] / steps}
              for s in [x for x, _ in STAGES] + ["other"] if s in per_stage]
    kernels = sorted(({"kernel": k, "stage": stage_of(k), "us_per_step": us / steps, "launches_per_step": c / steps}
                      for k, (us, c) in per_kernel.items()), key=lambda r: -r["us_per_step"])
    name, limits = gpu_info()
    out = {"config": args.config, "scale": args.scale, "steps": steps, "warmup": args.warmup, "topics": n,
           "distinct_topics": int(n_distinct), "tier2_topics": int(n_overflow), "label": args.label,
           "lib": N.LIB_PATH, "gpu": name, "power_limit_and_max_sm_clock": limits,
           "tier0_event_ms_mean": float(np.mean(tier0_ms)),
           "kernel_us_per_step_total": sum(r["us_per_step"] for r in stages), "stages": stages, "kernels": kernels}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "step_kernels.json"), "w") as f:
        json.dump(out, f, indent=1)
    lines = ["%s, %s x%g, %d steps (%s; power limit, max SM clock: %s)%s" % (args.config, "scale", args.scale, steps, name, limits,
                                                                             (" — " + args.label) if args.label else ""),
             "", "| stage | us / step | launches / step |", "|---|---:|---:|"]
    lines += ["| %s | %.1f | %.1f |" % (r["stage"], r["us_per_step"], r["launches_per_step"]) for r in stages]
    lines += ["| all kernels | %.1f | |" % out["kernel_us_per_step_total"], "",
              "| kernel | stage | us / step | launches / step |", "|---|---|---:|---:|"]
    lines += ["| %s | %s | %.1f | %.1f |" % (r["kernel"][:90], r["stage"], r["us_per_step"], r["launches_per_step"]) for r in kernels]
    text = "\n".join(lines) + "\n"
    with open(os.path.join(args.out, "step_kernels.md"), "w") as f:
        f.write(text)
    print(text)
    idx.close()


if __name__ == "__main__":
    main()
