"""Time the inverse match (retained-message match) on config C5: the host call against another build, concurrent callers on one
handle, the device-resident call, and retain keys gathered on the device against the host's.

Input: C5 at --scale (1.0 = 1M retained topics, 100k wildcard filters), seeded, the same for every build; limit 10
(RetainMessageMatchLimit's default) and unlimited. Every call ends in a device synchronise, so calls are timed with a host clock.

  single   bfq_rmatch from one thread: median and min of --iters calls after --warmup, per build. With --lib name=path, the
           builds alternate run by run (--runs), each run in a fresh process; each build prints the SHA-256 of its ids,
           which must agree between builds.
  threads  aggregate filters/s of 1, 2, 4 and 8 threads calling bfq_rmatch on one handle (--iters calls each).
  device   bfq_rmatch_device: wall time of the call, its device time (inputs resident to ids expanded) and rmatch_kernel's.
  keys     retain keys of one unlimited result: bfq_rretain_keys_device (sizing, scan and copy, ended by a synchronise)
           against bfq_rresult_retain_keys (sizing pass and copy pass on the host); the bytes must be identical.

    python tools/rmatch_device_bench.py [--lib name=path ...] [--runs 3] [--scale 1.0] [--iters 5] [--warmup 2]

threads, device and keys run on the in-tree library only. The card's name and power limit are printed with the numbers.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

_vp, _i32, _i64 = C.c_void_p, C.c_int32, C.c_int64
# the part of the C-ABI every build has: a build from before bfq_rmatch_device can be timed too
_HOST_ABI = {
    "bfq_last_error": (C.c_char_p, []),
    "bfq_rindex_create": (_i32, [_i32, C.POINTER(_vp)]),
    "bfq_rindex_destroy": (None, [_vp]),
    "bfq_rindex_add": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp]),
    "bfq_rindex_commit": (_i32, [_vp]),
    "bfq_rmatch": (_i32, [_vp, _vp, _vp, _i32, _vp, _vp, _vp, _i64, _vp, C.POINTER(_vp)]),
    "bfq_rresult_ids": (_vp, [_vp, C.POINTER(_i64)]),
    "bfq_rresult_retain_keys": (_i64, [_vp, _vp, _vp, _i64, _vp]),
    "bfq_rresult_free": (None, [_vp]),
}


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return {"gpu": name, "power_limit": limit}


class Setup:
    """C5 loaded into one committed handle of the library at `path`"""

    def __init__(self, path, scale):
        from bifromq_b200 import workload
        lib = C.CDLL(path)
        for name, (res, args) in _HOST_ABI.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        self.lib = lib
        self.w = w = workload.Workload("C5", scale=scale)
        bl = [t.encode() for t in w.tenants]
        self.tb = np.frombuffer(b"".join(bl), np.uint8).copy()
        self.toff = np.zeros(len(bl) + 1, np.int64)
        self.toff[1:] = np.cumsum([len(b) for b in bl])
        self.nt = len(bl)
        self.h = _vp()
        self.check(lib.bfq_rindex_create(0, C.byref(self.h)))
        self.ids_out = np.zeros(w.n_topics, np.int64)
        tt = np.ascontiguousarray(w.topic_tenant[:w.n_topics], np.int32)
        self.check(lib.bfq_rindex_add(self.h, self.tb.ctypes.data, self.toff.ctypes.data, self.nt, w.topics.ctypes.data,
                                      w.topic_off.ctypes.data, tt.ctypes.data, w.n_topics, self.ids_out.ctypes.data))
        self.check(lib.bfq_rindex_commit(self.h))
        self.n = w.n_query_filters
        self.ft = np.ascontiguousarray(w.filter_tenant[:self.n], np.int32)
        self.foff = np.ascontiguousarray(w.filter_off[:self.n + 1], np.int64)
        self.limits = {"limit10": np.full(self.n, 10, np.int64), "unlimited": None}

    def check(self, rc):
        if rc != 0:
            raise RuntimeError("bfq error %d: %s" % (rc, self.lib.bfq_last_error().decode()))

    def rmatch(self, lim):
        r = _vp()
        self.check(self.lib.bfq_rmatch(self.h, self.tb.ctypes.data, self.toff.ctypes.data, self.nt, self.w.filters.ctypes.data,
                                       self.foff.ctypes.data, self.ft.ctypes.data, self.n,
                                       None if lim is None else lim.ctypes.data, C.byref(r)))
        return r

    def ids(self, r):
        k = _i64(0)
        p = self.lib.bfq_rresult_ids(r, C.byref(k))
        return np.frombuffer((C.c_uint8 * (k.value * 8)).from_address(p), np.int64).copy() if k.value else np.zeros(0, np.int64)


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return {"median_ms": round(statistics.median(ts), 3), "min_ms": round(min(ts), 3)}


def child_single(a):
    """one run of the host call on the build at BFQ_LIB (or in tree) -> JSON line"""
    from bifromq_b200 import _native
    s = Setup(os.environ.get("BFQ_LIB") or _native.LIB_PATH, a.scale)
    out = {}
    for name, lim in s.limits.items():
        def one():
            s.lib.bfq_rresult_free(s.rmatch(lim))
        out[name] = timed(one, a.iters, a.warmup)
        out[name]["filters_per_s"] = round(s.n / (out[name]["median_ms"] / 1e3))
        r = s.rmatch(lim)
        ids = s.ids(r)
        s.lib.bfq_rresult_free(r)
        out[name]["ids"] = int(len(ids))
        out[name]["ids_sha256"] = hashlib.sha256(ids.tobytes()).hexdigest()[:16]
    print(json.dumps(out))


def in_tree(a):
    """threads, device and keys on the in-tree library"""
    import torch

    from bifromq_b200 import _native as N
    N.load_library()
    s = Setup(N.LIB_PATH, a.scale)
    lib = N.lib
    dev = torch.device("cuda", 0)
    out = {"threads": {}, "device": {}, "keys": {}}
    for name, lim in s.limits.items():
        rows = {}
        for k in (1, 2, 4, 8):
            def worker():
                for _ in range(a.iters):
                    s.lib.bfq_rresult_free(s.rmatch(lim))
            for _ in range(a.warmup):
                s.lib.bfq_rresult_free(s.rmatch(lim))
            ts = [threading.Thread(target=worker) for _ in range(k)]
            t0 = time.perf_counter()
            for t in ts:
                t.start()
            for t in ts:
                t.join()
            dt = time.perf_counter() - t0
            rows[str(k)] = {"filters_per_s": round(k * a.iters * s.n / dt), "wall_ms": round(dt * 1e3, 2)}
        base = rows["1"]["filters_per_s"]
        for r in rows.values():
            r["vs_1_thread"] = round(r["filters_per_s"] / base, 2)
        out["threads"][name] = rows
        # the device-resident call
        d_f = torch.from_numpy(s.w.filters).to(dev)
        d_off = torch.from_numpy(s.foff).to(dev)
        d_ft = torch.from_numpy(s.ft).to(dev)
        d_lim = None if lim is None else torch.from_numpy(lim).to(dev)
        torch.cuda.synchronize()
        res = N.BfqRDeviceResult()
        dev_ms, kern_ms = [], []

        def dcall():
            N.check(lib.bfq_rmatch_device(s.h, s.tb.ctypes.data, s.toff.ctypes.data, s.nt, d_f.data_ptr(), d_off.data_ptr(),
                                          d_ft.data_ptr(), s.n, None if d_lim is None else d_lim.data_ptr(), None, C.byref(res)))
            dev_ms.append(res.device_ms)
            kern_ms.append(res.kernel_ms)
            lib.bfq_rdevice_result_release(C.byref(res))
        wall = timed(dcall, a.iters, a.warmup)
        out["device"][name] = dict(wall, device_ms=round(statistics.median(dev_ms[a.warmup:]), 3),
                                   rmatch_kernel_ms=round(statistics.median(kern_ms[a.warmup:]), 3))
    # retain keys of one unlimited result: device gather against the host's
    N.check(lib.bfq_rmatch_device(s.h, s.tb.ctypes.data, s.toff.ctypes.data, s.nt, d_f.data_ptr(), d_off.data_ptr(),
                                  d_ft.data_ptr(), s.n, None, None, C.byref(res)))
    hr = s.rmatch(None)
    n_ids = res.n_ids
    d_koff = torch.zeros(n_ids + 1, dtype=torch.int64, device=dev)
    n_bytes = _i64(0)
    N.check(lib.bfq_rretain_keys_device(s.h, C.byref(res), d_koff.data_ptr(), None, 0, None, C.byref(n_bytes)))
    d_keys = torch.zeros(max(n_bytes.value, 1), dtype=torch.uint8, device=dev)

    def dkeys():
        N.check(lib.bfq_rretain_keys_device(s.h, C.byref(res), d_koff.data_ptr(), d_keys.data_ptr(), n_bytes.value, None,
                                            C.byref(n_bytes)))
        torch.cuda.synchronize()
    h_koff = np.zeros(n_ids + 1, np.int64)
    h_blob = np.zeros(max(n_bytes.value, 1), np.uint8)

    def hkeys():
        total = s.lib.bfq_rresult_retain_keys(s.h, hr, None, 0, h_koff.ctypes.data)
        assert s.lib.bfq_rresult_retain_keys(s.h, hr, h_blob.ctypes.data, total, h_koff.ctypes.data) == total
    out["keys"] = {"ids": int(n_ids), "bytes": int(n_bytes.value), "device": timed(dkeys, a.iters, a.warmup),
                   "host": timed(hkeys, a.iters, a.warmup)}
    same = (np.array_equal(d_koff.cpu().numpy(), h_koff) and
            np.array_equal(d_keys.cpu().numpy()[:n_bytes.value], h_blob[:n_bytes.value]))
    out["keys"]["identical"] = bool(same)
    s.lib.bfq_rresult_free(hr)
    lib.bfq_rdevice_result_release(C.byref(res))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], help="name=path of a build to A/B (default: the in-tree library)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child_single(a)
        return
    from bifromq_b200 import _native
    builds = [tuple(x.split("=", 1)) for x in a.lib] or [("this", _native.LIB_PATH)]
    single = {name: [] for name, _ in builds}
    for _ in range(a.runs):
        for name, path in builds:
            env = dict(os.environ, BFQ_LIB=os.path.abspath(path))
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--scale", str(a.scale), "--iters", str(a.iters),
                   "--warmup", str(a.warmup)]
            single[name].append(json.loads(subprocess.run(cmd, env=env, check=True, capture_output=True, text=True).stdout.strip().splitlines()[-1]))
    out = dict(gpu_info(), config="C5", scale=a.scale, single=single)
    out.update(in_tree(a))
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
