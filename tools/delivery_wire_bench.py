"""Time bfq_delivery_encode behind bfq_delivery_device, and the same encoding on the host.

Input: the shapes of tools/delivery_bench.py (the C4 workload's routes as generated, and re-keyed to about 10k and 100k
deliverers), matched once (MaxGroupFanout 100), with one publisher pack of --msg-bytes payload bytes per topic position. Per
shape, rounds alternate `--iters` bfq_delivery_device calls and `--iters` (bfq_delivery_device + bfq_delivery_encode) calls,
each block timed with CUDA events after warm-up (every call includes its stream synchronisations). Reported per shape: the
median per call of both legs and of their difference (the encode), the bytes written, the encode's output rate, and that rate
as a share of the H100 SXM's 3.35 TB/s HBM3 bandwidth counted as a write-plus-read bound (every output byte is read from a
table or the caller's packs and written once: 2 x bytes over the encode time). The host leg encodes the first --host-packs
packs of the same nesting with the restatement in tests/delivery_wire.py (MatchInfos built from the route KV) and reports
its rate and the time the whole batch would take at that rate (extrapolated, labelled so). Prints the GPU name and power limit.

    python tools/delivery_wire_bench.py [--scale 0.1] [--msg-bytes 1000] [--iters 10] [--rounds 5] [--warmup 3]
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

HBM_BYTES_PER_S = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C4")
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--msg-bytes", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=10, help="calls per timed block")
    ap.add_argument("--rounds", type=int, default=5, help="alternating (delivery block, delivery + encode block) rounds")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-packs", type=int, default=20000)
    ap.add_argument("--rekey", default="0,10000,100000", help="0 = the workload's own deliverer keys")
    args = ap.parse_args()
    import torch

    import bifromq_b200
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
    # one PublisherPack per position: {publisher = 1: a client id, message = 2: msg-bytes of payload}
    rng = np.random.default_rng(1)
    pack = W.field(1, b"client") + W.field(2, rng.integers(0, 256, args.msg_bytes, dtype=np.uint8).tobytes())
    pub_off = np.arange(n + 1, dtype=np.int64)
    d_pub_off = torch.from_numpy(pub_off).to(dev)
    d_pp = torch.from_numpy(np.frombuffer(pack * n, np.uint8).copy()).to(dev)
    d_pp_off = torch.from_numpy(np.arange(n + 1, dtype=np.int64) * len(pack)).to(dev)
    tblob = bifromq_b200.GpuRouteIndex.tenant_blob(tenants)
    kb, vb = w.keys.tobytes(), w.vals.tobytes()
    for nd in [int(x) for x in args.rekey.split(",")]:
        idx = bifromq_b200.GpuRouteIndex(0)
        if nd == 0:
            keys = [kb[w.key_off[i]:w.key_off[i + 1]] for i in range(w.n_routes)]
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
        wire_args = (tblob, d_topics.data_ptr(), d_off.data_ptr(), d_pub_off.data_ptr(), d_pp.data_ptr(), d_pp_off.data_ptr())
        dl = deliver()
        n_bytes = out.delivery_wire(dl, *wire_args, None, 0, stream).n_bytes
        buf = torch.empty(max(n_bytes, 1), dtype=torch.uint8, device=dev)

        def both():
            d = deliver()
            return d, out.delivery_wire(d, *wire_args, buf.data_ptr(), n_bytes, stream)
        for _ in range(args.warmup):
            deliver()
            both()
        torch.cuda.synchronize()
        ms = {"delivery": [], "delivery_encode": []}
        for _ in range(args.rounds):
            for leg, fn in (("delivery", deliver), ("delivery_encode", both)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    r = fn()
                e1.record()
                torch.cuda.synchronize()
                ms[leg].append(e0.elapsed_time(e1) / args.iters)
        dl, wr = r
        stats = idx.stats()
        # host leg: the first host-packs packs of the nesting, encoded with the restatement
        a = dl.arrays(dev)
        K = min(args.host_packs, dl.n_packs)
        t0 = time.perf_counter()
        infos, host_bytes = {}, 0
        pkg_of = np.repeat(np.arange(dl.n_packages), np.diff(a["pack_off"]))
        packs = []
        for k in range(K):
            t = int(a["pack_topic"][k])
            ms_ = []
            for j in range(int(a["match_off"][k]), int(a["match_off"][k + 1])):
                rnk, mem = int(a["match_rank"][j]), int(a["match_member"][j])
                if rnk not in infos:
                    v = vals_of[rnk] if nd else rnk
                    infos[rnk] = W.route_match_infos(keys[rnk], vb[w.val_off[v]:w.val_off[v + 1]])
                ms_.append(infos[rnk][0 if mem == 0xFFFFFFFF else mem])
            topic = bytes(w.topics[w.topic_off[t]:w.topic_off[t + 1]])
            packs.append((tenants[int(a["package_tenant"][pkg_of[k]])].encode(), [(W.topic_message_pack(topic, [pack]), ms_)]))
        host_bytes = sum(len(W.delivery_request([p])) for p in packs)
        host_s = time.perf_counter() - t0
        dl_ms, both_ms = float(np.median(ms["delivery"])), float(np.median(ms["delivery_encode"]))
        enc_ms = both_ms - dl_ms
        print(json.dumps({
            "config": args.config, "scale": args.scale, "rekey": nd, "msg_bytes": args.msg_bytes, "n_topics": n,
            "n_pairs": total, "n_packs": dl.n_packs, "n_deliverers": dl.n_deliverers, "n_bytes": wr.n_bytes,
            "n_match_infos": wr.n_match_infos, "n_skipped": wr.n_skipped, "wire_table_bytes": stats["wire_table_bytes"],
            "delivery_ms": round(dl_ms, 3), "delivery_ms_rounds": [round(x, 3) for x in ms["delivery"]],
            "delivery_encode_ms": round(both_ms, 3), "delivery_encode_ms_rounds": [round(x, 3) for x in ms["delivery_encode"]],
            "encode_ms": round(enc_ms, 3), "encode_bytes_per_s": round(wr.n_bytes / (enc_ms * 1e-3), 1) if enc_ms > 0 else None,
            "encode_hbm_share_write_plus_read": round(2 * wr.n_bytes / (enc_ms * 1e-3) / HBM_BYTES_PER_S, 4) if enc_ms > 0 else None,
            "host_sample_packs": K, "host_sample_s": round(host_s, 3), "host_sample_bytes": host_bytes,
            "host_full_batch_s_extrapolated": round(host_s * dl.n_packs / max(K, 1), 1),
            "gpu": name, "power_limit": limit}), flush=True)
        out.release()
        idx.close()
        del buf
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
