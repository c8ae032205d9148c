"""The workspace pool, the call lease and the use events both indexes lease their workspaces through
(bifromq_b200/csrc/lease.h), without a GPU.

tests/native/lease_harness.cc drives lease.h with a fake workspace, compiled with g++ against the stand-in cuda_runtime.h
(tests/native/) that numbers streams and events, logs every call and can make the next stream or event creation fail. The
pool's order is the one tests/test_gpu_workspace_lease.py predicts each forward call's workspace with (PoolModel): the same
model is run here over a long acquire / give-back sequence."""
import json
import os
import random
import re
import subprocess

import test_gpu_workspace_lease as WL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bifromq_b200", "csrc")
NATIVE = os.path.join(ROOT, "tests", "native")
BFQ_E_CUDA, BFQ_E_STATE = -2, -4


def sequence(seed=11, n=600):
    """acquire / give-back steps that alternately fill and drain the pool: up to a dozen leased at once, back to none. A
    give-back names the k-th leased workspace, so the steps mean the same to the pool and to the model."""
    rng = random.Random(seed)
    steps, leased = [], 0
    for i in range(n):
        filling = (i // 40) % 2 == 0
        if leased == 0 or (rng.random() < (0.75 if filling else 0.25) and leased < 12):
            steps.append("A")
            leased += 1
        else:
            steps.append("G%d" % rng.randrange(leased))
            leased -= 1
    return steps


def run_harness(tmp_path, args):
    exe = str(tmp_path / "lease_harness")
    # the stand-in runtime header comes first on the include path
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I" + NATIVE, "-I" + CSRC,
                           os.path.join(NATIVE, "lease_harness.cc"), os.path.join(CSRC, "errors.cc"), "-o", exe])
    r = subprocess.run([exe] + args, capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout)


def test_lease_rules(tmp_path):
    steps = sequence()
    o = run_harness(tmp_path, steps)
    assert o["pool_keep"] == WL.POOL_KEEP

    # the pool hands out what PoolModel predicts at every step: LIFO, at most POOL_KEEP idle, the rest freed on return;
    # live counts every workspace made and not freed, idle or leased (bfq_rindex_stats slot 11)
    model, leased = WL.PoolModel(), []
    assert len(o["steps"]) == len(steps)
    for i, (s, (got, live, idle, freed)) in enumerate(zip(steps, o["steps"])):
        if s == "A":
            w, _ = model.acquire(0)
            leased.append(w)
            assert got == w, i
        else:
            model.give_back(leased.pop(int(s[1:])))
        assert freed == model.freed, i
        assert live == model.made - len(model.freed), i
        assert idle == len(model.idle), i
    assert model.made > WL.POOL_KEEP + 4 and len(model.freed) > 4
    assert max(idle for _, _, idle, _ in o["steps"]) == WL.POOL_KEEP

    # close: the idle workspaces are freed at once on the pool's device; a leased one when it comes back, on that device
    a, b, c = o["close_ids"]
    assert [x for x in o["close_log"] if not x.startswith(("event_", "stream_"))] == ["set_device 7", "delete ws%d" % a,
                                                                                     "delete ws%d" % b]
    assert o["close_freed"] == [a, b] and o["close_live"] == 1 and o["close_idle"] == 0
    assert o["late_log"][:2] == ["set_device 7", "delete ws%d" % c]
    assert o["late_freed"] == [c] and o["late_live"] == 0 and o["late_idle"] == 0

    # a failed init: BFQ_E_CUDA "workspace: ...", the stream it made is destroyed with it, the pool's count is unchanged
    assert o["init_failed_rc"] == BFQ_E_CUDA and o["init_failed_error"] == "workspace: out of memory"
    log = o["init_failed_log"]
    assert len(log) == 3 and log[0].startswith("stream_create ") and log[1].startswith("delete ws")
    assert log[2] == "stream_destroy " + log[0].split()[1]
    assert o["init_failed_out_null"] == 1 and o["init_failed_streams_left"] == 0 and o["init_failed_events_left"] == 0
    assert o["init_failed_live"] == 1
    assert o["stream_failed_rc"] == BFQ_E_CUDA and o["stream_failed_live"] == 1

    # use events: stream A's first use creates an event and its second reuses it; stream B gets a second event; release
    # waits for both. The workspace's next lease creates none and waits for the streams it used only.
    ea, ea2, eb = o["use_events"]
    assert o["use_first_a_log"] == ["event_create " + ea] and o["use_second_a_log"] == [] and ea2 == ea
    assert o["use_b_log"] == ["event_create " + eb] and eb != ea
    assert o["use_wait_log"] == ["event_sync " + ea, "event_sync " + eb]
    assert o["use_same_workspace"] == 1
    assert o["use_next_lease_log"] == [] and o["use_next_lease_event"] == ea
    assert o["use_next_wait_log"] == ["event_sync " + o["use_next_lease_event"]]

    # the call lease: an error return drains the workspace and gives it back; once a result has taken it, neither
    assert o["lease_error_rc"] == BFQ_E_STATE
    made = [x for x in o["lease_error_log"] if x.startswith(("stream_create", "event_create"))]
    assert [x for x in o["lease_error_log"] if x not in made] == ["drain ws%d" % o["lease_error_ws"], "sync"]
    assert o["lease_error_idle"] == 1
    assert o["lease_taken_rc"] == 0 and o["lease_taken_log"] == [] and o["lease_taken_same"] == 1
    assert o["lease_taken_idle"] == 0 and o["lease_taken_live"] == 1

    # every stream and event made was destroyed once
    assert o["streams_created"] == o["streams_destroyed"] > 0
    assert o["events_created"] == o["events_destroyed"] > 0


def test_one_pool_policy_and_no_device_wide_synchronise():
    """POOL_KEEP is defined once, in lease.h; no library source waits for the whole device (a match waits for its own
    workspace's streams only)"""
    defs, syncs = [], []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".h", ".cc")):
            continue
        with open(os.path.join(CSRC, name)) as f:
            text = f.read()
        defs += [name for _ in re.finditer(r"\bPOOL_KEEP\s*=", text)]
        if "cudaDeviceSynchronize" in text:
            syncs.append(name)
    assert defs == ["lease.h"]
    assert syncs == []
