"""The owning CUDA buffer of every host-side source (bifromq_b200/csrc/cuda_buf.h), without a GPU.

tests/native/cuda_buf_harness.cc is compiled with g++ against a stand-in cuda_runtime.h (tests/native/) that backs device
and pinned memory with malloc, logs every call and counts allocations and frees per allocator. The sizes matter beyond
memory use: device_bytes in bfq_index_stats / bfq_rindex_stats is the sum of the buffers' bytes(), and the initial buffer
sizes tests/test_gpu_edges.py relies on come from reserve."""
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_OF_MEMORY = 2   # the stand-in's cudaErrorMemoryAllocation
BFQ_E_CUDA = -2


def test_cuda_buf_allocation_rules(tmp_path):
    csrc = os.path.join(ROOT, "bifromq_b200", "csrc")
    native = os.path.join(ROOT, "tests", "native")
    exe = str(tmp_path / "cuda_buf_harness")
    # the stand-in runtime header comes first on the include path
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-Wall", "-Wextra", "-Werror", "-I" + native, "-I" + csrc,
                           os.path.join(native, "cuda_buf_harness.cc"), os.path.join(csrc, "errors.cc"), "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    o = json.loads(r.stdout)

    # reserve: exactly n elements, nothing when they fit; reserve(0) allocates nothing at all
    assert o["reserve0_log"] == [] and o["reserve0_cap"] == 0 and o["reserve0_null"] == 1
    assert o["reserve10_log"] == ["malloc 40"] and o["reserve10_cap"] == 10 and o["reserve10_bytes"] == 40
    assert o["reserve_fits_log"] == [] and o["reserve_fits_cap"] == 10
    # a reserve that does not fit frees the old buffer before it allocates the new one
    assert o["reserve_grow_log"] == ["free", "malloc 44"] and o["reserve_grow_cap"] == 11

    # grow: at least 1.5x the capacity; the kept prefix is copied, the stream synchronised, then the old buffer freed
    assert o["grow_log"] == ["malloc 24", "memcpy 12", "sync", "free"] and o["grow_cap"] == 6
    assert o["grow_prefix"] == [100, 101, 102]
    assert o["grow_fits_log"] == []
    assert o["grow_again_cap"] == 9
    assert o["grow_failed_rc"] == OUT_OF_MEMORY and o["grow_failed_kept"] == 1   # a failed grow keeps the old buffer

    # moves hand the allocation over and leave the source empty; a move-assignment frees the target's old allocation
    assert o["move_assign_frees"] == 1 and o["move_assign_target"] == 1 and o["move_assign_source_empty"] == 1
    assert o["move_construct_target"] == 1 and o["move_construct_source_empty"] == 1

    # pinned buffers use the pinned calls only
    assert o["pinned_log"] == ["malloc_host 24", "free_host", "malloc_host 40", "free_host"]
    assert o["pinned_device_calls"] == 0

    # BFQ_CUDA_TRY returns BFQ_E_CUDA with the failed expression and CUDA's message in bfq_last_error()
    assert o["try_rc"] == BFQ_E_CUDA and o["try_error"] == "buf.reserve(n): out of memory"
    assert o["try_buffer_empty"] == 1 and o["try_ok_rc"] == 0

    # carve: the counting pass sizes the arena (3 bytes, 5 x 8 at 256, an empty array and 2 x 2 at 512); the placing pass
    # hands out those offsets. Arrays never overlap and each starts on a 256-byte boundary.
    assert o["carve_rc"] == 0 and o["carve_log"] == ["malloc 516"] and o["carve_offsets"] == [0, 256, 512, 512]
    assert o["carve_fits_log"] == []
    assert o["carve_grow_log"] == ["free", "malloc 1284"] and o["carve_grow_offsets"] == [0, 256, 1280, 1280]
    assert o["carve_failed_rc"] == BFQ_E_CUDA and o["carve_failed_error"] == "test arena: out of memory"

    # every allocation was freed exactly once
    assert o["device_allocs"] == o["device_frees"] > 0
    assert o["pinned_allocs"] == o["pinned_frees"] == 2
