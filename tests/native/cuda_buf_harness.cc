// cuda_buf_harness.cc — drives bifromq_b200/csrc/cuda_buf.h against the counting stand-in runtime next to it
// (tests/native/cuda_runtime.h) and prints what it observed as one JSON object; tests/test_host_cuda_buf_cpu.py asserts on it.
#include <cstdio>
#include <string>
#include <utility>
#include <vector>

#include "cuda_buf.h"

using bfq::DeviceBuf;
using bfq::PinnedBuf;

namespace {

std::string out = "{";
void put(const char* key, const std::string& json_value) {
    if (out.size() > 1) out += ", ";
    out += std::string("\"") + key + "\": " + json_value;
}
void put(const char* key, long v) { put(key, std::to_string(v)); }
void put(const char* key, const std::vector<std::string>& v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); i++) s += (i ? ", \"" : "\"") + v[i] + "\"";
    put(key, s + "]");
}
std::string quoted(const std::string& s) {
    std::string q = "\"";
    for (char c : s) q += c == '"' || c == '\\' ? std::string("\\") + c : std::string(1, c);
    return q + "\"";
}
// the log entries since `mark`
std::vector<std::string> since(size_t mark) {
    const auto& l = fake_cuda::state().log;
    return std::vector<std::string>(l.begin() + (long) mark, l.end());
}

int32_t reserve_or_fail(DeviceBuf<int>& buf, size_t n) {
    BFQ_CUDA_TRY(buf.reserve(n));
    return BFQ_OK;
}

}  // namespace

int main() {
    auto& st = fake_cuda::state();
    {
        // ---- reserve: exact sizes, no-op when it fits, free before the new allocation
        DeviceBuf<uint32_t> b;
        size_t m = st.log.size();
        b.reserve(0);
        put("reserve0_log", since(m));
        put("reserve0_cap", (long) b.cap);
        put("reserve0_null", (long) (b.p == nullptr));
        m = st.log.size();
        b.reserve(10);
        put("reserve10_log", since(m));
        put("reserve10_cap", (long) b.cap);
        put("reserve10_bytes", (long) b.bytes());
        m = st.log.size();
        b.reserve(7);
        put("reserve_fits_log", since(m));
        put("reserve_fits_cap", (long) b.cap);
        m = st.log.size();
        b.reserve(11);
        put("reserve_grow_log", since(m));
        put("reserve_grow_cap", (long) b.cap);

        // ---- grow: at least 1.5x, keeps its prefix, copies and synchronises before freeing the old buffer
        DeviceBuf<int> g;
        g.reserve(4);
        for (int i = 0; i < 4; i++) g.p[i] = 100 + i;
        m = st.log.size();
        g.grow(5, 3, nullptr);
        put("grow_log", since(m));
        put("grow_cap", (long) g.cap);
        put("grow_prefix", "[" + std::to_string(g.p[0]) + ", " + std::to_string(g.p[1]) + ", " + std::to_string(g.p[2]) + "]");
        m = st.log.size();
        g.grow(6, 6, nullptr);
        put("grow_fits_log", since(m));
        g.grow(7, 0, nullptr);
        put("grow_again_cap", (long) g.cap);
        int* before = g.p;
        st.fail_next_alloc = true;
        const cudaError_t ge = g.grow(100, 9, nullptr);
        put("grow_failed_rc", (long) ge);
        put("grow_failed_kept", (long) (g.p == before && g.cap == 9));

        // ---- moves: the source is left empty, the target's old allocation is freed
        DeviceBuf<int> a, t;
        a.reserve(8);
        t.reserve(16);
        int* ap = a.p;
        const long frees = st.device_frees;
        t = std::move(a);
        put("move_assign_frees", st.device_frees - frees);
        put("move_assign_target", (long) (t.p == ap && t.cap == 8));
        put("move_assign_source_empty", (long) (a.p == nullptr && a.cap == 0));
        DeviceBuf<int> c(std::move(t));
        put("move_construct_target", (long) (c.p == ap && c.cap == 8));
        put("move_construct_source_empty", (long) (t.p == nullptr && t.cap == 0));

        // ---- device and pinned allocations go to their own calls
        const long d0 = st.device_allocs, df0 = st.device_frees;
        PinnedBuf<unsigned long long> h;
        m = st.log.size();
        h.reserve(3);
        h.reserve(5);
        h.release();
        put("pinned_log", since(m));
        put("pinned_device_calls", (st.device_allocs - d0) + (st.device_frees - df0));

        // ---- BFQ_CUDA_TRY: BFQ_E_CUDA, the failed expression and CUDA's message in bfq_last_error(); the buffer is left empty
        DeviceBuf<int> e;
        e.reserve(2);
        st.fail_next_alloc = true;
        put("try_rc", (long) reserve_or_fail(e, 64));
        put("try_error", quoted(bfq_last_error()));
        put("try_buffer_empty", (long) (e.p == nullptr && e.cap == 0));
        put("try_ok_rc", (long) reserve_or_fail(e, 64));

        // ---- carve: one layout sizes the arena and hands out its arrays, each at a 256-byte boundary
        DeviceBuf<uint8_t> arena;
        uint8_t* a8 = nullptr;
        unsigned long long* a64 = nullptr;
        uint32_t* a32 = nullptr;
        uint16_t* a16 = nullptr;
        size_t n64 = 5;
        auto layout = [&](bfq::Carve& c) {
            a8 = c.take<uint8_t>(3);
            a64 = c.take<unsigned long long>(n64);
            a32 = c.take<uint32_t>(0);
            a16 = c.take<uint16_t>(2);
        };
        auto offsets = [&]() {
            const uint8_t* b = arena.p;
            return "[" + std::to_string((const uint8_t*) a8 - b) + ", " + std::to_string((const uint8_t*) a64 - b) + ", " +
                   std::to_string((const uint8_t*) a32 - b) + ", " + std::to_string((const uint8_t*) a16 - b) + "]";
        };
        m = st.log.size();
        put("carve_rc", (long) bfq::carve(arena, "arena", layout));
        put("carve_log", since(m));
        put("carve_offsets", offsets());
        m = st.log.size();
        bfq::carve(arena, "arena", layout);
        put("carve_fits_log", since(m));
        n64 = 100;
        m = st.log.size();
        bfq::carve(arena, "arena", layout);
        put("carve_grow_log", since(m));
        put("carve_grow_offsets", offsets());
        n64 = 1000;
        st.fail_next_alloc = true;
        put("carve_failed_rc", (long) bfq::carve(arena, "test arena", layout));
        put("carve_failed_error", quoted(bfq_last_error()));
    }
    // every buffer above is out of scope: each allocation has been freed exactly once
    put("device_allocs", st.device_allocs);
    put("device_frees", st.device_frees);
    put("pinned_allocs", st.pinned_allocs);
    put("pinned_frees", st.pinned_frees);
    printf("%s}\n", out.c_str());
    return 0;
}
