// lease_harness.cc — drives the workspace pool, the call lease and the use events of bifromq_b200/csrc/lease.h with a fake
// workspace, against the stand-in runtime next to it (tests/native/cuda_runtime.h), and prints what it observed as one JSON
// object; tests/test_host_lease_cpu.py asserts on it.
//
// argv: the pool sequence, one step per argument: "A" acquires, "G<k>" gives back the k-th of the workspaces leased so far
// (in the order they were acquired).
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "lease.h"

using bfq::CallLease;
using bfq::Pool;
using bfq::StreamUses;

namespace {

std::string out = "{";
void put(const char* key, const std::string& json_value) {
    if (out.size() > 1) out += ", ";
    out += std::string("\"") + key + "\": " + json_value;
}
void put(const char* key, long v) { put(key, std::to_string(v)); }
std::string quoted(const std::string& s) {
    std::string q = "\"";
    for (char c : s) q += c == '"' || c == '\\' ? std::string("\\") + c : std::string(1, c);
    return q + "\"";
}
void put(const char* key, const std::vector<std::string>& v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); i++) s += (i ? ", " : "") + quoted(v[i]);
    put(key, s + "]");
}
std::string list(const std::vector<long>& v) {
    std::string s = "[";
    for (size_t i = 0; i < v.size(); i++) s += (i ? ", " : "") + std::to_string(v[i]);
    return s + "]";
}
// the log entries since `mark`
std::vector<std::string> since(size_t mark) {
    const auto& l = fake_cuda::state().log;
    return std::vector<std::string>(l.begin() + (long) mark, l.end());
}
std::string name(cudaEvent_t e) { return fake_cuda::name(e, "e"); }

std::vector<long> freed;   // workspace ids in the order they were deleted

// A workspace as the pool sees it: numbered in the order it was made, one stream and one event of its own, its use events.
struct FakeWs {
    static long next_id;
    long id = next_id++;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev = nullptr;
    bfq::UseEvents use_events;
    cudaError_t init(int) {
        cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        return e;
    }
    cudaError_t drain() {
        fake_cuda::state().log.push_back("drain ws" + std::to_string(id));
        return cudaStreamSynchronize(stream);
    }
    ~FakeWs() {
        fake_cuda::state().log.push_back("delete ws" + std::to_string(id));
        freed.push_back(id);
        if (ev) cudaEventDestroy(ev);
        if (stream) cudaStreamDestroy(stream);
    }
};
long FakeWs::next_id = 0;

// one call on a leased workspace: an error return before a result takes it, or a result that takes it
int32_t call(Pool<FakeWs>& pool, bool fails, FakeWs** result) {
    CallLease<FakeWs> lease(pool);
    const int32_t rc = pool.acquire(&lease.w);
    if (rc != BFQ_OK) return rc;
    if (fails) return BFQ_E_STATE;
    *result = lease.take();
    return BFQ_OK;
}

}  // namespace

int main(int argc, char** argv) {
    auto& st = fake_cuda::state();
    put("pool_keep", (long) bfq::POOL_KEEP);
    {
        // ---- the sequence: per step the workspace acquired or given back, the live and idle counts, the deletions so far
        Pool<FakeWs> pool;
        std::vector<FakeWs*> leased;
        std::string steps = "[";
        for (int i = 1; i < argc; i++) {
            FakeWs* w = nullptr;
            if (argv[i][0] == 'A') {
                if (pool.acquire(&w) != BFQ_OK) return 1;
                leased.push_back(w);
            } else {
                const long k = atol(argv[i] + 1);
                w = leased[(size_t) k];
                leased.erase(leased.begin() + k);
                pool.give_back(w);
            }
            // a give-back prints -1: w may have been deleted
            steps += std::string(i > 1 ? ", " : "") + "[" + std::to_string(argv[i][0] == 'A' ? w->id : -1) + ", " +
                     std::to_string(pool.live.size()) + ", " + std::to_string(pool.idle.size()) + ", " + list(freed) + "]";
        }
        put("steps", steps + "]");
        for (FakeWs* w : leased) pool.give_back(w);
    }
    freed.clear();
    {
        // ---- close: idle workspaces are freed at once, a leased one when it comes back, each on the pool's device
        Pool<FakeWs> pool;
        pool.device = 7;
        FakeWs *a = nullptr, *b = nullptr, *c = nullptr;
        pool.acquire(&a);
        pool.acquire(&b);
        pool.acquire(&c);
        const std::string ids = list({a->id, b->id, c->id});
        pool.give_back(a);
        pool.give_back(b);
        size_t m = st.log.size();
        freed.clear();
        pool.close();
        put("close_ids", ids);
        put("close_log", since(m));
        put("close_freed", list(freed));
        put("close_live", (long) pool.live.size());
        put("close_idle", (long) pool.idle.size());
        m = st.log.size();
        freed.clear();
        pool.give_back(c);
        put("late_log", since(m));
        put("late_freed", list(freed));
        put("late_live", (long) pool.live.size());
        put("late_idle", (long) pool.idle.size());
    }
    {
        // ---- a failed init: BFQ_E_CUDA, what it made is freed, the count is unchanged
        Pool<FakeWs> pool;
        FakeWs* w = nullptr;
        pool.acquire(&w);
        pool.give_back(w);
        w = nullptr;
        pool.acquire(&w);   // the idle one
        const long streams = st.streams_created - st.streams_destroyed, events = st.events_created - st.events_destroyed;
        FakeWs* failed = nullptr;
        st.fail_next_event = true;
        const size_t m = st.log.size();
        put("init_failed_rc", (long) pool.acquire(&failed));
        put("init_failed_error", quoted(bfq_last_error()));
        put("init_failed_log", since(m));
        put("init_failed_out_null", (long) (failed == nullptr));
        put("init_failed_streams_left", st.streams_created - st.streams_destroyed - streams);
        put("init_failed_events_left", st.events_created - st.events_destroyed - events);
        put("init_failed_live", (long) pool.live.size());
        st.fail_next_stream = true;
        put("stream_failed_rc", (long) pool.acquire(&failed));
        put("stream_failed_live", (long) pool.live.size());
        pool.give_back(w);
    }
    {
        // ---- use events: one per stream of a lease, owned by the workspace and reused by its next lease
        Pool<FakeWs> pool;
        cudaStream_t sa = nullptr, sb = nullptr;
        cudaStreamCreateWithFlags(&sa, cudaStreamNonBlocking);
        cudaStreamCreateWithFlags(&sb, cudaStreamNonBlocking);
        FakeWs* w = nullptr;
        pool.acquire(&w);
        cudaEvent_t a1 = nullptr, a2 = nullptr, b1 = nullptr;
        {
            StreamUses uses;
            size_t m = st.log.size();
            uses.event_for(w->use_events, sa, &a1);
            put("use_first_a_log", since(m));
            m = st.log.size();
            uses.event_for(w->use_events, sa, &a2);
            put("use_second_a_log", since(m));
            m = st.log.size();
            uses.event_for(w->use_events, sb, &b1);
            put("use_b_log", since(m));
            put("use_events", std::vector<std::string>{name(a1), name(a2), name(b1)});
            m = st.log.size();
            uses.wait(w->use_events);
            put("use_wait_log", since(m));
        }
        pool.give_back(w);
        FakeWs* again = nullptr;
        pool.acquire(&again);
        put("use_same_workspace", (long) (again == w));
        {
            StreamUses uses;
            cudaEvent_t e = nullptr;
            size_t m = st.log.size();
            uses.event_for(again->use_events, sb, &e);
            put("use_next_lease_log", since(m));
            put("use_next_lease_event", quoted(name(e)));
            m = st.log.size();
            uses.wait(again->use_events);
            put("use_next_wait_log", since(m));
        }
        pool.give_back(again);
        cudaStreamDestroy(sa);
        cudaStreamDestroy(sb);
    }
    {
        // ---- the call lease: drained and given back on an error return, left alone once a result has taken the workspace
        Pool<FakeWs> pool;
        FakeWs* kept = nullptr;
        size_t m = st.log.size();
        put("lease_error_rc", (long) call(pool, true, &kept));
        const std::vector<std::string> error_log = since(m);
        put("lease_error_log", error_log);
        put("lease_error_idle", (long) pool.idle.size());
        FakeWs* first = pool.idle.empty() ? nullptr : pool.idle.back();
        put("lease_error_ws", first ? first->id : -1);
        m = st.log.size();
        put("lease_taken_rc", (long) call(pool, false, &kept));
        put("lease_taken_log", since(m));
        put("lease_taken_same", (long) (kept == first));
        put("lease_taken_idle", (long) pool.idle.size());
        put("lease_taken_live", (long) pool.live.size());
        pool.give_back(kept);
    }
    // every pool above is gone: every stream and event made has been destroyed
    put("streams_created", st.streams_created);
    put("streams_destroyed", st.streams_destroyed);
    put("events_created", st.events_created);
    put("events_destroyed", st.events_destroyed);
    printf("%s}\n", out.c_str());
    return 0;
}
