// range_lookup.cu — batched range pruning on the dist-server side (SURVEY.md §8f rank 2).
//
// Before a publish is sent to the dist-workers, TenantRangeLookupCache.lookup
// (bifromq-dist/bifromq-dist-server/src/main/java/org/apache/bifromq/dist/server/scheduler/TenantRangeLookupCache.java:70-106) decides
// which KV ranges of the tenant can hold a matching route: every range publishes a Fact {firstGlobalFilterLevels,
// lastGlobalFilterLevels} (the smallest and largest filter it stores, tenant id as level 0), and a range stays a candidate iff
// the topic's EXPANSION SET (every filter that matches the topic) has a member inside [first, last]. The reference builds a
// one-topic trie and runs its lazy expansion iterator: seek(first), then compares the filter found with `last` — per topic, per
// candidate, behind a Caffeine cache. Here the whole batch is answered by one kernel, one thread per (topic, candidate):
//
// The expansion set of a topic t_1/../t_n (global mode: level 0 is the tenant id and is never wildcard-matched,
// TopicTrieNode.java:146-152) is an implicit trie: after i matched levels the children are "#" (terminal; not under the tenant
// level when t_1 starts with '$'), "+" and t_{i+1} (the last two only while i < n; "+" not for a '$' first level), and the
// node with i == n is itself a filter. seek(B) = the least member >= B in level-wise String.compareTo order is a lower-bound
// walk of that trie: follow B while it is a path, remember the deepest level that has a greater sibling, and complete
// minimally ("#" as soon as it is the smallest child). No trie is materialised and no level is stored: the walk reads the
// topic and the bounds through cursors, and the member it finds is described by how far it follows the bound, the one greater
// child it takes there and where its minimal completion starts, so neither a topic nor a bound has a level limit. UTF-8 byte
// order equals UTF-16 code-unit order on BMP text (what the MQTT edge admits).
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "cuda_buf.h"

using bfq::DeviceBuf;
using bfq::fail;

namespace {

__device__ const uint8_t kWild[2] = {'#', '+'};   // the level of kind 0 and of kind 1 below

struct Str {
    const uint8_t* p;
    int n;
};
__device__ __forceinline__ int cmp(Str a, Str b) {   // bytewise, shorter prefix first
    const int m = a.n < b.n ? a.n : b.n;
    for (int i = 0; i < m; i++)
        if (a.p[i] != b.p[i]) return a.p[i] < b.p[i] ? -1 : 1;
    return a.n == b.n ? 0 : (a.n < b.n ? -1 : 1);
}
__device__ __forceinline__ Str wild(int kind) { return Str{kWild + kind, 1}; }
__device__ __forceinline__ bool below_hash(Str s) { return s.n == 0 || s.p[0] < '#'; }   // s < "#"

// cursor over the levels of a topic ('/') or of a NUL-joined bound: `pos` is where the next level starts, past `len` once every
// level has been read
struct Levels {
    const uint8_t* s;
    int len, pos;
    uint8_t sep;
    __device__ bool more() const { return pos <= len; }
    __device__ Str peek() const {
        int e = pos;
        while (e < len && s[e] != sep) e++;
        return Str{s + pos, e - pos};
    }
    __device__ void skip(Str l) { pos += l.n + 1; }
    __device__ Str next() {
        const Str l = peek();
        skip(l);
        return l;
    }
};

// children of the node behind i matched levels, smallest first; kinds: 0 = "#", 1 = "+", 2 = the topic's level i + 1 (tx; only
// while has_t, i.e. i < n). wild = false under the tenant level of a '$' topic: no "#" / "+" there
__device__ __forceinline__ int children(bool wild, bool has_t, Str tx, int* kind) {
    int c = 0;
    if (has_t) {
        // order "#" < "+" always; place the topic level among them
        const int ch = cmp(tx, Str{kWild, 1}), cp = cmp(tx, Str{kWild + 1, 1});
        if (!wild) {
            kind[c++] = 2;
        } else if (ch < 0) {
            kind[c++] = 2; kind[c++] = 0; kind[c++] = 1;
        } else if (ch == 0) {            // the topic level is literally "#" (not a valid topic, but keep the order total)
            kind[c++] = 0; kind[c++] = 1;
        } else if (cp < 0) {
            kind[c++] = 0; kind[c++] = 2; kind[c++] = 1;
        } else if (cp == 0) {
            kind[c++] = 0; kind[c++] = 1;
        } else {
            kind[c++] = 0; kind[c++] = 1; kind[c++] = 2;
        }
    } else if (wild) {
        kind[c++] = 0;   // "#" matches the parent level
    }
    return c;
}

// A member of the expansion set as seek finds it, after the tenant level: the bound's levels 1..pre, then at most one level
// that leaves the bound (div: -1 = none, 0 = "#", which ends the member, 1 = "+", 2 = the topic level at dpos), then the minimal
// completion from topic position `tail`. The smallest child of a node is "#" unless the topic level sorts below it, or no
// wildcard exists (under the tenant level of a '$' topic); it is never "+". So the completion follows topic levels while that
// holds and then ends in "#", or it ends with the topic.
struct Member {
    int pre, div, dpos, tail;
};

// yields the levels of a member after the tenant level, one per call; false once there are no more
struct MemberLevels {
    Levels bound, topic;   // the bound at its level 1, the topic at the completion's first level
    int pre, div, dpos;
    bool sys;
    int i;                 // levels yielded so far
    bool done;
    __device__ bool next(Str* out) {
        if (done) return false;
        if (i < pre) {
            *out = bound.next();
        } else if (i == pre && div >= 0) {
            *out = div == 2 ? Str{topic.s + dpos, topic.pos - 1 - dpos} : wild(div);
            done = div == 0;
        } else if (!topic.more()) {   // the full-length filter
            done = true;
            return false;
        } else {
            const Str tx = topic.peek();
            if ((i == 0 && sys) || below_hash(tx)) {
                topic.skip(tx);
                *out = tx;
            } else {
                *out = wild(0);
                done = true;
            }
        }
        i++;
        return true;
    }
};

// least member >= the bound whose level 1 `b` is at (the tenant levels are equal); false: none. *exact: the member is the bound
__device__ bool seek(Levels t, Levels b, bool sys, Member* out, bool* exact) {
    int fb_depth = -1, fb_kind = 0;   // deepest level on the tight path with a child greater than the bound's level
    int fb_tpos = 0;                  // ... and the topic position of its level fb_depth + 1
    int i = 0;                        // matched levels so far (tight)
    *exact = false;
    while (true) {
        if (!b.more()) {              // the bound is exhausted: everything below this node is >= it
            *out = Member{i, -1, 0, t.pos};
            *exact = !t.more();       // the node itself is the full-length filter
            return true;
        }
        const Str bl = b.next();
        const bool has_t = t.more();
        const Str tx = has_t ? t.peek() : Str{t.s, 0};
        int kind[3];
        const int nc = children(!(i == 0 && sys), has_t, tx, kind);
        int eq = -1, gt = -1;
        for (int j = 0; j < nc; j++) {
            const int r = cmp(kind[j] == 2 ? tx : wild(kind[j]), bl);
            if (r == 0) eq = kind[j];
            else if (r > 0 && gt < 0) gt = kind[j];
        }
        if (gt >= 0) {
            fb_depth = i;
            fb_kind = gt;
            fb_tpos = t.pos;
        }
        if (eq == 0) {                // "#": terminal. Equal to the bound iff the bound ends here too, else it is a proper prefix (<)
            if (!b.more()) {
                *out = Member{i, 0, 0, 0};
                *exact = true;
                return true;
            }
            break;
        }
        if (eq > 0) {                 // "+" or the topic level: both consume the topic level
            t.skip(tx);
            i++;
            continue;
        }
        break;                        // no child equals the bound's level: leave the tight path
    }
    if (fb_depth < 0) return false;
    if (fb_kind == 0) {
        *out = Member{fb_depth, 0, 0, 0};
        return true;
    }
    t.pos = fb_tpos;                  // "+" and the topic level exist only while the topic has a level fb_depth + 1
    t.skip(t.peek());
    *out = Member{fb_depth, fb_kind, fb_tpos, t.pos};
    return true;
}

// 0 = the range cannot hold a match, 1 = candidate, 2 = seek past the end (the reference stops looking at later candidates)
__global__ void __launch_bounds__(128) range_lookup_kernel(int64_t n_pairs, const int64_t* pair_off, int64_t n_topics, const uint8_t* topics,
                                                           const int64_t* topic_off, const int32_t* topic_tenant, const uint8_t* tenants,
                                                           const int64_t* tenant_off, const int64_t* cand_off, const uint8_t* first_blob,
                                                           const int64_t* first_off, const uint8_t* last_blob, const int64_t* last_off,
                                                           uint8_t* out) {
    const int64_t j = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n_pairs) return;
    int64_t lo = 0, hi = n_topics;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (pair_off[mid] <= j) lo = mid;
        else hi = mid;
    }
    const int64_t ti = lo;
    const int tn = topic_tenant[ti];
    const int64_t cand = cand_off[tn] + (j - pair_off[ti]);
    const uint8_t* topic = topics + topic_off[ti];
    const int tlen = (int) (topic_off[ti + 1] - topic_off[ti]);
    const bool sys = tlen > 0 && topic[0] == '$';
    const Levels t{topic, tlen, 0, '/'};
    Levels f{first_blob + first_off[cand], (int) (first_off[cand + 1] - first_off[cand]), 0, 0};
    Levels l{last_blob + last_off[cand], (int) (last_off[cand + 1] - last_off[cand]), 0, 0};
    const Str tenant{tenants + tenant_off[tn], (int) (tenant_off[tn + 1] - tenant_off[tn])};
    // level 0 is the tenant id: every member starts with it
    const int r0 = cmp(tenant, f.next());
    if (r0 < 0) {
        out[j] = 2;   // the bound's tenant sorts behind this tenant: nothing >= first
        return;
    }
    Member m{0, -1, 0, 0};   // r0 > 0: every member is greater, so the smallest one
    bool exact = false;
    if (r0 == 0 && !seek(t, f, sys, &m, &exact)) {
        out[j] = 2;
        return;
    }
    // found == first, or found <= last (level-wise)
    int r = cmp(tenant, l.next());
    MemberLevels g{f, Levels{topic, tlen, m.tail, '/'}, m.pre, m.div, m.dpos, sys, 0, false};
    while (r == 0) {
        Str ml;
        const bool me = !g.next(&ml), le_ = !l.more();
        if (me || le_) {
            r = me && le_ ? 0 : (me ? -1 : 1);
            break;
        }
        r = cmp(ml, l.next());
    }
    out[j] = (exact || r <= 0) ? 1 : 0;
}

}  // namespace

extern "C" int32_t bfq_range_lookup(int32_t device_ordinal, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                                    const uint8_t* topics, const int64_t* topic_off, const int32_t* topic_tenant, int64_t n_topics,
                                    const int64_t* cand_off, const uint8_t* cand_flags, const uint8_t* first_blob, const int64_t* first_off,
                                    const uint8_t* last_blob, const int64_t* last_off, int64_t* keep_off_out, uint8_t* keep_out) {
    if (n_tenants < 0 || n_topics < 0 || !keep_off_out || (n_topics > 0 && (!topics || !topic_off || !topic_tenant || !keep_out)) ||
        (n_tenants > 0 && (!tenants || !tenant_off || !cand_off)))
        return fail(BFQ_E_INVALID, "bad argument");
    const int64_t n_cand = n_tenants ? cand_off[n_tenants] : 0;
    if (n_cand > 0 && (!cand_flags || !first_off || !last_off)) return fail(BFQ_E_INVALID, "NULL candidate arrays");
    // rows: topic i has one cell per candidate of its tenant
    keep_off_out[0] = 0;
    for (int64_t i = 0; i < n_topics; i++) {
        const int t = topic_tenant[i];
        if (t < 0 || t >= n_tenants) return fail(BFQ_E_RANGE, "topic_tenant out of range");
        keep_off_out[i + 1] = keep_off_out[i] + (cand_off[t + 1] - cand_off[t]);
    }
    const int64_t n_pairs = keep_off_out[n_topics];
    if (n_pairs == 0) return BFQ_OK;
    BFQ_CUDA_TRY(cudaSetDevice(device_ordinal));
    // every input is uploaded into a buffer of its own, of at least 16 bytes
    auto up = [](const void* src, size_t bytes, DeviceBuf<uint8_t>* dst) -> cudaError_t {
        cudaError_t e = dst->reserve(std::max<size_t>(bytes, 16));
        if (e != cudaSuccess) return e;
        return bytes ? cudaMemcpy(dst->p, src, bytes, cudaMemcpyHostToDevice) : cudaSuccess;
    };
    DeviceBuf<uint8_t> d_pair_off, d_topics, d_topic_off, d_tt, d_tenants, d_tenant_off, d_cand_off, d_first, d_first_off, d_last,
        d_last_off, d_out;
    BFQ_CUDA_TRY(up(keep_off_out, (size_t) (n_topics + 1) * 8, &d_pair_off));
    BFQ_CUDA_TRY(up(topics + topic_off[0], (size_t) (topic_off[n_topics] - topic_off[0]), &d_topics));
    std::vector<int64_t> toff((size_t) n_topics + 1);
    for (int64_t i = 0; i <= n_topics; i++) toff[(size_t) i] = topic_off[i] - topic_off[0];
    BFQ_CUDA_TRY(up(toff.data(), toff.size() * 8, &d_topic_off));
    BFQ_CUDA_TRY(up(topic_tenant, (size_t) n_topics * 4, &d_tt));
    BFQ_CUDA_TRY(up(tenants, (size_t) tenant_off[n_tenants], &d_tenants));
    BFQ_CUDA_TRY(up(tenant_off, (size_t) (n_tenants + 1) * 8, &d_tenant_off));
    BFQ_CUDA_TRY(up(cand_off, (size_t) (n_tenants + 1) * 8, &d_cand_off));
    BFQ_CUDA_TRY(up(first_blob, (size_t) first_off[n_cand], &d_first));
    BFQ_CUDA_TRY(up(first_off, (size_t) (n_cand + 1) * 8, &d_first_off));
    BFQ_CUDA_TRY(up(last_blob, (size_t) last_off[n_cand], &d_last));
    BFQ_CUDA_TRY(up(last_off, (size_t) (n_cand + 1) * 8, &d_last_off));
    BFQ_CUDA_TRY(d_out.reserve((size_t) n_pairs));
    range_lookup_kernel<<<(unsigned) ((n_pairs + 127) / 128), 128>>>(n_pairs, (const int64_t*) d_pair_off.p, n_topics, d_topics.p,
                                                                    (const int64_t*) d_topic_off.p, (const int32_t*) d_tt.p, d_tenants.p,
                                                                    (const int64_t*) d_tenant_off.p, (const int64_t*) d_cand_off.p,
                                                                    d_first.p, (const int64_t*) d_first_off.p, d_last.p,
                                                                    (const int64_t*) d_last_off.p, d_out.p);
    BFQ_CUDA_TRY(cudaGetLastError());
    BFQ_CUDA_TRY(cudaMemcpy(keep_out, d_out.p, (size_t) n_pairs, cudaMemcpyDeviceToHost));
    // the reference's candidate loop (TenantRangeLookupCache.java:78-104): a range without a Fact is kept, one whose Fact lacks
    // first or last is empty (skipped), and the first range whose seek runs past the end ends the scan
    for (int64_t i = 0; i < n_topics; i++) {
        const int t = topic_tenant[i];
        bool stopped = false;
        for (int64_t k = 0; k < cand_off[t + 1] - cand_off[t]; k++) {
            uint8_t& cell = keep_out[keep_off_out[i] + k];
            const uint8_t fl = cand_flags[cand_off[t] + k];
            if (stopped) {
                cell = 0;
            } else if (!(fl & 1)) {
                cell = 1;
            } else if ((fl & 6) != 6) {
                cell = 0;
            } else if (cell == 2) {
                cell = 0;
                stopped = true;
            }
        }
    }
    return BFQ_OK;
}
