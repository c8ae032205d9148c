// match_kernels.cu — forward match on sm_90a (H100): a batch of publish topics against the flattened filter tries.
//
// Replaces the hot loop of TenantRouteMatcher.matchAll
// (bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/cache/TenantRouteMatcher.java:96-156)
// with a level-synchronous frontier walk: ONE WARP PER TOPIC.
//   * the topic bytes are staged in shared memory, '/' boundaries found with a warp ballot (device-side
//     TopicUtil.parse, bifromq-util/.../TopicUtil.java:206-225 — empty levels are kept);
//   * the frontier (trie nodes whose path matches the consumed prefix) lives in shared memory, one node
//     per lane; every lane probes the 64-byte hash slot of its node's exact child with four LDG.128 and,
//     independently, loads the '+' child record — all loads of a level are in flight together;
//   * '#' children are inlined in their parent record, so "prefix/#" (incl. the parent-level match) is
//     emitted at discovery without another access; the '$' rule masks the root's '+' and '#' only;
//   * results are emitted as RANGES of route ranks (one per matched filter) compacted with ballot/popc
//     into a shared staging area and flushed with one atomicAdd per topic.
// Tier 2 (kBig): the rare topic whose frontier or range count outgrows the shared buffers is re-run by the
// same code with per-warp buffers in global memory sized from the index statistics — never truncated.
#include "match_kernels.cuh"
#include "hash_probe.cuh"

#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <mutex>
#include <cstdlib>

namespace bfq {

namespace {

constexpr int WARPS_PER_CTA = 8;
constexpr int STAGE_BYTES = 256;
constexpr uint32_t FR_CAP = 64;
constexpr uint32_t RG_CAP = 48;
constexpr uint32_t NONE31 = 0x7FFFFFFFu;
constexpr unsigned FULL = 0xFFFFFFFFu;

struct WarpSmem {
    uint8_t stage[STAGE_BYTES];
    uint32_t keyw[8];
    uint4 fr[2][FR_CAP];     // frontier entry: {child ref a, '+' child slot or NONE31, meta, -}
    uint2 rg[RG_CAP];
};

// one saturating byte per counter in the node record: 255 means "255 or more" -> force the exact caps kernel
__device__ __forceinline__ uint64_t caps_value(uint32_t c8) { return c8 == 0xFFu ? (1ull << 32) : (uint64_t) c8; }

template <bool kBig>
__device__ __forceinline__ void match_one(const MatchParams& p, WarpSmem& ws, uint32_t t, int lane, uint4* fr_a, uint4* fr_b,
                                          uint2* rg, uint32_t capF, uint32_t capR) {
    const int64_t tb = p.topic_off[t];
    const int len = (int) (p.topic_off[t + 1] - tb);
    const uint8_t* src = p.topics + tb;
    const bool staged = len <= STAGE_BYTES;
    __syncwarp();
    if (staged)
        for (int i = lane; i < len; i += 32) ws.stage[i] = src[i];
    __syncwarp();
    auto byte_at = [&](int i) -> uint32_t { return staged ? (uint32_t) ws.stage[i] : (uint32_t) src[i]; };

    int tenant = p.topic_tenant[t];
    const bool tenant_ok = tenant >= 0 && tenant < p.n_tenants;
    if (!tenant_ok) tenant = 0;
    const int root_ord = tenant_ok ? p.tenant_root[tenant] : -1;
    uint32_t n_rg = 0;
    uint32_t acc_r = 0;
    uint64_t acc_p = 0, acc_g = 0;
    bool overflow = false;

    // warp-compacted append of one optional range per lane
    auto emit = [&](bool valid, uint32_t first, uint32_t count, bool multi, uint32_t caps) {
        const unsigned m = __ballot_sync(FULL, valid);
        if (m == 0) return;
        if (valid) {
            const uint32_t idx = n_rg + __popc(m & ((1u << lane) - 1));
            if (idx < capR) rg[idx] = make_uint2(first, multi ? (count | RANGE_MULTI) : count);
            acc_r += count;
            acc_p += caps_value(caps & 0xFFu);
            acc_g += caps_value((caps >> 8) & 0xFFu);
        }
        n_rg += __popc(m);
        if (n_rg > capR) overflow = true;
    };

    if (root_ord >= 0) {
        uint32_t rw[16];
        load_payload(p.roots + root_ord, rw);
        const bool sys = len > 0 && byte_at(0) == '$';
        // "#" at level 0 matches every non-'$' topic
        emit(lane == 0 && !sys && rw[W_HASH_COUNT] > 0, rw[W_HASH_FIRST], rw[W_HASH_COUNT], rw[W_META] & FLAG_HASH_MULTI,
             (rw[W_CAPS] >> 16));
        uint4* fr_cur = fr_a;
        uint4* fr_next = fr_b;
        uint32_t n_fr = 0;
        {
            const uint32_t plus = (sys || rw[W_PLUS] == NONE) ? NONE31 : rw[W_PLUS];   // '+' at level 0 skips '$' topics
            const uint32_t has_exact = rw[W_META] & FLAG_HAS_EXACT;
            if (has_exact || plus != NONE31) {
                if (lane == 0) fr_cur[0] = make_uint4(child_ref(ROOT_BASE + (uint32_t) root_ord, rw), plus, rw[W_META], 0u);
                n_fr = 1;
            }
        }
        int pos = 0;
        while (n_fr > 0 && !overflow) {
            // ---- next token [pos, e)
            int e = len;
            for (int b = pos; b < len; b += 32) {
                const int i = b + lane;
                const unsigned m = __ballot_sync(FULL, i < len && byte_at(i) == '/');
                if (m) {
                    e = b + __ffs(m) - 1;
                    break;
                }
            }
            const bool last = e == len;
            const int tlen = e - pos;
            const int nchunks = tlen <= (int) TOKEN_BYTES ? 1 : (tlen + (int) TOKEN_BYTES - 1) / (int) TOKEN_BYTES;
            uint32_t n_next = 0;
            __syncwarp();
            for (uint32_t base = 0; base < n_fr && !overflow; base += 32) {
                const bool active = base + lane < n_fr;
                const uint4 fe = active ? fr_cur[base + lane] : make_uint4(0u, NONE31, 0u, 0u);
                const uint32_t plus = fe.y;
                // '+' child record: independent of the token, issue its load first
                const bool has_plus = active && plus != NONE31;
                uint32_t pw[16];
                if (has_plus) load_payload(p.slots + plus, pw);
                // exact child: one probe per 24-byte chunk of the token (one chunk unless the level is > 24 B)
                bool alive = active && (fe.z & FLAG_HAS_EXACT);
                uint32_t node = fe.x, node_meta = fe.z, cid = 0;
                uint32_t cw[16];
                for (int c = 0; c < nchunks; c++) {
                    const int cpos = pos + c * (int) TOKEN_BYTES;
                    const int cend = min(e, cpos + (int) TOKEN_BYTES);
                    const uint32_t lenw = c == nchunks - 1 ? (uint32_t) tlen : (LEN_CONT | (uint32_t) c);
                    __syncwarp();
                    if (lane < (int) TOKEN_WORDS) {
                        uint32_t v = 0;
#pragma unroll
                        for (int b = 0; b < 4; b++) {
                            const int idx = cpos + lane * 4 + b;
                            if (idx < cend) v |= byte_at(idx) << (8 * b);
                        }
                        ws.keyw[lane] = v;
                    }
                    __syncwarp();
                    uint32_t k[6];
#pragma unroll
                    for (int j = 0; j < 6; j++) k[j] = ws.keyw[j];
                    const uint64_t tokh = token_hash(lenw, k);
                    if (alive) {
                        alive = find_child(p.slots, p.tags, p.n_blocks, node, node_meta, lenw, k, tokh, cw, cid);
                        if (alive) {   // an intermediate chunk node: its own children continue the chain
                            node = child_ref(cid, cw);
                            node_meta = cw[W_META];
                        }
                    }
                }
                // ---- emit ranges of the discovered children and build the next frontier
                emit(alive && cw[W_HASH_COUNT] > 0, cw[W_HASH_FIRST], cw[W_HASH_COUNT], alive && (cw[W_META] & FLAG_HASH_MULTI),
                     (cw[W_CAPS] >> 16));
                emit(has_plus && pw[W_HASH_COUNT] > 0, pw[W_HASH_FIRST], pw[W_HASH_COUNT],
                     has_plus && (pw[W_META] & FLAG_HASH_MULTI), (pw[W_CAPS] >> 16));
                if (last) {
                    emit(alive && cw[W_OWN_COUNT] > 0, cw[W_OWN_FIRST], cw[W_OWN_COUNT], alive && (cw[W_META] & FLAG_OWN_MULTI),
                         (cw[W_CAPS] & 0xFFFFu));
                    emit(has_plus && pw[W_OWN_COUNT] > 0, pw[W_OWN_FIRST], pw[W_OWN_COUNT],
                         has_plus && (pw[W_META] & FLAG_OWN_MULTI), (pw[W_CAPS] & 0xFFFFu));
                } else {
                    const bool push_c = alive && ((cw[W_META] & FLAG_HAS_EXACT) || cw[W_PLUS] != NONE);
                    const bool push_p = has_plus && ((pw[W_META] & FLAG_HAS_EXACT) || pw[W_PLUS] != NONE);
                    const unsigned mc = __ballot_sync(FULL, push_c);
                    const unsigned mp = __ballot_sync(FULL, push_p);
                    const uint32_t lt = (1u << lane) - 1;
                    if (push_c) {
                        const uint32_t idx = n_next + __popc(mc & lt);
                        if (idx < capF) fr_next[idx] = make_uint4(child_ref(cid, cw), cw[W_PLUS] == NONE ? NONE31 : cw[W_PLUS], cw[W_META], 0u);
                    }
                    n_next += __popc(mc);
                    if (push_p) {
                        const uint32_t idx = n_next + __popc(mp & lt);
                        if (idx < capF) fr_next[idx] = make_uint4(child_ref(plus, pw), pw[W_PLUS] == NONE ? NONE31 : pw[W_PLUS], pw[W_META], 0u);
                    }
                    n_next += __popc(mp);
                    if (n_next > capF) overflow = true;
                }
            }
            __syncwarp();
            uint4* tmp = fr_cur;
            fr_cur = fr_next;
            fr_next = tmp;
            n_fr = n_next;
            pos = e + 1;
            if (last) break;
        }
    }

    // ---- warp totals
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        acc_r += __shfl_xor_sync(FULL, acc_r, o);
        acc_p += __shfl_xor_sync(FULL, acc_p, o);
        acc_g += __shfl_xor_sync(FULL, acc_g, o);
    }
    if (overflow) {
        if (lane == 0) {
            if (!kBig) {
                const unsigned long long idx = atomicAdd(&p.counters[CTR_OVERFLOW], 1ull);
                p.overflow_list[idx] = t;
                p.span_begin[t] = 0;
                p.span_count[t] = SPAN_OVERFLOW;
                p.route_count[t] = 0;
            } else {
                atomicAdd(&p.counters[CTR_ERROR], 1ull);
                p.span_begin[t] = 0;
                p.span_count[t] = 0;
                p.route_count[t] = 0;
            }
        }
        return;
    }
    const int maxP = p.max_pfanout[tenant], maxG = p.max_gfanout[tenant];
    // ranks are < 2^31-1, so a cap of INT_MAX can never be exceeded
    const bool flag_p = maxP != 0x7FFFFFFF && acc_p > (uint64_t) (maxP < 0 ? 0 : maxP);
    const bool flag_g = maxG != 0x7FFFFFFF && acc_g > (uint64_t) (maxG < 0 ? 0 : maxG);
    const bool flagged = flag_p || flag_g;
    unsigned long long base = 0;
    if (n_rg > 0) {
        if (lane == 0) base = atomicAdd(&p.counters[CTR_RANGES], (unsigned long long) n_rg);
        base = __shfl_sync(FULL, base, 0);
        base += p.dyn_base;
        if (base + n_rg <= p.ranges_cap)
            for (uint32_t i = lane; i < n_rg; i += 32) p.ranges[base + i] = rg[i];
    }
    if (lane == 0) {
        p.span_begin[t] = (uint32_t) base;
        p.span_count[t] = n_rg | (flagged ? SPAN_FLAGGED : 0u);
        p.route_count[t] = acc_r;
        if (flagged) {
            const unsigned long long idx = atomicAdd(&p.counters[CTR_FLAGGED], 1ull);
            p.flagged_list[idx] = t;
        }
    }
}

template <bool kBig>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32) match_topics_kernel(const MatchParams p) {
    __shared__ WarpSmem sm[WARPS_PER_CTA];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    WarpSmem& ws = sm[wid];
    const int64_t gw = (int64_t) blockIdx.x * WARPS_PER_CTA + wid;
    const int64_t nw = (int64_t) gridDim.x * WARPS_PER_CTA;
    if (kBig) {
        // per-warp scratch, in uint2 units: two frontier buffers of uint4 entries, then the range staging
        uint2* basep = p.scratch + (uint64_t) gw * (4 * p.scratch_frontier_cap + p.scratch_ranges_cap);
        uint4* fr_a = reinterpret_cast<uint4*>(basep);
        uint4* fr_b = reinterpret_cast<uint4*>(basep + 2 * p.scratch_frontier_cap);
        uint2* rg = basep + 4 * p.scratch_frontier_cap;
        const uint32_t capF = (uint32_t) min((uint64_t) 0x3FFFFFFFull, p.scratch_frontier_cap);
        const uint32_t capR = (uint32_t) min((uint64_t) SPAN_COUNT_MASK, p.scratch_ranges_cap);
        for (int64_t it = gw; it < p.n_work; it += nw) match_one<true>(p, ws, p.work_list[it], lane, fr_a, fr_b, rg, capF, capR);
    } else if (p.work_list) {
        // tier 1 behind tier 0: the number of deferred topics is read from the device counter (no host round trip)
        const int64_t n_work = p.n_work >= 0 ? p.n_work : (int64_t) p.counters[CTR_DEFER];
        for (int64_t it = gw; it < n_work; it += nw)
            match_one<false>(p, ws, p.work_list[it], lane, ws.fr[0], ws.fr[1], ws.rg, FR_CAP, RG_CAP);
    } else {
        for (int64_t it = gw; it < p.n_topics; it += nw)
            match_one<false>(p, ws, (uint32_t) it, lane, ws.fr[0], ws.fr[1], ws.rg, FR_CAP, RG_CAP);
    }
}


// ------------------------------------------------------------------------------------------------ tier 0
// ONE LANE PER TOPIC, persistent lanes. The warp-per-topic walk above leaves most lanes idle when the frontier
// is a handful of nodes (the common case: ~4 per level on BASELINE config C4). Here every lane walks its own topic
// depth-first:
//   * a node has at most two continuations per level (exact child, '+' child), so the DFS parks at most ONE
//     pending '+' branch per level: a (L_MAXLV+1)-entry per-lane array plus a bitmask, never a growing frontier;
//   * per step a lane reads the 28 bytes at its current level start (up to three aligned 16-byte granules, word select +
//     funnel shift), finds the '/' with a SWAR zero-byte test — the level table is filled lazily, there is no tokenising
//     pre-pass —, issues the exact-child slot read (4 x LDG.128) and the '+' child payload read (2 x LDG.128) together and
//     writes the discovered ranges to the INLINE_RANGES inline slots of the topic's position in the work order, one whole
//     32-byte sector at a time from registers: no shared-memory staging, no output atomics;
//   * a lane that finishes takes the next topic at once (warp-uniform refill from 32-topic chunks claimed with
//     one atomicAdd per chunk), so a straggler never idles the other 31 lanes (a warp that waits for its whole batch of 32
//     runs with a third of its lanes active);
//   * chunks are runs of p.order — the batch sorted by (tenant, leading-level hashes), see launch_order — so the lanes of
//     a warp walk the same part of the trie, take the same branches and finish together.
// Anything that does not fit the bounded state (> L_MAXLV levels, a level > 24 B, > INLINE_RANGES ranges, topic > 64 KB)
// is handed, whole, to the warp-per-topic tier through defer_list.
constexpr int L_WARPS = 4;
constexpr int64_t LARGE_BATCH_TOPICS = 1 << 17;   // tier 0: batches of at least this many topics run with ...
constexpr int LARGE_BATCH_CTAS_PER_SM = 4;        // ... at most this many resident CTAs per SM (see launch_match_lanes)
constexpr int L_MAXLV = 12;
constexpr int L_CHUNK = 32;
constexpr int TENANT_CAPPED = 1 << 30;   // flag in the lane's tenant word: the tenant has a finite fan-out cap

struct LaneSmem {
    uint16_t lv[L_MAXLV + 1][32];   // start offset of each level of the lane's topic (lane-minor: conflict free)
    uint2 stk[L_MAXLV + 1][32];     // parked '+' branch per level: {child ref a, '+' child slot or NONE31}
    uint32_t stkm[L_MAXLV + 1][32]; //   ... and its meta word
    // metadata of the warp's current chunk of topics, loaded cooperatively (coalesced) when the chunk is claimed
    int64_t m_off[L_CHUNK];         // byte offset of the topic in the blob
    uint32_t m_t[L_CHUNK];          // topic index (the chunk is a run of positions of p.order, or of topic indices)
    uint32_t m_len[L_CHUNK];
    int32_t m_tenant[L_CHUNK];
    int32_t m_root[L_CHUNK];        // root ordinal of the topic's tenant, or -1
    // payload of the tenant root of the chunk's first topic: in locality order a chunk is almost always one tenant, and the
    // root read at every refill would be a dependent L2 access in the middle of a lock-step step
    uint32_t c_root[8];
    int32_t c_ord;
};

// 7 resident CTAs per SM (what the shared memory allows, and what a batch below LARGE_BATCH_TOPICS runs with) need <= 72
// registers per thread; left to itself the compiler takes 76-80 since the sector buffer below
constexpr int L_MIN_CTAS_PER_SM = 7;

template <bool kRootStep, bool kPrefetch, bool kNA>
__global__ void __launch_bounds__(L_WARPS * 32, L_MIN_CTAS_PER_SM) match_topics_lane_kernel(const MatchParams p) {
    __shared__ LaneSmem sm[L_WARPS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    LaneSmem& ws = sm[wid];
    const uint32_t lt_mask = (1u << lane) - 1;
    // in locality order only the batch's distinct topics are matched; their number was counted on the device
    const int64_t n = (p.order && p.order_count) ? (int64_t) *p.order_count : p.n_topics;

    // warp-uniform work cursor over the current chunk [cstart, end)
    int64_t next = 0, end = 0, cstart = 0;
    bool exhausted = false;
    // per-lane topic state; level < 0: the tenant root has not been expanded yet (`node` holds the root ordinal)
    bool have = false, bad = false;
    uint32_t t = 0, node = 0 /* child ref a (root ordinal while level < 0) */, plusf = NONE31, meta = 0, pending = 0, n_rg = 0, acc_r = 0;
    uint32_t pos = 0;   // the topic's position in the work order (= t without an order)
    // matched persistent / group routes so far; bit 31 = "a node's saturated count byte was seen" (then the true sum is
    // unknown but large: the topic is flagged unless the cap is INT_MAX). <= INLINE_RANGES * 254 otherwise.
    uint32_t acc_p = 0, acc_g = 0;
    // The ranges are written a whole 32-byte sector (4 ranges) at a time: rg_out is the first slot of the topic's current sector,
    // s0..s2 hold its first n_rg % 4 ranges. A sector written piecemeal over a walk is partial whenever L2 evicts it in between
    // (C4: range stores cost tier 0 71 us that way, issuing them ~0; see DESIGN §4). The inline runs (RANGE_SECTOR-aligned: INLINE_RANGES per
    // position) and the spill blocks (RANGE_SECTOR-aligned offsets, see capi.cu) start on sector boundaries.
    uint2* rg_out = nullptr;
    uint2 s0 = make_uint2(0u, 0u), s1 = s0, s2 = s0;
    int64_t my_off = 0;
    int len = 0, level = 0, tenant = 0;

    auto emit = [&](uint32_t first, uint32_t count, bool multi, uint32_t caps) {
        if (n_rg >= INLINE_RANGES) {
            // the topic's inline slots are full: move it to a SPILL_RANGES block of the cursor-allocated region once (topics with
            // many matched filters — '+'-heavy filter sets — stay in this kernel instead of queueing for the warp-per-topic tier)
            if (n_rg == INLINE_RANGES) {
                const unsigned long long at = p.dyn_base + atomicAdd(&p.counters[CTR_RANGES], (unsigned long long) SPILL_RANGES);
                if (at + SPILL_RANGES <= p.ranges_cap) {
                    // INLINE_RANGES is a whole number of sectors: all of them are written, none is pending
                    uint4* dst = reinterpret_cast<uint4*>(p.ranges + at);
                    const uint4* src = reinterpret_cast<const uint4*>(rg_out - INLINE_RANGES);
#pragma unroll
                    for (int j = 0; j < (int) INLINE_RANGES / 2; j++) dst[j] = src[j];
                    rg_out = p.ranges + at + INLINE_RANGES;
                } else {
                    bad = true;   // no room: the host grows the region and re-runs the batch
                }
            } else if (n_rg >= SPILL_RANGES) {
                bad = true;
            }
        }
        if (!bad) {
            const uint2 r = make_uint2(first, multi ? (count | RANGE_MULTI) : count);
            switch (n_rg & (RANGE_SECTOR - 1)) {
            case 0: s0 = r; break;
            case 1: s1 = r; break;
            case 2: s2 = r; break;
            default: {
                uint4* o = reinterpret_cast<uint4*>(rg_out);
                o[0] = make_uint4(s0.x, s0.y, s1.x, s1.y);
                o[1] = make_uint4(s2.x, s2.y, r.x, r.y);
                rg_out += RANGE_SECTOR;
            }
            }
        }
        n_rg++;
        acc_r += count;
        const uint32_t cp = caps & 0xFFu, cg = (caps >> 8) & 0xFFu;
        acc_p = (acc_p + cp) | (cp == 0xFFu ? 0x80000000u : 0u);   // <= SPILL_RANGES additions of <= 255: no carry into bit 31
        acc_g = (acc_g + cg) | (cg == 0xFFu ? 0x80000000u : 0u);
    };
    // the topic's span: one record at its position in an ordered batch (finalize_kernel gathers it), else the topic-indexed arrays
    auto put_span = [&](uint32_t begin, uint32_t count, uint32_t routes, uint32_t deferred) {
        if (p.order) {
            p.pos_rec[pos] = SpanRecord{begin, count, routes, deferred};
        } else {
            p.span_begin[t] = begin;
            p.span_count[t] = count;
            p.route_count[t] = routes;
        }
    };
    auto finish = [&]() {
        if (bad) {
            const unsigned long long idx = atomicAdd(&p.counters[CTR_DEFER], 1ull);
            p.defer_list[idx] = t;
            put_span(0u, SPAN_OVERFLOW, 0u, 1u);   // tier 1 writes the topic-indexed span
        } else {
            // the caps are only read for a topic that matched capped-kind routes in a tenant with a finite cap (bit 30 of
            // `tenant`, set when the chunk was claimed): the loads would otherwise stall the whole warp at every finish
            bool flagged = false;
            if ((tenant & TENANT_CAPPED) && (acc_p | acc_g)) {
                const int tn = tenant & ~TENANT_CAPPED;
                const int maxP = p.max_pfanout[tn], maxG = p.max_gfanout[tn];
                const bool flag_p = maxP != 0x7FFFFFFF && acc_p > (uint32_t) (maxP < 0 ? 0 : maxP);
                const bool flag_g = maxG != 0x7FFFFFFF && acc_g > (uint32_t) (maxG < 0 ? 0 : maxG);
                flagged = flag_p || flag_g;
            }
            if (n_rg & (RANGE_SECTOR - 1)) {
                // the last, partial sector, written whole: the slots past n_rg hold stale ranges no reader looks at
                uint4* o = reinterpret_cast<uint4*>(rg_out);
                o[0] = make_uint4(s0.x, s0.y, s1.x, s1.y);
                o[1] = make_uint4(s2.x, s2.y, s2.x, s2.y);
            }
            put_span((uint32_t) ((rg_out - (n_rg & ~(RANGE_SECTOR - 1))) - p.ranges),   // the inline slots, or the spill block
                     n_rg | (flagged ? SPAN_FLAGGED : 0u), acc_r, 0u);
            if (flagged) {
                const unsigned long long idx = atomicAdd(&p.counters[CTR_FLAGGED], 1ull);
                p.flagged_list[idx] = t;
            }
        }
        have = false;
    };

    while (true) {
        // ---- refill idle lanes with the next unclaimed topics
        const unsigned idle = __ballot_sync(FULL, !have);
        if (idle) {
            if (next >= end && !exhausted) {
                unsigned long long c = 0;
                if (lane == 0) c = atomicAdd(&p.counters[CTR_CHUNK], (unsigned long long) L_CHUNK);
                c = __shfl_sync(FULL, c, 0);
                if ((int64_t) c >= n) {
                    exhausted = true;
                } else {
                    cstart = next = (int64_t) c;
                    end = min(n, next + L_CHUNK);
                    __syncwarp();
                    for (int i = lane; i < (int) (end - cstart); i += 32) {
                        const uint32_t ti = p.order ? p.order[cstart + i] : (uint32_t) (cstart + i);
                        const int64_t o = p.topic_off[ti], o2 = p.topic_off[ti + 1];
                        int tn = p.topic_tenant[ti];
                        const bool tn_ok = tn >= 0 && tn < p.n_tenants;
                        if (!tn_ok) tn = 0;
                        if (kPrefetch) {
                            // pull the topic's bytes towards L2 now: the first key read of each topic would otherwise be a
                            // compulsory HBM miss in the middle of a lock-step warp step
                            // (the '$' test below reads the first line; a topic's first 28 bytes may straddle into a second)
                            if (((o + 28) >> 7) != (o >> 7)) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.topics + o + 28));
                        }
                        // bit 31 of m_len: the topic starts with '$' (first-level wildcards skip it) — read here, with the rest
                        // of the chunk's metadata, instead of as a dependent load in the middle of a refill
                        const bool sys = o2 > o && p.topics[o] == '$';
                        const bool capped = p.max_pfanout[tn] != 0x7FFFFFFF || p.max_gfanout[tn] != 0x7FFFFFFF;
                        ws.m_t[i] = ti;
                        ws.m_off[i] = o;
                        ws.m_len[i] = (uint32_t) min((int64_t) 0x7FFFFFFF, o2 - o) | (sys ? 0x80000000u : 0u);
                        ws.m_tenant[i] = tn | (capped ? TENANT_CAPPED : 0);
                        const int ro = tn_ok ? p.tenant_root[tn] : -1;
                        ws.m_root[i] = ro;
                        if (i == 0) {
                            ws.c_ord = ro;
                            if (ro >= 0) {
                                uint32_t rw[16];
                                load_payload(p.roots + ro, rw);
#pragma unroll
                                for (int j = 0; j < 8; j++) ws.c_root[j] = rw[8 + j];
                            }
                        }
                    }
                    __syncwarp();
                }
            }
            if (next < end) {
                const int64_t idx = next + __popc(idle & lt_mask);
                const bool take = !have && idx < end;
                next = min(end, next + (int64_t) __popc(idle));
                if (take) {
                    const int i = (int) (idx - cstart);
                    t = ws.m_t[i];
                    my_off = ws.m_off[i];
                    const uint32_t lenw = ws.m_len[i];
                    len = (int) (lenw & 0x7FFFFFFFu);
                    tenant = ws.m_tenant[i];
                    const int root_ord = ws.m_root[i];
                    n_rg = 0; acc_r = 0; acc_p = 0; acc_g = 0; pending = 0;
                    // the inline slots of the topic's POSITION in the work order (idx), not of its topic index t: a warp's topics come
                    // from the chunks it claimed, so its range writes stay in a few KB of the array instead of scattering over all
                    // of it (in locality order t is effectively random over an array larger than L2)
                    rg_out = p.ranges + (uint64_t) idx * INLINE_RANGES;
                    pos = (uint32_t) idx;
                    bad = len > 65535;
                    have = true;
                    ws.lv[0][lane] = 0;
                    level = -1;
                    node = (uint32_t) root_ord;
                    plusf = NONE31;
                    if (root_ord < 0 || bad) {
                        finish();   // tenant without routes: an empty result; oversized: tier 1
                    } else if (!kRootStep) {
                        // expand the tenant root right here instead of spending a lock-step DFS step on it
                        uint32_t rw[16];
                        if (root_ord == ws.c_ord) {
#pragma unroll
                            for (int j = 0; j < 8; j++) rw[8 + j] = ws.c_root[j];
                        } else {
                            load_payload(p.roots + root_ord, rw);
                        }
                        const bool sys = lenw >> 31;
                        if (!sys && rw[W_HASH_COUNT] > 0) emit(rw[W_HASH_FIRST], rw[W_HASH_COUNT], rw[W_META] & FLAG_HASH_MULTI, (rw[W_CAPS] >> 16));
                        const uint32_t rplus = (sys || rw[W_PLUS] == NONE) ? NONE31 : rw[W_PLUS];
                        const uint32_t has_exact = rw[W_META] & FLAG_HAS_EXACT;
                        if ((has_exact || rplus != NONE31) && !bad) {
                            node = child_ref(ROOT_BASE + (uint32_t) root_ord, rw);
                            plusf = rplus;
                            meta = rw[W_META];
                            level = 0;
                        } else {
                            finish();
                        }
                    }
                }
            } else if (idle == FULL) {
                break;   // nothing left to claim and every lane is done
            }
        }
        if (have) {
            // ---- one DFS step. level < 0: expand the tenant root (its record is loaded where a '+' child would be)
            const bool rootstep = kRootStep && level < 0;
            const int lvl = rootstep ? 0 : level;
            const int s = ws.lv[lvl][lane];
            const int rem = len - s;
            // 28 bytes at the level start from up to three ALIGNED 16-byte granules (each one holds at least one byte of the
            // topic, so the reads never leave the granules the blob occupies), then a word-select + funnel shift. Eight
            // 4-byte loads here were 25 % of the kernel's L1 tag lookups.
            const uint64_t a = (uint64_t) (uintptr_t) p.topics + (uint64_t) my_off + (uint64_t) s;
            const uint4* qp = reinterpret_cast<const uint4*>(a & ~15ull);
            const int o = (int) (a & 15);
            const int need = o + min(rem, 28);
            uint4 q0 = make_uint4(0u, 0u, 0u, 0u), q1 = q0, q2 = q0;
            if (need > 0) q0 = __ldg(qp);
            if (need > 16) q1 = __ldg(qp + 1);
            if (need > 32) q2 = __ldg(qp + 2);
            // the '+' child (or the tenant root) record: independent of the token, issue its load right away
            const uint32_t plus = plusf;
            const bool has_plus = rootstep || plus != NONE31;
            uint32_t pw[16];
            if (has_plus) {
                if (rootstep) load_payload<false>(p.roots + node, pw);
                else load_payload<kNA>(p.slots + plus, pw);
            }
            uint32_t k[7];
            {
                const uint32_t X[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
                const bool by2 = o & 8, by1 = o & 4;
                uint32_t Y[10], Z[8];
#pragma unroll
                for (int j = 0; j < 10; j++) Y[j] = by2 ? X[j + 2] : X[j];
#pragma unroll
                for (int j = 0; j < 8; j++) Z[j] = by1 ? Y[j + 1] : Y[j];
                const int sh = (o & 3) * 8;
#pragma unroll
                for (int j = 0; j < 7; j++) k[j] = __funnelshift_r(Z[j], Z[j + 1], sh);
            }
            const uint32_t first_byte = k[0] & 0xFFu;
            // first '/' within the 28 bytes (SWAR zero-byte test on w ^ "////")
            int q = 28;
#pragma unroll
            for (int j = 6; j >= 0; j--) {
                const uint32_t y = k[j] ^ 0x2F2F2F2Fu;
                const uint32_t hz = (y - 0x01010101u) & ~y & 0x80808080u;
                if (hz) q = 4 * j + ((__ffs(hz) - 1) >> 3);
            }
            const int tlen = min(q, rem);
            const bool last = tlen == rem;
            if (rootstep) {
                const bool sys = len > 0 && first_byte == '$';   // '+' and '#' at the first level skip '$' topics
                if (!sys && pw[W_HASH_COUNT] > 0) emit(pw[W_HASH_FIRST], pw[W_HASH_COUNT], pw[W_META] & FLAG_HASH_MULTI, (pw[W_CAPS] >> 16));
                const uint32_t rplus = (sys || pw[W_PLUS] == NONE) ? NONE31 : pw[W_PLUS];
                const uint32_t has_exact = pw[W_META] & FLAG_HAS_EXACT;
                if ((has_exact || rplus != NONE31) && !bad) {
                    node = child_ref(ROOT_BASE + node, pw);
                    plusf = rplus;
                    meta = pw[W_META];
                    level = 0;
                } else {
                    finish();
                }
            } else if (tlen > (int) TOKEN_BYTES || (!last && level >= L_MAXLV - 1)) {
                bad = true;   // a level longer than the inline key, or deeper than the level table: tier 1 takes it
                finish();
            } else {
                if (!last) ws.lv[level + 1][lane] = (uint16_t) (s + tlen + 1);
                const int tbits = 8 * tlen;
#pragma unroll
                for (int j = 0; j < 6; j++)   // clear the bytes at and after the token end: 0xFFFFFFFF >> clamp(32(j+1) - 8 tlen, 0, 32)
                    k[j] &= __funnelshift_rc(0xFFFFFFFFu, 0u, (uint32_t) max(32 * (j + 1) - tbits, 0));
                uint32_t cw[16], cid = 0;
                const uint32_t kk[6] = {k[0], k[1], k[2], k[3], k[4], k[5]};
                const bool alive = find_child_lanes<kNA>(p.slots, p.tags, p.n_blocks, meta & FLAG_HAS_EXACT, node, meta, (uint32_t) tlen, kk,
                                                         token_hash((uint32_t) tlen, kk), cw, cid);
                bool push_c = false, push_p = false;
                if (alive) {
                    if (cw[W_HASH_COUNT] > 0) emit(cw[W_HASH_FIRST], cw[W_HASH_COUNT], cw[W_META] & FLAG_HASH_MULTI, (cw[W_CAPS] >> 16));
                    if (last) {
                        if (cw[W_OWN_COUNT] > 0) emit(cw[W_OWN_FIRST], cw[W_OWN_COUNT], cw[W_META] & FLAG_OWN_MULTI, (cw[W_CAPS] & 0xFFFFu));
                    } else {
                        push_c = (cw[W_META] & FLAG_HAS_EXACT) || cw[W_PLUS] != NONE;
                    }
                }
                if (has_plus) {
                    if (pw[W_HASH_COUNT] > 0) emit(pw[W_HASH_FIRST], pw[W_HASH_COUNT], pw[W_META] & FLAG_HASH_MULTI, (pw[W_CAPS] >> 16));
                    if (last) {
                        if (pw[W_OWN_COUNT] > 0) emit(pw[W_OWN_FIRST], pw[W_OWN_COUNT], pw[W_META] & FLAG_OWN_MULTI, (pw[W_CAPS] & 0xFFFFu));
                    } else {
                        push_p = (pw[W_META] & FLAG_HAS_EXACT) || pw[W_PLUS] != NONE;
                    }
                }
                if (bad) {
                    finish();
                } else if (push_c) {
                    if (push_p) {   // park the '+' branch of this level, continue down the exact branch
                        ws.stk[level + 1][lane] = make_uint2(child_ref(plus, pw), pw[W_PLUS] == NONE ? NONE31 : pw[W_PLUS]);
                        ws.stkm[level + 1][lane] = pw[W_META];
                        pending |= 1u << (level + 1);
                    }
                    node = child_ref(cid, cw);
                    plusf = cw[W_PLUS] == NONE ? NONE31 : cw[W_PLUS];
                    meta = cw[W_META];
                    level++;
                } else if (push_p) {
                    node = child_ref(plus, pw);
                    plusf = pw[W_PLUS] == NONE ? NONE31 : pw[W_PLUS];
                    meta = pw[W_META];
                    level++;
                } else if (pending) {
                    const int l = 31 - __clz(pending);
                    pending &= ~(1u << l);
                    const uint2 it = ws.stk[l][lane];
                    node = it.x;
                    plusf = it.y;
                    meta = ws.stkm[l][lane];
                    level = l;
                } else {
                    finish();
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ locality order
// Reads a topic 16 bytes at a time as four topic-aligned 32-bit words (word i of block j = topic bytes 16j + 4i .. + 3), whatever
// the topic's alignment in the blob: one aligned 16-byte granule load per block, word select + funnel shift in registers. Bytes
// at and after len read as 0. Only granules that hold at least one byte of the topic are read, so the reads stay inside the
// 16-byte granules the blob occupies. (A word-at-a-time reader spends most of the prep kernel's instructions in its tail loop.)
struct TopicQuads {
    const uint4* qp;
    int off, len, j;
    uint4 cur;
    __device__ __forceinline__ TopicQuads(const uint8_t* topics, int64_t o, int len_) {
        const uint64_t a = (uint64_t) (uintptr_t) topics + (uint64_t) o;
        qp = reinterpret_cast<const uint4*>(a & ~15ull);
        off = (int) (a & 15);
        len = len_;
        j = 0;
        cur = len > 0 ? __ldg(qp) : make_uint4(0u, 0u, 0u, 0u);
    }
    __device__ __forceinline__ void next(uint32_t (&w)[4]) {
        // granule j+1 starts at topic byte 16(j+1) - off
        const uint4 nx = (16 * (j + 1) - off < len) ? __ldg(qp + j + 1) : make_uint4(0u, 0u, 0u, 0u);
        const uint32_t X[8] = {cur.x, cur.y, cur.z, cur.w, nx.x, nx.y, nx.z, nx.w};
        const bool by2 = off & 8, by1 = off & 4;
        const int sh = (off & 3) * 8;
        uint32_t Y[6], Z[5];
#pragma unroll
        for (int i = 0; i < 6; i++) Y[i] = by2 ? X[i + 2] : X[i];
#pragma unroll
        for (int i = 0; i < 5; i++) Z[i] = by1 ? Y[i + 1] : Y[i];
#pragma unroll
        for (int i = 0; i < 4; i++) w[i] = __funnelshift_r(Z[i], Z[i + 1], sh);
        const int rem = len - 16 * j;
        if (rem < 16) {
#pragma unroll
            for (int i = 0; i < 4; i++)   // 0xFFFFFFFF >> clamp(32(i+1) - 8 rem, 0, 32)
                w[i] &= __funnelshift_rc(0xFFFFFFFFu, 0u, (uint32_t) max(32 * (i + 1) - 8 * max(rem, 0), 0));
        }
        cur = nx;
        j++;
    }
};

// What the ordering kernels read: the caller's OrderParams with its scratch carved up by launch_order.
struct OrderKernelParams {
    int64_t n_topics;
    const uint8_t* topics;
    const int64_t* topic_off;
    const int32_t* topic_tenant;
    int32_t n_tenants;
    uint32_t* keys;
    uint32_t* leader;
    uint32_t* order;
    unsigned long long* hash_tab;
    uint32_t hash_mask;
    uint32_t* hist;                 // [n_buckets] zeroed; n_buckets = 2^hist_bits, a multiple of 4096
    uint32_t* blk_tot;              // [n_buckets / 4096]
    uint32_t* blk_pfx;              // [n_buckets / 4096]
    uint32_t* ticket;               // zeroed
    int hist_bits;
    int dedup;
    uint64_t dedup_hash_mask;
    unsigned long long* counters;
};

constexpr int ORDER_WINDOW_QUADS = 3;
constexpr int ORDER_WINDOW_WORDS = 4 * ORDER_WINDOW_QUADS;   // the order key looks at the first 48 bytes: three levels of ordinary topics end well before

// The (tenant, topic) pairs of topics a and b are equal: same tenant (every out-of-range index counts as one tenant), same
// length, same bytes.
__device__ __forceinline__ bool same_pair(const OrderKernelParams& q, uint32_t a, uint32_t b) {
    int ta = q.topic_tenant[a], tb = q.topic_tenant[b];
    if (ta < 0 || ta >= q.n_tenants) ta = -1;
    if (tb < 0 || tb >= q.n_tenants) tb = -1;
    const int64_t oa = q.topic_off[a], ob = q.topic_off[b];
    const int64_t len = max((int64_t) 0, q.topic_off[a + 1] - oa);
    if (ta != tb || max((int64_t) 0, q.topic_off[b + 1] - ob) != len || len > 0x3FFFFFFF) return false;
    TopicQuads wa(q.topics, oa, (int) len), wb(q.topics, ob, (int) len);
    for (int j = 0; 16 * j < len; j++) {
        uint32_t x[4], y[4];
        wa.next(x);
        wb.next(y);
        if ((x[0] ^ y[0]) | (x[1] ^ y[1]) | (x[2] ^ y[2]) | (x[3] ^ y[3])) return false;
    }
    return true;
}

// One pass over topic i: its first ORDER_WINDOW_WORDS words go to k (the order key's window, zero past the end), and the
// 64-bit de-dup hash of (tenant, length, bytes) is returned (two independent 32-bit multiply-xor lanes, one IMAD each per word,
// folded by fmix64 and cut to q.dedup_hash_mask). Without de-dup only the window is read.
__device__ __forceinline__ uint64_t read_topic(const OrderKernelParams& q, int64_t i, int& hlen, int& tn, uint32_t (&k)[ORDER_WINDOW_WORDS]) {
    const int64_t o = q.topic_off[i];
    hlen = (int) min(max((int64_t) 0, q.topic_off[i + 1] - o), (int64_t) 0x3FFFFFFF);
    tn = q.topic_tenant[i];
    if (tn < 0 || tn >= q.n_tenants) tn = -1;   // all out-of-range tenant indices match nothing: one group
    uint32_t h1 = (uint32_t) hlen * 0x9E3779B1u + (uint32_t) tn, h2 = (uint32_t) tn * 0x85EBCA77u ^ (uint32_t) hlen;
    TopicQuads tq(q.topics, o, hlen);
#pragma unroll
    for (int j = 0; j < ORDER_WINDOW_QUADS; j++) {
        uint32_t w[4] = {0u, 0u, 0u, 0u};
        if (16 * j < hlen) tq.next(w);
#pragma unroll
        for (int x = 0; x < 4; x++) {
            k[4 * j + x] = w[x];
            h1 = (h1 ^ w[x]) * 0xCC9E2D51u;
            h2 = (h2 + w[x]) * 0x1B873593u ^ (h2 >> 15);
        }
    }
    if (!q.dedup) return 0;
    for (int j = ORDER_WINDOW_QUADS; 16 * j < hlen; j++) {
        uint32_t w[4];
        tq.next(w);
#pragma unroll
        for (int x = 0; x < 4; x++) {
            h1 = (h1 ^ w[x]) * 0xCC9E2D51u;
            h2 = (h2 + w[x]) * 0x1B873593u ^ (h2 >> 15);
        }
    }
    return fmix64(((uint64_t) h1 << 32) | h2) & q.dedup_hash_mask;
}

// key = tenant index (T bits) | hash(level 0) | hash(levels 0..1) | hash(levels 0..2): equal leading levels => equal digits =>
// one bucket. Hash collisions only merge groups. Topics with fewer levels use digit 0. One digit per level among the first
// three, each the hash of the PREFIX that ends with the level; one pass over the window words with a running hash, a digit
// taken at each of the first three '/' (or at the end of the window for the last, unterminated level). Returns the bucket:
// the key's leading hist_bits bits.
__device__ __forceinline__ uint32_t order_bucket(const uint32_t (&k)[ORDER_WINDOW_WORDS], int hlen, int tn, int tenant_bits, int key_bits,
                                                 int hist_bits) {
    const int len = min(hlen, 4 * ORDER_WINDOW_WORDS);
    const int rest = key_bits - tenant_bits;
    const int b0 = rest / 3 + (rest % 3 > 0), b1 = rest / 3 + (rest % 3 > 1), b2 = rest / 3;
    uint32_t run = 0x9E3779B1u, dig[3] = {0u, 0u, 0u};
    int lvl = 0;   // levels closed so far
#pragma unroll
    for (int j = 0; j < ORDER_WINDOW_WORDS; j++) {
        uint32_t m = 4 * j < len ? match_bytes(k[j], 0x2F2F2F2Fu) : 0u;   // 0x80 flag in every byte that is '/' (a byte above a match may be flagged too)
        while (m && lvl < 3) {
            const int byte = (__ffs(m) - 1) >> 3;
            m &= m - 1;
            if (((k[j] >> (8 * byte)) & 0xFFu) != 0x2Fu) continue;   // the SWAR test's false positive
            const uint32_t part = byte ? (k[j] & (0xFFFFFFFFu >> (32 - 8 * byte))) : 0u;   // the word's bytes before the '/'
            const uint32_t hh = (run ^ part) * 0x85EBCA77u + (uint32_t) (4 * j + byte);
            dig[lvl++] = (hh ^ (hh >> 15)) * 0x9E3779B1u;
        }
        run = (run ^ k[j]) * 0xCC9E2D51u;
        run ^= run >> 13;
    }
    const int closed = lvl;                       // levels that ended with a '/' inside the window
    if (lvl < 3) dig[lvl] = ((run + (uint32_t) len) ^ (run >> 15)) * 0x9E3779B1u;   // the level that runs to the end of the window
    uint32_t key = tenant_bits ? ((uint32_t) max(tn, 0) & ((1u << tenant_bits) - 1u)) : 0u;
    key = (key << b0) | (b0 ? dig[0] >> (32 - b0) : 0u);
    key = (key << b1) | (b1 && closed >= 1 ? dig[1] >> (32 - b1) : 0u);
    key = (key << b2) | (b2 && closed >= 2 ? dig[2] >> (32 - b2) : 0u);
    return key_bits > hist_bits ? key >> (key_bits - hist_bits) : key;
}

// One thread per topic. The order key's bucket is computed first, so nothing of the topic's window is live across the de-dup
// probe: the kernel fits 48 registers, 5 CTAs per SM instead of 4, and the probe (a chain of dependent L2 round trips, with a
// byte compare against the leader at every tag match) is hidden by more resident warps. An empty slot is claimed with
// atomicCAS and no load before it: the CAS returns what it found, one L2 round trip per step. Slots never change once
// claimed, so the first inserter of a (tenant, topic) pair leads and every later one finds it. A leader counts itself into
// the bucket histogram.
__global__ void __launch_bounds__(256, 5) order_prep_kernel(const OrderKernelParams q, int tenant_bits, int key_bits) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= q.n_topics) return;
    uint32_t k[ORDER_WINDOW_WORDS];
    int hlen, tn;
    const uint64_t h = read_topic(q, i, hlen, tn, k);
    const uint32_t bucket = order_bucket(k, hlen, tn, tenant_bits, key_bits, q.hist_bits);
    uint32_t lead = (uint32_t) i;
    if (q.dedup) {
        const unsigned long long mine = ((unsigned long long) (uint32_t) (h >> 32) << 32) | (unsigned long long) (uint32_t) i;
        for (uint32_t slot = (uint32_t) h & q.hash_mask;; slot = (slot + 1) & q.hash_mask) {
            const unsigned long long cur = atomicCAS(&q.hash_tab[slot], ~0ull, mine);
            if (cur == ~0ull) break;   // claimed: this topic leads
            if ((uint32_t) (cur >> 32) == (uint32_t) (h >> 32) && same_pair(q, (uint32_t) i, (uint32_t) cur)) {
                lead = (uint32_t) cur;
                break;
            }
        }
    }
    q.leader[i] = lead;
    if (lead != (uint32_t) i) return;
    q.keys[i] = bucket;
    atomicAdd(&q.hist[bucket], 1u);
}

// exclusive scan of the bucket histogram, in place: every block scans its 4096 counters and publishes its total; the last
// block to finish (ticket) scans the <= 1024 block totals into blk_pfx and writes the grand total (= number of leaders)
constexpr int SCAN_THREADS = 1024, SCAN_PER_BLOCK = 4096;
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums, uint32_t& total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(FULL, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sums[wid] = inc;
    __syncthreads();
    if (wid == 0) {
        const uint32_t ws = warp_sums[lane];
        uint32_t winc = ws;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(FULL, winc, o);
            if (lane >= o) winc += y;
        }
        warp_sums[lane] = winc - ws;
        if (lane == 31) warp_sums[32] = winc;
    }
    __syncthreads();
    total = warp_sums[32];
    const uint32_t r = warp_sums[wid] + inc - v;
    __syncthreads();
    return r;
}
__global__ void __launch_bounds__(SCAN_THREADS) order_scan_kernel(const OrderKernelParams q) {
    __shared__ uint32_t warp_sums[33];
    __shared__ bool is_last;
    uint4* hv = reinterpret_cast<uint4*>(q.hist + (size_t) blockIdx.x * SCAN_PER_BLOCK) + threadIdx.x;
    const uint4 c = *hv;
    uint32_t total;
    const uint32_t ex = block_exclusive_scan(c.x + c.y + c.z + c.w, warp_sums, total);
    *hv = make_uint4(ex, ex + c.x, ex + c.x + c.y, ex + c.x + c.y + c.z);
    if (threadIdx.x == 0) {
        q.blk_tot[blockIdx.x] = total;
        __threadfence();
        is_last = atomicAdd(q.ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const uint32_t v = threadIdx.x < gridDim.x ? *((volatile uint32_t*) q.blk_tot + threadIdx.x) : 0u;
    const uint32_t pfx = block_exclusive_scan(v, warp_sums, total);
    if (threadIdx.x < gridDim.x) q.blk_pfx[threadIdx.x] = pfx;
    if (threadIdx.x == 0) q.counters[CTR_NLEAD] = total;
}
__global__ void __launch_bounds__(256) order_scatter_kernel(const OrderKernelParams q) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= q.n_topics || q.leader[i] != (uint32_t) i) return;
    const uint32_t b = q.keys[i];
    const uint32_t at = q.blk_pfx[b / SCAN_PER_BLOCK] + atomicAdd(&q.hist[b], 1u);
    q.order[at] = (uint32_t) i;
    q.keys[i] = at;   // the bucket is dead now: keep the position for finalize_kernel (a coalesced store)
}

// Topic order from tier 0's position records: a leader's record goes to its own index, a follower takes its leader's (spans
// index the sparse range array, so the ranges themselves are shared). Every access but the record read is coalesced.
__global__ void __launch_bounds__(256) finalize_kernel(const FinalizeParams p) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n_topics) return;
    const uint32_t l = p.leader[i];
    if (!p.second_pass) {
        const SpanRecord r = p.pos_rec[p.pos[l]];
        if (!r.deferred) {
            p.span_begin[i] = r.span_begin;
            p.span_count[i] = r.span_count;
            p.route_count[i] = r.route_count;
            // a flagged leader joined the list in tier 0
            if (l != (uint32_t) i && (r.span_count & SPAN_FLAGGED)) p.flagged_list[atomicAdd(&p.counters[CTR_FLAGGED], 1ull)] = (uint32_t) i;
            return;
        }
        // deferred to tier 1, which wrote the leader's topic-indexed span: a follower copies it below
    }
    if (l == (uint32_t) i) return;
    if (p.second_pass && p.span_count[i] != SPAN_OVERFLOW) return;
    const uint32_t sc = p.span_count[l];
    p.span_begin[i] = p.span_begin[l];
    p.span_count[i] = sc;
    p.route_count[i] = p.route_count[l];
    if (sc & SPAN_FLAGGED) p.flagged_list[atomicAdd(&p.counters[CTR_FLAGGED], 1ull)] = (uint32_t) i;
}

// ------------------------------------------------------------------------------------------------ compaction
// counts[i] = ranges topic i contributes to the dense array: its own, or none if it repeats an earlier (tenant, topic) pair —
// a repeat shares its leader's dense span instead of copying it (a third of BASELINE C4's batch: 13 MB less D2H per 1M topics)
__global__ void compact_counts_kernel(const CompactParams p) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n_topics) p.counts[i] = (p.leader && p.leader[i] != (uint32_t) i) ? 0u : (p.span_count[i] & SPAN_COUNT_MASK);
}
__global__ void compact_total_kernel(const CompactParams p) {
    *p.total_out = (unsigned long long) p.new_begin[p.n_topics - 1] + p.counts[p.n_topics - 1];
}
__global__ void compact_gather_kernel(const CompactParams p) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= p.n_topics) return;
    const uint32_t l = p.leader ? p.leader[i] : (uint32_t) i;
    const uint32_t c = p.span_count[i] & SPAN_COUNT_MASK;     // a repeat carries its leader's span (finalize_kernel)
    const uint32_t nb = p.new_begin[l];                       // the scan's output is not modified here: no race with the leader's thread
    if (l == (uint32_t) i) {
        const uint32_t ob = p.span_begin[i];
        if ((uint64_t) nb + c <= p.ranges_out_cap)
            for (uint32_t j = 0; j < c; j++) p.ranges_out[nb + j] = p.ranges[ob + j];
    }
    p.final_begin[i] = nb + p.out_base;   // position in the concatenated result
    p.final_count[i] = c;
}

// ------------------------------------------------------------------------------------------------ caps
// Fan-out caps of MatchedRoutes (bifromq-dist/bifromq-dist-worker/.../cache/MatchedRoutes.java:87-141): among a
// topic's matched routes taken in KV (rank) order, only the first maxPersistentFanout persistent normal routes
// (subBrokerId == 1) and the first maxGroupFanout group routes survive; every later one is dropped and reported.
// One CTA per flagged topic. A route's index among the matched persistent routes is
//   (# persistent routes in matched segments that start before its segment) + (# persistent before it in its segment),
// both read off exclusive prefix counts over the rank space, so no sort of the ranges is needed.
constexpr int CAPS_THREADS = 128;

struct SegIter {  // iterate the segments {first,count} behind a topic's ranges (resolving multi-segment ranges)
    const uint2* ranges;
    const uint32_t* segs;
    uint32_t n;
    template <typename F>
    __device__ __forceinline__ void for_range(uint32_t j, F&& f) const {
        const uint2 r = ranges[j];
        if (r.y & RANGE_MULTI) {
            const uint32_t nseg = segs[2 * (uint64_t) r.x];
            for (uint32_t s = 0; s < nseg; s++) f(segs[2 * ((uint64_t) r.x + 1 + s)], segs[2 * ((uint64_t) r.x + 1 + s) + 1]);
        } else {
            f(r.x, r.y);
        }
    }
};

__device__ __forceinline__ void caps_one(const CapsParams& p, uint32_t t);
__global__ void __launch_bounds__(CAPS_THREADS) caps_kernel(const CapsParams p) {
    if (p.n_flagged >= 0) {
        caps_one(p, p.flagged_list[blockIdx.x]);
        return;
    }
    // counts read on the device: a fixed grid strides over the flagged topics no earlier pass has handled
    const unsigned long long b = p.counters[CTR_FLAGGED2], e = p.counters[CTR_FLAGGED];
    for (unsigned long long j = b + blockIdx.x; j < e; j += gridDim.x) {
        caps_one(p, p.flagged_list[j]);
        __syncthreads();
    }
}
__device__ __forceinline__ void caps_one(const CapsParams& p, uint32_t t) {
    const int tenant = p.topic_tenant[t];
    const uint64_t maxP = (uint64_t) max(p.max_pfanout[tenant], 0), maxG = (uint64_t) max(p.max_gfanout[tenant], 0);
    SegIter it{p.ranges + p.span_begin[t], p.segs, p.span_count[t] & SPAN_COUNT_MASK};
    __shared__ unsigned long long kept;
    if (threadIdx.x == 0) kept = 0;
    __syncthreads();
    unsigned long long my_kept = 0;
    for (uint32_t j = threadIdx.x; j < it.n; j += CAPS_THREADS) {
        it.for_range(j, [&](uint32_t first, uint32_t count) {
            // persistent / group routes in matched segments that start before this one
            uint64_t baseP = 0, baseG = 0;
            for (uint32_t q = 0; q < it.n; q++)
                it.for_range(q, [&](uint32_t f2, uint32_t c2) {
                    if (f2 < first) {
                        baseP += p.pfx_persistent[f2 + c2] - p.pfx_persistent[f2];
                        baseG += p.pfx_group[f2 + c2] - p.pfx_group[f2];
                    }
                });
            const uint64_t cntP = p.pfx_persistent[first + count] - p.pfx_persistent[first];
            const uint64_t cntG = p.pfx_group[first + count] - p.pfx_group[first];
            if (baseP + cntP <= maxP && baseG + cntG <= maxG) {
                my_kept += count;
                return;
            }
            for (uint32_t r = first; r < first + count; r++) {
                const uint8_t kind = p.rkind[r];
                uint32_t drop = 0;
                if (kind == 1 && baseP + (p.pfx_persistent[r] - p.pfx_persistent[first]) >= maxP) drop = 1;
                else if (kind == 2 && baseG + (p.pfx_group[r] - p.pfx_group[first]) >= maxG) drop = 2;
                if (drop) {
                    const unsigned long long idx = atomicAdd(&p.counters[CTR_THROTTLED], 1ull);
                    if (idx < p.throttled_cap) p.throttled[idx] = make_uint3(t + p.topic_base, r, drop);
                } else {
                    my_kept++;
                }
            }
        });
    }
    atomicAdd(&kept, my_kept);
    __syncthreads();
    if (threadIdx.x == 0 && p.kept_count) p.kept_count[t] = (uint32_t) kept;
}
// marks everything flagged so far as handled (the next device-counted caps pass starts behind it)
__global__ void caps_advance_kernel(unsigned long long* counters) { counters[CTR_FLAGGED2] = counters[CTR_FLAGGED]; }

// ------------------------------------------------------------------------------------------------ expand (device CSR)
__global__ void expand_counts_kernel(const ExpandParams p) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < p.n_topics) p.counts[i] = (p.span_count[i] & SPAN_FLAGGED) ? p.kept_count[i] : p.route_count[i];
    if (i == p.n_topics) p.counts[i] = 0;
}
// one warp per topic that needs no caps: every rank of every range
__global__ void __launch_bounds__(256) expand_plain_kernel(const ExpandParams p) {
    const int lane = threadIdx.x & 31;
    const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= p.n_topics || (p.span_count[t] & SPAN_FLAGGED)) return;
    SegIter it{p.ranges + p.span_begin[t], p.segs, p.span_count[t] & SPAN_COUNT_MASK};
    int64_t pos = p.offsets[t];
    for (uint32_t j = 0; j < it.n; j++)
        it.for_range(j, [&](uint32_t first, uint32_t count) {
            for (uint32_t x = lane; x < count; x += 32)
                if (pos + x < p.rank_cap) p.ranks[pos + x] = (int64_t) first + x;
            pos += count;
        });
}
// Writes topic t's ranks that survive a persistent cap maxP and a group cap maxG (KV order, the classification of
// caps_kernel), dropping transient routes too if drop_t. One CTA of CAPS_THREADS per topic.
__device__ __forceinline__ void copy_capped(const ExpandParams& p, uint32_t t, uint64_t maxP, uint64_t maxG, bool drop_t);
// one CTA per cap-flagged topic: same classification as caps_kernel, the survivors are written
__global__ void __launch_bounds__(CAPS_THREADS) expand_flagged_kernel(const ExpandParams p) {
    const uint32_t t = p.flagged_list[blockIdx.x];
    const int tenant = p.topic_tenant[t];
    copy_capped(p, t, (uint64_t) max(p.max_pfanout[tenant], 0), (uint64_t) max(p.max_gfanout[tenant], 0), false);
}
__device__ __forceinline__ void copy_capped(const ExpandParams& p, uint32_t t, uint64_t maxP, uint64_t maxG, bool drop_t) {
    SegIter it{p.ranges + p.span_begin[t], p.segs, p.span_count[t] & SPAN_COUNT_MASK};
    __shared__ unsigned long long cursor;
    if (threadIdx.x == 0) cursor = 0;
    __syncthreads();
    const int64_t base = p.offsets[t];
    for (uint32_t j = threadIdx.x; j < it.n; j += CAPS_THREADS) {
        it.for_range(j, [&](uint32_t first, uint32_t count) {
            uint64_t baseP = 0, baseG = 0;
            for (uint32_t q = 0; q < it.n; q++)
                it.for_range(q, [&](uint32_t f2, uint32_t c2) {
                    if (f2 < first) {
                        baseP += p.pfx_persistent[f2 + c2] - p.pfx_persistent[f2];
                        baseG += p.pfx_group[f2 + c2] - p.pfx_group[f2];
                    }
                });
            for (uint32_t r = first; r < first + count; r++) {
                const uint8_t kind = p.rkind[r];
                const bool drop = (kind == 1 && baseP + (p.pfx_persistent[r] - p.pfx_persistent[first]) >= maxP) ||
                                  (kind == 2 && baseG + (p.pfx_group[r] - p.pfx_group[first]) >= maxG) ||
                                  (kind == 0 && drop_t);
                if (!drop) {
                    const unsigned long long k = atomicAdd(&cursor, 1ull);
                    if (base + (int64_t) k < p.rank_cap) p.ranks[base + k] = (int64_t) r;
                }
            }
        });
    }
}

// ------------------------------------------------------------------------------------------------ delivery budgets
// DeliverExecutorGroup.submit (bifromq-dist-worker .../DeliverExecutorGroup.java:112-231) over a topic's surviving routes R
// (the match's caps applied): |R| <= 1 is delivered as is; otherwise groups are delivered, transient routes only with
// transient bandwidth, and persistent routes only with persistent bandwidth and while sent * s < MaxPersistentFanoutBytes:
// the first k = min(P, ceil(B / s)) of them in KV order (all P when s == 0).
// One warp per topic: |R|, P and G from the prefix counts over the topic's ranges, then k, the flags and the delivered count.
__global__ void __launch_bounds__(256) budget_pass_kernel(const BudgetParams q) {
    const ExpandParams& p = q.e;
    const int lane = threadIdx.x & 31;
    const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= p.n_topics) {
        if (t == p.n_topics && lane == 0) p.counts[t] = 0;
        return;
    }
    const uint32_t sc = p.span_count[t];
    SegIter it{p.ranges + p.span_begin[t], p.segs, sc & SPAN_COUNT_MASK};
    uint64_t n = 0, np = 0, ng = 0;
    for (uint32_t j = lane; j < it.n; j += 32)
        it.for_range(j, [&](uint32_t first, uint32_t count) {
            n += count;
            np += p.pfx_persistent[first + count] - p.pfx_persistent[first];
            ng += p.pfx_group[first + count] - p.pfx_group[first];
        });
    for (int o = 16; o > 0; o >>= 1) {
        n += __shfl_xor_sync(0xFFFFFFFFu, n, o);
        np += __shfl_xor_sync(0xFFFFFFFFu, np, o);
        ng += __shfl_xor_sync(0xFFFFFFFFu, ng, o);
    }
    if (lane != 0) return;
    const int32_t s = q.msg_bytes[t];
    if (s < 0) atomicAdd(&q.ctr[BUD_BAD_SIZE], 1ull);
    const int tenant = p.topic_tenant[t];
    const bool known = tenant >= 0 && tenant < q.n_tenants;   // an unknown tenant matches nothing
    uint64_t P = np, G = ng;
    if ((sc & SPAN_FLAGGED) && known) {
        P = min(P, (uint64_t) max(p.max_pfanout[tenant], 0));
        G = min(G, (uint64_t) max(p.max_gfanout[tenant], 0));
    }
    const uint64_t T = n - np - ng, R = T + P + G;
    uint64_t k = P, tdel = T;
    uint8_t f = (R > 1 || P == 1) ? BUDGET_METERED : 0;
    if (R > 1 && known) {
        const uint8_t bw = q.bandwidth[tenant];
        if (!(bw & 2) && T > 0) {
            tdel = 0;
            f |= BUDGET_NO_TRANSIENT_BW;
            atomicAdd(&q.ctr[BUD_DROP_TBW], (unsigned long long) T);
        }
        if (!(bw & 1)) {
            if (P > 0) {
                k = 0;
                f |= BUDGET_NO_PERSISTENT_BW;
                atomicAdd(&q.ctr[BUD_DROP_PBW], (unsigned long long) P);
            }
        } else if (s > 0) {
            // ceil(B / s) without overflow (B >= 1): the number of sends for which sent * s < B still held
            const uint64_t m = ((uint64_t) q.max_bytes[tenant] - 1) / (uint64_t) s + 1;
            if (m < P) {
                k = m;
                f |= BUDGET_BYTES_THROTTLED;
                atomicAdd(&q.ctr[BUD_DROP_BYTES], (unsigned long long) (P - m));
            }
        }
        if (f & BUDGET_DROPS) q.list[atomicAdd(&q.ctr[BUD_LISTED], 1ull)] = (uint32_t) t;
    }
    p.counts[t] = tdel + k + G;
    q.delivered_p[t] = (uint32_t) k;
    q.flags[t] = f;
}
// one warp per topic the budget and the caps leave whole
__global__ void __launch_bounds__(256) budget_plain_kernel(const BudgetParams q) {
    const ExpandParams& p = q.e;
    const int lane = threadIdx.x & 31;
    const int64_t t = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= p.n_topics || (p.span_count[t] & SPAN_FLAGGED) || (q.flags[t] & BUDGET_DROPS)) return;
    SegIter it{p.ranges + p.span_begin[t], p.segs, p.span_count[t] & SPAN_COUNT_MASK};
    int64_t pos = p.offsets[t];
    for (uint32_t j = 0; j < it.n; j++)
        it.for_range(j, [&](uint32_t first, uint32_t count) {
            for (uint32_t x = lane; x < count; x += 32)
                if (pos + x < p.rank_cap) p.ranks[pos + x] = (int64_t) first + x;
            pos += count;
        });
}
// one CTA per cap-flagged topic (blocks [0, n_flagged)) and per budget-listed topic (the rest). A topic on both lists is
// copied by its listed block only, under min(maxP, k): the match's cap and the budget keep KV-order prefixes of the same
// persistent routes, so together they keep the shorter one.
__global__ void __launch_bounds__(CAPS_THREADS) budget_capped_kernel(const BudgetParams q) {
    const ExpandParams& p = q.e;
    const bool listed = blockIdx.x >= p.n_flagged;
    const uint32_t t = listed ? q.list[blockIdx.x - p.n_flagged] : p.flagged_list[blockIdx.x];
    const uint8_t f = q.flags[t];
    if (!listed && (f & BUDGET_DROPS)) return;
    uint64_t maxP = listed ? q.delivered_p[t] : ~0ull, maxG = ~0ull;
    if (p.span_count[t] & SPAN_FLAGGED) {
        const int tenant = p.topic_tenant[t];
        maxP = min(maxP, (uint64_t) max(p.max_pfanout[tenant], 0));
        maxG = (uint64_t) max(p.max_gfanout[tenant], 0);
    }
    copy_capped(p, t, maxP, maxG, (f & BUDGET_NO_TRANSIENT_BW) != 0);
}

}  // namespace

namespace {
// moves the ranks of one node record by d: its own / '#' first-rank words, unless the slot is free, the target is empty, or
// the word indexes the segment table (a MULTI target; its ranks are shifted on the host)
__device__ __forceinline__ void shift_record_ranks(uint32_t* w, uint32_t d) {
    if (w[W_PARENT] == EMPTY_PARENT) return;
    const uint32_t meta = w[W_META];
    if (w[W_OWN_COUNT] > 0 && !(meta & FLAG_OWN_MULTI)) w[W_OWN_FIRST] += d;
    if (w[W_HASH_COUNT] > 0 && !(meta & FLAG_HASH_MULTI)) w[W_HASH_FIRST] += d;
}
__global__ void __launch_bounds__(256) rank_shift_kernel(Slot* slots, const RankShiftRegion* regions, int n_regions) {
    // a CTA takes a region at a time; regions differ in size by orders of magnitude, so big ones are cut into pieces of 8192
    // slots that all CTAs pick up (piece index = blockIdx, striding)
    for (int r = 0; r < n_regions; r++) {
        const RankShiftRegion rg = regions[r];
        const uint32_t d = (uint32_t) rg.delta;
        for (uint64_t s = (uint64_t) blockIdx.x * blockDim.x + threadIdx.x; s < rg.len; s += (uint64_t) gridDim.x * blockDim.x)
            shift_record_ranks(slots[rg.base + s].w, d);
    }
}
// the tag-table records of the tenants whose ranks moved: one thread per listed slot (they are scattered over the table)
__global__ void __launch_bounds__(256) rank_shift_listed_kernel(Slot* slots, const RankShiftSlot* list, int64_t n) {
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x) {
        const RankShiftSlot e = list[i];
        shift_record_ranks(slots[e.slot].w, (uint32_t) e.delta);
    }
}
// rebuilt tenants' tag-table records to their slots: 16 threads per record, one word each (coalesced 64-byte stores)
__global__ void __launch_bounds__(256) scatter_records_kernel(Slot* slots, const uint32_t* ids, const Slot* recs, int64_t n) {
    for (int64_t t = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; t < n * 16; t += (int64_t) gridDim.x * blockDim.x) {
        const int64_t i = t >> 4;
        const uint32_t k = (uint32_t) t & 15u;
        slots[ids[i]].w[k] = recs[i].w[k];
    }
}
// one thread per rank (striding); a thread finds its run by binary search over the run starts (a warp's lanes almost always
// land in the same run, so the probes are broadcasts from L1)
__global__ void __launch_bounds__(256) assemble_rank_arrays_kernel(const AssembleRankParams p) {
    for (int64_t r = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; r <= p.n; r += (int64_t) gridDim.x * blockDim.x) {
        if (r == p.n) {
            p.pfxP[r] = p.tailP;
            p.pfxG[r] = p.tailG;
            continue;
        }
        int lo = 0, hi = p.n_runs - 1;   // the last run with new_lo <= r
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if ((int64_t) p.runs[mid].new_lo <= r) lo = mid;
            else hi = mid - 1;
        }
        const RankRun run = p.runs[lo];
        const uint32_t s = run.src_lo + (uint32_t) (r - run.new_lo);
        const uint8_t* rk = run.packed ? p.up_rkind : p.old_rkind;
        const uint32_t* pP = run.packed ? p.up_pfxP : p.old_pfxP;
        const uint32_t* pG = run.packed ? p.up_pfxG : p.old_pfxG;
        p.rkind[r] = rk[s];
        p.pfxP[r] = pP[s] + run.dP;
        p.pfxG[r] = pG[s] + run.dG;
    }
}
}  // namespace

int device_sm_count() {
    static std::mutex mu;
    static int sms_of[64] = {0};   // per device ordinal
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu);
    int& sms = sms_of[dev & 63];
    if (sms == 0 && (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1)) sms = 132;
    return sms;
}

void launch_rank_shift(Slot* slots, const RankShiftRegion* d_regions, int n_regions, cudaStream_t stream) {
    if (n_regions <= 0) return;
    rank_shift_kernel<<<device_sm_count() * 8, 256, 0, stream>>>(slots, d_regions, n_regions);
}
void launch_rank_shift_listed(Slot* slots, const RankShiftSlot* d_list, int64_t n, cudaStream_t stream) {
    if (n <= 0) return;
    rank_shift_listed_kernel<<<(unsigned) std::min<int64_t>((n + 255) / 256, (int64_t) device_sm_count() * 16), 256, 0, stream>>>(slots, d_list, n);
}
void launch_scatter_records(Slot* slots, const uint32_t* d_ids, const Slot* d_recs, int64_t n, cudaStream_t stream) {
    if (n <= 0) return;
    scatter_records_kernel<<<(unsigned) std::min<int64_t>((n * 16 + 255) / 256, (int64_t) device_sm_count() * 16), 256, 0, stream>>>(slots, d_ids, d_recs, n);
}
void launch_assemble_rank_arrays(const AssembleRankParams& p, cudaStream_t stream) {
    assemble_rank_arrays_kernel<<<(unsigned) std::min<int64_t>((p.n + 1 + 255) / 256, (int64_t) device_sm_count() * 16), 256, 0, stream>>>(p);
}

int match_kernel_smem_bytes() { return (int) sizeof(WarpSmem) * WARPS_PER_CTA; }

void launch_match(const MatchParams& p, bool tier2, int n_warps_tier2, cudaStream_t stream) {
    if (tier2) {
        const int ctas = (n_warps_tier2 + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
        match_topics_kernel<true><<<ctas, WARPS_PER_CTA * 32, 0, stream>>>(p);
        return;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    const int sms = device_sm_count();
    // occupancy is a property of the device / context: cached per device ordinal
    static std::mutex occ_mu;
    static int occ_of[64] = {0};
    int ctas_per_sm;
    {
        std::lock_guard<std::mutex> g(occ_mu);
        int& slot = occ_of[dev & 63];
        if (slot == 0) {
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&slot, match_topics_kernel<false>, WARPS_PER_CTA * 32, 0);
            if (slot < 1) slot = 1;
        }
        ctas_per_sm = slot;
    }
    // persistent grid: a whole number of waves (SM count x resident CTAs per SM), grid-stride over topics
    int64_t ctas = (int64_t) sms * ctas_per_sm;
    // chained behind tier 0 (n_work < 0: count read on the device) the deferral list is short: one CTA per SM
    if (p.work_list && p.n_work < 0) ctas = sms;
    const int64_t items = p.work_list ? (p.n_work >= 0 ? p.n_work : p.n_topics) : p.n_topics;
    const int64_t need = (items + WARPS_PER_CTA - 1) / WARPS_PER_CTA;
    if (need < ctas) ctas = need < 1 ? 1 : need;
    match_topics_kernel<false><<<(unsigned) ctas, WARPS_PER_CTA * 32, 0, stream>>>(p);
}

static int order_tenant_bits(int32_t n_tenants) {
    int tenant_bits = 0;
    while (tenant_bits < 20 && (1ll << tenant_bits) < (long long) n_tenants) tenant_bits++;
    return tenant_bits;
}
static int order_key_bits(int tenant_bits) {
    // width of the order key: tenant bits + ~14 bits of level hashes (1000 tenants: 24 bits). BFQ_ORDER_BITS overrides (experiments).
    static const int forced_bits = [] {
        const char* e = getenv("BFQ_ORDER_BITS");
        return e ? std::min(std::max(atoi(e), 8), 32) : 0;
    }();
    int kb = forced_bits ? forced_bits : std::min(32, (tenant_bits + 12 + 7) / 8 * 8);
    return std::max(kb, std::min(32, tenant_bits + 3));
}
static int order_hist_bits(int64_t n_topics, int32_t n_tenants) {
    // buckets = the key's leading bits: at most 2^22 (a 16 MB histogram: zeroed and scanned in a few microseconds) and about
    // four per topic for smaller batches; at least 2^12 (one scan block)
    int nb = 12;
    while (nb < 22 && (1ll << nb) < 4 * n_topics) nb++;
    return std::max(12, std::min(nb, order_key_bits(order_tenant_bits(n_tenants))));
}
// the scratch of one ordering: histogram | block totals | block prefixes | ticket (kept 256-byte aligned)
size_t order_scratch_words(int64_t n_topics, int32_t n_tenants) {
    const size_t buckets = (size_t) 1 << order_hist_bits(n_topics, n_tenants);
    return (buckets + 2 * (buckets / SCAN_PER_BLOCK) + 64 + 63) / 64 * 64;
}
uint32_t order_hash_entries(int64_t n_topics) {
    uint32_t e = 1024;
    while (e < (1u << 31) && (int64_t) e < 2 * n_topics) e <<= 1;
    return e;
}

cudaError_t launch_order(const OrderParams& p, cudaStream_t stream) {
    const int64_t n = p.n_topics;
    if (n <= 0) return cudaSuccess;
    const int hist_bits = order_hist_bits(n, p.n_tenants);
    const size_t buckets = (size_t) 1 << hist_bits, scan_blocks = buckets / SCAN_PER_BLOCK;
    uint32_t* blk_tot = p.hist + buckets;
    const OrderKernelParams q{p.n_topics, p.topics, p.topic_off, p.topic_tenant, p.n_tenants, p.keys, p.leader, p.order,
                              p.hash_tab, p.hash_mask, p.hist, blk_tot, blk_tot + scan_blocks, blk_tot + 2 * scan_blocks, hist_bits,
                              p.dedup, p.dedup_hash_mask, p.counters};
    cudaError_t e = cudaMemsetAsync(q.hist, 0, order_scratch_words(n, p.n_tenants) * sizeof(uint32_t), stream);
    if (e == cudaSuccess && q.dedup) e = cudaMemsetAsync(q.hash_tab, 0xFF, ((size_t) q.hash_mask + 1) * sizeof(unsigned long long), stream);
    if (e != cudaSuccess) return e;
    const int tenant_bits = order_tenant_bits(q.n_tenants);
    const int kb = order_key_bits(tenant_bits);
    const unsigned blocks = (unsigned) ((n + 255) / 256);
    order_prep_kernel<<<blocks, 256, 0, stream>>>(q, tenant_bits, kb);
    order_scan_kernel<<<(unsigned) scan_blocks, SCAN_THREADS, 0, stream>>>(q);
    order_scatter_kernel<<<blocks, 256, 0, stream>>>(q);
    return cudaGetLastError();
}

void launch_finalize(const FinalizeParams& p, cudaStream_t stream) {
    if (p.n_topics <= 0) return;
    finalize_kernel<<<(unsigned) ((p.n_topics + 255) / 256), 256, 0, stream>>>(p);
}

void launch_match_lanes(const MatchParams& p, cudaStream_t stream) {
    int dev = 0;
    cudaGetDevice(&dev);
    const int sms = device_sm_count();
    // experiment switches: BFQ_ROOTSTEP=0/1, BFQ_PREFETCH=0/1, BFQ_NOALLOC=0/1, BFQ_CTAS=n, BFQ_CARVEOUT=percent.
    // Node records allocate in L1: on an H100 that is faster than bypassing it (ld.global.nc.L1::no_allocate) in locality
    // order as well as in arrival order — neighbouring lanes walk the same top of the trie, which then stays in L1.
    typedef void (*kern_t)(const MatchParams);
    static const kern_t kerns[8] = {match_topics_lane_kernel<false, false, false>, match_topics_lane_kernel<false, true, false>,
                                    match_topics_lane_kernel<true, false, false>,  match_topics_lane_kernel<true, true, false>,
                                    match_topics_lane_kernel<false, false, true>,  match_topics_lane_kernel<false, true, true>,
                                    match_topics_lane_kernel<true, false, true>,   match_topics_lane_kernel<true, true, true>};
    static std::mutex setup_mu;
    static int ctas_by_dev[64][8] = {};   // function attributes (the carve-out) and occupancy are per device: cached per ordinal
    static const int rootstep = getenv("BFQ_ROOTSTEP") ? atoi(getenv("BFQ_ROOTSTEP")) : 0;
    static const int prefetch = getenv("BFQ_PREFETCH") ? atoi(getenv("BFQ_PREFETCH")) : 1;
    static const int noalloc_forced = getenv("BFQ_NOALLOC") ? atoi(getenv("BFQ_NOALLOC")) : -1;
    static const int ctas_forced = getenv("BFQ_CTAS") ? std::max(1, atoi(getenv("BFQ_CTAS"))) : 0;
    const int noalloc = noalloc_forced >= 0 ? noalloc_forced : 0;
    const int variant = (noalloc ? 4 : 0) + (rootstep ? 2 : 0) + (prefetch ? 1 : 0);
    int ctas_per_sm;
    {
        std::lock_guard<std::mutex> g(setup_mu);
        int* ctas_of = ctas_by_dev[dev & 63];
        if (ctas_of[variant] == 0) {
            // Shared memory and L1 share 256 KB per SM, and the kernel lives on L1 (topic bytes, top trie levels): the
            // 228 KB carve-out (what 8 resident CTAs need) would leave 28 KB of L1, leaving it to the driver is slower still.
            // Ask for the 196 KB carve-out (60 KB L1) and size the persistent grid for what fits there.
            cudaFuncAttributes fa{};
            cudaFuncGetAttributes(&fa, kerns[variant]);
            const char* cv = getenv("BFQ_CARVEOUT");   // experiment switch: percent of the 228 KB, 0 = leave it to the driver
            const int carve = cv ? atoi(cv) : 85;
            if (carve > 0) cudaFuncSetAttribute(kerns[variant], cudaFuncAttributePreferredSharedMemoryCarveout, carve);
            int occ = 0;
            cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kerns[variant], L_WARPS * 32, 0);
            const int fit = (int) ((196 * 1024) / (fa.sharedSizeBytes + 1024));
            if (occ > fit) occ = fit;
            if (ctas_forced) occ = std::min(occ, ctas_forced);
            ctas_of[variant] = occ < 1 ? 1 : occ;
        }
        ctas_per_sm = ctas_of[variant];
    }
    // A large batch runs faster with fewer resident CTAs than fit: on an H100, 4 per SM beat 5 / 6 / 7 on 1M-topic batches
    // (fewer requests contend for L1 and the memory system; there is work for every lane anyway). A smaller batch (below
    // LARGE_BATCH_TOPICS, e.g. 100k topics) keeps every CTA that fits, or it would leave lanes it needs unscheduled.
    if (!ctas_forced && p.n_topics >= LARGE_BATCH_TOPICS) ctas_per_sm = std::min(ctas_per_sm, LARGE_BATCH_CTAS_PER_SM);
    // persistent grid (SM count x resident CTAs); warps claim 32-topic chunks with one atomicAdd each
    if (p.max_ctas_per_sm > 0) ctas_per_sm = std::min(ctas_per_sm, (int) p.max_ctas_per_sm);
    int64_t ctas = (int64_t) sms * ctas_per_sm;
    const int64_t need = ((p.n_topics + L_CHUNK - 1) / L_CHUNK + L_WARPS - 1) / L_WARPS;
    if (need < ctas) ctas = need < 1 ? 1 : need;
    kerns[variant]<<<(unsigned) ctas, L_WARPS * 32, 0, stream>>>(p);
}

cudaError_t launch_compact(const CompactParams& p, void* d_scan_tmp, size_t* tmp_bytes, cudaStream_t stream, int phase) {
    if (!d_scan_tmp) return cub::DeviceScan::ExclusiveSum(nullptr, *tmp_bytes, p.counts, p.new_begin, (int) p.n_topics, stream);
    if (p.n_topics <= 0) return cudaSuccess;
    const unsigned blocks = (unsigned) ((p.n_topics + 255) / 256);
    if (phase == 1) {   // clean counts, exclusive scan, total
        compact_counts_kernel<<<blocks, 256, 0, stream>>>(p);
        cudaError_t e = cub::DeviceScan::ExclusiveSum(d_scan_tmp, *tmp_bytes, p.counts, p.new_begin, (int) p.n_topics, stream);
        if (e != cudaSuccess) return e;
        compact_total_kernel<<<1, 1, 0, stream>>>(p);
    } else {            // gather into the dense array at p.ranges_out (already offset by the caller), rebase new_begin
        compact_gather_kernel<<<blocks, 256, 0, stream>>>(p);
    }
    return cudaGetLastError();
}

cudaError_t launch_expand(const ExpandParams& p, void* d_scan_tmp, size_t* tmp_bytes, cudaStream_t stream, int phase) {
    const int n1 = (int) p.n_topics + 1;
    if (!d_scan_tmp) return cub::DeviceScan::ExclusiveSum(nullptr, *tmp_bytes, p.counts, reinterpret_cast<unsigned long long*>(p.offsets), n1, stream);
    if (phase == 1) {
        expand_counts_kernel<<<(unsigned) ((p.n_topics + 256) / 256), 256, 0, stream>>>(p);
        return cub::DeviceScan::ExclusiveSum(d_scan_tmp, *tmp_bytes, p.counts, reinterpret_cast<unsigned long long*>(p.offsets), n1, stream);
    }
    if (p.n_topics > 0) expand_plain_kernel<<<(unsigned) ((p.n_topics * 32 + 255) / 256), 256, 0, stream>>>(p);
    if (p.n_flagged > 0) expand_flagged_kernel<<<(unsigned) p.n_flagged, CAPS_THREADS, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_budget(const BudgetParams& q, void* d_scan_tmp, size_t* tmp_bytes, cudaStream_t stream, int phase) {
    const ExpandParams& p = q.e;
    const int n1 = (int) p.n_topics + 1;
    if (!d_scan_tmp) return cub::DeviceScan::ExclusiveSum(nullptr, *tmp_bytes, p.counts, reinterpret_cast<unsigned long long*>(p.offsets), n1, stream);
    if (phase == 1) {
        budget_pass_kernel<<<(unsigned) (((p.n_topics + 1) * 32 + 255) / 256), 256, 0, stream>>>(q);
        return cub::DeviceScan::ExclusiveSum(d_scan_tmp, *tmp_bytes, p.counts, reinterpret_cast<unsigned long long*>(p.offsets), n1, stream);
    }
    if (p.n_topics > 0) budget_plain_kernel<<<(unsigned) ((p.n_topics * 32 + 255) / 256), 256, 0, stream>>>(q);
    if (p.n_flagged + q.n_listed > 0) budget_capped_kernel<<<(unsigned) (p.n_flagged + q.n_listed), CAPS_THREADS, 0, stream>>>(q);
    return cudaGetLastError();
}

void launch_caps(const CapsParams& p, cudaStream_t stream) {
    if (p.n_flagged == 0) return;
    if (p.n_flagged > 0) {
        caps_kernel<<<(unsigned) p.n_flagged, CAPS_THREADS, 0, stream>>>(p);
        return;
    }
    // counts on the device (the optimistic, sync-free enqueue): a fixed grid, then advance the handled mark
    caps_kernel<<<device_sm_count() * 4, CAPS_THREADS, 0, stream>>>(p);
    caps_advance_kernel<<<1, 1, 0, stream>>>(p.counters);
}

}  // namespace bfq
