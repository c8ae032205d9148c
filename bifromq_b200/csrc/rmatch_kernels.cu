// rmatch_kernels.cu — inverse match on sm_90a (H100): a batch of topic FILTERS against an index of TOPICS.
//
// Replaces RetainTopicIndex.match / TopicIndex.match
//   (bifromq-retain/bifromq-retain-store/src/main/java/org/apache/bifromq/retain/store/index/RetainTopicIndex.java:36-138,
//    bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/TopicIndex.java:40-155,
//    traversal bifromq-util/src/main/java/org/apache/bifromq/util/index/TopicLevelTrie.java:190-249).
// Same machinery as the forward kernel with the roles swapped: ONE WARP PER FILTER walks the topic trie.
//
// Layout (HBM): each tenant's topic trie is one region of BFS-numbered node records (see the layout comment above
// rebuild_full; a delta commit appends the rebuilt tenants' regions), so
//   * the children of a node — and the children of any RUN of consecutive nodes of one depth — are one
//     contiguous id interval: a '+' level maps a frontier interval to ONE interval with two record loads,
//     it never explodes the frontier;
//   * topics get two ranks: their DFS (pre-order) rank, in which a whole subtree is a contiguous range
//     ("prefix/#" = one range per frontier node), and their BFS rank, in which the topics ending at a run of
//     consecutive nodes are contiguous (a final '+' = one range per frontier interval).
//   * exact levels use the same 64-byte (parent, token) hash slots as the forward index (trie_layout.h),
//     payload word W_PLUS holding the child's BFS id.
// Results are emitted as ranges {space|first, count}; a second kernel maps them to stable topic ids and
// applies the per-filter limit (RetainStoreCoProc.match stops after `limit` messages,
// bifromq-retain/bifromq-retain-store/.../RetainStoreCoProc.java:167-190).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <set>
#include <shared_mutex>
#include <string>
#include <tuple>
#include <unordered_map>
#include <vector>

#include <cub/device/device_scan.cuh>

#include "../../include/bfq_gpumatch.h"
#include "codec.h"
#include "cuda_buf.h"
#include "trie_layout.h"
#include "hash_probe.cuh"
#include "lease.h"
#include "match_kernels.cuh"

using namespace bfq;

namespace {

// one topic-trie node, indexed by node id; the node array has a sentinel entry at [n_nodes]
struct RNode {
    uint32_t child_begin;   // BFS id of the first child (children are consecutive)
    uint32_t child_count;
    uint32_t sub_begin;     // DFS-rank range of the topics in this subtree (own topic first)
    uint32_t sub_end;
    uint32_t own_prefix;    // BFS-rank of the first topic ending at a node with id >= this one
    uint32_t sys_begin;     // children whose name starts with '$' form the run [sys_begin, sys_begin+sys_count)
    uint32_t sys_count;
    uint32_t pad;
};
static_assert(sizeof(RNode) == 32, "RNode is one 32-byte sector");

constexpr uint32_t SPACE_BFS = 0x80000000u;   // tag in a range's `first` word: BFS-rank space (else DFS)
constexpr uint32_t VIRT_BASE = 0x80000000u;   // ids of the intermediate nodes of long-token chunk chains

enum : int { RC_RANGES = 0, RC_OVERFLOW = 1, RC_ERROR = 2, RC_COUNT = 4 };

struct RMatchParams {
    const RNode* nodes;
    const Slot* slots;
    const uint4* tags;
    uint32_t n_blocks;
    const uint8_t* filters;
    const int64_t* filter_off;
    const int32_t* filter_tenant;
    const int32_t* tenant_root;     // BFS id of the tenant's root or -1
    int64_t n_filters;
    const uint32_t* work_list;
    int64_t n_work;
    uint32_t* span_begin;
    uint32_t* span_count;
    unsigned long long* total;      // [n] matches before the limit
    uint2* ranges;
    uint64_t ranges_cap;
    uint32_t* overflow_list;
    unsigned long long* counters;
    uint2* scratch;
    uint64_t scratch_frontier_cap, scratch_ranges_cap;
};

constexpr int R_WARPS = 8;
constexpr int R_STAGE = 256;
constexpr uint32_t R_FR_CAP = 64, R_RG_CAP = 64;
constexpr unsigned RFULL = 0xFFFFFFFFu;
constexpr uint32_t SPAN_OVF = 0x40000000u;

struct RWarpSmem {
    uint8_t stage[R_STAGE];
    uint32_t keyw[8];
    uint2 fr[2][R_FR_CAP];   // frontier: intervals {first id, count}
    uint2 rg[R_RG_CAP];
};

__device__ __forceinline__ RNode load_node(const RNode* n) {
    const uint4* p = reinterpret_cast<const uint4*>(n);
    uint4 a = __ldg(p), b = __ldg(p + 1);
    RNode r;
    r.child_begin = a.x; r.child_count = a.y; r.sub_begin = a.z; r.sub_end = a.w;
    r.own_prefix = b.x; r.sys_begin = b.y; r.sys_count = b.z; r.pad = b.w;
    return r;
}

// (parent, lenw, k) -> child id, or NONE; *nd = the child's record (without its '$' run), *own_next = own_prefix of the node
// behind it — both carried in the slot's payload half (see build_tenant)
__device__ __forceinline__ uint32_t rprobe(const Slot* slots, const uint4* tags, uint32_t n_blocks, uint32_t parent, uint32_t lenw,
                                           const uint32_t (&k)[6], uint64_t tokh, RNode* nd, uint32_t* own_next) {
    uint32_t w[16], slot = 0;
    if (!probe(slots, tags, n_blocks, parent, lenw, k, tokh, w, slot)) return NONE;
    nd->child_begin = w[9]; nd->child_count = w[10]; nd->sub_begin = w[11]; nd->sub_end = w[12];
    nd->own_prefix = w[13]; nd->sys_begin = 0; nd->sys_count = 0; nd->pad = 0;
    *own_next = w[14];
    return w[W_PLUS];
}

template <bool kBig>
__device__ __forceinline__ void rmatch_one(const RMatchParams& p, RWarpSmem& ws, uint32_t f, int lane, uint2* fr_a, uint2* fr_b,
                                           uint2* rg, uint32_t capF, uint32_t capR) {
    const int64_t fb = p.filter_off[f];
    const int len = (int) (p.filter_off[f + 1] - fb);
    const uint8_t* src = p.filters + fb;
    const bool staged = len <= R_STAGE;
    __syncwarp();
    if (staged)
        for (int i = lane; i < len; i += 32) ws.stage[i] = src[i];
    __syncwarp();
    auto byte_at = [&](int i) -> uint32_t { return staged ? (uint32_t) ws.stage[i] : (uint32_t) src[i]; };

    const int root = p.tenant_root[p.filter_tenant[f]];
    uint32_t n_rg = 0;
    unsigned long long total = 0;   // lane-local, reduced at the end
    bool overflow = false;
    auto emit = [&](bool valid, uint32_t first, uint32_t count) {
        valid = valid && count > 0;
        const unsigned m = __ballot_sync(RFULL, valid);
        if (m == 0) return;
        if (valid) {
            const uint32_t idx = n_rg + __popc(m & ((1u << lane) - 1));
            if (idx < capR) rg[idx] = make_uint2(first, count);
            total += count;
        }
        n_rg += __popc(m);
        if (n_rg > capR) overflow = true;
    };
    // append intervals to the next frontier (one optional interval per lane)
    uint2* fr_cur = fr_a;
    uint2* fr_next = fr_b;
    uint32_t n_fr = 0, n_next = 0;
    auto push = [&](bool valid, uint32_t first, uint32_t count) {
        valid = valid && count > 0;
        const unsigned m = __ballot_sync(RFULL, valid);
        if (m == 0) return;
        if (valid) {
            const uint32_t idx = n_next + __popc(m & ((1u << lane) - 1));
            if (idx < capF) fr_next[idx] = make_uint2(first, count);
        }
        n_next += __popc(m);
        if (n_next > capF) overflow = true;
    };

    // Visits every NODE of every frontier interval, 32 nodes per round, one per lane: the intervals of a block of 32 are
    // flattened with a warp scan and each lane finds its (interval, offset) with a 5-step search over the scanned prefixes.
    // (Round 1 gave each lane one INTERVAL and walked it sequentially: after a '+' level the frontier is ONE interval of
    // hundreds of nodes, so one lane did hundreds of dependent probes while 31 idled.) fn(alive, node) is called by the whole
    // warp in lock step: it may use warp collectives.
    auto for_each_frontier_node = [&](auto&& fn) {
        for (uint32_t base = 0; base < n_fr && !overflow; base += 32) {
            const bool act = base + lane < n_fr;
            const uint2 iv = act ? fr_cur[base + lane] : make_uint2(0u, 0u);
            uint32_t inc = iv.y;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(RFULL, inc, o);
                if (lane >= o) inc += y;
            }
            const uint32_t pre = inc - iv.y, tot = __shfl_sync(RFULL, inc, 31);
            for (uint32_t t0 = 0; t0 < tot && !overflow; t0 += 32) {
                const uint32_t g = t0 + lane;
                int lo = 0, hi = 32;
#pragma unroll
                for (int it = 0; it < 5; it++) {   // largest lane whose exclusive prefix is <= g (prefixes are non-decreasing)
                    const int mid = (lo + hi) >> 1;
                    const uint32_t pm = __shfl_sync(RFULL, pre, mid);
                    if (pm <= g) lo = mid;
                    else hi = mid;
                }
                const uint32_t ix = __shfl_sync(RFULL, iv.x, lo), ip = __shfl_sync(RFULL, pre, lo);
                fn(g < tot, ix + (g - ip));
            }
        }
    };

    if (root >= 0) {
        if (lane == 0) fr_cur[0] = make_uint2((uint32_t) root, 1u);
        n_fr = 1;
        int pos = 0;
        int level = 0;
        while (n_fr > 0 && !overflow) {
            int e = len;
            for (int b = pos; b < len; b += 32) {
                const int i = b + lane;
                const unsigned m = __ballot_sync(RFULL, i < len && byte_at(i) == '/');
                if (m) {
                    e = b + __ffs(m) - 1;
                    break;
                }
            }
            const bool last = e == len;
            const int tlen = e - pos;
            const uint32_t c0 = tlen >= 1 ? byte_at(pos) : 0u;
            const bool is_plus = tlen == 1 && c0 == '+';
            const bool is_hash = last && tlen == 1 && c0 == '#';
            // does "/#" follow this level as the final level?  (matchParent of the reference selectors)
            bool hash_next = false;
            if (!last && e + 2 == len) hash_next = byte_at(e + 1) == '#';
            n_next = 0;
            __syncwarp();
            if (is_hash) {
                // '#': every child subtree of every frontier node. At level 0 the '$' children are skipped.
                for (uint32_t base = 0; base < n_fr && !overflow; base += 32) {
                    const bool act = base + lane < n_fr;
                    const uint2 iv = act ? fr_cur[base + lane] : make_uint2(0u, 0u);
                    // an interval of frontier nodes: emit per node (subtrees of different parents are not adjacent in DFS rank)
                    // intervals are short here except after '+' levels; lanes walk their interval sequentially
                    for (uint32_t j = 0; __any_sync(RFULL, act && j < iv.y); j++) {
                        const bool a2 = act && j < iv.y;
                        RNode nd{};
                        if (a2) nd = load_node(p.nodes + iv.x + j);
                        if (level == 0) {
                            // children subtrees minus the '$' run: [first child .. sys) and (sys .. last child]
                            RNode s0{}, s1{};
                            const bool has_sys = a2 && nd.sys_count > 0;
                            if (has_sys) {
                                s0 = load_node(p.nodes + nd.sys_begin);
                                s1 = load_node(p.nodes + nd.sys_begin + nd.sys_count - 1);
                            }
                            const uint32_t own = a2 ? (load_node(p.nodes + iv.x + j + 1).own_prefix - nd.own_prefix) : 0u;
                            const uint32_t lo = nd.sub_begin + own;
                            emit(a2 && !has_sys, lo, nd.sub_end - lo);
                            emit(has_sys, lo, s0.sub_begin - lo);
                            emit(has_sys, s1.sub_end, nd.sub_end - s1.sub_end);
                        } else {
                            // reached through "x/#" handling below, never here: kept for completeness
                            emit(a2, nd.sub_begin, nd.sub_end - nd.sub_begin);
                        }
                    }
                }
                break;
            }
            if (is_plus) {
                for (uint32_t base = 0; base < n_fr && !overflow; base += 32) {
                    const bool act = base + lane < n_fr;
                    const uint2 iv = act ? fr_cur[base + lane] : make_uint2(0u, 0u);
                    RNode n0{}, n1{};
                    if (act) {
                        n0 = load_node(p.nodes + iv.x);
                        n1 = iv.y > 1 ? load_node(p.nodes + iv.x + iv.y - 1) : n0;
                    }
                    // children of the whole interval = [first child of the first node, last child of the last node]
                    uint32_t cb = n0.child_begin, ce = n1.child_begin + n1.child_count;
                    // level 0: the frontier is the single tenant root; skip its '$' children
                    const bool split = act && level == 0 && n0.sys_count > 0;
                    const uint32_t sb = n0.sys_begin, se = n0.sys_begin + n0.sys_count;
                    if (last) {
                        // MATCH_AND_STOP on every child: the topics ending exactly at those nodes = one BFS-rank range
                        uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;
                        if (act && ce > cb) {
                            o0 = load_node(p.nodes + cb).own_prefix;
                            o3 = load_node(p.nodes + ce).own_prefix;
                            if (split) {
                                o1 = load_node(p.nodes + sb).own_prefix;
                                o2 = load_node(p.nodes + se).own_prefix;
                            }
                        }
                        emit(act && !split, SPACE_BFS | o0, o3 - o0);
                        emit(split, SPACE_BFS | o0, o1 - o0);
                        emit(split, SPACE_BFS | o2, o3 - o2);
                    } else if (hash_next) {
                        // "+/#": handled below, per frontier NODE
                    } else {
                        push(act && !split, cb, ce - cb);
                        push(split, cb, sb - cb);
                        push(split, se, ce - se);
                    }
                }
                if (hash_next && !last) {
                    // "+/#": whole subtrees of all children; per frontier node one DFS range (minus its own topic)
                    for_each_frontier_node([&](bool a2, uint32_t id) {
                        RNode nd{};
                        uint32_t own = 0;
                        if (a2) {
                            nd = load_node(p.nodes + id);
                            own = load_node(p.nodes + id + 1).own_prefix - nd.own_prefix;
                        }
                        const uint32_t lo = nd.sub_begin + own;
                        const bool sp = a2 && level == 0 && nd.sys_count > 0;
                        RNode s0{}, s1{};
                        if (sp) {
                            s0 = load_node(p.nodes + nd.sys_begin);
                            s1 = load_node(p.nodes + nd.sys_begin + nd.sys_count - 1);
                        }
                        emit(a2 && !sp, lo, nd.sub_end - lo);
                        emit(sp, lo, s0.sub_begin - lo);
                        emit(sp, s1.sub_end, nd.sub_end - s1.sub_end);
                    });
                }
                if (last || hash_next) break;
            } else {
                // exact level: probe every node of every frontier interval
                const int nchunks = tlen <= (int) TOKEN_BYTES ? 1 : (tlen + (int) TOKEN_BYTES - 1) / (int) TOKEN_BYTES;
                for_each_frontier_node([&](bool alive, uint32_t node) {
                    RNode cnd{};
                    uint32_t own_next = 0;
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
                        for (int q = 0; q < 6; q++) k[q] = ws.keyw[q];
                        const uint64_t tokh = token_hash(lenw, k);
                        if (alive) {
                            node = rprobe(p.slots, p.tags, p.n_blocks, node, lenw, k, tokh, &cnd, &own_next);
                            alive = node != NONE;
                        }
                    }
                    if (last) {
                        emit(alive, SPACE_BFS | cnd.own_prefix, own_next - cnd.own_prefix);
                    } else if (hash_next) {
                        emit(alive, cnd.sub_begin, cnd.sub_end - cnd.sub_begin);   // "x/#": x itself and everything below
                    } else {
                        push(alive, node, 1u);
                    }
                });
                if (last || hash_next) break;
            }
            __syncwarp();
            uint2* tmp = fr_cur;
            fr_cur = fr_next;
            fr_next = tmp;
            n_fr = n_next;
            pos = e + 1;
            level++;
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(RFULL, total, o);
    __syncwarp();
    if (overflow) {
        if (lane == 0) {
            if (!kBig) {
                const unsigned long long idx = atomicAdd(&p.counters[RC_OVERFLOW], 1ull);
                p.overflow_list[idx] = f;
                p.span_count[f] = SPAN_OVF;
            } else {
                atomicAdd(&p.counters[RC_ERROR], 1ull);
                p.span_count[f] = 0;
            }
            p.span_begin[f] = 0;
            p.total[f] = 0;
        }
        return;
    }
    unsigned long long base = 0;
    if (n_rg > 0) {
        if (lane == 0) base = atomicAdd(&p.counters[RC_RANGES], (unsigned long long) n_rg);
        base = __shfl_sync(RFULL, base, 0);
        if (base + n_rg <= p.ranges_cap)
            for (uint32_t i = lane; i < n_rg; i += 32) p.ranges[base + i] = rg[i];
    }
    if (lane == 0) {
        p.span_begin[f] = (uint32_t) base;
        p.span_count[f] = n_rg;
        p.total[f] = total;
    }
}

template <bool kBig>
__global__ void __launch_bounds__(R_WARPS * 32, 5) rmatch_kernel(const RMatchParams p) {
    __shared__ RWarpSmem sm[R_WARPS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    RWarpSmem& ws = sm[wid];
    const int64_t gw = (int64_t) blockIdx.x * R_WARPS + wid, nw = (int64_t) gridDim.x * R_WARPS;
    if (kBig) {
        uint2* basep = p.scratch + (uint64_t) gw * (2 * p.scratch_frontier_cap + p.scratch_ranges_cap);
        for (int64_t it = gw; it < p.n_work; it += nw)
            rmatch_one<true>(p, ws, p.work_list[it], lane, basep, basep + p.scratch_frontier_cap, basep + 2 * p.scratch_frontier_cap,
                             (uint32_t) min((uint64_t) 0x3FFFFFFFull, p.scratch_frontier_cap),
                             (uint32_t) min((uint64_t) 0x3FFFFFFFull, p.scratch_ranges_cap));
    } else {
        // p.work_list here = the locality order of the batch (filters grouped by tenant and leading levels), or nullptr
        for (int64_t it = gw; it < p.n_filters; it += nw)
            rmatch_one<false>(p, ws, p.work_list ? p.work_list[it] : (uint32_t) it, lane, ws.fr[0], ws.fr[1], ws.rg, R_FR_CAP, R_RG_CAP);
    }
}

// kept[i] = min(total[i], limit[i])
__global__ void rkept_kernel(int64_t n, const unsigned long long* total, const int64_t* limit, unsigned long long* kept) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const unsigned long long t = total[i];
        const long long l = limit ? limit[i] : -1;
        kept[i] = l < 0 ? t : (t < (unsigned long long) l ? t : (unsigned long long) l);
    }
}

// one warp per filter: map its ranges to topic ids, first `kept` of them
__global__ void __launch_bounds__(256) rexpand_kernel(int64_t n, const uint32_t* span_begin, const uint32_t* span_count,
                                                      const uint2* ranges, const unsigned long long* offsets,
                                                      const unsigned long long* kept, const int64_t* dfs_to_id,
                                                      const int64_t* bfs_to_id, int64_t* ids) {
    const int lane = threadIdx.x & 31;
    const int64_t f = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (f >= n) return;
    const unsigned long long out0 = offsets[f], want = kept[f];
    unsigned long long done = 0;
    const uint32_t b = span_begin[f], c = span_count[f];
    for (uint32_t j = 0; j < c && done < want; j++) {
        const uint2 r = ranges[b + j];
        const bool bfs = r.x & SPACE_BFS;
        const uint32_t first = r.x & ~SPACE_BFS;
        const unsigned long long take = min((unsigned long long) r.y, want - done);
        const int64_t* map = bfs ? bfs_to_id : dfs_to_id;
        for (unsigned long long x = lane; x < take; x += 32) ids[out0 + done + x] = map[first + x];
        done += take;
    }
}

// Inserts the exact edges of the regions a delta commit appended into the live tag table, one thread per edge. img[i] is the
// finished 64-byte slot (key words 0..7, payload 8..15). The probe sequence is EdgeTable::place's: the first free tag of the
// 15 usable ones in the home block, else mark the block overflowed (control byte) and go on to the next block. A tag byte is
// claimed with atomicCAS on its 32-bit tag word, retried while other threads change that word. The caller keeps the table
// below full (the occupancy bound of the delta path), so every thread finds a free slot.
__global__ void __launch_bounds__(256) rinsert_edges_kernel(const Slot* __restrict__ img, int64_t n, Slot* slots, uint32_t* tags,
                                                            uint32_t n_blocks, unsigned long long* overflowed) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint4* src = reinterpret_cast<const uint4*>(img + i);
    const uint4 a = src[0], b = src[1];
    const uint32_t k[6] = {a.z, a.w, b.x, b.y, b.z, b.w};
    const uint64_t h = edge_hash(token_hash(a.y, k), a.x);
    const uint32_t fp = fingerprint(h);
    uint32_t blk = home_block(h, n_blocks);
    while (true) {
        uint32_t* tw = tags + (size_t) blk * 4;
        for (int q = 0; q < 4; q++) {
            const int bytes = q == 3 ? 3 : 4;   // byte 15 of the block is the control byte
            uint32_t cur = *reinterpret_cast<volatile uint32_t*>(tw + q);
            while (true) {
                int j = -1;
                for (int t = 0; t < bytes; t++)
                    if (((cur >> (8 * t)) & 0xFFu) == 0) {
                        j = t;
                        break;
                    }
                if (j < 0) break;
                const uint32_t old = atomicCAS(tw + q, cur, cur | (fp << (8 * j)));
                if (old == cur) {
                    uint4* dst = reinterpret_cast<uint4*>(slots + (size_t) blk * BLOCK_SLOTS + (uint32_t) (q * 4 + j));
                    dst[0] = a;
                    dst[1] = b;
                    dst[2] = src[2];
                    dst[3] = src[3];
                    return;
                }
                cur = old;
            }
        }
        if ((atomicOr(tw + 3, 1u << 24) >> 24) == 0) atomicAdd(overflowed, 1ull);
        blk = blk + 1 == n_blocks ? 0 : blk + 1;
    }
}

// *bad = 1 if some filter_tenant of a device-resident batch lies outside [0, n_tenants): the match kernel indexes the tenant
// table with it, so the call fails before that kernel runs
__global__ void rcheck_tenants_kernel(int64_t n, const int32_t* filter_tenant, int32_t n_tenants, unsigned long long* bad) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && (filter_tenant[i] < 0 || filter_tenant[i] >= n_tenants)) *bad = 1;
}

// len[i] = length of the retain key of ids[i] (key_off: the id table's device key offsets)
__global__ void rkey_len_kernel(int64_t n, const int64_t* ids, const int64_t* key_off, int64_t* len) {
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const int64_t id = ids[i];
        len[i] = key_off[id + 1] - key_off[id];
    }
}

// one warp per id: its retain key to out[out_off[i] ..)
__global__ void __launch_bounds__(256) rkey_copy_kernel(int64_t n, const int64_t* ids, const int64_t* key_off,
                                                        const uint8_t* key_bytes, const int64_t* out_off, uint8_t* out) {
    const int lane = threadIdx.x & 31;
    const int64_t i = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (i >= n) return;
    const int64_t id = ids[i];
    const int64_t b = key_off[id], len = key_off[id + 1] - b;
    const uint8_t* src = key_bytes + b;
    uint8_t* dst = out + out_off[i];
    for (int64_t x = lane; x < len; x += 32) dst[x] = src[x];
}

}  // namespace

// The retain keys of an id table on the device: key i is bytes[off[i] .. off[i + 1]). Buffers that must grow are replaced, not
// reallocated: a gather still running on another stream keeps reading the old ones, which its result holds until released.
struct KeyBufs {
    int device = 0;
    DeviceBuf<uint8_t> bytes;
    DeviceBuf<int64_t> off;
    ~KeyBufs() { cudaSetDevice(device); }   // runs before the members are destroyed: the buffers are freed on this device
};

// id -> (tenant, topic); tombstones keep their slot. bfq_rindex_reset starts a new table, so ids restart at 0 there while the
// snapshot and its results still name ids of the old one. Append-only: add / load_keys push_back under the handle lock held
// exclusive, and every host reader of `e` (a match's result, key calls, lookup) holds it shared, so no reader sees a
// reallocation. The device key table belongs to the id table and goes with it.
struct IdTable {
    std::vector<std::pair<std::string, std::string>> e;
    std::mutex key_mu;                    // the key table below
    std::shared_ptr<KeyBufs> keys;        // built on the first key call, extended for ids added since
    int64_t key_ids = 0, key_bytes = 0;   // ids and bytes it holds
    std::atomic<int64_t> key_device_bytes{0};
};

struct bfq_rresult {
    std::vector<int64_t> offsets, ids, totals;
    double ms[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint64_t generation = 0;
    std::shared_ptr<IdTable> by_id;   // the id table of the snapshot the match ran on
};

// Everything ONE inverse match in flight needs: its stream, device scratch and outputs, pinned counters. Leased from the
// handle's pool for a call, and for a device result until bfq_rdevice_result_release (its arrays live here), so concurrent
// matches on one handle never share a buffer.
struct RWorkspace {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};   // [0,1] around all kernels of a match, [2,3] around rmatch_kernel
    cudaEvent_t ev_in = nullptr;        // device path: recorded on the caller's stream, where the batch was written
    std::vector<cudaEvent_t> ev_use;    // device result: one per stream a key gather ran on (RLease::used_on), created on demand
    std::atomic<int64_t> bytes_held{0}; // device_bytes() when the last call on it ended (bfq_rindex_stats)
    DeviceBuf<uint8_t> d_in, d_scan_tmp, d_key_tmp;   // d_in: the host path's batch, one block
    PinnedBuf<int32_t> h_tenant_root;
    PinnedBuf<unsigned long long> h_small;   // [0, RC_COUNT) the match counters, [RC_COUNT] a total read back
    DeviceBuf<int64_t> d_ids, d_key_len;
    DeviceBuf<int32_t> d_tenant_root;
    DeviceBuf<uint32_t> d_span_begin, d_span_count, d_overflow;
    DeviceBuf<unsigned long long> d_total, d_kept, d_offsets, d_counters;
    DeviceBuf<uint2> d_ranges, d_scratch;
    // locality order of a batch of filters (match_kernels.cu: launch_order, without de-duplication)
    DeviceBuf<uint32_t> d_ord_keys, d_ord_leader, d_order, d_hist;
    DeviceBuf<unsigned long long> d_ord_ctr;

    cudaError_t init(int dev) {
        device = dev;
        cudaError_t e = cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking);
        for (auto& x : ev)
            if (e == cudaSuccess) e = cudaEventCreate(&x);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ev_in, cudaEventDisableTiming);
        return e;
    }
    int64_t device_bytes() const {
        return (int64_t) (d_in.bytes() + d_scan_tmp.bytes() + d_key_tmp.bytes() + d_ids.bytes() + d_key_len.bytes() +
                          d_tenant_root.bytes() + d_span_begin.bytes() + d_span_count.bytes() + d_overflow.bytes() +
                          d_total.bytes() + d_kept.bytes() + d_offsets.bytes() + d_counters.bytes() + d_ranges.bytes() +
                          d_scratch.bytes() + d_ord_keys.bytes() + d_ord_leader.bytes() + d_order.bytes() + d_hist.bytes() +
                          d_ord_ctr.bytes());
    }
    ~RWorkspace() {
        cudaSetDevice(device);   // the buffers are freed after this body, on this device
        for (auto& e : ev) if (e) cudaEventDestroy(e);
        if (ev_in) cudaEventDestroy(ev_in);
        for (auto& e : ev_use) cudaEventDestroy(e);
        if (stream) cudaStreamDestroy(stream);
    }
};

// the workspaces of one handle. Shared with every device result in flight, so that releasing a result after its handle was
// destroyed still has a place to return its workspace to.
struct RPool {
    std::mutex mu;
    std::vector<RWorkspace*> idle;
    std::vector<RWorkspace*> held;   // every workspace alive: idle and leased
    int device = 0;
    bool closed = false;
    ~RPool() {
        cudaSetDevice(device);
        for (RWorkspace* w : idle) delete w;
    }
};

// a device result (bfq_rmatch_device .. bfq_rdevice_result_release)
struct RLease {
    bfq_rindex* h = nullptr;
    std::shared_ptr<RPool> pool;
    RWorkspace* ws = nullptr;
    std::shared_ptr<IdTable> by_id;   // the id table of the snapshot the match ran on
    std::mutex use_mu;                // key gathers on this result, one at a time (they share the workspace's scratch)
    std::vector<cudaStream_t> used_on;              // ws->ev_use[i]: the last gather on used_on[i]
    std::vector<std::shared_ptr<KeyBufs>> keys;     // key buffers the gathers read, held until release
};

// where a live tenant's trie sits in the snapshot (see the layout comment above rebuild_full)
struct TenantRegion {
    uint32_t root = 0;      // node id of the root = first node of the region
    uint32_t n_nodes = 0;
    int64_t n_topics = 0;
};

struct bfq_rindex {
    int device = 0;
    // Matches hold it shared from reading the snapshot's tables until their device reads of them have finished (a commit
    // patches the device tables in place); add / load_keys / remove / reset / commit hold it exclusive.
    std::shared_mutex mu;
    std::mutex gate;   // a writer holds it while it waits for and holds mu: matches arriving meanwhile queue behind it
    cudaStream_t stream = nullptr;   // commits
    std::shared_ptr<RPool> pool = std::make_shared<RPool>();
    // staging: (tenant, topic) -> id ; id -> (tenant, topic)
    std::map<std::pair<std::string, std::string>, int64_t> staged;
    std::shared_ptr<IdTable> by_id = std::make_shared<IdTable>();   // staging: add / load_keys append here
    std::vector<char> alive;
    std::set<std::string> dirty;   // tenants whose staged topic set changed since the last commit
    bool need_full = true;         // the next commit is a full build (no snapshot yet, reset, bulk load onto an empty handle)
    bool have_snapshot = false;
    uint64_t generation = 0;       // successful commits so far: the snapshot's generation
    std::shared_ptr<IdTable> committed;   // the table by_id was when the snapshot was built (append-only since)
    // snapshot
    std::unordered_map<std::string, int32_t> tenant_root;
    std::unordered_map<std::string, TenantRegion> regions;   // the live tenants' regions
    uint32_t n_blocks = 0;
    int64_t n_nodes = 0, max_nodes_per_depth = 0, n_topics = 0;   // n_nodes: records of every region, garbage included
    int64_t n_dfs = 0, n_bfs = 0;          // DFS / BFS ranks handed out, garbage included
    uint32_t next_virtual = 0;             // next free id of a long-name chunk node
    int64_t garbage_nodes = 0;             // records of replaced regions and vanished tenants
    int64_t used_slots = 0;                // occupied table slots, garbage included
    int64_t overflowed_blocks = 0;
    int64_t full_commits = 0, delta_commits = 0, last_rebuilt = 0;
    DeviceBuf<RNode> d_nodes;
    DeviceBuf<Slot> d_slots;
    DeviceBuf<uint8_t> d_tags;
    DeviceBuf<int64_t> d_dfs_to_id, d_bfs_to_id;
    DeviceBuf<Slot> d_new_slots;                // slot images of a delta commit
    DeviceBuf<unsigned long long> d_ins_ctr;
    std::atomic<int64_t> launches{0};

    int64_t snapshot_bytes() const {
        return (int64_t) (d_nodes.bytes() + d_slots.bytes() + d_tags.bytes() + d_dfs_to_id.bytes() + d_bfs_to_id.bytes() +
                          d_new_slots.bytes() + d_ins_ctr.bytes());
    }

    ~bfq_rindex() {
        cudaSetDevice(device);   // the buffers are freed after this body, on this device
        std::vector<RWorkspace*> idle;
        {
            std::lock_guard<std::mutex> g(pool->mu);
            pool->closed = true;   // workspaces still leased are freed when they come back
            idle.swap(pool->idle);
            pool->held.clear();
        }
        for (RWorkspace* w : idle) delete w;
        if (stream) cudaStreamDestroy(stream);
    }
};

namespace {

// The handle lock for matches and for writers. std::shared_mutex lets new readers in while a writer waits, so a steady stream
// of matches could hold a commit off indefinitely; the gate makes matches that arrive after a waiting writer wait behind it.
std::shared_lock<std::shared_mutex> read_lock(bfq_rindex* h) {
    { std::lock_guard<std::mutex> wait_for_writers(h->gate); }
    return std::shared_lock<std::shared_mutex>(h->mu);
}
struct WriteLock {
    std::lock_guard<std::mutex> gate;
    std::unique_lock<std::shared_mutex> g;
    explicit WriteLock(bfq_rindex* h) : gate(h->gate), g(h->mu) {}
};

struct HNode {  // host build node
    std::map<std::string, uint32_t> children;   // name -> host node index (sorted => '$' children form one run)
    int64_t own = -1;                           // topic id ending here
    uint32_t bfs = 0;
};

inline void make_tok(sv chunk, uint32_t* tok) {
    for (uint32_t k = 0; k < TOKEN_WORDS; k++) tok[k] = 0;
    for (size_t j = 0; j < chunk.size(); j++) tok[j >> 2] |= (uint32_t) (uint8_t) chunk[j] << (8 * (j & 3));
}

using Staged = std::map<std::pair<std::string, std::string>, int64_t>;

// Snapshot layout. Every live tenant owns one REGION of consecutive node ids: its root first, then its trie in BFS order from
// that root (level by level, children in bytewise name order, so the '$' children of a node are one run). Its topics get
// consecutive DFS ranks (pre-order, own topic first) and consecutive BFS ranks (by the id of the node they end at). A full build
// places the regions back to back in bytewise tenant order; a delta commit appends the rebuilt tenants' regions behind all
// existing ones, and the regions they replace (and those of tenants that vanished) stay in place as garbage that no tenant root
// reaches, until the next full build. The kernels rely on these invariants, which deltas keep:
//   * BFS ranks are assigned in node-id order over the whole array, garbage regions included, so own_prefix is monotone;
//   * the record after a region's last node carries that region's rank end in own_prefix: it is the next region's root, or
//     the one sentinel record at [n_nodes], which is rewritten on every append;
//   * node ids stay below VIRT_BASE, ranks below SPACE_BFS, and long-name chunk ids between VIRT_BASE and NONE.
// Within a region this is exactly the layout of one tenant in a single global BFS, so answers (ids and their order), range
// counts and tier hand-offs do not depend on where a tenant's region sits.
struct TenantImage {
    std::vector<RNode> rn;                    // the region's records, node_base.. (no sentinel)
    std::vector<int64_t> dfs_to_id, bfs_to_id;
    std::vector<Slot> slots;                  // the region's exact edges as finished slot images
    int64_t max_depth_nodes = 0;              // the largest number of the tenant's nodes at one depth
    uint32_t n_virtual = 0;                   // chunk-node ids used from virt_base on
};

constexpr uint64_t ID_LIMIT = 0x7FFFFFF0ull;     // node ids and ranks stay below this (VIRT_BASE / SPACE_BFS)
constexpr uint64_t VIRT_LIMIT = 0xFFFFFFF0ull;   // chunk-node ids stay below this (NONE / EMPTY_PARENT)

// The trie of one tenant's topics [first, last) of the staging map, with node ids from node_base, DFS ranks from dfs_base,
// BFS ranks from bfs_base and chunk-node ids from virt_base.
int32_t build_tenant(Staged::const_iterator first, Staged::const_iterator last, uint32_t node_base, uint32_t dfs_base,
                     uint32_t bfs_base, uint32_t virt_base, TenantImage* out) {
    std::vector<HNode> nodes(1);
    for (auto it = first; it != last; ++it) {
        uint32_t cur = 0;
        for_each_level(sv(it->first.second), '/', [&](sv l) {
            auto c = nodes[cur].children.find(std::string(l));
            if (c == nodes[cur].children.end()) {
                nodes.emplace_back();
                uint32_t idx = (uint32_t) nodes.size() - 1;
                nodes[cur].children.emplace(std::string(l), idx);
                cur = idx;
            } else {
                cur = c->second;
            }
        });
        nodes[cur].own = it->second;
    }
    const size_t N = nodes.size();
    if (N >= ID_LIMIT) return fail(BFQ_E_RANGE, "topic index too large");
    // ---- BFS numbering from the root, level by level in parent order
    std::vector<uint32_t> order;
    order.reserve(N);
    order.push_back(0);
    int64_t max_depth_nodes = 1;
    for (size_t lo = 0, hi = order.size(); lo < hi;) {
        for (size_t i = lo; i < hi; i++)
            for (const auto& c : nodes[order[i]].children) order.push_back(c.second);
        lo = hi;
        hi = order.size();
        max_depth_nodes = std::max<int64_t>(max_depth_nodes, (int64_t) (hi - lo));
    }
    for (size_t i = 0; i < N; i++) nodes[order[i]].bfs = (uint32_t) i;
    TenantImage& im = *out;
    im.rn.assign(N, RNode{});
    im.max_depth_nodes = max_depth_nodes;
    std::vector<RNode>& rn = im.rn;
    std::vector<int64_t>& bfs_to_id = im.bfs_to_id;
    std::vector<int64_t>& dfs_to_id = im.dfs_to_id;
    // child intervals + BFS topic ranks
    {
        uint32_t next_child = node_base + 1;
        for (size_t i = 0; i < N; i++) {
            const HNode& hn = nodes[order[i]];
            RNode& r = rn[i];
            r.child_begin = next_child;
            r.child_count = (uint32_t) hn.children.size();
            next_child += r.child_count;
            r.own_prefix = bfs_base + (uint32_t) bfs_to_id.size();
            if (hn.own >= 0) bfs_to_id.push_back(hn.own);
            uint32_t k = 0;
            for (const auto& c : hn.children) {
                if (!c.first.empty() && c.first[0] == '$') {
                    if (r.sys_count == 0) r.sys_begin = r.child_begin + k;
                    r.sys_count++;
                }
                k++;
            }
        }
    }
    const uint32_t rank_end = bfs_base + (uint32_t) bfs_to_id.size();   // own_prefix of the record behind the region
    // DFS (pre-order) topic ranks, iterative
    {
        std::vector<std::pair<uint32_t, std::map<std::string, uint32_t>::const_iterator>> st;
        rn[0].sub_begin = dfs_base;
        if (nodes[0].own >= 0) dfs_to_id.push_back(nodes[0].own);
        st.push_back({0u, nodes[0].children.begin()});
        while (!st.empty()) {
            auto& top = st.back();
            if (top.second == nodes[top.first].children.end()) {
                rn[nodes[top.first].bfs].sub_end = dfs_base + (uint32_t) dfs_to_id.size();
                st.pop_back();
                continue;
            }
            uint32_t c = top.second->second;
            ++top.second;
            rn[nodes[c].bfs].sub_begin = dfs_base + (uint32_t) dfs_to_id.size();
            if (nodes[c].own >= 0) dfs_to_id.push_back(nodes[c].own);
            st.push_back({c, nodes[c].children.begin()});
        }
    }
    // ---- exact edges keyed by the parent's node id (long names: chains of virtual nodes)
    auto slot_of = [](uint32_t parent, uint32_t lenw, sv chunk, uint32_t child) {
        Slot s{};
        s.w[W_PARENT] = parent;
        s.w[W_LEN] = lenw;
        make_tok(chunk, &s.w[W_TOK]);
        s.w[W_PLUS] = child;
        return s;
    };
    std::vector<Slot>& slots = im.slots;
    slots.reserve(N);
    uint64_t next_virtual = virt_base;
    std::map<std::tuple<uint32_t, uint32_t, std::string>, uint32_t> virt;
    for (size_t i = 0; i < N; i++) {
        const HNode& hn = nodes[order[i]];
        for (const auto& c : hn.children) {
            sv name(c.first);
            uint32_t parent = node_base + (uint32_t) i;
            size_t off = 0;
            uint32_t j = 0;
            while (name.size() - off > TOKEN_BYTES) {
                const sv chunk = name.substr(off, TOKEN_BYTES);
                // identical chunk prefixes under the same parent share one virtual node
                auto vk = std::make_tuple(parent, LEN_CONT | j, std::string(chunk));
                auto vit = virt.find(vk);
                if (vit == virt.end()) {
                    if (next_virtual >= VIRT_LIMIT) return fail(BFQ_E_RANGE, "topic index too large");
                    const uint32_t v = (uint32_t) next_virtual++;
                    slots.push_back(slot_of(parent, LEN_CONT | j, chunk, v));
                    virt.emplace(std::move(vk), v);
                    parent = v;
                } else {
                    parent = vit->second;
                }
                off += TOKEN_BYTES;
                j++;
            }
            const uint32_t local = nodes[c.second].bfs;
            Slot s = slot_of(parent, (uint32_t) name.size(), name.substr(off), node_base + local);
            // the child's node record rides in the slot's payload half: an exact step is tag + slot, with no third dependent
            // access for the record (words 9..14: child_begin, child_count, sub_begin, sub_end, own_prefix, own_prefix of the
            // next node; the '$' run is only needed for tenant roots, which are never reached through a slot)
            const RNode& r = rn[local];
            s.w[9] = r.child_begin;
            s.w[10] = r.child_count;
            s.w[11] = r.sub_begin;
            s.w[12] = r.sub_end;
            s.w[13] = r.own_prefix;
            s.w[14] = local + 1 < N ? rn[local + 1].own_prefix : rank_end;
            slots.push_back(s);
        }
    }
    im.n_virtual = (uint32_t) (next_virtual - virt_base);
    return BFQ_OK;
}

template <typename T>
void append(std::vector<T>& a, const std::vector<T>& b) {
    a.insert(a.end(), b.begin(), b.end());
}

// the half-open run of one tenant's topics in the staging map
std::pair<Staged::const_iterator, Staged::const_iterator> tenant_run(const Staged& staged, Staged::const_iterator first) {
    auto last = first;
    while (last != staged.end() && last->first.first == first->first.first) ++last;
    return {first, last};
}

// Full build: build_tenant over every tenant, regions back to back in bytewise tenant order, one fresh tag table.
int32_t rebuild_full(bfq_rindex* h) {
    std::vector<RNode> rn;
    std::vector<int64_t> dfs_to_id, bfs_to_id;
    std::vector<Slot> imgs;
    std::unordered_map<std::string, TenantRegion> regions;
    int64_t max_depth_nodes = 0;
    uint64_t next_virtual = VIRT_BASE;
    for (auto it = h->staged.cbegin(); it != h->staged.cend();) {
        const auto run = tenant_run(h->staged, it);
        TenantImage im;
        const int32_t rc = build_tenant(run.first, run.second, (uint32_t) rn.size(), (uint32_t) dfs_to_id.size(),
                                        (uint32_t) bfs_to_id.size(), (uint32_t) next_virtual, &im);
        if (rc != BFQ_OK) return rc;
        if (rn.size() + im.rn.size() + 1 >= ID_LIMIT || dfs_to_id.size() + im.dfs_to_id.size() >= ID_LIMIT)
            return fail(BFQ_E_RANGE, "topic index too large");
        TenantRegion reg;
        reg.root = (uint32_t) rn.size();
        reg.n_nodes = (uint32_t) im.rn.size();
        reg.n_topics = (int64_t) im.dfs_to_id.size();
        regions.emplace(it->first.first, reg);
        append(rn, im.rn);
        append(dfs_to_id, im.dfs_to_id);
        append(bfs_to_id, im.bfs_to_id);
        append(imgs, im.slots);
        next_virtual += im.n_virtual;
        max_depth_nodes = std::max(max_depth_nodes, im.max_depth_nodes);
        it = run.second;
    }
    const size_t N = rn.size();
    rn.push_back(RNode{(uint32_t) N, 0, 0, 0, (uint32_t) bfs_to_id.size(), 0, 0, 0});   // the sentinel
    if (((uint64_t) imgs.size() * 2 / BLOCK_USABLE + 64) * BLOCK_SLOTS >= ID_LIMIT) return fail(BFQ_E_RANGE, "topic index too large");
    EdgeTable table;
    table.init(imgs.size());
    for (const Slot& s : imgs) table.slots[table.place(s.w[W_PARENT], s.w[W_LEN], &s.w[W_TOK])] = s;
    SlotVec& slots = table.slots;
    // ---- upload
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    BFQ_CUDA_TRY(cudaStreamSynchronize(h->stream));
    h->need_full = true;   // until the upload is complete
    BFQ_CUDA_TRY(h->d_nodes.reserve(rn.size()));
    BFQ_CUDA_TRY(h->d_slots.reserve(slots.size()));
    BFQ_CUDA_TRY(h->d_tags.reserve(table.tags.size()));
    BFQ_CUDA_TRY(h->d_dfs_to_id.reserve(std::max<size_t>(dfs_to_id.size(), 1)));
    BFQ_CUDA_TRY(h->d_bfs_to_id.reserve(std::max<size_t>(bfs_to_id.size(), 1)));
    BFQ_CUDA_TRY(cudaMemcpy(h->d_nodes.p, rn.data(), rn.size() * sizeof(RNode), cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(h->d_slots.p, slots.data(), slots.size() * sizeof(Slot), cudaMemcpyHostToDevice));
    BFQ_CUDA_TRY(cudaMemcpy(h->d_tags.p, table.tags.data(), table.tags.size(), cudaMemcpyHostToDevice));
    if (!dfs_to_id.empty()) {
        BFQ_CUDA_TRY(cudaMemcpy(h->d_dfs_to_id.p, dfs_to_id.data(), dfs_to_id.size() * 8, cudaMemcpyHostToDevice));
        BFQ_CUDA_TRY(cudaMemcpy(h->d_bfs_to_id.p, bfs_to_id.data(), bfs_to_id.size() * 8, cudaMemcpyHostToDevice));
    }
    h->tenant_root.clear();
    for (const auto& e : regions) h->tenant_root[e.first] = (int32_t) e.second.root;
    h->last_rebuilt = (int64_t) regions.size();
    h->regions = std::move(regions);
    h->n_blocks = table.n_blocks;
    h->n_nodes = (int64_t) N;
    h->n_dfs = h->n_topics = (int64_t) dfs_to_id.size();
    h->n_bfs = (int64_t) bfs_to_id.size();
    h->next_virtual = (uint32_t) next_virtual;
    h->max_nodes_per_depth = max_depth_nodes;
    h->garbage_nodes = 0;
    h->used_slots = (int64_t) imgs.size();
    h->overflowed_blocks = table.overflowed_blocks;
    h->full_commits++;
    h->dirty.clear();
    h->need_full = false;
    h->have_snapshot = true;
    return BFQ_OK;
}

// Bounds of the delta path: past them a commit is a full build.
constexpr int64_t GARBAGE_SLACK = 4096;   // garbage nodes may exceed a quarter of the live nodes by this much
constexpr int64_t OCCUPANCY_NUM = 3, OCCUPANCY_DEN = 4;   // occupied table slots, garbage included, <= 3/4 of the usable ones
constexpr int32_t NEED_FULL = 1;

// Delta commit: rebuild only the dirty tenants, each into a fresh region appended behind the existing ones, and insert their
// edges into the live tag table on the device. Returns NEED_FULL (nothing changed) when the commit must be a full build.
int32_t commit_delta(bfq_rindex* h) {
    if (h->need_full || !h->have_snapshot) return NEED_FULL;
    if (h->dirty.empty()) {   // nothing changed: no device work
        h->last_rebuilt = 0;
        return BFQ_OK;
    }
    std::vector<RNode> rn;
    std::vector<int64_t> dfs_to_id, bfs_to_id;
    std::vector<Slot> imgs;
    std::vector<std::pair<std::string, TenantRegion>> fresh;   // rebuilt tenants and their new regions
    std::vector<std::string> gone;                              // tenants whose topics were all removed
    int64_t garbage = h->garbage_nodes, max_depth_nodes = h->max_nodes_per_depth, n_topics = h->n_topics;
    uint64_t next_virtual = h->next_virtual;
    const uint64_t node0 = (uint64_t) h->n_nodes, dfs0 = (uint64_t) h->n_dfs, bfs0 = (uint64_t) h->n_bfs;
    for (const std::string& t : h->dirty) {
        auto old = h->regions.find(t);
        if (old != h->regions.end()) {
            garbage += old->second.n_nodes;
            n_topics -= old->second.n_topics;
        }
        const auto run = tenant_run(h->staged, h->staged.lower_bound({t, std::string()}));
        if (run.first == run.second || run.first->first.first != t) {
            if (old != h->regions.end()) gone.push_back(t);
            continue;
        }
        const uint64_t nb = node0 + rn.size(), db = dfs0 + dfs_to_id.size(), bb = bfs0 + bfs_to_id.size();
        if (nb + 1 >= ID_LIMIT || db >= ID_LIMIT || bb >= ID_LIMIT || next_virtual >= VIRT_LIMIT) return NEED_FULL;
        TenantImage im;
        if (build_tenant(run.first, run.second, (uint32_t) nb, (uint32_t) db, (uint32_t) bb, (uint32_t) next_virtual, &im) != BFQ_OK)
            return NEED_FULL;
        TenantRegion reg;
        reg.root = (uint32_t) nb;
        reg.n_nodes = (uint32_t) im.rn.size();
        reg.n_topics = (int64_t) im.dfs_to_id.size();
        fresh.emplace_back(t, reg);
        n_topics += reg.n_topics;
        append(rn, im.rn);
        append(dfs_to_id, im.dfs_to_id);
        append(bfs_to_id, im.bfs_to_id);
        append(imgs, im.slots);
        next_virtual += im.n_virtual;
        max_depth_nodes = std::max(max_depth_nodes, im.max_depth_nodes);
    }
    const uint64_t n_nodes = node0 + rn.size(), n_dfs = dfs0 + dfs_to_id.size(), n_bfs = bfs0 + bfs_to_id.size();
    if (n_nodes + 1 >= ID_LIMIT || n_dfs >= ID_LIMIT || n_bfs >= ID_LIMIT) return NEED_FULL;
    if (garbage > ((int64_t) n_nodes - garbage) / 4 + GARBAGE_SLACK) return NEED_FULL;
    const int64_t used = h->used_slots + (int64_t) imgs.size();
    if (used * OCCUPANCY_DEN > (int64_t) h->n_blocks * BLOCK_USABLE * OCCUPANCY_NUM) return NEED_FULL;
    // ---- device patch, on the handle's stream, finished before the handle lock is released
    cudaStream_t st = h->stream;
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    h->need_full = true;   // until the patch is complete: a failed patch leaves the device arrays to the next full build
    BFQ_CUDA_TRY(h->d_nodes.grow(n_nodes + 1, node0, st));   // the old sentinel is overwritten by the first appended root
    BFQ_CUDA_TRY(h->d_dfs_to_id.grow(std::max<uint64_t>(n_dfs, 1), dfs0, st));
    BFQ_CUDA_TRY(h->d_bfs_to_id.grow(std::max<uint64_t>(n_bfs, 1), bfs0, st));
    rn.push_back(RNode{(uint32_t) n_nodes, 0, 0, 0, (uint32_t) n_bfs, 0, 0, 0});   // the new sentinel
    BFQ_CUDA_TRY(cudaMemcpyAsync(h->d_nodes.p + node0, rn.data(), rn.size() * sizeof(RNode), cudaMemcpyHostToDevice, st));
    if (!dfs_to_id.empty()) {
        BFQ_CUDA_TRY(cudaMemcpyAsync(h->d_dfs_to_id.p + dfs0, dfs_to_id.data(), dfs_to_id.size() * 8, cudaMemcpyHostToDevice, st));
        BFQ_CUDA_TRY(cudaMemcpyAsync(h->d_bfs_to_id.p + bfs0, bfs_to_id.data(), bfs_to_id.size() * 8, cudaMemcpyHostToDevice, st));
    }
    unsigned long long overflowed = 0;
    if (!imgs.empty()) {
        BFQ_CUDA_TRY(h->d_new_slots.reserve(imgs.size()));
        BFQ_CUDA_TRY(h->d_ins_ctr.reserve(1));
        BFQ_CUDA_TRY(cudaMemcpyAsync(h->d_new_slots.p, imgs.data(), imgs.size() * sizeof(Slot), cudaMemcpyHostToDevice, st));
        BFQ_CUDA_TRY(cudaMemsetAsync(h->d_ins_ctr.p, 0, sizeof(unsigned long long), st));
        const int64_t n = (int64_t) imgs.size();
        rinsert_edges_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(h->d_new_slots.p, n, h->d_slots.p,
                                                                           reinterpret_cast<uint32_t*>(h->d_tags.p), h->n_blocks,
                                                                           h->d_ins_ctr.p);
        h->launches++;
        BFQ_CUDA_TRY(cudaGetLastError());
        BFQ_CUDA_TRY(cudaMemcpyAsync(&overflowed, h->d_ins_ctr.p, sizeof(overflowed), cudaMemcpyDeviceToHost, st));
    }
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    // ---- publish
    for (const std::string& t : gone) {
        h->regions.erase(t);
        h->tenant_root.erase(t);
    }
    for (const auto& f : fresh) {
        h->regions[f.first] = f.second;
        h->tenant_root[f.first] = (int32_t) f.second.root;
    }
    h->n_nodes = (int64_t) n_nodes;
    h->n_dfs = (int64_t) n_dfs;
    h->n_bfs = (int64_t) n_bfs;
    h->n_topics = n_topics;
    h->next_virtual = (uint32_t) next_virtual;
    h->max_nodes_per_depth = max_depth_nodes;
    h->garbage_nodes = garbage;
    h->used_slots = used;
    h->overflowed_blocks += (int64_t) overflowed;
    h->last_rebuilt = (int64_t) fresh.size();
    h->delta_commits++;
    h->dirty.clear();
    h->need_full = false;
    return BFQ_OK;
}

// ------------------------------------------------------------------------------------------------ workspaces
constexpr size_t POOL_KEEP = 4;   // idle workspaces kept for reuse; more are freed when they come back

int32_t acquire(bfq_rindex* h, RWorkspace** out) {
    RPool& pool = *h->pool;
    {
        std::lock_guard<std::mutex> g(pool.mu);
        if (!pool.idle.empty()) {
            *out = pool.idle.back();
            pool.idle.pop_back();
            return BFQ_OK;
        }
    }
    auto* w = new RWorkspace();
    const cudaError_t e = w->init(h->device);
    if (e != cudaSuccess) {
        delete w;
        return fail(BFQ_E_CUDA, std::string("workspace: ") + cudaGetErrorString(e));
    }
    std::lock_guard<std::mutex> g(pool.mu);
    pool.held.push_back(w);
    *out = w;
    return BFQ_OK;
}

// the caller has waited for everything enqueued on w
void give_back(const std::shared_ptr<RPool>& pool, RWorkspace* w) {
    if (!w) return;
    w->bytes_held = w->device_bytes();
    {
        std::lock_guard<std::mutex> g(pool->mu);
        if (!pool->closed && pool->idle.size() < POOL_KEEP) {
            pool->idle.push_back(w);
            return;
        }
        pool->held.erase(std::remove(pool->held.begin(), pool->held.end(), w), pool->held.end());
    }
    cudaSetDevice(pool->device);
    delete w;
}

// a workspace for the length of one call: back to the pool on every return, after its stream has drained
struct CallLease {
    std::shared_ptr<RPool> pool;
    RWorkspace* w = nullptr;
    ~CallLease() {
        if (w) {
            cudaStreamSynchronize(w->stream);
            give_back(pool, w);
        }
    }
};

// ------------------------------------------------------------------------------------------------ retain keys on the device
// Brings the device key table of t up to every id t holds and returns its buffers. The caller holds the handle lock (the ids
// are read here); uploads run on st and are finished on return.
int32_t extend_keys(IdTable& t, int device, cudaStream_t st, std::shared_ptr<KeyBufs>* out) {
    std::lock_guard<std::mutex> g(t.key_mu);
    const int64_t n = (int64_t) t.e.size();
    if (t.keys && t.key_ids == n) {
        *out = t.keys;
        return BFQ_OK;
    }
    std::string blob;
    std::vector<int64_t> ends;   // off[key_ids + 1 .. n]
    ends.reserve((size_t) (n - t.key_ids));
    for (int64_t i = t.key_ids; i < n; i++) {
        blob += make_retain_key(t.e[(size_t) i].first, t.e[(size_t) i].second);
        ends.push_back(t.key_bytes + (int64_t) blob.size());
    }
    const int64_t n_bytes = t.key_bytes + (int64_t) blob.size();
    std::shared_ptr<KeyBufs> kb = t.keys;
    if (!kb || kb->off.cap < (size_t) n + 1 || kb->bytes.cap < (size_t) std::max<int64_t>(n_bytes, 1)) {
        auto nb = std::make_shared<KeyBufs>();
        nb->device = device;
        const size_t want_off = std::max((size_t) n + 1, kb ? kb->off.cap + kb->off.cap / 2 : 0);
        const size_t want_bytes = std::max((size_t) std::max<int64_t>(n_bytes, 1), kb ? kb->bytes.cap + kb->bytes.cap / 2 : 0);
        BFQ_CUDA_TRY(nb->off.reserve(want_off));
        BFQ_CUDA_TRY(nb->bytes.reserve(want_bytes));
        if (kb) {
            BFQ_CUDA_TRY(cudaMemcpyAsync(nb->off.p, kb->off.p, (size_t) (t.key_ids + 1) * 8, cudaMemcpyDeviceToDevice, st));
            if (t.key_bytes)
                BFQ_CUDA_TRY(cudaMemcpyAsync(nb->bytes.p, kb->bytes.p, (size_t) t.key_bytes, cudaMemcpyDeviceToDevice, st));
        } else {
            BFQ_CUDA_TRY(cudaMemsetAsync(nb->off.p, 0, 8, st));   // off[0]
        }
        kb = nb;
    }
    // appended past what earlier gathers read: they keep running on the same buffers
    if (!ends.empty())
        BFQ_CUDA_TRY(cudaMemcpyAsync(kb->off.p + t.key_ids + 1, ends.data(), ends.size() * 8, cudaMemcpyHostToDevice, st));
    if (!blob.empty()) BFQ_CUDA_TRY(cudaMemcpyAsync(kb->bytes.p + t.key_bytes, blob.data(), blob.size(), cudaMemcpyHostToDevice, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    t.keys = kb;
    t.key_ids = n;
    t.key_bytes = n_bytes;
    t.key_device_bytes = (int64_t) (kb->bytes.bytes() + kb->off.bytes());
    *out = kb;
    return BFQ_OK;
}

// ------------------------------------------------------------------------------------------------ the match
struct RCoreIn {
    const uint8_t* tenants;
    const int64_t* tenant_off;
    int32_t n_tenants;
    const uint8_t* d_filters;
    const int64_t* d_filter_off;
    const int32_t* d_filter_tenant;
    int64_t n;
    const int64_t* d_limit;      // nullptr = unlimited
    bool check_tenants;          // filter_tenant has not been range-checked on the host
};
struct RCoreOut {
    unsigned long long n_ids = 0, n_ranges = 0, n_overflow = 0;
};

// The match of a batch resident on the device, enqueued on w->stream: tenant roots, locality order, rmatch_kernel (re-run
// while the range buffer grows), the limit, the id offsets and rexpand_kernel. On return the ids are enqueued to
// w->d_ids, d_offsets[n + 1] / d_total[n] hold offsets and totals, and ev[1] follows the last kernel. The caller holds h->mu
// shared and keeps it until w->stream has drained: rexpand_kernel is the last to read the snapshot's tables.
int32_t rmatch_core(bfq_rindex* h, RWorkspace* w, const RCoreIn& in, RCoreOut* out) {
    cudaStream_t st = w->stream;
    const int64_t n = in.n;
    const int32_t n_tenants = in.n_tenants;
    const size_t nn = (size_t) std::max<int64_t>(n, 1), nt = (size_t) std::max(n_tenants, 1);
    unsigned long long* hc = nullptr;
    BFQ_CUDA_TRY(w->h_small.reserve(RC_COUNT + 1));
    hc = w->h_small.p;
    BFQ_CUDA_TRY(w->d_offsets.reserve(nn + 1));
    if (n == 0) {
        BFQ_CUDA_TRY(cudaMemsetAsync(w->d_offsets.p, 0, 8, st));
        return BFQ_OK;
    }
    BFQ_CUDA_TRY(w->h_tenant_root.reserve(nt));
    for (int32_t t = 0; t < n_tenants; t++) {
        auto it = h->tenant_root.find(std::string((const char*) in.tenants + in.tenant_off[t], (size_t) (in.tenant_off[t + 1] - in.tenant_off[t])));
        w->h_tenant_root.p[t] = it != h->tenant_root.end() ? it->second : -1;
    }
    BFQ_CUDA_TRY(w->d_tenant_root.reserve(nt));
    BFQ_CUDA_TRY(w->d_span_begin.reserve(nn));
    BFQ_CUDA_TRY(w->d_span_count.reserve(nn));
    BFQ_CUDA_TRY(w->d_overflow.reserve(nn));
    BFQ_CUDA_TRY(w->d_total.reserve(nn));
    BFQ_CUDA_TRY(w->d_kept.reserve(nn + 1));
    BFQ_CUDA_TRY(w->d_counters.reserve(RC_COUNT));
    if (w->d_ranges.cap == 0) BFQ_CUDA_TRY(w->d_ranges.reserve(std::max<size_t>(1 << 18, 8 * nn)));
    if (n_tenants > 0)
        BFQ_CUDA_TRY(cudaMemcpyAsync(w->d_tenant_root.p, w->h_tenant_root.p, (size_t) n_tenants * 4, cudaMemcpyHostToDevice, st));
    BFQ_CUDA_TRY(cudaEventRecord(w->ev[0], st));   // the inputs are (enqueued to be) resident: device time of the kernels from here
    if (in.check_tenants) {
        BFQ_CUDA_TRY(cudaMemsetAsync(w->d_counters.p, 0, RC_COUNT * sizeof(unsigned long long), st));
        rcheck_tenants_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(n, in.d_filter_tenant, n_tenants, w->d_counters.p + RC_COUNT - 1);
        h->launches++;
        BFQ_CUDA_TRY(cudaGetLastError());
        BFQ_CUDA_TRY(cudaMemcpyAsync(hc + RC_COUNT - 1, w->d_counters.p + RC_COUNT - 1, 8, cudaMemcpyDeviceToHost, st));
        BFQ_CUDA_TRY(cudaStreamSynchronize(st));
        if (hc[RC_COUNT - 1] != 0) return fail(BFQ_E_RANGE, "filter_tenant out of range");
    }

    RMatchParams p{};
    p.nodes = h->d_nodes.p;
    p.slots = h->d_slots.p;
    p.tags = reinterpret_cast<const uint4*>(h->d_tags.p);
    p.n_blocks = h->n_blocks;
    p.filters = in.d_filters;
    p.filter_off = in.d_filter_off;
    p.filter_tenant = in.d_filter_tenant;
    p.tenant_root = w->d_tenant_root.p;
    p.n_filters = n;
    p.span_begin = w->d_span_begin.p;
    p.span_count = w->d_span_count.p;
    p.total = w->d_total.p;
    p.overflow_list = w->d_overflow.p;
    p.counters = w->d_counters.p;
    const int sms = device_sm_count();
    int ctas_per_sm = 4;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctas_per_sm, rmatch_kernel<false>, R_WARPS * 32, 0);
    ctas_per_sm = std::max(1, ctas_per_sm);
    // filters that share a tenant and leading levels walk the same part of the topic trie: group them so that the warps
    // running at the same time hit the same node records in L2 (the forward path's locality order, reused)
    const uint32_t* order = nullptr;
    if (n >= 4096) {
        BFQ_CUDA_TRY(w->d_ord_keys.reserve(nn));
        BFQ_CUDA_TRY(w->d_ord_leader.reserve(nn));
        BFQ_CUDA_TRY(w->d_order.reserve(nn));
        BFQ_CUDA_TRY(w->d_hist.reserve(order_scratch_words(n, n_tenants)));
        BFQ_CUDA_TRY(w->d_ord_ctr.reserve(CTR_COUNT));
        OrderParams q{};
        q.n_topics = n;
        q.topics = in.d_filters;
        q.topic_off = in.d_filter_off;
        q.topic_tenant = in.d_filter_tenant;
        q.n_tenants = n_tenants;
        q.keys = w->d_ord_keys.p;
        q.leader = w->d_ord_leader.p;
        q.order = w->d_order.p;
        q.hash_tab = nullptr;
        q.hash_mask = 0;
        q.hist = w->d_hist.p;
        q.dedup = 0;
        q.counters = w->d_ord_ctr.p;
        BFQ_CUDA_TRY(launch_order(q, st));
        h->launches += 3;
        order = q.order;
    }
    for (int attempt = 0; attempt < 8; attempt++) {
        p.ranges = w->d_ranges.p;
        p.ranges_cap = w->d_ranges.cap;
        p.work_list = order;
        p.n_work = 0;
        BFQ_CUDA_TRY(cudaMemsetAsync(w->d_counters.p, 0, RC_COUNT * sizeof(unsigned long long), st));
        int64_t ctas = std::min<int64_t>((n + R_WARPS - 1) / R_WARPS, (int64_t) sms * ctas_per_sm);
        BFQ_CUDA_TRY(cudaEventRecord(w->ev[2], st));
        rmatch_kernel<false><<<(unsigned) std::max<int64_t>(ctas, 1), R_WARPS * 32, 0, st>>>(p);
        BFQ_CUDA_TRY(cudaEventRecord(w->ev[3], st));
        h->launches++;
        BFQ_CUDA_TRY(cudaGetLastError());
        BFQ_CUDA_TRY(cudaMemcpyAsync(hc, w->d_counters.p, RC_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
        BFQ_CUDA_TRY(cudaStreamSynchronize(st));
        if (hc[RC_OVERFLOW] > 0) {
            const uint64_t capF = (uint64_t) h->max_nodes_per_depth + 2;
            const uint64_t capR = 3 * ((uint64_t) h->n_nodes + 2) + 2;
            const uint64_t per_warp = 2 * capF + capR;
            uint64_t warps = std::min<uint64_t>(hc[RC_OVERFLOW], std::max<uint64_t>(8, (1ull << 31) / (per_warp * sizeof(uint2))));
            warps = std::min<uint64_t>((warps + 7) / 8 * 8, (uint64_t) sms * 8);
            BFQ_CUDA_TRY(w->d_scratch.reserve((size_t) (warps * per_warp)));
            p.scratch = w->d_scratch.p;
            p.scratch_frontier_cap = capF;
            p.scratch_ranges_cap = capR;
            p.work_list = w->d_overflow.p;
            p.n_work = (int64_t) hc[RC_OVERFLOW];
            rmatch_kernel<true><<<(unsigned) (warps / 8), R_WARPS * 32, 0, st>>>(p);
            h->launches++;
            BFQ_CUDA_TRY(cudaGetLastError());
            BFQ_CUDA_TRY(cudaMemcpyAsync(hc, w->d_counters.p, RC_COUNT * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
            BFQ_CUDA_TRY(cudaStreamSynchronize(st));
            if (hc[RC_ERROR] != 0) return fail(BFQ_E_STATE, "tier-2 scratch exhausted");
        }
        if (hc[RC_RANGES] <= w->d_ranges.cap) break;
        const size_t want = (size_t) (hc[RC_RANGES] + hc[RC_RANGES] / 4 + 1024);
        if (want >= 0xFFFFFFF0ull || attempt == 7) return fail(BFQ_E_RANGE, "too many matched ranges in one batch; split the batch");
        BFQ_CUDA_TRY(w->d_ranges.reserve(want));
    }
    out->n_ranges = hc[RC_RANGES];
    out->n_overflow = hc[RC_OVERFLOW];
    // kept = min(total, limit), kept[n] = 0; exclusive scan over n + 1, so offsets[n] is the grand total; expand to ids
    rkept_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(n, w->d_total.p, in.d_limit, w->d_kept.p);
    BFQ_CUDA_TRY(cudaMemsetAsync(w->d_kept.p + n, 0, 8, st));
    size_t tmp_bytes = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, w->d_kept.p, w->d_offsets.p, (int) (n + 1), st);
    BFQ_CUDA_TRY(w->d_scan_tmp.reserve(tmp_bytes));
    cub::DeviceScan::ExclusiveSum(w->d_scan_tmp.p, tmp_bytes, w->d_kept.p, w->d_offsets.p, (int) (n + 1), st);
    h->launches += 2;
    // only the grand total is needed on the host before the expansion (to size the id buffer)
    BFQ_CUDA_TRY(cudaMemcpyAsync(hc + RC_COUNT, w->d_offsets.p + n, 8, cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    out->n_ids = hc[RC_COUNT];
    BFQ_CUDA_TRY(w->d_ids.reserve((size_t) std::max<unsigned long long>(out->n_ids, 1)));
    rexpand_kernel<<<(unsigned) ((n * 32 + 255) / 256), 256, 0, st>>>(n, w->d_span_begin.p, w->d_span_count.p, w->d_ranges.p,
                                                                      w->d_offsets.p, w->d_kept.p, h->d_dfs_to_id.p,
                                                                      h->d_bfs_to_id.p, w->d_ids.p);
    h->launches++;
    BFQ_CUDA_TRY(cudaGetLastError());
    BFQ_CUDA_TRY(cudaEventRecord(w->ev[1], st));
    return BFQ_OK;
}

}  // namespace

extern "C" {

int32_t bfq_rindex_create(int32_t device_ordinal, bfq_rindex** out) {
    if (!out) return fail(BFQ_E_INVALID, "out is NULL");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(BFQ_E_CUDA, std::string("no usable CUDA device (there is no CPU fallback): ") + cudaGetErrorString(e));
    if (device_ordinal < 0 || device_ordinal >= count) return fail(BFQ_E_INVALID, "device ordinal out of range");
    BFQ_CUDA_TRY(cudaSetDevice(device_ordinal));
    auto* h = new bfq_rindex();
    h->device = device_ordinal;
    h->pool->device = device_ordinal;
    if (cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
        delete h;
        return fail(BFQ_E_CUDA, "cudaStreamCreate failed");
    }
    *out = h;
    return BFQ_OK;
}
void bfq_rindex_destroy(bfq_rindex* h) { delete h; }

int32_t bfq_rindex_reset(bfq_rindex* h) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    WriteLock g(h);
    h->staged.clear();
    h->by_id = std::make_shared<IdTable>();   // the committed table stays with the snapshot and its results
    h->alive.clear();
    h->dirty.clear();
    h->need_full = true;
    return BFQ_OK;
}

int32_t bfq_rindex_add(bfq_rindex* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                       const uint8_t* topics, const int64_t* topic_off, const int32_t* topic_tenant, int64_t n, int64_t* ids_out) {
    if (!h || n < 0 || n_tenants < 0) return fail(BFQ_E_INVALID, "bad argument");
    WriteLock g(h);
    std::vector<std::string> ts((size_t) n_tenants);
    for (int32_t t = 0; t < n_tenants; t++) ts[(size_t) t].assign((const char*) tenants + tenant_off[t], (size_t) (tenant_off[t + 1] - tenant_off[t]));
    for (int64_t i = 0; i < n; i++) {
        if (topic_tenant[i] < 0 || topic_tenant[i] >= n_tenants) return fail(BFQ_E_RANGE, "topic_tenant out of range");
        std::pair<std::string, std::string> key(ts[(size_t) topic_tenant[i]],
                                                std::string((const char*) topics + topic_off[i], (size_t) (topic_off[i + 1] - topic_off[i])));
        auto it = h->staged.find(key);
        int64_t id;
        if (it == h->staged.end()) {
            id = (int64_t) h->by_id->e.size();
            h->by_id->e.push_back(key);
            h->alive.push_back(1);
            h->dirty.insert(key.first);
            h->staged.emplace(std::move(key), id);
        } else {
            id = it->second;
        }
        if (ids_out) ids_out[i] = id;
    }
    return BFQ_OK;
}

// The feed of RetainStoreCoProc.load() (RS/RetainStoreCoProc.java:279-296): raw retain-store KV keys from a range scan. The
// reference parses every VALUE (a TopicMessage proto) for the topic; the key carries it too (escaped, behind the level-hash bytes),
// so the index is fed from the keys alone. ids_out[i] < 0 marks a key that is not a retain key (skipped, as the reference logs
// and skips an unparsable entry).
int32_t bfq_rindex_load_keys(bfq_rindex* h, const uint8_t* keys, const int64_t* key_off, int64_t n, int64_t* ids_out) {
    if (!h || n < 0 || (n > 0 && (!keys || !key_off))) return fail(BFQ_E_INVALID, "bad argument");
    WriteLock g(h);
    if (h->staged.empty()) h->need_full = true;   // a bulk load onto an empty handle: one full build beats a delta per tenant
    for (int64_t i = 0; i < n; i++) {
        sv tenant;
        std::string topic;
        if (key_off[i + 1] < key_off[i] || !decode_retain_key(sv((const char*) keys + key_off[i], (size_t) (key_off[i + 1] - key_off[i])), &tenant, &topic)) {
            if (ids_out) ids_out[i] = -1;
            continue;
        }
        std::pair<std::string, std::string> key(std::string(tenant), std::move(topic));
        auto it = h->staged.find(key);
        int64_t id;
        if (it == h->staged.end()) {
            id = (int64_t) h->by_id->e.size();
            h->by_id->e.push_back(key);
            h->alive.push_back(1);
            h->dirty.insert(key.first);
            h->staged.emplace(std::move(key), id);
        } else {
            id = it->second;
        }
        if (ids_out) ids_out[i] = id;
    }
    return BFQ_OK;
}

// retainMessageKey(tenant, topic) of every id in a match result, in result order: the keys of the follow-up reader.get calls of
// RetainStoreCoProc.match (RS/RetainStoreCoProc.java:177-188), as one batch. Returns the blob length; copies if it fits.
// The ids are resolved in the id table of the snapshot the match ran on, so a reset + reload between the match and this call
// does not change the answer. h->mu is taken shared: add / load_keys append to that same table until the next reset.
int64_t bfq_rresult_retain_keys(bfq_rindex* h, const bfq_rresult* r, uint8_t* blob_out, int64_t blob_cap, int64_t* key_off_out) {
    if (!h || !r) return BFQ_E_INVALID;
    std::shared_lock<std::shared_mutex> g(h->mu);
    int64_t at = 0;
    const int64_t n = (int64_t) r->ids.size();
    const auto& by_id = r->by_id->e;   // set by bfq_rmatch, which runs only after a commit
    for (int64_t i = 0; i < n; i++) {
        const int64_t id = r->ids[(size_t) i];
        if (id < 0 || id >= (int64_t) by_id.size()) return BFQ_E_RANGE;
        const std::string k = make_retain_key(by_id[(size_t) id].first, by_id[(size_t) id].second);
        if (key_off_out) key_off_out[i] = at;
        if (blob_out && at + (int64_t) k.size() <= blob_cap) memcpy(blob_out + at, k.data(), k.size());
        at += (int64_t) k.size();
    }
    if (key_off_out) key_off_out[n] = at;
    return at;
}

int32_t bfq_rindex_remove(bfq_rindex* h, const uint8_t* tenant, int64_t tn, const uint8_t* topic, int64_t n) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    WriteLock g(h);
    auto it = h->staged.find({std::string((const char*) tenant, (size_t) tn), std::string((const char*) topic, (size_t) n)});
    if (it != h->staged.end()) {
        h->alive[(size_t) it->second] = 0;
        h->dirty.insert(it->first.first);
        h->staged.erase(it);
    }
    return BFQ_OK;
}

int32_t bfq_rindex_commit(bfq_rindex* h) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    WriteLock g(h);
    int32_t rc = commit_delta(h);
    if (rc == NEED_FULL) rc = rebuild_full(h);
    if (rc == BFQ_OK) {
        h->committed = h->by_id;
        h->generation++;
    }
    return rc;
}

int32_t bfq_rindex_stats(bfq_rindex* h, int64_t* stats, int32_t n) {
    if (!h || (!stats && n > 0)) return fail(BFQ_E_INVALID, "bad argument");
    std::shared_lock<std::shared_mutex> g(h->mu);
    int64_t n_ws = 0, ws_bytes = 0;
    {
        std::lock_guard<std::mutex> p(h->pool->mu);
        n_ws = (int64_t) h->pool->held.size();
        for (const RWorkspace* w : h->pool->held) ws_bytes += w->bytes_held;
    }
    const int64_t key_bytes = h->by_id->key_device_bytes;
    const int64_t v[14] = {h->n_topics, (int64_t) h->regions.size(), h->n_nodes, h->garbage_nodes, h->used_slots,
                           (int64_t) h->n_blocks * BLOCK_USABLE, h->full_commits, h->delta_commits, h->last_rebuilt,
                           h->snapshot_bytes() + ws_bytes + key_bytes, h->overflowed_blocks, n_ws, ws_bytes, key_bytes};
    for (int32_t i = 0; i < n && i < 14; i++) stats[i] = v[i];
    return BFQ_OK;
}

int32_t bfq_rindex_lookup(bfq_rindex* h, int64_t id, uint8_t* tenant_out, int64_t tenant_cap, int64_t* tenant_len,
                          uint8_t* topic_out, int64_t topic_cap, int64_t* topic_len) {
    if (!h) return fail(BFQ_E_INVALID, "handle is NULL");
    std::shared_lock<std::shared_mutex> g(h->mu);
    if (id < 0 || id >= (int64_t) h->by_id->e.size()) return fail(BFQ_E_RANGE, "id out of range");
    const auto& e = h->by_id->e[(size_t) id];
    if (tenant_len) *tenant_len = (int64_t) e.first.size();
    if (topic_len) *topic_len = (int64_t) e.second.size();
    if (tenant_out && (int64_t) e.first.size() <= tenant_cap) memcpy(tenant_out, e.first.data(), e.first.size());
    if (topic_out && (int64_t) e.second.size() <= topic_cap) memcpy(topic_out, e.second.data(), e.second.size());
    return BFQ_OK;
}

int32_t bfq_rmatch(bfq_rindex* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                   const uint8_t* filters, const int64_t* filter_off, const int32_t* filter_tenant, int64_t n,
                   const int64_t* limit, bfq_rresult** out) {
    if (!h || !out || n < 0 || n_tenants < 0) return fail(BFQ_E_INVALID, "bad argument");
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    auto g = read_lock(h);   // declared first: released after the lease below has drained its stream
    CallLease lease{h->pool};
    int32_t rc = acquire(h, &lease.w);
    if (rc != BFQ_OK) return rc;
    RWorkspace* w = lease.w;
    if (!h->have_snapshot) return fail(BFQ_E_STATE, "bfq_rmatch before the first bfq_rindex_commit");
    for (int64_t i = 0; i < n; i++)
        if (filter_tenant[i] < 0 || filter_tenant[i] >= n_tenants) return fail(BFQ_E_RANGE, "filter_tenant out of range");
    cudaStream_t st = w->stream;
    auto t0 = std::chrono::steady_clock::now();
    std::unique_ptr<bfq_rresult> res(new bfq_rresult());
    res->by_id = h->committed;
    res->generation = h->generation;
    res->offsets.assign((size_t) n + 1, 0);
    res->totals.assign((size_t) n, 0);
    if (n == 0) {
        *out = res.release();
        return BFQ_OK;
    }
    // the batch into one device block of the workspace, straight from the caller's memory: the driver overlaps its own staging
    // of pageable memory with the transfer, where a copy into pinned memory first would add a host pass over the whole batch
    const int64_t fbytes = filter_off[n];
    uint8_t* d_filters = nullptr;
    int64_t *d_filter_off = nullptr, *d_limit = nullptr;
    int32_t* d_filter_tenant = nullptr;
    rc = carve(w->d_in, "bfq_rmatch inputs", [&](Carve& c) {
        d_filters = c.take<uint8_t>((size_t) fbytes);
        d_filter_off = c.take<int64_t>((size_t) n + 1);
        d_filter_tenant = c.take<int32_t>((size_t) n);
        d_limit = limit ? c.take<int64_t>((size_t) n) : nullptr;
    });
    if (rc != BFQ_OK) return rc;
    BFQ_CUDA_TRY(cudaMemcpyAsync(d_filters, filters, (size_t) fbytes, cudaMemcpyHostToDevice, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(d_filter_off, filter_off, (size_t) (n + 1) * 8, cudaMemcpyHostToDevice, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(d_filter_tenant, filter_tenant, (size_t) n * 4, cudaMemcpyHostToDevice, st));
    if (limit) BFQ_CUDA_TRY(cudaMemcpyAsync(d_limit, limit, (size_t) n * 8, cudaMemcpyHostToDevice, st));
    auto t1 = std::chrono::steady_clock::now();
    RCoreOut co;
    rc = rmatch_core(h, w, RCoreIn{tenants, tenant_off, n_tenants, d_filters, d_filter_off, d_filter_tenant, n, d_limit, false}, &co);
    if (rc != BFQ_OK) return rc;
    auto t2 = std::chrono::steady_clock::now();
    // the result owns its arrays: offsets / totals / ids are read back straight into them (same 8-byte element types)
    static_assert(sizeof(unsigned long long) == sizeof(int64_t), "offsets are copied without conversion");
    res->ids.resize((size_t) co.n_ids);
    BFQ_CUDA_TRY(cudaMemcpyAsync(res->offsets.data(), w->d_offsets.p, (size_t) (n + 1) * 8, cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaMemcpyAsync(res->totals.data(), w->d_total.p, (size_t) n * 8, cudaMemcpyDeviceToHost, st));
    if (co.n_ids) BFQ_CUDA_TRY(cudaMemcpyAsync(res->ids.data(), w->d_ids.p, (size_t) co.n_ids * 8, cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    g.unlock();
    auto t3 = std::chrono::steady_clock::now();
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    res->ms[0] = ms(t0, t1);
    res->ms[1] = ms(t1, t2);
    res->ms[2] = ms(t2, t3);
    res->ms[3] = ms(t0, t3);
    {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, w->ev[0], w->ev[1]);
        cudaEventElapsedTime(&b, w->ev[2], w->ev[3]);
        res->ms[4] = a;                       // device time from "inputs resident" to "ids expanded" (all kernels + the host's counter reads between them)
        res->ms[5] = b;                       // device time of rmatch_kernel (the last attempt)
        res->ms[6] = (double) co.n_ranges;    // rank ranges emitted (8 bytes each): the kernel's output size
        res->ms[7] = (double) co.n_overflow;
    }
    *out = res.release();
    return BFQ_OK;
}

int64_t bfq_rresult_num_filters(const bfq_rresult* r) { return r ? (int64_t) r->totals.size() : 0; }
const int64_t* bfq_rresult_offsets(const bfq_rresult* r) { return r->offsets.data(); }
const int64_t* bfq_rresult_ids(const bfq_rresult* r, int64_t* n) {
    if (n) *n = (int64_t) r->ids.size();
    return r->ids.data();
}
const int64_t* bfq_rresult_total_matches(const bfq_rresult* r) { return r->totals.data(); }
uint64_t bfq_rresult_generation(const bfq_rresult* r) { return r ? r->generation : 0; }
int32_t bfq_rresult_timings(const bfq_rresult* r, double* ms, int32_t n) {
    if (!r || !ms) return fail(BFQ_E_INVALID, "bad argument");
    for (int32_t i = 0; i < n && i < 8; i++) ms[i] = r->ms[i];
    return BFQ_OK;
}
void bfq_rresult_free(bfq_rresult* r) { delete r; }

int32_t bfq_rmatch_device(bfq_rindex* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                          const uint8_t* d_filters, const int64_t* d_filter_off, const int32_t* d_filter_tenant, int64_t n,
                          const int64_t* d_limit, void* stream, bfq_rdevice_result* out) {
    if (!h || !out || n < 0 || n_tenants < 0) return fail(BFQ_E_INVALID, "bad argument");
    if (n_tenants > 0 && (!tenants || !tenant_off)) return fail(BFQ_E_INVALID, "NULL tenant list");
    if (n > 0 && (!d_filters || !d_filter_off || !d_filter_tenant)) return fail(BFQ_E_INVALID, "NULL filter arrays");
    memset(out, 0, sizeof(*out));
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    auto g = read_lock(h);   // declared first: released after the lease below has drained its stream
    CallLease lease{h->pool};
    int32_t rc = acquire(h, &lease.w);
    if (rc != BFQ_OK) return rc;
    RWorkspace* w = lease.w;
    if (!h->have_snapshot) return fail(BFQ_E_STATE, "bfq_rmatch_device before the first bfq_rindex_commit");
    // the batch was written on the caller's stream: the match runs on the workspace's own stream, after it
    BFQ_CUDA_TRY(cudaEventRecord(w->ev_in, (cudaStream_t) stream));
    BFQ_CUDA_TRY(cudaStreamWaitEvent(w->stream, w->ev_in, 0));
    RCoreOut co;
    rc = rmatch_core(h, w, RCoreIn{tenants, tenant_off, n_tenants, d_filters, d_filter_off, d_filter_tenant, n, d_limit, true}, &co);
    if (rc != BFQ_OK) return rc;
    BFQ_CUDA_TRY(cudaStreamSynchronize(w->stream));
    auto* L = new RLease();
    L->h = h;
    L->pool = h->pool;
    L->by_id = h->committed;
    out->generation = h->generation;
    g.unlock();
    out->d_offsets = reinterpret_cast<const int64_t*>(w->d_offsets.p);
    out->d_ids = w->d_ids.p;
    out->d_total = reinterpret_cast<const int64_t*>(w->d_total.p);
    out->n_filters = n;
    out->n_ids = (int64_t) co.n_ids;
    out->n_ranges = (int64_t) co.n_ranges;
    out->n_overflow_filters = (int64_t) co.n_overflow;
    if (n > 0) {
        float a = 0, b = 0;
        cudaEventElapsedTime(&a, w->ev[0], w->ev[1]);
        cudaEventElapsedTime(&b, w->ev[2], w->ev[3]);
        out->device_ms = a;
        out->kernel_ms = b;
    }
    L->ws = w;
    lease.w = nullptr;   // the result keeps the workspace until bfq_rdevice_result_release
    out->lease = L;
    return BFQ_OK;
}

void bfq_rdevice_result_release(bfq_rdevice_result* res) {
    if (!res || !res->lease) return;
    auto* L = static_cast<RLease*>(res->lease);
    cudaSetDevice(L->pool->device);
    // never hand a busy workspace back: every key gather on the result, on each stream it ran on
    for (size_t i = 0; i < L->used_on.size(); i++) cudaEventSynchronize(L->ws->ev_use[i]);
    give_back(L->pool, L->ws);
    delete L;
    res->lease = nullptr;
}

int32_t bfq_rretain_keys_device(bfq_rindex* h, const bfq_rdevice_result* res, int64_t* d_key_off, uint8_t* d_keys, int64_t cap,
                                void* stream, int64_t* n_bytes) {
    if (!h || !res || !d_key_off || !n_bytes) return fail(BFQ_E_INVALID, "bad argument");
    if (!res->lease) return fail(BFQ_E_INVALID, "no match behind this result");
    auto* L = static_cast<RLease*>(res->lease);
    if (L->h != h) return fail(BFQ_E_INVALID, "the result belongs to another handle");
    const int64_t n = res->n_ids;
    if (n >= (int64_t) INT32_MAX) return fail(BFQ_E_RANGE, "too many ids in one result");
    BFQ_CUDA_TRY(cudaSetDevice(h->device));
    std::lock_guard<std::mutex> u(L->use_mu);
    RWorkspace* w = L->ws;
    std::shared_ptr<KeyBufs> kb;
    {
        auto g = read_lock(h);   // the id table is read while its key table is extended
        const int32_t rc = extend_keys(*L->by_id, h->device, w->stream, &kb);
        if (rc != BFQ_OK) return rc;
    }
    if (std::find(L->keys.begin(), L->keys.end(), kb) == L->keys.end()) L->keys.push_back(kb);
    cudaStream_t st = (cudaStream_t) stream;
    size_t k = 0;
    while (k < L->used_on.size() && L->used_on[k] != st) k++;
    if (k == L->used_on.size()) {
        if (k == w->ev_use.size()) {
            cudaEvent_t e = nullptr;
            BFQ_CUDA_TRY(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            w->ev_use.push_back(e);
        }
        L->used_on.push_back(st);
    }
    RecordOnExit rec(w->ev_use[k], st);
    // sizing pass, scan, then the bytes if they fit
    BFQ_CUDA_TRY(cudaMemsetAsync(d_key_off, 0, 8, st));
    if (n > 0) {
        BFQ_CUDA_TRY(w->d_key_len.reserve((size_t) n));
        rkey_len_kernel<<<(unsigned) ((n + 255) / 256), 256, 0, st>>>(n, w->d_ids.p, kb->off.p, w->d_key_len.p);
        BFQ_CUDA_TRY(cudaGetLastError());
        size_t tmp_bytes = 0;
        cub::DeviceScan::InclusiveSum(nullptr, tmp_bytes, w->d_key_len.p, d_key_off + 1, (int) n, st);
        BFQ_CUDA_TRY(w->d_key_tmp.reserve(tmp_bytes));
        BFQ_CUDA_TRY(cub::DeviceScan::InclusiveSum(w->d_key_tmp.p, tmp_bytes, w->d_key_len.p, d_key_off + 1, (int) n, st));
        h->launches += 2;
    }
    BFQ_CUDA_TRY(w->h_small.reserve(RC_COUNT + 1));
    BFQ_CUDA_TRY(cudaMemcpyAsync(w->h_small.p + RC_COUNT, d_key_off + n, 8, cudaMemcpyDeviceToHost, st));
    BFQ_CUDA_TRY(cudaStreamSynchronize(st));
    const int64_t total = (int64_t) w->h_small.p[RC_COUNT];
    *n_bytes = total;
    if (d_keys && n > 0 && total <= cap) {
        rkey_copy_kernel<<<(unsigned) ((n * 32 + 255) / 256), 256, 0, st>>>(n, w->d_ids.p, kb->off.p, kb->bytes.p, d_key_off, d_keys);
        h->launches++;
        BFQ_CUDA_TRY(cudaGetLastError());
    }
    return BFQ_OK;
}

}  // extern "C"
