// delivery_reply.cu — every deliverer's DeliveryReply joined back to the pairs of its request (bfq_delivery_reply).
//
// BatchDeliveryCall.execute (bifromq-deliverer/.../BatchDeliveryCall.java:108-172) completes each (tenant, MatchInfo, pack)
// task from the reply, keyed on (tenant, MatchInfo) through TypeUtil.toMap, and removes the NO_SUB / NO_RECEIVER routes:
//   DeliveryReply   { Code code = 1; map<string tenantId, DeliveryResults> result = 2 }     entry {key = 1, value = 2}
//   DeliveryResults { repeated DeliveryResult result = 1 }
//   DeliveryResult  { MatchInfo matchInfo = 1; Code code = 2 }                              (subbroker/type.proto:41-63)
// The join is on bytes: a reply MatchInfo resolves when it equals, byte for byte, the canonical MatchInfo (the snapshot's
// table entry) of a pair the deliverer's request carries under that tenant. Anything the device cannot be sure to answer as
// the reference does (malformed bytes, a repeated singular field or tenant, an unknown tenant or MatchInfo, a duplicate) makes
// the deliverer FALLBACK, for the host to handle.
//
// Stages: the top level of every reply on a thread (its code and map entries), each map entry on a warp (its tenant resolved
// to a package of the request), then every entry's DeliveryResults cut into chunks: a thread per chunk guesses the first record
// start and walks from it to the chunk's end, a warp per entry accepts a guess only where it equals the previous chunk's
// accepted exit (re-walking the chunk otherwise), and a thread per chunk decodes the records from its accepted start. The
// pairs' distinct (package, MatchInfo entry) keys sit in an open-addressing table the records probe by the hash of their bytes.
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "fanout.h"

namespace bfq {

namespace {

constexpr int RP_THREADS = 256;
constexpr unsigned RP_GRID = 132 * 8;   // grid-stride kernels over device-side counts
constexpr uint32_t NO_MEMBER = 0xFFFFFFFFu;
constexpr uint32_t CODE_UNSET = 0xFFFFFFFFu;
constexpr unsigned long long EMPTY_KEY = ~0ull;
constexpr long long NONE = -1;

__device__ __forceinline__ uint32_t fnv_bytes(const uint8_t* b, uint64_t n) {
    uint32_t h = 2166136261u;
    for (uint64_t i = 0; i < n; i++) h = (h ^ b[i]) * 16777619u;
    return h;
}
__device__ __forceinline__ uint64_t slot_hash(uint32_t pkg, uint32_t h) {
    uint64_t x = ((uint64_t) pkg << 32 | h) * 0x9E3779B97F4A7C15ull;
    return x ^ (x >> 29);
}

// a varint of at most `max_bytes` bytes inside [p, end): the value, or false (truncated or too long)
__device__ __forceinline__ bool get_varint(const uint8_t* b, long long& p, long long end, int max_bytes, uint64_t* v) {
    uint64_t x = 0;
    for (int i = 0; i < max_bytes; i++) {
        if (p >= end) return false;
        const uint8_t c = b[p++];
        x |= (uint64_t) (c & 0x7F) << (7 * i);
        if (!(c & 0x80)) {
            *v = x;
            return true;
        }
    }
    return false;
}
// one field's tag and extent: for wire type 2 [*vs, *ve) is its payload, for wire type 0 *val its value. False for a
// malformed field: field number 0, a tag past 5 bytes, a wire type other than 0, 1, 2, 5, a length past `end`.
__device__ __forceinline__ bool get_field(const uint8_t* b, long long& p, long long end, uint32_t* no, uint32_t* wt,
                                          long long* vs, long long* ve, uint64_t* val) {
    uint64_t tag;
    if (!get_varint(b, p, end, 5, &tag) || tag > 0xFFFFFFFFull || (tag >> 3) == 0) return false;
    *no = (uint32_t) (tag >> 3);
    *wt = (uint32_t) (tag & 7);
    switch (*wt) {
    case 0:
        return get_varint(b, p, end, 10, val);
    case 1:
        p += 8;
        return p <= end;
    case 5:
        p += 4;
        return p <= end;
    case 2: {
        uint64_t len;
        if (!get_varint(b, p, end, 5, &len) || len > 0x7FFFFFFFull || (long long) len > end - p) return false;
        *vs = p;
        p += (long long) len;
        *ve = p;
        return true;
    }
    default:
        return false;
    }
}

// a DeliveryResult body [s, e): its matchInfo payload (must be present) and code (0 when absent, Java's int otherwise)
__device__ __forceinline__ bool parse_result(const uint8_t* b, long long s, long long e, long long* ms, long long* me, int32_t* code) {
    bool seen_mi = false, seen_code = false;
    *code = 0;
    long long p = s;
    while (p < e) {
        uint32_t no, wt;
        long long vs = 0, ve = 0;
        uint64_t val = 0;
        if (!get_field(b, p, e, &no, &wt, &vs, &ve, &val)) return false;
        if (no == 1) {
            if (wt != 2 || seen_mi) return false;
            seen_mi = true;
            *ms = vs;
            *me = ve;
        } else if (no == 2) {
            if (wt != 0 || seen_code) return false;
            seen_code = true;
            *code = (int32_t) (uint32_t) val;
        }
    }
    return seen_mi;
}

// the DeliveryResults fields from p up to the first that starts at or past `stop` (bounded by `end`): where the walk stops,
// or NONE for a malformed field
__device__ __forceinline__ long long walk(const uint8_t* b, long long p, long long stop, long long end) {
    while (p < stop) {
        uint32_t no, wt;
        long long vs, ve;
        uint64_t val;
        if (!get_field(b, p, end, &no, &wt, &vs, &ve, &val) || (no == 1 && wt != 2)) return NONE;
    }
    return p;
}

// strict UTF-8 (no overlongs, surrogates or code points past U+10FFFF), as protobuf's string parsing checks it
__device__ bool valid_utf8(const uint8_t* s, long long n) {
    long long i = 0;
    while (i < n) {
        const uint8_t c = s[i];
        if (c < 0x80) {
            i++;
            continue;
        }
        int k;
        uint32_t lo = 0x80, hi = 0xBF;
        if (c >= 0xC2 && c <= 0xDF) k = 1;
        else if (c == 0xE0) k = 2, lo = 0xA0;
        else if (c >= 0xE1 && c <= 0xEC) k = 2;
        else if (c == 0xED) k = 2, hi = 0x9F;
        else if (c >= 0xEE && c <= 0xEF) k = 2;
        else if (c == 0xF0) k = 3, lo = 0x90;
        else if (c >= 0xF1 && c <= 0xF3) k = 3;
        else if (c == 0xF4) k = 3, hi = 0x8F;
        else return false;
        if (i + k >= n) return false;
        for (int j = 1; j <= k; j++) {
            const uint8_t x = s[i + j];
            if (j == 1 ? (x < lo || x > hi) : (x < 0x80 || x > 0xBF)) return false;
        }
        i += k + 1;
    }
    return true;
}

__device__ __forceinline__ int64_t upper_index(const long long* off, int64_t n, long long x) {
    // last i in [0, n) with off[i] <= x (off non-decreasing, off[0] <= x)
    int64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}
__device__ __forceinline__ int64_t upper_index_u(const unsigned long long* off, int64_t n, unsigned long long x) {
    int64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (off[mid] <= x) lo = mid;
        else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ int64_t skipped_package(const ReplyParams& p) { return p.package_off[p.n_deliverers - 1]; }
__device__ __forceinline__ int64_t skipped_pack(const ReplyParams& p) { return p.pack_off[skipped_package(p)]; }
__device__ __forceinline__ uint32_t pair_entry(const ReplyParams& p, int64_t j) {
    const uint32_t m = p.match_member[j];
    return p.mi_first[p.match_rank[j]] + (m == NO_MEMBER ? 0u : m);
}
// the MatchInfo message inside table entry e (the entry is the request's whole `matchInfo = 3` field)
__device__ __forceinline__ void entry_body(const ReplyParams& p, uint32_t e, const uint8_t** s, uint64_t* n) {
    long long q = (long long) p.mi_off[e] + 1;
    uint64_t len = 0;
    get_varint(p.mi_bytes, q, (long long) p.mi_off[e + 1], 5, &len);
    *s = p.mi_bytes + q;
    *n = len;
}
__device__ __forceinline__ bool deliverer_sent(const ReplyParams& p, int64_t d) {
    if (d >= (int64_t) p.n_deliverers - 1) return false;
    const long long k0 = p.pack_off[p.package_off[d]], k1 = p.pack_off[p.package_off[d + 1]];
    return p.match_off[k1] > p.match_off[k0];
}
__device__ __forceinline__ bool stopped(const ReplyParams& p) { return p.ctr[RP_BAD_OFF] != 0; }

__global__ void __launch_bounds__(RP_THREADS) mi_hash_kernel(const uint8_t* bytes, const unsigned long long* off, int64_t n,
                                                             uint32_t* out) {
    const int64_t e = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x;
    if (e >= n) return;
    long long q = (long long) off[e] + 1;
    uint64_t len = 0;
    get_varint(bytes, q, (long long) off[e + 1], 5, &len);
    out[e] = fnv_bytes(bytes + q, len);
}

// reply offsets never decrease
__global__ void __launch_bounds__(RP_THREADS) rp_check_kernel(const ReplyParams p) {
    for (int64_t d = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x; d < (int64_t) p.n_deliverers; d += (int64_t) gridDim.x * RP_THREADS)
        if (p.reply_off[d + 1] < p.reply_off[d]) atomicAdd(&p.ctr[RP_BAD_OFF], 1ull);
}

// every pair's (package, entry) key inserted; pair_slot names its slot. A thread per pack.
__global__ void __launch_bounds__(RP_THREADS) rp_insert_kernel(const ReplyParams p) {
    const int64_t k = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x;
    if (k >= p.n_packs || k >= skipped_pack(p)) return;
    const uint32_t g = (uint32_t) upper_index(p.pack_off, p.n_packages, k);
    for (long long j = p.match_off[k]; j < p.match_off[k + 1]; j++) {
        const uint32_t e = pair_entry(p, j);
        const unsigned long long key = (unsigned long long) g << 32 | e;
        for (uint64_t s = slot_hash(g, p.mi_hash[e]) & p.table_mask;; s = (s + 1) & p.table_mask) {
            unsigned long long cur = p.slot_key[s];
            if (cur == EMPTY_KEY) {
                cur = atomicCAS(&p.slot_key[s], EMPTY_KEY, key);
                if (cur == EMPTY_KEY) {
                    p.slot_pair[s] = (uint32_t) j;
                    p.slot_code[s] = CODE_UNSET;
                    cur = key;
                }
            }
            if (cur == key) {
                p.pair_slot[j] = (uint32_t) s;
                break;
            }
        }
    }
}

// the top level of deliverer d's reply: its code, and its map entries at ent_s / ent_e[package_off[d] + i]
__global__ void __launch_bounds__(RP_THREADS) rp_top_kernel(const ReplyParams p) {
    const int64_t d = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x;
    if (d >= (int64_t) p.n_deliverers || stopped(p)) return;
    p.dl_fail[d] = 0;
    p.dl_code[d] = 0;
    p.dl_entries[d] = 0;
    if (!deliverer_sent(p, d)) return;
    const long long g0 = p.package_off[d], cap = p.package_off[d + 1] - g0, end = p.reply_off[d + 1];
    long long q = p.reply_off[d], n = 0;
    int32_t code = 0;
    bool seen_code = false, ok = true;
    while (ok && q < end) {
        uint32_t no, wt;
        long long vs = 0, ve = 0;
        uint64_t val = 0;
        if (!get_field(p.reply, q, end, &no, &wt, &vs, &ve, &val)) ok = false;
        else if (no == 1) {
            ok = wt == 0 && !seen_code;
            seen_code = true;
            code = (int32_t) (uint32_t) val;
        } else if (no == 2) {
            ok = wt == 2 && n < cap;   // more entries than requested tenants: one repeats or was never sent
            if (ok) {
                p.ent_s[g0 + n] = vs;
                p.ent_e[g0 + n] = ve;
                n++;
            }
        }
    }
    p.dl_code[d] = code;
    p.dl_entries[d] = (uint32_t) n;
    if (!ok) p.dl_fail[d] = 1;
}

// map entry slot g on a warp: key and value, the key resolved to the one package of the deliverer whose tenant it is
__global__ void __launch_bounds__(RP_THREADS) rp_entry_kernel(const ReplyParams p) {
    const int64_t g = ((int64_t) blockIdx.x * RP_THREADS + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if (g >= p.n_packages || stopped(p)) return;
    const int64_t d = upper_index(p.package_off, p.n_deliverers, g);
    const long long g0 = p.package_off[d];
    if (lane == 0) p.ent_vs[g] = p.ent_ve[g] = 0;
    // other warps of this kernel may be setting dl_fail[d]: one lane reads it, so the whole warp leaves or stays
    const bool skip = __shfl_sync(0xFFFFFFFFu, lane == 0 && (g - g0 >= (long long) p.dl_entries[d] || p.dl_fail[d]), 0);
    if (skip) return;
    long long ks = 0, ke = 0, vs = 0, ve = 0;
    bool ok = true;
    if (lane == 0) {
        bool seen_k = false, seen_v = false;
        long long q = p.ent_s[g];
        const long long end = p.ent_e[g];
        while (ok && q < end) {
            uint32_t no, wt;
            long long s = 0, e = 0;
            uint64_t val;
            if (!get_field(p.reply, q, end, &no, &wt, &s, &e, &val)) ok = false;
            else if (no == 1) {
                ok = wt == 2 && !seen_k;
                seen_k = true;
                ks = s;
                ke = e;
            } else if (no == 2) {
                ok = wt == 2 && !seen_v;
                seen_v = true;
                vs = s;
                ve = e;
            }
        }
        ok = ok && valid_utf8(p.reply + ks, ke - ks);
    }
    ok = __shfl_sync(0xFFFFFFFFu, ok, 0);
    ks = __shfl_sync(0xFFFFFFFFu, ks, 0);
    ke = __shfl_sync(0xFFFFFFFFu, ke, 0);
    if (ok) {
        int matches = 0;
        long long hit = -1;
        const long long kl = ke - ks;
        for (long long base = g0; base < p.package_off[d + 1]; base += 32) {
            const long long pk = base + lane;
            bool eq = false;
            if (pk < p.package_off[d + 1]) {
                const uint32_t tn = p.package_tenant[pk];
                const long long a = p.tenant_off[tn];
                eq = p.tenant_off[tn + 1] - a == kl;
                for (long long i = 0; eq && i < kl; i++) eq = p.tenants[a + i] == p.reply[ks + i];
            }
            const unsigned m = __ballot_sync(0xFFFFFFFFu, eq);
            matches += __popc(m);
            if (m && hit < 0) hit = base + __ffs(m) - 1;
        }
        ok = matches == 1;
        if (ok && lane == 0) {
            ok = atomicExch(&p.pkg_claimed[hit], 1u) == 0;   // a tenant key seen twice
            if (ok) {
                p.ent_pkg[g] = (uint32_t) hit;
                p.ent_vs[g] = vs;
                p.ent_ve[g] = ve;
                atomicAdd(&p.ctr[RP_VALUE_BYTES], (unsigned long long) (ve - vs));
            }
        }
        ok = __shfl_sync(0xFFFFFFFFu, ok, 0);
    }
    if (!ok && lane == 0) {
        p.dl_fail[d] = 1;
        p.ent_vs[g] = p.ent_ve[g] = 0;
    }
}

__device__ __forceinline__ long long chunk_size(const ReplyParams& p) {
    const unsigned long long total = p.ctr[RP_VALUE_BYTES];
    return (long long) max((unsigned long long) RP_CHUNK_MIN, (total + RP_MAX_CHUNKS - 1) / RP_MAX_CHUNKS);
}

__global__ void __launch_bounds__(RP_THREADS) rp_chunk_count_kernel(const ReplyParams p) {
    const int64_t g = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x;
    if (g > p.n_packages) return;
    unsigned long long n = 0;
    if (g < p.n_packages && !stopped(p)) {
        const long long cs = chunk_size(p), len = p.ent_ve[g] - p.ent_vs[g];
        n = (unsigned long long) ((len + cs - 1) / cs);
    }
    p.chunk_base[g] = n;
}

struct Chunk {
    int64_t g;
    long long s, e;   // the chunk's bytes
    long long ve;     // its entry's value end
    bool first;
};
__device__ __forceinline__ Chunk chunk_at(const ReplyParams& p, unsigned long long c) {
    Chunk k;
    k.g = upper_index_u(p.chunk_base, p.n_packages + 1, c);
    const long long cs = chunk_size(p);
    const unsigned long long i = c - p.chunk_base[k.g];
    k.s = p.ent_vs[k.g] + (long long) i * cs;
    k.ve = p.ent_ve[k.g];
    k.e = min(k.s + cs, k.ve);
    k.first = i == 0;
    return k;
}

// every chunk's guess (the first position whose bytes pass as a whole DeliveryResult field) and the walk from it
__global__ void __launch_bounds__(RP_THREADS) rp_guess_kernel(const ReplyParams p) {
    if (stopped(p)) return;
    const unsigned long long n = p.chunk_base[p.n_packages];
    for (unsigned long long c = (unsigned long long) blockIdx.x * RP_THREADS + threadIdx.x; c < n;
         c += (unsigned long long) gridDim.x * RP_THREADS) {
        const Chunk k = chunk_at(p, c);
        long long guess = k.first ? k.s : NONE;
        for (long long q = k.s; guess == NONE && q < k.e; q++) {
            if (p.reply[q] != 0x0A) continue;
            long long r = q + 1;
            uint64_t len;
            if (!get_varint(p.reply, r, k.ve, 5, &len) || (long long) len > k.ve - r) continue;
            long long ms, me;
            int32_t code;
            if (parse_result(p.reply, r, r + (long long) len, &ms, &me, &code)) guess = q;
        }
        p.ch_guess[c] = guess;
        p.ch_exit[c] = guess == NONE ? NONE : walk(p.reply, guess, k.e, k.ve);
    }
}

// a warp per entry: chunk i + 1 starts where chunk i's accepted walk ended; a guess that says otherwise is re-walked from there
__global__ void __launch_bounds__(RP_THREADS) rp_fix_kernel(const ReplyParams p) {
    const int64_t g = ((int64_t) blockIdx.x * RP_THREADS + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if (g >= p.n_packages || stopped(p)) return;
    const unsigned long long c0 = p.chunk_base[g], n = p.chunk_base[g + 1] - c0;
    if (n == 0) return;
    long long cur = p.ent_vs[g];
    bool ok = true;
    for (unsigned long long i = 0; ok && i < n;) {
        const unsigned long long c = c0 + i + lane;
        const bool in = i + lane < n;
        const long long gs = in ? p.ch_guess[c] : NONE, ex = in ? p.ch_exit[c] : NONE;
        long long prev = __shfl_up_sync(0xFFFFFFFFu, ex, 1);
        if (lane == 0) prev = cur;
        const bool good = in && prev != NONE && gs == prev;
        const unsigned bad = __ballot_sync(0xFFFFFFFFu, !good);
        const uint32_t f = bad ? (uint32_t) (__ffs(bad) - 1) : 32u;   // chunks i .. i + f - 1 start at their guesses
        if (lane < f) p.ch_start[c] = gs;
        const long long last = __shfl_sync(0xFFFFFFFFu, ex, (f ? f : 1) - 1);
        if (f > 0) cur = last;
        i += f;
        if (i >= n || f == 32) continue;
        // chunk i starts at cur (the previous chunk's exit): walk it
        if (cur == NONE) {
            ok = false;
            break;
        }
        if (lane == 0) {
            const Chunk k = chunk_at(p, c0 + i);
            p.ch_start[c0 + i] = cur;
            cur = walk(p.reply, cur, k.e, k.ve);
        }
        cur = __shfl_sync(0xFFFFFFFFu, cur, 0);
        i++;
        ok = cur != NONE;
    }
    ok = ok && cur == p.ent_ve[g];
    if (!ok && lane == 0) {
        p.dl_fail[upper_index(p.package_off, p.n_deliverers, p.ent_pkg[g])] = 1;
        p.ent_bad[g] = 1;
    }
}

// every record from the chunks' accepted starts: decoded, its MatchInfo found in the table, its code set once
__global__ void __launch_bounds__(RP_THREADS) rp_decode_kernel(const ReplyParams p) {
    if (stopped(p)) return;
    const unsigned long long n = p.chunk_base[p.n_packages];
    for (unsigned long long c = (unsigned long long) blockIdx.x * RP_THREADS + threadIdx.x; c < n;
         c += (unsigned long long) gridDim.x * RP_THREADS) {
        const Chunk k = chunk_at(p, c);
        if (p.ent_bad[k.g]) continue;
        const uint32_t pkg = p.ent_pkg[k.g];
        const int64_t d = upper_index(p.package_off, p.n_deliverers, pkg);
        bool ok = true;
        long long q = p.ch_start[c];
        while (ok && q < k.e && !p.dl_fail[d]) {
            uint32_t no, wt;
            long long rs = 0, re = 0;
            uint64_t val;
            ok = get_field(p.reply, q, k.ve, &no, &wt, &rs, &re, &val) && (no != 1 || wt == 2);
            if (!ok || no != 1) continue;
            long long ms = 0, me = 0;
            int32_t code;
            ok = parse_result(p.reply, rs, re, &ms, &me, &code);
            if (!ok) continue;
            const uint8_t* mb = p.reply + ms;
            const uint64_t ml = (uint64_t) (me - ms);
            const uint32_t h = fnv_bytes(mb, ml);
            const uint32_t cv = code >= 0 && code <= 2 ? (uint32_t) code : 4u;   // an unrecognised code completes as ERROR
            bool found = false;
            for (uint64_t s = slot_hash(pkg, h) & p.table_mask;; s = (s + 1) & p.table_mask) {
                const unsigned long long key = p.slot_key[s];
                if (key == EMPTY_KEY) break;
                if ((uint32_t) (key >> 32) != pkg) continue;
                const uint32_t e = (uint32_t) key;
                if (p.mi_hash[e] != h) continue;
                const uint8_t* eb;
                uint64_t el;
                entry_body(p, e, &eb, &el);
                bool eq = el == ml;
                for (uint64_t i = 0; eq && i < ml; i++) eq = eb[i] == mb[i];
                if (!eq) continue;
                found = true;
                if (atomicCAS(&p.slot_code[s], CODE_UNSET, cv) != CODE_UNSET) ok = false;   // toMap's duplicate key
                p.slot_rpos[s] = (unsigned long long) ms;
                p.slot_rlen[s] = (uint32_t) ml;
            }
            ok = ok && found;
        }
        if (!ok) p.dl_fail[d] = 1;
    }
}

__global__ void __launch_bounds__(RP_THREADS) rp_status_kernel(const ReplyParams p) {
    const int64_t d = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x;
    if (d >= (int64_t) p.n_deliverers || stopped(p)) return;
    uint8_t s;
    if (!deliverer_sent(p, d)) s = RP_NOT_SENT;
    else if (p.dl_fail[d]) s = RP_UNDECIDED;
    else if (p.dl_code[d] == 0) s = 0;
    else if (p.dl_code[d] == 1) s = 3;
    else s = 4;
    p.status[d] = s;
    if (s == RP_UNDECIDED) atomicAdd(&p.ctr[RP_N_FALLBACK], 1ull);
}

// every pair's code, counted per code; a thread per pack
__global__ void __launch_bounds__(RP_THREADS) rp_pair_kernel(const ReplyParams p) {
    __shared__ unsigned long long cnt[8];
    if (threadIdx.x < 8) cnt[threadIdx.x] = 0;
    __syncthreads();
    const int64_t k = (int64_t) blockIdx.x * RP_THREADS + threadIdx.x;
    if (k < p.n_packs && !stopped(p)) {
        const int64_t g = upper_index(p.pack_off, p.n_packages, k);
        const uint8_t st = p.status[upper_index(p.package_off, p.n_deliverers, g)];
        const long long j0 = p.match_off[k], j1 = p.match_off[k + 1];
        for (long long j = j0; j < j1; j++) {
            uint8_t c = st;
            if (st == 0) {
                const uint32_t v = p.slot_code[p.pair_slot[j]];
                c = v == CODE_UNSET ? RP_NO_RESULT : (uint8_t) v;
            }
            p.pair_code[j] = c;
            atomicAdd(&cnt[c], 1ull);
        }
    }
    __syncthreads();
    if (threadIdx.x < 8 && cnt[threadIdx.x]) atomicAdd(&p.ctr[RP_N_CODE + threadIdx.x], cnt[threadIdx.x]);
}

// the stale keys (NO_SUB / NO_RECEIVER of a resolved deliverer): listed, and counted per package
__global__ void __launch_bounds__(RP_THREADS) rp_stale_list_kernel(const ReplyParams p) {
    if (stopped(p)) return;
    for (uint64_t s = (uint64_t) blockIdx.x * RP_THREADS + threadIdx.x; s <= p.table_mask; s += (uint64_t) gridDim.x * RP_THREADS) {
        const unsigned long long key = p.slot_key[s];
        if (key == EMPTY_KEY) continue;
        const uint32_t c = p.slot_code[s];
        if (c != 1 && c != 2) continue;
        const uint32_t pkg = (uint32_t) (key >> 32);
        if (p.status[upper_index(p.package_off, p.n_deliverers, pkg)] != 0) continue;
        p.stale_list[atomicAdd(&p.ctr[RP_N_STALE], 1ull)] = (uint32_t) s;
        atomicAdd(&p.pkg_stale[pkg], 1ull);
    }
}

// the listed slots placed in their package's segment (pkg_stale scanned), keyed by their entry
__global__ void __launch_bounds__(RP_THREADS) rp_stale_place_kernel(const ReplyParams p) {
    if (stopped(p)) return;
    const unsigned long long n = p.ctr[RP_N_STALE];
    for (unsigned long long i = (unsigned long long) blockIdx.x * RP_THREADS + threadIdx.x; i < n;
         i += (unsigned long long) gridDim.x * RP_THREADS) {
        const uint32_t s = p.stale_list[i];
        const unsigned long long key = p.slot_key[s];
        const unsigned long long at = atomicAdd(&p.pkg_cursor[key >> 32], 1ull);
        p.sort_key_in[at] = (uint32_t) key;
        p.sort_val_in[at] = s;
    }
}

__global__ void __launch_bounds__(RP_THREADS) rp_stale_out_kernel(const ReplyParams p) {
    if (stopped(p)) return;
    const unsigned long long n = p.ctr[RP_N_STALE];
    for (unsigned long long i = (unsigned long long) blockIdx.x * RP_THREADS + threadIdx.x; i < n;
         i += (unsigned long long) gridDim.x * RP_THREADS) {
        const uint32_t s = p.sort_val_out[i];
        const uint32_t pkg = (uint32_t) (p.slot_key[s] >> 32), j = p.slot_pair[s];
        bfq_stale_match m;
        m.deliverer = (int32_t) upper_index(p.package_off, p.n_deliverers, pkg);
        m.tenant = (int32_t) p.package_tenant[pkg];
        m.rank = p.match_rank[j];
        m.member = p.match_member[j];
        m.reply_off = (int64_t) p.slot_rpos[s];
        m.reply_len = (int32_t) p.slot_rlen[s];
        m.code = (int32_t) p.slot_code[s];
        p.stale[i] = m;
    }
}

unsigned rp_blocks(int64_t n) { return (unsigned) std::max<int64_t>(1, (n + RP_THREADS - 1) / RP_THREADS); }

}  // namespace

cudaError_t launch_mi_hash(const uint8_t* bytes, const unsigned long long* off, int64_t n_entries, uint32_t* out, cudaStream_t stream) {
    if (n_entries > 0) mi_hash_kernel<<<rp_blocks(n_entries), RP_THREADS, 0, stream>>>(bytes, off, n_entries, out);
    return cudaGetLastError();
}

cudaError_t launch_reply(const ReplyParams& p, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    const int64_t np = p.n_packages;
    if (!d_tmp) {
        size_t a = 0, b = 0;
        cudaError_t err = cub::DeviceScan::ExclusiveSum(nullptr, a, p.chunk_base, np + 1, stream);
        if (err != cudaSuccess) return err;
        if (np > 0)
            err = cub::DeviceSegmentedSort::SortPairs(nullptr, b, p.sort_key_in, p.sort_key_out, p.sort_val_in, p.sort_val_out,
                                                      std::max<int64_t>(p.stale_cap, 1), np, p.pkg_stale, p.pkg_stale + 1, stream);
        if (err != cudaSuccess) return err;
        *tmp_bytes = std::max(a, b);
        return cudaSuccess;
    }
    cudaError_t err;
    if ((err = cudaMemsetAsync(p.ctr, 0, RP_CTR_N * sizeof(unsigned long long), stream)) != cudaSuccess) return err;
    if ((err = cudaMemsetAsync(p.slot_key, 0xFF, (p.table_mask + 1) * sizeof(unsigned long long), stream)) != cudaSuccess) return err;
    if ((err = cudaMemsetAsync(p.pkg_claimed, 0, std::max<int64_t>(np, 1) * sizeof(uint32_t), stream)) != cudaSuccess) return err;
    if ((err = cudaMemsetAsync(p.ent_bad, 0, std::max<int64_t>(np, 1), stream)) != cudaSuccess) return err;
    if ((err = cudaMemsetAsync(p.pkg_stale, 0, (np + 1) * sizeof(unsigned long long), stream)) != cudaSuccess) return err;
    rp_check_kernel<<<rp_blocks(p.n_deliverers), RP_THREADS, 0, stream>>>(p);
    rp_insert_kernel<<<rp_blocks(p.n_packs), RP_THREADS, 0, stream>>>(p);
    rp_top_kernel<<<rp_blocks(p.n_deliverers), RP_THREADS, 0, stream>>>(p);
    rp_entry_kernel<<<rp_blocks(np * 32), RP_THREADS, 0, stream>>>(p);
    rp_chunk_count_kernel<<<rp_blocks(np + 1), RP_THREADS, 0, stream>>>(p);
    size_t bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, p.chunk_base, np + 1, stream)) != cudaSuccess) return err;
    rp_guess_kernel<<<RP_GRID, RP_THREADS, 0, stream>>>(p);
    rp_fix_kernel<<<rp_blocks(np * 32), RP_THREADS, 0, stream>>>(p);
    rp_decode_kernel<<<RP_GRID, RP_THREADS, 0, stream>>>(p);
    rp_status_kernel<<<rp_blocks(p.n_deliverers), RP_THREADS, 0, stream>>>(p);
    rp_pair_kernel<<<rp_blocks(p.n_packs), RP_THREADS, 0, stream>>>(p);
    rp_stale_list_kernel<<<RP_GRID, RP_THREADS, 0, stream>>>(p);
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, p.pkg_stale, np + 1, stream)) != cudaSuccess) return err;
    if ((err = cudaMemcpyAsync(p.pkg_cursor, p.pkg_stale, (np + 1) * sizeof(unsigned long long), cudaMemcpyDeviceToDevice,
                               stream)) != cudaSuccess)
        return err;
    rp_stale_place_kernel<<<RP_GRID, RP_THREADS, 0, stream>>>(p);
    bytes = *tmp_bytes;
    if (np > 0 && (err = cub::DeviceSegmentedSort::SortPairs(d_tmp, bytes, p.sort_key_in, p.sort_key_out, p.sort_val_in, p.sort_val_out,
                                                   std::max<int64_t>(p.stale_cap, 1), np, p.pkg_stale, p.pkg_stale + 1, stream)) !=
        cudaSuccess)
        return err;
    rp_stale_out_kernel<<<RP_GRID, RP_THREADS, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace bfq
