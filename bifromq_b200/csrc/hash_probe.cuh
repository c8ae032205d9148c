// hash_probe.cuh — device-side lookup in the tag-filtered blocked edge table (layout: trie_layout.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "trie_layout.h"

namespace bfq {

// kNA: bypass L1 allocation (ld.global.nc.L1::no_allocate) — node records are touched once per walk, keeping them out
// of L1 leaves it to the topic bytes / tenant roots that every step re-reads
template <bool kNA>
__device__ __forceinline__ uint4 ld16(const uint4* p) {
    if (kNA) {
        uint4 v;
        asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
        return v;
    }
    return __ldg(p);
}

// One 32-byte sector as two 16-byte loads (LDG.E.128 is the widest global load sm_90 has). Both halves are issued before
// either is used, so a lane still waits one memory round trip per sector.
template <bool kNA>
__device__ __forceinline__ void ld32(const void* p, uint32_t* w) {
    const uint4* q = reinterpret_cast<const uint4*>(p);
    const uint4 a = ld16<kNA>(q), b = ld16<kNA>(q + 1);
    w[0] = a.x; w[1] = a.y; w[2] = a.z; w[3] = a.w;
    w[4] = b.x; w[5] = b.y; w[6] = b.z; w[7] = b.w;
}

template <bool kNA = false>
__device__ __forceinline__ void load_slot(const Slot* s, uint32_t (&w)[16]) {
    ld32<kNA>(s, &w[0]);
    ld32<kNA>(reinterpret_cast<const uint8_t*>(s) + 32, &w[8]);
}

// payload half only (words 8..15): a '+' child or a tenant root is addressed directly, its key words are not needed —
// one 32-byte sector instead of two
template <bool kNA = false>
__device__ __forceinline__ void load_payload(const Slot* s, uint32_t (&w)[16]) {
    ld32<kNA>(reinterpret_cast<const uint8_t*>(s) + 32, &w[8]);
}

// bytes of w equal to fp -> 0x80 in that byte (SWAR zero-byte test; it can also flag a byte just above a true
// match — such a false candidate only costs one extra slot compare, a true match is never missed)
__device__ __forceinline__ uint32_t match_bytes(uint32_t w, uint32_t fp4) {
    const uint32_t y = w ^ fp4;
    return (y - 0x01010101u) & ~y & 0x80808080u;
}

// 0x80 flags in bytes 0..3 -> bits 0..3
__device__ __forceinline__ uint32_t nibble(uint32_t m) {
    return ((m >> 7) & 1u) | ((m >> 14) & 2u) | ((m >> 21) & 4u) | ((m >> 28) & 8u);
}

// Lookup of the edge (parent, lenw, k[0..5]). On success `w` holds the child record and `slot` its index.
template <bool kNA = false>
__device__ __forceinline__ bool probe(const Slot* slots, const uint4* tags, uint32_t n_blocks, uint32_t parent, uint32_t lenw,
                                      const uint32_t (&k)[6], uint64_t tokh, uint32_t (&w)[16], uint32_t& slot) {
    const uint64_t h = edge_hash(tokh, parent);
    uint32_t b = home_block(h, n_blocks);
    const uint32_t fp4 = fingerprint(h) * 0x01010101u;
    while (true) {
        const uint4 tg = __ldg(tags + b);
        // 16-bit candidate mask over the block's tags (bit j = tag j matches); byte 15 is the control byte.
        // All candidates are then tried from ONE loop so that every lane's slot load is issued at the same place
        // (a per-word candidate loop serialises the lanes by the word their match sits in: 4 HBM round trips).
        uint32_t cand = nibble(match_bytes(tg.x, fp4)) | (nibble(match_bytes(tg.y, fp4)) << 4) |
                        (nibble(match_bytes(tg.z, fp4)) << 8) | (nibble(match_bytes(tg.w & 0x00FFFFFFu, fp4)) << 12);
        cand &= 0x7FFFu;
        while (cand) {
            const uint32_t j = __ffs(cand) - 1;
            cand &= cand - 1;
            const uint32_t s = b * BLOCK_SLOTS + j;
            load_slot<kNA>(slots + s, w);
            if (w[W_PARENT] == parent && w[W_LEN] == lenw && w[2] == k[0] && w[3] == k[1] && w[4] == k[2] &&
                w[5] == k[3] && w[6] == k[4] && w[7] == k[5]) {
                slot = s;
                return true;
            }
        }
        if ((tg.w >> 24) == 0) return false;   // the block never overflowed: the edge does not exist
        b = b + 1 == n_blocks ? 0 : b + 1;
    }
}

// Exact child of a node described by (a, meta): a = the node id for BIG nodes (global tag table), else the base of the
// node's private child array (perfect hash: one access, hit or miss; single-child nodes filter by fingerprint first).
template <bool kNA = false>
__device__ __forceinline__ bool find_child(const Slot* slots, const uint4* tags, uint32_t n_blocks, uint32_t a, uint32_t meta,
                                           uint32_t lenw, const uint32_t (&k)[6], uint64_t tokh, uint32_t (&w)[16], uint32_t& slot) {
    if (meta & FLAG_BIG) return probe<kNA>(slots, tags, n_blocks, a, lenw, k, tokh, w, slot);
    const uint32_t lg = meta_log2size(meta), sd = meta >> 16, t32 = fold32(tokh);
    uint32_t idx = 0;
    if (lg == 0) {
        if ((t32 & 0xFFFFu) != sd) return false;
    } else {
        idx = child_index(t32, sd, lg);
    }
    slot = a + idx;
    load_slot<kNA>(slots + slot, w);
    return w[W_PARENT] != EMPTY_PARENT && w[W_LEN] == lenw && w[2] == k[0] && w[3] == k[1] && w[4] == k[2] && w[5] == k[3] &&
           w[6] == k[4] && w[7] == k[5];
}

// 15-bit candidate mask over a block's tags (bit j = tag j equals the fingerprint); byte 15 is the control byte
__device__ __forceinline__ uint32_t tag_candidates(const uint4& tg, uint32_t fp4) {
    return (nibble(match_bytes(tg.x, fp4)) | (nibble(match_bytes(tg.y, fp4)) << 4) | (nibble(match_bytes(tg.z, fp4)) << 8) |
            (nibble(match_bytes(tg.w & 0x00FFFFFFu, fp4)) << 12)) & 0x7FFFu;
}

// find_child for a warp whose lanes sit on different kinds of nodes (the lane-per-topic kernel). A plain
// `big ? probe : perfect-hash` branch serialises the two sides: the BIG lanes' tag read and slot read, THEN the other lanes'
// slot read — three dependent memory round trips per warp step.
// Here phase 1 is the BIG lanes' tag read only (16 bytes, L2-resident window), and phase 2 is ONE slot read issued by every
// lane at the same instruction, whatever kind of node it is on; second candidates / overflowed blocks (rare) loop afterwards.
template <bool kNA = false>
__device__ __forceinline__ bool find_child_lanes(const Slot* slots, const uint4* tags, uint32_t n_blocks, bool alive, uint32_t a,
                                                 uint32_t meta, uint32_t lenw, const uint32_t (&k)[6], uint64_t tokh,
                                                 uint32_t (&w)[16], uint32_t& slot) {
    const bool big = alive && (meta & FLAG_BIG);
    bool want = false, hit = false, chain = false;
    uint32_t cand = 0, b = 0, fp4 = 0;
    if (big) {
        const uint64_t h = edge_hash(tokh, a);
        b = home_block(h, n_blocks);
        fp4 = fingerprint(h) * 0x01010101u;
        const uint4 tg = __ldg(tags + b);
        cand = tag_candidates(tg, fp4);
        chain = (tg.w >> 24) != 0;
        if (cand) {
            slot = b * BLOCK_SLOTS + (__ffs(cand) - 1);
            cand &= cand - 1;
            want = true;
        }
    } else if (alive) {
        const uint32_t lg = meta_log2size(meta), sd = meta >> 16, t32 = fold32(tokh);
        want = lg != 0 || (t32 & 0xFFFFu) == sd;
        slot = a + (lg ? child_index(t32, sd, lg) : 0u);
    }
    if (want) {
        load_slot<kNA>(slots + slot, w);
        const bool parent_ok = big ? w[W_PARENT] == a : w[W_PARENT] != EMPTY_PARENT;
        hit = parent_ok && w[W_LEN] == lenw && w[2] == k[0] && w[3] == k[1] && w[4] == k[2] && w[5] == k[3] && w[6] == k[4] &&
              w[7] == k[5];
    }
    while (big && !hit) {
        if (!cand) {
            if (!chain) break;   // the block never overflowed: the edge does not exist
            b = b + 1 == n_blocks ? 0 : b + 1;
            const uint4 tg = __ldg(tags + b);
            cand = tag_candidates(tg, fp4);
            chain = (tg.w >> 24) != 0;
            continue;
        }
        slot = b * BLOCK_SLOTS + (__ffs(cand) - 1);
        cand &= cand - 1;
        load_slot<kNA>(slots + slot, w);
        hit = w[W_PARENT] == a && w[W_LEN] == lenw && w[2] == k[0] && w[3] == k[1] && w[4] == k[2] && w[5] == k[3] &&
              w[6] == k[4] && w[7] == k[5];
    }
    return hit;
}

// the `a` word of a node: what find_child needs to address its children
__device__ __forceinline__ uint32_t child_ref(uint32_t node_id, const uint32_t (&w)[16]) {
    return (w[W_META] & FLAG_BIG) ? node_id : w[W_CHILD_BASE];
}

}  // namespace bfq
