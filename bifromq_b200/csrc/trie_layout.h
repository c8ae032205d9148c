// trie_layout.h — HBM layout of the forward index, shared by the host builder and the kernels.
//
// The per-tenant filter tries are flattened into ONE hash table of 64-byte slots keyed by (parent node id,
// level token). A slot is the child NODE RECORD itself, so following an exact edge costs a single 64 B
// (two 32 B sectors) random access and no separate node fetch. Node id == slot index; tenant roots live in
// a small side array (id = ROOT_BASE + ordinal).
//
// Exact children are found in one of two ways, chosen per parent node at build time:
//   * SMALL fan-out (<= 16 exact children; > 90 % of all nodes have exactly one): the children sit in a private,
//     contiguous array of 2^k slots right in the slot array (CSR), addressed by a per-node PERFECT HASH:
//     slot = child_base + ((fold32(token hash) ^ seed * C1) * C2 >> (32 - k)); the parent record carries child_base,
//     k and the 16-bit seed (found by search at build time). A lookup is ONE 64 B access, hit or miss, no probing;
//     a single-child node stores a 16-bit fingerprint instead of a seed, so most misses cost no access at all.
//   * BIG fan-out: the global blocked, tag-filtered table below, keyed by (parent id, token).
//
// The global table is BLOCKED and TAG-FILTERED (Swiss-table style): slots are grouped in blocks of 16 (15 usable),
// and a parallel 16-byte tag word per block holds one fingerprint byte per slot (0 = free, 2..255 = fingerprint
// of the slot's key) plus a control byte (byte 15: 1 = the block overflowed into the next one). An edge hashes
// to ONE block; a lookup loads that block's 16 tags (the tag array is ~1/64 of the table and mostly L2
// resident), SWAR-compares them with the key's fingerprint and loads only the slot(s) whose tag matches:
//   hit  = 1 tag load (L2) + 1 slot load (HBM);  miss = 1 tag load, NO slot load (3% false positives);
// and — what matters for one-lane-per-topic SIMT — the number of dependent memory round trips per lookup is
// constant. (Linear probing over the slots themselves makes a warp step wait for its longest probe chain: several
// serial HBM round trips with most lanes idle.)
//
//   word  0      parent node id              (EMPTY_PARENT = free slot)
//   word  1      token length in bytes       (LEN_PLUS for the '+' child, LEN_CONT|j for the j-th
//                                             24-byte continuation chunk of a token longer than 24 B)
//   words 2..7   token bytes, zero padded    (exact compare: no hash collisions by construction)
//   word  8      slot of the '+' child       (NONE if absent)
//   word  9      child_base                  (first slot of the private child array; unused for BIG nodes)
//   words 10,11  own routes  [first rank, count)   routes of the filter ending at this node
//   words 12,13  '#' routes  [first rank, count)   routes of the filter "<this node>/#" ('#' is always the
//                                                   last level, so the '#' child is inlined into its parent)
//   word  14     caps counters, one saturating byte each: own persistent (subBrokerId==1), own group,
//                '#' persistent, '#' group   (255 = "255 or more": the exact caps kernel decides)
//   word  15     meta: bits 0-7 flags (HAS_EXACT, OWN_MULTI, HASH_MULTI, BIG), bits 8-11 k = log2(child array
//                size), bits 16-31 perfect-hash seed (k >= 1) or the only child's fingerprint (k == 0)
//
// A rank is the position of a route in the committed KV order (the reference's RocksDB order), so a
// filter's routes are one contiguous run [first, first+count) — except in the rare interleaving case
// (filters with an empty level after a common prefix, see DESIGN.md) where the run is split; then the
// *_MULTI flag is set, `count` still holds the total number of routes and `first` indexes the segment
// table: segs[first] = {n_segments, total}, followed by n_segments {first rank, count} pairs.
#pragma once
#include <stdint.h>

namespace bfq {

struct alignas(64) Slot {
    uint32_t w[16];
};
static_assert(sizeof(Slot) == 64, "slot must be one 64-byte burst");

enum : uint32_t {
    W_PARENT = 0, W_LEN = 1, W_TOK = 2, W_PLUS = 8, W_CHILD_BASE = 9,
    W_OWN_FIRST = 10, W_OWN_COUNT = 11, W_HASH_FIRST = 12, W_HASH_COUNT = 13, W_CAPS = 14, W_META = 15,
};
constexpr uint32_t EMPTY_PARENT = 0xFFFFFFFFu;
constexpr uint32_t NONE = 0xFFFFFFFFu;
constexpr uint32_t LEN_PLUS = 0xFFFFFFFFu;
constexpr uint32_t LEN_CONT = 0x80000000u;       // | chunk index
constexpr uint32_t ROOT_BASE = 0x80000000u;      // node id of tenant root = ROOT_BASE + tenant ordinal
constexpr uint32_t FLAG_HAS_EXACT = 1u, FLAG_OWN_MULTI = 2u, FLAG_HASH_MULTI = 4u, FLAG_BIG = 8u;
constexpr uint32_t PERFECT_LOG2_MAX = 16;       // largest private (perfect-hashed) child array: 2^16 slots; a fan-out whose
                                                //   array would be larger (> ~1000 children) goes to the global tag table
constexpr uint32_t TOKEN_WORDS = 6;              // 24 inline token bytes per edge
constexpr uint32_t TOKEN_BYTES = 24;
constexpr uint32_t RANGE_MULTI = 0x80000000u;    // marker in an emitted range's count word

// Hash of an edge key. tokh covers (length word, 6 token words); the parent id is mixed in afterwards so
// the per-level token hash is computed once per topic level and reused for every frontier node.
#if defined(__CUDACC__)
#define BFQ_HD __host__ __device__ __forceinline__
#else
#define BFQ_HD inline
#endif

BFQ_HD uint64_t fmix64(uint64_t k) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
}
BFQ_HD uint64_t token_hash(uint32_t lenw, const uint32_t* k /*[6]*/) {
    uint64_t h = (uint64_t) lenw * 0x9E3779B97F4A7C15ull;
    h += (uint64_t) k[0] * 0xA24BAED4963EE407ull;
    h += (uint64_t) k[1] * 0x9FB21C651E98DF25ull;
    h += (uint64_t) k[2] * 0xD6E8FEB86659FD93ull;
    h += (uint64_t) k[3] * 0xCA5A826395121157ull;
    h += (uint64_t) k[4] * 0x8CB92BA72F3D8DD7ull;
    h += (uint64_t) k[5] * 0xE7037ED1A0B428DBull;
    return h;
}
constexpr uint32_t BLOCK_SLOTS = 16;     // slots per block (slot 15 of every block is never used)
constexpr uint32_t BLOCK_USABLE = 15;
constexpr uint32_t TAG_CTRL = 15;        // control byte index inside the 16-byte tag word

// per-node perfect hash over the 32-bit fold of the token hash
BFQ_HD uint32_t fold32(uint64_t tokh) { return (uint32_t) (tokh ^ (tokh >> 32)); }
BFQ_HD uint32_t child_index(uint32_t t32, uint32_t seed, uint32_t log2size) {   // log2size >= 1
    return ((t32 ^ (seed * 0x9E3779B9u)) * 0x85EBCA6Bu) >> (32u - log2size);
}
BFQ_HD uint32_t meta_pack(uint32_t flags, uint32_t log2size, uint32_t seed) { return (flags & 0xFFu) | ((log2size & 31u) << 8) | (seed << 16); }
BFQ_HD uint32_t meta_log2size(uint32_t meta) { return (meta >> 8) & 31u; }

BFQ_HD uint64_t edge_hash(uint64_t tokh, uint32_t parent) { return fmix64(tokh + (uint64_t) parent * 0xC2B2AE3D27D4EB4Full); }
BFQ_HD uint32_t home_block(uint64_t h, uint32_t n_blocks) { return (uint32_t) (((h >> 32) * (uint64_t) n_blocks) >> 32); }
BFQ_HD uint32_t fingerprint(uint64_t h) {
    const uint32_t f = (uint32_t) (h & 0xFFu);
    return f < 2u ? f + 2u : f;          // 0 = free slot, 1 is reserved for the control byte
}

}  // namespace bfq

// ---- host-side placement shared by the forward and the inverse index builders
#include <memory>
#include <utility>
#include <vector>
namespace bfq {
// std::vector allocator that leaves trivially-constructible elements uninitialised on resize(): the 64-byte slot array is
// gigabytes at full size and is filled (and its pages first touched) by the builder's worker threads instead.
template <typename T>
struct NoInitAlloc : std::allocator<T> {
    template <typename U> struct rebind { using other = NoInitAlloc<U>; };
    NoInitAlloc() = default;
    template <typename U> NoInitAlloc(const NoInitAlloc<U>&) {}
    template <typename U> void construct(U* p) noexcept { ::new ((void*) p) U; }
    template <typename U, typename... A> void construct(U* p, A&&... a) { ::new ((void*) p) U(std::forward<A>(a)...); }
};
using SlotVec = std::vector<Slot, NoInitAlloc<Slot>>;

inline void fill_empty_slots(Slot* s, size_t n) {
    for (size_t i = 0; i < n; i++) {
        for (auto& w : s[i].w) w = 0;
        s[i].w[W_PARENT] = EMPTY_PARENT;
    }
}

struct EdgeTable {
    SlotVec slots;                  // n_blocks * BLOCK_SLOTS
    std::vector<uint8_t> tags;      // n_blocks * 16
    uint32_t n_blocks = 0;
    int64_t overflowed_blocks = 0;

    // sizes the table; with fill == false the caller resizes `slots` further and fills all of it itself
    void init(uint64_t n_edges, bool fill = true) {
        // target load 0.5 of the usable slots
        uint64_t nb = (n_edges * 2 + BLOCK_USABLE - 1) / BLOCK_USABLE;
        if (nb < 64) nb = 64;
        n_blocks = (uint32_t) nb;
        tags.assign((size_t) n_blocks * 16, 0);
        if (!fill) return;
        slots.resize((size_t) n_blocks * BLOCK_SLOTS);
        fill_empty_slots(slots.data(), slots.size());
    }
    // claims a tag for the edge key and returns its slot index; only the tag array is touched (the caller writes the whole
    // record). The table must have a free usable slot somewhere, or this never returns.
    uint32_t claim(uint32_t parent, uint32_t lenw, const uint32_t* tok) {
        const uint64_t h = edge_hash(token_hash(lenw, tok), parent);
        uint32_t b = home_block(h, n_blocks);
        const uint8_t fp = (uint8_t) fingerprint(h);
        while (true) {
            uint8_t* tg = &tags[(size_t) b * 16];
            for (uint32_t j = 0; j < BLOCK_USABLE; j++) {
                uint8_t expected = 0;   // claim a free tag atomically: tenants are placed by concurrent threads
                if (__atomic_load_n(&tg[j], __ATOMIC_RELAXED) == 0 &&
                    __atomic_compare_exchange_n(&tg[j], &expected, fp, false, __ATOMIC_ACQ_REL, __ATOMIC_RELAXED))
                    return b * BLOCK_SLOTS + j;
            }
            if (__atomic_exchange_n(&tg[TAG_CTRL], (uint8_t) 1, __ATOMIC_ACQ_REL) == 0)
                __atomic_fetch_add(&overflowed_blocks, (int64_t) 1, __ATOMIC_RELAXED);
            b = b + 1 == n_blocks ? 0 : b + 1;
        }
    }
    // claims a slot for the edge key and writes the key words (the caller fills the payload)
    uint32_t place(uint32_t parent, uint32_t lenw, const uint32_t* tok) {
        const uint32_t s = claim(parent, lenw, tok);
        slots[s].w[W_PARENT] = parent;
        slots[s].w[W_LEN] = lenw;
        for (uint32_t k = 0; k < TOKEN_WORDS; k++) slots[s].w[W_TOK + k] = tok[k];
        return s;
    }
    // Frees a claimed slot (a forward delta commit frees the slots of the tenants it replaces or removes, BEFORE it places
    // their new edges). Only the fingerprint byte is cleared; the record behind it stays as it was, and lookups stay exact:
    //   * the control byte of the slot's block is never cleared, so a key that was placed past this block (because the block
    //     was full when it was placed) is still reached: the probe still walks on from here;
    //   * a free tag (0) is never taken for a candidate. Fingerprints are 2..255. The device compares a block's tags four
    //     bytes at a time (match_bytes in hash_probe.cuh: (y - 0x01010101) & ~y & 0x80808080 with y = tags ^ fp), which
    //     flags a byte whose y is 0 (a true match) and, through the borrow of a true match below it, a byte whose y is 1.
    //     For a free tag y = fp >= 2: neither. The host lookup (find) compares bytes exactly;
    //   * so the stale record behind a freed slot is never loaded, even when a rebuilt tenant re-places the very same key (a
    //     root-level edge keeps its key: the tenant keeps its ordinal) into another slot of the probe sequence.
    // A later claim may reuse the slot; the caller then overwrites the whole record.
    void release(uint32_t slot) { tags[slot] = 0; }
    // host-side lookup (self-check only): slot index or NONE
    uint32_t find(uint32_t parent, uint32_t lenw, const uint32_t* tok) const {
        const uint64_t h = edge_hash(token_hash(lenw, tok), parent);
        uint32_t b = home_block(h, n_blocks);
        const uint8_t fp = (uint8_t) fingerprint(h);
        while (true) {
            const uint8_t* tg = &tags[(size_t) b * 16];
            for (uint32_t j = 0; j < BLOCK_USABLE; j++) {
                if (tg[j] != fp) continue;
                const Slot& sl = slots[(size_t) b * BLOCK_SLOTS + j];
                bool eq = sl.w[W_PARENT] == parent && sl.w[W_LEN] == lenw;
                for (uint32_t k = 0; k < TOKEN_WORDS && eq; k++) eq = sl.w[W_TOK + k] == tok[k];
                if (eq) return b * BLOCK_SLOTS + j;
            }
            if (tg[TAG_CTRL] == 0) return NONE;
            b = b + 1 == n_blocks ? 0 : b + 1;
        }
    }
};
}  // namespace bfq
