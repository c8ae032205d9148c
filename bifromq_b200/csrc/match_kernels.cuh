// match_kernels.cuh — launch parameters of the forward-match kernels (see match_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "trie_layout.h"

namespace bfq {

// device counters, one block of uint64
enum : int {
    CTR_RANGES = 0,      // cursor into out_ranges (total ranges requested, may exceed capacity)
    CTR_OVERFLOW = 1,    // topics deferred to the tier-2 kernel
    CTR_FLAGGED = 2,     // topics whose matched persistent / group route counts may exceed their caps
    CTR_THROTTLED = 3,   // cursor into the throttled list
    CTR_ROUTES = 4,      // total matched routes (before caps)
    CTR_ERROR = 5,       // tier-2 scratch exhausted (cannot happen with correctly sized scratch)
    CTR_DEFER = 6,       // topics the lane-per-topic tier handed to the warp-per-topic tier
    CTR_CHUNK = 7,       // tier-0 work distribution: next unclaimed topic index
    CTR_NLEAD = 8,       // number of distinct (tenant, topic) pairs of the batch = length of the locality order
    CTR_FLAGGED2 = 9,    // flagged topics already handled by an earlier caps pass (the rare tier-2 path runs a second one)
    CTR_COUNT = 12,
};

constexpr uint32_t SPAN_FLAGGED = 0x80000000u;   // in span_count: caps must be applied to this topic
constexpr uint32_t SPAN_OVERFLOW = 0x40000000u;  // in span_count: deferred to tier 2 (never visible to callers)
constexpr uint32_t SPAN_COUNT_MASK = 0x3FFFFFFFu;

// Tier 0's result for the topic at work-order position i when the batch is ordered (MatchParams::order set), written with one
// 16-byte store to pos_rec[i]: the 32 positions of a chunk are neighbours, so a warp's record writes stay within a few hundred
// bytes instead of scattering 3 x 32 words over the topic-indexed arrays. finalize_kernel gathers the records to topic order.
struct __align__(16) SpanRecord {
    uint32_t span_begin;
    uint32_t span_count;    // count | SPAN_FLAGGED
    uint32_t route_count;
    uint32_t deferred;      // != 0: tier 0 handed the topic to tier 1, which writes the topic-indexed arrays itself
};
static_assert(sizeof(SpanRecord) == 16, "a span record is one 16-byte store");

struct MatchParams {
    // index snapshot
    const Slot* slots;              // blocked edge table (trie_layout.h)
    const uint4* tags;              // one 16-byte tag word per block
    const Slot* roots;
    uint32_t n_blocks;
    // topic batch
    const uint8_t* topics;          // blob
    const int64_t* topic_off;       // [n+1]
    const int32_t* topic_tenant;    // [n] index into the per-call tenant tables
    const int32_t* tenant_root;     // [n_tenants] root ordinal or -1 (tenant has no routes)
    const int32_t* max_pfanout;     // [n_tenants]
    const int32_t* max_gfanout;     // [n_tenants]
    int32_t n_tenants;
    int64_t n_topics;
    // tier 0: optional processing order (topic indices grouped by tenant and leading levels, see launch_order); nullptr =>
    // 0..n_topics. With an order, tier 0 writes a topic's span record at its position in the order (pos_rec) and leaves the
    // topic-indexed span_begin / span_count / route_count to finalize_kernel; without one it writes those three directly.
    // Tiers 1 and 2 always write the topic-indexed arrays.
    const uint32_t* order;
    const unsigned long long* order_count;   // device scalar: entries of `order` (the batch's distinct topics); with order only
    SpanRecord* pos_rec;                     // [n] with order only: tier 0's record of the topic at each position
    int32_t max_ctas_per_sm;        // tier 0: cap of resident CTAs per SM (0 = as many as fit); one slot less leaves room for a
                                    // concurrently running exchange (NCCL) kernel
    // tiers 1/2: list of topic indices to process (nullptr => all topics 0..n_topics)
    const uint32_t* work_list;
    int64_t n_work;
    // outputs
    uint32_t* span_begin;           // [n]
    uint32_t* span_count;           // [n]  count | SPAN_FLAGGED
    uint32_t* route_count;          // [n]
    uint2* ranges;                  // [ranges_cap] {first, count | RANGE_MULTI}
    uint64_t ranges_cap;
    uint64_t dyn_base;              // ranges[0, dyn_base) = tier-0 inline slots (INLINE_RANGES per topic); the cursor
                                    // CTR_RANGES allocates from ranges[dyn_base, ranges_cap) for tiers 1 and 2
    uint32_t* overflow_list;        // [n] topic indices deferred to tier 2
    uint32_t* defer_list;           // [n] topic indices deferred from tier 0 to tier 1
    uint32_t* flagged_list;         // [n] topic indices needing caps
    unsigned long long* counters;   // [CTR_COUNT]
    // tier-2 scratch (global memory frontier / range staging), per warp
    uint2* scratch;
    uint64_t scratch_frontier_cap;  // entries per frontier buffer
    uint64_t scratch_ranges_cap;    // entries of range staging
};

struct CapsParams {
    const uint32_t* flagged_list;
    int64_t n_flagged;              // < 0: flagged_list[counters[CTR_FLAGGED2] ... counters[CTR_FLAGGED]) (counts read on the device)
    const int32_t* topic_tenant;
    const int32_t* max_pfanout;
    const int32_t* max_gfanout;
    const uint32_t* span_begin;
    const uint32_t* span_count;
    const uint2* ranges;
    const uint32_t* segs;
    const uint8_t* rkind;
    const uint32_t* pfx_persistent;
    const uint32_t* pfx_group;
    uint3* throttled;               // {topic, rank, kind}
    uint32_t topic_base;            // added to the (sub-batch relative) topic index
    uint64_t throttled_cap;
    uint32_t* kept_count;           // [n] (optional) routes surviving per flagged topic
    unsigned long long* counters;
};

struct ExpandParams {
    int64_t n_topics;
    const uint32_t* span_begin;
    const uint32_t* span_count;     // with SPAN_FLAGGED bits
    const uint32_t* route_count;    // matched routes before caps
    const uint32_t* kept_count;     // surviving routes of cap-flagged topics (written by the caps kernel)
    const uint2* ranges;            // sparse
    const uint32_t* segs;
    unsigned long long* counts;     // scratch [n+1]
    int64_t* offsets;               // out [n+1]
    int64_t* ranks;                 // out
    int64_t rank_cap;
    // caps inputs for the flagged topics
    const uint32_t* flagged_list;
    int64_t n_flagged;
    const int32_t* topic_tenant;
    const int32_t* max_pfanout;
    const int32_t* max_gfanout;
    const uint8_t* rkind;
    const uint32_t* pfx_persistent;
    const uint32_t* pfx_group;
};
// device CSR of the surviving routes: phase 1 = per-topic counts + exclusive scan into offsets (offsets[n] = total),
// phase 2 = write the ranks (unordered within a topic). tmp as for launch_compact.
cudaError_t launch_expand(const ExpandParams& p, void* d_scan_tmp, size_t* tmp_bytes, cudaStream_t stream, int phase);

// Delivery budgets of DeliverExecutorGroup.submit on top of the expand (bfq_expand_device_budget): per topic a tighter
// persistent cap k (MaxPersistentFanoutBytes, persistent bandwidth) and an on/off switch for transient routes.
enum : uint8_t {
    BUDGET_BYTES_THROTTLED = 1,      // k < P persistent routes delivered: PersistentFanoutBytesThrottled
    BUDGET_NO_PERSISTENT_BW = 2,     // persistent routes dropped: OutOfTenantResource(TotalPersistentFanOutBytesPerSeconds)
    BUDGET_NO_TRANSIENT_BW = 4,      // transient routes dropped: OutOfTenantResource(TotalTransientFanOutBytesPerSeconds)
    BUDGET_METERED = 8,              // the topic records MqttPersistentFanOutBytes (|R| > 1, or one persistent route)
    BUDGET_DROPS = 7,                // any of the first three: the topic's survivors are copied rank by rank
};
enum : int {
    BUD_LISTED = 0,                  // topics in BudgetParams::list
    BUD_BAD_SIZE = 1,                // topics with a negative message size
    BUD_DROP_BYTES = 2,              // persistent routes dropped by the bytes budget
    BUD_DROP_PBW = 3,                // ... by the persistent bandwidth switch
    BUD_DROP_TBW = 4,                // transient routes dropped by the transient bandwidth switch
    BUD_CTR_COUNT = 8,
};
struct BudgetParams {
    ExpandParams e;                  // the match's CSR inputs and the expand's outputs (e.counts / e.offsets / e.ranks)
    int32_t n_tenants;
    const int32_t* msg_bytes;        // [n_topics] message size of each topic position
    const long long* max_bytes;      // [n_tenants] MaxPersistentFanoutBytes (> 0)
    const uint8_t* bandwidth;        // [n_tenants] bit 0: persistent bandwidth, bit 1: transient bandwidth
    uint32_t* delivered_p;           // out [n_topics] persistent routes delivered (k)
    uint8_t* flags;                  // out [n_topics] BUDGET_* bits
    uint32_t* list;                  // out: topics with a BUDGET_DROPS bit
    int64_t n_listed;                // phase 2: entries of list (read back after phase 1)
    unsigned long long* ctr;         // [BUD_CTR_COUNT], zeroed before phase 1
};
// phase 1 = budget pass (counts, flags, list) + exclusive scan into e.offsets; phase 2 = write the delivered ranks
cudaError_t launch_budget(const BudgetParams& q, void* d_scan_tmp, size_t* tmp_bytes, cudaStream_t stream, int phase);

// Locality ordering + de-duplication for tier 0, all own kernels (no library sort):
//   prep     one thread per topic: 64-bit hash of (tenant, topic bytes) -> insert into an open-addressing table; the first
//            inserter of a (tenant, topic) pair is its LEADER, later identical ones (verified byte by byte) are followers that
//            only remember their leader. Leaders get an order key = tenant index | hashes of the level-0 / 0..1 / 0..2 prefixes
//            and count themselves into a bucket histogram (bucket = the key's leading bits).
//   scan     exclusive prefix sum of the histogram (block-local scans; the last block to finish scans the block totals)
//   scatter  leaders -> order[bucket base + atomic cursor]: a counting sort, unstable inside a bucket (only grouping matters);
//            each leader's position goes back to keys[leader] for finalize_kernel
// Tier 0 then matches order[0 .. n_leaders) — topics that walk the same top of the trie are matched by neighbouring lanes at
// the same time — and finalize_kernel gathers tier 0's span records back to topic order, giving each follower its leader's
// span (spans are indices into the sparse range array, so no range is copied). The reference never sees duplicates
// (matchAll takes a Set<String>, DW/cache/ITenantRouteMatcher.java:28-38; DW/cache/TenantRouteCache.java:100-139 serves
// repeats from its cache).
struct OrderParams {
    int64_t n_topics;
    const uint8_t* topics;
    const int64_t* topic_off;
    const int32_t* topic_tenant;
    int32_t n_tenants;
    uint32_t* keys;                 // [n] bucket of each leader; after the scatter: the leader's position in `order`
    uint32_t* leader;               // [n] out: i for a leader, else the index of the identical topic that leads
    uint32_t* order;                // [n] out: the leaders, grouped by bucket
    unsigned long long* hash_tab;   // [hash_mask + 1], filled with 0xFF bytes by launch_order when dedup is set
    uint32_t hash_mask;
    uint32_t* hist;                 // [order_scratch_words(n_topics, n_tenants)] scratch, zeroed and laid out by launch_order
    int dedup;                      // 0: every topic is its own leader
    uint64_t dedup_hash_mask;       // bits of the de-dup hash kept after fmix64 (all of them but in tests: forced collisions)
    unsigned long long* counters;   // CTR_NLEAD is written by the scan
};
size_t order_scratch_words(int64_t n_topics, int32_t n_tenants);   // 32-bit words of scratch launch_order needs
uint32_t order_hash_entries(int64_t n_topics);                     // dedup table entries (power of two)
// enqueues the scratch and hash-table fills and the three kernels on stream
cudaError_t launch_order(const OrderParams& q, cudaStream_t stream);

// Runs behind tiers 0 and 1 of every ordered batch. First pass: every topic takes its leader's span record from tier 0's
// position records (a repeat of a flagged record also joins the flagged list); a repeat of a leader that tier 0 deferred copies
// the leader's topic-indexed span, which tier 1 wrote. second_pass: only the repeats whose span still carries the tier-2 marker
// (their leader was finished by tier 2 after the first pass) copy it again.
struct FinalizeParams {
    int64_t n_topics;
    const uint32_t* leader;
    const uint32_t* pos;            // [n] OrderParams::keys after launch_order: position of each leader in the order
    const SpanRecord* pos_rec;      // MatchParams::pos_rec
    uint32_t* span_begin;
    uint32_t* span_count;
    uint32_t* route_count;
    uint32_t* flagged_list;
    unsigned long long* counters;
    int second_pass;
};
void launch_finalize(const FinalizeParams& p, cudaStream_t stream);

// tier 0: one LANE per topic (DFS, bounded smem); tier 1: one WARP per topic; tier 2: warp per topic, global scratch
void launch_match_lanes(const MatchParams& p, cudaStream_t stream);
void launch_match(const MatchParams& p, bool tier2, int n_warps_tier2, cudaStream_t stream);
void launch_caps(const CapsParams& p, cudaStream_t stream);

constexpr uint32_t INLINE_RANGES = 12;   // tier 0 writes the ranges of the topic at work-order position i at ranges[i * INLINE_RANGES ...)
constexpr uint32_t SPILL_RANGES = 64;    // ... and moves a topic with more of them, once, to a block of this many ranges
// Tier 0 writes its ranges one whole 32-byte sector (two 16-byte stores) at a time, so the inline runs and the spill blocks
// start on sector boundaries: ranges[0] is 256-byte aligned, INLINE_RANGES and SPILL_RANGES are multiples of RANGE_SECTOR, and
// the host cuts the cursor-allocated region into sub-batch slices of whole spill blocks.
constexpr uint32_t RANGE_SECTOR = 4;
static_assert(INLINE_RANGES % RANGE_SECTOR == 0 && SPILL_RANGES % RANGE_SECTOR == 0, "tier 0 writes whole 32-byte sectors");

// Compaction for the host path: gathers the sparse (inline + dynamic) ranges into one dense array in topic order.
// d_scan_tmp / tmp_bytes: scratch for the exclusive scan (query the size with d_scan_tmp == nullptr).
struct CompactParams {
    int64_t n_topics;
    const uint32_t* span_begin;     // in
    const uint32_t* span_count;     // in (flag bits allowed)
    const uint2* ranges;            // in
    const uint32_t* leader;         // optional [n]: leader[i] != i marks a repeat of topic leader[i] (shares its dense span)
    uint32_t* counts;               // scratch [n]
    uint32_t* new_begin;            // scratch [n]: exclusive scan of counts
    uint32_t* final_begin;          // out [n] (phase 2): first range of topic i in the concatenated result
    uint32_t* final_count;          // out [n] (phase 2): its number of ranges
    uint2* ranges_out;              // out [total]
    uint64_t ranges_out_cap;
    uint32_t out_base;              // index of ranges_out[0] in the concatenated result (added to new_begin in phase 2)
    unsigned long long* total_out;  // device scalar: total number of ranges (phase 1)
};
// phase 1: counts + exclusive scan + total; phase 2: gather (after the caller has read the total and placed ranges_out)
cudaError_t launch_compact(const CompactParams& p, void* d_scan_tmp, size_t* tmp_bytes, cudaStream_t stream, int phase);
int match_kernel_smem_bytes();
int device_sm_count();   // SMs of the current device (cached per ordinal): sizes the fixed and persistent grids

// bfq_index_commit's delta path: the records of the tenants BEHIND a tenant that grew or shrank carry dense KV ranks, so
// their own / '#' first-rank words move by the difference. One streaming pass over the listed slot regions.
struct RankShiftRegion {
    uint64_t base, len;     // slots [base, base + len)
    int32_t delta;
};
void launch_rank_shift(Slot* slots, const RankShiftRegion* d_regions, int n_regions, cudaStream_t stream);
// the same rule for single slots: the tag-table records (children of wide nodes) of those tenants
struct RankShiftSlot {
    uint32_t slot;
    int32_t delta;
};
void launch_rank_shift_listed(Slot* slots, const RankShiftSlot* d_list, int64_t n, cudaStream_t stream);
// slots[ids[i]] = recs[i]: the tag-table records of the tenants a delta commit rebuilt
void launch_scatter_records(Slot* slots, const uint32_t* d_ids, const Slot* d_recs, int64_t n, cudaStream_t stream);
// The per-rank arrays (rkind and the two prefix counts) of a delta commit's new snapshot, all ranks in one launch. The ranks
// are cut into runs sorted by new rank that tile [0, n): a run of untouched tenants is read from the old snapshot's arrays, a
// run of rebuilt tenants from the packed upload; the prefix counts of a run move by (dP, dG) (mod 2^32, like the counts).
struct RankRun {
    uint32_t new_lo, len;   // new ranks [new_lo, new_lo + len)
    uint32_t src_lo;        // first rank of the run in its source
    uint32_t packed;        // 1: the packed upload, 0: the old snapshot
    uint32_t dP, dG;
};
struct AssembleRankParams {
    uint8_t* rkind;                                 // out [n]
    uint32_t *pfxP, *pfxG;                          // out [n + 1]
    const uint8_t* old_rkind;                       // the old snapshot's arrays
    const uint32_t *old_pfxP, *old_pfxG;
    const uint8_t* up_rkind;                        // the rebuilt tenants' arrays, packed in new-rank order
    const uint32_t *up_pfxP, *up_pfxG;
    const RankRun* runs;
    int32_t n_runs;
    int64_t n;
    uint32_t tailP, tailG;                          // pfxP[n], pfxG[n]: the totals
};
void launch_assemble_rank_arrays(const AssembleRankParams& p, cudaStream_t stream);

}  // namespace bfq
