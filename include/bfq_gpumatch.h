/* bfq_gpumatch.h — C-ABI of the H100 topic-filter matcher (libbfq_gpumatch.so).
 *
 * This is the drop-in boundary: everything a JNI shim needs to put the CUDA matcher behind
 * apache/bifromq's dist-worker / retain-store co-processors without touching their Java API.
 * Nothing native exists in the reference today (it is 100% Java), so each entry point cites the
 * Java interface or call site it replaces. Paths are relative to the reference root; DW/ =
 * bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/, DWS/ =
 * bifromq-dist/bifromq-dist-worker-schema/src/main/java/org/apache/bifromq/dist/worker/schema/,
 * RS/ = bifromq-retain/bifromq-retain-store/src/main/java/org/apache/bifromq/retain/store/,
 * U/ = bifromq-util/src/main/java/org/apache/bifromq/util/.
 *
 * Conventions: every function returns 0 (BFQ_OK) or a negative BFQ_E_* code; bfq_last_error()
 * gives the text. All buffers are caller-owned plain memory (host unless the name says device);
 * strings are (blob, int64 offsets[n+1]) pairs, never NUL-terminated. There is no CPU fallback: every
 * match runs on the GPU and the library fails (BFQ_E_CUDA) if no device is usable.
 *
 * Threading (what ITenantRouteMatcher's callers need: matchAll runs on the shared "topic-matcher" ForkJoinPool,
 * DW/DistWorkerCoProcFactory.java:74-85, while mutate() runs on the range's raft-apply thread): a handle may be used
 * from any number of threads at once. Every match leases its own workspace (streams, device scratch, pinned result
 * buffers) and pins the snapshot it ran on; the result keeps both until it is freed, so results of concurrent matches
 * never share memory and a commit never changes what an existing result resolves to. load/apply/commit serialise
 * among themselves and never block matches.
 *
 * Semantics: the matcher implements the match PREDICATE of the reference (DESIGN.md section 2). It equals the reference's
 * literal merge-join (TenantRouteMatcher.java:96-156) whenever that neither skips routes after its 20 probes nor seeks
 * backwards, i.e. for filters/topics without empty levels next to a shared prefix; the two documented divergences are
 * pinned in tests/test_oracle_golden.py and cannot be cross-checked against a JVM in this repository.
 */
#ifndef BFQ_GPUMATCH_H
#define BFQ_GPUMATCH_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BFQ_OK 0
#define BFQ_E_INVALID (-1)   /* bad argument (unsorted keys, undecodable route key, ...) */
#define BFQ_E_CUDA (-2)      /* CUDA runtime / device error */
#define BFQ_E_NOMEM (-3)
#define BFQ_E_STATE (-4)     /* e.g. match before the first commit */
#define BFQ_E_RANGE (-5)     /* index out of range */

typedef struct bfq_index bfq_index;     /* forward index: topic filters (routes) of many tenants  */
typedef struct bfq_result bfq_result;   /* result of one bfq_match call                            */
typedef struct bfq_rindex bfq_rindex;   /* inverse index: topics, matched BY filters (retain)      */
typedef struct bfq_rresult bfq_rresult;

/* text of the last error raised on this thread */
const char* bfq_last_error(void);

/* ------------------------------------------------------------------------------------------------
 * Forward index life cycle. One bfq_index per dist-worker KV range == one DistWorkerCoProc
 * (DW/DistWorkerCoProc.java:105-125). It replaces the per-tenant TenantRouteMatcher instances
 * (DW/cache/TenantRouteCacheFactory.java:67-71) and their RocksDB merge-join.
 * ---------------------------------------------------------------------------------------------- */
int32_t bfq_index_create(int32_t device_ordinal, bfq_index** out);
void bfq_index_destroy(bfq_index* h);

/* Drop all staged routes. Called from DistWorkerCoProc.reset(Boundary) (DW/DistWorkerCoProc.java:283-291)
 * before re-loading the range. */
int32_t bfq_index_reset(bfq_index* h);

/* Bulk-stage raw KV pairs exactly as stored by the reference: key = route key
 * (DWS/KVSchemaUtil.java:91-130), value = 8-byte BE incarnation (normal) or RouteGroup proto (shared).
 * Keys must be strictly ascending in unsigned byte order (a KV range scan is). Decoding is native
 * (replaces DWS/cache/RouteDetailCache.java:53-109 on the load path). */
int32_t bfq_index_load(bfq_index* h, const uint8_t* keys, const int64_t* key_off, const uint8_t* vals,
                       const int64_t* val_off, int64_t n);

/* Incremental feed from the post-persist Supplier of DistWorkerCoProc.mutate
 * (DW/DistWorkerCoProc.java:188-209; batchAddRoute :304-413, batchRemoveRoute :415-513):
 * upsert n_add pairs, delete n_del keys (any order). */
int32_t bfq_index_apply(bfq_index* h, const uint8_t* add_keys, const int64_t* add_key_off, const uint8_t* add_vals,
                        const int64_t* add_val_off, int64_t n_add, const uint8_t* del_keys, const int64_t* del_key_off,
                        int64_t n_del);

/* Publish the staged state as a new immutable device snapshot. The host-side rebuild and the upload run while matches
 * continue on the previous snapshot; the swap is atomic with respect to matches (they always see a whole snapshot).
 * Every snapshot has a generation (1, 2, ...); results report the generation they were produced from. The previous
 * snapshot is freed when the last match / result that pins it is gone. bfq_index_apply is all-or-nothing: an
 * undecodable key leaves the staging area untouched.
 * Delta path: a commit rebuilds only the tenants its staged changes touch, however many and whatever their shape (one
 * batchAddRoute / batchRemoveRoute batch may span every tenant of the range); the touched tenants are rebuilt on all host
 * cores and the device work is a fixed number of copies and launches.
 * Each gets a fresh slot region behind the existing ones (the one it replaces stays behind as garbage); the children of its
 * wide nodes (too many children for a private perfect-hash array, about a thousand) go into the shared tag table: its old
 * tag slots are freed first, then its new edges are placed into the free ones. The rest of the snapshot is copied on the
 * device and the ranks of the tenants behind a grown or shrunk tenant are moved. The commit is a full build instead when:
 *   - there is no snapshot yet, or bfq_index_reset / bfq_index_load ran since the last commit;
 *   - garbage slots would exceed a quarter of the slots plus 4096;
 *   - claimed tag-table slots would exceed 3/4 of its usable slots (the table only grows with a full build);
 *   - tag-table blocks with their overflow byte set would exceed a quarter of the blocks (freed slots do not clear it, so
 *     churn lengthens probes until a full build resets them);
 *   - a slot id or rank would run out of 31 bits.
 * Both paths give the same answers as a handle fully built from the same KV. bfq_index_stats reports the path taken
 * (13, 14), the tag table's fill (18..20) and how many tenants the commit built (21). */
int32_t bfq_index_commit(bfq_index* h);
int32_t bfq_index_generation(bfq_index* h, uint64_t* generation);   /* 0 before the first commit */
/* Tuning knobs (defaults are the measured best for a handle that has the GPU to itself):
 *   "tier0_ctas_per_sm"  cap of the lane-per-topic kernel's resident CTAs per SM (0 = the default: as many as fit, 7 on an
 *                        H100, and at most 4 for batches of >= 131072 topics). One slot less leaves room for kernels that must run BESIDE the matching: the exchange of the previous batch
 *                        (bfq_exchange_gather on another stream) in a multi-GPU pipeline;
 *   "order_min_topics"   batches of at least this many topics are de-duplicated and matched in locality order (default 32768);
 *   "dedup"              0: match repeated (tenant, topic) pairs separately;
 *   "dedup_hash_bits"    test knob, 0..64 (default 64): keep only the low k bits of the de-dup hash, so that distinct topics
 *                        share table slots and 32-bit tags on purpose and only the byte-for-byte compare tells them apart.
 *                        Answers stay exact at any k; small k only makes the de-dup pass slower;
 *   "fanout_global"      test knob, 0/1 (default 0): 1 makes every bfq_fanout_device take the global-count pass that large
 *                        deliverer counts use, so it can be checked on small cases. The grouping is the same either way. */
int32_t bfq_index_set_option(bfq_index* h, const char* name, int64_t value);

/* stats[k], k < n: 0 routes, 1 tenants, 2 trie nodes, 3 hash-table slots, 4 device bytes, 5 max nodes per
 * depth, 6 kernel launches so far, 7 overflow (tier-2) topics so far, 8 cap-flagged topics so far,
 * 9 multi-segment filters, 10 long-token chunks, 11 topics handed from the lane-per-topic tier to the
 * warp-per-topic tier so far, 12 duplicate (tenant, topic) pairs answered from their first occurrence so far,
 * 13 full commits, 14 delta commits, 15 garbage slots of the current snapshot, 16 match calls that found a range or
 * throttle buffer too small, grew it and re-ran the batch so far, 17 bfq_fanout_device calls that took the global-count
 * pass (rather than the shared-memory tile pass) so far, 18 usable tag-table slots (15 per block), 19 claimed tag-table
 * slots (children of wide nodes), 20 tag-table blocks whose overflow byte is set (all three of the current snapshot), 21 tenants
 * the last bfq_index_commit built (0 when nothing changed, every tenant after a full build), 22 device bytes of the current
 * snapshot's MatchInfo table (0 until the first bfq_delivery_encode[_ordered] on it) */
int32_t bfq_index_stats(bfq_index* h, int64_t* stats, int32_t n);
/* device time of the tier-0 (lane-per-topic) match kernel of the latest completed match call on this handle, measured with
 * CUDA events recorded on the launching stream around the launch (for roofline accounting) */
int32_t bfq_index_last_kernel_ms(bfq_index* h, double* ms);

/* Host-only diagnostic: run the index builder on a sorted KV snapshot without touching a device and report
 * stats[0..7] = routes, tenants, trie nodes, hash slots, max nodes per depth, max nodes per tenant,
 * multi-segment filters, long-token chunks, 8 = tag-table blocks that overflowed, 9..13 = nodes with 0/1/2/3/>=4
 * exact children, 14 = staging microseconds, 15 = flatten microseconds, 16 = a checksum of the whole image the build would
 * upload, 17 = 1 if building from one concatenated KV blob gives that same image, 18 = tenants whose stand-alone image (what a delta
 * commit builds for a touched tenant) equals their part of the full image, 19 = tenants with wide edges whose delta rebuild,
 * simulated on the image (their tag slots freed, the tenant rebuilt into a fresh region and its wide edges placed again), is
 * found again node for node by the kernels' lookup rules (used by CPU tests and to time the build). */
int32_t bfq_host_build_stats(const uint8_t* keys, const int64_t* key_off, const uint8_t* vals, const int64_t* val_off,
                             int64_t n, int64_t* stats, int32_t n_stats);

/* Map a route rank (position in the committed KV order) back to its stored key/value so the Java side
 * re-hydrates Matching objects with its own KVSchemaUtil.buildMatchRoute (DWS/KVSchemaUtil.java:73-79).
 * Lengths are returned even if the capacities are too small (nothing is copied then).
 * These three resolve against the CURRENT snapshot: ranks shift with every add/remove, so a rank taken from a match
 * result must be resolved with bfq_result_route_lookup / bfq_result_route_kinds (below), which use the snapshot the
 * result was produced from — the reference reads keys and values from one consistent KV reader too. */
int32_t bfq_route_lookup(bfq_index* h, int64_t rank, uint8_t* key_out, int64_t key_cap, int64_t* key_len,
                         uint8_t* val_out, int64_t val_cap, int64_t* val_len);
/* per-rank route kind: 0 normal, 1 normal persistent (subBrokerId == 1), 2 group (shared subscription) */
int32_t bfq_route_kind(bfq_index* h, int64_t rank, int32_t* kind);
int32_t bfq_route_kinds(bfq_index* h, const int64_t* ranks, int64_t n, uint8_t* kinds_out);

/* ------------------------------------------------------------------------------------------------
 * Forward match == ITenantRouteMatcher.matchAll(Set<String> topics, int maxPersistentFanout,
 * int maxGroupFanout) (DW/cache/ITenantRouteMatcher.java:28-38; implementation replaced:
 * DW/cache/TenantRouteMatcher.java:68-161 + caps of DW/cache/MatchedRoutes.java:87-141),
 * batched over tenants. Topic i belongs to tenant topic_tenant[i] (index into the tenants list);
 * max_pfanout/max_gfanout are per tenant (Setting.MaxPersistentFanout / MaxGroupFanout).
 * Host buffers in, host result out (H2D + kernels + D2H inside the call; batches of >= 128k topics are cut into four
 * sub-batches pipelined over three streams so the copies overlap the kernels). A topic whose topic_tenant[i] is outside
 * [0, n_tenants) simply matches nothing. Pinned (page-locked) host buffers give the best H2D rate.
 * ---------------------------------------------------------------------------------------------- */
int32_t bfq_match(bfq_index* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                  const uint8_t* topics, const int64_t* topic_off, const int32_t* topic_tenant, int64_t n_topics,
                  const int32_t* max_pfanout, const int32_t* max_gfanout, bfq_result** out);

/* Result layout. The arrays live in pinned memory leased to this result: they stay valid, and private to it, until
 * bfq_result_free() — other matches on the same handle (from any thread) and commits do not touch them:
 *   span_begin[i], span_count[i]   topic i's matched route RANGES are ranges[span_begin[i] ... +span_count[i])
 *   ranges[j] = {first rank, count} a run of consecutive route ranks (one matched filter's routes)
 *   route_count[i]                 routes matched by topic i before caps
 *   throttled[k] = {topic, rank, kind} routes dropped by the fan-out caps, kind 1 = PersistentFanoutThrottled,
 *                                  2 = GroupFanoutThrottled (MatchedRoutes.java:95-100,128-133); the caller
 *                                  emits the events. Surviving routes of topic i = its ranges minus these. */
typedef struct { uint32_t first; uint32_t count; } bfq_range;
typedef struct { uint32_t topic; uint32_t rank; uint32_t kind; } bfq_throttled;
int64_t bfq_result_num_topics(const bfq_result* r);
const uint32_t* bfq_result_span_begin(const bfq_result* r);
const uint32_t* bfq_result_span_count(const bfq_result* r);
const uint32_t* bfq_result_route_count(const bfq_result* r);
const bfq_range* bfq_result_ranges(const bfq_result* r, int64_t* n_ranges);
const bfq_throttled* bfq_result_throttled(const bfq_result* r, int64_t* n_throttled);
/* Convenience: flatten to CSR of surviving ranks, ascending per topic. offsets[n_topics+1]; returns the
 * total, copies only if it fits rank_cap (large results are filled by several host threads). */
int64_t bfq_result_expand(const bfq_result* r, int64_t* offsets, int64_t* ranks, int64_t rank_cap);
/* rank -> stored key/value and route kind, resolved against the snapshot THIS result was produced from */
int32_t bfq_result_route_lookup(const bfq_result* r, int64_t rank, uint8_t* key_out, int64_t key_cap, int64_t* key_len,
                                uint8_t* val_out, int64_t val_cap, int64_t* val_len);
int32_t bfq_result_route_kinds(const bfq_result* r, const int64_t* ranks, int64_t n, uint8_t* kinds_out);
uint64_t bfq_result_generation(const bfq_result* r);
/* timings of the call in milliseconds: 0 busy time of the H2D copy stream (overlapped with kernels), 1 device time
 * of the tier-0 kernel of the first sub-batch, 2 number of pipelined sub-batches, 3 wall time of the whole call */
int32_t bfq_result_timings(const bfq_result* r, double* ms, int32_t n);
void bfq_result_free(bfq_result* r);

/* Same match with the topic batch already resident in device memory and the result left there
 * (used by bench.py's kernel-only leg and by callers that pipeline batches). d_* are device pointers
 * (the kernels read d_topics in whole aligned words / 16-byte granules that hold at least one topic byte, so the
 * blob must lie in memory that is readable up to its enclosing 16-byte boundaries: any cudaMalloc'd buffer),
 * stream is a cudaStream_t (NULL = default stream).
 *   bfq_match_device_async  enqueues every kernel of the match on `stream` and returns without synchronising: all
 *                           counts the later kernels need are read on the device. The d_* result pointers are valid
 *                           for work enqueued on the same stream afterwards; the n_* fields are not filled yet.
 *   bfq_device_result_wait  waits for the match, fills the n_* fields and handles the rare cases the optimistic
 *                           enqueue cannot (topics that need the global-scratch tier, buffers that must grow: the
 *                           batch is then re-run and the d_* pointers may change — read them after the wait).
 *   bfq_match_device        = async + wait.
 * The result buffers belong to a workspace leased to this result: they stay valid until bfq_device_result_release,
 * whatever else runs on the handle. Several matches may be in flight on one handle (and one stream) at a time.
 *   bfq_device_result_release  blocks until the match and everything the library enqueued for the result since
 *                           (bfq_expand_device, bfq_expand_device_budget, bfq_fanout_device, bfq_delivery_device,
 *                           bfq_delivery_device_ordered, bfq_delivery_encode[_ordered], bfq_delivery_reply, bfq_exchange_gather), on every stream it was used on, has finished; then the workspace goes back
 *                           to the handle's pool, where the next match may take it. The caller's own work that reads the
 *                           result's arrays (or the CSR and fan-out arrays that live in its workspace) must be ordered
 *                           before the release by the caller. */
typedef struct {
    const uint32_t* d_span_begin;   /* [n_topics] */
    const uint32_t* d_span_count;   /* [n_topics] */
    const uint32_t* d_route_count;  /* [n_topics] */
    const bfq_range* d_ranges;      /* sparse: topic i's ranges are d_ranges[d_span_begin[i] ... + d_span_count[i] & 0x3FFFFFFF);
                                       n_ranges is the extent of the array, not the number of ranges */
    const bfq_throttled* d_throttled; /* [n_throttled] */
    int64_t n_ranges, n_throttled, n_routes;
    int64_t n_overflow_topics, n_flagged_topics, n_launches;
    int64_t n_topics;               /* topics of the batch (length of the per-topic arrays) */
    int64_t n_distinct_topics;      /* (tenant, topic) pairs actually walked; duplicates share their first occurrence's span */
    double tier0_ms;                /* device time of the lane-per-topic kernel of this match (CUDA events on `stream`) */
    uint64_t generation;            /* snapshot the match ran on */
    void* lease;                    /* opaque; owned by the library until bfq_device_result_release */
} bfq_device_result;
int32_t bfq_match_device(bfq_index* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                         const uint8_t* d_topics, const int64_t* d_topic_off, const int32_t* d_topic_tenant,
                         int64_t n_topics, const int32_t* max_pfanout, const int32_t* max_gfanout, void* stream,
                         bfq_device_result* out);
int32_t bfq_match_device_async(bfq_index* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                               const uint8_t* d_topics, const int64_t* d_topic_off, const int32_t* d_topic_tenant,
                               int64_t n_topics, const int32_t* max_pfanout, const int32_t* max_gfanout, void* stream,
                               bfq_device_result* out);
int32_t bfq_device_result_wait(bfq_device_result* res);
void bfq_device_result_release(bfq_device_result* res);
/* Flatten a completed device result into a device CSR: d_offsets[n_topics+1] (int64) is always written, the surviving
 * ranks (caps applied, unordered within a topic) are written to d_ranks if the total fits rank_cap (pass
 * d_ranks = NULL to only size). Returns the total via *n_ranks. Resolves against the result's own snapshot and caps. */
int32_t bfq_expand_device(const bfq_device_result* res, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap,
                          void* stream, int64_t* n_ranks);

/* Delivery budgets of DeliverExecutorGroup.submit (DW/DeliverExecutorGroup.java:112-231) applied to a completed device match:
 * the same device CSR as bfq_expand_device, holding only the routes that are actually DELIVERED. It goes unchanged into
 * bfq_fanout_device. Per tenant i of the match's tenant list the host supplies max_pfanout_bytes[i]
 * (Setting.MaxPersistentFanoutBytes, > 0) and tenant_bandwidth[i] (bit 0: resourceThrottler.hasResource(tenant,
 * TotalPersistentFanOutBytesPerSeconds), bit 1: the same for TotalTransientFanOutBytesPerSeconds); per topic position t,
 * d_msg_bytes[t] (device, SizeUtil.estSizeOf of the topic's TopicMessagePack, >= 0). Repeated topics may carry different sizes.
 * For topic t with surviving routes R (the match's caps applied), kinds as in bfq_route_kind, P of them persistent:
 *   |R| <= 1       delivered whatever the budgets say (the reference's single-route branch)
 *   |R| > 1        groups: all delivered, no budget applies (a group of persistent members does not count toward the bytes)
 *                  transient: all delivered with transient bandwidth, else none (flag BFQ_BUDGET_NO_TRANSIENT_BW if any)
 *                  persistent: without persistent bandwidth none (flag BFQ_BUDGET_NO_PERSISTENT_BW if P > 0); with it the
 *                  first k = min(P, ceil(B / s)) in KV (rank) order, k = P if s == 0: the sends for which sent * s < B held
 *                  (flag BFQ_BUDGET_BYTES_THROTTLED iff k < P). Computed without overflow for any B <= 2^63 - 1, s <= 2^31 - 1.
 * The reference iterates a hash set, so WHICH k persistent routes it sends is unspecified; this call fixes it to KV order,
 * the rule of the match's own caps, so results are reproducible. With the match's caps applied first, submit's count checks
 * (MaxPersistentFanout, MaxGroupFanout) never drop a route or fire an event, so the call takes no count inputs.
 * What the host does with the result (the reference's events and meter):
 *   BFQ_BUDGET_BYTES_THROTTLED    report PersistentFanoutBytesThrottled(tenantId, topic, maxBytes) once for the topic
 *   BFQ_BUDGET_NO_*_BW            report OutOfTenantResource(reason) once per PUBLISHER of the topic's message pack
 *   BFQ_BUDGET_METERED            record MqttPersistentFanOutBytes = d_delivered_persistent[t] * s (zero included); set for
 *                                 |R| > 1 and for a single persistent route
 * The match result is not touched: route_count, throttled and the BatchDistReply fan-out count stay the match's.
 * Sizing and writing follow bfq_expand_device: d_offsets[n_topics + 1] is always written, d_ranks only if the total fits
 * rank_cap (d_ranks = NULL only sizes), ranks are unordered within a topic and resolve against the result's own snapshot.
 * The per-topic arrays live in the result's leased workspace until bfq_device_result_release (the next budget call on the
 * same result overwrites them). The call synchronises `stream` once (to read the total and the size check).
 * Errors: BFQ_E_INVALID for a NULL array the call needs, a max_pfanout_bytes[i] <= 0, or a negative d_msg_bytes entry (checked
 * on the device; offsets are written, ranks are not); BFQ_E_STATE for a match that has not completed. */
#define BFQ_BUDGET_BYTES_THROTTLED 1
#define BFQ_BUDGET_NO_PERSISTENT_BW 2
#define BFQ_BUDGET_NO_TRANSIENT_BW 4
#define BFQ_BUDGET_METERED 8
typedef struct {
    const uint32_t* d_delivered_persistent;  /* [n_topics] persistent routes delivered (k; 1 or 0 when |R| <= 1) */
    const uint8_t* d_topic_flags;            /* [n_topics] BFQ_BUDGET_* bits */
    int64_t n_delivered;                     /* routes delivered = d_offsets[n_topics] */
    int64_t n_dropped_bytes;                 /* persistent routes dropped by MaxPersistentFanoutBytes */
    int64_t n_dropped_persistent_bandwidth;  /* persistent routes dropped for lack of persistent bandwidth */
    int64_t n_dropped_transient_bandwidth;   /* transient routes dropped for lack of transient bandwidth */
} bfq_budget_result;
int32_t bfq_expand_device_budget(const bfq_device_result* res, const int32_t* d_msg_bytes, const int64_t* max_pfanout_bytes,
                                 const uint8_t* tenant_bandwidth, int64_t* d_offsets, int64_t* d_ranks, int64_t rank_cap,
                                 void* stream, bfq_budget_result* out);

/* ------------------------------------------------------------------------------------------------
 * Batched range pruning on the dist-server side (SURVEY.md 8f): TenantRangeLookupCache.lookup
 * (bifromq-dist/bifromq-dist-server/src/main/java/org/apache/bifromq/dist/server/scheduler/TenantRangeLookupCache.java:70-106)
 * decides, per publish topic, which of the tenant's KV ranges can hold a matching route: a range with a Fact
 * {firstGlobalFilterLevels, lastGlobalFilterLevels} stays a candidate iff the topic's expansion set (every filter that matches
 * it) has a member in [first, last]; the reference runs its expansion iterator per topic and candidate behind a cache. Here one
 * kernel answers a whole batch (one thread per (topic, candidate): a lower-bound walk of the implicit expansion trie).
 *   tenants / topics / topic_tenant   as for bfq_match
 *   cand_off[n_tenants + 1]           tenant t's candidate ranges are [cand_off[t], cand_off[t + 1]), in boundary order
 *   cand_flags[c]                     bit 0: the range has a Fact, bit 1: it has first, bit 2: it has last
 *   first / last (blob, off[n_cand + 1])   the global filter levels joined by NUL bytes, level 0 = the tenant id
 *   keep_off_out[n_topics + 1], keep_out[keep_off_out[n_topics]]   topic i's row = one byte per candidate of its tenant:
 *                                     1 = the range is returned by the reference's lookup, 0 = it is not
 * Semantics are the reference's loop, literally: no Fact -> kept; a Fact without first or last -> empty range, skipped; the
 * first range whose seek runs past the end of the expansion set ends the scan. Stateless; needs a CUDA device.
 * Depth: there is no level limit. A topic (up to MaxTopicLength) and a bound may have any number of levels; each thread reads
 * them through cursors and keeps no per-level state, so a deep topic in a batch costs time in its own rows only.
 * Errors: BFQ_E_INVALID for a NULL array the call needs, BFQ_E_RANGE for a topic_tenant outside [0, n_tenants).
 * ---------------------------------------------------------------------------------------------- */
int32_t bfq_range_lookup(int32_t device_ordinal, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                         const uint8_t* topics, const int64_t* topic_off, const int32_t* topic_tenant, int64_t n_topics,
                         const int64_t* cand_off, const uint8_t* cand_flags, const uint8_t* first_blob, const int64_t* first_off,
                         const uint8_t* last_blob, const int64_t* last_off, int64_t* keep_off_out, uint8_t* keep_out);

/* ------------------------------------------------------------------------------------------------
 * Fan-out expansion on the device (SURVEY.md 8f): the step right behind the match. DeliverExecutorGroup.submit
 * (DW/DeliverExecutorGroup.java:112-231) walks every matched route of a message, resolves a shared subscription to one
 * member (:242-278) and hands each route to the deliverer of its (subBrokerId, delivererKey) (DW/DeliverExecutor.java:89-93),
 * which batches per deliverer. bfq_fanout_device does that grouping for a whole batch: it takes the device CSR of a completed
 * match (bfq_expand_device: surviving ranks per topic, caps applied) and returns every (topic, route) pair grouped by
 * deliverer id: pairs [d_pack_offsets[d], d_pack_offsets[d + 1]) belong to deliverer d; d_pack_topic / d_pack_rank give the
 * pair, d_pack_member the member index a $share subscription was resolved to (0xFFFFFFFF for ordinary routes; members in the
 * order of the stored RouteGroup). An unordered share picks member hash(topic position, rank) mod n (the reference picks
 * uniformly at random: any member is valid); ORDERED shares need each message's publisher (rendezvous hash of ClientInfo) and
 * are grouped, unresolved, under the last id (ordered_share_id) for the host; a shared subscription whose stored RouteGroup
 * has no member is parked there too (member 0xFFFFFFFF). Order inside a deliverer's pairs is unspecified.
 * Deliverer ids: every (subBrokerId, delivererKey) pair the handle has interned since it was created, in first-seen order.
 * An id is never reused and never freed: it stays valid across commits, resets and reloads, and routes that were removed
 * keep their ids. So a handle with much deliverer churn carries every id it has seen, and each call writes
 * d_pack_offsets over all of them (8 bytes per id). Scratch: the tile pass (chosen while ids x 4096-pair tiles is at most
 * max(n_pairs, 4096), so for at most 4096 ids) needs 8 bytes per (id, tile) cell, at most 8 bytes per pair; the global pass
 * (every other case) needs 8 bytes per id. bfq_fanout_deliverer gives an
 * id's pair back. The ordered-share id is the number of ids interned when the result's snapshot was first fanned out:
 * always use the result's ordered_share_id; bfq_fanout_deliverer may resolve that number to a deliverer interned later.
 * Limits: fewer than 2^32 (topic, route) pairs per call (BFQ_E_RANGE; split the batch), route ranks below 2^32, and at most
 * 2^31 - 3 ids per handle (BFQ_E_RANGE). A receiver url without a subBrokerId or delivererKey makes the call fail with BFQ_E_INVALID.
 * The arrays live in the result's leased workspace: valid until bfq_device_result_release.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const int64_t* d_pack_offsets;   /* [n_deliverers + 1] */
    const uint32_t* d_pack_topic;    /* [n_pairs] topic position in the batch */
    const uint32_t* d_pack_rank;     /* [n_pairs] route rank (of the result's snapshot) */
    const uint32_t* d_pack_member;   /* [n_pairs] */
    int64_t n_pairs;
    int32_t n_deliverers;            /* ids [0, n_deliverers); the last one is ordered_share_id */
    int32_t ordered_share_id;
    uint64_t generation;
} bfq_fanout_result;
int32_t bfq_fanout_device(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs,
                          void* stream, bfq_fanout_result* out);
int32_t bfq_fanout_deliverer(bfq_index* h, int32_t id, int32_t* sub_broker_id, uint8_t* key_out, int64_t key_cap, int64_t* key_len);

/* ------------------------------------------------------------------------------------------------
 * Delivery requests on the device: the fan-out laid out the way a deliverer sends it. Every DeliveryCall goes to the
 * deliverer's batcher, BatchDeliveryCall (bifromq-deliverer/.../BatchDeliveryCall.java:58,75-104), which nests the calls as
 * tenantId -> TopicMessagePack -> Set<MatchInfo> and sends one DeliveryRequest
 * (map<tenantId, DeliveryPackage{repeated DeliveryPack{messagePack, repeated MatchInfo}}>, subbroker/type.proto:28-38).
 * bfq_delivery_device returns the pairs of a device CSR already in that nesting:
 *   deliverer d's packages  [d_package_off[d], d_package_off[d + 1]); a package is one (deliverer, tenant): its tenant is
 *                           d_package_tenant[p] (index into the match's tenant list), ascending within a deliverer, each tenant at
 *                           most once per deliverer even when the batch interleaves tenants
 *   package p's packs       [d_pack_off[p], d_pack_off[p + 1]); a pack is one (deliverer, topic position): d_pack_topic[k],
 *                           ascending within a package (the order BatchDeliveryCall.add sees when a request's packs are submitted
 *                           in order). Repeated (tenant, topic) positions stay separate packs (separate TopicMessagePacks), even
 *                           though the match de-duplicated them.
 *   pack k's MatchInfos     pairs [d_match_off[k], d_match_off[k + 1]): d_match_rank (route rank of the result's snapshot) and
 *                           d_match_member (member index of a $share, 0xFFFFFFFF otherwise). Order inside a pack is unspecified
 *                           (the reference keeps a HashSet); no pair appears twice.
 * Input: the device CSR bfq_fanout_device takes (bfq_expand_device or bfq_expand_device_budget) and d_topic_tenant, the device
 * array the match itself took. A topic whose tenant index is outside the match's list has no pairs (n_pairs counts the pairs
 * nested). Deliverer ids, ordered_share_id and the $share member pick are exactly those of bfq_fanout_device for the same
 * result and CSR (one device function resolves both); $oshare pairs and groups without members are nested under
 * ordered_share_id like any other deliverer.
 * The arrays live in the result's leased workspace until bfq_device_result_release, in buffers separate from the fan-out's (both
 * calls may be used on one result); calling this again on the same result overwrites them. The call synchronises `stream` once
 * (to read n_packages and n_packs). Limits as bfq_fanout_device: fewer than 2^32 pairs and ranks below 2^32, else BFQ_E_RANGE.
 * Errors: BFQ_E_INVALID for a NULL array the call needs, an n_pairs that disagrees with d_offsets[n_topics] (checked on the
 * device: nothing is nested) or a receiver url without a delivererKey; BFQ_E_STATE for a match that has not completed.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const int64_t* d_package_off;     /* [n_deliverers + 1] */
    const uint32_t* d_package_tenant; /* [n_packages] */
    const int64_t* d_pack_off;        /* [n_packages + 1] */
    const uint32_t* d_pack_topic;     /* [n_packs] */
    const int64_t* d_match_off;       /* [n_packs + 1] */
    const uint32_t* d_match_rank;     /* [n_pairs] */
    const uint32_t* d_match_member;   /* [n_pairs] */
    int64_t n_pairs, n_packages, n_packs;
    int32_t n_deliverers, ordered_share_id;
    uint64_t generation;
} bfq_delivery_result;
int32_t bfq_delivery_device(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks, int64_t n_pairs,
                            const int32_t* d_topic_tenant, void* stream, bfq_delivery_result* out);

/* ------------------------------------------------------------------------------------------------
 * Ordered shared subscriptions ($oshare) resolved in the delivery nesting. The ordered branch of DeliverExecutorGroup.send
 * (DW/DeliverExecutorGroup.java:242-278) sends, for every publisher pack of the topic's TopicMessagePack, to ONE member of the
 * group: RendezvousHash.get (base-util/.../RendezvousHash.java) scores member m as
 *   Hashing.murmur3_128() (seed 0).newHasher().putInt(publisher.hashCode()).putString(receiverUrl_m, UTF_8).hash().asLong()
 * i.e. h1 of MurmurHash3_x64_128 over LE32(hash) ‖ utf8(receiverUrl), as a signed 64-bit value, and picks the first member
 * (in the stored RouteGroup's wire order, the fan-out's member order) whose score is strictly greater than every earlier one
 * (the running best starts at Long.MIN_VALUE). Publishers with the same winner form one new TopicMessagePack (the topic, those
 * publisher packs in their original order), sent to the winner's deliverer with the winner's MatchInfo in a fresh
 * TopicMessagePackHolder; BatchDeliveryCall keys packs by holder identity, so every such sub-pack is a DeliveryPack of its own
 * with exactly one MatchInfo, even when two $oshare routes of a topic pick members on one deliverer.
 * bfq_delivery_device_ordered is bfq_delivery_device plus that pick. Per topic position t the host passes its publisher packs:
 * d_pub_off[n_topics + 1] (device, from 0 to n_pubs, never decreasing) and d_pub_hash[n_pubs] (device,
 * publisherPack.getPublisher().hashCode(): a protobuf object hash, which native code cannot recompute). Repeated topic
 * positions carry their own publishers.
 *   d                       the nesting of bfq_delivery_device (same deliverer ids, tenants, pack order and $share picks), with
 *                           every $oshare pair whose group has members replaced by its sub-packs: a sub-pack's MatchInfo is
 *                           (rank, winning member index). Only member-less groups stay under d.ordered_share_id (the reference
 *                           would fail on them), and so would a publisher for which every member scores exactly
 *                           Long.MIN_VALUE (the reference finds no winner: member 0xFFFFFFFF). A topic position with no
 *                           publisher packs gives no sub-pack for its $oshare routes; its other routes still get the whole pack.
 *                           d.n_pairs counts the MatchInfos nested. Within a package a topic position's whole pack comes first,
 *                           then its sub-packs ordered by (rank, member).
 *   d_pack_pub_off          [d.n_packs + 1]: pack k's publishers are d_pack_pub[d_pack_pub_off[k] .. d_pack_pub_off[k + 1]). An
 *                           empty span is the whole TopicMessagePack of d_pack_topic[k]; a non-empty span is an $oshare sub-pack.
 *   d_pack_pub              publisher positions (indices into d_pub_hash), ascending within a pack; n_pack_pubs of them
 *   n_ordered_packs         the sub-packs (packs with a non-empty span)
 * The pick is stateless: it scores the members of the result's own snapshot. The reference caches it per (tenantId,
 * mqttTopicFilter, ClientInfo) but drops that cache on every add or remove of the ordered filter's routes
 * (DistWorkerCoProc.mutate -> refreshOrderedShareSubRoutes), so a pick over the snapshot's members is the same answer.
 * The first call on a snapshot uploads its ordered groups' member receiverUrls; bfq_fanout_device and bfq_delivery_device never
 * need them. The arrays live in the result's leased workspace until bfq_device_result_release and share buffers with
 * bfq_delivery_device: a later call of either on the same result overwrites the earlier one's arrays. The call synchronises
 * `stream` twice (to size the (pair, publisher) items, and to read the totals).
 * Errors: BFQ_E_INVALID for a NULL array the call needs, an n_pairs that disagrees with d_offsets[n_topics], or a d_pub_off
 * that does not run from 0 to n_pubs without decreasing (both checked on the device: nothing is nested), or a receiver url
 * without a delivererKey; BFQ_E_RANGE for 2^32 or more pairs plus ($oshare pair, publisher) items; BFQ_E_STATE for a match that
 * has not completed.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    bfq_delivery_result d;          /* as bfq_delivery_device, with $oshare pairs resolved: only member-less groups stay
                                       under d.ordered_share_id; d.n_pairs counts the MatchInfos nested */
    const int64_t* d_pack_pub_off;  /* [d.n_packs + 1]: an empty span = the whole TopicMessagePack of d_pack_topic[k];
                                       a non-empty span = an $oshare sub-pack made of these publisher packs */
    const uint32_t* d_pack_pub;     /* publisher positions (indices into d_pub_hash), ascending within a pack */
    int64_t n_pack_pubs, n_ordered_packs;
} bfq_delivery_ordered_result;
int32_t bfq_delivery_device_ordered(const bfq_device_result* res, const int64_t* d_offsets, const int64_t* d_ranks,
                                    int64_t n_pairs, const int32_t* d_topic_tenant, const int64_t* d_pub_off,
                                    const int32_t* d_pub_hash, int64_t n_pubs, void* stream,
                                    bfq_delivery_ordered_result* out);

/* ------------------------------------------------------------------------------------------------
 * Delivery requests as wire bytes: a nesting of bfq_delivery_device or bfq_delivery_device_ordered encoded as one serialized
 * DeliveryRequest per deliverer, the message BatchDeliveryCall.execute (bifromq-deliverer/.../BatchDeliveryCall.java:91-108)
 * builds and sends. Deliverer d's request is d_out[d_req_off[d] .. d_req_off[d + 1]): DeliveryRequest.parseFrom takes the
 * slice as it is, so no MatchInfo or DeliveryRequest is ever built per pair on the host. Proto3, field numbers of
 * subbroker/type.proto, commontype/MatchInfo.proto, RouteMatcher.proto and TopicMessage.proto, every length a minimal varint:
 *   DeliveryRequest   package = 3: one map entry per package of the deliverer, in the nesting's tenant order; both entry fields
 *                     are written (key = 1: tenantId, the match's tenant list entry; value = 2: DeliveryPackage)
 *   DeliveryPackage   pack = 1 per pack, in the nesting's order
 *   DeliveryPack      messagePack = 2, then matchInfo = 3 per MatchInfo of the pack, in the nesting's order
 *   TopicMessagePack  topic = 1 (the topic position's topic, omitted when empty), message = 2 per publisher pack: every publisher
 *                     pack of the topic position for a whole pack, the sub-pack's own (d_pack_pub, in order) for an $oshare
 *                     sub-pack (DeliverExecutorGroup.java:271-273)
 *   MatchInfo         as NormalMatching / GroupMatching build it (DWS/cache/): matcher = 1 always; receiverId = 2 (the second
 *                     NUL-separated part of the receiverUrl, ReceiverCache) omitted when empty; incarnation = 3 (varint: the
 *                     normal route's 8-byte big-endian value, or the member's value in the stored RouteGroup) omitted when 0.
 *                     A $share / $oshare member carries the GROUP's RouteMatcher.
 *   RouteMatcher      as RouteDetailCache.get builds it from the route key: type = 1 omitted for Normal, 1 UnorderedShare,
 *                     2 OrderedShare; filterLevel = 2 for every NUL-separated level of the escaped filter, empty levels included;
 *                     group = 3 for shared routes only; mqttTopicFilter = 4 the unescaped filter, prefixed "$share/<group>/" or
 *                     "$oshare/<group>/" for groups (omitted when empty).
 * Inputs: the nesting (the latest delivery call on THIS result: one from another result, snapshot or an earlier call is
 * BFQ_E_RANGE; bfq_delivery_encode takes bfq_delivery_device's, bfq_delivery_encode_ordered bfq_delivery_device_ordered's);
 * the match's own tenant list (host) and topics (device, as the match took them); per topic position its publisher packs as
 * serialized TopicMessagePack.PublisherPack bytes (device): d_pub_off[n_topics + 1] as for bfq_delivery_device_ordered, and
 * pack q's bytes are d_pubpack_bytes[d_pubpack_off[q] .. d_pubpack_off[q + 1]).
 * Sizing follows bfq_expand_device: d_req_off [n_deliverers + 1] is always written; the bytes are written only if n_bytes fits
 * out_cap (d_out = NULL only sizes). The span of ordered_share_id is empty: its MatchInfos (member-less groups, and with
 * bfq_delivery_encode every $oshare pair) are counted in n_skipped and never encoded. d_req_off lives in the result's leased
 * workspace until bfq_device_result_release, which waits for the encode; the next encode on the result overwrites it. The
 * first call on a snapshot builds and uploads its MatchInfo table (bfq_index_stats slot 22); other calls never need it. The
 * call synchronises `stream` once (to read n_bytes) and returns while the write pass may still run.
 * Errors: BFQ_E_INVALID for a NULL array, a tenant list of another length than the match's, or a d_pub_off / d_pubpack_off
 * that does not start at 0 and never decrease or a publisher position outside it (checked on the device: nothing is
 * written); BFQ_E_STATE for a match that has not completed; BFQ_E_RANGE for a nesting that is not the result's latest.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    const int64_t* d_req_off;       /* [n_deliverers + 1]: deliverer d's DeliveryRequest = d_out[d_req_off[d] .. d_req_off[d + 1]) */
    int64_t n_bytes;                /* = d_req_off[n_deliverers] */
    int64_t n_match_infos;          /* MatchInfos encoded */
    int64_t n_skipped;              /* MatchInfos left under ordered_share_id: never encoded */
    int32_t n_deliverers, ordered_share_id;
    uint64_t generation;
} bfq_delivery_wire_result;
int32_t bfq_delivery_encode(const bfq_device_result* res, const bfq_delivery_result* nesting, const uint8_t* tenants,
                            const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_topics, const int64_t* d_topic_off,
                            const int64_t* d_pub_off, const uint8_t* d_pubpack_bytes, const int64_t* d_pubpack_off, uint8_t* d_out,
                            int64_t out_cap, void* stream, bfq_delivery_wire_result* out);
int32_t bfq_delivery_encode_ordered(const bfq_device_result* res, const bfq_delivery_ordered_result* nesting, const uint8_t* tenants,
                                    const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_topics, const int64_t* d_topic_off,
                                    const int64_t* d_pub_off, const uint8_t* d_pubpack_bytes, const int64_t* d_pubpack_off,
                                    uint8_t* d_out, int64_t out_cap, void* stream, bfq_delivery_wire_result* out);

/* ------------------------------------------------------------------------------------------------
 * Delivery replies: every deliverer's serialized DeliveryReply joined back to the pairs of its request, as the reply branch
 * of BatchDeliveryCall.execute (bifromq-deliverer/.../BatchDeliveryCall.java:108-172) with TypeUtil.toMap does it, so the
 * host never builds a MatchInfo per pair to key the join. subbroker/type.proto:41-63:
 *   DeliveryReply     code = 1 (0 OK, 1 BACK_PRESSURE_REJECTED, 2 ERROR); result = 2: map<tenantId, DeliveryResults>
 *   DeliveryResults   result = 1: repeated DeliveryResult
 *   DeliveryResult    matchInfo = 1; code = 2 (0 OK, 1 NO_SUB, 2 NO_RECEIVER)
 * Inputs: `nesting` is the latest delivery nesting of this result, the one bfq_delivery_encode[_ordered] encodes (for an ordered
 * nesting pass &ordered.d; an $oshare sub-pack's MatchInfo is its (rank, winning member)); anything else is BFQ_E_RANGE. The
 * match's own tenant list (host). Deliverer d's reply is d_reply[d_reply_off[d] .. d_reply_off[d + 1]) (device; the offsets
 * never decrease and need not start at 0): a failed call is the bytes 08 02 (the ERROR reply `.exceptionally` makes), an empty
 * slice a default reply (OK, no results). The slices of deliverers with an empty request (ordered_share_id among them) are
 * never read.
 * A deliverer is decided on the device only when its answer is certainly the reference's: its reply is well-formed protobuf
 * (known fields in any order; unknown fields of wire types 0, 1, 2 and 5 skipped at every level), every DeliveryResult's
 * matchInfo equals, byte for byte, a MatchInfo the deliverer's request carries under that map entry's tenant (the encode's
 * canonical bytes; for these messages canonical bytes are equal exactly when the messages are), and no MatchInfo appears
 * twice under a tenant (where toMap throws). A singular field or a tenant key given twice, a tenant key that is not valid
 * UTF-8 or not in the request, a MatchInfo that does not resolve (a non-canonical encoding of a requested one included),
 * truncated bytes or a wrong wire type on a known field make it FALLBACK instead: the host runs execute's loop on its request
 * and reply slices. Sub-brokers that echo the request's MatchInfo objects (LocalDistService.dist, DeliveryPipeline.deliver)
 * never cause it. Other deliverers of the call are unaffected.
 * Outputs (device arrays in the result's leased workspace until bfq_device_result_release, which waits for this call; the next
 * call on the result overwrites them):
 *   d_pair_code[nesting->n_pairs]  per pair of the nesting (aligned with d_match_rank / d_match_member), DeliveryCallResult:
 *                           0 OK, 1 NO_SUB, 2 NO_RECEIVER, 3 BACK_PRESSURE_REJECTED, 4 ERROR (also a DeliveryResult code
 *                           outside 0-2, which is not stale), and 5 NO_RESULT (no result for it: the reference completes it OK
 *                           and logs "No deliver result"), 6 NOT_SENT (the pairs under ordered_share_id), 7 UNDECIDED (its
 *                           deliverer is FALLBACK)
 *   d_status[n_deliverers]  0 OK, 3 BACK_PRESSURE_REJECTED, 4 ERROR (the reply code is ERROR or any value but 0 and 1),
 *                           6 NOT_SENT (an empty request), 7 FALLBACK
 *   d_stale[n_stale]        execute's staleMatchInfos: one entry per distinct (deliverer, tenant index, rank, member) whose code
 *                           is NO_SUB or NO_RECEIVER, sorted by those four fields, with the offset and length of its MatchInfo
 *                           in d_reply (MatchInfo.parseFrom of those bytes gives removeRoute's matcher, receiverId and
 *                           incarnation; delivererKey and subBrokerId come from bfq_fanout_deliverer)
 * The plain and the ordered nesting share the result's buffers and the nesting struct does not say which call made it: a
 * bfq_delivery_result copied before a later delivery call whose counts happen to equal it is taken for that later nesting, so
 * pass the struct of the latest call (it is what the requests were encoded from).
 * The first call on a snapshot also hashes its MatchInfo table (uploading the table first if no encode did). Workspace: the
 * key table has a power of two of at least 2 * nesting->n_pairs slots of 28 bytes, and the per-pair and stale arrays take
 * about 60 bytes per pair (all sized from n_pairs, an upper bound on the distinct keys, because the count is only known on the
 * device); about 3 GB at 23.6 M pairs, kept by the workspace for its next calls. The call synchronises `stream` once, to read
 * the counts.
 * Errors: BFQ_E_INVALID for a NULL array, a tenant list of another length than the match's, or a decreasing d_reply_off
 * (checked on the device: nothing is written); BFQ_E_STATE for a match that has not completed; BFQ_E_RANGE for a nesting that
 * is not the result's latest.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t deliverer, tenant;      /* deliverer id; tenant index in the match's list */
    uint32_t rank, member;          /* as in d_match_rank / d_match_member */
    int64_t reply_off;              /* the MatchInfo message: d_reply[reply_off .. reply_off + reply_len) */
    int32_t reply_len, code;        /* code: 1 NO_SUB or 2 NO_RECEIVER */
} bfq_stale_match;
typedef struct {
    const uint8_t* d_pair_code;     /* [n_pairs] */
    const uint8_t* d_status;        /* [n_deliverers] */
    const bfq_stale_match* d_stale; /* [n_stale] */
    int64_t n_code[8];              /* pairs per code of d_pair_code */
    int64_t n_pairs, n_stale;
    int32_t n_fallback, n_deliverers, ordered_share_id;
    uint64_t generation;
} bfq_delivery_reply_result;
int32_t bfq_delivery_reply(const bfq_device_result* res, const bfq_delivery_result* nesting, const uint8_t* tenants,
                           const int64_t* tenant_off, int32_t n_tenants, const uint8_t* d_reply, const int64_t* d_reply_off,
                           void* stream, bfq_delivery_reply_result* out);

/* ------------------------------------------------------------------------------------------------
 * Multi-GPU: the one exchange step of the tenant-sharded path (SURVEY.md 8e). Tenants are independent key ranges, so
 * every GPU (one process each) matches the topics of the tenants it hosts with NO data-path collective; what travels is
 * the reply, reassembled on every rank the way the dist-server reassembles the per-worker BatchDistReply messages
 * (bifromq-dist/bifromq-dist-server/src/main/java/org/apache/bifromq/dist/server/scheduler/BatchDistServerCall.java:186-205,
 * 245-271). bfq_exchange_gather all-gathers the device results of the ranks' matches over NCCL (NVLink / NVSwitch), in
 * rank order: per topic the matched-route count (what TopicFanout carries, DistWorkerCoProc.proto:34-131) and, with
 * BFQ_EXCHANGE_RANGES, the number of matched ranges plus the dense {first rank, count} ranges themselves (route ranks are
 * local to the rank that produced them: rank r's ranges refer to r's committed KV order). One host synchronisation per
 * call (NCCL needs the receive counts); no host-side copies. NCCL is taken from the process at run time (libnccl.so.2).
 *   rank 0: bfq_exchange_unique_id(id)  -> broadcast the 128 bytes to the other ranks out of band (the host's own RPC)
 *   every rank: bfq_exchange_create(device, rank, world, id, &x)       (collective: all ranks must call it)
 *   per batch, every rank: bfq_match_device(...) ; bfq_exchange_gather(x, &res, what, stream, &g)   (collective)
 * The gathered arrays live in device memory owned by the exchange, valid until the next gather on it; topic_base /
 * range_base (host, [world + 1]) give each rank's slice. A world of 1 is allowed (the gather is then a local compaction).
 * The gather reads the result's arrays on `stream` after its host synchronisation, so it returns while that work may still
 * run: bfq_device_result_release waits for it, and nothing else needs to. Errors: BFQ_E_STATE for a match that has not
 * completed (bfq_device_result_wait), BFQ_E_INVALID for a result without a match behind it.
 * ---------------------------------------------------------------------------------------------- */
#define BFQ_EXCHANGE_ID_BYTES 128
#define BFQ_EXCHANGE_COUNTS 1
#define BFQ_EXCHANGE_RANGES 2
typedef struct bfq_exchange bfq_exchange;
typedef struct {
    const uint32_t* d_route_count;   /* matched routes per topic; rank r's slice starts at topic_base[r] */
    const uint32_t* d_span_count;    /* matched ranges per topic, same slices (NULL with BFQ_EXCHANGE_COUNTS) */
    const bfq_range* d_ranges;       /* rank r's slice starts at range_base[r]; dense inside a slice: a topic's ranges follow
                                        those of the topic before it (NULL with BFQ_EXCHANGE_COUNTS) */
    const int64_t* topic_base;       /* host [world + 1]: rank r's topics are [topic_base[r], topic_base[r] + topic_count[r]) — the  */
    const int64_t* range_base;       /* host [world + 1]   slices have one padded stride (the payload travels as ncclAllGather)    */
    const int64_t* topic_count;      /* host [world] */
    const int64_t* range_count;      /* host [world] */
    int64_t n_topics_total, n_ranges_total;
    int64_t bytes_received;          /* payload bytes this rank received from its peers */
    int32_t world;
} bfq_gathered;
int32_t bfq_exchange_unique_id(uint8_t* id_out, int32_t cap);
int32_t bfq_exchange_create(int32_t device_ordinal, int32_t rank, int32_t world, const uint8_t* id, bfq_exchange** out);
void bfq_exchange_destroy(bfq_exchange* x);
int32_t bfq_exchange_gather(bfq_exchange* x, const bfq_device_result* res, int32_t what, void* stream, bfq_gathered* out);

/* ------------------------------------------------------------------------------------------------
 * Route key codec + tokeniser, native restatement of DWS/KVSchemaUtil.java:56-130 and
 * U/TopicUtil.java:42-163,206-225 (exported so the Java side / tests can cross-check bytes).
 * Each returns the produced length (or BFQ_E_*), copying only if it fits cap.
 * ---------------------------------------------------------------------------------------------- */
int64_t bfq_receiver_url(int32_t sub_broker_id, const uint8_t* receiver_id, int64_t rn, const uint8_t* deliverer_key,
                         int64_t dn, uint8_t* out, int64_t cap);
/* mqtt_topic_filter may carry a $share/<g>/ or $oshare/<g>/ prefix (=> toGroupRouteKey, receiver_url ignored) */
int64_t bfq_route_key(const uint8_t* tenant, int64_t tn, const uint8_t* mqtt_topic_filter, int64_t fn,
                      const uint8_t* receiver_url, int64_t un, uint8_t* out, int64_t cap);
int64_t bfq_tenant_begin_key(const uint8_t* tenant, int64_t tn, uint8_t* out, int64_t cap);
/* retain store key layout (bifromq-retain/bifromq-retain-store-schema/src/main/java/org/apache/bifromq/retain/store/schema/
 * KVSchemaUtil.java:44-73, LevelHash.java:31-49): retainMessageKey(tenant, topic) and retainKeyPrefix of a topic filter */
int64_t bfq_retain_key(const uint8_t* tenant, int64_t tn, const uint8_t* topic, int64_t n, uint8_t* out, int64_t cap);
int64_t bfq_retain_key_prefix(const uint8_t* tenant, int64_t tn, const uint8_t* topic_filter, int64_t fn, uint8_t* out, int64_t cap);
int32_t bfq_is_valid_topic(const uint8_t* topic, int64_t n, int32_t max_level_length, int32_t max_level, int32_t max_length);
int32_t bfq_is_valid_topic_filter(const uint8_t* tf, int64_t n, int32_t max_level_length, int32_t max_level, int32_t max_length);

/* ------------------------------------------------------------------------------------------------
 * Inverse index == IRetainTopicIndex (RS/index/IRetainTopicIndex.java:27-35; implementation replaced:
 * RS/index/RetainTopicIndex.java:35-144 over U/index/TopicLevelTrie.java:190-249) and, with
 * tenant == NULL levels, DW/TopicIndex.java:39-156. Topics are staged with add/remove, published with
 * commit, and matched BY a batch of topic filters.
 * ---------------------------------------------------------------------------------------------- */
int32_t bfq_rindex_create(int32_t device_ordinal, bfq_rindex** out);
void bfq_rindex_destroy(bfq_rindex* h);
int32_t bfq_rindex_reset(bfq_rindex* h);
/* add n topics; topic i belongs to tenant topic_tenant[i] of the tenants list; returns via ids_out[i] the
 * stable topic id (>= 0) used in match results. Adding an existing (tenant, topic) returns its id. */
int32_t bfq_rindex_add(bfq_rindex* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                       const uint8_t* topics, const int64_t* topic_off, const int32_t* topic_tenant, int64_t n,
                       int64_t* ids_out);
/* The feed of RetainStoreCoProc.load() (RS/RetainStoreCoProc.java:279-296): raw retain-store KV KEYS of a range scan. The
 * reference parses every value (a TopicMessage proto) for the topic; the key carries it too, so the index is fed from the keys
 * alone. ids_out[i] = the topic's id, or -1 for bytes that are not a retain key (skipped). */
int32_t bfq_rindex_load_keys(bfq_rindex* h, const uint8_t* keys, const int64_t* key_off, int64_t n, int64_t* ids_out);
int32_t bfq_rindex_remove(bfq_rindex* h, const uint8_t* tenant, int64_t tn, const uint8_t* topic, int64_t n);
/* Publishes the staged topics as the snapshot that bfq_rmatch reads; the snapshot's generation is the number of successful
 * commits on the handle so far (a commit with nothing changed counts too). Each tenant's trie is one region of the device arrays.
 * Delta path: a commit rebuilds only the tenants whose staged topic set changed since the last commit (an add of a new
 * (tenant, topic) or a remove of a staged one; re-adding an existing topic changes nothing). Each rebuilt tenant gets a
 * fresh region behind the existing ones, and its exact edges are inserted into the device hash table by a kernel. The
 * region it replaces, and that of a tenant whose topics were all removed, stay behind as garbage. A commit with nothing
 * changed does no device work. The commit is a full build instead (every tenant, fresh table, no garbage) when:
 *   - there is no snapshot yet, or bfq_rindex_reset ran, or bfq_rindex_load_keys ran on an empty staging set;
 *   - garbage nodes would exceed a quarter of the live nodes plus 4096;
 *   - occupied table slots, garbage included, would exceed 3/4 of the usable slots;
 *   - a node id, rank or long-name chunk id space would run out.
 * Both paths give the same answers (ids and their order) as a fresh handle given the same add / remove history and
 * committed once. The commit holds the handle lock and returns after the device is patched. */
int32_t bfq_rindex_commit(bfq_rindex* h);
/* stats[k], k < n, of the committed snapshot: 0 live topics, 1 live tenants, 2 node records (garbage included), 3 garbage
 * nodes, 4 occupied hash-table slots (garbage included), 5 usable hash-table slots, 6 full commits so far, 7 delta commits
 * so far (a commit with nothing changed counts as neither), 8 tenants whose region the last commit built (0 when nothing
 * changed), 9 device bytes held by the handle (snapshot, workspaces and key table: the sum of 12, 13 and the snapshot's),
 * 10 hash-table blocks that overflowed into the next block, 11 match workspaces the handle holds (idle in its pool or leased
 * to a call or a device result), 12 their device bytes (as each was when its last call ended), 13 device bytes of the
 * retain-key table of the current id table (bfq_rretain_keys_device; 0 until the first key call, and again after a reset) */
int32_t bfq_rindex_stats(bfq_rindex* h, int64_t* stats, int32_t n);
/* topic id -> (tenant, topic) strings, resolved against the STAGED ids: after bfq_rindex_reset ids restart at 0, so an id of an
 * earlier result may name another topic here (bfq_rresult_retain_keys resolves against the result's own snapshot instead) */
int32_t bfq_rindex_lookup(bfq_rindex* h, int64_t id, uint8_t* tenant_out, int64_t tenant_cap, int64_t* tenant_len,
                          uint8_t* topic_out, int64_t topic_cap, int64_t* topic_len);
/* match n filters; filter i is scoped to tenant filter_tenant[i]; limit[i] < 0 = unlimited, else at most
 * limit[i] ids are returned for filter i (RS/RetainStoreCoProc.java:167-190 stops after `limit` messages;
 * which ones is unspecified there too — it iterates a HashSet). NOTE: the reference applies its expiry filter INSIDE that
 * loop (it keeps iterating until `limit` LIVE messages are found, RetainStoreCoProc.java:177-188), whereas this call
 * truncates to `limit` topic ids before the caller has looked at any message: a caller that drops expired messages must
 * ask for more than `limit` (total_matches tells how many exist) or pass limit < 0 and cut after its own expiry check.
 * Thread-safe: any number of threads may match on one handle at once. Every match leases its own workspace (stream, device
 * scratch, pinned counters) from the handle's pool and holds the handle lock SHARED until its kernels have read the snapshot;
 * add / load_keys / remove / reset / commit take it exclusive, so a commit waits for the matches in flight and a match waits
 * for a running commit. A result owns its arrays; the workspace goes back to the pool when the call returns. */
int32_t bfq_rmatch(bfq_rindex* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                   const uint8_t* filters, const int64_t* filter_off, const int32_t* filter_tenant, int64_t n_filters,
                   const int64_t* limit, bfq_rresult** out);
int64_t bfq_rresult_num_filters(const bfq_rresult* r);
const int64_t* bfq_rresult_offsets(const bfq_rresult* r);            /* [n_filters+1] */
/* topic ids of filter i at [offsets[i], offsets[i + 1]). Ids are handed out in insertion order and returned in trie order, so
 * they are NOT sorted. What holds: the ids of a filter are distinct; a filter's answer depends only on the filter, its tenant
 * and the snapshot, not on the rest of the batch or where the filter sits in it; with limit[i] = k >= 0 the answer is the
 * first min(k, total) ids of the unlimited answer */
const int64_t* bfq_rresult_ids(const bfq_rresult* r, int64_t* n);
const int64_t* bfq_rresult_total_matches(const bfq_rresult* r);      /* [n_filters] matches before the limit */
/* ms[0..3]: wall time of the H2D section, the kernel section, the D2H section, the whole call; ms[4]: DEVICE time from
 * "inputs resident" to "ids expanded" (CUDA events on the call's stream); ms[5]: device time of rmatch_kernel alone;
 * ms[6]: rank ranges the kernel emitted (8 bytes each); ms[7]: filters that needed the global-scratch tier */
int32_t bfq_rresult_timings(const bfq_rresult* r, double* ms, int32_t n);
uint64_t bfq_rresult_generation(const bfq_rresult* r);               /* the snapshot the match ran on (bfq_rindex_commit) */
/* retainMessageKey of every id of the result, in result order, as one (blob, key_off[n_ids + 1]) batch: the keys of the
 * follow-up reader.get calls of RetainStoreCoProc.match (RS/RetainStoreCoProc.java:177-188). Returns the blob length (or a
 * negative BFQ_E_*); copies only if it fits blob_cap; key_off_out may be NULL. The ids are resolved against the id table of
 * the snapshot the match ran on, which the result keeps alive: a bfq_rindex_reset + reload (or a match run between a reset
 * and the next commit) still gets the keys of the topics the result matched. */
int64_t bfq_rresult_retain_keys(bfq_rindex* h, const bfq_rresult* r, uint8_t* blob_out, int64_t blob_cap, int64_t* key_off_out);
void bfq_rresult_free(bfq_rresult* r);

/* bfq_rmatch with the batch already in device memory and the answer left there. d_filters / d_filter_off[n + 1] /
 * d_filter_tenant[n] / d_limit[n] are device arrays written on `stream` (a cudaStream_t, NULL = default stream); d_limit NULL =
 * unlimited. The match runs on the leased workspace's own stream, after the work already enqueued on `stream`, and the call
 * returns once the ids are on the device: the arrays in *out are ready for any stream. The tenant list is host memory. A
 * filter_tenant outside [0, n_tenants) is found on the device and fails the whole call with BFQ_E_RANGE, leaving *out
 * empty. NULL arrays: BFQ_E_INVALID; before the first commit: BFQ_E_STATE; other errors as bfq_rmatch. Answers (offsets, ids
 * in order, totals) are bfq_rmatch's: both run the same match.
 * The arrays belong to a workspace leased to the result until bfq_rdevice_result_release, which first waits for everything
 * the library enqueued for the result (bfq_rretain_keys_device, on every stream it ran on) and then returns the workspace to
 * the handle's pool. The caller's own work that reads the arrays must be ordered before the release by the caller. */
typedef struct {
    const int64_t* d_offsets;       /* [n_filters + 1]: filter i's ids are d_ids[d_offsets[i] .. d_offsets[i + 1]) */
    const int64_t* d_ids;           /* [n_ids] */
    const int64_t* d_total;         /* [n_filters] matches before the limit */
    int64_t n_filters, n_ids;
    int64_t n_ranges;               /* rank ranges rmatch_kernel emitted (its last attempt) */
    int64_t n_overflow_filters;     /* filters that needed the global-scratch tier */
    uint64_t generation;            /* snapshot the match ran on */
    double device_ms;               /* device time from "inputs resident" to "ids expanded" (CUDA events) */
    double kernel_ms;               /* device time of rmatch_kernel (its last attempt) */
    void* lease;                    /* opaque; owned by the library until bfq_rdevice_result_release */
} bfq_rdevice_result;
int32_t bfq_rmatch_device(bfq_rindex* h, const uint8_t* tenants, const int64_t* tenant_off, int32_t n_tenants,
                          const uint8_t* d_filters, const int64_t* d_filter_off, const int32_t* d_filter_tenant, int64_t n_filters,
                          const int64_t* d_limit, void* stream, bfq_rdevice_result* out);
void bfq_rdevice_result_release(bfq_rdevice_result* res);
/* bfq_rresult_retain_keys for a device result, gathered on the device on `stream`: the retainMessageKey of every id, in result
 * order. Sizing follows bfq_expand_device: d_key_off[n_ids + 1] (int64, device) is always written, the bytes go to d_keys only
 * if *n_bytes <= cap (d_keys = NULL only sizes). Bytes are those of bfq_rresult_retain_keys on the same ids. The keys come
 * from a device table of the id table the match resolved against: built on the first key call, extended for ids added since,
 * dropped with the id table (a result taken before a reset and reload still gets its own snapshot's keys). The copy may
 * still run on `stream` when the call returns; bfq_rdevice_result_release waits for it. Calls on one result are serialised. */
int32_t bfq_rretain_keys_device(bfq_rindex* h, const bfq_rdevice_result* res, int64_t* d_key_off, uint8_t* d_keys, int64_t cap,
                                void* stream, int64_t* n_bytes);

#ifdef __cplusplus
}
#endif
#endif /* BFQ_GPUMATCH_H */
