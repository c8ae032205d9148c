// fanout.h — fan-out expansion (fanout.cu): parameters of the device pass and the host-side deliverer interning.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/bfq_gpumatch.h"
#include "codec.h"
#include "index_builder.h"

namespace bfq {

constexpr uint32_t FO_GROUP_BIT = 0x80000000u;   // in rdeliv[rank]: the route is a shared subscription, low bits = group index

struct FanoutParams {
    // the surviving routes of a completed match as a device CSR (bfq_expand_device)
    int64_t n_topics;
    const int64_t* offsets;          // [n_topics + 1]
    int64_t n_pairs;                 // offsets[n_topics]
    const int64_t* ranks;            // [n_pairs]
    // per-snapshot tables
    const uint32_t* rdeliv;          // [n_routes] deliverer id, or FO_GROUP_BIT | group index
    const uint32_t* gmem_off;        // [n_groups + 1] members of group g: gmem_deliv[gmem_off[g] .. gmem_off[g + 1])
    const uint32_t* gmem_deliv;      // deliverer id of every member
    const uint8_t* gordered;         // [n_groups] 1 = $oshare (left to the host)
    uint32_t n_deliverers;           // ids are [0, n_deliverers); the last one is the reserved "ordered share" id
    // scratch, fanout_scratch_words() each: the tile pass's [deliverer][tile] count matrix and its scan, or the global pass's
    // D + 1 counts and their scan (the write cursors)
    uint32_t* counts;
    uint32_t* base;
    // outputs
    long long* pack_offsets;         // [n_deliverers + 1]
    uint32_t* pack_topic;            // [n_pairs]
    uint32_t* pack_rank;             // [n_pairs]
    uint32_t* pack_member;           // [n_pairs] member index of a shared subscription, 0xFFFFFFFF otherwise
};
// true: the shared-memory tile pass fits (few deliverers for the batch); false: the global pass. Both give the same grouping.
bool fanout_tiled(uint32_t n_deliverers, int64_t n_pairs);
size_t fanout_scratch_words(uint32_t n_deliverers, int64_t n_pairs, bool tiled);
// d_tmp == nullptr: query the scan scratch size
cudaError_t launch_fanout(const FanoutParams& p, bool tiled, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream);

// The ordered shared subscriptions of a delivery nesting resolved per publisher (RendezvousHash over each member's
// receiverUrl). An "item" is one ($oshare pair, publisher); a "sub-pack" the publishers of one pair that picked the same member.
// Pair arrays below are sized for the pairs AND the sub-packs: the nesting then holds emit_cap = n_pairs + n_items slots.
struct OshareParams {
    // inputs
    const int64_t* pub_off;          // [n_topics + 1] publishers of topic position t: pub_hash[pub_off[t] .. pub_off[t + 1])
    const int32_t* pub_hash;         // [n_pubs] ClientInfo.hashCode() of each publisher
    int64_t n_pubs;
    // per-snapshot member receiverUrls: member m's bytes sit at byte 4 of the 8-byte words from url_word[m] on, zero before and
    // after, so LE32(hash) ‖ url is read as whole aligned words (bfq_delivery_device_ordered builds them on first use)
    const unsigned long long* url_words;
    const long long* url_word;       // [n_members]
    const uint32_t* url_len;         // [n_members]
    uint32_t member_bits;            // bits_for(largest $oshare group): a pick, or the group size for "no winner", fits
    // phase 1 (sized by the host): flags and item counts per CSR pair, their scans, the pub_off check
    uint32_t* oflag;                 // [n_pairs + 1] 1 = an $oshare pair with members in a nested topic; scanned in place
    unsigned long long* oitems;      // [n_pairs + 1] its publishers; scanned in place
    unsigned long long* check;       // [4]: opairs, items, bad pub_off, offsets[n_topics] (written by launch_oshare_count)
    // phase 2 (sized by the host after reading check[]): n_opairs and n_items known
    int64_t n_opairs, n_items;
    unsigned long long* okey[2];     // [n_opairs] each: (topic position << 32 | rank), sorted
    uint32_t* istart;                // [n_opairs + 1] first item of every sorted $oshare pair
    unsigned long long* ikey[2];     // [n_items] each: (sorted pair << member_bits | pick), sorted (stable: publishers in order)
    uint32_t* ival[2];               // [n_items] each: ... and the publisher position
    uint32_t* ihead;                 // [n_items + 1] 1 where (pair, pick) changes, scanned in place: the item's sub-pack
    uint32_t* sub_start;             // [n_items + 1] first item of every sub-pack ([n_subs] = n_items)
    uint32_t* sub_pack;              // [n_items] the pack each sub-pack became
    uint32_t* e_sub;                 // [emit_cap] per emit position: its sub-pack or 0xFFFFFFFF
    uint32_t* s_sub;                 // [emit_cap] per nested pair: ditto
    uint32_t* pub_count;             // [emit_cap + 1] publishers per pack (0 for a whole pack), scanned into pack_pub_off
    // outputs
    long long* pack_pub_off;         // [emit_cap + 1] (n_packs + 1 used)
    uint32_t* pack_pub;              // [n_items]
};

// The same pairs nested the way the deliverer's batcher sends them: deliverer -> package (tenant) -> pack (topic position)
// -> MatchInfos. Deliverer ids and member picks are the fan-out's (the same device function resolves both).
struct DeliveryParams {
    FanoutParams f;                  // the CSR and the per-snapshot tables; f's scratch and outputs are not used
    const int32_t* topic_tenant;     // [n_topics] the match's tenant index per topic position
    int32_t n_tenants;
    // scratch
    uint32_t* tkey[2];               // [n_topics] each: the tenant sort's keys (double buffer)
    uint32_t* tval[2];               // [n_topics] each: ... and topic positions
    uint32_t* tcount;                // [n_topics + 1] pairs per topic in tenant-major order
    uint32_t* tstart;                // [n_topics + 1] their exclusive scan: [n_topics] = pairs nested
    // the [n_pairs] arrays below are [n_pairs + o.n_items] with oshare (the sub-packs' emit positions)
    uint32_t* key[2];                // [n_pairs] each: the deliverer partition's keys (double buffer)
    uint32_t* val[2];                // [n_pairs] each: ... and emit positions
    uint32_t* e_topic;               // [n_pairs] per emit position: tenant-major topic index, rank, member
    uint32_t* e_rank;
    uint32_t* e_member;
    uint32_t* s_topic;               // [n_pairs] per nested pair: tenant-major topic index
    uint32_t* package_head;          // [n_pairs + 1] 1 where (deliverer, tenant) changes, scanned in place (exclusive)
    uint32_t* pack_head;             // [n_pairs + 1] 1 where (deliverer, topic) changes, scanned in place (exclusive)
    uint32_t* pcount;                // [n_deliverers + 1] packages per deliverer
    unsigned long long* totals;      // [4] pairs nested, packages, packs, offsets[n_topics] (+ [4] sub-packs with oshare)
    // outputs
    long long* package_off;          // [n_deliverers + 1]
    uint32_t* package_tenant;        // [n_pairs] (n_packages used)
    long long* pack_off;             // [n_pairs + 1] (n_packages + 1 used)
    uint32_t* pack_topic;            // [n_pairs] (n_packs used)
    long long* match_off;            // [n_pairs + 1] (n_packs + 1 used)
    uint32_t* match_rank;            // [n_pairs]
    uint32_t* match_member;          // [n_pairs]
    // $oshare resolution (bfq_delivery_device_ordered); oshare == false: $oshare pairs stay under the ordered-share id
    bool oshare;
    OshareParams o;
};

// d_tmp == nullptr: query the scratch size of the sorts and scans. Enqueues everything on `stream`; totals[] is written last
// (with q.oshare: [4] = sub-packs).
cudaError_t launch_delivery(const DeliveryParams& q, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream);
// Phase 1 of the $oshare resolution: flags, item counts and the pub_off check into o.check[] (the host reads them to size
// phase 2, which is launch_delivery with q.oshare set). d_tmp == nullptr: query the scan scratch size.
cudaError_t launch_oshare_count(const DeliveryParams& q, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream);

// (subBrokerId, delivererKey) -> dense id, append-only and shared by every snapshot of an index (ids stay valid across commits
// and resets, and are never freed)
struct DelivererTable {
    std::mutex mu;
    std::unordered_map<std::string, uint32_t> ids;
    std::vector<std::pair<int32_t, std::string>> list;
    uint32_t intern(int32_t broker, sv key);
};

// one tenant's routes resolved to deliverer ids (built once per tenant KV blob, reused by the snapshots that share the blob)
struct TenantFan {
    std::vector<uint32_t> rdeliv;        // per local rank; FO_GROUP_BIT | tenant-local group index for shared subscriptions
    std::vector<uint32_t> gmem_off;      // tenant-local
    std::vector<uint32_t> gmem_deliv;
    std::vector<uint8_t> gordered;
    // receiverUrl of every member of an ordered group (empty for the members of other groups): member m is
    // ourl[ourl_off[m] .. ourl_off[m + 1]); the $oshare pick hashes it
    std::vector<uint32_t> ourl_off;
    std::string ourl;
};
bool build_tenant_fan(const KVBlob& kv, DelivererTable* table, TenantFan* out, std::string* err);

// one tenant's MatchInfos as wire bytes (built once per tenant KV blob, like TenantFan): entry e is the whole `matchInfo = 3`
// field of a DeliveryPack (tag, length, MatchInfo) as NormalMatching / GroupMatching build it from the route key and value
// (DWS/cache/RouteDetailCache.java:53-109, ReceiverCache.java:32-36). One entry per normal route, one per member of a group in
// the fan-out's member order; a member-less group has none.
struct TenantWire {
    std::vector<uint32_t> first;         // per local rank: its entry (a group's first member's)
    std::vector<uint64_t> off;           // [entries + 1]: entry e is bytes[off[e] .. off[e + 1])
    std::string bytes;
};
bool build_tenant_wire(const KVBlob& kv, TenantWire* out, std::string* err);

// bfq_delivery_encode: a delivery nesting (launch_delivery's outputs) as one DeliveryRequest per deliverer (delivery_wire.cu)
struct WireParams {
    // the nesting
    int64_t n_packages, n_packs, n_pairs;
    uint32_t n_deliverers;               // the last id is ordered_share_id: its span is left empty
    const long long* package_off;        // [n_deliverers + 1]
    const uint32_t* package_tenant;      // [n_packages]
    const long long* pack_off;           // [n_packages + 1]
    const uint32_t* pack_topic;          // [n_packs]
    const long long* match_off;          // [n_packs + 1]
    const uint32_t* match_rank;          // [n_pairs]
    const uint32_t* match_member;        // [n_pairs]
    const long long* pack_pub_off;       // [n_packs + 1] or nullptr (every pack is whole)
    const uint32_t* pack_pub;
    // the batch: tenants (device copy of the match's list), topics, publisher packs
    const uint8_t* tenants;
    const long long* tenant_off;         // [n_tenants + 1]
    const uint8_t* topics;
    const long long* topic_off;          // [n_topics + 1]
    int64_t n_topics;
    const long long* pub_off;            // [n_topics + 1]
    const uint8_t* pubpack;
    const long long* pubpack_off;        // [n_pubs + 1], n_pubs = pub_off[n_topics]
    // the snapshot's MatchInfo table
    const uint32_t* mi_first;            // per rank
    const unsigned long long* mi_off;    // [entries + 1]
    const uint8_t* mi_bytes;
    // scratch
    unsigned long long* pair_pos;        // [n_pairs + 1] MatchInfo field bytes per pair, scanned
    unsigned long long* pack_pos;        // [n_packs + 1] pack field bytes, scanned
    unsigned long long* package_pos;     // [n_packages + 1] map entry field bytes, scanned
    unsigned long long* check;           // [4]: bad pub_off / pubpack_off / pack_pub, total bytes, MatchInfos encoded
    // outputs
    long long* req_off;                  // [n_deliverers + 1]
    uint8_t* out;
};
// pass 1 (sizes, req_off, check[]); d_tmp == nullptr: query the scan scratch size
cudaError_t launch_wire_size(const WireParams& p, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream);
// pass 2: the bytes (after pass 1 and a total that fits the caller's buffer)
cudaError_t launch_wire_write(const WireParams& p, cudaStream_t stream);

// bfq_delivery_reply: every deliverer's DeliveryReply joined back to the pairs of a nesting (delivery_reply.cu)
enum { RP_BAD_OFF = 0, RP_VALUE_BYTES = 1, RP_N_FALLBACK = 2, RP_N_STALE = 3, RP_N_CODE = 4, RP_CTR_N = 12 };
enum { RP_NO_RESULT = 5, RP_NOT_SENT = 6, RP_UNDECIDED = 7 };
// DeliveryResults spans are cut into chunks of RP_CHUNK_MIN bytes, or more when the replies' results exceed RP_MAX_CHUNKS of them
constexpr long long RP_CHUNK_MIN = 2048;
constexpr unsigned long long RP_MAX_CHUNKS = 1ull << 20;
struct ReplyParams {
    // the nesting
    int64_t n_packages, n_packs, n_pairs;
    uint32_t n_deliverers;               // the last id is ordered_share_id: its pairs were never sent
    const long long* package_off;        // [n_deliverers + 1]
    const uint32_t* package_tenant;      // [n_packages]
    const long long* pack_off;           // [n_packages + 1]
    const long long* match_off;          // [n_packs + 1]
    const uint32_t* match_rank;          // [n_pairs]
    const uint32_t* match_member;        // [n_pairs]
    // device copy of the match's tenant list
    const uint8_t* tenants;
    const long long* tenant_off;         // [n_tenants + 1]
    // the snapshot's MatchInfo table and the hash of every entry's MatchInfo
    const uint32_t* mi_first;
    const unsigned long long* mi_off;
    const uint8_t* mi_bytes;
    const uint32_t* mi_hash;
    // the replies
    const uint8_t* reply;
    const long long* reply_off;          // [n_deliverers + 1]
    // scratch
    unsigned long long* ctr;             // [RP_CTR_N]
    uint8_t* dl_fail;                    // per deliverer
    int32_t* dl_code;                    // per deliverer: the reply code
    uint32_t* dl_entries;                // per deliverer: its map entries, at slots package_off[d] ..
    long long *ent_s, *ent_e;            // per entry slot [n_packages]: the map entry's bytes
    long long *ent_vs, *ent_ve;          // its DeliveryResults bytes
    uint32_t* ent_pkg;                   // the package its tenant key names
    uint8_t* ent_bad;                    // its results could not be walked
    uint32_t* pkg_claimed;               // per package: a map entry named it
    unsigned long long* chunk_base;      // [n_packages + 1] chunks per entry slot, scanned
    long long *ch_guess, *ch_exit, *ch_start;   // per chunk [RP_MAX_CHUNKS + n_packages]
    unsigned long long* slot_key;        // [table_mask + 1]: package << 32 | MatchInfo entry, ~0 empty
    uint32_t *slot_pair, *slot_code, *slot_rlen;
    unsigned long long* slot_rpos;
    uint64_t table_mask;
    uint32_t* pair_slot;                 // [n_pairs]
    unsigned long long *pkg_stale, *pkg_cursor;   // [n_packages + 1]
    uint32_t *stale_list, *sort_key_in, *sort_key_out, *sort_val_in, *sort_val_out;   // [stale_cap]
    int64_t stale_cap;
    // outputs
    uint8_t* pair_code;                  // [n_pairs]
    uint8_t* status;                     // [n_deliverers]
    bfq_stale_match* stale;              // [stale_cap]
};
// the MatchInfo hash of every table entry (once per snapshot)
cudaError_t launch_mi_hash(const uint8_t* bytes, const unsigned long long* off, int64_t n_entries, uint32_t* out, cudaStream_t stream);
// every stage of the join; d_tmp == nullptr: query the scan / sort scratch size
cudaError_t launch_reply(const ReplyParams& p, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream);

}  // namespace bfq
