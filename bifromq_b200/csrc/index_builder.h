// index_builder.h — host side of the forward index: staging of raw route KV pairs and the flattening of
// all tenants' filter tries into the hash-table layout of trie_layout.h.
#pragma once
#include <cstdint>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "codec.h"
#include "trie_layout.h"

namespace bfq {

// Sorted KV snapshot stored as two blobs (keys / values) with int64 offsets.
struct KVBlob {
    std::vector<uint8_t> keys, vals;
    std::vector<int64_t> koff{0}, voff{0};
    int64_t n() const { return (int64_t) koff.size() - 1; }
    sv key(int64_t i) const { return sv((const char*) keys.data() + koff[i], (size_t) (koff[i + 1] - koff[i])); }
    sv val(int64_t i) const { return sv((const char*) vals.data() + voff[i], (size_t) (voff[i + 1] - voff[i])); }
    void push(sv k, sv v) {
        keys.insert(keys.end(), k.begin(), k.end());
        vals.insert(vals.end(), v.begin(), v.end());
        koff.push_back((int64_t) keys.size());
        voff.push_back((int64_t) vals.size());
    }
    void clear() { keys.clear(); vals.clear(); koff.assign(1, 0); voff.assign(1, 0); }
};

// Where one tenant lives in a snapshot (tenants are independent key ranges: the tenant id is the key prefix).
struct TenantMeta {
    std::string tenant;
    uint32_t ordinal = 0;                  // index of its root record; first-level nodes carry ROOT_BASE + ordinal as parent id
    int64_t lo = 0, n_routes = 0;          // its routes are the ranks [lo, lo + n_routes)
    uint64_t region_base = 0, csr_slots = 0;   // its private slot region
    uint64_t seg_base = 0, seg_words = 0;      // its slice of the segment table (uint32 words)
    uint32_t pp = 0, pg = 0;               // persistent / group routes
    uint32_t pp_base = 0, pg_base = 0;     // value of the prefix-count arrays at its first rank
    int64_t tenant_nodes = 0, max_depth_nodes = 0, walk_nodes = 0, n_multi = 0, n_cont = 0;
    uint64_t big_edges = 0;                // edges in the shared tag table (children of its wide nodes)
    std::vector<uint32_t> tag_slots;       // their slot ids, in placement order (big_edges of them): what a delta commit frees
                                           //   when it replaces or removes the tenant, and rank-shifts when the tenant moves
};

// One tenant built on its own (bfq_index_commit's delta path): records carry absolute slot ids / ranks for the given bases.
// It is made in two steps, so that a commit can build many tenants in parallel before it knows where each one goes:
// build_tenant_image (trie, child-array plans, sizes) and place_tenant_image (placement and records at given bases).
struct TenantBuildState;                   // the trie and plans between the two steps (index_builder.cc)
struct TenantImage {
    TenantMeta meta;                       // after the build step: every size and count; after placing: the bases too
    bool placed = false;                   // false: not placed (yet), see place_tenant_image
    SlotVec slots;                         // csr_slots records, slot region_base + i at [i] (unless placed into a caller's buffer)
    std::vector<Slot> tag_recs;            // records of the nodes placed in the tag table, slot meta.tag_slots[i] at [i]
    Slot root;
    std::vector<uint32_t> segs;            // seg_words
    std::vector<uint8_t> rkind;            // n
    std::vector<uint32_t> pfxP, pfxG;      // n + 1: tenant-local after the build step, offset by the given bases after placing
    std::shared_ptr<TenantBuildState> state;   // released by place_tenant_image
};
// The build step: decodes the tenant's keys, builds its trie and plans its child arrays. Its routes get the ranks
// [rank_lo, rank_lo + n): a tenant's ranks depend only on the sizes of the tenants before it. Fills meta's sizes and counts
// (n_routes, csr_slots, seg_words, pp, pg, big_edges, node counts), rkind and the tenant-local prefix counts. Thread-safe for
// distinct images.
bool build_tenant_image(const KVBlob& tenant_kv, sv tenant, uint32_t ordinal, int64_t rank_lo, TenantImage* img, std::string* err);
// The place step: places a built tenant at the given bases and emits its records, into `region` (csr_slots records) or, when
// it is null, into img->slots. The children of its wide nodes claim slots in `tags` (the live tag table of the index, whose
// slot array stays on the device: only the tag bytes are touched) exactly as the full build's placement does; their records
// come back in tag_recs instead of the region. A tenant with wide edges is left unplaced (placed = false, nothing claimed)
// when `tags` is null or when it has more than `tag_room` of them. Tenants without wide edges touch no shared state, so they
// can be placed in parallel; tenants with wide edges claim from `tags` and are placed one after another.
bool place_tenant_image(TenantImage* img, uint64_t region_base, uint64_t seg_base, uint32_t pp_base, uint32_t pg_base, EdgeTable* tags,
                        uint64_t tag_room, Slot* region, std::string* err);
// Both steps at once, without a tag table: a tenant with wide edges is built but not placed
inline bool build_tenant_image(const KVBlob& tenant_kv, sv tenant, uint32_t ordinal, int64_t rank_lo, uint64_t region_base, uint64_t seg_base,
                               uint32_t pp_base, uint32_t pg_base, TenantImage* out, std::string* err) {
    return build_tenant_image(tenant_kv, tenant, ordinal, rank_lo, out, err) &&
           place_tenant_image(out, region_base, seg_base, pp_base, pg_base, nullptr, 0, nullptr, err);
}
// Runs f(i) for every i of `order` on all host cores, taking them in that order (largest task first keeps the cores busy)
void parallel_for_each(const std::vector<uint32_t>& order, const std::function<void(uint32_t)>& f);

// Everything the device needs, in host memory, plus build statistics.
struct FlatIndex {
    SlotVec slots;                            // blocked hash table (n_blocks * BLOCK_SLOTS)
    std::vector<uint8_t> tags;                // 16 tag bytes per block (kept on the host: delta commits place into a copy)
    std::vector<Slot> roots;                  // one record per tenant (key words unused)
    std::vector<uint32_t> segs;               // segment table (pairs), see trie_layout.h
    std::vector<uint8_t> rkind;               // per rank RouteKind
    std::vector<uint32_t> pfx_persistent;     // [n_routes+1] exclusive prefix count of KIND_PERSISTENT
    std::vector<uint32_t> pfx_group;          // [n_routes+1] exclusive prefix count of KIND_GROUP
    std::unordered_map<std::string, uint32_t> tenant_ordinal;
    std::vector<TenantMeta> tenants;          // in key order
    std::vector<Slot> host_roots;             // kept on the host (roots is dropped after the upload)
    uint64_t n_big_edges = 0;                 // claimed tag-table slots (the tenants' big_edges summed)
    int64_t n_routes = 0, n_nodes = 0, max_nodes_per_depth = 0, max_tenant_nodes = 0, n_multi = 0, n_cont_chunks = 0;
    uint32_t n_slots = 0, n_blocks = 0;
    int64_t overflowed_blocks = 0;
    int64_t child_hist[5] = {0, 0, 0, 0, 0};   // nodes with 0, 1, 2, 3, >=4 exact children (diagnostic)
};

// Build the flat index from a sorted KV snapshot. Returns false and sets *err on undecodable input.
bool build_flat_index(const KVBlob& kv, FlatIndex* out, std::string* err);
// The same from per-tenant blobs (one tenant each, in key order, empty ones skipped): what bfq_index_commit's full build uses.
bool build_flat_index_parts(const std::vector<const KVBlob*>& parts, FlatIndex* out, std::string* err);

// Host staging area behind bfq_index_load / bfq_index_apply / bfq_index_commit, kept PER TENANT (tenants are independent key
// ranges: a SUB / UNSUB touches one tenant, and bfq_index_commit's delta path rebuilds only the touched ones). A tenant's
// committed KV blob is immutable and shared with the snapshots that were built from it (copy-on-write on the next change).
struct TenantStage {
    std::shared_ptr<const KVBlob> base = std::make_shared<KVBlob>();   // sorted
    std::map<std::string, std::pair<bool, std::string>> delta;         // key -> (present?, value)
};
// <0x00><u16 BE len><tenant id> of a route key, or an empty view if the key is too short to carry one. Byte order of these
// prefixes == KV order of the tenants.
inline sv tenant_prefix_of(sv key) {
    if (key.size() < 3 || key[0] != 0) return sv();
    const size_t tl = ((size_t) (uint8_t) key[1] << 8) | (uint8_t) key[2];
    return key.size() < 3 + tl ? sv() : key.substr(0, 3 + tl);
}
class Staging {
public:
    void reset();
    bool load(const uint8_t* keys, const int64_t* koff, const uint8_t* vals, const int64_t* voff, int64_t n, std::string* err);
    bool upsert(sv k, sv v);   // false: the key carries no tenant prefix
    bool erase(sv k);
    bool has_delta() const;
    // tenants (by key prefix, in key order) with staged changes
    std::vector<std::string> dirty_tenants() const;
    // merges one tenant's delta into a NEW base blob (the old one may be pinned by a snapshot); erases the tenant if it ends empty
    void merge_tenant(const std::string& prefix);
    // the same for many tenants, merged on all host cores (each merge rewrites only its own TenantStage); the tenants that end
    // empty are erased afterwards, on the calling thread
    void merge_tenants(const std::vector<std::string>& prefixes);
    void merge_all();
    const std::map<std::string, TenantStage>& tenants() const { return tenants_; }
    KVBlob concat() const;     // every tenant's base, in key order (the input of a full build)
    bool bulk_changed() const { return bulk_changed_; }   // reset / load since the last commit: the next commit is a full build
    void clear_bulk_changed() { bulk_changed_ = false; }
private:
    std::map<std::string, TenantStage> tenants_;
    std::string last_loaded_;
    bool bulk_changed_ = true;
};

}  // namespace bfq
