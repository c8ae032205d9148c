// index_builder.cc — see index_builder.h.
#include "index_builder.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>

namespace bfq {

// ------------------------------------------------------------------------------------------------ staging
void Staging::reset() {
    tenants_.clear();
    last_loaded_.clear();
    bulk_changed_ = true;
}

bool Staging::load(const uint8_t* keys, const int64_t* koff, const uint8_t* vals, const int64_t* voff, int64_t n,
                   std::string* err) {
    if (n <= 0) return true;
    auto key_at = [&](int64_t i) { return sv((const char*) keys + koff[i], (size_t) (koff[i + 1] - koff[i])); };
    // validate first (nothing is staged on failure): strictly ascending, after everything loaded before, tenant prefix present
    {
        sv prev = sv(last_loaded_);
        bool have_prev = !last_loaded_.empty();
        for (int64_t i = 0; i < n; i++) {
            const sv k = key_at(i);
            if (koff[i + 1] < koff[i] || voff[i + 1] < voff[i] || (have_prev && !(prev < k))) {
                if (err) *err = "bfq_index_load: keys must be strictly ascending (and follow the keys already staged)";
                return false;
            }
            if (tenant_prefix_of(k).empty()) {
                if (err) *err = "undecodable route key at position " + std::to_string(i);
                return false;
            }
            prev = k;
            have_prev = true;
        }
    }
    // append tenant by tenant (a run of keys with one prefix is one bulk copy)
    int64_t i = 0;
    while (i < n) {
        const sv pfx = tenant_prefix_of(key_at(i));
        int64_t j = i + 1;
        while (j < n) {
            const sv k = key_at(j);
            if (k.size() < pfx.size() || memcmp(k.data(), pfx.data(), pfx.size()) != 0) break;
            j++;
        }
        TenantStage& ts = tenants_[std::string(pfx)];
        auto nb = std::make_shared<KVBlob>(*ts.base);   // copy-on-write: the old blob may be pinned by a snapshot
        const size_t k0 = nb->keys.size(), v0 = nb->vals.size();
        nb->keys.insert(nb->keys.end(), keys + koff[i], keys + koff[j]);
        nb->vals.insert(nb->vals.end(), vals + voff[i], vals + voff[j]);
        for (int64_t r = i + 1; r <= j; r++) {
            nb->koff.push_back((int64_t) k0 + koff[r] - koff[i]);
            nb->voff.push_back((int64_t) v0 + voff[r] - voff[i]);
        }
        ts.base = std::move(nb);
        i = j;
    }
    last_loaded_ = std::string(key_at(n - 1));
    bulk_changed_ = true;
    return true;
}

bool Staging::upsert(sv k, sv v) {
    const sv pfx = tenant_prefix_of(k);
    if (pfx.empty()) return false;
    tenants_[std::string(pfx)].delta[std::string(k)] = {true, std::string(v)};
    return true;
}
bool Staging::erase(sv k) {
    const sv pfx = tenant_prefix_of(k);
    if (pfx.empty()) return false;
    auto it = tenants_.find(std::string(pfx));
    if (it == tenants_.end()) return true;   // nothing of this tenant is staged: nothing to delete
    it->second.delta[std::string(k)] = {false, std::string()};
    return true;
}
bool Staging::has_delta() const {
    for (auto& kv : tenants_)
        if (!kv.second.delta.empty()) return true;
    return false;
}
std::vector<std::string> Staging::dirty_tenants() const {
    std::vector<std::string> out;
    for (auto& kv : tenants_)
        if (!kv.second.delta.empty()) out.push_back(kv.first);
    return out;
}

namespace {
void merge_stage(TenantStage& ts) {
    if (!ts.delta.empty()) {
        const KVBlob& base = *ts.base;
        auto merged = std::make_shared<KVBlob>();
        merged->keys.reserve(base.keys.size() + 256);
        merged->vals.reserve(base.vals.size() + 64);
        // the delta is a handful of keys against a base of up to millions: the runs of base keys between two delta keys are
        // copied in bulk (one lower_bound per delta key), not key by key
        const int64_t n = base.n();
        merged->koff.reserve((size_t) n + ts.delta.size() + 1);
        merged->voff.reserve((size_t) n + ts.delta.size() + 1);
        auto copy_run = [&](int64_t a, int64_t b) {   // base keys [a, b)
            if (b <= a) return;
            const int64_t k0 = (int64_t) merged->keys.size() - base.koff[(size_t) a], v0 = (int64_t) merged->vals.size() - base.voff[(size_t) a];
            merged->keys.insert(merged->keys.end(), base.keys.begin() + base.koff[(size_t) a], base.keys.begin() + base.koff[(size_t) b]);
            merged->vals.insert(merged->vals.end(), base.vals.begin() + base.voff[(size_t) a], base.vals.begin() + base.voff[(size_t) b]);
            for (int64_t r = a + 1; r <= b; r++) {
                merged->koff.push_back(k0 + base.koff[(size_t) r]);
                merged->voff.push_back(v0 + base.voff[(size_t) r]);
            }
        };
        int64_t i = 0;
        for (auto d = ts.delta.begin(); d != ts.delta.end(); ++d) {
            int64_t lo = i, hi = n;   // first base key >= the delta key (delta keys ascend, so the search starts at i)
            const sv dk(d->first);
            while (lo < hi) {
                const int64_t mid = lo + (hi - lo) / 2;
                if (base.key(mid).compare(dk) < 0) lo = mid + 1;
                else hi = mid;
            }
            copy_run(i, lo);
            i = lo;
            if (d->second.first) merged->push(d->first, d->second.second);
            if (i < n && base.key(i) == dk) i++;   // replaced or removed
        }
        copy_run(i, n);
        ts.base = std::move(merged);
        ts.delta.clear();
    }
}
}  // namespace

void Staging::merge_tenant(const std::string& prefix) {
    auto it = tenants_.find(prefix);
    if (it == tenants_.end()) return;
    merge_stage(it->second);
    if (it->second.base->n() == 0) tenants_.erase(it);
}
void Staging::merge_tenants(const std::vector<std::string>& prefixes) {
    std::vector<TenantStage*> stages;
    std::vector<uint32_t> order;
    for (auto& p : prefixes) {
        auto it = tenants_.find(p);
        if (it == tenants_.end()) continue;
        order.push_back((uint32_t) stages.size());
        stages.push_back(&it->second);
    }
    parallel_for_each(order, [&](uint32_t i) { merge_stage(*stages[i]); });
    for (auto& p : prefixes) {   // erasing from the map is not thread-safe
        auto it = tenants_.find(p);
        if (it != tenants_.end() && it->second.base->n() == 0) tenants_.erase(it);
    }
}
void Staging::merge_all() {
    std::vector<std::string> names;
    for (auto& kv : tenants_) names.push_back(kv.first);
    merge_tenants(names);
}

KVBlob Staging::concat() const {
    KVBlob out;
    size_t kb = 0, vb = 0, nn = 0;
    for (auto& kv : tenants_) {
        kb += kv.second.base->keys.size();
        vb += kv.second.base->vals.size();
        nn += (size_t) kv.second.base->n();
    }
    out.keys.reserve(kb);
    out.vals.reserve(vb);
    out.koff.reserve(nn + 1);
    out.voff.reserve(nn + 1);
    for (auto& kv : tenants_) {
        const KVBlob& b = *kv.second.base;
        const int64_t k0 = (int64_t) out.keys.size(), v0 = (int64_t) out.vals.size();
        out.keys.insert(out.keys.end(), b.keys.begin(), b.keys.end());
        out.vals.insert(out.vals.end(), b.vals.begin(), b.vals.end());
        for (int64_t r = 1; r <= b.n(); r++) {
            out.koff.push_back(k0 + b.koff[(size_t) r]);
            out.voff.push_back(v0 + b.voff[(size_t) r]);
        }
    }
    return out;
}

// ------------------------------------------------------------------------------------------------ builder
namespace {

struct Target {
    uint32_t first = 0, count = 0, total = 0, pc = 0, gc = 0;
    int32_t multi = -1;
};
struct BNode {
    uint32_t parent = NONE;   // node index of the parent (NONE for tenant roots)
    uint32_t lenw = 0;
    uint32_t tok[TOKEN_WORDS] = {0, 0, 0, 0, 0, 0};
    uint32_t plus = NONE;     // node index of the '+' child
    uint32_t flags = 0;
    uint32_t root_ordinal = NONE;
    uint32_t last_child = NONE;   // most recently created exact child (sorted-order construction, see Builder::edge)
    Target own, hash;
};

inline void make_tok(sv chunk, uint32_t* tok) {
    for (uint32_t k = 0; k < TOKEN_WORDS; k++) tok[k] = 0;
    for (size_t j = 0; j < chunk.size(); j++) tok[j >> 2] |= (uint32_t) (uint8_t) chunk[j] << (8 * (j & 3));
}

class Builder {
public:
    std::vector<BNode> nodes;
    std::vector<std::vector<std::pair<uint32_t, uint32_t>>> multi_lists;
    int64_t n_cont = 0;

    // sorted == true: the keys arrive in KV order, i.e. the filters in level-wise order, so the levels descended from one
    // parent form a NON-DECREASING sequence (build_tenant checks exactly that against last_level and falls back to the hash
    // table if it ever fails). Then every distinct child of a parent is one contiguous run, and "does this child exist?" has
    // only one candidate: the parent's most recently created child. No hash table, no random probes: the 1.4M-key tenant of
    // C4 builds in a third of the time. (A parent's OWN keys may interleave with the subtree of its empty-named child — the
    // reference's bucket-byte quirk, DESIGN.md §2 — which is a revisit of the last child too.)
    explicit Builder(bool sorted_mode = false) : sorted(sorted_mode) {
        if (!sorted) table_.assign(1u << 8, NONE);
    }
    bool sorted;
    std::vector<sv> last_level;   // sorted mode: per node, the last level descended from it (order check)
    static sv unset() {
        static const char marker = 0;
        return sv(&marker, 0);
    }

    uint32_t new_root(uint32_t ordinal) {
        nodes.emplace_back();
        nodes.back().root_ordinal = ordinal;
        return (uint32_t) nodes.size() - 1;
    }
    // find-or-create the child of `parent` along one edge key
    uint32_t edge(uint32_t parent, uint32_t lenw, const uint32_t* tok, bool* created) {
        if (sorted) {
            const uint32_t lc = nodes[parent].last_child;
            if (lc != NONE && nodes[lc].lenw == lenw && memcmp(nodes[lc].tok, tok, sizeof(nodes[lc].tok)) == 0) {
                *created = false;
                return lc;
            }
            nodes.emplace_back();
            BNode& c = nodes.back();
            c.parent = parent;
            c.lenw = lenw;
            memcpy(c.tok, tok, sizeof(c.tok));
            const uint32_t idx = (uint32_t) nodes.size() - 1;
            if (lenw != LEN_PLUS) nodes[parent].last_child = idx;
            *created = true;
            return idx;
        }
        if ((nodes.size() + 1) * 2 > table_.size()) grow();
        uint64_t h = fmix64(token_hash(lenw, tok) + (uint64_t) parent * 0xC2B2AE3D27D4EB4Full);
        size_t mask = table_.size() - 1, s = (size_t) h & mask;
        while (true) {
            uint32_t idx = table_[s];
            if (idx == NONE) break;
            const BNode& c = nodes[idx];
            if (c.parent == parent && c.lenw == lenw && memcmp(c.tok, tok, sizeof(c.tok)) == 0) {
                *created = false;
                return idx;
            }
            s = (s + 1) & mask;
        }
        nodes.emplace_back();
        BNode& c = nodes.back();
        c.parent = parent;
        c.lenw = lenw;
        memcpy(c.tok, tok, sizeof(c.tok));
        uint32_t idx = (uint32_t) nodes.size() - 1;
        table_[s] = idx;
        *created = true;
        return idx;
    }
    // descend one filter level (not '#'); created_real reports whether the level's final node is new
    // *in_order = false (sorted mode only): `level` sorts before the last level descended from `node` — the input is not in
    // level-wise order and the caller must rebuild with the hash table
    uint32_t descend(uint32_t node, sv level, bool* created_real, bool* in_order) {
        uint32_t tok[TOKEN_WORDS];
        bool created;
        if (sorted) {
            if (last_level.size() < nodes.size()) last_level.resize(std::max(nodes.size(), last_level.size() * 2), unset());
            const sv prev = last_level[node];
            if (prev.data() != unset().data() && level.compare(prev) < 0) *in_order = false;   // unsigned byte order == KV order
            last_level[node] = level;
        }
        if (level.size() == 1 && level[0] == '+') {
            if (nodes[node].plus != NONE) {
                *created_real = false;
                return nodes[node].plus;
            }
            make_tok(sv(), tok);
            uint32_t c = edge(node, LEN_PLUS, tok, &created);
            nodes[node].plus = c;
            *created_real = created;
            return c;
        }
        nodes[node].flags |= FLAG_HAS_EXACT;
        size_t off = 0;
        uint32_t j = 0;
        while (level.size() - off > TOKEN_BYTES) {  // continuation chunks of a long token
            make_tok(level.substr(off, TOKEN_BYTES), tok);
            node = edge(node, LEN_CONT | j, tok, &created);
            if (created) n_cont++;
            nodes[node].flags |= FLAG_HAS_EXACT;
            off += TOKEN_BYTES;
            j++;
        }
        make_tok(level.substr(off), tok);
        uint32_t c = edge(node, (uint32_t) level.size(), tok, created_real);
        return c;
    }
    void add_route(Target& t, uint32_t rank, RouteKind kind) {
        if (t.total == 0) {
            t.first = rank;
            t.count = 1;
        } else if (t.first + t.count == rank) {
            t.count++;
        } else {
            if (t.multi < 0) {
                t.multi = (int32_t) multi_lists.size();
                multi_lists.emplace_back();
            }
            multi_lists[t.multi].push_back({t.first, t.count});
            t.first = rank;
            t.count = 1;
        }
        t.total++;
        if (kind == KIND_PERSISTENT) t.pc++;
        else if (kind == KIND_GROUP) t.gc++;
    }

private:
    std::vector<uint32_t> table_;
    void grow() {
        std::vector<uint32_t> nt(table_.size() * 2, NONE);
        size_t mask = nt.size() - 1;
        for (uint32_t idx = 0; idx < nodes.size(); idx++) {
            const BNode& c = nodes[idx];
            if (c.parent == NONE) continue;
            uint64_t h = fmix64(token_hash(c.lenw, c.tok) + (uint64_t) c.parent * 0xC2B2AE3D27D4EB4Full);
            size_t s = (size_t) h & mask;
            while (nt[s] != NONE) s = (s + 1) & mask;
            nt[s] = idx;
        }
        table_.swap(nt);
    }
};

inline uint32_t sat16(uint32_t v) { return v > 0xFFFFu ? 0xFFFFu : v; }

}  // namespace

namespace {

struct ChildPlan { uint8_t lg; uint8_t big; uint16_t seed; };

// Everything about one tenant's trie; tenants are independent, so phases B and D run one tenant per task in parallel.
struct TenantBuild {
    sv tenant;
    const KVBlob* kv = nullptr;           // the blob its keys live in: the whole snapshot, or the tenant's own staged blob
    int64_t lo = 0, hi = 0;               // its routes are the entries [lo, hi) of *kv ...
    int64_t glo = 0;                      // ... and the ranks [glo, glo + hi - lo) of the index
    uint32_t ordinal = 0;
    Builder b;                            // local node indices; node 0 is the tenant root
    std::vector<uint32_t> child_off, child_list;
    std::vector<ChildPlan> plan;
    uint64_t csr_slots = 0, big_edges = 0, seg_words = 0;
    uint32_t pp = 0, pg = 0;              // persistent / group routes of this tenant
    int64_t max_depth_nodes = 0, tenant_nodes = 0;
    int64_t child_hist[5] = {0, 0, 0, 0, 0};
    std::string err;
    // assigned between the phases
    uint64_t region_base = 0, seg_base = 0;
    uint32_t pp_base = 0, pg_base = 0;
    int64_t n_multi = 0;
    // where the phases write (the whole-index arrays of a full build, or one tenant's private buffers of a delta build):
    // rank r of `kv` is stored in the records as r + rank_off and indexes the per-rank arrays at r + index_off
    int64_t rank_off = 0, index_off = 0;
    uint8_t* rkind = nullptr;
    uint32_t *pfxP = nullptr, *pfxG = nullptr;
    Slot* slots = nullptr;        // slot s of the device array lives at slots[s - slot_origin]
    uint64_t slot_origin = 0;
    Slot* root_rec = nullptr;
    uint32_t* segs = nullptr;     // word w of the segment table lives at segs[w - seg_origin]
    uint64_t seg_origin = 0;
    std::vector<uint32_t> tag_slots;        // phase D: the tag-table slots its wide nodes' children claimed, in placement order
    std::vector<Slot>* tag_recs = nullptr;  // delta build: the records of those children go here (tag_slots order), not to `slots`
};

// phase B, first half: decode the tenant's keys and build its trie. Returns false if the sorted-order construction met a level
// out of order (then nothing of tb.b is usable and the caller rebuilds with the hash table).
bool insert_tenant_keys(const KVBlob& kv, TenantBuild& tb, std::vector<uint32_t>& depth_count) {
    Builder& b = tb.b;
    b.nodes.reserve((size_t) (tb.hi - tb.lo) * 3 / 2 + 16);   // about what a tenant needs (C4: 1.5 nodes per route); growth copies 100-byte nodes
    const uint32_t root = b.new_root(0);
    std::vector<sv> path_levels, levels;
    std::vector<uint32_t> path_nodes;
    uint32_t pp = 0, pg = 0;
    bool in_order = true;
    sv prev_filter;
    uint32_t prev_node = root;
    bool prev_multi_wild = false;
    for (int64_t r = tb.lo; r < tb.hi; r++) {
        DecodedKey d;
        if (!decode_route_key(kv.key(r), &d)) {
            tb.err = "undecodable route key at rank " + std::to_string(r);
            return true;
        }
        tb.rkind[(size_t) (r + tb.index_off)] = (uint8_t) d.kind;
        tb.pfxP[(size_t) (r + tb.index_off)] = pp;   // tenant-local for now, rebased in phase D
        tb.pfxG[(size_t) (r + tb.index_off)] = pg;
        if (d.kind == KIND_PERSISTENT) pp++;
        else if (d.kind == KIND_GROUP) pg++;
        if (r > tb.lo && d.escaped_filter == prev_filter) {   // another route of the previous key's filter: same node, same target
            b.add_route(prev_multi_wild ? b.nodes[prev_node].hash : b.nodes[prev_node].own, (uint32_t) (r + tb.rank_off), d.kind);
            continue;
        }
        levels.clear();
        for_each_level(d.escaped_filter, '\0', [&](sv l) { levels.push_back(l); });
        const bool multi_wild = levels.back().size() == 1 && levels.back()[0] == '#';
        const size_t walk = multi_wild ? levels.size() - 1 : levels.size();
        size_t k = 0;   // reuse the longest common prefix with the previous key's path
        while (k < walk && k < path_levels.size() && path_levels[k] == levels[k]) k++;
        path_levels.resize(k);
        path_nodes.resize(k);
        uint32_t node = k ? path_nodes[k - 1] : root;
        for (; k < walk; k++) {
            bool created = false;
            node = b.descend(node, levels[k], &created, &in_order);
            if (!in_order) return false;
            if (created) {
                if (depth_count.size() <= k) depth_count.resize(k + 1, 0);
                depth_count[k]++;
                tb.tenant_nodes++;
            }
            path_levels.push_back(levels[k]);
            path_nodes.push_back(node);
        }
        b.add_route(multi_wild ? b.nodes[node].hash : b.nodes[node].own, (uint32_t) (r + tb.rank_off), d.kind);
        prev_filter = d.escaped_filter;
        prev_node = node;
        prev_multi_wild = multi_wild;
    }
    tb.pp = pp;
    tb.pg = pg;
    return true;
}

// The first level of the filter in a route key (the bytes up to the first NUL of the escaped filter), or false if undecodable.
bool first_level_of_key(sv key, sv* level) {
    DecodedKey d;
    if (!decode_route_key(key, &d)) return false;
    const size_t nul = d.escaped_filter.find('\0');
    *level = nul == sv::npos ? d.escaped_filter : d.escaped_filter.substr(0, nul);
    return true;
}

// Sorted-order construction of a LARGE tenant on several threads. The sorted key range is cut where the filter's first EDGE from
// the root changes (the first level, or its first 24-byte chunk if it is longer than one token): the sub-tries under different
// root children share nothing but the root, so every piece is built on its own (same
// code, its own root), and the pieces are concatenated — piece after piece, each in its creation order — which is exactly the
// numbering the one-thread construction gives (it creates the nodes in key order too), hence the same image
// (tests compare it with the hash-table construction byte for byte). Returns 1 = built, 0 = not applicable or order
// violation (the caller falls back to one thread), and leaves tb.err set on undecodable keys like the one-thread path.
int insert_tenant_keys_parallel(const KVBlob& kv, TenantBuild& tb, std::vector<uint32_t>& depth_count, unsigned threads) {
    const int64_t lo = tb.lo, hi = tb.hi, nkeys = hi - lo;
    // ---- cut points
    std::vector<int64_t> cuts{lo};
    for (unsigned c = 1; c < threads; c++) {
        int64_t r = lo + nkeys * (int64_t) c / (int64_t) threads;
        if (r <= cuts.back()) continue;
        sv prev, cur;
        if (!first_level_of_key(kv.key(r - 1), &prev)) return 0;
        while (r < hi) {
            if (!first_level_of_key(kv.key(r), &cur)) return 0;
            const int cmp = cur.compare(prev);
            if (cmp < 0) return 0;   // not in level-wise order: the one-thread path decides what to do with it
            // same child of the root? equal levels, or two levels longer than one token that share their first 24-byte chunk
            // (they hang off the same continuation node)
            const bool same_edge = cmp == 0 || (prev.size() > TOKEN_BYTES && cur.size() > TOKEN_BYTES &&
                                                prev.substr(0, TOKEN_BYTES) == cur.substr(0, TOKEN_BYTES));
            if (!same_edge) break;
            prev = cur;
            r++;
        }
        if (r >= hi) break;   // the rest of the range hangs off one root child: no further cut exists (and no further scan)
        if (r > cuts.back()) cuts.push_back(r);
    }
    cuts.push_back(hi);
    const size_t P = cuts.size() - 1;
    if (P < 2) return 0;
    // ---- the pieces, each with the tenant's own output arrays (ranks are absolute; the prefix counts are rebased below)
    std::vector<TenantBuild> piece(P);
    std::vector<std::vector<uint32_t>> piece_depth(P);
    std::vector<char> piece_ok(P, 1);
    {
        std::atomic<size_t> next{0};
        auto worker = [&]() {
            while (true) {
                const size_t i = next.fetch_add(1);
                if (i >= P) break;
                TenantBuild& pb = piece[i];
                pb.kv = tb.kv;
                pb.lo = cuts[i];
                pb.hi = cuts[i + 1];
                pb.rank_off = tb.rank_off;
                pb.index_off = tb.index_off;
                pb.rkind = tb.rkind;
                pb.pfxP = tb.pfxP;
                pb.pfxG = tb.pfxG;
                pb.b = Builder(true);
                piece_ok[i] = insert_tenant_keys(kv, pb, piece_depth[i]) ? 1 : 0;
            }
        };
        std::vector<std::thread> th;
        for (unsigned t = 1; t < std::min<size_t>(threads, P); t++) th.emplace_back(worker);
        worker();
        for (auto& t : th) t.join();
    }
    for (size_t i = 0; i < P; i++) {
        if (!piece[i].err.empty()) {
            tb.err = piece[i].err;
            return 1;   // reported like the one-thread path does
        }
        if (!piece_ok[i]) return 0;
    }
    // ---- concatenate: node 0 = the root, then piece after piece without their own roots
    std::vector<size_t> node_off(P + 1, 1), multi_off(P + 1, 0);
    std::vector<uint32_t> pp_base(P + 1, 0), pg_base(P + 1, 0);
    int64_t n_cont_total = 0;
    for (size_t i = 0; i < P; i++) {
        n_cont_total += piece[i].b.n_cont;
        node_off[i + 1] = node_off[i] + piece[i].b.nodes.size() - 1;
        multi_off[i + 1] = multi_off[i] + piece[i].b.multi_lists.size();
        pp_base[i + 1] = pp_base[i] + piece[i].pp;
        pg_base[i + 1] = pg_base[i] + piece[i].pg;
    }
    if (node_off[P] >= 0x7FFFFFF0ull) return 0;
    Builder& b = tb.b;
    b = Builder(true);
    b.nodes.resize(node_off[P]);
    b.multi_lists.resize(multi_off[P]);
    BNode root;
    root.root_ordinal = 0;
    int plus_owner = -1, hash_owner = -1;
    for (size_t i = 0; i < P; i++) {
        const BNode& r = piece[i].b.nodes[0];
        root.flags |= r.flags;
        if (r.plus != NONE) {
            if (plus_owner >= 0) return 0;   // cannot happen when the cuts are first-level boundaries
            plus_owner = (int) i;
        }
        if (r.hash.total > 0) {
            if (hash_owner >= 0) return 0;
            hash_owner = (int) i;
        }
        if (r.own.total > 0) return 0;   // no filter has zero levels
    }
    auto map_node = [&](size_t i, uint32_t local) { return local == NONE ? NONE : local == 0 ? 0u : (uint32_t) (node_off[i] + local - 1); };
    auto map_target = [&](size_t i, Target t) {
        if (t.multi >= 0) t.multi += (int32_t) multi_off[i];
        return t;
    };
    if (plus_owner >= 0) root.plus = map_node((size_t) plus_owner, piece[(size_t) plus_owner].b.nodes[0].plus);
    if (hash_owner >= 0) root.hash = map_target((size_t) hash_owner, piece[(size_t) hash_owner].b.nodes[0].hash);
    b.nodes[0] = root;
    {
        std::atomic<size_t> next{0};
        auto worker = [&]() {
            while (true) {
                const size_t i = next.fetch_add(1);
                if (i >= P) break;
                Builder& pb = piece[i].b;
                for (size_t l = 1; l < pb.nodes.size(); l++) {
                    BNode nd = pb.nodes[l];
                    nd.parent = map_node(i, nd.parent);
                    nd.plus = map_node(i, nd.plus);
                    nd.last_child = NONE;
                    nd.own = map_target(i, nd.own);
                    nd.hash = map_target(i, nd.hash);
                    b.nodes[node_off[i] + l - 1] = nd;
                }
                for (size_t m = 0; m < pb.multi_lists.size(); m++) b.multi_lists[multi_off[i] + m] = std::move(pb.multi_lists[m]);
                // prefix counts were counted from the piece's first key: rebase to the tenant's
                if (pp_base[i] || pg_base[i])
                    for (int64_t r = piece[i].lo; r < piece[i].hi; r++) {
                        tb.pfxP[(size_t) (r + tb.index_off)] += pp_base[i];
                        tb.pfxG[(size_t) (r + tb.index_off)] += pg_base[i];
                    }
                pb = Builder(true);   // release the piece's nodes here, on this thread
            }
        };
        std::vector<std::thread> th;
        for (unsigned t = 1; t < std::min<size_t>(threads, P); t++) th.emplace_back(worker);
        worker();
        for (auto& t : th) t.join();
    }
    if (getenv("BFQ_BUILD_TRACE"))
        fprintf(stderr, "[bfq build] tenant of %lld routes inserted as %zu pieces (%zu nodes)\n", (long long) nkeys, P, b.nodes.size());
    tb.pp = pp_base[P];
    tb.pg = pg_base[P];
    tb.tenant_nodes = 0;
    depth_count.clear();
    b.n_cont = n_cont_total;
    for (size_t i = 0; i < P; i++) {
        tb.tenant_nodes += piece[i].tenant_nodes;
        if (piece_depth[i].size() > depth_count.size()) depth_count.resize(piece_depth[i].size(), 0);
        for (size_t k = 0; k < piece_depth[i].size(); k++) depth_count[k] += piece_depth[i][k];
    }
    return 1;
}

// phase B: the tenant's trie (sorted-order construction; hash-table construction if the keys turn out not to be in level-wise
// order, or when BFQ_BUILDER=hash asks for it — both give the same node numbering, hence the same image: tests compare them),
// then the plan of the child arrays
void build_tenant(const KVBlob& kv, TenantBuild& tb) {
    static const bool force_table = [] {
        const char* e = getenv("BFQ_BUILDER");
        return e && strcmp(e, "hash") == 0;
    }();
    // a tenant of >= 2^18 routes is inserted on several threads (experiment / test switches: BFQ_INSERT_PARALLEL_MIN,
    // BFQ_INSERT_THREADS)
    static const int64_t par_min = [] {
        const char* e = getenv("BFQ_INSERT_PARALLEL_MIN");
        return e ? std::max<int64_t>(2, atoll(e)) : (int64_t) 1 << 18;
    }();
    static const unsigned par_threads = [] {
        const char* e = getenv("BFQ_INSERT_THREADS");
        return e ? (unsigned) std::min(std::max(atoi(e), 1), 64) : std::min<unsigned>(std::max(1u, std::thread::hardware_concurrency()), 16u);
    }();
    std::vector<uint32_t> depth_count;
    bool done = false;
    if (!force_table) {
        if (par_threads > 1 && tb.hi - tb.lo >= par_min) done = insert_tenant_keys_parallel(kv, tb, depth_count, par_threads) == 1;
        if (!done) {
            tb.b = Builder(true);
            tb.tenant_nodes = 0;
            tb.err.clear();
            depth_count.clear();
            done = insert_tenant_keys(kv, tb, depth_count);
        }
    }
    if (!done) {
        tb.b = Builder(false);
        tb.tenant_nodes = 0;
        depth_count.clear();
        insert_tenant_keys(kv, tb, depth_count);
    }
    if (!tb.err.empty()) return;
    Builder& b = tb.b;
    b.last_level = std::vector<sv>();
    for (uint32_t c : depth_count) tb.max_depth_nodes = std::max<int64_t>(tb.max_depth_nodes, c);
    // group the exact children by parent (counting sort)
    const size_t N = b.nodes.size();
    tb.child_off.assign(N + 1, 0);
    for (size_t i = 0; i < N; i++) {
        const BNode& nd = b.nodes[i];
        if (nd.parent != NONE && nd.lenw != LEN_PLUS) tb.child_off[nd.parent + 1]++;
    }
    for (size_t i = 0; i < N; i++) tb.child_off[i + 1] += tb.child_off[i];
    tb.child_list.resize(tb.child_off[N]);
    {
        std::vector<uint32_t> fill(tb.child_off.begin(), tb.child_off.end() - 1);
        for (size_t i = 0; i < N; i++) {
            const BNode& nd = b.nodes[i];
            if (nd.parent != NONE && nd.lenw != LEN_PLUS) tb.child_list[fill[nd.parent]++] = (uint32_t) i;
        }
    }
    // per parent choose {single child + fingerprint, perfect hash of 2^lg slots with a seed, big (global tag table)}
    tb.plan.assign(N, ChildPlan{0, 0, 0});
    static const uint32_t perfect_max = [] {   // experiment switch BFQ_PERFECT_LOG2_MAX (default PERFECT_LOG2_MAX)
        const char* e = getenv("BFQ_PERFECT_LOG2_MAX");
        const int v = e ? atoi(e) : (int) PERFECT_LOG2_MAX;
        return (uint32_t) std::min(std::max(v, 1), (int) PERFECT_LOG2_MAX);
    }();
    // parents are independent: a large tenant's plan is spread over threads (block-cyclic), each with its own scratch and
    // counters; the result does not depend on the split
    struct PlanAcc {
        uint64_t csr_slots = 0, big_edges = 0, seg_words = 0;
        int64_t child_hist[5] = {0, 0, 0, 0, 0};
    };
    auto plan_nodes = [&](size_t i0, size_t i1, PlanAcc& acc, std::vector<uint32_t>& t32, std::vector<uint32_t>& sorted,
                          std::vector<uint32_t>& stamp, uint32_t& epoch) {
    for (size_t i = i0; i < i1; i++) {
        const BNode& nd = b.nodes[i];
        const uint32_t c = tb.child_off[i + 1] - tb.child_off[i];
        acc.child_hist[std::min<uint32_t>(c, 4)]++;
        if (nd.plus != NONE) acc.csr_slots++;
        for (const Target* t : {&nd.own, &nd.hash})
            if (t->multi >= 0) acc.seg_words += 2 + 2 * (b.multi_lists[t->multi].size() + 1);
        if (c == 0) continue;
        ChildPlan& pl = tb.plan[i];
        t32.clear();
        for (uint32_t j = tb.child_off[i]; j < tb.child_off[i + 1]; j++) {
            const BNode& ch = b.nodes[tb.child_list[j]];
            t32.push_back(fold32(token_hash(ch.lenw, ch.tok)));
        }
        // Private child array of 2^lg slots addressed by child_index(fold32(token hash), seed, lg) with a seed that makes it
        // collision-free: ONE memory access per lookup, hit or miss. A random seed works with probability
        // ~exp(-c^2 / 2^(lg+1)), so the array needs ~c^2/16 slots for the 16-bit seed space to contain one: cheap for the
        // common small fan-outs, 4096 slots for 256 children, and beyond 2^PERFECT_LOG2_MAX the global tag table takes over
        // (two dependent accesses, and a warp's lanes wait for the slowest of them).
        bool big = false;
        if (c == 1) {
            pl.lg = 0;
            pl.seed = (uint16_t) (t32[0] & 0xFFFFu);
        } else {
            sorted = t32;
            std::sort(sorted.begin(), sorted.end());
            if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) big = true;   // 32-bit fold collision
            uint32_t lg = 1;
            while ((1u << lg) < c) lg++;
            if (c > 4) lg++;
            while (lg <= perfect_max && ((uint64_t) c * c) / 16 > (1ull << lg)) lg++;
            bool found = false;
            for (; !big && !found && lg <= perfect_max; lg++) {
                if (stamp.size() < (1u << lg)) stamp.assign(1u << lg, 0), epoch = 0;
                for (uint32_t seed = 0; seed < 65536 && !found; seed++) {
                    if (++epoch == 0) {   // stamp wrap-around
                        std::fill(stamp.begin(), stamp.end(), 0u);
                        epoch = 1;
                    }
                    bool ok = true;
                    for (uint32_t v : t32) {
                        uint32_t& st = stamp[child_index(v, seed, lg)];
                        if (st == epoch) { ok = false; break; }
                        st = epoch;
                    }
                    if (ok) {
                        found = true;
                        pl.lg = (uint8_t) lg;
                        pl.seed = (uint16_t) seed;
                    }
                }
                if (found) break;
            }
            if (!found) big = true;
        }
        if (big) {
            pl.big = 1;
            acc.big_edges += c;
        } else {
            acc.csr_slots += 1ull << pl.lg;
        }
    }
    };
    constexpr size_t PLAN_BLOCK = 8192;
    unsigned nthreads = N >= (1u << 18) ? std::min<unsigned>(std::max(1u, std::thread::hardware_concurrency()), 16u) : 1u;
    std::vector<PlanAcc> accs(nthreads);
    std::atomic<size_t> next_block{0};
    auto worker = [&](unsigned t) {
        std::vector<uint32_t> t32, sorted, stamp;
        uint32_t epoch = 0;
        while (true) {
            const size_t i0 = next_block.fetch_add(1) * PLAN_BLOCK;
            if (i0 >= N) break;
            plan_nodes(i0, std::min(N, i0 + PLAN_BLOCK), accs[t], t32, sorted, stamp, epoch);
        }
    };
    if (nthreads <= 1) {
        worker(0);
    } else {
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nthreads; t++) th.emplace_back(worker, t);
        for (auto& t : th) t.join();
    }
    for (const PlanAcc& a : accs) {
        tb.csr_slots += a.csr_slots;
        tb.big_edges += a.big_edges;
        tb.seg_words += a.seg_words;
        for (int k = 0; k < 5; k++) tb.child_hist[k] += a.child_hist[k];
    }
}

inline uint32_t sat8(uint32_t v) { return v > 255u ? 255u : v; }

// phase D: place the tenant's nodes (BFS inside its private region; big fan-outs into the shared tag table) and emit records
void place_tenant(TenantBuild& tb, EdgeTable& table) {
    Builder& b = tb.b;
    const size_t N = b.nodes.size();
    std::vector<uint32_t> id_of(N, NONE), child_base(N, 0), order, tag_pos;
    order.reserve(N);
    tb.tag_slots.clear();
    tb.tag_slots.reserve((size_t) tb.big_edges);
    if (tb.tag_recs) tag_pos.assign(N, NONE);   // node -> its index in tag_slots / tag_recs
    id_of[0] = ROOT_BASE + tb.ordinal;
    order.push_back(0);
    uint64_t cursor = tb.region_base;
    for (size_t qi = 0; qi < order.size(); qi++) {
        const uint32_t pi = order[qi];
        const BNode& P = b.nodes[pi];
        if (P.plus != NONE) {
            id_of[P.plus] = (uint32_t) cursor++;
            order.push_back(P.plus);
        }
        const ChildPlan& pl = tb.plan[pi];
        const uint32_t c0 = tb.child_off[pi], c1 = tb.child_off[pi + 1];
        if (c1 == c0) continue;
        if (pl.big) {
            for (uint32_t j = c0; j < c1; j++) {
                const BNode& ch = b.nodes[tb.child_list[j]];
                const uint32_t s = table.claim(id_of[pi], ch.lenw, ch.tok);   // the record (key included) is emitted below
                id_of[tb.child_list[j]] = s;
                if (tb.tag_recs) tag_pos[tb.child_list[j]] = (uint32_t) tb.tag_slots.size();
                tb.tag_slots.push_back(s);
                order.push_back(tb.child_list[j]);
            }
        } else {
            child_base[pi] = (uint32_t) cursor;
            for (uint32_t j = c0; j < c1; j++) {
                const BNode& ch = b.nodes[tb.child_list[j]];
                const uint32_t idx = pl.lg ? child_index(fold32(token_hash(ch.lenw, ch.tok)), pl.seed, pl.lg) : 0u;
                id_of[tb.child_list[j]] = (uint32_t) (cursor + idx);
                order.push_back(tb.child_list[j]);
            }
            cursor += 1ull << pl.lg;
        }
    }
    if (order.size() != N || cursor != tb.region_base + tb.csr_slots || tb.tag_slots.size() != tb.big_edges) {
        tb.err = "internal error: BFS placement did not cover the trie";
        return;
    }
    if (tb.tag_recs) tb.tag_recs->assign(tb.tag_slots.size(), Slot());
    // segment-table offsets of the multi-segment targets, in node order (a sequential pass over the few that exist), so that
    // the records themselves can be written by several threads
    std::vector<uint64_t> seg_at(b.multi_lists.size(), 0);
    {
        uint64_t seg_cursor = tb.seg_base;   // in uint32 words
        if (!b.multi_lists.empty())
            for (size_t i = 0; i < N; i++)
                for (const Target* t : {&b.nodes[i].own, &b.nodes[i].hash})
                    if (t->multi >= 0) {
                        seg_at[t->multi] = seg_cursor;
                        seg_cursor += 2 + 2 * (b.multi_lists[t->multi].size() + 1);
                        tb.n_multi++;
                    }
    }
    auto emit_target = [&](Target& t, uint32_t* first, uint32_t* count, uint32_t multi_flag, uint32_t* flags) {
        if (t.multi >= 0) {
            auto& lst = b.multi_lists[t.multi];
            lst.push_back({t.first, t.count});
            uint64_t seg_cursor = seg_at[t.multi];
            *first = (uint32_t) (seg_cursor / 2);
            *count = t.total;
            *flags |= multi_flag;
            uint32_t* sg = tb.segs - tb.seg_origin;
            sg[seg_cursor++] = (uint32_t) lst.size();
            sg[seg_cursor++] = t.total;
            for (auto& p : lst) {
                sg[seg_cursor++] = p.first;
                sg[seg_cursor++] = p.second;
            }
        } else {
            *first = t.first;
            *count = t.total;
        }
    };
    auto emit_nodes = [&](size_t i0, size_t i1) {
    for (size_t i = i0; i < i1; i++) {
        BNode& nd = b.nodes[i];
        Slot* rec;
        if (nd.parent == NONE) {
            rec = tb.root_rec;
            memset(rec->w, 0, sizeof(rec->w));
            rec->w[W_PARENT] = NONE;
        } else {
            rec = !tag_pos.empty() && tag_pos[i] != NONE ? &(*tb.tag_recs)[tag_pos[i]] : &tb.slots[id_of[i] - tb.slot_origin];
            rec->w[W_PARENT] = id_of[nd.parent];
            rec->w[W_LEN] = nd.lenw;
            for (uint32_t k = 0; k < TOKEN_WORDS; k++) rec->w[W_TOK + k] = nd.tok[k];
        }
        uint32_t flags = nd.flags & FLAG_HAS_EXACT;
        emit_target(nd.own, &rec->w[W_OWN_FIRST], &rec->w[W_OWN_COUNT], FLAG_OWN_MULTI, &flags);
        emit_target(nd.hash, &rec->w[W_HASH_FIRST], &rec->w[W_HASH_COUNT], FLAG_HASH_MULTI, &flags);
        rec->w[W_CAPS] = sat8(nd.own.pc) | (sat8(nd.own.gc) << 8) | (sat8(nd.hash.pc) << 16) | (sat8(nd.hash.gc) << 24);
        if (tb.plan[i].big) flags |= FLAG_BIG;
        rec->w[W_META] = meta_pack(flags, tb.plan[i].lg, tb.plan[i].seed);
        rec->w[W_CHILD_BASE] = child_base[i];
        rec->w[W_PLUS] = nd.plus == NONE ? NONE : id_of[nd.plus];
    }
    };
    const unsigned nthreads = N >= (1u << 18) ? std::min<unsigned>(std::max(1u, std::thread::hardware_concurrency()), 16u) : 1u;
    if (nthreads <= 1) {
        emit_nodes(0, N);
    } else {   // every node owns its record (and its targets' segment lists): disjoint writes
        constexpr size_t EMIT_BLOCK = 16384;
        std::atomic<size_t> next_block{0};
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nthreads; t++)
            th.emplace_back([&]() {
                while (true) {
                    const size_t i0 = next_block.fetch_add(1) * EMIT_BLOCK;
                    if (i0 >= N) break;
                    emit_nodes(i0, std::min(N, i0 + EMIT_BLOCK));
                }
            });
        for (auto& t : th) t.join();
    }
    // rebase the tenant-local prefix counts
    for (int64_t r = tb.lo; r < tb.hi; r++) {
        tb.pfxP[(size_t) (r + tb.index_off)] += tb.pp_base;
        tb.pfxG[(size_t) (r + tb.index_off)] += tb.pg_base;
    }
}

template <typename F>
void parallel_for_tenants(std::vector<TenantBuild>& tenants, const std::vector<uint32_t>& by_size, F&& f) {
    parallel_for_each(by_size, [&](uint32_t i) { f(tenants[i]); });
}

}  // namespace

void parallel_for_each(const std::vector<uint32_t>& order, const std::function<void(uint32_t)>& f) {
    unsigned nthreads = std::thread::hardware_concurrency();
    if (nthreads == 0) nthreads = 1;
    nthreads = std::min<unsigned>(nthreads, 64);
    nthreads = (unsigned) std::min<size_t>(nthreads, std::max<size_t>(order.size(), 1));
    std::atomic<size_t> cursor{0};
    auto worker = [&]() {
        while (true) {
            const size_t i = cursor.fetch_add(1);
            if (i >= order.size()) break;
            f(order[i]);
        }
    };
    if (nthreads <= 1) {
        worker();
        return;
    }
    std::vector<std::thread> th;
    for (unsigned t = 0; t < nthreads; t++) th.emplace_back(worker);
    for (auto& t : th) t.join();
}

namespace {

struct BuildTrace {
    bool on = getenv("BFQ_BUILD_TRACE") != nullptr;
    std::chrono::steady_clock::time_point t_prev = std::chrono::steady_clock::now();
    void lap(const char* what) {
        if (!on) return;
        const auto now = std::chrono::steady_clock::now();
        fprintf(stderr, "[bfq build] %-28s %8.1f ms\n", what, std::chrono::duration<double, std::milli>(now - t_prev).count());
        t_prev = now;
    }
};

bool tenant_id_of_key(sv k, sv* tenant) {
    if (k.size() < 3 || k[0] != 0) return false;
    const size_t tl = ((size_t) (uint8_t) k[1] << 8) | (uint8_t) k[2];
    if (k.size() < 3 + tl) return false;
    *tenant = k.substr(3, tl);
    return true;
}

bool build_from_tenants(std::vector<TenantBuild>& tenants, int64_t n, FlatIndex* out, std::string* err, BuildTrace& tr);

}  // namespace

bool build_flat_index(const KVBlob& kv, FlatIndex* out, std::string* err) {
    *out = FlatIndex();
    BuildTrace tr;
    const int64_t n = kv.n();
    // ---- phase A (serial, cheap): tenant boundaries. The tenant id is the key prefix <0x00><u16 BE len><id>.
    std::vector<TenantBuild> tenants;
    {
        sv cur;
        for (int64_t r = 0; r < n; r++) {
            sv t;
            if (!tenant_id_of_key(kv.key(r), &t)) {
                if (err) *err = "undecodable route key at rank " + std::to_string(r);
                return false;
            }
            if (tenants.empty() || t != cur) {
                if (!tenants.empty()) tenants.back().hi = r;
                if (out->tenant_ordinal.count(std::string(t))) {
                    if (err) *err = "tenant keys are not contiguous";
                    return false;
                }
                tenants.emplace_back();
                tenants.back().tenant = t;
                tenants.back().kv = &kv;
                tenants.back().lo = tenants.back().glo = r;
                tenants.back().ordinal = (uint32_t) tenants.size() - 1;
                out->tenant_ordinal.emplace(std::string(t), tenants.back().ordinal);
                cur = t;
            }
        }
        if (!tenants.empty()) tenants.back().hi = n;
    }
    tr.lap("A tenant boundaries");
    return build_from_tenants(tenants, n, out, err, tr);
}

// The same build from the staging area's per-tenant blobs (every part = one tenant's sorted KV, parts in key order): no
// concatenated copy of the whole KV, no boundary scan.
bool build_flat_index_parts(const std::vector<const KVBlob*>& parts, FlatIndex* out, std::string* err) {
    *out = FlatIndex();
    BuildTrace tr;
    std::vector<TenantBuild> tenants;
    int64_t n = 0;
    sv prev;
    for (const KVBlob* part : parts) {
        if (!part || part->n() == 0) continue;
        sv t, t_last;
        if (!tenant_id_of_key(part->key(0), &t) || !tenant_id_of_key(part->key(part->n() - 1), &t_last) || t != t_last) {
            if (err) *err = "a staged tenant blob does not hold exactly one tenant's keys";
            return false;
        }
        if (!tenants.empty() && make_tenant_begin_key(prev) >= make_tenant_begin_key(t)) {
            if (err) *err = "staged tenants are not in key order";
            return false;
        }
        tenants.emplace_back();
        TenantBuild& tb = tenants.back();
        tb.tenant = t;
        tb.kv = part;
        tb.lo = 0;
        tb.hi = part->n();
        tb.glo = n;
        tb.rank_off = tb.index_off = n;
        tb.ordinal = (uint32_t) tenants.size() - 1;
        out->tenant_ordinal.emplace(std::string(t), tb.ordinal);
        n += part->n();
        prev = t;
    }
    tr.lap("A tenant list");
    return build_from_tenants(tenants, n, out, err, tr);
}

namespace {

bool build_from_tenants(std::vector<TenantBuild>& tenants, int64_t n, FlatIndex* out, std::string* err, BuildTrace& tr) {
    auto lap = [&](const char* what) { tr.lap(what); };
    const bool trace = tr.on;
    if (n >= (int64_t) 0x7FFFFFFF) {
        if (err) *err = "too many routes for 31-bit ranks";
        return false;
    }
    out->n_routes = n;
    out->rkind.resize((size_t) n);
    out->pfx_persistent.resize((size_t) n + 1);
    out->pfx_group.resize((size_t) n + 1);
    std::vector<uint32_t> by_size(tenants.size());
    for (size_t i = 0; i < tenants.size(); i++) by_size[i] = (uint32_t) i;
    std::sort(by_size.begin(), by_size.end(), [&](uint32_t a, uint32_t b) { return tenants[a].hi - tenants[a].lo > tenants[b].hi - tenants[b].lo; });
    // ---- phase B (parallel): per-tenant trie + child-array plans
    for (auto& tb : tenants) {
        tb.rkind = out->rkind.data();
        tb.pfxP = out->pfx_persistent.data();
        tb.pfxG = out->pfx_group.data();
    }
    parallel_for_tenants(tenants, by_size, [&](TenantBuild& tb) { build_tenant(*tb.kv, tb); });
    lap("B tries + plans (parallel)");
    if (trace) {
        uint64_t big_nodes = 0, big_edges = 0, hist[6] = {0, 0, 0, 0, 0, 0};
        for (auto& tb : tenants)
            for (size_t i = 0; i < tb.plan.size(); i++)
                if (tb.plan[i].big) {
                    const uint32_t c = tb.child_off[i + 1] - tb.child_off[i];
                    big_nodes++;
                    big_edges += c;
                    hist[c <= 16 ? 0 : c <= 32 ? 1 : c <= 64 ? 2 : c <= 256 ? 3 : c <= 4096 ? 4 : 5]++;
                }
        fprintf(stderr, "[bfq build] big nodes %llu (edges %llu): fan-out <=16: %llu, <=32: %llu, <=64: %llu, <=256: %llu, <=4096: %llu, more: %llu\n",
                (unsigned long long) big_nodes, (unsigned long long) big_edges, (unsigned long long) hist[0], (unsigned long long) hist[1],
                (unsigned long long) hist[2], (unsigned long long) hist[3], (unsigned long long) hist[4], (unsigned long long) hist[5]);
    }
    // ---- phase C (serial): regions, prefix bases, the shared tag table
    uint64_t n_big_edges = 0, csr_total = 0, seg_total = 0;
    uint32_t pp = 0, pg = 0;
    int64_t total_nodes = 0;
    for (auto& tb : tenants) {
        if (!tb.err.empty()) {
            if (err) *err = tb.err;
            return false;
        }
        n_big_edges += tb.big_edges;
        tb.pp_base = pp;
        tb.pg_base = pg;
        pp += tb.pp;
        pg += tb.pg;
        tb.seg_base = seg_total;
        seg_total += tb.seg_words;
        total_nodes += (int64_t) tb.b.nodes.size();
        out->max_nodes_per_depth = std::max(out->max_nodes_per_depth, tb.max_depth_nodes);
        out->max_tenant_nodes = std::max(out->max_tenant_nodes, tb.tenant_nodes);
        out->n_cont_chunks += tb.b.n_cont;
        for (int i = 0; i < 5; i++) out->child_hist[i] += tb.child_hist[i];
    }
    out->pfx_persistent[(size_t) n] = pp;
    out->pfx_group[(size_t) n] = pg;
    out->n_nodes = total_nodes;
    EdgeTable table;
    table.init(n_big_edges, /*fill=*/false);
    const uint64_t csr_base = (uint64_t) table.n_blocks * BLOCK_SLOTS;
    for (auto& tb : tenants) {
        tb.region_base = csr_base + csr_total;
        csr_total += tb.csr_slots;
    }
    if (csr_base + csr_total >= 0x7FFFFFF0ull) {
        if (err) *err = "index too large for 31-bit slot ids";
        return false;
    }
    table.slots.resize((size_t) (csr_base + csr_total));   // uninitialised; filled (first-touched) in parallel below
    {
        const size_t total = table.slots.size(), piece = 1u << 16;
        std::atomic<size_t> next{0};
        unsigned nt = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
        auto worker = [&]() {
            while (true) {
                const size_t at = next.fetch_add(piece);
                if (at >= total) break;
                fill_empty_slots(table.slots.data() + at, std::min(piece, total - at));
            }
        };
        std::vector<std::thread> th;
        for (unsigned t = 1; t < nt; t++) th.emplace_back(worker);
        worker();
        for (auto& t : th) t.join();
    }
    out->roots.assign(tenants.size(), Slot());
    out->segs.assign((size_t) std::max<uint64_t>(seg_total, 2), 0);
    lap("C regions + allocation");
    // ---- phase D (parallel): placement + record emission (tag-table claims are atomic)
    for (auto& tb : tenants) {
        tb.slots = table.slots.data();
        tb.root_rec = &out->roots[tb.ordinal];
        tb.segs = out->segs.data();
    }
    parallel_for_tenants(tenants, by_size, [&](TenantBuild& tb) { place_tenant(tb, table); });
    out->tenants.clear();
    out->tenants.reserve(tenants.size());
    for (auto& tb : tenants) {
        if (!tb.err.empty()) {
            if (err) *err = tb.err;
            return false;
        }
        out->n_multi += tb.n_multi;
        TenantMeta m;
        m.tenant = std::string(tb.tenant);
        m.ordinal = tb.ordinal;
        m.lo = tb.glo;
        m.n_routes = tb.hi - tb.lo;
        m.region_base = tb.region_base;
        m.csr_slots = tb.csr_slots;
        m.seg_base = tb.seg_base;
        m.seg_words = tb.seg_words;
        m.pp = tb.pp;
        m.pg = tb.pg;
        m.pp_base = tb.pp_base;
        m.pg_base = tb.pg_base;
        m.tenant_nodes = (int64_t) tb.b.nodes.size();
        m.max_depth_nodes = tb.max_depth_nodes;
        m.walk_nodes = tb.tenant_nodes;
        m.n_multi = tb.n_multi;
        m.n_cont = tb.b.n_cont;
        m.big_edges = tb.big_edges;
        m.tag_slots = std::move(tb.tag_slots);
        out->tenants.push_back(std::move(m));
    }
    out->n_big_edges = n_big_edges;
    out->host_roots = out->roots;
    lap("D placement (parallel)");
    out->n_blocks = table.n_blocks;
    out->n_slots = (uint32_t) table.slots.size();
    out->overflowed_blocks = table.overflowed_blocks;
    out->slots = std::move(table.slots);
    out->tags = std::move(table.tags);
    // the per-tenant build state (gigabytes of nodes at 10M filters) is released by the workers, not by one thread on return
    parallel_for_tenants(tenants, by_size, [](TenantBuild& tb) {
        tb.b = Builder();
        std::vector<uint32_t>().swap(tb.child_off);
        std::vector<uint32_t>().swap(tb.child_list);
        std::vector<ChildPlan>().swap(tb.plan);
    });
    lap("E release build state");
    return true;
}

}  // namespace

// the trie and plans of one tenant between build_tenant_image and place_tenant_image
struct TenantBuildState {
    std::string tenant;   // tb.tenant views it
    TenantBuild tb;
};

bool build_tenant_image(const KVBlob& tkv, sv tenant, uint32_t ordinal, int64_t rank_lo, TenantImage* img, std::string* err) {
    *img = TenantImage();
    auto state = std::make_shared<TenantBuildState>();
    state->tenant = std::string(tenant);
    TenantBuild& tb = state->tb;
    const int64_t n = tkv.n();
    tb.tenant = state->tenant;
    tb.lo = 0;
    tb.hi = n;
    tb.ordinal = ordinal;
    tb.rank_off = rank_lo;
    tb.index_off = 0;
    img->rkind.assign((size_t) n, 0);
    img->pfxP.assign((size_t) n + 1, 0);
    img->pfxG.assign((size_t) n + 1, 0);
    tb.rkind = img->rkind.data();
    tb.pfxP = img->pfxP.data();
    tb.pfxG = img->pfxG.data();
    build_tenant(tkv, tb);
    if (!tb.err.empty()) {
        if (err) *err = tb.err;
        return false;
    }
    TenantMeta& m = img->meta;
    m.tenant = state->tenant;
    m.ordinal = ordinal;
    m.lo = rank_lo;
    m.n_routes = n;
    m.csr_slots = tb.csr_slots;
    m.seg_words = tb.seg_words;
    m.pp = tb.pp;
    m.pg = tb.pg;
    m.tenant_nodes = (int64_t) tb.b.nodes.size();
    m.max_depth_nodes = tb.max_depth_nodes;
    m.walk_nodes = tb.tenant_nodes;
    m.n_cont = tb.b.n_cont;
    m.big_edges = tb.big_edges;
    img->state = std::move(state);
    return true;
}

bool place_tenant_image(TenantImage* img, uint64_t region_base, uint64_t seg_base, uint32_t pp_base, uint32_t pg_base, EdgeTable* tags,
                        uint64_t tag_room, Slot* region, std::string* err) {
    if (!img->state) {
        if (err) *err = "internal error: a tenant image is placed that was not built, or twice";
        return false;
    }
    TenantBuild& tb = img->state->tb;
    TenantMeta& m = img->meta;
    const int64_t n = m.n_routes;
    m.region_base = region_base;
    m.seg_base = seg_base;
    m.pp_base = pp_base;
    m.pg_base = pg_base;
    if (tb.big_edges > 0 && (!tags || tb.big_edges > tag_room)) return true;   // not placed: the caller decides
    tb.region_base = region_base;
    tb.seg_base = seg_base;
    tb.pp_base = pp_base;
    tb.pg_base = pg_base;
    tb.rkind = img->rkind.data();
    tb.pfxP = img->pfxP.data();
    tb.pfxG = img->pfxG.data();
    if (!region) {
        img->slots.resize((size_t) tb.csr_slots);
        region = img->slots.data();
    }
    {   // uninitialised; filled (first-touched) by several threads when the tenant is large
        const size_t total = (size_t) tb.csr_slots, piece = 1u << 16;
        const unsigned nt = total >= (1u << 20) ? std::min<unsigned>(std::max(1u, std::thread::hardware_concurrency()), 16u) : 1u;
        std::atomic<size_t> next{0};
        auto worker = [&]() {
            while (true) {
                const size_t at = next.fetch_add(piece);
                if (at >= total) break;
                fill_empty_slots(region + at, std::min(piece, total - at));
            }
        };
        std::vector<std::thread> th;
        for (unsigned t = 1; t < nt; t++) th.emplace_back(worker);
        worker();
        for (auto& t : th) t.join();
    }
    img->segs.assign((size_t) tb.seg_words, 0);
    tb.slots = region;
    tb.slot_origin = region_base;
    tb.root_rec = &img->root;
    tb.segs = img->segs.data();
    tb.seg_origin = seg_base;
    tb.tag_recs = &img->tag_recs;
    EdgeTable unused;
    place_tenant(tb, tags ? *tags : unused);
    if (!tb.err.empty()) {
        if (err) *err = tb.err;
        return false;
    }
    img->pfxP[(size_t) n] = pp_base + tb.pp;
    img->pfxG[(size_t) n] = pg_base + tb.pg;
    m.n_multi = tb.n_multi;
    m.tag_slots = std::move(tb.tag_slots);
    img->placed = true;
    img->state.reset();
    return true;
}

}  // namespace bfq
