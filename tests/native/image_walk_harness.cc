// image_walk_harness.cc — TEST INFRASTRUCTURE (never linked into the product): walks publish topics through the flat index image
// the host builder produces (bifromq_b200/csrc/index_builder.cc, layout bifromq_b200/csrc/trie_layout.h) on the CPU, the way the
// kernels look things up — tenant root, exact child through the single-child fingerprint / per-node perfect hash / global
// tag table, '+' child slot, inlined '#' range, continuation chunks of long levels, segment table of split rank runs, the
// '$' rule — and writes every topic's matched route ranks. tests/test_host_cpu.py compares them with the oracle's, so the host
// half of the product (staging, key decoding, trie construction, child-array plans, placement, record emission) is checked
// against the reference semantics without a GPU. It applies no caps (those are the caps kernel's).
//
//   image_walk <dir>      reads  <dir>/keys.bin koff.bin vals.bin voff.bin   (sorted route KV, int64 offsets)
//                                <dir>/tenants.bin tenant_off.bin            (tenant ids of the batch)
//                                <dir>/topics.bin topic_off.bin topic_tenant.bin (int32)
//                                <dir>/deltas.bin (optional)  records: u8 op (1 = upsert, 2 = erase), u32 klen, key, u32 vlen, val
//                         writes <dir>/out_off.bin (int64[n + 1]) out_ranks.bin (int64, ascending per topic)
//   image_walk <dir> dump  also writes <dir>/dump.txt: the image's tag-table size, then for every topic read as a node path
//                          (its levels as exact edges, '+' as the '+' child) the node reached at each depth with its record id
//                          and child lookup, then every tag block's 16 bytes:
//                            n_blocks <n>
//                            node <topic> <depth> <id or NONE> <none|single|perfect|big> <lg> <seed or fingerprint>
//                            tags <block> <32 hex digits, byte 0 first>
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "index_builder.h"
using namespace bfq;
int32_t bfq::set_error(int32_t code, const std::string&) { return code; }

template <typename T>
static std::vector<T> slurp(const std::string& path, bool optional = false) {
    std::ifstream f(path, std::ios::binary | std::ios::ate);
    if (!f) {
        if (optional) return {};
        fprintf(stderr, "cannot read %s\n", path.c_str());
        exit(2);
    }
    const std::streamsize bytes = f.tellg();
    f.seekg(0);
    std::vector<T> v((size_t) bytes / sizeof(T));
    if (bytes) f.read((char*) v.data(), bytes);
    return v;
}

struct Image {
    FlatIndex f;
    EdgeTable tag;   // view of the tag-table part (find())
    const Slot& rec(uint32_t id) const { return id >= ROOT_BASE ? f.host_roots[id - ROOT_BASE] : f.slots[id]; }
    uint32_t exact_child(uint32_t pid, uint32_t lenw, const uint32_t* tok) const {
        const Slot& p = rec(pid);
        const uint32_t meta = p.w[W_META];
        if (!(meta & FLAG_HAS_EXACT)) return NONE;
        uint32_t cand;
        if (meta & FLAG_BIG) {
            return tag.find(pid, lenw, tok);
        } else {
            const uint32_t lg = meta_log2size(meta), sd = meta >> 16, t32 = fold32(token_hash(lenw, tok));
            if (lg == 0) {
                if ((t32 & 0xFFFFu) != sd) return NONE;   // the fingerprint filters most misses without touching the slot
                cand = p.w[W_CHILD_BASE];
            } else {
                cand = p.w[W_CHILD_BASE] + child_index(t32, sd, lg);
            }
        }
        const Slot& c = f.slots[cand];
        if (c.w[W_PARENT] != pid || c.w[W_LEN] != lenw) return NONE;
        for (uint32_t k = 0; k < TOKEN_WORDS; k++)
            if (c.w[W_TOK + k] != tok[k]) return NONE;
        return cand;
    }
    // the child of `pid` along one topic level (any length: 24-byte continuation chunks, then the final edge)
    uint32_t level_child(uint32_t pid, sv level) const {
        uint32_t tok[TOKEN_WORDS];
        auto make = [&](sv chunk) {
            for (uint32_t k = 0; k < TOKEN_WORDS; k++) tok[k] = 0;
            for (size_t j = 0; j < chunk.size(); j++) tok[j >> 2] |= (uint32_t) (uint8_t) chunk[j] << (8 * (j & 3));
        };
        size_t off = 0;
        uint32_t j = 0, node = pid;
        while (level.size() - off > TOKEN_BYTES) {
            make(level.substr(off, TOKEN_BYTES));
            node = exact_child(node, LEN_CONT | j, tok);
            if (node == NONE) return NONE;
            off += TOKEN_BYTES;
            j++;
        }
        make(level.substr(off));
        return exact_child(node, (uint32_t) level.size(), tok);
    }
    void emit(uint32_t first, uint32_t count, bool multi, std::vector<int64_t>* out) const {
        if (count == 0) return;
        if (!multi) {
            for (uint32_t r = 0; r < count; r++) out->push_back((int64_t) first + r);
            return;
        }
        const uint32_t* sg = f.segs.data() + 2 * (size_t) first;
        const uint32_t nseg = sg[0];
        uint32_t total = 0;
        for (uint32_t s = 0; s < nseg; s++) {
            for (uint32_t r = 0; r < sg[2 + 2 * s + 1]; r++) out->push_back((int64_t) sg[2 + 2 * s] + r);
            total += sg[2 + 2 * s + 1];
        }
        if (total != count || sg[1] != count) {
            fprintf(stderr, "segment table disagrees with the record's route count\n");
            exit(3);
        }
    }
    void match(uint32_t root, sv topic, std::vector<int64_t>* out) const {
        std::vector<sv> levels;
        for_each_level(topic, '/', [&](sv l) { levels.push_back(l); });
        const bool sys = !levels.empty() && !levels[0].empty() && levels[0][0] == '$';
        std::vector<uint32_t> frontier{root}, next;
        const size_t n = levels.size();
        for (size_t i = 0; i <= n; i++) {
            next.clear();
            for (uint32_t pid : frontier) {
                const Slot& p = rec(pid);
                const uint32_t meta = p.w[W_META];
                if (!(i == 0 && sys)) emit(p.w[W_HASH_FIRST], p.w[W_HASH_COUNT], meta & FLAG_HASH_MULTI, out);   // "<p>/#", parent level included
                if (i == n) {
                    emit(p.w[W_OWN_FIRST], p.w[W_OWN_COUNT], meta & FLAG_OWN_MULTI, out);
                    continue;
                }
                if (p.w[W_PLUS] != NONE && !(i == 0 && sys)) next.push_back(p.w[W_PLUS]);
                const uint32_t c = level_child(pid, levels[i]);
                if (c != NONE) next.push_back(c);
            }
            frontier.swap(next);
        }
        std::sort(out->begin(), out->end());
    }
};

int main(int argc, char** argv) {
    if (argc < 2) return 2;
    const std::string dir = argv[1];
    auto keys = slurp<uint8_t>(dir + "/keys.bin"), vals = slurp<uint8_t>(dir + "/vals.bin");
    auto koff = slurp<int64_t>(dir + "/koff.bin"), voff = slurp<int64_t>(dir + "/voff.bin");
    auto tenants = slurp<uint8_t>(dir + "/tenants.bin"), topics = slurp<uint8_t>(dir + "/topics.bin");
    auto tenant_off = slurp<int64_t>(dir + "/tenant_off.bin"), topic_off = slurp<int64_t>(dir + "/topic_off.bin");
    auto topic_tenant = slurp<int32_t>(dir + "/topic_tenant.bin");
    auto deltas = slurp<uint8_t>(dir + "/deltas.bin", true);
    keys.push_back(0);
    vals.push_back(0);
    Staging st;
    std::string err;
    if (!st.load(keys.data(), koff.data(), vals.data(), voff.data(), (int64_t) koff.size() - 1, &err)) {
        fprintf(stderr, "load: %s\n", err.c_str());
        return 1;
    }
    for (size_t at = 0; at + 9 <= deltas.size();) {   // the staged delta of bfq_index_apply, merged like a commit does
        const uint8_t op = deltas[at];
        uint32_t kl, vl;
        memcpy(&kl, &deltas[at + 1], 4);
        const sv k((const char*) &deltas[at + 5], kl);
        memcpy(&vl, &deltas[at + 5 + kl], 4);
        const sv v((const char*) &deltas[at + 9 + kl], vl);
        if (op == 1) st.upsert(k, v);
        else st.erase(k);
        at += 9 + (size_t) kl + vl;
    }
    st.merge_all();
    std::vector<const KVBlob*> parts;
    for (auto& kvp : st.tenants()) parts.push_back(kvp.second.base.get());
    Image im;
    if (!build_flat_index_parts(parts, &im.f, &err)) {
        fprintf(stderr, "build: %s\n", err.c_str());
        return 1;
    }
    // the tag table is the head of the slot array; give find() a view of it (copy: test sizes are small)
    im.tag.n_blocks = im.f.n_blocks;
    im.tag.tags = im.f.tags;
    im.tag.slots.assign(im.f.slots.begin(), im.f.slots.begin() + (size_t) im.f.n_blocks * BLOCK_SLOTS);
    const int64_t n = (int64_t) topic_tenant.size();
    std::vector<int64_t> out_off{0}, out_ranks, one;
    for (int64_t i = 0; i < n; i++) {
        one.clear();
        const int32_t t = topic_tenant[(size_t) i];
        const std::string tid((const char*) tenants.data() + tenant_off[(size_t) t], (size_t) (tenant_off[(size_t) t + 1] - tenant_off[(size_t) t]));
        auto it = im.f.tenant_ordinal.find(tid);
        if (it != im.f.tenant_ordinal.end())
            im.match(ROOT_BASE + it->second, sv((const char*) topics.data() + topic_off[(size_t) i], (size_t) (topic_off[(size_t) i + 1] - topic_off[(size_t) i])), &one);
        out_ranks.insert(out_ranks.end(), one.begin(), one.end());
        out_off.push_back((int64_t) out_ranks.size());
    }
    if (argc > 2 && std::string(argv[2]) == "dump") {
        FILE* d = fopen((dir + "/dump.txt").c_str(), "w");
        fprintf(d, "n_blocks %u\n", im.f.n_blocks);
        for (int64_t i = 0; i < n; i++) {
            const int32_t t = topic_tenant[(size_t) i];
            const std::string tid((const char*) tenants.data() + tenant_off[(size_t) t], (size_t) (tenant_off[(size_t) t + 1] - tenant_off[(size_t) t]));
            auto it = im.f.tenant_ordinal.find(tid);
            uint32_t id = it == im.f.tenant_ordinal.end() ? NONE : ROOT_BASE + it->second;
            std::vector<sv> levels;
            for_each_level(sv((const char*) topics.data() + topic_off[(size_t) i], (size_t) (topic_off[(size_t) i + 1] - topic_off[(size_t) i])), '/',
                           [&](sv l) { levels.push_back(l); });
            for (size_t k = 0; k <= levels.size() && id != NONE; k++) {
                if (k > 0) id = levels[k - 1] == "+" ? im.rec(id).w[W_PLUS] : im.level_child(id, levels[k - 1]);
                if (id == NONE) {
                    fprintf(d, "node %lld %zu NONE none 0 0\n", (long long) i, k);
                    break;
                }
                const uint32_t meta = im.rec(id).w[W_META];
                const char* kind = !(meta & FLAG_HAS_EXACT) ? "none" : (meta & FLAG_BIG) ? "big" : meta_log2size(meta) ? "perfect" : "single";
                fprintf(d, "node %lld %zu %u %s %u %u\n", (long long) i, k, id, kind, meta_log2size(meta), meta >> 16);
            }
        }
        for (uint32_t b = 0; b < im.f.n_blocks; b++) {
            fprintf(d, "tags %u ", b);
            for (uint32_t j = 0; j < 16; j++) fprintf(d, "%02x", im.f.tags[(size_t) b * 16 + j]);
            fprintf(d, "\n");
        }
        fclose(d);
    }
    std::ofstream(dir + "/out_off.bin", std::ios::binary).write((const char*) out_off.data(), (std::streamsize) (out_off.size() * 8));
    std::ofstream(dir + "/out_ranks.bin", std::ios::binary).write((const char*) out_ranks.data(), (std::streamsize) (out_ranks.size() * 8));
    printf("walked %lld topics, %zu ranks, %lld nodes, %u slots, %u tag blocks\n", (long long) n, out_ranks.size(), (long long) im.f.n_nodes, im.f.n_slots, im.f.n_blocks);
    return 0;
}
