// oracle/oracle.h — CPU ORACLE (TEST INFRASTRUCTURE ONLY).
//
// A plain C++17 restatement of the apache/bifromq publish-topic -> routes path and its
// inverse (retain / TopicIndex) path. It exists to CHECK the CUDA product in
// bifromq_b200/csrc; nothing in the product may include, link or call it. Only tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs use it.
//
// Parity pinning: the reference is Java 17 and cannot run in this image (no JDK), so the
// oracle is pinned against every golden vector the reference's own tests carry for this
// path (see tests/test_oracle_golden.py; SURVEY.md §8c lists them).
//
// Paths below are relative to the reference repository's root. Abbreviations:
//   U/   = bifromq-util/src/main/java/org/apache/bifromq/util/
//   DCP/ = bifromq-dist/bifromq-dist-coproc-proto/src/main/java/org/apache/bifromq/dist/trie/
//   DW/  = bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/
//   DWS/ = bifromq-dist/bifromq-dist-worker-schema/src/main/java/org/apache/bifromq/dist/worker/schema/
//   RS/  = bifromq-retain/bifromq-retain-store/src/main/java/org/apache/bifromq/retain/store/
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

namespace orc {

using Levels = std::vector<std::string>;

// ---------------------------------------------------------------- JDK behaviours
// UTF-8 -> UTF-16 code units (Java strings are UTF-16; lengths / hashCode / compareTo
// are all defined on code units).
std::u16string to_utf16(const std::string& utf8);
// java.lang.String.hashCode(): s[0]*31^(n-1) + ... over UTF-16 units, int32 wrap.
int32_t java_hash(const std::string& utf8);
// java.lang.String.compareTo(): lexicographic over UTF-16 units.
int java_compare(const std::string& a, const std::string& b);
struct JavaLess {
    bool operator()(const std::string& a, const std::string& b) const { return java_compare(a, b) < 0; }
};
struct JavaLevelsLess {  // level-wise compareTo, shorter prefix first
    bool operator()(const Levels& a, const Levels& b) const;
};

// ---------------------------------------------------------------- U/TopicUtil.java
Levels parse(const std::string& topic, bool escaped);                                   // :206-225
bool is_valid_topic(const std::string& topic, int maxLevelLength, int maxLevel, int maxLength);        // :42-72
bool is_valid_topic_filter(const std::string& tf, int maxLevelLength, int maxLevel, int maxLength);    // :74-163
bool is_wildcard_topic_filter(const std::string& tf);                                   // :165-171
bool is_multi_wildcard_topic_filter(const std::string& tf);
bool is_shared_subscription(const std::string& tf);                                     // :173-187
bool is_unordered_shared(const std::string& tf);
bool is_ordered_shared(const std::string& tf);
std::string escape(const std::string& tf);                                              // :189-192
std::string unescape(const std::string& tf);                                            // :194-196
std::string join(const Levels& levels, char sep);                                       // fastJoin :227-237

// commontype.RouteMatcher (bifromq-common-type/src/main/proto/commontype/RouteMatcher.proto:27-37)
struct RouteMatcher {
    enum Type { Normal = 0, UnorderedShare = 1, OrderedShare = 2 } type = Normal;
    Levels filterLevels;
    std::string group;
    std::string mqttTopicFilter;
};
RouteMatcher route_matcher_from(const std::string& topicFilter);                        // TopicUtil.from :252-272

// ---------------------------------------------------------------- DWS/KVSchemaUtil.java
std::string to_receiver_url(int subBrokerId, const std::string& receiverId, const std::string& delivererKey);  // :56-58
std::string tenant_begin_key(const std::string& tenantId);                              // :91-94
// retain store schema (bifromq-retain/bifromq-retain-store-schema/src/main/java/org/apache/bifromq/retain/store/schema/):
uint8_t level_hash_byte(const std::string& level);                                      // LevelHash.java:41-48
std::string level_hash(const std::vector<std::string>& levels);                         // LevelHash.java:33-39
std::string retain_message_key(const std::string& tenantId, const std::string& topic);  // KVSchemaUtil.java:44-50
std::vector<std::string> retain_filter_prefix(const std::vector<std::string>& filterLevels);   // KVSchemaUtil.java:52-62
std::string retain_key_prefix(const std::string& tenantId, int levels, const std::vector<std::string>& filterPrefix);   // :64-68
std::string tenant_route_start_key(const std::string& tenantId, const Levels& filterLevels);  // :96-102
std::string to_normal_route_key(const std::string& tenantId, const RouteMatcher& m, const std::string& receiverUrl);  // :108-113
std::string to_group_route_key(const std::string& tenantId, const RouteMatcher& m);     // :115-120
uint8_t bucket(const std::string& receiver);                                            // :127-130
std::string upper_bound(const std::string& key, bool* open_end);                        // BoundaryUtil.upperBound :299-307
std::string u64_be(uint64_t v);                                                         // BSUtil.toByteString(long)
uint64_t u64_from_be(const std::string& b);                                             // BSUtil.toLong :29-33

struct Receiver {  // DWS/cache/ReceiverCache.java:32-36
    int subBrokerId = 0;
    std::string receiverId, delivererKey;
};
Receiver parse_receiver(const std::string& receiverUrl);

struct RouteDetail {  // DWS/cache/RouteDetailCache.java:53-109
    std::string tenantId;
    RouteMatcher matcher;
    std::string receiverUrl;  // normal routes only
};
RouteDetail decode_route_key(const std::string& key);
std::string parse_tenant_id(const std::string& key);                                    // KVSchemaUtil.parseTenantId :60-64
uint8_t parse_flag(const std::string& key);                                             // KVSchemaUtil.parseFlag :66-71

// distservice.RouteGroup { map<string,uint64> members = 1; }  (RouteGroup.proto:27-29)
std::string encode_route_group(const std::vector<std::pair<std::string, uint64_t>>& members);
std::map<std::string, uint64_t> decode_route_group(const std::string& bytes);

// Matching equality (DWS/cache/NormalMatching.java:30-41, GroupMatching.java:32-39):
// Normal = (tenantId, mqttTopicFilter, receiverUrl, incarnation); Group = (tenantId, mqttTopicFilter, members).
struct Matching {
    enum Type { Normal, Group } type = Normal;
    std::string tenantId, mqttTopicFilter;
    Levels filterLevels;
    std::string receiverUrl;
    uint64_t incarnation = 0;
    int subBrokerId = 0;
    std::map<std::string, uint64_t> members;
};
Matching build_match_route(const std::string& key, const std::string& value);           // KVSchemaUtil.buildMatchRoute :73-79

// ---------------------------------------------------------------- DCP/TopicTrieNode.java
struct TopicTrieNode {
    std::string levelName;
    bool wildcardMatchable = false;
    std::map<std::string, std::unique_ptr<TopicTrieNode>, JavaLess> children;  // TreeMap<String,...>
    std::vector<int> values;  // ids of the topics ending here
    Levels topic;
    bool is_user_topic() const { return !values.empty(); }
};
struct TopicTrie {
    explicit TopicTrie(bool isGlobal);
    void add_topic(const Levels& topicLevels, int value);                               // :135-161
    std::unique_ptr<TopicTrieNode> root;
    bool isGlobal;
};

// ---------------------------------------------------------------- DCP/TopicFilterIterator.java
// Cursor over the expansion set (every filter matching >= 1 topic of the trie), in
// level-wise String.compareTo order, built from virtual N / S(+) / M(#) filter nodes
// (DCP/NTopicFilterTrieNode.java:118-153, STopicFilterTrieNode.java:117-148,
//  MTopicFilterTrieNode.java:105-135).
class TopicFilterIterator {
public:
    explicit TopicFilterIterator(const TopicTrie& trie);
    ~TopicFilterIterator();
    void seek(const Levels& filterLevels);                                              // :62-122
    void next();                                                                        // :260-278
    bool is_valid() const;                                                              // :224-226
    Levels key() const;                                                                 // :280-288
    // value(): topics (by id) backing the current filter                               // :290-300
    std::vector<int> value() const;
    struct FNode;
private:
    const TopicTrie& trie_;
    std::vector<FNode*> stack_;
    void clear();
    void pop();
};

// ---------------------------------------------------------------- DW/cache/TenantRouteMatcher.java + MatchedRoutes.java
struct ThrottleEvent {  // PersistentFanoutThrottled / GroupFanoutThrottled (MatchedRoutes.java:95-100,128-133)
    enum Kind { Persistent = 1, Group = 2 } kind;
    int topicIdx;
    int64_t routeRank;  // rank (KV order index) of the route that was dropped
    int maxCount;
};
struct MatchStats {
    uint64_t seeks = 0, nexts = 0;          // KV iterator ops (TenantRouteMatcherTest.java:232-235)
    uint64_t backwardSeeks = 0;             // oracle-only guard, see matcher.cc
    uint64_t V = 0, P = 0, R = 0, ranges = 0;  // SURVEY.md §8(d) algorithmic-byte counters (trie walk only)
};
struct MatchResult {
    std::vector<std::vector<int64_t>> routes;  // per topic: KV ranks of surviving routes (sorted ascending)
    std::vector<int> persistentFanout, groupFanout;
    std::vector<ThrottleEvent> events;
    MatchStats stats;
};
// Sorted KV (RocksDB order == unsigned byte order; tests use a TreeMap with
// ByteString.unsignedLexicographicalComparator(), TenantRouteMatcherTest.java:73-75).
class SortedKV {
public:
    void put(const std::string& k, const std::string& v) { frozen_ = false; kv_[k] = v; }
    void erase(const std::string& k) { frozen_ = false; kv_.erase(k); }
    size_t size() const { return kv_.size(); }
    void freeze();                                   // materialise the rank-ordered view
    int64_t lower_bound(const std::string& k) const; // == IKVIterator.seek: first rank with key >= k
    const std::string& key(int64_t rank) const { return order_[rank]->first; }
    const std::string& value(int64_t rank) const { return order_[rank]->second; }
    int64_t n() const { return (int64_t) order_.size(); }
private:
    std::map<std::string, std::string> kv_;  // std::string compares as unsigned bytes (memcmp)
    std::vector<const std::pair<const std::string, std::string>*> order_;
    bool frozen_ = false;
};

// (1) literal restatement of TenantRouteMatcher.matchAll (DW/cache/TenantRouteMatcher.java:68-161)
MatchResult match_all_reference(const SortedKV& kv, const std::string& tenantId, const std::vector<std::string>& topics,
                                int maxPersistentFanout, int maxGroupFanout);
// (2) brute force: the §8a predicate applied to every (topic, route) of the tenant, caps in KV order
MatchResult match_all_brute(const SortedKV& kv, const std::string& tenantId, const std::vector<std::string>& topics,
                            int maxPersistentFanout, int maxGroupFanout);
// predicate, restating DCPT TopicMatcher (test helper of the reference) on parsed levels
bool topic_matches_filter(const Levels& topicLevels, const Levels& filterLevels);
// (3) straightforward filter-trie walk (strongest honest CPU competitor; also counts V/P/R)
class FilterTrie;
std::shared_ptr<FilterTrie> build_filter_trie(const SortedKV& kv);
MatchResult match_all_trie(const FilterTrie& trie, const SortedKV& kv, const std::string& tenantId,
                           const std::vector<std::string>& topics, int maxPersistentFanout, int maxGroupFanout);

// ---------------------------------------------------------------- inverse match
// U/index/TopicLevelTrie.java:190-249 driven by the selectors of DW/TopicIndex.java:40-117
// (levelShift = 0) and RS/index/RetainTopicIndex.java:36-124 (tenantId is level 0, levelShift = 1).
class TopicLevelIndex {
public:
    TopicLevelIndex();
    ~TopicLevelIndex();
    void add(const Levels& topicLevels, int64_t value);
    void remove(const Levels& topicLevels, int64_t value);
    // TopicIndex.match(filterLevels): sysLevel = 0 ; RetainTopicIndex.match(tenant, filter): sysLevel = 1
    std::vector<int64_t> match(const Levels& filterLevels, int sysLevel, uint64_t* visited = nullptr) const;
    std::vector<int64_t> get(const Levels& topicLevels) const;                           // TopicIndex.get (TopicGetter)
    std::vector<int64_t> find_all() const;                                              // RetainTopicIndex.findAll
    struct Node;
private:
    std::unique_ptr<Node> root_;
};

}  // namespace orc
