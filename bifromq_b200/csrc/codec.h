// codec.h — host-side route key codec and topic tokeniser/validators of the product.
//
// Native restatement of the pieces of apache/bifromq the index is fed with:
//   route key layout   bifromq-dist/bifromq-dist-worker-schema/.../schema/KVSchemaUtil.java:91-130,
//                      KVSchemaConstants.java:24-34, cache/RouteDetailCache.java:53-109 (decode),
//                      cache/ReceiverCache.java:32-36 (subBrokerId)
//   tokeniser          bifromq-util/.../util/TopicUtil.java:206-225 (parse), :42-163 (validators)
// Works on byte spans; no Java object graph is rebuilt — the matcher only needs (tenant, filter levels,
// route kind) per key.
#pragma once
#include <cstdint>
#include <string>
#include <string_view>
#include <vector>

namespace bfq {

using sv = std::string_view;

constexpr uint8_t FLAG_NORMAL = 0x01, FLAG_UNORDERED = 0x02, FLAG_ORDERED = 0x03;
enum RouteKind : uint8_t { KIND_NORMAL = 0, KIND_PERSISTENT = 1, KIND_GROUP = 2 };

struct DecodedKey {
    sv tenant;
    sv escaped_filter;   // filter levels joined by NUL
    sv receiver;         // receiverUrl (normal) or group name (shared)
    uint8_t flag = 0;
    uint8_t bucket = 0;
    RouteKind kind = KIND_NORMAL;
};
// returns false if the bytes cannot be a route key
bool decode_route_key(sv key, DecodedKey* out);

// iterate the NUL-separated levels of an escaped filter (or '/'-separated levels of a topic)
template <typename F>
inline void for_each_level(sv s, char sep, F&& f) {
    size_t start = 0;
    for (size_t i = 0; i <= s.size(); i++) {
        if (i == s.size() || s[i] == sep) {
            f(s.substr(start, i - start));
            start = i + 1;
        }
    }
}

int32_t java_string_hash(sv utf8);          // java.lang.String.hashCode over UTF-16 code units
uint8_t receiver_bucket(sv receiver);       // KVSchemaUtil.bucket :127-130
std::string make_receiver_url(int32_t sub_broker_id, sv receiver_id, sv deliverer_key);   // :56-58
std::string make_tenant_begin_key(sv tenant);                                              // :91-94
// mqtt_topic_filter may start with $share/<group>/ or $oshare/<group>/   (TopicUtil.from :252-272)
std::string make_route_key(sv tenant, sv mqtt_topic_filter, sv receiver_url);              // :108-125
std::string prefix_upper_bound(sv key, bool* open_end);

// thread-local error text behind bfq_last_error() (defined in errors.cc)
int32_t set_error(int32_t code, const std::string& msg);

// ---- retain store key layout (bifromq-retain/bifromq-retain-store-schema/.../schema/KVSchemaUtil.java:44-73, LevelHash.java:31-49):
//   key = <0x00> <u16 BE len> tenantId <u16 BE number of topic levels> <one FNV-1a byte per level> escape(topic)
// with escape = '/' -> NUL (U/TopicUtil.java:189-192). The topic is recoverable from the key, so the index is fed from a plain
// key scan (RetainStoreCoProc.load, RS/RetainStoreCoProc.java:279-296, parses every VALUE for it).
uint8_t level_hash_byte(sv level_utf8);                          // LevelHash.hashToByte :41-48 (FNV-1a over UTF-16 code units, low byte)
std::string make_retain_key(sv tenant, sv topic);                // retainMessageKey :44-50
// retainKeyPrefix(tenant, levels, filterPrefix(filter)) :52-72 with levels = the filter's level count (one less under a final '#')
std::string make_retain_key_prefix(sv tenant, sv topic_filter);
bool decode_retain_key(sv key, sv* tenant, std::string* topic);  // false if the bytes cannot be a retain key

bool is_valid_topic(sv topic, int max_level_length, int max_level, int max_length);
bool is_valid_topic_filter(sv tf, int max_level_length, int max_level, int max_length);

}  // namespace bfq
