// delivery_wire.cu — a delivery nesting encoded as protobuf bytes: one DeliveryRequest per deliverer (bfq_delivery_encode).
//
// BatchDeliveryCall.execute (bifromq-deliverer/.../BatchDeliveryCall.java:91-108) builds, per deliverer,
//   DeliveryRequest { map<tenantId, DeliveryPackage> package = 3 }      entry {key = 1: tenantId, value = 2: DeliveryPackage}
//   DeliveryPackage { repeated DeliveryPack pack = 1 }
//   DeliveryPack    { TopicMessagePack messagePack = 2; repeated MatchInfo matchInfo = 3 }
//   TopicMessagePack{ string topic = 1; repeated PublisherPack message = 2 }
// (subbroker/type.proto, commontype/TopicMessage.proto). The MatchInfo fields come whole from the snapshot's table (TenantWire);
// the publisher packs are the caller's serialized bytes. Every length is a minimal varint, so a field's size depends on its
// content's: pass 1 sizes bottom-up (MatchInfo -> pack -> package / map entry -> request) with one scan per level, which also
// gives every write offset; pass 2 writes each map entry's header on a thread and each pack on a warp, most of it copies.
// The span of the last deliverer id (ordered_share_id) is left empty: its MatchInfos are counted, never encoded.
#include <cuda_runtime.h>

#include <cub/device/device_scan.cuh>

#include "fanout.h"

namespace bfq {

namespace {

constexpr int WR_THREADS = 256;
constexpr uint32_t NO_MEMBER = 0xFFFFFFFFu;
enum { CHK_BAD_PUB = 0, CHK_TOTAL = 1, CHK_ENCODED = 2 };

__device__ __forceinline__ uint32_t vlen(uint64_t v) {
    uint32_t n = 1;
    while (v >= 0x80) {
        v >>= 7;
        n++;
    }
    return n;
}
// a length-delimited field's bytes: tag, varint length, payload
__device__ __forceinline__ uint64_t field_bytes(uint64_t payload) { return 1 + vlen(payload) + payload; }
__device__ __forceinline__ uint8_t* put_varint(uint8_t* o, uint64_t v) {
    while (v >= 0x80) {
        *o++ = (uint8_t) (v | 0x80);
        v >>= 7;
    }
    *o++ = (uint8_t) v;
    return o;
}
__device__ __forceinline__ uint8_t* put_header(uint8_t* o, uint8_t tag, uint64_t len) {
    *o++ = tag;
    return put_varint(o, len);
}

unsigned wr_blocks(int64_t n) { return (unsigned) std::max<int64_t>(1, (n + WR_THREADS - 1) / WR_THREADS); }

// first item of the ordered-share deliverer's span, per level: packages, packs, pairs
__device__ __forceinline__ int64_t skipped_package(const WireParams& p) { return p.package_off[p.n_deliverers - 1]; }
__device__ __forceinline__ int64_t skipped_pack(const WireParams& p) { return p.pack_off[skipped_package(p)]; }
__device__ __forceinline__ int64_t skipped_pair(const WireParams& p) { return p.match_off[skipped_pack(p)]; }

// pub_off (0 at the start, never decreasing) and pubpack_off (the same over pub_off[n_topics] publishers), grid-stride
__global__ void __launch_bounds__(WR_THREADS) wire_check_kernel(const WireParams p) {
    const int64_t stride = (int64_t) gridDim.x * WR_THREADS, i0 = (int64_t) blockIdx.x * WR_THREADS + threadIdx.x;
    bool bad = false;
    for (int64_t t = i0; t <= p.n_topics; t += stride) bad |= t == 0 ? p.pub_off[0] != 0 : p.pub_off[t] < p.pub_off[t - 1];
    const int64_t n_pubs = p.pub_off[p.n_topics];
    if (n_pubs >= 0)
        for (int64_t x = i0; x <= n_pubs; x += stride) bad |= x == 0 ? p.pubpack_off[0] != 0 : p.pubpack_off[x] < p.pubpack_off[x - 1];
    if (bad) atomicAdd(&p.check[CHK_BAD_PUB], 1ull);
}

// MatchInfo field bytes of every nested pair; none under the ordered-share id
__global__ void __launch_bounds__(WR_THREADS) wire_pair_kernel(const WireParams p) {
    const int64_t j = (int64_t) blockIdx.x * WR_THREADS + threadIdx.x;
    if (j >= p.n_pairs) return;
    uint64_t b = 0;
    if (j < skipped_pair(p)) {
        const uint32_t m = p.match_member[j];
        const uint32_t e = p.mi_first[p.match_rank[j]] + (m == NO_MEMBER ? 0u : m);
        b = p.mi_off[e + 1] - p.mi_off[e];
    }
    p.pair_pos[j] = b;
}

// pack k's publisher packs: [*a, *b) of pack_pub (a sub-pack) or of the topic's own publishers (a whole pack, *sub = false)
__device__ __forceinline__ void pack_pubs(const WireParams& p, int64_t k, int64_t* a, int64_t* b, bool* sub) {
    *sub = false;
    if (p.pack_pub_off) {
        *a = p.pack_pub_off[k];
        *b = p.pack_pub_off[k + 1];
        *sub = *b > *a;
    }
    if (!*sub) {
        const uint32_t t = p.pack_topic[k];
        *a = p.pub_off[t];
        *b = p.pub_off[t + 1];
    }
}
__device__ __forceinline__ int64_t pub_at(const WireParams& p, bool sub, int64_t x) { return sub ? (int64_t) p.pack_pub[x] : x; }

// TopicMessagePack bytes of pack k (topic field + every publisher pack field), or ~0 for a publisher outside pub_off's range
__device__ __forceinline__ uint64_t message_pack_bytes(const WireParams& p, int64_t k) {
    const uint32_t t = p.pack_topic[k];
    const uint64_t tl = (uint64_t) (p.topic_off[t + 1] - p.topic_off[t]);
    uint64_t s = tl ? field_bytes(tl) : 0;
    int64_t a, b;
    bool sub;
    pack_pubs(p, k, &a, &b, &sub);
    const int64_t n_pubs = p.pub_off[p.n_topics];
    for (int64_t x = a; x < b; x++) {
        const int64_t q = pub_at(p, sub, x);
        if (q < 0 || q >= n_pubs) return ~0ull;
        s += field_bytes((uint64_t) (p.pubpack_off[q + 1] - p.pubpack_off[q]));
    }
    return s;
}

// DeliveryPack field bytes of every pack (pair_pos scanned); none under the ordered-share id
__global__ void __launch_bounds__(WR_THREADS) wire_pack_kernel(const WireParams p) {
    const int64_t k = (int64_t) blockIdx.x * WR_THREADS + threadIdx.x;
    if (k >= p.n_packs) return;
    uint64_t b = 0;
    if (k < skipped_pack(p)) {
        const uint64_t mp = message_pack_bytes(p, k);
        if (mp == ~0ull) {
            atomicAdd(&p.check[CHK_BAD_PUB], 1ull);
        } else {
            const uint64_t infos = p.pair_pos[p.match_off[k + 1]] - p.pair_pos[p.match_off[k]];
            b = field_bytes(field_bytes(mp) + infos);
        }
    }
    p.pack_pos[k] = b;
}

__device__ __forceinline__ uint64_t tenant_bytes(const WireParams& p, uint32_t tn) {
    return (uint64_t) (p.tenant_off[tn + 1] - p.tenant_off[tn]);
}

// map entry field bytes of every package (pack_pos scanned); none under the ordered-share id
__global__ void __launch_bounds__(WR_THREADS) wire_package_kernel(const WireParams p) {
    const int64_t g = (int64_t) blockIdx.x * WR_THREADS + threadIdx.x;
    if (g >= p.n_packages) return;
    uint64_t b = 0;
    if (g < skipped_package(p)) {
        const uint64_t body = p.pack_pos[p.pack_off[g + 1]] - p.pack_pos[p.pack_off[g]];
        b = field_bytes(field_bytes(tenant_bytes(p, p.package_tenant[g])) + field_bytes(body));
    }
    p.package_pos[g] = b;
}

// package_pos scanned: every deliverer's request offset, the total and the MatchInfos encoded
__global__ void __launch_bounds__(WR_THREADS) wire_offsets_kernel(const WireParams p) {
    const int64_t d = (int64_t) blockIdx.x * WR_THREADS + threadIdx.x;
    if (d > (int64_t) p.n_deliverers) return;
    p.req_off[d] = (long long) p.package_pos[p.package_off[d]];
    if (d == 0) {
        p.check[CHK_TOTAL] = p.package_pos[p.n_packages];
        p.check[CHK_ENCODED] = (unsigned long long) skipped_pair(p);
    }
}

// ---- pass 2
// map entry header of package g: {entry tag, len, key field (tenantId), value tag, len}; its packs follow
__global__ void __launch_bounds__(WR_THREADS) wire_entry_kernel(const WireParams p) {
    const int64_t g = (int64_t) blockIdx.x * WR_THREADS + threadIdx.x;
    if (g >= p.n_packages || g >= skipped_package(p)) return;
    const uint32_t tn = p.package_tenant[g];
    const uint64_t tl = tenant_bytes(p, tn);
    const uint64_t body = p.pack_pos[p.pack_off[g + 1]] - p.pack_pos[p.pack_off[g]];
    uint8_t* o = p.out + p.package_pos[g];
    o = put_header(o, 0x1A, field_bytes(tl) + field_bytes(body));
    o = put_header(o, 0x0A, tl);
    const uint8_t* src = p.tenants + p.tenant_off[tn];
    for (uint64_t i = 0; i < tl; i++) o[i] = src[i];
    put_header(o + tl, 0x12, body);
}

// dst[0 .. n) = src[0 .. n) by the 32 lanes of a warp: 16-byte stores to dst's aligned middle, each built from 4-byte aligned
// loads of src funnel-shifted into place (a load never leaves the 4-byte words that hold src's bytes); bytes at the ends
__device__ __forceinline__ void warp_copy(uint8_t* dst, const uint8_t* src, uint64_t n, uint32_t lane) {
    const uint64_t head = min(n, (uint64_t) ((16u - ((uintptr_t) dst & 15u)) & 15u));
    for (uint64_t i = lane; i < head; i += 32) dst[i] = src[i];
    dst += head;
    src += head;
    n -= head;
    const uint64_t chunks = n >> 4;
    const uint32_t sh = (uint32_t) ((uintptr_t) src & 3u) * 8u;
    const uint32_t* sw = reinterpret_cast<const uint32_t*>((uintptr_t) src & ~(uintptr_t) 3);
    for (uint64_t c = lane; c < chunks; c += 32) {
        const uint32_t* s = sw + 4 * c;
        const uint32_t w0 = __ldg(s), w1 = __ldg(s + 1), w2 = __ldg(s + 2), w3 = __ldg(s + 3);
        const uint32_t w4 = sh ? __ldg(s + 4) : 0u;
        uint4 v;
        v.x = __funnelshift_r(w0, w1, sh);
        v.y = __funnelshift_r(w1, w2, sh);
        v.z = __funnelshift_r(w2, w3, sh);
        v.w = __funnelshift_r(w3, w4, sh);
        reinterpret_cast<uint4*>(dst)[c] = v;
    }
    for (uint64_t i = (chunks << 4) + lane; i < n; i += 32) dst[i] = src[i];
}

// one warp per pack: the pack's headers, topic, publisher packs and MatchInfos at its place in its package's value
__global__ void __launch_bounds__(WR_THREADS) wire_pack_write_kernel(const WireParams p) {
    const int64_t k = ((int64_t) blockIdx.x * WR_THREADS + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if (k >= p.n_packs || k >= skipped_pack(p)) return;
    // the package holding pack k: last g with pack_off[g] <= k
    int64_t lo = 0, hi = p.n_packages;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (p.pack_off[mid] <= k) lo = mid;
        else hi = mid;
    }
    const int64_t g = lo;
    const uint64_t tl = tenant_bytes(p, p.package_tenant[g]);
    const uint64_t body = p.pack_pos[p.pack_off[g + 1]] - p.pack_pos[p.pack_off[g]];
    // the entry header before the package's packs, as wire_entry_kernel writes it
    const uint64_t entry_hdr = 1 + vlen(field_bytes(tl) + field_bytes(body)) + field_bytes(tl) + 1 + vlen(body);
    uint8_t* o = p.out + p.package_pos[g] + entry_hdr + (p.pack_pos[k] - p.pack_pos[p.pack_off[g]]);
    const uint32_t t = p.pack_topic[k];
    const uint64_t topic_len = (uint64_t) (p.topic_off[t + 1] - p.topic_off[t]);
    const uint64_t mp = message_pack_bytes(p, k);
    const int64_t m0 = p.match_off[k], m1 = p.match_off[k + 1];
    const uint64_t infos = p.pair_pos[m1] - p.pair_pos[m0];
    if (lane == 0) {
        uint8_t* h = put_header(o, 0x0A, field_bytes(mp) + infos);
        h = put_header(h, 0x12, mp);
        if (topic_len) put_header(h, 0x0A, topic_len);
    }
    o += 1 + vlen(field_bytes(mp) + infos) + 1 + vlen(mp);
    if (topic_len) {
        o += 1 + vlen(topic_len);
        warp_copy(o, p.topics + p.topic_off[t], topic_len, lane);
        o += topic_len;
    }
    int64_t a, b;
    bool sub;
    pack_pubs(p, k, &a, &b, &sub);
    for (int64_t x = a; x < b; x++) {
        const int64_t q = pub_at(p, sub, x);
        const uint64_t len = (uint64_t) (p.pubpack_off[q + 1] - p.pubpack_off[q]);
        if (lane == 0) put_header(o, 0x12, len);
        o += 1 + vlen(len);
        warp_copy(o, p.pubpack + p.pubpack_off[q], len, lane);
        o += len;
    }
    for (int64_t j = m0; j < m1; j++) {
        const uint32_t m = p.match_member[j];
        const uint32_t e = p.mi_first[p.match_rank[j]] + (m == NO_MEMBER ? 0u : m);
        const uint64_t len = p.mi_off[e + 1] - p.mi_off[e];
        warp_copy(o, p.mi_bytes + p.mi_off[e], len, lane);
        o += len;
    }
}

}  // namespace

cudaError_t launch_wire_size(const WireParams& p, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    const int64_t n[3] = {p.n_pairs, p.n_packs, p.n_packages};
    unsigned long long* pos[3] = {p.pair_pos, p.pack_pos, p.package_pos};
    if (!d_tmp) {
        size_t most = 0;
        for (int i = 0; i < 3; i++) {
            size_t b = 0;
            const cudaError_t err = cub::DeviceScan::ExclusiveSum(nullptr, b, pos[i], n[i] + 1, stream);
            if (err != cudaSuccess) return err;
            most = std::max(most, b);
        }
        *tmp_bytes = most;
        return cudaSuccess;
    }
    cudaError_t err = cudaMemsetAsync(p.check, 0, 4 * sizeof(unsigned long long), stream);
    if (err != cudaSuccess) return err;
    // the scans are exclusive over n + 1 entries: the last one is the total
    if ((err = cudaMemsetAsync(p.pair_pos + p.n_pairs, 0, sizeof(unsigned long long), stream)) != cudaSuccess) return err;
    if ((err = cudaMemsetAsync(p.pack_pos + p.n_packs, 0, sizeof(unsigned long long), stream)) != cudaSuccess) return err;
    if ((err = cudaMemsetAsync(p.package_pos + p.n_packages, 0, sizeof(unsigned long long), stream)) != cudaSuccess) return err;
    wire_check_kernel<<<264, WR_THREADS, 0, stream>>>(p);
    size_t bytes;
    wire_pair_kernel<<<wr_blocks(p.n_pairs), WR_THREADS, 0, stream>>>(p);
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, p.pair_pos, p.n_pairs + 1, stream)) != cudaSuccess) return err;
    wire_pack_kernel<<<wr_blocks(p.n_packs), WR_THREADS, 0, stream>>>(p);
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, p.pack_pos, p.n_packs + 1, stream)) != cudaSuccess) return err;
    wire_package_kernel<<<wr_blocks(p.n_packages), WR_THREADS, 0, stream>>>(p);
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, p.package_pos, p.n_packages + 1, stream)) != cudaSuccess) return err;
    wire_offsets_kernel<<<wr_blocks((int64_t) p.n_deliverers + 1), WR_THREADS, 0, stream>>>(p);
    return cudaGetLastError();
}

cudaError_t launch_wire_write(const WireParams& p, cudaStream_t stream) {
    wire_entry_kernel<<<wr_blocks(p.n_packages), WR_THREADS, 0, stream>>>(p);
    wire_pack_write_kernel<<<wr_blocks(p.n_packs * 32), WR_THREADS, 0, stream>>>(p);
    return cudaGetLastError();
}

}  // namespace bfq
