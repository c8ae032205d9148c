// fanout.cu — fan-out expansion on the GPU (SURVEY.md §8f rank 3): the step right behind the match.
//
// The reference walks every matched route of a message on the CPU: DeliverExecutorGroup.submit
// (bifromq-dist/bifromq-dist-worker/src/main/java/org/apache/bifromq/dist/worker/DeliverExecutorGroup.java:112-231) iterates the
// route set, resolves a shared subscription to ONE member (send(GroupMatching) :242-278: a uniformly random member for
// $share, a rendezvous hash of the publisher for $oshare), and DeliverExecutor.send (DeliverExecutor.java:89-93) turns each
// route into a DeliveryCall keyed by (subBrokerId, delivererKey), which the deliverer batches into one DeliveryPack list per
// deliverer. With the matched route ranks already on the device that is a group-by:
//   input   the device CSR of a completed match (surviving ranks per topic, caps applied: bfq_expand_device)
//   output  every (topic, route) pair of the batch grouped by DELIVERER id: pack_offsets[D + 1], pack_topic[], pack_rank[]
//           (+ pack_member[] for shared subscriptions: the index of the member the pair was resolved to)
// A deliverer id is a dense index over the distinct (subBrokerId, delivererKey) pairs the handle has interned since it was
// created, interned on the host when a snapshot is first used for fan-out (bfq_fanout_deliverer gives the pair back); ids are
// never freed, so a handle that has seen many deliverers carries them all. Unordered shared subscriptions pick member
// hash(topic position, route rank) mod n — the reference picks uniformly at random (ThreadLocalRandom), so any member is a valid
// outcome and the pick here is reproducible; ORDERED shared subscriptions need the publisher of each message
// (RendezvousHash over ClientInfo.hashCode(), :253-270) which a topic batch does not carry: their pairs are grouped under the
// reserved deliverer id BFQ_FANOUT_ORDERED_SHARE with every member left to the host.
//
// Kernels: a two-pass radix partition on the deliverer id, in one of two forms.
//   tile pass    pass 1 counts per (CTA tile, deliverer) in shared memory; a scan over the [deliverer][tile] count matrix gives
//                every tile its write cursor per deliverer; pass 2 re-reads the tile and scatters. Used while the matrix has
//                no more cells than the batch has pairs (so at most FO_TILE ids: a 16 KB shared histogram).
//   global pass  pass 1 counts per deliverer in global memory (warp-aggregated atomics), an exclusive scan over the D + 1
//                counts gives every deliverer its segment, pass 2 re-reads the pairs and claims slots with the same atomics.
//                Scratch is 2 x (D + 1) words whatever the batch; used for many deliverers or a small batch.
// Per pair: one 8-byte rank read (streaming), one 4-byte deliverer-id read (the table is 4 bytes per route: L2 resident at
// 10M filters), 12 bytes written. HBM-streaming bound.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "../../include/bfq_gpumatch.h"
#include "codec.h"
#include "fanout.h"

namespace bfq {

namespace {

constexpr int FO_THREADS = 256;
constexpr int FO_TILE = 4096;          // pairs per tile

__device__ __forceinline__ uint32_t fo_mix(uint32_t a, uint32_t b) {
    uint32_t h = a * 0x9E3779B1u ^ (b + 0x7F4A7C15u + (a << 6) + (a >> 2));
    h ^= h >> 15;
    h *= 0x85EBCA6Bu;
    h ^= h >> 13;
    return h;
}

// deliverer of the pair (topic position t, rank r); *member = member index of a shared subscription or 0xFFFFFFFF
__device__ __forceinline__ uint32_t fo_deliverer(const FanoutParams& p, uint32_t t, int64_t r, uint32_t* member) {
    const uint32_t d = p.rdeliv[r];
    *member = 0xFFFFFFFFu;
    if (!(d & FO_GROUP_BIT)) return d;
    const uint32_t g = d & ~FO_GROUP_BIT;                 // index into the group table
    const uint32_t b = p.gmem_off[g], n = p.gmem_off[g + 1] - b;
    if (n == 0) return p.n_deliverers - 1;                // empty group: nothing to deliver (parked under the ordered-share id)
    if (p.gordered[g]) return p.n_deliverers - 1;         // BFQ_FANOUT_ORDERED_SHARE: the host picks per publisher
    const uint32_t m = fo_mix(t, (uint32_t) r) % n;
    *member = m;
    return p.gmem_deliv[b + m];
}

// topic of pair position j: binary search in offsets (monotone), amortised by doing it once per thread then walking
__device__ __forceinline__ uint32_t fo_topic_of(const int64_t* offsets, int64_t n_topics, int64_t j) {
    int64_t lo = 0, hi = n_topics;   // offsets[lo] <= j < offsets[hi]
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (offsets[mid] <= j) lo = mid;
        else hi = mid;
    }
    return (uint32_t) lo;
}

// global pass: the lanes of a warp that hold the same deliverer take consecutive slots of ctr[d] with one atomic (a batch whose
// pairs all go to one deliverer costs one atomic per warp step, not one per pair); returns this lane's slot
__device__ __forceinline__ uint32_t fo_claim(uint32_t* ctr, uint32_t d) {
    const uint32_t peers = __match_any_sync(__activemask(), d);
    const uint32_t lane = threadIdx.x & 31u;
    const int leader = __ffs(peers) - 1;
    uint32_t base = 0;
    if ((int) lane == leader) base = atomicAdd(&ctr[d], (uint32_t) __popc(peers));
    base = __shfl_sync(peers, base, leader);
    return base + (uint32_t) __popc(peers & ((1u << lane) - 1u));
}

template <bool GLOBAL>
__global__ void __launch_bounds__(FO_THREADS) fanout_count_kernel(const FanoutParams p) {
    extern __shared__ uint32_t hist[];
    if constexpr (!GLOBAL) {
        for (uint32_t i = threadIdx.x; i < p.n_deliverers; i += FO_THREADS) hist[i] = 0;
        __syncthreads();
    }
    // a thread owns FO_TILE / FO_THREADS consecutive pairs (one 128-byte line of ranks): one binary search for the first one's
    // topic, then the topic index only walks forward
    constexpr int PER = FO_TILE / FO_THREADS;
    const int64_t j0 = (int64_t) blockIdx.x * FO_TILE + (int64_t) threadIdx.x * PER;
    if (j0 < p.n_pairs) {
        uint32_t t = fo_topic_of(p.offsets, p.n_topics, j0);
        for (int q = 0; q < PER && j0 + q < p.n_pairs; q++) {
            const int64_t j = j0 + q;
            while (p.offsets[t + 1] <= j) t++;
            uint32_t member;
            const uint32_t d = fo_deliverer(p, t, p.ranks[j], &member);
            if constexpr (GLOBAL) fo_claim(p.counts, d);
            else atomicAdd(&hist[d], 1u);
        }
    }
    if constexpr (!GLOBAL) {
        __syncthreads();
        // count matrix in [deliverer][tile] order: its exclusive scan is, for every deliverer, the cursor of every tile
        for (uint32_t i = threadIdx.x; i < p.n_deliverers; i += FO_THREADS) p.counts[(uint64_t) i * gridDim.x + blockIdx.x] = hist[i];
    }
}

template <bool GLOBAL>
__global__ void __launch_bounds__(FO_THREADS) fanout_scatter_kernel(const FanoutParams p) {
    extern __shared__ uint32_t cur[];
    if constexpr (!GLOBAL) {
        for (uint32_t i = threadIdx.x; i < p.n_deliverers; i += FO_THREADS) cur[i] = 0;
        __syncthreads();
    }
    constexpr int PER = FO_TILE / FO_THREADS;
    const int64_t j0 = (int64_t) blockIdx.x * FO_TILE + (int64_t) threadIdx.x * PER;
    if (j0 < p.n_pairs) {
        uint32_t t = fo_topic_of(p.offsets, p.n_topics, j0);
        for (int q = 0; q < PER && j0 + q < p.n_pairs; q++) {
            const int64_t j = j0 + q;
            while (p.offsets[t + 1] <= j) t++;
            uint32_t member;
            const int64_t r = p.ranks[j];
            const uint32_t d = fo_deliverer(p, t, r, &member);
            uint32_t at;
            if constexpr (GLOBAL) at = fo_claim(p.base, d);   // base[d] is deliverer d's write cursor
            else at = p.base[(uint64_t) d * gridDim.x + blockIdx.x] + atomicAdd(&cur[d], 1u);
            p.pack_topic[at] = t;
            p.pack_rank[at] = (uint32_t) r;
            if (p.pack_member) p.pack_member[at] = member;
        }
    }
}

// pack_offsets[d] = base[d][0] (the first tile's cursor of deliverer d); pack_offsets[D] = n_pairs
__global__ void fanout_offsets_kernel(const FanoutParams p, uint32_t n_tiles) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d < p.n_deliverers) p.pack_offsets[d] = (long long) p.base[(uint64_t) d * n_tiles];
    if (d == p.n_deliverers) p.pack_offsets[d] = (long long) p.n_pairs;
}

uint32_t fo_tiles(int64_t n_pairs) { return (uint32_t) std::max<int64_t>(1, (n_pairs + FO_TILE - 1) / FO_TILE); }

}  // namespace

// The tile pass while its [deliverer][tile] matrix has at most one cell per pair (FO_TILE cells for a batch of less than one
// tile): its scratch stays at most 8 bytes per pair, and n_deliverers <= FO_TILE follows, so the histogram fits in 16 KB of
// shared memory. Otherwise the global pass, whose scratch is 8 bytes per deliverer id.
bool fanout_tiled(uint32_t n_deliverers, int64_t n_pairs) {
    const uint64_t cells = (uint64_t) n_deliverers * fo_tiles(n_pairs);
    return cells <= (uint64_t) std::min<int64_t>(std::max<int64_t>(n_pairs, FO_TILE), 0x7FFFFFFF);
}

size_t fanout_scratch_words(uint32_t n_deliverers, int64_t n_pairs, bool tiled) {
    return tiled ? (size_t) n_deliverers * fo_tiles(n_pairs) : (size_t) n_deliverers + 1;
}

cudaError_t launch_fanout(const FanoutParams& p, bool tiled, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    const uint32_t n_tiles = fo_tiles(p.n_pairs);
    const int cells = (int) fanout_scratch_words(p.n_deliverers, p.n_pairs, tiled);
    if (!d_tmp) return cub::DeviceScan::ExclusiveSum(nullptr, *tmp_bytes, p.counts, p.base, cells, stream);
    if (!tiled) {
        // counts[D] stays 0, so the exclusive scan's last entry is n_pairs
        cudaError_t e = cudaMemsetAsync(p.counts, 0, (size_t) cells * sizeof(uint32_t), stream);
        if (e != cudaSuccess) return e;
        fanout_count_kernel<true><<<n_tiles, FO_THREADS, 0, stream>>>(p);
        e = cub::DeviceScan::ExclusiveSum(d_tmp, *tmp_bytes, p.counts, p.base, cells, stream);
        if (e != cudaSuccess) return e;
        // offsets before the scatter: the scatter advances base[] as its cursors
        fanout_offsets_kernel<<<(p.n_deliverers + 1 + 255) / 256, 256, 0, stream>>>(p, 1);
        fanout_scatter_kernel<true><<<n_tiles, FO_THREADS, 0, stream>>>(p);
        return cudaGetLastError();
    }
    const size_t smem = (size_t) p.n_deliverers * sizeof(uint32_t);   // <= 16 KB (fanout_tiled)
    fanout_count_kernel<false><<<n_tiles, FO_THREADS, smem, stream>>>(p);
    cudaError_t e = cub::DeviceScan::ExclusiveSum(d_tmp, *tmp_bytes, p.counts, p.base, cells, stream);
    if (e != cudaSuccess) return e;
    fanout_scatter_kernel<false><<<n_tiles, FO_THREADS, smem, stream>>>(p);
    fanout_offsets_kernel<<<(p.n_deliverers + 1 + 255) / 256, 256, 0, stream>>>(p, n_tiles);
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ delivery nesting
// BatchDeliveryCall (bifromq-deliverer/.../BatchDeliveryCall.java:58,75-104) nests a deliverer's calls as
// tenantId -> TopicMessagePack -> Set<MatchInfo> and sends one DeliveryRequest. The pairs are emitted in (tenant, topic position)
// order, so a STABLE partition on the deliverer id alone leaves every deliverer's pairs in (tenant, topic position) order:
//   1. tenant-major topic order   stable radix sort of the topic positions by tenant index (work ~ topics, not pairs)
//   2. emit                       per pair in that order: key = deliverer id (fo_deliverer, as the fan-out), value = emit position
//   3. partition                  cub::DeviceRadixSort::SortPairs on the bits of the deliverer id (stable)
//   4. segments                   head flags where (deliverer, tenant) or (deliverer, topic) changes, their exclusive scans
//                                 (package / pack numbers), one scatter of the offsets
// Emit positions past the pairs nested (the CSR may hold pairs of a topic without a valid tenant, or disagree with n_pairs)
// carry the key n_deliverers, so they sort last and are never read back.
namespace {

constexpr int DL_THREADS = 256;

uint32_t bits_for(uint32_t v) { return v ? 32u - (uint32_t) __builtin_clz(v) : 1u; }

__global__ void __launch_bounds__(DL_THREADS) delivery_topic_keys_kernel(const DeliveryParams q) {
    const int64_t t = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (t >= q.f.n_topics) return;
    const int32_t tn = q.topic_tenant[t];
    q.tkey[0][t] = (tn >= 0 && tn < q.n_tenants) ? (uint32_t) tn : (uint32_t) q.n_tenants;
    q.tval[0][t] = (uint32_t) t;
}

// pairs of the i-th topic in tenant-major order; none for a topic without a valid tenant, none at all if the CSR's total is not n_pairs
__global__ void __launch_bounds__(DL_THREADS) delivery_topic_counts_kernel(const DeliveryParams q, const uint32_t* tkey, const uint32_t* order) {
    const int64_t i = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (i > q.f.n_topics) return;
    uint32_t c = 0;
    if (i < q.f.n_topics && tkey[i] < (uint32_t) q.n_tenants && q.f.offsets[q.f.n_topics] == q.f.n_pairs) {
        const uint32_t t = order[i];
        c = (uint32_t) (q.f.offsets[t + 1] - q.f.offsets[t]);
    }
    q.tcount[i] = c;
}

// last i with start[i] <= j (start monotone, start[0] = 0 <= j < start[n])
__device__ __forceinline__ uint32_t dl_segment_of(const uint32_t* start, int64_t n, uint32_t j) {
    int64_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (start[mid] <= j) lo = mid;
        else hi = mid;
    }
    return (uint32_t) lo;
}

// a thread owns FO_TILE / FO_THREADS consecutive emit positions, as the fan-out's passes do
__global__ void __launch_bounds__(FO_THREADS) delivery_emit_kernel(const DeliveryParams q, const uint32_t* order) {
    constexpr int PER = FO_TILE / FO_THREADS;
    const int64_t j0 = (int64_t) blockIdx.x * FO_TILE + (int64_t) threadIdx.x * PER;
    if (j0 >= q.f.n_pairs) return;
    const int64_t n_emit = q.tstart[q.f.n_topics];
    uint32_t i = j0 < n_emit ? dl_segment_of(q.tstart, q.f.n_topics, (uint32_t) j0) : 0;
    for (int k = 0; k < PER && j0 + k < q.f.n_pairs; k++) {
        const uint32_t j = (uint32_t) (j0 + k);
        q.val[0][j] = j;
        if (j >= n_emit) {
            q.key[0][j] = q.f.n_deliverers;
            continue;
        }
        while (q.tstart[i + 1] <= j) i++;
        const uint32_t t = order[i];
        const int64_t r = q.f.ranks[q.f.offsets[t] + (j - q.tstart[i])];
        uint32_t member;
        q.key[0][j] = fo_deliverer(q.f, t, r, &member);
        q.e_topic[j] = i;
        q.e_rank[j] = (uint32_t) r;
        q.e_member[j] = member;
    }
}

// nested pair k (deliverer-major): its pair, its tenant-major topic index and its head flags
__global__ void __launch_bounds__(DL_THREADS) delivery_gather_kernel(const DeliveryParams q, const uint32_t* skey, const uint32_t* sval,
                                                                     const uint32_t* tkey) {
    const int64_t k = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (k > q.f.n_pairs) return;
    if (k >= (int64_t) q.tstart[q.f.n_topics]) {
        q.package_head[k] = 0;
        q.pack_head[k] = 0;
        return;
    }
    const uint32_t j = sval[k], i = q.e_topic[j], d = skey[k];
    q.s_topic[k] = i;
    q.match_rank[k] = q.e_rank[j];
    q.match_member[k] = q.e_member[j];
    bool package = true, pack = true;
    if (k > 0) {
        const uint32_t i0 = q.e_topic[sval[k - 1]], d0 = skey[k - 1];
        package = d != d0 || tkey[i] != tkey[i0];
        pack = d != d0 || i != i0;
    }
    q.package_head[k] = package;
    q.pack_head[k] = pack;
}

// package_head[] / pack_head[] scanned (exclusive, n_pairs + 1 entries): a head's package / pack number, and the totals at
// [n_emit]. Thread 0 writes the terminators and the totals.
__global__ void __launch_bounds__(DL_THREADS) delivery_scatter_kernel(const DeliveryParams q, const uint32_t* skey, const uint32_t* tkey,
                                                                      const uint32_t* order) {
    const int64_t k = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    const int64_t n_emit = q.tstart[q.f.n_topics];
    if (k == 0) {
        const uint32_t n_packages = q.package_head[n_emit], n_packs = q.pack_head[n_emit];
        q.pack_off[n_packages] = n_packs;
        q.match_off[n_packs] = n_emit;
        q.totals[0] = (unsigned long long) n_emit;
        q.totals[1] = n_packages;
        q.totals[2] = n_packs;
        q.totals[3] = (unsigned long long) q.f.offsets[q.f.n_topics];
    }
    if (k >= n_emit) return;
    const uint32_t pk = q.pack_head[k], pg = q.package_head[k];
    const uint32_t i = q.s_topic[k];
    if (q.pack_head[k + 1] != pk) {
        q.pack_topic[pk] = order[i];
        q.match_off[pk] = k;
    }
    if (q.package_head[k + 1] != pg) {
        q.package_tenant[pg] = tkey[i];
        q.pack_off[pg] = pk;
        atomicAdd(&q.pcount[skey[k]], 1u);
    }
}

unsigned dl_blocks(int64_t n) { return (unsigned) std::max<int64_t>(1, (n + DL_THREADS - 1) / DL_THREADS); }

}  // namespace

cudaError_t launch_delivery(const DeliveryParams& q, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    // item counts as uint32 (pairs and topics are below 2^32): CUB then keeps 32-bit offsets
    const uint32_t T = (uint32_t) q.f.n_topics, n = (uint32_t) q.f.n_pairs;
    const uint32_t D = q.f.n_deliverers;
    const int tbits = (int) bits_for((uint32_t) q.n_tenants), dbits = (int) bits_for(D);
    cub::DoubleBuffer<uint32_t> tk(q.tkey[0], q.tkey[1]), tv(q.tval[0], q.tval[1]);
    cub::DoubleBuffer<uint32_t> dk(q.key[0], q.key[1]), dv(q.val[0], q.val[1]);
    if (!d_tmp) {
        size_t a = 0, b = 0, c = 0, d = 0, e = 0;
        cudaError_t err = cub::DeviceRadixSort::SortPairs(nullptr, a, tk, tv, T, 0, tbits, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, b, q.tcount, q.tstart, T + 1, stream);
        if (err == cudaSuccess) err = cub::DeviceRadixSort::SortPairs(nullptr, c, dk, dv, n, 0, dbits, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, d, q.pack_head, n + 1, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, e, q.pcount, q.package_off, D + 1, stream);
        *tmp_bytes = std::max({a, b, c, d, e});
        return err;
    }
    size_t bytes = *tmp_bytes;
    cudaError_t err = cudaMemsetAsync(q.pcount, 0, ((size_t) D + 1) * sizeof(uint32_t), stream);
    if (err != cudaSuccess) return err;
    delivery_topic_keys_kernel<<<dl_blocks(T), DL_THREADS, 0, stream>>>(q);
    if ((err = cub::DeviceRadixSort::SortPairs(d_tmp, bytes, tk, tv, T, 0, tbits, stream)) != cudaSuccess) return err;
    delivery_topic_counts_kernel<<<dl_blocks(T + 1), DL_THREADS, 0, stream>>>(q, tk.Current(), tv.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.tcount, q.tstart, T + 1, stream)) != cudaSuccess) return err;
    delivery_emit_kernel<<<fo_tiles(n), FO_THREADS, 0, stream>>>(q, tv.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceRadixSort::SortPairs(d_tmp, bytes, dk, dv, n, 0, dbits, stream)) != cudaSuccess) return err;
    delivery_gather_kernel<<<dl_blocks(n + 1), DL_THREADS, 0, stream>>>(q, dk.Current(), dv.Current(), tk.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.package_head, n + 1, stream)) != cudaSuccess) return err;
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.pack_head, n + 1, stream)) != cudaSuccess) return err;
    delivery_scatter_kernel<<<dl_blocks(n), DL_THREADS, 0, stream>>>(q, dk.Current(), tk.Current(), tv.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.pcount, q.package_off, D + 1, stream)) != cudaSuccess) return err;
    return cudaGetLastError();
}

// ------------------------------------------------------------------------------------------------ host: interning
namespace {
// "<decimal subBrokerId>\0<receiverId>\0<delivererKey>"  (DWS/KVSchemaUtil.java:56-58; parsed by cache/ReceiverCache.java:32-36)
bool split_receiver_url(sv url, int32_t* broker, sv* deliverer_key) {
    const size_t a = url.find('\0');
    if (a == sv::npos) return false;
    const size_t b = url.find('\0', a + 1);
    if (b == sv::npos) return false;
    int64_t v = 0;
    if (a == 0) return false;
    for (size_t i = 0; i < a; i++) {
        if (url[i] < '0' || url[i] > '9') return false;
        v = v * 10 + (url[i] - '0');
        if (v > 0x7FFFFFFF) return false;
    }
    *broker = (int32_t) v;
    *deliverer_key = url.substr(b + 1);
    return true;
}
// RouteGroup { map<string, uint64> members = 1; }  (bifromq-dist-worker-schema/src/main/proto/distservice/RouteGroup.proto:27-29):
// repeated field 1, each a nested message {1: string key, 2: varint value}. Calls f(receiverUrl) per member in wire order.
template <typename F>
bool for_each_group_member(sv b, F&& f) {
    size_t i = 0;
    auto varint = [&](uint64_t* out) {
        uint64_t v = 0;
        int shift = 0;
        while (i < b.size()) {
            const uint8_t c = (uint8_t) b[i++];
            v |= (uint64_t) (c & 0x7F) << shift;
            if (!(c & 0x80)) {
                *out = v;
                return true;
            }
            shift += 7;
            if (shift > 63) return false;
        }
        return false;
    };
    while (i < b.size()) {
        uint64_t tag, len;
        if (!varint(&tag)) return false;
        if (tag != ((1u << 3) | 2u)) return false;
        if (!varint(&len) || i + len > b.size()) return false;
        const size_t end = i + (size_t) len;
        sv key;
        while (i < end) {
            uint64_t t2;
            if (!varint(&t2)) return false;
            if (t2 == ((1u << 3) | 2u)) {
                uint64_t kl;
                if (!varint(&kl) || i + kl > end) return false;
                key = b.substr(i, (size_t) kl);
                i += (size_t) kl;
            } else if (t2 == (2u << 3)) {
                uint64_t v;
                if (!varint(&v)) return false;
            } else {
                return false;
            }
        }
        f(key);
    }
    return true;
}
}  // namespace

uint32_t DelivererTable::intern(int32_t broker, sv key) {
    std::string k = std::to_string(broker);
    k.push_back('\0');
    k.append(key);
    std::lock_guard<std::mutex> g(mu);
    auto it = ids.find(k);
    if (it != ids.end()) return it->second;
    const uint32_t id = (uint32_t) list.size();
    list.emplace_back(broker, std::string(key));
    ids.emplace(std::move(k), id);
    return id;
}

bool build_tenant_fan(const KVBlob& kv, DelivererTable* table, TenantFan* out, std::string* err) {
    const int64_t n = kv.n();
    out->rdeliv.assign((size_t) n, 0);
    out->gmem_off.assign(1, 0);
    out->gmem_deliv.clear();
    out->gordered.clear();
    for (int64_t r = 0; r < n; r++) {
        DecodedKey d;
        if (!decode_route_key(kv.key(r), &d)) {
            if (err) *err = "undecodable route key";
            return false;
        }
        if (d.kind != KIND_GROUP) {
            int32_t broker = 0;
            sv dk;
            if (!split_receiver_url(d.receiver, &broker, &dk)) {
                if (err) *err = "receiver url without subBrokerId / delivererKey";
                return false;
            }
            out->rdeliv[(size_t) r] = table->intern(broker, dk);
            continue;
        }
        out->rdeliv[(size_t) r] = FO_GROUP_BIT | (uint32_t) out->gordered.size();
        out->gordered.push_back(d.flag == FLAG_ORDERED ? 1 : 0);
        bool ok = true;
        const bool parsed = for_each_group_member(kv.val(r), [&](sv url) {
            int32_t broker = 0;
            sv dk;
            if (!split_receiver_url(url, &broker, &dk)) {
                ok = false;
                return;
            }
            out->gmem_deliv.push_back(table->intern(broker, dk));
        });
        if (!parsed || !ok) {
            if (err) *err = "undecodable RouteGroup value";
            return false;
        }
        out->gmem_off.push_back((uint32_t) out->gmem_deliv.size());
    }
    return true;
}

}  // namespace bfq
