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
//
// $oshare resolution (q.oshare, bfq_delivery_device_ordered) adds, between 1 and 2, the ordered branch of
// DeliverExecutorGroup.send (DW/DeliverExecutorGroup.java:242-278): per ($oshare pair, publisher of its topic position) an
// "item", per item the rendezvous winner (RendezvousHash.get: the first member whose Guava murmur3_128 score over
// LE32(publisher hash) ‖ receiverUrl is strictly greater than every earlier one), and per (pair, winner) a "sub-pack" of the
// publishers that picked it, in publisher order. Each topic then emits its ordinary pairs (the resolved $oshare pairs emit the
// key n_deliverers: dropped) and after them its sub-packs in (rank, member) order; a sub-pack is a pack of its own. The stable
// partition keeps that order per deliverer. Kernels templated on OSH: without it they compile to the plain nesting.
namespace {

constexpr int DL_THREADS = 256;
constexpr uint32_t NO_SUB = 0xFFFFFFFFu;

uint32_t bits_for(uint32_t v) { return v ? 32u - (uint32_t) __builtin_clz(v) : 1u; }

// emit positions of the nesting: the pairs, plus (with $oshare) room for one sub-pack per item
template <bool OSH>
__host__ __device__ __forceinline__ int64_t dl_emit_cap(const DeliveryParams& q) {
    if constexpr (OSH) return q.f.n_pairs + q.o.n_items;
    else return q.f.n_pairs;
}

__global__ void __launch_bounds__(DL_THREADS) delivery_topic_keys_kernel(const DeliveryParams q) {
    const int64_t t = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (t >= q.f.n_topics) return;
    const int32_t tn = q.topic_tenant[t];
    q.tkey[0][t] = (tn >= 0 && tn < q.n_tenants) ? (uint32_t) tn : (uint32_t) q.n_tenants;
    q.tval[0][t] = (uint32_t) t;
}

// the sub-packs of topic position t: [first, first + n) (OSH; the $oshare pairs of t are the scanned oflag's range over t's
// pairs, their items istart[] of those, and their sub-packs the item heads before them)
__device__ __forceinline__ void os_topic_subs(const DeliveryParams& q, uint32_t t, uint32_t* first, uint32_t* n) {
    const uint32_t olo = q.o.oflag[q.f.offsets[t]], ohi = q.o.oflag[q.f.offsets[t + 1]];
    *first = q.o.ihead[q.o.istart[olo]];
    *n = q.o.ihead[q.o.istart[ohi]] - *first;
}

// pairs of the i-th topic in tenant-major order; none for a topic without a valid tenant, none at all if the CSR's total is not n_pairs
template <bool OSH>
__global__ void __launch_bounds__(DL_THREADS) delivery_topic_counts_kernel(const DeliveryParams q, const uint32_t* tkey, const uint32_t* order) {
    const int64_t i = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (i > q.f.n_topics) return;
    uint32_t c = 0;
    if (i < q.f.n_topics && tkey[i] < (uint32_t) q.n_tenants && q.f.offsets[q.f.n_topics] == q.f.n_pairs) {
        const uint32_t t = order[i];
        c = (uint32_t) (q.f.offsets[t + 1] - q.f.offsets[t]);
        if constexpr (OSH) {
            uint32_t s0, ns;
            os_topic_subs(q, t, &s0, &ns);
            c += ns;
        }
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
template <bool OSH>
__global__ void __launch_bounds__(FO_THREADS) delivery_emit_kernel(const DeliveryParams q, const uint32_t* order) {
    constexpr int PER = FO_TILE / FO_THREADS;
    const int64_t cap = dl_emit_cap<OSH>(q);
    const int64_t j0 = (int64_t) blockIdx.x * FO_TILE + (int64_t) threadIdx.x * PER;
    if (j0 >= cap) return;
    const int64_t n_emit = q.tstart[q.f.n_topics];
    uint32_t i = j0 < n_emit ? dl_segment_of(q.tstart, q.f.n_topics, (uint32_t) j0) : 0;
    uint32_t cur = 0xFFFFFFFFu, s0 = 0, ns = 0;   // OSH: the topic whose sub-packs s0 / ns hold
    for (int k = 0; k < PER && j0 + k < cap; k++) {
        const uint32_t j = (uint32_t) (j0 + k);
        q.val[0][j] = j;
        if (j >= n_emit) {
            q.key[0][j] = q.f.n_deliverers;
            continue;
        }
        while (q.tstart[i + 1] <= j) i++;
        const uint32_t t = order[i];
        const uint32_t local = j - q.tstart[i];
        const uint32_t cnt = (uint32_t) (q.f.offsets[t + 1] - q.f.offsets[t]);
        int64_t r;
        uint32_t member = 0xFFFFFFFFu, d;
        if constexpr (OSH) {
            if (local < cnt) {
                const int64_t pj = q.f.offsets[t] + local;
                r = q.f.ranks[pj];
                // a resolved $oshare pair: its sub-packs stand for it
                d = q.o.oflag[pj + 1] != q.o.oflag[pj] ? q.f.n_deliverers : fo_deliverer(q.f, t, r, &member);
                q.o.e_sub[j] = NO_SUB;
            } else {
                if (cur != t) {
                    os_topic_subs(q, t, &s0, &ns);
                    cur = t;
                }
                const uint32_t s = s0 + (local - cnt);
                const unsigned long long kk = q.o.ikey[0][q.o.sub_start[s]];
                const uint32_t w = (uint32_t) (kk & ((1ull << q.o.member_bits) - 1));
                r = (int64_t) (q.o.okey[0][kk >> q.o.member_bits] & 0xFFFFFFFFu);
                const uint32_t g = q.f.rdeliv[r] & ~FO_GROUP_BIT;
                const uint32_t b = q.f.gmem_off[g], n = q.f.gmem_off[g + 1] - b;
                // w == n: every member scored Long.MIN_VALUE, no winner: parked like a member-less group
                member = w < n ? w : 0xFFFFFFFFu;
                d = w < n ? q.f.gmem_deliv[b + w] : q.f.n_deliverers - 1;
                q.o.e_sub[j] = s;
            }
        } else {
            r = q.f.ranks[q.f.offsets[t] + local];
            d = fo_deliverer(q.f, t, r, &member);
        }
        q.key[0][j] = d;
        q.e_topic[j] = i;
        q.e_rank[j] = (uint32_t) r;
        q.e_member[j] = member;
    }
}

// pairs nested: the emit positions, less the resolved $oshare pairs (their key was n_deliverers)
template <bool OSH>
__device__ __forceinline__ int64_t dl_nested(const DeliveryParams& q) {
    if constexpr (OSH) return (int64_t) q.tstart[q.f.n_topics] - q.o.n_opairs;
    else return (int64_t) q.tstart[q.f.n_topics];
}

// nested pair k (deliverer-major): its pair, its tenant-major topic index and its head flags
template <bool OSH>
__global__ void __launch_bounds__(DL_THREADS) delivery_gather_kernel(const DeliveryParams q, const uint32_t* skey, const uint32_t* sval,
                                                                     const uint32_t* tkey) {
    const int64_t k = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (k > dl_emit_cap<OSH>(q)) return;
    if (k >= dl_nested<OSH>(q)) {
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
        if constexpr (OSH) pack = pack || q.o.e_sub[j] != NO_SUB || q.o.e_sub[sval[k - 1]] != NO_SUB;
    }
    if constexpr (OSH) q.o.s_sub[k] = q.o.e_sub[j];
    q.package_head[k] = package;
    q.pack_head[k] = pack;
}

// package_head[] / pack_head[] scanned (exclusive, emit cap + 1 entries): a head's package / pack number, and the totals at
// [pairs nested]. Thread 0 writes the terminators and the totals.
template <bool OSH>
__global__ void __launch_bounds__(DL_THREADS) delivery_scatter_kernel(const DeliveryParams q, const uint32_t* skey, const uint32_t* tkey,
                                                                      const uint32_t* order) {
    const int64_t k = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    const int64_t n_emit = dl_nested<OSH>(q);
    if (k == 0) {
        const uint32_t n_packages = q.package_head[n_emit], n_packs = q.pack_head[n_emit];
        q.pack_off[n_packages] = n_packs;
        q.match_off[n_packs] = n_emit;
        q.totals[0] = (unsigned long long) n_emit;
        q.totals[1] = n_packages;
        q.totals[2] = n_packs;
        q.totals[3] = (unsigned long long) q.f.offsets[q.f.n_topics];
        if constexpr (OSH) q.totals[4] = q.o.ihead[q.o.n_items];
    }
    if (k >= n_emit) return;
    const uint32_t pk = q.pack_head[k], pg = q.package_head[k];
    const uint32_t i = q.s_topic[k];
    if (q.pack_head[k + 1] != pk) {
        q.pack_topic[pk] = order[i];
        q.match_off[pk] = k;
        if constexpr (OSH) {
            const uint32_t s = q.o.s_sub[k];
            if (s != NO_SUB) {
                q.o.pub_count[pk] = q.o.sub_start[s + 1] - q.o.sub_start[s];
                q.o.sub_pack[s] = pk;
            }
        }
    }
    if (q.package_head[k + 1] != pg) {
        q.package_tenant[pg] = tkey[i];
        q.pack_off[pg] = pk;
        atomicAdd(&q.pcount[skey[k]], 1u);
    }
}

unsigned dl_blocks(int64_t n) { return (unsigned) std::max<int64_t>(1, (n + DL_THREADS - 1) / DL_THREADS); }

// ---- $oshare: Guava's Hashing.murmur3_128() (MurmurHash3_x64_128, seed 0; Murmur3_128HashFunction.java) restated
__device__ __forceinline__ uint64_t mm3_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t mm3_fmix(uint64_t k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return k;
}
constexpr uint64_t MM3_C1 = 0x87c37b91114253d5ull, MM3_C2 = 0x4cf5ad432745937full;

// newHasher().putInt(hash).putString(url, UTF_8).hash().asLong(): h1 over the n = 4 + len bytes LE32(hash) ‖ url. The url sits
// at byte 4 of the aligned words w[], zero-padded to its last word, so every 16-byte block and the tail are whole word loads.
__device__ __forceinline__ int64_t rendezvous_score(uint32_t hash, const unsigned long long* w, uint32_t len) {
    const uint32_t n = len + 4, nb = n >> 4;
    uint64_t h1 = 0, h2 = 0;
    for (uint32_t i = 0; i < nb; i++) {
        uint64_t k1 = __ldg(w + 2 * i), k2 = __ldg(w + 2 * i + 1);
        if (i == 0) k1 |= hash;
        k1 *= MM3_C1; k1 = mm3_rotl(k1, 31); k1 *= MM3_C2; h1 ^= k1;
        h1 = mm3_rotl(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52dce729;
        k2 *= MM3_C2; k2 = mm3_rotl(k2, 33); k2 *= MM3_C1; h2 ^= k2;
        h2 = mm3_rotl(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495ab5;
    }
    const uint32_t rem = n & 15;
    if (rem) {
        uint64_t k1 = __ldg(w + 2 * nb);
        if (nb == 0) k1 |= hash;
        if (rem > 8) {
            uint64_t k2 = __ldg(w + 2 * nb + 1);
            k2 *= MM3_C2; k2 = mm3_rotl(k2, 33); k2 *= MM3_C1; h2 ^= k2;
        }
        k1 *= MM3_C1; k1 = mm3_rotl(k1, 31); k1 *= MM3_C2; h1 ^= k1;
    }
    h1 ^= n;
    h2 ^= n;
    h1 += h2;
    h2 += h1;
    h1 = mm3_fmix(h1);
    h2 = mm3_fmix(h2);
    return (int64_t) (h1 + h2);
}

// phase 1: d_pub_off must run from 0, never decrease and end at n_pubs (check[2] = 1 otherwise); the scans' last entries
__global__ void __launch_bounds__(DL_THREADS) oshare_check_kernel(const DeliveryParams q) {
    const int64_t t = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    const int64_t T = q.f.n_topics;
    if (t == 0) {
        q.o.oflag[q.f.n_pairs] = 0;
        q.o.oitems[q.f.n_pairs] = 0;
    }
    if (t > T) return;
    const int64_t* po = q.o.pub_off;
    const bool bad = (t == 0 && po[0] != 0) || (t == T && po[T] != q.o.n_pubs) || (t < T && po[t + 1] < po[t]);
    if (bad) atomicOr(&q.o.check[2], 1ull);
}

// phase 1, per CSR pair (the fan-out's walk): an $oshare pair with members in a topic the nesting keeps, and its publishers
__global__ void __launch_bounds__(FO_THREADS) oshare_flag_kernel(const DeliveryParams q) {
    constexpr int PER = FO_TILE / FO_THREADS;
    const int64_t j0 = (int64_t) blockIdx.x * FO_TILE + (int64_t) threadIdx.x * PER;
    if (j0 >= q.f.n_pairs) return;
    const bool csr_ok = q.f.offsets[q.f.n_topics] == q.f.n_pairs;   // else nothing is nested (and the walk has no bound)
    uint32_t t = csr_ok ? fo_topic_of(q.f.offsets, q.f.n_topics, j0) : 0;
    for (int k = 0; k < PER && j0 + k < q.f.n_pairs; k++) {
        const int64_t j = j0 + k;
        uint32_t fl = 0;
        unsigned long long items = 0;
        if (csr_ok) {
            while (q.f.offsets[t + 1] <= j) t++;
            const int32_t tn = q.topic_tenant[t];
            const uint32_t d = q.f.rdeliv[q.f.ranks[j]];
            if (tn >= 0 && tn < q.n_tenants && (d & FO_GROUP_BIT)) {
                const uint32_t g = d & ~FO_GROUP_BIT;
                if (q.f.gordered[g] && q.f.gmem_off[g + 1] > q.f.gmem_off[g]) {
                    fl = 1;
                    items = (unsigned long long) (q.o.pub_off[t + 1] - q.o.pub_off[t]);
                }
            }
        }
        q.o.oflag[j] = fl;
        q.o.oitems[j] = items;
    }
}

__global__ void oshare_total_kernel(const DeliveryParams q) {
    q.o.check[0] = q.o.oflag[q.f.n_pairs];
    q.o.check[1] = q.o.oitems[q.f.n_pairs];
    q.o.check[3] = (unsigned long long) q.f.offsets[q.f.n_topics];
}

// phase 2: the $oshare pairs compacted (scanned oflag), keyed (topic position, rank) so the sort puts each topic's in rank order
__global__ void __launch_bounds__(FO_THREADS) oshare_compact_kernel(const DeliveryParams q) {
    constexpr int PER = FO_TILE / FO_THREADS;
    const int64_t j0 = (int64_t) blockIdx.x * FO_TILE + (int64_t) threadIdx.x * PER;
    if (j0 >= q.f.n_pairs || q.o.n_opairs == 0) return;
    uint32_t t = fo_topic_of(q.f.offsets, q.f.n_topics, j0);
    for (int k = 0; k < PER && j0 + k < q.f.n_pairs; k++) {
        const int64_t j = j0 + k;
        const uint32_t o = q.o.oflag[j];
        if (q.o.oflag[j + 1] == o) continue;
        while (q.f.offsets[t + 1] <= j) t++;
        q.o.okey[0][o] = (unsigned long long) t << 32 | (uint32_t) q.f.ranks[j];
    }
}

// items per sorted $oshare pair (its topic's publishers), scanned in place into istart[]
__global__ void __launch_bounds__(DL_THREADS) oshare_items_kernel(const DeliveryParams q) {
    const int64_t o = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (o > q.o.n_opairs) return;
    uint32_t c = 0;
    if (o < q.o.n_opairs) {
        const uint32_t t = (uint32_t) (q.o.okey[0][o] >> 32);
        c = (uint32_t) (q.o.pub_off[t + 1] - q.o.pub_off[t]);
    }
    q.o.istart[o] = c;
}

// one warp per item: lanes over the group's members, each keeping its first strictly best score, then a warp argmax that
// breaks ties by the lower member index -- the reference's "first member with a strictly greater score". Key (pair, winner).
constexpr int RV_THREADS = 256;
__global__ void __launch_bounds__(RV_THREADS) oshare_rendezvous_kernel(const DeliveryParams q) {
    const int64_t item = ((int64_t) blockIdx.x * RV_THREADS + threadIdx.x) >> 5;
    const uint32_t lane = threadIdx.x & 31u;
    if (item >= q.o.n_items) return;
    const uint32_t o = dl_segment_of(q.o.istart, q.o.n_opairs, (uint32_t) item);
    const unsigned long long ok = q.o.okey[0][o];
    const uint32_t t = (uint32_t) (ok >> 32), r = (uint32_t) ok;
    const uint32_t p = (uint32_t) (q.o.pub_off[t] + ((uint32_t) item - q.o.istart[o]));
    const uint32_t hash = (uint32_t) q.o.pub_hash[p];
    const uint32_t g = q.f.rdeliv[r] & ~FO_GROUP_BIT;
    const uint32_t b = q.f.gmem_off[g], n = q.f.gmem_off[g + 1] - b;
    int64_t best = INT64_MIN;
    uint32_t bm = 0xFFFFFFFFu;
    for (uint32_t m = lane; m < n; m += 32) {
        const int64_t sc = rendezvous_score(hash, q.o.url_words + q.o.url_word[b + m], q.o.url_len[b + m]);
        if (sc > best) {
            best = sc;
            bm = m;
        }
    }
    for (int off = 16; off > 0; off >>= 1) {
        const int64_t ob = __shfl_xor_sync(0xFFFFFFFFu, best, off);
        const uint32_t om = __shfl_xor_sync(0xFFFFFFFFu, bm, off);
        if (ob > best || (ob == best && om < bm)) {
            best = ob;
            bm = om;
        }
    }
    if (lane == 0) {
        q.o.ikey[0][item] = (unsigned long long) o << q.o.member_bits | (bm == 0xFFFFFFFFu ? n : bm);
        q.o.ival[0][item] = p;
    }
}

// sorted items: 1 where (pair, winner) changes (exclusive scan: an item's heads before it), [n_items] = 0
__global__ void __launch_bounds__(DL_THREADS) oshare_heads_kernel(const DeliveryParams q) {
    const int64_t x = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (x > q.o.n_items) return;
    const unsigned long long* ikey = q.o.ikey[0];
    q.o.ihead[x] = x < q.o.n_items && (x == 0 || ikey[x] != ikey[x - 1]);
}

// sub-pack s starts at its head item; sub_start[n_subs] = n_items
__global__ void __launch_bounds__(DL_THREADS) oshare_subs_kernel(const DeliveryParams q) {
    const int64_t x = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (x == 0) q.o.sub_start[q.o.ihead[q.o.n_items]] = (uint32_t) q.o.n_items;
    if (x < q.o.n_items && q.o.ihead[x + 1] != q.o.ihead[x]) q.o.sub_start[q.o.ihead[x]] = (uint32_t) x;
}

// every item's publisher into its sub-pack's pack: pack_pub[pack_pub_off[pack] + its place in the sub-pack]
__global__ void __launch_bounds__(DL_THREADS) oshare_pubs_kernel(const DeliveryParams q, const uint32_t* ival) {
    const int64_t x = (int64_t) blockIdx.x * DL_THREADS + threadIdx.x;
    if (x >= q.o.n_items) return;
    const uint32_t s = q.o.ihead[x + 1] - 1;
    q.o.pack_pub[q.o.pack_pub_off[q.o.sub_pack[s]] + ((uint32_t) x - q.o.sub_start[s])] = ival[x];
}

template <bool OSH>
cudaError_t run_delivery(const DeliveryParams& q0, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    DeliveryParams q = q0;   // OSH: okey[0] / ikey[0] are re-pointed at the sorted buffers
    // item counts as uint32 (emit positions and topics are below 2^32): CUB then keeps 32-bit offsets
    const uint32_t T = (uint32_t) q.f.n_topics, n = (uint32_t) dl_emit_cap<OSH>(q);
    const uint32_t D = q.f.n_deliverers;
    const int tbits = (int) bits_for((uint32_t) q.n_tenants), dbits = (int) bits_for(D);
    cub::DoubleBuffer<uint32_t> tk(q.tkey[0], q.tkey[1]), tv(q.tval[0], q.tval[1]);
    cub::DoubleBuffer<uint32_t> dk(q.key[0], q.key[1]), dv(q.val[0], q.val[1]);
    // $oshare: pairs sorted on (topic position, rank), items on (pair, winner)
    const uint32_t O = OSH ? (uint32_t) q.o.n_opairs : 0, I = OSH ? (uint32_t) q.o.n_items : 0;
    const int okbits = 32 + (int) bits_for(T), ikbits = OSH ? (int) (q.o.member_bits + bits_for(O)) : 0;
    cub::DoubleBuffer<unsigned long long> ok(q.o.okey[0], q.o.okey[1]), ik(q.o.ikey[0], q.o.ikey[1]);
    cub::DoubleBuffer<uint32_t> iv(q.o.ival[0], q.o.ival[1]);
    if (!d_tmp) {
        size_t a = 0, b = 0, c = 0, d = 0, e = 0, f = 0, g = 0, h = 0, k = 0;
        cudaError_t err = cub::DeviceRadixSort::SortPairs(nullptr, a, tk, tv, T, 0, tbits, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, b, q.tcount, q.tstart, T + 1, stream);
        if (err == cudaSuccess) err = cub::DeviceRadixSort::SortPairs(nullptr, c, dk, dv, n, 0, dbits, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, d, q.pack_head, n + 1, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, e, q.pcount, q.package_off, D + 1, stream);
        if constexpr (OSH) {
            if (err == cudaSuccess) err = cub::DeviceRadixSort::SortKeys(nullptr, f, ok, O, 0, okbits, stream);
            if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, g, q.o.istart, O + 1, stream);
            if (err == cudaSuccess) err = cub::DeviceRadixSort::SortPairs(nullptr, h, ik, iv, I, 0, ikbits, stream);
            if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, k, q.o.pub_count, q.o.pack_pub_off, n + 1, stream);
            g = std::max(g, k);
        }
        *tmp_bytes = std::max({a, b, c, d, e, f, g, h});
        return err;
    }
    size_t bytes = *tmp_bytes;
    cudaError_t err = cudaMemsetAsync(q.pcount, 0, ((size_t) D + 1) * sizeof(uint32_t), stream);
    if (err != cudaSuccess) return err;
    delivery_topic_keys_kernel<<<dl_blocks(T), DL_THREADS, 0, stream>>>(q);
    if ((err = cub::DeviceRadixSort::SortPairs(d_tmp, bytes, tk, tv, T, 0, tbits, stream)) != cudaSuccess) return err;
    if constexpr (OSH) {
        if ((err = cudaMemsetAsync(q.o.pub_count, 0, ((size_t) n + 1) * sizeof(uint32_t), stream)) != cudaSuccess) return err;
        oshare_compact_kernel<<<fo_tiles(q.f.n_pairs), FO_THREADS, 0, stream>>>(q);
        bytes = *tmp_bytes;
        if ((err = cub::DeviceRadixSort::SortKeys(d_tmp, bytes, ok, O, 0, okbits, stream)) != cudaSuccess) return err;
        q.o.okey[0] = ok.Current();
        oshare_items_kernel<<<dl_blocks(O + 1), DL_THREADS, 0, stream>>>(q);
        bytes = *tmp_bytes;
        if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.o.istart, O + 1, stream)) != cudaSuccess) return err;
        if (I > 0) {
            const unsigned warps_per_block = RV_THREADS / 32;
            oshare_rendezvous_kernel<<<(unsigned) ((I + warps_per_block - 1) / warps_per_block), RV_THREADS, 0, stream>>>(q);
        }
        bytes = *tmp_bytes;
        if ((err = cub::DeviceRadixSort::SortPairs(d_tmp, bytes, ik, iv, I, 0, ikbits, stream)) != cudaSuccess) return err;
        q.o.ikey[0] = ik.Current();
        oshare_heads_kernel<<<dl_blocks(I + 1), DL_THREADS, 0, stream>>>(q);
        bytes = *tmp_bytes;
        if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.o.ihead, I + 1, stream)) != cudaSuccess) return err;
        oshare_subs_kernel<<<dl_blocks(I), DL_THREADS, 0, stream>>>(q);
    }
    delivery_topic_counts_kernel<OSH><<<dl_blocks(T + 1), DL_THREADS, 0, stream>>>(q, tk.Current(), tv.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.tcount, q.tstart, T + 1, stream)) != cudaSuccess) return err;
    delivery_emit_kernel<OSH><<<fo_tiles(n), FO_THREADS, 0, stream>>>(q, tv.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceRadixSort::SortPairs(d_tmp, bytes, dk, dv, n, 0, dbits, stream)) != cudaSuccess) return err;
    delivery_gather_kernel<OSH><<<dl_blocks(n + 1), DL_THREADS, 0, stream>>>(q, dk.Current(), dv.Current(), tk.Current());
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.package_head, n + 1, stream)) != cudaSuccess) return err;
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.pack_head, n + 1, stream)) != cudaSuccess) return err;
    delivery_scatter_kernel<OSH><<<dl_blocks(n), DL_THREADS, 0, stream>>>(q, dk.Current(), tk.Current(), tv.Current());
    if constexpr (OSH) {
        bytes = *tmp_bytes;
        if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.o.pub_count, q.o.pack_pub_off, n + 1, stream)) != cudaSuccess) return err;
        oshare_pubs_kernel<<<dl_blocks(I), DL_THREADS, 0, stream>>>(q, iv.Current());
    }
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.pcount, q.package_off, D + 1, stream)) != cudaSuccess) return err;
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_delivery(const DeliveryParams& q, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    return q.oshare ? run_delivery<true>(q, d_tmp, tmp_bytes, stream) : run_delivery<false>(q, d_tmp, tmp_bytes, stream);
}

cudaError_t launch_oshare_count(const DeliveryParams& q, void* d_tmp, size_t* tmp_bytes, cudaStream_t stream) {
    const uint32_t n = (uint32_t) q.f.n_pairs;
    if (!d_tmp) {
        size_t a = 0, b = 0;
        cudaError_t err = cub::DeviceScan::ExclusiveSum(nullptr, a, q.o.oflag, n + 1, stream);
        if (err == cudaSuccess) err = cub::DeviceScan::ExclusiveSum(nullptr, b, q.o.oitems, n + 1, stream);
        *tmp_bytes = std::max(a, b);
        return err;
    }
    cudaError_t err = cudaMemsetAsync(q.o.check, 0, 4 * sizeof(unsigned long long), stream);
    if (err != cudaSuccess) return err;
    oshare_check_kernel<<<dl_blocks(q.f.n_topics + 1), DL_THREADS, 0, stream>>>(q);
    oshare_flag_kernel<<<fo_tiles(n), FO_THREADS, 0, stream>>>(q);
    size_t bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.o.oflag, n + 1, stream)) != cudaSuccess) return err;
    bytes = *tmp_bytes;
    if ((err = cub::DeviceScan::ExclusiveSum(d_tmp, bytes, q.o.oitems, n + 1, stream)) != cudaSuccess) return err;
    oshare_total_kernel<<<1, 1, 0, stream>>>(q);
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
// repeated field 1, each a nested message {1: string key, 2: varint value}. Calls f(receiverUrl, incarnation) per member in wire
// order.
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
        uint64_t value = 0;
        while (i < end) {
            uint64_t t2;
            if (!varint(&t2)) return false;
            if (t2 == ((1u << 3) | 2u)) {
                uint64_t kl;
                if (!varint(&kl) || i + kl > end) return false;
                key = b.substr(i, (size_t) kl);
                i += (size_t) kl;
            } else if (t2 == (2u << 3)) {
                if (!varint(&value)) return false;
            } else {
                return false;
            }
        }
        f(key, value);
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
    out->ourl_off.assign(1, 0);
    out->ourl.clear();
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
        const bool ordered = d.flag == FLAG_ORDERED;
        out->gordered.push_back(ordered ? 1 : 0);
        bool ok = true;
        const bool parsed = for_each_group_member(kv.val(r), [&](sv url, uint64_t) {
            int32_t broker = 0;
            sv dk;
            if (!split_receiver_url(url, &broker, &dk)) {
                ok = false;
                return;
            }
            out->gmem_deliv.push_back(table->intern(broker, dk));
            if (ordered) out->ourl.append(url);
            out->ourl_off.push_back((uint32_t) out->ourl.size());
        });
        if (!parsed || !ok) {
            if (err) *err = "undecodable RouteGroup value";
            return false;
        }
        out->gmem_off.push_back((uint32_t) out->gmem_deliv.size());
    }
    return true;
}

// ------------------------------------------------------------------------------------------------ host: MatchInfo wire bytes
namespace {
void put_varint(std::string& s, uint64_t v) {
    while (v >= 0x80) {
        s.push_back((char) (uint8_t) (v | 0x80));
        v >>= 7;
    }
    s.push_back((char) (uint8_t) v);
}
void put_len_field(std::string& s, uint8_t tag, sv bytes) {
    s.push_back((char) tag);
    put_varint(s, bytes.size());
    s.append(bytes);
}
// RouteMatcher {type = 1, repeated filterLevel = 2, optional group = 3, mqttTopicFilter = 4} as RouteDetailCache.get builds it:
// Normal (type left at 0) with the unescaped filter; UnorderedShare / OrderedShare with the group set and
// "$share/<group>/<filter>" / "$oshare/<group>/<filter>". filterLevel = parse(escapedFilter, true): every NUL-separated level,
// empty ones included.
std::string route_matcher_bytes(const DecodedKey& d) {
    std::string m;
    const bool group = d.kind == KIND_GROUP;
    if (group) {
        m.push_back(0x08);
        put_varint(m, d.flag == FLAG_ORDERED ? 2 : 1);
    }
    for_each_level(d.escaped_filter, '\0', [&](sv level) { put_len_field(m, 0x12, level); });
    std::string filter(d.escaped_filter);
    std::replace(filter.begin(), filter.end(), '\0', '/');
    if (group) {
        put_len_field(m, 0x1A, d.receiver);
        filter = std::string(d.flag == FLAG_ORDERED ? "$oshare/" : "$share/") + std::string(d.receiver) + "/" + filter;
    }
    if (!filter.empty()) put_len_field(m, 0x22, filter);
    return m;
}
// MatchInfo {matcher = 1, receiverId = 2, incarnation = 3} (NormalMatching), as DeliveryPack's matchInfo = 3 field. receiverId is
// ReceiverCache's parts[1] of "<subBrokerId>\0<receiverId>\0<delivererKey>".
bool put_match_info(std::string& out, const std::string& matcher, sv receiver_url, uint64_t incarnation) {
    const size_t a = receiver_url.find('\0');
    const size_t b = a == sv::npos ? sv::npos : receiver_url.find('\0', a + 1);
    if (b == sv::npos) return false;
    std::string mi;
    put_len_field(mi, 0x0A, matcher);
    if (b > a + 1) put_len_field(mi, 0x12, receiver_url.substr(a + 1, b - a - 1));
    if (incarnation) {
        mi.push_back(0x18);
        put_varint(mi, incarnation);
    }
    put_len_field(out, 0x1A, mi);
    return true;
}
}  // namespace

bool build_tenant_wire(const KVBlob& kv, TenantWire* out, std::string* err) {
    const int64_t n = kv.n();
    out->first.assign((size_t) n, 0);
    out->off.assign(1, 0);
    out->bytes.clear();
    auto fail_with = [&](const char* what) {
        if (err) *err = what;
        return false;
    };
    for (int64_t r = 0; r < n; r++) {
        DecodedKey d;
        if (!decode_route_key(kv.key(r), &d)) return fail_with("undecodable route key");
        out->first[(size_t) r] = (uint32_t) (out->off.size() - 1);
        const std::string matcher = route_matcher_bytes(d);
        if (d.kind != KIND_GROUP) {
            const sv v = kv.val(r);   // BSUtil.toLong: 8 bytes, big-endian
            if (v.size() < 8) return fail_with("normal route value shorter than 8 bytes");
            uint64_t inc = 0;
            for (int i = 0; i < 8; i++) inc = inc << 8 | (uint8_t) v[(size_t) i];
            if (!put_match_info(out->bytes, matcher, d.receiver, inc)) return fail_with("receiver url without a receiverId");
            out->off.push_back(out->bytes.size());
            continue;
        }
        bool ok = true;
        const bool parsed = for_each_group_member(kv.val(r), [&](sv url, uint64_t inc) {
            ok = ok && put_match_info(out->bytes, matcher, url, inc);
            out->off.push_back(out->bytes.size());
        });
        if (!parsed) return fail_with("undecodable RouteGroup value");
        if (!ok) return fail_with("member receiver url without a receiverId");
    }
    if (out->off.size() - 1 >= 0xFFFFFFFFull) return fail_with("2^32 or more MatchInfos in one tenant");
    return true;
}

}  // namespace bfq
