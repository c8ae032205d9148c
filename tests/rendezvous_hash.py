"""Guava's Hashing.murmur3_128() and RendezvousHash.get restated in Python: the $oshare member pick of
DeliverExecutorGroup.send's ordered branch. Plain code (murmur3_128, score, rendezvous_pick) and a numpy form for many pairs
at once (scores_np); tests/test_host_oshare_cpu.py pins both on Guava's test vectors and on each other."""
import numpy as np

M64 = (1 << 64) - 1
C1, C2 = 0x87C37B91114253D5, 0x4CF5AD432745937F
LONG_MIN = -(1 << 63)


# ------------------------------------------------------------------ Guava's murmur3_128, restated
def _rotl(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def _fmix(k):
    k ^= k >> 33
    k = (k * 0xFF51AFD7ED558CCD) & M64
    k ^= k >> 33
    k = (k * 0xC4CEB9FE1A85EC53) & M64
    k ^= k >> 33
    return k


def murmur3_128(data, seed=0):
    """MurmurHash3_x64_128 over bytes -> (h1, h2) as unsigned 64-bit values (Guava's Murmur3_128HashFunction)"""
    h1 = h2 = seed
    n = len(data)
    for i in range(n // 16):
        k1 = int.from_bytes(data[16 * i:16 * i + 8], "little")
        k2 = int.from_bytes(data[16 * i + 8:16 * i + 16], "little")
        h1 ^= (_rotl((k1 * C1) & M64, 31) * C2) & M64
        h1 = (_rotl(h1, 27) + h2) & M64
        h1 = (h1 * 5 + 0x52DCE729) & M64
        h2 ^= (_rotl((k2 * C2) & M64, 33) * C1) & M64
        h2 = (_rotl(h2, 31) + h1) & M64
        h2 = (h2 * 5 + 0x38495AB5) & M64
    tail = data[n // 16 * 16:]
    if len(tail) > 8:
        h2 ^= (_rotl((int.from_bytes(tail[8:], "little") * C2) & M64, 33) * C1) & M64
    if tail:
        h1 ^= (_rotl((int.from_bytes(tail[:8], "little") * C1) & M64, 31) * C2) & M64
    h1 ^= n
    h2 ^= n
    h1 = (h1 + h2) & M64
    h2 = (h2 + h1) & M64
    h1, h2 = _fmix(h1), _fmix(h2)
    h1 = (h1 + h2) & M64
    h2 = (h2 + h1) & M64
    return h1, h2


def score(publisher_hash, receiver_url):
    """putInt(hash).putString(url, UTF_8).hash().asLong(): little-endian int, then the url's bytes; h1 as a signed long"""
    h1 = murmur3_128(int(publisher_hash).to_bytes(4, "little", signed=True) + bytes(receiver_url))[0]
    return h1 - (1 << 64) if h1 >> 63 else h1


def rendezvous_pick(publisher_hash, member_urls):
    """RendezvousHash.get: the first member whose score beats every earlier one, or None (every score Long.MIN_VALUE)"""
    best, winner = LONG_MIN, None
    for m, url in enumerate(member_urls):
        s = score(publisher_hash, url)
        if s > best:
            best, winner = s, m
    return winner


def scores_np(hashes, urls):
    """score() for many (hash, url) pairs at once (numpy, wrapping uint64 arithmetic): the same function, used where a batch
    has too many pairs for the plain loop. Cross-checked against score() below."""
    hashes = np.asarray(hashes, np.int64)
    streams = [int(h).to_bytes(4, "little", signed=True) + bytes(u) for h, u in zip(hashes.tolist(), urls)]
    n = np.array([len(s) for s in streams], np.uint64)
    width = int(max(n.max(initial=0), 1) + 15) // 16 * 16
    buf = np.zeros((len(streams), width), np.uint8)
    for i, s in enumerate(streams):
        buf[i, :len(s)] = np.frombuffer(s, np.uint8)
    words = buf.view("<u8")
    u = np.uint64
    rot = lambda x, r: (x << u(r)) | (x >> u(64 - r))
    h1 = np.zeros(len(streams), np.uint64)
    h2 = np.zeros(len(streams), np.uint64)
    with np.errstate(over="ignore"):
        for b in range(width // 16):
            full = n >= u(16 * (b + 1))
            k1, k2 = words[:, 2 * b], words[:, 2 * b + 1]
            x1 = h1 ^ (rot(k1 * u(C1), 31) * u(C2))
            x1 = (rot(x1, 27) + h2) * u(5) + u(0x52DCE729)
            x2 = h2 ^ (rot(k2 * u(C2), 33) * u(C1))
            x2 = (rot(x2, 31) + x1) * u(5) + u(0x38495AB5)
            # tail block: the padding is zero, so the partial words are the tail's little-endian values
            rem = n - u(16 * b)
            tail = (n // u(16)) == u(b)
            t2 = h2 ^ np.where(rem > u(8), rot(k2 * u(C2), 33) * u(C1), u(0))
            t1 = h1 ^ np.where(rem > u(0), rot(k1 * u(C1), 31) * u(C2), u(0))
            h1 = np.where(full, x1, np.where(tail, t1, h1))
            h2 = np.where(full, x2, np.where(tail, t2, h2))
        h1 ^= n
        h2 ^= n
        h1 = h1 + h2
        h2 = h2 + h1

        def fmix(k):
            k = k ^ (k >> u(33))
            k = k * u(0xFF51AFD7ED558CCD)
            k = k ^ (k >> u(33))
            k = k * u(0xC4CEB9FE1A85EC53)
            return k ^ (k >> u(33))
        h1, h2 = fmix(h1), fmix(h2)
        return (h1 + h2).view(np.int64)
