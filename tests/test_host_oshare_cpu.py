"""The ordered shared subscription ($oshare) pick and the delivery nesting it produces, restated in plain Python.

DeliverExecutorGroup.send's ordered branch (bifromq-dist-worker/.../DeliverExecutorGroup.java:242-278) sends every publisher
pack of a topic's TopicMessagePack to ONE member of the group, RendezvousHash.get (base-util/.../RendezvousHash.java): member
m scores Hashing.murmur3_128().newHasher().putInt(publisher.hashCode()).putString(receiverUrl_m, UTF_8).hash().asLong(), and
the first member whose score is strictly greater than every earlier one (the running best starts at Long.MIN_VALUE) wins.
Publishers with one winner become one new TopicMessagePack in a fresh TopicMessagePackHolder, so BatchDeliveryCall.add
(bifromq-deliverer/.../BatchDeliveryCall.java:75-80) files each as a DeliveryPack of its own with one MatchInfo.

rendezvous_hash.murmur3_128() restates Guava's Murmur3_128HashFunction and is pinned here on its published test vectors
(scores_np, its numpy form, on the plain one); batch_delivery_ordered()
extends test_gpu_delivery.batch_delivery with that branch. tests/test_gpu_delivery_oshare.py compares the device with both.
"""
import numpy as np

import test_gpu_delivery as D
from rendezvous_hash import murmur3_128, rendezvous_pick, score, scores_np

NO_MEMBER, ORDERED = D.NO_MEMBER, D.ORDERED


# ------------------------------------------------------------------ the ordered branch of send + BatchDeliveryCall.add
def batch_delivery_ordered(topic_tenant, n_tenants, offsets, ranks, route_of, pick, pub_off, pub_hash, winner=None):
    """batch_delivery with $oshare routes resolved. route_of(rank) -> as batch_delivery's, plus ('R', [(receiverUrl,
    deliverer), ...]) for an $oshare route whose group has members (wire order); ('O', None) stays for a member-less group.
    pub_off / pub_hash: the publisher packs of every topic position. winner(position, rank, publisher) may stand in for
    rendezvous_pick (the numpy scores at scale).
    -> {deliverer: {tenant: [(position, {(rank, member)}, (publisher, ...)), ...]}}: a position's whole pack (publishers ())
    first, then its sub-packs in (rank, member) order, positions in batch order"""
    offsets, ranks = np.asarray(offsets, np.int64), np.asarray(ranks, np.int64)
    keep = np.array([route_of(int(r))[0] != "R" for r in ranks], bool)
    kept = np.concatenate([[0], np.cumsum(keep)])[offsets]   # the CSR without the $oshare routes that are resolved
    whole = D.batch_delivery(topic_tenant, n_tenants, kept, ranks[keep], route_of, pick)
    packs = {}
    for d, pkgs in whole.items():
        for tn, lst in pkgs.items():
            for t, infos in lst:
                packs.setdefault(d, {}).setdefault(tn, []).append(((t, 0, 0, 0), (t, infos, ())))
    for t in range(len(offsets) - 1):
        tenant = int(topic_tenant[t])
        if not 0 <= tenant < n_tenants:
            continue
        pubs = range(int(pub_off[t]), int(pub_off[t + 1]))
        for r in sorted(int(x) for x in ranks[offsets[t]:offsets[t + 1]]):
            kind, members = route_of(r)
            if kind != "R":
                continue
            by_winner = {}                                  # send(): publisher packs grouped by their rendezvous pick
            for p in pubs:
                w = winner(t, r, p) if winner else rendezvous_pick(int(pub_hash[p]), [u for u, _ in members])
                by_winner.setdefault(w, []).append(p)
            for w, ps in by_winner.items():
                d, member = (ORDERED, NO_MEMBER) if w is None else (members[w][1], w)   # no winner: parked, as member-less
                # add(): a fresh TopicMessagePackHolder per sub-pack, so a pack of its own with one MatchInfo
                packs.setdefault(d, {}).setdefault(tenant, []).append(((t, 1, r, member), (t, {(r, member)}, tuple(ps))))
    return {d: {tn: [p for _, p in sorted(lst, key=lambda x: x[0])] for tn, lst in pkgs.items()} for d, pkgs in packs.items()}


# ------------------------------------------------------------------ pinned
GUAVA_VECTORS = [   # (seed, h1, h2, input): Guava's Murmur3Hash128Test
    (0, 0xE34BBC7BBC071B6C, 0x7A433CA9C49A9347, b"The quick brown fox jumps over the lazy dog"),
    (0, 0x629942693E10F867, 0x92DB0B82BAEB5347, b"hell"),
    (1, 0xA78DDFF5ADAE8D10, 0x128900EF20900135, b"hello"),
    (0, 0, 0, b""),
]


def test_murmur3_128_reproduces_guava_vectors():
    for seed, h1, h2, data in GUAVA_VECTORS:
        assert murmur3_128(data, seed) == (h1, h2), data


def test_numpy_scores_equal_the_plain_restatement_at_every_tail_length():
    urls = [("0\0r\0" + "x" * k).encode() for k in range(40)] + ["1\0é你\0\U0001F600d".encode()]
    hashes = [0, -1, -2 ** 31, 2 ** 31 - 1, 12345] * 9
    hashes = hashes[:len(urls)]
    assert scores_np(hashes, urls).tolist() == [score(h, u) for h, u in zip(hashes, urls)]


A, B2, C = b"0\0a\0d1", b"1\0b\0d2", b"0\0c\0d1"


def test_rendezvous_picks_pinned():
    assert [rendezvous_pick(h, [A, B2, C]) for h in (0, -1, -2 ** 31, 2 ** 31 - 1, 7, 8)] == [0, 0, 0, 2, 1, 0]
    assert [rendezvous_pick(h, [C, A]) for h in (0, -1, -2 ** 31, 2 ** 31 - 1, 7, 8)] == [1, 1, 1, 0, 1, 1]
    assert [score(h, A) for h in (0, -1)] == [667015427989259597, 4664953090929987489]
    assert rendezvous_pick(5, [A]) == 0 and rendezvous_pick(5, []) is None


def _route_table():
    """0 -> deliverer a, 1 -> $share(a, b), 5 -> b, 6 -> $oshare(A, B2, C) on deliverers a, b, a, 7 -> member-less group,
    8 -> a second $oshare(C, A) whose members both sit on deliverer a"""
    return {0: ("N", "a"), 1: ("S", ["a", "b"]), 5: ("N", "b"), 6: ("R", [(A, "a"), (B2, "b"), (C, "a")]), 7: ("O", None),
            8: ("R", [(C, "a"), (A, "a")])}


def test_restatement_splits_packs_per_winner_and_keeps_the_rest_whole():
    rows = [[8, 6, 0, 1, 7], [6, 5], [6]]                  # position 1 has no publishers, position 2 is another tenant's
    off, ranks = D.hand_csr(rows)
    pub_off = [0, 6, 6, 8]
    pub_hash = [0, -1, -2 ** 31, 2 ** 31 - 1, 7, 7, 8, 0]   # picks of rank 6: 0 0 0 2 1 1 | 0 0; of rank 8: 1 1 1 0 1 1
    got = batch_delivery_ordered([0, 0, 1], 2, off, ranks, _route_table().__getitem__, lambda t, r: 1, pub_off, pub_hash)
    assert got == {
        # position 0: the whole pack first, then sub-packs by (rank, member); ranks 6 and 8 never share a pack
        "a": {0: [(0, {(0, NO_MEMBER)}, ()), (0, {(6, 0)}, (0, 1, 2)), (0, {(6, 2)}, (3,)), (0, {(8, 0)}, (3,)),
                  (0, {(8, 1)}, (0, 1, 2, 4, 5))],
              1: [(2, {(6, 0)}, (6, 7))]},
        # position 1 has no publishers: no sub-pack for rank 6, its other route still gets the whole pack
        "b": {0: [(0, {(1, 1)}, ()), (0, {(6, 1)}, (4, 5)), (1, {(5, NO_MEMBER)}, ())]},
        ORDERED: {0: [(0, {(7, NO_MEMBER)}, ())]},        # the member-less group stays parked
    }


def test_restatement_without_oshare_routes_is_batch_delivery():
    routes = {r: v for r, v in _route_table().items() if v[0] != "R"}
    rows = [[0, 1, 7], [5]]
    off, ranks = D.hand_csr(rows)
    got = batch_delivery_ordered([0, 1], 2, off, ranks, routes.__getitem__, lambda t, r: 0, [0, 3, 3], [1, 2, 3])
    base = D.batch_delivery([0, 1], 2, off, ranks, routes.__getitem__, lambda t, r: 0)
    assert got == {d: {tn: [p + ((),) for p in lst] for tn, lst in pkgs.items()} for d, pkgs in base.items()}

