"""Descriptor sets, a checker of DBoW2's vocabulary layout and an independent Python transliteration of DBoW2's
TemplatedVocabulary::create (include/dfk.h, the DBoW2 training block) for tests/test_bow_train.py and
tests/test_gpu_bow_train.py.

The transliteration follows HKmeansStep's recursion with Python ints for the random streams and Python floats for
min_dist, as DBoW2 keeps it, so it must agree with the C oracle and the device bit for bit."""
from __future__ import annotations

import math

import numpy as np

M64 = 2 ** 64 - 1


def mix64(z: int) -> int:
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


class Stream:
    def __init__(self, key: int):
        self.s = key & M64

    def next(self) -> int:
        self.s = (self.s + 0x9E3779B97F4A7C15) & M64
        return mix64(self.s)

    def index(self, m: int) -> int:
        return (self.next() * m) >> 64

    def cut(self, dist_sum: float) -> float:
        while True:
            c = (float(self.next() >> 11) * 2.0 ** -53) * float(dist_sum)
            if c != 0.0:
                return c


def child_key(key: int, i: int) -> int:
    return mix64((key + (i + 1) * 0xD1B54A32D192ED03) & M64)


_POP = np.array([bin(i).count("1") for i in range(256)], np.int64)


def distances(x: np.ndarray, c: np.ndarray) -> np.ndarray:
    """popcount(x_i ^ c) for rows x [n, D] against one descriptor c [D]"""
    return _POP[np.bitwise_xor(x, c[None, :])].sum(axis=1)


def mean(rows: np.ndarray, D: int) -> np.ndarray:
    """FBrisk::meanValue: bit set iff its count > m / 2 (integer division)"""
    if len(rows) == 0:
        return np.zeros(D, np.uint8)
    counts = np.unpackbits(rows, axis=1, bitorder="little").sum(axis=0)
    return np.packbits((counts > len(rows) // 2).astype(np.uint8), bitorder="little")


def py_train(desc: np.ndarray, offsets, k: int, L: int, seed: int, max_rounds: int = 1000):
    """(vocabulary dict in save order, stats dict)"""
    desc = np.ascontiguousarray(desc, np.uint8)
    D = desc.shape[1]
    parent, descs, keys, kids = [-1], [np.zeros(D, np.uint8)], [seed & M64], [[]]
    stats = dict(max_rounds=0, capped_nodes=0, empty_clusters=0, level_max_rounds=[0] * 16)

    def step(pid: int, idx: np.ndarray, level: int):
        m = len(idx)
        if m == 0:
            return
        X = desc[idx]
        if m <= k:
            clusters = [X[i].copy() for i in range(m)]
            assoc = np.arange(m)
        else:
            s = Stream(keys[pid])
            clusters = [X[s.index(m)].copy()]
            min_dists = [float(d) for d in distances(X, clusters[0])]
            while len(clusters) < k:
                dl = distances(X, clusters[-1])
                for i in range(m):
                    if min_dists[i] > 0 and dl[i] < min_dists[i]:
                        min_dists[i] = float(dl[i])
                dist_sum = 0.0
                for v in min_dists:
                    dist_sum += v
                if not dist_sum > 0:
                    break
                cut = s.cut(dist_sum)
                up, i = 0.0, 0
                while i < m:
                    up += min_dists[i]
                    if up >= cut:
                        break
                    i += 1
                clusters.append(X[min(i, m - 1)].copy())
            rounds, last = 0, None
            while True:
                if last is not None:
                    clusters = [mean(X[assoc == c], D) for c in range(len(clusters))]
                dm = np.stack([distances(X, c) for c in clusters], axis=1)
                new = np.argmin(dm, axis=1)  # the first of equal distances: strict < in cluster order
                rounds += 1
                if last is None:
                    last = assoc = new
                    continue
                done = np.array_equal(new, assoc)
                assoc = new
                if done:
                    break
                if rounds == max_rounds:
                    stats["capped_nodes"] += 1
                    break
            stats["max_rounds"] = max(stats["max_rounds"], rounds)
            stats["level_max_rounds"][level - 1] = max(stats["level_max_rounds"][level - 1], rounds)
            stats["empty_clusters"] += sum(int((assoc == c).sum() == 0) for c in range(len(clusters)))
        first = len(parent)
        for c, cl in enumerate(clusters):
            parent.append(pid)
            descs.append(cl)
            keys.append(child_key(keys[pid], c))
            kids.append([])
            kids[pid].append(first + c)
        if level < L:
            for c in range(len(clusters)):
                g = idx[assoc == c]
                if len(g) > 1:
                    step(first + c, g, level + 1)

    step(0, np.arange(len(desc)), 1)
    n = len(parent) - 1
    leaves = [i for i in range(1, n + 1) if not kids[i]]
    word_of = {nid: j for j, nid in enumerate(leaves)}
    ni = [0] * len(leaves)
    off = [int(o) for o in offsets]
    for img in range(len(off) - 1):
        seen = set()
        for f in range(off[img], off[img + 1]):
            nid = 0
            while kids[nid]:
                dd = [int(_POP[np.bitwise_xor(desc[f], descs[c])].sum()) for c in kids[nid]]
                nid = kids[nid][int(np.argmin(dd))]
            seen.add(word_of[nid])
        for w in seen:
            ni[w] += 1
    weight = np.zeros(n + 1)
    for nid in leaves:
        c = ni[word_of[nid]]
        weight[nid] = math.log(float(len(off) - 1) / float(c)) if c > 0 else 0.0
    order, stack = [], [0]
    while stack:
        p = stack.pop()
        for c in kids[p]:
            order.append(c)
            if kids[c]:
                stack.append(c)
    order = np.array(order, np.int64)
    voc = dict(k=k, L=L, weighting=0, scoring=0, descriptor_bytes=D, node_ids=order.astype(np.int32),
               parent_ids=np.array(parent, np.int32)[order], weights=weight[order],
               descriptors=np.stack(descs)[order].astype(np.uint8), word_ids=np.arange(len(leaves), dtype=np.int32),
               word_nodes=np.array(leaves, np.int32))
    stats.update(num_nodes=n, num_words=len(leaves))
    return voc, stats


# ---------------------------------------------------------------------------------------------------- the layout
def check_dbow2_layout(voc: dict) -> None:
    """What a vocabulary DBoW2's create and save wrote looks like: ids 1..N numbered depth first (a node's children one
    block of consecutive ids, given when the node is visited), nodes listed in save's order, words = the leaves in
    ascending id with word ids 0..W-1 in order, inner nodes weighing 0"""
    ids = np.asarray(voc["node_ids"], np.int64)
    par = np.asarray(voc["parent_ids"], np.int64)
    n = len(ids)
    assert sorted(ids.tolist()) == list(range(1, n + 1))
    kids = {0: []}
    for i, p in zip(ids, par):
        kids.setdefault(int(p), []).append(int(i))
        kids.setdefault(int(i), [])
    for p, c in kids.items():
        assert c == list(range(c[0], c[0] + len(c))) if c else True, f"children of {p} are not consecutive"
    # depth-first numbering
    nxt, expect, stack = 1, {}, [0]

    def visit(p):
        nonlocal nxt
        for c in kids[p]:
            expect[c] = nxt
            nxt += 1
        for c in kids[p]:
            if kids[c]:
                visit(c)

    visit(0)
    assert all(expect[i] == i for i in expect), "ids are not DBoW2's depth-first numbering"
    # save order
    order = []
    while stack:
        p = stack.pop()
        for c in kids[p]:
            order.append(c)
            if kids[c]:
                stack.append(c)
    assert order == ids.tolist(), "nodes are not in save's order"
    leaves = sorted(i for i in kids if i and not kids[i])
    assert np.asarray(voc["word_ids"]).tolist() == list(range(len(leaves)))
    assert np.asarray(voc["word_nodes"]).tolist() == leaves
    w = dict(zip(ids.tolist(), np.asarray(voc["weights"]).tolist()))
    assert all(w[i] == 0.0 for i in kids if i and kids[i]), "an inner node weighs more than 0"


# ------------------------------------------------------------------------------------------------- descriptor sets
def planted(n: int, D: int, k: int, depth: int, flips: int, seed: int) -> np.ndarray:
    """n descriptors from a seeded planted hierarchy: k random centres, each with k children made by flipping `flips`
    bits, `depth` levels deep; every descriptor is a random leaf with `flips` more bits flipped"""
    rng = np.random.default_rng(seed)
    cents = rng.integers(0, 256, (k, D), np.uint8)
    for _ in range(depth - 1):
        cents = np.repeat(cents, k, axis=0)
        cents = _flip(cents, flips, rng)
    return _flip(cents[rng.integers(0, len(cents), n)], flips, rng)


def _flip(x: np.ndarray, flips: int, rng) -> np.ndarray:
    bits = np.unpackbits(x, axis=1)
    pos = rng.integers(0, bits.shape[1], (len(x), flips))
    np.bitwise_xor.at(bits, (np.arange(len(x))[:, None], pos), 1)
    return np.packbits(bits, axis=1)


def few_distinct(n: int, D: int, distinct: int, seed: int) -> np.ndarray:
    """n descriptors drawn from `distinct` random ones: seeding stops early when distinct < k"""
    rng = np.random.default_rng(seed)
    base = rng.integers(0, 256, (distinct, D), np.uint8)
    return base[rng.integers(0, distinct, n)]


def one_bit(n: int, D: int, seed: int) -> np.ndarray:
    """descriptors with one set bit each: every two distinct ones are at distance 2, exact ties everywhere"""
    rng = np.random.default_rng(seed)
    bits = np.zeros((n, 8 * D), np.uint8)
    bits[np.arange(n), rng.integers(0, 8 * D, n)] = 1
    return np.packbits(bits, axis=1)


def offsets_for(n: int, images: int, seed: int, empty: int = 0) -> np.ndarray:
    """image offsets of n descriptors in `images` images, `empty` of them empty"""
    rng = np.random.default_rng(seed + 1)
    cuts = np.sort(rng.integers(0, n + 1, images - 1))
    off = np.concatenate([[0], cuts, [n]]).astype(np.int64)
    for j in rng.choice(images - 1, min(empty, images - 1), replace=False):
        off[j + 1] = off[j]  # image j empty: its rows go to the next image (the last image is never emptied)
    return np.maximum.accumulate(off)


def make(kind: str, n: int, D: int, k: int, seed: int):
    if kind == "planted":
        return planted(n, D, k, 3, 6, seed)
    if kind == "random":
        return np.random.default_rng(seed).integers(0, 256, (n, D), np.uint8)
    if kind == "few":
        return few_distinct(n, D, max(1, k // 2), seed)
    if kind == "one_bit":
        return one_bit(n, D, seed)
    raise ValueError(kind)


# (kind, N, D, k, L, seed, images, empty images)
CASES = [
    ("random", 1, 32, 2, 1, 0, 1, 0),
    ("random", 2, 32, 2, 2, 1, 2, 1),
    ("random", 3, 48, 3, 2, 2, 2, 0),
    ("random", 9, 64, 9, 2, 3, 3, 1),
    ("random", 10, 32, 9, 2, 4, 3, 0),
    ("random", 32, 32, 32, 2, 5, 4, 0),
    ("random", 33, 64, 32, 2, 6, 4, 1),
    ("planted", 400, 32, 3, 4, 7, 8, 2),
    ("planted", 1500, 48, 9, 2, 8, 12, 0),
    ("planted", 3000, 32, 9, 4, 9, 20, 3),
    ("planted", 700, 64, 32, 2, 10, 6, 0),
    ("planted", 600, 32, 2, 4, 11, 5, 1),
    ("few", 500, 32, 9, 2, 12, 5, 0),
    ("few", 300, 48, 32, 4, 13, 4, 1),
    ("one_bit", 800, 32, 9, 4, 14, 6, 0),
    ("one_bit", 400, 64, 3, 4, 15, 4, 1),
    ("random", 2000, 32, 32, 1, 16, 10, 0),
]


def case_data(case):
    kind, n, D, k, L, seed, images, empty = case
    return make(kind, n, D, k, seed), offsets_for(n, images, seed, empty), k, L, seed


def case_id(case) -> str:
    kind, n, D, k, L, seed, _, _ = case
    return f"{kind}-N{n}-D{D}-k{k}-L{L}-s{seed}"
