"""Vocabularies, descriptor sets and an independent Python transliteration of DBoW2's retrieval (include/dfk.h, DBoW2
block, steps 1-6) for tests/test_bow.py and tests/test_gpu_bow.py.

The transliteration uses dicts for DBoW2's std::map and Python floats (IEEE doubles) in the specification's operation
order, so it must agree with the C oracle and the device bit for bit."""
from __future__ import annotations

import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL_VOC = os.path.join(ROOT, "tests", "golden", "dbow2_small_voc.yml.gz")


def small_voc() -> dict:
    from deepfactors_b200.aligners import load_dbow2_vocabulary
    return load_dbow2_vocabulary(SMALL_VOC)


def synthetic_voc(seed: int, k: int, L: int, D: int, zero_frac: float = 0.1, ties: bool = False,
                  shuffle: bool = True) -> dict:
    """A random tree of depth <= L with 1..k children per node, listed in a shuffled file order with shuffled ids.
    ties: every node's second child copies its first child's descriptor (exact ties between children)."""
    rng = np.random.default_rng(seed)
    nodes = []  # (parent index or -1 for the root, depth)
    frontier = [(-1, 0)]
    while frontier:
        p, d = frontier.pop()
        if d == L:
            continue
        nc = int(rng.integers(2 if d == 0 else 1, k + 1))
        if d > 0 and rng.random() < 0.15:
            nc = 0  # an early leaf
        for _ in range(nc):
            nodes.append((p, d + 1))
            frontier.append((len(nodes) - 1, d + 1))
    N = len(nodes)
    order = rng.permutation(N) if shuffle else np.arange(N)
    ids = rng.permutation(N) + 1 if shuffle else np.arange(1, N + 1)
    desc = rng.integers(0, 256, (N, D), dtype=np.uint8)
    has_child = np.zeros(N, bool)
    for p, _ in nodes:
        if p >= 0:
            has_child[p] = True
    weights = np.where(has_child, 0.0, rng.uniform(0.1, 3.0, N))
    leaves = np.nonzero(~has_child)[0]
    weights[leaves[rng.random(len(leaves)) < zero_frac]] = 0.0
    # listed in file order: the children order of a parent is the order its children appear in the file
    node_ids = ids[order]
    parent_ids = np.array([0 if nodes[i][0] < 0 else ids[nodes[i][0]] for i in order], np.int32)
    word_perm = rng.permutation(len(leaves))
    if ties:  # a parent's second child in file order copies its first
        seen = {}
        for i in order:
            p = nodes[i][0]
            if seen.get(p, 0) == 0:
                seen[p] = (i,)
            elif len(seen[p]) == 1:
                desc[i] = desc[seen[p][0]]
                seen[p] = (seen[p][0], i)
    return dict(k=k, L=L, weighting=0, scoring=0, descriptor_bytes=D, node_ids=node_ids.astype(np.int32),
                parent_ids=parent_ids, weights=weights[order].astype(np.float64), descriptors=desc[order],
                word_ids=np.arange(len(leaves), dtype=np.int32),
                word_nodes=ids[leaves[word_perm]].astype(np.int32))


def near_node_descriptors(voc: dict, seed: int, n: int, max_flips: int = 40) -> np.ndarray:
    """n descriptors, each a random node's descriptor with 0..max_flips random bits flipped"""
    rng = np.random.default_rng(seed)
    d = voc["descriptors"][rng.integers(0, len(voc["node_ids"]), n)].copy()
    bits = d.shape[1] * 8
    for r in range(n):
        for b in rng.choice(bits, int(rng.integers(0, max_flips + 1)), replace=False):
            d[r, b // 8] ^= np.uint8(1 << (b % 8))
    return d


class PyVocabulary:
    """Steps 1-3 with dicts: children lists in file order, descent by strict < in children order."""

    def __init__(self, voc: dict):
        self.children = {0: []}
        self.desc, self.weight, self.word = {}, {}, {}
        for nid, pid, w, d in zip(voc["node_ids"], voc["parent_ids"], voc["weights"], voc["descriptors"]):
            nid, pid = int(nid), int(pid)
            self.children.setdefault(pid, []).append(nid)
            self.children.setdefault(nid, [])
            self.desc[nid] = int.from_bytes(bytes(d), "little")
            self.weight[nid] = float(w)
        for wid, nid in zip(voc["word_ids"], voc["word_nodes"]):
            self.word[int(nid)] = int(wid)

    def word_of(self, f: bytes):
        x = int.from_bytes(bytes(f), "little")
        nid = 0
        while True:
            ch = self.children[nid]
            best = ch[0]
            best_d = (x ^ self.desc[best]).bit_count()
            for c in ch[1:]:
                d = (x ^ self.desc[c]).bit_count()
                if d < best_d:
                    best, best_d = c, d
            nid = best
            if not self.children[nid]:
                return self.word[nid], self.weight[nid]

    def transform(self, descriptors):
        v, fw = {}, []
        for f in np.asarray(descriptors, np.uint8):
            w, wt = self.word_of(f)
            if wt > 0:
                fw.append(w)
                v[w] = v[w] + wt if w in v else wt
            else:
                fw.append(-1)
        norm = 0.0
        for w in sorted(v):
            norm += abs(v[w])
        if norm > 0:
            for w in v:
                v[w] = v[w] / norm
        return fw, v


def py_query(entries: list, q: dict, max_results: int, max_id: int = -1):
    """queryL1: ([(entry, Score)], count before the cut), equal sums by ascending entry"""
    pairs = {}
    for w in sorted(q):
        for e, d in enumerate(entries):
            if w in d and (e < max_id or max_id == -1):
                t = abs(q[w] - d[w]) - abs(q[w]) - abs(d[w])
                pairs[e] = pairs[e] + t if e in pairs else t
    ret = sorted(pairs.items(), key=lambda p: (p[1], p[0]))
    count = len(ret)
    if max_results > 0:
        ret = ret[:max_results]
    return [(e, -s / 2.0) for e, s in ret], count


def py_score(a: dict, b: dict) -> float:
    """L1Scoring::score(a, b): vi from a, wi from b"""
    s = 0.0
    for w in sorted(a):
        if w in b:
            s += abs(a[w] - b[w]) - abs(a[w]) - abs(b[w])
    return -s / 2.0


def as_arrays(v: dict):
    ws = sorted(v)
    return np.array(ws, np.int32), np.array([v[w] for w in ws], np.float64)


def bits(x) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(x, np.float64)).view(np.int64)
