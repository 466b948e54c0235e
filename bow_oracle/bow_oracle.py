"""ctypes front-end of the DBoW2 retrieval's oracle (bow_oracle/libdfk_bow_oracle.so).

TEST INFRASTRUCTURE ONLY: tests/ and tools/bench_secondary.py use it as the checker of the dfk_bow_* calls.  A
vocabulary is the dict of deepfactors_b200.aligners.load_dbow2_vocabulary; descriptors are uint8 [N, descriptor_bytes];
a vector is (words int32 ascending, values float64).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfk_bow_oracle.so")
_CSRC = os.path.join(_HERE, "..", "deepfactors_b200", "csrc")


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc, -O2 -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in ("dfk_bow_oracle.c", "Makefile")] + [os.path.join(_CSRC, "dfk_bow_model.h")]
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(_LIB_PATH) for f in srcs):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


_lib = None
_P = C.c_void_p


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.dfkb_voc_create.restype = _P
        L.dfkb_voc_create.argtypes = [C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P]
        L.dfkb_voc_free.argtypes = [_P]
        L.dfkb_transform.restype = C.c_int
        L.dfkb_transform.argtypes = [_P, _P, C.c_int, _P, _P, _P]
        L.dfkb_query.restype = C.c_int
        L.dfkb_query.argtypes = [_P, _P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P]
        L.dfkb_score.restype = C.c_double
        L.dfkb_score.argtypes = [_P, _P, C.c_int, _P, _P, C.c_int]
        L.dfkb_train.restype = _P
        L.dfkb_train.argtypes = [_P, C.c_int64, C.c_int, _P, C.c_int, C.c_int, C.c_int, C.c_uint64]
        L.dfkb_train_nodes.restype = C.c_int
        L.dfkb_train_nodes.argtypes = [_P]
        L.dfkb_train_get.argtypes = [_P, _P, _P, _P, _P]
        L.dfkb_train_free.argtypes = [_P]
        _lib = L
    return _lib


def _a(x, dt):
    return np.ascontiguousarray(np.asarray(x, dt))


class Vocabulary:
    """Steps 1-3 (the tree as listed, children in file order)."""

    def __init__(self, voc: dict):
        self._keep = [_a(voc["node_ids"], np.int32), _a(voc["parent_ids"], np.int32), _a(voc["weights"], np.float64),
                      _a(voc["descriptors"], np.uint8), _a(voc["word_ids"], np.int32), _a(voc["word_nodes"], np.int32)]
        ids, par, wt, desc, wid, wn = self._keep
        self.descriptor_bytes = int(voc["descriptor_bytes"])
        self._p = lib().dfkb_voc_create(len(ids), ids.ctypes.data, par.ctypes.data, wt.ctypes.data, desc.ctypes.data,
                                        self.descriptor_bytes, len(wid), wid.ctypes.data, wn.ctypes.data)
        if not self._p:
            raise MemoryError("bow oracle: out of memory")

    def __del__(self):
        if getattr(self, "_p", None):
            lib().dfkb_voc_free(self._p)
            self._p = None

    def transform(self, descriptors):
        """(feature_words int32 [N] with -1 for a weight not > 0, words int32 [count], values float64 [count])"""
        d = _a(descriptors, np.uint8).reshape(-1, self.descriptor_bytes)
        m = d.shape[0]
        fw = np.zeros(max(m, 1), np.int32)
        w = np.zeros(max(m, 1), np.int32)
        v = np.zeros(max(m, 1), np.float64)
        c = lib().dfkb_transform(self._p, d.ctypes.data, m, fw.ctypes.data, w.ctypes.data, v.ctypes.data)
        return fw[:m], w[:c].copy(), v[:c].copy()


class Database:
    """Steps 4-6 over vectors kept on the host."""

    def __init__(self):
        self.entries = []

    def clear(self):
        self.entries = []

    def __len__(self):
        return len(self.entries)

    def add(self, words, values) -> int:
        self.entries.append((_a(words, np.int32), _a(values, np.float64)))
        return len(self.entries) - 1

    def _flat(self):
        counts = np.array([len(w) for w, _ in self.entries] or [0], np.int32)
        offsets = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.int64)
        ew = np.concatenate([w for w, _ in self.entries] + [np.zeros(1, np.int32)]).astype(np.int32)
        ev = np.concatenate([v for _, v in self.entries] + [np.zeros(1, np.float64)]).astype(np.float64)
        return offsets, counts, ew, ev

    def query(self, words, values, max_results: int, max_id: int = -1):
        """(ids int32, scores float64, count before the cut)"""
        qw, qv = _a(words, np.int32), _a(values, np.float64)
        offsets, counts, ew, ev = self._flat()
        ids = np.zeros(max(max_results, 1), np.int32)
        sc = np.zeros(max(max_results, 1), np.float64)
        c = lib().dfkb_query(qw.ctypes.data, qv.ctypes.data, len(qw), len(self.entries), offsets.ctypes.data,
                             counts.ctypes.data, ew.ctypes.data, ev.ctypes.data, int(max_results), int(max_id),
                             ids.ctypes.data, sc.ctypes.data)
        if c < 0:
            raise MemoryError("bow oracle: out of memory")
        k = min(c, max_results)
        return ids[:k].copy(), sc[:k].copy(), int(c)

    def score(self, entry: int, words, values) -> float:
        aw, av = self.entries[entry]
        return score(aw, av, words, values)


def score(aw, av, bw, bv) -> float:
    """L1Scoring::score(a, b)"""
    aw, av, bw, bv = _a(aw, np.int32), _a(av, np.float64), _a(bw, np.int32), _a(bv, np.float64)
    return float(lib().dfkb_score(aw.ctypes.data, av.ctypes.data, len(aw), bw.ctypes.data, bv.ctypes.data, len(bw)))


def save_order(parent_ids):
    """DBoW2 save's node order from parent ids by id (index id - 1, children as consecutive ascending ids): a stack of
    parents from the root; pop the last, list its children, push each that has children"""
    parent_ids = np.asarray(parent_ids)
    n = len(parent_ids)
    kids = [[] for _ in range(n + 1)]
    for i, p in enumerate(parent_ids):
        kids[int(p)].append(i + 1)
    order, stack = [], [0]
    while stack:
        p = stack.pop()
        for c in kids[p]:
            order.append(c)
            if kids[c]:
                stack.append(c)
    return np.array(order, np.int64), kids


def train(descriptors, image_offsets, k: int, L: int, seed: int):
    """TemplatedVocabulary::create of the block in include/dfk.h, sequential and depth first: (the vocabulary dict of
    load_dbow2_vocabulary in save order, stats dict)"""
    d = _a(descriptors, np.uint8)
    D = d.shape[1]
    off = _a(image_offsets, np.int64)
    p = lib().dfkb_train(d.ctypes.data, d.shape[0], D, off.ctypes.data, len(off) - 1, int(k), int(L),
                         C.c_uint64(int(seed) & (2 ** 64 - 1)))
    if not p:
        raise MemoryError("bow oracle: out of memory")
    try:
        n = lib().dfkb_train_nodes(p)
        par = np.zeros(n, np.int32)
        wt = np.zeros(n, np.float64)
        desc = np.zeros((n, D), np.uint8)
        st = np.zeros(5 + 16, np.int32)
        lib().dfkb_train_get(p, par.ctypes.data, wt.ctypes.data, desc.ctypes.data, st.ctypes.data)
    finally:
        lib().dfkb_train_free(p)
    order, kids = save_order(par)
    leaves = np.array([i for i in range(1, n + 1) if not kids[i]], np.int32)
    voc = dict(k=int(k), L=int(L), weighting=0, scoring=0, descriptor_bytes=D, node_ids=order.astype(np.int32),
               parent_ids=par[order - 1], weights=wt[order - 1], descriptors=desc[order - 1],
               word_ids=np.arange(len(leaves), dtype=np.int32), word_nodes=leaves)
    stats = dict(zip(("num_nodes", "num_words", "max_rounds", "capped_nodes", "empty_clusters"), map(int, st[:5])))
    stats["level_max_rounds"] = [int(v) for v in st[5:]]
    return voc, stats
