"""The dfk_bow_* calls on the device against the CPU oracle (bow_oracle/), bit for bit:
- transform of mixed batches (0, 1, 500 and 8192 descriptors) with 32-, 48- (the reference's small_voc) and 64-byte
  vocabularies: the word of every descriptor, the vector's words and value bits, its count;
- databases of 1, 100 and 5000 entries built from transform outputs with no synchronisation in between; queries with
  max_results 1, 3 and above the count, max_id -1 / 0 / middle; the score of every query against several entries;
  the same after clear;
- an item gives the same output alone, first in a batch and in a reversed batch, and two runs are equal;
- every validation rule is rejected, the call writes nothing (sentinels stay) and the message names the item and
  field; other weighting or scoring types are DFK_ERR_UNSUPPORTED."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import bow_cases as bc
from bow_oracle import bow_oracle as bo
from deepfactors_b200 import _lib
from deepfactors_b200 import aligners as A

pytestmark = pytest.mark.gpu

VOCS = {48: bc.small_voc, 32: lambda: bc.synthetic_voc(32, k=8, L=4, D=32),
        64: lambda: bc.synthetic_voc(64, k=10, L=3, D=64, ties=True)}


@pytest.fixture(scope="module", params=[32, 48, 64])
def voc(request):
    v = VOCS[request.param]()
    return v, A.BowVocabulary(v), bo.Vocabulary(v)


def _sets(v, seed, sizes):
    return [bc.near_node_descriptors(v, seed + i, n) for i, n in enumerate(sizes)]


def _dev(sets):
    return [torch.from_numpy(np.ascontiguousarray(s)).cuda() for s in sets]


def _host(batch, i):
    o, c = int(batch.offsets[i]), int(batch.counts[i].item())
    return batch.words[o:o + c].cpu().numpy(), batch.values[o:o + c].cpu().numpy()


def _check_item(batch, i, orc_out, num):
    fw, w, v = orc_out
    o = int(batch.offsets[i])
    assert np.array_equal(batch.feature_words[o:o + num].cpu().numpy(), fw), i
    gw, gv = _host(batch, i)
    assert np.array_equal(gw, w) and np.array_equal(bc.bits(gv), bc.bits(v)), i


def test_transform_mixed_batch(voc):
    v, gv, orc = voc
    sizes = [0, 1, 500, 8192, 37]
    sets = _sets(v, 100, sizes)
    batch = A.BowTransformBatch(gv, _dev(sets), capacities=[n + 3 for n in sizes])
    for i, s in enumerate(sets):
        _check_item(batch, i, orc.transform(s), len(s))


def test_item_independent_of_batch_and_repeatable(voc):
    v, gv, orc = voc
    sets = _sets(v, 200, [300, 0, 700, 5])
    dev = _dev(sets)
    ref = A.BowTransformBatch(gv, dev)
    for order in ([2], [2, 0, 1, 3], [3, 2, 1, 0]):
        b = A.BowTransformBatch(gv, [dev[i] for i in order])
        for j, i in enumerate(order):
            a, c = _host(ref, i), _host(b, j)
            assert np.array_equal(a[0], c[0]) and np.array_equal(bc.bits(a[1]), bc.bits(c[1]))
    again = A.BowTransformBatch(gv, dev)
    assert torch.equal(ref.words, again.words) and torch.equal(ref.values.view(torch.int64),
                                                               again.values.view(torch.int64))


@pytest.mark.parametrize("entries", [1, 100, 5000])
def test_database_query_and_score(voc, entries):
    v, gv, orc = voc
    rng = np.random.default_rng(entries)
    # a few distinct images, repeated so that equal sums occur, transformed in batches and added with no read-back
    base = _sets(v, 300, [int(rng.integers(1, 120)) for _ in range(min(entries, 40))])
    pick = [int(rng.integers(0, len(base))) for _ in range(entries)]
    db, odb = A.BowDatabase(gv), bo.Database()
    dev = _dev(base)
    for s in range(0, entries, 1000):
        idx = pick[s:s + 1000]
        b = A.BowTransformBatch(gv, [dev[i] for i in idx])
        assert db.add(b.vectors()) == s
    assert len(db) == entries
    oracle_vecs = [orc.transform(s)[1:] for s in base]
    for i in pick:
        odb.add(*oracle_vecs[i])
    qsets = _sets(v, 400, [200, 1, 0, 60])
    qb = A.BowTransformBatch(gv, _dev(qsets))
    qv = qb.vectors()
    qo = [orc.transform(s)[1:] for s in qsets]
    for mr in (1, 3, entries + 5):
        for mi in (-1, 0, entries // 2):
            res = db.query(qv, mr, mi)
            got = res.results()
            counts = res.counts.cpu().numpy()
            for k, (w, val) in enumerate(qo):
                ids, sc, c = odb.query(w, val, mr, mi)
                assert counts[k] == c
                assert [e for e, _ in got[k]] == ids.tolist()
                assert np.array_equal(bc.bits([s for _, s in got[k]]), bc.bits(sc))
    ents = [0, entries // 2, entries - 1]
    sc = db.score([e for e in ents for _ in qv], [q for _ in ents for q in qv]).cpu().numpy()
    want = [odb.score(e, *qo[k]) for e in ents for k in range(len(qv))]
    assert np.array_equal(bc.bits(sc), bc.bits(want))
    # after clear: empty, then a fresh entry is entry 0
    db.clear()
    assert len(db) == 0
    res = db.query(qv, 3)
    assert res.counts.cpu().tolist() == [0] * len(qv)
    assert db.add([qv[0]]) == 0
    got = db.query([qv[0]], 3).results()[0]
    o2 = bo.Database()
    o2.add(*qo[0])
    ids, scs, c = o2.query(*qo[0], 3)
    assert [e for e, _ in got] == ids.tolist() and np.array_equal(bc.bits([s for _, s in got]), bc.bits(scs))


def test_small_voc_retrieves_the_same_place():
    """a query made of an entry's descriptors with a few bits flipped finds that entry first"""
    v = bc.small_voc()
    gv = A.BowVocabulary(v)
    places = _sets(v, 500, [400] * 6)
    noisy = []
    rng = np.random.default_rng(1)
    for p in places:
        q = p.copy()
        m = rng.random(q.shape) < 0.02
        q[m] ^= np.uint8(1 << int(rng.integers(0, 8)))
        noisy.append(q)
    db = A.BowDatabase(gv)
    db.add(A.BowTransformBatch(gv, _dev(places)).vectors())
    res = db.query(A.BowTransformBatch(gv, _dev(noisy)).vectors(), 2).results()
    for k, r in enumerate(res):
        print(f"query {k}: top {r[0]}")
        assert r[0][0] == k


# ------------------------------------------------------------------------------------------- rejected arguments
def _voc_desc(v, **over):
    v = dict(v, **over)
    keep = {k: np.ascontiguousarray(v[k], dt) for k, dt in
            (("node_ids", np.int32), ("parent_ids", np.int32), ("weights", np.float64), ("descriptors", np.uint8),
             ("word_ids", np.int32), ("word_nodes", np.int32))}
    d = _lib.DfkBowVocabularyDesc(v["k"], v["L"], v["weighting"], v["scoring"], v["descriptor_bytes"],
                                  v.get("num_nodes", len(keep["node_ids"])), keep["node_ids"].ctypes.data,
                                  keep["parent_ids"].ctypes.data, keep["weights"].ctypes.data,
                                  keep["descriptors"].ctypes.data, v.get("num_words", len(keep["word_ids"])),
                                  keep["word_ids"].ctypes.data, keep["word_nodes"].ctypes.data)
    return d, keep


def test_vocabulary_validation():
    base = bc.synthetic_voc(3, k=4, L=3, D=32)
    hd = A._Handle()
    L = _lib.lib()
    N = len(base["node_ids"])
    ids, par, wn = base["node_ids"], base["parent_ids"], base["word_nodes"]
    leaf = int(wn[0])
    internal = int(par[par > 0][0])
    li = int(np.nonzero(ids == leaf)[0][0])
    cases = {
        "weighting": (dict(weighting=1), _lib.DFK_ERR_UNSUPPORTED),
        "scoring": (dict(scoring=2), _lib.DFK_ERR_UNSUPPORTED),
        "k not in": (dict(k=33), _lib.DFK_ERR_INVALID_ARG),
        "L not in": (dict(L=17), _lib.DFK_ERR_INVALID_ARG),
        "descriptor_bytes": (dict(descriptor_bytes=40), _lib.DFK_ERR_INVALID_ARG),
        "num_nodes": (dict(num_nodes=0), _lib.DFK_ERR_INVALID_ARG),
        "repeated": (dict(node_ids=np.where(ids == ids[1], ids[0], ids)), _lib.DFK_ERR_INVALID_ARG),
        "not in [1, N]": (dict(node_ids=np.where(ids == ids[1], N + 5, ids)), _lib.DFK_ERR_INVALID_ARG),
        "does not exist": (dict(parent_ids=np.where(np.arange(N) == 2, N + 7, par)), _lib.DFK_ERR_INVALID_ARG),
        "more than k children": (dict(k=1), _lib.DFK_ERR_INVALID_ARG),
        "depth > L": (dict(L=1), _lib.DFK_ERR_INVALID_ARG),
        "weight not finite": (dict(weights=np.where(np.arange(N) == li, np.nan, base["weights"])),
                              _lib.DFK_ERR_INVALID_ARG),
        "weight not finite ": (dict(weights=np.where(np.arange(N) == li, -1.0, base["weights"])),
                               _lib.DFK_ERR_INVALID_ARG),
        "wordId repeated": (dict(word_ids=np.where(np.arange(len(wn)) == 1, 0, base["word_ids"])),
                            _lib.DFK_ERR_INVALID_ARG),
        "wordId not in": (dict(word_ids=np.where(np.arange(len(wn)) == 1, 10 ** 6, base["word_ids"])),
                          _lib.DFK_ERR_INVALID_ARG),
        "not a leaf": (dict(word_nodes=np.where(np.arange(len(wn)) == 0, internal, wn)), _lib.DFK_ERR_INVALID_ARG),
        "a leaf without a word": (dict(word_ids=base["word_ids"][1:] - 1 * (base["word_ids"][1:] > 0),
                                       word_nodes=wn[1:]), _lib.DFK_ERR_INVALID_ARG),
    }
    # a cycle: two leaves each the other's parent, cut off from the root
    i0, i1 = [int(i) for i in np.nonzero(~np.isin(ids, par))[0][:2]]
    cyc = par.copy()
    cyc[i0], cyc[i1] = ids[i1], ids[i0]
    cases["not reachable"] = (dict(parent_ids=cyc), _lib.DFK_ERR_INVALID_ARG)
    for what, (over, want) in cases.items():
        d, keep = _voc_desc(base, **over)
        out = C.c_void_p(12345)
        st = L.dfk_bow_vocabulary_create(hd.h, C.byref(d), C.byref(out))
        msg = L.dfk_last_error(hd.h).decode()
        print(what, "->", msg)
        assert st == want, (what, st, msg)
        assert not out.value
        assert what.strip() in msg, (what, msg)
        where = {"repeated": "node 1:", "not in [1, N]": "node 1:", "does not exist": "node 2:",
                 "weight not finite": f"node {li}:", "wordId repeated": "word 1:", "wordId not in": "word 1:",
                 "not a leaf": "word 0:", "not reachable": f"node {i0}:",
                 "more than k children": "nodeId ", "depth > L": "node ", "a leaf without a word": "node "}.get(
                     what.strip())
        if where:
            assert where in msg, (what, where, msg)  # the message names the node or word
    d, keep = _voc_desc(base)
    out = C.c_void_p()
    assert L.dfk_bow_vocabulary_create(hd.h, C.byref(d), C.byref(out)) == _lib.DFK_OK
    L.dfk_bow_vocabulary_destroy(hd.h, out)


def test_call_validation_writes_nothing():
    v = bc.synthetic_voc(4, k=6, L=3, D=32)
    gv = A.BowVocabulary(v)
    hd, L = gv._hd, _lib.lib()
    hd.use_torch_stream()
    sets = _dev(_sets(v, 600, [50, 60]))
    words = torch.full((200,), -7, dtype=torch.int32, device="cuda")
    values = torch.full((200,), -7.0, dtype=torch.float64, device="cuda")
    counts = torch.full((2,), -7, dtype=torch.int32, device="cuda")

    def fs(t, D=32, num=None):
        return _lib.DfkFeatureSet(None, t.data_ptr(), t.shape[0] if num is None else num, D)

    bad = {
        "descriptor_bytes": ([fs(sets[0]), fs(sets[1], D=64)], [50, 60]),
        "num not in": ([fs(sets[0]), fs(sets[1], num=9000)], [50, 9000]),
        "capacity < num": ([fs(sets[0]), fs(sets[1])], [50, 10]),
        "16-byte aligned": ([fs(sets[0]), _lib.DfkFeatureSet(None, sets[1].data_ptr() + 4, 20, 32)], [50, 60]),
    }
    for what, (items, caps) in bad.items():
        arr = (_lib.DfkFeatureSet * 2)(*items)
        ca = (C.c_int32 * 2)(*caps)
        st = L.dfk_bow_transform_batch(hd.h, gv._p, arr, ca, 2, C.c_void_p(words.data_ptr()),
                                       C.c_void_p(values.data_ptr()), C.c_void_p(counts.data_ptr()), None)
        msg = L.dfk_last_error(hd.h).decode()
        assert st == _lib.DFK_ERR_INVALID_ARG and what in msg and "item 1" in msg, (what, msg)
    torch.cuda.synchronize()
    assert (words == -7).all() and (values == -7.0).all() and (counts == -7).all()
    # database: add, query and score with bad arguments add and write nothing
    b = A.BowTransformBatch(gv, sets)
    db = A.BowDatabase(gv)
    db.add(b.vectors())
    vec = b.vectors()[0].to_c()
    badvec = _lib.DfkBowVector(vec.words, vec.values + 4, vec.count, vec.capacity)
    st = L.dfk_bow_database_add(hd.h, db._p, (_lib.DfkBowVector * 2)(vec, badvec), 2, None)
    assert st == _lib.DFK_ERR_INVALID_ARG and "vector 1" in L.dfk_last_error(hd.h).decode()
    assert len(db) == 2
    ids = torch.full((10,), -7, dtype=torch.int32, device="cuda")
    scs = torch.full((10,), -7.0, dtype=torch.float64, device="cuda")
    qcounts = torch.full((2,), -7, dtype=torch.int32, device="cuda")
    for what, q2 in (("max_results < 1", _lib.DfkBowQuery(vec, 0, -1)), ("max_id < -1", _lib.DfkBowQuery(vec, 3, -2)),
                     ("vector", _lib.DfkBowQuery(badvec, 3, -1))):
        st = L.dfk_bow_database_query_batch(hd.h, db._p, (_lib.DfkBowQuery * 2)(_lib.DfkBowQuery(vec, 3, -1), q2), 2,
                                            C.c_void_p(ids.data_ptr()), C.c_void_p(scs.data_ptr()),
                                            C.c_void_p(qcounts.data_ptr()))
        msg = L.dfk_last_error(hd.h).decode()
        assert st == _lib.DFK_ERR_INVALID_ARG and what in msg and "query 1" in msg, (what, msg)
    for what, it in (("entry not in", _lib.DfkBowScoreItem(2, vec)), ("vector", _lib.DfkBowScoreItem(0, badvec))):
        st = L.dfk_bow_score_batch(hd.h, db._p, (_lib.DfkBowScoreItem * 2)(_lib.DfkBowScoreItem(0, vec), it), 2,
                                   C.c_void_p(scs.data_ptr()))
        msg = L.dfk_last_error(hd.h).decode()
        assert st == _lib.DFK_ERR_INVALID_ARG and what in msg and "item 1" in msg, (what, msg)
    torch.cuda.synchronize()
    assert (ids == -7).all() and (scs == -7.0).all() and (qcounts == -7).all()


# ------------------------------------------------------------------------------------------- more coverage
def _orb_voc():
    z = np.load(os.path.join(bc.ROOT, "tests", "golden", "bow_orb.npz"))
    voc = dict(k=int(z["voc_k"]), L=int(z["voc_L"]), weighting=0, scoring=0, descriptor_bytes=32,
               **{k: z["voc_" + k] for k in ("node_ids", "parent_ids", "weights", "descriptors", "word_ids",
                                             "word_nodes")})
    return z, voc


def test_device_orb_places_retrieve_their_partner():
    """device ORB of the reference's four test images -> transform of the detector's output slices -> database
    {0, 1047} -> queries {25, 1052}, against the oracle on the same descriptors read back; each query's partner (the
    other view of its place) is expected first"""
    z, voc = _orb_voc()
    t = np.load(os.path.join(bc.ROOT, "tests", "golden", "testimg.npz"))
    gv, ov = A.BowVocabulary(voc), bo.Vocabulary(voc)
    names = ["0", "1047", "25", "1052"]
    imgs = [z["gray_0"], t["gray_1047"], z["gray_25"], t["gray_1052"]]
    orb = A.OrbDetectBatch(gv, [torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in imgs])
    feats = orb.features()  # views of the detector's rows at its capacity offsets
    b = A.BowTransformBatch(gv, feats)
    vecs = b.vectors()
    db, odb = A.BowDatabase(gv), bo.Database()
    db.add(vecs[:2])
    host = [ov.transform(f.descriptors.cpu().numpy()) for f in feats]
    for i, f in enumerate(feats):
        _check_item(b, i, host[i], int(f.descriptors.shape[0]))
    for i in (0, 1):
        odb.add(*host[i][1:])
    res = db.query(vecs[2:], 2).results()
    for k, q in enumerate((2, 3)):
        ids, sc, c = odb.query(*host[q][1:], 2)
        assert [e for e, _ in res[k]] == ids.tolist()
        assert np.array_equal(bc.bits([s for _, s in res[k]]), bc.bits(sc))
        print(f"query {names[q]}: top {names[res[k][0][0]]} (Score {res[k][0][1]:.4f}), "
              f"then {names[res[k][1][0]]} ({res[k][1][1]:.4f})")
        assert res[k][0][0] == k, "the other view of the place is expected first"


def test_wide_nodes_and_full_shared_memory_query():
    """a vocabulary whose nodes have 32 children (every lane of the argmin active) and a query vector of capacity
    DFK_MATCH_MAX_QUERIES (96 KB of shared memory in the sums kernel)"""
    rng = np.random.default_rng(3)
    N1, k = 32, 32
    root = np.arange(1, N1 + 1)
    kids = np.arange(N1 + 1, N1 + 1 + N1 * k)
    ids = np.concatenate([root, kids]).astype(np.int32)
    par = np.concatenate([np.zeros(N1), np.repeat(root, k)]).astype(np.int32)
    desc = rng.integers(0, 256, (len(ids), 32), np.uint8)
    desc[N1 + 5] = desc[N1 + 4]  # a tie inside one node's children
    w = np.concatenate([np.zeros(N1), rng.uniform(0.1, 3, N1 * k)])
    voc = dict(k=32, L=2, weighting=0, scoring=0, descriptor_bytes=32, node_ids=ids, parent_ids=par, weights=w,
               descriptors=desc, word_ids=np.arange(N1 * k, dtype=np.int32), word_nodes=kids.astype(np.int32))
    gv, ov = A.BowVocabulary(voc), bo.Vocabulary(voc)
    sets = _sets(voc, 900, [8192, 700, 300])
    b = A.BowTransformBatch(gv, _dev(sets))
    host = [ov.transform(s) for s in sets]
    for i, s in enumerate(sets):
        _check_item(b, i, host[i], len(s))
    assert int(b.counts[0].item()) > 900  # most of the 1024 words in the big query
    db, odb = A.BowDatabase(gv), bo.Database()
    db.add(b.vectors()[1:])
    for h in host[1:]:
        odb.add(*h[1:])
    got = db.query(b.vectors()[:1], 5).results()[0]
    ids_, sc, c = odb.query(*host[0][1:], 5)
    assert [e for e, _ in got] == ids_.tolist() and np.array_equal(bc.bits([s for _, s in got]), bc.bits(sc))
    sc2 = db.score([0, 1], b.vectors()[:1] * 2).cpu().numpy()
    assert np.array_equal(bc.bits(sc2), bc.bits([odb.score(e, *host[0][1:]) for e in (0, 1)]))


def test_more_rejections():
    v = bc.synthetic_voc(5, k=4, L=3, D=32)
    hd, L = A._Handle(), _lib.lib()
    d, keep = _voc_desc(v, num_nodes=_lib.BOW_MAX_NODES + 1)
    out = C.c_void_p()
    assert L.dfk_bow_vocabulary_create(hd.h, C.byref(d), C.byref(out)) == _lib.DFK_ERR_INVALID_ARG
    assert "num_nodes" in L.dfk_last_error(hd.h).decode() and not out.value
    gv = A.BowVocabulary(v)
    hd = gv._hd
    hd.use_torch_stream()
    db = A.BowDatabase(gv)
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    empty = _lib.DfkBowVector(None, None, cnt.data_ptr(), 0)
    # a null count
    st = L.dfk_bow_database_add(hd.h, db._p, (_lib.DfkBowVector * 1)(_lib.DfkBowVector(None, None, None, 0)), 1, None)
    assert st == _lib.DFK_ERR_INVALID_ARG and "vector 0" in L.dfk_last_error(hd.h).decode() and len(db) == 0
    ids = torch.full((65535 * 2,), -7, dtype=torch.int32, device="cuda")
    scs = torch.full((65535 * 2,), -7.0, dtype=torch.float64, device="cuda")
    qc = torch.full((65535,), -7, dtype=torch.int32, device="cuda")
    big = torch.zeros(8193, dtype=torch.float64, device="cuda")
    bigw = torch.zeros(8193, dtype=torch.int32, device="cuda")

    def query(qs):
        arr = (_lib.DfkBowQuery * len(qs))(*qs)
        st = L.dfk_bow_database_query_batch(hd.h, db._p, arr, len(qs), C.c_void_p(ids.data_ptr()),
                                            C.c_void_p(scs.data_ptr()), C.c_void_p(qc.data_ptr()))
        return st, L.dfk_last_error(hd.h).decode()

    st, msg = query([_lib.DfkBowQuery(empty, 1, -1),
                     _lib.DfkBowQuery(_lib.DfkBowVector(bigw.data_ptr(), big.data_ptr(), cnt.data_ptr(), 8193), 1, -1)])
    assert st == _lib.DFK_ERR_INVALID_ARG and "capacity > DFK_MATCH_MAX_QUERIES" in msg and "query 1" in msg, msg
    # queries x entries > 2^26: 65535 queries against 1025 entries
    db.add([A.BowVector(bigw, big, cnt, 0)] * 1025)
    st, msg = query([_lib.DfkBowQuery(empty, 1, -1)] * 65535)
    assert st == _lib.DFK_ERR_INVALID_ARG and "2^26" in msg, msg
    # queries x entries^2 > 2^36: one query against 262,145 entries
    while len(db) < 262145:
        db.add([A.BowVector(bigw, big, cnt, 0)] * min(65535, 262145 - len(db)))
    st, msg = query([_lib.DfkBowQuery(empty, 1, -1)])
    assert st == _lib.DFK_ERR_INVALID_ARG and "2^36" in msg, msg
    torch.cuda.synchronize()
    assert (ids == -7).all() and (scs == -7.0).all() and (qc == -7).all()


def test_loop_detector_runs_on_the_device(golden, oracle):
    """aligners.LoopDetector end to end: AddKeyframe of two keyframes (a decoy, the true one), DetectLoop of the live
    frame: its result equals the plain functions applied to the query and a TrackFrameBatch of the same candidates"""
    from helpers import tracking_pyramid
    from deepfactors_b200 import se3
    cams, p0, p1, pd, pg = tracking_pyramid(golden, oracle, 3)
    up = lambda lst: [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in lst]
    mir0 = [np.ascontiguousarray(a[:, ::-1]) for a in p0]
    mird = [np.ascontiguousarray(a[:, ::-1]) for a in pd]
    z, voc = _orb_voc()
    t = np.load(os.path.join(bc.ROOT, "tests", "golden", "testimg.npz"))
    cfg = A.LoopDetectorConfig(iters=(10, 5, 4), min_similarity=0.0, max_dist=10.0, max_candidates=5,
                               active_window=2)
    ld = A.LoopDetector(voc, cams, cfg)
    g = lambda im: A.OrbDetectBatch(ld.voc_, [torch.from_numpy(np.ascontiguousarray(im)).cuda()]).features()[0]
    f1047, f1052 = g(t["gray_1047"]), g(t["gray_1052"])
    f_mirror = g(np.ascontiguousarray(t["gray_1047"][:, ::-1]))
    keyframes = {1: (up(mir0), up(mird), se3.identity()), 2: (up(p0), up(pd), se3.identity())}
    ld.AddKeyframe(1, f_mirror)
    ld.AddKeyframe(2, f1047)
    info = ld.DetectLoop(up(p1), [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in pg],
                         f1052, 9, keyframes)
    # the same steps by hand
    q = A.BowTransformBatch(ld.voc_, [f1052]).vectors()
    res = ld.db_.query(q, cfg.max_candidates, -1).results()[0]
    cands = A.loop_candidates(res, 9, cfg.active_window, cfg.min_similarity)
    assert cands, res
    poses_ck, frac, _ = ld.tracker_.TrackFrameBatch([keyframes[c] for c in cands], up(p1),
                                                    [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
                                                     for a in pg])
    pwk = [np.asarray(keyframes[c][2], np.float32) for c in cands]
    want = A.loop_select(cands, [se3.compose(w, se3.inverse(p)) for w, p in zip(pwk, poses_ck)], frac, pwk,
                         cfg.max_dist)
    print(f"query results {res}, candidates {cands}, inliers {frac}, loop {info.loop_id} detected {info.detected}")
    assert (info.detected, info.loop_id) == (want.detected, want.loop_id)
    if info.detected:
        assert np.array_equal(info.pose_wc, want.pose_wc)
    assert ld.last_min_score is None  # keyframe 9 was never added: no score against it
    ld.Reset()
    assert len(ld.db_) == 0


def test_facade_binary(tmp_path):
    """df::BowVocabulary / df::BowDatabase against the dfk_bow_* calls (tests/cpp/bow_test) on the reference's
    small_voc, read by the facade's LoadText"""
    import gzip
    import subprocess
    src = tmp_path / "voc.yml"
    with gzip.open(bc.SMALL_VOC, "rt") as f:
        src.write_text(f.read())
    exe = os.path.join(bc.ROOT, "tests", "cpp", "bow_test")
    r = subprocess.run([exe, str(src)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0 and "bow_test OK" in r.stdout
