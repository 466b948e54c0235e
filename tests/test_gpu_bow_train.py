"""dfk_bow_vocabulary_train / dfk_bow_vocabulary_export on the device against the sequential C oracle of include/dfk.h's
DBoW2 training block, bit for bit: every exported array (weights by bit pattern) and the stats."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import bow_cases as bc
import bow_train_cases as bt
from bow_oracle import bow_oracle as bo
from deepfactors_b200 import _lib
from deepfactors_b200 import aligners as A

pytestmark = pytest.mark.gpu

SMALL_MAX = 2048  # kBowTrainSmallMax: the largest node one CTA trains
KEYS = ("node_ids", "parent_ids", "descriptors", "word_ids", "word_nodes")


def _same(got: dict, want: dict):
    for key in ("k", "L", "descriptor_bytes"):
        assert int(got[key]) == int(want[key]), key
    for key in KEYS:
        assert np.array_equal(np.asarray(got[key]), np.asarray(want[key])), key
    assert np.array_equal(bc.bits(got["weights"]), bc.bits(want["weights"])), "weights"


def _train(x, off, k, L, seed):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    return A.TrainVocabulary(t, k=k, L=L, seed=seed, image_offsets=off)


def _against_oracle(x, off, k, L, seed):
    v = _train(x, off, k, L, seed)
    want, stats = bo.train(x, off, k, L, seed)
    _same(v.voc, want)
    assert v.stats == stats, (v.stats, stats)
    bt.check_dbow2_layout(v.voc)
    return v, stats


@pytest.mark.parametrize("case", bt.CASES, ids=[bt.case_id(c) for c in bt.CASES])
def test_case_matrix_matches_the_oracle(case):
    x, off, k, L, seed = bt.case_data(case)
    _, stats = _against_oracle(x, off, k, L, seed)
    assert stats["capped_nodes"] == 0


@pytest.mark.parametrize("n", [SMALL_MAX, SMALL_MAX + 1])
@pytest.mark.parametrize("D", [32, 48, 64])
def test_root_at_and_above_the_small_node_bound(n, D):
    """the root alone on the one-CTA path (n = 2048) and on the multi-CTA path (n = 2049)"""
    x = bt.planted(n, D, 9, 2, 8, seed=n + D)
    _against_oracle(x, bt.offsets_for(n, 7, n), 9, 1, 3)


@pytest.mark.parametrize("k,D", [(32, 64), (2, 32)])
def test_large_nodes_at_the_widest_and_narrowest_k(k, D):
    n = 9000
    x = bt.planted(n, D, k if k > 2 else 4, 2, 10, seed=k)
    _against_oracle(x, bt.offsets_for(n, 30, k, empty=2), k, 3, 11)


@pytest.mark.parametrize("kind,D", [("few", 32), ("few", 64), ("one_bit", 32), ("one_bit", 48)])
def test_large_roots_with_early_stopping_seeding_and_exact_ties(kind, D):
    """N = 5000 at the root, on the multi-CTA path: fewer distinct descriptors than k (the seeding stops in the draw
    kernel and the later seeding launches skip the node), or one set bit each (every distance ties)"""
    n = 5000
    x = bt.make(kind, n, D, 9, 3)
    _, stats = _against_oracle(x, bt.offsets_for(n, 12, 3, empty=1), 9, 3, 3)
    if kind == "few":
        assert stats["num_nodes"] < 9 * 2


@pytest.mark.parametrize("seed", [27, 31])
def test_large_root_with_an_emptied_cluster(seed):
    """a root of 3000 descriptors (multi-CTA) whose converged partition leaves a cluster empty (seeds found with the
    oracle); L = 1, so the root is the only clustered node"""
    n = 3000
    x = bt.planted(n, 32, 9, 2, 8, seed=100 + seed)
    _, stats = _against_oracle(x, bt.offsets_for(n, 10, seed), 9, 1, seed)
    assert stats["empty_clusters"] >= 1


def test_both_paths_across_levels_k10_L6():
    """k = 10, L = 6 over 60 k descriptors: large nodes at the top levels, small ones below"""
    n = 60000
    x = bt.planted(n, 32, 10, 4, 6, seed=21)
    _, stats = _against_oracle(x, bt.offsets_for(n, 120, 21, empty=3), 10, 6, 0)
    assert stats["num_nodes"] > 10000


def test_200k_descriptors_d48():
    n = 200000
    x = bt.planted(n, 48, 10, 3, 12, seed=5)
    _against_oracle(x, bt.offsets_for(n, 400, 5), 10, 4, 7)


def test_deterministic_across_calls_and_handles_and_seed_dependent():
    n = 20000
    x = bt.planted(n, 32, 8, 3, 8, seed=9)
    off = bt.offsets_for(n, 50, 9)
    a, b = _train(x, off, 8, 4, 1), _train(x, off, 8, 4, 1)  # each TrainVocabulary call has a handle of its own
    _same(a.voc, b.voc)
    assert a.stats == b.stats
    c = _train(x, off, 8, 4, 2)
    assert not all(np.array_equal(np.asarray(a.voc[key]), np.asarray(c.voc[key])) for key in KEYS)


def _raw_train(hd, **over):
    x = torch.from_numpy(bt.make("random", 100, 32, 4, 0)).cuda()
    off = np.array([0, 40, 100], np.int64)
    f = dict(k=4, L=2, descriptor_bytes=32, num_images=2, seed=0, num_descriptors=100, descriptors_dev=x.data_ptr(),
             image_offsets=off.ctypes.data)
    f.update(over)
    d = _lib.DfkBowTrainDesc(**f)
    p = C.c_void_p()
    st = _lib.lib().dfk_bow_vocabulary_train(hd.h, C.byref(d), None, C.byref(p))
    return st, p, _lib.lib().dfk_last_error(hd.h)


def test_rejected_calls_create_nothing():
    hd = A._Handle()
    big = np.array([0, 9000], np.int64)
    dec = np.array([0, 60, 40, 100], np.int64)
    short = np.array([0, 40, 99], np.int64)
    cases = [(dict(k=1), b"k not in"), (dict(k=33), b"k not in"), (dict(L=0), b"L not in"),
             (dict(L=17), b"L not in"), (dict(descriptor_bytes=16), b"descriptor_bytes"),
             (dict(num_images=0), b"num_images"),
             (dict(descriptors_dev=torch.zeros(4000, dtype=torch.uint8, device="cuda").data_ptr() + 4),
              b"16-byte aligned"),
             (dict(num_images=3, image_offsets=dec.ctypes.data), b"decrease"),
             (dict(image_offsets=short.ctypes.data), b"num_descriptors"),
             (dict(num_images=1, num_descriptors=9000, image_offsets=big.ctypes.data), b"DFK_MATCH_MAX_QUERIES"),
             # the size is checked before the offsets (a null pointer here) are read
             (dict(num_descriptors=2 ** 28 + 1, image_offsets=None), b"num_descriptors not in")]
    for over, msg in cases:
        st, p, err = _raw_train(hd, **over)
        assert st == _lib.DFK_ERR_INVALID_ARG, over
        assert not p.value, over
        assert msg in err, (over, err)
    st, p, _ = _raw_train(hd)
    assert st == _lib.DFK_OK and p.value
    _lib.lib().dfk_bow_vocabulary_destroy(hd.h, p)


def test_transform_with_the_trained_handle_equals_the_saved_file(tmp_path):
    n = 12000
    x = bt.planted(n, 32, 8, 3, 8, seed=4)
    off = bt.offsets_for(n, 40, 4, empty=1)
    v = _train(x, off, 8, 3, 5)
    for name in ("voc.yml", "voc.yml.gz"):
        path = os.path.join(tmp_path, name)
        A.save_dbow2_vocabulary(path, v)
        loaded = A.BowVocabulary(path)
        _same(loaded.export(), v.voc)
        rows = [torch.from_numpy(x[off[j]:off[j + 1]]).cuda() for j in range(len(off) - 1)]
        a, b = A.BowTransformBatch(v, rows), A.BowTransformBatch(loaded, rows)
        torch.cuda.synchronize()
        for key in ("words", "counts", "feature_words"):
            assert torch.equal(getattr(a, key), getattr(b, key)), key
        assert np.array_equal(bc.bits(a.values.cpu().numpy()), bc.bits(b.values.cpu().numpy()))


def test_device_orb_vocabulary_matches_the_oracle_and_retrieves_places():
    """device ORB of the images the test fixture's vocabulary is trained on, TrainVocabulary(k=8, L=3, seed=0) against
    the oracle on the same descriptors; then the place test of test_gpu_bow.py with that vocabulary"""
    import orb_images
    z = np.load(os.path.join(bc.ROOT, "tests", "golden", "bow_orb.npz"))
    t = np.load(os.path.join(bc.ROOT, "tests", "golden", "testimg.npz"))
    places = [z["gray_0"], t["gray_1047"], z["gray_25"], t["gray_1052"]]
    imgs = places + list(orb_images.images().values())
    hd_voc = A.BowVocabulary(bc.small_voc())  # any object with a handle runs the detector
    orb = A.OrbDetectBatch(hd_voc, [torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in imgs], nfeatures=500)
    feats = [f.descriptors for f in orb.features()]
    v = A.TrainVocabulary(feats, k=8, L=3, seed=0)
    flat = np.concatenate([f.cpu().numpy() for f in feats])
    off = np.concatenate([[0], np.cumsum([f.shape[0] for f in feats])]).astype(np.int64)
    want, stats = bo.train(flat, off, 8, 3, 0)
    _same(v.voc, want)
    assert v.stats == stats
    b = A.BowTransformBatch(v, feats[:4])
    vecs = b.vectors()
    db = A.BowDatabase(v)
    db.add(vecs[:2])
    res = db.query(vecs[2:], 2).results()
    names = ["0", "1047", "25", "1052"]
    for k in range(2):
        print(f"query {names[2 + k]}: top {names[res[k][0][0]]} (Score {res[k][0][1]:.4f}), "
              f"then {names[res[k][1][0]]} ({res[k][1][1]:.4f})")
        assert res[k][0][0] == k, "the other view of the place is expected first"


def test_facade_trains_exports_and_saves(tmp_path):
    """df::BowVocabulary(features, D, k, L, seed) (tests/cpp/bow_train_test train): its SaveText of Export equals the
    oracle's vocabulary and TrainVocabulary's file byte for byte; LoadText of it creates a vocabulary that exports and
    transforms the same"""
    n = 9000
    x = bt.planted(n, 32, 8, 3, 8, seed=31)
    off = bt.offsets_for(n, 25, 31, empty=2)
    desc, offs, out = (os.path.join(tmp_path, f) for f in ("d.bin", "o.bin", "v.yml"))
    x.tofile(desc)
    off.astype(np.int64).tofile(offs)
    exe = os.path.join(bc.ROOT, "tests", "cpp", "bow_train_test")
    import subprocess
    r = subprocess.run([exe, "train", desc, offs, "32", "8", "3", "4", out], capture_output=True, text=True,
                       timeout=300)
    assert r.returncode == 0 and "bow_train_test OK" in r.stdout, r.stdout + r.stderr
    want, stats = bo.train(x, off, 8, 3, 4)
    _same(A.load_dbow2_vocabulary(out), want)
    line = next(l for l in r.stdout.splitlines() if l.startswith("stats "))
    assert [int(v) for v in line.split()[1:6]] == [stats[k] for k in ("num_nodes", "num_words", "max_rounds",
                                                                      "capped_nodes", "empty_clusters")]
    py = os.path.join(tmp_path, "py.yml")
    A.save_dbow2_vocabulary(py, _train(x, off, 8, 3, 4))
    assert open(py).read() == open(out).read()
