"""CPU tests of the keypoint matching step of a reprojection factor (dfk_hamming_match_batch /
dfk_reprojection_match_batch): the oracle against OpenCV's brute-force matcher, the fp64 eight-point model and RANSAC
against known two-view geometry, the adaptive stop against a transliteration of the sequential loop, and the C struct
layouts against the Python binding."""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

from match_oracle import match_oracle as mo
from match_scenes import Cam, bearing, make_scene, rodrigues, rotation_angle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "match_features.npz")


@pytest.mark.parametrize("det", ["orb", "brisk"])
@pytest.mark.parametrize("a,b", [("1047", "1052"), ("1052", "1047")])
def test_oracle_matcher_equals_opencv(det, a, b):
    z = np.load(FIXTURE)
    m = mo.hamming(z[f"{det}_desc_{a}"], z[f"{det}_desc_{b}"])
    assert np.array_equal(m, z[f"{det}_match_{a}_{b}"])


def test_oracle_matcher_ties_and_empty_train():
    d0 = np.zeros((3, 32), np.uint8)
    d1 = np.zeros((4, 32), np.uint8)
    assert np.array_equal(mo.hamming(d0, d1), np.zeros((3, 2), np.int32))  # all equal: the lowest train index
    assert np.array_equal(mo.hamming(d0, d1[:0]), -np.ones((3, 2), np.int32))


def _views(seed, n=8):
    rng = np.random.default_rng(seed)
    R = rodrigues(rng.normal(size=3) * 0.1)
    t = rng.normal(size=3)
    X0 = np.c_[rng.uniform(-1, 1, (n, 2)), rng.uniform(2, 5, n)]
    X1 = X0 @ R.T + t
    return R, t, X0 / np.linalg.norm(X0, axis=1, keepdims=True), X1 / np.linalg.norm(X1, axis=1, keepdims=True)


@pytest.mark.parametrize("seed", range(5))
def test_eightpt_noise_free(seed):
    R, t, f0, f1 = _views(seed)
    E = mo.eightpt(f0, f1)
    assert np.abs(np.einsum("ki,ij,kj->k", f1, E, f0)).max() <= 1e-12
    Rm, tm = mo.model(f0, f1)
    assert rotation_angle(Rm, R) <= 1e-9
    assert np.abs(tm - t / np.linalg.norm(t)).max() <= 1e-9
    for k in range(8):  # every sample point scores ~0 under its own model
        assert abs(mo.score(Rm, tm, f0[k], f1[k])) <= 1e-12


def test_eightpt_degenerate_sample_is_invalid():
    R, t, f0, f1 = _views(0)
    f0[1], f1[1] = f0[0], f1[0]  # a repeated correspondence: rank 7
    assert mo.eightpt(f0, f1) is None and mo.model(f0, f1) is None


def test_sample_generator():
    for h in range(50):
        idx = mo.sample(7, h, 20)
        assert len(set(idx.tolist())) == 8 and idx.min() >= 0 and idx.max() < 20
    assert np.array_equal(mo.sample(7, 3, 20), mo.sample(7, 3, 20))
    assert not np.array_equal(mo.sample(7, 3, 20), mo.sample(8, 3, 20))
    assert sorted(mo.sample(1, 0, 8).tolist()) == list(range(8))


def _selected_rotation(sc, p, res):
    """the rotation of the selected hypothesis' model (the scenes match query q with train q)"""
    idx = mo.sample(p.seed, res.best, len(sc.kp0))
    return mo.model(bearing(sc.kp0[idx], sc.cam), bearing(sc.kp1[idx], sc.cam))[0]


@pytest.mark.parametrize("frac", [0.3, 0.45, 0.6])
@pytest.mark.parametrize("seed", [1, 2])
def test_ransac_separates_inliers_from_outliers(frac, seed):
    """opengv's default threshold (1e-4), 0.1 px noise, 30-60 % outliers off their epipolar lines"""
    thr = mo.params(Cam()).threshold
    sc = make_scene(600, frac, 0.1, seed, outlier_margin=10 * thr)
    p = mo.params(sc.cam, max_dist=1e9, seed=seed)
    matches = np.c_[np.arange(600), sc.flips].astype(np.int32)
    res = mo.reprojection_match(p, sc.kp0, sc.desc0, sc.kp1, sc.desc1, matches)
    kept = np.zeros(600, bool)
    kept[res.rows[:, 0]] = True
    assert kept[sc.inlier].mean() >= 0.95
    assert kept[~sc.inlier].mean() <= 0.01
    assert res.inliers == kept.sum()  # max_dist prunes nothing here
    assert 1 <= res.evaluated <= 1000


@pytest.mark.parametrize("frac", [0.3, 0.45])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_ransac_recovers_the_rotation(frac, seed):
    """The selected model is a minimal-sample model (no refit on the inliers, as in opengv's Ransac), so its rotation is
    only as sharp as the threshold makes the inlier count: with exact inliers (float32 keypoints) and a threshold of
    1e-7 it is the true rotation to 1e-3 rad."""
    sc = make_scene(600, frac, 0.0, seed, outlier_margin=1e-6)
    p = mo.params(sc.cam, max_dist=1e9, seed=seed, threshold=1e-7)
    matches = np.c_[np.arange(600), sc.flips].astype(np.int32)
    res = mo.reprojection_match(p, sc.kp0, sc.desc0, sc.kp1, sc.desc1, matches)
    assert res.best >= 0
    assert rotation_angle(_selected_rotation(sc, p, res), sc.R) <= 1e-3


def _sequential(counts, n, prob, max_it):
    """the sequential adaptive RANSAC loop, transliterated"""
    best, best_h, k, h = 0, -1, math.inf, 0
    while h < max_it:
        c = int(counts[h])
        if c > best:
            best, best_h = c, h
            w = best / n
            w2 = w * w
            w4 = w2 * w2
            q = min(max(1.0 - w4 * w4, 2.0 ** -52), 1.0 - 2.0 ** -52)
            k = math.log(1.0 - prob) / math.log(q)
        h += 1
        if h >= k:
            break
    return best_h, best, h


@pytest.mark.parametrize("frac,max_it,prob", [(0.3, 1000, 0.99), (0.6, 1000, 0.99), (0.6, 40, 0.99), (0.5, 300, 0.5)])
def test_adaptive_stop_matches_the_sequential_loop(frac, max_it, prob):
    sc = make_scene(200, frac, 0.5, 11)
    p = mo.params(sc.cam, max_iterations=max_it, probability=prob, seed=3)
    matches = np.c_[np.arange(200), sc.flips].astype(np.int32)
    counts = mo.hypothesis_counts(p, sc.kp0, sc.kp1, matches, max_it)
    res = mo.reprojection_match(p, sc.kp0, sc.desc0, sc.kp1, sc.desc1, matches)
    assert (res.best, res.inliers, res.evaluated) == _sequential(counts, 200, prob, max_it)


def test_pruning_sorts_by_distance_then_query():
    sc = make_scene(300, 0.2, 0.2, 5, max_flips=60)
    p = mo.params(sc.cam, max_dist=30.0, seed=1)
    res = mo.reprojection_match(p, sc.kp0, sc.desc0, sc.kp1, sc.desc1)
    assert len(res.rows) > 0 and res.rows[:, 2].max() <= 30
    assert np.array_equal(np.lexsort((res.rows[:, 0], res.rows[:, 2])), np.arange(len(res.rows)))
    inl = res.scores < p.threshold
    assert inl.sum() == res.inliers and len(res.rows) == (inl & (sc.flips <= 30)).sum()


def test_fewer_than_eight_matches_yield_nothing():
    sc = make_scene(7, 0.0, 0.1, 2)
    res = mo.reprojection_match(mo.params(sc.cam), sc.kp0, sc.desc0, sc.kp1, sc.desc1)
    assert len(res.rows) == 0 and (res.best, res.inliers, res.evaluated) == (-1, 0, 0)


def test_struct_layouts_match_the_header(tmp_path):
    """offsets and sizes of DfkFeatureSet / DfkMatchItem as the C compiler lays them out"""
    from deepfactors_b200 import _lib
    src = tmp_path / "layout.c"
    fields = {"DfkFeatureSet": [f[0] for f in _lib.DfkFeatureSet._fields_],
              "DfkMatchItem": [f[0] for f in _lib.DfkMatchItem._fields_]}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "dfk.h"', "int main(void) {"]
    for s, fs in fields.items():
        lines.append(f'printf("{s} %zu\\n", sizeof({s}));')
        lines += [f'printf("{s}.{f} %zu\\n", offsetof({s}, {f}));' for f in fs]
    lines += ["return 0; }"]
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                         check=True).stdout.splitlines())
    for s, fs in fields.items():
        cls = getattr(_lib, s)
        assert int(got[s]) == ctypes.sizeof(cls)
        for f in fs:
            assert int(got[f"{s}.{f}"]) == getattr(cls, f).offset, (s, f)
