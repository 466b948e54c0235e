"""Keypoint matching of reprojection factors on the device (dfk_hamming_match_batch, dfk_reprojection_match_batch)
against the CPU oracle (match_oracle) and OpenCV's matches (tests/golden/match_features.npz):

- the matcher bit for bit against cv2 for ORB and BRISK both ways, and on mixed batches with edge cases (one feature,
  all-equal descriptors, empty sets);
- per item, the selected hypothesis, its inlier count, the hypotheses evaluated and the sorted, pruned list bit for bit
  against the sequential oracle (matches scoring within 1e-12 relative of the threshold are printed);
- an item's output does not depend on the rest of the batch;
- links built on the device feed SfmWindowProblem and DeviceWindowOptimizer exactly as the same lists from the host;
- invalid items are rejected before anything is written;
- df::ReprojectionMatcher of the C++ facade (tests/cpp/match_test)."""
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib, se3
from match_oracle import match_oracle as mo
from match_scenes import Cam, make_scene

pytestmark = pytest.mark.gpu

FIXTURE_CAM = Cam(fx=262.5, fy=262.5, u0=160.0, v0=120.0, width=320.0, height=240.0)


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(scope="module")
def aligner(torch_mod):
    from deepfactors_b200.aligners import SfmAligner
    return SfmAligner(8)


def _feat(kp, desc):
    from deepfactors_b200.aligners import Features
    return Features.from_host(kp, desc)


def _fixture_items():
    z = np.load(__file__.replace("test_gpu_match.py", "golden/match_features.npz"))
    items, host = [], []
    for det in ("orb", "brisk"):
        f = {k: (z[f"{det}_kp_{k}"], z[f"{det}_desc_{k}"]) for k in ("1047", "1052")}
        dev = {k: _feat(*v) for k, v in f.items()}
        for a, b in (("1047", "1052"), ("1052", "1047")):
            items.append(dict(query=dev[a], train=dev[b], cam=FIXTURE_CAM))
            host.append((f[a], f[b], z[f"{det}_match_{a}_{b}"]))
    return items, host


def test_matcher_equals_opencv(aligner):
    from deepfactors_b200.aligners import HammingMatchBatch, match_offsets
    items, host = _fixture_items()
    got = HammingMatchBatch(aligner, items).cpu().numpy()
    off = match_offsets(items)
    for i, (_, _, want) in enumerate(host):
        assert np.array_equal(got[off[i]:off[i + 1]], want), i


def test_matcher_edge_cases_in_one_batch(aligner):
    from deepfactors_b200.aligners import HammingMatchBatch, match_offsets
    rng = np.random.default_rng(2)
    kp = lambda n: rng.uniform(0, 100, (n, 2)).astype(np.float32)  # noqa: E731
    d32 = lambda n: rng.integers(0, 256, (n, 32), dtype=np.uint8)  # noqa: E731
    d64 = lambda n: rng.integers(0, 256, (n, 64), dtype=np.uint8)  # noqa: E731
    sets = [
        ((kp(1), d32(1)), (kp(300), d32(300))),                       # one query
        ((kp(200), d64(200)), (kp(1), d64(1))),                       # one train feature
        ((kp(130), np.full((130, 32), 7, np.uint8)), (kp(260), np.full((260, 32), 7, np.uint8))),  # all ties
        ((kp(50), d64(50)), (kp(0), d64(0))),                         # empty train set
        ((kp(0), d32(0)), (kp(10), d32(10))),                         # empty query set
        ((kp(700), d32(700)), (kp(333), d32(333))),                   # several CTAs and tiles
        ((kp(129), d64(129)), (kp(129), d64(129))),
    ]
    items = [dict(query=_feat(*a), train=_feat(*b)) for a, b in sets]
    got = HammingMatchBatch(aligner, items).cpu().numpy()
    off = match_offsets(items)
    for i, (a, b) in enumerate(sets):
        assert np.array_equal(got[off[i]:off[i + 1]], mo.hamming(a[1], b[1])), i


def _scene_items(seeds=(1, 2, 3)):
    """synthetic scenes of the sizes a mapper sees: 500 ORB-sized and 1000 BRISK-sized features, 30-60 % outliers"""
    out = []
    for s in seeds:
        for n, nb, frac, noise in ((500, 32, 0.3, 0.5), (1000, 64, 0.5, 0.3), (800, 32, 0.6, 0.2)):
            sc = make_scene(n, frac, noise, 100 * s + n, desc_bytes=nb, max_flips=40)
            out.append((sc, s))
    return out


def _check_against_oracle(items, host, matches, counts, ransac, off):
    for i, (it, (q, t)) in enumerate(zip(items, host)):
        p = mo.params(it["cam"], max_dist=it.get("max_dist", 30.0), max_iterations=it.get("max_iterations", 1000),
                      threshold=it.get("threshold", float(np.float32(1e-4))), seed=it.get("seed", 0))
        want = mo.reprojection_match(p, q[0], q[1], t[0], t[1])
        near = np.flatnonzero(np.abs(want.scores - p.threshold) <= 1e-12 * p.threshold)
        for j in near:
            print(f"item {i}: match {j} scores {want.scores[j]!r}, within 1e-12 of the threshold {p.threshold!r}")
        got_rows = matches[off[i]:off[i] + counts[i]]
        print(f"item {i}: n0 {len(q[0])} best {want.best} inliers {want.inliers} evaluated {want.evaluated} "
              f"kept {len(want.rows)}")
        assert tuple(ransac[i]) == (want.best, want.inliers, want.evaluated), i
        assert counts[i] == len(want.rows) and np.array_equal(got_rows, want.rows), i


def test_ransac_equals_the_sequential_oracle(aligner):
    from deepfactors_b200.aligners import ReprojectionMatchBatch, match_offsets
    items, host = _fixture_items()
    host = [(a, b) for a, b, _ in host]
    for k, (sc, s) in enumerate(_scene_items()):
        items.append(dict(query=_feat(sc.kp0, sc.desc0), train=_feat(sc.kp1, sc.desc1), cam=sc.cam, seed=s + k))
        host.append(((sc.kp0, sc.desc0), (sc.kp1, sc.desc1)))
    # a short iteration budget, a tight threshold, a tight max_dist, fewer than 8 matches, an empty train set
    sc, _ = _scene_items((4,))[1]
    for extra in (dict(max_iterations=33, seed=9), dict(threshold=1e-6, seed=10), dict(max_dist=12.0, seed=11)):
        items.append(dict(query=_feat(sc.kp0, sc.desc0), train=_feat(sc.kp1, sc.desc1), cam=sc.cam, **extra))
        host.append(((sc.kp0, sc.desc0), (sc.kp1, sc.desc1)))
    items.append(dict(query=_feat(sc.kp0[:7], sc.desc0[:7]), train=_feat(sc.kp1, sc.desc1), cam=sc.cam))
    host.append(((sc.kp0[:7], sc.desc0[:7]), (sc.kp1, sc.desc1)))
    items.append(dict(query=_feat(sc.kp0, sc.desc0), train=_feat(sc.kp1[:0], sc.desc1[:0]), cam=sc.cam))
    host.append(((sc.kp0, sc.desc0), (sc.kp1[:0], sc.desc1[:0])))
    matches, counts, ransac = ReprojectionMatchBatch(aligner, items)
    _check_against_oracle(items, host, matches.cpu().numpy(), counts.cpu().numpy(), ransac.cpu().numpy(),
                          match_offsets(items))


def test_an_items_output_does_not_depend_on_the_batch(aligner):
    from deepfactors_b200.aligners import ReprojectionMatchBatch, match_offsets
    scenes = _scene_items((5,))
    items = [dict(query=_feat(sc.kp0, sc.desc0), train=_feat(sc.kp1, sc.desc1), cam=sc.cam, seed=k)
             for k, (sc, _) in enumerate(scenes)]
    full = [x.cpu().numpy() for x in ReprojectionMatchBatch(aligner, items)]
    off = match_offsets(items)
    for i in range(len(items)):
        for batch in ([items[i]], [items[i]] + items[:i] + items[i + 1:], items[::-1]):
            j = next(k for k, it in enumerate(batch) if it is items[i])
            m, c, r = [x.cpu().numpy() for x in ReprojectionMatchBatch(aligner, batch)]
            o = match_offsets(batch)
            assert np.array_equal(r[j], full[2][i]) and c[j] == full[1][i]
            assert np.array_equal(m[o[j]:o[j] + c[j]], full[0][off[i]:off[i] + full[1][i]])


def test_device_links_feed_the_window_as_host_lists(torch_mod, aligner):
    """match_reprojection_links against ReprojectionLinks built from the oracle's lists: equal lists, and
    DeviceWindowOptimizer gives the same result bit for bit on both problems"""
    torch = torch_mod
    import test_gpu_reprojection_batch as tr
    from test_oracle_ref import _keypoint_matches
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import (DeviceWindowOptimizer, LMParams, ReprojectionLink, SfmWindowProblem,
                                             match_reprojection_links)
    cs = 8
    base, cams, keyframes = tr._window_scene(torch, cs)
    L = base.levels[0]
    rng = np.random.default_rng(4)
    moved = se3.make_pose([0.01, -0.02, 0.015], [0.06, -0.03, 0.02], np.float64)
    q, t = _keypoint_matches(L.cam, se3.identity(np.float64), moved, L.prx_orig, n=400, seed=31)
    t[:120] = rng.uniform([0, 0], [L.width, L.height], (120, 2)).astype(np.float32)  # outliers
    d0 = rng.integers(0, 256, (400, 32), dtype=np.uint8)
    d2 = d0 ^ (rng.random((400, 32)) < 0.04).astype(np.uint8) * np.uint8(1 << 3)
    host_f = {0: (q, d0), 2: (t, d2)}
    feats = {k: _feat(*v) for k, v in host_f.items()}
    links = match_reprojection_links(aligner, feats, [(0, 2)], L.cam, cauchy_delta=3.0, sigma=1.5, seed=5)
    want = []
    for j, (a, b) in enumerate(((0, 2), (2, 0))):
        p = mo.params(L.cam, seed=5 + j)
        r = mo.reprojection_match(p, host_f[a][0], host_f[a][1], host_f[b][0], host_f[b][1])
        if len(r.rows):
            want.append(ReprojectionLink(a, b, host_f[a][0][r.rows[:, 0]], host_f[b][0][r.rows[:, 1]], 3.0, 1.5))
    assert len(links) == len(want) == 2
    for g, w in zip(links, want):
        print(f"link {g.k0} -> {g.k1}: {len(g.query_xy)} matches")
        assert (g.k0, g.k1) == (w.k0, w.k1) and len(g.query_xy) >= 100
        assert np.array_equal(g.query_xy, w.query_xy) and np.array_equal(g.train_xy, w.train_xy)
    poses = np.stack([se3.identity(np.float64), se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                      se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.006], np.float64)])
    codes = np.zeros((3, cs))
    out = []
    for lk in (links, want):
        prob = SfmWindowProblem(SfmAligner(cs), cams, keyframes, [(0, 1), (1, 2), (1, 0)], links=lk)
        out.append(DeviceWindowOptimizer(prob, LMParams(iterations=4)).run(poses, codes))
    (gp, gc, gt), (wp, wc, wt) = out
    assert np.array_equal(gp, wp) and np.array_equal(gc, wc) and gt.energy == wt.energy


def test_invalid_items_are_rejected(aligner, torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import HammingMatchBatch, ReprojectionMatchBatch
    rng = np.random.default_rng(0)
    kp = rng.uniform(0, 100, (20, 2)).astype(np.float32)
    a32, a64 = _feat(kp, rng.integers(0, 256, (20, 32), dtype=np.uint8)), _feat(kp, rng.integers(0, 256, (20, 64),
                                                                                                 dtype=np.uint8))
    a16 = _feat(kp, rng.integers(0, 256, (20, 16), dtype=np.uint8))
    out = torch.full((40, 2), -7, dtype=torch.int32, device="cuda")
    good = dict(query=a32, train=a32, cam=FIXTURE_CAM)
    with pytest.raises(_lib.DfkError) as e:
        HammingMatchBatch(aligner, [good, dict(query=a16, train=a16)], out=out)
    assert e.value.status == _lib.DFK_ERR_UNSUPPORTED and "item 1" in e.value.message
    with pytest.raises(_lib.DfkError) as e:
        HammingMatchBatch(aligner, [good, dict(query=a32, train=a64)], out=out)
    assert e.value.status == _lib.DFK_ERR_INVALID_ARG and "item 1" in e.value.message
    for bad in (dict(max_iterations=0), dict(probability=1.0), dict(threshold=0.0), dict(max_dist=float("nan")),
                dict(cam=Cam(fx=0.0))):
        with pytest.raises(_lib.DfkError) as e:
            ReprojectionMatchBatch(aligner, [good, dict(good, **bad)])
        assert e.value.status == _lib.DFK_ERR_INVALID_ARG and "item 1" in e.value.message, bad
    torch.cuda.synchronize()
    assert bool((out == -7).all())


def test_facade_matching_binary():
    """df::ReprojectionMatcher against the C calls it wraps (tests/cpp/match_test)"""
    exe = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "match_test")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "match_test OK" in r.stdout
