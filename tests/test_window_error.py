"""Host logic of the window energy without a linearisation (no GPU): WindowOptimizer(error=...) with injected
linearise / solve / error, the host sum of SfmWindowProblem.error (rescale, items without inliers, prior terms) against
a numpy restatement, and the in-place rewrite of the ctypes item arrays it reuses."""
import numpy as np
import pytest

from deepfactors_b200 import _lib
from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import (LMParams, WindowError, WindowOptimizer, _struct_floats, prior_energy,
                                         window_error_sum)

CS = 2
# steps on code 0 of keyframe 0 and the energy 100 (c - 1)^2 they lead to: x = 0 (100), 3 (400, rejected), 0.5 (25),
# no step (not positive definite), 1.25 (6.25), 0.25 (56.25, rejected); every energy is exact in fp32
STEPS = [3.0, 0.5, None, 0.75, -1.0]  # from the accepted point


def energy(codes):
    return 100.0 * (codes[0, 0] - 1.0) ** 2


def fake_problem():
    wb = WindowBlocks(2, CS, [(0, 1)])
    log = []

    def linearise(poses, codes, todo):
        log.append(("linearise", float(codes[0, 0])))
        NP = 12 + CS
        buf = wb.pack([0], np.eye(NP)[None], np.zeros((1, NP)), [energy(codes)], [5], [(1, 5)])  # W * H / inliers = 1
        return buf, None

    def solve(buf, lam, fixed, w, codes):
        log.append(("solve", float(buf[wb.offsets()[2]])))
        step = STEPS[sum(1 for k, _ in log if k == "solve") - 1]
        if step is None:
            return None
        dx = np.zeros(wb.dim)
        dx[6] = step
        return dx

    def error(poses, codes):
        log.append(("error", float(codes[0, 0])))
        return energy(codes), WindowError(photometric=energy(codes))

    return wb, linearise, solve, error, log


def run(with_error):
    wb, linearise, solve, error, log = fake_problem()
    opt = WindowOptimizer(wb, linearise, LMParams(iterations=len(STEPS)), solve=solve,
                          error=error if with_error else None)
    poses = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float64), (2, 1))
    p, c, tr = opt.run(poses, np.zeros((2, CS)))
    return p, c, tr, log


def test_without_error_the_loop_is_unchanged():
    p, c, tr, log = run(False)
    # a linearisation at the start and at every candidate; the solve after a rejection sees the accepted point's buffer
    assert log == [("linearise", 0.0), ("solve", 100.0), ("linearise", 3.0), ("solve", 100.0), ("linearise", 0.5),
                   ("solve", 25.0), ("solve", 25.0), ("linearise", 1.25), ("solve", 6.25), ("linearise", 0.25)]
    assert tr.accepted == [False, True, False, True, False]
    assert tr.energy == [100.0, 25.0, 6.25]
    assert np.allclose(tr.lam, [1e-4, 1e-3, 1e-4, 1e-3, 1e-4], rtol=1e-12)
    assert tr.factors_relinearised == [1, 1, 1, 1, 1]
    assert tr.linearisations == 5 and tr.error_evaluations == 0
    assert c[0, 0] == 1.25


def test_with_error_a_rejected_step_linearises_nothing():
    p0, c0, t0, _ = run(False)
    p, c, tr, log = run(True)
    assert log == [("linearise", 0.0), ("error", 0.0), ("solve", 100.0), ("error", 3.0), ("solve", 100.0),
                   ("error", 0.5), ("linearise", 0.5), ("solve", 25.0), ("solve", 25.0), ("error", 1.25),
                   ("linearise", 1.25), ("solve", 6.25), ("error", 0.25)]
    # the accept / reject sequence follows E, and ends where the linearising loop ends
    assert tr.accepted == t0.accepted and tr.energy == t0.energy and tr.lam == t0.lam
    assert np.array_equal(p, p0) and np.array_equal(c, c0)
    assert tr.linearisations == 1 + sum(tr.accepted) == 3
    assert tr.error_evaluations == 1 + sum(s is not None for s in STEPS) == 5
    assert tr.factors_relinearised == [1, 1, 1]


def test_with_error_the_code_prior_is_added_to_E():
    wb, linearise, solve, error, log = fake_problem()
    w = 0.5
    opt = WindowOptimizer(wb, linearise, LMParams(iterations=2, code_prior_weight=w), solve=solve, error=error)
    poses = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float64), (2, 1))
    codes = np.full((2, CS), 0.25)
    _, _, tr = opt.run(poses, codes)
    assert tr.energy[0] == energy(codes) + 0.5 * w * float((codes ** 2).sum())


def test_host_energy_sum_matches_numpy():
    rng = np.random.default_rng(0)
    n = 40
    res = (rng.random(n) * 50).astype(np.float32)
    inl = rng.integers(0, 300, n).astype(np.uint32)
    inl[[3, 17, 18]] = 0  # items without inliers add nothing, whatever their residual
    res[17] = 123.0
    dense = np.stack([res, inl.view(np.float32)], 1)
    areas = [float(w * h) for w, h in zip(rng.integers(1, 641, n), rng.integers(1, 481, n))]
    rep = np.stack([(rng.random(3) * 9).astype(np.float32), np.array([4, 0, 9], np.uint32).view(np.float32)], 1)
    geo = np.stack([(rng.random(2) * 3).astype(np.float32), np.array([40, 7], np.uint32).view(np.float32)], 1)
    B = 6 + 4
    rows, deltas = [], []
    for nb in (B, 2 * B):
        A = rng.standard_normal((nb, nb))
        rows.append(np.concatenate([(A @ A.T).ravel(), rng.standard_normal(nb), [2.5]]))
        deltas.append(rng.standard_normal(nb) * 0.1)
    terms = [prior_energy(r, d) for r, d in zip(rows, deltas)]
    for r, d, t in zip(rows, deltas, terms):
        nb = d.size
        G, g, f0 = r[:nb * nb].reshape(nb, nb), r[nb * nb:-1], r[-1]
        assert t == pytest.approx(f0 - 2 * g @ d + d @ G @ d, rel=1e-14)
    got = window_error_sum(dense, areas, rep, geo, terms)
    keep = inl > 0
    pho = float(np.sum(res[keep].astype(np.float64) / inl[keep] * np.asarray(areas)[keep]))
    want = pho + float(rep[:, 0].astype(np.float64).sum()) + float(geo[:, 0].astype(np.float64).sum()) + sum(terms)
    assert got.energy == pytest.approx(want, rel=1e-13)
    assert got.photometric == pytest.approx(pho, rel=1e-13)
    assert got.no_inliers == 3 and got.inliers == int(inl.sum())
    assert got.reprojection == pytest.approx(float(rep[:, 0].astype(np.float64).sum()), rel=1e-15)
    assert got.priors == pytest.approx(sum(terms), rel=1e-15)
    empty = window_error_sum(np.zeros((0, 2), np.float32), [], np.zeros((0, 2)), np.zeros((0, 2)), [])
    assert empty.energy == 0.0 and empty.no_inliers == 0


def test_item_arrays_are_rewritten_in_place():
    arr = (_lib.DfkSfmWorkItem * 3)()
    p1 = _struct_floats(arr, "pose1", 7)
    p1[:] = np.arange(21, dtype=np.float32).reshape(3, 7)
    assert list(arr[2].pose1) == list(range(14, 21)) and list(arr[2].pose0) == [0.0] * 7
    geo = (_lib.DfkSparseGeometricItem * 2)()
    _struct_floats(geo, "pose0", 7)[1] = 0.5
    assert list(geo[1].pose0) == [0.5] * 7 and list(geo[0].pose0) == [0.0] * 7
