"""The mapper's ISAM2 steps in the library (dfk_window_problem_isam2_update, dfk_window_map_steps) on the synthetic
window of test_gpu_window_error._window: photometric pairs, reprojection and geometric links, a tracked frame, and a
frame and a keyframe prior (or none).

- DeviceIncrementalOptimizer.update() against IncrementalOptimizer.from_problem(...).update() on a twin problem over
  ten updates: equal ISAM2Result counts, the same relinearised keys, the records bit for bit, and theta_lin / delta /
  the estimate within 1e-9 relative (the largest difference is printed);
- an unreached threshold: the second update launches no RunStep kernel, first_column == K, nothing changes;
- map_steps against window_opt.mapping_steps on twin problems, and a continued call against one longer run;
- grow_from after a new keyframe with its pairs, links and a frame: kept records bit for bit, then the updates of
  IncrementalOptimizer.grow_problem's path; a wrong map is rejected and writes nothing;
- rejected arguments write nothing;
- df::WindowProblem's UpdateIncremental / MappingSteps / GrowFrom of the C++ facade (tests/cpp/window_isam2_test)."""
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib, se3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _twin(torch, cs, priors):
    """the window, built afresh (its own keyframe buffers and records), with or without its priors; perturbed poses"""
    from test_gpu_window_error import _window
    from deepfactors_b200.window_opt import SfmWindowProblem
    prob, poses = _window(torch, cs)
    if not priors:
        prob = SfmWindowProblem(prob.al, prob.cams, prob.kf, prob.pairs[:prob._num_photometric], links=prob.links,
                                geometric=prob.geometric, frames=prob.frames)
    rng = np.random.default_rng(5)
    p0 = np.asarray(poses, np.float64).copy()
    p0[1:] = np.stack([se3.retract(p, rng.standard_normal(6) * 0.02, np.float64) for p in p0[1:]])
    fposes = np.stack([se3.make_pose([0.002, -0.001, 0.003], [0.01, 0.004, -0.006], np.float64)])
    return prob, p0, np.zeros((3, cs)), fposes


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def _records_equal(torch, a, b):
    return torch.equal(a.records.view(torch.int32), b.records.view(torch.int32)) and \
        torch.equal(a.geo_records.view(torch.int32), b.geo_records.view(torch.int32))


@pytest.mark.parametrize("cs", [8, 32, 128])
@pytest.mark.parametrize("priors", [False, True])
def test_device_update_is_incremental_optimizer(torch_mod, cs, priors):
    torch = torch_mod
    from deepfactors_b200.window_opt import DeviceIncrementalOptimizer, IncrementalOptimizer
    host_prob, p0, c0, f0 = _twin(torch, cs, priors)
    dev_prob, _, _, _ = _twin(torch, cs, priors)
    kw = dict(relinearize_threshold=0.004, code_prior_weight=1e-2)
    host = IncrementalOptimizer.from_problem(host_prob, p0, c0, f0, **kw)
    dev = DeviceIncrementalOptimizer(dev_prob, poses=p0, codes=c0, frame_poses=f0, **kw)
    worst, moved_total = 0.0, 0
    for step in range(10):
        lin_before = dev.linearization() if step else None
        rh, rd = host.update(), dev.update()
        assert rh == rd, (step, rh, rd)
        assert _records_equal(torch, host_prob, dev_prob), step
        lp, lc, lf, d = dev.linearization()
        # the relinearised keys: exactly those whose theta_lin moved
        if step:
            moved = [("pose", k) for k in range(3) if not np.array_equal(lp[k], lin_before[0][k])] + \
                    [("code", k) for k in range(3) if not np.array_equal(lc[k], lin_before[1][k])] + \
                    [("frame", f) for f in range(len(lf)) if not np.array_equal(lf[f], lin_before[2][f])]
            assert len(moved) == rd.variables_relinearized, step
            moved_total += len(moved)
        hp, hc, hf = host.estimate()
        ep, ec, ef = dev.estimate()
        errs = [_rel(lp, host.lin_poses), _rel(lc, host.lin_codes) if np.any(host.lin_codes) else
                float(np.abs(lc - host.lin_codes).max()), _rel(lf, host.lin_frames), _rel(d, host.delta),
                _rel(ep, hp), _rel(ec, hc) if np.any(hc) else float(np.abs(ec - hc).max()), _rel(ef, hf)]
        worst = max(worst, max(errs))
        assert max(errs) <= 1e-9, (step, errs)
    print(f"C={cs} priors={priors}: {moved_total} keys relinearised, largest relative difference {worst:.2e}")
    assert moved_total > 0


def test_unreached_threshold_relinearises_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.window_opt import DeviceIncrementalOptimizer
    cs = 8
    prob, p0, c0, f0 = _twin(torch, cs, True)
    dev = DeviceIncrementalOptimizer(prob, relinearize_threshold=1e9, poses=p0, codes=c0, frame_poses=f0)
    r1 = dev.update()
    assert r1.first_column == 0 and r1.factors_relinearised == len(prob.pairs) + len(prob.geometric)
    rec, geo = prob.records.clone(), prob.geo_records.clone()
    _, _, _, d1 = dev.linearization()
    h = dev.dev._al.handle
    lib = _lib.lib()
    lib.dfk_set_profiling(h, 1)
    import ctypes as C
    ms, main, total = C.c_double(), C.c_uint64(), C.c_uint64()
    lib.dfk_get_profile(h, C.byref(ms), C.byref(main), C.byref(total))
    r2 = dev.update()
    torch.cuda.synchronize()
    lib.dfk_get_profile(h, C.byref(ms), C.byref(main), C.byref(total))
    lib.dfk_set_profiling(h, 0)
    print(f"second update: {main.value} RunStep launches, {total.value} launches in all")
    assert main.value == 0
    assert r2.first_column == 3 and r2.factors_relinearised == 0 and r2.variables_relinearized == 0
    assert r2.variables_reeliminated == 6 * len(prob.frames)
    assert torch.equal(prob.records, rec) and torch.equal(prob.geo_records, geo)
    assert np.array_equal(dev.linearization()[3], d1)


def _works(prob, iters):
    from deepfactors_b200.window_opt import OptimizeWork
    n = len(prob.dense_pairs())
    return [OptimizeWork(iters, remove_after=(q % 2 == 1)) for q in range(n)]


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_map_steps_is_mapping_steps(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.window_opt import DeviceIncrementalOptimizer, IncrementalOptimizer, mapping_steps
    host_prob, p0, c0, f0 = _twin(torch, cs, False)
    dev_prob, _, _, _ = _twin(torch, cs, False)
    kw = dict(relinearize_threshold=0.004, code_prior_weight=1e-2)
    iters = [2] + [1] * (host_prob.levels - 1)
    host = IncrementalOptimizer.from_problem(host_prob, p0, c0, f0, **kw)
    dev = DeviceIncrementalOptimizer(dev_prob, poses=p0, codes=c0, frame_poses=f0, **kw)
    hw, dw = _works(host_prob, iters), _works(dev_prob, iters)
    sched = host_prob.level_schedule(iters, remove_after=[w.remove_after for w in hw])
    rh, lh = mapping_steps(host, host_prob, hw, 40, sched)
    rd, ld = dev.map_steps(dw, 40)
    print(f"C={cs}: {len(rh)} steps; levels {lh}; results {[tuple(vars(r).values()) for r in rd]}")
    assert rd == rh and ld == lh
    for a, b in zip(hw, dw):
        assert (a.active_level, a.iters, a.first, a.remove, a.factor, a.erased) == \
            (b.active_level, b.iters, b.first, b.remove, b.factor, b.erased)
    assert _records_equal(torch, host_prob, dev_prob)
    hp, hc, hf = host.estimate()
    ep, ec, ef = dev.estimate()
    assert _rel(ep, hp) <= 1e-9 and _rel(ec, hc) <= 1e-9 and _rel(ef, hf) <= 1e-9
    # a continued call equals one longer run
    split_prob, _, _, _ = _twin(torch, cs, False)
    split = DeviceIncrementalOptimizer(split_prob, poses=p0, codes=c0, frame_poses=f0, **kw)
    sw = _works(split_prob, iters)
    a, la = split.map_steps(sw, 3)
    b, lb = split.map_steps(sw, 40)
    assert a + b == rd and la + lb == ld
    assert np.array_equal(split.estimate()[0], ep) and np.array_equal(split.estimate()[1], ec)


def test_rejected_arguments_write_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.window_opt import DeviceIncrementalOptimizer
    prob, p0, c0, f0 = _twin(torch, 8, True)
    dev = DeviceIncrementalOptimizer(prob, poses=p0, codes=c0, frame_poses=f0)
    dev.update()
    torch.cuda.synchronize()
    state, rec = dev.dev.get_state(), prob.records.clone()
    lin = dev.linearization()
    for bad in (dict(relinearize_skip=0), dict(relinearize_threshold=float("nan")), dict(code_prior_weight=-1.0)):
        with pytest.raises(_lib.DfkError) as e:
            dev.dev.isam2_update(**bad)
        assert e.value.status == _lib.DFK_ERR_INVALID_ARG
    works = _works(prob, [1] * prob.levels)
    works[0].active_level = 7  # not a state of its schedule
    with pytest.raises(_lib.DfkError, match="work 0"):
        dev.map_steps(works, 5)
    assert works[0].active_level == 7
    sched = prob.level_schedule([1] * prob.levels)
    with pytest.raises(_lib.DfkError, match="num_levels"):
        dev.dev.map_steps(sched.__class__(**{**vars(sched), "iters": []}), None, 5)
    torch.cuda.synchronize()
    s2 = dev.dev.get_state()
    assert np.array_equal(s2[0], state[0]) and np.array_equal(s2[1], state[1])
    assert torch.equal(prob.records, rec)
    for x, y in zip(dev.linearization(), lin):
        assert np.array_equal(x, y)
    # a sharded window has no device problem
    prob.allreduce = lambda buf: buf
    prob._dev = None
    with pytest.raises(ValueError, match="all-reduce"):
        DeviceIncrementalOptimizer(prob)


@pytest.mark.parametrize("cs", [8, 32])
def test_grow_from_is_grow_problem(torch_mod, cs):
    """the window of test_gpu_window_incremental._grown_scene (three keyframes, grown by keyframe 3 with pairs (3, 2) /
    (2, 3), a reprojection link, a geometric link and a frame on keyframe 3): host and device runs of two updates, the
    growth, and three more updates"""
    torch = torch_mod
    from test_gpu_window_incremental import _grown_scene, _rows
    from deepfactors_b200.window_opt import DeviceIncrementalOptimizer, IncrementalOptimizer
    h_old, h_new, _, factor_of, frame_of, poses, fposes = _grown_scene(torch, cs)
    d_old, d_new, _, _, _, _, _ = _grown_scene(torch, cs)
    codes = np.random.default_rng(5).standard_normal((4, cs)) * 0.05
    kw = dict(relinearize_threshold=0.004, code_prior_weight=1e-2)
    host = IncrementalOptimizer.from_problem(h_old, poses[:3], codes[:3], fposes[:1], **kw)
    dev = DeviceIncrementalOptimizer(d_old, poses=poses[:3], codes=codes[:3], frame_poses=fposes[:1], **kw)
    for _ in range(2):
        assert host.update() == dev.update()
    # a kept item mapped to another item (pair (0, 1) as old pair (1, 2)) is rejected and writes nothing
    before = d_new.records.clone()
    bad = [1, 0] + list(factor_of[2:])
    with pytest.raises(_lib.DfkError, match="old item"):
        dev.grow_problem(d_old, d_new, poses, codes, fposes, bad, frame_of)
    torch.cuda.synchronize()
    assert torch.equal(d_new.records, before) and dev.prob is d_old
    host.grow_problem(h_old, h_new, poses, codes, fposes, factor_of, frame_of)
    dev.grow_problem(d_old, d_new, poses, codes, fposes, factor_of, frame_of)
    torch.cuda.synchronize()
    for i, o in enumerate(factor_of):  # the kept records, copied bit for bit
        if o is None:
            continue
        nb, n0, nr = _rows(d_new, i)
        ob, o0, _ = _rows(d_old, o)
        assert torch.equal(nb[n0:n0 + nr].view(torch.int32), ob[o0:o0 + nr].view(torch.int32)), i
    firsts = []
    for step in range(3):
        rh, rd = host.update(), dev.update()
        assert rh == rd, (step, rh, rd)
        firsts.append(rd.first_column)
        assert _records_equal(torch, h_new, d_new), step
        lp, lc, lf, d = dev.linearization()
        assert _rel(lp, host.lin_poses) <= 1e-9 and _rel(lf, host.lin_frames) <= 1e-9 and _rel(d, host.delta) <= 1e-9
        ep, ec, ef = dev.estimate()
        hp, hc, hf = host.estimate()
        assert _rel(ep, hp) <= 1e-9 and _rel(ec, hc) <= 1e-9 and _rel(ef, hf) <= 1e-9
    print(f"C={cs}: first columns after the growth {firsts}")
    assert firsts[0] < 3


def test_facade_window_isam2_binary():
    """df::WindowProblem<CS>'s ISAM2 calls against the C calls they wrap (tests/cpp/window_isam2_test)"""
    exe = os.path.join(ROOT, "tests", "cpp", "window_isam2_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "WINDOW_ISAM2_TEST_OK" in out.stdout, out.stdout + out.stderr
