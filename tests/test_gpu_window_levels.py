"""Coarse-to-fine on the device (dfk_window_problem_set_active, dfk_window_lm_levels) on the window of
test_gpu_window_error._window: every factor kind, a tracked frame, a frame prior and a keyframe prior.

- masked linearize: records bit for bit the masked SfmWindowProblem.linearise (all stale), the buffer bit for bit where
  no prior contributes and within 1 fp32 ulp where one does; all on again is today's linearize bit for bit.
- masked error: its parts against the masked SfmWindowProblem.error.
- DeviceWindowOptimizer(schedule=...) against WindowOptimizer(solve=prob.solve, schedule=...), with and without error.
- malformed masks and schedules are rejected and write nothing.
- df::WindowProblem::SetActive / OptimizeLevels of the C++ facade (tests/cpp/window_levels_test)."""
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _masks(prob):
    """named dense masks: one level per pair, mixed levels, one pair off, every item off, every item on"""
    L, n = prob.levels, prob._num_photometric + len(prob.frames)
    lvl = np.tile(np.arange(L), n)
    pair = np.repeat(np.arange(n), L)
    return {"coarsest": lvl == L - 1, "mixed": lvl == pair % L, "pair0_off": pair != 0,
            "all_off": np.zeros(n * L, bool), "all_on": np.ones(n * L, bool)}


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_masked_linearize_is_the_masked_python_linearisation(torch_mod, cs):
    torch = torch_mod
    from test_gpu_window_lm import _prior_touched, _scene, _states
    prob, poses, fposes = _scene(torch, cs)
    dp = prob.device_problem()
    todo = list(range(len(prob.pairs) + len(prob.geometric)))
    touched = _prior_touched(prob.layout, prob)
    states = _states(prob, poses, fposes, cs)[:2]
    p, c, f = states[0]
    dp.set_state(np.concatenate([p, f]), c)
    today = dp.linearize().clone()
    today_rec = prob.records.clone()
    for name, m in _masks(prob).items():
        for p, c, f in states:
            prob.set_active(m)
            want, _ = prob.linearise(p, c, todo, f)
            want = want.clone()
            rec = prob.records.clone()
            assert torch.all(rec[torch.as_tensor(np.flatnonzero(~m), device=rec.device)] == 0)
            prob.records.fill_(-7.0)
            dp.set_active(m)
            dp.set_state(np.concatenate([p, f]), c)
            got = dp.linearize()
            torch.cuda.synchronize()
            assert torch.equal(prob.records.view(torch.int32), rec.view(torch.int32)), name
            g, w = got.cpu().numpy().view(np.int32).astype(np.int64), want.cpu().numpy().view(np.int32).astype(np.int64)
            ulp = np.abs(g - w)
            print(f"C={cs} {name}: buffer entries differing {int((ulp > 0).sum())} of {ulp.size}, max {int(ulp.max())}")
            assert ulp.max() <= 1 and np.all(ulp[~touched] == 0), name
    # all on again after other masks: today's linearize, bit for bit
    p, c, f = states[0]
    dp.set_active(np.ones_like(_masks(prob)["all_on"]))
    dp.set_state(np.concatenate([p, f]), c)
    again = dp.linearize()
    torch.cuda.synchronize()
    assert torch.equal(again.view(torch.int32), today.view(torch.int32))
    assert torch.equal(prob.records.view(torch.int32), today_rec.view(torch.int32))
    prob.set_active(None)


@pytest.mark.parametrize("cs", [8, 32])
def test_masked_error_matches_the_masked_python_error(torch_mod, cs):
    torch = torch_mod
    from test_gpu_window_lm import _scene, _states
    prob, poses, fposes = _scene(torch, cs)
    dp = prob.device_problem()
    for name, m in _masks(prob).items():
        prob.set_active(m)
        dp.set_active(m)
        for p, c, f in _states(prob, poses, fposes, cs)[:2]:
            E, parts = prob.error(p, c, f)
            dp.set_state(np.concatenate([p, f]), c)
            out = dp.error().cpu().numpy()
            assert out[1] == parts.photometric and out[2] == parts.reprojection and out[3] == parts.geometric, name
            assert abs(out[4] - parts.priors) <= 1e-12 * abs(parts.priors)
            assert int(out[5]) == parts.no_inliers and int(out[6]) == parts.inliers, name
            assert abs(out[0] - E) <= 1e-12 * abs(E)
        if name == "all_off":
            assert out[1] == 0.0 and int(out[5]) == 0 and int(out[6]) == 0
    prob.set_active(None)


@pytest.mark.parametrize("cs", [8, 32])
@pytest.mark.parametrize("use_error", [False, True])
def test_device_level_optimizer_matches_window_optimizer(torch_mod, use_error, cs):
    torch = torch_mod
    from test_gpu_window_lm import _lm_start, _scene
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, WindowOptimizer
    prob, poses, fposes = _scene(torch, cs)
    p0, prm = _lm_start(prob, poses, fposes, cs)
    prm.iterations = 8
    c0 = np.zeros((3, cs))
    n = prob._num_photometric + len(prob.frames)
    sched = prob.level_schedule([1, 2], steps_done=[0, 1, 2, 0, 3], remove_after=[False, True, False, False, True])
    assert len(sched.steps_done) == n
    wp, wc, wt = WindowOptimizer(prob.layout, prob.linearise, prm, solve=prob.solve,
                                 error=prob.error if use_error else None,
                                 set_active=prob.set_active).run(p0, c0, fposes, schedule=sched)
    mw = prob.marginalize_keyframe(wp, wc, 0, wt.frame_poses).row
    dopt = DeviceWindowOptimizer(prob, prm, use_error=use_error, schedule=sched)
    gp, gc, gt = dopt.run(p0, c0, fposes)
    print(f"use_error={use_error}: accepted {gt.accepted} lam {gt.lam}; switches {wt.switch_energy} / "
          f"{gt.switch_energy}; levels {gt.pair_levels}")
    assert gt.accepted == wt.accepted and gt.lam == wt.lam
    assert gt.pair_levels == wt.pair_levels and gt.pair_steps_done == wt.pair_steps_done
    assert len(gt.switch_energy) == len(wt.switch_energy) > 0
    assert np.allclose(gt.energy, wt.energy, rtol=1e-6, atol=0)
    assert np.allclose(gt.switch_energy, wt.switch_energy, rtol=1e-6, atol=0)
    assert np.abs(gp - wp).max() <= 1e-6 and np.abs(gc - wc).max() <= 1e-6
    assert np.abs(gt.frame_poses - wt.frame_poses).max() <= 1e-6
    assert gt.linearisations == wt.linearisations and gt.error_evaluations == wt.error_evaluations
    mg = prob.marginalize_keyframe(gp, gc, 0, gt.frame_poses).row
    assert np.abs(mg - mw).max() <= 1e-6 * np.abs(mw).max()
    # the device problem keeps the masks of the last step: its records at the final point are the masked Python
    # records bit for bit (the Python problem holds the same masks after its run), so the marginalisation calls fed
    # the device records marginalise the active factors
    dm, _ = sched.masks(gt.pair_levels[-1])
    assert np.array_equal(prob._active if prob._active is not None else np.ones_like(dm), dm) and not dm.all()
    dopt.dev.set_state(np.concatenate([gp, gt.frame_poses]), gc)
    dopt.dev.linearize()
    torch.cuda.synchronize()
    dev_rec = prob.records.clone()
    prob.linearise(gp, gc, list(range(len(prob.pairs) + len(prob.geometric))), gt.frame_poses)
    assert torch.equal(dev_rec.view(torch.int32), prob.records.view(torch.int32))
    assert torch.all(dev_rec[torch.as_tensor(np.flatnonzero(~dm), device=dev_rec.device)] == 0)
    hp, hc, ht = dopt.run(p0, c0, fposes)
    assert np.array_equal(hp, gp) and np.array_equal(hc, gc) and ht.energy == gt.energy and ht.lam == gt.lam
    assert ht.switch_energy == gt.switch_energy
    prob.set_active(None)


def test_malformed_masks_and_schedules_are_rejected(torch_mod):
    torch = torch_mod
    from test_gpu_window_lm import _scene
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, LMParams, LevelSchedule
    prob, poses, fposes = _scene(torch, 8)
    dp = prob.device_problem()
    lib, hd = _lib.lib(), prob.al._hd
    nd = dp.num_dense
    c = np.zeros((3, 8))
    dp.set_state(np.concatenate([poses, fposes]), c)
    ref = dp.linearize().clone()
    # a NULL dense mask
    with pytest.raises(_lib.DfkError) as e:
        _lib.check(hd.h, lib.dfk_window_problem_set_active(hd.h, dp.p, None, None))
    assert e.value.status == _lib.DFK_ERR_INVALID_ARG
    # error_active NULL on a problem with num_error != num_dense (here without error items)
    from deepfactors_b200.aligners import WindowProblem
    from deepfactors_b200.window_opt import problem_slots
    sl = problem_slots(3, prob.levels, prob.pairs, prob._num_photometric, prob.links, prob.geometric)
    rec, geo = prob.records.clone(), prob.geo_records.clone()
    full = prob.device_problem()
    noerr = WindowProblem(prob.window, rec, geo, dense=full._keep[2], dense_slots=sl["dense"], reproj=full._keep[3],
                          reproj_slots=sl["reproj"], geo=full._keep[4], geo_slots=sl["geo"],
                          frame_prior_kf=[pr.k for pr in prob._mpriors],
                          frame_prior_rows=np.stack([np.asarray(pr.row, np.float64) for pr in prob._mpriors]),
                          frame_prior_x0=np.stack([np.concatenate([pr.pose0, pr.code0]) for pr in prob._mpriors]),
                          kf_prior_rows=np.concatenate([np.ravel(pr.row) for pr in prob._kpriors]),
                          kf_prior_x0=np.stack([np.concatenate([pr.poses0[a], pr.codes0[a]]) for pr in prob._kpriors
                                                for a in range(len(pr.keyframes))]))
    assert noerr.num_error == 0 and noerr.num_dense == nd
    half = np.zeros(nd, np.uint8)
    half[::2] = 1
    with pytest.raises(_lib.DfkError, match="error_active may be NULL only") as e:
        _lib.check(hd.h, lib.dfk_window_problem_set_active(hd.h, noerr.p, half.ctypes.data_as(_lib.C.c_void_p), None))
    assert e.value.status == _lib.DFK_ERR_INVALID_ARG
    with pytest.raises(ValueError):
        noerr.set_active(half.astype(bool))
    noerr.set_state(np.concatenate([poses, fposes]), c)
    got = noerr.linearize()
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int32), ref.view(torch.int32))  # the rejected call left every item active
    noerr.close()
    with pytest.raises(ValueError):
        dp.set_active(np.ones(nd - 1, bool))
    with pytest.raises(ValueError):
        prob.set_active(np.ones(nd + 1, bool))
    good = prob.level_schedule([1, 1])
    prm = LMParams(iterations=3)
    bad = [LevelSchedule(iters=[1, -1], item_level=good.item_level, item_pair=good.item_pair,
                         steps_done=good.steps_done, remove_after=good.remove_after),
           LevelSchedule(iters=[1, 1], item_level=[2] + list(good.item_level[1:]), item_pair=good.item_pair,
                         steps_done=good.steps_done, remove_after=good.remove_after),
           LevelSchedule(iters=[1, 1], item_level=good.item_level, item_pair=good.item_pair,
                         steps_done=[-1] + list(good.steps_done[1:]), remove_after=good.remove_after),
           LevelSchedule(iters=[1, 1], item_level=good.item_level, item_pair=good.item_pair,
                         steps_done=list(good.steps_done) + [0], remove_after=list(good.remove_after) + [False]),
           LevelSchedule(iters=[1, 1], item_level=good.item_level, item_pair=good.item_pair,
                         steps_done=good.steps_done, remove_after=good.remove_after, error_pair=[99] * nd)]
    p_before, c_before = dp.get_state()
    for sc in bad:
        with pytest.raises(_lib.DfkError) as e:
            dp.lm_levels(prm, sc)
        assert e.value.status == _lib.DFK_ERR_INVALID_ARG
    p_after, c_after = dp.get_state()
    assert np.array_equal(p_before, p_after) and np.array_equal(c_before, c_after)
    # the rejected calls left the mask (all on) as it was
    again = dp.linearize()
    torch.cuda.synchronize()
    assert torch.equal(again.view(torch.int32), ref.view(torch.int32))
    # a sharded window stays rejected
    # wrong lengths and a pairing other than the window's are rejected before the C call reads the arrays
    import dataclasses
    for over in (dict(item_level=list(good.item_level)[:-1]), dict(remove_after=list(good.remove_after)[:-1]),
                 dict(error_level=[0] * (nd - 1)), dict(item_pair=list(reversed(good.item_pair)))):
        with pytest.raises(ValueError):
            dp.lm_levels(prm, dataclasses.replace(good, **over))
    prob.allreduce = lambda buf: buf
    with pytest.raises(ValueError, match="all-reduce"):
        DeviceWindowOptimizer(prob, schedule=good)
    prob.allreduce = None


def test_facade_window_levels_binary():
    """df::WindowProblem<CS>::SetActive / OptimizeLevels against the C calls they wrap (tests/cpp/window_levels_test)"""
    exe = os.path.join(ROOT, "tests", "cpp", "window_levels_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "WINDOW_LEVELS_TEST_OK" in out.stdout, out.stdout + out.stderr
