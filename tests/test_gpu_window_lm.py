"""The keyframe window's Levenberg-Marquardt loop in the library (dfk_window_problem_*, dfk_window_lm) on the window of
test_gpu_window_error._window: every factor kind, a tracked frame, a frame prior and a keyframe prior.

- linearize: the records bit for bit an all-stale SfmWindowProblem.linearise at three states; the buffer bit for bit
  where no prior contributes and within 1 fp32 ulp where one does (Local in fp64 on the device against numpy).
- retract against apply_update; error's parts against SfmWindowProblem.error.
- DeviceWindowOptimizer against WindowOptimizer(solve=prob.solve), with and without error, through rejected steps;
  bit for bit repeatable; marginalize_keyframe afterwards.
- malformed descriptors are rejected and write nothing.
- df::WindowProblem of the C++ facade (tests/cpp/window_lm_test)."""
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


def _scene(torch, cs):
    from test_gpu_window_error import _window
    prob, poses = _window(torch, cs)
    fposes = np.stack([se3.make_pose([0.002, -0.001, 0.003], [0.01, 0.004, -0.006], np.float64)])
    return prob, np.asarray(poses, np.float64), fposes


def _states(prob, poses, fposes, cs):
    rng = np.random.default_rng(11)
    out = []
    for it in range(3):
        codes = rng.standard_normal((3, cs)) * 0.05 * it
        out.append((poses.copy(), codes, fposes.copy()))
        poses = np.stack([se3.retract(p, rng.standard_normal(6) * 0.003, np.float64) for p in poses])
        fposes = np.stack([se3.retract(p, rng.standard_normal(6) * 0.002, np.float64) for p in fposes])
    return out


def _prior_touched(layout, prob):
    """entries of the buffer a prior adds to: the diagonal blocks and gradients of the prior keyframes, the prior
    blocks and f"""
    mask = np.zeros(layout.floats, dtype=bool)
    B = layout.B
    o = layout.offsets()
    ks = {pr.k for pr in prob._mpriors} | {k for pr in prob._kpriors for k in pr.keyframes}
    for k in ks:
        mask[k * B * B:(k + 1) * B * B] = True
        mask[o[0] + k * B:o[0] + (k + 1) * B] = True
    mask[o[2]] = True
    mask[layout.prior_offset:] = True
    return mask


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_linearize_is_the_all_stale_python_linearisation(torch_mod, cs):
    torch = torch_mod
    prob, poses, fposes = _scene(torch, cs)
    dp = prob.device_problem()
    todo = list(range(len(prob.pairs) + len(prob.geometric)))
    mask = _prior_touched(prob.layout, prob)
    states = _states(prob, poses, fposes, cs)[: (1 if cs == 128 else 3)]
    for p, c, f in states:
        want, _ = prob.linearise(p, c, todo, f)
        want = want.clone()
        rec, geo = prob.records.clone(), prob.geo_records.clone()
        prob.records.fill_(-7.0)
        prob.geo_records.fill_(-7.0)
        dp.set_state(np.concatenate([p, f]), c)
        got = dp.linearize()
        torch.cuda.synchronize()
        assert torch.equal(prob.records.view(torch.int32), rec.view(torch.int32))
        assert torch.equal(prob.geo_records.view(torch.int32), geo.view(torch.int32))
        g, w = got.cpu().numpy().view(np.int32).astype(np.int64), want.cpu().numpy().view(np.int32).astype(np.int64)
        ulp = np.abs(g - w)
        print(f"C={cs}: buffer entries differing {int((ulp > 0).sum())} of {ulp.size}, max {int(ulp.max())} ulp")
        assert ulp.max() <= 1
        assert np.all(ulp[~mask] == 0)


@pytest.mark.parametrize("cs", [8, 32])
def test_retract_matches_apply_update(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.window_opt import apply_update
    prob, poses, fposes = _scene(torch, cs)
    dp = prob.device_problem()
    rng = np.random.default_rng(3)
    codes = rng.standard_normal((3, cs)) * 0.1
    for scale in (1e-12, 1e-3, 0.3):
        dx = rng.standard_normal(prob.layout.dim) * scale
        dp.set_state(np.concatenate([poses, fposes]), codes)
        dp.retract(torch.as_tensor(dx, device="cuda"))
        p, c = dp.get_state()
        wp, wc, wf = apply_update(poses, codes, dx, cs, fposes)
        assert np.abs(p[:3] - wp).max() <= 1e-15 and np.abs(p[3:] - wf).max() <= 1e-15
        assert np.abs(c - wc).max() <= 1e-15


@pytest.mark.parametrize("cs", [8, 32])
def test_error_parts_match_the_python_error(torch_mod, cs):
    torch = torch_mod
    prob, poses, fposes = _scene(torch, cs)
    dp = prob.device_problem()
    for p, c, f in _states(prob, poses, fposes, cs):
        E, parts = prob.error(p, c, f)
        rec = prob.records.clone()
        dp.set_state(np.concatenate([p, f]), c)
        out = dp.error().cpu().numpy()
        assert torch.equal(rec, prob.records)
        assert out[1] == parts.photometric and out[2] == parts.reprojection and out[3] == parts.geometric
        assert abs(out[4] - parts.priors) <= 1e-12 * abs(parts.priors)
        assert int(out[5]) == parts.no_inliers and int(out[6]) == parts.inliers
        assert abs(out[0] - E) <= 1e-12 * abs(E)


def _lm_start(prob, poses, fposes, cs):
    """perturbed poses and a damping small enough that the Python run rejects a step"""
    from deepfactors_b200.window_opt import LMParams, WindowOptimizer
    rng = np.random.default_rng(5)
    for scale, lam in ((0.02, 1e-9), (0.04, 1e-9), (0.02, 0.0), (0.06, 1e-10)):
        p0 = poses.copy()
        p0[1:] = np.stack([se3.retract(p, rng.standard_normal(6) * scale, np.float64) for p in poses[1:]])
        prm = LMParams(iterations=6, lambda_init=lam, code_prior_weight=1e-2)
        _, _, t = WindowOptimizer(prob.layout, prob.linearise, prm, solve=prob.solve).run(p0, np.zeros((3, cs)), fposes)
        if not all(t.accepted):
            return p0, prm
    raise AssertionError("no seeded start gave a rejected step")


@pytest.mark.parametrize("cs", [8, 32])
@pytest.mark.parametrize("use_error", [False, True])
def test_device_optimizer_matches_window_optimizer(torch_mod, use_error, cs):
    torch = torch_mod
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, WindowOptimizer
    prob, poses, fposes = _scene(torch, cs)
    p0, prm = _lm_start(prob, poses, fposes, cs)
    c0 = np.zeros((3, cs))
    wp, wc, wt = WindowOptimizer(prob.layout, prob.linearise, prm, solve=prob.solve,
                                 error=prob.error if use_error else None).run(p0, c0, fposes)
    mw = prob.marginalize_keyframe(wp, wc, 0, wt.frame_poses).row
    dopt = DeviceWindowOptimizer(prob, prm, use_error=use_error)
    gp, gc, gt = dopt.run(p0, c0, fposes)
    print(f"use_error={use_error}: accepted {gt.accepted} lam {gt.lam}; energy {wt.energy} / {gt.energy}; "
          f"linearisations {wt.linearisations} / {gt.linearisations}")
    assert not all(wt.accepted)
    assert gt.accepted == wt.accepted and gt.lam == wt.lam
    assert np.allclose(gt.energy, wt.energy, rtol=1e-6, atol=0)
    assert np.abs(gp - wp).max() <= 1e-6 and np.abs(gc - wc).max() <= 1e-6
    assert np.abs(gt.frame_poses - wt.frame_poses).max() <= 1e-6
    assert gt.linearisations == wt.linearisations and gt.error_evaluations == wt.error_evaluations
    if use_error:
        assert gt.linearisations == 1 + sum(gt.accepted)
    # marginalisation still works after a device run and gives the Python run's prior
    mg = prob.marginalize_keyframe(gp, gc, 0, gt.frame_poses).row
    assert np.abs(mg - mw).max() <= 1e-6 * np.abs(mw).max()
    # two runs are bit for bit equal
    hp, hc, ht = dopt.run(p0, c0, fposes)
    assert np.array_equal(hp, gp) and np.array_equal(hc, gc) and ht.energy == gt.energy and ht.lam == gt.lam


def test_device_optimizer_rejects_a_sharded_window(torch_mod):
    torch = torch_mod
    from deepfactors_b200.window_opt import DeviceWindowOptimizer
    prob, _, _ = _scene(torch, 8)
    prob.allreduce = lambda buf: buf
    with pytest.raises(ValueError, match="all-reduce"):
        DeviceWindowOptimizer(prob)
    # also once a device problem exists
    prob.allreduce = None
    DeviceWindowOptimizer(prob)
    prob.allreduce = lambda buf: buf
    with pytest.raises(ValueError, match="all-reduce"):
        DeviceWindowOptimizer(prob)


def test_malformed_descriptors_are_rejected_and_write_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import WindowProblem, make_geometric_items, make_reprojection_items
    from deepfactors_b200.window_opt import _photometric_items, problem_slots
    cs = 8
    prob, _, _ = _scene(torch, cs)
    K, L, P = 3, prob.levels, prob._num_photometric
    zero, zc = np.zeros(7, np.float32), np.zeros(cs, np.float32)
    ends = [prob.pairs[p] for p in list(range(P)) + list(range(P + len(prob.links), len(prob.pairs)))]
    dense = [it for a, b in ends for it in _photometric_items(prob, 0, prob.kf[a], prob.kf[b] if b < K else
                                                               prob.frames[b - K].levels, zero, zero, zc, zc)]
    sl = problem_slots(K, L, prob.pairs, P, prob.links, prob.geometric)
    rep = make_reprojection_items([dict(pose0=zero, pose1=zero, code0=zc, cam=prob.cams[0],
                                        prx_orig=prob.kf[ln.k0][0]["prx_orig"], prx_jac=prob.kf[ln.k0][0]["prx_jac"],
                                        query_xy=ln.query_xy, train_xy=ln.train_xy, cauchy_delta=ln.cauchy_delta,
                                        sigma=ln.sigma) for ln in prob.links], cs)
    geo = make_geometric_items([dict(pose0=zero, pose1=zero, code0=zc, code1=zc, cam=prob.cams[0],
                                     prx0_orig=prob.kf[g.k0][0]["prx_orig"], prx0_jac=prob.kf[g.k0][0]["prx_jac"],
                                     prx1_orig=prob.kf[g.k1][0]["prx_orig"], prx1_jac=prob.kf[g.k1][0]["prx_jac"],
                                     dpt_grad1=prob.kf[g.k1][0]["dpt_grad"], points_xy=g.points_xy,
                                     huber_delta=g.huber_delta) for g in prob.geometric], cs)
    prob.records.fill_(3.0)
    prob.geo_records.fill_(3.0)

    def make(dense_items=dense, **over):
        kw = dict(dense_slots=sl["dense"], reproj_slots=sl["reproj"], geo_slots=sl["geo"],
                  kf_prior_rows=np.concatenate([np.ravel(pr.row) for pr in prob._kpriors]),
                  kf_prior_x0=np.stack([np.concatenate([pr.poses0[a], pr.codes0[a]]) for pr in prob._kpriors
                                        for a in range(len(pr.keyframes))]))
        kw.update(over)
        return WindowProblem(prob.window, prob.records, prob.geo_records, dense=prob.al.make_work_items(dense_items),
                             reproj=rep, geo=geo, **kw)

    make().close()  # the well-formed descriptor is accepted
    bad_slot = list(sl["dense"])
    bad_slot[3] = (bad_slot[3][0], 9, bad_slot[3][2], -1)
    frame_code = list(sl["dense"])
    frame_code[-1] = (1, 3, 3, -1)  # the frame's slot as code0
    bad_geo = list(sl["geo"])
    bad_geo[0] = (0, 1, 0, -1)
    bad_item = list(dense)
    bad_item[2] = dict(bad_item[2], img1=prob.kf[0][1]["img"])  # a level of the wrong size
    for kw, msg in ((dict(dense_slots=bad_slot), "dense item 3: pose1"), (dict(dense_slots=frame_code), "code0"),
                    (dict(geo_slots=bad_geo), "geometric item 0: code1"), (dict(dense_items=bad_item), "work item 2")):
        with pytest.raises(_lib.DfkError, match=msg) as e:
            make(**kw)
        assert e.value.status == _lib.DFK_ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert torch.all(prob.records == 3.0) and torch.all(prob.geo_records == 3.0)


def test_facade_window_problem_binary():
    """df::WindowProblem<CS> of the C++ facade against the C calls it wraps (tests/cpp/window_lm_test)"""
    exe = os.path.join(ROOT, "tests", "cpp", "window_lm_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "WINDOW_LM_TEST_OK" in out.stdout, out.stdout + out.stderr

