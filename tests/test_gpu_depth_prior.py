"""Depth priors (DepthPriorFactor) on the device: the batched linearisation and error, the window's in-place addition and
SfmWindowProblem with depth priors.

- DepthPriorLinearizeBatch per entry against the fp64 DepthAligner reference (system_accuracy.depth_reference) with
  the bars of system_accuracy.py (Jtr: the small-item bar 1e-5 below 256 pixels), at C = 8, 32 and 128, one mixed batch of 1x1, 37x5, 97x33, 80x60 and 640x480 items
  with padded pitches, plus the one-signed target of the DepthAligner test; inliers exactly W * H.
- Two calls agree bit for bit, a permuted batch gives every item's record bit for bit, the error batch's residual is the
  record's bit for bit, malformed batches are rejected and write nothing.
- Window.add_depth_priors against the numpy mirror (WindowBlocks.add_depth_priors); every other entry untouched; zero
  priors touch nothing.
- SfmWindowProblem with depth priors on the window of test_gpu_window_error: linearise = the window without them plus
  the mirror's addition, error's depth part and E against the linearisation's f; keyframe marginalisation with a depth
  prior elsewhere bit for bit the window without it, and with one on m against a numpy Schur complement.
- The window problem (dfk_window_problem_set_depth_priors): linearize against the all-stale SfmWindowProblem.linearise,
  error_ex's parts against SfmWindowProblem.error, DeviceWindowOptimizer against WindowOptimizer(solve=prob.solve) with
  and without error, and with a level schedule (the depth priors stay active at every level).
- df::DepthPriorFactor of the C++ factor header (tests/cpp/depth_prior_test)."""
import ctypes as C

import numpy as np
import pytest

from deepfactors_b200 import _lib, se3
from system_accuracy import CODE_NAMES, JTR_BAR, assert_system_close, depth_reference
from test_gpu_tracker_depth_accuracy import upload

pytestmark = pytest.mark.gpu

SIZES = [(1, 1), (37, 5), (97, 33), (80, 60), (640, 480)]


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _case(cs, w, h, seed, one_signed=False, avg=2.0):
    """code, target, prx_orig, prx_jac (host); the one-signed case has non-negative Jacobian columns and code and the
    target one-signedly behind the decoded depth, so nothing in Jtr cancels"""
    from oracle import oracle as orc
    rng = np.random.default_rng(seed)
    prx = (0.3 + 0.4 * rng.random((h, w))).astype(np.float32)
    # the decode's dot product keeps the same spread at every C (std 0.017), so no proximity comes near 0 (a depth
    # near infinity, whose fp32 decode would swamp the comparison)
    jac = (rng.standard_normal((h, w, cs)) * (0.02 * np.sqrt(8.0 / cs))).astype(np.float32)
    code = (rng.standard_normal(cs) * 0.3).astype(np.float32)
    if one_signed:
        jac, code = np.abs(jac), np.abs(code)
    dpt = orc.update_depth(code, prx, jac, avg)
    if one_signed:
        tgt = (dpt * np.float32(1.1)).astype(np.float32)
    else:
        tgt = (dpt + np.float32(0.05) * rng.standard_normal((h, w)).astype(np.float32)).astype(np.float32)
    return code, tgt, prx, jac


def _items(torch, cases, extra=3):
    return [dict(code=c, target_dpt=upload(torch, t, extra), prx_orig=upload(torch, p, extra + 1),
                 prx_jac=upload(torch, j, extra)) for c, t, p, j in cases]


def _unpack(rec, cs):
    """a DFK_DEPTH_RECORD_FLOATS record as the code-only JTJJrReductionItem"""
    from deepfactors_b200.aligners import JTJJrReductionItem
    nh = cs * (cs + 1) // 2
    rec = np.ascontiguousarray(rec, dtype=np.float32)
    return JTJJrReductionItem(rec[:nh].copy(), rec[nh:nh + cs].copy(), float(rec[nh + cs]),
                              int(rec[nh + cs + 1:nh + cs + 2].view(np.uint32)[0]))


def _aligner(cs, avg=2.0):
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    return SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(avg_dpt=avg)))


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_batch_records_against_fp64(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.aligners import DepthPriorLinearizeBatch
    cases = [_case(cs, w, h, seed=cs + i) for i, (w, h) in enumerate(SIZES)]
    cases.append(_case(cs, 640, 480, seed=99, one_signed=True))
    al = _aligner(cs)
    rec = DepthPriorLinearizeBatch(al, _items(torch, cases)).cpu().numpy()
    worst = (0.0, 0.0)
    for i, (code, tgt, prx, jac) in enumerate(cases):
        h, w = tgt.shape
        got = _unpack(rec[i], cs)
        assert got.inliers == w * h
        ref = depth_reference(code, tgt, prx, jac, 2.0)
        # below 256 pixels the fp32 decode of single pixels (diff = target - dpt is a few percent of dpt; the per-pixel
        # arithmetic of dfk_depth_run_step) does not average out in the cancelling Jtr: the small-item bar 1e-5
        e = assert_system_close(got, ref, ref.S, ref.B, f"depth prior batch C={cs} {w}x{h} item {i}", names=CODE_NAMES,
                                jtr_bar=JTR_BAR if w * h >= 256 else 1e-5)
        worst = (max(worst[0], e["h"]), max(worst[1], e["jtr"]))
    print(f"C={cs}: worst JtJ {worst[0]:.2e} of S, worst Jtr {worst[1]:.2e} of B over the batch")


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_batch_is_deterministic_and_independent_of_the_batch(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.aligners import DepthPriorErrorBatch, DepthPriorLinearizeBatch
    cases = [_case(cs, w, h, seed=7 * cs + i) for i, (w, h) in enumerate(SIZES)]
    al = _aligner(cs)
    items = _items(torch, cases)
    a = DepthPriorLinearizeBatch(al, items).clone()
    b = DepthPriorLinearizeBatch(al, items)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    perm = [3, 0, 4, 2, 1]
    p = DepthPriorLinearizeBatch(al, [items[i] for i in perm])
    for j, i in enumerate(perm):
        assert torch.equal(p[j].view(torch.int32), a[i].view(torch.int32))
    one = DepthPriorLinearizeBatch(al, [items[2]])
    assert torch.equal(one[0].view(torch.int32), a[2].view(torch.int32))
    err = DepthPriorErrorBatch(al, items)
    nh = cs * (cs + 1) // 2
    assert torch.equal(err[:, 0].contiguous().view(torch.int32), a[:, nh + cs].contiguous().view(torch.int32))
    assert torch.equal(err[:, 1].contiguous().view(torch.int32), a[:, nh + cs + 1].contiguous().view(torch.int32))


def test_malformed_batches_are_rejected_and_write_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import make_depth_prior_items
    cs = 8
    al = _aligner(cs)
    good = _items(torch, [_case(cs, 37, 5, seed=1), _case(cs, 80, 60, seed=2)])
    L, h = _lib.lib(), al.handle
    rec = _lib.depth_record_floats(cs)
    out = torch.full((2, rec), -3.0, device="cuda")

    def call(arr, n, code_size=cs, fn="dfk_depth_prior_linearize_batch"):
        st = getattr(L, fn)(h, arr, n, code_size, C.c_void_p(out.data_ptr()))
        torch.cuda.synchronize()
        return st

    for fn in ("dfk_depth_prior_linearize_batch", "dfk_depth_prior_error_batch"):
        arr = make_depth_prior_items(good, cs)
        arr[1].code = C.POINTER(C.c_float)()
        assert call(arr, 2, fn=fn) == _lib.DFK_ERR_INVALID_ARG
        arr = make_depth_prior_items(good, cs)
        arr[0].prx_orig.width = 36
        assert call(arr, 2, fn=fn) == _lib.DFK_ERR_INVALID_ARG
        arr = make_depth_prior_items(good, cs)
        arr[1].prx_jac.pitch_bytes = 4 * cs * 80 - 4
        assert call(arr, 2, fn=fn) == _lib.DFK_ERR_INVALID_ARG
        arr = make_depth_prior_items(good, cs)
        arr[0].target_dpt.pitch_bytes = 4 * 37 + 2
        assert call(arr, 2, fn=fn) == _lib.DFK_ERR_INVALID_ARG
        assert call(make_depth_prior_items(good, cs), 0, fn=fn) == _lib.DFK_ERR_INVALID_ARG
        assert call(make_depth_prior_items(good, cs), 65536, fn=fn) == _lib.DFK_ERR_INVALID_ARG
        assert call(make_depth_prior_items(good, cs), 2, code_size=12, fn=fn) == _lib.DFK_ERR_UNSUPPORTED
        assert bool((out == -3.0).all())


def _window(al, K=4, cs=8):
    from deepfactors_b200.aligners import Window
    pairs = [(0, 1), (1, 2), (2, 3), (3, 0)]
    return Window(al, K, pairs, [0, 0, 1, 2, 3], [(64, 48), (32, 24), (64, 48), (64, 48), (64, 48)])


@pytest.mark.parametrize("cs", [8, 32])
def test_window_add_depth_priors_matches_the_mirror(torch_mod, cs):
    torch = torch_mod
    al = _aligner(cs)
    win = _window(al, cs=cs)
    lay = win.layout
    rng = np.random.default_rng(cs)
    base = rng.standard_normal(win.floats).astype(np.float32)
    rec = _lib.depth_record_floats(cs)
    records = (rng.standard_normal((5, rec)) * 10).astype(np.float32)
    kf, sigma, lp = [2, 0, 2], [0.5, 1.3, 0.07], [0, 2, 3, 5]
    buf = torch.from_numpy(base.copy()).cuda()
    win.add_depth_priors(buf, kf, sigma, lp, torch.from_numpy(records).cuda())
    got = buf.cpu().numpy()
    want = lay.add_depth_priors(base.copy(), kf, sigma, lp, records)
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    print(f"C={cs}: {int((ulp > 0).sum())} entries differ from the mirror, max {int(ulp.max())} ulp")
    assert ulp.max() <= 1
    B = lay.B
    touched = np.zeros(win.floats, dtype=bool)
    o_g, _, o_t = lay.offsets()
    for k in set(kf):
        touched[k * B * B:(k + 1) * B * B].reshape(B, B)[6:, 6:] = True
        touched[o_g + k * B + 6:o_g + (k + 1) * B] = True
    touched[o_t] = True
    assert np.array_equal(got[~touched].view(np.int32), base[~touched].view(np.int32))
    assert not np.array_equal(got[touched], base[touched])
    # zero priors: nothing written
    buf2 = torch.from_numpy(base.copy()).cuda()
    win.add_depth_priors(buf2, [], [], [0], torch.zeros(1, device="cuda"))
    assert np.array_equal(buf2.cpu().numpy().view(np.int32), base.view(np.int32))
    # rejected: keyframe outside, sigma <= 0 or not finite, level_ptr not increasing
    from deepfactors_b200._lib import DfkError
    for bad in (dict(kf=[4, 0, 2]), dict(sigma=[0.5, 0.0, 1.0]), dict(sigma=[0.5, float("nan"), 1.0]),
                dict(lp=[0, 2, 2, 5]), dict(lp=[1, 2, 3, 5])):
        args = dict(kf=kf, sigma=sigma, lp=lp)
        args.update(bad)
        buf3 = torch.from_numpy(base.copy()).cuda()
        with pytest.raises(DfkError):
            win.add_depth_priors(buf3, args["kf"], args["sigma"], args["lp"], torch.from_numpy(records).cuda())
        assert np.array_equal(buf3.cpu().numpy().view(np.int32), base.view(np.int32))


def _depth_window(torch, cs, on=(0, 2)):
    """test_gpu_window_error's window (every factor kind, a tracked frame, a frame and a keyframe prior) with depth
    priors on the keyframes `on`: targets 5 % behind the depth decoded at a small code, plus noise"""
    from test_gpu_window_error import _window
    from deepfactors_b200.window_opt import SfmWindowProblem, make_depth_prior
    from oracle import oracle as orc
    prob, poses = _window(torch, cs)
    rng = np.random.default_rng(23)
    dps = []
    for i, k in enumerate(on):
        lv = prob.kf[k][0]
        code = (rng.standard_normal(cs) * 0.05).astype(np.float32)
        d = orc.update_depth(code, lv["prx_orig"].cpu().numpy(), lv["prx_jac"].cpu().numpy(), 2.0)
        tgt = (d * np.float32(1.05) + np.float32(0.01) * rng.standard_normal(d.shape).astype(np.float32))
        dps.append(make_depth_prior(k, torch.from_numpy(tgt.astype(np.float32)).cuda(), 0.5 + i, prob.levels))
    dprob = SfmWindowProblem(prob.al, prob.cams, prob.kf, prob.pairs[:prob._num_photometric], links=prob.links,
                             geometric=prob.geometric, frames=prob.frames, priors=prob.priors, depth_priors=dps)
    fposes = np.stack([se3.make_pose([0.002, -0.001, 0.003], [0.01, 0.004, -0.006], np.float64)])
    return prob, dprob, np.asarray(poses, np.float64), fposes


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_window_problem_linearise_and_error(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.aligners import DepthPriorLinearizeBatch
    from deepfactors_b200.window_opt import LMParams, WindowOptimizer, _depth_prior_items
    prob, dprob, poses, fposes = _depth_window(torch, cs)
    rng = np.random.default_rng(4)
    todo = list(range(len(prob.pairs) + len(prob.geometric)))
    for it in range(1 if cs == 128 else 2):
        codes = rng.standard_normal((3, cs)) * 0.03 * it
        got, _ = dprob.linearise(poses, codes, todo, fposes)
        got = got.cpu().numpy()
        recs = DepthPriorLinearizeBatch(dprob.al, _depth_prior_items(dprob, dprob.depth_priors, codes)).cpu().numpy()
        assert np.array_equal(recs.view(np.int32), dprob.depth_records.cpu().numpy().view(np.int32))
        # the order of an unsharded linearise: the assembly, the frame and keyframe priors, then the depth priors
        wt = dprob.window.assemble(dprob.records, geo_records=dprob.geo_records)
        dprob.window.add_priors(wt, [pr.k for pr in dprob._mpriors], dprob._prior_rows,
                                torch.as_tensor(dprob._deltas(poses, codes), device="cuda"))
        dprob.window.add_keyframe_priors(wt, dprob._kprior_rows,
                                         torch.as_tensor(dprob._kf_deltas(poses, codes), device="cuda"))
        want = dprob.layout.add_depth_priors(wt.cpu().numpy().copy(), [d.k for d in dprob.depth_priors],
                                             [d.sigma for d in dprob.depth_priors], dprob._depth_level_ptr, recs)
        ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        print(f"C={cs} point {it}: {int((ulp > 0).sum())} entries differ from the mirror, max {int(ulp.max())} ulp")
        assert ulp.max() <= 1
        # error: the depth part from the error batch, E against the linearisation's energy
        E, parts = dprob.error(poses, codes, fposes)
        _, p0 = prob.error(poses, codes, fposes)
        nh = cs * (cs + 1) // 2
        dep = sum(float(np.float64(recs[i * dprob.levels + l, nh + cs]) / np.float64(np.float32(d.sigma)) ** 2)
                  for i, d in enumerate(dprob.depth_priors) for l in range(dprob.levels))
        assert parts.depth > 0 and abs(parts.depth - dep) <= 1e-12 * dep
        assert parts.photometric == p0.photometric and parts.priors == p0.priors
        f = WindowOptimizer(dprob.layout, dprob.linearise, LMParams())._energy(torch.from_numpy(got).cuda(), codes)
        print(f"C={cs} point {it}: E {E:.9e} f {f:.9e} depth part {parts.depth:.6e}")
        assert abs(E - f) <= 1e-5 * abs(f)


def _prior_touched(layout, prob):
    """entries the frame / keyframe priors and the depth priors add to (the window problem forms the priors' deltas
    Local(x0, x) on the device in fp64: within 1 fp32 ulp of numpy's there)"""
    from test_gpu_window_lm import _prior_touched as touched
    mask = touched(layout, prob)
    B, o_g = layout.B, layout.offsets()[0]
    for d in prob.depth_priors:
        mask[d.k * B * B:(d.k + 1) * B * B] = True
        mask[o_g + d.k * B:o_g + (d.k + 1) * B] = True
    return mask


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_device_problem_linearize_and_error_ex(torch_mod, cs):
    """dfk_window_problem_set_depth_priors: linearize against the all-stale SfmWindowProblem.linearise (bit for bit
    where no prior contributes, <= 1 ulp where one does), error_ex's parts against SfmWindowProblem.error"""
    torch = torch_mod
    _, dprob, poses, fposes = _depth_window(torch, cs, on=(1, 2))
    dp = dprob.device_problem()
    todo = list(range(len(dprob.pairs) + len(dprob.geometric)))
    mask = _prior_touched(dprob.layout, dprob)
    rng = np.random.default_rng(8)
    for it in range(1 if cs == 128 else 2):
        codes = rng.standard_normal((3, cs)) * 0.03 * it
        want, _ = dprob.linearise(poses, codes, todo, fposes)
        want = want.cpu().numpy().copy()
        dp.set_state(np.concatenate([poses, fposes]), codes)
        got = dp.linearize().cpu().numpy()
        ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        print(f"C={cs} point {it}: {int((ulp > 0).sum())} entries differ, max {int(ulp.max())} ulp")
        assert ulp.max() <= 1 and np.all(ulp[~mask] == 0)
        E, parts = dprob.error(poses, codes, fposes)
        out = dp.error_ex().cpu().numpy()
        assert out[7] == parts.depth > 0
        assert out[1] == parts.photometric and out[2] == parts.reprojection and out[3] == parts.geometric
        assert abs(out[4] - parts.priors) <= 1e-12 * abs(parts.priors)
        assert abs(out[0] - E) <= 1e-12 * abs(E)
        assert np.array_equal(dp.error().cpu().numpy(), out[:7])


def test_device_problem_without_depth_priors_is_unchanged(torch_mod):
    torch = torch_mod
    prob, _, poses, fposes = _depth_window(torch, 8)
    dp = prob.device_problem()
    dp.set_state(np.concatenate([poses, fposes]), np.zeros((3, 8)))
    out = dp.error_ex().cpu().numpy()
    assert out[7] == 0.0 and np.array_equal(out[:7], dp.error().cpu().numpy())


@pytest.mark.parametrize("cs", [8, 32])
@pytest.mark.parametrize("use_error", [False, True])
def test_device_optimizer_with_depth_priors_matches_window_optimizer(torch_mod, use_error, cs):
    torch = torch_mod
    from test_gpu_window_lm import _lm_start
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, WindowOptimizer
    prob, dprob, poses, fposes = _depth_window(torch, cs, on=(1, 2))
    p0, prm = _lm_start(prob, poses, fposes, cs)
    c0 = np.zeros((3, cs))
    wp, wc, wt = WindowOptimizer(dprob.layout, dprob.linearise, prm, solve=dprob.solve,
                                 error=dprob.error if use_error else None).run(p0, c0, fposes)
    gp, gc, gt = DeviceWindowOptimizer(dprob, prm, use_error=use_error).run(p0, c0, fposes)
    print(f"use_error={use_error}: accepted {gt.accepted} lam {gt.lam}; energy {wt.energy} / {gt.energy}")
    assert any(gt.accepted) and gt.energy[-1] < gt.energy[0]
    assert gt.accepted == wt.accepted and gt.lam == wt.lam
    assert np.allclose(gt.energy, wt.energy, rtol=1e-6, atol=0)
    assert np.abs(gp - wp).max() <= 1e-6 and np.abs(gc - wc).max() <= 1e-6
    assert gt.linearisations == wt.linearisations and gt.error_evaluations == wt.error_evaluations


@pytest.mark.parametrize("use_error", [False, True])
def test_level_schedule_keeps_the_depth_priors_active(torch_mod, use_error):
    torch = torch_mod
    from test_gpu_window_lm import _lm_start
    from deepfactors_b200.window_opt import DeviceWindowOptimizer, WindowOptimizer
    cs = 8
    prob, dprob, poses, fposes = _depth_window(torch, cs, on=(1, 2))
    p0, prm = _lm_start(prob, poses, fposes, cs)
    prm.iterations = 8
    c0 = np.zeros((3, cs))
    sched = dprob.level_schedule([1, 2], steps_done=[0, 1, 2, 0, 3], remove_after=[False, True, False, False, True])
    wp, wc, wt = WindowOptimizer(dprob.layout, dprob.linearise, prm, solve=dprob.solve,
                                 error=dprob.error if use_error else None,
                                 set_active=dprob.set_active).run(p0, c0, fposes, schedule=sched)
    dopt = DeviceWindowOptimizer(dprob, prm, use_error=use_error, schedule=sched)
    gp, gc, gt = dopt.run(p0, c0, fposes)
    assert gt.accepted == wt.accepted and gt.lam == wt.lam and gt.pair_levels == wt.pair_levels
    assert np.allclose(gt.energy, wt.energy, rtol=1e-6, atol=0)
    assert np.allclose(gt.switch_energy, wt.switch_energy, rtol=1e-6, atol=0)
    assert np.abs(gp - wp).max() <= 1e-6 and np.abs(gc - wc).max() <= 1e-6
    # under the last step's masks the depth part is still the whole depth-prior energy at the final point
    _, parts = dprob.error(gp, gc, gt.frame_poses)
    dopt.dev.set_state(np.concatenate([gp, gt.frame_poses]), gc)
    assert dopt.dev.error_ex().cpu().numpy()[7] == parts.depth > 0
    dprob.set_active(None)


def test_marginalise_keyframe_with_depth_priors(torch_mod):
    torch = torch_mod
    cs = 8
    prob, dprob, poses, fposes = _depth_window(torch, cs, on=(2,))
    codes = np.random.default_rng(2).standard_normal((3, cs)) * 0.02
    # no depth prior on m: bit for bit the window without depth priors
    a = prob.marginalize_keyframe(poses, codes, 0, fposes).row
    b = dprob.marginalize_keyframe(poses, codes, 0, fposes).row
    assert np.array_equal(a, b)
    # a depth prior on m: its code block, gradient and constant enter the local system before the elimination, so the
    # prior's f0 grows by at most the prior's energy and G stays symmetric
    _, dprob2, _, _ = _depth_window(torch, cs, on=(0,))
    c = dprob2.marginalize_keyframe(poses, codes, 0, fposes).row
    assert not np.array_equal(a, c)
    nb = len(dprob2.window.blanket(0)) * dprob2.layout.B
    G = c[:nb * nb].reshape(nb, nb)
    assert np.abs(G - G.T).max() <= 1e-9 * np.abs(G).max()
    # numpy Schur reference: the depth prior adds (G_d, g_d, f_d) to m's own block, gradient and f, so the prior changes
    # by Schur(H_mm + G_d, g_m + g_d) - Schur(H_mm, g_m) plus f_d, with H_mm, H_Nm, g_m from the dense linearisation
    from deepfactors_b200.window_opt import depth_prior_rows
    lay, B = prob.layout, prob.layout.B
    buf, _ = prob.linearise(poses, codes, list(range(len(prob.pairs) + len(prob.geometric))), fposes)
    H, g, _, _ = lay.to_dense(buf.cpu().numpy())
    nbl = dprob2.window.blanket(0)
    M = np.arange(B)
    N = np.concatenate([np.arange(k * B, (k + 1) * B) for k in nbl])
    Hmm, HNm, gm, gN = H[np.ix_(M, M)], H[np.ix_(N, M)], g[M], g[N]
    recs = dprob2._linearise_depth_priors(codes, records=torch.empty_like(dprob2.depth_records))
    row = depth_prior_rows(recs.cpu().numpy(), [dprob2.depth_priors[0].sigma], dprob2.levels, cs)[0]
    Gd, gd, fd = row[:B * B].reshape(B, B), row[B * B:B * B + B], row[-1]

    def schur(Hm, gmm):
        X = np.linalg.solve(Hm, np.concatenate([HNm.T, gmm[:, None]], axis=1))
        return -HNm @ X[:, :-1], -HNm @ X[:, -1], -gmm @ X[:, -1]

    G1, g1, f1 = schur(Hmm + Gd, gm + gd)
    G0, g0, f0 = schur(Hmm, gm)
    nn = N.size
    for what, got, want in (("G", (c - a)[:nn * nn], (G1 - G0).ravel()), ("g", (c - a)[nn * nn:nn * nn + nn], g1 - g0),
                            ("f0", (c - a)[-1:], np.array([f1 - f0 + fd]))):
        err = np.abs(got - want).max() / np.abs(want).max()
        print(f"marginal change {what}: {err:.2e} of its largest entry")
        assert err <= 1e-4, what
    nxt = dprob2.without_keyframe(0, dprob2.marginalize_keyframe(poses, codes, 0, fposes))
    assert nxt.depth_priors == []


def test_facade_depth_prior_binary(torch_mod):
    """df::DepthPriorFactor + WindowSystem::AddDepthPrior through the C++ factor header"""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "cpp", "depth_prior_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "DEPTH_PRIOR_TEST_OK" in out.stdout, out.stdout + out.stderr
