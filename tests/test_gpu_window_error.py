"""The error() half of the factors on the device and the window energy without a linearisation.

- dfk_update_depth_batch: every item bit for bit dfk_update_depth, at C = 8 ... 128 and an odd C, 1x1 to 1280x960,
  pitched and misaligned views, mixed sizes in one batch.
- dfk_sfm_evaluate_error_batch: every item bit for bit dfk_sfm_evaluate_error, whatever else is in the batch; inliers
  exact against the fp32 oracle and the residual against fp64 at the bar of test_sfm_evaluate_error_matches_oracle.
- dfk_reprojection_error_batch / dfk_sparse_geometric_error_batch: b^T b bit for bit the residual of the records
  kernels' record, and against sum b^2 of the fp64 oracle rows.
- SfmWindowProblem.error on a window with every factor kind, a tracked frame and both prior kinds: E equals the
  linearisation's f, and LM with and without `error` walks the same steps.
- df::SfmAligner::EvaluateErrorBatch of the C++ facade (tests/cpp/error_batch_test)."""
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib, se3, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def pitched(torch, arr, extra_px=0, offset_floats=0):
    """host [H, W(, K)] -> device view whose rows are padded by extra_px pixels, starting offset_floats into its buffer"""
    a = np.ascontiguousarray(arr, dtype=np.float32)
    h, w = a.shape[:2]
    k = a.shape[2] if a.ndim == 3 else 1
    row = (w + extra_px) * k + offset_floats
    buf = torch.zeros((h, row), dtype=torch.float32, device="cuda")
    buf[:, offset_floats:offset_floats + w * k] = torch.from_numpy(a.reshape(h, w * k)).cuda()
    return torch.as_strided(buf, (h, w, k), (row, k, 1), offset_floats) if a.ndim == 3 else \
        torch.as_strided(buf, (h, w), (row, 1), offset_floats)


def bits(t):
    import torch
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------ dfk_update_depth_batch
@pytest.mark.parametrize("cs", [8, 16, 32, 64, 128, 7])
def test_update_depth_batch_is_the_single_call_bit_for_bit(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner, UpdateDepth
    al = SfmAligner(cs)
    gen = torch.Generator(device="cuda").manual_seed(cs)
    rng = np.random.default_rng(cs)
    items = []
    # (w, h, extra pixels per row, misaligned code-Jacobian view); 1280 x 960 only where it fits comfortably
    sizes = [(1, 1, 0, False), (7, 3, 2, False), (160, 120, 3, False), (97, 61, 0, True), (640, 480, 0, False)]
    if cs <= 32:
        sizes.append((1280, 960, 1, False))
    for w, h, extra, mis in sizes:
        jac = torch.zeros((h, (w + extra) * cs + (1 if mis else 0)), device="cuda")
        jac.normal_(0.0, 0.02, generator=gen)
        jac = torch.as_strided(jac, (h, w, cs), (jac.shape[1], cs, 1), 1 if mis else 0)
        prx = torch.empty((h, w + extra), device="cuda").uniform_(0.3, 0.9, generator=gen)[:, :w]
        dpt = torch.full((h, w + extra), 7.0, device="cuda")[:, :w]
        items.append(dict(code=(rng.standard_normal(cs) * 0.5).astype(np.float32), prx_orig=prx, prx_jac=jac, dpt=dpt))
    al.UpdateDepthBatch(items + items[:2])  # a repeated item writes the same depth twice
    for it in items:
        want = torch.full_like(it["dpt"], -1.0)
        UpdateDepth(it["code"], it["prx_orig"], it["prx_jac"], 2.0, want)
        torch.cuda.synchronize()
        assert torch.equal(bits(it["dpt"]), bits(want)), (cs, tuple(it["dpt"].shape))


def test_update_depth_batch_rejects_bad_items_and_writes_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(8)
    dpt = torch.full((4, 5), 3.0, device="cuda")
    good = dict(code=np.zeros(8, np.float32), prx_orig=torch.ones((4, 5), device="cuda"),
                prx_jac=torch.zeros((4, 5, 8), device="cuda"), dpt=dpt)
    bad = dict(good, prx_orig=torch.ones((4, 6), device="cuda"))
    with pytest.raises(_lib.DfkError, match="item 1"):
        al.UpdateDepthBatch([good, bad])
    torch.cuda.synchronize()
    assert torch.all(dpt == 3.0)


# ------------------------------------------------------------------------------------------ dfk_sfm_evaluate_error_batch
def _error_items(torch, cs):
    """(work-item dicts, host levels): 320x240 and 97x61 levels, pitched and not, a cropped camera, an item whose frame
    lies far behind (no overlap), a 1x1 item and a tiny one"""
    pair = synth.make_pair(320, 240, cs, 2, seed=9, code_sigma=0.5)
    small = synth.make_level(97, 61, cs, seed=3)
    one = synth.make_level(1, 1, cs, seed=4)
    tiny = synth.make_level(5, 4, cs, seed=5)
    far = se3.make_pose([0, 0, 0], [0, 0, 30.0], np.float32)  # the scene falls behind the frame
    out = []
    for k, (L, extra, pose1) in enumerate([(pair.levels[0], 3, pair.pose1), (pair.levels[1], 0, pair.pose1),
                                           (small, 1, pair.pose1), (pair.levels[0], 0, far), (one, 0, pair.pose1),
                                           (tiny, 2, se3.identity()), (small, 0, se3.identity())]):
        cam = L.cam
        if k == 2:  # a camera viewport smaller than the views
            cam = synth.Camera(cam.fx, cam.fy, cam.u0, cam.v0, cam.width - 9, cam.height - 5)
        dev = dict(img0=pitched(torch, L.img0, extra), img1=pitched(torch, L.img1, extra), dpt0=pitched(torch, L.dpt0),
                   valid0=pitched(torch, np.zeros_like(L.img0)), prx0_jac=pitched(torch, L.prx_jac),
                   grad1=pitched(torch, L.grad1, extra))
        out.append((dict(pose0=pair.pose0, pose1=pose1, cam=cam, **dev), L))
    return out


def _single(al, it):
    r = al.EvaluateError(it["pose0"], it["pose1"], it["cam"], it["img0"], it["img1"], it["dpt0"], None, None)
    return np.float32(r.residual), r.inliers


@pytest.mark.parametrize("delta", [0.1, 0.5])
def test_evaluate_error_batch_is_the_single_call_bit_for_bit(torch_mod, delta):
    torch = torch_mod
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    cs = 32
    al = SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(huber_delta=delta)))
    its = [it for it, _ in _error_items(torch, cs)]
    want = [_single(al, it) for it in its]
    assert want[3][1] == 0 and want[4][1] == 0, "no overlap / a 1x1 image (outside the border) have no inliers"
    assert want[5][1] > 0 and want[0][1] > 1000
    orders = [list(range(len(its))), list(reversed(range(len(its)))), [2, 0, 2, 5, 1, 6, 3, 4, 0]]
    for order in orders:
        out = al.EvaluateErrorBatch(al.make_work_items([its[i] for i in order]))
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        assert got.shape == (len(order), 2)
        for row, i in zip(got, order):
            assert row[0].view(np.uint32) == want[i][0].view(np.uint32), (order, i, row[0], want[i][0])
            assert int(row[1:2].view(np.uint32)[0]) == want[i][1], (order, i)


def test_evaluate_error_batch_against_the_oracle(torch_mod, oracle):
    torch = torch_mod
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    cs = 32
    items = _error_items(torch, cs)
    for delta in (0.1, 0.5):
        al = SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(huber_delta=delta)))
        got = al.EvaluateErrorBatch(al.make_work_items([it for it, _ in items])).cpu().numpy()
        for (it, L), row in zip(items, got):
            c = it["cam"]
            cam = synth.Camera(c.fx, c.fy, c.u0, c.v0, c.width, c.height)
            p = oracle.default_params(huber_delta=delta)
            _, i32 = oracle.sfm_evaluate_error(it["pose0"], it["pose1"], cam, L.img0, L.img1, L.dpt0, p, precision="f32")
            r64, _ = oracle.sfm_evaluate_error(it["pose0"], it["pose1"], cam, L.img0, L.img1, L.dpt0, p, precision="f64")
            inl = int(row[1:2].view(np.uint32)[0])
            assert inl == i32
            assert abs(float(row[0]) - r64) <= 1e-5 * r64


def test_evaluate_error_batch_rejects_a_fused_decode_and_writes_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    cs = 8
    al = SfmAligner(cs)
    its = [it for it, _ in _error_items(torch, cs)][:2]
    its[1] = dict(its[1], prx_orig=its[1]["dpt0"], code=np.zeros(cs, np.float32))
    out = torch.full((2, 2), 5.0, device="cuda")
    with pytest.raises(_lib.DfkError, match="work item 1") as e:
        al.EvaluateErrorBatch(al.make_work_items(its), out)
    assert e.value.status == _lib.DFK_ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert torch.all(out == 5.0)


# ------------------------------------------------------------------------------------------------- sparse error batches
@pytest.mark.parametrize("cs", [8, 16, 32, 64, 128])
def test_sparse_error_batches_are_the_records_residual_bit_for_bit(torch_mod, cs):
    torch = torch_mod
    import test_gpu_geometric_batch as tg
    import test_gpu_reprojection_batch as tr
    from deepfactors_b200.aligners import (ReprojectionErrorBatch, ReprojectionLinearizeBatch, SfmAligner,
                                           SparseGeometricErrorBatch, SparseGeometricLinearizeBatch)
    al = SfmAligner(cs)
    NP, GNP = 12 + cs, 12 + 2 * cs
    for make, lin, err, np_ in ((tr.make_factors, ReprojectionLinearizeBatch, ReprojectionErrorBatch, NP),
                                (tg.make_factors, SparseGeometricLinearizeBatch, SparseGeometricErrorBatch, GNP)):
        fs = [{k: v for k, v in f.items() if k != "host"} for f in make(torch, cs)]
        rec = lin(al, fs).cpu().numpy()
        res = rec[:, np_ * (np_ + 1) // 2 + np_:np_ * (np_ + 1) // 2 + np_ + 2]
        for order in (list(range(len(fs))), list(reversed(range(len(fs))))):
            got = err(al, [fs[i] for i in order]).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), res[order].view(np.uint32)), (err.__name__, cs, order)
        assert res[:, 1].view(np.uint32).max() > 1000


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_sparse_error_batches_against_the_fp64_oracle_rows(torch_mod, oracle, cs):
    """b^T b (twice the factor's error) against sum b^2, each over its own size (a sum of positive terms): the fp32 sum
    against the fp64 sum of the same rows (the single call's, bit for bit the rows the kernel forms) at the residual bar
    of system_accuracy.py, and those fp32 rows against the fp64 oracle rows at 1e-4 (the rows' own rounding: the
    geometric b = w (dpt1 - dpt1') cancels, the reprojection b goes through a log and two square roots)"""
    torch = torch_mod
    import test_gpu_geometric_batch as tg
    import test_gpu_reprojection_batch as tr
    from system_accuracy import RES_BAR
    from deepfactors_b200.aligners import ReprojectionErrorBatch, SfmAligner, SparseGeometricErrorBatch
    al = SfmAligner(cs)
    fs = tr.make_factors(torch, cs)
    got = ReprojectionErrorBatch(al, [{k: v for k, v in f.items() if k != "host"} for f in fs]).cpu().numpy()
    worst_sum, worst_rows = 0.0, 0.0
    for f, row in zip(fs, got):
        L = f["host"]
        r64, _ = oracle.reprojection_rows(f["pose0"], f["pose1"], f["code0"], L.cam, L.prx_orig, L.prx_jac, f["query_xy"],
                                          f["train_xy"], f["cauchy_delta"], f["sigma"], precision="f64")
        ref = float(r64[:, -1] @ r64[:, -1])
        b = tr.single_rows(al, f)[:, -1].astype(np.float64)
        own = float(b @ b)
        if ref == 0.0:
            assert row[0] == 0.0 and own == 0.0
            continue
        worst_sum = max(worst_sum, abs(float(row[0]) - own) / own)
        worst_rows = max(worst_rows, abs(own - ref) / ref)
    print(f"reprojection b^T b C={cs}: fp32 sum vs fp64 sum of the same rows {worst_sum:.2e}, fp32 rows vs fp64 oracle "
          f"rows {worst_rows:.2e}")
    assert worst_sum <= RES_BAR
    assert worst_rows <= 1e-4
    fs = tg.make_factors(torch, cs)
    got = SparseGeometricErrorBatch(al, [tg._args(f) for f in fs]).cpu().numpy()
    worst_sum, worst_rows = 0.0, 0.0
    for f, row in zip(fs, got):
        hs = f["host"]
        r64, _ = oracle.sparse_geometric_rows(f["pose0"], f["pose1"], f["code0"], f["code1"], f["cam"], hs["prx0_orig"],
                                              hs["prx0_jac"], hs["prx1_orig"], hs["prx1_jac"], hs["dpt_grad1"],
                                              f["points_xy"], f["huber_delta"], precision="f64")
        ref = float(r64[:, -1] @ r64[:, -1])
        rows, _ = tg.single_rows(al, f)
        own = float(rows[:, -1].astype(np.float64) @ rows[:, -1].astype(np.float64))
        if ref == 0.0:
            assert row[0] == 0.0 and own == 0.0
            continue
        worst_sum = max(worst_sum, abs(float(row[0]) - own) / own)
        worst_rows = max(worst_rows, abs(own - ref) / ref)
    print(f"geometric b^T b C={cs}: fp32 sum vs fp64 sum of the same rows {worst_sum:.2e}, fp32 rows vs fp64 oracle "
          f"rows {worst_rows:.2e}")
    assert worst_sum <= RES_BAR
    assert worst_rows <= 1e-4


# ------------------------------------------------------------------------------------------------------- window energy
def _window(torch, cs=8):
    """three keyframes (test_gpu_geometric_batch's scene), photometric pairs, two reprojection and three geometric
    links, a tracked frame on keyframe 1, a frame prior on keyframe 2 and a keyframe prior over (0, 2).  Pixel validity
    as in EvaluateError (valid_border 1, min_dpt 0), so the two validity chains coincide."""
    import test_gpu_geometric_batch as tg
    import test_gpu_reprojection_batch as tr
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    from deepfactors_b200.window_opt import KeyframePrior, MarginalPrior, SfmWindowProblem, TrackedFrame
    base, cams, kf = tg._window_scene(torch, cs, 2)
    al = SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(valid_border=1, min_dpt=0.0)))
    frame_lv = []
    for l, L in enumerate(base.levels):
        img = synth.rotated_view(L, float(2 ** l), [0.004, -0.005, 0.003]).astype(np.float32)
        frame_lv.append(dict(img=torch.from_numpy(img).cuda(), grad=torch.from_numpy(synth.sobel_np(img)).cuda()))
    rng = np.random.default_rng(7)
    B = 6 + cs

    def spd(n):
        A = rng.standard_normal((n, n)) * 0.3
        return A @ A.T + n * np.eye(n)

    def row(n):
        return np.concatenate([spd(n).ravel(), rng.standard_normal(n), [abs(rng.standard_normal()) + 1.0]])

    poses0 = tg._window_poses()
    priors = [MarginalPrior(2, se3.identity(np.float64), np.zeros(cs), row(B)),
              KeyframePrior((0, 2), poses0[[0, 2]], rng.standard_normal((2, cs)) * 0.01, row(2 * B))]
    prob = SfmWindowProblem(al, cams, kf, [(0, 1), (1, 2), (2, 0), (1, 0)], links=tr._links(base),
                            geometric=tg._geo_links(base), frames=[TrackedFrame(1, frame_lv)], priors=priors)
    return prob, tg._window_poses()


def test_window_error_equals_the_linearisations_energy(torch_mod):
    """E(x) against _energy(linearise(x)) (everything re-linearised at x) at three points: the bar is 1e-5 of |f| for
    the fp32 rounding of the buffer's f and of the different summation orders of the per-item sums; the inlier totals
    are equal; E does not touch the keyframes' depth (the tracker's) or the records"""
    torch = torch_mod
    from deepfactors_b200.window_opt import LMParams, WindowOptimizer
    cs = 8
    prob, poses = _window(torch, cs)
    rng = np.random.default_rng(1)
    opt = WindowOptimizer(prob.layout, prob.linearise, LMParams())
    fposes = np.stack([se3.make_pose([0.002, -0.001, 0.003], [0.01, 0.004, -0.006], np.float64)])
    for it in range(3):
        codes = rng.standard_normal((3, cs)) * 0.05 * it
        buf, _ = prob.linearise(poses, codes, list(range(len(prob.pairs) + len(prob.geometric))), fposes)
        f = opt._energy(buf, codes)
        inl = float(buf[prob.layout.offsets()[2] + 1])
        dpt = [lv["dpt"].clone() for lv in prob.kf[0]]
        rec = prob.records.clone()
        E, parts = prob.error(poses, codes, fposes)
        torch.cuda.synchronize()
        print(f"point {it}: E {E:.9e} f {f:.9e} rel {abs(E - f) / abs(f):.2e}; {parts}")
        assert abs(E - f) <= 1e-5 * abs(f)
        assert parts.inliers == inl
        assert parts.reprojection > 0 and parts.geometric > 0 and parts.priors > 0 and parts.photometric > 0
        assert all(torch.equal(a, b["dpt"]) for a, b in zip(dpt, prob.kf[0]))
        assert torch.equal(rec, prob.records)
        E2, _ = prob.error(poses, codes, fposes)
        assert E2 == E
        poses = np.stack([se3.retract(p, rng.standard_normal(6) * 0.003, np.float64) for p in poses])


def test_lm_with_error_takes_the_same_steps_and_linearises_accepted_points_only(torch_mod):
    """the window above from perturbed poses; the first step is blown up 5x, so it is rejected in both modes"""
    torch = torch_mod
    from deepfactors_b200.window_opt import LMParams, WindowOptimizer
    cs = 8
    prob, poses = _window(torch, cs)
    fposes = np.stack([se3.make_pose([0.003, -0.002, 0.002], [0.012, 0.006, -0.008], np.float64)])
    codes = np.zeros((3, cs))
    prm = LMParams(iterations=6, lambda_init=1e-3, code_prior_weight=1e-2)

    def solve_first_blown_up():
        calls = [0]

        def solve(buf, lam, fixed, w, c):
            dx = prob.solve(buf, lam, fixed, w, c)
            calls[0] += 1
            return dx * 5.0 if calls[0] == 1 and dx is not None else dx
        return solve

    p0, c0, t0 = WindowOptimizer(prob.layout, prob.linearise, prm, solve=solve_first_blown_up()).run(poses, codes, fposes)
    p1, c1, t1 = WindowOptimizer(prob.layout, prob.linearise, prm, solve=solve_first_blown_up(),
                                 error=prob.error).run(poses, codes, fposes)
    print(f"accepted {t1.accepted}; linearisations {t0.linearisations} -> {t1.linearisations}, error evaluations "
          f"{t1.error_evaluations}; energy {t0.energy[0]:.6e} -> {t0.energy[-1]:.6e} / {t1.energy[-1]:.6e}")
    assert t1.accepted == t0.accepted
    assert not t1.accepted[0] and sum(t1.accepted) >= 3
    assert t1.lam == t0.lam
    assert np.abs(p1 - p0).max() <= 1e-6 and np.abs(c1 - c0).max() <= 1e-6
    assert np.abs(t1.frame_poses - t0.frame_poses).max() <= 1e-6
    assert t1.linearisations == 1 + sum(t1.accepted) < t0.linearisations == 1 + len(t0.accepted)
    assert t1.error_evaluations == 1 + len(t1.accepted) and t0.error_evaluations == 0
    assert np.allclose(t1.energy, t0.energy, rtol=1e-5, atol=0)


def test_facade_error_batch_binary():
    """df::SfmAligner::EvaluateErrorBatch against EvaluateError through the C++ facade"""
    exe = os.path.join(ROOT, "tests", "cpp", "error_batch_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "ERROR_BATCH_TEST_OK" in out.stdout, out.stdout + out.stderr
