"""The fp64 truth and the per-entry comparator of the tracker's SE3 step, DepthAligner and UpdateDepth (CPU only).

  * The oracle's new fp64 rows (se3_pixel_rows, depth_pixel_rows) sum to its fp64 RunSteps to 1e-12, and the fp64
    decode (update_depth(precision="f64")) agrees with the fp32 one to rounding.
  * The comparator (system_accuracy.RowGram / assert_system_close, update_depth_scale) accepts a correct fp32
    reduction of the rows at every bar, and the fp32 CPU flavours at the JtJ, residual and decode bars.  Their Jtr is
    one serial fp32 chain per entry over the level and misses 1e-6 B by up to 3.6x, which is the error class the Jtr
    bar is there to catch (the serial-chain bug below is the same thing at 1280x960).
  * It rejects emulated kernel bugs by at least 4x: a 256-thread block's second grid-stride pass dropped at 1280x960,
    the Huber weight applied to J but not to r, DepthAligner's Jtr summed as one serial fp32 chain over a 1280x960
    level with one-signed Jacobian columns, and UpdateDepth with a tf32-rounded code or one float4 lane dropped at
    C = 128.
  * One candidate bug falls below the bars and is only reported: the SE3 gradients sampled with tf32-rounded bilinear
    weights.  The rounding moves each pixel's J by about 2^-11 of the gradient difference across the pixel, with a
    sign that varies from pixel to pixel, so over n pixels it grows like sqrt(n) while S and B grow like n; on a
    160x120 level it sits at 1.2e-6 S / 6.1e-7 B, 0.6x the bars (test_tf32_gradient_weights_are_below_the_bars).
"""
import numpy as np
import pytest

from deepfactors_b200 import se3, synth
from oracle import oracle as orc
from system_accuracy import (CODE_NAMES, H_BAR, JTR_BAR, SE3_NAMES, UD_BAR, Reference, RowGram, assert_system_close,
                             depth_reference, se3_reference, system_errors, update_depth_errors, update_depth_scale)

POSE = se3.make_pose([0.01, -0.02, 0.005], [0.02, 0.01, -0.03])
REJECT = 4.0


def _level(w, h, cs=1, seed=0, **kw):
    return synth.make_level(w, h, cs, seed=seed, **kw)


def _se3_rows(L, delta=0.1, valid_f32=True):
    X, _, n = orc.se3_pixel_rows(POSE, L.cam, L.img0, L.img1, L.dpt0, L.grad1, delta, valid_f32=valid_f32)
    return X, n


def _worst(e, h_bar=H_BAR, jtr_bar=JTR_BAR):
    """how far above the bars a result is: max(h / h_bar, jtr / jtr_bar)"""
    return max(e["h"] / h_bar, e["jtr"] / jtr_bar)


def _sys(X, inliers):
    return RowGram(X.shape[1] - 1).add(X).reference(inliers)


def _as_got(ref: Reference):
    return Reference(ref.H, ref.Jtr, ref.residual, ref.inliers, ref.S, ref.B, None)


# ------------------------------------------------------------------------------------------------ identities
@pytest.mark.parametrize("w,h,delta", [(160, 120, 0.1), (97, 33, 0.01), (80, 60, 10.0)])
def test_se3_rows_sum_to_the_fp64_run_step(w, h, delta):
    L = _level(w, h, seed=w)
    X, n = _se3_rows(L, delta, valid_f32=False)
    o = orc.se3_run_step(POSE, L.cam, L.img0, L.img1, L.dpt0, L.grad1, delta, precision="f64")
    ref = _sys(X, n)
    assert n == o.inliers > 0.5 * w * h
    e = system_errors(o, ref, ref.S, ref.B)
    assert e["h"] <= 1e-12 and e["jtr"] <= 1e-12 and e["res"] <= 1e-12, e
    # the fp32 validity chain: the pixel set of the fp32 oracle (and of the kernels)
    _, n32 = _se3_rows(L, delta, valid_f32=True)
    assert n32 == orc.se3_run_step(POSE, L.cam, L.img0, L.img1, L.dpt0, L.grad1, delta).inliers


def test_se3_rows_follow_the_fp32_validity_chain_at_identity():
    """at the identity pose fp32 and fp64 disagree on border pixels; valid_f32 takes the fp32 set"""
    L = _level(80, 60, seed=3)
    ident = se3.identity()
    o32 = orc.se3_run_step(ident, L.cam, L.img0, L.img1, L.dpt0, L.grad1)
    o64 = orc.se3_run_step(ident, L.cam, L.img0, L.img1, L.dpt0, L.grad1, precision="f64")
    _, _, n32 = orc.se3_pixel_rows(ident, L.cam, L.img0, L.img1, L.dpt0, L.grad1, valid_f32=True)
    _, _, n64 = orc.se3_pixel_rows(ident, L.cam, L.img0, L.img1, L.dpt0, L.grad1, valid_f32=False)
    print(f"identity 80x60: fp32 chain {o32.inliers} pixels, fp64 chain {o64.inliers}")
    assert (n32, n64) == (o32.inliers, o64.inliers)


@pytest.mark.parametrize("cs,w,h,avg", [(8, 160, 120, 2.0), (32, 97, 33, 2.0), (16, 80, 60, 3.5)])
def test_depth_rows_sum_to_the_fp64_run_step(cs, w, h, avg):
    L = _level(w, h, cs, seed=cs, avg_dpt=avg)
    code = np.random.default_rng(cs).standard_normal(cs).astype(np.float32) * 0.3
    tgt = (L.dpt0 * np.float32(1.05) + np.float32(0.01)).astype(np.float32)
    ref = depth_reference(code, tgt, L.prx_orig, L.prx_jac, avg)
    o = orc.depth_run_step(code, tgt, L.prx_orig, L.prx_jac, avg, precision="f64")
    e = system_errors(o, ref, ref.S, ref.B)
    assert o.inliers == ref.inliers == w * h
    assert e["h"] <= 1e-12 and e["jtr"] <= 1e-12 and e["res"] <= 1e-12, e


@pytest.mark.parametrize("cs,avg", [(1, 2.0), (12, 2.0), (128, 2.0), (32, 0.7)])
def test_fp64_decode_agrees_with_the_fp32_oracle(cs, avg):
    L = _level(64, 48, cs, seed=cs)
    code = np.random.default_rng(cs).standard_normal(cs).astype(np.float32) * 0.5
    d32 = orc.update_depth(code, L.prx_orig, L.prx_jac, avg)
    d64 = orc.update_depth(code, L.prx_orig, L.prx_jac, avg, precision="f64")
    r, at = update_depth_errors(d32, d64, update_depth_scale(code, L.prx_orig, L.prx_jac, avg))
    print(f"fp32 oracle decode C={cs} avg={avg}: worst pixel {at} at {r:.2e} S_px (bar {UD_BAR:.0e})")
    assert r <= UD_BAR


# ------------------------------------------------------------------------------------------------ accepts
def _fp32_tree(X, inliers):
    """a correct fp32 reduction of rows [J | r]: J and r rounded to fp32, the products in fp32, each entry summed
    pairwise (numpy's fp32 sum) -- the error class of the kernels' short per-thread chains and tree reductions"""
    X32 = np.ascontiguousarray(X, dtype=np.float32)
    n = X.shape[1] - 1
    iu = np.triu_indices(n)
    col = [np.ascontiguousarray(X32[:, k]) for k in range(n + 1)]
    H = np.array([np.sum(col[i] * col[j], dtype=np.float32) for i, j in zip(*iu)], dtype=np.float32)
    Jtr = np.array([np.sum(col[i] * col[n], dtype=np.float32) for i in range(n)], dtype=np.float32)
    return orc.StepResult(H, Jtr, float(np.sum(col[n] * col[n], dtype=np.float32)), inliers)


def _depth_case(cs, w, h):
    L = _level(w, h, cs, seed=cs)
    code = np.random.default_rng(cs).standard_normal(cs).astype(np.float32) * 0.3
    tgt = (L.dpt0 + np.float32(0.02)).astype(np.float32)
    return L, code, tgt


@pytest.mark.parametrize("w,h,delta", [(160, 120, 0.1), (320, 240, 0.01), (80, 60, 10.0), (1280, 960, 0.1)])
def test_comparator_accepts_fp32_se3_systems(w, h, delta):
    """A correct fp32 reduction passes every bar.  The fp32 CPU flavour (dfko_se3_run_step_f) passes the JtJ and
    residual bars; its Jtr is one serial fp32 chain per entry over the whole level, the error the Jtr bar exists to
    catch, and it sits at 1.2e-6 - 2e-6 B here (reported, held to 1e-5 B)."""
    L = _level(w, h, seed=w + 1)
    ref = se3_reference(POSE, L.cam, L.img0, L.img1, L.dpt0, L.grad1, delta)
    X, n = _se3_rows(L, delta)
    assert_system_close(_fp32_tree(X, n), ref, ref.S, ref.B, f"fp32 tree SE3 {w}x{h} delta={delta}", names=SE3_NAMES)
    if w * h <= 320 * 240:
        o = orc.se3_run_step(POSE, L.cam, L.img0, L.img1, L.dpt0, L.grad1, delta)
        assert_system_close(o, ref, ref.S, ref.B, f"fp32 CPU SE3 {w}x{h} delta={delta}", jtr_bar=1e-5,
                            names=SE3_NAMES)


@pytest.mark.parametrize("cs,w,h", [(8, 160, 120), (32, 80, 60), (128, 64, 48)])
def test_comparator_accepts_fp32_depth_systems(cs, w, h):
    """as above for DepthAligner; the fp32 CPU flavour's serial Jtr chain reaches 3.6e-6 B at 160x120"""
    L, code, tgt = _depth_case(cs, w, h)
    ref = depth_reference(code, tgt, L.prx_orig, L.prx_jac)
    X = orc.depth_pixel_rows(code, tgt, L.prx_orig, L.prx_jac)
    assert_system_close(_fp32_tree(X, w * h), ref, ref.S, ref.B, f"fp32 tree depth C={cs} {w}x{h}", names=CODE_NAMES)
    o = orc.depth_run_step(code, tgt, L.prx_orig, L.prx_jac)
    assert_system_close(o, ref, ref.S, ref.B, f"fp32 CPU depth C={cs} {w}x{h}", jtr_bar=1e-5, names=CODE_NAMES)


# ------------------------------------------------------------------------------------------------ rejects
def test_rejects_a_dropped_second_grid_stride_pass_at_1280x960():
    """1280x960 = 4.7 pixels per thread of the 1024 x 256 grid: block 17 loses its second pass (256 pixels)"""
    L = _level(1280, 960, seed=9)
    X, n = _se3_rows(L)
    ref = _sys(X, n)
    drop = np.arange(1024 * 256 + 17 * 256, 1024 * 256 + 18 * 256)
    keep = np.ones(X.shape[0], bool)
    keep[drop] = False
    bug = _sys(X[keep], n)
    e = system_errors(_as_got(bug), ref, ref.S, ref.B)
    print(f"dropped pass: {e['h']:.2e} S, {e['jtr']:.2e} B -> {_worst(e):.0f}x the bars")
    assert _worst(e) >= REJECT


def test_rejects_huber_weight_on_j_but_not_on_r():
    L = _level(160, 120, seed=5)
    X, n = _se3_rows(L, 0.1)
    X0, _ = _se3_rows(L, 1e30)  # unweighted rows, same pixels
    ref = _sys(X, n)
    bug = _sys(np.concatenate([X[:, :6], X0[:, 6:]], axis=1), n)
    e = system_errors(_as_got(bug), ref, ref.S, ref.B)
    print(f"Huber on J only: {e['jtr']:.2e} B, residual {e['res']:.2e} -> {_worst(e):.0f}x the bars")
    assert _worst(e) >= REJECT


def _tf32(x):
    b = np.ascontiguousarray(x, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def test_tf32_gradient_weights_are_below_the_bars():
    """Not rejected (module docstring): sampling grad1 with tf32-rounded bilinear weights fu, fv.  Each valid pixel's
    pix1 and pose Jacobian come from the oracle's probe, J = -(gx A0 + gy A1) w is recomputed with exact and with
    rounded weights, and the difference is added to the fp64 rows."""
    L = _level(160, 120, seed=6)
    X, n = _se3_rows(L)
    ref = _sys(X, n)
    Xb = X.copy()
    g = L.grad1.astype(np.float64)
    for p in np.flatnonzero(np.any(X != 0, axis=1)):
        y, x = divmod(int(p), L.width)
        pr = orc.probe_pixel(x, y, float(L.dpt0[y, x]), L.cam, POSE.astype(np.float64))
        u, v = pr["pix1"]
        ix, iy = int(np.floor(u)), int(np.floor(v))
        fu, fv = u - ix, v - iy
        q = g[iy:iy + 2, ix:ix + 2]

        def lerp(a, b):
            top = q[0, 0] + a * (q[0, 1] - q[0, 0])
            return top + b * (q[1, 0] + a * (q[1, 1] - q[1, 0]) - top)

        d = lerp(float(_tf32(fu)[0]), float(_tf32(fv)[0])) - lerp(fu, fv)
        J = X[p, :6]
        J0 = -(pr["J_pose"][0] * lerp(fu, fv)[0] + pr["J_pose"][1] * lerp(fu, fv)[1])
        w = J[np.argmax(np.abs(J0))] / J0[np.argmax(np.abs(J0))]
        Xb[p, :6] += -(pr["J_pose"][0] * d[0] + pr["J_pose"][1] * d[1]) * w
    e = system_errors(_as_got(_sys(Xb, n)), ref, ref.S, ref.B)
    print(f"tf32 gradient weights: {e['h']:.2e} S, {e['jtr']:.2e} B -> {_worst(e):.2f}x the bars (below them)")
    assert e["h"] > 0 and e["jtr"] > 0


def test_rejects_depth_jtr_as_one_serial_fp32_chain():
    """one-signed Jacobian columns (and a target one-signedly behind the decoded depth) so nothing cancels: the whole
    1280x960 level summed as one fp32 chain per Jtr entry"""
    cs = 8
    L = _level(1280, 960, cs, seed=2, jac_sigma=0.0)
    jac = np.abs(np.random.default_rng(2).standard_normal((960, 1280, cs))).astype(np.float32) * np.float32(0.02)
    code = np.full(cs, 0.1, np.float32)
    dpt = orc.update_depth(code, L.prx_orig, jac)
    tgt = (dpt * np.float32(1.1)).astype(np.float32)
    ref = depth_reference(code, tgt, L.prx_orig, jac)
    X = orc.depth_pixel_rows(code, tgt, L.prx_orig, jac)
    prod = (X[:, :cs] * X[:, cs:]).astype(np.float32)
    jtr = np.cumsum(prod, axis=0, dtype=np.float32)[-1]
    rj = np.max(np.abs(jtr - ref.Jtr) / ref.B)
    print(f"serial fp32 Jtr chain over 1280x960: {rj:.2e} B -> {rj / JTR_BAR:.0f}x the bar")
    assert rj >= REJECT * JTR_BAR


@pytest.mark.parametrize("bug", ["tf32 code", "lane 5 dropped"])
def test_rejects_update_depth_bugs(bug):
    cs = 128
    L = _level(160, 120, cs, seed=7)
    code = np.random.default_rng(7).standard_normal(cs).astype(np.float32) * 0.5
    d64 = orc.update_depth(code, L.prx_orig, L.prx_jac, precision="f64")
    jac = L.prx_jac.astype(np.float64)
    if bug == "tf32 code":
        dot = jac @ _tf32(code).astype(np.float64)
    else:  # at C = 128 lane `sub` owns float4 chunk sub: terms 20..23 of lane 5
        c = code.astype(np.float64)
        c[20:24] = 0
        dot = jac @ c
    got = 2.0 / (L.prx_orig.astype(np.float64) + dot) - 2.0
    r, at = update_depth_errors(got, d64, update_depth_scale(code, L.prx_orig, L.prx_jac, 2.0))
    print(f"UpdateDepth {bug}: worst pixel {at} at {r:.2e} S_px -> {r / UD_BAR:.0f}x the bar")
    assert r >= REJECT * UD_BAR
