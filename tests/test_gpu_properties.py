"""GPU tests at BASELINE.json's full sizes (640x480, 4-level pyramid, C=32) through size-independent
properties -- the fp64 comparison of every entry at these sizes is in test_gpu_system_accuracy.py -- plus the
C++ facade test binary:
  * inliers == number of pixels flagged in valid0; valid0 idempotent (only ever set)
  * additivity: evaluating two complementary pixel sets (the other half made invalid through a negative
    depth) sums to the full evaluation, inliers exactly, JtJ/Jtr/residual to fp32 tolerance
  * the two Gram engines (fp32 CUDA cores, wgmma split-tf32) agree; both are bitwise reproducible
  * the reduced-system structure: the pose1 blocks are the congruent image of the pose0 blocks under the
    relative-pose Jacobians (JtJ = E^T G E)
  * EvaluateError (border 1) sees at least the inliers of RunStep (border 2)
"""
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import se3, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def full_pair():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    pair = synth.make_pair(640, 480, 32, 4, seed=2, code_sigma=0.5)
    dev = []
    for L in pair.levels:
        d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
            img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()}
        d["valid0"] = torch.zeros_like(d["img0"])
        d["cam"] = L.cam
        dev.append(d)
    return pair, dev


def run(al, pair, d, dpt0=None):
    return al.RunStep(pair.pose0, pair.pose1, pair.code, d["cam"], d["img0"], d["img1"], d["dpt0"] if dpt0 is None else dpt0,
                      None, d["valid0"], d["prx0_jac"], d["grad1"])


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_full_size_properties(full_pair, mode):
    import torch
    from deepfactors_b200.aligners import SfmAligner
    pair, dev = full_pair
    al = SfmAligner(32, gram_mode=mode)
    for lvl, d in enumerate(dev):
        d["valid0"].zero_()
        full = run(al, pair, d)
        again = run(al, pair, d)
        assert np.array_equal(full.JtJ, again.JtJ) and full.residual == again.residual, "not reproducible"
        assert full.inliers == int((d["valid0"] == 1).sum())
        assert set(torch.unique(d["valid0"]).tolist()) <= {0.0, 1.0}
        h = d["dpt0"].shape[0]
        top, bot = d["dpt0"].clone(), d["dpt0"].clone()
        top[h // 2:] = -1.0   # a negative depth lands behind the camera: invalid (warping.h:224)
        bot[:h // 2] = -1.0
        a, b = run(al, pair, d, top), run(al, pair, d, bot)
        assert a.inliers + b.inliers == full.inliers
        scale = np.abs(full.JtJ).max()
        assert np.abs((a.JtJ + b.JtJ) - full.JtJ).max() <= 2e-5 * scale, f"level {lvl}"
        assert np.abs((a.Jtr + b.Jtr) - full.Jtr).max() <= 1e-4 * np.abs(full.Jtr).max()
        assert abs((a.residual + b.residual) - full.residual) <= 1e-5 * full.residual
        # structure of JtJ = E^T G E
        from oracle import oracle as orc  # host-side relative-pose Jacobians (checker only)
        _, P1, P0 = orc.relative_pose(pair.pose1.astype(np.float64), pair.pose0.astype(np.float64))
        H = full.toDenseMatrix().astype(np.float64)
        Gaa = np.linalg.solve(P0.T, np.linalg.solve(P0.T, H[:6, :6].T).T)
        assert np.abs(P1.T @ Gaa @ P1 - H[6:12, 6:12]).max() <= 1e-4 * scale
        ev = al.EvaluateError(pair.pose0, pair.pose1, d["cam"], d["img0"], d["img1"], d["dpt0"], None, d["grad1"])
        assert ev.inliers >= full.inliers and ev.residual >= 0.999 * full.residual


def test_c128_full_size_properties():
    """BASELINE config (v): 640x480, C=128 (thread-owned-block kernel): reproducible, additive, inliers == mask"""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    pair = synth.make_pair(640, 480, 128, 1, seed=4)
    L = pair.levels[0]
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
        img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()}
    d["valid0"] = torch.zeros_like(d["img0"])
    d["cam"] = L.cam
    al = SfmAligner(128)
    full, again = run(al, pair, d), run(al, pair, d)
    assert np.array_equal(full.JtJ, again.JtJ) and full.residual == again.residual, "not reproducible"
    assert full.inliers == int((d["valid0"] == 1).sum()) and full.inliers > 100000
    top, bot = d["dpt0"].clone(), d["dpt0"].clone()
    top[240:] = -1.0
    bot[:240] = -1.0
    a, b = run(al, pair, d, top), run(al, pair, d, bot)
    assert a.inliers + b.inliers == full.inliers
    scale = np.abs(full.JtJ).max()
    assert np.abs((a.JtJ + b.JtJ) - full.JtJ).max() <= 2e-5 * scale
    assert np.abs((a.Jtr + b.Jtr) - full.Jtr).max() <= 1e-4 * np.abs(full.Jtr).max()
    H = full.toDenseMatrix()
    assert H.shape == (140, 140) and np.allclose(H, H.T)
    # the 32 leading code columns of a C=128 evaluation == a C=32 evaluation on the same leading Jacobian slices
    d32 = dict(d)
    d32["prx0_jac"] = d["prx0_jac"][:, :, :32].contiguous()
    al32 = SfmAligner(32, gram_mode="fp32")
    sub = run(al32, pair, d32)
    assert sub.inliers == full.inliers
    assert np.abs(sub.toDenseMatrix() - H[:44, :44]).max() <= 2e-5 * scale


def test_large_image_1280x960_properties():
    """four times BASELINE's largest level (1280x960, C=32): inliers == mask, reproducible, engines agree"""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    pair = synth.make_pair(1280, 960, 32, 1, seed=8)
    L = pair.levels[0]
    d = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in dict(
        img0=L.img0, img1=L.img1, dpt0=L.dpt0, prx0_jac=L.prx_jac, grad1=L.grad1).items()}
    d["valid0"] = torch.zeros_like(d["img0"])
    d["cam"] = L.cam
    res = {}
    for mode in ("tf32x3", "fp32"):
        al = SfmAligner(32, gram_mode=mode)
        d["valid0"].zero_()
        a, b = run(al, pair, d), run(al, pair, d)
        assert np.array_equal(a.JtJ, b.JtJ) and a.inliers == int((d["valid0"] == 1).sum()) > 500000
        res[mode] = a
    assert res["fp32"].inliers == res["tf32x3"].inliers
    scale = np.abs(res["fp32"].JtJ).max()
    assert np.abs(res["fp32"].JtJ - res["tf32x3"].JtJ).max() <= 2e-5 * scale


def test_gram_engines_agree_on_the_full_pyramid(full_pair):
    from deepfactors_b200.aligners import SfmAligner
    pair, dev = full_pair
    res = {}
    for mode in ("fp32", "tf32x3"):
        al = SfmAligner(32, gram_mode=mode)
        items = [dict(pose0=pair.pose0, pose1=pair.pose1, cam=d["cam"], img0=d["img0"], img1=d["img1"], dpt0=d["dpt0"],
                      valid0=d["valid0"], prx0_jac=d["prx0_jac"], grad1=d["grad1"]) for d in dev]
        res[mode] = al.unpack(al.RunStepBatch(al.make_work_items(items)))
    for a, b in zip(res["fp32"], res["tf32x3"]):
        assert a.inliers == b.inliers
        assert np.abs(a.JtJ - b.JtJ).max() <= 1e-5 * np.abs(a.JtJ).max()
        assert np.abs(a.Jtr - b.Jtr).max() <= 1e-4 * np.abs(a.Jtr).max()
        assert abs(a.residual - b.residual) <= 1e-5 * a.residual


def test_cpp_facade_binary_runs():
    """tests/cpp/facade_test.cpp: df::SfmAligner / df::SE3Aligner through the header-only facade vs the oracle
    (the reference's FullJacobianCompareWithCpu, tests/ut_sfmaligner.cpp:235-327)."""
    exe = os.path.join(ROOT, "tests", "cpp", "facade_test")
    if not os.path.exists(exe):
        pytest.skip("facade_test not built (run __graft_entry__.build())")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(out.stdout, out.stderr)
    assert out.returncode == 0 and "FACADE_TEST_OK" in out.stdout
