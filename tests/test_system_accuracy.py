"""CPU tests that pin the per-entry comparator of system_accuracy.py (no GPU needed).

  * the oracle's fp64 per-pixel rows, summed in fp64, are the fp64 RunStep system (so the GPU tests compare against the
    same truth as before, only per entry);
  * on the inputs the GPU tests use, the comparator accepts what a correct kernel computes -- a numpy emulation of the
    tensor-core kernel's split-tf32 Gram (HH + LH + LH^T on [J | r]) and the fp32 CPU path -- and rejects each emulated
    bug of that kernel by a margin, so that its bars cannot drift loose unnoticed.
"""
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import oracle as orc
from system_accuracy import (H_BAR, JTR_BAR, RES_BAR, assert_system_close, case_pair, level_reference, pitched_host,
                             reference_system, system_errors)


@pytest.fixture(scope="module", autouse=True)
def _built_oracle():
    orc.build()


def valid_rows(pair, L, params=None):
    """every valid pixel's fp64 row [J | r] and its linear pixel index (row major)"""
    valid = np.zeros((L.height, L.width), dtype=np.float32)
    X, _, _ = orc.sfm_pixel_rows(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, valid, L.prx_jac, L.grad1, params)
    idx = np.flatnonzero(valid.reshape(-1) > 0)
    return X[idx], idx


def tf32_split(x):
    """the kernel's split of an fp32 value: h = x with the low 13 mantissa bits cleared (exact in tf32), l = x - h"""
    x = np.asarray(x, dtype=np.float32)
    h = (x.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)
    return h, x - h


def gram_result(G, inliers):
    """a result of the kernels' form from an (NP+1)^2 Gram of [J | r] (only its upper triangle is read)"""
    n = G.shape[0] - 1
    return SimpleNamespace(JtJ=G[:n, :n], Jtr=G[:n, n], residual=G[n, n], inliers=inliers)


def emulated_gram(X, *, drop_lo=(), lh_t=True, lo=True):
    """split-tf32 Gram of the fp32-rounded rows X, products summed exactly (fp64 of 11-bit mantissas)"""
    h, l = tf32_split(X)
    h, l = h.astype(np.float64), l.astype(np.float64)
    if not lo:
        return h.T @ h
    l[:, list(drop_lo)] = 0.0
    LH = l.T @ h
    return h.T @ h + LH + (LH.T if lh_t else 0.0)


# ---------------------------------------------------------------------------------------------- rows == RunStep
@pytest.mark.parametrize("w,h,cs,extra", [(160, 120, 8, 12), (97, 33, 8, 0), (202, 96, 32, 1), (160, 120, 128, 4)])
@pytest.mark.parametrize("delta", [0.1, 0.5])
def test_pixel_rows_sum_to_the_fp64_run_step(w, h, cs, extra, delta):
    pair = case_pair(w, h, cs)
    L = pair.levels[0]
    prm = orc.default_params(huber_delta=delta)
    args = [pitched_host(a, extra) for a in (L.img0, L.img1, L.dpt0)]
    jac, grad = pitched_host(L.prx_jac, extra), pitched_host(L.grad1, extra)
    v64 = np.zeros((h, w), dtype=np.float32)
    o64 = orc.sfm_run_step(pair.pose0, pair.pose1, L.cam, *args, v64, jac, grad, prm, precision="f64")
    # chunks of a few image rows, the last one ragged
    ref = reference_system(pair.pose0, pair.pose1, L.cam, *args, jac, grad, prm, chunk_pixels=7 * w)
    assert ref.inliers == o64.inliers > 0
    assert np.array_equal(ref.valid, v64)
    X, _ = valid_rows(pair, L, prm)
    absG = np.abs(X).T @ np.abs(X)
    n = 12 + cs
    assert np.all(np.abs(ref.H - o64.dense()) <= 1e-12 * absG[:n, :n])
    assert np.all(np.abs(ref.Jtr - o64.Jtr) <= 1e-12 * absG[:n, n])
    assert abs(ref.residual - o64.residual) <= 1e-12 * o64.residual
    # a row range on its own: the rows of those image lines only
    rows, res, inl = orc.sfm_pixel_rows(pair.pose0, pair.pose1, L.cam, *args, None, jac, grad, prm, y_begin=5, y_end=9)
    assert rows.shape == (4 * w, n + 1)
    assert inl == int(v64[5:9].sum()) and np.array_equal(np.abs(rows).sum(1) > 0, v64[5:9].reshape(-1) > 0)


# ---------------------------------------------------------------------------------------------- the comparator
# (w, h, C): the single-call cases of test_gpu_system_accuracy.py that the CPU checks here afford
ACCEPT_CASES = [(160, 120, 8), (320, 240, 32), (160, 120, 32), (202, 96, 16), (160, 120, 128)]


@pytest.fixture(scope="module")
def c32_320():
    pair = case_pair(320, 240, 32)
    L = pair.levels[0]
    ref = level_reference(pair, L)
    X, idx = valid_rows(pair, L)
    return pair, L, ref, X, idx


@pytest.mark.parametrize("w,h,cs", ACCEPT_CASES)
def test_comparator_accepts_split_tf32_and_the_fp32_cpu_path(w, h, cs):
    pair = case_pair(w, h, cs)
    L = pair.levels[0]
    ref = level_reference(pair, L)
    X, _ = valid_rows(pair, L)
    e = assert_system_close(gram_result(emulated_gram(X), ref.inliers), ref, ref.S, ref.B, f"split-tf32 {w}x{h} C={cs}")
    assert e["h"] <= H_BAR / 50 and e["jtr"] <= JTR_BAR / 50  # a correct split-tf32 sum sits far below the bars
    o32 = orc.sfm_run_step(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, None, L.prx_jac, L.grad1)
    # its residual is one serial fp32 chain of up to 5e4 positive terms (1.4e-5 at 320x240); the kernels sum short
    # chains in a tree, and the GPU tests hold them to RES_BAR
    assert_system_close(o32, ref, ref.S, ref.B, f"fp32 CPU {w}x{h} C={cs}", res_bar=5 * RES_BAR)


def _rejected(got, ref, what):
    """the comparator must refuse `got`, and by a margin of 4 on at least one of its two bars"""
    with pytest.raises(AssertionError):
        assert_system_close(got, ref, ref.S, ref.B, what)
    e = system_errors(got, ref, ref.S, ref.B)
    print(f"{what}: H {e['h']:.2e} Jtr {e['jtr']:.2e}")
    assert e["h"] >= 4 * H_BAR or e["jtr"] >= 4 * JTR_BAR, (what, e["h"], e["jtr"])
    return e


def test_comparator_rejects_plain_tf32(c32_320):
    _, _, ref, X, _ = c32_320
    _rejected(gram_result(emulated_gram(X, lo=False), ref.inliers), ref, "plain tf32")


def test_comparator_rejects_lost_low_parts_of_code_features_24_to_31(c32_320):
    """the tensor-core kernel keeps the low rows of code features 24-31 in their own operand group (group 8) and reads
    them through their own branch of tc_lh: losing them leaves a quarter of the code block at plain-tf32 precision"""
    _, _, ref, X, _ = c32_320
    _rejected(gram_result(emulated_gram(X, drop_lo=range(12 + 24, 12 + 32)), ref.inliers), ref, "lo 24-31 lost")


def test_comparator_rejects_a_missing_lh_transpose(c32_320):
    _, _, ref, X, _ = c32_320
    _rejected(gram_result(emulated_gram(X, lh_t=False), ref.inliers), ref, "LH^T missing")


def test_comparator_rejects_one_dropped_tile(c32_320):
    """one 128-pixel tile's products lost (e.g. an accumulator chain that is never flushed) while the inlier counter,
    which the kernels keep apart from the Gram, still counts its pixels"""
    _, L, ref, X, idx = c32_320
    tiles = idx // 128
    t = np.bincount(tiles).argmax()
    keep = tiles != t
    assert (~keep).sum() > 64
    _rejected(gram_result(emulated_gram(X[keep]), ref.inliers), ref, "one tile dropped")


def test_comparator_rejects_a_code_jacobian_rounded_to_tf32(c32_320):
    pair, L, ref, _, _ = c32_320
    jac = (L.prx_jac.view(np.uint32) & np.uint32(0xffffe000)).view(np.float32)
    bad = reference_system(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, jac, L.grad1)
    assert np.array_equal(bad.valid, ref.valid)
    _rejected(bad, ref, "code Jacobian in tf32")
