"""Every entry of the RunStep normal equations against fp64, scaled to its own size (system_accuracy.py).

The fp64 truth is the oracle's per-pixel rows summed in fp64 (a 640x480, C = 32 level takes about 0.1 s on the CPU, a
1280x960 level is summed in chunks of image rows), so full sizes are affordable.  Bars: |H - H64| <= 5e-5 S and
|Jtr - Jtr64| <= 1e-6 B per entry, residual 1e-5 relative, inliers and the valid0 mask exactly.  The poses are those of
the reference's RunStep test, where the fp32 validity chain of the kernels and the fp64 one select the same pixels;
every test asserts that (the identity-pose border case keeps its own test in test_gpu_parity.py).

Covered: code sizes 8-128 on every Gram engine, 160x120 to 1280x960 and odd widths on pitched views, Huber thresholds
from "every pixel down-weighted" (0.01) to "none" (10), the single call, RunStepBatch over mixed sizes, the fused depth
decode, dfk_set_sm_limit at 1 and 7 SMs (the longest per-CTA fp32 chains), the fp32 and tensor-core engines against
each other, and the records of the batched reprojection factors.
"""
import numpy as np
import pytest

from deepfactors_b200 import factors, synth
from system_accuracy import H_BAR, JTR_BAR, Reference, assert_system_close, case_pair, level_reference, reference_system
from test_gpu_parity import upload_level

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _modes(cs):
    return ("fp32", "tf32x3") if cs == 32 else ("auto",)


def _aligner(cs, mode, delta=0.1):
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    return SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(huber_delta=delta)), gram_mode=mode)


def _check(got, ref, valid_gpu, what):
    # precondition: the kernels' fp32 validity chain selects the pixels of the fp64 truth
    assert np.array_equal(valid_gpu, ref.valid), f"{what}: fp32 and fp64 valid sets differ ({int(valid_gpu.sum())} vs " \
                                                 f"{ref.inliers}): choose a pose away from the validity border"
    return assert_system_close(got, ref, ref.S, ref.B, what)


def _item(pair, L, dev, **kw):
    return dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{k: dev[k] for k in (
        "img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")}, **kw)


# ---------------------------------------------------------------------------------------------- the single call
SINGLE = [(160, 120, 8, 12), (160, 120, 16, 0), (160, 120, 32, 0), (320, 240, 32, 20), (160, 120, 64, 0),
          (160, 120, 128, 4), (202, 96, 8, 1), (202, 96, 32, 1), (97, 33, 16, 3), (97, 33, 32, 0), (200, 96, 64, 4),
          (320, 240, 128, 0)]


@pytest.mark.parametrize("w,h,cs,extra", SINGLE)
@pytest.mark.parametrize("delta", [0.01, 0.1, 0.5, 10.0])
def test_run_step_per_entry(torch_mod, w, h, cs, extra, delta):
    from oracle import oracle as orc
    pair = case_pair(w, h, cs)
    L = pair.levels[0]
    dev = upload_level(torch_mod, L, extra)
    ref = level_reference(pair, L, orc.default_params(huber_delta=delta))
    assert ref.inliers > 0.3 * w * h
    for mode in _modes(cs):
        dev["valid0"].zero_()
        g = _aligner(cs, mode, delta).RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"],
                                              dev["dpt0"], dev["std0"], dev["valid0"], dev["prx0_jac"], dev["grad1"])
        _check(g, ref, dev["valid0"].cpu().numpy(), f"single {w}x{h}+{extra} C={cs} delta={delta} gram={mode}")


@pytest.mark.parametrize("cs", [32, 128])
@pytest.mark.parametrize("delta", [0.1, 0.5])
def test_run_step_per_entry_640x480(torch_mod, cs, delta):
    from oracle import oracle as orc
    pair = case_pair(640, 480, cs)
    L = pair.levels[0]
    dev = upload_level(torch_mod, L, 8)
    ref = level_reference(pair, L, orc.default_params(huber_delta=delta))
    for mode in _modes(cs):
        dev["valid0"].zero_()
        g = _aligner(cs, mode, delta).RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"],
                                              dev["dpt0"], None, dev["valid0"], dev["prx0_jac"], dev["grad1"])
        _check(g, ref, dev["valid0"].cpu().numpy(), f"single 640x480 C={cs} delta={delta} gram={mode}")


def test_run_step_per_entry_1280x960(torch_mod):
    """four times the largest benchmark level: 1.2 M pixels, fp64 rows summed in chunks of image rows"""
    pair = case_pair(1280, 960, 32, seed=8)
    L = pair.levels[0]
    dev = upload_level(torch_mod, L, 4)
    ref = level_reference(pair, L)
    assert ref.inliers > 500000
    for mode in ("tf32x3", "fp32"):
        dev["valid0"].zero_()
        g = _aligner(32, mode).RunStep(pair.pose0, pair.pose1, pair.code, L.cam, dev["img0"], dev["img1"], dev["dpt0"],
                                       None, dev["valid0"], dev["prx0_jac"], dev["grad1"])
        _check(g, ref, dev["valid0"].cpu().numpy(), f"single 1280x960 C=32 gram={mode}")


# ---------------------------------------------------------------------------------------------- batched paths
@pytest.mark.parametrize("cs", [8, 32, 128])
def test_batch_of_mixed_sizes_per_entry(torch_mod, cs):
    """one launch over items of very different sizes (a 320x240 level next to 7-row, 5x5 and odd-width images).

    Jtr of an item with fewer than 64 valid pixels is held to 1e-5 B instead of 1e-6 B.  Error analysis: each pixel's
    row carries the rounding of the fp32 front-end -- w*diff with diff = img0 - img1(u, v) about a tenth of the
    intensities loses ~3 bits, and the pose entries add the cancellation of a*P0 / a*P1 -- about 1e-6 of |J_i r| per
    pixel (1.1e-6 measured on the H100 for the one valid pixel of the 5x5 item at C = 8, Jtr entry w1 2).  These errors
    are independent across pixels and shrink as 1/sqrt(n) relative to B, which is why a full level sits near 1e-7;
    with a handful of pixels nothing averages.  JtJ has no such difference in it and keeps its bar."""
    torch = torch_mod
    sizes = [(320, 240), (33, 7), (5, 5), (160, 120), (64, 5), (31, 33), (97, 33)]
    items, refs, devs = [], [], []
    for k, (w, h) in enumerate(sizes):
        pair = case_pair(w, h, cs, seed=60 + k)
        L = pair.levels[0]
        dev = upload_level(torch, L, k % 3)
        items.append(_item(pair, L, dev))
        refs.append(level_reference(pair, L))
        devs.append(dev)
    for mode in _modes(cs):
        al = _aligner(cs, mode)
        for d in devs:
            d["valid0"].zero_()
        recs = al.unpack(al.RunStepBatch(al.make_work_items(items)))
        for (w, h), got, ref, d in zip(sizes, recs, refs, devs):
            what = f"batch item {w}x{h} C={cs} gram={mode}"
            if ref.inliers == 0:
                assert got.inliers == 0 and not np.any(got.JtJ) and not np.any(got.Jtr) and got.residual == 0.0, what
                continue
            assert np.array_equal(d["valid0"].cpu().numpy(), ref.valid), what
            assert_system_close(got, ref, ref.S, ref.B, what, jtr_bar=JTR_BAR if ref.inliers >= 64 else 1e-5)


@pytest.mark.parametrize("cs,w,h", [(8, 160, 120), (16, 200, 96), (32, 320, 240), (32, 202, 96), (64, 160, 120),
                                    (128, 160, 120)])
def test_fused_depth_decode_per_entry(torch_mod, cs, w, h):
    """code != NULL: the depth is decoded inside the launch (bit-equal to UpdateDepth, test_gpu_parity.py); the system
    is checked against fp64 rows computed on the depth the GPU decoded"""
    torch = torch_mod
    pair = synth.make_pair(w, h, cs, 2, seed=40 + cs, code_sigma=0.3)
    for mode in _modes(cs):
        al = _aligner(cs, mode)
        items, keep = [], []
        for L in pair.levels:
            dev = upload_level(torch, L, 0 if w % 4 else 4)
            dpt = torch.full_like(dev["dpt0"], -7.0)
            items.append(dict(_item(pair, L, dev), dpt0=dpt, prx_orig=dev["prx_orig"], code=pair.code))
            keep.append((L, dpt, dev))
        recs = al.unpack(al.RunStepBatch(al.make_work_items(items)))
        for got, (L, dpt, dev) in zip(recs, keep):
            decoded = np.ascontiguousarray(dpt.cpu().numpy())
            ref = reference_system(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, decoded, L.prx_jac, L.grad1)
            _check(got, ref, dev["valid0"].cpu().numpy(), f"fused {L.width}x{L.height} C={cs} gram={mode}")


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_sm_limit_per_entry(torch_mod, cs):
    """dfk_set_sm_limit at 1 and 7 SMs: a few CTAs walk the whole 640x480 pyramid, the longest fp32 accumulation
    chains of every engine.

    The C = 64 / 128 kernel (dfk_sfm_wide.cu) at 1 SM is held to 1e-4 S instead of 5e-5 S.  Error analysis: that kernel
    splits a CTA's pixels among only KS = 2 threads per 8x8 block at C = 128 and keeps each split in one fp32 chain until
    the CTA leaves the item; with one SM a single CTA walks the whole 640x480 level, so a code-diagonal entry is a
    chain of about 1e5 same-sign products.  Products far below the running sum lose their low bits, all in the same
    direction, so this error grows like n*eps rather than sqrt(n)*eps: 5.6e-5 S measured on the H100 at 1 SM (code 48,
    code 48, the sum short by 5.6 of 99838), against 3.7e-7 S on the full grid and 1.3e-6 S for the fp32 C = 32 kernel
    at 1 SM, whose lanes cut the chains 32 ways.  (The fp32 CPU path, one chain of 1.9e5 products at 640x480, sits at
    1.2e-4 S.)  Cutting the wide kernel's chains as the tensor-core kernel does (kFlushTiles) would bring it back under
    5e-5; until then this configuration keeps twice the bar."""
    torch = torch_mod
    pair = synth.make_pair(640, 480, cs, 3, seed=31, code_sigma=0.3)
    devs = [upload_level(torch, L) for L in pair.levels]
    refs = [level_reference(pair, L) for L in pair.levels]
    items = [_item(pair, L, d) for L, d in zip(pair.levels, devs)]
    for mode in _modes(cs):
        al = _aligner(cs, mode)
        for limit in (1, 7):
            al.SetSmLimit(limit)
            for d in devs:
                d["valid0"].zero_()
            recs = al.unpack(al.RunStepBatch(al.make_work_items(items)))
            for L, got, ref, d in zip(pair.levels, recs, refs, devs):
                what = f"sm_limit={limit} {L.width}x{L.height} C={cs} gram={mode}"
                assert np.array_equal(d["valid0"].cpu().numpy(), ref.valid), what
                assert_system_close(got, ref, ref.S, ref.B, what, h_bar=2 * H_BAR if (cs >= 64 and limit == 1) else H_BAR)
        al.SetSmLimit(0)


def test_gram_engines_agree_per_entry(torch_mod):
    """the fp32 CUDA-core and the split-tf32 tensor-core engines on the 640x480 4-level pyramid: each within the bar of
    the fp64 truth, so within twice the bar of each other"""
    torch = torch_mod
    pair = synth.make_pair(640, 480, 32, 4, seed=2, code_sigma=0.5)
    devs = [upload_level(torch, L) for L in pair.levels]
    refs = [level_reference(pair, L) for L in pair.levels]
    items = [_item(pair, L, d) for L, d in zip(pair.levels, devs)]
    res = {}
    for mode in ("fp32", "tf32x3"):
        al = _aligner(32, mode)
        res[mode] = al.unpack(al.RunStepBatch(al.make_work_items(items)))
    for L, a, b, ref in zip(pair.levels, res["fp32"], res["tf32x3"], refs):
        what = f"fp32 vs tf32x3 {L.width}x{L.height}"
        other = Reference(b.toDenseMatrix().astype(np.float64), b.Jtr.astype(np.float64), b.residual, b.inliers, ref.S,
                          ref.B, ref.valid)
        assert_system_close(a, other, ref.S, ref.B, what, h_bar=2 * H_BAR, jtr_bar=2 * JTR_BAR, res_bar=2e-5)
        for mode, got in (("fp32", a), ("tf32x3", b)):
            assert_system_close(got, ref, ref.S, ref.B, f"pyramid {L.width}x{L.height} gram={mode}")


# ---------------------------------------------------------------------------------------------- reprojection records
@pytest.mark.parametrize("cs", [8, 32, 128])
def test_reprojection_records_per_entry(torch_mod, cs):
    """each record of ReprojectionLinearizeBatch against the fp64 Gram of that factor's single-call rows [A | b]:
    JtJ = A^T A with S = |A|^T |A|, Jtr = -A^T b with B = |A|^T |b|, residual = b^T b"""
    from deepfactors_b200.aligners import JTJJrReductionItem, SfmAligner
    from test_gpu_reprojection_batch import batch, make_factors, single_rows
    al = SfmAligner(cs)
    fs = make_factors(torch_mod, cs)
    H, Jtr, res, inl = factors.unpack_records(batch(torch_mod, al, fs), cs)
    n = 12 + cs
    checked = 0
    for i, f in enumerate(fs):
        rows = single_rows(al, f).astype(np.float64)
        A, b = rows[:, :n], rows[:, n]
        valid = int((np.abs(rows[0::2]).sum(1) > 0).sum())
        if valid == 0:
            continue
        ref = Reference(A.T @ A, -(A.T @ b), float(b @ b), valid, np.abs(A).T @ np.abs(A), np.abs(A).T @ np.abs(b), None)
        got = JTJJrReductionItem(H[i], Jtr[i], float(res[i]), int(inl[i]))
        assert_system_close(got, ref, ref.S, ref.B, f"reprojection record {i} ({f['query_xy'].shape[0]} matches) C={cs}")
        checked += 1
    assert checked >= 4
