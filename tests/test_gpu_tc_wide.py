"""The tensor-core RunStep kernel of the wide code sizes (dfk_sfm_tc_wide.cu, C = 64 and 128), forced with
gram_mode="tf32x3", entry by entry against fp64 (system_accuracy.py): inliers and valid0 exact, H within 5e-5 S,
Jtr within 1e-6 B, the residual within 1e-5.

Covered: 160x120 to 640x480 and a pitched odd layout at four Huber thresholds, two calls bitwise equal, the fp32 wide
engine on the same 4-level pyramid, dfk_set_sm_limit at 1 and 7 SMs (one CTA walks a whole level in 8-tile chains),
a mixed batch down to a 1-pixel item without a valid pixel, code rows that are not 16-byte aligned, the fused depth
decode, and grad1 rows the tensor cores cannot gather (forced mode refuses them, AUTO runs the fp32 wide engine).
"""
import numpy as np
import pytest

from deepfactors_b200 import synth
from system_accuracy import JTR_BAR, assert_system_close, case_pair, level_reference
from test_gpu_parity import upload_level

pytestmark = pytest.mark.gpu

CODE_SIZES = [64, 128]


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _aligner(cs, mode="tf32x3", delta=0.1):
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    return SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(huber_delta=delta)), gram_mode=mode)


def _item(pair, L, dev, **kw):
    views = {k: dev[k] for k in ("img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")}
    return dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{**views, **kw})


def _check(got, ref, valid_gpu, what, **kw):
    assert np.array_equal(valid_gpu, ref.valid), f"{what}: valid0 differs from the fp64 truth"
    e = assert_system_close(got, ref, ref.S, ref.B, what, **kw)
    print(f"worst entries {what}: H {e['h']:.2e} S, Jtr {e['jtr']:.2e} B")  # the README's accuracy table (pytest -s)
    return e


@pytest.mark.parametrize("cs", CODE_SIZES)
@pytest.mark.parametrize("w,h,extra", [(160, 120, 0), (200, 96, 4), (320, 240, 0), (640, 480, 8)])
@pytest.mark.parametrize("delta", [0.01, 0.1, 0.5, 10.0])
def test_tc_wide_per_entry(torch_mod, cs, w, h, extra, delta):
    from oracle import oracle as orc
    pair = case_pair(w, h, cs)
    L = pair.levels[0]
    dev = upload_level(torch_mod, L, extra)
    ref = level_reference(pair, L, orc.default_params(huber_delta=delta))
    assert ref.inliers > 0.3 * w * h
    al = _aligner(cs, "tf32x3", delta)
    work = al.make_work_items([_item(pair, L, dev)])
    first = al.RunStepBatch(work).clone()
    torch_mod.cuda.synchronize()
    got = al.unpack(first)[0]
    _check(got, ref, dev["valid0"].cpu().numpy(), f"tf32x3 {w}x{h}+{extra} C={cs} delta={delta}")
    assert torch_mod.equal(al.RunStepBatch(work), first), "two calls differ"


@pytest.mark.parametrize("cs", CODE_SIZES)
def test_tc_wide_agrees_with_the_fp32_wide_engine(torch_mod, cs):
    """the 640x480 4-level pyramid through both engines: the same inliers and valid0 bit for bit, each within the bars"""
    torch = torch_mod
    pair = synth.make_pair(640, 480, cs, 4, seed=2, code_sigma=0.5)
    devs = [upload_level(torch, L) for L in pair.levels]
    refs = [level_reference(pair, L) for L in pair.levels]
    res, valid = {}, {}
    for mode in ("fp32", "tf32x3"):
        for d in devs:
            d["valid0"].zero_()
        al = _aligner(cs, mode)
        res[mode] = al.unpack(al.RunStepBatch(al.make_work_items([_item(pair, L, d) for L, d in zip(pair.levels, devs)])))
        valid[mode] = [d["valid0"].clone() for d in devs]
    for k, (L, ref) in enumerate(zip(pair.levels, refs)):
        assert torch.equal(valid["fp32"][k], valid["tf32x3"][k])
        assert res["fp32"][k].inliers == res["tf32x3"][k].inliers == ref.inliers
        for mode in ("fp32", "tf32x3"):
            what = f"pyramid {L.width}x{L.height} C={cs} gram={mode}"
            _check(res[mode][k], ref, valid[mode][k].cpu().numpy(), what)


@pytest.mark.parametrize("cs", CODE_SIZES)
def test_tc_wide_sm_limit(torch_mod, cs):
    """1 and 7 SMs: a few CTAs walk the whole 640x480 pyramid; the accumulation chains are still cut every 8 tiles"""
    torch = torch_mod
    pair = synth.make_pair(640, 480, cs, 3, seed=31, code_sigma=0.3)
    devs = [upload_level(torch, L) for L in pair.levels]
    refs = [level_reference(pair, L) for L in pair.levels]
    al = _aligner(cs)
    work = al.make_work_items([_item(pair, L, d) for L, d in zip(pair.levels, devs)])
    for limit in (1, 7):
        al.SetSmLimit(limit)
        for d in devs:
            d["valid0"].zero_()
        recs = al.unpack(al.RunStepBatch(work))
        for L, got, ref, d in zip(pair.levels, recs, refs, devs):
            _check(got, ref, d["valid0"].cpu().numpy(), f"sm_limit={limit} {L.width}x{L.height} C={cs}")
    al.SetSmLimit(0)


@pytest.mark.parametrize("cs", CODE_SIZES)
def test_tc_wide_mixed_batch(torch_mod, cs):
    """one launch over a 320x240 level next to tiny and odd-width items and a 1-pixel item with no valid pixel; the
    views are pitched by 0-2 floats, so most items' code rows are not 16-byte aligned (no bulk-copy flag)"""
    torch = torch_mod
    sizes = [(320, 240), (33, 7), (5, 5), (1, 1), (64, 5), (31, 33), (97, 33)]
    items, refs, devs = [], [], []
    for k, (w, h) in enumerate(sizes):
        pair = case_pair(w, h, cs, seed=60 + k)
        L = pair.levels[0]
        dev = upload_level(torch, L, k % 3)
        items.append(_item(pair, L, dev))
        refs.append(level_reference(pair, L))
        devs.append(dev)
    assert refs[3].inliers == 0
    al = _aligner(cs)
    recs = al.unpack(al.RunStepBatch(al.make_work_items(items)))
    for (w, h), got, ref, d in zip(sizes, recs, refs, devs):
        what = f"batch item {w}x{h} C={cs}"
        if ref.inliers == 0:
            assert got.inliers == 0 and not np.any(got.JtJ) and not np.any(got.Jtr) and got.residual == 0.0, what
            continue
        # Jtr of an item with a handful of valid pixels: 1e-5 B (test_gpu_system_accuracy.py explains why)
        _check(got, ref, d["valid0"].cpu().numpy(), what, jtr_bar=JTR_BAR if ref.inliers >= 64 else 1e-5)


@pytest.mark.parametrize("cs", CODE_SIZES)
@pytest.mark.parametrize("w,h,extra", [(160, 120, 4), (202, 96, 1)])
def test_tc_wide_fused_decode_equals_update_depth_then_run_step(torch_mod, cs, w, h, extra):
    """the depth decoded inside the launch and the records are bit-identical to UpdateDepth followed by RunStep, on
    16-byte aligned (extra = 4) and unaligned (extra = 1) code rows"""
    torch = torch_mod
    from deepfactors_b200.aligners import UpdateDepth
    pair = synth.make_pair(w, h, cs, 2, seed=40 + cs, code_sigma=0.3)
    al = _aligner(cs)
    two_step, fused, keep = [], [], []
    for L in pair.levels:
        dev = upload_level(torch, L, extra)
        dpt_a = torch.zeros_like(dev["dpt0"])
        UpdateDepth(pair.code, dev["prx_orig"], dev["prx0_jac"], 2.0, dpt_a)
        dpt_b = torch.full_like(dev["dpt0"], -7.0)
        va, vb = torch.zeros_like(dev["valid0"]), torch.zeros_like(dev["valid0"])
        base = dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, img0=dev["img0"], img1=dev["img1"],
                    prx0_jac=dev["prx0_jac"], grad1=dev["grad1"])
        two_step.append(dict(base, dpt0=dpt_a, valid0=va))
        fused.append(dict(base, dpt0=dpt_b, valid0=vb, prx_orig=dev["prx_orig"], code=pair.code))
        keep.append((dpt_a, dpt_b, va, vb))
    rec_a = al.RunStepBatch(al.make_work_items(two_step)).clone()
    rec_b = al.RunStepBatch(al.make_work_items(fused)).clone()
    torch.cuda.synchronize()
    for dpt_a, dpt_b, va, vb in keep:
        assert torch.equal(dpt_a, dpt_b), "decoded depth differs from UpdateDepth"
        assert torch.equal(va, vb)
    assert torch.equal(rec_a, rec_b), "fused records differ from UpdateDepth + RunStep"
    assert al.unpack(rec_b)[0].inliers > 0.3 * w * h


@pytest.mark.parametrize("cs", CODE_SIZES)
def test_tc_wide_misaligned_grad1(torch_mod, cs):
    """grad1 rows at a 4-byte offset: the forced tensor-core mode refuses them with the existing message, AUTO runs the
    fp32 wide engine and returns exactly its records"""
    torch = torch_mod
    pair = case_pair(160, 120, cs)
    L = pair.levels[0]
    dev = upload_level(torch, L)
    h, w = L.height, L.width
    base = torch.zeros((h, 2 * w + 1), device="cuda")
    grad = base[:, 1:].view(h, w, 2)
    grad.copy_(dev["grad1"])
    item = _item(pair, L, dev, grad1=grad)
    forced = _aligner(cs, "tf32x3")
    with pytest.raises(Exception, match="tensor-core path needs 8-byte aligned grad1 rows"):
        forced.RunStepBatch(forced.make_work_items([item]))
    out = {}
    for mode in ("auto", "fp32"):
        al = _aligner(cs, mode)
        out[mode] = al.RunStepBatch(al.make_work_items([item])).clone()
    assert torch.equal(out["auto"], out["fp32"])
    ref = level_reference(pair, L)
    assert_system_close(_aligner(cs).unpack(out["auto"])[0], ref, ref.S, ref.B, f"misaligned grad1 C={cs} auto")
