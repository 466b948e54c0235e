"""The binding's argument checks in front of the C calls (aligners.py), one case per call that once bypassed them:

- SfmAligner.RunStepBatch refuses a records tensor that is float64 or on the host before any C call reaches the step
  (the kernel would write float32 rows through its pointer).
- WindowProblem refuses record buffers of another type: linearize and lm write float32 records into them.
- An empty prebuilt item array (make_depth_items / make_depth_prior_items of []) is the empty batch it stands for:
  UpdateDepthBatch, DepthPriorLinearizeBatch and DepthPriorErrorBatch refuse it exactly as they refuse [], not as a
  batch of one zeroed item."""
import pytest

from deepfactors_b200 import _lib, synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _refusal(fn, items):
    with pytest.raises(_lib.DfkError) as e:
        fn(items)
    return e.value.status, e.value.message


def test_run_step_batch_refuses_records_of_another_type_before_any_c_call(torch_mod, monkeypatch):
    torch = torch_mod
    from deepfactors_b200 import aligners
    from test_gpu_parity import upload_level
    al = aligners.SfmAligner(32)
    pair = synth.make_pair(160, 120, 32, 1)
    L = pair.levels[0]
    dev = upload_level(torch, L)
    work = al.make_work_items([dict(pose0=pair.pose0, pose1=pair.pose1, cam=L.cam, **{
        k: dev[k] for k in ("img0", "img1", "dpt0", "valid0", "prx0_jac", "grad1")})])
    rec = torch.full((1, _lib.record_floats(32)), -3.0, device="cuda")

    class NoRunStep:
        def __getattr__(self, name):
            assert "run_step" not in name, name
            return getattr(_lib.lib(), name)

    monkeypatch.setattr(aligners, "lib", NoRunStep)
    for wrong in (rec.double(), rec.cpu()):  # big enough, but not float32 on the handle's device
        with pytest.raises(ValueError, match="records"):
            al.RunStepBatch(work, wrong)
        assert bool((wrong == -3.0).all())
    monkeypatch.undo()
    al.RunStepBatch(work, rec)  # and the same call with float32 device records runs
    torch.cuda.synchronize()
    assert not bool((rec == -3.0).all())


def test_window_problem_refuses_record_buffers_of_another_type(torch_mod):
    from test_gpu_window_lm import _scene
    prob, _, _ = _scene(torch_mod, 8)
    good = prob.records
    for wrong in (good.double(), good.cpu()):
        prob.records = wrong
        with pytest.raises(ValueError, match="records"):
            prob.device_problem()
    prob.records = good
    prob.device_problem()  # the same problem with its float32 device records is accepted


def test_an_empty_prebuilt_item_array_is_refused_as_the_empty_batch(torch_mod):
    from deepfactors_b200.aligners import (DepthPriorErrorBatch, DepthPriorLinearizeBatch, SfmAligner,
                                           make_depth_prior_items)
    cs = 8
    al = SfmAligner(cs)
    assert _refusal(al.UpdateDepthBatch, al.make_depth_items([])) == _refusal(al.UpdateDepthBatch, [])
    for fn in (DepthPriorLinearizeBatch, DepthPriorErrorBatch):
        call = lambda items: fn(al, items)
        assert _refusal(call, make_depth_prior_items([], cs)) == _refusal(call, []), fn.__name__
