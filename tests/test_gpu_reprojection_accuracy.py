"""The reprojection factor on the device against fp64 truth, entry by entry: the single-call rows
(dfk_reprojection_linearize), the batched records (dfk_reprojection_linearize_batch) and the error batch
(dfk_reprojection_error_batch) of every factor of tests/test_reprojection_accuracy.py's set, held to the checks stated
there (the Cauchy weight per match, the rows per column block, JtJ / Jtr / residual / inliers per entry, the error
batch bit for bit).  Every code size, every chunk edge of RepCfg<C> and a 20000-match chain, pitched and odd unpitched
levels, the reference test poses and a near-identity pair, sigma 0.5 and 2, and five residual regimes: 0.7 px noise,
the mapper's delta 0.1 (a << 1), near-exact matches (a >> 1) at delta 1.5 and 1e3, and 0.7 px noise at delta 1e3."""
import numpy as np
import pytest

from deepfactors_b200 import factors
from test_reprojection_accuracy import CODE_SIZES, REGIMES, Truth, evaluate, levels, make_factors, report

pytestmark = pytest.mark.gpu

_ALIGNERS = {}


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def pitched(torch, arr, extra_px=0):
    """host [H, W(, K)] -> device view whose rows are padded by extra_px pixels"""
    a = np.ascontiguousarray(arr, dtype=np.float32)
    h, w = a.shape[:2]
    k = a.shape[2] if a.ndim == 3 else 1
    row = (w + extra_px) * k
    buf = torch.zeros((h, row), dtype=torch.float32, device="cuda")
    buf[:, :w * k] = torch.from_numpy(a.reshape(h, w * k)).cuda()
    return buf[:, :w] if a.ndim == 2 else torch.as_strided(buf, (h, w, k), (row, k, 1))


def aligner(cs):
    from deepfactors_b200.aligners import SfmAligner
    if cs not in _ALIGNERS:
        _ALIGNERS[cs] = SfmAligner(cs)
    return _ALIGNERS[cs]


ARGS = ("pose0", "pose1", "code0", "cam", "prx_orig", "prx_jac", "query_xy", "train_xy", "cauchy_delta", "sigma")


@pytest.mark.parametrize("regime", sorted(REGIMES))
@pytest.mark.parametrize("cs", CODE_SIZES)
def test_reprojection_factor_against_fp64_per_entry(torch_mod, oracle, cs, regime):
    from deepfactors_b200.aligners import ReprojectionErrorBatch, ReprojectionLinearize, ReprojectionLinearizeBatch
    torch = torch_mod
    al = aligner(cs)
    fs = make_factors(cs, regime)
    dev = [(pitched(torch, L.prx_orig, extra), pitched(torch, L.prx_jac, extra)) for L, extra in levels(cs)]
    items = [dict({k: f[k] for k in ARGS}, prx_orig=dev[f["level"]][0], prx_jac=dev[f["level"]][1]) for f in fs]
    rec = ReprojectionLinearizeBatch(al, items)
    err = ReprojectionErrorBatch(al, items)
    torch.cuda.synchronize()
    rec, err = rec.cpu().numpy(), err.cpu().numpy()
    H, Jtr, res, inl = factors.unpack_records(rec, cs)
    failed = []
    for i, (f, it) in enumerate(zip(fs, items)):
        rows, _ = ReprojectionLinearize(al, *[it[k] for k in ARGS])
        t = Truth(oracle, f)
        what = f"C={cs} {regime} factor {i} ({f['query_xy'].shape[0]} matches, delta {f['cauchy_delta']}, " \
               f"sigma {f['sigma']})"
        if t.inliers == 0:  # every point behind the camera: nothing to add
            assert inl[i] == 0 and not rec[i].any() and not err[i].any() and not rows.any(), what
            continue
        checks = evaluate(t, rows, (H[i], Jtr[i], res[i], inl[i]),
                          err_batch=(err[i, 0], err[i, 1:2].view(np.uint32)[0]))
        report(what, checks)
        failed += [f"{what}: {k} {v[0]:.3g} x its bar at {v[1]}" for k, v in checks.items() if not v[0] <= 1.0]
    assert not failed, "\n".join(failed)
