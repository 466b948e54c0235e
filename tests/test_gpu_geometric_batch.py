"""dfk_sparse_geometric_linearize_batch / SparseGeometricLinearizeBatch on the GPU: sparse geometric factors linearised
in one launch straight into normal-equation records, and keyframe windows that hold them as links with their own
code-to-code coupling blocks (SfmWindowProblem geometric links).

A factor's rows [A | b] (sparse_geometric_factor.cpp:157-271) over [pose0 | pose1 | code0 | code1] contribute
H += A^T A, g += A^T b and |b|^2 to the energy, so its record must be the Gram of the rows dfk_sparse_geometric_linearize
returns for it: JtJ = A^T A, Jtr = -A^T b, residual = b^T b, inliers = points with a valid correspondence."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import factors, se3, synth
from system_accuracy import Reference, assert_system_close
from test_oracle_ref import _geometric_scene, _keypoint_matches

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = np.float32(-7.25)  # what "left untouched" looks like


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


def _level(torch, cs, w, h, extra):
    L0, L1, code0, code1, g1, _ = _geometric_scene(cs, w, h)
    dev = dict(prx0_orig=pitched(torch, L0.prx_orig, extra), prx0_jac=pitched(torch, L0.prx_jac, extra),
               prx1_orig=pitched(torch, L1.prx_orig, extra), prx1_jac=pitched(torch, L1.prx_jac, extra),
               dpt_grad1=pitched(torch, g1, extra))
    host = dict(prx0_orig=L0.prx_orig, prx0_jac=L0.prx_jac, prx1_orig=L1.prx_orig, prx1_jac=L1.prx_jac, dpt_grad1=g1)
    return L0.cam, code0, code1, dev, host, (w, h)


def make_factors(torch, cs):
    """factors over two level sizes (pitched 160x120, unpitched 97x61), different codes, poses and Huber deltas,
    M = 1, 7, 63, 64, 65, 129, 500 and 3000 points (chunk edges at 64 and 128), with points outside the image and points
    that warp out of it, and one factor whose points all fall behind the second camera"""
    pose0, pose1 = synth.reference_test_poses()
    rng = np.random.default_rng(100 + cs)
    levels = [_level(torch, cs, 160, 120, 3), _level(torch, cs, 97, 61, 0)]
    out = []
    for k, m in enumerate([3000, 1, 7, 63, 64, 65, 129, 500]):
        cam, code0, code1, dev, host, (w, h) = levels[k % 2]
        if m == 1:
            pts = np.array([[w // 3, h // 3]], dtype=np.int32)  # off the optical axis, where no entry vanishes
        else:
            pts = np.stack([rng.integers(-3, w + 3, m), rng.integers(-3, h + 3, m)], 1).astype(np.int32)
        c0 = (code0 + rng.standard_normal(cs).astype(np.float32) * 0.05).astype(np.float32)
        out.append(dict(pose0=pose0, pose1=pose1, code0=c0, code1=code1, cam=cam, points_xy=pts,
                        huber_delta=0.05 + 0.04 * k, host=host, **dev))
    cam, code0, code1, dev, host, _ = levels[0]
    far = se3.make_pose([0, 0, 0], [0, 0, 30.0], np.float32)
    pts = np.array([[10, 12], [40, 30], [-1, 5], [79, 59]], dtype=np.int32)
    out.append(dict(pose0=se3.identity(), pose1=far, code0=code0, code1=code1, cam=cam, points_xy=pts, huber_delta=0.1,
                    host=host, **dev))
    return out


def _args(f):
    return {k: v for k, v in f.items() if k != "host"}


def single_rows(al, f):
    from deepfactors_b200.aligners import SparseGeometricLinearize
    return SparseGeometricLinearize(al, f["pose0"], f["pose1"], f["code0"], f["code1"], f["cam"], f["prx0_orig"],
                                    f["prx0_jac"], f["prx1_orig"], f["prx1_jac"], f["dpt_grad1"], f["points_xy"],
                                    f["huber_delta"])


def batch(torch, al, fs, records=None):
    from deepfactors_b200.aligners import SparseGeometricLinearizeBatch
    rec = SparseGeometricLinearizeBatch(al, [_args(f) for f in fs], records)
    torch.cuda.synchronize()
    return rec.cpu().numpy()


def _gram_reference(A, b, valid):
    return Reference(A.T @ A, -(A.T @ b), float(b @ b), valid, np.abs(A).T @ np.abs(A), np.abs(A).T @ np.abs(b), None)


@pytest.mark.parametrize("cs", [8, 16, 32, 64, 128])
def test_records_are_the_gram_of_the_single_call_rows(torch_mod, cs):
    from deepfactors_b200.aligners import JTJJrReductionItem, SfmAligner
    al = SfmAligner(cs)
    fs = make_factors(torch_mod, cs)
    rec = batch(torch_mod, al, fs)
    assert rec.shape == (len(fs), factors.geo_record_layout(cs)[2])
    H, Jtr, res, inl = factors.unpack_geometric_records(rec, cs)
    n = 12 + 2 * cs
    for i, f in enumerate(fs):
        rows, nv = single_rows(al, f)
        assert inl[i] == nv, (i, inl[i], nv)
        if nv == 0:
            assert not rec[i].any(), i
            continue
        rows = rows.astype(np.float64)
        ref = _gram_reference(rows[:, :n], rows[:, n], nv)
        got = JTJJrReductionItem(H[i], Jtr[i], float(res[i]), int(inl[i]))
        assert_system_close(got, ref, ref.S, ref.B, f"geometric record {i} ({f['points_xy'].shape[0]} points) C={cs}")
    assert 1000 < inl[0] < 3000, "many points valid, some outside or warped out"
    assert inl[-1] == 0


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_records_per_entry_against_the_fp64_oracle_rows(torch_mod, oracle, cs):
    """each record against the fp64 Gram of oracle.sparse_geometric_rows(precision="f64") for the same factor, at the
    per-entry bars of tests/system_accuracy.py for JtJ and the residual; the worst ratios are printed.  Jtr: its error
    against fp64 rows is mostly that of the fp32 rows themselves (b = w (dpt1 - dpt1') cancels, so a point whose two
    depths nearly agree carries a relative error of about eps |dpt1| / |dpt1 - dpt1'| in b), which the single call shares
    bit for bit.  So every Jtr entry must lie within 1e-6 B of the gap that the fp64 Gram of the single call's rows
    already has to the oracle: what the Gram adds stays at the existing bar, and only the row error may exceed it."""
    from deepfactors_b200.aligners import JTJJrReductionItem, SfmAligner
    al = SfmAligner(cs)
    fs = make_factors(torch_mod, cs)
    H, Jtr, res, inl = factors.unpack_geometric_records(batch(torch_mod, al, fs), cs)
    n = 12 + 2 * cs
    checked = 0
    for i, f in enumerate(fs):
        hs = f["host"]
        r64, n64 = oracle.sparse_geometric_rows(f["pose0"], f["pose1"], f["code0"], f["code1"], f["cam"], hs["prx0_orig"],
                                                hs["prx0_jac"], hs["prx1_orig"], hs["prx1_jac"], hs["dpt_grad1"],
                                                f["points_xy"], f["huber_delta"], precision="f64")
        if n64 == 0:
            assert inl[i] == 0
            continue
        ref = _gram_reference(r64[:, :n], r64[:, n], n64)
        got = JTJJrReductionItem(H[i], Jtr[i], float(res[i]), int(inl[i]))
        rows, _ = single_rows(al, f)
        rows = rows.astype(np.float64)
        row_gap = np.abs(-(rows[:, :n].T @ rows[:, n]) - ref.Jtr)  # the fp32 rows' own Jtr error, Gram in fp64
        gap = np.abs(Jtr[i].astype(np.float64) - ref.Jtr)
        worst = float(np.max((gap - row_gap) / np.where(ref.B > 0, ref.B, 1.0)))
        print(f"geometric record {i} vs fp64 oracle C={cs}: Jtr beyond the rows' own gap {worst:.2e} B, rows' gap "
              f"{float(np.max(row_gap / np.where(ref.B > 0, ref.B, 1.0))):.2e} B")
        assert worst <= 1e-6, (i, worst)
        # JtJ and the residual at the existing bars; Jtr above (the sum of the rows' gap and the Gram's part)
        assert_system_close(got, ref, ref.S, ref.B, f"geometric record {i} vs fp64 oracle C={cs}", jtr_bar=np.inf)
        checked += 1
    assert checked >= 7


@pytest.mark.parametrize("cs", [8, 128])
def test_a_factor_record_does_not_depend_on_the_batch(torch_mod, cs):
    """bitwise: alone, permuted, repeated, across runs and in a slice of a larger buffer (C = 128: the split grid)"""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(cs)
    fs = make_factors(torch_mod, cs)
    full = batch(torch_mod, al, fs)
    assert np.array_equal(full, batch(torch_mod, al, fs))
    perm = [3, 0, 8, 5, 1, 7, 4, 2, 6]
    shuffled = batch(torch_mod, al, [fs[p] for p in perm])
    for j, p in enumerate(perm):
        assert np.array_equal(shuffled[j], full[p]), p
    rep = batch(torch_mod, al, [fs[2], fs[0], fs[2], fs[0]])
    for j, p in enumerate([2, 0, 2, 0]):
        assert np.array_equal(rep[j], full[p]), p
    for i, f in enumerate(fs):
        assert np.array_equal(batch(torch_mod, al, [f])[0], full[i]), i
    buf = torch.full((len(fs) + 2, full.shape[1]), float(SENTINEL), device="cuda")
    got = batch(torch_mod, al, fs, buf[1:1 + len(fs)])
    assert np.array_equal(got, full)
    b = buf.cpu().numpy()
    assert (b[0] == SENTINEL).all() and (b[-1] == SENTINEL).all()


def test_reprojection_and_geometric_batches_back_to_back(torch_mod):
    """both batched sparse launches enqueued on one handle with no sync in between: each gives its standalone records"""
    import torch
    from deepfactors_b200.aligners import ReprojectionLinearizeBatch, SfmAligner, SparseGeometricLinearizeBatch
    from test_gpu_reprojection_batch import make_factors as rep_factors
    cs = 32
    al = SfmAligner(cs)
    gfs = [_args(f) for f in make_factors(torch_mod, cs)]
    rfs = [{k: v for k, v in f.items() if k != "host"} for f in rep_factors(torch_mod, cs)]
    r_alone = ReprojectionLinearizeBatch(al, rfs).cpu().numpy()
    g_alone = SparseGeometricLinearizeBatch(al, gfs).cpu().numpy()
    torch.cuda.synchronize()
    r1 = ReprojectionLinearizeBatch(al, rfs)
    g1 = SparseGeometricLinearizeBatch(al, gfs)
    r2 = ReprojectionLinearizeBatch(al, rfs[::-1])
    g2 = SparseGeometricLinearizeBatch(al, gfs[:3])
    torch.cuda.synchronize()
    assert np.array_equal(r1.cpu().numpy(), r_alone) and np.array_equal(g1.cpu().numpy(), g_alone)
    assert np.array_equal(r2.cpu().numpy(), r_alone[::-1]) and np.array_equal(g2.cpu().numpy(), g_alone[:3])


def test_rejected_calls_name_the_item_and_write_nothing(torch_mod, monkeypatch):
    import torch
    from deepfactors_b200 import _lib, aligners
    from deepfactors_b200._lib import DfkSparseGeometricItem
    from deepfactors_b200.aligners import SfmAligner, SparseGeometricLinearize, _cam, _image, _pose
    cs = 8
    al = SfmAligner(cs)
    lib = _lib.lib()
    fs = make_factors(torch_mod, cs)[:3]
    rec = torch.full((3, _lib.geo_record_floats(cs)), float(SENTINEL), device="cuda")
    FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    keep = []

    def items():
        arr = (DfkSparseGeometricItem * 3)()
        for k, f in enumerate(fs):
            c0 = np.ascontiguousarray(f["code0"], np.float32)
            c1 = np.ascontiguousarray(f["code1"], np.float32)
            p = np.ascontiguousarray(f["points_xy"], np.int32)
            keep.extend([c0, c1, p])
            w = arr[k]
            w.pose0, w.pose1, w.cam = _pose(f["pose0"]), _pose(f["pose1"]), _cam(f["cam"])
            w.prx0_orig, w.prx0_jac = _image(f["prx0_orig"]), _image(f["prx0_jac"], cs)
            w.prx1_orig, w.prx1_jac = _image(f["prx1_orig"]), _image(f["prx1_jac"], cs)
            w.dpt_grad1 = _image(f["dpt_grad1"], 2)
            w.code0, w.code1, w.points_xy = c0.ctypes.data_as(FP), c1.ctypes.data_as(FP), p.ctypes.data_as(IP)
            w.num_points, w.huber_delta = p.shape[0], f["huber_delta"]
        return arr

    def call(arr, n=3, code_size=cs, ptr=None):
        al._hd.use_torch_stream()
        return lib.dfk_sparse_geometric_linearize_batch(al.handle, arr, n, code_size,
                                                        C.c_void_p(rec.data_ptr() if ptr is None else ptr))

    def mutate(field, value, k=2):
        arr = items()
        setattr(arr[k], field, value)
        return arr

    wide = _image(fs[1]["prx1_jac"], cs)
    wide.width += 1
    big_cam = _cam(fs[0]["cam"])
    big_cam.width += 8
    cases = [  # (call, status, words the error message must hold)
        (lambda: call(items(), n=0), _lib.DFK_ERR_INVALID_ARG, "empty batch"),
        (lambda: call(None), _lib.DFK_ERR_INVALID_ARG, "null"),
        (lambda: lib.dfk_sparse_geometric_linearize_batch(al.handle, items(), 3, cs, None), _lib.DFK_ERR_INVALID_ARG,
         "null"),
        (lambda: call(items(), code_size=12), _lib.DFK_ERR_UNSUPPORTED, "code size"),
        (lambda: call(mutate("num_points", 0)), _lib.DFK_ERR_INVALID_ARG, "item 2: no points"),
        (lambda: call(mutate("huber_delta", 0.0)), _lib.DFK_ERR_INVALID_ARG, "item 2: no points / non-positive"),
        (lambda: call(mutate("huber_delta", float("nan"), 1)), _lib.DFK_ERR_INVALID_ARG, "item 1"),
        (lambda: call(mutate("code0", None, 0)), _lib.DFK_ERR_INVALID_ARG, "item 0: null"),
        (lambda: call(mutate("code1", None)), _lib.DFK_ERR_INVALID_ARG, "item 2: null"),
        (lambda: call(mutate("points_xy", None)), _lib.DFK_ERR_INVALID_ARG, "item 2: null"),
        (lambda: call(mutate("prx1_jac", wide, 1)), _lib.DFK_ERR_INVALID_ARG, "item 1: inconsistent"),
        (lambda: call(mutate("prx0_orig", _lib.DfkImage(None, 4 * 97, 97, 61), 1)), _lib.DFK_ERR_INVALID_ARG,
         "item 1: inconsistent"),
        (lambda: call(mutate("cam", big_cam, 0)), _lib.DFK_ERR_INVALID_ARG, "item 0: camera larger"),
    ]
    for k, (fn, want, words) in enumerate(cases):
        st = fn()
        assert st == want, (k, st)
        assert words in lib.dfk_last_error(al.handle).decode(), (k, lib.dfk_last_error(al.handle))
    # the single call checks its arguments as a batch item: a short code would make the C side read past the host
    # array, so the call is refused before it reaches the linearise entry point
    class NoLinearize:
        def __getattr__(self, name):
            assert "linearize" not in name, name
            return getattr(lib, name)

    monkeypatch.setattr(aligners, "lib", NoLinearize)
    single = _args(fs[2])
    for bad in (dict(code0=single["code0"][:cs - 1]), dict(code1=single["code1"][:cs - 1])):
        with pytest.raises(ValueError):
            SparseGeometricLinearize(al, **{**single, **bad})
    # records the kernel would write float32 rows into: big enough, but float64 or on the host
    for wrong in (rec.double(), rec.cpu()):
        with pytest.raises(ValueError):
            aligners.SparseGeometricLinearizeBatch(al, [single], wrong)
    monkeypatch.undo()
    torch.cuda.synchronize()
    assert (rec.cpu().numpy() == SENTINEL).all()
    assert call(items()) == _lib.DFK_OK  # and the handle still works


# ----------------------------------------------------------------------------------------------------------- windows
def _window_scene(torch, cs=8, levels=2):
    """three keyframes of one scene (true poses identity); each carries the Sobel gradient of its level-0 depth at code
    zero (mapper.cpp:993-1000), which geometric links into it need"""
    base = synth.make_pair(160, 120, cs, levels, seed=5)
    cams = [L.cam for L in base.levels]
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    keyframes = []
    for k in range(3):
        lv = []
        for L in base.levels:
            img = up(L.img0)
            lv.append(dict(img=img, grad=up(synth.sobel_np(L.img0)), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac),
                           dpt=torch.zeros_like(img), valid=torch.zeros_like(img)))
        L = base.levels[0]
        dpt = (np.float32(2.0) / L.prx_orig - np.float32(2.0)).astype(np.float32)
        lv[0]["dpt_grad"] = up(synth.sobel_np(dpt))
        keyframes.append(lv)
    return base, cams, keyframes


def _geo_links(base, delta=0.1, step=5):
    from deepfactors_b200.window_opt import GeometricLink
    L = base.levels[0]
    ys, xs = np.mgrid[4:L.height - 4:step, 4:L.width - 4:step]
    pts = np.stack([xs.ravel(), ys.ravel()], 1).astype(np.int32)
    return [GeometricLink(0, 2, pts, delta), GeometricLink(2, 0, pts[::-1].copy(), delta),
            GeometricLink(1, 2, pts[::2].copy(), delta)]


def _window_poses():
    return np.stack([se3.identity(np.float64), se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                     se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.03], np.float64)])


def test_geometric_link_window_on_device_equals_host_mirror(torch_mod):
    import torch
    from deepfactors_b200.aligners import SfmAligner, SparseGeometricLinearizeBatch
    from deepfactors_b200.window_opt import SfmWindowProblem
    cs = 8
    base, cams, keyframes = _window_scene(torch, cs)
    al = SfmAligner(cs)
    pairs = [(0, 1), (1, 2), (1, 0)]
    geo = _geo_links(base)
    prob = SfmWindowProblem(al, cams, keyframes, pairs, geometric=geo)
    assert prob.layout.floats == prob.window.floats == factors.WindowBlocks(3, cs, pairs).floats + len(geo) * (6 + cs) ** 2
    poses = _window_poses()
    codes = np.random.default_rng(3).standard_normal((3, cs)) * 0.05
    everything = list(range(len(pairs) + len(geo)))
    buf = prob.linearise(poses, codes, everything)[0].cpu().numpy()
    rec = prob.records.cpu().numpy()
    grec = prob.geo_records.cpu().numpy()
    H, g, res, inl = factors.unpack_records(rec, cs)
    gH, gg, gres, ginl = factors.unpack_geometric_records(grec, cs)
    assert (ginl > 0).all() and (gres > 0).all()
    item_pair = [p for p in range(len(pairs)) for _ in range(2)]
    sizes = [(L.width, L.height) for _ in pairs for L in base.levels]
    want = prob.layout.pack(item_pair, H, g, res, inl, sizes, geo=(gH, gg, gres))
    assert np.abs(buf - want).max() <= 2e-6 * np.abs(want).max()
    o_t = prob.layout.offsets()[2]
    assert buf[o_t + 1] == float(inl.sum())  # links add no inliers
    assert abs(buf[o_t] - want[o_t]) <= 2e-6 * want[o_t]
    # the link records are those of SparseGeometricLinearizeBatch for the same arguments
    direct = SparseGeometricLinearizeBatch(al, prob._items("geometric", poses, codes, [0, 1, 2])).cpu().numpy()
    assert np.array_equal(direct, grec)
    # bitwise reproducible, and a partial re-linearisation (one link) lands in the same place
    assert np.array_equal(prob.linearise(poses, codes, everything)[0].cpu().numpy(), buf)
    assert np.array_equal(prob.linearise(poses, codes, [len(pairs) + 1])[0].cpu().numpy(), buf)
    # to_dense against a dense numpy scatter of the same records
    Hd, gd, f, _ = prob.layout.to_dense(buf)
    Hr, gr, fr = factors.assemble_window(factors.WindowLayout(3, cs), [pairs[p] for p in item_pair], H, g, res, inl, sizes)
    B = 6 + cs
    for l, gl in enumerate(geo):
        i0 = np.r_[0:6, 12:12 + cs]
        i1 = np.r_[6:12, 12 + cs:12 + 2 * cs]
        s0, s1 = slice(gl.k0 * B, (gl.k0 + 1) * B), slice(gl.k1 * B, (gl.k1 + 1) * B)
        G = gH[l].astype(np.float64)
        Hr[s0, s0] += G[np.ix_(i0, i0)]
        Hr[s1, s1] += G[np.ix_(i1, i1)]
        Hr[s0, s1] += G[np.ix_(i0, i1)]
        Hr[s1, s0] += G[np.ix_(i1, i0)]
        gr[s0] -= gg[l][i0]
        gr[s1] -= gg[l][i1]
        fr += float(gres[l])
    assert np.abs(Hd - Hr).max() <= 2e-6 * np.abs(Hr).max()
    assert np.abs(gd - gr).max() <= 2e-6 * np.abs(gr).max() and abs(f - fr) <= 1e-5 * abs(fr)


def test_window_relinearises_any_subset_of_its_factors_in_place(torch_mod):
    """photometric pairs, reprojection links and geometric links in one window: with the records of the factors in
    `todo` spoilt first, re-linearising any one factor, or every factor of one kind, at the same poses and codes writes
    each record back to its own rows and leaves every other row alone.  Photometric pair p owns records rows
    [p * levels, (p + 1) * levels), reprojection link j row len(pairs) * levels + j, geometric link j geo_records row j.
    A link's record does not depend on its batch, and a batch of all photometric pairs is the one of the full
    linearisation, so those come back bit for bit.  A batch of some photometric pairs sums their pixels in another
    order; its records come back within 1e-5 of their largest entry, and another pair's record would not."""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import ReprojectionLink, SfmWindowProblem
    cs, levels = 8, 2
    base, cams, keyframes = _window_scene(torch, cs, levels)
    al = SfmAligner(cs)
    L = base.levels[0]
    ident = se3.identity(np.float64)
    links = [ReprojectionLink(0, 2, *_keypoint_matches(L.cam, ident, ident, L.prx_orig, n=400, seed=31), 3.0, 1.5),
             ReprojectionLink(2, 1, *_keypoint_matches(L.cam, ident, ident, L.prx_orig, n=300, seed=32), 2.0, 1.0)]
    pairs = [(0, 1), (1, 2), (1, 0)]
    geo = _geo_links(base)
    prob = SfmWindowProblem(al, cams, keyframes, pairs, links=links, geometric=geo)
    poses = _window_poses()
    codes = np.random.default_rng(6).standard_normal((3, cs)) * 0.05
    P, R, G = len(pairs), len(links), len(geo)
    full = prob.linearise(poses, codes, list(range(P + R + G)))[0].cpu().numpy()
    rec, grec = prob.records.cpu().numpy(), prob.geo_records.cpu().numpy()
    assert np.isfinite(rec).all() and np.isfinite(grec).all()
    assert np.abs(rec).max(1).min() > 0 and np.abs(grec).max(1).min() > 0
    assert min(np.abs(rec[i] - rec[j]).max() / np.abs(rec[i]).max() for i in range(P * levels) for j in range(i)) > 1e-4

    def rows(p):  # (records rows, geo_records rows) of factor p in `todo` numbering
        if p < P:
            return list(range(p * levels, (p + 1) * levels)), []
        return ([P * levels + p - P], []) if p < P + R else ([], [p - P - R])

    kinds = [list(range(P)), list(range(P, P + R)), list(range(P + R, P + R + G))]
    for todo in [[p] for p in range(P + R + G)] + kinds:
        spoilt = [r for p in todo for r in rows(p)[0]], [r for p in todo for r in rows(p)[1]]
        r0, g0 = rec.copy(), grec.copy()
        r0[spoilt[0]], g0[spoilt[1]] = np.nan, np.nan
        prob.records.copy_(torch.from_numpy(r0))
        prob.geo_records.copy_(torch.from_numpy(g0))
        buf = prob.linearise(poses, codes, todo)[0].cpu().numpy()
        got, ggot = prob.records.cpu().numpy(), prob.geo_records.cpu().numpy()
        assert np.array_equal(ggot, grec), todo
        if 0 < len([p for p in todo if p < P]) < P:
            assert np.isfinite(got).all(), todo
            assert (np.abs(got - rec).max(1) <= 1e-5 * np.abs(rec).max(1)).all(), todo
            kept = np.setdiff1d(np.arange(len(rec)), spoilt[0])
            assert np.array_equal(got[kept], rec[kept]), todo
            assert np.abs(buf - full).max() <= 1e-5 * np.abs(full).max(), todo
        else:
            assert np.array_equal(got, rec) and np.array_equal(buf, full), todo


def test_window_entry_points_reject_bad_links(torch_mod):
    import torch
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner, Window
    cs = 8
    al = SfmAligner(cs)
    lib = _lib.lib()
    I32 = C.POINTER(C.c_int32)
    k0 = np.array([0, 1], np.int32)
    k1 = np.array([1, 0], np.int32)
    ip = np.array([0, 1], np.int32)
    wh = np.array([160, 160], np.int32)
    hh = np.array([120, 120], np.int32)
    desc = _lib.DfkWindowDesc(3, 2, 2, cs, k0.ctypes.data_as(I32), k1.ctypes.data_as(I32), ip.ctypes.data_as(I32),
                              wh.ctypes.data_as(I32), hh.ctypes.data_as(I32))
    for a, b, words in (([0, 3], [2, 1], "link 1 names a keyframe outside"), ([0, 1], [2, -1], "link 1 names"),
                        ([2, 0], [2, 1], "link 0 ties a keyframe to itself")):
        la, lb = np.array(a, np.int32), np.array(b, np.int32)
        out = C.c_void_p(12345)
        st = lib.dfk_window_create_geometric(al.handle, C.byref(desc), 2, la.ctypes.data_as(I32), lb.ctypes.data_as(I32),
                                             C.byref(out))
        assert st == _lib.DFK_ERR_INVALID_ARG and words in lib.dfk_last_error(al.handle).decode()
        assert not out.value
    win = Window(al, 3, [(0, 1), (1, 0)], [0, 1], [(160, 120), (160, 120)], geometric=[(0, 2)])
    rec = torch.zeros((2, _lib.record_floats(cs)), device="cuda")
    out = torch.full((win.floats,), float(SENTINEL), device="cuda")
    al._hd.use_torch_stream()
    st = lib.dfk_window_assemble(al.handle, win.w, C.c_void_p(rec.data_ptr()), C.c_void_p(out.data_ptr()))
    assert st == _lib.DFK_ERR_INVALID_ARG and "geometric links" in lib.dfk_last_error(al.handle).decode()
    st = lib.dfk_window_assemble_geometric(al.handle, win.w, C.c_void_p(rec.data_ptr()), None, C.c_void_p(out.data_ptr()))
    assert st == _lib.DFK_ERR_INVALID_ARG and "no geometric records" in lib.dfk_last_error(al.handle).decode()
    torch.cuda.synchronize()
    assert (out.cpu().numpy() == SENTINEL).all()
    geo = torch.zeros((1, _lib.geo_record_floats(cs)), device="cuda")
    win.assemble(rec, out, geo_records=geo)  # and the handle still works
    torch.cuda.synchronize()
    assert not (out.cpu().numpy() == SENTINEL).any()


def test_window_without_links_is_the_same_through_both_entry_points(torch_mod):
    import torch
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import SfmWindowProblem
    cs = 8
    base, cams, keyframes = _window_scene(torch, cs)
    al = SfmAligner(cs)
    prob = SfmWindowProblem(al, cams, keyframes, [(0, 1), (1, 2), (2, 0)])
    poses = _window_poses()
    codes = np.random.default_rng(4).standard_normal((3, cs)) * 0.05
    a = prob.linearise(poses, codes, [0, 1, 2])[0].cpu().numpy()
    out = torch.empty(prob.window.floats, device="cuda")
    al._hd.use_torch_stream()
    _lib.check(al.handle, _lib.lib().dfk_window_assemble_geometric(al.handle, prob.window.w,
                                                                   C.c_void_p(prob.records.data_ptr()), None,
                                                                   C.c_void_p(out.data_ptr())))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), a)


def test_geometric_links_pull_a_keyframe_back(torch_mod):
    """keyframes 0 and 1 tied photometrically, keyframe 2 only by geometric links 0 -> 2, 2 -> 0 and 1 -> 2; keyframe 2's
    pose perturbed, mostly along its optical axis, which the depth residual observes directly.  LM must cut the energy
    by > 10x, bring keyframe 2's translation error under 0.25x its start, and re-linearise a link exactly when pose0,
    pose1, code0 or code1 moved."""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, WindowOptimizer
    cs = 8
    base, cams, keyframes = _window_scene(torch, cs)
    al = SfmAligner(cs)
    pairs = [(0, 1), (1, 0)]
    prob = SfmWindowProblem(al, cams, keyframes, pairs, geometric=_geo_links(base, delta=0.5))
    poses = np.stack([se3.identity(np.float64), se3.identity(np.float64),
                      se3.make_pose([0.004, -0.003, 0.002], [0.01, -0.008, 0.08], np.float64)])
    codes = np.zeros((3, cs))
    calls = []

    def linearise(p, c, todo):
        calls.append((p.copy(), c.copy(), list(todo)))
        return prob.linearise(p, c, todo)

    opt = WindowOptimizer(prob.layout, linearise, LMParams(iterations=12, lambda_init=1e-3, code_prior_weight=1e-2))
    p, c, tr = opt.run(poses, codes)
    print("energy", tr.energy)
    assert tr.energy[-1] < tr.energy[0] / 10.0, tr.energy
    err0 = np.abs(poses[2][4:7] - poses[0][4:7]).max()
    err1 = np.abs(p[2][4:7] - p[0][4:7]).max()
    assert err1 < 0.25 * err0, (err0, err1)
    assert np.allclose(p[0], poses[0])
    last = {}
    for cp, cc, todo in calls:
        for j, gl in enumerate(prob.geometric):
            idx = len(pairs) + j
            key = np.concatenate([cp[gl.k0], cp[gl.k1], cc[gl.k0], cc[gl.k1]])
            moved = idx not in last or np.abs(last[idx] - key).max() > 1e-6
            assert (idx in todo) == moved, (idx, todo)
            if moved:
                last[idx] = key
    assert len(calls) > 1


def test_facade_batch_binary():
    """df::LinearizeSparseGeometricBatch + WindowSystem::AddGeometric through the C++ factor header"""
    exe = os.path.join(ROOT, "tests", "cpp", "geometric_batch_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "GEOMETRIC_BATCH_TEST_OK" in out.stdout, out.stdout + out.stderr
