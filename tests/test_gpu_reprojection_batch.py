"""dfk_reprojection_linearize_batch / ReprojectionLinearizeBatch on the GPU: reprojection factors linearised in one launch
straight into normal-equation records, and keyframe windows that hold them (SfmWindowProblem links).

A factor's rows [A | b] (reprojection_factor.cpp:157-269) contribute H += A^T A, g += A^T b and |b|^2 to the energy
(reprojection_factor.cpp:148,254-268), so its record must be the Gram of the rows dfk_reprojection_linearize returns for
it: JtJ = A^T A, Jtr = -A^T b, residual = b^T b, inliers = matches with a valid correspondence."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import factors, se3, synth
from test_oracle_ref import _keypoint_matches

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


def make_factors(torch, cs):
    """factors over two level sizes (pitched and not), different codes and poses, M = 1, 7, 129 and 3000 matches (chunk
    edges at 64 and 128), with matches outside the image and a factor whose points all fall behind the camera"""
    pose0, pose1 = synth.reference_test_poses()
    rng = np.random.default_rng(cs)
    out = []
    levels = [synth.make_level(160, 120, cs, seed=12), synth.make_level(97, 61, cs, seed=13)]
    dev = [(pitched(torch, levels[0].prx_orig, 3), pitched(torch, levels[0].prx_jac, 2)),
           (pitched(torch, levels[1].prx_orig), pitched(torch, levels[1].prx_jac))]
    for k, (m, lv, seed) in enumerate([(3000, 0, 4), (1, 1, 5), (7, 0, 6), (129, 1, 7), (400, 0, 8)]):
        L = levels[lv]
        code = (rng.standard_normal(cs) * 0.3).astype(np.float32)
        q, t = _keypoint_matches(L.cam, pose0, pose1, L.prx_orig, n=m, seed=seed)
        if m >= 7:
            q[3] = [-4.0, 7.0]                          # outside the image
            q[5] = [L.cam.width + 3.0, 9.5]
        out.append(dict(pose0=pose0, pose1=pose1, code0=code, cam=L.cam, prx_orig=dev[lv][0], prx_jac=dev[lv][1],
                        query_xy=q, train_xy=t, cauchy_delta=1.5 + 0.5 * k, sigma=2.0 - 0.25 * k, host=L))
    # every point behind the frame (test_reprojection_factor_marks_points_behind_the_camera): an all-zero record
    L = levels[0]
    far = synth.se3.make_pose([0, 0, 0], [0, 0, 30.0], np.float32)
    q = np.array([[10.3, 12.9], [40.0, 30.0], [80.5, 60.5]], dtype=np.float32)
    out.append(dict(pose0=synth.se3.identity(), pose1=far, code0=np.zeros(cs, np.float32), cam=L.cam, prx_orig=dev[0][0],
                    prx_jac=dev[0][1], query_xy=q, train_xy=q + 1.0, cauchy_delta=1.0, sigma=1.0, host=L))
    return out


def single_rows(al, f):
    from deepfactors_b200.aligners import ReprojectionLinearize
    return ReprojectionLinearize(al, f["pose0"], f["pose1"], f["code0"], f["cam"], f["prx_orig"], f["prx_jac"], f["query_xy"],
                                 f["train_xy"], f["cauchy_delta"], f["sigma"])[0]


def batch(torch, al, fs, records=None):
    from deepfactors_b200.aligners import ReprojectionLinearizeBatch
    rec = ReprojectionLinearizeBatch(al, [{k: v for k, v in f.items() if k != "host"} for f in fs], records)
    torch.cuda.synchronize()
    return rec.cpu().numpy()


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_records_are_the_gram_of_the_single_call_rows(torch_mod, oracle, cs):
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(cs)
    fs = make_factors(torch_mod, cs)
    rec = batch(torch_mod, al, fs)
    H, Jtr, res, inl = factors.unpack_records(rec, cs)
    for i, f in enumerate(fs):
        rows = single_rows(al, f).astype(np.float64)
        G = rows.T @ rows
        n = 12 + cs
        valid = int((np.abs(rows[0::2]).sum(1) > 0).sum())
        assert inl[i] == valid, i
        if valid == 0:  # behind the camera: nothing to add
            assert not rec[i].any(), i
            continue
        assert np.abs(H[i] - G[:n, :n]).max() <= 2e-5 * np.abs(G[:n, :n]).max(), i
        assert np.abs(-Jtr[i] - G[:n, n]).max() <= 1e-4 * np.abs(G[:n, n]).max(), i
        assert abs(res[i] - G[n, n]) <= 1e-5 * G[n, n], i
        L = f["host"]
        r64, _ = oracle.reprojection_rows(f["pose0"], f["pose1"], f["code0"], L.cam, L.prx_orig, L.prx_jac, f["query_xy"],
                                          f["train_xy"], f["cauchy_delta"], f["sigma"], precision="f64")
        G64 = r64.T @ r64
        assert np.abs(H[i] - G64[:n, :n]).max() <= 2e-4 * np.abs(G64[:n, :n]).max(), i
    assert inl[0] > 2900 and inl[1] == 1 and inl[-1] == 0


@pytest.mark.parametrize("cs", [8, 128])
def test_a_factor_record_does_not_depend_on_the_batch(torch_mod, cs):
    """bitwise: alone, in the batch, at any position, and across runs"""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(cs)
    fs = make_factors(torch_mod, cs)
    full = batch(torch_mod, al, fs)
    assert np.array_equal(full, batch(torch_mod, al, fs))
    perm = [3, 0, 5, 1, 4, 2]
    shuffled = batch(torch_mod, al, [fs[p] for p in perm])
    for j, p in enumerate(perm):
        assert np.array_equal(shuffled[j], full[p]), p
    for i, f in enumerate(fs):
        assert np.array_equal(batch(torch_mod, al, [f])[0], full[i]), i
    # into a slice of a larger record buffer: the rows around it stay as they were
    buf = torch.full((len(fs) + 2, full.shape[1]), float(SENTINEL), device="cuda")
    got = batch(torch_mod, al, fs, buf[1:1 + len(fs)])
    assert np.array_equal(got, full)
    b = buf.cpu().numpy()
    assert (b[0] == SENTINEL).all() and (b[-1] == SENTINEL).all()


def test_rejected_calls_name_the_item_and_write_nothing(torch_mod, monkeypatch):
    import torch
    from deepfactors_b200 import _lib, aligners
    from deepfactors_b200._lib import DfkReprojectionItem
    from deepfactors_b200.aligners import ReprojectionLinearize, SfmAligner, _cam, _image, _pose
    cs = 8
    al = SfmAligner(cs)
    lib = _lib.lib()
    fs = make_factors(torch_mod, cs)[:3]
    rec = torch.full((3, _lib.record_floats(cs)), float(SENTINEL), device="cuda")
    FP = C.POINTER(C.c_float)
    keep = []

    def items():
        arr = (DfkReprojectionItem * 3)()
        for k, f in enumerate(fs):
            q = np.ascontiguousarray(f["query_xy"], np.float32)
            t = np.ascontiguousarray(f["train_xy"], np.float32)
            c = np.ascontiguousarray(f["code0"], np.float32)
            keep.extend([q, t, c])
            w = arr[k]
            w.pose0, w.pose1, w.cam = _pose(f["pose0"]), _pose(f["pose1"]), _cam(f["cam"])
            w.prx_orig, w.prx_jac = _image(f["prx_orig"]), _image(f["prx_jac"], cs)
            w.code, w.query_xy, w.train_xy = c.ctypes.data_as(FP), q.ctypes.data_as(FP), t.ctypes.data_as(FP)
            w.num_matches, w.cauchy_delta, w.sigma = q.shape[0], f["cauchy_delta"], f["sigma"]
        return arr

    def call(arr, n=3, code_size=cs, ptr=None):
        al._hd.use_torch_stream()
        return lib.dfk_reprojection_linearize_batch(al.handle, arr, n, code_size,
                                                    C.c_void_p(rec.data_ptr() if ptr is None else ptr))

    def mutate(field, value, k=2):
        arr = items()
        setattr(arr[k], field, value)
        return arr

    wide = _image(fs[1]["prx_jac"], cs)
    wide.width += 1
    cases = [  # (call, status, words the error message must hold)
        (lambda: call(items(), n=0), _lib.DFK_ERR_INVALID_ARG, "empty batch"),
        (lambda: call(None), _lib.DFK_ERR_INVALID_ARG, "null"),
        (lambda: lib.dfk_reprojection_linearize_batch(al.handle, items(), 3, cs, None), _lib.DFK_ERR_INVALID_ARG, "null"),
        (lambda: call(items(), code_size=12), _lib.DFK_ERR_UNSUPPORTED, "code size"),
        (lambda: call(mutate("num_matches", 0)), _lib.DFK_ERR_INVALID_ARG, "item 2"),
        (lambda: call(mutate("sigma", 0.0)), _lib.DFK_ERR_INVALID_ARG, "item 2"),
        (lambda: call(mutate("sigma", float("nan"), 1)), _lib.DFK_ERR_INVALID_ARG, "item 1"),
        (lambda: call(mutate("code", None, 0)), _lib.DFK_ERR_INVALID_ARG, "item 0"),
        (lambda: call(mutate("query_xy", None)), _lib.DFK_ERR_INVALID_ARG, "item 2"),
        (lambda: call(mutate("train_xy", None)), _lib.DFK_ERR_INVALID_ARG, "item 2"),
        (lambda: call(mutate("prx_jac", wide, 1)), _lib.DFK_ERR_INVALID_ARG, "item 1"),
        (lambda: call(mutate("prx_orig", _lib.DfkImage(None, 4 * 97, 97, 61), 1)), _lib.DFK_ERR_INVALID_ARG, "item 1"),
    ]
    for k, (fn, want, words) in enumerate(cases):
        st = fn()
        assert st == want, (k, st)
        assert words in lib.dfk_last_error(al.handle).decode(), (k, lib.dfk_last_error(al.handle))
    # the single call checks its arguments as a batch item: a short code, or fewer train than query points, would make
    # the C side read past the host arrays, so the call is refused before it reaches the linearise entry point
    class NoLinearize:
        def __getattr__(self, name):
            assert "linearize" not in name, name
            return getattr(lib, name)

    monkeypatch.setattr(aligners, "lib", NoLinearize)
    single = {k: v for k, v in fs[2].items() if k != "host"}
    for bad in (dict(code0=single["code0"][:cs - 1]), dict(train_xy=single["train_xy"][:-1])):
        with pytest.raises(ValueError):
            ReprojectionLinearize(al, **{**single, **bad})
    # records the kernel would write float32 rows into: big enough, but float64 or on the host
    for wrong in (rec.double(), rec.cpu()):
        with pytest.raises(ValueError):
            aligners.ReprojectionLinearizeBatch(al, [single], wrong)
    monkeypatch.undo()
    torch.cuda.synchronize()
    assert (rec.cpu().numpy() == SENTINEL).all()
    assert call(items()) == _lib.DFK_OK  # and the handle still works


def _window_scene(torch, cs=8, levels=2):
    base = synth.make_pair(160, 120, cs, levels, seed=5)
    cams = [L.cam for L in base.levels]
    keyframes = []
    for k in range(3):
        lv = []
        for L in base.levels:
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
            img = up(L.img0)
            lv.append(dict(img=img, grad=up(synth.sobel_np(L.img0)), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac),
                           dpt=torch.zeros_like(img), valid=torch.zeros_like(img)))
        keyframes.append(lv)
    return base, cams, keyframes


def _links(base, delta=10.0, sigma=1.0):
    from deepfactors_b200.window_opt import ReprojectionLink
    L = base.levels[0]
    ident = se3.identity(np.float64)
    q02, t02 = _keypoint_matches(L.cam, ident, ident, L.prx_orig, n=400, seed=31)
    q20, t20 = _keypoint_matches(L.cam, ident, ident, L.prx_orig, n=400, seed=32)
    return [ReprojectionLink(0, 2, q02, t02, delta, sigma), ReprojectionLink(2, 0, q20, t20, delta, sigma)]


def test_reprojection_link_window_on_device_equals_host_mirror(torch_mod):
    import torch
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import SfmWindowProblem
    cs = 8
    base, cams, keyframes = _window_scene(torch, cs)
    al = SfmAligner(cs)
    pairs = [(0, 1), (1, 2), (1, 0)]
    links = _links(base, delta=3.0, sigma=1.5)
    prob = SfmWindowProblem(al, cams, keyframes, pairs, links=links)
    poses = np.stack([se3.identity(np.float64), se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                      se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.006], np.float64)])
    codes = np.random.default_rng(3).standard_normal((3, cs)) * 0.05
    everything = list(range(len(prob.pairs)))
    buf = prob.linearise(poses, codes, everything)[0].cpu().numpy()
    rec = prob.records.cpu().numpy()
    H, g, res, inl = factors.unpack_records(rec, cs)
    item_pair = [p for p in range(len(pairs)) for _ in range(2)] + [len(pairs), len(pairs) + 1]
    sizes = [(L.width, L.height) for _ in pairs for L in base.levels] + [(0, 0), (0, 0)]
    want = prob.layout.pack(item_pair, H, g, res, inl, sizes)
    assert np.abs(buf - want).max() <= 2e-6 * np.abs(want).max()
    o_t = prob.layout.offsets()[2]
    assert buf[o_t + 1] == float(inl[:-2].sum())                      # photometric inliers only
    assert res[-2:].min() > 0 and abs(buf[o_t] - want[o_t]) <= 1e-6 * want[o_t]
    # the link records are those of ReprojectionLinearizeBatch for the same arguments
    from deepfactors_b200.aligners import ReprojectionLinearizeBatch
    direct = ReprojectionLinearizeBatch(al, prob._items("reprojection", poses, codes, [0, 1])).cpu().numpy()
    assert np.array_equal(direct, rec[-2:])
    # bitwise reproducible, and a partial re-linearisation (one link) lands in the same place
    assert np.array_equal(prob.linearise(poses, codes, everything)[0].cpu().numpy(), buf)
    assert np.array_equal(prob.linearise(poses, codes, [len(pairs) + 1])[0].cpu().numpy(), buf)
    Hd, gd, f, ninl = prob.layout.to_dense(buf)
    Hr, gr, fr = factors.assemble_window(factors.WindowLayout(3, cs), [prob.pairs[p] for p in item_pair], H, g, res, inl,
                                         sizes)
    assert np.abs(Hd - Hr).max() <= 2e-6 * np.abs(Hr).max() and abs(f - fr) <= 1e-5 * abs(fr)


def test_loop_closure_links_pull_a_keyframe_back(torch_mod):
    """keyframes 0 and 1 tied photometrically, keyframe 2 only by reprojection links 0 -> 2 and 2 -> 0 (a global loop
    closure, mapper.cpp:367-376); pose 2 perturbed.  LM must cut the energy by > 10x, bring keyframe 2's translation
    error under 0.25x its start, and re-linearise a link only when its keyframes moved."""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, WindowOptimizer
    cs = 8
    base, cams, keyframes = _window_scene(torch, cs)
    al = SfmAligner(cs)
    pairs = [(0, 1), (1, 0)]
    prob = SfmWindowProblem(al, cams, keyframes, pairs, links=_links(base))
    poses = np.stack([se3.identity(np.float64), se3.identity(np.float64),
                      se3.make_pose([-0.015, 0.01, 0.012], [-0.06, 0.05, -0.03], np.float64)])
    codes = np.zeros((3, cs))
    calls = []

    def linearise(p, c, todo):
        calls.append((p.copy(), c.copy(), list(todo)))
        return prob.linearise(p, c, todo)

    opt = WindowOptimizer(prob.layout, linearise, LMParams(iterations=12, lambda_init=1e-3, code_prior_weight=1e-2))
    p, c, tr = opt.run(poses, codes)
    assert tr.energy[-1] < tr.energy[0] / 10.0, tr.energy
    err0 = np.abs(poses[2][4:7] - poses[0][4:7]).max()
    err1 = np.abs(p[2][4:7] - p[0][4:7]).max()
    assert err1 < 0.25 * err0, (err0, err1)
    assert np.allclose(p[0], poses[0])
    # a link (pair index 2 + j) is in `todo` exactly when pose0, pose1 or code0 moved since its last evaluation
    last = {}
    for cp, cc, todo in calls:
        for j, ln in enumerate(prob.links):
            idx = len(pairs) + j
            key = np.concatenate([cp[ln.k0], cp[ln.k1], cc[ln.k0]])
            moved = idx not in last or np.abs(last[idx] - key).max() > 1e-6
            assert (idx in todo) == moved, (idx, todo)
            if moved:
                last[idx] = key
    assert len(calls) > 1


def test_facade_batch_binary():
    """df::LinearizeReprojectionBatch + WindowSystem::AddUnscaled through the C++ factor header"""
    exe = os.path.join(ROOT, "tests", "cpp", "reprojection_batch_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "REPROJECTION_BATCH_TEST_OK" in out.stdout, out.stdout + out.stderr
