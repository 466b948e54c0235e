"""Keyframe meshes on the device (dfk_keyframe_mesh_batch, aligners.KeyframeMeshBatch) against the CPU oracle
(mesh_oracle) and dfk_update_depth_batch:

- every output (positions, normals, colours, pixel indices, triangles, counts, uint16 depth) bit for bit the oracle's
  on a mixed batch of sizes 1 x 1 to 640 x 480 with padded pitches, each optional input present and absent, planted
  depths at the range limits, NaN and +-inf, log-stdevs at the noise threshold, and several parameter sets;
- the fused decode at C = 8, 32 and 128 is dfk_update_depth_batch's depth followed by the depth path, bit for bit;
- meshes of a synthetic window's keyframes from a DeviceWindowOptimizer run's final poses and codes, likewise;
- an item one row short writes only its counts, and its neighbours' rows are unchanged (sentinel-filled outputs);
- rejected calls write nothing and name the item and the field;
- two calls are bit for bit equal;
- df::KeyframeMesher of the C++ facade (tests/cpp/keyframe_mesh_test)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib
from mesh_oracle import mesh_oracle as mo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


class Cam:
    def __init__(self, fx, fy, u0, v0, w, h):
        self.fx, self.fy, self.u0, self.v0 = (float(np.float32(v)) for v in (fx, fy, u0, v0))
        self.width, self.height = float(w), float(h)


def same_bits(a, b) -> bool:
    """bit for bit, any NaN equal to any NaN (the device's and the host's default NaNs differ)"""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind != "f":
        return np.array_equal(a, b)
    nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(nan | (a.view(np.uint32) == b.view(np.uint32))))


def scene(rng, w, h, specials=True):
    """host depth, log-stdev, validity and colour of a w x h keyframe"""
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    d = (1.5 + 0.4 * np.sin(xs / 7.0) * np.cos(ys / 5.0) + rng.normal(0, 0.01, (h, w))).astype(np.float32)
    tau = np.float32(mo.tau(4.2))
    s = rng.normal(float(tau), 0.5, (h, w)).astype(np.float32)
    v = rng.uniform(0.0, 1.0, (h, w)).astype(np.float32)
    if specials and w * h >= 16:
        k = rng.choice(w * h, size=min(w * h // 4, 40), replace=False)
        f = np.float32
        planted = [0.5, 10.0, np.nextafter(f(0.5), f(0)), np.nextafter(f(0.5), f(1)), np.nextafter(f(10), f(0)),
                   np.nextafter(f(10), f(11)), np.nan, np.inf, -np.inf, 0.0]
        d.flat[k[:len(planted)]] = np.array(planted[:len(k)], np.float32)
        s.flat[k[-6:]] = np.array([tau, np.nextafter(tau, f(0)), np.nextafter(tau, f(9)), np.nan, -np.inf, np.inf],
                                  np.float32)[:len(k[-6:])]
        v.flat[k[10:16]] = np.array([0.0, -0.0, np.nan, 1e-30, -1.0, 0.0], np.float32)[:len(k[10:16])]
    c = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return d, s, v, c


def dev(torch, a, pad=0):
    """a host array on the device, rows padded by `pad` elements"""
    a = np.ascontiguousarray(a)
    shape = (a.shape[0], a.shape[1] + pad) + a.shape[2:]
    t = torch.zeros(shape, dtype=getattr(torch, str(a.dtype)), device="cuda")
    t[:, :a.shape[1]] = torch.from_numpy(a).cuda()
    return t[:, :a.shape[1]]


def random_pose(rng):
    q = rng.normal(0, 1, 4)
    q /= np.linalg.norm(q)
    return np.concatenate([q, rng.normal(0, 1, 3)]).astype(np.float32)


def check_against_oracle(res, hosts, params):
    """every output of a KeyframeMeshes against mesh_oracle.mesh of each item's host inputs"""
    ms = res.meshes()
    for i, (hst, m) in enumerate(zip(hosts, ms)):
        o = mo.mesh(hst["dpt"], hst["cam"], hst["pose"], std=hst.get("std"), vld=hst.get("vld"),
                    color=hst.get("color"), stdev_thresh=params.stdev_thresh, slt_thresh=params.slt_thresh,
                    crop_pix=params.crop_pix, draw_noisy_pixels=params.draw_noisy_pixels)
        assert (m.num_vertices, m.num_triangles) == (len(o.positions), len(o.triangles)), i
        assert same_bits(m.positions.cpu().numpy(), o.positions), i
        assert same_bits(m.normals.cpu().numpy(), o.normals), i
        assert np.array_equal(m.pixels.cpu().numpy(), o.pixels), i
        assert np.array_equal(m.triangles.cpu().numpy(), o.triangles), i
        if m.colors is not None:
            assert np.array_equal(m.colors.cpu().numpy(), o.colors), i
        if res.depth_u16[i] is not None:
            assert np.array_equal(res.depth_u16[i].cpu().numpy(), o.depth_u16), i
    return ms


SIZES = [(1, 1), (8, 8), (9, 9), (37, 5), (256, 192), (640, 480), (64, 48)]
PARAMS = [dict(), dict(crop_pix=0), dict(crop_pix=1, slt_thresh=0.3), dict(crop_pix=4, slt_thresh=1.0),
          dict(crop_pix=4, draw_noisy_pixels=True), dict(crop_pix=500, stdev_thresh=0.0),
          dict(crop_pix=2, stdev_thresh=-1.0, draw_noisy_pixels=True)]


@pytest.mark.parametrize("pk", range(len(PARAMS)))
def test_mixed_batch_matches_the_oracle(torch_mod, pk):
    torch = torch_mod
    from deepfactors_b200.aligners import KeyframeMeshBatch, KeyframeMeshParams, SfmAligner
    params = KeyframeMeshParams(**PARAMS[pk])
    rng = np.random.default_rng(100 + pk)
    al = SfmAligner(8)
    items, hosts = [], []
    for j, (w, h) in enumerate(SIZES):
        d, s, v, c = scene(rng, w, h)
        cam = Cam(0.8 * w + 1, 0.8 * h + 1, (w - 1) / 2 + 0.25, (h - 1) / 2 - 0.25, w, h)
        pose = random_pose(rng)
        pad = 3 if j % 2 else 0
        it = dict(cam=cam, pose_wk=pose, dpt=dev(torch, d, pad), depth_u16=(j % 3 != 1))
        hst = dict(dpt=d, cam=cam, pose=pose)
        if j % 2 == 0:  # every other item with a stdev and validity view
            it.update(std=dev(torch, s, pad + 1), valid=dev(torch, v, pad))
            hst.update(std=s, vld=v)
        it["color"] = dev(torch, c, pad)
        hst["color"] = c
        items.append(it)
        hosts.append(hst)
    res = KeyframeMeshBatch(al, items, params)
    ms = check_against_oracle(res, hosts, params)
    print(f"params {PARAMS[pk]}: counts {[(m.num_vertices, m.num_triangles) for m in ms]}")
    if pk == 0:
        assert ms[4].num_triangles > 1000  # the default parameters do draw the 256 x 192 keyframe
    # without colour views, no colours are returned; the other outputs are unchanged
    for it in items:
        it.pop("color")
    res2 = KeyframeMeshBatch(al, items, params)
    assert res2.colors is None
    assert torch.equal(res2.positions.view(torch.int32), res.positions.view(torch.int32))
    assert torch.equal(res2.triangles, res.triangles)


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_fused_decode_is_update_depth_then_the_depth_path(torch_mod, cs):
    torch = torch_mod
    from deepfactors_b200.aligners import KeyframeMeshBatch, KeyframeMeshParams, SfmAligner
    al = SfmAligner(cs)
    rng = np.random.default_rng(cs)
    params = KeyframeMeshParams(crop_pix=4)
    dec, ref, hosts = [], [], []
    for j, (w, h) in enumerate([(64, 48), (256, 192), (37, 5)]):
        prx = rng.uniform(0.4, 0.8, (h, w)).astype(np.float32)
        jac = (rng.standard_normal((h, w, cs)) * 0.01).astype(np.float32)
        code = rng.standard_normal(cs).astype(np.float32)
        cam = Cam(0.9 * w, 0.9 * h, w / 2, h / 2, w, h)
        pose = random_pose(rng)
        _, s, v, c = scene(rng, w, h, specials=False)
        dpt = torch.zeros((h, w), dtype=torch.float32, device="cuda")
        ref.append(dict(code=code, prx_orig=dev(torch, prx), prx_jac=dev(torch, jac, 4 * (j % 2)), dpt=dpt))
        dec.append(dict(cam=cam, pose_wk=pose, prx_orig=ref[-1]["prx_orig"], prx_jac=ref[-1]["prx_jac"], code=code,
                        std=dev(torch, s), valid=dev(torch, v), color=dev(torch, c), depth_u16=True))
        hosts.append(dict(cam=cam, pose=pose, std=s, vld=v, color=c))
    al.UpdateDepthBatch(ref)
    res = KeyframeMeshBatch(al, dec, params)
    torch.cuda.synchronize()
    for hst, r in zip(hosts, ref):
        hst["dpt"] = r["dpt"].cpu().numpy()
    check_against_oracle(res, hosts, params)
    # the same items from the decoded depth: the same bits
    for it, r in zip(dec, ref):
        for k in ("prx_orig", "prx_jac", "code"):
            it.pop(k)
        it["dpt"] = r["dpt"]
    res2 = KeyframeMeshBatch(al, dec, params)
    assert torch.equal(res2.positions.view(torch.int32), res.positions.view(torch.int32))
    assert torch.equal(res2.counts, res.counts) and torch.equal(res2.triangles, res.triangles)
    for a, b in zip(res.depth_u16, res2.depth_u16):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_window_keyframes_after_the_device_optimizer(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import KeyframeMeshBatch, KeyframeMeshParams
    from deepfactors_b200.window_opt import DeviceWindowOptimizer
    from test_gpu_window_lm import _lm_start, _scene
    cs = 8
    prob, poses, fposes = _scene(torch, cs)
    p0, prm = _lm_start(prob, poses, fposes, cs)
    gp, gc, _ = DeviceWindowOptimizer(prob, prm).run(p0, np.zeros((3, cs)), fposes)
    cam = prob.cams[0]
    params = KeyframeMeshParams(crop_pix=4)
    items, ref = [], []
    for k in range(3):
        L = prob.kf[k][0]
        code = np.asarray(gc[k], np.float32)
        ref.append(dict(code=code, prx_orig=L["prx_orig"], prx_jac=L["prx_jac"],
                        dpt=torch.zeros_like(L["prx_orig"])))
        items.append(dict(cam=cam, pose_wk=np.asarray(gp[k], np.float32), prx_orig=L["prx_orig"],
                          prx_jac=L["prx_jac"], code=code, depth_u16=True))
    prob.al.UpdateDepthBatch(ref)
    res = KeyframeMeshBatch(prob.al, items, params)
    torch.cuda.synchronize()
    hosts = [dict(dpt=r["dpt"].cpu().numpy(), cam=cam, pose=np.asarray(gp[k], np.float32)) for k, r in enumerate(ref)]
    ms = check_against_oracle(res, hosts, params)
    assert all(m.num_triangles > 0 for m in ms)


def _raw_call(torch, items, n, outs, params, code_size=0, colors=None):
    prm = _lib.DfkKeyframeMeshParams(*params)
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    h = _raw_call.hd.h
    st = _lib.lib().dfk_keyframe_mesh_batch(h, items, n, code_size, C.byref(prm), ptr(outs["pos"]), ptr(outs["nrm"]),
                                            ptr(colors), ptr(outs["pix"]), ptr(outs["tri"]), ptr(outs["cnt"]))
    torch.cuda.synchronize()
    msg = _lib.lib().dfk_last_error(h).decode() if st else ""
    return st, msg


def _sentinel_outputs(torch, V, T, n):
    return dict(pos=torch.full((V, 3), -7.0, device="cuda"), nrm=torch.full((V, 3), -7.0, device="cuda"),
                pix=torch.full((V,), -7, dtype=torch.int32, device="cuda"),
                tri=torch.full((T, 3), -7, dtype=torch.int32, device="cuda"),
                cnt=torch.full((n, 2), -7, dtype=torch.int32, device="cuda"))


def _items(torch, rng, sizes, caps=None):
    from deepfactors_b200.aligners import _cam, _image, _pose
    arr = (_lib.DfkKeyframeMeshItem * len(sizes))()
    keep = []
    for k, (w, h) in enumerate(sizes):
        d = dev(torch, scene(rng, w, h, specials=False)[0])
        keep.append(d)
        a = arr[k]
        a.dpt = _image(d)
        a.cam = _cam(Cam(0.9 * w, 0.9 * h, w / 2, h / 2, w, h))
        a.pose_wk = _pose(random_pose(rng))
        a.vertex_capacity, a.triangle_capacity = caps[k] if caps else (w * h, 2 * w * h)
    arr._keep = keep
    return arr


def test_overflow_writes_only_the_counts(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(8)
    _raw_call.hd = al._hd
    al._hd.use_torch_stream()
    rng = np.random.default_rng(9)
    sizes = [(64, 48), (80, 60), (64, 48)]
    params = (4.2, 0.0, 4, 0)
    full = _items(torch, rng, sizes)
    V, T = sum(w * h for w, h in sizes), sum(2 * w * h for w, h in sizes)
    a = _sentinel_outputs(torch, V, T, 3)
    assert _raw_call(torch, full, 3, a, params) == (0, "")
    counts = a["cnt"].cpu().numpy()
    for which in (0, 1):  # one vertex row short, then one triangle row short
        caps = [(full[k].vertex_capacity, full[k].triangle_capacity) for k in range(3)]
        caps[1] = (int(counts[1, 0]) - (which == 0), int(counts[1, 1]) - (which == 1))
        short = _items(torch, np.random.default_rng(9), sizes, caps)
        b = _sentinel_outputs(torch, V, T, 3)
        assert _raw_call(torch, short, 3, b, params) == (0, "")
        assert np.array_equal(b["cnt"].cpu().numpy(), counts)
        vo = [0, caps[0][0], caps[0][0] + caps[1][0]]
        to = [0, caps[0][1], caps[0][1] + caps[1][1]]
        for key, offs, k_cnt in (("pos", vo, 0), ("nrm", vo, 0), ("pix", vo, 0), ("tri", to, 1)):
            got, ref = b[key], a[key]
            ao = [0, sizes[0][0] * sizes[0][1] * (1 + k_cnt), (sizes[0][0] * sizes[0][1] + 80 * 60) * (1 + k_cnt)]
            for i in (0, 2):  # the neighbours: the rows of the full call
                c = int(counts[i, k_cnt])
                assert torch.equal(got[offs[i]:offs[i] + c].view(torch.int32), ref[ao[i]:ao[i] + c].view(torch.int32))
            # the short item: its rows keep the sentinel
            rows = got[offs[1]:offs[2]]
            assert bool((rows.view(torch.int32) == torch.full_like(rows, -7).view(torch.int32)).all())


def test_rejected_calls_write_nothing(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import SfmAligner
    al = SfmAligner(8)
    _raw_call.hd = al._hd
    al._hd.use_torch_stream()
    rng = np.random.default_rng(4)
    sizes = [(32, 24), (40, 30)]
    params = (4.2, 0.0, 4, 0)
    cases = []

    def case(field, mutate, params=params, code_size=0, colors=False, n=2):
        arr = _items(torch, np.random.default_rng(4), sizes)
        mutate(arr)
        cases.append((field, arr, params, code_size, colors, n))

    case("cam", lambda a: setattr(a[1].cam, "fx", 0.0))
    case("cam", lambda a: setattr(a[1].cam, "width", 40.5))
    case("dpt", lambda a: setattr(a[1].dpt, "width", 39))
    case("dpt", lambda a: setattr(a[1].dpt, "ptr", None))
    case("pose_wk", lambda a: a[1].pose_wk.__setitem__(2, float("nan")))
    case("capacity", lambda a: setattr(a[1], "triangle_capacity", -1))
    case("color", lambda a: None, colors=True)
    case("std", lambda a: setattr(a[1], "std", _lib.DfkImage(a[1].dpt.ptr, a[1].dpt.pitch_bytes, 39, 30)))
    case("depth_u16", lambda a: setattr(a[1], "depth_u16", _lib.DfkImage(a[1].dpt.ptr, 81, 40, 30)))
    case("params", lambda a: None, params=(float("inf"), 0.0, 4, 0))
    case("params", lambda a: None, params=(4.2, 0.0, -1, 0))
    case("number of items", lambda a: None, n=0)
    for field, arr, prm, cs, colors, n in cases:
        out = _sentinel_outputs(torch, 4000, 8000, 2)
        col = torch.full((4000, 3), 7, dtype=torch.uint8, device="cuda") if colors else None
        st, msg = _raw_call(torch, arr, n, out, prm, cs, col)
        assert st != 0, field
        assert field in msg and ("item 1" in msg or field in ("params", "number of items", "color")), (field, msg)
        for t in out.values():
            assert bool((t.view(torch.int32) == torch.full_like(t, -7).view(torch.int32)).all()), field
        if col is not None:
            assert bool((col == 7).all())
    # a decode with an unsupported code size
    arr = _items(torch, np.random.default_rng(4), sizes)
    prx = dev(torch, np.ones((30, 40), np.float32))
    code = np.zeros(300, np.float32)
    arr[1].dpt = _lib.DfkImage()
    arr[1].prx_orig = _lib.DfkImage(C.c_void_p(prx.data_ptr()), 160, 40, 30)
    arr[1].prx_jac = _lib.DfkImage(C.c_void_p(prx.data_ptr()), 160, 40, 30)
    arr[1].code = code.ctypes.data_as(C.POINTER(C.c_float))
    st, msg = _raw_call(torch, arr, 2, _sentinel_outputs(torch, 4000, 8000, 2), params, 300)
    assert st == _lib.DFK_ERR_UNSUPPORTED and "code_size" in msg and "item 1" in msg


def test_two_calls_are_bit_equal(torch_mod):
    torch = torch_mod
    from deepfactors_b200.aligners import KeyframeMeshBatch, KeyframeMeshParams, SfmAligner
    al = SfmAligner(8)
    rng = np.random.default_rng(21)
    items = []
    for w, h in [(640, 480)] * 4 + [(256, 192)] * 4:
        d, s, v, c = scene(rng, w, h)
        items.append(dict(cam=Cam(0.8 * w, 0.8 * h, w / 2, h / 2, w, h), pose_wk=random_pose(rng), dpt=dev(torch, d),
                          std=dev(torch, s), valid=dev(torch, v), color=dev(torch, c), depth_u16=True))
    params = KeyframeMeshParams(crop_pix=4, slt_thresh=0.1, draw_noisy_pixels=True)
    a = KeyframeMeshBatch(al, items, params)
    b = KeyframeMeshBatch(al, items, params)
    for x, y in ((a.positions, b.positions), (a.normals, b.normals)):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    for x, y in ((a.colors, b.colors), (a.pixels, b.pixels), (a.triangles, b.triangles), (a.counts, b.counts)):
        assert torch.equal(x, y)


def test_keyframe_mesher_facade():
    """df::KeyframeMesher against the C call it wraps (tests/cpp/keyframe_mesh_test)"""
    exe = os.path.join(HERE, "cpp", "keyframe_mesh_test")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "keyframe_mesh_test OK" in r.stdout
