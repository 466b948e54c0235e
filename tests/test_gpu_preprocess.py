"""Frame preprocessing on the device (dfk_preprocess_batch, aligners.PreprocessBatch) against OpenCV
(tests/golden/preprocess_frames.npz) and the CPU oracle (preprocess_oracle, the SfM oracle's blur-down and Sobel):

- colour, gray and level 0 of every fixture run bit for bit, by digest and, for the stored run, row by row; the
  identity config returns the source unchanged;
- every output, all levels and gradients included, bit for bit the oracle's on random frames of mixed sizes with padded
  pitches on the sources and the outputs; the levels equal dfk_build_image_pyramid run on the device's level 0;
- with normalisation, (mu, sigma) equal the oracle's fixed-order fp64 sums and f' follows from them bit for bit;
- an item's output is the same alone and in a mixed batch of 64 frames, and two runs are bit for bit equal;
- the device gray fed to OrbDetectBatch gives exactly the features of the oracle's gray;
- rejected calls write nothing and name the item;
- df::FramePreprocessor of the C++ facade (tests/cpp/preprocess_test)."""
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib
from oracle import oracle as orc
from preprocess_oracle import preprocess_oracle as po

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def torch_mod():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


@pytest.fixture(scope="module")
def aligner(torch_mod):
    from deepfactors_b200.aligners import SfmAligner
    return SfmAligner(8)


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(os.path.join(HERE, "golden", "preprocess_frames.npz")))


class Cam:
    def __init__(self, c, w=0.0, h=0.0):
        self.fx, self.fy, self.u0, self.v0 = (float(v) for v in np.float32(c[:4]))
        self.width, self.height = float(w), float(h)


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def dev_frame(torch, img, pad=0):
    """uint8 [H, W, 3] on the device, rows padded by `pad` bytes"""
    h, w = img.shape[:2]
    buf = torch.zeros((h, 3 * w + pad), dtype=torch.uint8, device="cuda")
    buf[:, :3 * w] = torch.from_numpy(np.ascontiguousarray(img).reshape(h, 3 * w)).cuda()
    return buf[:, :3 * w].view(h, w, 3) if pad == 0 else torch.as_strided(buf, (h, w, 3), (3 * w + pad, 3, 1))


def run_frame(fx, run):
    name, img = str(run).rsplit("_", 1)
    c = fx[f"cfg_{name}"]
    frame = fx[f"image_{img}"]
    if int(c[0]) == 2:
        frame = np.ascontiguousarray(np.repeat(np.repeat(frame, 2, axis=0), 2, axis=1))
    return frame, np.float32(c[1:5]), np.float32(c[5:9]), int(c[9]), int(c[10])


def host(out):
    """one PreprocessedFrame on the host"""
    cv = lambda t: None if t is None else t.cpu().numpy()
    return dict(color=cv(out.color), gray=cv(out.gray), levels=[cv(t) for t in out.levels],
                grads=None if out.grads is None else [cv(t) for t in out.grads], stats=cv(out.stats))


def bits_equal(a, b):
    return np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8))


def frames_equal(a, b):
    for k in a:
        x, y = a[k], b[k]
        if x is None or y is None:
            ok = x is None and y is None
        elif isinstance(x, list):
            ok = len(x) == len(y) and all(bits_equal(u, v) for u, v in zip(x, y))
        else:
            ok = bits_equal(x, y)
        if not ok:
            return False
    return True


def oracle_frame(frame, cin, cout, w, h, levels, normalize=False):
    r = po.preprocess(frame, cin, cout, w, h, normalize)
    lv = [r.level0]
    for _ in range(1, levels):
        lv.append(orc.gaussian_blur_down(lv[-1]))
    return r, lv, [orc.sobel_gradients(x) for x in lv]


def test_equals_opencv_on_every_fixture(aligner, torch_mod, fx):
    from deepfactors_b200.aligners import PreprocessBatch
    runs = [str(r) for r in fx["runs"]]
    # the whole fixture in two batches: frames of one output camera each go together
    by_cam = {}
    for run in runs:
        frame, cin, cout, w, h = run_frame(fx, run)
        by_cam.setdefault((tuple(cout), w, h), []).append((run, frame, cin))
    for (cout, w, h), group in by_cam.items():
        outs = PreprocessBatch(aligner, [dev_frame(torch_mod, f) for _, f, _ in group], [Cam(c) for _, _, c in group],
                               Cam(cout, w, h), 1, grads=False)
        for (run, frame, _), o in zip(group, outs):
            o = host(o)
            assert [sha(o["color"]), sha(o["gray"]), sha(o["levels"][0])] == list(fx[f"sha_{run}"]), run
            if run == "a_1047":
                assert np.array_equal(o["color"], fx["rows_color"]) and np.array_equal(o["gray"], fx["rows_gray"])
                assert bits_equal(o["levels"][0], fx["rows_float"])
            if run.startswith("b_"):
                assert np.array_equal(o["color"], frame)


def random_items(rng, count):
    items = []
    for i in range(count):
        sw, sh = int(rng.integers(8, 400)), int(rng.integers(8, 300))
        f_in = np.float32(rng.uniform(0.4, 1.5) * sw)
        cin = np.float32([f_in, f_in * rng.uniform(0.8, 1.2), sw * rng.uniform(0.3, 0.7), sh * rng.uniform(0.3, 0.7)])
        items.append((rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8), cin, int(rng.integers(0, 13)) if i % 2 else 0))
    return items


def test_random_frames_with_padded_pitches_equal_the_oracle(aligner, torch_mod):
    from deepfactors_b200.aligners import BuildImagePyramid, PreprocessBatch
    torch = torch_mod
    rng = np.random.default_rng(5)
    for w, h, levels in ((256, 192, 4), (203, 117, 3), (64, 48, 1)):
        cout = np.float32([0.9 * w, 0.85 * w, 0.45 * w, 0.55 * h])
        items = random_items(rng, 9)
        norm = [i % 3 == 1 for i in range(len(items))]
        outs = PreprocessBatch(aligner, [dev_frame(torch, f, pad) for f, _, pad in items], [Cam(c) for _, c, _ in items],
                               Cam(cout, w, h), levels, normalize=norm)
        for (frame, cin, _), o, nz in zip(items, outs, norm):
            d = host(o)
            r, lv, gd = oracle_frame(frame, cin, cout, w, h, levels, nz)
            assert np.array_equal(d["color"], r.color) and np.array_equal(d["gray"], r.gray)
            assert all(bits_equal(a, b) for a, b in zip(d["levels"], lv))
            assert all(bits_equal(a, b) for a, b in zip(d["grads"], gd))
            if nz:
                assert tuple(d["stats"]) == r.stats
            else:
                assert d["stats"] is None
            # the levels equal dfk_build_image_pyramid run on the device's level 0
            imgs = [o.levels[0].clone()] + [torch.empty_like(t) for t in o.levels[1:]]
            grads = [torch.empty_like(t) for t in o.grads]
            BuildImagePyramid(imgs, grads)
            torch.cuda.synchronize()
            assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(imgs, o.levels))
            assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(grads, o.grads))


def test_padded_output_views(aligner, torch_mod):
    """the C call on outputs whose rows are padded writes only the W_o x H_o pixels, as the packed outputs hold them"""
    torch = torch_mod
    rng = np.random.default_rng(8)
    frame = rng.integers(0, 256, (120, 160, 3), dtype=np.uint8)
    cin, cout, w, h = np.float32([150, 150, 80, 60]), np.float32([100, 100, 50.5, 40.5]), 101, 77
    src = dev_frame(torch, frame, 5)
    color = torch.full((h, 3 * w + 13), 9, dtype=torch.uint8, device="cuda")
    gray = torch.full((h, w + 7), 9, dtype=torch.uint8, device="cuda")
    l0 = torch.full((h, w + 3), -9.0, device="cuda")
    l1 = torch.full((h // 2, w // 2 + 5), -9.0, device="cuda")
    g0 = torch.full((h, 2 * w + 6), -9.0, device="cuda")
    g1 = torch.full((h // 2, 2 * (w // 2) + 2), -9.0, device="cuda")
    img = lambda t, ww, hh: _lib.DfkImage(t.data_ptr(), t.stride(0) * t.element_size(), ww, hh)
    lv = (_lib.DfkImage * 2)(img(l0, w, h), img(l1, w // 2, h // 2))
    gd = (_lib.DfkImage * 2)(img(g0, w, h), img(g1, w // 2, h // 2))
    it = _lib.DfkPreprocessItem(_lib.DfkImage(src.data_ptr(), src.stride(0), 160, 120),
                                _lib.DfkCamera(*cin, 160, 120), _lib.DfkCamera(*cout, w, h),
                                img(color, w, h), img(gray, w, h), C.cast(lv, C.POINTER(_lib.DfkImage)),
                                C.cast(gd, C.POINTER(_lib.DfkImage)), 0)
    aligner._hd.use_torch_stream()
    _lib.check(aligner._hd.h, _lib.lib().dfk_preprocess_batch(aligner._hd.h, (_lib.DfkPreprocessItem * 1)(it), 1, 2,
                                                               None))
    torch.cuda.synchronize()
    r, lvs, gds = oracle_frame(frame, cin, cout, w, h, 2)
    assert np.array_equal(color[:, :3 * w].cpu().numpy().reshape(h, w, 3), r.color) and (color[:, 3 * w:] == 9).all()
    assert np.array_equal(gray[:, :w].cpu().numpy(), r.gray) and (gray[:, w:] == 9).all()
    assert bits_equal(l0[:, :w].cpu().numpy(), lvs[0]) and (l0[:, w:] == -9).all()
    assert bits_equal(l1[:, :w // 2].cpu().numpy(), lvs[1]) and (l1[:, w // 2:] == -9).all()
    assert bits_equal(g0[:, :2 * w].cpu().numpy().reshape(h, w, 2), gds[0]) and (g0[:, 2 * w:] == -9).all()
    assert bits_equal(g1[:, :2 * (w // 2)].cpu().numpy().reshape(h // 2, w // 2, 2), gds[1])


def test_batch_independence_and_repeatability(aligner, torch_mod):
    from deepfactors_b200.aligners import PreprocessBatch
    torch = torch_mod
    rng = np.random.default_rng(11)
    items = random_items(rng, 64)
    w, h = 96, 72
    cout = Cam(np.float32([80.0, 78.0, 47.5, 35.5]), w, h)
    norm = [i % 4 == 0 for i in range(64)]
    frames = [dev_frame(torch, f, pad) for f, _, pad in items]
    cams = [Cam(c) for _, c, _ in items]
    a = [host(o) for o in PreprocessBatch(aligner, frames, cams, cout, 3, normalize=norm)]
    b = [host(o) for o in PreprocessBatch(aligner, frames, cams, cout, 3, normalize=norm)]
    assert all(frames_equal(x, y) for x, y in zip(a, b))
    for i in (0, 1, 5, 63):
        alone = host(PreprocessBatch(aligner, [frames[i]], [cams[i]], cout, 3, normalize=norm[i])[0])
        assert frames_equal(alone, a[i]), i


def test_device_gray_drives_orb_as_the_oracle_gray(aligner, torch_mod, fx):
    from deepfactors_b200.aligners import OrbDetectBatch, PreprocessBatch
    torch = torch_mod
    frames, cams = [], []
    for run in ("a_1047", "a640_1052", "c_1047"):
        frame, cin, cout, w, h = run_frame(fx, run)
        out = PreprocessBatch(aligner, [dev_frame(torch, frame)], [Cam(cin)], Cam(cout, w, h), 0)[0]
        r = po.preprocess(frame, cin, cout, w, h)
        d = OrbDetectBatch(aligner, [out.gray, torch.from_numpy(r.gray).cuda()], 500, 20)
        c = d.host_counts()
        assert c[0] == c[1] > 0
        o = d.offsets
        for t in (d.keypoints, d.descriptors, d.angles, d.responses):
            assert torch.equal(t[o[0]:o[0] + c[0]], t[o[1]:o[1] + c[1]])


def test_rejected_calls_write_nothing(aligner, torch_mod):
    torch = torch_mod
    frame = dev_frame(torch, np.random.default_rng(3).integers(0, 256, (60, 80, 3), dtype=np.uint8))
    w, h = 40, 30
    color = torch.full((h, w, 3), 7, dtype=torch.uint8, device="cuda")
    gray = torch.full((h, w), 7, dtype=torch.uint8, device="cuda")
    l0 = torch.full((h, w), -7.0, device="cuda")
    l1 = torch.full((h // 2, w // 2), -7.0, device="cuda")
    g0 = torch.full((h, w, 2), -7.0, device="cuda")
    stats = torch.full((4, 2), -7.0, dtype=torch.float64, device="cuda")
    V = lambda t, p, ww, hh: _lib.DfkImage(t.data_ptr(), p, ww, hh)
    lv = (_lib.DfkImage * 2)(V(l0, 4 * w, w, h), V(l1, 4 * (w // 2), w // 2, h // 2))
    lv_bad = (_lib.DfkImage * 2)(V(l0, 4 * w, w, h), V(l1, 4 * (w // 2), w // 2 + 1, h // 2))  # not the halved size
    gd = (_lib.DfkImage * 2)(V(g0, 8 * w, w, h), V(g0, 8 * w, w, h))  # level 1 gradient of the wrong size
    src = V(frame, 240, 80, 60)
    cin, cout = _lib.DfkCamera(60, 60, 40, 30, 80, 60), _lib.DfkCamera(30, 30, 20, 15, w, h)
    P = lambda a: C.cast(a, C.POINTER(_lib.DfkImage))

    def item(**kw):
        d = dict(src=src, src_cam=cin, out_cam=cout, color=V(color, 3 * w, w, h), gray=V(gray, w, w, h), levels=P(lv),
                 grads=None, normalize=1)
        d.update(kw)
        return _lib.DfkPreprocessItem(**d)

    def call(items, levels=2, st=None):
        arr = (_lib.DfkPreprocessItem * len(items))(*items)
        s = _lib.lib().dfk_preprocess_batch(aligner._hd.h, arr, len(items), levels,
                                            st if st is not None else stats.data_ptr())
        return s, _lib.lib().dfk_last_error(aligner._hd.h)

    good = item()
    bad_items = [
        item(src=_lib.DfkImage(None, 240, 80, 60)),           # null source
        item(src=V(frame, 200, 80, 60)),                                          # pitch < 3 width
        item(src=V(frame, 240 * 300, 80, 20000)),                                 # too tall
        item(src_cam=_lib.DfkCamera(0, 60, 40, 30, 80, 60)),                      # fx = 0
        item(out_cam=_lib.DfkCamera(30, float("nan"), 20, 15, w, h)),             # NaN
        item(out_cam=_lib.DfkCamera(30, 30, 20, 15, w + 0.5, h)),                 # fractional size
        item(out_cam=_lib.DfkCamera(30, 30, 20, 15, 0, h)),                       # empty output
        item(color=V(color, 3 * w - 1, w, h)),                                    # colour pitch
        item(gray=V(gray, w, w + 1, h)),                                          # gray size
        item(levels=None),                                                        # no levels
        item(levels=P(lv_bad)),                                                   # level 1 size
        item(grads=P(gd)),                                                        # gradient size
        item(normalize=2),                                                        # normalize not 0 / 1
    ]
    for bad in bad_items:
        st, msg = call([good, good, bad])
        assert st == _lib.DFK_ERR_INVALID_ARG and b"item 2" in msg, msg
    # negative levels, more than DFK_PREPROCESS_MAX_LEVELS (rejected before any host buffer is sized by them),
    # misaligned stats
    for args in (dict(levels=-1), dict(levels=16), dict(levels=2 ** 31 - 1), dict(st=stats.data_ptr() + 4)):
        st, _ = call([good], **args)
        assert st == _lib.DFK_ERR_INVALID_ARG
    st, msg = call([item(out_cam=_lib.DfkCamera(30, 30, 20, 15, 1, 1))], levels=2)  # level 1 would be 0 x 0
    assert st == _lib.DFK_ERR_INVALID_ARG and b"item 0" in msg
    torch.cuda.synchronize()
    assert (color == 7).all() and (gray == 7).all() and (l0 == -7).all() and (l1 == -7).all() and (g0 == -7).all()
    assert (stats == -7).all()
    st, _ = call([good])
    torch.cuda.synchronize()
    r = po.preprocess(frame.cpu().numpy(), [60, 60, 40, 30], [30, 30, 20, 15], w, h, normalize=True)
    assert st == 0 and tuple(stats[0].cpu().numpy()) == r.stats and (stats[1:] == -7).all()


def test_frame_preprocessor_facade():
    """df::FramePreprocessor against the C call it wraps (tests/cpp/preprocess_test)"""
    exe = os.path.join(HERE, "cpp", "preprocess_test")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "preprocess_test OK" in r.stdout
