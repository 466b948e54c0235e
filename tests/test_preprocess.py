"""CPU checks of the frame preprocessing's specification (include/dfk.h dfk_preprocess_batch, DESIGN.md section 4.10)
through its oracle (preprocess_oracle/), against cv2 (skipped without it) and tests/golden/preprocess_frames.npz:
- the map equals cv2.initUndistortRectifyMap(..., CV_32FC1) bit for bit over 300 random cameras and sizes, and iR
  equals cv2.invert(DECOMP_LU);
- the colour equals cv2.remap(INTER_LINEAR) on both fixture images and on random images x random cameras, outputs that
  leave the source included; the gray equals cv2.cvtColor(COLOR_RGB2GRAY), the float convertTo(CV_32FC1, 1 / 255.0);
- (mu, sigma) agree with cv2.meanStdDev to 1e-12 relative, and f' follows from them;
- the oracle reproduces every fixture digest, and the stored run row by row;
- the weight table equals an independent computation (and whether its fix-up fired is reported);
- the ctypes layout of DfkPreprocessItem matches the header."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest

from preprocess_oracle import preprocess_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "preprocess_frames.npz")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(FIXTURE))


@pytest.fixture(scope="module")
def cv2():
    return pytest.importorskip("cv2")


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def K(c):
    c = np.asarray(c, np.float64)
    return np.array([[c[0], 0, c[2]], [0, c[1], c[3]], [0, 0, 1]], np.float64)


def run_frame(fx, run):
    """(frame, in_cam, out_cam, w, h) of a fixture run: a640 frames are the 2x pixel repeat of the stored image"""
    name, img = str(run).rsplit("_", 1)
    c = fx[f"cfg_{name}"]
    frame = fx[f"image_{img}"]
    if int(c[0]) == 2:
        frame = np.ascontiguousarray(np.repeat(np.repeat(frame, 2, axis=0), 2, axis=1))
    return frame, np.float32(c[1:5]), np.float32(c[5:9]), int(c[9]), int(c[10])


def random_cam(rng, sw, sh, w, h, leave=False):
    """a source camera at sw x sh and an output camera at w x h; leave: the output reaches well past the source"""
    f_in = np.float32(rng.uniform(0.4, 1.5) * sw)
    cin = np.float32([f_in, f_in * rng.uniform(0.8, 1.2), sw * rng.uniform(0.3, 0.7), sh * rng.uniform(0.3, 0.7)])
    zoom = rng.uniform(0.15, 0.6) if leave else rng.uniform(0.7, 2.5)
    f_out = np.float32(f_in * zoom * w / sw)
    cout = np.float32([f_out, f_out * rng.uniform(0.8, 1.2), w * rng.uniform(0.2, 0.8), h * rng.uniform(0.2, 0.8)])
    return cin, cout


def convert_to_float(cv2, gray):
    """gray.convertTo(CV_32FC1, 1 / 255.0): cv2.normalize with NORM_INF and alpha 1 calls exactly that when the
    largest value is 255 (a 255 row is appended and cropped)"""
    s = np.vstack([gray, np.full((1, gray.shape[1]), 255, np.uint8)])
    return cv2.normalize(s, None, alpha=1.0, beta=0.0, norm_type=cv2.NORM_INF, dtype=cv2.CV_32F)[:-1]


def test_map_equals_opencv_on_random_cameras(cv2):
    rng = np.random.default_rng(0)
    for _ in range(300):
        sw, sh = int(rng.integers(16, 700)), int(rng.integers(16, 500))
        w, h = int(rng.integers(1, 400)), int(rng.integers(1, 300))
        cin, cout = random_cam(rng, sw, sh, w, h, leave=bool(rng.integers(0, 2)))
        m1, m2 = cv2.initUndistortRectifyMap(K(cin), None, None, K(cout), (w, h), cv2.CV_32FC1)
        o1, o2 = po.init_map(cin, cout, w, h)
        assert np.array_equal(m1.view(np.int32), o1.view(np.int32)) and np.array_equal(m2.view(np.int32),
                                                                                        o2.view(np.int32))
        _, inv = cv2.invert(K(cout), flags=cv2.DECOMP_LU)
        assert np.array_equal(inv.view(np.int64), po.inverse(cout).view(np.int64))


def test_remap_gray_and_float_equal_opencv(cv2, fx):
    rng = np.random.default_rng(1)
    cases = []
    for img in ("1047", "1052"):
        for name in ("a", "c", "d", "e"):
            c = fx[f"cfg_{name}"]
            cases.append((fx[f"image_{img}"], np.float32(c[1:5]), np.float32(c[5:9]), int(c[9]), int(c[10])))
    for i in range(24):
        sw, sh = int(rng.integers(8, 400)), int(rng.integers(8, 300))
        w, h = int(rng.integers(1, 300)), int(rng.integers(1, 200))
        cases.append((rng.integers(0, 256, (sh, sw, 3), dtype=np.uint8), *random_cam(rng, sw, sh, w, h, i % 3 == 0),
                      w, h))
    left = 0
    for frame, cin, cout, w, h in cases:
        m1, m2 = cv2.initUndistortRectifyMap(K(cin), None, None, K(cout), (w, h), cv2.CV_32FC1)
        color = cv2.remap(frame, m1, m2, cv2.INTER_LINEAR).reshape(h, w, 3)
        gray = cv2.cvtColor(color, cv2.COLOR_RGB2GRAY).reshape(h, w)
        r = po.preprocess(frame, cin, cout, w, h)
        assert np.array_equal(r.color, color)
        assert np.array_equal(r.gray, gray)
        assert np.array_equal(r.level0.view(np.int32), convert_to_float(cv2, gray).view(np.int32))
        sh_, sw_ = frame.shape[:2]
        left += int(((m1 < 0) | (m2 < 0) | (m1 > sw_ - 1) | (m2 > sh_ - 1)).any())
    assert left >= 10  # outputs that reach outside the source (the BORDER_CONSTANT ring) are covered


def test_gray_rule_is_the_15_bit_one(cv2):
    img = np.random.default_rng(2).integers(0, 256, (300, 400, 3), dtype=np.uint8)
    g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY).astype(np.int64)
    c = img.astype(np.int64)
    assert np.array_equal(g, (9798 * c[..., 0] + 19235 * c[..., 1] + 3735 * c[..., 2] + (1 << 14)) >> 15)
    assert not np.array_equal(g, (4899 * c[..., 0] + 9617 * c[..., 1] + 1868 * c[..., 2] + (1 << 13)) >> 14)


def test_normalisation_stats_agree_with_meanstddev(cv2, fx):
    for run in fx["runs"]:
        frame, cin, cout, w, h = run_frame(fx, run)
        if w * h < 4:
            continue
        r = po.preprocess(frame, cin, cout, w, h)
        n = po.preprocess(frame, cin, cout, w, h, normalize=True)
        mean, sd = cv2.meanStdDev(r.level0)
        mu, sigma = n.stats
        assert abs(mu - mean[0, 0]) <= 1e-12 * abs(mean[0, 0]), run
        assert abs(sigma - sd[0, 0]) <= 1e-12 * abs(sd[0, 0]), run
        assert (mu, sigma) == po.stats_of(r.level0)
        want = ((r.level0.astype(np.float64) - mu) / sigma).astype(np.float32)
        assert np.array_equal(n.level0.view(np.int32), want.view(np.int32)), run


def test_oracle_reproduces_every_fixture_run(fx):
    assert len(fx["runs"]) == 14 and str(fx["cv2_version"]) == "4.13.0"
    for run in fx["runs"]:
        frame, cin, cout, w, h = run_frame(fx, run)
        r = po.preprocess(frame, cin, cout, w, h)
        assert [sha(r.color), sha(r.gray), sha(r.level0)] == list(fx[f"sha_{run}"]), run
        if str(run) == "a_1047":
            assert np.array_equal(r.color, fx["rows_color"]) and np.array_equal(r.gray, fx["rows_gray"])
            assert np.array_equal(r.level0.view(np.int32), fx["rows_float"].view(np.int32))
        if str(run).startswith("b_"):  # identity: the source unchanged
            assert np.array_equal(r.color, frame)


def test_weight_table():
    tab, fired = po.weights()
    t = np.arange(32, dtype=np.float32) * np.float32(1.0 / 32)
    wy = np.stack([np.float32(1) - t, t], axis=1)  # [ty, dy]
    wx = wy
    prod = (wy[:, None, :, None] * wx[None, :, None, :]).astype(np.float32)  # [ty, tx, dy, dx]
    want = np.rint(prod * np.float32(32768)).astype(np.int32).reshape(32, 32, 4)
    assert (want.sum(axis=2) == 32768).all()
    print(f"weight table fix-up fired for {fired} of 1024 entries")
    assert fired == 0
    assert np.array_equal(tab, want)


def test_struct_layouts_match_the_header(tmp_path):
    """offsets and sizes of DfkPreprocessItem as the C compiler lays them out"""
    from deepfactors_b200 import _lib
    src = tmp_path / "layout.c"
    fields = [f[0] for f in _lib.DfkPreprocessItem._fields_]
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "dfk.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(DfkPreprocessItem));']
    lines += [f'printf("{f} %zu\\n", offsetof(DfkPreprocessItem, {f}));' for f in fields]
    lines += ['printf("DFK_PREPROCESS_MAX_LEVELS %d\\n", DFK_PREPROCESS_MAX_LEVELS);', "return 0; }"]
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                         check=True).stdout.splitlines())
    assert int(got["size"]) == ctypes.sizeof(_lib.DfkPreprocessItem)
    for f in fields:
        assert int(got[f]) == getattr(_lib.DfkPreprocessItem, f).offset, f
    # 16384, 8192, ..., 1: the levels of a frame of DFK_ORB_MAX_SIDE
    assert int(got["DFK_PREPROCESS_MAX_LEVELS"]) == _lib.PREPROCESS_MAX_LEVELS == _lib.ORB_MAX_SIDE.bit_length()
