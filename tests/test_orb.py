"""CPU checks of the ORB detector's specification (include/dfk.h dfk_orb_detect_batch, DESIGN.md section 4.9) through
its oracle (orb_oracle/), against cv2.ORB_create(nfeatures, 1.2, 1) as recorded in tests/golden/orb_features.npz on the
images of tests/orb_images.py:
- the oracle equals cv2 bit for bit on every recorded image and setting: keypoint set, angles, responses, descriptors
  (their digest in the detector's order, and every row where the fixture holds the run in full);
- the generated pattern header equals the recovered table of the fixture;
- both cuts keep every tie (constructed cases);
- the ctypes layout of DfkOrbItem matches the header."""
import ctypes
import hashlib
import os
import re
import subprocess

import numpy as np
import pytest

from orb_images import CONFIGS, device_order, digest, images
from orb_oracle import orb_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "orb_features.npz")


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(FIXTURE))


@pytest.fixture(scope="module")
def imgs():
    return images()


def runs(imgs):
    return [(name, nf, t) for name in sorted(imgs) for nf, t in CONFIGS]


def test_fixture_covers_the_issue_settings(fx, imgs):
    assert {(int(a), int(b)) for a, b in fx["configs"]} == set(CONFIGS) == {(500, 20), (200, 20), (2000, 10)}
    assert {im.shape for im in imgs.values()} == {(240, 320), (480, 640), (192, 256)}
    for name, nf, t in runs(imgs):
        assert f"{name}_{nf}_{t}_digest" in fx
    # the tie-heavy image keeps more than nfeatures at the response cut
    assert int(fx["dots_clean_200_20_count"]) > 200 and int(fx["dots_clean_500_20_count"]) > 500


def test_images_are_reproducible(imgs):
    """the fixture's images are rebuilt in integer arithmetic: pin them"""
    want = {'1047_640': '48d53751cc2dcc7a', '1052_256': 'cce8ff7b74ee1c74', 'dots': '7fc161d0fa59171e', 'dots_clean': '4157bc2b498d7798'}
    for name, h in want.items():
        assert hashlib.sha256(imgs[name].tobytes()).hexdigest()[:16] == h, name


def test_oracle_equals_opencv_bit_for_bit(fx, imgs):
    for name, nf, t in runs(imgs):
        key = f"{name}_{nf}_{t}"
        r = oo.detect(imgs[name], nf, t)
        assert r.count == int(fx[f"{key}_count"]), key
        if f"{key}_kp" in fx:  # the run in full: row by row, cv2's rows permuted into the detector's order
            kp, ang, resp, desc = (fx[f"{key}_{s}"] for s in ("kp", "angle", "response", "desc"))
            perm = device_order(kp, resp)
            assert np.array_equal(r.keypoints, kp[perm]), key
            assert np.array_equal(r.angles.view(np.uint32), ang[perm].view(np.uint32)), key
            assert np.array_equal(r.responses.view(np.uint32), resp[perm].view(np.uint32)), key
            assert np.array_equal(r.descriptors, desc[perm]), key
        # the oracle's rows are in the detector's order already
        assert digest(r.keypoints, r.angles, r.responses, r.descriptors, order=False) == str(fx[f"{key}_digest"]), key


def test_keypoints_are_integer_positions_inside_the_border(fx, imgs):
    for name, nf, t in runs(imgs):
        key = f"{name}_{nf}_{t}_kp"
        if key not in fx:
            continue
        kp = fx[key]
        h, w = imgs[name].shape
        assert np.array_equal(kp, np.round(kp))
        assert (kp >= 31).all() and (kp[:, 0] < w - 31).all() and (kp[:, 1] < h - 31).all()


def test_pattern_header_equals_fixture(fx):
    with open(os.path.join(ROOT, "deepfactors_b200", "csrc", "dfk_orb_pattern.h")) as f:
        text = f.read()
    body = text.split("#define DFK_ORB_PATTERN_DATA", 1)[1].split("#endif", 1)[0]
    table = np.array([int(v) for v in re.findall(r"-?\d+", body)], np.int32).reshape(256, 4)
    assert np.array_equal(table, fx["pattern"])
    assert np.array_equal(oo.pattern(), fx["pattern"])  # the table the oracle was compiled with
    assert tuple(fx["pattern"][0]) == (8, -3, 9, 5) and tuple(fx["pattern"][1]) == (4, 2, 7, -12)


def test_small_images_have_no_features():
    rng = np.random.default_rng(0)
    for h, w in ((62, 200), (200, 62), (10, 10)):
        assert oo.detect(rng.integers(0, 256, (h, w), dtype=np.uint8), 500, 0).count == 0
    assert oo.detect(rng.integers(0, 256, (63, 63), dtype=np.uint8), 500, 0).count <= 1


def dot_grid(levels, step=9, size=(240, 320), background=40):
    """isolated single-pixel corners on a grid, brightness levels[k] for the k-th dot in raster order (cycled)"""
    img = np.full(size, background, np.uint8)
    k = 0
    for y in range(31 + 4, size[0] - 31, step):
        for x in range(31 + 4, size[1] - 31, step):
            img[y, x] = levels[k % len(levels)]
            k += 1
    return img, k


def test_first_cut_keeps_every_tie():
    # every dot has the same FAST score: the first cut (2 nfeatures) keeps them all, and so does the second, since
    # every response ties too
    img, ndots = dot_grid([200])
    nf = 10
    assert ndots > 2 * nf
    scores = oo.fast_scores(img, 20)
    assert len(np.unique(scores[scores >= 0])) == 1
    r = oo.detect(img, nf, 20)
    assert r.count == ndots
    assert len(np.unique(r.responses)) == 1
    # the ties come out in raster order
    assert np.array_equal(np.lexsort((r.keypoints[:, 0], r.keypoints[:, 1])), np.arange(ndots))


def test_second_cut_keeps_every_tie_and_only_those():
    # two brightness levels: the brighter dots respond more; with nfeatures inside the brighter group every brighter
    # dot is kept and no dimmer one
    img, ndots = dot_grid([250, 120, 120])
    nbright = (ndots + 2) // 3
    for nf in (1, nbright // 2, nbright):
        r = oo.detect(img, nf, 20)
        assert r.count == nbright, nf
        assert len(np.unique(r.responses)) == 1
    # one past the brighter group: every dimmer dot ties at the cut
    assert oo.detect(img, nbright + 1, 20).count == ndots
    # capacity: the count stays true, only the first rows are written
    r = oo.detect(img, 1, 20, capacity=5)
    assert r.count == nbright and len(r.keypoints) == 5


def test_struct_layouts_match_the_header(tmp_path):
    """offsets and sizes of DfkOrbItem as the C compiler lays them out"""
    from deepfactors_b200 import _lib
    src = tmp_path / "layout.c"
    fields = {"DfkOrbItem": [f[0] for f in _lib.DfkOrbItem._fields_]}
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "dfk.h"', "int main(void) {"]
    for s, fs in fields.items():
        lines.append(f'printf("{s} %zu\\n", sizeof({s}));')
        lines += [f'printf("{s}.{f} %zu\\n", offsetof({s}, {f}));' for f in fs]
    lines += ['printf("DFK_ORB_MAX_SIDE %d\\n", DFK_ORB_MAX_SIDE);', "return 0; }"]
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True,
                                                         check=True).stdout.splitlines())
    for s, fs in fields.items():
        cls = getattr(_lib, s)
        assert int(got[s]) == ctypes.sizeof(cls)
        for f in fs:
            assert int(got[f"{s}.{f}"]) == getattr(cls, f).offset, (s, f)
    assert int(got["DFK_ORB_MAX_SIDE"]) == _lib.ORB_MAX_SIDE
