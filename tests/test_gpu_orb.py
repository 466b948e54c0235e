"""ORB features on the device (dfk_orb_detect_batch, aligners.OrbDetectBatch) against OpenCV
(tests/golden/orb_features.npz, cv2.ORB_create(nfeatures, 1.2, 1) on the images of tests/orb_images.py) and the CPU
oracle (orb_oracle):

- every recorded image and setting bit for bit against cv2 -- keypoints, angles, responses and descriptors -- in the
  documented order (response descending, then y, then x): row by row where the fixture holds the run in full, by digest
  everywhere;
- random images bit for bit against the oracle, including a count above the capacity;
- an item's output does not depend on the rest of its batch (mixed sizes, one image below 63 x 63);
- two runs are bit for bit equal;
- invalid items are rejected before anything is written;
- device features -> dfk_reprojection_match_batch gives exactly the matches of cv2's features permuted into the
  device order;
- df::OrbDetector of the C++ facade (tests/cpp/orb_test)."""
import os
import subprocess

import numpy as np
import pytest

from deepfactors_b200 import _lib
from match_scenes import Cam
from orb_images import CONFIGS, device_order, digest, images
from orb_oracle import orb_oracle as oo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE_CAM = Cam(fx=262.5, fy=262.5, u0=160.0, v0=120.0, width=320.0, height=240.0)


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
    return dict(np.load(os.path.join(HERE, "golden", "orb_features.npz")))


def dev(torch, img):
    return torch.from_numpy(np.ascontiguousarray(img, np.uint8)).cuda()


def detect(aligner, torch, imgs, nf=500, t=20, capacity=None):
    """OrbDetectBatch, read back: per image (count, keypoints, angles, responses, descriptors) of the written rows"""
    from deepfactors_b200.aligners import OrbDetectBatch
    out = OrbDetectBatch(aligner, [dev(torch, im) for im in imgs], nf, t, capacity)
    counts = out.counts.cpu().numpy()
    kp, ang, resp, desc = (x.cpu().numpy() for x in (out.keypoints, out.angles, out.responses, out.descriptors))
    res = []
    for i, c in enumerate(counts):
        o, m = int(out.offsets[i]), min(int(c), int(out.capacities[i]))
        res.append((int(c), kp[o:o + m], ang[o:o + m], resp[o:o + m], desc[o:o + m]))
    return res


def same(a, b):
    """bit for bit: count and every written row"""
    return a[0] == b[0] and all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
                                for x, y in zip(a[1:], b[1:]))


def oracle(img, nf, t, capacity):
    r = oo.detect(img, nf, t, capacity)
    return (r.count, r.keypoints, r.angles, r.responses, r.descriptors)


def test_equals_opencv_on_every_fixture(aligner, torch_mod, fx):
    imgs = images()
    names = sorted(imgs)
    for nf, t in CONFIGS:
        got = detect(aligner, torch_mod, [imgs[n] for n in names], nf, t, capacity=4 * nf)
        for name, (count, kp, ang, resp, desc) in zip(names, got):
            key = f"{name}_{nf}_{t}"
            assert count == int(fx[f"{key}_count"]), key
            if f"{key}_kp" in fx:  # the run in full: row by row, cv2's rows permuted into the detector's order
                ckp, cang, cresp, cdesc = (fx[f"{key}_{s}"] for s in ("kp", "angle", "response", "desc"))
                perm = device_order(ckp, cresp)
                assert np.array_equal(kp, ckp[perm]), key
                assert np.array_equal(ang.view(np.uint32), cang[perm].view(np.uint32)), key
                assert np.array_equal(resp.view(np.uint32), cresp[perm].view(np.uint32)), key
                assert np.array_equal(desc, cdesc[perm]), key
            # every run: the device rows, as they come, hash to cv2's rows in the detector's order
            assert digest(kp, ang, resp, desc, order=False) == str(fx[f"{key}_digest"]), key


def random_image(rng, h, w):
    """smooth blobs plus noise: corners of many scores, responses and angles"""
    y, x = np.mgrid[0:h, 0:w]
    img = np.full((h, w), 80.0)
    for _ in range(h * w // 400):
        cy, cx, r, a = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(1.5, 6), rng.uniform(-70, 120)
        img += a * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2 * r * r))
    return np.clip(img + rng.normal(0, 4, (h, w)), 0, 255).astype(np.uint8)


def test_random_images_equal_the_oracle(aligner, torch_mod):
    rng = np.random.default_rng(5)
    cases = [((240, 320), 500, 20), ((192, 256), 200, 12), ((480, 640), 1000, 15), ((100, 300), 50, 30),
             ((333, 277), 300, 0), ((240, 320), 8192, 5)]
    for (h, w), nf, t in cases:
        img = random_image(rng, h, w)
        got = detect(aligner, torch_mod, [img], nf, t, capacity=2 * nf)[0]
        assert same(got, oracle(img, nf, t, 2 * nf)), ((h, w), nf, t)
    # a count above the capacity: the true count, and the first capacity rows
    img = dot_grid()
    want = oracle(img, 10, 20, 12)
    assert want[0] > 12
    got = detect(aligner, torch_mod, [img], 10, 20, capacity=12)[0]
    assert same(got, want)


def dot_grid(h=240, w=320, step=9):
    img = np.full((h, w), 40, np.uint8)
    img[35:h - 31:step, 35:w - 31:step] = 200  # isolated equal corners: every score and response ties
    return img


def test_batch_independence_and_repeatability(aligner, torch_mod):
    rng = np.random.default_rng(9)
    imgs = [random_image(rng, 240, 320), random_image(rng, 50, 80), random_image(rng, 480, 640),
            random_image(rng, 63, 63), random_image(rng, 192, 256), dot_grid()]
    nf = [500, 500, 300, 10, 200, 20]
    t = [20, 20, 10, 0, 25, 20]
    batch = None
    for rep in range(2):
        from deepfactors_b200.aligners import OrbDetectBatch
        out = OrbDetectBatch(aligner, [dev(torch_mod, im) for im in imgs], nf, t, [4 * x for x in nf])
        cur = [x.cpu().numpy().copy() for x in (out.keypoints, out.angles, out.responses, out.descriptors, out.counts)]
        if batch is None:
            batch = (cur, out.offsets)
        else:  # two runs, bit for bit
            for a, b in zip(batch[0], cur):
                assert np.array_equal(a.view(np.uint8), b.view(np.uint8))
    cur, offsets = batch
    counts = cur[4]
    assert counts[1] == 0
    for i, im in enumerate(imgs):
        alone = detect(aligner, torch_mod, [im], nf[i], t[i], 4 * nf[i])[0]
        o, m = int(offsets[i]), min(int(counts[i]), 4 * nf[i])
        assert same((int(counts[i]), *(x[o:o + m] for x in cur[:4])), alone), i
        assert same(alone, oracle(im, nf[i], t[i], 4 * nf[i])), i


def test_rejected_calls_write_nothing(aligner, torch_mod):
    torch = torch_mod
    img = dev(torch, random_image(np.random.default_rng(2), 240, 320))
    rows = 1000
    kp = torch.full((rows, 2), -7.0, device="cuda")
    desc = torch.full((rows, 32), 7, dtype=torch.uint8, device="cuda")
    ang = torch.full((rows,), -7.0, device="cuda")
    resp = torch.full((rows,), -7.0, device="cuda")
    counts = torch.full((4,), -7, dtype=torch.int32, device="cuda")
    good = _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 320, 320, 240), 200, 20, 200)

    def call(items, d=None):
        arr = (_lib.DfkOrbItem * len(items))(*items)
        st = _lib.lib().dfk_orb_detect_batch(aligner._hd.h, arr, len(items), kp.data_ptr(),
                                             d if d is not None else desc.data_ptr(), ang.data_ptr(),
                                             resp.data_ptr(), counts.data_ptr())
        return st, _lib.lib().dfk_last_error(aligner._hd.h)

    bad_items = [
        _lib.DfkOrbItem(_lib.DfkImage(None, 320, 320, 240), 200, 20, 200),     # null image
        _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 100, 320, 240), 200, 20, 200),  # pitch < width
        _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 320, 320, 240), 0, 20, 200),     # nfeatures 0
        _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 320, 320, 240), 9000, 20, 9000),  # > DFK_MATCH_MAX_QUERIES
        _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 320, 320, 240), 200, 256, 200),  # threshold
        _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 320, 320, 240), 200, 20, 199),   # capacity < nfeatures
        _lib.DfkOrbItem(_lib.DfkImage(img.data_ptr(), 20000, 20000, 10), 200, 20, 200),  # too wide
    ]
    for bad in bad_items:
        st, msg = call([good, good, bad])
        assert st == _lib.DFK_ERR_INVALID_ARG and b"item 2" in msg, msg
    st, _ = call([good], d=desc.data_ptr() + 4)  # misaligned descriptors
    assert st == _lib.DFK_ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert (kp == -7).all() and (desc == 7).all() and (ang == -7).all() and (resp == -7).all() and (counts == -7).all()
    st, _ = call([good])
    torch.cuda.synchronize()
    want = oo.detect(img.cpu().numpy(), 200, 20, 200).count
    assert st == 0 and int(counts[0]) == want > 0 and (counts[1:] == -7).all()


def test_device_features_drive_the_matcher_as_opencv_features(aligner, torch_mod, fx):
    from deepfactors_b200.aligners import Features, OrbDetectBatch, ReprojectionMatchBatch
    imgs = images()
    out = OrbDetectBatch(aligner, [dev(torch_mod, imgs["1047"]), dev(torch_mod, imgs["1052"])], 500, 20)
    f_dev = out.features()
    f_cv = []
    for name in ("1047", "1052"):
        kp, resp, desc = fx[f"{name}_500_20_kp"], fx[f"{name}_500_20_response"], fx[f"{name}_500_20_desc"]
        perm = device_order(kp, resp)
        f_cv.append(Features.from_host(kp[perm], desc[perm]))
    res = []
    for f in (f_dev, f_cv):
        items = [dict(query=f[0], train=f[1], cam=FIXTURE_CAM, seed=3), dict(query=f[1], train=f[0], cam=FIXTURE_CAM,
                                                                            seed=4)]
        m, c, r = ReprojectionMatchBatch(aligner, items)
        res.append((m.cpu().numpy(), c.cpu().numpy(), r.cpu().numpy()))
    assert res[0][1].min() > 0
    for a, b in zip(*res):
        assert np.array_equal(a, b)


def test_orb_detector_facade():
    """df::OrbDetector against the C call it wraps (tests/cpp/orb_test)"""
    exe = os.path.join(HERE, "cpp", "orb_test")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0 and "orb_test OK" in r.stdout
