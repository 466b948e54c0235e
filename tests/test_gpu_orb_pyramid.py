"""ORB features with several pyramid levels on the device (dfk_orb_detect_pyramid_batch,
aligners.OrbDetectPyramidBatch) against the CPU oracle (orb_oracle.detect_pyramid) and OpenCV
(tests/golden/orb_pyramid_features.npz), bit for bit:
- every fixture image and setting, all images of a setting in one batch: row by row against the oracle, and by
  digest against cv2 (the one run whose two descriptor bits the one-level model rounds differently is checked against
  the oracle only; tests/test_orb_pyramid.py pins those bits);
- one batch of mixed sizes, pitches and settings, with levels shrinking below 63 x 63 and an image smaller than that;
- nlevels = 1 equals dfk_orb_detect_batch;
- a count above the capacity: the true count, the first capacity rows, and features() raises;
- rejected calls write nothing;
- pyramid ORB -> BowTransformBatch against the BoW oracle on the oracle's descriptors;
- df::OrbPyramidDetector of the C++ facade (tests/cpp/orb_pyramid_test)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from orb_images import digest, dots, images
from orb_oracle import orb_oracle as oo

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = [(500, 1.2, 8, 20), (1000, 1.2, 8, 20), (500, 1.5, 4, 20), (2000, 1.2, 3, 10)]
KNOWN_BITS = {"1047_640_2000_1p2_3_10"}  # see tests/test_orb_pyramid.py


def key(name, cfg):
    nf, s, nl, t = cfg
    return f"{name}_{nf}_{str(s).replace('.', 'p')}_{nl}_{t}"


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


def dev(torch, img):
    return torch.from_numpy(np.ascontiguousarray(img, np.uint8)).cuda()


def unpack(out):
    """per image (count, keypoints, angles, responses, descriptors, octaves) of the written rows"""
    counts = out.counts.cpu().numpy()
    arrs = [x.cpu().numpy() for x in (out.keypoints, out.angles, out.responses, out.descriptors, out.octaves)]
    res = []
    for i, c in enumerate(counts):
        o, m = int(out.offsets[i]), min(int(c), int(out.capacities[i]))
        res.append((int(c),) + tuple(a[o:o + m] for a in arrs))
    return res


def detect(aligner, torch, imgs, nf=500, s=1.2, nl=8, t=20, capacity=None):
    from deepfactors_b200.aligners import OrbDetectPyramidBatch
    ims = [im if isinstance(im, torch.Tensor) else dev(torch, im) for im in imgs]
    return unpack(OrbDetectPyramidBatch(aligner, ims, nf, s, nl, t, capacity))


def oracle(img, nf, s, nl, t, capacity):
    r = oo.detect_pyramid(img, nf, s, nl, t, capacity)
    return (r.count, r.keypoints, r.angles, r.responses, r.descriptors, r.octaves)


def same(a, b):
    return a[0] == b[0] and all(np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8))
                                for x, y in zip(a[1:], b[1:]))


@pytest.mark.parametrize("cfg", CONFIGS, ids=[key("", c)[1:] for c in CONFIGS])
def test_equals_oracle_and_opencv_on_every_fixture(aligner, torch_mod, cfg):
    fx = np.load(os.path.join(HERE, "golden", "orb_pyramid_features.npz"))
    imgs = images()
    names = sorted(imgs)
    got = detect(aligner, torch_mod, [imgs[n] for n in names], *cfg, capacity=4 * cfg[0])
    for name, g in zip(names, got):
        k = key(name, cfg)
        assert same(g, oracle(imgs[name], *cfg, 4 * cfg[0])), k
        assert g[0] == int(fx[f"{k}_count"]), k
        assert np.array_equal(np.bincount(g[5], minlength=cfg[2]), fx[f"{k}_octaves"]), k
        if k not in KNOWN_BITS:
            assert digest(*g[1:5], order=False) == str(fx[f"{k}_digest"]), k


def random_image(rng, h, w):
    y, x = np.mgrid[0:h, 0:w]
    img = np.full((h, w), 80.0)
    for _ in range(h * w // 400):
        cy, cx, r, a = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(1.5, 6), rng.uniform(-70, 120)
        img += a * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2 * r * r))
    return np.clip(img + rng.normal(0, 4, (h, w)), 0, 255).astype(np.uint8)


def test_mixed_batch_equals_the_oracle(aligner, torch_mod):
    """sizes, pitches and every setting differ per image; levels fall below 63 x 63 part way; one image is below it"""
    torch = torch_mod
    rng = np.random.default_rng(21)
    sizes = [(480, 640), (240, 320), (100, 300), (50, 80), (333, 277), (192, 256), (64, 64), (700, 900)]
    nf = [500, 300, 100, 50, 1000, 7, 20, 2000]
    sf = [1.2, 1.5, 1.3, 1.2, 1.1, 2.0, 1.2, 1.25]
    nl = [8, 4, 5, 8, 16, 3, 2, 6]
    t = [20, 12, 25, 20, 5, 0, 20, 15]
    cap = [2 * x + 17 for x in nf]
    imgs = [random_image(rng, h, w) for h, w in sizes]
    tens = []
    for i, im in enumerate(imgs):
        if i % 2:  # a pitched view: a wider buffer's left columns
            big = torch.zeros((im.shape[0], im.shape[1] + 13 * i), dtype=torch.uint8, device="cuda")
            big[:, :im.shape[1]] = dev(torch, im)
            tens.append(big[:, :im.shape[1]])
        else:
            tens.append(dev(torch, im))
    got = detect(aligner, torch, tens, nf, sf, nl, t, cap)
    for i, im in enumerate(imgs):
        want = oracle(im, nf[i], sf[i], nl[i], t[i], cap[i])
        assert same(got[i], want), i
    assert got[3][0] == 0  # 50 x 80
    # each item alone gives the same rows
    for i in (0, 5):
        assert same(detect(aligner, torch, [tens[i]], nf[i], sf[i], nl[i], t[i], cap[i])[0], got[i]), i
    # and a second run
    assert all(same(a, b) for a, b in zip(detect(aligner, torch, tens, nf, sf, nl, t, cap), got))


def test_one_level_equals_the_one_level_call(aligner, torch_mod):
    from deepfactors_b200.aligners import OrbDetectBatch
    imgs = images()
    names = sorted(imgs)
    for nf, t in ((500, 20), (2000, 10)):
        ims = [dev(torch_mod, imgs[n]) for n in names]
        a = OrbDetectBatch(aligner, ims, nf, t, 4 * nf)
        b = detect(aligner, torch_mod, ims, nf, 1.2, 1, t, 4 * nf)
        ca = a.counts.cpu().numpy()
        for i, n in enumerate(names):
            o, m = int(a.offsets[i]), min(int(ca[i]), 4 * nf)
            one = (int(ca[i]),) + tuple(x[o:o + m].cpu().numpy() for x in (a.keypoints, a.angles, a.responses,
                                                                              a.descriptors))
            assert same(one, b[i][:5]) and (b[i][5] == 0).all(), n


def test_capacity_overflow(aligner, torch_mod):
    from deepfactors_b200.aligners import OrbDetectPyramidBatch
    img = dots(1, 0, 480, 640)  # level 0 keeps 721 tied keypoints
    out = OrbDetectPyramidBatch(aligner, [dev(torch_mod, img)], 500, 1.2, 8, 20, 800)
    got = unpack(out)[0]
    want = oracle(img, 500, 1.2, 8, 20, 800)
    assert want[0] == 1007 and same(got, want)
    with pytest.raises(RuntimeError, match="OrbDetectPyramidBatch: image 0 has 1007"):
        out.features()


def test_rejected_calls_write_nothing(aligner, torch_mod):
    from deepfactors_b200 import _lib
    from deepfactors_b200._lib import check, lib
    from deepfactors_b200.aligners import _orb_image
    torch = torch_mod
    hd = aligner._hd
    img = dev(torch, images()["1047"])
    rows = 4000
    outs = [torch.full((rows, 2), -7.0, device="cuda"), torch.full((rows, 32), 7, dtype=torch.uint8, device="cuda"),
            torch.full((rows,), -7.0, device="cuda"), torch.full((rows,), -7.0, device="cuda"),
            torch.full((rows,), -7, dtype=torch.int32, device="cuda"), torch.full((4,), -7, dtype=torch.int32,
                                                                                  device="cuda")]
    snap = [o.clone() for o in outs]
    good = dict(nf=500, s=1.2, nl=8, t=20, cap=1000)
    bad = [dict(s=1.0), dict(s=float("nan")), dict(s=0.5), dict(nl=0), dict(nl=17), dict(nf=0), dict(t=256),
           dict(cap=499)]
    for b in bad:
        p = {**good, **b}
        items = [(_lib.DfkOrbPyramidItem(_orb_image(img), good["nf"], good["s"], good["nl"], good["t"], good["cap"]))
                 for _ in range(3)]
        items.append(_lib.DfkOrbPyramidItem(_orb_image(img), p["nf"], p["s"], p["nl"], p["t"], p["cap"]))
        arr = (_lib.DfkOrbPyramidItem * 4)(*items)
        st = lib().dfk_orb_detect_pyramid_batch(hd.h, arr, 4, *[C.c_void_p(o.data_ptr()) for o in outs])
        assert st != 0, b
        assert "item 3" in lib().dfk_last_error(hd.h).decode(), b
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs, snap))
    # and a good call through the same buffers succeeds
    arr = (_lib.DfkOrbPyramidItem * 1)(_lib.DfkOrbPyramidItem(_orb_image(img), 500, 1.2, 8, 20, 1000))
    check(hd.h, lib().dfk_orb_detect_pyramid_batch(hd.h, arr, 1, *[C.c_void_p(o.data_ptr()) for o in outs]))


def test_pyramid_orb_feeds_bow(torch_mod):
    from bow_oracle import bow_oracle as bo
    from deepfactors_b200 import aligners as A
    z = np.load(os.path.join(HERE, "golden", "bow_orb.npz"))
    voc = dict(k=int(z["voc_k"]), L=int(z["voc_L"]), weighting=0, scoring=0, descriptor_bytes=32,
               **{k: z["voc_" + k] for k in ("node_ids", "parent_ids", "weights", "descriptors", "word_ids",
                                             "word_nodes")})
    gv, ov = A.BowVocabulary(voc), bo.Vocabulary(voc)
    imgs = [z["gray_0"], z["gray_25"], images()["1052_640"]]
    orb = A.OrbDetectPyramidBatch(gv, [dev(torch_mod, im) for im in imgs], 500, 1.2, 8)
    feats = orb.features()
    b = A.BowTransformBatch(gv, feats)
    for i, im in enumerate(imgs):
        want = oo.detect_pyramid(im, 500, 1.2, 8, 20, 1000)
        assert np.array_equal(feats[i].descriptors.cpu().numpy(), want.descriptors), i
        fw, w, v = ov.transform(want.descriptors)
        o, c = int(b.offsets[i]), int(b.counts[i].item())
        assert np.array_equal(b.feature_words[o:o + len(want.descriptors)].cpu().numpy(), fw), i
        assert np.array_equal(b.words[o:o + c].cpu().numpy(), w), i
        assert np.array_equal(b.values[o:o + c].cpu().numpy().view(np.uint64), np.asarray(v).view(np.uint64)), i


def test_facade_binary():
    exe = os.path.join(HERE, "cpp", "orb_pyramid_test")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/orb_pyramid_test not built")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "ok" in r.stdout
