"""Writes tests/golden/orb_pyramid_features.npz: cv2.ORB keypoints, angles, Harris responses, descriptors and octaves
with several pyramid levels -- the expected output of dfk_orb_detect_pyramid_batch and of the CPU oracle
(orb_oracle.detect_pyramid).

    python tests/golden/make_orb_pyramid_fixture.py [out.npz]

Needs OpenCV (cv2) on the host; the tests only read the .npz.

The images are those of tests/orb_images.py.  Each is run through cv2.ORB_create(nfeatures, scale_factor, nlevels,
fastThreshold=t).detectAndCompute for each entry of CONFIGS.  Keys per run {name}_{nfeatures}_{scale}_{nlevels}_{t}
(scale with '.' written 'p'): _count (cv2's number of keypoints), _octaves [nlevels] int32 (its count per octave) and
_digest (orb_images.digest of keypoints, angles, responses and descriptors in the pyramid detector's order: octaves
ascending, each in the one-level order).  The runs of FULL_RUNS are also stored in that order: _kp [N, 2] float32
(pt), _angle [N] float32, _response [N] float32, _desc [N, 32] uint8, _octave [N] int32."""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from orb_images import device_order, digest, images  # noqa: E402  (tests/orb_images.py)

CONFIGS = [(500, 1.2, 8, 20), (1000, 1.2, 8, 20), (500, 1.5, 4, 20), (2000, 1.2, 3, 10)]
FULL_RUNS = [("1047_640", (500, 1.2, 8, 20)), ("dots", (500, 1.2, 8, 20)), ("1052_256", (500, 1.5, 4, 20)),
             ("1047_640", (2000, 1.2, 3, 10))]


def key(name, cfg):
    nf, s, nl, t = cfg
    return f"{name}_{nf}_{str(s).replace('.', 'p')}_{nl}_{t}"


def pyramid_order(kp, response, octave) -> np.ndarray:
    octave = np.asarray(octave)
    return np.concatenate([np.nonzero(octave == k)[0][device_order(kp[octave == k], response[octave == k])]
                           for k in range(int(octave.max()) + 1)] if len(octave) else [np.zeros(0, np.int64)])


def run(img, cfg):
    """cv2's output in the pyramid detector's order: kp, angle, response, desc, octave"""
    nf, s, nl, t = cfg
    kps, desc = cv2.ORB_create(nf, s, nl, fastThreshold=t).detectAndCompute(img, None)
    kp = np.array([k.pt for k in kps], np.float32).reshape(-1, 2)
    angle = np.array([k.angle for k in kps], np.float32)
    resp = np.array([k.response for k in kps], np.float32)
    octave = np.array([k.octave for k in kps], np.int32)
    desc = np.zeros((0, 32), np.uint8) if desc is None else np.ascontiguousarray(desc, np.uint8)
    p = pyramid_order(kp, resp, octave)
    return kp[p], angle[p], resp[p], desc[p], octave[p]


def main(out):
    res = {"cv2_version": np.array(cv2.__version__), "configs": np.array(CONFIGS, np.float64)}
    for name, img in images().items():
        for cfg in CONFIGS:
            kp, angle, resp, desc, octave = run(img, cfg)
            k = key(name, cfg)
            res[f"{k}_count"] = np.array(len(kp), np.int32)
            res[f"{k}_octaves"] = np.bincount(octave, minlength=cfg[2]).astype(np.int32)
            res[f"{k}_digest"] = np.array(digest(kp, angle, resp, desc, order=False))
            if (name, cfg) in FULL_RUNS:
                res[f"{k}_kp"], res[f"{k}_angle"], res[f"{k}_response"] = kp, angle, resp
                res[f"{k}_desc"], res[f"{k}_octave"] = desc, octave
    np.savez_compressed(out, **res)
    print(out, {k: v.shape for k, v in res.items() if k.endswith("_kp")})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "orb_pyramid_features.npz"))
