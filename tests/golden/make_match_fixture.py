"""Writes tests/golden/match_features.npz: OpenCV keypoints, binary descriptors and brute-force Hamming matches of the
two test images gray_1047 / gray_1052 of testimg.npz, the inputs and the expected output of the keypoint matching calls.

    python tests/golden/make_match_fixture.py [out.npz]

Needs OpenCV (cv2) on the host; the tests only read the .npz.  Per detector:
  orb    cv2.ORB_create(500, 1.2, 1): the rep_nfeatures / rep_scale_factor / rep_nlevels options (32-byte descriptors)
  brisk  cv2.BRISK_create(): 64-byte descriptors.  OpenCV's BRISK is not the brisk library DeepFactors links; it is test
         data with the shape of BriskDetector's descriptors.
and for both directions a -> b (1047 -> 1052, 1052 -> 1047) cv2.BFMatcher(cv2.NORM_HAMMING).match: per query the train
index and the distance.  Keys: {det}_kp_{img} [N, 2] float32, {det}_desc_{img} [N, D] uint8, {det}_match_{a}_{b}
[N_a, 2] int32 (train index, distance), and the cv2 version."""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))


def features(det, img):
    kps, desc = det.detectAndCompute(img, None)
    kp = np.array([k.pt for k in kps], np.float32).reshape(-1, 2)
    return kp, np.ascontiguousarray(desc, np.uint8)


def main(out):
    z = np.load(os.path.join(HERE, "testimg.npz"))
    imgs = {"1047": z["gray_1047"], "1052": z["gray_1052"]}
    res = {"cv2_version": np.array(cv2.__version__)}
    dets = {"orb": cv2.ORB_create(500, 1.2, 1), "brisk": cv2.BRISK_create()}
    bf = cv2.BFMatcher(cv2.NORM_HAMMING)
    for name, det in dets.items():
        f = {k: features(det, im) for k, im in imgs.items()}
        for k, (kp, desc) in f.items():
            res[f"{name}_kp_{k}"] = kp
            res[f"{name}_desc_{k}"] = desc
        for a, b in (("1047", "1052"), ("1052", "1047")):
            ms = bf.match(f[a][1], f[b][1])
            m = np.full((len(f[a][1]), 2), -1, np.int32)
            for x in ms:
                m[x.queryIdx] = (x.trainIdx, int(round(x.distance)))
            res[f"{name}_match_{a}_{b}"] = m
    np.savez_compressed(out, **res)
    print(out, {k: v.shape for k, v in res.items()})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "match_features.npz"))
