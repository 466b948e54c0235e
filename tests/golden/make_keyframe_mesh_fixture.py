"""Writes tests/golden/keyframe_mesh_u16.npz: OpenCV's uint16 depth conversion for dfk_keyframe_mesh_batch's tests.

    python tests/golden/make_keyframe_mesh_fixture.py

SaveKeyframes (core/deepfactors.cpp:560) converts a keyframe's depth with cv::Mat::convertTo(CV_16UC1, 5000).  The
Python binding has no convertTo; cv2.normalize(NORM_INF, dtype=CV_16U) runs exactly src.convertTo(dst, CV_16U,
alpha / ||src||_inf, 0).  Each run puts an anchor m = FLT_MAX first (the largest magnitude, so the norm is m) and
alpha = 5000 m, an exact fp64 product, so the scale is exactly 5000.  A NaN after the anchor does not change the norm
(std::max keeps the anchor).  An infinite value would make the norm infinite, so +-inf themselves are not converted
here; their product with 5000 is the same +-inf as +-FLT_MAX's, whose conversion is stored.

The fixture holds the values and cv2's conversion of them as one row (the vectorised path) and one value at a time
(the scalar path): halves after the scaling, negatives, NaN, +-FLT_MAX, values around 65535.5 / 5000 and around
2^31 / 5000, and random depths.
"""
from __future__ import annotations

import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "keyframe_mesh_u16.npz")
FMAX = float(np.finfo(np.float32).max)


def values() -> np.ndarray:
    f = np.float32
    v = [0.0, -0.0, 1e-30, -1e-30, 0.5, 1.0, 10.0, -1.0, -1e-4, -0.5 / 5000, np.nan, FMAX, -FMAX,
         float(np.finfo(np.float32).tiny)]
    v += [(k + 0.5) / 5000 for k in range(-4, 40)]                     # products near halves
    v += [k * 0.0001 for k in range(0, 200)]                           # products near k / 2
    for c in (65535.0, 65535.5, 65536.0, 65534.5, 2.0 ** 31, 2.0 ** 31 - 128, 2.0 ** 31 + 256, 2.0 ** 32, 1e12):
        x = f(c / 5000)
        v += [np.nextafter(x, f(-np.inf)), x, np.nextafter(x, f(np.inf))]
        v += [-np.nextafter(x, f(-np.inf)), -x]
    rng = np.random.default_rng(5000)
    v += list(rng.uniform(0.0, 15.0, 500)) + list(rng.uniform(-3e5, 5e5, 200))
    return np.array(v, np.float32)


def convert(d: np.ndarray) -> np.ndarray:
    """convertTo(CV_16UC1, 5000) of a float32 row"""
    src = np.concatenate([np.float32([FMAX]), d]).reshape(1, -1)
    out = cv2.normalize(src, None, 5000.0 * FMAX, 0.0, cv2.NORM_INF, cv2.CV_16U)
    assert out[0, 0] == 0 and out.dtype == np.uint16  # the anchor's product is beyond int32
    return out[0, 1:]


def main():
    d = values()
    row = convert(d)
    scalar = np.array([convert(d[i:i + 1])[0] for i in range(d.size)], np.uint16)
    assert row[list(d).index(np.float32(0.5))] == 2500, "the scale is not 5000"
    np.savez_compressed(OUT, values=d, u16_row=row, u16_scalar=scalar, cv2_version=np.array(cv2.__version__))
    print(f"wrote {OUT}: {d.size} values, row and scalar paths agree: {bool((row == scalar).all())}")


if __name__ == "__main__":
    main()
