"""Writes tests/golden/preprocess_frames.npz: OpenCV's PreprocessImage outputs for dfk_preprocess_batch's tests.

    python tests/golden/make_preprocess_fixture.py /path/to/DeepFactors/data/testimg

The two colour test images of the reference (data/testimg/1047.jpg, 1052.jpg, decoded by cv2.imread as 320 x 240 x 3
uint8) are stored as data.  For every config below and both images (and, for config a640, their 640 x 480 2x pixel
repeat, rebuilt by the tests and not stored) the fixture holds the SHA-256 of cv2's
    colour  cv2.remap(frame, *cv2.initUndistortRectifyMap(K_in, None, None, K_out, size, CV_32FC1), INTER_LINEAR)
    gray    cv2.cvtColor(colour, COLOR_RGB2GRAY)
    float   gray.convertTo(CV_32FC1, 1 / 255.0) (cv2.normalize with NORM_INF and alpha 1 runs exactly that convertTo
            when the image's largest value is 255; a 255 row is appended and cropped)
as the reference's PreprocessImage (core/deepfactors.cpp:634-658) computes them, and config a / 1047 row by row.
Cameras are fp32 (fx, fy, u0, v0), K matrices their fp64 widening.
"""
from __future__ import annotations

import hashlib
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "preprocess_frames.npz")


def f32(*v):
    return np.array(v, np.float32)


def resize_viewport(cam, w0, h0, w, h):
    """PinholeCamera::ResizeViewport in fp32"""
    xr, yr = np.float32(w) / np.float32(w0), np.float32(h) / np.float32(h0)
    return f32(cam[0] * xr, cam[1] * yr, cam[2] * xr, cam[3] * yr)


def scenenet(w, h):
    """GetSceneNetCam (tests/testing_utils.h:34-40): w / 2 and h / 2 are integer divisions"""
    return f32(np.float32(w // 2) / np.float32(0.5773502691896257), np.float32(h // 2) / np.float32(0.41421356237309503),
               w // 2, h // 2)


TUM = f32(525.0, 525.0, 319.5, 239.5)  # at 640 x 480
TUM_320 = resize_viewport(TUM, 640, 480, 320, 240)
# name -> (source scale, source camera, output camera, output width, output height)
CONFIGS = {
    "a": (1, TUM_320, scenenet(256, 192), 256, 192),                  # the reference's test pair
    "a640": (2, TUM, scenenet(256, 192), 256, 192),                   # the same from a 640 x 480 frame
    "b": (1, TUM_320, TUM_320, 320, 240),                             # identity
    "c": (1, TUM_320, f32(525.0, 525.0, 331.25, 227.75), 640, 480),   # 640 x 480 output, shifted principal point
    "d": (1, TUM_320, f32(90.0, 80.0, 128.0, 96.0), 256, 192),        # zoom-out: the output runs past the source
    "e": (1, TUM_320, scenenet(257, 193), 257, 193),                  # odd sizes
    "e1": (1, TUM_320, f32(0.5, 0.5, 0.25, 0.75), 1, 1),              # a 1 x 1 output
}
IMAGES = ("1047", "1052")
ROWS = ("a", "1047")  # the run stored row by row


def K(c):
    c = np.asarray(c, np.float64)
    return np.array([[c[0], 0, c[2]], [0, c[1], c[3]], [0, 0, 1]], np.float64)


def convert_to_float(gray):
    s = np.vstack([gray, np.full((1, gray.shape[1]), 255, np.uint8)])
    return np.ascontiguousarray(cv2.normalize(s, None, alpha=1.0, beta=0.0, norm_type=cv2.NORM_INF,
                                              dtype=cv2.CV_32F)[:-1])


def cv_preprocess(frame, in_cam, out_cam, w, h):
    m1, m2 = cv2.initUndistortRectifyMap(K(in_cam), None, None, K(out_cam), (w, h), cv2.CV_32FC1)
    color = cv2.remap(frame, m1, m2, cv2.INTER_LINEAR).reshape(h, w, 3)
    gray = cv2.cvtColor(color, cv2.COLOR_RGB2GRAY).reshape(h, w)
    return color, gray, convert_to_float(gray)


def repeat2(img):
    return np.ascontiguousarray(np.repeat(np.repeat(img, 2, axis=0), 2, axis=1))


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main(testimg_dir: str) -> None:
    imgs = {k: cv2.imread(os.path.join(testimg_dir, k + ".jpg")) for k in IMAGES}
    for k, v in imgs.items():
        assert v is not None and v.shape == (240, 320, 3) and v.dtype == np.uint8, k
    out = {"image_" + k: v for k, v in imgs.items()}
    names = []
    for name, (scale, in_cam, out_cam, w, h) in CONFIGS.items():
        out[f"cfg_{name}"] = np.concatenate([[scale], in_cam, out_cam, [w, h]]).astype(np.float64)
        for k in IMAGES:
            frame = imgs[k] if scale == 1 else repeat2(imgs[k])
            color, gray, f = cv_preprocess(frame, in_cam, out_cam, w, h)
            run = f"{name}_{k}"
            names.append(run)
            out[f"sha_{run}"] = np.array([sha(color), sha(gray), sha(f)])
            if (name, k) == ROWS:
                out["rows_color"], out["rows_gray"], out["rows_float"] = color, gray, f
    out["runs"] = np.array(names)
    out["cv2_version"] = np.array(cv2.__version__)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, {len(names)} runs, cv2 {cv2.__version__})")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "data/testimg")
