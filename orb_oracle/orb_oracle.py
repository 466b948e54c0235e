"""ctypes front-end of the ORB detector's oracle (orb_oracle/libdfk_orb_oracle.so).

TEST INFRASTRUCTURE ONLY: tests/ and tools/bench_secondary.py use it as the checker of dfk_orb_detect_batch and
dfk_orb_detect_pyramid_batch.  Images are
uint8 [H, W]; the outputs are keypoints float32 [N, 2], angles float32 [N], responses float32 [N] and descriptors uint8
[N, 32], in the detector's order (response descending, then y, then x).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfk_orb_oracle.so")
_CSRC = os.path.join(_HERE, "..", "deepfactors_b200", "csrc")


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc, -O2 -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in ("dfk_orb_oracle.c", "Makefile")] + \
        [os.path.join(_CSRC, f) for f in ("dfk_orb_model.h", "dfk_orb_pattern.h", "dfk_orb_pyramid_model.h")]
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(_LIB_PATH) for f in srcs):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


_lib = None
_I = C.POINTER(C.c_int32)


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.dfko_pattern.argtypes = [_I]
        L.dfko_fast_scores.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, _I]
        L.dfko_harris.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.dfko_harris.restype = C.c_float
        L.dfko_angle.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
        L.dfko_angle.restype = C.c_float
        L.dfko_detect.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]
        L.dfko_detect.restype = C.c_int
        L.dfko_resize.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
        L.dfko_budgets.argtypes = [C.c_int, C.c_float, C.c_int, _I]
        L.dfko_detect_pyramid.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                          C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, _I]
        L.dfko_detect_pyramid.restype = C.c_int
        _lib = L
    return _lib


def pattern() -> np.ndarray:
    """[256, 4] int32 rows (p0.x, p0.y, p1.x, p1.y): the table the oracle and the kernels were built with"""
    out = np.zeros((256, 4), np.int32)
    lib().dfko_pattern(out.ctypes.data_as(_I))
    return out


def fast_scores(img, threshold: int = 20) -> np.ndarray:
    """[H, W] int32: the FAST-9 score of every corner before suppression, -1 elsewhere"""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    out = np.zeros((h, w), np.int32)
    lib().dfko_fast_scores(img.ctypes.data, w, h, w, int(threshold), out.ctypes.data_as(_I))
    return out


@dataclass
class OrbResult:
    count: int                 # the true count; the arrays hold min(count, capacity) rows
    keypoints: np.ndarray
    angles: np.ndarray
    responses: np.ndarray
    descriptors: np.ndarray


def detect(img, nfeatures: int = 500, fast_threshold: int = 20, capacity: int | None = None) -> OrbResult:
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = int(capacity if capacity is not None else 4 * nfeatures + max(w * h // 4, 1))
    kp = np.zeros((cap, 2), np.float32)
    ang = np.zeros(cap, np.float32)
    resp = np.zeros(cap, np.float32)
    desc = np.zeros((cap, 32), np.uint8)
    n = lib().dfko_detect(img.ctypes.data, w, h, w, int(nfeatures), int(fast_threshold), cap, kp.ctypes.data,
                          ang.ctypes.data, resp.ctypes.data, desc.ctypes.data)
    if n < 0:
        raise MemoryError("orb oracle: out of memory")
    m = min(n, cap)
    return OrbResult(n, kp[:m], ang[:m], resp[:m], desc[:m])


def resize(img, w: int, h: int) -> np.ndarray:
    """uint8 [h, w]: img resized as cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR_EXACT)"""
    img = np.ascontiguousarray(img, np.uint8)
    out = np.zeros((h, w), np.uint8)
    lib().dfko_resize(img.ctypes.data, img.shape[1], img.shape[0], img.shape[1], out.ctypes.data, int(w), int(h))
    return out


def budgets(nfeatures: int, scale_factor: float, nlevels: int) -> np.ndarray:
    """int32 [nlevels]: cv::ORB's feature budget of each level"""
    out = np.zeros(nlevels, np.int32)
    lib().dfko_budgets(int(nfeatures), float(scale_factor), int(nlevels), out.ctypes.data_as(_I))
    return out


@dataclass
class OrbPyramidResult(OrbResult):
    octaves: np.ndarray = None       # int32 [rows]: the level of each row
    level_counts: np.ndarray = None  # int32 [nlevels]: each level's true count (they sum to count)


def detect_pyramid(img, nfeatures: int = 500, scale_factor: float = 1.2, nlevels: int = 8, fast_threshold: int = 20,
                   capacity: int | None = None) -> OrbPyramidResult:
    """cv2.ORB_create(nfeatures, scale_factor, nlevels, fastThreshold=fast_threshold) in the pyramid detector's order:
    levels ascending, each in the one-level order"""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape
    cap = int(capacity if capacity is not None else 4 * nfeatures + max(w * h // 4, 1))
    kp = np.zeros((cap, 2), np.float32)
    ang = np.zeros(cap, np.float32)
    resp = np.zeros(cap, np.float32)
    desc = np.zeros((cap, 32), np.uint8)
    octv = np.zeros(cap, np.int32)
    lc = np.zeros(nlevels, np.int32)
    n = lib().dfko_detect_pyramid(img.ctypes.data, w, h, w, int(nfeatures), float(scale_factor), int(nlevels),
                                  int(fast_threshold), cap, kp.ctypes.data, ang.ctypes.data, resp.ctypes.data,
                                  desc.ctypes.data, octv.ctypes.data, lc.ctypes.data_as(_I))
    if n < 0:
        raise MemoryError("orb oracle: out of memory")
    m = min(n, cap)
    return OrbPyramidResult(n, kp[:m], ang[:m], resp[:m], desc[:m], octv[:m], lc)
