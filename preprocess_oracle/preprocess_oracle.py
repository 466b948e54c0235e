"""ctypes front-end of the frame preprocessing's oracle (preprocess_oracle/libdfk_preprocess_oracle.so).

TEST INFRASTRUCTURE ONLY: tests/ and tools/bench_secondary.py use it as the checker of dfk_preprocess_batch.  Frames are
uint8 [H, W, 3]; cameras are (fx, fy, u0, v0) in fp32.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfk_preprocess_oracle.so")
_CSRC = os.path.join(_HERE, "..", "deepfactors_b200", "csrc")


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc, -O2 -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in ("dfk_preprocess_oracle.c", "Makefile")] + \
        [os.path.join(_CSRC, "dfk_preprocess_model.h")]
    if force or not os.path.exists(_LIB_PATH) or any(os.path.getmtime(f) > os.path.getmtime(_LIB_PATH) for f in srcs):
        subprocess.run(["make", "-C", _HERE, "-s"], check=True)
    return _LIB_PATH


_lib = None
_P = C.c_void_p


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB_PATH)
        L.dfkp_map.argtypes = [_P, _P, C.c_int, C.c_int, _P, _P]
        L.dfkp_inverse.argtypes = [_P, _P]
        L.dfkp_weights.argtypes = [_P]
        L.dfkp_preprocess.argtypes = [_P, C.c_size_t, C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, _P]
        L.dfkp_normalize.argtypes = [_P, C.c_int, C.c_int, C.c_int, _P]
        _lib = L
    return _lib


def _cam(cam) -> np.ndarray:
    """(fx, fy, u0, v0) as fp32; cam is a sequence or an object with those attributes"""
    if hasattr(cam, "fx"):
        cam = (cam.fx, cam.fy, cam.u0, cam.v0)
    return np.ascontiguousarray(np.asarray(cam, np.float32)[:4])


def init_map(in_cam, out_cam, w: int, h: int):
    """(map1, map2) float32 [h, w]: cv::initUndistortRectifyMap(K_in, None, None, K_out, (w, h), CV_32FC1)"""
    a, b = _cam(in_cam), _cam(out_cam)
    m1 = np.zeros((h, w), np.float32)
    m2 = np.zeros((h, w), np.float32)
    if not lib().dfkp_map(a.ctypes.data, b.ctypes.data, w, h, m1.ctypes.data, m2.ctypes.data):
        raise ValueError("singular output camera")
    return m1, m2


def inverse(out_cam) -> np.ndarray:
    """K_out^-1 [3, 3] float64, as cv::Mat::inv(DECOMP_LU)"""
    b = _cam(out_cam)
    ir = np.zeros(9, np.float64)
    if not lib().dfkp_inverse(b.ctypes.data, ir.ctypes.data):
        raise ValueError("singular output camera")
    return ir.reshape(3, 3)


def weights():
    """(table int32 [32, 32, 4] indexed [ty, tx, tap], number of entries whose sum needed the fix-up)"""
    tab = np.zeros((32, 32, 4), np.int32)
    fired = lib().dfkp_weights(tab.ctypes.data)
    return tab, int(fired)


@dataclass
class Preprocessed:
    color: np.ndarray      # uint8 [h, w, 3]
    gray: np.ndarray       # uint8 [h, w]
    level0: np.ndarray     # float32 [h, w]: f, or f' when normalised
    stats: tuple | None    # (mu, sigma) when normalised


def preprocess(frame, in_cam, out_cam, w: int, h: int, normalize: bool = False) -> Preprocessed:
    """Steps 1-7 of dfk_preprocess_batch for one frame"""
    src = np.ascontiguousarray(frame, np.uint8)
    sh, sw = src.shape[:2]
    assert src.ndim == 3 and src.shape[2] == 3
    a, b = _cam(in_cam), _cam(out_cam)
    color = np.zeros((h, w, 3), np.uint8)
    gray = np.zeros((h, w), np.uint8)
    f = np.zeros((h, w), np.float32)
    if not lib().dfkp_preprocess(src.ctypes.data, 3 * sw, sw, sh, a.ctypes.data, b.ctypes.data, w, h,
                                 color.ctypes.data, gray.ctypes.data, f.ctypes.data):
        raise ValueError("singular output camera")
    stats = None
    if normalize:
        st = np.zeros(2, np.float64)
        if not lib().dfkp_normalize(f.ctypes.data, w, h, 1, st.ctypes.data):
            raise MemoryError("preprocess oracle: out of memory")
        stats = (float(st[0]), float(st[1]))
    return Preprocessed(color, gray, f, stats)


def stats_of(f) -> tuple:
    """(mu, sigma) of a float32 [h, w] image by the fixed-order fp64 sums"""
    f = np.array(f, np.float32, order="C")
    h, w = f.shape
    st = np.zeros(2, np.float64)
    if not lib().dfkp_normalize(f.ctypes.data, w, h, 0, st.ctypes.data):
        raise MemoryError("preprocess oracle: out of memory")
    return float(st[0]), float(st[1])
