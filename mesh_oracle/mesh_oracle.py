"""ctypes front-end of the keyframe meshes' oracle (mesh_oracle/libdfk_mesh_oracle.so).

TEST INFRASTRUCTURE ONLY: tests/ and tools/bench_secondary.py use it as the checker of dfk_keyframe_mesh_batch.  Images
are numpy arrays [H, W] (float32) or [H, W, 3] (uint8); a camera is (fx, fy, u0, v0) in fp32; a pose is pose_wk, 7
floats (quaternion x, y, z, w, translation).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libdfk_mesh_oracle.so")
_CSRC = os.path.join(_HERE, "..", "deepfactors_b200", "csrc")


def build(force: bool = False) -> str:
    """Compile the oracle with the committed Makefile (gcc, -O2 -ffp-contract=off)."""
    srcs = [os.path.join(_HERE, f) for f in ("dfk_mesh_oracle.c", "Makefile")] + \
        [os.path.join(_CSRC, "dfk_mesh_model.h")]
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
        L.dfkm_tau.argtypes = [C.c_float]
        L.dfkm_tau.restype = C.c_double
        L.dfkm_depth_u16.argtypes = [_P, C.c_longlong, _P]
        L.dfkm_mesh.argtypes = [C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, C.c_float, C.c_float, C.c_int, C.c_int,
                                C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P]
        L.dfkm_mesh.restype = C.c_int
        _lib = L
    return _lib


def tau(stdev_thresh: float) -> float:
    """log(stdev_thresh / sqrt 2) in fp64 (-inf for stdev_thresh <= 0): the noise test is (double)s > tau"""
    return float(lib().dfkm_tau(float(stdev_thresh)))


def depth_u16(d) -> np.ndarray:
    """convertTo(CV_16UC1, 5000) of a float32 array, elementwise"""
    a = np.ascontiguousarray(d, np.float32)
    out = np.zeros(a.shape, np.uint16)
    lib().dfkm_depth_u16(a.ctypes.data, a.size, out.ctypes.data)
    return out


@dataclass
class Mesh:
    positions: np.ndarray   # float32 [V, 3]
    normals: np.ndarray     # float32 [V, 3]
    colors: np.ndarray      # uint8 [V, 3] (zeros without a colour image)
    pixels: np.ndarray      # int32 [V]
    triangles: np.ndarray   # int32 [T, 3]
    depth_u16: np.ndarray   # uint16 [H, W]


def _opt(a, dtype):
    return None if a is None else np.ascontiguousarray(a, dtype)


def mesh(dpt, cam, pose, std=None, vld=None, color=None, stdev_thresh: float = 4.2, slt_thresh: float = 0.0,
         crop_pix: int = 20, draw_noisy_pixels: bool = False) -> Mesh:
    """dfk_keyframe_mesh_batch of one keyframe from its depth (float32 [H, W])"""
    d = np.ascontiguousarray(dpt, np.float32)
    H, W = d.shape
    s, v, c = _opt(std, np.float32), _opt(vld, np.float32), _opt(color, np.uint8)
    for a in (s, v):
        assert a is None or a.shape == (H, W)
    assert c is None or c.shape == (H, W, 3)
    cm = np.ascontiguousarray(np.asarray([cam.fx, cam.fy, cam.u0, cam.v0] if hasattr(cam, "fx") else cam,
                                         np.float32)[:4])
    ps = np.ascontiguousarray(pose, np.float32)
    assert ps.shape == (7,)
    vcap, tcap = W * H, 2 * W * H
    pos = np.zeros((vcap, 3), np.float32)
    nrm = np.zeros((vcap, 3), np.float32)
    col = np.zeros((vcap, 3), np.uint8)
    pix = np.zeros(vcap, np.int32)
    tri = np.zeros((tcap, 3), np.int32)
    u16 = np.zeros((H, W), np.uint16)
    counts = np.zeros(2, np.int32)
    ptr = lambda a: None if a is None else a.ctypes.data
    if not lib().dfkm_mesh(W, H, d.ctypes.data, ptr(s), ptr(v), ptr(c), cm.ctypes.data, ps.ctypes.data,
                           float(stdev_thresh), float(slt_thresh), int(crop_pix), int(bool(draw_noisy_pixels)), vcap,
                           tcap, pos.ctypes.data, nrm.ctypes.data, col.ctypes.data if c is not None else None,
                           pix.ctypes.data, tri.ctypes.data, u16.ctypes.data, counts.ctypes.data):
        raise MemoryError("mesh oracle: out of memory")
    nv, nt = int(counts[0]), int(counts[1])
    return Mesh(pos[:nv], nrm[:nv], col[:nv], pix[:nv], tri[:nt], u16)
