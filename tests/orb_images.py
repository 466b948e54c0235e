"""The images of the ORB fixture (tests/golden/orb_features.npz), rebuilt from testimg.npz in integer arithmetic so that
the fixture need not store them, and the digest that pins a detector's output to cv2's.

  images()        name -> uint8 [H, W]: gray_1047 / gray_1052 (320 x 240), their 640 x 480 and 256 x 192 resizes
                  (resize(): bilinear with 1/1024 fixed-point weights, exact on every machine), a 3 x 3 dot grid with
                  small noise and a grid of single-pixel dots without noise (many equal FAST scores and responses)
  device_order()  the detector's order of a result: response descending, then y, then x
  digest()        SHA-256 of a result in that order: keypoints, angles, responses (float32 bits), descriptors
"""
from __future__ import annotations

import hashlib
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = [(500, 20), (200, 20), (2000, 10)]


def resize(img: np.ndarray, w: int, h: int) -> np.ndarray:
    """bilinear resize with pixel centres aligned (x_src = (x + 0.5) W / w - 0.5, clamped), weights in 1/1024, rounded
    half up: integer arithmetic only"""
    H, W = img.shape

    def taps(n_out, n_in):
        # source coordinate in 1/1024 units: ((2 x + 1) n_in - n_out) / (2 n_out) * 1024, clamped to [0, n_in - 1]
        s = ((2 * np.arange(n_out, dtype=np.int64) + 1) * n_in - n_out) * 1024 // (2 * n_out)
        s = np.clip(s, 0, (n_in - 1) * 1024)
        i0 = s // 1024
        f = s - i0 * 1024
        return i0, np.minimum(i0 + 1, n_in - 1), f

    x0, x1, fx = taps(w, W)
    y0, y1, fy = taps(h, H)
    a = img.astype(np.int64)
    rows = a[:, x0] * (1024 - fx) + a[:, x1] * fx                    # [H, w], 1/1024
    out = rows[y0, :] * (1024 - fy)[:, None] + rows[y1, :] * fy[:, None]  # [h, w], 1/2^20
    return ((out + (1 << 19)) >> 20).astype(np.uint8)


def _hash(a: np.ndarray) -> np.ndarray:
    """a deterministic integer hash (no random-number generator whose stream could change between numpy versions)"""
    x = (a.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    x ^= x >> np.uint64(29)
    x = (x * np.uint64(0xBF58476D1CE4E5B9)) & np.uint64(0xFFFFFFFFFFFFFFFF)
    return x ^ (x >> np.uint64(32))


def dots(size: int, noise: int, h: int = 240, w: int = 320) -> np.ndarray:
    """size x size squares of four brightness levels on a 9-pixel grid, on a dark background, plus noise in
    [-noise, noise]"""
    y, x = np.mgrid[0:h, 0:w]
    cell = (y // 9) * 64 + (x // 9)
    level = np.array([120, 160, 200, 240])[(_hash(cell + 7) % np.uint64(4)).astype(np.int64)]
    img = np.where(((x % 9) < size) & ((y % 9) < size), level, 40)
    if noise:
        img = img + (_hash(y * w + x + 100003) % np.uint64(2 * noise + 1)).astype(np.int64) - noise
    return np.clip(img, 0, 255).astype(np.uint8)


def images() -> dict:
    z = np.load(os.path.join(HERE, "golden", "testimg.npz"))
    out = {}
    for k in ("1047", "1052"):
        g = z[f"gray_{k}"]
        out[k] = g
        out[f"{k}_640"] = resize(g, 640, 480)
        out[f"{k}_256"] = resize(g, 256, 192)
    out["dots"] = dots(3, 2)
    out["dots_clean"] = dots(1, 0)
    return out


def device_order(kp, response) -> np.ndarray:
    kp = np.asarray(kp, np.float32).reshape(-1, 2)
    return np.lexsort((kp[:, 0], kp[:, 1], -np.asarray(response, np.float64)))


def digest(kp, angle, response, desc, order: bool = True) -> str:
    """SHA-256 of (keypoints, angles, responses, descriptors); order=True first puts the rows in the device order"""
    kp = np.ascontiguousarray(np.asarray(kp, np.float32).reshape(-1, 2))
    angle = np.ascontiguousarray(angle, np.float32).ravel()
    response = np.ascontiguousarray(response, np.float32).ravel()
    desc = np.ascontiguousarray(np.asarray(desc, np.uint8).reshape(-1, 32))
    if order:
        p = device_order(kp, response)
        kp, angle, response, desc = kp[p], angle[p], response[p], desc[p]
    h = hashlib.sha256()
    for a in (kp, angle, response, desc):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()
