"""The keyframe meshes' CPU oracle (mesh_oracle, the model of dfk_keyframe_mesh_batch) against an independent
transliteration of the reference's geometry shader, OpenCV's uint16 conversion and the PLY writer:

- the oracle's vertex set, triangles, positions and normals are bit for bit those of a numpy transliteration of
  gui/shaders/drawkf.geom, written here, whose quads emit their triangle strips exactly as lines 152-183 do, the strips
  then cut into triangles; at sizes 1 x 1 to 256 x 192, with planted depths at 0.5 and 10 and one ulp either side,
  NaN and +-inf, log-stdevs at the noise threshold and next to it, zero validity, crops 0, 1, 4, 20 and larger than
  the image, slant thresholds 0, 0.3 and 1, and noisy pixels drawn and not;
- the uint16 depth is cv2's convertTo(CV_16UC1, 5000) on every value of tests/golden/keyframe_mesh_u16.npz;
- write_ply round-trips through a small PLY reader, concatenating items with index offsets, and refuses an item that
  overflowed its capacities."""
import os

import numpy as np
import pytest

from mesh_oracle import mesh_oracle as mo

# degenerate quads (a corner at depth 0 or NaN) give NaN normals, as the shader's do
pytestmark = pytest.mark.filterwarnings("ignore:invalid value encountered")

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32


# ------------------------------------------------------------------------------------------- drawkf.geom in numpy
def _normalize(v):
    x, y, z = v
    n = np.sqrt(f32(f32(x * x) + f32(y * y)) + f32(z * z))
    return (f32(x / n), f32(y / n), f32(z / n))


def _cross(a, b):
    return (f32(f32(a[1] * b[2]) - f32(a[2] * b[1])), f32(f32(a[2] * b[0]) - f32(a[0] * b[2])),
            f32(f32(a[0] * b[1]) - f32(a[1] * b[0])))


def _sub(a, b):
    return tuple(f32(p - q) for p, q in zip(a, b))


def _dot(a, b):
    return f32(f32(f32(a[0] * b[0]) + f32(a[1] * b[1])) + f32(a[2] * b[2]))


def _triangle_normal(a, b, c):  # :29-34
    return _normalize(_cross(_sub(c, a), _sub(b, a)))


def _lift(px, py, depth, cam):  # :36-46
    fx, fy, u0, v0 = cam
    return (f32(f32(f32(f32(px) - u0) / fx) * depth), f32(f32(f32(f32(py) - v0) / fy) * depth), f32(depth))


class Shader:
    """drawkf.geom for one keyframe.  Deviations, as dfk_keyframe_mesh_batch documents them: the noise test is
    (double)log-stdev > log(stdev_thresh / sqrt 2) (GLSL's exp is not exact), and a NaN depth is invalid."""

    def __init__(self, dpt, std, vld, color, cam, stdev_thresh, slt_thresh, crop, draw_noisy):
        self.d, self.s, self.v, self.c = dpt, std, vld, color
        self.H, self.W = dpt.shape
        self.cam = tuple(f32(x) for x in cam)
        self.tau = mo.tau(stdev_thresh)
        self.slt, self.crop, self.noisy_on = f32(slt_thresh), int(crop), bool(draw_noisy)

    def fetch_pixel(self, x, y):  # :80-89 with validate_pixel :57-78
        inside = 0 <= x < self.W and 0 <= y < self.H
        depth = self.d[y, x] if inside else f32(0)  # texelFetch outside the texture: 0 (invalid by the border rule)
        valid = (self.v[y, x] > 0) if (inside and self.v is not None) else inside
        color = tuple(int(k) for k in self.c[y, x]) if (inside and self.c is not None) else (0, 0, 0)
        if depth < 0.5 or depth > 10:
            valid = False
        if np.isnan(depth):  # deviation: a NaN depth is invalid
            valid = False
        if inside and self.s is not None and float(self.s[y, x]) > self.tau:
            if self.noisy_on:
                color = (255, 0, 0)
            else:
                valid = False
        border = 4
        if x < border or x > self.W - border or y < border or y > self.H - border:
            valid = False
        return dict(pos=(x, y), depth=depth, valid=valid, color=color)

    def normals(self, x, y):
        """n1, n2 of the quad at (x, y) (:113-120)"""
        tr, tl = self.fetch_pixel(x, y), self.fetch_pixel(x - 1, y)
        br, bl = self.fetch_pixel(x, y + 1), self.fetch_pixel(x - 1, y + 1)
        p = [_lift(q["pos"][0], q["pos"][1], q["depth"], self.cam) for q in (tr, tl, br, bl)]
        return _triangle_normal(p[0], p[1], p[2]), _triangle_normal(p[1], p[3], p[2])

    def main(self, x, y):
        """the strip of the quad at (x, y): a list of (pixel, colour) in emission order"""
        W, H, crop = self.W, self.H, self.crop
        if x < crop or x > W - crop or y < crop or y > H - crop:
            return []
        tr, tl = self.fetch_pixel(x, y), self.fetch_pixel(x - 1, y)
        br, bl = self.fetch_pixel(x, y + 1), self.fetch_pixel(x - 1, y + 1)
        n1, n2 = self.normals(x, y)
        fx, fy, u0, v0 = self.cam
        ray = _normalize((f32(f32(f32(x) - u0) / fx), f32(f32(f32(y) - v0) / fy), f32(1)))
        if abs(_dot(n1, ray)) < self.slt:
            return []
        if abs(_dot(n2, ray)) < self.slt:
            return []
        strip = []
        emit = lambda q: strip.append((q["pos"], q["color"]))
        if tr["valid"]:
            emit(tr)
        if not tl["valid"] or not br["valid"]:
            return strip
        emit(tl)
        emit(br)
        if bl["valid"]:
            emit(bl)
        return strip


def _strip_triangles(strip, has_tr):
    """GL_TRIANGLE_STRIP: triangle k is (v_k, v_k+1, v_k+2), the first two swapped for odd k.  The library winds T2 as
    T1 also when tr is missing (its documented deviation): the strip (tl, br, bl) becomes (br, tl, bl)."""
    out = []
    for k in range(len(strip) - 2):
        a, b, c = strip[k], strip[k + 1], strip[k + 2]
        out.append((b, a, c) if k % 2 else (a, b, c))
    if not has_tr and out:
        out = [(out[0][1], out[0][0], out[0][2])]
    return out


def _quat_rotate(q, v):
    """Eigen's q * v for q = (x, y, z, w): v + 2 w (q x v) + 2 q x (q x v), in its _transformVector order"""
    qv = (f32(q[0]), f32(q[1]), f32(q[2]))
    uv = _cross(qv, v)
    uv = tuple(f32(u + u) for u in uv)
    c = _cross(qv, uv)
    return tuple(f32(f32(v[k] + f32(f32(q[3]) * uv[k])) + c[k]) for k in range(3))


def shader_mesh(dpt, cam, pose, std, vld, color, stdev_thresh, slt_thresh, crop, draw_noisy):
    sh = Shader(dpt, std, vld, color, cam, stdev_thresh, slt_thresh, crop, draw_noisy)
    H, W = dpt.shape
    tris = []
    for y in range(H):  # gl_PrimitiveIDIn = y W + x
        for x in range(W):
            strip = sh.main(x, y)
            has_tr = bool(strip) and strip[0][0] == (x, y)
            tris += [tuple(q[0] for q in t) for t in _strip_triangles(strip, has_tr)]
    verts = sorted({p for t in tris for p in t}, key=lambda p: (p[1], p[0]))
    index = {p: i for i, p in enumerate(verts)}
    pos, nrm, col = [], [], []
    for (x, y) in verts:
        q = sh.fetch_pixel(x, y)
        pc = _lift(x, y, q["depth"], sh.cam)
        pw = _quat_rotate(pose[:4], pc)
        pos.append([f32(pw[k] + f32(pose[4 + k])) for k in range(3)])
        n1, n2 = sh.normals(x, y)
        n = tuple(f32(f32(n1[k] + n2[k]) * f32(0.5)) for k in range(3))
        nrm.append(_quat_rotate(pose[:4], n))
        col.append(q["color"])
    return dict(pixels=np.array([y * W + x for x, y in verts], np.int32).reshape(-1),
                triangles=np.array([[index[p] for p in t] for t in tris], np.int32).reshape(-1, 3),
                positions=np.array(pos, np.float32).reshape(-1, 3), normals=np.array(nrm, np.float32).reshape(-1, 3),
                colors=np.array(col, np.uint8).reshape(-1, 3))


def same_bits(a, b) -> bool:
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and bool(np.all((np.isnan(a) & np.isnan(b)) | (a.view(np.uint32) == b.view(np.uint32))))


def _keyframe(rng, w, h):
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    d = (1.5 + 0.6 * np.sin(xs / 3.0) * np.cos(ys / 4.0) + rng.normal(0, 0.02, (h, w))).astype(np.float32)
    tau = f32(mo.tau(4.2))
    s = rng.normal(float(tau), 0.4, (h, w)).astype(np.float32)
    v = rng.uniform(-0.1, 1.0, (h, w)).astype(np.float32)
    if w * h >= 30:
        k = rng.choice(w * h, size=30, replace=False)
        planted = [0.5, 10.0, np.nextafter(f32(0.5), f32(0)), np.nextafter(f32(0.5), f32(1)),
                   np.nextafter(f32(10), f32(0)), np.nextafter(f32(10), f32(11)), np.nan, np.inf, -np.inf, 0.0]
        d.flat[k[:10]] = np.array(planted, np.float32)
        s.flat[k[10:16]] = np.array([tau, np.nextafter(tau, f32(0)), np.nextafter(tau, f32(9)), np.nan, -np.inf, tau],
                                    np.float32)
        v.flat[k[16:20]] = np.array([0.0, -0.0, np.nan, 0.0], np.float32)
    c = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return d, s, v, c


CASES = [(1, 1, dict()), (8, 8, dict(crop_pix=0)), (9, 9, dict(crop_pix=1, slt_thresh=0.3)),
         (37, 5, dict(crop_pix=0)), (37, 5, dict(crop_pix=1, draw_noisy_pixels=True)),
         (48, 40, dict(crop_pix=4, draw_noisy_pixels=True)), (48, 40, dict(crop_pix=4, slt_thresh=1.0)),
         (48, 40, dict(crop_pix=4, slt_thresh=0.3)), (48, 40, dict(crop_pix=20)), (48, 40, dict(crop_pix=60)),
         (48, 40, dict(crop_pix=1, stdev_thresh=0.0)), (48, 40, dict(crop_pix=0, stdev_thresh=-2.0, draw_noisy_pixels=True)),
         (256, 192, dict()), (256, 192, dict(crop_pix=4, slt_thresh=0.3, draw_noisy_pixels=True))]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("views", ["all", "none"])
def test_oracle_is_the_shader(case, views):
    w, h, kw = CASES[case]
    if views == "none" and w * h > 10000:
        pytest.skip("one run of the largest size is enough")
    rng = np.random.default_rng(case)
    d, s, v, c = _keyframe(rng, w, h)
    if views == "none":
        s = v = c = None
    cam = (0.9 * w + 0.5, 0.85 * h + 0.5, w / 2 - 0.3, h / 2 + 0.2)
    q = rng.normal(0, 1, 4)
    pose = np.concatenate([q / np.linalg.norm(q), rng.normal(0, 1, 3)]).astype(np.float32)
    prm = dict(stdev_thresh=4.2, slt_thresh=0.0, crop_pix=20, draw_noisy_pixels=False)
    prm.update(kw)
    o = mo.mesh(d, cam, pose, std=s, vld=v, color=c, **prm)
    r = shader_mesh(d, cam, pose, s, v, c, prm["stdev_thresh"], prm["slt_thresh"], prm["crop_pix"],
                    prm["draw_noisy_pixels"])
    print(f"{w} x {h} {kw} {views}: {len(o.pixels)} vertices, {len(o.triangles)} triangles")
    assert np.array_equal(o.pixels, r["pixels"])
    assert np.array_equal(o.triangles, r["triangles"])
    assert same_bits(o.positions, r["positions"])
    assert same_bits(o.normals, r["normals"])
    if c is not None:
        assert np.array_equal(o.colors, r["colors"])
    if (w, h) == (256, 192) and not kw:
        assert len(o.triangles) > 1000


def test_u16_is_cv2_convert_to():
    z = np.load(os.path.join(HERE, "golden", "keyframe_mesh_u16.npz"))
    vals = z["values"]
    assert np.array_equal(mo.depth_u16(vals), z["u16_row"])
    assert np.array_equal(mo.depth_u16(vals), z["u16_scalar"])
    # +-inf scale to the same +-inf as +-FLT_MAX, whose conversion the fixture holds
    fmax = np.finfo(np.float32).max
    for inf, big in ((np.inf, fmax), (-np.inf, -fmax)):
        k = int(np.nonzero(vals == np.float32(big))[0][0])
        assert mo.depth_u16(np.float32([inf]))[0] == z["u16_row"][k] == 0


def _read_ply(path):
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").split("\n")
    assert head[0] == "ply" and head[1] == "format binary_little_endian 1.0"
    elements, cur = [], None
    for line in head[2:]:
        t = line.split()
        if t and t[0] == "element":
            cur = [t[1], int(t[2]), []]
            elements.append(cur)
        elif t and t[0] == "property":
            cur[2].append(t[1:])
    types = {"float": "<f4", "uchar": "u1", "int": "<i4"}
    out, off = {}, end
    for name, count, props in elements:
        if props[0][0] == "list":
            assert props[0][1:3] == ["uchar", "int"]
            rows = []
            for _ in range(count):
                k = data[off]
                rows.append(np.frombuffer(data, "<i4", k, off + 1))
                off += 1 + 4 * k
            out[name] = np.array(rows, np.int32).reshape(-1, 3)
        else:
            dt = np.dtype([(p[1], types[p[0]]) for p in props])
            out[name] = np.frombuffer(data, dt, count, off)
            off += dt.itemsize * count
    assert off == len(data)
    return out


def test_write_ply_round_trip(tmp_path):
    torch = pytest.importorskip("torch")
    from deepfactors_b200.aligners import KeyframeMeshes, write_ply
    rng = np.random.default_rng(3)
    meshes = []
    for w, h in ((48, 40), (37, 30)):
        d, s, v, c = _keyframe(rng, w, h)
        meshes.append(mo.mesh(d, (40, 40, w / 2, h / 2), [0, 0, 0, 1, 0.5, 0, 1], std=s, vld=v, color=c, crop_pix=4))
    caps_v = [len(meshes[0].positions) + 5, len(meshes[1].positions)]
    caps_t = [len(meshes[0].triangles), len(meshes[1].triangles) + 2]
    vo, to = np.array([0, caps_v[0], sum(caps_v)]), np.array([0, caps_t[0], sum(caps_t)])
    pos, nrm = np.zeros((vo[-1], 3), np.float32), np.zeros((vo[-1], 3), np.float32)
    col, pix = np.zeros((vo[-1], 3), np.uint8), np.zeros(vo[-1], np.int32)
    tri = np.zeros((to[-1], 3), np.int32)
    for i, m in enumerate(meshes):
        nv, nt = len(m.positions), len(m.triangles)
        pos[vo[i]:vo[i] + nv], nrm[vo[i]:vo[i] + nv], col[vo[i]:vo[i] + nv] = m.positions, m.normals, m.colors
        pix[vo[i]:vo[i] + nv], tri[to[i]:to[i] + nt] = m.pixels, m.triangles
    counts = np.array([[len(m.positions), len(m.triangles)] for m in meshes], np.int32)
    T = torch.from_numpy
    batch = KeyframeMeshes(T(pos), T(nrm), T(col), T(pix), T(tri), T(counts), vo, to, [None, None])
    path = str(tmp_path / "map.ply")
    write_ply(path, batch)
    got = _read_ply(path)
    v, f = got["vertex"], got["face"]
    assert list(v.dtype.names) == ["x", "y", "z", "nx", "ny", "nz", "red", "green", "blue"]
    allp = np.concatenate([m.positions for m in meshes])
    assert same_bits(np.stack([v["x"], v["y"], v["z"]], 1), allp)
    assert same_bits(np.stack([v["nx"], v["ny"], v["nz"]], 1), np.concatenate([m.normals for m in meshes]))
    assert np.array_equal(np.stack([v["red"], v["green"], v["blue"]], 1), np.concatenate([m.colors for m in meshes]))
    n0 = len(meshes[0].positions)
    assert np.array_equal(f, np.concatenate([meshes[0].triangles, meshes[1].triangles + n0]))
    # one item alone, then the other first
    write_ply(path, batch, items=[1, 0])
    f = _read_ply(path)["face"]
    assert np.array_equal(f, np.concatenate([meshes[1].triangles, meshes[0].triangles + len(meshes[1].positions)]))
    # an item past its capacity is refused
    batch.counts[1, 1] = caps_t[1] + 1
    with pytest.raises(RuntimeError, match="item 1"):
        write_ply(path, batch)
    write_ply(path, batch, items=[0])
    assert len(_read_ply(path)["vertex"]) == n0
