"""CPU tests of sparse geometric links in the keyframe window: the WindowBlocks layout and host mirror, the all-reduce
property of the buffer, the linearisation cache's code1 rule and the link indices WindowOptimizer passes through `todo`."""
import numpy as np

from deepfactors_b200 import factors, se3
from deepfactors_b200.window_opt import LinearisationCache, LMParams, WindowOptimizer

CS = 4
B = 6 + CS


def _photometric(rng, n, cs=CS):
    npar = 12 + cs
    J = rng.standard_normal((n, 3 * npar, npar)).astype(np.float32)
    H = np.einsum("nki,nkj->nij", J, J).astype(np.float32)
    g = rng.standard_normal((n, npar)).astype(np.float32)
    res = rng.random(n).astype(np.float32) * 10
    inl = rng.integers(1, 500, n)
    return H, g, res, inl


def _geo(rng, L, cs=CS):
    ng = 12 + 2 * cs
    J = rng.standard_normal((L, 2 * ng, ng)).astype(np.float32)
    H = np.einsum("nki,nkj->nij", J, J).astype(np.float32)
    return H, rng.standard_normal((L, ng)).astype(np.float32), rng.random(L).astype(np.float32) * 3


PAIRS = [(0, 1), (1, 0), (1, 2)]
LINKS = [(0, 2), (2, 0), (1, 2), (2, 3), (3, 1)]
ITEM_PAIR = [0, 0, 1, 1, 2]
SIZES = [(64, 48), (32, 24), (64, 48), (32, 24), (0, 0)]


def test_no_links_is_todays_layout_bitwise():
    rng = np.random.default_rng(1)
    H, g, res, inl = _photometric(rng, len(ITEM_PAIR))
    a = factors.WindowBlocks(4, CS, PAIRS)
    b = factors.WindowBlocks(4, CS, PAIRS, ())
    assert a.floats == b.floats == 4 * (B * B + B) + 3 * 6 * B + 2
    assert a.offsets() == b.offsets() and len(b.offsets()) == 3
    assert b.geometric_offset == b.floats
    assert np.array_equal(a.pack(ITEM_PAIR, H, g, res, inl, SIZES), b.pack(ITEM_PAIR, H, g, res, inl, SIZES, geo=None))


def _dense_scatter(H, g, res, inl, gH, gg, gres):
    Hd, gd, f = factors.assemble_window(factors.WindowLayout(4, CS), [PAIRS[p] for p in ITEM_PAIR], H, g, res, inl, SIZES)
    i0, i1 = np.r_[0:6, 12:12 + CS], np.r_[6:12, 12 + CS:12 + 2 * CS]
    for l, (k0, k1) in enumerate(LINKS):
        s0, s1 = slice(k0 * B, (k0 + 1) * B), slice(k1 * B, (k1 + 1) * B)
        G = gH[l].astype(np.float64)
        Hd[s0, s0] += G[np.ix_(i0, i0)]
        Hd[s1, s1] += G[np.ix_(i1, i1)]
        Hd[s0, s1] += G[np.ix_(i0, i1)]
        Hd[s1, s0] += G[np.ix_(i1, i0)]
        gd[s0] -= gg[l][i0]
        gd[s1] -= gg[l][i1]
        f += float(gres[l])
    return Hd, gd, f


def test_pack_and_to_dense_equal_a_dense_scatter_of_four_variable_records():
    rng = np.random.default_rng(2)
    H, g, res, inl = _photometric(rng, len(ITEM_PAIR))
    gH, gg, gres = _geo(rng, len(LINKS))
    lay = factors.WindowBlocks(4, CS, PAIRS, LINKS)
    assert lay.floats == factors.WindowBlocks(4, CS, PAIRS).floats + len(LINKS) * B * B
    buf = lay.pack(ITEM_PAIR, H, g, res, inl, SIZES, geo=(gH, gg, gres))
    assert buf.shape == (lay.floats,)
    Hd, gd, f, ninl = lay.to_dense(buf)
    Hr, gr, fr = _dense_scatter(H, g, res, inl, gH, gg, gres)
    assert np.abs(Hd - Hr).max() <= 1e-5 * np.abs(Hr).max()
    assert np.abs(gd - gr).max() <= 1e-5 * np.abs(gr).max()
    assert abs(f - fr) <= 1e-5 * abs(fr)
    assert ninl == float(inl[:-1].sum())  # links and the unscaled record add no inliers
    # the link block itself: rows k0's [pose0 | code0], columns k1's [pose1 | code1]
    l = 3
    blk = buf[lay.geometric_offset + l * B * B:lay.geometric_offset + (l + 1) * B * B].reshape(B, B)
    i0, i1 = np.r_[0:6, 12:12 + CS], np.r_[6:12, 12 + CS:12 + 2 * CS]
    assert np.array_equal(blk, gH[l][np.ix_(i0, i1)])
    assert np.allclose(Hd, Hd.T)


def test_two_halves_of_the_links_sum_to_the_full_pack():
    """the all-reduce property: each rank packs its share of the links (zero records for the rest) -- and, here, half
    the photometric items -- and the buffers add up to the full pack"""
    rng = np.random.default_rng(3)
    H, g, res, inl = _photometric(rng, len(ITEM_PAIR))
    gH, gg, gres = _geo(rng, len(LINKS))
    lay = factors.WindowBlocks(4, CS, PAIRS, LINKS)
    full = lay.pack(ITEM_PAIR, H, g, res, inl, SIZES, geo=(gH, gg, gres))
    mine = np.array([1, 0, 1, 0, 1], bool)
    zero = lambda a, m: np.where(m.reshape((-1,) + (1,) * (a.ndim - 1)), a, 0).astype(a.dtype)
    im = np.array([1, 1, 0, 0, 1], bool)
    inl0, inl1 = np.where(im, inl, 0), np.where(~im, inl, 0)
    a = lay.pack(ITEM_PAIR, zero(H, im), zero(g, im), zero(res, im), inl0, SIZES,
                 geo=(zero(gH, mine), zero(gg, mine), zero(gres, mine)))
    b = lay.pack(ITEM_PAIR, zero(H, ~im), zero(g, ~im), zero(res, ~im), inl1, SIZES,
                 geo=(zero(gH, ~mine), zero(gg, ~mine), zero(gres, ~mine)))
    assert np.abs((a + b) - full).max() <= 4 * np.finfo(np.float32).eps * np.abs(full).max()


def test_cache_marks_a_link_stale_when_code1_moves():
    poses = np.stack([se3.identity(np.float64)] * 3)
    codes = np.zeros((3, CS))
    c = LinearisationCache([(0, 1)], 1e-6, geometric=[(0, 2), (1, 2)])
    assert c.stale(poses, codes) == [0, 1, 2]
    c.store([0, 1, 2], poses, codes)
    assert c.stale(poses, codes) == []
    moved = codes.copy()
    moved[2, 1] += 1e-3   # code of keyframe 2: code1 of both links, of no pair
    assert c.stale(poses, moved) == [1, 2]
    moved = codes.copy()
    moved[1, 0] += 1e-3   # code0 of link 1 (1 -> 2); pair 0 (0 -> 1) does not depend on its frame's code
    assert c.stale(poses, moved) == [2]
    p = poses.copy()
    p[2, 6] += 1e-3       # pose1 of both links
    assert c.stale(p, codes) == [1, 2]
    c.invalidate()
    assert c.stale(poses, codes) == [0, 1, 2]


def test_window_optimizer_passes_link_indices_through_todo():
    rng = np.random.default_rng(4)
    pairs, links = [(0, 1), (1, 0)], [(0, 2), (2, 1)]
    lay = factors.WindowBlocks(3, CS, pairs, links)
    H, g, res, inl = _photometric(rng, 2)
    gH, gg, gres = _geo(rng, 2)
    seen = []

    def linearise(poses, codes, todo):
        seen.append(list(todo))
        buf = lay.pack([0, 1], H, g, res, inl, [(64, 48), (64, 48)], geo=(gH, gg, gres))
        return buf, None

    opt = WindowOptimizer(lay, linearise, LMParams(iterations=2))
    assert opt.cache.geometric == links
    opt.run(np.stack([se3.identity(np.float64)] * 3), np.zeros((3, CS)))
    assert seen[0] == [0, 1, 2, 3]  # pairs, then link j at len(pairs) + j
    assert all(set(t) <= {0, 1, 2, 3} for t in seen)
