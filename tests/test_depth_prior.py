"""CPU tests of the depth-prior host side: the numpy mirror of dfk_window_add_depth_priors (WindowBlocks.add_depth_priors),
depth_prior_rows, SfmWindowProblem's argument checks for depth priors and the target pyramid sizes."""
import numpy as np
import pytest

from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import DepthPrior, SfmWindowProblem, depth_prior_rows, depth_prior_sizes


def _records(rng, n, cs):
    return (rng.standard_normal((n, cs * (cs + 1) // 2 + cs + 2)) * 5).astype(np.float32)


def _dense_code(rec, cs):
    J = np.zeros((cs, cs))
    J[np.triu_indices(cs)] = rec[:cs * (cs + 1) // 2]
    return J + np.triu(J, 1).T


@pytest.mark.parametrize("cs", [8, 32])
def test_mirror_offsets_triangles_and_f(cs):
    lay = WindowBlocks(4, cs, [(0, 1), (1, 2), (2, 3)], [(0, 3)])
    rng = np.random.default_rng(cs)
    base = rng.standard_normal(lay.floats).astype(np.float32)
    recs = _records(rng, 5, cs)
    kf, sigma, lp = [3, 1, 3], [0.5, 2.0, 0.1], [0, 1, 3, 5]
    got = lay.add_depth_priors(base.copy(), kf, sigma, lp, recs)
    B = lay.B
    o_g, _, o_t = lay.offsets()
    nh = cs * (cs + 1) // 2
    touched = np.zeros(lay.floats, dtype=bool)
    for k in (1, 3):
        blk = got[k * B * B:(k + 1) * B * B].reshape(B, B)
        b0 = base[k * B * B:(k + 1) * B * B].reshape(B, B).astype(np.float64)
        add, gadd = np.zeros((cs, cs)), np.zeros(cs)
        for i, kk in enumerate(kf):
            if kk == k:
                for r in recs[lp[i]:lp[i + 1]]:
                    add += _dense_code(r.astype(np.float64), cs) / np.float64(np.float32(sigma[i])) ** 2
                    gadd -= r[nh:nh + cs].astype(np.float64) / np.float64(np.float32(sigma[i])) ** 2
        assert np.array_equal(blk[6:, 6:], (b0[6:, 6:] + add).astype(np.float32))  # both triangles
        assert np.array_equal(blk[:6], b0[:6].astype(np.float32)) and np.array_equal(blk[:, :6], b0[:, :6].astype(np.float32))
        g = got[o_g + k * B:o_g + (k + 1) * B]
        assert np.array_equal(g[6:], (base[o_g + k * B + 6:o_g + (k + 1) * B].astype(np.float64) + gadd).astype(np.float32))
        touched[k * B * B:(k + 1) * B * B].reshape(B, B)[6:, 6:] = True
        touched[o_g + k * B + 6:o_g + (k + 1) * B] = True
    f = np.float64(base[o_t])
    for i in range(3):
        for r in recs[lp[i]:lp[i + 1]]:
            f = f + np.float64(r[nh + cs]) / np.float64(np.float32(sigma[i])) ** 2
    assert got[o_t] == np.float32(f)
    touched[o_t] = True
    assert np.array_equal(got[~touched], base[~touched])  # inlier total, links, pose parts, other keyframes
    # no priors: untouched
    assert np.array_equal(lay.add_depth_priors(base.copy(), [], [], [0], recs[:0]), base)


def test_depth_prior_rows_are_linear_priors_at_zero_delta():
    cs, levels = 8, 3
    rng = np.random.default_rng(1)
    recs = _records(rng, 2 * levels, cs)
    rows = depth_prior_rows(recs, [0.5, 2.0], levels, cs)
    lay = WindowBlocks(1, cs, [])
    for i, sg in enumerate([0.5, 2.0]):
        # the prior row, taken at delta 0, adds what add_depth_priors adds
        buf = lay.add_depth_priors(np.zeros(lay.floats, np.float32), [0], [sg], [0, levels],
                                   recs[i * levels:(i + 1) * levels])
        B = lay.B
        G, g, f0 = rows[i][:B * B].reshape(B, B), rows[i][B * B:B * B + B], rows[i][-1]
        assert np.array_equal(G.astype(np.float32), buf[:B * B].reshape(B, B))
        assert np.array_equal(g.astype(np.float32), buf[B * B:B * B + B])
        assert np.float32(f0) == buf[lay.offsets()[2]]
        assert not G[:6].any() and not G[:, :6].any() and not g[:6].any()


def test_target_pyramid_sizes():
    assert depth_prior_sizes(640, 480, 4) == [(640, 480), (320, 240), (160, 120), (80, 60)]
    assert depth_prior_sizes(81, 61, 3) == [(81, 61), (40, 30), (20, 15)]
    assert depth_prior_sizes(5, 3, 1) == [(5, 3)]


class _T:
    """a stand-in for a device tensor: the checks read shapes only"""

    def __init__(self, h, w):
        self.shape = (h, w)


def _kf(sizes):
    return [dict(prx_orig=_T(h, w)) for w, h in sizes]


@pytest.mark.parametrize("dp,match", [
    (DepthPrior(2, [_T(48, 64), _T(24, 32)], 1.0), "outside the window"),
    (DepthPrior(-1, [_T(48, 64), _T(24, 32)], 1.0), "outside the window"),
    (DepthPrior(0, [_T(48, 64), _T(24, 32)], 0.0), "sigma"),
    (DepthPrior(0, [_T(48, 64), _T(24, 32)], -1.0), "sigma"),
    (DepthPrior(0, [_T(48, 64), _T(24, 32)], float("inf")), "sigma"),
    (DepthPrior(1, [_T(48, 64)], 1.0), "target levels"),
    (DepthPrior(1, [_T(48, 64), _T(24, 30)], 1.0), "level 1 target"),
])
def test_window_problem_rejects_bad_depth_priors(dp, match):
    kf = [_kf([(64, 48), (32, 24)]), _kf([(64, 48), (32, 24)])]
    with pytest.raises(ValueError, match=match):
        SfmWindowProblem(None, [None, None], kf, [(0, 1)], depth_priors=[dp])
