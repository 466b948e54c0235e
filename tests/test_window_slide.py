"""Sliding the keyframe window, host side: the buffer layout with keyframe priors (WindowBlocks.kf_priors, pack +
add_keyframe_priors + to_dense against a dense fp64 build), the Schur identity behind marginalising a keyframe (the slid
window with the keyframe's prior solves to the kept part of the full window's solution), chaining (two keyframes one
after the other equal both at once), and the renumbering of slide_factors.  The fp64 references here (dense_system,
local_system, schur_row) are the ones the GPU tests (test_gpu_window_slide.py) use."""
import numpy as np
import pytest

from deepfactors_b200.factors import WindowBlocks, is_unscaled
from deepfactors_b200.window_opt import (GeometricLink, KeyframePrior, MarginalPrior, ReprojectionLink, TrackedFrame,
                                         damped_solve, drop_keyframe, slide_factors)
from test_gpu_window_frames import random_geo
from test_window_frames import random_records


# ------------------------------------------------------------------------------------------------ fp64 references
def dense_system(K, cs, pairs, item_pair, JtJ, Jtr, res, inl, sizes, geo_pairs=(), geo=None, frame_priors=(),
                 kf_priors=(), w=0.0, codes=None, only=None):
    """(H, g, f) in fp64 of a window of K keyframes (no tracked frames) from unpacked records, geometric records
    geo = (JtJ, Jtr, res), frame priors [(k, row, delta)], keyframe priors [(keyframes, row, delta)] and the zero-code
    prior w on every keyframe.  only = m: just the factors that touch keyframe m (and the code prior on m)."""
    B = 6 + cs
    n = K * B
    H, g, f = np.zeros((n, n)), np.zeros(n), 0.0
    touches = lambda *ks: only is None or only in ks
    for i, p in enumerate(item_pair):
        k0, k1 = pairs[p]
        if not touches(k0, k1):
            continue
        cols = np.r_[k0 * B:k0 * B + 6, k1 * B:k1 * B + 6, k0 * B + 6:(k0 + 1) * B]
        np.add.at(H, np.ix_(cols, cols), np.asarray(JtJ[i], np.float64))
        np.add.at(g, cols, -np.asarray(Jtr[i], np.float64))
        if is_unscaled(sizes[i]):
            f += float(res[i])
        elif inl[i] > 0:
            f += float(res[i]) / float(inl[i]) * sizes[i][0] * sizes[i][1]
    for l, (k0, k1) in enumerate(geo_pairs):
        if not touches(k0, k1):
            continue
        cols = np.r_[k0 * B:k0 * B + 6, k1 * B:k1 * B + 6, k0 * B + 6:(k0 + 1) * B, k1 * B + 6:(k1 + 1) * B]
        H[np.ix_(cols, cols)] += np.asarray(geo[0][l], np.float64)
        g[cols] -= np.asarray(geo[1][l], np.float64)
        f += float(geo[2][l])
    for k, row, d in frame_priors:
        if not touches(k):
            continue
        G, gp, f0 = row[:B * B].reshape(B, B), row[B * B:B * B + B], row[-1]
        H[k * B:(k + 1) * B, k * B:(k + 1) * B] += G
        g[k * B:(k + 1) * B] += gp - G @ d
        f += f0 - 2 * gp @ d + d @ G @ d
    for kfs, row, d in kf_priors:
        if not touches(*kfs):
            continue
        nB = len(kfs) * B
        G, gp, f0 = row[:nB * nB].reshape(nB, nB), row[nB * nB:nB * nB + nB], row[-1]
        idx = np.concatenate([np.arange(k * B, (k + 1) * B) for k in kfs])
        H[np.ix_(idx, idx)] += G
        g[idx] += gp - G @ d
        f += f0 - 2 * gp @ d + d @ G @ d
    if w > 0:
        for k in range(K):
            if only is None or k == only:
                H[k * B + 6:(k + 1) * B, k * B + 6:(k + 1) * B] += w * np.eye(cs)
                g[k * B + 6:(k + 1) * B] -= w * codes[k]
                f += w * codes[k] @ codes[k]
    return H, g, f


def blanket(K, m, pairs, geo_pairs=(), kf_priors=()):
    nb = {a for p in pairs for a in p if p[1] < K and m in p} | {a for p in geo_pairs for a in p if m in p}
    for kfs in kf_priors:
        if m in kfs:
            nb |= set(kfs)
    return sorted(nb - {m})


def local_system(K, cs, m, nb, **kw):
    """(H, g, f) of the factors touching m over [m | nb] (dense_system(..., only=m) restricted)"""
    B = 6 + cs
    H, g, f = dense_system(K, cs, only=m, **kw)
    idx = np.concatenate([np.arange(k * B, (k + 1) * B) for k in [m] + list(nb)])
    return H[np.ix_(idx, idx)], g[idx], f


def schur_row(H, g, f, B):
    """[G | g | f0] of the Schur complement of the first B variables"""
    X = np.linalg.solve(H[:B, :B], np.column_stack([H[B:, :B].T, g[:B]]))
    G = H[B:, B:] - H[B:, :B] @ X[:, :-1]
    G = 0.5 * (G + G.T)
    return np.concatenate([G.ravel(), g[B:] - H[B:, :B] @ X[:, -1], [f - g[:B] @ X[:, -1]]])


def random_kf_prior(kfs, cs, rng, scale=0.3):
    """a random positive definite keyframe prior over kfs and a small delta"""
    nB = len(kfs) * (6 + cs)
    A = rng.standard_normal((nB + 4, nB)) * scale
    return (tuple(kfs), np.concatenate([(A.T @ A).ravel(), rng.standard_normal(nB), [abs(rng.standard_normal()) + 1]]),
            rng.standard_normal(nB) * 0.01)


def scene(cs, rng, K=5):
    pairs = [(k, (k + 1) % K) for k in range(K)] + [(2, 0), (4, 2)]
    item_pair = [p for p in range(len(pairs)) for _ in range(2)]
    sizes = [(40 >> l, 30 >> l) for _ in pairs for l in range(2)]
    JtJ, Jtr, res, inl = random_records(len(item_pair), cs, rng, 0.5)
    geo_pairs = [(0, 2), (3, 1)]
    geo = random_geo(len(geo_pairs), cs, rng)
    return pairs, item_pair, sizes, (JtJ, Jtr, res, inl), geo_pairs, geo


def renumber_records(m, pairs, item_pair, sizes, rec, geo_pairs, geo):
    """the records of the factors that do not touch m, their pairs / links renumbered as slide_factors does"""
    keep_p = [p for p, (a, b) in enumerate(pairs) if m not in (a, b)]
    items = [i for i, p in enumerate(item_pair) if p in keep_p]
    pairs2, _, _, _, _ = slide_factors(m, pairs)
    assert pairs2 == [(a - (a > m), b - (b > m)) for a, b in (pairs[p] for p in keep_p)]
    keep_l = [l for l, p in enumerate(geo_pairs) if m not in p]
    geo2 = [(a - (a > m), b - (b > m)) for a, b in (geo_pairs[l] for l in keep_l)]
    return (pairs2, [keep_p.index(item_pair[i]) for i in items], [sizes[i] for i in items],
            tuple(np.asarray(x)[items] for x in rec), geo2, tuple(np.asarray(x)[keep_l] for x in geo))


def kept_index(K, B, removed):
    return np.concatenate([np.arange(k * B, (k + 1) * B) for k in range(K) if k not in removed])


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("cs", [8, 32])
def test_layout_with_keyframe_priors_matches_a_dense_build(cs):
    rng = np.random.default_rng(cs + 1)
    K, B = 5, 6 + cs
    pairs, item_pair, sizes, rec, geo_pairs, geo = scene(cs, rng, K)
    kp = [random_kf_prior((0, 2, 3), cs, rng), random_kf_prior((1, 2), cs, rng), random_kf_prior((2, 3, 4), cs, rng)]
    plain = WindowBlocks(K, cs, pairs, geo_pairs)
    wb = WindowBlocks(K, cs, pairs, geo_pairs, kf_priors=[p[0] for p in kp])
    assert wb.prior_blocks == [(0, 2), (0, 3), (1, 2), (2, 3), (2, 4), (3, 4)]
    assert wb.prior_offset == plain.floats and wb.floats == plain.floats + 6 * B * B
    assert wb.offsets() == plain.offsets() and wb.frame_offset == plain.frame_offset
    buf = wb.pack(item_pair, *rec, sizes, geo=geo)
    assert np.all(buf[wb.prior_offset:] == 0)
    wb.add_keyframe_priors(buf, [p[1] for p in kp], [p[2] for p in kp])
    H, g, f, _ = wb.to_dense(buf)
    Hr, gr, fr = dense_system(K, cs, pairs, item_pair, *rec, sizes, geo_pairs, geo, kf_priors=kp)
    assert np.abs(H - Hr).max() <= 1e-5 * np.abs(Hr).max()
    assert np.abs(g - gr).max() <= 1e-5 * np.abs(gr).max()
    assert f == pytest.approx(fr, rel=1e-5)
    assert np.array_equal(H, H.T)
    # without keyframe priors nothing moves
    empty = WindowBlocks(K, cs, pairs, geo_pairs, kf_priors=())
    assert empty.floats == plain.floats and empty.prior_blocks == [] and empty.prior_offset == plain.floats
    assert np.array_equal(empty.pack(item_pair, *rec, sizes, geo=geo), plain.pack(item_pair, *rec, sizes, geo=geo))


@pytest.mark.parametrize("cs", [8, 32])
def test_without_keyframe_priors_pack_is_the_previous_builds(cs):
    from deepfactors_b200.factors import unpack_geometric_records, unpack_records
    from test_window_frames import load_parent_fixture
    fx = load_parent_fixture(cs)
    H, g, r_, n_ = unpack_records(fx["records"], cs)
    gH, gg, gres, _ = unpack_geometric_records(fx["geo_records"], cs)
    lay = WindowBlocks(fx["K"], cs, fx["pairs"], fx["geo_pairs"], num_frames=0, kf_priors=())
    assert lay.floats == fx["pack"].size
    assert np.array_equal(lay.pack(fx["item_pair"], H, g, r_, n_, fx["sizes"], geo=(gH, gg, gres)), fx["pack"])


def slide(K, cs, m, state, w, codes):
    """marginalise keyframe m of state = (pairs, item_pair, sizes, rec, geo_pairs, geo, kf_priors) in fp64 and return
    the next window's state and codes"""
    pairs, item_pair, sizes, rec, geo_pairs, geo, kp = state
    B = 6 + cs
    nb = blanket(K, m, pairs, geo_pairs, [p[0] for p in kp])
    Hl, gl, fl = local_system(K, cs, m, nb, pairs=pairs, item_pair=item_pair, JtJ=rec[0], Jtr=rec[1], res=rec[2],
                              inl=rec[3], sizes=sizes, geo_pairs=geo_pairs, geo=geo, kf_priors=kp, w=w, codes=codes)
    row = schur_row(Hl, gl, fl, B)
    prior = KeyframePrior(tuple(nb), np.zeros((len(nb), 7)), np.zeros((len(nb), cs)), row)
    old = [KeyframePrior(k, np.zeros((len(k), 7)), np.zeros((len(k), cs)), r) for k, r, _ in kp]
    _, _, _, _, priors2 = slide_factors(m, pairs, priors=old, prior=prior)
    deltas = {id(pr): d for pr, (_, _, d) in zip(old, kp)}
    kp2 = []
    for pr, src in zip(priors2, [p for p in old if m not in p.keyframes] + [prior]):
        kp2.append((pr.keyframes, pr.row, deltas.get(id(src), np.zeros(len(pr.keyframes) * B))))
    pairs2, ip2, sizes2, rec2, geo_pairs2, geo2 = renumber_records(m, pairs, item_pair, sizes, rec, geo_pairs, geo)
    return (pairs2, ip2, sizes2, rec2, geo_pairs2, geo2, kp2), np.delete(codes, m, axis=0)


def solve_state(K, cs, state, w, codes, fixed):
    pairs, item_pair, sizes, rec, geo_pairs, geo, kp = state
    H, g, _ = dense_system(K, cs, pairs, item_pair, *rec, sizes, geo_pairs, geo, kf_priors=kp, w=w, codes=codes)
    return damped_solve(H, g, 0.0, fixed), H, g


@pytest.mark.parametrize("cs", [8, 16])
@pytest.mark.parametrize("m", [0, 2, 4])
def test_schur_identity_of_a_marginalised_keyframe(cs, m):
    """marginalising keyframe m, then solving the slid window at lambda = 0, gives the kept part of the full window's
    solution; the gauge is the first kept keyframe's pose (after dropping keyframe 0, the new first pose)"""
    rng = np.random.default_rng(10 * cs + m)
    K, B, w = 5, 6 + cs, 1e-2
    pairs, item_pair, sizes, rec, geo_pairs, geo = scene(cs, rng, K)
    kp = [random_kf_prior((1, 2, 3), cs, rng)]
    codes = rng.standard_normal((K, cs)) * 0.3
    state = (pairs, item_pair, sizes, rec, geo_pairs, geo, kp)
    g0 = 0 if m != 0 else 1  # the gauge keyframe, kept
    dx, _, _ = solve_state(K, cs, state, w, codes, range(g0 * B, g0 * B + 6))
    state2, codes2 = slide(K, cs, m, state, w, codes)
    g2 = g0 - (g0 > m)
    dx2, _, _ = solve_state(K - 1, cs, state2, w, codes2, range(g2 * B, g2 * B + 6))
    want = dx[kept_index(K, B, [m])]
    assert np.abs(dx2 - want).max() <= 1e-12 * np.abs(want).max()


def test_chained_marginalisation_equals_eliminating_both_at_once():
    """m1 = 2, then m2 = 3 (old numbering; in m1's prior): the window left has the normal equations of the full window
    with both keyframes eliminated at once, and the same solution"""
    cs, K = 8, 6
    B = 6 + cs
    rng = np.random.default_rng(77)
    pairs = [(k, (k + 1) % K) for k in range(K)] + [(2, 4), (5, 3)]
    item_pair = list(range(len(pairs)))
    sizes = [(40, 30)] * len(pairs)
    rec = random_records(len(pairs), cs, rng, 0.5)
    geo_pairs = [(0, 3), (2, 5)]
    geo = random_geo(len(geo_pairs), cs, rng)
    kp = [random_kf_prior((1, 2, 4), cs, rng)]
    codes = np.zeros((K, cs))
    state = (pairs, item_pair, sizes, rec, geo_pairs, geo, kp)
    dx, H, g = solve_state(K, cs, state, 0.0, codes, range(6))
    state2, codes2 = slide(K, cs, 2, state, 0.0, codes)
    assert 2 in state2[6][-1][0]  # old keyframe 3 (now 2) is in keyframe 2's prior
    state3, codes3 = slide(K - 1, cs, 2, state2, 0.0, codes2)
    # both at once, on the full normal equations
    e = np.r_[2 * B:4 * B]
    k = kept_index(K, B, [2, 3])
    X = np.linalg.solve(H[np.ix_(e, e)], np.column_stack([H[np.ix_(e, k)], g[e]]))
    S = H[np.ix_(k, k)] - H[np.ix_(k, e)] @ X[:, :-1]
    s = g[k] - H[np.ix_(k, e)] @ X[:, -1]
    dx3, H3, g3 = solve_state(K - 2, cs, state3, 0.0, codes3, range(6))
    assert np.abs(H3 - S).max() <= 1e-12 * np.abs(S).max()
    assert np.abs(g3 - s).max() <= 1e-12 * np.abs(s).max()
    # damped_solve's 1e-12 max|d| diagonal term differs between the two systems; the conditioning amplifies it
    assert np.abs(dx3 - dx[k]).max() <= 1e-10 * np.abs(dx[k]).max()


def test_slide_factors_renumbers_every_factor_kind():
    K, m = 6, 2
    pairs = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5), (5, 0), (3, 1)]
    pts = np.zeros((4, 2), np.int32)
    links = [ReprojectionLink(2, 4, pts, pts, 1.0, 1.0), ReprojectionLink(5, 3, pts, pts, 1.0, 1.0)]
    geometric = [GeometricLink(0, 2, pts, 0.1), GeometricLink(4, 1, pts, 0.1)]
    frames = [TrackedFrame(0, []), TrackedFrame(3, []), TrackedFrame(5, [])]
    z = lambda n: np.zeros((n, 7))
    priors = [MarginalPrior(2, z(1)[0], np.zeros(8), np.ones(3)), MarginalPrior(4, z(1)[0], np.zeros(8), np.ones(3)),
              KeyframePrior((1, 2, 3), z(3), np.zeros((3, 8)), np.ones(3)),
              KeyframePrior((3, 5), z(2), np.zeros((2, 8)), 2 * np.ones(3))]
    prior = KeyframePrior((1, 3, 4), z(3), np.zeros((3, 8)), 3 * np.ones(3))
    p2, l2, g2, f2, pr2 = slide_factors(m, pairs, links, geometric, frames, priors, prior)
    assert p2 == [(0, 1), (2, 3), (3, 4), (4, 0), (2, 1)]
    assert [(ln.k0, ln.k1) for ln in l2] == [(4, 2)]
    assert [(gl.k0, gl.k1) for gl in g2] == [(3, 1)]
    assert [fr.k for fr in f2] == [0, 2, 4]
    assert isinstance(pr2[0], MarginalPrior) and pr2[0].k == 3
    assert [pr.keyframes for pr in pr2[1:]] == [(2, 4), (1, 2, 3)]
    assert np.array_equal(pr2[2].row, prior.row)
    # the inputs are left alone
    assert priors[3].keyframes == (3, 5) and links[1].k0 == 5 and frames[1].k == 3
    with pytest.raises(ValueError, match="tracked frames"):
        slide_factors(3, pairs, links, geometric, frames, priors, None)
    with pytest.raises(ValueError):
        slide_factors(m, pairs, prior=KeyframePrior((1, 2), z(2), np.zeros((2, 8)), np.ones(3)))
    poses, codes = np.arange(K * 7).reshape(K, 7), np.arange(K * 8).reshape(K, 8)
    p, c = drop_keyframe(poses, codes, m)
    assert np.array_equal(p, poses[[0, 1, 3, 4, 5]]) and np.array_equal(c, codes[[0, 1, 3, 4, 5]])
