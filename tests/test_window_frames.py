"""Tracked frames in the keyframe window, host side: the buffer layout (WindowBlocks.pack / to_dense with pose-only frame
variables), se3.local, the Schur identity behind marginalisation (a frame eliminated from the window equals its linear
prior on the keyframe), and the cache / retraction / LM loop with frames on a synthetic quadratic.  The numpy helpers
here are the fp64 references the GPU tests (test_gpu_window_frames.py) use too."""
import numpy as np
import pytest

from deepfactors_b200 import se3
from deepfactors_b200.factors import WindowBlocks, is_unscaled, record_layout
from deepfactors_b200.window_opt import LMParams, LinearisationCache, WindowOptimizer, apply_update, damped_solve


# ------------------------------------------------------------------------------------------------ fp64 references
def dense_from_records(K, cs, pairs, item_pair, JtJ, Jtr, residual, inliers, sizes, F):
    """(H, g, f) of a window with F frames built straight from unpacked records in fp64: pair (k0, k1) puts
    [pose0 | code0] on k0's variables and pose1 on k1's, or on frame k1 - K's (after the keyframes')"""
    B = 6 + cs
    n = K * B + 6 * F
    H, g, f = np.zeros((n, n)), np.zeros(n), 0.0
    for i, p in enumerate(item_pair):
        k0, k1 = pairs[p]
        v1 = k1 * B if k1 < K else K * B + 6 * (k1 - K)
        cols = np.r_[k0 * B:k0 * B + 6, v1:v1 + 6, k0 * B + 6:(k0 + 1) * B]  # record order [pose0 | pose1 | code0]
        H[np.ix_(cols, cols)] += np.asarray(JtJ[i], np.float64)
        g[cols] -= np.asarray(Jtr[i], np.float64)
        if is_unscaled(sizes[i]):
            f += float(residual[i])
        elif inliers[i] > 0:
            f += float(residual[i]) / float(inliers[i]) * sizes[i][0] * sizes[i][1]
    return H, g, f


def schur_prior(cs, JtJ, Jtr, residual, inliers, sizes):
    """fp64 Schur complement of the pose1 variables of one frame pair's items: the prior row [G | g | f0]"""
    B = 6 + cs
    a = np.r_[0:6, 12:12 + cs]
    Hs = np.sum(np.asarray(JtJ, np.float64), axis=0)
    gs = -np.sum(np.asarray(Jtr, np.float64), axis=0)
    fp = sum(float(r) / float(n) * w * h for r, n, (w, h) in zip(residual, inliers, sizes) if n > 0)
    Haa, Hab, Hbb = Hs[np.ix_(a, a)], Hs[np.ix_(a, np.arange(6, 12))], Hs[6:12, 6:12]
    X = np.linalg.solve(Hbb, np.column_stack([Hab.T, gs[6:12]]))
    G = Haa - Hab @ X[:, :B]
    G = 0.5 * (G + G.T)
    return np.concatenate([G.ravel(), gs[a] - Hab @ X[:, B], [fp - gs[6:12] @ X[:, B]]])


def random_records(n, cs, rng, scale=1.0):
    """n random Gram records (JtJ, Jtr, residual, inliers) of rank 2 NP: positive definite"""
    NP = 12 + cs
    A = rng.standard_normal((n, 2 * NP, NP + 1)) * scale
    JtJ = np.einsum("nri,nrj->nij", A[..., :NP], A[..., :NP]).astype(np.float32)
    Jtr = np.einsum("nri,nr->ni", A[..., :NP], A[..., NP]).astype(np.float32)
    res = np.einsum("nr,nr->n", A[..., NP], A[..., NP]).astype(np.float32)
    return JtJ, Jtr, res, rng.integers(50, 500, n)


def frame_window(K, frames_of, levels=2):
    """pairs of a K-keyframe ring plus one pair (k, K + f) per frame; item_pair / sizes with `levels` items per pair"""
    pairs = [(k, (k + 1) % K) for k in range(K)]
    F = 0
    for k, nf in enumerate(frames_of):
        for _ in range(nf):
            pairs.append((k, K + F))
            F += 1
    item_pair = [p for p in range(len(pairs)) for _ in range(levels)]
    sizes = [(40 >> l, 30 >> l) for _ in range(len(pairs)) for l in range(levels)]
    return pairs, F, item_pair, sizes


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("cs", [8, 32])
def test_pack_and_to_dense_with_frames_match_a_dense_build(cs):
    rng = np.random.default_rng(cs)
    K = 4
    pairs, F, item_pair, sizes = frame_window(K, [2, 0, 1, 3])
    JtJ, Jtr, res, inl = random_records(len(item_pair), cs, rng)
    wb = WindowBlocks(K, cs, pairs, num_frames=F)
    B = 6 + cs
    assert wb.floats == WindowBlocks(K, cs, pairs).floats + 42 * F
    assert wb.dim == K * B + 6 * F
    buf = wb.pack(item_pair, JtJ, Jtr, res, inl, sizes)
    H, g, f, ni = wb.to_dense(buf)
    Hr, gr, fr = dense_from_records(K, cs, pairs, item_pair, JtJ, Jtr, res, inl, sizes, F)
    scale = np.abs(Hr).max()
    assert np.abs(H - Hr).max() <= 1e-5 * scale
    assert np.abs(g - gr).max() <= 1e-5 * np.abs(gr).max()
    assert f == pytest.approx(fr, rel=1e-5) and ni == float(np.sum(inl))
    assert np.array_equal(H, H.T)
    # frame blocks: exactly the pose1 x pose1 sums of the frame pair's items (float32, item order)
    o = wb.frame_offset
    Df = buf[o:o + 36 * F].reshape(F, 6, 6)
    for f_ in range(F):
        p = pairs.index(next(pp for pp in pairs if pp[1] == K + f_))
        acc = np.zeros((6, 6), np.float32)
        for i in [i for i, q in enumerate(item_pair) if q == p]:
            acc += JtJ[i][6:12, 6:12]
        assert np.array_equal(Df[f_], acc)
    # torch mirror of to_dense
    import torch
    Ht, gt, _, _ = wb.to_dense(torch.from_numpy(buf))
    assert np.array_equal(Ht.numpy(), H) and np.array_equal(gt.numpy(), g)


def load_parent_fixture(cs):
    """inputs and buffers of windows without frames made by the build before tracked frames (make_window_f0_fixture.py)"""
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "window_without_frames.npz"))
    get = lambda k: z[f"c{cs}_{k}"]
    return dict(K=int(get("K")), pairs=[tuple(map(int, p)) for p in get("pairs")], item_pair=list(get("item_pair")),
                sizes=[tuple(map(int, s)) for s in get("sizes")], records=get("records"),
                geo_pairs=[tuple(map(int, p)) for p in get("geo_pairs")], geo_records=get("geo_records"),
                pack=get("pack"), device=get("device"))


@pytest.mark.parametrize("cs", [8, 32])
def test_without_frames_pack_is_the_previous_builds(cs):
    """WindowBlocks.pack of a window without frames (pairs, a self pair, geometric links) is bit for bit the buffer
    the build before tracked frames packed from the same records"""
    from deepfactors_b200.factors import unpack_geometric_records, unpack_records
    fx = load_parent_fixture(cs)
    H, g, r_, n_ = unpack_records(fx["records"], cs)
    gH, gg, gres, _ = unpack_geometric_records(fx["geo_records"], cs)
    for lay in (WindowBlocks(fx["K"], cs, fx["pairs"], fx["geo_pairs"]),
                WindowBlocks(fx["K"], cs, fx["pairs"], fx["geo_pairs"], num_frames=0)):
        assert lay.floats == fx["pack"].size and lay.frame_offset == lay.floats
        buf = lay.pack(fx["item_pair"], H, g, r_, n_, fx["sizes"], geo=(gH, gg, gres))
        assert np.array_equal(buf, fx["pack"])


def test_se3_local_inverts_retract():
    rng = np.random.default_rng(3)
    for _ in range(50):
        a = se3.make_pose(rng.standard_normal(3), rng.standard_normal(3), np.float64)
        w = rng.standard_normal(3)
        w *= rng.uniform(0, 3.1) / np.linalg.norm(w)  # log is the inverse of exp inside the ball |w| < pi
        d = np.concatenate([rng.standard_normal(3), w])
        assert np.abs(se3.local(a, se3.retract(a, d)) - d).max() <= 1e-12
        assert np.abs(se3.local(a, se3.retract(a, d * 1e-9)) - d * 1e-9).max() <= 1e-15
    assert np.all(se3.local(a, a) == 0)


@pytest.mark.parametrize("cs", [8, 32])
def test_frame_elimination_equals_its_marginal_prior(cs):
    """Schur identity in fp64: a window with frame f solved (undamped, gauge fixed) gives the keyframe dx of the same
    window without f plus f's prior at delta = 0; the prior's energy f0 - 2 g^T d + d^T G d is the frame-eliminated
    quadratic model at random d."""
    rng = np.random.default_rng(10 + cs)
    K = 3
    pairs, F, item_pair, sizes = frame_window(K, [1, 1, 0])
    JtJ, Jtr, res, inl = random_records(len(item_pair), cs, rng)
    B = 6 + cs
    H, g, f = dense_from_records(K, cs, pairs, item_pair, JtJ, Jtr, res, inl, sizes, F)
    fixed = list(range(6))
    keep = np.ones(len(g), bool)
    keep[fixed] = False
    dx = np.zeros(len(g))
    dx[keep] = np.linalg.solve(H[np.ix_(keep, keep)], g[keep])
    # drop frame 0 (pair K, on the gauge keyframe 0) into a prior on keyframe 0
    fp = K
    assert pairs[fp] == (0, K)
    mine = [i for i, p in enumerate(item_pair) if p == fp]
    row = schur_prior(cs, JtJ[mine], Jtr[mine], res[mine], inl[mine], [sizes[i] for i in mine])
    G, gp, f0 = row[:B * B].reshape(B, B), row[B * B:B * B + B], row[-1]
    rest = [i for i in range(len(item_pair)) if item_pair[i] != fp]
    pairs2 = pairs[:fp] + [(k0, k1 - 1) for k0, k1 in pairs[fp + 1:]]  # frame 1 becomes frame 0
    ip2 = [p if p < fp else p - 1 for p in np.asarray(item_pair)[rest]]
    H2, g2, f2 = dense_from_records(K, cs, pairs2, ip2, JtJ[rest], Jtr[rest], res[rest], inl[rest],
                                    [sizes[i] for i in rest], F - 1)
    H2[:B, :B] += G
    g2[:B] += gp
    keep2 = np.ones(len(g2), bool)
    keep2[fixed] = False
    dx2 = np.zeros(len(g2))
    dx2[keep2] = np.linalg.solve(H2[np.ix_(keep2, keep2)], g2[keep2])
    assert np.abs(dx2[:K * B] - dx[:K * B]).max() <= 1e-9 * np.abs(dx[:K * B]).max()
    assert np.abs(dx2[K * B:] - dx[K * B + 6:]).max() <= 1e-9 * np.abs(dx).max()
    # energy model of the frame's factor alone, minimised over the frame's pose, against the prior's
    Hs = sum(np.asarray(JtJ[i], np.float64) for i in mine)
    gs = -sum(np.asarray(Jtr[i], np.float64) for i in mine)
    a = np.r_[0:6, 12:12 + cs]
    for _ in range(5):
        d = rng.standard_normal(B) * 0.1
        db = np.linalg.solve(Hs[6:12, 6:12], gs[6:12] - Hs[np.ix_(np.arange(6, 12), a)] @ d)
        full = np.zeros(12 + cs)
        full[a], full[6:12] = d, db
        e_full = (f0 + gs[6:12] @ np.linalg.solve(Hs[6:12, 6:12], gs[6:12])) - 2 * gs @ full + full @ Hs @ full
        e_prior = f0 - 2 * gp @ d + d @ G @ d
        assert e_prior == pytest.approx(e_full, rel=1e-9, abs=1e-9 * abs(f0))


def test_cache_and_retraction_with_frames():
    K, cs = 2, 3
    pairs = [(0, 1), (1, 0), (0, 2)]  # frame 0 = variable K + 0, on keyframe 0
    c = LinearisationCache(pairs, 1e-6)
    poses = np.tile(se3.identity(np.float64), (K, 1))
    fposes = np.tile(se3.identity(np.float64), (1, 1))
    codes = np.zeros((K, cs))
    assert c.stale(poses, codes, fposes) == [0, 1, 2]
    c.store([0, 1, 2], poses, codes, fposes)
    assert c.stale(poses, codes, fposes) == []
    f2 = fposes.copy(); f2[0, 4] += 1e-3                   # the frame moved: only its pair
    assert c.stale(poses, codes, f2) == [2]
    c2 = codes.copy(); c2[0, 1] = 1e-3                      # keyframe 0's code: its pair to 1 and its frame's pair
    assert c.stale(poses, c2, fposes) == [0, 2]
    c2 = codes.copy(); c2[1, 1] = 1e-3
    assert c.stale(poses, c2, fposes) == [1]
    dx = np.arange(K * (6 + cs) + 6, dtype=np.float64) * 1e-3
    p2, co2, fp2 = apply_update(poses, codes, dx, cs, fposes)
    p1, co1 = apply_update(poses, codes, dx, cs)
    assert np.array_equal(p1, p2) and np.array_equal(co1, co2)
    assert np.allclose(fp2[0], se3.retract(fposes[0], dx[K * (6 + cs):], np.float64))


def test_lm_loop_moves_frames_on_a_quadratic():
    """two keyframes, one frame on keyframe 1: energy |t1 - goal|^2 + |code1 - cgoal|^2 + |t_frame - t1 - off|^2 through
    the window layout with the frame pair's records; the frame converges, the gauge stays"""
    cs = 2
    K = 2
    pairs = [(0, 1), (1, K)]
    wb = WindowBlocks(K, cs, pairs, num_frames=1)
    goal = np.array([0.05, -0.02, 0.03])
    cgoal = np.array([0.3, -0.1])
    off = np.array([0.01, 0.02, -0.04])
    NP = 12 + cs
    calls = []

    def linearise(poses, codes, todo, frame_poses):
        calls.append(list(todo))
        J0 = np.zeros((3, NP)); J0[:, 6:9] = np.eye(3)                          # pair 0: pose1 = keyframe 1
        r0 = poses[1][4:7] - goal
        J1 = np.zeros((5, NP)); J1[0:3, 6:9] = np.eye(3); J1[0:3, 0:3] = -np.eye(3)  # pair 1: frame - keyframe 1
        J1[3:5, 12:14] = np.eye(2)                                             # and keyframe 1's code
        r1 = np.concatenate([frame_poses[0][4:7] - poses[1][4:7] - off, codes[1] - cgoal])
        JtJ = np.stack([J0.T @ J0, J1.T @ J1])
        Jtr = np.stack([J0.T @ r0, J1.T @ r1])
        return wb.pack([0, 1], JtJ, Jtr, [r0 @ r0, r1 @ r1], [1, 1], [(1, 1), (1, 1)]), None

    poses = np.tile(se3.identity(np.float64), (K, 1))
    frames = np.tile(se3.identity(np.float64), (1, 1))
    codes = np.zeros((K, cs))
    opt = WindowOptimizer(wb, linearise, LMParams(iterations=10, lambda_init=1e-6))
    p, c, tr = opt.run(poses, codes, frames)
    assert tr.energy[-1] < 1e-10 < tr.energy[0]
    assert np.allclose(p[1][4:7], goal, atol=1e-5) and np.allclose(c[1], cgoal, atol=1e-5)
    assert np.allclose(tr.frame_poses[0][4:7], goal + off, atol=1e-5)
    assert np.array_equal(p[0], poses[0])
    assert calls[0] == [0, 1]
    # without frames the loop refuses frame poses it has no variables for, and a frame window needs them
    with pytest.raises(ValueError):
        opt.run(poses, codes)
    # the dense solve of the frame window equals damped_solve of to_dense
    buf, _ = linearise(poses, codes, [0, 1], frames)
    H, g, _, _ = wb.to_dense(buf)
    assert H.shape == (K * (6 + cs) + 6,) * 2
    dx = damped_solve(H, g, 1e-3, range(6))
    assert dx.shape == (K * (6 + cs) + 6,)
