"""dfk_window_solver_update / dfk_window_solver_create_from (WindowSolver.update / grown) and IncrementalOptimizer on the
device: an incremental update is bit for bit a fresh solver's first update of the same buffer, it re-factorises from
the first changed keyframe column, a grown solver takes over the unchanged prefix, and a mapping sequence driven by
IncrementalOptimizer equals one with a fresh solver every step."""
import numpy as np
import pytest

from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import IncrementalOptimizer, diag_eps_of, reusable_columns
from test_gpu_window_solve import damped_system
from test_window_frames import random_records

CODE_SIZES = [8, 32, 128]


def lastn_pairs(K, n=4):
    """every keyframe's back connections to its n predecessors, both directions (the mapper's LASTN)"""
    return [p for k in range(1, K) for m in range(max(0, k - n), k) for p in ((k, m), (m, k))]


def case(K, cs, frames_of=(), links=(), kf_priors=(), seed=0):
    pairs = lastn_pairs(K) + [(0, 0)]
    F = 0
    for k, nf in enumerate(frames_of):
        for _ in range(nf):
            pairs.append((k, K + F))
            F += 1
    layout = WindowBlocks(K, cs, pairs, list(links), F, list(kf_priors))
    rng = np.random.default_rng(seed)
    recs = random_records(len(pairs), cs, rng)
    geo = None
    if links:
        NG = 12 + 2 * cs
        G = rng.standard_normal((len(links), 2 * NG, NG + 1))
        geo = (np.einsum("nri,nrj->nij", G[..., :NG], G[..., :NG]).astype(np.float32),
               np.einsum("nri,nr->ni", G[..., :NG], G[..., NG]).astype(np.float32), np.ones(len(links), np.float32))
    buf = layout.pack(list(range(len(pairs))), *recs, [(4, 4)] * len(pairs), geo=geo)
    if kf_priors:  # small prior blocks keep the system positive definite
        o = layout.prior_offset
        buf[o:] = (rng.standard_normal(buf.size - o) * 0.05).astype(np.float32)
    return layout, buf


def window_of(al, layout):
    from deepfactors_b200.aligners import Window
    n = len(layout.pairs)
    return Window(al, layout.num_keyframes, layout.pairs, list(range(n)), [(4, 4)] * n, layout.geometric,
                  layout.num_frames, layout.kf_priors)


def touch_keyframe(layout, buf, j, rng):
    """the buffer with keyframe j's own terms changed (a unary factor on j): only column j's loaded system changes"""
    out = buf.copy()
    B = layout.B
    A = rng.standard_normal((B, B)).astype(np.float32) * 0.1
    D = out[:layout.num_keyframes * B * B].reshape(-1, B, B)
    D[j] += A @ A.T
    o_g = layout.offsets()[0]
    out[o_g + j * B:o_g + (j + 1) * B] += rng.standard_normal(B).astype(np.float32)
    return out


def fresh_update(win, fixed, buf, eps, w, codes):
    from deepfactors_b200.aligners import WindowSolver
    sol = WindowSolver(win, fixed)
    dx, j0 = sol.update(buf, eps, w, codes)
    assert j0 == 0
    return dx, sol.info.clone()


VARIANTS = {
    "plain": dict(),
    "frames": dict(frames_of=(1, 0, 2, 0, 1, 0, 0, 1)),
    "links": dict(links=((0, 3), (7, 2))),
    "priors": dict(kf_priors=((1, 2, 4),)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("cs", CODE_SIZES)
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_update_is_a_fresh_solver_bit_for_bit(cs, variant):
    import torch
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    K = 8
    layout, buf_h = case(K, cs, seed=cs, **VARIANTS[variant])
    al = SfmAligner(cs)
    win = window_of(al, layout)
    rng = np.random.default_rng(cs + 1)
    codes = rng.standard_normal((K, cs)) * 0.3
    for fixed, w in (((), 0.0), (tuple(range(6)), 1e-2)):
        eps = diag_eps_of(layout, buf_h, fixed, w)
        sol = WindowSolver(win, fixed)
        buf = torch.from_numpy(buf_h).cuda()
        dx, j0 = sol.update(buf, eps, w, codes)
        assert j0 == 0 and int(sol.info.item()) == 0
        prev = dx.clone()
        dx, j0 = sol.update(buf, eps, w, codes)  # nothing changed
        assert j0 == K and torch.equal(dx, prev) and int(sol.info.item()) == 0
        cur = buf_h
        for j in (0, K // 2, K - 1, 3):
            cur = touch_keyframe(layout, cur, j, rng)
            b = torch.from_numpy(cur).cuda()
            dx, j0 = sol.update(b, eps, w, codes)
            assert j0 == j, (j, j0)
            ref, info = fresh_update(win, fixed, b, eps, w, codes)
            assert torch.equal(dx, ref), j
            assert torch.equal(sol.info, info) and int(info.item()) == 0
        # the code prior's gradient moves with the codes: the first keyframe whose code changed
        if w > 0:
            codes = codes.copy()
            codes[5] += 0.1
            dx, j0 = sol.update(b, eps, w, codes)
            assert j0 == 5
            assert torch.equal(dx, fresh_update(win, fixed, b, eps, w, codes)[0])
        # a dfk_window_solve in between starts the next update over
        sol.solve(b, 0.0, w, codes)
        dx, j0 = sol.update(b, eps, w, codes)
        assert j0 == 0 and torch.equal(dx, fresh_update(win, fixed, b, eps, w, codes)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("cs", CODE_SIZES)
def test_update_matches_the_existing_solve_at_lambda_zero(cs):
    import torch
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    K = 8
    layout, buf_h = case(K, cs, seed=10 + cs, frames_of=(0, 1, 0, 1), links=((0, 4),))
    win = window_of(SfmAligner(cs), layout)
    codes = np.random.default_rng(3).standard_normal((K, cs)) * 0.3
    buf = torch.from_numpy(buf_h).cuda()
    for fixed, w in (((), 0.0), (tuple(range(6)), 1e-2)):
        eps = diag_eps_of(layout, buf_h, fixed, w)
        dx, j0 = WindowSolver(win, fixed).update(buf, eps, w, codes)
        ref, info = WindowSolver(win, fixed).solve(buf, 0.0, w, codes)
        assert int(info.item()) == 0
        x, r = dx.cpu().numpy(), ref.cpu().numpy()
        A, b, keep = damped_system(layout, buf_h, 0.0, fixed, w, codes)
        berr = np.abs(A @ x[keep] - b).max() / (np.abs(A).sum(1).max() * np.abs(x).max() + np.abs(b).max())
        assert berr <= 1e-12, berr
        assert np.abs(x - r).max() / np.abs(r).max() <= 1e-9


@pytest.mark.gpu
def test_update_reports_a_failed_pivot_like_the_solve():
    import torch
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    cs, K = 8, 8
    layout, good = case(K, cs, seed=4, frames_of=(0, 1, 0, 1))
    win = window_of(SfmAligner(cs), layout)
    B = layout.B
    bad = good.copy()
    bad[:K * B * B].reshape(K, B, B)[5] = -np.eye(B, dtype=np.float32) * 1e3
    sol = WindowSolver(win, range(6))
    eps = diag_eps_of(layout, good, range(6))
    sol.update(torch.from_numpy(good).cuda(), eps)
    _, finfo = fresh_update(win, range(6), torch.from_numpy(bad).cuda(), eps, 0.0, None)
    _, sinfo = sol.solve(torch.from_numpy(bad).cuda(), 0.0)
    assert int(finfo.item()) == int(sinfo.item()) == 1 + 5 * B  # keyframe 5's first pivot
    sol.update(torch.from_numpy(good).cuda(), eps)
    dx, j0 = sol.update(torch.from_numpy(bad).cuda(), eps)
    assert j0 == 5 and int(sol.info.item()) == int(finfo.item()) and torch.all(dx == 0)
    dx, j0 = sol.update(torch.from_numpy(bad).cuda(), eps)  # the kept failed column is reported again
    assert j0 == K and int(sol.info.item()) == int(finfo.item()) and torch.all(dx == 0)
    dx, j0 = sol.update(torch.from_numpy(good).cuda(), eps)  # and recovers
    assert j0 == 5 and int(sol.info.item()) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("cs", CODE_SIZES)
def test_grown_solver_reuses_the_unchanged_prefix(cs):
    import torch
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    al = SfmAligner(cs)
    K0 = 10
    rng = np.random.default_rng(20 + cs)
    old, _ = case(K0, cs)
    # one record per factor, the same for a factor in both windows: the old keyframes' terms sum alike
    grown = WindowBlocks(K0 + 1, cs, old.pairs + [p for m in range(K0 - 4, K0) for p in ((K0, m), (m, K0))])
    loop = WindowBlocks(K0 + 1, cs, grown.pairs, [(K0, 2)])
    recs = random_records(len(loop.pairs), cs, rng)
    NG = 12 + 2 * cs
    G = rng.standard_normal((1, 2 * NG, NG + 1))
    geo = (np.einsum("nri,nrj->nij", G[..., :NG], G[..., :NG]).astype(np.float32),
           np.einsum("nri,nr->ni", G[..., :NG], G[..., NG]).astype(np.float32), np.ones(1, np.float32))

    def packed(layout):
        n = len(layout.pairs)
        return layout.pack(list(range(n)), *(r[:n] for r in recs), [(4, 4)] * n,
                           geo=geo if layout.geometric else None)

    fixed = tuple(range(6))
    w_old, w_new, w_loop = window_of(al, old), window_of(al, grown), window_of(al, loop)
    sol = WindowSolver(w_old, fixed)
    eps = diag_eps_of(old, packed(old), fixed)
    sol.update(torch.from_numpy(packed(old)).cuda(), eps)
    assert reusable_columns(old, grown, fixed, fixed) == K0 - 4
    g = sol.grown(w_new, fixed)
    b = torch.from_numpy(packed(grown)).cuda()
    dx, j0 = g.update(b, eps)
    assert j0 == K0 - 4
    assert torch.equal(dx, fresh_update(w_new, fixed, b, eps, 0.0, None)[0])
    # a loop link (K - 1, 2) between keyframes the grown window already holds
    assert reusable_columns(grown, loop, fixed, fixed) == 2
    gl = g.grown(w_loop, fixed)
    b = torch.from_numpy(packed(loop)).cuda()
    dx, j0 = gl.update(b, eps)
    assert j0 == 2
    assert torch.equal(dx, fresh_update(w_loop, fixed, b, eps, 0.0, None)[0])
    # not an extension (fewer keyframes, other fixed variables among the old ones): rejected, nothing written
    smaller = window_of(al, WindowBlocks(K0 - 1, cs, lastn_pairs(K0 - 1)))
    for bad, fx in ((smaller, fixed), (w_new, ()), (w_new, tuple(range(7)))):
        with pytest.raises(_lib.DfkError):
            sol.grown(bad, fx)
    import ctypes as C
    s = C.c_void_p(12345)
    fx = np.arange(6, dtype=np.int32)
    st = _lib.lib().dfk_window_solver_create_from(al.handle, smaller.w, 6, fx.ctypes.data_as(C.POINTER(C.c_int32)),
                                                  sol.s, C.byref(s))
    assert st == _lib.DFK_ERR_INVALID_ARG and s.value == 12345
    # the old solver is left as it was: its next update of the same buffer reuses everything
    dx, j0 = sol.update(torch.from_numpy(packed(old)).cuda(), eps)
    assert j0 == K0


# ------------------------------------------------------------------------------------------- mapping sequence
VEC = [4, 5, 6, 0, 1, 2]  # a pose [q (x, y, z, w) | t]: t, then the quaternion's vector part


class ToyMap:
    """A nonlinear map on the window layout: every factor's record is a fixed Gram H and the gradient
    H (x + 0.1 sin(3 x) - t) of its keys' coordinates x (each pose's t and quaternion vector part, code0) towards a
    target t, packed with WindowBlocks.pack in factor order.  Gauss-Newton contracts towards the target, so deltas
    shrink through the relinearisation threshold.  Records are kept per factor identity, so a grown map keeps its kept
    factors'."""

    def __init__(self, cs, seed):
        self.cs, self.rng = cs, np.random.default_rng(seed)
        self.gram = {}
        self.recs = {}
        self.evaluated = []

    def factor(self, key):
        if key not in self.gram:
            NP = 12 + self.cs
            A = self.rng.standard_normal((2 * NP, NP)) * 0.5
            self.gram[key] = (A.T @ A, self.rng.standard_normal(NP) * 0.2)
        return self.gram[key]

    def linearise_fn(self, layout, keys):
        def lin(poses, codes, todo, frame_poses=None):
            K = layout.num_keyframes
            for i in todo:
                k0, k1 = layout.pairs[i]
                H, t = self.factor(keys[i])
                p1 = poses[k1] if k1 < K else frame_poses[k1 - K]
                x = np.concatenate([poses[k0][VEC], p1[VEC], codes[k0]])
                self.recs[keys[i]] = (H, H @ (x + 0.1 * np.sin(3 * x) - t))
                self.evaluated.append(keys[i])
            n = len(layout.pairs)
            JtJ = np.stack([self.recs[keys[i]][0] for i in range(n)]).astype(np.float32)
            Jtr = np.stack([self.recs[keys[i]][1] for i in range(n)]).astype(np.float32)
            buf = layout.pack(list(range(n)), JtJ, Jtr, np.ones(n, np.float32), np.full(n, 10), [(4, 4)] * n)
            import torch
            return torch.from_numpy(buf).cuda(), None
        return lin


def mapping_sequence(cs, fresh_every_step):
    """12 keyframes added one at a time with LASTN 4, a loop link (11, 2) at the end and two tracked frames, three
    updates per keyframe.  Returns every step's (estimate, delta, result)"""
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    al = SfmAligner(cs)
    toy = ToyMap(cs, 7)
    rng = np.random.default_rng(8)
    out = []
    opt = None
    for K in range(2, 13):
        pairs = lastn_pairs(K)
        keys = [("pair",) + p for p in pairs]
        frames = [k for k in (3, 6) if k < K]
        pairs += [(k, K + f) for f, k in enumerate(frames)]
        keys += [("frame", f) for f in range(len(frames))]
        if K == 12:  # the loop closure
            pairs.append((11, 2))
            keys.append(("pair", 11, 2))
        layout = WindowBlocks(K, cs, pairs, num_frames=len(frames))
        win = window_of(al, layout)
        poses = np.tile(np.array([0, 0, 0, 1.0, 0, 0, 0]), (K, 1))
        poses[:, 4:] = rng.standard_normal((K, 3)) * 0.1
        codes = rng.standard_normal((K, cs)) * 0.1
        fposes = np.tile(np.array([0, 0, 0, 1.0, 0, 0, 0]), (len(frames), 1))
        lin = toy.linearise_fn(layout, keys)
        if opt is None:
            opt = IncrementalOptimizer(layout, lin, None, poses, codes, fposes if frames else None,
                                       code_prior_weight=1e-2)
            opt.keys = keys
            opt._solver_of(win, None)
        else:
            old = {k: i for i, k in enumerate(opt.keys)}
            fmap = [f if f < len(opt.lin_frames) else None for f in range(len(frames))]
            opt.grow(layout, lin, poses, codes, fposes if frames else None, [old.get(k) for k in keys], fmap,
                     window=win)
            opt.keys = keys
        if fresh_every_step:
            def solve(buf, eps, c, win=win):
                dx, j0 = WindowSolver(win, opt.fixed).update(buf, eps, opt.code_prior_weight, c)
                return dx.cpu().numpy(), j0
            opt.solve = solve
        for _ in range(3):
            n0 = len(toy.evaluated)
            moved = opt.relinearize_keys() if (opt.update_count + 1) % opt.relinearize_skip == 0 else []
            res = opt.update()
            est = opt.estimate()
            out.append((est, opt.delta.copy(), res, list(toy.evaluated[n0:]), moved, layout, keys,
                        opt.lin_poses.copy(), opt.lin_codes.copy(), opt.lin_frames.copy(), opt.diag_eps))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [8, 32])
def test_mapping_sequence_incremental_equals_fresh(cs):
    inc = mapping_sequence(cs, False)
    ref = mapping_sequence(cs, True)
    assert len(inc) == len(ref) == 33
    reused = 0
    for step, (a, b) in enumerate(zip(inc, ref)):
        for x, y in zip(a[0], b[0]):
            assert np.array_equal(x, y), step
        assert np.array_equal(a[1], b[1]), step
        ra, rb = a[2], b[2]
        assert (ra.variables_relinearized, ra.factors_relinearised) == (rb.variables_relinearized,
                                                                         rb.factors_relinearised), step
        assert rb.first_column == 0
        reused += ra.first_column > 0
        # re-linearised factors: the new ones and those that depend on a relinearised key
        evaluated, moved, layout, keys = a[3], a[4], a[5], a[6]
        assert ra.factors_relinearised == len(evaluated)
        K = layout.num_keyframes
        prev_keys = set(inc[step - 1][6]) if step else set()
        want = set()
        for i, key in enumerate(keys):
            k0, k1 = layout.pairs[i]
            deps = {("pose", k0), ("code", k0), ("pose", k1) if k1 < K else ("frame", k1 - K)}
            if key not in prev_keys or deps & set(moved):
                want.add(key)
        assert set(evaluated) == want, step
    assert reused > 0
    print(f"C={cs}: {reused} of {len(inc)} updates reused a column prefix")


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [8, 32])
def test_mapping_sequence_against_dense_gauss_newton(cs):
    """every step's delta against damped_solve at lambda 0 of the dense system of the same buffer"""
    import torch
    captured = []
    import deepfactors_b200.window_opt as wo
    orig = wo.IncrementalOptimizer.update

    def spy(self):
        lin = self.linearise

        def keep(*args):
            buf, f = lin(*args)
            captured.append((self.layout, buf.clone(), self.lin_codes.copy()))
            return buf, f
        self.linearise = keep
        try:
            return orig(self)
        finally:
            self.linearise = lin
    wo.IncrementalOptimizer.update = spy
    try:
        seq = mapping_sequence(cs, False)
    finally:
        wo.IncrementalOptimizer.update = orig
    assert len(captured) == len(seq)
    worst = 0.0
    for (layout, buf, codes), step in zip(captured, seq):
        delta, eps = step[1], step[10]
        H, g, _, _ = layout.to_dense(buf)
        B, w = layout.B, 1e-2
        for k in range(layout.num_keyframes):
            sl = slice(k * B + 6, (k + 1) * B)
            H[sl, sl] += w * torch.eye(B - 6, dtype=H.dtype, device=H.device)
            g[sl] -= w * torch.as_tensor(codes[k], dtype=g.dtype, device=g.device)
        keep = torch.ones(H.shape[0], dtype=torch.bool, device=H.device)
        keep[:6] = False
        idx = torch.nonzero(keep).squeeze(1)
        Hk = H.index_select(0, idx).index_select(1, idx) + eps * torch.eye(len(idx), dtype=H.dtype, device=H.device)
        ref = torch.zeros_like(g)
        ref[idx] = torch.linalg.solve(Hk, g.index_select(0, idx))
        err = np.abs(delta - ref.cpu().numpy()).max()
        worst = max(worst, err)
        assert err <= 1e-6, err
    print(f"C={cs}: worst |delta - dense GN| {worst:.2e}")


def dense_mirror(cs):
    """The mapping sequence of mapping_sequence(cs) by an independent dense mirror of ISAM2's rules: theta_lin and
    delta in dicts per key (pose / code of each keyframe, pose of each frame), the full relinearisation check on the
    previous delta, every factor re-evaluated at theta_lin (ToyMap's formula), the dense system in fp64 with the code
    prior and diag_eps, numpy's solve, and theta_lin (+) delta.  Returns every step's (poses, codes, frame poses,
    relinearised keys)."""
    from deepfactors_b200 import se3
    toy = ToyMap(cs, 7)
    rng = np.random.default_rng(8)
    lin, delta, out, eps, w = {}, {}, [], None, 1e-2
    for K in range(2, 13):
        pairs = lastn_pairs(K)
        keys = [("pair",) + p for p in pairs]
        frames = [k for k in (3, 6) if k < K]
        pairs += [(k, K + f) for f, k in enumerate(frames)]
        keys += [("frame", f) for f in range(len(frames))]
        if K == 12:
            pairs.append((11, 2))
            keys.append(("pair", 11, 2))
        layout = WindowBlocks(K, cs, pairs, num_frames=len(frames))
        poses = np.tile(np.array([0, 0, 0, 1.0, 0, 0, 0]), (K, 1))
        poses[:, 4:] = rng.standard_normal((K, 3)) * 0.1
        codes = rng.standard_normal((K, cs)) * 0.1
        for k in range(K):
            lin.setdefault(("pose", k), poses[k].copy())
            lin.setdefault(("code", k), codes[k].copy())
        for f in range(len(frames)):
            lin.setdefault(("frame", f), np.array([0, 0, 0, 1.0, 0, 0, 0]))
        B = layout.B

        def sl(key):
            kind, i = key
            return slice(i * B, i * B + 6) if kind == "pose" else slice(i * B + 6, (i + 1) * B) if kind == "code" \
                else slice(K * B + 6 * i, K * B + 6 * i + 6)
        for _ in range(3):
            moved = sorted(k for k, d in delta.items() if np.abs(d).max() >= 0.05)
            for k in moved:
                lin[k] = lin[k] + delta[k] if k[0] == "code" else se3.retract(lin[k], delta[k], np.float64)
                delta[k] = np.zeros_like(delta[k])
            JtJ, Jtr = [], []
            for (k0, k1), key in zip(pairs, keys):
                H, t = toy.factor(key)
                p1 = lin[("pose", k1)] if k1 < K else lin[("frame", k1 - K)]
                x = np.concatenate([lin[("pose", k0)][VEC], p1[VEC], lin[("code", k0)]])
                JtJ.append(H)
                Jtr.append(H @ (x + 0.1 * np.sin(3 * x) - t))
            n = len(pairs)
            buf = layout.pack(list(range(n)), np.stack(JtJ).astype(np.float32), np.stack(Jtr).astype(np.float32),
                              np.ones(n, np.float32), np.full(n, 10), [(4, 4)] * n)
            Hd, g, _, _ = layout.to_dense(buf)
            for k in range(K):
                Hd[k * B + 6:(k + 1) * B, k * B + 6:(k + 1) * B] += w * np.eye(cs)
                g[k * B + 6:(k + 1) * B] -= w * lin[("code", k)]
            keep = np.ones(layout.dim, bool)
            keep[:6] = False
            if eps is None:
                eps = 1e-12 * np.abs(np.diag(Hd)[keep]).max()
            A = Hd[np.ix_(keep, keep)] + eps * np.eye(int(keep.sum()))
            dx = np.zeros(layout.dim)
            dx[keep] = np.linalg.solve(A, g[keep])
            for key in lin:
                if key[0] != "frame" or key[1] < len(frames):
                    delta[key] = dx[sl(key)].copy()
            est_p = np.stack([se3.retract(lin[("pose", k)], delta[("pose", k)], np.float64) for k in range(K)])
            est_c = np.stack([lin[("code", k)] + delta[("code", k)] for k in range(K)])
            est_f = np.stack([se3.retract(lin[("frame", f)], delta[("frame", f)], np.float64)
                              for f in range(len(frames))]) if frames else np.zeros((0, 7))
            out.append((est_p, est_c, est_f, moved))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [8, 32])
def test_mapping_sequence_against_an_independent_dense_mirror(cs):
    """IncrementalOptimizer's estimates and relinearised keys on the device against dense_mirror: the threshold, the
    theta_lin bookkeeping, the retraction and grow()'s carry of theta_lin and delta (frames included)"""
    inc = mapping_sequence(cs, False)
    ref = dense_mirror(cs)
    assert len(inc) == len(ref)
    worst = 0.0
    relinearised = 0
    for step, (a, (p, c, f, moved)) in enumerate(zip(inc, ref)):
        ep, ec, ef = a[0]
        assert sorted(a[4]) == moved, step
        relinearised += len(moved)
        err = max(np.abs(ep - p).max(), np.abs(ec - c).max(), np.abs(ef - f).max(initial=0.0))
        worst = max(worst, err)
        assert err <= 1e-6, (step, err)
    assert relinearised > 0
    print(f"C={cs}: worst |estimate - dense mirror| {worst:.2e}, {relinearised} keys relinearised")


# ------------------------------------------------------------------------------------------ growing a real problem
def _grown_scene(torch, cs):
    """the synthetic window of test_gpu_window_lm (three keyframes, photometric pairs, a reprojection link (0, 2), a
    geometric link (0, 2), a tracked frame on keyframe 1), and the same window grown by keyframe 3 with pairs (3, 2) /
    (2, 3), a reprojection link (2, 0), a geometric link (1, 2) and a tracked frame on keyframe 3.  Returns (old, new,
    a third copy of new, factor_of, frame_of, poses, frame poses)"""
    import test_gpu_geometric_batch as tg
    import test_gpu_reprojection_batch as tr
    from deepfactors_b200 import se3, synth
    from deepfactors_b200.aligners import DenseSfmParams, SfmAligner, SfmAlignerParams
    from deepfactors_b200.window_opt import SfmWindowProblem, TrackedFrame
    base, cams, kf = tg._window_scene(torch, cs, 2)
    kf3 = [{k: v.clone() for k, v in lv.items()} for lv in kf[2]]
    al = SfmAligner(cs, SfmAlignerParams(sfmparams=DenseSfmParams(valid_border=1, min_dpt=0.0)))
    frame_lv = []
    for l, L in enumerate(base.levels):
        img = synth.rotated_view(L, float(2 ** l), [0.004, -0.005, 0.003]).astype(np.float32)
        frame_lv.append(dict(img=torch.from_numpy(img).cuda(), grad=torch.from_numpy(synth.sobel_np(img)).cuda()))
    rep, geo = tr._links(base), tg._geo_links(base)
    pairs = [(0, 1), (1, 2), (2, 0), (1, 0)]

    def grown():
        return SfmWindowProblem(al, cams, kf + [kf3], pairs + [(3, 2), (2, 3)], links=[rep[0], rep[1]],
                                geometric=[geo[0], geo[2]], frames=[TrackedFrame(1, frame_lv), TrackedFrame(3, frame_lv)])
    old = SfmWindowProblem(al, cams, kf, pairs, links=[rep[0]], geometric=[geo[0]], frames=[TrackedFrame(1, frame_lv)])
    # old: photometric 0-3, reprojection 4, frame 5, geometric 6; new: photometric 0-5, reprojection 6-7, frames 8-9,
    # geometric 10-11
    factor_of = [0, 1, 2, 3, None, None, 4, None, 5, None, 6, None]
    poses = np.concatenate([tg._window_poses(), se3.make_pose([0.002, 0.003, -0.001], [0.01, -0.02, 0.005],
                                                               np.float64)[None]])
    fposes = np.stack([se3.make_pose([0.002, -0.001, 0.003], [0.01, 0.004, -0.006], np.float64),
                       se3.make_pose([-0.001, 0.002, 0.001], [0.004, 0.01, -0.003], np.float64)])
    return old, grown(), grown(), factor_of, [0, None], poses, fposes


def _rows(prob, i):
    """(buffer, first row, rows) of factor i's records"""
    for kd in prob._kinds.values():
        if kd.first <= i < kd.first + len(kd.ends):
            return kd.base, kd.row0 + (i - kd.first) * kd.rows, kd.rows
    raise IndexError(i)


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [8, 32])
def test_grown_problem_keeps_its_factors_records(cs):
    """IncrementalOptimizer.grow_problem on SfmWindowProblem: the grown problem re-evaluates only the new factors;
    every kept factor's records are bit for bit the old problem's records of that factor; every record and the buffer
    match an all-stale linearisation of the grown window at the same theta_lin.  The last comparison is within fp32
    rounding, not bit for bit: a RunStep batch's tile-to-CTA split follows its total tile count (DESIGN §4.7), so the
    same item rounds differently in another batch.  A record of another factor is orders of magnitude further off."""
    import torch
    old, new, ref, factor_of, frame_of, poses, fposes = _grown_scene(torch, cs)
    rng = np.random.default_rng(5)
    codes = rng.standard_normal((4, cs)) * 0.05
    opt = IncrementalOptimizer.from_problem(old, poses[:3], codes[:3], fposes[:1], relinearize_threshold=1e9,
                                            code_prior_weight=0.1)
    assert opt.update().factors_relinearised == 7
    assert opt.update().factors_relinearised == 0
    # a wrong map (pair (0, 1) as old pair (1, 2); a frame pair mapped to another frame) raises and copies nothing
    before = ref.records.clone()
    for bad_f, bad_fr in (([1, 0] + factor_of[2:], frame_of), (factor_of, [None, 0])):
        with pytest.raises(ValueError):
            ref.carry_records(old, bad_f, bad_fr)
    assert torch.equal(ref.records, before)
    opt.grow_problem(old, new, poses, codes, fposes, factor_of, frame_of)
    seen = {}
    lin = opt.linearise

    def capture(*args):
        seen["todo"] = list(args[2])
        buf, f = lin(*args)
        seen["buf"] = buf.clone()
        return buf, f
    opt.linearise = capture
    r = opt.update()
    assert seen["todo"] == [4, 5, 7, 9, 11] and r.factors_relinearised == 5
    for i, o in enumerate(factor_of):
        if o is None:
            continue
        nb, n0, nr = _rows(new, i)
        ob, o0, orows = _rows(old, o)
        assert nr == orows and torch.equal(nb[n0:n0 + nr].view(torch.int32), ob[o0:o0 + nr].view(torch.int32)), i
    everything = list(range(len(ref.pairs) + len(ref.geometric)))
    want, _ = ref.linearise(opt.lin_poses, opt.lin_codes, everything, opt.lin_frames)
    worst = 0.0
    for i in everything:
        nb, n0, nr = _rows(new, i)
        rb, r0, _ = _rows(ref, i)
        a, b = nb[n0:n0 + nr].double(), rb[r0:r0 + nr].double()
        err = float((a - b).abs().max() / b.abs().max())
        worst = max(worst, err)
        assert err <= 1e-5, (i, err)
    got = seen["buf"].double()
    berr = float((got - want.double()).abs().max() / want.double().abs().max())
    assert berr <= 1e-5, berr
    print(f"C={cs}: worst record difference {worst:.1e}, buffer {berr:.1e} (relative to the largest entry)")
