"""Tracked frames in the keyframe window on the device: assembly of frame windows (dfk_window_create_frames) against
WindowBlocks.pack, the device solve with frames eliminated first against the dense damped solve of to_dense,
marginalisation (dfk_window_marginalize_frames) and prior addition (dfk_window_add_priors) against fp64 numpy, and an
LM window with tracked frames run through both solves."""
import numpy as np
import pytest

from deepfactors_b200 import factors, se3, synth
from test_gpu_window_solve import damped_system
from test_window_frames import frame_window, random_records, schur_prior

pytestmark = pytest.mark.gpu


def pack_records(JtJ, Jtr, res, inl, cs):
    """device-format records [n, REC] (packed upper JtJ | Jtr | residual | inliers bits) of float32 systems"""
    n_, nh, rec = factors.record_layout(cs)
    iu = np.triu_indices(n_)
    out = np.zeros((len(JtJ), rec), np.float32)
    out[:, :nh] = np.asarray(JtJ, np.float32)[:, iu[0], iu[1]]
    out[:, nh:nh + n_] = Jtr
    out[:, nh + n_] = res
    out[:, nh + n_ + 1] = np.asarray(inl, np.uint32).view(np.float32)
    return out


def random_geo(L, cs, rng):
    NG = 12 + 2 * cs
    A = rng.standard_normal((L, 2 * NG, NG + 1))
    return (np.einsum("nri,nrj->nij", A[..., :NG], A[..., :NG]).astype(np.float32),
            np.einsum("nri,nr->ni", A[..., :NG], A[..., NG]).astype(np.float32), np.ones(L, np.float32))


def pack_geo(geo, cs):
    n_, nh, rec = factors.geo_record_layout(cs)
    iu = np.triu_indices(n_)
    out = np.zeros((len(geo[0]), rec), np.float32)
    out[:, :nh] = geo[0][:, iu[0], iu[1]]
    out[:, nh:nh + n_] = geo[1]
    out[:, nh + n_] = geo[2]
    return out


FRAMES_OF = {"none": [0, 0, 0, 0], "one_each": [1, 1, 1, 1], "mixed": [3, 0, 1, 2]}


@pytest.mark.parametrize("cs", [8, 32, 128])
@pytest.mark.parametrize("layout", list(FRAMES_OF))
@pytest.mark.parametrize("links", [False, True])
def test_frame_window_assembly_equals_pack(cs, layout, links):
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window
    rng = np.random.default_rng(cs + 7 * len(layout) + links)
    K = 4
    pairs, F, item_pair, sizes = frame_window(K, FRAMES_OF[layout])
    JtJ, Jtr, res, inl = random_records(len(item_pair), cs, rng)
    rec = pack_records(JtJ, Jtr, res, inl, cs)
    H, g, r_, n_ = factors.unpack_records(rec, cs)
    geo_pairs = [(0, 2), (3, 1)] if links else []
    geo = random_geo(len(geo_pairs), cs, rng) if links else None
    al = SfmAligner(cs)
    win = Window(al, K, pairs, item_pair, sizes, geo_pairs, F)
    assert win.floats == win.layout.floats == factors.WindowBlocks(K, cs, pairs, geo_pairs).floats + 42 * F
    grec = torch.from_numpy(pack_geo(geo, cs)).cuda() if links else None
    buf = win.assemble(torch.from_numpy(rec).cuda(), geo_records=grec).cpu().numpy()
    want = win.layout.pack(item_pair, H, g, r_, n_, sizes, geo=geo)
    assert np.abs(buf - want).max() <= 2e-6 * np.abs(want).max()
    # the new parts are the same chains of float32 adds in item order: bit for bit
    o_f = win.layout.frame_offset
    assert np.array_equal(buf[o_f:], want[o_f:])
    o_c, o_t = win.layout.offsets()[1:]
    assert np.array_equal(buf[o_c:o_t], want[o_c:o_t])
    assert buf[o_t + 1] == float(n_.sum())
    B = 6 + cs
    kf1 = {k1 for k0, k1 in pairs if k1 < K} | {k1 for _, k1 in geo_pairs}
    for k in set(range(K)) - kf1:  # no k1 items: the diagonal block sums in item order exactly as pack does
        assert np.array_equal(buf[k * B * B:(k + 1) * B * B], want[k * B * B:(k + 1) * B * B])
    # two launches, same bits
    assert np.array_equal(win.assemble(torch.from_numpy(rec).cuda(), geo_records=grec).cpu().numpy(), buf)


@pytest.mark.parametrize("cs", [8, 32])
def test_window_without_frames_is_the_previous_builds_bit_for_bit(cs):
    """a window without frames, created through dfk_window_create_frames (Window), assembles bit for bit the buffer the
    build before tracked frames assembled from the same records (tests/golden/window_without_frames.npz)"""
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window
    from test_window_frames import load_parent_fixture
    fx = load_parent_fixture(cs)
    win = Window(SfmAligner(cs), fx["K"], fx["pairs"], fx["item_pair"], fx["sizes"], fx["geo_pairs"], 0)
    buf = win.assemble(torch.from_numpy(fx["records"]).cuda(), geo_records=torch.from_numpy(fx["geo_records"]).cuda())
    assert np.array_equal(buf.cpu().numpy(), fx["device"])


def test_frame_window_rejects_bad_structures_and_writes_nothing():
    import torch
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner, Window
    al = SfmAligner(8)
    K = 3
    ok = [(0, 1), (1, 2), (0, 3)]
    Window(al, K, ok, [0, 1, 2], [(8, 6)] * 3, (), 1)
    bad = [
        ([(0, 1), (1, 2)], [0, 1], [(8, 6)] * 2, (), 1),                 # frame 0 is k1 of no pair
        ([(0, 1), (0, 3), (1, 3)], [0, 1, 2], [(8, 6)] * 3, (), 1),      # frame 0 is k1 of two pairs
        ([(0, 1), (3, 1), (0, 3)], [0, 1, 2], [(8, 6)] * 3, (), 1),      # frame 0 as k0
        ([(0, 1), (0, 3)], [0, 1], [(8, 6)] * 2, [(0, 3)], 1),           # frame 0 in a link
        ([(0, 1), (0, 3)], [0, 1], [(8, 6), (0, 0)], (), 1),             # unscaled item on a frame pair
        ([(0, 1), (0, 4)], [0, 1], [(8, 6)] * 2, (), 1),                 # beyond the frames
    ]
    for pairs, ip, sizes, geo, F in bad:
        with pytest.raises(_lib.DfkError):
            Window(al, K, pairs, ip, sizes, geo, F)
    win = Window(al, K, ok, [0, 1, 2], [(8, 6)] * 3, (), 1)
    rec = torch.zeros((3, _lib.record_floats(8)), device="cuda")
    for frames in ([1], [-1]):
        with pytest.raises(_lib.DfkError):
            win.marginalize_frames(rec, frames)
    buf = torch.full((win.floats,), 3.0, device="cuda")
    pr = torch.zeros((1, _lib.prior_doubles(8)), dtype=torch.float64, device="cuda")
    with pytest.raises(_lib.DfkError):
        win.add_priors(buf, [K], pr, torch.zeros((1, 14), dtype=torch.float64, device="cuda"))
    torch.cuda.synchronize()
    assert torch.all(buf == 3.0)


def solve_case(cs, rng, K=5, frames_of=(2, 0, 1, 3, 1), scale=1.0):
    from deepfactors_b200.factors import WindowBlocks
    pairs = [(k, k + 1) for k in range(K - 1)] + [(K - 1, 0), (2, 0)]
    F = 0
    for k, nf in enumerate(frames_of):
        for _ in range(nf):
            pairs.append((k, K + F))
            F += 1
    layout = WindowBlocks(K, cs, pairs, num_frames=F)
    JtJ, Jtr, res, inl = random_records(len(pairs), cs, rng, scale)
    buf = layout.pack(list(range(len(pairs))), JtJ, Jtr, res, inl, [(4, 4)] * len(pairs))
    return pairs, F, layout, buf


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_frame_window_solve_matches_dense_damped_solve(cs):
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window, WindowSolver
    from deepfactors_b200.window_opt import damped_solve
    rng = np.random.default_rng(200 + cs)
    K = 5
    pairs, F, layout, buf_h = solve_case(cs, rng, K)
    al = SfmAligner(cs)
    win = Window(al, K, pairs, list(range(len(pairs))), [(4, 4)] * len(pairs), (), F)
    buf = torch.from_numpy(buf_h).cuda()
    B = 6 + cs
    codes = rng.standard_normal((K, cs)) * 0.3
    worst = [0.0, 0.0]
    for fixed in ((), tuple(range(6))):
        sol = WindowSolver(win, fixed)
        for lam in (0.0, 1e-4, 1e3):
            for w in (0.0, 1e-2):
                dx, info = sol.solve(buf, lam, w, codes)
                assert dx.numel() == K * B + 6 * F
                dxh = dx.cpu().numpy()
                assert int(info.item()) == 0
                A, b, keep = damped_system(layout, buf_h, lam, fixed, w, codes)
                x = dxh[keep]
                berr = np.abs(A @ x - b).max() / (np.abs(A).sum(1).max() * np.abs(x).max() + np.abs(b).max())
                assert berr <= 1e-12, (fixed, lam, w, berr)
                assert np.all(dxh[list(fixed)] == 0.0)
                H, g, _, _ = layout.to_dense(buf)
                if w > 0:
                    for k in range(K):
                        sl = slice(k * B + 6, (k + 1) * B)
                        H[sl, sl] += w * torch.eye(cs, dtype=H.dtype, device=H.device)
                        g[sl] -= w * torch.as_tensor(codes[k], dtype=g.dtype, device=g.device)
                ref = damped_solve(H, g, lam, fixed).cpu().numpy()
                cond = np.linalg.cond(A)
                assert cond <= 1e6, cond
                ferr = np.abs(dxh - ref).max() / np.abs(ref).max()
                assert ferr <= 1e-9, (fixed, lam, w, ferr)
                worst = [max(worst[0], berr), max(worst[1], ferr)]
                dx2, _ = sol.solve(buf, lam, w, codes)
                assert torch.equal(dx, dx2)
    print(f"C={cs} F={F}: worst backward error {worst[0]:.2e} worst |dx - torch|/|dx| {worst[1]:.2e}")


def test_frame_window_solve_reports_a_bad_frame_then_recovers():
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window, WindowSolver
    from deepfactors_b200.window_opt import damped_solve
    cs, K = 16, 5
    rng = np.random.default_rng(5)
    pairs, F, layout, good = solve_case(cs, rng, K)
    al = SfmAligner(cs)
    win = Window(al, K, pairs, list(range(len(pairs))), [(4, 4)] * len(pairs), (), F)
    B = 6 + cs
    bad = good.copy()
    o = layout.frame_offset
    Df = bad[o:o + 36 * F].reshape(F, 6, 6)
    Df[3] = -np.eye(6, dtype=np.float32)   # frame 3's block negative definite: its first pivot fails at lambda = 0
    sol = WindowSolver(win, range(6))
    dx = torch.full((K * B + 6 * F,), 7.0, dtype=torch.float64, device="cuda")
    _, info = sol.solve(torch.from_numpy(bad).cuda(), 0.0, dx=dx)
    assert int(info.item()) == 1 + K * B + 6 * 3
    assert torch.all(dx == 0)
    _, info = sol.solve(torch.from_numpy(good).cuda(), 0.0, dx=dx)
    assert int(info.item()) == 0
    H, g, _, _ = layout.to_dense(torch.from_numpy(good).cuda())
    ref = damped_solve(H, g, 0.0, range(6))
    assert (dx - ref).abs().max() <= 1e-9 * ref.abs().max()


def entry_scale_prior(cs, JtJ, Jtr):
    """per-entry scale of the Schur complement's terms (|H_aa| + |H_ab| |H_bb^-1| |H_ab|^T, ...), for relative bars"""
    a = np.r_[0:6, 12:12 + cs]
    Hs = np.abs(np.sum(np.asarray(JtJ, np.float64), axis=0))
    Hsi = np.abs(np.linalg.inv(np.sum(np.asarray(JtJ, np.float64), axis=0)[6:12, 6:12]))
    gs = np.abs(np.sum(np.asarray(Jtr, np.float64), axis=0))
    Hab = Hs[np.ix_(a, np.arange(6, 12))]
    G = Hs[np.ix_(a, a)] + Hab @ Hsi @ Hab.T
    g = gs[a] + Hab @ Hsi @ gs[6:12]
    return G, g, gs[6:12] @ Hsi @ gs[6:12]


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_marginalize_frames_and_add_priors_match_numpy(cs):
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window
    rng = np.random.default_rng(300 + cs)
    K = 4
    pairs, F, item_pair, sizes = frame_window(K, [2, 0, 1, 1], levels=3)
    JtJ, Jtr, res, inl = random_records(len(item_pair), cs, rng)
    # frame 3's items see nothing of its pose: a singular block
    p3 = pairs.index((3, K + 3))
    for i in [i for i, p in enumerate(item_pair) if p == p3]:
        JtJ[i][6:12, :] = 0
        JtJ[i][:, 6:12] = 0
    rec = pack_records(JtJ, Jtr, res, inl, cs)
    H, g, r_, n_ = factors.unpack_records(rec, cs)
    al = SfmAligner(cs)
    win = Window(al, K, pairs, item_pair, sizes, (), F)
    rec_d = torch.from_numpy(rec).cuda()
    which = [2, 0, 3, 1]
    priors, info = win.marginalize_frames(rec_d, which)
    priors, info = priors.cpu().numpy(), info.cpu().numpy()
    B = 6 + cs
    worst = 0.0
    for i, f in enumerate(which):
        p = pairs.index(next(pp for pp in pairs if pp[1] == K + f))
        mine = [j for j, q in enumerate(item_pair) if q == p]
        if f == 3:
            assert info[i] == 1 and np.all(priors[i] == 0)
            continue
        assert info[i] == 0
        want = schur_prior(cs, H[mine], g[mine], r_[mine], n_[mine], [sizes[j] for j in mine])
        sG, sg, sf = entry_scale_prior(cs, H[mine], g[mine])
        scale = np.concatenate([sG.ravel(), sg, [abs(want[-1]) + sf]])
        err = np.abs(priors[i] - want) / scale
        worst = max(worst, err.max())
        assert err.max() <= 1e-11, (f, err.max())
        G = priors[i][:B * B].reshape(B, B)
        assert np.array_equal(G, G.T)
    print(f"C={cs}: marginal priors, worst entry error / entry scale {worst:.2e}")
    # add_priors: two priors on keyframe 0 and one on keyframe 2, in list order, at random deltas
    buf_h = win.layout.pack(item_pair, H, g, r_, n_, sizes)
    buf = torch.from_numpy(buf_h).cuda()
    use = [0, 1, 3]                   # priors of frames 2, 0, 1 (keyframes 2, 0, 0)
    kf = [pairs[pairs.index(next(pp for pp in pairs if pp[1] == K + which[i]))][0] for i in use]
    rows = priors[use]
    delta = rng.standard_normal((len(use), B)) * 0.01
    win.add_priors(buf, kf, torch.from_numpy(np.ascontiguousarray(rows)).cuda(), torch.from_numpy(delta).cuda())
    got = buf.cpu().numpy()
    want = buf_h.copy()
    D = want[:K * B * B].reshape(K, B, B)
    gk = want[K * B * B:K * (B * B + B)].reshape(K, B)
    o_t = win.layout.offsets()[2]
    for k in range(K):
        mine = [q for q in range(len(use)) if kf[q] == k]
        if not mine:
            continue
        Ds = D[k].astype(np.float64)
        gs = gk[k].astype(np.float64)
        for q in mine:
            G = rows[q][:B * B].reshape(B, B)
            Ds = Ds + G
            gs = gs + (rows[q][B * B:B * B + B] - G @ delta[q])
        D[k] = Ds.astype(np.float32)
        gk[k] = gs.astype(np.float32)
    f = np.float64(want[o_t])
    for q in range(len(use)):
        G, gp, f0 = rows[q][:B * B].reshape(B, B), rows[q][B * B:B * B + B], rows[q][-1]
        f = f + (f0 - 2 * gp @ delta[q] + delta[q] @ G @ delta[q])
    want[o_t] = np.float32(f)
    # D: the same fp64 chain rounded once, bit for bit; g and f within one float32 rounding of the fp64 value
    assert np.array_equal(got[:K * B * B], want[:K * B * B])
    assert np.abs(got - want).max() <= 2e-7 * np.abs(want).max()
    assert got[o_t + 1] == buf_h[o_t + 1]
    assert np.array_equal(got[K * (B * B + B):o_t], buf_h[K * (B * B + B):o_t])


def test_schur_identity_through_the_device_path():
    """A window with frame 0 (on the gauge keyframe) solved on the device gives the keyframe dx of the window without
    it plus its device-made prior added at delta = 0, to the float32 rounding of the two buffers."""
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window, WindowSolver
    cs = 32
    rng = np.random.default_rng(41)
    K = 3
    pairs, F, item_pair, sizes = frame_window(K, [1, 1, 1])
    JtJ, Jtr, res, inl = random_records(len(item_pair), cs, rng)
    rec = torch.from_numpy(pack_records(JtJ, Jtr, res, inl, cs)).cuda()
    al = SfmAligner(cs)
    B = 6 + cs
    win = Window(al, K, pairs, item_pair, sizes, (), F)
    dx, info = WindowSolver(win, range(6)).solve(win.assemble(rec), 0.0)
    assert int(info.item()) == 0
    prior, pinfo = win.marginalize_frames(rec, [0])
    assert int(pinfo.item()) == 0
    fp = pairs.index((0, K))
    rest = [i for i in range(len(item_pair)) if item_pair[i] != fp]
    pairs2 = pairs[:fp] + [(k0, k1 - 1) for k0, k1 in pairs[fp + 1:]]
    ip2 = [p if p < fp else p - 1 for p in np.asarray(item_pair)[rest]]
    win2 = Window(al, K, pairs2, ip2, [sizes[i] for i in rest], (), F - 1)
    buf2 = win2.assemble(rec[torch.as_tensor(rest, device="cuda")].contiguous())
    win2.add_priors(buf2, [0], prior, torch.zeros((1, B), dtype=torch.float64, device="cuda"))
    dx2, info2 = WindowSolver(win2, range(6)).solve(buf2, 0.0)
    assert int(info2.item()) == 0
    a, b = dx[:K * B].cpu().numpy(), dx2[:K * B].cpu().numpy()
    err = np.abs(a - b).max() / np.abs(a).max()
    print(f"Schur identity through the device: |dx_kf - dx_kf(prior)| / |dx_kf| = {err:.2e}")
    assert err <= 1e-4
    assert np.abs(dx[K * B + 6:].cpu().numpy() - dx2[K * B:].cpu().numpy()).max() <= 1e-4 * np.abs(a).max()


def _scene(cs, levels):
    import torch
    base = synth.make_pair(160, 120, cs, levels, seed=5)
    cams = [L.cam for L in base.levels]
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    keyframes = []
    for k in range(3):
        lv = []
        for L in base.levels:
            img = up(L.img0)
            lv.append(dict(img=img, grad=up(synth.sobel_np(L.img0)), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac),
                           dpt=torch.zeros_like(img), valid=torch.zeros_like(img)))
        keyframes.append(lv)
    return base, cams, keyframes


def test_window_lm_with_tracked_frames_device_solve_takes_the_torch_path_steps():
    """The 3-keyframe window of test_window_lm_with_device_solve_takes_the_torch_path_steps (every keyframe's true pose
    the identity) plus one tracked frame per keyframe, started at perturbed poses.  Frame 0 sees its keyframe's images
    (true pose the identity); frames 1 and 2 are views rendered at known rotations (synth.rotated_view).  The device
    solve takes the torch path's steps and the frames converge to their true poses; then the frames are marginalised and
    the window without them re-solved from the optimum stays there."""
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, TrackedFrame, WindowOptimizer
    import torch
    cs, levels = 8, 2
    base, cams, keyframes = _scene(cs, levels)
    al = SfmAligner(cs)
    pairs = [(0, 1), (1, 2), (2, 0), (1, 0), (2, 1)]
    omegas = [np.zeros(3), np.array([0.006, -0.008, 0.004]), np.array([-0.005, 0.004, 0.007])]
    truth = np.stack([se3.retract(se3.identity(np.float64), np.r_[0.0, 0.0, 0.0, w], np.float64) for w in omegas])
    frames = []
    for k in range(3):
        lv = []
        for l, L in enumerate(base.levels):
            img = synth.rotated_view(L, float(2 ** l), omegas[k]).astype(np.float32)
            lv.append(dict(img=torch.from_numpy(img).cuda(), grad=torch.from_numpy(synth.sobel_np(img)).cuda()))
        frames.append(TrackedFrame(k, lv))
    prob = SfmWindowProblem(al, cams, keyframes, pairs, frames=frames)
    assert prob.layout.num_frames == 3 and prob.layout.dim == 3 * (6 + cs) + 18
    poses = np.stack([se3.identity(np.float64),
                      se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                      se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.006], np.float64)])
    fposes = np.stack([se3.make_pose([0.003, 0.002, -0.002], [0.01, 0.008, -0.01], np.float64),
                       se3.make_pose([-0.002, 0.003, 0.001], [-0.012, 0.006, 0.01], np.float64),
                       se3.make_pose([0.002, -0.002, 0.003], [0.008, -0.01, 0.012], np.float64)])
    codes = np.zeros((3, cs))
    prm = LMParams(iterations=12, lambda_init=1e-3, code_prior_weight=1e-2)
    p0, c0, t0 = WindowOptimizer(prob.layout, prob.linearise, prm).run(poses, codes, fposes)
    p1, c1, t1 = WindowOptimizer(prob.layout, prob.linearise, prm, solve=prob.solve).run(poses, codes, fposes)
    assert t1.accepted == t0.accepted
    assert t1.lam == t0.lam
    assert t1.factors_relinearised == t0.factors_relinearised
    assert np.allclose(t1.energy, t0.energy, rtol=1e-6, atol=0)
    assert np.abs(p1 - p0).max() <= 1e-6 and np.abs(t1.frame_poses - t0.frame_poses).max() <= 1e-6
    assert t1.energy[-1] < t1.energy[0] / 20.0
    assert np.array_equal(p1[0], poses[0])
    # the frames converge to their true poses (and the keyframes to theirs, the identity)
    assert np.abs(truth[1:] - fposes[1:]).max() > 0.005  # rendered away from the start, not at the identity
    for f in range(3):
        e0 = np.abs(se3.local(truth[f], fposes[f])).max()
        e1 = np.abs(se3.local(truth[f], t1.frame_poses[f])).max()
        print(f"frame {f}: |local(truth, frame)| {e0:.2e} -> {e1:.2e}")
        assert e1 < 0.05 * e0 and e1 < 1e-3
    # marginalised where they are, the frames leave the same problem on the keyframes: at the start point the undamped
    # step of the window without frames, with their priors, is the keyframe part of the full window's (Schur identity,
    # both through the device; marginalize leaves prob's records alone, so linearise re-evaluates everything)
    w = prm.code_prior_weight
    priors0 = prob.marginalize(poses, codes, fposes, [0, 1, 2])
    prob_s = SfmWindowProblem(al, cams, keyframes, pairs, priors=priors0)
    buf_full, _ = prob.linearise(poses, codes, list(range(len(prob.pairs))), fposes)
    buf_red, _ = prob_s.linearise(poses, codes, list(range(len(prob_s.pairs))))
    dx_full = prob.solve(buf_full, 0.0, range(6), w, codes)
    dx_red = prob_s.solve(buf_red, 0.0, range(6), w, codes)
    n = prob_s.layout.dim
    step = np.abs(dx_red - dx_full[:n]).max() / np.abs(dx_full[:n]).max()
    # marginalised at the final point, LM on the window without frames keeps the keyframe poses (the codes, weakly
    # constrained, may still creep on)
    priors = prob.marginalize(p1, c1, t1.frame_poses, [0, 1, 2])
    assert [pr.k for pr in priors] == [0, 1, 2]
    prob2 = SfmWindowProblem(al, cams, keyframes, pairs, priors=priors)
    assert prob2.layout.num_frames == 0
    p2, c2, t2 = WindowOptimizer(prob2.layout, prob2.linearise, prm, solve=prob2.solve).run(p1, c1)
    moved = max(np.abs(se3.local(p1[k], p2[k])).max() for k in range(3))
    print(f"at the start: |dx_kf(priors) - dx_kf(frames)| / |dx_kf| = {step:.2e}; LM without the frames from the final "
          f"point moves the keyframe poses by {moved:.2e}, the codes by {np.abs(c2 - c1).max():.2e}")
    assert step <= 1e-3
    assert moved <= 1e-3
    assert t2.energy[-1] <= t2.energy[0]
