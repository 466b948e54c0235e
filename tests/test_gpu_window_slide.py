"""Sliding the keyframe window on the device: dfk_window_marginalize_keyframe against the fp64 numpy Schur complement of
test_window_slide.py (every factor kind touching the keyframe), dfk_window_add_keyframe_priors against
WindowBlocks.add_keyframe_priors, dfk_window_solve of a window with prior blocks against the dense damped solve, and the
end-to-end slide of a synthetic window: the slid window's step is the kept part of the full window's, and at the
optimum it stays put, once and twice slid."""
import numpy as np
import pytest

from deepfactors_b200 import _lib, se3
from test_gpu_window_frames import _scene, pack_geo, pack_records
from test_gpu_window_solve import damped_system
from test_window_slide import blanket, local_system, random_kf_prior, scene, schur_row

pytestmark = pytest.mark.gpu


def slide_case(cs, rng):
    """scene() plus an unscaled record on a pair of keyframe 2, a tracked frame on keyframe 4, two frame priors on 2 and
    three keyframe priors (two of them over 2)"""
    import torch
    K, B = 5, 6 + cs
    pairs, item_pair, sizes, rec, geo_pairs, geo = scene(cs, rng, K)
    from test_window_frames import random_records
    extra = random_records(2, cs, rng, 0.5)
    pairs = pairs + [(3, 2), (4, K)]               # (3, 2): one unscaled record; (4, K): frame 0 on keyframe 4
    item_pair = item_pair + [len(pairs) - 2, len(pairs) - 1]
    sizes = sizes + [(0, 0), (20, 15)]
    rec = tuple(np.concatenate([a, b]) for a, b in zip(rec, extra))
    kp = [random_kf_prior((1, 2, 3), cs, rng), random_kf_prior((0, 2), cs, rng), random_kf_prior((3, 4), cs, rng)]
    fp = [(2,) + random_kf_prior((2,), cs, rng)[1:], (2,) + random_kf_prior((2,), cs, rng)[1:]]
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dev = dict(rec=up(pack_records(*rec, cs)), geo=up(pack_geo(geo, cs)),
               kp=up(np.concatenate([r for _, r, _ in kp])), kd=up(np.concatenate([d for _, _, d in kp])),
               fp=up(np.stack([r for _, r, _ in fp])), fd=up(np.stack([d for _, _, d in fp])))
    return K, B, pairs, item_pair, sizes, rec, geo_pairs, geo, kp, fp, dev


def entry_scale(Hl, gl, fl, B):
    """per-entry scale of the Schur complement's terms: |H_NN| + |H_Nm| |H_mm^-1| |H_mN|, |g_N| + ..., |f| + ..."""
    A, a = np.abs(Hl), np.abs(gl)
    Mi = np.abs(np.linalg.inv(Hl[:B, :B]))
    G = A[B:, B:] + A[B:, :B] @ Mi @ A[:B, B:]
    g = a[B:] + A[B:, :B] @ Mi @ a[:B]
    return np.maximum(np.concatenate([G.ravel(), g, [abs(fl) + a[:B] @ Mi @ a[:B]]]), 1e-300)


@pytest.mark.parametrize("cs", [8, 32, 128])
@pytest.mark.parametrize("w", [0.0, 1e-2])
def test_marginalize_keyframe_matches_numpy(cs, w):
    from deepfactors_b200.aligners import SfmAligner, Window
    rng = np.random.default_rng(cs + int(w * 1000))
    K, B, pairs, item_pair, sizes, rec, geo_pairs, geo, kp, fp, dev = slide_case(cs, rng)
    win = Window(SfmAligner(cs), K, pairs, item_pair, sizes, geo_pairs, 1, [p[0] for p in kp])
    m = 2
    nb = win.blanket(m)
    assert nb == blanket(K, m, pairs, geo_pairs, [p[0] for p in kp]) == [0, 1, 3, 4]
    code = rng.standard_normal(cs) * 0.3
    codes = np.zeros((K, cs))
    codes[m] = code
    args = (dev["rec"], m, dev["geo"], dev["fp"], dev["fd"], dev["kp"], dev["kd"], w, code)
    prior, info = win.marginalize_keyframe(*args)
    assert int(info.item()) == 0
    got = prior.cpu().numpy()
    Hl, gl, fl = local_system(K, cs, m, nb, pairs=pairs, item_pair=item_pair, JtJ=rec[0], Jtr=rec[1], res=rec[2],
                              inl=rec[3], sizes=sizes, geo_pairs=geo_pairs, geo=geo, frame_priors=fp, kf_priors=kp,
                              w=w, codes=codes)
    want = schur_row(Hl, gl, fl, B)
    err = np.abs(got - want) / entry_scale(Hl, gl, fl, B)
    print(f"C={cs} w={w}: keyframe prior over {len(nb)} keyframes, worst entry error / entry scale {err.max():.2e}")
    assert err.max() <= 1e-11
    nB = len(nb) * B
    G = got[:nB * nB].reshape(nB, nB)
    assert np.array_equal(G, G.T)
    prior2, _ = win.marginalize_keyframe(*args)
    assert np.array_equal(prior2.cpu().numpy(), got)


def test_marginalize_keyframe_reports_a_singular_block_then_recovers_and_rejects_bad_calls():
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window
    cs = 16
    rng = np.random.default_rng(3)
    K, B, pairs, item_pair, sizes, rec, geo_pairs, geo, kp, fp, dev = slide_case(cs, rng)
    win = Window(SfmAligner(cs), K, pairs, item_pair, sizes, geo_pairs, 1, [p[0] for p in kp])
    bad_fp = dev["fp"].clone()
    bad_fp[0, :B * B] = -1e9 * torch.eye(B, dtype=torch.float64, device="cuda").reshape(-1)
    prior, info = win.marginalize_keyframe(dev["rec"], 2, dev["geo"], bad_fp, dev["fd"], dev["kp"], dev["kd"])
    assert int(info.item()) == 1
    assert torch.all(prior == 0)
    prior, info = win.marginalize_keyframe(dev["rec"], 2, dev["geo"], dev["fp"], dev["fd"], dev["kp"], dev["kd"],
                                           prior=prior, info=info)
    assert int(info.item()) == 0 and torch.any(prior != 0)
    # keyframe 4 still has a tracked frame; keyframe 0 of a 17-spoke star has a blanket of 17: nothing written
    out = torch.full((_lib.kf_prior_doubles(cs, 4),), 7.0, dtype=torch.float64, device="cuda")
    inf = torch.full((1,), 5, dtype=torch.int32, device="cuda")
    with pytest.raises(_lib.DfkError):
        win.marginalize_keyframe(dev["rec"], 4, dev["geo"], kf_priors=dev["kp"], kf_delta=dev["kd"], prior=out,
                                 info=inf)
    star = [(0, k) for k in range(1, 18)]
    swin = Window(SfmAligner(cs), 18, star, list(range(17)), [(8, 6)] * 17)
    assert swin.blanket(0) == list(range(1, 18)) and swin.blanket(5) == [0]
    srec = torch.zeros((17, _lib.record_floats(cs)), device="cuda")
    with pytest.raises(_lib.DfkError) as e:
        swin.marginalize_keyframe(srec, 0, prior=torch.full((_lib.kf_prior_doubles(cs, 17),), 7.0,
                                                            dtype=torch.float64, device="cuda"), info=inf)
    assert e.value.status == _lib.DFK_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert torch.all(out == 7.0) and int(inf.item()) == 5


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_add_keyframe_priors_matches_the_numpy_mirror(cs):
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window
    rng = np.random.default_rng(50 + cs)
    K, B, pairs, item_pair, sizes, rec, geo_pairs, geo, kp, fp, dev = slide_case(cs, rng)
    win = Window(SfmAligner(cs), K, pairs, item_pair, sizes, geo_pairs, 1, [p[0] for p in kp])
    lay = win.layout
    assert win.floats == lay.floats
    buf = win.assemble(dev["rec"], geo_records=dev["geo"])
    host = buf.cpu().numpy()
    assert np.all(host[lay.prior_offset:] == 0)
    win.add_keyframe_priors(buf, dev["kp"], dev["kd"])
    got = buf.cpu().numpy()
    want = lay.add_keyframe_priors(host.copy(), [r for _, r, _ in kp], [d for _, _, d in kp])
    # D and the prior blocks: the same fp64 chains rounded once, bit for bit; g and f within a float32 rounding
    o_g, o_c, o_t = lay.offsets()
    assert np.array_equal(got[:o_g], want[:o_g])
    assert np.array_equal(got[lay.prior_offset:], want[lay.prior_offset:])
    scale = np.abs(want[o_g:o_c]).max()
    assert np.abs(got[o_g:o_c] - want[o_g:o_c]).max() <= 2e-7 * scale
    assert got[o_t] == pytest.approx(want[o_t], rel=1e-6)
    assert np.array_equal(got[o_c:o_t], host[o_c:o_t]) and got[o_t + 1] == host[o_t + 1]
    assert np.array_equal(got[o_t + 2:lay.prior_offset], host[o_t + 2:lay.prior_offset])


@pytest.mark.parametrize("cs", [8, 32, 128])
def test_window_with_prior_blocks_solve_matches_dense_damped_solve(cs):
    import torch
    from deepfactors_b200.aligners import SfmAligner, Window, WindowSolver
    from deepfactors_b200.window_opt import damped_solve
    rng = np.random.default_rng(90 + cs)
    K = 6
    B = 6 + cs
    pairs = [(k, k + 1) for k in range(K - 1)] + [(3, 1)]
    from test_window_frames import random_records
    JtJ, Jtr, res, inl = random_records(len(pairs), cs, rng)
    kp = [random_kf_prior((0, 3, 5), cs, rng), random_kf_prior((2, 4), cs, rng), random_kf_prior((0, 5), cs, rng)]
    win = Window(SfmAligner(cs), K, pairs, list(range(len(pairs))), [(4, 4)] * len(pairs), (), 0, [p[0] for p in kp])
    lay = win.layout
    buf_h = lay.add_keyframe_priors(lay.pack(list(range(len(pairs))), JtJ, Jtr, res, inl, [(4, 4)] * len(pairs)),
                                    [r for _, r, _ in kp], [d for _, _, d in kp])
    buf = torch.from_numpy(buf_h).cuda()
    codes = rng.standard_normal((K, cs)) * 0.3
    worst = [0.0, 0.0]
    for fixed in ((), tuple(range(6))):
        sol = WindowSolver(win, fixed)
        for lam in (0.0, 1e-4, 1e3):
            for w in (0.0, 1e-2):
                dx, info = sol.solve(buf, lam, w, codes)
                assert int(info.item()) == 0
                dxh = dx.cpu().numpy()
                A, b, keep = damped_system(lay, buf_h, lam, fixed, w, codes)
                x = dxh[keep]
                berr = np.abs(A @ x - b).max() / (np.abs(A).sum(1).max() * np.abs(x).max() + np.abs(b).max())
                assert berr <= 1e-12, (fixed, lam, w, berr)
                H, g, _, _ = lay.to_dense(buf)
                if w > 0:
                    for k in range(K):
                        sl = slice(k * B + 6, (k + 1) * B)
                        H[sl, sl] += w * torch.eye(cs, dtype=H.dtype, device=H.device)
                        g[sl] -= w * torch.as_tensor(codes[k], dtype=g.dtype, device=g.device)
                ref = damped_solve(H, g, lam, fixed).cpu().numpy()
                ferr = np.abs(dxh - ref).max() / np.abs(ref).max()
                assert ferr <= 1e-9, (fixed, lam, w, ferr)
                worst = [max(worst[0], berr), max(worst[1], ferr)]
                dx2, _ = sol.solve(buf, lam, w, codes)
                assert torch.equal(dx, dx2)
    print(f"C={cs}: {sol.tiles} tiles with prior blocks; worst backward error {worst[0]:.2e}, "
          f"|dx - torch|/|dx| {worst[1]:.2e}")


def _scene4(cs, levels):
    """test_gpu_window_frames' synthetic scene with four keyframes (every keyframe's true pose the identity)"""
    base, cams, kf = _scene(cs, levels)
    import torch
    extra = [{k: (torch.zeros_like(v) if k in ("dpt", "valid") else v) for k, v in lv.items()} for lv in kf[0]]
    return base, cams, kf + [extra]


def test_slid_window_step_is_the_kept_part_and_stays_at_the_optimum():
    """On a 4-keyframe synthetic window: at lambda = 0, the step of the window slid past keyframe 0 (device
    marginalisation, then the device solve) is the kept part of the full window's step with the gauge on keyframe 1
    (after dropping the gauge keyframe, the new first pose is fixed).  Slid at the optimum, LM keeps the kept poses.  A
    second slide, whose marginalisation folds the first prior in, keeps both properties."""
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, WindowOptimizer, drop_keyframe
    cs, levels = 8, 2
    base, cams, keyframes = _scene4(cs, levels)
    al = SfmAligner(cs)
    B = 6 + cs
    pairs = [(0, 1), (1, 0), (1, 2), (2, 1), (2, 3), (3, 2), (0, 2), (3, 1)]
    prob = SfmWindowProblem(al, cams, keyframes, pairs)
    poses = np.stack([se3.identity(np.float64),
                      se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                      se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.006], np.float64),
                      se3.make_pose([0.002, 0.003, -0.003], [0.008, 0.01, -0.012], np.float64)])
    codes = np.zeros((4, cs))
    w = 1e-2
    prm = LMParams(iterations=12, lambda_init=1e-3, code_prior_weight=w)

    def step_check(p_full, p, c, removed):
        """|dx(slid) - dx(full)[kept]| / |dx(full)[kept]| at (p, c), gauge on the first kept keyframe"""
        K = len(prob.kf)
        g = removed
        buf, _ = prob.linearise(p, c, list(range(len(prob.pairs) + len(prob.geometric))))
        dx = prob.solve(buf, 0.0, range(g * B, g * B + 6), w, c)
        ps, cs_ = drop_keyframe(p, c, 0)
        for _ in range(removed - 1):
            ps, cs_ = drop_keyframe(ps, cs_, 0)
        bs, _ = p_full.linearise(ps, cs_, list(range(len(p_full.pairs) + len(p_full.geometric))))
        dxs = p_full.solve(bs, 0.0, range(6), w, cs_)
        keep = np.concatenate([np.arange(k * B, (k + 1) * B) for k in range(removed, K)])
        return np.abs(dxs - dx[keep]).max() / np.abs(dx[keep]).max()

    # slide once at the start point
    pr1 = prob.marginalize_keyframe(poses, codes, 0, code_prior_weight=w)
    assert pr1.keyframes == (1, 2)
    s1 = prob.without_keyframe(0, pr1)
    assert len(s1.kf) == 3 and s1.layout.kf_priors == [(0, 1)]
    e1 = step_check(s1, poses, codes, 1)
    # twice: keyframe 1 of the full window (0 of s1) is in pr1, which the second marginalisation folds in
    p1s, c1s = drop_keyframe(poses, codes, 0)
    pr2 = s1.marginalize_keyframe(p1s, c1s, 0, code_prior_weight=w)
    s2 = s1.without_keyframe(0, pr2)
    assert len(s2.kf) == 2 and s2.layout.kf_priors == [(0, 1)]
    e2 = step_check(s2, poses, codes, 2)
    print(f"slid step vs the full window's kept step: once {e1:.2e}, twice {e2:.2e}")
    assert e1 <= 1e-4 and e2 <= 1e-4
    # at the optimum of the full window, the slid windows stay put
    p_opt, c_opt, t = WindowOptimizer(prob.layout, prob.linearise, prm, solve=prob.solve).run(poses, codes)
    assert t.energy[-1] < t.energy[0] / 20.0
    q1 = prob.marginalize_keyframe(p_opt, c_opt, 0, code_prior_weight=w)
    w1 = prob.without_keyframe(0, q1)
    pa, ca = drop_keyframe(p_opt, c_opt, 0)
    pb, cb, tb = WindowOptimizer(w1.layout, w1.linearise, prm, solve=w1.solve).run(pa, ca)
    moved1 = max(np.abs(se3.local(pa[k], pb[k])).max() for k in range(len(pa)))
    q2 = w1.marginalize_keyframe(pa, ca, 0, code_prior_weight=w)
    w2 = w1.without_keyframe(0, q2)
    pc, cc = drop_keyframe(pa, ca, 0)
    pd, cd, td = WindowOptimizer(w2.layout, w2.linearise, prm, solve=w2.solve).run(pc, cc)
    moved2 = max(np.abs(se3.local(pc[k], pd[k])).max() for k in range(len(pc)))
    print(f"LM from the optimum moves the kept poses by {moved1:.2e} (slid once), {moved2:.2e} (twice)")
    assert moved1 <= 1e-3 and moved2 <= 1e-3
    assert tb.energy[-1] <= tb.energy[0] and td.energy[-1] <= td.energy[0]
