"""dfk_window_solve (aligners.WindowSolver): the damped block-sparse fp64 Cholesky of a window buffer against the dense
system WindowOptimizer solves on torch (WindowBlocks.to_dense + the code prior + damped_solve), on random positive
semi-definite records packed with WindowBlocks.pack."""
import ctypes as C

import numpy as np
import pytest

from deepfactors_b200 import se3, synth
from deepfactors_b200.factors import WindowBlocks

CODE_SIZES = [8, 16, 32, 64, 128]


def structure(name, K, rng):
    """(pairs, geometric links) of a test window; every keyframe is k0 of a pair, so every code block is covered"""
    if name == "chain":
        return [(k, k + 1) for k in range(K - 1)] + [(K - 1, K - 2)], []
    if name == "ring":  # the wrap-around pair fills the last row
        return [(k, (k + 1) % K) for k in range(K)], []
    if name == "dense":
        pairs = [(k, (k + 1) % K) for k in range(K)]
        pairs += [tuple(int(v) for v in rng.choice(K, 2, replace=False)) for _ in range(2 * K)]
        return pairs, []
    if name == "both_directions":
        return [(k, (k + 2) % K) for k in range(K)] + [((k + 2) % K, k) for k in range(K)], []
    if name == "duplicates":
        return [(k, (k + 1) % K) for k in range(K)] + [(0, 1), (0, 1), (3, 1)], []
    if name == "self_pair":
        return [(k, (k + 1) % K) for k in range(K)] + [(2, 2), (0, 0)], []
    if name == "geometric":
        return [(k, k + 1) for k in range(K - 1)] + [(K - 1, 0)], [(0, 2), (3, 1), (K - 1, 1)]
    raise ValueError(name)


STRUCTURES = ["chain", "ring", "dense", "both_directions", "duplicates", "self_pair", "geometric"]


def random_buffer(layout: WindowBlocks, rng, scale=1.0):
    """the packed buffer of random Gram records (2 x as many rows as variables: positive definite blocks)"""
    C_ = layout.code_size
    NP, NG = 12 + C_, 12 + 2 * C_
    n = len(layout.pairs)
    A = rng.standard_normal((n, 2 * NP, NP + 1)).astype(np.float32) * np.float32(scale)
    JtJ = np.einsum("nri,nrj->nij", A[..., :NP], A[..., :NP])
    Jtr = np.einsum("nri,nr->ni", A[..., :NP], A[..., NP])
    geo = None
    if layout.geometric:
        L = len(layout.geometric)
        G = rng.standard_normal((L, 2 * NG, NG + 1)).astype(np.float32) * np.float32(scale)
        geo = (np.einsum("nri,nrj->nij", G[..., :NG], G[..., :NG]), np.einsum("nri,nr->ni", G[..., :NG], G[..., NG]),
               np.ones(L, dtype=np.float32))
    return layout.pack(list(range(n)), JtJ, Jtr, np.ones(n, np.float32), np.zeros(n), [(0, 0)] * n, geo=geo)


def damped_system(layout, buf, lam, fixed, w, codes):
    """(A, b, keep) of the damped system over the kept variables, numpy fp64, as WindowOptimizer builds it"""
    H, g, _, _ = layout.to_dense(buf)
    B = layout.B
    if w > 0:
        for k in range(layout.num_keyframes):
            sl = slice(k * B + 6, (k + 1) * B)
            H[sl, sl] += w * np.eye(B - 6)
            g[sl] -= w * codes[k]
    keep = np.ones(H.shape[0], dtype=bool)
    keep[list(fixed)] = False
    A = H[np.ix_(keep, keep)]
    d = np.diag(A).copy()
    A = A + np.diag(lam * d + 1e-12 * np.abs(d).max())
    return A, g[keep], keep


def symbolic_tiles(K, pairs, links):
    below = [set() for _ in range(K)]
    for a, b in list(pairs) + list(links):
        if a != b:
            below[min(a, b)].add(max(a, b))
    for j in range(K):
        rows = sorted(below[j])
        for x in range(len(rows)):
            for y in range(x):
                below[rows[y]].add(rows[x])
    return K + sum(len(s) for s in below)


def make_window(al, K, pairs, links):
    from deepfactors_b200.aligners import Window
    return Window(al, K, pairs, list(range(len(pairs))), [(0, 0)] * len(pairs), links)


@pytest.mark.gpu
@pytest.mark.parametrize("cs", CODE_SIZES)
@pytest.mark.parametrize("name", STRUCTURES)
def test_window_solve_matches_dense_damped_solve(cs, name):
    import torch
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    from deepfactors_b200.window_opt import damped_solve
    rng = np.random.default_rng(100 + cs + STRUCTURES.index(name))
    K = 6
    pairs, links = structure(name, K, rng)
    al = SfmAligner(cs)
    win = make_window(al, K, pairs, links)
    buf_h = random_buffer(win.layout, rng)
    buf = torch.from_numpy(buf_h).cuda()
    B = win.layout.B
    codes = rng.standard_normal((K, cs)) * 0.3
    worst = [0.0, 0.0]
    for fixed in ((), tuple(range(6))):
        sol = WindowSolver(win, fixed)
        assert sol.tiles == symbolic_tiles(K, pairs, links)
        if name == "chain":
            assert sol.tiles == 2 * K - 1
        for lam in (0.0, 1e-4, 1e3):
            for w in (0.0, 1e-2):
                dx, info = sol.solve(buf, lam, w, codes)
                dxh = dx.cpu().numpy()
                assert int(info.item()) == 0
                A, b, keep = damped_system(win.layout, buf_h, lam, fixed, w, codes)
                x = dxh[keep]
                berr = np.abs(A @ x - b).max() / (np.abs(A).sum(1).max() * np.abs(x).max() + np.abs(b).max())
                assert berr <= 1e-12, (fixed, lam, w, berr)
                assert np.all(dxh[list(fixed)] == 0.0)
                # against damped_solve on torch (the system is built with cond <= 1e6)
                H, g, _, _ = win.layout.to_dense(buf)
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
                # deterministic: a second solve is bit for bit the first
                dx2, _ = sol.solve(buf, lam, w, codes)
                assert torch.equal(dx, dx2)
    print(f"C={cs} {name}: tiles {sol.tiles} worst backward error {worst[0]:.2e} worst |dx - torch|/|dx| {worst[1]:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("cs", [8, 128])
def test_window_solve_two_handles_bitwise_equal(cs):
    import torch
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    rng = np.random.default_rng(7)
    K = 7
    pairs, links = structure("dense", K, rng)
    outs = []
    for _ in range(2):
        al = SfmAligner(cs)
        win = make_window(al, K, pairs, links)
        buf = torch.from_numpy(random_buffer(win.layout, np.random.default_rng(8))).cuda()
        dx, info = WindowSolver(win, range(6)).solve(buf, 1e-3, 1e-2, np.ones((K, cs)))
        outs.append(dx.clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.gpu
def test_window_solve_reports_not_positive_definite_then_recovers():
    import torch
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    from deepfactors_b200.window_opt import damped_solve
    cs, K = 16, 5
    rng = np.random.default_rng(11)
    pairs, links = structure("ring", K, rng)
    al = SfmAligner(cs)
    win = make_window(al, K, pairs, links)
    good = random_buffer(win.layout, rng)
    bad = good.copy()
    B = win.layout.B
    D = bad[:K * B * B].reshape(K, B, B)
    D[2, 6:, 6:] = 0.0   # keyframe 2's code block zero, its couplings not: indefinite at lambda = 0
    sol = WindowSolver(win, range(6))
    dx = torch.full((K * B,), 7.0, dtype=torch.float64, device="cuda")
    _, info = sol.solve(torch.from_numpy(bad).cuda(), 0.0, dx=dx)
    assert int(info.item()) != 0
    assert int(info.item()) - 1 >= 2 * B
    assert torch.all(dx == 0)
    _, info = sol.solve(torch.from_numpy(good).cuda(), 0.0, dx=dx)
    assert int(info.item()) == 0
    H, g, _, _ = win.layout.to_dense(torch.from_numpy(good).cuda())
    ref = damped_solve(H, g, 0.0, range(6))
    assert (dx - ref).abs().max() <= 1e-9 * ref.abs().max()


@pytest.mark.gpu
def test_window_solve_rejects_bad_arguments_and_writes_nothing():
    import torch
    from deepfactors_b200 import _lib
    from deepfactors_b200.aligners import SfmAligner, WindowSolver
    cs, K = 8, 4
    rng = np.random.default_rng(3)
    pairs, links = structure("chain", K, rng)
    al = SfmAligner(cs)
    win = make_window(al, K, pairs, links)
    B = win.layout.B
    buf = torch.from_numpy(random_buffer(win.layout, rng)).cuda()
    for fixed in ((0, 0), (-1,), (K * B,)):
        with pytest.raises(_lib.DfkError):
            WindowSolver(win, fixed)
    sol = WindowSolver(win, range(6))
    dx = torch.full((K * B,), 5.0, dtype=torch.float64, device="cuda")
    info = torch.full((1,), 9, dtype=torch.int32, device="cuda")
    lib, h = _lib.lib(), al.handle

    def raw(lam, w, codes, window=buf, d=dx, i=info, s=None):
        prm = _lib.DfkWindowSolveParams(lam, w)
        return lib.dfk_window_solve(h, s or sol.s, C.c_void_p(window.data_ptr()) if window is not None else None,
                                    C.byref(prm), codes, C.c_void_p(d.data_ptr()) if d is not None else None,
                                    C.c_void_p(i.data_ptr()) if i is not None else None)

    cp = np.zeros(K * cs).ctypes.data_as(C.POINTER(C.c_double))
    for args in ((-1.0, 0.0, None), (float("nan"), 0.0, None), (float("inf"), 0.0, None), (0.0, -1e-3, cp),
                 (0.0, float("nan"), cp), (0.0, 1e-2, None)):
        assert raw(*args) == _lib.DFK_ERR_INVALID_ARG, args
        assert lib.dfk_last_error(h)
    assert raw(0.0, 0.0, None, window=None) == _lib.DFK_ERR_INVALID_ARG
    assert raw(0.0, 0.0, None, d=None) == _lib.DFK_ERR_INVALID_ARG
    assert raw(0.0, 0.0, None, i=None) == _lib.DFK_ERR_INVALID_ARG
    assert lib.dfk_window_solver_create(h, None, 0, None, C.byref(C.c_void_p())) == _lib.DFK_ERR_INVALID_ARG
    torch.cuda.synchronize()
    assert torch.all(dx == 5.0) and int(info.item()) == 9
    # the Python wrapper checks the buffers the way Window.assemble does
    for bad in (buf[:-1], buf.double(), buf.cpu()):
        with pytest.raises(ValueError):
            sol.solve(bad, 0.0)
    with pytest.raises(ValueError):
        sol.solve(buf, 0.0, 1e-2, None)
    with pytest.raises(_lib.DfkError):
        sol.solve(buf, -1.0)
    torch.cuda.synchronize()
    assert torch.all(dx == 5.0)


@pytest.mark.gpu
def test_window_lm_with_device_solve_takes_the_torch_path_steps():
    """The 3-keyframe LM window of test_window_gauss_newton_loop_on_device_recovers_perturbed_poses, once with the torch
    solve and once with SfmWindowProblem.solve: same accept / reject sequence, energies and poses within 1e-6."""
    import torch
    from deepfactors_b200.aligners import SfmAligner
    from deepfactors_b200.window_opt import LMParams, SfmWindowProblem, WindowOptimizer
    cs, levels = 8, 2
    base = synth.make_pair(160, 120, cs, levels, seed=5)
    cams = [L.cam for L in base.levels]
    al = SfmAligner(cs)
    keyframes = []
    for k in range(3):
        lv = []
        for L in base.levels:
            up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
            img = up(L.img0)
            lv.append(dict(img=img, grad=up(synth.sobel_np(L.img0)), prx_orig=up(L.prx_orig), prx_jac=up(L.prx_jac),
                           dpt=torch.zeros_like(img), valid=torch.zeros_like(img)))
        keyframes.append(lv)
    pairs = [(0, 1), (1, 2), (2, 0), (1, 0), (2, 1)]
    prob = SfmWindowProblem(al, cams, keyframes, pairs)
    poses = np.stack([se3.identity(np.float64),
                      se3.make_pose([0.004, -0.003, 0.002], [0.015, -0.01, 0.008], np.float64),
                      se3.make_pose([-0.003, 0.002, 0.004], [-0.01, 0.012, -0.006], np.float64)])
    codes = np.zeros((3, cs))
    prm = LMParams(iterations=12, lambda_init=1e-3, code_prior_weight=1e-2)
    p0, c0, t0 = WindowOptimizer(prob.layout, prob.linearise, prm).run(poses, codes)
    p1, c1, t1 = WindowOptimizer(prob.layout, prob.linearise, prm, solve=prob.solve).run(poses, codes)
    assert t1.accepted == t0.accepted
    assert t1.lam == t0.lam
    assert t1.factors_relinearised == t0.factors_relinearised
    assert np.allclose(t1.energy, t0.energy, rtol=1e-6, atol=0)
    assert np.abs(p1 - p0).max() <= 1e-6
    assert t1.energy[-1] < t1.energy[0] / 20.0
    assert np.array_equal(p1[0], poses[0])


@pytest.mark.gpu
def test_window_solve_cpp_binary():
    """dfk_window_solve from C++ against a host Cholesky of the same df::WindowSystem<CS>"""
    import os
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "cpp", "window_solve_test")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(out.stdout)
    assert out.returncode == 0 and "WINDOW_SOLVE_TEST_OK" in out.stdout, out.stdout + out.stderr
