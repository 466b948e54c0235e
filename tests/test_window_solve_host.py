"""Host logic of WindowOptimizer's injected `solve` (the hook SfmWindowProblem.solve fills with dfk_window_solve), without
a GPU: a numpy solve that wraps to_dense + damped_solve must reproduce the default path's trace exactly, f comes from the
buffer's scalar slot, and a solve that returns None is a rejected step."""
import numpy as np

from deepfactors_b200 import se3
from deepfactors_b200.factors import WindowBlocks
from deepfactors_b200.window_opt import LMParams, WindowOptimizer, damped_solve


def _problem(cs=3, seed=1):
    """a nonlinear least-squares window in the block-sparse layout: three keyframes, three pairs; residuals mix pose
    translations and codes through sin() so that LM takes rejected steps too"""
    pairs = [(0, 1), (1, 2), (2, 0)]
    wb = WindowBlocks(3, cs, pairs)
    rng = np.random.default_rng(seed)
    M = [rng.standard_normal((6, 12 + cs)) for _ in pairs]
    evals = []

    def linearise(poses, codes, todo):
        evals.append(list(todo))
        NP = 12 + cs
        JtJ, Jtr, res = [], [], []
        for p, (k0, k1) in enumerate(pairs):
            x = np.concatenate([poses[k0][4:7], [0, 0, 0], poses[k1][4:7], [0, 0, 0], codes[k0]])
            r = np.sin(3.0 * (M[p] @ x)) + 0.1 * (p + 1)
            J = (3.0 * np.cos(3.0 * (M[p] @ x)))[:, None] * M[p]
            J[:, 3:6] = 0.0
            J[:, 9:12] = 0.0
            JtJ.append(J.T @ J + 1e-3 * np.eye(NP))
            Jtr.append(J.T @ r)
            res.append(float(r @ r))
        buf = wb.pack(list(range(len(pairs))), np.array(JtJ), np.array(Jtr), res, [1] * len(pairs), [(0, 0)] * len(pairs))
        return buf, None

    poses = np.tile(se3.identity(np.float64), (3, 1))
    poses[1][4:7] = [0.3, -0.2, 0.1]
    poses[2][4:7] = [-0.1, 0.25, 0.2]
    codes = rng.standard_normal((3, cs)) * 0.2
    return wb, linearise, poses, codes, evals


def _numpy_solve(wb):
    def solve(buf, lam, fixed, w, codes):
        H, g, _, _ = wb.to_dense(buf)
        B = wb.B
        if w > 0:
            for k in range(wb.num_keyframes):
                sl = slice(k * B + 6, (k + 1) * B)
                H[sl, sl] += w * np.eye(B - 6)
                g[sl] -= w * codes[k]
        return damped_solve(H, g, lam, fixed)
    return solve


def test_injected_solve_reproduces_the_default_trace_exactly():
    for w in (0.0, 1e-2):
        wb, lin, poses, codes, _ = _problem()
        prm = LMParams(iterations=15, lambda_init=1e-2, code_prior_weight=w)
        p0, c0, t0 = WindowOptimizer(wb, lin, prm).run(poses, codes)
        p1, c1, t1 = WindowOptimizer(wb, lin, prm, solve=_numpy_solve(wb)).run(poses, codes)
        assert t1.energy == t0.energy and t1.lam == t0.lam and t1.accepted == t0.accepted
        assert t1.factors_relinearised == t0.factors_relinearised
        assert np.array_equal(p1, p0) and np.array_equal(c1, c0)
        assert any(t0.accepted) and len(t0.energy) > 2


def test_energy_from_the_buffer_is_to_dense_f_plus_the_code_prior():
    wb, lin, poses, codes, _ = _problem()
    buf, _ = lin(poses, codes, [0, 1, 2])
    for w in (0.0, 0.5):
        opt = WindowOptimizer(wb, lin, LMParams(code_prior_weight=w))
        assert opt._energy(buf, codes) == wb.to_dense(buf)[2] + 0.5 * w * float((codes ** 2).sum())
    assert WindowOptimizer(wb, lin)._energy(buf, codes) == wb.to_dense(buf)[2]


def test_solve_returning_none_rejects_the_step_without_relinearising():
    wb, lin, poses, codes, evals = _problem()
    calls = []

    def solve(buf, lam, fixed, w, c):
        calls.append(lam)
        return None if len(calls) <= 2 else _numpy_solve(wb)(buf, lam, fixed, w, c)

    prm = LMParams(iterations=4, lambda_init=1e-3, lambda_up=10.0)
    p, c, tr = WindowOptimizer(wb, lin, prm, solve=solve).run(poses, codes)
    assert calls[:3] == [1e-3, 1e-2, 1e-1]
    assert tr.accepted[:2] == [False, False] and tr.lam[:3] == [1e-3, 1e-2, 1e-1]
    assert len(evals) == 1 + (len(calls) - 2)     # the initial linearisation, then one per solved step only
    assert tr.factors_relinearised[0] == 3


def test_solve_returning_none_stops_past_lambda_max():
    wb, lin, poses, codes, evals = _problem()
    prm = LMParams(iterations=50, lambda_init=1e-3, lambda_up=10.0, lambda_max=1.0)
    p, c, tr = WindowOptimizer(wb, lin, prm, solve=lambda *a: None).run(poses, codes)
    assert len(evals) == 1 and not any(tr.accepted) and len(tr.accepted) == 4
    assert np.array_equal(p, poses) and np.array_equal(c, codes) and tr.energy == tr.energy[:1]
