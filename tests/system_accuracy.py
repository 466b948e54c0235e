"""Per-entry accuracy of a photometric (or reprojection) normal-equation system against fp64 truth.

The RunStep system mixes columns of very different size: code-code entries of JtJ are 3-4 orders of magnitude below
the pose entries, and the code part of Jtr 1-2 orders below its pose part.  A bar relative to max|H| therefore checks
the code block -- most of what the kernels compute -- only to a few per cent of its own size.  This module states the
error of every entry relative to the error scale of the algorithm the kernels run:

  * the kernels reduce the Gram G = sum_p m_p^T m_p of the reduced row m = [a (6) | code (C) | r], with
    J = [a P0 | a P1 | code] (P0 = d pose10 / d pose0, P1 = d pose10 / d pose1), and expand JtJ = E^T G E,
    E = [[P0, P1, 0], [0, 0, I_C]] (dfk_sfm_finalize.cu).  Any summation of the products m_i m_j in fp32 errs by
    about eps * sum_p |m_pi| |m_pj|, so the scale of JtJ entry (i, j) is  S = |E|^T (sum_p |m_p|^T |m_p|) |E|.
    On the code-code block S is the absolute Gram sum_p |J_pi| |J_pj|.
  * the scale of Jtr entry i is  B_i = sum_p |J_pi r_p|.

assert_system_close() bars (per entry, upper triangle):  |H - H64| <= 5e-5 S,  |Jtr - Jtr64| <= 1e-6 B, the residual to
1e-5 relative and the inliers exactly.  On the synthetic pairs of the suite a correct split-tf32 Gram sits near 2e-7 / 2e-9
of these scales, the reference-like fp32 CPU path (one serial chain per entry) at <= 2.4e-5 / 2e-7 up to 320x240, and
the kernel bugs emulated in tests/test_system_accuracy.py (tf32 without its low part, the low part of code features
24-31 lost, LH^T missing, a 128-pixel tile dropped, the code Jacobian rounded to tf32) at >= 3.6e-4 / 3.2e-6: the bars
sit 4x or more below every one of them.

The same bars apply to systems that reduce plain rows [J | r] with no expansion (E = I): RowGram builds H, Jtr and the
scales S = sum |J|^T |J|, B_i = sum |J_i r| from any row set, se3_reference() does it for the tracker's SE3 step and
depth_reference() for DepthAligner, from the oracle's fp64 per-pixel rows (entry names: SE3_NAMES, CODE_NAMES).
UpdateDepth, a per-pixel decode, is held per pixel to UD_BAR times an error scale derived from its own roundings
(update_depth_scale).  tests/test_tracker_depth_accuracy.py shows which emulated bugs these bars reject.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from deepfactors_b200 import synth
from oracle import oracle as orc

H_BAR = 5e-5
JTR_BAR = 1e-6
RES_BAR = 1e-5


def case_pair(w, h, cs, *, seed=None, code_sigma=0.5):
    """the one-level synthetic pair of a w x h, C = cs case (the seed formula of test_gpu_parity.py)"""
    return synth.make_pair(w, h, cs, 1, seed=w + cs if seed is None else seed, code_sigma=code_sigma)


def pitched_host(a, extra_px):
    """the same values as `a` [H, W(, K)] in a host array whose rows are padded by extra_px pixels"""
    a = np.ascontiguousarray(a, dtype=np.float32)
    buf = np.full((a.shape[0], a.shape[1] + extra_px) + a.shape[2:], np.nan, dtype=np.float32)
    buf[:, :a.shape[1]] = a
    return buf[:, :a.shape[1]]


@dataclass
class Reference:
    """fp64 truth of one RunStep: H (NP x NP), Jtr, residual, inliers, the per-entry scales S and B, the valid mask"""
    H: np.ndarray
    Jtr: np.ndarray
    residual: float
    inliers: int
    S: np.ndarray
    B: np.ndarray
    valid: np.ndarray


def pose_jacobians(pose0, pose1):
    """P0 = d pose10 / d pose0 and P1 = d pose10 / d pose1 (fp64, from the fp32 poses the kernels get)"""
    _, P1, P0 = orc.relative_pose(np.asarray(pose1, np.float32).astype(np.float64),
                                  np.asarray(pose0, np.float32).astype(np.float64))
    return P0, P1


def reference_system(pose0, pose1, cam, img0, img1, dpt0, prx0_jac, grad1, params=None, *,
                     chunk_pixels=1 << 17) -> Reference:
    """Sum the oracle's fp64 per-pixel rows [J | r] in fp64, chunk by chunk of image rows (a 1280x960 level at C = 32
    has 440 MB of rows), and build the scales S and B."""
    H_, W_ = img0.shape
    Cs = prx0_jac.shape[2]
    NP = 12 + Cs
    P0, P1 = pose_jacobians(pose0, pose1)
    P0inv = np.linalg.inv(P0)
    E = np.zeros((6 + Cs, NP))
    E[:6, :6], E[:6, 6:12], E[6:, 12:] = P0, P1, np.eye(Cs)
    G = np.zeros((NP + 1, NP + 1))
    A = np.zeros((6 + Cs, 6 + Cs))
    B = np.zeros(NP)
    valid = np.zeros((H_, W_), dtype=np.float32)
    inliers = 0
    step = max(1, chunk_pixels // W_)
    for y0 in range(0, H_, step):
        X, _, n_ = orc.sfm_pixel_rows(pose0, pose1, cam, img0, img1, dpt0, valid, prx0_jac, grad1, params,
                                       y_begin=y0, y_end=y0 + step)
        X = X[valid[y0:y0 + step].reshape(-1) > 0]
        inliers += n_
        G += X.T @ X
        m = np.abs(np.concatenate([X[:, :6] @ P0inv, X[:, 12:NP]], axis=1))  # |[a | code]|
        A += m.T @ m
        B += np.abs(X[:, :NP] * X[:, NP:]).sum(0)
    Ea = np.abs(E)
    return Reference(G[:NP, :NP], G[:NP, NP].copy(), float(G[NP, NP]), inliers, Ea.T @ A @ Ea, B, valid)


def level_reference(pair, L, params=None, **kw) -> Reference:
    return reference_system(pair.pose0, pair.pose1, L.cam, L.img0, L.img1, L.dpt0, L.prx_jac, L.grad1, params, **kw)


def _dense(JtJ, n):
    JtJ = np.asarray(JtJ, dtype=np.float64)
    if JtJ.ndim == 2:
        return JtJ
    H = np.zeros((n, n))
    H[np.triu_indices(n)] = JtJ
    return H + np.triu(H, 1).T


class RowGram:
    """fp64 Gram of plain rows [J (n) | r], fed chunk by chunk: H = sum J^T J, Jtr = sum J r, residual = sum r^2, and the
    scales S = sum |J|^T |J| and B_i = sum |J_i r| (the rows are what the kernel reduces, so E = I above)."""

    def __init__(self, n):
        self.n = n
        self.G = np.zeros((n + 1, n + 1))
        self.A = np.zeros((n, n))
        self.B = np.zeros(n)

    def add(self, X):
        X = np.asarray(X, dtype=np.float64)
        self.G += X.T @ X
        a = np.abs(X[:, :self.n])
        self.A += a.T @ a
        self.B += (a * np.abs(X[:, self.n:])).sum(0)
        return self

    def reference(self, inliers, valid=None) -> Reference:
        n = self.n
        return Reference(self.G[:n, :n].copy(), self.G[:n, n].copy(), float(self.G[n, n]), int(inliers), self.A.copy(),
                         self.B.copy(), valid)


def se3_reference(se3, cam, img0, img1, dpt0, grad1, huber_delta=0.1, *, valid_f32=True,
                  chunk_pixels=1 << 18) -> Reference:
    """fp64 truth of one SE3Aligner::RunStep from the oracle's per-pixel rows.  valid_f32 (default): the pixel set of
    the fp32 validity chain, which the kernels run -- so the system stays comparable entry by entry at poses where
    fp32 and fp64 disagree on a border pixel (identity-like poses, small levels)."""
    H_, W_ = img0.shape
    g = RowGram(6)
    inliers = 0
    step = max(1, chunk_pixels // W_)
    for y0 in range(0, H_, step):
        X, _, n_ = orc.se3_pixel_rows(se3, cam, img0, img1, dpt0, grad1, huber_delta, valid_f32=valid_f32,
                                      y_begin=y0, y_end=y0 + step)
        g.add(X)
        inliers += n_
    return g.reference(inliers)


def depth_reference(code, target_dpt, prx_orig, prx_jac, avg_dpt=2.0, *, chunk_pixels=1 << 16) -> Reference:
    """fp64 truth of one DepthAligner::RunStep from the oracle's per-pixel rows (every pixel is an inlier)"""
    H_, W_ = target_dpt.shape
    g = RowGram(np.asarray(code).shape[0])
    step = max(1, chunk_pixels // W_)
    for y0 in range(0, H_, step):
        g.add(orc.depth_pixel_rows(code, target_dpt, prx_orig, prx_jac, avg_dpt, y_begin=y0, y_end=y0 + step))
    return g.reference(H_ * W_)


# --------------------------------------------------------------------------------------------- UpdateDepth
UD_BAR = 1e-6


def update_depth_scale(code, prx_orig, prx_jac, avg_dpt, *, chunk_pixels=1 << 16):
    """per-pixel error scale of the fp32 decode dpt = avg / (prx_orig + j . c) - avg, from its own roundings:

        S_px = (avg / prx^2) (|prx_orig| + sum_k |j_k c_k|) + avg / |prx|

    The first term carries the rounding of the dot product and of the add (each at most eps times the sum of the
    magnitudes that went into it) through d dpt / d prx = -avg / prx^2; the second is the division and the final
    subtraction (|dpt| <= avg / |prx| wherever 0 < prx < 1, the range a proximity lives in).

    UpdateDepth is held to |dpt - dpt64| <= UD_BAR S_px = 1e-6 S_px, about 17 eps (eps = 2^-24).  Worst cases: a
    serial fp32 chain over C terms errs by at most C eps of sum |j c| but, with the rounding errors independent and the
    partial sums a random walk, typically by about 0.5 eps of it, and the worst of 1.2 M pixels by a few eps; a tree
    (the vectorised kernel's lane split and shuffle sum) errs by log2(C) eps at most.  The add, division and
    subtraction are one rounding each.  So a correct decode sits at a few eps, the bar leaves room for the serial
    C = 256 generic kernel, and any lost term (one float4 lane dropped: 4 of C terms, about 3 % of sum |j c| at
    C = 128) or a tf32-rounded operand (2^-11 relative per term, 4e-4 of sum |j c| / sqrt(C)) is far above it."""
    code = np.asarray(code, dtype=np.float64)
    H_, W_ = prx_orig.shape
    ac = np.abs(code)
    s = np.empty((H_, W_))
    prx = np.empty((H_, W_))
    step = max(1, chunk_pixels // W_)
    for y0 in range(0, H_, step):
        J = np.asarray(prx_jac[y0:y0 + step], dtype=np.float64)
        po = np.asarray(prx_orig[y0:y0 + step], dtype=np.float64)
        prx[y0:y0 + step] = po + J @ code
        s[y0:y0 + step] = np.abs(po) + np.abs(J) @ ac
    avg = float(avg_dpt)
    return avg / prx ** 2 * s + avg / np.abs(prx)


def update_depth_errors(got, ref64, scale):
    """worst per-pixel ratio |got - ref64| / scale and where it is"""
    r = np.abs(np.asarray(got, np.float64) - ref64) / scale
    k = int(np.argmax(r))
    return float(r.reshape(-1)[k]), np.unravel_index(k, r.shape)


# --------------------------------------------------------------------------------------------- entry names
def _name(i):
    if i >= 12:
        return f"code {i - 12}"
    return ("t0", "w0", "t1", "w1")[i // 3] + f" {i % 3}"


def _block(i):
    return "code" if i >= 12 else ("t0", "w0", "t1", "w1")[i // 3]


SFM_NAMES = (_name, _block)
SE3_NAMES = (lambda i: ("t", "w")[i // 3] + f" {i % 3}", lambda i: ("t", "w")[i // 3])
CODE_NAMES = (lambda i: f"code {i}", lambda i: "code")


def _ratio(err, scale):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(scale > 0, err / np.where(scale > 0, scale, 1.0), np.where(err > 0, np.inf, 0.0))
    return r


def system_errors(got, ref, S, B):
    """worst per-entry ratios of a result (JtJ packed or dense, Jtr, residual) against the fp64 reference:
    dict(h=..., h_at=(i, j), jtr=..., jtr_at=i, res=relative residual error)"""
    n = ref.Jtr.shape[0]
    Hg = _dense(got.JtJ if hasattr(got, "JtJ") else got.H, n)
    iu = np.triu_indices(n)
    rh = _ratio(np.abs(Hg - ref.H)[iu], S[iu])
    k = int(np.argmax(rh))
    rj = _ratio(np.abs(np.asarray(got.Jtr, np.float64) - ref.Jtr), B)
    q = int(np.argmax(rj))
    rres = abs(float(got.residual) - ref.residual) / ref.residual if ref.residual > 0 else (
        0.0 if float(got.residual) == 0.0 else np.inf)
    return dict(h=float(rh[k]), h_at=(int(iu[0][k]), int(iu[1][k])), jtr=float(rj[q]), jtr_at=q, res=rres, Hg=Hg)


def assert_system_close(got, ref, S, B, what, *, h_bar=H_BAR, jtr_bar=JTR_BAR, res_bar=RES_BAR, names=SFM_NAMES):
    """inliers exactly; max_ij |H - H64|_ij / S_ij <= h_bar (upper triangle); max_i |Jtr - Jtr64|_i / B_i <= jtr_bar;
    residual to res_bar relative.  The message names the worst entry, its block, value and scale (names: SFM_NAMES for
    the [pose0 | pose1 | code] system, SE3_NAMES for the tracker's [t | w], CODE_NAMES for DepthAligner's code-only
    one).  Returns the errors."""
    assert int(got.inliers) == int(ref.inliers), f"{what}: inliers {got.inliers} != {ref.inliers}"
    e = system_errors(got, ref, S, B)
    i, j = e["h_at"]
    q = e["jtr_at"]
    _name, _block = names
    msg = (f"{what}: worst H entry [{_block(i)}/{_block(j)}] ({_name(i)}, {_name(j)}): got {e['Hg'][i, j]:.9e} "
           f"ref {ref.H[i, j]:.9e} scale S {S[i, j]:.3e} -> {e['h']:.2e} (bar {h_bar:.0e}); "
           f"worst Jtr entry [{_block(q)}] ({_name(q)}): got {float(got.Jtr[q]):.9e} ref {ref.Jtr[q]:.9e} "
           f"scale B {B[q]:.3e} -> {e['jtr']:.2e} (bar {jtr_bar:.0e}); residual {e['res']:.2e} (bar {res_bar:.0e})")
    print(msg)
    assert e["h"] <= h_bar, msg
    assert e["jtr"] <= jtr_bar, msg
    assert e["res"] <= res_bar, msg
    return e
