"""GPU-driven Gauss-Newton / Levenberg-Marquardt over a keyframe window.

The reference runs this loop on the host, one factor at a time: ISAM2::update (sources/core/mapping/mapper.cpp:518-519)
calls PhotometricFactor::linearize for every relinearised factor (sources/core/gtsam/photometric_factor.cpp:84-181),
which consults its linearisation cache (:296-328, keyed on pose0 / pose1 / code0 within 1e-6), re-decodes the keyframe's
depth from its code (UpdateDepthMaps, :229,331-341), runs SfmAligner::RunStep synchronously (:267-274), rescales the
residual (:275-282) and slices the 44x44 system into HessianFactor blocks (:126-161); the solver adds the factors up and
solves.  Here every heavy step of one iteration is ONE device operation over the whole window:

    linearise   one batched RunStep launch over all (pair, level) factors whose variables moved, with the depth decode
                fused in (the code of keyframe k0 rides in the work item)               dfk_sfm_run_step_batch
    assemble    block-sparse normal equations of the window, on the device              dfk_window_assemble_geometric
                (+ one all-reduce across ranks when the pairs are sharded)
    solve       damped dense solve on the device (dense_solve: Cholesky, float64)       torch.linalg
                or, with WindowOptimizer(solve=...), the damped block-sparse Cholesky      dfk_window_solve
                straight from the window buffer (SfmWindowProblem.solve)
    (links)     one batched launch over the stale reprojection links (global loop closures, use_reprojection),
                straight into normal-equation records                                  dfk_reprojection_linearize_batch
                and one over the stale sparse geometric links (use_geometric)          dfk_sparse_geometric_linearize_batch
    retract     pose: t += dt, R = exp(w) R (gtsam_traits.h:48-58); code += dc           (tiny, host)
    accept      Levenberg-Marquardt on the energy f: rescaled photometric residuals + b^T b of the links (what the
                factors' error() return)

The host side (cache, retraction, damping schedule) is plain Python / numpy; nothing here needs GTSAM.
"""
from __future__ import annotations

import functools
from dataclasses import dataclass, field
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np

from . import se3
from .factors import WindowBlocks


@dataclass
class LMParams:
    iterations: int = 10
    lambda_init: float = 1e-4
    lambda_up: float = 10.0
    lambda_down: float = 0.1
    lambda_max: float = 1e6
    fix_first_pose: bool = True       # gauge: the window's first keyframe keeps its pose (the reference adds a pose prior)
    code_prior_weight: float = 0.0    # zero-code prior: adds w * I to every code block and -w * code to its gradient
    cache_eps: float = 1e-6           # photometric_factor.cpp:302-316


@dataclass
class LMTrace:
    energy: List[float] = field(default_factory=list)       # accepted energies, energy[0] = initial
    lam: List[float] = field(default_factory=list)
    accepted: List[bool] = field(default_factory=list)
    factors_relinearised: List[int] = field(default_factory=list)  # per linearisation: pairs that were re-evaluated


def damped_solve(H, g, lam: float, fixed: Sequence[int] = ()):
    """(H + lam * diag(H)) dx = g with the variables in `fixed` held (rows / columns removed).  H, g: torch (any device,
    float64) or numpy.  Returns dx of full dimension (zeros at the fixed variables)."""
    if hasattr(H, "detach"):
        import torch
        n = H.shape[0]
        keep = torch.ones(n, dtype=torch.bool, device=H.device)
        if len(fixed):
            keep[torch.as_tensor(list(fixed), device=H.device)] = False
        idx = torch.nonzero(keep).squeeze(1)
        Hk = H.index_select(0, idx).index_select(1, idx)
        d = torch.diagonal(Hk).clone()
        Hk = Hk + torch.diag(lam * d + 1e-12 * d.abs().max())
        gk = g.index_select(0, idx)
        L, info = torch.linalg.cholesky_ex(Hk)
        if int(info.item()) != 0:  # not positive definite at this damping: least squares keeps the loop alive
            sol = torch.linalg.lstsq(Hk, gk.unsqueeze(1)).solution.squeeze(1)
        else:
            sol = torch.cholesky_solve(gk.unsqueeze(1), L).squeeze(1)
        dx = torch.zeros(n, dtype=H.dtype, device=H.device)
        dx[idx] = sol
        return dx
    Hn = np.asarray(H, dtype=np.float64)
    gn = np.asarray(g, dtype=np.float64)
    n = Hn.shape[0]
    keep = np.ones(n, dtype=bool)
    keep[list(fixed)] = False
    Hk = Hn[np.ix_(keep, keep)]
    d = np.diag(Hk).copy()
    Hk = Hk + np.diag(lam * d + 1e-12 * np.abs(d).max())
    dx = np.zeros(n)
    dx[keep] = np.linalg.lstsq(Hk, gn[keep], rcond=None)[0]
    return dx


def dense_solve(layout: WindowBlocks, buf, lam: float, fixed: Sequence[int], code_prior_weight: float, codes):
    """WindowOptimizer's default solve: to_dense of the buffer plus the zero-code prior (w * I on every code block,
    -w * code on its gradient), then damped_solve.  buf: numpy, or torch on any device (H is built and solved there).
    Returns dx (numpy float64)."""
    H, g, _, _ = layout.to_dense(buf)
    w = code_prior_weight
    if w > 0:
        B = layout.B
        for k in range(layout.num_keyframes):
            sl = slice(k * B + 6, (k + 1) * B)
            if hasattr(H, "detach"):
                import torch
                H[sl, sl] += w * torch.eye(B - 6, dtype=H.dtype, device=H.device)
                g[sl] -= w * torch.as_tensor(codes[k], dtype=g.dtype, device=g.device)
            else:
                H[sl, sl] += w * np.eye(B - 6)
                g[sl] -= w * codes[k]
    dx = damped_solve(H, g, lam, fixed)
    return dx.detach().cpu().numpy() if hasattr(dx, "detach") else dx


class LinearisationCache:
    """photometric_factor.cpp:296-328 GetJacobiansIfNeeded for a whole window: a pair's factors are re-evaluated only when
    pose0, pose1 or code0 moved by more than eps since the evaluation whose records are still in the record buffer.
    Geometric links (k0, k1) follow the pairs (link j is index len(pairs) + j); a link also depends on code1, so it is
    stale when pose0, pose1, code0 or code1 moved."""

    def __init__(self, pairs: Sequence[Tuple[int, int]], eps: float = 1e-6, geometric: Sequence[Tuple[int, int]] = ()):
        self.pairs = list(pairs)
        self.geometric = [tuple(p) for p in geometric]
        self.eps = eps
        self.invalidate()

    def _keys(self):
        return [(k0, k1, False) for k0, k1 in self.pairs] + [(k0, k1, True) for k0, k1 in self.geometric]

    def stale(self, poses: np.ndarray, codes: np.ndarray) -> List[int]:
        out = []
        for p, (k0, k1, geo) in enumerate(self._keys()):
            at = self._at[p]
            if at is None or np.abs(at[0] - poses[k0]).max() > self.eps or np.abs(at[1] - poses[k1]).max() > self.eps or \
                    np.abs(at[2] - codes[k0]).max() > self.eps or (geo and np.abs(at[3] - codes[k1]).max() > self.eps):
                out.append(p)
        return out

    def store(self, done: Sequence[int], poses: np.ndarray, codes: np.ndarray):
        keys = self._keys()
        for p in done:
            k0, k1, _ = keys[p]
            # (pose0, pose1, code0, code1) the stored records were evaluated at
            self._at[p] = (poses[k0].copy(), poses[k1].copy(), codes[k0].copy(), codes[k1].copy())

    def invalidate(self):
        self._at = [None] * (len(self.pairs) + len(self.geometric))


def apply_update(poses: np.ndarray, codes: np.ndarray, dx: np.ndarray, code_size: int):
    """variables [pose_k (6: t, w) | code_k (C)] per keyframe; pose retraction of gtsam_traits.h:48-58"""
    B = 6 + code_size
    new_p, new_c = poses.copy(), codes.copy()
    for k in range(poses.shape[0]):
        d = dx[k * B:(k + 1) * B]
        new_p[k] = se3.retract(poses[k].astype(np.float64), d[:6], np.float64)
        new_c[k] = codes[k] + d[6:]
    return new_p, new_c


class WindowOptimizer:
    """Levenberg-Marquardt over the poses and codes of a keyframe window.

    `linearise(poses, codes, pairs_to_eval) -> (window_buffer, f)` is the device pipeline (see SfmWindowProblem below for
    the one built on SfmAligner / Window); injected so that the host logic is testable without a GPU.  It must return a
    buffer that its next call does not overwrite: the loop keeps the accepted point's buffer across a rejected candidate.

    `solve(buf, lam, fixed, code_prior_weight, codes) -> dx (numpy float64) | None` solves the damped system of a buffer;
    None (not positive definite) counts as a rejected step.  The default is dense_solve; SfmWindowProblem.solve is the
    block-sparse one on the device.  f is the buffer's scalar slot plus the host prior term."""

    def __init__(self, layout: WindowBlocks, linearise: Callable, params: Optional[LMParams] = None,
                 solve: Optional[Callable] = None):
        self.layout = layout
        self.linearise = linearise
        self.params = params or LMParams()
        self.solve = solve or functools.partial(dense_solve, layout)
        self.cache = LinearisationCache(layout.pairs, self.params.cache_eps, layout.geometric)

    def _energy(self, buf, codes) -> float:
        """f: the buffer's scalar slot (what to_dense returns) plus the prior term"""
        f = float(buf[self.layout.offsets()[2]])
        w = self.params.code_prior_weight
        if w > 0:
            f += 0.5 * w * float((codes ** 2).sum())
        return f

    def _evaluate(self, poses, codes, trace: LMTrace):
        todo = self.cache.stale(poses, codes)
        buf, _ = self.linearise(poses, codes, todo)
        self.cache.store(todo, poses, codes)
        trace.factors_relinearised.append(len(todo))
        return buf

    def run(self, poses, codes) -> Tuple[np.ndarray, np.ndarray, LMTrace]:
        prm = self.params
        poses = np.asarray(poses, dtype=np.float64).copy()
        codes = np.asarray(codes, dtype=np.float64).copy()
        trace = LMTrace()
        fixed = list(range(6)) if prm.fix_first_pose else []
        lam = prm.lambda_init
        buf = self._evaluate(poses, codes, trace)
        f = self._energy(buf, codes)
        trace.energy.append(f)
        for _ in range(prm.iterations):
            dx = self.solve(buf, lam, fixed, prm.code_prior_weight, codes)
            trace.lam.append(lam)
            ok = False
            if dx is not None:  # None: not positive definite at this damping, a rejected step with nothing re-linearised
                cand_p, cand_c = apply_update(poses, codes, np.asarray(dx, dtype=np.float64), self.layout.code_size)
                cbuf = self._evaluate(cand_p, cand_c, trace)
                cf = self._energy(cbuf, cand_c)
                ok = bool(np.isfinite(cf) and cf < f)
            trace.accepted.append(ok)
            if ok:
                poses, codes, buf, f = cand_p, cand_c, cbuf, cf
                trace.energy.append(f)
                lam = max(lam * prm.lambda_down, 1e-12)
            else:
                # buf and f of the accepted point are still at hand; the record buffer (and with it the cache) now
                # describes the rejected candidate, which the next candidate is compared against
                lam = lam * prm.lambda_up
                if lam > prm.lambda_max:
                    break
        return poses, codes, trace


@dataclass
class ReprojectionLink:
    """A reprojection factor between keyframes k0 -> k1 (ReprojectionFactor, reprojection_factor.cpp): matched keypoints
    query_xy [M, 2] in k0 and train_xy [M, 2] in k1 (host), Cauchy delta and sigma.  A global loop closure is one link
    each way with sigma = loop_sigma (mapper.cpp:367-376); use_reprojection adds them with rep_huber / rep_sigma
    (mapper.cpp:314-325)."""
    k0: int
    k1: int
    query_xy: np.ndarray
    train_xy: np.ndarray
    cauchy_delta: float
    sigma: float


@dataclass
class GeometricLink:
    """A sparse geometric factor between keyframes k0 -> k1 (SparseGeometricFactor, sparse_geometric_factor.cpp): the
    sampled pixels points_xy [M, 2] of k0 (host ints) and the Huber delta.  use_geometric adds one per new keyframe
    connection and per enqueued link (mapper.cpp:328-337, 379-388)."""
    k0: int
    k1: int
    points_xy: np.ndarray
    huber_delta: float


@dataclass
class _FactorKind:
    """One kind of factor of a SfmWindowProblem.  Factor j joins keyframes ends[j], is index first + j of linearise's
    `todo` and owns rows [j * rows, (j + 1) * rows) of `records`.  items(prob, j, kf0, kf1, pose0, pose1, code0, code1)
    are factor j's batch items (float32 poses and codes); batch(aligner, items, records=None) linearises items in one
    launch, into `records` when given."""
    ends: List[Tuple[int, int]]
    first: int
    records: object
    rows: int
    items: Callable
    batch: Callable


def _photometric_items(prob, p, a, b, pose0, pose1, code0, code1):
    """one RunStep work item per level, the depth decode of keyframe k0 fused in"""
    return [dict(pose0=pose0, pose1=pose1, cam=prob.cams[l], img0=a[l]["img"], img1=b[l]["img"], dpt0=a[l]["dpt"],
                 valid0=a[l]["valid"], prx0_jac=a[l]["prx_jac"], grad1=b[l]["grad"], prx_orig=a[l]["prx_orig"], code=code0)
            for l in range(prob.levels)]


def _reprojection_items(prob, j, a, b, pose0, pose1, code0, code1):
    ln = prob.links[j]
    return [dict(pose0=pose0, pose1=pose1, code0=code0, cam=prob.cams[0], prx_orig=a[0]["prx_orig"],
                 prx_jac=a[0]["prx_jac"], query_xy=ln.query_xy, train_xy=ln.train_xy, cauchy_delta=ln.cauchy_delta,
                 sigma=ln.sigma)]


def _geometric_items(prob, j, a, b, pose0, pose1, code0, code1):
    gl = prob.geometric[j]
    return [dict(pose0=pose0, pose1=pose1, code0=code0, code1=code1, cam=prob.cams[0], prx0_orig=a[0]["prx_orig"],
                 prx0_jac=a[0]["prx_jac"], prx1_orig=b[0]["prx_orig"], prx1_jac=b[0]["prx_jac"],
                 dpt_grad1=b[0]["dpt_grad"], points_xy=gl.points_xy, huber_delta=gl.huber_delta)]


def _run_step_batch(aligner, items, records=None):
    return aligner.RunStepBatch(aligner.make_work_items(items), records)


class SfmWindowProblem:
    """The device pipeline of one linearisation, on SfmAligner + Window: keyframes hold their pyramids on the device
    (img, grad, prx_orig, prx_jac per level + the dpt / valid buffers the fused decode writes); `linearise` re-evaluates
    the factors of the given pairs in one launch (depth decode fused in) and re-assembles the window.

    `links` (optional) are reprojection factors: they follow the photometric pairs in the window's pair list (same
    variables pose0, pose1, code0, so the linearisation cache covers them), each owns one unscaled record at the end of
    the record buffer, and the stale ones are re-linearised in one dfk_reprojection_linearize_batch launch.

    `geometric` (optional) are sparse geometric links: keyframe k1 of each must carry kf[k1][0]["dpt_grad"], the Sobel
    gradient of its level-0 depth (mapper.cpp:993-1000).  They own a record buffer of their own and a link block of the
    window; link j is index len(self.pairs) + j of the cache, and the stale ones are re-linearised in one
    dfk_sparse_geometric_linearize_batch launch."""

    def __init__(self, aligner, cams, keyframes, pairs, allreduce: Optional[Callable] = None,
                 links: Optional[Sequence[ReprojectionLink]] = None, geometric: Optional[Sequence[GeometricLink]] = None):
        import torch
        from . import _lib
        from .aligners import ReprojectionLinearizeBatch, SparseGeometricLinearizeBatch, Window
        self.al = aligner
        self.cams = list(cams)
        self.kf = keyframes          # kf[k][l] = dict(img, grad, prx_orig, prx_jac, dpt, valid) of device tensors
        self.links = list(links or [])
        P = len(pairs)
        self.pairs = [tuple(p) for p in pairs] + [(int(ln.k0), int(ln.k1)) for ln in self.links]
        self.levels = len(self.cams)
        item_pair, sizes = [], []
        for p in range(P):
            for l in range(self.levels):
                item_pair.append(p)
                t = self.kf[self.pairs[p][0]][l]["img"]
                sizes.append((int(t.shape[1]), int(t.shape[0])))
        for j in range(len(self.links)):
            item_pair.append(P + j)
            sizes.append((0, 0))  # unscaled record: b^T b enters f as it is
        self.geometric = list(geometric or [])
        for gl in self.geometric:
            if "dpt_grad" not in self.kf[gl.k1][0]:
                raise ValueError(f"keyframe {gl.k1} is k1 of a geometric link but carries no level-0 dpt_grad")
        geo_ends = [(int(gl.k0), int(gl.k1)) for gl in self.geometric]
        self.window = Window(aligner, len(keyframes), self.pairs, item_pair, sizes, geo_ends)
        self.layout = self.window.layout
        dev = self.kf[0][0]["img"].device
        self.records = torch.zeros((len(item_pair), _lib.record_floats(aligner.CS)), dtype=torch.float32, device=dev)
        self.geo_records = torch.zeros((len(self.geometric), _lib.geo_record_floats(aligner.CS)), dtype=torch.float32,
                                       device=dev) if self.geometric else None
        L = P * self.levels
        self._kinds = {  # in `todo` numbering: the photometric pairs, then the reprojection links, then the geometric links
            "photometric": _FactorKind(self.pairs[:P], 0, self.records[:L], self.levels, _photometric_items,
                                       _run_step_batch),
            "reprojection": _FactorKind(self.pairs[P:], P, self.records[L:], 1, _reprojection_items,
                                        ReprojectionLinearizeBatch),
            "geometric": _FactorKind(geo_ends, len(self.pairs), self.geo_records, 1, _geometric_items,
                                     SparseGeometricLinearizeBatch)}
        self.allreduce = allreduce
        self._solvers = {}  # fixed variables -> WindowSolver, created on first use

    def solve(self, buf, lam, fixed, code_prior_weight=0.0, codes=None):
        """WindowOptimizer's `solve` on the device: dfk_window_solve of the window buffer, then one read-back of dx and
        info together.  Returns dx (numpy float64), or None when the damped system is not positive definite."""
        import torch
        from .aligners import WindowSolver
        key = tuple(int(v) for v in fixed)
        if key not in self._solvers:
            self._solvers[key] = WindowSolver(self.window, key)
        n = self.layout.num_keyframes * self.layout.B
        out = torch.empty(8 * n + 8, dtype=torch.uint8, device=buf.device)  # [dx float64 | info int32 | pad]
        dx, info = out[:8 * n].view(torch.float64), out[8 * n:8 * n + 4].view(torch.int32)
        self._solvers[key].solve(buf, lam, code_prior_weight, codes if code_prior_weight > 0 else None, dx=dx, info=info)
        host = out.cpu().numpy()
        if int(host[8 * n:8 * n + 4].view(np.int32)[0]) != 0:
            return None
        return host[:8 * n].view(np.float64).copy()

    def _items(self, kind, poses, codes, todo):
        """the batch items of the factors `todo` of one kind (numbered within the kind) at these poses and codes"""
        kd = self._kinds[kind]
        items = []
        for j in todo:
            k0, k1 = kd.ends[j]
            items += kd.items(self, j, self.kf[k0], self.kf[k1], poses[k0].astype(np.float32),
                              poses[k1].astype(np.float32), codes[k0].astype(np.float32), codes[k1].astype(np.float32))
        return items

    def linearise(self, poses, codes, todo):
        import torch
        for kind, kd in self._kinds.items():
            sel = [p - kd.first for p in todo if kd.first <= p < kd.first + len(kd.ends)]
            if not sel:
                continue
            items = self._items(kind, poses, codes, sel)
            if len(sel) == len(kd.ends):  # the whole kind: straight into its records
                kd.batch(self.al, items, kd.records)
            else:  # some factors: one batch of their own, copied to their rows
                rows = torch.as_tensor([j * kd.rows + r for j in sel for r in range(kd.rows)], device=kd.records.device)
                kd.records.index_copy_(0, rows, kd.batch(self.al, items))
        buf = self.window.assemble(self.records, geo_records=self.geo_records)
        if self.allreduce is not None:
            self.allreduce(buf)
        return buf, None
