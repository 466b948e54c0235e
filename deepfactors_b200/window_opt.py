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
    (frames)    tracked frames (Mapper::EnqueueFrame): pose-only variables with one photometric pair each, eliminated
                first in the device solve; marginalised into linear keyframe priors     dfk_window_marginalize_frames
                which later windows add after the all-reduce                            dfk_window_add_priors
    (depth)     depth priors (DepthPriorFactor): one launch linearises every (prior, level) item, one adds them to the
                buffer                            dfk_depth_prior_linearize_batch / dfk_window_add_depth_priors
    (slide)     a keyframe leaves the window: eliminated from the factors that touch it into a dense linear prior
                over its blanket                                                        dfk_window_marginalize_keyframe
                which the next window (without_keyframe) adds after the all-reduce      dfk_window_add_keyframe_priors
    error       the window energy without linearising (SfmWindowProblem.error): every keyframe level decoded
                into the problem's depth scratch in one launch                           dfk_update_depth_batch
                every photometric and frame (pair, level) item's error in one launch      dfk_sfm_evaluate_error_batch
                b^T b of every link, one launch per kind           dfk_reprojection_error_batch / dfk_sparse_geometric_error_batch
                one read-back, summed on the host in fp64 with the priors; WindowOptimizer(error=...) then linearises
                accepted points only
    retract     pose: t += dt, R = exp(w) R (gtsam_traits.h:48-58); code += dc           (tiny, host)
    accept      Levenberg-Marquardt on the energy f: rescaled photometric residuals + b^T b of the links (what the
                factors' error() return)

The host side (cache, retraction, damping schedule) is plain Python / numpy; nothing here needs GTSAM.
"""
from __future__ import annotations

import ctypes
import dataclasses
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
    frame_poses: Optional[np.ndarray] = None  # run(..., frame_poses): the frames' poses at the returned point
    linearisations: int = 0       # calls of `linearise`
    error_evaluations: int = 0    # calls of `error` (WindowOptimizer(error=...) only)
    # run(..., schedule=...) only: the energy every level switch re-linearised to, the level of every pair at every
    # step (-1: inactive) and every pair's position at the end (LevelSchedule.steps_done of a continuing schedule)
    switch_energy: List[float] = field(default_factory=list)
    pair_levels: List[List[int]] = field(default_factory=list)
    pair_steps_done: List[int] = field(default_factory=list)


def level_at(iters: Sequence[int], s: int, remove_after: bool = False) -> int:
    """The active level of a pair after s steps of its schedule (-1: inactive): level len(iters) - 1 for its first
    iters[-1] + 1 steps, then each finer level l for iters[l] + 1 steps; afterwards level 0, or -1 with remove_after"""
    for l in range(len(iters) - 1, -1, -1):
        if s < iters[l] + 1:
            return l
        s -= iters[l] + 1
    return -1 if remove_after else 0


def level_start(iters: Sequence[int], l: int) -> int:
    """the position of the first step at level l"""
    return sum(int(iters[m]) + 1 for m in range(l + 1, len(iters)))


@dataclass
class LevelSchedule:
    """The coarse-to-fine schedule of WindowOptimizer.run(schedule=...) and dfk_window_lm_levels (the reference's
    OptimizePhoto works, df_work.cpp:100-225, with pho_iters = iters).  The schedule's pairs are the window pairs of the
    dense items (photometric, then frame pairs, in window order); item_pair / item_level give every dense item's pair
    and pyramid level.  Error items are the dense items' twins unless error_pair / error_level say otherwise.  steps_done
    is each pair's position (0 for a new pair; trace.pair_steps_done continues a schedule), remove_after marks the pairs
    that leave once their schedule has run out (mapper.cpp:306-311: the backward direction of a new connection)."""
    iters: Sequence[int]
    item_level: Sequence[int]
    item_pair: Sequence[int]
    steps_done: Sequence[int]
    remove_after: Sequence[bool]
    error_pair: Optional[Sequence[int]] = None
    error_level: Optional[Sequence[int]] = None

    def levels(self, pos: Sequence[int]) -> List[int]:
        return [level_at(self.iters, int(s), bool(r)) for s, r in zip(pos, self.remove_after)]

    def masks(self, lvl: Sequence[int]):
        """(dense mask, error mask or None) of the pair levels lvl"""
        dm = np.asarray([lvl[q] == l for q, l in zip(self.item_pair, self.item_level)], dtype=bool)
        if self.error_pair is None and self.error_level is None:
            return dm, None
        ep = self.item_pair if self.error_pair is None else self.error_pair
        el = self.item_level if self.error_level is None else self.error_level
        return dm, np.asarray([lvl[q] == l for q, l in zip(ep, el)], dtype=bool)


class OptimizeWork:
    """A transliteration of the reference's OptimizeWork for one pair (df_work.cpp:100-190): the readable statement of
    the per-pair rule level_at / WindowOptimizer.run(schedule=...) implement.  Per mapping step the mapper calls
    bookkeeping (the factor the pair holds: constructed at a level start, removed after remove_after), then update
    (the counter), and signal_no_relinearize when ISAM2 relinearised nothing (mapper.cpp:440-538)."""

    def __init__(self, iters: Sequence[int], remove_after: bool = False):
        self.iters, self.orig = list(iters), list(iters)
        self.active_level = len(iters) - 1
        self.first, self.remove, self.remove_after = True, False, remove_after
        self.factor: Optional[int] = None  # the level of the PhotometricFactor in the graph
        self.erased = False  # mapping_steps: the work manager dropped it (finished at an update); its factor stays

    def is_new_level_start(self) -> bool:
        return self.active_level >= 0 and self.iters[self.active_level] == self.orig[self.active_level]

    def bookkeeping(self) -> Optional[int]:
        if self.remove:
            self.factor = None
            self.active_level = -2
        if self.first or (self.active_level >= 0 and self.is_new_level_start()):
            self.first = False
            self.factor = self.active_level
        return self.factor

    def update(self):
        if self.active_level >= 0:
            self.iters[self.active_level] -= 1
            if self.iters[self.active_level] < 0:
                self.active_level -= 1
        if self.remove_after and self.active_level < 0:
            self.remove = True

    def signal_no_relinearize(self):
        if not self.first:
            self.active_level -= 1

    def finished(self) -> bool:
        return self.active_level == (-2 if self.remove_after else -1)


@dataclass
class WindowError:
    """The parts of SfmWindowProblem.error's energy, each summed in fp64 in factor order (buffer units)."""
    photometric: float = 0.0   # photometric and frame (pair, level) items: res / inliers * W * H, 0 without inliers
    reprojection: float = 0.0  # b^T b of the reprojection links
    geometric: float = 0.0     # b^T b of the sparse geometric links
    priors: float = 0.0        # f0 - 2 g^T d + d^T G d of the frame priors, then of the keyframe priors
    no_inliers: int = 0        # photometric and frame items without inliers (they add 0)
    inliers: int = 0           # total inliers of the photometric and frame items
    depth: float = 0.0         # sum diff^2 / sigma^2 of the depth priors, prior by prior, level by level

    @property
    def energy(self) -> float:
        e = self.photometric + self.reprojection + self.geometric + self.priors
        return e + self.depth if self.depth else e


def prior_energy(row, delta) -> float:
    """f0 - 2 g^T d + d^T G d of a linear prior row [G (n x n) | g (n) | f0] at d = delta (n), in fp64"""
    d = np.asarray(delta, dtype=np.float64).ravel()
    n = d.size
    row = np.asarray(row, dtype=np.float64).ravel()
    G, g, f0 = row[:n * n].reshape(n, n), row[n * n:n * n + n], float(row[n * n + n])
    return f0 - 2.0 * float(g @ d) + float(d @ G @ d)


def window_error_sum(dense, areas, reprojection, geometric, prior_terms, active=None) -> WindowError:
    """The host half of SfmWindowProblem.error.  dense: [n, 2] float32 rows [residual | inliers as uint32 bits] of the
    photometric and frame items (dfk_sfm_evaluate_error_batch) with their W * H in `areas`; reprojection / geometric:
    [m, 2] rows [b^T b | valid (uint32 bits)] of the links; prior_terms: each prior's energy (prior_energy).  An item
    without inliers adds 0, as in the window assembly (PhotometricFactor::error would return inf for it).  active
    (optional, n bools): the inactive rows are skipped, counted neither as items without inliers nor in the inliers."""
    dense = np.ascontiguousarray(dense, dtype=np.float32).reshape(-1, 2)
    areas = list(areas)
    if active is not None:
        keep = np.asarray(active, dtype=bool)
        dense, areas = dense[keep], [a for a, k in zip(areas, keep) if k]
    res, inl = dense[:, 0].astype(np.float64), dense[:, 1].view(np.uint32).astype(np.int64)
    out = WindowError()
    for r, n, a in zip(res, inl, areas):
        if n > 0:
            out.photometric += float(r / n * a)
    out.no_inliers = int((inl == 0).sum())
    out.inliers = int(inl.sum())
    for b in np.asarray(reprojection, dtype=np.float32).reshape(-1, 2)[:, 0]:
        out.reprojection += float(b)
    for b in np.asarray(geometric, dtype=np.float32).reshape(-1, 2)[:, 0]:
        out.geometric += float(b)
    for t in prior_terms:
        out.priors += float(t)
    return out


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
    stale when pose0, pose1, code0 or code1 moved.  A frame pair (k, K + f) is stale when k's pose or code or frame f's
    pose moved: pass the frame poses to stale / store."""

    def __init__(self, pairs: Sequence[Tuple[int, int]], eps: float = 1e-6, geometric: Sequence[Tuple[int, int]] = ()):
        self.pairs = list(pairs)
        self.geometric = [tuple(p) for p in geometric]
        self.eps = eps
        self.invalidate()

    def _keys(self):
        return [(k0, k1, False) for k0, k1 in self.pairs] + [(k0, k1, True) for k0, k1 in self.geometric]

    @staticmethod
    def _pose1(poses, frame_poses, k1):
        return poses[k1] if k1 < len(poses) else frame_poses[k1 - len(poses)]

    def stale(self, poses: np.ndarray, codes: np.ndarray, frame_poses: Optional[np.ndarray] = None) -> List[int]:
        out = []
        for p, (k0, k1, geo) in enumerate(self._keys()):
            at = self._at[p]
            if at is None or np.abs(at[0] - poses[k0]).max() > self.eps or \
                    np.abs(at[1] - self._pose1(poses, frame_poses, k1)).max() > self.eps or \
                    np.abs(at[2] - codes[k0]).max() > self.eps or (geo and np.abs(at[3] - codes[k1]).max() > self.eps):
                out.append(p)
        return out

    def store(self, done: Sequence[int], poses: np.ndarray, codes: np.ndarray, frame_poses: Optional[np.ndarray] = None):
        keys = self._keys()
        for p in done:
            k0, k1, geo = keys[p]
            # (pose0, pose1, code0, code1) the stored records were evaluated at (a frame has no code)
            self._at[p] = (poses[k0].copy(), self._pose1(poses, frame_poses, k1).copy(), codes[k0].copy(),
                           codes[k1].copy() if geo else None)

    def invalidate(self, which: Optional[Sequence[int]] = None):
        """forget the evaluation of the factors `which` (default: all)"""
        if which is None:
            self._at = [None] * (len(self.pairs) + len(self.geometric))
        else:
            for i in which:
                self._at[i] = None


def apply_update(poses: np.ndarray, codes: np.ndarray, dx: np.ndarray, code_size: int,
                 frame_poses: Optional[np.ndarray] = None):
    """variables [pose_k (6: t, w) | code_k (C)] per keyframe; pose retraction of gtsam_traits.h:48-58.  With frame_poses
    [F, 7], frame f's pose retracts by dx[K * B + 6 f: + 6] and (poses, codes, frame_poses) is returned."""
    B = 6 + code_size
    new_p, new_c = poses.copy(), codes.copy()
    for k in range(poses.shape[0]):
        d = dx[k * B:(k + 1) * B]
        new_p[k] = se3.retract(poses[k].astype(np.float64), d[:6], np.float64)
        new_c[k] = codes[k] + d[6:]
    if frame_poses is None:
        return new_p, new_c
    o = poses.shape[0] * B
    new_f = np.stack([se3.retract(np.asarray(fp, dtype=np.float64), dx[o + 6 * f:o + 6 * f + 6], np.float64)
                      for f, fp in enumerate(frame_poses)]) if len(frame_poses) else np.zeros((0, 7))
    return new_p, new_c, new_f


def diag_eps_of(layout: WindowBlocks, buf, fixed: Sequence[int] = (), code_prior_weight: float = 0.0) -> float:
    """1e-12 max|d| of a buffer's system over the kept variables, the code prior included (what damped_solve and
    dfk_window_solve add to the diagonal): IncrementalOptimizer's fixed diag_eps"""
    H, _, _, _ = layout.to_dense(buf)
    d = np.array(H.diagonal().cpu().numpy() if hasattr(H, "detach") else np.diag(H), dtype=np.float64)
    if code_prior_weight > 0:
        B = layout.B
        for k in range(layout.num_keyframes):
            d[k * B + 6:(k + 1) * B] += code_prior_weight
    keep = np.ones(d.size, dtype=bool)
    keep[list(fixed)] = False
    return 1e-12 * float(np.abs(d[keep]).max())


def solver_columns(K: int, pairs, links=(), kf_priors=()) -> List[List[int]]:
    """The tile pattern of the window solver's factor (dfk_window_solver_create's symbolic analysis): the rows i > j of
    the nonzero tiles of every keyframe column j, fill included.  A frame pair (k1 >= K) makes no tile."""
    below = [set() for _ in range(K)]
    for a, b in list(pairs) + list(links):
        if a != b and a < K and b < K:
            below[min(a, b)].add(max(a, b))
    for p in kf_priors:
        p = sorted(int(v) for v in p)
        for x in range(len(p)):
            for y in range(x + 1, len(p)):
                below[p[x]].add(p[y])
    for j in range(K):
        rows = sorted(below[j])
        for x in range(len(rows)):
            for y in range(x):
                below[rows[y]].add(rows[x])
    return [sorted(b) for b in below]


def reusable_columns(old: WindowBlocks, new: WindowBlocks, old_fixed: Sequence[int] = (),
                     new_fixed: Sequence[int] = ()) -> int:
    """The growth rule of dfk_window_solver_create_from: the longest prefix of keyframe columns whose tile pattern the
    grown window keeps.  Raises ValueError when `new` does not extend `old` (fewer keyframes, another code size, other
    fixed variables among the old keyframes)."""
    K0 = old.num_keyframes
    if new.code_size != old.code_size or new.num_keyframes < K0:
        raise ValueError("the window does not extend the old one")
    n0 = K0 * old.B
    if sorted(int(v) for v in old_fixed) != sorted(int(v) for v in new_fixed if int(v) < n0):
        raise ValueError("the window fixes other variables among the old keyframes")
    a = solver_columns(K0, old.pairs, old.geometric, old.kf_priors)
    b = solver_columns(new.num_keyframes, new.pairs, new.geometric, new.kf_priors)
    j = 0
    while j < K0 and a[j] == b[j]:
        j += 1
    return j


@dataclass
class ISAM2Result:
    """What one IncrementalOptimizer.update did (gtsam::ISAM2Result's counts)"""
    variables_relinearized: int   # keys whose linearisation point moved (pose and code keys counted apart)
    variables_reeliminated: int   # scalar variables re-factorised: (K - first_column) B + 6 F
    factors_relinearised: int     # factors re-evaluated: the new ones and those that depend on a relinearised key
    first_column: int             # the solver's first re-factorised keyframe column (K: none)


class IncrementalOptimizer:
    """The reference's mapping step (Mapper::MappingStep, one ISAM2::update per step) on the incremental window solver:
    Gauss-Newton, Cholesky in keyframe order, relinearize_threshold / relinearize_skip as ISAM2Params.

    Every key -- the pose and the code of each keyframe, the pose of each tracked frame -- has a linearisation point
    theta_lin and the last full delta.  update() runs, in GTSAM's order:
      1. every relinearize_skip-th update, the relinearisation check on the previous delta: a key with
         max|delta_key| >= relinearize_threshold gets theta_lin <- theta_lin (+) delta_key;
      2. linearise at theta_lin: the linearisation cache re-evaluates only the new factors and those that depend on a
         relinearised key (every other key's theta_lin is unchanged bit for bit);
      3. the incremental solve gives the full delta from theta_lin (re-factorising from the first changed column);
      4. the estimate is theta_lin (+) delta (apply_update's retraction).
    The check is GTSAM's full one (not the partial check), and back-substitution always runs in full.
    MappingStep calls update with force_relinearize = true (mapper.cpp:520-521), which runs the check every step
    whatever relinearizeSkip is: reproduce it with relinearize_skip = 1.  Its threshold is the float 0.05f
    (0.0500000007 as a double); relinearize_threshold=float(np.float32(0.05)) reproduces that edge exactly.

    `linearise(poses, codes, todo[, frame_poses]) -> (buf, _)` is WindowOptimizer's; `solve(buf, diag_eps, codes) ->
    (dx, first_column)` the incremental solve (from_problem: WindowSolver.update).  diag_eps is fixed for the optimiser's
    lifetime: 1e-12 max|d| of the first linearisation, so that later solves can reuse columns.  grow() adds keyframes,
    factors and frames and carries the kept factors' cache entries over."""

    def __init__(self, layout: WindowBlocks, linearise: Callable, solve: Callable, poses, codes, frame_poses=None,
                 relinearize_threshold: float = 0.05, relinearize_skip: int = 1, code_prior_weight: float = 0.0,
                 fix_first_pose: bool = True, cache_eps: float = 1e-6):
        if relinearize_skip < 1:
            raise ValueError("relinearize_skip must be >= 1")
        self.relinearize_threshold = float(relinearize_threshold)
        self.relinearize_skip = int(relinearize_skip)
        self.code_prior_weight = float(code_prior_weight)
        self.fixed = list(range(6)) if fix_first_pose else []
        self.cache_eps = cache_eps
        self.diag_eps: Optional[float] = None
        self.update_count = 0
        self._adopt(layout, linearise, solve)
        self.cache = LinearisationCache(layout.pairs, cache_eps, layout.geometric)
        self.lin_poses = np.asarray(poses, dtype=np.float64).copy()
        self.lin_codes = np.asarray(codes, dtype=np.float64).copy()
        self.lin_frames = np.asarray(frame_poses if frame_poses is not None else np.zeros((0, 7)),
                                     dtype=np.float64).reshape(-1, 7).copy()
        self._check_sizes()
        self.delta = np.zeros(layout.dim)

    @classmethod
    def from_problem(cls, prob: "SfmWindowProblem", poses, codes, frame_poses=None, **kw) -> "IncrementalOptimizer":
        """the optimiser of an SfmWindowProblem: its linearise, and WindowSolver.update on its window"""
        opt = cls(prob.layout, prob.linearise, None, poses, codes, frame_poses, **kw)
        opt._solver_of(prob.window, None)
        return opt

    def _adopt(self, layout, linearise, solve):
        self.layout, self.linearise, self.solve = layout, linearise, solve

    def _solver_of(self, window, prev):
        from .aligners import WindowSolver
        sol = WindowSolver(window, self.fixed) if prev is None else prev.grown(window, self.fixed)
        self.solver = sol

        def solve(buf, diag_eps, codes):
            dx, j0 = sol.update(buf, diag_eps, self.code_prior_weight, codes if self.code_prior_weight > 0 else None)
            if int(sol.info.cpu().item()) != 0:
                raise RuntimeError(f"the window's system is not positive definite (variable {int(sol.info.item()) - 1})")
            return dx.cpu().numpy(), j0
        self.solve = solve

    def _check_sizes(self):
        K, F = self.layout.num_keyframes, self.layout.num_frames
        if self.lin_poses.shape != (K, 7) or self.lin_codes.shape != (K, self.layout.code_size) or \
                self.lin_frames.shape != (F, 7):
            raise ValueError(f"the window has {K} keyframes of code size {self.layout.code_size} and {F} frames")

    def _keys(self):
        """(kind, index, slice of the delta) of every key: pose and code of each keyframe, then each frame's pose"""
        K, B = self.layout.num_keyframes, self.layout.B
        out = []
        for k in range(K):
            out += [("pose", k, slice(k * B, k * B + 6)), ("code", k, slice(k * B + 6, (k + 1) * B))]
        return out + [("frame", f, slice(K * B + 6 * f, K * B + 6 * f + 6)) for f in range(self.layout.num_frames)]

    def relinearize_keys(self) -> List[Tuple[str, int]]:
        """the keys whose previous delta reaches the threshold (max |delta_key| >= relinearize_threshold)"""
        return [(kind, i) for kind, i, sl in self._keys()
                if np.abs(self.delta[sl]).max(initial=0.0) >= self.relinearize_threshold]

    def estimate(self):
        """theta_lin (+) delta: (poses, codes, frame_poses)"""
        return apply_update(self.lin_poses, self.lin_codes, self.delta, self.layout.code_size, self.lin_frames)

    def update(self) -> ISAM2Result:
        self.update_count += 1
        moved = []
        if self.update_count % self.relinearize_skip == 0:
            moved = self.relinearize_keys()
            for kind, i, sl in self._keys():
                if (kind, i) not in moved:
                    continue
                d = self.delta[sl]
                if kind == "pose":
                    self.lin_poses[i] = se3.retract(self.lin_poses[i], d, np.float64)
                elif kind == "code":
                    self.lin_codes[i] = self.lin_codes[i] + d
                else:
                    self.lin_frames[i] = se3.retract(self.lin_frames[i], d, np.float64)
                self.delta[sl] = 0.0
        frames = self.lin_frames if self.layout.num_frames else None
        todo = self.cache.stale(self.lin_poses, self.lin_codes, frames)
        if frames is None:
            buf, _ = self.linearise(self.lin_poses, self.lin_codes, todo)
        else:
            buf, _ = self.linearise(self.lin_poses, self.lin_codes, todo, frames)
        self.cache.store(todo, self.lin_poses, self.lin_codes, frames)
        if self.diag_eps is None:
            self.diag_eps = diag_eps_of(self.layout, buf, self.fixed, self.code_prior_weight)
        dx, j0 = self.solve(buf, self.diag_eps, self.lin_codes)
        self.delta = np.asarray(dx, dtype=np.float64).copy()
        K, B = self.layout.num_keyframes, self.layout.B
        return ISAM2Result(len(moved), (K - int(j0)) * B + 6 * self.layout.num_frames, len(todo), int(j0))

    def grow(self, layout: WindowBlocks, linearise: Callable, poses, codes, frame_poses=None,
             factor_of: Optional[Sequence[Optional[int]]] = None, frame_of: Optional[Sequence[Optional[int]]] = None,
             window=None, solve: Optional[Callable] = None):
        """Move to a grown window whose first keyframes are this one's (keyframes appended in index order, factors and
        frames added or removed; no slide).  poses / codes: the new keyframes' initial estimates after the old ones'
        (the old rows are ignored: the old keys keep theta_lin and delta); frame_poses: every frame's estimate, kept
        frames' rows ignored.  factor_of[i] / frame_of[f]: the old index of new factor i (cache numbering) / frame f,
        None for a new one (default: the old ones first, in order).  window: the new Window when the optimiser runs on
        WindowSolver (from_problem): the solver grows from the old one (WindowSolver.grown); else `solve`."""
        K0, B0 = self.layout.num_keyframes, self.layout.B
        K, F = layout.num_keyframes, layout.num_frames
        if layout.code_size != self.layout.code_size or K < K0:
            raise ValueError("a grown window keeps the old keyframes first, with the same code size")
        old_keys = len(self.cache._at)
        factor_of = list(factor_of) if factor_of is not None else \
            [i if i < old_keys else None for i in range(len(layout.pairs) + len(layout.geometric))]
        frame_of = list(frame_of) if frame_of is not None else [f if f < len(self.lin_frames) else None for f in range(F)]
        poses, codes = np.asarray(poses, np.float64), np.asarray(codes, np.float64)
        lin_p = np.concatenate([self.lin_poses, poses[K0:K]]).reshape(K, 7)
        lin_c = np.concatenate([self.lin_codes, codes[K0:K]]).reshape(K, layout.code_size)
        fp = np.asarray(frame_poses if frame_poses is not None else np.zeros((0, 7)), np.float64).reshape(-1, 7)
        lin_f = np.stack([self.lin_frames[o] if o is not None else fp[f] for f, o in enumerate(frame_of)]) \
            if F else np.zeros((0, 7))
        delta = np.zeros(layout.dim)
        delta[:K0 * B0] = self.delta[:K0 * B0]
        for f, o in enumerate(frame_of):
            if o is not None:
                delta[K * B0 + 6 * f:K * B0 + 6 * f + 6] = self.delta[K0 * B0 + 6 * o:K0 * B0 + 6 * o + 6]
        cache = LinearisationCache(layout.pairs, self.cache_eps, layout.geometric)
        for i, o in enumerate(factor_of):
            if o is not None:
                cache._at[i] = self.cache._at[o]
        prev = getattr(self, "solver", None)
        self._adopt(layout, linearise, solve)
        self.cache, self.lin_poses, self.lin_codes, self.lin_frames, self.delta = cache, lin_p, lin_c, lin_f, delta
        self._check_sizes()
        if window is not None:
            self._solver_of(window, prev)
        elif solve is None:
            raise ValueError("grow needs the new window (WindowSolver) or a solve")

    def grow_problem(self, old: "SfmWindowProblem", prob: "SfmWindowProblem", poses, codes,
                     frame_poses: Optional[np.ndarray], factor_of: Sequence[Optional[int]],
                     frame_of: Sequence[Optional[int]]):
        """grow() onto a grown SfmWindowProblem (from_problem's optimiser): the kept factors' records are copied from
        the old problem (carry_records, which checks every kept factor's kind and ends) with their cache entries, and
        the solver grows from the old window's.  factor_of and frame_of are required: SfmWindowProblem numbers its
        factors by kind (photometric pairs, reprojection links, frame pairs, geometric links), so a new photometric
        pair shifts every later factor and no positional default is right."""
        factor_of, frame_of = list(factor_of), list(frame_of)
        prob.carry_records(old, factor_of, frame_of)
        self.grow(prob.layout, prob.linearise, poses, codes, frame_poses, factor_of, frame_of, window=prob.window)


def mapping_steps(opt: IncrementalOptimizer, prob, works: Sequence[OptimizeWork], max_steps: int,
                  schedule: Optional[LevelSchedule] = None) -> Tuple[List[ISAM2Result], List[List[int]]]:
    """Up to max_steps of the reference's mapping steps (Mapper::MappingStep, repeated by DeepFactors::ProcessFrame while
    the work manager has work) with one OptimizeWork per pair of prob's level schedule: the host mirror of
    dfk_window_map_steps.  Each step, in the reference's order:
      1. bookkeeping of every work the manager still holds (WorkManager::Bookkeeping);
      2. their update; a work that has finished is erased from the manager, its factor stays in the graph;
      3. prob.set_active to the pairs' factor levels; a pair whose factor changed holds a new factor, so its cache
         entry is invalidated and it is linearised at theta_lin;
      4. opt.update();
      5. signal_no_relinearize of every work the manager holds when nothing was relinearised.
    It stops early once every work is erased.  schedule (default prob.level_schedule(works[0].orig)) gives the dense
    items' pairs and levels; prob.dense_pairs() the cache index of every schedule pair.  The works are updated in
    place, so a later call continues the run.  Returns every step's ISAM2Result and pair factor levels (-1: none)."""
    sched = prob.level_schedule(works[0].orig) if schedule is None else schedule
    ids = prob.dense_pairs()
    results, levels = [], []
    for _ in range(int(max_steps)):
        if all(w.erased for w in works):
            break
        prev = [w.factor for w in works]
        for w in works:
            if not w.erased:
                w.bookkeeping()
        for w in works:
            if not w.erased:
                w.update()
                w.erased = w.finished()
        lvl = [-1 if w.factor is None else w.factor for w in works]
        prob.set_active(*sched.masks(lvl))
        opt.cache.invalidate([ids[q] for q, w in enumerate(works) if w.factor != prev[q]])
        r = opt.update()
        results.append(r)
        levels.append(lvl)
        if r.variables_relinearized == 0:
            for w in works:
                if not w.erased:
                    w.signal_no_relinearize()
    return results, levels


class DeviceIncrementalOptimizer:
    """IncrementalOptimizer on the device (dfk_window_problem_isam2_update on SfmWindowProblem.device_problem()):
    theta_lin, the last delta and the estimate stay on the device, the stale items are found from the keys the check
    moved, and only those are re-linearised.  The run starts from the device problem's state: pass poses / codes /
    frame_poses to set it (any later set_state starts a new run).  update() returns IncrementalOptimizer.update's
    ISAM2Result; estimate() reads theta_lin (+) delta back.  grow_problem moves the run onto a grown window
    (dfk_window_problem_grow_from).  map_steps runs mapping_steps' loop as one call (dfk_window_map_steps).  A sharded
    window (allreduce) cannot run here."""

    def __init__(self, prob: "SfmWindowProblem", relinearize_threshold: float = 0.05, relinearize_skip: int = 1,
                 code_prior_weight: float = 0.0, fix_first_pose: bool = True, poses=None, codes=None,
                 frame_poses=None):
        if relinearize_skip < 1:
            raise ValueError("relinearize_skip must be >= 1")
        self.prob, self.layout = prob, prob.layout
        self.dev = prob.device_problem()
        self.params = dict(relinearize_threshold=float(relinearize_threshold), relinearize_skip=int(relinearize_skip),
                           code_prior_weight=float(code_prior_weight), fix_first_pose=bool(fix_first_pose))
        if poses is not None:
            frames = np.zeros((0, 7)) if frame_poses is None else np.asarray(frame_poses, np.float64).reshape(-1, 7)
            if len(frames) != self.layout.num_frames:
                raise ValueError(f"the window has {self.layout.num_frames} tracked frames: pass as many frame_poses")
            self.dev.set_state(np.concatenate([np.asarray(poses, np.float64).reshape(-1, 7), frames]),
                               np.asarray(codes, np.float64))

    def update(self) -> ISAM2Result:
        return ISAM2Result(*self.dev.isam2_update(**self.params))

    def estimate(self):
        """theta_lin (+) delta: (poses, codes, frame_poses)"""
        p, c = self.dev.get_state()
        K = self.layout.num_keyframes
        return p[:K], c, p[K:]

    def linearization(self):
        """(theta_lin poses, theta_lin codes, theta_lin frame poses, delta) of the last update"""
        p, c, d = self.dev.get_linearization()
        K = self.layout.num_keyframes
        return p[:K], c, p[K:], d

    def grow_problem(self, old: "SfmWindowProblem", prob: "SfmWindowProblem", poses, codes,
                     frame_poses: Optional[np.ndarray], factor_of: Sequence[Optional[int]],
                     frame_of: Sequence[Optional[int]]):
        """IncrementalOptimizer.grow_problem on the device (dfk_window_problem_grow_from): the run moves onto `prob`,
        the window `old` grew into.  poses / codes / frame_poses: the new keyframes' and frames' initial estimates (the
        kept ones keep theta_lin and delta); factor_of / frame_of as grow_problem takes them, turned into item maps"""
        if old is not self.prob:
            raise ValueError("grow_problem continues the run of the optimiser's own problem")
        if len(factor_of) != len(prob.pairs) + len(prob.geometric) or len(frame_of) != len(prob.frames):
            raise ValueError("factor_of needs one entry per factor and frame_of one per frame")
        L = prob.levels

        def kind_of(pr, i):
            P, PF, NP = pr._num_photometric, pr._num_photometric + len(pr.links), len(pr.pairs)
            return ("dense", i) if i < P else ("rep", i - P) if i < PF else ("frame", i - PF) if i < NP else \
                ("geo", i - NP)
        dense, rep, geo = [], [], []
        order = list(range(prob._num_photometric)) + \
            list(range(prob._num_photometric + len(prob.links), len(prob.pairs)))
        for i in order:  # the dense items in record order: photometric pairs, then frame pairs
            o = factor_of[i]
            ok, oi = kind_of(old, o) if o is not None else (None, None)
            kn = kind_of(prob, i)[0]
            if o is not None and ok != kn:
                raise ValueError(f"factor {i} ({kn}) is old factor {o} of another kind ({ok})")
            base = None if o is None else (oi if ok == "dense" else old._num_photometric + oi) * L
            dense += [-1 if base is None else base + l for l in range(L)]
        for i in range(len(prob.pairs) + len(prob.geometric)):
            kn, j = kind_of(prob, i)
            if kn not in ("rep", "geo"):
                continue
            o = factor_of[i]
            if o is not None and kind_of(old, o)[0] != kn:
                raise ValueError(f"factor {i} ({kn}) is old factor {o} of another kind")
            (rep if kn == "rep" else geo).append(-1 if o is None else kind_of(old, o)[1])
        dev = prob.device_problem()
        K = prob.layout.num_keyframes
        fr = np.zeros((0, 7)) if frame_poses is None else np.asarray(frame_poses, np.float64).reshape(-1, 7)
        dev.set_state(np.concatenate([np.asarray(poses, np.float64).reshape(K, 7), fr]), np.asarray(codes, np.float64))
        dev.grow_from(self.dev, dense, rep, geo, [-1 if o is None else o for o in frame_of])
        self.prob, self.layout, self.dev = prob, prob.layout, dev

    def map_steps(self, works: Sequence[OptimizeWork], max_steps: int, schedule: Optional[LevelSchedule] = None
                  ) -> Tuple[List[ISAM2Result], List[List[int]]]:
        """mapping_steps(opt, prob, works, max_steps, schedule) on the device: the works are updated in place"""
        sched = self.prob.level_schedule(works[0].orig) if schedule is None else schedule
        sched = dataclasses.replace(sched, remove_after=[w.remove_after for w in works])
        t = self.dev.map_steps(sched, list(works), max_steps, **self.params)
        res = [ISAM2Result(*v) for v in zip(t["variables_relinearized"], t["variables_reeliminated"],
                                            t["factors_relinearised"], t["first_column"])]
        return res, t["pair_levels"]


class WindowOptimizer:
    """Levenberg-Marquardt over the poses and codes of a keyframe window.

    `linearise(poses, codes, pairs_to_eval) -> (window_buffer, f)` is the device pipeline (see SfmWindowProblem below for
    the one built on SfmAligner / Window); injected so that the host logic is testable without a GPU.  It must return a
    buffer that its next call does not overwrite: the loop keeps the accepted point's buffer across a rejected candidate.

    `solve(buf, lam, fixed, code_prior_weight, codes) -> dx (numpy float64) | None` solves the damped system of a buffer;
    None (not positive definite) counts as a rejected step.  The default is dense_solve; SfmWindowProblem.solve is the
    block-sparse one on the device.  f is the buffer's scalar slot plus the host prior term.

    With tracked frames (layout.num_frames > 0) run takes their poses, `linearise` is called as
    linearise(poses, codes, todo, frame_poses), dx carries the frames' steps after the keyframes' and the frames' final
    poses come back on the trace (trace.frame_poses).

    `error(poses, codes[, frame_poses]) -> (E, breakdown)` (optional; SfmWindowProblem.error) is the energy at a point
    without linearising it, in the units of the buffer's f.  With it the loop evaluates E at every candidate and
    linearises only the points it accepts (the start point and every accepted step), so a rejected step costs one error
    evaluation and leaves the record buffer and the cache at the accepted point.  f is then E plus the host prior term.
    The masks of SfmWindowProblem.set_active hold for every run until the next set_active call, also for a run
    without a schedule.

    run(..., schedule=LevelSchedule) optimises coarse to fine: the policy of dfk_levels.h, with `set_active(dense_mask,
    error_mask)` (SfmWindowProblem.set_active) making the levels of the pairs the active items.  Every step moves every
    active pair one position along its schedule (level_at); when lambda would exceed lambda_max every pair above level 0
    jumps to its next finer level and lambda restarts (the run ends only when no pair is above level 0); whenever a
    level changes, the accepted point is re-linearised under the new masks and its energy becomes f."""

    def __init__(self, layout: WindowBlocks, linearise: Callable, params: Optional[LMParams] = None,
                 solve: Optional[Callable] = None, error: Optional[Callable] = None,
                 set_active: Optional[Callable] = None):
        self.layout = layout
        self.linearise = linearise
        self.params = params or LMParams()
        self.solve = solve or functools.partial(dense_solve, layout)
        self.error = error
        self.set_active = set_active
        self.cache = LinearisationCache(layout.pairs, self.params.cache_eps, layout.geometric)

    def _set_levels(self, schedule: "LevelSchedule", lvl):
        """the masks of the pair levels lvl (set_active(dense_mask, error_mask)); the records of the items that were
        off are zero, so the cache starts over"""
        self.set_active(*schedule.masks(lvl))
        self.cache.invalidate()

    def _code_prior(self, codes) -> float:
        w = self.params.code_prior_weight
        return 0.5 * w * float((codes ** 2).sum()) if w > 0 else 0.0

    def _energy(self, buf, codes) -> float:
        """f: the buffer's scalar slot (what to_dense returns) plus the prior term"""
        f = float(buf[self.layout.offsets()[2]])
        if self.params.code_prior_weight > 0:
            f += self._code_prior(codes)
        return f

    def _error(self, poses, codes, trace: LMTrace, frame_poses=None) -> float:
        """f from `error`: E plus the prior term"""
        e, _ = self.error(poses, codes) if frame_poses is None else self.error(poses, codes, frame_poses)
        trace.error_evaluations += 1
        return float(e) + self._code_prior(codes)

    def _evaluate(self, poses, codes, trace: LMTrace, frame_poses=None):
        todo = self.cache.stale(poses, codes, frame_poses)
        if frame_poses is None:
            buf, _ = self.linearise(poses, codes, todo)
        else:
            buf, _ = self.linearise(poses, codes, todo, frame_poses)
        self.cache.store(todo, poses, codes, frame_poses)
        trace.factors_relinearised.append(len(todo))
        trace.linearisations += 1
        return buf

    def run(self, poses, codes, frame_poses=None, schedule: Optional[LevelSchedule] = None
            ) -> Tuple[np.ndarray, np.ndarray, LMTrace]:
        prm = self.params
        poses = np.asarray(poses, dtype=np.float64).copy()
        codes = np.asarray(codes, dtype=np.float64).copy()
        frames = None if frame_poses is None else np.asarray(frame_poses, dtype=np.float64).reshape(-1, 7).copy()
        if (frames is None and self.layout.num_frames) or (frames is not None and len(frames) != self.layout.num_frames):
            raise ValueError(f"the window has {self.layout.num_frames} tracked frames: pass as many frame_poses")
        trace = LMTrace()
        fixed = list(range(6)) if prm.fix_first_pose else []
        lam = prm.lambda_init
        if schedule is not None:
            if self.set_active is None:
                raise ValueError("run(schedule=...) needs WindowOptimizer(..., set_active=...), e.g. prob.set_active")
            pos = [int(v) for v in schedule.steps_done]
            lvl = schedule.levels(pos)
            self._set_levels(schedule, lvl)
        buf = self._evaluate(poses, codes, trace, frames)
        f = self._energy(buf, codes) if self.error is None else self._error(poses, codes, trace, frames)
        trace.energy.append(f)
        for it in range(prm.iterations):
            if schedule is not None:
                trace.pair_levels.append(list(lvl))
            dx = self.solve(buf, lam, fixed, prm.code_prior_weight, codes)
            trace.lam.append(lam)
            ok = False
            if dx is not None:  # None: not positive definite at this damping, a rejected step with nothing re-linearised
                dx = np.asarray(dx, dtype=np.float64)
                if frames is None:
                    cand_p, cand_c = apply_update(poses, codes, dx, self.layout.code_size)
                    cand_f = None
                else:
                    cand_p, cand_c, cand_f = apply_update(poses, codes, dx, self.layout.code_size, frames)
                if self.error is None:
                    cbuf = self._evaluate(cand_p, cand_c, trace, cand_f)
                    cf = self._energy(cbuf, cand_c)
                else:
                    cf = self._error(cand_p, cand_c, trace, cand_f)
                ok = bool(np.isfinite(cf) and cf < f)
            trace.accepted.append(ok)
            if ok:
                if self.error is not None:  # only an accepted point is linearised
                    cbuf = self._evaluate(cand_p, cand_c, trace, cand_f)
                poses, codes, buf, f, frames = cand_p, cand_c, cbuf, cf, cand_f
                trace.energy.append(f)
                lam = max(lam * prm.lambda_down, 1e-12)
            else:
                # buf and f of the accepted point are still at hand; without `error` the record buffer (and with it the
                # cache) now describes the rejected candidate, which the next candidate is compared against
                lam = lam * prm.lambda_up
                if lam > prm.lambda_max and schedule is None:
                    break
            if schedule is None:
                continue
            pos = [p + 1 if l >= 0 else p for p, l in zip(pos, lvl)]
            if not ok and lam > prm.lambda_max:  # stall: every pair above level 0 moves one level finer
                now = schedule.levels(pos)
                if not any(l > 0 for l in now):
                    break
                pos = [level_start(schedule.iters, l - 1) if l > 0 else p for p, l in zip(pos, now)]
                lam = prm.lambda_init
            if it + 1 == prm.iterations:
                break
            nxt = schedule.levels(pos)
            if nxt != lvl:
                lvl = nxt
                self._set_levels(schedule, lvl)
                buf = self._evaluate(poses, codes, trace, frames)
                f = self._energy(buf, codes) if self.error is None else self._error(poses, codes, trace, frames)
                trace.switch_energy.append(f)
        if schedule is not None:
            trace.pair_steps_done = pos
        trace.frame_poses = frames
        return poses, codes, trace


class DeviceWindowOptimizer:
    """WindowOptimizer's loop as one library call (dfk_window_lm on SfmWindowProblem.device_problem()): the state and
    the accepted and candidate window buffers stay on the device, and each step reads back the solve's info and the
    candidate's energy.  The policy is WindowOptimizer's with solve=prob.solve (and error=prob.error when
    params.use_error), except that every linearisation re-evaluates every factor: an LM step moves every code, so the
    linearisation cache would re-evaluate everything anyway.  run returns what WindowOptimizer.run returns.  A run
    rewrites prob.records (see SfmWindowProblem.device_problem): invalidate the cache of a WindowOptimizer over the same
    problem before its next run.  With a schedule (LevelSchedule, e.g. prob.level_schedule(...)) run is
    dfk_window_lm_levels, WindowOptimizer.run(schedule=...)'s policy; the device problem keeps the masks of the last
    step."""

    def __init__(self, prob: "SfmWindowProblem", params: Optional[LMParams] = None, use_error: bool = False,
                 schedule: Optional[LevelSchedule] = None):
        self.prob = prob
        self.params = params or LMParams()
        self.use_error = bool(use_error)
        self.schedule = schedule
        self.dev = prob.device_problem()

    def run(self, poses, codes, frame_poses=None) -> Tuple[np.ndarray, np.ndarray, LMTrace]:
        layout = self.prob.layout
        K, F = layout.num_keyframes, layout.num_frames
        frames = np.zeros((0, 7)) if frame_poses is None else np.asarray(frame_poses, np.float64).reshape(-1, 7)
        if len(frames) != F:
            raise ValueError(f"the window has {F} tracked frames: pass as many frame_poses")
        self.dev.set_state(np.concatenate([np.asarray(poses, np.float64).reshape(-1, 7), frames]),
                           np.asarray(codes, np.float64))
        if self.schedule is None:
            # a scheduled run leaves its last masks on the device problem: an unscheduled run uses every item
            self.dev.set_active(np.ones(self.dev.num_dense, bool), np.ones(self.dev.num_error, bool))
            t = self.dev.lm(self.params, self.use_error)
        else:
            t = self.dev.lm_levels(self.params, self.schedule, self.use_error)
        p, c = self.dev.get_state()
        n = len(self.prob.pairs) + len(self.prob.geometric)
        trace = LMTrace(energy=t["energy"], lam=t["lam"], accepted=t["accepted"],
                        factors_relinearised=[n] * t["linearisations"], frame_poses=p[K:] if F else None,
                        linearisations=t["linearisations"], error_evaluations=t["error_evaluations"],
                        switch_energy=t.get("switch_energy", []), pair_levels=t.get("pair_levels", []),
                        pair_steps_done=t.get("pair_steps_done", []))
        return p[:K], c, trace


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


REP_HUBER = 0.1  # rep_huber (deepfactors_options.h:97)
REP_SIGMA = 1.0  # rep_sigma (deepfactors_options.h:99)


def match_reprojection_links(aligner, features, connections, cam, cauchy_delta: float = REP_HUBER,
                             sigma: float = REP_SIGMA, seed: int = 0, **options) -> List[ReprojectionLink]:
    """The ReprojectionLinks of keyframe connections with their matches built on the device
    (aligners.ReprojectionMatchBatch: Hamming matching, eight-point RANSAC, distance pruning).  features[k] is keyframe
    k's aligners.Features, cam its level-0 camera, connections (k0, k1) pairs; each gives the factor k0 -> k1, then
    k1 -> k0, as use_reprojection and a loop closure add them (mapper.cpp:314-325, 367-376; pass sigma = loop_sigma for
    a loop closure).  options override the rep_* RANSAC defaults (max_dist, max_iterations, threshold, probability);
    factor j of the batch has seed + j.  A factor without matches is dropped, as OptimizeRep::ConstructFactors does
    (df_work.cpp:336).  The keypoints of every list are gathered on the device and read back once with the counts."""
    import torch

    from .aligners import ReprojectionMatchBatch, match_offsets

    ends, items = [], []
    for k0, k1 in connections:
        for a, b in ((k0, k1), (k1, k0)):
            items.append(dict(options, query=features[a], train=features[b], cam=cam, seed=seed + len(items)))
            ends.append((a, b))
    if not items:
        return []
    matches, counts, _ = ReprojectionMatchBatch(aligner, items)
    off = match_offsets(items)
    parts = [counts.view(torch.float32)]
    for j, (a, b) in enumerate(ends):
        rows = matches[off[j]:off[j + 1]].long()
        if features[b].keypoints.shape[0] == 0:  # no train features: no matches, nothing to gather
            rows = rows[:0]
        parts += [features[a].keypoints[rows[:, 0]].reshape(-1), features[b].keypoints[rows[:, 1]].reshape(-1)]
    host = torch.cat(parts).cpu().numpy()
    num = host[:len(items)].view(np.int32)
    links, pos = [], len(items)
    for j, (a, b) in enumerate(ends):
        seg = int(off[j + 1] - off[j]) if features[b].keypoints.shape[0] else 0
        q = host[pos:pos + 2 * seg].reshape(-1, 2)[:num[j]]
        t = host[pos + 2 * seg:pos + 4 * seg].reshape(-1, 2)[:num[j]]
        pos += 4 * seg
        if num[j] > 0:
            links.append(ReprojectionLink(a, b, q.copy(), t.copy(), float(cauchy_delta), float(sigma)))
    return links


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
class TrackedFrame:
    """A tracked frame that did not become a keyframe (Mapper::EnqueueFrame, df_work.cpp:59-65): a pose-only variable
    with one photometric factor from keyframe k over the pyramid levels (OptimizePhoto(kf, fr), df_work.cpp:212-225).
    levels[l] = dict(img, grad) of device tensors, the frame's pyramid (the img1 / grad1 of the factor's work items)."""
    k: int
    levels: List[dict]


@dataclass
class MarginalPrior:
    """What marginalising a tracked frame leaves (MarginalizeFrames, mapper.cpp:396-436): a linear factor on keyframe
    k's [pose | code] frozen at (pose0, code0), row = [G (B x B) | g (B) | f0] (DFK_PRIOR_DOUBLES).  Its energy at x is
    f0 - 2 g^T d + d^T G d with d = [local(pose0, pose) | code - code0], in window buffer units."""
    k: int
    pose0: np.ndarray
    code0: np.ndarray
    row: np.ndarray


@dataclass
class KeyframePrior:
    """What marginalising a keyframe out of a window leaves (SfmWindowProblem.marginalize_keyframe): a dense linear factor
    over the ascending keyframes `keyframes` (the blanket of the keyframe that left), frozen at (poses0 [n, 7], codes0
    [n, C]), row = [G (nB x nB) | g (nB) | f0] (DFK_KF_PRIOR_DOUBLES).  Its energy at x is f0 - 2 g^T d + d^T G d with
    d = [local(poses0[a], pose_{keyframes[a]}) | code_{keyframes[a]} - codes0[a]] stacked over a, in window buffer
    units.  Like MarginalPrior it is never re-linearised."""
    keyframes: Tuple[int, ...]
    poses0: np.ndarray
    codes0: np.ndarray
    row: np.ndarray


@dataclass
class DepthPrior:
    """DepthPriorFactor (sources/core/gtsam/depth_prior_factor.cpp:29-137): a unary factor on keyframe k's code that
    pulls the depth decoded from it towards a measured depth map, with standard deviation sigma.  target_dpt[l] is the
    target at pyramid level l (float32 device tensors [H_l, W_l], the keyframe's level sizes); make_depth_prior builds
    them from level 0 as the factor's constructor does.  Its energy is 0.5 sum diff^2 / sigma^2 over every pixel of every
    level (in buffer units, twice that); it has no active level: every level always counts."""
    k: int
    target_dpt: List[object]
    sigma: float


def depth_prior_sizes(width: int, height: int, levels: int) -> List[Tuple[int, int]]:
    """(W_l, H_l) of a target pyramid: each level GaussianBlurDown's half of the one above (cu_image_proc.cpp:166-184)"""
    out = [(int(width), int(height))]
    for _ in range(1, levels):
        out.append((out[-1][0] // 2, out[-1][1] // 2))
    return out


def make_depth_prior(k: int, target_dpt, sigma: float, levels: int) -> DepthPrior:
    """A DepthPrior from a level-0 target depth (a float32 [H, W] device tensor): T_0 = target, T_l =
    GaussianBlurDown(T_{l-1}) (the constructor, depth_prior_factor.cpp:29-53), in one dfk_build_image_pyramid call."""
    import torch
    from .aligners import BuildImagePyramid
    t0 = target_dpt.contiguous()
    sizes = depth_prior_sizes(t0.shape[1], t0.shape[0], levels)
    pyr = [t0] + [torch.empty((h, w), dtype=torch.float32, device=t0.device) for w, h in sizes[1:]]
    if levels > 1:
        BuildImagePyramid(pyr)
    return DepthPrior(int(k), pyr, float(sigma))


def _depth_prior_items(prob, priors, codes):
    """the (prior, level) items of `priors` at these codes, prior by prior, level by level"""
    return [dict(code=np.asarray(codes[dp.k], np.float32), target_dpt=dp.target_dpt[l],
                 prx_orig=prob.kf[dp.k][l]["prx_orig"], prx_jac=prob.kf[dp.k][l]["prx_jac"])
            for dp in priors for l in range(prob.levels)]


def depth_prior_rows(records, sigma, levels: int, code_size: int) -> np.ndarray:
    """Depth priors as linear priors on their keyframe's [pose | code] (DFK_PRIOR_DOUBLES rows [G | g | f0], to be taken
    at delta = 0): records [n * levels, DFK_DEPTH_RECORD_FLOATS] of n priors, each prior's levels summed in fp64 in level
    order: G's code block = sum JtJ / sigma^2, g's code part = -sum Jtr / sigma^2, f0 = sum residual / sigma^2."""
    C, B = code_size, 6 + code_size
    nh = C * (C + 1) // 2
    iu = np.triu_indices(C)
    recs = np.asarray(records, np.float32).reshape(len(sigma), levels, nh + C + 2)
    rows = np.zeros((len(sigma), B * B + B + 1))
    for i, sg in enumerate(sigma):
        s2 = np.float64(np.float32(sg)) * np.float64(np.float32(sg))
        G, g, f0 = np.zeros((B, B)), np.zeros(B), np.float64(0.0)
        for r in recs[i]:
            J = np.zeros((C, C))
            J[iu] = r[:nh].astype(np.float64)
            J[(iu[1], iu[0])] = r[:nh].astype(np.float64)
            G[6:, 6:] += J / s2
            g[6:] -= r[nh:nh + C].astype(np.float64) / s2
            f0 = f0 + np.float64(r[nh + C]) / s2
        rows[i] = np.concatenate([G.ravel(), g, [f0]])
    return rows


def slide_factors(m: int, pairs, links=(), geometric=(), frames=(), priors=(), prior: Optional[KeyframePrior] = None):
    """The factors of a window without keyframe m, renumbered (keyframes above m move down by one): pairs and links that
    touch m are dropped, frames and the priors that do not contain m are kept, and the priors that contain m (frame priors
    on m, keyframe priors over m) are replaced by `prior`, m's KeyframePrior in the old numbering, appended last.
    Raises when a frame still sits on m (marginalise it first).  Returns (pairs, links, geometric, frames, priors)."""
    import dataclasses
    if any(fr.k == m for fr in frames):
        raise ValueError(f"keyframe {m} still has tracked frames: marginalise them first")
    ren = lambda k: int(k) - (int(k) > m)
    keep = lambda a, b: a != m and b != m
    pairs2 = [(ren(a), ren(b)) for a, b in pairs if keep(a, b)]
    links2 = [dataclasses.replace(ln, k0=ren(ln.k0), k1=ren(ln.k1)) for ln in links if keep(ln.k0, ln.k1)]
    geo2 = [dataclasses.replace(gl, k0=ren(gl.k0), k1=ren(gl.k1)) for gl in geometric if keep(gl.k0, gl.k1)]
    frames2 = [dataclasses.replace(fr, k=ren(fr.k)) for fr in frames]
    priors2 = []
    for pr in priors:
        if isinstance(pr, KeyframePrior):
            if m not in pr.keyframes:
                priors2.append(dataclasses.replace(pr, keyframes=tuple(ren(k) for k in pr.keyframes)))
        elif pr.k != m:
            priors2.append(dataclasses.replace(pr, k=ren(pr.k)))
    if prior is not None:
        if m in prior.keyframes:
            raise ValueError(f"the prior that replaces keyframe {m} cannot contain it")
        priors2.append(dataclasses.replace(prior, keyframes=tuple(ren(k) for k in prior.keyframes)))
    return pairs2, links2, geo2, frames2, priors2


def drop_keyframe(poses, codes, m: int):
    """(poses, codes) of the window without keyframe m, in the numbering of slide_factors / without_keyframe"""
    return np.delete(np.asarray(poses), m, axis=0), np.delete(np.asarray(codes), m, axis=0)


@dataclass
class _FactorKind:
    """One kind of factor of a SfmWindowProblem.  Factor j joins keyframes ends[j], is index first + j of linearise's
    `todo` and owns rows row0 + [j * rows, (j + 1) * rows) of the record buffer `base`.  items(prob, j, kf0, kf1, pose0,
    pose1, code0, code1) are factor j's batch items (float32 poses and codes); batch(aligner, items, records=None)
    linearises items in one launch, into `records` when given.  Kinds with the same batch function share one launch."""
    ends: List[Tuple[int, int]]
    first: int
    base: object
    row0: int
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


def problem_slots(K: int, levels: int, pairs, num_photometric: int, links=(), geometric=()) -> dict:
    """The state slots (pose0, pose1, code0, code1; -1 unused) of every item of SfmWindowProblem.device_problem: pairs
    are the problem's pair list (photometric pairs, then one per reprojection link, then one (k, K + f) per tracked
    frame); a pose slot >= K is frame slot - K.  dense: the photometric then the frame (pair, level) items in record
    order; reproj / geo: one per link; depth: one decode per (keyframe, level); error: the dense items' error twins,
    error_depth the decode each reads."""
    P, PF = num_photometric, num_photometric + len(links)
    ends = [tuple(pairs[p]) for p in list(range(P)) + list(range(PF, len(pairs)))]
    return dict(dense=[(a, b, a, -1) for a, b in ends for _ in range(levels)],
                reproj=[(int(ln.k0), int(ln.k1), int(ln.k0), -1) for ln in links],
                geo=[(int(gl.k0), int(gl.k1), int(gl.k0), int(gl.k1)) for gl in geometric],
                depth=[(-1, -1, k, -1) for k in range(K) for _ in range(levels)],
                error=[(a, b, -1, -1) for a, b in ends for _ in range(levels)],
                error_depth=[a * levels + l for a, b in ends for l in range(levels)])


def _struct_floats(arr, name: str, count: int) -> np.ndarray:
    """[len(arr), count] float32 numpy view of the float-array field `name` of every struct of a ctypes array: writing
    the view rewrites the array in place"""
    T = arr._type_
    off = getattr(T, name).offset
    raw = np.frombuffer(arr, dtype=np.uint8).reshape(len(arr), ctypes.sizeof(T))
    return raw[:, off:off + 4 * count].view(np.float32)


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
    dfk_sparse_geometric_linearize_batch launch.

    `frames` (optional) are tracked frames: frame f is the window's pose-only variable K + f with one photometric pair
    (k, K + f), after the photometric pairs and the reprojection links, whose items warp keyframe k into the frame's
    levels; `linearise` then takes the frames' poses.  `priors` (optional) are MarginalPriors of frames marginalised
    out of an earlier window and KeyframePriors of keyframes marginalised out of it: `linearise` adds both kinds to the
    buffer after the all-reduce.  `marginalize` turns frames into MarginalPriors, `marginalize_keyframe` a keyframe into
    a KeyframePrior, and `without_keyframe` builds the window that slides past it.

    `depth_priors` (optional) are DepthPriors: `linearise` re-evaluates every (prior, level) item in one
    dfk_depth_prior_linearize_batch launch and adds them with dfk_window_add_depth_priors after the assembly and before
    the all-reduce on rank 0 only when the pairs are sharded, else after the frame and keyframe priors (the order of the
    device problem); `error` adds their sum diff^2 / sigma^2 (WindowError.depth); `marginalize_keyframe` eliminates those
    on m with the rest of its factors and `without_keyframe` drops them; `device_problem` hands them to the window
    problem (dfk_window_problem_set_depth_priors), so DeviceWindowOptimizer runs such a window."""

    def __init__(self, aligner, cams, keyframes, pairs, allreduce: Optional[Callable] = None,
                 links: Optional[Sequence[ReprojectionLink]] = None, geometric: Optional[Sequence[GeometricLink]] = None,
                 frames: Optional[Sequence[TrackedFrame]] = None, priors: Optional[Sequence] = None,
                 depth_priors: Optional[Sequence[DepthPrior]] = None):
        import torch
        from . import _lib
        from .aligners import ReprojectionLinearizeBatch, SparseGeometricLinearizeBatch, Window
        self.al = aligner
        self.cams = list(cams)
        self.kf = keyframes          # kf[k][l] = dict(img, grad, prx_orig, prx_jac, dpt, valid) of device tensors
        self.links = list(links or [])
        self.frames = list(frames or [])
        P, K = len(pairs), len(keyframes)
        self._num_photometric = P
        self.priors = list(priors or [])
        self.depth_priors = list(depth_priors or [])
        self._mpriors = [pr for pr in self.priors if isinstance(pr, MarginalPrior)]
        self._kpriors = [pr for pr in self.priors if isinstance(pr, KeyframePrior)]
        for pr in self._mpriors:
            if not 0 <= pr.k < K:
                raise ValueError(f"prior on keyframe {pr.k}, outside the window")
        self.pairs = [tuple(p) for p in pairs] + [(int(ln.k0), int(ln.k1)) for ln in self.links] + \
            [(int(fr.k), K + f) for f, fr in enumerate(self.frames)]
        self.levels = len(self.cams)
        self._check_depth_priors()
        item_pair, sizes = [], []
        for p in range(P):
            for l in range(self.levels):
                item_pair.append(p)
                t = self.kf[self.pairs[p][0]][l]["img"]
                sizes.append((int(t.shape[1]), int(t.shape[0])))
        for j in range(len(self.links)):
            item_pair.append(P + j)
            sizes.append((0, 0))  # unscaled record: b^T b enters f as it is
        # records: the photometric items, then the frame pairs' (one RunStep launch covers both), then the links'
        PF = P + len(self.links)
        frame_items, frame_sizes = [], []
        for f in range(len(self.frames)):
            for l in range(self.levels):
                frame_items.append(PF + f)
                t = self.kf[self.pairs[PF + f][0]][l]["img"]
                frame_sizes.append((int(t.shape[1]), int(t.shape[0])))
        L = P * self.levels
        item_pair[L:L] = frame_items
        sizes[L:L] = frame_sizes
        self.geometric = list(geometric or [])
        for gl in self.geometric:
            if "dpt_grad" not in self.kf[gl.k1][0]:
                raise ValueError(f"keyframe {gl.k1} is k1 of a geometric link but carries no level-0 dpt_grad")
        geo_ends = [(int(gl.k0), int(gl.k1)) for gl in self.geometric]
        self.window = Window(aligner, len(keyframes), self.pairs, item_pair, sizes, geo_ends, len(self.frames),
                             [pr.keyframes for pr in self._kpriors])
        self.layout = self.window.layout
        dev = self.kf[0][0]["img"].device
        self.records = torch.zeros((len(item_pair), _lib.record_floats(aligner.CS)), dtype=torch.float32, device=dev)
        self.geo_records = torch.zeros((len(self.geometric), _lib.geo_record_floats(aligner.CS)), dtype=torch.float32,
                                       device=dev) if self.geometric else None
        LF = L + len(frame_items)
        # in `todo` numbering: the photometric pairs, the reprojection links, the frame pairs, then the geometric links
        self._kinds = {
            "photometric": _FactorKind(self.pairs[:P], 0, self.records, 0, self.levels, _photometric_items,
                                       _run_step_batch),
            "frame": _FactorKind(self.pairs[PF:], PF, self.records, L, self.levels, _photometric_items,
                                 _run_step_batch),
            "reprojection": _FactorKind(self.pairs[P:PF], P, self.records, LF, 1, _reprojection_items,
                                        ReprojectionLinearizeBatch),
            "geometric": _FactorKind(geo_ends, len(self.pairs), self.geo_records, 0, 1, _geometric_items,
                                     SparseGeometricLinearizeBatch)}
        self.allreduce = allreduce
        self._active = None  # set_active: the dense items' mask (None: every item active)
        self._solvers = {}  # fixed variables -> WindowSolver, created on first use
        self._prior_rows = torch.as_tensor(np.stack([np.asarray(pr.row, dtype=np.float64) for pr in self._mpriors]),
                                           device=dev) if self._mpriors else None
        self._kprior_rows = torch.as_tensor(np.concatenate([np.asarray(pr.row, dtype=np.float64).ravel()
                                                            for pr in self._kpriors]),
                                            device=dev) if self._kpriors else None
        nl = len(self.depth_priors) * self.levels
        self.depth_records = torch.zeros((nl, _lib.depth_record_floats(aligner.CS)), dtype=torch.float32,
                                         device=dev) if nl else None
        self._depth_level_ptr = [i * self.levels for i in range(len(self.depth_priors) + 1)]

    def _check_depth_priors(self):
        K = len(self.kf)
        for i, dp in enumerate(self.depth_priors):
            if not 0 <= int(dp.k) < K:
                raise ValueError(f"depth prior {i} on keyframe {dp.k}, outside the window")
            if not (np.isfinite(dp.sigma) and dp.sigma > 0):
                raise ValueError(f"depth prior {i}: sigma must be finite and > 0, got {dp.sigma}")
            if len(dp.target_dpt) != self.levels:
                raise ValueError(f"depth prior {i}: {len(dp.target_dpt)} target levels for a {self.levels}-level window")
            for l, t in enumerate(dp.target_dpt):
                want = tuple(self.kf[dp.k][l]["prx_orig"].shape[:2])
                if tuple(t.shape[:2]) != want:
                    raise ValueError(f"depth prior {i}: level {l} target is {tuple(t.shape[:2])}, keyframe {dp.k}'s "
                                     f"level is {want}")

    def _counts_depth_priors(self) -> bool:
        """the sharding rule of dfk_window_add_depth_priors: on a sharded window only rank 0 adds the depth priors, before
        the all-reduce, so each is counted once"""
        if self.allreduce is None:
            return True
        import torch.distributed as dist
        return not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0

    def _linearise_depth_priors(self, codes, records=None, priors=None):
        """every (prior, level) item of `priors` (default: all) at `codes`, in one launch, into `records`"""
        from .aligners import DepthPriorLinearizeBatch
        items = _depth_prior_items(self, self.depth_priors if priors is None else priors, codes)
        return DepthPriorLinearizeBatch(self.al, items, self.depth_records if records is None else records)

    def set_active(self, mask, error_mask=None):
        """Make only the dense items of `mask` (bools, record order: the photometric then the frame (pair, level)
        items) active: linearise evaluates the active items only and writes all-zero records for the others, error
        skips the inactive rows, and marginalize / marginalize_keyframe see the active factors.  The error items are
        the dense items' twins, so error_mask, when given, must equal mask.  All true (or None) restores every item."""
        m = None if mask is None else np.asarray(mask, dtype=bool).ravel()
        nd = self._kinds["frame"].row0 + len(self._kinds["frame"].ends) * self.levels
        if m is not None and m.size != nd:
            raise ValueError(f"a mask of {nd} dense items expected")
        if error_mask is not None and not np.array_equal(np.asarray(error_mask, dtype=bool).ravel(), m):
            raise ValueError("the error items are the dense items' twins: their mask is the dense mask")
        self._active = None if m is None or m.all() else m

    def dense_pairs(self) -> List[int]:
        """the cache index (linearise's `todo` numbering) of every pair of level_schedule: the photometric pairs, then
        the frame pairs"""
        P, PF = self._num_photometric, self._num_photometric + len(self.links)
        return list(range(P)) + list(range(PF, len(self.pairs)))

    def level_schedule(self, iters, steps_done=None, remove_after=None) -> LevelSchedule:
        """The LevelSchedule of this window's photometric and frame pairs with pho_iters = iters: item (pair, l) has
        level l; steps_done / remove_after per pair (photometric pairs, then frame pairs), default 0 / False."""
        P, F = self._num_photometric, len(self.frames)
        n = P + F
        return LevelSchedule(iters=[int(v) for v in iters], item_level=[l for _ in range(n) for l in range(self.levels)],
                             item_pair=[q for q in range(n) for _ in range(self.levels)],
                             steps_done=[0] * n if steps_done is None else [int(v) for v in steps_done],
                             remove_after=[False] * n if remove_after is None else [bool(v) for v in remove_after])

    def _zero_inactive(self, records):
        """the all-zero records of the inactive dense items"""
        if self._active is not None:
            import torch
            off = torch.as_tensor(np.flatnonzero(~self._active), device=records.device)
            records.index_fill_(0, off, 0.0)

    def solve(self, buf, lam, fixed, code_prior_weight=0.0, codes=None):
        """WindowOptimizer's `solve` on the device: dfk_window_solve of the window buffer, then one read-back of dx and
        info together.  Returns dx (numpy float64), or None when the damped system is not positive definite."""
        import torch
        from .aligners import WindowSolver
        key = tuple(int(v) for v in fixed)
        if key not in self._solvers:
            self._solvers[key] = WindowSolver(self.window, key)
        n = self.layout.dim
        out = torch.empty(8 * n + 8, dtype=torch.uint8, device=buf.device)  # [dx float64 | info int32 | pad]
        dx, info = out[:8 * n].view(torch.float64), out[8 * n:8 * n + 4].view(torch.int32)
        self._solvers[key].solve(buf, lam, code_prior_weight, codes if code_prior_weight > 0 else None, dx=dx, info=info)
        host = out.cpu().numpy()
        if int(host[8 * n:8 * n + 4].view(np.int32)[0]) != 0:
            return None
        return host[:8 * n].view(np.float64).copy()

    def _items(self, kind, poses, codes, todo, frame_poses=None):
        """the batch items of the factors `todo` of one kind (numbered within the kind) at these poses and codes"""
        kd = self._kinds[kind]
        K = len(self.kf)
        items = []
        for j in todo:
            k0, k1 = kd.ends[j]
            if k1 < K:
                lv1, pose1, code1 = self.kf[k1], poses[k1], codes[k1]
            else:  # a tracked frame: its levels and pose, no code
                lv1, pose1, code1 = self.frames[k1 - K].levels, frame_poses[k1 - K], codes[k0]
            items += kd.items(self, j, self.kf[k0], lv1, poses[k0].astype(np.float32), pose1.astype(np.float32),
                              codes[k0].astype(np.float32), code1.astype(np.float32))
        return items

    def _deltas(self, poses, codes, priors=None):
        """[m, B] Local(x0_i, x) of every frame prior's keyframe: [t - t0 | log(R R0^T) | c - c0] (gtsam_traits.h:66-72)"""
        return np.stack([np.concatenate([se3.local(pr.pose0, poses[pr.k]), np.asarray(codes[pr.k], np.float64) -
                                         np.asarray(pr.code0, np.float64)])
                         for pr in (self._mpriors if priors is None else priors)])

    def _kf_deltas(self, poses, codes):
        """the keyframe priors' deltas back to back: Local(x0, x) of every member, prior by prior"""
        return np.concatenate([np.concatenate([se3.local(pr.poses0[a], poses[k]), np.asarray(codes[k], np.float64) -
                                               np.asarray(pr.codes0[a], np.float64)])
                               for pr in self._kpriors for a, k in enumerate(pr.keyframes)])

    def error(self, poses, codes, frame_poses=None):
        """The window energy E at (poses, codes) without linearising: PhotometricFactor / ReprojectionFactor /
        SparseGeometricFactor::error of every factor plus the priors, in the units of the buffer's f (WindowOptimizer adds
        the code prior as for a linearisation).  Four launches and one read-back: every keyframe level decoded into depth
        scratch owned by this problem (dfk_update_depth_batch; the keyframes' own dpt keeps the last linearised point),
        the error of every photometric and frame (pair, level) item from that scratch (dfk_sfm_evaluate_error_batch), and
        b^T b of the reprojection and the geometric links.  Summed on the host in fp64 (window_error_sum): an item with
        inliers adds res / inliers * W * H, one without adds 0 (as in the assembly; PhotometricFactor::error would return
        inf), a link its b^T b, a prior f0 - 2 g^T d + d^T G d at the d linearise uses.  The pixel validity rule is
        EvaluateError's (border 1, min_dpt 0): E equals the linearisation's f when valid_border = 1 and min_dpt = 0.  With
        sharded pairs, E covers this rank's items and every prior: sum the factor parts across ranks and add the priors
        once.  Returns (E, WindowError)."""
        from .aligners import ReprojectionErrorBatch, SparseGeometricErrorBatch
        if self.frames and frame_poses is None:
            raise ValueError("the window has tracked frames: error needs their poses")
        st = self._err if getattr(self, "_err", None) is not None else self._error_state()
        c32 = np.asarray(codes, dtype=np.float32)
        st["depth_codes"][:] = np.repeat(c32, self.levels, axis=0)
        self.al.UpdateDepthBatch(st["depth_items"])
        allp = np.asarray(poses, dtype=np.float64)
        if self.frames:
            allp = np.concatenate([allp, np.asarray(frame_poses, dtype=np.float64).reshape(-1, 7)])
        allp = allp.astype(np.float32)
        out, nd, nr = st["out"], st["nd"], st["nr"]
        if nd:
            st["dense_p0"][:], st["dense_p1"][:] = allp[st["dense_k0"]], allp[st["dense_k1"]]
            self.al.EvaluateErrorBatch(st["dense_items"], out[:nd])
        for kind, fn, lo, hi in (("rep", ReprojectionErrorBatch, nd, nd + nr),
                                 ("geo", SparseGeometricErrorBatch, nd + nr, out.shape[0])):
            if hi > lo:
                k0, k1 = st[kind + "_k0"], st[kind + "_k1"]
                st[kind + "_p0"][:], st[kind + "_p1"][:] = allp[k0], allp[k1]
                st[kind + "_code0"][:] = c32[k0]
                if kind == "geo":
                    st["geo_code1"][:] = c32[k1]
                fn(self.al, st[kind + "_items"], out[lo:hi])
        host = out.cpu().numpy()
        terms = []
        if self._mpriors:
            terms += [prior_energy(pr.row, d) for pr, d in zip(self._mpriors, self._deltas(poses, codes))]
        if self._kpriors:
            d, at = self._kf_deltas(poses, codes), 0
            for pr in self._kpriors:
                n = len(pr.keyframes) * self.layout.B
                terms.append(prior_energy(pr.row, d[at:at + n]))
                at += n
        ew = window_error_sum(host[:nd], st["areas"], host[nd:nd + nr], host[nd + nr:], terms, self._active)
        if self.depth_priors and self._counts_depth_priors():
            ew.depth = self._depth_error(codes)
        return ew.energy, ew

    def _depth_error(self, codes) -> float:
        """sum diff^2 / sigma^2 of the depth priors at `codes` (dfk_depth_prior_error_batch, one launch), summed in fp64
        prior by prior, level by level"""
        from .aligners import DepthPriorErrorBatch
        res = DepthPriorErrorBatch(self.al, _depth_prior_items(self, self.depth_priors, codes)).cpu().numpy()[:, 0]
        e = 0.0
        for i, dp in enumerate(self.depth_priors):
            s2 = np.float64(np.float32(dp.sigma)) * np.float64(np.float32(dp.sigma))
            for l in range(self.levels):
                e += float(np.float64(res[i * self.levels + l]) / s2)
        return e

    def _error_state(self):
        """what error() builds once: the depth scratch and the ctypes item arrays, whose poses and codes each call
        rewrites in place through numpy views"""
        import torch
        from .aligners import make_geometric_items, make_reprojection_items
        K, L, C, P, PF = len(self.kf), self.levels, self.al.CS, self._num_photometric, \
            self._num_photometric + len(self.links)
        st = {"dpt": [[torch.empty_like(self.kf[k][l]["dpt"]) for l in range(L)] for k in range(K)]}
        st["depth_codes"] = np.zeros((K * L, C), dtype=np.float32)
        st["depth_items"] = self.al.make_depth_items(
            [dict(code=st["depth_codes"][k * L + l], prx_orig=self.kf[k][l]["prx_orig"], prx_jac=self.kf[k][l]["prx_jac"],
                  dpt=st["dpt"][k][l]) for k in range(K) for l in range(L)])
        zero = np.zeros(7, dtype=np.float32)
        # the dense items in record order: the photometric pairs' levels, then the frame pairs'
        ends = [(p, self.pairs[p]) for p in range(P)] + [(p, self.pairs[p]) for p in range(PF, len(self.pairs))]
        dense, k0s, k1s, areas = [], [], [], []
        for _, (a, b) in ends:
            lv1 = self.kf[b] if b < K else self.frames[b - K].levels
            for l in range(L):
                img0 = self.kf[a][l]["img"]
                dense.append(dict(pose0=zero, pose1=zero, cam=self.cams[l], img0=img0, img1=lv1[l]["img"],
                                  dpt0=st["dpt"][a][l], valid0=self.kf[a][l]["valid"], prx0_jac=self.kf[a][l]["prx_jac"],
                                  grad1=lv1[l]["grad"]))
                k0s.append(a)
                k1s.append(b)
                areas.append(float(img0.shape[0] * img0.shape[1]))
        st["nd"], st["areas"] = len(dense), areas
        st["dense_k0"], st["dense_k1"] = np.asarray(k0s, dtype=np.int64), np.asarray(k1s, dtype=np.int64)
        if dense:
            st["dense_items"] = self.al.make_work_items(dense)
            st["dense_p0"] = _struct_floats(st["dense_items"], "pose0", 7)
            st["dense_p1"] = _struct_floats(st["dense_items"], "pose1", 7)
        st["rep_k0"] = np.asarray([ln.k0 for ln in self.links], dtype=np.int64)
        st["rep_k1"] = np.asarray([ln.k1 for ln in self.links], dtype=np.int64)
        st["nr"] = len(self.links)
        if self.links:
            st["rep_code0"] = np.zeros((len(self.links), C), dtype=np.float32)
            st["rep_items"] = make_reprojection_items(
                [dict(it, code0=st["rep_code0"][j]) for j in range(len(self.links))
                 for it in _reprojection_items(self, j, self.kf[self.links[j].k0], None, zero, zero, None, None)], C)
            st["rep_p0"] = _struct_floats(st["rep_items"], "pose0", 7)
            st["rep_p1"] = _struct_floats(st["rep_items"], "pose1", 7)
        st["geo_k0"] = np.asarray([gl.k0 for gl in self.geometric], dtype=np.int64)
        st["geo_k1"] = np.asarray([gl.k1 for gl in self.geometric], dtype=np.int64)
        if self.geometric:
            st["geo_code0"] = np.zeros((len(self.geometric), C), dtype=np.float32)
            st["geo_code1"] = np.zeros((len(self.geometric), C), dtype=np.float32)
            st["geo_items"] = make_geometric_items(
                [dict(it, code0=st["geo_code0"][j], code1=st["geo_code1"][j]) for j, gl in enumerate(self.geometric)
                 for it in _geometric_items(self, j, self.kf[gl.k0], self.kf[gl.k1], zero, zero, None, None)], C)
            st["geo_p0"] = _struct_floats(st["geo_items"], "pose0", 7)
            st["geo_p1"] = _struct_floats(st["geo_items"], "pose1", 7)
        n = st["nd"] + st["nr"] + len(self.geometric)
        st["out"] = torch.empty((max(n, 1), 2), dtype=torch.float32, device=self.records.device)[:n]
        self._err = st
        return st

    def device_problem(self):
        """This window as one problem of the C ABI (aligners.WindowProblem, built once): the items linearise and error
        use, each with the state slots it reads -- the photometric then the frame (pair, level) items (fused decode),
        the reprojection links and the geometric links in record order, writing this problem's own record buffers (so
        marginalize / marginalize_keyframe keep working), and error()'s depth decodes and error items -- and both prior
        kinds with their frozen points.  DeviceWindowOptimizer runs on it.  A sharded window (allreduce) cannot.
        The device problem writes self.records / self.geo_records: after a device run they hold its last linearised
        point, so a WindowOptimizer over this problem that keeps running afterwards must start from an empty
        linearisation cache (opt.cache.invalidate())."""
        if self.allreduce is not None:
            raise ValueError("a window with an all-reduce (sharded pairs) cannot run as one device problem")
        if getattr(self, "_dev", None) is not None:
            return self._dev
        from .aligners import WindowProblem, make_geometric_items, make_reprojection_items
        st = self._err if getattr(self, "_err", None) is not None else self._error_state()
        K, L, C, P = len(self.kf), self.levels, self.al.CS, self._num_photometric
        PF = P + len(self.links)
        zero, zc = np.zeros(7, np.float32), np.zeros(C, np.float32)
        dense = []
        for p in list(range(P)) + list(range(PF, len(self.pairs))):
            a, b = self.pairs[p]
            lv1 = self.kf[b] if b < K else self.frames[b - K].levels
            dense += _photometric_items(self, p, self.kf[a], lv1, zero, zero, zc, zc)
        rep = [it for j, ln in enumerate(self.links)
               for it in _reprojection_items(self, j, self.kf[ln.k0], None, zero, zero, zc, None)]
        geo = [it for j, gl in enumerate(self.geometric)
               for it in _geometric_items(self, j, self.kf[gl.k0], self.kf[gl.k1], zero, zero, zc, zc)]
        kw = {}
        if self._mpriors:
            kw.update(frame_prior_kf=[pr.k for pr in self._mpriors],
                      frame_prior_rows=np.stack([np.asarray(pr.row, np.float64) for pr in self._mpriors]),
                      frame_prior_x0=np.stack([np.concatenate([pr.pose0, pr.code0]) for pr in self._mpriors]))
        if self._kpriors:
            kw.update(kf_prior_rows=np.concatenate([np.asarray(pr.row, np.float64).ravel() for pr in self._kpriors]),
                      kf_prior_x0=np.stack([np.concatenate([pr.poses0[a], pr.codes0[a]])
                                            for pr in self._kpriors for a in range(len(pr.keyframes))]))
        sl = problem_slots(K, L, self.pairs, P, self.links, self.geometric)
        self._dev = WindowProblem(
            self.window, self.records, self.geo_records,
            dense=self.al.make_work_items(dense) if dense else None, dense_slots=sl["dense"],
            reproj=make_reprojection_items(rep, C) if rep else None, reproj_slots=sl["reproj"],
            geo=make_geometric_items(geo, C) if geo else None, geo_slots=sl["geo"],
            depth=st["depth_items"], depth_slots=sl["depth"],
            error=st["dense_items"] if st["nd"] else None, error_slots=sl["error"], error_depth=sl["error_depth"], **kw)
        if self.depth_priors:
            items = _depth_prior_items(self, self.depth_priors, np.zeros((len(self.kf), C)))
            self._dev.set_depth_priors([dp.k for dp in self.depth_priors], [dp.sigma for dp in self.depth_priors],
                                       self._depth_level_ptr, items)
        return self._dev

    def linearise(self, poses, codes, todo, frame_poses=None):
        import torch
        if self.frames and frame_poses is None:
            raise ValueError("the window has tracked frames: linearise needs their poses")
        self._linearise_factors(poses, codes, todo, frame_poses)
        buf = self.window.assemble(self.records, geo_records=self.geo_records)
        sharded = self.allreduce is not None
        if sharded and self.depth_priors and self._counts_depth_priors():  # one rank, before the all-reduce
            self._add_depth_priors(buf, codes)
        if sharded:
            self.allreduce(buf)
        # after the all-reduce: every rank adds the priors once
        if self._mpriors:
            delta = torch.as_tensor(self._deltas(poses, codes), device=buf.device)
            self.window.add_priors(buf, [pr.k for pr in self._mpriors], self._prior_rows, delta)
        if self._kpriors:
            delta = torch.as_tensor(self._kf_deltas(poses, codes), device=buf.device)
            self.window.add_keyframe_priors(buf, self._kprior_rows, delta)
        if not sharded and self.depth_priors:  # after the priors, the order of dfk_window_problem_linearize
            self._add_depth_priors(buf, codes)
        return buf, None

    def _add_depth_priors(self, buf, codes):
        self._linearise_depth_priors(codes)
        self.window.add_depth_priors(buf, [dp.k for dp in self.depth_priors], [dp.sigma for dp in self.depth_priors],
                                     self._depth_level_ptr, self.depth_records)

    def marginalize_keyframe(self, poses, codes, m: int, frame_poses=None, code_prior_weight: float = 0.0
                             ) -> KeyframePrior:
        """Marginalise keyframe m at the current point: every factor that touches m (its pairs in both directions, its
        reprojection and geometric links) is re-evaluated at (poses, codes) into a copy of the record buffers, so a
        WindowOptimizer's linearisation cache stays valid, and together with the frame priors on m, the keyframe priors
        that contain m and, with code_prior_weight > 0, the zero-code prior on m, eliminated on the device
        (dfk_window_marginalize_keyframe).  Returns the KeyframePrior over m's blanket, frozen at its current poses and
        codes.  Every rank of a sharded window computes the same prior (no collective is involved).  Raises when m still
        has tracked frames or its block is singular."""
        import torch
        K, PF = len(self.kf), self._num_photometric + len(self.links)
        if any(fr.k == m for fr in self.frames):
            raise ValueError(f"keyframe {m} still has tracked frames: marginalise them first")
        todo = [p for p, (a, b) in enumerate(self.pairs[:PF]) if b < K and m in (a, b)]
        todo += [len(self.pairs) + j for j, gl in enumerate(self.geometric) if m in (gl.k0, gl.k1)]
        records = self.records.clone()
        geo = self.geo_records.clone() if self.geo_records is not None else None
        self._linearise_factors(poses, codes, todo, frame_poses, records, geo)
        dev = records.device
        fp = [pr for pr in self._mpriors if pr.k == m]
        frows = fdelta = krows = kdelta = None
        if fp:
            frows = torch.as_tensor(np.stack([np.asarray(pr.row, np.float64) for pr in fp]), device=dev)
            fdelta = torch.as_tensor(self._deltas(poses, codes, fp), device=dev)
        dp = [d for d in self.depth_priors if d.k == m]
        if dp:  # each a linear prior on m at delta 0, after m's frame priors
            recs = self._linearise_depth_priors(codes, records=torch.empty(
                (len(dp) * self.levels, self.depth_records.shape[1]), dtype=torch.float32, device=dev), priors=dp)
            drows = torch.as_tensor(depth_prior_rows(recs.cpu().numpy(), [d.sigma for d in dp], self.levels,
                                                     self.al.CS), device=dev)
            dzero = torch.zeros((len(dp), self.layout.B), dtype=torch.float64, device=dev)
            frows = drows if frows is None else torch.cat([frows, drows])
            fdelta = dzero if fdelta is None else torch.cat([fdelta, dzero])
        if self._kpriors:
            krows = self._kprior_rows
            kdelta = torch.as_tensor(self._kf_deltas(poses, codes), device=dev)
        prior, info = self.window.marginalize_keyframe(records, m, geo, frows, fdelta, krows, kdelta,
                                                       code_prior_weight, np.asarray(codes[m], np.float64))
        row = prior.cpu().numpy()
        if int(info.cpu().item()) != 0:
            raise RuntimeError(f"keyframe {m} has a singular block (row {int(info.cpu().item()) - 1})")
        nb = self.window.blanket(m)
        return KeyframePrior(tuple(nb), np.asarray(poses, np.float64)[nb].copy(),
                             np.asarray(codes, np.float64)[nb].copy(), row.copy())

    def without_keyframe(self, m: int, prior: KeyframePrior) -> "SfmWindowProblem":
        """The next window of a sliding window: keyframe m removed and the rest renumbered, the factors that touch m
        dropped, the priors that contain m replaced by `prior` (marginalize_keyframe's, old numbering), every other
        factor and prior renumbered (slide_factors).  drop_keyframe gives the matching poses and codes."""
        import dataclasses
        pairs, links, geo, frames, priors = slide_factors(m, self.pairs[:self._num_photometric], self.links,
                                                          self.geometric, self.frames, self.priors, prior)
        depth = [dataclasses.replace(dp, k=int(dp.k) - (int(dp.k) > m)) for dp in self.depth_priors if dp.k != m]
        return SfmWindowProblem(self.al, self.cams, self.kf[:m] + self.kf[m + 1:], pairs, self.allreduce, links, geo,
                                frames, priors, depth)

    def carry_records(self, old: "SfmWindowProblem", factor_of: Sequence[Optional[int]],
                      frame_of: Sequence[Optional[int]]):
        """Copy the records of the factors this problem keeps from `old` (a grown map: IncrementalOptimizer.grow_problem).
        factor_of[i]: the old `todo` index of this problem's factor i (photometric pairs, reprojection links, frame
        pairs, geometric links), None for a new one; frame_of[f]: the old index of frame f, None for a new one.  A kept
        factor must keep its kind and its ends (keyframes keep their indices; a frame pair's frame maps by frame_of):
        anything else raises ValueError before a record is copied."""
        import torch
        K, K0 = len(self.kf), len(old.kf)
        if len(factor_of) != len(self.pairs) + len(self.geometric) or len(frame_of) != len(self.frames):
            raise ValueError("factor_of needs one entry per factor and frame_of one per frame")
        copies = []
        for kind, kd in self._kinds.items():
            okd = old._kinds[kind]
            src, dst = [], []
            for j in range(len(kd.ends)):
                o = factor_of[kd.first + j]
                if o is None:
                    continue
                if not okd.first <= o < okd.first + len(okd.ends):
                    raise ValueError(f"factor {kd.first + j} ({kind}) is old factor {o} of another kind")
                (a, b), (oa, ob) = kd.ends[j], okd.ends[o - okd.first]
                same = a == oa and (b == ob if b < K else ob >= K0 and frame_of[b - K] == ob - K0)
                if not same:
                    raise ValueError(f"factor {kd.first + j} ({kind}, ends {(a, b)}) is not old factor {o} "
                                     f"(ends {(oa, ob)})")
                src += range(okd.row0 + (o - okd.first) * okd.rows, okd.row0 + (o - okd.first + 1) * okd.rows)
                dst += range(kd.row0 + j * kd.rows, kd.row0 + (j + 1) * kd.rows)
            if dst:
                copies.append((kd.base, okd.base, dst, src))
        for base, obase, dst, src in copies:
            dev = base.device
            base.index_copy_(0, torch.as_tensor(dst, device=dev), obase.index_select(0, torch.as_tensor(src, device=dev)))

    def marginalize(self, poses, codes, frame_poses, which) -> List[MarginalPrior]:
        """Marginalise the frames `which` at the current point (MarginalizeFrames): their pairs are re-evaluated at
        (poses, codes, frame_poses) and each becomes a MarginalPrior on its keyframe, frozen at the keyframe's current
        pose and code, for a later window that no longer holds the frame.  Raises when a frame's block is singular.
        The re-evaluated records go to a copy of the record buffer, so a WindowOptimizer's linearisation cache still
        describes this problem's records afterwards."""
        import torch
        kd = self._kinds["frame"]
        which = [int(f) for f in which]
        records = self.records.clone()
        if which:
            rows = torch.as_tensor([kd.row0 + f * kd.rows + r for f in which for r in range(kd.rows)],
                                   device=records.device)
            records.index_copy_(0, rows, kd.batch(self.al, self._items("frame", poses, codes, which, frame_poses)))
            self._zero_inactive(records)
        priors, info = self.window.marginalize_frames(records, which)
        rows, info = priors.cpu().numpy(), info.cpu().numpy()
        if np.any(info != 0):
            raise RuntimeError(f"frames {[f for f, i in zip(which, info) if i]} have a singular pose block")
        return [MarginalPrior(self.frames[f].k, np.asarray(poses[self.frames[f].k], np.float64).copy(),
                              np.asarray(codes[self.frames[f].k], np.float64).copy(), rows[i].copy())
                for i, f in enumerate(which)]

    def _linearise_factors(self, poses, codes, todo, frame_poses, records=None, geo_records=None):
        """the stale factors `todo` into their record rows: one launch per batch function (photometric and frame pairs
        share RunStepBatch), straight into the records when the rows it covers are contiguous.  records / geo_records:
        buffers to write instead of the problem's own (copies of them)"""
        import torch
        swap = {id(self.records): records, id(self.geo_records): geo_records}
        launches = {}  # batch function -> (base, items, rows)
        for kind, kd in self._kinds.items():
            sel = [p - kd.first for p in todo if kd.first <= p < kd.first + len(kd.ends)]
            if not sel:
                continue
            its = self._items(kind, poses, codes, sel, frame_poses)
            rws = [kd.row0 + j * kd.rows + r for j in sel for r in range(kd.rows)]
            if self._active is not None and kd.batch is _run_step_batch:  # the active (pair, level) items only
                keep = [i for i, r in enumerate(rws) if self._active[r]]
                its, rws = [its[i] for i in keep], [rws[i] for i in keep]
                if not rws:
                    continue
            target = swap.get(id(kd.base))
            base, items, rows = launches.setdefault(kd.batch, (kd.base if target is None else target, [], []))
            items += its
            rows += rws
        for batch, (base, items, rows) in launches.items():
            if rows == list(range(rows[0], rows[0] + len(rows))):  # contiguous rows: straight into the records
                batch(self.al, items, base[rows[0]:rows[0] + len(rows)])
            else:  # one batch of their own, copied to their rows
                base.index_copy_(0, torch.as_tensor(rows, device=base.device), batch(self.al, items))
        self._zero_inactive(self.records if records is None else records)
