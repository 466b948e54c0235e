"""The consumer side of the hot path: what the factor graph does with an aligner result.

Restates (host logic only, no GTSAM here) the parts of the reference that sit immediately above the
aligners, so that a sharded evaluation can be reduced into one set of normal equations:

  * `photometric_factor_blocks`  PhotometricFactor::linearize + RunAlignmentStep
        (sources/core/gtsam/photometric_factor.cpp:84-181, 223-293): residual rescale
        res/inliers*W*H (:275-282), JtJ to double, Jtr negated (:105-106), slicing into the
        HessianFactor blocks G11 G12 G13 G22 G23 G33 / g1 g2 g3 (:126-161).
  * `WindowLayout` / `assemble_window`   the block-sparse -> dense normal equations of a keyframe window
        (SURVEY section 8e): variables [pose_k (6) | code_k (C)] per keyframe; a pair (k0 -> k1) adds
        its pose0/code0 blocks to keyframe k0's diagonal block, pose1 to k1's and the pose0-pose1 /
        pose1-code0 couplings off the diagonal.
  * `shard_pairs` / `allreduce_window`   pairs shard across ranks with no data-path collective; ONE
        all-reduce (sum) of the window's normal equations per Gauss-Newton step joins them
        (torch.distributed: NCCL over NVLink on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import List, Sequence, Tuple

import numpy as np


def record_layout(code_size: int) -> Tuple[int, int, int]:
    """(NP, NH, record_floats) of a device result record [JtJ packed | Jtr | residual | inliers bits]."""
    n = 12 + code_size
    nh = n * (n + 1) // 2
    return n, nh, nh + n + 2


def geo_record_layout(code_size: int) -> Tuple[int, int, int]:
    """(NG, NH, record_floats) of a sparse geometric record over [pose0 | pose1 | code0 | code1] (DFK_GEO_RECORD_FLOATS)."""
    n = 12 + 2 * code_size
    nh = n * (n + 1) // 2
    return n, nh, nh + n + 2


def unpack_records(records, code_size: int):
    """records: [n, REC] float32 (numpy or torch, host or device) -> dense JtJ [n,NP,NP], Jtr [n,NP], residual [n],
    inliers [n] (int64), computed with the array library the input comes from."""
    n, nh, _ = record_layout(code_size)
    return _unpack(records, n, nh)


def unpack_geometric_records(records, code_size: int):
    """unpack_records for sparse geometric records: JtJ [n, NG, NG] over [pose0 | pose1 | code0 | code1], Jtr [n, NG],
    residual [n], inliers [n] = valid points."""
    n, nh, _ = geo_record_layout(code_size)
    return _unpack(records, n, nh)


def _unpack(records, n: int, nh: int):
    if hasattr(records, "detach"):  # torch
        import torch
        r = records
        iu = torch.triu_indices(n, n, device=r.device)
        H = torch.zeros((r.shape[0], n, n), dtype=r.dtype, device=r.device)
        H[:, iu[0], iu[1]] = r[:, :nh]
        H = H + torch.triu(H, 1).transpose(1, 2)
        inl = r[:, nh + n + 1].contiguous().view(torch.int32).to(torch.int64)
        return H, r[:, nh:nh + n], r[:, nh + n], inl
    r = np.asarray(records, dtype=np.float32)
    iu = np.triu_indices(n)
    H = np.zeros((r.shape[0], n, n), dtype=r.dtype)
    H[:, iu[0], iu[1]] = r[:, :nh]
    H = H + np.transpose(np.triu(H, 1), (0, 2, 1))
    inl = np.ascontiguousarray(r[:, nh + n + 1]).view(np.uint32).astype(np.int64)
    return H, r[:, nh:nh + n], r[:, nh + n], inl


def photometric_factor_blocks(JtJ_dense, Jtr, residual, inliers, width, height, code_size):
    """photometric_factor.cpp:84-181,275-282 for one aligner result.
    Returns (Gs, gs, f): Gs = [G11, G12, G13, G22, G23, G33], gs = [g1, g2, g3] (= -Jtr blocks), f = rescaled
    residual (inf when there is no overlap, :279-282).  float64 like the reference's cast."""
    H = np.asarray(JtJ_dense, dtype=np.float64)
    g = -np.asarray(Jtr, dtype=np.float64)
    c = code_size
    Gs = [H[0:6, 0:6], H[0:6, 6:12], H[0:6, 12:12 + c], H[6:12, 6:12], H[6:12, 12:12 + c], H[12:12 + c, 12:12 + c]]
    gs = [g[0:6], g[6:12], g[12:12 + c]]
    f = float(residual) / float(inliers) * float(width) * float(height) if inliers > 0 else float("inf")
    return Gs, gs, f


@dataclass
class WindowLayout:
    """Variable order of a keyframe window: keyframe k owns [pose (6) | code (C)] at offset k * (6 + C)."""
    num_keyframes: int
    code_size: int

    @property
    def block(self) -> int:
        return 6 + self.code_size

    @property
    def dim(self) -> int:
        return self.num_keyframes * self.block


def assemble_window(layout: WindowLayout, pairs: Sequence[Tuple[int, int]], JtJ, Jtr, residual, inliers, sizes):
    """Scatter-add the per-(pair, level) systems into the window's dense normal equations.

    pairs[i] = (k0, k1): keyframe k0 is warped into frame k1 (pose0/code0 belong to k0, pose1 to k1).
    JtJ [n, NP, NP], Jtr [n, NP] in the aligner's column order [pose0 | pose1 | code0].  sizes[i] = (W, H) of the
    level (for the residual rescale); (0, 0) marks an unscaled record (a reprojection factor, whose residual b^T b enters f
    as it is).  Works on numpy arrays or torch tensors (any device).
    Returns (H [dim, dim], g [dim], f) with g = -sum Jtr (photometric_factor.cpp:106) and f = sum of rescaled residuals
    over items with overlap plus the residuals of the unscaled records."""
    c, b = layout.code_size, layout.block
    is_torch = hasattr(JtJ, "detach")
    if is_torch:
        import torch
        H = torch.zeros((layout.dim, layout.dim), dtype=torch.float64, device=JtJ.device)
        g = torch.zeros((layout.dim,), dtype=torch.float64, device=JtJ.device)
        J64, r64 = JtJ.to(torch.float64), Jtr.to(torch.float64)
    else:
        H = np.zeros((layout.dim, layout.dim))
        g = np.zeros(layout.dim)
        J64, r64 = np.asarray(JtJ, dtype=np.float64), np.asarray(Jtr, dtype=np.float64)
    f = 0.0
    for i, (k0, k1) in enumerate(pairs):
        p0, c0, p1 = k0 * b, k0 * b + 6, k1 * b
        # local column ranges: pose0 [0,6), pose1 [6,12), code0 [12,12+c)
        loc = [(slice(0, 6), slice(p0, p0 + 6)), (slice(6, 12), slice(p1, p1 + 6)), (slice(12, 12 + c), slice(c0, c0 + c))]
        for la, ga in loc:
            g[ga] -= r64[i, la]
            for lb, gb in loc:
                H[ga, gb] += J64[i, la, lb]
        inl = int(inliers[i])
        if is_unscaled(sizes[i]):
            f += float(residual[i])
        elif inl > 0:
            f += float(residual[i]) / inl * sizes[i][0] * sizes[i][1]
    return H, g, f


def is_unscaled(size) -> bool:
    """item size (0, 0): a record whose residual is not rescaled (dfk_reprojection_linearize_batch)"""
    return size[0] == 0 and size[1] == 0


@dataclass
class WindowBlocks:
    """The packed block-sparse buffer dfk_window_assemble writes (include/dfk.h, SURVEY 8e): K diagonal blocks B x B,
    K gradients B, P coupling blocks B x 6 ([pose0 | code0] of k0 x pose1 of k1), then f and the inlier total of the
    photometric (scaled) records, then L link blocks B x B ([pose0 | code0] of k0 x [pose1 | code1] of k1), one per
    sparse geometric link in `geometric`, then F frame blocks 6 x 6 and F frame gradients 6 (dfk_window_create_frames).

    Tracked frames are pose-only variables: a pair (k0, K + f) is frame f's one pair, its coupling block is [pose0 |
    code0] of k0 x the frame's pose, and its pose1 parts go to frame f's block and gradient.  The dense system orders
    the frames' variables after the keyframes': frame f at K * B + 6 f.

    Keyframe priors (dfk_window_create_priors): kf_priors[q] is the ascending keyframe list of prior q, and the buffer
    ends with one B x B prior block per distinct keyframe pair (i < j) of some prior (`prior_blocks`, ascending; rows =
    keyframe i's [pose | code], columns = j's), at `prior_offset`.  pack leaves them zero; add_keyframe_priors fills
    them."""
    num_keyframes: int
    code_size: int
    pairs: Sequence[Tuple[int, int]]
    geometric: Sequence[Tuple[int, int]] = field(default=())
    num_frames: int = 0
    kf_priors: Sequence[Tuple[int, ...]] = field(default=())

    @property
    def B(self) -> int:
        return 6 + self.code_size

    @property
    def prior_blocks(self) -> List[Tuple[int, int]]:
        return sorted({(int(p[a]), int(p[c])) for p in self.kf_priors for a in range(len(p))
                       for c in range(a + 1, len(p))})

    @property
    def prior_offset(self) -> int:
        """start of the prior blocks, after the frames' blocks and gradients"""
        return self.frame_offset + 42 * self.num_frames

    @property
    def floats(self) -> int:
        K, P, B = self.num_keyframes, len(self.pairs), self.B
        return K * (B * B + B) + P * 6 * B + 2 + len(self.geometric) * B * B + 42 * self.num_frames + \
            len(self.prior_blocks) * B * B

    @property
    def dim(self) -> int:
        """variables of the dense system: K keyframes [pose | code], then F frame poses"""
        return self.num_keyframes * self.B + 6 * self.num_frames

    def offsets(self):
        K, P, B = self.num_keyframes, len(self.pairs), self.B
        o_g = K * B * B
        o_c = o_g + K * B
        o_t = o_c + P * 6 * B
        return o_g, o_c, o_t

    @property
    def geometric_offset(self) -> int:
        """start of the link blocks, after f and the inlier total"""
        return self.offsets()[2] + 2

    @property
    def frame_offset(self) -> int:
        """start of the frame blocks (F x 36), followed by the frame gradients (F x 6)"""
        return self.geometric_offset + len(self.geometric) * self.B * self.B

    def pack(self, item_pair, JtJ, Jtr, residual, inliers, sizes, geo=None):
        """Host mirror of dfk_window_assemble (numpy, float32 sums in item order): item i belongs to pair item_pair[i];
        JtJ [n, NP, NP] dense, Jtr [n, NP], sizes[i] = (W, H), or (0, 0) for an unscaled record: its residual is added
        to f as it is and its inliers are left out of the inlier total.  geo = (JtJ [L, NG, NG], Jtr [L, NG],
        residual [L]) of the geometric links (dfk_window_assemble_geometric): after the items, the links where a
        keyframe is k0, then those where it is k1, in link order.  A frame pair's pose1 parts go to its frame's block and
        gradient.  Returns the flat buffer."""
        K, B, c = self.num_keyframes, self.B, self.code_size
        out = np.zeros(self.floats, dtype=np.float32)
        o_g, o_c, o_t = self.offsets()
        D = out[:o_g].reshape(K, B, B)
        g = out[o_g:o_c].reshape(K, B)
        O = out[o_c:o_t].reshape(len(self.pairs), B, 6)
        F, o_f = self.num_frames, self.frame_offset
        Df = out[o_f:o_f + 36 * F].reshape(F, 6, 6)
        gf = out[o_f + 36 * F:o_f + 42 * F].reshape(F, 6)
        loc0 = np.r_[0:6, 12:12 + c]  # [pose0 | code0] rows of a record
        f = np.float32(0)
        ninl = np.float32(0)
        for i, p in enumerate(item_pair):
            k0, k1 = self.pairs[p]
            H = np.asarray(JtJ[i], dtype=np.float32)
            r = np.asarray(Jtr[i], dtype=np.float32)
            D[k0] += H[np.ix_(loc0, loc0)]
            if k1 < K:
                D[k1][:6, :6] += H[6:12, 6:12]
            else:
                Df[k1 - K] += H[6:12, 6:12]
            g[k0] -= r[loc0]
            if k1 < K:
                g[k1][:6] -= r[6:12]
            else:
                gf[k1 - K] -= r[6:12]
            O[p] += H[np.ix_(loc0, np.arange(6, 12))]
            inl = int(inliers[i])
            if is_unscaled(sizes[i]):
                f += np.float32(residual[i])
                continue
            if inl > 0:
                f += np.float32(residual[i]) / np.float32(inl) * np.float32(sizes[i][0] * sizes[i][1])
            ninl += np.float32(inl)
        if self.geometric:
            gJ, gr, gres = geo
            loc1 = np.r_[6:12, 12 + c:12 + 2 * c]  # [pose1 | code1] rows of a geometric record
            Lb = out[self.geometric_offset:self.frame_offset].reshape(len(self.geometric), B, B)
            for l, (k0, k1) in enumerate(self.geometric):
                H = np.asarray(gJ[l], dtype=np.float32)
                D[k0] += H[np.ix_(loc0, loc0)]
                g[k0] -= np.asarray(gr[l], dtype=np.float32)[loc0]
                Lb[l] = H[np.ix_(loc0, loc1)]
            for l, (k0, k1) in enumerate(self.geometric):
                H = np.asarray(gJ[l], dtype=np.float32)
                D[k1] += H[np.ix_(loc1, loc1)]
                g[k1] -= np.asarray(gr[l], dtype=np.float32)[loc1]
            for l in range(len(self.geometric)):
                f += np.float32(gres[l])
        out[o_t] = f
        out[o_t + 1] = ninl
        return out

    def to_dense(self, buf):
        """(H [dim, dim], g [dim], f, inliers) of the dense normal equations the buffer stands for (numpy float64, or
        torch float64 on the buffer's device); frame f's pose is variables K * B + 6 f ... + 6."""
        K, B, F, n = self.num_keyframes, self.B, self.num_frames, self.dim
        o_g, o_c, o_t = self.offsets()
        is_torch = hasattr(buf, "detach")
        if is_torch:
            import torch
            b64 = buf.detach().to(torch.float64)
            H = torch.zeros((n, n), dtype=torch.float64, device=buf.device)
        else:
            b64 = np.asarray(buf, dtype=np.float64)
            H = np.zeros((n, n))
        D = b64[:o_g].reshape(K, B, B)
        for k in range(K):
            H[k * B:(k + 1) * B, k * B:(k + 1) * B] += D[k]
        O = b64[o_c:o_t].reshape(len(self.pairs), B, 6)
        for p, (k0, k1) in enumerate(self.pairs):
            v1 = k1 * B if k1 < K else K * B + 6 * (k1 - K)  # pose1: a keyframe's, or a frame's
            H[k0 * B:(k0 + 1) * B, v1:v1 + 6] += O[p]
            H[v1:v1 + 6, k0 * B:(k0 + 1) * B] += O[p].T if not is_torch else O[p].transpose(0, 1)
        if self.geometric:
            Lb = b64[self.geometric_offset:self.frame_offset].reshape(len(self.geometric), B, B)
            for l, (k0, k1) in enumerate(self.geometric):
                H[k0 * B:(k0 + 1) * B, k1 * B:(k1 + 1) * B] += Lb[l]
                H[k1 * B:(k1 + 1) * B, k0 * B:(k0 + 1) * B] += Lb[l].T if not is_torch else Lb[l].transpose(0, 1)
        g = b64[o_g:o_c].reshape(K * B)
        if F:
            o_f = self.frame_offset
            Df = b64[o_f:o_f + 36 * F].reshape(F, 6, 6)
            for f in range(F):
                H[K * B + 6 * f:K * B + 6 * f + 6, K * B + 6 * f:K * B + 6 * f + 6] += Df[f]
            gf = b64[o_f + 36 * F:o_f + 42 * F].reshape(6 * F)
            g = torch.cat([g, gf]) if is_torch else np.concatenate([g, gf])
        o_p = self.prior_offset
        for b, (i, j) in enumerate(self.prior_blocks):
            Pb = b64[o_p + b * B * B:o_p + (b + 1) * B * B].reshape(B, B)
            H[i * B:(i + 1) * B, j * B:(j + 1) * B] += Pb
            H[j * B:(j + 1) * B, i * B:(i + 1) * B] += Pb.T if not is_torch else Pb.transpose(0, 1)
        return H, g, float(b64[o_t]), float(b64[o_t + 1])

    def add_keyframe_priors(self, buf, rows, deltas):
        """Host mirror of dfk_window_add_keyframe_priors, in place on a numpy float32 buffer: rows[q] = keyframe prior q
        [G | g | f0] over kf_priors[q], deltas[q] its n_q B deltas Local(x0, x).  Each entry sums its priors' terms in fp64
        in prior order onto its float32 value, rounded once.  Returns buf."""
        K, B = self.num_keyframes, self.B
        o_g, _, o_t = self.offsets()
        blocks = {ij: b for b, ij in enumerate(self.prior_blocks)}
        acc = {}  # float offset of a B x B block or B gradient -> fp64 running value

        def add(off, size, v):
            if off not in acc:
                acc[off] = np.asarray(buf[off:off + size], np.float64).copy()
            acc[off] = acc[off] + v

        fsum = np.float64(buf[o_t])
        for q, kfs in enumerate(self.kf_priors):
            n = len(kfs)
            row = np.asarray(rows[q], np.float64)
            d = np.asarray(deltas[q], np.float64).reshape(n * B)
            G, g, f0 = row[:(n * B) ** 2].reshape(n * B, n * B), row[(n * B) ** 2:(n * B) ** 2 + n * B], row[-1]
            gr = g - G @ d
            for a, k in enumerate(kfs):
                add(k * B * B, B * B, G[a * B:(a + 1) * B, a * B:(a + 1) * B].ravel())
                add(o_g + k * B, B, gr[a * B:(a + 1) * B])
                for c in range(a + 1, n):
                    off = self.prior_offset + blocks[(int(k), int(kfs[c]))] * B * B
                    add(off, B * B, G[a * B:(a + 1) * B, c * B:(c + 1) * B].ravel())
            fsum = fsum + (f0 - 2 * g @ d + d @ G @ d)
        for off, v in acc.items():
            buf[off:off + v.size] = v.astype(np.float32)
        buf[o_t] = np.float32(fsum)
        return buf

    def add_depth_priors(self, buf, prior_kf, sigma, level_ptr, records):
        """Host mirror of dfk_window_add_depth_priors, in place on a numpy float32 buffer: depth prior i on keyframe
        prior_kf[i] with standard deviation sigma[i] owns records[level_ptr[i]:level_ptr[i + 1]] (rows of
        DFK_DEPTH_RECORD_FLOATS(C) floats: [JtJ packed upper | Jtr | residual | inliers]).  JtJ / sigma^2 goes to the
        keyframe's code x code block (both triangles), -Jtr / sigma^2 to its code gradient and residual / sigma^2 to f.
        Each entry sums its terms in fp64, in prior order then level order, onto its float32 value, rounded once.
        Returns buf."""
        K, B, c = self.num_keyframes, self.B, self.code_size
        o_g, _, o_t = self.offsets()
        nh = c * (c + 1) // 2
        iu = np.triu_indices(c)
        recs = np.asarray(records, np.float32).reshape(-1, nh + c + 2)
        acc = {}  # keyframe -> (fp64 code block, fp64 code gradient)
        fsum = np.float64(buf[o_t])
        for i, k in enumerate(prior_kf):
            k = int(k)
            if k not in acc:
                D = np.asarray(buf[k * B * B:(k + 1) * B * B], np.float64).reshape(B, B)[6:, 6:].copy()
                acc[k] = (D, np.asarray(buf[o_g + k * B + 6:o_g + (k + 1) * B], np.float64).copy())
            D, g = acc[k]
            s2 = np.float64(np.float32(sigma[i])) * np.float64(np.float32(sigma[i]))
            for r in recs[int(level_ptr[i]):int(level_ptr[i + 1])]:
                J = np.zeros((c, c))
                J[iu] = r[:nh].astype(np.float64)
                J[(iu[1], iu[0])] = r[:nh].astype(np.float64)
                D += J / s2
                g -= r[nh:nh + c].astype(np.float64) / s2
                fsum = fsum + np.float64(r[nh + c]) / s2
        for k, (D, g) in acc.items():
            blk = buf[k * B * B:(k + 1) * B * B].reshape(B, B)
            blk[6:, 6:] = D.astype(np.float32)
            buf[o_g + k * B + 6:o_g + (k + 1) * B] = g.astype(np.float32)
        if len(prior_kf):
            buf[o_t] = np.float32(fsum)
        return buf


def shard_pairs(num_pairs: int, world_size: int, rank: int) -> range:
    """Contiguous, balanced shard of the pair list for `rank` (sizes differ by at most one)."""
    lo = (num_pairs * rank) // world_size
    hi = (num_pairs * (rank + 1)) // world_size
    return range(lo, hi)


def allreduce_window(H, g, group=None):
    """The one collective of a sharded Gauss-Newton step: sum the window's normal equations over ranks.
    H, g are torch tensors (CUDA with NCCL, CPU with gloo); reduced in place, also returned."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(H, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(g, op=dist.ReduceOp.SUM, group=group)
    return H, g


def gauss_newton_step(H, g, damping: float = 0.0):
    """Solve H dx = g (g already carries the sign flip) with optional Levenberg damping; numpy, float64."""
    Hn = np.asarray(H, dtype=np.float64)
    gn = np.asarray(g, dtype=np.float64)
    if damping > 0:
        Hn = Hn + damping * np.diag(np.diag(Hn))
    return np.linalg.lstsq(Hn, gn, rcond=None)[0]
