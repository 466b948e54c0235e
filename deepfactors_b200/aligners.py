"""Host-side mirror of the reference's aligner API over libdfk.so.

Same class / method names, argument order and result types as
  df::SfmAligner<float,CS>   sources/cuda/cu_sfmaligner.h:50-97
  df::SE3Aligner<float>      sources/cuda/cu_se3aligner.h:38-86
  df::UpdateDepth / SobelGradients / GaussianBlurDown / SquaredError   sources/cuda/cu_image_proc.h:27-44
  df::JTJJrReductionItem / CorrespondenceReductionItem                  sources/cuda/reduction_items.h:35-143
(the C++ facade with the real template signatures is include/df/*.h; this module exists so the
parity tests and the benchmark can drive the C ABI from Python).  Image arguments are torch CUDA
float32 tensors standing in for vc::Image2DView<float, TargetDeviceCUDA>: [H, W] scalar images,
[H, W, 2] gradients, [H, W, C] code Jacobians; the row stride may exceed the row length (pitched).

PyTorch is plumbing only (device memory + streams).  Every computation is a libdfk.so call; there
is no CPU or torch fallback.
"""
from __future__ import annotations

import ctypes as C
import gzip
import os
import re
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np
import torch

from . import _lib
from ._lib import (DfkCamera, DfkDenseSfmParams, DfkDepthDecodeItem, DfkImage, DfkReprojectionItem, DfkSfmAlignerParams, DfkSparseGeometricItem, DfkSfmWorkItem,
                   DfkTrackLevel, check, lib)


# ------------------------------------------------------------------------------------------- params
@dataclass
class DenseSfmParams:
    """df::DenseSfmParams (sources/common/algorithm/dense_sfm.h:36-43)."""
    huber_delta: float = 0.1
    ocl_th: float = 1000.0
    avg_dpt: float = 2.0
    min_dpt: float = 0.0
    valid_border: int = 2


@dataclass
class SfmAlignerParams:
    """df::SfmAlignerParams (sources/cuda/cu_sfmaligner.h:41-48)."""
    sfmparams: DenseSfmParams = field(default_factory=DenseSfmParams)
    step_threads: int = 32
    step_blocks: int = 11
    eval_threads: int = 224
    eval_blocks: int = 66

    def to_c(self) -> DfkSfmAlignerParams:
        s = self.sfmparams
        return DfkSfmAlignerParams(DfkDenseSfmParams(s.huber_delta, s.ocl_th, s.avg_dpt, s.min_dpt, s.valid_border),
                                   self.step_threads, self.step_blocks, self.eval_threads, self.eval_blocks)


# ------------------------------------------------------------------------------------------- results
@dataclass
class CorrespondenceReductionItem:
    """sources/cuda/reduction_items.h:35-71"""
    residual: float = 0.0
    inliers: int = 0


@dataclass
class JTJJrReductionItem:
    """sources/cuda/reduction_items.h:77-143.  JtJ is the packed upper triangle (row major)."""
    JtJ: np.ndarray
    Jtr: np.ndarray
    residual: float
    inliers: int

    @property
    def NP(self) -> int:
        return int(self.Jtr.shape[0])

    def toDenseMatrix(self) -> np.ndarray:
        """SquareUpperTriangularMatrix::toDenseMatrix(): full symmetric NP x NP."""
        n = self.NP
        H = np.zeros((n, n), dtype=self.JtJ.dtype)
        H[np.triu_indices(n)] = self.JtJ
        return H + np.triu(H, 1).T

    @staticmethod
    def from_record(rec: np.ndarray, code_size: int) -> "JTJJrReductionItem":
        n = 12 + code_size
        nh = n * (n + 1) // 2
        rec = np.ascontiguousarray(rec, dtype=np.float32)
        inl = int(rec[nh + n + 1:nh + n + 2].view(np.uint32)[0])
        return JTJJrReductionItem(rec[:nh].copy(), rec[nh:nh + n].copy(), float(rec[nh + n]), inl)


# ------------------------------------------------------------------------------------------- views
def _image(t: torch.Tensor, floats_per_px: int = 1) -> DfkImage:
    """vc::Image2DView over a torch CUDA tensor (no copy)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32:
        raise TypeError("expected a float32 CUDA tensor")
    if floats_per_px == 1:
        if t.dim() != 2 or t.stride(1) != 1:
            raise ValueError("scalar image must be [H, W] with unit column stride")
    else:
        if t.dim() == 3:
            if t.shape[2] != floats_per_px or t.stride(2) != 1 or t.stride(1) != floats_per_px:
                raise ValueError("interleaved image must be [H, W, K] with contiguous pixels")
        elif t.dim() == 2:  # the reference's (W*K) x H float-image view
            if t.shape[1] % floats_per_px != 0 or t.stride(1) != 1:
                raise ValueError("flat interleaved image must be [H, W*K]")
        else:
            raise ValueError("bad image rank")
    h = t.shape[0]
    w = t.shape[1] if (t.dim() == 3 or floats_per_px == 1) else t.shape[1] // floats_per_px
    return DfkImage(C.c_void_p(t.data_ptr()), t.stride(0) * 4, w, h)


def _cam(cam) -> DfkCamera:
    return DfkCamera(cam.fx, cam.fy, cam.u0, cam.v0, cam.width, cam.height)


def _pose(p) -> "C.Array":
    a = np.ascontiguousarray(np.asarray(p, dtype=np.float32))
    if a.shape != (7,):
        raise ValueError("pose must be 7 floats: quaternion (x,y,z,w), translation")
    return (C.c_float * 7)(*a.tolist())


class _Handle:
    def __init__(self, device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("deepfactors_b200 needs a CUDA device (no CPU fallback)")
        dev = torch.cuda.current_device() if device is None else torch.device(device).index
        self.device = dev if dev is not None else torch.cuda.current_device()
        torch.cuda.init()
        with torch.cuda.device(self.device):
            torch.zeros(1, device="cuda")  # make sure the primary context exists
        self.h = C.c_void_p()
        st = lib().dfk_create(int(self.device), C.byref(self.h))
        if st != _lib.DFK_OK:
            raise _lib.DfkError(st, "dfk_create failed")

    def use_torch_stream(self):
        """launch on torch's current stream (so torch-side events and allocations order correctly)"""
        s = torch.cuda.current_stream(self.device).cuda_stream
        check(self.h, lib().dfk_set_stream(self.h, C.c_void_p(s)))

    def close(self):
        if getattr(self, "h", None) is not None and self.h:
            lib().dfk_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------- SfmAligner
class SfmAligner:
    """df::SfmAligner<float, CS> (sources/cuda/cu_sfmaligner.h:50-97)."""

    def __init__(self, code_size: int, params: SfmAlignerParams | None = None, device=None, gram_mode: str = "auto"):
        self.CS = int(code_size)
        self.params_ = params or SfmAlignerParams()
        self._hd = _Handle(device)
        self._hd.use_torch_stream()
        cp = self.params_.to_c()
        check(self._hd.h, lib().dfk_sfm_set_params(self._hd.h, C.byref(cp)))
        self.SetGramMode(gram_mode)

    @property
    def handle(self):
        return self._hd.h

    def SetSmLimit(self, num_sms: int):
        """size the persistent RunStep grids for `num_sms` SMs (0 = all): leaves room for a kernel on another stream, e.g.
        the window's all-reduce of the previous step (dfk_set_sm_limit)"""
        check(self._hd.h, lib().dfk_set_sm_limit(self._hd.h, int(num_sms)))

    def SetGramMode(self, mode: str):
        m = {"auto": _lib.DFK_GRAM_AUTO, "fp32": _lib.DFK_GRAM_FP32, "tf32x3": _lib.DFK_GRAM_TF32X3}[mode]
        check(self._hd.h, lib().dfk_sfm_set_gram_mode(self._hd.h, m))

    def SetEvalThreadsBlocks(self, threads: int, blocks: int):
        self.params_.eval_threads, self.params_.eval_blocks = threads, blocks
        cp = self.params_.to_c()
        check(self._hd.h, lib().dfk_sfm_set_params(self._hd.h, C.byref(cp)))

    def SetStepThreadsBlocks(self, threads: int, blocks: int):
        self.params_.step_threads, self.params_.step_blocks = threads, blocks
        cp = self.params_.to_c()
        check(self._hd.h, lib().dfk_sfm_set_params(self._hd.h, C.byref(cp)))

    def RunStep(self, pose0, pose1, code0, cam, img0, img1, dpt0, std0, valid0, prx0_jac, grad1) -> JTJJrReductionItem:
        """cu_sfmaligner.h:76-86.  Synchronous, result by value."""
        self._hd.use_torch_stream()
        n = 12 + self.CS
        JtJ = np.zeros(n * (n + 1) // 2, dtype=np.float32)
        Jtr = np.zeros(n, dtype=np.float32)
        res = C.c_float(0)
        inl = C.c_uint64(0)
        code = None if code0 is None else np.ascontiguousarray(code0, dtype=np.float32)
        F = C.POINTER(C.c_float)
        i0, i1, d0 = _image(img0), _image(img1), _image(dpt0)
        s0 = None if std0 is None else _image(std0)
        v0, jc, g1 = _image(valid0), _image(prx0_jac, self.CS), _image(grad1, 2)
        cc = _cam(cam)
        st = lib().dfk_sfm_run_step(self._hd.h, _pose(pose0), _pose(pose1),
                                    None if code is None else code.ctypes.data_as(F), self.CS, C.byref(cc),
                                    C.byref(i0), C.byref(i1), C.byref(d0), None if s0 is None else C.byref(s0),
                                    C.byref(v0), C.byref(jc), C.byref(g1),
                                    JtJ.ctypes.data_as(F), Jtr.ctypes.data_as(F), C.byref(res), C.byref(inl))
        check(self._hd.h, st)
        return JTJJrReductionItem(JtJ, Jtr, float(res.value), int(inl.value))

    def EvaluateError(self, pose0, pose1, cam, img0, img1, dpt0, std0, grad1) -> CorrespondenceReductionItem:
        """cu_sfmaligner.h:67-74."""
        self._hd.use_torch_stream()
        res = C.c_float(0)
        inl = C.c_uint64(0)
        i0, i1, d0 = _image(img0), _image(img1), _image(dpt0)
        cc = _cam(cam)
        st = lib().dfk_sfm_evaluate_error(self._hd.h, _pose(pose0), _pose(pose1), C.byref(cc), C.byref(i0),
                                          C.byref(i1), C.byref(d0), None, None, C.byref(res), C.byref(inl))
        check(self._hd.h, st)
        return CorrespondenceReductionItem(float(res.value), int(inl.value))

    # ---- batched extension (one persistent launch for many (pair, level) items) -----------------
    def make_work_items(self, items: Sequence[dict]):
        """items: dicts with pose0, pose1, cam, img0, img1, dpt0, valid0, prx0_jac, grad1; optionally prx_orig + code
        (fused depth decode: UpdateDepth(code, prx_orig, prx0_jac, avg_dpt, dpt0) happens inside the launch and dpt0
        becomes an output)."""
        arr = (DfkSfmWorkItem * len(items))()
        keep = []  # the code arrays must outlive the ctypes pointers
        for k, it in enumerate(items):
            w = arr[k]
            w.pose0 = _pose(it["pose0"])
            w.pose1 = _pose(it["pose1"])
            w.cam = _cam(it["cam"])
            w.img0, w.img1, w.dpt0 = _image(it["img0"]), _image(it["img1"]), _image(it["dpt0"])
            w.valid0, w.prx0_jac, w.grad1 = _image(it["valid0"]), _image(it["prx0_jac"], self.CS), _image(it["grad1"], 2)
            if it.get("code") is not None:
                code = np.ascontiguousarray(it["code"], dtype=np.float32)
                if code.shape != (self.CS,):
                    raise ValueError(f"code must have {self.CS} entries")
                keep.append(code)
                w.prx_orig = _image(it["prx_orig"])
                w.code = code.ctypes.data_as(C.POINTER(C.c_float))
        arr._keepalive = keep
        return arr

    def RunStepBatch(self, work_items, records: torch.Tensor | None = None) -> torch.Tensor:
        """Asynchronous: returns a device tensor [n, DFK_SFM_RECORD_FLOATS(CS)] on torch's current stream."""
        self._hd.use_torch_stream()
        n = len(work_items)
        rec = _lib.record_floats(self.CS)
        if records is None:
            records = torch.empty((n, rec), dtype=torch.float32, device=f"cuda:{self._hd.device}")
        assert records.is_contiguous() and records.numel() >= n * rec
        st = lib().dfk_sfm_run_step_batch(self._hd.h, work_items, n, self.CS, C.c_void_p(records.data_ptr()))
        check(self._hd.h, st)
        return records

    def EvaluateErrorBatch(self, work_items, out: torch.Tensor | None = None) -> torch.Tensor:
        """Many EvaluateError items in one launch (dfk_sfm_evaluate_error_batch): work_items from make_work_items, without
        the fused decode (no `code`: the depth is read from dpt0).  Asynchronous: returns a device tensor [n, 2] float32
        on torch's current stream, row i = [residual | inliers as uint32 bits] (view column 1 as int32 for the count),
        each bit for bit what EvaluateError gives for item i alone."""
        self._hd.use_torch_stream()
        n = len(work_items)
        out = _batch_records(self, n, 2, out)
        check(self._hd.h, lib().dfk_sfm_evaluate_error_batch(self._hd.h, work_items, n, C.c_void_p(out.data_ptr())))
        return out

    def UpdateDepthBatch(self, items):
        """Many UpdateDepth calls in one launch (dfk_update_depth_batch): items are dicts with code (host, CS floats),
        prx_orig, prx_jac and dpt (the output), e.g. one per (keyframe, level), or the array of make_depth_items.
        avg_dpt is params.sfmparams.avg_dpt.  Item i is bit for bit UpdateDepth(code, prx_orig, prx_jac, avg_dpt, dpt).
        Asynchronous."""
        self._hd.use_torch_stream()
        arr = items if isinstance(items, C.Array) else self.make_depth_items(items)
        check(self._hd.h, lib().dfk_update_depth_batch(self._hd.h, arr, len(items), self.CS))

    def make_depth_items(self, items: Sequence[dict]):
        """the ctypes array of UpdateDepthBatch; a float32 C-contiguous code is referenced, not copied, so a caller may
        build the array once and rewrite the codes in place"""
        arr = (DfkDepthDecodeItem * max(len(items), 1))()
        keep = []
        for k, it in enumerate(items):
            code = np.ascontiguousarray(it["code"], dtype=np.float32)
            if code.shape != (self.CS,):
                raise ValueError(f"code must have {self.CS} entries")
            keep.append(code)
            w = arr[k]
            w.prx_orig, w.prx_jac, w.dpt = _image(it["prx_orig"]), _image(it["prx_jac"], self.CS), _image(it["dpt"])
            w.code = code.ctypes.data_as(C.POINTER(C.c_float))
        arr._keepalive = keep
        return arr

    def unpack(self, records: torch.Tensor):
        r = records.detach().cpu().numpy()
        return [JTJJrReductionItem.from_record(r[i], self.CS) for i in range(r.shape[0])]


# ------------------------------------------------------------------------------------------- sparse keypoint factor
def _reprojection_item(it: dict, cs: int, keep: list) -> DfkReprojectionItem:
    """one ReprojectionFactor's arguments as the C item; the host arrays go into `keep`, which must outlive the call"""
    code = np.ascontiguousarray(it["code0"], dtype=np.float32)
    if code.shape != (cs,):
        raise ValueError(f"code0 must have {cs} entries")
    q = np.ascontiguousarray(it["query_xy"], dtype=np.float32).reshape(-1, 2)
    t = np.ascontiguousarray(it["train_xy"], dtype=np.float32).reshape(-1, 2)
    if q.shape != t.shape:
        raise ValueError("query_xy and train_xy must hold the same number of matches")
    keep += [code, q, t]
    FP = C.POINTER(C.c_float)
    w = DfkReprojectionItem()
    w.pose0, w.pose1, w.cam = _pose(it["pose0"]), _pose(it["pose1"]), _cam(it["cam"])
    w.prx_orig, w.prx_jac = _image(it["prx_orig"]), _image(it["prx_jac"], cs)
    w.code, w.query_xy, w.train_xy = code.ctypes.data_as(FP), q.ctypes.data_as(FP), t.ctypes.data_as(FP)
    w.num_matches = q.shape[0]
    w.cauchy_delta, w.sigma = float(it["cauchy_delta"]), float(it["sigma"])
    return w


def _geometric_item(it: dict, cs: int, keep: list) -> DfkSparseGeometricItem:
    """one SparseGeometricFactor's arguments as the C item; the host arrays go into `keep`, which must outlive the call"""
    c0 = np.ascontiguousarray(it["code0"], dtype=np.float32)
    c1 = np.ascontiguousarray(it["code1"], dtype=np.float32)
    if c0.shape != (cs,) or c1.shape != (cs,):
        raise ValueError(f"code0 and code1 must have {cs} entries")
    pts = np.ascontiguousarray(it["points_xy"], dtype=np.int32).reshape(-1, 2)
    keep += [c0, c1, pts]
    FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    w = DfkSparseGeometricItem()
    w.pose0, w.pose1, w.cam = _pose(it["pose0"]), _pose(it["pose1"]), _cam(it["cam"])
    w.prx0_orig, w.prx0_jac = _image(it["prx0_orig"]), _image(it["prx0_jac"], cs)
    w.prx1_orig, w.prx1_jac = _image(it["prx1_orig"]), _image(it["prx1_jac"], cs)
    w.dpt_grad1 = _image(it["dpt_grad1"], 2)
    w.code0, w.code1, w.points_xy = c0.ctypes.data_as(FP), c1.ctypes.data_as(FP), pts.ctypes.data_as(IP)
    w.num_points = pts.shape[0]
    w.huber_delta = float(it["huber_delta"])
    return w


def _check_tensor(hd: _Handle, t: torch.Tensor, dtype: torch.dtype, n: int, what: str):
    """a kernel reads or writes n elements of t, on the handle's device: refuse any other tensor before the C call"""
    dev = torch.device("cuda", hd.device)
    if not (t.dtype == dtype and t.device == dev and t.is_contiguous() and t.numel() >= n):
        raise ValueError(f"{what} must be a contiguous {dtype} tensor of at least {n} entries on {dev}")


def _batch_records(aligner, n: int, rec: int, records: torch.Tensor | None) -> torch.Tensor:
    if records is None:
        return torch.empty((n, rec), dtype=torch.float32, device=f"cuda:{aligner._hd.device}")
    _check_tensor(aligner._hd, records, torch.float32, n * rec, "records")
    return records


def ReprojectionLinearize(aligner, pose0, pose1, code0, cam, prx_orig, prx_jac, query_xy, train_xy, cauchy_delta: float,
                          sigma: float):
    """ReprojectionFactor::linearize (sources/core/gtsam/reprojection_factor.cpp:157-269) with the rows gathered on the
    device: prx_orig / prx_jac are the keyframe's level-0 DEVICE buffers, query_xy / train_xy the matched keypoints [M, 2]
    (host).  Returns (rows [2M, 13 + C] float32 = the blocks of the JacobianFactor [J_pose0 | J_pose1 | J_code0 | b],
    total_err)."""
    aligner._hd.use_torch_stream()
    cs, keep = aligner.CS, []
    w = _reprojection_item(dict(pose0=pose0, pose1=pose1, code0=code0, cam=cam, prx_orig=prx_orig, prx_jac=prx_jac,
                                query_xy=query_xy, train_xy=train_xy, cauchy_delta=cauchy_delta, sigma=sigma), cs, keep)
    rows = np.zeros((2 * w.num_matches, 13 + cs), dtype=np.float32)
    tot = C.c_float(0)
    check(aligner.handle, lib().dfk_reprojection_linearize(
        aligner.handle, w.pose0, w.pose1, w.code, cs, C.byref(w.cam), C.byref(w.prx_orig), C.byref(w.prx_jac),
        w.num_matches, w.query_xy, w.train_xy, w.cauchy_delta, w.sigma, rows.ctypes.data_as(C.POINTER(C.c_float)),
        C.byref(tot)))
    return rows, float(tot.value)


def ReprojectionLinearizeBatch(aligner, items: Sequence[dict], records: torch.Tensor | None = None) -> torch.Tensor:
    """Many ReprojectionFactors linearised in one launch straight into normal-equation records
    (dfk_reprojection_linearize_batch): items are dicts with the arguments of ReprojectionLinearize (pose0, pose1, code0,
    cam, prx_orig, prx_jac, query_xy, train_xy, cauchy_delta, sigma).  Record i = [A^T A packed | -A^T b | b^T b | valid
    matches] of factor i's rows, in the RunStep record layout, so it goes into Window.assemble as an unscaled record
    (item size (0, 0)).  `records` may be a slice of a larger record buffer.  Asynchronous: returns a device tensor
    [n, DFK_SFM_RECORD_FLOATS(CS)] on torch's current stream."""
    aligner._hd.use_torch_stream()
    cs, n, keep = aligner.CS, len(items), []
    records = _batch_records(aligner, n, _lib.record_floats(cs), records)
    arr = (DfkReprojectionItem * max(n, 1))(*[_reprojection_item(it, cs, keep) for it in items])
    check(aligner.handle, lib().dfk_reprojection_linearize_batch(aligner.handle, arr, n, cs,
                                                                 C.c_void_p(records.data_ptr())))
    return records


def SparseGeometricLinearize(aligner, pose0, pose1, code0, code1, cam, prx0_orig, prx0_jac, prx1_orig, prx1_jac, dpt_grad1,
                             points_xy, huber_delta: float):
    """SparseGeometricFactor::linearize (sources/core/gtsam/sparse_geometric_factor.cpp:157-271) on the device: prx*_orig /
    prx*_jac are the two keyframes' level-0 DEVICE buffers, dpt_grad1 keyframe 1's depth gradient [H, W, 2] (device),
    points_xy the sampled integer pixels [M, 2] (host).  Returns (rows [M, 13 + 2C] float32 = the blocks of the
    JacobianFactor [J_pose0 | J_pose1 | J_code0 | J_code1 | b], number of valid rows)."""
    aligner._hd.use_torch_stream()
    cs, keep = aligner.CS, []
    w = _geometric_item(dict(pose0=pose0, pose1=pose1, code0=code0, code1=code1, cam=cam, prx0_orig=prx0_orig,
                             prx0_jac=prx0_jac, prx1_orig=prx1_orig, prx1_jac=prx1_jac, dpt_grad1=dpt_grad1,
                             points_xy=points_xy, huber_delta=huber_delta), cs, keep)
    rows = np.zeros((w.num_points, 13 + 2 * cs), dtype=np.float32)
    nv = C.c_int(0)
    check(aligner.handle, lib().dfk_sparse_geometric_linearize(
        aligner.handle, w.pose0, w.pose1, w.code0, w.code1, cs, C.byref(w.cam), C.byref(w.prx0_orig), C.byref(w.prx0_jac),
        C.byref(w.prx1_orig), C.byref(w.prx1_jac), C.byref(w.dpt_grad1), w.num_points, w.points_xy, w.huber_delta,
        rows.ctypes.data_as(C.POINTER(C.c_float)), C.byref(nv)))
    return rows, int(nv.value)


def SparseGeometricLinearizeBatch(aligner, items: Sequence[dict], records: torch.Tensor | None = None) -> torch.Tensor:
    """Many SparseGeometricFactors linearised in one launch straight into normal-equation records
    (dfk_sparse_geometric_linearize_batch): items are dicts with the arguments of SparseGeometricLinearize (pose0, pose1,
    code0, code1, cam, prx0_orig, prx0_jac, prx1_orig, prx1_jac, dpt_grad1, points_xy, huber_delta).  Record i =
    [A^T A packed | -A^T b | b^T b | valid points] of factor i's rows over [pose0 | pose1 | code0 | code1]
    (DFK_GEO_RECORD_FLOATS(CS) floats), which goes into Window.assemble(geo_records=...).  `records` may be a slice of a
    larger record buffer.  Asynchronous: returns a device tensor [n, DFK_GEO_RECORD_FLOATS(CS)] on torch's current
    stream."""
    aligner._hd.use_torch_stream()
    cs, n, keep = aligner.CS, len(items), []
    records = _batch_records(aligner, n, _lib.geo_record_floats(cs), records)
    arr = (DfkSparseGeometricItem * max(n, 1))(*[_geometric_item(it, cs, keep) for it in items])
    check(aligner.handle, lib().dfk_sparse_geometric_linearize_batch(aligner.handle, arr, n, cs,
                                                                     C.c_void_p(records.data_ptr())))
    return records


def make_reprojection_items(items: Sequence[dict], cs: int):
    """the ctypes array of ReprojectionErrorBatch; a float32 C-contiguous code0 is referenced, not copied, so a caller
    may build the array once and rewrite poses and codes in place"""
    keep = []
    arr = (DfkReprojectionItem * max(len(items), 1))(*[_reprojection_item(it, cs, keep) for it in items])
    arr._keepalive = keep
    return arr


def make_geometric_items(items: Sequence[dict], cs: int):
    """the ctypes array of SparseGeometricErrorBatch (code0 / code1 referenced as in make_reprojection_items)"""
    keep = []
    arr = (DfkSparseGeometricItem * max(len(items), 1))(*[_geometric_item(it, cs, keep) for it in items])
    arr._keepalive = keep
    return arr


def ReprojectionErrorBatch(aligner, items, out: torch.Tensor | None = None) -> torch.Tensor:
    """ReprojectionFactor::error of many factors in one launch (dfk_reprojection_error_batch): the items of
    ReprojectionLinearizeBatch (dicts, or the array of make_reprojection_items).  Asynchronous: returns a device tensor [n, 2] float32, row i = [b^T b | valid matches as
    uint32 bits], b^T b bit for bit the residual of factor i's ReprojectionLinearizeBatch record."""
    aligner._hd.use_torch_stream()
    cs, n = aligner.CS, len(items)
    out = _batch_records(aligner, n, 2, out)
    arr = items if isinstance(items, C.Array) else make_reprojection_items(items, cs)
    check(aligner.handle, lib().dfk_reprojection_error_batch(aligner.handle, arr, n, cs, C.c_void_p(out.data_ptr())))
    return out


# ------------------------------------------------------------------------------------------- keypoint matching
# the reference's rep_* options (deepfactors_options.h:93-101) and PruneMatchesEightPoint's probability (matching.h:48-50);
# the threshold is the float option widened to double, as the reference passes it
REP_MAX_DIST = 30.0
REP_RANSAC_MAXITERS = 1000
REP_RANSAC_THRESHOLD = float(np.float32(1e-4))
REP_RANSAC_PROBABILITY = 0.99


@dataclass
class Features:
    """A keyframe's keypoints and binary descriptors on the device (kf->features of the reference): keypoints [N, 2]
    float32 (keypoints[i].pt at level 0), descriptors [N, D] uint8 with D = 32 (ORB) or 64 (BRISK)."""
    keypoints: torch.Tensor
    descriptors: torch.Tensor

    @staticmethod
    def from_host(keypoints, descriptors, device="cuda") -> "Features":
        kp = np.ascontiguousarray(np.asarray(keypoints, np.float32).reshape(-1, 2))
        d = np.ascontiguousarray(np.asarray(descriptors, np.uint8))
        if d.ndim != 2 or d.shape[0] != kp.shape[0]:
            raise ValueError("descriptors must be [N, D] with one row per keypoint")
        return Features(torch.from_numpy(kp).to(device), torch.from_numpy(d).to(device))


def _feature_set(hd: _Handle, f: Features) -> _lib.DfkFeatureSet:
    kp, d = f.keypoints, f.descriptors
    n = int(kp.shape[0]) if kp.dim() == 2 else -1
    if kp.dim() != 2 or kp.shape[1] != 2 or d.dim() != 2 or d.shape[0] != n:
        raise ValueError("features: keypoints must be [N, 2] and descriptors [N, D]")
    _check_tensor(hd, kp, torch.float32, 2 * n, "keypoints")
    _check_tensor(hd, d, torch.uint8, n * int(d.shape[1]), "descriptors")
    return _lib.DfkFeatureSet(kp.data_ptr() if n else None, d.data_ptr() if n else None, n, int(d.shape[1]))


def _match_item(hd: _Handle, it: dict) -> _lib.DfkMatchItem:
    w = _lib.DfkMatchItem()
    w.query, w.train = _feature_set(hd, it["query"]), _feature_set(hd, it["train"])
    if it.get("cam") is not None:
        w.cam = _cam(it["cam"])
    w.max_dist = float(it.get("max_dist", REP_MAX_DIST))
    w.max_iterations = int(it.get("max_iterations", REP_RANSAC_MAXITERS))
    w.threshold = float(it.get("threshold", REP_RANSAC_THRESHOLD))
    w.probability = float(it.get("probability", REP_RANSAC_PROBABILITY))
    w.seed = int(it.get("seed", 0))
    return w


def match_offsets(items: Sequence[dict]) -> np.ndarray:
    """[n + 1]: item i's rows of the match outputs are [offsets[i], offsets[i + 1]) (the prefix sum of the query counts)"""
    return np.concatenate([[0], np.cumsum([int(it["query"].keypoints.shape[0]) for it in items])]).astype(np.int64)


def HammingMatchBatch(aligner, items: Sequence[dict], out: torch.Tensor | None = None) -> torch.Tensor:
    """cv::BFMatcher(NORM_HAMMING).match(query, train) of many factors in one launch (dfk_hamming_match_batch): items are
    dicts with query / train (Features).  Asynchronous: returns a device tensor [sum of query counts, 2] int32, item i's
    rows at match_offsets(items)[i], row q = (train index, Hamming distance), ties to the lowest train index, (-1, -1)
    when the train set is empty."""
    hd = aligner._hd
    hd.use_torch_stream()
    n = len(items)
    arr = (_lib.DfkMatchItem * max(n, 1))(*[_match_item(hd, it) for it in items])
    total = int(match_offsets(items)[-1])
    if out is None:
        out = torch.empty((max(total, 1), 2), dtype=torch.int32, device=f"cuda:{hd.device}")
    _check_tensor(hd, out, torch.int32, 2 * total, "out")
    check(hd.h, lib().dfk_hamming_match_batch(hd.h, arr, n, C.c_void_p(out.data_ptr())))
    return out[:total]


def ReprojectionMatchBatch(aligner, items: Sequence[dict]):
    """The match lists of many ReprojectionFactors in four launches (dfk_reprojection_match_batch): Hamming matching,
    eight-point RANSAC and distance pruning (reprojection_factor.cpp:56-65).  items are dicts with query / train
    (Features), cam (level 0) and optionally max_dist, max_iterations, threshold, probability (the rep_* defaults above)
    and seed (0).  Asynchronous: returns device tensors (matches [sum of query counts, 3] int32, counts [n] int32,
    ransac [n, 3] int32): item i's list is matches[offsets[i] : offsets[i] + counts[i]] (offsets = match_offsets(items)),
    rows (query index, train index, distance) sorted by (distance, query); ransac[i] = (selected hypothesis or -1, its
    inliers, hypotheses evaluated)."""
    hd = aligner._hd
    hd.use_torch_stream()
    n = len(items)
    for it in items:
        if it.get("cam") is None:
            raise ValueError("ReprojectionMatchBatch: every item needs its level-0 camera")
    arr = (_lib.DfkMatchItem * max(n, 1))(*[_match_item(hd, it) for it in items])
    total = int(match_offsets(items)[-1])
    dev = f"cuda:{hd.device}"
    matches = torch.zeros((max(total, 1), 3), dtype=torch.int32, device=dev)  # rows past an item's count stay 0
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    ransac = torch.empty((max(n, 1), 3), dtype=torch.int32, device=dev)
    check(hd.h, lib().dfk_reprojection_match_batch(hd.h, arr, n, C.c_void_p(matches.data_ptr()),
                                                   C.c_void_p(counts.data_ptr()), C.c_void_p(ransac.data_ptr())))
    return matches[:total], counts[:n], ransac[:n]


# ------------------------------------------------------------------------------------------- ORB features
# the reference's rep_nfeatures (deepfactors_options.h) and cv::ORB's default FAST threshold
REP_NFEATURES = 500
ORB_FAST_THRESHOLD = 20


@dataclass
class OrbBatch:
    """The device output of OrbDetectBatch: item i's rows are [offsets[i], offsets[i] + min(counts[i], capacity_i)),
    in the detector's order (response descending, then y, then x).  keypoints [rows, 2] float32, descriptors [rows, 32]
    uint8, angles [rows] float32 (degrees), responses [rows] float32, counts [n] int32 (the true counts)."""
    keypoints: torch.Tensor
    descriptors: torch.Tensor
    angles: torch.Tensor
    responses: torch.Tensor
    counts: torch.Tensor
    offsets: np.ndarray
    capacities: np.ndarray
    _call = "OrbDetectBatch"  # the call named by host_counts' error

    def host_counts(self) -> np.ndarray:
        """The counts on the host (synchronises with the stream); raises when an image's count exceeds its capacity,
        since its output then lacks the keypoints past the capacity"""
        c = self.counts.cpu().numpy().astype(np.int64)
        over = np.nonzero(c > self.capacities)[0]
        if len(over):
            i = int(over[0])
            raise RuntimeError(f"{self._call}: image {i} has {int(c[i])} keypoints (ties at the cut) but capacity "
                               f"{int(self.capacities[i])}; pass a larger capacity")
        return c

    def features(self) -> list:
        """One Features per image (views into the batch's tensors), ready for HammingMatchBatch /
        ReprojectionMatchBatch / window_opt.match_reprojection_links; one read-back of the counts"""
        c = self.host_counts()
        return [Features(self.keypoints[o:o + k], self.descriptors[o:o + k]) for o, k in zip(self.offsets[:-1], c)]


def _orb_image(t: torch.Tensor) -> DfkImage:
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8:
        raise TypeError("OrbDetectBatch: images must be uint8 CUDA tensors")
    if t.dim() != 2 or t.stride(1) != 1 or (t.shape[0] > 1 and t.stride(0) < t.shape[1]):
        raise ValueError("OrbDetectBatch: an image must be [H, W] with unit column stride")
    return DfkImage(C.c_void_p(t.data_ptr()), max(int(t.stride(0)), int(t.shape[1])), int(t.shape[1]),
                    int(t.shape[0]))


def OrbDetectBatch(aligner, images: Sequence[torch.Tensor], nfeatures: int = REP_NFEATURES,
                   fast_threshold: int = ORB_FAST_THRESHOLD, capacity: int | None = None) -> OrbBatch:
    """cv::ORB_create(nfeatures, 1.2, 1).detectAndCompute of many gray images in one call (dfk_orb_detect_batch): the
    reference's OrbDetector with rep_nlevels = 1, bit for bit.  images: uint8 [H, W] CUDA tensors of any sizes (below
    63 x 63 an image has no features).  nfeatures, fast_threshold and capacity (default 2 nfeatures: ties at the
    response cut can add keypoints) are one value for all images or one per image.  Asynchronous: returns an OrbBatch
    of device tensors; OrbBatch.features() splits it into per-image Features."""
    hd = aligner._hd
    hd.use_torch_stream()
    n = len(images)
    per = lambda v: [int(x) for x in (v if isinstance(v, (list, tuple, np.ndarray)) else [v] * n)]
    nf, t = per(nfeatures), per(fast_threshold)
    cap = per(capacity) if capacity is not None else [2 * x for x in nf]
    if not (len(nf) == len(t) == len(cap) == n):
        raise ValueError("OrbDetectBatch: per-image settings need one entry per image")
    for im in images:
        if im.device != torch.device("cuda", hd.device):
            raise ValueError(f"OrbDetectBatch: images must be on cuda:{hd.device}")
    arr = (_lib.DfkOrbItem * max(n, 1))(*[_lib.DfkOrbItem(_orb_image(im), a, b, c)
                                          for im, a, b, c in zip(images, nf, t, cap)])
    offsets = np.concatenate([[0], np.cumsum(cap)]).astype(np.int64)
    rows = int(offsets[-1])
    dev = f"cuda:{hd.device}"
    kp = torch.zeros((max(rows, 1), 2), dtype=torch.float32, device=dev)  # rows past a count stay 0
    desc = torch.zeros((max(rows, 1), 32), dtype=torch.uint8, device=dev)
    ang = torch.zeros(max(rows, 1), dtype=torch.float32, device=dev)
    resp = torch.zeros(max(rows, 1), dtype=torch.float32, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    check(hd.h, lib().dfk_orb_detect_batch(hd.h, arr, n, C.c_void_p(kp.data_ptr()), C.c_void_p(desc.data_ptr()),
                                           C.c_void_p(ang.data_ptr()), C.c_void_p(resp.data_ptr()),
                                           C.c_void_p(counts.data_ptr())))
    return OrbBatch(kp[:rows], desc[:rows], ang[:rows], resp[:rows], counts[:n], offsets, np.array(cap, np.int64))


@dataclass
class OrbPyramidBatch(OrbBatch):
    """The device output of OrbDetectPyramidBatch: OrbBatch's fields, item i's rows in level order (each level in the
    one-level order), keypoints at level 0, plus octaves [rows] int32 (each row's level)."""
    octaves: torch.Tensor = None
    _call = "OrbDetectPyramidBatch"


def OrbDetectPyramidBatch(aligner, images: Sequence[torch.Tensor], nfeatures: int = REP_NFEATURES,
                          scale_factor: float = 1.2, nlevels: int = 8, fast_threshold: int = ORB_FAST_THRESHOLD,
                          capacity: int | None = None) -> OrbPyramidBatch:
    """cv::ORB_create(nfeatures, scale_factor, nlevels).detectAndCompute of many gray images in one call
    (dfk_orb_detect_pyramid_batch): the reference's OrbDetector with rep_nlevels > 1, bit for bit.  images: uint8
    [H, W] CUDA tensors of any sizes; every setting is one value for all images or one per image, capacity by default
    2 nfeatures.  Asynchronous: returns an OrbPyramidBatch of device tensors; .features() feeds HammingMatchBatch,
    ReprojectionMatchBatch, window_opt.match_reprojection_links and BowTransformBatch as OrbDetectBatch's does."""
    hd = aligner._hd
    hd.use_torch_stream()
    n = len(images)
    per = lambda v, f=int: [f(x) for x in (v if isinstance(v, (list, tuple, np.ndarray)) else [v] * n)]
    nf, s, nl, t = per(nfeatures), per(scale_factor, float), per(nlevels), per(fast_threshold)
    cap = per(capacity) if capacity is not None else [2 * x for x in nf]
    if not (len(nf) == len(s) == len(nl) == len(t) == len(cap) == n):
        raise ValueError("OrbDetectPyramidBatch: per-image settings need one entry per image")
    for im in images:
        if im.device != torch.device("cuda", hd.device):
            raise ValueError(f"OrbDetectPyramidBatch: images must be on cuda:{hd.device}")
    arr = (_lib.DfkOrbPyramidItem * max(n, 1))(*[_lib.DfkOrbPyramidItem(_orb_image(im), a, b, c, d, e)
                                                 for im, a, b, c, d, e in zip(images, nf, s, nl, t, cap)])
    offsets = np.concatenate([[0], np.cumsum(cap)]).astype(np.int64)
    rows = int(offsets[-1])
    dev = f"cuda:{hd.device}"
    kp = torch.zeros((max(rows, 1), 2), dtype=torch.float32, device=dev)  # rows past a count stay 0
    desc = torch.zeros((max(rows, 1), 32), dtype=torch.uint8, device=dev)
    ang = torch.zeros(max(rows, 1), dtype=torch.float32, device=dev)
    resp = torch.zeros(max(rows, 1), dtype=torch.float32, device=dev)
    octv = torch.zeros(max(rows, 1), dtype=torch.int32, device=dev)
    counts = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    check(hd.h, lib().dfk_orb_detect_pyramid_batch(hd.h, arr, n, C.c_void_p(kp.data_ptr()),
                                                   C.c_void_p(desc.data_ptr()), C.c_void_p(ang.data_ptr()),
                                                   C.c_void_p(resp.data_ptr()), C.c_void_p(octv.data_ptr()),
                                                   C.c_void_p(counts.data_ptr())))
    return OrbPyramidBatch(kp[:rows], desc[:rows], ang[:rows], resp[:rows], counts[:n], offsets,
                           np.array(cap, np.int64), octv[:rows])


# ------------------------------------------------------------------------------------------- frame preprocessing
def resize_viewport(cam, w: int, h: int):
    """PinholeCamera::ResizeViewport (pinhole_camera_impl.h:126-136) in the reference's fp32 arithmetic: the camera of a
    frame of w x h pixels (orig_cam_ in PreprocessImage, deepfactors.cpp:638)"""
    from .synth import Camera
    return Camera(cam.fx, cam.fy, cam.u0, cam.v0, cam.width, cam.height).resized(int(w), int(h))


@dataclass
class PreprocessedFrame:
    """One frame's output of PreprocessBatch, device tensors: color uint8 [H_o, W_o, 3] (kf->color_img) and gray uint8
    [H_o, W_o] (OrbDetectBatch's image), or None when not asked for; levels float32 [h_l, w_l] (level 0 = f, or f'
    when normalised) and grads float32 [h_l, w_l, 2] (or None); stats float64 [2] = (mu, sigma) of a normalised
    frame, else None."""
    color: torch.Tensor | None
    gray: torch.Tensor | None
    levels: list
    grads: list | None
    stats: torch.Tensor | None


def _frame_view(t: torch.Tensor) -> DfkImage:
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8:
        raise TypeError("PreprocessBatch: frames must be uint8 CUDA tensors")
    if t.dim() != 3 or t.shape[2] != 3 or t.stride(2) != 1 or t.stride(1) != 3:
        raise ValueError("PreprocessBatch: a frame must be [H, W, 3] with interleaved contiguous pixels")
    return DfkImage(C.c_void_p(t.data_ptr()), int(t.stride(0)), int(t.shape[1]), int(t.shape[0]))


def pyramid_sizes(w: int, h: int, num_levels: int) -> list:
    """(w, h) of each level: integer halving (camera_pyramid.h:43-44)"""
    sizes = [(int(w), int(h))]
    for _ in range(1, num_levels):
        sizes.append((sizes[-1][0] // 2, sizes[-1][1] // 2))
    return sizes[:num_levels]


def PreprocessBatch(aligner, frames: Sequence[torch.Tensor], src_cams, out_cam, num_levels: int,
                    normalize=False, color: bool = True, gray: bool = True, grads: bool = True) -> list:
    """DeepFactors::PreprocessImage and the frame's image pyramid for many camera frames in one call
    (dfk_preprocess_batch): the remap to out_cam, the gray and float conversion bit for bit cv::remap / cv::cvtColor /
    convertTo, optionally the normalisation, then num_levels levels by GaussianBlurDown and their Sobel gradients.
    frames: uint8 [H, W, 3] CUDA tensors of any sizes; src_cams: the camera of each frame at its size (one for all, or
    one per frame; resize_viewport gives it); out_cam: the network camera, whose width x height is the output size;
    normalize: one bool for all frames or one per frame.  Asynchronous: returns one PreprocessedFrame per frame."""
    hd = aligner._hd
    hd.use_torch_stream()
    n = len(frames)
    cams = list(src_cams) if isinstance(src_cams, (list, tuple)) else [src_cams] * n
    norm = [bool(x) for x in normalize] if isinstance(normalize, (list, tuple, np.ndarray)) else [bool(normalize)] * n
    if len(cams) != n or len(norm) != n:
        raise ValueError("PreprocessBatch: per-frame settings need one entry per frame")
    W, H = int(out_cam.width), int(out_cam.height)
    if W != out_cam.width or H != out_cam.height or W < 1 or H < 1:
        raise ValueError("PreprocessBatch: the output camera's size must be whole numbers >= 1")
    dev = torch.device("cuda", hd.device)
    for f in frames:
        if f.device != dev:
            raise ValueError(f"PreprocessBatch: frames must be on cuda:{hd.device}")
    sizes = pyramid_sizes(W, H, num_levels)
    stats = torch.zeros((max(n, 1), 2), dtype=torch.float64, device=dev) if any(norm) else None
    out, items, keep = [], [], []
    for i, f in enumerate(frames):
        col = torch.empty((H, W, 3), dtype=torch.uint8, device=dev) if color else None
        gr = torch.empty((H, W), dtype=torch.uint8, device=dev) if gray else None
        lv = [torch.empty((h, w), dtype=torch.float32, device=dev) for w, h in sizes]
        gd = [torch.empty((h, w, 2), dtype=torch.float32, device=dev) for w, h in sizes] if grads else None
        la = (DfkImage * max(num_levels, 1))(*[_image(t) for t in lv])
        ga = (DfkImage * max(num_levels, 1))(*[_image(t, 2) for t in gd]) if grads else None
        keep += [la, ga]
        items.append(_lib.DfkPreprocessItem(
            _frame_view(f), _cam(cams[i]), _cam(out_cam),
            DfkImage(C.c_void_p(col.data_ptr()), 3 * W, W, H) if color else DfkImage(),
            DfkImage(C.c_void_p(gr.data_ptr()), W, W, H) if gray else DfkImage(),
            C.cast(la, C.POINTER(DfkImage)) if num_levels > 0 else None,
            C.cast(ga, C.POINTER(DfkImage)) if grads and num_levels > 0 else None, int(norm[i])))
        out.append(PreprocessedFrame(col, gr, lv, gd, stats[i] if norm[i] else None))
    arr = (_lib.DfkPreprocessItem * max(n, 1))(*items)
    check(hd.h, lib().dfk_preprocess_batch(hd.h, arr, n, int(num_levels),
                                           C.c_void_p(stats.data_ptr()) if stats is not None else None))
    return out


# ------------------------------------------------------------------------------------------- keyframe meshes
@dataclass
class KeyframeMeshParams:
    """The keyframe renderer's parameters (gui/visualizer.cpp:657-661)."""
    stdev_thresh: float = 4.2
    slt_thresh: float = 0.0
    crop_pix: int = 20
    draw_noisy_pixels: bool = False

    def to_c(self) -> "_lib.DfkKeyframeMeshParams":
        return _lib.DfkKeyframeMeshParams(self.stdev_thresh, self.slt_thresh, int(self.crop_pix),
                                          int(bool(self.draw_noisy_pixels)))


@dataclass
class KeyframeMesh:
    """One keyframe's mesh: views into a KeyframeMeshes batch (None where the batch has no such output).  positions
    and normals float32 [V, 3] in the world frame, colors uint8 [V, 3], pixels int32 [V] (y W + x), triangles int32
    [T, 3] of item-local vertex indices.  overflow: the item's counts exceed its capacities, so it has no rows."""
    positions: torch.Tensor
    normals: torch.Tensor | None
    colors: torch.Tensor | None
    pixels: torch.Tensor | None
    triangles: torch.Tensor | None
    num_vertices: int
    num_triangles: int
    overflow: bool


@dataclass
class KeyframeMeshes:
    """The device output of KeyframeMeshBatch: item i's vertex rows start at vertex_offsets[i] and its triangle rows at
    triangle_offsets[i] (the capacities of the items before it); counts int32 [n, 2] holds each item's true vertex and
    triangle counts; depth_u16[i] is item i's uint16 [H, W] depth image, or None."""
    positions: torch.Tensor
    normals: torch.Tensor | None
    colors: torch.Tensor | None
    pixels: torch.Tensor | None
    triangles: torch.Tensor | None
    counts: torch.Tensor
    vertex_offsets: np.ndarray
    triangle_offsets: np.ndarray
    depth_u16: list

    def meshes(self) -> list:
        """One KeyframeMesh per item (one read-back of the counts)"""
        c = self.counts.cpu().numpy().astype(np.int64)
        out = []
        for i, (nv, nt) in enumerate(c):
            vo, to = int(self.vertex_offsets[i]), int(self.triangle_offsets[i])
            over = nv > self.vertex_offsets[i + 1] - vo or nt > self.triangle_offsets[i + 1] - to
            v, t = (0, 0) if over else (int(nv), int(nt))
            sl = lambda a, o, k: None if a is None else a[o:o + k]
            out.append(KeyframeMesh(sl(self.positions, vo, v), sl(self.normals, vo, v), sl(self.colors, vo, v),
                                    sl(self.pixels, vo, v), sl(self.triangles, to, t), int(nv), int(nt), bool(over)))
        return out


def _u8_view(t: torch.Tensor, channels: int, what: str) -> DfkImage:
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8:
        raise TypeError(f"KeyframeMeshBatch: {what} must be a uint8 CUDA tensor")
    if t.dim() != 3 or t.shape[2] != channels or t.stride(2) != 1 or t.stride(1) != channels:
        raise ValueError(f"KeyframeMeshBatch: {what} must be [H, W, {channels}] with interleaved contiguous pixels")
    return DfkImage(C.c_void_p(t.data_ptr()), int(t.stride(0)), int(t.shape[1]), int(t.shape[0]))


def KeyframeMeshBatch(aligner, items: Sequence[dict], params: KeyframeMeshParams | None = None,
                      code_size: int | None = None, normals: bool = True, pixels: bool = True,
                      triangles: bool = True) -> KeyframeMeshes:
    """What the keyframe renderer (gui/shaders/drawkf.geom) draws for many keyframes, as world-frame meshes, in one call
    (dfk_keyframe_mesh_batch).  items are dicts with cam (the keyframe's camera, whose size is every view's), pose_wk
    (7 floats), the depth as dpt (float32 [H, W], pyr_dpt level 0) or as prx_orig, prx_jac and a host code (decoded
    bit for bit as UpdateDepthBatch decodes it, avg_dpt the aligner's), and optionally std (log-stdev), valid (float32
    [H, W]), color (uint8 [H, W, 3]), vertex_capacity (default H W), triangle_capacity (default 2 H W) and depth_u16
    (True: also return SaveKeyframes' uint16 depth image).  Colours are returned when every item has a color view.
    code_size defaults to the aligner's.  Asynchronous: returns a KeyframeMeshes of device tensors."""
    hd = aligner._hd
    hd.use_torch_stream()
    params = params or KeyframeMeshParams()
    cs = int(code_size if code_size is not None else getattr(aligner, "CS", 0))
    n = len(items)
    dev = torch.device("cuda", hd.device)
    arr = (_lib.DfkKeyframeMeshItem * max(n, 1))()
    keep, u16s, vcap, tcap = [], [], [], []
    with_colors = n > 0 and all(it.get("color") is not None for it in items)
    for k, it in enumerate(items):
        cam = it["cam"]
        W, H = int(cam.width), int(cam.height)
        a = arr[k]
        a.cam = _cam(cam)
        a.pose_wk = _pose(it["pose_wk"])
        if it.get("dpt") is not None:
            a.dpt = _image(it["dpt"])
        else:
            code = np.ascontiguousarray(it["code"], dtype=np.float32)
            if code.shape != (cs,):
                raise ValueError(f"KeyframeMeshBatch: item {k}'s code must have code_size = {cs} entries")
            keep.append(code)
            a.prx_orig, a.prx_jac = _image(it["prx_orig"]), _image(it["prx_jac"], cs)
            a.code = code.ctypes.data_as(C.POINTER(C.c_float))
        if it.get("std") is not None:
            a.std = _image(it["std"])
        if it.get("valid") is not None:
            a.valid = _image(it["valid"])
        if it.get("color") is not None:
            a.color = _u8_view(it["color"], 3, "color")
        vcap.append(int(it.get("vertex_capacity", W * H)))
        tcap.append(int(it.get("triangle_capacity", 2 * W * H)))
        a.vertex_capacity, a.triangle_capacity = vcap[-1], tcap[-1]
        u16 = torch.empty((H, W), dtype=torch.uint16, device=dev) if it.get("depth_u16") else None
        if u16 is not None:
            a.depth_u16 = DfkImage(C.c_void_p(u16.data_ptr()), 2 * W, W, H)
        u16s.append(u16)
    vo = np.concatenate([[0], np.cumsum(vcap)]).astype(np.int64)
    to = np.concatenate([[0], np.cumsum(tcap)]).astype(np.int64)
    V, T = int(vo[-1]), int(to[-1])
    pos = torch.zeros((max(V, 1), 3), dtype=torch.float32, device=dev)  # rows past a count stay 0
    nrm = torch.zeros((max(V, 1), 3), dtype=torch.float32, device=dev) if normals else None
    col = torch.zeros((max(V, 1), 3), dtype=torch.uint8, device=dev) if with_colors else None
    pix = torch.zeros(max(V, 1), dtype=torch.int32, device=dev) if pixels else None
    tri = torch.zeros((max(T, 1), 3), dtype=torch.int32, device=dev) if triangles else None
    counts = torch.empty((max(n, 1), 2), dtype=torch.int32, device=dev)
    ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    prm = params.to_c()
    check(hd.h, lib().dfk_keyframe_mesh_batch(hd.h, arr, n, cs, C.byref(prm), ptr(pos), ptr(nrm), ptr(col), ptr(pix),
                                              ptr(tri), ptr(counts)))
    cut = lambda t, r: None if t is None else t[:r]
    return KeyframeMeshes(pos[:V], cut(nrm, V), cut(col, V), cut(pix, V), cut(tri, T), counts[:n], vo, to, u16s)


def write_ply(path, meshes: KeyframeMeshes, items=None) -> None:
    """Writes the meshes of KeyframeMeshBatch to one binary little-endian PLY file: vertices x y z (nx ny nz when the
    batch has normals, red green blue when it has colours), faces as `list uchar int vertex_indices` when it has
    triangles.  items: the item indices to write (default all), concatenated in that order with their triangles'
    indices offset by the vertices before them.  Raises when a written item overflowed its capacities."""
    ms = meshes.meshes()
    idx = range(len(ms)) if items is None else [int(i) for i in items]
    for i in idx:
        if ms[i].overflow:
            raise RuntimeError(f"write_ply: item {i} has {ms[i].num_vertices} vertices and {ms[i].num_triangles} "
                               "triangles, more than its capacities; call KeyframeMeshBatch again with larger ones")
    fields = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if meshes.normals is not None:
        fields += [("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    if meshes.colors is not None:
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    verts, faces, base = [], [], 0
    for i in idx:
        m = ms[i]
        v = np.zeros(m.num_vertices, dtype=fields)
        p = m.positions.cpu().numpy()
        v["x"], v["y"], v["z"] = p[:, 0], p[:, 1], p[:, 2]
        if m.normals is not None:
            q = m.normals.cpu().numpy()
            v["nx"], v["ny"], v["nz"] = q[:, 0], q[:, 1], q[:, 2]
        if m.colors is not None:
            c = m.colors.cpu().numpy()
            v["red"], v["green"], v["blue"] = c[:, 0], c[:, 1], c[:, 2]
        verts.append(v)
        if m.triangles is not None:
            f = np.zeros(m.num_triangles, dtype=[("n", "u1"), ("v", "<i4", (3,))])
            f["n"] = 3
            f["v"] = m.triangles.cpu().numpy().astype(np.int64) + base
            faces.append(f)
        base += m.num_vertices
    vall = np.concatenate(verts) if verts else np.zeros(0, dtype=fields)
    names = {"<f4": "float", "u1": "uchar"}
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(vall)}"]
    head += [f"property {names[t]} {nm}" for nm, t in fields]
    if meshes.triangles is not None:
        fall = np.concatenate(faces) if faces else np.zeros(0, dtype=[("n", "u1"), ("v", "<i4", (3,))])
        head += [f"element face {len(fall)}", "property list uchar int vertex_indices"]
    head.append("end_header")
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(vall.tobytes())
        if meshes.triangles is not None:
            fh.write(fall.tobytes())


def SparseGeometricErrorBatch(aligner, items, out: torch.Tensor | None = None) -> torch.Tensor:
    """SparseGeometricFactor::error of many factors in one launch (dfk_sparse_geometric_error_batch): the items of
    SparseGeometricLinearizeBatch (dicts, or the array of make_geometric_items).  Asynchronous: returns a device tensor [n, 2] float32, row i = [b^T b | valid points
    as uint32 bits], b^T b bit for bit the residual of factor i's SparseGeometricLinearizeBatch record."""
    aligner._hd.use_torch_stream()
    cs, n = aligner.CS, len(items)
    out = _batch_records(aligner, n, 2, out)
    arr = items if isinstance(items, C.Array) else make_geometric_items(items, cs)
    check(aligner.handle, lib().dfk_sparse_geometric_error_batch(aligner.handle, arr, n, cs, C.c_void_p(out.data_ptr())))
    return out


# ------------------------------------------------------------------------------------------- DepthAligner
class DepthAligner:
    """df::DepthAligner<float, CS> (sources/cuda/cu_depthaligner.h:38-54): code-only alignment of the decoded depth to a
    target depth map; the result is a JTJJrReductionItem over the CS code parameters.  The decode uses
    params.sfmparams.avg_dpt (default 2, the value the reference hard-codes in this kernel)."""

    def __init__(self, code_size: int, device=None, params: SfmAlignerParams | None = None):
        self.CS = int(code_size)
        self._hd = _Handle(device)
        if params is not None:
            cp = params.to_c()
            check(self._hd.h, lib().dfk_sfm_set_params(self._hd.h, C.byref(cp)))

    @property
    def handle(self):
        return self._hd.h

    def RunStep(self, code, target_dpt, prx_orig, prx_jac) -> JTJJrReductionItem:
        self._hd.use_torch_stream()
        code = np.ascontiguousarray(code, dtype=np.float32)
        if code.shape != (self.CS,):
            raise ValueError(f"code must have {self.CS} entries")
        nh = self.CS * (self.CS + 1) // 2
        JtJ = np.zeros(nh, dtype=np.float32)
        Jtr = np.zeros(self.CS, dtype=np.float32)
        res, inl = C.c_float(0), C.c_uint64(0)
        t, p, j = _image(target_dpt), _image(prx_orig), _image(prx_jac, self.CS)
        FP = C.POINTER(C.c_float)
        check(self._hd.h, lib().dfk_depth_run_step(self._hd.h, code.ctypes.data_as(FP), self.CS, C.byref(t), C.byref(p),
                                                  C.byref(j), JtJ.ctypes.data_as(FP), Jtr.ctypes.data_as(FP),
                                                  C.byref(res), C.byref(inl)))
        return JTJJrReductionItem(JtJ, Jtr, float(res.value), int(inl.value))


# ------------------------------------------------------------------------------------------- keyframe window
class Window:
    """Device-side assembly of a keyframe window's block-sparse normal equations (dfk_window_* of include/dfk.h):
    what the factor graph does with the RunStep records of a window -- PhotometricFactor::linearize's block slicing,
    sign flip and residual rescale (sources/core/gtsam/photometric_factor.cpp:105-161,275-282) summed over the window's
    factors (one per pair and level, core/mapping/df_work.cpp:211-225).  `layout` (factors.WindowBlocks) describes the
    buffer; it is the one buffer a multi-GPU Gauss-Newton step all-reduces.  `geometric` lists the window's sparse
    geometric links (k0, k1), one record each (SparseGeometricLinearizeBatch); their blocks follow the scalars.
    `num_frames` tracked frames (pose-only variables, dfk_window_create_frames): a pair (k, K + f) is frame f's one
    photometric pair; the frames' blocks follow the links'.  `kf_priors` lists the keyframes of each keyframe prior
    (dfk_window_create_priors, ascending lists); their prior blocks follow the frames'."""

    def __init__(self, aligner: "SfmAligner", num_keyframes: int, pairs, item_pair, item_sizes, geometric=(),
                 num_frames: int = 0, kf_priors=()):
        from .factors import WindowBlocks
        self._al = aligner
        self.layout = WindowBlocks(int(num_keyframes), aligner.CS, [tuple(map(int, p)) for p in pairs],
                                   [tuple(map(int, p)) for p in geometric], int(num_frames),
                                   [tuple(int(k) for k in p) for p in kf_priors])
        k0 = np.ascontiguousarray([p[0] for p in self.layout.pairs], dtype=np.int32)
        k1 = np.ascontiguousarray([p[1] for p in self.layout.pairs], dtype=np.int32)
        ip = np.ascontiguousarray(item_pair, dtype=np.int32)
        self.item_pair = ip.copy()
        iw = np.ascontiguousarray([s[0] for s in item_sizes], dtype=np.int32)
        ih = np.ascontiguousarray([s[1] for s in item_sizes], dtype=np.int32)
        I32 = C.POINTER(C.c_int32)
        desc = _lib.DfkWindowDesc(int(num_keyframes), len(k0), len(ip), aligner.CS, k0.ctypes.data_as(I32),
                                  k1.ctypes.data_as(I32), ip.ctypes.data_as(I32), iw.ctypes.data_as(I32),
                                  ih.ctypes.data_as(I32))
        g0 = np.ascontiguousarray([p[0] for p in self.layout.geometric], dtype=np.int32)
        g1 = np.ascontiguousarray([p[1] for p in self.layout.geometric], dtype=np.int32)
        L = len(g0)
        self.w = C.c_void_p()
        kp = self.layout.kf_priors
        if kp:
            pp = np.ascontiguousarray(np.cumsum([0] + [len(p) for p in kp]), dtype=np.int32)
            pk = np.ascontiguousarray([k for p in kp for k in p], dtype=np.int32)
            check(aligner.handle, lib().dfk_window_create_priors(aligner.handle, C.byref(desc), L,
                                                                 g0.ctypes.data_as(I32) if L else None,
                                                                 g1.ctypes.data_as(I32) if L else None, int(num_frames),
                                                                 len(kp), pp.ctypes.data_as(I32),
                                                                 pk.ctypes.data_as(I32), C.byref(self.w)))
        else:
            check(aligner.handle, lib().dfk_window_create_frames(aligner.handle, C.byref(desc), L,
                                                                 g0.ctypes.data_as(I32) if L else None,
                                                                 g1.ctypes.data_as(I32) if L else None, int(num_frames),
                                                                 C.byref(self.w)))
        # doubles of each keyframe prior and of its deltas, and where each starts in the back-to-back buffers
        self.kf_prior_sizes = [_lib.kf_prior_doubles(aligner.CS, len(p)) for p in kp]
        self.kf_prior_doubles = int(sum(self.kf_prior_sizes))
        self.kf_delta_doubles = int(sum(len(p) for p in kp)) * self.layout.B
        self.num_items = len(ip)
        self.floats = int(lib().dfk_window_floats(self.w))
        assert self.floats == self.layout.floats

    def assemble(self, records: torch.Tensor, out: torch.Tensor | None = None,
                 geo_records: torch.Tensor | None = None) -> torch.Tensor:
        """records: [num_items, REC] device tensor written by RunStepBatch; geo_records: [num_links, GEO_REC] written by
        SparseGeometricLinearizeBatch (required when the window has links).  Asynchronous on torch's current stream."""
        hd = self._al._hd
        hd.use_torch_stream()
        _check_tensor(hd, records, torch.float32, self.num_items * _lib.record_floats(self.layout.code_size), "records")
        if out is None:
            out = torch.empty(self.floats, dtype=torch.float32, device=records.device)
        _check_tensor(hd, out, torch.float32, self.floats, "out")
        if self.layout.geometric and geo_records is None:
            raise ValueError("the window has geometric links: geo_records is required")
        geo = None
        if geo_records is not None:
            _check_tensor(hd, geo_records, torch.float32,
                          len(self.layout.geometric) * _lib.geo_record_floats(self.layout.code_size), "geo_records")
            geo = C.c_void_p(geo_records.data_ptr())
        check(hd.h, lib().dfk_window_assemble_geometric(hd.h, self.w, C.c_void_p(records.data_ptr()), geo,
                                                        C.c_void_p(out.data_ptr())))
        return out

    def marginalize_frames(self, records: torch.Tensor, frames, priors: torch.Tensor | None = None,
                           info: torch.Tensor | None = None):
        """dfk_window_marginalize_frames: the linear prior each listed frame leaves on its keyframe (the Schur complement
        of the frame's pose in its pair's records, undamped).  records: [num_items, REC] on the device.  Returns
        (priors [n, DFK_PRIOR_DOUBLES] float64, info [n] int32), device tensors written asynchronously on torch's
        current stream; info[i] = 0, or 1 + the row of the frame block whose pivot failed (prior i is then zero)."""
        hd = self._al._hd
        hd.use_torch_stream()
        _check_tensor(hd, records, torch.float32, self.num_items * _lib.record_floats(self.layout.code_size), "records")
        fr = np.ascontiguousarray([int(f) for f in frames], dtype=np.int32)
        n, pd = len(fr), _lib.prior_doubles(self.layout.code_size)
        if priors is None:
            priors = torch.empty((n, pd), dtype=torch.float64, device=records.device)
        _check_tensor(hd, priors, torch.float64, n * pd, "priors")
        if info is None:
            info = torch.empty(n, dtype=torch.int32, device=records.device)
        _check_tensor(hd, info, torch.int32, n, "info")
        check(hd.h, lib().dfk_window_marginalize_frames(hd.h, self.w, C.c_void_p(records.data_ptr()), n,
                                                        fr.ctypes.data_as(C.POINTER(C.c_int32)),
                                                        C.c_void_p(priors.data_ptr()), C.c_void_p(info.data_ptr())))
        return priors, info

    def add_priors(self, buf: torch.Tensor, prior_kf, priors: torch.Tensor, delta: torch.Tensor) -> torch.Tensor:
        """dfk_window_add_priors, in place on an assembled buffer: prior i (a row of `priors`, [m, DFK_PRIOR_DOUBLES]
        float64 on the device) on keyframe prior_kf[i] at delta[i] ([m, B] float64 on the device) = Local(x0_i, x).
        With sharded pairs, call it after the all-reduce.  Asynchronous on torch's current stream."""
        hd = self._al._hd
        hd.use_torch_stream()
        kf = np.ascontiguousarray([int(k) for k in prior_kf], dtype=np.int32)
        m, B = len(kf), self.layout.B
        _check_tensor(hd, buf, torch.float32, self.floats, "buf")
        _check_tensor(hd, priors, torch.float64, m * _lib.prior_doubles(self.layout.code_size), "priors")
        _check_tensor(hd, delta, torch.float64, m * B, "delta")
        check(hd.h, lib().dfk_window_add_priors(hd.h, self.w, m, kf.ctypes.data_as(C.POINTER(C.c_int32)),
                                                C.c_void_p(priors.data_ptr()), C.c_void_p(delta.data_ptr()),
                                                C.c_void_p(buf.data_ptr())))
        return buf

    def add_keyframe_priors(self, buf: torch.Tensor, priors: torch.Tensor, delta: torch.Tensor) -> torch.Tensor:
        """dfk_window_add_keyframe_priors, in place on an assembled buffer: the window's keyframe priors back to back in
        `priors` (float64 on the device, kf_prior_doubles entries) at `delta` (float64, kf_delta_doubles: Local(x0, x) of
        every member, prior by prior).  With sharded pairs, call it after the all-reduce.  Asynchronous on torch's current
        stream."""
        hd = self._al._hd
        hd.use_torch_stream()
        _check_tensor(hd, buf, torch.float32, self.floats, "buf")
        if not self.layout.kf_priors:
            return buf
        _check_tensor(hd, priors, torch.float64, self.kf_prior_doubles, "priors")
        _check_tensor(hd, delta, torch.float64, self.kf_delta_doubles, "delta")
        check(hd.h, lib().dfk_window_add_keyframe_priors(hd.h, self.w, C.c_void_p(priors.data_ptr()),
                                                         C.c_void_p(delta.data_ptr()), C.c_void_p(buf.data_ptr())))
        return buf

    def blanket(self, m: int):
        """dfk_window_blanket: the ascending keyframes that share a factor with keyframe m"""
        out = np.zeros(max(self.layout.num_keyframes, 1), dtype=np.int32)
        n = C.c_int32(0)
        check(self._al.handle, lib().dfk_window_blanket(self._al.handle, self.w, int(m),
                                                        out.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(n)))
        return [int(k) for k in out[:n.value]]

    def marginalize_keyframe(self, records: torch.Tensor, m: int, geo_records: torch.Tensor | None = None,
                             frame_priors: torch.Tensor | None = None, frame_delta: torch.Tensor | None = None,
                             kf_priors: torch.Tensor | None = None, kf_delta: torch.Tensor | None = None,
                             code_prior_weight: float = 0.0, code=None, prior: torch.Tensor | None = None,
                             info: torch.Tensor | None = None):
        """dfk_window_marginalize_keyframe: the keyframe prior over blanket(m) that eliminating keyframe m leaves (the
        Schur complement of m's [pose | code], undamped, of every factor touching m).  records / geo_records: the
        window's records on the device; frame_priors [r, DFK_PRIOR_DOUBLES] / frame_delta [r, B]: the frame priors on m
        and their deltas; kf_priors / kf_delta: the window's keyframe priors as add_keyframe_priors takes them (needed
        when one contains m); code_prior_weight / code (host, C): the zero-code prior on m.  Returns (prior
        [DFK_KF_PRIOR_DOUBLES(C, n)] float64, info [1] int32), device tensors written asynchronously on torch's current
        stream; info = 0, or 1 + the row of m's block whose pivot failed (the prior is then zero)."""
        hd = self._al._hd
        hd.use_torch_stream()
        cs, B = self.layout.code_size, self.layout.B
        _check_tensor(hd, records, torch.float32, self.num_items * _lib.record_floats(cs), "records")
        geo = None
        if geo_records is not None:
            _check_tensor(hd, geo_records, torch.float32, len(self.layout.geometric) * _lib.geo_record_floats(cs),
                          "geo_records")
            geo = C.c_void_p(geo_records.data_ptr())
        r = 0
        if frame_priors is not None:
            r = frame_priors.numel() // _lib.prior_doubles(cs)
            _check_tensor(hd, frame_priors, torch.float64, r * _lib.prior_doubles(cs), "frame_priors")
            _check_tensor(hd, frame_delta, torch.float64, r * B, "frame_delta")
        if kf_priors is not None:
            _check_tensor(hd, kf_priors, torch.float64, self.kf_prior_doubles, "kf_priors")
            _check_tensor(hd, kf_delta, torch.float64, self.kf_delta_doubles, "kf_delta")
        n = len(self.blanket(m))
        dev = records.device
        if prior is None:
            prior = torch.empty(_lib.kf_prior_doubles(cs, n), dtype=torch.float64, device=dev)
        _check_tensor(hd, prior, torch.float64, _lib.kf_prior_doubles(cs, n), "prior")
        if info is None:
            info = torch.empty(1, dtype=torch.int32, device=dev)
        _check_tensor(hd, info, torch.int32, 1, "info")
        cp = None
        if code_prior_weight > 0:
            c64 = np.ascontiguousarray(code, dtype=np.float64).reshape(-1)
            if c64.shape != (cs,):
                raise ValueError(f"code must have {cs} entries")
            cp = c64.ctypes.data_as(C.POINTER(C.c_double))
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        check(hd.h, lib().dfk_window_marginalize_keyframe(
            hd.h, self.w, C.c_void_p(records.data_ptr()), geo, int(m), r, ptr(frame_priors) if r else None,
            ptr(frame_delta) if r else None, ptr(kf_priors), ptr(kf_delta), float(code_prior_weight), cp,
            C.c_void_p(prior.data_ptr()), C.c_void_p(info.data_ptr())))
        return prior, info

    def close(self):
        if getattr(self, "w", None):
            lib().dfk_window_destroy(self._al.handle, self.w)
            self.w = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class WindowSolver:
    """Damped block-sparse fp64 Cholesky of a Window's normal equations on the device (dfk_window_solve): the system
    WindowOptimizer solves with to_dense + damped_solve, straight from the packed buffer.  `fixed` lists the window
    variables k * B + r held at zero (e.g. range(6): the gauge keyframe's pose).  `tiles` is the number of structurally
    nonzero B x B tiles of the factor, fill included.  With tracked frames dx has K * B + 6 F entries (frame f's pose
    at K * B + 6 f)."""

    def __init__(self, window: Window, fixed=()):
        self._win = window  # keeps the window (and its handle) alive
        self._al = window._al
        self.layout = window.layout
        fx = np.ascontiguousarray([int(v) for v in fixed], dtype=np.int32)
        self.fixed = tuple(int(v) for v in fx)
        self.s = C.c_void_p()
        check(self._al.handle, lib().dfk_window_solver_create(self._al.handle, window.w, len(fx),
                                                              fx.ctypes.data_as(C.POINTER(C.c_int32)), C.byref(self.s)))
        tiles = C.c_size_t(0)
        check(self._al.handle, lib().dfk_window_solver_tiles(self._al.handle, self.s, C.byref(tiles)))
        self.tiles = int(tiles.value)

    def solve(self, buf: torch.Tensor, lam: float, code_prior_weight: float = 0.0, codes=None,
              dx: torch.Tensor | None = None, info: torch.Tensor | None = None):
        """buf: the window buffer (contiguous float32 on the handle's device).  codes: [K, C] (host), required when
        code_prior_weight > 0.  Returns (dx [K * B + 6 F] float64, info [1] int32), device tensors written asynchronously on
        torch's current stream; info = 0, or 1 + the first variable whose pivot was not positive (dx is then zero)."""
        hd = self._al._hd
        hd.use_torch_stream()
        n = self.layout.dim
        _check_tensor(hd, buf, torch.float32, self.layout.floats, "buf")
        if dx is None:
            dx = torch.empty(n, dtype=torch.float64, device=buf.device)
        _check_tensor(hd, dx, torch.float64, n, "dx")
        if info is None:
            info = torch.empty(1, dtype=torch.int32, device=buf.device)
        _check_tensor(hd, info, torch.int32, 1, "info")
        cp = None
        if code_prior_weight > 0:
            if codes is None:
                raise ValueError("code_prior_weight > 0 needs the codes")
            c64 = np.ascontiguousarray(codes, dtype=np.float64)
            if c64.shape != (self.layout.num_keyframes, self.layout.code_size):
                raise ValueError(f"codes must be [{self.layout.num_keyframes}, {self.layout.code_size}]")
            cp = c64.ctypes.data_as(C.POINTER(C.c_double))
        prm = _lib.DfkWindowSolveParams(float(lam), float(code_prior_weight))
        check(self._al.handle, lib().dfk_window_solve(self._al.handle, self.s, C.c_void_p(buf.data_ptr()), C.byref(prm),
                                                      cp, C.c_void_p(dx.data_ptr()), C.c_void_p(info.data_ptr())))
        return dx, info

    def close(self):
        if getattr(self, "s", None):
            lib().dfk_window_solver_destroy(self._al.handle, self.s)
            self.s = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class WindowProblem:
    """A window problem of the C ABI (dfk_window_problem_*): every work item of a window held on the device once, the
    window's state (poses and codes, fp64) on the device, and the Levenberg-Marquardt loop as one call (dfk_window_lm).
    Item arrays are the ctypes arrays of make_work_items / make_reprojection_items / make_geometric_items /
    make_depth_items (their poses and codes are ignored); slots are [n, 4] ints (pose0, pose1, code0, code1; -1 where
    unused); records / geo_records are the caller's record buffers, which linearize writes.  The problem keeps every
    array it was given alive (the image views inside them must stay valid)."""

    def __init__(self, window: Window, records: torch.Tensor, geo_records=None, dense=None, dense_slots=(),
                 reproj=None, reproj_slots=(), geo=None, geo_slots=(), depth=None, depth_slots=(), error=None,
                 error_slots=(), error_depth=(), frame_prior_kf=(), frame_prior_rows=None, frame_prior_x0=None,
                 kf_prior_rows=None, kf_prior_x0=None):
        self._win = window
        self._al = window._al
        self.layout = window.layout
        keep = [records, geo_records, dense, reproj, geo, depth, error]
        S = _lib.DfkWindowItemSlots

        def slots(rows):
            a = np.ascontiguousarray(np.asarray(rows, dtype=np.int32).reshape(-1, 4))
            keep.append(a)
            return len(a), (a.ctypes.data_as(C.POINTER(S)) if len(a) else None)

        def f64(x):
            if x is None:
                return None
            a = np.ascontiguousarray(np.asarray(x, dtype=np.float64).ravel())
            keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_double))

        def i32(x):
            a = np.ascontiguousarray(np.asarray(x, dtype=np.int32).ravel())
            keep.append(a)
            return a.ctypes.data_as(C.POINTER(C.c_int32)) if a.size else None

        nd, ds = slots(dense_slots)
        nr, rs = slots(reproj_slots)
        ng, gs = slots(geo_slots)
        ndep, dps = slots(depth_slots)
        ne, es = slots(error_slots)
        mf = len(frame_prior_kf)
        d = _lib.DfkWindowProblemDesc(
            window.w, nd, dense if nd else None, ds, nr, reproj if nr else None, rs, ng, geo if ng else None, gs,
            ndep, depth if ndep else None, dps, ne, error if ne else None, es, i32(error_depth), mf, i32(frame_prior_kf),
            f64(frame_prior_rows), f64(frame_prior_x0), f64(kf_prior_rows), f64(kf_prior_x0),
            C.c_void_p(records.data_ptr()), C.c_void_p(geo_records.data_ptr()) if geo_records is not None else None)
        self._keep = keep
        self.p = C.c_void_p()
        self._al._hd.use_torch_stream()
        check(self._al.handle, lib().dfk_window_problem_create(self._al.handle, C.byref(d), C.byref(self.p)))
        L = self.layout
        self.num_poses, self.num_codes = L.num_keyframes + L.num_frames, L.num_keyframes * L.code_size
        self.num_dense, self.num_error = nd, ne

    def set_state(self, poses, codes):
        """poses [(K + F), 7] (keyframes then frames), codes [K, C]: host arrays or device tensors (float64)"""
        hd = self._al._hd
        hd.use_torch_stream()
        args, keep = [], []
        for x, n in ((poses, self.num_poses * 7), (codes, self.num_codes)):
            if isinstance(x, torch.Tensor):
                _check_tensor(hd, x, torch.float64, n, "state")
                args.append(C.c_void_p(x.data_ptr()))
            else:
                a = np.ascontiguousarray(np.asarray(x, dtype=np.float64))
                if a.size != n:
                    raise ValueError(f"the state is {self.num_poses} poses and a [K, C] code array")
                keep.append(a)
                args.append(a.ctypes.data_as(C.c_void_p))
        check(hd.h, lib().dfk_window_problem_set_state(hd.h, self.p, *args))

    def get_state(self):
        """(poses [(K + F), 7], codes [K, C]) float64 host arrays"""
        self._al._hd.use_torch_stream()
        P = np.zeros((self.num_poses, 7))
        Q = np.zeros((self.layout.num_keyframes, self.layout.code_size))
        check(self._al.handle, lib().dfk_window_problem_get_state(self._al.handle, self.p, P.ctypes.data_as(C.c_void_p),
                                                                   Q.ctypes.data_as(C.c_void_p)))
        check(self._al.handle, lib().dfk_synchronize(self._al.handle))
        return P, Q

    def linearize(self, out: torch.Tensor | None = None) -> torch.Tensor:
        """dfk_window_problem_linearize: the window buffer at the state (asynchronous on torch's current stream)"""
        hd = self._al._hd
        hd.use_torch_stream()
        if out is None:
            out = torch.empty(self._win.floats, dtype=torch.float32, device=f"cuda:{hd.device}")
        _check_tensor(hd, out, torch.float32, self._win.floats, "out")
        check(hd.h, lib().dfk_window_problem_linearize(hd.h, self.p, C.c_void_p(out.data_ptr())))
        return out

    def error(self, out: torch.Tensor | None = None) -> torch.Tensor:
        """dfk_window_problem_error: [E | photometric | reprojection | geometric | priors | items without inliers |
        inliers] float64 on the device (asynchronous)"""
        hd = self._al._hd
        hd.use_torch_stream()
        if out is None:
            out = torch.empty(_lib.WINDOW_ERROR_DOUBLES, dtype=torch.float64, device=f"cuda:{hd.device}")
        _check_tensor(hd, out, torch.float64, _lib.WINDOW_ERROR_DOUBLES, "out")
        check(hd.h, lib().dfk_window_problem_error(hd.h, self.p, C.c_void_p(out.data_ptr())))
        return out

    def retract(self, dx: torch.Tensor):
        """dfk_window_problem_retract: state <- retract(state, dx), dx [K B + 6 F] float64 on the device"""
        hd = self._al._hd
        hd.use_torch_stream()
        _check_tensor(hd, dx, torch.float64, self.layout.dim, "dx")
        check(hd.h, lib().dfk_window_problem_retract(hd.h, self.p, C.c_void_p(dx.data_ptr())))

    def lm(self, params, use_error: bool = False) -> dict:
        """dfk_window_lm with window_opt.LMParams; returns the trace as a dict"""
        hd = self._al._hd
        hd.use_torch_stream()
        it = int(params.iterations)
        prm = _lib.DfkLMParams(it, float(params.lambda_init), float(params.lambda_up), float(params.lambda_down),
                               float(params.lambda_max), int(bool(params.fix_first_pose)),
                               float(params.code_prior_weight), int(bool(use_error)))
        e, lam, acc = np.zeros(it + 1), np.zeros(max(it, 1)), np.zeros(max(it, 1), dtype=np.int32)
        tr = _lib.DfkLMTrace(e.ctypes.data_as(C.POINTER(C.c_double)), lam.ctypes.data_as(C.POINTER(C.c_double)),
                             acc.ctypes.data_as(C.POINTER(C.c_int32)), 0, 0, 0, 0)
        check(hd.h, lib().dfk_window_lm(hd.h, self.p, C.byref(prm), C.byref(tr)))
        return dict(energy=e[:tr.num_energies].tolist(), lam=lam[:tr.num_steps].tolist(),
                    accepted=[bool(a) for a in acc[:tr.num_steps]], linearisations=int(tr.linearisations),
                    error_evaluations=int(tr.error_evaluations))

    def set_active(self, dense_active, error_active=None):
        """dfk_window_problem_set_active: bool masks over the dense and the error items (error_active None: the dense
        mask, which needs as many error items as dense items)"""
        hd = self._al._hd
        hd.use_torch_stream()
        d = np.ascontiguousarray(np.asarray(dense_active, dtype=bool).astype(np.uint8).ravel())
        e = None if error_active is None else np.ascontiguousarray(np.asarray(error_active, bool).astype(np.uint8).ravel())
        if d.size != self.num_dense or (e is not None and e.size != self.num_error) or \
                (e is None and self.num_error != self.num_dense):
            raise ValueError(f"masks of {self.num_dense} dense and {self.num_error} error items expected (error_active "
                             "may be None only with as many error as dense items)")
        check(hd.h, lib().dfk_window_problem_set_active(hd.h, self.p, d.ctypes.data_as(C.c_void_p),
                                                         None if e is None else e.ctypes.data_as(C.c_void_p)))

    def lm_levels(self, params, schedule, use_error: bool = False) -> dict:
        """dfk_window_lm_levels with window_opt.LMParams and window_opt.LevelSchedule; returns dfk_window_lm's trace
        dict plus switch_energy, pair_levels (per step, per pair; -1 = off) and pair_steps_done"""
        hd = self._al._hd
        hd.use_torch_stream()
        it = int(params.iterations)
        prm = _lib.DfkLMParams(it, float(params.lambda_init), float(params.lambda_up), float(params.lambda_down),
                               float(params.lambda_max), int(bool(params.fix_first_pose)),
                               float(params.code_prior_weight), int(bool(use_error)))
        P = len(schedule.steps_done)
        # the C call reads num_dense / num_error / num_pairs entries: wrong lengths are rejected here
        ln = lambda x: len(np.ravel(x))
        if ln(schedule.item_level) != self.num_dense or ln(schedule.item_pair) != self.num_dense or \
                ln(schedule.remove_after) != P or \
                any(x is not None and ln(x) != self.num_error for x in (schedule.error_pair, schedule.error_level)):
            raise ValueError(f"a schedule of {self.num_dense} dense items, {self.num_error} error items and "
                             f"{P} pairs expected")
        # the device takes each dense item's pair from the window: the schedule's pairing must be the same
        ids = self._win.item_pair[:self.num_dense]
        if not np.array_equal(np.searchsorted(np.unique(ids), ids), np.asarray(schedule.item_pair)):
            raise ValueError("schedule.item_pair is not the window's pairing of the dense items (the distinct window "
                             "pairs of the dense items in window order)")
        i32 = lambda x: np.ascontiguousarray(np.asarray(x, dtype=np.int32).ravel())
        iters, dl, steps = i32(schedule.iters), i32(schedule.item_level), i32(schedule.steps_done)
        rem = np.ascontiguousarray(np.asarray(schedule.remove_after, dtype=bool).astype(np.uint8).ravel())
        ep = None if schedule.error_pair is None else i32(schedule.error_pair)
        el = None if schedule.error_level is None else i32(schedule.error_level)
        ip = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_int32))
        sc = _lib.DfkLevelSchedule(len(iters), ip(iters), ip(dl), ip(ep), ip(el), P, ip(steps),
                                   rem.ctypes.data_as(C.POINTER(C.c_uint8)) if rem.size else None)
        e, lam, acc = np.zeros(it + 1), np.zeros(max(it, 1)), np.zeros(max(it, 1), dtype=np.int32)
        sw, lv, done = np.zeros(max(it, 1)), np.zeros(max(it * P, 1), dtype=np.int32), np.zeros(max(P, 1), np.int32)
        tr = _lib.DfkLMTrace(e.ctypes.data_as(C.POINTER(C.c_double)), lam.ctypes.data_as(C.POINTER(C.c_double)),
                             acc.ctypes.data_as(C.POINTER(C.c_int32)), 0, 0, 0, 0)
        lt = _lib.DfkLevelTrace(sw.ctypes.data_as(C.POINTER(C.c_double)), ip(lv), ip(done), 0)
        check(hd.h, lib().dfk_window_lm_levels(hd.h, self.p, C.byref(prm), C.byref(sc), C.byref(tr), C.byref(lt)))
        n = tr.num_steps
        return dict(energy=e[:tr.num_energies].tolist(), lam=lam[:n].tolist(), accepted=[bool(a) for a in acc[:n]],
                    linearisations=int(tr.linearisations), error_evaluations=int(tr.error_evaluations),
                    switch_energy=sw[:lt.num_switches].tolist(),
                    pair_levels=[lv[s * P:(s + 1) * P].tolist() for s in range(n)], pair_steps_done=done[:P].tolist())

    def close(self):
        if getattr(self, "p", None):
            lib().dfk_window_problem_destroy(self._al.handle, self.p)
            self.p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------- SE3Aligner
class SE3Aligner:
    """df::SE3Aligner<float> (sources/cuda/cu_se3aligner.h:38-86)."""

    def __init__(self, device=None):
        self._hd = _Handle(device)
        self._hd.use_torch_stream()
        self.huber_delta_ = 0.1

    def SetHuberDelta(self, val: float):
        self.huber_delta_ = float(val)
        check(self._hd.h, lib().dfk_se3_set_huber_delta(self._hd.h, C.c_float(val)))

    def RunStep(self, se3, cam, img0, img1, dpt0, grad1) -> JTJJrReductionItem:
        self._hd.use_torch_stream()
        JtJ = np.zeros(21, dtype=np.float32)
        Jtr = np.zeros(6, dtype=np.float32)
        res = C.c_float(0)
        inl = C.c_uint64(0)
        F = C.POINTER(C.c_float)
        i0, i1, d0, g1 = _image(img0), _image(img1), _image(dpt0), _image(grad1, 2)
        cc = _cam(cam)
        st = lib().dfk_se3_run_step(self._hd.h, _pose(se3), C.byref(cc), C.byref(i0), C.byref(i1), C.byref(d0),
                                    C.byref(g1), JtJ.ctypes.data_as(F), Jtr.ctypes.data_as(F), C.byref(res),
                                    C.byref(inl))
        check(self._hd.h, st)
        return JTJJrReductionItem(JtJ, Jtr, float(res.value), int(inl.value))

    def Warp(self, se3, cam, img0, img1, dpt0, img2) -> CorrespondenceReductionItem:
        self._hd.use_torch_stream()
        res = C.c_float(0)
        inl = C.c_uint64(0)
        i0, i1, d0, i2 = _image(img0), _image(img1), _image(dpt0), _image(img2)
        cc = _cam(cam)
        st = lib().dfk_se3_warp(self._hd.h, _pose(se3), C.byref(cc), C.byref(i0), C.byref(i1), C.byref(d0),
                                C.byref(i2), C.byref(res), C.byref(inl))
        check(self._hd.h, st)
        return CorrespondenceReductionItem(float(res.value), int(inl.value))


# ------------------------------------------------------------------------------------------- CameraTracker
@dataclass
class TrackerConfig:
    """CameraTracker::TrackerConfig (core/system/camera_tracker.h:45-50)"""
    pyramid_levels: int = 3
    iterations_per_level: Sequence[int] = (10, 5, 4)   # index = pyramid level, 0 = finest
    huber_delta: float = 0.1


class CameraTracker:
    """df::CameraTracker (core/system/camera_tracker.{h,cpp}), the part that touches the GPU: TrackFrame's
    coarse-to-fine Gauss-Newton on pose_ck.  The reference synchronises and solves on the host after every SE3 step
    (camera_tracker.cpp:53-63); here the whole loop is enqueued at once (dfk_se3_track) and the 6x6 solve + retraction
    run in the last block of every step kernel.  Keyframe bookkeeping (SetKeyframe / GetPoseEstimate pose algebra,
    camera_tracker.cpp:94-121) is host-side and kept as plain methods."""

    def __init__(self, camera_pyr, config: TrackerConfig, device=None):
        if len(config.iterations_per_level) != config.pyramid_levels:
            # the reference LOG(FATAL)s here (camera_tracker.cpp:32-33)
            raise ValueError("CameraTracker config error: iterations_per_level size not equal pyramid_levels")
        self.config_ = config
        self.camera_pyr_ = list(camera_pyr)
        self._hd = _Handle(device)
        check(self._hd.h, lib().dfk_se3_set_huber_delta(self._hd.h, C.c_float(config.huber_delta)))
        self.pose_ck_ = np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float32)
        self.kf_ = None
        self.inliers_ = 0.0
        self.error_ = float("inf")
        self.history_ = None

    def Reset(self):
        self.pose_ck_ = np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float32)

    def SetKeyframe(self, kf_pyr_img, kf_pyr_dpt, pose_wk=None):
        """kf_pyr_img / kf_pyr_dpt: per-level keyframe image and depth (level 0 = finest)"""
        from . import se3 as _se3
        if self.kf_ is not None and pose_wk is not None and self.kf_[2] is not None:
            wc = _se3.compose(self.kf_[2], _se3.inverse(self.pose_ck_))
            self.pose_ck_ = _se3.compose(_se3.inverse(wc), pose_wk).astype(np.float32)
        self.kf_ = (list(kf_pyr_img), list(kf_pyr_dpt), None if pose_wk is None else np.asarray(pose_wk, np.float32))

    def GetPoseEstimate(self):
        from . import se3 as _se3
        pose_wk = self.kf_[2] if self.kf_[2] is not None else np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float32)
        return _se3.compose(pose_wk, _se3.inverse(self.pose_ck_))

    def GetInliers(self) -> float:
        return self.inliers_

    def GetError(self) -> float:
        return self.error_

    def TrackFrame(self, pyr_img1, pyr_grad1, keep_history: bool = False):
        if self.kf_ is None:
            raise RuntimeError("Calling CameraTracker::TrackFrame before a keyframe was set")
        self._hd.use_torch_stream()
        n = self.config_.pyramid_levels
        levels = (DfkTrackLevel * n)()
        for l in range(n):
            levels[l].cam = _cam(self.camera_pyr_[l])
            levels[l].img0 = _image(self.kf_[0][l])
            levels[l].img1 = _image(pyr_img1[l])
            levels[l].dpt0 = _image(self.kf_[1][l])
            levels[l].grad1 = _image(pyr_grad1[l], 2)
            levels[l].iterations = int(self.config_.iterations_per_level[l])
        total = int(sum(self.config_.iterations_per_level))
        pose = np.ascontiguousarray(self.pose_ck_, dtype=np.float32).copy()
        frac, err = C.c_float(0), C.c_float(0)
        last = np.zeros(29, dtype=np.float32)
        hist = np.zeros((max(total, 1), 36), dtype=np.float32) if keep_history else None
        F = C.POINTER(C.c_float)
        st = lib().dfk_se3_track(self._hd.h, pose.ctypes.data_as(F), levels, n, C.byref(frac), C.byref(err),
                                 last.ctypes.data_as(F), hist.ctypes.data_as(F) if keep_history else None,
                                 total if keep_history else 0)
        check(self._hd.h, st)
        self.pose_ck_ = pose
        self.inliers_ = float(frac.value)
        self.error_ = float(err.value)
        self.history_ = hist[:total] if keep_history else None
        return pose

    def TrackFrameBatch(self, keyframes, pyr_img1, pyr_grad1, poses_ck=None):
        """The live frame (pyr_img1, pyr_grad1) tracked against every keyframe of `keyframes` at once
        (dfk_se3_track_batch): one launch per Gauss-Newton iteration for all of them, one read-back.  `keyframes` is a
        sequence of (pyr_img, pyr_dpt[, pose_wk]); `poses_ck` [N, 7] are the start poses, identity for every keyframe when
        omitted (what Reset does before each TrackFrame in Relocalize / DetectLoop).  Keyframe n gives bit for bit what
        SetKeyframe(keyframe n) + TrackFrame from poses_ck[n] gives.  Returns (poses_ck [N, 7], inlier_fractions [N],
        errors [N]); the tracker's own keyframe, pose and statistics are left alone."""
        poses = batch_start_poses(keyframes, self.config_.pyramid_levels, poses_ck)
        n, L = poses.shape[0], self.config_.pyramid_levels
        if len(pyr_img1) < L or len(pyr_grad1) < L:
            raise ValueError(f"the live frame needs {L} pyramid levels")
        self._hd.use_torch_stream()
        levels = (DfkTrackLevel * (n * L))()
        for k, kf in enumerate(keyframes):
            for l in range(L):
                lv = levels[k * L + l]
                lv.cam = _cam(self.camera_pyr_[l])
                lv.img0 = _image(kf[0][l])
                lv.img1 = _image(pyr_img1[l])
                lv.dpt0 = _image(kf[1][l])
                lv.grad1 = _image(pyr_grad1[l], 2)
                lv.iterations = int(self.config_.iterations_per_level[l])
        frac = np.zeros(n, dtype=np.float32)
        err = np.zeros(n, dtype=np.float32)
        F = C.POINTER(C.c_float)
        check(self._hd.h, lib().dfk_se3_track_batch(self._hd.h, n, L, poses.ctypes.data_as(F), levels,
                                                    frac.ctypes.data_as(F), err.ctypes.data_as(F), None))
        return poses, frac, err

    def Relocalize(self, keyframes, pyr_img1, pyr_grad1):
        """DeepFactors::Relocalize (core/deepfactors.cpp:713-743): track the live frame against every keyframe from
        identity, keep the first keyframe with the strictly smallest error; when no error is finite, the first keyframe
        at its own pose_wk (pose_ck = identity).  `keyframes` as in TrackFrameBatch; all of them are tracked in one
        batched call.  Afterwards the tracker's keyframe is the winner and pose_ck_ its tracked pose, so the next
        TrackFrame continues from there.  Returns (index, pose_wc, errors).

        One deliberate difference: after the reference's loop GetError() / GetInliers() still hold the LAST keyframe
        tracked, whichever won; here they report the winner's."""
        poses, frac, err = self.TrackFrameBatch(keyframes, pyr_img1, pyr_grad1)
        idx, pose_ck, pose_wc = relocalize_select(err, poses, [kf[2] if len(kf) > 2 else None for kf in keyframes])
        kf = keyframes[idx]
        self.kf_ = None  # SetKeyframe without the pose hand-over: pose_ck_ is set directly below
        self.SetKeyframe(kf[0], kf[1], kf[2] if len(kf) > 2 else None)
        self.pose_ck_ = pose_ck
        self.inliers_ = float(frac[idx])
        self.error_ = float(err[idx])
        return idx, pose_wc, err


def batch_start_poses(keyframes, pyramid_levels: int, poses_ck=None) -> np.ndarray:
    """Argument checks of CameraTracker.TrackFrameBatch; returns the start poses as a fresh [N, 7] float32 array."""
    n = len(keyframes)
    if n < 1 or n > 65535:
        raise ValueError(f"need 1 to 65535 keyframes, got {n}")
    for k, kf in enumerate(keyframes):
        if len(kf) not in (2, 3):
            raise ValueError(f"keyframe {k} must be (pyr_img, pyr_dpt[, pose_wk])")
        if len(kf[0]) < pyramid_levels or len(kf[1]) < pyramid_levels:
            raise ValueError(f"keyframe {k} needs {pyramid_levels} pyramid levels of image and depth")
    if poses_ck is None:
        poses = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float32), (n, 1))
    else:
        poses = np.array(poses_ck, dtype=np.float32).reshape(-1, 7) if np.size(poses_ck) == 7 * n else None
        if poses is None:
            raise ValueError(f"poses_ck must be {n} x 7 floats")
    return np.ascontiguousarray(poses)


def relocalize_select(errors, poses_ck, poses_wk):
    """The selection rule of DeepFactors::Relocalize (core/deepfactors.cpp:717-733): the first keyframe whose error is
    strictly smaller than every earlier one (and than +inf), else keyframe 0 at its own pose_wk with pose_ck = identity.
    poses_wk[k] may be None (identity).  Returns (index, pose_ck, pose_wc = pose_wk * pose_ck^-1, GetPoseEstimate)."""
    from . import se3 as _se3
    best, best_err = 0, float("inf")
    for k, e in enumerate(np.asarray(errors, dtype=np.float64)):
        if e < best_err:
            best, best_err = k, float(e)
    if best_err == float("inf"):  # nothing tracked: best_pose = keyframe 1's pose_wk in the reference
        pose_ck = np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float32)
    else:
        pose_ck = np.asarray(poses_ck[best], dtype=np.float32).copy()
    pose_wk = poses_wk[best] if poses_wk[best] is not None else np.array([0, 0, 0, 1, 0, 0, 0], dtype=np.float32)
    return best, pose_ck, _se3.compose(np.asarray(pose_wk, np.float32), _se3.inverse(pose_ck))


# ------------------------------------------------------------------------------------------- DBoW2 retrieval
_BOW_NODE = re.compile(r'\{\s*nodeId\s*:\s*(\d+)\s*,\s*parentId\s*:\s*(\d+)\s*,\s*weight\s*:\s*([^,\s}]+)\s*,'
                       r'\s*descriptor\s*:\s*"([^"]*)"\s*\}')
_BOW_WORD = re.compile(r'\{\s*wordId\s*:\s*(\d+)\s*,\s*nodeId\s*:\s*(\d+)\s*\}')


def parse_dbow2_vocabulary(text: str) -> dict:
    """DBoW2's TemplatedVocabulary::save text (cv::FileStorage YAML) as the arrays of DfkBowVocabularyDesc: k, L,
    weighting, scoring, descriptor_bytes, node_ids / parent_ids int32 [N], weights float64 [N] (float() rounds as strtod),
    descriptors uint8 [N, D], word_ids / word_nodes int32 [W], all in file order.  A line break inside a quoted
    descriptor, with or without a trailing backslash, reads as the writer meant it."""
    text = re.sub(r'\\\r?\n\s*', '', text)  # an escaped line break joins the two lines

    def head(key):
        m = re.search(r'^\s*' + key + r'\s*:\s*(-?\d+)\s*$', text, re.M)
        if not m:
            raise ValueError(f"DBoW2 vocabulary: no {key}")
        return int(m.group(1))

    nodes = _BOW_NODE.findall(text)
    words = _BOW_WORD.findall(text)
    if not nodes or not words:
        raise ValueError("DBoW2 vocabulary: no nodes or no words")
    desc = [[int(t) for t in d.split()] for _, _, _, d in nodes]
    D = len(desc[0])
    if any(len(d) != D for d in desc):
        raise ValueError("DBoW2 vocabulary: descriptors of different lengths")
    return dict(k=head("k"), L=head("L"), weighting=head("weightingType"), scoring=head("scoringType"),
                descriptor_bytes=D,
                node_ids=np.array([int(n[0]) for n in nodes], np.int32),
                parent_ids=np.array([int(n[1]) for n in nodes], np.int32),
                weights=np.array([float(n[2]) for n in nodes], np.float64),
                descriptors=np.array(desc, np.uint8).reshape(-1, D),
                word_ids=np.array([int(w[0]) for w in words], np.int32),
                word_nodes=np.array([int(w[1]) for w in words], np.int32))


def load_dbow2_vocabulary(path) -> dict:
    """parse_dbow2_vocabulary of a .yml or .yml.gz file; needs no OpenCV"""
    path = os.fspath(path)
    opener = gzip.open if path.endswith(".gz") else open
    with opener(path, "rt", encoding="ascii") as f:
        return parse_dbow2_vocabulary(f.read())


class BowVocabulary:
    """A DBoW2 vocabulary on the device (dfk_bow_vocabulary_create): a path or the dict of load_dbow2_vocabulary.  The
    tree is validated when it is created; TF_IDF / L1_NORM only."""

    def __init__(self, voc, device=None):
        if not isinstance(voc, dict):
            voc = load_dbow2_vocabulary(voc)
        self.voc = voc
        self._hd = _Handle(device)
        arr = {k: np.ascontiguousarray(voc[k], dt) for k, dt in
               (("node_ids", np.int32), ("parent_ids", np.int32), ("weights", np.float64), ("descriptors", np.uint8),
                ("word_ids", np.int32), ("word_nodes", np.int32))}
        d = _lib.DfkBowVocabularyDesc(int(voc["k"]), int(voc["L"]), int(voc["weighting"]), int(voc["scoring"]),
                                      int(voc["descriptor_bytes"]), len(arr["node_ids"]), arr["node_ids"].ctypes.data,
                                      arr["parent_ids"].ctypes.data, arr["weights"].ctypes.data,
                                      arr["descriptors"].ctypes.data, len(arr["word_ids"]), arr["word_ids"].ctypes.data,
                                      arr["word_nodes"].ctypes.data)
        self._p = C.c_void_p()
        check(self._hd.h, lib().dfk_bow_vocabulary_create(self._hd.h, C.byref(d), C.byref(self._p)))

    @property
    def descriptor_bytes(self) -> int:
        return int(self.voc["descriptor_bytes"])

    def close(self):
        if getattr(self, "_p", None) and self._hd.h:
            lib().dfk_bow_vocabulary_destroy(self._hd.h, self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


@dataclass
class BowVector:
    """A bag-of-words vector on the device (DfkBowVector): words int32 [capacity] ascending, values float64 [capacity],
    count int32 [1] (a view into a transform's counts); only the first count rows hold the vector."""
    words: torch.Tensor
    values: torch.Tensor
    count: torch.Tensor
    capacity: int

    def to_c(self) -> "_lib.DfkBowVector":
        return _lib.DfkBowVector(self.words.data_ptr(), self.values.data_ptr(), self.count.data_ptr(), self.capacity)

    def host(self):
        """(words, values) on the host (synchronises)"""
        c = int(self.count.item())
        return self.words[:c].cpu().numpy(), self.values[:c].cpu().numpy()

    @staticmethod
    def from_host(words, values, device="cuda", capacity: int | None = None) -> "BowVector":
        w = np.ascontiguousarray(words, np.int32)
        v = np.ascontiguousarray(values, np.float64)
        cap = len(w) if capacity is None else int(capacity)
        tw = torch.zeros(max(cap, 1), dtype=torch.int32, device=device)
        tv = torch.zeros(max(cap, 1), dtype=torch.float64, device=device)
        tw[:len(w)] = torch.from_numpy(w).to(device)
        tv[:len(v)] = torch.from_numpy(v).to(device)
        return BowVector(tw, tv, torch.tensor([len(w)], dtype=torch.int32, device=device), cap)


@dataclass
class BowBatch:
    """The device output of BowTransformBatch: item i's rows are [offsets[i], offsets[i] + capacities[i]); words int32,
    values float64, feature_words int32 (the word of each descriptor, -1 when its weight is not > 0), counts int32 [n]."""
    words: torch.Tensor
    values: torch.Tensor
    counts: torch.Tensor
    feature_words: torch.Tensor
    offsets: np.ndarray
    capacities: np.ndarray

    def vectors(self) -> list:
        """one BowVector per item (views, no read-back): they feed BowDatabase.add / query / score as they are"""
        return [BowVector(self.words[o:o + c], self.values[o:o + c], self.counts[i:i + 1], int(c))
                for i, (o, c) in enumerate(zip(self.offsets[:-1], self.capacities))]


def _descriptor_rows(d) -> torch.Tensor:
    d = d.descriptors if isinstance(d, Features) else d
    if not isinstance(d, torch.Tensor) or not d.is_cuda or d.dtype != torch.uint8 or d.dim() != 2 or \
            (d.shape[0] > 1 and not d.is_contiguous()):
        raise TypeError("BowTransformBatch: descriptors must be contiguous uint8 [N, D] CUDA tensors")
    return d


def BowTransformBatch(voc: BowVocabulary, descriptors: Sequence, capacities=None) -> BowBatch:
    """voc_.transform(features, bow_vec) of many images in one call (dfk_bow_transform_batch), bit for bit DBoW2:
    descriptors are uint8 [N, D] CUDA tensors (or Features), D the vocabulary's.  capacities (default N) reserve each
    item's output rows.  Asynchronous: returns a BowBatch of device tensors."""
    hd = voc._hd
    hd.use_torch_stream()
    rows = [_descriptor_rows(d) for d in descriptors]
    n = len(rows)
    caps = [int(r.shape[0]) for r in rows] if capacities is None else [int(c) for c in capacities]
    if len(caps) != n:
        raise ValueError("BowTransformBatch: one capacity per item")
    sets = (_lib.DfkFeatureSet * max(n, 1))(*[_lib.DfkFeatureSet(None, r.data_ptr() if r.shape[0] else None,
                                                                 int(r.shape[0]), int(r.shape[1])) for r in rows])
    cap_arr = (C.c_int32 * max(n, 1))(*caps)
    offsets = np.concatenate([[0], np.cumsum(caps)]).astype(np.int64)
    total = int(offsets[-1])
    dev = f"cuda:{hd.device}"
    words = torch.zeros(max(total, 1), dtype=torch.int32, device=dev)
    values = torch.zeros(max(total, 1), dtype=torch.float64, device=dev)
    fw = torch.zeros(max(total, 1), dtype=torch.int32, device=dev)
    counts = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
    check(hd.h, lib().dfk_bow_transform_batch(hd.h, voc._p, sets, cap_arr, n, C.c_void_p(words.data_ptr()),
                                              C.c_void_p(values.data_ptr()), C.c_void_p(counts.data_ptr()),
                                              C.c_void_p(fw.data_ptr())))
    return BowBatch(words, values, counts[:n], fw, offsets, np.array(caps, np.int64))


@dataclass
class BowQueryResult:
    """BowDatabase.query's device output: query i's rows are [offsets[i], offsets[i] + min(counts[i], max_results[i]));
    ids int32 entry ids, scores float64, best first; counts int32 [n] (DBoW2's ret.size() before the cut)."""
    ids: torch.Tensor
    scores: torch.Tensor
    counts: torch.Tensor
    offsets: np.ndarray
    max_results: np.ndarray

    def results(self) -> list:
        """per query the list of (Id, Score), as DBoW2's QueryResults (one read-back)"""
        c, ids, sc = self.counts.cpu().numpy(), self.ids.cpu().numpy(), self.scores.cpu().numpy()
        return [[(int(ids[o + k]), float(sc[o + k])) for k in range(min(int(c[i]), int(m)))]
                for i, (o, m) in enumerate(zip(self.offsets[:-1], self.max_results))]


class BowDatabase:
    """TemplatedDatabase(voc, false, 0) on the device (dfk_bow_database_*): add, query, score, clear, len."""

    def __init__(self, voc: BowVocabulary):
        self.voc = voc
        self._hd = voc._hd
        self._p = C.c_void_p()
        check(self._hd.h, lib().dfk_bow_database_create(self._hd.h, voc._p, C.byref(self._p)))

    def __len__(self) -> int:
        n = C.c_int32()
        check(self._hd.h, lib().dfk_bow_database_size(self._hd.h, self._p, C.byref(n)))
        return int(n.value)

    def clear(self):
        check(self._hd.h, lib().dfk_bow_database_clear(self._hd.h, self._p))

    def add(self, vectors: Sequence[BowVector]) -> int:
        """adds the vectors in order (copied on the device, no read-back); returns the first entry id"""
        self._hd.use_torch_stream()
        n = len(vectors)
        arr = (_lib.DfkBowVector * max(n, 1))(*[v.to_c() for v in vectors])
        first = C.c_int32(-1)
        check(self._hd.h, lib().dfk_bow_database_add(self._hd.h, self._p, arr, n, C.byref(first)))
        return int(first.value)

    def query(self, vectors: Sequence[BowVector], max_results=1, max_id=-1) -> BowQueryResult:
        """db_.query(vec, ret, max_results, max_id) for every vector in one call (dfk_bow_database_query_batch);
        max_results and max_id are one value for all or one per vector.  Asynchronous."""
        self._hd.use_torch_stream()
        n = len(vectors)
        per = lambda v: [int(x) for x in (v if isinstance(v, (list, tuple, np.ndarray)) else [v] * n)]
        mr, mi = per(max_results), per(max_id)
        arr = (_lib.DfkBowQuery * max(n, 1))(*[_lib.DfkBowQuery(v.to_c(), a, b) for v, a, b in zip(vectors, mr, mi)])
        offsets = np.concatenate([[0], np.cumsum(mr)]).astype(np.int64)
        dev = f"cuda:{self._hd.device}"
        ids = torch.full((max(int(offsets[-1]), 1),), -1, dtype=torch.int32, device=dev)
        scores = torch.zeros(max(int(offsets[-1]), 1), dtype=torch.float64, device=dev)
        counts = torch.zeros(max(n, 1), dtype=torch.int32, device=dev)
        check(self._hd.h, lib().dfk_bow_database_query_batch(self._hd.h, self._p, arr, n, C.c_void_p(ids.data_ptr()),
                                                             C.c_void_p(scores.data_ptr()),
                                                             C.c_void_p(counts.data_ptr())))
        return BowQueryResult(ids, scores, counts[:n], offsets, np.array(mr, np.int64))

    def score(self, entries: Sequence[int], vectors: Sequence[BowVector]) -> torch.Tensor:
        """voc_.score(entry's vector, vector) per pair (dfk_bow_score_batch): float64 [n] on the device"""
        self._hd.use_torch_stream()
        n = len(vectors)
        arr = (_lib.DfkBowScoreItem * max(n, 1))(*[_lib.DfkBowScoreItem(int(e), v.to_c())
                                                   for e, v in zip(entries, vectors)])
        out = torch.zeros(max(n, 1), dtype=torch.float64, device=f"cuda:{self._hd.device}")
        check(self._hd.h, lib().dfk_bow_score_batch(self._hd.h, self._p, arr, n, C.c_void_p(out.data_ptr())))
        return out[:n]

    def close(self):
        if getattr(self, "_p", None) and self._hd.h:
            lib().dfk_bow_database_destroy(self._hd.h, self._p)
            self._p = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ------------------------------------------------------------------------------------------- LoopDetector
@dataclass
class LoopDetectorConfig:
    """LoopDetectorConfig (core/system/loop_detector.h:44-53)"""
    tracker_cfg: TrackerConfig = field(default_factory=TrackerConfig)
    iters: Sequence[int] = (10, 5, 4)
    min_similarity: float = 0.35
    max_error: float = 0.5
    max_dist: float = 0.1
    max_candidates: int = 3
    active_window: int = 5


@dataclass
class LoopInfo:
    """LoopDetector::LoopInfo (loop_detector.h:73-78)"""
    loop_id: int = 1
    pose_wc: np.ndarray | None = None
    detected: bool = False


def _translation_dist(a, b) -> np.float32:
    """(a.translation() - b.translation()).norm() in fp32 (poses: quaternion (x, y, z, w), translation)"""
    d = np.asarray(a, np.float32)[4:7] - np.asarray(b, np.float32)[4:7]
    return np.sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2], dtype=np.float32)


def loop_candidates(results, curr_kf_id: int, active_window: int, min_similarity: float, entry_to_id=None) -> list:
    """The candidate filter of LoopDetector::DetectLoop (loop_detector.cpp:117-139): results are the query's (Id, Score)
    best first, keyframe id = entry_to_id(Id) (Id + 1 by default, as the reference assumes).  Skips the current
    keyframe, ids > curr - active_window and Score < min_similarity.  The ids are size_t there, so curr - active_window
    wraps when curr < active_window and then skips nothing; so does this."""
    to_id = entry_to_id or (lambda e: e + 1)
    thr = (int(curr_kf_id) - int(active_window)) % (1 << 64)
    ms = float(np.float32(min_similarity))
    out = []
    for e, s in results:
        kfid = int(to_id(e))
        if kfid == curr_kf_id or kfid > thr or s < ms:
            continue
        out.append(kfid)
    return out


def loop_select(candidates, poses_wc, inliers, poses_wk, max_dist: float) -> LoopInfo:
    """The geometry check's selection of LoopDetector::DetectLoop (loop_detector.cpp:146-184): per candidate its tracked
    pose_wc, inlier fraction and pose_wk; skip inliers < 0.5, keep the strictly smallest translation distance, accept it
    below max_dist."""
    best_dist, best_id, best_pose = np.float32(np.inf), candidates[0], None
    for cid, pwc, inl, pwk in zip(candidates, poses_wc, inliers, poses_wk):
        dist = _translation_dist(pwc, pwk)
        if np.float32(inl) < np.float32(0.5):
            continue
        if dist < best_dist:
            best_dist, best_id, best_pose = dist, cid, pwc
    if best_dist < np.float32(max_dist):
        return LoopInfo(int(best_id), np.asarray(best_pose, np.float32), True)
    return LoopInfo()


def detect_local_loop(keyframe_poses, pose_cam, curr_kf_id: int, active_window: int, max_dist: float) -> int:
    """LoopDetector::DetectLocalLoop (loop_detector.cpp:190-224), host only: keyframe_poses is (id, pose_wk) in the map's
    order; the last active_window of them, newest first, the strictly closest by translation that is not the current
    keyframe; its id when closer than max_dist, else 0."""
    kp = list(keyframe_poses)
    best_dist, best_id = np.float32(np.inf), (kp[-1][0] if kp else 0)
    for kid, pwk in kp[::-1][:max(int(active_window), 0)]:
        dist = _translation_dist(pose_cam, pwk)
        if dist < best_dist and kid != curr_kf_id:
            best_dist, best_id = dist, kid
    if best_id != curr_kf_id and best_dist < np.float32(max_dist):
        return int(best_id)
    return 0


class LoopDetector:
    """df::LoopDetector (core/system/loop_detector.{h,cpp}) on the device: the vocabulary transform, the database and
    its query run in libdfk.so (no descriptor leaves the device), the geometric check is one batched track of every
    surviving candidate (CameraTracker.TrackFrameBatch).  Keyframes are passed as a mapping id -> (pyr_img, pyr_dpt,
    pose_wk); entry e of the database is keyframe entry_to_id(e), e + 1 by default."""

    def __init__(self, vocabulary, camera_pyr, config: LoopDetectorConfig | None = None, entry_to_id=None, device=None):
        self.cfg_ = config or LoopDetectorConfig()
        self.voc_ = vocabulary if isinstance(vocabulary, BowVocabulary) else BowVocabulary(vocabulary, device)
        self.db_ = BowDatabase(self.voc_)
        tc = self.cfg_.tracker_cfg
        self.tracker_ = CameraTracker(camera_pyr, TrackerConfig(len(self.cfg_.iters), tuple(self.cfg_.iters),
                                                                tc.huber_delta), device)
        self.entry_to_id = entry_to_id or (lambda e: e + 1)
        self.dmap_ = {}  # keyframe id -> (entry, BowVector)
        self.last_min_score = None

    def AddKeyframe(self, kf_id: int, descriptors) -> BowVector:
        """transform the keyframe's descriptors and add them to the database (loop_detector.cpp:38-44)"""
        vec = BowTransformBatch(self.voc_, [descriptors]).vectors()[0]
        entry = self.db_.add([vec])
        self.dmap_[kf_id] = (entry, vec)
        return vec

    def DetectLoop(self, pyr_img, pyr_grad, descriptors, curr_kf_id: int, keyframes) -> LoopInfo:
        """LoopDetector::DetectLoop (loop_detector.cpp:96-185): transform, the score against the current keyframe
        (kept in last_min_score; the reference only logs it), the query (max_id -1, max_candidates), the candidate
        filter, one batched track of the survivors and the selection"""
        vec = BowTransformBatch(self.voc_, [descriptors]).vectors()[0]
        cur = self.dmap_.get(curr_kf_id)
        score = self.db_.score([cur[0]], [vec]) if cur is not None else None
        res = self.db_.query([vec], self.cfg_.max_candidates, -1).results()[0]
        self.last_min_score = float(score.item()) if score is not None else None
        cands = loop_candidates(res, curr_kf_id, self.cfg_.active_window, self.cfg_.min_similarity, self.entry_to_id)
        if not cands:
            return LoopInfo()
        from . import se3 as _se3
        kfs = [keyframes[c] for c in cands]
        poses_ck, frac, _ = self.tracker_.TrackFrameBatch(kfs, pyr_img, pyr_grad)
        ident = np.array([0, 0, 0, 1, 0, 0, 0], np.float32)
        pwk = [np.asarray(kf[2], np.float32) if len(kf) > 2 and kf[2] is not None else ident for kf in kfs]
        pwc = [_se3.compose(w, _se3.inverse(p)) for w, p in zip(pwk, poses_ck)]
        return loop_select(cands, pwc, frac, pwk, self.cfg_.max_dist)

    def DetectLocalLoop(self, keyframe_poses, pose_cam, curr_kf_id: int) -> int:
        return detect_local_loop(keyframe_poses, pose_cam, curr_kf_id, self.cfg_.active_window, self.cfg_.max_dist)

    def Reset(self):
        self.db_.clear()
        self.dmap_.clear()


# ------------------------------------------------------------------------------------------- free functions
_default_handle = {}


def _free_handle(device=None) -> _Handle:
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    if dev not in _default_handle:
        _default_handle[dev] = _Handle(dev)
    hd = _default_handle[dev]
    hd.use_torch_stream()
    return hd


def UpdateDepth(code, prx_orig, prx_jac, avg_dpt, dpt_out):
    """df::UpdateDepth (cu_image_proc.cpp:266-277): dpt = avg/(prx_orig + prx_jac.code) - avg."""
    hd = _free_handle(dpt_out.device)
    code = np.ascontiguousarray(code, dtype=np.float32)
    cs = int(code.shape[0])
    p, j, d = _image(prx_orig), _image(prx_jac, cs), _image(dpt_out)
    st = lib().dfk_update_depth(hd.h, code.ctypes.data_as(C.POINTER(C.c_float)), cs, C.byref(p), C.byref(j),
                                C.c_float(avg_dpt), C.byref(d))
    check(hd.h, st)


def SobelGradients(img, grad):
    """df::SobelGradients (cu_image_proc.cpp:95-113)."""
    hd = _free_handle(img.device)
    i, g = _image(img), _image(grad, 2)
    check(hd.h, lib().dfk_sobel_gradients(hd.h, C.byref(i), C.byref(g)))


def GaussianBlurDown(inp, out):
    """df::GaussianBlurDown (cu_image_proc.cpp:166-184)."""
    hd = _free_handle(inp.device)
    i, o = _image(inp), _image(out)
    check(hd.h, lib().dfk_gaussian_blur_down(hd.h, C.byref(i), C.byref(o)))


def BuildImagePyramid(imgs, grads=None):
    """imgs[0] given; fills imgs[1:] by GaussianBlurDown and grads[:] by SobelGradients, all enqueued at once
    (Frame::FillPyramids, core/mapping/frame.h:80-94)."""
    hd = _free_handle()
    n = len(imgs)
    ia = (DfkImage * n)(*[_image(t) for t in imgs])
    ga = (DfkImage * n)(*[_image(t, 2) for t in grads]) if grads is not None else None
    check(hd.h, lib().dfk_build_image_pyramid(hd.h, ia, ga, n))


def SquaredError(buf1, buf2) -> float:
    """df::SquaredError (cu_image_proc.cpp:208-242)."""
    hd = _free_handle(buf1.device)
    a, b = _image(buf1), _image(buf2)
    out = C.c_float(0)
    check(hd.h, lib().dfk_squared_error(hd.h, C.byref(a), C.byref(b), C.byref(out)))
    return float(out.value)
