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
from dataclasses import dataclass, field
from typing import Sequence

import numpy as np
import torch

from . import _lib
from ._lib import (DfkCamera, DfkDenseSfmParams, DfkImage, DfkReprojectionItem, DfkSfmAlignerParams, DfkSparseGeometricItem, DfkSfmWorkItem,
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

    def unpack(self, records: torch.Tensor):
        r = records.detach().cpu().numpy()
        return [JTJJrReductionItem.from_record(r[i], self.CS) for i in range(r.shape[0])]


# ------------------------------------------------------------------------------------------- sparse keypoint factor
def ReprojectionLinearize(aligner, pose0, pose1, code0, cam, prx_orig, prx_jac, query_xy, train_xy, cauchy_delta: float,
                          sigma: float):
    """ReprojectionFactor::linearize (sources/core/gtsam/reprojection_factor.cpp:157-269) with the rows gathered on the
    device: prx_orig / prx_jac are the keyframe's level-0 DEVICE buffers, query_xy / train_xy the matched keypoints [M, 2]
    (host).  Returns (rows [2M, 13 + C] float32 = the blocks of the JacobianFactor [J_pose0 | J_pose1 | J_code0 | b],
    total_err)."""
    aligner._hd.use_torch_stream()
    cs = aligner.CS
    code = np.ascontiguousarray(code0, dtype=np.float32)
    q = np.ascontiguousarray(query_xy, dtype=np.float32).reshape(-1, 2)
    t = np.ascontiguousarray(train_xy, dtype=np.float32).reshape(-1, 2)
    M = q.shape[0]
    rows = np.zeros((2 * M, 13 + cs), dtype=np.float32)
    tot = C.c_float(0)
    FP = C.POINTER(C.c_float)
    c, p, j = _cam(cam), _image(prx_orig), _image(prx_jac, cs)
    check(aligner.handle, lib().dfk_reprojection_linearize(
        aligner.handle, _pose(pose0), _pose(pose1), code.ctypes.data_as(FP), cs, C.byref(c), C.byref(p), C.byref(j), M,
        q.ctypes.data_as(FP), t.ctypes.data_as(FP), C.c_float(cauchy_delta), C.c_float(sigma), rows.ctypes.data_as(FP),
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
    cs, n = aligner.CS, len(items)
    rec = _lib.record_floats(cs)
    if records is None:
        records = torch.empty((n, rec), dtype=torch.float32, device=f"cuda:{aligner._hd.device}")
    if not (records.is_contiguous() and records.numel() >= n * rec):
        raise ValueError(f"records must be a contiguous device tensor of at least {n} x {rec} floats")
    arr = (DfkReprojectionItem * max(n, 1))()
    keep = []  # the host arrays must outlive the ctypes pointers until the call returns
    FP = C.POINTER(C.c_float)
    for k, it in enumerate(items):
        code = np.ascontiguousarray(it["code0"], dtype=np.float32)
        if code.shape != (cs,):
            raise ValueError(f"code0 must have {cs} entries")
        q = np.ascontiguousarray(it["query_xy"], dtype=np.float32).reshape(-1, 2)
        t = np.ascontiguousarray(it["train_xy"], dtype=np.float32).reshape(-1, 2)
        if q.shape != t.shape:
            raise ValueError("query_xy and train_xy must hold the same number of matches")
        keep += [code, q, t]
        w = arr[k]
        w.pose0, w.pose1, w.cam = _pose(it["pose0"]), _pose(it["pose1"]), _cam(it["cam"])
        w.prx_orig, w.prx_jac = _image(it["prx_orig"]), _image(it["prx_jac"], cs)
        w.code, w.query_xy, w.train_xy = code.ctypes.data_as(FP), q.ctypes.data_as(FP), t.ctypes.data_as(FP)
        w.num_matches = q.shape[0]
        w.cauchy_delta, w.sigma = float(it["cauchy_delta"]), float(it["sigma"])
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
    cs = aligner.CS
    c0 = np.ascontiguousarray(code0, dtype=np.float32)
    c1 = np.ascontiguousarray(code1, dtype=np.float32)
    pts = np.ascontiguousarray(points_xy, dtype=np.int32).reshape(-1, 2)
    M = pts.shape[0]
    rows = np.zeros((M, 13 + 2 * cs), dtype=np.float32)
    nv = C.c_int(0)
    FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int)
    c = _cam(cam)
    i0, j0, i1, j1, g1 = _image(prx0_orig), _image(prx0_jac, cs), _image(prx1_orig), _image(prx1_jac, cs), _image(dpt_grad1, 2)
    check(aligner.handle, lib().dfk_sparse_geometric_linearize(
        aligner.handle, _pose(pose0), _pose(pose1), c0.ctypes.data_as(FP), c1.ctypes.data_as(FP), cs, C.byref(c), C.byref(i0),
        C.byref(j0), C.byref(i1), C.byref(j1), C.byref(g1), M, pts.ctypes.data_as(IP), C.c_float(huber_delta),
        rows.ctypes.data_as(FP), C.byref(nv)))
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
    cs, n = aligner.CS, len(items)
    rec = _lib.geo_record_floats(cs)
    if records is None:
        records = torch.empty((n, rec), dtype=torch.float32, device=f"cuda:{aligner._hd.device}")
    if not (records.is_contiguous() and records.numel() >= n * rec):
        raise ValueError(f"records must be a contiguous device tensor of at least {n} x {rec} floats")
    arr = (DfkSparseGeometricItem * max(n, 1))()
    keep = []  # the host arrays must outlive the ctypes pointers until the call returns
    FP, IP = C.POINTER(C.c_float), C.POINTER(C.c_int32)
    for k, it in enumerate(items):
        c0 = np.ascontiguousarray(it["code0"], dtype=np.float32)
        c1 = np.ascontiguousarray(it["code1"], dtype=np.float32)
        if c0.shape != (cs,) or c1.shape != (cs,):
            raise ValueError(f"code0 and code1 must have {cs} entries")
        pts = np.ascontiguousarray(it["points_xy"], dtype=np.int32).reshape(-1, 2)
        keep += [c0, c1, pts]
        w = arr[k]
        w.pose0, w.pose1, w.cam = _pose(it["pose0"]), _pose(it["pose1"]), _cam(it["cam"])
        w.prx0_orig, w.prx0_jac = _image(it["prx0_orig"]), _image(it["prx0_jac"], cs)
        w.prx1_orig, w.prx1_jac = _image(it["prx1_orig"]), _image(it["prx1_jac"], cs)
        w.dpt_grad1 = _image(it["dpt_grad1"], 2)
        w.code0, w.code1, w.points_xy = c0.ctypes.data_as(FP), c1.ctypes.data_as(FP), pts.ctypes.data_as(IP)
        w.num_points = pts.shape[0]
        w.huber_delta = float(it["huber_delta"])
    check(aligner.handle, lib().dfk_sparse_geometric_linearize_batch(aligner.handle, arr, n, cs,
                                                                     C.c_void_p(records.data_ptr())))
    return records


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
    geometric links (k0, k1), one record each (SparseGeometricLinearizeBatch); their blocks follow the scalars."""

    def __init__(self, aligner: "SfmAligner", num_keyframes: int, pairs, item_pair, item_sizes, geometric=()):
        from .factors import WindowBlocks
        self._al = aligner
        self.layout = WindowBlocks(int(num_keyframes), aligner.CS, [tuple(map(int, p)) for p in pairs],
                                   [tuple(map(int, p)) for p in geometric])
        k0 = np.ascontiguousarray([p[0] for p in self.layout.pairs], dtype=np.int32)
        k1 = np.ascontiguousarray([p[1] for p in self.layout.pairs], dtype=np.int32)
        ip = np.ascontiguousarray(item_pair, dtype=np.int32)
        iw = np.ascontiguousarray([s[0] for s in item_sizes], dtype=np.int32)
        ih = np.ascontiguousarray([s[1] for s in item_sizes], dtype=np.int32)
        I32 = C.POINTER(C.c_int32)
        desc = _lib.DfkWindowDesc(int(num_keyframes), len(k0), len(ip), aligner.CS, k0.ctypes.data_as(I32),
                                  k1.ctypes.data_as(I32), ip.ctypes.data_as(I32), iw.ctypes.data_as(I32),
                                  ih.ctypes.data_as(I32))
        self.w = C.c_void_p()
        L = len(self.layout.geometric)
        if L:
            g0 = np.ascontiguousarray([p[0] for p in self.layout.geometric], dtype=np.int32)
            g1 = np.ascontiguousarray([p[1] for p in self.layout.geometric], dtype=np.int32)
            check(aligner.handle, lib().dfk_window_create_geometric(aligner.handle, C.byref(desc), L, g0.ctypes.data_as(I32),
                                                                    g1.ctypes.data_as(I32), C.byref(self.w)))
        else:
            check(aligner.handle, lib().dfk_window_create(aligner.handle, C.byref(desc), C.byref(self.w)))
        self.num_items = len(ip)
        self.floats = int(lib().dfk_window_floats(self.w))
        assert self.floats == self.layout.floats

    def assemble(self, records: torch.Tensor, out: torch.Tensor | None = None,
                 geo_records: torch.Tensor | None = None) -> torch.Tensor:
        """records: [num_items, REC] device tensor written by RunStepBatch; geo_records: [num_links, GEO_REC] written by
        SparseGeometricLinearizeBatch (required when the window has links).  Asynchronous on torch's current stream."""
        self._al._hd.use_torch_stream()
        dev = torch.device(f"cuda:{self._al._hd.device}")

        def need(t, n, what):  # the kernel reads / writes n floats of t on the handle's device
            if not (t.dtype == torch.float32 and t.device == dev and t.is_contiguous() and t.numel() >= n):
                raise ValueError(f"{what} must be a contiguous float32 tensor of at least {n} floats on {dev}")

        rec = _lib.record_floats(self.layout.code_size)
        need(records, self.num_items * rec, "records")
        if out is None:
            out = torch.empty(self.floats, dtype=torch.float32, device=records.device)
        need(out, self.floats, "out")
        if self.layout.geometric and geo_records is None:
            raise ValueError("the window has geometric links: geo_records is required")
        if geo_records is not None:
            need(geo_records, len(self.layout.geometric) * _lib.geo_record_floats(self.layout.code_size), "geo_records")
        if geo_records is None and not self.layout.geometric:
            check(self._al.handle, lib().dfk_window_assemble(self._al.handle, self.w, C.c_void_p(records.data_ptr()),
                                                             C.c_void_p(out.data_ptr())))
            return out
        geo = C.c_void_p(geo_records.data_ptr()) if geo_records is not None else None
        check(self._al.handle, lib().dfk_window_assemble_geometric(self._al.handle, self.w,
                                                                   C.c_void_p(records.data_ptr()), geo,
                                                                   C.c_void_p(out.data_ptr())))
        return out

    def close(self):
        if getattr(self, "w", None):
            lib().dfk_window_destroy(self._al.handle, self.w)
            self.w = None

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
