"""The C ABI of libdfk.so called through ctypes: every argument check an entry point can reach without a CUDA failure,
and the scratch a handle owns.

Argument checks: each row makes one bad call and pins the exact status, the exact dfk_last_error string (DFK promises
the message the reference would have thrown) and that the call wrote nothing to its outputs.  Before each row the handle
holds a known message, so a rejection that sets none (a null parameter block, for example) is pinned as well.

Scratch: a handle that linearised reprojection and sparse geometric factors holds device and pinned host scratch sized
by its largest call; destroying it must give both back."""
import ctypes as C

import numpy as np
import pytest

from deepfactors_b200 import _lib
from deepfactors_b200._lib import (DfkCamera, DfkImage, DfkReprojectionItem, DfkSfmAlignerParams, DfkSfmWorkItem,
                                   DfkTrackLevel, DfkWindowDesc)

pytestmark = pytest.mark.gpu

INV, UNS = _lib.DFK_ERR_INVALID_ARG, _lib.DFK_ERR_UNSUPPORTED
W, H, CS = 32, 24, 8
SENT = -7.25  # what "left untouched" looks like
PRIME = "[dfk_set_sm_limit] num_sms < 0"  # the handle's message before every row
FP = C.POINTER(C.c_float)
GRAM_AUTO, GRAM_TF32X3 = _lib.DFK_GRAM_AUTO, _lib.DFK_GRAM_TF32X3
_KEEP = []


@pytest.fixture(scope="module")
def env():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = _lib.lib()
    h = C.c_void_p()
    assert lib.dfk_create(torch.cuda.current_device(), C.byref(h)) == _lib.DFK_OK
    e = Env(torch, lib, h)
    yield e
    for s in e.streams:
        lib.dfk_sfm_stream_destroy(h, s)
    lib.dfk_destroy(h)


class Env:
    def __init__(self, torch, lib, h):
        self.torch, self.lib, self.h = torch, lib, h
        # every device view points into this buffer: a check that unexpectedly passes reads real memory
        self.dev = torch.zeros(W * H * 260, device="cuda")
        self.host = np.zeros(W * H * 260, np.float32)  # the same for the host views of the stream
        self.records = torch.full((4, _lib.record_floats(128)), SENT, device="cuda")
        self.code = np.zeros(256, np.float32)
        self.streams = []
        self.defaults = DfkSfmAlignerParams()
        assert lib.dfk_sfm_get_params(h, C.byref(self.defaults)) == _lib.DFK_OK

    def img(self, fpp=1, w=W, h=H, off=0, pitch=None, host=False, null=False):
        base = self.host.ctypes.data if host else self.dev.data_ptr()
        return DfkImage(None if null else base + off, w * fpp * 4 if pitch is None else pitch, w, h)

    def stream(self, code_size=CS, max_items=2, depth=1):
        s = C.c_void_p()
        assert self.lib.dfk_sfm_stream_create(self.h, code_size, max_items, 1 << 16, depth, C.byref(s)) == _lib.DFK_OK
        self.streams.append(s)
        return s


class Outs:
    """host outputs of one row, filled with a sentinel; a rejected call must leave them as they are"""

    def __init__(self):
        self.arrays = []
        self.ptrs = []

    def _keep(self, a):
        self.arrays.append((a, a.copy()))
        return a

    def f(self, n=1):
        return self._keep(np.full(n, SENT, np.float32)).ctypes.data_as(FP)

    def u64(self):
        return self._keep(np.full(1, 0xDEADBEEF, np.uint64)).ctypes.data_as(C.POINTER(C.c_uint64))

    def i32(self, n=1):
        return self._keep(np.full(n, -7, np.int32)).ctypes.data_as(C.POINTER(C.c_int))

    def ptr(self, expect_after):
        """an object out-parameter preset to 0xBAD0; expect_after: its value after the rejected call"""
        p = C.c_void_p(0xBAD0)
        self.ptrs.append((p, expect_after))
        return C.byref(p)

    def check(self):
        for a, before in self.arrays:
            assert np.array_equal(a, before)
        for p, want in self.ptrs:
            assert p.value == want


def pose():
    return (C.c_float * 7)(0, 0, 0, 1, 0, 0, 0)


def cam(w=W, h=H):
    return DfkCamera(20.0, 20.0, W / 2, H / 2, float(w), float(h))


def ref(x):
    return C.byref(x)


def sfm_item(e, host=False, **kw):
    it = DfkSfmWorkItem()
    it.pose0, it.pose1, it.cam = pose(), pose(), cam()
    for name, fpp in (("img0", 1), ("img1", 1), ("dpt0", 1), ("valid0", 1), ("prx0_jac", CS), ("grad1", 2)):
        setattr(it, name, e.img(fpp, host=host))
    for k, v in kw.items():
        setattr(it, k, v)
    return it


def sfm_items(*its):
    return (DfkSfmWorkItem * len(its))(*its)


def level(e, iterations=2, **kw):
    L = DfkTrackLevel(cam(), e.img(), e.img(), e.img(), e.img(2), iterations)
    for k, v in kw.items():
        setattr(L, k, v)
    return L


def levels(*ls):
    return (DfkTrackLevel * len(ls))(*ls)


def rep_item(e, code_size=CS, **kw):
    q = e.code.ctypes.data_as(FP)
    it = DfkReprojectionItem(pose(), pose(), cam(), e.img(), e.img(code_size), q, 1, q, q, 1.0, 1.0)
    for k, v in kw.items():
        setattr(it, k, v)
    return it


def rep_items(*its):
    return (DfkReprojectionItem * len(its))(*its)


def window(K=2, P=1, n=2, code_size=CS, k0=(0,), k1=(1,), pair=(0, 0), wh=((W, H), (W // 2, H // 2))):
    arrs = [np.array(a, np.int32) for a in (k0, k1, pair, [x for x, _ in wh], [y for _, y in wh])]
    ip = C.POINTER(C.c_int32)
    _KEEP.extend(arrs)  # the descriptor only points at them
    return DfkWindowDesc(K, P, n, code_size, *[a.ctypes.data_as(ip) for a in arrs])


def with_gram(e, mode, fn):
    assert e.lib.dfk_sfm_set_gram_mode(e.h, mode) == _lib.DFK_OK
    try:
        return fn()
    finally:
        assert e.lib.dfk_sfm_set_gram_mode(e.h, GRAM_AUTO) == _lib.DFK_OK


def params(e, **kw):
    p = DfkSfmAlignerParams.from_buffer_copy(e.defaults)
    for k, v in kw.items():
        if k == "valid_border":
            p.sfmparams.valid_border = v
        else:
            setattr(p, k, v)
    return p


def tracking_rows():
    RS = "[SfmAligner::RunStep] "
    TF = "[CameraTracker::TrackFrame] "
    TB = "[CameraTracker::TrackFrame batch] "
    BAD_LEVEL = "inconsistent image views / camera larger than them / negative iteration count at "
    return [
        # ---- handle settings
        ("set_sm_limit", lambda e, o: e.lib.dfk_set_sm_limit(e.h, -1), INV, PRIME),
        ("set_params/null", lambda e, o: e.lib.dfk_sfm_set_params(e.h, None), INV, PRIME),
        ("set_params/step_threads", lambda e, o: e.lib.dfk_sfm_set_params(e.h, ref(params(e, step_threads=33))), INV,
         "threads must be a multiple of 32!"),
        ("set_params/eval_threads", lambda e, o: e.lib.dfk_sfm_set_params(e.h, ref(params(e, eval_threads=48))), INV,
         "threads must be a multiple of 32!"),
        ("set_params/step_blocks", lambda e, o: e.lib.dfk_sfm_set_params(e.h, ref(params(e, step_blocks=1025))), INV,
         "blocks must be less than 1024"),
        ("set_params/eval_blocks", lambda e, o: e.lib.dfk_sfm_set_params(e.h, ref(params(e, eval_blocks=1025))), INV,
         "blocks must be less than 1024"),
        ("set_params/valid_border", lambda e, o: e.lib.dfk_sfm_set_params(e.h, ref(params(e, valid_border=0))), INV,
         "valid_border must be >= 1 (bilinear sampling reads ix+1, iy+1)"),
        ("get_params/null", lambda e, o: e.lib.dfk_sfm_get_params(e.h, None), INV, PRIME),
        ("set_gram_mode", lambda e, o: e.lib.dfk_sfm_set_gram_mode(e.h, 7), INV, "unknown gram mode"),
        # ---- SfmAligner::RunStep, batched into device records
        ("run_step_batch/null_items", lambda e, o: e.lib.dfk_sfm_run_step_batch(e.h, None, 1, CS, e.records.data_ptr()),
         INV, RS + "null/empty batch"),
        ("run_step_batch/n0", lambda e, o: e.lib.dfk_sfm_run_step_batch(e.h, sfm_items(sfm_item(e)), 0, CS,
                                                                         e.records.data_ptr()), INV, RS + "null/empty batch"),
        ("run_step_batch/null_records", lambda e, o: e.lib.dfk_sfm_run_step_batch(e.h, sfm_items(sfm_item(e)), 1, CS, None),
         INV, RS + "null/empty batch"),
        ("run_step_batch/code_size", lambda e, o: e.lib.dfk_sfm_run_step_batch(e.h, sfm_items(sfm_item(e)), 1, 12,
                                                                                e.records.data_ptr()),
         UNS, RS + "no kernel instantiated for code size 12"),
        ("run_step_batch/tc_misaligned_grad", lambda e, o: with_gram(e, GRAM_TF32X3, lambda: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e, grad1=e.img(2, off=4))), 1, 32, e.records.data_ptr())),
         UNS, RS + "tensor-core path needs 8-byte aligned grad1 rows"),
        ("run_step_batch/tc_null_grad", lambda e, o: with_gram(e, GRAM_TF32X3, lambda: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e, grad1=e.img(2, null=True))), 1, 32, e.records.data_ptr())),
         UNS, RS + "tensor-core path needs 8-byte aligned grad1 rows"),
        ("run_step_batch/tc_code_size", lambda e, o: with_gram(e, GRAM_TF32X3, lambda: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e)), 1, CS, e.records.data_ptr())),
         UNS, RS + "tensor-core Gram path is not instantiated for code size 8"),
        ("run_step_batch/empty_image", lambda e, o: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e), sfm_item(e, img0=e.img(w=0))), 2, CS, e.records.data_ptr()),
         INV, RS + "empty image"),
        ("run_step_batch/views", lambda e, o: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e), sfm_item(e, prx0_jac=e.img(CS, pitch=4 * CS * W - 4))), 2, CS, e.records.data_ptr()),
         INV, RS + "inconsistent image views (size, pitch or null pointer) in work item 1"),
        ("run_step_batch/camera", lambda e, o: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e, cam=cam(W + 1))), 1, CS, e.records.data_ptr()),
         INV, RS + "camera viewport larger than the image views in work item 0"),
        ("run_step_batch/fused_prx_orig", lambda e, o: e.lib.dfk_sfm_run_step_batch(
            e.h, sfm_items(sfm_item(e), sfm_item(e, code=e.code.ctypes.data_as(FP))), 2, CS, e.records.data_ptr()),
         INV, RS + "fused depth decode: inconsistent prx_orig view in work item 1"),
        # ---- ... into host records
        ("run_step_batch_host/n0", lambda e, o: e.lib.dfk_sfm_run_step_batch_host(e.h, sfm_items(sfm_item(e)), 0, CS,
                                                                                   o.f(2000)), INV, RS + "null/empty batch"),
        ("run_step_batch_host/null_records", lambda e, o: e.lib.dfk_sfm_run_step_batch_host(
            e.h, sfm_items(sfm_item(e)), 1, CS, None), INV, RS + "null/empty batch"),
        ("run_step_batch_host/code_size", lambda e, o: e.lib.dfk_sfm_run_step_batch_host(
            e.h, sfm_items(sfm_item(e)), 1, 12, o.f(2000)), UNS, RS + "no kernel instantiated for code size 12"),
        ("run_step_batch_host/null_items", lambda e, o: e.lib.dfk_sfm_run_step_batch_host(e.h, None, 1, CS, o.f(2000)),
         INV, RS + "null/empty batch"),
        ("run_step_batch_host/views", lambda e, o: e.lib.dfk_sfm_run_step_batch_host(
            e.h, sfm_items(sfm_item(e, dpt0=e.img(h=H - 1))), 1, CS, o.f(2000)),
         INV, RS + "inconsistent image views (size, pitch or null pointer) in work item 0"),
        # ---- single RunStep
        ("run_step/null", lambda e, o: e.lib.dfk_sfm_run_step(
            e.h, None, pose(), None, CS, cam(), ref(e.img()), ref(e.img()), ref(e.img()), None, ref(e.img()),
            ref(e.img(CS)), ref(e.img(2)), o.f(210), o.f(20), o.f(), o.u64()), INV, RS + "null argument"),
        ("run_step/code_size", lambda e, o: e.lib.dfk_sfm_run_step(
            e.h, pose(), pose(), None, 12, cam(), ref(e.img()), ref(e.img()), ref(e.img()), None, ref(e.img()),
            ref(e.img(12)), ref(e.img(2)), o.f(210), o.f(20), o.f(), o.u64()),
         UNS, RS + "no kernel instantiated for code size 12"),
        ("run_step/camera", lambda e, o: e.lib.dfk_sfm_run_step(
            e.h, pose(), pose(), None, CS, cam(h=H + 1), ref(e.img()), ref(e.img()), ref(e.img()), None, ref(e.img()),
            ref(e.img(CS)), ref(e.img(2)), o.f(210), o.f(20), o.f(), o.u64()),
         INV, RS + "camera viewport larger than the image views in work item 0"),
        # ---- EvaluateError
        ("evaluate_error/null", lambda e, o: e.lib.dfk_sfm_evaluate_error(
            e.h, pose(), pose(), cam(), ref(e.img()), ref(e.img()), None, None, None, o.f(), o.u64()),
         INV, "[SfmAligner::EvaluateError] null argument"),
        ("evaluate_error/views", lambda e, o: e.lib.dfk_sfm_evaluate_error(
            e.h, pose(), pose(), cam(), ref(e.img()), ref(e.img(w=W - 1)), ref(e.img()), None, None, o.f(), o.u64()),
         INV, "[SfmAligner::EvaluateError] inconsistent image views"),
        ("evaluate_error/camera", lambda e, o: e.lib.dfk_sfm_evaluate_error(
            e.h, pose(), pose(), cam(-1.0), ref(e.img()), ref(e.img()), ref(e.img()), None, None, o.f(), o.u64()),
         INV, "[SfmAligner::EvaluateError] camera viewport larger than the image views"),
        # ---- SE3Aligner
        ("se3_run_step/null", lambda e, o: e.lib.dfk_se3_run_step(
            e.h, pose(), cam(), ref(e.img()), ref(e.img()), ref(e.img()), ref(e.img(2)), o.f(21), o.f(6), o.f(), None),
         INV, "[SE3Aligner::RunStep] null argument"),
        ("se3_run_step/views", lambda e, o: e.lib.dfk_se3_run_step(
            e.h, pose(), cam(), ref(e.img()), ref(e.img()), ref(e.img()), ref(e.img(1)), o.f(21), o.f(6), o.f(), o.u64()),
         INV, "[SE3Aligner::RunStep] inconsistent image views"),
        ("se3_run_step/camera", lambda e, o: e.lib.dfk_se3_run_step(
            e.h, pose(), cam(W + 1), ref(e.img()), ref(e.img()), ref(e.img()), ref(e.img(2)), o.f(21), o.f(6), o.f(),
            o.u64()), INV, "[SE3Aligner::RunStep] camera viewport larger than the image views"),
        ("se3_warp/null", lambda e, o: e.lib.dfk_se3_warp(
            e.h, pose(), cam(), ref(e.img()), ref(e.img()), ref(e.img()), None, o.f(), o.u64()),
         INV, "[SE3Aligner::Warp] null argument"),
        ("se3_warp/views", lambda e, o: e.lib.dfk_se3_warp(
            e.h, pose(), cam(), ref(e.img()), ref(e.img()), ref(e.img()), ref(e.img(null=True)), o.f(), o.u64()),
         INV, "[SE3Aligner::Warp] inconsistent image views"),
        ("se3_warp/camera", lambda e, o: e.lib.dfk_se3_warp(
            e.h, pose(), cam(h=H + 0.5), ref(e.img()), ref(e.img()), ref(e.img()), ref(e.img()), o.f(), o.u64()),
         INV, "[SE3Aligner::Warp] camera viewport larger than the image views"),
        # ---- tracker
        ("se3_track/null_pose", lambda e, o: e.lib.dfk_se3_track(
            e.h, None, levels(level(e)), 1, o.f(), o.f(), o.f(29), o.f(72), 2), INV, TF + "null argument / no pyramid levels"),
        ("se3_track/null_levels", lambda e, o: e.lib.dfk_se3_track(
            e.h, o.f(7), None, 1, o.f(), o.f(), o.f(29), o.f(72), 2), INV, TF + "null argument / no pyramid levels"),
        ("se3_track/no_levels", lambda e, o: e.lib.dfk_se3_track(
            e.h, o.f(7), levels(level(e)), 0, o.f(), o.f(), o.f(29), o.f(72), 2), INV, TF + "null argument / no pyramid levels"),
        ("se3_track/negative_iterations", lambda e, o: e.lib.dfk_se3_track(
            e.h, o.f(7), levels(level(e), level(e, -1)), 2, o.f(), o.f(), o.f(29), None, 0), INV, TF + BAD_LEVEL + "level 1"),
        ("se3_track/camera", lambda e, o: e.lib.dfk_se3_track(
            e.h, o.f(7), levels(level(e, cam=cam(W + 1)), level(e)), 2, o.f(), o.f(), o.f(29), None, 0),
         INV, TF + BAD_LEVEL + "level 0"),
        ("se3_track/views", lambda e, o: e.lib.dfk_se3_track(
            e.h, o.f(7), levels(level(e), level(e, grad1=e.img(2, w=W - 1))), 2, o.f(), o.f(), o.f(29), None, 0),
         INV, TF + BAD_LEVEL + "level 1"),
        ("se3_track/history", lambda e, o: e.lib.dfk_se3_track(
            e.h, o.f(7), levels(level(e, 2), level(e, 3)), 2, o.f(), o.f(), o.f(29), o.f(36 * 5), 4),
         INV, TF + "history buffer too small"),
        ("se3_track_batch/null_poses", lambda e, o: e.lib.dfk_se3_track_batch(
            e.h, 1, 1, None, levels(level(e)), o.f(), o.f(), o.f(29)), INV, TB + "null argument / no pyramid levels"),
        ("se3_track_batch/no_levels", lambda e, o: e.lib.dfk_se3_track_batch(
            e.h, 1, 0, o.f(7), levels(level(e)), o.f(), o.f(), o.f(29)), INV, TB + "null argument / no pyramid levels"),
        ("se3_track_batch/n0", lambda e, o: e.lib.dfk_se3_track_batch(
            e.h, 0, 1, o.f(7), levels(level(e)), o.f(), o.f(), o.f(29)),
         INV, TB + "number of problems must be in [1, 65535]"),
        ("se3_track_batch/n65536", lambda e, o: e.lib.dfk_se3_track_batch(
            e.h, 65536, 1, o.f(7), levels(level(e)), o.f(), o.f(), o.f(29)),
         INV, TB + "number of problems must be in [1, 65535]"),
        ("se3_track_batch/views", lambda e, o: e.lib.dfk_se3_track_batch(
            e.h, 2, 2, o.f(14), levels(level(e), level(e), level(e), level(e, img1=e.img(null=True))), o.f(2), o.f(2),
            o.f(58)), INV, TB + BAD_LEVEL + "problem 1 level 1"),
        ("se3_track_batch/schedule", lambda e, o: e.lib.dfk_se3_track_batch(
            e.h, 2, 2, o.f(14), levels(level(e, 2), level(e, 1), level(e, 3), level(e, 1)), o.f(2), o.f(2), o.f(58)),
         INV, TB + "problem 1 has 3 iterations at level 0, problem 0 has 2"),
    ]


def image_and_factor_rows():
    RF = "[ReprojectionFactor::linearize] "
    RB = "[ReprojectionFactor::linearize batch] "
    SG = "[SparseGeometricFactor::linearize] "
    DA = "[DepthAligner::RunStep] "
    code = lambda e: e.code.ctypes.data_as(FP)  # noqa: E731

    def rep(e, o, code_size=CS, num_matches=5, sigma=1.0, prx_jac=None, null_query=False):
        return e.lib.dfk_reprojection_linearize(
            e.h, pose(), pose(), code(e), code_size, cam(), ref(e.img()), ref(prx_jac or e.img(code_size)), num_matches,
            None if null_query else code(e), code(e), 1.0, sigma, o.f(2 * 5 * (13 + 128)), o.f())

    def sg(e, o, code_size=CS, num_points=5, huber=0.1, cam_=None, dpt_grad1=None, null_points=False):
        pts = np.ones(10, np.int32)
        o._keep(pts)
        return e.lib.dfk_sparse_geometric_linearize(
            e.h, pose(), pose(), code(e), code(e), code_size, cam_ or cam(), ref(e.img()), ref(e.img(code_size)),
            ref(e.img()), ref(e.img(code_size)), ref(dpt_grad1 or e.img(2)), num_points,
            None if null_points else pts.ctypes.data_as(C.POINTER(C.c_int)), huber, o.f(5 * (13 + 256)), o.i32())

    big = 2 ** 31 - 1
    return [
        ("update_depth/null", lambda e, o: e.lib.dfk_update_depth(e.h, None, CS, ref(e.img()), ref(e.img(CS)), 2.0,
                                                                  ref(e.img())), INV, "[UpdateDepth] null argument"),
        ("update_depth/code_size0", lambda e, o: e.lib.dfk_update_depth(e.h, code(e), 0, ref(e.img()), ref(e.img()), 2.0,
                                                                        ref(e.img())), UNS, "[UpdateDepth] code size out of range"),
        ("update_depth/code_size257", lambda e, o: e.lib.dfk_update_depth(e.h, code(e), 257, ref(e.img()), ref(e.img()),
                                                                          2.0, ref(e.img())),
         UNS, "[UpdateDepth] code size out of range"),
        ("update_depth/views", lambda e, o: e.lib.dfk_update_depth(e.h, code(e), CS, ref(e.img()), ref(e.img(CS - 1)), 2.0,
                                                                   ref(e.img())), INV, "[UpdateDepth] inconsistent image views"),
        ("sobel/null", lambda e, o: e.lib.dfk_sobel_gradients(e.h, ref(e.img()), None), INV, "[SobelGradients] null argument"),
        ("sobel/views", lambda e, o: e.lib.dfk_sobel_gradients(e.h, ref(e.img()), ref(e.img(1))),
         INV, "[SobelGradients] inconsistent image views"),
        ("blur_down/null", lambda e, o: e.lib.dfk_gaussian_blur_down(e.h, None, ref(e.img())),
         INV, "[GaussianBlurDown] null argument"),
        ("blur_down/views", lambda e, o: e.lib.dfk_gaussian_blur_down(e.h, ref(e.img()), ref(e.img(w=0))),
         INV, "[GaussianBlurDown] inconsistent image views"),
        ("pyramid/null", lambda e, o: e.lib.dfk_build_image_pyramid(e.h, None, None, 2),
         INV, "[BuildImagePyramid] null argument / no levels"),
        ("pyramid/no_levels", lambda e, o: e.lib.dfk_build_image_pyramid(e.h, (DfkImage * 1)(e.img()), None, 0),
         INV, "[BuildImagePyramid] null argument / no levels"),
        ("pyramid/level_view", lambda e, o: e.lib.dfk_build_image_pyramid(
            e.h, (DfkImage * 2)(e.img(), e.img(pitch=3)), None, 2), INV, "[GaussianBlurDown] inconsistent image views"),
        ("pyramid/grad_view", lambda e, o: e.lib.dfk_build_image_pyramid(
            e.h, (DfkImage * 1)(e.img()), (DfkImage * 1)(e.img()), 1), INV, "[SobelGradients] inconsistent image views"),
        ("squared_error/null", lambda e, o: e.lib.dfk_squared_error(e.h, ref(e.img()), ref(e.img()), None),
         INV, "[SquaredError] null argument"),
        ("squared_error/views", lambda e, o: e.lib.dfk_squared_error(e.h, ref(e.img()), ref(e.img(h=H - 1)), o.f()),
         INV, "[SquaredError] inconsistent image views"),
        # ---- DepthAligner
        ("depth_run_step/null", lambda e, o: e.lib.dfk_depth_run_step(
            e.h, code(e), CS, ref(e.img()), ref(e.img()), ref(e.img(CS)), o.f(36), None, o.f(), o.u64()),
         INV, DA + "null argument"),
        ("depth_run_step/code_size", lambda e, o: e.lib.dfk_depth_run_step(
            e.h, code(e), 12, ref(e.img()), ref(e.img()), ref(e.img(12)), o.f(80), o.f(12), o.f(), o.u64()),
         UNS, "DepthAligner used with a different code size than it was compiled for: 12"),
        ("depth_run_step/code_size256", lambda e, o: e.lib.dfk_depth_run_step(
            e.h, code(e), 256, ref(e.img()), ref(e.img()), ref(e.img(256)), o.f(10), o.f(10), o.f(), o.u64()),
         UNS, "DepthAligner used with a different code size than it was compiled for: 256"),
        ("depth_run_step/views", lambda e, o: e.lib.dfk_depth_run_step(
            e.h, code(e), CS, ref(e.img()), ref(e.img(null=True)), ref(e.img(CS)), o.f(36), o.f(8), o.f(), o.u64()),
         INV, DA + "inconsistent image views"),
        # ---- ReprojectionFactor
        ("reprojection/null", lambda e, o: rep(e, o, null_query=True), INV, RF + "null argument"),
        ("reprojection/code_size", lambda e, o: rep(e, o, code_size=12), UNS, RF + "code size not instantiated: 12"),
        ("reprojection/no_matches", lambda e, o: rep(e, o, num_matches=0), INV, RF + "no matches / non-positive sigma"),
        ("reprojection/sigma", lambda e, o: rep(e, o, sigma=0.0), INV, RF + "no matches / non-positive sigma"),
        ("reprojection/sigma_nan", lambda e, o: rep(e, o, sigma=float("nan")), INV, RF + "no matches / non-positive sigma"),
        ("reprojection/views", lambda e, o: rep(e, o, prx_jac=e.img(CS, h=H + 1)), INV, RF + "inconsistent image views"),
        ("reprojection_batch/null_items", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, None, 1, CS, e.records.data_ptr()), INV, RB + "null argument / empty batch"),
        ("reprojection_batch/n0", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e)), 0, CS, e.records.data_ptr()), INV, RB + "null argument / empty batch"),
        ("reprojection_batch/null_records", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e)), 1, CS, None), INV, RB + "null argument / empty batch"),
        ("reprojection_batch/code_size", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e)), 1, 12, e.records.data_ptr()), UNS, RB + "code size not instantiated: 12"),
        ("reprojection_batch/null_code", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e), rep_item(e, code=None)), 2, CS, e.records.data_ptr()),
         INV, RB + "item 1: null argument"),
        ("reprojection_batch/no_matches", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e), rep_item(e, num_matches=0)), 2, CS, e.records.data_ptr()),
         INV, RB + "item 1: no matches / non-positive sigma"),
        ("reprojection_batch/sigma", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e, sigma=-1.0)), 1, CS, e.records.data_ptr()),
         INV, RB + "item 0: no matches / non-positive sigma"),
        ("reprojection_batch/views", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e), rep_item(e, prx_orig=e.img(pitch=4 * W - 4))), 2, CS, e.records.data_ptr()),
         INV, RB + "item 1: inconsistent image views"),
        ("reprojection_batch/too_many_matches", lambda e, o: e.lib.dfk_reprojection_linearize_batch(
            e.h, rep_items(rep_item(e, num_matches=big), rep_item(e)), 2, CS, e.records.data_ptr()),
         INV, RB + "more than 2^31 - 1 matches in one call"),
        # ---- SparseGeometricFactor
        ("sparse_geometric/null", lambda e, o: sg(e, o, null_points=True), INV, SG + "null argument"),
        ("sparse_geometric/code_size", lambda e, o: sg(e, o, code_size=12), UNS, SG + "code size not instantiated: 12"),
        ("sparse_geometric/no_points", lambda e, o: sg(e, o, num_points=0), INV, SG + "no points / non-positive huber delta"),
        ("sparse_geometric/huber", lambda e, o: sg(e, o, huber=0.0), INV, SG + "no points / non-positive huber delta"),
        ("sparse_geometric/views", lambda e, o: sg(e, o, dpt_grad1=e.img(2, w=W + 1)), INV, SG + "inconsistent image views"),
        ("sparse_geometric/camera", lambda e, o: sg(e, o, cam_=cam(W + 1)), INV, SG + "camera larger than the image views"),
    ]


def window_and_stream_rows():
    WN = "[Window] "
    ST = "[SfmStream] "
    BAD = ST + "bad argument (1 <= depth <= 16, max_items > 0, max_bytes > 0)"

    def create(e, o, d, expect_out=0):
        return e.lib.dfk_window_create(e.h, ref(d) if d is not None else None, o.ptr(expect_out or None))

    def stream_create(e, o, code_size=CS, max_items=2, max_bytes=1 << 16, depth=2, null_out=False, cleared=True):
        return e.lib.dfk_sfm_stream_create(e.h, code_size, max_items, max_bytes, depth,
                                           None if null_out else o.ptr(None if cleared else 0xBAD0))

    def submit(e, o, n=1, its=None, null_ticket=False):
        s = e.stream(max_items=2)
        its = its if its is not None else sfm_items(sfm_item(e, host=True))
        t = C.c_uint64(77)
        st = e.lib.dfk_sfm_stream_submit(e.h, s, its, n, None if null_ticket else C.byref(t))
        assert t.value == 77
        return st

    return [
        ("window_create/null_desc", lambda e, o: create(e, o, None, 0xBAD0), INV, WN + "null argument"),
        ("window_create/null_out", lambda e, o: e.lib.dfk_window_create(e.h, ref(window()), None), INV, WN + "null argument"),
        ("window_create/empty", lambda e, o: create(e, o, window(K=0)), INV, WN + "empty window / null index array"),
        ("window_create/no_items", lambda e, o: create(e, o, window(n=0)), INV, WN + "empty window / null index array"),
        ("window_create/code_size", lambda e, o: create(e, o, window(code_size=12)),
         UNS, WN + "no RunStep kernel for code size 12"),
        ("window_create/pair", lambda e, o: create(e, o, window(P=2, k0=(0, 1), k1=(1, 2))),
         INV, WN + "pair 1 names a keyframe outside the window"),
        ("window_create/record_pair", lambda e, o: create(e, o, window(pair=(0, 1))),
         INV, WN + "record 1 names a pair outside the window"),
        ("window_create/record_size", lambda e, o: create(e, o, window(wh=((W, H), (W, 0)))),
         INV, WN + "record 1 names a pair outside the window"),
        ("window_assemble/null", lambda e, o: e.lib.dfk_window_assemble(e.h, None, e.records.data_ptr(),
                                                                        e.records.data_ptr()), INV, WN + "null argument"),
        ("stream_create/null_out", lambda e, o: stream_create(e, o, null_out=True), INV, BAD),
        ("stream_create/depth0", lambda e, o: stream_create(e, o, depth=0, cleared=False), INV, BAD),
        ("stream_create/depth17", lambda e, o: stream_create(e, o, depth=17, cleared=False), INV, BAD),
        ("stream_create/max_items", lambda e, o: stream_create(e, o, max_items=0, cleared=False), INV, BAD),
        ("stream_create/max_bytes", lambda e, o: stream_create(e, o, max_bytes=0, cleared=False), INV, BAD),
        ("stream_create/code_size", lambda e, o: stream_create(e, o, code_size=12),
         UNS, ST + "no RunStep kernel for code size 12"),
        ("stream_submit/null_stream", lambda e, o: e.lib.dfk_sfm_stream_submit(
            e.h, None, sfm_items(sfm_item(e, host=True)), 1, C.byref(C.c_uint64())), INV, ST + "null argument / empty submission"),
        ("stream_submit/null_items", lambda e, o: submit(e, o, its=C.POINTER(DfkSfmWorkItem)()),
         INV, ST + "null argument / empty submission"),
        ("stream_submit/null_ticket", lambda e, o: submit(e, o, null_ticket=True), INV, ST + "null argument / empty submission"),
        ("stream_submit/n0", lambda e, o: submit(e, o, n=0), INV, ST + "null argument / empty submission"),
        ("stream_submit/too_many", lambda e, o: submit(e, o, n=3, its=sfm_items(*[sfm_item(e, host=True)] * 3)),
         INV, ST + "more work items than the stream was created for"),
        ("stream_submit/views", lambda e, o: submit(e, o, n=2, its=sfm_items(
            sfm_item(e, host=True), sfm_item(e, host=True, grad1=e.img(1, host=True)))),
         INV, ST + "inconsistent host image views in work item 1"),
        ("stream_submit/fused_views", lambda e, o: submit(e, o, its=sfm_items(sfm_item(e, host=True, code=e.code.ctypes.data_as(FP)))),
         INV, ST + "inconsistent host image views in work item 0"),
        ("stream_wait/null_stream", lambda e, o: e.lib.dfk_sfm_stream_wait(e.h, None, 0, o.f(2000)), INV, ST + "null argument"),
        ("stream_wait/null_records", lambda e, o: e.lib.dfk_sfm_stream_wait(e.h, e.stream(), 0, None),
         INV, ST + "null argument"),
        ("stream_wait/nothing_submitted", lambda e, o: e.lib.dfk_sfm_stream_wait(e.h, e.stream(), 0, o.f(2000)),
         INV, ST + "tickets must be waited for once, in submission order"),
    ]


ROWS = tracking_rows() + image_and_factor_rows() + window_and_stream_rows()


@pytest.mark.parametrize("row", ROWS, ids=[r[0] for r in ROWS])
def test_rejected_call(env, row):
    _, fn, want_status, want_msg = row
    e = env
    assert e.lib.dfk_set_sm_limit(e.h, -1) == INV  # the message a row that sets none must leave in place
    assert e.lib.dfk_last_error(e.h).decode() == PRIME
    o = Outs()
    st = fn(e, o)
    msg = e.lib.dfk_last_error(e.h).decode()
    assert (st, msg) == (want_status, want_msg)
    o.check()
    assert e.lib.dfk_synchronize(e.h) == _lib.DFK_OK
    e.torch.cuda.synchronize()
    assert (e.records == SENT).all()
    p = DfkSfmAlignerParams()
    assert e.lib.dfk_sfm_get_params(e.h, C.byref(p)) == _lib.DFK_OK
    assert bytes(p) == bytes(e.defaults)


def test_stream_tickets_are_checked(env):
    """a stream of depth 1: a second submission before the wait, a wait out of order and a second wait are refused"""
    e = env
    lib, s = e.lib, e.stream(max_items=1, depth=1)
    ST = "[SfmStream] "
    t = C.c_uint64(77)
    rec = np.full(_lib.record_floats(CS), SENT, np.float32)
    assert lib.dfk_sfm_stream_submit(e.h, s, sfm_items(sfm_item(e, host=True)), 1, C.byref(t)) == _lib.DFK_OK
    assert t.value == 0
    assert lib.dfk_sfm_stream_submit(e.h, s, sfm_items(sfm_item(e, host=True)), 1, C.byref(t)) == INV
    assert lib.dfk_last_error(e.h).decode() == ST + "1 submissions outstanding: wait for ticket 0 first"
    assert t.value == 0
    wait = lambda ticket: lib.dfk_sfm_stream_wait(e.h, s, ticket, rec.ctypes.data_as(FP))  # noqa: E731
    order = ST + "tickets must be waited for once, in submission order"
    assert wait(1) == INV and lib.dfk_last_error(e.h).decode() == order
    assert (rec == SENT).all()
    assert wait(0) == _lib.DFK_OK
    rec[:] = SENT
    assert wait(0) == INV and lib.dfk_last_error(e.h).decode() == order
    assert (rec == SENT).all()


def test_null_handle():
    """every entry point that takes a handle refuses a null one and writes no message anywhere; destroy calls accept
    null"""
    lib = _lib.lib()
    no_handle = {"dfk_version", "dfk_status_string", "dfk_sfm_supports_code_size", "dfk_create", "dfk_window_floats"}
    accepts_null = {"dfk_destroy", "dfk_window_destroy", "dfk_sfm_stream_destroy"}
    for name, (res, args) in _lib.SYMBOLS.items():
        if name in no_handle:
            continue
        zero = [0.0 if a in (C.c_float, C.c_double) else (0 if a in (C.c_int, C.c_size_t, C.c_uint64) else None)
                for a in args]
        got = getattr(lib, name)(*zero)
        if name == "dfk_last_error":
            assert got == b"null handle"
        elif name == "dfk_get_stream":
            assert got is None
        else:
            assert got == (_lib.DFK_OK if name in accepts_null else INV), name
    assert lib.dfk_create(0, None) == INV
    assert lib.dfk_window_floats(None) == 0


def _vmrss():
    with open("/proc/self/status") as f:
        for line in f:
            if line.startswith("VmRSS:"):
                return int(line.split()[1]) * 1024
    raise RuntimeError("no VmRSS")


def test_destroy_frees_the_sparse_factor_scratch():
    """dfk_reprojection_linearize (400k matches) and dfk_sparse_geometric_linearize (300k points) at C = 128 leave
    ~460 MB of device scratch and as much pinned host memory in the handle; three create / linearise / destroy cycles
    after a warm-up one must not grow device use or the resident set by more than 96 MB (a quarter of one cycle's
    scratch, so a leak of either buffer fails by 4x or more per cycle).  The sizes are chosen for that margin on a shared
    card: shrinking them, or raising the allowance, needs the margin rechecked (the assert on `scratch` below)"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = _lib.lib()
    cs, M, P, w, h = 128, 400_000, 300_000, 64, 48
    rng = np.random.default_rng(0)
    prx = torch.from_numpy(rng.uniform(0.5, 1.5, (h, w)).astype(np.float32)).cuda()
    jac = torch.from_numpy(rng.uniform(-0.01, 0.01, (h, w, cs)).astype(np.float32)).cuda()
    grad = torch.from_numpy(rng.uniform(-1, 1, (h, w, 2)).astype(np.float32)).cuda()
    im = lambda t, k: DfkImage(t.data_ptr(), w * k * 4, w, h)  # noqa: E731
    camera = DfkCamera(50.0, 50.0, w / 2, h / 2, float(w), float(h))
    code = np.zeros(cs, np.float32)
    query = rng.uniform(0, [w, h], (M, 2)).astype(np.float32)
    train = rng.uniform(0, [w, h], (M, 2)).astype(np.float32)
    points = rng.integers([2, 2], [w - 2, h - 2], (P, 2)).astype(np.int32)
    rep_rows = np.empty(2 * M * (13 + cs), np.float32)
    sg_rows = np.empty(P * (13 + 2 * cs), np.float32)
    tot, nv = C.c_float(), C.c_int()
    p0 = (C.c_float * 7)(0, 0, 0, 1, 0, 0, 0)
    p1 = (C.c_float * 7)(0, 0, 0, 1, 0.01, 0, 0)
    c = code.ctypes.data_as(FP)

    def cycle():
        hd = C.c_void_p()
        assert lib.dfk_create(torch.cuda.current_device(), C.byref(hd)) == _lib.DFK_OK
        try:
            assert lib.dfk_reprojection_linearize(hd, p0, p1, c, cs, C.byref(camera), C.byref(im(prx, 1)),
                                                  C.byref(im(jac, cs)), M, query.ctypes.data_as(FP),
                                                  train.ctypes.data_as(FP), 1.0, 1.0, rep_rows.ctypes.data_as(FP),
                                                  C.byref(tot)) == _lib.DFK_OK, lib.dfk_last_error(hd)
            assert lib.dfk_sparse_geometric_linearize(hd, p0, p1, c, c, cs, C.byref(camera), C.byref(im(prx, 1)),
                                                      C.byref(im(jac, cs)), C.byref(im(prx, 1)), C.byref(im(jac, cs)),
                                                      C.byref(im(grad, 2)), P,
                                                      points.ctypes.data_as(C.POINTER(C.c_int)), 0.1,
                                                      sg_rows.ctypes.data_as(FP), C.byref(nv)) == _lib.DFK_OK
        finally:
            assert lib.dfk_destroy(hd) == _lib.DFK_OK

    scratch = 4 * (4 * M + 2 * M * (13 + cs) + M)  # bytes of each of the two buffers after one cycle
    allowed = 96 << 20
    assert scratch >= 4 * allowed
    cycle()  # warm-up: module loading, first touch of the row buffers
    torch.cuda.synchronize()
    free0, rss0 = torch.cuda.mem_get_info()[0], _vmrss()
    for _ in range(3):
        cycle()
    torch.cuda.synchronize()
    dev_growth, rss_growth = free0 - torch.cuda.mem_get_info()[0], _vmrss() - rss0
    print(f"scratch per buffer and cycle {scratch / 2**20:.0f} MiB; after 3 cycles: device use grew "
          f"{dev_growth / 2**20:.0f} MiB, VmRSS grew {rss_growth / 2**20:.0f} MiB (allowed {allowed / 2**20:.0f} MiB)")
    assert dev_growth < allowed
    assert rss_growth < allowed
