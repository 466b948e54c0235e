"""ctypes binding of libdfk.so (the C ABI declared in include/dfk.h).

The library is built in-tree by `__graft_entry__.build()` / `make -C deepfactors_b200/csrc`.
There is NO fallback: if the shared library is missing or a call fails, this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# DFK_LIB: another build of the same library (A/B measurements of kernel variants); default = the in-tree build
LIB_PATH = os.environ.get("DFK_LIB") or os.path.join(_HERE, "libdfk.so")

DFK_OK = 0
DFK_ERR_INVALID_ARG = 1
DFK_ERR_CUDA = 2
DFK_ERR_UNSUPPORTED = 3
DFK_ERR_NOMEM = 4

DFK_GRAM_AUTO, DFK_GRAM_FP32, DFK_GRAM_TF32X3 = 0, 1, 2


class DfkError(RuntimeError):
    """std::runtime_error / vc::CUDAException stand-in carrying the status code."""

    def __init__(self, status: int, message: str):
        super().__init__(f"dfk status {status}: {message}")
        self.status = status
        self.message = message


class DfkImage(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("pitch_bytes", C.c_size_t), ("width", C.c_uint32), ("height", C.c_uint32)]


class DfkCamera(C.Structure):
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("u0", C.c_float), ("v0", C.c_float),
                ("width", C.c_float), ("height", C.c_float)]


class DfkDenseSfmParams(C.Structure):
    _fields_ = [("huber_delta", C.c_float), ("ocl_th", C.c_float), ("avg_dpt", C.c_float),
                ("min_dpt", C.c_float), ("valid_border", C.c_int32)]


class DfkSfmAlignerParams(C.Structure):
    _fields_ = [("sfmparams", DfkDenseSfmParams), ("step_threads", C.c_int32), ("step_blocks", C.c_int32),
                ("eval_threads", C.c_int32), ("eval_blocks", C.c_int32)]


class DfkSfmWorkItem(C.Structure):
    _fields_ = [("pose0", C.c_float * 7), ("pose1", C.c_float * 7), ("cam", DfkCamera),
                ("img0", DfkImage), ("img1", DfkImage), ("dpt0", DfkImage), ("valid0", DfkImage),
                ("prx0_jac", DfkImage), ("grad1", DfkImage),
                ("prx_orig", DfkImage), ("code", C.POINTER(C.c_float))]  # optional fused depth decode


class DfkTrackLevel(C.Structure):
    _fields_ = [("cam", DfkCamera), ("img0", DfkImage), ("img1", DfkImage), ("dpt0", DfkImage), ("grad1", DfkImage),
                ("iterations", C.c_int)]


class DfkReprojectionItem(C.Structure):
    _fields_ = [("pose0", C.c_float * 7), ("pose1", C.c_float * 7), ("cam", DfkCamera), ("prx_orig", DfkImage),
                ("prx_jac", DfkImage), ("code", C.POINTER(C.c_float)), ("num_matches", C.c_int32),
                ("query_xy", C.POINTER(C.c_float)), ("train_xy", C.POINTER(C.c_float)), ("cauchy_delta", C.c_float),
                ("sigma", C.c_float)]


class DfkSparseGeometricItem(C.Structure):
    _fields_ = [("pose0", C.c_float * 7), ("pose1", C.c_float * 7), ("cam", DfkCamera), ("prx0_orig", DfkImage),
                ("prx0_jac", DfkImage), ("prx1_orig", DfkImage), ("prx1_jac", DfkImage), ("dpt_grad1", DfkImage),
                ("code0", C.POINTER(C.c_float)), ("code1", C.POINTER(C.c_float)), ("num_points", C.c_int32),
                ("points_xy", C.POINTER(C.c_int32)), ("huber_delta", C.c_float)]


class DfkDepthDecodeItem(C.Structure):
    _fields_ = [("prx_orig", DfkImage), ("prx_jac", DfkImage), ("dpt", DfkImage), ("code", C.POINTER(C.c_float))]


class DfkDepthPriorItem(C.Structure):
    _fields_ = [("target_dpt", DfkImage), ("prx_orig", DfkImage), ("prx_jac", DfkImage), ("code", C.POINTER(C.c_float))]


class DfkWindowDesc(C.Structure):
    _fields_ = [("num_keyframes", C.c_int32), ("num_pairs", C.c_int32), ("num_items", C.c_int32), ("code_size", C.c_int32),
                ("pair_k0", C.POINTER(C.c_int32)), ("pair_k1", C.POINTER(C.c_int32)), ("item_pair", C.POINTER(C.c_int32)),
                ("item_width", C.POINTER(C.c_int32)), ("item_height", C.POINTER(C.c_int32))]


class DfkWindowSolveParams(C.Structure):
    _fields_ = [("lambda_", C.c_double), ("code_prior_weight", C.c_double)]


class DfkWindowUpdateParams(C.Structure):
    _fields_ = [("code_prior_weight", C.c_double), ("diag_eps", C.c_double)]


class DfkWindowItemSlots(C.Structure):
    _fields_ = [("pose0", C.c_int32), ("pose1", C.c_int32), ("code0", C.c_int32), ("code1", C.c_int32)]


class DfkWindowProblemDesc(C.Structure):
    _fields_ = [("window", C.c_void_p),
                ("num_dense", C.c_int32), ("dense", C.POINTER(DfkSfmWorkItem)),
                ("dense_slots", C.POINTER(DfkWindowItemSlots)),
                ("num_reproj", C.c_int32), ("reproj", C.POINTER(DfkReprojectionItem)),
                ("reproj_slots", C.POINTER(DfkWindowItemSlots)),
                ("num_geo", C.c_int32), ("geo", C.POINTER(DfkSparseGeometricItem)),
                ("geo_slots", C.POINTER(DfkWindowItemSlots)),
                ("num_depth", C.c_int32), ("depth", C.POINTER(DfkDepthDecodeItem)),
                ("depth_slots", C.POINTER(DfkWindowItemSlots)),
                ("num_error", C.c_int32), ("error", C.POINTER(DfkSfmWorkItem)),
                ("error_slots", C.POINTER(DfkWindowItemSlots)), ("error_depth", C.POINTER(C.c_int32)),
                ("num_frame_priors", C.c_int32), ("frame_prior_kf", C.POINTER(C.c_int32)),
                ("frame_prior_rows", C.POINTER(C.c_double)), ("frame_prior_x0", C.POINTER(C.c_double)),
                ("kf_prior_rows", C.POINTER(C.c_double)), ("kf_prior_x0", C.POINTER(C.c_double)),
                ("records_dev", C.c_void_p), ("geo_records_dev", C.c_void_p)]


class DfkLMParams(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("lambda_init", C.c_double), ("lambda_up", C.c_double),
                ("lambda_down", C.c_double), ("lambda_max", C.c_double), ("fix_first_pose", C.c_int32),
                ("code_prior_weight", C.c_double), ("use_error", C.c_int32)]


class DfkLMTrace(C.Structure):
    _fields_ = [("energy", C.POINTER(C.c_double)), ("lambda_", C.POINTER(C.c_double)),
                ("accepted", C.POINTER(C.c_int32)), ("num_energies", C.c_int32), ("num_steps", C.c_int32),
                ("linearisations", C.c_int32), ("error_evaluations", C.c_int32)]


class DfkLevelSchedule(C.Structure):
    _fields_ = [("num_levels", C.c_int32), ("iters", C.POINTER(C.c_int32)), ("dense_level", C.POINTER(C.c_int32)),
                ("error_pair", C.POINTER(C.c_int32)), ("error_level", C.POINTER(C.c_int32)), ("num_pairs", C.c_int32),
                ("pair_steps_done", C.POINTER(C.c_int32)), ("pair_remove_after", C.POINTER(C.c_uint8))]


class DfkLevelTrace(C.Structure):
    _fields_ = [("switch_energy", C.POINTER(C.c_double)), ("pair_levels", C.POINTER(C.c_int32)),
                ("pair_steps_done", C.POINTER(C.c_int32)), ("num_switches", C.c_int32)]


class DfkIsam2Params(C.Structure):
    _fields_ = [("relinearize_threshold", C.c_double), ("relinearize_skip", C.c_int32),
                ("code_prior_weight", C.c_double), ("fix_first_pose", C.c_int32)]


class DfkIsam2Result(C.Structure):
    _fields_ = [("variables_relinearized", C.c_int32), ("variables_reeliminated", C.c_int32),
                ("factors_relinearised", C.c_int32), ("first_column", C.c_int32)]


MAX_WORK_LEVELS = 8  # DFK_MAX_WORK_LEVELS


class DfkWorkState(C.Structure):
    _fields_ = [("active_level", C.c_int32), ("iters", C.c_int32 * MAX_WORK_LEVELS), ("first", C.c_int32),
                ("remove", C.c_int32), ("factor", C.c_int32), ("erased", C.c_int32)]


class DfkMapTrace(C.Structure):
    _fields_ = [("variables_relinearized", C.POINTER(C.c_int32)), ("variables_reeliminated", C.POINTER(C.c_int32)),
                ("factors_relinearised", C.POINTER(C.c_int32)), ("first_column", C.POINTER(C.c_int32)),
                ("pair_levels", C.POINTER(C.c_int32)), ("num_steps", C.c_int32)]


class DfkFeatureSet(C.Structure):
    _fields_ = [("keypoints", C.c_void_p), ("descriptors", C.c_void_p), ("num", C.c_int32),
                ("descriptor_bytes", C.c_int32)]


class DfkMatchItem(C.Structure):
    _fields_ = [("query", DfkFeatureSet), ("train", DfkFeatureSet), ("cam", DfkCamera), ("max_dist", C.c_float),
                ("max_iterations", C.c_int32), ("threshold", C.c_double), ("probability", C.c_double),
                ("seed", C.c_uint64)]


MATCH_MAX_QUERIES = 8192  # DFK_MATCH_MAX_QUERIES
MATCH_MAX_ITERATIONS = 1000000  # DFK_MATCH_MAX_ITERATIONS


class DfkOrbItem(C.Structure):
    _fields_ = [("image", DfkImage), ("nfeatures", C.c_int32), ("fast_threshold", C.c_int32),
                ("capacity", C.c_int32)]


ORB_MAX_SIDE = 16384  # DFK_ORB_MAX_SIDE
ORB_MAX_LEVELS = 16  # DFK_ORB_MAX_LEVELS


class DfkOrbPyramidItem(C.Structure):
    _fields_ = [("image", DfkImage), ("nfeatures", C.c_int32), ("scale_factor", C.c_float), ("nlevels", C.c_int32),
                ("fast_threshold", C.c_int32), ("capacity", C.c_int32)]
PREPROCESS_MAX_LEVELS = 15  # DFK_PREPROCESS_MAX_LEVELS


class DfkPreprocessItem(C.Structure):
    _fields_ = [("src", DfkImage), ("src_cam", DfkCamera), ("out_cam", DfkCamera), ("color", DfkImage),
                ("gray", DfkImage), ("levels", C.POINTER(DfkImage)), ("grads", C.POINTER(DfkImage)),
                ("normalize", C.c_int32)]


class DfkKeyframeMeshParams(C.Structure):
    _fields_ = [("stdev_thresh", C.c_float), ("slt_thresh", C.c_float), ("crop_pix", C.c_int32),
                ("draw_noisy_pixels", C.c_int32)]


class DfkKeyframeMeshItem(C.Structure):
    _fields_ = [("dpt", DfkImage), ("prx_orig", DfkImage), ("prx_jac", DfkImage), ("code", C.POINTER(C.c_float)),
                ("std", DfkImage), ("valid", DfkImage), ("color", DfkImage), ("cam", DfkCamera),
                ("pose_wk", C.c_float * 7), ("vertex_capacity", C.c_int32), ("triangle_capacity", C.c_int32),
                ("depth_u16", DfkImage)]


BOW_MAX_DEPTH = 16  # DFK_BOW_MAX_DEPTH
BOW_MAX_NODES = 4194304  # DFK_BOW_MAX_NODES


class DfkBowVocabularyDesc(C.Structure):
    _fields_ = [("k", C.c_int32), ("L", C.c_int32), ("weighting", C.c_int32), ("scoring", C.c_int32),
                ("descriptor_bytes", C.c_int32), ("num_nodes", C.c_int32), ("node_ids", C.c_void_p),
                ("parent_ids", C.c_void_p), ("weights", C.c_void_p), ("descriptors", C.c_void_p),
                ("num_words", C.c_int32), ("word_ids", C.c_void_p), ("word_nodes", C.c_void_p)]


class DfkBowVector(C.Structure):
    _fields_ = [("words", C.c_void_p), ("values", C.c_void_p), ("count", C.c_void_p), ("capacity", C.c_int32)]


class DfkBowQuery(C.Structure):
    _fields_ = [("vector", DfkBowVector), ("max_results", C.c_int32), ("max_id", C.c_int32)]


class DfkBowScoreItem(C.Structure):
    _fields_ = [("entry", C.c_int32), ("vector", DfkBowVector)]


BOW_TRAIN_MAX_ROUNDS = 1000  # DFK_BOW_TRAIN_MAX_ROUNDS
BOW_TRAIN_MAX_DESCRIPTORS = 268435456  # DFK_BOW_TRAIN_MAX_DESCRIPTORS


class DfkBowTrainDesc(C.Structure):
    _fields_ = [("k", C.c_int32), ("L", C.c_int32), ("descriptor_bytes", C.c_int32), ("num_images", C.c_int32),
                ("seed", C.c_uint64), ("num_descriptors", C.c_int64), ("descriptors_dev", C.c_void_p),
                ("image_offsets", C.c_void_p)]


class DfkBowTrainStats(C.Structure):
    _fields_ = [("num_nodes", C.c_int32), ("num_words", C.c_int32), ("max_rounds", C.c_int32),
                ("capped_nodes", C.c_int32), ("empty_clusters", C.c_int32),
                ("level_max_rounds", C.c_int32 * BOW_MAX_DEPTH)]


class DfkBowVocabularyShape(C.Structure):
    _fields_ = [("k", C.c_int32), ("L", C.c_int32), ("weighting", C.c_int32), ("scoring", C.c_int32),
                ("descriptor_bytes", C.c_int32), ("num_nodes", C.c_int32), ("num_words", C.c_int32)]


WINDOW_ERROR_DOUBLES = 7  # DFK_WINDOW_ERROR_DOUBLES
WINDOW_ERROR_EX_DOUBLES = 8  # DFK_WINDOW_ERROR_EX_DOUBLES


# every symbol include/dfk.h declares: (name, restype, argtypes)
_F = C.POINTER(C.c_float)
_IMG = C.POINTER(DfkImage)
_CAM = C.POINTER(DfkCamera)
_H = C.c_void_p
SYMBOLS = {
    "dfk_create": (C.c_int, [C.c_int, C.POINTER(_H)]),
    "dfk_destroy": (C.c_int, [_H]),
    "dfk_set_stream": (C.c_int, [_H, C.c_void_p]),
    "dfk_set_sm_limit": (C.c_int, [_H, C.c_int]),
    "dfk_use_own_stream": (C.c_int, [_H]),
    "dfk_get_stream": (C.c_void_p, [_H]),
    "dfk_synchronize": (C.c_int, [_H]),
    "dfk_last_error": (C.c_char_p, [_H]),
    "dfk_status_string": (C.c_char_p, [C.c_int]),
    "dfk_version": (C.c_int, []),
    "dfk_sfm_supports_code_size": (C.c_int, [C.c_int]),
    "dfk_set_profiling": (C.c_int, [_H, C.c_int]),
    "dfk_get_profile": (C.c_int, [_H, C.POINTER(C.c_double), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "dfk_sfm_set_params": (C.c_int, [_H, C.POINTER(DfkSfmAlignerParams)]),
    "dfk_sfm_get_params": (C.c_int, [_H, C.POINTER(DfkSfmAlignerParams)]),
    "dfk_sfm_set_gram_mode": (C.c_int, [_H, C.c_int]),
    "dfk_se3_set_huber_delta": (C.c_int, [_H, C.c_float]),
    "dfk_sfm_run_step": (C.c_int, [_H, _F, _F, _F, C.c_int, _CAM, _IMG, _IMG, _IMG, _IMG, _IMG, _IMG, _IMG,
                                   _F, _F, _F, C.POINTER(C.c_uint64)]),
    "dfk_sfm_evaluate_error": (C.c_int, [_H, _F, _F, _CAM, _IMG, _IMG, _IMG, _IMG, _IMG, _F,
                                         C.POINTER(C.c_uint64)]),
    "dfk_sfm_evaluate_error_batch": (C.c_int, [_H, C.POINTER(DfkSfmWorkItem), C.c_int, C.c_void_p]),
    "dfk_sfm_run_step_batch": (C.c_int, [_H, C.POINTER(DfkSfmWorkItem), C.c_int, C.c_int, C.c_void_p]),
    "dfk_sfm_run_step_batch_host": (C.c_int, [_H, C.POINTER(DfkSfmWorkItem), C.c_int, C.c_int, _F]),
    "dfk_sfm_stream_create": (C.c_int, [_H, C.c_int, C.c_int, C.c_size_t, C.c_int, C.POINTER(C.c_void_p)]),
    "dfk_sfm_stream_destroy": (C.c_int, [_H, C.c_void_p]),
    "dfk_sfm_stream_submit": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkSfmWorkItem), C.c_int, C.POINTER(C.c_uint64)]),
    "dfk_sfm_stream_wait": (C.c_int, [_H, C.c_void_p, C.c_uint64, _F]),
    "dfk_window_create": (C.c_int, [_H, C.POINTER(DfkWindowDesc), C.POINTER(C.c_void_p)]),
    "dfk_window_destroy": (C.c_int, [_H, C.c_void_p]),
    "dfk_window_floats": (C.c_size_t, [C.c_void_p]),
    "dfk_window_assemble": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_create_geometric": (C.c_int, [_H, C.POINTER(DfkWindowDesc), C.c_int, C.POINTER(C.c_int32),
                                              C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]),
    "dfk_window_assemble_geometric": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_create_frames": (C.c_int, [_H, C.POINTER(DfkWindowDesc), C.c_int, C.POINTER(C.c_int32),
                                           C.POINTER(C.c_int32), C.c_int, C.POINTER(C.c_void_p)]),
    "dfk_window_marginalize_frames": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_void_p,
                                                C.c_void_p]),
    "dfk_window_add_priors": (C.c_int, [_H, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "dfk_window_create_priors": (C.c_int, [_H, C.POINTER(DfkWindowDesc), C.c_int, C.POINTER(C.c_int32),
                                           C.POINTER(C.c_int32), C.c_int, C.c_int, C.POINTER(C.c_int32),
                                           C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]),
    "dfk_window_add_keyframe_priors": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_blanket": (C.c_int, [_H, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "dfk_window_marginalize_keyframe": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_double,
                                                  C.POINTER(C.c_double), C.c_void_p, C.c_void_p]),
    "dfk_window_solver_create": (C.c_int, [_H, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_void_p)]),
    "dfk_window_solver_destroy": (C.c_int, [_H, C.c_void_p]),
    "dfk_window_solver_tiles": (C.c_int, [_H, C.c_void_p, C.POINTER(C.c_size_t)]),
    "dfk_window_solve": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.POINTER(DfkWindowSolveParams), C.POINTER(C.c_double),
                                   C.c_void_p, C.c_void_p]),
    "dfk_window_solver_update": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.POINTER(DfkWindowUpdateParams),
                                           C.POINTER(C.c_double), C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]),
    "dfk_window_solver_create_from": (C.c_int, [_H, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.c_void_p,
                                                C.POINTER(C.c_void_p)]),
    "dfk_window_problem_create": (C.c_int, [_H, C.POINTER(DfkWindowProblemDesc), C.POINTER(C.c_void_p)]),
    "dfk_window_problem_destroy": (C.c_int, [_H, C.c_void_p]),
    "dfk_window_problem_set_state": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_get_state": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_linearize": (C.c_int, [_H, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_error": (C.c_int, [_H, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_retract": (C.c_int, [_H, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_error_ex": (C.c_int, [_H, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_set_depth_priors": (C.c_int, [_H, C.c_void_p, C.c_int, C.POINTER(C.c_int32),
                                                      C.POINTER(C.c_float), C.POINTER(C.c_int32),
                                                      C.POINTER(DfkDepthPriorItem)]),
    "dfk_window_lm": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkLMParams), C.POINTER(DfkLMTrace)]),
    "dfk_window_problem_set_active": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_lm_levels": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkLMParams), C.POINTER(DfkLevelSchedule),
                                       C.POINTER(DfkLMTrace), C.POINTER(DfkLevelTrace)]),
    "dfk_window_problem_isam2_update": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkIsam2Params),
                                                  C.POINTER(DfkIsam2Result)]),
    "dfk_window_problem_get_linearization": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_window_problem_grow_from": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32),
                                               C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "dfk_window_map_steps": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkIsam2Params), C.POINTER(DfkLevelSchedule),
                                       C.POINTER(DfkWorkState), C.c_int, C.POINTER(DfkMapTrace)]),
    "dfk_se3_run_step": (C.c_int, [_H, _F, _CAM, _IMG, _IMG, _IMG, _IMG, _F, _F, _F, C.POINTER(C.c_uint64)]),
    "dfk_se3_track": (C.c_int, [_H, _F, C.POINTER(DfkTrackLevel), C.c_int, _F, _F, _F, _F, C.c_int]),
    "dfk_se3_track_batch": (C.c_int, [_H, C.c_int, C.c_int, _F, C.POINTER(DfkTrackLevel), _F, _F, _F]),
    "dfk_se3_warp": (C.c_int, [_H, _F, _CAM, _IMG, _IMG, _IMG, _IMG, _F, C.POINTER(C.c_uint64)]),
    "dfk_depth_run_step": (C.c_int, [_H, _F, C.c_int, _IMG, _IMG, _IMG, _F, _F, _F, C.POINTER(C.c_uint64)]),
    "dfk_depth_prior_linearize_batch": (C.c_int, [_H, C.POINTER(DfkDepthPriorItem), C.c_int, C.c_int, C.c_void_p]),
    "dfk_depth_prior_error_batch": (C.c_int, [_H, C.POINTER(DfkDepthPriorItem), C.c_int, C.c_int, C.c_void_p]),
    "dfk_window_add_depth_priors": (C.c_int, [_H, C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_float),
                                              C.POINTER(C.c_int32), C.c_void_p, C.c_void_p]),
    "dfk_reprojection_linearize": (C.c_int, [_H, _F, _F, _F, C.c_int, _CAM, _IMG, _IMG, C.c_int, _F, _F, C.c_float,
                                             C.c_float, _F, _F]),
    "dfk_reprojection_linearize_batch": (C.c_int, [_H, C.POINTER(DfkReprojectionItem), C.c_int, C.c_int, C.c_void_p]),
    "dfk_sparse_geometric_linearize": (C.c_int, [_H, _F, _F, _F, _F, C.c_int, _CAM, _IMG, _IMG, _IMG, _IMG, _IMG, C.c_int,
                                                 C.POINTER(C.c_int), C.c_float, _F, C.POINTER(C.c_int)]),
    "dfk_sparse_geometric_linearize_batch": (C.c_int, [_H, C.POINTER(DfkSparseGeometricItem), C.c_int, C.c_int,
                                                       C.c_void_p]),
    "dfk_reprojection_error_batch": (C.c_int, [_H, C.POINTER(DfkReprojectionItem), C.c_int, C.c_int, C.c_void_p]),
    "dfk_sparse_geometric_error_batch": (C.c_int, [_H, C.POINTER(DfkSparseGeometricItem), C.c_int, C.c_int,
                                                   C.c_void_p]),
    "dfk_hamming_match_batch": (C.c_int, [_H, C.POINTER(DfkMatchItem), C.c_int, C.c_void_p]),
    "dfk_reprojection_match_batch": (C.c_int, [_H, C.POINTER(DfkMatchItem), C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p]),
    "dfk_orb_detect_batch": (C.c_int, [_H, C.POINTER(DfkOrbItem), C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                       C.c_void_p, C.c_void_p]),
    "dfk_orb_detect_pyramid_batch": (C.c_int, [_H, C.POINTER(DfkOrbPyramidItem), C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_update_depth": (C.c_int, [_H, _F, C.c_int, _IMG, _IMG, C.c_float, _IMG]),
    "dfk_update_depth_batch": (C.c_int, [_H, C.POINTER(DfkDepthDecodeItem), C.c_int, C.c_int]),
    "dfk_sobel_gradients": (C.c_int, [_H, _IMG, _IMG]),
    "dfk_gaussian_blur_down": (C.c_int, [_H, _IMG, _IMG]),
    "dfk_build_image_pyramid": (C.c_int, [_H, _IMG, _IMG, C.c_int]),
    "dfk_squared_error": (C.c_int, [_H, _IMG, _IMG, _F]),
    "dfk_preprocess_batch": (C.c_int, [_H, C.POINTER(DfkPreprocessItem), C.c_int, C.c_int, C.c_void_p]),
    "dfk_keyframe_mesh_batch": (C.c_int, [_H, C.POINTER(DfkKeyframeMeshItem), C.c_int, C.c_int,
                                          C.POINTER(DfkKeyframeMeshParams), C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_bow_vocabulary_create": (C.c_int, [_H, C.POINTER(DfkBowVocabularyDesc), C.POINTER(C.c_void_p)]),
    "dfk_bow_vocabulary_destroy": (C.c_int, [_H, C.c_void_p]),
    "dfk_bow_transform_batch": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkFeatureSet), C.POINTER(C.c_int32), C.c_int,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "dfk_bow_database_create": (C.c_int, [_H, C.c_void_p, C.POINTER(C.c_void_p)]),
    "dfk_bow_database_destroy": (C.c_int, [_H, C.c_void_p]),
    "dfk_bow_database_clear": (C.c_int, [_H, C.c_void_p]),
    "dfk_bow_database_size": (C.c_int, [_H, C.c_void_p, C.POINTER(C.c_int32)]),
    "dfk_bow_database_add": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkBowVector), C.c_int, C.POINTER(C.c_int32)]),
    "dfk_bow_database_query_batch": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkBowQuery), C.c_int, C.c_void_p, C.c_void_p,
                                               C.c_void_p]),
    "dfk_bow_score_batch": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkBowScoreItem), C.c_int, C.c_void_p]),
    "dfk_bow_vocabulary_train": (C.c_int, [_H, C.POINTER(DfkBowTrainDesc), C.POINTER(DfkBowTrainStats),
                                           C.POINTER(C.c_void_p)]),
    "dfk_bow_vocabulary_export": (C.c_int, [_H, C.c_void_p, C.POINTER(DfkBowVocabularyShape), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}

_lib = None


def lib():
    """Load libdfk.so; raises if it has not been built (no CPU fallback exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; "
                "g.build()' or make -C deepfactors_b200/csrc). deepfactors_b200 has no CPU fallback.")
        handle = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(handle, name)  # AttributeError if the library does not export it
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(handle, status: int):
    if status != DFK_OK:
        msg = lib().dfk_last_error(handle)
        raise DfkError(status, (msg or b"").decode() or lib().dfk_status_string(status).decode())


def record_floats(code_size: int) -> int:
    npar = 12 + code_size
    return npar * (npar + 1) // 2 + npar + 2


def geo_record_floats(code_size: int) -> int:
    """DFK_GEO_RECORD_FLOATS: a sparse geometric record over [pose0 | pose1 | code0 | code1]"""
    npar = 12 + 2 * code_size
    return npar * (npar + 1) // 2 + npar + 2


def depth_record_floats(code_size: int) -> int:
    """DFK_DEPTH_RECORD_FLOATS: a depth-prior record [JtJ packed upper | Jtr | residual | inliers]"""
    return code_size * (code_size + 1) // 2 + code_size + 2


def prior_doubles(code_size: int) -> int:
    """DFK_PRIOR_DOUBLES: a linear keyframe prior [G (B x B) | g (B) | f0], B = 6 + code_size"""
    b = 6 + code_size
    return b * b + b + 1


def kf_prior_doubles(code_size: int, n: int) -> int:
    """DFK_KF_PRIOR_DOUBLES: a keyframe prior over n keyframes [G (nB x nB) | g (nB) | f0], B = 6 + code_size"""
    nb = n * (6 + code_size)
    return nb * nb + nb + 1


MAX_BLANKET = 16  # DFK_MAX_BLANKET
