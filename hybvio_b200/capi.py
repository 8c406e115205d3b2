"""ctypes binding of libhybvio_b200.so (include/hybvio_b200.h).

Harness-side plumbing only: tests/ and bench.py drive the C ABI through this module exactly the way the
reference-side C++ adapters (hybvio_b200/host/) do. There is no CPU fallback: a missing library or a missing
GPU raises.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# HV_LIB_PATH: tools/ only (e.g. the -DHV_EKF_TIMING build used by tools/ekf_phases.py)
LIB_PATH = os.environ.get("HV_LIB_PATH") or os.path.join(_HERE, "libhybvio_b200.so")

c_int, c_double, c_void_p, c_size_t = ctypes.c_int, ctypes.c_double, ctypes.c_void_p, ctypes.c_size_t


class HvError(RuntimeError):
    pass


class EkfParams(ctypes.Structure):
    _fields_ = [
        ("camera_trail_length", c_int), ("hybrid_map_size", c_int),
        ("noise_scale", c_double), ("gravity", c_double),
        ("noise_initial_pos", c_double), ("noise_initial_vel", c_double), ("noise_initial_ori", c_double),
        ("noise_initial_bga", c_double), ("noise_initial_baa", c_double), ("noise_initial_bat", c_double),
        ("noise_initial_sft", c_double),
        ("noise_initial_pos_trail", c_double), ("noise_initial_ori_trail", c_double),
        ("noise_process_acc", c_double), ("noise_process_gyro", c_double),
        ("noise_process_baa", c_double), ("noise_process_baa_rev", c_double),
        ("noise_process_bga", c_double), ("noise_process_bga_rev", c_double),
        ("augment_r", c_double), ("init_zupt_r", c_double), ("rotation_zupt_r", c_double),
    ]


class CameraModel(ctypes.Structure):
    """hv_camera_model (include/hybvio_b200.h)"""
    _fields_ = [("imu_to_camera", c_double * 16), ("second_imu_to_camera", c_double * 16), ("use_stereo", c_int),
                ("estimate_imu_camera_time_shift", c_int), ("gauss_newton_iterations", ctypes.c_uint),
                ("convergence_threshold", c_double), ("convergence_r", c_double), ("rcond_threshold", c_double),
                ("min_dist", c_double), ("max_dist", c_double)]


class TrackObs(ctypes.Structure):
    _fields_ = [("npose", c_int), ("pose_trail_index", c_void_p), ("ip", c_void_p), ("velocities", c_void_p)]


class TrackModel(ctypes.Structure):
    _fields_ = [("triangulator_status", c_int), ("prepare_vu_status", c_int), ("rows", c_int), ("cols", c_int),
                ("pf", c_double * 3), ("depth", c_double), ("d_H", c_void_p), ("d_f", c_void_p), ("d_y", c_void_p)]


class VisualUpdateParams(ctypes.Structure):
    _fields_ = [("chi_outlier_r", c_double), ("track_rmse_threshold", c_double), ("visual_r", c_double),
                ("max_successful_updates", c_int), ("lookahead", c_int)]


class TrackResult(ctypes.Structure):
    _fields_ = [("triangulator_status", c_int), ("prepare_vu_status", c_int), ("outlier_status", c_int), ("updated", c_int),
                ("chi2", c_double), ("pf", c_double * 3), ("depth", c_double)]


class EkfOp(ctypes.Structure):
    _fields_ = [("kind", c_int), ("n", c_int), ("l", c_int), ("mode", c_int), ("index", c_int),
                ("t", c_double), ("r", c_double), ("rmse_thr", c_double), ("gyro", c_double * 3), ("acc", c_double * 3),
                ("H", c_void_p), ("f", c_void_p), ("y", c_void_p)]


OP_PREDICT, OP_VISUAL, OP_SYMMETRIZE, OP_AUGMENT, OP_UNAUGMENT, OP_NORMALIZE = range(6)


class LkJob(ctypes.Structure):
    _fields_ = [("prev", c_void_p), ("next", c_void_p), ("d_prev_xy", c_void_p), ("d_next_xy", c_void_p),
                ("d_status", c_void_p), ("d_track_status", c_void_p), ("n", c_int), ("use_initial", c_int)]


class CornerJob(ctypes.Structure):
    """hv_corner_job: one session's list in the batched detect / select calls"""
    _fields_ = [("pyr", c_void_p), ("d_kp", c_void_p), ("nkp", c_int), ("d_prev_xy", c_void_p), ("nprev", c_int),
                ("mask_radius", c_int), ("max_tracks", c_int), ("d_corners", c_void_p), ("capacity", c_int), ("d_count", c_void_p)]


class SubpixJob(ctypes.Structure):
    """hv_subpix_job: one session's points in the batched sub-pixel refinement"""
    _fields_ = [("pyr", c_void_p), ("d_xy", c_void_p), ("n", c_int)]


class FastJob(ctypes.Structure):
    """hv_fast_job: one session's pyramid and outputs in the batched FAST detection (see fast_job)"""
    _fields_ = [("pyr", c_void_p), ("d_xy", c_void_p), ("d_response", c_void_p), ("capacity", c_int), ("d_count", c_void_p)]


class GoodFeaturesJob(ctypes.Structure):
    """hv_good_features_job: one session's pyramid, corner budget, mask and outputs in the batched Shi-Tomasi detection (see
    good_features_job)"""
    _fields_ = [("pyr", c_void_p), ("max_corners", c_int), ("d_mask", c_void_p), ("mask_stride", c_size_t), ("d_xy", c_void_p),
                ("d_response", c_void_p), ("capacity", c_int), ("d_count", c_void_p)]


CORNER_BATCH_MAX = 64   # HV_CORNER_BATCH_MAX


class EssentialJob(ctypes.Structure):
    """hv_essential_job: one session's correspondences, intrinsics and outputs in the batched essential-matrix RANSAC (see
    essential_job)"""
    _fields_ = [("d_xy1", c_void_p), ("d_xy2", c_void_p), ("d_status", c_void_p), ("n", c_int),
                ("fx", c_double), ("fy", c_double), ("cx", c_double), ("cy", c_double),
                ("d_E", c_void_p), ("d_nsol", c_void_p), ("d_mask", c_void_p), ("d_inliers", c_void_p)]


ESSENTIAL_BATCH_MAX = 64       # HV_ESSENTIAL_BATCH_MAX
ESSENTIAL_MAX_POINTS = 4096    # HV_ESSENTIAL_MAX_POINTS
ESSENTIAL_MAX_ITERS = 4096     # HV_ESSENTIAL_MAX_ITERS


class PoseJob(ctypes.Structure):
    """hv_pose_job: one session's essential matrix, correspondences, intrinsics and outputs in the batched relative pose (see
    pose_job)"""
    _fields_ = [("d_E", c_void_p), ("d_nsol", c_void_p), ("d_xy1", c_void_p), ("d_xy2", c_void_p), ("d_mask_in", c_void_p), ("n", c_int),
                ("fx", c_double), ("fy", c_double), ("cx", c_double), ("cy", c_double),
                ("d_R", c_void_p), ("d_t", c_void_p), ("d_mask_out", c_void_p), ("d_good", c_void_p)]


class IngestJob(ctypes.Structure):
    """hv_ingest_job: one frame of hv_ingest_frames (see ingest_job)"""
    _fields_ = [("ing", c_void_p), ("src", c_void_p), ("stride_bytes", c_size_t), ("channels", c_int), ("coeff", c_void_p),
                ("dst", c_void_p), ("gray_out", c_void_p)]


INGEST_BATCH_MAX = 128  # HV_INGEST_BATCH_MAX

_lib = None


def load():
    """Loads the CUDA library; fails loudly when it has not been built (python -c 'import __graft_entry__ as g; g.build()')."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `make` (nvcc, sm_90a). hybvio_b200 has no CPU fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    lib.hv_version.restype = ctypes.c_char_p
    lib.hv_last_error.restype = ctypes.c_char_p
    lib.hv_ctx_stream.restype = c_void_p
    lib.hv_ctx_stream.argtypes = [c_void_p]
    lib.hv_ctx_launch_count.restype = ctypes.c_longlong
    lib.hv_ctx_launch_count.argtypes = [c_void_p]
    lib.hv_ctx_create.argtypes = [c_int, ctypes.POINTER(c_void_p)]
    lib.hv_ctx_create_on_stream.argtypes = [c_int, c_void_p, ctypes.POINTER(c_void_p)]
    lib.hv_ctx_destroy.argtypes = [c_void_p]
    lib.hv_ctx_sync.argtypes = [c_void_p]
    lib.hv_pyr_create.argtypes = [c_void_p, c_int, c_int, c_int, c_int, ctypes.POINTER(c_void_p)]
    lib.hv_pyr_release.argtypes = [c_void_p]
    lib.hv_pyr_levels.argtypes = [c_void_p]
    lib.hv_pyr_level_size.argtypes = [c_void_p, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]
    lib.hv_pyr_build.argtypes = [c_void_p, c_void_p, c_size_t]
    lib.hv_pyr_build_batch.argtypes = [ctypes.POINTER(c_void_p), ctypes.POINTER(c_void_p), ctypes.POINTER(c_size_t), c_int, c_int]
    lib.hv_pyr_download_level.argtypes = [c_void_p, c_int, c_void_p, c_void_p]
    lib.hv_pyr_download_level_padded.argtypes = [c_void_p, c_int, c_void_p, c_void_p]
    lib.hv_lk_track.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_double, c_double]
    lib.hv_lk_track_device.argtypes = lib.hv_lk_track.argtypes
    lib.hv_lk_track_device_on_stream.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_double, c_double]
    lib.hv_lk_track_batch_device.argtypes = [c_void_p, ctypes.POINTER(LkJob), c_int, c_int, c_double, c_double]
    lib.hv_ingest_create.argtypes = [c_void_p, c_int, c_int, ctypes.POINTER(c_void_p)]
    lib.hv_ingest_destroy.argtypes = [c_void_p]
    lib.hv_ingest_set_remap.argtypes = [c_void_p, c_void_p]
    lib.hv_ingest_frame.argtypes = [c_void_p, c_void_p, c_size_t, c_int, c_void_p, c_void_p, c_void_p]
    lib.hv_ingest_frames.argtypes = [ctypes.POINTER(IngestJob), c_int, c_int]
    lib.hv_gftt_cells.argtypes = [c_void_p, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]
    lib.hv_gftt_detect.argtypes = [c_void_p, c_void_p, c_int, c_int, ctypes.c_float, c_void_p]
    lib.hv_gftt_detect_device.argtypes = [c_void_p, c_void_p, c_int, c_int, ctypes.c_float, c_void_p]
    lib.hv_gftt_select_device.argtypes = [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]
    lib.hv_gftt_corners.argtypes = [c_void_p, c_void_p, c_int, c_int, ctypes.c_float, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]
    lib.hv_subpix_refine.argtypes = [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_double]
    lib.hv_subpix_refine_device.argtypes = lib.hv_subpix_refine.argtypes
    lib.hv_gftt_detect_batch_device.argtypes = [c_void_p, ctypes.POINTER(CornerJob), c_int, c_int, c_int, ctypes.c_float]
    lib.hv_gftt_select_batch_device.argtypes = [c_void_p, ctypes.POINTER(CornerJob), c_int]
    lib.hv_subpix_refine_batch_device.argtypes = [c_void_p, ctypes.POINTER(SubpixJob), c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_double]
    lib.hv_fast_detect.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p]
    lib.hv_fast_detect_device.argtypes = lib.hv_fast_detect.argtypes
    lib.hv_fast_detect_batch_device.argtypes = [c_void_p, ctypes.POINTER(FastJob), c_int, c_int, c_int]
    lib.hv_good_features.argtypes = [c_void_p, c_void_p, c_int, c_int, c_double, c_double, c_void_p, c_size_t, c_void_p, c_void_p, c_int, c_void_p]
    lib.hv_good_features_device.argtypes = lib.hv_good_features.argtypes
    lib.hv_good_features_batch_device.argtypes = [c_void_p, ctypes.POINTER(GoodFeaturesJob), c_int, c_int, c_double, c_double]
    lib.hv_find_essential.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_double, c_double,
                                      c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.hv_find_essential_device.argtypes = lib.hv_find_essential.argtypes
    lib.hv_find_essential_batch_device.argtypes = [c_void_p, ctypes.POINTER(EssentialJob), c_int, c_double, c_double, c_int]
    lib.hv_recover_pose.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_double,
                                    c_double, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.hv_recover_pose_device.argtypes = [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_double, c_double,
                                           c_double, c_double, c_double, c_void_p, c_void_p, c_void_p, c_void_p]
    lib.hv_recover_pose_batch_device.argtypes = [c_void_p, ctypes.POINTER(PoseJob), c_int, c_double]
    _bind_ekf(lib)
    _lib = lib
    return lib


def _bind_ekf(lib):
    if not hasattr(lib, "hv_ekf_create"):
        return
    dp = ctypes.POINTER(c_double)
    lib.hv_ekf_default_params.argtypes = [ctypes.POINTER(EkfParams)]
    lib.hv_ekf_default_params.restype = None
    lib.hv_ekf_create.argtypes = [c_void_p, ctypes.POINTER(EkfParams), ctypes.POINTER(c_void_p)]
    lib.hv_ekf_destroy.argtypes = [c_void_p]
    lib.hv_ekf_clone.argtypes = [c_void_p, ctypes.POINTER(c_void_p)]
    for name in ("hv_ekf_state_dim", "hv_ekf_pose_count", "hv_ekf_was_stationary", "hv_ekf_unaugment", "hv_ekf_symmetrize",
                 "hv_ekf_condition_on_last_pose", "hv_ekf_lock_biases", "hv_ekf_update_zupt_initialization", "hv_ekf_flush"):
        getattr(lib, name).argtypes = [c_void_p]
    lib.hv_ekf_platform_time.argtypes = [c_void_p]
    lib.hv_ekf_platform_time.restype = c_double
    lib.hv_ekf_history_time.argtypes = [c_void_p, c_int]
    lib.hv_ekf_history_time.restype = c_double
    lib.hv_ekf_set_first_sample_time.argtypes = [c_void_p, c_double]
    lib.hv_ekf_upload.argtypes = [c_void_p, c_void_p, c_void_p]
    lib.hv_ekf_download.argtypes = [c_void_p, c_void_p, c_void_p]
    lib.hv_ekf_download_inertial.argtypes = [c_void_p, c_void_p, c_void_p]
    lib.hv_ekf_set_inertial_state.argtypes = [c_void_p, c_void_p, c_void_p]
    lib.hv_ekf_set_process_noise.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_get_dydx.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_initialize_orientation.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_predict.argtypes = [c_void_p, c_double, c_void_p, c_void_p]
    lib.hv_ekf_update_zupt.argtypes = [c_void_p, c_double]
    lib.hv_ekf_update_zrupt.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_update_pseudo_velocity.argtypes = [c_void_p, c_double, c_double]
    lib.hv_ekf_update_position.argtypes = [c_void_p, c_void_p, c_double]
    lib.hv_ekf_update_zero_height.argtypes = [c_void_p, c_double]
    lib.hv_ekf_update_orientation.argtypes = [c_void_p, c_void_p, c_double]
    lib.hv_ekf_visual_check.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_double, c_double,
                                        ctypes.POINTER(c_int), dp]
    lib.hv_ekf_visual_update.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_double]
    lib.hv_ekf_visual_check_update.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_double, c_double,
                                               ctypes.POINTER(c_int), dp, c_void_p]
    lib.hv_camera_model_defaults.argtypes = [ctypes.POINTER(CameraModel)]
    lib.hv_camera_model_defaults.restype = None
    lib.hv_ekf_set_camera_model.argtypes = [c_void_p, ctypes.POINTER(CameraModel)]
    lib.hv_ekf_track_models.argtypes = [c_void_p, ctypes.POINTER(TrackObs), c_int, ctypes.POINTER(TrackModel)]
    lib.hv_ekf_track_model_download.argtypes = [c_void_p, c_int, c_void_p, c_void_p, c_void_p]
    lib.hv_ekf_visual_tracks.argtypes = [c_void_p, ctypes.POINTER(TrackObs), c_int, ctypes.POINTER(VisualUpdateParams), ctypes.POINTER(TrackResult),
                                         ctypes.POINTER(c_int)]
    lib.hv_ekf_track_models_time.argtypes = [c_void_p, c_int, ctypes.POINTER(ctypes.c_float)]
    lib.hv_ekf_debug_result_words.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_debug_host_times.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_visual_track.argtypes = [c_void_p, ctypes.POINTER(TrackModel), c_double, c_double, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_double)]
    lib.hv_ekf_visual_device.argtypes = [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_double, c_double, c_int, c_void_p]
    lib.hv_ekf_augment.argtypes = [c_void_p, c_int]
    lib.hv_ekf_set_imu_batching.argtypes = [c_void_p, c_int]
    lib.hv_ekf_run_device.argtypes = [c_void_p, ctypes.POINTER(EkfOp), c_int]
    lib.hv_ekf_predicted_mean_device.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_predicted_mean.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_run_device_results.argtypes = [c_void_p, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_double)]
    lib.hv_ekf_run_host.argtypes = [c_void_p, ctypes.POINTER(EkfOp), c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_double), c_void_p]
    lib.hv_ekf_group_run_device.argtypes = [ctypes.POINTER(c_void_p), c_int, ctypes.POINTER(ctypes.POINTER(EkfOp)), ctypes.POINTER(c_int)]
    lib.hv_ekf_group_visual_tracks.argtypes = [ctypes.POINTER(c_void_p), c_int, ctypes.POINTER(ctypes.POINTER(TrackObs)), ctypes.POINTER(c_int),
                                               ctypes.POINTER(VisualUpdateParams), ctypes.POINTER(ctypes.POINTER(TrackResult)), ctypes.POINTER(c_int)]
    lib.hv_ekf_group_visual_tracks.restype = c_int
    lib.hv_ekf_normalize_quaternions.argtypes = [c_void_p, c_int]
    lib.hv_ekf_translate_to.argtypes = [c_void_p, c_void_p]
    lib.hv_ekf_transform_to.argtypes = [c_void_p, c_void_p, c_void_p, c_int]
    lib.hv_ekf_insert_map_point.argtypes = [c_void_p, c_int, c_void_p]


def check(rc, what=""):
    if rc != 0:
        raise HvError(f"{what} failed with hv_status {rc}: {load().hv_last_error().decode()}")


def _ptr(a):
    """Address of a numpy array / torch tensor / raw int."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    return a.data_ptr()   # torch tensor


GROUP_MAX = 64      # HV_EKF_GROUP_MAX


def ekf_group_run_device(ekfs, lists):
    """hv_ekf_group_run_device: steps several filters of one context with the launches of one. lists[i] is filter i's op list, as for
    Ekf.run_device: an (EkfOp array, nops) pair or an EkfOp array (all of it). Asynchronous; raises HvError on a refusal (the filters
    are then untouched and the caller steps them one by one)."""
    n = len(ekfs)
    pairs = [x if isinstance(x, tuple) else (x, len(x)) for x in lists]
    E = (c_void_p * n)(*[e.h for e in ekfs])
    O = (ctypes.POINTER(EkfOp) * n)(*[ctypes.cast(ops, ctypes.POINTER(EkfOp)) for ops, _ in pairs])
    K = (c_int * n)(*[k for _, k in pairs])
    check(load().hv_ekf_group_run_device(E, n, O, K), "hv_ekf_group_run_device")


def ekf_group_visual_tracks(ekfs, tracks_per_filter, params_per_filter):
    """hv_ekf_group_visual_tracks: the visual-update chains of several filters of one context with the launches of one chain.
    tracks_per_filter[i]: filter i's tracks, as for Ekf.visual_tracks (may be empty); params_per_filter[i]: a VisualUpdateParams or a
    dict of Ekf.visual_tracks' keyword arguments (chi_outlier_r, visual_r, track_rmse_threshold, max_successful_updates, lookahead).
    Returns, per filter, what Ekf.visual_tracks returns: (list of dicts per track, number of successful updates). Raises HvError on a
    refusal (the filters are then untouched) and on a numerical failure."""
    n = len(ekfs)
    packed = [ekfs[i]._pack_tracks(t) if len(t) else (None, None) for i, t in enumerate(tracks_per_filter)]
    outs = [(TrackResult * len(t))() if len(t) else None for t in tracks_per_filter]
    E = (c_void_p * n)(*[e.h for e in ekfs])
    T = (ctypes.POINTER(TrackObs) * n)(*[ctypes.cast(obs, ctypes.POINTER(TrackObs)) if obs is not None else None for obs, _ in packed])
    K = (c_int * n)(*[len(t) for t in tracks_per_filter])
    P = (VisualUpdateParams * n)(*[p if isinstance(p, VisualUpdateParams) else _visual_params(**p) for p in params_per_filter])
    O = (ctypes.POINTER(TrackResult) * n)(*[ctypes.cast(o, ctypes.POINTER(TrackResult)) if o is not None else None for o in outs])
    succ = (c_int * n)()
    check(load().hv_ekf_group_visual_tracks(E, n, T, K, P, O, succ), "hv_ekf_group_visual_tracks")
    return [(_track_results(o) if o is not None else [], succ[i]) for i, o in enumerate(outs)]


def _visual_params(chi_outlier_r, visual_r, track_rmse_threshold=-1.0, max_successful_updates=5, lookahead=0):
    return VisualUpdateParams(chi_outlier_r, track_rmse_threshold, visual_r, max_successful_updates, lookahead)


def _track_results(out):
    return [{"tri_status": o.triangulator_status, "vu_status": o.prepare_vu_status, "outlier_status": o.outlier_status, "updated": bool(o.updated),
             "chi2": o.chi2, "pf": np.array(o.pf[:]), "depth": o.depth} for o in out]


class Context:
    """hv_ctx: one CUDA stream's worth of tracker + EKF work (the reference's Session, src/odometry/backend.cpp)."""

    def __init__(self, device=0, stream=None):
        self.lib = load()
        h = c_void_p()
        if stream is None:
            check(self.lib.hv_ctx_create(device, ctypes.byref(h)), "hv_ctx_create")
        else:
            check(self.lib.hv_ctx_create_on_stream(device, c_void_p(stream), ctypes.byref(h)), "hv_ctx_create_on_stream")
        self.h = h
        self.device = device

    def sync(self):
        check(self.lib.hv_ctx_sync(self.h), "hv_ctx_sync")

    @property
    def stream(self):
        return self.lib.hv_ctx_stream(self.h)

    @property
    def launches(self):
        return self.lib.hv_ctx_launch_count(self.h)

    def close(self):
        if self.h:
            self.lib.hv_ctx_destroy(self.h)
            self.h = None

    # ---- tracker::ImagePyramid::Factory::compute
    def pyramid(self, width, height, win=31, max_level=3):
        return Pyramid(self, width, height, win, max_level)

    def build_pyramids(self, pyrs, images, device=False):
        """One launch for several images (stereo pair). images: numpy (host) or torch tensors (host pinned / device)."""
        n = len(pyrs)
        P = (c_void_p * n)(*[p.h for p in pyrs])
        G = (c_void_p * n)(*[_ptr(im) for im in images])
        S = (c_size_t * n)(*[_stride0(im) for im in images])
        check(self.lib.hv_pyr_build_batch(P, G, S, n, 1 if device else 0), "hv_pyr_build_batch")

    def ingest_frames(self, jobs, device=False):
        """hv_ingest_frames: Ingest.frame for every job (see ingest_job) with the launches of one; asynchronous (synchronise before
        reading a gray_out). device: every source is a CUDA tensor, read in place; otherwise every source is host memory."""
        assert all(j.on_device == bool(device) for j in jobs), "sources must all be on the device (device=True) or all on the host"
        J = (IngestJob * len(jobs))(*jobs)
        check(self.lib.hv_ingest_frames(J, len(jobs), 1 if device else 0), "hv_ingest_frames")

    # ---- tracker::OpticalFlow::compute
    def lk_track(self, prev, nxt, prev_xy, next_xy=None, max_iter=20, eps=0.03, min_eig=1e-3):
        """Host-buffer LK. Returns (next_xy float32 (n,2), status uint8 (n,), track_status int32 (n,))."""
        prev_xy = np.ascontiguousarray(prev_xy, dtype=np.float32)
        n = prev_xy.shape[0]
        use_initial = next_xy is not None
        out = np.ascontiguousarray(next_xy, dtype=np.float32).copy() if use_initial else np.zeros((n, 2), np.float32)
        status = np.zeros(n, np.uint8)
        ts = np.zeros(n, np.int32)
        check(self.lib.hv_lk_track(self.h, prev.h, nxt.h, _ptr(prev_xy), _ptr(out), _ptr(status), _ptr(ts), n,
                                   1 if use_initial else 0, max_iter, eps, min_eig), "hv_lk_track")
        return out, status, ts

    def gftt_select_device(self, d_kp, d_corners, d_count, d_prev=None, mask_radius=0, max_tracks=150):
        """hv_gftt_select_device on contiguous CUDA tensors: d_kp (nkp, 3) float32 key points, d_prev (nprev, 2) float32 or None,
        d_corners (capacity, 2) float32 and d_count (1,) int32 outputs; asynchronous on the context's stream."""
        for t in (d_kp, d_corners, d_count) + (() if d_prev is None else (d_prev,)):
            assert t.is_cuda and t.is_contiguous() and t.element_size() == 4
        nprev = 0 if d_prev is None else d_prev.numel() // 2
        check(self.lib.hv_gftt_select_device(self.h, _ptr(d_kp), d_kp.numel() // 3, _ptr(d_prev), nprev, mask_radius, max_tracks,
                                             _ptr(d_corners), d_corners.numel() // 2, _ptr(d_count)), "hv_gftt_select_device")

    # ---- the new-corner step of many sessions: one launch per call (see corner_job / subpix_job for the jobs)
    def gftt_detect_batch_device(self, jobs, block_size=3, cell=32, min_response=1e-3):
        """hv_gftt_detect_batch_device: every job's key points (d_kp) from level 0 of its pyramid; asynchronous."""
        J = (CornerJob * len(jobs))(*jobs)
        check(self.lib.hv_gftt_detect_batch_device(self.h, J, len(jobs), block_size, cell, min_response), "hv_gftt_detect_batch_device")

    def gftt_select_batch_device(self, jobs):
        """hv_gftt_select_batch_device: every job's corner list and count from its nkp key points; asynchronous."""
        J = (CornerJob * len(jobs))(*jobs)
        check(self.lib.hv_gftt_select_batch_device(self.h, J, len(jobs)), "hv_gftt_select_batch_device")

    def subpix_refine_batch_device(self, jobs, win=(5, 5), zero_zone=(-1, -1), criteria=(3, 30, 0.01)):
        """hv_subpix_refine_batch_device: every job's points refined in place on level 0 of its pyramid; asynchronous."""
        J = (SubpixJob * len(jobs))(*jobs)
        check(self.lib.hv_subpix_refine_batch_device(self.h, J, len(jobs), win[0], win[1], zero_zone[0], zero_zone[1],
                                                     criteria[0], criteria[1], criteria[2]), "hv_subpix_refine_batch_device")

    def fast_detect_batch_device(self, jobs, threshold=10, nonmax=True):
        """hv_fast_detect_batch_device: cv::FAST on level 0 of every job's pyramid (see fast_job), two launches; asynchronous."""
        J = (FastJob * len(jobs))(*jobs)
        check(self.lib.hv_fast_detect_batch_device(self.h, J, len(jobs), threshold, 1 if nonmax else 0), "hv_fast_detect_batch_device")

    def good_features_batch_device(self, jobs, quality_level=0.01, min_distance=10.0, block_size=3):
        """hv_good_features_batch_device: cv::goodFeaturesToTrack on level 0 of every job's pyramid (see good_features_job), three
        launches; asynchronous."""
        J = (GoodFeaturesJob * len(jobs))(*jobs)
        check(self.lib.hv_good_features_batch_device(self.h, J, len(jobs), block_size, quality_level, min_distance),
              "hv_good_features_batch_device")

    # ---- cv::findEssentialMat(..., RANSAC, prob, threshold, max_iters): one launch per call
    def find_essential(self, xy1, xy2, fx, fy, cx, cy, prob=0.999, threshold=1.0, max_iters=1000, status=None):
        """hv_find_essential on host arrays: xy1, xy2 (n, 2) float32 (converted), status (n,) uint8 or None. Returns (E, mask) as
        cv2.findEssentialMat returns them: E (nsol, 3, 3) float64 row-major (nsol 0 where cv2 returns None), mask (n,) uint8."""
        a = np.ascontiguousarray(xy1, np.float32).reshape(-1, 2)
        b = np.ascontiguousarray(xy2, np.float32).reshape(-1, 2)
        if a.shape != b.shape:
            raise ValueError(f"xy1 {a.shape} and xy2 {b.shape} differ")
        n = a.shape[0]
        st = None if status is None else np.ascontiguousarray(status, np.uint8)
        if st is not None and st.shape != (n,):
            raise ValueError(f"status {st.shape} is not ({n},)")
        E = np.zeros(90, np.float64)
        mask = np.zeros(max(n, 1), np.uint8)
        nsol, inl = ctypes.c_int(), ctypes.c_int()
        check(self.lib.hv_find_essential(self.h, _ptr(a), _ptr(b), _ptr(st), n, fx, fy, cx, cy, prob, threshold, max_iters, _ptr(E),
                                         ctypes.byref(nsol), _ptr(mask), ctypes.byref(inl)), "hv_find_essential")
        return np.ascontiguousarray(E.reshape(10, 3, 3)[:nsol.value].transpose(0, 2, 1)), mask[:n]

    def find_essential_device(self, d_xy1, d_xy2, d_E, d_nsol, d_mask, d_inliers, fx, fy, cx, cy, prob=0.999, threshold=1.0,
                              max_iters=1000, d_status=None, n=None):
        """hv_find_essential_device on CUDA tensors (see essential_job for the buffers); asynchronous on the context's stream."""
        j = essential_job(d_xy1, d_xy2, d_E, d_nsol, d_mask, d_inliers, fx, fy, cx, cy, d_status, n)
        check(self.lib.hv_find_essential_device(self.h, j.d_xy1, j.d_xy2, j.d_status, j.n, fx, fy, cx, cy, prob, threshold, max_iters,
                                                j.d_E, j.d_nsol, j.d_mask, j.d_inliers), "hv_find_essential_device")

    def find_essential_batch_device(self, jobs, prob=0.999, threshold=1.0, max_iters=1000):
        """hv_find_essential_batch_device: every job (see essential_job) in one launch; asynchronous."""
        J = (EssentialJob * len(jobs))(*jobs)
        check(self.lib.hv_find_essential_batch_device(self.h, J, len(jobs), prob, threshold, max_iters), "hv_find_essential_batch_device")

    # ---- cv::recoverPose(E, xy1, xy2, K, R, t, distance_thresh, mask): one launch per call
    def recover_pose(self, E, xy1, xy2, fx, fy, cx, cy, distance_thresh=50.0, mask=None):
        """hv_recover_pose on host arrays: E (3, 3) row-major, xy1, xy2 (n, 2) float32 (converted), mask (n,) or (n, 1) uint8 or None.
        Returns (good, R (3, 3), t (3, 1), mask (n, 1) uint8) as cv2.recoverPose returns them: the mask holds mask's value where a
        point is good (255 without a mask), 0 elsewhere."""
        E = np.asarray(E, np.float64)
        if E.shape != (3, 3):
            raise ValueError(f"E {E.shape} is not (3, 3) (cv2.recoverPose refuses a stacked E; pass its first matrix)")
        Ecm = np.ascontiguousarray(E.T)
        a = np.ascontiguousarray(xy1, np.float32).reshape(-1, 2)
        b = np.ascontiguousarray(xy2, np.float32).reshape(-1, 2)
        if a.shape != b.shape:
            raise ValueError(f"xy1 {a.shape} and xy2 {b.shape} differ")
        n = a.shape[0]
        mi = None if mask is None else np.ascontiguousarray(mask, np.uint8).reshape(-1)
        if mi is not None and mi.shape != (n,):
            raise ValueError(f"mask {np.shape(mask)} does not hold {n} points")
        R, t = np.zeros(9, np.float64), np.zeros(3, np.float64)
        out = np.zeros(max(n, 1), np.uint8)
        good = ctypes.c_int()
        check(self.lib.hv_recover_pose(self.h, _ptr(Ecm), _ptr(a), _ptr(b), _ptr(mi), n, fx, fy, cx, cy, distance_thresh, _ptr(R), _ptr(t),
                                       _ptr(out), ctypes.byref(good)), "hv_recover_pose")
        keep = np.uint8(255) if mi is None else mi
        return good.value, R.reshape(3, 3).T.copy(), t.reshape(3, 1), np.where(out[:n] != 0, keep, 0).astype(np.uint8).reshape(n, 1)

    def recover_pose_device(self, d_E, d_xy1, d_xy2, d_R, d_t, d_mask_out, d_good, fx, fy, cx, cy, distance_thresh=50.0, d_nsol=None,
                            d_mask_in=None, n=None):
        """hv_recover_pose_device on CUDA tensors (see pose_job for the buffers); asynchronous on the context's stream."""
        j = pose_job(d_E, d_xy1, d_xy2, d_R, d_t, d_mask_out, d_good, fx, fy, cx, cy, d_nsol, d_mask_in, n)
        check(self.lib.hv_recover_pose_device(self.h, j.d_E, j.d_nsol, j.d_xy1, j.d_xy2, j.d_mask_in, j.n, fx, fy, cx, cy, distance_thresh,
                                              j.d_R, j.d_t, j.d_mask_out, j.d_good), "hv_recover_pose_device")

    def recover_pose_batch_device(self, jobs, distance_thresh=50.0):
        """hv_recover_pose_batch_device: every job (see pose_job) in one launch; asynchronous."""
        J = (PoseJob * len(jobs))(*jobs)
        check(self.lib.hv_recover_pose_batch_device(self.h, J, len(jobs), distance_thresh), "hv_recover_pose_batch_device")

    def lk_track_device(self, prev, nxt, d_prev, d_next, d_status, d_ts, n, use_initial, max_iter=20, eps=0.03, min_eig=1e-3):
        check(self.lib.hv_lk_track_device(self.h, prev.h, nxt.h, _ptr(d_prev), _ptr(d_next), _ptr(d_status), _ptr(d_ts), n,
                                          1 if use_initial else 0, max_iter, eps, min_eig), "hv_lk_track_device")


    def lk_track_device_on_stream(self, cuda_stream, prev, nxt, d_prev, d_init, d_next, d_status, d_ts, n, max_iter=20, eps=0.03, min_eig=1e-3):
        """The same launch on a stream of the caller; d_init (or None): predicted end points, read from their own buffer."""
        check(self.lib.hv_lk_track_device_on_stream(self.h, c_void_p(int(cuda_stream)), prev.h, nxt.h, _ptr(d_prev), _ptr(d_init), _ptr(d_next),
                                                    _ptr(d_status), _ptr(d_ts), n, max_iter, eps, min_eig), "hv_lk_track_device_on_stream")


def _check_cuda_buffer(t):
    assert t.is_cuda and t.is_contiguous() and t.element_size() == 4
    return t


def corner_job(pyr=None, d_kp=None, d_corners=None, d_count=None, d_prev=None, mask_radius=0, max_tracks=150, nkp=None):
    """A CornerJob on contiguous CUDA tensors: d_kp (nkp, 3) float32 (nkp: all its rows unless given), d_corners (capacity, 2) float32,
    d_count (1,) int32, d_prev (nprev, 2) float32 or None; pyr a Pyramid (detect) or None (select only). The tensors must outlive the
    calls that use the job."""
    for t in (d_kp, d_corners, d_count, d_prev):
        if t is not None:
            _check_cuda_buffer(t)
    if nkp is None:
        nkp = 0 if d_kp is None else d_kp.numel() // 3
    return CornerJob(None if pyr is None else pyr.h.value, _ptr(d_kp), nkp,
                     _ptr(d_prev), 0 if d_prev is None else d_prev.numel() // 2, mask_radius, max_tracks,
                     _ptr(d_corners), 0 if d_corners is None else d_corners.numel() // 2, _ptr(d_count))


def subpix_job(pyr, d_xy, n=None):
    """A SubpixJob: the first n (all) points of a contiguous (m, 2) float32 CUDA tensor on level 0 of pyr."""
    _check_cuda_buffer(d_xy)
    return SubpixJob(pyr.h.value, _ptr(d_xy), d_xy.numel() // 2 if n is None else n)


def fast_job(pyr, d_xy, d_count, d_response=None):
    """A FastJob on contiguous CUDA tensors: d_xy (capacity, 2) float32, d_count (1,) int32, d_response (capacity,) float32 or None.
    The tensors must outlive the call that uses the job."""
    for t in (d_xy, d_count) + (() if d_response is None else (d_response,)):
        _check_cuda_buffer(t)
    return FastJob(pyr.h.value, _ptr(d_xy), _ptr(d_response), d_xy.numel() // 2, _ptr(d_count))


def _mask_tensor(d_mask, pyr):
    """A CUDA uint8 mask of level 0's shape (h, w) whose rows are dense: (pointer, row stride in bytes); None: (None, 0)."""
    if d_mask is None:
        return None, 0
    import torch
    w, h = pyr.level_size(0)
    if not d_mask.is_cuda or d_mask.dtype != torch.uint8 or d_mask.dim() != 2 or d_mask.stride(1) != 1:
        raise ValueError("the mask must be a 2-D uint8 CUDA tensor with dense rows")
    if tuple(d_mask.shape) != (h, w):
        raise ValueError(f"the mask is {tuple(d_mask.shape)}, level 0 is {(h, w)}")
    return d_mask.data_ptr(), d_mask.stride(0)


def good_features_job(pyr, d_xy, d_count, max_corners, d_response=None, d_mask=None):
    """A GoodFeaturesJob on CUDA tensors: d_xy (capacity, 2) float32, d_count (1,) int32, d_response (capacity,) float32 or None,
    d_mask (h, w) uint8 with dense rows (any row stride) or None. The tensors must outlive the call that uses the job."""
    for t in (d_xy, d_count) + (() if d_response is None else (d_response,)):
        _check_cuda_buffer(t)
    mp, ms = _mask_tensor(d_mask, pyr)
    return GoodFeaturesJob(pyr.h.value, max_corners, mp, ms, _ptr(d_xy), _ptr(d_response), d_xy.numel() // 2, _ptr(d_count))


def essential_job(d_xy1, d_xy2, d_E, d_nsol, d_mask, d_inliers, fx, fy, cx, cy, d_status=None, n=None):
    """An EssentialJob on contiguous CUDA tensors: d_xy1, d_xy2 (capacity, 2) float32, d_status (capacity,) uint8 or None, d_E (90,) or
    (10, 3, 3) float64 (column-major slots), d_nsol and d_inliers (1,) int32, d_mask (capacity,) uint8; n: the first n points (all).
    The tensors must outlive the call that uses the job."""
    for t, size in ((d_xy1, 4), (d_xy2, 4), (d_E, 8), (d_nsol, 4), (d_mask, 1), (d_inliers, 4)) + (() if d_status is None else ((d_status, 1),)):
        if not t.is_cuda or not t.is_contiguous() or t.element_size() != size:
            raise ValueError("essential_job: every buffer must be a contiguous CUDA tensor of the documented dtype")
    cap = d_xy1.numel() // 2
    n = cap if n is None else n
    if d_xy2.numel() // 2 < n or d_mask.numel() < n or d_E.numel() < 90 or (d_status is not None and d_status.numel() < n) or n > cap:
        raise ValueError("essential_job: a buffer is smaller than n points (or E smaller than 90 doubles)")
    return EssentialJob(_ptr(d_xy1), _ptr(d_xy2), _ptr(d_status), n, fx, fy, cx, cy, _ptr(d_E), _ptr(d_nsol), _ptr(d_mask), _ptr(d_inliers))


def pose_job(d_E, d_xy1, d_xy2, d_R, d_t, d_mask_out, d_good, fx, fy, cx, cy, d_nsol=None, d_mask_in=None, n=None):
    """A PoseJob on contiguous CUDA tensors: d_E float64 (at least 9: column-major, the first slot is used), d_nsol (1,) int32 or None
    (E holds one matrix), d_xy1, d_xy2 (capacity, 2) float32, d_mask_in (capacity,) uint8 or None, d_R (9,) or (3, 3) float64
    (column-major), d_t (3,) float64, d_mask_out (capacity,) uint8 (may be d_mask_in), d_good (1,) int32; n: the first n points (all).
    The tensors must outlive the call that uses the job."""
    opt = tuple((t, s) for t, s in ((d_nsol, 4), (d_mask_in, 1)) if t is not None)
    for t, size in ((d_E, 8), (d_xy1, 4), (d_xy2, 4), (d_R, 8), (d_t, 8), (d_mask_out, 1), (d_good, 4)) + opt:
        if not t.is_cuda or not t.is_contiguous() or t.element_size() != size:
            raise ValueError("pose_job: every buffer must be a contiguous CUDA tensor of the documented dtype")
    cap = d_xy1.numel() // 2
    n = cap if n is None else n
    if (d_xy2.numel() // 2 < n or d_mask_out.numel() < n or (d_mask_in is not None and d_mask_in.numel() < n) or n > cap
            or d_E.numel() < 9 or d_R.numel() < 9 or d_t.numel() < 3):
        raise ValueError("pose_job: a buffer is smaller than n points (or E, R, t smaller than 9, 9, 3 doubles)")
    return PoseJob(_ptr(d_E), _ptr(d_nsol), _ptr(d_xy1), _ptr(d_xy2), _ptr(d_mask_in), n, fx, fy, cx, cy, _ptr(d_R), _ptr(d_t),
                   _ptr(d_mask_out), _ptr(d_good))


def _dense_rows(img):
    """A host image as Ingest.frame passes it: a uint8 view whose rows are dense keeps its own row stride, any other layout is copied."""
    img = np.asarray(img)
    channels = 1 if img.ndim == 2 else img.shape[2]
    if img.dtype != np.uint8 or img.strides[1:] != ((channels, 1) if img.ndim == 3 else (1,)) or img.strides[0] < img.shape[1] * channels:
        img = np.ascontiguousarray(img, np.uint8)
    return img, channels


def _coeff_array(coeff):
    return None if coeff is None else np.ascontiguousarray(list(coeff) + [0.0] * (4 - len(coeff)), np.float64)


def ingest_job(ing, img, pyr, coeff=None, gray_out=None):
    """An IngestJob: frame img ((h, w) gray or (h, w, channels) uint8) through `ing` into `pyr`. img is a numpy array (host; a view whose
    rows are dense keeps its own row stride, as Ingest.frame passes it) or a torch uint8 tensor with dense rows (a CUDA tensor for
    Context.ingest_frames(..., device=True), else host memory, pinned for an asynchronous copy). gray_out: None or a (h, w) uint8 C-contiguous
    numpy array that receives the ingested image. The job keeps img, the coefficients and gray_out alive."""
    if isinstance(img, np.ndarray) or not hasattr(img, "data_ptr"):
        img, channels = _dense_rows(img)
        on_device = False
    else:
        channels = 1 if img.dim() == 2 else img.shape[2]
        assert img.dtype.itemsize == 1 and img.stride()[1:] == ((channels, 1) if img.dim() == 3 else (1,)), "rows must be dense"
        on_device = img.is_cuda
    if gray_out is not None:
        assert gray_out.dtype == np.uint8 and gray_out.shape == (ing.h, ing.w) and gray_out.flags.c_contiguous
    cf = _coeff_array(coeff)
    job = IngestJob(ing.h_.value, _ptr(img), _stride0(img), channels, _ptr(cf), pyr.h.value, _ptr(gray_out))
    job.on_device, job.keep = on_device, (img, cf, gray_out)
    return job


def gftt_select_capacity(nkp, mask_radius, max_tracks):
    """Corner slots a selection over nkp key points can fill (the capacity hv_gftt_select_device / hv_gftt_corners require)."""
    return min(max_tracks, 2 * nkp) if mask_radius > 0 else 2 * nkp


def _stride0(im):
    if isinstance(im, np.ndarray):
        return im.strides[0]
    return im.stride(0) * im.element_size()


class Pyramid:
    """hv_pyr: tracker::ImagePyramid (src/tracker/image_pyramid.hpp:18-42)."""

    def __init__(self, ctx, width, height, win, max_level):
        self.ctx, self.lib = ctx, ctx.lib
        h = c_void_p()
        check(self.lib.hv_pyr_create(ctx.h, width, height, win, max_level, ctypes.byref(h)), "hv_pyr_create")
        self.h = h
        self.win = win
        self.levels = self.lib.hv_pyr_levels(h)

    def level_size(self, level):
        w, h = c_int(), c_int()
        check(self.lib.hv_pyr_level_size(self.h, level, ctypes.byref(w), ctypes.byref(h)), "hv_pyr_level_size")
        return w.value, h.value

    def build(self, gray):
        assert gray.dtype == np.uint8 and gray.ndim == 2
        check(self.lib.hv_pyr_build(self.h, _ptr(gray), gray.strides[0]), "hv_pyr_build")

    def download(self, level, padded=False):
        w, h = self.level_size(level)
        if padded:
            w, h = w + 2 * self.win, h + 2 * self.win
        g = np.zeros((h, w), np.uint8)
        d = np.zeros((h, w, 2), np.int16)
        fn = self.lib.hv_pyr_download_level_padded if padded else self.lib.hv_pyr_download_level
        check(fn(self.h, level, _ptr(g), _ptr(d)), "hv_pyr_download_level")
        return g, d

    def gftt_cells(self, cell=32):
        cx, cy = c_int(), c_int()
        check(self.lib.hv_gftt_cells(self.h, cell, ctypes.byref(cx), ctypes.byref(cy)), "hv_gftt_cells")
        return cx.value, cy.value

    def gftt_detect(self, block_size=3, cell=32, min_response=1e-3):
        """Device part of tracker::FeatureDetector::detect on the level-0 image of this pyramid: (cells, 3) float32 (x, y, response)."""
        cx, cy = self.gftt_cells(cell)
        kp = np.zeros((cx * cy, 3), np.float32)
        check(self.lib.hv_gftt_detect(self.ctx.h, self.h, block_size, cell, min_response, _ptr(kp)), "hv_gftt_detect")
        return kp

    def gftt_detect_device(self, d_kp, block_size=3, cell=32, min_response=1e-3):
        check(self.lib.hv_gftt_detect_device(self.ctx.h, self.h, block_size, cell, min_response, d_kp), "hv_gftt_detect_device")

    def gftt_corners(self, prev=None, mask_radius=0, max_tracks=150, block_size=3, cell=32, min_response=1e-3):
        """tracker::FeatureDetector::detect on the level-0 image of this pyramid: detection, stable sort, resize quirk and applyMinDistance
        against `prev` ((nprev, 2) corners already tracked) on the device, one synchronisation. Returns the corners, (n, 2) float32."""
        prev = np.zeros((0, 2), np.float32) if prev is None else np.ascontiguousarray(prev, np.float32).reshape(-1, 2)
        cap = gftt_select_capacity(int(np.prod(self.gftt_cells(cell))), mask_radius, max_tracks)
        out = np.zeros((max(cap, 1), 2), np.float32)
        n = c_int(0)
        check(self.lib.hv_gftt_corners(self.ctx.h, self.h, block_size, cell, min_response, _ptr(prev), len(prev), mask_radius, max_tracks,
                                       _ptr(out), cap, ctypes.byref(n)), "hv_gftt_corners")
        return out[:n.value].copy()

    def subpix_refine(self, xy, win=(5, 5), zero_zone=(-1, -1), criteria=(3, 30, 0.01)):
        """cv::cornerSubPix on the level-0 image of this pyramid; criteria = (type: 1 COUNT | 2 EPS, max_count, epsilon).
        Returns the refined points as a new (n, 2) float32 array."""
        out = np.ascontiguousarray(xy, dtype=np.float32).reshape(-1, 2).copy()
        check(self.lib.hv_subpix_refine(self.ctx.h, self.h, _ptr(out), len(out), win[0], win[1], zero_zone[0], zero_zone[1],
                                        criteria[0], criteria[1], criteria[2]), "hv_subpix_refine")
        return out

    def subpix_refine_device(self, d_xy, win=(5, 5), zero_zone=(-1, -1), criteria=(3, 30, 0.01)):
        """The same on a contiguous (n, 2) float32 CUDA tensor, refined in place on the context's stream (asynchronous)."""
        assert d_xy.is_cuda and d_xy.is_contiguous() and d_xy.is_floating_point() and d_xy.element_size() == 4
        n = d_xy.numel() // 2
        check(self.lib.hv_subpix_refine_device(self.ctx.h, self.h, _ptr(d_xy), n, win[0], win[1], zero_zone[0], zero_zone[1],
                                               criteria[0], criteria[1], criteria[2]), "hv_subpix_refine_device")

    def fast_detect(self, threshold=10, nonmax=True, capacity=None):
        """cv::FAST (TYPE_9_16) on the level-0 image of this pyramid. Returns (xy (n, 2) float32, response (n,) float32) in OpenCV's
        order: every keypoint, or the first `capacity` of them when a capacity is given (a second call fetches the rest when the
        first guess of 4096 was too small)."""
        cap = 4096 if capacity is None else capacity
        while True:
            xy = np.zeros((max(cap, 1), 2), np.float32)
            resp = np.zeros(max(cap, 1), np.float32)
            n = c_int(0)
            check(self.lib.hv_fast_detect(self.ctx.h, self.h, threshold, 1 if nonmax else 0, _ptr(xy), _ptr(resp), cap, ctypes.byref(n)),
                  "hv_fast_detect")
            if capacity is not None or n.value <= cap:
                m = min(n.value, cap)
                return xy[:m].copy(), resp[:m].copy()
            cap = n.value

    def fast_detect_device(self, d_xy, d_count, d_response=None, threshold=10, nonmax=True):
        """hv_fast_detect_device on contiguous CUDA tensors: d_xy (capacity, 2) float32, d_count (1,) int32, d_response (capacity,)
        float32 or None; asynchronous on the context's stream."""
        for t in (d_xy, d_count) + (() if d_response is None else (d_response,)):
            _check_cuda_buffer(t)
        check(self.lib.hv_fast_detect_device(self.ctx.h, self.h, threshold, 1 if nonmax else 0, _ptr(d_xy), _ptr(d_response),
                                             d_xy.numel() // 2, _ptr(d_count)), "hv_fast_detect_device")

    def good_features(self, max_corners, quality_level, min_distance, mask=None, block_size=3):
        """cv::goodFeaturesToTrack (minimum-eigenvalue response) on the level-0 image of this pyramid. mask: None or an (h, w) uint8
        array (non-zero: allowed). Returns (xy (n, 2) float32, response (n,) float32) in OpenCV's order, n <= max_corners."""
        mp, ms = None, 0
        if mask is not None:
            mask = np.asarray(mask)
            w, h = self.level_size(0)
            if mask.shape != (h, w):
                raise ValueError(f"the mask is {mask.shape}, level 0 is {(h, w)}")
            if mask.dtype != np.uint8 or mask.strides[1] != 1 or mask.strides[0] < w:
                mask = np.ascontiguousarray(mask, np.uint8)
            mp, ms = mask.ctypes.data, mask.strides[0]
        cap = max(int(max_corners), 1)
        xy = np.zeros((cap, 2), np.float32)
        resp = np.zeros(cap, np.float32)
        n = c_int(0)
        check(self.lib.hv_good_features(self.ctx.h, self.h, block_size, max_corners, quality_level, min_distance, mp, ms, _ptr(xy),
                                        _ptr(resp), cap, ctypes.byref(n)), "hv_good_features")
        return xy[:n.value].copy(), resp[:n.value].copy()

    def good_features_device(self, d_xy, d_count, max_corners, quality_level, min_distance, d_response=None, d_mask=None, block_size=3):
        """hv_good_features_device on CUDA tensors: d_xy (capacity, 2) float32, d_count (1,) int32, d_response (capacity,) float32 or
        None, d_mask (h, w) uint8 with dense rows or None; asynchronous on the context's stream."""
        for t in (d_xy, d_count) + (() if d_response is None else (d_response,)):
            _check_cuda_buffer(t)
        mp, ms = _mask_tensor(d_mask, self)
        check(self.lib.hv_good_features_device(self.ctx.h, self.h, block_size, max_corners, quality_level, min_distance, mp, ms,
                                               _ptr(d_xy), _ptr(d_response), d_xy.numel() // 2, _ptr(d_count)), "hv_good_features_device")

    def release(self):
        if self.h:
            self.lib.hv_pyr_release(self.h)
            self.h = None


class Ingest:
    """hv_ingest: device part of tracker::Image::Factory::build (colour -> gray, undistortion / rectification) feeding a pyramid."""

    def __init__(self, ctx, width, height):
        self.ctx, self.lib, self.w, self.h = ctx, ctx.lib, width, height
        h = c_void_p()
        check(self.lib.hv_ingest_create(ctx.h, width, height, ctypes.byref(h)), "hv_ingest_create")
        self.h_ = h

    def set_remap(self, table):
        if table is None:
            check(self.lib.hv_ingest_set_remap(self.h_, None), "hv_ingest_set_remap")
            return
        assert table.dtype.itemsize == 12 and table.size == self.w * self.h
        check(self.lib.hv_ingest_set_remap(self.h_, _ptr(np.ascontiguousarray(table))), "hv_ingest_set_remap")

    def frame(self, img, pyr, coeff=None, want_gray=True):
        """img: (h, w) gray or (h, w, channels) uint8. A view whose rows are dense (e.g. a crop of a wider buffer) is passed with its own
        row stride, as the C adapters pass an image's bytesPerRow(); any other layout is copied first."""
        img, channels = _dense_rows(img)
        out = np.zeros((self.h, self.w), np.uint8) if want_gray else None
        cf = _coeff_array(coeff)
        check(self.lib.hv_ingest_frame(self.h_, _ptr(img), img.strides[0], channels, None if cf is None else _ptr(cf), pyr.h, None if out is None else _ptr(out)),
              "hv_ingest_frame")
        self.ctx.sync()
        return out

    def close(self):
        if self.h_:
            self.lib.hv_ingest_destroy(self.h_)
            self.h_ = None


def _dd(a):
    return np.ascontiguousarray(a, dtype=np.float64)


class Ekf:
    """hv_ekf: odometry::EKF (src/odometry/ekf.hpp:62-174) with m and P resident on the device."""
    name = "cuda"

    def __init__(self, ctx, params=None, handle=None):
        self.ctx, self.lib = ctx, ctx.lib
        if handle is None:
            if params is None:
                params = EkfParams()
                self.lib.hv_ekf_default_params(ctypes.byref(params))
            h = c_void_p()
            check(self.lib.hv_ekf_create(ctx.h, ctypes.byref(params), ctypes.byref(h)), "hv_ekf_create")
            handle = h
        self.params = params
        self.h = handle
        self.N = self.lib.hv_ekf_state_dim(self.h)

    def clone(self):
        h = c_void_p()
        check(self.lib.hv_ekf_clone(self.h, ctypes.byref(h)), "hv_ekf_clone")
        return Ekf(self.ctx, self.params, h)

    def close(self):
        if self.h:
            self.lib.hv_ekf_destroy(self.h)
            self.h = None

    def upload(self, m=None, P=None):
        m = None if m is None else _dd(m)
        P = None if P is None else np.asfortranarray(P, dtype=np.float64)
        check(self.lib.hv_ekf_upload(self.h, _ptr(m), _ptr(P)), "hv_ekf_upload")

    def download(self):
        m = np.zeros(self.N); P = np.zeros((self.N, self.N), order="F")
        check(self.lib.hv_ekf_download(self.h, _ptr(m), _ptr(P)), "hv_ekf_download")
        return m, P

    def download_inertial(self):
        m = np.zeros(20); P = np.zeros((20, 20), order="F")
        check(self.lib.hv_ekf_download_inertial(self.h, _ptr(m), _ptr(P)), "hv_ekf_download_inertial")
        return m, P

    def set_inertial_state(self, m20, P20):
        m20 = _dd(m20); P20 = np.asfortranarray(P20, dtype=np.float64)
        check(self.lib.hv_ekf_set_inertial_state(self.h, _ptr(m20), _ptr(P20)), "hv_ekf_set_inertial_state")

    def set_process_noise(self, Q):
        Q = np.asfortranarray(Q, dtype=np.float64)
        check(self.lib.hv_ekf_set_process_noise(self.h, _ptr(Q)), "hv_ekf_set_process_noise")

    def get_dydx(self):
        d = np.zeros((20, 20), order="F")
        check(self.lib.hv_ekf_get_dydx(self.h, _ptr(d)), "hv_ekf_get_dydx")
        return d

    def pose_count(self): return self.lib.hv_ekf_pose_count(self.h)
    def platform_time(self): return self.lib.hv_ekf_platform_time(self.h)
    def history_time(self, i): return self.lib.hv_ekf_history_time(self.h, i)
    def was_stationary(self): return bool(self.lib.hv_ekf_was_stationary(self.h))
    def set_first_sample_time(self, t): check(self.lib.hv_ekf_set_first_sample_time(self.h, t), "hv_ekf_set_first_sample_time")

    def initialize_orientation(self, acc): check(self.lib.hv_ekf_initialize_orientation(self.h, _ptr(_dd(acc))), "hv_ekf_initialize_orientation")

    def predict(self, t, gyro, acc):
        g, a = _dd(gyro), _dd(acc)
        check(self.lib.hv_ekf_predict(self.h, t, _ptr(g), _ptr(a)), "hv_ekf_predict")

    def update_zupt(self, r): check(self.lib.hv_ekf_update_zupt(self.h, r), "hv_ekf_update_zupt")
    def update_zupt_initialization(self): check(self.lib.hv_ekf_update_zupt_initialization(self.h), "hv_ekf_update_zupt_initialization")
    def update_zrupt(self, gyro): check(self.lib.hv_ekf_update_zrupt(self.h, _ptr(_dd(gyro))), "hv_ekf_update_zrupt")
    def update_pseudo_velocity(self, speed, r): check(self.lib.hv_ekf_update_pseudo_velocity(self.h, speed, r), "hv_ekf_update_pseudo_velocity")
    def update_position(self, pos, r): check(self.lib.hv_ekf_update_position(self.h, _ptr(_dd(pos)), r), "hv_ekf_update_position")
    def update_zero_height(self, r): check(self.lib.hv_ekf_update_zero_height(self.h, r), "hv_ekf_update_zero_height")
    def update_orientation(self, q, r): check(self.lib.hv_ekf_update_orientation(self.h, _ptr(_dd(q)), r), "hv_ekf_update_orientation")

    def visual_check(self, H, f, y, r, rmse_thr=-1.0):
        H = np.asfortranarray(H, dtype=np.float64); f, y = _dd(f), _dd(y)
        st, chi2 = c_int(-1), c_double(0.0)
        check(self.lib.hv_ekf_visual_check(self.h, _ptr(H), H.shape[0], H.shape[1], _ptr(f), _ptr(y), r, rmse_thr,
                                           ctypes.byref(st), ctypes.byref(chi2)), "hv_ekf_visual_check")
        return st.value, chi2.value

    def visual_update(self, H, f, y, r):
        H = np.asfortranarray(H, dtype=np.float64); f, y = _dd(f), _dd(y)
        check(self.lib.hv_ekf_visual_update(self.h, _ptr(H), H.shape[0], H.shape[1], _ptr(f), _ptr(y), r), "hv_ekf_visual_update")

    def visual_check_update(self, H, f, y, r, rmse_thr=-1.0):
        H = np.asfortranarray(H, dtype=np.float64); f, y = _dd(f), _dd(y)
        st, chi2 = c_int(-1), c_double(0.0)
        m = np.zeros(self.N)
        check(self.lib.hv_ekf_visual_check_update(self.h, _ptr(H), H.shape[0], H.shape[1], _ptr(f), _ptr(y), r, rmse_thr,
                                                  ctypes.byref(st), ctypes.byref(chi2), _ptr(m)), "hv_ekf_visual_check_update")
        return st.value, chi2.value, m

    def visual_device(self, d_H, n, l, d_f, d_y, r, rmse_thr, mode, d_result=None):
        check(self.lib.hv_ekf_visual_device(self.h, _ptr(d_H), n, l, _ptr(d_f), _ptr(d_y), r, rmse_thr, mode, _ptr(d_result)),
              "hv_ekf_visual_device")

    def run_device(self, ops, nops):
        """ops: (EkfOp * k) array with DEVICE pointers; asynchronous."""
        check(self.lib.hv_ekf_run_device(self.h, ops, nops), "hv_ekf_run_device")

    def predicted_mean_device(self, d_ptr):
        """Mean part of the queued IMU samples into 20 doubles of DEVICE memory (own small launch; the full predict stays queued)."""
        check(self.lib.hv_ekf_predicted_mean_device(self.h, c_void_p(int(d_ptr))), "hv_ekf_predicted_mean_device")

    def predicted_mean(self):
        """The 20 inertial states the queued IMU samples lead to (host array); the full predict stays queued."""
        m = np.zeros(20)
        check(self.lib.hv_ekf_predicted_mean(self.h, _ptr(m)), "hv_ekf_predicted_mean")
        return m

    def run_device_results(self, nops):
        """(vu_status, chi2) arrays of the last run_device list (entries of non-VISUAL ops: -1 / nan); waits for the list."""
        st = np.full(nops, -1, dtype=np.int32); chi2 = np.full(nops, np.nan)
        check(self.lib.hv_ekf_run_device_results(self.h, nops, st.ctypes.data_as(ctypes.POINTER(c_int)), chi2.ctypes.data_as(ctypes.POINTER(c_double))),
              "hv_ekf_run_device_results")
        return st, chi2

    def run_host(self, ops, nops, want_m=False):
        """ops with HOST pointers; returns (vu_status int32[nops], chi2 float64[nops], m or None)."""
        st = (c_int * nops)(*([-1] * nops))
        chi2 = (c_double * nops)()
        m = np.zeros(self.N) if want_m else None
        check(self.lib.hv_ekf_run_host(self.h, ops, nops, st, chi2, _ptr(m)), "hv_ekf_run_host")
        return np.frombuffer(st, dtype=np.int32).copy(), np.frombuffer(chi2, dtype=np.float64).copy(), m

    def augment(self, drop=-1): check(self.lib.hv_ekf_augment(self.h, drop), "hv_ekf_augment")
    def unaugment(self): check(self.lib.hv_ekf_unaugment(self.h), "hv_ekf_unaugment")
    def symmetrize(self): check(self.lib.hv_ekf_symmetrize(self.h), "hv_ekf_symmetrize")
    def set_camera_model(self, imu_to_camera, second_imu_to_camera=None, use_stereo=False, estimate_time_shift=True, **kw):
        """hv_ekf_set_camera_model: 4x4 matrices as numpy (row, col); kw: other hv_camera_model fields."""
        c = CameraModel()
        self.lib.hv_camera_model_defaults(ctypes.byref(c))
        c.imu_to_camera[:] = list(np.asarray(imu_to_camera, np.float64).flatten(order="F"))
        if second_imu_to_camera is not None:
            c.second_imu_to_camera[:] = list(np.asarray(second_imu_to_camera, np.float64).flatten(order="F"))
        c.use_stereo = 1 if use_stereo else 0
        c.estimate_imu_camera_time_shift = 1 if estimate_time_shift else 0
        for k, v in kw.items():
            setattr(c, k, v)
        check(self.lib.hv_ekf_set_camera_model(self.h, ctypes.byref(c)), "hv_ekf_set_camera_model")
        self._stereo = bool(use_stereo)

    def track_models(self, tracks, download=True):
        """hv_ekf_track_models. tracks: list of (pose_trail_index, ip, velocities). Returns one dict per track: tri_status,
        vu_status, pf, depth, rows, cols, device pointers d_H / d_f / d_y and (download=True) H, f, dpf on the host."""
        n = len(tracks)
        obs = (TrackObs * n)()
        keep = []
        for k, (idx, ip, vel) in enumerate(tracks):
            idx = np.ascontiguousarray(idx, np.int32); ip = _dd(np.asarray(ip).ravel()); vel = _dd(np.asarray(vel).ravel())
            keep.append((idx, ip, vel))
            obs[k].npose = len(idx); obs[k].pose_trail_index = idx.ctypes.data; obs[k].ip = ip.ctypes.data; obs[k].velocities = vel.ctypes.data
        out = (TrackModel * n)()
        check(self.lib.hv_ekf_track_models(self.h, obs, n, out), "hv_ekf_track_models")
        res = []
        for k in range(n):
            o = out[k]
            d = {"tri_status": o.triangulator_status, "vu_status": o.prepare_vu_status, "rows": o.rows, "cols": o.cols,
                 "pf": np.array(o.pf[:]), "depth": o.depth, "d_H": o.d_H, "d_f": o.d_f, "d_y": o.d_y}
            if download:
                npose = len(keep[k][0])
                H = np.zeros((o.rows, o.cols), order="F"); f = np.zeros(o.rows); dpf = np.zeros((3, 7 * npose + 1), order="F")
                check(self.lib.hv_ekf_track_model_download(self.h, k, _ptr(H) if H.size else None, _ptr(f) if f.size else None, _ptr(dpf)),
                      "hv_ekf_track_model_download")
                d.update(H=H, f=f, dpf=dpf)
            res.append(d)
        return res

    def _pack_tracks(self, tracks):
        n = len(tracks)
        obs = (TrackObs * n)()
        keep = []
        for k, (idx, ip, vel) in enumerate(tracks):
            idx = np.ascontiguousarray(idx, np.int32); ip = _dd(np.asarray(ip).ravel()); vel = _dd(np.asarray(vel).ravel())
            keep.append((idx, ip, vel))
            obs[k].npose = len(idx); obs[k].pose_trail_index = idx.ctypes.data; obs[k].ip = ip.ctypes.data; obs[k].velocities = vel.ctypes.data
        return obs, keep

    def visual_tracks(self, tracks, chi_outlier_r, visual_r, track_rmse_threshold=-1.0, max_successful_updates=5, lookahead=0):
        """hv_ekf_visual_tracks: the per-track model -> check -> update chain with the control flow on the device.
        Returns (list of dicts per track, number of successful updates)."""
        obs, keep = self._pack_tracks(tracks)
        prm = _visual_params(chi_outlier_r, visual_r, track_rmse_threshold, max_successful_updates, lookahead)
        out = (TrackResult * len(tracks))()
        succ = c_int(0)
        check(self.lib.hv_ekf_visual_tracks(self.h, obs, len(tracks), ctypes.byref(prm), out, ctypes.byref(succ)), "hv_ekf_visual_tracks")
        return _track_results(out), succ.value

    def track_models_time(self, reps=50):
        """Average device time (us) of the kernel of the last track_models call."""
        ms = ctypes.c_float(0)
        check(self.lib.hv_ekf_track_models_time(self.h, reps, ctypes.byref(ms)), "hv_ekf_track_models_time")
        return ms.value * 1e3

    def visual_track(self, model, r, rmse_thr=-1.0, mode=0):
        """hv_ekf_visual_track on one dict returned by track_models: (VuOutlierStatus, chi2), or None for mode 1 (asynchronous)."""
        t = TrackModel()
        t.triangulator_status, t.prepare_vu_status, t.rows, t.cols = model["tri_status"], model["vu_status"], model["rows"], model["cols"]
        t.d_H, t.d_f, t.d_y = model["d_H"], model["d_f"], model["d_y"]
        st, chi2 = c_int(-1), c_double(0.0)
        check(self.lib.hv_ekf_visual_track(self.h, ctypes.byref(t), r, rmse_thr, mode, ctypes.byref(st), ctypes.byref(chi2)), "hv_ekf_visual_track")
        return None if mode == 1 else (st.value, chi2.value)

    def flush(self): check(self.lib.hv_ekf_flush(self.h), "hv_ekf_flush")
    def set_imu_batching(self, max_samples): check(self.lib.hv_ekf_set_imu_batching(self.h, int(max_samples)), "hv_ekf_set_imu_batching")
    def normalize_quaternions(self, only_current=False): check(self.lib.hv_ekf_normalize_quaternions(self.h, 1 if only_current else 0), "hv_ekf_normalize_quaternions")
    def translate_to(self, pos): check(self.lib.hv_ekf_translate_to(self.h, _ptr(_dd(pos))), "hv_ekf_translate_to")
    def transform_to(self, pos, q, i=-1): check(self.lib.hv_ekf_transform_to(self.h, _ptr(_dd(pos)), _ptr(_dd(q)), i), "hv_ekf_transform_to")
    def insert_map_point(self, idx, pf): check(self.lib.hv_ekf_insert_map_point(self.h, idx, _ptr(_dd(pf))), "hv_ekf_insert_map_point")
    def condition_on_last_pose(self): check(self.lib.hv_ekf_condition_on_last_pose(self.h), "hv_ekf_condition_on_last_pose")
    def lock_biases(self): check(self.lib.hv_ekf_lock_biases(self.h), "hv_ekf_lock_biases")
