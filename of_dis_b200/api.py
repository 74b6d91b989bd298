"""Python host side of the C-ABI (include/ofdis_b200.h), via ctypes.

`Context` is the batch engine; `OFClass`, `PatGridClass`, `VarRefClass` mirror the
reference's three classes (oflow.h:84-111, patchgrid.h:19-44,
refine_variational.h:37-39) with the same argument meaning, so the parity tests
read like calls into the reference.  There is NO CPU fallback: importing this
module loads of_dis_b200/lib/libofdis_b200.so and raises if it is missing.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from .params import CParams, DisParams
from .preprocess import (CONF_PARAM_FIELDS, DISP_FILTER_FIELDS, EGO_PARAM_FIELDS, FUSE_PARAM_FIELDS, FUSE_POINT_DTYPE,
                         FUSE_TRACK_PARAM_FIELDS, FUSE_TRACK_STATS_DTYPE, FISHER_MAX_BLOCKS, FISHER_STATS_DTYPE, MOTION_PARAM_FIELDS, MOTION_STATS_DTYPE, RELPOSE_PARAM_FIELDS, SF_STATS_DTYPE,
                         STAB_FRAME_DTYPE, STAB_PARAM_FIELDS, STEREO_CAMERA_FIELDS, TRACK_PARAM_FIELDS,
                         TRACK_POINT_DTYPE, TRACK_STATS_FIELDS, TRAJ_PARAM_FIELDS, TRAJ_RECORD_DTYPE, TRAJ_STATS_FIELDS,
                         fisher_fit, fisher_pack, fisher_sizes, gaussian_weights, motion_params,
                         traj_bound, traj_dim)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OFDIS_LIB") or os.path.join(_HERE, "lib", "libofdis_b200.so")  # OFDIS_LIB: experiments only
_FP = ctypes.POINTER(ctypes.c_float)
_IP = ctypes.POINTER(ctypes.c_int)

MEM_HOST, MEM_DEVICE = 0, 1

EXPORTS = [
    "ofdis_create", "ofdis_destroy", "ofdis_last_error", "ofdis_version", "ofdis_level_info",
    "ofdis_upload_level", "ofdis_packed_frame_floats", "ofdis_packed_offset", "ofdis_upload_packed",
    "ofdis_patgrid_optimize", "ofdis_patgrid_aggregate", "ofdis_varref_refine", "ofdis_run", "ofdis_sync",
    "ofdis_get_flow", "ofdis_set_flow", "ofdis_get_flow_batch", "ofdis_get_patches", "ofdis_debug_get",
    "ofdis_debug_varref_iters", "ofdis_launch_count", "ofdis_set_graph_mode", "ofdis_profile_run",
    "ofdis_set_camlr", "ofdis_set_dp_thresh_sq", "ofdis_packed_images_frame_floats", "ofdis_upload_packed_images",
    "ofdis_upload_frames_u8", "ofdis_finest_level_frame_floats", "ofdis_upload_finest_level", "ofdis_get_flow_fullres",
    "ofdis_get_level", "ofdis_upload_level_fb", "ofdis_set_option", "ofdis_profile_levels", "ofdis_set_direction",
    "ofdis_debug_div", "ofdis_debug_sor_div_fallbacks", "ofdis_upload_sequence_u8", "ofdis_set_initflow_fullres",
    "ofdis_set_initflow_from_result", "ofdis_upload_sequence_bidir_u8", "ofdis_set_swapped_slots",
    "ofdis_consistency_fullres", "ofdis_flow_error_fullres", "ofdis_debug_sor_plan",
    "ofdis_get_flow_fullres_encoded", "ofdis_flow_color_fullres", "ofdis_interpolate_fullres",
    "ofdis_track_begin", "ofdis_track_advance", "ofdis_track_stats_get", "ofdis_disparity_fullres",
    "ofdis_global_motion_fullres", "ofdis_stab_begin", "ofdis_stab_push", "ofdis_stab_finish",
    "ofdis_traj_begin", "ofdis_traj_advance", "ofdis_traj_stats_get", "ofdis_scene_flow_fullres",
    "ofdis_fisher_begin", "ofdis_fisher_push", "ofdis_fisher_take", "ofdis_traj_advance_fisher",
    "ofdis_egomotion_fullres", "ofdis_fuse_begin", "ofdis_fuse_push", "ofdis_fuse_extract", "ofdis_fuse_render",
    "ofdis_fuse_get_volume", "ofdis_fuse_set_volume", "ofdis_fuse_mesh", "ofdis_fuse_track",
    "ofdis_confidence_fullres", "ofdis_fuse_push_weighted", "ofdis_fuse_track_weighted", "ofdis_relpose_fullres",
]

# outputs of disparity_fullres, in the C-ABI's argument order
DISP_OUTPUTS = ("disp", "status", "depth", "xyz")

# outputs of scene_flow_fullres, in the C-ABI's argument order
SF_OUTPUTS = ("disp1", "status", "motion")

# per-pixel outputs of egomotion_fullres, in the C-ABI's argument order
EGO_OUTPUTS = ("mask", "residual", "object_motion")

# per-pixel outputs of relpose_fullres, in the C-ABI's argument order
RELPOSE_OUTPUTS = ("mask", "sampson", "depth")

# encodings of get_flow_fullres_encoded (OFDIS_ENC_F16, OFDIS_ENC_KITTI)
ENCODINGS = {"f16": 1, "kitti": 2}

# kind of ofdis_debug_sor_plan (SorKind)
SOR_KINDS = ("wave_single", "wave_cluster", "wave_chain", "lane", "redblack")
SOR_PLAN_FIELDS = ("kind", "hpad", "rt", "ml", "nb", "sweeps", "tail_sweeps", "assemble_rows", "assemble_mode")

# default thresholds of consistency_fullres: flow (Sundaram, Brox, Keutzer, ECCV 2010) and stereo (|d_L + d_R| <= 1)
CONSISTENCY_DEFAULTS = {2: (0.01, 0.5), 1: (0.0, 1.0)}

# ofdis_error_stats (include/ofdis_b200.h), field for field: counts of one (pair, class) of flow_error_fullres
ERROR_STATS_DTYPE = np.dtype([("n", "<i8"), ("n_over", "<i8", (3,)), ("n_outlier", "<i8"), ("sum_err", "<f8")])


class TrackParams(ctypes.Structure):
    """ofdis_track_params (include/ofdis_b200.h)."""
    _fields_ = [("capacity", ctypes.c_int), ("spacing", ctypes.c_int)] + \
        [(k, ctypes.c_float) for k in TRACK_PARAM_FIELDS[2:]]


class TrackStats(ctypes.Structure):
    """ofdis_track_stats (include/ofdis_b200.h)."""
    _fields_ = [(k, ctypes.c_longlong) for k in TRACK_STATS_FIELDS[:5]] + \
        [(k, ctypes.c_int) for k in TRACK_STATS_FIELDS[5:]]


class DispFilter(ctypes.Structure):
    """ofdis_disp_filter (include/ofdis_b200.h)."""
    _fields_ = [("lr_check", ctypes.c_int), ("alpha", ctypes.c_float), ("beta", ctypes.c_float),
                ("speckle_size", ctypes.c_int), ("speckle_diff", ctypes.c_float), ("fill", ctypes.c_int)]


class StereoCamera(ctypes.Structure):
    """ofdis_stereo_camera (include/ofdis_b200.h)."""
    _fields_ = [(k, ctypes.c_float) for k in STEREO_CAMERA_FIELDS]


assert tuple(k for k, _ in DispFilter._fields_) == DISP_FILTER_FIELDS


class SfGt(ctypes.Structure):
    """ofdis_sf_gt (include/ofdis_b200.h)."""
    _fields_ = [("disp0", ctypes.c_void_p), ("disp1", ctypes.c_void_p), ("flow", ctypes.c_void_p)]


class MotionParams(ctypes.Structure):
    """ofdis_motion_params (include/ofdis_b200.h)."""
    _fields_ = [("model", ctypes.c_int), ("step", ctypes.c_int), ("fb_check", ctypes.c_int), ("alpha", ctypes.c_float),
                ("beta", ctypes.c_float), ("hypotheses", ctypes.c_int), ("threshold", ctypes.c_float),
                ("refine", ctypes.c_int), ("seed", ctypes.c_ulonglong)]


class MotionStats(ctypes.Structure):
    """ofdis_motion_stats (include/ofdis_b200.h); MOTION_STATS_DTYPE is the same record as numpy sees it."""
    _fields_ = [(k, ctypes.c_int) for k in MOTION_STATS_DTYPE.names]


assert tuple(k for k, _ in MotionParams._fields_) == MOTION_PARAM_FIELDS
assert ctypes.sizeof(MotionStats) == MOTION_STATS_DTYPE.itemsize


class EgoParams(ctypes.Structure):
    """ofdis_egomotion_params (include/ofdis_b200.h)."""
    _fields_ = [("step", ctypes.c_int), ("fb_check", ctypes.c_int), ("alpha", ctypes.c_float),
                ("beta", ctypes.c_float), ("edge_diff", ctypes.c_float), ("hypotheses", ctypes.c_int),
                ("threshold", ctypes.c_float), ("refine", ctypes.c_int), ("seed", ctypes.c_ulonglong)]


assert tuple(k for k, _ in EgoParams._fields_) == EGO_PARAM_FIELDS


class RelposeParams(ctypes.Structure):
    """ofdis_relpose_params (include/ofdis_b200.h)."""
    _fields_ = [(k, ctypes.c_float) for k in ("fx", "fy", "cx", "cy")] + \
        [("step", ctypes.c_int), ("fb_check", ctypes.c_int), ("alpha", ctypes.c_float), ("beta", ctypes.c_float),
         ("hypotheses", ctypes.c_int), ("threshold", ctypes.c_float), ("refine", ctypes.c_int),
         ("min_parallax", ctypes.c_float), ("seed", ctypes.c_ulonglong)]


assert tuple(k for k, _ in RelposeParams._fields_) == RELPOSE_PARAM_FIELDS


class FuseParams(ctypes.Structure):
    """ofdis_fuse_params (include/ofdis_b200.h)."""
    _fields_ = [("nx", ctypes.c_int), ("ny", ctypes.c_int), ("nz", ctypes.c_int), ("origin", ctypes.c_float * 3),
                ("voxel", ctypes.c_float), ("trunc", ctypes.c_float), ("max_weight", ctypes.c_float),
                ("color", ctypes.c_int)]


assert tuple(k for k, _ in FuseParams._fields_) == FUSE_PARAM_FIELDS
assert FUSE_POINT_DTYPE.itemsize == 28


class FuseTrackParams(ctypes.Structure):
    """ofdis_fuse_track_params (include/ofdis_b200.h)."""
    _fields_ = [("step", ctypes.c_int), ("rounds", ctypes.c_int), ("min_weight", ctypes.c_float),
                ("max_depth", ctypes.c_float), ("huber", ctypes.c_float), ("damping", ctypes.c_double),
                ("min_corr", ctypes.c_int), ("max_shift", ctypes.c_double), ("min_cos", ctypes.c_double),
                ("eps", ctypes.c_double), ("integrate", ctypes.c_int)]


class ConfParams(ctypes.Structure):
    """ofdis_conf_params (include/ofdis_b200.h)."""
    _fields_ = [("radius", ctypes.c_int), ("s_fb", ctypes.c_float), ("s_tex", ctypes.c_float),
                ("min_count", ctypes.c_int)]


assert tuple(k for k, _ in ConfParams._fields_) == CONF_PARAM_FIELDS


class FuseTrackStats(ctypes.Structure):
    """ofdis_fuse_track_stats (include/ofdis_b200.h); FUSE_TRACK_STATS_DTYPE is the same record as numpy sees it."""
    _fields_ = [("status", ctypes.c_int), ("n_corr", ctypes.c_int), ("rounds", ctypes.c_int),
                ("cost0", ctypes.c_double), ("cost", ctypes.c_double)]


assert tuple(k for k, _ in FuseTrackParams._fields_) == FUSE_TRACK_PARAM_FIELDS
assert ctypes.sizeof(FuseTrackStats) == FUSE_TRACK_STATS_DTYPE.itemsize == 32


class StabParams(ctypes.Structure):
    """ofdis_stab_params (include/ofdis_b200.h)."""
    _fields_ = [("radius", ctypes.c_int), ("crop", ctypes.c_float), ("limit", ctypes.c_int)]


class StabFrame(ctypes.Structure):
    """ofdis_stab_frame (include/ofdis_b200.h); STAB_FRAME_DTYPE is the same record as numpy sees it."""
    _fields_ = [("frame", ctypes.c_longlong), ("status", ctypes.c_int), ("lambda", ctypes.c_double),
                ("correction", ctypes.c_double * 9)]


assert tuple(k for k, _ in StabParams._fields_) == STAB_PARAM_FIELDS
assert ctypes.sizeof(StabFrame) == STAB_FRAME_DTYPE.itemsize


class TrajParams(ctypes.Structure):
    """ofdis_traj_params (include/ofdis_b200.h)."""
    _fields_ = [(k, ctypes.c_int) for k in TRAJ_PARAM_FIELDS[:4]] + [(k, ctypes.c_float) for k in TRAJ_PARAM_FIELDS[4:]]


class TrajStats(ctypes.Structure):
    """ofdis_traj_stats (include/ofdis_b200.h)."""
    _fields_ = [(k, ctypes.c_longlong) for k in TRAJ_STATS_FIELDS]


class FisherBlock(ctypes.Structure):
    """ofdis_fisher_block (include/ofdis_b200.h)."""
    _fields_ = [("offset", ctypes.c_int), ("dim_in", ctypes.c_int), ("dim", ctypes.c_int)]


class FisherCodebook(ctypes.Structure):
    """ofdis_fisher_codebook (include/ofdis_b200.h); params points at a packed float32 body the caller keeps alive."""
    _fields_ = [("K", ctypes.c_int), ("desc_dim", ctypes.c_int), ("nblocks", ctypes.c_int),
                ("blocks", FisherBlock * FISHER_MAX_BLOCKS), ("params", ctypes.c_void_p)]


class FisherStats(ctypes.Structure):
    """ofdis_fisher_stats (include/ofdis_b200.h); FISHER_STATS_DTYPE is the same record as numpy sees it."""
    _fields_ = [("pushed", ctypes.c_longlong), ("n", ctypes.c_longlong * FISHER_MAX_BLOCKS),
                ("skipped", ctypes.c_longlong * FISHER_MAX_BLOCKS)]


assert ctypes.sizeof(FisherStats) == FISHER_STATS_DTYPE.itemsize


class OfdisError(RuntimeError):
    pass


_lib = None


def lib():
    """Loads the CUDA library; raises loudly when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise OfdisError("%s not found: run `python -m of_dis_b200.build` (no CPU fallback exists)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        L.ofdis_last_error.restype = ctypes.c_char_p
        L.ofdis_version.restype = ctypes.c_char_p
        L.ofdis_packed_frame_floats.restype = ctypes.c_size_t
        L.ofdis_packed_images_frame_floats.restype = ctypes.c_size_t
        L.ofdis_packed_offset.restype = ctypes.c_size_t
        L.ofdis_debug_get.restype = ctypes.c_long
        L.ofdis_launch_count.restype = ctypes.c_long
        L.ofdis_create.argtypes = [ctypes.POINTER(ctypes.c_void_p), ctypes.c_int, ctypes.c_void_p,
                                   ctypes.POINTER(CParams), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_int]
        for name in ("ofdis_destroy", "ofdis_sync"):
            getattr(L, name).argtypes = [ctypes.c_void_p]
        L.ofdis_last_error.argtypes = [ctypes.c_void_p]
        L.ofdis_launch_count.argtypes = [ctypes.c_void_p]
        L.ofdis_packed_frame_floats.argtypes = [ctypes.c_void_p]
        L.ofdis_packed_images_frame_floats.argtypes = [ctypes.c_void_p]
        L.ofdis_upload_packed_images.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_packed_offset.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.ofdis_get_level.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_finest_level_frame_floats.restype = ctypes.c_size_t
        L.ofdis_finest_level_frame_floats.argtypes = [ctypes.c_void_p]
        L.ofdis_upload_finest_level.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_upload_frames_u8.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int]
        L.ofdis_upload_sequence_u8.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                               ctypes.c_int, ctypes.c_int]
        L.ofdis_upload_sequence_bidir_u8.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                     ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ofdis_set_swapped_slots.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3
        L.ofdis_consistency_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + \
            [ctypes.c_float] * 2 + [ctypes.c_int] * 3
        L.ofdis_flow_error_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 2 + \
            [ctypes.c_int] + [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3
        L.ofdis_get_flow_fullres.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int]
        L.ofdis_get_flow_fullres_encoded.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] + \
            [ctypes.c_int] * 3
        L.ofdis_flow_color_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 2 + \
            [ctypes.c_float] + [ctypes.c_int] * 3
        L.ofdis_interpolate_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + \
            [ctypes.c_size_t] + [ctypes.c_float] * 3 + [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3
        L.ofdis_track_begin.argtypes = [ctypes.c_void_p, ctypes.POINTER(TrackParams)] + [ctypes.c_void_p] * 3 + \
            [ctypes.c_int] * 3
        L.ofdis_track_advance.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3
        L.ofdis_disparity_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.POINTER(DispFilter), ctypes.POINTER(StereoCamera)] + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3
        L.ofdis_scene_flow_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 2 + [ctypes.c_void_p] * 2 + \
            [ctypes.c_size_t, ctypes.c_float, ctypes.POINTER(StereoCamera)] + [ctypes.c_void_p] * 3 + \
            [ctypes.POINTER(SfGt), ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p] + [ctypes.c_int] * 3
        L.ofdis_global_motion_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.POINTER(MotionParams), ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 5 + [ctypes.c_int] * 3
        L.ofdis_egomotion_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.POINTER(EgoParams)] + [ctypes.c_void_p] * 2 + [ctypes.c_size_t, ctypes.POINTER(StereoCamera)] + \
            [ctypes.c_void_p] * 5 + [ctypes.c_int] * 3
        L.ofdis_relpose_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.POINTER(RelposeParams)] + [ctypes.c_void_p] * 5 + [ctypes.c_int] * 3
        L.ofdis_track_stats_get.argtypes = [ctypes.c_void_p, ctypes.POINTER(TrackStats)]
        L.ofdis_traj_begin.argtypes = [ctypes.c_void_p, ctypes.POINTER(TrackParams), ctypes.POINTER(TrajParams)] + \
            [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3
        L.ofdis_traj_advance.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_void_p] * 6 + [ctypes.c_int] * 3
        L.ofdis_traj_stats_get.argtypes = [ctypes.c_void_p, ctypes.POINTER(TrajStats)]
        L.ofdis_stab_begin.argtypes = [ctypes.c_void_p, ctypes.POINTER(StabParams)] + [ctypes.c_void_p] * 2 + \
            [ctypes.c_int] * 3
        L.ofdis_stab_push.argtypes = [ctypes.c_void_p, ctypes.c_int] + [ctypes.c_void_p] * 2 + [ctypes.c_size_t] + \
            [ctypes.c_void_p] * 3 + [ctypes.c_int]
        L.ofdis_stab_finish.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_int]
        L.ofdis_fisher_begin.argtypes = [ctypes.c_void_p, ctypes.POINTER(FisherCodebook)]
        L.ofdis_fisher_push.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long, ctypes.c_int]
        L.ofdis_fisher_take.argtypes = [ctypes.c_void_p] + [ctypes.c_void_p] * 3 + [ctypes.c_int]
        L.ofdis_traj_advance_fisher.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3
        L.ofdis_fuse_begin.argtypes = [ctypes.c_void_p, ctypes.POINTER(FuseParams)]
        L.ofdis_fuse_push.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p,
                                      ctypes.POINTER(StereoCamera), ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_int] * 3
        L.ofdis_fuse_extract.argtypes = [ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_long,
                                         ctypes.POINTER(ctypes.c_long), ctypes.c_int]
        L.ofdis_fuse_render.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.POINTER(StereoCamera)] + \
            [ctypes.c_float] * 4 + [ctypes.c_void_p] + [ctypes.c_int] * 3
        L.ofdis_fuse_get_volume.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int]
        L.ofdis_fuse_set_volume.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int]
        L.ofdis_fuse_mesh.argtypes = [ctypes.c_void_p, ctypes.c_float] + \
            [ctypes.c_void_p, ctypes.c_long, ctypes.POINTER(ctypes.c_long)] * 2 + [ctypes.c_int]
        L.ofdis_fuse_track.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_void_p] * 2 + [ctypes.POINTER(StereoCamera), ctypes.POINTER(FuseTrackParams), ctypes.c_void_p,
                                     ctypes.c_size_t] + [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3
        L.ofdis_fuse_track_weighted.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t] + \
            [ctypes.c_void_p] * 2 + [ctypes.POINTER(StereoCamera), ctypes.POINTER(FuseTrackParams)] + \
            [ctypes.c_void_p, ctypes.c_size_t] * 2 + [ctypes.c_void_p] * 2 + [ctypes.c_int] * 3
        L.ofdis_fuse_push_weighted.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t,
                                               ctypes.c_void_p, ctypes.POINTER(StereoCamera), ctypes.c_float] + \
            [ctypes.c_void_p, ctypes.c_size_t] * 2 + [ctypes.c_int] * 3
        L.ofdis_confidence_fullres.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + \
            [ctypes.POINTER(ConfParams), ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t] + [ctypes.c_void_p] * 2 + \
            [ctypes.c_int] * 3
        L.ofdis_set_initflow_fullres.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                                 ctypes.c_int, ctypes.c_int, ctypes.c_int]
        L.ofdis_set_initflow_from_result.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 5
        L.ofdis_upload_packed.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_upload_level.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 4 + [ctypes.c_int]
        L.ofdis_upload_level_fb.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_int]
        L.ofdis_level_info.argtypes = [ctypes.c_void_p, ctypes.c_int] + [_IP] * 5
        L.ofdis_patgrid_optimize.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 4
        L.ofdis_patgrid_aggregate.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3
        L.ofdis_varref_refine.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3
        L.ofdis_debug_varref_iters.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 4
        L.ofdis_debug_div.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_long] + [ctypes.c_void_p] * 3
        L.ofdis_debug_sor_div_fallbacks.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_ulonglong), ctypes.c_int]
        L.ofdis_debug_sor_plan.argtypes = [ctypes.c_int] * 11 + [_IP]
        L.ofdis_run.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int]
        L.ofdis_get_flow.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_set_flow.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_get_flow_batch.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int]
        L.ofdis_get_patches.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 4
        L.ofdis_debug_get.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t]
        L.ofdis_set_graph_mode.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.ofdis_set_option.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
        L.ofdis_set_direction.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.ofdis_set_camlr.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.ofdis_set_dp_thresh_sq.argtypes = [ctypes.c_void_p, ctypes.c_float]
        L.ofdis_profile_run.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
        L.ofdis_profile_levels.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
        _lib = L
    return _lib


def debug_sor_plan(w, h, nop, noc, solverit, frames, lane=2, fast=0, rt=1, single_max=128, max_cluster=8):
    """The refinement's launch plan of a w x h level for `frames` internal frames per launch (ofdis_debug_sor_plan;
    no device needed): a dict of SOR_PLAN_FIELDS, kind named by SOR_KINDS, or None where no plan exists."""
    out = (ctypes.c_int * len(SOR_PLAN_FIELDS))()
    rc = lib().ofdis_debug_sor_plan(w, h, nop, noc, solverit, frames, lane, fast, rt, single_max, max_cluster, out)
    if rc == -3:
        return None
    if rc != 0:
        raise OfdisError("debug_sor_plan: status %d" % rc)
    d = dict(zip(SOR_PLAN_FIELDS, list(out)))
    d["kind"] = SOR_KINDS[d["kind"]]
    return d


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data_as(ctypes.c_void_p)
    return ctypes.c_void_p(int(a))  # raw address (e.g. torch tensor .data_ptr())


class Context:
    """One device, one stream, frames [0, max_frames) per launch."""

    def __init__(self, prm: DisParams, width: int, height: int, imgpadding: int | None = None, max_frames: int = 1,
                 device: int = 0, stream: int | None = None):
        self.prm = prm
        self.width, self.height = width, height
        self.pad = prm.p_samp_s if imgpadding is None else imgpadding
        self.max_frames = max_frames
        self._h = ctypes.c_void_p()
        cp = prm.to_c()
        rc = lib().ofdis_create(ctypes.byref(self._h), device, ctypes.c_void_p(stream or 0), ctypes.byref(cp), prm.nop,
                                width, height, self.pad, max_frames)
        if rc != 0:
            self._h = ctypes.c_void_p()
            raise OfdisError("ofdis_create failed with status %d" % rc)

    # -- lifetime ---------------------------------------------------------
    def close(self):
        if self._h:
            lib().ofdis_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise OfdisError("status %d: %s" % (rc, lib().ofdis_last_error(self._h).decode()))

    # -- geometry ----------------------------------------------------------
    def level_info(self, level: int):
        v = [ctypes.c_int() for _ in range(5)]
        self._ck(lib().ofdis_level_info(self._h, level, *[ctypes.byref(x) for x in v]))
        return dict(zip(("w", "h", "nopw", "noph", "steps"), [x.value for x in v]))

    @property
    def packed_frame_floats(self) -> int:
        return lib().ofdis_packed_frame_floats(self._h)

    def packed_offset(self, level: int, which: int) -> int:
        return lib().ofdis_packed_offset(self._h, level, which)

    def pack_frame(self, pyr, out: np.ndarray | None = None) -> np.ndarray:
        """Lays one PairPyramids out in the context's packed transfer format."""
        buf = np.zeros(self.packed_frame_floats, np.float32) if out is None else out
        for lv in range(self.prm.sc_l, self.prm.sc_f + 1):
            for k, arr in enumerate((pyr.i0[lv], pyr.i0x[lv], pyr.i0y[lv], pyr.i1[lv])):
                o = self.packed_offset(lv, k)
                buf[o:o + arr.size] = arr.reshape(-1)
        return buf

    # -- transfers ----------------------------------------------------------
    def upload_level(self, frame, level, i0, i0x, i0y, i1, memkind=MEM_HOST):
        self._ck(lib().ofdis_upload_level(self._h, frame, level, _ptr(i0), _ptr(i0x), _ptr(i0y), _ptr(i1), memkind))

    def upload_level_fb(self, frame, level, i0, i0x, i0y, i1, i1x, i1y, memkind=MEM_HOST):
        """All six arrays of OFClass (oflow.h:84-86); the last two are only used with usefbcon."""
        self._ck(lib().ofdis_upload_level_fb(self._h, frame, level, _ptr(i0), _ptr(i0x), _ptr(i0y), _ptr(i1), _ptr(i1x),
                                             _ptr(i1y), memkind))

    def upload_pyramids(self, frame: int, pyr):
        for lv in range(self.prm.sc_l, self.prm.sc_f + 1):
            if self.prm.usefbcon:
                self.upload_level_fb(frame, lv, pyr.i0[lv], pyr.i0x[lv], pyr.i0y[lv], pyr.i1[lv], pyr.i1x[lv], pyr.i1y[lv])
            else:
                self.upload_level(frame, lv, pyr.i0[lv], pyr.i0x[lv], pyr.i0y[lv], pyr.i1[lv])

    @property
    def packed_images_frame_floats(self) -> int:
        return lib().ofdis_packed_images_frame_floats(self._h)

    def upload_packed_images(self, f0, f1, packed, memkind=MEM_HOST):
        """I0,I1 only (the leading part of the packed layout); gradients are derived on the device."""
        self._ck(lib().ofdis_upload_packed_images(self._h, f0, f1, _ptr(packed), memkind))

    def get_level(self, frame, level, which) -> np.ndarray:
        """Padded device array `which` (0 I0, 1 I0x, 2 I0y, 3 I1) of one level."""
        h, w = (self.height >> level) + 2 * self.pad, (self.width >> level) + 2 * self.pad
        out = np.empty((h, w) if self.prm.noc == 1 else (h, w, self.prm.noc), np.float32)
        self._ck(lib().ofdis_get_level(self._h, frame, level, which, _ptr(out), MEM_HOST))
        return out

    @property
    def finest_level_frame_floats(self) -> int:
        return lib().ofdis_finest_level_frame_floats(self._h)

    def upload_finest_level(self, f0, f1, packed, memkind=MEM_HOST):
        """[frame][2][h][w][noc] un-padded float images of level sc_l; the rest is derived on the device."""
        self._ck(lib().ofdis_upload_finest_level(self._h, f0, f1, _ptr(packed), memkind))

    def upload_frames_u8(self, f0, f1, frames, width_org, height_org, memkind=MEM_HOST):
        """[frame][2][height_org][width_org][noc] 8-bit pairs; whole pyramid built on the device."""
        self._ck(lib().ofdis_upload_frames_u8(self._h, f0, f1, _ptr(frames), width_org, height_org, memkind))

    def upload_sequence_u8(self, f0, f1, frames, width_org, height_org, memkind=MEM_HOST):
        """[f1-f0+1][height_org][width_org][noc] 8-bit consecutive frames; pair f0+i = (frames[i], frames[i+1]).
        Bitwise the pyramids upload_frames_u8 builds from the duplicated pairs, each frame uploaded once."""
        self._ck(lib().ofdis_upload_sequence_u8(self._h, f0, f1, _ptr(frames), width_org, height_org, memkind))

    def upload_sequence_bidir_u8(self, f0, n, frames, width_org, height_org, memkind=MEM_HOST):
        """[n+1][height_org][width_org][noc] 8-bit consecutive frames -> slot f0+t = (frames[t], frames[t+1]) and
        slot f0+n+t = (frames[t+1], frames[t]), the latter marked swapped (set_swapped_slots).  Bitwise the pyramids
        upload_frames_u8 builds from the forward and the swapped pairs, each frame uploaded once."""
        self._ck(lib().ofdis_upload_sequence_bidir_u8(self._h, f0, n, _ptr(frames), width_org, height_org, memkind))

    def set_swapped_slots(self, f0, f1, swapped):
        """Stereo: slots [f0, f1) hold (right, left) pairs and run as the right camera (camlr inverted)."""
        self._ck(lib().ofdis_set_swapped_slots(self._h, f0, f1, int(swapped)))

    def consistency_fullres(self, f0, f1, b0, width_org, height_org, alpha=None, beta=None, with_err=False,
                            memkind=MEM_HOST, mask=None, err=None):
        """Forward-backward (flow) / left-right (stereo) check of the last run's slots [f0, f1) against slots
        [b0, b0 + f1 - f0) at the original frame size (preprocess.consistency_check on the device).  Returns
        (mask, err): [f1-f0][height_org][width_org] uint8 (0 consistent, 1 inconsistent, 2 leaves the frame) and
        float32, err None unless with_err.  alpha/beta None: CONSISTENCY_DEFAULTS of the context's nop.  Host output
        goes to new arrays, or to `mask` / `err` given as numpy arrays of exactly that shape and dtype.  With
        memkind=MEM_DEVICE, mask (and err) are device addresses the caller owns."""
        da, db = CONSISTENCY_DEFAULTS[self.prm.nop]
        alpha = da if alpha is None else alpha
        beta = db if beta is None else beta
        shape = (f1 - f0, height_org, width_org)
        if memkind == MEM_HOST:
            mask = np.empty(shape, np.uint8) if mask is None else mask
            err = (np.empty(shape, np.float32) if err is None else err) if with_err else None
            for name, arr, dt in (("mask", mask, np.uint8), ("err", err, np.float32)):
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shape
                                            and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("consistency_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shape))
        self._ck(lib().ofdis_consistency_fullres(self._h, f0, f1, b0, _ptr(mask), _ptr(err), alpha, beta, width_org,
                                                 height_org, memkind))
        if memkind == MEM_HOST:
            self.sync()
        return mask, err

    def confidence_fullres(self, f0, f1, b0, frames0, frames1, params, width_org, height_org, with_conf=True,
                           with_terms=False, memkind=MEM_HOST, conf=None, terms=None, frame_stride=None):
        """Per-pixel confidence of the last run's slots [f0, f1) (ofdis_confidence_fullres; preprocess.confidence
        restates it), with the forward-backward term against slots [b0, b0 + f1 - f0), or without it for b0 < 0.
        params: a mapping with preprocess.CONF_PARAM_FIELDS or a ConfParams.  Returns (conf, terms): [f1-f0][H][W]
        and [f1-f0][H][W][3] (z, e, lambda) float32, each None unless asked for.  Host: frames0 and frames1 as
        interpolate_fullres takes them (frames[:-1] / frames[1:] of a clip qualify), outputs new or given as numpy
        arrays of exactly that shape; the call synchronises the stream.  With memkind=MEM_DEVICE frames0, frames1,
        conf and terms are device addresses (conf or terms may be None) and frame_stride the bytes between frames
        (default one frame)."""
        if not isinstance(params, ConfParams):
            params = ConfParams(int(params["radius"]), float(params["s_fb"]), float(params["s_tex"]),
                                int(params["min_count"]))
        n = max(f1 - f0, 0)
        hwc = height_org * width_org * self.prm.noc
        if memkind == MEM_HOST:
            strides = [self._frames_u8("confidence_fullres: %s" % name, arr, n, width_org, height_org)
                       for name, arr in (("frames0", frames0), ("frames1", frames1))]
            if strides[0] != strides[1]:
                raise ValueError("confidence_fullres: frames0 and frames1 must have the same strides[0]")
            frame_stride = strides[0]
            frames0, frames1 = frames0.ctypes.data, frames1.ctypes.data
            shapes = {"conf": (n, height_org, width_org), "terms": (n, height_org, width_org, 3)}
            conf = (np.empty(shapes["conf"], np.float32) if conf is None else conf) if with_conf else None
            terms = (np.empty(shapes["terms"], np.float32) if terms is None else terms) if with_terms else None
            for name, arr in (("conf", conf), ("terms", terms)):
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == np.float32 and
                                            arr.shape == shapes[name] and arr.flags["C_CONTIGUOUS"] and
                                            arr.flags["WRITEABLE"]):
                    raise ValueError("confidence_fullres: %s must be a writeable C-contiguous float32 array of shape %s"
                                     % (name, shapes[name]))
        else:
            frame_stride = hwc if frame_stride is None else frame_stride
        self._ck(lib().ofdis_confidence_fullres(self._h, f0, f1, b0, ctypes.byref(params), _ptr(frames0),
                                                _ptr(frames1), frame_stride, _ptr(conf), _ptr(terms), width_org,
                                                height_org, memkind))
        return conf, terms

    def disparity_fullres(self, f0, f1, b0, width_org, height_org, lr_check=0, alpha=0.0, beta=1.0, speckle_size=0,
                          speckle_diff=1.0, fill=0, camera=None, outputs=("disp", "status"), memkind=MEM_HOST,
                          out=None):
        """Filtered disparities of the last run's stereo slots [f0, f1), left-right checked against slots
        [b0, b0 + f1 - f0) with lr_check, and from them depth and xyz with a camera (ofdis_disparity_fullres;
        preprocess.disparity_filter restates it).  camera: None or a mapping with STEREO_CAMERA_FIELDS (required for
        "depth" and "xyz").  Returns a dict of the requested DISP_OUTPUTS.  Host: "disp" and "depth" (f1-f0,
        height_org, width_org) float32, "status" the same in uint8, "xyz" (f1-f0, height_org, width_org, 3) float32,
        new or given in `out` as numpy arrays of exactly that dtype and shape; the call synchronises the stream.
        With memkind=MEM_DEVICE, `out` maps the requested outputs to device addresses the caller owns, and the
        call is enqueued on the context's stream."""
        unknown = set(outputs) - set(DISP_OUTPUTS)
        if unknown:
            raise ValueError("disparity_fullres: unknown outputs %s" % sorted(unknown))
        out = dict(out or {})
        if memkind == MEM_HOST:
            n = max(f1 - f0, 0)
            for name in outputs:
                shape = (n, height_org, width_org) + ((3,) if name == "xyz" else ())
                dt = np.uint8 if name == "status" else np.float32
                arr = out.setdefault(name, np.empty(shape, dt))
                if not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shape
                        and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("disparity_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shape))
        else:
            missing = [name for name in outputs if out.get(name) is None]
            if missing:
                raise ValueError("disparity_fullres: no device address for the requested outputs %s" % missing)
        filt = DispFilter(int(lr_check), alpha, beta, int(speckle_size), speckle_diff, int(fill))
        cam = None if camera is None else ctypes.byref(StereoCamera(*[camera[k] for k in STEREO_CAMERA_FIELDS]))
        ptrs = [_ptr(out.get(k)) if k in outputs else None for k in DISP_OUTPUTS]
        self._ck(lib().ofdis_disparity_fullres(self._h, f0, f1, b0, ctypes.byref(filt), cam, *ptrs, width_org,
                                               height_org, memkind))
        return {k: out.get(k) for k in outputs}

    def scene_flow_fullres(self, f0, f1, disp0, disp1, *, width_org, height_org, edge_diff=1.0, camera=None,
                           outputs=("disp1", "status"), gt=None, classes=None, nclasses=None, memkind=MEM_HOST,
                           out=None, disp_stride=None):
        """Scene flow of the last run's flow slots [f0, f1) (ofdis_scene_flow_fullres; preprocess.scene_flow restates
        it): pair k's flow F with the disparities disp0[k] at t and disp1[k] at t+1 (positive, NaN unknown) gives
        "disp1" (the t+1 disparity warped to frame t), "status" and, with a camera (a mapping with
        STEREO_CAMERA_FIELDS), "motion" (the 3-D motion).  gt: None or (disp0, disp1, flow) ground truth, with classes
        and nclasses as flow_error_fullres takes them.  Returns (outs, stats): a dict of the requested SF_OUTPUTS and,
        with gt, a (f1-f0, nclasses) array of SF_STATS_DTYPE (else None), always on the host.
        Host: disp0 and disp1 float32 (f1-f0, height_org, width_org) arrays whose frames are C-contiguous and equally
        spaced (a clip's maps[:-1] and maps[1:] qualify); gt and classes C-contiguous float32 / uint8 arrays; the
        outputs new or given in `out` as numpy arrays of exactly their dtype and shape ("motion" has a last axis of 3);
        the call synchronises the stream.  With memkind=MEM_DEVICE every array is a device address the caller owns,
        disp_stride the floats between consecutive maps (default one frame), and the call only synchronises for
        stats."""
        unknown = set(outputs) - set(SF_OUTPUTS)
        if unknown:
            raise ValueError("scene_flow_fullres: unknown outputs %s" % sorted(unknown))
        if nclasses is None:
            if classes is not None:
                raise ValueError("scene_flow_fullres: nclasses is required with classes")
            nclasses = 1
        n = max(f1 - f0, 0)
        shape = (n, height_org, width_org)
        out = dict(out or {})
        if gt is not None:
            gt = tuple(gt)
            if len(gt) != 3:
                raise ValueError("scene_flow_fullres: gt is (disp0, disp1, flow)")
        if memkind == MEM_HOST:
            strides = []
            for name, arr in (("disp0", disp0), ("disp1", disp1)):
                if not (isinstance(arr, np.ndarray) and arr.dtype == np.float32 and arr.shape == shape
                        and (n == 0 or arr[0].flags["C_CONTIGUOUS"])):
                    raise ValueError("scene_flow_fullres: %s must be a float32 array of shape %s whose frames are "
                                     "C-contiguous" % (name, shape))
                strides.append(arr.strides[0] // 4 if n > 1 else height_org * width_org)
            if strides[0] != strides[1] or (n > 1 and disp0.strides[0] % 4):
                raise ValueError("scene_flow_fullres: disp0 and disp1 must space their frames equally")
            disp_stride = strides[0]
            inputs = (("classes", classes, np.uint8, shape),)
            if gt is not None:
                inputs += (("gt disp0", gt[0], np.float32, shape), ("gt disp1", gt[1], np.float32, shape),
                           ("gt flow", gt[2], np.float32, shape + (2,)))
            for name, arr, dt, shp in inputs:
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shp
                                            and arr.flags["C_CONTIGUOUS"]):
                    raise ValueError("scene_flow_fullres: %s must be a C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shp))
            for name in outputs:
                shp = shape + ((3,) if name == "motion" else ())
                dt = np.uint8 if name == "status" else np.float32
                arr = out.setdefault(name, np.empty(shp, dt))
                if not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shp
                        and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("scene_flow_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shp))
        else:
            missing = [name for name in outputs if out.get(name) is None]
            if missing:
                raise ValueError("scene_flow_fullres: no device address for the requested outputs %s" % missing)
            if disp_stride is None:
                disp_stride = height_org * width_org
        cam = None if camera is None else ctypes.byref(StereoCamera(*[camera[k] for k in STEREO_CAMERA_FIELDS]))
        gts = None if gt is None else ctypes.byref(SfGt(*[_ptr(a) for a in gt]))
        stats = None if gt is None else np.zeros((n, max(nclasses, 0)), SF_STATS_DTYPE)
        ptrs = [_ptr(out.get(k)) if k in outputs else None for k in SF_OUTPUTS]
        self._ck(lib().ofdis_scene_flow_fullres(self._h, f0, f1, _ptr(disp0), _ptr(disp1), disp_stride, edge_diff, cam,
                                                *ptrs, gts, _ptr(classes), nclasses, _ptr(stats), width_org,
                                                height_org, memkind))
        return {k: out.get(k) for k in outputs}, stats

    def global_motion_fullres(self, f0, f1, params, *, width_org, height_org, b0=None, i1=None, frame_stride=None,
                              mask=None, residual=None, registered=None, memkind=MEM_HOST):
        """The camera motion of the last run's slots [f0, f1): one RANSAC model per pair, refitted on its inliers, and
        optionally the per-pixel residual flows, moving-pixel masks and registered I1 (ofdis_global_motion_fullres;
        preprocess.global_motion restates it).  params: a mapping with preprocess.MOTION_PARAM_FIELDS (the model as a
        number or a name of preprocess.MOTION_MODELS) or a MotionParams; b0: the partner slots of fb_check.  Returns
        (models, stats): (f1-f0, 3, 3) float64 and (f1-f0,) of MOTION_STATS_DTYPE, always on the host; the call
        synchronises the stream.  Host: mask (f1-f0, height_org, width_org) uint8, residual (..., 2) float32 and
        registered (f1-f0, height_org, width_org[, noc]) uint8 are writeable C-contiguous numpy arrays to fill (None
        skips them); i1 the pairs' I1, a uint8 (f1-f0, height_org, width_org[, noc]) array whose frames are
        C-contiguous -- clip[1:] or pairs[:, 1] qualify.  With memkind=MEM_DEVICE they are device addresses the
        caller owns and frame_stride the bytes between the frames of i1 (default one frame)."""
        if not isinstance(params, MotionParams):
            p = motion_params(params)
            params = MotionParams(*[p[k] for k in MOTION_PARAM_FIELDS])
        n = max(f1 - f0, 0)
        noc = self.prm.noc
        frame = (height_org, width_org) + ((noc,) if noc > 1 else ())
        if memkind == MEM_HOST:
            for name, arr, dt, shapes in (("mask", mask, np.uint8, ((n, height_org, width_org),)),
                                          ("residual", residual, np.float32, ((n, height_org, width_org, 2),)),
                                          ("registered", registered, np.uint8,
                                           ((n,) + frame, (n, height_org, width_org, noc)))):
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape in shapes
                                            and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("global_motion_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shapes[0]))
            if i1 is not None:
                frame_stride = self._frames_u8("global_motion_fullres: i1", i1, n, width_org, height_org)
                i1 = i1.ctypes.data
        if frame_stride is None:
            frame_stride = height_org * width_org * noc
        models = np.empty((n, 3, 3), np.float64)
        stats = np.zeros(n, MOTION_STATS_DTYPE)
        self._ck(lib().ofdis_global_motion_fullres(self._h, f0, f1, -1 if b0 is None else b0, ctypes.byref(params),
                                                   _ptr(i1), frame_stride, _ptr(models), _ptr(stats), _ptr(mask),
                                                   _ptr(residual), _ptr(registered), width_org, height_org, memkind))
        return models, stats

    def egomotion_fullres(self, f0, f1, disp0, disp1, params, *, camera, width_org, height_org, b0=None,
                          disp_stride=None, outputs=(), out=None, memkind=MEM_HOST):
        """The stereo ego-motion of the last run's flow slots [f0, f1) (ofdis_egomotion_fullres;
        preprocess.egomotion restates it): pair k's flow with the disparities disp0[k] at t and disp1[k] at t+1
        (positive, NaN unknown) and the stereo camera (a mapping with STEREO_CAMERA_FIELDS) give one rigid pose per
        pair, camera t to camera t+1.  params: a mapping with preprocess.EGO_PARAM_FIELDS or an EgoParams; b0: the
        partner slots of fb_check.  outputs: any of EGO_OUTPUTS ("mask" uint8 (n, H, W), "residual" float32
        (n, H, W, 2), "object_motion" float32 (n, H, W, 3)).  Returns (pose (n, 3, 4) float64, stats (n,) of
        MOTION_STATS_DTYPE, outs), pose and stats always on the host; the call synchronises the stream.  Host: disp0
        and disp1 float32 (n, H, W) arrays whose frames are C-contiguous and equally spaced (a clip's maps[:-1] and
        maps[1:] qualify); the outputs new or given in `out` as numpy arrays of exactly their dtype and shape.  With
        memkind=MEM_DEVICE every array is a device address the caller owns and disp_stride the floats between
        consecutive maps (default one frame)."""
        unknown = set(outputs) - set(EGO_OUTPUTS)
        if unknown:
            raise ValueError("egomotion_fullres: unknown outputs %s" % sorted(unknown))
        if not isinstance(params, EgoParams):
            params = EgoParams(*[params[k] for k in EGO_PARAM_FIELDS])
        n = max(f1 - f0, 0)
        shape = (n, height_org, width_org)
        out = dict(out or {})
        if memkind == MEM_HOST:
            strides = []
            for name, arr in (("disp0", disp0), ("disp1", disp1)):
                if not (isinstance(arr, np.ndarray) and arr.dtype == np.float32 and arr.shape == shape
                        and (n == 0 or arr[0].flags["C_CONTIGUOUS"])):
                    raise ValueError("egomotion_fullres: %s must be a float32 array of shape %s whose frames are "
                                     "C-contiguous" % (name, shape))
                strides.append(arr.strides[0] // 4 if n > 1 else height_org * width_org)
            if strides[0] != strides[1] or (n > 1 and disp0.strides[0] % 4):
                raise ValueError("egomotion_fullres: disp0 and disp1 must space their frames equally")
            disp_stride = strides[0]
            for name in outputs:
                shp = shape + {"mask": (), "residual": (2,), "object_motion": (3,)}[name]
                dt = np.uint8 if name == "mask" else np.float32
                arr = out.setdefault(name, np.empty(shp, dt))
                if not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shp
                        and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("egomotion_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shp))
        else:
            missing = [name for name in outputs if out.get(name) is None]
            if missing:
                raise ValueError("egomotion_fullres: no device address for the requested outputs %s" % missing)
            if disp_stride is None:
                disp_stride = height_org * width_org
        cam = None if camera is None else ctypes.byref(StereoCamera(*[camera[k] for k in STEREO_CAMERA_FIELDS]))
        pose = np.empty((n, 3, 4), np.float64)
        stats = np.zeros(n, MOTION_STATS_DTYPE)
        ptrs = [_ptr(out.get(k)) if k in outputs else None for k in EGO_OUTPUTS]
        self._ck(lib().ofdis_egomotion_fullres(self._h, f0, f1, -1 if b0 is None else b0, ctypes.byref(params),
                                               _ptr(disp0), _ptr(disp1), disp_stride, cam, _ptr(pose), _ptr(stats),
                                               *ptrs, width_org, height_org, memkind))
        return pose, stats, {k: out.get(k) for k in outputs}

    def relpose_fullres(self, f0, f1, params, *, width_org, height_org, b0=None, outputs=(), out=None,
                        memkind=MEM_HOST):
        """The monocular relative pose of the last run's flow slots [f0, f1) (ofdis_relpose_fullres; preprocess.relpose
        restates it): one essential-matrix fit per pair with one calibrated camera, camera t to camera t+1 with a unit
        translation.  params: a mapping with preprocess.RELPOSE_PARAM_FIELDS or a RelposeParams; b0: the partner slots
        of fb_check.  outputs: any of RELPOSE_OUTPUTS ("mask" uint8, "sampson" and "depth" float32, each (n, H, W)).
        Returns (pose (n, 3, 4) float64, stats (n,) of MOTION_STATS_DTYPE, outs), pose and stats always on the host;
        the call synchronises the stream.  Host: the outputs new or given in `out` as numpy arrays of exactly their
        dtype and shape.  With memkind=MEM_DEVICE every output is a device address the caller owns."""
        unknown = set(outputs) - set(RELPOSE_OUTPUTS)
        if unknown:
            raise ValueError("relpose_fullres: unknown outputs %s" % sorted(unknown))
        if not isinstance(params, RelposeParams):
            params = RelposeParams(*[params[k] for k in RELPOSE_PARAM_FIELDS])
        n = max(f1 - f0, 0)
        shape = (n, height_org, width_org)
        out = dict(out or {})
        if memkind == MEM_HOST:
            for name in outputs:
                dt = np.uint8 if name == "mask" else np.float32
                arr = out.setdefault(name, np.empty(shape, dt))
                if not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shape
                        and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("relpose_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shape))
        else:
            missing = [name for name in outputs if out.get(name) is None]
            if missing:
                raise ValueError("relpose_fullres: no device address for the requested outputs %s" % missing)
        pose = np.empty((n, 3, 4), np.float64)
        stats = np.zeros(n, MOTION_STATS_DTYPE)
        ptrs = [_ptr(out.get(k)) if k in outputs else None for k in RELPOSE_OUTPUTS]
        self._ck(lib().ofdis_relpose_fullres(self._h, f0, f1, -1 if b0 is None else b0, ctypes.byref(params),
                                             _ptr(pose), _ptr(stats), *ptrs, width_org, height_org, memkind))
        return pose, stats, {k: out.get(k) for k in outputs}

    def flow_error_fullres(self, f0, f1, gt, width_org, height_org, classes=None, nclasses=None, with_err=False,
                           memkind=MEM_HOST, err=None):
        """Evaluation of the last run's slots [f0, f1) against ground truth at the original frame size
        (preprocess.flow_error on the device, bitwise).  gt: [f1-f0][height_org][width_org][nop] float32 (stereo also
        without the last axis); classes: [f1-f0][height_org][width_org] uint8, e.g. a consistency mask (then nclasses
        is required; without classes it is 1).  Returns (stats, err): stats a (f1-f0, nclasses) array of
        ERROR_STATS_DTYPE, err the float32 error map (NaN where the ground truth is unknown), None unless with_err
        (host: a new array, or `err` given as a numpy array of exactly that shape).  With memkind=MEM_DEVICE, gt,
        classes and err are device addresses the caller owns (err None: no map); stats are always returned on the
        host.  The call synchronises the context's stream."""
        if nclasses is None:
            if classes is not None:
                raise ValueError("flow_error_fullres: nclasses is required with classes")
            nclasses = 1
        shape = (f1 - f0, height_org, width_org)
        if memkind == MEM_HOST:
            nop = self.prm.nop
            gt_shapes = (shape + (nop,),) + ((shape,) if nop == 1 else ())
            err = (np.empty(shape, np.float32) if err is None else err) if with_err else None
            for name, arr, dt, shapes, write in (("gt", gt, np.float32, gt_shapes, False),
                                                 ("classes", classes, np.uint8, (shape,), False),
                                                 ("err", err, np.float32, (shape,), True)):
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape in shapes
                                            and arr.flags["C_CONTIGUOUS"] and (arr.flags["WRITEABLE"] or not write)):
                    raise ValueError("flow_error_fullres: %s must be a %sC-contiguous %s array of shape %s"
                                     % (name, "writeable " if write else "", np.dtype(dt).name,
                                        " or ".join(map(str, shapes))))
        stats = np.zeros((max(f1 - f0, 0), max(nclasses, 0)), ERROR_STATS_DTYPE)
        self._ck(lib().ofdis_flow_error_fullres(self._h, f0, f1, _ptr(gt), _ptr(classes), nclasses, _ptr(stats),
                                                _ptr(err), width_org, height_org, memkind))
        return stats, err

    def get_flow_fullres(self, f0, f1, dst, width_org, height_org, memkind=MEM_HOST):
        """Flow x 2^sc_l, upsampled to the original frame size and cropped (run_dense.cpp:407-414)."""
        self._ck(lib().ofdis_get_flow_fullres(self._h, f0, f1, _ptr(dst), width_org, height_org, memkind))

    def get_flow_fullres_encoded(self, f0, f1, encoding, width_org, height_org, out=None, memkind=MEM_HOST):
        """get_flow_fullres of slots [f0, f1), encoded on the device as `encoding` (a key of ENCODINGS; the format
        contract is ofdis_get_flow_fullres_encoded's, restated by preprocess.encode_f16 / encode_kitti).  Host result:
        "f16" a (f1-f0, height_org, width_org, nop) float16 array, "kitti" a (f1-f0, height_org, width_org, 3) uint16
        array for flow and (f1-f0, height_org, width_org) for stereo -- a new array, or `out` given as a numpy array
        of exactly that dtype and shape; the call then synchronises the stream.  With memkind=MEM_DEVICE, out is a
        device address the caller owns (e.g. a torch.float16 tensor's data_ptr()) and is returned as given."""
        if encoding not in ENCODINGS:
            raise ValueError("get_flow_fullres_encoded: encoding must be one of %s" % ", ".join(ENCODINGS))
        if memkind == MEM_HOST:
            nop = self.prm.nop
            shape = (max(f1 - f0, 0), height_org, width_org)
            if encoding == "f16":
                shape, dt = shape + (nop,), np.float16
            else:
                shape, dt = shape + ((3,) if nop == 2 else ()), np.uint16
            out = np.empty(shape, dt) if out is None else out
            if not (isinstance(out, np.ndarray) and out.dtype == dt and out.shape == shape
                    and out.flags["C_CONTIGUOUS"] and out.flags["WRITEABLE"]):
                raise ValueError("get_flow_fullres_encoded: out must be a writeable C-contiguous %s array of shape %s"
                                 % (np.dtype(dt).name, shape))
        self._ck(lib().ofdis_get_flow_fullres_encoded(self._h, f0, f1, ENCODINGS[encoding], _ptr(out), width_org,
                                                      height_org, memkind))
        if memkind == MEM_HOST:
            self.sync()
        return out

    def flow_color_fullres(self, f0, f1, width_org, height_org, max_value=0.0, out=None, with_scale=False,
                           memkind=MEM_HOST, scale=None):
        """The color images of slots [f0, f1) computed on the device: Middlebury's color wheel for flow, KITTI's
        disparity map for stereo (the contract is ofdis_flow_color_fullres's, restated by preprocess.flow_to_color /
        disp_to_color).  max_value > 0 fixes the scale; 0 takes each slot's own maximum.  Returns (rgb, scale).  Host:
        rgb a (f1-f0, height_org, width_org, 3) uint8 array and scale a (f1-f0,) float32 array (None unless
        with_scale), each new or given as a numpy array of exactly that dtype and shape; the call then synchronises
        the stream.  With memkind=MEM_DEVICE, out and scale are device addresses the caller owns (scale may be None)
        and are returned as given."""
        if memkind == MEM_HOST:
            n = max(f1 - f0, 0)
            out = np.empty((n, height_org, width_org, 3), np.uint8) if out is None else out
            scale = (np.empty(n, np.float32) if scale is None else scale) if with_scale else None
            for name, arr, dt, shape in (("out", out, np.uint8, (n, height_org, width_org, 3)),
                                         ("scale", scale, np.float32, (n,))):
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shape
                                            and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("flow_color_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shape))
        self._ck(lib().ofdis_flow_color_fullres(self._h, f0, f1, _ptr(out), _ptr(scale), max_value, width_org,
                                                height_org, memkind))
        if memkind == MEM_HOST:
            self.sync()
        return out, scale

    def interpolate_fullres(self, f0, f1, b0, frames0, frames1, t, width_org, height_org, alpha=None, beta=None,
                            out=None, with_flow=False, memkind=MEM_HOST, flow_t=None, frame_stride=None):
        """The frame at time t (0 < t < 1) between frames0[k] and frames1[k], from the last run's forward flow in slot
        f0 + k and its backward partner in slot b0 + k (ofdis_interpolate_fullres; preprocess.interpolate_frames
        restates it).  alpha/beta None: CONSISTENCY_DEFAULTS of the context's nop.  Returns (out, flow_t).  Host:
        frames0, frames1 uint8 arrays (f1-f0, height_org, width_org[, noc]) whose frames are C-contiguous and whose
        strides[0] agree -- frames[:-1] / frames[1:] of a clip and pairs[:, 0] / pairs[:, 1] both qualify; out a
        (f1-f0, height_org, width_org[, noc]) uint8 array (no channel axis for gray) and flow_t a (f1-f0, height_org,
        width_org, nop) float32 array (None unless with_flow), each new or given as a numpy array of exactly that
        dtype and shape; the call then synchronises the stream.  With memkind=MEM_DEVICE, frames0, frames1, out and
        flow_t are device addresses the caller owns (flow_t may be None) and frame_stride the bytes between frames
        (default: one frame); out and flow_t are returned as given and are ready when the context's stream is.  The
        hole filling synchronises the stream on the way."""
        da, db = CONSISTENCY_DEFAULTS[self.prm.nop]
        alpha = da if alpha is None else alpha
        beta = db if beta is None else beta
        noc, nop = self.prm.noc, self.prm.nop
        n = max(f1 - f0, 0)
        hwc = height_org * width_org * noc
        frame = (height_org, width_org) + ((noc,) if noc > 1 else ())
        if memkind == MEM_HOST:
            strides = []
            for name, arr in (("frames0", frames0), ("frames1", frames1)):
                ok = isinstance(arr, np.ndarray) and arr.dtype == np.uint8 and arr.ndim >= 3 and arr.shape[0] == n \
                    and arr.shape[1:] in (frame, (height_org, width_org, noc)) \
                    and (n == 0 or arr[0].flags["C_CONTIGUOUS"]) and (n < 2 or arr.strides[0] >= hwc)
                if not ok:
                    raise ValueError("interpolate_fullres: %s must be a uint8 array of shape %s whose frames are "
                                     "C-contiguous" % (name, (n,) + frame))
                strides.append(arr.strides[0] if n > 1 else hwc)
            if strides[0] != strides[1]:
                raise ValueError("interpolate_fullres: frames0 and frames1 must have the same strides[0]")
            frame_stride = strides[0]
            out = np.empty((n,) + frame, np.uint8) if out is None else out
            flow_t = (np.empty((n, height_org, width_org, nop), np.float32) if flow_t is None else flow_t) \
                if with_flow else None
            for name, arr, dt, shape in (("out", out, np.uint8, (n,) + frame),
                                         ("flow_t", flow_t, np.float32, (n, height_org, width_org, nop))):
                if arr is not None and not (isinstance(arr, np.ndarray) and arr.dtype == dt and arr.shape == shape
                                            and arr.flags["C_CONTIGUOUS"] and arr.flags["WRITEABLE"]):
                    raise ValueError("interpolate_fullres: %s must be a writeable C-contiguous %s array of shape %s"
                                     % (name, np.dtype(dt).name, shape))
            p0, p1 = frames0.ctypes.data, frames1.ctypes.data
        else:
            frame_stride = hwc if frame_stride is None else frame_stride
            p0, p1 = frames0, frames1
        self._ck(lib().ofdis_interpolate_fullres(self._h, f0, f1, b0, _ptr(p0), _ptr(p1), frame_stride, t, alpha,
                                                 beta, _ptr(out), _ptr(flow_t), width_org, height_org, memkind))
        if memkind == MEM_HOST:
            self.sync()
        return out, flow_t

    def _frames_u8(self, name, frames, n, width_org, height_org):
        """Checks a host array of n 8-bit frames of the context's channel count whose frames are C-contiguous and
        returns its frame stride in bytes."""
        noc = self.prm.noc
        hwc = height_org * width_org * noc
        frame = (height_org, width_org) + ((noc,) if noc > 1 else ())
        ok = isinstance(frames, np.ndarray) and frames.dtype == np.uint8 and frames.ndim >= 3 and \
            frames.shape[0] == n and frames.shape[1:] in (frame, (height_org, width_org, noc)) and \
            (n == 0 or frames[0].flags["C_CONTIGUOUS"]) and (n < 2 or frames.strides[0] >= hwc)
        if not ok:
            raise ValueError("%s must be a uint8 array of shape %s whose frames are C-contiguous" % (name, (n,) + frame))
        return frames.strides[0] if n > 1 else hwc

    def track_begin(self, params, frame, width_org, height_org, memkind=MEM_HOST, points=None):
        """Resets the context's tracker and seeds `frame` (ofdis_track_begin; preprocess.track_points restates it).
        params: a mapping with the keys of preprocess.TRACK_PARAM_FIELDS (or a TrackParams).  Host: frame a uint8
        (height_org, width_org[, noc]) array; returns frame 0's tracks as an array of TRACK_POINT_DTYPE.  With
        memkind=MEM_DEVICE, frame and points are device addresses the caller owns (points: `capacity` records) and
        the count of records written is returned."""
        if not isinstance(params, TrackParams):
            params = TrackParams(*[params[k] for k in TRACK_PARAM_FIELDS])
        self._track_capacity = params.capacity
        count = ctypes.c_int(0)
        if memkind == MEM_HOST:
            self._frames_u8("track_begin: frame", np.asarray(frame)[None], 1, width_org, height_org)
            frame = np.ascontiguousarray(frame)
            points = np.empty(max(params.capacity, 0), TRACK_POINT_DTYPE)
        self._ck(lib().ofdis_track_begin(self._h, ctypes.byref(params), _ptr(frame), _ptr(points), ctypes.byref(count),
                                         width_org, height_org, memkind))
        return points[:count.value].copy() if memkind == MEM_HOST else count.value

    def track_advance(self, f0, f1, b0, frames, width_org, height_org, frame_stride=None, memkind=MEM_HOST,
                      points=None):
        """Advances the tracker through the last run's slots f0 + k (forward) and b0 + k (backward), seeding frames[k]
        after pair k (ofdis_track_advance).  Host: frames a uint8 (f1-f0, height_org, width_org[, noc]) array whose
        frames are C-contiguous -- clip[1:] of a clip, or pairs[:, 1] of a pair array; returns the f1-f0 lists of
        TRACK_POINT_DTYPE.  With memkind=MEM_DEVICE, frames and points are device addresses the caller owns (points:
        (f1-f0) x capacity records, list k at record k*capacity), frame_stride the bytes between frames (default one
        frame), and the int32 counts of the lists are returned."""
        n = max(f1 - f0, 0)
        cap = getattr(self, "_track_capacity", 0)
        counts = np.zeros(n, np.int32)
        if memkind == MEM_HOST:
            frame_stride = self._frames_u8("track_advance: frames", frames, n, width_org, height_org)
            points = np.empty(n * cap, TRACK_POINT_DTYPE)
            pf = frames.ctypes.data
        else:
            frame_stride = height_org * width_org * self.prm.noc if frame_stride is None else frame_stride
            pf = frames
        self._ck(lib().ofdis_track_advance(self._h, f0, f1, b0, _ptr(pf), frame_stride, _ptr(points), _ptr(counts),
                                           width_org, height_org, memkind))
        if memkind != MEM_HOST:
            return counts
        return [points[k * cap:k * cap + counts[k]].copy() for k in range(n)]

    def track_stats(self):
        """The tracker's counters since track_begin (ofdis_track_stats_get): a dict of preprocess.TRACK_STATS_FIELDS."""
        st = TrackStats()
        rc = lib().ofdis_track_stats_get(self._h, ctypes.byref(st))
        if rc != 0:
            raise OfdisError("track_stats: status %d" % rc)
        return {k: int(getattr(st, k)) for k in TRACK_STATS_FIELDS}

    def traj_begin(self, track_params, traj_params, frame, width_org, height_org, memkind=MEM_HOST, points=None):
        """Resets the context's tracker and its descriptor stage and seeds `frame` (ofdis_traj_begin;
        preprocess.traj_descriptors restates the whole stage).  track_params as track_begin's; traj_params a mapping
        with the keys of preprocess.TRAJ_PARAM_FIELDS (or a TrajParams).  Returns what track_begin returns."""
        if not isinstance(track_params, TrackParams):
            track_params = TrackParams(*[track_params[k] for k in TRACK_PARAM_FIELDS])
        if not isinstance(traj_params, TrajParams):
            traj_params = TrajParams(*[traj_params[k] for k in TRAJ_PARAM_FIELDS])
        count = ctypes.c_int(0)
        if memkind == MEM_HOST:
            self._frames_u8("traj_begin: frame", np.asarray(frame)[None], 1, width_org, height_org)
            frame = np.ascontiguousarray(frame)
            points = np.empty(max(track_params.capacity, 0), TRACK_POINT_DTYPE)
        self._ck(lib().ofdis_traj_begin(self._h, ctypes.byref(track_params), ctypes.byref(traj_params), _ptr(frame),
                                        _ptr(points), ctypes.byref(count), width_org, height_org, memkind))
        # only a stage the library accepted sizes the host outputs of traj_advance: a refused begin leaves the
        # previous stage, and its parameters, live
        self._track_capacity = track_params.capacity
        self._traj = {k: getattr(traj_params, k) for k in TRAJ_PARAM_FIELDS}
        return points[:count.value].copy() if memkind == MEM_HOST else count.value

    def traj_advance(self, f0, f1, b0, frames, width_org, height_org, models=None, frame_stride=None,
                     memkind=MEM_HOST, points=None, records=None, desc=None):
        """track_advance with the descriptors of every pair (ofdis_traj_advance).  models: None (no compensation) or
        (f1-f0, 9) float64 as global_motion_fullres returns them, always on the host.  Host: returns (lists, records,
        desc, n_desc) -- the tracker's lists, the emitted segments' TRAJ_RECORD_DTYPE records and (count, dim) float32
        descriptors, and the int32 segments per pair.  With memkind=MEM_DEVICE frames, points, records and desc are
        device addresses the caller owns (records and desc: preprocess.traj_bound(capacity, f1-f0, L) entries) and
        (counts, n_desc) is returned."""
        n = max(f1 - f0, 0)
        cap = getattr(self, "_track_capacity", 0)
        tp = getattr(self, "_traj", None)
        L = tp["L"] if tp else 1
        dim = traj_dim(tp) if tp else 0
        bound = traj_bound(cap, n, L)
        counts = np.zeros(n, np.int32)
        n_desc = np.zeros(n, np.int32)
        pm = None
        if models is not None:
            pm = np.ascontiguousarray(models, np.float64)
            if pm.shape != (n, 9) and pm.shape != (n, 3, 3):
                raise ValueError("traj_advance: models must be (%d, 9) float64" % n)
        if memkind == MEM_HOST:
            frame_stride = self._frames_u8("traj_advance: frames", frames, n, width_org, height_org)
            points = np.empty(n * cap, TRACK_POINT_DTYPE)
            records = np.empty(bound, TRAJ_RECORD_DTYPE)
            desc = np.empty((bound, dim), np.float32)
            pf = frames.ctypes.data
        else:
            frame_stride = height_org * width_org * self.prm.noc if frame_stride is None else frame_stride
            pf = frames
        self._ck(lib().ofdis_traj_advance(self._h, f0, f1, b0, _ptr(pf), frame_stride, _ptr(pm), _ptr(points),
                                          _ptr(counts), _ptr(records), _ptr(desc), _ptr(n_desc), width_org,
                                          height_org, memkind))
        if memkind != MEM_HOST:
            return counts, n_desc
        total = int(n_desc.sum())
        lists = [points[k * cap:k * cap + counts[k]].copy() for k in range(n)]
        return lists, records[:total].copy(), desc[:total].copy(), n_desc

    def traj_stats(self):
        """The descriptor stage's counters since traj_begin (ofdis_traj_stats_get): a dict of
        preprocess.TRAJ_STATS_FIELDS."""
        st = TrajStats()
        rc = lib().ofdis_traj_stats_get(self._h, ctypes.byref(st))
        if rc != 0:
            raise OfdisError("traj_stats: status %d" % rc)
        return {k: int(getattr(st, k)) for k in TRAJ_STATS_FIELDS}

    def stab_begin(self, params, frame0, width_org, height_org, weights=None, memkind=MEM_HOST):
        """Resets the context's stabiliser on frame 0 (ofdis_stab_begin; preprocess.stabilize restates the whole clip).
        params: a mapping with preprocess.STAB_PARAM_FIELDS or a StabParams; weights: r+1 floats, by default
        preprocess.gaussian_weights(radius).  Host: frame0 a uint8 (height_org, width_org[, noc]) array; with
        memkind=MEM_DEVICE a device address the caller owns."""
        if not isinstance(params, StabParams):
            params = StabParams(*[params[k] for k in STAB_PARAM_FIELDS])
        wts = np.ascontiguousarray(gaussian_weights(params.radius) if weights is None else weights, np.float64)
        if wts.shape != (max(params.radius, 0) + 1,):
            raise ValueError("stab_begin: weights must hold radius + 1 = %d values" % (params.radius + 1))
        if memkind == MEM_HOST:
            self._frames_u8("stab_begin: frame0", np.asarray(frame0)[None], 1, width_org, height_org)
            frame0 = np.ascontiguousarray(frame0)
        self._ck(lib().ofdis_stab_begin(self._h, ctypes.byref(params), _ptr(wts), _ptr(frame0), width_org, height_org,
                                        memkind))
        self._stab = (params.radius, width_org, height_org)

    def _stab_out(self, frames, out, memkind):
        _, w, h = getattr(self, "_stab", (0, 0, 0))
        noc = self.prm.noc
        shape = (frames, h, w) + ((noc,) if noc > 1 else ())
        if memkind == MEM_HOST:
            return np.empty(shape, np.uint8)
        if out is None:
            raise ValueError("stab: memkind=MEM_DEVICE needs out, a device address of %s bytes" % (shape,))
        return out

    def stab_push(self, models, frames, frame_stride=None, memkind=MEM_HOST, out=None):
        """Appends n frames and their n models (ofdis_stab_push) and returns (out[:n_out], info): the frames whose
        smoothing window is complete, and their records (n_out,) of STAB_FRAME_DTYPE.  models: (n, 3, 3) float64 on the
        host, model k mapping the previous frame onto frames[k] -- what global_motion_fullres returns.  Host: frames a
        uint8 (n, height_org, width_org[, noc]) array whose frames are C-contiguous (clip[1:] or pairs[:, 1]).  With
        memkind=MEM_DEVICE, frames and out ([n] frames) are device addresses the caller owns, frame_stride the bytes
        between frames (default one frame), and out is returned as given with n_out."""
        models = np.ascontiguousarray(models, np.float64).reshape(-1, 9)
        n = models.shape[0]
        _, w, h = getattr(self, "_stab", (0, 0, 0))
        if memkind == MEM_HOST:
            frame_stride = self._frames_u8("stab_push: frames", frames, n, w, h)
            pf = frames.ctypes.data
        else:
            frame_stride = h * w * self.prm.noc if frame_stride is None else frame_stride
            pf = frames
        dst = self._stab_out(max(n, 1), out, memkind)
        info = np.zeros(max(n, 1), STAB_FRAME_DTYPE)
        n_out = ctypes.c_int(0)
        self._ck(lib().ofdis_stab_push(self._h, n, _ptr(models), _ptr(pf), frame_stride, _ptr(dst), _ptr(info),
                                       ctypes.byref(n_out), memkind))
        k = n_out.value
        return (dst[:k] if memkind == MEM_HOST else (dst, k)), info[:k].copy()

    def stab_finish(self, memkind=MEM_HOST, out=None):
        """Emits the remaining frames and ends the stabiliser (ofdis_stab_finish): (out[:n_out], info) as stab_push,
        out holding radius frames."""
        r = getattr(self, "_stab", (0, 0, 0))[0]
        dst = self._stab_out(max(r, 1), out, memkind)
        info = np.zeros(max(r, 1), STAB_FRAME_DTYPE)
        n_out = ctypes.c_int(0)
        self._ck(lib().ofdis_stab_finish(self._h, _ptr(dst), _ptr(info), ctypes.byref(n_out), memkind))
        k = n_out.value
        return (dst[:k] if memkind == MEM_HOST else (dst, k)), info[:k].copy()

    def fisher_begin(self, codebook):
        """Resets the context's Fisher encoder on `codebook` (ofdis_fisher_begin; preprocess.FisherStream restates the
        encoder): a dict of preprocess.fisher_unpack / read_fisher_codebook."""
        K, blocks = int(codebook["K"]), [tuple(int(v) for v in b) for b in codebook["blocks"]]
        body = np.ascontiguousarray(fisher_pack(codebook), np.float32)
        c = FisherCodebook()
        c.K, c.desc_dim, c.nblocks = K, int(codebook["desc_dim"]), len(blocks)
        if len(blocks) > FISHER_MAX_BLOCKS or body.size != fisher_sizes(K, blocks)["body"]:
            raise ValueError("fisher_begin: %d blocks, body of %d floats" % (len(blocks), body.size))
        for b, (o, di, d) in enumerate(blocks):
            c.blocks[b] = FisherBlock(o, di, d)
        c.params = body.ctypes.data
        self._ck(lib().ofdis_fisher_begin(self._h, ctypes.byref(c)))
        self._fisher = (K, blocks, int(codebook["desc_dim"]))

    def fisher_push(self, desc, memkind=MEM_HOST, n=None):
        """Adds descriptors to the clip (ofdis_fisher_push): host (n, desc_dim) float32, or with memkind=MEM_DEVICE
        a device address of n descriptors."""
        if memkind == MEM_HOST:
            D = getattr(self, "_fisher", (0, [], 0))[2]
            desc = np.ascontiguousarray(desc, np.float32)
            if desc.size and (desc.ndim != 2 or desc.shape[1] != D):
                raise ValueError("fisher_push: desc must be (n, %d) float32" % D)
            n = desc.shape[0] if desc.ndim == 2 else 0
        elif n is None:
            raise ValueError("fisher_push: device input needs n, the number of descriptors at the address")
        self._ck(lib().ofdis_fisher_push(self._h, _ptr(desc), int(n), memkind))

    def fisher_take(self, memkind=MEM_HOST, fv=None, stats=None, with_fv=True, with_stats=True):
        """Ends the clip (ofdis_fisher_take).  Host: returns (fv float32 (2K sum dim,), stats float64, counters) --
        counters a dict with `pushed` and per-block `n` and `skipped` arrays -- fv or stats None where not asked for.
        With memkind=MEM_DEVICE fv and stats are device addresses the caller owns (or None) and counters is returned."""
        K, blocks, _ = getattr(self, "_fisher", (1, [(0, 1, 1)], 1))
        sz = fisher_sizes(K, blocks)
        if memkind == MEM_HOST:
            fv = np.empty(sz["fv"], np.float32) if with_fv else None
            stats = np.empty(sz["stats"], np.float64) if with_stats else None
        st = FisherStats()
        self._ck(lib().ofdis_fisher_take(self._h, _ptr(fv), _ptr(stats), ctypes.byref(st), memkind))
        nb = len(blocks)
        counters = {"pushed": int(st.pushed), "n": np.array(st.n[:nb], np.int64),
                    "skipped": np.array(st.skipped[:nb], np.int64)}
        return counters if memkind != MEM_HOST else (fv, stats, counters)

    def fisher_fit(self, samples, blocks, dims, K=256, iters=10, seed=0, var_floor=1e-3):
        """preprocess.fisher_fit with the E-step on the device: each iteration is a fisher_begin, one push of the
        samples and a take of the statistics; the M-step runs on the host.  Returns the same codebook bytes as
        preprocess.fisher_fit."""
        x = np.ascontiguousarray(samples, np.float32)

        def estep(cb, xs):
            self.fisher_begin(cb)
            self.fisher_push(xs)
            return self.fisher_take(with_fv=False)[1]

        return fisher_fit(x, blocks, dims, K, iters, seed, var_floor, estep=estep)

    def fuse_begin(self, params):
        """Resets the context's fusion volume (ofdis_fuse_begin; preprocess.fuse_new_volume is its restatement).
        params: a mapping with preprocess.FUSE_PARAM_FIELDS (origin three numbers) or a FuseParams."""
        if not isinstance(params, FuseParams):
            params = FuseParams(int(params["nx"]), int(params["ny"]), int(params["nz"]),
                                (ctypes.c_float * 3)(*[float(v) for v in params["origin"]]), float(params["voxel"]),
                                float(params["trunc"]), float(params["max_weight"]), int(params["color"]))
        self._ck(lib().ofdis_fuse_begin(self._h, ctypes.byref(params)))
        self._fuse = (params.nx, params.ny, params.nz, params.color)

    @staticmethod
    def _fuse_cam(camera):
        return None if camera is None else ctypes.byref(StereoCamera(*[camera[k] for k in STEREO_CAMERA_FIELDS]))

    @staticmethod
    def _fuse_poses(poses):
        poses = np.ascontiguousarray(poses, np.float64)
        if poses.size % 12:
            raise ValueError("fuse: poses must be (n, 3, 4) float64")
        return poses.reshape(-1, 12)

    def fuse_push(self, disp, poses, camera, *, width_org, height_org, max_depth=float("inf"), frames=None,
                  disp_stride=None, frame_stride=None, memkind=MEM_HOST, weights=None, weight_stride=None):
        """Integrates n frames into the volume (ofdis_fuse_push; preprocess.fuse_integrate restates it): disp (n, H, W)
        positive disparities (NaN unknown), poses (n, 3, 4) camera-to-world float64 on the host, camera a mapping
        with STEREO_CAMERA_FIELDS and, when the volume keeps colour, frames (n, H, W[, noc]) uint8.  Host arrays'
        frames must be C-contiguous and equally spaced; with memkind=MEM_DEVICE disp and frames are device addresses
        the caller owns and the strides count floats and bytes between frames (default one frame).  weights (n, H, W)
        float32 (e.g. confidence_fullres's conf), or a device address with weight_stride floats between frames,
        calls ofdis_fuse_push_weighted instead."""
        poses = self._fuse_poses(poses)
        n = poses.shape[0]
        pix = width_org * height_org
        if memkind == MEM_HOST:
            ok = isinstance(disp, np.ndarray) and disp.dtype == np.float32 and disp.shape == (n, height_org, width_org) \
                and (n == 0 or disp[0].flags["C_CONTIGUOUS"]) and disp.strides[0] % 4 == 0
            if not ok:
                raise ValueError("fuse_push: disp must be a float32 array of shape %s whose frames are C-contiguous"
                                 % ((n, height_org, width_org),))
            disp_stride = disp.strides[0] // 4 if n > 1 else pix
            if frames is not None:
                frame_stride = self._frames_u8("fuse_push: frames", frames, n, width_org, height_org)
                frames = frames.ctypes.data
            if weights is not None:
                weight_stride = self._weights_f32("fuse_push: weights", weights, n, width_org, height_org)
        else:
            disp_stride = pix if disp_stride is None else disp_stride
            frame_stride = pix * self.prm.noc if frame_stride is None else frame_stride
            weight_stride = pix if weight_stride is None else weight_stride
        if weights is None:
            self._ck(lib().ofdis_fuse_push(self._h, n, _ptr(disp), disp_stride, _ptr(poses), self._fuse_cam(camera),
                                           max_depth, _ptr(frames), frame_stride or 0, width_org, height_org, memkind))
        else:
            self._ck(lib().ofdis_fuse_push_weighted(self._h, n, _ptr(disp), disp_stride, _ptr(poses),
                                                    self._fuse_cam(camera), max_depth, _ptr(frames), frame_stride or 0,
                                                    _ptr(weights), weight_stride, width_org, height_org, memkind))

    @staticmethod
    def _weights_f32(name, weights, n, width_org, height_org):
        """Checks a host float32 array of n (height_org, width_org) maps whose maps are C-contiguous and returns its
        stride in floats."""
        ok = isinstance(weights, np.ndarray) and weights.dtype == np.float32 and \
            weights.shape == (n, height_org, width_org) and (n == 0 or weights[0].flags["C_CONTIGUOUS"]) and \
            weights.strides[0] % 4 == 0 and (n < 2 or weights.strides[0] >= 4 * height_org * width_org)
        if not ok:
            raise ValueError("%s must be a float32 array of shape %s whose maps are C-contiguous"
                             % (name, (n, height_org, width_org)))
        return weights.strides[0] // 4 if n > 1 else width_org * height_org

    def fuse_extract(self, min_weight=1.0, capacity=None, memkind=MEM_HOST, out=None):
        """The volume's zero crossings (ofdis_fuse_extract; preprocess.fuse_extract restates it).  Host: returns
        (points of FUSE_POINT_DTYPE, total); capacity None counts first and takes them all, else at most capacity.
        With memkind=MEM_DEVICE out is a device address of capacity records the caller owns; returns (out, total)."""
        total = ctypes.c_long(0)
        if memkind != MEM_HOST:
            self._ck(lib().ofdis_fuse_extract(self._h, min_weight, _ptr(out), capacity or 0, ctypes.byref(total),
                                              memkind))
            return out, total.value
        if capacity is None:
            self._ck(lib().ofdis_fuse_extract(self._h, min_weight, None, 0, ctypes.byref(total), memkind))
            capacity = total.value
        pts = np.zeros(capacity, FUSE_POINT_DTYPE)
        self._ck(lib().ofdis_fuse_extract(self._h, min_weight, _ptr(pts) if capacity else None, capacity,
                                          ctypes.byref(total), memkind))
        return pts[:min(capacity, total.value)], total.value

    def fuse_render(self, poses, camera, *, z_near, z_far, step, width_org, height_org, min_weight=1.0,
                    memkind=MEM_HOST, out=None):
        """Ray-cast depth of the volume from n camera-to-world poses (ofdis_fuse_render; preprocess.fuse_render
        restates it): host (n, height_org, width_org) float32, qNaN where no ray meets the surface; with
        memkind=MEM_DEVICE out is a device address the caller owns and is returned as given."""
        poses = self._fuse_poses(poses)
        n = poses.shape[0]
        if memkind == MEM_HOST:
            out = np.empty((n, height_org, width_org), np.float32)
        self._ck(lib().ofdis_fuse_render(self._h, n, _ptr(poses), self._fuse_cam(camera), z_near, z_far, step,
                                         min_weight, _ptr(out), width_org, height_org, memkind))
        return out

    def fuse_volume(self, memkind=MEM_HOST, T=None, W=None, color=None):
        """The volume (ofdis_fuse_get_volume): host returns {"T", "W", "C"} as preprocess.fuse_new_volume lays them
        out (C None without colour); with memkind=MEM_DEVICE T, W and color are device addresses (or None)."""
        if memkind == MEM_HOST:
            nx, ny, nz, col = getattr(self, "_fuse", (0, 0, 0, 0))
            T, W = np.empty((nz, ny, nx), np.float32), np.empty((nz, ny, nx), np.float32)
            color = np.empty((nz, ny, nx, 3), np.uint8) if col else None
        self._ck(lib().ofdis_fuse_get_volume(self._h, _ptr(T), _ptr(W), _ptr(color), memkind))
        return {"T": T, "W": W, "C": color}

    def fuse_set_volume(self, T=None, W=None, color=None, memkind=MEM_HOST):
        """Loads the volume (ofdis_fuse_set_volume, the inverse of fuse_volume): host T and W float32 and color uint8
        as preprocess.fuse_new_volume lays them out, or device addresses with memkind=MEM_DEVICE; None leaves that
        array as it was."""
        if memkind == MEM_HOST:
            nx, ny, nz, _ = getattr(self, "_fuse", (0, 0, 0, 0))
            arrs = []
            for a, dt, shape in ((T, np.float32, (nz, ny, nx)), (W, np.float32, (nz, ny, nx)),
                                 (color, np.uint8, (nz, ny, nx, 3))):
                if a is not None:
                    a = np.ascontiguousarray(a, dt)
                    if a.shape != shape:
                        raise ValueError("fuse_set_volume: an array of shape %s, expected %s" % (a.shape, shape))
                arrs.append(a)
            T, W, color = arrs
        self._ck(lib().ofdis_fuse_set_volume(self._h, _ptr(T), _ptr(W), _ptr(color), memkind))

    def fuse_mesh(self, min_weight=1.0, pt_capacity=None, face_capacity=None, memkind=MEM_HOST, pts_out=None,
                  faces_out=None):
        """The volume's triangle mesh (ofdis_fuse_mesh; preprocess.fuse_mesh restates it): returns (points, faces,
        n_points, n_faces).  Host: points of FUSE_POINT_DTYPE (the points of fuse_extract) and faces (F, 3) uint32; a
        capacity None counts first and takes them all, else at most that many.  With memkind=MEM_DEVICE pts_out and
        faces_out are device addresses of the capacities' records the caller owns and are returned as given."""
        n_pts, n_faces = ctypes.c_long(0), ctypes.c_long(0)
        if memkind != MEM_HOST:
            self._ck(lib().ofdis_fuse_mesh(self._h, min_weight, _ptr(pts_out), pt_capacity or 0, ctypes.byref(n_pts),
                                           _ptr(faces_out), face_capacity or 0, ctypes.byref(n_faces), memkind))
            return pts_out, faces_out, n_pts.value, n_faces.value
        if pt_capacity is None or face_capacity is None:
            self._ck(lib().ofdis_fuse_mesh(self._h, min_weight, None, 0, ctypes.byref(n_pts), None, 0,
                                           ctypes.byref(n_faces), memkind))
            pt_capacity = n_pts.value if pt_capacity is None else pt_capacity
            face_capacity = n_faces.value if face_capacity is None else face_capacity
        pts = np.zeros(pt_capacity, FUSE_POINT_DTYPE)
        faces = np.zeros((face_capacity, 3), np.uint32)
        self._ck(lib().ofdis_fuse_mesh(self._h, min_weight, _ptr(pts) if pt_capacity else None, pt_capacity,
                                       ctypes.byref(n_pts), _ptr(faces) if face_capacity else None, face_capacity,
                                       ctypes.byref(n_faces), memkind))
        return pts[:min(pt_capacity, n_pts.value)], faces[:min(face_capacity, n_faces.value)], n_pts.value, \
            n_faces.value

    def fuse_track(self, disp, motions, prev, camera, params, *, width_org, height_org, frames=None, disp_stride=None,
                   frame_stride=None, n=None, memkind=MEM_HOST, weights=None, weight_stride=None):
        """Aligns n frames to the volume, each before the next, and with params["integrate"] pushes each at its final
        pose (ofdis_fuse_track; preprocess.fuse_track restates it).  disp (n, H, W) float32 positive disparities (NaN
        unknown), motions (n, 3, 4) float64 camera k-1 to camera k or None (the identity), prev (3, 4) the
        camera-to-world pose before frame 0, params a mapping with preprocess.FUSE_TRACK_PARAM_FIELDS or a
        FuseTrackParams, frames (n, H, W[, noc]) uint8 when integrating into a volume with colour.  With
        memkind=MEM_DEVICE disp and frames are device addresses the caller owns, n is required and the strides count
        floats and bytes between frames (default one frame).  weights (n, H, W) float32, or a device address with
        weight_stride floats between frames, calls ofdis_fuse_track_weighted instead.  Returns (poses (n, 3, 4)
        float64, stats (n,) FUSE_TRACK_STATS_DTYPE)."""
        if not isinstance(params, FuseTrackParams):
            params = FuseTrackParams(*[params[k] for k in FUSE_TRACK_PARAM_FIELDS])
        pix = width_org * height_org
        if memkind == MEM_HOST:
            n = disp.shape[0] if isinstance(disp, np.ndarray) and disp.ndim == 3 else -1
            ok = isinstance(disp, np.ndarray) and disp.dtype == np.float32 and disp.shape == (n, height_org, width_org) \
                and (n == 0 or disp[0].flags["C_CONTIGUOUS"]) and disp.strides[0] % 4 == 0
            if not ok:
                raise ValueError("fuse_track: disp must be a float32 array (n, %d, %d) whose frames are C-contiguous"
                                 % (height_org, width_org))
            disp_stride = disp.strides[0] // 4 if n > 1 else pix
            if frames is not None:
                frame_stride = self._frames_u8("fuse_track: frames", frames, n, width_org, height_org)
                frames = frames.ctypes.data
            if weights is not None:
                weight_stride = self._weights_f32("fuse_track: weights", weights, n, width_org, height_org)
        else:
            if n is None:
                raise ValueError("fuse_track: device input needs n, the number of frames at the address")
            disp_stride = pix if disp_stride is None else disp_stride
            frame_stride = pix * self.prm.noc if frame_stride is None else frame_stride
            weight_stride = pix if weight_stride is None else weight_stride
        if motions is not None:
            motions = np.ascontiguousarray(motions, np.float64)
            if motions.size != 12 * n:
                raise ValueError("fuse_track: motions must be (n, 3, 4) float64")
        prev = np.ascontiguousarray(prev, np.float64)
        if prev.size != 12:
            raise ValueError("fuse_track: prev must be (3, 4) float64")
        poses = np.zeros((max(n, 1), 3, 4))
        stats = np.zeros(max(n, 1), FUSE_TRACK_STATS_DTYPE)
        st = (FuseTrackStats * max(n, 1))()
        if weights is None:
            self._ck(lib().ofdis_fuse_track(self._h, n, _ptr(disp), disp_stride, _ptr(motions), _ptr(prev),
                                            self._fuse_cam(camera), ctypes.byref(params), _ptr(frames),
                                            frame_stride or 0, _ptr(poses), st, width_org, height_org, memkind))
        else:
            self._ck(lib().ofdis_fuse_track_weighted(self._h, n, _ptr(disp), disp_stride, _ptr(motions), _ptr(prev),
                                                     self._fuse_cam(camera), ctypes.byref(params), _ptr(frames),
                                                     frame_stride or 0, _ptr(weights), weight_stride, _ptr(poses), st,
                                                     width_org, height_org, memkind))
        for k in range(n):
            stats[k] = (st[k].status, st[k].n_corr, st[k].rounds, st[k].cost0, st[k].cost)
        return poses[:n], stats[:n]

    def set_initflow_fullres(self, f0, f1, flow, width_org, height_org, memkind=MEM_HOST):
        """[f1-f0][height_org][width_org][nop] flows of the original frame size -> the init flow of pairs [f0, f1)
        that run(n, use_initflow=True) starts from (preprocess.initflow_from_fullres on the device).  The context's
        width and height must be multiples of 2^(sc_f+1)."""
        if isinstance(flow, np.ndarray):
            flow = np.ascontiguousarray(flow, np.float32)
        self._ck(lib().ofdis_set_initflow_fullres(self._h, f0, f1, _ptr(flow), width_org, height_org, memkind))

    def set_initflow_from_result(self, f0, f1, src_f0, width_org, height_org):
        """Warm start: the init flow of pairs [f0, f1) from the last run's flows of pairs [src_f0, src_f0 + f1 - f0),
        bitwise get_flow_fullres (device) followed by set_initflow_fullres (device)."""
        self._ck(lib().ofdis_set_initflow_from_result(self._h, f0, f1, src_f0, width_org, height_org))

    def upload_packed(self, f0, f1, packed, memkind=MEM_HOST):
        self._ck(lib().ofdis_upload_packed(self._h, f0, f1, _ptr(packed), memkind))

    def set_flow(self, frame, level, flow, memkind=MEM_HOST):
        if isinstance(flow, np.ndarray):
            flow = np.ascontiguousarray(flow, np.float32)
        self._ck(lib().ofdis_set_flow(self._h, frame, level, _ptr(flow), memkind))
        if memkind == MEM_HOST:
            self.sync()

    def get_flow(self, frame, level) -> np.ndarray:
        h, w = self.height >> level, self.width >> level
        out = np.empty((h, w, self.prm.nop), np.float32)
        self._ck(lib().ofdis_get_flow(self._h, frame, level, _ptr(out), MEM_HOST))
        return out

    def get_flow_batch(self, f0, f1, dst, memkind=MEM_HOST):
        self._ck(lib().ofdis_get_flow_batch(self._h, f0, f1, _ptr(dst), memkind))

    def get_patches(self, frame, level):
        li = self.level_info(level)
        n_p = li["nopw"] * li["noph"]
        novals = self.prm.noc * self.prm.p_samp_s ** 2
        p = np.empty((n_p, self.prm.nop), np.float32)
        pw = np.empty((n_p, novals), np.float32)
        conv = np.empty(n_p, np.int32)
        cnt = np.empty(n_p, np.int32)
        self._ck(lib().ofdis_get_patches(self._h, frame, level, _ptr(p), _ptr(pw), _ptr(conv), _ptr(cnt)))
        return dict(p=p, pweight=pw, conv=conv, cnt=cnt, **li)

    # -- stage operators ------------------------------------------------------
    def patgrid_optimize(self, level, f0=0, f1=1, init_from_coarser=True):
        self._ck(lib().ofdis_patgrid_optimize(self._h, level, f0, f1, 1 if init_from_coarser else 0))

    def patgrid_aggregate(self, level, f0=0, f1=1):
        self._ck(lib().ofdis_patgrid_aggregate(self._h, level, f0, f1))

    def varref_refine(self, level, f0=0, f1=1, n_inner=None):
        if n_inner is None:
            self._ck(lib().ofdis_varref_refine(self._h, level, f0, f1))
        else:
            self._ck(lib().ofdis_debug_varref_iters(self._h, level, f0, f1, n_inner))

    def run(self, nframes=1, use_initflow=False):
        self._ck(lib().ofdis_run(self._h, nframes, 1 if use_initflow else 0))

    def sync(self):
        self._ck(lib().ofdis_sync(self._h))

    def set_camlr(self, camlr: int):
        self._ck(lib().ofdis_set_camlr(self._h, camlr))

    def set_option(self, name: str, value: int):
        """Launch-geometry options of ofdis_set_option (results are bit-identical under every setting)."""
        self._ck(lib().ofdis_set_option(self._h, name.encode(), int(value)))

    def set_graph_mode(self, on: bool):
        self._ck(lib().ofdis_set_graph_mode(self._h, 1 if on else 0))

    def profile_kernels(self, nframes: int, steps: int = 5):
        """Eager runs with CUDA events around each stage: {class: ms_per_step, launches_per_step}."""
        ms = (ctypes.c_double * 5)()
        n = (ctypes.c_long * 5)()
        self._ck(lib().ofdis_profile_run(self._h, nframes, steps, ms, n))
        names = ("patch", "densify", "vr_setup", "assemble", "sor")
        return {k: {"ms_per_step": ms[i] / steps, "launches_per_step": n[i] / steps} for i, k in enumerate(names)}

    def profile_levels(self, nframes: int, steps: int = 3):
        """Like profile_kernels, split by pyramid level: {level: {class: ms_per_step}}."""
        nlev = self.prm.sc_f - self.prm.sc_l + 1
        ms = (ctypes.c_double * 5)()
        n = (ctypes.c_long * 5)()
        lv = (ctypes.c_double * (5 * nlev))()
        self._ck(lib().ofdis_profile_levels(self._h, nframes, steps, ms, n, lv))
        names = ("patch", "densify", "vr_setup", "assemble", "sor")
        return {self.prm.sc_l + i: {k: lv[i * 5 + j] / steps for j, k in enumerate(names)} for i in range(nlev)}

    @property
    def launch_count(self) -> int:
        return lib().ofdis_launch_count(self._h)

    def debug_get(self, name: str, frame: int, level: int) -> np.ndarray:
        li = self.level_info(level)
        pitch = (li["w"] + 3) // 4 * 4
        C = self.prm.noc
        per = {"mask": 1, "dudv": 2, "rec": 8 if self.prm.nop == 2 else 5}.get(name, C)
        buf = np.empty(pitch * li["h"] * per, np.float32)
        n = lib().ofdis_debug_get(self._h, name.encode(), frame, _ptr(buf), buf.size)
        if n < 0:
            raise OfdisError("debug_get(%s) failed: %d" % (name, n))
        if name in ("dudv", "rec"):
            return buf.reshape(li["h"], pitch, per)[:, :li["w"]]
        return buf.reshape(per, li["h"], pitch)[:, :, :li["w"]]

    def debug_div(self, a: np.ndarray, b: np.ndarray):
        """The stereo SOR's division b / a on the device: (q_fast, q_plain, unsafe) -- the SOR kernels' written-out
        IEEE division, the compiler's `/`, and where the kernels' range test sends the pair to the latter."""
        a = np.ascontiguousarray(a, np.float32).reshape(-1)
        b = np.ascontiguousarray(b, np.float32).reshape(-1)
        assert a.shape == b.shape
        q_fast, q_plain = np.empty_like(a), np.empty_like(a)
        unsafe = np.empty(a.shape, np.uint8)
        self._ck(lib().ofdis_debug_div(self._h, _ptr(a), _ptr(b), a.size, _ptr(q_fast), _ptr(q_plain), _ptr(unsafe)))
        return q_fast, q_plain, unsafe.astype(bool)

    def sor_div_fallbacks(self, reset: bool = False) -> int:
        """How often the stereo SOR redid work with the plain division since create or the last reset."""
        v = ctypes.c_ulonglong()
        self._ck(lib().ofdis_debug_sor_div_fallbacks(self._h, ctypes.byref(v), 1 if reset else 0))
        return v.value


# ---------------------------------------------------------------------------
# Reference-shaped classes (same names, same argument meaning).
# ---------------------------------------------------------------------------
class OFClass:
    """OFC::OFClass (oflow.h:84-111): all work happens in the constructor; the flow of
    level sc_l is written into `outflow` (numpy, (h, w, nop) float32)."""

    def __init__(self, im_ao, im_ao_dx, im_ao_dy, im_bo, im_bo_dx, im_bo_dy, imgpadding, outflow, initflow, width,
                 height, sc_f, sc_l, max_iter, min_iter, dp_thresh, dr_thresh, res_thresh, p_samp_s, patove, usefbcon,
                 costfct, noc, patnorm, usetvref, tv_alpha, tv_gamma, tv_delta, tv_innerit, tv_solverit, tv_sor,
                 verbosity, nop=2, device=0):
        prm = DisParams(sc_f=sc_f, sc_l=sc_l, max_iter=max_iter, min_iter=min_iter, dp_thresh=dp_thresh,
                        dr_thresh=dr_thresh, res_thresh=res_thresh, p_samp_s=p_samp_s, patove=patove,
                        usefbcon=int(usefbcon), costfct=costfct, noc=noc, patnorm=patnorm, usetvref=int(usetvref),
                        tv_alpha=tv_alpha, tv_gamma=tv_gamma, tv_delta=tv_delta, tv_innerit=tv_innerit,
                        tv_solverit=tv_solverit, tv_sor=tv_sor, verbosity=verbosity, nop=nop)
        ctx = Context(prm, width, height, imgpadding, 1, device)
        try:
            for lv in range(sc_l, sc_f + 1):
                if usefbcon:  # the backward grid's template gradients (oflow.cpp:193-197)
                    ctx.upload_level_fb(0, lv, im_ao[lv], im_ao_dx[lv], im_ao_dy[lv], im_bo[lv], im_bo_dx[lv], im_bo_dy[lv])
                else:
                    ctx.upload_level(0, lv, im_ao[lv], im_ao_dx[lv], im_ao_dy[lv], im_bo[lv])
            if initflow is not None:
                ctx.set_flow(0, sc_f + 1, initflow)
            ctx.run(1, use_initflow=initflow is not None)
            outflow[...] = ctx.get_flow(0, sc_l).reshape(outflow.shape)
        finally:
            ctx.close()


class PatGridClass:
    """OFC::PatGridClass (patchgrid.h:19-44) on one pyramid level of a Context."""

    def __init__(self, ctx: Context, level: int, frame: int = 0):
        self.ctx, self.level, self.frame = ctx, level, frame
        self._i0 = self._i1 = None
        self._from_coarser = False

    def InitializeGrid(self, im_ao, im_ao_dx, im_ao_dy):
        self._i0 = (im_ao, im_ao_dx, im_ao_dy)

    def SetTargetImage(self, im_bo, im_bo_dx=None, im_bo_dy=None):
        self._i1 = im_bo
        self.ctx.upload_level(self.frame, self.level, self._i0[0], self._i0[1], self._i0[2], im_bo)

    def InitializeFromCoarserOF(self, flow_prev):
        self.ctx.set_flow(self.frame, self.level + 1, flow_prev)
        self._from_coarser = True

    def Optimize(self):
        self.ctx.patgrid_optimize(self.level, self.frame, self.frame + 1, self._from_coarser)

    def AggregateFlowDense(self, flowout):
        self.ctx.patgrid_aggregate(self.level, self.frame, self.frame + 1)
        flowout[...] = self.ctx.get_flow(self.frame, self.level).reshape(flowout.shape)

    def GetNoPatches(self):
        li = self.ctx.level_info(self.level)
        return li["nopw"] * li["noph"]

    def GetNopw(self):
        return self.ctx.level_info(self.level)["nopw"]

    def GetNoph(self):
        return self.ctx.level_info(self.level)["noph"]

    def GetRefPatchPos(self, i):
        li = self.ctx.level_info(self.level)
        offw = (li["w"] - (li["nopw"] - 1) * li["steps"]) // 2
        offh = (li["h"] - (li["noph"] - 1) * li["steps"]) // 2
        x, y = divmod(i, li["noph"])
        return np.array([x * li["steps"] + offw, y * li["steps"] + offh], np.float32)

    def GetQuePatchDis(self, i):
        """pt_ref - pt_iter (patchgrid.h:44)."""
        p = self.ctx.get_patches(self.frame, self.level)["p"][i]
        ref = self.GetRefPatchPos(i)
        que = ref.copy()
        que[:len(p)] = ref[:len(p)] + p
        return ref - que


class VarRefClass:
    """OFC::VarRefClass (refine_variational.h:37-39): refines `flowout` in place."""

    def __init__(self, ctx: Context, level: int, flowout: np.ndarray, frame: int = 0):
        ctx.set_flow(frame, level, flowout)
        ctx.varref_refine(level, frame, frame + 1)
        flowout[...] = ctx.get_flow(frame, level).reshape(flowout.shape)
