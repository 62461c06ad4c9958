"""ctypes binding of include/b200mvs.h.  There is no CPU fallback: if the CUDA library is
missing or no GPU is present, calls raise."""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

ABI_VERSION = 7  # B200MVS_ABI_VERSION of include/b200mvs.h these structs mirror
SGM_MAX_LEVELS = 9  # B200MVS_SGM_MAX_LEVELS: entries of the level-size arrays of b200mvs_sgm_levels
SGM_MAX_PAIRS = 32  # B200MVS_SGM_MAX_PAIRS: pairs one b200mvs_sgm_fuse call takes
MAX_POINT_NEIGHBORS = 32  # B200MVS_MAX_POINT_NEIGHBORS: the largest numNeighbors of the point-normal and k-NN calls


class View(C.Structure):
	"""b200mvs_view"""
	_fields_ = [("image", C.c_void_p), ("width", C.c_int), ("height", C.c_int), ("stride_bytes", C.c_int),
		("K", C.c_double*9), ("R", C.c_double*9), ("C", C.c_double*3),
		("depth", C.c_void_p), ("dwidth", C.c_int), ("dheight", C.c_int), ("dstride_bytes", C.c_int),
		("Kd", C.c_double*9), ("Rd", C.c_double*9), ("Cd", C.c_double*3),
		("image8", C.c_void_p), ("channels8", C.c_int), ("bgr8", C.c_int), ("stride8_bytes", C.c_int)]


class Params(C.Structure):
	"""b200mvs_params"""
	_fields_ = [("nEstimationIters", C.c_int), ("nEstimationGeometricIters", C.c_int), ("nRandomIters", C.c_int),
		("nSubResolutionLevels", C.c_int),
		("fNCCThresholdKeep", C.c_float), ("fDescriptorMinMagnitudeThreshold", C.c_float),
		("fRandomDepthRatio", C.c_float), ("fRandomAngle1Range", C.c_float), ("fRandomAngle2Range", C.c_float),
		("fRandomSmoothDepth", C.c_float), ("fRandomSmoothNormal", C.c_float), ("fRandomSmoothBonus", C.c_float),
		("fEstimationGeometricWeight", C.c_float),
		("nSweepsPerIter", C.c_int), ("nPropagation", C.c_int), ("seed", C.c_uint32),
		("nPropagationFar", C.c_int), ("bSkipUnchanged", C.c_int), ("nEvalCap", C.c_int)]


class Debug(C.Structure):
	"""b200mvs_debug"""
	_fields_ = [("reserved0", C.c_int), ("reserved1", C.c_int), ("sgmAggregation", C.c_int), ("sgmCost", C.c_int),
		("reserved2", C.c_int), ("reserved3", C.c_int), ("reserved4", C.c_int), ("reserved5", C.c_int), ("reserved6", C.c_int),
		("reserved7", C.c_int), ("reserved8", C.c_int), ("reserved9", C.c_int), ("reserved", C.c_int*4)]


class Stats(C.Structure):
	"""b200mvs_stats"""
	_fields_ = [("ms_total", C.c_double), ("ms_device", C.c_double), ("bytes_h2d", C.c_uint64), ("bytes_d2h", C.c_uint64),
		("kernel_launches", C.c_int), ("levels", C.c_int),
		("ms_sweep_kernels", C.c_double), ("sweep_launches", C.c_int), ("tma_active", C.c_int)]


class Job(C.Structure):
	"""b200mvs_job"""
	_fields_ = [("views", C.POINTER(View)), ("nViews", C.c_int), ("dMin", C.c_float), ("dMax", C.c_float), ("nGeometricIter", C.c_int),
		("depth", C.c_void_p), ("normal", C.c_void_p), ("conf", C.c_void_p), ("viewsMap", C.c_void_p), ("status", C.c_int)]


class SgmPixel(C.Structure):
	"""b200mvs_sgm_pixel"""
	_fields_ = [("idx", C.c_uint64), ("dmin", C.c_int16), ("dmax", C.c_int16), ("reserved", C.c_int32)]


class SgmParams(C.Structure):
	"""b200mvs_sgm_params"""
	_fields_ = [("P1", C.c_int), ("P2", C.c_int), ("P2alpha", C.c_float), ("P2beta", C.c_float)]


class SgmPair(C.Structure):
	"""b200mvs_sgm_pair"""
	_fields_ = [("disparity", C.c_void_p), ("cost", C.c_void_p), ("width", C.c_int), ("height", C.c_int), ("subpixelSteps", C.c_int),
		("Q", C.c_double*16)]


class DMap(C.Structure):
	"""b200mvs_dmap"""
	_fields_ = [("depth", C.c_void_p), ("conf", C.c_void_p), ("width", C.c_int), ("height", C.c_int),
		("K", C.c_double*9), ("R", C.c_double*9), ("C", C.c_double*3)]


class FilterParams(C.Structure):
	"""b200mvs_filter_params"""
	_fields_ = [("nMinViews", C.c_int), ("nMinViewsAdjust", C.c_int), ("fDepthDiffThreshold", C.c_float), ("bAdjust", C.c_int)]


class FuseView(C.Structure):
	"""b200mvs_fuse_view"""
	_fields_ = [("width", C.c_int), ("height", C.c_int), ("depth", C.c_void_p), ("normal", C.c_void_p), ("conf", C.c_void_p),
		("color", C.c_void_p), ("K", C.c_double*9), ("R", C.c_double*9), ("C", C.c_double*3), ("neighbors", C.c_void_p),
		("nNeighbors", C.c_int), ("nSceneNeighbors", C.c_int)]


class FuseParams(C.Structure):
	"""b200mvs_fuse_params"""
	_fields_ = [("nMinViewsFuse", C.c_int), ("fDepthDiffThreshold", C.c_float), ("fNormalDiffThreshold", C.c_float),
		("bEstimateColor", C.c_int), ("bEstimateNormal", C.c_int)]


I, U, F, P, U64 = C.c_int, C.c_uint, C.c_float, C.c_void_p, C.c_uint64
IP, PP = C.POINTER(C.c_int), C.POINTER(C.c_void_p)
PView, PStats, PSgmParams, PDMap = C.POINTER(View), C.POINTER(Stats), C.POINTER(SgmParams), C.POINTER(DMap)

# name -> (restype, argtypes) of every function include/b200mvs.h declares, in header order; contexts, device buffers and
# streams are c_void_p (checked against the header's prototypes by tests/test_capi_symbols.py)
PROTOTYPES = {
	"b200mvs_create": (I, [I, PP]),
	"b200mvs_destroy": (I, [P]),
	"b200mvs_default_params": (None, [C.POINTER(Params)]),
	"b200mvs_set_params": (I, [P, C.POINTER(Params)]),
	"b200mvs_set_debug": (I, [P, C.POINTER(Debug)]),
	"b200mvs_get_schedule": (I, [C.POINTER(Params), I, IP, IP]),
	"b200mvs_abi_version": (I, []),
	"b200mvs_sizeof": (C.c_size_t, [I]),
	"b200mvs_set_ignore_mask": (I, [P, P, I, I, I, I]),
	"b200mvs_last_error": (C.c_char_p, [P]),
	"b200mvs_device_count": (I, []),
	"b200mvs_estimate": (I, [P, PView, I, F, F, I, P, P, P, P, PStats]),
	"b200mvs_estimate_async": (I, [P, PView, I, F, F, I, P, P, P, P]),
	"b200mvs_sync": (I, [P, PStats]),
	"b200mvs_estimate_batch": (I, [PP, I, C.POINTER(Job), I]),
	"b200mvs_estimate_device": (I, [P, PView, I, F, F, I, P, P, P, P, P, PStats]),
	"b200mvs_pm_pack": (I, [P, I, I, P, P, P, P]),
	"b200mvs_pm_unpack": (I, [P, I, I, P, P, P, P]),
	"b200mvs_pm_score": (I, [P, PView, I, F, F, P, P, P, P]),
	"b200mvs_pm_sweep": (I, [P, PView, I, F, F, P, I, I, I, P, P, P]),
	"b200mvs_pm_finalize": (I, [P, I, I, F, P, P, P, P, P, P]),
	"b200mvs_sgm_default_params": (None, [PSgmParams]),
	"b200mvs_sgm_match": (I, [P, P, P, P, I, I, P, U64, PSgmParams, P, P, PStats]),
	"b200mvs_sgm_match_device": (I, [P, P, P, P, I, I, P, U64, PSgmParams, I, P, P, P, P, P, PStats]),
	"b200mvs_sgm_cross_check_device": (I, [P, P, P, I, I, I, P]),
	"b200mvs_sgm_refine_device": (I, [P, P, P, P, I, I, P]),
	"b200mvs_sgm_levels": (I, [I, I, I, IP, IP, IP, IP, IP]),
	"b200mvs_sgm_match_hierarchical_device": (I, [P, P, P, P, P, I, I, P, I, I, P, P, I, I, I, I, PSgmParams, P, P, P, P]),
	"b200mvs_sgm_range_map_device": (I, [P, P, I, I, P, I, I, I, I, P, C.POINTER(U64), P]),
	"b200mvs_sgm_flip_direction_device": (I, [P, P, P, I, I, P]),
	"b200mvs_sgm_upscale_mask_device": (I, [P, P, I, I, P, I, I, P]),
	"b200mvs_sgm_extract_mask_device": (I, [P, P, P, I, I, I, P]),
	"b200mvs_sgm_filter_speckles_device": (I, [P, P, I, I, I, I, I, P]),
	"b200mvs_resize_area_u8_device": (I, [P, P, I, I, I, I, P, P]),
	"b200mvs_sgm_level_mask_device": (I, [P, P, I, I, I, I, P, P]),
	"b200mvs_sgm_pair_q": (I, [P, P, P, P, P, P, P, P]),
	"b200mvs_sgm_project_disparity_device": (I, [P, P, I, I, P, P, P, P]),
	"b200mvs_sgm_fuse_device": (I, [P, P, I, I, I, I, P, P, P, P, P]),
	"b200mvs_sgm_fuse": (I, [P, P, I, I, I, I, P, P, P, P, PStats]),
	"b200mvs_estimate_normal_map_device": (I, [P, P, I, I, P, P, P]),
	"b200mvs_filter_default_params": (None, [C.POINTER(FilterParams)]),
	"b200mvs_filter_depth_map": (I, [P, PDMap, PDMap, I, C.POINTER(FilterParams), F, F, P, P, IP, PStats]),
	"b200mvs_filter_depth_map_device": (I, [P, PDMap, PDMap, I, C.POINTER(FilterParams), F, F, P, P, P, P, IP, P]),
	"b200mvs_remove_small_segments": (I, [P, P, P, P, I, I, F, U, PStats]),
	"b200mvs_remove_small_segments_device": (I, [P, P, P, P, I, I, F, U, P]),
	"b200mvs_gap_interpolation": (I, [P, P, P, P, I, I, F, U, PStats]),
	"b200mvs_gap_interpolation_device": (I, [P, P, P, P, I, I, F, U, P]),
	"b200mvs_to_gray_device": (I, [P, P, I, I, I, I, I, P, I, P]),
	"b200mvs_scaled_size": (I, [I, I, F, IP, IP]),
	"b200mvs_scale_image_device": (I, [P, P, I, I, I, F, P, IP, P]),
	"b200mvs_fuse_default_params": (None, [C.POINTER(FuseParams)]),
	"b200mvs_fuse_depth_maps": (I, [C.POINTER(FuseView), I, C.POINTER(FuseParams), PP]),
	"b200mvs_fuse_depth_maps_device": (I, [P, C.POINTER(FuseView), I, C.POINTER(FuseParams), PP, P, PStats]),
	"b200mvs_fuse_round_stats": (I, [P, I, IP, IP, IP, P, P, P, P]),
	"b200mvs_pointcloud_size": (U64, [P]),
	"b200mvs_pointcloud_depths": (U64, [P]),
	"b200mvs_pointcloud_points": (C.POINTER(F), [P]),
	"b200mvs_pointcloud_normals": (C.POINTER(F), [P]),
	"b200mvs_pointcloud_colors": (C.POINTER(C.c_uint8), [P]),
	"b200mvs_pointcloud_view_offsets": (C.POINTER(C.c_uint32), [P]),
	"b200mvs_pointcloud_views": (C.POINTER(C.c_uint32), [P]),
	"b200mvs_pointcloud_weights": (C.POINTER(F), [P]),
	"b200mvs_pointcloud_projs": (C.POINTER(C.c_uint16), [P]),
	"b200mvs_pointcloud_free": (None, [P]),
	"b200mvs_merge_depth_maps": (I, [C.POINTER(FuseView), I, C.POINTER(FuseParams), PP]),
	"b200mvs_merge_depth_maps_device": (I, [P, C.POINTER(FuseView), I, C.POINTER(FuseParams), PP, P, PStats]),
	"b200mvs_estimate_point_colors": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, P, PStats]),
	"b200mvs_estimate_point_colors_device": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, P, P]),
	"b200mvs_estimate_point_normals": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, I, P, PStats]),
	"b200mvs_estimate_point_normals_device": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, I, P, P]),
	"b200mvs_point_knn_device": (I, [P, P, U64, I, P, P]),
	"b200mvs_point_cloud_visibility": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, P, PStats]),
	"b200mvs_point_cloud_visibility_device": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, P, P]),
	"b200mvs_pointcloud_remove_order": (I, [P, U64, P, C.POINTER(U64)]),
	"b200mvs_pointcloud_remove_order_device": (I, [P, P, U64, P, C.POINTER(U64), P]),
	"b200mvs_pointcloud_compact_device": (I, [P, P, U64, U64, P, P, P, P, P, P, P, P, P, P, P, P, P, P, C.POINTER(U64), P]),
	"b200mvs_point_cloud_outside_obb": (I, [P, U64, P, P, P, F, P]),
	"b200mvs_point_cloud_outside_obb_device": (I, [P, P, U64, P, P, P, F, P, P]),
	"b200mvs_point_cloud_min_views": (I, [P, U64, C.c_uint32, P]),
	"b200mvs_point_cloud_min_views_device": (I, [P, P, U64, C.c_uint32, P, P]),
	"b200mvs_estimate_roi": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, I, F, P, P, P, IP]),
	"b200mvs_estimate_roi_device": (I, [P, P, U64, P, P, C.POINTER(FuseView), I, I, F, P, P, P, IP, P]),
}
SYMBOLS = list(PROTOTYPES)

_LIB = None


def load(build_if_missing: bool = True):
	"""Load libb200mvs.so (building it in-tree when stale and nvcc is available)."""
	global _LIB
	if _LIB is not None:
		return _LIB
	path = _build.LIB_PATH
	if build_if_missing:
		# a stale library whose rebuild fails is NOT used: its struct layouts may differ from these bindings
		path = _build.build_extension()
	if not os.path.exists(path):
		raise RuntimeError("CUDA extension %s is missing: run __graft_entry__.build() (no CPU fallback exists)" % path)
	lib = C.CDLL(path)
	if not hasattr(lib, "b200mvs_abi_version") or lib.b200mvs_abi_version() != ABI_VERSION:
		raise RuntimeError("%s was built from another version of include/b200mvs.h (ABI %s, bindings %d): rebuild it" % (
			path, lib.b200mvs_abi_version() if hasattr(lib, "b200mvs_abi_version") else "?", ABI_VERSION))
	for name, (restype, argtypes) in PROTOTYPES.items():
		f = getattr(lib, name)
		f.restype, f.argtypes = restype, argtypes
	for what, T in enumerate((View, Params, Stats, Job, SgmPixel, SgmParams, DMap, FilterParams, Debug, SgmPair)):
		if lib.b200mvs_sizeof(what) != C.sizeof(T):
			raise RuntimeError("struct %s: library %d bytes, bindings %d bytes" % (T.__name__, lib.b200mvs_sizeof(what), C.sizeof(T)))
	_LIB = lib
	return lib


class B200MVSError(RuntimeError):
	pass


def check(lib, ctx, rc: int, what: str):
	if rc != 0:
		msg = lib.b200mvs_last_error(ctx).decode() if ctx else ""
		raise B200MVSError("%s failed with status %d: %s" % (what, rc, msg))
