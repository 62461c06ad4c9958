"""ctypes binding of tests/cpp/visibility_oracle.cpp, the exhaustive CPU restatement of Scene::PointCloudFilter: the visibility
counts of every (point, view) cone over every point, and the reference's literal removal loop.  Compiled once per session into
a temporary directory with -O2 -ffp-contract=off (each float operation rounded as written)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCE = os.path.join(HERE, "cpp", "visibility_oracle.cpp")
_LIB = None


def lib():
	global _LIB
	if _LIB is None:
		out = os.path.join(tempfile.mkdtemp(prefix="visibility_oracle_"), "libvisibility_oracle.so")
		subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-pthread", "-o", out, SOURCE])
		L = C.CDLL(out)
		P, U64, I = C.c_void_p, C.c_uint64, C.c_int
		L.vis_oracle.restype, L.vis_oracle.argtypes = I, [P, U64, P, P, I, P, P, P, I, P]
		L.vis_oracle_filter.restype, L.vis_oracle_filter.argtypes = U64, [P, U64, I, P]
		_LIB = L
	return _LIB


def flat(pointViews):
	"""per-point view lists -> (offsets (n+1,) uint32, IDs uint32)"""
	off = np.zeros(len(pointViews)+1, np.uint32)
	off[1:] = np.cumsum([len(v) for v in pointViews])
	ids = np.concatenate([np.asarray(v, np.uint32).ravel() for v in pointViews]) if off[-1] else np.zeros(1, np.uint32)
	return off, np.ascontiguousarray(ids, np.uint32)


def visibility(points, pointViews, views, threads=None):
	"""the counts of the single-threaded reference: points (n, 3) float32, pointViews per-point image IDs, views dicts with K, C
	and width (or a depth / colour map) -> (n,) int32"""
	pts = np.ascontiguousarray(points, np.float32)
	off, ids = flat(pointViews)
	K = np.ascontiguousarray([np.asarray(v["K"], np.float64).ravel() for v in views], np.float64)
	Cs = np.ascontiguousarray([np.asarray(v["C"], np.float64).ravel() for v in views], np.float64)
	W = np.array([v["width"] if v.get("width") is not None else (v["depth"] if v.get("depth") is not None else v["color"]).shape[1]
		for v in views], np.int32)
	out = np.zeros(len(pts), np.int32)
	lib().vis_oracle(pts.ctypes.data, len(pts), off.ctypes.data, ids.ctypes.data, len(views), K.ctypes.data, Cs.ctypes.data,
		W.ctypes.data, int(threads or os.cpu_count() or 1), out.ctypes.data)
	return out


def filter_order(vis, thRemove):
	"""the original indices of the kept points in the slots the reference's removal loop leaves them in"""
	vis = np.ascontiguousarray(vis, np.int32)
	order = np.zeros(max(len(vis), 1), np.uint32)
	k = lib().vis_oracle_filter(vis.ctypes.data, len(vis), int(thRemove), order.ctypes.data)
	return order[:k].copy()
