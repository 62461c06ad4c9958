"""CPU restatements of the point-cloud removals (DESIGN.md §5.8), in numpy and plain Python where that is exact: the order
cList::RemoveAt leaves after RFOREACH(i) if (remove[i]) RemovePoint(i) (libs/Common/List.h:1630-1636), the remove mask of
PointCloud::RemovePointsOutside with DenseReconstruction's fBorderROI (libs/Common/OBB.inl:388-400, SceneDensify.cpp:1728), and
Scene::EstimateROI (libs/MVS/Scene.cpp:1652-1740).  Float steps are numpy float32 scalars or arrays (one rounding per operation,
no FMA), double steps Python floats, and tanf / asinf are the C library's, as the reference calls them."""
from __future__ import annotations

import ctypes as C
import ctypes.util

import numpy as np

f32 = np.float32
_LIBM = C.CDLL(ctypes.util.find_library("m"))
for _name in ("tanf", "asinf"):
	getattr(_LIBM, _name).restype = C.c_float
	getattr(_LIBM, _name).argtypes = [C.c_float]


def remove_order(remove):
	"""the kept original indices in the order the removal loop leaves them, by the chain formulation the device resolves: step t
	removes the t-th removed slot from the top and takes tail slot j = n-1-t, which holds point j when j is kept and otherwise
	what the earlier step s(j) = #{removed slots > j} moved"""
	remove = np.asarray(remove).astype(bool).ravel()
	n = len(remove)
	P = np.concatenate([[0], np.cumsum(remove)]).astype(np.int64)   # P[i] = #{removed slots < i}
	m = int(P[n])
	value = np.zeros(m, np.int64)
	for t in range(m):
		j = n-1-t
		s = m - P[j] - 1 if remove[j] else t
		value[t] = value[s] if s < t else j
	order = np.arange(n-m, dtype=np.int64)
	for k in np.flatnonzero(remove[:n-m]):
		order[k] = value[m - P[k] - 1]
	return order


def roi_extent(ext, fBorderROI):
	"""OBB3f(obb).EnlargePercent(b) for b > 0 (ext * b), Enlarge(-b) for b < 0 (ext + -b), the box itself for 0"""
	ext = np.asarray(ext, f32)
	b = f32(fBorderROI)
	return ext*b if b > 0 else ext + (-b) if b < 0 else ext.copy()


def outside_obb(points, rot, pos, ext, fBorderROI=0.0):
	"""!OBB3f::Intersects(X) per point -> uint8: d = rot (X - pos) in float, each row summed r0 + (r1 + r2) (Eigen's order for
	three terms); inside when |d| <= ext on every axis"""
	X = np.asarray(points, f32).reshape(-1, 3)
	R = np.asarray(rot, f32).reshape(3, 3)
	d = X - np.asarray(pos, f32)
	e = roi_extent(ext, fBorderROI)
	inside = np.ones(len(X), bool)
	for a in range(3):
		v = R[a, 0]*d[:, 0] + (R[a, 1]*d[:, 1] + R[a, 2]*d[:, 2])
		inside &= np.abs(v) <= e[a]
	return (~inside).astype(np.uint8)


def _median(v):
	"""cList::GetMedian of floats: the middle value, or the float mean of the two middle values"""
	v = sorted(f32(x) for x in v)
	h = len(v) >> 1
	return v[h] if len(v) % 2 else (v[h-1] + v[h]) / f32(2)


def _depth_row(K, R, C_):
	"""the third row of AssembleProjectionMatrix's P = [K R | -K R C] (Camera::PointDepth), each sum left to right in double"""
	K = np.asarray(K, np.float64).reshape(3, 3); R = np.asarray(R, np.float64).reshape(3, 3); C_ = np.asarray(C_, np.float64).ravel()
	M = [(float(K[2, 0])*float(R[0, j]) + float(K[2, 1])*float(R[1, j])) + float(K[2, 2])*float(R[2, j]) for j in range(3)]
	return M + [(M[0]*-float(C_[0]) + M[1]*-float(C_[1])) + M[2]*-float(C_[2])]


def _key(x):
	"""the order of the bounds: -0 below +0"""
	u = np.asarray(x, f32).view(np.uint32).astype(np.int64)
	return np.where(u & 0x80000000, -(u & 0x7FFFFFFF) - 1, u)


def estimate_roi(points, offsets, views, cameras, nEstimateROI=2, scale=1.1):
	"""Scene::EstimateROI -> (rot, pos, ext) float32 arrays, or None for an unbounded scene.  cameras: per image (K, R, C, valid)."""
	if nEstimateROI == 0 or len(points) == 0:
		return None
	valid = [i for i, c in enumerate(cameras) if c[3]]
	if len(valid) < 3:
		return None
	Cs = [np.asarray(cameras[i][2], np.float64).ravel() for i in valid]
	Rs = [np.asarray(cameras[i][1], np.float64).reshape(3, 3) for i in valid]
	center = [float(_median([f32(c[a]) for c in Cs])) for a in range(3)]
	mean = []
	for a in range(3):
		s = f32(0)
		for R in Rs:
			s = f32(s + f32(R[2, a]))
		mean.append(float(s / f32(len(valid))))
	length = f32(np.sqrt(mean[0]*mean[0] + mean[1]*mean[1] + mean[2]*mean[2]))
	if not abs(length) < f32(0.0001):
		mean = [m / float(length) for m in mean]
	if length > f32(np.sqrt(2.0))/f32(2) and nEstimateROI == 2:
		return None

	def distance(C_, X):
		r = [X[0]-C_[0], X[1]-C_[1], X[2]-C_[2]]
		return f32(np.sqrt(r[0]*r[0] + r[1]*r[1] + r[2]*r[2]))
	shift = f32(_LIBM.tanf(_LIBM.asinf(float(min(max(length, f32(0)), f32(0.999)))))) * _median([distance(c, center) for c in Cs])
	scene = [center[a] + float(shift)*mean[a] for a in range(3)]
	Ps = [_depth_row(*c[:3]) for c in cameras]
	radius = None
	for i, c in zip(valid, Cs):
		p = Ps[i]
		if p[0]*scene[0] + p[1]*scene[1] + p[2]*scene[2] + p[3] <= 0 and nEstimateROI == 2:
			return None
		d = distance(c, scene)
		radius = d if radius is None else max(radius, d)
	lim = float(f32(radius*f32(2)))
	X = np.asarray(points, f32).reshape(-1, 3)
	off = np.asarray(offsets, np.int64)
	views = np.asarray(views, np.int64)[:off[-1]]
	x = X.astype(np.float64)[np.repeat(np.arange(len(X)), np.diff(off))]   # one row per view entry
	P = np.asarray(Ps, np.float64).reshape(-1, 4)[views]
	depth = ((P[:, 0]*x[:, 0] + P[:, 1]*x[:, 1]) + P[:, 2]*x[:, 2]) + P[:, 3]
	hit = np.asarray([bool(c[3]) for c in cameras], bool)[views] & (depth < lim)
	core = np.bincount(np.repeat(np.arange(len(X)), np.diff(off))[hit], minlength=len(X)) > 0
	if not core.any():
		return None
	Y = X[core]
	lo = np.array([Y[np.argmin(_key(Y[:, a])), a] for a in range(3)], f32)
	hi = np.array([Y[np.argmax(_key(Y[:, a])), a] for a in range(3)], f32)
	delta = (hi - lo) * (f32(scale) - f32(1)) / f32(2)
	mn, mx = lo - delta, hi + delta
	return np.eye(3, dtype=f32), (mx + mn) * f32(0.5), (mx - mn) / f32(2)
