"""CPU restatements of the point-cloud tail of Scene::DenseReconstruction — TEST INFRASTRUCTURE ONLY.

  merge_depth_maps       DepthMapsData::MergeDepthMaps     libs/MVS/SceneDensify.cpp:1305-1366
  estimate_point_colors  EstimatePointColors               libs/MVS/DepthMap.cpp:1429-1465
  knn                    the neighbourhoods of EstimatePointNormals, brute force (DESIGN.md §5.6)
  estimate_point_normals EstimatePointNormals              libs/MVS/DepthMap.cpp:1469-1519

Plain numpy, with the float32 / float64 operations in the reference's order, one elementwise operation at a time (numpy does
not contract them), so the merge and the colours are bit-exact restatements.  Only tests/ and scripts/ may import this module;
the product path is b200mvs_merge_depth_maps / b200mvs_estimate_point_* (openmvs_b200/csrc/cloud_host.cu).
parity unpinned: the reference has no golden vectors for these functions, and the normals come from CGAL, which is not in the
reference tree (DESIGN.md §3, §8).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def projection_matrix(K, R, C):
	"""AssembleProjectionMatrix (libs/MVS/Camera.cpp:173-180), P = [K R | -K R C] summed left to right in double"""
	K = np.asarray(K, np.float64).reshape(3, 3); R = np.asarray(R, np.float64).reshape(3, 3); C = np.asarray(C, np.float64).reshape(3)
	M = np.zeros((3, 3))
	for i in range(3):
		for j in range(3):
			M[i, j] = (K[i, 0]*R[0, j] + K[i, 1]*R[1, j]) + K[i, 2]*R[2, j]
	P = np.zeros((3, 4))
	P[:, :3] = M
	for i in range(3):
		P[i, 3] = (M[i, 0]*-C[0] + M[i, 1]*-C[1]) + M[i, 2]*-C[2]
	return P


def image_to_world(K, R, C, x, y, depth):
	"""Camera::TransformPointI2W(Point3(x, y, depth)) (libs/MVS/Camera.h:339-356) on arrays, double, summed left to right"""
	K = np.asarray(K, np.float64).reshape(3, 3); R = np.asarray(R, np.float64).reshape(3, 3); C = np.asarray(C, np.float64).reshape(3)
	z = np.asarray(depth, np.float32).astype(np.float64)
	cx = ((np.asarray(x, np.float64)-K[0, 2])*z)/K[0, 0]
	cy = ((np.asarray(y, np.float64)-K[1, 2])*z)/K[1, 1]
	return np.stack([((R[0, a]*cx + R[1, a]*cy) + R[2, a]*z) + C[a] for a in range(3)], -1)


def normal_to_world(R, n):
	"""R^T n (libs/MVS/DepthMap.cpp:137-146 with a normal map): double sums of the float normal, float result"""
	R = np.asarray(R, np.float64).reshape(3, 3)
	n = np.asarray(n, np.float32).astype(np.float64)
	return np.stack([(R[0, a]*n[..., 0] + R[1, a]*n[..., 1]) + R[2, a]*n[..., 2] for a in range(3)], -1).astype(F32)


def merge_depth_maps(views, estimate_color=True, estimate_normal=True):
	"""SceneDensify.cpp:1325-1360: images in index order (a view takes part when it has a depth-map), pixels in raster order,
	every depth != 0 one point seen by its image.  views: dicts with depth (h, w) float32 or None, normal (h, w, 3), color
	(h, w, 3) uint8, K, R, C.  -> dict(points (n, 3) f32, views (n,) u32, projs (n, 2) u16, colors, normals, nDepths)"""
	pts, ids, projs, cols, nrms = [], [], [], [], []
	for i, v in enumerate(views):
		d = v.get("depth")
		if d is None:
			continue
		d = np.asarray(d, np.float32)
		ys, xs = np.nonzero(d != 0)          # row-major: raster order
		pts.append(image_to_world(v["K"], v["R"], v["C"], xs, ys, d[ys, xs]).astype(F32))
		ids.append(np.full(len(xs), i, np.uint32))
		projs.append(np.stack([xs, ys], -1).astype(np.uint16))
		if estimate_color:
			cols.append(np.asarray(v["color"], np.uint8)[ys, xs])
		if estimate_normal:
			nrms.append(normal_to_world(v["R"], np.asarray(v["normal"], np.float32)[ys, xs]))
	cat = lambda a, shape, dt: np.concatenate(a) if a else np.zeros(shape, dt)
	points = cat(pts, (0, 3), F32)
	return dict(points=points, views=cat(ids, (0,), np.uint32), projs=cat(projs, (0, 2), np.uint16),
		colors=cat(cols, (0, 3), np.uint8) if estimate_color else None, normals=cat(nrms, (0, 3), F32) if estimate_normal else None,
		nDepths=len(points))


def _px_mul(p, v):
	"""TPixel<uint8_t> * float (libs/Common/Types.h:1965): float product truncated to uint8"""
	return (F32(v)*np.asarray(p, np.uint8).astype(F32)).astype(F32).astype(np.uint8)


def _px_add(a, b):
	"""TPixel<uint8_t> + TPixel<uint8_t> (libs/Common/Types.h:1970): a uint8 sum"""
	return ((a.astype(np.int32) + b.astype(np.int32)) & 0xFF).astype(np.uint8)


def sample(image, x, y):
	"""TImage<Pixel8U>::sample (libs/Common/Types.inl:2273-2281) at float32 arrays x, y (inside the 1-pixel border)"""
	x = np.asarray(x, F32); y = np.asarray(y, F32)
	lx = x.astype(np.int32); ly = y.astype(np.int32)
	fx = (x - lx.astype(F32)).astype(F32); fx1 = (F32(1) - fx).astype(F32)
	fy = (y - ly.astype(F32)).astype(F32); fy1 = (F32(1) - fy).astype(F32)
	w = lambda a: a[:, None]
	top = _px_add(_px_mul(image[ly, lx], w(fx1)), _px_mul(image[ly, lx+1], w(fx)))
	bottom = _px_add(_px_mul(image[ly+1, lx], w(fx1)), _px_mul(image[ly+1, lx+1], w(fx)))
	return _px_add(_px_mul(top, w(fy1)), _px_mul(bottom, w(fy)))


def project_point_p(P, points):
	"""Camera::ProjectPointP (libs/MVS/Camera.h:308-320) of float32 points (n, 3): float components of double row sums, then
	INVERT (libs/Common/Types.h:1234, FINV_ZERO for 0) -> float32 (x, y)"""
	X = np.asarray(points, F32).reshape(-1, 3).astype(np.float64)
	q = [(((P[r, 0]*X[:, 0] + P[r, 1]*X[:, 1]) + P[r, 2]*X[:, 2]) + P[r, 3]).astype(F32) for r in range(3)]
	with np.errstate(divide="ignore"):
		inv = np.where(q[2] == 0, F32(1000000.0), (F32(1)/q[2]).astype(F32)).astype(F32)
	return (q[0]*inv).astype(F32), (q[1]*inv).astype(F32)


def estimate_point_colors(points, offsets, ids, images):
	"""DepthMap.cpp:1433-1462.  points (n, 3) float32; the views of point i are ids[offsets[i]:offsets[i+1]]; images: dicts with
	color ((h, w, 3) uint8 or None: empty), K, R, C.  -> (n, 3) uint8"""
	points = np.asarray(points, F32)
	n = len(points)
	offsets = np.asarray(offsets, np.int64); ids = np.asarray(ids, np.int64)
	Ps = [projection_matrix(im["K"], im["R"], im["C"]) for im in images]
	has = np.array([im.get("color") is not None for im in images], bool)
	X = points.astype(np.float64)
	# Camera::PointDepth (libs/MVS/Camera.cpp:112-115) of every view, the least one strictly, from REAL(FLT_MAX)
	best = np.full(n, float(np.finfo(F32).max)); bv = np.full(n, -1, np.int64)
	lens = offsets[1:] - offsets[:-1]
	for j in range(int(lens.max()) if n else 0):
		live = np.nonzero(lens > j)[0]
		v = ids[offsets[live]+j]
		live, v = live[has[v]], v[has[v]]
		P = np.stack([Ps[k][2] for k in v]) if len(v) else np.zeros((0, 4))
		d = ((P[:, 0]*X[live, 0] + P[:, 1]*X[live, 1]) + P[:, 2]*X[live, 2]) + P[:, 3]
		upd = best[live] > d
		best[live[upd]] = d[upd]; bv[live[upd]] = v[upd]
	out = np.full((n, 3), 255, np.uint8)
	for k, im in enumerate(images):
		sel = np.nonzero(bv == k)[0]
		if not len(sel):
			continue
		x, y = project_point_p(Ps[k], points[sel])
		img = np.asarray(im["color"], np.uint8)
		h, w = img.shape[:2]
		# isInsideWithBorder<float,1> (libs/Common/Types.h:1649-1651)
		ok = (x >= F32(1)) & (y >= F32(1)) & (x <= F32(w-2)) & (y <= F32(h-2))
		if ok.any():
			out[sel[ok]] = sample(img, x[ok], y[ok])
	return out


def knn(points, k, chunk=256):
	"""per point the min(k, n) points with the least (squared distance in double, index), itself included, by brute force.
	-> (n, min(k, n)) int64"""
	X = np.asarray(points, F32).astype(np.float64)
	n = len(X)
	k = min(k, n)
	out = np.zeros((n, k), np.int64)
	for s in range(0, n, chunk):
		q = X[s:s+chunk]
		dx = X[None, :, 0] - q[:, None, 0]; dy = X[None, :, 1] - q[:, None, 1]; dz = X[None, :, 2] - q[:, None, 2]
		d2 = (dx*dx + dy*dy) + dz*dz
		part = np.argpartition(d2, k-1, axis=1)[:, :k] if k < n else np.tile(np.arange(n), (len(q), 1))
		dp = np.take_along_axis(d2, part, 1)
		order = np.lexsort((part, dp), axis=-1)
		out[s:s+len(q)] = np.take_along_axis(part, order, 1)
		# a row with more points at its k-th distance than fit: every point at or inside it, ties resolved by index
		for r in np.nonzero((d2 <= dp.max(1)[:, None]).sum(1) > k)[0]:
			cand = np.nonzero(d2[r] <= dp[r].max())[0]
			out[s+r] = cand[np.lexsort((cand, d2[r, cand]))[:k]]
	return out


def estimate_point_normals(points, offsets, ids, Cs, nbr):
	"""DESIGN.md §5.6: the scatter matrix of each point's neighbours nbr (n, k) in double, the eigenvector of its least eigenvalue
	(numpy.linalg.eigh), cast to float, and turned towards Cast<float>(C) of the point's first view in float
	(libs/MVS/DepthMap.cpp:1511-1515).  Cs: (nImages, 3) camera centres.  nbr may have fewer rows than there are points: the
	normals of the first len(nbr) points.  -> (normals (len(nbr), 3) f32, eigenvalues (len(nbr), 3) ascending)"""
	X = np.asarray(points, F32).astype(np.float64)
	P = np.asarray(points, F32)[:len(nbr)]
	nb = X[np.asarray(nbr)]
	c = nb.sum(1)/nb.shape[1]
	d = nb - c[:, None]
	A = np.einsum("nki,nkj->nij", d, d)
	w, V = np.linalg.eigh(A)
	v = V[:, :, 0]
	v = v/np.linalg.norm(v, axis=1, keepdims=True)
	nf = v.astype(F32)
	Cf = np.asarray(Cs, np.float64).astype(F32)[np.asarray(ids, np.int64)[np.asarray(offsets, np.int64)[:-1]]]
	dv = (Cf - P).astype(F32)
	dot = ((nf[:, 0]*dv[:, 0]).astype(F32) + (nf[:, 1]*dv[:, 1]).astype(F32)).astype(F32) + (nf[:, 2]*dv[:, 2]).astype(F32)
	nf[dot < 0] = -nf[dot < 0]
	return nf, w
