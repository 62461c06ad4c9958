"""The point cloud after the fusion: DepthMapsData::MergeDepthMaps (libs/MVS/SceneDensify.cpp:1305-1366), EstimatePointColors
(libs/MVS/DepthMap.cpp:1429-1465), EstimatePointNormals (libs/MVS/DepthMap.cpp:1469-1519) with the exact k-NN search of the
normals, and Scene::PointCloudFilter (libs/MVS/SceneDensify.cpp:2226-2360), above the C-ABI (include/b200mvs.h); the kernels are
openmvs_b200/csrc/cloud_kernels.cu.  Re-exported by depth_estimator.  numpy inputs take the host forms, CUDA tensors the device
forms on the context kept per device."""
from __future__ import annotations

import ctypes as C
import dataclasses

import numpy as np

from . import lib as _lib
from .depth_estimator import PointCloud, _arg, _cuda_index, _device_context, _host, _is_torch, _point_cloud, _stream_handle


def _image_table(where: str, views, device, maps):
	"""the b200mvs_fuse_view table of the merge and point-cloud calls -> (table, keepalive).  maps: (key, dtype, channels) of the
	maps the call reads; a map's size is the size of the first map given (depth, else color)."""
	arr = (_lib.FuseView*len(views))()
	keep = []
	for i, v in enumerate(views):
		o = arr[i]
		size = None
		for key, dt, ch in maps:
			a = v.get(key)
			a = a.contiguous() if _is_torch(a) and a.is_cuda else _host(a, dt, device)
			keep.append(a)
			shape = (None, None)+ch if size is None else size+ch
			setattr(o, key, _arg(where, "views[%d].%s" % (i, key), a, dt, shape, device))
			if a is not None and size is None:
				size = tuple(a.shape[:2])
				o.height, o.width = size
		for name in ("K", "R", "C"):
			getattr(o, name)[:] = list(np.asarray(v[name], np.float64).ravel())
	return arr, keep


def MergeDepthMaps(views, bEstimateColor: bool = True, bEstimateNormal: bool = True) -> PointCloud:
	"""DepthMapsData::MergeDepthMaps (libs/MVS/SceneDensify.cpp:1305-1366), the nMinViewsFuse < 2 branch of DenseReconstruction:
	every depth != 0 of every depth-map becomes one point seen by its own image.  views: the dicts of FuseDepthMaps (depth, normal,
	color, K, R, C are read; depth is not modified).  numpy maps take b200mvs_merge_depth_maps (host code), CUDA tensors (every map
	on one device) b200mvs_merge_depth_maps_device on a context kept per device: the same cloud, bit for bit.  pointWeights is
	None (the reference leaves them empty); an image with a depth-map needs a colour map with bEstimateColor and a normal map
	with bEstimateNormal."""
	lib = _lib.load()
	first = next((v["depth"] for v in views if _is_torch(v.get("depth"))), None)
	device = None if first is None else _cuda_index(first)
	maps = (("depth", "float32", ()), ("normal", "float32", (3,)), ("color", "uint8", (3,)))
	arr, keep = _image_table("MergeDepthMaps", views, device, maps)
	prm = _lib.FuseParams(1, 0.01, 25.0, int(bool(bEstimateColor)), int(bool(bEstimateNormal)))
	cloud = C.c_void_p()
	if device is not None:
		ctx = _device_context(first.device)
		ctx._call("merge_depth_maps_device", arr, len(views), C.byref(prm), C.byref(cloud), _stream_handle(ctx.device), C.byref(ctx.stats))
	else:
		rc = lib.b200mvs_merge_depth_maps(arr, len(views), C.byref(prm), C.byref(cloud))
		if rc:
			raise _lib.B200MVSError("b200mvs_merge_depth_maps failed with status %d (bad view description)" % rc)
	try:
		return _point_cloud(lib, cloud, weights=False)
	finally:
		lib.b200mvs_pointcloud_free(cloud)


def _cloud_args(where: str, views, pointcloud, maps):
	"""the cloud and image arguments of EstimatePointColors / EstimatePointNormals -> (device index or None, context or None,
	points, offsets, ids, image table, keepalive).  CUDA points take the device form: the view lists are flattened and copied to
	the points' device."""
	pts = pointcloud.points
	device = _cuda_index(pts) if _is_torch(pts) and pts.is_cuda else None
	pv = pointcloud.pointViews
	lens = np.fromiter((len(v) for v in pv), np.int64, len(pv))
	off = np.zeros(len(pv)+1, np.uint32)
	if len(pv):
		off[1:] = np.cumsum(lens)
	ids = np.concatenate([np.asarray(v, np.uint32).ravel() for v in pv]) if int(lens.sum()) else np.zeros(1, np.uint32)
	if device is None:
		pts = _host(pts, np.float32)
	else:
		import torch
		off = torch.from_numpy(off).to(pts.device)
		ids = torch.from_numpy(ids.astype(np.int32)).to(pts.device)
	p = _arg(where, "pointcloud.points", pts, "float32", (None, 3), device)
	po = _arg(where, "pointcloud view offsets", off, ("uint32", "int32"), (len(pv)+1,), device)
	pi = _arg(where, "pointcloud view IDs", ids, ("uint32", "int32"), None, device)
	arr, keep = _image_table(where, views, device, maps)
	ctx = None if device is None else _device_context(pts.device)
	return device, ctx, (p, len(pv), po, pi, arr, len(views)), [pts, off, ids, keep]


def EstimatePointColors(views, pointcloud: PointCloud) -> PointCloud:
	"""MVS::EstimatePointColors (libs/MVS/DepthMap.cpp:1429-1465): fills pointcloud.colors ((n, 3) uint8) with the colour of each
	point's view of least depth, sampled bilinearly as the reference does (white without a view or outside the border).  views:
	the scene images as dicts with color ((h, w, 3) uint8, None: empty image), K, R, C.  numpy points take the host-buffer form;
	CUDA points (and colour maps on the same device) the device form, and colors is then a tensor."""
	lib = _lib.load()
	device, ctx, args, keep = _cloud_args("EstimatePointColors", views, pointcloud, (("color", "uint8", (3,)),))
	n = args[1]
	if device is None:
		colors = np.zeros((n, 3), np.uint8)
		ctx = _device_context(0)
		ctx._call("estimate_point_colors", *args, colors.ctypes.data, C.byref(ctx.stats))
	else:
		import torch
		colors = torch.empty((n, 3), dtype=torch.uint8, device=pointcloud.points.device)
		ctx._call("estimate_point_colors_device", *args, colors.data_ptr(), _stream_handle(ctx.device))
	pointcloud.colors = colors
	return pointcloud


def EstimatePointNormals(views, pointcloud: PointCloud, numNeighbors: int = 16) -> PointCloud:
	"""MVS::EstimatePointNormals (libs/MVS/DepthMap.cpp:1469-1519): fills pointcloud.normals ((n, 3) float32) with the PCA normal
	of each point's numNeighbors nearest points (exact search, ties to the lower index; DESIGN.md §5.6), turned towards the
	camera of its first view.  views: the scene images as dicts with K, R, C.  numpy points take the host-buffer form, CUDA
	points the device form (normals is then a tensor)."""
	lib = _lib.load()
	device, ctx, args, keep = _cloud_args("EstimatePointNormals", views, pointcloud, ())
	n = args[1]
	if device is None:
		normals = np.zeros((n, 3), np.float32)
		ctx = _device_context(0)
		ctx._call("estimate_point_normals", *args, int(numNeighbors), normals.ctypes.data, C.byref(ctx.stats))
	else:
		import torch
		normals = torch.empty((n, 3), dtype=torch.float32, device=pointcloud.points.device)
		ctx._call("estimate_point_normals_device", *args, int(numNeighbors), normals.data_ptr(), _stream_handle(ctx.device))
	pointcloud.normals = normals
	return pointcloud


def PointKNN(points, numNeighbors: int = 16):
	"""the exact neighbour search of EstimatePointNormals on an (n, 3) float32 CUDA tensor -> (n, min(numNeighbors, n)) int32
	tensor of point indices, ascending by (squared distance in double, index); every point is its own first neighbour unless
	an exact duplicate with a lower index precedes it"""
	import torch
	ptr = _arg("PointKNN", "points", points, "float32", (None, 3), _cuda_index(points))
	ctx = _device_context(points.device)
	n = points.shape[0]
	out = torch.empty((n, max(min(int(numNeighbors), n), 0)), dtype=torch.int32, device=points.device)
	ctx._call("point_knn_device", ptr, n, int(numNeighbors), out.data_ptr() if n else None, _stream_handle(ctx.device))
	return out


def PointCloudVisibility(views, pointcloud: PointCloud):
	"""The visibility counts of Scene::PointCloudFilter (libs/MVS/SceneDensify.cpp:2226-2360): for every point and every view of
	it, the cone from the view's camera centre through the point with a half-angle of one pixel classifies every point of the
	cloud, and each VISIBLE point at least 1 % farther (nearer) along the axis than the apex-to-point distance gains the size of
	its own view list (loses the size of the point's view list).  Exactly the counts of the single-threaded reference
	(DESIGN.md §5.7).  views: the scene images as dicts with K, R, C and their size, given as width and height or by a depth or
	colour map (only the size and the camera are read).  -> (n,) int32: a numpy array for numpy points (host-buffer form), a
	tensor on the points' device for CUDA points (device form)."""
	return _visibility("PointCloudVisibility", views, pointcloud)


def _visibility(where: str, views, pointcloud: PointCloud):
	rows = len(pointcloud.points) if hasattr(pointcloud.points, "__len__") else None
	if rows is not None and rows != len(pointcloud.pointViews):
		raise ValueError("%s: pointcloud.points must have one row per view list; got %d rows and %d lists" % (where, rows,
			len(pointcloud.pointViews)))
	device, ctx, args, keep = _cloud_args(where, views, pointcloud, ())
	table = args[4]
	for i, v in enumerate(views):
		if v.get("width") is not None and v.get("height") is not None:
			size = (v["height"], v["width"])
		else:
			m = next((v[k] for k in ("depth", "color") if v.get(k) is not None), None)
			if m is None:
				raise ValueError("%s: views[%d] needs width and height, or a depth or colour map to take them from" % (where, i))
			size = tuple(m.shape[:2])
		if not all(isinstance(s, (int, np.integer)) and 0 < int(s) < 2**31 for s in size):
			raise ValueError("%s: views[%d] width and height must be positive integers; got %r" % (where, i, size[::-1]))
		table[i].height, table[i].width = int(size[0]), int(size[1])
	n = args[1]
	if device is None:
		vis = np.zeros(n, np.int32)
		ctx = _device_context(0)
		ctx._call("point_cloud_visibility", *args, vis.ctypes.data, C.byref(ctx.stats))
	else:
		import torch
		vis = torch.empty(n, dtype=torch.int32, device=pointcloud.points.device)
		ctx._call("point_cloud_visibility_device", *args, vis.data_ptr(), _stream_handle(ctx.device))
	return vis


def PointCloudFilter(views, pointcloud: PointCloud, thRemove: int = 0) -> PointCloud:
	"""Scene::PointCloudFilter(thRemove) (libs/MVS/SceneDensify.cpp:2226-2360): the cloud without the points whose visibility
	count (PointCloudVisibility) is <= thRemove, in the order the reference's removal loop leaves them (from the last point down,
	each removed point replaced by the current last one: b200mvs_pointcloud_remove_order).  points, pointViews, pointWeights,
	colors, normals and projs are reordered alike, where present; a CUDA cloud stays on its device.  -> a new PointCloud."""
	if isinstance(thRemove, bool) or not isinstance(thRemove, (int, np.integer)) or not -2**31 <= int(thRemove) < 2**31:
		raise ValueError("PointCloudFilter: thRemove must be an int32 integer; got %r" % (thRemove,))
	vis = _visibility("PointCloudFilter", views, pointcloud)
	remove = vis <= int(thRemove)
	remove = np.ascontiguousarray(remove.cpu().numpy() if _is_torch(remove) else remove, np.uint8)
	n = len(remove)
	order = np.zeros(max(n, 1), np.uint32)
	kept = C.c_uint64()
	rc = _lib.load().b200mvs_pointcloud_remove_order(remove.ctypes.data, n, order.ctypes.data, C.byref(kept))
	if rc:
		raise _lib.B200MVSError("b200mvs_pointcloud_remove_order failed with status %d" % rc)
	order = order[:kept.value].astype(np.int64)

	def take(a):
		if a is None:
			return None
		if isinstance(a, list):
			return [a[k] for k in order]
		if _is_torch(a):
			import torch
			return a[torch.from_numpy(order).to(a.device)]
		return np.asarray(a)[order]
	return dataclasses.replace(pointcloud, points=take(pointcloud.points), pointViews=take(pointcloud.pointViews),
		pointWeights=take(pointcloud.pointWeights), colors=take(pointcloud.colors), normals=take(pointcloud.normals),
		projs=take(pointcloud.projs))
