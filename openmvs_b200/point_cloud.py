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
from .depth_estimator import (PointCloud, _arg, _cloud_call, _cuda_index, _device_context, _host, _image_table, _is_torch,
	_stream_handle)


def MergeDepthMaps(views, bEstimateColor: bool = True, bEstimateNormal: bool = True) -> PointCloud:
	"""DepthMapsData::MergeDepthMaps (libs/MVS/SceneDensify.cpp:1305-1366), the nMinViewsFuse < 2 branch of DenseReconstruction:
	every depth != 0 of every depth-map becomes one point seen by its own image.  views: the dicts of FuseDepthMaps (depth, normal,
	color, K, R, C are read; depth is not modified).  numpy maps take b200mvs_merge_depth_maps (host code), CUDA tensors (every map
	on one device) b200mvs_merge_depth_maps_device on a context kept per device: the same cloud, bit for bit.  pointWeights is
	None (the reference leaves them empty); an image with a depth-map needs a colour map with bEstimateColor and a normal map
	with bEstimateNormal."""
	maps = (("depth", "float32", ()), ("normal", "float32", (3,)), ("color", "uint8", (3,)))
	return _cloud_call("MergeDepthMaps", "merge_depth_maps", views, maps, (1, 0.01, 25.0, bEstimateColor, bEstimateNormal))


def _per_point(where: str, name: str, views, pointcloud, maps, cols, dtype: str, extra=(), view_size=None):
	"""b200mvs_<name> of the points of pointcloud -> the (n,)+cols output of dtype: the host-buffer form on device 0's context for
	numpy points, a numpy array; the device form on the context of the points' device for CUDA points (the view lists are flattened
	and copied there), a tensor on that device.  extra: the int arguments between the image count and the output; view_size(where,
	i, view) -> (height, width) of each image in the table, where the call takes them from elsewhere than its maps."""
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
	for i, v in enumerate(views if view_size else ()):
		arr[i].height, arr[i].width = view_size(where, i, v)
	n = len(pv)
	args = (p, n, po, pi, arr, len(views)) + tuple(int(e) for e in extra)
	if device is None:
		out = np.zeros((n,)+cols, dtype)
		ctx = _device_context(0)
		ctx._call(name, *args, out.ctypes.data, C.byref(ctx.stats))
	else:
		import torch
		out = torch.empty((n,)+cols, dtype=getattr(torch, dtype), device=pts.device)
		ctx = _device_context(pts.device)
		ctx._call(name + "_device", *args, out.data_ptr(), _stream_handle(ctx.device))
	return out


def EstimatePointColors(views, pointcloud: PointCloud) -> PointCloud:
	"""MVS::EstimatePointColors (libs/MVS/DepthMap.cpp:1429-1465): fills pointcloud.colors ((n, 3) uint8) with the colour of each
	point's view of least depth, sampled bilinearly as the reference does (white without a view or outside the border).  views:
	the scene images as dicts with color ((h, w, 3) uint8, None: empty image), K, R, C.  numpy points take the host-buffer form;
	CUDA points (and colour maps on the same device) the device form, and colors is then a tensor."""
	pointcloud.colors = _per_point("EstimatePointColors", "estimate_point_colors", views, pointcloud, (("color", "uint8", (3,)),),
		(3,), "uint8")
	return pointcloud


def EstimatePointNormals(views, pointcloud: PointCloud, numNeighbors: int = 16) -> PointCloud:
	"""MVS::EstimatePointNormals (libs/MVS/DepthMap.cpp:1469-1519): fills pointcloud.normals ((n, 3) float32) with the PCA normal
	of each point's numNeighbors nearest points (exact search, ties to the lower index; DESIGN.md §5.6), turned towards the
	camera of its first view.  views: the scene images as dicts with K, R, C.  numpy points take the host-buffer form, CUDA
	points the device form (normals is then a tensor)."""
	pointcloud.normals = _per_point("EstimatePointNormals", "estimate_point_normals", views, pointcloud, (), (3,), "float32",
		(numNeighbors,))
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


def _view_size(where: str, i: int, v):
	"""the size of a view of the visibility counts: width and height, or the shape of a depth or colour map"""
	if v.get("width") is not None and v.get("height") is not None:
		size = (v["height"], v["width"])
	else:
		m = next((v[k] for k in ("depth", "color") if v.get(k) is not None), None)
		if m is None:
			raise ValueError("%s: views[%d] needs width and height, or a depth or colour map to take them from" % (where, i))
		size = tuple(m.shape[:2])
	if not all(isinstance(s, (int, np.integer)) and 0 < int(s) < 2**31 for s in size):
		raise ValueError("%s: views[%d] width and height must be positive integers; got %r" % (where, i, size[::-1]))
	return int(size[0]), int(size[1])


def _visibility(where: str, views, pointcloud: PointCloud):
	rows = len(pointcloud.points) if hasattr(pointcloud.points, "__len__") else None
	if rows is not None and rows != len(pointcloud.pointViews):
		raise ValueError("%s: pointcloud.points must have one row per view list; got %d rows and %d lists" % (where, rows,
			len(pointcloud.pointViews)))
	return _per_point(where, "point_cloud_visibility", views, pointcloud, (), (), "int32", view_size=_view_size)


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
