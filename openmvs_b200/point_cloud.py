"""The point cloud after the fusion: DepthMapsData::MergeDepthMaps (libs/MVS/SceneDensify.cpp:1305-1366), EstimatePointColors
(libs/MVS/DepthMap.cpp:1429-1465) and EstimatePointNormals (libs/MVS/DepthMap.cpp:1469-1519), and the exact k-NN search of the
normals, above the C-ABI (include/b200mvs.h); the kernels are openmvs_b200/csrc/cloud_kernels.cu.  Re-exported by
depth_estimator.  numpy inputs take the host forms, CUDA tensors the device forms on the context kept per device."""
from __future__ import annotations

import ctypes as C

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
