"""The point-cloud tail on 12 views at 1920x1080 with 9 neighbours each: MergeDepthMaps (device form), EstimatePointColors,
EstimatePointNormals (k = 16) and the visibility counts of PointCloudFilter on the fused and on the merged cloud.

  python scripts/profile_point_cloud.py [--width W] [--height H] [--iters N] [--subset M] [--out FILE]

The depth-maps are those of scripts/profile_fuse.py, fused on the device.  Prints one JSON object: the cloud sizes; the device
time of the merge (its events, without the read-back of the cloud), of the colours and of the normals (CUDA events around the
call on device buffers, which includes its checks' read-back), best of --iters runs after one warm-up, on the fused cloud, the
merged cloud and the fused cloud with 16 far outliers; the normals split into grid build (checks, bounding box, sample, keys,
sort, cells), k-NN and PCA from the kernel times under torch.profiler, each the best of --iters profiled runs after a warm-up;
the visibility counts' device time (CUDA events around the call on device buffers), best of --iters runs after one warm-up, with
its split into checks, binning (query sort, per-view keys, sorts, cell starts, gather) and queries (binned and exhaustive) from
the kernel times under torch.profiler, and the queries (entries of the view lists) per second; the numpy ORACLE's time for the
normals of --subset points (brute-force k-NN and PCA, scaled per point), which is not the reference (CGAL); and the card name and power limit (read-only nvidia-smi query)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmvs_b200 import synth  # noqa: E402
from openmvs_b200.depth_estimator import FuseDepthMaps, _device_context, _stream_handle  # noqa: E402
from openmvs_b200.point_cloud import _image_table  # noqa: E402
from oracle import point_cloud_oracle as PO  # noqa: E402


def gpu_info():
	try:
		out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
		name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
		return name, power
	except Exception as e:  # noqa: BLE001
		return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def make_views(W, H, n=12, n_nb=9, seed=0):
	"""the depth-maps of scripts/profile_fuse.py: ground truth, 0.2 % noise, 10 % holes, a band of outliers"""
	sc = synth.make_scene(W, H, n, step_deg=5.0)
	rng = np.random.RandomState(seed)
	views = []
	for i, v in enumerate(sc.views):
		d = v.depth_gt.astype(np.float32)*(1+2e-3*rng.randn(H, W)).astype(np.float32)
		d[rng.rand(H, W) < 0.1] = 0
		d[H//3:H//3+2, :] *= np.float32(0.8)
		nb = list(sc.neighbors(i, n_nb))
		color = (np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1)
		views.append(dict(depth=d, normal=v.normal_gt.astype(np.float32), conf=rng.rand(H, W).astype(np.float32), color=color,
			K=v.K, R=v.R, C=v.C, neighbors=nb, n_scene_neighbors=len(nb)))
	return views


def to_device(views):
	return [dict(v, **{k: torch.from_numpy(np.ascontiguousarray(v[k])).cuda() for k in ("depth", "normal", "conf", "color")}) for v in views]


def flat(pointViews):
	"""per-point view lists -> (offsets, IDs)"""
	off = np.zeros(len(pointViews)+1, np.int64)
	off[1:] = np.cumsum(np.fromiter((len(v) for v in pointViews), np.int64, len(pointViews)))
	return off, np.concatenate(pointViews)


def merge_raw(ctx, dev):
	"""b200mvs_merge_depth_maps_device without the per-point lists of MergeDepthMaps -> (points, offsets, IDs)"""
	lib = ctx._lib
	maps = (("depth", "float32", ()), ("normal", "float32", (3,)), ("color", "uint8", (3,)))
	arr, keep = _image_table("profile", dev, torch.cuda.current_device(), maps)
	cloud = C.c_void_p()
	ctx._call("merge_depth_maps_device", arr, len(dev), None, C.byref(cloud), _stream_handle(ctx.device), C.byref(ctx.stats))
	try:
		n = int(lib.b200mvs_pointcloud_size(cloud))
		get = lambda fn, count: np.ctypeslib.as_array(fn(cloud), shape=(count,)).copy()
		return (get(lib.b200mvs_pointcloud_points, 3*n).reshape(-1, 3), get(lib.b200mvs_pointcloud_view_offsets, n+1),
			get(lib.b200mvs_pointcloud_views, n))
	finally:
		lib.b200mvs_pointcloud_free(cloud)


def timed(fn, iters):
	"""best device time in ms of fn() over iters runs after one warm-up"""
	best = float("inf")
	for it in range(iters+1):
		a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
		torch.cuda.synchronize()
		a.record(); fn(); b.record()
		torch.cuda.synchronize()
		if it > 0:
			best = min(best, a.elapsed_time(b))
	return best


def split(fn, iters):
	"""device ms of the normals' grid build (the checks, bounding box and sample, keys, sort, cells, and the call's memsets of its
	check words and cell ranges: the only memsets in the window), k-NN and PCA kernels, each the best of iters runs under
	torch.profiler after one warm-up run"""
	from torch.profiler import ProfilerActivity, profile
	fn(); torch.cuda.synchronize()
	best = {"grid": float("inf"), "knn": float("inf"), "pca": float("inf")}
	for _ in range(iters):
		with profile(activities=[ProfilerActivity.CUDA]) as prof:
			fn(); torch.cuda.synchronize()
		out = {"grid": 0.0, "knn": 0.0, "pca": 0.0}
		for e in prof.key_averages():
			name, ms = e.key, e.device_time_total/1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total/1000.0
			if "k_knn" in name:
				out["knn"] += ms
			elif "k_pca" in name:
				out["pca"] += ms
			elif any(s in name for s in ("k_bbox", "k_check_views", "k_sample", "k_keys", "k_cells", "RadixSort", "Memset", "memset")):
				out["grid"] += ms
		best = {k: min(best[k], out[k]) for k in best}
	return {k: round(v, 3) for k, v in best.items()}


def split_visibility(fn, iters):
	"""device ms of the visibility call's checks, binning and query kernels, each the best of iters profiled runs after a warm-up"""
	from torch.profiler import ProfilerActivity, profile
	fn(); torch.cuda.synchronize()
	keys = ("checks", "binning", "queries", "exhaustive")
	best = dict.fromkeys(keys, float("inf"))
	for _ in range(iters):
		with profile(activities=[ProfilerActivity.CUDA]) as prof:
			fn(); torch.cuda.synchronize()
		out = dict.fromkeys(keys, 0.0)
		for e in prof.key_averages():
			name, ms = e.key, e.device_time_total/1000.0 if hasattr(e, "device_time_total") else e.cuda_time_total/1000.0
			if "k_vis_query" in name:
				out["queries"] += ms
			elif "k_vis_exhaustive" in name:
				out["exhaustive"] += ms
			elif any(s in name for s in ("k_vis_entries", "k_vis_starts", "k_vis_keys", "k_vis_gather", "RadixSort", "Onesweep")):
				out["binning"] += ms
			elif any(s in name for s in ("k_check_views", "k_bbox", "Memset", "memset")):
				out["checks"] += ms
		best = {k: min(best[k], out[k]) for k in keys}
	return {k: round(v, 3) for k, v in best.items()}


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--width", type=int, default=1920)
	ap.add_argument("--height", type=int, default=1080)
	ap.add_argument("--iters", type=int, default=3)
	ap.add_argument("--subset", type=int, default=200)
	ap.add_argument("--out", default=None)
	a = ap.parse_args()
	name, power = gpu_info()
	views = make_views(a.width, a.height)
	dev = to_device(views)
	row = {"size": [a.width, a.height], "views": len(views), "neighbors": 9}
	fused = FuseDepthMaps(to_device(views))
	ctx = _device_context(torch.device("cuda", torch.cuda.current_device()))
	merged, ms = None, []
	for it in range(a.iters+1):
		merged = merge_raw(ctx, dev)
		ms.append(ctx.stats.ms_device)
	row["ms_merge_device"] = min(ms[1:])
	fused = (fused.points, *flat(fused.pointViews))
	arr, keep = _image_table("profile", dev, 0, (("color", "uint8", (3,)),))
	stream = _stream_handle(ctx.device)
	# the fused cloud with 16 far outliers (1000 times the scene's extent away), one view each
	rng = np.random.RandomState(1)
	far = (fused[0].mean(0) + rng.randn(16, 3)*1000*np.ptp(fused[0], 0)).astype(np.float32)
	outliers = (np.concatenate([fused[0], far]), np.concatenate([fused[1], fused[1][-1] + np.arange(1, 17)]),
		np.concatenate([fused[2], np.zeros(16, fused[2].dtype)]))
	for label, (points, off, ids) in (("fused", fused), ("merged", merged), ("fused_outliers", outliers)):
		n = len(points)
		pts = torch.from_numpy(points).cuda()
		doff = torch.from_numpy(off.astype(np.int32)).cuda()
		ids = torch.from_numpy(ids.astype(np.int32)).cuda()
		colors = torch.empty((n, 3), dtype=torch.uint8, device="cuda")
		normals = torch.empty((n, 3), dtype=torch.float32, device="cuda")
		args = (pts.data_ptr(), n, doff.data_ptr(), ids.data_ptr(), arr, len(dev))
		row["points_"+label] = n
		row["ms_colors_"+label] = timed(lambda: ctx._call("estimate_point_colors_device", *args, colors.data_ptr(), stream), a.iters)
		run = lambda: ctx._call("estimate_point_normals_device", *args, 16, normals.data_ptr(), stream)
		row["ms_normals_"+label] = timed(run, a.iters)
		row["normals_split_ms_"+label] = split(run, a.iters)
		if label == "fused_outliers":
			continue
		vis = torch.empty(n, dtype=torch.int32, device="cuda")
		run = lambda: ctx._call("point_cloud_visibility_device", *args, vis.data_ptr(), stream)
		row["ms_visibility_"+label] = timed(run, a.iters)
		row["visibility_split_ms_"+label] = split_visibility(run, a.iters)
		row["visibility_queries_"+label] = int(off[-1])
		row["visibility_queries_per_s_"+label] = int(off[-1])/(row["ms_visibility_"+label]/1000.0)
		v = vis.cpu().numpy()
		row["visibility_removed_at_0_"+label] = int((v <= 0).sum())
	# the numpy oracle on a subset: brute force over the whole fused cloud for --subset queries, then PCA
	X = fused[0]
	rng = np.random.RandomState(0)
	q = rng.choice(len(X), min(a.subset, len(X)), replace=False)
	t = time.perf_counter()
	Xd = X.astype(np.float64)
	nbr = np.zeros((len(q), 16), np.int64)
	for i, j in enumerate(q):
		d = Xd - Xd[j]
		d2 = (d[:, 0]*d[:, 0] + d[:, 1]*d[:, 1]) + d[:, 2]*d[:, 2]
		p = np.argpartition(d2, 15)[:16]
		nbr[i] = p[np.lexsort((p, d2[p]))]
	# the queries first, then the whole cloud, so that the neighbour indices stay valid
	off = np.arange(len(q)+1, dtype=np.uint32)
	PO.estimate_point_normals(np.concatenate([X[q], X]), off, np.zeros(len(q), np.uint32), np.zeros((1, 3)), nbr + len(q))
	row["oracle_normals_ms_per_point"] = (time.perf_counter()-t)*1000.0/len(q)
	row["oracle_normals_s_estimated_fused"] = row["oracle_normals_ms_per_point"]*len(X)/1000.0
	row["oracle_subset"] = len(q)
	row["gpu"], row["power_limit"] = name, power
	print(json.dumps(row))
	if a.out:
		with open(a.out, "w") as f:
			json.dump(row, f, indent=1)


if __name__ == "__main__":
	main()
