"""The point-cloud removals on the fused and the merged cloud of 12 views at 1920x1080 (the clouds of
scripts/profile_point_cloud.py): device time of EstimateROI, the ROI mask, the removal order and the compaction, and the whole
crop on the device against the crop through the host (read the cloud back, mask and order on the host, gather with numpy,
upload it again).

  python scripts/profile_removal.py [--width W] [--height H] [--iters N] [--shrink S] [--out FILE]

The ROI is EstimateROI(1, 1.1) (the synthetic rig faces one way, so mode 2 leaves it unbounded) of the fused cloud with its extent multiplied by --shrink (fBorderROI), so that the crop removes
part of each cloud.  Device times are CUDA events around each call on device buffers (the removal order and the compaction
include their one read-back), best of --iters runs after one warm-up.  The host path is timed by the host clock from the first
read-back to the end of the upload, with a device synchronisation at both ends, best of --iters runs.  Both crops return the
same cloud, which the script checks.  Prints one JSON object with the card name and power limit (read-only nvidia-smi query)."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from profile_point_cloud import gpu_info, make_views, merge_raw, timed, to_device  # noqa: E402
from openmvs_b200 import lib as L  # noqa: E402
from openmvs_b200.depth_estimator import FuseDepthMaps, _device_context, _stream_handle  # noqa: E402
from openmvs_b200.point_cloud import _image_table  # noqa: E402


def fields_of(points, off, views, weights, projs, colors, normals):
	"""the device copy of a cloud: name -> contiguous CUDA tensor (None where the cloud has no such field)"""
	T = lambda a, dt=None: None if a is None else torch.from_numpy(np.ascontiguousarray(a if dt is None else a.view(dt))).cuda()
	return dict(points=T(points), off=T(off, np.int32), views=T(views, np.int32), weights=T(weights), projs=T(projs, np.int16),
		colors=T(colors), normals=T(normals))


def crop_device(ctx, d, box, border, out):
	"""mask, order and compaction on device buffers -> (kept points, kept views); the outputs are carved in `out`"""
	s = _stream_handle(ctx.device)
	n = d["points"].shape[0]
	p = lambda t: None if t is None else t.data_ptr()
	ctx._call("point_cloud_outside_obb_device", p(d["points"]), n, *(b.ctypes.data for b in box), border, p(out["remove"]), s)
	kept = C.c_uint64()
	ctx._call("pointcloud_remove_order_device", p(out["remove"]), n, p(out["order"]), C.byref(kept), s)
	nv = C.c_uint64()
	ctx._call("pointcloud_compact_device", p(out["order"]), kept.value, n, p(d["points"]), p(d["normals"]), p(d["colors"]), p(d["off"]),
		p(d["views"]), p(d["weights"]), p(d["projs"]), p(out["points"]), p(out["normals"]), p(out["colors"]), p(out["off"]),
		p(out["views"]), p(out["weights"]), p(out["projs"]), C.byref(nv), s)
	return kept.value, nv.value


def crop_host(lib, d, box, border):
	"""the same crop through the host: read the device cloud back, mask and order with the host forms, gather with numpy, upload"""
	torch.cuda.synchronize()
	h = {k: None if v is None else v.cpu().numpy() for k, v in d.items()}
	n = len(h["points"])
	remove = np.zeros(n, np.uint8)
	assert lib.b200mvs_point_cloud_outside_obb(h["points"].ctypes.data, n, *(b.ctypes.data for b in box), border, remove.ctypes.data) == 0
	order = np.zeros(n, np.uint32)
	kept = C.c_uint64()
	assert lib.b200mvs_pointcloud_remove_order(remove.ctypes.data, n, order.ctypes.data, C.byref(kept)) == 0
	order = order[:kept.value].astype(np.int64)
	off = h["off"].view(np.uint32).astype(np.int64)
	lens = np.diff(off)[order]
	new_off = np.concatenate([[0], np.cumsum(lens)])
	src = np.repeat(off[order] - new_off[:-1], lens) + np.arange(new_off[-1])
	g = dict(points=h["points"][order], off=new_off.astype(np.int32), views=h["views"][src],
		weights=None if h["weights"] is None else h["weights"][src], projs=None if h["projs"] is None else h["projs"].reshape(-1, 2)[src],
		colors=None if h["colors"] is None else h["colors"][order], normals=None if h["normals"] is None else h["normals"][order])
	up = {k: None if v is None else torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in g.items()}
	torch.cuda.synchronize()
	return up


def measure(ctx, lib, d, box, border, iters, images, nImages):
	n = d["points"].shape[0]
	total = d["views"].shape[0]
	dev = d["points"].device
	out = dict(remove=torch.empty(n, dtype=torch.uint8, device=dev), order=torch.empty(n, dtype=torch.int32, device=dev),
		points=torch.empty((n, 3), dtype=torch.float32, device=dev), off=torch.empty(n+1, dtype=torch.int32, device=dev),
		views=torch.empty(total, dtype=torch.int32, device=dev),
		weights=torch.empty(total, dtype=torch.float32, device=dev) if d["weights"] is not None else None,
		projs=torch.empty(2*total, dtype=torch.int16, device=dev),
		colors=torch.empty((n, 3), dtype=torch.uint8, device=dev) if d["colors"] is not None else None,
		normals=torch.empty((n, 3), dtype=torch.float32, device=dev) if d["normals"] is not None else None)
	s = _stream_handle(ctx.device)
	p = lambda t: None if t is None else t.data_ptr()
	row = dict(points=n, views=total)
	rot, pos, ext, bounded = np.zeros(9, np.float32), np.zeros(3, np.float32), np.zeros(3, np.float32), C.c_int()
	row["estimate_roi_ms"] = timed(lambda: ctx._call("estimate_roi_device", p(d["points"]), n, p(d["off"]), p(d["views"]), images,
		nImages, 1, 1.1, rot.ctypes.data, pos.ctypes.data, ext.ctypes.data, C.byref(bounded), s), iters)
	row["mask_ms"] = timed(lambda: ctx._call("point_cloud_outside_obb_device", p(d["points"]), n, *(b.ctypes.data for b in box), border,
		p(out["remove"]), s), iters)
	kept = C.c_uint64()
	row["order_ms"] = timed(lambda: ctx._call("pointcloud_remove_order_device", p(out["remove"]), n, p(out["order"]), C.byref(kept), s),
		iters)
	nv = C.c_uint64()
	row["compact_ms"] = timed(lambda: ctx._call("pointcloud_compact_device", p(out["order"]), kept.value, n, p(d["points"]),
		p(d["normals"]), p(d["colors"]), p(d["off"]), p(d["views"]), p(d["weights"]), p(d["projs"]), p(out["points"]), p(out["normals"]),
		p(out["colors"]), p(out["off"]), p(out["views"]), p(out["weights"]), p(out["projs"]), C.byref(nv), s), iters)
	row["kept"] = kept.value
	row["device_crop_ms"] = timed(lambda: crop_device(ctx, d, box, border, out), iters)
	best = float("inf")
	for _ in range(iters):
		t0 = time.perf_counter()
		up = crop_host(lib, d, box, border)
		best = min(best, 1e3*(time.perf_counter() - t0))
	row["host_round_trip_ms"] = best
	k, nvk = crop_device(ctx, d, box, border, out)
	torch.cuda.synchronize()
	same = k == up["points"].shape[0] and torch.equal(out["points"][:k], up["points"]) and torch.equal(out["off"][:k+1], up["off"]) and \
		torch.equal(out["views"][:nvk], up["views"])
	for f in ("weights", "colors", "normals"):
		if up[f] is not None:
			same &= torch.equal(out[f][:k if f != "weights" else nvk], up[f])
	same &= torch.equal(out["projs"][:2*nvk], up["projs"].reshape(-1))
	row["device_equals_host"] = bool(same)
	return row


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--width", type=int, default=1920)
	ap.add_argument("--height", type=int, default=1080)
	ap.add_argument("--iters", type=int, default=3)
	ap.add_argument("--shrink", type=float, default=0.8)
	ap.add_argument("--out", default=None)
	a = ap.parse_args()
	name, power = gpu_info()
	lib = L.load()
	ctx = _device_context(0)
	views = make_views(a.width, a.height)
	dev = to_device(views)
	fused = FuseDepthMaps([dict(v) for v in dev])
	off = np.zeros(len(fused.pointViews)+1, np.uint32)
	off[1:] = np.cumsum([len(v) for v in fused.pointViews])
	ids = np.concatenate(fused.pointViews).astype(np.uint32)
	images, keep = _image_table("profile", [dict(K=v["K"], R=v["R"], C=v["C"]) for v in views], None, ())
	for i in range(len(views)):
		images[i].width, images[i].height = a.width, a.height
	fd = fields_of(fused.points, off, ids, np.concatenate(fused.pointWeights).astype(np.float32),
		np.concatenate(fused.projs).astype(np.uint16).ravel(), fused.colors, fused.normals)
	rot, pos, ext, bounded = np.zeros(9, np.float32), np.zeros(3, np.float32), np.zeros(3, np.float32), C.c_int()
	ctx._call("estimate_roi_device", fd["points"].data_ptr(), len(off)-1, fd["off"].data_ptr(), fd["views"].data_ptr(), images, len(views),
		1, 1.1, rot.ctypes.data, pos.ctypes.data, ext.ctypes.data, C.byref(bounded), _stream_handle(0))
	assert bounded.value, "EstimateROI found no ROI on the fused cloud"
	box = (rot, pos, ext)
	row = dict(gpu=name, power_limit=power, width=a.width, height=a.height, iters=a.iters, roi=dict(pos=pos.tolist(), ext=ext.tolist()),
		fBorderROI=a.shrink)
	row["fused"] = measure(ctx, lib, fd, box, a.shrink, a.iters, images, len(views))
	del fd
	torch.cuda.empty_cache()
	pts, moff, mids = merge_raw(ctx, dev)
	md = fields_of(pts, moff, mids, None, np.zeros(2*len(mids), np.uint16), None, None)
	row["merged"] = measure(ctx, lib, md, box, a.shrink, a.iters, images, len(views))
	print(json.dumps(row))
	if a.out:
		with open(a.out, "w") as f:
			json.dump(row, f, indent=1)


if __name__ == "__main__":
	main()
