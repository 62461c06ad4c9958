"""The point-cloud removals on the device against their host forms and the CPU oracle (oracle/removal_oracle.py): the removal
order (pointer jumping) on the masks of the CPU test and at 10^7 points, the compaction against a numpy gather, the ROI mask and
EstimateROI bit for bit, and the chain FuseDepthMaps -> EstimateROI -> RemovePointsOutside -> colours -> normals ->
RemoveMinViews on a 12-view scene, device against host and oracle."""
import copy
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from openmvs_b200 import lib as L, synth  # noqa: E402
from openmvs_b200.depth_estimator import (EstimatePointColors, EstimatePointNormals, EstimateROI, FuseDepthMaps, PointCloud,  # noqa: E402
	RemoveMinViews, RemovePointsOutside, _device_context, _stream_handle)
from oracle import point_cloud_oracle as PO, removal_oracle as R  # noqa: E402
from test_point_cloud_removal_oracle import cloud, literal_order, masks, ring, rotated_box, face_points  # noqa: E402


def _ctx():
	return _device_context(0)


def device_order(remove):
	remove = torch.from_numpy(np.ascontiguousarray(remove, np.uint8)).cuda()
	n = remove.numel()
	order = torch.full((max(n, 1),), -1, dtype=torch.int32, device="cuda")
	kept = C.c_uint64(12345)
	_ctx()._call("pointcloud_remove_order_device", remove.data_ptr() if n else None, n, order.data_ptr(), C.byref(kept),
		_stream_handle(0))
	return order[:kept.value].cpu().numpy().astype(np.int64), kept.value


def test_remove_order_device_equals_the_loop():
	for m in masks():
		got, k = device_order(m)
		assert list(got) == literal_order(m), m.astype(int)


def test_remove_order_device_at_ten_million_points():
	lib = L.load()
	rng = np.random.default_rng(3)
	n = 10**7
	for density in (0.001, 0.3, 0.97):
		m = (rng.random(n) < density).astype(np.uint8)
		order = np.zeros(n, np.uint32)
		kept = C.c_uint64()
		assert lib.b200mvs_pointcloud_remove_order(m.ctypes.data, n, order.ctypes.data, C.byref(kept)) == 0
		got, k = device_order(m)
		assert k == kept.value and np.array_equal(got, order[:k].astype(np.int64))
	# a long chain: a removed block followed by a shorter kept tail, scaled up
	m = (np.arange(n) < (3*n)//5).astype(np.uint8)
	assert np.array_equal(device_order(m)[0], R.remove_order(m))


def _compact(order, n, pts, nrm, col, off, views, weights, projs):
	T = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()
	d = dict(order=T(order.astype(np.uint32).view(np.int32)), pts=T(pts), nrm=T(nrm), col=T(col), off=T(off.view(np.int32) if off is not None else None),
		views=T(views.view(np.int32) if views is not None else None), w=T(weights), pj=T(projs.view(np.int16) if projs is not None else None))
	k = len(order)
	total = int(off[-1]) if off is not None else 0
	out = dict(pts=torch.zeros((k, 3), dtype=torch.float32, device="cuda") if pts is not None else None,
		nrm=torch.zeros((k, 3), dtype=torch.float32, device="cuda") if nrm is not None else None,
		col=torch.zeros((k, 3), dtype=torch.uint8, device="cuda") if col is not None else None,
		off=torch.zeros(k+1, dtype=torch.int32, device="cuda") if off is not None else None,
		views=torch.zeros(max(total, 1), dtype=torch.int32, device="cuda") if off is not None else None,
		w=torch.zeros(max(total, 1), dtype=torch.float32, device="cuda") if weights is not None else None,
		pj=torch.zeros(max(2*total, 2), dtype=torch.int16, device="cuda") if projs is not None else None)
	p = lambda t: None if t is None or t.numel() == 0 else t.data_ptr()
	nv = C.c_uint64(99)
	_ctx()._call("pointcloud_compact_device", p(d["order"]), k, n, p(d["pts"]), p(d["nrm"]), p(d["col"]), p(d["off"]), p(d["views"]),
		p(d["w"]), p(d["pj"]), p(out["pts"]), p(out["nrm"]), p(out["col"]), p(out["off"]), p(out["views"]), p(out["w"]), p(out["pj"]),
		C.byref(nv), _stream_handle(0))
	return {key: None if t is None else t.cpu().numpy() for key, t in out.items()}, nv.value


@pytest.mark.parametrize("fields", ["all", "no weights", "points only", "no lists"])
def test_compact_device_equals_a_numpy_gather(fields):
	rng = np.random.default_rng(5)
	n = 5000
	lens = rng.integers(0, 5, n)   # empty lists included
	off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
	views = rng.integers(0, 12, int(off[-1])).astype(np.uint32)
	weights = rng.random(int(off[-1])).astype(np.float32)
	projs = rng.integers(0, 65535, 2*int(off[-1])).astype(np.uint16)
	pts = rng.normal(size=(n, 3)).astype(np.float32)
	nrm = rng.normal(size=(n, 3)).astype(np.float32)
	col = rng.integers(0, 256, (n, 3)).astype(np.uint8)
	if fields == "no weights":
		weights = None
	if fields in ("points only", "no lists"):
		nrm = col = None
	if fields == "points only":
		off = views = weights = projs = None
	if fields == "no lists":
		pts = None
	remove = rng.random(n) < 0.4
	order = R.remove_order(remove)
	got, nv = _compact(order, n, pts, nrm, col, off, views, weights, projs)
	for key, a in (("pts", pts), ("nrm", nrm), ("col", col)):
		assert (got[key] is None) if a is None else np.array_equal(got[key], a[order])
	if off is None:
		assert nv == 0
		return
	new_off = np.concatenate([[0], np.cumsum(lens[order])])
	assert nv == new_off[-1] and np.array_equal(got["off"], new_off)
	src = np.concatenate([np.arange(off[i], off[i+1]) for i in order])
	assert np.array_equal(got["views"][:nv].astype(np.uint32), views[src])
	if weights is not None:
		assert np.array_equal(got["w"][:nv], weights[src])
	assert np.array_equal(got["pj"][:2*nv].view(np.uint16).reshape(-1, 2), projs.reshape(-1, 2)[src])


@pytest.mark.parametrize("border", [0.0, 1.25, -0.05])
def test_roi_mask_device_equals_the_oracle(border):
	rng = np.random.default_rng(2)
	for seed in range(4):
		rot, pos, ext = rotated_box(seed)
		P = np.concatenate([face_points(rot, pos, ext, border), rng.normal(scale=2, size=(100000, 3)).astype(np.float32),
			np.array([[np.nan, 0, 0], [np.inf, 0, 0]], np.float32)])
		pc = PointCloud(torch.from_numpy(np.ascontiguousarray(P)).cuda(), [np.zeros(0, np.uint32)]*len(P), None)
		box = [np.ascontiguousarray(a, np.float32).ravel() for a in (rot, pos, ext)]
		remove = torch.empty(len(P), dtype=torch.uint8, device="cuda")
		_ctx()._call("point_cloud_outside_obb_device", pc.points.data_ptr(), len(P), *(b.ctypes.data for b in box), border,
			remove.data_ptr(), _stream_handle(0))
		assert np.array_equal(remove.cpu().numpy(), R.outside_obb(P, rot, pos, ext, border))


def _images(cams):
	return [dict(K=K, R=Rm, C=C_, valid=v) for K, Rm, C_, v in cams]


@pytest.mark.parametrize("n", [5, 6])
def test_estimate_roi_device_equals_host_and_oracle(n):
	cams = ring(n) + [(ring(1)[0][0], np.eye(3), np.array([9.0, 9, 9]), False)]
	pts, off, ids = cloud(20000, cams[:n])
	pv = [ids[off[i]:off[i+1]] for i in range(len(off)-1)]
	for mode, scale in ((2, 1.1), (1, 1.0), (0, 1.1)):
		want = R.estimate_roi(pts, off, ids, cams, mode, scale)
		host = EstimateROI(_images(cams), PointCloud(pts, pv, None), mode, scale)
		dev = EstimateROI(_images(cams), PointCloud(torch.from_numpy(pts).cuda(), pv, None), mode, scale)
		if want is None:
			assert host is None and dev is None
			continue
		for got in (host, dev):
			for a, b in zip((got.rot, got.pos, got.ext), want):
				assert np.array_equal(np.asarray(a).ravel(), np.asarray(b).ravel())


def _scene_views(w, h, n, seed=0):
	sc = synth.make_scene(w, h, n, step_deg=5.0)
	rng = np.random.RandomState(seed)
	views = []
	for i, v in enumerate(sc.views):
		d = v.depth_gt.astype(np.float32)*(1+2e-3*rng.randn(h, w)).astype(np.float32)
		d[rng.rand(h, w) < 0.1] = 0
		color = (np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1)
		nb = list(sc.neighbors(i, min(n-1, 4)))
		views.append(dict(depth=d, normal=v.normal_gt.astype(np.float32), conf=rng.rand(h, w).astype(np.float32), color=color,
			K=np.asarray(v.K, np.float64), R=np.asarray(v.R, np.float64), C=np.asarray(v.C, np.float64), neighbors=nb,
			n_scene_neighbors=len(nb)))
	return views


def _chain(views, pc, border, device):
	"""EstimateROI(1), RemovePointsOutside(border), EstimatePointColors, EstimatePointNormals, RemoveMinViews(3)"""
	images = [dict(K=v["K"], R=v["R"], C=v["C"], color=torch.from_numpy(v["color"]).cuda() if device else v["color"]) for v in views]
	if device:
		pc = PointCloud(torch.from_numpy(np.ascontiguousarray(pc.points)).cuda(), pc.pointViews, pc.pointWeights, None, None, pc.projs)
	else:
		pc = PointCloud(pc.points, pc.pointViews, pc.pointWeights, None, None, pc.projs)
	obb = EstimateROI(images, pc, 1, 1.1)   # the synthetic rig faces one way: mode 2 leaves it unbounded
	assert obb is not None
	pc = RemovePointsOutside(pc, obb, border)
	pc = EstimatePointColors(images, pc)
	pc = EstimatePointNormals(images, pc)
	return obb, RemoveMinViews(pc, 3)


def _host_arrays(pc):
	a = lambda x: x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)
	return a(pc.points), a(pc.colors), a(pc.normals)


@pytest.mark.parametrize("border", [0.0, 0.9, -0.02])
def test_device_chain_equals_host_chain_and_oracle(border):
	views = _scene_views(160, 120, 12)
	fused = FuseDepthMaps([dict(v, depth=torch.from_numpy(v["depth"].copy()).cuda(), normal=torch.from_numpy(v["normal"]).cuda(),
		conf=torch.from_numpy(v["conf"]).cuda(), color=torch.from_numpy(v["color"]).cuda()) for v in copy.deepcopy(views)],
		bEstimateColor=False, bEstimateNormal=False)
	obb_h, host = _chain(views, fused, border, False)
	obb_d, dev = _chain(views, fused, border, True)
	for a, b in zip((obb_h.rot, obb_h.pos, obb_h.ext), (obb_d.rot, obb_d.pos, obb_d.ext)):
		assert np.array_equal(a, b)
	for a, b in zip(_host_arrays(host), _host_arrays(dev)):
		assert a.dtype == b.dtype and np.array_equal(a, b)
	for f in ("pointViews", "pointWeights", "projs"):
		assert all(np.array_equal(x, y) for x, y in zip(getattr(host, f), getattr(dev, f))) and len(getattr(host, f)) == len(getattr(dev, f))
	# the oracle: ROI, crop order, colours and the minimum-views cut
	off, ids = PO.flat(fused.pointViews)
	cams = [(v["K"], v["R"], v["C"], True) for v in views]
	want = R.estimate_roi(fused.points, off, ids, cams, 1, 1.1)
	assert all(np.array_equal(np.asarray(x).ravel(), np.asarray(y).ravel()) for x, y in zip((obb_h.rot, obb_h.pos, obb_h.ext), want))
	crop = R.remove_order(R.outside_obb(fused.points, *want, border))
	assert 0 < len(crop) <= len(fused.points)
	X = fused.points[crop]
	pv = [fused.pointViews[k] for k in crop]
	o2, i2 = PO.flat(pv)
	colors = PO.estimate_point_colors(X, o2, i2, [dict(color=v["color"], K=v["K"], R=v["R"], C=v["C"]) for v in views])
	keep = R.remove_order((np.diff(o2) < 3).astype(np.uint8))
	assert np.array_equal(host.points, X[keep]) and np.array_equal(host.colors, colors[keep])
	assert all(np.array_equal(a, pv[k]) for a, k in zip(host.pointViews, keep))
