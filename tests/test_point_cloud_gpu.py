"""MergeDepthMaps, EstimatePointColors and EstimatePointNormals on the device, against their host forms and the numpy oracle
(oracle/point_cloud_oracle.py): the merge and the colours bit for bit, the k-NN search index for index, the normals within the
tolerances of DESIGN.md §5.6; bad clouds are refused before any launch can fault."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from openmvs_b200 import lib, synth  # noqa: E402
from openmvs_b200.depth_estimator import (EstimatePointColors, EstimatePointNormals, FuseDepthMaps, MergeDepthMaps, PointCloud,  # noqa: E402
	PointKNN)
from oracle import point_cloud_oracle as PO  # noqa: E402


def _scene_views(w, h, n, noise, seed, drop=0.1, n_nb=4):
	"""noisy depth-maps of the synthetic scene with holes and a band of outliers, colour and camera-space normal maps"""
	sc = synth.make_scene(w, h, n, step_deg=5.0)
	rng = np.random.RandomState(seed)
	views = []
	for i, v in enumerate(sc.views):
		d = v.depth_gt.astype(np.float32)*(1+noise*rng.randn(h, w)).astype(np.float32)
		d[rng.rand(h, w) < drop] = 0
		d[h//3:h//3+2, :] *= np.float32(0.8)
		color = (np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1)
		color[..., 1] = rng.randint(0, 256, (h, w))
		nb = list(sc.neighbors(i, min(n-1, n_nb)))
		views.append(dict(depth=d, normal=v.normal_gt.astype(np.float32), conf=rng.rand(h, w).astype(np.float32), color=color,
			K=np.asarray(v.K, np.float64), R=np.asarray(v.R, np.float64), C=np.asarray(v.C, np.float64), neighbors=nb,
			n_scene_neighbors=len(nb)))
	return views


def _to_device(views):
	return [dict(v, **{k: torch.from_numpy(np.ascontiguousarray(v[k])).cuda() for k in ("depth", "normal", "conf", "color")
		if v.get(k) is not None}) for v in views]


def _flat(pc):
	lens = np.array([len(v) for v in pc.pointViews], np.int64)
	off = np.zeros(len(lens)+1, np.uint32); off[1:] = np.cumsum(lens)
	ids = np.concatenate(pc.pointViews) if len(lens) else np.zeros(0, np.uint32)
	return off, ids


# ---- MergeDepthMaps ----

def _check_merge(views, **kw):
	ph = MergeDepthMaps(copy.deepcopy(views), **kw)
	pd = MergeDepthMaps(_to_device(views), **kw)
	po = PO.merge_depth_maps(views, kw.get("bEstimateColor", True), kw.get("bEstimateNormal", True))
	assert len(ph.points) > 0 and ph.pointWeights is None and pd.pointWeights is None
	assert ph.nDepths == pd.nDepths == po["nDepths"] == len(po["points"])
	assert np.array_equal(pd.points, ph.points) and np.array_equal(ph.points, po["points"])
	for pc in (ph, pd):
		off, ids = _flat(pc)
		assert np.array_equal(off, np.arange(len(off))) and np.array_equal(ids, po["views"])
		assert np.array_equal(np.concatenate(pc.projs), po["projs"])
		for name in ("colors", "normals"):
			a, b = getattr(pc, name), po[name]
			assert (a is None) == (b is None) or (b is not None and len(b) == 0 and a is None), name
			if a is not None:
				assert np.array_equal(a, b), name
	return ph


@pytest.mark.parametrize("color,normal", [(True, True), (False, True), (True, False)])
def test_merge_equals_host_and_oracle(color, normal):
	views = _scene_views(64, 48, 5, 2e-3, 1)
	views[1]["depth"] = None                 # no depth-map
	views[3]["depth"][:] = 0                 # no depth
	views[2]["depth"][5, 7] = np.float32(-1.5)   # any value but 0 is a point
	_check_merge(views, bEstimateColor=color, bEstimateNormal=normal)


def test_merge_twelve_views_640x480():
	ph = _check_merge(_scene_views(640, 480, 12, 2e-3, 2))
	assert len(ph.points) > 1000000


def test_merge_refuses_a_missing_colour_or_normal_map():
	views = _scene_views(32, 24, 3, 2e-3, 3)
	for key, flag in (("color", "bEstimateColor"), ("normal", "bEstimateNormal")):
		bad = copy.deepcopy(views)
		bad[1][key] = None
		with pytest.raises(lib.B200MVSError, match="status 1"):
			MergeDepthMaps(bad)
		with pytest.raises(lib.B200MVSError, match="status 1"):
			MergeDepthMaps(_to_device(bad))
		MergeDepthMaps(_to_device(bad), **{flag: False})


# ---- EstimatePointColors ----

def _images(views):
	return [dict(color=v.get("color"), K=v["K"], R=v["R"], C=v["C"]) for v in views]


def _on_line(P, X, axis, value):
	"""float32 points next to X (a few ulps per coordinate) whose float projection has coordinate `axis` exactly `value`, and
	points whose projection lies one float step outside it"""
	steps = np.arange(-40, 41).astype(np.float32)
	axes = [np.float32(c) + steps*np.spacing(np.float32(c)) for c in X]
	cand = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
	proj = PO.project_point_p(P, cand)[axis]
	on = cand[proj == np.float32(value)]
	outside = np.nextafter(np.float32(value), np.float32(-np.inf if value < 10 else np.inf))
	off = cand[proj == outside]
	return on[:3], off[:3]


def test_colours_equal_the_oracle_on_a_fused_cloud_with_border_and_behind_points():
	views = _scene_views(96, 72, 5, 2e-3, 4)
	pc = FuseDepthMaps(copy.deepcopy(views))
	v0 = views[0]
	K, R, C = v0["K"], v0["R"], v0["C"]
	P = PO.projection_matrix(K, R, C)
	extra = []
	# points projecting exactly onto the border lines x = 1, x = W - 2, y = 1, y = H - 2 of isInsideWithBorder<float,1>, and one
	# float step outside them
	for axis, value, other in ((0, 1.0, 30.0), (0, 94.0, 40.0), (1, 1.0, 50.0), (1, 70.0, 20.0)):
		xy = (value, other) if axis == 0 else (other, value)
		X = PO.image_to_world(K, R, C, np.array([xy[0]]), np.array([xy[1]]), np.array([4.0], np.float32))[0].astype(np.float32)
		on, off = _on_line(P, X, axis, value)
		assert len(on) and len(off), (axis, value)
		assert np.all(PO.project_point_p(P, on)[axis] == np.float32(value))
		extra += list(on) + list(off)
	n_line = len(extra)
	extra.append(np.asarray(C) - 5*np.asarray(R)[2])           # behind image 0
	extra = np.asarray(extra, np.float32)
	pts = np.concatenate([pc.points, extra])
	pv = pc.pointViews + [np.array([0], np.uint32)]*(len(extra)-1) + [np.array([0, 2], np.uint32)]
	images = _images(views)
	images[3]["color"] = None                                   # an empty image
	cloud = PointCloud(points=pts, pointViews=pv, pointWeights=None)
	off, ids = _flat(cloud)
	want = PO.estimate_point_colors(pts, off, ids, images)
	assert (want == 255).all(1).sum() > 0 and (want != 255).any(1).sum() > 1000
	on_line = want[len(pc.points):len(pc.points)+n_line]
	assert (on_line != 255).any(1).sum() >= 4 and (on_line == 255).all(1).sum() >= 4   # inside on the lines, white beyond them
	EstimatePointColors(images, cloud)
	assert np.array_equal(cloud.colors, want)
	dcloud = PointCloud(points=torch.from_numpy(pts).cuda(), pointViews=pv, pointWeights=None)
	EstimatePointColors([dict(im, color=None if im["color"] is None else torch.from_numpy(im["color"]).cuda()) for im in images], dcloud)
	assert np.array_equal(dcloud.colors.cpu().numpy(), want)


# ---- k-NN and EstimatePointNormals ----

def _clouds():
	rng = np.random.RandomState(5)
	uniform = rng.rand(20000, 3).astype(np.float32)
	clusters = np.concatenate([rng.rand(10000, 3)*0.01, rng.rand(10000, 3)*10 + 20]).astype(np.float32)
	views = _scene_views(128, 96, 3, 2e-3, 6)
	surf = MergeDepthMaps(views, bEstimateColor=False, bEstimateNormal=False).points[::2][:20000]
	surf = (surf.astype(np.float64) + 1e5).astype(np.float32)
	dup = rng.rand(5000, 3).astype(np.float32)
	dup = np.concatenate([dup, dup[:2000], dup[:300]])
	small = rng.rand(11, 3).astype(np.float32)
	# the surface with a few far outliers, which the grid's robust extent leaves in its border cells
	far = (rng.randn(8, 3)*1e4).astype(np.float32)
	outliers = np.concatenate([surf[:10000] - np.float32(1e5), far, surf[10000:12000] - np.float32(1e5)])
	return dict(uniform=uniform, clusters=clusters, surface=surf, duplicates=dup, small=small, outliers=outliers)


CLOUDS = {}


def _cloud(name):
	if not CLOUDS:
		CLOUDS.update(_clouds())
		CLOUDS["oracle"] = {k: PO.knn(v, 32) for k, v in CLOUDS.items()}
	return CLOUDS[name], CLOUDS["oracle"][name]


@pytest.mark.parametrize("name", ["uniform", "clusters", "surface", "duplicates", "small", "outliers"])
def test_knn_equals_the_oracle(name):
	X, want = _cloud(name)
	for k in (1, 16, 32):
		got = PointKNN(torch.from_numpy(X).cuda(), k).cpu().numpy()
		assert got.shape == (len(X), min(k, len(X)))
		assert np.array_equal(got, want[:, :min(k, len(X))]), (name, k)


@pytest.mark.parametrize("name", ["uniform", "clusters", "surface", "duplicates", "small", "outliers"])
def test_normals_match_the_oracle(name):
	X, nbr = _cloud(name)
	n = len(X)
	rng = np.random.RandomState(7)
	Cs = (X.mean(0) + rng.randn(4, 3)*50).astype(np.float64)
	pv = [np.array(sorted(set(rng.randint(0, 4, 1+i % 3).tolist())), np.uint32) for i in range(n)]
	images = [dict(K=np.eye(3), R=np.eye(3), C=c) for c in Cs]
	off, ids = _flat(PointCloud(X, pv, None))
	for k in (16, 32) if name != "small" else (16,):
		kk = min(k, n)
		want, w = PO.estimate_point_normals(X, off, ids, Cs, nbr[:, :kk])
		host = EstimatePointNormals(images, PointCloud(X, pv, None), k).normals
		dev = EstimatePointNormals(images, PointCloud(torch.from_numpy(X).cuda(), pv, None), k).normals.cpu().numpy()
		assert np.array_equal(host, dev)
		assert np.isfinite(dev).all() and np.all(np.abs(np.linalg.norm(dev.astype(np.float64), axis=1) - 1) <= 1e-6)
		gap = (w[:, 1] - w[:, 0]) >= 1e-4*w[:, 2]
		a, b = dev.astype(np.float64), want.astype(np.float64)
		angle = np.arctan2(np.linalg.norm(np.cross(a, b), axis=1), np.abs(np.einsum("ij,ij->i", a, b)))   # well conditioned near 0
		assert np.all(angle[gap] <= 1e-5), (name, angle[gap].max())
		Cf = Cs.astype(np.float32)[ids[off[:-1]]].astype(np.float64)
		dv = Cf - X.astype(np.float64)
		sure = gap & (np.abs(np.einsum("ij,ij->i", want.astype(np.float64), dv)) > 1e-6*np.linalg.norm(dv, axis=1))
		assert np.array_equal(np.sign(np.einsum("ij,ij->i", dev[sure].astype(np.float64), dv[sure])),
			np.sign(np.einsum("ij,ij->i", want[sure].astype(np.float64), dv[sure])))
		if name in ("uniform", "surface"):
			assert gap.mean() > 0.9


def test_knn_on_the_fused_full_hd_cloud():
	views = _scene_views(1920, 1080, 12, 2e-3, 8, n_nb=9)
	pc = FuseDepthMaps(_to_device(views))
	X = torch.from_numpy(pc.points).cuda()
	assert len(X) > 2000000
	got = PointKNN(X, 16)
	rng = np.random.RandomState(9)
	Xd = X.double()
	for q in rng.choice(len(X), 500, replace=False):
		d = Xd - Xd[q]
		d2 = (d[:, 0]*d[:, 0] + d[:, 1]*d[:, 1]) + d[:, 2]*d[:, 2]
		order = torch.sort(d2, stable=True).indices[:16]
		assert torch.equal(got[q].long(), order), q


# ---- bad input ----

def test_bad_clouds_are_refused():
	rng = np.random.RandomState(10)
	X = rng.rand(1000, 3).astype(np.float32)
	pv = [np.array([i % 2], np.uint32) for i in range(1000)]
	images = [dict(K=np.eye(3), R=np.eye(3), C=np.zeros(3), color=np.zeros((8, 8, 3), np.uint8))]*2
	nan = X.copy(); nan[17, 1] = np.nan
	empty = list(pv); empty[5] = np.zeros(0, np.uint32)
	far = list(pv); far[9] = np.array([2], np.uint32)
	for dev in (False, True):
		T = (lambda a: torch.from_numpy(a).cuda()) if dev else (lambda a: a)
		ims = [dict(im, color=T(im["color"])) for im in images]
		for pts, views, k in ((nan, pv, 16), (X, empty, 16), (X, far, 16), (X, pv, 0), (X, pv, 33)):
			with pytest.raises(lib.B200MVSError, match="status 1"):
				EstimatePointNormals(ims, PointCloud(T(pts), views, None), k)
		with pytest.raises(lib.B200MVSError, match="status 1"):
			EstimatePointColors(ims, PointCloud(T(X), far, None))
	for k in (0, 33):
		with pytest.raises(lib.B200MVSError, match="status 1"):
			PointKNN(torch.from_numpy(X).cuda(), k)
	with pytest.raises(lib.B200MVSError, match="status 1"):
		PointKNN(torch.from_numpy(nan).cuda(), 16)
	# a view table given as NULL with views to read: refused in every form of the C-ABI
	import ctypes as C
	from openmvs_b200.depth_estimator import _device_context
	from openmvs_b200.point_cloud import _image_table
	ctx = _device_context(0)
	arr, keep = _image_table("test", images, None, ())
	off = np.arange(1001, dtype=np.uint32)
	out = np.zeros((1000, 3), np.float32)
	for name, extra in (("estimate_point_normals", (16, out.ctypes.data, None)), ("estimate_point_colors", (out.ctypes.data, None))):
		with pytest.raises(lib.B200MVSError, match="status 1"):
			ctx._call(name, X.ctypes.data, 1000, off.ctypes.data, None, arr, 2, *extra)
	dX, doff, dout = torch.from_numpy(X).cuda(), torch.from_numpy(off.astype(np.int32)).cuda(), torch.zeros((1000, 3), device="cuda")
	for name, extra in (("estimate_point_normals_device", (16, dout.data_ptr(), None)), ("estimate_point_colors_device", (dout.data_ptr(), None))):
		with pytest.raises(lib.B200MVSError, match="status 1"):
			ctx._call(name, dX.data_ptr(), 1000, doff.data_ptr(), None, arr, 2, *extra)
	# the context still works after the refusals
	assert PointKNN(torch.from_numpy(X).cuda(), 4).shape == (1000, 4)
	torch.cuda.synchronize()
