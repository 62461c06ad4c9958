"""The entry points of the point-cloud calls (MergeDepthMaps, FuseDepthMaps, EstimatePointColors, EstimatePointNormals, PointKNN and
the visibility counts of PointCloudFilter), run with -m gpu:
- the bytes each host-buffer form copies and its kernel launches, as formulas in the cloud and the views, with host and device
  forms equal bit for bit; the read-back bytes and launches of the device merge and fusion;
- the status and exact error text of every refusal the calls share, in each form;
- one context reused across these calls at growing and shrinking sizes computes what a fresh context computes, bit for bit."""
import copy
import ctypes as C

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from openmvs_b200 import lib  # noqa: E402
from openmvs_b200 import depth_estimator as de  # noqa: E402
from openmvs_b200.depth_estimator import (EstimatePointColors, EstimatePointNormals, FuseDepthMaps, FuseRoundStats,  # noqa: E402
	MergeDepthMaps, PointCloud, PointCloudVisibility, PointKNN)
from openmvs_b200.point_cloud import _image_table  # noqa: E402
from test_point_cloud_gpu import _scene_views, _to_device  # noqa: E402

COUNTERS = 40   # sizeof(FuseCounters): the device fusion's counters, read back with its cloud


@pytest.fixture(scope="module")
def scene():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	views = _scene_views(96, 72, 5, 2e-3, 21)
	pc = FuseDepthMaps(copy.deepcopy(views))
	assert len(pc.points) > 5000
	return views, pc


def _stats():
	s = de._device_context(0).stats
	return s.bytes_h2d, s.bytes_d2h, s.kernel_launches


def _images(views, sized=False, device=False):
	out = []
	for v in views:
		im = dict(K=v["K"], R=v["R"], C=v["C"], color=v["color"])
		if device:
			im["color"] = torch.from_numpy(v["color"]).cuda()
		if sized:
			im["height"], im["width"] = v["depth"].shape
		out.append(im)
	return out


def _on_device(pc):
	return PointCloud(torch.from_numpy(np.ascontiguousarray(pc.points)).cuda(), pc.pointViews, None)


# ---- what each form copies and launches ----

def test_host_forms_copy_and_launch_what_the_cloud_needs(scene):
	views, pc = scene
	n = len(pc.points)
	staged = 12*n + 4*(n+1) + 4*sum(len(v) for v in pc.pointViews)
	images = _images(views)
	images[2]["color"] = None                                           # an empty image is not staged
	maps = sum(3*v["color"].shape[0]*v["color"].shape[1] for v, im in zip(views, images) if im["color"] is not None)
	host = EstimatePointColors(images, PointCloud(pc.points, pc.pointViews, None)).colors
	assert _stats() == (staged + maps, 3*n, 2)                           # view checks, colours
	dev_images = [dict(im, color=None if im["color"] is None else torch.from_numpy(im["color"]).cuda()) for im in images]
	assert np.array_equal(EstimatePointColors(dev_images, _on_device(pc)).colors.cpu().numpy(), host)
	host = EstimatePointNormals(images, PointCloud(pc.points, pc.pointViews, None), 16).normals
	assert _stats() == (staged, 12*n, 8)                                 # checks, box, sample; keys, sort, cells, k-NN; PCA
	assert np.array_equal(EstimatePointNormals(images, _on_device(pc), 16).normals.cpu().numpy(), host)
	sized = _images(views, sized=True)
	host = PointCloudVisibility(sized, pc)
	queried = len(set(np.concatenate(pc.pointViews).tolist()))
	# checks, box; entries, sort, view starts; per view with queries: keys, sort, cell starts, gather, queries, exhaustive
	assert _stats() == (staged, 4*n, 5 + 6*queried)
	assert np.array_equal(PointCloudVisibility(sized, _on_device(pc)).cpu().numpy(), host)


def test_device_merge_and_fusion_read_back_and_launches(scene):
	views, _ = scene
	ctx = de._device_context(0)
	merged = MergeDepthMaps(_to_device(views))
	N, nd = len(merged.points), sum(v["depth"] is not None for v in views)
	# the point count, then points, pixels, views, colours and normals; per image flags, one base scan, per image select + assemble
	assert (ctx.stats.bytes_d2h, ctx.stats.kernel_launches) == (8 + N*(12+4+4+3+12), nd + 1 + 2*nd)
	host = MergeDepthMaps(copy.deepcopy(views))
	assert np.array_equal(merged.points, host.points) and np.array_equal(merged.colors, host.colors)
	assert np.array_equal(merged.normals, host.normals) and np.array_equal(np.concatenate(merged.projs), np.concatenate(host.projs))
	# nMinViewsFuse = 1: a round with candidates always makes points, so its launches follow from its round statistics
	fused = FuseDepthMaps(_to_device(views), nMinViewsFuse=1)
	host = FuseDepthMaps(copy.deepcopy(views), nMinViewsFuse=1)
	assert np.array_equal(fused.points, host.points) and np.array_equal(fused.normals, host.normals)
	assert np.array_equal(np.concatenate(fused.pointViews), np.concatenate(host.pointViews))
	launches, d2h = len(views), 4*len(views)                            # which images have a depth, read back
	for r in FuseRoundStats()[0]:
		nb, it, edges = len(views[r["image"]]["neighbors"]), r["iterations"], r["edges"] > 0
		launches += 2
		d2h += 4
		if r["candidates"]:
			launches += 2*(nb > 0) + 3*edges + it*(1 + edges) + edges + 4 + 1
			d2h += 4*(nb > 0) + 4*it + COUNTERS
	nP, nV = len(fused.points), int(sum(len(v) for v in fused.pointViews))
	d2h += nP*(12 + 12 + 3 + 4) + nV*(4 + 4 + 4) + COUNTERS
	assert (ctx.stats.bytes_d2h, ctx.stats.kernel_launches) == (d2h, launches)


# ---- refusals ----

def _refused(call, text):
	with pytest.raises(lib.B200MVSError) as e:
		call()
	assert str(e.value).endswith("failed with status 1: %s" % text), str(e.value)


CALLS = {"colors": ("estimate_point_colors", (), 3, np.uint8), "normals": ("estimate_point_normals", (16,), 3, np.float32),
	"visibility": ("point_cloud_visibility", (), 1, np.int32)}


class Form:
	"""one entry point with its arguments as buffers in the right memory: f(points, n, offsets, ids, table, nImages, *extra)"""

	def __init__(self, call, device):
		self.name, self.extra, cols, dt = CALLS[call]
		self.device = device
		self.ctx = de._device_context(0)
		self.cols, self.dt = cols, dt

	def buf(self, a):
		a = np.ascontiguousarray(a)
		if not self.device:
			self.keep.append(a)
			return a.ctypes.data
		t = torch.from_numpy(a).cuda()
		self.keep.append(t)
		return t.data_ptr()

	def __call__(self, X, off, ids, table, nImages, n=None, extra=None, points=None):
		"""points: an address to pass in place of X's (0: NULL)"""
		self.keep = []
		n = len(X) if n is None else n
		out = self.buf(np.zeros((max(len(X), 1), self.cols), self.dt))
		args = (self.buf(X) if points is None else points, n, self.buf(off), self.buf(ids), table, nImages) + \
			(self.extra if extra is None else extra) + (out,)
		if self.device:
			self.ctx._call(self.name + "_device", *args, None)
		else:
			self.ctx._call(self.name, *args, C.byref(self.ctx.stats))


def _table(images, device):
	return _image_table("test", images, 0 if device else None, (("color", "uint8", (3,)),))


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("call", ["colors", "normals", "visibility"])
def test_refusals(call, device):
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	rng = np.random.RandomState(3)
	X = rng.rand(500, 3).astype(np.float32)
	off = np.arange(501, dtype=np.uint32)
	ids = (np.arange(500) % 2).astype(np.uint32)
	col = np.zeros((8, 8, 3), np.uint8)
	images = [dict(K=np.eye(3), R=np.eye(3), C=np.zeros(3), color=torch.from_numpy(col).cuda() if device else col)]*2
	table, keep = _table(images, device)
	f = Form(call, device)
	what = {"colors": "point colors: ", "normals": "point normals: ", "visibility": "point visibility: "}[call]
	f(X, off, ids, table, 2)                                             # the arguments below differ from these in one place
	_refused(lambda: f(X, off, ids, table, 2, points=0), "point cloud: null pointer")
	_refused(lambda: f(X, off, ids, table, 2, n=2**31), "point cloud: more than 2^31 - 1 points")
	_refused(lambda: f(X, off, ids, None, 2), "point cloud: bad image table")
	_refused(lambda: f(X, off, ids, table, -1), "point cloud: bad image table")
	bad = off.copy(); bad[0] = 1
	_refused(lambda: f(X, bad, ids, table, 2), "point cloud: the view offsets do not start at 0" + (" or are not monotone" if device else ""))
	bad = off.copy(); bad[7] = 9
	_refused(lambda: f(X, bad, ids, table, 2), "point cloud: the view offsets " + ("do not start at 0 or " if device else "") + "are not monotone")
	bad = ids.copy(); bad[11] = 2
	_refused(lambda: f(X, off, bad, table, 2), "point cloud: a view ID is not below nImages")
	empty = np.concatenate([off[:6], off[5:-1]])                          # point 5 has no view
	if call == "normals":
		_refused(lambda: f(X, empty, ids, table, 2), "point cloud: a point has no view")
	else:
		f(X, empty, ids, table, 2)
	nan = X.copy(); nan[17, 1] = np.nan
	if call == "colors":
		f(nan, off, ids, table, 2)                                       # the colours read no coordinate they cannot project
	else:
		_refused(lambda: f(nan, off, ids, table, 2), "point cloud: a coordinate is not finite")
	if device:
		_refused(lambda: f(X, off, ids, table, 2, points=X.ctypes.data), what + "a buffer is not in device memory of the context's device")
	if call == "normals":
		for k in (0, 33):
			_refused(lambda: f(X, off, ids, table, 2, extra=(k,)), what + "numNeighbors out of [1, 32]")
			_refused(lambda: f(X[:0], off[:1], ids, table, 2, extra=(k,)), what + "numNeighbors out of [1, 32]")   # before the empty return
	if call in ("colors", "visibility"):
		table[1].width = 0
		_refused(lambda: f(X, off, ids, table, 2), what + "image size out of range")
		if call == "colors":
			f(X[:0], off[:1], ids, table, 2)                               # an empty cloud reads no image
		table[1].width = 8
	if call == "colors" and device:
		host_table, host_keep = _table([dict(im, color=col) for im in images], False)
		_refused(lambda: f(X, off, ids, host_table, 2), what + "an image is not in device memory of the context's device")
	f(X, off, ids, table, 2)                                             # the context still works


# ---- one context across the point-cloud calls ----

def _bits(a):
	a = a.cpu().numpy() if torch.is_tensor(a) else np.asarray(a)
	return np.ascontiguousarray(a).view(np.uint8)


def _cloud_steps(w, h, n, k, seed):
	views = _scene_views(w, h, n, 2e-3, seed)
	fused = FuseDepthMaps(copy.deepcopy(views))

	def run():
		merged = MergeDepthMaps(_to_device(views))
		dev = _on_device(fused)
		out = [merged.points, merged.colors, merged.normals, np.concatenate(merged.projs)]
		out.append(EstimatePointColors(_images(views, device=True), dev).colors)
		out.append(EstimatePointColors(_images(views), PointCloud(fused.points, fused.pointViews, None)).colors)
		out.append(EstimatePointNormals(_images(views), dev, k).normals)
		out.append(EstimatePointNormals(_images(views), PointCloud(fused.points, fused.pointViews, None), k).normals)
		out.append(PointKNN(dev.points, k))
		out.append(PointKNN(torch.from_numpy(merged.points).cuda(), k))
		out.append(PointCloudVisibility(_images(views, sized=True), dev))
		out.append(PointCloudVisibility(_images(views, sized=True), fused))
		return out
	return run


def _fuse_steps(w, h, n, seed):
	views = _scene_views(w, h, n, 2e-3, seed)

	def run():
		dev = _to_device(views)
		pc = FuseDepthMaps(dev)
		return [pc.points, pc.colors, pc.normals, np.concatenate(pc.pointViews), np.concatenate(pc.pointWeights),
			np.concatenate(pc.projs)] + [v["depth"] for v in dev]
	return run


def _on(ctx, run):
	saved = de._DEVICE_CTX.get(0)
	de._DEVICE_CTX[0] = ctx
	try:
		return [_bits(a) for a in run() if a is not None]
	finally:
		de._DEVICE_CTX[0] = saved


def test_one_context_across_the_point_cloud_calls():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	steps = [
		("cloud 96x72 x4", _cloud_steps(96, 72, 4, 8, 31)),
		("fuse 160x120 x4", _fuse_steps(160, 120, 4, 32)),
		("cloud 320x240 x6", _cloud_steps(320, 240, 6, 32, 33)),
		("fuse 320x240 x6", _fuse_steps(320, 240, 6, 34)),
		("cloud 160x120 x5", _cloud_steps(160, 120, 5, 16, 35)),
		("fuse 96x72 x3", _fuse_steps(96, 72, 3, 36)),
		("cloud 64x48 x3", _cloud_steps(64, 48, 3, 4, 37)),
	]
	shared = de._Context(0)
	try:
		reused = [_on(shared, run) for _, run in steps]
	finally:
		shared.Release()
	for (name, run), got in zip(steps, reused):
		fresh = de._Context(0)
		try:
			want = _on(fresh, run)
		finally:
			fresh.Release()
		assert len(got) == len(want), name
		for k, (a, b) in enumerate(zip(got, want)):
			assert a.shape == b.shape and np.array_equal(a, b), "%s: output %d differs from a fresh context" % (name, k)
