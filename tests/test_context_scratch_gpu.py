"""One engine context reused across subsystems and sizes: every call's scratch is carved from its subsystem's arena, so a call that
follows larger or smaller calls of any kind on the same context, or nests other calls, computes what it computes on a fresh
context, bit for bit.  The sequence grows and then shrinks every arena (PatchMatch, SGM match, tSGM, SGM fusion, post-processing,
FuseDepthMaps), runs hierarchical pairs (which nest SGM matches) between plain matches, and checks that the accumulated costs of
the last match stay readable by RefineDisparityMap(accums=None) until a hierarchical call clears them (run with -m gpu)."""
import ctypes as C

import numpy as np
import pytest

from openmvs_b200 import synth

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


class Engine:
	"""PatchMatch, SGM, post-processing and device FuseDepthMaps calls, all on one native context"""

	def __init__(self):
		from openmvs_b200.depth_estimator import DepthMapsData, PatchMatchB200, SemiGlobalMatcher
		self.pm = PatchMatchB200(0)
		self.m = SemiGlobalMatcher()
		self.m._lib.b200mvs_destroy(self.m._ctx)
		self.m._ctx = self.pm._ctx
		self.dm = DepthMapsData([], 0, nCalibratedImages=12)
		self.dm.pmCUDA.Release()
		self.dm.pmCUDA = self.pm

	def release(self):
		self.m._ctx = C.c_void_p()
		self.pm.Release()


def _cuda(a):
	return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _np(a):
	return a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def _estimate(w, h, colour):
	from openmvs_b200.depth_estimator import Camera, DepthData, ViewData
	sc = synth.make_scene(w, h, 2, step_deg=5.0)
	images = [(np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1) if colour else v.image for v in sc.views]

	def run(e):
		dd = DepthData([ViewData(im, Camera(v.K, v.R, v.C)) for im, v in zip(images, sc.views)], sc.dmin, sc.dmax)
		e.pm.EstimateDepthMap(dd)
		return dd.depthMap, dd.normalMap, dd.confMap, dd.viewsMap
	return run


def _pixel_map(w, h, lo, hi):
	px, num = synth.sgm_pixel_map(w, h, lo, hi)
	return _cuda(px.view(np.uint8).reshape(-1, 16)), num


def _match_and_refine(w, h, num_disp):
	lg, lc, rg, _ = synth.make_stereo_pair(w, h)

	def run(e):
		pxd, num = _pixel_map(w, h, 0, num_disp)
		disp, cost = e.m.MatchDevice(_cuda(lg), _cuda(lc), _cuda(rg), pxd, num)
		refined = e.m.RefineDisparityMap(disp.clone(), pxd, None, 4)   # the sums of this match, kept on the context
		return disp, cost, refined
	return run


def _hierarchical(w, h, min_res, masked):
	lg, lc, rg, _, rc = synth.make_stereo_pair(w, h, right_color=True)
	lm = np.full((h, w), 255, np.uint8)
	lm[:, w//3:w//3+25] = 0

	def run(e):
		from openmvs_b200 import lib
		disp, cost, levels = e.m.MatchPairHierarchicalDevice(_cuda(lg), _cuda(lc), _cuda(rg), _cuda(rc), None,
			_cuda(lm) if masked else None, None, minResolution=min_res)
		# the pixel maps of the hierarchy are internal: a refinement without sums of its own is refused afterwards
		pxd, _ = _pixel_map(w, h, 0, 32)
		with pytest.raises(lib.B200MVSError):
			e.m.RefineDisparityMap(torch.zeros((h-6, w-6), dtype=torch.int16, device="cuda"), pxd, None, 4)
		return disp, cost, np.array([l["numCosts"] for l in levels])
	return run


def _tsgm_blocks(w, h):
	lg, lc, rg, d, rc = synth.make_stereo_pair(w, h, right_color=True)
	disp = np.rint(d[3:-3, 3:-3]*4).astype(np.int16)
	disp[::7, ::5] = 32767
	mask2 = np.full((2*(h-6)+8, 2*(w-6)+8), 255, np.uint8)
	mask = np.full((h, w), 255, np.uint8)
	mask[h//2:h//2+9, :] = 0

	def run(e):
		px, num = e.m.Disparity2RangeMap(_cuda(disp), _cuda(mask2))
		flipped = e.m.FlipDirection(_cuda(disp))
		speckles = e.m.FilterSpeckles(_cuda(disp), maxSpeckleSize=40)
		level = e.m.LevelMask(_cuda(mask), (w//2, h//2))
		return px, np.array([num]), flipped, speckles, level
	return run


def _sgm_fuse(W, H, seed):
	from test_sgm_fuse_gpu import random_pairs
	pairs = random_pairs(W, H, 3, seed=seed)
	K = np.array([[0.9*W, 0, (W-1)/2.0], [0, 0.9*W, (H-1)/2.0], [0, 0, 1.0]])

	def run(e):
		return e.m.Fuse([(_cuda(d), _cuda(c), Q, s) for d, c, Q, s in pairs], (W, H), 2, K)
	return run


def _post(w, h):
	from test_filter_oracle import segment_test_map
	from test_filter_parity_gpu import _depth_data, _gap_inputs
	from openmvs_b200.depth_estimator import DepthData
	sc = synth.make_scene(w, h, 6, step_deg=4.0)
	maps = synth.make_noisy_dmaps(sc)
	seg = segment_test_map(sc)
	gd, gn, gc = _gap_inputs(sc)

	def run(e):
		out = list(e.dm.FilterDepthMap(_depth_data(sc, maps, 2, "cuda"), [_depth_data(sc, maps, i, "cuda") for i in sc.neighbors(2, 5)]))
		for name, (d, n, c) in (("RemoveSmallSegments", (seg, gn, gc)), ("GapInterpolation", (gd, gn, gc))):
			dd = DepthData([], 0, 0, _cuda(d), _cuda(n), _cuda(c))
			getattr(e.dm, name)(dd)
			out += [dd.depthMap, dd.normalMap, dd.confMap]
		return out
	return run


def _fuse_depth_maps(w, h, n):
	from test_fuse_device_gpu import _scene_views, _to_device
	views = _scene_views(w, h, n, 2e-3, 3)

	def run(e):
		from openmvs_b200 import depth_estimator as de
		dev = _to_device(views)
		saved = de._DEVICE_CTX.get(0)
		de._DEVICE_CTX[0] = e.pm
		try:
			pc = de.FuseDepthMaps(dev, nMinViewsFuse=2)
			rounds = de.FuseRoundStats()[0]
		finally:
			if saved is None:
				del de._DEVICE_CTX[0]
			else:
				de._DEVICE_CTX[0] = saved
		assert len(rounds) == n
		return [pc.points, pc.colors, pc.normals, np.array([pc.nDepths]), np.concatenate(pc.pointViews),
			np.concatenate(pc.pointWeights), np.concatenate(pc.projs)] + [v["depth"] for v in dev]
	return run


def _bits(a):
	return np.ascontiguousarray(_np(a)).view(np.uint8)


def test_one_context_across_subsystems_and_sizes():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	steps = [
		("estimate 640x480", _estimate(640, 480, False)),
		("estimate 1920x1080", _estimate(1920, 1080, False)),
		("estimate 320x240", _estimate(320, 240, False)),
		("estimate 322x242 colour", _estimate(322, 242, True)),   # gray copies, and a reference pitch TMA cannot address
		("match 200x120", _match_and_refine(200, 120, 32)),
		("hierarchical 640x360", _hierarchical(640, 360, 160, True)),
		("match 960x540", _match_and_refine(960, 540, 64)),
		("tsgm blocks 400x240", _tsgm_blocks(400, 240)),
		("hierarchical 400x240", _hierarchical(400, 240, 160, False)),
		("match 200x120 again", _match_and_refine(200, 120, 32)),
		("tsgm blocks 200x120", _tsgm_blocks(200, 120)),
		("post 400x300", _post(400, 300)),
		("post 200x150", _post(200, 150)),
		("fuse depth maps 320x240 x6", _fuse_depth_maps(320, 240, 6)),
		("fuse depth maps 160x120 x4", _fuse_depth_maps(160, 120, 4)),
		("sgm fuse 301x203", _sgm_fuse(301, 203, 5)),
		("sgm fuse 97x61", _sgm_fuse(97, 61, 11)),
	]
	shared = Engine()
	try:
		reused = [[_bits(a) for a in run(shared) if a is not None] for _, run in steps]
	finally:
		shared.release()
	for (name, run), got in zip(steps, reused):
		fresh = Engine()
		try:
			want = [_bits(a) for a in run(fresh) if a is not None]
		finally:
			fresh.release()
		assert len(got) == len(want), name
		for k, (a, b) in enumerate(zip(got, want)):
			assert a.shape == b.shape and np.array_equal(a, b), "%s: output %d differs from a fresh context" % (name, k)
