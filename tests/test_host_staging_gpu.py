"""The host forms of the C-ABI (numpy maps in, numpy maps out) against their device forms on the same inputs: bit-identical outputs,
the bytes each call copies (bytes_h2d / bytes_d2h), its kernel launches, and the status and error text of refused arguments
(run with -m gpu)."""
import ctypes as C

import numpy as np
import pytest

from openmvs_b200 import synth

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu
f32 = np.float32
bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def eng():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	from openmvs_b200.depth_estimator import DepthMapsData, SemiGlobalMatcher
	dm, m = DepthMapsData([], 0, nCalibratedImages=12), SemiGlobalMatcher()
	yield dm, m
	dm.pmCUDA.Release(); m.Release()


def cuda(a):
	return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def counts(stats):
	return stats.bytes_h2d, stats.bytes_d2h, stats.kernel_launches


def refused(call, status, text):
	from openmvs_b200.lib import B200MVSError
	with pytest.raises(B200MVSError) as e:
		call()
	assert str(e.value).endswith("failed with status %d: %s" % (status, text)), str(e.value)


def test_match(eng):
	_, m = eng
	w, h = 200, 120
	n, nv = w*h, (w-6)*(h-6)
	lg, lc, rg, _ = synth.make_stereo_pair(w, h)
	px, num = synth.sgm_pixel_map(w, h, 0, 32)
	hd, hc = m.Match(lg, lc, rg, px, num)
	host = counts(m.stats)
	gd, gc = m.MatchDevice(cuda(lg), cuda(lc), cuda(rg), cuda(px.view(np.uint8).reshape(-1, 16)), num)
	assert np.array_equal(hd, gd.cpu().numpy()) and np.array_equal(hc.view(np.int16), gc.cpu().numpy())
	assert host == (11*n+16*nv, 4*nv, m.stats.kernel_launches) and host[2] == 2+1+8+1
	px2, num2 = synth.sgm_pixel_map(w, h, 0, 300)
	refused(lambda: m.Match(lg, lc, rg, px2, num2), 1, "sgm: more than 256 disparities per pixel")
	out = np.zeros((h-6, w-6), np.int16)
	refused(lambda: m._call("sgm_match", None, lc.ctypes.data, rg.ctypes.data, w, h, px.ctypes.data, num, C.byref(m.prm),
		out.ctypes.data, out.ctypes.data, C.byref(m.stats)), 1, "sgm: null pointer or image too small")


@pytest.mark.parametrize("costs", [True, False])
@pytest.mark.parametrize("with_k", [True, False])
def test_fuse(eng, costs, with_k):
	from test_sgm_fuse_gpu import random_pairs
	_, m = eng
	W, H = 97, 61
	pairs = random_pairs(W, H, 3, seed=11, costs=costs)
	K = np.array([[0.9*W, 0, (W-1)/2.0], [0, 0.9*W, (H-1)/2.0], [0, 0, 1.0]]) if with_k else None
	hd, hc, hn = m.Fuse(pairs, (W, H), 2, K)
	maps = sum(d.size*2*(2 if costs else 1) for d, _, _, _ in pairs)
	assert counts(m.stats) == (maps, W*H*(8+(12 if with_k else 0)), 4 if with_k else 3)
	gd, gc, gn = m.Fuse([(cuda(d), None if c is None else cuda(c), Q, s) for d, c, Q, s in pairs], (W, H), 2, K)
	assert np.array_equal(bits(hd), bits(gd.cpu().numpy())) and np.array_equal(bits(hc), bits(gc.cpu().numpy()))
	assert (hn is None) == (gn is None) and (hn is None or np.array_equal(bits(hn), bits(gn.cpu().numpy())))
	refused(lambda: m.Fuse(pairs, (W, H), -1, K), 1, "sgm fuse: null depth map, negative minViews, or K without a normal map")
	mixed = [pairs[0], (pairs[1][0], np.zeros_like(pairs[1][0], np.uint16) if not costs else None, pairs[1][2], 4)]
	refused(lambda: m.Fuse(mixed, (W, H), 2, K), 1, "sgm fuse: either every pair has a cost map or none has one")


@pytest.fixture(scope="module")
def scene():
	sc = synth.make_scene(200, 150, 6, step_deg=4.0)
	return sc, synth.make_noisy_dmaps(sc)


@pytest.mark.parametrize("adjust", [True, False])
def test_filter_depth_map(eng, scene, adjust):
	from test_filter_parity_gpu import _depth_data
	from openmvs_b200.depth_estimator import OPTDENSE
	dm, _ = eng
	sc, maps = scene
	ref, nb = 2, sc.neighbors(2, 5)
	hd, hc = dm.FilterDepthMap(_depth_data(sc, maps, ref), [_depth_data(sc, maps, i, None, adjust) for i in nb], adjust)
	n = 200*150
	assert counts(dm.stats) == (n*8+len(nb)*n*(8 if adjust else 4), n*8, 2)
	gd, gc = dm.FilterDepthMap(_depth_data(sc, maps, ref, "cuda"), [_depth_data(sc, maps, i, "cuda", adjust) for i in nb], adjust)
	assert np.array_equal(bits(hd), bits(gd.cpu().numpy())) and np.array_equal(bits(hc), bits(gc.cpu().numpy()))
	# too few neighbours: not filtered, nothing copied
	dm.stats.bytes_h2d = 12345
	assert dm.FilterDepthMap(_depth_data(sc, maps, ref), [_depth_data(sc, maps, nb[0])], adjust) is None
	assert dm.stats.bytes_h2d == 12345
	refused(lambda: dm.FilterDepthMap(_depth_data(sc, maps, ref), [_depth_data(sc, maps, nb[0])]*17, adjust),
		1, "filter: too many neighbour depth-maps")
	th = OPTDENSE.fDepthDiffThreshold
	try:
		OPTDENSE.fDepthDiffThreshold = 0.0
		refused(lambda: dm.FilterDepthMap(_depth_data(sc, maps, ref), [_depth_data(sc, maps, i) for i in nb], adjust),
			1, "filter: invalid parameter block")
	finally:
		OPTDENSE.fDepthDiffThreshold = th


def _post_maps(sc, name, extras):
	from test_filter_oracle import segment_test_map
	from test_filter_parity_gpu import _gap_inputs
	d, n, c = _gap_inputs(sc)
	if name == "RemoveSmallSegments":
		d = segment_test_map(sc)
	return d, (n if "normal" in extras else None), (c if "conf" in extras else None)


def _host_and_device(dm, name, d, n, c):
	"""the host and the device form of one in-place pass on copies of (d, n, c) -> (host maps, device maps, host counts)"""
	from openmvs_b200.depth_estimator import DepthData
	copy = lambda a: None if a is None else a.copy()
	hm = DepthData([], 0, 0, copy(d), copy(n), copy(c))
	getattr(dm, name)(hm)
	host = counts(dm.stats)
	gm = DepthData([], 0, 0, *[None if a is None else cuda(a) for a in (d, n, c)])
	getattr(dm, name)(gm)
	torch.cuda.synchronize()
	out = lambda mm: [None if a is None else (a if isinstance(a, np.ndarray) else a.cpu().numpy()) for a in (mm.depthMap, mm.normalMap, mm.confMap)]
	return out(hm), out(gm), host


def _rounds(w, h):
	r = 1
	while (1 << r) < w+h:
		r += 1
	return r


@pytest.mark.parametrize("extras", [(), ("normal",), ("conf",), ("normal", "conf")], ids=lambda e: "+".join(e) or "depth")
@pytest.mark.parametrize("name", ["RemoveSmallSegments", "GapInterpolation"])
def test_remove_small_segments_and_gap_interpolation(eng, scene, name, extras):
	from oracle import oracle as O
	dm, _ = eng
	sc, _ = scene
	d, n, c = _post_maps(sc, name, extras)
	h, w = d.shape
	if name == "RemoveSmallSegments":
		assert O.count_asymmetric_edges(d, f32(f32(0.01)*f32(0.7))) == 0   # no arcs: no patch launch
	hm, gm, host = _host_and_device(dm, name, d, n, c)
	for a, b in zip(hm, gm):
		assert (a is None) == (b is None) and (a is None or np.array_equal(bits(a), bits(b)))
	b = d.nbytes+(n.nbytes if n is not None else 0)+(c.nbytes if c is not None else 0)
	assert host == (b, b, 5+2*_rounds(w, h) if name == "RemoveSmallSegments" else 2)


def test_post_processing_refused_arguments(eng):
	from openmvs_b200.depth_estimator import DepthData, OPTDENSE
	dm, _ = eng
	d = np.ones((20, 30), f32)
	for name, call in (("remove_small_segments", dm.RemoveSmallSegments), ("gap_interpolation", dm.GapInterpolation)):
		refused(lambda: dm.pmCUDA._call(name, None, None, None, 30, 20, 0.01, 100, C.byref(dm.stats)), 1, "post-processing: invalid argument")
		refused(lambda: dm.pmCUDA._call(name, d.ctypes.data, None, None, 0, 20, 0.01, 100, C.byref(dm.stats)), 1,
			"post-processing: invalid argument")
		th = OPTDENSE.fDepthDiffThreshold
		try:
			OPTDENSE.fDepthDiffThreshold = 0.0
			refused(lambda: call(DepthData([], 0, 0, d.copy())), 1, name+": invalid argument")
		finally:
			OPTDENSE.fDepthDiffThreshold = th


def test_remove_small_segments_many_direction_dependent_edges(eng):
	"""a staircase whose steps sit right at the threshold, large enough for thousands of one-way edges between its components, its
	depth falling left to right, so that the one-way edges point from earlier seeds (column-major) to later ones: the reference's
	segments then differ from both the two-way components and the components of the undirected edges.  The host replay of its seed
	order is bit-identical to the breadth-first oracle on the host and device paths."""
	from oracle import oracle as O
	from openmvs_b200.depth_estimator import OPTDENSE
	from test_filter_oracle import component_sizes
	dm, _ = eng
	th = f32(f32(0.01)*f32(0.7))
	rng = np.random.RandomState(4)
	stairs = np.full((300, 400), 5.0, f32)
	for k in range(1, 80):
		stairs[:, 5*k:] *= f32(1.0+float(th)*(0.9965+0.007*rng.rand()))
	stairs[rng.rand(*stairs.shape) < 0.08] = 0
	stairs = np.ascontiguousarray(stairs[:, ::-1])
	assert O.count_asymmetric_edges(stairs, th) > 4096
	two_way, undirected = component_sizes(stairs, th, True), component_sizes(stairs, th, False)
	for speckle in (20, 100, 1000, 5000):   # 5000: above the size of one step's stripe
		od, _, _ = O.remove_small_segments(stairs, None, None, th, speckle)
		for sizes in (two_way, undirected):
			assert not np.array_equal(np.where(sizes < speckle, 0, stairs), od)
		OPTDENSE.nSpeckleSize = speckle
		try:
			hm, gm, host = _host_and_device(dm, "RemoveSmallSegments", stairs, None, None)
		finally:
			OPTDENSE.nSpeckleSize = 100
		assert np.array_equal(hm[0], od) and np.array_equal(gm[0], od)
		assert host == (stairs.nbytes, stairs.nbytes, 5+2*_rounds(400, 300)+1)
