"""GPU parity of the SGM pair matcher against the oracle (run with -m gpu).
Integer stages (8-path aggregation, WTA) must be bit-exact; the WZNCC cost is a float
rounded to uint8 and may differ by one level on a small fraction of entries."""
import numpy as np
import pytest
import torch

from openmvs_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sgm():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	from oracle import oracle as O
	from openmvs_b200.depth_estimator import SemiGlobalMatcher
	m = SemiGlobalMatcher()
	yield m, O
	m.Release()


def _dev(a):
	return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _px_dev(px):
	return torch.from_numpy(px.view(np.uint8).reshape(-1, 16).copy()).cuda()


def test_cost_volume_parity(sgm):
	m, O = sgm
	w, h = 240, 136
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, -4, 28)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n, stage=1)
	costs = torch.zeros(n, dtype=torch.uint8, device="cuda")
	m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=1, costs=costs)
	g = costs.cpu().numpy().astype(np.int32)
	diff = np.abs(g-c.astype(np.int32))
	assert diff.max() <= 1 and (diff > 0).mean() < 5e-3
	assert np.array_equal(g == 255, c == 255) or ((g == 255) != (c == 255)).mean() < 1e-4


@pytest.mark.parametrize("num,dmin,w", [(128, 0, 403), (128, -40, 300), (64, 5, 261), (64, -70, 200), (256, -100, 330), (192, 3, 290)])
def test_cost_volume_on_tensor_cores(sgm, num, dmin, w):
	"""The banded-GEMM cost kernel (wgmma, fp16 hi/lo split operands, fp32 accumulation in registers; sgm_cost_tc.cu) against the
	oracle and against the SIMT kernel: within one uint8 level on a small fraction of the entries, out-of-image windows exact."""
	m, O = sgm
	h = 61
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, dmin, dmin+num)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n, stage=1)
	simt = torch.zeros(n, dtype=torch.uint8, device="cuda"); tc = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
	args = (_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n)
	try:
		m.SetDebug(sgmCost=1); m.MatchDevice(*args, stages=1, costs=simt)
		m.SetDebug(sgmCost=2); m.MatchDevice(*args, stages=1, costs=tc)
	finally:
		m.SetDebug()
	g = tc.cpu().numpy().astype(np.int32); s = simt.cpu().numpy().astype(np.int32)
	for name, ref in (("oracle", c.astype(np.int32)), ("simt", s)):
		diff = np.abs(g-ref)
		assert diff.max() <= 1, (name, int(diff.max()), float((diff > 1).mean()))
		assert (diff > 0).mean() < 5e-3, (name, float((diff > 0).mean()))
	assert ((g == 255) != (c == 255)).mean() < 1e-4


@pytest.mark.parametrize("ragged", [False, True])
def test_aggregation_and_wta_bit_exact(sgm, ragged):
	m, O = sgm
	w, h = 200, 120
	rng = np.random.RandomState(11)
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	vw, vh = w-6, h-6
	if ragged:
		# tSGM-like ragged ranges around the true disparity, with invalid pixels and range jumps
		base = np.rint(d[3:-3, 3:-3]).astype(np.int16)
		lo = base-rng.randint(2, 9, (vh, vw)).astype(np.int16)
		hi = base+rng.randint(2, 40, (vh, vw)).astype(np.int16)
		hi[10:14] = lo[10:14]+256   # the widest range the kernel supports
		px, n = synth.sgm_pixel_map(w, h, lo, hi, rng.rand(vh, vw) < 0.07)
	else:
		px, n = synth.sgm_pixel_map(w, h, 0, 64)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n)
	accums = torch.zeros(n, dtype=torch.int16, device="cuda")
	gd, gc = m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=6, costs=_dev(c), accums=accums)
	assert np.array_equal(accums.cpu().numpy().view(np.uint16), a)
	assert np.array_equal(gd.cpu().numpy(), disp)
	assert np.array_equal(gc.cpu().numpy().view(np.uint16), cost)


def test_host_api_full_match_and_errors(sgm):
	m, O = sgm
	w, h = 200, 120
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, 0, 32)
	gd, gc = m.Match(lg, lc, rg, px, n)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n)
	# end to end the two pipelines differ only through the +-1 cost roundings
	assert (gd != disp).mean() < 0.01
	gt = d[3:-3, 3:-3]
	assert (np.abs(gd-gt)[5:-5, 5:-40] <= 1).mean() > 0.97
	assert m.stats.kernel_launches == 2+1+8+1 and m.stats.bytes_d2h == (w-6)*(h-6)*4
	# more than 256 disparities per pixel is refused loudly
	from openmvs_b200 import lib
	px2, n2 = synth.sgm_pixel_map(w, h, 0, 300)
	with pytest.raises(lib.B200MVSError):
		m.Match(lg, lc, rg, px2, n2)
	# same input twice -> identical output
	gd2, gc2 = m.Match(lg, lc, rg, px, n)
	assert np.array_equal(gd, gd2) and np.array_equal(gc, gc2)


def test_full_size_sgm_properties_1080p(sgm):
	"""BASELINE configs[2] size: 1920x1080 pair, fixed range D=128 (the non-tSGM branch,
	SemiGlobalMatcher.cpp:643-669): determinism and ground-truth disparity."""
	m, O = sgm
	w, h = 1920, 1080
	lg, lc, rg, d = synth.make_stereo_pair(w, h, d0=40.0, amp=25.0)
	px, n = synth.sgm_pixel_map(w, h, 0, 128)
	args = (_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n)
	gd, gc = m.MatchDevice(*args)
	ms = m.stats.ms_device
	gd2, gc2 = m.MatchDevice(*args)
	assert torch.equal(gd, gd2) and torch.equal(gc, gc2)
	# the per-direction ring kernel gives the same integers
	try:
		m.SetDebug(sgmAggregation=3)
		gd3, gc3 = m.MatchDevice(*args)
	finally:
		m.SetDebug()
	assert torch.equal(gd, gd3) and torch.equal(gc, gc3)
	gt = d[3:-3, 3:-3]
	err = np.abs(gd.cpu().numpy()-gt)[8:-8, 8:-140]
	assert (err <= 1).mean() > 0.97
	print("sgm 1080p D=128: %.2f ms device" % ms)


def test_cross_check_and_subpixel_refinement_parity(sgm):
	"""ConsistencyCrossCheck (exact) and RefineDisparityMap / LC-blend (float -> quarter-pixel integer)."""
	m, O = sgm
	w, h = 200, 120
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, 0, 32)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n)
	# right-to-left map of the same pair: swap the roles, negative disparities
	pxr, nr = synth.sgm_pixel_map(w, h, -32, 0)
	bgr_r = np.repeat(np.rint(rg*255).astype(np.uint8)[..., None], 3, -1)
	cr, ar, dispr, costr = O.sgm_match(rg, bgr_r, lg, pxr, nr)
	rng = np.random.RandomState(2)
	disp_in = disp.copy(); disp_in[rng.rand(*disp.shape) < 0.05] = 32767
	want = O.sgm_cross_check(disp_in, dispr, 1)
	got = m.ConsistencyCrossCheck(_dev(disp_in), _dev(dispr), 1).cpu().numpy()
	assert np.array_equal(got, want)
	assert 0.3 < (want != 32767).mean() < 0.999
	# sub-pixel refinement on the oracle's accumulated costs
	want = O.sgm_refine(px, a, disp_in, 4)
	got = m.RefineDisparityMap(_dev(disp_in), _px_dev(px), accums=_dev(a.view(np.int16)), subpixelSteps=4).cpu().numpy()
	diff = np.abs(got.astype(np.int32)-want.astype(np.int32))
	assert diff.max() <= 1 and (diff > 0).mean() < 1e-3
	valid = want != 32767
	assert np.abs(want[valid]/4.0-disp_in[valid]).max() <= 0.5+1e-6  # the offset stays within half a pixel


_UNIFORM_CASES = [(num, 0) for num in (4, 36, 48, 128, 132, 144, 192, 256)] + [(num, 2) for num in (48, 128, 144, 192, 256)]


@pytest.mark.parametrize("num,mode", _UNIFORM_CASES, ids=[str(n) if mode == 0 else "%d-register" % n for n, mode in _UNIFORM_CASES])
def test_uniform_range_fast_path_bit_exact(sgm, num, mode):
	"""One global disparity range (the non-tSGM branch) against the oracle, with some invalid pixels: the packed
	register-pipelined aggregation kernel (4, 36, 132: slices not 16-byte aligned) and the bulk-copy ring kernel
	(48, 128: 4 disparities per lane; 144, 192, 256: 8 per lane), and the register-pipelined kernel forced
	(sgmAggregation = 2) on the 16-byte aligned widths, so that both kernels run the shared packed step at 4 and 8 per lane."""
	m, O = sgm
	w, h = 150, 90
	rng = np.random.RandomState(num)
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, -7, -7+num, rng.rand(h-6, w-6) < 0.05)
	costs = rng.randint(0, 256, n).astype(np.uint8)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n, costs=costs)
	accums = torch.zeros(n, dtype=torch.int16, device="cuda")
	try:
		m.SetDebug(sgmAggregation=mode)
		gd, gc = m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=6, costs=_dev(costs), accums=accums)
	finally:
		m.SetDebug()
	assert np.array_equal(accums.cpu().numpy().view(np.uint16), a)
	assert np.array_equal(gd.cpu().numpy(), disp) and np.array_equal(gc.cpu().numpy().view(np.uint16), cost)


@pytest.mark.parametrize("w,h", [(151, 92), (263, 143)])
@pytest.mark.parametrize("num", [64, 128, 256])
def test_wave_front_aggregation_bit_exact(sgm, num, w, h):
	"""The wave-front kernel (dense volume, one range of 64 / 128 / 256 disparities; the default of the non-tSGM branch) against the
	oracle.  Valid regions 145 x 86 and 257 x 137: neither a multiple of the 4-path bands, three and five sub-cell columns, and
	paths that cross up to 9 and 14 front blocks, so that their segments hand the path state over on the GPU."""
	m, O = sgm
	rng = np.random.RandomState(num)
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, -9, -9+num)
	costs = rng.randint(0, 256, n).astype(np.uint8)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n, costs=costs)
	accums = torch.full((n,), -1, dtype=torch.int16, device="cuda")   # phase 0 of each pass stores: no memset needed
	try:
		m.SetDebug(sgmAggregation=4)
		gd, gc = m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=6, costs=_dev(costs), accums=accums)
	finally:
		m.SetDebug()
	assert np.array_equal(accums.cpu().numpy().view(np.uint16), a)
	assert np.array_equal(gd.cpu().numpy(), disp) and np.array_equal(gc.cpu().numpy().view(np.uint16), cost)


def test_wide_image_tensor_core_cost_and_wave_fronts(sgm):
	"""A 4100-pixel-wide strip (wider than C5's 4032): 32 pixel blocks per row in the tensor-core cost kernel, sub-cell columns of
	the wave-front dependencies clamped to 30 (137 pixels each), bands at the image corners that span every sub-cell column."""
	m, O = sgm
	w, h, num = 4100, 61, 64
	lg, lc, rg, d = synth.make_stereo_pair(w, h, d0=20.0, amp=8.0)
	px, n = synth.sgm_pixel_map(w, h, 0, num)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n)
	costs = torch.zeros(n, dtype=torch.uint8, device="cuda"); accums = torch.full((n,), -1, dtype=torch.int16, device="cuda")
	m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=1, costs=costs)
	diff = np.abs(costs.cpu().numpy().astype(np.int32)-c.astype(np.int32))
	assert diff.max() <= 1 and (diff > 0).mean() < 5e-3
	# aggregation + WTA on the ORACLE's cost volume: bit-exact
	gd, gc = m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=6, costs=_dev(c), accums=accums)
	assert np.array_equal(accums.cpu().numpy().view(np.uint16), a)
	assert np.array_equal(gd.cpu().numpy(), disp)


def test_wave_front_aggregation_larger_image_and_variants_agree(sgm):
	"""403 x 251, D = 128: default (wave fronts) == bulk-copy ring kernel == register-pipelined kernel == general kernel == oracle"""
	m, O = sgm
	w, h = 403, 251
	rng = np.random.RandomState(5)
	lg, lc, rg, d = synth.make_stereo_pair(w, h)
	px, n = synth.sgm_pixel_map(w, h, 0, 128)
	costs = rng.randint(0, 256, n).astype(np.uint8)
	c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n, costs=costs)
	try:
		for mode in (0, 3, 2, 1):
			m.SetDebug(sgmAggregation=mode)
			accums = torch.zeros(n, dtype=torch.int16, device="cuda")
			gd, gc = m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=6, costs=_dev(costs), accums=accums)
			assert np.array_equal(accums.cpu().numpy().view(np.uint16), a), mode
			assert np.array_equal(gd.cpu().numpy(), disp), mode
			assert m.stats.kernel_launches == (2+1+1 if mode == 0 else 2+8+1)
		# aggregation alone (stages = 2): the two volumes of the default are added by a launch of their own; then the
		# winner-takes-all stage alone over the stored sums
		m.SetDebug()
		accums = torch.zeros(n, dtype=torch.int16, device="cuda")
		m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=2, costs=_dev(costs), accums=accums)
		assert np.array_equal(accums.cpu().numpy().view(np.uint16), a)
		gd, gc = m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=4, costs=_dev(costs), accums=accums)
		assert np.array_equal(accums.cpu().numpy().view(np.uint16), a) and np.array_equal(gd.cpu().numpy(), disp)
	finally:
		m.SetDebug()


def test_pair_pipeline_matches_oracle_and_ground_truth(sgm):
	"""Right->left match, left->right match with mirrored ranges, cross-check, quarter-pixel refinement
	(the non-tSGM level body, SemiGlobalMatcher.cpp:643-725) against the same chain of oracle calls."""
	m, O = sgm
	w, h = 240, 136
	lg, lc, rg, d, rc = synth.make_stereo_pair(w, h, right_color=True)
	# left(x) = right(x + d): the left->right disparity is +d, the right->left one about -d
	ld, rd = m.MatchPairDevice(_dev(lg), _dev(lc), _dev(rg), _dev(rc), -32, 0)
	# default: the two matches on two contexts / streams; one after the other on one context gives the same integers
	ld1, rd1 = m.MatchPairDevice(_dev(lg), _dev(lc), _dev(rg), _dev(rc), -32, 0, overlap=False)
	assert torch.equal(ld, ld1) and torch.equal(rd, rd1)
	ld, rd = ld.cpu().numpy(), rd.cpu().numpy()
	pxr, n = synth.sgm_pixel_map(w, h, -32, 0)
	cr, ar, odr, _ = O.sgm_match(rg, rc, lg, pxr, n)
	pxl, n = synth.sgm_pixel_map(w, h, 0, 32)
	cl, al, odl, _ = O.sgm_match(lg, lc, rg, pxl, n)
	want = O.sgm_refine(pxl, al, O.sgm_cross_check(odl, odr, 1), 4)
	assert (rd != odr).mean() < 0.01
	both = (ld != 32767) & (want != 32767)
	assert ((ld != 32767) != (want != 32767)).mean() < 0.02
	assert (np.abs(ld.astype(np.int32)-want.astype(np.int32))[both] > 1).mean() < 0.02
	gt = d[3:-3, 3:-3]
	err = np.abs(ld[both]/4.0-gt[both])
	assert both.mean() > 0.75 and np.median(err) < 0.2 and (err < 0.5).mean() > 0.9
