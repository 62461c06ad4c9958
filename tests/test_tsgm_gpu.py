"""GPU checks of the hierarchical (tSGM) matcher (run with -m gpu): its building blocks bit for bit against the oracle and OpenCV,
the whole level loop statistically against tsgm_match of oracle/tsgm.py (the WZNCC cost may differ by one uint8 level, see
test_sgm_parity_gpu.py), and the context state it leaves behind."""
import numpy as np
import pytest
import torch

from openmvs_b200 import synth

pytestmark = pytest.mark.gpu
NO = 32767


@pytest.fixture(scope="module")
def sgm():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	from oracle import tsgm as O
	from openmvs_b200.depth_estimator import SemiGlobalMatcher
	m = SemiGlobalMatcher()
	yield m, O
	m.Release()


def _dev(a):
	return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _estimator_like_map(rng, h, w):
	"""int16 disparities as a matcher leaves them: smooth surfaces with steps, noise, NO_DISP holes and speckles"""
	ys, xs = np.mgrid[0:h, 0:w]
	d = 20+8*np.sin(xs/17.0)*np.cos(ys/23.0)+6*((xs//40+ys//30) % 3)
	d = np.rint(d+rng.randn(h, w)*1.5).astype(np.int16)
	d[rng.rand(h, w) < 0.15] = NO
	spk = rng.rand(h, w) < 0.03
	d[spk] = rng.randint(-60, 60, int(spk.sum()))
	d[10:30, 40:90] = NO
	return d


@pytest.mark.parametrize("first", [True, False])
def test_range_map_bit_exact(sgm, first):
	m, O = sgm
	rng = np.random.RandomState(3)
	h, w = 61, 87
	D = _estimator_like_map(rng, h, w)
	M = np.full((2*h+6, 2*w+7), 255, np.uint8)
	M[rng.rand(*M.shape) < 0.05] = 0
	args = (11, 33) if first else (5, 7)
	px, n = O.tsgm_range_map(D, M, *args)
	gpx, gn = m.Disparity2RangeMap(_dev(D), _dev(M), *args)
	assert gn == n
	assert np.array_equal(gpx.cpu().numpy().view(O.SGM_PIXEL).ravel(), px)


def test_flip_upscale_extract_bit_exact(sgm):
	m, O = sgm
	rng = np.random.RandomState(4)
	h, w = 70, 130
	D = _estimator_like_map(rng, h, w)
	assert np.array_equal(m.FlipDirection(_dev(D)).cpu().numpy(), O.tsgm_flip_direction(D))
	mask = (rng.rand(h, w) < 0.8).astype(np.uint8)*255
	for size2x in ((2*w+7, 2*h+6), (2*w+5, 2*h+5)):
		assert np.array_equal(m.UpscaleMask(_dev(mask), size2x).cpu().numpy(), O.tsgm_upscale_mask(mask, size2x))
	for th in (1, 3, 7):
		assert np.array_equal(m.ExtractMask(_dev(D), _dev(mask), th).cpu().numpy(), O.tsgm_extract_mask(D, mask, th))


@pytest.mark.parametrize("size", [20, 100, 1000])
def test_filter_speckles_matches_opencv(sgm, size):
	import cv2
	m, O = sgm
	rng = np.random.RandomState(size)
	for h, w in ((120, 200), (263, 471)):
		D = _estimator_like_map(rng, h, w)
		want = D.copy()
		cv2.filterSpeckles(want, NO, size, 5)
		got = m.FilterSpeckles(_dev(D), NO, size, 5).cpu().numpy()
		assert np.array_equal(got, want)
		assert (want != D).any()


def test_area_pyramid_and_level_mask_match_opencv(sgm):
	import cv2
	m, O = sgm
	rng = np.random.RandomState(5)
	for h, w in ((270, 480), (271, 483), (135, 241), (1080, 1920)):
		img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
		for f in (2, 4, 8):
			want = cv2.resize(img, None, fx=1.0/f, fy=1.0/f, interpolation=cv2.INTER_AREA)
			got = m.ResizeAreaU8(_dev(img), f).cpu().numpy()
			assert got.shape == want.shape and np.array_equal(got, want), (h, w, f)
	mask = np.full((361, 641), 255, np.uint8)
	mask[rng.rand(361, 641) < 0.3] = 0
	mask[:, 500:520] = 0
	for lw, lh in ((160, 90), (321, 181), (641, 361)):
		want = cv2.resize(mask, (lw, lh), interpolation=cv2.INTER_NEAREST)[3:lh-3, 3:lw-3]
		assert np.array_equal(m.LevelMask(_dev(mask), (lw, lh)).cpu().numpy(), want)


def _init_map(d, sizes, init_size):
	"""the initial map a caller derives from sparse points: ground truth at half the coarsest level, every other pixel"""
	lw, lh = sizes[0]
	iw, ih = init_size
	s = 0.5*lw/d.shape[1]
	ys, xs = np.mgrid[0:ih, 0:iw]
	src = d[np.clip(np.rint((ys+3)/s).astype(int), 0, d.shape[0]-1), np.clip(np.rint((xs+3)/s).astype(int), 0, d.shape[1]-1)]
	init = np.rint(src*s).astype(np.int16)
	init[(xs+ys) % 2 == 1] = NO
	return init


CASES = [
	# (w, h, minResolution, initial map, masked band)
	(400, 240, 160, False, False),
	(400, 240, 160, True, False),
	(640, 360, 160, False, False),
	(640, 360, 160, True, True),
	(400, 240, 160, False, True),
	(400, 240, 0, True, False),
]


@pytest.mark.parametrize("w,h,minRes,with_init,masked", CASES)
def test_hierarchical_match_against_oracle(sgm, w, h, minRes, with_init, masked):
	m, O = sgm
	lg, lc, rg, d, rc = synth.make_stereo_pair(w, h, right_color=True)
	sizes, init_size = m.HierarchyLevels(w, h, minRes)
	init = _init_map(d, sizes, init_size) if with_init else None
	lm = rm = None
	if masked:
		lm = np.full((h, w), 255, np.uint8); lm[:, w//3:w//3+25] = 0
		rm = np.full((h, w), 255, np.uint8); rm[h//2:h//2+20, :] = 0
	if minRes == 0:
		init = -init   # the fixed-range branch searches the initial map's range for the right->left match, its mirror for the left one
	od, oc, olev = O.tsgm_match(lg, lc, rg, rc, init, lm, rm, minResolution=minRes)
	gd, gc, glev = m.MatchPairHierarchicalDevice(_dev(lg), _dev(lc), _dev(rg), _dev(rc), None if init is None else _dev(init),
		None if lm is None else _dev(lm), None if rm is None else _dev(rm), minResolution=minRes)
	gd = gd.cpu().numpy()
	assert [l["size"] for l in glev] == [l["size"] for l in olev] == sizes
	gv, ov = gd != NO, od != NO
	both = gv & ov
	equal = float((gd == od)[both].mean())
	valid_agree = float((gv == ov).mean())
	gt = d[3:-3, 3:-3]*4
	inner = np.zeros_like(gv); inner[8:-8, 8:-8] = True
	acc = lambda disp, v: float(((np.abs(disp.astype(np.float64)-gt) <= 4) & v & inner).sum()/inner.sum())
	gacc, oacc = acc(gd, gv), acc(od, ov)
	print("tsgm %dx%d min %d init %d mask %d: levels %s numCosts gpu %s oracle %s; equal %.4f valid-agree %.4f acc gpu %.4f oracle %.4f" % (
		w, h, minRes, with_init, masked, sizes, [l["numCosts"] for l in glev], [l["numCosts"] for l in olev], equal, valid_agree, gacc, oacc))
	assert equal >= 0.99 and valid_agree >= 0.99
	assert gacc >= oacc-0.005
	if masked:
		assert not gv[:, w//3:w//3+25-6].any()


def test_fixed_range_without_valid_initial_value_is_refused(sgm):
	m, O = sgm
	from openmvs_b200 import lib
	lg, lc, rg, d, rc = synth.make_stereo_pair(200, 120, right_color=True)
	sizes, (iw, ih) = m.HierarchyLevels(200, 120, 0)
	init = torch.full((ih, iw), NO, dtype=torch.int16, device="cuda")
	with pytest.raises(lib.B200MVSError):
		m.MatchPairHierarchicalDevice(_dev(lg), _dev(lc), _dev(rg), _dev(rc), init, minResolution=0)
	with pytest.raises(lib.B200MVSError):
		m.MatchPairHierarchicalDevice(_dev(lg), _dev(lc), _dev(rg), _dev(rc), None, minResolution=0)


def test_fixed_range_pair_unchanged_by_a_hierarchical_call(sgm):
	m, O = sgm
	lg, lc, rg, d, rc = synth.make_stereo_pair(240, 136, right_color=True)
	args = (_dev(lg), _dev(lc), _dev(rg), _dev(rc))
	ld0, rd0 = m.MatchPairDevice(*args, -32, 0)
	ld0, rd0 = ld0.clone(), rd0.clone()
	# a match of another caller on this context, whose accumulated costs a refinement could take (accums = NULL) ...
	from openmvs_b200 import lib
	px, n = synth.sgm_pixel_map(240, 136, 0, 32)
	pxd = _dev(px.view(np.uint8).reshape(-1, 16))
	disp, _ = m.MatchDevice(args[0], args[1], args[2], pxd, n)
	m.RefineDisparityMap(disp.clone(), pxd, None, 4)
	m.MatchPairHierarchicalDevice(*args, minResolution=100)
	# ... is no longer on the context after the hierarchy: the refinement refuses instead of reading another volume
	with pytest.raises(lib.B200MVSError):
		m.RefineDisparityMap(disp.clone(), pxd, None, 4)
	ld1, rd1 = m.MatchPairDevice(*args, -32, 0)
	assert torch.equal(ld0, ld1) and torch.equal(rd0, rd1)
