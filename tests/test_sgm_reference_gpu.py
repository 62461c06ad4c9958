"""The SGM matcher's floating-point kernels against the float64 references of tests/test_sgm_reference.py (run with -m gpu).

Both cost kernels (`sgm_cost_kernel`, SIMT, `SetDebug(sgmCost=1)`; `sgm_cost_tc_kernel`, tensor cores, `sgmCost=2`) must equal
`wzncc64` on every decidable entry, differ by at most one level elsewhere, and equal it wherever the window leaves the right image.
The sub-pixel refinement must equal `lc_blend64` where decidable, the cross-check `cross_check_ref` everywhere."""
import numpy as np
import pytest
import torch

from openmvs_b200 import synth
from test_sgm_reference import (CONTENT, NO_DISP, check_refine, check_volume, cross_check_case, cross_check_ref, lc_blend64,
	make_content, max_undecidable, refine_case, wzncc64)

pytestmark = pytest.mark.gpu

# power checks of the tensor-core kernel: its margin is 4x the float32 one (U_TC), and so is its undecidable fraction (measured:
# up to 6.4 % per case, 17.2 % on the textureless one)
MAX_UNDECIDABLE_TC = 0.08
MAX_UNDECIDABLE_TC_TEXTURELESS = 0.20


@pytest.fixture(scope="module")
def sgm():
	if not torch.cuda.is_available():
		pytest.skip("no CUDA device")
	from openmvs_b200.depth_estimator import SemiGlobalMatcher
	m = SemiGlobalMatcher()
	yield m
	m.Release()


def _dev(a):
	return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _px_dev(px):
	return torch.from_numpy(px.view(np.uint8).reshape(-1, 16).copy()).cuda()


def _costs(m, lg, lc, rg, px, n, kernel):
	out = torch.full((n,), 7, dtype=torch.uint8, device="cuda")
	try:
		m.SetDebug(sgmCost=kernel)
		m.MatchDevice(_dev(lg), _dev(lc), _dev(rg), _px_dev(px), n, stages=1, costs=out)
	finally:
		m.SetDebug()
	return out.cpu().numpy()


def _tc_cap(kind):
	return MAX_UNDECIDABLE_TC_TEXTURELESS if kind == "textureless" else MAX_UNDECIDABLE_TC


@pytest.mark.parametrize("kind", CONTENT)
@pytest.mark.parametrize("num,dmin,w", [(64, -70, 262), (128, -40, 135), (192, 3, 261), (256, -100, 262), (128, 60, 134)])
def test_tensor_core_cost_kernel(sgm, kind, num, dmin, w):
	"""D = 64 / 128 / 192 / 256; valid widths 256, 129, 255, 128 (vw % 128 = 0, 1, 127, 0); windows leave the right image on the
	left (dmin < 0) and on the right (dmin + D beyond the image)"""
	h = 26
	lg, lc, rg = make_content(w, h, kind, d0=12.0 if dmin < 40 else 70.0)
	px, n = synth.sgm_pixel_map(w, h, dmin, dmin+num)
	ref = wzncc64(lg, lc, rg, px, tc=True)
	check_volume("tc %s D=%d dmin=%d vw=%d" % (kind, num, dmin, w-6), _costs(sgm, lg, lc, rg, px, n, 2), ref, max_undecidable=_tc_cap(kind))


def test_tensor_core_cost_kernel_many_rows_per_cta(sgm):
	"""More than twice as many valid rows as SMs: every persistent CTA computes at least three rows, so the window prefetched for
	the CTA's next row during the last block of a row, and the restart of the B-tile ring, are compared entry by entry"""
	sms = torch.cuda.get_device_properties(0).multi_processor_count
	w, vh = 135, 2*sms+sms//2+5
	h = vh+6
	lg, lc, rg, _ = synth.make_stereo_pair(w, h, d0=20.0, amp=8.0)
	px, n = synth.sgm_pixel_map(w, h, 0, 64)
	ref = wzncc64(lg, lc, rg, px, tc=True)
	check_volume("tc %d rows" % vh, _costs(sgm, lg, lc, rg, px, n, 2), ref, max_undecidable=MAX_UNDECIDABLE_TC)


@pytest.mark.parametrize("kind", CONTENT)
def test_simt_cost_kernel_ragged(sgm, kind):
	"""Per-pixel ranges of widths 1-256 (every width % 4, so the 4-disparity chunk loop ends with 0-3 lanes of a chunk), 7 %
	invalid pixels between valid ones, ranges wholly left and wholly right of the right image (all 255), negative and positive
	dmin"""
	w, h = 90, 24
	vw, vh = w-6, h-6
	rng = np.random.RandomState(CONTENT.index(kind))
	lg, lc, rg = make_content(w, h, kind)
	lo = rng.randint(-60, 40, (vh, vw)); wd = rng.randint(1, 257, (vh, vw))
	wd[0, :16] = np.arange(1, 17)                      # widths 1-16: every width % 4, ranges 1-3 wide
	wd[1, :4] = 256
	lo[2, :8] = -300; wd[2, :8] = 40                   # wholly left of the right image
	lo[3, :8] = w; wd[3, :8] = 9                       # wholly right of it
	invalid = rng.rand(vh, vw) < 0.07
	invalid[:4] = False
	px, n = synth.sgm_pixel_map(w, h, lo, lo+wd, invalid)
	ref = wzncc64(lg, lc, rg, px)
	check_volume("simt ragged %s" % kind, _costs(sgm, lg, lc, rg, px, n, 1), ref, max_undecidable=max_undecidable(kind))
	for r in (2, 3):   # the wholly outside ranges: 255, margin 0 (exact)
		o = int(px["idx"][r*vw])
		assert (ref[0][o:o+8*int(wd[r, 0])] == 255).all() and (ref[2][o:o+8*int(wd[r, 0])] == 0).all()


@pytest.mark.parametrize("kind", CONTENT)
@pytest.mark.parametrize("num,dmin", [(36, -20), (100, 5)])
def test_simt_cost_kernel_uniform(sgm, kind, num, dmin):
	"""one range of 36 or 100 disparities (not a tensor-core width: the SIMT kernel is the default there)"""
	w, h = 131, 22
	lg, lc, rg = make_content(w, h, kind)
	px, n = synth.sgm_pixel_map(w, h, dmin, dmin+num)
	ref = wzncc64(lg, lc, rg, px)
	check_volume("simt %s [%d,%d)" % (kind, dmin, dmin+num), _costs(sgm, lg, lc, rg, px, n, 1), ref, max_undecidable=max_undecidable(kind))
	# the automatic choice is the SIMT kernel too
	assert np.array_equal(_costs(sgm, lg, lc, rg, px, n, 0), _costs(sgm, lg, lc, rg, px, n, 1))


@pytest.mark.parametrize("steps", [2, 4, 8, 16])
def test_refinement_kernel(sgm, steps):
	"""sgm_refine_kernel on accumulated costs and disparities built directly: every branch of the LC blend, uint16 costs up to
	65535, wrapped differences, widths 1 and 2, NO_DISP, negative ranges, and disparities past the range (left unchanged)"""
	px, a, disp = refine_case(steps, vw=121, vh=41)
	got = sgm.RefineDisparityMap(_dev(disp), _px_dev(px), accums=_dev(a.view(np.int16)), subpixelSteps=steps).cpu().numpy()
	ref = lc_blend64(px, a, disp, steps)
	check_refine("refine steps=%d" % steps, got, ref)
	lo, hi = px["dmin"].reshape(disp.shape), px["dmax"].reshape(disp.shape)
	untouched = (disp == NO_DISP) | (hi-lo < 2) | (disp < lo) | (disp >= hi)
	assert np.array_equal(got[untouched], disp[untouched])
	assert ((disp >= hi) & (hi-lo >= 2) & (disp != NO_DISP)).sum() > 20


@pytest.mark.parametrize("th", [0, 1, 2, 5])
@pytest.mark.parametrize("sign", [1, -1])
def test_cross_check_kernel(sgm, th, sign):
	l2r, r2l = cross_check_case(257, 31, sign, th, seed=10+th)
	want = cross_check_ref(l2r, r2l, th)
	got = sgm.ConsistencyCrossCheck(_dev(l2r), _dev(r2l), th).cpu().numpy()
	assert np.array_equal(got, want)
