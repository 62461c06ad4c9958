"""Float64 references of the SGM matcher's floating-point stages, and the CPU oracle pinned to them (no GPU).

* `wzncc64`       the WZNCC cost volume (SemiGlobalMatcher.cpp:875-985) in float64, with a first-order forward-error margin
* `lc_blend64`    RefineDisparityMap with SUBPIXEL_LC_BLEND (SemiGlobalMatcher.cpp:1693-1811) in float64, with a margin
* `cross_check_ref` ConsistencyCrossCheck (SemiGlobalMatcher.cpp:1449-1489) on integers

An entry is *decidable* when its unrounded value lies farther than the margin from every rounding boundary: a float32
evaluation of the same formula then rounds to the same integer, so the oracle and both cost kernels must equal the reference
there, and may differ by at most one level elsewhere.  `tests/test_sgm_reference_gpu.py` holds the kernels to the same rule.
"""
import numpy as np
import pytest

from openmvs_b200 import synth

HW = 3
NO_DISP = 32767
_f32 = np.float32

# the reference's float32 constants (SemiGlobalMatcher.cpp:877,912,917), promoted to float64; everything after them is float64
SIGMA_COLOR = float(_f32(-1)/(_f32(2)*(_f32(0.3)*_f32(255))*(_f32(0.3)*_f32(255))))
SIGMA_SPATIAL = float(_f32(-1)/(_f32(2)*(_f32(0.4)*_f32(7))*(_f32(0.4)*_f32(7))))
EPS = float(_f32(1e-3))

U_SIMT = 2.0**-22
"""Unit roundoff of the cost margin for a float32 evaluation (the oracle, `sgm_cost_kernel`).

The margin charges one U per elementary operation (relative to its result) and one U per accumulated sum (relative to the sum
of the absolute values of its terms); each weight carries U (1 + |a|), a = its exponent.  U = 2^-22 = 4 u, u = 2^-24 the float32
unit roundoff, covers:
* every correctly rounded operation (u), and CUDA's `expf` / `sqrtf` / division (<= 2 ulp = 2u);
* the exponent of a weight, s*sigmaColor + r*sigmaSpatial, rounded up to three times (product, product, sum; or one FMA and
  a rounded constant): <= 3u |a|, which `exp` turns into a relative error of the weight of 3u |a| <= U |a|;
* a 49-term sum in any order, with or without FMA.  Its rounding errors are independent and of either sign, so they add like a
  random walk: a sum of positive terms whose partial sums grow to S errs by sqrt(sum_k (S_k)^2 / 3) u ~ 2.3 u S (standard
  deviation) in sequential order, less in a tree.  The margin adds the bounds of all sums and operations of an entry in absolute
  value (about fifteen independent contributions), so the level's total error is far inside it although a single sum may exceed
  4u of its absolute sum: a float32 evaluation that rounds to a different integer than the float64 value on a decidable entry
  is a bug, not noise.
The constant is fixed by this argument, not by any kernel's output."""

U_TC = 2.0**-20
"""Unit roundoff of the cost margin for the tensor-core kernel (`sgm_cost_tc_kernel`).

Each operand x (weight, weight * (g - mean), right gray f, f^2) is split into fp16 hi = rn(x) and lo = rn(x - hi), and the
product x y is taken as hi_x hi_y + hi_x lo_y + lo_x hi_y.  With the fp16 unit roundoff 2^-11, |x - hi - lo| <= 2^-22 |x| for each
operand and the dropped lo_x lo_y is <= 2^-22 |x y|: a product errs by <= 3 * 2^-22 relative.  The fp32 accumulation inside the
MMA (alignment and normalisation may truncate) and across the 12 MMAs of a sum adds about 2^-22 more.  So U_TC = 2^-20 = 4 * 2^-22
bounds the per-product error and the accumulation as U_SIMT does for float32.  `ex2.approx` (<= 2 ulp) and the rounded
log2(e) factor in its argument are covered as `expf` is for U_SIMT.  Operands in the fp16 subnormal range lose relative
precision: see FP16_ABS."""

FP16_ABS = 2.0**-25
"""Absolute error of one fp16 hi/lo split below the normal range.  Below 2^-14 the fp16 spacing is 2^-24, so hi and lo each
round with an absolute error of at most 2^-25: a weight as small as exp(-17.8) ~ 1.9e-8 (saturated colour contrast at the window
corner) keeps no relative precision at all, and neither does a lo part below 2^-14 (an operand below 2^-3).  For the tensor-core
kernel each product x y therefore errs by up to FP16_ABS (|x| + |y|) on top of the relative U_TC: this term is added to the
sums' error bounds separately."""


# ---- WZNCC cost ------------------------------------------------------------------------------------------------------------------

_TI, _TJ = np.divmod(np.arange(49), 7)
_TI = _TI-HW
_TJ = _TJ-HW


def _pixels(px, vw):
	valid = np.flatnonzero(px["dmin"] < px["dmax"])
	r, c = np.divmod(valid, vw)
	return valid, r, c


def wzncc64(left_gray, left_bgr, right_gray, pixel_map, tc=False, chunk=40000):
	"""-> (expected u8 as int32, unrounded level float64, margin float64), one entry per cost of the volume (numCosts = the end
	of the last slice).  Expected: 255 where the window leaves the right image or ncc <= 0, floor((1 - min(ncc, 1)) * 255 + .5)
	otherwise.  The level is 255 (1 - clip(ncc, 0, 1)), so the ncc = 0 and ncc = 1 switches are boundaries of the rounded value
	exactly where they change it (they never do: the level is continuous across both).  Entries outside the right image have
	margin 0.  tc: the tensor-core kernel's error model (U_TC and the fp16 absolute error), else float32 (U_SIMT)."""
	lg = np.asarray(left_gray, np.float64); rg = np.asarray(right_gray, np.float64)
	lc = np.asarray(left_bgr, np.int64)
	h, w = lg.shape
	vw = w-2*HW
	px = np.ascontiguousarray(pixel_map)
	U = U_TC if tc else U_SIMT
	e16 = FP16_ABS if tc else 0.0
	num = np.maximum(px["dmax"].astype(np.int64)-px["dmin"].astype(np.int64), 0)
	n_costs = int((px["idx"].astype(np.int64)+num).max()) if len(px) else 0
	exp_ = np.full(n_costs, -1, np.int32); lev = np.zeros(n_costs); mar = np.zeros(n_costs)
	valid, R, Cc = _pixels(px, vw)
	if not len(valid):
		return exp_, lev, mar
	uy, ux = R+HW, Cc+HW
	# per pixel: bilateral weights, their relative error (in units of U), the patch mean and tempWeights
	yy, xx = uy[:, None]+_TI, ux[:, None]+_TJ
	dc = lc[yy, xx]-lc[uy, ux][:, None, :]
	s = (dc*dc).sum(-1).astype(np.float64)
	a = s*SIGMA_COLOR+(_TI*_TI+_TJ*_TJ).astype(np.float64)*SIGMA_SPATIAL
	wt = np.exp(a)
	ew = 1.0+np.abs(a)
	g = lg[yy, xx]
	sumW = wt.sum(1)
	eW = (wt*(1.0+ew)).sum(1)                                  # sumW: accumulation + weights
	accG = (g*wt).sum(1)
	tm = accG/sumW
	t = g-tm[:, None]
	# the mean: accumulations of acc (with its products) and sumW, the division; the weights' errors enter a weighted mean only
	# through g - tm
	etm = 2.0*accG/sumW+accG/sumW+np.abs(tm)+(wt*ew*np.abs(t)).sum(1)/sumW
	tw = wt*t
	N0 = (tw*t).sum(1)
	# dN0/dtm = -2 sum w t (zero in exact arithmetic): the mean's error enters only through it
	eN0 = (tw*t*(ew+4.0)).sum(1)+2.0*np.abs((wt*t).sum(1))*etm
	# entries
	lo = px["dmin"][valid].astype(np.int64); cnt = num[valid]
	e_pix = np.repeat(np.arange(len(valid)), cnt)
	first = np.repeat(np.cumsum(cnt)-cnt, cnt)
	e_k = np.arange(len(e_pix))-first
	e_d = lo[e_pix]+e_k
	e_pos = px["idx"][valid].astype(np.int64)[e_pix]+e_k
	for b in range(0, len(e_pix), chunk):
		sl = slice(b, b+chunk)
		p, d, pos = e_pix[sl], e_d[sl], e_pos[sl]
		x0 = ux[p]+d
		outside = (x0-HW < 0) | (x0+HW >= w)
		cols = np.clip(x0[:, None]+_TJ, 0, w-1)
		f = rg[uy[p][:, None]+_TI, cols]
		W, TW, EW = wt[p], tw[p], ew[p]
		fw = f*W
		sm = fw.sum(1); sq = (f*fw).sum(1); nom = (f*TW).sum(1)
		e_sm = U*(fw*(EW+2.0)).sum(1)+e16*(f+W).sum(1)
		e_sq = U*(f*fw*(EW+3.0)).sum(1)+e16*(f*f+W).sum(1)
		e_nom = U*((np.abs(f*TW)*(EW+4.0)).sum(1)+np.abs(sm)*etm[p])+e16*(np.abs(f)+np.abs(TW)).sum(1)
		sw = sumW[p]
		N1 = sq-sm*sm/sw
		e_N1 = e_sq+2.0*np.abs(sm)/sw*e_sm+sm*sm/sw**2*U*eW[p]+U*(np.abs(sq)+2.0*sm*sm/sw)
		n0 = N0[p]
		D = n0*N1+EPS
		e_D = np.abs(N1)*U*eN0[p]+np.abs(n0)*e_N1+2.0*U*(np.abs(n0*N1)+EPS)
		ncc = nom/np.sqrt(D)
		e_ncc = e_nom/np.sqrt(D)+np.abs(ncc)/(2.0*D)*e_D+2.0*U*np.abs(ncc)
		L = 255.0*(1.0-np.clip(ncc, 0.0, 1.0))
		M = 255.0*e_ncc+U*766.0                                  # 1 - ncc, * 255, + .5
		E = np.floor(L+0.5).astype(np.int32)
		E[outside] = 255; L[outside] = 255.0; M[outside] = 0.0
		exp_[pos] = E; lev[pos] = L; mar[pos] = M
	return exp_, lev, mar


def decidable(level, margin):
	"""no rounding boundary k + 1/2 within the margin of the unrounded value"""
	return np.floor(level-margin+0.5) == np.floor(level+margin+0.5)


def check_volume(name, got, ref, report=True, max_undecidable=None):
	"""got: uint8 volume; ref: wzncc64's triple.  Equal on every decidable entry, within one level elsewhere.
	-> (entries, undecidable fraction, entries that differ by one)"""
	want, level, margin = ref
	got = np.asarray(got).astype(np.int32)
	assert got.shape == want.shape and (want >= 0).all()
	dec = decidable(level, margin)
	diff = np.abs(got-want)
	bad = np.flatnonzero(dec & (diff != 0))
	assert len(bad) == 0, "%s: %d decidable entries differ, e.g. %s" % (name, len(bad), [
		(int(i), int(got[i]), int(want[i]), float(level[i]), float(margin[i])) for i in bad[:5]])
	assert diff.max(initial=0) <= 1, (name, int(diff.max()))
	und = float(1.0-dec.mean())
	if report:
		print("%s: %d entries, undecidable %.3f %%, %d differ by one" % (name, len(want), 100*und, int((diff == 1).sum())))
	if max_undecidable is not None:
		assert und <= max_undecidable, (name, und)
	return len(want), und, int((diff == 1).sum())


# ---- images where the formula changes regime -------------------------------------------------------------------------------------

CONTENT = ("smooth", "textureless", "anticorrelated", "identical", "saturated", "gray01")


def make_content(w, h, kind, seed=0, d0=12.0):
	"""A rectified pair (left gray, left BGR, right gray) on which one regime of the cost formula covers about half of the image:
	smooth          synth.make_stereo_pair as it is
	textureless     both images flattened to a contrast of 2 %: normSq0 * normSq1 << eps, eps decides the cost
	anticorrelated  right = 1 - right: at the true disparity ncc ~ -1 (cost 255)
	identical       left(x) = right(x + d0) with an integer d0, contrast x3: at d0 the windows are equal and ncc ~ 1 (cost 0)
	saturated       left BGR random 0 / 255 per channel: colour distances up to 3 * 255^2, weights down to exp(-17.8) ~ 1.9e-8
	gray01          gray values exactly 0 and 1 (thresholded texture) and constant 0 / 1 patches"""
	lg, lc, rg, d = synth.make_stereo_pair(w, h, seed=7+seed, d0=d0, amp=0.0 if kind == "identical" else 6.0)
	lg = lg.copy(); lc = lc.copy(); rg = rg.copy()
	rng = np.random.RandomState(100+seed)
	blk = np.s_[:, w//4:3*w//4]
	if kind == "textureless":
		for im in (lg, rg):
			im[blk] = (0.5+0.02*(im[blk]-0.5)).astype(np.float32)
	elif kind == "anticorrelated":
		rg[blk] = (1.0-rg[blk]).astype(np.float32)
	elif kind == "identical":
		# amp = 0: the true disparity is d0 everywhere, and the left image is the right one shifted by whole pixels
		k = int(round(d0))
		rg[:] = np.clip(0.5+3.0*(rg-0.5), 0.0, 1.0)            # strong contrast: normSq0 >> eps, so ncc reaches 1 - 1e-4
		lg[:, :w-k] = rg[:, k:]
	elif kind == "saturated":
		lc[blk] = (rng.randint(0, 2, lc[blk].shape)*255).astype(np.uint8)
	elif kind == "gray01":
		for im in (lg, rg):
			im[blk] = np.where(im[blk] < 0.5, 0.0, 1.0).astype(np.float32)
		lg[:h//3, :w//3] = 0.0; rg[:h//3, :w//3] = 0.0
		lg[2*h//3:, 2*w//3:] = 1.0; rg[2*h//3:, 2*w//3:] = 1.0
	elif kind != "smooth":
		raise ValueError(kind)
	return lg, lc, rg


# ---- sub-pixel refinement ------------------------------------------------------------------------------------------------------

_C13 = float(_f32(np.pi/3.0))
_C23 = float(_f32(np.pi/2.3))
_F1195 = float(_f32(1.195))


def lc_blend64(pixel_map, accums, disparity, steps):
	"""RefineDisparityMap, SUBPIXEL_LC_BLEND, in float64 -> (expected int16, unrounded disparity * steps, margin).
	Untouched (margin 0): ranges narrower than 2, NO_DISP, and disparities outside the pixel's [dmin, dmax).  prev - center and
	next - center are uint16 differences, so they wrap when the disparity is not the slice's minimum, as the reference's AccumCost
	arithmetic does.  semisubpixel(primary, 0) is 0 (the reference would divide by zero).  The constants are the reference's
	float32 ones.  Margin: float32 disp = d + off at |d| <= 256 rounds by <= u (|d| + 1); the offset itself (a rounded ratio, two
	cosf of <= 2 ulp, about ten more roundings of values below 1.2, slopes below 2) by <= 40 u; the product with steps and the
	+ 0.5 by <= u steps (|d| + 2) each; u = 2^-24."""
	px = np.ascontiguousarray(pixel_map)
	a = np.asarray(accums).view(np.uint16).astype(np.int64)
	d = np.asarray(disparity, np.int16).ravel().astype(np.int64)
	lo = px["dmin"].astype(np.int64); hi = px["dmax"].astype(np.int64); idx = px["idx"].astype(np.int64)
	out = d.copy(); val = d.astype(np.float64)*steps; mar = np.zeros(len(d))
	act = (hi-lo >= 2) & (d != NO_DISP) & (d >= lo) & (d < hi)
	i = np.flatnonzero(act)
	if steps <= 1 or not len(i):
		return out.astype(np.int16).reshape(np.shape(disparity)), val.reshape(np.shape(disparity)), mar.reshape(np.shape(disparity))
	k = idx[i]+d[i]-lo[i]
	at_lo = d[i] == lo[i]; at_hi = (~at_lo) & (d[i]+1 == hi[i]); mid = ~(at_lo | at_hi)
	last = len(a)-1
	cen = a[k]; prv = a[np.clip(k-1, 0, last)]; nxt = a[np.clip(k+1, 0, last)]

	def semi(p, o):
		return np.where(o == 0, 0.0, 0.5*p/np.where(o == 0, 1, o))

	def blend(x):
		cosine = 1.0-np.cos(x*_C13)
		factor = _F1195-np.cos(x*_C23)
		return cosine*factor+x/2.0*(1.0-factor)

	off = np.zeros(len(i))
	off[at_lo] = semi(cen, nxt)[at_lo]
	off[at_hi] = -semi(cen, prv)[at_hi]
	pc, cn = prv == cen, cen == nxt
	ld = (prv-cen) & 0xFFFF; rd = (nxt-cen) & 0xFFFF
	lt = ld < rd
	x = np.where(lt, ld/np.maximum(rd, 1), rd/np.maximum(ld, 1))
	lcb = (blend(x)-0.5)*np.where(lt, 1.0, -1.0)
	m = np.where(pc, np.where(cn, 0.0, semi(cen, nxt)), np.where(cn, -semi(cen, prv), lcb))
	off[mid] = m[mid]
	v = (d[i]+off)*steps
	out[i] = np.floor(v+0.5).astype(np.int64)
	val[i] = v
	mar[i] = 2.0**-24*(np.abs(d[i])+1+40+2*steps*(np.abs(d[i])+2))
	shape = np.shape(disparity)
	return out.astype(np.int16).reshape(shape), val.reshape(shape), mar.reshape(shape)


def check_refine(name, got, ref, report=True):
	want, value, margin = ref
	got = np.asarray(got).astype(np.int32); want = want.astype(np.int32)
	dec = decidable(value, margin)
	diff = np.abs(got-want)
	bad = np.flatnonzero((dec & (diff != 0)).ravel())
	assert len(bad) == 0, "%s: %d decidable entries differ, e.g. %s" % (name, len(bad), [
		(int(j), int(got.ravel()[j]), int(want.ravel()[j]), float(value.ravel()[j])) for j in bad[:5]])
	assert diff.max(initial=0) <= 1, (name, int(diff.max()))
	und = float(1.0-dec.mean())
	if report:
		print("%s: %d pixels, undecidable %.3f %%, %d differ by one" % (name, got.size, 100*und, int((diff == 1).sum())))
	return und


def refine_case(steps, seed=0, vw=61, vh=23):
	"""A pixel map, accumulated costs and disparities built directly (no matching) -> (px, accums u16, disparity i16).
	Ranges: widths 1 and 2 (left untouched: width 1; width 2 has only the two end branches), negative and positive dmin, up to 256
	wide; invalid pixels.  Costs: random uint16 up to 65535, with rows of plateaus (prev == center == next, prev == center,
	center == next), equal neighbour differences (ld == rd), ratios near 0 and near 1, and zero neighbours (other == 0).
	Disparities: the slice's arg-min mostly, also dmin, dmax - 1, NO_DISP, an interior non-minimum (the uint16 differences wrap),
	and a value past dmax - 1 at pixels that have a following slice (left unchanged)."""
	rng = np.random.RandomState(1000*steps+seed)
	n = vw*vh
	width = rng.choice([1, 2, 3, 5, 17, 64, 255, 256], n, p=[.06, .1, .14, .2, .2, .15, .1, .05])
	dmin = rng.randint(-300, 60, n)
	inval = rng.rand(n) < 0.05
	px = np.zeros(n, dtype=np.dtype([("idx", "<u8"), ("dmin", "<i2"), ("dmax", "<i2"), ("reserved", "<i4")]))
	px["dmin"] = np.where(inval, NO_DISP, dmin); px["dmax"] = np.where(inval, NO_DISP, dmin+width)
	cnt = np.where(inval, 0, width)
	px["idx"] = np.concatenate([[0], np.cumsum(cnt)[:-1]])
	a = np.zeros(int(cnt.sum()), np.int64)
	disp = np.full(n, NO_DISP, np.int64)
	for p in range(n):
		if inval[p]:
			continue
		W = int(width[p]); o = int(px["idx"][p]); lo = int(dmin[p])
		kind = p % 9
		seg = rng.randint(0, 65536, W)
		if kind == 1:
			seg = rng.randint(0, 4, W)*rng.randint(1, 20000)       # plateaus and zeros
		elif kind == 2:
			seg = np.full(W, rng.randint(0, 65536))                # flat
		elif kind == 3 and W >= 3:
			j = rng.randint(1, W-1); c = rng.randint(0, 30000); dd = rng.randint(1, 30000)
			seg[j] = c; seg[j-1] = c+dd; seg[j+1] = c+dd               # ld == rd
		elif kind == 4 and W >= 3:
			j = rng.randint(1, W-1); c = rng.randint(0, 1000)
			seg[j] = c; seg[j-1] = c+rng.randint(1, 4); seg[j+1] = c+rng.randint(30000, 65535-c)   # ratio near 0
		elif kind == 5 and W >= 3:
			j = rng.randint(1, W-1); c = rng.randint(0, 20000); dd = rng.randint(20000, 40000)
			seg[j] = c; seg[j-1] = c+dd; seg[j+1] = c+dd+rng.randint(1, 3)                        # ratio near 1
		elif kind == 6:
			seg[:] = np.sort(seg)                                   # minimum at dmin, next may be 0
			seg[0] = 0
		a[o:o+W] = seg
		sel = rng.rand()
		if sel < 0.6:
			k = int(np.argmin(seg))
		elif sel < 0.7:
			k = 0
		elif sel < 0.8:
			k = W-1
		elif sel < 0.9 and W >= 3:
			k = rng.randint(1, W-1)                                 # interior, usually not the minimum: wrapped differences
		elif sel < 0.95:
			disp[p] = NO_DISP
			continue
		else:
			# outside the range, but with a following slice: the parent kernel's stray reads stay inside the volume
			k = W if p+1 < n and o+W+1 < len(a) else 0
		disp[p] = lo+k
	return px, a.astype(np.uint16), disp.astype(np.int16).reshape(vh, vw)


# ---- cross-check ---------------------------------------------------------------------------------------------------------------

def cross_check_ref(l2r, r2l, th):
	"""ConsistencyCrossCheck on integers: a left disparity survives if it points inside the row, at a valid right disparity rd,
	with |ld + rd| <= th"""
	ld = np.asarray(l2r, np.int16).astype(np.int64)
	rd_map = np.asarray(r2l, np.int16).astype(np.int64)
	h, w = ld.shape
	c = np.arange(w)[None, :]
	vx = c+ld
	inside = (vx >= 0) & (vx < w)
	rd = np.take_along_axis(rd_map, np.clip(vx, 0, w-1), 1)
	ok = inside & (rd != NO_DISP) & (np.abs(ld+rd) <= th)
	keep = (ld == NO_DISP) | ok
	return np.where(keep, ld, NO_DISP).astype(np.int16)


def cross_check_case(w, h, sign, th, seed=0):
	"""l2r / r2l maps with disparities of one sign (positive: left -> right as the matcher's right -> left map; negative: the
	mirror), targets at column 0 and w-1 and outside the image, and NO_DISP on either side; consistent pairs miss by up to th + 1"""
	rng = np.random.RandomState(seed)
	c = np.arange(w)[None, :].repeat(h, 0)
	l2r = (sign*rng.randint(0, 40, (h, w))).astype(np.int64)
	# exact edges: targets at column 0 and at w-1, and one step outside each
	e = rng.rand(h, w)
	l2r = np.where(e < 0.05, -c, l2r); l2r = np.where((e >= 0.05) & (e < 0.1), w-1-c, l2r)
	l2r = np.where((e >= 0.1) & (e < 0.13), -c-1, l2r); l2r = np.where((e >= 0.13) & (e < 0.16), w-c, l2r)
	# right map: mostly consistent (rd = -ld +- small), some NO_DISP
	r2l = rng.randint(-60, 60, (h, w)).astype(np.int64)
	vx = np.clip(c+l2r, 0, w-1)
	cons = rng.rand(h, w) < 0.7
	np.put_along_axis(r2l, vx, np.where(cons, -l2r+rng.randint(-th-1, th+2, (h, w)), np.take_along_axis(r2l, vx, 1)), 1)
	l2r[rng.rand(h, w) < 0.05] = NO_DISP
	r2l[rng.rand(h, w) < 0.05] = NO_DISP
	return l2r.astype(np.int16), r2l.astype(np.int16)


# ---- the oracle pinned to the references ---------------------------------------------------------------------------------------

# Power checks for a float32 evaluation (the oracle and the SIMT kernel): 0.3-1.5 % of the entries are undecidable per case
# (measured on the reference alone, for every case of this file and of the SIMT kernel's tests); the checks allow 2 %.  Textureless
# windows are the exception: there eps makes the level about 8000 times as sensitive to `nom` (255 / sqrt(eps)) as a textured
# window, and the rounding of the patch mean moves `nom` by sum * error(mean), so 3.5-4.8 % of those entries are genuinely
# undecidable; the check allows 6 %.  A margin loosened by a factor of two fails these checks.
MAX_UNDECIDABLE = 0.02
MAX_UNDECIDABLE_TEXTURELESS = 0.06


def max_undecidable(kind):
	return MAX_UNDECIDABLE_TEXTURELESS if kind == "textureless" else MAX_UNDECIDABLE


@pytest.fixture(scope="module")
def O():
	from oracle import oracle
	return oracle


@pytest.mark.parametrize("kind", CONTENT)
@pytest.mark.parametrize("w,h,dmin,dmax", [(114, 34, -4, 28), (94, 24, -30, 70)])
def test_oracle_cost_volume_equals_float64_reference(O, kind, w, h, dmin, dmax):
	lg, lc, rg = make_content(w, h, kind)
	px, n = synth.sgm_pixel_map(w, h, dmin, dmax)
	c, _, _, _ = O.sgm_match(lg, lc, rg, px, n, stage=1)
	ref = wzncc64(lg, lc, rg, px)
	check_volume("oracle %s %dx%d [%d,%d)" % (kind, w, h, dmin, dmax), c, ref, max_undecidable=max_undecidable(kind))


def test_oracle_cost_volume_ragged_ranges(O):
	"""per-pixel ranges of widths 1-256 (every width % 4), ranges wholly outside the right image, invalid pixels"""
	w, h = 70, 16
	vw, vh = w-6, h-6
	rng = np.random.RandomState(4)
	lg, lc, rg = make_content(w, h, "smooth")
	lo = rng.randint(-80, 40, (vh, vw)); wd = rng.randint(1, 257, (vh, vw))
	lo[0, :8] = -200; wd[0, :8] = 50                                  # wholly left of the right image
	lo[1, :8] = w; wd[1, :8] = 5                                      # wholly right of it
	px, n = synth.sgm_pixel_map(w, h, lo, lo+wd, rng.rand(vh, vw) < 0.07)
	c, _, _, _ = O.sgm_match(lg, lc, rg, px, n, stage=1)
	ref = wzncc64(lg, lc, rg, px)
	check_volume("oracle ragged", c, ref, max_undecidable=MAX_UNDECIDABLE)
	assert (ref[0][:int(px["idx"][8])] == 255).all()


def test_float64_reference_regimes():
	"""The content cases reach the regimes they are built for: eps-dominated windows, ncc <= 0 at the true disparity, cost 0 at
	the true disparity of identical windows, weights near exp(-17.8), exactly flat windows (cost 255)."""
	w, h, d0 = 74, 20, 12
	px, n = synth.sgm_pixel_map(w, h, d0, d0+1)
	vw = w-6
	mid = np.s_[:, vw//4+8:3*vw//4-8]
	lev = {k: wzncc64(*make_content(w, h, k, d0=d0), px)[0].reshape(h-6, vw) for k in CONTENT}
	assert (lev["identical"] == 0).mean() > 0.3
	assert (lev["anticorrelated"][mid] == 255).mean() > 0.7
	assert (lev["textureless"][mid] > 200).mean() > 0.9 and np.median(lev["smooth"][mid]) < 150
	assert (lev["gray01"][:h//3-6, :w//3-6] == 255).all()
	lg, lc, rg = make_content(w, h, "saturated")
	dc = lc[1:, 1:].astype(np.int64)-lc[:-1, :-1]
	assert ((dc*dc).sum(-1) == 3*255*255).any()


def test_margin_is_first_order_and_not_vacuous():
	"""Perturbing the inputs by float32 rounding moves the level by far less than the margin, and the margin is small: a bound
	loosened by 10x would make more than the power checks allow undecidable."""
	w, h = 60, 20
	lg, lc, rg = make_content(w, h, "smooth")
	px, n = synth.sgm_pixel_map(w, h, -4, 28)
	want, level, margin = wzncc64(lg, lc, rg, px)
	inside = margin > 0
	assert np.median(margin[inside]) < 0.02
	und10 = 1.0-decidable(level, 10*margin).mean()
	assert und10 > MAX_UNDECIDABLE


@pytest.mark.parametrize("steps", [2, 4, 8, 16])
def test_oracle_refinement_equals_float64_reference(O, steps):
	px, a, disp = refine_case(steps)
	# the oracle, like the reference, expects the disparity inside the pixel's range
	lo, hi = px["dmin"].reshape(disp.shape), px["dmax"].reshape(disp.shape)
	inr = (disp == NO_DISP) | ((disp >= lo) & (disp < hi)) | (hi-lo < 2)
	d_in = np.where(inr, disp, NO_DISP).astype(np.int16)
	got = O.sgm_refine(px, a, d_in, steps)
	ref = lc_blend64(px, a, d_in, steps)
	und = check_refine("oracle refine steps=%d" % steps, got, ref)
	assert und <= MAX_UNDECIDABLE
	# untouched: widths < 2 and NO_DISP
	w1 = (hi-lo < 2) | (d_in == NO_DISP)
	assert np.array_equal(got[w1], d_in[w1])


def test_refinement_reference_branches():
	"""Hand-derived values of lc_blend64: each branch of the LC blend and the uint16 wrap"""
	px = np.zeros(6, dtype=np.dtype([("idx", "<u8"), ("dmin", "<i2"), ("dmax", "<i2"), ("reserved", "<i4")]))
	px["dmin"] = -10; px["dmax"] = -7; px["idx"] = np.arange(6)*3
	a = np.array([100, 50, 200,   100, 100, 200,   100, 50, 50,   90, 50, 90,   10, 20, 30,   0, 7, 0], np.uint16)
	d = np.array([-9, -9, -9, -9, -9, -10], np.int16)
	want, val, _ = lc_blend64(px, a, d, 4)
	blend = lambda x: (1-np.cos(x*_C13))*(_F1195-np.cos(x*_C23))+x/2*(1-(_F1195-np.cos(x*_C23)))
	assert val[0] == pytest.approx(4*(-9+blend(50/150)-0.5))                # ld < rd
	assert val[1] == pytest.approx(4*(-9+0.5*100/200))                      # prev == center: + semi(center, next)
	assert val[2] == pytest.approx(4*(-9-0.5*50/100))                       # center == next: - semi(center, prev)
	assert val[3] == pytest.approx(4*(-9-(blend(1.0)-0.5)))                 # ld == rd: mult -1
	# not the minimum: ld = (10 - 20) mod 2^16 = 65526 > rd = 10 -> x = 10 / 65526, mult -1
	assert val[4] == pytest.approx(4*(-9-(blend(10/65526)-0.5)))
	assert val[5] == -40 and want[5] == -40                                 # d == dmin, other == 0
	assert want[0] == np.floor(val[0]+0.5)


@pytest.mark.parametrize("th", [0, 1, 2, 5])
@pytest.mark.parametrize("sign", [1, -1])
def test_oracle_cross_check_equals_integer_reference(O, th, sign):
	l2r, r2l = cross_check_case(97, 23, sign, th, seed=th)
	want = cross_check_ref(l2r, r2l, th)
	assert np.array_equal(O.sgm_cross_check(l2r, r2l, th), want)
	kept = (want != NO_DISP)
	assert 0.1 < kept.mean() < 0.9
