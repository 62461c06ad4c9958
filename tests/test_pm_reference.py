"""Float64 references of the PatchMatch score and of the sweep's propagation step, and the CPU oracle pinned to them (no GPU).

* `score64`      ScorePixelImage + ScorePixel (MINMEAN, DepthMap.cpp:465-626), the patch fill and weights (DepthMap.cpp:422-462),
                 the pass-A pixel rules (SceneDensify.cpp:490-517, the prior DepthMap.cpp:552-561) and the geometric term
                 (DepthMap.cpp:535-551) in float64, vectorised over pixels x views x taps, for planes given per pixel
* `propagate64`  one red-black half-sweep without refinement tries (nRandomIters = 0): the far-candidate choice, InterpolatePixel
                 (DepthMap.cpp:915-959), CorrectNormal (DepthMap.h:447-453), the smoothness factor (DepthMap.cpp:522-534) and
                 the accept chain `conf > nconf`

Every value carries a first-order forward-error margin for a float32 evaluation of the same formula (`F`, `U`), and every
discontinuity of the formula its signed distance from the switch point with its own margin.  A hypothesis is *decidable* when
every discontinuity lies farther from its switch than its margin: a float32 evaluation must then equal the float64 value within
the margin.  Elsewhere it must equal, within the margin, the value of one side of each undecided switch.  The references do
not use `oracle/` or the kernels; `tests/test_pm_reference_gpu.py` holds the kernels to the same rules.
"""
import dataclasses

import numpy as np
import pytest
from scipy.ndimage import maximum_filter

from openmvs_b200 import synth

HALF = 4
_f32 = np.float32

# the float32 constants of the engine (PMParams, pm_host.cu build_params) and of the oracle, promoted exactly to float64
KEEP = float(_f32(0.9))
TH_ROBUST = float(_f32(_f32(0.9)*_f32(4))/_f32(3))
TH_MAG_SQ = float(_f32(0.02)*_f32(0.02))
SIGMA_COLOR = float(_f32(-1)/(_f32(2)*(_f32(0.1)*_f32(0.1))))
SIGMA_SPATIAL = float(_f32(-1)/(_f32(2)*_f32(9)))
NRM_EPS = float(_f32(1e-16))
PRIOR_SIGMA = float(_f32(-1)/_f32(0.02))
GEOM_W = float(_f32(0.1))
SIM_TH = float(_f32(0.03))
IPOL_EPS = float(_f32(1e-4))
_PI = _f32(np.pi)
SMOOTH_BONUS_DEPTH = float(_f32(1)-_f32(0.93))
SMOOTH_BONUS_NORMAL = float((_f32(1)-_f32(0.93))*_f32(0.96))
SMOOTH_SIGMA_DEPTH = float(_f32(-1)/(_f32(2)*_f32(0.02)*_f32(0.02)))
_R13 = _f32(13)*(_PI/_f32(180))
SMOOTH_SIGMA_NORMAL = float(_f32(-1)/(_f32(2)*_R13*_R13))

U = 2.0**-22
"""Unit roundoff of every margin: one U per elementary operation (relative to its result) and one U per accumulated sum
(relative to the sum of the absolute values of its terms).  U = 2^-22 = 4u (u = 2^-24, the float32 unit roundoff) covers every
correctly rounded operation (u), CUDA's `expf` / `sqrtf` / `acosf` / division and libm's float functions (<= 2 ulp), an FMA
counted as two operations, a float constant whose grouping differs between the engine and the oracle (1 ulp), and a 25-term sum
in any order: its independent roundings add like a random walk (~2.3u of the absolute sum in sequential order), and the margin of
a value adds the bounds of all its sums and operations in absolute value.  `F` propagates these charges to first order and adds
the product of two errors, so a bound stays valid where a factor is smaller than its own error (`sqrt` and `acos` use their
Hoelder bounds there).  Fixed by this argument, not fitted to any kernel's output."""

U_POS = 2.0**-24
K_TAP_A = 14
K_TAP_M = 20
"""Tap-position term, in units of U_POS = u: every operation of the tap position is a correctly rounded float32 FMA, product
or sum (no transcendental function), so each rounds by at most u of its result.  The host folds A = Hl Hr and Hm in double and rounds them to float (1 U relative to each term of
A p and Hm (ms . p)); the kernel forms ms = n^T Kref^-1 / (n . X0 d) in float (6 operations on the Hm part); the homogeneous
centre H (x, y, 1) takes three FMAs, the top-left tap two more, and a tap is reached by up to 4 accumulated steps along its row
and 4 down its column (8 roundings of a running value bounded by the same absolute sum).  So |error of X_i| <= u (K_TAP_A
sum_j |A_ij p_j| + K_TAP_M |Hm_i| sum_j |ms_j p_j|) with K_TAP_A = 1 + 3 + 2 + 8 = 14 and K_TAP_M = K_TAP_A + 6 = 20; the oracle
(double H rounded to float, 3 operations for the top-left tap, the same 8 steps) stays inside it.  The perspective divide
p = X * rcp.approx.ftz.f32(Z): the PTX ISA gives rcp.approx.f32 a maximum error of 1 ulp over the full range (ftz only flushes
subnormals, far below any |Z| here), so with the product the projected position errs by 3u |p| < U |p| more than X / Z does.  The
position error enters the texel value through the bilinear cell's gradient: the largest difference of horizontally (vertically)
adjacent texels in the 3 x 3 cells around the tap bounds |dv/dx| (|dv/dy|) for any position within one texel, and the three
FMAs of the interpolation add 3 U."""


# ---- first-order error arithmetic ----------------------------------------------------------------------------------------------

class F:
	"""a float64 value and a bound on the error of its float32 evaluation (see U)"""
	__slots__ = ("v", "e")

	def __init__(self, v, e=0.0):
		self.v = np.asarray(v, np.float64)
		self.e = np.broadcast_to(np.asarray(e, np.float64), self.v.shape) if np.ndim(e) < self.v.ndim else np.asarray(e, np.float64)

	def __add__(a, b):
		b = _F(b); v = a.v+b.v
		return F(v, a.e+b.e+U*np.abs(v))
	__radd__ = __add__

	def __sub__(a, b):
		b = _F(b); v = a.v-b.v
		return F(v, a.e+b.e+U*np.abs(v))

	def __rsub__(a, b):
		return _F(b)-a

	def __neg__(a):
		return F(-a.v, a.e)

	def __mul__(a, b):
		b = _F(b); v = a.v*b.v
		with np.errstate(invalid="ignore"):      # 0 * inf: a bound that is already infinite elsewhere
			e = np.abs(a.v)*b.e+np.abs(b.v)*a.e+a.e*b.e+U*np.abs(v)
		return F(v, e)
	__rmul__ = __mul__

	def __truediv__(a, b):
		b = _F(b)
		with np.errstate(divide="ignore", invalid="ignore"):
			q = a.v/b.v
			den = np.abs(b.v)-b.e
			e = np.where(den > 0, (a.e+np.abs(q)*b.e)/np.where(den > 0, den, 1.0)+U*np.abs(q), np.inf)
		return F(q, e)

	def __rtruediv__(a, b):
		return _F(b)/a

	def __getitem__(self, k):
		return F(self.v[k], self.e[k])


def _F(x):
	return x if isinstance(x, F) else F(x)


def fsum(a, axis=-1):
	"""an accumulated sum: one U of the absolute sum of its terms"""
	return F(a.v.sum(axis), a.e.sum(axis)+U*np.abs(a.v).sum(axis))


def fexp(a):
	y = np.exp(a.v)
	return F(y, y*np.expm1(a.e)+U*y)


def fsqrt(a):
	s = np.sqrt(np.maximum(a.v, 0.0))
	lo = np.maximum(a.v-a.e, 0.0)
	with np.errstate(divide="ignore", invalid="ignore"):
		lin = np.where(lo > 0, a.e/(2.0*np.sqrt(lo)), np.inf)
	return F(s, np.minimum(np.sqrt(a.e), lin)+U*s)


def facos(a):
	c = np.clip(a.v, -1.0, 1.0)
	y = np.arccos(c)
	hi = np.minimum(np.abs(c)+a.e, 1.0)
	with np.errstate(divide="ignore", invalid="ignore"):
		lin = np.where(hi < 1.0, a.e/np.sqrt(1.0-hi*hi), np.inf)
	return F(y, np.minimum(lin, np.pi*np.sqrt(a.e/2.0))+U*(1.0+y))


def fclip(a, lo, hi):
	"""clamping is 1-Lipschitz: the error bound carries over"""
	return F(np.clip(a.v, lo, hi), a.e)


def fmin(a, c):
	return F(np.minimum(a.v, c), a.e)


# ---- cameras and views ---------------------------------------------------------------------------------------------------------

@dataclasses.dataclass
class View:
	image: np.ndarray            # (h, w) float32
	K: np.ndarray
	R: np.ndarray
	C: np.ndarray
	depth_gt: np.ndarray = None
	normal_gt: np.ndarray = None


@dataclasses.dataclass
class Case:
	name: str
	views: list                  # reference first
	dmin: float
	dmax: float
	depth: np.ndarray            # (H, W) float32 plane depth per pixel
	normal: np.ndarray           # (H, W, 3) float32
	lowres: np.ndarray = None    # (H, W) float32 prior or None
	depths: list = None          # per view None or (dmap, Kd, Rd, Cd)


def _texture(w, h, seed, lam=(4.0, 30.0), n=16, contrast=0.17):
	rng = np.random.RandomState(seed)
	yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
	acc = np.zeros((h, w))
	for _ in range(n):
		f = 2*np.pi/np.exp(rng.uniform(np.log(lam[0]), np.log(lam[1])))
		a = rng.uniform(0, np.pi)
		acc += np.sin(f*(np.cos(a)*xx+np.sin(a)*yy)+rng.uniform(0, 2*np.pi))
	return np.clip(0.5+contrast*acc/np.sqrt(n/2.0), 0.0, 1.0).astype(np.float32)


def _K(w, h, f=None, fy=None, cx=None, cy=None):
	f = 0.9*w if f is None else f
	return np.array([[f, 0, (w-1)/2.0 if cx is None else cx], [0, f if fy is None else fy, (h-1)/2.0 if cy is None else cy], [0, 0, 1.0]])


def _ray(K, x, y):
	"""X0 = Kref^-1 (x, y, 1) (zero skew) as the engine forms it in float: x ifx + ox with rounded constants, 3 operations"""
	X0x = (np.asarray(x, np.float64)-K[0, 2])/K[0, 0]
	X0y = (np.asarray(y, np.float64)-K[1, 2])/K[1, 1]
	sx = (np.abs(np.asarray(x, np.float64))+abs(K[0, 2]))/abs(K[0, 0])
	sy = (np.abs(np.asarray(y, np.float64))+abs(K[1, 2]))/abs(K[1, 1])
	return F(X0x, 3*U*sx), F(X0y, 3*U*sy)


def _view_consts(ref, v):
	"""A = K R Rref^T Kref^-1, Hm = K R (Cref - C) in double (ViewData::Init, DepthMap.h:175-185)"""
	KR = v.K@v.R
	A = KR@ref.R.T@np.linalg.inv(ref.K)
	Hm = KR@(ref.C-v.C)
	return A, Hm


def _geo_consts(ref, dm):
	d, Kd, Rd, Cd = dm
	KdRd = Kd@Rd
	Tl = KdRd@ref.R.T
	Tm = KdRd@(ref.C-Cd)
	Tr = ref.K@ref.R@Rd.T@np.linalg.inv(Kd)
	Tn = ref.K@ref.R@(Cd-ref.C)
	return Tl, Tm, Tr, Tn


# ---- the patch of the reference pixel ------------------------------------------------------------------------------------------

_TI, _TJ = np.divmod(np.arange(25), 5)
DY = 2*_TI-HALF
DX = 2*_TJ-HALF
CORNERS = (0, 4, 20, 24)


def patch64(img, xs, ys):
	"""FillPixelPatch: weights w, tempWeights tw, sumW, normSq0 of the 5x5 taps of each pixel (P, 25) / (P,).
	The error of the weighted mean tm enters tw (and through it the NCC numerator) in full, but normSq0 = sum w (I - tm)^2
	only to second order: d normSq0 / d tm = -2 sum w (I - tm) = 0."""
	I = img.astype(np.float64)[ys[:, None]+DY, xs[:, None]+DX]
	c = img.astype(np.float64)[ys, xs][:, None]
	dI = F(I)-F(c)
	w = fexp(dI*dI*SIGMA_COLOR+F((DX*DX+DY*DY).astype(np.float64))*SIGMA_SPATIAL)
	sumW = fsum(w)
	tm = fsum(F(I)*w)/sumW
	tv = I-tm.v[:, None]
	t = F(tv, U*np.abs(tv))
	etm = tm.e[:, None]
	tw = F(w.v*tv, (w*t).e+w.v*etm)
	n0 = fsum(F(w.v*tv, (w*t).e)*t)
	return w, tw, sumW, F(n0.v, n0.e+(w.v*etm*etm).sum(1))


def prior_of(case, xs, ys):
	return np.zeros(len(xs)) if case.lowres is None else np.maximum(case.lowres[ys, xs].astype(np.float64), 0.0)


def pixels_active(case, xs, ys, normSq0):
	"""-> (active for sure, undecided): inside the image with the patch, and the magnitude reject unless a prior vouches"""
	H, W = case.views[0].image.shape
	inside = (xs >= HALF) & (ys >= HALF) & (xs < W-HALF) & (ys < H-HALF)
	d0 = prior_of(case, xs, ys)
	gap = normSq0.v-TH_MAG_SQ
	strong = (d0 > 0) | (gap > normSq0.e)
	weak = (d0 <= 0) & (gap < -normSq0.e)
	return inside & strong, inside & ~strong & ~weak


# ---- one neighbour view --------------------------------------------------------------------------------------------------------

class ViewScore:
	"""ScorePixelImage of one neighbour for P pixels.  Fields (P,):
	rej      the reference rejects (thRobust) for sure: a tap outside the 1-pixel border or nrmSq <= 1e-16
	maybe    a rejection switch is undecided (then thRobust and the value both count)
	sc, sc_und  the depth Z of the four corner taps changes sign (decided / undecided): the kernel rejects the view
	alt_v, alt_e, alt_ok (P, G): the values of the score after the geometric term, the prior and min(2, .) for every side of
	         the undecided geometric switches (G = 1 without a depth-map), their margins and which of them are reachable
	dist     signed distance of each discontinuity from its switch, with its margin: name -> (distance, margin)"""


def _bilinear(img, px, py):
	h, w = img.shape
	lx = np.clip(np.floor(np.nan_to_num(px, nan=1.0, posinf=1.0, neginf=1.0)), 0, w-2).astype(np.int64)
	ly = np.clip(np.floor(np.nan_to_num(py, nan=1.0, posinf=1.0, neginf=1.0)), 0, h-2).astype(np.int64)
	ax = np.clip(np.nan_to_num(px)-lx, -1, 2); ay = np.clip(np.nan_to_num(py)-ly, -1, 2)
	I = img
	v00, v10, v01, v11 = I[ly, lx], I[ly, lx+1], I[ly+1, lx], I[ly+1, lx+1]
	return lx, ly, (v00*(1-ax)+v10*ax)*(1-ay)+(v01*(1-ax)+v11*ax)*ay, np.maximum.reduce([np.abs(v00), np.abs(v10), np.abs(v01), np.abs(v11)])


class _Img:
	"""a neighbour image in float64 with the Lipschitz bounds of its bilinear interpolant around every cell"""

	def __init__(self, img):
		self.I = img.astype(np.float64)
		gx = np.zeros_like(self.I); gy = np.zeros_like(self.I)
		gx[:, :-1] = np.abs(np.diff(self.I, axis=1)); gy[:-1] = np.abs(np.diff(self.I, axis=0))
		self.Gx = maximum_filter(gx, size=4, origin=(-1, 0), mode="nearest")
		self.Gy = maximum_filter(gy, size=4, origin=(0, -1), mode="nearest")


def _geometric(case, vi, X0x, X0y, d, xs, ys):
	"""the geometric term of view vi for every side of its undecided switches -> (cons (P, G), margin (P, G), ok (P, G), dist)"""
	ref = case.views[0]
	dmap, Kd, Rd, Cd = case.depths[vi]
	Tl, Tm, Tr, Tn = _geo_consts(ref, case.depths[vi])
	dh, dw = dmap.shape
	D = dmap.astype(np.float64)
	T = lambda a: F(a, U*np.abs(a))                 # a double constant rounded to float
	Xc = (X0x*F(d), X0y*F(d), F(d))
	X1 = [Xc[0]*T(Tl[i, 0])+Xc[1]*T(Tl[i, 1])+Xc[2]*T(Tl[i, 2])+T(Tm[i]) for i in range(3)]
	z = X1[2]
	zpos = z.v > z.e; zneg = z.v < -z.e
	x1 = X1[0]/z; y1 = X1[1]/z
	ex = np.where(np.isfinite(x1.e), x1.e, 1e30); ey = np.where(np.isfinite(y1.e), y1.e, 1e30)
	bd = np.minimum.reduce([x1.v-1, dw-2-x1.v, y1.v-1, dh-2-y1.v])
	be = np.maximum(ex, ey)
	bin_ = bd > be; bout = bd < -be
	dist = {"X1z": (z.v, z.e), "dmap_border": (bd, be)}
	P = len(xs)
	vals, errs, oks = [], [], []
	xv = np.nan_to_num(x1.v, nan=1.0); yv = np.nan_to_num(y1.v, nan=1.0)
	cells_x = [np.clip(np.floor(xv-np.minimum(ex, 1.0)), 0, dw-2).astype(np.int64), np.clip(np.floor(xv+np.minimum(ex, 1.0)), 0, dw-2).astype(np.int64)]
	cells_y = [np.clip(np.floor(yv-np.minimum(ey, 1.0)), 0, dh-2).astype(np.int64), np.clip(np.floor(yv+np.minimum(ey, 1.0)), 0, dh-2).astype(np.int64)]
	sim_dist = []
	none_any = np.zeros(P, bool)
	for ix, cx_ in enumerate(cells_x):
		for iy, cy_ in enumerate(cells_y):
			# a second cell only where the position's error interval crosses a cell boundary
			fresh = np.ones(P, bool)
			if ix: fresh &= cells_x[1] != cells_x[0]
			if iy: fresh &= cells_y[1] != cells_y[0]
			t = [D[cy_, cx_], D[cy_, cx_+1], D[cy_+1, cx_], D[cy_+1, cx_+1]]
			rel = [F(np.abs(z.v-tk), z.e)/z for tk in t]
			sure = [r.v-SIM_TH < -r.e for r in rel]                               # similar for sure
			never = [(r.v-SIM_TH > r.e) | ~np.isfinite(r.v) for r in rel]      # dissimilar for sure
			sim_dist.append(np.where(fresh, np.min(np.stack([np.abs(r.v-SIM_TH)-r.e for r in rel]), 0), np.inf))
			fx = x1-F(cx_.astype(np.float64)); fy = y1-F(cy_.astype(np.float64))
			fx1 = 1.0-fx; fy1 = 1.0-fy
			for m in range(1, 16):
				b = [(m >> k) & 1 == 1 for k in range(4)]
				ok = fresh.copy()
				for k in range(4):
					ok &= ~sure[k] if not b[k] else ~never[k]
				# the masked bilinear sample's fallbacks (TImage::sample with functor, Types.inl:2297-2313)
				sel = lambda order: t[next(k for k in order if b[k])]
				a00 = sel((0, 1, 2, 3)); a10 = sel((1, 0, 3, 2)); a01 = sel((2, 3, 0, 1)); a11 = sel((3, 2, 1, 0))
				v = fy1*(fx1*F(a00)+fx*F(a10))+fy*(fx1*F(a01)+fx*F(a11))
				Px, Py = x1*v, y1*v
				B = [Px*T(Tr[i, 0])+Py*T(Tr[i, 1])+v*T(Tr[i, 2])+T(Tn[i]) for i in range(3)]
				ex_ = F(xs.astype(np.float64))-B[0]/B[2]; ey_ = F(ys.astype(np.float64))-B[1]/B[2]
				dd = fsqrt(ex_*ex_+ey_*ey_)
				cons = fmin(fsqrt(dd*(dd+2.0)), 4.0)
				vals.append(cons.v); errs.append(cons.e); oks.append(ok & ~zneg & ~bout)
			# no tap similar: the consistency stays 4
			none = fresh.copy()
			for k in range(4):
				none &= ~sure[k]
			none_any |= none
	# behind the depth-map's camera, outside its border or no similar tap: 4
	vals.append(np.full(P, 4.0)); errs.append(np.zeros(P)); oks.append(none_any | ~(zpos & bin_))
	dist["similarity"] = (np.min(np.stack(sim_dist), 0), np.zeros(P))
	return np.stack(vals, 1), np.nan_to_num(np.stack(errs, 1), nan=np.inf), np.stack(oks, 1), dist


def score_view64(case, vi, pt, xs, ys, d, n, smooth, img=None):
	ref, v = case.views[0], case.views[vi]
	A, Hm = _view_consts(ref, v)
	Kinv = np.linalg.inv(ref.K)
	X0x, X0y = _ray(ref.K, xs, ys)
	nX0 = n[:, 0]*X0x.v+n[:, 1]*X0y.v+n[:, 2]
	ms = (n@Kinv)/(nX0*d)[:, None]                                       # (P, 3)
	p = np.stack([xs[:, None]+DX, ys[:, None]+DY, np.ones((len(xs), 25))], -1).astype(np.float64)   # (P, 25, 3)
	mp = (ms[:, None, :]*p).sum(-1)                                       # (P, 25)
	amp = np.abs(ms[:, None, :]*p).sum(-1)
	X = p@A.T+Hm[None, None, :]*mp[..., None]                            # (P, 25, 3)
	eX = U_POS*(K_TAP_A*(np.abs(p)@np.abs(A).T)+K_TAP_M*np.abs(Hm)[None, None, :]*amp[..., None])
	Z, eZ = X[..., 2], eX[..., 2]
	with np.errstate(divide="ignore", invalid="ignore"):
		px = X[..., 0]/Z; py = X[..., 1]/Z
		den = np.abs(Z)-eZ
		epx = np.where(den > 0, (eX[..., 0]+np.abs(px)*eZ)/np.where(den > 0, den, 1), np.inf)+U*np.abs(px)
		epy = np.where(den > 0, (eX[..., 1]+np.abs(py)*eZ)/np.where(den > 0, den, 1), np.inf)+U*np.abs(py)
	epx = np.nan_to_num(epx, nan=np.inf); epy = np.nan_to_num(epy, nan=np.inf)
	h, w = v.image.shape
	# the inside test of every tap (isInsideWithBorder<float,1>: 1 <= x <= w-2, 1 <= y <= h-2)
	ind = np.nan_to_num(np.minimum.reduce([px-1, (w-2)-px, py-1, (h-2)-py]), nan=-1e30)
	ine = np.maximum(epx, epy)
	out_sure = (ind < -ine).any(1)
	in_sure = (ind > ine).all(1)
	# corner depths: the kernel decides "all taps inside" from the four corners, valid while Z keeps its sign
	zc, ezc = Z[:, CORNERS], eZ[:, CORNERS]
	sc_und = (np.abs(zc) <= ezc).any(1)
	sc = ~sc_und & (zc > 0).any(1) & (zc < 0).any(1)
	# texels
	if img is None:
		img = _Img(v.image)
	lx, ly, val, vmax = _bilinear(img.I, px, py)
	ev = img.Gx[ly, lx]*epx+img.Gy[ly, lx]*epy+3*U*vmax
	ev = np.where((epx < 0.5) & (epy < 0.5), ev, np.inf)
	# The sums in float arithmetic on the exact texels and weights; the texels' position errors (ev) and the weights' errors
	# enter through the derivatives of the centred forms: d normSq1 / d v_k = 2 w_k (v_k - m1), d normSq1 / d w_k = (v_k - m1)^2
	# (m1 = sum / sumW), d num / d v_k = tw_k.
	wk, twk, sumW, normSq0 = pt
	tv = F(val)
	W = F(wk.v)
	vw = tv*W
	sm = fsum(vw); sq = fsum(tv*vw); num = fsum(tv*twk)
	S = F(sumW.v, U*sumW.v)
	normSq1 = sq-sm*sm/S
	m1 = (sm.v/sumW.v)[:, None]
	normSq1 = F(normSq1.v, normSq1.e+(2*wk.v*np.abs(val-m1)*ev).sum(1)+((val-m1)**2*wk.e).sum(1))
	num = F(num.v, num.e+(np.abs(twk.v)*ev).sum(1))
	normSq1.e = np.nan_to_num(normSq1.e, nan=np.inf); num.e = np.nan_to_num(num.e, nan=np.inf)
	nrm = normSq0*normSq1
	nrm_small = nrm.v-NRM_EPS < -nrm.e
	nrm_big = nrm.v-NRM_EPS > nrm.e
	with np.errstate(invalid="ignore", divide="ignore"):
		ncc = fclip(num/fsqrt(F(np.maximum(nrm.v, NRM_EPS), nrm.e)), -1.0, 1.0)
	score = (1.0-ncc)*smooth
	res = ViewScore()
	res.rej = out_sure | (in_sure & nrm_small)
	res.maybe = ~res.rej & ~(in_sure & nrm_big)
	res.sc, res.sc_und = sc, sc_und
	res.dist = {"tap_inside": (ind.min(1), ine[np.arange(len(xs)), ind.argmin(1)]), "nrmSq": (nrm.v-NRM_EPS, nrm.e),
		"corner_z": (np.abs(zc).min(1), ezc.max(1))}
	if case.depths is not None and case.depths[vi] is not None:
		cons, econs, cok, gd = _geometric(case, vi, X0x, X0y, d, xs, ys)
		res.dist.update(gd)
		alt = F(score.v[:, None], score.e[:, None])+F(cons, econs)*GEOM_W
	else:
		alt = F(score.v[:, None], score.e[:, None]); cok = np.ones((len(xs), 1), bool)
	d0 = prior_of(case, xs, ys)
	if (d0 > 0).any():
		f = fexp(normSq0*PRIOR_SIGMA)
		delta = fmin(F(np.abs(d0-d)/np.where(d0 > 0, d0, 1.0), 3*U*np.abs(d0-d)/np.where(d0 > 0, d0, 1.0)), 0.5)
		fc = F(f.v[:, None], f.e[:, None]); dc = F(delta.v[:, None], delta.e[:, None])
		mixed = (1.0-fc)*alt+fc*dc
		has = (d0 > 0)[:, None]
		alt = F(np.where(has, mixed.v, alt.v), np.where(has, mixed.e, alt.e))
		res.dist["prior_clamp"] = (np.abs(d0-d)/np.where(d0 > 0, d0, 1.0)-0.5, delta.e)
	alt = fmin(alt, 2.0)
	res.alt_v, res.alt_e, res.alt_ok = alt.v, np.nan_to_num(alt.e, nan=np.inf), cok
	return res


# ---- ScorePixel ----------------------------------------------------------------------------------------------------------------

@dataclasses.dataclass
class PixelScores:
	dec: np.ndarray        # (P,) decidable
	val: np.ndarray        # (P,) float64 value (decidable pixels)
	mar: np.ndarray        # (P,) its margin
	cands: list            # per pixel: (values, margins) arrays of the values that count where it is undecidable
	views: list            # the ViewScore of every view
	vdec: np.ndarray       # (P, V) decidable per view


def _view_alternatives(r, kernel):
	"""(P, G+1) values / margins / reachable of one view, the last column the rejection thRobust (exact)"""
	rej_ok = r.rej | r.maybe
	val_ok = r.alt_ok & ~r.rej[:, None]
	if kernel:
		rej_ok = rej_ok | r.sc | r.sc_und
		val_ok = val_ok & ~r.sc[:, None]
	v = np.concatenate([r.alt_v, np.full((len(r.rej), 1), TH_ROBUST)], 1)
	e = np.concatenate([r.alt_e, np.zeros((len(r.rej), 1))], 1)
	ok = np.concatenate([val_ok, rej_ok[:, None]], 1)
	return v, e, ok


def score64(case, xs, ys, d, n, smooth=None, kernel=True, views=None):
	"""ScorePixel (MINMEAN) of the planes (d, n) at pixels (xs, ys) -> PixelScores.  kernel: the engine's documented difference
	(a view whose four corner taps have depths of both signs scores thRobust) instead of the reference's per-tap test.
	smooth: F (P,) product of the smoothness factors (1 in pass A)."""
	xs = np.asarray(xs, np.int64); ys = np.asarray(ys, np.int64)
	d = np.asarray(d, np.float64); n = np.asarray(n, np.float64)
	P = len(xs)
	smooth = F(np.ones(P)) if smooth is None else smooth
	pt = patch64(case.views[0].image, xs, ys)
	imgs = views if views is not None else [_Img(v.image) for v in case.views[1:]]
	res = [score_view64(case, i+1, pt, xs, ys, d, n, smooth, imgs[i]) for i in range(len(case.views)-1)]
	alts = [_view_alternatives(r, kernel) for r in res]
	N = len(res)
	V = np.stack([a[0] for a in alts], 1); E = np.stack([a[1] for a in alts], 1); OK = np.stack([a[2] for a in alts], 1)  # (P, N, G+1)
	cnt = OK.sum(2)
	assert (cnt >= 1).all()
	vdec = cnt == 1
	g = OK.argmax(2)
	sv = np.take_along_axis(V, g[..., None], 2)[..., 0]; se = np.take_along_axis(E, g[..., None], 2)[..., 0]
	order = np.argsort(sv, 1, kind="stable")
	s = np.take_along_axis(sv, order, 1); m = np.take_along_axis(se, order, 1)
	dec = vdec.all(1) & np.isfinite(m).all(1)
	# The two smallest scores are continuous functions of the views' scores (their order only decides which views are reported),
	# so the one switch of MINMEAN is s2 >= thRobust.  The k-th smallest errs by at most the largest margin among the views whose
	# values may swap places with it.
	def order_margin(k):
		near = np.abs(s-s[:, k:k+1]) <= m+m[:, k:k+1]
		return np.where(near, m, 0.0).max(1)
	if N == 1:
		val, mar = s[:, 0], m[:, 0]
	else:
		exact2 = (m[:, 1] == 0) & (s[:, 1] >= TH_ROBUST)
		hi2 = exact2 | (s[:, 1]-m[:, 1] > TH_ROBUST)
		lo2 = s[:, 1]+m[:, 1] < TH_ROBUST
		dec &= hi2 | lo2
		m0, m1 = order_margin(0), order_margin(1)
		mean = 0.5*(s[:, 0]+s[:, 1])
		val = np.where(hi2, s[:, 0], mean)
		mar = np.where(hi2, m0, 0.5*(m0+m1)+U*np.abs(mean))
	cands = [None]*P
	for i in np.flatnonzero(~dec):
		ok = OK[i]
		vv, ee = V[i][ok], E[i][ok]
		owner = np.nonzero(ok)[0]
		top = np.array([(V[i][j][OK[i][j]]+E[i][j][OK[i][j]]).max() for j in range(N)])
		u2 = np.sort(top)[min(1, N-1)]
		keep = vv-ee <= u2
		vv, ee, owner = vv[keep], ee[keep], owner[keep]
		cv, ce = [vv], [ee]
		if N > 1 and len(vv) > 1:
			a, b = np.triu_indices(len(vv), 1)
			two = owner[a] != owner[b]
			mean = 0.5*(vv[a]+vv[b])
			cv.append(mean[two]); ce.append((0.5*(ee[a]+ee[b])+U*np.abs(mean))[two])
		cands[i] = (np.concatenate(cv), np.concatenate(ce))
	return PixelScores(dec, val, mar, cands, res, vdec)


def check_scores(name, got, ps, sel=None):
	"""got (P,) float32 costs -> (undecidable fraction, margins of the decidable pixels); every decidable pixel within its margin
	of the float64 value, every undecidable one within the margin of one of its sides"""
	got = np.asarray(got, np.float64)
	dec = ps.dec if sel is None else ps.dec & sel
	bad = np.flatnonzero(dec & ~(np.abs(got-ps.val) <= ps.mar))
	assert len(bad) == 0, "%s: %d decidable scores differ, e.g. %s" % (name, len(bad), [
		(int(i), float(got[i]), float(ps.val[i]), float(ps.mar[i])) for i in bad[:5]])
	und = np.flatnonzero(~ps.dec if sel is None else (~ps.dec & sel))
	wrong = [i for i in und if not (np.abs(got[i]-ps.cands[i][0]) <= ps.cands[i][1]).any()]
	assert not wrong, "%s: %d undecidable scores match no side of their switches, e.g. %s" % (name, len(wrong), [
		(int(i), float(got[i]), ps.cands[i][0][:6].tolist()) for i in wrong[:5]])
	n = int(dec.sum()+len(und))
	return len(und)/max(n, 1), ps.mar[dec]


# ---- pass A --------------------------------------------------------------------------------------------------------------------

def pass_a_expect(case, kernel=True):
	"""-> (active (H, W) for sure, undecided activity (H, W), pixel coordinates of the active pixels, their PixelScores)"""
	H, W = case.views[0].image.shape
	ys, xs = np.mgrid[HALF:H-HALF, HALF:W-HALF]
	xs, ys = xs.ravel(), ys.ravel()
	pt = patch64(case.views[0].image, xs, ys)
	act, und = pixels_active(case, xs, ys, pt[3])
	A = np.zeros((H, W), bool); Ua = np.zeros((H, W), bool)
	A[ys, xs] = act; Ua[ys, xs] = und
	sel = act | und
	xs, ys = xs[sel], ys[sel]
	ps = score64(case, xs, ys, case.depth[ys, xs], case.normal[ys, xs], kernel=kernel)
	return A, Ua, xs, ys, ps


def check_pass_a(name, case, plane_d, plane_n, cost, expect):
	"""the output of pass A (kernel or oracle) against the rules -> (undecidable fraction, decidable margins)"""
	A, Ua, xs, ys, ps = expect
	rejected = ~A & ~Ua
	assert np.all(plane_d[rejected] == 0) and np.all(plane_n[rejected] == 0) and np.all(cost[rejected] == 2), name
	# a given valid plane is scored as it is
	assert np.array_equal(plane_d[A], case.depth[A]) and np.array_equal(plane_n[A], case.normal[A]), name
	scored = plane_d[ys, xs] > 0
	assert scored[A[ys, xs]].all()
	und, mar = check_scores(name, cost[ys, xs], ps, sel=scored)
	return und, mar


# ---- the cases -----------------------------------------------------------------------------------------------------------------

def _valid_normals(K, d, n, H, W):
	"""normals that face the camera with margin (n . X0 < -0.2): the engine keeps a given plane only when it faces the camera"""
	yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
	X0 = np.stack([(xx-K[0, 2])/K[0, 0], (yy-K[1, 2])/K[1, 1], np.ones_like(xx)], -1)
	c = (n*X0).sum(-1)/np.linalg.norm(X0, axis=-1)
	bad = c > -0.2
	n = n.copy()
	n[bad] = -X0[bad]/np.linalg.norm(X0[bad], axis=-1, keepdims=True)
	return n.astype(np.float32)


def _fronto(H, W):
	n = np.zeros((H, W, 3), np.float32); n[..., 2] = -1
	return n


def _shift_case(axis, w=96, h=72, seed=0):
	"""A neighbour translated purely along x (axis 0) or y (axis 1), same orientation, principal point offset by 50 pixels:
	the homography of a fronto-parallel plane is a shift by 50 - f b / d.  Per pixel the depth puts the first (or last) tap of the
	row/column at 1 + delta (or at w-2 + delta) with delta in {+-1e-4, +-1e-2, +-0.3}."""
	K0 = _K(w, h)
	nw, nh = w, h
	Kn = _K(nw, nh, f=K0[0, 0], fy=K0[1, 1])
	off = 50.0
	Kn[axis, 2] = K0[axis, 2]+off
	b = 0.5
	ref = View(_texture(w, h, seed+1), K0, np.eye(3), np.zeros(3))
	C = np.zeros(3); C[axis] = b
	nb = View(_texture(nw, nh, seed+2), Kn, np.eye(3), C)
	deltas = np.array([1e-4, -1e-4, 1e-2, -1e-2, 0.3, -0.3])
	f = K0[axis, axis]
	yy, xx = np.mgrid[0:h, 0:w]
	u = (xx if axis == 0 else yy).astype(np.float64)
	other = yy if axis == 0 else xx
	size = nw if axis == 0 else nh
	delta = deltas[(other+u.astype(int)) % len(deltas)]
	# shift s = f b / d: a tap at u + k maps to u + k + off - s
	s_first = u-HALF+off-(1+delta)                 # first tap (u-4) at 1 + delta
	s_last = u+HALF+off-(size-2+delta)             # last tap (u+4) at size-2 + delta
	s = np.where(u < (w if axis == 0 else h)/2, s_first, s_last)
	s = np.where(s > 2.0, s, s_first)
	depth = (f*b/s).astype(np.float32)
	return Case("shift" + "xy"[axis], [ref, nb], 0.3, 200.0,
		depth, _fronto(h, w))


def _scene_case(name, w, h, nv, seed=1234, perturb=0.01, step=5.0):
	sc = synth.make_scene(w, h, nv+1, seed=seed, step_deg=step)
	ref = len(sc.views)//2
	views = [sc.views[ref]]+[sc.views[i] for i in sc.neighbors(ref, nv)]
	views = [View(v.image, v.K, v.R, v.C, v.depth_gt, v.normal_gt) for v in views]
	rng = np.random.RandomState(seed+nv)
	d = (views[0].depth_gt*(1+perturb*rng.randn(h, w))).astype(np.float32)
	n = views[0].normal_gt+5*perturb*rng.randn(h, w, 3)
	n = n/np.linalg.norm(n, axis=-1, keepdims=True)
	n = _valid_normals(views[0].K, d, n, h, w)
	return Case(name, views, sc.dmin, sc.dmax, d, n)


def _resized(v, sw, sh):
	import cv2
	h, w = v.image.shape
	small = cv2.resize(v.image, (sw, sh), interpolation=cv2.INTER_AREA)
	K = v.K.copy(); sx, sy = sw/w, sh/h
	K[0] *= sx; K[1] *= sy; K[0, 2] = (v.K[0, 2]+0.5)*sx-0.5; K[1, 2] = (v.K[1, 2]+0.5)*sy-0.5
	return View(small.astype(np.float32), K, v.R, v.C)


def _sizes_case():
	"""neighbours of 10x10 and of 0.8x the reference's size (K scaled), and one 4032 wide: tap coordinates beyond 2^11"""
	c = _scene_case("sizes", 96, 72, 3)
	v1, v2, v3 = c.views[1:]
	c.views[1] = _resized(v1, 10, 10)
	c.views[2] = _resized(v2, int(round(96*0.8)), int(round(72*0.8)))
	# a wide strip camera: the focal length along x 42 times the reference's, same centre shifted along x
	K = v3.K.copy(); K[0, 0] *= 42; K[0, 2] = 2016.0
	wide = _texture(4032, 72, 77, lam=(3.0, 40.0))
	c.views[3] = View(wide, K, v3.R, v3.C)
	return c


def _content_case(kind, w=96, h=72):
	"""identical: a neighbour with the reference's camera and image (ncc -> +1, score 0); inverse: 1 - I (ncc -> -1, score 2,
	and the MINMEAN switch s1 >= thRobust); textureless: flat bands (the magnitude reject and nrmSq <= 1e-16); gray01: gray
	values exactly 0 and 1 (weights down to exp(-52))"""
	c = _scene_case(kind, w, h, 2)
	ref = c.views[0]
	if kind == "identical":
		c.views[1] = View(ref.image.copy(), ref.K, ref.R, ref.C)
	elif kind == "inverse":
		c.views[1] = View((1-ref.image).astype(np.float32), ref.K, ref.R, ref.C)
		c.views.append(View(ref.image.copy(), ref.K, ref.R, ref.C))
	elif kind == "textureless":
		img = ref.image.copy(); img[30:46] = 0.5
		c.views[0] = View(img, ref.K, ref.R, ref.C)
		nb = c.views[1].image.copy(); nb[:, 40:60] = 0.25
		c.views[1] = View(nb, c.views[1].K, c.views[1].R, c.views[1].C)
	elif kind == "gray01":
		# the neighbours and a band of the reference thresholded (the band's patches are mostly rejected as too flat)
		for i in range(len(c.views)):
			v = c.views[i]
			img = np.where(v.image < 0.5, 0.0, 1.0).astype(np.float32)
			if i == 0:
				img = v.image.copy(); img[:, 30:50] = np.where(v.image[:, 30:50] < 0.5, 0.0, 1.0)
			c.views[i] = View(img, v.K, v.R, v.C)
	return c


def _rot(axis, ang):
	c, s = np.cos(ang), np.sin(ang)
	if axis == 1:
		return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
	return np.array([[1, 0, 0], [0, c, -s], [0, s, c]])


def _zsign_case(w=96, h=72):
	"""A neighbour whose optical axis is perpendicular to the reference's, its centre beside the surface: the patches of the
	pixels near the reference's centre column straddle the neighbour's Z = 0 plane (the documented sign-change case); a
	second neighbour looks away from the surface, so all four corners of every patch have Z < 0."""
	K0 = _K(w, h)
	ref = View(_texture(w, h, 5), K0, np.eye(3), np.zeros(3))
	R1 = _rot(1, -np.pi/2)             # camera z axis = world +x
	nb1 = View(_texture(w, h, 6), _K(w, h, f=0.3*w), R1, np.array([0.0, 0.0, 4.0]))
	R2 = _rot(1, np.pi)                # camera z axis = world -z: the surface is behind it
	nb2 = View(_texture(w, h, 7), _K(w, h, f=0.9*w), R2, np.array([0.0, 0.0, 1.0]))
	yy, xx = np.mgrid[0:h, 0:w]
	d = (4.0+0.3*np.sin(0.3*xx)+0.2*np.cos(0.25*yy)).astype(np.float32)
	return Case("zsign", [ref, nb1, nb2], 0.5, 20.0, d, _fronto(h, w))


def _geometric_case(w=96, h=72):
	"""Neighbours carrying depth-maps: holes, texels at 0.97 / 1.03 of the reprojected depth +- a few ulp and between 3 and
	4 %, a depth-map at half the image's resolution, reprojections at the depth-map's border, a depth-map camera behind the
	surface (X1.z <= 0), and a 1 - I neighbour whose score exceeds 2 before min(2, .)"""
	c = _scene_case("geometric", w, h, 3, perturb=0.0)
	ref = c.views[0]
	rng = np.random.RandomState(9)
	depths = [None]
	# view 1: its own depth, holes, per-pixel factors around the 3 % switch
	v1 = c.views[1]
	dm = v1.depth_gt.copy()
	fac = np.array([0.97, 1.03, 0.965, 1.035, 0.9701, 1.0299, 1.0, 1.0, 1.2])
	k = rng.randint(0, len(fac), dm.shape)
	dm = (dm*fac[k]).astype(np.float32)
	ulp = rng.randint(-3, 4, dm.shape)
	near = (k < 2)
	dm[near] = np.nextafter(dm[near], np.where(ulp[near] > 0, np.inf, -np.inf).astype(np.float32))
	dm[rng.rand(*dm.shape) < 0.08] = 0
	depths.append((dm, v1.K, v1.R, v1.C))
	# view 2: depth-map at half resolution with its camera scaled; a band of it pushed 5 pixels in from the border
	v2 = c.views[2]
	import cv2
	dm2 = cv2.resize(v2.depth_gt, (w//2, h//2), interpolation=cv2.INTER_NEAREST)
	K2 = v2.K.copy(); K2[0] *= 0.5; K2[1] *= 0.5; K2[0, 2] = (v2.K[0, 2]+0.5)*0.5-0.5; K2[1, 2] = (v2.K[1, 2]+0.5)*0.5-0.5
	depths.append((dm2.astype(np.float32), K2, v2.R, v2.C))
	# view 3: 1 - I with the reference's camera, and a depth-map camera behind the surface
	c.views[3] = View((1-ref.image).astype(np.float32), ref.K, ref.R, ref.C)
	Rb = _rot(1, np.pi)@ref.R
	depths.append((np.full((h, w), 5.0, np.float32), ref.K, Rb, ref.C))
	c.depths = depths
	c.depth = ref.depth_gt.copy()
	c.normal = _valid_normals(ref.K, c.depth, ref.normal_gt, h, w)
	return c


def _geometric_inverse_case(w=96, h=72):
	"""every neighbour 1 - I with the reference's camera and an inconsistent depth-map: each view scores 2 + 0.1 * 4 before
	the clamp min(2, .)"""
	c = _scene_case("geometric_inverse", w, h, 2, perturb=0.0)
	ref = c.views[0]
	c.views = [ref]+[View((1-ref.image).astype(np.float32), ref.K, ref.R, ref.C) for _ in range(2)]
	c.depths = [None]+[((ref.depth_gt*f).astype(np.float32), ref.K, ref.R, ref.C) for f in (1.5, 0.5)]
	c.depth = ref.depth_gt.copy()
	c.normal = _valid_normals(ref.K, c.depth, ref.normal_gt, h, w)
	return c


def _prior_case(w=96, h=72):
	"""a low-resolution prior: d0 = 0 and d0 > 0, |d0 - d| / d0 around the 0.5 clamp, textureless pixels that the prior keeps"""
	c = _scene_case("prior", w, h, 2)
	img = c.views[0].image.copy(); img[20:36, 10:60] = 0.5
	c.views[0] = View(img, c.views[0].K, c.views[0].R, c.views[0].C)
	rng = np.random.RandomState(3)
	ratio = np.array([0.0, 0.1, 0.45, 0.49, 0.51, 0.55, 0.65, 0.9, -0.3, -0.6])
	k = rng.randint(0, len(ratio), (h, w))
	# d0 with |d0 - d| / d0 = |ratio|
	d0 = (c.depth/(1-ratio[k])).astype(np.float32)
	d0[rng.rand(h, w) < 0.15] = 0
	c.lowres = d0
	c.dmax = float(max(c.dmax, d0.max()+1))
	return c


def score_cases():
	cs = [_shift_case(0), _shift_case(1)]
	for nv in (1, 2, 3, 9, 32):
		cs.append(_scene_case("views%d" % nv, 96, 72, nv, perturb=0.03))
	cs += [_sizes_case()]+[_content_case(k) for k in ("identical", "inverse", "textureless", "gray01")]
	cs += [_zsign_case(), _geometric_case(), _geometric_inverse_case(), _prior_case()]
	cs += [_scene_case("shape64x14", 64, 14, 2), _scene_case("shape203x151", 203, 151, 2)]
	return cs


CASES = {}


def case(name):
	if not CASES:
		for c in score_cases():
			CASES[c.name] = c
	return CASES[name]


SCORE_CASES = ["shiftx", "shifty", "views1", "views2", "views3", "views9", "views32", "sizes", "identical", "inverse",
	"textureless", "gray01", "zsign", "geometric", "geometric_inverse", "prior", "shape64x14", "shape203x151"]


# ---- the sweep's propagation step ------------------------------------------------------------------------------------------------

def _close_offset(dirn, k):
	kk = (k ^ 2) if dirn else k
	return kk, (-1 if kk == 0 else 1 if kk == 2 else 0), (-1 if kk == 1 else 1 if kk == 3 else 0)


def interpolate64(case, xs, ys, qx, qy, qd, qn, vertical):
	"""InterpolatePixel (DepthMap.cpp:915-959) with the skew-free x offset -> (depth F, undecided switch, the other side's
	depth).  Sides: |denom| < 1e-4 and a result outside [dMin, dMax) keep the candidate's depth."""
	K = case.views[0].K
	X0x, X0y = _ray(K, xs, ys)
	Qx, Qy = _ray(K, qx, qy)
	n1 = F(np.where(vertical, X0y.v, X0x.v), np.where(vertical, X0y.e, X0x.e))
	x1 = F(np.where(vertical, Qy.v, Qx.v), np.where(vertical, Qy.e, Qx.e))
	nc = F(np.where(vertical, qn[:, 1], qn[:, 0]))
	denom = F(qn[:, 2])+n1*nc
	dn = F(qd)*(F(qn[:, 2])+x1*nc)/denom
	dmin, dmax = float(_f32(case.dmin)), float(_f32(case.dmax))
	small = np.abs(denom.v) < IPOL_EPS
	und = np.abs(np.abs(denom.v)-IPOL_EPS) <= denom.e
	inr = (dmin <= dn.v) & (dn.v < dmax)
	und |= ~small & (np.minimum(np.abs(dn.v-dmin), np.abs(dmax-dn.v)) <= dn.e)
	use = ~small & inr
	val = np.where(use, dn.v, qd)
	err = np.where(use, dn.e, 0.0)
	other = np.where(use, qd, np.where(np.isfinite(dn.v), dn.v, qd))
	return F(val, err), und, other


def correct_normal64(n, X0x, X0y):
	"""CorrectNormal (DepthMap.h:447-453) -> (normal, error bound, undecided switch)"""
	X0 = np.stack([X0x.v, X0y.v, np.ones_like(X0x.v)], -1)
	c = (n*X0).sum(-1)
	vlen = np.linalg.norm(X0, axis=-1)
	rot = c >= 0
	und = np.abs(c) <= 8*U*(np.abs(n)*np.abs(X0)).sum(-1)+np.abs(n[:, 0])*X0x.e+np.abs(n[:, 1])*X0y.e
	out = n.copy()
	e = np.zeros(len(n))
	if rot.any():
		ang = np.minimum((np.arccos(np.clip(c[rot]/vlen[rot], -1, 1))-np.pi/2)*1.01, -0.001)
		w = np.cross(n[rot], X0[rot])
		with np.errstate(invalid="ignore", divide="ignore"):     # zero normals of invalid planes (never candidates)
			w /= np.linalg.norm(w, axis=-1, keepdims=True)
		v = n[rot]
		wv = np.cross(w, v); wwv = np.cross(w, wv)
		out[rot] = v+np.sin(ang)[:, None]*wv+(1-np.cos(ang))[:, None]*wwv
		e[rot] = 40*U
	return out, e, und


def smooth64(case, xs, ys, d, n, close):
	"""the product of the smoothness factors over the valid close neighbours (DepthMap.cpp:522-534); close: list of
	(mask, cx, cy, cd, cn) -> F"""
	K = case.views[0].K
	X0x, X0y = _ray(K, xs, ys)
	nx, ny, nz = F(n[:, 0]), F(n[:, 1]), F(n[:, 2])
	nX0 = nx*X0x+ny*X0y+nz
	planeD = -(F(d)*nX0)
	nn = nx*nx+ny*ny+nz*nz
	s = F(np.ones(len(xs)))
	for mask, cx, cy, cd, cn in close:
		Rx, Ry = _ray(K, cx, cy)
		dist = (nx*Rx+ny*Ry+nz)*F(cd)+planeD
		rd = dist/F(d)
		fD = fexp(rd*rd*SMOOTH_SIGMA_DEPTH)
		cnx, cny, cnz = F(cn[:, 0]), F(cn[:, 1]), F(cn[:, 2])
		ca = fclip((nx*cnx+ny*cny+nz*cnz)/fsqrt(nn*(cnx*cnx+cny*cny+cnz*cnz)), -1.0, 1.0)
		ang = facos(ca)
		fN = fexp(ang*ang*SMOOTH_SIGMA_NORMAL)
		f = (1.0-fD*SMOOTH_BONUS_DEPTH)*(1.0-fN*SMOOTH_BONUS_NORMAL)
		s = F(np.where(mask, (s*f).v, s.v), np.where(mask, (s*f).e, s.e))
	return s


@dataclasses.dataclass
class Sweep:
	xs: np.ndarray; ys: np.ndarray      # the active pixels of the colour
	winner: np.ndarray                  # -1 own plane, else candidate slot k
	dec: np.ndarray
	cost: np.ndarray; cost_mar: np.ndarray
	hyps: list                          # per slot k: (has candidate, depth F, normal, normal error, other-side depth, undecided)
	undecidable: float = 0.0


def propagate64(case, d, n, cost, colour, sweep, nprop, far, kernel=True, imgs=None):
	"""one half-sweep of colour `colour` with no refinement tries -> Sweep.  cost: the stored costs (the sign bit is the
	kernel's changed memory; every comparison takes |cost|)."""
	H, W = d.shape
	dirn = sweep & 1
	ys, xs = np.mgrid[HALF:H-HALF, HALF:W-HALF]
	sel = ((xs+ys+colour) & 1) == 0
	xs, ys = xs[sel], ys[sel]
	pt = patch64(case.views[0].image, xs, ys)
	act, und_act = pixels_active(case, xs, ys, pt[3])
	assert not und_act.any(), "a sweep state with an undecided magnitude reject"
	xs, ys = xs[act], ys[act]
	P = len(xs)
	ac = np.abs(cost)
	close, slots = [], []
	for k in range(4):
		kk, ox, oy = _close_offset(dirn, k)
		ok = xs > HALF if kk == 0 else ys > HALF if kk == 1 else xs < W-HALF if kk == 2 else ys < H-HALF
		nxs, nys = xs+ox, ys+oy
		valid = ok & (d[nys, nxs] > 0)
		close.append((valid, nxs, nys, d[nys, nxs].astype(np.float64), n[nys, nxs].astype(np.float64)))
		best = np.where(valid, ac[nys, nxs], 3.0).astype(np.float32)
		ring = np.zeros(P, np.int64)
		if k < nprop:
			alive = ok.copy()
			for f in range(1, far+1):
				qx, qy = xs+ox*(2*f+1), ys+oy*(2*f+1)
				alive &= (qx >= HALF) & (qy >= HALF) & (qx < W-HALF) & (qy < H-HALF)
				fc = ac[np.clip(qy, 0, H-1), np.clip(qx, 0, W-1)]
				better = alive & (fc < best)
				best = np.where(better, fc, best); ring = np.where(better, f, ring)
			has = ok & (best < _f32(KEEP))
		else:
			has = np.zeros(P, bool)
		dist = 2*ring+1
		qx, qy = xs+ox*dist, ys+oy*dist
		slots.append((has, kk, qx, qy))
	X0x, X0y = _ray(case.views[0].K, xs, ys)
	imgs = imgs or [_Img(v.image) for v in case.views[1:]]
	hyps = []
	for has, kk, qx, qy in slots:
		qd = d[qy, qx].astype(np.float64); qn = n[qy, qx].astype(np.float64)
		hd, und_i, other = interpolate64(case, xs, ys, qx, qy, qd, qn, bool(kk & 1))
		hn, en, und_n = correct_normal64(qn, X0x, X0y)
		hd_v = np.where(has, hd.v, 5.0); hn_v = np.where(has[:, None], hn, [0, 0, -1.0])
		ps = score64(case, xs, ys, hd_v, hn_v, smooth64(case, xs, ys, hd_v, hn_v, close), kernel=kernel, views=imgs)
		# hypothesis rounding: the float rounding of the interpolated depth (and of a corrected normal) moves the score by
		# about its central difference over the rounding bound
		step = np.maximum(hd.e, 0.0)
		sp = score64(case, xs, ys, hd_v+step, hn_v, smooth64(case, xs, ys, hd_v+step, hn_v, close), kernel=kernel, views=imgs).val
		sm = score64(case, xs, ys, hd_v-step, hn_v, smooth64(case, xs, ys, hd_v-step, hn_v, close), kernel=kernel, views=imgs).val
		rnd = np.abs(sp-sm)/2
		if (en[has] > 0).any():
			t1 = np.cross(hn_v, [0.0, 1.0, 0.0]); t1 /= np.linalg.norm(t1, axis=-1, keepdims=True)
			t2 = np.cross(hn_v, t1)
			for t in (t1, t2):
				a = score64(case, xs, ys, hd_v, hn_v+en[:, None]*t, smooth64(case, xs, ys, hd_v, hn_v+en[:, None]*t, close), kernel=kernel, views=imgs).val
				b = score64(case, xs, ys, hd_v, hn_v-en[:, None]*t, smooth64(case, xs, ys, hd_v, hn_v-en[:, None]*t, close), kernel=kernel, views=imgs).val
				rnd = rnd+np.where(en > 0, np.abs(a-b)/2, 0.0)
		hyps.append(dict(has=has, hd=hd, hn=hn, en=en, other=other, und=(und_i | und_n) & has, ps=ps, rnd=rnd, q=(qx, qy)))
	conf = ac[ys, xs].astype(np.float64); cm = np.zeros(P)
	winner = np.full(P, -1); dec = np.ones(P, bool)
	for k, h in enumerate(hyps):
		ps = h["ps"]
		nm = ps.mar+h["rnd"]
		gap = conf-ps.val
		decided = ps.dec & ~h["und"] & (np.abs(gap) > cm+nm)
		dec &= ~h["has"] | decided
		acc = h["has"] & (gap > 0)
		conf = np.where(acc, ps.val, conf); cm = np.where(acc, nm, cm); winner = np.where(acc, k, winner)
	return Sweep(xs, ys, winner, dec, conf, cm, hyps, 1.0-dec.mean() if P else 0.0)


def check_sweep(name, case, d, n, cost, colour, sw, od, on, oc):
	"""the state after a half-sweep (kernel or oracle: od, on, oc) against propagate64's Sweep sw -> undecidable fraction"""
	H, W = d.shape
	act = np.zeros((H, W), bool); act[sw.ys, sw.xs] = True
	same = ~act
	assert np.array_equal(od[same], d[same]) and np.array_equal(on[same], n[same]), name+": a pixel outside the half-sweep changed"
	assert np.array_equal(oc[same].view(np.uint32), cost[same].view(np.uint32)), name+": a cost outside the half-sweep changed"
	xs, ys = sw.xs, sw.ys
	gd, gn, gc = od[ys, xs], on[ys, xs], oc[ys, xs]
	kept = (gd == d[ys, xs]) & (gn == n[ys, xs]).all(1)
	nocand = ~np.any([h["has"] for h in sw.hyps], 0)
	assert kept[nocand].all() and np.array_equal(gc[nocand], np.abs(cost[ys, xs][nocand])), name+": a pixel without candidates changed"
	# every output plane is the own one or a candidate's hypothesis (either side of an undecided InterpolatePixel switch)
	match = np.full((len(xs), 4), False)
	for k, h in enumerate(sw.hyps):
		tol_d = 2*h["hd"].e+np.abs(h["hd"].v)*2**-23
		md = (np.abs(gd-h["hd"].v) <= tol_d) | (h["und"] & (np.abs(gd-h["other"]) <= np.abs(h["other"])*2**-20))
		mn = np.abs(gn-h["hn"]).max(1) <= h["en"]+2**-23
		match[:, k] = h["has"] & md & mn
	okp = kept | match.any(1)
	bad = np.flatnonzero(~okp)
	assert len(bad) == 0, "%s: %d planes are neither kept nor a candidate's, e.g. %s" % (name, len(bad), [
		(int(xs[i]), int(ys[i]), float(gd[i]), [float(h["hd"].v[i]) for h in sw.hyps if h["has"][i]]) for i in bad[:4]])
	# decidable pixels: the expected winner and its score
	dec = sw.dec
	w = sw.winner
	wrong = dec & (((w < 0) & ~kept) | ((w >= 0) & ~match[np.arange(len(xs)), np.maximum(w, 0)]))
	bad = np.flatnonzero(wrong)
	assert len(bad) == 0, "%s: %d decidable pixels took another plane, e.g. %s" % (name, len(bad), [
		(int(xs[i]), int(ys[i]), int(w[i]), float(gd[i]), float(d[ys[i], xs[i]])) for i in bad[:4]])
	bad = np.flatnonzero(dec & (w >= 0) & ~(np.abs(gc-sw.cost) <= sw.cost_mar))
	assert len(bad) == 0, "%s: %d decidable costs differ, e.g. %s" % (name, len(bad), [
		(int(xs[i]), int(ys[i]), float(gc[i]), float(sw.cost[i]), float(sw.cost_mar[i])) for i in bad[:4]])
	return float(1.0-dec.mean()) if len(dec) else 0.0


def sweep_state(c, seed=0):
	"""a consistent state of the case's planes: costs from score64 (an invalid plane has cost 2), with exact ties between
	rings, costs equal to keep, sign-bit costs and invalid close neighbours"""
	H, W = c.depth.shape
	rng = np.random.RandomState(seed)
	d = (c.depth*(1+0.04*rng.randn(H, W))).astype(np.float32)
	n = c.normal+0.2*rng.randn(H, W, 3)
	n = _valid_normals(c.views[0].K, d, n/np.linalg.norm(n, axis=-1, keepdims=True), H, W)
	inval = rng.rand(H, W) < 0.12
	border = np.ones((H, W), bool); border[HALF:H-HALF, HALF:W-HALF] = False
	ys, xs = np.mgrid[HALF:H-HALF, HALF:W-HALF]
	xs, ys = xs.ravel(), ys.ravel()
	pt = patch64(c.views[0].image, xs, ys)
	act, und = pixels_active(c, xs, ys, pt[3])
	rej = np.zeros((H, W), bool); rej[ys[~act], xs[~act]] = True
	dead = inval | border | rej
	d[dead] = 0; n[dead] = 0
	cost = np.full((H, W), 2.0, np.float32)
	live = ~dead
	ly, lx = np.nonzero(live)
	ps = score64(c, lx, ly, d[ly, lx], n[ly, lx])
	cost[ly, lx] = ps.val.astype(np.float32)
	# exact ties between rings: the pixels two apart along a row / a column share a cost
	t = rng.rand(H, W) < 0.15
	ty, tx = np.nonzero(t[:, :-2] & live[:, :-2] & live[:, 2:]); cost[ty, tx+2] = cost[ty, tx]
	t = rng.rand(H, W) < 0.15
	ty, tx = np.nonzero(t[:-2] & live[:-2] & live[2:]); cost[ty+2, tx] = cost[ty, tx]
	cost[live & (rng.rand(H, W) < 0.05)] = _f32(KEEP)
	neg = rng.rand(H, W) < 0.2
	cost[neg] = -cost[neg]
	return d, n, cost


SWEEP_CASES = ["views3", "shape203x151", "shape64x14"]
# (sweep, half, nPropagation, nPropagationFar)
SWEEP_CONFIGS = [(0, 0, 4, 2), (1, 1, 4, 2), (0, 1, 2, 1), (1, 0, 4, 0), (0, 0, 2, 2), (1, 1, 2, 0)]


def sweep_configs(name):
	return SWEEP_CONFIGS if name == "views3" else SWEEP_CONFIGS[:2]


# ---- the oracle pinned to the references -------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def O():
	from oracle import oracle
	return oracle


def oracle_params(O, **kw):
	return O.default_params(schedule=1, nSubResolutionLevels=0, threads=8, **kw)


@pytest.mark.parametrize("name", SCORE_CASES)
def test_oracle_pass_a_equals_float64_reference(O, name):
	c = case(name)
	d, n, cost = O.pm_score(c.views, oracle_params(O), c.dmin, c.dmax, depth=c.depth, normal=c.normal, lowres=c.lowres, depths=c.depths)
	und, mar = check_pass_a("oracle " + name, c, d, n, cost, pass_a_expect(c, kernel=False))
	print("oracle pass A %s: undecidable %.4f, margin median %.2e" % (name, und, np.median(mar) if len(mar) else 0))


@pytest.mark.parametrize("name", SWEEP_CASES)
def test_oracle_propagation_equals_float64_reference(O, name):
	"""pm_iterate with nRandomIters = 0 and the building blocks' propagation settings (bSkipUnchanged = 0); the oracle keeps its
	changed memory apart from the costs, so it is given |cost|"""
	c = case(name)
	d, n, cost = sweep_state(c)
	for sweep, half, nprop, far in sweep_configs(name):
		prm = oracle_params(O, propagation=O.rb_propagation(nprop, far, 0), nRandomIters=0)
		od, on, oc = O.pm_iterate(c.views, prm, c.dmin, c.dmax, d, n, np.abs(cost), sweep, half=half)
		sw = propagate64(c, d, n, cost, half, sweep, nprop, far, kernel=False)
		und = check_sweep("oracle %s %s" % (name, (sweep, half, nprop, far)), c, d, n, np.abs(cost), half, sw, od, on, oc)
		assert und < 0.5


def test_cases_reach_their_regimes():
	"""The cases reach the switches they are built for: taps within 1e-4 / 1e-2 / 0.3 of both inside borders, views rejected for
	sure beside views that score, NCC at +1 and -1, nrmSq <= 1e-16, rejected flat pixels and flat pixels a prior keeps, corner
	depths of both signs and all negative, every geometric switch, scores above 2 before the clamp, the prior's 0.5 clamp"""
	for name in ("shiftx", "shifty"):
		c = case(name)
		A, Ua, xs, ys, ps = pass_a_expect(c)
		dist = np.abs(ps.views[0].dist["tap_inside"][0])
		for delta in (1e-4, 1e-2, 0.3):
			assert (np.abs(dist-delta) < 1e-6+1e-3*delta).sum() > 100, (name, delta)
		assert ps.views[0].rej.any() and (~ps.views[0].rej & ~ps.views[0].maybe).any()
	A, Ua, xs, ys, ps = pass_a_expect(case("identical"))
	r = ps.views[0]
	assert (r.alt_v[~r.rej, 0] < 1e-5).mean() > 0.9                    # ncc -> +1, score 0
	A, Ua, xs, ys, ps = pass_a_expect(case("inverse"))
	r = ps.views[0]
	assert (r.alt_v[~r.rej, 0] > 2-1e-3).mean() > 0.9                  # ncc -> -1, score 2 >= thRobust: the min branch
	c = case("textureless")
	A, Ua, xs, ys, ps = pass_a_expect(c)
	assert not A[34:42, 10:80].any() and ps.views[0].rej.sum() > 200     # magnitude reject; nrmSq <= 1e-16 in the flat band
	A, Ua, xs, ys, ps = pass_a_expect(case("zsign"))
	assert (ps.views[0].sc).sum() > 100
	zc = ps.views[1].dist["corner_z"][0]
	assert len(zc)
	A, Ua, xs, ys, ps = pass_a_expect(case("geometric"))
	g = ps.views[0].dist
	assert (np.abs(g["similarity"][0]) < 1e-3).sum() > 10 and ps.views[2].dist["X1z"][0].max() < 0
	assert any((np.abs(ps.views[i].dist["dmap_border"][0]) < 1).sum() > 10 for i in (0, 1)) and (ps.views[0].alt_ok.sum(1) > 1).any()
	A, Ua, xs, ys, ps = pass_a_expect(case("geometric_inverse"))
	assert (ps.val[ps.dec] == 2).mean() > 0.9
	c = case("prior")
	A, Ua, xs, ys, ps = pass_a_expect(c)
	pc = ps.views[0].dist["prior_clamp"][0]
	assert ((pc > 0) & (pc < 0.2)).sum() > 100 and A[22:34, 14:56].mean() > 0.5


def test_margin_is_first_order_and_not_vacuous():
	"""The margins are small against the scores' range (median below 1e-3), so almost every hypothesis of a textured case is
	decidable and held to its float64 value."""
	c = case("views3")
	A, Ua, xs, ys, ps = pass_a_expect(c)
	assert np.median(ps.mar[ps.dec]) < 1e-3
	assert ps.dec.mean() > 0.99
