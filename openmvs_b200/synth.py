"""Seeded synthetic multi-view scenes with analytic ground truth (SURVEY.md §8(d)).

A smooth textured height-field z = h(x, y) seen by pinhole cameras placed on a spherical
cap and looking at the origin.  Images are rendered by exact ray casting (Newton on the
height function) and an analytic band-limited texture, so depth and normal ground truth
are exact and there is no resampling blur.  Camera convention is the reference's:
X_cam = R (X - C), x ~ K X_cam, pixel centres at integer coordinates
(libs/MVS/Camera.h:331-344).

Pure numpy; deterministic for a given seed (inputs of parity tests are generated once on
the CPU and fed to both the oracle and the CUDA engine).
"""
from __future__ import annotations

import dataclasses
import numpy as np


@dataclasses.dataclass
class View:
	image: np.ndarray      # (H, W) float32 gray in [0, 1]
	K: np.ndarray          # (3, 3) float64
	R: np.ndarray          # (3, 3) float64
	C: np.ndarray          # (3,) float64
	depth_gt: np.ndarray   # (H, W) float32
	normal_gt: np.ndarray  # (H, W, 3) float32 camera space, facing the camera


@dataclasses.dataclass
class Scene:
	views: list
	dmin: float
	dmax: float

	def neighbors(self, ref: int, n: int) -> list:
		"""indices of the n nearest views (by camera centre) of `ref`"""
		c = np.stack([v.C for v in self.views])
		d = np.linalg.norm(c - c[ref], axis=1)
		order = [int(i) for i in np.argsort(d, kind="stable") if i != ref]
		return order[:n]


def _height(x, y, xp=np):
	h = 0.22*xp.sin(1.7*x + 0.3)*xp.cos(1.3*y - 0.2) + 0.08*xp.sin(3.1*x - 1.0)*xp.sin(2.7*y + 0.5)
	hx = 0.22*1.7*xp.cos(1.7*x + 0.3)*xp.cos(1.3*y - 0.2) + 0.08*3.1*xp.cos(3.1*x - 1.0)*xp.sin(2.7*y + 0.5)
	hy = -0.22*1.3*xp.sin(1.7*x + 0.3)*xp.sin(1.3*y - 0.2) + 0.08*2.7*xp.sin(3.1*x - 1.0)*xp.cos(2.7*y + 0.5)
	return h, hx, hy


class _Texture:
	def __init__(self, seed: int, px_per_unit: float, n_waves: int = 20):
		rng = np.random.RandomState(seed)
		# wavelengths between 5 and 48 pixels in the image (log-uniform)
		lam_px = np.exp(rng.uniform(np.log(5.0), np.log(48.0), n_waves))
		freq = 2*np.pi*px_per_unit/lam_px
		ang = rng.uniform(0, np.pi, n_waves)
		self.fx = freq*np.cos(ang)
		self.fy = freq*np.sin(ang)
		self.ph = rng.uniform(0, 2*np.pi, n_waves)
		amp = rng.uniform(0.6, 1.0, n_waves)
		self.amp = amp/np.sqrt((amp**2).sum()/2.0)  # unit variance of the sum

	def __call__(self, x, y, xp=np):
		acc = xp.zeros_like(x)
		for fx, fy, ph, a in zip(self.fx, self.fy, self.ph, self.amp):
			acc += float(a)*xp.sin(float(fx)*x + float(fy)*y + float(ph))
		return xp.clip(0.5 + 0.17*acc, 0.0, 1.0)


def look_at(C, target=np.zeros(3)):
	z = target - C
	z = z/np.linalg.norm(z)
	x = np.cross(np.array([0.0, 1.0, 0.0]), z)
	x = x/np.linalg.norm(x)
	y = np.cross(z, x)
	return np.stack([x, y, z])


def _render(K, R, C, tex, xs, ys, xp):
	"""ray cast of the height-field through the pixel centres (xs, ys) of camera (K, R, C) -> (image, depth, camera-space normal)"""
	# rays in world space, parameterised so that t == camera-space depth: D = R^T K^-1 (x,y,1)
	dx = (xs-K[0, 2])/K[0, 0]
	dy = (ys-K[1, 2])/K[1, 1]
	D = [dx*R[0, k] + dy*R[1, k] + R[2, k] for k in range(3)]
	t = (0.0-C[2])/D[2]
	for _ in range(12):
		px = C[0]+t*D[0]
		py = C[1]+t*D[1]
		h, hx, hy = _height(px, py, xp)
		F = C[2]+t*D[2]-h
		dF = D[2]-(hx*D[0]+hy*D[1])
		t = t-F/dF
	px = C[0]+t*D[0]
	py = C[1]+t*D[1]
	h, hx, hy = _height(px, py, xp)
	inv = 1.0/xp.sqrt(hx*hx + hy*hy + 1.0)
	nw = [-hx*inv, -hy*inv, inv]
	nc = xp.stack([nw[0]*R[k, 0] + nw[1]*R[k, 1] + nw[2]*R[k, 2] for k in range(3)], -1)
	return tex(px, py, xp), t, nc


def render_view(K, R, C, width: int, height: int, seed: int = 1234, px_per_unit: float | None = None, radius: float = 5.5) -> View:
	"""The surface and texture of make_scene seen through any pinhole camera (K, R, C) at width x height: gray image, ground-truth
	depth and normal, exact per pixel (no resampling).  The texture is make_scene's for the same seed and px_per_unit (make_scene uses
	its focal length / radius; default here: K[0, 0] / radius).  Cameras that share R and K and differ by a shift along their x axis
	give a rectified pair directly."""
	K = np.asarray(K, np.float64); R = np.asarray(R, np.float64); C = np.asarray(C, np.float64)
	tex = _Texture(seed, px_per_unit=(K[0, 0]/radius) if px_per_unit is None else px_per_unit)
	ys, xs = np.mgrid[0:height, 0:width].astype(np.float64)
	img, t, nc = _render(K, R, C, tex, xs, ys, np)
	return View(img.astype(np.float32), K.copy(), R.copy(), C.copy(), t.astype(np.float32), nc.astype(np.float32))


def make_scene(width: int, height: int, n_views: int, seed: int = 1234, radius: float = 5.5,
		step_deg: float = 4.0, focal_ratio: float = 0.9, cols: int | None = None, device=None, gt_views=None) -> Scene:
	"""n_views cameras on a (rows x cols) angular grid `step_deg` apart, radius `radius`.
	device: None -> numpy float64 (bit-reproducible inputs for the parity tests);
	a torch device -> the same arithmetic in torch float64 on that device (fast, for the bench)."""
	if cols is None:
		cols = int(np.ceil(np.sqrt(n_views*4/3.0))) if n_views > 2 else n_views
	rows = int(np.ceil(n_views/cols))
	f = focal_ratio*width
	K = np.array([[f, 0, (width-1)/2.0], [0, f, (height-1)/2.0], [0, 0, 1.0]])
	tex = _Texture(seed, px_per_unit=f/radius)
	views = []
	if device is None:
		xp = np
		ys, xs = np.mgrid[0:height, 0:width].astype(np.float64)
	else:
		import torch
		xp = torch
		ys, xs = torch.meshgrid(torch.arange(height, dtype=torch.float64, device=device),
			torch.arange(width, dtype=torch.float64, device=device), indexing="ij")
	for i in range(n_views):
		r, c = divmod(i, cols)
		ax = np.deg2rad(step_deg*(c-(cols-1)/2.0))
		ay = np.deg2rad(step_deg*(r-(rows-1)/2.0))
		C = radius*np.array([np.sin(ax)*np.cos(ay), np.sin(ay), np.cos(ax)*np.cos(ay)])
		R = look_at(C)
		img, t, nc = _render(K, R, C, tex, xs, ys, xp)
		keep = gt_views is None or i in gt_views   # large scenes: ground truth only for the views that are checked (16 B per pixel)
		if device is None:
			views.append(View(img.astype(np.float32), K.copy(), R, C, t.astype(np.float32) if keep else None, nc.astype(np.float32) if keep else None))
		else:
			views.append(View(img.float().cpu().numpy(), K.copy(), R, C, t.float().cpu().numpy() if keep else None, nc.float().cpu().numpy() if keep else None))
	return Scene(views, dmin=float(radius-1.5), dmax=float(radius+1.5))


def make_stereo_pair(width: int, height: int, seed: int = 7, d0: float = 12.0, amp: float = 6.0, right_color: bool = False):
	"""Rectified synthetic pair for the SGM path: left(x, y) = right(x + d(x, y), y) with a smooth
	analytic disparity d = d0 + amp*sin(.)cos(.) (the reference's convention: the cost of
	disparity d compares left x with right x+d, libs/MVS/SemiGlobalMatcher.cpp:960).
	Returns left gray float32, left BGR uint8, right gray float32, ground-truth disparity."""
	tex = _Texture(seed, px_per_unit=1.0)
	tex_c = [_Texture(seed+11+k, px_per_unit=1.0, n_waves=6) for k in range(3)]
	ys, xs = np.mgrid[0:height, 0:width].astype(np.float64)
	d = d0 + amp*np.sin(2*np.pi*xs/(0.9*width)+0.4)*np.cos(2*np.pi*ys/(1.3*height)-0.3)
	left = tex(xs+d, ys)
	right = tex(xs, ys)
	bgr = np.stack([np.clip(0.8*left+0.2*t(xs+d, ys), 0, 1) for t in tex_c], -1)
	out = (left.astype(np.float32), np.rint(bgr*255).astype(np.uint8), right.astype(np.float32), d.astype(np.float32))
	if right_color:  # + right BGR uint8
		bgr_r = np.stack([np.clip(0.8*right+0.2*t(xs, ys), 0, 1) for t in tex_c], -1)
		out = out+(np.rint(bgr_r*255).astype(np.uint8),)
	return out


def sgm_pixel_map(width: int, height: int, dmin, dmax, invalid=None):
	"""PixelMap of the valid region (width-6) x (height-6): per-pixel [dmin, dmax) (scalars or
	arrays), idx = running offset into the ragged cost volume (SemiGlobalMatcher.cpp:660-667).
	Returns (structured array {idx u8, dmin i2, dmax i2, reserved i4}, numCosts)."""
	vw, vh = width-6, height-6
	lo = np.broadcast_to(np.asarray(dmin, np.int16), (vh, vw)).copy()
	hi = np.broadcast_to(np.asarray(dmax, np.int16), (vh, vw)).copy()
	if invalid is not None:
		lo[invalid] = np.iinfo(np.int16).max
		hi[invalid] = np.iinfo(np.int16).max
	num = np.maximum(hi.astype(np.int64)-lo.astype(np.int64), 0).ravel()
	px = np.zeros(vh*vw, dtype=np.dtype([("idx", "<u8"), ("dmin", "<i2"), ("dmax", "<i2"), ("reserved", "<i4")]))
	px["idx"] = np.concatenate([[0], np.cumsum(num)[:-1]])
	px["dmin"] = lo.ravel(); px["dmax"] = hi.ravel()
	return px, int(num.sum())


def make_noisy_dmaps(scene: Scene, seed: int = 7, noise: float = 0.002, outliers: float = 0.03, holes: float = 0.05):
	"""Per view (depth, conf) float32 maps as an estimator would leave them: ground-truth depth with
	relative Gaussian noise, a fraction of gross outliers (x U(0.7, 1.3)), a fraction of rejected pixels
	(depth 0, conf 0), confidence U(0.1, 1).  Inputs of the FilterDepthMap parity tests."""
	rng = np.random.RandomState(seed)
	out = []
	for v in scene.views:
		h, w = v.depth_gt.shape
		d = v.depth_gt.astype(np.float64)*(1.0+noise*rng.randn(h, w))
		o = rng.rand(h, w) < outliers
		d[o] *= rng.uniform(0.7, 1.3, int(o.sum()))
		c = rng.uniform(0.1, 1.0, (h, w))
		z = rng.rand(h, w) < holes
		d[z] = 0; c[z] = 0
		out.append((d.astype(np.float32), c.astype(np.float32)))
	return out
