"""Fusion-mode -2 without a GPU: the sequential oracle of SemiGlobalMatcher::ProjectDisparity2DepthMap / ::Fuse / EstimateNormalMap
(oracle/sgm_fuse_oracle.cpp) against an independent pure-Python transcription, hand-built fusion cases, known answers, the Q of a
reversed pair, the .dimap files and the whole chain on rendered rectified pairs.  The helpers here also feed test_sgm_fuse_gpu.py."""
import struct

import numpy as np
import pytest

from oracle import sgm_fuse as F

NO_DISP = 32767
f32 = np.float32


# ---- an independent transcription of ProjectDisparity2DepthMap (libs/MVS/SemiGlobalMatcher.cpp:1925-2039) ----

def py_project(disp, cost, Q, steps, W, H, stats=None):
	"""Python floats for the double arithmetic, numpy float32 scalars for the float arithmetic, the reference's loops and its four
	buffers with the sequential `ndepth > 0 && ndistSq <= distSq` test.  stats (dict, optional) counts the branches taken."""
	st = stats if stats is not None else {}
	inc = lambda k: st.__setitem__(k, st.get(k, 0)+1)
	q = [float(x) for x in np.asarray(Q, np.float64).ravel()]
	bufs = [{} for _ in range(4)]   # (y, x) -> [dist, depth, lo, hi, conf]

	def d2d(ux, uy, d):
		w = q[12]*ux + q[13]*uy - q[14]*float(d) + q[15]
		if abs(w) < 1e-7:
			return f32(0)
		z = q[8]*ux + q[9]*uy - q[10]*float(d) + q[11]
		dep = f32(z/w)
		return f32(0) if dep < f32(0.0001) else dep

	vh, vw = disp.shape
	for r in range(vh):
		for c in range(vw):
			dint = int(disp[r, c])
			if dint == NO_DISP:
				inc("holes"); continue
			d = f32(dint)/f32(steps)
			ux, uy = c+3, r+3
			w = q[12]*ux + q[13]*uy - q[14]*float(d) + q[15]
			if abs(w) < 1e-7:
				inc("w0"); continue
			z = (q[8]*ux + q[9]*uy - q[10]*float(d) + q[11])/w
			if z < 1e-7:
				inc("behind"); continue
			nrm = 1.0/(w*z)
			px = f32((q[0]*ux + q[1]*uy - q[2]*float(d) + q[3])*nrm)
			py = f32((q[4]*ux + q[5]*uy - q[6]*float(d) + q[7])*nrm)
			dep = f32(z)
			fx, fy = np.floor(px), np.floor(py)
			if not (-1 <= fx <= W and -1 <= fy <= H):
				inc("outside"); continue
			dc = int(np.int16(int(np.floor(d))))
			lo, hi = d2d(ux, uy, f32(dc-1)), d2d(ux, uy, f32(dc+1))
			cf = f32(1)/f32(int(cost[r, c])+1) if cost is not None else f32(0)
			x0, y0 = int(fx), int(fy)
			pxm, pym = px-f32(0.5), py-f32(0.5)
			for i in (-1, 0, 1):
				for j in (-1, 0, 1):
					nx, ny = x0+j, y0+i
					if not (0 <= nx < W and 0 <= ny < H):
						inc("clipped"); continue
					dx, dy = f32(nx)-pxm, f32(ny)-pym
					if abs(dx) > f32(0.75) or abs(dy) > f32(0.75):
						continue
					k = (1 if dx < 0 else 0)+(2 if dy < 0 else 0)
					inc("quadrant%d" % k)
					if nx in (0, W-1) or ny in (0, H-1):
						inc("border")
					dsq = dx*dx+dy*dy
					old = bufs[k].get((ny, nx))
					if old is not None and old[0] <= dsq:
						if old[0] == dsq:
							inc("tie")
						continue
					bufs[k][(ny, nx)] = [dsq, dep, lo, hi, cf]
	depth = np.zeros((H, W), f32); rng = np.zeros((H, W, 2), f32); conf = np.zeros((H, W), f32)
	for y in range(H):
		for x in range(W):
			ent = [b.get((y, x)) for b in bufs]
			distC, depC = f32(np.finfo(f32).max), f32(0)
			for e in ent:
				if e is not None and distC > e[0]:
					distC, depC = e[0], e[1]
			if distC > f32(0.75)*f32(0.75):
				continue
			v = [f32(0)]*4
			wsum = f32(0)
			for e in ent:
				if e is None or not (abs(depC-e[1])/depC < f32(0.02)):
					continue
				wt = np.sqrt(e[0])
				v = [v[i]+e[1+i]*wt for i in range(4)]
				wsum = wsum+wt
			if not wsum > 0:
				inc("zero_weight"); continue
			inv = f32(1)/wsum
			depth[y, x], rng[y, x, 0], rng[y, x, 1], conf[y, x] = (vi*inv for vi in v)
	return depth, rng, conf


def scaled_q(sx, ox, sy, oy, qw=0.25):
	"""Q of a synthetic pair: pixel (sx x + ox, sy y + oy), depth 1/(-qw d): quarter-pixel positions for sx, sy in quarters"""
	return np.array([[sx, 0, 0, ox], [0, sy, 0, oy], [0, 0, 0, 1.0], [0, 0, qw, 0]], np.float64)


def projection_cases():
	"""(name, disparity, cost or None, Q, subpixelSteps, (W, H)) small enough for the Python transcription"""
	out = []
	rng = np.random.RandomState(5)
	def disp_map(vh, vw, lo=-80, hi=8, holes=0.15):
		d = rng.randint(lo, hi, (vh, vw)).astype(np.int16)   # includes 0 (w == 0) and positive values (negative depth)
		d[rng.rand(vh, vw) < holes] = NO_DISP
		return d
	cost = lambda d: rng.randint(0, 3000, d.shape).astype(np.uint16)
	d = disp_map(24, 40)
	out.append(("quarters", d, cost(d), scaled_q(0.25, 0.0, 0.25, 0.0), 4, (10, 7)))
	d = disp_map(24, 40)
	out.append(("quarters_shifted_nocost", d, None, scaled_q(0.25, -0.5, 0.25, -0.25), 4, (11, 8)))
	# every column of a row lands on the same x: equal distances in one quadrant, the earliest source wins
	d = disp_map(12, 30, -40, -8, 0.1)
	out.append(("ties", d, cost(d), scaled_q(0.0, 3.25, 0.5, 0.25), 4, (8, 9)))
	# depth-similar neighbours around exact quarter pixels: the weighted means
	d = np.full((20, 36), -32, np.int16) + rng.randint(-1, 2, (20, 36)).astype(np.int16)
	out.append(("smooth", d, cost(d), scaled_q(0.5, 0.25, 0.5, -0.25), 4, (21, 12)))
	# a general Q with off-diagonal terms and subpixelSteps 1 / 16
	Qg = np.array([[0.3, 0.02, 0.01, 0.7], [-0.015, 0.28, 0.004, 0.2], [0.0005, 0.0002, 0.003, 1.0], [0.0, 0.0, 0.2, 0.01]])
	d = disp_map(20, 30, -60, 4)
	out.append(("general_steps1", d, cost(d), Qg, 1, (12, 9)))
	d = disp_map(20, 30, -900, 40)
	out.append(("general_steps16", d, cost(d), Qg, 16, (12, 9)))
	return out


@pytest.mark.parametrize("case", projection_cases(), ids=lambda c: c[0])
def test_oracle_projection_matches_python_transcription(case):
	name, d, c, Q, steps, (W, H) = case
	st = {}
	pd, pr, pc = py_project(d, c, Q, steps, W, H, st)
	od, orng, oc, n = F.project(d, c, Q, steps, (W, H))
	bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)
	assert np.array_equal(bits(od), bits(pd)) and np.array_equal(bits(orng), bits(pr)) and np.array_equal(bits(oc), bits(pc))
	assert n == int((pd > 0).sum()) and n > 0
	if c is None:
		assert not oc.any()


def test_projection_cases_reach_every_branch():
	"""the cases above take every branch of the projection at least once"""
	total = {}
	for name, d, c, Q, steps, (W, H) in projection_cases():
		st = {}
		py_project(d, c, Q, steps, W, H, st)
		for k, v in st.items():
			total[k] = total.get(k, 0)+v
	for k in ("holes", "w0", "behind", "clipped", "border", "tie", "zero_weight", "quadrant0", "quadrant1", "quadrant2", "quadrant3"):
		assert total.get(k, 0) > 0, (k, total)


# ---- the cluster vote of Fuse (SemiGlobalMatcher.cpp:795-848) ----

def _maps(entries, n):
	"""entries: per pair (depth, lo, hi, conf) or None for one pixel -> per-pair 1x1 maps"""
	D = [np.zeros((1, 1), f32) for _ in range(n)]; R = [np.zeros((1, 1, 2), f32) for _ in range(n)]; Cf = [np.zeros((1, 1), f32) for _ in range(n)]
	for p, e in enumerate(entries):
		if e is not None:
			D[p][0, 0], R[p][0, 0, 0], R[p][0, 0, 1], Cf[p][0, 0] = e
	return D, R, Cf


FUSION_CASES = [
	# pair 2 lies in both clusters and joins both; both then hold 2 pairs: the first cluster (pairs 0, 2) wins
	("inside_two", [(1.0, 0.9, 1.1, 0.5), (1.2, 1.05, 1.3, 0.25), (1.07, 1.0, 1.15, 0.125)], 2, (f32(1.0)+f32(1.07))/f32(2), f32(0.625)/f32(2)),
	# two disjoint clusters of one pair each, minViews 1: the first wins
	("tie_first", [(2.0, 1.9, 2.1, 0.5), (3.0, 2.9, 3.1, 0.25)], 1, f32(2.0), f32(0.5)),
	("below_min_views", [(2.0, 1.9, 2.1, 0.5), (3.0, 2.9, 3.1, 0.25)], 2, f32(0), f32(0)),
	# depth exactly on the lower bound joins ([lo, hi)), exactly on the upper bound does not
	("on_lower_bound", [(2.0, 1.9, 2.1, 0.5), (1.9, 1.8, 2.0, 0.25)], 2, (f32(2.0)+f32(1.9))/f32(2), f32(0.75)/f32(2)),
	("on_upper_bound", [(2.0, 1.9, 2.1, 0.5), (2.1, 2.0, 2.2, 0.25)], 2, f32(0), f32(0)),
	# a narrowed range: pair 2 would fit the first range but not the narrowed one; it opens a cluster
	("narrowed", [(2.0, 1.5, 2.5, 1.0), (2.05, 1.95, 2.15, 1.0), (1.9, 1.8, 2.0, 1.0), (2.1, 2.0, 2.2, 1.0)], 2,
		(f32(2.0)+f32(2.05)+f32(2.1))/f32(3), f32(3)/f32(3)),
	("no_depth", [None, (0.0, 0.0, 0.0, 0.0)], 1, f32(0), f32(0)),
]


def py_fuse(D, R, Cf, minViews):
	"""pure-Python cluster vote of one pixel"""
	clusters = []
	for p in range(len(D)):
		d = D[p][0, 0]
		if not d > 0:
			continue
		lo, hi = R[p][0, 0]
		joined = 0
		for cl in clusters:
			if cl[1] <= d < cl[2]:
				cl[0].append(p)
				if cl[1] < lo:
					cl[1] = lo
				if cl[2] > hi:
					cl[2] = hi
				joined += 1
		if not joined:
			clusters.append([[p], lo, hi])
	if not clusters:
		return f32(0), f32(0)
	best = clusters[0]
	for cl in clusters[1:]:
		if len(best[0]) < len(cl[0]):
			best = cl
	if len(best[0]) < minViews:
		return f32(0), f32(0)
	sd, sc = f32(0), f32(0)
	for p in best[0]:
		sd, sc = sd+D[p][0, 0], sc+Cf[p][0, 0]
	return sd/f32(len(best[0])), sc/f32(len(best[0]))


@pytest.mark.parametrize("case", FUSION_CASES, ids=lambda c: c[0])
def test_fusion_cases(case):
	name, entries, minViews, want_d, want_c = case
	D, R, Cf = _maps(entries, len(entries))
	od, oc = F.fuse_maps(D, R, Cf, minViews)
	assert (od[0, 0], oc[0, 0]) == (want_d, want_c)
	assert py_fuse(D, R, Cf, minViews) == (want_d, want_c)


def test_fusion_random_pixels_match_python():
	rng = np.random.RandomState(3)
	n, H, W = 6, 9, 11
	base = rng.uniform(2, 3, (H, W)).astype(f32)
	D = [(base*rng.choice([1.0, 1.005, 1.3], (H, W))*(rng.rand(H, W) > 0.2)).astype(f32) for _ in range(n)]
	R = [np.stack([d*f32(0.99), d*f32(1.01)], -1).astype(f32) for d in D]
	Cf = [rng.rand(H, W).astype(f32) for _ in range(n)]
	od, oc = F.fuse_maps(D, R, Cf, 2)
	for y in range(H):
		for x in range(W):
			pick = lambda ms: [m[y:y+1, x:x+1] for m in ms]
			assert (od[y, x], oc[y, x]) == py_fuse(pick(D), pick(R), pick(Cf), 2), (y, x)
	assert (od > 0).mean() > 0.5


# ---- known answers ----

def rect_q(f, b):
	"""Q of a rectified pair whose left camera is unrectified (H = I), focal f, right camera b to the right: pixel (x, y),
	depth -f b / d"""
	return np.array([[f, 0, 0, 0], [0, f, 0, 0], [0, 0, 0, f], [0, 0, 1.0/b, 0]], np.float64)


def test_fronto_parallel_plane_gives_the_analytic_depth():
	f, b, W, H = 200.0, 0.25, 64, 48
	disp = np.full((H-6, W-6), -40*4, np.int16)   # d = -40: depth = f b / 40
	cost = np.full(disp.shape, 99, np.uint16)
	depth, conf, normal = F.fuse([(disp, cost, rect_q(f, b), 4)]*2, (W, H), 2, K=np.array([[f, 0, W/2.0], [0, f, H/2.0], [0, 0, 1]]))
	inner = depth[3:-3, 3:-3]
	assert (inner > 0).all() and np.allclose(inner, f*b/40.0, rtol=1e-6, atol=0)
	assert np.all(conf[3:-3, 3:-3] == f32(1)/f32(100))
	assert np.allclose(normal[4:-4, 4:-4], [0, 0, -1], atol=1e-6)
	# the depth range of one pair: the depths at d -/+ 1
	_, rng, _, _ = F.project(disp, cost, rect_q(f, b), 4, (W, H))
	assert np.allclose(rng[3:-3, 3:-3, 0], f*b/41.0, rtol=1e-6) and np.allclose(rng[3:-3, 3:-3, 1], f*b/39.0, rtol=1e-6)


def test_tilted_plane_normals():
	"""EstimateNormalMap of the depth of a plane n.X = c seen by a pinhole camera gives n (camera space, facing the camera)"""
	W, H, f = 40, 30, 50.0
	K = np.array([[f, 0, 19.5], [0, f, 14.5], [0, 0, 1.0]])
	n = np.array([0.2, -0.1, -1.0]); n /= np.linalg.norm(n)
	ys, xs = np.mgrid[0:H, 0:W].astype(np.float64)
	rays = np.stack([(xs-K[0, 2])/f, (ys-K[1, 2])/f, np.ones_like(xs)], -1)
	depth = (-3.0/(rays @ n)).astype(f32)
	N = F.normals(depth, K)
	assert np.allclose(N[1:-1, 1:-1], n, atol=2e-3)


# ---- the Q of a reversed pair (SemiGlobalMatcher.cpp:770-779) ----

def _rotation(a, b, c):
	ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
	return np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]]) @ np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]]) @ np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])


def test_reversed_pair_q_lands_on_the_image_pixel_and_depth():
	from openmvs_b200.depth_estimator import SemiGlobalMatcher
	rng = np.random.RandomState(11)
	R = _rotation(0.3, -0.2, 0.1)
	K = np.array([[310.0, 0, 160.2], [0, 310.0, 119.7], [0, 0, 1]])
	b = 0.4
	Cl = np.array([0.3, -0.2, 5.0])   # the pair's left camera (the other view)
	C = Cl + b*R[0]                   # this image: the pair's right camera, shifted along the shared x axis
	Kr = K
	Q = rect_q(Kr[0, 0], b)
	Q2 = F.pair_q(Q, Kr, R, Cl, Kr, R, C)
	assert np.array_equal(Q2, SemiGlobalMatcher.PairQ(Q, Kr, R, Cl, Kr, R, C))
	for _ in range(20):
		X = Cl + R.T @ np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(4, 7)])
		xl = Kr @ (R @ (X-Cl)); xl = xl[:2]/xl[2]
		xr = Kr @ (R @ (X-C)); zr = xr[2]; xr = xr[:2]/xr[2]
		d = xr[0]-xl[0]
		v = Q2 @ np.array([xl[0], xl[1], -d, 1.0])
		z = v[2]/v[3]
		pt = v[:2]/(v[3]*z)
		assert abs(z-zr) <= 1e-9*zr and np.all(np.abs(pt-xr) <= 1e-9*np.abs(xr).max())


# ---- .dimap files (SemiGlobalMatcher.cpp:2094-2184) ----

def test_dimap_round_trip(tmp_path):
	from openmvs_b200 import dmap_io
	rng = np.random.RandomState(2)
	disp = rng.randint(-300, 300, (9, 13)).astype(np.int16); disp[0, 0] = NO_DISP
	cost = rng.randint(0, 65535, (9, 13)).astype(np.uint16)
	H = rng.randn(3, 3); Q = rng.randn(4, 4)
	for c in (cost, None):
		p = str(tmp_path/"a.dimap")
		dmap_io.ExportDisparityDataRawFull(p, disp, c, (19, 15), H, Q, 4)
		full = dmap_io.ImportDisparityDataRaw(p)
		assert full["disparityMap"].shape == (15, 19) and (full["disparityMap"][:3] == NO_DISP).all()
		if c is not None:
			assert (full["costMap"][:, -3:] == dmap_io.NO_ACCUMCOST).all()
		d = dmap_io.ImportDisparityDataRawFull(p)
		assert np.array_equal(d["disparityMap"], disp) and np.array_equal(d["H"], H) and np.array_equal(d["Q"], Q)
		assert d["imageSize"] == (19, 15) and d["subpixelSteps"] == 4
		assert (d["costMap"] is None) if c is None else np.array_equal(d["costMap"], c)


def test_dimap_known_bytes(tmp_path):
	"""a file assembled byte by byte in the reference's fwrite order"""
	from openmvs_b200 import dmap_io
	Hm = np.arange(9, dtype=np.float64)*0.5; Q = np.arange(16, dtype=np.float64)-3.25
	disp = np.array([[1, -2, 3], [NO_DISP, 5, -6]], np.int16); cost = np.array([[7, 8, 9], [65535, 0, 1]], np.uint16)
	raw = struct.pack("<2i", 640, 480) + struct.pack("<9d", *Hm) + struct.pack("<16d", *Q) + struct.pack("<h", 4) + struct.pack("<2i", 3, 2)
	raw += struct.pack("<6h", *disp.ravel())
	for with_cost in (False, True):
		data = raw + (struct.pack("<6H", *cost.ravel()) if with_cost else b"")
		p = str(tmp_path/("c%d.dimap" % with_cost))
		with open(p, "wb") as f:
			f.write(data)
		d = dmap_io.ImportDisparityDataRaw(p)
		assert d["imageSize"] == (640, 480) and d["subpixelSteps"] == 4
		assert np.array_equal(d["H"].ravel(), Hm) and np.array_equal(d["Q"].ravel(), Q) and np.array_equal(d["disparityMap"], disp)
		assert np.array_equal(d["costMap"], cost) if with_cost else d["costMap"] is None
		q = str(tmp_path/"w.dimap")
		dmap_io.ExportDisparityDataRaw(q, disp, cost if with_cost else None, (640, 480), Hm.reshape(3, 3), Q.reshape(4, 4), 4)
		with open(q, "rb") as f:
			assert f.read() == data
	with open(p, "wb") as f:
		f.write(raw + b"\x00")   # a partial cost map
	with pytest.raises(ValueError):
		dmap_io.ImportDisparityDataRaw(p)


# ---- the whole chain on rendered rectified pairs ----

def rectified_scene(W, H, baseline=0.3):
	"""the reference view and two neighbours shifted by -/+ baseline along its x axis (shared K and R: every pair is rectified as
	rendered, H = I) -> (views [ref, left neighbour, right neighbour], K, pairs [(left index, right index, Q)]) with the pairs in
	fusion order: (ref, right neighbour) and (left neighbour, ref), whose Q is re-targeted to the reference with pair_q"""
	from openmvs_b200 import synth
	f = 0.9*W
	K = np.array([[f, 0, (W-1)/2.0], [0, f, (H-1)/2.0], [0, 0, 1.0]])
	ax = np.deg2rad(3.0)
	C0 = 5.5*np.array([np.sin(ax), 0.0, np.cos(ax)])
	R = synth.look_at(C0)
	views = [synth.render_view(K, R, C0 + s*baseline*R[0], W, H, px_per_unit=f/5.5) for s in (0, -1, 1)]
	Q = rect_q(f, baseline)
	pairs = [(0, 2, Q), (1, 0, F.pair_q(Q, K, R, views[1].C, K, R, views[0].C))]
	return views, K, pairs


def bgr(view):
	return np.repeat(np.rint(view.image*255).astype(np.uint8)[..., None], 3, -1)


def depth_quality(depth, gt):
	"""(fraction of pixels with a depth, fraction of those within 1 % of the ground truth)"""
	valid = depth > 0
	return float(valid.mean()), float((np.abs(depth-gt)/gt < 0.01)[valid].mean()) if valid.any() else 0.0


E2E_SIZE = (256, 192)


def test_end_to_end_on_rendered_pairs():
	"""tSGM matching of both pairs by the oracle (oracle.tsgm.tsgm_match, subpixelSteps 4), then the oracle's projection and fusion
	(minViews 2) against the rendered depth of the reference view at 256 x 192.  Measured: coverage 0.7804, and 0.7431 of the covered
	pixels within 1 % of the ground truth (each pair alone: coverage 0.838 / 0.835, within 1 % 0.724 / 0.728).  The reversed pair,
	re-targeted by pair_q, is as good as the direct one."""
	from oracle import tsgm
	views, K, pairs = rectified_scene(*E2E_SIZE)
	maps = []
	for l, r, Q in pairs:
		d, c, _ = tsgm.tsgm_match(views[l].image, bgr(views[l]), views[r].image, bgr(views[r]))
		maps.append((d, c, Q, 4))
		cov, ok = depth_quality(F.project(d, c, Q, 4, E2E_SIZE)[0], views[0].depth_gt)
		assert cov > 0.8 and ok > 0.7, (l, r, cov, ok)
	depth, conf, normal = F.fuse(maps, E2E_SIZE, 2, K)
	cov, ok = depth_quality(depth, views[0].depth_gt)
	assert cov > 0.76 and ok > 0.72, (cov, ok)
	assert ((conf > 0) == (depth > 0)).all() and (conf <= 1).all()
