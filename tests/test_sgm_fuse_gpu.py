"""Fusion-mode -2 on the H100: the projection, fusion and normal kernels bit-identical to the sequential oracle
(oracle/sgm_fuse_oracle.cpp), the host and device forms in agreement, the chain from the device tSGM matcher, and argument checks
that refuse before any launch."""
import numpy as np
import pytest

from oracle import sgm_fuse as F
from test_sgm_fuse import (E2E_SIZE, bgr, depth_quality, projection_cases, rect_q, rectified_scene)

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.fixture(scope="module")
def sgm():
	from openmvs_b200.depth_estimator import SemiGlobalMatcher
	m = SemiGlobalMatcher()
	yield m
	m.Release()


def cuda(a):
	return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def random_pairs(W, H, n, seed, costs=True):
	"""n pairs of smooth noisy disparity maps with holes, rectified-pair Q's of different baselines and principal points, so that the
	projections of the pairs overlap, disagree in places and cover the border"""
	rng = np.random.RandomState(seed)
	f = 0.9*W
	out = []
	for p in range(n):
		vw, vh = W-6+rng.randint(-8, 9), H-6+rng.randint(-8, 9)
		b = rng.uniform(0.2, 0.4)
		ys, xs = np.mgrid[0:vh, 0:vw].astype(np.float64)
		depth = 5.5 + 0.3*np.sin(xs/37.0+p)*np.cos(ys/23.0) + (rng.rand(vh, vw) < 0.05)*rng.uniform(-1, 1, (vh, vw))
		d = np.rint(-f*b/depth*4 + rng.randint(-2, 3, (vh, vw))).astype(np.int16)
		d[rng.rand(vh, vw) < 0.1] = 32767
		Q = rect_q(f, b)
		Q[0, 3], Q[1, 3] = rng.uniform(-3, 3)*f, rng.uniform(-3, 3)*f   # shifted positions
		cost = rng.randint(0, 4000, (vh, vw)).astype(np.uint16) if costs else None
		out.append((d, cost, Q, 4))
	return out


@pytest.mark.parametrize("case", projection_cases(), ids=lambda c: c[0])
def test_projection_bit_identical(sgm, case):
	name, d, c, Q, steps, (W, H) = case
	od, orng, oc, _ = F.project(d, c, Q, steps, (W, H))
	gd, gr, gc = sgm.ProjectDisparity2DepthMap(cuda(d), None if c is None else cuda(c), Q, steps, (W, H))
	assert np.array_equal(bits(gd.cpu().numpy()), bits(od)) and np.array_equal(bits(gr.cpu().numpy()), bits(orng))
	assert np.array_equal(bits(gc.cpu().numpy()), bits(oc))


@pytest.mark.parametrize("size,n,costs", [((97, 61), 3, True), ((160, 120), 5, False), ((1920, 1080), 8, True)],
	ids=["97x61x3", "160x120x5_nocost", "1080p_x8"])
def test_fuse_bit_identical_and_host_equals_device(sgm, size, n, costs):
	W, H = size
	pairs = random_pairs(W, H, n, seed=W+n, costs=costs)
	f = 0.9*W
	K = np.array([[f, 0, (W-1)/2.0], [0, f*1.01, (H-1)/2.0], [0, 0, 1.0]])
	od, oc, on = F.fuse(pairs, size, 2, K)
	assert (od > 0).mean() > 0.3
	dev = [(cuda(d), None if c is None else cuda(c), Q, s) for d, c, Q, s in pairs]
	gd, gc, gn = sgm.Fuse(dev, size, 2, K)
	gd, gc, gn = gd.cpu().numpy(), gc.cpu().numpy(), gn.cpu().numpy()
	assert np.array_equal(bits(gd), bits(od)) and np.array_equal(bits(gc), bits(oc)) and np.array_equal(bits(gn), bits(on))
	hd, hc, hn = sgm.Fuse(pairs, size, 2, K)
	assert np.array_equal(bits(hd), bits(gd)) and np.array_equal(bits(hc), bits(gc)) and np.array_equal(bits(hn), bits(gn))
	assert sgm.stats.kernel_launches == 4
	# the per-pair projections of the fusion are the building block's
	for d, c, Q, s in pairs[:2]:
		pd, pr, pc, _ = F.project(d, c, Q, s, size)
		qd, qr, qc = sgm.ProjectDisparity2DepthMap(cuda(d), None if c is None else cuda(c), Q, s, size)
		assert np.array_equal(bits(qd.cpu().numpy()), bits(pd)) and np.array_equal(bits(qr.cpu().numpy()), bits(pr))


def test_estimate_normal_map_bit_identical():
	from openmvs_b200.depth_estimator import EstimateNormalMap
	rng = np.random.RandomState(4)
	H, W = 77, 131
	ys, xs = np.mgrid[0:H, 0:W]
	depth = (4 + 0.01*xs + 0.02*np.sin(ys/5.0) + 0.05*(rng.rand(H, W) < 0.05)).astype(np.float32)
	depth[rng.rand(H, W) < 0.1] = 0
	K = np.array([[120.3, 0, 65.1], [0, 119.7, 38.2], [0, 0, 1]])
	gn = EstimateNormalMap(K, cuda(depth)).cpu().numpy()
	assert np.array_equal(bits(gn), bits(F.normals(depth, K)))
	assert (np.abs(np.linalg.norm(gn, axis=-1)-1) < 1e-6)[np.abs(gn).sum(-1) > 0].all()


def test_end_to_end_from_the_device_matcher(sgm):
	"""MatchPairHierarchicalDevice on both rendered pairs, then Fuse on the device.  The matcher differs from the oracle's tsgm_match
	at single pixels (its cost volume at one level, DESIGN §5.3), so the chain is held to the quality the CPU chain reaches
	(test_sgm_fuse.test_end_to_end_on_rendered_pairs: coverage 0.7804, 0.7431 within 1 %) minus a margin, not to bits."""
	views, K, pairs = rectified_scene(*E2E_SIZE)
	maps = []
	for l, r, Q in pairs:
		lv, rv = views[l], views[r]
		d, c, _ = sgm.MatchPairHierarchicalDevice(cuda(lv.image), cuda(bgr(lv)), cuda(rv.image), cuda(bgr(rv)), subpixelSteps=4)
		maps.append((d, c, Q, 4))
	depth, conf, normal = sgm.Fuse(maps, E2E_SIZE, 2, K)
	cov, ok = depth_quality(depth.cpu().numpy(), views[0].depth_gt)
	assert cov > 0.74 and ok > 0.70, (cov, ok)
	assert normal is not None and bool(((conf > 0) == (depth > 0)).all())


def test_bad_arguments_launch_nothing(sgm):
	from openmvs_b200 import lib
	dll = lib.load()
	W, H = 64, 48
	pairs = random_pairs(W, H, 2, seed=1)
	dev = [(cuda(d), cuda(c), Q, s) for d, c, Q, s in pairs]
	depth = torch.full((H, W), 7.0, device="cuda"); conf = torch.full((H, W), 7.0, device="cuda")
	def call(plist, n, w=W, h=H):
		arr, keep = sgm._pairs(plist, True)
		rc = dll.b200mvs_sgm_fuse_device(sgm._ctx, arr, n, w, h, 2, None, depth.data_ptr(), conf.data_ptr(), None, None)
		torch.cuda.synchronize()
		return rc
	base = sgm._pairs(dev, True)[0]
	many = (lib.SgmPair*(lib.SGM_MAX_PAIRS+1))(*([base[0]]*(lib.SGM_MAX_PAIRS+1)))
	assert dll.b200mvs_sgm_fuse_device(sgm._ctx, many, lib.SGM_MAX_PAIRS+1, W, H, 2, None, depth.data_ptr(), conf.data_ptr(), None,
		None) == 1                                                 # above B200MVS_SGM_MAX_PAIRS
	assert dll.b200mvs_sgm_fuse_device(sgm._ctx, many, 0, W, H, 2, None, depth.data_ptr(), conf.data_ptr(), None, None) == 1
	assert call([dev[0], (dev[1][0], None, dev[1][2], 4)], 2) == 1  # a cost map on one pair only
	assert call(dev, 2, 0, H) == 1 and call(dev, 2, W, -1) == 1    # empty target
	bad = sgm._pairs(dev, True)[0]
	bad[1].width = 0                                               # a map without pixels
	assert dll.b200mvs_sgm_fuse_device(sgm._ctx, bad, 2, W, H, 2, None, depth.data_ptr(), conf.data_ptr(), None, None) == 1
	bad[1].width, bad[1].subpixelSteps = dev[1][0].shape[1], 0
	assert dll.b200mvs_sgm_fuse_device(sgm._ctx, bad, 2, W, H, 2, None, depth.data_ptr(), conf.data_ptr(), None, None) == 1
	k = np.eye(3).ravel()
	assert dll.b200mvs_sgm_fuse_device(sgm._ctx, sgm._pairs(dev, True)[0], 2, W, H, 2, k.ctypes.data, depth.data_ptr(), conf.data_ptr(),
		None, None) == 1                                           # K without a normal map
	torch.cuda.synchronize()
	assert bool((depth == 7).all()) and bool((conf == 7).all())
	with pytest.raises(ValueError):
		sgm.Fuse([(dev[0][0], dev[0][1][:-1], dev[0][2], 4)], (W, H))  # cost and disparity of different sizes
	with pytest.raises(lib.B200MVSError):
		sgm.Fuse([(dev[0][0], None, dev[0][2], 4), dev[1]], (W, H))
