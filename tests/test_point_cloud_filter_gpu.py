"""Scene::PointCloudFilter on the device: the visibility counts of the host-buffer and device forms equal the exhaustive CPU
restatement (tests/cpp/visibility_oracle.cpp) exactly, on the fused and the merged cloud of a synthetic scene and on adversarial
clouds; PointCloudFilter keeps the oracle's points in the reference's order; two runs are identical; and a 12 x 1080p fused cloud
runs through both forms to the same counts."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

import visibility_oracle as VO  # noqa: E402
from openmvs_b200 import synth  # noqa: E402
from openmvs_b200.depth_estimator import FuseDepthMaps, MergeDepthMaps, PointCloud, PointCloudFilter, PointCloudVisibility  # noqa: E402


def _scene_views(w, h, n, noise, seed, drop=0.1, n_nb=4):
	"""noisy depth-maps of the synthetic scene with holes and a band of outliers, colour and camera-space normal maps"""
	sc = synth.make_scene(w, h, n, step_deg=5.0)
	rng = np.random.RandomState(seed)
	views = []
	for i, v in enumerate(sc.views):
		d = v.depth_gt.astype(np.float32)*(1+noise*rng.randn(h, w)).astype(np.float32)
		d[rng.rand(h, w) < drop] = 0
		d[h//3:h//3+2, :] *= np.float32(0.8)
		color = (np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1)
		nb = list(sc.neighbors(i, min(n-1, n_nb)))
		views.append(dict(depth=d, normal=v.normal_gt.astype(np.float32), conf=rng.rand(h, w).astype(np.float32), color=color,
			K=np.asarray(v.K, np.float64), R=np.asarray(v.R, np.float64), C=np.asarray(v.C, np.float64), neighbors=nb,
			n_scene_neighbors=len(nb)))
	return views


def _on_device(pc):
	return PointCloud(torch.from_numpy(np.ascontiguousarray(pc.points)).cuda(), pc.pointViews, pc.pointWeights, pc.colors, pc.normals,
		pc.projs, pc.nDepths)


def _check(views, pc):
	"""both forms equal the oracle exactly and each other on a second run -> the counts"""
	want = VO.visibility(pc.points, pc.pointViews, views)
	host = PointCloudVisibility(views, pc)
	dev = PointCloudVisibility(views, _on_device(pc))
	assert host.dtype == np.int32 and dev.dtype == torch.int32
	assert np.array_equal(host, want), np.flatnonzero(host != want)[:20]
	assert np.array_equal(dev.cpu().numpy(), want), np.flatnonzero(dev.cpu().numpy() != want)[:20]
	assert np.array_equal(PointCloudVisibility(views, _on_device(pc)).cpu().numpy(), want)
	assert np.array_equal(PointCloudVisibility(views, pc), want)
	return want


@pytest.fixture(scope="module")
def scene():
	views = _scene_views(200, 150, 6, 2e-3, 3)
	fused = FuseDepthMaps(copy.deepcopy(views))
	merged = MergeDepthMaps(copy.deepcopy(views))
	return views, fused, merged


def test_fused_cloud_equals_oracle(scene):
	views, fused, _ = scene
	assert len(fused.points) > 30000
	want = _check(views, fused)
	assert (want < 0).any() and (want > 0).any()


def test_merged_cloud_equals_oracle(scene):
	views, _, merged = scene
	assert len(merged.points) > 100000 and merged.pointWeights is None
	_check(views, merged)


@pytest.mark.parametrize("th", [0, -1, -10, 5])
def test_filter_equals_oracle_in_reference_order(scene, th):
	views, fused, _ = scene
	want = VO.visibility(fused.points, fused.pointViews, views)
	order = VO.filter_order(want, th)
	for pc in (fused, _on_device(fused)):
		out = PointCloudFilter(views, pc, th)
		pts = out.points.cpu().numpy() if torch.is_tensor(out.points) else out.points
		assert np.array_equal(pts, fused.points[order])
		assert len(out.pointViews) == len(out.pointWeights) == len(out.projs) == len(order)
		for k, o in enumerate(order[:: max(1, len(order)//500)]):
			j = k*max(1, len(order)//500)
			assert np.array_equal(out.pointViews[j], fused.pointViews[o]) and np.array_equal(out.pointWeights[j], fused.pointWeights[o])
			assert np.array_equal(out.projs[j], fused.projs[o])
		assert np.array_equal(out.colors, fused.colors[order]) and np.array_equal(out.normals, fused.normals[order])
		assert out.nDepths == fused.nDepths
	assert len(fused.points) == len(fused.pointViews)   # the input is not modified


def _camera(fx, w, h, C, look, up=(0.0, -1.0, 0.0)):
	z = np.asarray(look, np.float64) - C
	z /= np.linalg.norm(z)
	x = np.cross(np.asarray(up, np.float64), z); x /= np.linalg.norm(x)
	y = np.cross(z, x)
	K = np.array([[fx, 0, w/2], [0, fx, h/2], [0, 0, 1]])
	return dict(K=K, R=np.stack([x, y, z]), C=np.asarray(C, np.float64), width=w, height=h)


def _backproject(cam, u, v, depth):
	"""world points at pixels (u, v) and camera depths"""
	K, R, C = cam["K"], cam["R"], cam["C"]
	x = (u - K[0, 2])/K[0, 0]*depth
	y = (v - K[1, 2])/K[1, 1]*depth
	return (np.stack([x, y, depth], -1) @ R) + C


def _adversarial(seed):
	"""three cameras (one of them wide-angle) looking at a slab of points, with duplicate points, points along shared rays,
	points just outside an image and behind a camera, and points whose own view does not see them"""
	rng = np.random.RandomState(seed)
	cams = [_camera(500.0, 320, 240, (0.0, 0, 0), (0, 0, 10)), _camera(520.0, 320, 240, (2.0, 0.5, 0), (0, 0, 10)),
		_camera(60.0, 320, 240, (-1.0, -0.5, 1), (0, 0, 10))]          # 139 degrees across
	pts, views = [], []

	def add(p, vs):
		pts.append(np.asarray(p, np.float32).reshape(-1, 3))
		views.extend([np.asarray(sorted(v), np.uint32) for v in vs])

	n = 3000
	base = _backproject(cams[0], rng.uniform(0, 320, n), rng.uniform(0, 240, n), rng.uniform(8, 12, n))
	add(base, [rng.choice(3, rng.randint(1, 4), replace=False) for _ in range(n)])
	add(base[:300], [[0]]*300)                                           # exact duplicates
	u, v = rng.uniform(0, 320, 40), rng.uniform(0, 240, 40)
	for k in range(40):                                                  # 30 points along each of 40 rays of camera 0
		ray = _backproject(cams[0], np.full(30, u[k]), np.full(30, v[k]), np.sort(rng.uniform(2, 20, 30)))
		add(ray, [[0]]*10 + [[0, 1]]*10 + [[1, 2]]*10)
	m = 400                                                              # just outside camera 0's image, either side of the border
	add(_backproject(cams[0], np.r_[rng.uniform(-4, 0, m//2), rng.uniform(320, 324, m//2)], rng.uniform(-4, 244, m), rng.uniform(8, 12, m)),
		[[0]]*(m//2) + [[0, 2]]*(m//2))
	add(_backproject(cams[0], rng.uniform(-200, -40, 100), rng.uniform(0, 240, 100), rng.uniform(8, 12, 100)), [[0]]*100)   # far outside
	add(rng.uniform(-3, 3, (100, 3))*[1, 1, 0] + [0, 0, -4], [[0]]*50 + [[1]]*50)   # behind cameras 0 and 1
	add(rng.uniform(-3, 3, (50, 3))*[1, 1, 0.01], [[]]*50)              # near the apex plane, no view
	add([[0, 0, 0], [2, 0.5, 0]], [[0], [1]])                            # at an apex: a degenerate cone
	return cams, PointCloud(np.concatenate(pts), views, None)


@pytest.mark.parametrize("seed", [0, 1])
def test_adversarial_clouds_equal_oracle(seed):
	cams, pc = _adversarial(seed)
	want = _check(cams, pc)
	assert (want != 0).sum() > 100
	# a camera looking the other way, with a rotation that is not orthonormal and one with K(2,2) != 1: every query of those
	# views tests every point, and the counts do not change (they depend on width, K(0,0) and C alone)
	odd = copy.deepcopy(cams)
	odd[1]["R"] = odd[1]["R"]*1.001
	odd[2]["K"] = odd[2]["K"]*2.0
	odd[2]["K"][0, 0] = cams[2]["K"][0, 0]
	odd[0]["R"] = -odd[0]["R"]                                           # camera 0 now looks away from every point
	assert np.array_equal(PointCloudVisibility(odd, _on_device(pc)).cpu().numpy(), want)


def test_fused_twelve_views_1080p_host_and_device_agree():
	W, H = 1920, 1080
	views = _scene_views(W, H, 12, 2e-3, 0, n_nb=9)
	dev = [dict(v, **{k: torch.from_numpy(np.ascontiguousarray(v[k])).cuda() for k in ("depth", "normal", "conf", "color")}) for v in views]
	fused = FuseDepthMaps(dev)
	assert len(fused.points) > 4_000_000
	host = PointCloudVisibility(views, fused)
	device = PointCloudVisibility(views, _on_device(fused))
	assert np.array_equal(host, device.cpu().numpy())
	assert (host < 0).any() and (host > 0).any()
