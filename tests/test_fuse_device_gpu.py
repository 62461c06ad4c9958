"""FuseDepthMaps on the device (b200mvs_fuse_depth_maps_device) against the host form (b200mvs_fuse_depth_maps) on identical copies
of the same inputs: the same points, view lists, weights, projections, colours, normals and nDepths, bit for bit, and the same
modified depth-maps.  The scenes cover shared neighbour pixels (a half-resolution neighbour), rejections that release claims and
zero depths (nMin 3, heavy noise, the outlier band), equal connection scores, missing normal / confidence / colour maps, images
without a depth-map or without a depth, and a 12 x 640x480 scene."""
import copy

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from openmvs_b200 import lib, synth  # noqa: E402
from openmvs_b200.depth_estimator import FuseDepthMaps, FuseRoundStats  # noqa: E402


def _scene_views(w, h, n, noise, seed, drop=0.1, with_color=True, n_nb=4):
	"""depth-maps of the synthetic scene as an estimator delivers them: ground truth + relative noise, holes, a band of gross
	outliers in front of the surface, random confidences, camera-space normals"""
	sc = synth.make_scene(w, h, n, step_deg=5.0)
	rng = np.random.RandomState(seed)
	views = []
	for i, v in enumerate(sc.views):
		d = v.depth_gt.astype(np.float32).copy()
		d *= (1+noise*rng.randn(h, w)).astype(np.float32)
		d[rng.rand(h, w) < drop] = 0
		d[h//3:h//3+2, :] *= np.float32(0.8)
		nb = list(sc.neighbors(i, min(n-1, n_nb)))
		color = (np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1) if with_color else None
		views.append(dict(depth=d, normal=v.normal_gt.astype(np.float32), conf=rng.rand(h, w).astype(np.float32), color=color,
			K=np.asarray(v.K, np.float64), R=v.R, C=v.C, neighbors=nb, n_scene_neighbors=len(nb)+(i % 2)))
	return views


def _to_device(views):
	out = []
	for v in views:
		d = dict(v)
		for key in ("depth", "normal", "conf", "color"):
			if v.get(key) is not None:
				d[key] = torch.from_numpy(np.ascontiguousarray(v[key])).cuda()
		out.append(d)
	return out


def _assert_same(views, **kw):
	host = copy.deepcopy(views)
	dev = _to_device(views)
	ph = FuseDepthMaps(host, **kw)
	pd = FuseDepthMaps(dev, **kw)
	assert len(ph.points) > 0
	assert pd.nDepths == ph.nDepths
	assert np.array_equal(pd.points, ph.points)
	assert len(pd.pointViews) == len(ph.pointViews)
	assert all(np.array_equal(a, b) for a, b in zip(pd.pointViews, ph.pointViews))
	assert all(np.array_equal(a, b) for a, b in zip(pd.pointWeights, ph.pointWeights))
	assert all(np.array_equal(a, b) for a, b in zip(pd.projs, ph.projs))
	for name in ("colors", "normals"):
		a, b = getattr(pd, name), getattr(ph, name)
		assert (a is None) == (b is None), name
		if a is not None:
			assert np.array_equal(a, b), name
	for h, d in zip(host, dev):
		if h["depth"] is not None:
			assert np.array_equal(d["depth"].cpu().numpy(), h["depth"])
	return ph, host


@pytest.mark.parametrize("nmin,with_color,seed", [(2, True, 0), (3, True, 1), (1, False, 2)])
def test_equals_host_on_the_oracle_configurations(nmin, with_color, seed):
	views = _scene_views(56, 42, 5, 2e-3, seed, with_color=with_color)
	if seed == 2:
		views[3]["depth"] = None
	ph, host = _assert_same(views, nMinViewsFuse=nmin)
	assert len(ph.points) > 500


def test_half_resolution_neighbour_shares_targets():
	views = _scene_views(96, 72, 5, 2e-3, 3)
	v = views[2]
	S = np.diag([0.5, 0.5, 1.0])
	for key in ("depth", "normal", "conf", "color"):
		v[key] = np.ascontiguousarray(v[key][::2, ::2])
	v["K"] = S @ v["K"]
	_assert_same(views, nMinViewsFuse=2)
	stats = FuseRoundStats()[torch.cuda.current_device()]
	assert any(r["shared"] > 0 for r in stats) and all(r["iterations"] >= 1 for r in stats)


def test_rejections_release_claims_and_zero_depths():
	views = _scene_views(80, 60, 6, 1e-2, 4, drop=0.2)
	ph, host = _assert_same(views, nMinViewsFuse=3)
	assert sum(int((h["depth"] != v["depth"]).sum()) for h, v in zip(host, views)) > 0


def test_equal_connection_scores():
	views = _scene_views(64, 48, 6, 2e-3, 5)
	for v in views:
		v["n_scene_neighbors"] = 3
	_assert_same(views, nMinViewsFuse=2)


def test_views_without_normal_conf_or_color_maps():
	views = _scene_views(64, 48, 5, 2e-3, 6, with_color=False)
	views[1]["normal"] = None
	views[2]["conf"] = None; views[4]["conf"] = None
	ph, _ = _assert_same(views, nMinViewsFuse=2)
	assert ph.normals is None and ph.colors is None


def test_image_without_depth_map_and_image_without_depth():
	views = _scene_views(64, 48, 5, 2e-3, 7)
	views[1]["depth"] = None
	views[4]["depth"][:] = 0
	_assert_same(views, nMinViewsFuse=2, bEstimateNormal=False)


def test_twelve_views_640x480():
	views = _scene_views(640, 480, 12, 2e-3, 8, n_nb=9)
	ph, _ = _assert_same(views, nMinViewsFuse=3)
	assert len(ph.points) > 100000


def test_bad_arguments_are_refused_and_leave_the_maps_untouched():
	views = _scene_views(32, 24, 3, 2e-3, 9)
	for bad in ([1, 1], [7]):
		dev = _to_device(views)
		dev[0]["neighbors"] = bad
		before = [d["depth"].clone() for d in dev]
		with pytest.raises(lib.B200MVSError, match="status 1"):
			FuseDepthMaps(dev)
		assert all(torch.equal(b, d["depth"]) for b, d in zip(before, dev))
	dev = _to_device(views)
	dev.append(dict(depth=torch.ones((1, 70000), dtype=torch.float32, device="cuda"), K=np.eye(3), R=np.eye(3), C=np.zeros(3),
		neighbors=[0]))
	before = [d["depth"].clone() for d in dev]
	with pytest.raises(lib.B200MVSError, match="status 1"):
		FuseDepthMaps(dev)
	assert all(torch.equal(b, d["depth"]) for b, d in zip(before, dev))
