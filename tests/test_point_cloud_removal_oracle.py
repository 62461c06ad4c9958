"""The point-cloud removals on the CPU: the removal order of the oracle (the chain formulation the device resolves) against the
host b200mvs_pointcloud_remove_order and a literal restatement of the RFOREACH / cList::RemoveAt loop; the ROI test on box
faces; EstimateROI on hand-built camera rigs, host form against the oracle."""
import ctypes as C

import numpy as np
import pytest

from oracle import removal_oracle as R


def literal_order(remove):
	"""RFOREACH(i, points) if (remove[i]) RemovePoint(i), with RemoveAt moving the last element into slot i"""
	a = list(range(len(remove)))
	for i in reversed(range(len(remove))):
		if remove[i]:
			a[i] = a[-1]
			a.pop()
	return a


def host_order(remove):
	from openmvs_b200 import lib as L
	lib = L.load()
	remove = np.ascontiguousarray(remove, np.uint8)
	n = len(remove)
	order = np.zeros(max(n, 1), np.uint32)
	kept = C.c_uint64()
	assert lib.b200mvs_pointcloud_remove_order(remove.ctypes.data if n else None, n, order.ctypes.data, C.byref(kept)) == 0
	return [int(v) for v in order[:kept.value]]


def adversarial(n):
	"""all, none, a prefix, a suffix, alternating slots, and long chains ([1,1,1,0,0] scaled up)"""
	k = n // 2
	yield np.ones(n, bool)
	yield np.zeros(n, bool)
	yield np.arange(n) < k
	yield np.arange(n) >= k
	yield np.arange(n) % 2 == 0
	yield np.arange(n) % 2 == 1
	yield np.arange(n) < (3*n)//5


def masks():
	rng = np.random.default_rng(7)
	for _ in range(4000):
		n = int(rng.integers(0, 65))
		yield rng.random(n) < rng.random()
	for n in (0, 1, 2, 3, 5, 17, 64, 1000):
		yield from adversarial(n)


def test_removal_order_matches_the_loop_and_the_host_function():
	for m in masks():
		want = literal_order(m)
		assert list(R.remove_order(m)) == want, m.astype(int)
		assert host_order(m) == want, m.astype(int)
	assert literal_order([1, 1, 1, 0, 0]) == [4, 3]


def rotated_box(seed):
	rng = np.random.default_rng(seed)
	q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
	return q.astype(np.float32), rng.normal(size=3).astype(np.float32), (rng.random(3) + 0.5).astype(np.float32)


def face_points(rot, pos, ext, border):
	"""points whose box coordinate is exactly on each face of the box with its border, and one ulp to either side, as the float
	arithmetic of the test computes it: searched along the face normal from a point of the face"""
	e = R.roi_extent(ext, border)
	pts = []
	rng = np.random.default_rng(1)
	for a in range(3):
		for sgn in (-1, 1):
			local = (rng.random(3).astype(np.float32) - 0.5) * e
			for t in np.linspace(-3, 3, 61):
				local[a] = sgn*e[a]
				X = (pos.astype(np.float64) + rot.T.astype(np.float64) @ local.astype(np.float64)).astype(np.float32)
				X = X + np.float32(t)*np.float32(1e-7)*rot[a]*sgn
				pts.append(X.astype(np.float32))
	P = np.array(pts, np.float32)
	# one ulp to either side of every coordinate of every point
	return np.concatenate([P, np.nextafter(P, np.float32(np.inf)), np.nextafter(P, np.float32(-np.inf))])


@pytest.mark.parametrize("border", [0.0, 1.25, -0.05])
def test_roi_mask_on_box_faces(border):
	from openmvs_b200 import lib as L
	lib = L.load()
	for seed in range(4):
		rot, pos, ext = rotated_box(seed)
		P = np.ascontiguousarray(face_points(rot, pos, ext, border))
		want = R.outside_obb(P, rot, pos, ext, border)
		assert 0 < want.sum() < len(want)   # the set straddles the faces
		got = np.zeros(len(P), np.uint8)
		box = [np.ascontiguousarray(a, np.float32).ravel() for a in (rot, pos, ext)]
		assert lib.b200mvs_point_cloud_outside_obb(P.ctypes.data, len(P), *(b.ctypes.data for b in box), border, got.ctypes.data) == 0
		assert np.array_equal(got, want)


def test_min_views_mask():
	from openmvs_b200 import lib as L
	lib = L.load()
	off = np.array([0, 0, 1, 3, 6, 6, 8], np.uint32)
	for th in range(5):
		got = np.zeros(6, np.uint8)
		assert lib.b200mvs_point_cloud_min_views(off.ctypes.data, 6, th, got.ctypes.data) == 0
		assert np.array_equal(got, (np.diff(off) < th).astype(np.uint8))


def look_at(C_, target):
	z = np.asarray(target, np.float64) - C_
	z /= np.linalg.norm(z)
	x = np.cross([0.0, 1.0, 0.0], z)
	x /= np.linalg.norm(x)
	return np.stack([x, np.cross(z, x), z])


def ring(n, radius=4.0, height=1.0, target=(0.0, 0.0, 0.0)):
	"""n cameras on a ring looking at target: (K, R, C, valid) per camera"""
	K = np.array([[500.0, 0, 320], [0, 500.0, 240], [0, 0, 1]])
	cams = []
	for i in range(n):
		a = 2*np.pi*i/n + 0.1
		C_ = np.array([radius*np.cos(a), height, radius*np.sin(a)])
		cams.append((K, look_at(C_, target), C_, True))
	return cams


def cloud(n, cams, seed=0):
	rng = np.random.default_rng(seed)
	pts = rng.normal(scale=[1.0, 0.5, 1.0], size=(n, 3)).astype(np.float32)
	pts[:5] *= 40   # far points
	lists = [np.sort(rng.choice(len(cams), size=int(rng.integers(1, min(4, len(cams)+1))), replace=False)).astype(np.uint32) for _ in range(n)]
	off = np.concatenate([[0], np.cumsum([len(v) for v in lists])]).astype(np.uint32)
	return pts, off, np.concatenate(lists).astype(np.uint32)


def host_roi(pts, off, ids, cams, mode=2, scale=1.1):
	from openmvs_b200 import lib as L
	lib = L.load()
	arr = (L.FuseView*len(cams))()
	for i, (K, Rm, C_, valid) in enumerate(cams):
		arr[i].K[:] = list(np.ravel(K)); arr[i].R[:] = list(np.ravel(Rm)); arr[i].C[:] = list(np.ravel(C_))
		arr[i].width = arr[i].height = int(valid)
	rot, pos, ext = np.zeros(9, np.float32), np.zeros(3, np.float32), np.zeros(3, np.float32)
	bounded = C.c_int(-1)
	pts = np.ascontiguousarray(pts, np.float32)
	assert lib.b200mvs_estimate_roi(None, pts.ctypes.data, len(off)-1, off.ctypes.data, ids.ctypes.data, arr, len(cams), mode,
		scale, rot.ctypes.data, pos.ctypes.data, ext.ctypes.data, C.byref(bounded)) == 0
	return (rot.reshape(3, 3), pos, ext) if bounded.value else None


def same_roi(a, b):
	if a is None or b is None:
		return a is None and b is None
	return all(np.array_equal(np.asarray(x, np.float32).ravel(), np.asarray(y, np.float32).ravel()) for x, y in zip(a, b))


@pytest.mark.parametrize("n", [5, 6])   # an odd and an even camera count: the median rule
def test_estimate_roi_rigs(n):
	cams = ring(n)
	pts, off, ids = cloud(400, cams)
	want = R.estimate_roi(pts, off, ids, cams, 2, 1.1)
	assert want is not None
	assert same_roi(host_roi(pts, off, ids, cams, 2, 1.1), want)
	# an image without a pose is skipped
	cams2 = cams + [(cams[0][0], cams[0][1], np.array([50.0, 0, 0]), False)]
	assert same_roi(host_roi(pts, off, ids, cams2, 2, 1.3), R.estimate_roi(pts, off, ids, cams2, 2, 1.3))


def test_estimate_roi_unbounded():
	cams = ring(5)
	pts, off, ids = cloud(200, cams)
	# mode 0, fewer than 3 cameras (or valid ones)
	assert R.estimate_roi(pts, off, ids, cams, 0) is None and host_roi(pts, off, ids, cams, 0) is None
	two = ring(2)
	p2, o2, i2 = cloud(50, two)
	assert R.estimate_roi(p2, o2, i2, two) is None and host_roi(p2, o2, i2, two) is None
	few = [c if i < 2 else c[:3] + (False,) for i, c in enumerate(cams)]
	assert R.estimate_roi(pts, off, ids, few) is None and host_roi(pts, off, ids, few) is None
	# mode 2: unbalanced directions (all cameras on one side, looking the same way)
	K = cams[0][0]
	fwd = [(K, np.eye(3), np.array([x, 0.0, -5.0]), True) for x in (-1.0, 0.0, 1.0, 2.0)]
	pf, of, idf = cloud(100, fwd)
	assert R.estimate_roi(pf, of, idf, fwd, 2) is None and host_roi(pf, of, idf, fwd, 2) is None
	# mode 1 accepts the same rig
	assert same_roi(host_roi(pf, of, idf, fwd, 1), R.estimate_roi(pf, of, idf, fwd, 1))
	assert R.estimate_roi(pf, of, idf, fwd, 1) is not None
	# mode 2: a camera not facing the scene centre
	away = list(cams)
	K0, R0, C0, _ = away[0]
	away[0] = (K0, -R0, C0, True)
	assert R.estimate_roi(pts, off, ids, away, 2) is None and host_roi(pts, off, ids, away, 2) is None
	assert same_roi(host_roi(pts, off, ids, away, 1), R.estimate_roi(pts, off, ids, away, 1))
