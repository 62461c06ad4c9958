"""Known answers of the point-cloud oracle (oracle/point_cloud_oracle.py), which the GPU tests of MergeDepthMaps,
EstimatePointColors and EstimatePointNormals compare against: merge counts and positions, a hand-computed bilinear colour,
white outside the border or without an image, brute-force k-NN with ties to the lower index, and PCA normals of a plane and a
sphere turned towards the first view's camera."""
import numpy as np

from oracle import point_cloud_oracle as PO

K = np.array([[2.0, 0, 1.5], [0, 2.0, 1.0], [0, 0, 1]])


def test_merge_counts_and_positions_on_a_4x3_map():
	d = np.array([[0, 1, 2, 0], [4, 0, 0, 8], [0, 0, 3, 0]], np.float32)
	n = np.zeros((3, 4, 3), np.float32); n[..., 2] = -1
	col = np.arange(36, dtype=np.uint8).reshape(3, 4, 3)
	views = [dict(depth=None), dict(depth=d, normal=n, color=col, K=K, R=np.eye(3), C=np.array([1.0, 2.0, 3.0]))]
	m = PO.merge_depth_maps(views)
	assert m["nDepths"] == 5 and m["views"].tolist() == [1]*5
	assert m["projs"].tolist() == [[1, 0], [2, 0], [0, 1], [3, 1], [2, 2]]
	# pixel (3, 1), depth 8: ((3 - 1.5)*8/2, (1 - 1)*8/2, 8) + C
	assert np.array_equal(m["points"][3], np.array([7.0, 2.0, 11.0], np.float32))
	assert np.array_equal(m["colors"][0], col[0, 1]) and np.array_equal(m["normals"][4], [0, 0, -1])


def test_colour_truncates_every_product():
	img = np.zeros((4, 4, 3), np.uint8)
	img[1, 1] = 101; img[1, 2] = 203; img[2, 1] = 7; img[2, 2] = 255
	x, y = np.float32(1.3), np.float32(1.6)
	got = PO.sample(img, np.array([x]), np.array([y]))[0]
	fx = np.float32(x - np.float32(1)); fy = np.float32(y - np.float32(1))
	t = lambda p, v: int(np.float32(v)*np.float32(p))
	top = (t(101, np.float32(1)-fx) + t(203, fx)) & 255
	bot = (t(7, np.float32(1)-fx) + t(255, fx)) & 255
	want = (t(top, np.float32(1)-fy) + t(bot, fy)) & 255
	assert got.tolist() == [want]*3
	exact = (101*(1-0.3) + 203*0.3)*(1-0.6) + (7*(1-0.3) + 255*0.3)*0.6
	assert want != int(round(exact))          # rounding would give another colour here


def test_colour_outside_the_border_and_without_an_image_is_white():
	img = np.full((6, 8, 3), 9, np.uint8)
	cam = dict(K=np.array([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1]]), R=np.eye(3), C=np.zeros(3))
	# projections (x, y) = (X/Z, Y/Z): on the border lines x = 1 and x = W - 2 inside, x = 0.5 and x = W - 1.5 outside
	pts = np.array([[1, 1, 1], [6, 4, 1], [0.5, 2, 1], [6.5, 2, 1], [2, 2, 1]], np.float32)
	off = np.arange(6, dtype=np.uint32)
	ids = np.array([0, 0, 0, 0, 1], np.uint32)
	c = PO.estimate_point_colors(pts, off, ids, [dict(cam, color=img), dict(cam, color=None)])
	assert c.tolist() == [[9]*3, [9]*3, [255]*3, [255]*3, [255]*3]


def _brute(X, k):
	X = X.astype(np.float64)
	out = []
	for q in X:
		d = ((X[:, 0]-q[0])*(X[:, 0]-q[0]) + (X[:, 1]-q[1])*(X[:, 1]-q[1])) + (X[:, 2]-q[2])*(X[:, 2]-q[2])
		out.append(sorted(range(len(X)), key=lambda j: (d[j], j))[:k])
	return np.array(out)


def test_knn_equals_an_independent_sort_with_ties_to_the_lower_index():
	rng = np.random.RandomState(0)
	X = rng.rand(300, 3).astype(np.float32)
	X[100:110] = X[5]                            # exact duplicates of point 5
	got = PO.knn(X, 16, chunk=64)
	assert np.array_equal(got, _brute(X, 16))
	assert got[107].tolist()[:11] == [5] + list(range(100, 110))
	assert PO.knn(X[:7], 16).shape == (7, 7)


def _normals(X, C, k=16):
	n = len(X)
	off = np.arange(n+1, dtype=np.uint32)
	return PO.estimate_point_normals(X, off, np.zeros(n, np.uint32), C[None], PO.knn(X, k))


def test_normals_of_a_tilted_plane_and_a_sphere():
	rng = np.random.RandomState(1)
	uv = rng.rand(2000, 2)*4 - 2
	nrm = np.array([1.0, 2.0, 3.0])/np.sqrt(14.0)
	a = np.cross(nrm, [1, 0, 0]); a /= np.linalg.norm(a); b = np.cross(nrm, a)
	X = (uv[:, :1]*a + uv[:, 1:]*b + 10).astype(np.float32)
	n, w = _normals(X, np.array([50.0, 50, 50]))
	assert np.all(np.abs(n.astype(np.float64) @ nrm - 1) < 1e-5)   # turned towards the camera
	n2, _ = _normals(X, np.array([-50.0, -50, -50]))
	assert np.array_equal(n2, -n)
	s = rng.randn(4000, 3); s /= np.linalg.norm(s, axis=1, keepdims=True)
	S = (s*5).astype(np.float32)
	n, w = _normals(S, np.zeros(3))
	assert np.all(np.einsum("ij,ij->i", n.astype(np.float64), -s) > 0.99)  # inward, towards the centre camera
