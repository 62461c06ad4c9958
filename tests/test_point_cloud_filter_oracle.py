"""Scene::PointCloudFilter without a GPU: hand-computed counts of the exhaustive CPU restatement
(oracle/visibility_oracle.cpp) for points on and around one ray, the library's removal order
(b200mvs_pointcloud_remove_order) against the reference's literal loop, and the argument checks of the binding."""
import numpy as np
import pytest

from openmvs_b200.depth_estimator import PointCloud, PointCloudFilter, PointCloudVisibility
from oracle import point_cloud_oracle as VO

K = np.array([[500.0, 0, 320], [0, 500, 240], [0, 0, 1]])
# camera 0 at the origin looking down +z; camera 1 at (0, 10, 10) looking down -y at the first point, so that its cone (and that
# of the point seen by it alone) holds no other point
CAMS = [dict(K=K, R=np.eye(3), C=np.zeros(3), width=640, height=480),
	dict(K=K, R=np.array([[1.0, 0, 0], [0, 0, -1], [0, 1, 0]]), C=np.array([0.0, 10, 10]), width=640, height=480)]
ANGLE = np.float32(2*np.arctan(640/1000)/640)   # one pixel of camera 0: float(ComputeFOV(0)/width)


def test_known_answers_on_one_ray():
	off_axis = np.float32(5*np.tan(0.5*ANGLE))    # half the cone's angle from the axis, 5 units in front of X
	pts = np.array([
		[0, 0, 10],         # X: seen by both cameras, so its cones weigh 2
		[0, 0, 5],          # in front of X inside the cone: -2
		[0, 0, 10.15],      # 1.5 % behind X: + its own view count, 1
		[0, 0, 10.05],      # 0.5 % behind X: depth-similar, 0
		[0, 0, 10.3],       # beyond 1.02 |X - C|: FRONT, 0
		[0.1, 0, 7],        # 0.8 degrees off the axis, far outside the one-pixel cone: 0
		[0, 0, -3],         # behind the camera: BACK, 0
		[0, 0, 5e-5],       # |t| < 1e-4: PLANAR, 0
		[off_axis, 0, 5],   # in front of X at half the cone's angle: -2
	], np.float32)
	views = [[0, 1], [], [1], [], [], [], [], [], []]
	want = np.array([0, -2, 1, 0, 0, 0, 0, 0, -2], np.int32)
	assert np.array_equal(VO.visibility(pts, views, CAMS, threads=1), want)
	assert np.array_equal(VO.visibility(pts, views, CAMS, threads=3), want)
	# the cone's angle is exclusive of its surface and the similarity threshold of 1 % exclusive of equality: a point just
	# outside the cone (1.5 times its angle) counts nothing
	outside = pts.copy()
	outside[8, 0] = np.float32(5*np.tan(1.5*ANGLE))
	assert VO.visibility(outside, views, CAMS, threads=1)[8] == 0
	# with thRemove = 0 the two points in front of X and every point without counts go
	order = VO.filter_order(want, 0)
	assert list(order) == [2]


def _literal(remove):
	return VO.filter_order(np.where(remove, 0, 1).astype(np.int32), 0)


def _library(remove):
	from openmvs_b200 import lib
	import ctypes as C
	L = lib.load()
	remove = np.ascontiguousarray(remove, np.uint8)
	order = np.zeros(max(len(remove), 1), np.uint32)
	kept = C.c_uint64()
	assert L.b200mvs_pointcloud_remove_order(remove.ctypes.data, len(remove), order.ctypes.data, C.byref(kept)) == 0
	return order[:kept.value]


@pytest.mark.parametrize("n", [0, 1, 2, 7, 100, 1001])
def test_remove_order_equals_the_literal_loop(n):
	rng = np.random.RandomState(n)
	masks = [np.zeros(n, bool), np.ones(n, bool), np.arange(n) == n-1, np.arange(n) == 0]
	masks += [rng.rand(n) < p for p in (0.1, 0.5, 0.9)]
	for m in masks:
		got, want = _library(m), _literal(m)
		assert np.array_equal(got, want), m
		assert len(got) == n - int(m.sum()) and not m[got].any()


def test_remove_order_refuses_null_buffers():
	from openmvs_b200 import lib
	import ctypes as C
	L = lib.load()
	kept = C.c_uint64()
	assert L.b200mvs_pointcloud_remove_order(None, 3, None, C.byref(kept)) != 0
	assert L.b200mvs_pointcloud_remove_order(None, 0, None, None) != 0
	assert L.b200mvs_pointcloud_remove_order(None, 0, None, C.byref(kept)) == 0 and kept.value == 0


def _cloud(n=3):
	return PointCloud(np.zeros((n, 3), np.float32), [np.array([0], np.uint32)]*n, None)


def test_visibility_refuses_bad_arguments():
	with pytest.raises(ValueError, match="PointCloudVisibility: pointcloud.points"):
		PointCloudVisibility(CAMS, PointCloud(np.zeros((3, 2), np.float32), [np.array([0], np.uint32)]*3, None))
	with pytest.raises(ValueError, match="PointCloudVisibility: pointcloud.points must have one row per view list"):
		PointCloudVisibility(CAMS, PointCloud(np.zeros((2, 3), np.float32), [np.array([0], np.uint32)]*3, None))
	with pytest.raises(ValueError, match="PointCloudVisibility: views\\[1\\] needs width and height"):
		PointCloudVisibility([CAMS[0], dict(K=K, R=np.eye(3), C=np.zeros(3))], _cloud())
	with pytest.raises(ValueError, match="PointCloudVisibility: views\\[0\\] width and height"):
		PointCloudVisibility([dict(CAMS[0], width=0)], _cloud())
	with pytest.raises(ValueError, match="PointCloudVisibility: views\\[0\\] width and height"):
		PointCloudVisibility([dict(CAMS[0], width=640.5)], _cloud())


def test_filter_refuses_bad_arguments():
	for th in (0.5, "0", None, True, 2**31):
		with pytest.raises(ValueError, match="PointCloudFilter: thRemove"):
			PointCloudFilter(CAMS, _cloud(), th)
	with pytest.raises(ValueError, match="PointCloudFilter: pointcloud.points"):
		PointCloudFilter(CAMS, PointCloud(np.zeros((3, 3, 1), np.float32), [np.array([0], np.uint32)]*3, None), 0)
