"""The point-cloud calls (openmvs_b200/point_cloud.py) check every buffer before it reaches the C-ABI: a map or cloud of the
wrong type, shape or memory is refused with a ValueError naming the call and the argument (no GPU needed)."""
import numpy as np
import pytest

from openmvs_b200.depth_estimator import EstimatePointColors, EstimatePointNormals, MergeDepthMaps, PointCloud

CAM = dict(K=np.eye(3), R=np.eye(3), C=np.zeros(3))


@pytest.mark.parametrize("key,bad", [("depth", np.zeros((4, 5, 2), np.float32)), ("normal", np.zeros((4, 5), np.float32)),
	("color", np.zeros((4, 5, 4), np.uint8))])
def test_merge_refuses_a_bad_map(key, bad):
	v = dict(CAM, depth=np.zeros((4, 5), np.float32), normal=np.zeros((4, 5, 3), np.float32), color=np.zeros((4, 5, 3), np.uint8))
	v[key] = bad
	with pytest.raises(ValueError, match="MergeDepthMaps: views\\[0\\].%s" % key):
		MergeDepthMaps([v])


def test_colours_and_normals_refuse_a_bad_cloud():
	pv = [np.array([0], np.uint32)]*3
	with pytest.raises(ValueError, match="EstimatePointNormals: pointcloud.points"):
		EstimatePointNormals([CAM], PointCloud(np.zeros((3, 2), np.float32), pv, None))
	with pytest.raises(ValueError, match="EstimatePointColors: views\\[0\\].color"):
		EstimatePointColors([dict(CAM, color=np.zeros((4, 5), np.uint8))], PointCloud(np.zeros((3, 3), np.float32), pv, None))
