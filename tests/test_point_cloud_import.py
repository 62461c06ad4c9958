"""The point-cloud calls import on their own and through depth_estimator, in either order, in a fresh interpreter (no GPU needed:
importing loads no library)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("code", [
	"import openmvs_b200.point_cloud",
	"from openmvs_b200.point_cloud import MergeDepthMaps, EstimatePointColors, EstimatePointNormals, PointKNN",
	"from openmvs_b200.depth_estimator import MergeDepthMaps, EstimatePointColors, EstimatePointNormals, PointKNN",
	"import openmvs_b200.point_cloud as P, openmvs_b200.depth_estimator as D; assert D.MergeDepthMaps is P.MergeDepthMaps",
])
def test_import_in_a_fresh_interpreter(code):
	env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
	subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, env=env, check=True, timeout=300)
