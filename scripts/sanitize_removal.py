"""Small runs of the point-cloud removal kernels (ROI and minimum-views masks, removal order, compaction, EstimateROI), host and
device forms, for compute-sanitizer: python scripts/sanitize_removal.py."""
import copy, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from openmvs_b200 import synth
from openmvs_b200.depth_estimator import EstimateROI, FuseDepthMaps, PointCloud, RemoveMinViews, RemovePointsOutside
sc = synth.make_scene(131, 97, 4, step_deg=5.0)
rng = np.random.RandomState(0)
views = [dict(depth=(v.depth_gt*(rng.rand(97, 131) > 0.1)).astype(np.float32), normal=v.normal_gt.astype(np.float32), conf=None,
	color=(np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1), K=v.K, R=v.R, C=v.C,
	neighbors=[j for j in range(4) if j != i], n_scene_neighbors=3) for i, v in enumerate(sc.views)]
host = FuseDepthMaps(copy.deepcopy(views))
dev = PointCloud(torch.from_numpy(host.points).cuda(), host.pointViews, host.pointWeights, torch.from_numpy(host.colors).cuda(),
	torch.from_numpy(host.normals).cuda(), host.projs)
images = [dict(K=v["K"], R=v["R"], C=v["C"]) for v in views]
for pc in (host, dev):
	obb = EstimateROI(images, pc, 1)
	for border in (0.0, 0.7, -0.01):
		cut = RemoveMinViews(RemovePointsOutside(pc, obb, border), 3)
		print(type(pc.points).__module__, "border", border, "kept", len(cut.pointViews), "of", len(pc.pointViews))
empty = PointCloud(torch.zeros((0, 3), device="cuda"), [], None)
print("empty", len(RemoveMinViews(empty, 2).pointViews), EstimateROI(images, empty))
torch.cuda.synchronize()
