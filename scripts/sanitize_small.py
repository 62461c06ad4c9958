"""Small PatchMatch (photometric, multi-scale, geometric) + SGM + post-processing runs for compute-sanitizer.
SANITIZE_ONLY=post runs the post-processing part alone."""
import copy, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from openmvs_b200 import synth
from openmvs_b200.depth_estimator import OPTDENSE, Camera, ViewData, DepthData, PatchMatchB200, SemiGlobalMatcher
sc = synth.make_scene(203, 151, 3, step_deg=5.0, cols=3)
views = [sc.views[1], sc.views[0], sc.views[2]]
OPTDENSE.nEstimationIters = 1; OPTDENSE.nEstimationGeometricIters = 1
ONLY = os.environ.get("SANITIZE_ONLY", "")
pm = PatchMatchB200(0)
if ONLY:
	pm.Release()
if ONLY == "":
	for levels in (0, 1):
		OPTDENSE.nSubResolutionLevels = levels
		dd = DepthData([ViewData(np.ascontiguousarray(v.image), Camera(v.K, v.R, v.C)) for v in views], sc.dmin, sc.dmax)
		pm.EstimateDepthMap(dd)
		print("pm levels", levels, "valid", (dd.depthMap > 0).mean(), "tma", pm.stats.tma_active)
	OPTDENSE.nSubResolutionLevels = 0
	g = DepthData([ViewData(np.ascontiguousarray(v.image), Camera(v.K, v.R, v.C), depthMap=(v.depth_gt if i else None), cameraDepthMap=Camera(v.K, v.R, v.C)) for i, v in enumerate(views)],
		sc.dmin, sc.dmax, depthMap=dd.depthMap.copy(), normalMap=dd.normalMap.copy())
	pm.Init(True); pm.EstimateDepthMap(g, 0); pm.Release()
	print("geo valid", (g.depthMap > 0).mean())
	lg, lc, rg, d = synth.make_stereo_pair(131, 77)
	rng = np.random.RandomState(0)
	lo = rng.randint(-3, 3, (71, 125)); hi = lo+rng.randint(1, 40, (71, 125))
	px, n = synth.sgm_pixel_map(131, 77, lo, hi, rng.rand(71, 125) < 0.1)
	m = SemiGlobalMatcher(); disp, cost = m.Match(lg, lc, rg, px, n); m.Release()
	print("sgm ok", disp.shape, int((disp != 32767).sum()))
if ONLY in ("", "sgm"):
	# uniform 16-byte aligned ranges: the bulk-copy ring aggregation kernel (mbarrier + cp.async.bulk)
	lg, lc, rg, d = synth.make_stereo_pair(150, 90)
	for num in (32, 144, 64, 128):   # ring kernel; wave-front aggregation + tensor-core cost kernel
		px, n = synth.sgm_pixel_map(150, 90, -8, -8+num)
		m = SemiGlobalMatcher(); disp, cost = m.Match(lg, lc, rg, px, n); m.Release()
		print("sgm ring num", num, "ok", int((disp != 32767).sum()))
if ONLY == "sgm":
	sys.exit(0)
# depth-map post-processing: filter (both branches), speckles, gaps
from openmvs_b200.depth_estimator import DepthMapsData
maps = synth.make_noisy_dmaps(sc)
def _dd(i, conf=True):
	v = sc.views[i]
	return DepthData([ViewData(None, Camera(v.K, v.R, v.C))], sc.dmin, sc.dmax, depthMap=maps[i][0].copy(), confMap=maps[i][1].copy() if conf else None)
dm = DepthMapsData([], 0, nCalibratedImages=3)
for adjust in (True, False):
	fd, fc = dm.FilterDepthMap(_dd(1), [_dd(0, adjust), _dd(2, adjust)], adjust)
	print("filter adjust", adjust, "kept", (fd > 0).mean())
p = DepthData([], 0, 0, fd.copy(), np.ascontiguousarray(sc.views[1].normal_gt*(fd > 0)[..., None]), fc.copy())
dm.RemoveSmallSegments(p); print("segments kept", (p.depthMap > 0).mean())
dm.GapInterpolation(p); print("gaps filled to", (p.depthMap > 0).mean())
dm.pmCUDA.Release()
# the point-cloud tail: merge (both forms), colours and normals (host-buffer and device forms), k-NN
from openmvs_b200.depth_estimator import EstimatePointColors, EstimatePointNormals, MergeDepthMaps, PointKNN
pv = [dict(depth=maps[i][0].copy(), normal=np.ascontiguousarray(sc.views[i].normal_gt), K=sc.views[i].K, R=sc.views[i].R, C=sc.views[i].C,
	color=(np.clip(sc.views[i].image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1)) for i in range(3)]
MergeDepthMaps(pv)
pc = MergeDepthMaps([dict(v, **{k: torch.from_numpy(np.ascontiguousarray(v[k])).cuda() for k in ("depth", "normal", "color")}) for v in pv])
EstimatePointColors(pv, pc); EstimatePointNormals(pv, pc)
pc.points = torch.from_numpy(pc.points).cuda()
EstimatePointColors([dict(v, color=torch.from_numpy(v["color"]).cuda()) for v in pv], pc); EstimatePointNormals(pv, pc, 32)
print("point cloud", len(pc.points), "knn", tuple(PointKNN(pc.points, 16).shape))
# PointCloudFilter: the visibility counts (host-buffer and device forms, binned and exhaustive paths) and the filter
from openmvs_b200.depth_estimator import FuseDepthMaps, PointCloudFilter, PointCloudVisibility
fv = [dict(v, conf=None, neighbors=[j for j in range(3) if j != i], n_scene_neighbors=2) for i, v in enumerate(copy.deepcopy(pv))]
fc = FuseDepthMaps(fv)
vh = PointCloudVisibility(pv, fc)
fc.points = torch.from_numpy(fc.points).cuda()
vd = PointCloudVisibility(pv, fc).cpu().numpy()
away = [dict(v, R=-np.asarray(v["R"])) for v in pv]   # every query of every view takes the exhaustive path
ve = PointCloudVisibility(away, fc).cpu().numpy()
print("visibility", len(vh), "host == device", bool((vh == vd).all()), "exhaustive == binned", bool((ve == vd).all()),
	"kept", len(PointCloudFilter(pv, fc, 0).points))
