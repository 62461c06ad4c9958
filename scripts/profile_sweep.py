"""Single-view 1080p run (one reference view, 9 neighbours) for ncu captures and schedule comparisons: prints the per-sweep
kernel times of the engine's schedule, from random initialisation and continuing from the converged state.
usage: profile_sweep.py [iters] [far] [skip] [sweepsPerIter] [unused] [evalCap]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from openmvs_b200 import synth
from openmvs_b200.depth_estimator import OPTDENSE, Camera, ViewData, DepthData, PatchMatchB200

iters = int(sys.argv[1]) if len(sys.argv) > 1 else 6
OPTDENSE.nPropagationFar = int(sys.argv[2]) if len(sys.argv) > 2 else 2
OPTDENSE.bSkipUnchanged = int(sys.argv[3]) if len(sys.argv) > 3 else 1
OPTDENSE.nSweepsPerIter = int(sys.argv[4]) if len(sys.argv) > 4 else 0
if len(sys.argv) > 6: OPTDENSE.nEvalCap = int(sys.argv[6])
dev = torch.device("cuda:0")
sc = synth.make_scene(1920, 1080, 12, step_deg=4.0, device=dev)
r = 5
views = [sc.views[r]]+[sc.views[i] for i in sc.neighbors(r, 9)]
imgs = [ViewData(torch.from_numpy(v.image).to(dev), Camera(v.K, v.R, v.C)) for v in views]
OPTDENSE.nSubResolutionLevels = 0; OPTDENSE.nEstimationGeometricIters = 0; OPTDENSE.nEstimationIters = iters
pm = PatchMatchB200(0)
gt = sc.views[r].depth_gt; gtn = sc.views[r].normal_gt
for tag in ("random init", "warm, random init", "continued"):
	dd = DepthData(imgs, sc.dmin, sc.dmax) if tag != "continued" else dd
	pm.EstimateDepthMap(dd)
	gd = dd.depthMap.cpu().numpy(); gn = dd.normalMap.cpu().numpy(); m = gd > 0
	ang = np.degrees(np.arccos(np.clip((gn*gtn).sum(-1), -1, 1)))[m]
	print("%-18s cap %d schedule %s far %d skip %d | device ms %.2f launches %d | sweep launches %d avg %.3f ms | valid %.4f gt<1e-3 %.4f med ang %.2f" % (
		tag, OPTDENSE.nEvalCap, OPTDENSE.schedule(), OPTDENSE.nPropagationFar, OPTDENSE.bSkipUnchanged, pm.stats.ms_device, pm.stats.kernel_launches,
		pm.stats.sweep_launches, pm.stats.ms_sweep_kernels/max(1, pm.stats.sweep_launches), m.mean(),
		(np.abs(gd-gt)[m]/gt[m] < 1e-3).mean(), np.median(ang)), flush=True)
