"""1080p SGM pair for profiling: per-stage device times of the default kernels and of the aggregation and cost variants
(b200mvs_debug.sgmAggregation / sgmCost), with an identity check against the register-pipelined kernel.
usage: profile_sgm.py [D]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from openmvs_b200 import synth
from openmvs_b200.depth_estimator import SemiGlobalMatcher
D = int(sys.argv[1]) if len(sys.argv) > 1 else 128
w, h = 1920, 1080
lg, lc, rg, d = synth.make_stereo_pair(w, h, d0=40.0, amp=25.0)
px, n = synth.sgm_pixel_map(w, h, 0, D)
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
args = (dev(lg), dev(lc), dev(rg), torch.from_numpy(px.view(np.uint8).reshape(-1, 16).copy()).cuda(), n)
m = SemiGlobalMatcher()
costs = torch.zeros(n, dtype=torch.uint8, device="cuda"); accums = torch.zeros(n, dtype=torch.int16, device="cuda")
ref = None
MODES = [("register pipeline", dict(sgmAggregation=2)), ("bulk-copy ring, 8 launches", dict(sgmAggregation=3)),
	("wave fronts (default)", dict()), ("SIMT cost kernel + wave fronts", dict(sgmCost=1))]
for name, dbg in MODES:
	m.SetDebug(**dbg)
	for rep in range(2):
		t = {}
		for stage_name, st in (("cost", 1), ("aggregate", 2), ("wta", 4), ("all", 7)):
			disp, cost = m.MatchDevice(*args, stages=st, costs=costs, accums=accums)
			t[stage_name] = m.stats.ms_device
	same = ""
	if ref is None:
		ref = (accums.clone(), disp.clone())
	else:
		same = "| identical to the register pipeline: %s" % (torch.equal(ref[0], accums) and torch.equal(ref[1], disp))
		if "sgmCost" in dbg:
			same = "| disparities equal to the tensor-core-cost run on %.4f of the pixels" % float((ref[1] == disp).float().mean())
	print("D=%d %-40s" % (D, name), " ".join("%s %.2f ms" % kv for kv in t.items()), "| %.2f G(px.d)/s" % (n/t["all"]/1e6), same, flush=True)
