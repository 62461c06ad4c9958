"""Hierarchical (tSGM) matching of bench.py's 1920x1080 SGM pair against the fixed-range pair, in one process.

  python scripts/profile_tsgm.py [--iters N] [--min-resolution R] [--out FILE]

Reports, as one JSON object: ms per hierarchical pair and per fixed-range MatchPairDevice(-128, 0) pair (CUDA events, the two
alternated after warm-up), the kernel time per level and per stage (pyramid, range maps, matches, filters) from one torch.profiler
run, numCosts per level, the fraction of interior pixels within 1 px of the ground truth for both, and the card name and power limit
(read-only nvidia-smi query)."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmvs_b200 import synth  # noqa: E402
from openmvs_b200.depth_estimator import SemiGlobalMatcher  # noqa: E402

PYRAMID = ("resize_area_kernel", "tsgm_area_u8", "tsgm_upscale_mask", "resize_nearest_u8")
RANGES = ("tsgm_range", "tsgm_expand", "tsgm_offsets", "tsgm_flip", "DeviceScan", "tsgm_fill", "tsgm_minmax", "tsgm_dense_map")
FILTERS = ("sgm_cross_check", "tsgm_speckle", "tsgm_extract_mask", "sgm_refine")


def stage_of(name):
	for stage, keys in (("pyramid", PYRAMID), ("range_maps", RANGES), ("filters", FILTERS)):
		if any(k in name for k in keys):
			return stage
	return "matches" if "sgm_" in name or "Memset" in name or "memset" in name else "other"


def gpu_info():
	try:
		out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
		name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
		return name, power
	except Exception as e:  # noqa: BLE001
		return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--iters", type=int, default=10)
	ap.add_argument("--min-resolution", type=int, default=320)
	ap.add_argument("--out", default=None)
	a = ap.parse_args()
	w, h = 1920, 1080
	lg, lc, rg, d, rc = synth.make_stereo_pair(w, h, d0=40.0, amp=25.0, right_color=True)
	dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
	L, LC, R, RC = dev(lg), dev(lc), dev(rg), dev(rc)
	m = SemiGlobalMatcher()
	hier = lambda: m.MatchPairHierarchicalDevice(L, LC, R, RC, minResolution=a.min_resolution)
	fixed = lambda: m.MatchPairDevice(L, LC, R, RC, -128, 0)
	for _ in range(2):
		hd, _, levels = hier()
		fd, _ = fixed()
	torch.cuda.synchronize()
	ms = {"hierarchical": [], "fixed": []}
	for _ in range(a.iters):
		for key, fn in (("hierarchical", hier), ("fixed", fixed)):
			e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
			e0.record(); fn(); e1.record(); torch.cuda.synchronize()
			ms[key].append(e0.elapsed_time(e1))
	# kernel time per level and stage; a level's range maps start with its FlipDirection launch, its pyramid and mask upscaling
	# run just before that
	from torch.profiler import profile, ProfilerActivity
	with profile(activities=[ProfilerActivity.CUDA]) as prof:
		hier(); torch.cuda.synchronize()
	evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA], key=lambda e: e.time_range.start)
	per = [{"pyramid": 0.0, "range_maps": 0.0, "matches": 0.0, "filters": 0.0, "other": 0.0} for _ in levels]
	flips = 0
	for e in evs:
		if "tsgm_flip_scatter" in e.name:
			flips += 1
		st = stage_of(e.name)
		lev = flips if st == "pyramid" else max(flips-1, 0)
		lev = min(lev, len(levels)-1)
		per[lev][st] += e.time_range.elapsed_us()/1000.0
	gt = d[3:-3, 3:-3]
	inner = (slice(8, -8), slice(8, -140))
	within = lambda disp: float((np.abs(disp.cpu().numpy()[inner]/4.0-gt[inner]) <= 1).mean())
	name, power = gpu_info()
	res = {
		"gpu": name, "power_limit": power, "size": [w, h], "minResolution": a.min_resolution, "iters": a.iters,
		"ms_hierarchical_pair": {"median": float(np.median(ms["hierarchical"])), "min": float(np.min(ms["hierarchical"]))},
		"ms_fixed_pair_-128_0": {"median": float(np.median(ms["fixed"])), "min": float(np.min(ms["fixed"]))},
		"levels": [{"size": l["size"], "numCosts": l["numCosts"], "kernel_ms": {k: round(v, 3) for k, v in p.items()}} for l, p in zip(levels, per)],
		"fixed_numCosts": 2*(w-6)*(h-6)*128,
		"within_1px_hierarchical": within(hd), "within_1px_fixed": within(fd),
	}
	s = json.dumps(res)
	print(s)
	if a.out:
		os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
		open(a.out, "w").write(s+"\n")
	m.Release()


if __name__ == "__main__":
	main()
