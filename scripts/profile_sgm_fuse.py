"""Fusion-mode -2 at 1920x1080 with 4 and 8 pairs: SemiGlobalMatcher.Fuse on the device against the single-threaded oracle.

  python scripts/profile_sgm_fuse.py [--iters N] [--out FILE]

Reports, as one JSON object per pair count: ms per device Fuse call without and with normals (CUDA events, after warm-up), the kernel
time of each stage (key reset + splat, gather, cluster vote, normals) from one torch.profiler run, the oracle's time on the same inputs
(one run), whether the two agree bit for bit, and the card name and power limit (read-only nvidia-smi query)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmvs_b200.depth_estimator import SemiGlobalMatcher  # noqa: E402
from oracle import sgm_fuse as F  # noqa: E402

STAGES = (("splat", ("sgmf_project", "emset")), ("gather", ("sgmf_gather",)), ("vote", ("sgmf_fuse",)), ("normals", ("sgmf_normal",)))


def gpu_info():
	try:
		out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
		name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
		return name, power
	except Exception as e:  # noqa: BLE001
		return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def make_pairs(W, H, n, seed=1):
	"""n disparity maps of a smooth surface seen from pairs of different baselines (subpixelSteps 4, 10 % holes, costs), with Q's
	that shift the projections by up to 3 pixels"""
	rng = np.random.RandomState(seed)
	f = 0.9*W
	ys, xs = np.mgrid[0:H-6, 0:W-6].astype(np.float64)
	out = []
	for p in range(n):
		b = rng.uniform(0.2, 0.4)
		depth = 5.5 + 0.3*np.sin(xs/37.0+p)*np.cos(ys/23.0)
		d = np.rint(-f*b/depth*4 + rng.randint(-2, 3, depth.shape)).astype(np.int16)
		d[rng.rand(*d.shape) < 0.1] = 32767
		Q = np.array([[f, 0, 0, rng.uniform(-3, 3)*f], [0, f, 0, rng.uniform(-3, 3)*f], [0, 0, 0, f], [0, 0, 1.0/b, 0]])
		out.append((d, rng.randint(0, 4000, d.shape).astype(np.uint16), Q, 4))
	return out


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--iters", type=int, default=20)
	ap.add_argument("--out", default=None)
	a = ap.parse_args()
	W, H = 1920, 1080
	K = np.array([[0.9*W, 0, (W-1)/2.0], [0, 0.9*W, (H-1)/2.0], [0, 0, 1.0]])
	name, power = gpu_info()
	m = SemiGlobalMatcher()
	results = []
	for n in (4, 8):
		pairs = make_pairs(W, H, n)
		dev = [(torch.from_numpy(d).cuda(), torch.from_numpy(c).cuda(), Q, s) for d, c, Q, s in pairs]
		row = {"size": [W, H], "pairs": n}
		for key, k in (("ms_fuse", None), ("ms_fuse_normals", K)):
			for _ in range(3):
				m.Fuse(dev, (W, H), 2, k)
			torch.cuda.synchronize()
			e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
			e0.record()
			for _ in range(a.iters):
				m.Fuse(dev, (W, H), 2, k)
			e1.record()
			torch.cuda.synchronize()
			row[key] = e0.elapsed_time(e1)/a.iters
		with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
			gd, gc, gn = m.Fuse(dev, (W, H), 2, K)
			torch.cuda.synchronize()
		stage_us = {s: 0.0 for s, _ in STAGES}
		for ev in prof.key_averages():
			for s, keys in STAGES:
				if any(k in ev.key for k in keys):
					stage_us[s] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
		row["ms_stages"] = {s: round(v/1000.0, 4) for s, v in stage_us.items()}
		t = time.perf_counter()
		od, oc, on = F.fuse(pairs, (W, H), 2, K)
		row["ms_oracle_single_thread"] = (time.perf_counter()-t)*1000.0
		row["bit_identical"] = bool(np.array_equal(gd.cpu().numpy().view(np.uint32), od.view(np.uint32)) and
			np.array_equal(gc.cpu().numpy().view(np.uint32), oc.view(np.uint32)) and np.array_equal(gn.cpu().numpy().view(np.uint32), on.view(np.uint32)))
		row["coverage"] = float((od > 0).mean())
		row["gpu"], row["power_limit"] = name, power
		results.append(row)
		print(json.dumps(row))
	m.Release()
	if a.out:
		with open(a.out, "w") as f:
			json.dump(results, f, indent=1)


if __name__ == "__main__":
	main()
