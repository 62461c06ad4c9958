"""FuseDepthMaps of 12 views at 1920x1080 with 9 neighbours each: the host form (sequential loop) and the device form in the same run.

  python scripts/profile_fuse.py [--width W] [--height H] [--iters N] [--out FILE]

The depth-maps are the synthetic scene's ground truth with 0.2 % noise, 10 % holes and a band of outliers.  Prints one JSON object:
the host time (one run), the device time per call (wall and device, best of --iters runs after one warm-up, each on a fresh copy of
the maps), the device time, fixed-point iterations, candidates, edges and shared-target edges of every round, whether both forms
give the same point cloud and depth-maps bit for bit, and the card name and power limit (read-only nvidia-smi query).  The host and
wall times leave out the conversion of the point cloud into per-point numpy arrays (ms_to_numpy), which both forms share."""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from openmvs_b200 import synth  # noqa: E402
from openmvs_b200 import depth_estimator as DE  # noqa: E402
from openmvs_b200.depth_estimator import FuseDepthMaps, FuseRoundStats, _device_context  # noqa: E402

# the time FuseDepthMaps spends turning the C point cloud into per-point numpy arrays (the same for both forms), so that the
# fusion itself can be reported apart from it
_CONVERT_MS = []
_point_cloud = DE._point_cloud


def _timed_point_cloud(lib, cloud):
	t = time.perf_counter()
	try:
		return _point_cloud(lib, cloud)
	finally:
		_CONVERT_MS.append((time.perf_counter()-t)*1000.0)


DE._point_cloud = _timed_point_cloud


def gpu_info():
	try:
		out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True, timeout=30)
		name, power = [s.strip() for s in out.strip().splitlines()[0].split(",")]
		return name, power
	except Exception as e:  # noqa: BLE001
		return torch.cuda.get_device_name(0), "unknown (%s)" % type(e).__name__


def make_views(W, H, n=12, n_nb=9, seed=0):
	sc = synth.make_scene(W, H, n, step_deg=5.0)
	rng = np.random.RandomState(seed)
	views = []
	for i, v in enumerate(sc.views):
		d = v.depth_gt.astype(np.float32)*(1+2e-3*rng.randn(H, W)).astype(np.float32)
		d[rng.rand(H, W) < 0.1] = 0
		d[H//3:H//3+2, :] *= np.float32(0.8)
		nb = list(sc.neighbors(i, n_nb))
		color = (np.clip(v.image, 0, 1)[..., None]*255).astype(np.uint8).repeat(3, -1)
		views.append(dict(depth=d, normal=v.normal_gt.astype(np.float32), conf=rng.rand(H, W).astype(np.float32), color=color,
			K=v.K, R=v.R, C=v.C, neighbors=nb, n_scene_neighbors=len(nb)))
	return views


def to_device(views):
	return [dict(v, **{k: torch.from_numpy(np.ascontiguousarray(v[k])).cuda() for k in ("depth", "normal", "conf", "color")}) for v in views]


def same(a, b):
	return (np.array_equal(a.points, b.points) and a.nDepths == b.nDepths and np.array_equal(a.colors, b.colors) and
		np.array_equal(a.normals, b.normals) and len(a.pointViews) == len(b.pointViews) and
		all(np.array_equal(x, y) for x, y in zip(a.pointViews, b.pointViews)) and
		all(np.array_equal(x, y) for x, y in zip(a.pointWeights, b.pointWeights)) and
		all(np.array_equal(x, y) for x, y in zip(a.projs, b.projs)))


def main():
	ap = argparse.ArgumentParser()
	ap.add_argument("--width", type=int, default=1920)
	ap.add_argument("--height", type=int, default=1080)
	ap.add_argument("--iters", type=int, default=2)
	ap.add_argument("--out", default=None)
	a = ap.parse_args()
	name, power = gpu_info()
	t = time.perf_counter()
	views = make_views(a.width, a.height)
	row = {"size": [a.width, a.height], "views": len(views), "neighbors": 9, "s_scene": round(time.perf_counter()-t, 1)}
	host = copy.deepcopy(views)
	t = time.perf_counter()
	ph = FuseDepthMaps(host)
	row["ms_host"] = (time.perf_counter()-t)*1000.0 - _CONVERT_MS[-1]
	row["ms_to_numpy"] = _CONVERT_MS[-1]
	ctx = _device_context(torch.device("cuda", torch.cuda.current_device()))
	walls, devs = [], []
	for it in range(a.iters+1):
		dev = to_device(views)
		torch.cuda.synchronize()
		t = time.perf_counter()
		pd = FuseDepthMaps(dev)
		wall = (time.perf_counter()-t)*1000.0 - _CONVERT_MS[-1]
		if it > 0:
			walls.append(wall); devs.append(ctx.stats.ms_device)
	row["ms_device_wall"] = min(walls)
	row["ms_device_events"] = min(devs)
	row["kernel_launches"] = ctx.stats.kernel_launches
	row["bytes_d2h"] = ctx.stats.bytes_d2h
	row["speedup_wall"] = row["ms_host"]/row["ms_device_wall"]
	row["points"] = len(ph.points)
	row["nDepths"] = ph.nDepths
	row["bit_identical"] = bool(same(pd, ph) and all(np.array_equal(d["depth"].cpu().numpy(), h["depth"]) for d, h in zip(dev, host)))
	row["rounds"] = FuseRoundStats()[torch.cuda.current_device()]
	row["gpu"], row["power_limit"] = name, power
	print(json.dumps(row))
	if a.out:
		with open(a.out, "w") as f:
			json.dump(row, f, indent=1)


if __name__ == "__main__":
	main()
