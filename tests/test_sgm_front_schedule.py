"""CPU simulation of the wave-front SGM aggregation schedule (tests/cpp/front_sched_main.cpp over
openmvs_b200/csrc/sgm_front_sched.h — the header the kernel and the host driver share) against the oracle: the driver's
schedule (32 fronts per block, lag 1, its sub-cell width) and other block sizes, lags and sub-cell widths process every (pixel,
direction) exactly once, in a queue order that meets every dependency, and hand the path state over between segments correctly
— the summed path costs equal the oracle's bit for bit."""
import os
import struct
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
	out = str(tmp_path_factory.mktemp("front")/"front_sched")
	subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(ROOT, "tests", "cpp", "front_sched_main.cpp")])
	return out


# (fronts per block, lag, sub-cell width; 0: the driver's); (32, 1, 0) is the schedule the driver runs
@pytest.mark.parametrize("block,lag,subcell", [(32, 1, 0), (32, 1, 48), (32, 1, 16), (64, 0, 0), (32, 2, 0), (32, 0, 0), (8, 1, 0), (16, 0, 0), (5, 3, 0), (7, 0, 0), (3, 1, 0)])
def test_schedule_simulation_equals_oracle(exe, tmp_path, block, lag, subcell):
	from oracle import oracle as O
	from openmvs_b200 import synth
	num = 64
	for (w, h) in ((61, 47), (38, 73), (301, 40)):   # the last one spans three sub-cell columns   # wider than high and higher than wide; valid regions not multiples of 4
		rng = np.random.RandomState(w)
		lg, lc, rg, d = synth.make_stereo_pair(w, h)
		px, n = synth.sgm_pixel_map(w, h, -5, -5+num)
		costs = rng.randint(0, 256, n).astype(np.uint8)
		c, a, disp, cost = O.sgm_match(lg, lc, rg, px, n, costs=costs)
		P2s = O.sgm_p2s() if hasattr(O, "sgm_p2s") else None
		if P2s is None:
			import ctypes as C
			buf = (C.c_uint16*256)()
			O.lib().oracle_sgm_p2s(C.c_uint16(4), C.c_float(14.0), C.c_float(38.0), buf)
			P2s = np.frombuffer(buf, np.uint16).copy()
		fin, fout = str(tmp_path/"in.bin"), str(tmp_path/"out.bin")
		with open(fin, "wb") as f:
			f.write(struct.pack("7i", w, h, num, block, lag, 3, subcell))
			f.write(P2s.tobytes()); f.write(np.ascontiguousarray(lg, np.float32).tobytes()); f.write(costs.tobytes())
		r = subprocess.run([exe, fin, fout], capture_output=True, text=True)
		assert r.returncode == 0, r.stdout+r.stderr
		got = np.fromfile(fout, np.uint16)
		assert np.array_equal(got, a), (w, h, int((got != a).sum()))
