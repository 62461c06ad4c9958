"""GPU tests (run on an H100 with -m gpu): the sweep kernel scores a warp's propagation candidates as one packed list, lane l
of packed step s taking entry 32s+l of the concatenated per-pixel lists, and each pixel then applies the accept test to its own
candidates in order.  One sweep from an identical state must follow the per-pixel rule of the oracle's red-black schedule
(same candidates, same Philox slots) with the thresholds of the single-sweep parity test, for warps whose candidate counts are
even, uneven, all four, all zero, for rows shorter than a warp, with the evaluation cap on and for the geometric kernel.
"""
import numpy as np
import pytest
import torch

from test_pm_parity_gpu import _crop_reference, _dev_views, _plane, _record, _set, env  # noqa: F401  (env: fixture)

pytestmark = pytest.mark.gpu

KEEP = 0.9  # OPTDENSE.fNCCThresholdKeep: a candidate whose stored cost is not below it is not tested


def _costs(d, c, pattern):
	"""the pass-A state with the costs of the estimated pixels rewritten so that every warp gets the candidate counts of
	`pattern` (costs of the other colour decide which directions have a candidate)"""
	c = c.copy()
	m = d > 0
	low = np.minimum(c, 0.5)
	if pattern == "all4":      # every direction of every pixel away from the border has a candidate
		c[m] = low[m]
	elif pattern == "all0":    # no candidate anywhere: the warps only refine
		c[m] = 1.9
	elif pattern == "uneven":  # columns x with x//2 even score above KEEP: their pixels keep 2 candidates, the others 4,
		cols = (np.arange(c.shape[1])//2) % 2 == 0  # so neighbouring lanes of a warp alternate between 2 and 4
		hi = m & cols[None, :]
		c[m] = low[m]
		c[hi] = 1.9
	return c


def _candidates(d, c, far):
	"""candidate count of every pixel (the rule of pm_sweep_kernel: per direction, the lowest stored cost among the
	other-colour pixels at distance 1, 3, .. 2*far+1 inside the border is below KEEP)"""
	H, W = c.shape
	cnt = np.zeros((H, W), np.int32)
	ys, xs = np.nonzero(d > 0)
	for x, y in zip(xs, ys):
		for ox, oy in ((-1, 0), (1, 0), (0, -1), (0, 1)):
			best = abs(c[y+oy, x+ox]) if d[y+oy, x+ox] > 0 else 3.0
			for f in range(1, far+1):
				qx, qy = x+ox*(2*f+1), y+oy*(2*f+1)
				if not (4 <= qx < W-4 and 4 <= qy < H-4):
					break
				best = min(best, abs(c[qy, qx]))
			cnt[y, x] += best < KEEP
	return cnt


CASES = {
	# name: (cost pattern, reference crop (x0, y0, w, h) or None, nEvalCap, neighbour depth-maps)
	"uneven": ("uneven", None, 0, False),
	"all4": ("all4", None, 0, False),
	"all0": ("all0", None, 0, False),
	"narrow_rows": ("all4", (140, 0, 40, 240), 0, False),  # 16 pixels of a colour per row: lanes 16-31 have no pixel
	"eval_cap": ("uneven", None, 7, False),
	"geometric": ("uneven", None, 0, True),
}


@pytest.mark.parametrize("name", list(CASES))
def test_packed_sweep_follows_the_per_pixel_rule(env, small_scene, name):
	e = env
	pattern, crop, cap, geometric = CASES[name]
	sc, ref, views = small_scene
	if crop is not None:
		views = _crop_reference(views, *crop)
	depths = None
	if geometric:
		rng = np.random.RandomState(11)
		depths = [None]
		for v in views[1:]:
			dm = v.depth_gt.copy()
			dm[rng.rand(*dm.shape) < 0.05] = 0
			depths.append((dm, v.K, v.R, v.C))
	nR, far = 3, 2
	_set(e, nSubResolutionLevels=0, nEstimationGeometricIters=0, nPropagation=4, nPropagationFar=far, bSkipUnchanged=1,
		nEvalCap=cap, fNCCThresholdKeep=KEEP, fEstimationGeometricWeight=0.1)
	try:
		prm = e.O.default_params(schedule=1, propagation=e.O.rb_propagation(4, far, 0, cap), nRandomIters=nR, nSubResolutionLevels=0,
			threads=4)
		d, n, c = e.O.pm_score(views, prm, sc.dmin, sc.dmax, depths=depths)
		c = _costs(d, c, pattern)
		cnt = _candidates(d, c, far)
		live = d > 0
		if pattern == "all4":
			assert (cnt[live] == 4).mean() > 0.9
		elif pattern == "all0":
			assert not cnt.any()
		else:
			assert set(np.unique(cnt[live])) >= {2, 4}
		dv = _dev_views(e, views, depths)
		for sweep in range(2):
			plane = _plane(e, d, n); cost = torch.from_numpy(c).to(e.dev)
			e.pm.SweepDepthMap(dv, sc.dmin, sc.dmax, plane, cost, sweep, nRandomIters=nR)
			od, on, oc = e.O.pm_iterate(views, prm, sc.dmin, sc.dmax, d, n, c, sweep, depths=depths)
			pg, cg = plane.cpu().numpy(), np.abs(cost.cpu().numpy())
			m = od > 0
			rel = np.abs(pg[..., 3]-od)[m]/od[m]
			_record("packing_%s_s%d" % (name, sweep), frac_rel_gt_1e3=(rel > 1e-3).mean(), frac_rel_gt_1e5=(rel > 1e-5).mean(),
				cost_mean_abs_diff=np.abs(cg-oc)[m].mean())
			# the thresholds of test_single_sweep_parity_from_identical_state: only accept tests decided by the last float
			# bits may differ
			assert np.array_equal(pg[..., 3] > 0, m)
			assert (rel > 1e-3).mean() < 2e-3, (name, sweep, (rel > 1e-3).mean())
			assert (rel > 1e-5).mean() < 0.12, (name, sweep, (rel > 1e-5).mean())
			assert np.abs(cg-oc)[m].mean() < 5e-5
	finally:
		_set(e, nEvalCap=0, nPropagationFar=2, bSkipUnchanged=1, fNCCThresholdKeep=0.9)
