"""ctypes binding of sgm_fuse_oracle.cpp: fusion-mode -2 of the SGM path (TEST INFRASTRUCTURE, like oracle.py: only tests/ and scripts
may import it; the product package openmvs_b200 never does).

sgm_fuse_oracle.cpp (part of liboracle.so) restates ProjectDisparity2DepthMap, the cluster vote of Fuse, the Q of a reversed pair
and EstimateNormalMap in the reference's sequential loop order.
"""
from __future__ import annotations

import numpy as np

from . import oracle as O
from .oracle import NO_DISP  # noqa: F401


def project(disparity, cost, Q, subpixelSteps, size):
	"""ProjectDisparity2DepthMap of one pair into an image of size = (W, H) -> (depth, range (H, W, 2), conf, numDepths);
	conf is all 0 without a cost map"""
	d = np.ascontiguousarray(disparity, np.int16)
	c = None if cost is None else np.ascontiguousarray(cost, np.uint16)
	q = np.ascontiguousarray(Q, np.float64).reshape(16)
	W, H = int(size[0]), int(size[1])
	depth = np.zeros((H, W), np.float32); rng = np.zeros((H, W, 2), np.float32); conf = np.zeros((H, W), np.float32)
	n = O.lib().oracle_sgmf_project(O._fptr(d), None if c is None else O._fptr(c), d.shape[1], d.shape[0], int(subpixelSteps), O._fptr(q),
		W, H, O._fptr(depth), O._fptr(rng), O._fptr(conf))
	return depth, rng, conf, int(n)


def fuse_maps(depths, ranges, confs, minViews=2):
	"""the cluster vote of Fuse over per-pair projected maps (lists of (H, W), (H, W, 2), (H, W)) -> (depth, conf)"""
	D = np.ascontiguousarray(np.stack(depths), np.float32); R = np.ascontiguousarray(np.stack(ranges), np.float32)
	Cf = np.ascontiguousarray(np.stack(confs), np.float32)
	n, H, W = D.shape
	depth = np.zeros((H, W), np.float32); conf = np.zeros((H, W), np.float32)
	O.lib().oracle_sgmf_fuse(n, O._fptr(D), O._fptr(R), O._fptr(Cf), W, H, int(minViews), O._fptr(depth), O._fptr(conf))
	return depth, conf


def fuse(pairs, size, minViews=2, K=None):
	"""SemiGlobalMatcher::Fuse of pairs = [(disparity, cost or None, Q, subpixelSteps), ...] into an image of size = (W, H)
	-> (depth, conf, normal or None)"""
	maps = [project(d, c, Q, s, size) for d, c, Q, s in pairs]
	depth, conf = fuse_maps([m[0] for m in maps], [m[1] for m in maps], [m[2] for m in maps], minViews)
	return depth, conf, None if K is None else normals(depth, K)


def pair_q(Q, Kleft, Rleft, Cleft, K, R, C):
	"""Q of a pair whose left camera is (Kleft, Rleft, Cleft), re-targeted to the image of camera (K, R, C)"""
	arrs = [np.ascontiguousarray(a, np.float64).ravel() for a in (Q, Kleft, Rleft, Cleft, K, R, C)]
	out = np.zeros(16, np.float64)
	O.lib().oracle_sgmf_pair_q(*[O._fptr(a) for a in arrs], O._fptr(out))
	return out.reshape(4, 4)


def normals(depth, K):
	"""EstimateNormalMap(Matrix3x3f(K), depth) -> (H, W, 3) float32"""
	d = np.ascontiguousarray(depth, np.float32)
	k = np.ascontiguousarray(K, np.float64).ravel()
	out = np.zeros(d.shape+(3,), np.float32)
	O.lib().oracle_sgmf_normals(O._fptr(d), d.shape[1], d.shape[0], O._fptr(k), O._fptr(out))
	return out
