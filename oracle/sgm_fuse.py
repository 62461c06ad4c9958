"""ctypes binding of sgm_fuse_oracle.cpp: fusion-mode -2 of the SGM path (TEST INFRASTRUCTURE, like oracle.py: only tests/ and scripts
may import it; the product package openmvs_b200 never does).

sgm_fuse_oracle.cpp restates ProjectDisparity2DepthMap, the cluster vote of Fuse, the Q of a reversed pair and EstimateNormalMap in the
reference's sequential loop order.  It is built into a library of its own (the parity flags of the main oracle build), next to this file
when the tree is writable, else in a per-user temporary directory.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sgm_fuse_oracle.cpp")
_CXXFLAGS = ["-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-Wall", "-shared"]
_LIB = None

NO_DISP = 32767


def build(force: bool = False) -> str:
	"""-> path of libsgm_fuse_oracle.so, (re)built with g++ when missing or older than its source"""
	for out in (_HERE, os.path.join(tempfile.gettempdir(), "openmvs_b200_sgm_fuse_oracle_%d" % os.getuid())):
		so = os.path.join(out, "libsgm_fuse_oracle.so")
		if not force and os.path.exists(so) and os.path.getmtime(_SRC) <= os.path.getmtime(so):
			return so
		# build to a temporary name and rename: a concurrent process never loads a half-written library
		tmp = "%s.tmp.%d" % (so, os.getpid())
		try:
			os.makedirs(out, exist_ok=True)
			subprocess.check_call([os.environ.get("CXX", "g++")] + _CXXFLAGS + ["-o", tmp, _SRC])
			os.replace(tmp, so)
			return so
		except (OSError, subprocess.CalledProcessError):
			if out != _HERE:
				raise
		finally:
			if os.path.exists(tmp):
				os.unlink(tmp)
	raise RuntimeError("libsgm_fuse_oracle.so could not be built")


def lib():
	global _LIB
	if _LIB is None:
		L = C.CDLL(build())
		P, I = C.c_void_p, C.c_int
		L.oracle_sgmf_project.restype = I
		L.oracle_sgmf_project.argtypes = [P, P, I, I, I, P, I, I, P, P, P]
		L.oracle_sgmf_fuse.restype = None
		L.oracle_sgmf_fuse.argtypes = [I, P, P, P, I, I, C.c_uint, P, P]
		L.oracle_sgmf_pair_q.restype = None
		L.oracle_sgmf_pair_q.argtypes = [P]*8
		L.oracle_sgmf_normals.restype = None
		L.oracle_sgmf_normals.argtypes = [P, I, I, P, P]
		_LIB = L
	return _LIB


def _p(a):
	return None if a is None else a.ctypes.data


def project(disparity, cost, Q, subpixelSteps, size):
	"""ProjectDisparity2DepthMap of one pair into an image of size = (W, H) -> (depth, range (H, W, 2), conf, numDepths);
	conf is all 0 without a cost map"""
	d = np.ascontiguousarray(disparity, np.int16)
	c = None if cost is None else np.ascontiguousarray(cost, np.uint16)
	q = np.ascontiguousarray(Q, np.float64).reshape(16)
	W, H = int(size[0]), int(size[1])
	depth = np.zeros((H, W), np.float32); rng = np.zeros((H, W, 2), np.float32); conf = np.zeros((H, W), np.float32)
	n = lib().oracle_sgmf_project(_p(d), _p(c), d.shape[1], d.shape[0], int(subpixelSteps), _p(q), W, H, _p(depth), _p(rng), _p(conf))
	return depth, rng, conf, int(n)


def fuse_maps(depths, ranges, confs, minViews=2):
	"""the cluster vote of Fuse over per-pair projected maps (lists of (H, W), (H, W, 2), (H, W)) -> (depth, conf)"""
	D = np.ascontiguousarray(np.stack(depths), np.float32); R = np.ascontiguousarray(np.stack(ranges), np.float32)
	Cf = np.ascontiguousarray(np.stack(confs), np.float32)
	n, H, W = D.shape
	depth = np.zeros((H, W), np.float32); conf = np.zeros((H, W), np.float32)
	lib().oracle_sgmf_fuse(n, _p(D), _p(R), _p(Cf), W, H, int(minViews), _p(depth), _p(conf))
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
	lib().oracle_sgmf_pair_q(*[_p(a) for a in arrs], _p(out))
	return out.reshape(4, 4)


def normals(depth, K):
	"""EstimateNormalMap(Matrix3x3f(K), depth) -> (H, W, 3) float32"""
	d = np.ascontiguousarray(depth, np.float32)
	k = np.ascontiguousarray(K, np.float64).ravel()
	out = np.zeros(d.shape+(3,), np.float32)
	lib().oracle_sgmf_normals(_p(d), d.shape[1], d.shape[0], _p(k), _p(out))
	return out
