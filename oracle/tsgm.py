"""ctypes binding of tsgm_oracle.cpp and the level loop of the hierarchical (tSGM) pair matcher (TEST INFRASTRUCTURE, like
oracle.py: only tests/ and scripts may import it; the product package openmvs_b200 never does).

tsgm_oracle.cpp (part of liboracle.so) restates the reference's Disparity2RangeMap, FlipDirection, UpscaleMask and ExtractMask.
tsgm_match composes the whole loop from these helpers, oracle.py's sgm_match / sgm_cross_check / sgm_refine, and OpenCV (cv2) for
the pyramid, the mask resize and filterSpeckles.
"""
from __future__ import annotations

import numpy as np

from . import oracle as O
from .oracle import NO_DISP, SGM_PIXEL


def tsgm_range_map(disparity, mask, minNumDisp, minNumDispInvalid):
	"""Disparity2RangeMap -> (pixel records of the mask's 2x grid, numCosts)"""
	d = np.ascontiguousarray(disparity, np.int16); m = np.ascontiguousarray(mask, np.uint8)
	px = np.zeros(m.size, SGM_PIXEL)
	n = O.lib().oracle_tsgm_range_map(O._fptr(d), d.shape[1], d.shape[0], O._fptr(m), m.shape[1], m.shape[0], int(minNumDisp),
		int(minNumDispInvalid), O._fptr(px))
	return px, int(n)


def tsgm_flip_direction(l2r):
	a = np.ascontiguousarray(l2r, np.int16); out = np.zeros_like(a)
	O.lib().oracle_tsgm_flip_direction(O._fptr(a), O._fptr(out), a.shape[1], a.shape[0])
	return out


def tsgm_upscale_mask(mask, size2x):
	m = np.ascontiguousarray(mask, np.uint8); out = np.zeros((size2x[1], size2x[0]), np.uint8)
	O.lib().oracle_tsgm_upscale_mask(O._fptr(m), m.shape[1], m.shape[0], O._fptr(out), int(size2x[0]), int(size2x[1]))
	return out


def tsgm_extract_mask(disparity, mask, thValid=3):
	d = np.ascontiguousarray(disparity, np.int16); m = np.array(mask, np.uint8, copy=True, order="C")
	O.lib().oracle_tsgm_extract_mask(O._fptr(d), O._fptr(m), d.shape[1], d.shape[0], int(thValid))
	return m


def tsgm_levels(width, height, minResolution):
	"""level sizes (coarsest first) and the initial map's size, as SemiGlobalMatcher::Match(scene, ...) derives them"""
	scale = 1.0
	if minResolution > 0:
		size = max(width, height)
		level = 8
		if (size >> level) < minResolution:
			level = 0
			while (size >> (level+1)) >= minResolution:
				level += 1
		scale = 1.0/max(2, 2**level)
	sizes = []
	while True:
		sizes.append((int(np.rint(width*scale)), int(np.rint(height*scale))))
		scale *= 2
		if not scale < 1+1e-9:
			break
	return sizes, (int(np.rint(sizes[0][0]*0.5))-6, int(np.rint(sizes[0][1]*0.5))-6)


def tsgm_match(left_gray, left_bgr, right_gray, right_bgr, init=None, left_mask=None, right_mask=None, minResolution=320,
		nSpeckleSize=100, thCross=1, subpixelSteps=4, P1=3, P2=4, alpha=14.0, beta=38.0):
	"""The level loop of SemiGlobalMatcher::Match(scene, ...) for one rectified pair: cv2.resize for the pyramid and the masks,
	cv2.filterSpeckles, oracle.py's sgm_match / sgm_cross_check / sgm_refine and this module's tsgm_* helpers.
	-> (left disparity * subpixelSteps, cost, [{"size", "numCosts"}] per level)"""
	import cv2
	h, w = left_gray.shape
	sizes, (iw, ih) = tsgm_levels(w, h, minResolution)
	tsgm = minResolution > 0
	dL = np.full((ih, iw), NO_DISP, np.int16) if init is None else np.array(init, np.int16, copy=True)
	dR = None
	if not tsgm:
		v = dL[dL != NO_DISP].astype(np.int32)
		if v.size == 0:
			raise ValueError("minResolution = 0 needs an initial map with a valid disparity")
		numDisp = np.int16(np.int16(v.max()-v.min())+16); disp = np.int16(v.min()+v.max())
		lo, hi = int(np.int16(disp-numDisp)), int(np.int16(disp+numDisp))
	full = lambda m: np.full((h, w), 255, np.uint8) if m is None else np.ascontiguousarray(m, np.uint8)
	mL, mR = full(left_mask), full(right_mask)
	levels = []
	for k, (lw, lh) in enumerate(sizes):
		vw, vh = lw-6, lh-6
		first = k == 0
		if (lw, lh) == (w, h):
			lg, lc, rg, rc = left_gray, left_bgr, right_gray, right_bgr
		else:
			s = 1.0/(1 << (len(sizes)-1-k))
			rs = lambda a: np.ascontiguousarray(cv2.resize(a, None, fx=s, fy=s, interpolation=cv2.INTER_AREA))
			lg, lc, rg, rc = rs(left_gray), rs(left_bgr), rs(right_gray), rs(right_bgr)
			assert lg.shape == (lh, lw)
		if first:
			crop = lambda m: np.ascontiguousarray(cv2.resize(m, (lw, lh), interpolation=cv2.INTER_NEAREST)[3:3+vh, 3:3+vw])
			mL, mR = crop(mL), crop(mR)
		else:
			mL, mR = tsgm_upscale_mask(mL, (vw, vh)), tsgm_upscale_mask(mR, (vw, vh))
		def match(g0, c0, g1, px, n):
			if n == 0:
				return np.zeros(0, np.uint16), np.full((vh, vw), NO_DISP, np.int16), np.full((vh, vw), 65535, np.uint16)
			_, a, d, c = O.sgm_match(g0, c0, g1, px, n, P1, P2, alpha, beta)
			return a, d, c
		if tsgm:
			pxR, nR = tsgm_range_map(tsgm_flip_direction(dL), mR, 11 if first else 5, 33 if first else 7)
		else:
			pxR = np.zeros(vw*vh, SGM_PIXEL); nR = vw*vh*(hi-lo)
			pxR["idx"] = np.arange(vw*vh, dtype=np.uint64)*np.uint64(hi-lo); pxR["dmin"] = lo; pxR["dmax"] = hi
		_, dR, _ = match(rg, rc, lg, pxR, nR)
		if tsgm:
			pxL, nL = tsgm_range_map(dL, mL, 11 if first else 5, 33 if first else 7)
		else:
			pxL = pxR.copy(); nL = nR
			pxL["dmin"] = -hi; pxL["dmax"] = -lo
		aL, dL, cost = match(lg, lc, rg, pxL, nL)
		levels.append({"size": (lw, lh), "numCosts": (nR, nL)})
		if first:
			dL = O.sgm_cross_check(dL, dR, thCross)
			dR = O.sgm_cross_check(dR, dL, thCross)
			cv2.filterSpeckles(dL, NO_DISP, nSpeckleSize, 5)
			cv2.filterSpeckles(dR, NO_DISP, nSpeckleSize, 5)
			mL = tsgm_extract_mask(dL, mL, 3)
			mR = tsgm_extract_mask(dR, mR, 3)
		else:
			dL = O.sgm_cross_check(dL, dR, thCross)
	if subpixelSteps > 1 and nL > 0:
		dL = O.sgm_refine(pxL, aL, dL, subpixelSteps)
	return dL, cost, levels
