"""CPU checks of the hierarchical (tSGM) level loop: the oracle's Disparity2RangeMap against an independent transcription,
FlipDirection / UpscaleMask / ExtractMask against hand-derived answers, the level arithmetic, and the argument errors of the
new C-ABI entry points (which return before touching a device)."""
import ctypes as C

import numpy as np
import pytest

from oracle import tsgm as O

NO = 32767


def _trunc_div(a, b):
	q = abs(a)//abs(b)
	return q if (a >= 0) == (b >= 0) else -q


def _i16(v):
	return ((int(v)+32768) % 65536)-32768


def _range_map_py(D, M, minNumDisp, minNumDispInvalid):
	"""Disparity2RangeMap restated from the expansion rules: a range per coarse pixel, then the 2x grid
	(row 0 -> rows 0..4, row r -> 2r+3, 2r+4, the last row to the end; columns alike), idx = running sum in raster order."""
	rows, cols = D.shape
	mh, mw = M.shape
	rng = {}
	for r in range(rows):
		for c in range(cols):
			if M[2*r+3, 2*c+3] == 0:
				rng[r, c] = (NO, NO)
				continue
			bad = D[r, c] == NO
			hw = 20 if bad else 3
			win = D[max(r-hw, 0):r+hw+1, max(c-hw, 0):c+hw+1].ravel().astype(int)
			v = sorted(x for x in win if x != NO)
			if len(v) < 3:
				hi = min(_i16(cols*2//3), minNumDispInvalid)
				rng[r, c] = (-hi, hi)
				continue
			n = len(v)
			med = v[n//2] if n % 2 else _trunc_div(v[n//2-1]+v[n//2], 2)
			disp = _i16(med*2)
			mn, mx = v[0], v[-1]
			num = _i16((mx-mn)*2)
			if num < minNumDisp:
				num = minNumDisp
				rng[r, c] = (_i16(disp-_trunc_div(num, 2)), _i16(disp+_trunc_div(num+1, 2)))
			else:
				mnd = 64 if bad else 32
				if num > mnd:
					rng[r, c] = (_i16(disp-_trunc_div(mnd*(disp-mn*2)+1, num)), _i16(disp+_trunc_div(mnd*(mx*2+1-disp)+1, num)))
				else:
					rng[r, c] = (_i16(disp-_trunc_div(num, 2)), _i16(disp+_trunc_div(num+1, 2)))
	lo = np.zeros((mh, mw), np.int64); hi = np.zeros((mh, mw), np.int64)
	for y in range(mh):
		r = 0 if y < 5 else min((y-3)//2, rows-1)
		for x in range(mw):
			c = 0 if x < 5 else min((x-3)//2, cols-1)
			lo[y, x], hi[y, x] = rng[r, c]
	width = np.maximum(hi-lo, 0).ravel()
	idx = np.concatenate([[0], np.cumsum(width)[:-1]])
	return lo.ravel(), hi.ravel(), idx, int(width.sum())


def _random_map(rng, rows, cols, holes, lo=-40, hi=40):
	base = rng.randint(lo, hi, (rows, cols))
	# smooth-ish field with outliers, NO_DISP holes (also whole blocks, so that 41x41 windows fall back)
	D = (base//3 + np.arange(cols)[None, :]//5).astype(np.int16)
	D[rng.rand(rows, cols) < holes] = NO
	D[:rows//3, :cols//4] = NO
	return D


@pytest.mark.parametrize("first", [True, False])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_range_map_matches_transcription(first, seed):
	rng = np.random.RandomState(seed)
	rows, cols = 23+seed, 31+2*seed
	D = _random_map(rng, rows, cols, 0.25)
	mh, mw = 2*rows+5+seed, 2*cols+6+seed
	M = np.full((mh, mw), 255, np.uint8)
	M[rng.rand(mh, mw) < 0.1] = 0
	mnd, mndi = (11, 33) if first else (5, 7)
	px, n = O.tsgm_range_map(D, M, mnd, mndi)
	lo, hi, idx, total = _range_map_py(D, M, mnd, mndi)
	assert n == total
	assert np.array_equal(px["dmin"], lo) and np.array_equal(px["dmax"], hi)
	assert np.array_equal(px["idx"], idx.astype(np.uint64))
	# masked pixels and wide (clipped) ranges occur; the narrow branch is pinned by the even-count test below
	w = (hi-lo)
	assert (w == 0).any() and (w > mnd).any()
	# no estimate at all: every unmasked pixel falls back to +-min(cols*2/3, minNumDispInvalid)
	px, n = O.tsgm_range_map(np.full_like(D, NO), M, mnd, mndi)
	lo, hi, idx, total = _range_map_py(np.full_like(D, NO), M, mnd, mndi)
	f = min(cols*2//3, mndi)
	assert n == total and np.array_equal(px["idx"], idx.astype(np.uint64)) and set(np.unique(hi-lo)) <= {0, 2*f}


def test_range_map_even_count_median_truncates_toward_zero():
	# one coarse pixel with a 7x7 window of 4 valid values -3, -2, 5, 6 -> median (-2+5)/2 = 1 -> disp 2
	D = np.full((7, 7), NO, np.int16)
	D[3, 3] = -3; D[3, 4] = -2; D[2, 3] = 5; D[4, 4] = 6
	M = np.full((19, 21), 255, np.uint8)
	px, n = O.tsgm_range_map(D, M, 3, 16)
	lo, hi, idx, total = _range_map_py(D, M, 3, 16)
	assert n == total and np.array_equal(px["dmin"], lo) and np.array_equal(px["dmax"], hi)
	# pixel (3, 3): numDisp = (6+3)*2 = 18 <= 32 -> [2-9, 2+9)
	r, c = 2*3+3, 2*3+3
	assert (px["dmin"][r*21+c], px["dmax"][r*21+c]) == (-7, 11)
	# a negative odd sum: -3, -2 -> (-5)/2 = -2 (not -3)
	D2 = np.full((7, 7), NO, np.int16)
	D2[3, 3] = -3; D2[3, 4] = -2; D2[2, 2] = -2; D2[4, 4] = -3
	px2, _ = O.tsgm_range_map(D2, M, 3, 16)
	lo2, hi2, _, _ = _range_map_py(D2, M, 3, 16)
	assert np.array_equal(px2["dmin"], lo2)
	assert (px2["dmin"][r*21+c], px2["dmax"][r*21+c]) == (-4-1, -4+2)   # median -2.5 -> -2, disp -4, numDisp 2 < 3 -> 3


def test_flip_direction_collisions_last_column_wins():
	l2r = np.full((2, 10), NO, np.int16)
	l2r[0, 2] = 3    # writes -3 to columns 4, 5, 6
	l2r[0, 3] = 2    # writes -2 to columns 4, 5, 6 (later c wins)
	l2r[0, 5] = 0    # writes 0 to columns 4, 5, 6
	l2r[0, 9] = -1   # writes 1 to columns 7, 8, 9... c+d-1 = 7 .. c+d+1 = 9
	l2r[1, 0] = -1   # columns -2 .. 0: only column 0
	l2r[1, 8] = 1    # columns 8, 9 (10 is outside)
	want = np.full((2, 10), NO, np.int16)
	want[0, 4:7] = 0; want[0, 7:10] = 1
	want[1, 0] = 1; want[1, 8:10] = -1
	assert np.array_equal(O.tsgm_flip_direction(l2r), want)


def test_upscale_mask_hand_derived():
	m = np.array([[255, 0], [0, 255]], np.uint8)
	got = O.tsgm_upscale_mask(m, (8, 8))
	want = np.zeros((8, 8), np.uint8)
	want[3:5, 3:5] = 255; want[5:7, 5:7] = 255
	assert np.array_equal(got, want)
	# a 2x grid that cuts the last block
	got = O.tsgm_upscale_mask(m, (6, 6))
	want = np.zeros((6, 6), np.uint8); want[3:5, 3:5] = 255; want[5, 5] = 255
	assert np.array_equal(got, want)


def test_extract_mask_hand_derived():
	d = np.array([[NO, 1, NO, 2, 3, 4, 5, NO, 6, 7, 8, NO]], np.int16)
	m = np.full(d.shape, 255, np.uint8)
	m[0, 6] = 0
	got = O.tsgm_extract_mask(d, m, 3)
	# from the left: columns 0..4 invalidated (3 valid values passed at column 4); from the right: 11, 10, 9, 8 (valid 8, 7, 6 at 10, 9, 8)
	want = np.array([[0, 0, 0, 0, 0, 255, 0, 255, 0, 0, 0, 0]], np.uint8)
	assert np.array_equal(got, want)


def test_level_arithmetic():
	from openmvs_b200.depth_estimator import SemiGlobalMatcher as S
	table = [
		((1920, 1080, 320), [(480, 270), (960, 540), (1920, 1080)], (234, 129)),
		((640, 480, 320), [(320, 240), (640, 480)], (154, 114)),
		((640, 360, 160), [(160, 90), (320, 180), (640, 360)], (74, 39)),
		((400, 240, 160), [(200, 120), (400, 240)], (94, 54)),
		((640, 480, 0), [(640, 480)], (314, 234)),
	]
	for (w, h, mr), sizes, init in table:
		assert O.tsgm_levels(w, h, mr) == (sizes, init), (w, h, mr)
		assert S.HierarchyLevels(w, h, mr) == (sizes, init), (w, h, mr)
	# odd sizes round half to even like cv::saturate_cast: 1081 x 0.25 = 270.25, 270 x 0.5 = 135 -> 135 x 0.5 = 67.5 -> 68
	assert S.HierarchyLevels(1921, 1081, 320) == O.tsgm_levels(1921, 1081, 320)
	assert S.HierarchyLevels(1921, 1081, 320)[1] == (int(np.rint(480*0.5))-6, int(np.rint(270*0.5))-6)
	from openmvs_b200 import lib
	with pytest.raises(lib.B200MVSError):
		S.HierarchyLevels(20, 20, 320)


def test_entry_points_refuse_bad_arguments_without_a_device():
	from openmvs_b200 import lib as L
	lib = L.load()
	P = C.c_void_p
	ERR = 1
	n = C.c_uint64()
	assert lib.b200mvs_sgm_match_hierarchical_device(None, P(8), P(8), P(8), P(8), 64, 64, None, 0, 0, None, None, 32, 100, 1, 4, None,
		P(8), P(8), None, None) == ERR
	assert lib.b200mvs_sgm_range_map_device(None, P(8), 4, 4, P(8), 16, 16, 3, 16, P(8), C.byref(n), None) == ERR
	assert lib.b200mvs_sgm_flip_direction_device(None, P(8), P(16), 4, 4, None) == ERR
	assert lib.b200mvs_sgm_upscale_mask_device(None, P(8), 4, 4, P(16), 8, 8, None) == ERR
	assert lib.b200mvs_sgm_extract_mask_device(None, P(8), P(16), 4, 4, 3, None) == ERR
	assert lib.b200mvs_sgm_filter_speckles_device(None, P(8), 4, 4, NO, 10, 5, None) == ERR
	assert lib.b200mvs_resize_area_u8_device(None, P(8), 4, 4, 3, 2, P(16), None) == ERR
	assert lib.b200mvs_sgm_level_mask_device(None, P(8), 16, 16, 8, 8, P(16), None) == ERR
	nl = C.c_int()
	assert lib.b200mvs_sgm_levels(6, 100, 0, C.byref(nl), None, None, None, None) == ERR
	assert lib.b200mvs_sgm_levels(100, 100, -1, C.byref(nl), None, None, None, None) == ERR
	assert lib.b200mvs_sgm_levels(100, 100, 0, C.byref(nl), None, None, None, None) == 0 and nl.value == 1
