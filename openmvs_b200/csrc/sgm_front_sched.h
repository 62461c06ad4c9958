// sgm_front_sched.h — the scanline geometry of every SGM aggregation kernel (sgm_front.cu, sgm_kernels.cu), and the work items and
// schedule of the wave-front aggregation, shared by its kernel, the host driver (sgm_host.cu) and the CPU simulation of the schedule
// (tests/cpp/front_sched_main.cpp, run by tests/test_sgm_front_schedule.py).
#pragma once
#include <stdint.h>
#include <algorithm>
#include <vector>
#if defined(__CUDACC__)
#define FRONT_HD __host__ __device__
#else
#define FRONT_HD
#endif
#ifndef __CUDACC__
using std::min; using std::max;
struct float2;
#endif

// one work item: direction `dir & 0xFF` (phase `ph` of pass `dir >> 8` of the launch), paths k0 .. k0+3, fronts [fb*FB, fb*FB+FB)
struct FrontItem {
	int k0; short dir; short ph;
	int fb;
	int seq;       // number of earlier items of the same band: wait until progress[chain] >= seq
	int chain;     // index into progress[]
	int depCell;   // first sub-cell of (phase - 1, fb) whose completion this item waits for, or -1
	int depNeed;   // bits 0-7: number of consecutive sub-cells waited for (each until cellDone >= cellNeed); bits 8-15: own sub-cells
	int cell;      // this item's first sub-cell (completion counters to bump)
};
struct FrontArgs {
	const FrontItem* items; int nItems;
	int* ticket;         // queue head
	int* progress;       // per (pass, phase, band): segments completed
	int* cellDone;       // per (pass, phase, front block, sub-cell): items completed
	const int* cellNeed; // ... items that touch it
	int* error;          // set to 1 when a wait timed out (never in a correct schedule)
	uint16_t* state;     // per (pass, phase, path): the normalised previous line, num u16
	float2* meta;        // per (pass, phase, path): {previous intensity, have-previous flag}
	int maxPaths;        // paths per phase slot in state / meta
	int FB;              // fronts per block
	int num;             // disparities per pixel (16 * NW)
	// the (up to two) passes that share the launch's queue; each accumulates into its own sum volume
	int fa[2], fb[2], fc[2];   // front f(x,y) = fa*x + fb*y + fc >= 0
	int storePhase0[2];        // 1: phase 0 stores the sum instead of adding to it (the volume's first pass)
	uint16_t* sum[2];
};

// number of scanlines of direction `dir` in a W x H region
FRONT_HD inline int front_path_count(int dir, int W, int H) { return dir == 0 || dir == 2 ? W : dir == 1 || dir == 3 ? H : W+H-1; }
// start pixel and step of scanline `k` of direction `dir` (order of SemiGlobalMatcher.cpp:1084-1199); host and device
FRONT_HD inline bool front_path_start(int dir, int k, int W, int H, int& x, int& y, int& dx, int& dy) {
	switch (dir) {
	case 0: if (k >= W) return false; x = k; y = 0; dx = 0; dy = 1; return true;        // width-down
	case 1: if (k >= H) return false; x = 0; y = k; dx = 1; dy = 0; return true;        // height-right
	case 2: if (k >= W) return false; x = k; y = H-1; dx = 0; dy = -1; return true;     // width-up
	case 3: if (k >= H) return false; x = W-1; y = k; dx = -1; dy = 0; return true;     // height-left
	case 4: dx = 1; dy = 1;                                                             // right-down
		if (k < W) { x = k; y = 0; return true; } k -= W; if (k >= H-1) return false; x = 0; y = k+1; return true;
	case 5: dx = -1; dy = 1;                                                            // left-down
		if (k < W-1) { x = k; y = 0; return true; } k -= W-1; if (k >= H) return false; x = W-1; y = k; return true;
	case 6: dx = 1; dy = -1;                                                            // right-up
		if (k < W-1) { x = k+1; y = H-1; return true; } k -= W-1; if (k >= H) return false; x = 0; y = k; return true;
	default: dx = -1; dy = -1;                                                          // left-up
		if (k < W) { x = k; y = H-1; return true; } k -= W; if (k >= H-1) return false; x = W-1; y = k; return true;
	}
}
// steps until the scanline leaves the region
FRONT_HD inline int front_path_len(int x0, int y0, int dx, int dy, int W, int H) {
	int n = 0x7FFFFFFF;
	if (dx > 0) n = min(n, W-x0); else if (dx < 0) n = min(n, x0+1);
	if (dy > 0) n = min(n, H-y0); else if (dy < 0) n = min(n, y0+1);
	return n;
}
// first step s >= 0 of a path with f(s) = f0 + s*df (df > 0) at or beyond front `lo`
FRONT_HD inline int front_first_step(int lo, int f0, int df) {
	const int a = lo-f0;
	return a <= 0 ? 0 : (a+df-1)/df;
}

// ---- host side: schedule --------------------------------------------------------------------------------------------
struct FrontPassDesc { int fa, fb; int nDirs; int dirs[4]; };

// Phase dependencies are tracked per SUB-CELL: a front block cut into column ranges of SW (default FRONT_SW) pixels.  An item touches the one
// to three sub-cells its pixels fall into (its paths are adjacent and its segment is at most a block long); it waits until every
// item of the previous phase that touches one of them is complete, and bumps the counters of its own when it is done.  With
// dependencies this local the phases of a block can follow each other directly in the queue (lag 0): the slice of the sum
// volume a block owns is read-modify-written by its four directions while it sits in the L2.
constexpr int FRONT_SW = 64;    // default width; b200mvs_debug.frontSubCell overrides it (the driver keeps at most 30 columns of sub-cells)

// Work items of one pass in queue order; returns the number of front blocks, bands and sub-cell columns through nFB / maxBands /
// nSX, and the number of items touching each sub-cell through cellCount (index (ph*nFB + fb)*nSX + sx).
// lag: queue distance (in front blocks) between consecutive phases of the same block (0: the phases of a block are adjacent).
inline void sgm_front_build(int vw, int vh, const FrontPassDesc& pd, int FB, int lag, int SW, std::vector<FrontItem>& items, int& nFB, int& maxBands, int& fc,
	int& nSX, std::vector<int>& cellCount)
{
	// offset that makes the front coordinate non-negative
	const int cx[2] = {0, vw-1}, cy[2] = {0, vh-1};
	int fmin = 0x7FFFFFFF, fmax = -0x7FFFFFFF;
	for (int a = 0; a < 2; ++a) for (int b = 0; b < 2; ++b) { const int f = pd.fa*cx[a] + pd.fb*cy[b]; fmin = std::min(fmin, f); fmax = std::max(fmax, f); }
	fc = -fmin;
	nFB = (fmax-fmin)/FB + 1;
	maxBands = (vw+vh+3)/4 + 1;
	nSX = (vw+SW-1)/SW;
	const bool phases = pd.nDirs > 1;      // a pass of one direction has no phase dependencies: no counters
	items.clear();
	std::vector<int> xkey;                // first column of every item: position along the front
	cellCount.assign((size_t)pd.nDirs*nFB*nSX, 0);
	for (int ph = 0; ph < pd.nDirs; ++ph) {
		const int dir = pd.dirs[ph];
		const int nPaths = front_path_count(dir, vw, vh);
		for (int band = 0; band*4 < nPaths; ++band) {
			int nv[4], f0v[4], dfv[4], xsv[4], dxv[4]; bool pv[4];
			int blo = 0x7FFFFFFF, bhi = -1;
			for (int g = 0; g < 4; ++g) {
				int x, y, dx, dy;
				pv[g] = front_path_start(dir, band*4+g, vw, vh, x, y, dx, dy);
				nv[g] = 0; f0v[g] = 0; dfv[g] = 1; xsv[g] = 0; dxv[g] = 0;
				if (!pv[g]) continue;
				nv[g] = front_path_len(x, y, dx, dy, vw, vh);
				f0v[g] = pd.fa*x + pd.fb*y + fc; dfv[g] = pd.fa*dx + pd.fb*dy;
				xsv[g] = x; dxv[g] = dx;
				blo = std::min(blo, f0v[g]/FB); bhi = std::max(bhi, (f0v[g]+(nv[g]-1)*dfv[g])/FB);
			}
			int seq = 0;
			for (int fb = blo; fb <= bhi; ++fb) {
				int xlo = 0x7FFFFFFF, xhi = -1;
				for (int g = 0; g < 4; ++g) {
					if (!pv[g]) continue;
					const int a = std::min(nv[g], front_first_step(fb*FB, f0v[g], dfv[g])), b = std::min(nv[g], front_first_step((fb+1)*FB, f0v[g], dfv[g]));
					if (b <= a) continue;
					const int xa = xsv[g]+a*dxv[g], xb = xsv[g]+(b-1)*dxv[g];
					xlo = std::min(xlo, std::min(xa, xb)); xhi = std::max(xhi, std::max(xa, xb));
				}
				if (xhi < 0) continue;
				const int sx0 = xlo/SW, nsx = phases ? xhi/SW-sx0+1 : 0;
				FrontItem it;
				it.k0 = band*4; it.dir = (short)dir; it.ph = (short)ph; it.fb = fb; it.seq = seq++;
				it.chain = ph*maxBands + band;
				it.cell = (ph*nFB + fb)*nSX + sx0;                                   // first own sub-cell
				it.depCell = ph > 0 ? ((ph-1)*nFB + fb)*nSX + sx0 : -1;              // first sub-cell of the previous phase waited for
				it.depNeed = (ph > 0 ? nsx : 0) | (nsx<<8);                           // number of sub-cells waited for | number of own sub-cells
				items.push_back(it); xkey.push_back(xlo);
				for (int i = 0; i < nsx; ++i) ++cellCount[(size_t)it.cell+i];
			}
		}
	}
	// queue order: front blocks advance, phase ph runs `lag` blocks behind phase ph-1; every dependency is earlier in the queue.
	// Within a (block, phase) the items run along the front in the same direction (ascending column) in every phase, so the
	// sub-cells of the previous phase complete in the order in which their dependents are handed out.
	std::vector<int> order(items.size());
	for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
	std::stable_sort(order.begin(), order.end(), [&](int ia, int ib) {
		const FrontItem& a = items[ia]; const FrontItem& b = items[ib];
		const int ta = a.fb + lag*a.ph, tb = b.fb + lag*b.ph;
		if (ta != tb) return ta < tb;
		if (a.fb != b.fb) return a.fb < b.fb;
		if (a.ph != b.ph) return a.ph < b.ph;
		return xkey[ia] < xkey[ib];
	});
	std::vector<FrontItem> sorted(items.size());
	for (size_t i = 0; i < order.size(); ++i) sorted[i] = items[order[i]];
	items.swap(sorted);
}


// One kernel launch: one pass, or two passes whose items share one queue (interleaved, each pass in its own order).  Two
// passes never touch the same sum volume, so they are independent chains of dependencies: while an item of one waits for
// its predecessors the warps find ready work in the other.
struct FrontLaunch {
	int nPasses; FrontPassDesc pass[2];
	int fc[2], nFB[2], maxBands;
	int nChains, nCells;           // sizes of progress[] / cellDone[]
	int subCell;                   // width of a sub-cell in columns
	std::vector<FrontItem> items;
	std::vector<int> cellNeed;     // items touching each sub-cell (nCells entries)
};
inline void sgm_front_build_launch(int vw, int vh, const FrontPassDesc* pds, int nPasses, int FB, int lag, int SW, FrontLaunch& L) {
	L.subCell = SW;
	L.nPasses = nPasses; L.items.clear(); L.cellNeed.clear(); L.nChains = 0; L.nCells = 0; L.maxBands = 0;
	std::vector<FrontItem> part[2];
	for (int p = 0; p < nPasses; ++p) {
		L.pass[p] = pds[p];
		int nSX = 0; std::vector<int> cnt;
		sgm_front_build(vw, vh, pds[p], FB, lag, SW, part[p], L.nFB[p], L.maxBands, L.fc[p], nSX, cnt);
		for (FrontItem& it: part[p]) {
			it.dir = (short)(it.dir | (p<<8));
			it.chain += L.nChains; it.cell += L.nCells;
			if (it.depCell >= 0) it.depCell += L.nCells;
		}
		L.cellNeed.insert(L.cellNeed.end(), cnt.begin(), cnt.end());
		L.nChains += 4*L.maxBands; L.nCells += (int)cnt.size();
	}
	if (nPasses == 1) { L.items.swap(part[0]); return; }
	// proportional interleave: both passes reach the end of their queues together
	const size_t na = part[0].size(), nb = part[1].size();
	L.items.reserve(na+nb);
	size_t ia = 0, ib = 0;
	while (ia < na || ib < nb) {
		if (ib >= nb || (ia < na && ia*nb <= ib*na)) L.items.push_back(part[0][ia++]);
		else L.items.push_back(part[1][ib++]);
	}
}

// Pass layouts of the wave-front aggregation (b200mvs_debug.frontLayout - 1):
//   0 (default) two tilted fronts f = +-(x + 2y): {right, right-down, down, left-down} then {left, left-up, up, right-up};
//   1 four straight fronts: top-down {down, right-down, left-down}, bottom-up {up, right-up, left-up}, left-right, right-left;
//   2 eight passes of one direction each (the traffic of the per-direction kernels with the new step).
inline std::vector<FrontPassDesc> sgm_front_layout(int layout) {
	std::vector<FrontPassDesc> descs;
	if (layout == 0) {
		descs.push_back(FrontPassDesc{1, 2, 4, {1, 4, 0, 5}});
		descs.push_back(FrontPassDesc{-1, -2, 4, {3, 7, 2, 6}});
	} else if (layout == 1) {
		descs.push_back(FrontPassDesc{0, 1, 3, {0, 4, 5, 0}});
		descs.push_back(FrontPassDesc{0, -1, 3, {2, 6, 7, 0}});
		descs.push_back(FrontPassDesc{1, 0, 1, {1, 0, 0, 0}});
		descs.push_back(FrontPassDesc{-1, 0, 1, {3, 0, 0, 0}});
	} else {
		const int f[8][2] = {{0, 1}, {1, 0}, {0, -1}, {-1, 0}, {1, 1}, {-1, 1}, {1, -1}, {-1, -1}};
		for (int d = 0; d < 8; ++d) descs.push_back(FrontPassDesc{f[d][0], f[d][1], 1, {d, 0, 0, 0}});
	}
	return descs;
}
// The launches of a layout: `concurrent` pairs consecutive passes (pass 2j into volume 0, pass 2j+1 into volume 1; the caller adds
// the two volumes at the end), otherwise one pass per launch, all into volume 0.
inline std::vector<FrontLaunch> sgm_front_plan(int vw, int vh, int layout, bool concurrent, int FB, int lag, int SW = FRONT_SW) {
	const std::vector<FrontPassDesc> descs = sgm_front_layout(layout);
	const int fbSize = layout == 2 ? (1<<28) : FB;   // one-direction passes need no blocks: one item per band walks the whole path
	std::vector<FrontLaunch> out;
	const size_t per = concurrent ? 2 : 1;
	for (size_t i = 0; i < descs.size(); i += per) {
		out.emplace_back();
		sgm_front_build_launch(vw, vh, &descs[i], (int)std::min(per, descs.size()-i), fbSize, lag, SW, out.back());
	}
	return out;
}
