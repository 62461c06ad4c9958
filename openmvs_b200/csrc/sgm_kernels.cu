// sgm_kernels.cu — SGM pair matcher kernels for sm_90a.
//
// Behaviour follows SemiGlobalMatcher::Match(left, right, disparityMap, costMap)
// (libs/MVS/SemiGlobalMatcher.cpp:863-1302, SGM_SIMILARITY_WZNCC, 8 paths):
//   sgm_cost_kernel       WZNCC 7x7 cost, bilateral weights from the colour image -> uint8   :875-985
//   sgm_aggregate_kernel  one warp per scanline, disparities across lanes; the previous line
//                         lives in shared memory so that ragged per-pixel ranges [dmin,dmax)
//                         (tSGM) can be intersected and shifted freely                       :1003-1201
//   sgm_wta_kernel        first arg-min of the summed path costs                            :1272-1301
// The cost volume is ragged: pixel p owns costs[p.idx .. p.idx + (dmax-dmin)) (PixelData,
// libs/MVS/SemiGlobalMatcher.h:78-81); it is uint8, the path sum uint16 — HBM-bound integer work.
// The scanline geometry (start, step, length and number of the paths of a direction) is sgm_front_sched.h's.
#include "sgm_common.cuh"
#include "sgm_front_sched.h"
#include <string.h>
#include <stdlib.h>

namespace {

constexpr int COST_THREADS = 128;

// ---- (1) cost ----------------------------------------------------------------------------
__global__ void __launch_bounds__(COST_THREADS)
sgm_cost_kernel(const __grid_constant__ SGMParams P)
{
	extern __shared__ float2 sw[]; // {weight, tempWeight}[tap][thread]
	const int col = blockIdx.x*COST_THREADS + threadIdx.x;
	const int r = blockIdx.y;
	if (col >= P.vw) return;
	const SGMPixel p = P.px[(size_t)r*P.vw + col];
	if (!(p.dmin < p.dmax)) return;
	const int ux = col+SGM_HW, uy = r+SGM_HW;
	const float sigmaColor = -1.f/(2.f*(0.3f*255)*(0.3f*255));
	const float sigmaSpatial = -1.f/(2.f*(0.4f*7)*(0.4f*7));
	float2* w = sw + threadIdx.x;
	const uchar3 cc = P.lbgr[(size_t)uy*P.w + ux];
	float acc = 0.f, sumW = 0.f;
	#pragma unroll 1
	for (int i = -SGM_HW; i <= SGM_HW; ++i) {
		#pragma unroll
		for (int j = -SGM_HW; j <= SGM_HW; ++j) {
			const size_t o = (size_t)(uy+i)*P.w + (ux+j);
			const uchar3 pc = P.lbgr[o];
			const int d0 = abs((int)pc.x-(int)cc.x), d1 = abs((int)pc.y-(int)cc.y), d2 = abs((int)pc.z-(int)cc.z);
			const float wgt = expf(float(d0*d0+d1*d1+d2*d2)*sigmaColor + float(j*j+i*i)*sigmaSpatial);
			const float g = __ldg(P.lgray + o);
			w[((i+SGM_HW)*7+(j+SGM_HW))*COST_THREADS] = make_float2(wgt, g);
			acc += g*wgt;
			sumW += wgt;
		}
	}
	const float tm = acc/sumW;
	float normSq0 = 0.f;
	#pragma unroll 7
	for (int n = 0; n < SGM_NT; ++n) {
		float2 e = w[n*COST_THREADS];
		const float t = e.y-tm;
		e.y = e.x*t;
		normSq0 += e.y*t;
		w[n*COST_THREADS] = e;
	}
	uint8_t* costs = P.costs + p.idx;
	const float eps = 1e-3f;
	// four disparities per pass over the 7x7 taps: one LDS of a tap's weights and ten loads of a right
	// image row serve 4 x 7 products.  Columns are clamped for the loads; windows that leave the right
	// image are overwritten with 255 afterwards (SemiGlobalMatcher.cpp:959-963).
	constexpr int DCH = 4;
	#pragma unroll 1
	for (int d = p.dmin; d < p.dmax; d += DCH) {
		const int x0 = ux-SGM_HW+d;
		float sum[DCH], sumSq[DCH], nom[DCH];
		#pragma unroll
		for (int q = 0; q < DCH; ++q) { sum[q] = 0.f; sumSq[q] = 0.f; nom[q] = 0.f; }
		int col[2*SGM_HW+DCH];
		#pragma unroll
		for (int t = 0; t < 2*SGM_HW+DCH; ++t) col[t] = min(max(x0+t, 0), P.w-1);
		#pragma unroll
		for (int i = 0; i < 7; ++i) {
			const float* rp = P.rgray + (size_t)(uy-SGM_HW+i)*P.w;
			float f[2*SGM_HW+DCH];
			#pragma unroll
			for (int t = 0; t < 2*SGM_HW+DCH; ++t) f[t] = __ldg(rp + col[t]);
			#pragma unroll
			for (int j = 0; j < 7; ++j) {
				const float2 e = w[(i*7+j)*COST_THREADS];
				#pragma unroll
				for (int q = 0; q < DCH; ++q) {
					const float fv = f[j+q];
					const float fw = fv*e.x;
					sum[q] += fw;
					sumSq[q] = fmaf(fv, fw, sumSq[q]);
					nom[q] = fmaf(fv, e.y, nom[q]);
				}
			}
		}
		#pragma unroll
		for (int q = 0; q < DCH; ++q) {
			if (d+q < p.dmax) {
				const float normSq1 = sumSq[q] - sum[q]*sum[q]/sumW;
				const float ncc = nom[q]/sqrtf(normSq0*normSq1+eps);
				uint8_t cst = ncc <= 0.f ? (uint8_t)255 : (uint8_t)(int)floorf((1.f-fminf(ncc, 1.f))*255.f+.5f);
				if (x0+q < 0 || x0+q+2*SGM_HW >= P.w) cst = 255;
				costs[d-p.dmin+q] = cst;
			}
		}
	}
}

// ---- (2) path aggregation ------------------------------------------------------------------
constexpr int AGG_WARPS = 4;
constexpr int LPAD = 8;
constexpr int AGG_PD = 2;           // prefetch distance (steps) of the scanline pipeline (general kernel)
constexpr int AGG_PD_UNIFORM = 4;   // the packed uniform kernel keeps only 3 registers per stage in flight

// penalty of a path step from intensity Ip to I: P2s[|round(255 (I - Ip))|] (SemiGlobalMatcher.cpp:1009, 518-524)
__device__ __forceinline__ int path_penalty(const SGMParams& P, float I, float Ip) { return P.P2s[abs((int)floorf(255.f*(I-Ip)+.5f))]; }

// One warp walks one scanline; lane l owns disparities l, l+32, ... (NPL per lane) of every pixel.
// The scanline is a chain of dependent steps, so it is software-pipelined: the pixel record of
// step t+PD+1 and the cost / accumulator values of step t+PD are in flight while step t computes.
// ADD = false: the launch owns its sum volume (P.accums) and stores the path costs instead of adding them — the eight directions
// then run side by side on eight streams, and the winner-takes-all kernel adds the volumes (sgm_wta_kernel, nVol = 8).
template <int NPL, int PD, bool ADD>
__global__ void __launch_bounds__(AGG_WARPS*32)
sgm_aggregate_kernel(const __grid_constant__ SGMParams P, int dir)
{
	__shared__ uint16_t lines[AGG_WARPS][2][SGM_MAX_DISP+2*LPAD];
	const int warp = threadIdx.x>>5, lane = threadIdx.x&31;
	const int k = blockIdx.x*AGG_WARPS + warp;
	int x, y, dx, dy;
	if (!front_path_start(dir, k, P.vw, P.vh, x, y, dx, dy))
		return;
	int cur = 0;
	int pmin = 0, pmax = 0;     // previous range (empty at the start of a scanline)
	unsigned minPrev = 0xFFFFu; // minimum of the previous line over its whole range
	float Ip = 0.5f;
	// pixels of the scanline (one comparison per step instead of four)
	const int len = front_path_len(x, y, dx, dy, P.vw, P.vh);
	SGMPixel none; none.idx = 0; none.dmin = 0; none.dmax = 0; none.pad = 0;
	// pipeline registers: pr[i] / Ir[i] = record and intensity of pixel t+i (i <= PD),
	// c[i] / a[i] = its costs and accumulators (i < PD)
	SGMPixel pr[PD+1]; float Ir[PD+1];
	uint8_t c[PD][NPL]; uint16_t a[PD][NPL];
	#pragma unroll
	for (int i = 0; i <= PD; ++i) {
		pr[i] = none; Ir[i] = 0.f;
		const int xx = x+i*dx, yy = y+i*dy;
		if (i < len) { pr[i] = P.px[(size_t)yy*P.vw + xx]; Ir[i] = __ldg(P.lgray + (size_t)yy*P.w + xx); }
	}
	#pragma unroll
	for (int i = 0; i < PD; ++i) {
		#pragma unroll
		for (int j = 0; j < NPL; ++j) {
			const int kk = lane+32*j;
			const bool v = kk < pr[i].dmax-pr[i].dmin;
			c[i][j] = v ? P.costs[pr[i].idx+kk] : 0; a[i][j] = (ADD && v) ? P.accums[pr[i].idx+kk] : 0;
		}
	}
	for (int t = 0; t < len; ++t, x += dx, y += dy) {
		// stage A: pixel record PD+1 steps ahead
		SGMPixel pnew = none; float Inew = 0.f;
		{
			const int xx = x+(PD+1)*dx, yy = y+(PD+1)*dy;
			if (t+PD+1 < len) { pnew = P.px[(size_t)yy*P.vw + xx]; Inew = __ldg(P.lgray + (size_t)yy*P.w + xx); }
		}
		// stage B: costs and accumulators PD steps ahead
		uint8_t cn[NPL]; uint16_t an[NPL];
		#pragma unroll
		for (int j = 0; j < NPL; ++j) {
			const int kk = lane+32*j;
			const bool v = kk < pr[PD].dmax-pr[PD].dmin;
			cn[j] = v ? P.costs[pr[PD].idx+kk] : 0; an[j] = (ADD && v) ? P.accums[pr[PD].idx+kk] : 0;
		}
		uint8_t* c0 = c[0]; uint16_t* a0 = a[0];
		const float I0 = Ir[0];
		const SGMPixel p0 = pr[0];
		// stage C: this pixel
		const SGMPixel p = p0;
		if (p.dmin < p.dmax) {
			// NB: the reference reads the intensity at the valid-region coordinates (no half-window offset)
			const float I = I0;
			const int P2 = path_penalty(P, I, Ip);
			Ip = I;
			const uint16_t* Lp = lines[warp][cur] + LPAD;
			uint16_t* Ls = lines[warp][cur^1] + LPAD;
			const int imin = max(pmin, (int)p.dmin), imax = min(pmax, (int)p.dmax);
			const int num = p.dmax-p.dmin;
			uint16_t* accums = P.accums + p.idx;
			unsigned Lnew[NPL];
			if (imin >= imax) {
				#pragma unroll
				for (int j = 0; j < NPL; ++j) {
					const int kk = lane+32*j;
					Lnew[j] = 0xFFFFu;
					if (kk < num) {
						Lnew[j] = (unsigned)(c0[j]+P2);
						Ls[kk] = (uint16_t)Lnew[j];
						accums[kk] = (uint16_t)(a0[j]+Lnew[j]);
					}
				}
			} else if (p.dmin == pmin && p.dmax == pmax && num >= 4) {
				// fast path: same range as the previous pixel of the scanline (always, for fixed ranges).
				// The line is padded with 0xFFFF on both sides, so d-1 / d+1 need no range test, and
				// the minimum of the previous line was reduced when it was written.
				const int minLp = (int)minPrev;
				#pragma unroll
				for (int j = 0; j < NPL; ++j) {
					const int kk = lane+32*j;
					Lnew[j] = 0xFFFFu;
					if (kk < num) {
						const int l0 = Lp[kk], lm = Lp[kk-1], lp1 = Lp[kk+1];
						const int best = min(min(l0, min(lm, lp1)+P.P1), minLp+P2);
						Lnew[j] = (unsigned)(c0[j]+best-minLp);
						Ls[kk] = (uint16_t)Lnew[j];
						accums[kk] = (uint16_t)(a0[j]+Lnew[j]);
					}
				}
			} else {
				// general (ragged) path: min of the previous line over the intersection
				unsigned m = 0xFFFFu;
				// the intersection is at most as wide as the current range (<= 32*NPL): NPL predicated reads, no loop control
				#pragma unroll
				for (int j = 0; j < NPL; ++j) {
					const int d = imin+lane+32*j;
					if (d < imax) m = min(m, (unsigned)Lp[d-pmin]);
				}
				m = __reduce_min_sync(0xFFFFFFFFu, m); // redux.sync: one instruction instead of a 5-shuffle chain
				const int minLp = (int)m;
				#pragma unroll
				for (int j = 0; j < NPL; ++j) {
					const int kk = lane+32*j;
					Lnew[j] = 0xFFFFu;
					if (kk < num) {
						const int d = p.dmin+kk;
						// The reference takes min over dp in the intersection I of Lp(dp)+{0 | P1 | P2}.
						// Because P1 <= P2 this is min(Lp(d), Lp(d+-1)+P1, minLp+P2): if the arg-min of Lp
						// is one of d-1,d,d+1 its cheaper 0/P1 term wins anyway.  The P2 term only exists
						// when I holds a dp with |dp-d| > 1.
						const bool hasFar = (imin < d-1) || (imax > d+2);
						int best = hasFar ? minLp+P2 : 0x7FFFFFFF;
						if (d >= imin && d < imax) best = min(best, (int)Lp[d-pmin]);
						if (d-1 >= imin && d-1 < imax) best = min(best, (int)Lp[d-1-pmin]+P.P1);
						if (d+1 >= imin && d+1 < imax) best = min(best, (int)Lp[d+1-pmin]+P.P1);
						Lnew[j] = (unsigned)(c0[j]+best-minLp);
						Ls[kk] = (uint16_t)Lnew[j];
						accums[kk] = (uint16_t)(a0[j]+Lnew[j]);
					}
				}
			}
			// sentinels around the new line and its minimum, for the next step's fast path
			if (lane == 0) { Ls[-1] = 0xFFFFu; Ls[num] = 0xFFFFu; }
			unsigned mn = Lnew[0];
			#pragma unroll
			for (int j = 1; j < NPL; ++j) mn = min(mn, Lnew[j]);
			mn = __reduce_min_sync(0xFFFFFFFFu, mn); // redux.sync: one instruction instead of a 5-shuffle chain
			minPrev = mn;
			__syncwarp();
			pmin = p.dmin; pmax = p.dmax;
			cur ^= 1;
		}
		// advance the pipeline
		#pragma unroll
		for (int i = 0; i < PD; ++i) { pr[i] = pr[i+1]; Ir[i] = Ir[i+1]; }
		pr[PD] = pnew; Ir[PD] = Inew;
		#pragma unroll
		for (int i = 0; i+1 < PD; ++i) {
			#pragma unroll
			for (int j = 0; j < NPL; ++j) { c[i][j] = c[i+1][j]; a[i][j] = a[i+1][j]; }
		}
		#pragma unroll
		for (int j = 0; j < NPL; ++j) { c[PD-1][j] = cn[j]; a[PD-1][j] = an[j]; }
	}
}

// Uniform ranges (the reference's non-tSGM branch gives every pixel one global range, SemiGlobalMatcher.cpp:643-669): all valid
// pixels share [dmin, dmin+num), the count is a multiple of 4 and every pixel's slice of the volume is 4-aligned.  Lane l owns the NPL
// consecutive disparities [l*NPL, l*NPL+NPL): its costs are one packed 32-bit (NPL=4) or 64-bit (NPL=8) word, its sums one 64/128-bit
// word, d-1 / d+1 live in the lane's own registers except at the two ends (one shuffle each), and the line never touches shared
// memory.  The two uniform kernels below differ only in how a step's inputs reach the registers; PackedPath is the rest.
template <int NPL> struct Pack;
template <> struct Pack<4> { typedef uint32_t C; typedef uint2 A; };
template <> struct Pack<8> { typedef uint2 C; typedef uint4 A; };

// One warp's scanline in the packed lane layout: the lane's share of the volume, the path state and the step.
template <int NPL> struct PackedPath {
	typedef typename Pack<NPL>::C CW;
	typedef typename Pack<NPL>::A AW;
	const int lane;
	const bool active;   // num % 4 == 0 and NPL in {4, 8}: a lane is all in or all out ...
	const int nval;      // ... except with NPL = 8 and num % 8 == 4: then the last active lane owns 4 disparities
	unsigned Lp[NPL];    // the previous line
	unsigned minLp;      // its minimum over the warp
	bool havePrev;       // false before the first valid pixel of the scanline
	float Ip;            // intensity of the previous valid pixel

	__device__ __forceinline__ PackedPath(int l, int num)
		: lane(l), active(l*NPL < num), nval(min(NPL, max(0, num-l*NPL))), minLp(0xFFFFu), havePrev(false), Ip(0.5f) {
		#pragma unroll
		for (int j = 0; j < NPL; ++j) Lp[j] = 0xFFFFu;
	}

	// The lane's packed costs and sums of a slice (costs / sums: the slice's first entries, 4-byte aligned, in global memory or in
	// a shared-memory stage); zero when the pixel is not valid or the lane owns no disparity.  Word i holds disparities 4i .. 4i+3.
	__device__ __forceinline__ void load(bool valid, const uint8_t* costs, const uint16_t* sums, CW& c, AW& a) const {
		uint32_t cw[NPL/4]; uint2 aw[NPL/4];
		#pragma unroll
		for (int i = 0; i < NPL/4; ++i) { cw[i] = 0u; aw[i] = make_uint2(0u, 0u); }
		if (valid && active) {
			const uint32_t* cs = (const uint32_t*)costs + lane*(NPL/4);
			const uint2* as = (const uint2*)sums + lane*(NPL/4);
			#pragma unroll
			for (int i = 0; i < NPL/4; ++i)
				if (i == 0 || nval > 4) { cw[i] = cs[i]; aw[i] = as[i]; }
		}
		memcpy(&c, cw, sizeof(c)); memcpy(&a, aw, sizeof(a));
	}

	// One step at a valid pixel of intensity I with the lane's costs c and sums a: the new line, its sum with a stored to the
	// pixel's slice `sums`, and the line's minimum over the warp.
	__device__ __forceinline__ void step(const SGMParams& P, float I, CW c, AW a, uint16_t* sums) {
		const int P2 = path_penalty(P, I, Ip);
		Ip = I;
		uint8_t cb[NPL]; uint16_t ab[NPL];
		memcpy(cb, &c, NPL); memcpy(ab, &a, 2*NPL);
		unsigned Ln[NPL];
		if (!havePrev) {
			#pragma unroll
			for (int j = 0; j < NPL; ++j) Ln[j] = j < nval ? (unsigned)(cb[j]+P2) : 0xFFFFu;
		} else {
			const unsigned below = __shfl_up_sync(0xFFFFFFFFu, Lp[NPL-1], 1);
			const unsigned above = __shfl_down_sync(0xFFFFFFFFu, Lp[0], 1);
			const int far = (int)minLp+P2;
			#pragma unroll
			for (int j = 0; j < NPL; ++j) {
				const int lm = j > 0 ? (int)Lp[j-1] : (lane > 0 ? (int)below : 0xFFFF);
				const int lq = j < NPL-1 ? (int)Lp[j+1] : (lane < 31 ? (int)above : 0xFFFF);
				const int best = min(min((int)Lp[j], min(lm, lq)+P.P1), far);
				Ln[j] = j < nval ? (unsigned)((int)cb[j]+best-(int)minLp) : 0xFFFFu;
			}
		}
		if (active) {
			#pragma unroll
			for (int j = 0; j < NPL; ++j) ab[j] = (uint16_t)(ab[j]+(j < nval ? Ln[j] : 0u));
			uint2* dst = (uint2*)sums + lane*(NPL/4);
			#pragma unroll
			for (int i = 0; i < NPL/4; ++i)
				if (i == 0 || nval > 4) { uint2 w; memcpy(&w, ab+4*i, 8); dst[i] = w; }
		}
		unsigned mn = Ln[0];
		#pragma unroll
		for (int j = 0; j < NPL; ++j) { Lp[j] = Ln[j]; mn = min(mn, Ln[j]); }
		minLp = __reduce_min_sync(0xFFFFFFFFu, mn); // redux.sync: one instruction instead of a 5-shuffle chain
		havePrev = true;
	}
};

// Register pipeline: any 4-aligned slices.  The pixel record and intensity of step t+PD+1 and the packed words of step t+PD are in
// flight while step t computes.
template <int NPL, int PD>
__global__ void __launch_bounds__(AGG_WARPS*32)
sgm_aggregate_uniform_kernel(const __grid_constant__ SGMParams P, int dir, int dmin, int num)
{
	typedef PackedPath<NPL> Path;
	const int warp = threadIdx.x>>5, lane = threadIdx.x&31;
	const int k = blockIdx.x*AGG_WARPS + warp;
	int x, y, dx, dy;
	if (!front_path_start(dir, k, P.vw, P.vh, x, y, dx, dy))
		return;
	const int len = front_path_len(x, y, dx, dy, P.vw, P.vh);
	Path path(lane, num);
	auto valid = [](const SGMPixel& p) { return p.dmin < p.dmax; };
	SGMPixel none; none.idx = 0; none.dmin = 0; none.dmax = 0; none.pad = 0;
	SGMPixel pr[PD+1]; float Ir[PD+1];
	typename Path::CW c[PD]; typename Path::AW a[PD];
	#pragma unroll
	for (int i = 0; i <= PD; ++i) {
		pr[i] = none; Ir[i] = 0.f;
		const int xx = x+i*dx, yy = y+i*dy;
		if (i < len) { pr[i] = P.px[(size_t)yy*P.vw + xx]; Ir[i] = __ldg(P.lgray + (size_t)yy*P.w + xx); }
	}
	#pragma unroll
	for (int i = 0; i < PD; ++i) path.load(valid(pr[i]), P.costs + pr[i].idx, P.accums + pr[i].idx, c[i], a[i]);
	for (int t = 0; t < len; ++t, x += dx, y += dy) {
		SGMPixel pnew = none; float Inew = 0.f;
		{
			const int xx = x+(PD+1)*dx, yy = y+(PD+1)*dy;
			if (t+PD+1 < len) { pnew = P.px[(size_t)yy*P.vw + xx]; Inew = __ldg(P.lgray + (size_t)yy*P.w + xx); }
		}
		typename Path::CW cn; typename Path::AW an;
		path.load(valid(pr[PD]), P.costs + pr[PD].idx, P.accums + pr[PD].idx, cn, an);
		if (valid(pr[0]))
			path.step(P, Ir[0], c[0], a[0], P.accums + pr[0].idx);
		#pragma unroll
		for (int i = 0; i < PD; ++i) { pr[i] = pr[i+1]; Ir[i] = Ir[i+1]; }
		pr[PD] = pnew; Ir[PD] = Inew;
		#pragma unroll
		for (int i = 0; i+1 < PD; ++i) { c[i] = c[i+1]; a[i] = a[i+1]; }
		c[PD-1] = cn; a[PD-1] = an;
	}
}

// Bulk-copy ring (cp.async.bulk + mbarrier): every slice of the volume 16-byte aligned (num % 16 == 0, idx % 16 == 0).
// A scanline is a chain of dependent steps, so its bandwidth is set by the bytes it keeps in flight.  Every warp owns a ring of 2E
// stages in shared memory.  The steps are grouped in epochs of E: while epoch e is computed, the copies of epoch e+1
// are in flight, and when epoch e is done its E stages are refilled for epoch e+2 — lane l < E reads the
// pixel record of "its" step, posts the expected byte count on that stage's mbarrier and issues the two bulk
// copies (num cost bytes + 2*num accumulator bytes) itself, so no lane ever waits for another lane's address.
// 1.5 E stages = 9 KB (num = 128, E = 16) per warp are in flight on average without holding a register.
// The consumer side reads the record (one broadcast LDS.128), waits on the stage's mbarrier, reads its
// packed costs / accumulators from the stage (LDS.32 / LDS.64), one step ahead of the arithmetic.
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, unsigned parity) {
	unsigned ok;
	asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
		: "=r"(ok) : "r"(bar), "r"(parity) : "memory");
	return ok != 0;
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, unsigned bytes, uint32_t bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
		:: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
// shared memory of one warp's ring: 2E stages of num cost bytes and 2*num sum bytes, 2E 16-byte records, 2E mbarriers
__host__ __device__ constexpr unsigned ring_warp_bytes(int E, int num) { return 2u*E*(3u*num+16u+8u); }

template <int NPL, int E>
__global__ void __launch_bounds__(AGG_WARPS*32)
sgm_aggregate_uniform_ring_kernel(const __grid_constant__ SGMParams P, int dir, int dmin, int num)
{
	typedef typename PackedPath<NPL>::CW CW;
	typedef typename PackedPath<NPL>::AW AW;
	constexpr int RING = 2*E;
	static_assert(RING <= 32, "one lane per stage");
	extern __shared__ __align__(128) unsigned char ring_smem[];
	const int warp = threadIdx.x>>5, lane = threadIdx.x&31;
	const int k = blockIdx.x*AGG_WARPS + warp;
	int x0, y0, dx, dy;
	if (!front_path_start(dir, k, P.vw, P.vh, x0, y0, dx, dy))
		return;
	const int n = front_path_len(x0, y0, dx, dy, P.vw, P.vh);
	const unsigned stageBytes = 3u*(unsigned)num;                        // costs | accumulators
	unsigned char* base = ring_smem + (size_t)warp*ring_warp_bytes(E, num);
	unsigned char* stages = base;                                        // RING x stageBytes (16-byte aligned: num % 16 == 0)
	uint4* recs = (uint4*)(base + RING*stageBytes);                      // RING x {idx lo, idx hi, intensity, valid | parity << 1}
	uint64_t* bars = (uint64_t*)(base + RING*(stageBytes+16u));          // RING mbarriers
	if (lane < RING)
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_addr(bars+lane)) : "memory");
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");         // the init is visible to the async proxy
	__syncwarp();
	PackedPath<NPL> path(lane, num);
	unsigned phase = 0;                                                  // bit h: completions so far (mod 2) of this lane's stage in half h
	// producer: lane l < E owns step e*E+l of epoch e, stage (e & 1)*E + l
	auto issue_epoch = [&](int e) {
		if (lane < E) {
			const int t = e*E+lane, h = e&1, slot = h*E+lane;
			uint4 r = make_uint4(0u, 0u, 0u, 0u);
			if (t < n) {
				const int xx = x0+t*dx, yy = y0+t*dy;
				const SGMPixel p = P.px[(size_t)yy*P.vw + xx];
				r.z = __float_as_uint(__ldg(P.lgray + (size_t)yy*P.w + xx));
				if (p.dmin < p.dmax) {
					r.x = (unsigned)p.idx; r.y = (unsigned)(p.idx>>32);
					r.w = 1u | (((phase>>h)&1u)<<1);
					phase ^= 1u<<h;
					const uint32_t bar = smem_addr(bars+slot), dst = smem_addr(stages+(size_t)slot*stageBytes);
					asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(stageBytes) : "memory");
					bulk_load(dst, P.costs+p.idx, (unsigned)num, bar);
					bulk_load(dst+(unsigned)num, P.accums+p.idx, 2u*(unsigned)num, bar);
				}
			}
			recs[slot] = r;
		}
		__syncwarp();
	};
	// consumer: record, wait, packed words of step t
	auto fetch = [&](int t, uint4& r, CW& c, AW& a) {
		const int slot = t & (RING-1);
		r = recs[slot];
		memset(&c, 0, sizeof(c)); memset(&a, 0, sizeof(a));
		if (r.w & 1u) {
			const uint32_t bar = smem_addr(bars+slot);
			while (!mbar_try_wait(bar, (r.w>>1)&1u)) {}
			const unsigned char* st = stages+(size_t)slot*stageBytes;
			path.load(true, st, (const uint16_t*)(st+num), c, a);
		}
	};
	issue_epoch(0);
	issue_epoch(1);
	uint4 rec; CW c; AW a;
	fetch(0, rec, c, a);
	#pragma unroll 1
	for (int t = 0; t < n; ++t) {
		if (t > 0 && (t & (E-1)) == 0) {
			// epoch t/E-1 is consumed (its last stage was read into registers one step ago): refill its stages
			__syncwarp();
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			issue_epoch(t/E+1);
		}
		uint4 recN = make_uint4(0u, 0u, 0u, 0u); CW cN; AW aN;
		memset(&cN, 0, sizeof(cN)); memset(&aN, 0, sizeof(aN));
		if (t+1 < n) fetch(t+1, recN, cN, aN);
		if (rec.w & 1u)
			path.step(P, __uint_as_float(rec.z), c, a, P.accums + ((unsigned long long)rec.x | ((unsigned long long)rec.y<<32)));
		rec = recN; c = cN; a = aN;
	}
}

// ---- (3) winner takes all ------------------------------------------------------------------------
__global__ void sgm_wta_kernel(const __grid_constant__ SGMParams P, int nVol, unsigned long long volStride, const uint16_t* __restrict__ more,
	int16_t* __restrict__ disparity, uint16_t* __restrict__ cost)
{
	const int gw = (blockIdx.x*blockDim.x + threadIdx.x)>>5, lane = threadIdx.x&31;
	if (gw >= P.vw*P.vh) return;
	const SGMPixel p = P.px[gw];
	if (!(p.dmin < p.dmax)) {
		if (lane == 0 && disparity) { disparity[gw] = p.dmin; cost[gw] = 0xFFFFu; }
		return;
	}
	uint16_t* a = P.accums + p.idx;
	unsigned best = 0xFFFFFFFFu; // (value << 16) | index: the minimum is the first arg-min
	for (int k = lane; k < p.dmax-p.dmin; k += 32) {
		unsigned v = a[k];
		if (nVol > 1) {
			// the directions ran side by side into their own volumes (`more` holds volumes 1 .. nVol-1): the sum goes back to volume 0
			for (int i = 0; i+1 < nVol; ++i) v += more[(size_t)i*volStride + p.idx + k];
			v &= 0xFFFFu;
			a[k] = (uint16_t)v;
		}
		best = min(best, (v<<16) | (unsigned)k);
	}
	best = __reduce_min_sync(0xFFFFFFFFu, best); // redux.sync: one instruction instead of a 5-shuffle chain
	if (lane == 0 && disparity) { disparity[gw] = (int16_t)(p.dmin+(int)(best&0xFFFFu)); cost[gw] = (uint16_t)(best>>16); }
}

// Uniform dense volumes (num % 16 == 0, 16-byte aligned slices): 8 lanes per pixel, 16-byte loads, the arg-min carried as
// (value << 16 | index) per lane.  HBM-bound: one read of the u16 sum volume.  TWO: the wave-front aggregation ran its two
// passes side by side into two volumes; their sum is formed here (packed u16x2 adds), written back to the first volume (the
// caller's accumulated costs, read again by the sub-pixel refinement) and searched in the same pass.
template <bool TWO>
__global__ void sgm_wta_uniform_kernel(uint16_t* __restrict__ accums, const uint16_t* __restrict__ second, int nPixels, int dmin, int num,
	int16_t* __restrict__ disparity, uint16_t* __restrict__ cost)
{
	const int gp = (blockIdx.x*blockDim.x + threadIdx.x)>>3, sub = threadIdx.x&7;
	const bool live = gp < nPixels;                         // every lane stays for the full-mask shuffles
	uint16_t* a = accums + (size_t)(live ? gp : 0)*num;
	const uint16_t* b = TWO ? second + (size_t)(live ? gp : 0)*num : nullptr;
	unsigned best = 0xFFFFFFFFu;
	for (int k = sub*8; k < num; k += 64) {
		uint4 v = TWO ? __ldcg((const uint4*)(a+k)) : __ldcs((const uint4*)(a+k));
		if (TWO) {
			const uint4 u = __ldcs((const uint4*)(b+k));
			v.x = __vadd2(v.x, u.x); v.y = __vadd2(v.y, u.y); v.z = __vadd2(v.z, u.z); v.w = __vadd2(v.w, u.w);
			if (live) __stcs((uint4*)(a+k), v);
		}
		const unsigned w[4] = {v.x, v.y, v.z, v.w};
		#pragma unroll
		for (int i = 0; i < 4; ++i) {
			best = min(best, ((w[i]&0xFFFFu)<<16) | (unsigned)(k+2*i));
			best = min(best, (w[i]&0xFFFF0000u) | (unsigned)(k+2*i+1));
		}
	}
	best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, 4));
	best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, 2));
	best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, 1));
	if (live && sub == 0 && disparity) { disparity[gp] = (int16_t)(dmin+(int)(best&0xFFFFu)); cost[gp] = (uint16_t)(best>>16); }
}

// ConsistencyCrossCheck (SemiGlobalMatcher.cpp:1449-1489): every pixel reads r2l and writes only
// its own l2r entry, so the in-place update is race-free
__global__ void sgm_cross_check_kernel(int16_t* __restrict__ l2r, const int16_t* __restrict__ r2l, int w, int h, int th) {
	const int c = blockIdx.x*blockDim.x + threadIdx.x, r = blockIdx.y;
	if (c >= w) return;
	const int16_t ld = l2r[(size_t)r*w+c];
	if (ld == SGM_NO_DISP) return;
	const int vx = c+ld;
	int16_t out = ld;
	if (vx < 0 || vx >= w) out = SGM_NO_DISP;
	else {
		const int16_t rd = r2l[(size_t)r*w+vx];
		if (rd == SGM_NO_DISP || abs((int)ld+(int)rd) > th) out = SGM_NO_DISP;
	}
	l2r[(size_t)r*w+c] = out;
}

// RefineDisparityMap with SUBPIXEL_LC_BLEND (SemiGlobalMatcher.cpp:1693-1811)
__global__ void sgm_refine_kernel(const SGMPixel* __restrict__ px, const uint16_t* __restrict__ accums, int16_t* __restrict__ disparity, int n, int steps) {
	const int i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const SGMPixel p = px[i];
	if (p.dmax-p.dmin < 2) return;
	const int16_t d = disparity[i];
	// NO_DISP, and a disparity outside the pixel's range (the caller's map need not come from this volume): left unchanged
	// instead of reading another pixel's slice
	if (d == SGM_NO_DISP || d < p.dmin || d >= p.dmax) return;
	const uint16_t* a = accums + p.idx;
	const int k = d-p.dmin;
	float disp = (float)d;
	auto semi = [](uint16_t primary, uint16_t other) { return other == 0 ? 0.f : 0.5f*((float)primary/(float)other); };
	if (d == p.dmin) disp += semi(a[k], a[k+1]);
	else if (d+1 == p.dmax) disp -= semi(a[k], a[k-1]);
	else {
		const uint16_t prev = a[k-1], center = a[k], next = a[k+1];
		float off;
		if (prev == center) off = center == next ? 0.f : semi(center, next);
		else if (center == next) off = -semi(center, prev);
		else {
			const uint16_t ld = (uint16_t)(prev-center), rd = (uint16_t)(next-center);
			float x, mult;
			if (ld < rd) { x = (float)ld/(float)rd; mult = 1.f; } else { x = (float)rd/(float)ld; mult = -1.f; }
			const float cosine = 1.f-cosf(x*(float)(3.14159265358979323846/3.0));
			const float factor = 1.195f-cosf(x*(float)(3.14159265358979323846/2.3));
			off = (cosine*factor + (x*0.5f)*(1.f-factor) - 0.5f)*mult;
		}
		disp += off;
	}
	disparity[i] = (int16_t)(int)floorf(disp*steps+.5f);
}

// statistics of the pixel map (SGMMapStats), reduced per warp and combined with atomics into *out (set up by sgm_stats_init_kernel)
__global__ void sgm_map_stats_kernel(const SGMPixel* __restrict__ px, int n, unsigned long long numCosts, SGMMapStats* __restrict__ out) {
	int m = 0, lo0 = 0x7FFFFFFF, hi0 = -0x7FFFFFFF, lo1 = 0x7FFFFFFF, hi1 = -0x7FFFFFFF, al = 0, sparse = 0, oob = 0;
	for (int i = blockIdx.x*blockDim.x + threadIdx.x; i < n; i += gridDim.x*blockDim.x) {
		const SGMPixel p = px[i];
		if (p.dmin < p.dmax) {
			m = max(m, p.dmax-p.dmin);
			lo0 = min(lo0, (int)p.dmin); hi0 = max(hi0, (int)p.dmin);
			lo1 = min(lo1, (int)p.dmax); hi1 = max(hi1, (int)p.dmax);
			al |= (int)(p.idx & 15ull);
			if (p.idx != (unsigned long long)i*(unsigned long long)(p.dmax-p.dmin)) sparse = 1;
			if (p.idx+(unsigned long long)(p.dmax-p.dmin) > numCosts) oob = 1;
		} else sparse = 1;
	}
	#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		m = max(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
		lo0 = min(lo0, __shfl_xor_sync(0xFFFFFFFFu, lo0, o)); hi0 = max(hi0, __shfl_xor_sync(0xFFFFFFFFu, hi0, o));
		lo1 = min(lo1, __shfl_xor_sync(0xFFFFFFFFu, lo1, o)); hi1 = max(hi1, __shfl_xor_sync(0xFFFFFFFFu, hi1, o));
		al |= __shfl_xor_sync(0xFFFFFFFFu, al, o);
		sparse |= __shfl_xor_sync(0xFFFFFFFFu, sparse, o); oob |= __shfl_xor_sync(0xFFFFFFFFu, oob, o);
	}
	if ((threadIdx.x&31) == 0) {
		atomicMax(&out->maxNum, m); atomicMin(&out->dminLo, lo0); atomicMax(&out->dminHi, hi0);
		atomicMin(&out->dmaxLo, lo1); atomicMax(&out->dmaxHi, hi1); atomicOr(&out->idxLowBits, al);
		if (sparse) atomicOr(&out->notDense, 1);
		if (oob) atomicOr(&out->overflow, 1);
	}
}
__global__ void sgm_stats_init_kernel(SGMMapStats* out) {
	out->maxNum = 0; out->dminLo = 0x7FFFFFFF; out->dminHi = -0x7FFFFFFF; out->dmaxLo = 0x7FFFFFFF; out->dmaxHi = -0x7FFFFFFF;
	out->idxLowBits = 0; out->notDense = 0; out->overflow = 0;
}

} // namespace

template <int NPL, int E>
static cudaError_t configure_ring() {
	return cudaFuncSetAttribute(sgm_aggregate_uniform_ring_kernel<NPL, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, AGG_WARPS*ring_warp_bytes(E, NPL*32));
}
// dynamic shared memory opt-in of the SGM kernels on the current device (called by b200mvs_create; idempotent)
cudaError_t sgm_configure_device() {
	cudaError_t e;
	if ((e = configure_ring<4, 16>()) != cudaSuccess) return e;
	if ((e = configure_ring<8, 8>()) != cudaSuccess) return e;
	return cudaFuncSetAttribute(sgm_cost_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)SGM_NT*COST_THREADS*sizeof(float2)));
}
cudaError_t sgm_launch_map_stats(const SGMPixel* px, int n, unsigned long long numCosts, SGMMapStats* out, cudaStream_t s) {
	int dev = 0, sms = 0;
	cudaError_t e = cudaGetDevice(&dev);
	if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
	if (e != cudaSuccess) return e;
	sgm_stats_init_kernel<<<1, 1, 0, s>>>(out);
	sgm_map_stats_kernel<<<sms*4, 256, 0, s>>>(px, n, numCosts, out);
	return cudaGetLastError();
}
// blocks of the per-direction kernels: one warp per scanline
static int aggregate_grid(const SGMParams& P, int dir) { return (front_path_count(dir, P.vw, P.vh)+AGG_WARPS-1)/AGG_WARPS; }
// uniform-range fast path: every valid pixel has the range [dmin, dmin+num), num % 4 == 0, 4-aligned slices;
// ring: slices are 16-byte aligned (num % 16 == 0, idx % 16 == 0, aligned base pointers) -> bulk-copy ring kernel
template <int NPL, int E>
static cudaError_t launch_ring(const SGMParams& P, int dir, int dmin, int num, int grid, cudaStream_t s) {
	sgm_aggregate_uniform_ring_kernel<NPL, E><<<grid, AGG_WARPS*32, AGG_WARPS*ring_warp_bytes(E, num), s>>>(P, dir, dmin, num);
	return cudaGetLastError();
}
cudaError_t sgm_launch_aggregate_uniform(const SGMParams& P, int dir, int dmin, int num, bool ring, cudaStream_t s) {
	const int grid = aggregate_grid(P, dir);
	if (ring && (num & 15) == 0)
		return num <= 128 ? launch_ring<4, 16>(P, dir, dmin, num, grid, s) : launch_ring<8, 8>(P, dir, dmin, num, grid, s);
	if (num <= 128) sgm_aggregate_uniform_kernel<4, AGG_PD_UNIFORM><<<grid, AGG_WARPS*32, 0, s>>>(P, dir, dmin, num);
	else sgm_aggregate_uniform_kernel<8, AGG_PD_UNIFORM><<<grid, AGG_WARPS*32, 0, s>>>(P, dir, dmin, num);
	return cudaGetLastError();
}
cudaError_t sgm_launch_cost(const SGMParams& P, cudaStream_t s) {
	const size_t smem = (size_t)SGM_NT*COST_THREADS*sizeof(float2);
	dim3 grid((P.vw+COST_THREADS-1)/COST_THREADS, P.vh);
	sgm_cost_kernel<<<grid, COST_THREADS, smem, s>>>(P);
	return cudaGetLastError();
}
template <bool ADD>
static void launch_aggregate(const SGMParams& P, int dir, int grid, cudaStream_t s) {
	const int npl = (P.maxNumDisp+31)/32;
	if (npl <= 1) sgm_aggregate_kernel<1, AGG_PD, ADD><<<grid, AGG_WARPS*32, 0, s>>>(P, dir);
	else if (npl <= 2) sgm_aggregate_kernel<2, AGG_PD, ADD><<<grid, AGG_WARPS*32, 0, s>>>(P, dir);
	else if (npl <= 4) sgm_aggregate_kernel<4, AGG_PD, ADD><<<grid, AGG_WARPS*32, 0, s>>>(P, dir);
	else sgm_aggregate_kernel<8, AGG_PD, ADD><<<grid, AGG_WARPS*32, 0, s>>>(P, dir);
}
// store: P.accums is this direction's own volume, written without reading it (see sgm_aggregate_kernel)
cudaError_t sgm_launch_aggregate(const SGMParams& P, int dir, bool store, cudaStream_t s) {
	const int grid = aggregate_grid(P, dir);
	if (store) launch_aggregate<false>(P, dir, grid, s); else launch_aggregate<true>(P, dir, grid, s);
	return cudaGetLastError();
}
// nVol > 1: P.accums += the nVol-1 volumes at more + i*volStride first (disparity / cost may then be null: the addition alone)
cudaError_t sgm_launch_wta(const SGMParams& P, int nVol, unsigned long long volStride, const uint16_t* more, int16_t* disparity, uint16_t* cost, cudaStream_t s) {
	const long long threads = (long long)P.vw*P.vh*32;
	sgm_wta_kernel<<<(unsigned)((threads+255)/256), 256, 0, s>>>(P, nVol, volStride, more, disparity, cost);
	return cudaGetLastError();
}

// dense uniform volume: every pixel valid, slice of pixel i at i*num
// second != nullptr: accums += second first (disparity / cost may then be null: the addition alone)
cudaError_t sgm_launch_wta_uniform(const SGMParams& P, const uint16_t* second, int dmin, int num, int16_t* disparity, uint16_t* cost, cudaStream_t s) {
	const long long threads = (long long)P.vw*P.vh*8;
	if (second) sgm_wta_uniform_kernel<true><<<(unsigned)((threads+255)/256), 256, 0, s>>>(P.accums, second, P.vw*P.vh, dmin, num, disparity, cost);
	else sgm_wta_uniform_kernel<false><<<(unsigned)((threads+255)/256), 256, 0, s>>>(P.accums, nullptr, P.vw*P.vh, dmin, num, disparity, cost);
	return cudaGetLastError();
}
cudaError_t sgm_launch_cross_check(int16_t* l2r, const int16_t* r2l, int w, int h, int th, cudaStream_t s) {
	sgm_cross_check_kernel<<<dim3((w+255)/256, h), 256, 0, s>>>(l2r, r2l, w, h, th);
	return cudaGetLastError();
}
cudaError_t sgm_launch_refine(const SGMPixel* px, const uint16_t* accums, int16_t* disparity, int n, int steps, cudaStream_t s) {
	sgm_refine_kernel<<<(n+255)/256, 256, 0, s>>>(px, accums, disparity, n, steps);
	return cudaGetLastError();
}
