// sgm_host.cu — host side of the SGM entry points of the C-ABI: the pair matcher (SemiGlobalMatcher::Match, cost / aggregation
// / winner-takes-all), cross-check, sub-pixel refinement and the hierarchical (tSGM) level loop.
#include "host_ctx.h"
#include "sgm_common.cuh"
#include "resize_common.cuh"

namespace {

// SGM path aggregation with the wave-front kernel (sgm_front.cu).  Pass layouts (b200mvs_debug.frontLayout, 0 = auto = 1):
//   1 two tilted fronts f = +-(x + 2y): {right, right-down, down, left-down} and {left, left-up, up, right-up};
//   2 four straight fronts: top-down {down, right-down, left-down}, bottom-up {up, right-up, left-up}, left-right, right-left;
//   3 eight passes of one direction each (the traffic of the per-direction kernels with the new step).
// With a `second` volume, consecutive passes share a launch: pass 2j accumulates into the caller's volume, pass 2j+1 into
// `second`, and the caller adds the two (the winner-takes-all kernel does).  Without one, every pass has a launch of its own.
int sgm_aggregate_fronts(b200mvs_ctx* ctx, const SGMParams& P, int num, uint16_t* second, cudaStream_t s) {
	const b200mvs_debug& D = ctx->dbg;
	const int layout = std::min(std::max(D.frontLayout-1, 0), 2);
	const bool concurrent = second != nullptr;
	const int FB = D.frontBlock > 0 ? D.frontBlock : 32;   // fronts per block: larger blocks widen the window of the sum volume kept in the L2
	// frontLag = lag + 1.  The sub-cell dependencies make every lag legal.  A larger lag lets more blocks be in flight at once, but
	// the window of blocks between a block's first and last phase then outgrows the L2 and the sums go to DRAM and back; lag 0
	// leaves the resident warps all holding items of one block, waiting for each other.  Default: lag 1.
	const int lag = D.frontLag > 0 ? D.frontLag-1 : 1;
	const int vw = P.vw, vh = P.vh;
	// sub-cell width: one lane polls one counter, and a band at an image corner can span the whole width: at most 30 sub-cell columns
	const int SW = std::max(D.frontSubCell >= 16 ? D.frontSubCell : FRONT_SW, (vw+29)/30);
	const int key[6] = {vw, vh, layout, FB, lag | (SW<<8), concurrent ? 2 : 1};
	if (memcmp(key, ctx->sgFrontKey, sizeof(key)) != 0) {
		ctx->sgFront.clear();
		std::vector<FrontLaunch> plan = sgm_front_plan(vw, vh, layout, concurrent, FB, lag, SW);
		ctx->sgFront.resize(plan.size());
		for (size_t i = 0; i < plan.size(); ++i) {
			b200mvs_ctx::FrontPass& fp = ctx->sgFront[i];
			CK(fp.items.reserve(plan[i].items.size()*sizeof(FrontItem)));
			CK(cudaMemcpyAsync(fp.items.p, plan[i].items.data(), plan[i].items.size()*sizeof(FrontItem), cudaMemcpyHostToDevice, s));
			CK(fp.need.reserve(std::max<size_t>(1, plan[i].cellNeed.size())*sizeof(int)));
			CK(cudaMemcpyAsync(fp.need.p, plan[i].cellNeed.data(), plan[i].cellNeed.size()*sizeof(int), cudaMemcpyHostToDevice, s));
			CK(cudaStreamSynchronize(s)); // the pageable source vectors are released below
			fp.nItems = (int)plan[i].items.size();
			plan[i].items.clear(); plan[i].items.shrink_to_fit(); plan[i].cellNeed.clear(); plan[i].cellNeed.shrink_to_fit();
			fp.launch = plan[i];
		}
		CK(cudaStreamSynchronize(s)); // the pageable source vectors die with `plan`
		memcpy(ctx->sgFrontKey, key, sizeof(key));
	}
	const int maxPaths = vw+vh+8;
	int maxCtl = 0;
	for (auto& fp: ctx->sgFront) maxCtl = std::max(maxCtl, fp.launch.nChains + fp.launch.nCells);
	CK(ctx->sgFrontCtl.reserve((size_t)(4+maxCtl)*sizeof(int)));
	CK(ctx->sgFrontState.reserve((size_t)8*maxPaths*num*sizeof(uint16_t)));
	CK(ctx->sgFrontMeta.reserve((size_t)8*maxPaths*sizeof(float2)));
	int* ctl = ctx->sgFrontCtl.as<int>();
	// resident CTAs: the queue needs no particular number; frontCtas = CTAs per SM, frontDepth = ring slots per warp (8 default, 4)
	const int pd = D.frontDepth == 4 ? 4 : 8;
	int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
	const int perSm = std::min(sgm_front_blocks_per_sm(num, pd), D.frontCtas > 0 ? D.frontCtas : 2);
	const int blocks = sms*perSm;
	const int FBeff = layout == 2 ? (1<<28) : FB;
	for (size_t i = 0; i < ctx->sgFront.size(); ++i) {
		b200mvs_ctx::FrontPass& fp = ctx->sgFront[i];
		const FrontLaunch& L = fp.launch;
		// [ticket, error, -, - | progress | cellDone]; the error word survives the launches of one call
		if (i == 0) CK(cudaMemsetAsync(ctl, 0, (size_t)(4+maxCtl)*sizeof(int), s));
		else { CK(cudaMemsetAsync(ctl, 0, sizeof(int), s)); CK(cudaMemsetAsync(ctl+4, 0, (size_t)maxCtl*sizeof(int), s)); }
		FrontArgs A; memset(&A, 0, sizeof(A));
		A.items = fp.items.as<FrontItem>(); A.nItems = fp.nItems;
		A.ticket = ctl; A.error = ctl+1; A.progress = ctl+4; A.cellDone = ctl+4+L.nChains; A.cellNeed = fp.need.as<int>();
		A.state = ctx->sgFrontState.as<uint16_t>(); A.meta = ctx->sgFrontMeta.as<float2>(); A.maxPaths = maxPaths;
		A.FB = FBeff; A.num = num;
		for (int p = 0; p < L.nPasses; ++p) {
			A.fa[p] = L.pass[p].fa; A.fb[p] = L.pass[p].fb; A.fc[p] = L.fc[p];
			A.storePhase0[p] = i == 0 ? 1 : 0;
			A.sum[p] = p == 0 ? P.accums : second;
		}
		CK(sgm_front_launch(P, A, blocks, pd, s)); ++ctx->launches;
	}
	return B200MVS_OK;
}

// The kernels of one match (sgm_plan).
struct SGMPlan {
	enum Aggregation { FRONTS, UNIFORM_RING, UNIFORM, RAGGED_STREAMS, RAGGED } agg;
	bool tcCost;     // the tensor-core cost kernel (sgm_cost_tc.cu), else sgm_cost_kernel
	bool denseWta;   // sgm_wta_uniform_kernel, else sgm_wta_kernel
	int volumes;     // sum volumes the aggregation leaves for the winner-takes-all to add: 1, 2 (paired wave-front passes) or 8
};

// Picks the kernels from the pixel map's statistics, the debug switches (b200mvs_debug.sgmAggregation / sgmCost / frontSerial),
// the 16-byte alignment of the cost and sum volumes' base pointers and the largest P2.
SGMPlan sgm_plan(const SGMMapStats& st, const b200mvs_debug& D, bool costsAligned, bool accumsAligned, int maxP2, uint64_t numCosts) {
	const int mode = D.sgmAggregation;
	// one global range (the non-tSGM branch): packed, shared-memory-free aggregation kernels
	const bool uniform = st.maxNum >= 4 && st.dminLo == st.dminHi && st.dmaxLo == st.dmaxHi && (st.maxNum & 3) == 0 && (st.idxLowBits & 3) == 0
		&& mode != 1;
	// ... every pixel valid, pixel i's slice at i*num, num % 16 == 0
	const bool dense = uniform && (st.maxNum & 15) == 0 && !st.notDense;
	// every slice 16-byte aligned: bulk-copy ring kernel (one launch per direction)
	const bool ring = uniform && (st.maxNum & 15) == 0 && st.idxLowBits == 0 && costsAligned && accumsAligned && mode != 2;
	// dense volume of a supported width: wave-front kernel (fused directions) — the default
	// (its step carries P2 + the previous line's minimum in 16 bits: P2 <= 16000; sums of eight paths overflow far earlier)
	const bool front = ring && !st.notDense && sgm_front_supports(st.maxNum) && maxP2 <= 16000 && (mode == 0 || mode == 4);
	SGMPlan p;
	// ragged (tSGM) ranges: one volume per direction (RAGGED_STREAMS) while the seven extra volumes take at most 3.5 GiB, else
	// the eight directions add into one volume in turn
	p.agg = front ? SGMPlan::FRONTS : ring ? SGMPlan::UNIFORM_RING : uniform ? SGMPlan::UNIFORM
		: numCosts <= (1ull<<28) ? SGMPlan::RAGGED_STREAMS : SGMPlan::RAGGED;
	// dense volume with one range of 64 / 128 / 192 / 256 disparities: the banded-GEMM cost kernel on the tensor cores
	p.tcCost = dense && costsAligned && sgm_cost_tc_supports(st.maxNum) && D.sgmCost != 1;
	p.denseWta = dense && accumsAligned;
	// every wave-front layout has at least two passes, so unless frontSerial is set two of them share a launch
	p.volumes = front ? (D.frontSerial ? 1 : 2) : p.agg == SGMPlan::RAGGED_STREAMS ? 8 : 1;
	return p;
}

} // namespace

extern "C" {

void b200mvs_sgm_default_params(b200mvs_sgm_params* p) { p->P1 = 3; p->P2 = 4; p->P2alpha = 14.f; p->P2beta = 38.f; }

int b200mvs_sgm_match_device(b200mvs_ctx* ctx, const float* leftGray, const uint8_t* leftBGR, const float* rightGray,
	int width, int height, const b200mvs_sgm_pixel* pixels, uint64_t numCosts, const b200mvs_sgm_params* prm,
	int stages, uint8_t* costs, uint16_t* accums, int16_t* disparity, uint16_t* cost, void* stream, b200mvs_stats* stats)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!leftGray || !leftBGR || !rightGray || !pixels || width <= 6 || height <= 6 || numCosts == 0)
		return fail(ctx, B200MVS_ERR_ARG, "sgm: null image/pixel map or image too small");
	if ((stages & 4) && (!disparity || !cost))
		return fail(ctx, B200MVS_ERR_ARG, "sgm: null output map");
	b200mvs_sgm_params def; b200mvs_sgm_default_params(&def);
	if (!prm) prm = &def;
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	SGMParams P; memset(&P, 0, sizeof(P));
	P.lgray = leftGray; P.lbgr = (const uchar3*)leftBGR; P.rgray = rightGray;
	P.w = width; P.h = height; P.vw = width-6; P.vh = height-6;
	P.px = (const SGMPixel*)pixels;
	P.P1 = prm->P1;
	int minP2 = 1<<30, maxP2 = 0;
	for (int i = 0; i < 256; ++i) {
		// GenerateP2s (libs/MVS/SemiGlobalMatcher.cpp:518-524)
		P.P2s[i] = (uint16_t)(int)std::floor(prm->P2*(1.f+prm->P2alpha*std::exp(-float(i)*float(i)/(2.f*prm->P2beta*prm->P2beta)))+.5f);
		minP2 = std::min(minP2, (int)P.P2s[i]); maxP2 = std::max(maxP2, (int)P.P2s[i]);
	}
	if (prm->P1 < 0 || prm->P1 > minP2)
		return fail(ctx, B200MVS_ERR_ARG, "sgm: needs 0 <= P1 <= min(P2s)");
	if (!costs) { CK(ctx->sgCosts.reserve(numCosts)); costs = ctx->sgCosts.as<uint8_t>(); }
	if (!accums) { CK(ctx->sgAccums.reserve(numCosts*sizeof(uint16_t))); accums = ctx->sgAccums.as<uint16_t>(); }
	P.costs = costs; P.accums = accums;
	const auto t0 = std::chrono::steady_clock::now();
	ctx->launches = 0;
	SGMMapStats st = {};
	SGMPlan plan = {};
	if (stats) CK(cudaEventRecord(ctx->ev0, s));
	if (stages & 7) {
		CK(ctx->sgMax.reserve(sizeof(SGMMapStats)));
		CK(sgm_launch_map_stats(P.px, P.vw*P.vh, numCosts, ctx->sgMax.as<SGMMapStats>(), s)); ctx->launches += 2;
		CK(cudaMemcpyAsync(&st, ctx->sgMax.p, sizeof(st), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		if (st.overflow)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: a pixel's slice [idx, idx+dmax-dmin) ends beyond numCosts");
		// the warp-per-scanline kernel keeps one line of at most SGM_MAX_DISP values
		if (st.maxNum > SGM_MAX_DISP)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: more than 256 disparities per pixel");
		P.maxNumDisp = st.maxNum;
		plan = sgm_plan(st, ctx->dbg, !((uintptr_t)P.costs & 15), !((uintptr_t)P.accums & 15), maxP2, numCosts);
		if (ctx->dbg.sgmAggregation == 4 && plan.agg != SGMPlan::FRONTS)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: the wave-front kernel needs a dense volume with one range of 64, 128 or 256 disparities");
	}
	if (stages & 1) {
		if (ctx->dbg.sgmCost == 2 && !plan.tcCost)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: the tensor-core cost kernel needs a dense volume with one range of 64, 128, 192 or 256 disparities");
		if (plan.tcCost) { CK(sgm_cost_tc_launch(P, st.dminLo, st.maxNum, s)); ctx->launches += (st.maxNum+127)/128; }
		else { CK(sgm_launch_cost(P, s)); ++ctx->launches; }
	}
	// the sum volumes the winner-takes-all adds: accums, then nVol-1 more at `more` (ctx->sgAccums2)
	const int nVol = (stages & 2) ? plan.volumes : 1;
	uint16_t* more = nullptr;
	if ((stages & 2) && plan.agg == SGMPlan::FRONTS) {
		if (nVol == 2) {
			CK(ctx->sgAccums2.reserve((size_t)P.vw*P.vh*st.maxNum*sizeof(uint16_t)));
			more = ctx->sgAccums2.as<uint16_t>();
		}
		const int rc = sgm_aggregate_fronts(ctx, P, st.maxNum, more, s);
		if (rc) return rc;
	} else
	if ((stages & 2) && plan.agg == SGMPlan::RAGGED_STREAMS) {
		// ragged (tSGM) ranges: a direction has only 1000-3000 scanlines, one warp each — far too few to fill the GPU.  The eight
		// directions run side by side on eight streams, each STORING its path costs into a volume of its own (no memset, no
		// read-modify-write, no races); the winner-takes-all kernel adds the volumes.
		CK(ctx->sgAccums2.reserve((size_t)7*numCosts*sizeof(uint16_t)));
		more = ctx->sgAccums2.as<uint16_t>();
		if (!ctx->sgSide[0]) {
			for (int i = 0; i < 7; ++i) { CK(cudaStreamCreateWithFlags(&ctx->sgSide[i], cudaStreamNonBlocking)); CK(cudaEventCreateWithFlags(&ctx->sgJoin[i], cudaEventDisableTiming)); }
			CK(cudaEventCreateWithFlags(&ctx->sgFork, cudaEventDisableTiming));
		}
		CK(cudaEventRecord(ctx->sgFork, s));
		for (int dir = 0; dir < 8; ++dir) {
			SGMParams Pd = P;
			cudaStream_t sd = s;
			if (dir > 0) {
				Pd.accums = more + (size_t)(dir-1)*numCosts;
				sd = ctx->sgSide[dir-1];
				CK(cudaStreamWaitEvent(sd, ctx->sgFork, 0));
			}
			CK(sgm_launch_aggregate(Pd, dir, true, sd));
			++ctx->launches;
			if (dir > 0) { CK(cudaEventRecord(ctx->sgJoin[dir-1], sd)); CK(cudaStreamWaitEvent(s, ctx->sgJoin[dir-1], 0)); }
		}
	} else
	if (stages & 2) {
		CK(cudaMemsetAsync(accums, 0, numCosts*sizeof(uint16_t), s));
		for (int dir = 0; dir < 8; ++dir) {
			if (plan.agg == SGMPlan::RAGGED) CK(sgm_launch_aggregate(P, dir, false, s));
			else CK(sgm_launch_aggregate_uniform(P, dir, st.dminLo, st.maxNum, plan.agg == SGMPlan::UNIFORM_RING, s));
			++ctx->launches;
		}
	}
	if (stages & 2) ctx->sgLastPx = (accums == ctx->sgAccums.as<uint16_t>()) ? (const void*)pixels : nullptr;
	// the winner-takes-all; without stage 4, several volumes are still added into accums (no disparity / cost maps)
	if ((stages & 4) || nVol > 1) {
		int16_t* d = (stages & 4) ? disparity : nullptr;
		uint16_t* c = (stages & 4) ? cost : nullptr;
		if (plan.denseWta) CK(sgm_launch_wta_uniform(P, more, st.dminLo, st.maxNum, d, c, s));
		else CK(sgm_launch_wta(P, nVol, numCosts, more, d, c, s));
		++ctx->launches;
	}
	if (stats) {
		CK(cudaEventRecord(ctx->ev1, s));
		CK(cudaStreamSynchronize(s));
		const int rc = fill_stats(ctx, stats, t0, 1);
		if (rc) return rc;
		if ((stages & 2) && plan.agg == SGMPlan::FRONTS) {
			// the wave-front kernel flags a dependency wait that timed out (never in a correct schedule): the stream is idle here
			int err = 0;
			CK(cudaMemcpy(&err, ctx->sgFrontCtl.as<int>()+1, sizeof(int), cudaMemcpyDeviceToHost));
			if (err) return fail(ctx, B200MVS_ERR_CUDA, "sgm: the wave-front aggregation timed out waiting for a predecessor");
		}
	}
	return B200MVS_OK;
}

int b200mvs_sgm_match(b200mvs_ctx* ctx, const float* leftGray, const uint8_t* leftBGR, const float* rightGray,
	int width, int height, const b200mvs_sgm_pixel* pixels, uint64_t numCosts, const b200mvs_sgm_params* prm,
	int16_t* disparity, uint16_t* cost, b200mvs_stats* stats)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!leftGray || !leftBGR || !rightGray || !pixels || !disparity || !cost || width <= 6 || height <= 6)
		return fail(ctx, B200MVS_ERR_ARG, "sgm: null pointer or image too small");
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = ctx->stream;
	const auto t0 = std::chrono::steady_clock::now();
	const size_t n = (size_t)width*height, nv = (size_t)(width-6)*(height-6);
	CK(ctx->sgL.reserve(n*4)); CK(ctx->sgR.reserve(n*4)); CK(ctx->sgC.reserve(n*3)); CK(ctx->sgPx.reserve(nv*sizeof(SGMPixel)));
	CK(ctx->sgDisp.reserve(nv*2)); CK(ctx->sgCost.reserve(nv*2));
	CK(cudaMemcpyAsync(ctx->sgL.p, leftGray, n*4, cudaMemcpyHostToDevice, s));
	CK(cudaMemcpyAsync(ctx->sgR.p, rightGray, n*4, cudaMemcpyHostToDevice, s));
	CK(cudaMemcpyAsync(ctx->sgC.p, leftBGR, n*3, cudaMemcpyHostToDevice, s));
	CK(cudaMemcpyAsync(ctx->sgPx.p, pixels, nv*sizeof(SGMPixel), cudaMemcpyHostToDevice, s));
	b200mvs_stats st; // the match records ev0 / ev1 around its kernels only when asked for statistics
	int rc = b200mvs_sgm_match_device(ctx, ctx->sgL.as<float>(), ctx->sgC.as<uint8_t>(), ctx->sgR.as<float>(), width, height,
		(const b200mvs_sgm_pixel*)ctx->sgPx.p, numCosts, prm, 7, nullptr, nullptr, ctx->sgDisp.as<int16_t>(), ctx->sgCost.as<uint16_t>(), s, &st);
	if (rc) return rc;
	CK(cudaMemcpyAsync(disparity, ctx->sgDisp.p, nv*2, cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(cost, ctx->sgCost.p, nv*2, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	if (stats) return fill_stats(ctx, stats, t0, 1, n*11+nv*sizeof(SGMPixel), nv*4);
	return B200MVS_OK;
}

int b200mvs_sgm_cross_check_device(b200mvs_ctx* ctx, int16_t* l2r, const int16_t* r2l, int width, int height, int thCross, void* stream) {
	if (!ctx || !l2r || !r2l || width <= 0 || height <= 0 || thCross < 0) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	CK(sgm_launch_cross_check(l2r, r2l, width, height, thCross, stream_of(ctx, stream)));
	return B200MVS_OK;
}

int b200mvs_sgm_refine_device(b200mvs_ctx* ctx, const b200mvs_sgm_pixel* pixels, const uint16_t* accums, int16_t* disparity,
	int nPixels, int subpixelSteps, void* stream)
{
	if (!ctx || !pixels || !disparity || nPixels <= 0) return B200MVS_ERR_ARG;
	if (!accums) {
		// the accumulated costs of the last match on this context: only valid for the pixel map they were computed for
		accums = ctx->sgAccums.as<uint16_t>();
		if (!accums || ctx->sgLastPx != (const void*)pixels)
			return fail(ctx, B200MVS_ERR_ARG, "sgm refine: no accumulated costs of a match with this pixel map on the context");
	}
	if (subpixelSteps <= 1) return B200MVS_OK;
	CK(cudaSetDevice(ctx->device));
	CK(sgm_launch_refine((const SGMPixel*)pixels, accums, disparity, nPixels, subpixelSteps, stream_of(ctx, stream)));
	return B200MVS_OK;
}

// ---- hierarchical (tSGM) matching ----------------------------------------------------------------
static int tsgm_levels(int width, int height, int minResolution, int& n, int* ws, int* hs, int& iw, int& ih) {
	if (width <= 6 || height <= 6 || minResolution < 0) return B200MVS_ERR_ARG;
	double scale = 1;
	if (minResolution > 0) {
		// Image8U::computeMaxResolution(w, h, level = 8, minResolution) (libs/Common/Types.inl:2459-2477)
		const unsigned imageSize = (unsigned)std::max(width, height), minSize = (unsigned)minResolution;
		unsigned level = 8;
		if ((imageSize >> level) < minSize) {
			level = 0;
			while ((imageSize >> (level+1)) >= minSize) ++level;
		}
		scale = 1.0/std::max(2.0, std::pow(2.0, (double)level));
	}
	n = 0;
	do {
		// computeResize / cv::resize(..., Size(), scale, scale): saturate_cast<int>(size * scale) rounds to nearest even
		ws[n] = (int)std::nearbyint(width*scale); hs[n] = (int)std::nearbyint(height*scale);
		if (ws[n] <= 6 || hs[n] <= 6) return B200MVS_ERR_ARG;
		++n;
	} while ((scale *= 2) < 1+1e-9 && n < B200MVS_SGM_MAX_LEVELS);
	iw = (int)std::nearbyint(ws[0]*0.5)-6; ih = (int)std::nearbyint(hs[0]*0.5)-6;
	if (iw < 1 || ih < 1) return B200MVS_ERR_ARG;
	// Disparity2RangeMap reads the mask of the 2x grid at (2r+3, 2c+3) and needs the grid to end beyond column 2w+3
	for (int k = 0, pw = iw, ph = ih; minResolution > 0 && k < n; pw = ws[k]-6, ph = hs[k]-6, ++k)
		if (2*pw+3 >= ws[k]-6 || 2*ph+1 >= hs[k]-6) return B200MVS_ERR_ARG;
	return B200MVS_OK;
}

int b200mvs_sgm_levels(int width, int height, int minResolution, int* numLevels, int* levelWidths, int* levelHeights, int* initWidth, int* initHeight) {
	int n = 0, ws[B200MVS_SGM_MAX_LEVELS], hs[B200MVS_SGM_MAX_LEVELS], iw = 0, ih = 0;
	const int rc = tsgm_levels(width, height, minResolution, n, ws, hs, iw, ih);
	if (rc) return rc;
	if (numLevels) *numLevels = n;
	for (int k = 0; k < n; ++k) { if (levelWidths) levelWidths[k] = ws[k]; if (levelHeights) levelHeights[k] = hs[k]; }
	if (initWidth) *initWidth = iw;
	if (initHeight) *initHeight = ih;
	return B200MVS_OK;
}

static int tsgm_range_map(b200mvs_ctx* ctx, const int16_t* disparity, int width, int height, const uint8_t* mask, int mw, int mh,
	int minNumDisp, int minNumDispInvalid, b200mvs_sgm_pixel* pixels, uint64_t* numCosts, cudaStream_t s)
{
	const size_t n2 = (size_t)mw*mh;
	CK(ctx->ts[b200mvs_ctx::TS_RANGES].reserve((size_t)width*height*sizeof(short2)));
	CK(ctx->ts[b200mvs_ctx::TS_SCAN].reserve(tsgm_range_map_scratch(n2)));
	CK(ctx->ts[b200mvs_ctx::TS_SMALL].reserve(64));
	unsigned long long* total = ctx->ts[b200mvs_ctx::TS_SMALL].as<unsigned long long>();
	CK(tsgm_launch_range_map(disparity, width, height, mask, mw, mh, minNumDisp, minNumDispInvalid,
		ctx->ts[b200mvs_ctx::TS_RANGES].as<short2>(), (SGMPixel*)pixels, ctx->ts[b200mvs_ctx::TS_SCAN].p, total, s));
	// the size of the volume: one 8-byte read per pixel map (the match that follows sizes its scratch with it)
	unsigned long long num = 0;
	CK(cudaMemcpyAsync(&num, total, sizeof(num), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	*numCosts = num;
	return B200MVS_OK;
}

int b200mvs_sgm_range_map_device(b200mvs_ctx* ctx, const int16_t* disparity, int width, int height, const uint8_t* mask,
	int maskWidth, int maskHeight, int minNumDisp, int minNumDispInvalid, b200mvs_sgm_pixel* pixels, uint64_t* numCosts, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!disparity || !mask || !pixels || !numCosts || width <= 0 || height <= 0)
		return fail(ctx, B200MVS_ERR_ARG, "range map: null pointer or empty map");
	if (maskWidth <= 2*width+3 || maskHeight <= 2*height+1 || (size_t)maskWidth*maskHeight >= (1u<<31))
		return fail(ctx, B200MVS_ERR_ARG, "range map: the 2x grid must extend beyond (2 width + 3, 2 height + 1)");
	CK(cudaSetDevice(ctx->device));
	return tsgm_range_map(ctx, disparity, width, height, mask, maskWidth, maskHeight, minNumDisp, minNumDispInvalid, pixels, numCosts,
		stream_of(ctx, stream));
}

int b200mvs_sgm_flip_direction_device(b200mvs_ctx* ctx, const int16_t* l2r, int16_t* r2l, int width, int height, void* stream) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!l2r || !r2l || l2r == r2l || width <= 0 || height <= 0 || width >= 65535)
		return fail(ctx, B200MVS_ERR_ARG, "flip direction: null or aliased maps, or a width outside [1, 65534]");
	CK(cudaSetDevice(ctx->device));
	CK(ctx->ts[b200mvs_ctx::TS_KEYS].reserve((size_t)width*height*sizeof(unsigned)));
	CK(tsgm_launch_flip(l2r, r2l, width, height, ctx->ts[b200mvs_ctx::TS_KEYS].as<unsigned>(), stream_of(ctx, stream)));
	return B200MVS_OK;
}

int b200mvs_sgm_upscale_mask_device(b200mvs_ctx* ctx, const uint8_t* mask, int width, int height, uint8_t* mask2x, int width2x, int height2x, void* stream) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!mask || !mask2x || mask == mask2x || width <= 0 || height <= 0 || width2x <= 0 || height2x <= 0)
		return fail(ctx, B200MVS_ERR_ARG, "upscale mask: null or aliased masks, or an empty size");
	CK(cudaSetDevice(ctx->device));
	CK(tsgm_launch_upscale_mask(mask, width, height, mask2x, width2x, height2x, stream_of(ctx, stream)));
	return B200MVS_OK;
}

int b200mvs_sgm_extract_mask_device(b200mvs_ctx* ctx, const int16_t* disparity, uint8_t* mask, int width, int height, int thValid, void* stream) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!disparity || !mask || width <= 0 || height <= 0)
		return fail(ctx, B200MVS_ERR_ARG, "extract mask: null pointer or empty map");
	CK(cudaSetDevice(ctx->device));
	CK(tsgm_launch_extract_mask(disparity, mask, width, height, thValid, stream_of(ctx, stream)));
	return B200MVS_OK;
}

int b200mvs_sgm_filter_speckles_device(b200mvs_ctx* ctx, int16_t* disparity, int width, int height, int newVal, int maxSpeckleSize,
	int maxDiff, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!disparity || width <= 0 || height <= 0 || (size_t)width*height >= (1u<<31) || maxSpeckleSize < 0 || maxDiff < 0)
		return fail(ctx, B200MVS_ERR_ARG, "filter speckles: null map, bad size or negative limits");
	CK(cudaSetDevice(ctx->device));
	const size_t n = (size_t)width*height;
	CK(ctx->ts[b200mvs_ctx::TS_LABELS].reserve(n*sizeof(int))); CK(ctx->ts[b200mvs_ctx::TS_SIZES].reserve(n*sizeof(int)));
	CK(tsgm_launch_speckles(disparity, width, height, newVal, maxSpeckleSize, maxDiff, ctx->ts[b200mvs_ctx::TS_LABELS].as<int>(),
		ctx->ts[b200mvs_ctx::TS_SIZES].as<int>(), stream_of(ctx, stream)));
	return B200MVS_OK;
}

int b200mvs_resize_area_u8_device(b200mvs_ctx* ctx, const uint8_t* src, int width, int height, int channels, int factor, uint8_t* dst, void* stream) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!src || !dst || width <= 0 || height <= 0 || factor < 1 || (channels != 1 && channels != 3 && channels != 4))
		return fail(ctx, B200MVS_ERR_ARG, "resize area u8: null pointer, empty image, factor < 1 or channels not 1, 3 or 4");
	const int dw = (int)std::nearbyint(width*(1.0/factor)), dh = (int)std::nearbyint(height*(1.0/factor));
	if (dw <= 0 || dh <= 0) return fail(ctx, B200MVS_ERR_ARG, "resize area u8: empty result");
	CK(cudaSetDevice(ctx->device));
	CK(tsgm_launch_area_u8(src, width, height, channels, dst, dw, dh, factor, stream_of(ctx, stream)));
	return B200MVS_OK;
}

static int tsgm_level_mask(b200mvs_ctx* ctx, const uint8_t* mask, int width, int height, int lw, int lh, uint8_t* valid, cudaStream_t s) {
	DevBuf& t = ctx->ts[b200mvs_ctx::TS_MASKT];
	CK(t.reserve((size_t)lw*lh));
	CK(rs_launch_nearest_u8(mask, width, height, width, t.as<uint8_t>(), lw, lh, s));
	CK(cudaMemcpy2DAsync(valid, lw-6, t.as<uint8_t>()+3*lw+3, lw, lw-6, lh-6, cudaMemcpyDeviceToDevice, s));
	return B200MVS_OK;
}

int b200mvs_sgm_level_mask_device(b200mvs_ctx* ctx, const uint8_t* mask, int width, int height, int levelWidth, int levelHeight,
	uint8_t* validMask, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!mask || !validMask || width <= 0 || height <= 0 || levelWidth <= 6 || levelHeight <= 6)
		return fail(ctx, B200MVS_ERR_ARG, "level mask: null pointer or a level of at most 6 pixels");
	CK(cudaSetDevice(ctx->device));
	return tsgm_level_mask(ctx, mask, width, height, levelWidth, levelHeight, validMask, stream_of(ctx, stream));
}

int b200mvs_sgm_match_hierarchical_device(b200mvs_ctx* ctx,
	const float* leftGray, const uint8_t* leftBGR, const float* rightGray, const uint8_t* rightBGR, int width, int height,
	const int16_t* initDisparity, int initWidth, int initHeight, const uint8_t* leftMask, const uint8_t* rightMask,
	int minResolution, int nSpeckleSize, int thCross, int subpixelSteps, const b200mvs_sgm_params* prm,
	int16_t* outDisparity, uint16_t* outCost, uint64_t* numCostsPerLevel, void* stream)
{
	typedef b200mvs_ctx X;
	if (!ctx) return B200MVS_ERR_ARG;
	if (!leftGray || !leftBGR || !rightGray || !rightBGR || !outDisparity || !outCost)
		return fail(ctx, B200MVS_ERR_ARG, "hierarchical sgm: null image or output map");
	if (nSpeckleSize < 0 || thCross < 0 || width >= 65535)
		return fail(ctx, B200MVS_ERR_ARG, "hierarchical sgm: negative nSpeckleSize / thCross or a width above 65534");
	int nl = 0, lw[B200MVS_SGM_MAX_LEVELS], lh[B200MVS_SGM_MAX_LEVELS], iw = 0, ih = 0;
	if (tsgm_levels(width, height, minResolution, nl, lw, lh, iw, ih))
		return fail(ctx, B200MVS_ERR_ARG, "hierarchical sgm: negative minResolution, or the image is too small for its levels");
	if (initDisparity && (initWidth != iw || initHeight != ih))
		return fail(ctx, B200MVS_ERR_ARG, "hierarchical sgm: the initial disparity map must have the size b200mvs_sgm_levels gives");
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	const bool tsgm = minResolution > 0;
	const size_t n = (size_t)width*height, nv = (size_t)(width-6)*(height-6);
	// grow-only scratch, sized for the full-resolution level up front (nothing is reallocated while kernels use it)
	const size_t nImg = nl > 1 ? (size_t)lw[nl-2]*lh[nl-2] : 0;
	CK(ctx->ts[X::TS_IMG].reserve(nImg*14+64));
	CK(ctx->ts[X::TS_MASKL].reserve(nv)); CK(ctx->ts[X::TS_MASKR].reserve(nv)); CK(ctx->ts[X::TS_MASKT].reserve(n));
	for (int b: {X::TS_DL, X::TS_DR, X::TS_DL0, X::TS_DR0}) CK(ctx->ts[b].reserve(nv*sizeof(int16_t)));
	CK(ctx->ts[X::TS_PXL].reserve(nv*sizeof(SGMPixel))); CK(ctx->ts[X::TS_PXR].reserve(nv*sizeof(SGMPixel)));
	CK(ctx->ts[X::TS_RANGES].reserve(nv*sizeof(short2))); CK(ctx->ts[X::TS_SCAN].reserve(tsgm_range_map_scratch(nv)));
	CK(ctx->ts[X::TS_KEYS].reserve(nv*sizeof(unsigned))); CK(ctx->ts[X::TS_LABELS].reserve(nv*sizeof(int)));
	CK(ctx->ts[X::TS_SIZES].reserve(nv*sizeof(int))); CK(ctx->ts[X::TS_SMALL].reserve(64));
	uint8_t* maskL = ctx->ts[X::TS_MASKL].as<uint8_t>(); uint8_t* maskR = ctx->ts[X::TS_MASKR].as<uint8_t>();
	uint8_t* maskT = ctx->ts[X::TS_MASKT].as<uint8_t>();
	b200mvs_sgm_pixel* pxL = ctx->ts[X::TS_PXL].as<b200mvs_sgm_pixel>(); b200mvs_sgm_pixel* pxR = ctx->ts[X::TS_PXR].as<b200mvs_sgm_pixel>();
	// dL / dR: the maps of the previous level (pw x ph; first level: the initial map), nL / nR: the maps of this level
	int16_t *dL = ctx->ts[X::TS_DL0].as<int16_t>(), *dR = ctx->ts[X::TS_DR0].as<int16_t>();
	int16_t *nL = ctx->ts[X::TS_DL].as<int16_t>(), *nR = ctx->ts[X::TS_DR].as<int16_t>();
	int pw = iw, ph = ih;
	if (initDisparity) CK(cudaMemcpyAsync(dL, initDisparity, (size_t)iw*ih*sizeof(int16_t), cudaMemcpyDeviceToDevice, s));
	else CK(tsgm_launch_fill(dL, (size_t)iw*ih, (int16_t)SGM_NO_DISP, s));
	int fixLo = 0, fixHi = 0;
	if (!tsgm) {
		// the global range of the initial map (SemiGlobalMatcher.cpp:643-668) over its valid values
		int mm[2] = {0, 0};
		int* dmm = (int*)(ctx->ts[X::TS_SMALL].as<unsigned long long>()+1);
		CK(tsgm_launch_minmax(dL, (size_t)iw*ih, dmm, s));
		CK(cudaMemcpyAsync(mm, dmm, sizeof(mm), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		if (mm[0] > mm[1]) return fail(ctx, B200MVS_ERR_ARG, "hierarchical sgm: minResolution = 0 needs an initial map with a valid disparity");
		const int16_t numDisp = (int16_t)((int16_t)(mm[1]-mm[0])+16), disp = (int16_t)(mm[0]+mm[1]);
		fixLo = (int16_t)(disp-numDisp); fixHi = (int16_t)(disp+numDisp);
		if (fixHi-fixLo > SGM_MAX_DISP)
			return fail(ctx, B200MVS_ERR_ARG, "hierarchical sgm: the initial map spans more than 256 disparities with its margins");
	}
	// one match; an empty volume (every pixel masked) leaves NO_DISP / NO_ACCUMCOST like the winner-takes-all of invalid pixels
	auto match = [&](const float* g0, const uint8_t* c0, const float* g1, int w, int h, const b200mvs_sgm_pixel* px, uint64_t num,
			int16_t* disp, uint16_t* cost) -> int {
		if (num == 0) {
			CK(tsgm_launch_fill(disp, (size_t)(w-6)*(h-6), (int16_t)SGM_NO_DISP, s));
			CK(cudaMemsetAsync(cost, 0xFF, (size_t)(w-6)*(h-6)*sizeof(uint16_t), s));
			return B200MVS_OK;
		}
		return b200mvs_sgm_match_device(ctx, g0, c0, g1, w, h, px, num, prm, 7, nullptr, nullptr, disp, cost, s, nullptr);
	};
	int rc = 0;
	for (int lev = 0; lev < nl; ++lev) {
		const int w = lw[lev], h = lh[lev], vw = w-6, vh = h-6;
		const bool first = lev == 0;
		// ViewData::GetImage(scale): INTER_AREA from the full-resolution images
		const float *lg = leftGray, *rg = rightGray; const uint8_t *lc = leftBGR, *rcol = rightBGR;
		if (lev+1 < nl) {
			const int f = 1 << (nl-1-lev);
			const size_t m = (size_t)w*h;
			float* g = (float*)ctx->ts[X::TS_IMG].p; uint8_t* c = (uint8_t*)(g+2*m);
			CK(rs_launch_area(leftGray, width, height, width, g, w, h, f, f, s));
			CK(rs_launch_area(rightGray, width, height, width, g+m, w, h, f, f, s));
			CK(tsgm_launch_area_u8(leftBGR, width, height, 3, c, w, h, f, s));
			CK(tsgm_launch_area_u8(rightBGR, width, height, 3, c+3*m, w, h, f, s));
			lg = g; rg = g+m; lc = c; rcol = c+3*m;
		}
		if (first) {
			// masks: NEAREST to the level size, cropped to the valid region (SemiGlobalMatcher.cpp:627-631)
			if (leftMask) { if ((rc = tsgm_level_mask(ctx, leftMask, width, height, w, h, maskL, s))) return rc; }
			else CK(cudaMemsetAsync(maskL, 0xFF, (size_t)vw*vh, s));
			if (rightMask) { if ((rc = tsgm_level_mask(ctx, rightMask, width, height, w, h, maskR, s))) return rc; }
			else CK(cudaMemsetAsync(maskR, 0xFF, (size_t)vw*vh, s));
		} else {
			for (uint8_t* m: {maskL, maskR}) {
				CK(tsgm_launch_upscale_mask(m, pw, ph, maskT, vw, vh, s));
				CK(cudaMemcpyAsync(m, maskT, (size_t)vw*vh, cudaMemcpyDeviceToDevice, s));
			}
		}
		uint64_t numR = 0, numL = 0;
		if (tsgm) {
			CK(tsgm_launch_flip(dL, dR, pw, ph, ctx->ts[X::TS_KEYS].as<unsigned>(), s));
			if ((rc = tsgm_range_map(ctx, dR, pw, ph, maskR, vw, vh, first ? 11 : 5, first ? 33 : 7, pxR, &numR, s))) return rc;
		} else {
			numR = (uint64_t)nv*(uint64_t)(fixHi-fixLo);
			CK(tsgm_launch_dense_map((SGMPixel*)pxR, nv, fixLo, fixHi, s));
		}
		if ((rc = match(rg, rcol, lg, w, h, pxR, numR, nR, outCost))) return rc;
		if (tsgm) {
			if ((rc = tsgm_range_map(ctx, dL, pw, ph, maskL, vw, vh, first ? 11 : 5, first ? 33 : 7, pxL, &numL, s))) return rc;
		} else {
			numL = numR;
			CK(tsgm_launch_dense_map((SGMPixel*)pxL, nv, -fixHi, -fixLo, s));
		}
		if ((rc = match(lg, lc, rg, w, h, pxL, numL, nL, outCost))) return rc;
		if (numCostsPerLevel) { numCostsPerLevel[2*lev] = numR; numCostsPerLevel[2*lev+1] = numL; }
		if (first) {
			// SemiGlobalMatcher.cpp:698-706
			CK(sgm_launch_cross_check(nL, nR, vw, vh, thCross, s));
			CK(sgm_launch_cross_check(nR, nL, vw, vh, thCross, s));
			for (int16_t* d: {nL, nR})
				CK(tsgm_launch_speckles(d, vw, vh, SGM_NO_DISP, nSpeckleSize, 5, ctx->ts[X::TS_LABELS].as<int>(), ctx->ts[X::TS_SIZES].as<int>(), s));
			CK(tsgm_launch_extract_mask(nL, maskL, vw, vh, 3, s));
			CK(tsgm_launch_extract_mask(nR, maskR, vw, vh, 3, s));
		} else {
			CK(sgm_launch_cross_check(nL, nR, vw, vh, thCross, s));
		}
		std::swap(dL, nL); std::swap(dR, nR);
		pw = vw; ph = vh;
	}
	// RefineDisparityMap(left) with the accumulated costs of the last left match (SemiGlobalMatcher.cpp:718)
	if (subpixelSteps > 1 && ctx->sgAccums.p)
		CK(sgm_launch_refine((const SGMPixel*)pxL, ctx->sgAccums.as<uint16_t>(), dL, (int)nv, subpixelSteps, s));
	CK(cudaMemcpyAsync(outDisparity, dL, nv*sizeof(int16_t), cudaMemcpyDeviceToDevice, s));
	// the pixel maps of the hierarchy are internal: no later refine call may take sgAccums for its own map
	ctx->sgLastPx = nullptr;
	CK(cudaStreamSynchronize(s));
	return B200MVS_OK;
}

} // extern "C"
