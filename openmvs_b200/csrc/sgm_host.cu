// sgm_host.cu — host side of the SGM entry points of the C-ABI: the pair matcher (SemiGlobalMatcher::Match, cost / aggregation
// / winner-takes-all), cross-check, sub-pixel refinement and the hierarchical (tSGM) level loop.
#include "host_ctx.h"
#include "sgm_common.cuh"
#include "resize_common.cuh"

namespace {

// One wave-front aggregation: the shape of its schedule (sgm_front_schedule) and the scratch of its launch, carved by the match
struct FrontRun {
	int maxPaths, maxCtl;
	int* ctl; uint16_t* state; float2* meta;   // [ticket, error, -, - | progress | cellDone] (4+maxCtl ints), path state, path meta
};

// SGM path aggregation with the wave-front kernel (sgm_front.cu): the two tilted passes f = +-(x + 2y) of sgm_front_sched.h share
// one launch and one queue; pass 0 accumulates into the caller's volume, pass 1 into `second`, and the winner-takes-all kernel
// adds the two.  The schedule is fixed (32 fronts per block, lag 1, sub-cells of at least 64 columns, DESIGN §5.3) and depends
// only on the size of the valid region: sgm_front_schedule builds and uploads it when the size changes (ctx->sgFront), and
// sgm_aggregate_fronts launches it.
int sgm_front_schedule(b200mvs_ctx* ctx, int vw, int vh, cudaStream_t s, FrontRun& F) {
	b200mvs_ctx::FrontSchedule& S = ctx->sgFront;
	if (S.vw != vw || S.vh != vh) {
		FrontLaunch L;
		sgm_front_build_launch(vw, vh, FRONT_FB, FRONT_LAG, sgm_front_sub_cell(vw), L);
		S.vw = S.vh = 0;   // no schedule until the upload has completed
		CK(S.items.reserve(L.items.size()*sizeof(FrontItem)));
		CK(cudaMemcpyAsync(S.items.p, L.items.data(), L.items.size()*sizeof(FrontItem), cudaMemcpyHostToDevice, s));
		CK(S.need.reserve(std::max<size_t>(1, L.cellNeed.size())*sizeof(int)));
		CK(cudaMemcpyAsync(S.need.p, L.cellNeed.data(), L.cellNeed.size()*sizeof(int), cudaMemcpyHostToDevice, s));
		CK(cudaStreamSynchronize(s)); // the pageable source vectors are released below
		S.nItems = (int)L.items.size();
		L.items.clear(); L.items.shrink_to_fit(); L.cellNeed.clear(); L.cellNeed.shrink_to_fit();
		S.launch = L; S.vw = vw; S.vh = vh;
	}
	F.maxPaths = vw+vh+8; F.maxCtl = S.launch.nChains + S.launch.nCells;
	return B200MVS_OK;
}

int sgm_aggregate_fronts(b200mvs_ctx* ctx, const SGMParams& P, int num, uint16_t* second, const FrontRun& F, cudaStream_t s) {
	const b200mvs_ctx::FrontSchedule& S = ctx->sgFront;
	const FrontLaunch& L = S.launch;
	// resident CTAs: the queue needs no particular number; at most 2 per SM (DESIGN §5.3)
	int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ctx->device));
	const int blocks = sms*std::min(sgm_front_blocks_per_sm(num), 2);
	// [ticket, error, -, - | progress | cellDone]
	CK(cudaMemsetAsync(F.ctl, 0, (size_t)(4+F.maxCtl)*sizeof(int), s));
	FrontArgs A; memset(&A, 0, sizeof(A));
	A.items = S.items.as<FrontItem>(); A.nItems = S.nItems;
	A.ticket = F.ctl; A.error = F.ctl+1; A.progress = F.ctl+4; A.cellDone = F.ctl+4+L.nChains; A.cellNeed = S.need.as<int>();
	A.state = F.state; A.meta = F.meta; A.maxPaths = F.maxPaths;
	A.FB = L.FB; A.num = num;
	for (int p = 0; p < 2; ++p) { A.fa[p] = FRONT_PASSES[p].fa; A.fb[p] = FRONT_PASSES[p].fb; A.fc[p] = L.fc[p]; }
	A.sum[0] = P.accums; A.sum[1] = second;
	CK(sgm_front_launch(P, A, blocks, s)); ++ctx->launches;
	return B200MVS_OK;
}

// The kernels of one match (sgm_plan).
struct SGMPlan {
	enum Aggregation { FRONTS, UNIFORM_RING, UNIFORM, RAGGED_STREAMS, RAGGED } agg;
	bool tcCost;     // the tensor-core cost kernel (sgm_cost_tc.cu), else sgm_cost_kernel
	bool denseWta;   // sgm_wta_uniform_kernel, else sgm_wta_kernel
	int volumes;     // sum volumes the aggregation leaves for the winner-takes-all to add: 1, 2 (the wave-front passes) or 8
};

// Picks the kernels from the pixel map's statistics, the debug switches (b200mvs_debug.sgmAggregation / sgmCost),
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
	p.volumes = front ? 2 : p.agg == SGMPlan::RAGGED_STREAMS ? 8 : 1;
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
	const auto t0 = std::chrono::steady_clock::now();
	ctx->launches = 0;
	SGMMapStats st = {};
	SGMPlan plan = {};
	if (stats) CK(cudaEventRecord(ctx->ev0, s));
	if (stages & 7) {
		ReadBack* rb; CK(read_back(ctx, rb));
		CK(sgm_launch_map_stats(P.px, P.vw*P.vh, numCosts, &rb->mapStats, s)); ctx->launches += 2;
		CK(cudaMemcpyAsync(&st, &rb->mapStats, sizeof(st), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		if (st.overflow)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: a pixel's slice [idx, idx+dmax-dmin) ends beyond numCosts");
		// the warp-per-scanline kernel keeps one line of at most SGM_MAX_DISP values
		if (st.maxNum > SGM_MAX_DISP)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: more than 256 disparities per pixel");
		P.maxNumDisp = st.maxNum;
		// a volume the caller does not pass (null here) is carved below, 256-byte aligned
		plan = sgm_plan(st, ctx->dbg, !((uintptr_t)costs & 15), !((uintptr_t)accums & 15), maxP2, numCosts);
		if (ctx->dbg.sgmAggregation == 4 && plan.agg != SGMPlan::FRONTS)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: the wave-front kernel needs a dense volume with one range of 64, 128 or 256 disparities");
	}
	// the sum volumes the winner-takes-all adds: accums, then nVol-1 more at `more`
	const int nVol = (stages & 2) ? plan.volumes : 1;
	const bool fronts = (stages & 2) && plan.agg == SGMPlan::FRONTS, streams = (stages & 2) && plan.agg == SGMPlan::RAGGED_STREAMS;
	FrontRun F = {};
	if (fronts) { const int rc = sgm_front_schedule(ctx, P.vw, P.vh, s, F); if (rc) return rc; }
	// the match's scratch: the volumes the caller does not pass, the second sum volume(s) and the wave-front state
	Carve scratch(ctx->sgmScratch);
	const bool ownAccums = !accums;
	if (ownAccums) scratch.take(accums, numCosts);
	if (!costs) scratch.take(costs, numCosts);
	uint16_t* more = nullptr;
	if (fronts) scratch.take(more, (size_t)P.vw*P.vh*st.maxNum);
	if (streams) scratch.take(more, (size_t)7*numCosts);
	if (fronts) { scratch.take(F.ctl, 4+F.maxCtl); scratch.take(F.state, (size_t)8*F.maxPaths*st.maxNum); scratch.take(F.meta, 8*F.maxPaths); }
	CK(scratch.commit());
	P.costs = costs; P.accums = accums;
	// b200mvs_sgm_refine_device(accums = NULL) reads the last match's own sum volume, for the pixel map it aggregated
	if (ownAccums) ctx->sgLastAccums = accums;
	else if (!scratch.empty()) { ctx->sgLastAccums = nullptr; ctx->sgLastPx = nullptr; }   // the carve may have moved them
	if (stages & 2) ctx->sgLastPx = ownAccums ? (const void*)pixels : nullptr;
	if (stages & 1) {
		if (ctx->dbg.sgmCost == 2 && !plan.tcCost)
			return fail(ctx, B200MVS_ERR_ARG, "sgm: the tensor-core cost kernel needs a dense volume with one range of 64, 128, 192 or 256 disparities");
		if (plan.tcCost) { CK(sgm_cost_tc_launch(P, st.dminLo, st.maxNum, s)); ctx->launches += (st.maxNum+127)/128; }
		else { CK(sgm_launch_cost(P, s)); ++ctx->launches; }
	}
	if (fronts) {
		const int rc = sgm_aggregate_fronts(ctx, P, st.maxNum, more, F, s);
		if (rc) return rc;
	} else
	if (streams) {
		// ragged (tSGM) ranges: a direction has only 1000-3000 scanlines, one warp each — far too few to fill the GPU.  The eight
		// directions run side by side on eight streams, each STORING its path costs into a volume of its own (no memset, no
		// read-modify-write, no races); the winner-takes-all kernel adds the volumes.
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
		if (fronts) {
			// the wave-front kernel flags a dependency wait that timed out (never in a correct schedule): the stream is idle here
			int err = 0;
			CK(cudaMemcpy(&err, F.ctl+1, sizeof(int), cudaMemcpyDeviceToHost));
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
	HostCall call(ctx);
	const size_t n = (size_t)width*height, nv = (size_t)(width-6)*(height-6);
	const float *dL, *dR; const uint8_t* dC; const b200mvs_sgm_pixel* dPx; int16_t* dDisp; uint16_t* dCost;
	call.in(dL, leftGray, n*sizeof(float)); call.in(dR, rightGray, n*sizeof(float)); call.in(dC, leftBGR, n*3);
	call.in(dPx, pixels, nv*sizeof(SGMPixel));
	call.out(dDisp, disparity, nv*sizeof(int16_t)); call.out(dCost, cost, nv*sizeof(uint16_t));
	if (int rc = call.stage()) return rc;
	// with statistics the match records ev0 / ev1 around its kernels and checks the wave-front aggregation's error word
	call.formRecordsEvents = true;
	b200mvs_stats st;
	return call.run([&](cudaStream_t s) {
		return b200mvs_sgm_match_device(ctx, dL, dC, dR, width, height, dPx, numCosts, prm, 7, nullptr, nullptr, dDisp, dCost, s, &st);
	}, stats);
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
		accums = ctx->sgLastAccums;
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

// Disparity2RangeMap of a width x height map onto the mw x mh grid.  ranges: width x height, scan: tsgm_range_map_scratch(mw x mh)
// bytes, from the caller's carve.
static int tsgm_range_map(b200mvs_ctx* ctx, const int16_t* disparity, int width, int height, const uint8_t* mask, int mw, int mh,
	int minNumDisp, int minNumDispInvalid, short2* ranges, uint8_t* scan, b200mvs_sgm_pixel* pixels, uint64_t* numCosts, cudaStream_t s)
{
	ReadBack* rb; CK(read_back(ctx, rb));
	unsigned long long* total = &rb->rangeTotal;
	CK(tsgm_launch_range_map(disparity, width, height, mask, mw, mh, minNumDisp, minNumDispInvalid, ranges, (SGMPixel*)pixels, scan,
		total, s));
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
	Carve scratch(ctx->tsgmScratch);
	short2* ranges; uint8_t* scan;
	scratch.take(ranges, (size_t)width*height); scratch.take(scan, tsgm_range_map_scratch((size_t)maskWidth*maskHeight));
	CK(scratch.commit());
	return tsgm_range_map(ctx, disparity, width, height, mask, maskWidth, maskHeight, minNumDisp, minNumDispInvalid, ranges, scan,
		pixels, numCosts, stream_of(ctx, stream));
}

int b200mvs_sgm_flip_direction_device(b200mvs_ctx* ctx, const int16_t* l2r, int16_t* r2l, int width, int height, void* stream) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!l2r || !r2l || l2r == r2l || width <= 0 || height <= 0 || width >= 65535)
		return fail(ctx, B200MVS_ERR_ARG, "flip direction: null or aliased maps, or a width outside [1, 65534]");
	CK(cudaSetDevice(ctx->device));
	Carve scratch(ctx->tsgmScratch);
	unsigned* keys;
	scratch.take(keys, (size_t)width*height);
	CK(scratch.commit());
	CK(tsgm_launch_flip(l2r, r2l, width, height, keys, stream_of(ctx, stream)));
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
	Carve scratch(ctx->tsgmScratch);
	int *labels, *sizes;
	scratch.take(labels, n); scratch.take(sizes, n);
	CK(scratch.commit());
	CK(tsgm_launch_speckles(disparity, width, height, newVal, maxSpeckleSize, maxDiff, labels, sizes, stream_of(ctx, stream)));
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

// the mask of an lw x lh level, cropped to its valid region; t: lw x lh bytes from the caller's carve
static int tsgm_level_mask(b200mvs_ctx* ctx, const uint8_t* mask, int width, int height, int lw, int lh, uint8_t* t, uint8_t* valid,
	cudaStream_t s)
{
	CK(rs_launch_nearest_u8(mask, width, height, width, t, lw, lh, s));
	CK(cudaMemcpy2DAsync(valid, lw-6, t+3*lw+3, lw, lw-6, lh-6, cudaMemcpyDeviceToDevice, s));
	return B200MVS_OK;
}

int b200mvs_sgm_level_mask_device(b200mvs_ctx* ctx, const uint8_t* mask, int width, int height, int levelWidth, int levelHeight,
	uint8_t* validMask, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!mask || !validMask || width <= 0 || height <= 0 || levelWidth <= 6 || levelHeight <= 6)
		return fail(ctx, B200MVS_ERR_ARG, "level mask: null pointer or a level of at most 6 pixels");
	CK(cudaSetDevice(ctx->device));
	Carve scratch(ctx->tsgmScratch);
	uint8_t* t;
	scratch.take(t, (size_t)levelWidth*levelHeight);
	CK(scratch.commit());
	return tsgm_level_mask(ctx, mask, width, height, levelWidth, levelHeight, t, validMask, stream_of(ctx, stream));
}

int b200mvs_sgm_match_hierarchical_device(b200mvs_ctx* ctx,
	const float* leftGray, const uint8_t* leftBGR, const float* rightGray, const uint8_t* rightBGR, int width, int height,
	const int16_t* initDisparity, int initWidth, int initHeight, const uint8_t* leftMask, const uint8_t* rightMask,
	int minResolution, int nSpeckleSize, int thCross, int subpixelSteps, const b200mvs_sgm_params* prm,
	int16_t* outDisparity, uint16_t* outCost, uint64_t* numCostsPerLevel, void* stream)
{
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
	// the scratch of every level, sized for the largest: the level images (gray, then BGR, of the left and the right image; the
	// last level reads the caller's), the valid masks, the disparity maps of the previous level (dL / dR: pw x ph; first level:
	// the initial map) and of this one (nL / nR), the pixel maps, and the Disparity2RangeMap / FlipDirection / speckle scratch
	const size_t nImg = nl > 1 ? (size_t)lw[nl-2]*lh[nl-2] : 0;
	Carve scratch(ctx->tsgmScratch);
	float *grayL, *grayR; uint8_t *bgrL, *bgrR, *maskL, *maskR, *maskT, *scan;
	int16_t *dL, *dR, *nL, *nR; b200mvs_sgm_pixel *pxL, *pxR; short2* ranges; unsigned* keys; int *labels, *sizes;
	scratch.take(grayL, nImg); scratch.take(grayR, nImg); scratch.take(bgrL, 3*nImg); scratch.take(bgrR, 3*nImg);
	scratch.take(maskL, nv); scratch.take(maskR, nv); scratch.take(maskT, n);
	for (int16_t** d: {&dL, &dR, &nL, &nR}) scratch.take(*d, nv);
	scratch.take(pxL, nv); scratch.take(pxR, nv);
	scratch.take(ranges, nv); scratch.take(scan, tsgm_range_map_scratch(nv));
	scratch.take(keys, nv); scratch.take(labels, nv); scratch.take(sizes, nv);
	CK(scratch.commit());
	int pw = iw, ph = ih;
	if (initDisparity) CK(cudaMemcpyAsync(dL, initDisparity, (size_t)iw*ih*sizeof(int16_t), cudaMemcpyDeviceToDevice, s));
	else CK(tsgm_launch_fill(dL, (size_t)iw*ih, (int16_t)SGM_NO_DISP, s));
	int fixLo = 0, fixHi = 0;
	if (!tsgm) {
		// the global range of the initial map (SemiGlobalMatcher.cpp:643-668) over its valid values
		int mm[2] = {0, 0};
		ReadBack* rb; CK(read_back(ctx, rb));
		int* dmm = rb->minMax;
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
			CK(rs_launch_area(leftGray, width, height, width, grayL, w, h, f, f, s));
			CK(rs_launch_area(rightGray, width, height, width, grayR, w, h, f, f, s));
			CK(tsgm_launch_area_u8(leftBGR, width, height, 3, bgrL, w, h, f, s));
			CK(tsgm_launch_area_u8(rightBGR, width, height, 3, bgrR, w, h, f, s));
			lg = grayL; rg = grayR; lc = bgrL; rcol = bgrR;
		}
		if (first) {
			// masks: NEAREST to the level size, cropped to the valid region (SemiGlobalMatcher.cpp:627-631)
			if (leftMask) { if ((rc = tsgm_level_mask(ctx, leftMask, width, height, w, h, maskT, maskL, s))) return rc; }
			else CK(cudaMemsetAsync(maskL, 0xFF, (size_t)vw*vh, s));
			if (rightMask) { if ((rc = tsgm_level_mask(ctx, rightMask, width, height, w, h, maskT, maskR, s))) return rc; }
			else CK(cudaMemsetAsync(maskR, 0xFF, (size_t)vw*vh, s));
		} else {
			for (uint8_t* m: {maskL, maskR}) {
				CK(tsgm_launch_upscale_mask(m, pw, ph, maskT, vw, vh, s));
				CK(cudaMemcpyAsync(m, maskT, (size_t)vw*vh, cudaMemcpyDeviceToDevice, s));
			}
		}
		uint64_t numR = 0, numL = 0;
		if (tsgm) {
			CK(tsgm_launch_flip(dL, dR, pw, ph, keys, s));
			if ((rc = tsgm_range_map(ctx, dR, pw, ph, maskR, vw, vh, first ? 11 : 5, first ? 33 : 7, ranges, scan, pxR, &numR, s))) return rc;
		} else {
			numR = (uint64_t)nv*(uint64_t)(fixHi-fixLo);
			CK(tsgm_launch_dense_map((SGMPixel*)pxR, nv, fixLo, fixHi, s));
		}
		if ((rc = match(rg, rcol, lg, w, h, pxR, numR, nR, outCost))) return rc;
		if (tsgm) {
			if ((rc = tsgm_range_map(ctx, dL, pw, ph, maskL, vw, vh, first ? 11 : 5, first ? 33 : 7, ranges, scan, pxL, &numL, s))) return rc;
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
				CK(tsgm_launch_speckles(d, vw, vh, SGM_NO_DISP, nSpeckleSize, 5, labels, sizes, s));
			CK(tsgm_launch_extract_mask(nL, maskL, vw, vh, 3, s));
			CK(tsgm_launch_extract_mask(nR, maskR, vw, vh, 3, s));
		} else {
			CK(sgm_launch_cross_check(nL, nR, vw, vh, thCross, s));
		}
		std::swap(dL, nL); std::swap(dR, nR);
		pw = vw; ph = vh;
	}
	// RefineDisparityMap(left) with the accumulated costs of the last left match (SemiGlobalMatcher.cpp:718)
	if (subpixelSteps > 1 && ctx->sgLastAccums)
		CK(sgm_launch_refine((const SGMPixel*)pxL, ctx->sgLastAccums, dL, (int)nv, subpixelSteps, s));
	CK(cudaMemcpyAsync(outDisparity, dL, nv*sizeof(int16_t), cudaMemcpyDeviceToDevice, s));
	// the pixel maps of the hierarchy are internal: no later refine call may take the last match's sums for its own map
	ctx->sgLastPx = nullptr;
	CK(cudaStreamSynchronize(s));
	return B200MVS_OK;
}

// ---- fusion-mode -2: the pairs' disparity maps projected into an image and fused (SemiGlobalMatcher::Fuse) ----

// Q of a reversed pair (SemiGlobalMatcher.cpp:770-779), products as cv::Matx computes them (s = 0; s += a(i,k) b(k,j))
int b200mvs_sgm_pair_q(const double* Q, const double* Kl, const double* Rl, const double* Cl, const double* K, const double* R,
	const double* C, double* Qout)
{
	if (!Q || !Kl || !Rl || !Cl || !K || !R || !C || !Qout) return B200MVS_ERR_ARG;
	if (Kl[0] == 0 || Kl[4] == 0) return B200MVS_ERR_ARG;
	// ComputeRelativePose(Rl, Cl, R, C): Rrel = R Rl^T, Crel = Rl (C - Cl) (libs/Common/Util.inl:39-42)
	double Rr[9], Cr[3], dC[3] = {C[0]-Cl[0], C[1]-Cl[1], C[2]-Cl[2]};
	for (int i = 0; i < 3; ++i) {
		for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += R[i*3+k]*Rl[j*3+k]; Rr[i*3+j] = s; }
		double s = 0; for (int k = 0; k < 3; ++k) s += Rl[i*3+k]*dC[k]; Cr[i] = s;
	}
	// P = [K Rrel | K Rrel (-Crel)] over the last row of the identity (AssembleProjectionMatrix, libs/MVS/Camera.cpp:173-180)
	double P[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1};
	for (int i = 0; i < 3; ++i) {
		for (int j = 0; j < 3; ++j) { double s = 0; for (int k = 0; k < 3; ++k) s += K[i*3+k]*Rr[k*3+j]; P[i*4+j] = s; }
		double s = 0; for (int k = 0; k < 3; ++k) s += P[i*4+k]*(-Cr[k]); P[i*4+3] = s;
	}
	// invK of the pair's left camera in the identity (Camera::InvK, libs/MVS/Camera.h:177-185)
	double iK[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
	iK[0] = 1.0/Kl[0]; iK[5] = 1.0/Kl[4]; iK[2] = -Kl[2]*iK[0]; iK[6] = -Kl[5]*iK[5];
	double T[16], O[16];
	auto mul4 = [](const double* a, const double* b, double* c) {
		for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { double s = 0; for (int k = 0; k < 4; ++k) s += a[i*4+k]*b[k*4+j]; c[i*4+j] = s; }
	};
	mul4(P, iK, T); mul4(T, Q, O);
	memcpy(Qout, O, sizeof(O));
	return B200MVS_OK;
}

// checks the pairs and target size of a projection / fusion call and fills the kernels' parameter block; no device work
static int sgmf_args(b200mvs_ctx* ctx, const b200mvs_sgm_pair* pairs, int nPairs, int width, int height, SGMFuseArgs& A) {
	if (!pairs || nPairs < 1 || nPairs > B200MVS_SGM_MAX_PAIRS)
		return fail(ctx, B200MVS_ERR_ARG, "sgm fuse: null pair array or a pair count outside [1, B200MVS_SGM_MAX_PAIRS]");
	if (width <= 0 || height <= 0 || (size_t)width*height >= (1u<<31))
		return fail(ctx, B200MVS_ERR_ARG, "sgm fuse: empty image or one of 2^31 pixels or more");
	memset(&A, 0, sizeof(A));
	A.n = nPairs;
	for (int p = 0; p < nPairs; ++p) {
		const b200mvs_sgm_pair& q = pairs[p];
		if (!q.disparity || q.width <= 0 || q.height <= 0 || (size_t)q.width*q.height >= (1u<<31) || q.subpixelSteps < 1 || q.subpixelSteps > 32767)
			return fail(ctx, B200MVS_ERR_ARG, "sgm fuse: a pair without a disparity map, with an empty or oversized map, or subpixelSteps outside [1, 32767]");
		// the reference would read the released confidence map of a pair without costs (SemiGlobalMatcher.cpp:2036-2037, :842)
		if ((q.cost != nullptr) != (pairs[0].cost != nullptr))
			return fail(ctx, B200MVS_ERR_ARG, "sgm fuse: either every pair has a cost map or none has one");
		SGMFusePair& d = A.pair[p];
		d.disp = q.disparity; d.cost = q.cost; d.vw = q.width; d.vh = q.height; d.steps = q.subpixelSteps;
		memcpy(d.Q, q.Q, sizeof(d.Q));
	}
	return B200MVS_OK;
}

int b200mvs_sgm_project_disparity_device(b200mvs_ctx* ctx, const b200mvs_sgm_pair* pair, int width, int height, float* depth,
	float* depthRange, float* conf, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	SGMFuseArgs A;
	if (int rc = sgmf_args(ctx, pair, 1, width, height, A)) return rc;
	if (!depth || !depthRange || ((uintptr_t)depthRange & 7))
		return fail(ctx, B200MVS_ERR_ARG, "project disparity: null depth or range map, or a range map not 8-byte aligned");
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	const size_t n = (size_t)width*height;
	Carve scratch(ctx->sfScratch);
	unsigned long long* keys;
	scratch.take(keys, 4*n);
	CK(scratch.commit());
	CK(sgmf_launch_project(A, width, height, keys, s));
	CK(sgmf_launch_gather(A, width, height, keys, depth, (float2*)depthRange, conf, n, s));
	ctx->launches = 2;
	return B200MVS_OK;
}

static int sgmf_normals(b200mvs_ctx* ctx, const float* depth, int width, int height, const double* K, float* normal, cudaStream_t s) {
	// EstimateNormalMap takes Matrix3x3f: the caller's double K converted element by element
	CK(sgmf_launch_normals(depth, width, height, make_float4((float)K[0], (float)K[4], (float)K[2], (float)K[5]), normal, s));
	return B200MVS_OK;
}

int b200mvs_sgm_fuse_device(b200mvs_ctx* ctx, const b200mvs_sgm_pair* pairs, int nPairs, int width, int height, int minViews,
	const double* K, float* depth, float* conf, float* normal, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	SGMFuseArgs A;
	if (int rc = sgmf_args(ctx, pairs, nPairs, width, height, A)) return rc;
	if (!depth || minViews < 0 || (K && !normal))
		return fail(ctx, B200MVS_ERR_ARG, "sgm fuse: null depth map, negative minViews, or K without a normal map");
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	const size_t n = (size_t)width*height, np = (size_t)nPairs*n;
	// the splat keys, then every pair's range, depth and confidence maps (pair p at p x n)
	Carve scratch(ctx->sfScratch);
	unsigned long long* keys; float2* range; float *pd, *pc;
	scratch.take(keys, 4*np); scratch.take(range, np); scratch.take(pd, np); scratch.take(pc, np);
	CK(scratch.commit());
	CK(sgmf_launch_project(A, width, height, keys, s));
	CK(sgmf_launch_gather(A, width, height, keys, pd, range, pc, n, s));
	CK(sgmf_launch_fuse(nPairs, width, height, pd, range, pc, n, minViews, depth, conf, s));
	ctx->launches = 3;
	if (K) {
		if (int rc = sgmf_normals(ctx, depth, width, height, K, normal, s)) return rc;
		++ctx->launches;
	}
	return B200MVS_OK;
}

int b200mvs_sgm_fuse(b200mvs_ctx* ctx, const b200mvs_sgm_pair* pairs, int nPairs, int width, int height, int minViews,
	const double* K, float* depth, float* conf, float* normal, b200mvs_stats* stats)
{
	if (!ctx) return B200MVS_ERR_ARG;
	SGMFuseArgs A;
	if (int rc = sgmf_args(ctx, pairs, nPairs, width, height, A)) return rc;
	if (!depth || minViews < 0 || (K && !normal))
		return fail(ctx, B200MVS_ERR_ARG, "sgm fuse: null depth map, negative minViews, or K without a normal map");
	CK(cudaSetDevice(ctx->device));
	HostCall call(ctx);
	std::vector<b200mvs_sgm_pair> dev(pairs, pairs+nPairs);   // the pairs with staged disparity (and cost) maps
	for (b200mvs_sgm_pair& q: dev) {
		const size_t bytes = (size_t)q.width*q.height*sizeof(int16_t);
		call.in(q.disparity, q.disparity, bytes);
		if (q.cost) call.in(q.cost, q.cost, bytes);
	}
	const size_t n = (size_t)width*height;
	float *dD, *dC = nullptr, *dN = nullptr;
	call.out(dD, depth, n*sizeof(float));
	if (conf) call.out(dC, conf, n*sizeof(float));
	if (K) call.out(dN, normal, n*3*sizeof(float));
	if (int rc = call.stage()) return rc;
	return call.run([&](cudaStream_t s) { return b200mvs_sgm_fuse_device(ctx, dev.data(), nPairs, width, height, minViews, K, dD, dC, dN, s); },
		stats);
}

int b200mvs_estimate_normal_map_device(b200mvs_ctx* ctx, const float* depth, int width, int height, const double* K, float* normal,
	void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!depth || !K || !normal || depth == normal || width <= 0 || height <= 0 || (size_t)width*height >= (1u<<31))
		return fail(ctx, B200MVS_ERR_ARG, "estimate normal map: null or aliased maps, null K, or an empty or oversized map");
	CK(cudaSetDevice(ctx->device));
	if (int rc = sgmf_normals(ctx, depth, width, height, K, normal, stream_of(ctx, stream))) return rc;
	ctx->launches = 1;
	return B200MVS_OK;
}

} // extern "C"
