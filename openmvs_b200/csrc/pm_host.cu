// pm_host.cu — host side of the PatchMatch entry points of the C-ABI (b200mvs_estimate* and the pm_* building blocks).
//
// Mirrors the control flow of DepthMapsData::EstimateDepthMap (libs/MVS/SceneDensify.cpp:616-805)
// and of the accelerator seam PatchMatchCUDA::EstimateDepthMap (libs/MVS/PatchMatchCUDA.cpp:174-416):
// scale loop -> pass A (score) -> pass B (sweeps) -> pass C (threshold), all on one stream,
// no host synchronisation between kernels.
#include "host_ctx.h"
#include "pm_common.cuh"
#include "resize_common.cuh"

namespace {

void mul33(const double* A, const double* B, double* C) {
	double T[9];
	for (int i=0;i<3;++i) for (int j=0;j<3;++j) T[i*3+j] = A[i*3]*B[j] + A[i*3+1]*B[3+j] + A[i*3+2]*B[6+j];
	memcpy(C, T, sizeof(T));
}
void mul31(const double* A, const double* v, double* r) {
	double t[3];
	for (int i=0;i<3;++i) t[i] = A[i*3]*v[0] + A[i*3+1]*v[1] + A[i*3+2]*v[2];
	memcpy(r, t, sizeof(t));
}
void transpose33(const double* A, double* T) {
	double R[9];
	for (int i=0;i<3;++i) for (int j=0;j<3;++j) R[j*3+i] = A[i*3+j];
	memcpy(T, R, sizeof(R));
}
void inv33(const double* A, double* I) {
	const double a=A[0],b=A[1],c=A[2],d=A[3],e=A[4],f=A[5],g=A[6],h=A[7],i=A[8];
	const double id = 1.0/(a*(e*i-f*h) - b*(d*i-f*g) + c*(d*h-e*g));
	double R[9] = {(e*i-f*h)*id, (c*h-b*i)*id, (b*f-c*e)*id, (f*g-d*i)*id, (a*i-c*g)*id, (c*d-a*f)*id, (d*h-e*g)*id, (b*g-a*h)*id, (a*e-b*d)*id};
	memcpy(I, R, sizeof(R));
}
// Camera::ScaleK (libs/MVS/Camera.h:160-173)
void scaleK(const double* K, int sw, int sh, int dw, int dh, double* Ko) {
	const double sx = (double)dw/sw, sy = (double)dh/sh;
	Ko[0] = K[0]*sx; Ko[1] = K[1]*sx; Ko[2] = (K[2]+0.5)*sx-0.5;
	Ko[3] = 0; Ko[4] = K[4]*sy; Ko[5] = (K[5]+0.5)*sy-0.5;
	Ko[6] = 0; Ko[7] = 0; Ko[8] = 1;
}
inline float d2r(float d) { return d*(3.14159265358979323846f/180.f); }

// a view whose image (and optional depth-map) pointers are device pointers, pitch in floats
struct DView {
	const float* img; int w, h, pitch;
	double K[9], R[9], C[3];
	const float* dmap; int dw, dh, dpitch;
	double Kd[9], Rd[9], Cd[3];
};

// fill the kernel parameter block for one resolution level (DepthEstimator ctor constants,
// libs/MVS/DepthMap.cpp:361-412, and ViewData::Init, libs/MVS/DepthMap.h:175-185)
void build_params(const b200mvs_params& o, const DView* v, int nViews, float dMin, float dMax,
	const float* lowres, float4* plane, float* cost, uint32_t* best, PMParams& P, bool& geom)
{
	memset(&P, 0, sizeof(P));
	P.img0 = v[0].img; P.W = v[0].w; P.H = v[0].h; P.pitch0 = v[0].pitch;
	P.nViews = nViews-1;
	const double* K = v[0].K;
	P.ifx = (float)(1.0/K[0]); P.sk = (float)(-K[1]/(K[0]*K[4])); P.ox = (float)((K[1]*K[5]-K[2]*K[4])/(K[0]*K[4]));
	P.ify = (float)(1.0/K[4]); P.oy = (float)(-K[5]/K[4]);
	P.ox0 = (float)(-K[2]/K[0]);
	P.dMin = dMin; P.dMax = dMax; P.dMinSqr = std::sqrt(dMin); P.dMaxSqr = std::sqrt(dMax);
	P.keep = o.fNCCThresholdKeep;
	P.thMagnitudeSq = o.fDescriptorMinMagnitudeThreshold > 0 ? o.fDescriptorMinMagnitudeThreshold*o.fDescriptorMinMagnitudeThreshold : -1.f;
	P.thConfSmall = o.fNCCThresholdKeep*0.66f; P.thConfBig = o.fNCCThresholdKeep*0.9f;
	P.thConfRand = o.fNCCThresholdKeep*1.1f; P.thRobust = o.fNCCThresholdKeep*4.f/3.f;
	P.smoothBonusDepth = 1.f-o.fRandomSmoothBonus; P.smoothBonusNormal = (1.f-o.fRandomSmoothBonus)*0.96f;
	P.smoothSigmaDepth = -1.f/(2.f*o.fRandomSmoothDepth*o.fRandomSmoothDepth);
	P.smoothSigmaNormal = -1.f/(2.f*d2r(o.fRandomSmoothNormal)*d2r(o.fRandomSmoothNormal));
	P.depthRatio = o.fRandomDepthRatio; P.angle1Range = d2r(o.fRandomAngle1Range); P.angle2Range = d2r(o.fRandomAngle2Range);
	P.geomWeight = o.fEstimationGeometricWeight;
	P.nRandomIters = o.nRandomIters; P.propagation = o.nPropagation;
	P.farRings = o.nPropagationFar; P.evalCap = o.nEvalCap; P.skipUnchanged = 0; // the estimate call turns the changed-flag rule on; building blocks keep costs unsigned
	P.seed = o.seed;
	P.lowres = lowres; P.plane = plane; P.cost = cost; P.bestViews = best;
	double RrT[9], Hr[9], KrRr[9];
	transpose33(v[0].R, RrT);
	inv33(v[0].K, Hr);
	mul33(v[0].K, v[0].R, KrRr);
	geom = false;
	for (int i = 1; i < nViews; ++i) {
		PMView& V = P.views[i-1];
		double KR[9], Hl[9], A[9], dC[3], Hm[3];
		mul33(v[i].K, v[i].R, KR);
		mul33(KR, RrT, Hl);
		mul33(Hl, Hr, A);
		for (int k=0;k<3;++k) dC[k] = v[0].C[k]-v[i].C[k];
		mul31(KR, dC, Hm);
		for (int k=0;k<9;++k) V.A[k] = (float)A[k];
		for (int k=0;k<3;++k) V.Hm[k] = (float)Hm[k];
		V.img = v[i].img; V.w = v[i].w; V.h = v[i].h; V.pitch = v[i].pitch;
		V.dmap = v[i].dmap; V.dw = v[i].dw; V.dh = v[i].dh; V.dpitch = v[i].dpitch;
		if (v[i].dmap) {
			geom = true;
			double KdRd[9], T[9], t[3], RdT[9], iKd[9];
			mul33(v[i].Kd, v[i].Rd, KdRd);
			mul33(KdRd, RrT, T);
			for (int k=0;k<9;++k) V.Tl[k] = (float)T[k];
			for (int k=0;k<3;++k) dC[k] = v[0].C[k]-v[i].Cd[k];
			mul31(KdRd, dC, t);
			for (int k=0;k<3;++k) V.Tm[k] = (float)t[k];
			transpose33(v[i].Rd, RdT);
			inv33(v[i].Kd, iKd);
			mul33(KrRr, RdT, T); mul33(T, iKd, T);
			for (int k=0;k<9;++k) V.Tr[k] = (float)T[k];
			for (int k=0;k<3;++k) dC[k] = v[i].Cd[k]-v[0].C[k];
			mul31(KrRr, dC, t);
			for (int k=0;k<3;++k) V.Tn[k] = (float)t[k];
		}
	}
}

int check_views(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!views || nViews < 2 || nViews > B200MVS_MAX_VIEWS+1)
		return fail(ctx, B200MVS_ERR_ARG, "need 2..33 views (reference first)");
	for (int i = 0; i < nViews; ++i) {
		if ((!views[i].image && !views[i].image8) || views[i].width < 2*PM_HALF+2 || views[i].height < 2*PM_HALF+2)
			return fail(ctx, B200MVS_ERR_ARG, "view without image or image too small");
		if (!views[i].image && views[i].channels8 != 3 && views[i].channels8 != 4)
			return fail(ctx, B200MVS_ERR_ARG, "8-bit image needs 3 or 4 channels");
	}
	return B200MVS_OK;
}

// the arguments b200mvs_estimate_device and b200mvs_estimate_async share
int check_estimate(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax,
	const float* depth, const float* normal, const float* conf)
{
	const int rc = check_views(ctx, views, nViews);
	if (rc) return rc;
	if (!depth || !normal || !conf || !(dMin > 0 && dMin < dMax))
		return fail(ctx, B200MVS_ERR_ARG, "null map pointer or invalid depth range");
	return B200MVS_OK;
}

void to_dview(const b200mvs_view& s, const float* img, int pitch, const float* dmap, int dpitch, DView& d) {
	d.img = img; d.w = s.width; d.h = s.height; d.pitch = pitch;
	memcpy(d.K, s.K, sizeof(d.K)); memcpy(d.R, s.R, sizeof(d.R)); memcpy(d.C, s.C, sizeof(d.C));
	d.dmap = dmap; d.dw = s.dwidth; d.dh = s.dheight; d.dpitch = dpitch;
	memcpy(d.Kd, s.Kd, sizeof(d.Kd)); memcpy(d.Rd, s.Rd, sizeof(d.Rd)); memcpy(d.Cd, s.Cd, sizeof(d.Cd));
}

inline int cvRoundI(double v) { return (int)std::nearbyint(v); }

// The engine's red-black schedule for nEstimationIters reference iterations (DESIGN.md §2): nSweeps red-black sweeps with nR
// refinement tries each.  nSweepsPerIter > 0 pins it (nSweeps = nSweepsPerIter x iterations, nR = ceil(nRandomIters /
// nSweepsPerIter)); 0 (default) = max(8, ceil(1.5 x iterations)) sweeps sharing the reference's nRandomIters x iterations
// tries.  A geometric pass (one reference iteration on a converged estimate) is 2 sweeps (or nSweepsPerIter).
void engine_schedule(const b200mvs_params& o, bool geometric, int& nSweeps, int& nR) {
	const int I = std::max(0, o.nEstimationIters);
	if (o.nSweepsPerIter > 0 || geometric) {
		const int spi = o.nSweepsPerIter > 0 ? o.nSweepsPerIter : 2;
		nSweeps = geometric ? spi : spi*I;
		nR = (o.nRandomIters+spi-1)/spi;
	} else {
		nSweeps = I > 0 ? std::max(8, (3*I+1)/2) : 0;
		nR = nSweeps > 0 ? (o.nRandomIters*I+nSweeps-1)/nSweeps : 0;
	}
}

// cuTensorMapEncodeTiled through the runtime (no link against libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
	const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
	static EncodeTiledFn fn = nullptr; static bool tried = false;
	if (!tried) {
		tried = true;
		void* p = nullptr; cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
			fn = (EncodeTiledFn)p;
	}
	return fn;
}

// TMA descriptor of the reference image of one level: 2-D float tensor {W, H}, box = the tile a CTA
// of the sweep kernel stages (72 x 16).  TMA needs a 16-byte aligned base and row pitch; an image that
// does not satisfy this (odd width, cv::Mat ROI) is first copied to an aligned scratch image.
int prepare_ref_tmap(b200mvs_ctx* ctx, const DView& ref, cudaStream_t s) {
	ctx->tmapValid = false;
	EncodeTiledFn enc = ctx->dbg.noTMA ? nullptr : encode_tiled_fn();
	if (!enc) return B200MVS_OK;
	const float* base = ref.img; size_t pitchB = (size_t)ref.pitch*4;
	if (((uintptr_t)base & 15) || (pitchB & 15)) {
		pitchB = (((size_t)ref.w*4)+15)&~(size_t)15;
		CK(ctx->refPad.reserve(pitchB*ref.h));
		CK(cudaMemcpy2DAsync(ctx->refPad.p, pitchB, ref.img, (size_t)ref.pitch*4, (size_t)ref.w*4, ref.h, cudaMemcpyDeviceToDevice, s));
		base = ctx->refPad.as<float>();
	}
	int bw, bh; pm_tma_box(&bw, &bh);
	const cuuint64_t dims[2] = {(cuuint64_t)ref.w, (cuuint64_t)ref.h};
	const cuuint64_t strides[1] = {(cuuint64_t)pitchB};
	const cuuint32_t box[2] = {(cuuint32_t)bw, (cuuint32_t)bh};
	const cuuint32_t estr[2] = {1, 1};
	const CUresult r = enc(&ctx->tmapRef, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr,
		CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	ctx->tmapValid = (r == CUDA_SUCCESS);
	return B200MVS_OK;
}

int launch_sweep_timed(b200mvs_ctx* ctx, const PMParams& P, bool geom, cudaStream_t s) {
	if (ctx->timeSweeps) {
		while ((int)ctx->sweepEv.size() < 2*(ctx->nSweepEv+1)) {
			cudaEvent_t e; CK(cudaEventCreate(&e)); ctx->sweepEv.push_back(e);
		}
		CK(cudaEventRecord(ctx->sweepEv[2*ctx->nSweepEv], s));
	}
	CK(pm_launch_sweep(P, ctx->tmapValid ? &ctx->tmapRef : nullptr, geom, s)); ++ctx->launches;
	if (ctx->timeSweeps) {
		CK(cudaEventRecord(ctx->sweepEv[2*ctx->nSweepEv+1], s));
		++ctx->nSweepEv;
	}
	return B200MVS_OK;
}

// The whole EstimateDepthMap on device-resident views.  d_depth/d_normal hold the initial
// estimate (full resolution) and receive the result together with d_conf / d_views.
int estimate_on_device(b200mvs_ctx* ctx, const DView* views, int nViews, float dMin, float dMax, int nGeometricIter,
	float* d_depth, float* d_normal, float* d_conf, uint32_t* d_views, cudaStream_t s)
{
	const b200mvs_params& o = ctx->prm;
	const int W = views[0].w, H = views[0].h;
	const bool geometric = nGeometricIter >= 0;
	int nSweepsPhoto, nRPhoto, nSweeps, nR;
	engine_schedule(o, false, nSweepsPhoto, nRPhoto);
	engine_schedule(o, geometric, nSweeps, nR);
	// Philox phase of the first sweep of this call: photometric sweeps 0 .. nSweepsPhoto-1, then the geometric passes
	const int sweepBase = geometric ? nSweepsPhoto + nGeometricIter*nSweeps : 0;
	const int totalScale = !geometric ? std::max(0, o.nSubResolutionLevels) : 0;
	const size_t P0 = (size_t)W*H;
	if (ctx->mask && (ctx->maskW != W || ctx->maskH != H))
		return fail(ctx, B200MVS_ERR_ARG, "ignore-mask size differs from the reference image");
	CK(ctx->plane.reserve(P0*sizeof(float4)));
	CK(ctx->cost.reserve(P0*sizeof(float)));
	CK(ctx->best.reserve(P0*sizeof(uint32_t)));
	if (totalScale > 0) {
		CK(ctx->prior.reserve(P0*sizeof(float)));
		CK(ctx->lowPlane.reserve((size_t)(W/2+2)*(H/2+2)*sizeof(float4)));
		if (ctx->mask) CK(ctx->maskLevel.reserve((size_t)(W/2+2)*(H/2+2)));
		if ((int)ctx->pyr.size() < nViews) ctx->pyr.resize(nViews);
		// level 1 is the largest pyramid level: size the buffers once, so that no level re-allocates mid-stream
		for (int i = 0; i < nViews; ++i) {
			const size_t dw = (size_t)cvRoundI(views[i].w*0.5), dh = (size_t)cvRoundI(views[i].h*0.5);
			CK(ctx->pyr[i].reserve(dw*dh*sizeof(float)*(views[i].dmap ? 2 : 1)));
		}
	}
	float4* plane = ctx->plane.as<float4>();
	float* cost = ctx->cost.as<float>();
	uint32_t* best = ctx->best.as<uint32_t>();
	int lowW = 0, lowH = 0;
	for (int sc = totalScale; sc >= 0; --sc) {
		// ScaleDepthData (SceneDensify.cpp:578-601): INTER_AREA images, rescaled K
		std::vector<DView> lv(views, views+nViews);
		if (sc > 0) {
			const double scale = 1.0/(double)(1<<sc);
			for (int i = 0; i < nViews; ++i) {
				const int dw = cvRoundI(views[i].w*scale), dh = cvRoundI(views[i].h*scale);
				if (dw < 2*PM_HALF+2 || dh < 2*PM_HALF+2)
					return fail(ctx, B200MVS_ERR_ARG, "image too small for nSubResolutionLevels");
				const size_t need = (size_t)dw*dh*sizeof(float)*(views[i].dmap ? 2 : 1);
				CK(ctx->pyr[i].reserve(need));
				float* im = ctx->pyr[i].as<float>();
				CK(rs_launch_area(views[i].img, views[i].w, views[i].h, views[i].pitch, im, dw, dh, 1.0/scale, 1.0/scale, s)); ++ctx->launches;
				lv[i].img = im; lv[i].w = dw; lv[i].h = dh; lv[i].pitch = dw;
				scaleK(views[i].K, views[i].w, views[i].h, dw, dh, lv[i].K);
				if (views[i].dmap) {
					float* dm = im + (size_t)dw*dh;
					CK(rs_launch_area(views[i].dmap, views[i].dw, views[i].dh, views[i].dpitch, dm, dw, dh, 0, 0, s)); ++ctx->launches;
					lv[i].dmap = dm; lv[i].dw = dw; lv[i].dh = dh; lv[i].dpitch = dw;
					scaleK(views[i].Kd, views[i].dw, views[i].dh, dw, dh, lv[i].Kd);
				}
			}
		}
		const int w = lv[0].w, h = lv[0].h;
		{ const int rc = prepare_ref_tmap(ctx, lv[0], s); if (rc) return rc; }
		const float* lowres = nullptr;
		if (sc != totalScale) {
			// depth LINEAR / normal NEAREST up-sampling of the coarser level; the up-sampled
			// depth is also the prior of this level (SceneDensify.cpp:660-664)
			CK(rs_launch_plane_up(ctx->lowPlane.as<float4>(), lowW, lowH, plane, ctx->prior.as<float>(), w, h, ctx->mask != nullptr, s)); ++ctx->launches;
			lowres = ctx->prior.as<float>();
		} else if (sc == 0) {
			CK(pm_launch_pack((int)P0, d_depth, d_normal, plane, s)); ++ctx->launches;
		} else {
			// coarsest level: the caller's initial estimate, NEAREST down-sampled
			CK(ctx->dDepth.reserve((size_t)w*h*sizeof(float)));
			CK(ctx->dNormal.reserve((size_t)w*h*3*sizeof(float)));
			CK(rs_launch_nearest(d_depth, W, H, 1, ctx->dDepth.as<float>(), w, h, (double)(1<<sc), (double)(1<<sc), s));
			CK(rs_launch_nearest(d_normal, W, H, 3, ctx->dNormal.as<float>(), w, h, (double)(1<<sc), (double)(1<<sc), s));
			CK(pm_launch_pack(w*h, ctx->dDepth.as<float>(), ctx->dNormal.as<float>(), plane, s)); ctx->launches += 3;
		}
		PMParams P; bool geom;
		build_params(o, lv.data(), nViews, dMin, dMax, lowres, plane, cost, best, P, geom);
		P.nRandomIters = nR;
		P.skipUnchanged = o.bSkipUnchanged ? 1 : 0;
		P.tma = ctx->tmapValid ? 1 : 0;
		if (ctx->mask) {
			// the mask of this level: cv::resize(..., INTER_NEAREST) of the full-resolution mask (DepthMap.cpp:309)
			if (sc > 0) {
				CK(rs_launch_nearest_u8(ctx->mask, W, H, ctx->maskPitch, ctx->maskLevel.as<uint8_t>(), w, h, s)); ++ctx->launches;
				P.mask = ctx->maskLevel.as<uint8_t>(); P.maskPitch = w;
			} else { P.mask = ctx->mask; P.maskPitch = ctx->maskPitch; }
		}
		CK(pm_launch_score(P, geom, s)); ++ctx->launches;
		for (int k = 0; k < nSweeps; ++k) {
			P.sweep = sweepBase+k;
			for (int colour = 0; colour < 2; ++colour) {
				P.colour = colour;
				{ const int rc = launch_sweep_timed(ctx, P, geom, s); if (rc) return rc; }
			}
		}
		if (sc > 0) {
			CK(cudaMemcpyAsync(ctx->lowPlane.p, plane, (size_t)w*h*sizeof(float4), cudaMemcpyDeviceToDevice, s));
			lowW = w; lowH = h;
		}
	}
	float keep = o.fNCCThresholdKeep;
	if (nGeometricIter < 0 && o.nEstimationGeometricIters)
		keep *= 1.333f;
	CK(pm_launch_finalize((int)P0, keep, plane, cost, best, d_depth, d_normal, d_conf, d_views, s)); ++ctx->launches;
	return B200MVS_OK;
}

// fill_stats plus the sweep timings of an estimate call
int pm_stats(b200mvs_ctx* ctx, b200mvs_stats* stats, std::chrono::steady_clock::time_point t0, int levels, uint64_t h2d, uint64_t d2h) {
	const int rc = fill_stats(ctx, stats, t0, levels, h2d, d2h);
	if (rc) return rc;
	for (int k = 0; k < ctx->nSweepEv; ++k) { float t = 0; CK(cudaEventElapsedTime(&t, ctx->sweepEv[2*k], ctx->sweepEv[2*k+1])); stats->ms_sweep_kernels += t; }
	stats->sweep_launches = ctx->nSweepEv;
	stats->tma_active = ctx->tmapValid ? 1 : 0;
	return B200MVS_OK;
}

// Page-locks the caller's buffers for the duration of a batch: cudaMemcpyAsync from / to pageable memory blocks the host
// (and serialises the contexts); already pinned or unregistrable ranges are left alone.
struct PinGuard {
	std::vector<void*> regs;
	void add(const void* p, size_t bytes) {
		if (!p || !bytes) return;
		if (cudaHostRegister((void*)p, bytes, cudaHostRegisterPortable) == cudaSuccess) regs.push_back((void*)p);
		else (void)cudaGetLastError(); // already registered (pinned by the caller, or shared between jobs): fine
	}
	~PinGuard() { for (void* p: regs) cudaHostUnregister(p); }
};

} // namespace

extern "C" {

int b200mvs_get_schedule(const b200mvs_params* p, int geometric, int* nSweeps, int* nRefinePerSweep) {
	if (!p || !nSweeps || !nRefinePerSweep) return B200MVS_ERR_ARG;
	engine_schedule(*p, geometric != 0, *nSweeps, *nRefinePerSweep);
	return B200MVS_OK;
}

int b200mvs_estimate_device(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax, int nGeometricIter,
	float* depth, float* normal, float* conf, uint8_t* viewsMap, void* stream, b200mvs_stats* stats)
{
	int rc = check_estimate(ctx, views, nViews, dMin, dMax, depth, normal, conf);
	if (rc) return rc;
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	std::vector<DView> dv(nViews);
	ctx->launches = 0;
	for (int i = 0; i < nViews; ++i) {
		const float* img = views[i].image; int pitch = views[i].stride_bytes ? views[i].stride_bytes/4 : views[i].width;
		if (!img) {
			// 8-bit colour image resident in HBM: toGray into the context's scratch
			if ((int)ctx->imgs.size() < nViews) { ctx->imgs.resize(nViews); ctx->dmaps.resize(nViews); ctx->img8.resize(nViews); }
			CK(ctx->imgs[i].reserve((size_t)views[i].width*views[i].height*sizeof(float)));
			CK(rs_launch_to_gray(views[i].image8, views[i].width, views[i].height, views[i].stride8_bytes ? views[i].stride8_bytes : views[i].width*views[i].channels8,
				views[i].channels8, views[i].bgr8 != 0, ctx->imgs[i].as<float>(), views[i].width, s)); ++ctx->launches;
			img = ctx->imgs[i].as<float>(); pitch = views[i].width;
		}
		to_dview(views[i], img, pitch, views[i].depth, views[i].dstride_bytes ? views[i].dstride_bytes/4 : views[i].dwidth, dv[i]);
	}
	const auto t0 = std::chrono::steady_clock::now();
	ctx->nSweepEv = 0; ctx->timeSweeps = stats != nullptr;
	if (stats) CK(cudaEventRecord(ctx->ev0, s));
	rc = estimate_on_device(ctx, dv.data(), nViews, dMin, dMax, nGeometricIter, depth, normal, conf, (uint32_t*)viewsMap, s);
	if (rc) return rc;
	if (stats) {
		CK(cudaEventRecord(ctx->ev1, s));
		CK(cudaStreamSynchronize(s));
		return pm_stats(ctx, stats, t0, (nGeometricIter < 0 ? ctx->prm.nSubResolutionLevels : 0)+1, 0, 0);
	}
	return B200MVS_OK;
}

int b200mvs_estimate_async(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax, int nGeometricIter,
	float* depth, float* normal, float* conf, uint8_t* viewsMap)
{
	int rc = check_estimate(ctx, views, nViews, dMin, dMax, depth, normal, conf);
	if (rc) return rc;
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = ctx->stream;
	ctx->t0 = std::chrono::steady_clock::now();
	if ((int)ctx->imgs.size() < nViews) { ctx->imgs.resize(nViews); ctx->dmaps.resize(nViews); ctx->img8.resize(nViews); }
	std::vector<DView> dv(nViews);
	uint64_t h2d = 0, d2h = 0;
	ctx->launches = 0;
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_view& v = views[i];
		const size_t row = (size_t)v.width*sizeof(float);
		CK(ctx->imgs[i].reserve(row*v.height));
		if (v.image) {
			CK(cudaMemcpy2DAsync(ctx->imgs[i].p, row, v.image, v.stride_bytes ? v.stride_bytes : row, row, v.height, cudaMemcpyHostToDevice, s));
			h2d += row*v.height;
		} else {
			// 8-bit colour image: upload channels8 bytes per pixel, convert on the device (toGray)
			const size_t row8 = (size_t)v.width*v.channels8;
			CK(ctx->img8[i].reserve(row8*v.height));
			CK(cudaMemcpy2DAsync(ctx->img8[i].p, row8, v.image8, v.stride8_bytes ? v.stride8_bytes : row8, row8, v.height, cudaMemcpyHostToDevice, s));
			h2d += row8*v.height;
			CK(rs_launch_to_gray(ctx->img8[i].as<uint8_t>(), v.width, v.height, (int)row8, v.channels8, v.bgr8 != 0, ctx->imgs[i].as<float>(), v.width, s)); ++ctx->launches;
		}
		const float* dm = nullptr;
		if (v.depth) {
			const size_t drow = (size_t)v.dwidth*sizeof(float);
			CK(ctx->dmaps[i].reserve(drow*v.dheight));
			CK(cudaMemcpy2DAsync(ctx->dmaps[i].p, drow, v.depth, v.dstride_bytes ? v.dstride_bytes : drow, drow, v.dheight, cudaMemcpyHostToDevice, s));
			h2d += drow*v.dheight;
			dm = ctx->dmaps[i].as<float>();
		}
		to_dview(v, ctx->imgs[i].as<float>(), v.width, dm, v.dwidth, dv[i]);
	}
	const size_t P0 = (size_t)views[0].width*views[0].height;
	DevBuf& dD = ctx->mapD; DevBuf& dN = ctx->mapN;
	CK(dD.reserve(P0*sizeof(float))); CK(dN.reserve(P0*3*sizeof(float)));
	CK(ctx->dConf.reserve(P0*sizeof(float))); CK(ctx->dViews.reserve(P0*sizeof(uint32_t)));
	CK(cudaMemcpyAsync(dD.p, depth, P0*sizeof(float), cudaMemcpyHostToDevice, s));
	CK(cudaMemcpyAsync(dN.p, normal, P0*3*sizeof(float), cudaMemcpyHostToDevice, s));
	h2d += P0*16;
	ctx->nSweepEv = 0; ctx->timeSweeps = true;
	CK(cudaEventRecord(ctx->ev0, s));
	rc = estimate_on_device(ctx, dv.data(), nViews, dMin, dMax, nGeometricIter, dD.as<float>(), dN.as<float>(),
		ctx->dConf.as<float>(), ctx->dViews.as<uint32_t>(), s);
	if (rc) return rc;
	CK(cudaEventRecord(ctx->ev1, s));
	CK(cudaMemcpyAsync(depth, dD.p, P0*sizeof(float), cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(normal, dN.p, P0*3*sizeof(float), cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(conf, ctx->dConf.p, P0*sizeof(float), cudaMemcpyDeviceToHost, s));
	d2h += P0*20;
	if (viewsMap) { CK(cudaMemcpyAsync(viewsMap, ctx->dViews.p, P0*4, cudaMemcpyDeviceToHost, s)); d2h += P0*4; }
	ctx->pendH2D = h2d; ctx->pendD2H = d2h; ctx->pendLevels = (nGeometricIter < 0 ? ctx->prm.nSubResolutionLevels : 0)+1;
	ctx->pending = true;
	return B200MVS_OK;
}

int b200mvs_sync(b200mvs_ctx* ctx, b200mvs_stats* stats) {
	if (!ctx) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	CK(cudaStreamSynchronize(ctx->stream));
	if (stats) {
		memset(stats, 0, sizeof(*stats));
		if (ctx->pending) {
			const int rc = pm_stats(ctx, stats, ctx->t0, ctx->pendLevels, ctx->pendH2D, ctx->pendD2H);
			if (rc) return rc;
		}
	}
	ctx->pending = false;
	return B200MVS_OK;
}

int b200mvs_estimate(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax, int nGeometricIter,
	float* depth, float* normal, float* conf, uint8_t* viewsMap, b200mvs_stats* stats)
{
	const int rc = b200mvs_estimate_async(ctx, views, nViews, dMin, dMax, nGeometricIter, depth, normal, conf, viewsMap);
	if (rc) return rc;
	return b200mvs_sync(ctx, stats);
}

int b200mvs_estimate_batch(b200mvs_ctx** ctxs, int nCtx, b200mvs_job* jobs, int nJobs) {
	if (!ctxs || nCtx <= 0 || (!jobs && nJobs > 0) || nJobs < 0) return B200MVS_ERR_ARG;
	for (int k = 0; k < nCtx; ++k) if (!ctxs[k]) return B200MVS_ERR_ARG;
	PinGuard pin;
	for (int j = 0; j < nJobs; ++j) {
		const b200mvs_job& J = jobs[j];
		if (!J.views || J.nViews <= 0) continue;
		for (int i = 0; i < J.nViews; ++i) {
			const b200mvs_view& v = J.views[i];
			if (v.image) pin.add(v.image, (size_t)(v.stride_bytes ? v.stride_bytes : v.width*4)*v.height);
			else if (v.image8) pin.add(v.image8, (size_t)(v.stride8_bytes ? v.stride8_bytes : v.width*v.channels8)*v.height);
			if (v.depth) pin.add(v.depth, (size_t)(v.dstride_bytes ? v.dstride_bytes : v.dwidth*4)*v.dheight);
		}
		const size_t P0 = (size_t)J.views[0].width*J.views[0].height;
		pin.add(J.depth, P0*4); pin.add(J.normal, P0*12); pin.add(J.conf, P0*4); pin.add(J.viewsMap, P0*4);
	}
	int first = B200MVS_OK;
	std::vector<int> inflight(nCtx, -1); // job running on each context
	auto drain = [&](int k) {
		if (inflight[k] < 0) return;
		const int rc = b200mvs_sync(ctxs[k], nullptr);
		if (rc && !jobs[inflight[k]].status) jobs[inflight[k]].status = rc;
		if (jobs[inflight[k]].status && !first) first = jobs[inflight[k]].status;
		inflight[k] = -1;
	};
	for (int j = 0; j < nJobs; ++j) {
		const int k = j % nCtx;
		drain(k);
		b200mvs_job& J = jobs[j];
		J.status = b200mvs_estimate_async(ctxs[k], J.views, J.nViews, J.dMin, J.dMax, J.nGeometricIter, J.depth, J.normal, J.conf, J.viewsMap);
		if (J.status) { if (!first) first = J.status; continue; }
		inflight[k] = j;
	}
	for (int k = 0; k < nCtx; ++k) drain(k);
	return first;
}

// ---- building blocks ----------------------------------------------------------------------
int b200mvs_pm_pack(b200mvs_ctx* ctx, int width, int height, const float* depth, const float* normal, float* plane4, void* stream) {
	if (!ctx || !depth || !normal || !plane4) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	CK(pm_launch_pack(width*height, depth, normal, (float4*)plane4, stream_of(ctx, stream)));
	return B200MVS_OK;
}
int b200mvs_pm_unpack(b200mvs_ctx* ctx, int width, int height, const float* plane4, float* depth, float* normal, void* stream) {
	if (!ctx || !depth || !normal || !plane4) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	CK(pm_launch_unpack(width*height, (const float4*)plane4, depth, normal, stream_of(ctx, stream)));
	return B200MVS_OK;
}
static int block_params(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax, const float* lowres,
	float* plane4, float* cost, cudaStream_t s, PMParams& P, bool& geom)
{
	int rc = check_views(ctx, views, nViews);
	if (rc) return rc;
	if (!plane4 || !cost) return fail(ctx, B200MVS_ERR_ARG, "null state pointer");
	for (int i = 0; i < nViews; ++i)
		if (!views[i].image) return fail(ctx, B200MVS_ERR_ARG, "the building blocks take float gray images");
	std::vector<DView> dv(nViews);
	for (int i = 0; i < nViews; ++i)
		to_dview(views[i], views[i].image, views[i].stride_bytes ? views[i].stride_bytes/4 : views[i].width,
			views[i].depth, views[i].dstride_bytes ? views[i].dstride_bytes/4 : views[i].dwidth, dv[i]);
	{ const int rc2 = prepare_ref_tmap(ctx, dv[0], s); if (rc2) return rc2; }
	build_params(ctx->prm, dv.data(), nViews, dMin, dMax, lowres, (float4*)plane4, cost, nullptr, P, geom);
	P.tma = ctx->tmapValid ? 1 : 0;
	return B200MVS_OK;
}
int b200mvs_pm_score(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax,
	const float* lowres, float* plane4, float* cost, void* stream)
{
	PMParams P; bool geom;
	if (!ctx) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	int rc = block_params(ctx, views, nViews, dMin, dMax, lowres, plane4, cost, s, P, geom);
	if (rc) return rc;
	CK(pm_launch_score(P, geom, s));
	return B200MVS_OK;
}
int b200mvs_pm_sweep(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax,
	const float* lowres, int sweep, int half, int nRandomIters, float* plane4, float* cost, void* stream)
{
	PMParams P; bool geom;
	if (!ctx) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	int rc = block_params(ctx, views, nViews, dMin, dMax, lowres, plane4, cost, s, P, geom);
	if (rc) return rc;
	P.sweep = sweep; P.nRandomIters = nRandomIters;
	for (int colour = 0; colour < 2; ++colour) {
		if (half >= 0 && half != colour) continue;
		P.colour = colour;
		CK(pm_launch_sweep(P, ctx->tmapValid ? &ctx->tmapRef : nullptr, geom, s));
	}
	return B200MVS_OK;
}
int b200mvs_pm_finalize(b200mvs_ctx* ctx, int width, int height, float keep, const float* plane4, const float* cost,
	float* depth, float* normal, float* conf, void* stream)
{
	if (!ctx || !plane4 || !cost || !depth || !normal || !conf) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	CK(pm_launch_finalize(width*height, keep, (const float4*)plane4, cost, nullptr, depth, normal, conf, nullptr,
		stream_of(ctx, stream)));
	return B200MVS_OK;
}

} // extern "C"
