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

// One image of a caller's view as it lies in memory: `rows` rows of `row` bytes, `pitch` bytes apart (stride 0: packed rows)
struct Rows { const void* p; size_t row, pitch; int rows; size_t extent() const { return pitch*rows; } };
Rows rows_of(const void* p, size_t row, int stride, int rows) { return {p, row, stride ? (size_t)stride : row, rows}; }
// the float gray image, or else the 8-bit colour image
Rows image_rows(const b200mvs_view& v) {
	return v.image ? rows_of(v.image, (size_t)v.width*sizeof(float), v.stride_bytes, v.height)
	               : rows_of(v.image8, (size_t)v.width*v.channels8, v.stride8_bytes, v.height);
}
Rows depth_rows(const b200mvs_view& v) { return rows_of(v.depth, (size_t)v.dwidth*sizeof(float), v.dstride_bytes, v.dheight); }

// The engine's views of the caller's device views: float images and depth-maps with their pitch in floats.  Float images and
// depth-maps are used in place; an 8-bit colour image is converted to gray (toGray) into gray[i] on stream s.
int stage_views(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, const std::vector<float*>& gray, cudaStream_t s,
	std::vector<DView>& dv)
{
	dv.resize(nViews);
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_view& v = views[i];
		const Rows im = image_rows(v), dm = depth_rows(v);
		DView& d = dv[i];
		d.w = v.width; d.h = v.height; d.dw = v.dwidth; d.dh = v.dheight;
		memcpy(d.K, v.K, sizeof(d.K)); memcpy(d.R, v.R, sizeof(d.R)); memcpy(d.C, v.C, sizeof(d.C));
		memcpy(d.Kd, v.Kd, sizeof(d.Kd)); memcpy(d.Rd, v.Rd, sizeof(d.Rd)); memcpy(d.Cd, v.Cd, sizeof(d.Cd));
		if (v.image) {
			d.img = v.image; d.pitch = (int)(im.pitch/sizeof(float));
		} else {
			d.img = gray[i]; d.pitch = v.width;
			CK(rs_launch_to_gray(v.image8, v.width, v.height, (int)im.pitch, v.channels8, v.bgr8 != 0, gray[i], v.width, s));
			++ctx->launches;
		}
		d.dmap = v.depth; d.dpitch = (int)(dm.pitch/sizeof(float));
	}
	return B200MVS_OK;
}

inline int cvRoundI(double v) { return (int)std::nearbyint(v); }

// width or height n of an image at pyramid level sc (ScaleDepthData, SceneDensify.cpp:578-601: cvRound of the scaled size)
int level_size(int n, int sc) { return cvRoundI(n*(1.0/(double)(1<<sc))); }

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

// TMA needs a 16-byte aligned base and row pitch: the bytes of the aligned copy of a w x h float image at `base`, rows `pitchB`
// bytes apart, that the sweep reads instead (0: the image is read in place)
size_t ref_pad_bytes(const void* base, size_t pitchB, int w, int h) {
	return ((uintptr_t)base & 15) || (pitchB & 15) ? ((((size_t)w*4)+15)&~(size_t)15)*h : 0;
}

// TMA descriptor of the reference image of one level: 2-D float tensor {W, H}, box = the tile a CTA
// of the sweep kernel stages (72 x 16; the box may exceed the image, TMA zero-fills the outside).  An image that TMA cannot
// address (odd width, cv::Mat ROI) is first copied to `pad`, of ref_pad_bytes.  The sweep kernel has no other way to read the
// reference patch, so a missing encoder or a refused descriptor fails the call.
int prepare_ref_tmap(b200mvs_ctx* ctx, const DView& ref, float* pad, cudaStream_t s) {
	EncodeTiledFn enc = encode_tiled_fn();
	if (!enc) return fail(ctx, B200MVS_ERR_CUDA, "cuTensorMapEncodeTiled: the driver does not provide the entry point");
	const float* base = ref.img; size_t pitchB = (size_t)ref.pitch*4;
	if (ref_pad_bytes(base, pitchB, ref.w, ref.h)) {
		pitchB = (((size_t)ref.w*4)+15)&~(size_t)15;
		CK(cudaMemcpy2DAsync(pad, pitchB, ref.img, (size_t)ref.pitch*4, (size_t)ref.w*4, ref.h, cudaMemcpyDeviceToDevice, s));
		base = pad;
	}
	int bw, bh; pm_tma_box(&bw, &bh);
	const cuuint64_t dims[2] = {(cuuint64_t)ref.w, (cuuint64_t)ref.h};
	const cuuint64_t strides[1] = {(cuuint64_t)pitchB};
	const cuuint32_t box[2] = {(cuuint32_t)bw, (cuuint32_t)bh};
	const cuuint32_t estr[2] = {1, 1};
	const CUresult r = enc(&ctx->tmapRef, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)base, dims, strides, box, estr,
		CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS)
		return fail(ctx, B200MVS_ERR_CUDA, ("cuTensorMapEncodeTiled failed for the reference image (CUresult " + std::to_string((int)r) + ")").c_str());
	return B200MVS_OK;
}

int launch_sweep_timed(b200mvs_ctx* ctx, const PMParams& P, bool geom, cudaStream_t s) {
	if (ctx->timeSweeps) {
		while ((int)ctx->sweepEv.size() < 2*(ctx->nSweepEv+1)) {
			cudaEvent_t e; CK(cudaEventCreate(&e)); ctx->sweepEv.push_back(e);
		}
		CK(cudaEventRecord(ctx->sweepEv[2*ctx->nSweepEv], s));
	}
	CK(pm_launch_sweep(P, ctx->tmapRef, geom, s)); ++ctx->launches;
	if (ctx->timeSweeps) {
		CK(cudaEventRecord(ctx->sweepEv[2*ctx->nSweepEv+1], s));
		++ctx->nSweepEv;
	}
	return B200MVS_OK;
}

// sub-resolution levels of an estimate call: none for a geometric pass
int scale_levels(const b200mvs_params& o, int nGeometricIter) { return nGeometricIter < 0 ? std::max(0, o.nSubResolutionLevels) : 0; }

// The scratch of an estimate call, carved from the PatchMatch arena: the gray images of 8-bit colour views, the pyramid levels
// of every view (image, then depth-map), the state of the current and of the coarser level, the initial estimate at the
// coarsest level, the mask of the current level and the TMA-aligned copy of the reference image
struct PMScratch {
	std::vector<float*> gray, pyr;
	float4 *plane = nullptr, *lowPlane = nullptr;
	float *cost = nullptr, *prior = nullptr, *dDepth = nullptr, *dNormal = nullptr, *refPad = nullptr;
	uint32_t* best = nullptr;
	uint8_t* maskLevel = nullptr;
};
int carve_estimate(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, int nGeometricIter, PMScratch& S) {
	Carve c(ctx->pmScratch);
	const int W = views[0].width, H = views[0].height, totalScale = scale_levels(ctx->prm, nGeometricIter);
	const size_t P0 = (size_t)W*H;
	S.gray.assign(nViews, nullptr);
	for (int i = 0; i < nViews; ++i) if (!views[i].image) c.take(S.gray[i], (size_t)views[i].width*views[i].height);
	c.take(S.plane, P0); c.take(S.cost, P0); c.take(S.best, P0);
	// the TMA pad of the reference image at level 0 (as stage_views describes it; a gray image is packed in the arena), then of the
	// packed pyramid levels
	const size_t pitch0 = views[0].image ? image_rows(views[0]).pitch/sizeof(float)*sizeof(float) : (size_t)W*sizeof(float);
	size_t pad = ref_pad_bytes(views[0].image, pitch0, W, H);
	if (totalScale > 0) {
		c.take(S.prior, P0);
		c.take(S.lowPlane, (size_t)(W/2+2)*(H/2+2));
		if (ctx->mask) c.take(S.maskLevel, (size_t)(W/2+2)*(H/2+2));
		const int wc = level_size(W, totalScale), hc = level_size(H, totalScale);
		c.take(S.dDepth, (size_t)wc*hc); c.take(S.dNormal, (size_t)wc*hc*3);
		// level 1 is the largest pyramid level
		S.pyr.assign(nViews, nullptr);
		for (int i = 0; i < nViews; ++i)
			c.take(S.pyr[i], (size_t)level_size(views[i].width, 1)*level_size(views[i].height, 1)*(views[i].depth ? 2 : 1));
		for (int sc = 1; sc <= totalScale; ++sc) {
			const int w = level_size(W, sc), h = level_size(H, sc);
			pad = std::max(pad, ref_pad_bytes(nullptr, (size_t)w*4, w, h));
		}
	}
	if (pad) c.take(S.refPad, pad/sizeof(float));
	CK(c.commit());
	return B200MVS_OK;
}

// The whole EstimateDepthMap on device-resident views, in the scratch of carve_estimate.  d_depth/d_normal hold the initial
// estimate (full resolution) and receive the result together with d_conf / d_views.
int estimate_on_device(b200mvs_ctx* ctx, const DView* views, int nViews, float dMin, float dMax, int nGeometricIter,
	const PMScratch& S, float* d_depth, float* d_normal, float* d_conf, uint32_t* d_views, cudaStream_t s)
{
	const b200mvs_params& o = ctx->prm;
	const int W = views[0].w, H = views[0].h;
	const bool geometric = nGeometricIter >= 0;
	int nSweepsPhoto, nRPhoto, nSweeps, nR;
	engine_schedule(o, false, nSweepsPhoto, nRPhoto);
	engine_schedule(o, geometric, nSweeps, nR);
	// Philox phase of the first sweep of this call: photometric sweeps 0 .. nSweepsPhoto-1, then the geometric passes
	const int sweepBase = geometric ? nSweepsPhoto + nGeometricIter*nSweeps : 0;
	const int totalScale = scale_levels(o, nGeometricIter);
	const size_t P0 = (size_t)W*H;
	if (ctx->mask && (ctx->maskW != W || ctx->maskH != H))
		return fail(ctx, B200MVS_ERR_ARG, "ignore-mask size differs from the reference image");
	float4* plane = S.plane;
	float* cost = S.cost;
	uint32_t* best = S.best;
	int lowW = 0, lowH = 0;
	for (int sc = totalScale; sc >= 0; --sc) {
		// ScaleDepthData (SceneDensify.cpp:578-601): INTER_AREA images, rescaled K
		std::vector<DView> lv(views, views+nViews);
		if (sc > 0) {
			const double inv = (double)(1<<sc);
			for (int i = 0; i < nViews; ++i) {
				const int dw = level_size(views[i].w, sc), dh = level_size(views[i].h, sc);
				if (dw < 2*PM_HALF+2 || dh < 2*PM_HALF+2)
					return fail(ctx, B200MVS_ERR_ARG, "image too small for nSubResolutionLevels");
				float* im = S.pyr[i];
				CK(rs_launch_area(views[i].img, views[i].w, views[i].h, views[i].pitch, im, dw, dh, inv, inv, s)); ++ctx->launches;
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
		{ const int rc = prepare_ref_tmap(ctx, lv[0], S.refPad, s); if (rc) return rc; }
		const float* lowres = nullptr;
		if (sc != totalScale) {
			// depth LINEAR / normal NEAREST up-sampling of the coarser level; the up-sampled
			// depth is also the prior of this level (SceneDensify.cpp:660-664)
			CK(rs_launch_plane_up(S.lowPlane, lowW, lowH, plane, S.prior, w, h, ctx->mask != nullptr, s)); ++ctx->launches;
			lowres = S.prior;
		} else if (sc == 0) {
			CK(pm_launch_pack((int)P0, d_depth, d_normal, plane, s)); ++ctx->launches;
		} else {
			// coarsest level: the caller's initial estimate, NEAREST down-sampled
			CK(rs_launch_nearest(d_depth, W, H, 1, S.dDepth, w, h, (double)(1<<sc), (double)(1<<sc), s));
			CK(rs_launch_nearest(d_normal, W, H, 3, S.dNormal, w, h, (double)(1<<sc), (double)(1<<sc), s));
			CK(pm_launch_pack(w*h, S.dDepth, S.dNormal, plane, s)); ctx->launches += 3;
		}
		PMParams P; bool geom;
		build_params(o, lv.data(), nViews, dMin, dMax, lowres, plane, cost, best, P, geom);
		P.nRandomIters = nR;
		P.skipUnchanged = o.bSkipUnchanged ? 1 : 0;
		if (ctx->mask) {
			// the mask of this level: cv::resize(..., INTER_NEAREST) of the full-resolution mask (DepthMap.cpp:309)
			if (sc > 0) {
				CK(rs_launch_nearest_u8(ctx->mask, W, H, ctx->maskPitch, S.maskLevel, w, h, s)); ++ctx->launches;
				P.mask = S.maskLevel; P.maskPitch = w;
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
			CK(cudaMemcpyAsync(S.lowPlane, plane, (size_t)w*h*sizeof(float4), cudaMemcpyDeviceToDevice, s));
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
	stats->tma_active = 1;   // every sweep stages its reference tile by TMA (the call fails without a descriptor)
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
	PMScratch S;
	if ((rc = carve_estimate(ctx, views, nViews, nGeometricIter, S))) return rc;
	std::vector<DView> dv;
	ctx->launches = 0;
	rc = stage_views(ctx, views, nViews, S.gray, s, dv);
	if (rc) return rc;
	const auto t0 = std::chrono::steady_clock::now();
	ctx->nSweepEv = 0; ctx->timeSweeps = stats != nullptr;
	if (stats) CK(cudaEventRecord(ctx->ev0, s));
	rc = estimate_on_device(ctx, dv.data(), nViews, dMin, dMax, nGeometricIter, S, depth, normal, conf, (uint32_t*)viewsMap, s);
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
	HostCall call(ctx);
	std::vector<b200mvs_view> dev(views, views+nViews);   // the views with staged, packed images and depth-maps
	for (b200mvs_view& v: dev) {
		const Rows im = image_rows(v), dm = depth_rows(v);
		if (v.image) call.in(v.image, im.p, im.row, im.rows, im.pitch);
		else call.in(v.image8, im.p, im.row, im.rows, im.pitch);
		if (v.depth) call.in(v.depth, dm.p, dm.row, dm.rows, dm.pitch);
		v.stride_bytes = v.stride8_bytes = v.dstride_bytes = 0;
	}
	const size_t P0 = (size_t)views[0].width*views[0].height;
	float *dD, *dN, *dC; uint32_t* dV = nullptr;
	call.inout(dD, depth, P0*sizeof(float)); call.inout(dN, normal, P0*3*sizeof(float)); call.out(dC, conf, P0*sizeof(float));
	if (viewsMap) call.out(dV, viewsMap, P0*sizeof(uint32_t));
	if ((rc = call.stage())) return rc;
	PMScratch S;
	if ((rc = carve_estimate(ctx, dev.data(), nViews, nGeometricIter, S))) return rc;
	std::vector<DView> dv;
	ctx->launches = 0;
	rc = stage_views(ctx, dev.data(), nViews, S.gray, ctx->stream, dv);   // toGray runs before ev0, as in b200mvs_estimate_device
	if (rc) return rc;
	ctx->nSweepEv = 0; ctx->timeSweeps = true;
	return call.enqueue([&](cudaStream_t s) {
		return estimate_on_device(ctx, dv.data(), nViews, dMin, dMax, nGeometricIter, S, dD, dN, dC, dV, s);
	}, (nGeometricIter < 0 ? ctx->prm.nSubResolutionLevels : 0)+1);
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
			const Rows im = image_rows(J.views[i]), dm = depth_rows(J.views[i]);
			pin.add(im.p, im.extent());
			pin.add(dm.p, dm.extent());
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
// tmap: also encode the reference image's TMA descriptor (the sweep needs it, the score kernel does not)
static int block_params(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax, const float* lowres,
	float* plane4, float* cost, bool tmap, cudaStream_t s, PMParams& P, bool& geom)
{
	int rc = check_views(ctx, views, nViews);
	if (rc) return rc;
	if (!plane4 || !cost) return fail(ctx, B200MVS_ERR_ARG, "null state pointer");
	for (int i = 0; i < nViews; ++i)
		if (!views[i].image) return fail(ctx, B200MVS_ERR_ARG, "the building blocks take float gray images");
	std::vector<DView> dv;
	rc = stage_views(ctx, views, nViews, {}, s, dv);
	if (rc) return rc;
	if (tmap) {
		float* pad = nullptr;
		Carve c(ctx->pmScratch);
		if (size_t bytes = ref_pad_bytes(dv[0].img, (size_t)dv[0].pitch*4, dv[0].w, dv[0].h)) c.take(pad, bytes/sizeof(float));
		CK(c.commit());
		if ((rc = prepare_ref_tmap(ctx, dv[0], pad, s))) return rc;
	}
	build_params(ctx->prm, dv.data(), nViews, dMin, dMax, lowres, (float4*)plane4, cost, nullptr, P, geom);
	return B200MVS_OK;
}
int b200mvs_pm_score(b200mvs_ctx* ctx, const b200mvs_view* views, int nViews, float dMin, float dMax,
	const float* lowres, float* plane4, float* cost, void* stream)
{
	PMParams P; bool geom;
	if (!ctx) return B200MVS_ERR_ARG;
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	int rc = block_params(ctx, views, nViews, dMin, dMax, lowres, plane4, cost, false, s, P, geom);
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
	int rc = block_params(ctx, views, nViews, dMin, dMax, lowres, plane4, cost, true, s, P, geom);
	if (rc) return rc;
	P.sweep = sweep; P.nRandomIters = nRandomIters;
	for (int colour = 0; colour < 2; ++colour) {
		if (half >= 0 && half != colour) continue;
		P.colour = colour;
		CK(pm_launch_sweep(P, ctx->tmapRef, geom, s));
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
