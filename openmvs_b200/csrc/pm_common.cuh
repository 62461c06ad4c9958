// pm_common.cuh — shared definitions of the PatchMatch kernels (sm_90a) and their launch functions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define PM_MAX_VIEWS 32
#define PM_HALF 4      // nSizeHalfWindow (libs/MVS/DepthMap.h:277)
#define PM_TEXELS 25   // 5x5 taps, window 9x9 step 2

// per-neighbour-view constants (DepthData::ViewData::Init, libs/MVS/DepthMap.h:175-185),
// folded on the host in double: A = Hl*Hr, so that H(d,n) = A + Hm (n^T Hr)/(n.X0 d)
struct PMView {
	float A[9];
	float Hm[3];
	const float* img; int w, h, pitch;       // plain float image, pitch in floats
	const float* dmap; int dw, dh, dpitch;   // known depth-map (geometric pass) or null
	float Tl[9], Tm[3], Tr[9], Tn[3];
};

struct PMParams {
	const float* img0; int W, H, pitch0;
	int nViews;
	float ifx, sk, ox, ify, oy;              // Kref^-1 = [[ifx, sk, ox],[0, ify, oy],[0,0,1]]
	float ox0;                               // -cx/fx: the skew-free x offset InterpolatePixel uses (DepthMap.cpp:915-959)
	float dMin, dMax, dMinSqr, dMaxSqr;
	float keep;                              // fNCCThresholdKeep
	float thMagnitudeSq, thConfSmall, thConfBig, thConfRand, thRobust;
	float smoothBonusDepth, smoothBonusNormal, smoothSigmaDepth, smoothSigmaNormal;
	float depthRatio, angle1Range, angle2Range, geomWeight;
	int nRandomIters, propagation;           // refinement tries per sweep; directions that propagate (2 causal / 4)
	int farRings;                            // propagation candidates per direction: distances 1, 3, .. 2*farRings+1
	int evalCap;                             // > 0: tries per pixel and sweep <= max(1, evalCap - propagation candidates tested)
	int skipUnchanged;                       // 1: a direction whose candidates kept their plane is not re-tested (sign bit of cost)
	int sweep, colour;
	int tma;                                 // reference tile staged by TMA (tensor map passed beside the params)
	uint32_t seed;
	const float* lowres;                     // low-resolution depth prior or null
	const uint8_t* mask; int maskPitch;      // ignore-mask of this level (0 = skip the pixel) or null; pitch in bytes
	float4* plane; float* cost; uint32_t* bestViews;
	PMView views[PM_MAX_VIEWS];
};

// Philox4x32-10 (Salmon et al. 2011); counter = (pixel, phase, slot, 0), key = (seed, 0xB200C0DE)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
	#pragma unroll
	for (int r = 0; r < 10; ++r) {
		const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u*c.x;
		const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u*c.z;
		c = make_uint4(hi1^c.y^k.x, lo1, hi0^c.w^k.y, lo0);
		k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
	}
	return c;
}
__device__ __forceinline__ float u32_to_unit(uint32_t u) { return (float)u*(1.0f/4294967296.0f); }

// launch functions (pm_kernels.cu)
cudaError_t pm_configure_device();
cudaError_t pm_launch_score(const PMParams& P, bool geom, cudaStream_t s);
cudaError_t pm_launch_sweep(const PMParams& P, const void* tmapRef, bool geom, cudaStream_t s);
void pm_tma_box(int* w, int* h);
cudaError_t pm_launch_finalize(int n, float keep, const float4* plane, const float* cost, const uint32_t* bestViews,
	float* depth, float* normal, float* conf, uint32_t* viewsMap, cudaStream_t s);
cudaError_t pm_launch_pack(int n, const float* depth, const float* normal, float4* plane, cudaStream_t s);
cudaError_t pm_launch_unpack(int n, const float4* plane, float* depth, float* normal, cudaStream_t s);
