// fuse_common.cuh — the arithmetic of DepthMapsData::FuseDepthMaps, one definition for the host form (fuse_host.cu) and the device
// form (fuse_kernels.cu), and the interface between the fusion kernels and their host driver.
//
// Bit-identical results on both sides: every double and float operation goes through the helpers below, which are the correctly
// rounded intrinsics on the device (so nvcc cannot contract a multiply and an add into an FMA) and the plain operators on the host
// (the host build, -O3 without -march, does not contract either).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/b200mvs.h"

#define FUSE_HD __host__ __device__ __forceinline__

namespace fuse {

#ifdef __CUDA_ARCH__
FUSE_HD double mul_d(double a, double b) { return __dmul_rn(a, b); }
FUSE_HD double add_d(double a, double b) { return __dadd_rn(a, b); }
FUSE_HD double sub_d(double a, double b) { return __dsub_rn(a, b); }
FUSE_HD double div_d(double a, double b) { return __ddiv_rn(a, b); }
FUSE_HD float mul_f(float a, float b) { return __fmul_rn(a, b); }
FUSE_HD float add_f(float a, float b) { return __fadd_rn(a, b); }
FUSE_HD float sub_f(float a, float b) { return __fsub_rn(a, b); }
FUSE_HD float div_f(float a, float b) { return __fdiv_rn(a, b); }
FUSE_HD float sqrt_f(float a) { return __fsqrt_rn(a); }
#else
FUSE_HD double mul_d(double a, double b) { return a*b; }
FUSE_HD double add_d(double a, double b) { return a+b; }
FUSE_HD double sub_d(double a, double b) { return a-b; }
FUSE_HD double div_d(double a, double b) { return a/b; }
FUSE_HD float mul_f(float a, float b) { return a*b; }
FUSE_HD float add_f(float a, float b) { return a+b; }
FUSE_HD float sub_f(float a, float b) { return a-b; }
FUSE_HD float div_f(float a, float b) { return a/b; }
FUSE_HD float sqrt_f(float a) { return sqrtf(a); }
#endif

struct Cam {
	double K[9], R[9], C[3], P[12];
};

// AssembleProjectionMatrix (libs/MVS/Camera.cpp:173-180): P = [K R | -K R C]
FUSE_HD void compose(const double* K, const double* R, const double* C, Cam& c) {
	for (int i = 0; i < 9; ++i) { c.K[i] = K[i]; c.R[i] = R[i]; }
	for (int i = 0; i < 3; ++i) c.C[i] = C[i];
	double M[9];
	for (int i = 0; i < 3; ++i)
		for (int j = 0; j < 3; ++j)
			M[3*i+j] = add_d(add_d(mul_d(c.K[3*i], c.R[j]), mul_d(c.K[3*i+1], c.R[3+j])), mul_d(c.K[3*i+2], c.R[6+j]));
	for (int i = 0; i < 3; ++i) {
		c.P[4*i] = M[3*i]; c.P[4*i+1] = M[3*i+1]; c.P[4*i+2] = M[3*i+2];
		c.P[4*i+3] = add_d(add_d(mul_d(M[3*i], -c.C[0]), mul_d(M[3*i+1], -c.C[1])), mul_d(M[3*i+2], -c.C[2]));
	}
}

// Camera::TransformPointI2W(Point3(x, y, depth)) (libs/MVS/Camera.h:339-356), double
FUSE_HD void image_to_world(const Cam& c, int x, int y, float depth, double out[3]) {
	const double z = (double)depth;
	const double cx = div_d(mul_d(sub_d((double)x, c.K[2]), z), c.K[0]), cy = div_d(mul_d(sub_d((double)y, c.K[5]), z), c.K[4]);
	out[0] = add_d(add_d(add_d(mul_d(c.R[0], cx), mul_d(c.R[3], cy)), mul_d(c.R[6], z)), c.C[0]);
	out[1] = add_d(add_d(add_d(mul_d(c.R[1], cx), mul_d(c.R[4], cy)), mul_d(c.R[7], z)), c.C[1]);
	out[2] = add_d(add_d(add_d(mul_d(c.R[2], cx), mul_d(c.R[5], cy)), mul_d(c.R[8], z)), c.C[2]);
}

// R^T n: camera-space normal of the depth-map to world space (SceneDensify.cpp:1526,1554), double sums, float result
FUSE_HD void normal_to_world(const Cam& c, const float* n, float out[3]) {
	const double nx = n[0], ny = n[1], nz = n[2];
	out[0] = (float)add_d(add_d(mul_d(c.R[0], nx), mul_d(c.R[3], ny)), mul_d(c.R[6], nz));
	out[1] = (float)add_d(add_d(mul_d(c.R[1], nx), mul_d(c.R[4], ny)), mul_d(c.R[7], nz));
	out[2] = (float)add_d(add_d(mul_d(c.R[2], nx), mul_d(c.R[5], ny)), mul_d(c.R[8], nz));
}

// Conf2Weight (SceneDensify.cpp:120-122)
FUSE_HD float conf2weight(float conf, float depth) { return div_f(1.f, mul_f(mul_f(fmaxf(sub_f(1.f, conf), 0.03f), depth), depth)); }

// one row of P applied to a float point widened to double; row 2 is Camera::PointDepth (libs/MVS/Camera.cpp:112-115)
FUSE_HD double project_row_d(const double* P, const float pt[3]) {
	return add_d(add_d(add_d(mul_d(P[0], (double)pt[0]), mul_d(P[1], (double)pt[1])), mul_d(P[2], (double)pt[2])), P[3]);
}

// Camera::ProjectPointP3<float> (Camera.h:308-314): double sums, float components
FUSE_HD float project_row(const double* P, const float pt[3]) { return (float)project_row_d(P, pt); }

// The pixel of neighbour B a point falls on: false when it is behind B (pz <= 0) or outside its w x h map.  ROUND2INT
// (libs/Common/Types.h:947-953) is floor(v + 0.5); the range test is made on the rounded float, so a value beyond int (or NaN)
// is outside, as the x86 conversion to INT_MIN makes it on the host.
FUSE_HD bool project_to_pixel(const Cam& c, const float pt[3], int w, int h, float& pz, int& xb, int& yb) {
	const float px = project_row(c.P, pt), py = project_row(c.P+4, pt);
	pz = project_row(c.P+8, pt);
	if (pz <= 0) return false;
	const float fx = floorf(add_f(div_f(px, pz), .5f)), fy = floorf(add_f(div_f(py, pz), .5f));
	if (!(fx >= 0.f && fy >= 0.f && fx < (float)w && fy < (float)h)) return false;
	xb = (int)fx; yb = (int)fy;
	return true;
}

// IsDepthSimilar(pt.z, depthB) (libs/Common/Util.inl:797-809)
FUSE_HD bool depth_similar(float pz, float depthB, float th) { return div_f(fabsf(sub_f(pz, depthB)), pz) < th; }

FUSE_HD float dot3(const float a[3], const float b[3]) { return add_f(add_f(mul_f(a[0], b[0]), mul_f(a[1], b[1])), mul_f(a[2], b[2])); }

} // namespace fuse

// ---- the device form: kernel interface ----

// One image as the fusion kernels see it: its maps (device), its claim map (1 = pixel belongs to a point) and its camera.
struct FuseDevView {
	float* depth; const float* normal; const float* conf; const uint8_t* color;
	uint8_t* claim;
	int w, h;
	fuse::Cam cam;
};

// One image's round: candidate c is pixel cand[c] of image a; edge e = c*nNb + k goes to neighbour nb[k], whose pixels are the
// round-local targets [base[k], base[k] + w*h).
struct FuseRound {
	const FuseDevView* views;
	int a, nNb;
	const int* nb;                 // nNb image IDs (device)
	const uint32_t* base;          // nNb target bases (device)
	bool bNormalMap, bColor, bNormal;
	unsigned nMin;
	float thDepth, normalError;
};

// edge types of the round (fixed at its start) and the per-edge / per-candidate states of the fixed point
enum : uint8_t { FE_NONE = 0, FE_CLAIM = 1, FE_ZERO = 2 };
enum : uint8_t { FS_UNKNOWN = 0, FS_LIVE = 1, FS_DEAD = 2 };
enum : uint8_t { FA_UNKNOWN = 0, FA_YES = 1, FA_NO = 2 };

// the outputs of one round: points / normals / colors / offsets start at the round's first point; views / weights / projs are the
// whole arrays, and the round's views start at viewBase
struct FuseOut {
	float* points; float* normals; uint8_t* colors;
	uint32_t* offsets; uint32_t* views; float* weights; uint16_t* projs;
	uint32_t viewBase;
};

cudaError_t fuse_launch_any_positive(const float* depth, size_t n, int* flag, cudaStream_t s);
cudaError_t fuse_launch_candidates(const float* depth, const uint8_t* claim, size_t n, uint8_t* flags, unsigned long long* nDepths,
	cudaStream_t s);
cudaError_t fuse_select(void* tmp, size_t& tmpBytes, const uint8_t* flags, uint32_t* out, uint32_t* nOut, size_t n, cudaStream_t s);
cudaError_t fuse_launch_classify(const FuseRound& R, const uint32_t* cand, uint32_t nCand, uint8_t* typ, uint32_t* tgt, cudaStream_t s);
cudaError_t fuse_launch_gather_keys(const uint32_t* tgt, const uint32_t* edges, uint32_t nEdges, uint32_t* keys, cudaStream_t s);
cudaError_t fuse_sort(void* tmp, size_t& tmpBytes, const uint32_t* keysIn, uint32_t* keysOut, const uint32_t* valsIn, uint32_t* valsOut,
	uint32_t n, int endBit, cudaStream_t s);
cudaError_t fuse_launch_shared(const uint32_t* keys, uint32_t nEdges, unsigned long long* shared, cudaStream_t s);
cudaError_t fuse_launch_walk(const uint32_t* keys, const uint32_t* edges, uint32_t nEdges, int nNb, const uint8_t* acc, uint8_t* status,
	cudaStream_t s);
cudaError_t fuse_launch_decide(const FuseRound& R, uint32_t nCand, const uint8_t* typ, const uint8_t* status, uint8_t* acc,
	uint32_t* undecided, cudaStream_t s);
cudaError_t fuse_launch_count(const FuseRound& R, uint32_t nCand, const uint8_t* typ, const uint8_t* status, const uint8_t* acc,
	uint32_t* isPoint, uint32_t* nViews, cudaStream_t s);
cudaError_t fuse_scan(void* tmp, size_t& tmpBytes, const uint32_t* in, uint32_t* out, uint32_t n, cudaStream_t s);
cudaError_t fuse_launch_totals(const uint32_t* isPoint, const uint32_t* pointId, const uint32_t* nViews, const uint32_t* viewOff,
	uint32_t n, uint32_t* out, cudaStream_t s);
cudaError_t fuse_launch_assemble(const FuseRound& R, const uint32_t* cand, uint32_t nCand, const uint8_t* typ, const uint32_t* tgt,
	const uint8_t* status, const uint8_t* acc, const uint32_t* pointId, const uint32_t* viewOff, const FuseOut& O, cudaStream_t s);
