// sgm_common.cuh — the interface between the SGM kernels (sgm_kernels.cu, sgm_cost_tc.cu, sgm_front.cu, sgm_tsgm.cu) and the
// host driver (sgm_host.cu): the parameter blocks the kernels receive and the launch functions that start them.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>
#include "../../include/b200mvs.h"

// one pixel of the ragged cost volume: costs[idx .. idx + dmax-dmin) (the device view of b200mvs_sgm_pixel)
struct SGMPixel { unsigned long long idx; short dmin, dmax; int pad; };
static_assert(sizeof(SGMPixel) == sizeof(b200mvs_sgm_pixel), "pixel record layout");
static_assert(offsetof(SGMPixel, idx) == offsetof(b200mvs_sgm_pixel, idx) && offsetof(SGMPixel, dmin) == offsetof(b200mvs_sgm_pixel, dmin) &&
	offsetof(SGMPixel, dmax) == offsetof(b200mvs_sgm_pixel, dmax), "pixel record layout");

struct SGMParams {
	const float* lgray; const uchar3* lbgr; const float* rgray;
	int w, h, vw, vh;           // image size, valid-region size (w-6, h-6)
	const SGMPixel* px;
	uint8_t* costs; uint16_t* accums;
	int P1;
	uint16_t P2s[256];
	int maxNumDisp;
};

constexpr int SGM_HW = 3, SGM_NT = 49;   // half width and taps of the 7x7 WZNCC window
constexpr int SGM_NO_DISP = 32767;       // invalid disparity (NO_DISP, libs/MVS/SemiGlobalMatcher.h:68)
constexpr int SGM_MAX_DISP = 256;        // disparities per pixel: the warp-per-scanline kernel keeps one line of at most this many

// statistics of a pixel map, over its valid pixels unless stated (sgm_launch_map_stats); the kernel writes the fields in this order
struct SGMMapStats {
	int maxNum;           // largest disparity count dmax-dmin
	int dminLo, dminHi;   // min / max of dmin
	int dmaxLo, dmaxHi;   // min / max of dmax
	int idxLowBits;       // OR of (idx & 15)
	int notDense;         // 1: an invalid pixel, or idx != pixel index x disparity count
	int overflow;         // 1: a slice ends beyond numCosts
};
static_assert(sizeof(SGMMapStats) == 8*sizeof(int), "pixel-map statistics layout");

// sgm_kernels.cu
cudaError_t sgm_configure_device();
cudaError_t sgm_launch_map_stats(const SGMPixel* px, int n, unsigned long long numCosts, SGMMapStats* out, cudaStream_t s);
cudaError_t sgm_launch_cost(const SGMParams& P, cudaStream_t s);
cudaError_t sgm_launch_aggregate(const SGMParams& P, int dir, bool store, cudaStream_t s);
cudaError_t sgm_launch_aggregate_uniform(const SGMParams& P, int dir, int dmin, int num, bool ring, cudaStream_t s);
cudaError_t sgm_launch_wta(const SGMParams& P, int nVol, unsigned long long volStride, const uint16_t* more, int16_t* disparity, uint16_t* cost, cudaStream_t s);
cudaError_t sgm_launch_wta_uniform(const SGMParams& P, const uint16_t* second, int dmin, int num, int16_t* disparity, uint16_t* cost, cudaStream_t s);
cudaError_t sgm_launch_cross_check(int16_t* l2r, const int16_t* r2l, int w, int h, int th, cudaStream_t s);
cudaError_t sgm_launch_refine(const SGMPixel* px, const uint16_t* accums, int16_t* disparity, int n, int steps, cudaStream_t s);
// sgm_cost_tc.cu
cudaError_t sgm_cost_tc_configure();
bool sgm_cost_tc_supports(int num);
cudaError_t sgm_cost_tc_launch(const SGMParams& P, int dmin, int num, cudaStream_t s);
// sgm_front.cu (FrontArgs: sgm_front_sched.h)
struct FrontArgs;
cudaError_t sgm_front_launch(const SGMParams& P, const FrontArgs& A, int blocks, int pd, cudaStream_t s);
int sgm_front_blocks_per_sm(int num, int pd);
bool sgm_front_supports(int num);
// sgm_tsgm.cu
size_t tsgm_range_map_scratch(size_t n);
cudaError_t tsgm_launch_range_map(const int16_t* D, int W, int H, const uint8_t* mask, int W2, int H2, int minNumDisp, int minNumDispInvalid,
	short2* ranges, SGMPixel* px, void* scratch, unsigned long long* total, cudaStream_t s);
cudaError_t tsgm_launch_flip(const int16_t* l2r, int16_t* r2l, int W, int H, unsigned* keys, cudaStream_t s);
cudaError_t tsgm_launch_upscale_mask(const uint8_t* m, int W, int H, uint8_t* m2, int W2, int H2, cudaStream_t s);
cudaError_t tsgm_launch_extract_mask(const int16_t* D, uint8_t* M, int W, int H, int thValid, cudaStream_t s);
cudaError_t tsgm_launch_speckles(int16_t* D, int W, int H, int newVal, int maxSpeckleSize, int maxDiff, int* labels, int* sizes, cudaStream_t s);
cudaError_t tsgm_launch_area_u8(const uint8_t* src, int sw, int sh, int cn, uint8_t* dst, int dw, int dh, int k, cudaStream_t s);
cudaError_t tsgm_launch_fill(int16_t* d, size_t n, int16_t v, cudaStream_t s);
cudaError_t tsgm_launch_minmax(const int16_t* d, size_t n, int* out2, cudaStream_t s);
cudaError_t tsgm_launch_dense_map(SGMPixel* px, size_t n, int lo, int hi, cudaStream_t s);
