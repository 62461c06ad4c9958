// filter_common.cuh — the interface between the depth-map post-processing kernels (filter_kernels.cu) and the host driver
// (post_host.cu): the parameter blocks the kernels receive and the launch functions that start them.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#define FLT_MAX_NBR 16

struct FltView {
	const float* depth; const float* conf;
	int w, h;
	double fx, fy, cx, cy;
	double R[9], C[3];
};
struct FltParams {
	FltView ref;
	FltView nbr[FLT_MAX_NBR];
	int N, nMinViews, nMinViewsAdjust;
	float thDepthDiff, thStrict, dMin, dMax;
	unsigned long long* zbuf; // N x ref.h x ref.w keys
	float* outDepth; float* outConf;
};

// RemoveSmallSegments: one-way edges between two-way components: arcs[k] = {source label, target label, sizes, seed keys}.
// Internal linkage (seg_launch_label takes the array as void*): the kernel that writes it keeps its symbol name.
namespace {
struct SegArc { int src, dst, srcSize, dstSize, srcKey, dstKey; };
}

cudaError_t flt_launch_filter(const FltParams& P, int maxNbrPixels, bool adjust, cudaStream_t s);
cudaError_t flt_launch_resolve(const unsigned long long* z, const float* nbrConf, size_t np, float* depth, float* conf, cudaStream_t s);
// the two RemoveSmallSegments launchers add the number of kernels they start to `launches`
cudaError_t seg_launch_label(const float* depth, int W, int H, float th, int* labels, int* sizes, int* minKey, void* arcs, int* count, int cap,
	int& launches, cudaStream_t s);
cudaError_t seg_launch_remove(float* depth, float* normal, float* conf, int W, int H, unsigned speckle, const int* labels, int* sizes,
	const int* patch, int nPatch, int& launches, cudaStream_t s);
cudaError_t gap_launch(float* depth, float* normal, float* conf, float* tDepth, float* tNormal, float* tConf, int W, int H, float th, int gap, cudaStream_t s);
