// cloud_common.cuh — the interface between the point-cloud kernels (cloud_kernels.cu) and their host driver (cloud_host.cu):
// DepthMapsData::MergeDepthMaps, EstimatePointColors and EstimatePointNormals.  The arithmetic they share with the fusion
// (compose, image_to_world, normal_to_world, project_row and the correctly rounded helpers) is fuse_common.cuh's.
#pragma once
#include <string.h>
#include "fuse_common.cuh"

// MergeDepthMaps: one image with a depth-map, as the assembly kernel sees it
struct MergeImage {
	const float* depth; const float* normal; const uint8_t* color;   // device maps; normal / color null when not asked for
	int w;
	uint32_t id;                  // the image ID: the one view of its points
	fuse::Cam cam;
};

// One scene image as the colour and normal kernels see it
struct CloudImage {
	const uint8_t* color;         // w x h x 3 (device), or null: the image is empty
	int w, h;
	double P[12];                 // the projection matrix (compose)
	float C[3];                   // Cast<float>(camera.C): the orientation of the normals
};

// What the checks of a call found: one bit per kind of bad input
enum : int { CLOUD_BAD_OFFSETS = 1, CLOUD_BAD_VIEW = 2, CLOUD_NO_VIEW = 4, CLOUD_NOT_FINITE = 8 };

// an order-preserving map of a float onto unsigned (so that atomicMin / atomicMax order floats), and back
FUSE_HD unsigned box_key(float f) {
	unsigned u; memcpy(&u, &f, 4);
	return (u & 0x80000000u) ? ~u : u | 0x80000000u;
}
FUSE_HD float box_value(unsigned k) {
	const unsigned u = (k & 0x80000000u) ? k & 0x7FFFFFFFu : ~k;
	float f; memcpy(&f, &u, 4);
	return f;
}

// The uniform grid of the neighbour search: cell (i, j, k) holds the points with floor((p - lo) / h) = (i, j, k), clamped to
// the grid, in double (the grid need not cover far outliers: they go to the border cells).  Its key is the Morton interleave
// of the three cell coordinates (at most 1024 cells per axis).
constexpr int CLOUD_GRID_MAX_DIM = 1024;
struct CloudGrid {
	double lo[3], h, invH;
	int dim[3];
};

cudaError_t cloud_launch_merge_flags(const float* depth, size_t n, uint8_t* flags, unsigned long long* count, cudaStream_t s);
cudaError_t cloud_launch_merge_bases(const unsigned long long* counts, int nImages, unsigned long long* bases, unsigned long long* total,
	cudaStream_t s);
cudaError_t cloud_launch_merge_assemble(const MergeImage& I, const uint32_t* idx, const uint32_t* nSel, size_t maxSel,
	const unsigned long long* base, float* points, uint16_t* projs, uint32_t* views, uint8_t* colors, float* normals, cudaStream_t s);
cudaError_t cloud_launch_check_views(const uint32_t* offsets, const uint32_t* views, uint32_t n, int nImages, bool needView, int* bad,
	cudaStream_t s);
// box: min x, y, z, max x, y, z as box_key, starting from 0xFFFFFFFF (minima) and 0 (maxima)
cudaError_t cloud_launch_bbox(const float* points, uint32_t n, unsigned* box, int* bad, cudaStream_t s);
// the extent of the grid is estimated from CLOUD_SAMPLE points spread over the cloud (cloud_host.cu, make_grid)
constexpr int CLOUD_SAMPLE = 1024;
cudaError_t cloud_launch_sample(const float* points, uint32_t n, int m, float* out, cudaStream_t s);
cudaError_t cloud_launch_colors(const float* points, uint32_t n, const uint32_t* offsets, const uint32_t* views, const CloudImage* images,
	uint8_t* colors, cudaStream_t s);
cudaError_t cloud_launch_keys(const float* points, uint32_t n, const CloudGrid& g, uint32_t* keys, uint32_t* idx, cudaStream_t s);
cudaError_t cloud_launch_cells(const float* points, const uint32_t* keys, const uint32_t* idx, uint32_t n, const CloudGrid& g,
	float4* sorted, uint32_t* cellStart, uint32_t* cellEnd, cudaStream_t s);
cudaError_t cloud_launch_knn(const float4* sorted, uint32_t n, const uint32_t* cellStart, const uint32_t* cellEnd, const CloudGrid& g,
	int k, uint32_t* indices, cudaStream_t s);
cudaError_t cloud_launch_pca(const float* points, uint32_t n, const uint32_t* indices, int k, const uint32_t* offsets,
	const uint32_t* views, const CloudImage* images, float* normals, cudaStream_t s);
