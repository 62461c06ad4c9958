// cloud_common.cuh — the interface between the point-cloud kernels (cloud_kernels.cu) and their host driver (cloud_host.cu):
// DepthMapsData::MergeDepthMaps, EstimatePointColors, EstimatePointNormals and the visibility counts of Scene::PointCloudFilter.
// The arithmetic they share with the fusion (compose, image_to_world, normal_to_world, project_row, depth_similar and the
// correctly rounded helpers) is fuse_common.cuh's.
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

// Scene::PointCloudFilter (DESIGN.md §5.7): one view v as the visibility kernels see it.  The cones of v share the apex o and
// cosSq; o, R and K also define the pixel cells its points are binned into (a pinhole at o, so that every point of a cone
// projects near the projection of the cone's axis).  binned = false: the view is not binned and all its queries test every point.
constexpr int VIS_CELL = 2;               // pixels per side of a cell
constexpr int VIS_MARGIN = 16;            // pixels the binned rectangle reaches beyond the image on every side
struct VisView {
	float o[3];                   // Cast<float>(C): the apex of the cones
	float cosSq;                  // SQUARE(COS(angle)), angle = float(ComputeFOV(0)/width), on the host
	double cosB, sinB;            // a conservative bound beta on the angle between a VISIBLE point and the axis (cloud_host.cu)
	double R[9];                  // rotation (checked orthonormal when binned)
	double fx, skew, cx, fy, cy;  // K = [fx skew cx; 0 fy cy; 0 0 1]
	int w, h, ncx, ncy;           // image size; cells per row and per column of the binned rectangle
	uint32_t nCells;              // ncx * ncy: the key of a point outside the rectangle
	bool binned;
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
// the entries of the view lists: entryPoint[j] = the point whose list holds entry j
cudaError_t cloud_launch_vis_entries(const uint32_t* offsets, uint32_t n, uint32_t* entryPoint, cudaStream_t s);
// start[k] (k <= nKeys) = the first i with min(keys[i], nKeys) >= k, over n keys sorted ascending (n >= 1)
cudaError_t cloud_launch_vis_starts(const uint32_t* keys, uint32_t n, uint32_t nKeys, uint32_t* start, cudaStream_t s);
// the cell of every point in view V (V.nCells when it is not binned) and the identity permutation
cudaError_t cloud_launch_vis_keys(const VisView& V, const float* points, uint32_t n, uint32_t* keys, uint32_t* idx, cudaStream_t s);
// the binned points in cell order: (x, y, z, original index) for i < cellStart[V.nCells]
cudaError_t cloud_launch_vis_gather(const float* points, const uint32_t* idxSorted, uint32_t n, const uint32_t* binnedCount, float4* sorted,
	cudaStream_t s);
// The nq queries of view V (query q: point qPoint[q]) over the bins, atomically into visibility; the queries the bins cannot
// answer are appended to flagged (*nFlagged counts them), then cloud_launch_vis_exhaustive tests every point for them.
cudaError_t cloud_launch_vis_query(const VisView& V, const uint32_t* qPoint, uint32_t nq, const float* points, const uint32_t* offsets,
	const float4* sorted, const uint32_t* cellStart, int* visibility, uint32_t* flagged, uint32_t* nFlagged, cudaStream_t s);
cudaError_t cloud_launch_vis_exhaustive(const VisView& V, const uint32_t* flagged, const uint32_t* nFlagged, uint32_t maxFlagged,
	const float* points, uint32_t n, const uint32_t* offsets, int* visibility, cudaStream_t s);
