// cloud_remove.cu — the removals of the dense point cloud behind the C-ABI, with their kernels (DESIGN.md §5.8):
//  - the order cList::RemoveAt leaves a cloud in after RFOREACH(i) if (remove[i]) RemovePoint(i) (libs/Common/List.h:1630-1636),
//    resolved on the device by pointer jumping, and the compaction of a device cloud by that order;
//  - the remove masks of PointCloud::RemovePointsOutside (the ROI crop, OBB3f::Intersects, libs/Common/OBB.inl:388-400) and
//    PointCloud::RemoveMinViews (libs/MVS/PointCloud.cpp:82-93);
//  - Scene::EstimateROI (libs/MVS/Scene.cpp:1652-1740): the cameras on the host, the core points and their box on the device.
// Each mask and EstimateROI has a host form (plain host code, the specification) and a device form that agree bit for bit.  The
// kernels are private to this file: no other call shares them.  The CPU restatements used by the tests are in
// oracle/removal_oracle.py.
#include <float.h>
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <algorithm>
#include <vector>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>
#include "host_ctx.h"
#include "cloud_common.cuh"

namespace {

using fuse::add_f; using fuse::sub_f; using fuse::mul_f; using fuse::add_d; using fuse::mul_d;

constexpr int TPB = 256;
constexpr uint32_t NO_LINK = 0xFFFFFFFFu;

inline unsigned blocks(size_t n) { return (unsigned)std::max<size_t>((n+TPB-1)/TPB, 1); }

// ---- the removal order ----
//
// Let m points be removed, r_0 > r_1 > ... > r_{m-1} their slots.  The loop visits them in that order, and step t (size n - t
// before it) moves the content of the tail slot n-1-t into slot r_t.  A slot is written only by the step that removes it, so
// the tail slot j = n-1-t still holds point j unless j was removed by an earlier step s(j) = #{removed slots > j} < t, in which
// case it holds what step s(j) moved: value(t) = j when j is kept, else value(s(j)).  (s(j) = t only when r_t = j: the removed
// slot is the tail itself, which is dropped.)  These links point to strictly earlier steps, so they form chains that end at a
// kept point, and log2(n) rounds of pointer jumping resolve every one.  Afterwards slot k < n - m holds point k when k is kept,
// and value(s(k)) when k was removed.

// remove[i] != 0 as a count, for the exclusive scan P[i] = #{removed slots < i}, i <= n
struct Removed {
	const uint8_t* remove; uint32_t n;
	__host__ __device__ uint32_t operator()(uint32_t i) const { return i < n && remove[i] != 0; }
};

// step t's link: (earlier step, 0), or (NO_LINK, the point it moves)
__global__ void k_order_links(const uint8_t* __restrict__ remove, const uint32_t* __restrict__ P, uint32_t n, uint2* __restrict__ link) {
	const uint32_t t = blockIdx.x*blockDim.x + threadIdx.x, m = P[n];
	if (t >= m) return;
	const uint32_t j = n-1-t;
	const uint32_t s = remove[j] ? m - P[j] - 1 : t;
	link[t] = s < t ? make_uint2(s, 0) : make_uint2(NO_LINK, j);
}

// one round of pointer jumping
__global__ void k_order_jump(const uint32_t* __restrict__ P, uint32_t n, const uint2* __restrict__ in, uint2* __restrict__ out) {
	const uint32_t t = blockIdx.x*blockDim.x + threadIdx.x;
	if (t >= P[n]) return;
	uint2 a = in[t];
	if (a.x != NO_LINK) {
		const uint2 b = in[a.x];
		a = b.x == NO_LINK ? b : make_uint2(b.x, 0);
	}
	out[t] = a;
}

__global__ void k_order_write(const uint8_t* __restrict__ remove, const uint32_t* __restrict__ P, uint32_t n, const uint2* __restrict__ link,
	uint32_t* __restrict__ order)
{
	const uint32_t k = blockIdx.x*blockDim.x + threadIdx.x, m = P[n];
	if (k >= n - m) return;
	order[k] = remove[k] ? link[m - P[k] - 1].y : k;
}

// ---- the compaction ----

// the view count of kept point k (0 past the end or for an order entry out of range, which the gather reports)
struct KeptViews {
	const uint32_t *order, *off; uint32_t nKept, n;
	__host__ __device__ uint32_t operator()(uint32_t k) const {
		if (k >= nKept) return 0;
		const uint32_t i = order[k];
		return i < n ? off[i+1] - off[i] : 0;
	}
};

struct CompactBufs {
	const float *points, *normals, *weights; const uint8_t* colors;
	const uint32_t *off, *views; const uint16_t* projs;
	float *oPoints, *oNormals, *oWeights; uint8_t* oColors;
	const uint32_t* oOff; uint32_t* oViews; uint16_t* oProjs;
};

// one thread per kept point: its fields, and its view list from off[i] to oOff[k]
__global__ void k_compact(const uint32_t* __restrict__ order, uint32_t nKept, uint32_t n, const CompactBufs b, int* bad) {
	const uint32_t k = blockIdx.x*blockDim.x + threadIdx.x;
	if (k >= nKept) return;
	const uint32_t i = order[k];
	if (i >= n) { atomicOr(bad, 1); return; }
	for (int c = 0; c < 3; ++c) {
		if (b.points) b.oPoints[3*(size_t)k+c] = b.points[3*(size_t)i+c];
		if (b.normals) b.oNormals[3*(size_t)k+c] = b.normals[3*(size_t)i+c];
		if (b.colors) b.oColors[3*(size_t)k+c] = b.colors[3*(size_t)i+c];
	}
	if (!b.off) return;
	const uint32_t src = b.off[i], len = b.off[i+1] - src, dst = b.oOff[k];
	for (uint32_t e = 0; e < len; ++e) {
		b.oViews[dst+e] = b.views[src+e];
		if (b.weights) b.oWeights[dst+e] = b.weights[src+e];
		if (b.projs) { b.oProjs[2*(size_t)(dst+e)] = b.projs[2*(size_t)(src+e)]; b.oProjs[2*(size_t)(dst+e)+1] = b.projs[2*(size_t)(src+e)+1]; }
	}
}

// ---- the masks ----

// OBB3f as Intersects reads it: m_rot row-major, m_pos, m_ext (the border already applied)
struct Box { float rot[9], pos[3], ext[3]; };

// !OBB3f::Intersects(X): dist = m_rot * (X - m_pos) in float, each row summed in Eigen's order for three terms, r0 + (r1 + r2),
// without FMA contraction; the point is inside when |dist[a]| <= m_ext[a] on every axis (a NaN is outside)
FUSE_HD uint8_t outside(const Box& B, const float* X) {
	const float d[3] = {sub_f(X[0], B.pos[0]), sub_f(X[1], B.pos[1]), sub_f(X[2], B.pos[2])};
	bool in = true;
	for (int a = 0; a < 3; ++a) {
		const float* r = B.rot + 3*a;
		const float v = add_f(mul_f(r[0], d[0]), add_f(mul_f(r[1], d[1]), mul_f(r[2], d[2])));
		in = in && fabsf(v) <= B.ext[a];
	}
	return !in;
}

// the ROI of DenseReconstruction (SceneDensify.cpp:1728): fBorderROI > 0 enlarges the extent by that factor (EnlargePercent),
// < 0 by -fBorderROI (Enlarge), 0 keeps it
Box roi_box(const float* rot, const float* pos, const float* ext, float fBorderROI) {
	Box B;
	memcpy(B.rot, rot, sizeof(B.rot)); memcpy(B.pos, pos, sizeof(B.pos)); memcpy(B.ext, ext, sizeof(B.ext));
	for (int a = 0; a < 3; ++a)
		B.ext[a] = fBorderROI > 0 ? B.ext[a]*fBorderROI : fBorderROI < 0 ? B.ext[a] + -fBorderROI : B.ext[a];
	return B;
}

__global__ void k_outside(const float* __restrict__ points, uint32_t n, const Box B, uint8_t* __restrict__ remove) {
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i < n) remove[i] = outside(B, points + 3*(size_t)i);
}

__global__ void k_min_views(const uint32_t* __restrict__ off, uint32_t n, uint32_t th, uint8_t* __restrict__ remove) {
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i < n) remove[i] = off[i+1] - off[i] < th;
}

// ---- EstimateROI ----

// the third row of an image's projection matrix (Camera::PointDepth); valid: Image::IsValid (a positive size in the table)
struct RoiCam { double p[4]; int valid; };

// Camera::PointDepth(X) (Camera.cpp:112-115): P(2,0) x + P(2,1) y + P(2,2) z + P(2,3), left to right, in double
FUSE_HD double point_depth(const RoiCam& c, const float* X) {
	return add_d(add_d(add_d(mul_d(c.p[0], (double)X[0]), mul_d(c.p[1], (double)X[1])), mul_d(c.p[2], (double)X[2])), c.p[3]);
}

// a core point: a valid view of it sees it at a depth below lim = sceneRadius * 2.0f (Scene.cpp:1719-1731)
FUSE_HD bool core_point(const RoiCam* cams, const float* X, const uint32_t* views, uint32_t a, uint32_t b, double lim) {
	for (uint32_t j = a; j < b; ++j) {
		const RoiCam& c = cams[views[j]];
		if (c.valid && point_depth(c, X) < lim) return true;
	}
	return false;
}

// the box of the core points as box_key minima and maxima, and their count; bad: a view ID not below nImages, or offsets that do
// not start at 0 or are not monotone
__global__ void k_roi_core(const float* __restrict__ points, uint32_t n, const uint32_t* __restrict__ off, const uint32_t* __restrict__ views,
	const RoiCam* __restrict__ cams, uint32_t nImages, double lim, unsigned* box, unsigned long long* count, int* bad)
{
	unsigned lo[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, hi[3] = {0u, 0u, 0u};
	unsigned cnt = 0; bool ok = true;
	for (uint32_t i = blockIdx.x*blockDim.x + threadIdx.x; i < n; i += gridDim.x*blockDim.x) {
		const uint32_t a = off[i], b = off[i+1];
		if (a > b || (i == 0 && a != 0)) { ok = false; continue; }
		bool ids = true;
		for (uint32_t j = a; j < b; ++j) ids &= views[j] < nImages;
		if (!ids) { ok = false; continue; }
		const float* X = points + 3*(size_t)i;
		if (!core_point(cams, X, views, a, b, lim)) continue;
		++cnt;
		for (int c = 0; c < 3; ++c) { const unsigned k = box_key(X[c]); lo[c] = min(lo[c], k); hi[c] = max(hi[c], k); }
	}
	for (int c = 0; c < 3; ++c) { lo[c] = __reduce_min_sync(0xFFFFFFFFu, lo[c]); hi[c] = __reduce_max_sync(0xFFFFFFFFu, hi[c]); }
	cnt = __reduce_add_sync(0xFFFFFFFFu, cnt);
	const bool all = __all_sync(0xFFFFFFFFu, ok);
	if ((threadIdx.x & 31) == 0) {
		if (cnt) {
			for (int c = 0; c < 3; ++c) { atomicMin(box+c, lo[c]); atomicMax(box+3+c, hi[c]); }
			atomicAdd(count, (unsigned long long)cnt);
		}
		if (!all) atomicOr(bad, 1);
	}
}

// cList::GetMedian of floats (List.h:668-678): the middle value, or for an even count the float mean of the two middle values
float median(std::vector<float> v) {
	std::sort(v.begin(), v.end());
	const size_t h = v.size() >> 1;
	return v.size() % 2 ? v[h] : (v[h-1] + v[h]) / 2.f;
}

// The camera half of Scene::EstimateROI (Scene.cpp:1652-1711) in the reference's types and order: the cameras of the valid
// images (cams, per image), and the radius whose double bounds the depth of a core point.  -> false: no ROI (mode 0, fewer than 3
// valid images, or a refusal of mode 2).
bool roi_cameras(const b200mvs_fuse_view* images, int nImages, int mode, std::vector<RoiCam>& cams, double& lim) {
	cams.assign(nImages, RoiCam{});
	std::vector<int> valid;
	for (int i = 0; i < nImages; ++i) {
		fuse::Cam cam;
		fuse::compose(images[i].K, images[i].R, images[i].C, cam);
		for (int a = 0; a < 4; ++a) cams[i].p[a] = cam.P[8+a];
		cams[i].valid = images[i].width > 0 && images[i].height > 0;
		if (cams[i].valid) valid.push_back(i);
	}
	const size_t nc = valid.size();
	if (mode == 0 || nc < 3) return false;
	std::vector<float> x(nc), y(nc), z(nc);
	float nx = 0, ny = 0, nz = 0;   // std::accumulate in float, in camera order
	for (size_t i = 0; i < nc; ++i) {
		const b200mvs_fuse_view& I = images[valid[i]];
		x[i] = (float)I.C[0]; y[i] = (float)I.C[1]; z[i] = (float)I.C[2];
		nx += (float)I.R[6]; ny += (float)I.R[7]; nz += (float)I.R[8];   // Camera::Direction() = R.row(2)
	}
	const double center[3] = {median(x), median(y), median(z)};
	double dir[3] = {nx/(float)nc, ny/(float)nc, nz/(float)nc};
	const float len = (float)sqrt(dir[0]*dir[0] + dir[1]*dir[1] + dir[2]*dir[2]);
	if (!(fabsf(len) < 0.0001f))   // !ISZERO
		for (double& d: dir) d /= len;
	if (len > (float)M_SQRT2/2.f && mode == 2) return false;
	auto distance = [&](const b200mvs_fuse_view& I, const double* X) {
		const double r[3] = {X[0]-I.C[0], X[1]-I.C[1], X[2]-I.C[2]};
		return (float)sqrt(r[0]*r[0] + r[1]*r[1] + r[2]*r[2]);
	};
	std::vector<float> dist(nc);
	for (size_t i = 0; i < nc; ++i) dist[i] = distance(images[valid[i]], center);
	const float shift = tanf(asinf(std::min(std::max(len, 0.f), 0.999f))) * median(dist);
	double sceneCenter[3];
	for (int a = 0; a < 3; ++a) sceneCenter[a] = center[a] + (double)shift*dir[a];
	float radius = 0;
	for (size_t i = 0; i < nc; ++i) {
		const double* p = cams[valid[i]].p;
		if (p[0]*sceneCenter[0] + p[1]*sceneCenter[1] + p[2]*sceneCenter[2] + p[3] <= 0 && mode == 2) return false;
		const float d = distance(images[valid[i]], sceneCenter);
		radius = i ? std::max(radius, d) : d;
	}
	lim = (double)(radius*2.0f);
	return true;
}

// obb.Set(AABB3f(core points).EnlargePercent(scale)) (Scene.cpp:1732, AABB.inl:109-115, OBB.inl:55-60)
void roi_obb(const float lo[3], const float hi[3], float scale, float* rot, float* pos, float* ext) {
	for (int a = 0; a < 9; ++a) rot[a] = a % 4 == 0;
	for (int a = 0; a < 3; ++a) {
		const float delta = (hi[a] - lo[a]) * (scale - 1.f) / 2.f;
		const float mn = lo[a] - delta, mx = hi[a] + delta;
		pos[a] = (mx + mn) * 0.5f;
		ext[a] = (mx - mn) / 2.f;
	}
}

// the checks both EstimateROI forms make before anything is read
int roi_args(b200mvs_ctx* ctx, const float* points, uint64_t n, const uint32_t* off, const uint32_t* views, const b200mvs_fuse_view* images,
	int nImages, int mode, float scale, const float* rot, const float* pos, const float* ext, const int* bounded)
{
	if (!rot || !pos || !ext || !bounded) return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: null pointer");
	if (mode < 0 || mode > 2) return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: nEstimateROI out of [0, 2]");
	if (!(scale > 0)) return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: scale must be positive");
	if (n > 0x7FFFFFFFull) return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: more than 2^31 - 1 points");
	if (n > 0 && (!points || !off || !views)) return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: null pointer");
	if (nImages < 0 || (nImages > 0 && !images)) return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: bad image table");
	return B200MVS_OK;
}

const char* const ROI_BAD_VIEWS = "EstimateROI: the view offsets do not start at 0 or are not monotone, or a view ID is not below nImages";

} // namespace

extern "C" {

int b200mvs_pointcloud_remove_order_device(b200mvs_ctx* ctx, const uint8_t* remove, uint64_t n, uint32_t* order, uint64_t* nKept,
	void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!nKept || (n && (!remove || !order))) return fail(ctx, B200MVS_ERR_ARG, "remove order: null pointer");
	if (n > 0x7FFFFFFEull) return fail(ctx, B200MVS_ERR_ARG, "remove order: more than 2^31 - 2 points");
	if (n == 0) { *nKept = 0; return B200MVS_OK; }
	CK(cudaSetDevice(ctx->device));
	if (!on_device(ctx, remove) || !on_device(ctx, order))
		return fail(ctx, B200MVS_ERR_ARG, "remove order: a buffer is not in device memory of the context's device");
	cudaStream_t s = stream_of(ctx, stream);
	const uint32_t N = (uint32_t)n;
	auto removed = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), Removed{remove, N});
	size_t cubBytes;
	CK(cub_reserve(ctx->pcCub, cubBytes, [&](void* tmp, size_t& bytes) {
		return cub::DeviceScan::ExclusiveSum(tmp, bytes, removed, (uint32_t*)nullptr, (int)N+1, (cudaStream_t)nullptr);
	}));
	Carve scratch(ctx->pcScratch);
	uint32_t* P; uint2 *A, *B;
	scratch.take(P, (size_t)N+1); scratch.take(A, N); scratch.take(B, N);
	CK(scratch.commit());
	ctx->launches = 0;
	CK(cub::DeviceScan::ExclusiveSum(ctx->pcCub.p, cubBytes, removed, P, (int)N+1, s));
	k_order_links<<<blocks(N), TPB, 0, s>>>(remove, P, N, A);
	CK(cudaGetLastError());
	ctx->launches += 2;
	// a chain has fewer than n links, and each round doubles the links a step spans
	for (uint64_t span = 1; span < n; span *= 2) {
		k_order_jump<<<blocks(N), TPB, 0, s>>>(P, N, A, B);
		CK(cudaGetLastError());
		std::swap(A, B);
		++ctx->launches;
	}
	k_order_write<<<blocks(N), TPB, 0, s>>>(remove, P, N, A, order);
	CK(cudaGetLastError());
	++ctx->launches;
	uint32_t m = 0;
	CK(cudaMemcpyAsync(&m, P + N, sizeof(m), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	*nKept = n - m;
	return B200MVS_OK;
}

int b200mvs_pointcloud_compact_device(b200mvs_ctx* ctx, const uint32_t* order, uint64_t nKept, uint64_t nPoints, const float* points,
	const float* normals, const uint8_t* colors, const uint32_t* viewOffsets, const uint32_t* views, const float* weights,
	const uint16_t* projs, float* outPoints, float* outNormals, uint8_t* outColors, uint32_t* outViewOffsets, uint32_t* outViews,
	float* outWeights, uint16_t* outProjs, uint64_t* nViewsKept, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!nViewsKept) return fail(ctx, B200MVS_ERR_ARG, "compact: null pointer");
	if (nPoints > 0x7FFFFFFEull || nKept > nPoints) return fail(ctx, B200MVS_ERR_ARG, "compact: more than 2^31 - 2 points, or nKept above nPoints");
	if ((points && !outPoints) || (normals && !outNormals) || (colors && !outColors) ||
		(viewOffsets && (!views || !outViewOffsets || !outViews || (weights && !outWeights) || (projs && !outProjs))))
		return fail(ctx, B200MVS_ERR_ARG, "compact: a field is given without its output, or view lists without views");
	if (nKept && !order) return fail(ctx, B200MVS_ERR_ARG, "compact: null pointer");
	CK(cudaSetDevice(ctx->device));
	const void* bufs[] = {order, points, normals, colors, viewOffsets, views, weights, projs, outPoints, outNormals, outColors,
		outViewOffsets, outViews, outWeights, outProjs};
	for (const void* p: bufs)
		if (!on_device(ctx, p)) return fail(ctx, B200MVS_ERR_ARG, "compact: a buffer is not in device memory of the context's device");
	cudaStream_t s = stream_of(ctx, stream);
	const uint32_t K = (uint32_t)nKept, N = (uint32_t)nPoints;
	auto lens = thrust::make_transform_iterator(thrust::counting_iterator<uint32_t>(0), KeptViews{order, viewOffsets, K, N});
	size_t cubBytes = 0;
	if (viewOffsets)
		CK(cub_reserve(ctx->pcCub, cubBytes, [&](void* tmp, size_t& bytes) {
			return cub::DeviceScan::ExclusiveSum(tmp, bytes, lens, (uint32_t*)nullptr, (int)K+1, (cudaStream_t)nullptr);
		}));
	ReadBack* rb; CK(read_back(ctx, rb));
	ctx->launches = 0;
	CK(cudaMemsetAsync(&rb->cloudBad, 0, sizeof(int), s));
	if (viewOffsets) {
		CK(cub::DeviceScan::ExclusiveSum(ctx->pcCub.p, cubBytes, lens, outViewOffsets, (int)K+1, s));
		++ctx->launches;
	}
	if (K) {
		const CompactBufs b{points, normals, weights, colors, viewOffsets, views, projs, outPoints, outNormals, outWeights, outColors,
			outViewOffsets, outViews, outProjs};
		k_compact<<<blocks(K), TPB, 0, s>>>(order, K, N, b, &rb->cloudBad);
		CK(cudaGetLastError());
		++ctx->launches;
	}
	int bad = 0; uint32_t total = 0;
	CK(cudaMemcpyAsync(&bad, &rb->cloudBad, sizeof(int), cudaMemcpyDeviceToHost, s));
	if (viewOffsets) CK(cudaMemcpyAsync(&total, outViewOffsets + K, sizeof(total), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	if (bad) return fail(ctx, B200MVS_ERR_ARG, "compact: an order entry is not below nPoints");
	*nViewsKept = total;
	return B200MVS_OK;
}

int b200mvs_point_cloud_outside_obb(const float* points, uint64_t nPoints, const float* rot, const float* pos, const float* ext,
	float fBorderROI, uint8_t* remove)
{
	if (!rot || !pos || !ext || (nPoints && (!points || !remove))) return B200MVS_ERR_ARG;
	const Box B = roi_box(rot, pos, ext, fBorderROI);
	for (uint64_t i = 0; i < nPoints; ++i) remove[i] = outside(B, points + 3*i);
	return B200MVS_OK;
}

int b200mvs_point_cloud_outside_obb_device(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const float* rot, const float* pos,
	const float* ext, float fBorderROI, uint8_t* remove, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!rot || !pos || !ext || (nPoints && (!points || !remove))) return fail(ctx, B200MVS_ERR_ARG, "outside OBB: null pointer");
	if (nPoints >= 0xFFFFFFFFull) return fail(ctx, B200MVS_ERR_ARG, "outside OBB: more than 2^32 - 2 points");
	if (nPoints == 0) return B200MVS_OK;
	CK(cudaSetDevice(ctx->device));
	if (!on_device(ctx, points) || !on_device(ctx, remove))
		return fail(ctx, B200MVS_ERR_ARG, "outside OBB: a buffer is not in device memory of the context's device");
	ctx->launches = 1;
	k_outside<<<blocks(nPoints), TPB, 0, stream_of(ctx, stream)>>>(points, (uint32_t)nPoints, roi_box(rot, pos, ext, fBorderROI), remove);
	CK(cudaGetLastError());
	return B200MVS_OK;
}

int b200mvs_point_cloud_min_views(const uint32_t* viewOffsets, uint64_t nPoints, uint32_t thMinViews, uint8_t* remove) {
	if (nPoints && (!viewOffsets || !remove)) return B200MVS_ERR_ARG;
	for (uint64_t i = 0; i < nPoints; ++i) remove[i] = viewOffsets[i+1] - viewOffsets[i] < thMinViews;
	return B200MVS_OK;
}

int b200mvs_point_cloud_min_views_device(b200mvs_ctx* ctx, const uint32_t* viewOffsets, uint64_t nPoints, uint32_t thMinViews,
	uint8_t* remove, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (nPoints && (!viewOffsets || !remove)) return fail(ctx, B200MVS_ERR_ARG, "min views: null pointer");
	if (nPoints >= 0xFFFFFFFFull) return fail(ctx, B200MVS_ERR_ARG, "min views: more than 2^32 - 2 points");
	if (nPoints == 0) return B200MVS_OK;
	CK(cudaSetDevice(ctx->device));
	if (!on_device(ctx, viewOffsets) || !on_device(ctx, remove))
		return fail(ctx, B200MVS_ERR_ARG, "min views: a buffer is not in device memory of the context's device");
	ctx->launches = 1;
	k_min_views<<<blocks(nPoints), TPB, 0, stream_of(ctx, stream)>>>(viewOffsets, (uint32_t)nPoints, thMinViews, remove);
	CK(cudaGetLastError());
	return B200MVS_OK;
}

int b200mvs_estimate_roi(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets, const uint32_t* views,
	const b200mvs_fuse_view* images, int nImages, int nEstimateROI, float scale, float* rot, float* pos, float* ext, int* bounded)
{
	if (int rc = roi_args(ctx, points, nPoints, viewOffsets, views, images, nImages, nEstimateROI, scale, rot, pos, ext, bounded))
		return rc;
	*bounded = 0;
	if (nPoints && viewOffsets[0] != 0) return fail(ctx, B200MVS_ERR_ARG, ROI_BAD_VIEWS);
	for (uint64_t i = 0; i < nPoints; ++i) {
		if (viewOffsets[i] > viewOffsets[i+1]) return fail(ctx, B200MVS_ERR_ARG, ROI_BAD_VIEWS);
		for (uint32_t j = viewOffsets[i]; j < viewOffsets[i+1]; ++j)
			if (views[j] >= (uint32_t)nImages) return fail(ctx, B200MVS_ERR_ARG, ROI_BAD_VIEWS);
	}
	std::vector<RoiCam> cams; double lim;
	// no point: the reference's point cloud is not valid
	if (nPoints == 0 || !roi_cameras(images, nImages, nEstimateROI, cams, lim)) return B200MVS_OK;
	unsigned keys[6] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u, 0u, 0u};
	uint64_t count = 0;
	for (uint64_t i = 0; i < nPoints; ++i) {
		const float* X = points + 3*i;
		if (!core_point(cams.data(), X, views, viewOffsets[i], viewOffsets[i+1], lim)) continue;
		for (int a = 0; a < 3; ++a) { keys[a] = std::min(keys[a], box_key(X[a])); keys[3+a] = std::max(keys[3+a], box_key(X[a])); }
		++count;
	}
	if (!count) return B200MVS_OK;
	float lo[3], hi[3];
	for (int a = 0; a < 3; ++a) { lo[a] = box_value(keys[a]); hi[a] = box_value(keys[3+a]); }
	roi_obb(lo, hi, scale, rot, pos, ext);
	*bounded = 1;
	return B200MVS_OK;
}

int b200mvs_estimate_roi_device(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets, const uint32_t* views,
	const b200mvs_fuse_view* images, int nImages, int nEstimateROI, float scale, float* rot, float* pos, float* ext, int* bounded,
	void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (int rc = roi_args(ctx, points, nPoints, viewOffsets, views, images, nImages, nEstimateROI, scale, rot, pos, ext, bounded))
		return rc;
	*bounded = 0;
	if (nPoints == 0) return B200MVS_OK;
	CK(cudaSetDevice(ctx->device));
	if (!on_device(ctx, points) || !on_device(ctx, viewOffsets) || !on_device(ctx, views))
		return fail(ctx, B200MVS_ERR_ARG, "EstimateROI: a buffer is not in device memory of the context's device");
	std::vector<RoiCam> cams; double lim = 0;
	const bool roi = roi_cameras(images, nImages, nEstimateROI, cams, lim);
	cudaStream_t s = stream_of(ctx, stream);
	Carve scratch(ctx->pcScratch);
	RoiCam* dCams; unsigned long long* count;
	scratch.take(dCams, std::max(nImages, 1)); scratch.take(count, 1);
	CK(scratch.commit());
	ReadBack* rb; CK(read_back(ctx, rb));
	ctx->launches = 0;
	if (nImages) CK(cudaMemcpyAsync(dCams, cams.data(), sizeof(RoiCam)*nImages, cudaMemcpyHostToDevice, s));
	CK(cudaMemsetAsync(&rb->cloudBad, 0, sizeof(int), s));
	CK(cudaMemsetAsync(rb->cloudBox, 0xFF, 3*sizeof(unsigned), s));
	CK(cudaMemsetAsync(rb->cloudBox+3, 0, 3*sizeof(unsigned), s));
	CK(cudaMemsetAsync(count, 0, sizeof(*count), s));
	// without an ROI the views are still checked, as the host form checks them; every depth is then below +inf
	k_roi_core<<<std::min(blocks(nPoints), 1024u), TPB, 0, s>>>(points, (uint32_t)nPoints, viewOffsets, views, dCams, (uint32_t)nImages,
		roi ? lim : INFINITY, rb->cloudBox, count, &rb->cloudBad);
	CK(cudaGetLastError());
	ctx->launches = 1;
	int bad = 0; unsigned keys[6]; unsigned long long n = 0;
	CK(cudaMemcpyAsync(&bad, &rb->cloudBad, sizeof(int), cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(keys, rb->cloudBox, sizeof(keys), cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(&n, count, sizeof(n), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));   // also ends the read of `cams`
	if (bad) return fail(ctx, B200MVS_ERR_ARG, ROI_BAD_VIEWS);
	if (!roi || !n) return B200MVS_OK;
	float lo[3], hi[3];
	for (int a = 0; a < 3; ++a) { lo[a] = box_value(keys[a]); hi[a] = box_value(keys[3+a]); }
	roi_obb(lo, hi, scale, rot, pos, ext);
	*bounded = 1;
	return B200MVS_OK;
}

} // extern "C"
