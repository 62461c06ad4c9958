// cloud_host.cu — the point-cloud tail of Scene::DenseReconstruction behind the C-ABI (kernels: cloud_kernels.cu):
//  - DepthMapsData::MergeDepthMaps (libs/MVS/SceneDensify.cpp:1305-1366), the nMinViewsFuse < 2 branch: every valid depth of
//    every depth-map becomes a point seen by its own image.  A host form (the plain loop, the specification) and a device form
//    that agree bit for bit.
//  - EstimatePointColors (libs/MVS/DepthMap.cpp:1429-1465): the colour of the closest view, sampled bilinearly.
//  - EstimatePointNormals (libs/MVS/DepthMap.cpp:1469-1519): PCA over the k nearest points, turned towards the first view.  The
//    neighbour search is exact (DESIGN.md §5.6): a uniform grid in Morton order and a shell-by-shell search per point.
//  - Scene::PointCloudFilter (libs/MVS/SceneDensify.cpp:2226-2360): the visibility counts of every (point, view) cone, exactly
//    those of the single-threaded reference (DESIGN.md §5.7), and the order its removal loop leaves the kept points in.
// The CPU restatements used by the tests are in oracle/point_cloud_oracle.py and oracle/visibility_oracle.cpp.
#include <float.h>
#include <stdint.h>
#include <string.h>
#include <math.h>
#include <vector>
#include <algorithm>
#include <new>
#include "host_ctx.h"
#include "cloud_common.cuh"

namespace {

using fuse::Cam;
static_assert(sizeof(ReadBack::cloudSample) == sizeof(float)*3*CLOUD_SAMPLE, "ReadBack::cloudSample holds CLOUD_SAMPLE points");

// the checks both merge forms make; only `depth`, `normal`, `color`, the size and the camera of a view are read
const char* merge_check(const b200mvs_fuse_view* views, int nViews, bool bColor, bool bNormal) {
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (!v.depth) continue;
		if (v.width <= 0 || v.height <= 0 || v.width > 65535 || v.height > 65535) return "merge: map size out of range";
		if (bColor && !v.color) return "merge: bEstimateColor is set and an image with a depth-map has no colour map";
		// without a normal map, DepthData::GetNormal fits a plane by RANSAC (DepthMap.cpp:147-204), which is not reproduced
		if (bNormal && !v.normal) return "merge: bEstimateNormal is set and an image with a depth-map has no normal map";
	}
	return nullptr;
}

// the view lists of a host cloud: offsets from 0, monotone, IDs below nImages; with needView, no empty list
int check_views_host(b200mvs_ctx* ctx, const uint32_t* off, const uint32_t* views, uint64_t n, int nImages, bool needView) {
	if (off[0] != 0) return fail(ctx, B200MVS_ERR_ARG, "point cloud: the view offsets do not start at 0");
	for (uint64_t i = 0; i < n; ++i) {
		if (off[i] > off[i+1]) return fail(ctx, B200MVS_ERR_ARG, "point cloud: the view offsets are not monotone");
		if (needView && off[i] == off[i+1]) return fail(ctx, B200MVS_ERR_ARG, "point cloud: a point has no view");
	}
	for (uint64_t j = 0; j < off[n]; ++j)
		if (views[j] >= (uint32_t)nImages) return fail(ctx, B200MVS_ERR_ARG, "point cloud: a view ID is not below nImages");
	return B200MVS_OK;
}

int cloud_bad(b200mvs_ctx* ctx, int bad) {
	if (bad & CLOUD_BAD_OFFSETS) return fail(ctx, B200MVS_ERR_ARG, "point cloud: the view offsets do not start at 0 or are not monotone");
	if (bad & CLOUD_BAD_VIEW) return fail(ctx, B200MVS_ERR_ARG, "point cloud: a view ID is not below nImages");
	if (bad & CLOUD_NO_VIEW) return fail(ctx, B200MVS_ERR_ARG, "point cloud: a point has no view");
	if (bad & CLOUD_NOT_FINITE) return fail(ctx, B200MVS_ERR_ARG, "point cloud: a coordinate is not finite");
	return B200MVS_OK;
}

// What sets the per-point cloud calls apart at their entry: the prefix of their messages, whether every point needs a view, whether
// they read the images' colour maps, and the bytes of one point's output
struct CloudCall { const char* what; bool needView, colorMaps; size_t outBytes; };
const CloudCall COLORS{"point colors: ", false, true, 3}, NORMALS{"point normals: ", true, false, 12},
	VISIBILITY{"point visibility: ", false, false, 4};

int refuse(b200mvs_ctx* ctx, const CloudCall& c, const char* why) {
	return fail(ctx, B200MVS_ERR_ARG, (std::string(c.what) + why).c_str());
}

// A per-point call's buffers where its device form reads them (the caller's, or staged by the host form): the n points with their
// view lists, image i's colour map color[i] (null: empty, or not read), and the output
struct CloudBufs {
	const float* points; uint32_t n; const uint32_t *off, *views;
	std::vector<const uint8_t*> color;
	void* out;
};

// the arguments every per-point call shares; refused: the call's own refusal of one of its other arguments, if any
int cloud_args(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* offsets, const uint32_t* views,
	const b200mvs_fuse_view* images, int nImages, const void* out, const char* refused)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (nPoints > 0x7FFFFFFFull) return fail(ctx, B200MVS_ERR_ARG, "point cloud: more than 2^31 - 1 points");
	// every point reads views unless the offsets are bad (refused then anyway)
	if (nPoints > 0 && (!points || !offsets || !views || !out)) return fail(ctx, B200MVS_ERR_ARG, "point cloud: null pointer");
	if (nImages < 0 || (nImages > 0 && !images)) return fail(ctx, B200MVS_ERR_ARG, "point cloud: bad image table");
	return refused ? fail(ctx, B200MVS_ERR_ARG, refused) : B200MVS_OK;
}

// The scene images as the kernels see them, copied to dImages on s; color[i] is image i's colour map where the kernels read it.
// The copy reads `table`, which the caller keeps until it synchronises s.
int upload_images(b200mvs_ctx* ctx, CloudImage* dImages, std::vector<CloudImage>& table, const b200mvs_fuse_view* images,
	int nImages, const std::vector<const uint8_t*>& color, cudaStream_t s)
{
	table.resize(nImages);
	for (int i = 0; i < nImages; ++i) {
		Cam cam;
		fuse::compose(images[i].K, images[i].R, images[i].C, cam);
		CloudImage& t = table[i];
		t.color = color[i]; t.w = images[i].width; t.h = images[i].height;
		memcpy(t.P, cam.P, sizeof(cam.P));
		for (int a = 0; a < 3; ++a) t.C[a] = (float)images[i].C[a];
	}
	if (nImages) CK(cudaMemcpyAsync(dImages, table.data(), sizeof(CloudImage)*nImages, cudaMemcpyHostToDevice, s));
	return B200MVS_OK;
}

// Run the view checks (and with a box, the bounding box, the finite check and the sample of make_grid) of a device cloud, with
// one read-back
int cloud_check(b200mvs_ctx* ctx, const float* points, uint32_t n, const uint32_t* off, const uint32_t* views, int nImages,
	bool needView, float box[6], std::vector<float>* sample, cudaStream_t s)
{
	ReadBack* rb; CK(read_back(ctx, rb));
	CK(cudaMemsetAsync(&rb->cloudBad, 0, sizeof(int), s));
	CK(cudaMemsetAsync(rb->cloudBox, 0xFF, 3*sizeof(unsigned), s));
	CK(cudaMemsetAsync(rb->cloudBox+3, 0, 3*sizeof(unsigned), s));
	if (off) { CK(cloud_launch_check_views(off, views, n, nImages, needView, &rb->cloudBad, s)); ++ctx->launches; }
	if (box) { CK(cloud_launch_bbox(points, n, rb->cloudBox, &rb->cloudBad, s)); ++ctx->launches; }
	const int m = (int)std::min<uint32_t>(n, CLOUD_SAMPLE);
	if (sample) { CK(cloud_launch_sample(points, n, m, rb->cloudSample, s)); ++ctx->launches; }
	int bad = 0; unsigned keys[6];
	CK(cudaMemcpyAsync(&bad, &rb->cloudBad, sizeof(int), cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(keys, rb->cloudBox, sizeof(keys), cudaMemcpyDeviceToHost, s));
	if (sample) {
		sample->resize(3*(size_t)m);
		CK(cudaMemcpyAsync(sample->data(), rb->cloudSample, sizeof(float)*3*m, cudaMemcpyDeviceToHost, s));
	}
	CK(cudaStreamSynchronize(s));
	if (box) for (int a = 0; a < 6; ++a) box[a] = box_value(keys[a]);
	return cloud_bad(ctx, bad);
}

// The grid of n points for k neighbours.  Its extent is robust: per axis, the 0.5 % and 99.5 % quantiles of a sample spread over
// the cloud, widened by 5 % of their distance and kept inside the bounding box, so that a few far outliers (they go to the border
// cells) do not blow up the cells of everything else.  The points of a dense cloud lie on a surface, so the cell size is chosen
// for about k points per cell on a surface as large as half that extent's surface area (DESIGN.md §5.6), and then widened until
// there are at most 1024 cells per axis and 2n + 4096 cells in all.  Any extent and cell size give the same neighbours.
CloudGrid make_grid(const float box[6], const std::vector<float>& sample, uint32_t n, int k) {
	CloudGrid g;
	double e[3], L = 0;
	const size_t m = sample.size()/3;
	std::vector<float> v(m);
	for (int a = 0; a < 3; ++a) {
		for (size_t i = 0; i < m; ++i) v[i] = sample[3*i+a];
		std::sort(v.begin(), v.end());
		const double qlo = v[(size_t)floor(0.005*(m-1))], qhi = v[(size_t)ceil(0.995*(m-1))], margin = 0.05*(qhi-qlo);
		const double lo = std::max((double)box[a], qlo-margin), hi = std::min((double)box[3+a], qhi+margin);
		g.lo[a] = lo; e[a] = hi - lo; L = std::max(L, e[a]);
	}
	const double S = e[0]*e[1] + e[1]*e[2] + e[2]*e[0];
	double h = S > 0 ? sqrt(S*k/n) : L*k/n;
	h = std::max(h, L/(CLOUD_GRID_MAX_DIM-1));
	if (!(h > 0)) h = 1;
	const double cap = 2.0*n + 4096;
	for (;;) {
		double cells = 1;
		for (int a = 0; a < 3; ++a) { g.dim[a] = std::max(1, (int)std::min(ceil(e[a]/h), (double)CLOUD_GRID_MAX_DIM)); cells *= g.dim[a]; }
		if (cells <= cap) break;
		h *= 1.25;
	}
	g.h = h; g.invH = 1.0/h;
	return g;
}

// The exact k nearest neighbours (k <= n) of n points into nbr (n x k), with the checks of the cloud (and of its view lists when off
// is given, each point with a view) and the grid's scratch joining the caller's slices in `scratch`, which this commits before its
// first launch.  nbr may be one of those slices: it is read after the commit.
int grid_knn(b200mvs_ctx* ctx, Carve& scratch, const float* points, uint32_t n, const uint32_t* off, const uint32_t* views,
	int nImages, int k, uint32_t* const& nbr, cudaStream_t s)
{
	size_t cubBytes;
	CK(cub_reserve(ctx->pcCub, cubBytes, [&](void* tmp, size_t& bytes) {
		return fuse_sort(tmp, bytes, nullptr, nullptr, nullptr, nullptr, n, 30, nullptr);
	}));
	float box[6]; std::vector<float> sample;
	if (int rc = cloud_check(ctx, points, n, off, views, nImages, true, box, &sample, s)) return rc;
	const CloudGrid g = make_grid(box, sample, n, k);
	// the grid: keys, the sort by key, the cells
	const size_t nCells = (size_t)g.dim[0]*g.dim[1]*g.dim[2];
	uint32_t *keys, *keysSorted, *idx, *idxSorted, *cellStart, *cellEnd;
	float4* sorted;
	scratch.take(keys, n); scratch.take(keysSorted, n); scratch.take(idx, n); scratch.take(idxSorted, n); scratch.take(sorted, n);
	scratch.take(cellStart, nCells); scratch.take(cellEnd, nCells);
	CK(scratch.commit());
	CK(cloud_launch_keys(points, n, g, keys, idx, s));
	CK(fuse_sort(ctx->pcCub.p, cubBytes, keys, keysSorted, idx, idxSorted, n, 30, s));
	CK(cudaMemsetAsync(cellStart, 0, nCells*4, s));
	CK(cudaMemsetAsync(cellEnd, 0, nCells*4, s));
	CK(cloud_launch_cells(points, keysSorted, idxSorted, n, g, sorted, cellStart, cellEnd, s));
	CK(cloud_launch_knn(sorted, n, cellStart, cellEnd, g, k, nbr, s));
	ctx->launches += 4;
	return B200MVS_OK;
}

// EstimatePointColors on device buffers
int colors_device(b200mvs_ctx* ctx, const CloudBufs& b, const b200mvs_fuse_view* images, int nImages, cudaStream_t s) {
	if (int rc = cloud_check(ctx, b.points, b.n, b.off, b.views, nImages, false, nullptr, nullptr, s)) return rc;
	Carve scratch(ctx->pcScratch);
	CloudImage* dImages;
	scratch.take(dImages, std::max(nImages, 1));
	CK(scratch.commit());
	std::vector<CloudImage> table;
	if (int rc = upload_images(ctx, dImages, table, images, nImages, b.color, s)) return rc;
	CK(cloud_launch_colors(b.points, b.n, b.off, b.views, dImages, (uint8_t*)b.out, s));
	++ctx->launches;
	CK(cudaStreamSynchronize(s));   // the table is read from host memory that ends with this call
	return B200MVS_OK;
}

// EstimatePointNormals on device buffers
int normals_device(b200mvs_ctx* ctx, const CloudBufs& b, const b200mvs_fuse_view* images, int nImages, int k, cudaStream_t s) {
	const int kk = (int)std::min<uint64_t>(k, b.n);
	Carve scratch(ctx->pcScratch);
	uint32_t* nbr; CloudImage* dImages;
	scratch.take(nbr, (size_t)b.n*kk); scratch.take(dImages, std::max(nImages, 1));
	if (int rc = grid_knn(ctx, scratch, b.points, b.n, b.off, b.views, nImages, kk, nbr, s)) return rc;
	std::vector<CloudImage> table;
	if (int rc = upload_images(ctx, dImages, table, images, nImages, b.color, s)) return rc;
	CK(cloud_launch_pca(b.points, b.n, nbr, kk, b.off, b.views, dImages, (float*)b.out, s));
	++ctx->launches;
	CK(cudaStreamSynchronize(s));
	return B200MVS_OK;
}

// The cone parameters of image I and its bins (DESIGN.md §5.7).  angle and cosSq are the reference's expressions in its types
// (SceneDensify.cpp:2295, Ray.h:209-212): ComputeFOV(0) = 2*atan(width/(2 K(0,0))) in double (Image.cpp:209-216), over width, cast
// to float; COS is std::cos of that float.
//
// beta bounds the angle phi between the axis dir and D = P - o of a point P the kernel classifies VISIBLE.  With u = 2^-24 and the
// float rounding of each step: |t - dir.D| <= 2u |dir| |D| (the dot product), fl(|D|^2) >= (1 - 2u) |D|^2, and VISIBLE means
// fl(t^2) > fl(cosSq fl(|D|^2)), so t > sqrt(cosSq) |D| (1 - 2.1u).  The kernel's binned path also requires | |dir|^2 - 1 | <= 16u,
// so |dir| <= 1 + 8u, and then cos(phi) = dir.D / (|dir| |D|) >= sqrt(cosSq) - 12.1u.  beta = acos(sqrt(cosSq) - 16u), plus 1e-6
// rad for the rounding of D itself against the exact P - o (at most ~2u) and of the double arithmetic.  The bins need a rotation
// (angles are kept), K = [fx skew cx; 0 fy cy; 0 0 1], beta below 80 degrees and at most 2^28 cells; otherwise the view is not
// binned and each of its queries tests every point.
VisView vis_view(const b200mvs_fuse_view& I) {
	VisView V;
	memset(&V, 0, sizeof(V));
	for (int a = 0; a < 3; ++a) V.o[a] = (float)I.C[a];
	const float angle = (float)(2*atan((double)I.width/(I.K[0]*2))/I.width);
	const float c = cosf(angle);
	V.cosSq = c*c;
	const double cb = sqrt((double)V.cosSq) - 16.0*FLT_EPSILON/2;
	const double beta = (cb > -1 ? acos(cb) : M_PI) + 1e-6;
	V.cosB = cos(beta); V.sinB = sin(beta);
	memcpy(V.R, I.R, sizeof(V.R));
	V.fx = I.K[0]; V.skew = I.K[1]; V.cx = I.K[2]; V.fy = I.K[4]; V.cy = I.K[5];
	V.w = I.width; V.h = I.height;
	double err = 0;
	for (int r = 0; r < 3; ++r)
		for (int s = 0; s < 3; ++s)
			err = std::max(err, fabs(I.R[r]*I.R[s] + I.R[3+r]*I.R[3+s] + I.R[6+r]*I.R[6+s] - (r == s)));
	const double ncx = ceil((I.width + 2.0*VIS_MARGIN)/VIS_CELL), ncy = ceil((I.height + 2.0*VIS_MARGIN)/VIS_CELL);
	bool finite = true;
	for (int a = 0; a < 9; ++a) finite &= std::isfinite(I.K[a]);
	V.binned = err <= 1e-9 && finite && I.K[3] == 0 && I.K[6] == 0 && I.K[7] == 0 && I.K[8] == 1 && beta < 80*M_PI/180 &&
		ncx*ncy <= (double)(1u << 28);
	if (V.binned) { V.ncx = (int)ncx; V.ncy = (int)ncy; V.nCells = (uint32_t)(ncx*ncy); }
	return V;
}

// the number of key bits of a radix sort of keys up to maxKey
int key_bits(uint32_t maxKey) {
	int b = 1;
	while (b < 32 && (maxKey >> b)) ++b;
	return b;
}

// PointCloudFilter's visibility counts on device buffers: the queries (the entries of the view lists) sorted by view, then per
// view with queries: bin every point by its cell, sort the bins, answer the queries from the bins and the flagged ones by testing
// every point.  One carve of the call's scratch, one read-back of the per-view query ranges.
int visibility_device(b200mvs_ctx* ctx, const CloudBufs& b, const b200mvs_fuse_view* images, int nImages, cudaStream_t s) {
	const float* points = b.points; const uint32_t *off = b.off, *views = b.views; const uint32_t n = b.n;
	int32_t* visibility = (int32_t*)b.out;
	for (int i = 0; i < nImages; ++i)
		if (images[i].width <= 0 || images[i].height <= 0) return fail(ctx, B200MVS_ERR_ARG, "point visibility: image size out of range");
	float box[6];
	if (int rc = cloud_check(ctx, points, n, off, views, nImages, false, box, nullptr, s)) return rc;
	uint32_t nEntries = 0;
	CK(cudaMemcpyAsync(&nEntries, off + n, sizeof(nEntries), cudaMemcpyDeviceToHost, s));
	CK(cudaMemsetAsync(visibility, 0, sizeof(int32_t)*n, s));
	CK(cudaStreamSynchronize(s));
	if (nEntries == 0) return B200MVS_OK;
	std::vector<VisView> V(nImages);
	uint32_t maxCells = 0;
	for (int i = 0; i < nImages; ++i) { V[i] = vis_view(images[i]); maxCells = std::max(maxCells, V[i].nCells); }
	// CUB's temporary storage for both sorts, reserved before the first launch of the call's work
	const int viewBits = key_bits((uint32_t)std::max(nImages-1, 0)), cellBits = key_bits(maxCells);
	size_t cubBytes;
	CK(cub_reserve(ctx->pcCub, cubBytes,
		[&](void* tmp, size_t& bytes) { return fuse_sort(tmp, bytes, nullptr, nullptr, nullptr, nullptr, nEntries, viewBits, nullptr); },
		[&](void* tmp, size_t& bytes) { return fuse_sort(tmp, bytes, nullptr, nullptr, nullptr, nullptr, n, cellBits, nullptr); }));
	Carve scratch(ctx->pcScratch);
	uint32_t *entryPoint, *viewSorted, *qPoint, *viewStart, *keys, *keysSorted, *idx, *idxSorted, *cellStart, *flagged, *nFlagged;
	float4* sorted;
	scratch.take(entryPoint, nEntries); scratch.take(viewSorted, nEntries); scratch.take(qPoint, nEntries);
	scratch.take(viewStart, nImages+1); scratch.take(flagged, nEntries); scratch.take(nFlagged, 1);
	scratch.take(keys, n); scratch.take(keysSorted, n); scratch.take(idx, n); scratch.take(idxSorted, n); scratch.take(sorted, n);
	scratch.take(cellStart, (size_t)maxCells+1);
	CK(scratch.commit());
	CK(cloud_launch_vis_entries(off, n, entryPoint, s));
	CK(fuse_sort(ctx->pcCub.p, cubBytes, views, viewSorted, entryPoint, qPoint, nEntries, viewBits, s));
	CK(cloud_launch_vis_starts(viewSorted, nEntries, (uint32_t)nImages, viewStart, s));
	ctx->launches += 3;
	std::vector<uint32_t> start(nImages+1);
	CK(cudaMemcpyAsync(start.data(), viewStart, sizeof(uint32_t)*(nImages+1), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	for (int v = 0; v < nImages; ++v) {
		const uint32_t nq = start[v+1] - start[v];
		if (!nq) continue;
		CK(cudaMemsetAsync(nFlagged, 0, sizeof(uint32_t), s));
		if (V[v].binned) {
			CK(cloud_launch_vis_keys(V[v], points, n, keys, idx, s));
			CK(fuse_sort(ctx->pcCub.p, cubBytes, keys, keysSorted, idx, idxSorted, n, cellBits, s));
			CK(cloud_launch_vis_starts(keysSorted, n, V[v].nCells, cellStart, s));
			CK(cloud_launch_vis_gather(points, idxSorted, n, cellStart + V[v].nCells, sorted, s));
			ctx->launches += 4;
		}
		CK(cloud_launch_vis_query(V[v], qPoint + start[v], nq, points, off, sorted, cellStart, visibility, flagged, nFlagged, s));
		CK(cloud_launch_vis_exhaustive(V[v], flagged, nFlagged, nq, points, n, off, visibility, s));
		ctx->launches += 2;
	}
	CK(cudaStreamSynchronize(s));
	return B200MVS_OK;
}

// The device form of a per-point call: the shared checks, then form(buffers, stream) on the caller's buffers
template <typename F>
int cloud_device(b200mvs_ctx* ctx, const CloudCall& c, const char* refused, const float* points, uint64_t nPoints,
	const uint32_t* off, const uint32_t* views, const b200mvs_fuse_view* images, int nImages, void* out, void* stream, F&& form)
{
	if (int rc = cloud_args(ctx, points, nPoints, off, views, images, nImages, out, refused)) return rc;
	if (nPoints == 0) return B200MVS_OK;
	CK(cudaSetDevice(ctx->device));
	CloudBufs b{points, (uint32_t)nPoints, off, views, std::vector<const uint8_t*>(nImages, nullptr), out};
	for (int i = 0; c.colorMaps && i < nImages; ++i) {
		b.color[i] = images[i].color;
		if (b.color[i] && (images[i].width <= 0 || images[i].height <= 0)) return refuse(ctx, c, "image size out of range");
		if (!on_device(ctx, b.color[i])) return refuse(ctx, c, "an image is not in device memory of the context's device");
	}
	if (!on_device(ctx, points) || !on_device(ctx, off) || !on_device(ctx, views) || !on_device(ctx, out))
		return refuse(ctx, c, "a buffer is not in device memory of the context's device");
	ctx->launches = 0;
	return form(b, stream_of(ctx, stream));
}

// The host-buffer form of a per-point call: the shared checks, then the caller's buffers staged for form(buffers, stream) and its
// output copied back (HostCall)
template <typename F>
int cloud_host(b200mvs_ctx* ctx, const CloudCall& c, const char* refused, const float* points, uint64_t nPoints,
	const uint32_t* off, const uint32_t* views, const b200mvs_fuse_view* images, int nImages, void* out, b200mvs_stats* stats,
	F&& form)
{
	if (int rc = cloud_args(ctx, points, nPoints, off, views, images, nImages, out, refused)) return rc;
	if (nPoints == 0) return stats ? (memset(stats, 0, sizeof(*stats)), B200MVS_OK) : B200MVS_OK;
	if (int rc = check_views_host(ctx, off, views, nPoints, nImages, c.needView)) return rc;
	CK(cudaSetDevice(ctx->device));
	ctx->launches = 0;
	HostCall call(ctx);
	CloudBufs b{nullptr, (uint32_t)nPoints, nullptr, nullptr, std::vector<const uint8_t*>(nImages, nullptr), nullptr};
	call.in(b.points, points, 12*nPoints); call.in(b.off, off, 4*(nPoints+1)); call.in(b.views, views, 4*(size_t)off[nPoints]);
	for (int i = 0; c.colorMaps && i < nImages; ++i) {
		if (!images[i].color) continue;
		if (images[i].width <= 0 || images[i].height <= 0) return refuse(ctx, c, "image size out of range");
		call.in(b.color[i], images[i].color, 3*(size_t)images[i].width*images[i].height);
	}
	call.out(b.out, out, c.outBytes*nPoints);
	if (int rc = call.stage()) return rc;
	return call.run([&](cudaStream_t s) { return form(b, s); }, stats);
}

// EstimatePointNormals' own refusal
const char* normals_refused(int numNeighbors) {
	return numNeighbors < 1 || numNeighbors > B200MVS_MAX_POINT_NEIGHBORS ? "point normals: numNeighbors out of [1, 32]" : nullptr;
}

} // namespace

extern "C" {

int b200mvs_merge_depth_maps(const b200mvs_fuse_view* views, int nViews, const b200mvs_fuse_params* prm, b200mvs_pointcloud** out) {
	b200mvs_fuse_params def; b200mvs_fuse_default_params(&def);
	if (!prm) prm = &def;
	const bool bColor = prm->bEstimateColor != 0, bNormal = prm->bEstimateNormal != 0;
	if (!views || nViews <= 0 || !out || merge_check(views, nViews, bColor, bNormal)) return B200MVS_ERR_ARG;
	b200mvs_pointcloud* pc = new (std::nothrow) b200mvs_pointcloud;
	if (!pc) return B200MVS_ERR_CUDA;
	pc->offsets.push_back(0);
	// images in index order, pixels in raster order (SceneDensify.cpp:1325-1360)
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (!v.depth) continue;
		Cam cam;
		fuse::compose(v.K, v.R, v.C, cam);
		for (int y = 0; y < v.height; ++y)
			for (int x = 0; x < v.width; ++x) {
				const size_t ia = (size_t)y*v.width + x;
				const float depth = v.depth[ia];
				if (depth == 0) continue;
				double X[3];
				fuse::image_to_world(cam, x, y, depth, X);
				for (int c = 0; c < 3; ++c) pc->points.push_back((float)X[c]);
				pc->views.push_back((uint32_t)i);
				pc->projs.push_back((uint16_t)x); pc->projs.push_back((uint16_t)y);
				if (bColor) for (int c = 0; c < 3; ++c) pc->colors.push_back(v.color[3*ia+c]);
				if (bNormal) {
					float n[3];
					fuse::normal_to_world(cam, v.normal+3*ia, n);
					pc->normals.insert(pc->normals.end(), n, n+3);
				}
				pc->offsets.push_back((uint32_t)pc->views.size());
				if (pc->views.size() >= 0xFFFFFFFFull) { delete pc; return B200MVS_ERR_ARG; }
			}
	}
	pc->nDepths = pc->views.size();
	*out = pc;
	return B200MVS_OK;
}

int b200mvs_merge_depth_maps_device(b200mvs_ctx* ctx, const b200mvs_fuse_view* views, int nViews, const b200mvs_fuse_params* prm,
	b200mvs_pointcloud** out, void* stream, b200mvs_stats* stats)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!views || nViews <= 0 || !out) return fail(ctx, B200MVS_ERR_ARG, "merge: null pointer");
	b200mvs_fuse_params def; b200mvs_fuse_default_params(&def);
	if (!prm) prm = &def;
	const bool bColor = prm->bEstimateColor != 0, bNormal = prm->bEstimateNormal != 0;
	if (const char* why = merge_check(views, nViews, bColor, bNormal)) return fail(ctx, B200MVS_ERR_ARG, why);
	CK(cudaSetDevice(ctx->device));
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (v.depth && (!on_device(ctx, v.depth) || (bNormal && !on_device(ctx, v.normal)) || (bColor && !on_device(ctx, v.color))))
			return fail(ctx, B200MVS_ERR_ARG, "merge: a map is not in device memory of the context's device");
	}
	const auto t0 = std::chrono::steady_clock::now();
	cudaStream_t s = stream_of(ctx, stream);
	ctx->launches = 0;
	// the call's scratch: per image its depth count and first point, the flags of all its pixels, and the selected pixels of one
	// image at a time with their count
	std::vector<size_t> flagOff(nViews, 0);
	size_t flagBytes = 0, maxNp = 0;
	for (int i = 0; i < nViews; ++i)
		if (views[i].depth) {
			const size_t np = (size_t)views[i].width*views[i].height;
			flagOff[i] = flagBytes; flagBytes += np; maxNp = std::max(maxNp, np);
		}
	size_t cubBytes;
	CK(cub_reserve(ctx->pcCub, cubBytes, [&](void* tmp, size_t& bytes) {
		return fuse_select(tmp, bytes, nullptr, nullptr, nullptr, std::max<size_t>(maxNp, 1), nullptr);
	}));
	Carve scratch(ctx->pcScratch);
	unsigned long long *counts, *bases; uint8_t* flags; uint32_t *idx, *nSel;
	scratch.take(counts, nViews); scratch.take(bases, nViews); scratch.take(flags, std::max<size_t>(flagBytes, 1));
	scratch.take(idx, std::max<size_t>(maxNp, 1)); scratch.take(nSel, 1);
	CK(scratch.commit());
	ReadBack* rb; CK(read_back(ctx, rb));
	CK(cudaEventRecord(ctx->ev0, s));
	CK(cudaMemsetAsync(counts, 0, sizeof(unsigned long long)*nViews, s));
	for (int i = 0; i < nViews; ++i)
		if (views[i].depth) {
			CK(cloud_launch_merge_flags(views[i].depth, (size_t)views[i].width*views[i].height, flags+flagOff[i], counts+i, s));
			++ctx->launches;
		}
	CK(cloud_launch_merge_bases(counts, nViews, bases, &rb->mergePoints, s));
	++ctx->launches;
	unsigned long long total = 0;
	CK(cudaMemcpyAsync(&total, &rb->mergePoints, sizeof(total), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	uint64_t d2h = sizeof(total);
	if (total >= 0xFFFFFFFFull) return fail(ctx, B200MVS_ERR_ARG, "merge: more than 2^32 - 2 points");
	// the outputs, carved once now that their size is known
	const size_t N = std::max<size_t>(total, 1);
	Carve outs(ctx->pcOut);
	float *points, *normals = nullptr; uint16_t* projs; uint8_t* colors = nullptr; uint32_t* pviews;
	outs.take(points, 3*N); outs.take(projs, 2*N); outs.take(pviews, N);
	if (bColor) outs.take(colors, 3*N);
	if (bNormal) outs.take(normals, 3*N);
	CK(outs.commit());
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (!v.depth) continue;
		const size_t np = (size_t)v.width*v.height;
		MergeImage I;
		I.depth = v.depth; I.normal = bNormal ? v.normal : nullptr; I.color = bColor ? v.color : nullptr; I.w = v.width; I.id = (uint32_t)i;
		fuse::compose(v.K, v.R, v.C, I.cam);
		CK(fuse_select(ctx->pcCub.p, cubBytes, flags+flagOff[i], idx, nSel, np, s));
		CK(cloud_launch_merge_assemble(I, idx, nSel, np, bases+i, points, projs, pviews, colors, normals, s));
		ctx->launches += 2;
	}
	CK(cudaEventRecord(ctx->ev1, s));
	const DeviceCloud cloud{total, total, bColor ? total : 0, points, normals, nullptr, colors, nullptr, pviews, projs, nullptr};
	return read_cloud(ctx, "merge: out of host memory", cloud, s, t0, d2h, stats, out);
}

int b200mvs_estimate_point_colors_device(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets,
	const uint32_t* views, const b200mvs_fuse_view* images, int nImages, uint8_t* colors, void* stream)
{
	return cloud_device(ctx, COLORS, nullptr, points, nPoints, viewOffsets, views, images, nImages, colors, stream,
		[&](const CloudBufs& b, cudaStream_t s) { return colors_device(ctx, b, images, nImages, s); });
}

int b200mvs_estimate_point_colors(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets,
	const uint32_t* views, const b200mvs_fuse_view* images, int nImages, uint8_t* colors, b200mvs_stats* stats)
{
	return cloud_host(ctx, COLORS, nullptr, points, nPoints, viewOffsets, views, images, nImages, colors, stats,
		[&](const CloudBufs& b, cudaStream_t s) { return colors_device(ctx, b, images, nImages, s); });
}

int b200mvs_estimate_point_normals_device(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets,
	const uint32_t* views, const b200mvs_fuse_view* images, int nImages, int numNeighbors, float* normals, void* stream)
{
	return cloud_device(ctx, NORMALS, normals_refused(numNeighbors), points, nPoints, viewOffsets, views, images, nImages,
		normals, stream,
		[&](const CloudBufs& b, cudaStream_t s) { return normals_device(ctx, b, images, nImages, numNeighbors, s); });
}

int b200mvs_estimate_point_normals(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets,
	const uint32_t* views, const b200mvs_fuse_view* images, int nImages, int numNeighbors, float* normals, b200mvs_stats* stats)
{
	return cloud_host(ctx, NORMALS, normals_refused(numNeighbors), points, nPoints, viewOffsets, views, images, nImages,
		normals, stats,
		[&](const CloudBufs& b, cudaStream_t s) { return normals_device(ctx, b, images, nImages, numNeighbors, s); });
}

int b200mvs_point_cloud_visibility_device(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets,
	const uint32_t* views, const b200mvs_fuse_view* images, int nImages, int32_t* visibility, void* stream)
{
	return cloud_device(ctx, VISIBILITY, nullptr, points, nPoints, viewOffsets, views, images, nImages, visibility, stream,
		[&](const CloudBufs& b, cudaStream_t s) { return visibility_device(ctx, b, images, nImages, s); });
}

int b200mvs_point_cloud_visibility(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, const uint32_t* viewOffsets,
	const uint32_t* views, const b200mvs_fuse_view* images, int nImages, int32_t* visibility, b200mvs_stats* stats)
{
	return cloud_host(ctx, VISIBILITY, nullptr, points, nPoints, viewOffsets, views, images, nImages, visibility, stats,
		[&](const CloudBufs& b, cudaStream_t s) { return visibility_device(ctx, b, images, nImages, s); });
}

int b200mvs_pointcloud_remove_order(const uint8_t* remove, uint64_t n, uint32_t* order, uint64_t* nKept) {
	if (!nKept || n > 0xFFFFFFFFull || (n && (!remove || !order))) return B200MVS_ERR_ARG;
	// RFOREACH(i, points) if (remove[i]) RemovePoint(i): slot i still holds point i when the loop reaches it, and RemoveAt moves
	// the last point into it
	uint64_t size = n;
	for (uint64_t i = 0; i < n; ++i) order[i] = (uint32_t)i;
	for (uint64_t i = n; i-- > 0; )
		if (remove[i]) order[i] = order[--size];
	*nKept = size;
	return B200MVS_OK;
}

int b200mvs_point_knn_device(b200mvs_ctx* ctx, const float* points, uint64_t nPoints, int numNeighbors, uint32_t* indices, void* stream) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (nPoints > 0x7FFFFFFFull) return fail(ctx, B200MVS_ERR_ARG, "k-NN: more than 2^31 - 1 points");
	if (numNeighbors < 1 || numNeighbors > B200MVS_MAX_POINT_NEIGHBORS) return fail(ctx, B200MVS_ERR_ARG, "k-NN: numNeighbors out of [1, 32]");
	if (nPoints == 0) return B200MVS_OK;
	if (!points || !indices) return fail(ctx, B200MVS_ERR_ARG, "k-NN: null pointer");
	CK(cudaSetDevice(ctx->device));
	if (!on_device(ctx, points) || !on_device(ctx, indices))
		return fail(ctx, B200MVS_ERR_ARG, "k-NN: a buffer is not in device memory of the context's device");
	ctx->launches = 0;
	cudaStream_t s = stream_of(ctx, stream);
	Carve scratch(ctx->pcScratch);
	if (int rc = grid_knn(ctx, scratch, points, (uint32_t)nPoints, nullptr, nullptr, 0, (int)std::min<uint64_t>(numNeighbors, nPoints),
		indices, s)) return rc;
	CK(cudaStreamSynchronize(s));
	return B200MVS_OK;
}

} // extern "C"
