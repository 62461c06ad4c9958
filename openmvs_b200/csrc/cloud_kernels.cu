// cloud_kernels.cu — the point-cloud tail of the densification on the device (host driver: cloud_host.cu): MergeDepthMaps,
// EstimatePointColors, the exact k-nearest-neighbour search and PCA of EstimatePointNormals (DESIGN.md §5.6), and the visibility
// counts of PointCloudFilter (§5.7).
#include <cfloat>
#include <cub/cub.cuh>
#include "cloud_common.cuh"

namespace {

constexpr int TPB = 256;

inline unsigned blocks(size_t n) { return (unsigned)std::max<size_t>((n+TPB-1)/TPB, 1); }

// ---- MergeDepthMaps ----

// every depth != 0 becomes a point (SceneDensify.cpp:1337-1340): the flag of each pixel and the image's count, one atomic per warp
__global__ void k_merge_flags(const float* __restrict__ depth, size_t n, uint8_t* __restrict__ flags, unsigned long long* count) {
	const size_t i = blockIdx.x*(size_t)blockDim.x + threadIdx.x;
	const bool nz = i < n && depth[i] != 0;
	if (i < n) flags[i] = nz;
	const unsigned m = __ballot_sync(0xFFFFFFFFu, nz);
	if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, (unsigned long long)__popc(m));
}

// the first point of every image (images in index order) and the total
__global__ void k_merge_bases(const unsigned long long* counts, int nImages, unsigned long long* bases, unsigned long long* total) {
	unsigned long long sum = 0;
	for (int i = 0; i < nImages; ++i) { bases[i] = sum; sum += counts[i]; }
	*total = sum;
}

// one thread per selected pixel, in raster order: the point, its projection and, when asked for, its colour and world normal
__global__ void k_merge_assemble(const MergeImage I, const uint32_t* __restrict__ idx, const uint32_t* nSel,
	const unsigned long long* base, float* __restrict__ points, uint16_t* __restrict__ projs, uint32_t* __restrict__ views,
	uint8_t* __restrict__ colors, float* __restrict__ normals)
{
	const uint32_t t = blockIdx.x*blockDim.x + threadIdx.x;
	if (t >= *nSel) return;
	const uint32_t ia = idx[t];
	const int x = (int)(ia % (uint32_t)I.w), y = (int)(ia / (uint32_t)I.w);
	const size_t j = (size_t)*base + t;
	double X[3];
	fuse::image_to_world(I.cam, x, y, I.depth[ia], X);
	for (int c = 0; c < 3; ++c) points[3*j+c] = (float)X[c];
	projs[2*j] = (uint16_t)x; projs[2*j+1] = (uint16_t)y;
	views[j] = I.id;
	if (colors) for (int c = 0; c < 3; ++c) colors[3*j+c] = I.color[3*(size_t)ia+c];
	if (normals) fuse::normal_to_world(I.cam, I.normal+3*(size_t)ia, normals+3*j);
}

// ---- checks of a cloud ----

// Offsets start at 0 and every range lies in [0, offsets[n]] (a thread reads views only then, so a bad table is never followed
// outside the views array); every view ID is below nImages; with needView, no point has an empty list.
__global__ void k_check_views(const uint32_t* __restrict__ off, const uint32_t* __restrict__ views, uint32_t n, int nImages,
	bool needView, int* bad)
{
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t a = off[i], b = off[i+1], end = off[n];
	int why = 0;
	if ((i == 0 && a != 0) || a > b || b > end) why = CLOUD_BAD_OFFSETS;
	else {
		if (needView && a == b) why |= CLOUD_NO_VIEW;
		for (uint32_t j = a; j < b; ++j)
			if (views[j] >= (uint32_t)nImages) { why |= CLOUD_BAD_VIEW; break; }
	}
	if (why) atomicOr(bad, why);
}

// the bounding box of the points and whether every coordinate is finite: per-thread extrema, a warp reduction, one atomic per warp
__global__ void k_bbox(const float* __restrict__ pts, uint32_t n, unsigned* box, int* bad) {
	unsigned lo[3] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu}, hi[3] = {0u, 0u, 0u};
	bool finite = true;
	for (uint32_t i = blockIdx.x*blockDim.x + threadIdx.x; i < n; i += gridDim.x*blockDim.x)
		for (int c = 0; c < 3; ++c) {
			const float v = pts[3*(size_t)i+c];
			finite &= isfinite(v);
			const unsigned k = box_key(v);
			lo[c] = min(lo[c], k); hi[c] = max(hi[c], k);
		}
	for (int c = 0; c < 3; ++c) { lo[c] = __reduce_min_sync(0xFFFFFFFFu, lo[c]); hi[c] = __reduce_max_sync(0xFFFFFFFFu, hi[c]); }
	const bool all = __all_sync(0xFFFFFFFFu, finite);
	if ((threadIdx.x & 31) == 0) {
		for (int c = 0; c < 3; ++c) { atomicMin(box+c, lo[c]); atomicMax(box+3+c, hi[c]); }
		if (!all) atomicOr(bad, CLOUD_NOT_FINITE);
	}
}

// m points at i*n/m (i < m <= n), the sample the grid's extent is estimated from
__global__ void k_sample(const float* __restrict__ pts, uint32_t n, int m, float* __restrict__ out) {
	const int i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= m) return;
	const size_t j = (size_t)i*n/(uint32_t)m;
	for (int c = 0; c < 3; ++c) out[3*i+c] = pts[3*j+c];
}

// ---- EstimatePointColors (libs/MVS/DepthMap.cpp:1433-1462) ----

// TPixel<uint8_t> * float (libs/Common/Types.h:1965): the product is truncated to uint8
__device__ __forceinline__ uint8_t px_mul(uint8_t p, float v) { return (uint8_t)(unsigned)fuse::mul_f(v, (float)p); }

// TImage<Pixel8U>::sample (libs/Common/Types.inl:2273-2281): products truncated to uint8, sums of uint8 (Types.h:1970)
__device__ __forceinline__ void sample(const CloudImage& I, float px, float py, uint8_t out[3]) {
	const int lx = (int)px, ly = (int)py;
	const float x = fuse::sub_f(px, (float)lx), x1 = fuse::sub_f(1.f, x);
	const float y = fuse::sub_f(py, (float)ly), y1 = fuse::sub_f(1.f, y);
	const uint8_t* r0 = I.color + 3*((size_t)ly*I.w + lx);
	const uint8_t* r1 = r0 + 3*(size_t)I.w;
	for (int c = 0; c < 3; ++c) {
		const uint8_t top = (uint8_t)(px_mul(r0[c], x1) + px_mul(r0[3+c], x));
		const uint8_t bottom = (uint8_t)(px_mul(r1[c], x1) + px_mul(r1[3+c], x));
		out[c] = (uint8_t)(px_mul(top, y1) + px_mul(bottom, y));
	}
}

__global__ void k_colors(const float* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ off, const uint32_t* __restrict__ views,
	const CloudImage* __restrict__ images, uint8_t* __restrict__ colors)
{
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float p[3] = {pts[3*(size_t)i], pts[3*(size_t)i+1], pts[3*(size_t)i+2]};
	// the view closest in depth, the first of equal ones; empty images are skipped
	double best = (double)FLT_MAX;
	int bestView = -1;
	for (uint32_t j = off[i], e = off[i+1]; j < e; ++j) {
		const uint32_t v = views[j];
		if (!images[v].color) continue;
		const double d = fuse::project_row_d(images[v].P+8, p);   // Camera::PointDepth
		if (best > d) { best = d; bestView = (int)v; }
	}
	uint8_t rgb[3] = {255, 255, 255};
	if (bestView >= 0) {
		// Camera::ProjectPointP (libs/MVS/Camera.h:315-320) with INVERT (libs/Common/Types.h:1234, FINV_ZERO for 0), then
		// isInsideWithBorder<float,1> (libs/Common/Types.h:1649-1651)
		const CloudImage& I = images[bestView];
		const float qx = fuse::project_row(I.P, p), qy = fuse::project_row(I.P+4, p), qz = fuse::project_row(I.P+8, p);
		const float inv = qz == 0.f ? 1000000.f : fuse::div_f(1.f, qz);
		const float x = fuse::mul_f(qx, inv), y = fuse::mul_f(qy, inv);
		if (x >= 1.f && y >= 1.f && x <= (float)(I.w-2) && y <= (float)(I.h-2)) sample(I, x, y, rgb);
	}
	for (int c = 0; c < 3; ++c) colors[3*(size_t)i+c] = rgb[c];
}

// ---- EstimatePointNormals: uniform grid, exact k-NN, PCA ----

__device__ __forceinline__ void cell_of(const CloudGrid& g, const double p[3], int c[3]) {
	for (int a = 0; a < 3; ++a) {
		const double f = floor((p[a] - g.lo[a])*g.invH);
		c[a] = f < 0 ? 0 : f >= (double)g.dim[a] ? g.dim[a]-1 : (int)f;
	}
}

__device__ __forceinline__ uint32_t spread10(uint32_t v) {
	v &= 0x3FFu;
	v = (v | (v << 16)) & 0x030000FFu;
	v = (v | (v << 8)) & 0x0300F00Fu;
	v = (v | (v << 4)) & 0x030C30C3u;
	v = (v | (v << 2)) & 0x09249249u;
	return v;
}

__global__ void k_keys(const float* __restrict__ pts, uint32_t n, const CloudGrid g, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx) {
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const double p[3] = {pts[3*(size_t)i], pts[3*(size_t)i+1], pts[3*(size_t)i+2]};
	int c[3];
	cell_of(g, p, c);
	keys[i] = spread10(c[0]) | (spread10(c[1]) << 1) | (spread10(c[2]) << 2);
	idx[i] = i;
}

// the points in key order (x, y, z, original index) and the range of every non-empty cell, indexed linearly
__global__ void k_cells(const float* __restrict__ pts, const uint32_t* __restrict__ keys, const uint32_t* __restrict__ idx, uint32_t n,
	const CloudGrid g, float4* __restrict__ sorted, uint32_t* __restrict__ cellStart, uint32_t* __restrict__ cellEnd)
{
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t o = idx[i];
	const float x = pts[3*(size_t)o], y = pts[3*(size_t)o+1], z = pts[3*(size_t)o+2];
	sorted[i] = make_float4(x, y, z, __uint_as_float(o));
	const double p[3] = {x, y, z};
	int c[3];
	cell_of(g, p, c);
	const size_t lin = ((size_t)c[2]*g.dim[1] + c[1])*g.dim[0] + c[0];
	if (i == 0 || keys[i] != keys[i-1]) cellStart[lin] = i;
	if (i == n-1 || keys[i] != keys[i+1]) cellEnd[lin] = i+1;
}

// (d, i) < (e, j): squared distance first, then the point index
__device__ __forceinline__ bool closer(double d, uint32_t i, double e, uint32_t j) { return d < e || (d == e && i < j); }

// One query per thread, the queries in key order so that a warp's queries are neighbours.  The K best (squared distance, index)
// pairs stay sorted in registers (every index into them is a compile-time constant).  The search visits shells of cells at
// Chebyshev distance r = 0, 1, 2, ... from the query's cell.  An unvisited point lies in a cell beyond the shell along some axis,
// so it is at least as far as the nearest face of the visited block that still has cells behind it (a point clamped into a
// border cell lies beyond that cell, so farther still; a query outside the grid is farther from every face than its cell).  The
// search stops when the k-th best squared distance is at most that distance squared (shrunk by 1e-6 for the rounding of the
// cell coordinates), or when no cell is left.  The cell size only changes how many shells that takes: the result is exact for
// any density.
template <int K>
__global__ void k_knn(const float4* __restrict__ sorted, uint32_t n, const uint32_t* __restrict__ cellStart,
	const uint32_t* __restrict__ cellEnd, const CloudGrid g, int k, uint32_t* __restrict__ out)
{
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 q4 = sorted[i];
	const double q[3] = {q4.x, q4.y, q4.z};
	int c[3];
	cell_of(g, q, c);
	double bd[K]; uint32_t bi[K];
#pragma unroll
	for (int j = 0; j < K; ++j) { bd[j] = INFINITY; bi[j] = 0xFFFFFFFFu; }
	int rMax = 0;
	for (int a = 0; a < 3; ++a) rMax = max(rMax, max(c[a], g.dim[a]-1-c[a]));
	for (int r = 0; r <= rMax; ++r) {
		const int z0 = max(c[2]-r, 0), z1 = min(c[2]+r, g.dim[2]-1), y0 = max(c[1]-r, 0), y1 = min(c[1]+r, g.dim[1]-1);
		for (int z = z0; z <= z1; ++z)
			for (int y = y0; y <= y1; ++y) {
				// the whole row on the shell's faces, its two ends inside
				const bool face = abs(z-c[2]) == r || abs(y-c[1]) == r;
				const int step = face ? 1 : 2*r;
				for (int x = c[0]-r; x <= c[0]+r; x += max(step, 1)) {
					if (x < 0 || x >= g.dim[0]) continue;
					const size_t lin = ((size_t)z*g.dim[1] + y)*g.dim[0] + x;
					for (uint32_t s = cellStart[lin], e = cellEnd[lin]; s < e; ++s) {
						const float4 p = sorted[s];
						const double dx = (double)p.x - q[0], dy = (double)p.y - q[1], dz = (double)p.z - q[2];
						const double d = fuse::add_d(fuse::add_d(fuse::mul_d(dx, dx), fuse::mul_d(dy, dy)), fuse::mul_d(dz, dz));
						const uint32_t id = __float_as_uint(p.w);
						if (!closer(d, id, bd[K-1], bi[K-1])) continue;
						bd[K-1] = d; bi[K-1] = id;
#pragma unroll
						for (int j = K-1; j > 0; --j)
							if (closer(bd[j], bi[j], bd[j-1], bi[j-1])) {
								const double td = bd[j]; bd[j] = bd[j-1]; bd[j-1] = td;
								const uint32_t ti = bi[j]; bi[j] = bi[j-1]; bi[j-1] = ti;
							}
					}
				}
			}
		// bd[k-1] as the least of bd[k-1..K-1] (the list is sorted): no index into the list depends on k
		double kth = INFINITY;
#pragma unroll
		for (int j = 0; j < K; ++j) kth = fmin(kth, j >= k-1 ? bd[j] : INFINITY);
		double bound = INFINITY;
		for (int a = 0; a < 3; ++a) {
			if (c[a]-r-1 >= 0) bound = fmin(bound, q[a] - (g.lo[a] + (double)(c[a]-r)*g.h));
			if (c[a]+r+1 < g.dim[a]) bound = fmin(bound, g.lo[a] + (double)(c[a]+r+1)*g.h - q[a]);
		}
		if (bound == INFINITY) break;   // every cell visited
		bound = fmax(bound, 0.0)*(1.0 - 1e-6);
		if (r > 0 && kth <= bound*bound) break;
	}
	const uint32_t o = __float_as_uint(q4.w);
#pragma unroll
	for (int j = 0; j < K; ++j) if (j < k) out[(size_t)o*k + j] = bi[j];
}

// one cyclic-Jacobi rotation of the symmetric A that zeroes A[p][q], accumulated into the eigenvector columns of V
template <int p, int q>
__device__ __forceinline__ void jacobi_rotate(double (&A)[3][3], double (&V)[3][3]) {
	constexpr int r = 3 - p - q;
	const double apq = A[p][q];
	if (apq == 0.0) return;
	const double theta = (A[q][q] - A[p][p])/(2.0*apq);
	double t = fabs(theta) > 1e150 ? 0.5/fabs(theta) : 1.0/(fabs(theta) + sqrt(theta*theta + 1.0));
	if (theta < 0) t = -t;
	const double cs = 1.0/sqrt(t*t + 1.0), sn = t*cs;
	const double arp = A[r][p], arq = A[r][q];
	A[r][p] = A[p][r] = cs*arp - sn*arq;
	A[r][q] = A[q][r] = sn*arp + cs*arq;
	A[p][p] -= t*apq; A[q][q] += t*apq;
	A[p][q] = A[q][p] = 0.0;
#pragma unroll
	for (int m = 0; m < 3; ++m) {
		const double vp = V[m][p], vq = V[m][q];
		V[m][p] = cs*vp - sn*vq; V[m][q] = sn*vp + cs*vq;
	}
}

// One thread per point: the centroid and scatter matrix of its k neighbours in double, the unit eigenvector of the smallest
// eigenvalue (cyclic Jacobi), cast to float, and turned towards the camera of the point's first view in float
// (libs/MVS/DepthMap.cpp:1511-1515).  A rank-deficient matrix still gives a column of the orthogonal V: finite and of unit length.
__global__ void __launch_bounds__(TPB) k_pca(const float* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ nbr, int k,
	const uint32_t* __restrict__ off, const uint32_t* __restrict__ views, const CloudImage* __restrict__ images, float* __restrict__ normals)
{
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t* nb = nbr + (size_t)i*k;
	double m[3] = {0, 0, 0};
	for (int j = 0; j < k; ++j)
		for (int a = 0; a < 3; ++a) m[a] += (double)pts[3*(size_t)nb[j]+a];
	for (int a = 0; a < 3; ++a) m[a] /= (double)k;
	double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
	for (int j = 0; j < k; ++j) {
		double d[3];
		for (int a = 0; a < 3; ++a) d[a] = (double)pts[3*(size_t)nb[j]+a] - m[a];
#pragma unroll
		for (int a = 0; a < 3; ++a)
#pragma unroll
			for (int b = a; b < 3; ++b) A[a][b] += d[a]*d[b];
	}
	A[1][0] = A[0][1]; A[2][0] = A[0][2]; A[2][1] = A[1][2];
	double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
	for (int sweep = 0; sweep < 16; ++sweep) {
		const double off2 = fabs(A[0][1]) + fabs(A[0][2]) + fabs(A[1][2]);
		if (off2 <= 1e-18*(fabs(A[0][0]) + fabs(A[1][1]) + fabs(A[2][2])) || !(off2 > 0)) break;
		jacobi_rotate<0, 1>(A, V); jacobi_rotate<0, 2>(A, V); jacobi_rotate<1, 2>(A, V);
	}
	int e = 0;
	if (A[1][1] < A[e][e]) e = 1;
	if (A[2][2] < (e ? A[1][1] : A[0][0])) e = 2;
	const double v0 = e == 0 ? V[0][0] : e == 1 ? V[0][1] : V[0][2];
	const double v1 = e == 0 ? V[1][0] : e == 1 ? V[1][1] : V[1][2];
	const double v2 = e == 0 ? V[2][0] : e == 1 ? V[2][1] : V[2][2];
	const double len = sqrt(v0*v0 + v1*v1 + v2*v2);
	float nf[3] = {(float)(v0/len), (float)(v1/len), (float)(v2/len)};
	const float* C = images[views[off[i]]].C;
	const float d[3] = {fuse::sub_f(C[0], pts[3*(size_t)i]), fuse::sub_f(C[1], pts[3*(size_t)i+1]), fuse::sub_f(C[2], pts[3*(size_t)i+2])};
	if (fuse::dot3(nf, d) < 0) for (int a = 0; a < 3; ++a) nf[a] = -nf[a];
	for (int a = 0; a < 3; ++a) normals[3*(size_t)i+a] = nf[a];
}

// ---- PointCloudFilter (libs/MVS/SceneDensify.cpp:2226-2360): the visibility counts ----

// Eigen's sum of three terms (Redux.h, redux_novec_unroller halves the range): a0 + (a1 + a2), as in VECTOR::dot and squaredNorm
__device__ __forceinline__ float sum3(float a0, float a1, float a2) { return fuse::add_f(a0, fuse::add_f(a1, a2)); }

// One cone: Collector::Init (SceneDensify.cpp:2258-2266) for point X and its view list of `weight` entries
struct VisCone {
	float dir[3], distance, maxHeight;
	int weight;
};

__device__ __forceinline__ void vis_cone(const VisView& V, const float* __restrict__ X, int weight, VisCone& c) {
	const float D0 = fuse::sub_f(X[0], V.o[0]), D1 = fuse::sub_f(X[1], V.o[1]), D2 = fuse::sub_f(X[2], V.o[2]);
	c.distance = fuse::sqrt_f(sum3(fuse::mul_f(D0, D0), fuse::mul_f(D1, D1), fuse::mul_f(D2, D2)));
	c.dir[0] = fuse::div_f(D0, c.distance); c.dir[1] = fuse::div_f(D1, c.distance); c.dir[2] = fuse::div_f(D2, c.distance);
	c.maxHeight = fuse::mul_f(c.distance, 1.02f);   // MaxDepthDifference (libs/Common/Util.inl:790)
	c.weight = weight;
}

// Collector::operator() on point P (index idx): TConeIntersect::Classify (libs/Common/Ray.inl:905-920), then IsDepthSimilar with
// 0.01; a VISIBLE point that is not similar gains the size of its own view list beyond X and loses the weight of X before it
__device__ __forceinline__ void vis_count(const VisView& V, const VisCone& c, float px, float py, float pz, uint32_t idx,
	const uint32_t* __restrict__ off, int* __restrict__ vis)
{
	const float D0 = fuse::sub_f(px, V.o[0]), D1 = fuse::sub_f(py, V.o[1]), D2 = fuse::sub_f(pz, V.o[2]);
	const float t = sum3(fuse::mul_f(c.dir[0], D0), fuse::mul_f(c.dir[1], D1), fuse::mul_f(c.dir[2], D2));
	if (fabsf(t) < 0.0001f || t < 0.f || t > c.maxHeight) return;   // PLANAR (ISZERO), BACK, FRONT
	const float tSq = fuse::mul_f(t, t);
	const float dSq = fuse::mul_f(V.cosSq, sum3(fuse::mul_f(D0, D0), fuse::mul_f(D1, D1), fuse::mul_f(D2, D2)));
	if (!(tSq > dSq)) return;                                         // CULLED or PLANAR
	if (fuse::depth_similar(c.distance, t, 0.01f)) return;
	atomicAdd(vis + idx, t > c.distance ? (int)(off[idx+1] - off[idx]) : -c.weight);
}

// The pixel of P in the binning camera of V (a pinhole at the apex o): false when P is behind it or outside the binned rectangle
__device__ __forceinline__ bool vis_pixel(const VisView& V, const float* p, double& u, double& v) {
	const double d0 = (double)p[0] - V.o[0], d1 = (double)p[1] - V.o[1], d2 = (double)p[2] - V.o[2];
	const double x = V.R[0]*d0 + V.R[1]*d1 + V.R[2]*d2, y = V.R[3]*d0 + V.R[4]*d1 + V.R[5]*d2, z = V.R[6]*d0 + V.R[7]*d1 + V.R[8]*d2;
	if (!(z > 0)) return false;
	const double nx = x/z, ny = y/z;
	u = V.fx*nx + V.skew*ny + V.cx; v = V.fy*ny + V.cy;
	return u >= -VIS_MARGIN && u < V.w + VIS_MARGIN && v >= -VIS_MARGIN && v < V.h + VIS_MARGIN;
}

__device__ __forceinline__ int vis_cell(double u) { return (int)floor((u + VIS_MARGIN)*(1.0/VIS_CELL)); }

// The cells a cone's VISIBLE points can lie in: columns [cx0, cx1] of rows [cy0, cy1]; false when the bins cannot answer the cone.
//
// Bound.  Let d be the unit axis in camera space, at angle theta to the optical axis e, and u the unit direction of a VISIBLE point
// P from the apex, at angle phi <= beta to d (beta: the host's bound on phi, cloud_host.cu vis_view).  If theta + beta < 90 deg,
// the normalised image points p(u) = u_xy/u_z and p(d) = d_xy/d_z satisfy
//     |p(u) - p(d)| = |u_xy d_z - d_xy u_z| / (u_z d_z) <= |u x d| / (u_z d_z) <= sin(beta) / (cos(theta) cos(theta + beta))
// because (u_xy d_z - d_xy u_z) is, up to sign and order, the xy part of u x d, |u x d| = sin(phi) <= sin(beta), d_z = cos(theta)
// and u_z = cos(angle(u, e)) >= cos(theta + beta) by the triangle inequality of angles.  (It equals tan(theta + beta) - tan(theta).)
// The pixel offset is K's upper-left 2x2 block times p(u) - p(d): at most (|fx| + |skew|) rho across and |fy| rho down.  One pixel
// more absorbs the double rounding of both projections (relative 1e-16).  A cone with theta + beta near 90 deg, a degenerate
// cone (distance 0 or infinite: then nothing is VISIBLE anyway) or one whose rectangle leaves the binned rectangle is flagged.
__device__ __forceinline__ bool vis_cells(const VisView& V, const VisCone& c, int& cx0, int& cx1, int& cy0, int& cy1) {
	if (!V.binned) return false;
	const double d0 = c.dir[0], d1 = c.dir[1], d2 = c.dir[2], n2 = d0*d0 + d1*d1 + d2*d2;
	if (!(fabs(n2 - 1.0) <= 8.0*FLT_EPSILON)) return false;    // |dir|^2 within 16 u of 1, as the bound on beta assumes
	const double ax = V.R[0]*d0 + V.R[1]*d1 + V.R[2]*d2, ay = V.R[3]*d0 + V.R[4]*d1 + V.R[5]*d2, az = V.R[6]*d0 + V.R[7]*d1 + V.R[8]*d2;
	const double cosT = az/sqrt(n2), sinT = sqrt(fmax(0.0, 1.0 - cosT*cosT));
	const double cosTB = cosT*V.cosB - sinT*V.sinB;             // cos(theta + beta)
	if (!(cosT > 0.1 && cosTB > 0.1)) return false;              // theta + beta beyond 84 deg
	const double rho = V.sinB/(cosT*cosTB);
	const double u = V.fx*(ax/az) + V.skew*(ay/az) + V.cx, v = V.fy*(ay/az) + V.cy;
	const double rx = (fabs(V.fx) + fabs(V.skew))*rho + 1.0, ry = fabs(V.fy)*rho + 1.0;
	if (!(u - rx >= -VIS_MARGIN && u + rx < V.w + VIS_MARGIN && v - ry >= -VIS_MARGIN && v + ry < V.h + VIS_MARGIN)) return false;
	cx0 = max(vis_cell(u - rx), 0); cx1 = min(vis_cell(u + rx), V.ncx - 1);
	cy0 = max(vis_cell(v - ry), 0); cy1 = min(vis_cell(v + ry), V.ncy - 1);
	return true;
}

__global__ void k_vis_entries(const uint32_t* __restrict__ off, uint32_t n, uint32_t* __restrict__ entryPoint) {
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	for (uint32_t j = off[i], e = off[i+1]; j < e; ++j) entryPoint[j] = i;
}

// every thread fills the starts of the keys from its predecessor's (exclusive) to its own (inclusive); the last one the rest
__global__ void k_vis_starts(const uint32_t* __restrict__ keys, uint32_t n, uint32_t nKeys, uint32_t* __restrict__ start) {
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t k = min(keys[i], nKeys);
	for (uint32_t j = i ? min(keys[i-1], nKeys) + 1 : 0; j <= k; ++j) start[j] = i;
	if (i == n-1) for (uint32_t j = k + 1; j <= nKeys; ++j) start[j] = n;
}

__global__ void k_vis_keys(const VisView V, const float* __restrict__ pts, uint32_t n, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx) {
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	double u, v;
	const bool in = vis_pixel(V, pts + 3*(size_t)i, u, v);
	keys[i] = in ? (uint32_t)min(vis_cell(v), V.ncy - 1)*V.ncx + min(vis_cell(u), V.ncx - 1) : V.nCells;
	idx[i] = i;
}

__global__ void k_vis_gather(const float* __restrict__ pts, const uint32_t* __restrict__ idxSorted, uint32_t n, const uint32_t* binned,
	float4* __restrict__ sorted)
{
	const uint32_t i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n || i >= *binned) return;
	const uint32_t o = idxSorted[i];
	sorted[i] = make_float4(pts[3*(size_t)o], pts[3*(size_t)o+1], pts[3*(size_t)o+2], __uint_as_float(o));
}

// One warp per query: the lanes stride over the binned points of each cell row of the cone's rectangle (one contiguous range per
// row, since the keys are row-major), so a warp's loads are coalesced and all its lanes run the same trip count.
__global__ void __launch_bounds__(TPB) k_vis_query(const VisView V, const uint32_t* __restrict__ qPoint, uint32_t nq,
	const float* __restrict__ pts, const uint32_t* __restrict__ off, const float4* __restrict__ sorted,
	const uint32_t* __restrict__ cellStart, int* __restrict__ vis, uint32_t* __restrict__ flagged, uint32_t* nFlagged)
{
	const uint32_t q = (blockIdx.x*blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
	if (q >= nq) return;
	const uint32_t i = qPoint[q];
	VisCone c;
	vis_cone(V, pts + 3*(size_t)i, (int)(off[i+1] - off[i]), c);
	int cx0, cx1, cy0, cy1;
	if (!vis_cells(V, c, cx0, cx1, cy0, cy1)) {
		if (lane == 0) flagged[atomicAdd(nFlagged, 1u)] = i;
		return;
	}
	for (int cy = cy0; cy <= cy1; ++cy) {
		const uint32_t row = (uint32_t)cy*V.ncx;
		for (uint32_t s = cellStart[row + cx0] + lane, e = cellStart[row + cx1 + 1]; s < e; s += 32) {
			const float4 p = sorted[s];
			vis_count(V, c, p.x, p.y, p.z, __float_as_uint(p.w), off, vis);
		}
	}
}

// One block per flagged query (grid-stride over the list): its threads test every point of the cloud
__global__ void __launch_bounds__(TPB) k_vis_exhaustive(const VisView V, const uint32_t* __restrict__ flagged, const uint32_t* nFlagged,
	const float* __restrict__ pts, uint32_t n, const uint32_t* __restrict__ off, int* __restrict__ vis)
{
	for (uint32_t f = blockIdx.x; f < *nFlagged; f += gridDim.x) {
		const uint32_t i = flagged[f];
		VisCone c;
		vis_cone(V, pts + 3*(size_t)i, (int)(off[i+1] - off[i]), c);
		for (uint32_t j = threadIdx.x; j < n; j += blockDim.x)
			vis_count(V, c, pts[3*(size_t)j], pts[3*(size_t)j+1], pts[3*(size_t)j+2], j, off, vis);
	}
}

} // namespace

cudaError_t cloud_launch_merge_flags(const float* depth, size_t n, uint8_t* flags, unsigned long long* count, cudaStream_t s) {
	k_merge_flags<<<blocks(n), TPB, 0, s>>>(depth, n, flags, count);
	return cudaGetLastError();
}

cudaError_t cloud_launch_merge_bases(const unsigned long long* counts, int nImages, unsigned long long* bases, unsigned long long* total,
	cudaStream_t s)
{
	k_merge_bases<<<1, 1, 0, s>>>(counts, nImages, bases, total);
	return cudaGetLastError();
}

cudaError_t cloud_launch_merge_assemble(const MergeImage& I, const uint32_t* idx, const uint32_t* nSel, size_t maxSel,
	const unsigned long long* base, float* points, uint16_t* projs, uint32_t* views, uint8_t* colors, float* normals, cudaStream_t s)
{
	k_merge_assemble<<<blocks(maxSel), TPB, 0, s>>>(I, idx, nSel, base, points, projs, views, colors, normals);
	return cudaGetLastError();
}

cudaError_t cloud_launch_check_views(const uint32_t* offsets, const uint32_t* views, uint32_t n, int nImages, bool needView, int* bad,
	cudaStream_t s)
{
	k_check_views<<<blocks(n), TPB, 0, s>>>(offsets, views, n, nImages, needView, bad);
	return cudaGetLastError();
}

cudaError_t cloud_launch_bbox(const float* points, uint32_t n, unsigned* box, int* bad, cudaStream_t s) {
	k_bbox<<<std::min(blocks(n), 1024u), TPB, 0, s>>>(points, n, box, bad);
	return cudaGetLastError();
}

cudaError_t cloud_launch_sample(const float* points, uint32_t n, int m, float* out, cudaStream_t s) {
	k_sample<<<blocks(m), TPB, 0, s>>>(points, n, m, out);
	return cudaGetLastError();
}

cudaError_t cloud_launch_colors(const float* points, uint32_t n, const uint32_t* offsets, const uint32_t* views, const CloudImage* images,
	uint8_t* colors, cudaStream_t s)
{
	k_colors<<<blocks(n), TPB, 0, s>>>(points, n, offsets, views, images, colors);
	return cudaGetLastError();
}

cudaError_t cloud_launch_keys(const float* points, uint32_t n, const CloudGrid& g, uint32_t* keys, uint32_t* idx, cudaStream_t s) {
	k_keys<<<blocks(n), TPB, 0, s>>>(points, n, g, keys, idx);
	return cudaGetLastError();
}

cudaError_t cloud_launch_cells(const float* points, const uint32_t* keys, const uint32_t* idx, uint32_t n, const CloudGrid& g,
	float4* sorted, uint32_t* cellStart, uint32_t* cellEnd, cudaStream_t s)
{
	k_cells<<<blocks(n), TPB, 0, s>>>(points, keys, idx, n, g, sorted, cellStart, cellEnd);
	return cudaGetLastError();
}

cudaError_t cloud_launch_knn(const float4* sorted, uint32_t n, const uint32_t* cellStart, const uint32_t* cellEnd, const CloudGrid& g,
	int k, uint32_t* indices, cudaStream_t s)
{
	// the smallest register list that holds k
	if (k <= 8) k_knn<8><<<blocks(n), TPB, 0, s>>>(sorted, n, cellStart, cellEnd, g, k, indices);
	else if (k <= 16) k_knn<16><<<blocks(n), TPB, 0, s>>>(sorted, n, cellStart, cellEnd, g, k, indices);
	else k_knn<32><<<blocks(n), TPB, 0, s>>>(sorted, n, cellStart, cellEnd, g, k, indices);
	return cudaGetLastError();
}

cudaError_t cloud_launch_pca(const float* points, uint32_t n, const uint32_t* indices, int k, const uint32_t* offsets,
	const uint32_t* views, const CloudImage* images, float* normals, cudaStream_t s)
{
	k_pca<<<blocks(n), TPB, 0, s>>>(points, n, indices, k, offsets, views, images, normals);
	return cudaGetLastError();
}

cudaError_t cloud_launch_vis_entries(const uint32_t* offsets, uint32_t n, uint32_t* entryPoint, cudaStream_t s) {
	k_vis_entries<<<blocks(n), TPB, 0, s>>>(offsets, n, entryPoint);
	return cudaGetLastError();
}

cudaError_t cloud_launch_vis_starts(const uint32_t* keys, uint32_t n, uint32_t nKeys, uint32_t* start, cudaStream_t s) {
	k_vis_starts<<<blocks(n), TPB, 0, s>>>(keys, n, nKeys, start);
	return cudaGetLastError();
}

cudaError_t cloud_launch_vis_keys(const VisView& V, const float* points, uint32_t n, uint32_t* keys, uint32_t* idx, cudaStream_t s) {
	k_vis_keys<<<blocks(n), TPB, 0, s>>>(V, points, n, keys, idx);
	return cudaGetLastError();
}

cudaError_t cloud_launch_vis_gather(const float* points, const uint32_t* idxSorted, uint32_t n, const uint32_t* binnedCount, float4* sorted,
	cudaStream_t s)
{
	k_vis_gather<<<blocks(n), TPB, 0, s>>>(points, idxSorted, n, binnedCount, sorted);
	return cudaGetLastError();
}

cudaError_t cloud_launch_vis_query(const VisView& V, const uint32_t* qPoint, uint32_t nq, const float* points, const uint32_t* offsets,
	const float4* sorted, const uint32_t* cellStart, int* visibility, uint32_t* flagged, uint32_t* nFlagged, cudaStream_t s)
{
	k_vis_query<<<blocks(32*(size_t)nq), TPB, 0, s>>>(V, qPoint, nq, points, offsets, sorted, cellStart, visibility, flagged, nFlagged);
	return cudaGetLastError();
}

cudaError_t cloud_launch_vis_exhaustive(const VisView& V, const uint32_t* flagged, const uint32_t* nFlagged, uint32_t maxFlagged,
	const float* points, uint32_t n, const uint32_t* offsets, int* visibility, cudaStream_t s)
{
	// the count stays on the device: enough blocks for every SM, each taking flagged queries in turn
	k_vis_exhaustive<<<std::max(std::min(maxFlagged, 4096u), 1u), TPB, 0, s>>>(V, flagged, nFlagged, points, n, offsets, visibility);
	return cudaGetLastError();
}
