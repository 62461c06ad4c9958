// cloud_kernels.cu — the point-cloud tail of the densification on the device (host driver: cloud_host.cu): MergeDepthMaps,
// EstimatePointColors, and the exact k-nearest-neighbour search and PCA of EstimatePointNormals (DESIGN.md §5.6).
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
