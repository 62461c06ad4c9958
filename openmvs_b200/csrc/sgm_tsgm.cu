// sgm_tsgm.cu — the level loop of the hierarchical (tSGM) pair matcher, on the device.
//
// SemiGlobalMatcher::Match(scene, ...) (libs/MVS/SemiGlobalMatcher.cpp:583-718) wraps the pair matcher in a coarse-to-fine loop.
// Between two matches it runs small sequential routines on the CPU; these are their device forms:
//   tsgm_range_kernel / tsgm_expand_kernel   Disparity2RangeMap: per-pixel ranges at twice the scale   :1350-1444
//   tsgm_flip_*                              FlipDirection: left->right map to right->left map          :1630-1657
//   tsgm_upscale_mask_kernel                 UpscaleMask                                               :1662-1690
//   tsgm_extract_mask_kernel                 ExtractMask: invalid border runs of each row              :1518-1576
//   tsgm_speckle_*                           cv::filterSpeckles (OpenCV): small 4-connected regions of similar disparity
//   tsgm_area_u8_kernel                      cv::resize(INTER_AREA) of the 8-bit colour pyramid (ViewData::GetImage,
//                                            SemiGlobalMatcher.h:127-142) at an integer factor
// All integer work on a few MB; one thread per pixel (per row for ExtractMask).  Every result is bit-exact to the sequential code.
#include "sgm_common.cuh"
#include "label_common.cuh"
#include <cub/device/device_scan.cuh>

namespace {

inline dim3 grid2(int w, int h, dim3 b) { return dim3((w+b.x-1)/b.x, (h+b.y-1)/b.y); }

// k-th smallest (0-based) valid value of the window [r-hw, r+hw] x [c-hw, c+hw] clipped to the map, by bisection over the value
// range [lo, hi]: the same integer as the nth_element of cList::GetMedian (libs/Common/List.h:668-678) without a per-thread list
__device__ int window_kth(const int16_t* __restrict__ D, int W, int H, int r, int c, int hw, int k, int lo, int hi) {
	const int i0 = max(r-hw, 0), i1 = min(r+hw, H-1), j0 = max(c-hw, 0), j1 = min(c+hw, W-1);
	while (lo < hi) {
		const int mid = lo+((hi-lo)>>1);
		int cnt = 0;
		for (int i = i0; i <= i1; ++i)
			for (int j = j0; j <= j1; ++j) {
				const int d = D[(size_t)i*W+j];
				cnt += (d != SGM_NO_DISP && d <= mid) ? 1 : 0;
			}
		if (cnt > k) hi = mid; else lo = mid+1;
	}
	return lo;
}

// Disparity2RangeMap, part 1: the range of every pixel of the (coarse) disparity map, read with the mask of the 2x grid at
// (2r+3, 2c+3).  Disparity arithmetic in int16 like the reference's Disparity type.
__global__ void tsgm_range_kernel(const int16_t* __restrict__ D, int W, int H, const uint8_t* __restrict__ mask, int mw,
	int minNumDisp, int minNumDispInvalid, short2* __restrict__ ranges)
{
	const int c = blockIdx.x*blockDim.x+threadIdx.x, r = blockIdx.y*blockDim.y+threadIdx.y;
	if (c >= W || r >= H) return;
	short lo = SGM_NO_DISP, hi = SGM_NO_DISP;
	if (mask[(size_t)(2*r+3)*mw + 2*c+3] != 0) {
		const bool bInvalid = D[(size_t)r*W+c] == SGM_NO_DISP;
		const int hw = bInvalid ? 20 : 3;
		int n = 0, mn = 0x7FFFFFFF, mx = -0x7FFFFFFF;
		for (int i = max(r-hw, 0); i <= min(r+hw, H-1); ++i)
			for (int j = max(c-hw, 0); j <= min(c+hw, W-1); ++j) {
				const int d = D[(size_t)i*W+j];
				if (d != SGM_NO_DISP) { ++n; mn = min(mn, d); mx = max(mx, d); }
			}
		if (n < 3) {
			hi = (short)min((int)(short)(W*2/3), minNumDispInvalid);
			lo = (short)-hi;
		} else {
			short med;
			if (n & 1) med = (short)window_kth(D, W, H, r, c, hw, n>>1, mn, mx);
			else med = (short)((window_kth(D, W, H, r, c, hw, (n>>1)-1, mn, mx) + window_kth(D, W, H, r, c, hw, n>>1, mn, mx))/2);
			const short disp = (short)(med*2);
			short numDisp = (short)((mx-mn)*2);
			if (numDisp < minNumDisp) {
				numDisp = (short)minNumDisp;
				lo = (short)(disp-numDisp/2);
				hi = (short)(disp+(numDisp+1)/2);
			} else {
				const short maxNumDisp = bInvalid ? 64 : 32;
				if (numDisp > maxNumDisp) {
					lo = (short)(disp-(maxNumDisp*(disp-mn*2)+1)/numDisp);
					hi = (short)(disp+(maxNumDisp*(mx*2+1-disp)+1)/numDisp);
				} else {
					lo = (short)(disp-numDisp/2);
					hi = (short)(disp+(numDisp+1)/2);
				}
			}
		}
	}
	ranges[(size_t)r*W+c] = make_short2(lo, hi);
}

// Disparity2RangeMap, part 2: the 2x grid.  Coarse row 0 covers rows 0..4, row r > 0 rows 2r+3 and 2r+4, the last row every row
// to the end; columns alike (the tail copies the last range).  widths = disparities per pixel, scanned into the idx offsets.
__global__ void tsgm_expand_kernel(const short2* __restrict__ ranges, int W, int H, int W2, int H2, SGMPixel* __restrict__ px,
	unsigned long long* __restrict__ widths)
{
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= W2 || y >= H2) return;
	const int r = y < 5 ? 0 : min((y-3)>>1, H-1), c = x < 5 ? 0 : min((x-3)>>1, W-1);
	const short2 rg = ranges[(size_t)r*W+c];
	const size_t i = (size_t)y*W2+x;
	SGMPixel p; p.idx = 0; p.dmin = rg.x; p.dmax = rg.y; p.pad = 0;
	px[i] = p;
	widths[i] = (unsigned long long)max((int)rg.y-(int)rg.x, 0);
}

__global__ void tsgm_offsets_kernel(SGMPixel* __restrict__ px, const unsigned long long* __restrict__ offs,
	const unsigned long long* __restrict__ widths, size_t n, unsigned long long* __restrict__ total)
{
	const size_t i = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	px[i].idx = offs[i];
	if (i+1 == n) *total = offs[i]+widths[i];
}

// FlipDirection: pixel (r, c) with disparity d writes -d to columns c+d-1 .. c+d+1 of the right map.  The reference loops over c
// in order, so the largest c wins a column: every write is an atomicMax of the key (c+1) << 16 | (uint16)(-d).
__global__ void tsgm_flip_scatter_kernel(const int16_t* __restrict__ l2r, int W, int H, unsigned* __restrict__ keys) {
	const int c = blockIdx.x*blockDim.x+threadIdx.x, r = blockIdx.y*blockDim.y+threadIdx.y;
	if (c >= W || r >= H) return;
	const int d = l2r[(size_t)r*W+c];
	if (d == SGM_NO_DISP) return;
	const unsigned key = ((unsigned)(c+1) << 16) | (unsigned)(uint16_t)(int16_t)(-d);
	for (int x = max(c+d-1, 0), xe = min(c+d+2, W); x < xe; ++x)
		atomicMax(keys+(size_t)r*W+x, key);
}
__global__ void tsgm_flip_resolve_kernel(const unsigned* __restrict__ keys, int16_t* __restrict__ r2l, size_t n) {
	const size_t i = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	const unsigned k = keys[i];
	r2l[i] = k ? (int16_t)(uint16_t)(k & 0xFFFFu) : (int16_t)SGM_NO_DISP;
}

// UpscaleMask: coarse (r, c) owns the 2x2 block at (2r+3, 2c+3); everything else is INVALID
__global__ void tsgm_upscale_mask_kernel(const uint8_t* __restrict__ m, int W, int H, uint8_t* __restrict__ m2, int W2, int H2) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= W2 || y >= H2) return;
	uint8_t v = 0;
	if (x >= 3 && y >= 3) {
		const int r = (y-3)>>1, c = (x-3)>>1;
		if (r < H && c < W) v = m[(size_t)r*W+c];
	}
	m2[(size_t)y*W2+x] = v;
}

// ExtractMask: each row is walked from the left and from the right, invalidating mask pixels until thValid valid disparities
// were passed (the pixel that reaches the count is invalidated too); already invalid mask pixels are skipped
__global__ void tsgm_extract_mask_kernel(const int16_t* __restrict__ D, uint8_t* __restrict__ M, int W, int H, int thValid) {
	const int r = blockIdx.x*blockDim.x+threadIdx.x;
	if (r >= H) return;
	const int16_t* d = D+(size_t)r*W;
	uint8_t* m = M+(size_t)r*W;
	int numValid = 0;
	for (int c = 0; c < W; ++c) {
		if (m[c] == 0) continue;
		m[c] = 0;
		if (d[c] == SGM_NO_DISP) continue;
		if (++numValid >= thValid) break;
	}
	numValid = 0;
	for (int c = W; --c >= 0; ) {
		if (m[c] == 0) continue;
		m[c] = 0;
		if (d[c] == SGM_NO_DISP) continue;
		if (++numValid >= thValid) break;
	}
}

// cv::filterSpeckles(img, newVal, maxSpeckleSize, maxDiff) on int16: the regions are the connected components of the pixels
// != newVal under the symmetric 4-neighbour relation |d1 - d2| <= maxDiff, so any labelling gives OpenCV's regions: the
// components of label_common.cuh, then the removal of the regions of at most maxSpeckleSize pixels.
struct SpeckleEdge {
	const int16_t* D; int newVal, maxDiff;
	__device__ int at(int i) const { return __ldg(D+i); }
	__device__ bool valid(int a) const { return a != newVal; }
	__device__ bool edge(int a, int b) const { return b != newVal && abs(a-b) <= maxDiff; }
};
__global__ void tsgm_speckle_remove_kernel(int16_t* __restrict__ D, const int* __restrict__ L, const int* __restrict__ size, int n,
	int newVal, int maxSpeckleSize)
{
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	const int r = L[i];
	if (r >= 0 && size[r] <= maxSpeckleSize) D[i] = (int16_t)newVal;
}

// cv::resize(src, dst, Size(), 1/k, 1/k, INTER_AREA) of an 8-bit image with 1, 3 or 4 channels (OpenCV's resizeAreaFast): a full
// k x k cell is (sum + 2) >> 2 for k = 2 and round-half-even(sum * (1/k^2)) otherwise; a cell cut by the right or bottom border is
// round-half-even(sum / count) over its pixels inside the image
__global__ void tsgm_area_u8_kernel(const uint8_t* __restrict__ src, int sw, int sh, int cn, uint8_t* __restrict__ dst, int dw, int dh, int k) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= dw || y >= dh) return;
	const int sx0 = x*k, sy0 = y*k;
	const int nx = min(k, sw-sx0), ny = min(k, sh-sy0);
	const bool full = nx == k && ny == k;
	const float scale = 1.f/(float)(k*k);
	for (int ch = 0; ch < cn; ++ch) {
		int s = 0;
		for (int j = 0; j < ny; ++j)
			for (int i = 0; i < nx; ++i) s += src[((size_t)(sy0+j)*sw + sx0+i)*cn + ch];
		int v;
		if (full) v = k == 2 ? (s+2)>>2 : __float2int_rn(__fmul_rn((float)s, scale));
		else v = __float2int_rn(__fdiv_rn((float)s, (float)(nx*ny)));
		dst[((size_t)y*dw+x)*cn+ch] = (uint8_t)min(max(v, 0), 255);
	}
}

__global__ void tsgm_fill_kernel(int16_t* __restrict__ d, size_t n, int16_t v) {
	const size_t i = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (i < n) d[i] = v;
}

__global__ void tsgm_minmax_init_kernel(int* out) { out[0] = 0x7FFFFFFF; out[1] = -0x7FFFFFFF-1; }
// out[0] = min, out[1] = max of the values != SGM_NO_DISP (initialised to INT_MAX / INT_MIN by tsgm_minmax_init_kernel)
__global__ void tsgm_minmax_kernel(const int16_t* __restrict__ d, size_t n, int* out) {
	int lo = 0x7FFFFFFF, hi = -0x7FFFFFFF-1;
	for (size_t i = (size_t)blockIdx.x*blockDim.x+threadIdx.x; i < n; i += (size_t)gridDim.x*blockDim.x) {
		const int v = d[i];
		if (v != SGM_NO_DISP) { lo = min(lo, v); hi = max(hi, v); }
	}
	lo = __reduce_min_sync(0xFFFFFFFFu, lo); hi = __reduce_max_sync(0xFFFFFFFFu, hi);
	if ((threadIdx.x&31) == 0) { atomicMin(out, lo); atomicMax(out+1, hi); }
}

// one range [lo, hi) for every pixel of a dense volume (the fixed-range branch)
__global__ void tsgm_dense_map_kernel(SGMPixel* __restrict__ px, size_t n, int lo, int hi) {
	const size_t i = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	SGMPixel p; p.idx = (unsigned long long)i*(unsigned long long)(hi-lo); p.dmin = (short)lo; p.dmax = (short)hi; p.pad = 0;
	px[i] = p;
}

} // namespace

// scratch bytes tsgm_launch_range_map needs for a 2x grid of n pixels (widths, offsets, scan temporaries, total)
size_t tsgm_range_map_scratch(size_t n) {
	size_t tmp = 0;
	cub::DeviceScan::ExclusiveSum(nullptr, tmp, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n);
	return 2*n*sizeof(unsigned long long) + ((tmp+255)&~(size_t)255) + 256;
}
// Disparity2RangeMap into px (W2 x H2 records); *total (device) receives numCosts.  scratch: tsgm_range_map_scratch(W2*H2) bytes,
// 256-byte aligned; ranges: W x H short2
cudaError_t tsgm_launch_range_map(const int16_t* D, int W, int H, const uint8_t* mask, int W2, int H2, int minNumDisp, int minNumDispInvalid,
	short2* ranges, SGMPixel* px, void* scratch, unsigned long long* total, cudaStream_t s)
{
	const size_t n = (size_t)W2*H2;
	unsigned long long* widths = (unsigned long long*)scratch;
	unsigned long long* offs = widths+n;
	void* tmp = (void*)(((uintptr_t)(offs+n)+255)&~(uintptr_t)255);
	size_t tmpBytes = 0;
	cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, tmpBytes, widths, offs, (int)n, s);
	if (e != cudaSuccess) return e;
	const dim3 b(32, 8);
	tsgm_range_kernel<<<grid2(W, H, b), b, 0, s>>>(D, W, H, mask, W2, minNumDisp, minNumDispInvalid, ranges);
	tsgm_expand_kernel<<<grid2(W2, H2, b), b, 0, s>>>(ranges, W, H, W2, H2, px, widths);
	if ((e = cub::DeviceScan::ExclusiveSum(tmp, tmpBytes, widths, offs, (int)n, s)) != cudaSuccess) return e;
	tsgm_offsets_kernel<<<(unsigned)((n+255)/256), 256, 0, s>>>(px, offs, widths, n, total);
	return cudaGetLastError();
}
// keys: W x H unsigned scratch
cudaError_t tsgm_launch_flip(const int16_t* l2r, int16_t* r2l, int W, int H, unsigned* keys, cudaStream_t s) {
	const size_t n = (size_t)W*H;
	cudaError_t e = cudaMemsetAsync(keys, 0, n*sizeof(unsigned), s);
	if (e != cudaSuccess) return e;
	const dim3 b(32, 8);
	tsgm_flip_scatter_kernel<<<grid2(W, H, b), b, 0, s>>>(l2r, W, H, keys);
	tsgm_flip_resolve_kernel<<<(unsigned)((n+255)/256), 256, 0, s>>>(keys, r2l, n);
	return cudaGetLastError();
}
cudaError_t tsgm_launch_upscale_mask(const uint8_t* m, int W, int H, uint8_t* m2, int W2, int H2, cudaStream_t s) {
	const dim3 b(32, 8);
	tsgm_upscale_mask_kernel<<<grid2(W2, H2, b), b, 0, s>>>(m, W, H, m2, W2, H2);
	return cudaGetLastError();
}
cudaError_t tsgm_launch_extract_mask(const int16_t* D, uint8_t* M, int W, int H, int thValid, cudaStream_t s) {
	tsgm_extract_mask_kernel<<<(H+63)/64, 64, 0, s>>>(D, M, W, H, thValid);
	return cudaGetLastError();
}
// labels / sizes: W x H int scratch each
cudaError_t tsgm_launch_speckles(int16_t* D, int W, int H, int newVal, int maxSpeckleSize, int maxDiff, int* labels, int* sizes, cudaStream_t s) {
	const int n = W*H;
	label_launch(SpeckleEdge{D, newVal, maxDiff}, W, H, labels, sizes, nullptr, s);
	tsgm_speckle_remove_kernel<<<(n+255)/256, 256, 0, s>>>(D, labels, sizes, n, newVal, maxSpeckleSize);
	return cudaGetLastError();
}
cudaError_t tsgm_launch_area_u8(const uint8_t* src, int sw, int sh, int cn, uint8_t* dst, int dw, int dh, int k, cudaStream_t s) {
	const dim3 b(32, 8);
	tsgm_area_u8_kernel<<<grid2(dw, dh, b), b, 0, s>>>(src, sw, sh, cn, dst, dw, dh, k);
	return cudaGetLastError();
}
cudaError_t tsgm_launch_fill(int16_t* d, size_t n, int16_t v, cudaStream_t s) {
	tsgm_fill_kernel<<<(unsigned)((n+255)/256), 256, 0, s>>>(d, n, v);
	return cudaGetLastError();
}
// out2: two device ints, min / max of the valid values (INT_MAX / INT_MIN when there is none)
cudaError_t tsgm_launch_minmax(const int16_t* d, size_t n, int* out2, cudaStream_t s) {
	tsgm_minmax_init_kernel<<<1, 1, 0, s>>>(out2);
	const size_t blocks = (n+255)/256;
	tsgm_minmax_kernel<<<(unsigned)(blocks < 1024 ? blocks : 1024), 256, 0, s>>>(d, n, out2);
	return cudaGetLastError();
}
cudaError_t tsgm_launch_dense_map(SGMPixel* px, size_t n, int lo, int hi, cudaStream_t s) {
	tsgm_dense_map_kernel<<<(unsigned)((n+255)/256), 256, 0, s>>>(px, n, lo, hi);
	return cudaGetLastError();
}
