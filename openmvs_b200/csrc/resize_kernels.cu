// resize_kernels.cu — the image-pyramid arithmetic of the scale loop, on device.
//
// The reference calls OpenCV for these (third-party arithmetic, see DESIGN.md):
//   cv::resize(..., INTER_AREA)    images / known depth-maps   libs/MVS/SceneDensify.cpp:586,590
//   cv::resize(..., INTER_LINEAR)  low-res depth  -> next level libs/MVS/SceneDensify.cpp:661
//   cv::resize(..., INTER_NEAREST) low-res normal -> next level libs/MVS/SceneDensify.cpp:662
// One thread per destination pixel; HBM-bound, a few MB per level.
#include "resize_common.cuh"

namespace {

// area taps of one destination index: at most a leading partial cell, full cells, trailing partial cell
struct AreaSpan { int s0, s1; float a0, a, a1; bool lead, trail; };

__device__ __forceinline__ AreaSpan area_span(int d, int ssize, double scale) {
	AreaSpan t;
	const double fsx1 = d*scale, fsx2 = fsx1+scale;
	const double cell = fmin(scale, ssize-fsx1);
	int sx1 = (int)ceil(fsx1), sx2 = (int)floor(fsx2);
	sx2 = min(sx2, ssize-1);
	sx1 = min(sx1, sx2);
	t.s0 = sx1; t.s1 = sx2;
	t.lead = (sx1-fsx1) > 1e-3;
	t.a0 = (float)((sx1-fsx1)/cell);
	t.a = (float)(1.0/cell);
	t.trail = (fsx2-sx2) > 1e-3;
	t.a1 = (float)(fmin(fmin(fsx2-sx2, 1.0), cell)/cell);
	return t;
}

__global__ void resize_area_kernel(const float* __restrict__ src, int sw, int sh, int spitch,
	float* __restrict__ dst, int dw, int dh, double scx, double scy, int ix, int iy)
{
	const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
	if (x >= dw || y >= dh) return;
	if (ix > 0) {
		// integer ratio: box mean over the part of the box that lies inside the image
		float s = 0.f; int count = 0;
		for (int j = 0; j < iy && y*iy+j < sh; ++j)
			for (int i = 0; i < ix && x*ix+i < sw; ++i) { s += __ldg(src + (size_t)(y*iy+j)*spitch + x*ix+i); ++count; }
		dst[(size_t)y*dw+x] = count == ix*iy ? s*(1.f/(ix*iy)) : s/count;
		return;
	}
	const AreaSpan tx = area_span(x, sw, scx), ty = area_span(y, sh, scy);
	float sum = 0.f;
	bool first = true;
	for (int r = ty.s0-(ty.lead ? 1 : 0); r <= ty.s1; ++r) {
		float beta;
		if (r < ty.s0) beta = ty.a0;
		else if (r < ty.s1) beta = ty.a;
		else { if (!ty.trail) break; beta = ty.a1; }
		const float* row = src + (size_t)r*spitch;
		float buf = 0.f;
		if (tx.lead) buf += __ldg(row+tx.s0-1)*tx.a0;
		for (int c = tx.s0; c < tx.s1; ++c) buf += __ldg(row+c)*tx.a;
		if (tx.trail) buf += __ldg(row+tx.s1)*tx.a1;
		if (first) { sum = beta*buf; first = false; } else sum += beta*buf;
	}
	dst[(size_t)y*dw+x] = sum;
}

__device__ __forceinline__ void linear_tap(int d, int ssize, double scale, int& s, float& f) {
	f = (float)((d+0.5)*scale-0.5);
	s = (int)floorf(f);
	f -= s;
	if (s < 0) { f = 0.f; s = 0; }
	if (s >= ssize-1) { f = 0.f; s = ssize-1; }
}

__global__ void resize_nearest_kernel(const float* __restrict__ src, int sw, int sh, int ch, float* __restrict__ dst, int dw, int dh, double ifx, double ify) {
	const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
	if (x >= dw || y >= dh) return;
	const int sx = min((int)floor(x*ifx), sw-1), sy = min((int)floor(y*ify), sh-1);
	for (int c = 0; c < ch; ++c)
		dst[((size_t)y*dw+x)*ch+c] = src[((size_t)sy*sw+sx)*ch+c];
}

// next-level initialisation: depth bilinear (INTER_LINEAR), normal nearest, from the packed
// low-resolution plane field; also writes the depth prior of the level
// cv::resize(mask, mask, size, 0, 0, INTER_NEAREST) of the ignore-mask (DepthEstimator::ImportIgnoreMask, DepthMap.cpp:309)
__global__ void resize_nearest_u8_kernel(const uint8_t* __restrict__ src, int sw, int sh, int spitch, uint8_t* __restrict__ dst, int dw, int dh, double ifx, double ify) {
	const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
	if (x >= dw || y >= dh) return;
	const int sx = min((int)floor(x*ifx), sw-1), sy = min((int)floor(y*ify), sh-1);
	dst[(size_t)y*dw+x] = src[(size_t)sy*spitch+sx];
}

// nearestDepth: the depth is up-sampled NEAREST instead of LINEAR (an ignore-mask is set, SceneDensify.cpp:661)
__global__ void plane_up_kernel(const float4* __restrict__ src, int sw, int sh, float4* __restrict__ dst, float* __restrict__ prior,
	int dw, int dh, double scx, double scy, int nearestDepth)
{
	const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
	if (x >= dw || y >= dh) return;
	int x0, y0; float fx, fy;
	linear_tap(x, sw, scx, x0, fx);
	linear_tap(y, sh, scy, y0, fy);
	const int x1 = min(x0+1, sw-1), y1 = min(y0+1, sh-1);
	const float r0 = src[(size_t)y0*sw+x0].w*(1.f-fx) + src[(size_t)y0*sw+x1].w*fx;
	const float r1 = src[(size_t)y1*sw+x0].w*(1.f-fx) + src[(size_t)y1*sw+x1].w*fx;
	const int sx = min((int)floor(x*scx), sw-1), sy = min((int)floor(y*scy), sh-1);
	const float4 n = src[(size_t)sy*sw+sx];
	const float d = nearestDepth ? n.w : r0*(1.f-fy) + r1*fy;
	dst[(size_t)y*dw+x] = make_float4(n.x, n.y, n.z, d);
	prior[(size_t)y*dw+x] = d;
}

// cv::resize(..., INTER_CUBIC) of a float image (ViewData::ScaleImage with scale > 1, DepthMap.h:197-203): OpenCV's bicubic
// kernel (A = -0.75), source coordinate (d + 0.5) * scale - 0.5, taps clamped to the image, horizontal pass then vertical pass,
// all in float like cv::resize's generic float path
__device__ __forceinline__ void cubic_taps(int d, int ssize, double scale, int* idx, float* cf) {
	float f = (float)((d+0.5)*scale-0.5);
	const int s = (int)floorf(f);
	f -= s;
	const float A = -0.75f;
	cf[0] = ((A*(f+1.f) - 5.f*A)*(f+1.f) + 8.f*A)*(f+1.f) - 4.f*A;
	cf[1] = ((A+2.f)*f - (A+3.f))*f*f + 1.f;
	cf[2] = ((A+2.f)*(1.f-f) - (A+3.f))*(1.f-f)*(1.f-f) + 1.f;
	cf[3] = 1.f - cf[0] - cf[1] - cf[2];
	#pragma unroll
	for (int k = 0; k < 4; ++k) idx[k] = min(max(s-1+k, 0), ssize-1);
}
__global__ void resize_cubic_kernel(const float* __restrict__ src, int sw, int sh, int spitch, float* __restrict__ dst, int dw, int dh, int dpitch, double scx, double scy) {
	const int x = blockIdx.x*blockDim.x + threadIdx.x, y = blockIdx.y*blockDim.y + threadIdx.y;
	if (x >= dw || y >= dh) return;
	int ix[4], iy[4]; float cx[4], cy[4];
	cubic_taps(x, sw, scx, ix, cx);
	cubic_taps(y, sh, scy, iy, cy);
	float rows[4];
	#pragma unroll
	for (int k = 0; k < 4; ++k) {
		const float* r = src + (size_t)iy[k]*spitch;
		rows[k] = __ldg(r+ix[0])*cx[0] + __ldg(r+ix[1])*cx[1] + __ldg(r+ix[2])*cx[2] + __ldg(r+ix[3])*cx[3];
	}
	dst[(size_t)y*dpitch+x] = rows[0]*cy[0] + rows[1]*cy[1] + rows[2]*cy[2] + rows[3]*cy[3];
}

inline dim3 grid2(int w, int h, dim3 b) { return dim3((w+b.x-1)/b.x, (h+b.y-1)/b.y); }

} // namespace

// scx/scy: source/destination scale; pass 1/factor for cv::resize(..., Size(), fx, fy) and <= 0 for
// the destination-size form (sw/dw)
cudaError_t rs_launch_area(const float* src, int sw, int sh, int spitch, float* dst, int dw, int dh, double scx, double scy, cudaStream_t s) {
	if (!(scx > 0)) scx = (double)sw/dw;
	if (!(scy > 0)) scy = (double)sh/dh;
	const int ix = (int)(scx+0.5), iy = (int)(scy+0.5);
	const bool integer = (double)ix == scx && (double)iy == scy;
	dim3 b(32, 8);
	resize_area_kernel<<<grid2(dw, dh, b), b, 0, s>>>(src, sw, sh, spitch, dst, dw, dh, scx, scy, integer ? ix : 0, integer ? iy : 0);
	return cudaGetLastError();
}
cudaError_t rs_launch_cubic(const float* src, int sw, int sh, int spitch, float* dst, int dw, int dh, int dpitch, double scx, double scy, cudaStream_t s) {
	dim3 b(32, 8);
	resize_cubic_kernel<<<grid2(dw, dh, b), b, 0, s>>>(src, sw, sh, spitch, dst, dw, dh, dpitch, scx, scy);
	return cudaGetLastError();
}
// scx/scy: source/destination scale; 1/factor for the factor form cv::resize(..., Size(), fx, fy, INTER_NEAREST)
// (ScaleDepthData, SceneDensify.cpp:596-599), <= 0 for the destination-size form (sw/dw)
cudaError_t rs_launch_nearest(const float* src, int sw, int sh, int ch, float* dst, int dw, int dh, double scx, double scy, cudaStream_t s) {
	dim3 b(32, 8);
	resize_nearest_kernel<<<grid2(dw, dh, b), b, 0, s>>>(src, sw, sh, ch, dst, dw, dh, scx > 0 ? scx : (double)sw/dw, scy > 0 ? scy : (double)sh/dh);
	return cudaGetLastError();
}
cudaError_t rs_launch_nearest_u8(const uint8_t* src, int sw, int sh, int spitch, uint8_t* dst, int dw, int dh, cudaStream_t s) {
	dim3 b(32, 8);
	resize_nearest_u8_kernel<<<grid2(dw, dh, b), b, 0, s>>>(src, sw, sh, spitch, dst, dw, dh, (double)sw/dw, (double)sh/dh);
	return cudaGetLastError();
}
cudaError_t rs_launch_plane_up(const float4* src, int sw, int sh, float4* dst, float* prior, int dw, int dh, bool nearestDepth, cudaStream_t s) {
	dim3 b(32, 8);
	plane_up_kernel<<<grid2(dw, dh, b), b, 0, s>>>(src, sw, sh, dst, prior, dw, dh, (double)sw/dw, (double)sh/dh, nearestDepth ? 1 : 0);
	return cudaGetLastError();
}

// TImage<Pixel8U>::toGray(out, COLOR_BGR2GRAY / COLOR_RGB2GRAY, bNormalize = true) (libs/Common/Types.inl:2377-2431), the
// conversion DepthMapsData::InitViews applies to every image (SceneDensify.cpp:324,345): each channel is scaled by
// float(1)/float(255) first (NormRGB_t, Types.inl:1610-1615), then gray = (cb*B + cg*G) + cr*R with cb, cg, cr = .114, .587, .299
// in float.  Explicit _rn intrinsics: no FMA contraction, same bits as the oracle.
__global__ void to_gray_kernel(const uint8_t* __restrict__ src, int w, int h, int sstride, int channels, int bgr, float* __restrict__ dst, int dpitch) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= w || y >= h) return;
	const uint8_t* p = src + (size_t)y*sstride + (size_t)x*channels;
	const float inv = 1.f/255.f;
	const float c0 = __fmul_rn((float)p[0], inv), c1 = __fmul_rn((float)p[1], inv), c2 = __fmul_rn((float)p[2], inv);
	const float k0 = bgr ? 0.114f : 0.299f, k2 = bgr ? 0.299f : 0.114f;
	dst[(size_t)y*dpitch+x] = __fadd_rn(__fadd_rn(__fmul_rn(k0, c0), __fmul_rn(0.587f, c1)), __fmul_rn(k2, c2));
}
cudaError_t rs_launch_to_gray(const uint8_t* src, int w, int h, int sstride, int channels, int bgr, float* dst, int dpitch, cudaStream_t s) {
	dim3 b(32, 8);
	to_gray_kernel<<<grid2(w, h, b), b, 0, s>>>(src, w, h, sstride, channels, bgr, dst, dpitch);
	return cudaGetLastError();
}
