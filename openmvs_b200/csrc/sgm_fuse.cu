// sgm_fuse.cu — fusion-mode -2 on the device: the disparity maps of the SGM pairs that contain an image, projected into the image and
// fused into its depth-map (SemiGlobalMatcher::Fuse, libs/MVS/SemiGlobalMatcher.cpp:739-859), and the normal map of a depth-map.
//
//   sgmf_project_kernel   ProjectDisparity2DepthMap, splat (:1950-1993): every source's 64-bit atomicMin into the key map of its
//                         quadrant at the up to 9 targets it reaches; key = (bits of dist^2) << 32 | source index, so the minimum is
//                         "nearest, then earliest in raster order", the sequential loop's `ndepth > 0 && ndistSq <= distSq` rule
//   sgmf_gather_kernel    ProjectDisparity2DepthMap, combination (:1994-2035): reads the four keys of a target, recomputes the
//                         winning sources' values (a pure function of the source index) and writes depth, range and conf
//   sgmf_fuse_kernel      the cluster vote of Fuse (:795-848), one thread per pixel, clusters as pair bit masks
//   sgmf_normal_kernel    EstimateNormalMap (libs/MVS/DepthMap.cpp:1522-1613), a 3x3 stencil
// Disparity2Depth runs in double (Image.cpp:373-404); every float and double operation is an explicitly rounded intrinsic, so no FMA
// contraction separates the kernels from the sequential restatement compiled without contraction.  No value is written by racing
// threads: the splat only orders keys, and each output has one writer.
#include "sgm_common.cuh"
#include <cfloat>

namespace {

// Image::Disparity2Depth(Q, u, d) (Image.cpp:373-381): depth of the rectified pixel u at disparity d, 0 when w is ~0 or depth < 1e-4
__device__ float d2d(const double* __restrict__ Q, double x, double y, float d) {
	const double dd = d;
	const double w = __dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(Q[12], x), __dmul_rn(Q[13], y)), __dmul_rn(Q[14], dd)), Q[15]);
	if (fabs(w) < 1e-7) return 0.f;
	const double z = __dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(Q[8], x), __dmul_rn(Q[9], y)), __dmul_rn(Q[10], dd)), Q[11]);
	const float depth = __double2float_rn(__ddiv_rn(z, w));
	return depth < 1e-4f ? 0.f : depth;
}

// One valid source of a pair: its depth, range, confidence and position in the target image.  false: NO_DISP, no positive depth
// (Image.cpp:392-404), or a position whose 3x3 block lies outside the image (the sequential loop then writes nothing either; the test
// also keeps the float -> int conversion of the position defined).
struct Source { float depth, lo, hi, conf, ux, uy; int x0, y0; };

__device__ bool source(const SGMFusePair& P, int s, int W, int H, Source& o) {
	const int dint = P.disp[s];
	if (dint == SGM_NO_DISP) return false;
	const int r = s / P.vw, c = s - r*P.vw;
	const double x = c+SGM_HW, y = r+SGM_HW;
	const float disparity = __fdiv_rn((float)dint, (float)P.steps);
	const double* Q = P.Q;
	const double dd = disparity;
	const double w = __dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(Q[12], x), __dmul_rn(Q[13], y)), __dmul_rn(Q[14], dd)), Q[15]);
	if (fabs(w) < 1e-7) return false;
	const double z = __ddiv_rn(__dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(Q[8], x), __dmul_rn(Q[9], y)), __dmul_rn(Q[10], dd)), Q[11]), w);
	if (z < 1e-7) return false;
	const double nrm = __ddiv_rn(1.0, __dmul_rn(w, z));
	const float ux = __double2float_rn(__dmul_rn(__dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(Q[0], x), __dmul_rn(Q[1], y)), __dmul_rn(Q[2], dd)), Q[3]), nrm));
	const float uy = __double2float_rn(__dmul_rn(__dadd_rn(__dsub_rn(__dadd_rn(__dmul_rn(Q[4], x), __dmul_rn(Q[5], y)), __dmul_rn(Q[6], dd)), Q[7]), nrm));
	o.depth = __double2float_rn(z);
	if (!(o.depth > 0.f)) return false;
	const float fx = floorf(ux), fy = floorf(uy);
	if (!(fx >= -1.f && fx <= (float)W && fy >= -1.f && fy <= (float)H)) return false;
	const int dc = (int)(short)(int)floorf(disparity);
	o.lo = d2d(Q, x, y, (float)(dc-1));
	o.hi = d2d(Q, x, y, (float)(dc+1));
	o.conf = P.cost ? __fdiv_rn(1.f, (float)((int)P.cost[s]+1)) : 0.f;
	o.x0 = (int)fx; o.y0 = (int)fy;
	o.ux = __fsub_rn(ux, 0.5f); o.uy = __fsub_rn(uy, 0.5f);
	return true;
}

constexpr float OVERLAP = 0.75f;   // 0.5f+0.25f
constexpr unsigned long long NO_KEY = ~0ull;

__global__ void sgmf_project_kernel(const SGMFuseArgs A, int W, int H, unsigned long long* __restrict__ keys) {
	const SGMFusePair& P = A.pair[blockIdx.z];
	const int c = blockIdx.x*blockDim.x+threadIdx.x, r = blockIdx.y*blockDim.y+threadIdx.y;
	if (c >= P.vw || r >= P.vh) return;
	const int s = r*P.vw+c;
	Source S;
	if (!source(P, s, W, H, S)) return;
	const size_t n = (size_t)W*H;
	unsigned long long* K = keys + (size_t)blockIdx.z*4*n;
	for (int i = -1; i <= 1; ++i) {
		for (int j = -1; j <= 1; ++j) {
			const int nx = S.x0+j, ny = S.y0+i;
			if (nx < 0 || ny < 0 || nx >= W || ny >= H) continue;
			const float dx = __fsub_rn((float)nx, S.ux), dy = __fsub_rn((float)ny, S.uy);
			if (fabsf(dx) > OVERLAP || fabsf(dy) > OVERLAP) continue;
			const int q = (dx < 0.f ? 1 : 0) + (dy < 0.f ? 2 : 0);
			const float dsq = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
			atomicMin(K + (size_t)q*n + (size_t)ny*W + nx, ((unsigned long long)__float_as_uint(dsq) << 32) | (unsigned)s);
		}
	}
}

__device__ __forceinline__ bool depth_similar(float d0, float d1, float th) { return __fdiv_rn(fabsf(__fsub_rn(d0, d1)), d0) < th; }

__global__ void sgmf_gather_kernel(const SGMFuseArgs A, int W, int H, const unsigned long long* __restrict__ keys, float* __restrict__ depth,
	float2* __restrict__ range, float* __restrict__ conf, size_t pairStride)
{
	const int c = blockIdx.x*blockDim.x+threadIdx.x, r = blockIdx.y*blockDim.y+threadIdx.y;
	if (c >= W || r >= H) return;
	const SGMFusePair& P = A.pair[blockIdx.z];
	const size_t n = (size_t)W*H, i = (size_t)r*W+c, o = (size_t)blockIdx.z*pairStride+i;
	const unsigned long long* K = keys + (size_t)blockIdx.z*4*n;
	unsigned long long key[4];
	#pragma unroll
	for (int q = 0; q < 4; ++q) key[q] = K[q*n+i];
	// the nearest entry, the first in quadrant order on ties (:2002-2014)
	float distCenter = FLT_MAX, depthCenter = 0.f;
	Source S[4];
	#pragma unroll
	for (int q = 0; q < 4; ++q) {
		if (key[q] == NO_KEY) continue;
		source(P, (int)(unsigned)key[q], W, H, S[q]);
		const float dist = __uint_as_float((unsigned)(key[q] >> 32));
		if (distCenter > dist) { distCenter = dist; depthCenter = S[q].depth; }
	}
	float v0 = 0.f, v1 = 0.f, v2 = 0.f, v3 = 0.f, wsum = 0.f;
	if (!(distCenter > OVERLAP*OVERLAP)) {
		// TAccumulator<Vec4f>: value += v*w, weight += w, in quadrant order (:2019-2027)
		#pragma unroll
		for (int q = 0; q < 4; ++q) {
			if (key[q] == NO_KEY || !depth_similar(depthCenter, S[q].depth, 0.02f)) continue;
			const float w = __fsqrt_rn(__uint_as_float((unsigned)(key[q] >> 32)));
			v0 = __fadd_rn(v0, __fmul_rn(S[q].depth, w)); v1 = __fadd_rn(v1, __fmul_rn(S[q].lo, w));
			v2 = __fadd_rn(v2, __fmul_rn(S[q].hi, w)); v3 = __fadd_rn(v3, __fmul_rn(S[q].conf, w));
			wsum = __fadd_rn(wsum, w);
		}
	}
	if (wsum > 0.f) {
		// Normalized(): value * (1/weight) (TMatrix operator /, libs/Common/Types.inl:1466-1470)
		const float inv = __fdiv_rn(1.f, wsum);
		v0 = __fmul_rn(v0, inv); v1 = __fmul_rn(v1, inv); v2 = __fmul_rn(v2, inv); v3 = __fmul_rn(v3, inv);
	} else {
		// no entry within 0.75 pixel, or the only agreeing one sits on the centre (weight 0; 0/0 in the reference): rejected
		v0 = v1 = v2 = v3 = 0.f;
	}
	depth[o] = v0;
	range[o] = make_float2(v1, v2);
	if (conf) conf[o] = v3;
}

__global__ void sgmf_fuse_kernel(int nPairs, int W, int H, const float* __restrict__ depth, const float2* __restrict__ range,
	const float* __restrict__ conf, size_t pairStride, int minViews, float* __restrict__ outDepth, float* __restrict__ outConf)
{
	const int c = blockIdx.x*blockDim.x+threadIdx.x, r = blockIdx.y*blockDim.y+threadIdx.y;
	if (c >= W || r >= H) return;
	const size_t i = (size_t)r*W+c;
	// clusters in the order they were opened; a cluster's members are the set bits of its mask, joined in ascending pair order
	unsigned mask[B200MVS_SGM_MAX_PAIRS]; float lo[B200MVS_SGM_MAX_PAIRS], hi[B200MVS_SGM_MAX_PAIRS];
	int nc = 0;
	for (int p = 0; p < nPairs; ++p) {
		const float d = depth[(size_t)p*pairStride+i];
		if (!(d > 0.f)) continue;
		const float2 rg = range[(size_t)p*pairStride+i];
		bool joined = false;
		for (int k = 0; k < nc; ++k) {
			if (!(lo[k] <= d && d < hi[k])) continue;   // ISINSIDE
			mask[k] |= 1u << p;
			if (lo[k] < rg.x) lo[k] = rg.x;
			if (hi[k] > rg.y) hi[k] = rg.y;
			joined = true;
		}
		if (!joined) { mask[nc] = 1u << p; lo[nc] = rg.x; hi[nc] = rg.y; ++nc; }
	}
	float od = 0.f, oc = 0.f;
	if (nc > 0) {
		// the largest cluster, the first one on ties (std::max_element)
		int best = 0, bestN = __popc(mask[0]);
		for (int k = 1; k < nc; ++k) { const int m = __popc(mask[k]); if (bestN < m) { best = k; bestN = m; } }
		if (bestN >= minViews) {
			for (unsigned m = mask[best]; m; m &= m-1) {
				const size_t o = (size_t)(__ffs(m)-1)*pairStride+i;
				od = __fadd_rn(od, depth[o]);
				oc = __fadd_rn(oc, conf[o]);
			}
			od = __fdiv_rn(od, (float)bestN); oc = __fdiv_rn(oc, (float)bestN);
		}
	}
	outDepth[i] = od;
	if (outConf) outConf[i] = oc;
}

__global__ void sgmf_normal_kernel(const float* __restrict__ D, int W, int H, float4 K, float* __restrict__ N) {
	const int c = blockIdx.x*blockDim.x+threadIdx.x, r = blockIdx.y*blockDim.y+threadIdx.y;
	if (c >= W || r >= H) return;
	const size_t i = (size_t)r*W+c;
	float nx = 0.f, ny = 0.f, nz = 0.f;
	const float w = D[i];
	if (w > 0.f) {
		// DepthGradient: least-squares plane over the valid 8-neighbours
		int whxx = 0, whxy = 0, whyy = 0, n = 0;
		float wgx = 0.f, wgy = 0.f;
		for (int y = -1; y <= 1; ++y) {
			for (int x = -1; x <= 1; ++x) {
				if (x == 0 && y == 0) continue;
				const int px = c+x, py = r+y;
				if (px < 0 || py < 0 || px >= W || py >= H) continue;
				const float wi = D[(size_t)py*W+px];
				if (!(wi > 0.f && depth_similar(w, wi, 0.03f))) continue;
				whxx += x*x; whxy += x*y; whyy += y*y;
				const float dw = __fsub_rn(wi, w);
				wgx = __fadd_rn(wgx, __fmul_rn(dw, (float)x)); wgy = __fadd_rn(wgy, __fmul_rn(dw, (float)y));
				++n;
			}
		}
		const int det = whxx*whyy - whxy*whxy;
		if (n >= 3 && det != 0) {
			const float invDet = __fdiv_rn(1.f, (float)det);
			const float wx = __fmul_rn(__fsub_rn(__fmul_rn((float)whyy, wgx), __fmul_rn((float)whxy, wgy)), invDet);
			const float wy = __fmul_rn(__fadd_rn(__fmul_rn((float)(-whxy), wgx), __fmul_rn((float)whxx, wgy)), invDet);
			// ComputeNormal, then normalized(): cv::normalize, the norm in double and a double scale rounded to float
			const float ax = __fmul_rn(K.x, wx), ay = __fmul_rn(K.y, wy);
			const float az = __fsub_rn(__fadd_rn(__fmul_rn(__fsub_rn(K.z, (float)c), wx), __fmul_rn(__fsub_rn(K.w, (float)r), wy)), w);
			double s = __dmul_rn((double)ax, (double)ax);
			s = __dadd_rn(s, __dmul_rn((double)ay, (double)ay));
			s = __dadd_rn(s, __dmul_rn((double)az, (double)az));
			const double nv = __dsqrt_rn(s);
			const double k = nv != 0.0 ? __ddiv_rn(1.0, nv) : 0.0;
			nx = __double2float_rn(__dmul_rn((double)ax, k)); ny = __double2float_rn(__dmul_rn((double)ay, k)); nz = __double2float_rn(__dmul_rn((double)az, k));
		}
	}
	N[3*i] = nx; N[3*i+1] = ny; N[3*i+2] = nz;
}

const dim3 BLOCK(32, 8);
inline dim3 grid3(int w, int h, int z) { return dim3((w+BLOCK.x-1)/BLOCK.x, (h+BLOCK.y-1)/BLOCK.y, z); }

} // namespace

cudaError_t sgmf_launch_project(const SGMFuseArgs& A, int W, int H, unsigned long long* keys, cudaStream_t s) {
	int mw = 0, mh = 0;
	for (int p = 0; p < A.n; ++p) { mw = max(mw, A.pair[p].vw); mh = max(mh, A.pair[p].vh); }
	cudaError_t e = cudaMemsetAsync(keys, 0xFF, (size_t)A.n*4*W*H*sizeof(unsigned long long), s);
	if (e != cudaSuccess) return e;
	sgmf_project_kernel<<<grid3(mw, mh, A.n), BLOCK, 0, s>>>(A, W, H, keys);
	return cudaGetLastError();
}

cudaError_t sgmf_launch_gather(const SGMFuseArgs& A, int W, int H, const unsigned long long* keys, float* depth, float2* range, float* conf,
	size_t pairStride, cudaStream_t s)
{
	sgmf_gather_kernel<<<grid3(W, H, A.n), BLOCK, 0, s>>>(A, W, H, keys, depth, range, conf, pairStride);
	return cudaGetLastError();
}

cudaError_t sgmf_launch_fuse(int nPairs, int W, int H, const float* depth, const float2* range, const float* conf, size_t pairStride,
	int minViews, float* outDepth, float* outConf, cudaStream_t s)
{
	sgmf_fuse_kernel<<<grid3(W, H, 1), BLOCK, 0, s>>>(nPairs, W, H, depth, range, conf, pairStride, minViews, outDepth, outConf);
	return cudaGetLastError();
}

cudaError_t sgmf_launch_normals(const float* depth, int W, int H, float4 K, float* normal, cudaStream_t s) {
	sgmf_normal_kernel<<<grid3(W, H, 1), BLOCK, 0, s>>>(depth, W, H, K, normal);
	return cudaGetLastError();
}
