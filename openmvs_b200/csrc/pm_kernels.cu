// pm_kernels.cu — PatchMatch depth+normal estimation kernels, hand-written for sm_90a.
//
// What they compute (behaviour, not code, follows the reference CPU estimator):
//   pm_score_kernel   pass A  ScoreDepthMapTmp            libs/MVS/SceneDensify.cpp:490-517
//   pm_sweep_kernel   pass B  DepthEstimator::ProcessPixel libs/MVS/DepthMap.cpp:630-852
//                             scored by ScorePixel/ScorePixelImage (DepthMap.cpp:465-626)
//   pm_finalize_kernel pass C EndDepthMapTmp              libs/MVS/SceneDensify.cpp:528-548
//
// Schedule: red-black.  One thread owns one pixel of the active colour; a warp owns 32
// same-colour pixels of one image row (64-pixel span), so the homography-warped taps of
// the 32 lanes fall on 2-3 cache lines of two neighbour-image rows.  The bilateral
// weights of the 5x5 reference patch are computed once per pixel and sweep from a reference
// tile that TMA stages into shared memory, kept in shared memory as float2{w, tw}[tap][thread]
// (80 registers per thread, 24 warps per SM) and reused by every hypothesis x view.
// All four 4-neighbours belong to the other colour, so in-place updates are race-free.
// Measured design history and the variants that were dropped: DESIGN.md section 5.1.
#include "pm_common.cuh"
#include <math_constants.h>

namespace {

constexpr int BLOCK_X = 32;  // lanes: 32 same-colour pixels = 64-pixel span
constexpr int BLOCK_Y = 8;

constexpr int NTHREADS = BLOCK_X*BLOCK_Y;
static_assert(BLOCK_X == 32, "pm_sweep_kernel: a warp is one row of the CTA");

// bilateral weights of the 5x5 reference patch (WeightedPatchFix<25>, DepthMap.h:145-155), kept in shared
// memory as float2{w,tw}[tap][thread] (conflict-free LDS.64): 50 registers per thread less than a register copy
struct PatchW {
	float2* s; // &smem[threadIndex]; tap k at s[k*NTHREADS]
	float sumW, normSq0;
	__device__ __forceinline__ void set(int k, float a, float b) { s[k*NTHREADS] = make_float2(a, b); }
	__device__ __forceinline__ float2 get(int k) const { return s[k*NTHREADS]; }
};

// ---- TMA staging of the reference tile ---------------------------------------------------------
// A CTA of the sweep kernel covers 64 x 8 pixels; their 9x9 patches need a (64+8) x (8+8) float tile
// of the reference image.  One elected thread issues a cp.async.bulk.tensor.2d (TMA) into shared
// memory and everybody waits on the mbarrier; out-of-image parts of the box are zero-filled by the
// TMA unit (those pixels are rejected by the patch-inside test anyway).
constexpr int TILE_W = 2*BLOCK_X+2*PM_HALF;   // 72 floats = 288 B (multiple of 16 B)
constexpr int TILE_H = BLOCK_Y+2*PM_HALF;     // 16 rows
constexpr int TILE_BYTES = TILE_W*TILE_H*4;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity) {
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_LOOP:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra WAIT_DONE;\n"
		"bra WAIT_LOOP;\n"
		"WAIT_DONE:\n"
		"}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
	asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
		:: "r"(smem_u32(dst)), "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar)) : "memory");
}

// The reference texel at offset (dx, dy) from the pixel: from the image in global memory (pass A) or from the staged tile
// (pass B; (lx, ly) = pixel position inside the tile)
struct ImageTexels {
	const float* __restrict__ img; int pitch, x, y;
	__device__ __forceinline__ float operator()(int dx, int dy) const { return __ldg(img + (size_t)(y+dy)*pitch + (x+dx)); }
};
struct TileTexels {
	const float* tile; int lx, ly;
	__device__ __forceinline__ float operator()(int dx, int dy) const { return tile[(ly+dy)*TILE_W + (lx+dx)]; }
};

// FillPixelPatch + GetWeight (DepthMap.cpp:422-462, DepthMap.h:403-412).  WEIGHTS_ALIAS_TILE: the weights share their
// shared memory with the tile the texels come from (pm_sweep_kernel), so every thread of the CTA calls this, and the
// weights are written only after all threads have read their patch.
template <bool WEIGHTS_ALIAS_TILE, typename Texels>
__device__ __forceinline__ void fill_patch(const Texels& texel, PatchW& p) {
	const float sigmaColor = -1.f/(2.f*0.1f*0.1f);
	const float sigmaSpatial = -1.f/(2.f*9.f);
	const float center = texel(0, 0);
	float acc = 0.f, sumW = 0.f;
	float w[PM_TEXELS], I[PM_TEXELS];
	#pragma unroll
	for (int i = 0; i < 5; ++i) {
		#pragma unroll
		for (int j = 0; j < 5; ++j) {
			const int dy = 2*i-PM_HALF, dx = 2*j-PM_HALF;
			const float v = texel(dx, dy);
			const float dI = v-center;
			const float wgt = expf(dI*dI*sigmaColor + float(dx*dx+dy*dy)*sigmaSpatial);
			w[i*5+j] = wgt;
			I[i*5+j] = v;
			acc += v*wgt;
			sumW += wgt;
		}
	}
	const float tm = acc/sumW;
	float nsq = 0.f, tw[PM_TEXELS];
	#pragma unroll
	for (int k = 0; k < PM_TEXELS; ++k) {
		const float t = I[k]-tm;
		tw[k] = w[k]*t;
		nsq += tw[k]*t;
	}
	if (WEIGHTS_ALIAS_TILE)
		__syncthreads();
	#pragma unroll
	for (int k = 0; k < PM_TEXELS; ++k)
		p.set(k, w[k], tw[k]);
	p.sumW = sumW;
	p.normSq0 = nsq;
}

struct Hyp {      // one plane hypothesis at the current pixel
	float d;      // depth
	float3 n;     // unit normal, camera space
	float invd;   // 1/d
	float3 ms;    // (n^T Kref^-1) / (n.X0 d)
	float smooth; // product of the smoothness factors (view independent)
};

__device__ __forceinline__ float fast_rcp(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float pow2neg(unsigned i) { return __int_as_float((int)(127u-i)<<23); } // 2^-i, scaleRanges[] (DepthMap.cpp:358-359)
__device__ __forceinline__ float dot3(const float3& a, const float3& b) { return a.x*b.x + a.y*b.y + a.z*b.z; }

// the viewing ray X0 = Kref^-1 (x, y, 1) of pixel (x, y); its z component is 1
__device__ __forceinline__ float2 pixel_ray(const PMParams& P, float fx, float fy) {
	return make_float2(fx*P.ifx + fy*P.sk + P.ox, fy*P.ify + P.oy);
}

// A pixel that is estimated: its patch lies inside the image and the ignore-mask (DepthData::ApplyIgnoreMask,
// DepthMap.cpp:215-230; masked pixels are not in the pixel list, DepthMap.cpp:343) keeps it
__device__ __forceinline__ bool pixel_active(const PMParams& P, int x, int y) {
	return x >= PM_HALF && y >= PM_HALF && x < P.W-PM_HALF && y < P.H-PM_HALF
		&& !(P.mask && P.mask[(size_t)y*P.maskPitch + x] == 0);
}

// The low-resolution depth prior of pixel idx and its weight (DepthMap.cpp:552-561); false when the patch is too flat
// (fDescriptorMinMagnitudeThreshold) and no prior vouches for the pixel
__device__ __forceinline__ bool pixel_prior(const PMParams& P, size_t idx, float normSq0, float& priorD, float& priorF) {
	priorD = 0.f; priorF = 0.f;
	if (P.lowres)
		priorD = fmaxf(__ldg(P.lowres + idx), 0.f);
	if (normSq0 < P.thMagnitudeSq && !(priorD > 0.f))
		return false;
	if (priorD > 0.f)
		priorF = expf(normSq0*(-1.f/0.02f));
	return true;
}

// masked bilinear depth sample (TImage::sample with functor, libs/Common/Types.inl:2297-2313)
__device__ __forceinline__ bool sample_depth_masked(const float* __restrict__ img, int pitch, float px, float py, float ref, float& v) {
	const int lx = (int)px, ly = (int)py;
	const float x = px-lx, x1 = 1.f-x, y = py-ly, y1 = 1.f-y;
	const float* r0 = img + (size_t)ly*pitch + lx;
	const float x0y0 = __ldg(r0), x1y0 = __ldg(r0+1), x0y1 = __ldg(r0+pitch), x1y1 = __ldg(r0+pitch+1);
	const bool b00 = fabsf(ref-x0y0)/ref < 0.03f, b10 = fabsf(ref-x1y0)/ref < 0.03f;
	const bool b01 = fabsf(ref-x0y1)/ref < 0.03f, b11 = fabsf(ref-x1y1)/ref < 0.03f;
	if (!b00 && !b10 && !b01 && !b11)
		return false;
	v = y1*(x1*(b00 ? x0y0 : (b10 ? x1y0 : (b01 ? x0y1 : x1y1))) + x*(b10 ? x1y0 : (b00 ? x0y0 : (b11 ? x1y1 : x0y1)))) +
	    y *(x1*(b01 ? x0y1 : (b11 ? x1y1 : (b00 ? x0y0 : x1y0))) + x*(b11 ? x1y1 : (b01 ? x0y1 : (b10 ? x1y0 : x0y0))));
	return true;
}

// Tap addressing without float<->int conversions (those run on the XU pipe beside the reciprocal).  For
// 0 <= p < 2^23, p + 2^23 lies in [2^23, 2^24), where consecutive floats are 1 apart, so the sum rounded toward
// zero is t = 2^23 + floor(p) exactly: t - 2^23 is floor(p) (exact, and equal to (float)(int)p since p >= 0), and
// the bit pattern of t is TAP_BIAS + floor(p).  Every lane that loads satisfies 0 <= p < 2^23: a lane that passed
// the corner test has its taps inside [1, w-2] up to rounding, and a rejected lane samples (1, 1).
constexpr unsigned TAP_BIAS = 0x4B000000u;  // bit pattern of 2^23
__device__ __forceinline__ float tap_floor(float p, unsigned& bits) {
	const float t = __fadd_rz(p, 0x1p23f);
	bits = __float_as_uint(t);
	return t - 0x1p23f;
}

// The four texels of one warped tap of a plain float image (pitch in floats).  xb / yb: bit patterns from
// tap_floor (TAP_BIAS + column / row); base: image pointer minus 4*TAP_BIAS bytes (tap_base), so that the column
// bias cancels inside the 64-bit address; the row bias is taken off before the multiply.  The element index
// (yb-TAP_BIAS)*pitch + xb = TAP_BIAS + y*pitch + x stays below 2^32 for images of fewer than 3e9 floats.
// L1 evict-last: the warped footprints of successive hypotheses and of the CTA's other rows overlap, keeping
// them in L1 against the streaming plane/cost traffic.
// (alternatives tried and dropped, DESIGN.md §5.1: row-pair and float4 quad layouts, column-parity planes, texture
//  gather TLD4, a TLD4/LDG split across views)
__device__ __forceinline__ unsigned long long tap_base(const float* img) { return (unsigned long long)img - 4ull*TAP_BIAS; }
__device__ __forceinline__ void fetch_texels(unsigned long long base, int pitch, unsigned xb, unsigned yb,
	float& v00, float& v10, float& v01, float& v11)
{
	unsigned long long addr;
	const unsigned idx = (yb-TAP_BIAS)*(unsigned)pitch + xb;
	asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(addr) : "r"(idx), "r"(4u), "l"(base));
	const float* r0 = (const float*)addr;
	const float* r1 = r0+pitch;
	asm("ld.global.nc.L1::evict_last.f32 %0, [%1];" : "=f"(v00) : "l"(r0));
	asm("ld.global.nc.L1::evict_last.f32 %0, [%1+4];" : "=f"(v10) : "l"(r0));
	asm("ld.global.nc.L1::evict_last.f32 %0, [%1];" : "=f"(v01) : "l"(r1));
	asm("ld.global.nc.L1::evict_last.f32 %0, [%1+4];" : "=f"(v11) : "l"(r1));
}

// ScorePixelImage (DepthMap.cpp:465-564) for one neighbour view.
// The reference rejects a hypothesis as soon as one warped tap leaves the neighbour image
// (1-pixel border).  A homography maps the convex patch quad onto the convex quad of its
// projected corners as long as the depth Z keeps its sign, so "all 25 taps inside" is decided
// once from the 4 corner taps; the tap loop itself is then branch-free and test-free, and the
// loads of a whole tap row are in flight together.  Rejected lanes run the loop on texel (1,1).
template <bool GEOM>
__device__ __forceinline__ float score_view(const PMParams& P, const PMView& V, const PatchW& pt,
	float fx, float fy, float X0x, float X0y, const Hyp& h, float priorF, float priorD)
{
	// H = A + Hm (n^T Kref^-1)/(n.X0 d); columns 0/1 and the centre point H*(x,y,1)
	float c0x = fmaf(V.Hm[0], h.ms.x, V.A[0]), c0y = fmaf(V.Hm[1], h.ms.x, V.A[3]), c0z = fmaf(V.Hm[2], h.ms.x, V.A[6]);
	float c1x = fmaf(V.Hm[0], h.ms.y, V.A[1]), c1y = fmaf(V.Hm[1], h.ms.y, V.A[4]), c1z = fmaf(V.Hm[2], h.ms.y, V.A[7]);
	const float xc = fmaf(V.Hm[0], h.invd, fmaf(V.A[0], fx, fmaf(V.A[1], fy, V.A[2])));
	const float yc = fmaf(V.Hm[1], h.invd, fmaf(V.A[3], fx, fmaf(V.A[4], fy, V.A[5])));
	const float zc = fmaf(V.Hm[2], h.invd, fmaf(V.A[6], fx, fmaf(V.A[7], fy, V.A[8])));
	// top-left tap, then steps of 2 pixels
	float bx = fmaf(-4.f, c0x+c1x, xc), by = fmaf(-4.f, c0y+c1y, yc), bz = fmaf(-4.f, c0z+c1z, zc);
	c0x *= 2.f; c0y *= 2.f; c0z *= 2.f; c1x *= 2.f; c1y *= 2.f; c1z *= 2.f;
	const float xmax = float(V.w-2), ymax = float(V.h-2);
	bool ok;
	{
		// the four corner taps (0,0) (4,0) (0,4) (4,4)
		const float x1 = fmaf(4.f, c0x, bx), y1 = fmaf(4.f, c0y, by), z1 = fmaf(4.f, c0z, bz);
		const float x2 = fmaf(4.f, c1x, bx), y2 = fmaf(4.f, c1y, by), z2 = fmaf(4.f, c1z, bz);
		const float x3 = fmaf(4.f, c1x, x1), y3 = fmaf(4.f, c1y, y1), z3 = fmaf(4.f, c1z, z1);
		const float zmin = fminf(fminf(bz, z1), fminf(z2, z3)), zmax = fmaxf(fmaxf(bz, z1), fmaxf(z2, z3));
		const float i0 = fast_rcp(bz), i1 = fast_rcp(z1), i2 = fast_rcp(z2), i3 = fast_rcp(z3);
		const float pxmin = fminf(fminf(bx*i0, x1*i1), fminf(x2*i2, x3*i3)), pxmax = fmaxf(fmaxf(bx*i0, x1*i1), fmaxf(x2*i2, x3*i3));
		const float pymin = fminf(fminf(by*i0, y1*i1), fminf(y2*i2, y3*i3)), pymax = fmaxf(fmaxf(by*i0, y1*i1), fmaxf(y2*i2, y3*i3));
		ok = (zmin > 0.f || zmax < 0.f) && pxmin >= 1.f && pymin >= 1.f && pxmax <= xmax && pymax <= ymax;
		// NaN anywhere makes a comparison false (fminf/fmaxf drop NaNs, so test them explicitly)
		ok = ok && (bx*i0 == bx*i0) && (x1*i1 == x1*i1) && (x2*i2 == x2*i2) && (x3*i3 == x3*i3)
		        && (by*i0 == by*i0) && (y1*i1 == y1*i1) && (y2*i2 == y2*i2) && (y3*i3 == y3*i3);
	}
	if (!__any_sync(__activemask(), ok))
		return P.thRobust;
	if (!ok) { bx = by = bz = 1.f; c0x = c0y = c0z = c1x = c1y = c1z = 0.f; }
	unsigned long long base = tap_base(V.img);
	int pitch = V.pitch;
	// keep the per-view constants in registers (otherwise re-read from the constant bank per tap)
	asm volatile("" : "+r"(pitch), "+l"(base));
	float sum = 0.f, sumSq = 0.f, num = 0.f;
	#pragma unroll
	for (int i = 0; i < 5; ++i) {
		float X = bx, Y = by, Z = bz;
		#pragma unroll
		for (int j = 0; j < 5; ++j) {
			const float iz = fast_rcp(Z);
			const float px = X*iz, py = Y*iz;
			unsigned xb, yb;
			const float ax = px-tap_floor(px, xb), ay = py-tap_floor(py, yb);
			float v00, v10, v01, v11;
			fetch_texels(base, pitch, xb, yb, v00, v10, v01, v11);
			const float top = fmaf(ax, v10-v00, v00), bot = fmaf(ax, v11-v01, v01);
			const float v = fmaf(ay, bot-top, top);
			const float2 wk = pt.get(i*5+j);
			const float vw = v*wk.x;
			sum += vw; sumSq = fmaf(v, vw, sumSq); num = fmaf(v, wk.y, num);
			X += c0x; Y += c0y; Z += c0z;
		}
		bx += c1x; by += c1y; bz += c1z;
	}
	const bool bad = !ok;
	if (bad)
		return P.thRobust;
	const float normSq1 = sumSq - sum*sum/pt.sumW;
	const float nrmSq = pt.normSq0*normSq1;
	if (nrmSq <= 1e-16f)
		return P.thRobust;
	const float ncc = fminf(fmaxf(num/sqrtf(nrmSq), -1.f), 1.f);
	float score = (1.f-ncc)*h.smooth;
	if (GEOM) {
		if (V.dmap) {
			// forward/backward reprojection through the neighbour's depth-map (DepthMap.cpp:535-551)
			float consistency = 4.f;
			const float Xx = X0x*h.d, Xy = X0y*h.d, Xz = h.d;
			const float X1x = V.Tl[0]*Xx + V.Tl[1]*Xy + V.Tl[2]*Xz + V.Tm[0];
			const float X1y = V.Tl[3]*Xx + V.Tl[4]*Xy + V.Tl[5]*Xz + V.Tm[1];
			const float X1z = V.Tl[6]*Xx + V.Tl[7]*Xy + V.Tl[8]*Xz + V.Tm[2];
			if (X1z > 0.f) {
				const float x1x = X1x/X1z, x1y = X1y/X1z;
				if (x1x >= 1.f && x1y >= 1.f && x1x <= float(V.dw-2) && x1y <= float(V.dh-2)) {
					float depth1;
					if (sample_depth_masked(V.dmap, V.dpitch, x1x, x1y, X1z, depth1)) {
						const float Px = x1x*depth1, Py = x1y*depth1, Pz = depth1;
						const float Bx = V.Tr[0]*Px + V.Tr[1]*Py + V.Tr[2]*Pz + V.Tn[0];
						const float By = V.Tr[3]*Px + V.Tr[4]*Py + V.Tr[5]*Pz + V.Tn[1];
						const float Bz = V.Tr[6]*Px + V.Tr[7]*Py + V.Tr[8]*Pz + V.Tn[2];
						const float ex = fx-Bx/Bz, ey = fy-By/Bz;
						const float dist = sqrtf(ex*ex + ey*ey);
						consistency = fminf(sqrtf(dist*(dist+2.f)), consistency);
					}
				}
			}
			score += P.geomWeight*consistency;
		}
	}
	if (priorD > 0.f) {
		// low-resolution depth prior (DepthMap.cpp:552-561)
		const float deltaDepth = fminf(fabsf(priorD-h.d)/priorD, 0.5f);
		score = (1.f-priorF)*score + priorF*deltaDepth;
	}
	return fminf(2.f, score);
}

// ScorePixel (DepthMap.cpp:567-626): MINMEAN over the views; also reports the two best views
template <bool GEOM>
__device__ __forceinline__ float score_pixel(const PMParams& P, const PatchW& pt,
	float fx, float fy, float X0x, float X0y, const Hyp& h, float priorF, float priorD, uint32_t& best)
{
	float s0 = CUDART_INF_F, s1 = CUDART_INF_F;
	int i0 = 255, i1 = 255;
	#pragma unroll 1
	for (int v = 0; v < P.nViews; ++v) {
		const float s = score_view<GEOM>(P, P.views[v], pt, fx, fy, X0x, X0y, h, priorF, priorD);
		if (s < s0) { s1 = s0; i1 = i0; s0 = s; i0 = v; }
		else if (s < s1) { s1 = s; i1 = v; }
	}
	if (P.nViews <= 1 || s1 >= P.thRobust) {
		best = 0xFFFFFF00u | (uint32_t)i0;
		return s0;
	}
	best = 0xFFFF0000u | ((uint32_t)i1<<8) | (uint32_t)i0;
	return (s0+s1)*0.5f;
}

// offset of close neighbour k (sweep direction dir 0: left, up, right, down;  dir 1: right, down, left, up)
__device__ __forceinline__ void close_offset(int dir, int k, int& ox, int& oy) {
	const int kk = dir ? (k^2) : k;
	ox = (kk == 0) ? -1 : (kk == 2) ? 1 : 0;
	oy = (kk == 1) ? -1 : (kk == 3) ? 1 : 0;
}

// build a hypothesis: homography terms + smoothness factor over the close neighbours
// (InitPlane DepthMap.cpp:963-971 and the smoothness loop DepthMap.cpp:522-534).
// closeMask bit k: close neighbour k (close_offset) holds a valid plane.  The close neighbours are of the other
// colour, so their planes do not change during a half-sweep: they are re-read here (L1 hits) and their rays
// recomputed instead of being kept in registers across the hypothesis loop.
__device__ __forceinline__ void make_hyp(const PMParams& P, int x, int y, float X0x, float X0y, float d, const float3& n,
	int dir, unsigned closeMask, Hyp& h)
{
	h.d = d; h.n = n;
	h.invd = 1.f/d;
	const float nX0 = n.x*X0x + n.y*X0y + n.z;
	const float s = 1.f/(nX0*d);
	h.ms = make_float3(n.x*P.ifx*s, (n.x*P.sk + n.y*P.ify)*s, (n.x*P.ox + n.y*P.oy + n.z)*s);
	float smooth = 1.f;
	if (closeMask != 0u) {
		// keep the compiler from hoisting the neighbour addresses and rays out of the hypothesis loop
		asm volatile("" : "+r"(x), "+r"(y));
		const float planeD = -d*nX0;
		const float nn = dot3(n, n);
		#pragma unroll
		for (int k = 0; k < 4; ++k) {
			if (closeMask & (1u<<k)) {
				int ox, oy;
				close_offset(dir, k, ox, oy);
				const float4 np = P.plane[(size_t)(y+oy)*P.W + (x+ox)];
				const float3 cn = make_float3(np.x, np.y, np.z);
				const float2 r = pixel_ray(P, float(x+ox), float(y+oy));
				const float dist = (n.x*r.x + n.y*r.y + n.z)*np.w + planeD;
				const float rd = dist/d;
				const float factorDepth = expf(rd*rd*P.smoothSigmaDepth);
				float ca = dot3(n, cn)/sqrtf(nn*dot3(cn, cn));
				ca = fminf(fmaxf(ca, -1.f), 1.f);
				const float ang = acosf(ca);
				const float factorNormal = expf(ang*ang*P.smoothSigmaNormal);
				smooth *= (1.f-P.smoothBonusDepth*factorDepth)*(1.f-P.smoothBonusNormal*factorNormal);
			}
		}
	}
	h.smooth = smooth;
}

__device__ __forceinline__ float3 dir2normal(float a, float b) {
	float sa, ca, sb, cb;
	sincosf(a, &sa, &ca);
	sincosf(b, &sb, &cb);
	return make_float3(ca*sb, sa*sb, cb);
}
// RandomNormal (DepthMap.h:439-444)
__device__ __forceinline__ float3 random_normal(float u1, float u2, float X0x, float X0y) {
	const float kPI = 3.14159265358979323846f;
	const float a = 0.f + (kPI-0.f)*u1;
	const float b = 0.5f*kPI + (kPI-0.5f*kPI)*u2;
	float3 n = dir2normal(a, b);
	if (n.x*X0x + n.y*X0y + n.z > 0.f)
		n = make_float3(-n.x, -n.y, -n.z);
	return n;
}
// CorrectNormal (DepthMap.h:447-453): rotate n to at most ~90 deg from the viewing ray
__device__ __forceinline__ void correct_normal(float3& n, float X0x, float X0y) {
	const float cosAngLen = n.x*X0x + n.y*X0y + n.z;
	if (cosAngLen >= 0.f) {
		const float kPI = 3.14159265358979323846f;
		const float vlen = sqrtf(X0x*X0x + X0y*X0y + 1.f);
		const float ang = fminf((acosf(cosAngLen/vlen) - 0.5f*kPI)*1.01f, -0.001f);
		float3 w = make_float3(n.y*1.f - n.z*X0y, n.z*X0x - n.x*1.f, n.x*X0y - n.y*X0x); // n x viewDir
		const float inv = 1.f/sqrtf(dot3(w, w));
		w.x *= inv; w.y *= inv; w.z *= inv;
		float s, c;
		sincosf(ang, &s, &c);
		// Rodrigues: R v = v + s (w x v) + (1-c) w x (w x v)
		const float3 wv = make_float3(w.y*n.z - w.z*n.y, w.z*n.x - w.x*n.z, w.x*n.y - w.y*n.x);
		const float3 wwv = make_float3(w.y*wv.z - w.z*wv.y, w.z*wv.x - w.x*wv.z, w.x*wv.y - w.y*wv.x);
		const float c1 = 1.f-c;
		n = make_float3(n.x + s*wv.x + c1*wwv.x, n.y + s*wv.y + c1*wwv.y, n.z + s*wv.z + c1*wwv.z);
	}
}

// The cost field doubles as the "changed" memory of the red-black schedule: the sign bit of a pixel's stored
// cost is set when its last update left its plane unchanged (costs are >= 0, so the bit is free; -0.f counts).
__device__ __forceinline__ bool cost_unchanged(float c) { return (__float_as_uint(c)>>31) != 0u; }

// ------------------------------------------------------------------------------------
// pass A: score the initial estimate of every pixel (random where invalid)
template <bool GEOM>
__global__ void __launch_bounds__(BLOCK_X*BLOCK_Y, 3)
pm_score_kernel(const __grid_constant__ PMParams P)
{
	extern __shared__ float2 smemW[];
	const int x = blockIdx.x*BLOCK_X + threadIdx.x;
	const int y = blockIdx.y*BLOCK_Y + threadIdx.y;
	if (x >= P.W || y >= P.H)
		return;
	const size_t idx = (size_t)y*P.W + x;
	PatchW pt;
	pt.s = smemW + threadIdx.y*BLOCK_X + threadIdx.x;
	float priorD = 0.f, priorF = 0.f;
	// a rejected or masked pixel: depth / normal zero, never scored; internally its cost is 2
	bool ok = pixel_active(P, x, y);
	if (ok) {
		fill_patch<false>(ImageTexels{P.img0, P.pitch0, x, y}, pt);
		ok = pixel_prior(P, idx, pt.normSq0, priorD, priorF);
	}
	if (!ok) {
		P.plane[idx] = make_float4(0.f, 0.f, 0.f, 0.f);
		P.cost[idx] = 2.f;
		if (P.bestViews) P.bestViews[idx] = 0xFFFFFFFFu;
		return;
	}
	const float fx = float(x), fy = float(y);
	const float2 X0 = pixel_ray(P, fx, fy);
	const float X0x = X0.x, X0y = X0.y;
	float4 pl = P.plane[idx];
	float3 n = make_float3(pl.x, pl.y, pl.z);
	float d = pl.w;
	const uint4 r = philox4x32_10(make_uint4((uint32_t)idx, 0u, 0u, 0u), make_uint2(P.seed, 0xB200C0DEu));
	if (!(P.dMin <= d && d < P.dMax)) {
		const float s = P.dMinSqr + (P.dMaxSqr-P.dMinSqr)*u32_to_unit(r.x);
		d = s*s;
		n = random_normal(u32_to_unit(r.y), u32_to_unit(r.z), X0x, X0y);
	} else if (n.x*X0x + n.y*X0y + n.z >= 0.f) {
		n = random_normal(u32_to_unit(r.x), u32_to_unit(r.y), X0x, X0y);
	}
	Hyp h;
	make_hyp(P, x, y, X0x, X0y, d, n, 0, 0u, h);
	uint32_t best;
	const float c = score_pixel<GEOM>(P, pt, fx, fy, X0x, X0y, h, priorF, priorD, best);
	P.plane[idx] = make_float4(n.x, n.y, n.z, d);
	P.cost[idx] = c;
	if (P.bestViews) P.bestViews[idx] = best;
}

// ------------------------------------------------------------------------------------
// pass B: one red-black half-sweep (ProcessPixel, DepthMap.cpp:630-852, on the engine schedule):
//   1. gather the four 4-neighbours (smoothing set "close", DepthMap.cpp:641-766) and, per direction, the
//      propagation candidate: the pixel of the other colour at distance 1, 3, .. 2*farRings+1 with the lowest
//      stored cost (the nearest on ties) — the red-black stand-in for the transport along the scanline that
//      the reference's sequential sweep performs within one iteration;
//   2. test the candidates' planes (InterpolatePixel + CorrectNormal), skipping a direction whose candidates
//      all kept their plane in their last update (they lost against this pixel one sweep ago) — P.skipUnchanged;
//   3. the refinement state machine (DepthMap.cpp:800-852).
// Every lane keeps its own to-do list of directions; the warp scores the lists of its 32 pixels as one packed list, so it
// runs ceil(sum of list lengths / 32) test steps instead of max-over-lanes(list length).
// 3 CTAs per SM: 80 registers without spills (a 64-register, 4-CTA build spills and measured slower, DESIGN.md §5.1)
template <bool GEOM>
__global__ void __launch_bounds__(BLOCK_X*BLOCK_Y, 3)
pm_sweep_kernel(const __grid_constant__ PMParams P, const __grid_constant__ CUtensorMap tmapRef)
{
	extern __shared__ __align__(128) unsigned char smemRaw[];
	// [ patch weights | {sumW, normSq0} per thread | mbarrier ]; the reference tile occupies the start of the weights
	// until the weights are written (fill_patch): 4.6 KB less shared memory per CTA, which the SM's L1/shared array gives
	// to L1.  A lane scores hypotheses of other pixels of its row (propagation candidates), so a pixel's patch statistics
	// live in shared memory beside its weights.
	float2* smemW = (float2*)smemRaw;
	float* tile = (float*)smemRaw;
	float2* smemStats = (float2*)(smemRaw + PM_TEXELS*NTHREADS*sizeof(float2));
	uint64_t* bar = (uint64_t*)(smemStats + NTHREADS);
	const int tid = threadIdx.y*BLOCK_X + threadIdx.x;
	if (tid == 0) {
		mbar_init(bar, 1);
		asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); // make the init visible to the async proxy
	}
	__syncthreads();
	if (tid == 0) {
		mbar_expect_tx(bar, TILE_BYTES);
		tma_load_2d(tile, &tmapRef, (int)blockIdx.x*(2*BLOCK_X)-PM_HALF, (int)blockIdx.y*BLOCK_Y-PM_HALF, bar);
	}
	mbar_wait(bar, 0);
	const int y = blockIdx.y*BLOCK_Y + threadIdx.y;
	const int lane = threadIdx.x;  // BLOCK_X == 32: a warp is one row of the CTA
	const int x0 = blockIdx.x*(2*BLOCK_X) + ((y+P.colour)&1);  // x of lane l: x0 + 2*l
	const int x = x0 + 2*lane;
	const bool active = pixel_active(P, x, y);
	const int W = P.W, H = P.H;
	const size_t idx = (size_t)y*W + x;
	{
		PatchW pt;
		pt.s = smemW + tid;
		fill_patch<true>(TileTexels{tile, 2*lane + ((y+P.colour)&1) + PM_HALF, (int)threadIdx.y + PM_HALF}, pt);
		smemStats[tid] = make_float2(pt.sumW, pt.normSq0);
	}
	__syncwarp(); // the other lanes of the row read this pixel's weights and statistics
	// A lane whose pixel is not estimated stays in the loop below without hypotheses of its own, so that the warp's
	// shuffles always have all 32 lanes and the packed list maps onto every lane
	float priorD, priorF;
	const bool live = active && pixel_prior(P, idx, smemStats[tid].y, priorD, priorF);
	const float fy = float(y);

	// neighbours: causal pair of the sweep direction first (DepthMap.cpp:641-766)
	const int dir = P.sweep & 1;
	const int nProp = P.propagation, farRings = P.farRings;
	unsigned closeMask = 0; // bit k: close neighbour k holds a valid plane (make_hyp)
	unsigned todo = 0;    // bit k: direction k has a candidate to test
	unsigned farSel = 0;  // 2 bits per direction: ring of the candidate (distance 2*ring+1)
	#pragma unroll
	for (int k = 0; k < 4 && live; ++k) {
		const int kk = dir ? (k^2) : k;
		int ox, oy;
		close_offset(dir, k, ox, oy);
		const bool ok = (kk == 0) ? (x > PM_HALF) : (kk == 1) ? (y > PM_HALF) : (kk == 2) ? (x < W-PM_HALF) : (y < H-PM_HALF);
		if (ok) {
			const size_t nidx = (size_t)(y+oy)*W + (x+ox);
			const float4 np = P.plane[nidx];
			const float nc = P.cost[nidx];
			bool changed = !cost_unchanged(nc);
			float bestC = 3.f;
			if (np.w > 0.f) {
				closeMask |= 1u<<k;
				bestC = fabsf(nc);
			}
			if (k < nProp) {
				unsigned ring = 0;
				for (int f = 1; f <= farRings; ++f) {
					const int qx = x+ox*(2*f+1), qy = y+oy*(2*f+1);
					if (qx < PM_HALF || qy < PM_HALF || qx >= W-PM_HALF || qy >= H-PM_HALF)
						break;
					const float fc = P.cost[(size_t)qy*W + qx];
					changed = changed || !cost_unchanged(fc);
					if (fabsf(fc) < bestC) { bestC = fabsf(fc); ring = (unsigned)f; }
				}
				if (bestC < P.keep && (changed || !P.skipUnchanged)) {
					todo |= 1u<<k;
					farSel |= ring<<(2*k);
				}
			}
		}
	}
	const unsigned nOwn = __popc(todo);               // this pixel's propagation candidates
	const unsigned info = todo | farSel<<4 | closeMask<<12;
	float depth = 0.f, conf = 0.f;
	float3 normal = make_float3(0.f, 0.f, 0.f);
	uint32_t bestViews = 0xFFFFFFFFu;
	if (live) {
		const float4 pl = P.plane[idx];
		depth = pl.w; normal = make_float3(pl.x, pl.y, pl.z);
		conf = fabsf(P.cost[idx]);
		if (P.bestViews) bestViews = P.bestViews[idx];
	}

	// The warp's propagation candidates as one list: lane after lane, each lane's in __ffs order.  The bits of the
	// candidate counts (0-4) as three ballots give every lane the prefix sum of any lane: listed(m) = candidates of
	// the lanes in mask m.  Packed step s scores list entries 32s .. 32s+31, entry 32s+l on lane l, for the pixel that
	// owns it; so the candidate phase takes ceil(total/32) steps instead of the largest count of a lane.
	const unsigned c0 = __ballot_sync(0xFFFFFFFFu, nOwn & 1u), c1 = __ballot_sync(0xFFFFFFFFu, nOwn & 2u), c2 = __ballot_sync(0xFFFFFFFFu, nOwn & 4u);
	const auto listed = [&](unsigned m) { return __popc(c0 & m) + 2*__popc(c1 & m) + 4*__popc(c2 & m); };
	const int nList = listed(0xFFFFFFFFu);

	// ---- propagation (DepthMap.cpp:775-799), then the refinement state machine (DepthMap.cpp:800-852) ----
	// One loop and one copy of the scoring code for both: the packed candidate steps, then every lane runs its own
	// refinement tries.  A candidate's plane comes from a pixel of the other colour and its hypothesis depends only on
	// the owner pixel, so any lane can score it; the owner then takes the scores in its candidate order (conf > nconf),
	// as the reference does.  Every try has its own Philox slot (restart try k: slot k, refinement try k: slot nR+k).
	// evalCap > 0 (engine schedule, b200mvs_params.nEvalCap): a pixel that tests c candidates spends at most
	// max(1, evalCap - c) tries of each kind — pixels whose four directions all changed give up their finest perturbation.
	const int nR = P.nRandomIters;
	// (the pixel's own count, listed(1u<<lane), and nRl are recomputed where they are used: 80 registers without spills)
	const auto nRl = [&]() { return P.evalCap > 0 ? min(nR, max(P.evalCap-listed(1u<<lane), 1)) : nR; };
	const uint2 key = make_uint2(P.seed, 0xB200C0DEu);
	const uint32_t pix = (uint32_t)idx; // Philox counter
	const uint32_t phase = 1u + (uint32_t)P.sweep;
	int mode = live ? 0 : 3;    // 0 undecided, 1 restart (fully random), 2 refine, 3 done
	bool entered = !live;       // the state machine has taken its first decision
	bool useClose = true;
	unsigned idxScale = 0;
	float depthRange = 0.f, pa = 0.f, pb = 0.f;
	int nTry = 0; // tries spent in the current mode (restart or refine)
	#pragma unroll 1
	for (int step = 0;; ++step) {
		const bool packed = 32*step < nList; // warp-uniform
		bool have = false, isRefine = false, alive = packed, uc = true;
		float hd = 0.f, na = 0.f, nb = 0.f; float3 hn = make_float3(0.f, 0.f, 1.f);
		int owner = lane, k = 0;  // the hypothesis is for the pixel of lane `owner`
		if (packed) {
			const int j = 32*step + lane;
			have = j < nList;
			if (have) {
				// owner: the lane whose candidates end after entry j (listed() of lanes 0..m grows with m)
				owner = 0;
				#pragma unroll
				for (int b = 16; b > 0; b >>= 1)
					if (listed((2u<<(owner+b-1))-1u) <= j) owner += b;
				k = j - listed((1u<<owner)-1u); // the owner's k-th candidate
			}
		}
		const unsigned oinfo = __shfl_sync(0xFFFFFFFFu, info, owner);
		const int sx = x0 + 2*owner;
		const float sfx = float(sx);
		const float2 X0 = pixel_ray(P, sfx, fy);
		const float X0x = X0.x, X0y = X0.y;
		if (packed) {
			if (have) {
				unsigned t = oinfo & 15u;
				for (int i = 0; i < k; ++i) t &= t-1u;
				const int d4 = __ffs((int)t)-1;
				const int kk = dir ? (d4^2) : d4;
				const int dist = 2*(int)((oinfo>>(4+2*d4))&3u)+1;
				const int qx = sx + ((kk == 0) ? -dist : (kk == 2) ? dist : 0);
				const int qy = y + ((kk == 1) ? -dist : (kk == 3) ? dist : 0);
				const float4 qp = P.plane[(size_t)qy*W + qx];
				// InterpolatePixel (DepthMap.cpp:915-959): the candidate's plane intersected with this pixel's ray,
				// restricted to the row / column; the reference's ray coordinates carry no skew term
				const bool vertical = (kk & 1) != 0;
				const float ncomp = vertical ? qp.y : qp.x;
				const float nx1 = vertical ? X0y : fmaf(sfx, P.ifx, P.ox0);
				const float x1 = vertical ? fmaf(float(qy), P.ify, P.oy) : fmaf(float(qx), P.ifx, P.ox0);
				const float denom = qp.z + nx1*ncomp;
				hd = qp.w;
				if (!(fabsf(denom) < 0.0001f)) {
					const float dn = qp.w*(qp.z + x1*ncomp)/denom;
					if (P.dMin <= dn && dn < P.dMax)
						hd = dn;
				}
				hn = make_float3(qp.x, qp.y, qp.z);
				correct_normal(hn, X0x, X0y);
			}
		} else {
			if (!entered || (mode == 1 && conf < P.thConfRand)) {
				// RefineIters: choose the perturbation scale from the current score
				entered = true;
				bool toRefine = true;
				if (conf <= P.thConfSmall) idxScale = 2;
				else if (conf <= P.thConfBig) idxScale = 1;
				else if (conf >= P.thConfRand && mode == 0) { mode = 1; useClose = false; toRefine = false; }
				if (toRefine) {
					mode = 2;
					nTry = 0;
					depthRange = depth*P.depthRatio;
					pa = atan2f(normal.y, normal.x);
					pb = acosf(normal.z);
				}
			}
			if (mode == 1 && nTry >= nRl()) mode = 3; // all random tries failed: no refinement this sweep
			alive = (mode == 1) || (mode == 2 && nTry < nRl());
			uc = useClose;
			if (mode == 1) {
				// completely random plane (DepthMap.cpp:810-825)
				const uint4 r = philox4x32_10(make_uint4(pix, phase, (uint32_t)nTry, 0u), key);
				++nTry;
				const float s = P.dMinSqr + (P.dMaxSqr-P.dMinSqr)*u32_to_unit(r.x);
				hd = s*s;
				hn = random_normal(u32_to_unit(r.y), u32_to_unit(r.z), X0x, X0y);
				have = true;
			} else if (mode == 2 && nTry < nRl()) {
				// perturb around the current estimate (DepthMap.cpp:832-851)
				const uint4 r = philox4x32_10(make_uint4(pix, phase, (uint32_t)(nR+nTry), 0u), key);
				++nTry;
				const float scaleRange = pow2neg(idxScale);
				hd = depth + depthRange*scaleRange*(2.f*u32_to_unit(r.x)-1.f);
				if (P.dMin <= hd && hd < P.dMax) {
					na = pa + P.angle1Range*scaleRange*(2.f*u32_to_unit(r.y)-1.f);
					nb = pb + P.angle2Range*scaleRange*(2.f*u32_to_unit(r.z)-1.f);
					hn = dir2normal(na, nb);
					have = hn.x*X0x + hn.y*X0y + hn.z < 0.f;
					isRefine = true;
				}
			}
		}
		if (!__any_sync(0xFFFFFFFFu, alive))
			break;
		if (!__any_sync(0xFFFFFFFFu, have))
			continue;
		float nconf = 0.f;
		uint32_t bv = 0u;
		if (have) {
			const int otid = threadIdx.y*BLOCK_X + owner;
			PatchW pt;
			pt.s = smemW + otid;
			const float2 st = smemStats[otid];
			pt.sumW = st.x; pt.normSq0 = st.y;
			float oPriorD, oPriorF;
			pixel_prior(P, (size_t)y*W + sx, st.y, oPriorD, oPriorF);
			Hyp h;
			make_hyp(P, sx, y, X0x, X0y, hd, hn, dir, uc ? (oinfo>>12) : 0u, h);
			nconf = score_pixel<GEOM>(P, pt, sfx, fy, X0x, X0y, h, oPriorF, oPriorD, bv);
		}
		if (packed) {
			// the owner takes the scores of its candidates of this step (at most four, contiguous lanes) in order
			#pragma unroll
			for (int i = 0; i < 4; ++i) {
				const int src = listed((1u<<lane)-1u) + i - 32*step; // list position of this pixel's candidate i, in this step
				const bool mine = i < listed(1u<<lane) && src >= 0 && src < 32;
				const int l = mine ? src : lane;
				const float c = __shfl_sync(0xFFFFFFFFu, nconf, l);
				const uint32_t b = __shfl_sync(0xFFFFFFFFu, bv, l);
				const float d = __shfl_sync(0xFFFFFFFFu, hd, l);
				const float n0 = __shfl_sync(0xFFFFFFFFu, hn.x, l), n1 = __shfl_sync(0xFFFFFFFFu, hn.y, l), n2 = __shfl_sync(0xFFFFFFFFu, hn.z, l);
				if (mine && conf > c) {
					conf = c; depth = d; normal = make_float3(n0, n1, n2); bestViews = b;
				}
			}
		} else if (have && conf > nconf) {
			conf = nconf; depth = hd; normal = hn; bestViews = bv;
			if (isRefine) {
				pa = na; pb = nb;
				++idxScale;
			}
		}
	}
	if (!live)
		return;
	const float4 pl = P.plane[idx]; // re-read (only this thread writes it) rather than kept live across the loop
	const bool same = depth == pl.w && normal.x == pl.x && normal.y == pl.y && normal.z == pl.z;
	P.plane[idx] = make_float4(normal.x, normal.y, normal.z, depth);
	P.cost[idx] = (same && P.skipUnchanged) ? -conf : conf;
	if (P.bestViews) P.bestViews[idx] = bestViews;
}

// pass C: threshold and convert cost to confidence (EndDepthMapTmp).  viewsMap: the (at most two) views of the
// MINMEAN score in ascending order, 255 padding — the order PatchMatchCUDA.cpp:374-391 emits its view ids in
__global__ void pm_finalize_kernel(int n, float keep, const float4* __restrict__ plane, const float* __restrict__ cost,
	const uint32_t* __restrict__ bestViews, float* __restrict__ depth, float* __restrict__ normal, float* __restrict__ conf,
	uint32_t* __restrict__ viewsMap)
{
	const int i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 p = plane[i];
	const float c = fabsf(cost[i]);
	float d = p.w, cf; float3 nn = make_float3(p.x, p.y, p.z);
	uint32_t bv = bestViews ? bestViews[i] : 0xFFFFFFFFu;
	if (d <= 0.f || c >= keep) {
		d = 0.f; cf = 0.f; nn = make_float3(0.f, 0.f, 0.f); bv = 0xFFFFFFFFu;
	} else {
		cf = c >= 1.f ? 0.f : 1.f-c;
		const uint32_t a = bv & 0xFFu, b = (bv>>8) & 0xFFu;
		bv = 0xFFFF0000u | (max(a, b)<<8) | min(a, b);
	}
	depth[i] = d; conf[i] = cf;
	normal[3*(size_t)i] = nn.x; normal[3*(size_t)i+1] = nn.y; normal[3*(size_t)i+2] = nn.z;
	if (viewsMap) viewsMap[i] = bv;
}

__global__ void pm_pack_kernel(int n, const float* __restrict__ depth, const float* __restrict__ normal, float4* __restrict__ plane) {
	const int i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	plane[i] = make_float4(normal[3*(size_t)i], normal[3*(size_t)i+1], normal[3*(size_t)i+2], depth[i]);
}
__global__ void pm_unpack_kernel(int n, const float4* __restrict__ plane, float* __restrict__ depth, float* __restrict__ normal) {
	const int i = blockIdx.x*blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 p = plane[i];
	depth[i] = p.w;
	normal[3*(size_t)i] = p.x; normal[3*(size_t)i+1] = p.y; normal[3*(size_t)i+2] = p.z;
}

// ---- host launchers ---------------------------------------------------------------------
constexpr size_t W_BYTES = (size_t)PM_TEXELS*NTHREADS*sizeof(float2);
// weights, per-thread patch statistics, mbarrier; the reference tile lives inside the weights (pm_sweep_kernel).  3 CTAs
// (53.3 KB + 1 KB reserved each) fit the SM's 164 KB shared-memory carveout, which leaves 92 KB of L1
constexpr size_t SWEEP_SMEM = W_BYTES + NTHREADS*sizeof(float2) + 16;
static_assert(TILE_BYTES <= W_BYTES, "the reference tile must fit inside the patch weights");

template <bool GEOM>
cudaError_t configure_one() {
	cudaError_t e = cudaFuncSetAttribute(pm_sweep_kernel<GEOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SWEEP_SMEM);
	if (e != cudaSuccess) return e;
	return cudaFuncSetAttribute(pm_score_kernel<GEOM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)W_BYTES);
}

} // namespace

// Opt the kernels of the current device into their dynamic shared memory sizes.  Called by b200mvs_create for its
// device (function attributes are per device; the call is idempotent and safe from several host threads).
cudaError_t pm_configure_device() {
	cudaError_t e;
	if ((e = configure_one<false>()) != cudaSuccess) return e;
	return configure_one<true>();
}
cudaError_t pm_launch_score(const PMParams& P, bool geom, cudaStream_t s) {
	dim3 block(BLOCK_X, BLOCK_Y), grid((P.W+BLOCK_X-1)/BLOCK_X, (P.H+BLOCK_Y-1)/BLOCK_Y);
	if (geom) pm_score_kernel<true><<<grid, block, W_BYTES, s>>>(P); else pm_score_kernel<false><<<grid, block, W_BYTES, s>>>(P);
	return cudaGetLastError();
}
// tmapRef: TMA descriptor of the reference image P.img0 with box {72, 16} (pm_tma_box)
cudaError_t pm_launch_sweep(const PMParams& P, const CUtensorMap& tmapRef, bool geom, cudaStream_t s) {
	dim3 block(BLOCK_X, BLOCK_Y), grid((P.W+2*BLOCK_X-1)/(2*BLOCK_X), (P.H+BLOCK_Y-1)/BLOCK_Y);
	if (geom) pm_sweep_kernel<true><<<grid, block, SWEEP_SMEM, s>>>(P, tmapRef); else pm_sweep_kernel<false><<<grid, block, SWEEP_SMEM, s>>>(P, tmapRef);
	return cudaGetLastError();
}
void pm_tma_box(int* w, int* h) { *w = TILE_W; *h = TILE_H; }
cudaError_t pm_launch_finalize(int n, float keep, const float4* plane, const float* cost, const uint32_t* bestViews,
	float* depth, float* normal, float* conf, uint32_t* viewsMap, cudaStream_t s) {
	pm_finalize_kernel<<<(n+255)/256, 256, 0, s>>>(n, keep, plane, cost, bestViews, depth, normal, conf, viewsMap);
	return cudaGetLastError();
}
cudaError_t pm_launch_pack(int n, const float* depth, const float* normal, float4* plane, cudaStream_t s) {
	pm_pack_kernel<<<(n+255)/256, 256, 0, s>>>(n, depth, normal, plane);
	return cudaGetLastError();
}
cudaError_t pm_launch_unpack(int n, const float4* plane, float* depth, float* normal, cudaStream_t s) {
	pm_unpack_kernel<<<(n+255)/256, 256, 0, s>>>(n, plane, depth, normal);
	return cudaGetLastError();
}
