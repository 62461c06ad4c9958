// sgm_cost_tc.cu — the WZNCC 7x7 cost volume of the SGM pair matcher on the Hopper tensor cores (wgmma, sm_90a).
//
// What it computes: per valid pixel x of a row and disparity d, the three weighted sums of the 49-tap window
//   sum = S_n w_x(n) f_n,  sumSq = S_n w_x(n) f_n^2,  nom = S_n tw_x(n) f_n,   f_n = right(y+i, x+d+j), n = (i,j)
// and from them the uint8 cost (SemiGlobalMatcher.cpp:875-985; the SIMT form is sgm_cost_kernel in sgm_kernels.cu).
//
// Why tensor cores fit: for a block of 128 pixels of one row the sums are a banded GEMM.  With A[x, n] = w_x(n) (M = 128 pixels,
// K = 49 taps padded to 64) and the Toeplitz matrix B[n, u] = right(y+i, u+j) (u = x + d, the right-image column), the wanted
// entries are D[x, u] for u - x in [dmin, dmin+D).  The band is cut into 64-column tiles of u; a tile serves two pixel blocks, a
// block needs (128+D)/64 tiles (band utilisation 50 % at D = 128).  Precision: the operands are split into fp16 high and low
// parts (w = wh + wl) and every sum is three f16 MMAs with fp32 accumulation (wh fh + wh fl + wl fh).  For operands of 2^-3 and
// more the split keeps 22 bits (error 2^-22 relative, and the dropped wl fl term is 2^-22 relative too); below that the low part,
// and below 2^-14 the high part, are fp16 subnormals with an absolute error of up to 2^-25 each.  Bilateral weights of saturated
// colour contrast reach exp(-17.8) ~ 1.9e-8 and keep no relative precision, but their absolute error is what enters the sums:
// tests/test_sgm_reference_gpu.py bounds it as 2^-25 per operand and product, and the kernel equals the float64 cost on every
// entry that this bound (with 2^-20 relative per product) leaves decidable.
//
// Structure (one CTA of 16 warps = 4 warpgroups per SM, persistent over the rows of the valid region):
//   all warps stage the seven image rows of the block in shared memory (left colour packed to a word, left and right gray) and
//              build A (bilateral weights of the block's 128 pixels: one warp-uniform tap quarter per warp, so tap offsets and
//              spatial weights are immediates; colour distance by VABSDIFF4 + DP4A, weight by one EX2; fp16 split; 16-byte stores
//              in the GMMA K-major no-swizzle core-matrix layout) and the two new B tiles (im2col of the staged right rows);
//   each warpgroup then owns one quarter of every tile — 64 pixels x 32 columns — and computes it with 36 wgmma.m64n32k16
//              (9 products x 4 K-steps) into 3 x 16 fp32 registers per thread; a quarter wholly outside the diagonal band is
//              skipped (warpgroup-uniform), which saves about a third of the MMAs at D = 128;
//   the same warpgroup turns its registers into costs and scatters them into a shared cost tile, which is finally written to
//              the volume with coalesced 16-byte stores.  The B tiles live in a ring of four: a block re-uses the last
//              nTiles - 2 tiles of the block before it.
// SASS: HGMMA (wgmma.mma_async), WARPGROUP.ARRIVE / WARPGROUP.DEPBAR (fence, wait).
#include "sgm_common.cuh"
#include <cuda_fp16.h>
#include <string.h>

namespace {

constexpr int BM = 128;          // pixels per block (two wgmma M = 64 halves)
constexpr int BN = 64;           // right-image columns per tile (two wgmma N = 32 halves)
constexpr int KP = 64;           // taps padded to the MMA K granularity (4 x 16)
constexpr int TC_THREADS = 512;  // 16 warps: operand builders, MMA issue and epilogue
constexpr int A_ARRAY = BM*KP*2;         // one fp16 operand array of a block: 16 KB
constexpr int B_ARRAY = BN*KP*2;         // one fp16 operand array of a tile: 8 KB
constexpr int B_SLOT = 4*B_ARRAY;        // fh, fl, qh, ql
constexpr int RING = 4;                  // B tiles kept (a block of D <= 128 needs (128+D)/64 <= 4)
constexpr int TILE_PITCH = 132;          // bytes per pixel row of the shared cost tile (bank-conflict-free byte scatter)
constexpr int SP = BM+8;                 // pitch of the staged image rows (128 columns + 6 of the window, padded)
constexpr int SMEM_A = 4*A_ARRAY;        // wh, wl, th, tl
constexpr int SMEM_B = RING*B_SLOT;
constexpr int SMEM_TILE = BM*TILE_PITCH; // the block's costs; while the operands are built: the staged image rows and partial sums
constexpr int SMEM_CONST = 4*BM*4 + BM*4;   // normSq0 partial of each tap quarter, 1/sumW per pixel
constexpr int SMEM_TOTAL = SMEM_A + SMEM_B + SMEM_TILE + SMEM_CONST;
// staging area inside the cost tile (free between the store of a block and the epilogue of the next)
constexpr int ST_LC = 0;                 // left colour rows, packed B | G<<8 | R<<16: 7 x SP u32
constexpr int ST_LG = ST_LC + 7*SP*4;    // left gray rows: 7 x SP float
constexpr int ST_RG = ST_LG + 7*SP*4;    // right gray rows of the two new tiles: 7 x SP float
constexpr int ST_PART = ST_RG + 7*SP*4;  // {sum w g, sum w} of each tap quarter: 4 x BM float2
static_assert(ST_PART + 4*BM*8 <= SMEM_TILE, "staging area exceeds the cost tile");
static_assert(SMEM_TOTAL <= 232448, "shared memory of one CTA (227 KB)");
// named barrier of all 16 warps (id 0 is __syncthreads; a named barrier may be reached from different code locations)
constexpr int BAR_WORKERS = 1;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bar_sync(int id, int n) { asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(n) : "memory"); }

// K-major, no swizzle (INTERLEAVE): a K-chunk of 8 halves (16 B) of row r sits at chunk*rows*16 + r*16; 8 consecutive rows are one
// 128-byte core matrix: stride between 8-row groups SBO = 128 B, between the two 16-byte K-chunks of one MMA LBO = rows*16 B
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes) {
	uint64_t d = 0;
	d |= (uint64_t)((saddr>>4) & 0x3FFFu);
	d |= (uint64_t)((lbo_bytes>>4) & 0x3FFFu) << 16;
	d |= (uint64_t)((128u>>4) & 0x3FFFu) << 32;
	return d;                 // base offset 0, layout type 0 = no swizzle
}
// D[64 x 32] (+)= A[64 x 16] B[16 x 32]: f16 operands from shared memory, both K-major, fp32 accumulators in registers
__device__ __forceinline__ void wgmma_m64n32k16(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
	asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
		"wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n}"
		: "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
		  "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
		: "l"(adesc), "l"(bdesc), "r"(accumulate) : "memory");
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) { return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b)<<16); }
// x = hi + lo with hi = fp16(x): two fp16 numbers carrying 22 bits of x for |x| >= 2^-3 (an absolute error <= 2^-25 below, where
// lo, and below 2^-14 hi, is subnormal)
__device__ __forceinline__ void split_h(float x, __half& hi, __half& lo) { hi = __float2half_rn(x); lo = __float2half_rn(x-__half2float(hi)); }
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

constexpr float LOG2E = 1.4426950408889634f;
constexpr float SIGMA_COLOR = -1.f/(2.f*(0.3f*255)*(0.3f*255));
constexpr float SIGMA_SPATIAL = -1.f/(2.f*(0.4f*7)*(0.4f*7));

// One tap quarter (taps 16 Q .. 16 Q + 15; Q = 3: tap 48) of the A operands of pixel `row` of the block, from the staged left
// rows.  Q is a template parameter so that the tap geometry (i, j) and the spatial weight are compile-time constants.
// Bilateral weight (SemiGlobalMatcher.cpp:889-905): exp(colour distance^2 sigmaColor + spatial distance^2 sigmaSpatial) as one
// ex2 of a fused multiply-add; the colour distance is |dB|^2 + |dG|^2 + |dR|^2 = dp4a of the packed absolute differences.
template <int Q>
__device__ __forceinline__ void build_a_quarter(unsigned char* sA, const unsigned char* sStage, float* sNorm, float* sInv, int row, bool valid) {
	constexpr int N0 = 16*Q, NN = Q == 3 ? 1 : 16;
	const uint32_t* lc = (const uint32_t*)(sStage + ST_LC);
	const float* lg = (const float*)(sStage + ST_LG);
	float2* part = (float2*)(sStage + ST_PART);
	float wv[NN], gv[NN];
	float sumW = 0.f, acc = 0.f;
	const uint32_t cc = lc[SGM_HW*SP + row+SGM_HW];
	#pragma unroll
	for (int k = 0; k < NN; ++k) {
		const int n = N0+k, i = n/7, j = n-7*i;   // compile-time after unrolling
		const uint32_t d = __vabsdiffu4(lc[i*SP + row+j], cc);
		const int dist2 = (int)__dp4a(d, d, 0u);
		const float spatial = float((j-SGM_HW)*(j-SGM_HW)+(i-SGM_HW)*(i-SGM_HW))*(SIGMA_SPATIAL*LOG2E);
		float wgt = ex2_approx(fmaf((float)dist2, SIGMA_COLOR*LOG2E, spatial));
		if (!valid) wgt = 0.f;
		const float g = lg[i*SP + row+j];
		wv[k] = wgt; gv[k] = g;
		acc = fmaf(g, wgt, acc);
		sumW += wgt;
	}
	part[Q*BM + row] = make_float2(acc, sumW);
	bar_sync(BAR_WORKERS, TC_THREADS);
	{
		const float2 p0 = part[row], p1 = part[BM+row], p2 = part[2*BM+row], p3 = part[3*BM+row];
		acc = (p0.x+p1.x)+(p2.x+p3.x); sumW = (p0.y+p1.y)+(p2.y+p3.y);
	}
	if (!valid) sumW = 1.f;
	const float tm = acc/sumW;
	float normSq0 = 0.f;
	#pragma unroll
	for (int k = 0; k < NN; ++k) {
		const float t = gv[k]-tm;
		gv[k] = wv[k]*t;          // tempWeight
		normSq0 = fmaf(gv[k], t, normSq0);
	}
	sNorm[Q*BM + row] = normSq0;
	if (Q == 0) sInv[row] = 1.f/sumW;
	#pragma unroll
	for (int c2 = 0; c2 < (Q == 3 ? 1 : 2); ++c2) {
		const int kc = 2*Q+c2;
		__half wh[8], wl[8], th[8], tl[8];
		#pragma unroll
		for (int e = 0; e < 8; ++e) {
			const int k = c2*8+e;
			if (k < NN) { split_h(wv[k], wh[e], wl[e]); split_h(gv[k], th[e], tl[e]); }
			else { wh[e] = wl[e] = th[e] = tl[e] = __float2half_rn(0.f); }
		}
		const size_t off = (size_t)kc*(BM*16) + (size_t)row*16;
		*(uint4*)(sA+0*A_ARRAY+off) = make_uint4(pack_h2(wh[0], wh[1]), pack_h2(wh[2], wh[3]), pack_h2(wh[4], wh[5]), pack_h2(wh[6], wh[7]));
		*(uint4*)(sA+1*A_ARRAY+off) = make_uint4(pack_h2(wl[0], wl[1]), pack_h2(wl[2], wl[3]), pack_h2(wl[4], wl[5]), pack_h2(wl[6], wl[7]));
		*(uint4*)(sA+2*A_ARRAY+off) = make_uint4(pack_h2(th[0], th[1]), pack_h2(th[2], th[3]), pack_h2(th[4], th[5]), pack_h2(th[6], th[7]));
		*(uint4*)(sA+3*A_ARRAY+off) = make_uint4(pack_h2(tl[0], tl[1]), pack_h2(tl[2], tl[3]), pack_h2(tl[4], tl[5]), pack_h2(tl[6], tl[7]));
	}
}
// One tap quarter of column c of a B tile (slot) from the staged right rows; cs = column of the tile's first window in the stage
template <int Q>
__device__ __forceinline__ void build_b_quarter(unsigned char* slot, const unsigned char* sStage, int cs, int c) {
	const float* rg = (const float*)(sStage + ST_RG);
	#pragma unroll
	for (int c2 = 0; c2 < (Q == 3 ? 1 : 2); ++c2) {
		const int kc = 2*Q+c2;
		__half fh[8], fl[8], qh[8], ql[8];
		#pragma unroll
		for (int e = 0; e < 8; ++e) {
			const int n = kc*8+e;
			float f = 0.f;
			if (n < SGM_NT) { const int i = n/7, j = n-7*i; f = rg[i*SP + cs+c+j]; }
			split_h(f, fh[e], fl[e]);
			split_h(f*f, qh[e], ql[e]);
		}
		const size_t off = (size_t)kc*(BN*16) + (size_t)c*16;
		*(uint4*)(slot+0*B_ARRAY+off) = make_uint4(pack_h2(fh[0], fh[1]), pack_h2(fh[2], fh[3]), pack_h2(fh[4], fh[5]), pack_h2(fh[6], fh[7]));
		*(uint4*)(slot+1*B_ARRAY+off) = make_uint4(pack_h2(fl[0], fl[1]), pack_h2(fl[2], fl[3]), pack_h2(fl[4], fl[5]), pack_h2(fl[6], fl[7]));
		*(uint4*)(slot+2*B_ARRAY+off) = make_uint4(pack_h2(qh[0], qh[1]), pack_h2(qh[2], qh[3]), pack_h2(qh[4], qh[5]), pack_h2(qh[6], qh[7]));
		*(uint4*)(slot+3*B_ARRAY+off) = make_uint4(pack_h2(ql[0], ql[1]), pack_h2(ql[2], ql[3]), pack_h2(ql[4], ql[5]), pack_h2(ql[6], ql[7]));
	}
}

// The three sums of one 64 x 32 quarter of a tile: aBase / bBase = the quarter's first row / column in the wh / fh arrays.
// {A array, B array, accumulator}: wh fh, wh fl, wl fh -> sum | wh qh, wh ql, wl qh -> sumSq | th fh, th fl, tl fh -> nom
__device__ __forceinline__ void mma_quarter(float (&acc)[3][16], uint32_t aBase, uint32_t bBase) {
	constexpr int prod[9][3] = {{0, 0, 0}, {0, 1, 0}, {1, 0, 0}, {0, 2, 1}, {0, 3, 1}, {1, 2, 1}, {2, 0, 2}, {2, 1, 2}, {3, 0, 2}};
	asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
	#pragma unroll
	for (int p = 0; p < 9; ++p) {
		#pragma unroll
		for (int kk = 0; kk < KP/16; ++kk) {
			const uint64_t ad = gmma_desc(aBase + prod[p][0]*A_ARRAY + kk*2*(BM*16), BM*16);
			const uint64_t bd = gmma_desc(bBase + prod[p][1]*B_ARRAY + kk*2*(BN*16), BN*16);
			wgmma_m64n32k16(acc[prod[p][2]], ad, bd, (p % 3 == 0 && kk == 0) ? 0u : 1u);
		}
	}
	asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
	asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
}

// Dense volumes only (every pixel valid with one range, idx = pixel index x numAll).  One launch computes the disparities
// [dmin, dmin+num), num in {64, 128}, and stores them at offset dOff of every pixel's numAll-wide slice: wider ranges (192, 256)
// are covered by two launches.
__global__ void __launch_bounds__(TC_THREADS, 1)
sgm_cost_tc_kernel(const __grid_constant__ SGMParams P, int dmin, int num, int numAll, int dOff)
{
	extern __shared__ __align__(1024) unsigned char smem[];
	unsigned char* sA = smem;
	unsigned char* sB = smem + SMEM_A;
	unsigned char* sTile = sB + SMEM_B;
	float* sNorm = (float*)(sTile + SMEM_TILE);           // 4 x BM: normSq0 of each tap quarter
	float* sInv = sNorm + 4*BM;                           // 1/sumW
	const int tid = threadIdx.x, warp = tid>>5, lane = tid&31;
	const int w = P.w, vw = P.vw, vh = P.vh;
	// the K padding (taps 49..63) of every operand array is zero and stays zero: only chunks 0..6 are rewritten (chunk 6 holds
	// taps 48..55, its upper seven halves are written as zeros by the builders)
	for (int i = tid; i < (SMEM_A+SMEM_B)/16; i += TC_THREADS) ((uint4*)smem)[i] = make_uint4(0u, 0u, 0u, 0u);
	__syncthreads();
	const int nTiles = (BM+num)/BN;             // u tiles a block needs: 3 (D = 64) or 4 (D = 128)
	const int nBlocks = (vw+BM-1)/BM;
	const int wq = warp&3;                       // tap quarter of this warp (operand builders)
	// the quarter of every tile this warpgroup multiplies: pixels r0 .. r0+63, columns c0 .. c0+31; the thread's two pixel rows
	// and columns of the accumulator fragment (wgmma D layout: warp w of the group holds rows 16 w .. 16 w + 15)
	const int r0 = 64*((warp>>2)&1), c0 = 32*(warp>>3);
	const int rowA = r0 + 16*(warp&3) + (lane>>2), rowB = rowA+8;
	const int colF = c0 + 2*(lane&3);
	const uint32_t aQuarter = smem_u32(sA) + (uint32_t)r0*16u;
	float acc[3][16];
	#pragma unroll
	for (int s = 0; s < 3; ++s)
		#pragma unroll
		for (int e = 0; e < 16; ++e) acc[s][e] = 0.f;
	// The staged pixels of a block's first tile pair are loaded into registers while the block before it is in its epilogue:
	// thread t owns elements t and t + 512 of the 7 x 134 window (left colour packed to a word, left gray, right gray).
	struct Pre { uint32_t c[2]; float lg[2], rg[2]; } pre;
	auto prefetch = [&](int rr, int bb) {
		const int xx0 = BM*bb, tt0 = bb == 0 ? 0 : 2*bb+nTiles-2;
		#pragma unroll
		for (int k = 0; k < 2; ++k) {
			const int i = tid + k*TC_THREADS;
			pre.c[k] = 0u; pre.lg[k] = 0.f; pre.rg[k] = 0.f;
			if (i < 7*(BM+6)) {
				const int ry = i/(BM+6), cx = i-ry*(BM+6);
				const int col = min(xx0+cx, w-1);
				const uchar3 c3 = P.lbgr[(size_t)(rr+ry)*w + col];
				pre.c[k] = (uint32_t)c3.x | ((uint32_t)c3.y<<8) | ((uint32_t)c3.z<<16);
				pre.lg[k] = __ldg(P.lgray + (size_t)(rr+ry)*w + col);
				const int rc = min(max(BN*tt0 + cx + dmin, 0), w-1);
				pre.rg[k] = __ldg(P.rgray + (size_t)(rr+ry)*w + rc);
			}
		}
	};
	if ((int)blockIdx.x < vh) prefetch((int)blockIdx.x, 0);
	#pragma unroll 1
	for (int r = blockIdx.x; r < vh; r += gridDim.x) {
		#pragma unroll 1
		for (int b = 0; b < nBlocks; ++b) {
			const int x0 = BM*b;
			// B tiles not yet in the ring: the last two of the block (all of them for the first block of a row), two at a time
			for (int t0 = (b == 0 ? 0 : 2*b+nTiles-2); t0 < 2*b+nTiles; t0 += 2) {
				if (t0 != (b == 0 ? 0 : 2*b+nTiles-2)) bar_sync(BAR_WORKERS, TC_THREADS);   // the stage is read by the previous pair
				// stage the image rows r .. r+6: left colour / gray columns x0 .. x0+133 (first pair only), right gray columns of the pair.
				// The first pair of a block comes out of registers: its global loads were issued a block earlier (see below).
				const bool first = t0 == (b == 0 ? 0 : 2*b+nTiles-2);
				if (first) {
					#pragma unroll
					for (int k = 0; k < 2; ++k) {
						const int i = tid + k*TC_THREADS;
						if (i < 7*(BM+6)) {
							const int ry = i/(BM+6), cx = i-ry*(BM+6);
							((uint32_t*)(sTile+ST_LC))[ry*SP+cx] = pre.c[k];
							((float*)(sTile+ST_LG))[ry*SP+cx] = pre.lg[k];
							((float*)(sTile+ST_RG))[ry*SP+cx] = pre.rg[k];
						}
					}
				} else {
					for (int i = tid; i < 7*(BM+6); i += TC_THREADS) {
						const int ry = i/(BM+6), cx = i-ry*(BM+6);
						const int rc = min(max(BN*t0 + cx + dmin, 0), w-1);
						((float*)(sTile+ST_RG))[ry*SP+cx] = __ldg(P.rgray + (size_t)(r+ry)*w + rc);
					}
				}
				bar_sync(BAR_WORKERS, TC_THREADS);
				if (first) {
					const int row = (warp>>2)*32 + lane;
					const bool valid = x0+row < vw;
					switch (wq) {
					case 0: build_a_quarter<0>(sA, sTile, sNorm, sInv, row, valid); break;
					case 1: build_a_quarter<1>(sA, sTile, sNorm, sInv, row, valid); break;
					case 2: build_a_quarter<2>(sA, sTile, sNorm, sInv, row, valid); break;
					default: build_a_quarter<3>(sA, sTile, sNorm, sInv, row, valid); break;
					}
				}
				{
					const int tsel = warp>>3, q = (warp>>1)&3, c = (warp&1)*32 + lane;
					if (t0+tsel < 2*b+nTiles) {
						unsigned char* slot = sB + (size_t)((t0+tsel)&(RING-1))*B_SLOT;
						switch (q) {
						case 0: build_b_quarter<0>(slot, sTile, BN*tsel, c); break;
						case 1: build_b_quarter<1>(slot, sTile, BN*tsel, c); break;
						case 2: build_b_quarter<2>(slot, sTile, BN*tsel, c); break;
						default: build_b_quarter<3>(slot, sTile, BN*tsel, c); break;
						}
					}
				}
			}
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
			bar_sync(BAR_WORKERS, TC_THREADS);     // operands complete; every warp is done with the stage (the cost tile is written next)
			// the next block's window: requested now, consumed after this block's epilogue
			if (b+1 < nBlocks) prefetch(r, b+1);
			else if (r+(int)gridDim.x < vh) prefetch(r+(int)gridDim.x, 0);
			// per pixel row of the fragment: normSq0, 1/sumW and the disparities whose right window lies inside the image
			// (0 <= col + d + dmin, col + d + dmin + 6 < w, col = valid-region column of the pixel)
			float normSq0[2], invW[2];
			int dlo[2], dhi[2];
			#pragma unroll
			for (int h = 0; h < 2; ++h) {
				const int row = h ? rowB : rowA, col = x0+row;
				normSq0[h] = (sNorm[row]+sNorm[BM+row])+(sNorm[2*BM+row]+sNorm[3*BM+row]);
				invW[h] = sInv[row];
				dlo[h] = max(0, -(col+dmin)); dhi[h] = min(num, w-2*SGM_HW-col-dmin);
			}
			// sums -> costs, tile by tile, into the shared cost tile
			#pragma unroll 1
			for (int k = 0; k < nTiles; ++k) {
				const int kq = BN*k;                             // disparity index of (row 0, column 0) of this tile
				// the band 0 <= d < num covers about half of a tile: a quarter wholly outside it is skipped (warpgroup-uniform)
				if (kq+c0+31-r0 < 0 || kq+c0-(r0+63) >= num)
					continue;
				const uint32_t bQuarter = smem_u32(sB + (size_t)((2*b+k)&(RING-1))*B_SLOT) + (uint32_t)c0*16u;
				mma_quarter(acc, aQuarter, bQuarter);
				#pragma unroll
				for (int e = 0; e < 16; ++e) {
					const int h = (e>>1)&1;
					const int row = h ? rowB : rowA;
					const int d = kq + colF + 8*(e>>2) + (e&1) - row;   // disparity index of (pixel, column)
					if (d >= 0 && d < num) {
						const float sum = acc[0][e], sumSq = acc[1][e], nom = acc[2][e];
						const float normSq1 = fmaf(-sum*invW[h], sum, sumSq);
						const float ncc = nom*rsqrtf(fmaf(normSq0[h], normSq1, 1e-3f));
						// ncc <= 0 ? 255 : floor((1 - min(ncc, 1)) * 255 + .5); 255 for windows that leave the right image
						int cv = ncc <= 0.f ? 255 : __float2int_rd(fmaf(-255.f, fminf(ncc, 1.f), 255.5f));
						if (d < dlo[h] || d >= dhi[h]) cv = 255;
						sTile[row*TILE_PITCH + d] = (uint8_t)cv;
					}
				}
			}
			bar_sync(BAR_WORKERS, TC_THREADS);
			// the block's costs: num bytes per pixel, coalesced 16-byte stores
			const int chunks = num/16;
			for (int i = tid; i < BM*chunks; i += TC_THREADS) {
				const int prow = i/chunks, c16 = i-prow*chunks;
				const int pcol = x0+prow;
				if (pcol < vw) {
					const uint32_t* src = (const uint32_t*)(sTile + prow*TILE_PITCH + 16*c16);
					const uint4 v = make_uint4(src[0], src[1], src[2], src[3]);
					*(uint4*)(P.costs + ((size_t)r*vw + pcol)*(size_t)numAll + dOff + 16*c16) = v;
				}
			}
			bar_sync(BAR_WORKERS, TC_THREADS);                  // the tile is free: the next block stages into it
		}
	}
}

} // namespace

cudaError_t sgm_cost_tc_configure() {
	return cudaFuncSetAttribute(sgm_cost_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL);
}
bool sgm_cost_tc_supports(int num) { return num == 64 || num == 128 || num == 192 || num == 256; }
cudaError_t sgm_cost_tc_launch(const SGMParams& P, int dmin, int num, cudaStream_t s) {
	int dev = 0, sms = 0;
	cudaError_t e = cudaGetDevice(&dev);
	if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
	if (e != cudaSuccess) return e;
	// slices of at most 128 disparities (the ring holds the four B tiles a block of 128 pixels x 128 disparities needs)
	for (int off = 0; off < num; off += 128)
		sgm_cost_tc_kernel<<<sms, TC_THREADS, SMEM_TOTAL, s>>>(P, dmin+off, num-off >= 128 ? 128 : num-off, num, off);
	return cudaGetLastError();
}
