// sgm_front.cu — SGM path aggregation as wave fronts (sm_90a), the default for uniform disparity ranges.
//
// What it computes: the eight path recursions of SemiGlobalMatcher::Match and their sum
//   L_r(p,d) = C(p,d) + min(L_r(q,d), L_r(q,d+-1)+P1, min_d' L_r(q,d')+P2) - min_d' L_r(q,d'),  S = sum_r L_r
// (pixelAccum + path drivers, libs/MVS/SemiGlobalMatcher.cpp:1003-1269; exact O(D) form under P1 <= P2 as in sgm_kernels.cu).
//
// Why a new organisation: one launch per direction read-modify-writes the u16 sum volume eight times (for 1914 x 1074 x 128
// about 10.4 GB of DRAM traffic against 2.9 GB algorithmic) and spends about 170 warp instructions per pixel and direction on
// a 128-wide scanline step.  Here
//   * 8 lanes own one pixel (16 disparities per lane as 8 packed u16x2 words): the step is SIMD-in-a-word arithmetic
//     (VIADD.16x2 / VIMNMX.U16x2 / the DPX three-input minimum VIMNMX3.U16x2), a warp advances 4 adjacent paths, the per-step
//     fixed cost (penalty lookup, neighbour shuffles, minimum reduction, loop) is shared by 4 pixels: about 25 warp
//     instructions per pixel and direction;
//   * directions whose step moves a tilted wave front f = x + 2y forward (right, right-down, down, left-down — and their
//     mirror images in the other pass) are processed TOGETHER, front block by front block: a work item is (direction,
//     band of 4 adjacent paths, block of FB consecutive fronts); items are handed out from one queue in front order, so all
//     four directions touch a block's slice of the sum volume while it is resident in the L2 (50 MB on H100): for
//     1914 x 1074 x 128 the algorithmic traffic is 2 x 263 MB of costs read and 2 x 526 MB of sums written, the other
//     phases' read-modify-writes stay in the L2;
//   * the two passes share ONE launch and one queue, each accumulating into its own sum volume (the winner-takes-all kernel
//     adds them): two independent chains of dependencies keep the warps busy;
//   * ordering instead of atomics: within a block the directions are phases; an item waits until the items of the previous
//     phase that touch its sub-cells (column ranges of the block, sgm_front_sched.h) are complete and until its own paths'
//     previous segment has been stored (path state: the normalised previous line, 256 B per path, kept in a small L2-resident
//     buffer between the segments).  Phase 0 stores the sum, so the volumes need no memset;
//   * the inputs of a step reach the warp through a ring in shared memory filled by cp.async (no destination registers:
//     the prefetch distance does not depend on the register allocator), and the whole step is branch-free, so that the warp
//     never splits (a split warp runs every shuffle through a collective re-synchronisation).
// Bit-exact against the oracle (tests/test_sgm_parity_gpu.py); the per-direction kernels of sgm_kernels.cu remain for
// ragged (tSGM) ranges and as debug variants (b200mvs_debug.sgmAggregation).
#include "sgm_common.cuh"
#include "sgm_front_sched.h"
#include <string.h>
#include <algorithm>
#include <vector>
#include <type_traits>

namespace {

constexpr int FRONT_WARPS = 4;

__device__ __forceinline__ uint4 ldcg4(const void* p) { return __ldcg((const uint4*)p); }
__device__ __forceinline__ void stcg4(void* p, uint4 v) { __stcg((uint4*)p, v); }
__device__ __forceinline__ void st_cg4_if(bool on, void* p, unsigned a, unsigned b, unsigned c, unsigned d) {
	asm volatile("{\n.reg .pred q;\nsetp.ne.b32 q, %0, 0;\n@q st.global.cg.v4.u32 [%1], {%2, %3, %4, %5};\n}"
		:: "r"((unsigned)on), "l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// asynchronous global -> shared copies (LDGSTS): no destination registers, so the prefetch distance does not depend on the
// register allocator; .cg is served by the L2 (coherent with the other SMs' st.cg after the acquire fence)
__device__ __forceinline__ void cp16(unsigned dst, const void* src) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp8(unsigned dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp4(unsigned dst, const void* src) { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(dst), "l"(src) : "memory"); }
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

// One step's inputs of a warp in shared memory: planes of 32 lanes x 16 B (costs: 2*NW bytes per lane, sums: 4*NW bytes per
// lane), then 32 x 4 B of intensities.  A lane reads back exactly what it copied.
template <int NW> struct FrontSlot {
	static constexpr int CB = 2*NW, SB = 4*NW;
	static constexpr int NC = (CB+15)/16, NS = SB/16;
	static constexpr int IOFF = (NC+NS)*512;
	static constexpr int BYTES = IOFF+128;
};

// NW words per lane (2*NW disparities), 8 lanes per pixel, 4 pixels (adjacent paths) per warp; PD = ring slots = steps whose
// loads are in flight.  Dense volumes only: every pixel of the valid region is valid, owns `num` = 16*NW entries at
// idx = (y*vw + x)*num (checked by the caller).  Per-item overhead is kept off the critical path: the ticket of the item after
// next and the record of the next item are requested while the current item runs; the copies of the first steps' read-only
// inputs (costs, intensities) are issued before the dependency wait; the wait polls with relaxed loads and fences once.
template <int NW, int PD>
__global__ void __launch_bounds__(FRONT_WARPS*32)
sgm_front_kernel(const __grid_constant__ SGMParams P, const __grid_constant__ FrontArgs A)
{
	typedef FrontSlot<NW> SL;
	extern __shared__ uint4 ringMem[];
	__shared__ unsigned sP2[256];   // adaptive P2 replicated in both halfwords (GenerateP2s, SemiGlobalMatcher.cpp:518-524)
	for (int i = threadIdx.x; i < 256; i += blockDim.x) sP2[i] = (unsigned)P.P2s[i]*0x10001u;
	__syncthreads();
	const int lane = threadIdx.x&31;
	const int g = lane>>3, sub = lane&7;
	const unsigned P1x2 = (unsigned)P.P1*0x10001u;
	const int vw = P.vw, vh = P.vh, num = A.num;
	char* const ring = (char*)ringMem + (size_t)(threadIdx.x>>5)*PD*SL::BYTES;
	const unsigned ringS = (unsigned)__cvta_generic_to_shared(ring);
	// queue: `ticket` is being processed, `next` is already claimed, the one after is requested at the top of the loop
	int ticket = 0, next = 0;
	if (lane == 0) { ticket = atomicAdd(A.ticket, 1); next = atomicAdd(A.ticket, 1); }
	ticket = __shfl_sync(0xFFFFFFFFu, ticket, 0); next = __shfl_sync(0xFFFFFFFFu, next, 0);
	uint4 r0 = make_uint4(0u, 0u, 0u, 0u), r1 = r0;
	if (ticket < A.nItems) { r0 = __ldg((const uint4*)(A.items+ticket)); r1 = __ldg((const uint4*)(A.items+ticket)+1); }
	#pragma unroll 1
	while (ticket < A.nItems) {
		int next2 = 0;
		if (lane == 0) next2 = atomicAdd(A.ticket, 1);
		uint4 n0 = make_uint4(0u, 0u, 0u, 0u), n1 = n0;
		if (next < A.nItems) { n0 = __ldg((const uint4*)(A.items+next)); n1 = __ldg((const uint4*)(A.items+next)+1); }
		const int k0 = (int)r0.x, dir = (int)(r0.y&0xFFu), pass = (int)((r0.y>>8)&1u), ph = (int)(short)(r0.y>>16), fblk = (int)r0.z, seq = (int)r0.w;
		const int chain = (int)r1.x, depCell = (int)r1.y, depNeed = (int)r1.z, cell = (int)r1.w;
		// geometry of this lane's path
		int xs = 0, ys = 0, dx = 0, dy = 0;
		const bool pv = front_path_start(dir, k0+g, vw, vh, xs, ys, dx, dy);
		const int n = pv ? front_path_len(xs, ys, dx, dy, vw, vh) : 0;
		const int f0 = A.fa[pass]*xs + A.fb[pass]*ys + A.fc[pass], df = max(1, A.fa[pass]*dx + A.fb[pass]*dy);
		const int s0 = min(n, front_first_step(fblk*A.FB, f0, df)), s1 = min(n, front_first_step((fblk+1)*A.FB, f0, df));
		const int cnt = s1-s0;
		const int maxcnt = __reduce_max_sync(0xFFFFFFFFu, cnt);
		const bool add = __any_sync(0xFFFFFFFFu, !(A.storePhase0[pass] && ph == 0));   // item-wide, and known to be warp-uniform
		uint16_t* const sum = A.sum[pass];
		// Step k of this lane's segment lies at base + min(k, last)*stride: every lane takes part in every copy (lanes whose
		// segment is shorter re-read their last step, lanes without steps the first slice of the volume).
		const int last = max(cnt-1, 0);
		const long long pix0 = cnt > 0 ? (long long)(ys+s0*dy)*vw + (xs+s0*dx) : 0;
		const uint8_t* const cbase = P.costs + (size_t)pix0*(size_t)num + (size_t)sub*(2*NW);
		uint16_t* const sbase = sum + (size_t)pix0*(size_t)num + (size_t)sub*(2*NW);
		const float* const ibase = P.lgray + (cnt > 0 ? (size_t)(ys+s0*dy)*P.w + (xs+s0*dx) : 0);
		const int cstep = (dy*vw + dx)*num, istep = dy*P.w + dx;          // element strides of one step (|cstep| < 2^31: checked by the host)
		auto copy_ci = [&](int j, int k) {   // costs and intensity of step k into slot j
			const uint8_t* c = cbase + (long long)min(k, last)*cstep;
			const unsigned d = ringS + (unsigned)(j*SL::BYTES + lane*16);
			if (SL::CB >= 16) {
				#pragma unroll
				for (int p = 0; p < SL::NC; ++p) cp16(d + p*512, c + p*16);
			} else cp8(d, c);
			cp4(ringS + (unsigned)(j*SL::BYTES + SL::IOFF + lane*4), ibase + (long long)min(k, last)*istep);
		};
		auto copy_s = [&](int j, int k) {    // sums of step k into slot j
			const uint16_t* sp = sbase + (long long)min(k, last)*cstep;
			const unsigned d = ringS + (unsigned)(j*SL::BYTES + SL::NC*512 + lane*16);
			#pragma unroll
			for (int p = 0; p < SL::NS; ++p) cp16(d + p*512, sp + p*8);
		};
		// read-only inputs of the first PD steps: no dependency, requested before the wait (one group)
		#pragma unroll
		for (int j = 0; j < PD; ++j) if (j < maxcnt) copy_ci(j, j);
		cp_commit();
		// wait for the predecessors: the previous segment of this band (progress[chain] >= seq) and the items of the previous phase
		// that touch this item's sub-cells (cellDone >= cellNeed for nDep consecutive counters).  Lane i < nDep polls counter i,
		// the other lanes the band's progress word — one load instruction per poll — and the exit is a vote: a loop run by one
		// lane alone leaves the warp split in two (measured: the steps after it then ran once per half, every shuffle through a
		// collective re-synchronisation).
		{
			const int nDep = depCell >= 0 ? (depNeed & 0xFF) : 0;
			const int* pw = lane < nDep ? A.cellDone+depCell+lane : A.progress+chain;
			const int need = lane < nDep ? __ldg(A.cellNeed+depCell+lane) : seq;
			unsigned spins = 0;
			for (;;) {
				int v;
				asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(pw) : "memory");
				if (__all_sync(0xFFFFFFFFu, v >= need)) break;
				__nanosleep(64);
				if (++spins > (1u<<21)) { if (lane == 0) *A.error = 1; break; }
			}
			// acquire: one acquire load per lane once satisfied (not a fence: a fence would also wait for the cost copies requested
			// above); the predecessors' stores are then visible to the loads below (ld.cg / cp.async.cg: served by the L2)
			int v;
			asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(pw) : "memory");
			if (v < need) *A.error = 2;   // cannot happen: the counters only grow
		}
		// the sums of the first PD steps: one group per step (empty when the phase stores)
		#pragma unroll
		for (int j = 0; j < PD; ++j) { if (add && j < maxcnt) copy_s(j, j); cp_commit(); }
		// path state: the previous line minus its minimum (all 0xFFFF at the start of a path: the step then yields C + P2,
		// SemiGlobalMatcher.cpp:1003-1006) and the previous intensity
		const size_t slot = (size_t)(pass*4+ph)*A.maxPaths + (size_t)(k0+g);
		unsigned w[NW];
		float Ip = 0.5f;
		#pragma unroll
		for (int i = 0; i < NW; ++i) w[i] = 0xFFFFFFFFu;
		if (s0 > 0 && cnt > 0) {
			Ip = __ldcg(A.meta+slot).x;
			const uint16_t* st = A.state + slot*(size_t)num + (size_t)sub*(2*NW);
			#pragma unroll
			for (int i = 0; i < NW; i += 4) { const uint4 v = ldcg4(st+2*i); w[i] = v.x; w[i+1] = v.y; w[i+2] = v.z; w[i+3] = v.w; }
		}
		unsigned mp2 = 0u;   // minimum of the line in w, in both halfwords (0: normalised)
		uint16_t* optr = sbase;
		#pragma unroll 1
		for (int t = 0; t < maxcnt; t += PD) {
			#pragma unroll
			for (int j = 0; j < PD; ++j) {
				const int tt = t+j;
				if (tt >= maxcnt) break;
				const bool act = tt < cnt;
				// the group of step tt has landed when at most the PD-1 younger ones are pending
				cp_wait<PD-1>();
				const char* sl = ring + j*SL::BYTES + lane*16;
				unsigned C[NW], S[NW];
				if (SL::CB >= 16) {
					#pragma unroll
					for (int p = 0; p < SL::NC; ++p) {
						const uint4 v = *(const uint4*)(sl + p*512);
						C[8*p+0] = __byte_perm(v.x, 0u, 0x4140); C[8*p+1] = __byte_perm(v.x, 0u, 0x4342);
						C[8*p+2] = __byte_perm(v.y, 0u, 0x4140); C[8*p+3] = __byte_perm(v.y, 0u, 0x4342);
						C[8*p+4] = __byte_perm(v.z, 0u, 0x4140); C[8*p+5] = __byte_perm(v.z, 0u, 0x4342);
						C[8*p+6] = __byte_perm(v.w, 0u, 0x4140); C[8*p+7] = __byte_perm(v.w, 0u, 0x4342);
					}
				} else {
					const uint2 v = *(const uint2*)sl;
					C[0] = __byte_perm(v.x, 0u, 0x4140); C[1] = __byte_perm(v.x, 0u, 0x4342);
					C[2] = __byte_perm(v.y, 0u, 0x4140); C[3] = __byte_perm(v.y, 0u, 0x4342);
				}
				if (add) {
					#pragma unroll
					for (int p = 0; p < SL::NS; ++p) {
						const uint4 v = *(const uint4*)(sl + (SL::NC+p)*512);
						S[4*p] = v.x; S[4*p+1] = v.y; S[4*p+2] = v.z; S[4*p+3] = v.w;
					}
				} else {
					#pragma unroll
					for (int i = 0; i < NW; ++i) S[i] = 0u;
				}
				const float I = *(const float*)(ring + j*SL::BYTES + SL::IOFF + lane*4);
				// penalty of this step: P2s[|round(255 (I - Ip))|] (SemiGlobalMatcher.cpp:1009, 518-524)
				const int di = min(255, abs((int)floorf(255.f*(I-Ip)+.5f)));
				const unsigned P2x2 = sP2[di];
				// With w = previous line (not normalised) and mp its minimum:
				//   L = C + min(w - mp, min(w[d-1], w[d+1]) - mp + P1, P2) = C + min(w, min(w[d-1], w[d+1]) + P1, P2 + mp) - mp,
				// so the neighbour exchange does not wait for the minimum of the previous step (shorter dependent chain).
				// Neighbours d-1 / d+1 across the lanes of the pixel: 0xFFFF beyond the two ends of the range.
				unsigned below = __shfl_up_sync(0xFFFFFFFFu, w[NW-1]>>16, 1), above = __shfl_down_sync(0xFFFFFFFFu, w[0]&0xFFFFu, 1);
				if (sub == 0) below = 0xFFFFu;
				if (sub == 7) above = 0xFFFFu;
				unsigned q[NW+1], L[NW];
				q[0] = __byte_perm(below, w[0], 0x5410);               // (L[-1], L[0])
				#pragma unroll
				for (int i = 1; i < NW; ++i) q[i] = __byte_perm(w[i-1], w[i], 0x5432);   // (L[2i-1], L[2i])
				q[NW] = __byte_perm(w[NW-1], above, 0x5432);
				const unsigned cap = __vadd2(P2x2, mp2);
				#pragma unroll
				for (int i = 0; i < NW; ++i) {
					const unsigned nb = __vaddus2(__vminu2(q[i], q[i+1]), P1x2);
					L[i] = __vsub2(__vadd2(C[i], __vimin3_u16x2(w[i], nb, cap)), mp2);
				}
				// minimum of the new line: within the lane, then three butterfly steps over the pixel's 8 lanes on the packed pair
				// (a sub-warp redux.sync with a per-group mask compiles to a WARPSYNC.COLLECTIVE loop: about 2000 cycles per step)
				unsigned m = L[0];
				#pragma unroll
				for (int i = 1; i+1 < NW; i += 2) m = __vimin3_u16x2(m, L[i], L[i+1]);
				if ((NW&1) == 0) m = __vminu2(m, L[NW-1]);
				m = __vminu2(m, __shfl_xor_sync(0xFFFFFFFFu, m, 4));
				m = __vminu2(m, __shfl_xor_sync(0xFFFFFFFFu, m, 2));
				m = __vminu2(m, __shfl_xor_sync(0xFFFFFFFFu, m, 1));
				m = min(m&0xFFFFu, m>>16);
				// lanes whose segment has ended keep their line (predicated moves and stores: no branch, the warp stays converged)
				#pragma unroll
				for (int i = 0; i < NW; ++i) w[i] = act ? L[i] : w[i];
				#pragma unroll
				for (int i = 0; i < NW; i += 4)
					st_cg4_if(act, optr+2*i, __vadd2(S[i], L[i]), __vadd2(S[i+1], L[i+1]), __vadd2(S[i+2], L[i+2]), __vadd2(S[i+3], L[i+3]));
				optr += act ? cstep : 0;
				mp2 = act ? m*0x10001u : mp2;
				Ip = act ? I : Ip;
				// refill the slot (its contents are in registers that have been consumed) with step tt+PD
				if (tt+PD < maxcnt) { copy_ci(j, tt+PD); if (add) copy_s(j, tt+PD); }
				cp_commit();
			}
		}
		// store the state for the next segment of these paths, then publish
		if (cnt > 0 && s1 < n) {
			uint16_t* st = A.state + slot*(size_t)num + (size_t)sub*(2*NW);
			#pragma unroll
			for (int i = 0; i < NW; i += 4) stcg4(st+2*i, make_uint4(__vsub2(w[i], mp2), __vsub2(w[i+1], mp2), __vsub2(w[i+2], mp2), __vsub2(w[i+3], mp2)));
			if (sub == 0) __stcg(A.meta+slot, make_float2(Ip, 1.f));
		}
		// publish: every lane fences its own stores (one MEMBAR per warp), the barrier makes all of them happen before the signals
		// that lane 0 (band progress) and lanes < nOwn (sub-cell counters) then send
		asm volatile("fence.acq_rel.gpu;" ::: "memory");
		__syncwarp();
		{
			const int nOwn = (depNeed>>8) & 0xFF;
			if (lane == 0) asm volatile("st.relaxed.gpu.global.s32 [%0], %1;" :: "l"(A.progress+chain), "r"(seq+1) : "memory");
			if (lane < nOwn) asm volatile("red.relaxed.gpu.global.add.s32 [%0], 1;" :: "l"(A.cellDone+cell+lane) : "memory");
		}
		ticket = next; next = __shfl_sync(0xFFFFFFFFu, next2, 0);
		r0 = n0; r1 = n1;
	}
}

template <int NW, int PD> cudaError_t front_launch(const SGMParams& P, const FrontArgs& A, int blocks, cudaStream_t s) {
	const int smem = FRONT_WARPS*PD*FrontSlot<NW>::BYTES;
	cudaError_t e = cudaFuncSetAttribute(sgm_front_kernel<NW, PD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
	if (e != cudaSuccess) return e;
	sgm_front_kernel<NW, PD><<<blocks, FRONT_WARPS*32, smem, s>>>(P, A);
	return cudaGetLastError();
}
template <int NW, int PD> int front_blocks_per_sm() {
	int per = 1;
	const int smem = FRONT_WARPS*PD*FrontSlot<NW>::BYTES;
	cudaFuncSetAttribute(sgm_front_kernel<NW, PD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
	cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, sgm_front_kernel<NW, PD>, FRONT_WARPS*32, smem);
	return std::max(1, per);
}

} // namespace

// pd: ring slots per warp (4 or 8 steps in flight)
cudaError_t sgm_front_launch(const SGMParams& P, const FrontArgs& A, int blocks, int pd, cudaStream_t s) {
	const int NW = A.num/16;
	if (NW == 8) return pd == 4 ? front_launch<8, 4>(P, A, blocks, s) : front_launch<8, 8>(P, A, blocks, s);
	if (NW == 4) return pd == 4 ? front_launch<4, 4>(P, A, blocks, s) : front_launch<4, 8>(P, A, blocks, s);
	if (NW == 16) return pd == 4 ? front_launch<16, 4>(P, A, blocks, s) : front_launch<16, 8>(P, A, blocks, s);
	return cudaErrorInvalidValue;
}
// resident CTAs of the kernel per SM on the current device
int sgm_front_blocks_per_sm(int num, int pd) {
	const int NW = num/16;
	if (NW == 8) return pd == 4 ? front_blocks_per_sm<8, 4>() : front_blocks_per_sm<8, 8>();
	if (NW == 4) return pd == 4 ? front_blocks_per_sm<4, 4>() : front_blocks_per_sm<4, 8>();
	if (NW == 16) return pd == 4 ? front_blocks_per_sm<16, 4>() : front_blocks_per_sm<16, 8>();
	return 1;
}
bool sgm_front_supports(int num) { return num == 64 || num == 128 || num == 256; }
