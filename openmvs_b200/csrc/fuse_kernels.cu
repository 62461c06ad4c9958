// fuse_kernels.cu — DepthMapsData::FuseDepthMaps on the device: the kernels of one image's round (host driver: fuse_host.cu).
//
// A round fuses the pixels of one image A into points.  The reference visits them in raster order, and a point claims neighbour
// pixels, releases them again when it is rejected, and zeroes neighbour depths in front of which it lies when it is accepted.
// Within a round every neighbour pixel q (a "target") can only go from live (depth > 0, unclaimed) to dead, so each edge
// (candidate p, neighbour slot k) has a type fixed at the start of the round: claim, zero or none.  q is live at p exactly when
// every earlier owner of an edge to q was rejected, and p is accepted exactly when 1 + (its live claim edges) >= nMinViewsFuse.
// The kernels resolve that by a monotone fixed point over the edges grouped by target in raster order of their owners; the
// earliest undecided candidate always decides, so it ends, and it reproduces the sequential loop exactly (DESIGN.md §5.5).
#include <algorithm>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include "fuse_common.cuh"

namespace {

constexpr int TPB = 256;

inline unsigned blocks(size_t n) { return (unsigned)((n+TPB-1)/TPB); }

// adds the number of lanes with `pred` to *counter, one atomic per warp; every lane of the warp must call it
template <typename T>
__device__ __forceinline__ void warp_count(bool pred, T* counter) {
	const unsigned m = __ballot_sync(0xFFFFFFFFu, pred);
	if ((threadIdx.x & 31) == 0 && m) atomicAdd(counter, (T)__popc(m));
}

__global__ void k_any_positive(const float* __restrict__ depth, size_t n, int* flag) {
	for (size_t i = blockIdx.x*(size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x*blockDim.x)
		if (depth[i] > 0) { *flag = 1; return; }
}

// the candidates of the round: depth != 0 and not claimed; every depth != 0 is a visited depth (nDepths)
__global__ void k_candidates(const float* __restrict__ depth, const uint8_t* __restrict__ claim, size_t n, uint8_t* __restrict__ flags,
	unsigned long long* nDepths)
{
	const size_t i = blockIdx.x*(size_t)blockDim.x + threadIdx.x;
	const bool nz = i < n && depth[i] != 0;
	if (i < n) flags[i] = nz && !claim[i];
	warp_count(nz, nDepths);
}

__device__ __forceinline__ void view_normal(const FuseRound& R, const FuseDevView& V, size_t i, float n[3]) {
	n[0] = 0.f; n[1] = 0.f; n[2] = -1.f;
	if (R.bNormalMap && V.normal) fuse::normal_to_world(V.cam, V.normal+3*i, n);
}

// one thread per candidate: the type and the target of each of its edges, from the maps as they are at the start of the round
__global__ void k_classify(const FuseRound R, const uint32_t* __restrict__ cand, uint32_t nCand, uint8_t* __restrict__ typ,
	uint32_t* __restrict__ tgt)
{
	const uint32_t c = blockIdx.x*blockDim.x + threadIdx.x;
	if (c >= nCand) return;
	const FuseDevView& A = R.views[R.a];
	const uint32_t ia = cand[c];
	const int x = (int)(ia % (uint32_t)A.w), y = (int)(ia / (uint32_t)A.w);
	double Xw[3];
	fuse::image_to_world(A.cam, x, y, A.depth[ia], Xw);
	const float point[3] = {(float)Xw[0], (float)Xw[1], (float)Xw[2]};
	float normal[3];
	view_normal(R, A, ia, normal);
	for (int k = 0; k < R.nNb; ++k) {
		const size_t e = (size_t)c*R.nNb + k;
		uint8_t t = FE_NONE;
		uint32_t target = 0;
		const FuseDevView& B = R.views[R.nb[k]];
		float pz; int xb, yb;
		if (B.depth && fuse::project_to_pixel(B.cam, point, B.w, B.h, pz, xb, yb)) {
			const uint32_t ib = (uint32_t)yb*(uint32_t)B.w + (uint32_t)xb;
			const float depthB = B.depth[ib];
			if (depthB != 0 && !B.claim[ib]) {
				target = R.base[k] + ib;
				bool claim = false;
				if (fuse::depth_similar(pz, depthB, R.thDepth)) {
					float normalB[3];
					view_normal(R, B, ib, normalB);
					claim = fuse::dot3(normal, normalB) > R.normalError;
				}
				t = claim ? FE_CLAIM : pz < depthB ? FE_ZERO : FE_NONE;
			}
		}
		typ[e] = t; tgt[e] = target;
	}
}

__global__ void k_gather_keys(const uint32_t* __restrict__ tgt, const uint32_t* __restrict__ edges, uint32_t n, uint32_t* __restrict__ keys) {
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	if (j < n) keys[j] = tgt[edges[j]];
}

// edges whose target is shared with another candidate's edge (statistics)
__global__ void k_shared(const uint32_t* __restrict__ keys, uint32_t n, unsigned long long* shared) {
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	const bool s = j < n && ((j > 0 && keys[j-1] == keys[j]) || (j+1 < n && keys[j+1] == keys[j]));
	warp_count(s, shared);
}

// one thread per target (the head of its run of sorted edges): an edge is live while every earlier owner is rejected, dead from
// the first accepted owner on, unknown after an undecided owner
__global__ void k_walk(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ edges, uint32_t n, int nNb,
	const uint8_t* __restrict__ acc, uint8_t* __restrict__ status)
{
	const uint32_t j = blockIdx.x*blockDim.x + threadIdx.x;
	if (j >= n || (j > 0 && keys[j-1] == keys[j])) return;
	const uint32_t key = keys[j];
	uint8_t state = FS_LIVE;
	for (uint32_t t = j; t < n && keys[t] == key; ++t) {
		const uint32_t e = edges[t];
		status[e] = state;
		if (state == FS_DEAD) continue;
		const uint8_t a = acc[e/(uint32_t)nNb];
		if (a == FA_YES) state = FS_DEAD;
		else if (a == FA_UNKNOWN) state = FS_UNKNOWN;
	}
}

__global__ void k_decide(const FuseRound R, uint32_t nCand, const uint8_t* __restrict__ typ, const uint8_t* __restrict__ status,
	uint8_t* __restrict__ acc, uint32_t* undecided)
{
	const uint32_t c = blockIdx.x*blockDim.x + threadIdx.x;
	bool open = false;
	if (c < nCand && acc[c] == FA_UNKNOWN) {
		unsigned live = 0, possible = 0;
		for (int k = 0; k < R.nNb; ++k) {
			const size_t e = (size_t)c*R.nNb + k;
			if (typ[e] != FE_CLAIM) continue;
			const uint8_t s = status[e];
			live += s == FS_LIVE; possible += s != FS_DEAD;
		}
		if (1+live >= R.nMin) acc[c] = FA_YES;
		else if (1+possible < R.nMin) acc[c] = FA_NO;
		else open = true;
	}
	warp_count(open, undecided);
}

__device__ __forceinline__ bool live_claim(const uint8_t* typ, const uint8_t* status, size_t e) {
	return typ[e] == FE_CLAIM && status[e] == FS_LIVE;
}

__global__ void k_count(const FuseRound R, uint32_t nCand, const uint8_t* __restrict__ typ, const uint8_t* __restrict__ status,
	const uint8_t* __restrict__ acc, uint32_t* __restrict__ isPoint, uint32_t* __restrict__ nViews)
{
	const uint32_t c = blockIdx.x*blockDim.x + threadIdx.x;
	if (c >= nCand) return;
	const bool yes = acc[c] == FA_YES;
	uint32_t n = 0;
	if (yes) {
		n = 1;
		for (int k = 0; k < R.nNb; ++k) n += live_claim(typ, status, (size_t)c*R.nNb + k);
	}
	isPoint[c] = yes; nViews[c] = n;
}

// [points, views] of the round: the last exclusive sums plus the last counts
__global__ void k_totals(const uint32_t* isPoint, const uint32_t* pointId, const uint32_t* nViews, const uint32_t* viewOff, uint32_t n,
	uint32_t* out)
{
	out[0] = pointId[n-1] + isPoint[n-1];
	out[1] = viewOff[n-1] + nViews[n-1];
}

// one thread per accepted candidate: the point, its views ascending by image ID (InsertSort) with the sums in neighbour-list order
// as the sequential loop forms them, then the claims and the zeroed depths of the point
__global__ void k_assemble(const FuseRound R, const uint32_t* __restrict__ cand, uint32_t nCand, const uint8_t* __restrict__ typ,
	const uint32_t* __restrict__ tgt, const uint8_t* __restrict__ status, const uint8_t* __restrict__ acc,
	const uint32_t* __restrict__ pointId, const uint32_t* __restrict__ viewOff, const FuseOut O)
{
	using namespace fuse;
	const uint32_t c = blockIdx.x*blockDim.x + threadIdx.x;
	if (c >= nCand || acc[c] != FA_YES) return;
	const FuseDevView& A = R.views[R.a];
	const uint32_t ia = cand[c];
	const int x = (int)(ia % (uint32_t)A.w), y = (int)(ia / (uint32_t)A.w);
	const uint32_t id = pointId[c], v0 = viewOff[c];
	const size_t e0 = (size_t)c*R.nNb;
	O.offsets[id] = O.viewBase + v0;
	const float depth = A.depth[ia];
	double Xw[3];
	image_to_world(A.cam, x, y, depth, Xw);
	const float point[3] = {(float)Xw[0], (float)Xw[1], (float)Xw[2]};
	const float wA = conf2weight(A.conf ? A.conf[ia] : 1.f, depth);
	double confidence = (double)wA;
	float normal[3];
	view_normal(R, A, ia, normal);
	double X[3] = {mul_d((double)point[0], confidence), mul_d((double)point[1], confidence), mul_d((double)point[2], confidence)};
	const bool colorA = R.bColor && A.color;
	float Cc[3] = {0.f, 0.f, 0.f};
	if (colorA) for (int i = 0; i < 3; ++i) Cc[i] = mul_f((float)A.color[3*(size_t)ia+i], (float)confidence);
	float N[3] = {mul_f(normal[0], (float)confidence), mul_f(normal[1], (float)confidence), mul_f(normal[2], (float)confidence)};
	// position of image `v` in the point's ascending view list
	auto rank = [&](int v) {
		uint32_t p = R.a < v;
		for (int k = 0; k < R.nNb; ++k) p += live_claim(typ, status, e0+k) && R.nb[k] < v;
		return p;
	};
	{
		const uint32_t p = O.viewBase + v0 + rank(R.a);
		O.views[p] = (uint32_t)R.a; O.weights[p] = wA; O.projs[2*(size_t)p] = (uint16_t)x; O.projs[2*(size_t)p+1] = (uint16_t)y;
		A.claim[ia] = 1;
	}
	for (int k = 0; k < R.nNb; ++k) {
		const size_t e = e0+k;
		const uint8_t t = typ[e];
		if (t == FE_NONE || status[e] != FS_LIVE) continue;
		const int b = R.nb[k];
		const FuseDevView& B = R.views[b];
		const uint32_t ib = tgt[e] - R.base[k];
		if (t == FE_ZERO) { B.depth[ib] = 0; continue; }
		const int xb = (int)(ib % (uint32_t)B.w), yb = (int)(ib / (uint32_t)B.w);
		const float depthB = B.depth[ib];
		const float confB = conf2weight(B.conf ? B.conf[ib] : 1.f, depthB);
		float normalB[3];
		view_normal(R, B, ib, normalB);
		const uint32_t p = O.viewBase + v0 + rank(b);
		O.views[p] = (uint32_t)b; O.weights[p] = confB; O.projs[2*(size_t)p] = (uint16_t)xb; O.projs[2*(size_t)p+1] = (uint16_t)yb;
		B.claim[ib] = 1;
		double Xb[3];
		image_to_world(B.cam, xb, yb, depthB, Xb);
		for (int i = 0; i < 3; ++i) X[i] = add_d(X[i], mul_d(Xb[i], (double)confB));
		if (R.bColor && B.color) for (int i = 0; i < 3; ++i) Cc[i] = add_f(Cc[i], mul_f((float)B.color[3*(size_t)ib+i], confB));
		if (R.bNormal) for (int i = 0; i < 3; ++i) N[i] = add_f(N[i], mul_f(normalB[i], confB));
		confidence = add_d(confidence, (double)confB);
	}
	const double nrm = div_d(1.0, confidence);
	for (int i = 0; i < 3; ++i) O.points[3*(size_t)id+i] = (float)mul_d(X[i], nrm);
	if (colorA) for (int i = 0; i < 3; ++i) O.colors[3*(size_t)id+i] = (uint8_t)mul_f(Cc[i], (float)nrm);
	if (R.bNormal) {
		const float n0 = mul_f(N[0], (float)nrm), n1 = mul_f(N[1], (float)nrm), n2 = mul_f(N[2], (float)nrm);
		const float len = sqrt_f(add_f(add_f(mul_f(n0, n0), mul_f(n1, n1)), mul_f(n2, n2)));
		O.normals[3*(size_t)id] = div_f(n0, len); O.normals[3*(size_t)id+1] = div_f(n1, len); O.normals[3*(size_t)id+2] = div_f(n2, len);
	}
}

} // namespace

cudaError_t fuse_launch_any_positive(const float* depth, size_t n, int* flag, cudaStream_t s) {
	k_any_positive<<<std::min(blocks(n), 1024u), TPB, 0, s>>>(depth, n, flag);
	return cudaGetLastError();
}

cudaError_t fuse_launch_candidates(const float* depth, const uint8_t* claim, size_t n, uint8_t* flags, unsigned long long* nDepths,
	cudaStream_t s)
{
	k_candidates<<<blocks(n), TPB, 0, s>>>(depth, claim, n, flags, nDepths);
	return cudaGetLastError();
}

cudaError_t fuse_select(void* tmp, size_t& tmpBytes, const uint8_t* flags, uint32_t* out, uint32_t* nOut, size_t n, cudaStream_t s) {
	return cub::DeviceSelect::Flagged(tmp, tmpBytes, thrust::counting_iterator<uint32_t>(0), flags, out, nOut, (int)n, s);
}

cudaError_t fuse_launch_classify(const FuseRound& R, const uint32_t* cand, uint32_t nCand, uint8_t* typ, uint32_t* tgt, cudaStream_t s) {
	k_classify<<<blocks(nCand), TPB, 0, s>>>(R, cand, nCand, typ, tgt);
	return cudaGetLastError();
}

cudaError_t fuse_launch_gather_keys(const uint32_t* tgt, const uint32_t* edges, uint32_t nEdges, uint32_t* keys, cudaStream_t s) {
	k_gather_keys<<<blocks(nEdges), TPB, 0, s>>>(tgt, edges, nEdges, keys);
	return cudaGetLastError();
}

cudaError_t fuse_sort(void* tmp, size_t& tmpBytes, const uint32_t* keysIn, uint32_t* keysOut, const uint32_t* valsIn, uint32_t* valsOut,
	uint32_t n, int endBit, cudaStream_t s)
{
	return cub::DeviceRadixSort::SortPairs(tmp, tmpBytes, keysIn, keysOut, valsIn, valsOut, (int)n, 0, endBit, s);
}

cudaError_t fuse_launch_shared(const uint32_t* keys, uint32_t nEdges, unsigned long long* shared, cudaStream_t s) {
	k_shared<<<blocks(nEdges), TPB, 0, s>>>(keys, nEdges, shared);
	return cudaGetLastError();
}

cudaError_t fuse_launch_walk(const uint32_t* keys, const uint32_t* edges, uint32_t nEdges, int nNb, const uint8_t* acc, uint8_t* status,
	cudaStream_t s)
{
	k_walk<<<blocks(nEdges), TPB, 0, s>>>(keys, edges, nEdges, nNb, acc, status);
	return cudaGetLastError();
}

cudaError_t fuse_launch_decide(const FuseRound& R, uint32_t nCand, const uint8_t* typ, const uint8_t* status, uint8_t* acc,
	uint32_t* undecided, cudaStream_t s)
{
	k_decide<<<blocks(nCand), TPB, 0, s>>>(R, nCand, typ, status, acc, undecided);
	return cudaGetLastError();
}

cudaError_t fuse_launch_count(const FuseRound& R, uint32_t nCand, const uint8_t* typ, const uint8_t* status, const uint8_t* acc,
	uint32_t* isPoint, uint32_t* nViews, cudaStream_t s)
{
	k_count<<<blocks(nCand), TPB, 0, s>>>(R, nCand, typ, status, acc, isPoint, nViews);
	return cudaGetLastError();
}

cudaError_t fuse_scan(void* tmp, size_t& tmpBytes, const uint32_t* in, uint32_t* out, uint32_t n, cudaStream_t s) {
	return cub::DeviceScan::ExclusiveSum(tmp, tmpBytes, in, out, (int)n, s);
}

cudaError_t fuse_launch_totals(const uint32_t* isPoint, const uint32_t* pointId, const uint32_t* nViews, const uint32_t* viewOff,
	uint32_t n, uint32_t* out, cudaStream_t s)
{
	k_totals<<<1, 1, 0, s>>>(isPoint, pointId, nViews, viewOff, n, out);
	return cudaGetLastError();
}

cudaError_t fuse_launch_assemble(const FuseRound& R, const uint32_t* cand, uint32_t nCand, const uint8_t* typ, const uint32_t* tgt,
	const uint8_t* status, const uint8_t* acc, const uint32_t* pointId, const uint32_t* viewOff, const FuseOut& O, cudaStream_t s)
{
	k_assemble<<<blocks(nCand), TPB, 0, s>>>(R, cand, nCand, typ, tgt, status, acc, pointId, viewOff, O);
	return cudaGetLastError();
}
