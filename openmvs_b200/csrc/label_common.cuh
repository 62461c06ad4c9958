// label_common.cuh — connected components of a 4-neighbour pixel grid on the device (union-find), shared by RemoveSmallSegments
// (filter_kernels.cu) and cv::filterSpeckles (sgm_tsgm.cu).  The two differ only in their edge functor E:
//   E::at(i)        the value of pixel i (the map is read-only for the whole labelling: the functors load it with __ldg);
//   E::valid(a)     a pixel of value a takes part (a label >= 0), else its label is -1;
//   E::edge(a, b)   a valid pixel of value a and its left or upper neighbour of value b belong to one component (symmetric).
// Labelling: every pixel first links to its left (else upper) connected neighbour — a region that is reasonably convex becomes
// one tree: row runs hang on their first pixel, which hangs on the row above — pointer jumping flattens these chains in
// ceil(log2(W+H)) rounds, the upper edges the links did not take are merged by an atomicMin union on the
// flat trees (mostly "same root already"), and a second series of jumps flattens whatever chains of roots the unions built.
// The count pass leaves every label on its root and the component's size at size[root]; with a minKey array also the
// component's first pixel in column-major order (x outer, y inner: key = x*H + y) at minKey[root].
#pragma once
#include <cuda_runtime.h>

namespace {

__device__ __forceinline__ int label_find(int* L, int i) {
	int p;
	while ((p = ((volatile int*)L)[i]) != i) i = p;
	return i;
}
__device__ void label_union(int* L, int a, int b) {
	bool done;
	do {
		a = label_find(L, a); b = label_find(L, b);
		if (a < b) { const int old = atomicMin(L+b, a); done = (old == b); b = old; }
		else if (b < a) { const int old = atomicMin(L+a, b); done = (old == a); a = old; }
		else done = true;
	} while (!done);
}
template <class E>
__global__ void label_init_kernel(const E e, int* L, int* size, int* minKey, int W, int H) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= W || y >= H) return;
	const int i = y*W+x;
	const auto a = e.at(i);
	int l = -1;
	if (e.valid(a)) {
		l = i;
		if (x > 0 && e.edge(a, e.at(i-1))) l = i-1;
		else if (y > 0 && e.edge(a, e.at(i-W))) l = i-W;
	}
	L[i] = l;
	size[i] = 0;
	if (minKey) minKey[i] = 0x7FFFFFFF;
}
__global__ void label_jump_kernel(int* L, int n) {
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	const int p = L[i];
	if (p >= 0 && p != i) L[i] = ((volatile int*)L)[p]; // labels only ever move towards the root: safe in place
}
template <class E>
__global__ void label_merge_kernel(const E e, int* L, int W, int H) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x < 1 || x >= W || y < 1 || y >= H) return;
	const int i = y*W+x;
	const auto a = e.at(i);
	if (!e.valid(a)) return;
	// the link went left; the upper edge is still open
	if (e.edge(a, e.at(i-1)) && e.edge(a, e.at(i-W))) label_union(L, i, i-W);
}
template <bool KEYS>
__global__ void label_count_kernel(int* L, int* size, int* minKey, int W, int H) {
	const int n = W*H;
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	int r = -1;
	if (i < n && L[i] >= 0) {
		r = label_find(L, i);
		L[i] = r;                   // roots keep L[r] == r, so concurrent finds stay correct
	}
	// one atomic per distinct root in the warp (large components would otherwise serialise on one address)
	const unsigned peers = __match_any_sync(0xFFFFFFFFu, r);
	const bool leader = r >= 0 && (threadIdx.x&31) == __ffs(peers)-1;
	if (leader) atomicAdd(size+r, __popc(peers));
	if (KEYS) {
		const int kmin = __reduce_min_sync(peers, r >= 0 ? (i%W)*H + i/W : 0x7FFFFFFF);
		if (leader) atomicMin(minKey+r, kmin);
	}
}

// labels, sizes (and minKey, or null): W x H ints each.  Returns the number of kernels launched.
template <class E>
int label_launch(const E& e, int W, int H, int* labels, int* sizes, int* minKey, cudaStream_t s) {
	const int n = W*H;
	int rounds = 1;
	while ((1<<rounds) < W+H) ++rounds;
	const dim3 b2(32, 8), g2((W+31)/32, (H+7)/8);
	label_init_kernel<<<g2, b2, 0, s>>>(e, labels, sizes, minKey, W, H);
	for (int r = 0; r < rounds; ++r) label_jump_kernel<<<(n+255)/256, 256, 0, s>>>(labels, n);
	label_merge_kernel<<<g2, b2, 0, s>>>(e, labels, W, H);
	for (int r = 0; r < rounds; ++r) label_jump_kernel<<<(n+255)/256, 256, 0, s>>>(labels, n);
	if (minKey) label_count_kernel<true><<<(n+255)/256, 256, 0, s>>>(labels, sizes, minKey, W, H);
	else label_count_kernel<false><<<(n+255)/256, 256, 0, s>>>(labels, sizes, nullptr, W, H);
	return 3+2*rounds;
}

} // namespace
