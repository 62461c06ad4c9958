// filter_kernels.cu — depth-map post-processing that follows the estimation path:
//   DepthMapsData::FilterDepthMap       libs/MVS/SceneDensify.cpp:1050-1299
//   DepthMapsData::RemoveSmallSegments  libs/MVS/SceneDensify.cpp:810-900
//   DepthMapsData::GapInterpolation     libs/MVS/SceneDensify.cpp:904-1045
//
// FilterDepthMap on the reference is two sequential loops: a z-buffered forward splat of every
// neighbour depth-map into the reference view, then a per-pixel vote.  Here the splat is one
// thread per neighbour pixel with a 64-bit atomicMin per touched reference pixel: the key is
// (float bits of the projected depth << 32) | (0xFFFFFFFF - source pixel index), so the minimum
// is the smallest depth and, among equal depths, the LAST source pixel in row-major order —
// exactly what the reference's sequential `if (depthRef != 0 && depthRef < z) continue;` leaves
// behind.  The vote is one thread per reference pixel and decodes the keys directly.
// All camera arithmetic is double with explicit _rn intrinsics (no FMA contraction), in the
// evaluation order oracle/filter_oracle.cpp writes out, so results are bit-identical to it.
// HBM-bound integer/float work: per reference pixel the vote reads 8 B x N keys + 8 B and
// writes 8 B; the splat reads 4 B and issues <= 4 atomics per neighbour pixel.
#include "filter_common.cuh"

namespace {

// IsDepthSimilar (libs/Common/Util.inl:797-809), not symmetric
__device__ __forceinline__ bool depth_similar(float d0, float d1, float th) { return __fdiv_rn(fabsf(__fsub_rn(d0, d1)), d0) < th; }

// Camera::TransformPointI2W(Point3(x,y,z)) (libs/MVS/Camera.h:339-356)
__device__ __forceinline__ void i2w(const FltView& v, double x, double y, double z, double X[3]) {
	const double cx = __ddiv_rn(__dmul_rn(__dsub_rn(x, v.cx), z), v.fx);
	const double cy = __ddiv_rn(__dmul_rn(__dsub_rn(y, v.cy), z), v.fy);
	#pragma unroll
	for (int i = 0; i < 3; ++i)
		X[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(v.R[i], cx), __dmul_rn(v.R[3+i], cy)), __dmul_rn(v.R[6+i], z)), v.C[i]);
}
// Camera::TransformPointW2C (Camera.h:388-390)
__device__ __forceinline__ void w2c(const FltView& v, const double X[3], double c[3]) {
	const double t0 = __dsub_rn(X[0], v.C[0]), t1 = __dsub_rn(X[1], v.C[1]), t2 = __dsub_rn(X[2], v.C[2]);
	#pragma unroll
	for (int i = 0; i < 3; ++i)
		c[i] = __dadd_rn(__dadd_rn(__dmul_rn(v.R[i*3], t0), __dmul_rn(v.R[i*3+1], t1)), __dmul_rn(v.R[i*3+2], t2));
}
// Camera::TransformPointC2I(Point3) (Camera.h:370-386)
__device__ __forceinline__ void c2i(const FltView& v, const double c[3], double& u, double& w) {
	u = __dadd_rn(v.cx, __dmul_rn(v.fx, __ddiv_rn(c[0], c[2])));
	w = __dadd_rn(v.cy, __dmul_rn(v.fy, __ddiv_rn(c[1], c[2])));
}

__global__ void __launch_bounds__(256) flt_project_kernel(const __grid_constant__ FltParams P) {
	const int n = blockIdx.y;
	const FltView& nb = P.nbr[n];
	const unsigned idx = blockIdx.x*blockDim.x+threadIdx.x;
	if (idx >= (unsigned)(nb.w*nb.h)) return;
	const float depth = nb.depth[idx];
	if (depth == 0) return;
	const int j = idx%nb.w, i = idx/nb.w;
	double X[3], c[3], u, v;
	i2w(nb, (double)j, (double)i, (double)depth, X);
	w2c(P.ref, X, c);
	if (c[2] <= 0) return;
	c2i(P.ref, c, u, v);
	const double xs[2] = {floor(u), ceil(u)}, ys[2] = {floor(v), ceil(v)};
	const unsigned long long key = ((unsigned long long)__float_as_uint((float)c[2]) << 32) | (unsigned long long)(0xFFFFFFFFu-idx);
	const int W = P.ref.w, H = P.ref.h;
	unsigned long long* z = P.zbuf+(size_t)n*W*H;
	#pragma unroll
	for (int p = 0; p < 4; ++p) {
		const double px = xs[p>>1], py = ys[p&1];
		if (!(px >= 0 && py >= 0 && px < W && py < H)) continue;
		if (p == 1 && ys[1] == ys[0]) continue;                     // same pixel again: the key is identical
		if (p >= 2 && xs[1] == xs[0]) continue;
		atomicMin(z+(size_t)py*W+(size_t)px, key);
	}
}

__device__ __forceinline__ float key_depth(unsigned long long k) { return k == ~0ull ? 0.f : __uint_as_float((unsigned)(k>>32)); }
__device__ __forceinline__ unsigned key_src(unsigned long long k) { return 0xFFFFFFFFu-(unsigned)k; }

// bAdjust branch (:1141-1210): confidence-weighted average of the agreeing depths
__global__ void __launch_bounds__(256) flt_adjust_kernel(const __grid_constant__ FltParams P) {
	const int W = P.ref.w, H = P.ref.h;
	const size_t np = (size_t)W*H;
	const size_t o = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (o >= np) return;
	const float depth = P.ref.depth[o];
	float od = 0, oc = 0;
	if (depth != 0) {
		float posConf = P.ref.conf[o], negConf = 0;
		float avgDepth = __fmul_rn(depth, posConf);
		unsigned nPos = 0, nNeg = 0;
		unsigned n = (unsigned)P.N;
		bool discard = false;
		do {
			--n;
			const unsigned long long k = P.zbuf[np*n+o];
			const float d = key_depth(k);
			if (d == 0) {
				if (nPos+nNeg+n < (unsigned)P.nMinViews) { discard = true; break; }
				continue;
			}
			const FltView& nb = P.nbr[n];
			const float cproj = nb.conf[key_src(k)];
			if (depth_similar(depth, d, P.thDepthDiff)) {
				avgDepth = __fadd_rn(avgDepth, __fmul_rn(d, cproj));
				posConf = __fadd_rn(posConf, cproj);
				++nPos;
			} else {
				if (depth > d) {
					negConf = __fadd_rn(negConf, cproj);              // occlusion
				} else {                                               // free-space violation
					double X[3], c3[3], u, v;
					i2w(P.ref, (double)(o%W), (double)(o/W), (double)depth, X);
					w2c(nb, X, c3);
					c2i(nb, c3, u, v);
					const double rx = floor(__dadd_rn(u, .5)), ry = floor(__dadd_rn(v, .5));
					float c = 0;
					if (rx >= 0 && ry >= 0 && rx < nb.w && ry < nb.h)
						c = nb.conf[(size_t)ry*nb.w+(size_t)rx];
					negConf = __fadd_rn(negConf, c > 0 ? c : cproj);
				}
				++nNeg;
			}
		} while (n);
		if (!discard && nPos >= (unsigned)P.nMinViewsAdjust && posConf > negConf) {
			avgDepth = __fdiv_rn(avgDepth, posConf);
			if (P.dMin <= avgDepth && avgDepth < P.dMax) { od = avgDepth; oc = __fsub_rn(posConf, negConf); }
		}
	}
	P.outDepth[o] = od; P.outConf[o] = oc;
}

// !bAdjust branch (:1211-1289): keep the depth if enough projected neighbours agree at the pixel
// and around it
__global__ void __launch_bounds__(256) flt_strict_kernel(const __grid_constant__ FltParams P) {
	const int W = P.ref.w, H = P.ref.h;
	const size_t np = (size_t)W*H;
	const size_t o = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (o >= np) return;
	const float depth = P.ref.depth[o];
	float od = 0, oc = 0;
	if (depth != 0) {
		unsigned good = 0, views = 0;
		for (int n = P.N; n-- > 0; ) {
			const float d = key_depth(P.zbuf[np*n+o]);
			if (d > 0) { ++views; if (depth_similar(depth, d, P.thStrict)) ++good; }
		}
		if (!(good < (unsigned)P.nMinViews || good < views*75/100)) {
			const int x0 = (int)(o%W), y0 = (int)(o/W);
			good = views = 0;
			#pragma unroll
			for (int k = 0; k < 4; ++k) {
				const int x = x0+(k == 0 ? -1 : k == 1 ? 1 : 0), y = y0+(k == 2 ? -1 : k == 3 ? 1 : 0);
				if (x < 0 || y < 0 || x >= W || y >= H) continue;
				for (int n = P.N; n-- > 0; ) {
					const float d = key_depth(P.zbuf[np*n+(size_t)y*W+x]);
					if (d > 0) { ++views; if (depth_similar(depth, d, P.thDepthDiff)) ++good; }
				}
			}
			if (!(good < (unsigned)P.nMinViews*2 || good < views*65/100)) { od = depth; oc = P.ref.conf[o]; }
		}
	}
	P.outDepth[o] = od; P.outConf[o] = oc;
}

// decode the keys of one neighbour into plain depth / confidence maps (inspection and tests)
__global__ void flt_resolve_kernel(const unsigned long long* z, const float* nbrConf, size_t np, float* depth, float* conf) {
	const size_t o = (size_t)blockIdx.x*blockDim.x+threadIdx.x;
	if (o >= np) return;
	const unsigned long long k = z[o];
	depth[o] = key_depth(k);
	if (conf) conf[o] = (k == ~0ull || !nbrConf) ? 0.f : nbrConf[key_src(k)];
}

// ---- RemoveSmallSegments: connected components over the 4-neighbour grid ----
// The reference grows segments breadth-first, seeds in column-major order, with a DIRECTED test
// IsDepthSimilar(current, neighbour) = |d0-d1|/d0 < th (SceneDensify.cpp:810-900).  Where a pair passes in both directions the
// segment does not depend on the order; where it passes in one direction only (relative difference within th^2 of the threshold)
// it does.  Exact parallel form:
//   1. label the components over TWO-WAY edges (every breadth-first segment is a union of such components);
//   2. list the one-way edges between different components ("arcs": a handful per map) with the sizes and the first pixel (in the
//      reference's seed order) of the components they join;
//   3. replay the reference's loop on that condensed graph on the host — components in seed order, a segment = every
//      not-yet-visited component reachable along arcs — and patch the sizes of the components involved;
//   4. remove the pixels whose segment is smaller than nSpeckleSize.
// Labelling: every pixel first links to its left (else upper) connected neighbour — a region that is
// reasonably convex becomes one tree: row runs hang on their first pixel, which hangs on the row above —
// pointer jumping flattens these chains in ceil(log2(W+H)) rounds, the upper edges the links did not
// take are merged by an atomicMin union on the flat trees (mostly "same root already"), and a second
// series of jumps flattens whatever chains of roots the unions built.
__device__ __forceinline__ bool seg_edge(float a, float b, float th) {
	return b > 0 && depth_similar(a, b, th) && depth_similar(b, a, th);
}
__device__ __forceinline__ int uf_find(int* L, int i) {
	int p;
	while ((p = ((volatile int*)L)[i]) != i) i = p;
	return i;
}
__device__ void uf_union(int* L, int a, int b) {
	bool done;
	do {
		a = uf_find(L, a); b = uf_find(L, b);
		if (a < b) { const int old = atomicMin(L+b, a); done = (old == b); b = old; }
		else if (b < a) { const int old = atomicMin(L+a, b); done = (old == a); a = old; }
		else done = true;
	} while (!done);
}
__global__ void seg_init_kernel(const float* __restrict__ depth, int* L, int* size, int* minKey, int W, int H, float th) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= W || y >= H) return;
	const int i = y*W+x;
	const float a = depth[i];
	int l = -1;
	if (a > 0) {
		l = i;
		if (x > 0 && seg_edge(a, depth[i-1], th)) l = i-1;
		else if (y > 0 && seg_edge(a, depth[i-W], th)) l = i-W;
	}
	L[i] = l;
	size[i] = 0;
	minKey[i] = 0x7FFFFFFF;
}
__global__ void seg_jump_kernel(int* L, int n) {
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	const int p = L[i];
	if (p >= 0 && p != i) L[i] = ((volatile int*)L)[p]; // labels only ever move towards the root: safe in place
}
__global__ void seg_merge_kernel(const float* __restrict__ depth, int* L, int W, int H, float th) {
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x < 1 || x >= W || y < 1 || y >= H) return;
	const int i = y*W+x;
	const float a = depth[i];
	if (!(a > 0)) return;
	// the link went left; the upper edge is still open
	if (seg_edge(a, depth[i-1], th) && seg_edge(a, depth[i-W], th)) uf_union(L, i, i-W);
}
// sizes of the components and their first pixel in the reference's seed order (x outer, y inner: key = x*H + y)
__global__ void seg_count_kernel(int* L, int* size, int* minKey, int W, int H) {
	const int n = W*H;
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	int r = -1, key = 0x7FFFFFFF;
	if (i < n && L[i] >= 0) {
		r = uf_find(L, i);
		L[i] = r;                   // roots keep L[r] == r, so concurrent finds stay correct
		key = (i%W)*H + i/W;
	}
	// one atomic per distinct root in the warp (large segments would otherwise serialise on one address)
	const unsigned peers = __match_any_sync(0xFFFFFFFFu, r);
	const int kmin = __reduce_min_sync(peers, key);
	if (r >= 0 && (threadIdx.x&31) == __ffs(peers)-1) { atomicAdd(size+r, __popc(peers)); atomicMin(minKey+r, kmin); }
}
__global__ void seg_arcs_kernel(const float* __restrict__ depth, const int* __restrict__ L, const int* __restrict__ size, const int* __restrict__ minKey,
	int W, int H, float th, SegArc* arcs, int* count, int cap)
{
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y*blockDim.y+threadIdx.y;
	if (x >= W || y >= H) return;
	const int i = y*W+x;
	const float a = depth[i];
	if (!(a > 0)) return;
	#pragma unroll
	for (int k = 0; k < 2; ++k) {
		if (k == 0 ? x+1 >= W : y+1 >= H) continue;
		const int j = k == 0 ? i+1 : i+W;
		const float b = depth[j];
		if (!(b > 0)) continue;
		const bool ab = depth_similar(a, b, th), ba = depth_similar(b, a, th);
		if (ab == ba) continue;
		const int li = L[i], lj = L[j];
		if (li == lj) continue;
		const int src = ab ? li : lj, dst = ab ? lj : li;
		const int slot = atomicAdd(count, 1);
		if (slot < cap) arcs[slot] = SegArc{src, dst, size[src], size[dst], minKey[src], minKey[dst]};
	}
}
__global__ void seg_patch_kernel(const int2* __restrict__ patch, int n, int* size) {
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	if (i < n) size[patch[i].x] = patch[i].y;
}
__global__ void seg_remove_kernel(const int* L, const int* size, int n, unsigned speckle, float* depth, float* normal, float* conf) {
	const int i = blockIdx.x*blockDim.x+threadIdx.x;
	if (i >= n) return;
	// an invalid pixel is a segment of one in the reference, so its normal / confidence are cleared too
	if (L[i] < 0 ? 1u < speckle : (unsigned)size[L[i]] < speckle) {
		depth[i] = 0;
		if (normal) { normal[i*3] = 0; normal[i*3+1] = 0; normal[i*3+2] = 0; }
		if (conf) conf[i] = 0;
	}
}

// ---- GapInterpolation: one thread per pixel of a line-wise pass, out of place ----
// PASS 0 walks rows, PASS 1 columns.  A pixel inside a gap of `count` <= gap invalid pixels
// between two valid, similar ones gets the k-th partial sum of the reference's running
// interpolation (d += diff, k times, so the rounding is the same).
template <int PASS>
__global__ void __launch_bounds__(256) gap_kernel(const float* __restrict__ sd, const float* __restrict__ sn, const float* __restrict__ sc,
	float* __restrict__ dd, float* __restrict__ dn, float* __restrict__ dc, int W, int H, float th, int gap)
{
	const int x = blockIdx.x*blockDim.x+threadIdx.x, y = blockIdx.y;
	if (x >= W) return;
	const int o = y*W+x;
	const int step = PASS == 0 ? 1 : W, pos = PASS == 0 ? x : y, len = PASS == 0 ? W : H;
	float d = sd[o];
	float nx = 0, ny = 0, nz = 0, c = 0;
	if (sn) { nx = sn[o*3]; ny = sn[o*3+1]; nz = sn[o*3+2]; }
	if (sc) c = sc[o];
	if (d <= 0) {
		int l = 1, r = 1;
		while (l <= gap && pos-l >= 0 && sd[o-l*step] <= 0) ++l;
		if (l <= gap && pos-l >= 0) {                        // first valid pixel before the gap
			while (l+r-1 <= gap && pos+r < len && sd[o+r*step] <= 0) ++r;
			const int count = l+r-1;
			if (count <= gap && pos+r < len) {
				const int of = o-l*step, ol = o+r*step;
				const float d0 = sd[of], d1 = sd[ol];
				if (depth_similar(d0, d1, th)) {
					const float den = (float)(count+1);
					const float diff = __fdiv_rn(__fsub_rn(d1, d0), den);
					d = d0;
					for (int k = 0; k < l; ++k) d = __fadd_rn(d, diff);
					if (sc) { const float c0 = sc[of], c1 = sc[ol]; c = c0 < c1 ? c0 : c1; }
					if (sn) {
						float a1 = atan2f(sn[of*3+1], sn[of*3]), b1 = acosf(sn[of*3+2]);
						const float a2 = atan2f(sn[ol*3+1], sn[ol*3]), b2 = acosf(sn[ol*3+2]);
						const float da = __fdiv_rn(__fsub_rn(a2, a1), den), db = __fdiv_rn(__fsub_rn(b2, b1), den);
						for (int k = 0; k < l; ++k) { a1 = __fadd_rn(a1, da); b1 = __fadd_rn(b1, db); }
						const float sy = sinf(b1);
						nx = __fmul_rn(cosf(a1), sy); ny = __fmul_rn(sinf(a1), sy); nz = cosf(b1);
					}
				}
			}
		}
	}
	dd[o] = d;
	if (dn) { dn[o*3] = nx; dn[o*3+1] = ny; dn[o*3+2] = nz; }
	if (dc) dc[o] = c;
}

} // namespace

cudaError_t flt_launch_filter(const FltParams& P, int maxNbrPixels, bool adjust, cudaStream_t s) {
	const size_t np = (size_t)P.ref.w*P.ref.h;
	cudaError_t e = cudaMemsetAsync(P.zbuf, 0xFF, np*8*(size_t)P.N, s);
	if (e != cudaSuccess) return e;
	if (P.N > 0 && maxNbrPixels > 0)
		flt_project_kernel<<<dim3((maxNbrPixels+255)/256, P.N), 256, 0, s>>>(P);
	const unsigned nb = (unsigned)((np+255)/256);
	if (adjust) flt_adjust_kernel<<<nb, 256, 0, s>>>(P);
	else flt_strict_kernel<<<nb, 256, 0, s>>>(P);
	return cudaGetLastError();
}

cudaError_t flt_launch_resolve(const unsigned long long* z, const float* nbrConf, size_t np, float* depth, float* conf, cudaStream_t s) {
	flt_resolve_kernel<<<(unsigned)((np+255)/256), 256, 0, s>>>(z, nbrConf, np, depth, conf);
	return cudaGetLastError();
}

// phase 1: two-way components, their sizes / seed keys, the arcs; *count (device) receives the number of arcs found
cudaError_t seg_launch_label(const float* depth, int W, int H, float th, int* labels, int* sizes, int* minKey, void* arcs, int* count, int cap, cudaStream_t s) {
	const int n = W*H;
	const dim3 b2(32, 8), g2((W+31)/32, (H+7)/8);
	cudaMemsetAsync(count, 0, sizeof(int), s);
	seg_init_kernel<<<g2, b2, 0, s>>>(depth, labels, sizes, minKey, W, H, th);
	int rounds = 1;
	while ((1<<rounds) < W+H) ++rounds;
	for (int r = 0; r < rounds; ++r)
		seg_jump_kernel<<<(n+255)/256, 256, 0, s>>>(labels, n);
	seg_merge_kernel<<<g2, b2, 0, s>>>(depth, labels, W, H, th);
	for (int r = 0; r < rounds; ++r)
		seg_jump_kernel<<<(n+255)/256, 256, 0, s>>>(labels, n);
	seg_count_kernel<<<(n+255)/256, 256, 0, s>>>(labels, sizes, minKey, W, H);
	seg_arcs_kernel<<<g2, b2, 0, s>>>(depth, labels, sizes, minKey, W, H, th, (SegArc*)arcs, count, cap);
	return cudaGetLastError();
}
// phase 2: sizes of the components the arcs join replaced by the sizes of their breadth-first segments, then the removal
cudaError_t seg_launch_remove(float* depth, float* normal, float* conf, int W, int H, unsigned speckle, const int* labels, int* sizes,
	const int* patch, int nPatch, cudaStream_t s) {
	const int n = W*H;
	if (nPatch > 0) seg_patch_kernel<<<(nPatch+255)/256, 256, 0, s>>>((const int2*)patch, nPatch, sizes);
	seg_remove_kernel<<<(n+255)/256, 256, 0, s>>>(labels, sizes, n, speckle, depth, normal, conf);
	return cudaGetLastError();
}

// rows: (depth, normal, conf) -> tmp; columns: tmp -> (depth, normal, conf)
cudaError_t gap_launch(float* depth, float* normal, float* conf, float* tDepth, float* tNormal, float* tConf, int W, int H, float th, int gap, cudaStream_t s) {
	const dim3 g((W+255)/256, H);
	gap_kernel<0><<<g, 256, 0, s>>>(depth, normal, conf, tDepth, normal ? tNormal : nullptr, conf ? tConf : nullptr, W, H, th, gap);
	gap_kernel<1><<<g, 256, 0, s>>>(tDepth, normal ? tNormal : nullptr, conf ? tConf : nullptr, depth, normal, conf, W, H, th, gap);
	return cudaGetLastError();
}
