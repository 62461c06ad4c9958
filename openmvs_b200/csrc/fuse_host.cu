// fuse_host.cu — DepthMapsData::FuseDepthMaps behind the C-ABI (SURVEY.md §8(f) rank 4): the host form (host code over host
// arrays) and the host driver of the device form (kernels: fuse_kernels.cu).
//
// What it computes (libs/MVS/SceneDensify.cpp:1372-1646): all valid depth-maps are fused into one point cloud, the best
// connected images first and every pixel in raster order; a pixel that is not yet part of a point creates one, projects it
// into the neighbour depth-maps, merges the neighbour pixels whose depth (1 % relative) and normal (25 deg) agree — position,
// colour and normal are confidence-weighted means — drops the point when fewer than nMinViewsFuse views agree, and zeroes the
// neighbour depths that lie behind an accepted point (they would block its view).
//
// The result depends on the order — a neighbour pixel claimed by an earlier point is not available to a later one, and a zeroed
// depth changes what later pixels see — so the reference's sequential loop is the specification.  The host form is that loop,
// written for throughput: flat arrays, the projection matrices composed once, no per-point allocations.  The device form keeps
// the images sequential (one round per image) and resolves each round's pixels in parallel with the exact fixed point of
// fuse_kernels.cu (DESIGN.md §5.5); both take their arithmetic from fuse_common.cuh.
// The CPU restatement used by the tests is oracle/fuse_oracle.py (independent, plain Python loops).
#include <stdint.h>
#include <string.h>
#include <math.h>
#include <vector>
#include <algorithm>
#include <new>
#include "host_ctx.h"
#include "fuse_common.cuh"

namespace {

constexpr uint32_t NO_ID = 0xFFFFFFFFu;
using fuse::Cam;
using namespace fuse;

// the argument checks both forms make: map sizes and neighbour IDs; the device form also refuses a neighbour list that repeats an
// ID (the reference asserts it never does, SceneDensify.cpp:1557), because its rounds need at most one edge per point and target
const char* fuse_check(const b200mvs_fuse_view* views, int nViews, bool device) {
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (v.depth && (v.width <= 0 || v.height <= 0 || v.width > 65535 || v.height > 65535)) return "fuse: map size out of range";
		for (int k = 0; k < v.nNeighbors; ++k) {
			if (!v.neighbors || v.neighbors[k] >= (uint32_t)nViews || v.neighbors[k] == (uint32_t)i) return "fuse: invalid neighbour ID";
			if (device)
				for (int j = 0; j < k; ++j)
					if (v.neighbors[j] == v.neighbors[k]) return "fuse: repeated neighbour ID";
		}
	}
	return nullptr;
}

// what both forms derive from the views before fusing: the order of the images and the switches of the loop
struct FusePlan {
	std::vector<int> order;
	bool bNormalMap, bColor, bNormal;
	unsigned nMin;
	float normalError, thDepth;
};
// any[i]: image i has a depth-map with a depth > 0 in it
FusePlan fuse_plan(const b200mvs_fuse_view* views, int nViews, const b200mvs_fuse_params* prm, const std::vector<char>& any) {
	// best connected images first (SceneDensify.cpp:1392-1449); a view is valid when it has a depth-map with a depth in it.
	// std::sort's order among equal scores is unspecified in the reference: ties go to the lower index here.
	struct Conn { int idx; float score; };
	std::vector<Conn> conns;
	FusePlan p;
	p.bNormalMap = true;
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (!v.depth || v.nSceneNeighbors <= 0 || !any[i]) continue;
		conns.push_back(Conn{i, (float)v.nSceneNeighbors});
		if (!v.normal) p.bNormalMap = false;
	}
	std::stable_sort(conns.begin(), conns.end(), [](const Conn& a, const Conn& b) { return a.score > b.score; });
	for (const Conn& c: conns) p.order.push_back(c.idx);
	p.bColor = prm->bEstimateColor != 0;
	p.bNormal = prm->bEstimateNormal != 0 && p.bNormalMap;
	p.nMin = (unsigned)std::min(prm->nMinViewsFuse, nViews);
	p.normalError = cosf(prm->fNormalDiffThreshold*0.017453292519943295f);
	p.thDepth = prm->fDepthDiffThreshold;
	return p;
}

} // namespace

extern "C" {

void b200mvs_fuse_default_params(b200mvs_fuse_params* p) {
	p->nMinViewsFuse = 2; p->fDepthDiffThreshold = 0.01f; p->fNormalDiffThreshold = 25.f; p->bEstimateColor = 1; p->bEstimateNormal = 1;
}

int b200mvs_fuse_depth_maps(b200mvs_fuse_view* views, int nViews, const b200mvs_fuse_params* prm, b200mvs_pointcloud** out) {
	if (!views || nViews <= 0 || !out || fuse_check(views, nViews, false)) return B200MVS_ERR_ARG;
	b200mvs_fuse_params def; b200mvs_fuse_default_params(&def);
	if (!prm) prm = &def;
	b200mvs_pointcloud* pc = new (std::nothrow) b200mvs_pointcloud;
	if (!pc) return B200MVS_ERR_CUDA;
	std::vector<Cam> cams(nViews);
	for (int i = 0; i < nViews; ++i) compose(views[i].K, views[i].R, views[i].C, cams[i]);
	std::vector<char> any(nViews, 0);
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (!v.depth || v.nSceneNeighbors <= 0) continue;
		for (size_t k = 0, n = (size_t)v.width*v.height; k < n && !any[i]; ++k) any[i] = v.depth[k] > 0;
	}
	const FusePlan plan = fuse_plan(views, nViews, prm, any);
	const bool bColor = plan.bColor, bNormal = plan.bNormal, bNormalMap = plan.bNormalMap;
	const unsigned nMinViewsFuse = plan.nMin;
	const float normalError = plan.normalError, thDepth = plan.thDepth;
	std::vector<std::vector<uint32_t>> idxMaps(nViews);
	pc->offsets.push_back(0);
	// scratch of the point under construction (a point has at most 1 + nNeighbors views)
	std::vector<uint32_t> pv; std::vector<float> pw; std::vector<uint16_t> pp; std::vector<float*> invalid;
	for (const int a: plan.order) {
		b200mvs_fuse_view& A = views[a];
		const Cam& camA = cams[a];
		for (int k = 0; k < A.nNeighbors; ++k) {
			const uint32_t b = A.neighbors[k];
			if (idxMaps[b].empty() && views[b].depth) idxMaps[b].assign((size_t)views[b].width*views[b].height, NO_ID);
		}
		if (idxMaps[a].empty()) idxMaps[a].assign((size_t)A.width*A.height, NO_ID);
		uint32_t* idxA = idxMaps[a].data();
		for (int y = 0; y < A.height; ++y) {
			for (int x = 0; x < A.width; ++x) {
				const size_t ia = (size_t)y*A.width + x;
				const float depth = A.depth[ia];
				if (depth == 0) continue;
				++pc->nDepths;
				if (idxA[ia] != NO_ID) continue;
				const uint32_t idxPoint = (uint32_t)(pc->offsets.size()-1);
				idxA[ia] = idxPoint;
				double Xw[3];
				image_to_world(camA, x, y, depth, Xw);
				const float point[3] = {(float)Xw[0], (float)Xw[1], (float)Xw[2]};
				pv.assign(1, (uint32_t)a); pp.assign(2, 0); pp[0] = (uint16_t)x; pp[1] = (uint16_t)y;
				pw.assign(1, conf2weight(A.conf ? A.conf[ia] : 1.f, depth));
				double confidence = (double)pw[0];
				float normal[3] = {0.f, 0.f, -1.f};
				if (bNormalMap) normal_to_world(camA, A.normal+3*ia, normal);
				double X[3] = {mul_d((double)point[0], confidence), mul_d((double)point[1], confidence), mul_d((double)point[2], confidence)};
				float Cc[3] = {0.f, 0.f, 0.f};
				if (bColor && A.color) for (int c = 0; c < 3; ++c) Cc[c] = mul_f((float)A.color[3*ia+c], (float)confidence);
				float N[3] = {mul_f(normal[0], (float)confidence), mul_f(normal[1], (float)confidence), mul_f(normal[2], (float)confidence)};
				invalid.clear();
				for (int k = 0; k < A.nNeighbors; ++k) {
					const uint32_t b = A.neighbors[k];
					b200mvs_fuse_view& B = views[b];
					if (!B.depth) continue;
					const Cam& camB = cams[b];
					float pz; int xb, yb;
					if (!project_to_pixel(camB, point, B.width, B.height, pz, xb, yb)) continue;
					const size_t ib = (size_t)yb*B.width + xb;
					float& depthB = B.depth[ib];
					if (depthB == 0) continue;
					uint32_t& idxPointB = idxMaps[b][ib];
					if (idxPointB != NO_ID) continue;
					if (depth_similar(pz, depthB, thDepth)) {
						float normalB[3] = {0.f, 0.f, -1.f};
						if (bNormalMap) normal_to_world(camB, B.normal+3*ib, normalB);
						if (dot3(normal, normalB) > normalError) {
							const float confB = conf2weight(B.conf ? B.conf[ib] : 1.f, depthB);
							size_t pos = 0;                      // views stay sorted by image index (InsertSort)
							while (pos < pv.size() && pv[pos] < b) ++pos;
							pv.insert(pv.begin()+pos, b); pw.insert(pw.begin()+pos, confB);
							pp.insert(pp.begin()+2*pos, (uint16_t)yb); pp.insert(pp.begin()+2*pos, (uint16_t)xb);
							idxPointB = idxPoint;
							double Xb[3];
							image_to_world(camB, xb, yb, depthB, Xb);
							for (int c = 0; c < 3; ++c) X[c] = add_d(X[c], mul_d(Xb[c], (double)confB));
							if (bColor && B.color) for (int c = 0; c < 3; ++c) Cc[c] = add_f(Cc[c], mul_f((float)B.color[3*ib+c], confB));
							if (bNormal) for (int c = 0; c < 3; ++c) N[c] = add_f(N[c], mul_f(normalB[c], confB));
							confidence = add_d(confidence, (double)confB);
							continue;
						}
					}
					if (pz < depthB) invalid.push_back(&depthB);   // in front of the neighbour's estimate: that depth blocks the view
				}
				if (pv.size() < nMinViewsFuse) {
					for (size_t v = 0; v < pv.size(); ++v)
						idxMaps[pv[v]][(size_t)pp[2*v+1]*views[pv[v]].width + pp[2*v]] = NO_ID;
					continue;
				}
				const double nrm = div_d(1.0, confidence);
				for (int c = 0; c < 3; ++c) pc->points.push_back((float)mul_d(X[c], nrm));
				if (bColor && A.color) for (int c = 0; c < 3; ++c) pc->colors.push_back((uint8_t)mul_f(Cc[c], (float)nrm));
				if (bNormal) {
					const float n0 = mul_f(N[0], (float)nrm), n1 = mul_f(N[1], (float)nrm), n2 = mul_f(N[2], (float)nrm);
					const float len = sqrt_f(add_f(add_f(mul_f(n0, n0), mul_f(n1, n1)), mul_f(n2, n2)));
					pc->normals.push_back(div_f(n0, len)); pc->normals.push_back(div_f(n1, len)); pc->normals.push_back(div_f(n2, len));
				}
				pc->views.insert(pc->views.end(), pv.begin(), pv.end());
				pc->weights.insert(pc->weights.end(), pw.begin(), pw.end());
				pc->projs.insert(pc->projs.end(), pp.begin(), pp.end());
				pc->offsets.push_back((uint32_t)pc->views.size());
				for (float* d: invalid) *d = 0;
			}
		}
	}
	*out = pc;
	return B200MVS_OK;
}

} // extern "C"

namespace {

// grow a device buffer to `need` bytes, keeping its first `used` bytes (enqueued on s)
cudaError_t grow_keep(DevBuf& b, size_t used, size_t need, cudaStream_t s) {
	if (need <= b.cap) return cudaSuccess;
	DevBuf n;
	cudaError_t e = n.reserve(std::max(need, b.cap + b.cap/2));
	if (e == cudaSuccess && used) e = cudaMemcpyAsync(n.p, b.p, used, cudaMemcpyDeviceToDevice, s);
	if (e != cudaSuccess) return e;
	e = cudaStreamSynchronize(s);
	std::swap(b.p, n.p); std::swap(b.cap, n.cap);
	return e;
}

} // namespace

extern "C" {

int b200mvs_fuse_depth_maps_device(b200mvs_ctx* ctx, b200mvs_fuse_view* views, int nViews, const b200mvs_fuse_params* prm,
	b200mvs_pointcloud** out, void* stream, b200mvs_stats* stats)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!views || nViews <= 0 || !out) return fail(ctx, B200MVS_ERR_ARG, "fuse: null pointer");
	if (const char* why = fuse_check(views, nViews, true)) return fail(ctx, B200MVS_ERR_ARG, why);
	b200mvs_fuse_params def; b200mvs_fuse_default_params(&def);
	if (!prm) prm = &def;
	CK(cudaSetDevice(ctx->device));
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		if (!on_device(ctx, v.depth) || !on_device(ctx, v.normal) || !on_device(ctx, v.conf) || !on_device(ctx, v.color))
			return fail(ctx, B200MVS_ERR_ARG, "fuse: a map is not in device memory of the context's device");
	}
	// the view table, the claim maps and the neighbour lists with their round-local target bases
	std::vector<FuseDevView> dv(nViews);
	std::vector<size_t> claimOff(nViews, 0), nbOff(nViews+1, 0);
	size_t claimBytes = 0;
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		FuseDevView& d = dv[i];
		d.depth = v.depth; d.normal = v.normal; d.conf = v.conf; d.color = v.color; d.claim = nullptr;
		d.w = v.depth ? v.width : 0; d.h = v.depth ? v.height : 0;
		compose(v.K, v.R, v.C, d.cam);
		claimOff[i] = claimBytes; claimBytes += (size_t)d.w*d.h;
		nbOff[i+1] = nbOff[i] + v.nNeighbors;
	}
	std::vector<int> nbIds(nbOff[nViews]);
	std::vector<uint32_t> nbBase(nbOff[nViews]);
	for (int i = 0; i < nViews; ++i) {
		const b200mvs_fuse_view& v = views[i];
		uint64_t base = 0;
		for (int k = 0; k < v.nNeighbors; ++k) {
			nbIds[nbOff[i]+k] = (int)v.neighbors[k];
			nbBase[nbOff[i]+k] = (uint32_t)base;
			base += (uint64_t)dv[v.neighbors[k]].w*dv[v.neighbors[k]].h;
		}
		if (v.depth && (base >= 0xFFFFFFFFull || (uint64_t)v.width*v.height*(uint64_t)std::max(v.nNeighbors, 1) >= 0x7FFFFFFFull))
			return fail(ctx, B200MVS_ERR_ARG, "fuse: the maps of an image and its neighbours are too large for one round");
	}
	const auto t0 = std::chrono::steady_clock::now();
	cudaStream_t s = stream_of(ctx, stream);
	ctx->launches = 0;
	ctx->fsRounds.clear();
	// the call's scratch: the view table, the neighbour IDs and bases, the claim maps, which images have a depth, and the
	// candidate flags and list of a round, sized for the largest image a round can fuse
	size_t maxNp = 0;
	for (int i = 0; i < nViews; ++i) if (views[i].depth && views[i].nSceneNeighbors > 0) maxNp = std::max(maxNp, (size_t)dv[i].w*dv[i].h);
	Carve scratch(ctx->fsScratch);
	FuseDevView* dViews; int *dNb, *dAny; uint32_t *dBase, *cand; uint8_t *claim, *flags;
	scratch.take(dViews, nViews); scratch.take(dNb, nbIds.size()); scratch.take(dBase, nbBase.size());
	scratch.take(claim, std::max<size_t>(claimBytes, 1)); scratch.take(dAny, nViews); scratch.take(flags, maxNp); scratch.take(cand, maxNp);
	CK(scratch.commit());
	for (int i = 0; i < nViews; ++i) if (views[i].depth) dv[i].claim = claim + claimOff[i];
	ReadBack* rb; CK(read_back(ctx, rb));
	FuseCounters* cnt = &rb->fuse;
	CK(cudaEventRecord(ctx->ev0, s));
	CK(cudaMemcpyAsync(dViews, dv.data(), sizeof(FuseDevView)*nViews, cudaMemcpyHostToDevice, s));
	if (!nbIds.empty()) {
		CK(cudaMemcpyAsync(dNb, nbIds.data(), nbIds.size()*4, cudaMemcpyHostToDevice, s));
		CK(cudaMemcpyAsync(dBase, nbBase.data(), nbBase.size()*4, cudaMemcpyHostToDevice, s));
	}
	if (claimBytes) CK(cudaMemsetAsync(claim, 0, claimBytes, s));
	CK(cudaMemsetAsync(dAny, 0, sizeof(int)*nViews, s));
	CK(cudaMemsetAsync(cnt, 0, sizeof(FuseCounters), s));
	// which images have a depth > 0 (the host form's validity test), then the same order of the images as the host form
	for (int i = 0; i < nViews; ++i)
		if (views[i].depth && views[i].nSceneNeighbors > 0) {
			CK(fuse_launch_any_positive(views[i].depth, (size_t)views[i].width*views[i].height, dAny+i, s));
			++ctx->launches;
		}
	std::vector<int> anyI(nViews);
	CK(cudaMemcpyAsync(anyI.data(), dAny, sizeof(int)*nViews, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	uint64_t d2h = sizeof(int)*nViews;
	const FusePlan plan = fuse_plan(views, nViews, prm, std::vector<char>(anyI.begin(), anyI.end()));

	struct Events {
		cudaEvent_t b = nullptr, e = nullptr;
		~Events() { if (b) cudaEventDestroy(b); if (e) cudaEventDestroy(e); }
	} ev;
	CK(cudaEventCreate(&ev.b)); CK(cudaEventCreate(&ev.e));
	// the outputs grow with the rounds: points, normals, colors, offsets (per point), views, weights, projs (per view)
	DevBuf* O = ctx->fsOut;
	const size_t perPoint[4] = {12, 12, 3, 4}, perView[3] = {4, 4, 4};
	uint64_t nPts = 0, nVw = 0, nCol = 0, shared = 0;
	for (const int a: plan.order) {
		const b200mvs_fuse_view& A = views[a];
		const size_t np = (size_t)A.width*A.height;
		const int nNb = A.nNeighbors;
		FuseRound R;
		R.views = dViews; R.a = a; R.nNb = nNb; R.nb = dNb + nbOff[a]; R.base = dBase + nbOff[a];
		R.bNormalMap = plan.bNormalMap; R.bColor = plan.bColor; R.bNormal = plan.bNormal;
		R.nMin = plan.nMin; R.thDepth = plan.thDepth; R.normalError = plan.normalError;
		b200mvs_ctx::FuseRoundStat st{a, 0, 0, 0, 0, 0.f};
		CK(cudaEventRecord(ev.b, s));
		// the candidates: pixels with a depth and no claim, in raster order
		CK(fuse_launch_candidates(A.depth, dv[a].claim, np, flags, &cnt->nDepths, s));
		CK(cub_run(ctx->fsCub, [&](void* tmp, size_t& bytes) { return fuse_select(tmp, bytes, flags, cand, &cnt->nCand, np, s); }));
		ctx->launches += 2;
		uint32_t nCand = 0, nEdges = 0;
		CK(cudaMemcpyAsync(&nCand, &cnt->nCand, 4, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		d2h += 4;
		st.candidates = nCand;
		if (nCand > 0) {
			// the round's scratch, carved again by the next round (this one has finished when its events have): per candidate the
			// acceptance, the point flag, ID, view count and view offset; per (candidate, neighbour) edge its type, status and
			// target, the selected edges and their sort keys
			const size_t ne = (size_t)nCand*nNb;
			Carve round(ctx->fsRoundScratch);
			uint8_t *acc, *typ, *status; uint32_t *isPt, *ptId, *nv, *vOff, *tgt, *e1 = nullptr, *k1 = nullptr, *keys = nullptr, *edges = nullptr;
			round.take(acc, nCand); round.take(isPt, nCand); round.take(ptId, nCand); round.take(nv, nCand); round.take(vOff, nCand);
			round.take(typ, std::max<size_t>(ne, 1)); round.take(status, std::max<size_t>(ne, 1)); round.take(tgt, std::max<size_t>(ne, 1));
			if (ne > 0) { round.take(e1, ne); round.take(edges, ne); round.take(k1, ne); round.take(keys, ne); }
			CK(round.commit());
			CK(cudaMemsetAsync(acc, 0, nCand, s));
			if (ne > 0) {
				// the edges: type and target from the maps at the start of the round; the claim and zero edges, grouped by target in
				// raster order of their owners (the radix sort is stable and its input is in edge order)
				CK(fuse_launch_classify(R, cand, nCand, typ, tgt, s));
				CK(cub_run(ctx->fsCub, [&](void* tmp, size_t& bytes) { return fuse_select(tmp, bytes, typ, e1, &cnt->nEdges, ne, s); }));
				ctx->launches += 2;
				CK(cudaMemcpyAsync(&nEdges, &cnt->nEdges, 4, cudaMemcpyDeviceToHost, s));
				CK(cudaStreamSynchronize(s));
				d2h += 4;
				if (nEdges > 0) {
					int endBit = 1;
					while (endBit < 32 && (1ull << endBit) < (uint64_t)nbBase[nbOff[a]+nNb-1] + (uint64_t)dv[nbIds[nbOff[a]+nNb-1]].w*dv[nbIds[nbOff[a]+nNb-1]].h)
						++endBit;
					CK(fuse_launch_gather_keys(tgt, e1, nEdges, k1, s));
					CK(cub_run(ctx->fsCub, [&](void* tmp, size_t& bytes) { return fuse_sort(tmp, bytes, k1, keys, e1, edges, nEdges, endBit, s); }));
					CK(fuse_launch_shared(keys, nEdges, &cnt->shared, s));
					ctx->launches += 3;
				}
			}
			// the fixed point: every iteration decides at least the earliest undecided candidate
			for (uint32_t undecided = nCand, last = nCand + 1; undecided > 0; ) {
				if (undecided >= last) return fail(ctx, B200MVS_ERR_CUDA, "fuse: the acceptance fixed point made no progress");
				last = undecided;
				CK(cudaMemsetAsync(&cnt->undecided, 0, 4, s));
				if (nEdges > 0) { CK(fuse_launch_walk(keys, edges, nEdges, nNb, acc, status, s)); ++ctx->launches; }
				CK(fuse_launch_decide(R, nCand, typ, status, acc, &cnt->undecided, s));
				++ctx->launches;
				CK(cudaMemcpyAsync(&undecided, &cnt->undecided, 4, cudaMemcpyDeviceToHost, s));
				CK(cudaStreamSynchronize(s));
				d2h += 4;
				++st.iterations;
			}
			// a candidate can decide while some of its edges are still unknown: one more walk with every candidate decided makes
			// every edge live or dead, which the views of a point and its zeroed depths need
			if (nEdges > 0) { CK(fuse_launch_walk(keys, edges, nEdges, nNb, acc, status, s)); ++ctx->launches; }
			// point IDs and view offsets in raster order, then the points
			CK(fuse_launch_count(R, nCand, typ, status, acc, isPt, nv, s));
			CK(cub_run(ctx->fsCub, [&](void* tmp, size_t& bytes) { return fuse_scan(tmp, bytes, isPt, ptId, nCand, s); }));
			CK(cub_run(ctx->fsCub, [&](void* tmp, size_t& bytes) { return fuse_scan(tmp, bytes, nv, vOff, nCand, s); }));
			CK(fuse_launch_totals(isPt, ptId, nv, vOff, nCand, cnt->totals, s));
			ctx->launches += 4;
			FuseCounters hc;
			CK(cudaMemcpyAsync(&hc, cnt, sizeof(hc), cudaMemcpyDeviceToHost, s));
			CK(cudaStreamSynchronize(s));
			d2h += sizeof(hc);
			const uint64_t nP = hc.totals[0], nV = hc.totals[1];
			st.edges = nEdges; st.shared = hc.shared - shared; shared = hc.shared;
			if (nPts + nP + 1 >= 0xFFFFFFFFull || nVw + nV >= 0xFFFFFFFFull)
				return fail(ctx, B200MVS_ERR_ARG, "fuse: more than 2^32 points or views");
			const bool colorA = plan.bColor && A.color;
			if (nP > 0) {
				for (int i = 0; i < 4; ++i) {
					if ((i == 1 && !plan.bNormal) || (i == 2 && !colorA)) continue;
					const uint64_t used = i == 2 ? nCol : nPts;
					CK(grow_keep(O[i], used*perPoint[i], (used + nP + (i == 3))*perPoint[i], s));
				}
				for (int i = 0; i < 3; ++i) CK(grow_keep(O[4+i], nVw*perView[i], (nVw + nV)*perView[i], s));
				FuseOut fo;
				fo.points = O[0].as<float>() + 3*nPts; fo.normals = plan.bNormal ? O[1].as<float>() + 3*nPts : nullptr;
				fo.colors = colorA ? O[2].as<uint8_t>() + 3*nCol : nullptr; fo.offsets = O[3].as<uint32_t>() + nPts;
				fo.views = O[4].as<uint32_t>(); fo.weights = O[5].as<float>(); fo.projs = O[6].as<uint16_t>(); fo.viewBase = (uint32_t)nVw;
				CK(fuse_launch_assemble(R, cand, nCand, typ, tgt, status, acc, ptId, vOff, fo, s));
				++ctx->launches;
				nPts += nP; nVw += nV; nCol += colorA ? nP : 0;
			}
		}
		CK(cudaEventRecord(ev.e, s));
		CK(cudaEventSynchronize(ev.e));
		CK(cudaEventElapsedTime(&st.ms, ev.b, ev.e));
		ctx->fsRounds.push_back(st);
	}
	CK(cudaEventRecord(ctx->ev1, s));
	const DeviceCloud cloud{nPts, nVw, nCol, O[0].as<float>(), plan.bNormal ? O[1].as<float>() : nullptr, O[5].as<float>(),
		O[2].as<uint8_t>(), O[3].as<uint32_t>(), O[4].as<uint32_t>(), O[6].as<uint16_t>(), cnt};
	return read_cloud(ctx, "fuse: out of host memory", cloud, s, t0, d2h, stats, out);
}

int b200mvs_fuse_round_stats(b200mvs_ctx* ctx, int maxRounds, int* nRounds, int* image, int* iterations, uint64_t* candidates,
	uint64_t* edges, uint64_t* sharedEdges, float* ms)
{
	if (!ctx || maxRounds < 0 || !nRounds) return B200MVS_ERR_ARG;
	*nRounds = (int)ctx->fsRounds.size();
	for (int i = 0; i < std::min(maxRounds, *nRounds); ++i) {
		const b200mvs_ctx::FuseRoundStat& r = ctx->fsRounds[i];
		if (image) image[i] = r.image;
		if (iterations) iterations[i] = r.iterations;
		if (candidates) candidates[i] = r.candidates;
		if (edges) edges[i] = r.edges;
		if (sharedEdges) sharedEdges[i] = r.shared;
		if (ms) ms[i] = r.ms;
	}
	return B200MVS_OK;
}

uint64_t b200mvs_pointcloud_size(const b200mvs_pointcloud* pc) { return pc ? pc->offsets.size()-1 : 0; }
uint64_t b200mvs_pointcloud_depths(const b200mvs_pointcloud* pc) { return pc ? pc->nDepths : 0; }
const float* b200mvs_pointcloud_points(const b200mvs_pointcloud* pc) { return pc && !pc->points.empty() ? pc->points.data() : nullptr; }
const float* b200mvs_pointcloud_normals(const b200mvs_pointcloud* pc) { return pc && !pc->normals.empty() ? pc->normals.data() : nullptr; }
const uint8_t* b200mvs_pointcloud_colors(const b200mvs_pointcloud* pc) { return pc && !pc->colors.empty() ? pc->colors.data() : nullptr; }
const uint32_t* b200mvs_pointcloud_view_offsets(const b200mvs_pointcloud* pc) { return pc ? pc->offsets.data() : nullptr; }
const uint32_t* b200mvs_pointcloud_views(const b200mvs_pointcloud* pc) { return pc && !pc->views.empty() ? pc->views.data() : nullptr; }
const float* b200mvs_pointcloud_weights(const b200mvs_pointcloud* pc) { return pc && !pc->weights.empty() ? pc->weights.data() : nullptr; }
const uint16_t* b200mvs_pointcloud_projs(const b200mvs_pointcloud* pc) { return pc && !pc->projs.empty() ? pc->projs.data() : nullptr; }
void b200mvs_pointcloud_free(b200mvs_pointcloud* pc) { delete pc; }

} // extern "C"
