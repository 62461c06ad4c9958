// post_host.cu — host side of the depth-map post-processing (FilterDepthMap, RemoveSmallSegments, GapInterpolation) and of the
// image preparation (toGray, ScaleImage) entry points of the C-ABI.
#include "host_ctx.h"
#include "filter_common.cuh"
#include "resize_common.cuh"

extern "C" {

// ---- depth-map post-processing (SceneDensify.cpp:810-1299) ----

void b200mvs_filter_default_params(b200mvs_filter_params* p) {
	p->nMinViews = 2; p->nMinViewsAdjust = 1; p->fDepthDiffThreshold = 0.01f; p->bAdjust = 1;
}

static void flt_view(const b200mvs_dmap& m, const float* depth, const float* conf, FltView& v) {
	v.depth = depth; v.conf = conf; v.w = m.width; v.h = m.height;
	v.fx = m.K[0]; v.fy = m.K[4]; v.cx = m.K[2]; v.cy = m.K[5];
	memcpy(v.R, m.R, sizeof(v.R)); memcpy(v.C, m.C, sizeof(v.C));
}

static int flt_check(b200mvs_ctx* ctx, const b200mvs_dmap* ref, const b200mvs_dmap* nbrs, int nNbrs, const b200mvs_filter_params* prm,
	const float* outDepth, const float* outConf)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!ref || !prm || !outDepth || !outConf || nNbrs < 0 || (nNbrs > 0 && !nbrs))
		return fail(ctx, B200MVS_ERR_ARG, "filter: null pointer");
	if (nNbrs > B200MVS_MAX_FILTER_VIEWS) return fail(ctx, B200MVS_ERR_ARG, "filter: too many neighbour depth-maps");
	if (!ref->depth || !ref->conf || ref->width <= 0 || ref->height <= 0 || (size_t)ref->width*ref->height >= 0xFFFFFFFFull)
		return fail(ctx, B200MVS_ERR_ARG, "filter: invalid reference depth-map");
	if (prm->nMinViews < 1 || prm->nMinViewsAdjust < 0 || !(prm->fDepthDiffThreshold > 0))
		return fail(ctx, B200MVS_ERR_ARG, "filter: invalid parameter block"); // nMinViewsFilter > 0 is asserted by the reference (:1057)
	for (int i = 0; i < nNbrs; ++i) {
		const b200mvs_dmap& m = nbrs[i];
		if (!m.depth || (prm->bAdjust && !m.conf) || m.width <= 0 || m.height <= 0 || (size_t)m.width*m.height >= 0xFFFFFFFFull)
			return fail(ctx, B200MVS_ERR_ARG, "filter: invalid neighbour depth-map");
	}
	return B200MVS_OK;
}

int b200mvs_filter_depth_map_device(b200mvs_ctx* ctx, const b200mvs_dmap* ref, const b200mvs_dmap* nbrs, int nNbrs,
	const b200mvs_filter_params* prm, float dMin, float dMax, float* outDepth, float* outConf,
	float* projDepth, float* projConf, int* filtered, void* stream)
{
	int rc = flt_check(ctx, ref, nbrs, nNbrs, prm, outDepth, outConf);
	if (rc) return rc;
	if (nNbrs < prm->nMinViews || nNbrs < prm->nMinViewsAdjust) { // "can not be filtered" (:1060-1063)
		if (filtered) *filtered = 0;
		return B200MVS_OK;
	}
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	const size_t np = (size_t)ref->width*ref->height;
	CK(ctx->fltZ.reserve(np*8*(size_t)nNbrs));
	FltParams P;
	memset(&P, 0, sizeof(P));
	flt_view(*ref, ref->depth, ref->conf, P.ref);
	int maxPix = 0;
	for (int i = 0; i < nNbrs; ++i) {
		flt_view(nbrs[i], nbrs[i].depth, nbrs[i].conf, P.nbr[i]);
		maxPix = std::max(maxPix, nbrs[i].width*nbrs[i].height);
	}
	P.N = nNbrs; P.nMinViews = prm->nMinViews; P.nMinViewsAdjust = prm->nMinViewsAdjust;
	P.thDepthDiff = prm->fDepthDiffThreshold*1.2f; P.thStrict = prm->fDepthDiffThreshold*0.8f;
	P.dMin = dMin; P.dMax = dMax;
	P.zbuf = ctx->fltZ.as<unsigned long long>(); P.outDepth = outDepth; P.outConf = outConf;
	CK(flt_launch_filter(P, maxPix, prm->bAdjust != 0, s));
	ctx->launches = 2;
	if (projDepth) {
		for (int i = 0; i < nNbrs; ++i)
			CK(flt_launch_resolve(P.zbuf+np*i, nbrs[i].conf, np, projDepth+np*i, projConf ? projConf+np*i : nullptr, s));
		ctx->launches += nNbrs;
	}
	if (filtered) *filtered = 1;
	return B200MVS_OK;
}

int b200mvs_filter_depth_map(b200mvs_ctx* ctx, const b200mvs_dmap* ref, const b200mvs_dmap* nbrs, int nNbrs,
	const b200mvs_filter_params* prm, float dMin, float dMax, float* outDepth, float* outConf, int* filtered, b200mvs_stats* stats)
{
	int rc = flt_check(ctx, ref, nbrs, nNbrs, prm, outDepth, outConf);
	if (rc) return rc;
	if (nNbrs < prm->nMinViews || nNbrs < prm->nMinViewsAdjust) { if (filtered) *filtered = 0; return B200MVS_OK; }
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = ctx->stream;
	const auto t0 = std::chrono::steady_clock::now();
	// stage every map once: [ref depth | ref conf | nbr0 depth | nbr0 conf | ...]
	size_t total = 0;
	for (int i = -1; i < nNbrs; ++i) { const b200mvs_dmap& m = i < 0 ? *ref : nbrs[i]; total += (size_t)m.width*m.height*2; }
	const size_t np = (size_t)ref->width*ref->height;
	CK(ctx->fltIn.reserve(total*4)); CK(ctx->fltOutD.reserve(np*4)); CK(ctx->fltOutC.reserve(np*4));
	std::vector<b200mvs_dmap> dv(nNbrs+1);
	float* p = ctx->fltIn.as<float>();
	uint64_t h2d = 0;
	for (int i = -1; i < nNbrs; ++i) {
		const b200mvs_dmap& m = i < 0 ? *ref : nbrs[i];
		const size_t n = (size_t)m.width*m.height;
		b200mvs_dmap& d = dv[i+1];
		d = m;
		CK(cudaMemcpyAsync(p, m.depth, n*4, cudaMemcpyHostToDevice, s)); d.depth = p; p += n; h2d += n*4;
		d.conf = nullptr;
		if (m.conf) { CK(cudaMemcpyAsync(p, m.conf, n*4, cudaMemcpyHostToDevice, s)); d.conf = p; h2d += n*4; }
		p += n;
	}
	CK(cudaEventRecord(ctx->ev0, s));
	rc = b200mvs_filter_depth_map_device(ctx, &dv[0], dv.data()+1, nNbrs, prm, dMin, dMax, ctx->fltOutD.as<float>(), ctx->fltOutC.as<float>(),
		nullptr, nullptr, filtered, s);
	if (rc) return rc;
	CK(cudaEventRecord(ctx->ev1, s));
	CK(cudaMemcpyAsync(outDepth, ctx->fltOutD.p, np*4, cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(outConf, ctx->fltOutC.p, np*4, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	if (stats) return fill_stats(ctx, stats, t0, 1, h2d, np*8);
	return B200MVS_OK;
}

int b200mvs_remove_small_segments_device(b200mvs_ctx* ctx, float* depth, float* normal, float* conf, int width, int height,
	float fDepthDiffThreshold, unsigned nSpeckleSize, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!depth || width <= 0 || height <= 0 || (size_t)width*height > 0x7FFFFFFFull || !(fDepthDiffThreshold > 0))
		return fail(ctx, B200MVS_ERR_ARG, "remove_small_segments: invalid argument");
	CK(cudaSetDevice(ctx->device));
	const size_t n = (size_t)width*height;
	cudaStream_t s = stream_of(ctx, stream);
	const float th = fDepthDiffThreshold*0.7f;
	const int cap = 1<<18;   // one-way edges kept (a 1080p map has tens); beyond it the call fails loudly
	CK(ctx->ppA.reserve(n*4)); CK(ctx->ppB.reserve(n*4)); CK(ctx->ppK.reserve(n*4));
	CK(ctx->ppArcs.reserve(sizeof(int)*4 + (size_t)cap*sizeof(SegArc)));
	int* count = ctx->ppArcs.as<int>();
	SegArc* arcs = (SegArc*)(ctx->ppArcs.as<int>()+4);
	CK(seg_launch_label(depth, width, height, th, ctx->ppA.as<int>(), ctx->ppB.as<int>(), ctx->ppK.as<int>(), arcs, count, cap, s));
	// the condensed graph is resolved on the host: one small read-back (the call synchronises the stream)
	int nArcs = 0;
	CK(cudaMemcpyAsync(&nArcs, count, sizeof(int), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	if (nArcs > cap) return fail(ctx, B200MVS_ERR_ARG, "remove_small_segments: too many direction-dependent edges in the depth-map");
	int nPatch = 0;
	if (nArcs > 0) {
		std::vector<SegArc> h(nArcs);
		CK(cudaMemcpyAsync(h.data(), arcs, (size_t)nArcs*sizeof(SegArc), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		// nodes: the components an arc touches; replay of the reference's loop (SceneDensify.cpp:828-895) on them
		struct Node { int label, size, key; std::vector<int> out; int seg = -1; };
		std::vector<Node> nodes;
		std::vector<std::pair<int, int>> index; // (label, node)
		auto node_of = [&](int label, int size, int key) {
			for (auto& p: index) if (p.first == label) return p.second;  // few nodes: linear search is fine ...
			index.push_back({label, (int)nodes.size()});
			Node nd; nd.label = label; nd.size = size; nd.key = key; nodes.push_back(nd);
			return (int)nodes.size()-1;
		};
		if (nArcs > 4096) {  // ... but not for pathological maps: sort once and search
			std::sort(h.begin(), h.end(), [](const SegArc& a, const SegArc& b) { return a.src != b.src ? a.src < b.src : a.dst < b.dst; });
		}
		std::vector<std::pair<int, int>> sortedIndex;
		if (nArcs > 4096) {
			std::vector<std::pair<int, std::pair<int, int>>> all; // label -> (size, key)
			for (auto& a: h) { all.push_back({a.src, {a.srcSize, a.srcKey}}); all.push_back({a.dst, {a.dstSize, a.dstKey}}); }
			std::sort(all.begin(), all.end());
			all.erase(std::unique(all.begin(), all.end(), [](const auto& x, const auto& y) { return x.first == y.first; }), all.end());
			for (auto& e: all) { Node nd; nd.label = e.first; nd.size = e.second.first; nd.key = e.second.second; sortedIndex.push_back({e.first, (int)nodes.size()}); nodes.push_back(nd); }
		}
		auto find_node = [&](int label, int size, int key) {
			if (sortedIndex.empty()) return node_of(label, size, key);
			return std::lower_bound(sortedIndex.begin(), sortedIndex.end(), std::make_pair(label, -1))->second;
		};
		for (auto& a: h) {
			const int u = find_node(a.src, a.srcSize, a.srcKey), v = find_node(a.dst, a.dstSize, a.dstKey);
			nodes[u].out.push_back(v);
		}
		std::vector<int> order(nodes.size());
		for (size_t i = 0; i < order.size(); ++i) order[i] = (int)i;
		std::sort(order.begin(), order.end(), [&](int a, int b) { return nodes[a].key < nodes[b].key; });
		std::vector<int> patch; std::vector<int> stack, members;
		for (int seed: order) {
			if (nodes[seed].seg >= 0) continue;
			// the segment grown from this seed: every unvisited component reachable along one-way edges
			long long total = 0;
			stack.assign(1, seed); members.clear(); nodes[seed].seg = seed;
			while (!stack.empty()) {
				const int u = stack.back(); stack.pop_back();
				members.push_back(u); total += nodes[u].size;
				for (int v: nodes[u].out) if (nodes[v].seg < 0) { nodes[v].seg = seed; stack.push_back(v); }
			}
			for (int u: members) { patch.push_back(nodes[u].label); patch.push_back((int)std::min<long long>(total, 0x7FFFFFFF)); }
		}
		nPatch = (int)patch.size()/2;
		CK(ctx->ppPatch.reserve(patch.size()*sizeof(int)));
		CK(cudaMemcpyAsync(ctx->ppPatch.p, patch.data(), patch.size()*sizeof(int), cudaMemcpyHostToDevice, s));
		CK(cudaStreamSynchronize(s)); // `patch` is a local
	}
	CK(seg_launch_remove(depth, normal, conf, width, height, nSpeckleSize, ctx->ppA.as<int>(), ctx->ppB.as<int>(), ctx->ppPatch.as<int>(), nPatch, s));
	{ int rounds = 1; while ((1<<rounds) < width+height) ++rounds; ctx->launches = 5+2*rounds+(nPatch > 0 ? 1 : 0); }
	return B200MVS_OK;
}

int b200mvs_gap_interpolation_device(b200mvs_ctx* ctx, float* depth, float* normal, float* conf, int width, int height,
	float fDepthDiffThreshold, unsigned nIpolGapSize, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!depth || width <= 0 || height <= 0 || (size_t)width*height > 0x7FFFFFFFull/3 || !(fDepthDiffThreshold > 0))
		return fail(ctx, B200MVS_ERR_ARG, "gap_interpolation: invalid argument");
	CK(cudaSetDevice(ctx->device));
	const size_t n = (size_t)width*height;
	CK(ctx->ppA.reserve(n*4)); CK(ctx->ppB.reserve(n*4)); CK(ctx->ppN.reserve(n*12));
	const int gap = (int)std::min<unsigned>(nIpolGapSize, (unsigned)std::max(width, height));
	CK(gap_launch(depth, normal, conf, ctx->ppA.as<float>(), ctx->ppN.as<float>(), ctx->ppB.as<float>(), width, height,
		fDepthDiffThreshold*2.5f, gap, stream_of(ctx, stream)));
	ctx->launches = 2;
	return B200MVS_OK;
}

// host form of the two in-place passes: stage, run, copy back
static int pp_host(b200mvs_ctx* ctx, int which, float* depth, float* normal, float* conf, int width, int height, float th, unsigned arg, b200mvs_stats* stats) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!depth || width <= 0 || height <= 0) return fail(ctx, B200MVS_ERR_ARG, "post-processing: invalid argument");
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = ctx->stream;
	const auto t0 = std::chrono::steady_clock::now();
	const size_t n = (size_t)width*height;
	CK(ctx->ppD.reserve(n*4+n*12)); CK(ctx->ppC.reserve(n*4));
	float* dD = ctx->ppD.as<float>(); float* dN = normal ? dD+n : nullptr; float* dC = conf ? ctx->ppC.as<float>() : nullptr;
	CK(cudaMemcpyAsync(dD, depth, n*4, cudaMemcpyHostToDevice, s));
	if (normal) CK(cudaMemcpyAsync(dN, normal, n*12, cudaMemcpyHostToDevice, s));
	if (conf) CK(cudaMemcpyAsync(dC, conf, n*4, cudaMemcpyHostToDevice, s));
	CK(cudaEventRecord(ctx->ev0, s));
	const int rc = which == 0 ? b200mvs_remove_small_segments_device(ctx, dD, dN, dC, width, height, th, arg, s)
		: b200mvs_gap_interpolation_device(ctx, dD, dN, dC, width, height, th, arg, s);
	if (rc) return rc;
	CK(cudaEventRecord(ctx->ev1, s));
	CK(cudaMemcpyAsync(depth, dD, n*4, cudaMemcpyDeviceToHost, s));
	if (normal) CK(cudaMemcpyAsync(normal, dN, n*12, cudaMemcpyDeviceToHost, s));
	if (conf) CK(cudaMemcpyAsync(conf, dC, n*4, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	const uint64_t b = n*4+(normal ? n*12 : 0)+(conf ? n*4 : 0);
	if (stats) return fill_stats(ctx, stats, t0, 1, b, b);
	return B200MVS_OK;
}

int b200mvs_remove_small_segments(b200mvs_ctx* ctx, float* depth, float* normal, float* conf, int width, int height,
	float fDepthDiffThreshold, unsigned nSpeckleSize, b200mvs_stats* stats)
{
	return pp_host(ctx, 0, depth, normal, conf, width, height, fDepthDiffThreshold, nSpeckleSize, stats);
}

int b200mvs_gap_interpolation(b200mvs_ctx* ctx, float* depth, float* normal, float* conf, int width, int height,
	float fDepthDiffThreshold, unsigned nIpolGapSize, b200mvs_stats* stats)
{
	return pp_host(ctx, 1, depth, normal, conf, width, height, fDepthDiffThreshold, nIpolGapSize, stats);
}

// ---- image preparation (SURVEY §8f rank 3): toGray on the device ----
int b200mvs_to_gray_device(b200mvs_ctx* ctx, const uint8_t* image, int width, int height, int stride_bytes, int channels, int bgr,
	float* gray, int gray_stride_bytes, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!image || !gray || width <= 0 || height <= 0 || (channels != 3 && channels != 4))
		return fail(ctx, B200MVS_ERR_ARG, "to_gray: null pointer, empty image or channel count other than 3 / 4");
	if (stride_bytes == 0) stride_bytes = width*channels;
	if (gray_stride_bytes == 0) gray_stride_bytes = width*4;
	if (stride_bytes < width*channels || gray_stride_bytes < width*4 || (gray_stride_bytes & 3))
		return fail(ctx, B200MVS_ERR_ARG, "to_gray: invalid stride");
	CK(cudaSetDevice(ctx->device));
	CK(rs_launch_to_gray(image, width, height, stride_bytes, channels, bgr != 0, gray, gray_stride_bytes/4, stream_of(ctx, stream)));
	ctx->launches = 1;
	return B200MVS_OK;
}

// DepthData::ViewData::ScaleImage (libs/MVS/DepthMap.h:193-203): a neighbour whose footprint differs from the reference's by
// 15 % or more is resampled by `scale` — cv::resize(image, Size(), scale, scale, scale > 1 ? INTER_CUBIC : INTER_AREA)
int b200mvs_scaled_size(int width, int height, float scale, int* scaledWidth, int* scaledHeight) {
	if (!scaledWidth || !scaledHeight || width <= 0 || height <= 0 || !(scale > 0)) return B200MVS_ERR_ARG;
	// cv::resize with dsize = Size(): saturate_cast<int>(src.cols * fx) = cvRound
	*scaledWidth = (int)std::nearbyint(width*(double)scale); *scaledHeight = (int)std::nearbyint(height*(double)scale);
	return B200MVS_OK;
}
int b200mvs_scale_image_device(b200mvs_ctx* ctx, const float* image, int width, int height, int stride_bytes, float scale,
	float* scaled, int* applied, void* stream)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!image || !scaled || width <= 0 || height <= 0 || !(scale > 0) || (stride_bytes & 3))
		return fail(ctx, B200MVS_ERR_ARG, "scale_image: null pointer, empty image, scale <= 0 or stride not a multiple of 4");
	if (applied) *applied = 0;
	if (std::fabs(scale-1.f) < 0.15f) return B200MVS_OK;  // !NeedScaleImage: the caller keeps the image and its camera
	int dw, dh; b200mvs_scaled_size(width, height, scale, &dw, &dh);
	if (dw <= 0 || dh <= 0) return fail(ctx, B200MVS_ERR_ARG, "scale_image: scaled image is empty");
	CK(cudaSetDevice(ctx->device));
	cudaStream_t s = stream_of(ctx, stream);
	const int pitch = stride_bytes ? stride_bytes/4 : width;
	const double inv = 1.0/(double)scale;
	if (scale > 1.f) CK(rs_launch_cubic(image, width, height, pitch, scaled, dw, dh, dw, inv, inv, s));
	else CK(rs_launch_area(image, width, height, pitch, scaled, dw, dh, inv, inv, s));
	ctx->launches = 1;
	if (applied) *applied = 1;
	return B200MVS_OK;
}

} // extern "C"
