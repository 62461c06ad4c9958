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
	Carve scratch(ctx->ppScratch);
	scratch.take(P.zbuf, np*nNbrs);   // z-buffer keys
	CK(scratch.commit());
	P.outDepth = outDepth; P.outConf = outConf;
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
	HostCall call(ctx);
	std::vector<b200mvs_dmap> dv(ref, ref+1);   // the reference, then the neighbours, with staged maps
	dv.insert(dv.end(), nbrs, nbrs+nNbrs);
	for (b200mvs_dmap& d: dv) {
		const size_t bytes = (size_t)d.width*d.height*sizeof(float);
		call.in(d.depth, d.depth, bytes);
		if (d.conf) call.in(d.conf, d.conf, bytes);
	}
	const size_t np = (size_t)ref->width*ref->height;
	float *dOutD, *dOutC;
	call.out(dOutD, outDepth, np*sizeof(float)); call.out(dOutC, outConf, np*sizeof(float));
	if ((rc = call.stage())) return rc;
	return call.run([&](cudaStream_t s) {
		return b200mvs_filter_depth_map_device(ctx, &dv[0], dv.data()+1, nNbrs, prm, dMin, dMax, dOutD, dOutC, nullptr, nullptr, filtered, s);
	}, stats);
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
	// labels, segment sizes, seed keys, the one-way edges and the patched segment sizes: (label, size) of each of the at most
	// 2 cap components the edges touch
	Carve scratch(ctx->ppScratch);
	int *labels, *sizes, *keys, *patched; SegArc* arcs;
	scratch.take(labels, n); scratch.take(sizes, n); scratch.take(keys, n); scratch.take(arcs, cap); scratch.take(patched, 4*(size_t)cap);
	CK(scratch.commit());
	ReadBack* rb; CK(read_back(ctx, rb));
	int* count = &rb->nArcs;
	int launches = 0;
	CK(seg_launch_label(depth, width, height, th, labels, sizes, keys, arcs, count, cap, launches, s));
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
		// nodes: the components an arc touches, sorted by label; replay of the reference's loop (SceneDensify.cpp:828-895) on them
		struct Node { int label, size, key; std::vector<int> out; int seg = -1; };
		std::vector<Node> nodes;
		for (const SegArc& a: h) { nodes.push_back({a.src, a.srcSize, a.srcKey}); nodes.push_back({a.dst, a.dstSize, a.dstKey}); }
		std::sort(nodes.begin(), nodes.end(), [](const Node& x, const Node& y) { return x.label < y.label; });
		nodes.erase(std::unique(nodes.begin(), nodes.end(), [](const Node& x, const Node& y) { return x.label == y.label; }), nodes.end());
		auto node_of = [&](int label) {
			return (int)(std::lower_bound(nodes.begin(), nodes.end(), label, [](const Node& x, int l) { return x.label < l; })-nodes.begin());
		};
		for (const SegArc& a: h) nodes[node_of(a.src)].out.push_back(node_of(a.dst));
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
		CK(cudaMemcpyAsync(patched, patch.data(), patch.size()*sizeof(int), cudaMemcpyHostToDevice, s));
		CK(cudaStreamSynchronize(s)); // `patch` is a local
	}
	CK(seg_launch_remove(depth, normal, conf, width, height, nSpeckleSize, labels, sizes, patched, nPatch, launches, s));
	ctx->launches = launches;
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
	Carve scratch(ctx->ppScratch);
	float *tDepth, *tNormal, *tConf;
	scratch.take(tDepth, n); scratch.take(tNormal, 3*n); scratch.take(tConf, n);
	CK(scratch.commit());
	const int gap = (int)std::min<unsigned>(nIpolGapSize, (unsigned)std::max(width, height));
	CK(gap_launch(depth, normal, conf, tDepth, tNormal, tConf, width, height, fDepthDiffThreshold*2.5f, gap, stream_of(ctx, stream)));
	ctx->launches = 2;
	return B200MVS_OK;
}

// host form of the two in-place passes: stage the maps, run the device form on them, copy them back
typedef int (*PPDeviceForm)(b200mvs_ctx*, float*, float*, float*, int, int, float, unsigned, void*);
static int pp_host(b200mvs_ctx* ctx, PPDeviceForm form, float* depth, float* normal, float* conf, int width, int height, float th, unsigned arg,
	b200mvs_stats* stats)
{
	if (!ctx) return B200MVS_ERR_ARG;
	if (!depth || width <= 0 || height <= 0) return fail(ctx, B200MVS_ERR_ARG, "post-processing: invalid argument");
	CK(cudaSetDevice(ctx->device));
	HostCall call(ctx);
	const size_t n = (size_t)width*height;
	float *dD, *dN = nullptr, *dC = nullptr;
	call.inout(dD, depth, n*sizeof(float));
	if (normal) call.inout(dN, normal, n*3*sizeof(float));
	if (conf) call.inout(dC, conf, n*sizeof(float));
	if (int rc = call.stage()) return rc;
	return call.run([&](cudaStream_t s) { return form(ctx, dD, dN, dC, width, height, th, arg, s); }, stats);
}

int b200mvs_remove_small_segments(b200mvs_ctx* ctx, float* depth, float* normal, float* conf, int width, int height,
	float fDepthDiffThreshold, unsigned nSpeckleSize, b200mvs_stats* stats)
{
	return pp_host(ctx, b200mvs_remove_small_segments_device, depth, normal, conf, width, height, fDepthDiffThreshold, nSpeckleSize, stats);
}

int b200mvs_gap_interpolation(b200mvs_ctx* ctx, float* depth, float* normal, float* conf, int width, int height,
	float fDepthDiffThreshold, unsigned nIpolGapSize, b200mvs_stats* stats)
{
	return pp_host(ctx, b200mvs_gap_interpolation_device, depth, normal, conf, width, height, fDepthDiffThreshold, nIpolGapSize, stats);
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
