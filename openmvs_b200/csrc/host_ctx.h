// host_ctx.h — the engine context behind the C-ABI (b200mvs_ctx) and the helpers shared by its host files: capi.cu (lifecycle
// and settings), pm_host.cu (PatchMatch), sgm_host.cu (SGM), post_host.cu (post-processing and image preparation).
// Internal to the library; include/b200mvs.h is the interface.
#pragma once
#include "../../include/b200mvs.h"
#include "sgm_front_sched.h"
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

// Grow-only device scratch that owns its memory: freed when the buffer (and so the context) is destroyed.  Move-only: the
// move constructor deletes the implicit copies.
struct DevBuf {
	void* p = nullptr; size_t cap = 0;
	DevBuf() = default;
	DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
	~DevBuf() { if (p) cudaFree(p); }
	cudaError_t reserve(size_t n) {
		if (n <= cap) return cudaSuccess;
		if (p) cudaFree(p);
		p = nullptr; cap = 0;
		cudaError_t e = cudaMalloc(&p, n);
		if (e == cudaSuccess) cap = n;
		return e;
	}
	template <typename T> T* as() const { return (T*)p; }
};

struct b200mvs_ctx {
	int device = 0;
	b200mvs_params prm;
	std::string err;
	cudaStream_t stream = nullptr;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	// grow-only device scratch
	std::vector<DevBuf> imgs, dmaps, img8;    // staged images / depth-maps / 8-bit colour images (host API; gray images converted on the device)
	std::vector<DevBuf> pyr;                  // per-view pyramid levels (all levels packed)
	DevBuf plane, cost, best, prior, lowPlane;
	DevBuf dDepth, dNormal, dConf, dViews;    // level scratch / staging of the maps (host API)
	DevBuf mapD, mapN;                        // full-resolution in/out maps (host API)
	DevBuf sgL, sgC, sgR, sgPx, sgCosts, sgAccums, sgAccums2, sgDisp, sgCost, sgMax; // SGM staging / scratch
	// wave-front aggregation: cached schedule of the last (size, mode) and its scratch
	struct FrontPass { FrontLaunch launch; DevBuf items, need; int nItems = 0; };   // launch.items is emptied once uploaded
	std::vector<FrontPass> sgFront; int sgFrontKey[6] = {0, 0, 0, 0, 0, 0};
	DevBuf sgFrontCtl, sgFrontState, sgFrontMeta;
	cudaStream_t sgSide[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // side streams of the ragged aggregation
	cudaEvent_t sgJoin[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, sgFork = nullptr;
	const void* sgLastPx = nullptr;           // pixel map of the volume in sgAccums (b200mvs_sgm_refine_device check)
	// hierarchical matcher: level images, masks, disparity maps, pixel maps, Disparity2RangeMap / FlipDirection / speckle scratch
	enum { TS_IMG, TS_MASKL, TS_MASKR, TS_MASKT, TS_DL, TS_DR, TS_DL0, TS_DR0, TS_PXL, TS_PXR, TS_RANGES, TS_SCAN, TS_KEYS, TS_LABELS,
		TS_SIZES, TS_SMALL, TS_COUNT };
	DevBuf ts[TS_COUNT];
	DevBuf fltZ, fltIn, fltOutD, fltOutC;     // FilterDepthMap: z-buffer keys, staged maps (host API), outputs
	DevBuf ppA, ppB, ppD, ppN, ppC;           // RemoveSmallSegments labels/sizes, GapInterpolation temporaries, staging
	DevBuf ppK, ppArcs, ppPatch;              // RemoveSmallSegments: seed keys, one-way edges (+ counter), patched segment sizes
	b200mvs_debug dbg;                        // diagnostic switches (b200mvs_set_debug); all zero = the shipped kernels
	const uint8_t* mask = nullptr; int maskW = 0, maskH = 0, maskPitch = 0; // ignore-mask of the reference view (device) or null
	DevBuf maskBuf, maskLevel;                // staged host mask, mask of the current pyramid level
	DevBuf refPad;                            // 16-byte aligned copy of a reference image whose pitch TMA cannot address
	CUtensorMap tmapRef;                      // descriptor of the current level's reference image
	bool tmapValid = false;
	std::vector<cudaEvent_t> sweepEv;         // event pairs around the sweep launches (stats only)
	int nSweepEv = 0; bool timeSweeps = false;
	int launches = 0;
	// state of an enqueued b200mvs_estimate_async call
	bool pending = false; uint64_t pendH2D = 0, pendD2H = 0; int pendLevels = 1;
	std::chrono::steady_clock::time_point t0;
};

inline int fail(b200mvs_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess) {
	if (c) {
		c->err = what;
		if (e != cudaSuccess) { c->err += ": "; c->err += cudaGetErrorString(e); }
	}
	return code;
}
#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail(ctx, B200MVS_ERR_CUDA, #call, _e); } while (0)

// the caller's stream, or the context's when it passes none
inline cudaStream_t stream_of(b200mvs_ctx* ctx, void* stream) { return stream ? (cudaStream_t)stream : ctx->stream; }

// The statistics every timed call reports.  ctx->ev0 and ctx->ev1 bracket the call's device work and have completed;
// t0 is the host clock at the start of the call.
inline int fill_stats(b200mvs_ctx* ctx, b200mvs_stats* stats, std::chrono::steady_clock::time_point t0, int levels,
	uint64_t h2d = 0, uint64_t d2h = 0)
{
	memset(stats, 0, sizeof(*stats));
	float ms = 0; CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
	stats->ms_device = ms;
	stats->ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now()-t0).count();
	stats->kernel_launches = ctx->launches; stats->levels = levels;
	stats->bytes_h2d = h2d; stats->bytes_d2h = d2h;
	return B200MVS_OK;
}
