// host_ctx.h — the engine context behind the C-ABI (b200mvs_ctx) and the helpers shared by its host files: capi.cu (lifecycle
// and settings), pm_host.cu (PatchMatch), sgm_host.cu (SGM), post_host.cu (post-processing and image preparation), fuse_host.cu
// (FuseDepthMaps), cloud_host.cu (MergeDepthMaps, point colours and normals).
// Internal to the library; include/b200mvs.h is the interface.
//
// Device scratch is owned by subsystem: the context keeps one arena per subsystem, and each entry point carves all of its
// temporaries from its arena once, before its first launch (Carve), so no pointer it hands a kernel moves during the call.
// The few words the host reads back before it can size a carve sit in one small block (ReadBack, read_back); the other
// device buffers of the context are state that outlives a call.
#pragma once
#include "../../include/b200mvs.h"
#include "sgm_common.cuh"
#include "sgm_front_sched.h"
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

// Grow-only device memory that owns its allocation: freed when the buffer (and so the context) is destroyed.  Move-only: the
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

// One call's scratch carved from an arena: take() declares each slice with the pointer it sets, commit() reserves the total
// once and only then sets the pointers, each 256-byte aligned as cudaMalloc's.  A carve's pointers stay valid until its arena
// is carved again, so an entry point commits once, before its first launch, and calls that nest carve different arenas.
struct Carve {
	explicit Carve(DevBuf& arena) : arena(arena) {}
	template <typename T> void take(T*& p, size_t n) { take_bytes(&p, n*sizeof(T)); }
	void take_bytes(void* ptrAddr, size_t bytes) { slices.push_back({ptrAddr, bytes, 0}); }
	bool empty() const { return slices.empty(); }
	cudaError_t commit() {
		size_t total = 0;
		for (Slice& s: slices) { s.off = total; total += (s.bytes+255) & ~(size_t)255; }
		const cudaError_t e = arena.reserve(total);
		if (e != cudaSuccess) return e;
		for (Slice& s: slices) { void* p = arena.as<uint8_t>()+s.off; memcpy(s.ptrAddr, &p, sizeof(p)); }
		return cudaSuccess;
	}
private:
	struct Slice { void* ptrAddr; size_t bytes, off; };
	DevBuf& arena;
	std::vector<Slice> slices;
};

// FuseDepthMaps (device form): the counters of one call
struct FuseCounters {
	unsigned long long nDepths, shared;
	uint32_t nCand, nEdges, undecided, totals[2];
};

// The device words the host reads back before it can size a call's scratch, one field per user (read_back)
struct ReadBack {
	SGMMapStats mapStats;                     // SGM match: statistics of the pixel map
	unsigned long long rangeTotal;            // tSGM range map: the size of the volume
	int minMax[2];                            // tSGM without levels: the disparity range of the initial map
	int nArcs;                                // RemoveSmallSegments: one-way edges between segments
	FuseCounters fuse;                        // FuseDepthMaps (device form)
	unsigned long long mergePoints;           // MergeDepthMaps (device form): the number of points
	int cloudBad;                             // point colours / normals / k-NN: what the checks found (CLOUD_* bits)
	unsigned cloudBox[6];                     // point normals / k-NN: bounding box as ordered keys (box_key, cloud_common.cuh)
	float cloudSample[3*1024];                // point normals / k-NN: the points the grid's extent is estimated from (CLOUD_SAMPLE)
};

// PointCloud as the fusion and the merge return it (b200mvs_pointcloud accessors)
struct b200mvs_pointcloud {
	std::vector<float> points, normals, weights;
	std::vector<uint8_t> colors;
	std::vector<uint32_t> views, offsets;   // views / weights of point i: [offsets[i], offsets[i+1])
	std::vector<uint16_t> projs;            // pixel (x, y) of every view of every point, parallel to `views`
	uint64_t nDepths = 0;
};

struct b200mvs_ctx {
	int device = 0;
	b200mvs_params prm;
	std::string err;
	cudaStream_t stream = nullptr;
	cudaEvent_t ev0 = nullptr, ev1 = nullptr;
	// scratch arenas
	DevBuf stage;                             // the host forms' staged inputs and outputs (HostCall)
	DevBuf pmScratch;                         // PatchMatch estimate and building blocks
	DevBuf sgmScratch;                        // SGM match
	DevBuf tsgmScratch;                       // hierarchical (tSGM) level loop and its building blocks
	DevBuf sfScratch;                         // SGM fusion and the normal map
	DevBuf ppScratch;                         // post-processing: filter, small segments, gap interpolation
	DevBuf fsScratch, fsRoundScratch;         // FuseDepthMaps (device form): the call, and one round of it
	DevBuf pcScratch, pcCub;                  // MergeDepthMaps, point colours / normals, k-NN: the call, and CUB's temporary storage
	DevBuf pcOut;                             // MergeDepthMaps (device form): the point cloud before its read-back
	ReadBack* words = nullptr;                // allocated on first use, never moved
	// wave-front aggregation: the schedule of the last valid-region size vw x vh, uploaded (launch.items is emptied then)
	struct FrontSchedule { int vw = 0, vh = 0; FrontLaunch launch; DevBuf items, need; int nItems = 0; };
	FrontSchedule sgFront;
	cudaStream_t sgSide[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // side streams of the ragged aggregation
	cudaEvent_t sgJoin[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr}, sgFork = nullptr;
	// the accumulated costs of the last SGM match in its own scratch, and their pixel map (b200mvs_sgm_refine_device check)
	const uint16_t* sgLastAccums = nullptr; const void* sgLastPx = nullptr;
	// FuseDepthMaps (device form): CUB's temporary storage, the growing point-cloud outputs, and what each round of the last call
	// did (b200mvs_fuse_round_stats)
	DevBuf fsCub;
	DevBuf fsOut[7];                          // points, normals, colors, offsets, views, weights, projs
	struct FuseRoundStat { int image, iterations; uint64_t candidates, edges, shared; float ms; };
	std::vector<FuseRoundStat> fsRounds;
	b200mvs_debug dbg;                        // diagnostic switches (b200mvs_set_debug); all zero = the shipped kernels
	const uint8_t* mask = nullptr; int maskW = 0, maskH = 0, maskPitch = 0; // ignore-mask of the reference view (device) or null
	DevBuf maskBuf;                           // staged host mask
	CUtensorMap tmapRef;                      // descriptor of the current level's reference image
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

// The context's read-back block, allocated by the first call that needs it (a small allocation takes a page of its own)
inline cudaError_t read_back(b200mvs_ctx* ctx, ReadBack*& words) {
	if (!ctx->words) {
		void* p = nullptr;
		if (cudaError_t e = cudaMalloc(&p, sizeof(ReadBack))) return e;
		ctx->words = (ReadBack*)p;
	}
	words = ctx->words;
	return cudaSuccess;
}

// map pointers of a device form must be device (or managed) memory of the context's device
inline bool on_device(const b200mvs_ctx* ctx, const void* p) {
	if (!p) return true;
	cudaPointerAttributes a;
	if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
	return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == ctx->device;
}

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

// One call of a host form on ctx->stream: the caller's host buffers are staged in the context's device arena (ctx->stage), the
// device form runs between ctx->ev0 and ctx->ev1, and the outputs are copied back.  Declare every buffer with in / out / inout,
// each with the device pointer the call should set; stage() sets them and enqueues the H2D copies; run() then does the rest and
// waits, or enqueue() leaves it pending for b200mvs_sync.  bytes_h2d / bytes_d2h are the bytes copied.
struct HostCall {
	b200mvs_ctx* ctx;
	const std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
	uint64_t h2d = 0, d2h = 0;
	bool formRecordsEvents = false;   // the device form records ev0 / ev1 itself (b200mvs_sgm_match_device with statistics)

	explicit HostCall(b200mvs_ctx* c) : ctx(c), carve(c->stage) {}
	// `rows` rows of `row` bytes, `pitch` bytes apart on the host (0: packed); packed on the device
	template <typename T> void in(T*& dev, const void* host, size_t row, int rows = 1, size_t pitch = 0) {
		add(&dev, host, nullptr, row, rows, pitch ? pitch : row);
	}
	template <typename T> void out(T*& dev, void* host, size_t bytes) { add(&dev, nullptr, host, bytes, 1, bytes); }
	template <typename T> void inout(T*& dev, void* host, size_t bytes) { add(&dev, host, host, bytes, 1, bytes); }

	int stage() {
		CK(carve.commit());
		for (Copy& c: copies) {
			memcpy(&c.p, c.dev, sizeof(c.p));
			if (!c.src) continue;
			if (c.pitch == c.row) CK(cudaMemcpyAsync(c.p, c.src, c.row*c.rows, cudaMemcpyHostToDevice, ctx->stream));
			else CK(cudaMemcpy2DAsync(c.p, c.row, c.src, c.pitch, c.row, c.rows, cudaMemcpyHostToDevice, ctx->stream));
			h2d += c.row*c.rows;
		}
		return B200MVS_OK;
	}
	// form(stream) is the device form on the staged buffers
	template <typename F> int run(F&& form, b200mvs_stats* stats) {
		if (int rc = launch(form)) return rc;
		CK(cudaStreamSynchronize(ctx->stream));
		return stats ? fill_stats(ctx, stats, t0, 1, h2d, d2h) : B200MVS_OK;
	}
	template <typename F> int enqueue(F&& form, int levels) {
		if (int rc = launch(form)) return rc;
		ctx->t0 = t0; ctx->pendH2D = h2d; ctx->pendD2H = d2h; ctx->pendLevels = levels;
		ctx->pending = true;
		return B200MVS_OK;
	}

private:
	// one staged buffer: the caller's device pointer (set by stage(), copied to p) and its host side
	struct Copy { void* dev; void* p; const void* src; void* dst; size_t row, pitch; int rows; };
	Carve carve;
	std::vector<Copy> copies;

	void add(void* dev, const void* src, void* dst, size_t row, int rows, size_t pitch) {
		carve.take_bytes(dev, row*rows);
		copies.push_back({dev, nullptr, src, dst, row, pitch, rows});
	}
	template <typename F> int launch(F& form) {
		if (!formRecordsEvents) CK(cudaEventRecord(ctx->ev0, ctx->stream));
		if (int rc = form(ctx->stream)) return rc;
		if (!formRecordsEvents) CK(cudaEventRecord(ctx->ev1, ctx->stream));
		for (const Copy& c: copies) {
			if (!c.dst) continue;
			CK(cudaMemcpyAsync(c.dst, c.p, c.row, cudaMemcpyDeviceToHost, ctx->stream));
			d2h += c.row;
		}
		return B200MVS_OK;
	}
};
