// capi.cu — host side of the C-ABI declared in include/b200mvs.h: device query, context lifecycle and settings.
// The estimation, matching and post-processing entry points are in pm_host.cu, sgm_host.cu, post_host.cu and fuse_host.cu.
#include "host_ctx.h"
#include "pm_common.cuh"
#include "sgm_common.cuh"

extern "C" {

int b200mvs_device_count(void) {
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
	return n;
}

void b200mvs_default_params(b200mvs_params* p) {
	p->nEstimationIters = 3; p->nEstimationGeometricIters = 2; p->nRandomIters = 6; p->nSubResolutionLevels = 2;
	p->fNCCThresholdKeep = 0.9f; p->fDescriptorMinMagnitudeThreshold = 0.02f;
	p->fRandomDepthRatio = 0.003f; p->fRandomAngle1Range = 16.f; p->fRandomAngle2Range = 10.f;
	p->fRandomSmoothDepth = 0.02f; p->fRandomSmoothNormal = 13.f; p->fRandomSmoothBonus = 0.93f;
	p->fEstimationGeometricWeight = 0.1f;
	p->nSweepsPerIter = 0; p->nPropagation = 4; p->seed = 1234u;
	p->nPropagationFar = 2; p->bSkipUnchanged = 1; p->nEvalCap = 0;
}

/* bumped whenever a struct of b200mvs.h changes layout; bindings compare it (and the struct sizes) at load time */
int b200mvs_abi_version(void) { return B200MVS_ABI_VERSION; }
size_t b200mvs_sizeof(int what) {
	switch (what) {
	case 0: return sizeof(b200mvs_view);
	case 1: return sizeof(b200mvs_params);
	case 2: return sizeof(b200mvs_stats);
	case 3: return sizeof(b200mvs_job);
	case 4: return sizeof(b200mvs_sgm_pixel);
	case 5: return sizeof(b200mvs_sgm_params);
	case 6: return sizeof(b200mvs_dmap);
	case 7: return sizeof(b200mvs_filter_params);
	case 8: return sizeof(b200mvs_debug);
	default: return 0;
	}
}

int b200mvs_create(int device, b200mvs_ctx** out) {
	if (!out) return B200MVS_ERR_ARG;
	*out = nullptr;
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0)
		return B200MVS_ERR_NOGPU; // never falls back to a CPU path
	if (device < 0) device = 0;
	if (device >= n) return B200MVS_ERR_ARG;
	if (cudaSetDevice(device) != cudaSuccess) return B200MVS_ERR_CUDA;
	b200mvs_ctx* c = new b200mvs_ctx();
	c->device = device;
	b200mvs_default_params(&c->prm);
	memset(&c->dbg, 0, sizeof(c->dbg));
	// dynamic shared memory opt-in of the kernels on this device (per-device attributes; idempotent, thread-safe)
	if (pm_configure_device() != cudaSuccess || sgm_configure_device() != cudaSuccess || sgm_cost_tc_configure() != cudaSuccess) { delete c; return B200MVS_ERR_CUDA; }
	if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
		cudaEventCreate(&c->ev0) != cudaSuccess || cudaEventCreate(&c->ev1) != cudaSuccess) {
		delete c;
		return B200MVS_ERR_CUDA;
	}
	*out = c;
	return B200MVS_OK;
}

int b200mvs_destroy(b200mvs_ctx* c) {
	if (!c) return B200MVS_ERR_ARG;
	cudaSetDevice(c->device);
	if (c->stream) cudaStreamSynchronize(c->stream); // an enqueued asynchronous call may still use the buffers
	for (auto e: c->sweepEv) cudaEventDestroy(e);
	for (int i = 0; i < 7; ++i) { if (c->sgSide[i]) cudaStreamDestroy(c->sgSide[i]); if (c->sgJoin[i]) cudaEventDestroy(c->sgJoin[i]); }
	if (c->sgFork) cudaEventDestroy(c->sgFork);
	if (c->ev0) cudaEventDestroy(c->ev0);
	if (c->ev1) cudaEventDestroy(c->ev1);
	if (c->stream) cudaStreamDestroy(c->stream);
	delete c; // frees the device buffers
	return B200MVS_OK;
}

int b200mvs_set_params(b200mvs_ctx* ctx, const b200mvs_params* p) {
	if (!ctx || !p) return B200MVS_ERR_ARG;
	if (p->nEstimationIters < 0 || p->nRandomIters < 0 || p->nSweepsPerIter < 0 || (p->nPropagation != 2 && p->nPropagation != 4) ||
		p->nPropagationFar < 0 || p->nPropagationFar > 3 || p->nEvalCap < 0 || p->nEvalCap > 15 || p->nSubResolutionLevels < 0 || !(p->fNCCThresholdKeep > 0))
		return fail(ctx, B200MVS_ERR_ARG, "invalid parameter block");
	ctx->prm = *p;
	return B200MVS_OK;
}

int b200mvs_set_debug(b200mvs_ctx* ctx, const b200mvs_debug* d) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (d) ctx->dbg = *d; else memset(&ctx->dbg, 0, sizeof(ctx->dbg));
	return B200MVS_OK;
}

int b200mvs_set_ignore_mask(b200mvs_ctx* ctx, const uint8_t* mask, int width, int height, int stride_bytes, int on_device) {
	if (!ctx) return B200MVS_ERR_ARG;
	if (!mask) { ctx->mask = nullptr; ctx->maskW = ctx->maskH = ctx->maskPitch = 0; return B200MVS_OK; }
	if (width <= 0 || height <= 0 || (stride_bytes != 0 && stride_bytes < width))
		return fail(ctx, B200MVS_ERR_ARG, "ignore-mask: invalid size or stride");
	if (stride_bytes == 0) stride_bytes = width;
	CK(cudaSetDevice(ctx->device));
	if (on_device) { ctx->mask = mask; ctx->maskPitch = stride_bytes; }
	else {
		CK(ctx->maskBuf.reserve((size_t)width*height));
		CK(cudaMemcpy2DAsync(ctx->maskBuf.p, width, mask, stride_bytes, width, height, cudaMemcpyHostToDevice, ctx->stream));
		CK(cudaStreamSynchronize(ctx->stream)); // the caller's buffer may be released after the call
		ctx->mask = ctx->maskBuf.as<uint8_t>(); ctx->maskPitch = width;
	}
	ctx->maskW = width; ctx->maskH = height;
	return B200MVS_OK;
}

const char* b200mvs_last_error(const b200mvs_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }

} // extern "C"
