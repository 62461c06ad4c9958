// resize_common.cuh — launch functions of the image-pyramid kernels (resize_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

cudaError_t rs_launch_area(const float* src, int sw, int sh, int spitch, float* dst, int dw, int dh, double scx, double scy, cudaStream_t s);
cudaError_t rs_launch_cubic(const float* src, int sw, int sh, int spitch, float* dst, int dw, int dh, int dpitch, double scx, double scy, cudaStream_t s);
cudaError_t rs_launch_nearest(const float* src, int sw, int sh, int ch, float* dst, int dw, int dh, double scx, double scy, cudaStream_t s);
cudaError_t rs_launch_nearest_u8(const uint8_t* src, int sw, int sh, int spitch, uint8_t* dst, int dw, int dh, cudaStream_t s);
cudaError_t rs_launch_to_gray(const uint8_t* src, int w, int h, int sstride, int channels, int bgr, float* dst, int dpitch, cudaStream_t s);
cudaError_t rs_launch_plane_up(const float4* src, int sw, int sh, float4* dst, float* prior, int dw, int dh, bool nearestDepth, cudaStream_t s);
