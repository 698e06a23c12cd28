// Keyframe image pyramids on the device: 16-byte texels (I, dI/dx, dI/dy, 0) so that one bilinear tap is one
// LDG.128. Either repacked from the reference's Eigen::Vector3f arrays (FrameHessian::dIp) or built on the device
// from the raw irradiance image exactly as FrameHessian::makeImages does (src/internal/FrameHessian.cc:44-98).
#pragma once
#include "common.cuh"

__global__ void k_repack_aos3(const float *__restrict__ src, float4 *__restrict__ dst, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    dst[i] = make_float4(src[3 * i], src[3 * i + 1], src[3 * i + 2], 0.f);
}

__global__ void k_unpack_aos3(const float4 *__restrict__ src, float *__restrict__ dst, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = src[i];
    dst[3 * i] = v.x; dst[3 * i + 1] = v.y; dst[3 * i + 2] = v.z;
}

// One launch per pyramid level: intensity (raw image at level 0, 2x2 box filter of level l-1 above) and the central
// differences of the same level over the flat index range [wl, wl*(hl-1)) (FrameHessian.cc:69-92; dx at a row border
// reads the neighbouring row's pixel exactly like the reference's flat indexing does). The four neighbours'
// intensities are recomputed with the same expression instead of being read back, so one launch per level suffices.
__device__ __forceinline__ float pyr_val(const float *__restrict__ color, const float4 *__restrict__ prev, int j, int wl, int wlm1) {
    if (prev == nullptr) return color[j];
    const int x = j % wl, y = j / wl;
    const float4 *b = prev + 2 * x + 2 * y * wlm1;
    return 0.25f * (b[0].x + b[1].x + b[wlm1].x + b[wlm1 + 1].x);
}
__global__ void k_pyr_level(const float *__restrict__ color, const float4 *__restrict__ prev, float4 *__restrict__ dst,
                            int wl, int hl, int wlm1) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= wl * hl) return;
    const float v = pyr_val(color, prev, idx, wl, wlm1);
    float dx = 0.f, dy = 0.f;
    if (idx >= wl && idx < wl * (hl - 1)) {
        dx = 0.5f * (pyr_val(color, prev, idx + 1, wl, wlm1) - pyr_val(color, prev, idx - 1, wl, wlm1));
        dy = 0.5f * (pyr_val(color, prev, idx + wl, wl, wlm1) - pyr_val(color, prev, idx - wl, wl, wlm1));
        if (isnan(dx) || fabsf(dx) > 255.0f) dx = 0;
        if (isnan(dy) || fabsf(dy) > 255.0f) dy = 0;
    }
    dst[idx] = make_float4(v, dx, dy, 0.f);
}

// absSquaredGrad[l][idx] as makeImages forms it (FrameHessian.cc:91-97) from a level-l texel: dx^2 + dy^2, times the square of
// CalibHessian::getBGradOnly(I) when B is given (nullptr = identity, setting_gammaWeightsPixelSelect = 1). Each product and sum is
// rounded on its own. On a pyramid built here (k_pyr_level) rows 0 and h_l-1, which makeImages never writes, give 0: their texels
// hold dx = dy = 0.
__device__ __forceinline__ float pyr_abs_sq_grad(const float4 *img, const float *B, int idx) {
    const float4 t = img[idx];
    float g = __fadd_rn(__fmul_rn(t.y, t.y), __fmul_rn(t.z, t.z));
    if (B) {
        int c = (int) __fadd_rn(t.x, 0.5f);            // CalibHessian::getBGradOnly
        if (c < 5) c = 5;
        if (c > 250) c = 250;
        const float gw = __fsub_rn(__ldg(B + c + 1), __ldg(B + c));
        g = __fmul_rn(g, __fmul_rn(gw, gw));
    }
    return g;
}
