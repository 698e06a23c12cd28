// Per-frame undistortion on the device: LDSO's PhotometricUndistorter::processFrame<T> (src/frontend/Undistort.cc:189-227) and
// Undistort::undistort<T>'s bilinear remap onto the rectified pinhole grid (Undistort.cc:357-457) in one kernel. Each thread
// writes one rectified pixel; each of its four taps is the photometric value of one raw pixel, computed on the fly from the raw
// 8- / 16-bit frame exactly as processFrame would have stored it, so the float image of the raw frame is never formed.
// Every product and sum is rounded on its own (__fmul_rn / __fadd_rn / __fsub_rn): nvcc contracts nothing into an FMA, and the
// result is the reference's expression evaluated in IEEE float, term by term, in the reference's order.
//
// Edge rule: the reference's range check (src_offset > (hOrg-1)*wOrg) lets through two offsets whose taps lie past the end of
// the image, src_offset == (hOrg-1)*wOrg (taps +wOrg, +1+wOrg) and (hOrg-1)*wOrg - 1 (tap +1+wOrg); the reference reads beyond
// its buffer there. Here any tap at index >= wOrg*hOrg reads 0. The raw frame is staged with wOrg + 1 zero pixels behind it so
// that no tap address leaves the buffer. A tap at xxi = wOrg-1 wraps to the next row, as the reference's linear indexing does.
#pragma once
#include "common.cuh"

struct UndistortArgs {
    const float2 *remap;        // (remapX, remapY) per rectified pixel; nullptr = passthrough (wOrg == w, hOrg == h)
    const float *G;             // inverse response, g_entries floats; nullptr = no valid calibration
    const float *vinv;          // vignetteMapInv, wOrg*hOrg floats (read in mode 2)
    int wOrg, hOrg, w, h;
    int use_G;                  // G valid && exposure > 0 && mode != 0 (processFrame's branch), decided on the host per frame
    int mode2;                  // multiply by vignetteMapInv (setting_photometricCalibration == 2)
    float factor;               // the other branch: factor * raw
};

template<typename T>
__device__ __forceinline__ float ud_tap(const T *__restrict__ raw, int k, const UndistortArgs &a) {
    if (k >= a.wOrg * a.hOrg) return 0.f;
    const int v = raw[k];
    if (!a.use_G) return __fmul_rn(a.factor, (float) v);
    const float g = __ldg(a.G + v);
    return a.mode2 ? __fmul_rn(g, __ldg(a.vinv + k)) : g;
}

template<typename T>
__global__ void __launch_bounds__(256) k_undistort(const T *__restrict__ raw, UndistortArgs a, float *__restrict__ out) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.w * a.h) return;
    if (a.remap == nullptr) {
        out[idx] = ud_tap(raw, idx, a);
        return;
    }
    const float2 r = __ldg(a.remap + idx);
    float xx = r.x, yy = r.y;
    if (xx < 0) {
        out[idx] = 0.f;
        return;
    }
    const int xxi = (int) xx;           // truncation toward zero, as the reference's int conversion
    const int yyi = (int) yy;
    xx = __fsub_rn(xx, (float) xxi);
    yy = __fsub_rn(yy, (float) yyi);
    const float xxyy = __fmul_rn(xx, yy);
    const int src_offset = xxi + yyi * a.wOrg;
    if (src_offset < 0 || src_offset > (a.hOrg - 1) * a.wOrg) {
        out[idx] = 0.f;
        return;
    }
    const float s0 = ud_tap(raw, src_offset, a), s1 = ud_tap(raw, src_offset + 1, a);
    const float s2 = ud_tap(raw, src_offset + a.wOrg, a), s3 = ud_tap(raw, src_offset + 1 + a.wOrg, a);
    // xxyy*s[1+wOrg] + (yy-xxyy)*s[wOrg] + (xx-xxyy)*s[1] + (1-xx-yy+xxyy)*s[0], left to right
    const float t3 = __fmul_rn(xxyy, s3);
    const float t2 = __fmul_rn(__fsub_rn(yy, xxyy), s2);
    const float t1 = __fmul_rn(__fsub_rn(xx, xxyy), s1);
    const float t0 = __fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(1.f, xx), yy), xxyy), s0);
    out[idx] = __fadd_rn(__fadd_rn(__fadd_rn(t3, t2), t1), t0);
}
