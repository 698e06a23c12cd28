// Immature-point candidates on the device (SURVEY.md §8f rank 2): ImmaturePoint's constructor and ImmaturePoint::traceOn
// (src/internal/ImmaturePoint.cc:14-38, :46-314), driven like FullSystem::traceNewCoarse drives them (FullSystem.cc:1012-1050).
// One WARP per candidate. The discrete epipolar search runs 32 steps at a time (lane = step; every lane re-creates the
// reference's running `ptx += dx` by repeated addition so the sample positions are bit-identical, and adds its 8 pattern
// residuals in the reference's order); the 1-D Gauss-Newton refinement evaluates the 8 pattern pixels on lanes 0..7 and
// accumulates them in pattern order. All control flow is warp-uniform (every lane carries the same scalars).
#pragma once
#include "trace_types.h"

__constant__ int c_trace_pattern[8][2] = {{0, -2}, {-1, -1}, {1, -1}, {-2, 0}, {0, 0}, {2, 0}, {-1, 1}, {0, 2}};

// getInterpolatedElement31 / 33 (GlobalFuncs.h:145-159, :89-103); samples outside the image count as non-finite (the reference
// would read out of bounds there)
__device__ __forceinline__ float trace_tap1(const float4 *img, int w, int h, float x, float y) {
    const int ix = (int) x, iy = (int) y;
    if (!(x >= 0.f && y >= 0.f && ix < w - 1 && iy < h - 1)) return NAN;
    const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
    const float4 *bp = img + ix + iy * w;
    return dxdy * bp[1 + w].x + (dy - dxdy) * bp[w].x + (dx - dxdy) * bp[1].x + (1 - dx - dy + dxdy) * bp[0].x;
}
__device__ __forceinline__ float3 trace_tap3(const float4 *img, int w, int h, float x, float y) {
    const int ix = (int) x, iy = (int) y;
    if (!(x >= 0.f && y >= 0.f && ix < w - 1 && iy < h - 1)) return make_float3(NAN, 0.f, 0.f);
    const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
    const float4 *bp = img + ix + iy * w;
    const float4 p11 = bp[1 + w], p01 = bp[w], p10 = bp[1], p00 = bp[0];
    const float w11 = dxdy, w01 = dy - dxdy, w10 = dx - dxdy, w00 = 1 - dx - dy + dxdy;
    return make_float3(w11 * p11.x + w01 * p01.x + w10 * p10.x + w00 * p00.x, w11 * p11.y + w01 * p01.y + w10 * p10.y + w00 * p00.y,
                       w11 * p11.z + w01 * p01.z + w10 * p10.z + w00 * p00.z);
}

// ImmaturePoint::ImmaturePoint (:14-38) of candidate i: one thread per candidate on its host keyframe. color8 / weights8 past the first
// non-finite pattern pixel are left as they are.
__device__ __forceinline__ void immature_init_one(int i, const float4 *img, int w, const float *u, const float *v, const TraceSettingsDev &S,
                                                  float *color8, float *weights8, float *gradH4, float *energyTH) {
    float g00 = 0, g01 = 0, g10 = 0, g11 = 0;
    bool bad = false;
    for (int idx = 0; idx < 8 && !bad; idx++) {
        const float x = u[i] + c_trace_pattern[idx][0], y = v[i] + c_trace_pattern[idx][1];
        // getInterpolatedElement33BiLin (GlobalFuncs.h:185-207)
        const int ix = (int) x, iy = (int) y;
        const float4 *bp = img + ix + iy * w;
        const float tl = bp[0].x, tr = bp[1].x, bl = bp[w].x, br = bp[w + 1].x;
        const float dx = x - ix, dy = y - iy;
        const float topInt = dx * tr + (1 - dx) * tl, botInt = dx * br + (1 - dx) * bl;
        const float leftInt = dy * bl + (1 - dy) * tl, rightInt = dy * br + (1 - dy) * tr;
        const float c = dx * rightInt + (1 - dx) * leftInt, gx = rightInt - leftInt, gy = botInt - topInt;
        color8[8 * i + idx] = c;
        if (!isfinite(c)) { bad = true; break; }
        g00 += gx * gx; g01 += gx * gy; g10 += gy * gx; g11 += gy * gy;
        weights8[8 * i + idx] = sqrtf(S.outlierTHSumComponent / (S.outlierTHSumComponent + (gx * gx + gy * gy)));
    }
    gradH4[4 * i] = g00; gradH4[4 * i + 1] = g01; gradH4[4 * i + 2] = g10; gradH4[4 * i + 3] = g11;
    float e = 8 * S.outlierTH;
    e *= S.overallEnergyTHWeight * S.overallEnergyTHWeight;
    energyTH[i] = bad ? NAN : e;
}

__global__ void k_immature_init(int n, const float4 *img, int w, const float *u, const float *v, TraceSettingsDev S, float *color8,
                                float *weights8, float *gradH4, float *energyTH) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    immature_init_one(i, img, w, u, v, S, color8, weights8, gradH4, energyTH);
}

#define KTR_WARPS 8
// ImmaturePoint::traceOn of candidate i (one warp; every lane returns the same status, the candidate's lastTraceStatus afterwards).
// A's per-candidate arrays are indexed by i; KRKi / Kt / aff are the candidate's host transform; s_err is this warp's 100 floats.
__device__ __forceinline__ int trace_on_one(const TraceArgs &A, int i, const float *KRKi, const float *Kt, const float *aff, float *s_err) {
    const int lane = threadIdx.x & 31;
    const unsigned FULL = 0xffffffffu;
    const TraceSettingsDev &S = A.S;
    int st = A.status[i];
    if (st == IPS_OOB) return st;                                                // :52
    const int w = A.w, h = A.h;
    const float pu = A.u[i], pv = A.v[i];
    float idmin = A.idepth_min[i], idmax = A.idepth_max[i], quality = A.quality[i];
    const float maxPixSearch = (w + h) * S.maxPixSearch;
    float uvx = -1.f, uvy = -1.f, interval = 0.f;
    int result = -1;          // >= 0: finished with this status
#define TR_RETURN(status_, ux_, uy_, iv_) do { result = (status_); uvx = (ux_); uvy = (uy_); interval = (iv_); } while (0)

    float pr[3], ptpMin[3], ptpMax[3];
    for (int k = 0; k < 3; k++) pr[k] = KRKi[k * 3 + 0] * pu + KRKi[k * 3 + 1] * pv + KRKi[k * 3 + 2] * 1.0f;
    for (int k = 0; k < 3; k++) ptpMin[k] = pr[k] + Kt[k] * idmin;
    float uMin = ptpMin[0] / ptpMin[2], vMin = ptpMin[1] / ptpMin[2];
    float dist = 0.f, uMax = 0.f, vMax = 0.f;
    if (!(uMin > 4 && vMin > 4 && uMin < w - 5 && vMin < h - 5)) TR_RETURN(IPS_OOB, -1.f, -1.f, 0.f);
    if (result < 0) {
        if (isfinite(idmax)) {                                                   // :77-98
            for (int k = 0; k < 3; k++) ptpMax[k] = pr[k] + Kt[k] * idmax;
            uMax = ptpMax[0] / ptpMax[2]; vMax = ptpMax[1] / ptpMax[2];
            if (!(uMax > 4 && vMax > 4 && uMax < w - 5 && vMax < h - 5)) TR_RETURN(IPS_OOB, -1.f, -1.f, 0.f);
            else {
                dist = (uMin - uMax) * (uMin - uMax) + (vMin - vMax) * (vMin - vMax);
                dist = sqrtf(dist);
                if (dist < S.trace_slackInterval) TR_RETURN(IPS_SKIPPED, (uMax + uMin) * 0.5f, (vMax + vMin) * 0.5f, dist);
            }
        } else {                                                                 // :99-124
            dist = maxPixSearch;
            for (int k = 0; k < 3; k++) ptpMax[k] = pr[k] + Kt[k] * 0.01f;
            uMax = ptpMax[0] / ptpMax[2]; vMax = ptpMax[1] / ptpMax[2];
            const float ddx = uMax - uMin, ddy = vMax - vMin;
            const float d = 1.0f / sqrtf(ddx * ddx + ddy * ddy);
            uMax = uMin + dist * ddx * d;
            vMax = vMin + dist * ddy * d;
            if (!(uMax > 4 && vMax > 4 && uMax < w - 5 && vMax < h - 5)) TR_RETURN(IPS_OOB, -1.f, -1.f, 0.f);
        }
    }
    if (result < 0 && !(idmin < 0 || (ptpMin[2] > 0.75f && ptpMin[2] < 1.5f))) TR_RETURN(IPS_OOB, -1.f, -1.f, 0.f);   // :127-131

    float dx = 0.f, dy = 0.f, errorInPixel = 0.f;
    if (result < 0) {                                                            // :134-148
        const float *G = A.gradH4 + 4 * i;
        dx = S.trace_stepsize * (uMax - uMin);
        dy = S.trace_stepsize * (vMax - vMin);
        const float a = (dx * G[0] + dy * G[2]) * dx + (dx * G[1] + dy * G[3]) * dy;
        const float b = (dy * G[0] + (-dx) * G[2]) * dy + (dy * G[1] + (-dx) * G[3]) * (-dx);
        errorInPixel = 0.2f + 0.2f * (a + b) / a;
        if (errorInPixel * S.trace_minImprovementFactor > dist && isfinite(idmax)) TR_RETURN(IPS_BADCONDITION, (uMax + uMin) * 0.5f, (vMax + vMin) * 0.5f, dist);
        if (errorInPixel > 10) errorInPixel = 10;
    }
    float bestU = 0.f, bestV = 0.f, bestEnergy = 1e10f;
    float rx = 0.f, ry = 0.f, col = 0.f, wgt = 0.f;        // lane < 8: rotated pattern offset, colour, weight of pattern pixel `lane`
    if (result < 0) {                                                            // :151-217 discrete search
        dx /= dist;
        dy /= dist;
        if (dist > maxPixSearch) {
            uMax = uMin + maxPixSearch * dx;
            vMax = vMin + maxPixSearch * dy;
            dist = maxPixSearch;
        }
        int numSteps = 1.9999f + dist / S.trace_stepsize;
        const float randShift = uMin * 1000 - floorf(uMin * 1000);
        const float ptx0 = uMin - randShift * dx, pty0 = vMin - randShift * dy;
        if (!isfinite(dx) || !isfinite(dy)) TR_RETURN(IPS_OOB, -1.f, -1.f, 0.f);
        else {
            if (lane < 8) {
                rx = KRKi[0] * c_trace_pattern[lane][0] + KRKi[1] * c_trace_pattern[lane][1];
                ry = KRKi[3] * c_trace_pattern[lane][0] + KRKi[4] * c_trace_pattern[lane][1];
                col = A.color8[8 * i + lane]; wgt = A.weights8[8 * i + lane];
            }
            if (numSteps >= 100) numSteps = 99;
            // every lane needs all 8 pattern offsets / colours for its own steps
            float prx[8], pry[8], pcol[8];
#pragma unroll
            for (int idx = 0; idx < 8; idx++) { prx[idx] = __shfl_sync(FULL, rx, idx); pry[idx] = __shfl_sync(FULL, ry, idx); pcol[idx] = __shfl_sync(FULL, col, idx); }
            float ptx = ptx0, pty = pty0;
            for (int k = 0; k < lane; k++) { ptx += dx; pty += dy; }             // the reference's running sum, replayed
            float myBestE = 1e10f, myBestU = 0.f, myBestV = 0.f;
            int myBestI = 1 << 30;
            for (int s0 = 0; s0 < numSteps; s0 += 32) {
                const int si = s0 + lane;
                if (si < numSteps) {
                    float energy = 0;
#pragma unroll
                    for (int idx = 0; idx < 8; idx++) {
                        const float hit = trace_tap1(A.img, w, h, ptx + prx[idx], pty + pry[idx]);
                        if (!isfinite(hit)) { energy += 1e5f; continue; }
                        const float residual = hit - (aff[0] * pcol[idx] + aff[1]);
                        const float hw = fabsf(residual) < S.huberTH ? 1 : S.huberTH / fabsf(residual);
                        energy += hw * residual * residual * (2 - hw);
                    }
                    s_err[si] = energy;
                    if (energy < myBestE) { myBestE = energy; myBestU = ptx; myBestV = pty; myBestI = si; }
                }
                for (int k = 0; k < 32; k++) { ptx += dx; pty += dy; }
            }
            // first index of the minimum (the reference's strict `<` scan)
            float be = myBestE; int bi = myBestI;
            for (int o = 16; o > 0; o >>= 1) {
                const float oe = __shfl_xor_sync(FULL, be, o); const int oi = __shfl_xor_sync(FULL, bi, o);
                if (oe < be || (oe == be && oi < bi)) { be = oe; bi = oi; }
            }
            const int src = bi & 31;        // lane that evaluated step bi (bi = 1<<30 only if no step beat 1e10: src 0, bestIdx -1)
            int bestIdx = (bi == (1 << 30)) ? -1 : bi;
            bestEnergy = (bestIdx < 0) ? 1e10f : be;
            bestU = __shfl_sync(FULL, (myBestI == bi) ? myBestU : 0.f, src);
            bestV = __shfl_sync(FULL, (myBestI == bi) ? myBestV : 0.f, src);
            if (bestIdx < 0) { bestU = 0.f; bestV = 0.f; }
            __syncwarp();
            float second = 1e10f;                                                // :220-227
            for (int si = lane; si < numSteps; si += 32)
                if ((si < bestIdx - S.minTraceTestRadius || si > bestIdx + S.minTraceTestRadius) && s_err[si] < second) second = s_err[si];
            for (int o = 16; o > 0; o >>= 1) second = fminf(second, __shfl_xor_sync(FULL, second, o));
            const float newQuality = second / bestEnergy;
            if (newQuality < quality || numSteps > 10) quality = newQuality;
        }
    }
    if (result < 0) {                                                            // :231-278 GN optimisation
        float uBak = bestU, vBak = bestV, stepBack = 0;
        const float gnstepsize = 1;
        if (S.trace_GNIterations > 0) bestEnergy = 1e5f;
        for (int it = 0; it < S.trace_GNIterations; it++) {
            float tH = 0.f, tb = 0.f, te = 0.f;
            int valid = 0;
            if (lane < 8) {
                const float3 hit = trace_tap3(A.img, w, h, bestU + rx, bestV + ry);
                if (isfinite(hit.x)) {
                    valid = 1;
                    const float residual = hit.x - (aff[0] * col + aff[1]);
                    const float dResdDist = dx * hit.y + dy * hit.z;
                    const float hw = fabsf(residual) < S.huberTH ? 1 : S.huberTH / fabsf(residual);
                    tH = hw * dResdDist * dResdDist;
                    tb = hw * residual * dResdDist;
                    te = wgt * wgt * hw * residual * residual * (2 - hw);
                }
            }
            float H = 1, b = 0, energy = 0;
#pragma unroll
            for (int idx = 0; idx < 8; idx++) {
                const int vd = __shfl_sync(FULL, valid, idx);
                const float xH = __shfl_sync(FULL, tH, idx), xb = __shfl_sync(FULL, tb, idx), xe = __shfl_sync(FULL, te, idx);
                if (!vd) { energy += 1e5f; continue; }
                H += xH; b += xb; energy += xe;
            }
            if (energy > bestEnergy) {
                stepBack *= 0.5f;
                bestU = uBak + stepBack * dx;
                bestV = vBak + stepBack * dy;
            } else {
                float step = -gnstepsize * b / H;
                if (step < -0.5f) step = -0.5f;
                else if (step > 0.5f) step = 0.5f;
                if (!isfinite(step)) step = 0;
                uBak = bestU; vBak = bestV; stepBack = step;
                bestU += step * dx;
                bestV += step * dy;
                bestEnergy = energy;
            }
            if (fabsf(stepBack) < S.trace_GNThreshold) break;
        }
        if (!(bestEnergy < A.energyTH[i] * S.trace_extraSlackOnTH)) {            // :281-288
            TR_RETURN((st == IPS_OUTLIER) ? IPS_OOB : IPS_OUTLIER, -1.f, -1.f, 0.f);
        } else {                                                                 // :291-313
            if (dx * dx > dy * dy) {
                idmin = (pr[2] * (bestU - errorInPixel * dx) - pr[0]) / (Kt[0] - Kt[2] * (bestU - errorInPixel * dx));
                idmax = (pr[2] * (bestU + errorInPixel * dx) - pr[0]) / (Kt[0] - Kt[2] * (bestU + errorInPixel * dx));
            } else {
                idmin = (pr[2] * (bestV - errorInPixel * dy) - pr[1]) / (Kt[1] - Kt[2] * (bestV - errorInPixel * dy));
                idmax = (pr[2] * (bestV + errorInPixel * dy) - pr[1]) / (Kt[1] - Kt[2] * (bestV + errorInPixel * dy));
            }
            if (idmin > idmax) { const float t = idmin; idmin = idmax; idmax = t; }
            if (!isfinite(idmin) || !isfinite(idmax) || (idmax < 0)) TR_RETURN(IPS_OUTLIER, -1.f, -1.f, 0.f);
            else TR_RETURN(IPS_GOOD, bestU, bestV, 2 * errorInPixel);
        }
    }
#undef TR_RETURN
    if (lane == 0) {
        A.status[i] = result;
        A.idepth_min[i] = idmin; A.idepth_max[i] = idmax; A.quality[i] = quality;
        A.uv2[2 * i] = uvx; A.uv2[2 * i + 1] = uvy; A.interval[i] = interval;
    }
    return result;
}

__global__ void __launch_bounds__(32 * KTR_WARPS) k_trace_on(TraceArgs A) {
    __shared__ float s_err[KTR_WARPS][100];
    const int wib = threadIdx.x >> 5;
    const int i = blockIdx.x * KTR_WARPS + wib;
    if (i >= A.n) return;
    trace_on_one(A, i, A.KRKi9 + 9 * A.host[i], A.Kt3 + 3 * A.host[i], A.aff2 + 2 * A.host[i], s_err[wib]);
}

// ---------------------------------------------------------------------------------------------------------
// FullSystem::optimizeImmaturePoint (src/frontend/FullSystem.cc:892-978) with ImmaturePoint::linearizeResidual
// (ImmaturePoint.cc:316-383): Levenberg-Marquardt on the inverse depth of a candidate over its residuals to all other
// keyframes of the device-resident window (frame-pair records, calibration and images as the GN loop left them).
// One warp per candidate: lane = (residual, pattern pixel) in two rounds of 32; the per-pixel terms are then folded by all
// lanes in the reference's order (residual by residual, pixel by pixel, stopping a residual at its first out-of-bounds pixel
// exactly like the early return of linearizeResidual, partial Hdd/bd contributions included).
#define RS_IN_ 0
#define RS_OOB_ 1
#define RS_OUTLIER_ 2
struct ImmatureEval { float E, H, B; int ns[MAXF - 1]; float ne[MAXF - 1]; };

__device__ __forceinline__ void immature_eval(const WinState *ws, int nF, int host, float pu, float pv, const float *col8, const float *w8,
                                              float energyTH, float idepth, float slack, const int *st, const float *en, ImmatureEval &R) {
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31, nres = nF - 1;
    int okp[2]; float ep[2], hp[2], bp[2];
    const CalibDev &C = ws->calib;
#pragma unroll
    for (int pass = 0; pass < 2; pass++) {
        const int q = 32 * pass + lane, r = q >> 3, idx = q & 7;
        okp[pass] = 0; ep[pass] = 0.f; hp[pass] = 0.f; bp[pass] = 0.f;
        if (r < nres) {
            const int t = (r < host) ? r : r + 1;
            const PairRecFull &pf = ws->pairFull[host + nF * t];
            const float *aff = ws->pair[host + nF * t].aff;
            const int dx = c_trace_pattern[idx][0], dy = c_trace_pattern[idx][1];
            // projectPoint (ResidualProjections.h:57-84)
            const float k0 = (pu + dx - C.cxl) * C.fxli, k1 = (pv + dy - C.cyl) * C.fyli, k2 = 1;
            float ptp[3];
#pragma unroll
            for (int a = 0; a < 3; a++) {
                float s = pf.RTll[a * 3 + 0] * k0;
                s += pf.RTll[a * 3 + 1] * k1;
                s += pf.RTll[a * 3 + 2] * k2;
                ptp[a] = s + pf.tTll[a] * idepth;
            }
            const float drescale = 1.0f / ptp[2];
            if (drescale > 0) {
                const float uu = ptp[0] * drescale, vv = ptp[1] * drescale;
                const float Ku = uu * C.fxl + C.cxl, Kv = vv * C.fyl + C.cyl;
                if (Ku > 1.1f && Kv > 1.1f && Ku < ws->wM3G && Kv < ws->hM3G) {
                    const float3 hit = trace_tap3(ws->img0[t], ws->w, ws->h, Ku, Kv);
                    if (isfinite(hit.x)) {
                        const float residual = hit.x - (aff[0] * col8[idx] + aff[1]);
                        float hw = fabsf(residual) < ws->S.huberTH ? 1 : ws->S.huberTH / fabsf(residual);
                        ep[pass] = w8[idx] * w8[idx] * hw * residual * residual * (2 - hw);
                        const float dxInterp = hit.y * C.fxl, dyInterp = hit.z * C.fyl;
                        const float d_idepth = (dxInterp * drescale * (pf.tTll[0] - pf.tTll[2] * uu) + dyInterp * drescale * (pf.tTll[1] - pf.tTll[2] * vv)) * SCALE_IDEPTH;
                        hw *= w8[idx] * w8[idx];
                        hp[pass] = (hw * d_idepth) * d_idepth;
                        bp[pass] = (hw * residual) * d_idepth;
                        okp[pass] = 1;
                    }
                }
            }
        }
    }
    R.E = 0.f;
#pragma unroll
    for (int r = 0; r < MAXF - 1; r++) {
        float el = 0.f;
        bool broke = false;
#pragma unroll
        for (int idx = 0; idx < 8; idx++) {
            const int q = r * 8 + idx, src = q & 31, pass = q >> 5;         // compile-time
            const int ok = __shfl_sync(FULL, okp[pass], src);
            const float e = __shfl_sync(FULL, ep[pass], src), hd = __shfl_sync(FULL, hp[pass], src), bd = __shfl_sync(FULL, bp[pass], src);
            if (r < nres && st[r] != RS_OOB_ && !broke) {
                if (!ok) broke = true;
                else { el += e; R.H += hd; R.B += bd; }
            }
        }
        if (r < nres) {
            float ret;
            if (st[r] == RS_OOB_ || broke) { R.ns[r] = RS_OOB_; R.ne[r] = en[r]; ret = en[r]; }     // state_NewEnergy untouched on these paths
            else {
                if (el > energyTH * slack) { el = energyTH * slack; R.ns[r] = RS_OUTLIER_; }
                else R.ns[r] = RS_IN_;
                R.ne[r] = el;
                ret = el;
            }
            R.E += ret;
        }
    }
}

// optimizeImmaturePoint of candidate i (one warp)
__device__ __forceinline__ void optimize_immature_one(int i, const WinState *ws, const float *u, const float *v, const int *host, const float *idmin,
                                                      const float *idmax, const float *color8, const float *weights8, const float *energyTH,
                                                      int minObs, int *ok_out, float *idepth_out, unsigned char *res_state) {
    const int lane = threadIdx.x & 31;
    const int nF = ws->nF, nres = nF - 1, h = host[i];
    const float setting_minIdepthH_act = 100;          // Setting.cc:25
    const int setting_GNItsOnPointActivation = 3;      // Setting.cc:47
    float col8[8], w8[8];
#pragma unroll
    for (int k = 0; k < 8; k++) { col8[k] = color8[8 * i + k]; w8[k] = weights8[8 * i + k]; }
    const float pu = u[i], pv = v[i], eTH = energyTH[i];
    int st[MAXF - 1]; float en[MAXF - 1];
#pragma unroll
    for (int r = 0; r < MAXF - 1; r++) { st[r] = RS_IN_; en[r] = 0.f; }
    float currentIdepth = (idmax[i] + idmin[i]) * 0.5f;
    ImmatureEval R;
    R.H = 0.f; R.B = 0.f;
    immature_eval(ws, nF, h, pu, pv, col8, w8, eTH, currentIdepth, 1000.f, st, en, R);
    float lastEnergy = R.E, lastHdd = R.H, lastbd = R.B;
#pragma unroll
    for (int r = 0; r < MAXF - 1; r++) if (r < nres) { st[r] = R.ns[r]; en[r] = R.ne[r]; }
    bool success = true;
    if (!isfinite(lastEnergy) || lastHdd < setting_minIdepthH_act) success = false;
    if (success) {
        float lambda = 0.1f;
        for (int iteration = 0; iteration < setting_GNItsOnPointActivation; iteration++) {
            float H = lastHdd;
            H *= 1 + lambda;
            const float step = (float) ((1.0 / (double) H) * (double) lastbd);
            const float newIdepth = currentIdepth - step;
            R.H = 0.f; R.B = 0.f;
            immature_eval(ws, nF, h, pu, pv, col8, w8, eTH, newIdepth, 1.f, st, en, R);
            if (!isfinite(lastEnergy) || R.H < setting_minIdepthH_act) { success = false; break; }
            if (R.E < lastEnergy) {
                currentIdepth = newIdepth;
                lastHdd = R.H; lastbd = R.B; lastEnergy = R.E;
#pragma unroll
                for (int r = 0; r < MAXF - 1; r++) if (r < nres) { st[r] = R.ns[r]; en[r] = R.ne[r]; }
                lambda = (float) ((double) lambda * 0.5);
            } else {
                lambda *= 5;
            }
            if ((double) fabsf(step) < 0.0001 * (double) currentIdepth) break;
        }
    }
    if (success && !isfinite(currentIdepth)) success = false;
    int numGoodRes = 0;
#pragma unroll
    for (int r = 0; r < MAXF - 1; r++) if (r < nres && st[r] == RS_IN_) numGoodRes++;
    if (success && numGoodRes < minObs) success = false;
    if (lane == 0) {
        ok_out[i] = success ? 1 : 0;
        idepth_out[i] = currentIdepth;
        for (int t = 0; t < nF; t++) res_state[(size_t) i * nF + t] = 255;
#pragma unroll
        for (int r = 0; r < MAXF - 1; r++) if (r < nres) res_state[(size_t) i * nF + ((r < h) ? r : r + 1)] = (unsigned char) st[r];
    }
}

__global__ void __launch_bounds__(32 * KTR_WARPS) k_optimize_immature(int n, const WinState *ws, const float *u, const float *v, const int *host,
                                                                      const float *idmin, const float *idmax, const float *color8,
                                                                      const float *weights8, const float *energyTH, int minObs, int *ok_out,
                                                                      float *idepth_out, unsigned char *res_state) {
    const int i = blockIdx.x * KTR_WARPS + (threadIdx.x >> 5);
    if (i >= n) return;
    optimize_immature_one(i, ws, u, v, host, idmin, idmax, color8, weights8, energyTH, minObs, ok_out, idepth_out, res_state);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Which immature points become active points: FullSystem::activatePointsMT's selection loop (FullSystem.cc:1088-1150) over the
// CoarseDistanceMap (CoarseTracker.cc:634-870). The loop is a greedy, order-dependent pass — every accepted candidate is added
// to the distance map before the next one is tested — so ONE CTA owns the map (one byte per level-1 pixel, in shared memory when
// it fits: 75 KB for 640x480): all 1024 threads build it (projection of the window's points, then the 39-step alternating
// 4-/8-neighbourhood BFS as a frontier expansion, each cell claimed once by a byte-wide compare-and-swap), all threads
// precompute each candidate's static test (status gates, projection, sub-pixel term, threshold), then one warp replays the
// reference's sequential pass, growing the map from every accepted point with a warp-wide frontier BFS that stops when
// nothing improves. Float arithmetic as in the reference (this TU is compiled with -fmad=false).
__device__ __forceinline__ bool actsel_improve(unsigned char *map, int idx, unsigned k) {      // map[idx] = k if map[idx] > k; true for the one winner
    if (((volatile unsigned char *) map)[idx] <= k) return false;          // most probes fail: settle them with a byte load
    unsigned *wp = (unsigned *) (map + (idx & ~3));
    const int sh = (idx & 3) * 8;
    unsigned old = *(volatile unsigned *) wp;
    while (true) {
        if (((old >> sh) & 255u) <= k) return false;
        const unsigned nw = (old & ~(255u << sh)) | (k << sh);
        const unsigned prev = atomicCAS(wp, old, nw);
        if (prev == old) return true;
        old = prev;
    }
}
// frontier entries are (x | y << 16); neighbour q in growDistBFS's visiting order (:747-806): +x, -x, +y, -y, then the four diagonals
__device__ __forceinline__ int actsel_dx(int q) { return (int) ((0x8252u >> (2 * q)) & 3u) - 1; }      // 1,-1,0,0,1,-1,-1,1
__device__ __forceinline__ int actsel_dy(int q) { return (int) ((0x0a25u >> (2 * q)) & 3u) - 1; }      // 0,0,1,-1,1,1,-1,-1
__device__ __forceinline__ void actsel_m33_mul(const float *a, const float *b, float *c) {
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            float s = a[i * 3 + 0] * b[0 * 3 + j];
            s += a[i * 3 + 1] * b[1 * 3 + j];
            s += a[i * 3 + 2] * b[2 * 3 + j];
            c[i * 3 + j] = s;
        }
}

__global__ void __launch_bounds__(ACTSEL_THREADS, 1) k_activation_select(ActSelArgs A) {
    extern __shared__ __align__(16) unsigned char actsel_smem[];
    __shared__ float sKRKi[MAXF][9], sKt[MAXF][3];
    __shared__ int sCnt[2];
    __shared__ int sLocal[2][ACTSEL_LOCAL_CAP];
    const int tid = threadIdx.x, w1 = A.w1, h1 = A.h1, nF = A.ws->nF;
    unsigned char *map = A.use_smem ? actsel_smem : A.map;

    // CoarseDistanceMap::makeK (:657-685) for levels 0 and 1, then K[1] * R * Ki[0] and K[1] * t per host keyframe (:705-706)
    if (tid < nF && tid != A.newest) {
        const CalibDev &cal = A.ws->calib;
        const float fx0 = cal.fxl, fy0 = cal.fyl, cx0 = cal.cxl, cy0 = cal.cyl;
        const float fx1 = fx0 * 0.5, fy1 = fy0 * 0.5;
        const float cx1 = (cx0 + 0.5) / ((int) 1 << 1) - 0.5, cy1 = (cy0 + 0.5) / ((int) 1 << 1) - 0.5;
        const float K1[9] = {fx1, 0, cx1, 0, fy1, cy1, 0, 0, 1}, m[9] = {fx0, 0, cx0, 0, fy0, cy0, 0, 0, 1};
        float inv[9];                                  // Eigen's 3x3 inverse: cofactors * (1 / det)
        const float c00 = m[4] * m[8] - m[5] * m[7], c01 = m[5] * m[6] - m[3] * m[8], c02 = m[3] * m[7] - m[4] * m[6];
        const float det = m[0] * c00 + m[1] * c01 + m[2] * c02;
        const float invdet = 1.0f / det;
        inv[0] = c00 * invdet; inv[3] = c01 * invdet; inv[6] = c02 * invdet;
        inv[1] = (m[2] * m[7] - m[1] * m[8]) * invdet; inv[4] = (m[0] * m[8] - m[2] * m[6]) * invdet; inv[7] = (m[1] * m[6] - m[0] * m[7]) * invdet;
        inv[2] = (m[1] * m[5] - m[2] * m[4]) * invdet; inv[5] = (m[2] * m[3] - m[0] * m[5]) * invdet; inv[8] = (m[0] * m[4] - m[1] * m[3]) * invdet;
        const PairRecFull &pf = A.ws->pairFull[tid + nF * A.newest];
        float KR[9];
        actsel_m33_mul(K1, pf.RTll, KR);
        actsel_m33_mul(KR, inv, sKRKi[tid]);
        for (int i = 0; i < 3; i++) {
            float s = K1[i * 3 + 0] * pf.tTll[0];
            s += K1[i * 3 + 1] * pf.tTll[1];
            s += K1[i * 3 + 2] * pf.tTll[2];
            sKt[tid][i] = s;
        }
    }
    if (tid == 0 && A.dbg) A.dbg[0] = clock64();
    for (int i = tid; i < A.map_bytes / 4; i += ACTSEL_THREADS) ((unsigned *) map)[i] = 0xffffffffu;      // :690-692 (1000 everywhere)
    if (tid < 2) sCnt[tid] = 0;
    __syncthreads();

    // makeDistanceMap :699-722 — seeds: the ACTIVE points of the other keyframes projected into level 1 of the newest
    for (int p = tid; p < A.nP; p += ACTSEL_THREADS) {
        const int hst = A.pt_host[p];
        if (hst == A.newest) continue;
        const float *KRKi = sKRKi[hst], *Kt = sKt[hst];
        const float pu = A.pt_u[p], pv = A.pt_v[p], pid = A.pt_idepth[p];
        float ptp[3];
        for (int r = 0; r < 3; r++) {
            float s = KRKi[r * 3 + 0] * pu;
            s += KRKi[r * 3 + 1] * pv;
            s += KRKi[r * 3 + 2] * 1.0f;
            ptp[r] = s + Kt[r] * pid;
        }
        const int u = (int) (ptp[0] / ptp[2] + 0.5f), v = (int) (ptp[1] / ptp[2] + 0.5f);
        if (!(u > 0 && v > 0 && u < w1 && v < h1)) continue;
        if (actsel_improve(map, u + w1 * v, 0u)) A.front0[atomicAdd(&sCnt[0], 1)] = u | (v << 16);
    }
    __syncthreads();

    // growDistBFS (:728-812): step k claims every cell > k next to a cell claimed at step k-1; even steps 4-neighbourhood, odd steps 8
    {
        int *fin = A.front0, *fout = A.front1;
        int cur = 0;
        for (int k = 1; k < 40; k++) {
            const int nin = sCnt[cur], lg = (k % 2 == 0) ? 2 : 3;
            if (nin == 0) break;
            for (int t = tid; t < (nin << lg); t += ACTSEL_THREADS) {
                const int xy = fin[t >> lg], x = xy & 0xffff, y = xy >> 16, q = t & ((1 << lg) - 1);
                if (x == 0 || y == 0 || x == w1 - 1 || y == h1 - 1) continue;
                const int nx = x + actsel_dx(q), ny = y + actsel_dy(q);
                if (actsel_improve(map, nx + ny * w1, (unsigned) k)) fout[atomicAdd(&sCnt[cur ^ 1], 1)] = nx | (ny << 16);
            }
            __syncthreads();
            if (tid == 0) sCnt[cur] = 0;
            cur ^= 1;
            int *tmp = fin; fin = fout; fout = tmp;
            __syncthreads();
        }
    }
    __syncthreads();

    if (tid == 0 && A.dbg) A.dbg[1] = clock64();
    // the static part of every candidate's test (FullSystem.cc:1103-1131, :1144-1148)
    for (int i = tid; i < A.n; i += ACTSEL_THREADS) {
        const int st = A.status[i], hst = A.host[i];
        const float idmax = A.idmax[i], idmin = A.idmin[i];
        unsigned char act;
        int cell = -1; float frac = 0.f;
        if (!isfinite(idmax) || st == IPS_OUTLIER) act = 2;
        else {
            const bool canActivate = (st == IPS_GOOD || st == IPS_SKIPPED || st == IPS_BADCONDITION || st == IPS_OOB) && A.interval[i] < 8 &&
                                     A.quality[i] > A.minTraceQuality && (idmax + idmin) > 0;
            if (!canActivate) act = (A.flagged[hst] || st == IPS_OOB) ? 2 : 0;
            else {
                const float *KRKi = sKRKi[hst], *Kt = sKt[hst];
                const float idm = 0.5f * (idmax + idmin), cu = A.u[i], cv = A.v[i];
                float ptp[3];
                for (int r = 0; r < 3; r++) {
                    float s = KRKi[r * 3 + 0] * cu;
                    s += KRKi[r * 3 + 1] * cv;
                    s += KRKi[r * 3 + 2] * 1.0f;
                    ptp[r] = s + Kt[r] * idm;
                }
                const int u = (int) (ptp[0] / ptp[2] + 0.5f), v = (int) (ptp[1] / ptp[2] + 0.5f);
                if (u > 0 && v > 0 && u < w1 && v < h1) { act = 3; cell = u + w1 * v; frac = ptp[0] - floorf(ptp[0]); }
                else act = 2;
            }
        }
        A.action[i] = act;                 // 3 = decided by the sequential pass below
        A.pre_idx[i] = cell < 0 ? -1 : ((cell % w1) | ((cell / w1) << 16)); A.pre_frac[i] = frac; A.pre_thresh[i] = A.currentMinActDist * A.my_type[i];
    }
    __syncthreads();

    if (tid == 0 && A.dbg) A.dbg[2] = clock64();
    // the sequential pass (:1133-1143), one warp; 32 candidates' precomputed terms are fetched at a time
    if (tid < 32) {
        const int lane = tid;
        for (int base = 0; base < A.n; base += 32) {
            const int i = base + lane;
            unsigned char myAct = 0; int myCell = -1; float myFrac = 0.f, myTh = 0.f;
            if (i < A.n) { myAct = A.action[i]; myCell = A.pre_idx[i]; myFrac = A.pre_frac[i]; myTh = A.pre_thresh[i]; }
            const int cnt = min(32, A.n - base);
            for (int j = 0; j < cnt; j++) {
                const int act = __shfl_sync(0xffffffffu, (int) myAct, j);
                if (act != 3) continue;
                const int cxy = __shfl_sync(0xffffffffu, myCell, j), cell = (cxy & 0xffff) + (cxy >> 16) * w1;
                const float frac = __shfl_sync(0xffffffffu, myFrac, j), th = __shfl_sync(0xffffffffu, myTh, j);
                const unsigned char b = map[cell];
                const float dist = (b == 255 ? 1000.f : (float) b) + frac;
                const bool accept = dist >= th;
                if (lane == j) myAct = accept ? 1 : 0;
                if (!accept) continue;
                // addIntoDistFinal (:814-819): the cell becomes 0 and the map grows from it
                if (lane == 0) { map[cell] = 0; sLocal[0][0] = cxy; }
                __syncwarp();
                int nin = 1, cur = 0;
                for (int k = 1; k < 40 && nin > 0; k++) {
                    const int lg = (k % 2 == 0) ? 2 : 3;
                    int nout = 0;
                    for (int t0 = 0; t0 < (nin << lg); t0 += 32) {
                        const int t = t0 + lane;
                        bool won = false; int nxy = 0;
                        if (t < (nin << lg)) {
                            const int xy = sLocal[cur][t >> lg], x = xy & 0xffff, y = xy >> 16, q = t & ((1 << lg) - 1);
                            if (!(x == 0 || y == 0 || x == w1 - 1 || y == h1 - 1)) {
                                const int nx = x + actsel_dx(q), ny = y + actsel_dy(q);
                                nxy = nx | (ny << 16);
                                won = actsel_improve(map, nx + ny * w1, (unsigned) k);
                            }
                        }
                        const unsigned m = __ballot_sync(0xffffffffu, won);
                        if (won) sLocal[cur ^ 1][nout + __popc(m & ((1u << lane) - 1u))] = nxy;
                        nout += __popc(m);
                    }
                    __syncwarp();
                    nin = nout; cur ^= 1;
                }
            }
            if (i < A.n) A.action[i] = myAct;
        }
    }
    __syncthreads();
    if (tid == 0 && A.dbg) A.dbg[3] = clock64();
    if (A.use_smem) for (int i = tid; i < A.map_bytes / 4; i += ACTSEL_THREADS) ((unsigned *) A.map)[i] = ((unsigned *) map)[i];
}

// ---------------------------------------------------------------------------------------------------------------------------
// CoarseInitializer::calcResAndGS (src/frontend/CoarseInitializer.cc:181-405): 8 lanes per point (lane = pattern pixel), 4 points
// per warp. The reference walks the pattern in order and leaves at the first pixel that projects outside or samples a non-finite
// value; here every lane evaluates its pixel, the group finds the first failing index and the ordered sums (energy, the ten
// JbBuffer entries) are folded in pattern order up to it, so the per-point outputs — including the partial JbBuffer / maxstep of
// a rejected point — are the reference's bit for bit. The 45 + 45 Hessian entries and the energy are summed across points by
// warp shuffles, per-CTA partials and a last-CTA fold (their order differs from the reference's SSE lanes: compared to tolerance).
__device__ __forceinline__ float init_tap1(const float4 *img, int w, float x, float y) {        // getInterpolatedElement31
    const int ix = (int) x, iy = (int) y;
    const float dx = x - ix, dy = y - iy, dxdy = dx * dy;
    const float4 *bp = img + ix + iy * w;
    return dxdy * bp[1 + w].x + (dy - dxdy) * bp[w].x + (dx - dxdy) * bp[1].x + (1 - dx - dy + dxdy) * bp[0].x;
}

__global__ void __launch_bounds__(INIT_THREADS) k_init_calc_res(InitArgs A) {
    __shared__ float s_part[(INIT_THREADS / 32) * INIT_NACC];
    __shared__ double s_sum[INIT_NACC];
    __shared__ bool s_last;
    const int lane = threadIdx.x & 31, idx = threadIdx.x & 7, gbase = lane & ~7;
    const int p = blockIdx.x * (INIT_THREADS / 8) + (threadIdx.x >> 3);
    const bool valid = p < A.n;
    float acc[INIT_NACC];
#pragma unroll
    for (int k = 0; k < INIT_NACC; k++) acc[k] = 0.f;

    const float pu = valid ? A.u[p] : 0.f, pv = valid ? A.v[p] : 0.f, idn = valid ? A.idepth_new[p] : 1.f;
    const bool goodOld = valid && A.isGood[p] != 0;
    // this lane's pattern pixel (:235-291)
    bool bad = true;
    float J[9], dd = 0.f, eterm = 0.f, ms = 1e10f;
#pragma unroll
    for (int k = 0; k < 9; k++) J[k] = 0.f;
    if (goodOld) {
        const int dx = c_trace_pattern[idx][0], dy = c_trace_pattern[idx][1];
        const float px = pu + dx, py = pv + dy;
        float pt0 = A.RKi[0] * px; pt0 += A.RKi[1] * py; pt0 += A.RKi[2] * 1.0f; pt0 = pt0 + A.t[0] * idn;
        float pt1 = A.RKi[3] * px; pt1 += A.RKi[4] * py; pt1 += A.RKi[5] * 1.0f; pt1 = pt1 + A.t[1] * idn;
        float pt2 = A.RKi[6] * px; pt2 += A.RKi[7] * py; pt2 += A.RKi[8] * 1.0f; pt2 = pt2 + A.t[2] * idn;
        const float u = pt0 / pt2, v = pt1 / pt2;
        const float Ku = A.fx * u + A.cx, Kv = A.fy * v + A.cy;
        const float new_idepth = idn / pt2;
        if (Ku > 1 && Kv > 1 && Ku < A.w - 2 && Kv < A.h - 2 && new_idepth > 0) {
            const float3 hit = trace_tap3(A.imgNew, A.w, A.h, Ku, Kv);
            const float rlR = init_tap1(A.imgRef, A.w, px, py);
            if (isfinite(rlR) && isfinite(hit.x)) {
                bad = false;
                const float residual = hit.x - A.aff0 * rlR - A.aff1;
                float hw = fabsf(residual) < A.huberTH ? 1.f : A.huberTH / fabsf(residual);
                eterm = hw * residual * residual * (2 - hw);
                const float dxdd = (A.t[0] - A.t[2] * u) / pt2;
                const float dydd = (A.t[1] - A.t[2] * v) / pt2;
                if (hw < 1) hw = sqrtf(hw);
                const float dxInterp = hw * hit.y * A.fx;
                const float dyInterp = hw * hit.z * A.fy;
                J[0] = new_idepth * dxInterp;
                J[1] = new_idepth * dyInterp;
                J[2] = -new_idepth * (u * dxInterp + v * dyInterp);
                J[3] = -u * v * dxInterp - (1 + v * v) * dyInterp;
                J[4] = (1 + u * u) * dxInterp + u * v * dyInterp;
                J[5] = -v * dxInterp + u * dyInterp;
                J[6] = -hw * A.aff0 * rlR;
                J[7] = -hw * 1;
                dd = dxInterp * dxdd + dyInterp * dydd;
                J[8] = hw * residual;
                const float a = dxdd * A.fx, b = dydd * A.fy;
                ms = 1.0f / sqrtf(a * a + b * b);
            }
        }
    }
    // first failing pattern index of the group; sums in pattern order up to it
    const unsigned badmask = (__ballot_sync(0xffffffffu, bad) >> gbase) & 0xffu;
    const int firstBad = badmask ? (__ffs(badmask) - 1) : 8;
    float energy = 0.f, Jb[10];
#pragma unroll
    for (int k = 0; k < 10; k++) Jb[k] = 0.f;
    float prod[10];
#pragma unroll
    for (int k = 0; k < 8; k++) prod[k] = J[k] * dd;
    prod[8] = J[8] * dd; prod[9] = dd * dd;
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const float ei = __shfl_sync(0xffffffffu, eterm, gbase + i);
        if (i < firstBad) energy += ei;
#pragma unroll
        for (int k = 0; k < 10; k++) {
            const float pk = __shfl_sync(0xffffffffu, prod[k], gbase + i);
            if (i < firstBad) Jb[k] += pk;
        }
    }
    // point->maxstep starts at 1e10 and takes `maxstep < point->maxstep` per visited pixel (:74, :125-126): an infinite step
    // (zero translation) or a NaN never wins that comparison, so such lanes enter the minimum as 1e10
    float msg = (idx < firstBad && ms < 1e10f) ? ms : 1e10f;
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) { const float other = __shfl_xor_sync(0xffffffffu, msg, o); if (other < msg) msg = other; }

    const float e0 = valid ? A.energy2[2 * p] : 0.f, e1 = valid ? A.energy2[2 * p + 1] : 0.f;
    const bool accepted = goodOld && firstBad == 8 && !(energy > (valid ? A.outlierTH[p] : 0.f) * 20);
    if (accepted) {      // acc9.updateSSE / updateSingle (:309-329): this lane's residual
        int k = 0;
#pragma unroll
        for (int r = 0; r < 9; r++)
#pragma unroll
            for (int c = r; c < 9; c++) acc[k++] += J[r] * J[c];
    }
    if (valid && idx == 0) {
        acc[90] += accepted ? energy : e0;                       // E.updateSingle (:211, :296, :303)
        A.isGood_new[p] = accepted ? 1 : 0;
        A.maxstep[p] = goodOld ? msg : 1e10f;
        if (!accepted) { A.energy_new2[2 * p] = e0; A.energy_new2[2 * p + 1] = e1; }
        if (goodOld && !accepted) for (int k = 0; k < 10; k++) A.Jb[10 * p + k] = Jb[k];
        if (accepted) {      // :344, :365-388
            A.energy_new2[2 * p] = energy;
            A.energy_new2[2 * p + 1] = (idn - 1) * (idn - 1);
            A.lastHessian_new[p] = Jb[9];
            Jb[8] += A.alphaOpt * (idn - 1);
            Jb[9] += A.alphaOpt;
            if (A.alphaOpt == 0) {
                Jb[8] += A.couplingWeight * (idn - A.iR[p]);
                Jb[9] += A.couplingWeight;
            }
            Jb[9] = 1 / (1 + Jb[9]);
            for (int k = 0; k < 10; k++) A.Jb[10 * p + k] = Jb[k];
            // acc9SC.updateSingleWeighted(Jb[0..8], w = Jb[9]) (MatrixAccumulators.h:1489-1604)
            float Jw[9];
#pragma unroll
            for (int k = 0; k < 9; k++) Jw[k] = Jb[k];
            const float wgt = Jb[9];
            int k = 45;
#pragma unroll
            for (int r = 0; r < 9; r++) {
                acc[k++] += Jw[r] * Jw[r] * wgt;
                if (r < 8) Jw[r] *= wgt;
#pragma unroll
                for (int c = r + 1; c < 9; c++) acc[k++] += Jw[c] * Jw[r];
            }
        }
    }
    // block sum -> per-CTA partial -> the last CTA folds all partials in CTA order
    const int warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < INIT_NACC; k++) {
        float vsum = acc[k];
        for (int o = 16; o > 0; o >>= 1) vsum += __shfl_xor_sync(0xffffffffu, vsum, o);
        if (lane == 0) s_part[warp * INIT_NACC + k] = vsum;
    }
    __syncthreads();
    if (threadIdx.x < INIT_NACC) {
        double s = 0.0;
        for (int w8 = 0; w8 < INIT_THREADS / 32; w8++) s += (double) s_part[w8 * INIT_NACC + threadIdx.x];
        A.partials[blockIdx.x * INIT_NACC + threadIdx.x] = (float) s;
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(A.counter, 1u) == gridDim.x - 1);
    __syncthreads();
    if (!s_last) return;
    if (threadIdx.x < INIT_NACC) {
        double s = 0.0;
        for (unsigned bI = 0; bI < gridDim.x; bI++) s += (double) ((volatile float *) A.partials)[bI * INIT_NACC + threadIdx.x];
        s_sum[threadIdx.x] = s;
        A.out[threadIdx.x] = s;
    }
    if (threadIdx.x == 0) *A.counter = 0;
}
