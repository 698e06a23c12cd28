// Keyframe corner detection on the device: LDSO's FeatureDetector::DetectCorners (src/frontend/FeatureDetector.cc:34-130) with
// ShiTomasiScore and IC_Angle (include/frontend/FeatureDetector.h:50-114) and ComputeDescriptor (FeatureDetector.cc:132-189), on
// level 0 of a keyframe's resident pyramid. absSquaredGrad[0] is formed on the fly from the texels as makeImages forms it
// (FrameHessian.cc:91-97). Every float product and sum is rounded on its own (__fmul_rn / __fadd_rn / __fsub_rn), so nvcc contracts
// nothing into an FMA; the double steps of the reference (gradTH, the score's divisions and 0.5*, scoreTH) stay double.
//   k_corner_cells     one CTA per grid cell: maxGrad, gradTH, the Shi-Tomasi score of every candidate, the cell's first k picks in
//                      the order rule (score descending, NaN last, ties in push order) and the cell's largest score
//   k_corner_scan      one CTA: exclusive scan of the per-cell counts (gx outer, gy inner), maxScore, scoreTH
//   k_corner_emit      one thread per pick: the features in the reference's order, and the initial isCorner = score > scoreTH
//   k_corner_describe  one thread per feature: suppression against the initial corners of the neighbouring cells, then IC_Angle
//                      and the ORB descriptor of every surviving corner (atan2 / cos / sin in double, rounded to float)
#pragma once
#include "common.cuh"
#include "img_kernels.cuh"

#define CORNER_HALF_PATCH 15
#define CORNER_THREADS 256
#define CORNER_FEATURE_BYTES (4 * 4 + 1 + 32)     // u, v, score, angle, is_corner, descriptor

struct CornerArgs {
    const float4 *img;            // level 0: (I, dx, dy, 0)
    const float *B;               // CalibHessian::B (256), nullptr = identity
    const int *pattern;           // bit_pattern_31_, 256 x 4
    int w, h;
    int gs, skip, ncx, ncy, kcap; // grid: cell size, skipped border cells, cells processed along x / y, picks per cell
    float nfeatInGrid;
    int umax[CORNER_HALF_PATCH + 1];
    // scratch
    unsigned long long *keys;     // per cell pixel: the order key of a candidate, ~0 for a non-candidate (ncx*ncy*gs*gs)
    int *cell_count, *cell_off;   // [ncx*ncy]
    float *cell_max;              // [ncx*ncy] the largest candidate score (s > m, from 0)
    int *pick_px;                 // [ncx*ncy*kcap] the picks' pixel index inside their cell (y*gs + x)
    float *pick_score;
    uint8_t *initial;             // [cap] isCorner before suppression
    int *hdr;                     // [0] n, [1] scoreTH bits
    // outputs, `cap` entries each
    int cap;
    float *u, *v, *score, *angle;
    uint8_t *is_corner, *desc;
};

__device__ __forceinline__ float corner_grad(const CornerArgs &a, int idx) { return pyr_abs_sq_grad(a.img, a.B, idx); }

__device__ float corner_shi_tomasi(const CornerArgs &a, int u, int v) {
    const int x_min = u - 4, x_max = u + 4, y_min = v - 4, y_max = v + 4;
    if (x_min < 1 || x_max >= a.w - 1 || y_min < 1 || y_max >= a.h - 1) return 0.f;
    float dXX = 0.f, dYY = 0.f, dXY = 0.f;
    for (int y = y_min; y < y_max; ++y)
        for (int x = x_min; x < x_max; ++x) {
            const float4 t = a.img[y * a.w + x];
            dXX = __fadd_rn(dXX, __fmul_rn(t.y, t.y));
            dYY = __fadd_rn(dYY, __fmul_rn(t.z, t.z));
            dXY = __fadd_rn(dXY, __fmul_rn(t.y, t.z));
        }
    dXX = (float) ((double) dXX / 128.0);              // / (2.0 * box_area)
    dYY = (float) ((double) dYY / 128.0);
    dXY = (float) ((double) dXY / 128.0);
    const float t = __fadd_rn(dXX, dYY);
    const float disc = __fsub_rn(__fmul_rn(t, t), __fmul_rn(4.f, __fsub_rn(__fmul_rn(dXX, dYY), __fmul_rn(dXY, dXY))));
    return (float) (0.5 * (double) __fsub_rn(t, __fsqrt_rn(disc)));
}

// order key of a candidate: score descending (NaN after every number), then push index ascending; smaller = earlier. -0 is keyed
// as +0 so that the two tie as they do in the reference's comparison (a score cannot be -0: dXX + dYY starts from +0 and grows, and
// t - sqrt(disc) of equal operands is +0)
__device__ __forceinline__ unsigned long long corner_key(float s, int push) {
    unsigned u = __float_as_uint(s == 0.f ? 0.f : s);
    unsigned kf;
    if (isnan(s)) kf = 0xFFFFFFFFu;
    else kf = ~((u & 0x80000000u) ? ~u : (u | 0x80000000u));
    return ((unsigned long long) kf << 32) | (unsigned) push;
}

// the score a key was made from; a NaN comes back as 0xFFC00000, the quiet NaN x86's sqrtss returns for a negative argument, which is
// what the reference stores for such a score
__device__ __forceinline__ float corner_key_score(unsigned long long key) {
    const unsigned kf = (unsigned) (key >> 32);
    if (kf == 0xFFFFFFFFu) return __uint_as_float(0xFFC00000u);
    const unsigned o = ~kf;
    return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}

template<typename T, typename Op>
__device__ __forceinline__ T corner_block_reduce(T v, Op op, T *sh) {
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[wid] = v;
    __syncthreads();
    if (wid == 0) {
        v = lane < (CORNER_THREADS / 32) ? sh[lane] : sh[0];
        for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
        if (lane == 0) sh[0] = v;
    }
    __syncthreads();
    return sh[0];
}

struct CornerMaxGT {      // the reference's running maximum: m = v > m ? v : m (NaN never wins)
    __device__ float operator()(float a, float b) const { return b > a ? b : a; }
};
struct CornerMinU64 {
    __device__ unsigned long long operator()(unsigned long long a, unsigned long long b) const { return b < a ? b : a; }
};

__global__ void __launch_bounds__(CORNER_THREADS) k_corner_cells(CornerArgs a) {
    __shared__ float shf[CORNER_THREADS / 32];
    __shared__ unsigned long long shk[CORNER_THREADS / 32];
    const int cell = blockIdx.x;
    const int gx = a.skip + cell / a.ncy, gy = a.skip + cell % a.ncy;
    const int gs = a.gs, npx = gs * gs;
    const int base = gy * gs * a.w + gx * gs;
    unsigned long long *keys = a.keys + (size_t) cell * npx;
    // push order: x outer, y inner -> push index i = x * gs + y
    float m = 0.f;
    for (int i = threadIdx.x; i < npx; i += CORNER_THREADS) {
        const int x = i / gs, y = i % gs;
        m = CornerMaxGT()(m, corner_grad(a, base + y * a.w + x));
    }
    const float maxGrad = corner_block_reduce(m, CornerMaxGT(), shf);
    const double gradTH = (0.5 * maxGrad) > 5 ? 0.5 * maxGrad : 5;
    float ms = 0.f;
    for (int i = threadIdx.x; i < npx; i += CORNER_THREADS) {
        const int x = i / gs, y = i % gs;
        unsigned long long k = ~0ull;
        if ((double) corner_grad(a, base + y * a.w + x) > gradTH) {
            const float s = corner_shi_tomasi(a, gx * gs + x, gy * gs + y);
            ms = CornerMaxGT()(ms, s);
            k = corner_key(s, i);
        }
        keys[i] = k;
    }
    const float cmax = corner_block_reduce(ms, CornerMaxGT(), shf);       // (the barriers inside also publish keys[])
    int r = 0;
    unsigned long long prev = 0;
    for (; r < a.kcap; r++) {
        unsigned long long best = ~0ull;
        for (int i = threadIdx.x; i < npx; i += CORNER_THREADS) {
            const unsigned long long k = keys[i];
            if ((r == 0 || k > prev) && k < best) best = k;
        }
        best = corner_block_reduce(best, CornerMinU64(), shk);
        if (best == ~0ull) break;
        if (threadIdx.x == 0) {
            const int i = (int) (best & 0xFFFFFFFFu);
            const int x = i / gs, y = i % gs;
            a.pick_px[cell * a.kcap + r] = y * gs + x;
            a.pick_score[cell * a.kcap + r] = corner_key_score(best);
        }
        prev = best;
    }
    if (threadIdx.x == 0) { a.cell_count[cell] = r; a.cell_max[cell] = cmax; }
}

__global__ void __launch_bounds__(1024) k_corner_scan(CornerArgs a) {
    __shared__ int shs[1024];
    __shared__ float shm[1024];
    __shared__ int carry;
    const int ncell = a.ncx * a.ncy;
    if (threadIdx.x == 0) carry = 0;
    float m = 0.f;
    for (int c0 = 0; c0 < ncell; c0 += 1024) {
        const int c = c0 + threadIdx.x;
        const int cnt = c < ncell ? a.cell_count[c] : 0;
        if (c < ncell) m = CornerMaxGT()(m, a.cell_max[c]);
        shs[threadIdx.x] = cnt;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {             // inclusive Hillis-Steele scan
            const int t = threadIdx.x >= o ? shs[threadIdx.x - o] : 0;
            __syncthreads();
            shs[threadIdx.x] += t;
            __syncthreads();
        }
        if (c < ncell) a.cell_off[c] = carry + shs[threadIdx.x] - cnt;
        __syncthreads();
        if (threadIdx.x == 1023) carry += shs[1023];
        __syncthreads();
    }
    shm[threadIdx.x] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        float mx = 0.f;                                   // maxScore, from 0 as the reference starts it
        for (int i = 0; i < 1024; i++) mx = CornerMaxGT()(mx, shm[i]);
        const float scoreTH = 0.01 * mx;
        a.hdr[0] = carry;
        a.hdr[1] = __float_as_int(scoreTH);
    }
}

__global__ void __launch_bounds__(256) k_corner_emit(CornerArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.ncx * a.ncy * a.kcap) return;
    const int cell = t / a.kcap, r = t % a.kcap;
    if (r >= a.cell_count[cell]) return;
    const int j = a.cell_off[cell] + r;
    const int gx = a.skip + cell / a.ncy, gy = a.skip + cell % a.ncy;
    const int p = a.pick_px[t];
    const float s = a.pick_score[t];
    a.u[j] = (float) (gx * a.gs + p % a.gs);
    a.v[j] = (float) (gy * a.gs + p / a.gs);
    a.score[j] = s;
    a.initial[j] = s > __int_as_float(a.hdr[1]);
}

__device__ float corner_ic_angle(const CornerArgs &a, int c) {
    float m_01 = 0.f, m_10 = 0.f;
    for (int u = -CORNER_HALF_PATCH; u <= CORNER_HALF_PATCH; ++u) m_10 = __fadd_rn(m_10, __fmul_rn((float) u, a.img[c + u].x));
    for (int v = 1; v <= CORNER_HALF_PATCH; ++v) {
        float v_sum = 0.f;
        const int d = a.umax[v];
        for (int u = -d; u <= d; ++u) {
            const float val_plus = a.img[c + u + v * a.w].x, val_minus = a.img[c + u - v * a.w].x;
            v_sum = __fadd_rn(v_sum, __fsub_rn(val_plus, val_minus));
            m_10 = __fadd_rn(m_10, __fmul_rn((float) u, __fadd_rn(val_plus, val_minus)));
        }
        m_01 = __fadd_rn(m_01, __fmul_rn((float) v, v_sum));
    }
    return (float) atan2((double) m_01, (double) m_10);
}

__device__ void corner_descriptor(const CornerArgs &a, int c, float angle_in, uint8_t *out) {
    const float factorPI = (float) (3.1415926535897932384626433832795 / 180.f);
    const float angle = __fmul_rn(angle_in, factorPI);
    const float ca = (float) cos((double) angle), sb = (float) sin((double) angle);
    for (int i = 0; i < 32; ++i) {
        int val = 0;
        for (int j = 0; j < 8; j++) {
            const int *p = a.pattern + 32 * i + 4 * j;
            const float p0 = (float) __ldg(p), p1 = (float) __ldg(p + 1), p2 = (float) __ldg(p + 2), p3 = (float) __ldg(p + 3);
            const int y0 = (int) __fadd_rn(__fmul_rn(p0, sb), __fmul_rn(p1, ca)), x0 = (int) __fsub_rn(__fmul_rn(p0, ca), __fmul_rn(p1, sb));
            const int y1 = (int) __fadd_rn(__fmul_rn(p2, sb), __fmul_rn(p3, ca)), x1 = (int) __fsub_rn(__fmul_rn(p2, ca), __fmul_rn(p3, sb));
            const int t0 = (int) a.img[c + y0 * a.w + x0].x, t1 = (int) a.img[c + y1 * a.w + x1].x;
            val |= (t0 < t1) << j;
        }
        out[i] = (uint8_t) val;
    }
}

__global__ void __launch_bounds__(128) k_corner_describe(CornerArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.ncx * a.ncy * a.kcap) return;
    const int cell = t / a.kcap, r = t % a.kcap;
    if (r >= a.cell_count[cell]) return;
    const int k = a.cell_off[cell] + r;
    bool c = a.initial[k];
    const float uk = a.u[k], vk = a.v[k], sk = a.score[k];
    if (c) {
        // suppression: any initial corner p closer than 5 pixels with p < k && s_p > s_k, or p > k && s_p >= s_k
        const int R = (4 + a.gs - 1) / a.gs;
        const int cx = cell / a.ncy, cy = cell % a.ncy;
        for (int nx = max(0, cx - R); c && nx <= min(a.ncx - 1, cx + R); nx++)
            for (int ny = max(0, cy - R); c && ny <= min(a.ncy - 1, cy + R); ny++) {
                const int nc = nx * a.ncy + ny, off = a.cell_off[nc], cnt = a.cell_count[nc];
                for (int p = off; p < off + cnt; p++) {
                    if (p == k || !a.initial[p]) continue;
                    const float dx = __fsub_rn(a.u[p], uk), dy = __fsub_rn(a.v[p], vk);
                    if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) >= 25.f) continue;
                    const float sp = a.score[p];
                    if ((p < k && sp > sk) || (p > k && sp >= sk)) { c = false; break; }
                }
            }
    }
    a.is_corner[k] = c;
    uint8_t *d = a.desc + 32 * (size_t) k;
    if (!c) {
        a.angle[k] = 0.f;
        for (int i = 0; i < 32; i++) d[i] = 0;
        return;
    }
    const int ctr = (int) vk * a.w + (int) uk;
    const float ang = corner_ic_angle(a, ctr);
    a.angle[k] = ang;
    corner_descriptor(a, ctr, ang, d);
}
