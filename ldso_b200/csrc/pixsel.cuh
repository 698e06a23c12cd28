// Keyframe candidate pixels on the device: DSO's PixelSelector::makeHists, select and makeMaps (src/frontend/PixelSelector2.cc:36-315)
// on levels 0-2 of a resident pyramid. absSquaredGrad[l] is formed on the fly from the level's texels (pyr_abs_sq_grad). Every float
// product and sum is rounded on its own; the reference's mixed expressions keep their types. DESIGN.md "Pixel selection" states the
// rules where the reference reads memory it never wrote.
//   k_pixsel_hist     one CTA per 32x32 cell: the gradient histogram, computeHistQuantil + minGradHistAdd -> ths
//   k_pixsel_smooth   one thread per cell: thsSmoothed, the neighbours summed in the reference's order
// per potential:
//   k_pixsel_mask     one thread per pot cell: bit d of the cell's mask is set iff the cell picks a level-0 pixel with direction d
//   k_pixsel_walk     one warp: the pot cells in select()'s nested order, carrying n2 (the level-0 picks so far) and recording the
//                     direction index randomPattern[n2] & 15 each cell starts with
//   k_pixsel_pick     one thread per 4pot block: select()'s loop body with the recorded directions; writes the map and n2, n3, n4
// after the last pass:
//   k_pixsel_rows / k_pixsel_row_scan / k_pixsel_emit   the selected pixels in raster order (a scan over per-row counts)
//   k_pixsel_finish   one CTA: makeMaps' subsampling (rank rn in raster order, kept iff randomPattern[rn] <= charTH) and the output
//                     lists: every kept pixel, and the kept pixels inside makeNewTraces' range [3, w-4) x [3, h-4)
#pragma once
#include "common.cuh"
#include "img_kernels.cuh"

#define PIXSEL_HDR_INTS 16
// header words (device, read back by the host)
#define PIXSEL_N2 0        // this pass's level-0, level-1 and level-2 picks
#define PIXSEL_N3 1
#define PIXSEL_N4 2
#define PIXSEL_MIXED 3     // pot cells of this pass whose direction mask is neither empty nor full
#define PIXSEL_NSEL 4      // selected pixels of the last pass (before subsampling)
#define PIXSEL_NKEPT 5     // ... kept by the subsampling: makeMaps' return value
#define PIXSEL_NFEAT 6     // ... of which inside [3, w-4) x [3, h-4)
#define PIXSEL_NSEED 7     // ... of which with a finite energyTH (k_store_compact)

struct PixselArgs {
    const float4 *img0, *img1, *img2;   // pyramid levels 0, 1, 2: (I, dx, dy, 0)
    const float *B;                     // CalibHessian::B (256), nullptr = identity
    int w, h, w1, w2;                   // wG[0], hG[0], wG[1], wG[2]
    int w32, h32;                       // full 32 x 32 cells along x / y
    float minGradHistCut, minGradHistAdd;
    float *ths, *thsS;                  // [w32*h32] ths and thsSmoothed
    const uint8_t *rp;                  // randomPattern, w*h bytes
    // one pass
    int pot, cw, ch, bw4, bh4;          // potential; pot cells (ceil(w/pot) x ceil(h/pot)); 4pot blocks
    float thFactor, dw1, dw2;
    int dirDist;                        // setting_selectDirectionDistribution
    uint16_t *mask;                     // [cw*ch]
    uint8_t *dir;                       // [cw*ch] direction index each pot cell starts with
    uint8_t *map;                       // [w*h] 0 or PixelSelectorStatus 1 / 2 / 4
    int *hdr;                           // PIXSEL_HDR_INTS
    // the selected pixels
    int *rowcnt, *rowoff;               // [h]
    int *list;                          // [w*h] pixel indices in raster order
    int charTH;                         // 255 keeps every pixel
    int32_t *sx, *sy; uint8_t *stype;   // kept pixels (may be null)
    float *fu, *fv, *ftype;             // kept pixels in makeNewTraces' range (may be null)
};

// select()'s 16 directions (PixelSelector2.cc:185-201), the double literals rounded to float as Vec2f's constructor does
__constant__ float c_pixsel_dir[16][2] = {
    {0, 1.0000}, {0.3827, 0.9239}, {0.1951, 0.9808}, {0.9239, 0.3827}, {0.7071, 0.7071}, {0.3827, -0.9239}, {0.8315, 0.5556},
    {0.8315, -0.5556}, {0.5556, -0.8315}, {0.9808, 0.1951}, {0.9239, -0.3827}, {0.7071, -0.7071}, {0.5556, 0.8315},
    {0.9808, -0.1951}, {1.0000, 0.0000}, {0.1951, -0.9808}};

// thsSmoothed[(xf>>5) + (yf>>5)*thsStep]: the flat index wraps into the next row as the reference's does; entries at or past
// w32*h32, which makeHists never writes, read 0
__device__ __forceinline__ float pixsel_th(const PixselArgs &a, int xf, int yf) {
    const int i = (xf >> 5) + (yf >> 5) * a.w32;
    return i < a.w32 * a.h32 ? a.thsS[i] : 0.f;
}

// |dot(grad, dir)| of Vec2f::dot (a0*b0 + a1*b1), or ag when selectDirectionDistribution is off
__device__ __forceinline__ float pixsel_dirnorm(const PixselArgs &a, float4 t, int d, float ag) {
    if (!a.dirDist) return ag;
    return fabsf(__fadd_rn(__fmul_rn(t.y, c_pixsel_dir[d][0]), __fmul_rn(t.z, c_pixsel_dir[d][1])));
}

__global__ void __launch_bounds__(1024) k_pixsel_hist(PixselArgs a) {
    __shared__ int hist[50];
    const int cx = blockIdx.x % a.w32, cy = blockIdx.x / a.w32;
    if (threadIdx.x < 50) hist[threadIdx.x] = 0;
    __syncthreads();
    const int it = 32 * cx + (threadIdx.x & 31), jt = 32 * cy + (threadIdx.x >> 5);
    if (!(it > a.w - 2 || jt > a.h - 2 || it < 1 || jt < 1)) {
        const float s = __fsqrt_rn(pyr_abs_sq_grad(a.img0, a.B, it + jt * a.w));
        int g = isnan(s) ? 48 : (int) s;               // a NaN gradient goes to bin 48 (DESIGN.md)
        if (g > 48) g = 48;
        atomicAdd(&hist[g + 1], 1);
        atomicAdd(&hist[0], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        // computeHistQuantil (:27-34); the bins past 49, never written by makeHists, read 0
        int th = (int) __fadd_rn(__fmul_rn((float) hist[0], a.minGradHistCut), 0.5f);
        int q = 90;
        for (int i = 0; i < 90; i++) {
            th -= i + 1 < 50 ? hist[i + 1] : 0;
            if (th < 0) { q = i; break; }
        }
        a.ths[blockIdx.x] = __fadd_rn((float) q, a.minGradHistAdd);
    }
}

__global__ void k_pixsel_smooth(PixselArgs a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.w32 * a.h32) return;
    const int x = i % a.w32, y = i / a.w32, w32 = a.w32, h32 = a.h32;
    const float *ths = a.ths;
    float sum = 0, num = 0;
    if (x > 0) {
        if (y > 0) { num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x - 1 + (y - 1) * w32]); }
        if (y < h32 - 1) { num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x - 1 + (y + 1) * w32]); }
        num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x - 1 + y * w32]);
    }
    if (x < w32 - 1) {
        if (y > 0) { num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x + 1 + (y - 1) * w32]); }
        if (y < h32 - 1) { num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x + 1 + (y + 1) * w32]); }
        num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x + 1 + y * w32]);
    }
    if (y > 0) { num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x + (y - 1) * w32]); }
    if (y < h32 - 1) { num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x + (y + 1) * w32]); }
    num = __fadd_rn(num, 1.f); sum = __fadd_rn(sum, ths[x + y * w32]);
    const float q = __fdiv_rn(sum, num);
    a.thsS[i] = __fmul_rn(q, q);
}

__global__ void k_pixsel_mask(PixselArgs a) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= a.cw * a.ch) return;
    const int pot = a.pot, x0 = (c % a.cw) * pot, y0 = (c / a.cw) * pot;
    const int my1 = min(pot, a.h - y0), mx1 = min(pot, a.w - x0);
    unsigned m = 0;
    for (int y1 = 0; y1 < my1 && m != 0xFFFFu; y1++)
        for (int x1 = 0; x1 < mx1 && m != 0xFFFFu; x1++) {
            const int xf = x0 + x1, yf = y0 + y1;
            if (xf < 4 || xf >= a.w - 5 || yf < 4 || yf > a.h - 4) continue;
            const int idx = xf + yf * a.w;
            const float ag0 = pyr_abs_sq_grad(a.img0, a.B, idx);
            if (!(ag0 > __fmul_rn(pixsel_th(a, xf, yf), a.thFactor))) continue;
            const float4 t = a.img0[idx];
            for (int d = 0; d < 16; d++)
                if (pixsel_dirnorm(a, t, d, ag0) > 0.f) m |= 1u << d;
        }
    a.mask[c] = (uint16_t) m;
}

// One warp. Lane l of a round takes 4pot block 2*round + l/16 (raster order) and, inside it, the pot cell s = l%16 in the nested
// order: 2pot block s/4 (y outer), pot cell s%4 (y outer). Cells past the image edge do not exist and never pick. A cell whose mask
// is empty or full picks whatever its direction; the mixed ones are resolved in lane order from the running n2.
__global__ void __launch_bounds__(32) k_pixsel_walk(PixselArgs a) {
    const int lane = threadIdx.x;
    const unsigned lt = (1u << lane) - 1u;
    const int nb = a.bw4 * a.bh4;
    int base = 0, mixed = 0;
    for (int b0 = 0; b0 < nb; b0 += 2) {
        const int b = b0 + (lane >> 4), s = lane & 15;
        const int cx = (b % a.bw4) * 4 + ((s >> 2) & 1) * 2 + (s & 1), cy = (b / a.bw4) * 4 + (s >> 3) * 2 + ((s >> 1) & 1);
        const bool exists = b < nb && cx < a.cw && cy < a.ch;
        const unsigned m = exists ? a.mask[cy * a.cw + cx] : 0u;
        unsigned picks = __ballot_sync(0xffffffffu, m == 0xFFFFu);
        unsigned mix = __ballot_sync(0xffffffffu, m != 0u && m != 0xFFFFu);
        mixed += __popc(mix);
        while (mix) {
            const int j = __ffs(mix) - 1;
            mix &= mix - 1;
            const unsigned mj = __shfl_sync(0xffffffffu, m, j);
            const int d = a.rp[base + __popc(picks & ((1u << j) - 1u))] & 15;
            if ((mj >> d) & 1u) picks |= 1u << j;
        }
        if (exists) a.dir[cy * a.cw + cx] = a.rp[base + __popc(picks & lt)] & 15;
        base += __popc(picks);
    }
    if (lane == 0) a.hdr[PIXSEL_MIXED] = mixed;
}

__global__ void k_pixsel_pick(PixselArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.bw4 * a.bh4) return;
    const int pot = a.pot, w = a.w, h = a.h;
    const int x4 = (b % a.bw4) * 4 * pot, y4 = (b / a.bw4) * 4 * pot;
    const float dw1 = a.dw1, dw2 = a.dw2, thFactor = a.thFactor;
    int n2 = 0, n3 = 0, n4 = 0;
    const int my3 = min(4 * pot, h - y4), mx3 = min(4 * pot, w - x4);
    int bestIdx4 = -1;
    float bestVal4 = 0;
    const int dir4 = a.dir[(y4 / pot) * a.cw + x4 / pot];
    for (int y3 = 0; y3 < my3; y3 += 2 * pot)
        for (int x3 = 0; x3 < mx3; x3 += 2 * pot) {
            const int x34 = x3 + x4, y34 = y3 + y4;
            const int my2 = min(2 * pot, h - y34), mx2 = min(2 * pot, w - x34);
            int bestIdx3 = -1;
            float bestVal3 = 0;
            const int dir3 = a.dir[(y34 / pot) * a.cw + x34 / pot];
            for (int y2 = 0; y2 < my2; y2 += pot)
                for (int x2 = 0; x2 < mx2; x2 += pot) {
                    const int x234 = x2 + x34, y234 = y2 + y34;
                    const int my1 = min(pot, h - y234), mx1 = min(pot, w - x234);
                    int bestIdx2 = -1;
                    float bestVal2 = 0;
                    const int dir2 = a.dir[(y234 / pot) * a.cw + x234 / pot];
                    for (int y1 = 0; y1 < my1; y1 += 1)
                        for (int x1 = 0; x1 < mx1; x1 += 1) {
                            const int idx = x1 + x234 + w * (y1 + y234);
                            const int xf = x1 + x234, yf = y1 + y234;
                            if (xf < 4 || xf >= w - 5 || yf < 4 || yf > h - 4) continue;
                            const float pixelTH0 = pixsel_th(a, xf, yf);
                            const float pixelTH1 = __fmul_rn(pixelTH0, dw1);
                            const float pixelTH2 = __fmul_rn(pixelTH1, dw2);
                            const float ag0 = pyr_abs_sq_grad(a.img0, a.B, idx);
                            if (ag0 > __fmul_rn(pixelTH0, thFactor)) {
                                const float dirNorm = pixsel_dirnorm(a, a.img0[idx], dir2, ag0);
                                if (dirNorm > bestVal2) { bestVal2 = dirNorm; bestIdx2 = idx; bestIdx3 = -2; bestIdx4 = -2; }
                            }
                            if (bestIdx3 == -2) continue;
                            const float ag1 = pyr_abs_sq_grad(a.img1, a.B, (int) __fadd_rn(__fmul_rn((float) xf, 0.5f), 0.25f) +
                                                                           (int) __fadd_rn(__fmul_rn((float) yf, 0.5f), 0.25f) * a.w1);
                            if (ag1 > __fmul_rn(pixelTH1, thFactor)) {
                                const float dirNorm = pixsel_dirnorm(a, a.img0[idx], dir3, ag1);
                                if (dirNorm > bestVal3) { bestVal3 = dirNorm; bestIdx3 = idx; bestIdx4 = -2; }
                            }
                            if (bestIdx4 == -2) continue;
                            // (int)(xf*0.25f + 0.125): a float product and a double sum
                            const float ag2 = pyr_abs_sq_grad(a.img2, a.B, (int) ((double) __fmul_rn((float) xf, 0.25f) + 0.125) +
                                                                           (int) ((double) __fmul_rn((float) yf, 0.25f) + 0.125) * a.w2);
                            if (ag2 > __fmul_rn(pixelTH2, thFactor)) {
                                const float dirNorm = pixsel_dirnorm(a, a.img0[idx], dir4, ag2);
                                if (dirNorm > bestVal4) { bestVal4 = dirNorm; bestIdx4 = idx; }
                            }
                        }
                    if (bestIdx2 > 0) { a.map[bestIdx2] = 1; bestVal3 = 1e10f; n2++; }
                }
            if (bestIdx3 > 0) { a.map[bestIdx3] = 2; bestVal4 = 1e10f; n3++; }
        }
    if (bestIdx4 > 0) { a.map[bestIdx4] = 4; n4++; }
    if (n2) atomicAdd(&a.hdr[PIXSEL_N2], n2);
    if (n3) atomicAdd(&a.hdr[PIXSEL_N3], n3);
    if (n4) atomicAdd(&a.hdr[PIXSEL_N4], n4);
}

// one warp per row: the row's selected pixels
__global__ void k_pixsel_rows(PixselArgs a) {
    const int y = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (y >= a.h) return;
    const uint8_t *row = a.map + (size_t) y * a.w;
    int n = 0;
    for (int x = lane; x < a.w; x += 32) n += row[x] != 0;
    for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if (lane == 0) a.rowcnt[y] = n;
}

__global__ void __launch_bounds__(1024) k_pixsel_row_scan(PixselArgs a) {
    __shared__ int s[33];
    int carry = 0;
    for (int y0 = 0; y0 < a.h; y0 += 1024) {
        const int y = y0 + threadIdx.x;
        const int n = y < a.h ? a.rowcnt[y] : 0;
        int tot;
        const int o = imm_block_scan(n, s, &tot);
        if (y < a.h) a.rowoff[y] = carry + o;
        carry += tot;
    }
    if (threadIdx.x == 0) a.hdr[PIXSEL_NSEL] = carry;
}

__global__ void k_pixsel_emit(PixselArgs a) {
    const int y = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (y >= a.h) return;
    const uint8_t *row = a.map + (size_t) y * a.w;
    int o = a.rowoff[y];
    for (int x0 = 0; x0 < a.w; x0 += 32) {
        const int x = x0 + lane;
        const bool sel = x < a.w && row[x] != 0;
        const unsigned b = __ballot_sync(0xffffffffu, sel);
        if (sel) a.list[o + __popc(b & ((1u << lane) - 1u))] = y * a.w + x;
        o += __popc(b);
    }
}

// makeMaps' subsampling (:150-163) over the selected pixels in raster order, and the output lists
__global__ void __launch_bounds__(1024) k_pixsel_finish(PixselArgs a) {
    __shared__ int s[33];
    const int n = a.hdr[PIXSEL_NSEL];
    int ok = 0, of = 0;
    for (int r0 = 0; r0 < n; r0 += 1024) {
        const int r = r0 + threadIdx.x;
        int idx = 0, t = 0;
        bool keep = false;
        if (r < n) {
            idx = a.list[r];
            t = a.map[idx];
            keep = (int) a.rp[r] <= a.charTH;
            if (!keep) a.map[idx] = 0;
        }
        const int x = idx % a.w, y = idx / a.w;
        const bool feat = keep && x >= 3 && x < a.w - 4 && y >= 3 && y < a.h - 4;
        int tk, tf;
        const int pk = ok + imm_block_scan(keep, s, &tk);
        const int pf = of + imm_block_scan(feat, s, &tf);
        if (keep && a.sx) { a.sx[pk] = x; a.sy[pk] = y; a.stype[pk] = (uint8_t) t; }
        if (feat && a.fu) { a.fu[pf] = (float) x; a.fv[pf] = (float) y; a.ftype[pf] = (float) t; }
        ok += tk; of += tf;
    }
    if (threadIdx.x == 0) { a.hdr[PIXSEL_NKEPT] = ok; a.hdr[PIXSEL_NFEAT] = of; }
}
