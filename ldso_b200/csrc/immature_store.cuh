// The immature-point store: every keyframe's ImmaturePoints kept on the device between calls (DESIGN.md "Immature-point store").
// One segment per image slot, holding the candidates of the keyframe seeded from that slot in feature-index order, as a structure
// of arrays with the segment's capacity as stride. Included by trace.cu only (built with -fmad=false): seeding, tracing and the
// activation LM reuse the constructor, traceOn and optimizeImmaturePoint bodies of trace_kernels.cuh, so their bits are the
// one-shot entry points' bits.
#pragma once
#include "trace_kernels.cuh"
#include "immature_store.h"

// The ImmaturePoint constructor for entries 0..n-1 of a segment (n from n_dev when given): u, v and my_type are copied in from src_*
// (my_type 1 when src_type is null; the sources may be the segment's own arrays), then the fresh trace state: idepth_min 0,
// idepth_max NaN, quality 10000, UNINITIALIZED (ImmaturePoint.h:103-121).
__global__ void k_store_seed(const int *n_dev, int n, const float *src_u, const float *src_v, const float *src_type, const float4 *img, int w,
                             TraceSettingsDev S, float *store, int cap, int slot) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (n_dev ? *n_dev : n)) return;
    const ImmSeg g = imm_seg(store, cap, slot);
    const float u = src_u[i], v = src_v[i], t = src_type ? src_type[i] : 1.f;
    g.u[i] = u; g.v[i] = v; g.my_type[i] = t;
    for (int k = 0; k < 8; k++) { g.color8[8 * i + k] = 0.f; g.weights8[8 * i + k] = 0.f; }
    immature_init_one(i, img, w, g.u, g.v, S, g.color8, g.weights8, g.gradH4, g.energyTH);
    g.idmin[i] = 0.f; g.idmax[i] = NAN; g.quality[i] = 10000.f; g.status[i] = IPS_UNINITIALIZED;
    g.uv2[2 * i] = 0.f; g.uv2[2 * i + 1] = 0.f; g.interval[i] = 0.f; g.live[i] = 1;
}

// makeNewTraces' energyTH check (FullSystem.cc:1298-1302): entries 0..n-1 of a freshly seeded segment whose energyTH is not finite
// are dropped, the others move down in order; *n_out gets the count kept. One CTA, in rounds of 1024 entries: a round reads its
// entries before any of them is written, and an entry only ever moves to a lower index, so no entry is overwritten before it moved.
__global__ void __launch_bounds__(1024) k_store_compact(float *store, int cap, int slot, int n, int *n_out) {
    __shared__ int s[33];
    const ImmSeg g = imm_seg(store, cap, slot);
    float *const f1[] = {g.u, g.v, g.my_type, g.energyTH, g.idmin, g.idmax, g.quality, (float *) g.status, g.interval, (float *) g.live};
    int o = 0;
    for (int r0 = 0; r0 < n; r0 += 1024) {
        const int i = r0 + threadIdx.x;
        const bool keep = i < n && isfinite(g.energyTH[i]);
        int tot;
        const int d = o + imm_block_scan(keep, s, &tot);
        if (o != r0 || tot != min(1024, n - r0)) {       // something moves in this round
            float r[IMM_SEG_WORDS];
            if (keep) {
                for (int k = 0; k < 10; k++) r[k] = f1[k][i];
                for (int k = 0; k < 8; k++) { r[10 + k] = g.color8[8 * i + k]; r[18 + k] = g.weights8[8 * i + k]; }
                for (int k = 0; k < 4; k++) r[26 + k] = g.gradH4[4 * i + k];
                r[30] = g.uv2[2 * i]; r[31] = g.uv2[2 * i + 1];
            }
            __syncthreads();
            if (keep) {
                for (int k = 0; k < 10; k++) f1[k][d] = r[k];
                for (int k = 0; k < 8; k++) { g.color8[8 * d + k] = r[10 + k]; g.weights8[8 * d + k] = r[18 + k]; }
                for (int k = 0; k < 4; k++) g.gradH4[4 * d + k] = r[26 + k];
                g.uv2[2 * d] = r[30]; g.uv2[2 * d + 1] = r[31];
            }
            __syncthreads();
        }
        o += tot;
    }
    if (threadIdx.x == 0) *n_out = o;
}

// One traceNewCoarse pass over the listed segments: warp w takes entry w - begin[j] of segment j, skips it when it is not live, and
// runs traceOn with segment j's host transform. counts (optional) accumulates traceNewCoarse's seven counters.
__global__ void __launch_bounds__(32 * KTR_WARPS) k_store_trace(const __grid_constant__ StoreTraceArgs P) {
    __shared__ float s_err[KTR_WARPS][100];
    __shared__ int s_cnt[7];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int gw = blockIdx.x * KTR_WARPS + wib;
    if (P.counts && threadIdx.x < 7) s_cnt[threadIdx.x] = 0;
    if (P.counts) __syncthreads();
    if (gw < P.begin[P.nseg]) {
        int j = 0;
        while (gw >= P.begin[j + 1]) j++;
        const int k = gw - P.begin[j];
        const ImmSeg g = imm_seg(P.store, P.cap, P.slot[j]);
        if (g.live[k]) {
            TraceArgs A = P.T;
            A.u = g.u; A.v = g.v; A.color8 = g.color8; A.weights8 = g.weights8; A.gradH4 = g.gradH4; A.energyTH = g.energyTH;
            A.idepth_min = g.idmin; A.idepth_max = g.idmax; A.quality = g.quality; A.status = g.status; A.uv2 = g.uv2; A.interval = g.interval;
            const int st = trace_on_one(A, k, P.KRKi[j], P.Kt[j], P.aff[j], s_err[wib]);
            if (P.counts && lane == 0) {
                atomicAdd(&s_cnt[0], 1);
                if (st >= 0 && st <= IPS_UNINITIALIZED) atomicAdd(&s_cnt[1 + st], 1);
            }
        }
    }
    if (P.counts) {
        __syncthreads();
        if (threadIdx.x < 7 && s_cnt[threadIdx.x]) atomicAdd(&P.counts[threadIdx.x], s_cnt[threadIdx.x]);
    }
}

// activatePointsMT's candidates: the live entries of the window's frames 0..nF-2 in window order, then feature-index order, gathered
// into the arrays k_activation_select reads (host = window frame). One CTA.
__global__ void __launch_bounds__(1024) k_store_gather(const __grid_constant__ StoreActArgs P) {
    __shared__ int s[33];
    const int total = P.begin[P.nseg];
    const int per = (total + 1023) / 1024, a = min(total, (int) threadIdx.x * per), b = min(total, a + per);
    int j = 0;
    while (j < P.nseg && a >= P.begin[j + 1]) j++;
    int cnt = 0;
    for (int e = a, jj = j; e < b; e++) {
        while (e >= P.begin[jj + 1]) jj++;
        cnt += imm_seg(P.store, P.cap, P.slot[jj]).live[e - P.begin[jj]] != 0;
    }
    int ntot;
    int o = imm_block_scan(cnt, s, &ntot);
    for (int e = a; e < b; e++) {
        while (e >= P.begin[j + 1]) j++;
        const int k = e - P.begin[j];
        const ImmSeg g = imm_seg(P.store, P.cap, P.slot[j]);
        if (!g.live[k]) continue;
        P.c_u[o] = g.u[k]; P.c_v[o] = g.v[k]; P.c_idmin[o] = g.idmin[k]; P.c_idmax[o] = g.idmax[k]; P.c_quality[o] = g.quality[k];
        P.c_interval[o] = g.interval[k]; P.c_type[o] = g.my_type[k]; P.c_status[o] = g.status[k]; P.c_host[o] = j; P.c_index[o] = k;
        o++;
    }
}

// the selected candidates (action 1), compacted in visiting order for the activation LM; c_sel[i] = position among them or -1
__global__ void __launch_bounds__(1024) k_store_pick(const __grid_constant__ StoreActArgs P) {
    __shared__ int s[33];
    const int n = P.n, per = (n + 1023) / 1024, a = min(n, (int) threadIdx.x * per), b = min(n, a + per);
    int cnt = 0;
    for (int i = a; i < b; i++) cnt += P.action[i] == 1;
    int ntot;
    int o = imm_block_scan(cnt, s, &ntot);
    for (int i = a; i < b; i++) {
        if (P.action[i] != 1) { P.c_sel[i] = -1; continue; }
        const ImmSeg g = imm_seg(P.store, P.cap, P.slot[P.c_host[i]]);
        const int k = P.c_index[i];
        P.c_sel[i] = o;
        P.s_u[o] = g.u[k]; P.s_v[o] = g.v[k]; P.s_host[o] = P.c_host[i]; P.s_idmin[o] = g.idmin[k]; P.s_idmax[o] = g.idmax[k];
        P.s_energyTH[o] = g.energyTH[k];
        for (int q = 0; q < 8; q++) { P.s_color8[8 * o + q] = g.color8[8 * k + q]; P.s_weights8[8 * o + q] = g.weights8[8 * k + q]; }
        o++;
    }
    if (threadIdx.x == 0) P.hdr[0] = ntot;
}

// optimizeImmaturePoint of the selected candidates; the grid covers every candidate, warps past the selected count leave at once
__global__ void __launch_bounds__(32 * KTR_WARPS) k_store_optimize(const __grid_constant__ StoreActArgs P, int minObs) {
    const int i = blockIdx.x * KTR_WARPS + (threadIdx.x >> 5);
    if (i >= P.hdr[0]) return;
    optimize_immature_one(i, P.ws, P.s_u, P.s_v, P.s_host, P.s_idmin, P.s_idmax, P.s_color8, P.s_weights8, P.s_energyTH, minObs, P.s_ok,
                          P.s_idepth, P.s_res);
}

// activatePointsMT's bookkeeping (FullSystem.cc:1104-1109, 1119-1126, 1145-1149, 1167-1186): action 2 releases the entry as OUTLIER,
// a selected one is released as VALID when its LM succeeded and as OUTLIER otherwise, action 0 stays live. The released entries are
// written as records in visiting order; hdr[1] / hdr[2] get their count and the VALID count.
__global__ void __launch_bounds__(1024) k_store_apply(const __grid_constant__ StoreActArgs P) {
    __shared__ int s[33];
    const int n = P.n, nF = P.nF, per = (n + 1023) / 1024, a = min(n, (int) threadIdx.x * per), b = min(n, a + per);
    int cnt = 0, nvalid = 0;
    for (int i = a; i < b; i++) {
        cnt += P.action[i] != 0;
        nvalid += P.action[i] == 1 && P.s_ok[P.c_sel[i]] != 0;
    }
    int ntot, vtot;
    int o = imm_block_scan(cnt, s, &ntot);
    imm_block_scan(nvalid, s, &vtot);
    for (int i = a; i < b; i++) {
        const int act = P.action[i];
        if (act == 0) continue;
        const int f = P.c_host[i], k = P.c_index[i], si = P.c_sel[i];
        const ImmSeg g = imm_seg(P.store, P.cap, P.slot[f]);
        ImmRecord &r = P.rec[o++];
        r.frame = f; r.index = k;
        r.status = (act == 1 && P.s_ok[si]) ? IMM_FEATURE_VALID : IMM_FEATURE_OUTLIER;
        r.idepth_min = g.idmin[k]; r.idepth_max = g.idmax[k]; r.idepth = act == 1 ? P.s_idepth[si] : NAN;
        r.energyTH = g.energyTH[k]; r.my_type = g.my_type[k];
        for (int q = 0; q < 8; q++) { r.color8[q] = g.color8[8 * k + q]; r.weights8[q] = g.weights8[8 * k + q]; }
        for (int t = 0; t < MAXF; t++) r.res_state[t] = (act == 1 && t < nF) ? P.s_res[(size_t) si * nF + t] : 255;
        g.live[k] = 0;
    }
    if (threadIdx.x == 0) { P.hdr[1] = ntot; P.hdr[2] = vtot; }
}
