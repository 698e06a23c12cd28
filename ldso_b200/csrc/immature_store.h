// Layout, kernel arguments and launchers of the immature-point store (immature_store.cuh, built into trace.cu).
#pragma once
#include "trace_types.h"

#define IMM_NSEG (2 * MAXF)            // one segment per image slot
#define IMM_SEG_WORDS 32               // 4-byte words per entry
#define IMM_FEATURE_VALID 1            // Feature::FeatureStatus (Feature.h:38-42)
#define IMM_FEATURE_OUTLIER 2

// One segment: cap entries of each field, fields one after another (an ImmaturePoint's members, ImmaturePoint.h:103-121, and
// the live flag: feat->status == IMMATURE && feat->ip). The whole segment is IMM_SEG_WORDS * cap words from its first field.
struct ImmSeg {
    float *u, *v, *my_type, *color8, *weights8, *gradH4, *energyTH, *idmin, *idmax, *quality;
    int *status;
    float *uv2, *interval;
    int *live;
};
__host__ __device__ inline ImmSeg imm_seg(float *store, int cap, int slot) {
    float *b = store + (size_t) slot * IMM_SEG_WORDS * cap;
    const size_t C = (size_t) cap;
    ImmSeg g;
    g.u = b; g.v = b + C; g.my_type = b + 2 * C; g.color8 = b + 3 * C; g.weights8 = b + 11 * C; g.gradH4 = b + 19 * C;
    g.energyTH = b + 23 * C; g.idmin = b + 24 * C; g.idmax = b + 25 * C; g.quality = b + 26 * C; g.status = (int *) (b + 27 * C);
    g.uv2 = b + 28 * C; g.interval = b + 30 * C; g.live = (int *) (b + 31 * C);
    return g;
}

struct StoreTraceArgs {
    TraceArgs T;                               // image, size and settings (its per-candidate pointers are set per segment)
    float *store; int cap;
    int nseg, slot[IMM_NSEG], begin[IMM_NSEG + 1];   // listed segments and the prefix sums of their entry counts
    float KRKi[IMM_NSEG][9], Kt[IMM_NSEG][3], aff[IMM_NSEG][2];
    int *counts;                               // [7] traceNewCoarse's counters, or null
};

// one released candidate of activate_immature, in the order the reference visits them
struct ImmRecord {
    int frame, index, status;
    float idepth_min, idepth_max, idepth, energyTH, my_type, color8[8], weights8[8];
    unsigned char res_state[MAXF];
};

struct StoreActArgs {
    float *store; int cap;
    int nseg, slot[IMM_NSEG], begin[IMM_NSEG + 1];   // window frames 0..nF-2 (gather) / 0..nF-1 (slot[f] for pick and apply)
    int n, nF;                                 // candidates (live entries gathered), window frames
    const WinState *ws;
    // gathered candidates, as k_activation_select reads them, with their feature index and selected position
    float *c_u, *c_v, *c_idmin, *c_idmax, *c_quality, *c_interval, *c_type;
    int *c_status, *c_host, *c_index, *c_sel;
    unsigned char *action;
    // the selected candidates and optimizeImmaturePoint's results
    float *s_u, *s_v, *s_idmin, *s_idmax, *s_color8, *s_weights8, *s_energyTH, *s_idepth;
    int *s_host, *s_ok;
    unsigned char *s_res;
    int *hdr;                                  // [0] selected, [1] released, [2] released as VALID
    ImmRecord *rec;
};

void launch_store_seed(const int *n_dev, int n, const float *src_u, const float *src_v, const float *src_type, const float4 *img, int w,
                       const TraceSettingsDev &S, float *store, int cap, int slot, cudaStream_t stream);
void launch_store_compact(float *store, int cap, int slot, int n, int *n_out, cudaStream_t stream);
void launch_store_trace(const StoreTraceArgs &P, cudaStream_t stream);
void launch_store_gather(const StoreActArgs &P, cudaStream_t stream);
void launch_store_pick(const StoreActArgs &P, cudaStream_t stream);
void launch_store_optimize(const StoreActArgs &P, int minObs, cudaStream_t stream);
void launch_store_apply(const StoreActArgs &P, cudaStream_t stream);
