// ldso_b200 — shared device/host definitions for the sm_90a kernels and the C ABI (include/ldso_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include "../../include/ldso_b200.h"

#define MAXF LDSO_B200_MAX_FRAMES
#define MAXPAIR (MAXF * MAXF)
#define MAXN (8 * MAXF + 4)          // 68
#define MAXLVL LDSO_B200_MAX_LEVELS
#define CPARS 4

// scale constants, include/Settings.h:26-43 of the reference
#define SCALE_IDEPTH 1.0f
#define SCALE_XI_ROT 1.0f
#define SCALE_XI_TRANS 0.5f
#define SCALE_F 50.0f
#define SCALE_C 50.0f
#define SCALE_A 10.0f
#define SCALE_B 1000.0f

// ---- K1 (linearize + accumulate) geometry ---------------------------------------------------------------
#define K1_THREADS 256
#define K1_GROUPS (K1_THREADS / 8)    // 8-lane groups (one residual each) per CTA round
#define REC 52                        // floats per residual record staged in shared memory
// record layout (floats)
#define REC_X 0        // [0..9]   x = [Jpdc[0](4) | Jpdxi[0](6)]
#define REC_Y 10       // [10..19] y = [Jpdc[1](4) | Jpdxi[1](6)]
#define REC_A 20       // JIdx2(0,0)
#define REC_B 21       // JIdx2(0,1)
#define REC_C 22       // JIdx2(1,1)
#define REC_JABJI 23   // [23..26] JabJIdx 00 01 10 11
#define REC_JIR 27     // [27,28]  JI_r
#define REC_JAB2 29    // [29..31] Jab2 00 01 11
#define REC_JABR 32    // [32,33]  Jab_r
#define REC_RR 34
#define REC_ACTIVE 35
#define REC_JPJD 36    // [36..43] JpJdF
#define REC_HDD 44
#define REC_BD 45
#define REC_HCD 46     // [46..49]
#define REC_JPDD 50    // [50,51]

// per-work-item partial accumulator layout (floats)
#define PART_TOP 0                       // [MAXF][96]  (91 used) per target
#define PART_D (MAXF * 96)               // 768: [MAXF][MAXF][64] blocked (t1,t2) 8x8 row-major
#define PART_E (PART_D + 4096)           // 4864: [MAXF][8][4]
#define PART_EB (PART_E + 256)           // 5120: [MAXF][8]
#define PART_HCC (PART_EB + 64)          // 5184: [4][4]
#define PART_BC (PART_HCC + 16)          // 5200: [4]
#define PART_USED (PART_BC + 4)          // 5204
#define PART_STRIDE 5216

// reduced (double) buffer layout: [MAXF hosts][PART_USED] then the scalar stats, then the newest-frame energies
#define RED_STATS (MAXF * PART_USED)     // 41632
#define RED_NSTATS 8                     // energy, nres_active, sumNID, numID, ...
#define RED_SELECT (RED_STATS + RED_NSTATS)

// K1 flags
#define K1F_APPLY_STEP 1      // resubstitute + idepth step from the previous solve, before linearizing
#define K1F_LINEARIZE 2       // linearize from images (else: rebuild records from the stored J)
#define K1F_ACCUMULATE 4      // run the Hessian accumulation phases and write partials
#define K1F_STORE_J 8         // write RawResidualJacobian/projectedTo/centerProjectedTo to global
#define K1F_APPLY_RES 16      // fused PointFrameResidual::applyRes(true)
#define K1F_RESET_OOB 32      // PointFrameResidual::resetOOB before linearizing
#define K1F_MODE_SHIFT 8      // bits 8..9: accumulate mode 0/1/2 (AccumulatedTopHessian.cc:9)
#define K1F_NO_SHIFT_PRIOR 1024  // SC addPoint(p, shiftPriorToZero=false) (marginalizePointsF)

struct PairRec {          // FrameFramePrecalc fields the residual reads (FrameFramePrecalc.h:35-44), 32 floats
    float R0[9];          // PRE_RTll_0
    float t0[3];          // PRE_tTll_0
    float KRKi[9];        // PRE_KRKiTll
    float Kt[3];          // PRE_KtTll
    float aff[2];         // PRE_aff_mode
    float b0;             // PRE_b0_mode
    float distanceLL;
    float pad[4];
};

struct PairRecFull {      // the fields only the host mirrors read
    float RTll[9];
    float tTll[3];
};

struct FrameDev {
    double evalR[9], evalT[3];
    double state[10], state_zero[10], state_backup[10], step[10];
    double preR[9], preT[3];            // PRE_worldToCam
    double prior[8], delta_prior[8], delta[8];
    float frameEnergyTH;
    float ab_exposure;
    int frame_id;
    int slot;
};

struct CalibDev {
    double value[4], value_zero[4], value_backup[4], step[4], value_scaled[4];
    float fxl, fyl, cxl, cyl, fxli, fyli, cxli, cyli;
    float cDeltaF[4];
};

struct ImgLevel {
    const float4 *p;
    int w, h;
};

// Everything about the keyframe window that changes per Gauss-Newton step; lives in global memory.
struct WinState {
    int nF, n;
    int w, h;
    float wM3G, hM3G;
    ldso_b200_settings S;
    FrameDev fr[MAXF];
    CalibDev calib;
    alignas(16) PairRec pair[MAXPAIR];            // index h + nF*t
    PairRecFull pairFull[MAXPAIR];
    alignas(16) float adHTdeltaF[MAXPAIR][8];     // index h + nF*t
    alignas(16) float xAd[MAXPAIR][8];            // index h*nF + t  (EnergyFunctional.cc:503)
    float cstep[4];
    double adHost[MAXPAIR][64], adTarget[MAXPAIR][64];   // index h + nF*t, 8x8 row-major
    float adHostF[MAXPAIR][64], adTargetF[MAXPAIR][64];
    double cPrior[4];
    const float4 *img0[MAXF];         // level-0 texels of each window frame
    // scalars produced on the device
    double energy;                    // last linearizeAll energy (lastEnergyP)
    int resInA;
    int resInA_solved;                // resInA of the system the last K3 solve used (EnergyFunctional::resInA after solveSystemF)
    int canbreak;
    int iteration_count;
    float sumNID, numID;
    float frameEnergyTH[MAXF];       // FrameHessian::frameEnergyTH of the window frames (the newest one is moved by setNewFrameEnergyTH on the device)
    long long dbg[64];               // clock64() phase stamps of the last K3 (development aid)
};

// device pointers of the flattened window
struct DevWindow {
    int nP, nR, nItems;
    const int *pt_host, *pt_res_begin;
    float *pt_u, *pt_v, *pt_idepth, *pt_idepth_zero, *pt_idepth_backup, *pt_step;
    float *pt_color, *pt_weights, *pt_priorF;
    float *pt_HdiF, *pt_bdSumF, *pt_Hcd, *pt_Hdd, *pt_bd;      // current solve (A + L sums)
    float *pt_HddL, *pt_bdL, *pt_HcdL;                          // Hdd_accLF etc. (modes 1/2)
    const int *res_point, *res_target;
    uint8_t *res_state, *res_new_state, *res_active, *res_lin;
    float *res_energy, *res_new_energy, *res_new_energy_wo;
    float *res_JpJdF, *res_JpJdF_new;
    float *res_J, *res_proj, *res_cpt, *res_toZero;
    const int *res_newest_slot;
    const int4 *items;            // (host, p0, p1, 0)
    const int *host_item_begin;   // [MAXF+1]
    float *partials;              // [nItems][PART_STRIDE]
    double *item_stats;           // [nItems][4]: energy, nres, sumNID, numID
    double *red;                  // reduced buffer (RED_* layout)
    int newest_offset, newest_total;
    int pts_per_item;
    long long *dbg;               // clock64() phase stamps of K1's CTA 0 (development aid)
};

// Programmatic dependent launch (sm_90+): the four kernels of a Gauss-Newton iteration are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization, so kernel N+1 may become resident and run its prologue while
// kernel N is still executing. RULE: before pdl_wait() a kernel may only read data that is constant for the whole
// iteration (window inputs, set_frames constants, settings) and may not write global memory; everything produced by
// an earlier kernel of the chain is touched only after pdl_wait() (which returns once all prerequisite grids have
// completed and flushed). Both are no-ops for a kernel launched without the attribute.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// Development instrumentation (clock64 / globaltimer stamps written by the kernels, tools/k3clk.py): compiled in only with
// -DLDSO_B200_PROFILE (LDSO_B200_CFLAGS=-DLDSO_B200_PROFILE python -m ldso_b200.build --force); production kernels carry none.
#ifdef LDSO_B200_PROFILE
#define PROF_ONLY(...) __VA_ARGS__
#else
#define PROF_ONLY(...)
#endif

#define CUDA_CHECK_RET(ctx, call)                                                         \
    do {                                                                                  \
        cudaError_t e__ = (call);                                                         \
        if (e__ != cudaSuccess) return (ctx)->fail_cuda(e__, #call, __FILE__, __LINE__);  \
    } while (0)

// exclusive prefix sum over a 1024-thread block; *total gets the block's sum (s holds 33 ints)
__device__ __forceinline__ int imm_block_scan(int x, int *s, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = x;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int t = s[lane], ti = t;
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += y; }
        s[lane] = ti - t;
        if (lane == 31) s[32] = ti;
    }
    __syncthreads();
    const int r = s[warp] + inc - x;
    *total = s[32];
    __syncthreads();
    return r;
}
