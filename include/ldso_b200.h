/* ldso_b200 — C ABI of the H100-native (sm_90a) photometric bundle-adjustment / coarse-tracker hot path of LDSO.
 *
 * This is the drop-in boundary (SURVEY.md §8b, DESIGN.md §2). LDSO has no FFI of its own; the entry points
 * below are what link-compatible replacements of the reference's
 *     src/internal/Residuals.cc, src/internal/OptimizationBackend/{AccumulatedTopHessian,AccumulatedSCHessian,
 *     EnergyFunctional}.cc, src/internal/FrameFramePrecalc.cc and src/frontend/CoarseTracker.cc
 * forward to (see INTEGRATION.md for the C++ side). Each function cites the reference interface it replaces
 * (paths relative to the LDSO source tree).
 *
 * Conventions: plain pointers and sizes only; every pointer is HOST memory unless the name says `_dev`;
 * the library copies and never retains host pointers past a call; matrices are column-major like Eigen's
 * MatXX (dimension n = 8*nFrames + 4, order [fx fy cx cy | frame0(8) | frame1(8) ...]); all functions return
 * 0 on success and a negative code on failure (ldso_b200_last_error() gives the text). There is NO CPU
 * fallback: without a CUDA device every compute entry point fails with LDSO_B200_ERR_CUDA.
 */
#ifndef LDSO_B200_H_
#define LDSO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LDSO_B200_MAX_FRAMES 8      /* setting_maxFrames(7)+1, src/Setting.cc:33 */
#define LDSO_B200_MAX_LEVELS 6      /* PYR_LEVELS, include/Settings.h:8 */
#define LDSO_B200_PATTERN 8         /* patternNum, include/Settings.h:163 */

#define LDSO_B200_OK 0
#define LDSO_B200_ERR_ARG (-1)
#define LDSO_B200_ERR_CUDA (-2)
#define LDSO_B200_ERR_STATE (-3)

/* ResState, include/internal/Residuals.h:32-34 */
#define LDSO_B200_RES_IN 0
#define LDSO_B200_RES_OOB 1
#define LDSO_B200_RES_OUTLIER 2

typedef struct ldso_b200_ctx ldso_b200_ctx;

/* The mutable globals of src/Setting.cc the path reads (reference defaults in ldso_b200_default_settings). */
typedef struct ldso_b200_settings {
    float huberTH;                    /* setting_huberTH                 Setting.cc:76 */
    float outlierTHSumComponent;      /* setting_outlierTHSumComponent   :41 */
    float affineOptModeA;             /* setting_affineOptModeA          :65 */
    float affineOptModeB;             /* setting_affineOptModeB          :66 */
    float idepthFixPrior;             /* setting_idepthFixPrior          :16 */
    float initialTransPrior;          /* :19 */
    float initialRotPrior;            /* :18 */
    float initialAffAPrior;           /* :21 */
    float initialAffBPrior;           /* :20 */
    float initialCalibHessian;        /* :22 */
    float frameEnergyTHN;             /* :78 */
    float frameEnergyTHFacMedian;     /* :80 */
    float frameEnergyTHConstWeight;   /* :77 */
    float overallEnergyTHWeight;      /* :81 */
    float coarseCutoffTH;             /* :82 */
    float thOptIterations;            /* :37 */
    double solverModeDelta;           /* :24 */
    float margWeightFac;              /* setting_margWeightFac           :45 */
    /* immature-point tracing (ImmaturePoint::traceOn) */
    float maxPixSearch;               /* setting_maxPixSearch            :28 */
    float outlierTH;                  /* setting_outlierTH               :39 */
    float trace_stepsize;             /* :89 */
    float trace_GNThreshold;          /* :91 */
    float trace_extraSlackOnTH;       /* :92 */
    float trace_slackInterval;        /* :93 */
    float trace_minImprovementFactor; /* :94 */
    int32_t minTraceTestRadius;       /* :52 */
    int32_t trace_GNIterations;       /* :90 */
} ldso_b200_settings;

void ldso_b200_default_settings(ldso_b200_settings *s);

/* ---- context ------------------------------------------------------------------------------------------ */
/* w,h = wG[0],hG[0]; pyr_levels = pyrLevelsUsed (src/internal/GlobalCalib.cc:20-75). */
ldso_b200_ctx *ldso_b200_create(int device, int w, int h, int pyr_levels, const ldso_b200_settings *settings);
void ldso_b200_destroy(ldso_b200_ctx *ctx);
const char *ldso_b200_last_error(const ldso_b200_ctx *ctx);
/* Run all work of this context on the caller's CUDA stream (cudaStream_t passed as void*). */
int ldso_b200_set_stream(ldso_b200_ctx *ctx, void *cuda_stream);
int ldso_b200_synchronize(ldso_b200_ctx *ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
long long ldso_b200_launch_count(const ldso_b200_ctx *ctx);

/* ---- keyframe images -----------------------------------------------------------------------------------
 * Replaces the host-resident FrameHessian::dIp[lvl] (include/internal/FrameHessian.h:169): `dIp[l]` is the
 * (I,dx,dy) Eigen::Vector3f array of level l exactly as FrameHessian::makeImages leaves it
 * (src/internal/FrameHessian.cc:44-98). Stored on the device as 16-byte texels. slot in [0, 2*MAX_FRAMES). */
int ldso_b200_upload_frame(ldso_b200_ctx *ctx, int slot, const float *const *dIp, int n_levels);
/* Device-side FrameHessian::makeImages: upload the raw irradiance image (w*h floats) and build the pyramid
 * with gradients on the GPU (SURVEY.md §8f rank 1). */
int ldso_b200_make_images(ldso_b200_ctx *ctx, int slot, const float *color);
/* read a level back as (I,dx,dy) AoS — tests only */
int ldso_b200_download_frame_level(ldso_b200_ctx *ctx, int slot, int lvl, float *dIp_out);

/* ---- raw camera frames: LDSO's per-frame undistortion on the device ------------------------------------
 * Undistort::undistort<T> (src/frontend/Undistort.cc:357-457) with PhotometricUndistorter::processFrame<T> (:189-227) in front
 * of makeImages: the raw 8- or 16-bit frame goes through the inverse response G (and the vignette in mode 2) and is bilinearly
 * remapped onto the rectified grid in one kernel, and the pyramid is built from the result as ldso_b200_make_images does.
 * The tables are the ones LDSO's Undistort built from its calibration files. Every output pixel equals the reference's bit for bit,
 * except where the reference reads past the end of its raw buffer (a remap offset of exactly (hOrg-1)*wOrg or (hOrg-1)*wOrg - 1):
 * those taps read 0 here. The benchmark noise settings (benchmark_varNoise, benchmark_varBlurNoise) are not supported. */
typedef struct ldso_b200_undistort_calib {
    int wOrg, hOrg;                 /* raw frame size (Undistort::getOriginalSize) */
    int w, h;                       /* rectified size (Undistort::getSize): must be the context's w x h */
    const float *remapX, *remapY;   /* w*h each (Undistort::remapX / remapY); both NULL = passthrough (needs wOrg x hOrg == w x h) */
    const float *G;                 /* PhotometricUndistorter::G, g_entries floats (256 or 65536); NULL = no valid calibration
                                     * (getG() == 0): every frame takes the factor path */
    int g_entries;
    const float *vignetteMapInv;    /* wOrg*hOrg floats; needed when G is given and photometric_mode == 2 */
    int photometric_mode;           /* setting_photometricCalibration: 0, 1 or 2 */
    int use_exposure;               /* setting_useExposure */
} ldso_b200_undistort_calib;
/* Copies the tables to the device (synchronising the context's stream). LDSO_B200_ERR_ARG for an inconsistent calibration: a
 * rectified size other than the context's, one of remapX / remapY missing, passthrough with wOrg x hOrg != w x h, g_entries
 * other than 256 / 65536 with G, photometric_mode 2 with G but no vignetteMapInv, photometric_mode outside 0..2. */
int ldso_b200_set_undistort(ldso_b200_ctx *ctx, const ldso_b200_undistort_calib *calib);
/* One raw frame (wOrg*hOrg pixels of bytes_per_pixel = 1 or 2 bytes) -> rectified irradiance -> the pyramid of `slot`, as
 * undistort<T>(raw, exposure, 0, factor) followed by makeImages. *exposure_time_out (may be NULL) gets processFrame's exposure
 * time: `exposure`, or 1 when use_exposure == 0. Asynchronous like ldso_b200_make_images; `raw` must stay valid until the next
 * synchronising call on the context. LDSO_B200_ERR_STATE before any set_undistort; LDSO_B200_ERR_ARG for a NULL raw, a
 * bytes_per_pixel other than 1 / 2, or a 16-bit frame with a 256-entry G. The level-0 image comes back through
 * ldso_b200_download_frame_level. */
int ldso_b200_undistort_frame(ldso_b200_ctx *ctx, int slot, const void *raw, int bytes_per_pixel, float exposure, float factor,
                              float *exposure_time_out);

/* ---- the optimisation window ---------------------------------------------------------------------------
 * Flattened EnergyFunctional::allPoints (EnergyFunctional.cc:385-401, points ordered by host keyframe as
 * makeIDX produces them) with each point's PointHessian::residuals list (CSR). */
typedef struct ldso_b200_window {
    int nPoints;
    int nResiduals;
    const int32_t *pt_host;          /* [nPoints]  FrameHessian::idx of the host, non-decreasing */
    const float *pt_u, *pt_v;        /* [nPoints]  PointHessian::u,v                 PointHessian.h:83 */
    const float *pt_idepth;          /* [nPoints]  idepth      (== idepth_scaled, SCALE_IDEPTH = 1) */
    const float *pt_idepth_zero;     /* [nPoints]  idepth_zero */
    const uint8_t *pt_has_prior;     /* [nPoints]  hasDepthPrior                     PointHessian.h:86 */
    const float *pt_color;           /* [nPoints*8] color[]                          PointHessian.h:106 */
    const float *pt_weights;         /* [nPoints*8] weights[]                        PointHessian.h:107 */
    const int32_t *res_begin;        /* [nPoints+1] CSR offsets into the residual arrays */
    const int32_t *res_target;       /* [nResiduals] targetIDX                       Residuals.h:109 */
    const uint8_t *res_state;        /* [nResiduals] state_state, may be NULL (=> IN after resetOOB) */
    const uint8_t *res_is_linearized;/* [nResiduals] isLinearized, may be NULL (=> 0) */
    const float *res_toZeroF;        /* [nResiduals*8] res_toZeroF, may be NULL */
} ldso_b200_window;

int ldso_b200_set_window(ldso_b200_ctx *ctx, const ldso_b200_window *win);

/* One keyframe's state record (include/internal/FrameHessian.h:163-201). */
typedef struct ldso_b200_frame_state {
    double evalR[9];       /* worldToCam_evalPT rotation, row-major */
    double evalT[3];       /* worldToCam_evalPT translation */
    double state_zero[10]; /* get_state_zero() (unscaled) */
    double state[10];      /* get_state()      (unscaled) */
    float ab_exposure;
    float frameEnergyTH;
    int32_t frame_id;      /* Frame::id; 0 => the gauge priors of FrameHessian::getPrior (FrameHessian.h:125-150) */
    int32_t image_slot;    /* slot given to ldso_b200_upload_frame */
} ldso_b200_frame_state;

/* Replaces EnergyFunctional::insertFrame/setAdjointsF/setDeltaF and FullSystem::setPrecalcValues
 * (EnergyFunctional.cc:30-61,403-489; FullSystem.cc:1423-1431; FrameFramePrecalc.cc:6-35): uploads the nF
 * keyframe states and the calibration (value_scaled = [fx fy cx cy] of CalibHessian, value_zero its
 * unscaled linearisation point; CalibHessian.h:71-100), computes adjoints, the 64 frame-pair precalc
 * records, adHTdeltaF and the null-space projector of EnergyFunctional::orthogonalize (:685-717). */
int ldso_b200_set_frames(ldso_b200_ctx *ctx, int nFrames, const ldso_b200_frame_state *frames,
                         const double calib_value_scaled[4], const double calib_value_zero[4]);

/* EnergyFunctional::HM / bM (EnergyFunctional.h:153-154). NULL => zero prior. */
int ldso_b200_set_marg_prior(ldso_b200_ctx *ctx, const double *HM, const double *bM);
int ldso_b200_get_marg_prior(ldso_b200_ctx *ctx, double *HM, double *bM);

/* ---- piecewise operations (each maps to one reference call) ------------------------------------------- */
/* FullSystem::linearizeAll(fixLinearization) restricted to the path (FullSystem.cc:1442-1543):
 * PointFrameResidual::linearize on every active residual (Residuals.cc:13-214), energy sum,
 * setNewFrameEnergyTH (:1762-1793), and for fixLinearization: applyRes(true).
 * flags: bit0 = store the full RawResidualJacobian / projectedTo / centerProjectedTo for read-back. */
int ldso_b200_linearize_all(ldso_b200_ctx *ctx, int fixLinearization, int flags, double *energy_out);
/* FullSystem::applyRes_Reductor -> PointFrameResidual::applyRes(true) (Residuals.h:70-87, FullSystem.cc:1706) */
int ldso_b200_apply_res(ldso_b200_ctx *ctx);
/* FullSystem::backupState (non-momentum branch), FullSystem.cc:1662-1676 */
int ldso_b200_backup_state(ldso_b200_ctx *ctx);
/* EnergyFunctional::solveSystemF(iteration, lambda, HCalib) (EnergyFunctional.cc:240-351) for the default
 * solver mode (SOLVER_FIX_LAMBDA | SOLVER_ORTHOGONALIZE_X_LATER): accumulateAF/LF/SCF_MT, the scaled 68x68
 * LDLT, orthogonalize, resubstituteF_MT. Needs a stored Jacobian (linearize_all with flags bit0) or uses the
 * on-chip records of the last linearize. Outputs may be NULL. */
int ldso_b200_solve_system(ldso_b200_ctx *ctx, int iteration, double *lastHS, double *lastbS, double *lastX);
/* The four stitched pieces of the last solve: AccumulatedTopHessianSSE::stitchDoubleMT (mode A, no priors;
 * AccumulatedTopHessian.h:64-105) and AccumulatedSCHessianSSE::stitchDoubleMT (AccumulatedSCHessian.h:64-98). */
int ldso_b200_get_system(ldso_b200_ctx *ctx, double *H_A, double *b_A, double *H_sc, double *b_sc, int *resInA);
/* FullSystem::doStepFromBackup(1,1,1,1,1) + setPrecalcValues (FullSystem.cc:1587-1622); returns canbreak. */
int ldso_b200_do_step(ldso_b200_ctx *ctx, int *canbreak);

/* FullSystem::flagPointsForRemoval's re-linearisation (FullSystem.cc:1241-1249: resetOOB, linearize, applyRes(true),
 * fixLinearizationF, Residuals.cc:216-242) of the n listed points followed by EnergyFunctional::marginalizePointsF
 * (EnergyFunctional.cc:165-222): priorF *= prior_fac (setting_idepthFixPriorMargFac), addPoint<2> + SC addPoint(p,false),
 * stitchDouble without priors, HM += setting_margWeightFac (M - Msc), bM likewise (read back with get_marg_prior;
 * get_system returns M, Mb, Msc, Mbsc). The caller then removes the points from its window (removePoint). */
int ldso_b200_marginalize_points(ldso_b200_ctx *ctx, int n, const int32_t *point_idx, float prior_fac, int *resInM);
/* EnergyFunctional::marginalizeFrame (EnergyFunctional.cc:72-129), the HM/bM algebra, on the device-resident prior:
 * the frame's block is moved to the end, its own prior added, and the 8 variables are eliminated by a scaled Schur
 * complement. HM, bM shrink to 8(nF-1)+4 (returned in *new_dim; get_marg_prior returns that size) until the next
 * set_frames. set_frames then KEEPS the prior when it is called with the remaining nF-1 frames, and extends it with a
 * zero block when one keyframe is appended (EnergyFunctional::insertFrame, :38-44); any other dimension clears it.
 * The bookkeeping half of the reference function (frame list, makeIDX, :131-150) is the caller's set_frames/set_window. */
int ldso_b200_marginalize_frame(ldso_b200_ctx *ctx, int frame_idx, int *new_dim);

/* AccumulatedTopHessianSSE::addPoint<mode> over a set of points followed by stitchDouble(usePrior = false), and
 * AccumulatedSCHessianSSE::addPoint(p, shiftPriorToZero) + stitchDouble on the same set
 * (include/internal/OptimizationBackend/AccumulatedTopHessian.h:20-125, AccumulatedSCHessian.h:17-118;
 * AccumulatedTopHessian.cc:9-118,129-255, AccumulatedSCHessian.cc:9-119): the calls behind EnergyFunctional::accumulateAF_MT /
 * accumulateLF_MT / accumulateSCF_MT (EnergyFunctional.cc:550-625) and marginalizePointsF. mode = the reference's template argument
 * (0: active, not linearized, resF; 1: active, linearized, res_toZeroF + J delta; 2: all active, res_toZeroF), 3 = modes 0 and 1 in
 * one pass (what solveSystemF sums: HA + HL). point_idx == NULL means every point. Works from the Jacobians ldso_b200_linearize_all
 * stored. Outputs are n x n / n column-major doubles without the frame / calibration priors; any of them may be NULL. */
int ldso_b200_accumulate(ldso_b200_ctx *ctx, int mode, int n_points, const int32_t *point_idx, int shift_prior_to_zero,
                         double *H_top, double *b_top, double *H_sc, double *b_sc, int *nres);

/* EnergyFunctional::calcLEnergyF_MT and calcMEnergyF (include/internal/OptimizationBackend/EnergyFunctional.h:120,126;
 * EnergyFunctional.cc:353-378, calcLEnergyPt :627-682) at the current state: energyL = frame / calibration / point priors plus the
 * linearised residuals' (2 res_toZeroF + J delta) . (J delta); energyM = delta . (2 bM + HM delta) with the device-resident prior.
 * FullSystem::optimize reads both around every step (FullSystem.cc:1697-1703). Either pointer may be NULL. */
int ldso_b200_calc_energies(ldso_b200_ctx *ctx, double *energyL, double *energyM);

/* ---- the fused, device-resident Gauss-Newton loop ------------------------------------------------------
 * FullSystem::optimize's prologue (resetOOB + linearizeAll(false) + applyRes, FullSystem.cc:734-771). */
int ldso_b200_optimize_begin(ldso_b200_ctx *ctx, double *energy_out);
/* n_iterations bodies of the loop FullSystem.cc:777-831 (forceAcceptStep) without any host round trip:
 * backupState, solveSystemF, doStepFromBackup, linearizeAll(false), applyRes. Iteration numbers
 * first_iteration.. are passed to solveSystemF (orthogonalize from iteration 2). Asynchronous on the
 * context's stream; results are fetched with the getters below (which synchronise). */
int ldso_b200_gn_iterations(ldso_b200_ctx *ctx, int first_iteration, int n_iterations);
/* FullSystem::optimize's loop with its exit (FullSystem.cc:777-831): at most max_iterations bodies (as gn_iterations runs them)
 * numbered from first_iteration; the loop stops after the body whose doStepFromBackup returned canbreak once that body's
 * iteration >= min_iterations (`if (canbreak && iteration >= setting_minOptIterations) break;`, :829; setting_minOptIterations
 * = 1, Setting.cc:37). max_iterations == 0 launches nothing. Asynchronous like gn_iterations: the decision is taken on the
 * device, inside one CUDA graph with a conditional WHILE node. Where the driver cannot build that node, without CUDA graphs
 * (LDSO_B200_NO_GRAPH) and while kernel_times is collecting, the same kernels run host-driven with one synchronise per body.
 * Either way the results are the same bits. With the peer exchange every rank takes the same decision after the same body. */
int ldso_b200_gn_iterations_until(ldso_b200_ctx *ctx, int first_iteration, int max_iterations, int min_iterations);
/* number of bodies the last gn_iterations_until (or optimize_from_host_until*) ran; synchronises */
int ldso_b200_get_iterations_run(ldso_b200_ctx *ctx, int *n);
/* which form the last gn_iterations_until ran in */
#define LDSO_B200_UNTIL_HOST 0          /* host-driven, one synchronise per body */
#define LDSO_B200_UNTIL_GRAPH_PDL 1     /* conditional WHILE node, programmatic dependent launch between the body's kernels */
#define LDSO_B200_UNTIL_GRAPH 2         /* conditional WHILE node, full dependencies between the body's kernels */
int ldso_b200_get_until_form(ldso_b200_ctx *ctx, int *form);
/* FullSystem::optimize's iteration budget (FullSystem.cc:727-732): 0 for nFrames < 2, 15 for nFrames < 4 (the `< 3 -> 20`
 * assignment is overwritten by the `< 4 -> 15` one), else max_opt_iterations (setting_maxOptIterations = 6, Setting.cc:36).
 * Needs no context; returns the budget, or LDSO_B200_ERR_ARG for a negative max_opt_iterations. */
int ldso_b200_optimize_iteration_budget(int nFrames, int max_opt_iterations);
/* ---- one call per keyframe optimisation, from host buffers ------------------------------------------------
 * What FullSystem::optimize does around the loop, as ONE call: (optionally) the newest keyframe's raw image -> device
 * makeImages, set_frames, set_window, the optimize() prologue, n_iterations Gauss-Newton iterations, and the read-back of the
 * results. The library orders the work itself: the image copy is queued first and travels while the host packs the
 * window; nothing blocks before the final wait. Inputs must stay valid until the call returns (they always do: it
 * returns after the read-back). Any output pointer may be NULL. Equivalent to the individual calls in that order. */
typedef struct ldso_b200_fused_io {
    int image_slot;                 /* slot of `image` (ignored when image == NULL) */
    const float *image;             /* w*h raw irradiance of the newest keyframe (pinned memory copies fastest), or NULL */
    int nFrames;
    const ldso_b200_frame_state *frames;
    const double *calib_value_scaled, *calib_value_zero;    /* [4] each */
    const ldso_b200_window *window;
    int first_iteration, n_iterations;
    /* outputs */
    double *lastHS, *lastbS, *lastX;                 /* (8nF+4)^2 column-major, 8nF+4, 8nF+4 */
    double *energy; int *canbreak;                   /* lastEnergyP of the final linearisation, canbreak of the last step */
    float *pt_idepth, *pt_step, *pt_HdiF;            /* [nPoints] */
    uint8_t *res_state, *res_new_state;              /* [nResiduals] */
    float *res_energy;                               /* [nResiduals] */
} ldso_b200_fused_io;
int ldso_b200_optimize_from_host(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io);
/* The same call split at its only synchronisation point: _submit queues uploads, prologue, iterations and the result read-back on the
 * context's stream and returns at once (io->image must stay valid until _wait; every other input is consumed before _submit returns);
 * _wait blocks until they are done and fills the outputs. One process may feed two contexts alternately (submit k+1, wait k): the
 * uploads of one window then overlap the kernels of the other (FullSystem keeps mapping and tracking on separate threads the same way). */
int ldso_b200_optimize_from_host_submit(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io);
int ldso_b200_optimize_from_host_wait(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io);
/* The same three calls with FullSystem::optimize's exit: the loop is gn_iterations_until(io->first_iteration, io->n_iterations,
 * min_iterations), so io->n_iterations is the MAXIMUM (pass ldso_b200_optimize_iteration_budget(nFrames, setting_maxOptIterations)).
 * *iterations_run (may be NULL) receives the number of bodies run; it rides back with the other results, so _until_submit /
 * _until_wait keep the two-context overlap of the pair above. */
int ldso_b200_optimize_from_host_until(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io, int min_iterations, int *iterations_run);
int ldso_b200_optimize_from_host_until_submit(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io, int min_iterations);
int ldso_b200_optimize_from_host_until_wait(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io, int *iterations_run);

/* ---- the end of FullSystem::optimize (FullSystem.cc:833-863), after the loop above ---------------------------------------------
 * ldso_b200_optimize_finish: the newest keyframe's new evaluation point (setEvalPT(PRE_worldToCam, newStateZero): eval pose = current
 * pose, state = state_zero = 0 except [6..7] = the current state[6..7]), setAdjointsF and setPrecalcValues for every pair, then
 * linearizeAll(true) over the window's non-linearised residuals: linearize, applyRes(true), energy, setNewFrameEnergyTH, and per
 * point the max relative baseline and the count of the residuals still active, per residual whether it is dropped
 * (ef->dropResidual). The RMSE is sqrtf((float) (energy / (patternNum * resInA))) with the resInA of the last solve; the frame is
 * lost when the energy is not finite. Asynchronous like gn_iterations_until; with fewer than 2 frames it launches nothing and
 * get_finish reports zeros (optimize returns 0, FullSystem.cc:727-728). Single, unsharded contexts only.
 * State rule: afterwards the device window still holds the dropped residuals and the null-space projector belongs to the old
 * evaluation point. Every entry point that computes on the window returns LDSO_B200_ERR_STATE until the next set_window, and the
 * solve entry points (optimize_begin, gn_iterations*, solve_system, do_step, gn_phase_a) also until the next set_frames --
 * the order LDSO keeps (the next keyframe's insertFrame / makeIDX come first). marginalize_points needs set_window only.
 * The getters keep working: get_frames returns the new adjoints and pair records, get_points / get_residuals the fixed linearisation. */
int ldso_b200_optimize_finish(ldso_b200_ctx *ctx);
/* Synchronises; any pointer may be NULL. res_state / res_dropped [nResiduals]; pt_relBS_max / pt_n_good [nPoints]: pt_relBS_max is 0
 * for a point without an active residual. The caller applies maxRelBaseline = max(maxRelBaseline, pt_relBS_max) and
 * numGoodResiduals += pt_n_good (host state the window does not carry), and removes the dropped residuals. newest_evalR (row-major),
 * newest_evalT, newest_state_zero: the newest frame's new evaluation point. Readable until the next set_window or set_frames
 * (LDSO_B200_ERR_STATE afterwards). */
int ldso_b200_get_finish(ldso_b200_ctx *ctx, double *energy, float *rmse, int *is_lost, uint8_t *res_state, uint8_t *res_dropped,
                         float *pt_relBS_max, int32_t *pt_n_good, double newest_evalR[9], double newest_evalT[3], double newest_state_zero[10]);
/* What get_finish returns, for the one-call form below; any pointer may be NULL. */
typedef struct ldso_b200_finish_out {
    int *iterations_run;                 /* bodies the loop ran */
    double *energy; float *rmse; int *is_lost;
    uint8_t *res_state, *res_dropped;    /* [nResiduals] */
    float *pt_relBS_max; int32_t *pt_n_good;     /* [nPoints] */
    double *newest_evalR, *newest_evalT, *newest_state_zero;     /* [9], [3], [10] */
} ldso_b200_finish_out;
/* One keyframe's FullSystem::optimize from host buffers: optimize_from_host_until followed by optimize_finish. io's outputs are
 * the loop's results exactly as optimize_from_host_until returns them; *out receives what get_finish returns. _full_submit /
 * _full_wait split it like the pairs above and keep their two-context overlap. */
int ldso_b200_optimize_from_host_full(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io, int min_iterations, const ldso_b200_finish_out *out);
int ldso_b200_optimize_from_host_full_submit(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io, int min_iterations);
int ldso_b200_optimize_from_host_full_wait(ldso_b200_ctx *ctx, const ldso_b200_fused_io *io, const ldso_b200_finish_out *out);

/* Multi-GPU (SURVEY §8e): points are sharded over ranks (one context per GPU), frames/images replicated. A GN
 * iteration is split around the ONE collective: gn_phase_a(iteration) runs [solve + frame step of `iteration`
 * (skipped when iteration < 0 = the optimize() prologue)] + resubstitute/linearize/accumulate on this rank's
 * shard and leaves the reduced system (doubles) in the buffer ldso_b200_reduce_buffer returns (device pointer);
 * the caller all-reduces (sum) that buffer over ranks on the same stream (NCCL through torch.distributed);
 * gn_phase_b() stitches the all-reduced accumulators and updates the newest frame's energy threshold. Every
 * rank then solves the 68x68 system redundantly in its next gn_phase_a. set_shard positions this rank's
 * newest-frame residual energies inside the shared select array (offset, global total) and switches the
 * context to sharded mode; call it before the first launch. */
int ldso_b200_reduce_buffer(ldso_b200_ctx *ctx, void **buf_dev, size_t *n_doubles);
int ldso_b200_set_shard(ldso_b200_ctx *ctx, int newest_slot_offset, int newest_total);
/* Device-side exchange instead of the caller's all-reduce: ONE kernel (k2r_peer_allreduce) sums the ranks' reduced buffers
 * over NVLink peer memory (CUDA IPC mappings; every rank pushes its values, tagged with the exchange number, into the peers'
 * inboxes and polls its own; fixed rank order = identical bits on every rank), so a sharded iteration is K3 -> K1 -> K2a -> K2r -> K2b on the device, captured in one CUDA graph, with no NCCL call
 * and no host round trip. Setup, once per window topology, one process per GPU on one node:
 *   set_shard(...); peer_export(handle64);  <all-gather the 64-byte handles, e.g. torch.distributed>;
 *   peer_connect(rank, world, handles);     then optimize_begin / gn_iterations exactly as on a single GPU.
 * A peer that never arrives does not hang the GPU: the wait is bounded and peer_error() then reports 1. */
int ldso_b200_peer_export(ldso_b200_ctx *ctx, void *ipc_handle_64);
int ldso_b200_peer_connect(ldso_b200_ctx *ctx, int rank, int world, const void *ipc_handles_64_each);
int ldso_b200_peer_error(ldso_b200_ctx *ctx, int *error);
int ldso_b200_gn_phase_a(ldso_b200_ctx *ctx, int iteration);
int ldso_b200_gn_phase_b(ldso_b200_ctx *ctx);

/* Per-kernel CUDA-event timing of the GN loop (bench.py's roofline leg): enable != 0 starts collecting (CUDA graphs off),
 * enable == 0 stops and returns the average duration in microseconds of K1, K2a, K2b, K3, K2r (peer exchange; 0 on a
 * single GPU) since it was enabled. */
int ldso_b200_kernel_times(ldso_b200_ctx *ctx, int enable, double out_us[5]);

/* ---- read-back (host mirrors of PointHessian / PointFrameResidual / FrameHessian fields) --------------- */
/* Optional, non-blocking: queue the device->host copy of everything get_last_solution / get_points / get_residuals
 * return (into the context's pinned staging memory) behind the work already on the stream. The next getter then
 * waits for that one copy instead of issuing and synchronising its own. The reference has no counterpart (its state is
 * host-resident); a caller that skips it gets the same values, one synchronise later. */
int ldso_b200_prefetch_results(ldso_b200_ctx *ctx);
int ldso_b200_get_energy(ldso_b200_ctx *ctx, double *energy, int *canbreak);
int ldso_b200_get_last_solution(ldso_b200_ctx *ctx, double *lastHS, double *lastbS, double *lastX);
/* any pointer may be NULL. Hcd4 is [nPoints*4]. */
int ldso_b200_get_points(ldso_b200_ctx *ctx, float *idepth, float *idepth_zero, float *step, float *HdiF,
                         float *bdSumF, float *Hdd_accAF, float *bd_accAF, float *Hcd4_accAF);
/* J74 per residual: resF[8] Jpdxi[2][6] Jpdc[2][4] Jpdd[2] JIdx[2][8] JabF[2][8] JIdx2[4] JabJIdx[4] Jab2[4]
 * (RawResidualJacobian.h:13-39); valid after linearize_all with flags bit0. */
int ldso_b200_get_residuals(ldso_b200_ctx *ctx, uint8_t *state_state, uint8_t *state_NewState, float *state_energy,
                            float *state_NewEnergy, float *state_NewEnergyWithOutlier, uint8_t *isActive,
                            float *JpJdF8, float *J74, float *projectedTo16, float *centerProjectedTo3);
/* per frame: state[10], step[10], frameEnergyTH; per pair (h + nF*t): precalc40 =
 * [RTll_0(9) tTll_0(3) RTll(9) tTll(3) KRKiTll(9) KtTll(3) aff(2) b0 distanceLL], adHost/adTarget 8x8 row-major
 * doubles, adHTdeltaF[8]; calib_value[4] (unscaled CalibHessian::value). */
int ldso_b200_get_frames(ldso_b200_ctx *ctx, double *state10, double *step10, float *frameEnergyTH, float *precalc40,
                         double *adHost64, double *adTarget64, float *adHTdeltaF8, double *calib_value4);
int ldso_b200_get_nullspace_projector(ldso_b200_ctx *ctx, double *P);

/* ---- immature points (src/internal/ImmaturePoint.cc; SURVEY.md 8f rank 2) -------------------------------
 * Candidate points whose inverse depth is still an interval [idepth_min, idepth_max]; SoA mirror of the ImmaturePoint fields
 * (include/internal/ImmaturePoint.h:103-121). status = ImmaturePointStatus (0 GOOD, 1 OOB, 2 OUTLIER, 3 SKIPPED,
 * 4 BADCONDITION, 5 UNINITIALIZED). */
typedef struct ldso_b200_immature {
    int n;
    const float *u, *v;                 /* [n] feature->uv on the host keyframe */
    const int32_t *host;                /* [n] index into the per-host KRKi/Kt/aff arrays of trace_immature */
    const float *color8, *weights8;     /* [n*8] color[], weights[] */
    const float *gradH4;                /* [n*4] gradH row-major */
    const float *energyTH;              /* [n] */
    float *idepth_min, *idepth_max;     /* [n] in/out */
    float *quality;                     /* [n] in/out */
    int32_t *lastTraceStatus;           /* [n] in/out */
    float *lastTraceUV2;                /* [n*2] out */
    float *lastTracePixelInterval;      /* [n] out */
} ldso_b200_immature;
/* ImmaturePoint::ImmaturePoint (ImmaturePoint.cc:14-38) for n candidates of the keyframe in image slot host_slot:
 * fills color8, weights8, gradH4, energyTH (NaN where a pattern pixel is not finite). */
int ldso_b200_immature_init(ldso_b200_ctx *ctx, int host_slot, int n, const float *u, const float *v, float *color8,
                            float *weights8, float *gradH4, float *energyTH);
/* One FullSystem::traceNewCoarse pass (FullSystem.cc:1012-1050): ImmaturePoint::traceOn (ImmaturePoint.cc:46-314) of every
 * candidate on the frame in image slot new_slot. KRKi9 (row-major 3x3), Kt3, aff2 per host keyframe, computed by the caller
 * exactly as FullSystem.cc:1027-1032 does. One warp per candidate. */
int ldso_b200_trace_immature(ldso_b200_ctx *ctx, int new_slot, const ldso_b200_immature *pts, int n_hosts, const float *KRKi9,
                             const float *Kt3, const float *aff2);

/* FullSystem::optimizeImmaturePoint (FullSystem.cc:892-978, with ImmaturePoint::linearizeResidual, ImmaturePoint.cc:316-383) for n
 * candidates against the device-resident window (set_frames: frame states, calibration, images; the candidates' hosts index
 * those frames): Levenberg-Marquardt on the inverse depth starting from (idepth_min + idepth_max)/2. ok[i] != 0 means the
 * reference would have created the PointHessian (finite depth, Hdd >= setting_minIdepthH_act, >= min_obs residuals IN);
 * idepth[i] is its idepth (= idepth_zero); res_state[i*nFrames + t] is the final ResState of the residual to frame t (0 IN, 1 OOB,
 * 2 OUTLIER; 255 for the host itself) - every residual left IN becomes a PointFrameResidual (:995-1008). */
int ldso_b200_optimize_immature(ldso_b200_ctx *ctx, int n, const float *u, const float *v, const int32_t *host, const float *idepth_min,
                                const float *idepth_max, const float *color8, const float *weights8, const float *energyTH, int min_obs,
                                int32_t *ok, float *idepth, uint8_t *res_state);

/* The selection loop of FullSystem::activatePointsMT (FullSystem.cc:1076-1150) with CoarseDistanceMap::makeK / makeDistanceMap /
 * addIntoDistFinal (src/frontend/CoarseTracker.cc:657-819), against the device-resident window (set_frames + set_window: the
 * window's points are the ACTIVE points that seed the distance map, projected into pyramid level 1 of frame newest_frame).
 * Candidates are visited in the order given (the reference walks the keyframes in window order and each keyframe's features in
 * index order); host[i] must not be newest_frame. current_min_act_dist = FullSystem::currentMinActDist after its update
 * (:1054-1074), min_trace_quality = setting_minTraceQuality (Setting.cc:51), frame_flagged[f] = flaggedForMarginalization.
 * action[i]: 0 = stays immature, 1 = selected (pass it to ldso_b200_optimize_immature; it is already in the distance map),
 * 2 = the reference deletes it (never traced / outlier / cannot activate and leaving / projects outside). dist_map (optional,
 * (w/2)*(h/2) floats) receives fwdWarpedIDDistFinal as the loop leaves it. Limit: (w/2)*(h/2) <= 204800 pixels (the map lives in
 * shared memory, one byte per pixel); larger images return LDSO_B200_ERR_ARG. */
int ldso_b200_select_activation(ldso_b200_ctx *ctx, int newest_frame, float current_min_act_dist, float min_trace_quality, int n,
                                const float *u, const float *v, const int32_t *host, const float *idepth_min, const float *idepth_max,
                                const int32_t *lastTraceStatus, const float *lastTracePixelInterval, const float *quality,
                                const float *my_type, const uint8_t *frame_flagged, uint8_t *action, float *dist_map);

/* EXPERIMENTAL (written at the end of round 1 against the pinned oracle, compiled, not yet run on hardware):
 * CoarseInitializer::calcResAndGS (src/frontend/CoarseInitializer.cc:181-405) for the n points of pyramid level lvl. Images: slot
 * first_slot = firstFrame, new_slot = newFrame (upload_frame / make_images). (R, t) = refToNew, tlog3 = refToNew.log().head<3>(),
 * (aff_a, aff_b) = refToNew_aff, (fx0 .. cy0) = Hcalib's level-0 intrinsics (makeK, :689-715). Per point in: Pnt::u, v, idepth_new, iR,
 * isGood, energy (2 floats), outlierTH; out: isGood_new, energy_new (2), maxstep, lastHessian_new (accepted points), JbBuffer_new
 * (10 floats; zero for points with isGood == 0). H64 / Hsc64 row-major 8x8, b8 / bsc8, res3 = the returned Vec3f. alphaK, alphaW,
 * couplingWeight as trackFrame sets them (:44-47). Points must keep the pattern radius (2 px) + 1 from the image border. */
int ldso_b200_init_calc_res(ldso_b200_ctx *ctx, int first_slot, int new_slot, int lvl, const double R[9], const double t[3], const double tlog3[3],
                            float aff_a, float aff_b, float fx0, float fy0, float cx0, float cy0, int n, const float *u, const float *v,
                            const float *idepth_new, const float *iR, const uint8_t *isGood, const float *energy2, const float *outlierTH,
                            float alphaK, float alphaW, float couplingWeight, uint8_t *isGood_new, float *energy_new2, float *maxstep,
                            float *lastHessian_new, float *JbBuffer_new10, float *H64, float *b8, float *Hsc64, float *bsc8, float *res3);

/* ---- coarse tracker (src/frontend/CoarseTracker.cc) ---------------------------------------------------- */
/* CoarseTracker::makeK (:219-246) */
int ldso_b200_tracker_make_k(ldso_b200_ctx *ctx, float fx, float fy, float cx, float cy);
/* Point cloud of the reference keyframe as makeCoarseDepthL0 leaves it (:398-437): pc_u, pc_v, pc_idepth,
 * pc_color of level lvl. */
int ldso_b200_tracker_set_ref_level(ldso_b200_ctx *ctx, int lvl, int n, const float *pc_u, const float *pc_v,
                                    const float *pc_idepth, const float *pc_color);
/* Device-side CoarseTracker::makeCoarseDepthL0 (:258-438): n contributions (centerProjectedTo[3], HdiF) of the
 * ACTIVE points whose newest residual is IN; ref_slot = image slot of lastRef. */
int ldso_b200_tracker_make_coarse_depth(ldso_b200_ctx *ctx, int ref_slot, int n, const float *centerProjectedTo3,
                                        const float *HdiF);
int ldso_b200_tracker_get_ref_level(ldso_b200_ctx *ctx, int lvl, int *n, float *pc_u, float *pc_v, float *pc_idepth,
                                    float *pc_color);
/* lastRef_aff_g2l, lastRef->ab_exposure, newFrame image slot and newFrame->ab_exposure */
int ldso_b200_tracker_set_frames(ldso_b200_ctx *ctx, float ref_aff_a, float ref_aff_b, float ref_exposure, int new_slot,
                                 float new_exposure);
/* One CoarseTracker::calcRes (:440-572) followed by calcGSSSE (:574-632) at the given pose: res6 =
 * [E, numTermsInE, flowT, 0, flowRT, satRatio]; H (8x8 row-major) and b as calcGSSSE scales them.
 * refToNew given as rotation R (row-major) and translation t. H/b may be NULL (calcRes only). */
int ldso_b200_tracker_eval(ldso_b200_ctx *ctx, int lvl, const double R[9], const double t[3], float aff_a, float aff_b,
                           float cutoffTH, double res6[6], double H[64], double b[8]);
/* CoarseTracker::trackNewestCoarse (:61-217) with the LM loop resident on the device. R,t,aff in/out.
 * Returns 1/0 (tracking good / bad) in *ok. */
int ldso_b200_tracker_track(ldso_b200_ctx *ctx, double R[9], double t[3], float *aff_a, float *aff_b, int coarsestLvl,
                            const double minResForAbort[5], double lastResiduals[5], double lastFlowIndicators[3],
                            int *ok);
/* Map::runPoseGraphOptimization (src/Map.cc:75-165; SURVEY 8f rank 4, BASELINE configs[4]): g2o Gauss-Newton over VertexSim3 /
 * EdgeSim3 (include/internal/PR.h:57-76,151-179: error = log(measurement^-1 * v1 * v2^-1), oplus: estimate = Sim3::exp(update) *
 * estimate) with g2o's numeric Jacobians (thirdparty/g2o/g2o/core/base_binary_edge.hpp:131-148, delta 1e-9), `iterations` rounds
 * (Map.cc:141: 25), vertex `fixed` held (Map.cc:109-111). Poses q4[nV][4] / t3[nV][3] (in / out): Sophus' Sim3 storage, quaternion
 * (w, x, y, z) with norm = scale + translation; edges ei / ej [nE] vertex indices, measurement mq4 / mt3, information info49[nE][49]
 * row-major. Each round's normal equations are solved by block-Jacobi preconditioned conjugate gradients to the relative residual
 * pcg_tol (at most pcg_max_iter iterations). chi2_out[iterations + 1]: sum e^T O e before every round and after the last (may be
 * NULL); *pcg_iterations_total: CG iterations spent (may be NULL). */
int ldso_b200_posegraph_optimize(ldso_b200_ctx *ctx, int nV, double *q4, double *t3, int nE, const int32_t *ei, const int32_t *ej,
                                 const double *mq4, const double *mt3, const double *info49, int fixed, int iterations,
                                 double pcg_tol, int pcg_max_iter, double *chi2_out, int *pcg_iterations_total);

/* FullSystem::trackNewCoarse's hypothesis loop (src/frontend/FullSystem.cc:290-357: constant / double / half / zero motion and
 * 26 x 3 small rotations, up to 83 calls of CoarseTracker::trackNewestCoarse per frame) as ONE launch: n <= 128 starting poses
 * (R9_each[n][9] row-major refToNew rotations, t3_each[n][3], aff2_each[n][2]), each tracked through all levels by its own CTA,
 * without abort thresholds. Per hypothesis: the refined pose / brightness, lastResiduals[5], lastFlowIndicators[3], the bool the
 * reference returns. The caller applies the reference's acceptance rule (:337-356) to the results. Output arrays other than
 * ok_each may be NULL. */
int ldso_b200_tracker_track_batch(ldso_b200_ctx *ctx, int n, const double *R9_each, const double *t3_each, const float *aff2_each, int coarsestLvl,
                                  double *R9_out, double *t3_out, float *aff2_out, double *lastResiduals5_each, double *lastFlow3_each, int *ok_each);

#ifdef __cplusplus
}
#endif
#endif /* LDSO_B200_H_ */
