// ldso_b200 C ABI implementation (include/ldso_b200.h): context, device memory, kernel launches.
// No CPU fallback anywhere: every compute entry point launches sm_90a kernels or fails.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <algorithm>
#include <cstddef>

#include "common.cuh"
#include "se3_math.cuh"
#include "host_math.h"
#include "img_kernels.cuh"
#include "ba_k1.cuh"
#include "ba_k2.cuh"
#include "ba_k3.cuh"
#include "tracker_kernels.cuh"
#include "trace_types.h"
#include "immature_store.h"
#include "posegraph.cuh"
#include "gn_loop.cuh"
#include "finish.cuh"
#include "undistort.cuh"
#include "corners.cuh"
#include "pixsel.cuh"
#include "scratch_layout.cuh"

static_assert(K1_THREADS / 32 == MAXF, "phase B maps one warp to one target frame");

#define NSLOTS (2 * MAXF)
static_assert(NSLOTS == IMM_NSEG, "one immature-point segment per image slot");

struct ldso_b200_ctx {
    int device = 0, w = 0, h = 0, levels = 0;
    int lw[MAXLVL], lh[MAXLVL];
    ldso_b200_settings S;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;
    long long launches = 0;
    int sm_count = 132;

    float4 *img[NSLOTS][MAXLVL];
    float *scratch = nullptr;          // upload staging (w*h*3 floats)
    cudaEvent_t copy_done = nullptr, frames_copied = nullptr;
    size_t scratch_floats = 0;
    // per-frame undistortion (set_undistort / undistort_frame): device tables, the raw frame buffer (wOrg*hOrg + wOrg + 1 pixels of
    // 2 bytes, zero behind the frame) and its pinned staging copy
    bool have_undistort = false;
    ldso_b200_undistort_calib ud = {};     // the pointers in it are the device copies
    float2 *ud_remap = nullptr;
    float *ud_G = nullptr, *ud_vinv = nullptr;
    void *ud_raw = nullptr, *ud_pin = nullptr;
    cudaEvent_t ud_copied = nullptr;       // the staging buffer has been read by the last frame's copy
    // keyframe corners (detect_corners), sized at creation for the most features any density can give (one per pixel): the ORB
    // pattern, B, the per-cell scratch, and the output block [n, scoreTH | u | v | score | angle | is_corner | descriptor] with its
    // pinned read-back copy
    int *orb_pattern = nullptr;
    bool have_orb_pattern = false;
    float *corner_B = nullptr;
    char *corner_mem = nullptr, *corner_pin = nullptr;
    // keyframe candidate pixels (select_pixels / make_new_traces_pixels): device block and pinned read-back block, allocated on
    // first use (pixsel_ensure); randomPattern is uploaded once, with the block
    char *pix_mem = nullptr, *pix_pin = nullptr;

    // window
    DevWindow d;
    std::vector<void *> win_allocs;
    std::vector<void *> derived_allocs;      // work items, partials, reduced buffer: rebuilt by build_derived
    bool have_window = false, have_frames = false, derived_dirty = true;
    bool select_pending = false;     // the newest frame's energy threshold of the last fused iteration has not been computed yet (flush_select)
    bool has_lin = false;            // the window holds linearized (isLinearized) residuals: solve_system accumulates HA + HL in one pass
    std::vector<unsigned char> h_scratch_bytes;     // select_activation's map read-back
    char *actsel_pin = nullptr; size_t actsel_pin_cap = 0;      // its pinned staging block
    std::vector<int> h_pt_host, h_res_begin, h_res_target;
    int nF = 0, n = 0;
    int slots[MAXF];
    WinState *ws_dev = nullptr;
    WinState *ws_host = nullptr;       // pinned staging copy
    SolveBufs sb;
    double *solve_mem = nullptr;
    double *sol_host = nullptr;      // pinned staging for get_last_solution
    // K2b(do_assemble) has produced the system K3 solves and nothing it depends on changed since
    bool solve_ready = false;
    // dimension of the device-resident marginalisation prior HM, bM (0 = all zero, any dimension): set_marg_prior,
    // marginalize_points -> n; marginalize_frame -> n - 8; set_frames keeps / grows / clears it accordingly
    int prior_dim = 0;
    // the reduced accumulators still describe the current window state (a re-stitch is enough to get solve_ready back)
    bool restitch_ok = false;
    int *iteration_dev = nullptr;
    uint8_t *pt_sel_dev = nullptr;
    char *arena_dev = nullptr, *arena_host = nullptr;
    struct Layout {
        size_t pt_host, pt_res_begin, res_point, res_target, topo_end, pt_u, pt_v, pt_color, pt_weights, pt_priorF, pt_idepth_backup,
            res_lin, res_state, dl_begin, pt_idepth, pt_idepth_zero, ul_end, pt_step, pt_HdiF, pt_bdSumF, pt_Hdd, pt_bd, pt_Hcd,
            res_new_state, res_active, res_energy, res_new_energy, res_new_energy_wo, dl_light_end, res_JpJdF, dl_end, res_JpJdF_new, total;
    } lay;
    bool mirror_valid = false;       // pinned mirror holds the current [res_state, dl_light_end) arrays
    bool mirror_full_valid = false;  // ... and the bulky [dl_light_end, dl_end) tail (JpJdF) as well
    bool sol_valid = false;          // sol_host holds the current [lastHS | lastbS | lastX]
    bool results_inflight = false;   // prefetch_results queued the read-back copies; results_ready marks their end
    cudaEvent_t results_ready = nullptr;
    std::vector<double> evalpt_key, Pns_host;
    cudaEvent_t window_copied = nullptr;
    // one GN iteration (K3 -> K1 -> K2a -> K2b) captured as a CUDA graph; re-captured when the window arena changes
    cudaGraphExec_t gn_graph = nullptr;
    bool gn_graph_valid = false;
    // the same body closed by k_gn_continue inside a conditional WHILE node (gn_iterations_until); same validity as gn_graph
    cudaGraphExec_t until_graph = nullptr;
    bool until_graph_valid = false;
    int until_form = LDSO_B200_UNTIL_HOST;    // which form the last gn_iterations_until ran (ldso_b200_get_until_form)
    int until_graph_form = LDSO_B200_UNTIL_GRAPH;     // ... and which one until_graph holds
    bool until_cond = true;          // cleared for good when the driver refuses the conditional node
    int until_launches_per_body = 0; // kernels per body of the last WHILE-node launch, not yet in `launches`
    int *loop_dev = nullptr;         // k_gn_continue's parameters and counters (LOOP_*)
    int *loop_pin = nullptr;         // pinned: the host-driven form reads LOOP_CONT back here
    // optimize_finish: per-point / per-residual outputs (window arrays) and the two scalars; fin_state 0 = nothing to read,
    // 1 = the last finish had fewer than 2 frames (nothing ran, get_finish reports zeros), 2 = results on the device
    FinishBufs fb = {};
    int fin_state = 0;
    // after optimize_finish the window still holds the dropped residuals and the null-space projector is stale: the window
    // entry points wait for the next set_window, the solve entry points also for the next set_frames
    bool fin_window_stale = false, fin_frames_stale = false;
    bool use_graph = true;
    bool use_pdl = true;             // programmatic dependent launch inside the GN iteration (env LDSO_B200_NO_PDL disables)
    bool pdl_now = false;            // set while launch_gn_body issues its four kernels
    size_t k1_smem = 0;
    char *trace_buf = nullptr;       // device scratch of the one-shot entry points (trace_carve)
    size_t trace_cap = 0;
    // immature-point store (immature_store.h): the segments (imm_cap entries each), activate_immature's scratch and the pinned
    // read-back block, allocated together on first use; per slot the entries seeded and how many of them are still live
    float *imm_store = nullptr;
    char *imm_scratch = nullptr, *imm_pin = nullptr;
    int imm_cap = 0;
    int imm_n[NSLOTS] = {}, imm_live[NSLOTS] = {};
    bool multi = false;
    // peer-memory exchange (k2r_peer_allreduce): this rank's exported inbox, the peers' mapped inboxes, and the local
    // epoch / completion / error words
    char *peer_local = nullptr;
    void *peer_opened[K2R_MAX_PEERS] = {};
    int *peer_words = nullptr;       // [0] epoch, [1] done, [2] error
    double *red_sum = nullptr;
    PeerExchange px;
    bool peers_connected = false;

    // tracker
    TrkLevel trk[MAXLVL];
    float *trk_pc[MAXLVL][4];
    int trk_cap[MAXLVL];
    float trk_fx[MAXLVL], trk_fy[MAXLVL], trk_cx[MAXLVL], trk_cy[MAXLVL];
    float trk_Ki[MAXLVL][9];
    float ref_aff_a = 0, ref_aff_b = 0, ref_exposure = 1, new_exposure = 1;
    int new_slot = -1;
    float *cd_id[MAXLVL] = {}, *cd_ws[MAXLVL] = {}, *cd_bak[MAXLVL] = {};
    int *cd_pos[MAXLVL] = {};
    int *cd_rows = nullptr, *cd_tot = nullptr;
    float *cd_in = nullptr;
    int cd_in_cap = 0;
    float *trk_partials = nullptr;
    unsigned *trk_counter = nullptr;
    double *trk_out_dev = nullptr;
    TrkTrackOut *trk_track_out = nullptr;

    // optional per-kernel CUDA-event timing of the GN loop (env LDSO_B200_KTIME=1), printed at destroy
    bool ktime = false;
    struct KT { const char *name; cudaEvent_t a, b; };
    std::vector<KT> kt;
    void kt_begin(const char *name) {
        if (!ktime) return;
        KT k; k.name = name;
        cudaEventCreate(&k.a); cudaEventCreate(&k.b);
        cudaEventRecord(k.a, stream);
        kt.push_back(k);
    }
    void kt_end() { if (ktime) cudaEventRecord(kt.back().b, stream); }
    void kt_report() {
        if (!ktime || kt.empty()) return;
        cudaStreamSynchronize(stream);
        std::vector<std::string> names; std::vector<double> tot; std::vector<int> cnt;
        for (auto &k : kt) {
            float ms = 0; cudaEventElapsedTime(&ms, k.a, k.b);
            size_t i = 0;
            for (; i < names.size(); i++) if (names[i] == k.name) break;
            if (i == names.size()) { names.push_back(k.name); tot.push_back(0); cnt.push_back(0); }
            tot[i] += ms; cnt[i]++;
            cudaEventDestroy(k.a); cudaEventDestroy(k.b);
        }
        for (size_t i = 0; i < names.size(); i++)
            fprintf(stderr, "[ldso_b200 ktime] %-12s n=%6d avg=%8.2f us\n", names[i].c_str(), cnt[i], 1e3 * tot[i] / cnt[i]);
        kt.clear();
    }

    int fail(int code, const char *msg) { err = msg; return code; }
    int fail_cuda(cudaError_t e, const char *call, const char *file, int line) {
        char buf[512];
        snprintf(buf, sizeof(buf), "CUDA error %s (%s) at %s:%d in %s", cudaGetErrorName(e), cudaGetErrorString(e), file, line, call);
        err = buf;
        return LDSO_B200_ERR_CUDA;
    }
};

extern "C" void ldso_b200_default_settings(ldso_b200_settings *s) {
    s->huberTH = 9;
    s->outlierTHSumComponent = 50 * 50;
    s->affineOptModeA = 1e12f;
    s->affineOptModeB = 1e8f;
    s->idepthFixPrior = 50 * 50;
    s->initialTransPrior = 1e10f;
    s->initialRotPrior = 1e11f;
    s->initialAffAPrior = 1e14f;
    s->initialAffBPrior = 1e14f;
    s->initialCalibHessian = 5e9f;
    s->frameEnergyTHN = 0.7f;
    s->frameEnergyTHFacMedian = 1.5f;
    s->frameEnergyTHConstWeight = 0.5f;
    s->overallEnergyTHWeight = 1;
    s->coarseCutoffTH = 20;
    s->thOptIterations = 1.2f;
    s->solverModeDelta = 0.00001;
    s->margWeightFac = 0.5f * 0.5f;
    s->maxPixSearch = 0.027f;
    s->outlierTH = 12 * 12;
    s->trace_stepsize = 1.0f;
    s->trace_GNThreshold = 0.1f;
    s->trace_extraSlackOnTH = 1.2f;
    s->trace_slackInterval = 1.5f;
    s->trace_minImprovementFactor = 2;
    s->minTraceTestRadius = 2;
    s->trace_GNIterations = 3;
}

extern "C" ldso_b200_ctx *ldso_b200_create(int device, int w, int h, int pyr_levels, const ldso_b200_settings *settings) {
    if (w <= 0 || h <= 0 || pyr_levels < 1 || pyr_levels > MAXLVL) return nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0 || device >= ndev) {
        fprintf(stderr, "ldso_b200: no CUDA device available (there is no CPU fallback)\n");
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) return nullptr;
    ldso_b200_ctx *c = new ldso_b200_ctx();
    c->device = device; c->w = w; c->h = h; c->levels = pyr_levels;
    if (settings) c->S = *settings; else ldso_b200_default_settings(&c->S);
    for (int l = 0; l < MAXLVL; l++) { c->lw[l] = w >> l; c->lh[l] = h >> l; }
    memset(c->img, 0, sizeof(c->img));
    memset(&c->d, 0, sizeof(c->d));
    memset(&c->sb, 0, sizeof(c->sb));
    memset(c->trk, 0, sizeof(c->trk));
    memset(c->trk_pc, 0, sizeof(c->trk_pc));
    memset(c->trk_cap, 0, sizeof(c->trk_cap));
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) c->sm_count = prop.multiProcessorCount;
    bool ok = true;
    ok = ok && cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) == cudaSuccess;
    c->own_stream = true;
    ok = ok && cudaMalloc(&c->ws_dev, sizeof(WinState)) == cudaSuccess;
    ok = ok && cudaMallocHost(&c->ws_host, sizeof(WinState)) == cudaSuccess;
    ok = ok && cudaMalloc(&c->iteration_dev, sizeof(int)) == cudaSuccess;
    ok = ok && cudaMalloc(&c->loop_dev, sizeof(int) * LOOP_WORDS) == cudaSuccess;
    ok = ok && cudaMallocHost(&c->loop_pin, sizeof(int) * LOOP_WORDS) == cudaSuccess;
    ok = ok && cudaMalloc(&c->fb.rmse, sizeof(float) + sizeof(int)) == cudaSuccess;
    // solve buffers: 4 + 1 + 1 + 1 matrices (n x n) and 6 vectors
    const size_t nn = (size_t) MAXN * MAXN;
    ok = ok && cudaMalloc(&c->solve_mem, sizeof(double) * (7 * nn + 8 * MAXN)) == cudaSuccess;
    ok = ok && cudaMalloc(&c->trk_partials, sizeof(float) * 1024 * TRK_NACC) == cudaSuccess;
    ok = ok && cudaMalloc(&c->trk_counter, sizeof(unsigned)) == cudaSuccess;
    ok = ok && cudaMalloc(&c->trk_out_dev, sizeof(double) * 80) == cudaSuccess;
    ok = ok && cudaMalloc(&c->trk_track_out, sizeof(TrkTrackOut)) == cudaSuccess;
    if (!ok) { fprintf(stderr, "ldso_b200: context allocation failed: %s\n", cudaGetErrorString(cudaGetLastError())); delete c; return nullptr; }
    cudaMemset(c->solve_mem, 0, sizeof(double) * (7 * nn + 8 * MAXN));
    cudaMemset(c->trk_counter, 0, sizeof(unsigned));
    cudaMemset(c->iteration_dev, 0, sizeof(int));
    cudaMemset(c->loop_dev, 0, sizeof(int) * LOOP_WORDS);
    c->fb.is_lost = (int *) (c->fb.rmse + 1);
    cudaMemset(c->ws_dev, 0, sizeof(WinState));
    memset(c->ws_host, 0, sizeof(WinState));
    double *p = c->solve_mem;
    c->sb.H_A = p; p += nn; c->sb.H_sc = p; p += nn; c->sb.HM = p; p += nn; c->sb.Pns = p; p += nn;
    c->sb.A0g = p; p += nn; c->sb.HSg = p; p += nn;     // assembled system handed from K2b to K3
    // lastHS | lastbS | lastX are contiguous: get_last_solution reads them back with one copy
    c->sb.lastHS = p; p += nn; c->sb.lastbS = p; p += MAXN; c->sb.lastX = p; p += MAXN;
    c->sb.b_A = p; p += MAXN; c->sb.b_sc = p; p += MAXN; c->sb.bM = p; p += MAXN;
    c->sb.dg = p; p += MAXN; c->sb.bFg = p; p += MAXN;
    ok = cudaMallocHost(&c->sol_host, sizeof(double) * (nn + 3 * MAXN)) == cudaSuccess;      // [lastHS | lastbS | lastX | scalars]
    if (!ok) { fprintf(stderr, "ldso_b200: pinned allocation failed\n"); delete c; return nullptr; }
    {
        const size_t px = (size_t) w * h;
        CornerArgs a;
        Arena S;
        corner_regions(S, px, 0, a);
        ok = cudaMalloc(&c->corner_mem, S.off) == cudaSuccess && cudaMallocHost(&c->corner_pin, corner_out_bytes(px)) == cudaSuccess;
        if (!ok) { fprintf(stderr, "ldso_b200: corner scratch allocation failed\n"); delete c; return nullptr; }
        Arena D(c->corner_mem);
        const CornerFixed f = corner_regions(D, px, 0, a);
        c->orb_pattern = f.pattern;
        c->corner_B = f.B;
    }
    c->ktime = getenv("LDSO_B200_KTIME") != nullptr;
    c->use_graph = !c->ktime && getenv("LDSO_B200_NO_GRAPH") == nullptr;
    c->use_pdl = getenv("LDSO_B200_NO_PDL") == nullptr;
    cudaEventCreateWithFlags(&c->frames_copied, cudaEventDisableTiming);
    cudaFuncSetAttribute(k1_linearize_accumulate, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) k1_smem_bytes(64));
    cudaFuncSetAttribute(k3_solve_step, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) K3_SMEM_BYTES);
    cudaFuncSetAttribute(k2b_stitch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) K2B_SMEM_BYTES);
    return c;
}

static void free_undistort(ldso_b200_ctx *c) {
    if (c->ud_remap) cudaFree(c->ud_remap);
    if (c->ud_G) cudaFree(c->ud_G);
    if (c->ud_vinv) cudaFree(c->ud_vinv);
    if (c->ud_raw) cudaFree(c->ud_raw);
    if (c->ud_pin) cudaFreeHost(c->ud_pin);
    if (c->ud_copied) cudaEventDestroy(c->ud_copied);
    c->ud_remap = nullptr; c->ud_G = c->ud_vinv = nullptr; c->ud_raw = c->ud_pin = nullptr; c->ud_copied = nullptr;
    c->have_undistort = false;
}

static void free_derived(ldso_b200_ctx *c) {
    for (void *p : c->derived_allocs) cudaFree(p);
    c->derived_allocs.clear();
    c->d.items = nullptr; c->d.host_item_begin = nullptr; c->d.res_newest_slot = nullptr;
    c->d.partials = nullptr; c->d.item_stats = nullptr; c->d.red = nullptr; c->d.dbg = nullptr;
}

static void free_window(ldso_b200_ctx *c) {
    for (void *p : c->win_allocs) cudaFree(p);
    c->win_allocs.clear();
    free_derived(c);
    if (c->arena_dev) { cudaFree(c->arena_dev); c->arena_dev = nullptr; }
    if (c->arena_host) { cudaFreeHost(c->arena_host); c->arena_host = nullptr; }
    { c->mirror_valid = false; c->results_inflight = false; c->sol_valid = false; c->mirror_full_valid = false; }
    c->gn_graph_valid = false; c->until_graph_valid = false;
    c->have_window = false;
}

extern "C" void ldso_b200_destroy(ldso_b200_ctx *c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    c->kt_report();
    if (c->gn_graph) cudaGraphExecDestroy(c->gn_graph);
    if (c->until_graph) cudaGraphExecDestroy(c->until_graph);
    free_window(c);
    for (int s = 0; s < NSLOTS; s++) for (int l = 0; l < MAXLVL; l++) if (c->img[s][l]) cudaFree(c->img[s][l]);
    for (int l = 0; l < MAXLVL; l++) for (int k = 0; k < 4; k++) if (c->trk_pc[l][k]) cudaFree(c->trk_pc[l][k]);
    for (int l = 0; l < MAXLVL; l++) { if (c->cd_id[l]) cudaFree(c->cd_id[l]); if (c->cd_ws[l]) cudaFree(c->cd_ws[l]); if (c->cd_bak[l]) cudaFree(c->cd_bak[l]); if (c->cd_pos[l]) cudaFree(c->cd_pos[l]); }
    if (c->cd_rows) cudaFree(c->cd_rows);
    if (c->cd_tot) cudaFree(c->cd_tot);
    if (c->cd_in) cudaFree(c->cd_in);
    if (c->scratch) cudaFree(c->scratch);
    free_undistort(c);
    if (c->corner_mem) cudaFree(c->corner_mem);
    if (c->corner_pin) cudaFreeHost(c->corner_pin);
    if (c->pix_mem) cudaFree(c->pix_mem);
    if (c->pix_pin) cudaFreeHost(c->pix_pin);
    if (c->ws_dev) cudaFree(c->ws_dev);
    if (c->ws_host) cudaFreeHost(c->ws_host);
    if (c->sol_host) cudaFreeHost(c->sol_host);
    if (c->actsel_pin) cudaFreeHost(c->actsel_pin);
    if (c->trace_buf) cudaFree(c->trace_buf);
    if (c->imm_store) cudaFree(c->imm_store);
    if (c->imm_scratch) cudaFree(c->imm_scratch);
    if (c->imm_pin) cudaFreeHost(c->imm_pin);
    for (int r = 0; r < K2R_MAX_PEERS; r++) if (c->peer_opened[r]) cudaIpcCloseMemHandle(c->peer_opened[r]);
    if (c->peer_local) cudaFree(c->peer_local);
    if (c->peer_words) cudaFree(c->peer_words);
    if (c->red_sum) cudaFree(c->red_sum);
    if (c->iteration_dev) cudaFree(c->iteration_dev);
    if (c->loop_dev) cudaFree(c->loop_dev);
    if (c->loop_pin) cudaFreeHost(c->loop_pin);
    if (c->fb.rmse) cudaFree(c->fb.rmse);
    if (c->solve_mem) cudaFree(c->solve_mem);
    if (c->trk_partials) cudaFree(c->trk_partials);
    if (c->trk_counter) cudaFree(c->trk_counter);
    if (c->trk_out_dev) cudaFree(c->trk_out_dev);
    if (c->trk_track_out) cudaFree(c->trk_track_out);
    if (c->own_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" const char *ldso_b200_last_error(const ldso_b200_ctx *c) { return c ? c->err.c_str() : "null context"; }
extern "C" long long ldso_b200_launch_count(const ldso_b200_ctx *c) { return c ? c->launches : 0; }

extern "C" int ldso_b200_set_stream(ldso_b200_ctx *c, void *cuda_stream) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    if (c->own_stream && c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
    c->stream = (cudaStream_t) cuda_stream;
    c->own_stream = false;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_synchronize(ldso_b200_ctx *c) {
    if (!c) return LDSO_B200_ERR_ARG;
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

#define LAUNCH_CHECK(c)                                            \
    do {                                                           \
        (c)->launches++;                                           \
        (c)->mirror_valid = false; (c)->results_inflight = false; (c)->sol_valid = false; (c)->mirror_full_valid = false;                                 \
        cudaError_t e__ = cudaGetLastError();                      \
        if (e__ != cudaSuccess) return (c)->fail_cuda(e__, "kernel launch", __FILE__, __LINE__); \
    } while (0)

#define RET_IF(x) do { int rc__ = (x); if (rc__) return rc__; } while (0)
#define D2H(dst, src, bytes) do { if (dst) CUDA_CHECK_RET(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream)); } while (0)
// dst may be a const member of a kernel's argument struct: the host fills what the kernel only reads
#define H2D(dst, src, bytes) CUDA_CHECK_RET(c, cudaMemcpyAsync((void *) (dst), src, bytes, cudaMemcpyHostToDevice, c->stream))

static int wait_results(ldso_b200_ctx *c);

// ---------------------------------------------------------------------------------------------- images
static int ensure_slot(ldso_b200_ctx *c, int slot) {
    if (slot < 0 || slot >= NSLOTS) return c->fail(LDSO_B200_ERR_ARG, "image slot out of range");
    for (int l = 0; l < c->levels; l++)
        if (!c->img[slot][l]) CUDA_CHECK_RET(c, cudaMalloc(&c->img[slot][l], sizeof(float4) * (size_t) c->lw[l] * c->lh[l]));
    if (!c->scratch) {
        c->scratch_floats = (size_t) c->w * c->h * 3;
        CUDA_CHECK_RET(c, cudaMalloc(&c->scratch, sizeof(float) * c->scratch_floats));
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_upload_frame(ldso_b200_ctx *c, int slot, const float *const *dIp, int n_levels) {
    if (!c || !dIp) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    if (n_levels != c->levels) return c->fail(LDSO_B200_ERR_ARG, "n_levels != pyr_levels of the context");
    int rc = ensure_slot(c, slot);
    if (rc) return rc;
    for (int l = 0; l < c->levels; l++) {
        const int npx = c->lw[l] * c->lh[l];
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->scratch, dIp[l], sizeof(float) * 3 * npx, cudaMemcpyHostToDevice, c->stream));
        k_repack_aos3<<<(npx + 255) / 256, 256, 0, c->stream>>>(c->scratch, c->img[slot][l], npx);
        LAUNCH_CHECK(c);
        // the staging buffer is reused by the next level: the copies are stream-ordered, but the host buffer
        // of a pageable cudaMemcpyAsync is consumed before the call returns, so this is safe.
    }
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

// FrameHessian::makeImages on the device from the w*h irradiance image in c->scratch into slot's pyramid (ensure_slot done)
static int pyramid_from_scratch(ldso_b200_ctx *c, int slot) {
    for (int l = 0; l < c->levels; l++) {
        const int npx = c->lw[l] * c->lh[l];
        k_pyr_level<<<(npx + 255) / 256, 256, 0, c->stream>>>(c->scratch, l == 0 ? nullptr : c->img[slot][l - 1], c->img[slot][l],
                                                                c->lw[l], c->lh[l], l == 0 ? 0 : c->lw[l - 1]);
        LAUNCH_CHECK(c);
    }
    return LDSO_B200_OK;
}

static int make_images_impl(ldso_b200_ctx *c, int slot, const float *color, bool wait_copy) {
    if (!c || !color) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    int rc = ensure_slot(c, slot);
    if (rc) return rc;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->scratch, color, sizeof(float) * c->w * c->h, cudaMemcpyHostToDevice, c->stream));
    if (!c->copy_done) CUDA_CHECK_RET(c, cudaEventCreateWithFlags(&c->copy_done, cudaEventDisableTiming));
    CUDA_CHECK_RET(c, cudaEventRecord(c->copy_done, c->stream));
    RET_IF(pyramid_from_scratch(c, slot));
    // the caller's buffer is free once the copy has landed; the pyramid kernels keep running asynchronously
    if (wait_copy) CUDA_CHECK_RET(c, cudaEventSynchronize(c->copy_done));
    return LDSO_B200_OK;
}
extern "C" int ldso_b200_make_images(ldso_b200_ctx *c, int slot, const float *color) { return make_images_impl(c, slot, color, true); }

// ---------------------------------------------------------------------------------------------- undistortion (undistort.cuh)
extern "C" int ldso_b200_set_undistort(ldso_b200_ctx *c, const ldso_b200_undistort_calib *u) {
    if (!c || !u) return LDSO_B200_ERR_ARG;
    if (u->wOrg <= 0 || u->hOrg <= 0) return c->fail(LDSO_B200_ERR_ARG, "set_undistort: wOrg and hOrg must be positive");
    if ((long long) u->wOrg * u->hOrg + u->wOrg + 1 > (1LL << 30)) return c->fail(LDSO_B200_ERR_ARG, "set_undistort: raw frame too large");
    if (u->w != c->w || u->h != c->h) return c->fail(LDSO_B200_ERR_ARG, "set_undistort: the rectified size must be the context's w x h");
    if ((u->remapX == nullptr) != (u->remapY == nullptr)) return c->fail(LDSO_B200_ERR_ARG, "set_undistort: remapX and remapY go together");
    if (!u->remapX && (u->wOrg != c->w || u->hOrg != c->h))
        return c->fail(LDSO_B200_ERR_ARG, "set_undistort: passthrough (no remap) needs wOrg x hOrg == the context's w x h");
    if (u->photometric_mode < 0 || u->photometric_mode > 2) return c->fail(LDSO_B200_ERR_ARG, "set_undistort: photometric_mode must be 0, 1 or 2");
    if (u->G && u->g_entries != 256 && u->g_entries != 65536) return c->fail(LDSO_B200_ERR_ARG, "set_undistort: g_entries must be 256 or 65536");
    if (u->G && u->photometric_mode == 2 && !u->vignetteMapInv)
        return c->fail(LDSO_B200_ERR_ARG, "set_undistort: photometric_mode 2 with a valid G needs vignetteMapInv");
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    free_undistort(c);
    const size_t nOrg = (size_t) u->wOrg * u->hOrg, n = (size_t) c->w * c->h;
    CUDA_CHECK_RET(c, cudaMalloc(&c->ud_raw, 2 * (nOrg + u->wOrg + 1)));
    CUDA_CHECK_RET(c, cudaMemset(c->ud_raw, 0, 2 * (nOrg + u->wOrg + 1)));     // the zero pixels behind the frame stay zero
    CUDA_CHECK_RET(c, cudaMallocHost(&c->ud_pin, 2 * nOrg));
    CUDA_CHECK_RET(c, cudaEventCreateWithFlags(&c->ud_copied, cudaEventDisableTiming));
    if (u->remapX) {
        std::vector<float2> rm(n);
        for (size_t i = 0; i < n; i++) rm[i] = make_float2(u->remapX[i], u->remapY[i]);
        CUDA_CHECK_RET(c, cudaMalloc(&c->ud_remap, sizeof(float2) * n));
        CUDA_CHECK_RET(c, cudaMemcpy(c->ud_remap, rm.data(), sizeof(float2) * n, cudaMemcpyHostToDevice));
    }
    if (u->G) {
        CUDA_CHECK_RET(c, cudaMalloc(&c->ud_G, sizeof(float) * u->g_entries));
        CUDA_CHECK_RET(c, cudaMemcpy(c->ud_G, u->G, sizeof(float) * u->g_entries, cudaMemcpyHostToDevice));
    }
    if (u->vignetteMapInv) {
        CUDA_CHECK_RET(c, cudaMalloc(&c->ud_vinv, sizeof(float) * nOrg));
        CUDA_CHECK_RET(c, cudaMemcpy(c->ud_vinv, u->vignetteMapInv, sizeof(float) * nOrg, cudaMemcpyHostToDevice));
    }
    c->ud = *u;
    c->ud.remapX = c->ud.remapY = nullptr;
    c->ud.G = c->ud_G;
    c->ud.vignetteMapInv = c->ud_vinv;
    c->have_undistort = true;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_undistort_frame(ldso_b200_ctx *c, int slot, const void *raw, int bytes_per_pixel, float exposure, float factor,
                                         float *exposure_time_out) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (!c->have_undistort) return c->fail(LDSO_B200_ERR_STATE, "undistort_frame: call set_undistort first");
    if (!raw) return c->fail(LDSO_B200_ERR_ARG, "undistort_frame: raw is NULL");
    if (bytes_per_pixel != 1 && bytes_per_pixel != 2) return c->fail(LDSO_B200_ERR_ARG, "undistort_frame: bytes_per_pixel must be 1 or 2");
    if (bytes_per_pixel == 2 && c->ud.G && c->ud.g_entries < 65536)
        return c->fail(LDSO_B200_ERR_ARG, "undistort_frame: a 16-bit frame needs a 65536-entry G");
    cudaSetDevice(c->device);
    RET_IF(ensure_slot(c, slot));
    const size_t bytes = (size_t) bytes_per_pixel * c->ud.wOrg * c->ud.hOrg;
    // the staging buffer is free once the previous frame's copy has read it
    CUDA_CHECK_RET(c, cudaEventSynchronize(c->ud_copied));
    memcpy(c->ud_pin, raw, bytes);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->ud_raw, c->ud_pin, bytes, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(c, cudaEventRecord(c->ud_copied, c->stream));
    UndistortArgs a;
    a.remap = c->ud_remap; a.G = c->ud_G; a.vinv = c->ud_vinv;
    a.wOrg = c->ud.wOrg; a.hOrg = c->ud.hOrg; a.w = c->w; a.h = c->h;
    a.use_G = c->ud_G != nullptr && !(exposure <= 0) && c->ud.photometric_mode != 0;      // processFrame's branch (Undistort.cc:197)
    a.mode2 = c->ud.photometric_mode == 2;
    a.factor = factor;
    const int npx = c->w * c->h;
    if (bytes_per_pixel == 1) k_undistort<uint8_t><<<(npx + 255) / 256, 256, 0, c->stream>>>((const uint8_t *) c->ud_raw, a, c->scratch);
    else k_undistort<uint16_t><<<(npx + 255) / 256, 256, 0, c->stream>>>((const uint16_t *) c->ud_raw, a, c->scratch);
    LAUNCH_CHECK(c);
    RET_IF(pyramid_from_scratch(c, slot));
    if (exposure_time_out) *exposure_time_out = c->ud.use_exposure ? exposure : 1.f;
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- keyframe corners (corners.cuh)
namespace {
struct CornerGrid { int gs, gridX, gridY, skip, ncx, ncy, kcap; float nfeatInGrid; };
}
// DetectCorners' grid (FeatureDetector.cc:37-42); false for nFeatures <= 0, gridsize 0, or a grid whose angle / descriptor footprints
// (+-15 pixels around every pixel of a processed cell: IC_Angle's circle; the descriptor's rotated pattern reaches at most 13) can
// leave the image, where the reference reads outside its buffer
static bool corner_grid(int w, int h, int nFeatures, CornerGrid &g) {
    if (w <= 0 || h <= 0 || nFeatures <= 0) return false;
    g.gs = int(sqrtf((float) (w * h / nFeatures)) + 0.5);
    if (g.gs <= 0) return false;
    g.gridX = w / g.gs + 1;
    g.gridY = h / g.gs + 1;
    g.nfeatInGrid = float(nFeatures) / (w * h) * (g.gs * g.gs);
    g.skip = CORNER_HALF_PATCH * 2 / g.gs + 1;
    g.ncx = std::max(0, g.gridX - 2 * g.skip);
    g.ncy = std::max(0, g.gridY - 2 * g.skip);
    int k = 0;                        // the reference stops after the pick that makes `picked > nfeatInGrid`
    while (!((float) k > g.nfeatInGrid)) k++;
    g.kcap = std::min(k, g.gs * g.gs);
    if (g.ncx > 0 && g.ncy > 0) {
        const int x0 = g.skip * g.gs, x1 = (g.gridX - g.skip) * g.gs - 1, y0 = g.skip * g.gs, y1 = (g.gridY - g.skip) * g.gs - 1;
        if (x0 - CORNER_HALF_PATCH < 0 || x1 + CORNER_HALF_PATCH > w - 1 || y0 - CORNER_HALF_PATCH < 0 || y1 + CORNER_HALF_PATCH > h - 1)
            return false;
    }
    return true;
}

extern "C" int ldso_b200_feature_capacity(int w, int h, int nFeatures) {
    CornerGrid g;
    if (!corner_grid(w, h, nFeatures, g)) return LDSO_B200_ERR_ARG;
    return g.ncx * g.ncy * g.kcap;
}

extern "C" int ldso_b200_set_orb_pattern(ldso_b200_ctx *c, const int32_t *pattern) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (!pattern) return c->fail(LDSO_B200_ERR_ARG, "set_orb_pattern: pattern is NULL");
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    CUDA_CHECK_RET(c, cudaMemcpy(c->orb_pattern, pattern, sizeof(int32_t) * 1024, cudaMemcpyHostToDevice));
    c->have_orb_pattern = true;
    return LDSO_B200_OK;
}

// detect_corners' checks and launches on the context's stream; corners_read brings the output block back into *out. Between the two
// the features are on the device: a.hdr[0] = n, a.u / a.v = their coordinates.
static int corners_launch(ldso_b200_ctx *c, int slot, int nFeatures, const float *B, const ldso_b200_features *out, CornerArgs &a) {
    if (!c->have_orb_pattern) return c->fail(LDSO_B200_ERR_STATE, "detect_corners: call set_orb_pattern first");
    if (slot < 0 || slot >= NSLOTS || !c->img[slot][0]) return c->fail(LDSO_B200_ERR_ARG, "detect_corners: image slot out of range or never filled");
    if (!out || !out->u || !out->v || !out->score || !out->is_corner || !out->angle || !out->descriptor)
        return c->fail(LDSO_B200_ERR_ARG, "detect_corners: missing output array");
    CornerGrid g;
    if (!corner_grid(c->w, c->h, nFeatures, g))
        return c->fail(LDSO_B200_ERR_ARG, "detect_corners: nFeatures must be positive and give a grid whose patches stay inside the image");
    const int cap = g.ncx * g.ncy * g.kcap;
    if (out->capacity < cap) return c->fail(LDSO_B200_ERR_ARG, "detect_corners: capacity below ldso_b200_feature_capacity(w, h, nFeatures)");
    cudaSetDevice(c->device);
    Arena D(c->corner_mem);
    corner_regions(D, (size_t) c->w * c->h, cap, a);
    a.img = c->img[slot][0];
    a.B = nullptr;
    if (B) {
        H2D(c->corner_B, B, sizeof(float) * 256);
        a.B = c->corner_B;
    }
    a.pattern = c->orb_pattern;
    a.w = c->w; a.h = c->h;
    a.gs = g.gs; a.skip = g.skip; a.ncx = g.ncx; a.ncy = g.ncy; a.kcap = g.kcap; a.nfeatInGrid = g.nfeatInGrid;
    {   // FeatureDetector's constructor (:10-28): umax with cvFloor / cvCeil / cvRound (round half to even)
        int v, v0, vmax = (int) floor(CORNER_HALF_PATCH * sqrtf(2.f) / 2 + 1), vmin = (int) ceil(CORNER_HALF_PATCH * sqrtf(2.f) / 2);
        const double hp2 = CORNER_HALF_PATCH * CORNER_HALF_PATCH;
        for (v = 0; v <= vmax; ++v) a.umax[v] = (int) lrint(sqrt(hp2 - v * v));
        for (v = CORNER_HALF_PATCH, v0 = 0; v >= vmin; --v) {
            while (a.umax[v0] == a.umax[v0 + 1]) ++v0;
            a.umax[v] = v0;
            ++v0;
        }
    }
    const int ncell = g.ncx * g.ncy;
    if (ncell == 0) {
        CUDA_CHECK_RET(c, cudaMemsetAsync(a.hdr, 0, 16, c->stream));
    } else {
        k_corner_cells<<<ncell, CORNER_THREADS, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        k_corner_scan<<<1, 1024, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        const int npick = ncell * g.kcap;
        k_corner_emit<<<(npick + 255) / 256, 256, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        k_corner_describe<<<(npick + 127) / 128, 128, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
    }
    return LDSO_B200_OK;
}

static int corners_read(ldso_b200_ctx *c, const CornerArgs &a, ldso_b200_features *out) {
    CornerArgs h;      // the output block's split, at the pinned copy
    corner_split(c->corner_pin, a.cap, h);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(h.hdr, a.hdr, corner_out_bytes(a.cap), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    const int n = h.hdr[0];
    memcpy(out->u, h.u, sizeof(float) * n);
    memcpy(out->v, h.v, sizeof(float) * n);
    memcpy(out->score, h.score, sizeof(float) * n);
    memcpy(out->angle, h.angle, sizeof(float) * n);
    memcpy(out->is_corner, h.is_corner, n);
    memcpy(out->descriptor, h.desc, (size_t) 32 * n);
    int nc = 0;
    for (int i = 0; i < n; i++) nc += h.is_corner[i] != 0;
    out->n = n;
    out->n_corners = nc;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_detect_corners(ldso_b200_ctx *c, int slot, int nFeatures, const float *B, ldso_b200_features *out) {
    if (!c) return LDSO_B200_ERR_ARG;
    CornerArgs a;
    RET_IF(corners_launch(c, slot, nFeatures, B, out, a));
    return corners_read(c, a, out);
}

// ---------------------------------------------------------------------------------------------- keyframe candidate pixels (pixsel.cuh)
// PixelSelector's randomPattern (PixelSelector2.cc:11-13): rand() & 0xFF after srand(3141592). glibc's rand() is random() on a
// TYPE_3 state of 128 bytes; initstate_r seeds a private state of that type exactly as srand seeds the global one, so the caller's
// rand() sequence is left alone.
static void pixsel_pattern(uint8_t *out, size_t n) {
    struct random_data rd;
    memset(&rd, 0, sizeof(rd));
    char state[128];
    initstate_r(3141592, state, sizeof(state), &rd);
    for (size_t i = 0; i < n; i++) {
        int32_t r;
        random_r(&rd, &r);
        out[i] = (uint8_t) (r & 0xFF);
    }
}

extern "C" int ldso_b200_pixsel_pattern(int n, uint8_t *out) {
    if (n < 0 || (n > 0 && !out)) return LDSO_B200_ERR_ARG;
    pixsel_pattern(out, (size_t) n);
    return LDSO_B200_OK;
}

// the device block (pixsel_regions) and the pinned block (pixsel_pin_regions), allocated on first use; randomPattern is uploaded once
static int pixsel_ensure(ldso_b200_ctx *c) {
    if (c->pix_mem) return LDSO_B200_OK;
    const size_t px = (size_t) c->w * c->h;
    PixselArgs a;
    Arena S, P, Q;
    pixsel_regions(S, c->w, c->h, true, a);
    pixsel_pin_regions(P, px, px, true, a);
    pixsel_pin_regions(Q, px, px, false, a);
    char *m = nullptr, *pin = nullptr;
    cudaError_t e = cudaMalloc(&m, S.off);
    if (e == cudaSuccess) e = cudaMallocHost(&pin, std::max(P.off, Q.off));
    if (e == cudaSuccess) {
        Arena D(m);
        const PixselFixed f = pixsel_regions(D, c->w, c->h, true, a);
        pixsel_pattern((uint8_t *) pin, px);
        e = cudaMemcpy(f.rp, pin, px, cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) {
        if (m) cudaFree(m);
        if (pin) cudaFreeHost(pin);
        return c->fail_cuda(e, "pixel selection scratch", __FILE__, __LINE__);
    }
    c->pix_mem = m; c->pix_pin = pin;
    return LDSO_B200_OK;
}

// float -> int as the reference's x86 build converts (cvttss2si): truncation, INT_MIN for NaN and out-of-range values
static int pixsel_f2i(float f) { return (f >= -2147483648.f && f < 2147483648.f) ? (int) f : INT_MIN; }

struct PixselResult { int n2, n3, n4, nsel, nkept, nfeat, pot; };

// makeMaps (PixelSelector2.cc:111-168) up to the output lists: the histogram once, one select() pass per recursion with a 16-byte
// read-back of its counts, the recursion and currentPotential on the host with the reference's float arithmetic, then the
// subsampling and the lists: every kept pixel as x / y / type, or (traces) the kept pixels in makeNewTraces' range as u / v / my_type.
// Ends with the header on the host.
static int pixsel_run(ldso_b200_ctx *c, const char *what, int slot, const ldso_b200_pixsel_params *p, const float *B, const int *current_potential,
                      bool traces, PixselArgs &a, PixselResult &R) {
    char msg[160];
#define PIXSEL_FAIL(text) do { snprintf(msg, sizeof(msg), "%s: %s", what, text); return c->fail(LDSO_B200_ERR_ARG, msg); } while (0)
    if (c->levels < 3) PIXSEL_FAIL("needs a context with at least 3 pyramid levels");
    if (slot < 0 || slot >= NSLOTS || !c->img[slot][0]) PIXSEL_FAIL("image slot out of range or never filled");
    if (!p || !current_potential) PIXSEL_FAIL("params or current_potential is NULL");
    if (!(p->density > 0)) PIXSEL_FAIL("density must be positive");
    if (*current_potential < 1) PIXSEL_FAIL("current_potential must be at least 1");
#undef PIXSEL_FAIL
    cudaSetDevice(c->device);
    RET_IF(pixsel_ensure(c));
    const int w = c->w, h = c->h;
    const size_t px = (size_t) w * h;
    Arena D(c->pix_mem);
    const PixselFixed f = pixsel_regions(D, w, h, traces, a);
    a.img0 = c->img[slot][0]; a.img1 = c->img[slot][1]; a.img2 = c->img[slot][2];
    a.B = nullptr;
    if (B) {
        H2D(f.B, B, sizeof(float) * 256);
        a.B = f.B;
    }
    a.w = w; a.h = h; a.w1 = c->lw[1]; a.w2 = c->lw[2];
    a.w32 = w / 32; a.h32 = h / 32;
    a.minGradHistCut = p->minGradHistCut; a.minGradHistAdd = p->minGradHistAdd;
    a.rp = f.rp;
    a.thFactor = p->th_factor; a.dw1 = p->gradDownweightPerLevel; a.dw2 = a.dw1 * a.dw1;
    a.dirDist = p->selectDirectionDistribution != 0;
    const int ncell32 = a.w32 * a.h32;
    if (ncell32 > 0) {                  // makeHists: once per call, whatever the potential
        k_pixsel_hist<<<ncell32, 1024, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        k_pixsel_smooth<<<(ncell32 + 255) / 256, 256, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
    }
    int pot = *current_potential, rec = p->recursions_left, ideal = pot;
    float quotia = 0.f;
    PixselArgs hp;
    Arena P(c->pix_pin);
    pixsel_pin_regions(P, 0, px, traces, hp);
    const int *hh = hp.hdr;
    for (;;) {
        // a potential of max(w, h) or more gives one cell, one 2pot and one 4pot block covering the image: the same pass
        const int pg = std::min(pot, std::max(w, h));
        a.pot = pg; a.cw = (w + pg - 1) / pg; a.ch = (h + pg - 1) / pg; a.bw4 = (w + 4 * pg - 1) / (4 * pg); a.bh4 = (h + 4 * pg - 1) / (4 * pg);
        CUDA_CHECK_RET(c, cudaMemsetAsync(a.map, 0, px, c->stream));
        CUDA_CHECK_RET(c, cudaMemsetAsync(a.hdr, 0, 4 * PIXSEL_HDR_INTS, c->stream));
        k_pixsel_mask<<<(a.cw * a.ch + 255) / 256, 256, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        k_pixsel_walk<<<1, 32, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        k_pixsel_pick<<<(a.bw4 * a.bh4 + 127) / 128, 128, 0, c->stream>>>(a);
        LAUNCH_CHECK(c);
        CUDA_CHECK_RET(c, cudaMemcpyAsync(hp.hdr, a.hdr, 16, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        R.n2 = hh[PIXSEL_N2]; R.n3 = hh[PIXSEL_N3]; R.n4 = hh[PIXSEL_N4];
        const float numHave = (float) (R.n2 + R.n3 + R.n4), numWant = p->density;
        quotia = numWant / numHave;
        const float K = numHave * (pot + 1) * (pot + 1);
        ideal = pixsel_f2i(sqrtf(K / numWant) - 1);
        if (ideal < 1) ideal = 1;
        if (rec > 0 && quotia > 1.25 && pot > 1) {
            if (ideal >= pot) ideal = pot - 1;
            pot = ideal; rec--;
        } else if (rec > 0 && quotia < 0.25) {
            if (ideal <= pot) ideal = pot + 1;
            pot = ideal; rec--;
        } else {
            break;
        }
    }
    a.charTH = quotia < 0.95 ? (int) (unsigned char) (255 * quotia) : 255;
    const int rows = (h * 32 + 255) / 256;
    k_pixsel_rows<<<rows, 256, 0, c->stream>>>(a);
    LAUNCH_CHECK(c);
    k_pixsel_row_scan<<<1, 1024, 0, c->stream>>>(a);
    LAUNCH_CHECK(c);
    k_pixsel_emit<<<rows, 256, 0, c->stream>>>(a);
    LAUNCH_CHECK(c);
    k_pixsel_finish<<<1, 1024, 0, c->stream>>>(a);
    LAUNCH_CHECK(c);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(hp.hdr, a.hdr, 4 * PIXSEL_HDR_INTS, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    R.nsel = hh[PIXSEL_NSEL]; R.nkept = hh[PIXSEL_NKEPT]; R.nfeat = hh[PIXSEL_NFEAT]; R.pot = ideal;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_select_pixels(ldso_b200_ctx *c, int slot, const ldso_b200_pixsel_params *params, const float *B, int *current_potential,
                                       ldso_b200_pixels *out) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (!out || !out->x || !out->y || !out->type) return c->fail(LDSO_B200_ERR_ARG, "select_pixels: missing output array");
    PixselArgs a;
    PixselResult R;
    RET_IF(pixsel_run(c, "select_pixels", slot, params, B, current_potential, false, a, R));
    const size_t px = (size_t) c->w * c->h;
    const int n = R.nkept;
    if (out->capacity < n) return c->fail(LDSO_B200_ERR_ARG, "select_pixels: capacity below the number of selected pixels");
    PixselArgs h;
    Arena P(c->pix_pin);
    pixsel_pin_regions(P, (size_t) n, px, false, h);
    D2H(h.sx, a.sx, 4 * (size_t) n);
    D2H(h.sy, a.sy, 4 * (size_t) n);
    D2H(h.stype, a.stype, (size_t) n);
    if (out->map) D2H(h.map, a.map, px);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    memcpy(out->x, h.sx, 4 * (size_t) n);
    memcpy(out->y, h.sy, 4 * (size_t) n);
    memcpy(out->type, h.stype, (size_t) n);
    if (out->map) memcpy(out->map, h.map, px);
    out->n = n; out->n2 = R.n2; out->n3 = R.n3; out->n4 = R.n4;
    *current_potential = R.pot;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_download_frame_level(ldso_b200_ctx *c, int slot, int lvl, float *out) {
    if (!c || !out || slot < 0 || slot >= NSLOTS || lvl < 0 || lvl >= c->levels || !c->img[slot][lvl]) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    const int npx = c->lw[lvl] * c->lh[lvl];
    k_unpack_aos3<<<(npx + 255) / 256, 256, 0, c->stream>>>(c->img[slot][lvl], c->scratch, npx);
    LAUNCH_CHECK(c);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(out, c->scratch, sizeof(float) * 3 * npx, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- window
template<typename T>
static int dev_alloc(ldso_b200_ctx *c, T **p, size_t count, std::vector<void *> *owner = nullptr) {
    void *q = nullptr;
    CUDA_CHECK_RET(c, cudaMalloc(&q, sizeof(T) * std::max<size_t>(count, 128)));   // empty windows still get valid buffers
    (owner ? *owner : c->win_allocs).push_back(q);
    *p = (T *) q;
    return 0;
}
template<typename T>
static int dev_upload(ldso_b200_ctx *c, T *dst, const T *src, size_t count) {
    if (count == 0) return 0;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(dst, src, sizeof(T) * count, cudaMemcpyHostToDevice, c->stream));
    return 0;
}

// Window memory: ONE device arena + ONE pinned host mirror with the same layout.
//   [topology | inputs ......................... | pt_idepth pt_idepth_zero | results ............ ]
//    ^ uploaded only when the CSR changes         ^---- upload range ------^
//                                                 ^----------- download range (one D2H) ----------^
// so a set_window is one pack + one cudaMemcpyAsync + one memset, and reading points/residuals back is one copy.
static int alloc_window(ldso_b200_ctx *c, int nP, int nR) {
    DevWindow &d = c->d;
    Arena A;
    // every region starts and ends on a 256-byte boundary, so the range ends below (topo_end, ...) are region starts as well
    auto take = [&](size_t bytes) { return (size_t) A.take((bytes + 255) & ~(size_t) 255, 256); };
    const size_t nPs = std::max(nP, 32), nRs = std::max(nR, 32);
    auto &L = c->lay;
    L.pt_host = take(4 * nPs); L.pt_res_begin = take(4 * (nPs + 1)); L.res_point = take(4 * nRs); L.res_target = take(4 * nRs);
    L.topo_end = A.off;
    L.pt_u = take(4 * nPs); L.pt_v = take(4 * nPs); L.pt_color = take(32 * nPs); L.pt_weights = take(32 * nPs);
    L.pt_priorF = take(4 * nPs); L.pt_idepth_backup = take(4 * nPs); L.res_lin = take(nRs);
    L.res_state = take(nRs);
    L.dl_begin = A.off;
    L.pt_idepth = take(4 * nPs); L.pt_idepth_zero = take(4 * nPs);
    L.ul_end = A.off;
    L.pt_step = take(4 * nPs); L.pt_HdiF = take(4 * nPs); L.pt_bdSumF = take(4 * nPs); L.pt_Hdd = take(4 * nPs);
    L.pt_bd = take(4 * nPs); L.pt_Hcd = take(16 * nPs);
    L.res_new_state = take(nRs); L.res_active = take(nRs); L.res_energy = take(4 * nRs); L.res_new_energy = take(4 * nRs);
    L.res_new_energy_wo = take(4 * nRs);
    L.dl_light_end = A.off;
    L.res_JpJdF = take(32 * nRs);
    L.dl_end = A.off;
    L.res_JpJdF_new = take(32 * nRs);
    L.total = A.off;
    // res_state is both an input and a result: it sits right before dl_begin and is fetched separately (tiny)
    CUDA_CHECK_RET(c, cudaMalloc(&c->arena_dev, L.total));
    CUDA_CHECK_RET(c, cudaMallocHost(&c->arena_host, L.total));
    memset(c->arena_host, 0, L.total);
    char *B = c->arena_dev;
    d.pt_host = (int *) (B + L.pt_host); d.pt_res_begin = (int *) (B + L.pt_res_begin);
    d.res_point = (int *) (B + L.res_point); d.res_target = (int *) (B + L.res_target);
    d.pt_u = (float *) (B + L.pt_u); d.pt_v = (float *) (B + L.pt_v); d.pt_color = (float *) (B + L.pt_color);
    d.pt_weights = (float *) (B + L.pt_weights); d.pt_priorF = (float *) (B + L.pt_priorF);
    d.pt_idepth_backup = (float *) (B + L.pt_idepth_backup); d.res_lin = (uint8_t *) (B + L.res_lin);
    d.res_state = (uint8_t *) (B + L.res_state);
    d.pt_idepth = (float *) (B + L.pt_idepth); d.pt_idepth_zero = (float *) (B + L.pt_idepth_zero);
    d.pt_step = (float *) (B + L.pt_step); d.pt_HdiF = (float *) (B + L.pt_HdiF); d.pt_bdSumF = (float *) (B + L.pt_bdSumF);
    d.pt_Hdd = (float *) (B + L.pt_Hdd); d.pt_bd = (float *) (B + L.pt_bd); d.pt_Hcd = (float *) (B + L.pt_Hcd);
    d.res_new_state = (uint8_t *) (B + L.res_new_state); d.res_active = (uint8_t *) (B + L.res_active);
    d.res_energy = (float *) (B + L.res_energy); d.res_new_energy = (float *) (B + L.res_new_energy);
    d.res_new_energy_wo = (float *) (B + L.res_new_energy_wo); d.res_JpJdF = (float *) (B + L.res_JpJdF);
    d.res_JpJdF_new = (float *) (B + L.res_JpJdF_new);
    // big arrays only the piecewise API / tests touch
    int rc = 0;
    rc |= dev_alloc(c, &d.res_J, (size_t) nR * 74);
    rc |= dev_alloc(c, &d.res_proj, (size_t) nR * 16); rc |= dev_alloc(c, &d.res_cpt, (size_t) nR * 3);
    rc |= dev_alloc(c, &d.res_toZero, (size_t) nR * 8);
    rc |= dev_alloc(c, &c->pt_sel_dev, nP);
    rc |= dev_alloc(c, &c->fb.pt_relBS_max, nP); rc |= dev_alloc(c, &c->fb.pt_n_good, nP); rc |= dev_alloc(c, &c->fb.res_dropped, nR);
    return rc ? LDSO_B200_ERR_CUDA : LDSO_B200_OK;
}

extern "C" int ldso_b200_set_window(ldso_b200_ctx *c, const ldso_b200_window *win) {
    if (!c || !win) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    const int nP = win->nPoints, nR = win->nResiduals;
    if (nP < 0 || nR < 0) return c->fail(LDSO_B200_ERR_ARG, "negative sizes");
    for (int p = 0; p < nP; p++) {
        if (win->pt_host[p] < 0 || win->pt_host[p] >= MAXF) return c->fail(LDSO_B200_ERR_ARG, "pt_host out of range");
        if (p > 0 && win->pt_host[p] < win->pt_host[p - 1]) return c->fail(LDSO_B200_ERR_ARG, "points must be ordered by host frame");
        if (win->res_begin[p + 1] < win->res_begin[p]) return c->fail(LDSO_B200_ERR_ARG, "res_begin must be non-decreasing");
        if (win->res_begin[p + 1] - win->res_begin[p] > MAXF) return c->fail(LDSO_B200_ERR_ARG, "more than MAX_FRAMES residuals on a point");
    }
    if (nP > 0 && (win->res_begin[0] != 0 || win->res_begin[nP] != nR)) return c->fail(LDSO_B200_ERR_ARG, "res_begin does not cover the residual arrays");
    for (int r = 0; r < nR; r++) if (win->res_target[r] < 0 || win->res_target[r] >= MAXF) return c->fail(LDSO_B200_ERR_ARG, "res_target out of range");
    if (c->window_copied) CUDA_CHECK_RET(c, cudaEventSynchronize(c->window_copied));     // the pinned mirror may still be in flight
    RET_IF(wait_results(c));                                                              // ... or be the target of a queued read-back
    DevWindow &d = c->d;
    const bool same_topology = c->have_window && d.nP == nP && d.nR == nR && (int) c->h_pt_host.size() == nP && nP > 0 &&
                               std::equal(win->pt_host, win->pt_host + nP, c->h_pt_host.begin()) &&
                               std::equal(win->res_begin, win->res_begin + nP + 1, c->h_res_begin.begin()) &&
                               std::equal(win->res_target, win->res_target + nR, c->h_res_target.begin());
    auto &L = c->lay;
    if (!same_topology) {
        free_window(c);
        memset(&d, 0, sizeof(d));
        d.nP = nP; d.nR = nR;
        c->h_pt_host.assign(win->pt_host, win->pt_host + nP);
        c->h_res_begin.assign(win->res_begin, win->res_begin + nP + 1);
        if (nP == 0) c->h_res_begin.assign(1, 0);
        c->h_res_target.assign(win->res_target, win->res_target + nR);
        int rc = alloc_window(c, nP, nR);
        if (rc) return rc;
        d.newest_offset = 0;
        d.newest_total = -1;   // derived
        c->derived_dirty = true;
        char *H = c->arena_host;
        memcpy(H + L.pt_host, win->pt_host, 4 * (size_t) nP);
        memcpy(H + L.pt_res_begin, c->h_res_begin.data(), 4 * ((size_t) nP + 1));
        int *rp = (int *) (H + L.res_point);
        for (int p = 0; p < nP; p++) for (int r = c->h_res_begin[p]; r < c->h_res_begin[p + 1]; r++) rp[r] = p;
        memcpy(H + L.res_target, win->res_target, 4 * (size_t) nR);
    }
    // ---- pack the per-call inputs into the pinned mirror
    char *H = c->arena_host;
    memcpy(H + L.pt_u, win->pt_u, 4 * (size_t) nP); memcpy(H + L.pt_v, win->pt_v, 4 * (size_t) nP);
    memcpy(H + L.pt_color, win->pt_color, 32 * (size_t) nP); memcpy(H + L.pt_weights, win->pt_weights, 32 * (size_t) nP);
    float *priorF = (float *) (H + L.pt_priorF);
    for (int p = 0; p < nP; p++)   // PointHessian::takeData (PointHessian.h:112-117)
        priorF[p] = (win->pt_has_prior && win->pt_has_prior[p]) ? c->S.idepthFixPrior * SCALE_IDEPTH * SCALE_IDEPTH : 0.f;
    memcpy(H + L.pt_idepth_backup, win->pt_idepth, 4 * (size_t) nP);
    if (win->res_is_linearized) memcpy(H + L.res_lin, win->res_is_linearized, nR); else memset(H + L.res_lin, 0, std::max(nR, 1));
    c->has_lin = false;
    if (win->res_is_linearized) for (int r = 0; r < nR; r++) if (win->res_is_linearized[r]) { c->has_lin = true; break; }
    if (win->res_state) memcpy(H + L.res_state, win->res_state, nR); else memset(H + L.res_state, LDSO_B200_RES_IN, std::max(nR, 1));
    memcpy(H + L.pt_idepth, win->pt_idepth, 4 * (size_t) nP); memcpy(H + L.pt_idepth_zero, win->pt_idepth_zero, 4 * (size_t) nP);
    const size_t ul_begin = same_topology ? L.topo_end : 0;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->arena_dev + ul_begin, H + ul_begin, L.ul_end - ul_begin, cudaMemcpyHostToDevice, c->stream));
    if (!c->window_copied) CUDA_CHECK_RET(c, cudaEventCreateWithFlags(&c->window_copied, cudaEventDisableTiming));
    CUDA_CHECK_RET(c, cudaEventRecord(c->window_copied, c->stream));
    CUDA_CHECK_RET(c, cudaMemsetAsync(c->arena_dev + L.ul_end, 0, L.total - L.ul_end, c->stream));    // all result/state arrays
    if (win->res_toZeroF && nR > 0) CUDA_CHECK_RET(c, cudaMemcpyAsync(d.res_toZero, win->res_toZeroF, 32 * (size_t) nR, cudaMemcpyHostToDevice, c->stream));
    if (!same_topology) CUDA_CHECK_RET(c, cudaMemsetAsync(d.res_J, 0, sizeof(float) * 74 * (size_t) std::max(nR, 1), c->stream));
    if (win->res_toZeroF) CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));   // pageable source
    { c->mirror_valid = false; c->results_inflight = false; c->sol_valid = false; c->mirror_full_valid = false; }
    c->solve_ready = false; c->restitch_ok = false;
    c->have_window = true;
    c->fin_window_stale = false; c->fin_state = 0;
    return LDSO_B200_OK;
}

// work items, newest-frame slots, partial buffers: need both the window and nF
static int build_derived(ldso_b200_ctx *c) {
    if (!c->have_window || !c->have_frames) return c->fail(LDSO_B200_ERR_STATE, "set_frames and set_window must both be called first");
    if (c->fin_window_stale) return c->fail(LDSO_B200_ERR_STATE, "optimize_finish left dropped residuals in the window: call set_window first");
    if (!c->derived_dirty) return LDSO_B200_OK;
    DevWindow &d = c->d;
    const int nP = d.nP, nR = d.nR, nF = c->nF;
    for (int p = 0; p < nP; p++) if (c->h_pt_host[p] >= nF) return c->fail(LDSO_B200_ERR_ARG, "pt_host >= nFrames");
    for (int r = 0; r < nR; r++) if (c->h_res_target[r] >= nF) return c->fail(LDSO_B200_ERR_ARG, "res_target >= nFrames");
    // two co-resident CTAs per SM hide each other's phase latencies (K1 is a chain of short, barrier-separated phases)
    // ... and large windows are cut into whole waves of 2*SMs items (at most 64 points each: the records of an item live in
    // shared memory), so that the last wave is as full as the first
    const int slots = 2 * std::max(c->sm_count, 1);
    const int waves = std::max(1, (nP + 64 * slots - 1) / (64 * slots));
    const int target_items = waves * slots;
    int ppi = (nP + target_items - 1) / target_items;
    ppi = std::max(4, std::min(64, ppi));
    d.pts_per_item = ppi;
    c->k1_smem = k1_smem_bytes(ppi);
    std::vector<int4> items;
    std::vector<int> hib(MAXF + 1, 0);
    int p = 0;
    for (int h = 0; h < MAXF; h++) {
        hib[h] = (int) items.size();
        while (p < nP && c->h_pt_host[p] == h) {
            int e = p;
            while (e < nP && c->h_pt_host[e] == h && e - p < ppi) e++;
            items.push_back(make_int4(h, p, e, 0));
            p = e;
        }
    }
    hib[MAXF] = (int) items.size();
    d.nItems = (int) items.size();
    std::vector<int> slot(nR, -1);
    int ns = 0;
    for (int r = 0; r < nR; r++) if (c->h_res_target[r] == nF - 1) slot[r] = ns++;
    const int local_newest = ns;
    if (d.newest_total < 0 || !c->multi) { d.newest_total = local_newest; d.newest_offset = 0; }
    for (int r = 0; r < nR; r++) if (slot[r] >= 0) slot[r] += d.newest_offset;

    int4 *items_dev; int *hib_dev, *slot_dev;
    int rc = 0;
    // the previous derived buffers (same window, other nF / shard description) may still be read by queued kernels
    if (!c->derived_allocs.empty()) { CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream)); free_derived(c); }
    std::vector<void *> *own = &c->derived_allocs;
    rc |= dev_alloc(c, &items_dev, items.size(), own); rc |= dev_alloc(c, &hib_dev, MAXF + 1, own); rc |= dev_alloc(c, &slot_dev, nR, own);
    rc |= dev_alloc(c, &d.partials, (size_t) std::max(d.nItems, 1) * PART_STRIDE, own);
    rc |= dev_alloc(c, &d.item_stats, (size_t) std::max(d.nItems, 1) * 4, own);
    rc |= dev_alloc(c, &d.red, (size_t) RED_SELECT + std::max(d.newest_total, 1) + 16, own);
    rc |= dev_alloc(c, &d.dbg, 32 + 3 * (size_t) std::max(d.nItems, 1), own);
    if (rc) return LDSO_B200_ERR_CUDA;
    rc |= dev_upload(c, items_dev, items.data(), items.size());
    rc |= dev_upload(c, hib_dev, hib.data(), MAXF + 1);
    rc |= dev_upload(c, slot_dev, slot.data(), nR);
    if (rc) return LDSO_B200_ERR_CUDA;
    CUDA_CHECK_RET(c, cudaMemsetAsync(d.red, 0, sizeof(double) * ((size_t) RED_SELECT + std::max(d.newest_total, 1) + 16), c->stream));
    CUDA_CHECK_RET(c, cudaMemsetAsync(d.partials, 0, sizeof(float) * (size_t) std::max(d.nItems, 1) * PART_STRIDE, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    if (c->peers_connected && c->px.n_doubles != RED_SELECT + std::max(d.newest_total, 0))
        return c->fail(LDSO_B200_ERR_STATE, "the window's newest-frame residual count changed: the peer exchange buffers must be re-exported");
    d.items = items_dev; d.host_item_begin = hib_dev; d.res_newest_slot = slot_dev;
    c->derived_dirty = false;
    c->gn_graph_valid = false; c->until_graph_valid = false;
    return LDSO_B200_OK;
}

// the solve entry points also need the null-space projector of the current evaluation points (set_frames after optimize_finish)
static int check_solve_frames(ldso_b200_ctx *c) {
    if (c->fin_frames_stale) return c->fail(LDSO_B200_ERR_STATE, "optimize_finish moved the newest evaluation point: call set_frames first");
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- frames
extern "C" int ldso_b200_set_frames(ldso_b200_ctx *c, int nFrames, const ldso_b200_frame_state *frames,
                                    const double calib_value_scaled[4], const double calib_value_zero[4]) {
    if (!c || !frames || !calib_value_scaled || !calib_value_zero) return LDSO_B200_ERR_ARG;
    if (nFrames < 1 || nFrames > MAXF) return c->fail(LDSO_B200_ERR_ARG, "nFrames must be in [1, LDSO_B200_MAX_FRAMES]");
    cudaSetDevice(c->device);
    // ws_host (pinned) may still be the source of the previous call's upload: wait for that copy only (not for the
    // kernels queued behind it), so that back-to-back calls overlap host packing with device work
    CUDA_CHECK_RET(c, cudaEventSynchronize(c->frames_copied));
    using namespace hostmath;
    WinState &W = *c->ws_host;
    // the adjoints and the null-space projector depend only on the evaluation points (worldToCam_evalPT, state_zero's
    // affine part, exposures): they change once per keyframe, so they are recomputed only when those inputs change
    std::vector<double> key;
    key.reserve((size_t) nFrames * 16 + 1);
    key.push_back((double) nFrames);
    for (int i = 0; i < nFrames; i++) {
        key.insert(key.end(), frames[i].evalR, frames[i].evalR + 9);
        key.insert(key.end(), frames[i].evalT, frames[i].evalT + 3);
        key.push_back(frames[i].state_zero[6]); key.push_back(frames[i].state_zero[7]); key.push_back(frames[i].ab_exposure);
    }
    const bool evalpt_cached = c->have_frames && key == c->evalpt_key;
    if (evalpt_cached) {
        // keep adHost/adTarget(/F) of the previous call; everything else is rewritten below
        memset(&W, 0, offsetof(WinState, adHost));
        memset((char *) &W + offsetof(WinState, cPrior), 0, sizeof(WinState) - offsetof(WinState, cPrior));
    } else {
        memset(&W, 0, sizeof(W));
    }
    const int nF = nFrames, n = 8 * nF + CPARS;
    const int prev_nF = c->have_frames ? c->nF : -1;
    W.nF = nF; W.n = n; W.w = c->w; W.h = c->h;
    W.wM3G = (float) (c->w - 3); W.hM3G = (float) (c->h - 3);      // GlobalCalib.cc:42-43
    W.S = c->S;
    std::vector<Pose> ev(nF);
    for (int i = 0; i < nF; i++) {
        const ldso_b200_frame_state &f = frames[i];
        if (f.image_slot < 0 || f.image_slot >= NSLOTS || !c->img[f.image_slot][0]) return c->fail(LDSO_B200_ERR_ARG, "frame image slot not uploaded");
        FrameDev &D = W.fr[i];
        memcpy(D.evalR, f.evalR, sizeof(D.evalR)); memcpy(D.evalT, f.evalT, sizeof(D.evalT));
        memcpy(D.state, f.state, sizeof(D.state)); memcpy(D.state_zero, f.state_zero, sizeof(D.state_zero));
        memcpy(D.state_backup, f.state, sizeof(D.state));
        D.frameEnergyTH = f.frameEnergyTH; W.frameEnergyTH[i] = f.frameEnergyTH; D.ab_exposure = f.ab_exposure; D.frame_id = f.frame_id; D.slot = f.image_slot;
        // FrameHessian::getPrior (FrameHessian.h:125-150), takeData (FrameHessian.cc:108-112)
        double p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        if (f.frame_id == 0) {
            p[0] = p[1] = p[2] = c->S.initialTransPrior;
            p[3] = p[4] = p[5] = c->S.initialRotPrior;
            p[6] = c->S.initialAffAPrior;
            p[7] = c->S.initialAffBPrior;
        } else {
            p[6] = (c->S.affineOptModeA < 0) ? c->S.initialAffAPrior : c->S.affineOptModeA;
            p[7] = (c->S.affineOptModeB < 0) ? c->S.initialAffBPrior : c->S.affineOptModeB;
        }
        for (int k = 0; k < 8; k++) D.prior[k] = p[k];
        memcpy(ev[i].R, f.evalR, sizeof(ev[i].R)); memcpy(ev[i].t, f.evalT, sizeof(ev[i].t));
        W.img0[i] = c->img[f.image_slot][0];
        c->slots[i] = f.image_slot;
    }
    // calibration (CalibHessian::setValueScaled, CalibHessian.h:87-100)
    CalibDev &C = W.calib;
    for (int i = 0; i < 4; i++) { C.value_scaled[i] = calib_value_scaled[i]; C.value_zero[i] = calib_value_zero[i]; }
    C.value[0] = (double) (1.0f / SCALE_F) * C.value_scaled[0]; C.value[1] = (double) (1.0f / SCALE_F) * C.value_scaled[1];
    C.value[2] = (double) (1.0f / SCALE_C) * C.value_scaled[2]; C.value[3] = (double) (1.0f / SCALE_C) * C.value_scaled[3];
    for (int i = 0; i < 4; i++) C.value_backup[i] = C.value[i];
    C.fxl = (float) C.value_scaled[0]; C.fyl = (float) C.value_scaled[1]; C.cxl = (float) C.value_scaled[2]; C.cyl = (float) C.value_scaled[3];
    C.fxli = 1.0f / C.fxl; C.fyli = 1.0f / C.fyl; C.cxli = -C.cxl / C.fxl; C.cyli = -C.cyl / C.fyl;
    for (int i = 0; i < 4; i++) { C.cDeltaF[i] = (float) (C.value[i] - C.value_zero[i]); W.cPrior[i] = c->S.initialCalibHessian; }

    // EnergyFunctional::setAdjointsF (EnergyFunctional.cc:431-489)
    if (!evalpt_cached)
    for (int h = 0; h < nF; h++)
        for (int t = 0; t < nF; t++) {
            Pose hostToTarget = mul(ev[t], inv(ev[h]));
            double Adj[36];
            adjoint(hostToTarget, Adj);
            double *AH = W.adHost[h + nF * t], *AT = W.adTarget[h + nF * t];
            for (int i = 0; i < 8; i++) AH[i * 8 + i] = AT[i * 8 + i] = 1.0;
            for (int i = 0; i < 6; i++) for (int j = 0; j < 6; j++) AH[i * 8 + j] = -Adj[j * 6 + i];
            float eF = frames[h].ab_exposure, eT = frames[t].ab_exposure;
            if (eF == 0 || eT == 0) eT = eF = 1;
            const float a0h = (float) (frames[h].state_zero[6] * SCALE_A), a0t = (float) (frames[t].state_zero[6] * SCALE_A);
            const float affLL0 = expf(a0t - a0h) * eT / eF;
            AT[6 * 8 + 6] = -affLL0; AH[6 * 8 + 6] = affLL0; AT[7 * 8 + 7] = -1; AH[7 * 8 + 7] = affLL0;
            for (int j = 0; j < 8; j++) {
                for (int i = 0; i < 3; i++) { AH[i * 8 + j] *= SCALE_XI_TRANS; AT[i * 8 + j] *= SCALE_XI_TRANS; }
                for (int i = 3; i < 6; i++) { AH[i * 8 + j] *= SCALE_XI_ROT; AT[i * 8 + j] *= SCALE_XI_ROT; }
                AH[6 * 8 + j] *= SCALE_A; AT[6 * 8 + j] *= SCALE_A;
                AH[7 * 8 + j] *= SCALE_B; AT[7 * 8 + j] *= SCALE_B;
            }
            for (int i = 0; i < 64; i++) { W.adHostF[h + nF * t][i] = (float) AH[i]; W.adTargetF[h + nF * t][i] = (float) AT[i]; }
        }

    // null spaces (FrameHessian::setStateZero, FrameHessian.cc:11-42; FullSystem::getNullspaces, FullSystem.cc:1711-1760)
    // and the projector EnergyFunctional::orthogonalize applies (pose + scale, EnergyFunctional.cc:687-716)
    std::vector<double> N((size_t) n * 7, 0.0);
    if (!evalpt_cached) {
    for (int f = 0; f < nF; f++) {
        const Pose evI = inv(ev[f]);
        for (int i = 0; i < 6; i++) {
            double e[6] = {0, 0, 0, 0, 0, 0}, m[6] = {0, 0, 0, 0, 0, 0};
            e[i] = 1e-3; m[i] = -1e-3;
            double lp[6], lm[6];
            logm(mul(mul(ev[f], expm(e)), evI), lp);
            logm(mul(mul(ev[f], expm(m)), evI), lm);
            for (int r = 0; r < 6; r++) {
                double v = (lp[r] - lm[r]) / 2e-3;
                v *= (r < 3) ? (double) (1.0f / SCALE_XI_TRANS) : (double) (1.0f / SCALE_XI_ROT);
                N[(size_t) i * n + CPARS + 8 * f + r] = v;
            }
        }
        Pose P = ev[f], M = ev[f];
        for (int k = 0; k < 3; k++) { P.t[k] *= 1.00001; M.t[k] /= 1.00001; }
        double lp[6], lm[6];
        logm(mul(P, evI), lp);
        logm(mul(M, evI), lm);
        for (int r = 0; r < 6; r++) {
            double v = (lp[r] - lm[r]) / 2e-3;
            v *= (r < 3) ? (double) (1.0f / SCALE_XI_TRANS) : (double) (1.0f / SCALE_XI_ROT);
            N[(size_t) 6 * n + CPARS + 8 * f + r] = v;
        }
    }
    for (int j = 0; j < 7; j++) {   // N.col(i) = ns[i].normalized()
        double s = 0;
        for (int r = 0; r < n; r++) s += N[(size_t) j * n + r] * N[(size_t) j * n + r];
        s = sqrt(s);
        if (s > 0) for (int r = 0; r < n; r++) N[(size_t) j * n + r] /= s;
    }
    range_projector(N, n, 7, c->S.solverModeDelta, c->Pns_host);
    c->evalpt_key = key;
    }

    c->nF = nF; c->n = n;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->ws_dev, c->ws_host, sizeof(WinState), cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(c, cudaEventRecord(c->frames_copied, c->stream));
    if (!evalpt_cached)     // pageable source: staged before the call returns
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sb.Pns, c->Pns_host.data(), sizeof(double) * n * n, cudaMemcpyHostToDevice, c->stream));
    if (c->prior_dim == n) {
        // same frames as the prior describes (a repeated set_frames, or the window after marginalize_frame + insertFrame)
    } else if (c->prior_dim > 0 && c->prior_dim == n - 8) {
        // one keyframe appended since the prior was last touched: EnergyFunctional::insertFrame (EnergyFunctional.cc:38-44)
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sb.A0g, c->sb.HM, sizeof(double) * (n - 8) * (n - 8), cudaMemcpyDeviceToDevice, c->stream));
        k_grow_prior<<<(n * n + 255) / 256, 256, 0, c->stream>>>(c->sb, c->sb.A0g, n);
        LAUNCH_CHECK(c);
        c->prior_dim = n;
    } else {
        CUDA_CHECK_RET(c, cudaMemsetAsync(c->sb.HM, 0, sizeof(double) * n * n, c->stream));
        CUDA_CHECK_RET(c, cudaMemsetAsync(c->sb.bM, 0, sizeof(double) * n, c->stream));
        c->prior_dim = 0;
    }
    k_frames_refresh<<<1, 128, 0, c->stream>>>(c->ws_dev);
    LAUNCH_CHECK(c);
    c->solve_ready = false; c->restitch_ok = false; c->select_pending = false;
    c->have_frames = true;
    c->fin_frames_stale = false;
    c->fin_state = 0;        // get_finish describes the frames the finish ran on, not these
    if (prev_nF != nF) c->derived_dirty = true;    // work items / newest-frame slots depend on nF only
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_set_marg_prior(ldso_b200_ctx *c, const double *HM, const double *bM) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    const int n = c->n;
    if (HM) CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sb.HM, HM, sizeof(double) * n * n, cudaMemcpyHostToDevice, c->stream));
    else CUDA_CHECK_RET(c, cudaMemsetAsync(c->sb.HM, 0, sizeof(double) * n * n, c->stream));
    if (bM) CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sb.bM, bM, sizeof(double) * n, cudaMemcpyHostToDevice, c->stream));
    else CUDA_CHECK_RET(c, cudaMemsetAsync(c->sb.bM, 0, sizeof(double) * n, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    c->solve_ready = false;      // HM/bM enter the assembled system
    c->prior_dim = (HM || bM) ? n : 0;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_marg_prior(ldso_b200_ctx *c, double *HM, double *bM) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    const int n = (c->prior_dim > 0) ? c->prior_dim : c->n;      // n - 8 between marginalize_frame and the next set_frames
    if (HM) CUDA_CHECK_RET(c, cudaMemcpyAsync(HM, c->sb.HM, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
    if (bM) CUDA_CHECK_RET(c, cudaMemcpyAsync(bM, c->sb.bM, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- launches
// One launch path for the loop kernels: inside launch_gn_body the kernel is allowed to start (and run its constant-data
// prologue up to pdl_wait()) while its predecessor on the stream is still executing.
template<typename... KArgs, typename... Args>
static cudaError_t launch_loop_kernel(ldso_b200_ctx *c, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, Args... args) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = c->stream;
    cudaLaunchAttribute at[1];
    memset(at, 0, sizeof(at));
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = (c->pdl_now && c->use_pdl && !c->ktime) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

static int launch_k1(ldso_b200_ctx *c, int flags, const uint8_t *sel = nullptr) {
    if (c->d.nItems == 0) return LDSO_B200_OK;
    c->kt_begin("k1");
    launch_loop_kernel(c, k1_linearize_accumulate, dim3(c->d.nItems), dim3(K1_THREADS), c->k1_smem, c->d, (const WinState *) c->ws_dev, flags, sel);
    c->kt_end();
    LAUNCH_CHECK(c);
    return LDSO_B200_OK;
}
static int launch_k2a(ldso_b200_ctx *c, int full) {
    const int nb = (MAXF * PART_USED + 63) / 64 + 1;
    c->kt_begin("k2a");
    launch_loop_kernel(c, k2a_reduce, dim3(nb), dim3(K2A_THREADS), 0, c->d, c->ws_dev, full, c->multi ? 1 : 0);
    c->kt_end();
    LAUNCH_CHECK(c);
    if (full) { c->restitch_ok = true; c->solve_ready = false; }
    return LDSO_B200_OK;
}
static int launch_k2b(ldso_b200_ctx *c, int do_stitch, int do_select, int do_assemble) {
    if (do_stitch && do_assemble && c->prior_dim != 0 && c->prior_dim != c->n)
        return c->fail(LDSO_B200_ERR_STATE, "the marginalisation prior has a different dimension than the frames (marginalize_frame): call set_frames with the remaining frames first");
    const int nb = c->nF * c->nF + c->nF + 2;
    c->kt_begin("k2b");
    DevWindow dw = c->d;
    if (c->peers_connected) dw.red = c->red_sum;      // the stitch reads the all-reduced accumulators
    launch_loop_kernel(c, k2b_stitch, dim3(nb), dim3(K2B_THREADS), K2B_SMEM_BYTES, dw, c->ws_dev, c->sb, do_stitch, do_select, (int) (do_stitch && do_assemble));
    c->kt_end();
    LAUNCH_CHECK(c);
    if (do_stitch) c->solve_ready = do_assemble != 0;
    if (do_select) c->select_pending = false;
    return LDSO_B200_OK;
}
static int launch_k2r(ldso_b200_ctx *c) {
    c->kt_begin("k2r");
    launch_loop_kernel(c, k2r_peer_allreduce, dim3(c->px.n_chunks), dim3(K2R_THREADS), 0, c->d, c->px);
    c->kt_end();
    LAUNCH_CHECK(c);
    return LDSO_B200_OK;
}
// K3(SOLVE) consumes what K2b(do_assemble) left behind; re-stitch if only the prior changed in between
static int ensure_solve_ready(ldso_b200_ctx *c) {
    if (c->solve_ready) return LDSO_B200_OK;
    if (!c->restitch_ok) return c->fail(LDSO_B200_ERR_STATE, "no stitched system for the current window state: call optimize_begin / solve_system first");
    return launch_k2b(c, 1, 0, 1);
}
static int launch_k3(ldso_b200_ctx *c, int flags) {
    c->kt_begin("k3");
    const double *sel_red = c->peers_connected ? c->red_sum : c->d.red;
    launch_loop_kernel(c, k3_solve_step, dim3((flags & K3F_SELECT) ? 2 : 1), dim3(K3_THREADS), K3_SMEM_BYTES, c->ws_dev, c->sb, flags, c->iteration_dev,
                       sel_red, std::max(c->d.newest_total, 0), c->d.dbg);
    c->kt_end();
    LAUNCH_CHECK(c);
    return LDSO_B200_OK;
}
static int set_iteration(ldso_b200_ctx *c, int it) {
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->iteration_dev, &it, sizeof(int), cudaMemcpyHostToDevice, c->stream));
    return LDSO_B200_OK;
}
static int clear_select(ldso_b200_ctx *c) {   // multi-GPU: slots owned by other ranks must be zero before the all-reduce
    if (c->multi && c->d.newest_total > 0)
        CUDA_CHECK_RET(c, cudaMemsetAsync(c->d.red + RED_SELECT, 0, sizeof(double) * c->d.newest_total, c->stream));
    return LDSO_B200_OK;
}

// grows a one-shot scratch block, device or pinned, to at least `bytes`; what it held is not kept
static int scratch_reserve(ldso_b200_ctx *c, char *&buf, size_t &cap, size_t bytes, bool pinned) {
    if (bytes <= cap) return LDSO_B200_OK;
    if (buf) { if (pinned) cudaFreeHost(buf); else cudaFree(buf); }
    buf = nullptr; cap = 0;
    CUDA_CHECK_RET(c, pinned ? cudaMallocHost(&buf, bytes) : cudaMalloc(&buf, bytes));
    cap = bytes;
    return LDSO_B200_OK;
}
// sizes one call's device scratch with its region list (scratch_layout.cuh), grows trace_buf to fit, and carves it with the same list
template <typename List>
static int trace_carve(ldso_b200_ctx *c, List &&list) {
    Arena S;
    list(S);
    RET_IF(scratch_reserve(c, c->trace_buf, c->trace_cap, S.off, false));
    Arena D(c->trace_buf);
    list(D);
    return LDSO_B200_OK;
}
static int flush_select(ldso_b200_ctx *c);                      // run a deferred setNewFrameEnergyTH select (fused loop)
extern "C" int ldso_b200_linearize_all(ldso_b200_ctx *c, int fixLinearization, int flags, double *energy_out) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    (void) flags;   // the piecewise path always keeps the full Jacobian: solve_system rebuilds its records from it
    RET_IF(flush_select(c));
    int f = K1F_LINEARIZE | K1F_STORE_J;
    if (fixLinearization) f |= K1F_APPLY_RES;
    RET_IF(clear_select(c));
    RET_IF(launch_k1(c, f));
    RET_IF(launch_k2a(c, 0));
    RET_IF(launch_k2b(c, 0, 1, 0));
    if (energy_out) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(energy_out, &c->ws_dev->energy, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_apply_res(ldso_b200_ctx *c) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    if (c->d.nR > 0) {
        k_apply_res<<<(c->d.nR + 255) / 256, 256, 0, c->stream>>>(c->d);
        LAUNCH_CHECK(c);
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_backup_state(ldso_b200_ctx *c) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(launch_k3(c, K3F_BACKUP));
    if (c->d.nP > 0) {
        k_points<<<(c->d.nP + 255) / 256, 256, 0, c->stream>>>(c->d, c->ws_dev, 1);
        LAUNCH_CHECK(c);
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_solve_system(ldso_b200_ctx *c, int iteration, double *lastHS, double *lastbS, double *lastX) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(check_solve_frames(c));
    // records from the stored Jacobians: accumulateAF (mode 0); with linearized residuals in the window, accumulateLF's terms
    // (mode 1: res_toZeroF + J delta) ride in the same pass -- solveSystemF only ever uses HA + HL and the summed point terms
    RET_IF(launch_k1(c, K1F_ACCUMULATE | ((c->has_lin ? 3 : 0) << K1F_MODE_SHIFT)));
    RET_IF(launch_k2a(c, 1));
    RET_IF(launch_k2b(c, 1, 0, 1));
    RET_IF(set_iteration(c, iteration));
    RET_IF(launch_k3(c, K3F_SOLVE));
    if (c->d.nP > 0) {
        k_points<<<(c->d.nP + 255) / 256, 256, 0, c->stream>>>(c->d, c->ws_dev, 2);
        LAUNCH_CHECK(c);
    }
    return ldso_b200_get_last_solution(c, lastHS, lastbS, lastX);
}

// AccumulatedTopHessianSSE::addPoint<mode> over a set of points + stitchDouble, and AccumulatedSCHessianSSE::addPoint + stitchDouble
// on the same set (AccumulatedTopHessian.cc:9-118,129-255; AccumulatedSCHessian.cc:9-119): what EnergyFunctional::accumulateAF_MT /
// accumulateLF_MT / accumulateSCF_MT and marginalizePointsF call. Records are rebuilt from the stored Jacobians (linearize_all).
// mode 0/1/2 as the reference's template argument, 3 = modes 0 and 1 in one pass. point_idx == NULL: all points. H, b WITHOUT the
// frame / calibration priors (stitchDouble(usePrior = false)); the caller adds them where the reference passes usePrior = true.
extern "C" int ldso_b200_accumulate(ldso_b200_ctx *c, int mode, int n_points, const int32_t *point_idx, int shift_prior_to_zero,
                                    double *H_top, double *b_top, double *H_sc, double *b_sc, int *nres) {
    if (!c || mode < 0 || mode > 3 || n_points < 0) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    const uint8_t *sel = nullptr;
    if (point_idx) {
        std::vector<uint8_t> hsel(std::max(c->d.nP, 1), 0);
        for (int i = 0; i < n_points; i++) {
            if (point_idx[i] < 0 || point_idx[i] >= c->d.nP) return c->fail(LDSO_B200_ERR_ARG, "point index out of range");
            hsel[point_idx[i]] = 1;
        }
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->pt_sel_dev, hsel.data(), c->d.nP, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        sel = c->pt_sel_dev;
    }
    RET_IF(launch_k1(c, K1F_ACCUMULATE | (shift_prior_to_zero ? 0 : K1F_NO_SHIFT_PRIOR) | (mode << K1F_MODE_SHIFT), sel));
    RET_IF(launch_k2a(c, 1));
    RET_IF(launch_k2b(c, 1, 0, 0));
    c->restitch_ok = false;      // the reduced buffer describes this call's selection / mode, not the window's system
    return ldso_b200_get_system(c, H_top, b_top, H_sc, b_sc, nres);
}

extern "C" int ldso_b200_get_last_solution(ldso_b200_ctx *c, double *lastHS, double *lastbS, double *lastX) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    const int n = c->n;
    // one copy of [lastHS | lastbS | lastX] into pinned staging memory, then plain memcpy into the caller's buffers
    const size_t nn = (size_t) MAXN * MAXN;
    RET_IF(wait_results(c));
    if (!c->sol_valid) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sol_host, c->sb.lastHS, sizeof(double) * (nn + 2 * MAXN), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        c->sol_valid = true;
    }
    if (lastHS) memcpy(lastHS, c->sol_host, sizeof(double) * n * n);
    if (lastbS) memcpy(lastbS, c->sol_host + nn, sizeof(double) * n);
    if (lastX) memcpy(lastX, c->sol_host + nn + MAXN, sizeof(double) * n);
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_system(ldso_b200_ctx *c, double *H_A, double *b_A, double *H_sc, double *b_sc, int *resInA) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    const int n = c->n;
    if (H_A) CUDA_CHECK_RET(c, cudaMemcpyAsync(H_A, c->sb.H_A, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
    if (b_A) CUDA_CHECK_RET(c, cudaMemcpyAsync(b_A, c->sb.b_A, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
    if (H_sc) CUDA_CHECK_RET(c, cudaMemcpyAsync(H_sc, c->sb.H_sc, sizeof(double) * n * n, cudaMemcpyDeviceToHost, c->stream));
    if (b_sc) CUDA_CHECK_RET(c, cudaMemcpyAsync(b_sc, c->sb.b_sc, sizeof(double) * n, cudaMemcpyDeviceToHost, c->stream));
    if (resInA) CUDA_CHECK_RET(c, cudaMemcpyAsync(resInA, &c->ws_dev->resInA, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_do_step(ldso_b200_ctx *c, int *canbreak) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(check_solve_frames(c));
    k_sum_nid<<<1, 256, 0, c->stream>>>(c->d, c->ws_dev);
    LAUNCH_CHECK(c);
    RET_IF(launch_k3(c, K3F_STEP));
    if (c->d.nP > 0) {
        k_points<<<(c->d.nP + 255) / 256, 256, 0, c->stream>>>(c->d, c->ws_dev, 4);
        LAUNCH_CHECK(c);
    }
    if (canbreak) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(canbreak, &c->ws_dev->canbreak, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    }
    return LDSO_B200_OK;
}

// FullSystem::flagPointsForRemoval's re-linearisation of the points to marginalise (FullSystem.cc:1241-1249:
// resetOOB, linearize, applyRes(true), fixLinearizationF) followed by EnergyFunctional::marginalizePointsF
// (EnergyFunctional.cc:165-222): priorF *= prior_fac, addPoint<2> + SC addPoint(p, false), stitchDouble without priors,
// HM += margWeightFac (M - Msc), bM likewise. The caller then drops the points from its window.
extern "C" int ldso_b200_marginalize_points(ldso_b200_ctx *c, int n, const int32_t *point_idx, float prior_fac, int *resInM) {
    if (!c || n < 0 || (n > 0 && !point_idx)) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    std::vector<uint8_t> sel(std::max(c->d.nP, 1), 0);
    for (int i = 0; i < n; i++) {
        if (point_idx[i] < 0 || point_idx[i] >= c->d.nP) return c->fail(LDSO_B200_ERR_ARG, "point index out of range");
        sel[point_idx[i]] = 1;
    }
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->pt_sel_dev, sel.data(), c->d.nP, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    RET_IF(flush_select(c));
    RET_IF(launch_k1(c, K1F_LINEARIZE | K1F_STORE_J | K1F_APPLY_RES | K1F_RESET_OOB, c->pt_sel_dev));
    if (c->d.nR > 0) {
        k_fix_linearization<<<(c->d.nR + 255) / 256, 256, 0, c->stream>>>(c->d, c->ws_dev, c->pt_sel_dev);
        LAUNCH_CHECK(c);
        k_scale_prior<<<(c->d.nP + 255) / 256, 256, 0, c->stream>>>(c->d, c->pt_sel_dev, prior_fac);
        LAUNCH_CHECK(c);
    }
    c->has_lin = c->has_lin || n > 0;
    RET_IF(launch_k1(c, K1F_ACCUMULATE | K1F_NO_SHIFT_PRIOR | (2 << K1F_MODE_SHIFT), c->pt_sel_dev));
    RET_IF(launch_k2a(c, 1));
    RET_IF(launch_k2b(c, 1, 0, 0));
    c->restitch_ok = false;      // the reduced buffer now holds the mode-2 (marginalisation) accumulators
    c->prior_dim = c->n;
    const int nn = c->n;
    k_add_marg<<<(nn * nn + 255) / 256, 256, 0, c->stream>>>(c->sb, nn, (double) c->S.margWeightFac);
    LAUNCH_CHECK(c);
    if (resInM) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(resInM, &c->ws_dev->resInA, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    }
    return LDSO_B200_OK;
}

// EnergyFunctional::calcLEnergyF_MT / calcMEnergyF (EnergyFunctional.cc:353-378): the prior + linearised-residual energy and the
// marginalisation energy at the current state (FullSystem::optimize reads both around every step, FullSystem.cc:1697-1703).
extern "C" int ldso_b200_calc_energies(ldso_b200_ctx *c, double *energyL, double *energyM) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    if (c->prior_dim != 0 && c->prior_dim != c->n) return c->fail(LDSO_B200_ERR_STATE, "prior dimension does not match the frames: call set_frames first");
    const int nb = std::max(1, (c->d.nP + KEN_THREADS - 1) / KEN_THREADS);
    EnergyScratch E;
    RET_IF(trace_carve(c, [&](Arena &A) { calc_energies_regions(A, nb, E); }));
    CUDA_CHECK_RET(c, cudaMemsetAsync(E.counter, 0, sizeof(unsigned), c->stream));
    k_calc_energies<<<nb, KEN_THREADS, 0, c->stream>>>(c->d, c->ws_dev, c->sb, E.part, E.counter, E.out);
    LAUNCH_CHECK(c);
    double h[2];
    CUDA_CHECK_RET(c, cudaMemcpyAsync(h, E.out, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    if (energyL) *energyL = h[0];
    if (energyM) *energyM = h[1];
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_marginalize_frame(ldso_b200_ctx *c, int frame_idx, int *new_dim) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    if (frame_idx < 0 || frame_idx >= c->nF) return c->fail(LDSO_B200_ERR_ARG, "frame index out of range");
    if (c->nF < 2) return c->fail(LDSO_B200_ERR_STATE, "cannot marginalise the only frame");
    if (c->prior_dim != 0 && c->prior_dim != c->n) return c->fail(LDSO_B200_ERR_STATE, "prior dimension does not match the frames: call set_frames first");
    cudaSetDevice(c->device);
    const int n = c->n;
    if (c->prior_dim == 0) {     // an all-zero prior of the current dimension
        CUDA_CHECK_RET(c, cudaMemsetAsync(c->sb.HM, 0, sizeof(double) * n * n, c->stream));
        CUDA_CHECK_RET(c, cudaMemsetAsync(c->sb.bM, 0, sizeof(double) * n, c->stream));
    }
    k_marginalize_frame<<<1, KMF_THREADS, KMF_SMEM_BYTES(n), c->stream>>>(c->sb, c->ws_dev, n, frame_idx);
    LAUNCH_CHECK(c);
    c->prior_dim = n - 8;
    c->solve_ready = false; c->restitch_ok = false;
    if (new_dim) *new_dim = n - 8;
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- immature points
static TraceSettingsDev trace_settings(const ldso_b200_ctx *c) {
    TraceSettingsDev T;
    T.maxPixSearch = c->S.maxPixSearch; T.outlierTH = c->S.outlierTH; T.outlierTHSumComponent = c->S.outlierTHSumComponent;
    T.huberTH = c->S.huberTH; T.overallEnergyTHWeight = c->S.overallEnergyTHWeight;
    T.minTraceTestRadius = c->S.minTraceTestRadius; T.trace_GNIterations = c->S.trace_GNIterations;
    T.trace_stepsize = c->S.trace_stepsize; T.trace_GNThreshold = c->S.trace_GNThreshold;
    T.trace_extraSlackOnTH = c->S.trace_extraSlackOnTH; T.trace_slackInterval = c->S.trace_slackInterval;
    T.trace_minImprovementFactor = c->S.trace_minImprovementFactor;
    return T;
}

extern "C" int ldso_b200_immature_init(ldso_b200_ctx *c, int host_slot, int n, const float *u, const float *v, float *color8,
                                       float *weights8, float *gradH4, float *energyTH) {
    if (!c || n < 0 || (n > 0 && (!u || !v || !color8 || !weights8 || !gradH4 || !energyTH))) return LDSO_B200_ERR_ARG;
    if (host_slot < 0 || host_slot >= NSLOTS || !c->img[host_slot][0]) return c->fail(LDSO_B200_ERR_ARG, "host image slot not uploaded");
    if (n == 0) return LDSO_B200_OK;
    cudaSetDevice(c->device);
    const size_t N = (size_t) n;
    ImmInitScratch s;
    RET_IF(trace_carve(c, [&](Arena &A) { immature_init_regions(A, N, s); }));
    H2D(s.u, u, 4 * N);
    H2D(s.v, v, 4 * N);
    CUDA_CHECK_RET(c, cudaMemsetAsync(s.color8, 0, sizeof(float) * N * 21, c->stream));      // the outputs' region
    launch_immature_init(n, c->img[host_slot][0], c->w, s.u, s.v, trace_settings(c), s.color8, s.weights8, s.gradH4, s.energyTH, c->stream);
    LAUNCH_CHECK(c);
    D2H(color8, s.color8, 32 * N); D2H(weights8, s.weights8, 32 * N); D2H(gradH4, s.gradH4, 16 * N); D2H(energyTH, s.energyTH, 4 * N);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_trace_immature(ldso_b200_ctx *c, int new_slot, const ldso_b200_immature *p, int n_hosts, const float *KRKi9,
                                        const float *Kt3, const float *aff2) {
    if (!c || !p || !KRKi9 || !Kt3 || !aff2 || n_hosts < 1) return LDSO_B200_ERR_ARG;
    if (new_slot < 0 || new_slot >= NSLOTS || !c->img[new_slot][0]) return c->fail(LDSO_B200_ERR_ARG, "image slot of the traced frame not uploaded");
    const int n = p->n;
    if (n < 0) return c->fail(LDSO_B200_ERR_ARG, "negative candidate count");
    if (n == 0) return LDSO_B200_OK;
    if (!p->u || !p->v || !p->host || !p->color8 || !p->weights8 || !p->gradH4 || !p->energyTH || !p->idepth_min || !p->idepth_max ||
        !p->quality || !p->lastTraceStatus || !p->lastTraceUV2 || !p->lastTracePixelInterval) return c->fail(LDSO_B200_ERR_ARG, "null candidate array");
    for (int i = 0; i < n; i++) if (p->host[i] < 0 || p->host[i] >= n_hosts) return c->fail(LDSO_B200_ERR_ARG, "candidate host index out of range");
    cudaSetDevice(c->device);
    const size_t N = (size_t) n, H = (size_t) n_hosts;
    TraceArgs A;
    RET_IF(trace_carve(c, [&](Arena &R) { trace_immature_regions(R, N, H, A); }));
    A.n = n; A.w = c->w; A.h = c->h; A.img = c->img[new_slot][0]; A.S = trace_settings(c);
    H2D(A.u, p->u, 4 * N); H2D(A.v, p->v, 4 * N); H2D(A.color8, p->color8, 32 * N); H2D(A.weights8, p->weights8, 32 * N);
    H2D(A.gradH4, p->gradH4, 16 * N); H2D(A.energyTH, p->energyTH, 4 * N); H2D(A.idepth_min, p->idepth_min, 4 * N); H2D(A.idepth_max, p->idepth_max, 4 * N);
    H2D(A.quality, p->quality, 4 * N); H2D(A.uv2, p->lastTraceUV2, 8 * N); H2D(A.interval, p->lastTracePixelInterval, 4 * N);
    H2D(A.host, p->host, 4 * N); H2D(A.status, p->lastTraceStatus, 4 * N);
    H2D(A.KRKi9, KRKi9, 36 * H); H2D(A.Kt3, Kt3, 12 * H); H2D(A.aff2, aff2, 8 * H);
    launch_trace_on(A, c->stream);
    LAUNCH_CHECK(c);
    D2H(p->idepth_min, A.idepth_min, 4 * N); D2H(p->idepth_max, A.idepth_max, 4 * N); D2H(p->quality, A.quality, 4 * N); D2H(p->lastTraceStatus, A.status, 4 * N);
    D2H(p->lastTraceUV2, A.uv2, 8 * N); D2H(p->lastTracePixelInterval, A.interval, 4 * N);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_optimize_immature(ldso_b200_ctx *c, int n, const float *u, const float *v, const int32_t *host, const float *idepth_min,
                                           const float *idepth_max, const float *color8, const float *weights8, const float *energyTH,
                                           int min_obs, int32_t *ok, float *idepth, uint8_t *res_state) {
    if (!c || n < 0) return LDSO_B200_ERR_ARG;
    if (!c->have_frames) return c->fail(LDSO_B200_ERR_STATE, "optimize_immature needs set_frames first");
    if (n == 0) return LDSO_B200_OK;
    if (!u || !v || !host || !idepth_min || !idepth_max || !color8 || !weights8 || !energyTH || !ok || !idepth || !res_state)
        return c->fail(LDSO_B200_ERR_ARG, "null candidate array");
    const int nF = c->nF;
    if (nF < 2) return c->fail(LDSO_B200_ERR_STATE, "optimize_immature needs at least two frames");
    for (int i = 0; i < n; i++) if (host[i] < 0 || host[i] >= nF) return c->fail(LDSO_B200_ERR_ARG, "candidate host index out of range");
    cudaSetDevice(c->device);
    const size_t N = (size_t) n;
    OptImmScratch s;
    RET_IF(trace_carve(c, [&](Arena &A) { optimize_immature_regions(A, N, nF, s); }));
    H2D(s.u, u, 4 * N); H2D(s.v, v, 4 * N); H2D(s.idmin, idepth_min, 4 * N); H2D(s.idmax, idepth_max, 4 * N); H2D(s.color8, color8, 32 * N);
    H2D(s.weights8, weights8, 32 * N); H2D(s.energyTH, energyTH, 4 * N); H2D(s.host, host, 4 * N);
    launch_optimize_immature(n, c->ws_dev, s.u, s.v, s.host, s.idmin, s.idmax, s.color8, s.weights8, s.energyTH, min_obs, s.ok, s.idepth, s.res_state,
                             c->stream);
    LAUNCH_CHECK(c);
    D2H(ok, s.ok, 4 * N); D2H(idepth, s.idepth, 4 * N); D2H(res_state, s.res_state, N * nF);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

// FullSystem::activatePointsMT's selection (FullSystem.cc:1076-1150): distance map of the window's points in the newest keyframe,
// then the greedy pass over the candidates. One kernel, one CTA (the pass is order-dependent by construction).
extern "C" int ldso_b200_select_activation(ldso_b200_ctx *c, int newest_frame, float current_min_act_dist, float min_trace_quality, int n,
                                           const float *u, const float *v, const int32_t *host, const float *idepth_min, const float *idepth_max,
                                           const int32_t *lastTraceStatus, const float *lastTracePixelInterval, const float *quality,
                                           const float *my_type, const uint8_t *frame_flagged, uint8_t *action, float *dist_map) {
    if (!c || n < 0) return LDSO_B200_ERR_ARG;
    if (!c->have_frames || !c->have_window) return c->fail(LDSO_B200_ERR_STATE, "select_activation needs set_frames and set_window first");
    const int nF = c->nF;
    if (newest_frame < 0 || newest_frame >= nF) return c->fail(LDSO_B200_ERR_ARG, "newest_frame out of range");
    if (n > 0 && (!u || !v || !host || !idepth_min || !idepth_max || !lastTraceStatus || !lastTracePixelInterval || !quality || !my_type || !action))
        return c->fail(LDSO_B200_ERR_ARG, "null candidate array");
    if (!frame_flagged) return c->fail(LDSO_B200_ERR_ARG, "frame_flagged must hold one byte per frame");
    for (int i = 0; i < n; i++) if (host[i] < 0 || host[i] >= nF || host[i] == newest_frame) return c->fail(LDSO_B200_ERR_ARG, "candidate host must be a window frame other than the newest");
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    const int w1 = c->w >> 1, h1 = c->h >> 1;
    const size_t N = (size_t) std::max(n, 1), cells = (size_t) w1 * h1;
    ActSelArgs A;
    RET_IF(trace_carve(c, [&](Arena &R) { actsel_regions(R, c->w, c->h, N, A); }));
    const size_t map_bytes = A.map_bytes;
    A.ws = c->ws_dev; A.newest = newest_frame; A.w1 = w1; A.h1 = h1;
    A.nP = c->d.nP; A.pt_host = c->d.pt_host; A.pt_u = c->d.pt_u; A.pt_v = c->d.pt_v; A.pt_idepth = c->d.pt_idepth;
    A.n = n;
    A.currentMinActDist = current_min_act_dist; A.minTraceQuality = min_trace_quality;
    // the kernel also has a global-memory map path (use_smem = 0) for larger images; it has not been exercised on hardware yet, so
    // larger images are refused rather than served by an unvalidated path (level 1 of 1240x376 needs 114 KB)
    if (map_bytes > 200 * 1024) return c->fail(LDSO_B200_ERR_ARG, "select_activation: level-1 image larger than 200 KB (one byte per pixel must fit in shared memory)");
    A.use_smem = 1;
    // the candidates and the frame flags travel through a pinned stage laid out like the device's inputs (actsel_inputs)
    ActSelArgs S;
    Arena P;
    actsel_stage_regions(P, N, S);
    RET_IF(scratch_reserve(c, c->actsel_pin, c->actsel_pin_cap, P.off, true));
    P = Arena(c->actsel_pin);
    actsel_stage_regions(P, N, S);
    {
        const struct { const void *dst, *src; } in[] = {{S.u, u}, {S.v, v}, {S.idmin, idepth_min}, {S.idmax, idepth_max}, {S.quality, quality},
                                                        {S.interval, lastTracePixelInterval}, {S.my_type, my_type}, {S.status, lastTraceStatus}, {S.host, host}};
        if (n > 0) for (const auto &x : in) memcpy((void *) x.dst, x.src, 4 * (size_t) n);
        H2D(A.u, S.u, 36 * N);      // the nine arrays are one region
        memcpy((void *) S.flagged, frame_flagged, (size_t) nF);
        H2D(A.flagged, S.flagged, (size_t) nF);
    }
    if (!c->ktime) A.dbg = nullptr;
    c->kt_begin("actsel");
    launch_activation_select(A, c->stream);
    c->kt_end();
    LAUNCH_CHECK(c);
    if (n > 0) D2H(S.action, A.action, (size_t) n);
    if (dist_map) {
        c->h_scratch_bytes.resize(map_bytes);
        D2H(c->h_scratch_bytes.data(), A.map, map_bytes);
    }
    long long stamps[4] = {0, 0, 0, 0};
    if (A.dbg) D2H(stamps, A.dbg, sizeof(stamps));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    if (n > 0) memcpy(action, S.action, (size_t) n);
    if (A.dbg) fprintf(stderr, "[ldso_b200 actsel] cycles: map+seeds+grow %lld, candidate terms %lld, sequential pass %lld\n", stamps[1] - stamps[0],
                       stamps[2] - stamps[1], stamps[3] - stamps[2]);
    if (dist_map) for (size_t i = 0; i < cells; i++) dist_map[i] = c->h_scratch_bytes[i] == 255 ? 1000.f : (float) c->h_scratch_bytes[i];   // fwdWarpedIDDistFinal's values
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- immature-point store
static cudaError_t imm_copy_segment(const ImmSeg &d, const ImmSeg &s, size_t n, cudaStream_t st) {
    const struct { void *dst; const void *src; size_t words; } f[] = {
        {d.u, s.u, 1}, {d.v, s.v, 1}, {d.my_type, s.my_type, 1}, {d.color8, s.color8, 8}, {d.weights8, s.weights8, 8}, {d.gradH4, s.gradH4, 4},
        {d.energyTH, s.energyTH, 1}, {d.idmin, s.idmin, 1}, {d.idmax, s.idmax, 1}, {d.quality, s.quality, 1}, {d.status, s.status, 1},
        {d.uv2, s.uv2, 2}, {d.interval, s.interval, 1}, {d.live, s.live, 1}};
    size_t words = 0;
    for (const auto &x : f) words += x.words;
    if (words != IMM_SEG_WORDS) return cudaErrorInvalidValue;       // a field of imm_seg missing here
    for (const auto &x : f) {
        const cudaError_t e = cudaMemcpyAsync(x.dst, x.src, 4 * x.words * n, cudaMemcpyDeviceToDevice, st);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}
// grows the store to at least cap entries per segment; every segment keeps its entries (live or released), copied to the new stride
static int imm_reserve(ldso_b200_ctx *c, int cap) {
    if (cap <= c->imm_cap) return LDSO_B200_OK;
    StoreActArgs P;
    ActSelArgs A;
    Arena S, H;
    imm_scratch_regions(S, cap, c->w, c->h, P, A);
    imm_pin_regions(H, cap);
    float *store = nullptr;
    char *scratch = nullptr, *pin = nullptr;
    cudaError_t e = cudaMalloc(&store, sizeof(float) * IMM_SEG_WORDS * (size_t) cap * NSLOTS);
    if (e == cudaSuccess) e = cudaMalloc(&scratch, S.off);
    if (e == cudaSuccess) e = cudaMallocHost(&pin, H.off);
    for (int s = 0; s < NSLOTS && e == cudaSuccess; s++)
        if (c->imm_n[s] > 0) e = imm_copy_segment(imm_seg(store, cap, s), imm_seg(c->imm_store, c->imm_cap, s), (size_t) c->imm_n[s], c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) {
        if (store) cudaFree(store);
        if (scratch) cudaFree(scratch);
        if (pin) cudaFreeHost(pin);
        return c->fail_cuda(e, "immature store growth", __FILE__, __LINE__);
    }
    if (c->imm_store) cudaFree(c->imm_store);
    if (c->imm_scratch) cudaFree(c->imm_scratch);
    if (c->imm_pin) cudaFreeHost(c->imm_pin);
    c->imm_store = store; c->imm_scratch = scratch; c->imm_pin = pin; c->imm_cap = cap;
    return LDSO_B200_OK;
}
#define IMM_SINGLE(c, what) do { if ((c)->multi) return (c)->fail(LDSO_B200_ERR_STATE, what " runs on a single, unsharded context"); } while (0)

extern "C" int ldso_b200_make_new_traces(ldso_b200_ctx *c, int slot, int nFeatures, const float *B, ldso_b200_features *out) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "make_new_traces");
    CornerGrid g;
    if (!corner_grid(c->w, c->h, nFeatures, g))
        return c->fail(LDSO_B200_ERR_ARG, "make_new_traces: nFeatures must be positive and give a grid whose patches stay inside the image");
    CornerArgs a;
    RET_IF(corners_launch(c, slot, nFeatures, B, out, a));
    const int need = std::max(1, g.ncx * g.ncy * g.kcap);
    if (need > c->imm_cap)          // the density fixes the store's capacity: it may change only while nothing is live
        for (int s = 0; s < NSLOTS; s++)
            if (c->imm_live[s]) return c->fail(LDSO_B200_ERR_STATE, "make_new_traces: a density with a larger capacity while entries are live");
    RET_IF(imm_reserve(c, need));
    c->imm_n[slot] = c->imm_live[slot] = 0;
    if (a.cap > 0) {                // a grid without cells: detect_corners returns no features, and the segment stays empty
        launch_store_seed(a.hdr, a.cap, a.u, a.v, nullptr, c->img[slot][0], c->w, trace_settings(c), c->imm_store, c->imm_cap, slot, c->stream);
        LAUNCH_CHECK(c);
    }
    RET_IF(corners_read(c, a, out));
    c->imm_n[slot] = c->imm_live[slot] = out->n;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_immature_seed(ldso_b200_ctx *c, int slot, int n, const float *u, const float *v, const float *my_type) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "immature_seed");
    if (slot < 0 || slot >= NSLOTS || !c->img[slot][0]) return c->fail(LDSO_B200_ERR_ARG, "immature_seed: image slot out of range or never filled");
    if (n < 0 || (n > 0 && (!u || !v))) return c->fail(LDSO_B200_ERR_ARG, "immature_seed: negative count or missing coordinates");
    for (int i = 0; i < n; i++)
        if (!(u[i] >= 2 && u[i] < c->w - 3 && v[i] >= 2 && v[i] < c->h - 3))
            return c->fail(LDSO_B200_ERR_ARG, "immature_seed: a candidate's pattern leaves the image");
    cudaSetDevice(c->device);
    RET_IF(imm_reserve(c, n));
    c->imm_live[slot] = 0;
    c->imm_n[slot] = 0;
    if (n == 0) return LDSO_B200_OK;
    const ImmSeg g = imm_seg(c->imm_store, c->imm_cap, slot);
    Arena H(c->imm_pin);
    float *hp = (float *) imm_pin_regions(H, c->imm_cap).body;      // u, v, my_type: n each
    const size_t N = (size_t) n;
    memcpy(hp, u, 4 * N); memcpy(hp + N, v, 4 * N);
    if (my_type) memcpy(hp + 2 * N, my_type, 4 * N);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(g.u, hp, 4 * N, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(c, cudaMemcpyAsync(g.v, hp + N, 4 * N, cudaMemcpyHostToDevice, c->stream));
    if (my_type) CUDA_CHECK_RET(c, cudaMemcpyAsync(g.my_type, hp + 2 * N, 4 * N, cudaMemcpyHostToDevice, c->stream));
    launch_store_seed(nullptr, n, g.u, g.v, my_type ? g.my_type : nullptr, c->img[slot][0], c->w, trace_settings(c), c->imm_store, c->imm_cap,
                      slot, c->stream);
    LAUNCH_CHECK(c);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    c->imm_n[slot] = c->imm_live[slot] = n;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_make_new_traces_pixels(ldso_b200_ctx *c, int slot, const ldso_b200_pixsel_params *params, const float *B,
                                                int *current_potential, ldso_b200_pixel_traces *out) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "make_new_traces_pixels");
    if (!out || !out->u || !out->v || !out->my_type) return c->fail(LDSO_B200_ERR_ARG, "make_new_traces_pixels: missing output array");
    PixselArgs a;
    PixselResult R;
    RET_IF(pixsel_run(c, "make_new_traces_pixels", slot, params, B, current_potential, true, a, R));
    if (out->capacity < R.nkept) return c->fail(LDSO_B200_ERR_ARG, "make_new_traces_pixels: capacity below the number of selected pixels");
    const int nf = R.nfeat;
    RET_IF(imm_reserve(c, nf));
    c->imm_n[slot] = c->imm_live[slot] = 0;
    int n = 0;
    if (nf > 0) {
        // the constructor for every pixel in range, then the entries whose energyTH is not finite leave the segment
        launch_store_seed(nullptr, nf, a.fu, a.fv, a.ftype, c->img[slot][0], c->w, trace_settings(c), c->imm_store, c->imm_cap, slot, c->stream);
        LAUNCH_CHECK(c);
        launch_store_compact(c->imm_store, c->imm_cap, slot, nf, a.hdr + PIXSEL_NSEED, c->stream);
        LAUNCH_CHECK(c);
        const ImmSeg g = imm_seg(c->imm_store, c->imm_cap, slot);
        const size_t N = (size_t) nf;
        PixselArgs h;
        Arena P(c->pix_pin);
        pixsel_pin_regions(P, N, (size_t) c->w * c->h, true, h);
        D2H(h.hdr, a.hdr, 4 * PIXSEL_HDR_INTS);
        D2H(h.fu, g.u, 4 * N);
        D2H(h.fv, g.v, 4 * N);
        D2H(h.ftype, g.my_type, 4 * N);
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        n = h.hdr[PIXSEL_NSEED];
        memcpy(out->u, h.fu, 4 * (size_t) n);
        memcpy(out->v, h.fv, 4 * (size_t) n);
        memcpy(out->my_type, h.ftype, 4 * (size_t) n);
    }
    c->imm_n[slot] = c->imm_live[slot] = n;
    out->n_selected = R.nkept; out->n = n;
    *current_potential = R.pot;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_trace_new_coarse(ldso_b200_ctx *c, int new_slot, int n_hosts, const int32_t *host_slots, const float *KRKi9,
                                          const float *Kt3, const float *aff2, int32_t counts7[7]) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "trace_new_coarse");
    if (new_slot < 0 || new_slot >= NSLOTS || !c->img[new_slot][0]) return c->fail(LDSO_B200_ERR_ARG, "trace_new_coarse: image slot of the traced frame not filled");
    if (n_hosts < 0 || n_hosts > NSLOTS || (n_hosts > 0 && (!host_slots || !KRKi9 || !Kt3 || !aff2)))
        return c->fail(LDSO_B200_ERR_ARG, "trace_new_coarse: bad host list");
    StoreTraceArgs P;
    P.nseg = n_hosts;
    P.begin[0] = 0;
    for (int j = 0; j < n_hosts; j++) {
        const int s = host_slots[j];
        if (s < 0 || s >= NSLOTS) return c->fail(LDSO_B200_ERR_ARG, "trace_new_coarse: host slot out of range");
        for (int q = 0; q < j; q++) if (host_slots[q] == s) return c->fail(LDSO_B200_ERR_ARG, "trace_new_coarse: host slot listed twice");
        P.slot[j] = s;
        P.begin[j + 1] = P.begin[j] + (c->imm_live[s] ? c->imm_n[s] : 0);
        memcpy(P.KRKi[j], KRKi9 + 9 * j, sizeof(float) * 9); memcpy(P.Kt[j], Kt3 + 3 * j, sizeof(float) * 3); memcpy(P.aff[j], aff2 + 2 * j, sizeof(float) * 2);
    }
    if (counts7) memset(counts7, 0, sizeof(int32_t) * 7);
    if (P.begin[n_hosts] == 0) return LDSO_B200_OK;
    cudaSetDevice(c->device);
    memset(&P.T, 0, sizeof(P.T));
    P.T.w = c->w; P.T.h = c->h; P.T.img = c->img[new_slot][0]; P.T.S = trace_settings(c);
    P.store = c->imm_store; P.cap = c->imm_cap;
    StoreActArgs act;      // activate_immature's regions: only the counters are used here
    ActSelArgs sel;
    Arena D(c->imm_scratch), H(c->imm_pin);
    const ImmSmall small = imm_scratch_regions(D, c->imm_cap, c->w, c->h, act, sel);
    P.counts = counts7 ? small.counts : nullptr;
    if (P.counts) CUDA_CHECK_RET(c, cudaMemsetAsync(P.counts, 0, sizeof(int) * 7, c->stream));
    launch_store_trace(P, c->stream);
    LAUNCH_CHECK(c);
    if (counts7) {
        int *hc = imm_pin_regions(H, c->imm_cap).small.counts;
        CUDA_CHECK_RET(c, cudaMemcpyAsync(hc, P.counts, sizeof(int) * 7, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        memcpy(counts7, hc, sizeof(int32_t) * 7);
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_activate_immature(ldso_b200_ctx *c, float current_min_act_dist, float min_trace_quality, const uint8_t *frame_flagged,
                                           int min_obs, ldso_b200_activation_out *out) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "activate_immature");
    if (!c->have_frames || !c->have_window) return c->fail(LDSO_B200_ERR_STATE, "activate_immature needs set_frames and set_window first");
    if (!frame_flagged) return c->fail(LDSO_B200_ERR_ARG, "frame_flagged must hold one byte per frame");
    if (!out || !out->frame || !out->index || !out->status || !out->idepth_min || !out->idepth_max || !out->idepth || !out->color8 ||
        !out->weights8 || !out->energyTH || !out->my_type || !out->res_state) return c->fail(LDSO_B200_ERR_ARG, "activate_immature: missing output array");
    const int nF = c->nF, w1 = c->w >> 1, h1 = c->h >> 1;
    const size_t cells = (size_t) w1 * h1, map_bytes = (cells + 3) & ~(size_t) 3;
    if (map_bytes > 200 * 1024) return c->fail(LDSO_B200_ERR_ARG, "activate_immature: level-1 image larger than 200 KB (one byte per pixel must fit in shared memory)");
    StoreActArgs P;
    P.nseg = std::max(nF - 1, 0);
    P.begin[0] = 0;
    for (int f = 0; f < nF; f++) {
        P.slot[f] = c->slots[f];
        if (f < P.nseg) P.begin[f + 1] = P.begin[f] + (c->imm_live[c->slots[f]] ? c->imm_n[c->slots[f]] : 0);
    }
    int ncand = 0;
    for (int f = 0; f < P.nseg; f++) ncand += c->imm_live[c->slots[f]];
    if (out->capacity < ncand) return c->fail(LDSO_B200_ERR_ARG, "activate_immature: capacity below the number of live candidates");
    out->n = 0; out->n_valid = 0;
    if (ncand == 0) return LDSO_B200_OK;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    P.store = c->imm_store; P.cap = c->imm_cap; P.n = ncand; P.nF = nF; P.ws = c->ws_dev;
    ActSelArgs A;
    Arena D(c->imm_scratch), H(c->imm_pin);
    imm_scratch_regions(D, c->imm_cap, c->w, c->h, P, A);
    const ImmPin pin = imm_pin_regions(H, c->imm_cap);
    // candidates, selection, activation LM, bookkeeping
    launch_store_gather(P, c->stream);
    LAUNCH_CHECK(c);
    memcpy(pin.small.flags, frame_flagged, (size_t) nF);
    H2D(A.flagged, pin.small.flags, (size_t) nF);
    A.ws = c->ws_dev; A.newest = nF - 1; A.w1 = w1; A.h1 = h1;
    A.nP = c->d.nP; A.pt_host = c->d.pt_host; A.pt_u = c->d.pt_u; A.pt_v = c->d.pt_v; A.pt_idepth = c->d.pt_idepth;
    A.n = ncand;
    A.u = P.c_u; A.v = P.c_v; A.idmin = P.c_idmin; A.idmax = P.c_idmax; A.quality = P.c_quality; A.interval = P.c_interval; A.my_type = P.c_type;
    A.status = P.c_status; A.host = P.c_host;
    A.currentMinActDist = current_min_act_dist; A.minTraceQuality = min_trace_quality;
    A.action = P.action; A.use_smem = 1; A.dbg = nullptr;
    launch_activation_select(A, c->stream);
    LAUNCH_CHECK(c);
    launch_store_pick(P, c->stream);
    LAUNCH_CHECK(c);
    launch_store_optimize(P, min_obs, c->stream);
    LAUNCH_CHECK(c);
    launch_store_apply(P, c->stream);
    LAUNCH_CHECK(c);
    int *hh = pin.small.hdr;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(hh, P.hdr, sizeof(int) * 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    const int nrel = hh[1], nvalid = hh[2];
    const ImmRecord *hr = (const ImmRecord *) pin.body;
    if (nrel > 0) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync((void *) hr, P.rec, sizeof(ImmRecord) * nrel, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    }
    for (int i = 0; i < nrel; i++) {
        const ImmRecord &r = hr[i];
        out->frame[i] = r.frame; out->index[i] = r.index; out->status[i] = r.status;
        out->idepth_min[i] = r.idepth_min; out->idepth_max[i] = r.idepth_max; out->idepth[i] = r.idepth;
        out->energyTH[i] = r.energyTH; out->my_type[i] = r.my_type;
        memcpy(out->color8 + 8 * i, r.color8, sizeof(r.color8)); memcpy(out->weights8 + 8 * i, r.weights8, sizeof(r.weights8));
        memcpy(out->res_state + (size_t) nF * i, r.res_state, (size_t) nF);
        c->imm_live[c->slots[r.frame]]--;
    }
    out->n = nrel; out->n_valid = nvalid;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_immature_release(ldso_b200_ctx *c, int slot) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "immature_release");
    if (slot < 0 || slot >= NSLOTS) return c->fail(LDSO_B200_ERR_ARG, "immature_release: slot out of range");
    if (c->imm_live[slot]) {
        cudaSetDevice(c->device);
        CUDA_CHECK_RET(c, cudaMemsetAsync(imm_seg(c->imm_store, c->imm_cap, slot).live, 0, sizeof(int) * c->imm_n[slot], c->stream));
    }
    c->imm_live[slot] = 0;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_immature_read(ldso_b200_ctx *c, int slot, ldso_b200_immature_segment *out) {
    if (!c) return LDSO_B200_ERR_ARG;
    IMM_SINGLE(c, "immature_read");
    if (slot < 0 || slot >= NSLOTS) return c->fail(LDSO_B200_ERR_ARG, "immature_read: slot out of range");
    if (!out) return c->fail(LDSO_B200_ERR_ARG, "immature_read: out is NULL");
    const int n = c->imm_n[slot];
    if (out->capacity < n) return c->fail(LDSO_B200_ERR_ARG, "immature_read: capacity below the segment's entry count");
    if (n > 0 && (!out->u || !out->v || !out->my_type || !out->color8 || !out->weights8 || !out->gradH4 || !out->energyTH || !out->idepth_min ||
                  !out->idepth_max || !out->quality || !out->lastTraceStatus || !out->lastTraceUV2 || !out->lastTracePixelInterval || !out->live))
        return c->fail(LDSO_B200_ERR_ARG, "immature_read: missing output array");
    out->n = n;
    if (n == 0) return LDSO_B200_OK;
    cudaSetDevice(c->device);
    const size_t cap = c->imm_cap, N = n;
    Arena H(c->imm_pin);
    float *hp = (float *) imm_pin_regions(H, c->imm_cap).body;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(hp, imm_seg(c->imm_store, c->imm_cap, slot).u, sizeof(float) * IMM_SEG_WORDS * cap, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    const ImmSeg g = imm_seg(hp, c->imm_cap, 0);      // the segment's layout, at the staging copy
    memcpy(out->u, g.u, 4 * N); memcpy(out->v, g.v, 4 * N); memcpy(out->my_type, g.my_type, 4 * N);
    memcpy(out->color8, g.color8, 32 * N); memcpy(out->weights8, g.weights8, 32 * N); memcpy(out->gradH4, g.gradH4, 16 * N);
    memcpy(out->energyTH, g.energyTH, 4 * N); memcpy(out->idepth_min, g.idmin, 4 * N); memcpy(out->idepth_max, g.idmax, 4 * N);
    memcpy(out->quality, g.quality, 4 * N); memcpy(out->lastTraceStatus, g.status, 4 * N); memcpy(out->lastTraceUV2, g.uv2, 8 * N);
    memcpy(out->lastTracePixelInterval, g.interval, 4 * N);
    for (int i = 0; i < n; i++) out->live[i] = g.live[i] != 0;
    return LDSO_B200_OK;
}

// CoarseInitializer::calcResAndGS (src/frontend/CoarseInitializer.cc:181-405) for the points of one pyramid level. EXPERIMENTAL: written
// at the end of round 1 against the pinned oracle (oracle/initializer.cc), compiled, NOT yet run on hardware (tests/test_gpu_init.py is
// skipped unless LDSO_B200_RUN_UNVALIDATED is set).
extern "C" int ldso_b200_init_calc_res(ldso_b200_ctx *c, int first_slot, int new_slot, int lvl, const double R[9], const double t[3], const double tlog3[3],
                                       float aff_a, float aff_b, float fx0, float fy0, float cx0, float cy0, int n, const float *u, const float *v,
                                       const float *idepth_new, const float *iR, const uint8_t *isGood, const float *energy2, const float *outlierTH,
                                       float alphaK, float alphaW, float couplingWeight, uint8_t *isGood_new, float *energy_new2, float *maxstep,
                                       float *lastHessian_new, float *JbBuffer_new10, float *H64, float *b8, float *Hsc64, float *bsc8, float *res3) {
    if (!c || n <= 0 || !R || !t || !tlog3) return LDSO_B200_ERR_ARG;
    if (lvl < 0 || lvl >= c->levels) return c->fail(LDSO_B200_ERR_ARG, "pyramid level out of range");
    if (first_slot < 0 || first_slot >= NSLOTS || new_slot < 0 || new_slot >= NSLOTS || !c->img[first_slot][lvl] || !c->img[new_slot][lvl])
        return c->fail(LDSO_B200_ERR_ARG, "image slot not uploaded");
    if (!u || !v || !idepth_new || !iR || !isGood || !energy2 || !outlierTH || !isGood_new || !energy_new2 || !maxstep || !lastHessian_new ||
        !JbBuffer_new10 || !H64 || !b8 || !Hsc64 || !bsc8 || !res3) return c->fail(LDSO_B200_ERR_ARG, "null array");
    const int wl = c->w >> lvl, hl = c->h >> lvl;
    for (int i = 0; i < n; i++)      // the reference samples the first frame at (u + dx, v + dy) without a bounds check (its selector keeps a margin)
        if (!(u[i] >= 2 && v[i] >= 2 && u[i] < wl - 3 && v[i] < hl - 3)) return c->fail(LDSO_B200_ERR_ARG, "initializer point closer than the pattern radius to the image border");
    cudaSetDevice(c->device);
    // CoarseInitializer::makeK (:689-715) in double, K^-1 by Eigen's 3x3 cofactor formula
    double fx = fx0, fy = fy0, cx = cx0, cy = cy0;
    for (int level = 1; level <= lvl; ++level) { fx = fx * 0.5; fy = fy * 0.5; }
    if (lvl > 0) { cx = ((double) cx0 + 0.5) / ((int) 1 << lvl) - 0.5; cy = ((double) cy0 + 0.5) / ((int) 1 << lvl) - 0.5; }
    const double K[9] = {fx, 0, cx, 0, fy, cy, 0, 0, 1};
    double Ki[9];
    {
        const double c00 = K[4] * K[8] - K[5] * K[7], c01 = K[5] * K[6] - K[3] * K[8], c02 = K[3] * K[7] - K[4] * K[6];
        const double det = K[0] * c00 + K[1] * c01 + K[2] * c02, invdet = 1.0 / det;
        Ki[0] = c00 * invdet; Ki[3] = c01 * invdet; Ki[6] = c02 * invdet;
        Ki[1] = (K[2] * K[7] - K[1] * K[8]) * invdet; Ki[4] = (K[0] * K[8] - K[2] * K[6]) * invdet; Ki[7] = (K[1] * K[6] - K[0] * K[7]) * invdet;
        Ki[2] = (K[1] * K[5] - K[2] * K[4]) * invdet; Ki[5] = (K[2] * K[3] - K[0] * K[5]) * invdet; Ki[8] = (K[0] * K[4] - K[1] * K[3]) * invdet;
    }
    InitArgs A;
    A.n = n; A.w = wl; A.h = hl;
    A.imgRef = c->img[first_slot][lvl]; A.imgNew = c->img[new_slot][lvl];
    for (int i = 0; i < 3; i++) {
        for (int j = 0; j < 3; j++) { double s = R[i * 3] * Ki[j]; s += R[i * 3 + 1] * Ki[3 + j]; s += R[i * 3 + 2] * Ki[6 + j]; A.RKi[i * 3 + j] = (float) s; }
        A.t[i] = (float) t[i];
    }
    A.aff0 = std::exp(aff_a); A.aff1 = aff_b;
    A.fx = (float) fx; A.fy = (float) fy; A.cx = (float) cx; A.cy = (float) cy; A.huberTH = c->S.huberTH;
    // alpha energy (:336-356): the reference's EAlpha accumulator never receives a term, so it depends on the translation only
    const double tsq = t[0] * t[0] + t[1] * t[1] + t[2] * t[2];
    float alphaEnergy = (float) ((double) alphaW * ((double) 0.0f + tsq * n));
    float alphaOpt;
    if (alphaEnergy > alphaK * n) { alphaOpt = 0; alphaEnergy = alphaK * n; } else alphaOpt = alphaW;
    A.alphaOpt = alphaOpt; A.couplingWeight = couplingWeight;
    const size_t N = (size_t) n, grid = (N + INIT_THREADS / 8 - 1) / (INIT_THREADS / 8);
    RET_IF(trace_carve(c, [&](Arena &R) { init_calc_res_regions(R, N, grid, A); }));
    H2D(A.u, u, 4 * N); H2D(A.v, v, 4 * N); H2D(A.idepth_new, idepth_new, 4 * N); H2D(A.iR, iR, 4 * N); H2D(A.energy2, energy2, 8 * N);
    H2D(A.outlierTH, outlierTH, 4 * N); H2D(A.isGood, isGood, N);
    CUDA_CHECK_RET(c, cudaMemsetAsync(A.energy_new2, 0, 4 * (size_t) (2 + 1 + 1 + 10) * N, c->stream));      // energy_new, maxstep, lastHessian_new, Jb
    CUDA_CHECK_RET(c, cudaMemsetAsync(A.counter, 0, 16, c->stream));
    launch_init_calc_res(A, c->stream);
    LAUNCH_CHECK(c);
    double sums[INIT_NACC];
    D2H(isGood_new, A.isGood_new, N); D2H(energy_new2, A.energy_new2, 8 * N); D2H(maxstep, A.maxstep, 4 * N); D2H(lastHessian_new, A.lastHessian_new, 4 * N);
    D2H(JbBuffer_new10, A.Jb, 40 * N);
    D2H(sums, A.out, sizeof(sums));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    // acc9.H / acc9SC.H -> H_out, b_out, H_out_sc, b_out_sc (:390-403)
    int k = 0;
    for (int r = 0; r < 9; r++)
        for (int cc = r; cc < 9; cc++, k++) {
            const float hv = (float) sums[k], sv = (float) sums[45 + k];
            if (cc < 8) { H64[r * 8 + cc] = H64[cc * 8 + r] = hv; Hsc64[r * 8 + cc] = Hsc64[cc * 8 + r] = sv; }
            else if (r < 8) { b8[r] = hv; bsc8[r] = sv; }
        }
    for (int i = 0; i < 3; i++) { H64[i * 8 + i] += alphaOpt * n; b8[i] += (float) tlog3[i] * alphaOpt * n; }
    res3[0] = (float) sums[90]; res3[1] = alphaEnergy; res3[2] = (float) (2 * n);      // E.num counts both loops (:211-303 and :339-347)
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- fused loop
static const int K1_FUSED = K1F_LINEARIZE | K1F_ACCUMULATE | K1F_APPLY_RES;

extern "C" int ldso_b200_optimize_begin(ldso_b200_ctx *c, double *energy_out) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(check_solve_frames(c));
    RET_IF(clear_select(c));
    RET_IF(launch_k1(c, K1_FUSED | K1F_RESET_OOB));
    RET_IF(launch_k2a(c, 1));
    if (c->multi && !c->peers_connected) return LDSO_B200_OK;     // caller all-reduces, then gn_phase_b
    if (c->peers_connected) RET_IF(launch_k2r(c));
    RET_IF(launch_k2b(c, 1, 1, 1));
    if (energy_out) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(energy_out, &c->ws_dev->energy, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    }
    return LDSO_B200_OK;
}

// One fused Gauss-Newton iteration: K3 (solve + step, and -- second CTA -- the energy-threshold select of the PREVIOUS linearisation)
// -> K1 -> K2a -> [K2r] -> K2b (stitch + assemble). The select of the linearisation this body ends with stays pending: the next
// body's K3 runs it, or flush_select() when something else needs the threshold first.
static int launch_gn_body(ldso_b200_ctx *c) {
    struct Scope { ldso_b200_ctx *c; Scope(ldso_b200_ctx *c_) : c(c_) { c->pdl_now = true; } ~Scope() { c->pdl_now = false; } } scope(c);
    RET_IF(launch_k3(c, K3F_BACKUP | K3F_SOLVE | K3F_STEP | K3F_SELECT));
    RET_IF(launch_k1(c, K1_FUSED | K1F_APPLY_STEP));
    RET_IF(launch_k2a(c, 1));
    if (c->peers_connected) RET_IF(launch_k2r(c));
    RET_IF(launch_k2b(c, 1, 0, 1));
    c->select_pending = true;
    return LDSO_B200_OK;
}
static int flush_select(ldso_b200_ctx *c) {
    if (!c->select_pending) return LDSO_B200_OK;
    c->select_pending = false;
    const bool sr = c->solve_ready;
    RET_IF(launch_k2b(c, 0, 1, 0));
    c->solve_ready = sr;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_gn_iterations(ldso_b200_ctx *c, int first_iteration, int n_iterations) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (c->multi && !c->peers_connected) return c->fail(LDSO_B200_ERR_STATE, "sharded context without peer exchange: use gn_phase_a / all-reduce / gn_phase_b, or peer_export + peer_connect");
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(check_solve_frames(c));
    RET_IF(ensure_solve_ready(c));
    RET_IF(set_iteration(c, first_iteration));     // K3 reads the iteration number from device memory and increments it
    if (c->use_graph && c->d.nItems > 0) {
        if (!c->gn_graph_valid) {
            if (c->gn_graph) { cudaGraphExecDestroy(c->gn_graph); c->gn_graph = nullptr; }
            cudaGraph_t g = nullptr;
            if (cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) {
                // e.g. the legacy default stream cannot be captured: run the plain launches instead
                cudaGetLastError();
                c->use_graph = false;
                for (int i = 0; i < n_iterations; i++) RET_IF(launch_gn_body(c));
                return LDSO_B200_OK;
            }
            const long long l0 = c->launches;
            int rc = launch_gn_body(c);
            cudaError_t e = cudaStreamEndCapture(c->stream, &g);
            c->launches = l0;
            if (rc == 0 && e == cudaSuccess) {
                e = cudaGraphInstantiate(&c->gn_graph, g, 0);
                if (e != cudaSuccess) c->gn_graph = nullptr;
            }
            if (g) cudaGraphDestroy(g);
            if (rc || e != cudaSuccess) {
                cudaGetLastError();
                if (c->use_pdl) {        // programmatic edges not capturable here: same graph with full dependencies
                    c->use_pdl = false;
                    return ldso_b200_gn_iterations(c, first_iteration, n_iterations);
                }
                if (rc) return rc;
                return c->fail_cuda(e, "CUDA graph capture of the GN iteration", __FILE__, __LINE__);
            }
            c->gn_graph_valid = true;
        }
        for (int i = 0; i < n_iterations; i++) {
            CUDA_CHECK_RET(c, cudaGraphLaunch(c->gn_graph, c->stream));
            c->launches += c->peers_connected ? 5 : 4;
            c->select_pending = true;
            { c->mirror_valid = false; c->results_inflight = false; c->sol_valid = false; c->mirror_full_valid = false; }
        }
        return LDSO_B200_OK;
    }
    for (int i = 0; i < n_iterations; i++) RET_IF(launch_gn_body(c));
    return LDSO_B200_OK;
}

// ---- FullSystem::optimize's iteration budget and convergence exit (FullSystem.cc:727-732, :829)
extern "C" int ldso_b200_optimize_iteration_budget(int nFrames, int max_opt_iterations) {
    if (max_opt_iterations < 0) return LDSO_B200_ERR_ARG;
    if (nFrames < 2) return 0;
    if (nFrames < 4) return 15;          // the `< 3 -> 20` assignment (:729-730) is overwritten by `< 4 -> 15` (:731-732)
    return max_opt_iterations;
}

static int launch_continue(ldso_b200_ctx *c, cudaGraphConditionalHandle cond, int use_cond) {
    c->pdl_now = true;
    launch_loop_kernel(c, k_gn_continue, dim3(1), dim3(32), 0, (const WinState *) c->ws_dev, (const int *) c->iteration_dev, c->loop_dev,
                       cond, use_cond);
    c->pdl_now = false;
    LAUNCH_CHECK(c);
    return LDSO_B200_OK;
}

// One graph holding a conditional WHILE node whose body is the captured GN body + k_gn_continue. The node's condition starts at 1
// on every launch; the continue kernel clears it after the body that ends the loop. Where the driver refuses programmatic edges
// inside the body the capture is repeated with full dependencies; where it refuses conditional nodes at all, until_cond is
// cleared and gn_iterations_until runs its host-driven form from then on. Returns an error only for a launch the body itself
// rejects (the same errors gn_iterations reports).
static int capture_until_graph(ldso_b200_ctx *c) {
    if (c->until_graph) { cudaGraphExecDestroy(c->until_graph); c->until_graph = nullptr; }
    const bool pdl_saved = c->use_pdl;
    int rc_last = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
        if (attempt == 1) {
            if (!pdl_saved) break;
            c->use_pdl = false;
        }
        cudaGraph_t g = nullptr;
        cudaGraphConditionalHandle cond = 0;
        cudaGraphNode_t node = nullptr;
        cudaGraphNodeParams p = {cudaGraphNodeTypeConditional};
        int rc = 0;
        cudaError_t e = cudaGraphCreate(&g, 0);
        if (e == cudaSuccess) e = cudaGraphConditionalHandleCreate(&cond, g, 1, cudaGraphCondAssignDefault);
        if (e == cudaSuccess) {
            p.conditional.handle = cond;
            p.conditional.type = cudaGraphCondTypeWhile;
            p.conditional.size = 1;
            e = cudaGraphAddNode(&node, g, nullptr, 0, &p);
        }
        if (e == cudaSuccess) e = cudaStreamBeginCaptureToGraph(c->stream, p.conditional.phGraph_out[0], nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal);
        if (e == cudaSuccess) {
            const long long l0 = c->launches;
            rc = launch_gn_body(c);
            if (!rc) rc = launch_continue(c, cond, 1);
            cudaGraph_t body = nullptr;      // the node's own body graph, owned by g
            const cudaError_t e2 = cudaStreamEndCapture(c->stream, &body);
            c->launches = l0;
            e = e2;
        }
        if (rc == 0 && e == cudaSuccess) {
            e = cudaGraphInstantiate(&c->until_graph, g, 0);
            if (e != cudaSuccess) c->until_graph = nullptr;
        }
        if (g) cudaGraphDestroy(g);
        c->use_pdl = pdl_saved;
        if (rc == 0 && e == cudaSuccess) {
            c->until_graph_valid = true;
            c->until_graph_form = (attempt == 0 && pdl_saved) ? LDSO_B200_UNTIL_GRAPH_PDL : LDSO_B200_UNTIL_GRAPH;
            return LDSO_B200_OK;
        }
        cudaGetLastError();
        rc_last = rc;
    }
    if (rc_last) return rc_last;
    c->until_cond = false;
    return LDSO_B200_OK;
}

// bodies a WHILE-node launch ran enter launch_count once their number is known on the host
static void count_until_launches(ldso_b200_ctx *c, int bodies) {
    c->launches += (long long) bodies * c->until_launches_per_body;
    c->until_launches_per_body = 0;
}

extern "C" int ldso_b200_gn_iterations_until(ldso_b200_ctx *c, int first_iteration, int max_iterations, int min_iterations) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (max_iterations < 0) return c->fail(LDSO_B200_ERR_ARG, "negative iteration count");
    if (c->multi && !c->peers_connected) return c->fail(LDSO_B200_ERR_STATE, "sharded context without peer exchange: use gn_phase_a / all-reduce / gn_phase_b, or peer_export + peer_connect");
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(check_solve_frames(c));
    RET_IF(ensure_solve_ready(c));
    const int params[LOOP_CONT] = {max_iterations, min_iterations, 0};      // LOOP_MAX, LOOP_MIN, LOOP_RUN
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->loop_dev, params, sizeof(params), cudaMemcpyHostToDevice, c->stream));
    c->until_launches_per_body = 0;
    if (max_iterations == 0) return LDSO_B200_OK;
    RET_IF(set_iteration(c, first_iteration));
    if (c->use_graph && c->until_cond && c->d.nItems > 0) {
        if (!c->until_graph_valid) RET_IF(capture_until_graph(c));
        if (c->until_graph_valid) {
            CUDA_CHECK_RET(c, cudaGraphLaunch(c->until_graph, c->stream));
            c->until_form = c->until_graph_form;
            c->until_launches_per_body = c->peers_connected ? 6 : 5;
            c->select_pending = true;
            { c->mirror_valid = false; c->results_inflight = false; c->sol_valid = false; c->mirror_full_valid = false; }
            return LDSO_B200_OK;
        }
    }
    // host-driven: the same kernels, one synchronise per body to read the continue kernel's decision
    c->until_form = LDSO_B200_UNTIL_HOST;
    for (int i = 0; i < max_iterations; i++) {
        RET_IF(launch_gn_body(c));
        RET_IF(launch_continue(c, 0, 0));
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->loop_pin, c->loop_dev + LOOP_CONT, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        if (!*c->loop_pin) break;
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_iterations_run(ldso_b200_ctx *c, int *n) {
    if (!c || !n) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->loop_pin + LOOP_RUN, c->loop_dev + LOOP_RUN, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    *n = c->loop_pin[LOOP_RUN];
    count_until_launches(c, *n);
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_until_form(ldso_b200_ctx *c, int *form) {
    if (!c || !form) return LDSO_B200_ERR_ARG;
    *form = c->until_form;
    return LDSO_B200_OK;
}

static int wait_results(ldso_b200_ctx *c);
extern "C" int ldso_b200_prefetch_results(ldso_b200_ctx *c);
extern "C" int ldso_b200_get_points(ldso_b200_ctx *c, float *idepth, float *idepth_zero, float *step, float *HdiF, float *bdSumF, float *Hdd,
                                    float *bd, float *Hcd4);
extern "C" int ldso_b200_get_residuals(ldso_b200_ctx *c, uint8_t *state_state, uint8_t *state_NewState, float *state_energy,
                                       float *state_NewEnergy, float *state_NewEnergyWithOutlier, uint8_t *isActive, float *JpJdF8, float *J74,
                                       float *projectedTo16, float *centerProjectedTo3);
// Queue one whole FullSystem::optimize (uploads, prologue, n iterations, result read-back into pinned staging) on the context's
// stream and return WITHOUT waiting. The caller's buffers (io->image, frames, window arrays) are consumed before this returns except
// io->image, which must stay valid until the matching _wait. Two contexts fed alternately overlap one window's uploads with the
// other's kernels (bench.py's pipelined end-to-end leg); a single context just splits the call at its only synchronisation point.
// until: the loop runs with FullSystem::optimize's exit (gn_iterations_until, io->n_iterations the maximum) and the number of bodies
// it ran rides into pinned staging behind the other two scalars
static int submit_impl(ldso_b200_ctx *c, const ldso_b200_fused_io *io, bool until, int min_iterations) {
    if (!c || !io || !io->frames || !io->window || !io->calib_value_scaled || !io->calib_value_zero) return LDSO_B200_ERR_ARG;
    if (io->n_iterations < 0) return c->fail(LDSO_B200_ERR_ARG, "negative iteration count");
    // the image first: 1.2 MB over PCIe, in flight while the host packs the frame states and the window
    if (io->image) RET_IF(make_images_impl(c, io->image_slot, io->image, false));
    RET_IF(ldso_b200_set_frames(c, io->nFrames, io->frames, io->calib_value_scaled, io->calib_value_zero));
    RET_IF(ldso_b200_set_window(c, io->window));
    RET_IF(ldso_b200_optimize_begin(c, nullptr));
    if (until) RET_IF(ldso_b200_gn_iterations_until(c, io->first_iteration, io->n_iterations, min_iterations));
    else if (io->n_iterations > 0) RET_IF(ldso_b200_gn_iterations(c, io->first_iteration, io->n_iterations));
    RET_IF(ldso_b200_prefetch_results(c));
    // the scalars ride behind the prefetch into pinned staging (sol_host has MAXN spare doubles behind lastX)
    const size_t nn = (size_t) MAXN * MAXN;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sol_host + nn + 2 * MAXN, &c->ws_dev->energy, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sol_host + nn + 2 * MAXN + 1, &c->ws_dev->canbreak, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    if (until) CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sol_host + nn + 2 * MAXN + 2, c->loop_dev + LOOP_RUN, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_optimize_from_host_submit(ldso_b200_ctx *c, const ldso_b200_fused_io *io) { return submit_impl(c, io, false, 0); }

extern "C" int ldso_b200_optimize_from_host_wait(ldso_b200_ctx *c, const ldso_b200_fused_io *io) {
    if (!c || !io) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));       // one wait covers everything (and frees the caller's image buffer)
    const size_t nn = (size_t) MAXN * MAXN;
    if (io->energy) *io->energy = c->sol_host[nn + 2 * MAXN];
    if (io->canbreak) memcpy(io->canbreak, c->sol_host + nn + 2 * MAXN + 1, sizeof(int));
    if (io->lastHS || io->lastbS || io->lastX) RET_IF(ldso_b200_get_last_solution(c, io->lastHS, io->lastbS, io->lastX));
    if (io->pt_idepth || io->pt_step || io->pt_HdiF)
        RET_IF(ldso_b200_get_points(c, io->pt_idepth, nullptr, io->pt_step, io->pt_HdiF, nullptr, nullptr, nullptr, nullptr));
    if (io->res_state || io->res_new_state || io->res_energy)
        RET_IF(ldso_b200_get_residuals(c, io->res_state, io->res_new_state, io->res_energy, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_optimize_from_host(ldso_b200_ctx *c, const ldso_b200_fused_io *io) {
    RET_IF(ldso_b200_optimize_from_host_submit(c, io));
    return ldso_b200_optimize_from_host_wait(c, io);
}

extern "C" int ldso_b200_optimize_from_host_until_submit(ldso_b200_ctx *c, const ldso_b200_fused_io *io, int min_iterations) {
    return submit_impl(c, io, true, min_iterations);
}

extern "C" int ldso_b200_optimize_from_host_until_wait(ldso_b200_ctx *c, const ldso_b200_fused_io *io, int *iterations_run) {
    RET_IF(ldso_b200_optimize_from_host_wait(c, io));
    int n = 0;
    memcpy(&n, c->sol_host + (size_t) MAXN * MAXN + 2 * MAXN + 2, sizeof(int));
    count_until_launches(c, n);
    if (iterations_run) *iterations_run = n;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_optimize_from_host_until(ldso_b200_ctx *c, const ldso_b200_fused_io *io, int min_iterations, int *iterations_run) {
    RET_IF(ldso_b200_optimize_from_host_until_submit(c, io, min_iterations));
    return ldso_b200_optimize_from_host_until_wait(c, io, iterations_run);
}

// ---- the end of FullSystem::optimize (FullSystem.cc:833-863)
// k_finish_frames (new evaluation point of the newest frame, adjoints, pair records) -> K1 (linearize + applyRes(true), as
// linearize_all(1)) -> K2a / K2b (energy, setNewFrameEnergyTH) -> k_finish_points (relBS, numGoodResiduals, dropped residuals)
// -> k_finish_tail (RMSE, lost). The pending setNewFrameEnergyTH of the loop's last linearisation runs first: LDSO's last
// linearizeAll(false) finished it before the epilogue began.
extern "C" int ldso_b200_optimize_finish(ldso_b200_ctx *c) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (c->multi) return c->fail(LDSO_B200_ERR_STATE, "optimize_finish runs on a single, unsharded context");
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    if (c->nF < 2) { c->fin_state = 1; return LDSO_B200_OK; }     // FullSystem.cc:727-728: optimize returns 0 before anything runs
    RET_IF(flush_select(c));
    k_finish_frames<<<1, 128, 0, c->stream>>>(c->ws_dev);
    LAUNCH_CHECK(c);
    RET_IF(launch_k1(c, K1F_LINEARIZE | K1F_STORE_J | K1F_APPLY_RES));       // as linearize_all(1): get_residuals reads its Jacobians
    RET_IF(launch_k2a(c, 0));
    RET_IF(launch_k2b(c, 0, 1, 0));
    if (c->d.nP > 0) {
        k_finish_points<<<(c->d.nP + 127) / 128, 128, 0, c->stream>>>(c->d, (const WinState *) c->ws_dev, c->fb);
        LAUNCH_CHECK(c);
    }
    k_finish_tail<<<1, 32, 0, c->stream>>>((const WinState *) c->ws_dev, c->fb);
    LAUNCH_CHECK(c);
    c->fin_state = 2;
    c->fin_window_stale = true; c->fin_frames_stale = true;
    c->solve_ready = false; c->restitch_ok = false;
    c->evalpt_key.clear();      // the device adjoints now belong to the new evaluation point: the next set_frames recomputes them
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_finish(ldso_b200_ctx *c, double *energy, float *rmse, int *is_lost, uint8_t *res_state, uint8_t *res_dropped,
                                    float *pt_relBS_max, int32_t *pt_n_good, double newest_evalR[9], double newest_evalT[3],
                                    double newest_state_zero[10]) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (c->fin_state == 0 || !c->have_window || !c->have_frames) return c->fail(LDSO_B200_ERR_STATE, "no optimize_finish to read");
    cudaSetDevice(c->device);
    const size_t nP = c->d.nP, nR = c->d.nR;
    FrameDev fr;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(&fr, &c->ws_dev->fr[c->nF - 1], sizeof(FrameDev), cudaMemcpyDeviceToHost, c->stream));
    if (c->fin_state == 2) {
        D2H(energy, &c->ws_dev->energy, sizeof(double));
        D2H(rmse, c->fb.rmse, sizeof(float));
        D2H(is_lost, c->fb.is_lost, sizeof(int));
        D2H(res_state, c->d.res_state, nR);
        D2H(res_dropped, c->fb.res_dropped, nR);
        D2H(pt_relBS_max, c->fb.pt_relBS_max, 4 * nP);
        D2H(pt_n_good, c->fb.pt_n_good, 4 * nP);
    } else {
        if (energy) *energy = 0.0;
        if (rmse) *rmse = 0.f;
        if (is_lost) *is_lost = 0;
        D2H(res_state, c->d.res_state, nR);
        if (res_dropped) memset(res_dropped, 0, nR);
        if (pt_relBS_max) memset(pt_relBS_max, 0, 4 * nP);
        if (pt_n_good) memset(pt_n_good, 0, 4 * nP);
    }
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    if (newest_evalR) memcpy(newest_evalR, fr.evalR, sizeof(fr.evalR));
    if (newest_evalT) memcpy(newest_evalT, fr.evalT, sizeof(fr.evalT));
    if (newest_state_zero) memcpy(newest_state_zero, fr.state_zero, sizeof(fr.state_zero));
    return LDSO_B200_OK;
}

// optimize_from_host_until + optimize_finish. io's outputs are the loop's results (read back into pinned staging before the finish
// runs, as optimize_from_host_until returns them); `out` receives what get_finish returns.
extern "C" int ldso_b200_optimize_from_host_full_submit(ldso_b200_ctx *c, const ldso_b200_fused_io *io, int min_iterations) {
    RET_IF(submit_impl(c, io, true, min_iterations));
    RET_IF(ldso_b200_optimize_finish(c));
    // the finish's launches do not touch what the prefetch queued before them: keep waiting on that copy
    c->results_inflight = true;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_optimize_from_host_full_wait(ldso_b200_ctx *c, const ldso_b200_fused_io *io, const ldso_b200_finish_out *out) {
    if (!c || !out) return LDSO_B200_ERR_ARG;
    RET_IF(ldso_b200_optimize_from_host_until_wait(c, io, out->iterations_run));
    // the mirror holds the loop's results, the device the finish's
    { c->mirror_valid = false; c->sol_valid = false; c->mirror_full_valid = false; }
    return ldso_b200_get_finish(c, out->energy, out->rmse, out->is_lost, out->res_state, out->res_dropped, out->pt_relBS_max, out->pt_n_good,
                                out->newest_evalR, out->newest_evalT, out->newest_state_zero);
}

extern "C" int ldso_b200_optimize_from_host_full(ldso_b200_ctx *c, const ldso_b200_fused_io *io, int min_iterations, const ldso_b200_finish_out *out) {
    if (!c || !out) return LDSO_B200_ERR_ARG;
    RET_IF(ldso_b200_optimize_from_host_full_submit(c, io, min_iterations));
    return ldso_b200_optimize_from_host_full_wait(c, io, out);
}

extern "C" int ldso_b200_reduce_buffer(ldso_b200_ctx *c, void **buf_dev, size_t *n_doubles) {
    if (!c || !buf_dev || !n_doubles) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    *buf_dev = c->d.red;
    *n_doubles = (size_t) RED_SELECT + std::max(c->d.newest_total, 0);
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_set_shard(ldso_b200_ctx *c, int newest_slot_offset, int newest_total) {
    if (!c) return LDSO_B200_ERR_ARG;
    if (newest_slot_offset < 0 || newest_total < newest_slot_offset) return c->fail(LDSO_B200_ERR_ARG, "bad shard description");
    c->multi = true;
    c->d.newest_offset = newest_slot_offset;
    c->d.newest_total = newest_total;
    c->derived_dirty = true;
    return LDSO_B200_OK;
}

// ---- peer-memory exchange: export this rank's block, map the peers', then gn_iterations / optimize_begin run the whole
// sharded iteration on the device (K3 -> K1 -> K2a -> K2r -> K2b) with no NCCL call and no host round trip
extern "C" int ldso_b200_peer_export(ldso_b200_ctx *c, void *ipc_handle_64) {
    if (!c || !ipc_handle_64) return LDSO_B200_ERR_ARG;
    if (!c->multi) return c->fail(LDSO_B200_ERR_STATE, "peer_export needs set_shard first");
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    const int n = RED_SELECT + std::max(c->d.newest_total, 0);
    const int nch = (n + K2R_THREADS - 1) / K2R_THREADS;
    if (c->peers_connected || c->peer_local) return c->fail(LDSO_B200_ERR_STATE, "peer exchange already set up for this context");
    const size_t bytes = sizeof(uint4) * (2 * K2R_MAX_PEERS + 2) * (size_t) n;      // the inbox: [2 parities][8 senders][n] 16-byte slots + the all-gather region [2][n]
    CUDA_CHECK_RET(c, cudaMalloc(&c->peer_local, bytes));
    CUDA_CHECK_RET(c, cudaMalloc(&c->peer_words, sizeof(int) * 4));
    CUDA_CHECK_RET(c, cudaMalloc(&c->red_sum, sizeof(double) * ((size_t) n + 16)));
    // cleared on the context's own (non-blocking) stream and completed before the handle is handed out: a peer's first push
    // and this rank's first exchange kernel must find zeroed tags
    CUDA_CHECK_RET(c, cudaMemsetAsync(c->peer_local, 0, bytes, c->stream));
    CUDA_CHECK_RET(c, cudaMemsetAsync(c->peer_words, 0, sizeof(int) * 4, c->stream));
    CUDA_CHECK_RET(c, cudaMemsetAsync(c->red_sum, 0, sizeof(double) * ((size_t) n + 16), c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    memset(&c->px, 0, sizeof(c->px));
    c->px.n_doubles = n; c->px.n_chunks = nch;
    cudaIpcMemHandle_t h;
    CUDA_CHECK_RET(c, cudaIpcGetMemHandle(&h, c->peer_local));
    memcpy(ipc_handle_64, &h, 64);
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_peer_connect(ldso_b200_ctx *c, int rank, int world, const void *ipc_handles_64_each) {
    if (!c || !ipc_handles_64_each) return LDSO_B200_ERR_ARG;
    if (!c->peer_local) return c->fail(LDSO_B200_ERR_STATE, "peer_connect needs peer_export first");
    if (world < 1 || world > K2R_MAX_PEERS || rank < 0 || rank >= world) return c->fail(LDSO_B200_ERR_ARG, "rank/world out of range (max 8 peers)");
    cudaSetDevice(c->device);
    for (int r = 0; r < world; r++) {
        char *base = c->peer_local;
        if (r != rank) {
            cudaIpcMemHandle_t h;
            memcpy(&h, (const char *) ipc_handles_64_each + 64 * r, 64);
            void *p = nullptr;
            CUDA_CHECK_RET(c, cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
            c->peer_opened[r] = p;
            base = (char *) p;
        }
        c->px.inbox[r] = (uint4 *) base;
    }
    c->px.rank = rank; c->px.world = world;
    c->px.two_hop = (world > 2 && getenv("LDSO_B200_K2R_ONESHOT") == nullptr) ? 1 : 0;
    c->px.epoch = c->peer_words; c->px.done = (unsigned *) (c->peer_words + 1); c->px.error = c->peer_words + 2;
    c->px.out = c->red_sum;
    c->peers_connected = true;
    c->gn_graph_valid = false; c->until_graph_valid = false;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_peer_error(ldso_b200_ctx *c, int *error) {
    if (!c || !error || !c->peer_words) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(error, c->peer_words + 2, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}


extern "C" int ldso_b200_gn_phase_a(ldso_b200_ctx *c, int iteration) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(check_solve_frames(c));
    RET_IF(clear_select(c));
    if (iteration < 0) {
        RET_IF(launch_k1(c, K1_FUSED | K1F_RESET_OOB));
    } else {
        if (!c->solve_ready) return c->fail(LDSO_B200_ERR_STATE, "gn_phase_a(iteration >= 0) needs a preceding gn_phase_b");
        RET_IF(flush_select(c));
        RET_IF(set_iteration(c, iteration));
        RET_IF(launch_k3(c, K3F_BACKUP | K3F_SOLVE | K3F_STEP));
        RET_IF(launch_k1(c, K1_FUSED | K1F_APPLY_STEP));
    }
    RET_IF(launch_k2a(c, 1));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_gn_phase_b(ldso_b200_ctx *c) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    RET_IF(build_derived(c));
    RET_IF(launch_k2b(c, 1, 1, 1));
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- read-back
extern "C" int ldso_b200_get_energy(ldso_b200_ctx *c, double *energy, int *canbreak) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    if (energy) CUDA_CHECK_RET(c, cudaMemcpyAsync(energy, &c->ws_dev->energy, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (canbreak) CUDA_CHECK_RET(c, cudaMemcpyAsync(canbreak, &c->ws_dev->canbreak, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

// one D2H of the contiguous result range into the pinned mirror (valid until the next launch)
// Optional hint: queue the read-back of everything the getters below return (solution, point and residual arrays) into
// pinned staging memory right behind the work already on the stream, without blocking. The next getter then only waits
// for that one event instead of issuing its own copy + synchronize.
extern "C" int ldso_b200_prefetch_results(ldso_b200_ctx *c) {
    if (!c || !c->have_window || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    auto &L = c->lay;
    const size_t nn = (size_t) MAXN * MAXN;
    if (!c->mirror_valid)
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->arena_host + L.res_state, c->arena_dev + L.res_state, L.dl_light_end - L.res_state, cudaMemcpyDeviceToHost, c->stream));
    if (!c->sol_valid)
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->sol_host, c->sb.lastHS, sizeof(double) * (nn + 2 * MAXN), cudaMemcpyDeviceToHost, c->stream));
    if (!c->results_ready) CUDA_CHECK_RET(c, cudaEventCreateWithFlags(&c->results_ready, cudaEventDisableTiming));
    CUDA_CHECK_RET(c, cudaEventRecord(c->results_ready, c->stream));
    c->results_inflight = true;
    return LDSO_B200_OK;
}
static int wait_results(ldso_b200_ctx *c) {
    if (!c->results_inflight) return LDSO_B200_OK;
    CUDA_CHECK_RET(c, cudaEventSynchronize(c->results_ready));
    c->results_inflight = false;
    c->mirror_valid = true;
    c->sol_valid = true;
    return LDSO_B200_OK;
}

static int refresh_mirror(ldso_b200_ctx *c, bool full = false) {
    RET_IF(wait_results(c));
    auto &L = c->lay;
    bool copied = false;
    if (!c->mirror_valid) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->arena_host + L.res_state, c->arena_dev + L.res_state, L.dl_light_end - L.res_state, cudaMemcpyDeviceToHost, c->stream));
        copied = true;
    }
    if (full && !c->mirror_full_valid) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->arena_host + L.dl_light_end, c->arena_dev + L.dl_light_end, L.dl_end - L.dl_light_end, cudaMemcpyDeviceToHost, c->stream));
        copied = true;
    }
    if (copied) CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    c->mirror_valid = true;
    if (full) c->mirror_full_valid = true;
    return LDSO_B200_OK;
}
#define FROM_MIRROR(dst, off, bytes) do { if (dst) memcpy(dst, c->arena_host + (off), (bytes)); } while (0)

extern "C" int ldso_b200_get_points(ldso_b200_ctx *c, float *idepth, float *idepth_zero, float *step, float *HdiF,
                                    float *bdSumF, float *Hdd, float *bd, float *Hcd4) {
    if (!c || !c->have_window) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    RET_IF(refresh_mirror(c));
    const size_t nP = c->d.nP;
    auto &L = c->lay;
    FROM_MIRROR(idepth, L.pt_idepth, 4 * nP); FROM_MIRROR(idepth_zero, L.pt_idepth_zero, 4 * nP); FROM_MIRROR(step, L.pt_step, 4 * nP);
    FROM_MIRROR(HdiF, L.pt_HdiF, 4 * nP); FROM_MIRROR(bdSumF, L.pt_bdSumF, 4 * nP); FROM_MIRROR(Hdd, L.pt_Hdd, 4 * nP);
    FROM_MIRROR(bd, L.pt_bd, 4 * nP); FROM_MIRROR(Hcd4, L.pt_Hcd, 16 * nP);
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_residuals(ldso_b200_ctx *c, uint8_t *state_state, uint8_t *state_NewState, float *state_energy,
                                       float *state_NewEnergy, float *state_NewEnergyWithOutlier, uint8_t *isActive,
                                       float *JpJdF8, float *J74, float *projectedTo16, float *centerProjectedTo3) {
    if (!c || !c->have_window) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    RET_IF(refresh_mirror(c, JpJdF8 != nullptr));
    const size_t nR = c->d.nR;
    auto &L = c->lay;
    FROM_MIRROR(state_state, L.res_state, nR); FROM_MIRROR(state_NewState, L.res_new_state, nR); FROM_MIRROR(state_energy, L.res_energy, 4 * nR);
    FROM_MIRROR(state_NewEnergy, L.res_new_energy, 4 * nR); FROM_MIRROR(state_NewEnergyWithOutlier, L.res_new_energy_wo, 4 * nR);
    FROM_MIRROR(isActive, L.res_active, nR); FROM_MIRROR(JpJdF8, L.res_JpJdF, 32 * nR);
    if (J74 || projectedTo16 || centerProjectedTo3) {
        D2H(J74, c->d.res_J, 296 * nR); D2H(projectedTo16, c->d.res_proj, 64 * nR); D2H(centerProjectedTo3, c->d.res_cpt, 12 * nR);
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_get_frames(ldso_b200_ctx *c, double *state10, double *step10, float *frameEnergyTH, float *precalc40,
                                    double *adHost64, double *adTarget64, float *adHTdeltaF8, double *calib_value4) {
    if (!c || !c->have_frames) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    if (c->have_window && !c->derived_dirty) RET_IF(flush_select(c));
    CUDA_CHECK_RET(c, cudaMemcpyAsync(c->ws_host, c->ws_dev, sizeof(WinState), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    const WinState &W = *c->ws_host;
    const int nF = W.nF;
    for (int h = 0; h < nF; h++) {
        if (state10) memcpy(state10 + 10 * h, W.fr[h].state, 80);
        if (step10) memcpy(step10 + 10 * h, W.fr[h].step, 80);
        if (frameEnergyTH) frameEnergyTH[h] = W.frameEnergyTH[h];
    }
    for (int q = 0; q < nF * nF; q++) {
        if (precalc40) {
            float *d = precalc40 + 40 * q;
            const PairRec &p = W.pair[q];
            const PairRecFull &f = W.pairFull[q];
            memcpy(d, p.R0, 36); memcpy(d + 9, p.t0, 12); memcpy(d + 12, f.RTll, 36); memcpy(d + 21, f.tTll, 12);
            memcpy(d + 24, p.KRKi, 36); memcpy(d + 33, p.Kt, 12);
            d[36] = p.aff[0]; d[37] = p.aff[1]; d[38] = p.b0; d[39] = p.distanceLL;
        }
        if (adHost64) memcpy(adHost64 + 64 * q, W.adHost[q], 512);
        if (adTarget64) memcpy(adTarget64 + 64 * q, W.adTarget[q], 512);
        if (adHTdeltaF8) memcpy(adHTdeltaF8 + 8 * q, W.adHTdeltaF[q], 32);
    }
    if (calib_value4) memcpy(calib_value4, W.calib.value, 32);
    return LDSO_B200_OK;
}

// Per-kernel CUDA-event timing of the GN loop (bench.py's roofline leg): enable != 0 starts collecting (graphs off),
// enable == 0 stops and returns the average duration in microseconds of K1, K2a, K2b, K3 since it was enabled.
extern "C" int ldso_b200_kernel_times(ldso_b200_ctx *c, int enable, double out_us[5]) {
    if (!c) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    if (enable) {
        for (auto &k : c->kt) { cudaEventDestroy(k.a); cudaEventDestroy(k.b); }
        c->kt.clear();
        c->ktime = true;
        c->use_graph = false;
        return LDSO_B200_OK;
    }
    const char *names[5] = {"k1", "k2a", "k2b", "k3", "k2r"};
    double tot[5] = {0, 0, 0, 0, 0};
    int cnt[5] = {0, 0, 0, 0, 0};
    for (auto &k : c->kt) {
        float ms = 0;
        cudaEventElapsedTime(&ms, k.a, k.b);
        for (int i = 0; i < 5; i++) if (!strcmp(names[i], k.name)) { tot[i] += ms; cnt[i]++; }
        cudaEventDestroy(k.a); cudaEventDestroy(k.b);
    }
    c->kt.clear();
    c->ktime = getenv("LDSO_B200_KTIME") != nullptr;
    c->use_graph = !c->ktime && getenv("LDSO_B200_NO_GRAPH") == nullptr;
    if (out_us) for (int i = 0; i < 5; i++) out_us[i] = cnt[i] ? 1e3 * tot[i] / cnt[i] : 0.0;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_debug_res_to_zero(ldso_b200_ctx *c, float *out8) {
    if (!c || !out8 || !c->have_window) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(out8, c->d.res_toZero, 32 * (size_t) c->d.nR, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_debug_clocks(ldso_b200_ctx *c, long long *out32) {
    if (!c || !out32) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    // out: 80 values = WinState::dbg[0..63] then DevWindow::dbg[0..15]
    CUDA_CHECK_RET(c, cudaMemcpyAsync(out32, c->ws_dev->dbg, sizeof(long long) * 64, cudaMemcpyDeviceToHost, c->stream));
    if (c->d.dbg) CUDA_CHECK_RET(c, cudaMemcpyAsync(out32 + 64, c->d.dbg, sizeof(long long) * 16, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_debug_cta_spans(ldso_b200_ctx *c, long long *out, int cap_items) {
    if (!c || !out || !c->d.dbg) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    const int n = std::min(cap_items, c->d.nItems);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(out, c->d.dbg + 32, sizeof(long long) * 3 * n, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return n;
}

extern "C" int ldso_b200_get_nullspace_projector(ldso_b200_ctx *c, double *P) {
    if (!c || !c->have_frames || !P) return LDSO_B200_ERR_STATE;
    cudaSetDevice(c->device);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(P, c->sb.Pns, sizeof(double) * c->n * c->n, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- pose graph
// Map::runPoseGraphOptimization (src/Map.cc:75-165): g2o Gauss-Newton over VertexSim3 / EdgeSim3 with numeric Jacobians, `iterations`
// rounds (25 in the reference), vertex `fixed` held (the current keyframe). The linear system of a round is solved by block-Jacobi
// preconditioned conjugate gradients to a relative residual of pcg_tol (g2o factorises it; both are exact solves of the same normal
// equations up to pcg_tol). Poses in / out as Sim3 = quaternion (w, x, y, z) with norm = scale + translation (Sophus' storage).
extern "C" int ldso_b200_posegraph_optimize(ldso_b200_ctx *c, int nV, double *q4, double *t3, int nE, const int32_t *ei, const int32_t *ej,
                                            const double *mq4, const double *mt3, const double *info49, int fixed, int iterations,
                                            double pcg_tol, int pcg_max_iter, double *chi2_out, int *pcg_iterations_total) {
    if (!c || nV < 2 || nE < 1 || !q4 || !t3 || !ei || !ej || !mq4 || !mt3 || !info49 || iterations < 0) return LDSO_B200_ERR_ARG;
    if (fixed < 0 || fixed >= nV) return c->fail(LDSO_B200_ERR_ARG, "fixed vertex out of range");
    for (int e = 0; e < nE; e++) if (ei[e] < 0 || ei[e] >= nV || ej[e] < 0 || ej[e] >= nV || ei[e] == ej[e]) return c->fail(LDSO_B200_ERR_ARG, "edge vertex index out of range");
    cudaSetDevice(c->device);
    // incidence lists (vertex -> edge * 2 + side), edge order
    std::vector<int> ib(nV + 1, 0), inc(2 * (size_t) nE);
    for (int e = 0; e < nE; e++) { ib[ei[e] + 1]++; ib[ej[e] + 1]++; }
    for (int v = 0; v < nV; v++) ib[v + 1] += ib[v];
    { std::vector<int> pos(ib.begin(), ib.end() - 1); for (int e = 0; e < nE; e++) { inc[pos[ei[e]]++] = 2 * e; inc[pos[ej[e]]++] = 2 * e + 1; } }
    const int nbv = (nV + PG_WARPS - 1) / PG_WARPS, nbe = (nE + PG_WARPS - 1) / PG_WARPS;
    PgGraph g;
    Arena S;
    posegraph_regions(S, nV, nE, g);
    char *B = nullptr;
    CUDA_CHECK_RET(c, cudaMalloc(&B, S.off));
    struct Free { char *p; ~Free() { if (p) cudaFree(p); } } guard{B};
    Arena D(B);
    posegraph_regions(D, nV, nE, g);
    CUDA_CHECK_RET(c, cudaMemsetAsync(B, 0, S.off, c->stream));
    H2D(g.q, q4, 32 * (size_t) nV); H2D(g.t, t3, 24 * (size_t) nV); H2D(g.ei, ei, 4 * (size_t) nE); H2D(g.ej, ej, 4 * (size_t) nE);
    H2D(g.mq, mq4, 32 * (size_t) nE); H2D(g.mt, mt3, 24 * (size_t) nE); H2D(g.info, info49, 392 * (size_t) nE);
    H2D(g.inc_begin, ib.data(), 4 * ((size_t) nV + 1)); H2D(g.inc, inc.data(), 8 * (size_t) nE);
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));      // pageable sources
    g.nV = nV; g.nE = nE; g.fixed = fixed;
    int total_cg = 0;
    const int chunk = 10;
    for (int it = 0; it <= iterations; it++) {
        k_pg_linearize<<<nbe, 32 * PG_WARPS, 0, c->stream>>>(g);
        LAUNCH_CHECK(c);
        k_pg_chi2<<<1, 256, 0, c->stream>>>(g, g.scal + 5);
        LAUNCH_CHECK(c);
        if (chi2_out) CUDA_CHECK_RET(c, cudaMemcpyAsync(chi2_out + it, g.scal + 5, 8, cudaMemcpyDeviceToHost, c->stream));
        if (it == iterations) break;
        k_pg_assemble<<<nbv, 32 * PG_WARPS, 0, c->stream>>>(g);
        LAUNCH_CHECK(c);
        double rz0 = 0.0, rz = 0.0;
        CUDA_CHECK_RET(c, cudaMemcpyAsync(&rz0, g.scal, 8, cudaMemcpyDeviceToHost, c->stream));
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        rz = rz0;
        int k = 0;
        while (k < pcg_max_iter && rz > pcg_tol * pcg_tol * rz0 && rz0 > 0.0) {
            for (int j = 0; j < chunk && k < pcg_max_iter; j++, k++) {
                double *pin = (k & 1) ? g.p0 : g.p1, *pout = (k & 1) ? g.p1 : g.p0;
                k_pg_cg_a<<<nbv, 32 * PG_WARPS, 0, c->stream>>>(g, pin, pout, k == 0 ? 1 : 0);
                k_pg_cg_b<<<nbv, 32 * PG_WARPS, 0, c->stream>>>(g, pout);
                c->launches += 2;
            }
            CUDA_CHECK_RET(c, cudaMemcpyAsync(&rz, g.scal, 8, cudaMemcpyDeviceToHost, c->stream));
            CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
            if (!(rz == rz)) return c->fail(LDSO_B200_ERR_STATE, "pose graph: the normal equations are not positive definite (CG broke down)");
        }
        total_cg += k;
        k_pg_update<<<(nV + 127) / 128, 128, 0, c->stream>>>(g);
        LAUNCH_CHECK(c);
    }
    CUDA_CHECK_RET(c, cudaMemcpyAsync(q4, g.q, 32 * (size_t) nV, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaMemcpyAsync(t3, g.t, 24 * (size_t) nV, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    { cudaError_t e__ = cudaGetLastError(); if (e__ != cudaSuccess) return c->fail_cuda(e__, "pose graph kernels", __FILE__, __LINE__); }
    if (pcg_iterations_total) *pcg_iterations_total = total_cg;
    return LDSO_B200_OK;
}

// ---------------------------------------------------------------------------------------------- tracker
extern "C" int ldso_b200_tracker_make_k(ldso_b200_ctx *c, float fx, float fy, float cx, float cy) {
    if (!c) return LDSO_B200_ERR_ARG;
    // CoarseTracker::makeK (CoarseTracker.cc:219-246)
    c->trk_fx[0] = fx; c->trk_fy[0] = fy; c->trk_cx[0] = cx; c->trk_cy[0] = cy;
    for (int l = 1; l < c->levels; l++) {
        c->trk_fx[l] = c->trk_fx[l - 1] * 0.5;
        c->trk_fy[l] = c->trk_fy[l - 1] * 0.5;
        c->trk_cx[l] = (c->trk_cx[0] + 0.5) / ((int) 1 << l) - 0.5;
        c->trk_cy[l] = (c->trk_cy[0] + 0.5) / ((int) 1 << l) - 0.5;
    }
    for (int l = 0; l < c->levels; l++) {
        const float K[9] = {c->trk_fx[l], 0, c->trk_cx[l], 0, c->trk_fy[l], c->trk_cy[l], 0, 0, 1};
        m33f_inverse(K, c->trk_Ki[l]);
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_tracker_set_ref_level(ldso_b200_ctx *c, int lvl, int n, const float *pc_u, const float *pc_v,
                                               const float *pc_idepth, const float *pc_color) {
    if (!c || lvl < 0 || lvl >= c->levels || n < 0) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    if (n > c->trk_cap[lvl]) {
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        for (int k = 0; k < 4; k++) {
            if (c->trk_pc[lvl][k]) cudaFree(c->trk_pc[lvl][k]);
            CUDA_CHECK_RET(c, cudaMalloc(&c->trk_pc[lvl][k], sizeof(float) * n));
        }
        c->trk_cap[lvl] = n;
    }
    const float *src[4] = {pc_u, pc_v, pc_idepth, pc_color};
    for (int k = 0; k < 4; k++)
        if (n > 0) CUDA_CHECK_RET(c, cudaMemcpyAsync(c->trk_pc[lvl][k], src[k], sizeof(float) * n, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    c->trk[lvl].n = n;
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_tracker_get_ref_level(ldso_b200_ctx *c, int lvl, int *n, float *pc_u, float *pc_v, float *pc_idepth, float *pc_color) {
    if (!c || lvl < 0 || lvl >= c->levels) return LDSO_B200_ERR_ARG;
    cudaSetDevice(c->device);
    const int m = c->trk[lvl].n;
    if (n) *n = m;
    float *dst[4] = {pc_u, pc_v, pc_idepth, pc_color};
    for (int k = 0; k < 4; k++) if (dst[k] && m > 0) CUDA_CHECK_RET(c, cudaMemcpyAsync(dst[k], c->trk_pc[lvl][k], sizeof(float) * m, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_tracker_set_frames(ldso_b200_ctx *c, float ref_aff_a, float ref_aff_b, float ref_exposure, int new_slot, float new_exposure) {
    if (!c || new_slot < 0 || new_slot >= NSLOTS || !c->img[new_slot][0]) return LDSO_B200_ERR_ARG;
    c->ref_aff_a = ref_aff_a; c->ref_aff_b = ref_aff_b; c->ref_exposure = ref_exposure;
    c->new_slot = new_slot; c->new_exposure = new_exposure;
    return LDSO_B200_OK;
}

static void fill_level(ldso_b200_ctx *c, int l, TrkLevel &L) {
    L.pc_u = c->trk_pc[l][0]; L.pc_v = c->trk_pc[l][1]; L.pc_idepth = c->trk_pc[l][2]; L.pc_color = c->trk_pc[l][3];
    L.n = c->trk[l].n;
    L.img = c->img[c->new_slot][l];
    L.w = c->lw[l]; L.h = c->lh[l];
    L.fx = c->trk_fx[l]; L.fy = c->trk_fy[l]; L.cx = c->trk_cx[l]; L.cy = c->trk_cy[l];
    memcpy(L.Ki, c->trk_Ki[l], sizeof(L.Ki));
}

extern "C" int ldso_b200_tracker_eval(ldso_b200_ctx *c, int lvl, const double R[9], const double t[3], float aff_a, float aff_b,
                                      float cutoffTH, double res6[6], double H[64], double b[8]) {
    if (!c || lvl < 0 || lvl >= c->levels || !R || !t || !res6) return LDSO_B200_ERR_ARG;
    if (c->new_slot < 0) return c->fail(LDSO_B200_ERR_STATE, "tracker_set_frames not called");
    cudaSetDevice(c->device);
    TrkLevel L;
    fill_level(c, lvl, L);
    TrkPose P;
    float Rf[9];
    for (int i = 0; i < 9; i++) Rf[i] = (float) R[i];
    m33f_mul(Rf, L.Ki, P.RKi);
    for (int i = 0; i < 3; i++) P.t[i] = (float) t[i];
    float eF = c->ref_exposure, eT = c->new_exposure;
    if (eF == 0 || eT == 0) eT = eF = 1;
    const float a = expf(aff_a - c->ref_aff_a) * eT / eF;
    P.affLL0 = a; P.affLL1 = aff_b - a * c->ref_aff_b; P.b0 = c->ref_aff_b;
    P.cutoffTH = cutoffTH; P.huberTH = c->S.huberTH;
    P.maxEnergy = 2 * c->S.huberTH * cutoffTH - c->S.huberTH * c->S.huberTH;
    int grid = std::max(1, std::min(1024, (L.n + TRK_EVAL_THREADS - 1) / TRK_EVAL_THREADS));
    k_trk_eval<<<grid, TRK_EVAL_THREADS, 0, c->stream>>>(L, P, lvl == 0 ? 1 : 0, c->trk_partials, c->trk_counter, c->trk_out_dev, (H && b) ? 1 : 0);
    LAUNCH_CHECK(c);
    double out[78];
    CUDA_CHECK_RET(c, cudaMemcpyAsync(out, c->trk_out_dev, sizeof(out), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    memcpy(res6, out, 48);
    if (H && b) { memcpy(H, out + 6, 512); memcpy(b, out + 70, 64); }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_tracker_track(ldso_b200_ctx *c, double R[9], double t[3], float *aff_a, float *aff_b, int coarsestLvl,
                                       const double minResForAbort[5], double lastResiduals[5], double lastFlowIndicators[3], int *ok) {
    if (!c || !R || !t || !aff_a || !aff_b || !ok) return LDSO_B200_ERR_ARG;
    if (coarsestLvl < 0 || coarsestLvl >= 5 || coarsestLvl >= c->levels) return c->fail(LDSO_B200_ERR_ARG, "coarsestLvl out of range");
    if (c->new_slot < 0) return c->fail(LDSO_B200_ERR_STATE, "tracker_set_frames not called");
    cudaSetDevice(c->device);
    TrkTrackArgs A;
    memset(&A, 0, sizeof(A));
    for (int l = 0; l < c->levels; l++) fill_level(c, l, A.L[l]);
    A.nLevels = c->levels;
    A.ref_aff_a = c->ref_aff_a; A.ref_aff_b = c->ref_aff_b; A.ref_exposure = c->ref_exposure; A.new_exposure = c->new_exposure;
    A.huberTH = c->S.huberTH; A.coarseCutoffTH = c->S.coarseCutoffTH; A.affineOptModeA = c->S.affineOptModeA; A.affineOptModeB = c->S.affineOptModeB;
    memcpy(A.R, R, 72); memcpy(A.t, t, 24);
    A.aff_a = *aff_a; A.aff_b = *aff_b;
    A.coarsestLvl = coarsestLvl;
    for (int i = 0; i < 5; i++) A.minResForAbort[i] = minResForAbort ? minResForAbort[i] : NAN;
    k_trk_track<<<1, TRK_TRACK_THREADS, 0, c->stream>>>(A, c->trk_track_out, nullptr);
    LAUNCH_CHECK(c);
    TrkTrackOut o;
    CUDA_CHECK_RET(c, cudaMemcpyAsync(&o, c->trk_track_out, sizeof(o), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    memcpy(R, o.R, 72); memcpy(t, o.t, 24);
    *aff_a = o.aff_a; *aff_b = o.aff_b;
    if (lastResiduals) memcpy(lastResiduals, o.lastResiduals, 40);
    if (lastFlowIndicators) memcpy(lastFlowIndicators, o.lastFlowIndicators, 24);
    *ok = o.ok;
    return LDSO_B200_OK;
}

// FullSystem::trackNewCoarse's hypothesis loop (FullSystem.cc:290-357) as ONE launch: n starting poses (the constant-motion,
// double-motion, half-motion, zero-motion guesses and the 26 x 3 small rotations), each tracked by its own CTA through all levels,
// all without an abort threshold (the reference passes the best residuals so far as minResForAbort to the later tries: a pruning
// of work that a parallel batch does not need). The caller applies the reference's acceptance rule to the n results.
extern "C" int ldso_b200_tracker_track_batch(ldso_b200_ctx *c, int n, const double *R9_each, const double *t3_each, const float *aff2_each, int coarsestLvl,
                                             double *R9_out, double *t3_out, float *aff2_out, double *lastResiduals5_each, double *lastFlow3_each, int *ok_each) {
    if (!c || n <= 0 || !R9_each || !t3_each || !aff2_each || !ok_each) return LDSO_B200_ERR_ARG;
    if (n > 128) return c->fail(LDSO_B200_ERR_ARG, "at most 128 hypotheses per batch");
    if (coarsestLvl < 0 || coarsestLvl >= 5 || coarsestLvl >= c->levels) return c->fail(LDSO_B200_ERR_ARG, "coarsestLvl out of range");
    if (c->new_slot < 0) return c->fail(LDSO_B200_ERR_STATE, "tracker_set_frames not called");
    cudaSetDevice(c->device);
    TrkTrackArgs A;
    memset(&A, 0, sizeof(A));
    for (int l = 0; l < c->levels; l++) fill_level(c, l, A.L[l]);
    A.nLevels = c->levels;
    A.ref_aff_a = c->ref_aff_a; A.ref_aff_b = c->ref_aff_b; A.ref_exposure = c->ref_exposure; A.new_exposure = c->new_exposure;
    A.huberTH = c->S.huberTH; A.coarseCutoffTH = c->S.coarseCutoffTH; A.affineOptModeA = c->S.affineOptModeA; A.affineOptModeB = c->S.affineOptModeB;
    A.coarsestLvl = coarsestLvl;
    for (int i = 0; i < 5; i++) A.minResForAbort[i] = NAN;
    TrackBatchScratch s;
    RET_IF(trace_carve(c, [&](Arena &R) { track_batch_regions(R, (size_t) n, s); }));
    std::vector<TrkHypothesis> hh(n);
    for (int i = 0; i < n; i++) {
        memcpy(hh[i].R, R9_each + 9 * i, 72); memcpy(hh[i].t, t3_each + 3 * i, 24);
        hh[i].aff_a = aff2_each[2 * i]; hh[i].aff_b = aff2_each[2 * i + 1];
    }
    H2D(s.hyp, hh.data(), sizeof(TrkHypothesis) * n);
    k_trk_track<<<n, TRK_TRACK_THREADS, 0, c->stream>>>(A, s.out, s.hyp);
    LAUNCH_CHECK(c);
    std::vector<TrkTrackOut> ho(n);
    CUDA_CHECK_RET(c, cudaMemcpyAsync(ho.data(), s.out, sizeof(TrkTrackOut) * n, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    for (int i = 0; i < n; i++) {
        if (R9_out) memcpy(R9_out + 9 * i, ho[i].R, 72);
        if (t3_out) memcpy(t3_out + 3 * i, ho[i].t, 24);
        if (aff2_out) { aff2_out[2 * i] = ho[i].aff_a; aff2_out[2 * i + 1] = ho[i].aff_b; }
        if (lastResiduals5_each) memcpy(lastResiduals5_each + 5 * i, ho[i].lastResiduals, 40);
        if (lastFlow3_each) memcpy(lastFlow3_each + 3 * i, ho[i].lastFlowIndicators, 24);
        ok_each[i] = ho[i].ok;
    }
    return LDSO_B200_OK;
}

extern "C" int ldso_b200_tracker_make_coarse_depth(ldso_b200_ctx *c, int ref_slot, int n, const float *centerProjectedTo3, const float *HdiF) {
    if (!c || n < 0 || (n > 0 && (!centerProjectedTo3 || !HdiF))) return LDSO_B200_ERR_ARG;
    if (ref_slot < 0 || ref_slot >= NSLOTS || !c->img[ref_slot][0]) return c->fail(LDSO_B200_ERR_ARG, "reference image slot not uploaded");
    if (c->lh[0] > 1024) return c->fail(LDSO_B200_ERR_ARG, "image height > 1024 not supported by the row scan");
    cudaSetDevice(c->device);
    // buffers: idepth / weightSums / weightSums_bak / pos per level, point-cloud arrays with wl*hl capacity (CoarseTracker.cc:36-45)
    for (int l = 0; l < c->levels; l++) {
        const size_t npx = (size_t) c->lw[l] * c->lh[l];
        if (!c->cd_id[l]) {
            CUDA_CHECK_RET(c, cudaMalloc(&c->cd_id[l], 4 * npx)); CUDA_CHECK_RET(c, cudaMalloc(&c->cd_ws[l], 4 * npx));
            CUDA_CHECK_RET(c, cudaMalloc(&c->cd_bak[l], 4 * npx)); CUDA_CHECK_RET(c, cudaMalloc(&c->cd_pos[l], 4 * npx));
        }
        if ((int) npx > c->trk_cap[l]) {
            CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
            for (int k = 0; k < 4; k++) { if (c->trk_pc[l][k]) cudaFree(c->trk_pc[l][k]); CUDA_CHECK_RET(c, cudaMalloc(&c->trk_pc[l][k], 4 * npx)); }
            c->trk_cap[l] = (int) npx;
        }
    }
    if (!c->cd_rows) { CUDA_CHECK_RET(c, cudaMalloc(&c->cd_rows, sizeof(int) * 1024)); CUDA_CHECK_RET(c, cudaMalloc(&c->cd_tot, sizeof(int) * MAXLVL)); }
    if (n > c->cd_in_cap) {
        CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
        if (c->cd_in) cudaFree(c->cd_in);
        CUDA_CHECK_RET(c, cudaMalloc(&c->cd_in, sizeof(float) * 4 * (size_t) n));
        c->cd_in_cap = n;
    }
    const size_t np0 = (size_t) c->lw[0] * c->lh[0];
    CUDA_CHECK_RET(c, cudaMemsetAsync(c->cd_id[0], 0, 4 * np0, c->stream));
    CUDA_CHECK_RET(c, cudaMemsetAsync(c->cd_ws[0], 0, 4 * np0, c->stream));
    if (n > 0) {
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->cd_in, centerProjectedTo3, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, c->stream));
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->cd_in + 3 * (size_t) n, HdiF, sizeof(float) * n, cudaMemcpyHostToDevice, c->stream));
        k_cd_scatter<<<(n + 255) / 256, 256, 0, c->stream>>>(n, c->cd_in, c->cd_in + 3 * (size_t) n, c->cd_id[0], c->cd_ws[0], c->lw[0], c->lh[0]);
        LAUNCH_CHECK(c);
    }
    for (int l = 1; l < c->levels; l++) {
        const int npx = c->lw[l] * c->lh[l];
        k_cd_down<<<(npx + 255) / 256, 256, 0, c->stream>>>(c->cd_id[l - 1], c->cd_ws[l - 1], c->cd_id[l], c->cd_ws[l], c->lw[l], c->lh[l], c->lw[l - 1]);
        LAUNCH_CHECK(c);
    }
    for (int l = 0; l < c->levels; l++) {
        const int npx = c->lw[l] * c->lh[l];
        CUDA_CHECK_RET(c, cudaMemcpyAsync(c->cd_bak[l], c->cd_ws[l], 4 * (size_t) npx, cudaMemcpyDeviceToDevice, c->stream));
        k_cd_dilate<<<(npx + 255) / 256, 256, 0, c->stream>>>(c->cd_id[l], c->cd_ws[l], c->cd_bak[l], c->lw[l], c->lh[l], l < 2 ? 1 : 0);
        LAUNCH_CHECK(c);
    }
    for (int l = 0; l < c->levels; l++) {
        const int npx = c->lw[l] * c->lh[l];
        k_cd_rowcount<<<c->lh[l], 128, 0, c->stream>>>(c->cd_id[l], c->cd_ws[l], c->img[ref_slot][l], c->lw[l], c->lh[l], c->cd_pos[l], c->cd_rows);
        LAUNCH_CHECK(c);
        k_cd_rowscan<<<1, 1024, 0, c->stream>>>(c->cd_rows, c->lh[l], c->cd_tot + l);
        LAUNCH_CHECK(c);
        k_cd_emit<<<(npx + 255) / 256, 256, 0, c->stream>>>(c->cd_id[l], c->cd_ws[l], c->img[ref_slot][l], c->cd_pos[l], c->cd_rows, c->lw[l], c->lh[l],
                                                             c->trk_pc[l][0], c->trk_pc[l][1], c->trk_pc[l][2], c->trk_pc[l][3]);
        LAUNCH_CHECK(c);
    }
    int tot[MAXLVL];
    CUDA_CHECK_RET(c, cudaMemcpyAsync(tot, c->cd_tot, sizeof(int) * c->levels, cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK_RET(c, cudaStreamSynchronize(c->stream));
    for (int l = 0; l < c->levels; l++) c->trk[l].n = tot[l];
    return LDSO_B200_OK;
}
