// The end of FullSystem::optimize on the device (FullSystem.cc:833-863): the newest keyframe's new evaluation point with the adjoints
// and pair records it implies, the per-point bookkeeping of linearizeAll(true) (FullSystem.cc:1494-1530), and the returned RMSE.
// ldso_b200_optimize_finish launches k_finish_frames -> K1 (linearize + applyRes(true)) -> K2a/K2b (energy, setNewFrameEnergyTH)
// -> k_finish_points -> k_finish_tail on the context's stream.
#pragma once
#include "common.cuh"
#include "se3_math.cuh"
#include "ba_k3.cuh"

// per-point outputs of the fixed linearisation (device arrays of the window)
struct FinishBufs {
    float *pt_relBS_max;     // [nP] max relBS over the point's residuals still active after applyRes(true), 0 if none
    int *pt_n_good;          // [nP] number of those residuals (numGoodResiduals increment)
    uint8_t *res_dropped;    // [nR] 1 = ef->dropResidual (active set, not active after applyRes(true))
    float *rmse;             // sqrtf((float) (energy / (patternNum * resInA of the last solve)))
    int *is_lost;            // !isfinite(energy)
};

// One CTA of 128 threads.
//   FullSystem.cc:833-836  newStateZero = 0 except [6..7] = the newest frame's state[6..7];
//                          setEvalPT(PRE_worldToCam, newStateZero) (FrameHessian.h:107-112): eval pose := current pose,
//                          state = state_zero = newStateZero
//   FullSystem.cc:838-841  EnergyFunctional::setAdjointsF for every pair (EnergyFunctional.cc:431-489), setPrecalcValues
//                          (FrameFramePrecalc::Set for every pair and setDeltaF)
// The newest frame's null spaces (FrameHessian::setStateZero) feed only the next orthogonalize; they and the projector are not
// rebuilt here, which is why the solve entry points refuse to run until the next set_frames.
__global__ void __launch_bounds__(128) k_finish_frames(WinState *ws) {
    __shared__ K3Frames S;
    __shared__ double sR[MAXF][9], sT[MAXF][3];
    stage_in(&S, ws);
    const int nF = ws->nF, tid = threadIdx.x;
    if (tid == 0) {
        FrameDev &f = S.fr[nF - 1];
        for (int i = 0; i < 9; i++) f.evalR[i] = f.preR[i];
        for (int i = 0; i < 3; i++) f.evalT[i] = f.preT[i];
        const double a = f.state[6], b = f.state[7];
        for (int i = 0; i < 10; i++) f.state[i] = f.state_zero[i] = 0.0;
        f.state[6] = f.state_zero[6] = a;
        f.state[7] = f.state_zero[7] = b;
    }
    __syncthreads();
    if (tid < nF) {
        for (int i = 0; i < 9; i++) sR[tid][i] = S.fr[tid].evalR[i];
        for (int i = 0; i < 3; i++) sT[tid][i] = S.fr[tid].evalT[i];
    }
    __syncthreads();
    // setAdjointsF: hostToTarget = target.evalPT * host.evalPT^-1; AH = -Adj^T (pose block), AT = I; then the affine entries and
    // the SCALE_* row scaling, in double, with float copies for the residual-side products
    for (int q = tid; q < nF * nF; q += blockDim.x) {
        const int h = q % nF, t = q / nF;
        double R[9], tt[3];
        se3_mul_inv(sR[t], sT[t], sR[h], sT[h], R, tt);
        double O[9], tR[9];
        hat3(tt, O);
        m3_mul(O, R, tR);
        double *AH = ws->adHost[q], *AT = ws->adTarget[q];
        for (int i = 0; i < 64; i++) AH[i] = AT[i] = 0.0;
        for (int i = 0; i < 8; i++) AH[i * 8 + i] = AT[i * 8 + i] = 1.0;
        // Adj = [R, hat(t) R; 0, R] (row-major 6x6); AH(i, j) = -Adj(j, i)
        for (int i = 0; i < 6; i++)
            for (int j = 0; j < 6; j++) {
                double adj;
                if (j < 3) adj = (i < 3) ? R[j * 3 + i] : tR[j * 3 + (i - 3)];
                else adj = (i < 3) ? 0.0 : R[(j - 3) * 3 + (i - 3)];
                AH[i * 8 + j] = -adj;
            }
        const FrameDev &fh = S.fr[h], &ft = S.fr[t];
        float eF = fh.ab_exposure, eT = ft.ab_exposure;
        if (eF == 0 || eT == 0) eT = eF = 1;
        const float a0h = (float) (fh.state_zero[6] * SCALE_A), a0t = (float) (ft.state_zero[6] * SCALE_A);
        // exp of the float difference, rounded once to float: the correctly rounded expf, which set_frames' host expf (glibc, not
        // guaranteed correctly rounded) gives in all but rare cases; the device's expf is further off (up to 2 ulp)
        const float affLL0 = (float) exp((double) (a0t - a0h)) * eT / eF;
        AT[6 * 8 + 6] = -affLL0; AH[6 * 8 + 6] = affLL0; AT[7 * 8 + 7] = -1; AH[7 * 8 + 7] = affLL0;
        for (int j = 0; j < 8; j++) {
            for (int i = 0; i < 3; i++) { AH[i * 8 + j] *= SCALE_XI_TRANS; AT[i * 8 + j] *= SCALE_XI_TRANS; }
            for (int i = 3; i < 6; i++) { AH[i * 8 + j] *= SCALE_XI_ROT; AT[i * 8 + j] *= SCALE_XI_ROT; }
            AH[6 * 8 + j] *= SCALE_A; AT[6 * 8 + j] *= SCALE_A;
            AH[7 * 8 + j] *= SCALE_B; AT[7 * 8 + j] *= SCALE_B;
        }
        for (int i = 0; i < 64; i++) { ws->adHostF[q][i] = (float) AH[i]; ws->adTargetF[q][i] = (float) AT[i]; }
    }
    __syncthreads();      // frames_adHTdelta reads the float adjoints this CTA just wrote
    frames_refresh(&S, ws, true, &ws->adHostF[0][0], &ws->adTargetF[0][0]);
    stage_out(&S, ws);
}

// One thread per point, after K1 ran linearize + applyRes(true) over the window's non-linearised residuals (FullSystem.cc:1505-1527).
// A point's residuals are contiguous, so each point's max and count are formed in residual order without atomics.
//   relBS = 0.01 * |pi(KRKi (u, v, 1)) - pi(KRKi (u, v, 1) + Kt idepth_scaled)|  with the pair records of the NEW precalc
__global__ void k_finish_points(DevWindow d, const WinState *__restrict__ ws, FinishBufs fb) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.nP) return;
    const int nF = ws->nF, host = d.pt_host[p];
    const float u = d.pt_u[p], v = d.pt_v[p], id = d.pt_idepth[p] * SCALE_IDEPTH;
    float mx = 0.f;
    int n_good = 0;
    for (int r = d.pt_res_begin[p]; r < d.pt_res_begin[p + 1]; r++) {
        uint8_t dropped = 0;
        if (!d.res_lin[r]) {
            if (d.res_active[r]) {
                const PairRec &pc = ws->pair[host + nF * d.res_target[r]];
                float inf[3], ptp[3];
                for (int i = 0; i < 3; i++) {
                    float s = __fmul_rn(pc.KRKi[i * 3], u);
                    s = __fadd_rn(s, __fmul_rn(pc.KRKi[i * 3 + 1], v));
                    s = __fadd_rn(s, pc.KRKi[i * 3 + 2]);
                    inf[i] = s;
                    ptp[i] = __fadd_rn(s, __fmul_rn(pc.Kt[i], id));
                }
                const float ex = __fsub_rn(__fdiv_rn(inf[0], inf[2]), __fdiv_rn(ptp[0], ptp[2]));
                const float ey = __fsub_rn(__fdiv_rn(inf[1], inf[2]), __fdiv_rn(ptp[1], ptp[2]));
                const float relBS = (float) (0.01 * (double) __fsqrt_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey))));
                if (relBS > mx) mx = relBS;
                n_good++;
            } else {
                dropped = 1;
            }
        }
        fb.res_dropped[r] = dropped;
    }
    fb.pt_relBS_max[p] = mx;
    fb.pt_n_good[p] = n_good;
}

// One warp: the value FullSystem::optimize returns (FullSystem.cc:863) and its lost test (:845-849). lastEnergy[1..2] are
// always 0 (linearizeAll returns (lastEnergyP, 0, 0)), so only the energy decides.
__global__ void __launch_bounds__(32) k_finish_tail(const WinState *ws, FinishBufs fb) {
    if (threadIdx.x != 0) return;
    const double e = ws->energy;
    *fb.rmse = sqrtf((float) (e / (double) (LDSO_B200_PATTERN * ws->resInA_solved)));
    *fb.is_lost = isfinite(e) ? 0 : 1;
}
