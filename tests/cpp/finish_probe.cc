// TEST INFRASTRUCTURE ONLY: the end of FullSystem::optimize (FullSystem.cc:833-863) driven on the oracle's own Window, compiled by
// tests/finish_oracle.py together with the oracle's sources (oracle/*.cc, unmodified) into a temporary shared object. Every step is
// the oracle's pinned code -- Frame::setState / setStateZero (FrameHessian.h:78-91, FrameHessian.cc:11-42), setAdjointsF,
// setPrecalcValues, linearizeAll(true) with its relBS / maxRelBaseline and dropResidual (FullSystem.cc:1494-1530) -- only the few
// lines of FullSystem.cc's driver that the oracle does not expose are restated here.
#include "../../oracle/ba.h"
#include <algorithm>
#include <cstring>

using namespace oracle;

extern "C" {

// The residual states a loop left behind (state_state, state_energy) and, from them, the activeResiduals optimize() collected at its
// start (FullSystem.cc:735-745: the non-linearised residuals of the window's points), without resetOOB. For a window rebuilt from
// another implementation's loop results.
void finish_probe_set_residuals(void *o, const int *state, const double *energy) {
    Window *W = (Window *) o;
    for (size_t r = 0; r < W->residuals.size(); r++) {
        Residual &R = W->residuals[r];
        R.state_state = (ResState) state[r];
        R.state_energy = energy[r];
        // applyRes(true) left isActiveAndIsGoodNEW = (NewState == IN); an OOB residual kept the false it got when it went OOB
        R.isActiveAndIsGoodNEW = state[r] == RS_IN;
    }
    W->activeResiduals.clear();
    for (auto &p : W->points)
        for (int ri : p.residuals)
            if (!W->residuals[ri].isLinearized) W->activeResiduals.push_back(ri);
}

// FullSystem.cc:833-863 on the window as the loop left it. Returns lastEnergyP of linearizeAll(true). Outputs: the newest frame's new
// evaluation point (row-major R, t) and state_zero; per point the maxRelBaseline this pass produced (it starts from 0 here, so a point
// without an active residual reports 0) and the count of its residuals still active (numGoodResiduals' increment); per residual the
// state and whether linearizeAll removed it (ef->dropResidual); EnergyFunctional::resInA.
double finish_probe_run(void *o, double evalR[9], double evalT[3], double state_zero[10], float *maxRelBaseline, int *numGood,
                        int *state, unsigned char *dropped, int *resInA) {
    Window *W = (Window *) o;
    Frame &f = W->frames.back();
    // :833-836  newStateZero; setEvalPT(PRE_worldToCam, newStateZero) = evalPT, setState, setStateZero (FrameHessian.h:106-111)
    double nsz[10];
    memset(nsz, 0, sizeof(nsz));
    nsz[6] = f.state[6];
    nsz[7] = f.state[7];
    f.worldToCam_evalPT = f.PRE_worldToCam;
    f.setState(nsz);
    f.setStateZero(nsz);
    // :838-841
    W->setAdjointsF();
    W->setPrecalcValues();
    // :843  linearizeAll(true)
    for (auto &p : W->points) p.maxRelBaseline = 0;
    const std::vector<std::vector<int>> before = [&] { std::vector<std::vector<int>> b; for (auto &p : W->points) b.push_back(p.residuals); return b; }();
    const double e = W->linearizeAll(true);
    M3 R = f.worldToCam_evalPT.rotationMatrix();
    memcpy(evalR, R.m, 72);
    for (int i = 0; i < 3; i++) evalT[i] = f.worldToCam_evalPT.t[i];
    memcpy(state_zero, f.state_zero, 80);
    for (size_t p = 0; p < W->points.size(); p++) {
        const Point &P = W->points[p];
        maxRelBaseline[p] = P.maxRelBaseline;
        int n = 0;
        for (int ri : P.residuals) if (!W->residuals[ri].isLinearized && W->residuals[ri].isActive()) n++;
        numGood[p] = n;
        for (int ri : before[p]) dropped[ri] = std::find(P.residuals.begin(), P.residuals.end(), ri) == P.residuals.end() ? 1 : 0;
    }
    for (size_t r = 0; r < W->residuals.size(); r++) state[r] = W->residuals[r].state_state;
    *resInA = W->resInA;
    return e;
}

}  // extern "C"
