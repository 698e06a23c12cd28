// FullSystem::optimize's loop exit on the device (FullSystem.cc:777-831): the kernel that closes every Gauss-Newton body of
// ldso_b200_gn_iterations_until and decides whether another body runs.
#pragma once
#include <cuda_runtime.h>
#include "common.cuh"

// device-resident loop parameters and counters (ctx->loop_dev); the host writes MAX / MIN and clears RUN before each call
enum { LOOP_MAX = 0, LOOP_MIN = 1, LOOP_RUN = 2, LOOP_CONT = 3, LOOP_WORDS = 4 };

// One warp, launched after the body's K2b. K3 of this body wrote ws->canbreak (doStepFromBackup's return value) and advanced
// *iteration_dev past the iteration it solved, so that iteration is *iteration_dev - 1 -- FullSystem's `iteration`.
//   cont = !(canbreak && iteration >= min) && bodies_run < max
// Inside the conditional WHILE node (use_cond != 0) the decision sets the node's condition; the host-driven form reads
// loop[LOOP_CONT] back instead. Both count the bodies run in loop[LOOP_RUN].
__global__ void __launch_bounds__(32) k_gn_continue(const WinState *ws, const int *iteration_dev, int *loop,
                                                    cudaGraphConditionalHandle cond, int use_cond) {
    pdl_wait();
    if (threadIdx.x != 0) return;
    const int run = loop[LOOP_RUN] + 1;
    const int iteration = *iteration_dev - 1;
    const int cont = (!(ws->canbreak && iteration >= loop[LOOP_MIN]) && run < loop[LOOP_MAX]) ? 1 : 0;
    loop[LOOP_RUN] = run;
    loop[LOOP_CONT] = cont;
    if (use_cond) cudaGraphSetConditional(cond, cont);
}
