// Immature-point kernels: separate translation unit, compiled with -fmad=false (see trace_types.h).
#include "trace_kernels.cuh"
#include "immature_store.cuh"

void launch_immature_init(int n, const float4 *img, int w, const float *u, const float *v, const TraceSettingsDev &S, float *color8,
                          float *weights8, float *gradH4, float *energyTH, cudaStream_t stream) {
    k_immature_init<<<(n + 127) / 128, 128, 0, stream>>>(n, img, w, u, v, S, color8, weights8, gradH4, energyTH);
}
void launch_trace_on(const TraceArgs &A, cudaStream_t stream) {
    k_trace_on<<<(A.n + KTR_WARPS - 1) / KTR_WARPS, 32 * KTR_WARPS, 0, stream>>>(A);
}
void launch_optimize_immature(int n, const WinState *ws, const float *u, const float *v, const int *host, const float *idmin, const float *idmax,
                              const float *color8, const float *weights8, const float *energyTH, int minObs, int *ok, float *idepth,
                              unsigned char *res_state, cudaStream_t stream) {
    k_optimize_immature<<<(n + KTR_WARPS - 1) / KTR_WARPS, 32 * KTR_WARPS, 0, stream>>>(n, ws, u, v, host, idmin, idmax, color8, weights8, energyTH,
                                                                                      minObs, ok, idepth, res_state);
}
size_t actsel_smem_bytes(const ActSelArgs &A) { return A.use_smem ? (size_t) A.map_bytes : 0; }
void launch_activation_select(const ActSelArgs &A, cudaStream_t stream) {
    const size_t smem = actsel_smem_bytes(A);
    static size_t configured = 0;
    if (smem > configured) { cudaFuncSetAttribute(k_activation_select, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) smem); configured = smem; }
    k_activation_select<<<1, ACTSEL_THREADS, smem, stream>>>(A);
}
void launch_init_calc_res(const InitArgs &A, cudaStream_t stream) {
    const int grid = (A.n + INIT_THREADS / 8 - 1) / (INIT_THREADS / 8);
    k_init_calc_res<<<grid, INIT_THREADS, 0, stream>>>(A);
}

void launch_store_seed(const int *n_dev, int n, const float *src_u, const float *src_v, const float *src_type, const float4 *img, int w,
                       const TraceSettingsDev &S, float *store, int cap, int slot, cudaStream_t stream) {
    k_store_seed<<<(n + 127) / 128, 128, 0, stream>>>(n_dev, n, src_u, src_v, src_type, img, w, S, store, cap, slot);
}
void launch_store_compact(float *store, int cap, int slot, int n, int *n_out, cudaStream_t stream) {
    k_store_compact<<<1, 1024, 0, stream>>>(store, cap, slot, n, n_out);
}
void launch_store_trace(const StoreTraceArgs &P, cudaStream_t stream) {
    k_store_trace<<<(P.begin[P.nseg] + KTR_WARPS - 1) / KTR_WARPS, 32 * KTR_WARPS, 0, stream>>>(P);
}
void launch_store_gather(const StoreActArgs &P, cudaStream_t stream) { k_store_gather<<<1, 1024, 0, stream>>>(P); }
void launch_store_pick(const StoreActArgs &P, cudaStream_t stream) { k_store_pick<<<1, 1024, 0, stream>>>(P); }
void launch_store_optimize(const StoreActArgs &P, int minObs, cudaStream_t stream) {
    k_store_optimize<<<(P.n + KTR_WARPS - 1) / KTR_WARPS, 32 * KTR_WARPS, 0, stream>>>(P, minObs);
}
void launch_store_apply(const StoreActArgs &P, cudaStream_t stream) { k_store_apply<<<1, 1024, 0, stream>>>(P); }
