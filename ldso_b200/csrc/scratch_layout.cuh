// Layout of the C ABI's scratch and staging blocks (api.cu). Each block has one region list: a function that takes the block's regions
// from an Arena and fills the kernel's argument struct with them. Run on an Arena without a base, the list sizes the block (the
// pointers it fills are then offsets from the block's start); run on the block, it carves it. A group of arrays that one copy or one
// memset covers is taken as one region and split inside, so that it stays contiguous whatever the sizes.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <algorithm>

#include "corners.cuh"
#include "pixsel.cuh"
#include "posegraph.cuh"
#include "tracker_kernels.cuh"
#include "trace_types.h"
#include "immature_store.h"

struct Arena {
    uintptr_t base = 0;            // 0: a sizing pass
    size_t off = 0;                // bytes taken so far: the block's size at the end of a sizing pass
    Arena() = default;
    explicit Arena(void *block) : base((uintptr_t) block) {}
    // count T's at the next multiple of align (a power of two, at least alignof(T)): base + offset, or the offset in a sizing pass
    template <typename T = char>
    T *take(size_t count, size_t align = 16) {
        off = (off + align - 1) & ~(align - 1);
        T *p = (T *) (base + off);
        off += sizeof(T) * count;
        return p;
    }
};

// ---------------------------------------------------------------------------------------------- detect_corners (corners.cuh)
// The output block: n and scoreTH in a 16-byte header, then u | v | score | angle (cap each), is_corner, the descriptors. One copy
// brings it back, and corners_read parses the pinned copy with the same split.
inline size_t corner_out_bytes(size_t cap) { return 16 + cap * CORNER_FEATURE_BYTES; }
inline void corner_split(char *o, int cap, CornerArgs &a) {
    a.hdr = (int *) o;
    a.cap = cap;
    a.u = (float *) (o + 16); a.v = a.u + cap; a.score = a.v + cap; a.angle = a.score + cap;
    a.is_corner = (uint8_t *) (a.angle + cap); a.desc = a.is_corner + cap;
}
// The device block, sized at context creation for one feature per pixel (px = w*h, the most any density gives): the output block
// (split with the call's capacity), the ORB pattern and B, then the per-cell scratch. The pattern and B sit at offsets that depend on
// px alone: set_orb_pattern writes the pattern once per context.
struct CornerFixed { int *pattern; float *B; };
inline CornerFixed corner_regions(Arena &A, size_t px, int cap, CornerArgs &a) {
    corner_split(A.take(corner_out_bytes(px)), cap, a);
    CornerFixed f;
    f.pattern = A.take<int>(1024);
    f.B = A.take<float>(256);
    a.keys = A.take<unsigned long long>(px);
    a.cell_count = A.take<int>(px);
    a.cell_off = A.take<int>(px);
    a.pick_px = A.take<int>(px);
    a.cell_max = A.take<float>(px);
    a.pick_score = A.take<float>(px);
    a.initial = A.take<uint8_t>(px);
    return f;
}

// ---------------------------------------------------------------------------------------------- pixel selection (pixsel.cuh)
// The output lists, cap entries each: x, y as int32 and type as uint8 (select_pixels), or u, v, my_type as floats
// (make_new_traces_pixels), from the same start
inline void pixsel_split(char *o, size_t cap, bool traces, PixselArgs &a) {
    a.sx = a.sy = nullptr; a.stype = nullptr; a.fu = a.fv = a.ftype = nullptr;
    if (traces) { a.fu = (float *) o; a.fv = a.fu + cap; a.ftype = a.fv + cap; }
    else { a.sx = (int32_t *) o; a.sy = a.sx + cap; a.stype = (uint8_t *) (a.sy + cap); }
}
// The device block, sized by w and h alone (potential 1: one pot cell per pixel), so that randomPattern, uploaded once with the block,
// stays put. The output lists take 12 bytes for every pixel, enough for either kind.
struct PixselFixed { float *B; uint8_t *rp; };
inline PixselFixed pixsel_regions(Arena &A, int w, int h, bool traces, PixselArgs &a) {
    const size_t px = (size_t) w * h, cells = (size_t) (w / 32) * (h / 32);
    PixselFixed f;
    a.hdr = A.take<int>(PIXSEL_HDR_INTS);
    f.B = A.take<float>(256);
    f.rp = A.take<uint8_t>(px);
    a.map = A.take<uint8_t>(px);
    a.dir = A.take<uint8_t>(px);
    a.mask = A.take<uint16_t>(px);
    a.ths = A.take<float>(cells);
    a.thsS = A.take<float>(cells);
    a.rowcnt = A.take<int>(h);
    a.rowoff = A.take<int>(h);
    a.list = A.take<int>(px);
    pixsel_split(A.take(12 * px), px, traces, a);
    return f;
}
// The pinned read-back block: the header (64 bytes), then n entries of the lists, then (select_pixels) the map. Allocated for n = w*h
// and either kind; the header's place does not depend on n.
inline void pixsel_pin_regions(Arena &A, size_t n, size_t px, bool traces, PixselArgs &h) {
    h.hdr = A.take<int>(PIXSEL_HDR_INTS);
    pixsel_split(A.take((traces ? 12 : 9) * n), n, traces, h);
    h.map = traces ? nullptr : A.take<uint8_t>(px, 1);
}

// ---------------------------------------------------------------------------------------------- select_activation
// The nine candidate arrays as one region, in the order u, v, idmin, idmax, quality, interval, my_type, status, host, then the frame
// flags: the same on the device and in the pinned stage, so that one copy moves the candidates
inline void actsel_inputs(Arena &A, size_t N, ActSelArgs &a) {
    float *f = A.take<float>(9 * N);
    a.u = f; a.v = f + N; a.idmin = f + 2 * N; a.idmax = f + 3 * N; a.quality = f + 4 * N; a.interval = f + 5 * N; a.my_type = f + 6 * N;
    a.status = (const int *) (f + 7 * N); a.host = (const int *) (f + 8 * N);
    a.flagged = A.take<unsigned char>(MAXF);
}
// the device block (the one-shot scratch), N = max(n, 1) candidates on a w x h image
inline void actsel_regions(Arena &A, int w, int h, size_t N, ActSelArgs &a) {
    const size_t cells = (size_t) (w >> 1) * (h >> 1);
    actsel_inputs(A, N, a);
    a.front0 = A.take<int>(cells);
    a.front1 = A.take<int>(cells);
    a.pre_idx = A.take<int>(N);
    a.pre_frac = A.take<float>(N);
    a.pre_thresh = A.take<float>(N);
    a.map_bytes = (int) ((cells + 3) & ~(size_t) 3);
    a.map = A.take<unsigned char>(a.map_bytes);
    a.action = A.take<unsigned char>(N);
    a.dbg = A.take<long long>(4);
}
// the pinned stage: the inputs, then the action bytes read back
inline void actsel_stage_regions(Arena &A, size_t N, ActSelArgs &s) {
    actsel_inputs(A, N, s);
    s.action = A.take<unsigned char>(N);
}

// ---------------------------------------------------------------------------------------------- immature-point store
// The 64 bytes both of its blocks hold: the frame flags at +0, the header at +16, traceNewCoarse's counters (7) at +32
struct ImmSmall { unsigned char *flags; int *hdr, *counts; };
static_assert(MAXF <= 16, "the frame flags fit in the small region's first 16 bytes");
inline ImmSmall imm_small(Arena &A) {
    char *s = A.take(64);
    return {(unsigned char *) s, (int *) (s + 16), (int *) (s + 32)};
}
// activate_immature's device scratch, sized for every candidate of a full window ((MAXF - 1) segments of cap entries)
inline ImmSmall imm_scratch_regions(Arena &A, int cap, int w, int h, StoreActArgs &P, ActSelArgs &S) {
    const size_t M = (size_t) (MAXF - 1) * cap, cells = (size_t) (w >> 1) * (h >> 1);
    // the gathered candidates and k_activation_select's terms
    P.c_u = A.take<float>(M); P.c_v = A.take<float>(M); P.c_idmin = A.take<float>(M); P.c_idmax = A.take<float>(M);
    P.c_quality = A.take<float>(M); P.c_interval = A.take<float>(M); P.c_type = A.take<float>(M);
    P.c_status = A.take<int>(M); P.c_host = A.take<int>(M); P.c_index = A.take<int>(M); P.c_sel = A.take<int>(M);
    S.pre_idx = A.take<int>(M); S.pre_frac = A.take<float>(M); S.pre_thresh = A.take<float>(M);
    // the selected candidates and the activation LM's results
    P.s_u = A.take<float>(M); P.s_v = A.take<float>(M); P.s_idmin = A.take<float>(M); P.s_idmax = A.take<float>(M);
    P.s_energyTH = A.take<float>(M); P.s_idepth = A.take<float>(M); P.s_host = A.take<int>(M); P.s_ok = A.take<int>(M);
    P.s_color8 = A.take<float>(8 * M); P.s_weights8 = A.take<float>(8 * M);
    P.s_res = A.take<unsigned char>(M * MAXF);
    P.action = A.take<unsigned char>(M);
    // the distance map and its BFS frontiers
    S.front0 = A.take<int>(cells);
    S.front1 = A.take<int>(cells);
    S.map_bytes = (int) ((cells + 3) & ~(size_t) 3);
    S.map = A.take<unsigned char>(S.map_bytes);
    const ImmSmall s = imm_small(A);
    S.flagged = s.flags;
    P.hdr = s.hdr;
    P.rec = A.take<ImmRecord>(M);
    return s;
}
// The pinned block: the 64 bytes above, then the body: one segment (immature_read), the released records (activate_immature) or
// immature_seed's staged coordinates
struct ImmPin { ImmSmall small; char *body; };
inline ImmPin imm_pin_regions(Arena &A, int cap) {
    ImmPin p;
    p.small = imm_small(A);
    p.body = A.take(std::max((size_t) IMM_SEG_WORDS * 4 * cap, (size_t) (MAXF - 1) * cap * sizeof(ImmRecord)));
    return p;
}

// ---------------------------------------------------------------------------------------------- the one-shot entry points
// Each lists the one-shot scratch (trace_buf) of one call.
struct EnergyScratch { double *part, *out; unsigned *counter; };
inline void calc_energies_regions(Arena &A, size_t nblocks, EnergyScratch &s) {
    s.part = A.take<double>(nblocks);
    s.out = A.take<double>(2);
    s.counter = A.take<unsigned>(1);
}

// immature_init: the outputs are one region, cleared by one memset
struct ImmInitScratch { float *u, *v, *color8, *weights8, *gradH4, *energyTH; };
inline void immature_init_regions(Arena &A, size_t N, ImmInitScratch &s) {
    s.u = A.take<float>(N);
    s.v = A.take<float>(N);
    float *o = A.take<float>(21 * N);
    s.color8 = o; s.weights8 = o + 8 * N; s.gradH4 = o + 16 * N; s.energyTH = o + 20 * N;
}

// trace_immature: N candidates, H host keyframes
inline void trace_immature_regions(Arena &A, size_t N, size_t H, TraceArgs &T) {
    T.u = A.take<float>(N); T.v = A.take<float>(N);
    T.color8 = A.take<float>(8 * N); T.weights8 = A.take<float>(8 * N); T.gradH4 = A.take<float>(4 * N); T.energyTH = A.take<float>(N);
    T.idepth_min = A.take<float>(N); T.idepth_max = A.take<float>(N); T.quality = A.take<float>(N);
    T.uv2 = A.take<float>(2 * N); T.interval = A.take<float>(N);
    T.host = A.take<int>(N); T.status = A.take<int>(N);
    T.KRKi9 = A.take<float>(9 * H); T.Kt3 = A.take<float>(3 * H); T.aff2 = A.take<float>(2 * H);
}

// optimize_immature: N candidates in a window of nF frames
struct OptImmScratch { float *u, *v, *idmin, *idmax, *color8, *weights8, *energyTH, *idepth; int *host, *ok; unsigned char *res_state; };
inline void optimize_immature_regions(Arena &A, size_t N, size_t nF, OptImmScratch &s) {
    s.u = A.take<float>(N); s.v = A.take<float>(N); s.idmin = A.take<float>(N); s.idmax = A.take<float>(N);
    s.color8 = A.take<float>(8 * N); s.weights8 = A.take<float>(8 * N); s.energyTH = A.take<float>(N);
    s.host = A.take<int>(N); s.ok = A.take<int>(N); s.idepth = A.take<float>(N);
    s.res_state = A.take<unsigned char>(N * nF);
}

// init_calc_res: N points, `grid` CTAs. energy_new, maxstep, lastHessian_new and Jb are one region, cleared by one memset; the
// counter's region is cleared by a 16-byte memset.
inline void init_calc_res_regions(Arena &A, size_t N, size_t grid, InitArgs &a) {
    a.u = A.take<float>(N); a.v = A.take<float>(N); a.idepth_new = A.take<float>(N); a.iR = A.take<float>(N);
    a.energy2 = A.take<float>(2 * N); a.outlierTH = A.take<float>(N);
    float *o = A.take<float>(14 * N);
    a.energy_new2 = o; a.maxstep = o + 2 * N; a.lastHessian_new = o + 3 * N; a.Jb = o + 4 * N;
    a.partials = A.take<float>(grid * INIT_NACC);
    a.counter = A.take<unsigned>(4);
    a.out = A.take<double>(INIT_NACC);
    a.isGood = A.take<unsigned char>(N);
    a.isGood_new = A.take<unsigned char>(N);
}

// tracker_track_batch: n hypotheses and their results
struct TrackBatchScratch { TrkHypothesis *hyp; TrkTrackOut *out; };
inline void track_batch_regions(Arena &A, size_t n, TrackBatchScratch &s) {
    s.hyp = A.take<TrkHypothesis>(n);
    s.out = A.take<TrkTrackOut>(n);
}

// ---------------------------------------------------------------------------------------------- pose graph (posegraph.cuh)
// posegraph_optimize's device block, allocated per call and cleared as a whole
inline void posegraph_regions(Arena &A, int nV, int nE, PgGraph &g) {
    const size_t V = nV, E = nE, nb = std::max((nV + PG_WARPS - 1) / PG_WARPS, (nE + PG_WARPS - 1) / PG_WARPS);
    g.q = A.take<double>(4 * V); g.t = A.take<double>(3 * V);
    g.ei = A.take<int>(E); g.ej = A.take<int>(E);
    g.mq = A.take<double>(4 * E); g.mt = A.take<double>(3 * E); g.info = A.take<double>(49 * E);
    g.Hii = A.take<double>(49 * E); g.Hij = A.take<double>(49 * E); g.Hjj = A.take<double>(49 * E);
    g.bi = A.take<double>(7 * E); g.bj = A.take<double>(7 * E); g.chi2e = A.take<double>(E);
    g.inc_begin = A.take<int>(V + 1); g.inc = A.take<int>(2 * E);
    g.D = A.take<double>(49 * V); g.Dinv = A.take<double>(49 * V); g.b = A.take<double>(7 * V);
    g.x = A.take<double>(7 * V); g.r = A.take<double>(7 * V); g.z = A.take<double>(7 * V);
    g.p0 = A.take<double>(7 * V); g.p1 = A.take<double>(7 * V); g.Ap = A.take<double>(7 * V);
    g.part = A.take<double>(nb);
    g.scal = A.take<double>(8);
    g.counter = A.take<unsigned>(4);
}
