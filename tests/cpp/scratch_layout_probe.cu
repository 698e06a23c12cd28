// TEST INFRASTRUCTURE ONLY: checks the region lists of the C ABI's scratch and staging blocks (ldso_b200/csrc/scratch_layout.cuh) on
// the host, over a grid of sizes; compiled by tests/test_scratch_layout_cpu.py into a temporary shared object. No CUDA call runs.
// Each list is run as a sizing pass (the pointers it fills are offsets) and as a carving pass on a made-up base; every region a
// kernel or a copy uses is listed here with the extent it needs, independently of the list, and checked: inside the block, pairwise
// disjoint, aligned for its type, the contiguous groups contiguous, and the regions set once per context at fixed offsets.
#include "../../ldso_b200/csrc/scratch_layout.cuh"
#include <stdarg.h>
#include <stdio.h>
#include <string>
#include <vector>

namespace {

const uintptr_t kBase = (uintptr_t) 1 << 40;      // the carving pass's block

struct Region { std::string name; uintptr_t off; size_t bytes, align; };

struct Checker {
    std::string err;
    long long cases = 0;
    bool fail(const char *fmt, ...) {
        if (!err.empty()) return false;
        char buf[512];
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(buf, sizeof(buf), fmt, ap);
        va_end(ap);
        err = buf;
        return false;
    }
    // the regions of one block: inside [0, total), aligned for their type, pairwise disjoint (empty ones excepted)
    bool block(const char *what, const std::vector<Region> &R, size_t total) {
        cases++;
        for (const Region &r : R) {
            if (r.off > total || r.bytes > total - r.off)
                return fail("%s: %s [%zu, +%zu) outside the block of %zu bytes", what, r.name.c_str(), (size_t) r.off, r.bytes, total);
            if (r.off % r.align) return fail("%s: %s at %zu not aligned to %zu", what, r.name.c_str(), (size_t) r.off, r.align);
        }
        for (size_t i = 0; i < R.size(); i++)
            for (size_t j = i + 1; j < R.size(); j++) {
                const Region &a = R[i], &b = R[j];
                if (a.bytes && b.bytes && a.off < b.off + b.bytes && b.off < a.off + a.bytes)
                    return fail("%s: %s and %s overlap", what, a.name.c_str(), b.name.c_str());
            }
        return true;
    }
    bool expect(bool ok, const char *what, const char *msg) { return ok || fail("%s: %s", what, msg); }
};

// regions are collected as offsets from the block's start: `at` is the block's base in the pass that filled the pointers
struct Regions {
    uintptr_t at;
    std::vector<Region> R;
    template <typename T> void add(const char *name, const T *p, size_t count) {
        R.push_back({name, (uintptr_t) p - at, sizeof(T) * count, alignof(T)});
    }
};
// the carving pass gives the sizing pass's offsets on the block
bool same(Checker &K, const char *what, const Regions &a, const Regions &b) {
    if (a.R.size() != b.R.size()) return K.fail("%s: the passes list different regions", what);
    for (size_t i = 0; i < a.R.size(); i++)
        if (a.R[i].off != b.R[i].off) return K.fail("%s: %s differs between the sizing and the carving pass", what, a.R[i].name.c_str());
    return true;
}
template <typename T> uintptr_t off(const T *p) { return (uintptr_t) p; }

const int kSizes[][2] = {{64, 48}, {100, 75}, {320, 240}, {640, 480}, {635, 480}, {752, 480}, {1232, 368}, {1920, 1080}};
const size_t kN[] = {0, 1, 3, 64, 1001, 4096, 20000};

// ---------------------------------------------------------------------------------------------- corners
Regions corner_list(Arena &A, size_t px, int cap, CornerFixed &f) {
    CornerArgs a;
    f = corner_regions(A, px, cap, a);
    Regions r{A.base};
    r.add("hdr", a.hdr, 4); r.add("u", a.u, cap); r.add("v", a.v, cap); r.add("score", a.score, cap); r.add("angle", a.angle, cap);
    r.add("is_corner", a.is_corner, cap); r.add("desc", a.desc, 32 * (size_t) cap);
    r.add("pattern", f.pattern, 1024); r.add("B", f.B, 256);
    r.add("keys", a.keys, px); r.add("cell_count", a.cell_count, px); r.add("cell_off", a.cell_off, px); r.add("pick_px", a.pick_px, cap);
    r.add("cell_max", a.cell_max, px); r.add("pick_score", a.pick_score, cap); r.add("initial", a.initial, cap);
    return r;
}
bool check_corners(Checker &K) {
    for (const auto &s : kSizes) {
        const size_t px = (size_t) s[0] * s[1];
        Arena S0;
        CornerFixed f0;
        corner_list(S0, px, 0, f0);
        const size_t pin = corner_out_bytes(px);
        // capacities: the golden fixtures' (a few thousand at 640x480) and the extremes, up to one feature per pixel
        for (size_t cap : {(size_t) 0, (size_t) 1, (size_t) 807, (size_t) 2000, (size_t) 4437, (size_t) 9000, px / 3, px}) {
            if (cap > px) continue;
            Arena S, D((void *) kBase);
            CornerFixed fs, fd;
            const Regions rs = corner_list(S, px, (int) cap, fs), rd = corner_list(D, px, (int) cap, fd);
            if (!K.block("corners", rs.R, S.off) || !same(K, "corners", rs, rd)) return false;
            CornerArgs a;
            Arena S2;
            corner_regions(S2, px, (int) cap, a);
            // the output block: header, u | v | score | angle, is_corner, descriptor back to back, covered by one copy
            const uintptr_t o = off(a.hdr);
            bool ok = off(a.u) == o + 16 && off(a.v) == off(a.u) + 4 * cap && off(a.score) == off(a.v) + 4 * cap &&
                      off(a.angle) == off(a.score) + 4 * cap && off(a.is_corner) == off(a.angle) + 4 * cap &&
                      off(a.desc) == off(a.is_corner) + cap && off(a.desc) + 32 * cap == o + corner_out_bytes(cap);
            if (!K.expect(ok, "corners", "the output block is not contiguous")) return false;
            if (!K.expect(corner_out_bytes(cap) <= pin, "corners", "the pinned block is smaller than the output block")) return false;
            CornerArgs h;
            corner_split((char *) kBase, (int) cap, h);
            if (!K.expect(off(h.desc) - kBase == off(a.desc) - o, "corners", "the pinned split differs from the device's")) return false;
            if (!K.expect(off(fs.pattern) == off(f0.pattern) && off(fs.B) == off(f0.B) && S.off == S0.off, "corners",
                          "the ORB pattern or B moves with the capacity"))
                return false;
        }
    }
    return true;
}

// ---------------------------------------------------------------------------------------------- pixel selection
Regions pixsel_list(Arena &A, int w, int h, bool traces, PixselFixed &f) {
    PixselArgs a;
    f = pixsel_regions(A, w, h, traces, a);
    const size_t px = (size_t) w * h, cells = (size_t) (w / 32) * (h / 32);
    Regions r{A.base};
    r.add("hdr", a.hdr, PIXSEL_HDR_INTS); r.add("B", f.B, 256); r.add("rp", f.rp, px); r.add("map", a.map, px);
    r.add("dir", a.dir, px); r.add("mask", a.mask, px); r.add("ths", a.ths, cells); r.add("thsS", a.thsS, cells);
    r.add("rowcnt", a.rowcnt, h); r.add("rowoff", a.rowoff, h); r.add("list", a.list, px);
    if (traces) { r.add("fu", a.fu, px); r.add("fv", a.fv, px); r.add("ftype", a.ftype, px); }
    else { r.add("sx", a.sx, px); r.add("sy", a.sy, px); r.add("stype", a.stype, px); }
    return r;
}
Regions pixsel_pin_list(Arena &A, size_t n, size_t px, bool traces) {
    PixselArgs h;
    pixsel_pin_regions(A, n, px, traces, h);
    Regions r{A.base};
    r.add("hdr", h.hdr, PIXSEL_HDR_INTS);
    if (traces) { r.add("fu", h.fu, n); r.add("fv", h.fv, n); r.add("ftype", h.ftype, n); }
    else { r.add("sx", h.sx, n); r.add("sy", h.sy, n); r.add("stype", h.stype, n); r.add("map", h.map, px); }
    return r;
}
bool check_pixsel(Checker &K) {
    // the potential and the recursion do not enter the lists: w and h alone size and place every region
    for (const auto &s : kSizes) {
        const int w = s[0], h = s[1];
        const size_t px = (size_t) w * h;
        Arena P1, P2;
        pixsel_pin_list(P1, px, px, true);
        pixsel_pin_list(P2, px, px, false);
        const size_t pin = std::max(P1.off, P2.off);
        Regions first;
        size_t first_total = 0;
        for (bool traces : {false, true}) {
            Arena S, D((void *) kBase);
            PixselFixed fs, fd;
            const Regions rs = pixsel_list(S, w, h, traces, fs), rd = pixsel_list(D, w, h, traces, fd);
            if (!K.block("pixsel", rs.R, S.off) || !same(K, "pixsel", rs, rd)) return false;
            if (!traces) { first = rs; first_total = S.off; continue; }
            // both kinds of list start in the same place, and every other region (randomPattern among them) stays put
            bool ok = S.off == first_total;
            for (size_t i = 0; i + 3 < rs.R.size(); i++) ok = ok && rs.R[i].off == first.R[i].off;
            ok = ok && rs.R[rs.R.size() - 3].off == first.R[first.R.size() - 3].off;
            if (!K.expect(ok, "pixsel", "a region moves with the kind of list")) return false;
        }
        for (size_t n : {(size_t) 0, (size_t) 1, (size_t) 777, px / 2, px})
            for (bool traces : {false, true}) {
                Arena P;
                const Regions r = pixsel_pin_list(P, n, px, traces);
                if (!K.block("pixsel pinned", r.R, pin)) return false;
                if (!K.expect(r.R[0].off == 0 && r.R[1].off == 64, "pixsel pinned", "the lists do not follow the 64-byte header")) return false;
                if (!K.expect(r.R[2].off == 64 + 4 * n && r.R[3].off == 64 + 8 * n, "pixsel pinned", "the lists are not back to back")) return false;
            }
    }
    return true;
}

// ---------------------------------------------------------------------------------------------- select_activation
void actsel_inputs_add(Regions &r, const ActSelArgs &a, size_t N) {
    r.add("u", a.u, N); r.add("v", a.v, N); r.add("idmin", a.idmin, N); r.add("idmax", a.idmax, N); r.add("quality", a.quality, N);
    r.add("interval", a.interval, N); r.add("my_type", a.my_type, N); r.add("status", a.status, N); r.add("host", a.host, N);
    r.add("flagged", a.flagged, MAXF);
}
bool actsel_inputs_ok(Checker &K, const char *what, const ActSelArgs &a, size_t N) {
    const uintptr_t u = off(a.u);
    const bool ok = off(a.v) == u + 4 * N && off(a.idmin) == u + 8 * N && off(a.idmax) == u + 12 * N && off(a.quality) == u + 16 * N &&
                    off(a.interval) == u + 20 * N && off(a.my_type) == u + 24 * N && off(a.status) == u + 28 * N && off(a.host) == u + 32 * N &&
                    off(a.flagged) >= u + 36 * N;
    return K.expect(ok, what, "the nine candidate arrays are not one region in order, followed by the flags");
}
bool check_actsel(Checker &K) {
    for (const auto &s : kSizes)
        for (size_t n : kN) {
            const size_t N = std::max(n, (size_t) 1), cells = (size_t) (s[0] >> 1) * (s[1] >> 1);
            Regions rr[2];
            size_t total = 0;
            for (int pass = 0; pass < 2; pass++) {
                Arena A = pass ? Arena((void *) kBase) : Arena();
                ActSelArgs a;
                actsel_regions(A, s[0], s[1], N, a);
                Regions &r = rr[pass];
                r.at = A.base;
                actsel_inputs_add(r, a, N);
                r.add("front0", a.front0, cells); r.add("front1", a.front1, cells);
                r.add("pre_idx", a.pre_idx, N); r.add("pre_frac", a.pre_frac, N); r.add("pre_thresh", a.pre_thresh, N);
                r.add("map", a.map, a.map_bytes); r.add("action", a.action, N); r.add("dbg", a.dbg, 4);
                if (pass == 0) {
                    total = A.off;
                    if (!actsel_inputs_ok(K, "actsel", a, N)) return false;
                    if (!K.expect((size_t) a.map_bytes >= cells && a.map_bytes % 4 == 0, "actsel", "map_bytes")) return false;
                }
            }
            if (!K.block("actsel", rr[0].R, total) || !same(K, "actsel", rr[0], rr[1])) return false;
            Arena P;
            ActSelArgs h;
            actsel_stage_regions(P, N, h);
            Regions r{0};
            actsel_inputs_add(r, h, N);
            r.add("action", h.action, N);
            if (!K.block("actsel pinned", r.R, P.off) || !actsel_inputs_ok(K, "actsel pinned", h, N)) return false;
        }
    return true;
}

// ---------------------------------------------------------------------------------------------- immature-point store
void imm_small_add(Regions &r, const ImmSmall &s, uintptr_t start, const char *what, Checker &K, bool &ok) {
    r.add("flags", s.flags, MAXF); r.add("hdr", s.hdr, 4); r.add("counts", s.counts, 7);
    ok = ok && K.expect(off(s.flags) == start && off(s.hdr) == start + 16 && off(s.counts) == start + 32, what,
                        "the small region is not flags +0, header +16, counters +32");
}
bool check_imm(Checker &K) {
    for (const auto &s : kSizes)
        for (int cap : {1, 64, 800, 4437, 20000}) {
            const size_t M = (size_t) (MAXF - 1) * cap, cells = (size_t) (s[0] >> 1) * (s[1] >> 1);
            Regions rr[2];
            size_t total = 0;
            bool ok = true;
            for (int pass = 0; pass < 2; pass++) {
                Arena A = pass ? Arena((void *) kBase) : Arena();
                StoreActArgs P;
                ActSelArgs S;
                const ImmSmall sm = imm_scratch_regions(A, cap, s[0], s[1], P, S);
                Regions &r = rr[pass];
                r.at = A.base;
                r.add("c_u", P.c_u, M); r.add("c_v", P.c_v, M); r.add("c_idmin", P.c_idmin, M); r.add("c_idmax", P.c_idmax, M);
                r.add("c_quality", P.c_quality, M); r.add("c_interval", P.c_interval, M); r.add("c_type", P.c_type, M);
                r.add("c_status", P.c_status, M); r.add("c_host", P.c_host, M); r.add("c_index", P.c_index, M); r.add("c_sel", P.c_sel, M);
                r.add("pre_idx", S.pre_idx, M); r.add("pre_frac", S.pre_frac, M); r.add("pre_thresh", S.pre_thresh, M);
                r.add("s_u", P.s_u, M); r.add("s_v", P.s_v, M); r.add("s_idmin", P.s_idmin, M); r.add("s_idmax", P.s_idmax, M);
                r.add("s_energyTH", P.s_energyTH, M); r.add("s_idepth", P.s_idepth, M); r.add("s_host", P.s_host, M); r.add("s_ok", P.s_ok, M);
                r.add("s_color8", P.s_color8, 8 * M); r.add("s_weights8", P.s_weights8, 8 * M);
                r.add("s_res", P.s_res, M * MAXF); r.add("action", P.action, M);
                r.add("front0", S.front0, cells); r.add("front1", S.front1, cells); r.add("map", S.map, S.map_bytes);
                imm_small_add(r, sm, off(sm.flags), "imm scratch", K, ok);
                r.add("rec", P.rec, M);
                ok = ok && K.expect(S.flagged == sm.flags && P.hdr == sm.hdr, "imm scratch", "flags / header not in the small region");
                ok = ok && K.expect((size_t) S.map_bytes >= cells && S.map_bytes % 4 == 0, "imm scratch", "map_bytes");
                if (pass == 0) total = A.off;
            }
            if (!ok || !K.block("imm scratch", rr[0].R, total) || !same(K, "imm scratch", rr[0], rr[1])) return false;
            Arena H;
            const ImmPin p = imm_pin_regions(H, cap);
            Regions r{0};
            imm_small_add(r, p.small, 0, "imm pinned", K, ok);
            const size_t body = std::max({(size_t) IMM_SEG_WORDS * 4 * cap, M * sizeof(ImmRecord), (size_t) 12 * cap});
            r.add("body", p.body, body);
            if (!ok || !K.block("imm pinned", r.R, H.off)) return false;
            if (!K.expect(off(p.body) % alignof(ImmRecord) == 0, "imm pinned", "records misaligned")) return false;
        }
    return true;
}

// ---------------------------------------------------------------------------------------------- one-shot scratch
// runs `fill` (which lists the regions of a pass) on a sizing and a carving Arena and checks the block
template <typename F> bool one_shot(Checker &K, const char *what, F &&fill) {
    Arena S, D((void *) kBase);
    Regions rs{0}, rd{kBase};
    fill(S, rs);
    fill(D, rd);
    return K.block(what, rs.R, S.off) && same(K, what, rs, rd);
}
bool check_one_shot(Checker &K) {
    for (size_t n : kN) {
        const size_t N = n;
        if (!one_shot(K, "calc_energies", [&](Arena &A, Regions &r) {
                const size_t nb = std::max<size_t>(1, (n + 255) / 256);
                EnergyScratch e;
                calc_energies_regions(A, nb, e);
                r.add("part", e.part, nb); r.add("out", e.out, 2); r.add("counter", e.counter, 1);
            }))
            return false;
        bool ok = true;
        if (!one_shot(K, "immature_init", [&](Arena &A, Regions &r) {
                ImmInitScratch s;
                immature_init_regions(A, N, s);
                r.add("u", s.u, N); r.add("v", s.v, N); r.add("color8", s.color8, 8 * N); r.add("weights8", s.weights8, 8 * N);
                r.add("gradH4", s.gradH4, 4 * N); r.add("energyTH", s.energyTH, N);
                // one memset of 21 N floats from color8 clears the outputs
                ok = ok && off(s.weights8) == off(s.color8) + 32 * N && off(s.gradH4) == off(s.weights8) + 32 * N &&
                     off(s.energyTH) == off(s.gradH4) + 16 * N;
            }) || !K.expect(ok, "immature_init", "the outputs are not one region"))
            return false;
        for (size_t H : {1, 2, 7, 16})
            if (!one_shot(K, "trace_immature", [&](Arena &A, Regions &r) {
                    TraceArgs T;
                    trace_immature_regions(A, N, H, T);
                    r.add("u", T.u, N); r.add("v", T.v, N); r.add("color8", T.color8, 8 * N); r.add("weights8", T.weights8, 8 * N);
                    r.add("gradH4", T.gradH4, 4 * N); r.add("energyTH", T.energyTH, N); r.add("idepth_min", T.idepth_min, N);
                    r.add("idepth_max", T.idepth_max, N); r.add("quality", T.quality, N); r.add("uv2", T.uv2, 2 * N); r.add("interval", T.interval, N);
                    r.add("host", T.host, N); r.add("status", T.status, N);
                    r.add("KRKi9", T.KRKi9, 9 * H); r.add("Kt3", T.Kt3, 3 * H); r.add("aff2", T.aff2, 2 * H);
                }))
                return false;
        for (size_t nF = 2; nF <= MAXF; nF++)
            if (!one_shot(K, "optimize_immature", [&](Arena &A, Regions &r) {
                    OptImmScratch s;
                    optimize_immature_regions(A, N, nF, s);
                    r.add("u", s.u, N); r.add("v", s.v, N); r.add("idmin", s.idmin, N); r.add("idmax", s.idmax, N);
                    r.add("color8", s.color8, 8 * N); r.add("weights8", s.weights8, 8 * N); r.add("energyTH", s.energyTH, N);
                    r.add("host", s.host, N); r.add("ok", s.ok, N); r.add("idepth", s.idepth, N); r.add("res_state", s.res_state, N * nF);
                }))
                return false;
        const size_t grid = (N + INIT_THREADS / 8 - 1) / (INIT_THREADS / 8);
        if (!one_shot(K, "init_calc_res", [&](Arena &A, Regions &r) {
                InitArgs a;
                init_calc_res_regions(A, N, grid, a);
                r.add("u", a.u, N); r.add("v", a.v, N); r.add("idepth_new", a.idepth_new, N); r.add("iR", a.iR, N);
                r.add("energy2", a.energy2, 2 * N); r.add("outlierTH", a.outlierTH, N);
                r.add("energy_new2", a.energy_new2, 2 * N); r.add("maxstep", a.maxstep, N); r.add("lastHessian_new", a.lastHessian_new, N);
                r.add("Jb", a.Jb, 10 * N); r.add("partials", a.partials, grid * INIT_NACC); r.add("counter", a.counter, 4);
                r.add("out", a.out, INIT_NACC); r.add("isGood", a.isGood, N); r.add("isGood_new", a.isGood_new, N);
                // one memset of 14 N floats from energy_new clears energy_new, maxstep, lastHessian_new and Jb
                ok = ok && off(a.maxstep) == off(a.energy_new2) + 8 * N && off(a.lastHessian_new) == off(a.maxstep) + 4 * N &&
                     off(a.Jb) == off(a.lastHessian_new) + 4 * N;
            }) || !K.expect(ok, "init_calc_res", "energy_new .. Jb are not one region"))
            return false;
    }
    for (size_t n : {1, 2, 30, 81, 128})
        if (!one_shot(K, "track_batch", [&](Arena &A, Regions &r) {
                TrackBatchScratch s;
                track_batch_regions(A, n, s);
                r.add("hyp", s.hyp, n); r.add("out", s.out, n);
            }))
            return false;
    return true;
}

// ---------------------------------------------------------------------------------------------- pose graph
bool check_posegraph(Checker &K) {
    for (int nV : {2, 3, 17, 200, 2000})
        for (int nE : {1, 2, 16, 199, 5000}) {
            const size_t V = nV, E = nE, nb = std::max((nV + PG_WARPS - 1) / PG_WARPS, (nE + PG_WARPS - 1) / PG_WARPS);
            if (!one_shot(K, "posegraph", [&](Arena &A, Regions &r) {
                    PgGraph g;
                    posegraph_regions(A, nV, nE, g);
                    r.add("q", g.q, 4 * V); r.add("t", g.t, 3 * V); r.add("ei", g.ei, E); r.add("ej", g.ej, E);
                    r.add("mq", g.mq, 4 * E); r.add("mt", g.mt, 3 * E); r.add("info", g.info, 49 * E);
                    r.add("Hii", g.Hii, 49 * E); r.add("Hij", g.Hij, 49 * E); r.add("Hjj", g.Hjj, 49 * E);
                    r.add("bi", g.bi, 7 * E); r.add("bj", g.bj, 7 * E); r.add("chi2e", g.chi2e, E);
                    r.add("inc_begin", g.inc_begin, V + 1); r.add("inc", g.inc, 2 * E);
                    r.add("D", g.D, 49 * V); r.add("Dinv", g.Dinv, 49 * V); r.add("b", g.b, 7 * V); r.add("x", g.x, 7 * V);
                    r.add("r", g.r, 7 * V); r.add("z", g.z, 7 * V); r.add("p0", g.p0, 7 * V); r.add("p1", g.p1, 7 * V); r.add("Ap", g.Ap, 7 * V);
                    r.add("part", g.part, nb); r.add("scal", g.scal, 8); r.add("counter", g.counter, 4);
                }))
                return false;
        }
    return true;
}

}  // namespace

// Runs the checks of one block ("corners", "pixsel", "actsel", "immature_store", "one_shot", "posegraph"): the number of layouts
// checked, or -1 with the first failure in err.
extern "C" long long scratch_layout_check(const char *block, char *err, int errlen) {
    Checker K;
    const std::string b = block;
    bool ok;
    if (b == "corners") ok = check_corners(K);
    else if (b == "pixsel") ok = check_pixsel(K);
    else if (b == "actsel") ok = check_actsel(K);
    else if (b == "immature_store") ok = check_imm(K);
    else if (b == "one_shot") ok = check_one_shot(K);
    else if (b == "posegraph") ok = check_posegraph(K);
    else ok = K.fail("unknown block %s", block);
    if (ok) return K.cases;
    snprintf(err, errlen, "%s", K.err.c_str());
    return -1;
}
