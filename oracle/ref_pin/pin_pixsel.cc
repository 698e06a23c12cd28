// PIN of the pixel-selection restatement (../pixsel.cc) against the reference's own PixelSelector2.cc — TEST INFRASTRUCTURE ONLY, built
// by ../pixsel.mk where a reference checkout exists. The reference's src/frontend/PixelSelector2.cc, src/internal/FrameHessian.cc and
// src/Setting.cc are compiled unmodified (-Dprivate=public, against ../ref_shim). Two steps make the reference deterministic where it
// reads memory it never wrote, and state the restatement's rules in its own terms:
//   - after the selector is constructed, ths and thsSmoothed are zeroed across their whole allocation ((w/32)*(h/32) + 100 floats);
//   - after makeImages, rows 0 and h_l-1 of every absSquaredGrad[l] are zeroed.
// (gradHist's bins past 49 are read only when minGradHistCut >= 1; the allocation is zeroed too.) tests/pixsel_oracle.py loads this
// library beside liboracle_pixsel.so.
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <vector>

#include "frontend/PixelSelector2.h"

namespace ldso {
namespace internal { float wM3G, hM3G; int wG[ldso::PYR_LEVELS], hG[ldso::PYR_LEVELS]; }
Camera::Camera(double fx_, double fy_, double cx_, double cy_) { fx = fx_; fy = fy_; cx = cx_; cy = cy_; }
}

namespace {
struct RefFrame {
    shared_ptr<ldso::Frame> frame;
    RefFrame(int w, int h, const float *color, const float *B) {
        for (int l = 0; l < ldso::PYR_LEVELS; l++) { ldso::internal::wG[l] = w >> l; ldso::internal::hG[l] = h >> l; }
        ldso::internal::wM3G = w - 3; ldso::internal::hM3G = h - 3;
        auto HC = std::make_shared<ldso::internal::CalibHessian>(std::make_shared<ldso::Camera>(500, 500, w / 2.0, h / 2.0));
        if (B) for (int i = 0; i < 256; i++) HC->B[i] = B[i];
        frame = std::make_shared<ldso::Frame>();
        frame->frameHessian = std::make_shared<ldso::internal::FrameHessian>(frame);
        std::vector<float> col(color, color + (size_t) w * h);
        frame->frameHessian->makeImages(col.data(), HC);
        for (int l = 0; l < ldso::pyrLevelsUsed; l++) {
            const int wl = ldso::internal::wG[l], hl = ldso::internal::hG[l];
            float *a = frame->frameHessian->absSquaredGrad[l];
            std::fill(a, a + wl, 0.f);
            std::fill(a + (size_t) wl * (hl - 1), a + (size_t) wl * hl, 0.f);
        }
    }
    ~RefFrame() {
        frame->frameHessian->frame.reset();
        frame->frameHessian.reset();
    }
};
}  // namespace

extern "C" {

void *cref_pixsel_new(int w, int h) {
    ldso::PixelSelector *s = new ldso::PixelSelector(w, h);
    std::fill(s->ths, s->ths + (w / 32) * (h / 32) + 100, 0.f);
    std::fill(s->thsSmoothed, s->thsSmoothed + (w / 32) * (h / 32) + 100, 0.f);
    std::fill(s->gradHist, s->gradHist + 100 * (1 + w / 32) * (1 + h / 32), 0);
    return s;
}
void cref_pixsel_free(void *s) { delete (ldso::PixelSelector *) s; }
void cref_pixsel_pattern(void *s, int n, uint8_t *out) { std::memcpy(out, ((ldso::PixelSelector *) s)->randomPattern, (size_t) n); }
int cref_pixsel_get_potential(void *s) { return ((ldso::PixelSelector *) s)->currentPotential; }
void cref_pixsel_set_potential(void *s, int p) { ((ldso::PixelSelector *) s)->currentPotential = p; }

static void set_settings(float cut, float add, float dw, int dirDist) {
    ldso::setting_minGradHistCut = cut;
    ldso::setting_minGradHistAdd = add;
    ldso::setting_gradDownweightPerLevel = dw;
    ldso::setting_selectDirectionDistribution = dirDist != 0;
    ldso::setting_gammaWeightsPixelSelect = 1;
}

// makeImages of (color, B) and makeMaps(fh, map, density, recursionsLeft, false, thFactor) with the selector's currentPotential;
// map_out gets makeMaps' float map (w*h)
int cref_pixsel_make_maps(void *sp, int w, int h, const float *color, const float *B, float density, int recursionsLeft, float thFactor,
                          float cut, float add, float dw, int dirDist, float *map_out) {
    set_settings(cut, add, dw, dirDist);
    RefFrame f(w, h, color, B);
    return ((ldso::PixelSelector *) sp)->makeMaps(f.frame->frameHessian, map_out, density, recursionsLeft, false, thFactor);
}

// seconds per makeMaps call on a frame whose pyramid is built (a new frame each keyframe: the histogram is made in every call):
// the median of `runs` runs of `reps` calls each; *n_out gets the last call's value
double cref_pixsel_time(int w, int h, const float *color, const float *B, float density, int reps, int runs, int *n_out) {
    set_settings(0.5f, 7.f, 0.75f, 1);
    RefFrame f(w, h, color, B);
    ldso::PixelSelector sel(w, h);
    std::vector<float> map((size_t) w * h);
    std::vector<double> t;
    for (int k = 0; k < runs; k++) {
        const auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < reps; i++) {
            sel.gradHistFrame = nullptr;
            *n_out = sel.makeMaps(f.frame->frameHessian, map.data(), density);
        }
        t.push_back(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() / reps);
    }
    std::sort(t.begin(), t.end());
    return t[t.size() / 2];
}

}
