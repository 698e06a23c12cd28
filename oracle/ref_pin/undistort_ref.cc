// The reference's own undistorters behind a small C interface — TEST INFRASTRUCTURE ONLY, built by ../undistort.mk where a
// reference checkout exists. It writes a camera file (FOV, RadTan, Equidistant, KB or Pinhole model; crop, explicit output
// calibration or no rectification) and a gamma file into a directory, builds the reference's Undistort through
// Undistort::getUndistorterForFile (src/frontend/Undistort.cc, compiled unmodified), and runs Undistort::undistort<T>. The vignette
// image comes from memory: IOWrap::readImageBW_8U / readImageBW_16U below stand in for the reference's OpenCV image reader.
// Compiled with -Dprivate=public so that the tables the reference built (G, vignetteMapInv, valid) can be read back; the protected
// remapX / remapY / passthrough members are reached through pointers to members of a derived class.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <string>
#include <vector>

#include "Settings.h"
#include "frontend/Undistort.h"
#include "frontend/ImageRW.h"

namespace {
int g_vig_bits = 0;          // which vignette image the stand-in reader serves: 8, 16 or none
int g_vig_w = 0, g_vig_h = 0;

// a radial fall-off with no zero, as a real vignette image has
template<typename T>
ldso::MinimalImage<T> *make_vignette(int w, int h, float lo, float hi) {
    auto *img = new ldso::MinimalImage<T>(w, h);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const double dx = (x - 0.5 * (w - 1)) / w, dy = (y - 0.5 * (h - 1)) / h;
            const double r2 = std::min(1.0, 2.0 * (dx * dx + dy * dy));
            img->at(x, y) = (T) std::lround(lo + (hi - lo) * (1.0 - r2) + ((x * 7 + y * 13) % 5));
        }
    return img;
}

const char *model_line(int model) {
    switch (model) {
        case 0: return "FOV 0.52 0.68 0.5 0.5 0.92";
        case 1: return "RadTan 0.55 0.72 0.49 0.51 -0.28 0.072 0.0011 -0.0007";
        case 2: return "EquiDistant 0.5 0.66 0.5 0.5 0.012 -0.0051 0.0013 -0.0002";
        case 3: return "KannalaBrandt 0.5 0.66 0.51 0.49 0.011 -0.0042 0.0009 -0.0001";
        default: return "Pinhole 0.53 0.7 0.5 0.5 0";
    }
}

struct Access : ldso::Undistort {       // protected members of the reference's Undistort
    static float *ldso::Undistort::*rx() { return &Access::remapX; }
    static float *ldso::Undistort::*ry() { return &Access::remapY; }
    static bool ldso::Undistort::*pt() { return &Access::passthrough; }
};
}  // namespace

namespace ldso {
namespace IOWrap {
MinimalImageB *readImageBW_8U(std::string) { return g_vig_bits == 8 ? make_vignette<unsigned char>(g_vig_w, g_vig_h, 110, 250) : nullptr; }
MinimalImage<unsigned short> *readImageBW_16U(std::string) {
    return g_vig_bits == 16 ? make_vignette<unsigned short>(g_vig_w, g_vig_h, 21000, 65000) : nullptr;
}
}  // namespace IOWrap
}  // namespace ldso

extern "C" {

// model 0..4 = FOV, RadTan, Equidistant, KB, Pinhole; rect 0 = crop, 1 = explicit output calibration, 2 = none (w == wOrg, h == hOrg);
// gamma_entries 256 (8-bit vignette), 65536 (16-bit vignette) or 0 (no gamma file: the calibration is invalid).
// mode / use_exposure set setting_photometricCalibration / setting_useExposure, which the constructor and processFrame read.
void *uref_open(const char *dir, int model, int rect, int wOrg, int hOrg, int w, int h, int gamma_entries, int mode, int use_exposure) {
    ldso::setting_photometricCalibration = mode;
    ldso::setting_useExposure = use_exposure != 0;
    const std::string cam = std::string(dir) + "/camera.txt", gamma = std::string(dir) + "/pcalib.txt";
    FILE *f = fopen(cam.c_str(), "w");
    if (!f) return nullptr;
    const char *out = rect == 0 ? "crop" : rect == 1 ? "0.42 0.56 0.5 0.5 0" : "none";
    fprintf(f, "%s\n%d %d\n%s\n%d %d\n", model_line(model), wOrg, hOrg, out, w, h);
    fclose(f);
    std::remove(gamma.c_str());
    if (gamma_entries > 0) {
        f = fopen(gamma.c_str(), "w");
        if (!f) return nullptr;
        for (int i = 0; i < gamma_entries; i++)      // strictly increasing, exactly representable in float
            fprintf(f, "%s%.9g", i ? " " : "", (float) (i + 0.35 * gamma_entries * std::pow(i / (double) (gamma_entries - 1), 0.6)));
        fprintf(f, "\n");
        fclose(f);
    }
    g_vig_bits = gamma_entries == 256 ? 8 : gamma_entries == 65536 ? 16 : 0;
    g_vig_w = wOrg; g_vig_h = hOrg;
    return ldso::Undistort::getUndistorterForFile(cam, gamma, "vignette");
}

void uref_close(void *u) { delete (ldso::Undistort *) u; }

// the reference's tables; returns 1 in passthrough (remap unused). g_entries gets GDepth when the calibration is valid, else 0.
int uref_tables(void *u_, int *wh, float *remapX, float *remapY, float *G, float *vinv, int *g_entries) {
    ldso::Undistort *u = (ldso::Undistort *) u_;
    ldso::PhotometricUndistorter *p = u->photometricUndist;
    const int w = u->getSize()[0], h = u->getSize()[1], wOrg = u->getOriginalSize()[0], hOrg = u->getOriginalSize()[1];
    wh[0] = w; wh[1] = h; wh[2] = wOrg; wh[3] = hOrg;
    if (remapX) for (int i = 0; i < w * h; i++) { remapX[i] = (u->*Access::rx())[i]; remapY[i] = (u->*Access::ry())[i]; }
    *g_entries = p->valid ? p->GDepth : 0;
    if (G && p->valid) for (int i = 0; i < p->GDepth; i++) G[i] = p->G[i];
    if (vinv && p->vignetteMapInv) for (int i = 0; i < wOrg * hOrg; i++) vinv[i] = p->vignetteMapInv[i];
    return u->*Access::pt() ? 1 : 0;
}

// Undistort::undistort<T> of one raw frame into out (w*h floats); returns the exposure time of the result
float uref_undistort(void *u_, const void *raw, int bytes_per_pixel, float exposure, float factor, float *out) {
    ldso::Undistort *u = (ldso::Undistort *) u_;
    const int wOrg = u->getOriginalSize()[0], hOrg = u->getOriginalSize()[1];
    ldso::ImageAndExposure *r;
    if (bytes_per_pixel == 1) {
        ldso::MinimalImage<unsigned char> img(wOrg, hOrg, (unsigned char *) raw);
        r = u->undistort<unsigned char>(&img, exposure, 0, factor);
    } else {
        ldso::MinimalImage<unsigned short> img(wOrg, hOrg, (unsigned short *) raw);
        r = u->undistort<unsigned short>(&img, exposure, 0, factor);
    }
    for (int i = 0; i < r->w * r->h; i++) out[i] = r->image[i];
    const float e = r->exposure_time;
    delete r;
    return e;
}

// seconds per Undistort::undistort<T> call (the result's allocation and release included, as in the reference's frame loop),
// the median of `runs` runs of `reps` calls each
double uref_time(void *u_, const void *raw, int bytes_per_pixel, float exposure, int reps, int runs) {
    ldso::Undistort *u = (ldso::Undistort *) u_;
    const int wOrg = u->getOriginalSize()[0], hOrg = u->getOriginalSize()[1];
    ldso::MinimalImage<unsigned char> i8(wOrg, hOrg, (unsigned char *) raw);
    ldso::MinimalImage<unsigned short> i16(wOrg, hOrg, (unsigned short *) raw);
    std::vector<double> t;
    for (int k = 0; k < runs; k++) {
        const auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < reps; i++)
            delete (bytes_per_pixel == 1 ? u->undistort<unsigned char>(&i8, exposure, 0, 1) : u->undistort<unsigned short>(&i16, exposure, 0, 1));
        t.push_back(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() / reps);
    }
    std::sort(t.begin(), t.end());
    return t[t.size() / 2];
}

}
