// PIN of the undistortion restatement (../undistort.cc) against the reference's own Undistort.cc — TEST INFRASTRUCTURE ONLY.
// For every camera (five models in crop mode, two with an explicit output calibration, one without rectification) and every case
// (8- and 16-bit frames, photometric modes 0 / 1 / 2, the factor path through exposure <= 0 and through a missing gamma file,
// setting_useExposure off), it builds the reference's undistorter from files (undistort_ref.cc), runs Undistort::undistort<T>, runs
// the restatement on the tables the reference built, and compares the two images bit for bit. Pixels whose taps the reference reads
// past the end of its buffer are excluded and counted. One line per case on stdout, starting with "PIN "; exit status 1 on any
// mismatch.
//
//     pin_undistort [DIR]      DIR: also write the tables, frames and the restatement's outputs there (tests/golden/make_undistort_golden.py)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unistd.h>
#include <vector>

extern "C" {
void *uref_open(const char *dir, int model, int rect, int wOrg, int hOrg, int w, int h, int gamma_entries, int mode, int use_exposure);
void uref_close(void *u);
int uref_tables(void *u, int *wh, float *remapX, float *remapY, float *G, float *vinv, int *g_entries);
float uref_undistort(void *u, const void *raw, int bytes_per_pixel, float exposure, float factor, float *out);
float oracle_undistort(int wOrg, int hOrg, int w, int h, const float *remapX, const float *remapY, const float *G, const float *vinv,
                       int mode, int use_exposure, const void *raw, int bytes_per_pixel, float exposure, float factor, float *out,
                       unsigned char *past_end);
}

static const char *MODEL[] = {"fov", "radtan", "equidistant", "kb", "pinhole"};
static const char *RECT[] = {"crop", "calib", "none"};
struct Cam { int model, rect; };
struct Case { const char *name; int bpp, gamma_entries, mode, use_exposure; float exposure, factor; };

static const Cam CAMS[] = {{0, 0}, {1, 0}, {2, 0}, {3, 0}, {4, 0}, {0, 1}, {1, 1}, {4, 2}};
static const Case CASES[] = {
    {"u8_m0", 1, 256, 0, 1, 1.5f, 1.0f},      {"u8_m1", 1, 256, 1, 1, 1.5f, 1.0f},      {"u8_m2", 1, 256, 2, 1, 1.5f, 1.0f},
    {"u16_m0", 2, 65536, 0, 1, 2.0f, 0.25f},  {"u16_m1", 2, 65536, 1, 1, 2.0f, 1.0f},   {"u16_m2", 2, 65536, 2, 1, 2.0f, 1.0f},
    {"u8_g16_m2", 1, 65536, 2, 1, 1.0f, 1.0f}, {"u8_exp0", 1, 256, 2, 1, 0.0f, 0.75f},  {"u16_expneg", 2, 65536, 2, 1, -2.0f, 1.25f},
    {"u8_nogamma", 1, 0, 2, 1, 1.0f, 0.5f},   {"u16_noexp", 2, 65536, 1, 0, 3.0f, 1.0f},
};
static const int WORG = 48, HORG = 36, W = 32, H = 24;

static void dump(const std::string &dir, const std::string &name, const void *p, size_t bytes) {
    FILE *f = fopen((dir + "/" + name).c_str(), "wb");
    if (!f || fwrite(p, 1, bytes, f) != bytes) { fprintf(stderr, "cannot write %s\n", name.c_str()); exit(2); }
    fclose(f);
}

int main(int argc, char **argv) {
    const std::string out_dir = argc > 1 ? argv[1] : "";
    char tmpl[] = "/tmp/pin_undistort_XXXXXX";
    const char *dir = mkdtemp(tmpl);
    if (!dir) { perror("mkdtemp"); return 2; }
    // raw frames: a fixed LCG over the whole 8- / 16-bit range
    std::vector<uint8_t> raw8(WORG * HORG);
    std::vector<uint16_t> raw16(WORG * HORG);
    uint32_t s = 12345;
    for (int i = 0; i < WORG * HORG; i++) {
        s = s * 1664525u + 1013904223u; raw8[i] = s >> 24;
        s = s * 1664525u + 1013904223u; raw16[i] = s >> 16;
    }
    FILE *manifest = nullptr;
    if (!out_dir.empty()) {
        dump(out_dir, "raw8.bin", raw8.data(), raw8.size());
        dump(out_dir, "raw16.bin", raw16.data(), 2 * raw16.size());
        manifest = fopen((out_dir + "/manifest.txt").c_str(), "w");
    }
    long total_bad = 0;
    for (const Cam &cam : CAMS) {
        const int w = cam.rect == 2 ? WORG : W, h = cam.rect == 2 ? HORG : H;
        const std::string cname = std::string(MODEL[cam.model]) + "_" + RECT[cam.rect];
        for (const Case &cs : CASES) {
            void *u = uref_open(dir, cam.model, cam.rect, WORG, HORG, w, h, cs.gamma_entries, cs.mode, cs.use_exposure);
            if (!u) { fprintf(stderr, "cannot build the reference's undistorter for %s\n", cname.c_str()); return 2; }
            int wh[4], g_entries = 0;
            std::vector<float> rx(w * h), ry(w * h), G(65536), vinv(WORG * HORG);
            const int passthrough = uref_tables(u, wh, rx.data(), ry.data(), G.data(), vinv.data(), &g_entries);
            if (wh[0] != w || wh[1] != h || wh[2] != WORG || wh[3] != HORG) { fprintf(stderr, "unexpected sizes\n"); return 2; }
            const void *raw = cs.bpp == 1 ? (const void *) raw8.data() : (const void *) raw16.data();
            std::vector<float> ref(w * h), ora(w * h);
            std::vector<unsigned char> past(w * h);
            const float e_ref = uref_undistort(u, raw, cs.bpp, cs.exposure, cs.factor, ref.data());
            const float e_ora = oracle_undistort(WORG, HORG, w, h, passthrough ? nullptr : rx.data(), passthrough ? nullptr : ry.data(),
                                                 g_entries ? G.data() : nullptr, vinv.data(), cs.mode, cs.use_exposure, raw, cs.bpp,
                                                 cs.exposure, cs.factor, ora.data(), past.data());
            long bad = 0, excluded = 0, nonzero = 0;
            for (int i = 0; i < w * h; i++) {
                if (past[i]) { excluded++; continue; }
                if (std::memcmp(&ref[i], &ora[i], sizeof(float)) != 0) bad++;
                nonzero += ora[i] != 0;
            }
            if (std::memcmp(&e_ref, &e_ora, sizeof(float)) != 0) bad++;
            total_bad += bad;
            printf("PIN %s %s mismatches=%ld excluded=%ld nonzero=%ld pixels=%d g_entries=%d passthrough=%d\n", cname.c_str(), cs.name,
                   bad, excluded, nonzero, w * h, g_entries, passthrough);
            if (manifest) {
                const std::string stem = cname + "." + cs.name;
                if (!passthrough) { dump(out_dir, stem + ".remapX.bin", rx.data(), 4 * rx.size()); dump(out_dir, stem + ".remapY.bin", ry.data(), 4 * ry.size()); }
                if (g_entries) dump(out_dir, stem + ".G.bin", G.data(), 4 * g_entries);
                if (g_entries) dump(out_dir, stem + ".vinv.bin", vinv.data(), 4 * vinv.size());
                dump(out_dir, stem + ".out.bin", ora.data(), 4 * ora.size());
                dump(out_dir, stem + ".past.bin", past.data(), past.size());
                fprintf(manifest, "%s %s %d %d %d %d %d %d %d %d %d %.9g %.9g %.9g %ld\n", cname.c_str(), cs.name, w, h, WORG, HORG, passthrough,
                        g_entries, cs.mode, cs.use_exposure, cs.bpp, cs.exposure, cs.factor, e_ora, excluded);
            }
            uref_close(u);
        }
    }
    if (manifest) fclose(manifest);
    std::remove((std::string(dir) + "/camera.txt").c_str());
    std::remove((std::string(dir) + "/pcalib.txt").c_str());
    rmdir(dir);
    printf("PIN total mismatches=%ld\n", total_bad);
    return total_bad ? 1 : 0;
}
