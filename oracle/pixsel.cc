// ORACLE restatement of DSO's pixel selection — TEST INFRASTRUCTURE ONLY (built by pixsel.mk with -ffp-contract=off).
// FrameHessian::makeImages' levels 0-2 (src/internal/FrameHessian.cc:44-98), PixelSelector's constructor, makeHists, select and
// makeMaps (src/frontend/PixelSelector2.cc) restated with the rules the device follows where the reference reads memory it never
// wrote (DESIGN.md "Pixel selection"):
//   - thsSmoothed entries at or past w32*h32 read 0; the flat index wraps into the next row as the reference's does;
//   - absSquaredGrad is 0 on rows 0 and h_l-1 of every level; gradHist bins past 49 read 0;
//   - a NaN gradient goes to histogram bin 48.
// It also counts, per select() pass, the pot cells whose level-0 pick depends on the direction (mixed direction masks).
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {

struct Selector {
    int w, h, currentPotential = 3;
    std::vector<unsigned char> randomPattern;
    std::vector<float> ths, thsSmoothed;
    std::vector<float> ag[3];            // absSquaredGrad[0..2]
    std::vector<float> dx0, dy0;         // level-0 gradient (dI[idx][1], [2])
    int w32 = 0, h32 = 0, mixed = 0;
};

void make_images(Selector &s, const float *color, const float *B) {
    std::vector<float> I(color, color + (size_t) s.w * s.h), Iprev;
    int wl = s.w, hl = s.h;
    for (int lvl = 0; lvl < 3; lvl++) {
        if (lvl > 0) {
            const int wlm1 = wl;
            Iprev.swap(I);
            wl = s.w >> lvl; hl = s.h >> lvl;
            I.assign((size_t) wl * hl, 0.f);
            for (int y = 0; y < hl; y++)
                for (int x = 0; x < wl; x++)
                    I[x + y * wl] = 0.25f * (Iprev[2 * x + 2 * y * wlm1] + Iprev[2 * x + 1 + 2 * y * wlm1] + Iprev[2 * x + 2 * y * wlm1 + wlm1] +
                                             Iprev[2 * x + 1 + 2 * y * wlm1 + wlm1]);
        }
        std::vector<float> &dabs = s.ag[lvl];
        dabs.assign((size_t) wl * hl, 0.f);          // rows 0 and hl-1 stay 0
        if (lvl == 0) { s.dx0.assign((size_t) wl * hl, 0.f); s.dy0.assign((size_t) wl * hl, 0.f); }
        for (int idx = wl; idx < wl * (hl - 1); idx++) {
            float dx = 0.5f * (I[idx + 1] - I[idx - 1]);
            float dy = 0.5f * (I[idx + wl] - I[idx - wl]);
            if (std::isnan(dx) || std::fabs(dx) > 255.0) dx = 0;
            if (std::isnan(dy) || std::fabs(dy) > 255.0) dy = 0;
            if (lvl == 0) { s.dx0[idx] = dx; s.dy0[idx] = dy; }
            dabs[idx] = dx * dx + dy * dy;
            if (B) {
                int c = I[idx] + 0.5f;
                if (c < 5) c = 5;
                if (c > 250) c = 250;
                const float gw = B[c + 1] - B[c];
                dabs[idx] *= gw * gw;
            }
        }
    }
}

int computeHistQuantil(const int *hist, float below) {
    int th = hist[0] * below + 0.5f;
    for (int i = 0; i < 90; i++) {
        th -= i + 1 < 50 ? hist[i + 1] : 0;
        if (th < 0) return i;
    }
    return 90;
}

void make_hists(Selector &s, float cut, float add) {
    const int w = s.w, h = s.h, w32 = s.w32, h32 = s.h32;
    const float *mapmax0 = s.ag[0].data();
    s.ths.assign((size_t) w32 * h32, 0.f);
    s.thsSmoothed.assign((size_t) w32 * h32, 0.f);
    for (int y = 0; y < h32; y++)
        for (int x = 0; x < w32; x++) {
            const float *map0 = mapmax0 + 32 * x + 32 * y * w;
            int hist0[50];
            memset(hist0, 0, sizeof(hist0));
            for (int j = 0; j < 32; j++)
                for (int i = 0; i < 32; i++) {
                    const int it = i + 32 * x, jt = j + 32 * y;
                    if (it > w - 2 || jt > h - 2 || it < 1 || jt < 1) continue;
                    const float r = sqrtf(map0[i + j * w]);
                    int g = std::isnan(r) ? 48 : (int) r;
                    if (g > 48) g = 48;
                    hist0[g + 1]++;
                    hist0[0]++;
                }
            s.ths[x + y * w32] = computeHistQuantil(hist0, cut) + add;
        }
    const float *ths = s.ths.data();
    for (int y = 0; y < h32; y++)
        for (int x = 0; x < w32; x++) {
            float sum = 0, num = 0;
            if (x > 0) {
                if (y > 0) { num++; sum += ths[x - 1 + (y - 1) * w32]; }
                if (y < h32 - 1) { num++; sum += ths[x - 1 + (y + 1) * w32]; }
                num++; sum += ths[x - 1 + (y) * w32];
            }
            if (x < w32 - 1) {
                if (y > 0) { num++; sum += ths[x + 1 + (y - 1) * w32]; }
                if (y < h32 - 1) { num++; sum += ths[x + 1 + (y + 1) * w32]; }
                num++; sum += ths[x + 1 + (y) * w32];
            }
            if (y > 0) { num++; sum += ths[x + (y - 1) * w32]; }
            if (y < h32 - 1) { num++; sum += ths[x + (y + 1) * w32]; }
            num++; sum += ths[x + y * w32];
            s.thsSmoothed[x + y * w32] = (sum / num) * (sum / num);
        }
}

float th_at(const Selector &s, int xf, int yf) {
    const int i = (xf >> 5) + (yf >> 5) * s.w32;
    return i < s.w32 * s.h32 ? s.thsSmoothed[i] : 0.f;
}

const float directions[16][2] = {{0, 1.0000}, {0.3827, 0.9239}, {0.1951, 0.9808}, {0.9239, 0.3827}, {0.7071, 0.7071}, {0.3827, -0.9239},
                                 {0.8315, 0.5556}, {0.8315, -0.5556}, {0.5556, -0.8315}, {0.9808, 0.1951}, {0.9239, -0.3827},
                                 {0.7071, -0.7071}, {0.5556, 0.8315}, {0.9808, -0.1951}, {1.0000, 0.0000}, {0.1951, -0.9808}};

struct Params { float thFactor, dw1; int dirDist; };

float dir_norm(const Selector &s, const Params &P, int idx, int d, float ag) {
    if (!P.dirDist) return ag;
    return fabsf((float) (s.dx0[idx] * directions[d][0] + s.dy0[idx] * directions[d][1]));
}

// the pot cell at (x234, y234): does it pick at level 0 with direction d, for every d? (mixed: some do, some do not)
bool cell_mixed(const Selector &s, const Params &P, int x234, int y234, int my1, int mx1) {
    unsigned m = 0;
    for (int y1 = 0; y1 < my1; y1++)
        for (int x1 = 0; x1 < mx1; x1++) {
            const int xf = x1 + x234, yf = y1 + y234, idx = xf + yf * s.w;
            if (xf < 4 || xf >= s.w - 5 || yf < 4 || yf > s.h - 4) continue;
            const float ag0 = s.ag[0][idx];
            if (!(ag0 > th_at(s, xf, yf) * P.thFactor)) continue;
            for (int d = 0; d < 16; d++)
                if (dir_norm(s, P, idx, d, ag0) > 0) m |= 1u << d;
        }
    return m != 0 && m != 0xFFFFu;
}

void select(Selector &s, const Params &P, uint8_t *map_out, int pot, int n[3]) {
    const int w = s.w, h = s.h, w1 = s.w >> 1, w2 = s.w >> 2;
    const float *mapmax0 = s.ag[0].data(), *mapmax1 = s.ag[1].data(), *mapmax2 = s.ag[2].data();
    memset(map_out, 0, (size_t) w * h);
    const float dw1 = P.dw1, dw2 = dw1 * dw1, thFactor = P.thFactor;
    const unsigned char *randomPattern = s.randomPattern.data();
    int n3 = 0, n2 = 0, n4 = 0;
    s.mixed = 0;
    for (int y4 = 0; y4 < h; y4 += (4 * pot))
        for (int x4 = 0; x4 < w; x4 += (4 * pot)) {
            const int my3 = std::min((4 * pot), h - y4), mx3 = std::min((4 * pot), w - x4);
            int bestIdx4 = -1;
            float bestVal4 = 0;
            const int dir4 = randomPattern[n2] & 0xF;
            for (int y3 = 0; y3 < my3; y3 += (2 * pot))
                for (int x3 = 0; x3 < mx3; x3 += (2 * pot)) {
                    const int x34 = x3 + x4, y34 = y3 + y4;
                    const int my2 = std::min((2 * pot), h - y34), mx2 = std::min((2 * pot), w - x34);
                    int bestIdx3 = -1;
                    float bestVal3 = 0;
                    const int dir3 = randomPattern[n2] & 0xF;
                    for (int y2 = 0; y2 < my2; y2 += pot)
                        for (int x2 = 0; x2 < mx2; x2 += pot) {
                            const int x234 = x2 + x34, y234 = y2 + y34;
                            const int my1 = std::min(pot, h - y234), mx1 = std::min(pot, w - x234);
                            int bestIdx2 = -1;
                            float bestVal2 = 0;
                            const int dir2 = randomPattern[n2] & 0xF;
                            s.mixed += cell_mixed(s, P, x234, y234, my1, mx1);
                            for (int y1 = 0; y1 < my1; y1 += 1)
                                for (int x1 = 0; x1 < mx1; x1 += 1) {
                                    const int idx = x1 + x234 + w * (y1 + y234);
                                    const int xf = x1 + x234, yf = y1 + y234;
                                    if (xf < 4 || xf >= w - 5 || yf < 4 || yf > h - 4) continue;
                                    const float pixelTH0 = th_at(s, xf, yf);
                                    const float pixelTH1 = pixelTH0 * dw1;
                                    const float pixelTH2 = pixelTH1 * dw2;
                                    const float ag0 = mapmax0[idx];
                                    if (ag0 > pixelTH0 * thFactor) {
                                        const float dirNorm = dir_norm(s, P, idx, dir2, ag0);
                                        if (dirNorm > bestVal2) { bestVal2 = dirNorm; bestIdx2 = idx; bestIdx3 = -2; bestIdx4 = -2; }
                                    }
                                    if (bestIdx3 == -2) continue;
                                    const float ag1 = mapmax1[(int) (xf * 0.5f + 0.25f) + (int) (yf * 0.5f + 0.25f) * w1];
                                    if (ag1 > pixelTH1 * thFactor) {
                                        const float dirNorm = dir_norm(s, P, idx, dir3, ag1);
                                        if (dirNorm > bestVal3) { bestVal3 = dirNorm; bestIdx3 = idx; bestIdx4 = -2; }
                                    }
                                    if (bestIdx4 == -2) continue;
                                    const float ag2 = mapmax2[(int) (xf * 0.25f + 0.125) + (int) (yf * 0.25f + 0.125) * w2];
                                    if (ag2 > pixelTH2 * thFactor) {
                                        const float dirNorm = dir_norm(s, P, idx, dir4, ag2);
                                        if (dirNorm > bestVal4) { bestVal4 = dirNorm; bestIdx4 = idx; }
                                    }
                                }
                            if (bestIdx2 > 0) { map_out[bestIdx2] = 1; bestVal3 = 1e10; n2++; }
                        }
                    if (bestIdx3 > 0) { map_out[bestIdx3] = 2; bestVal4 = 1e10; n3++; }
                }
            if (bestIdx4 > 0) { map_out[bestIdx4] = 4; n4++; }
        }
    n[0] = n2; n[1] = n3; n[2] = n4;
}

// float -> int as x86's cvttss2si converts it
int f2i(float f) { return (f >= -2147483648.f && f < 2147483648.f) ? (int) f : INT32_MIN; }

int make_maps(Selector &s, const Params &P, uint8_t *map_out, float density, int recursionsLeft, int counts[3]) {
    float numHave = 0;
    float numWant = density;
    float quotia;
    int idealPotential = s.currentPotential;
    int n[3];
    select(s, P, map_out, s.currentPotential, n);
    numHave = n[0] + n[1] + n[2];
    quotia = numWant / numHave;
    float K = numHave * (s.currentPotential + 1) * (s.currentPotential + 1);
    idealPotential = f2i(sqrtf(K / numWant) - 1);
    if (idealPotential < 1) idealPotential = 1;
    if (recursionsLeft > 0 && quotia > 1.25 && s.currentPotential > 1) {
        if (idealPotential >= s.currentPotential) idealPotential = s.currentPotential - 1;
        s.currentPotential = idealPotential;
        return make_maps(s, P, map_out, density, recursionsLeft - 1, counts);
    } else if (recursionsLeft > 0 && quotia < 0.25) {
        if (idealPotential <= s.currentPotential) idealPotential = s.currentPotential + 1;
        s.currentPotential = idealPotential;
        return make_maps(s, P, map_out, density, recursionsLeft - 1, counts);
    }
    int numHaveSub = numHave;
    if (quotia < 0.95) {
        const int wh = s.w * s.h;
        int rn = 0;
        unsigned char charTH = 255 * quotia;
        for (int i = 0; i < wh; i++) {
            if (map_out[i] != 0) {
                if (s.randomPattern[rn] > charTH) { map_out[i] = 0; numHaveSub--; }
                rn++;
            }
        }
    }
    s.currentPotential = idealPotential;
    counts[0] = n[0]; counts[1] = n[1]; counts[2] = n[2];
    return numHaveSub;
}

}  // namespace

extern "C" {

void *oracle_pixsel_new(int w, int h) {
    Selector *s = new Selector;
    s->w = w; s->h = h; s->w32 = w / 32; s->h32 = h / 32;
    s->randomPattern.resize((size_t) w * h);
    std::srand(3141592);
    for (int i = 0; i < w * h; i++) s->randomPattern[i] = rand() & 0xFF;
    return s;
}
void oracle_pixsel_free(void *s) { delete (Selector *) s; }
int oracle_pixsel_get_potential(void *s) { return ((Selector *) s)->currentPotential; }
void oracle_pixsel_set_potential(void *s, int p) { ((Selector *) s)->currentPotential = p; }
void oracle_pixsel_pattern(void *s, uint8_t *out) {
    const Selector &S = *(Selector *) s;
    memcpy(out, S.randomPattern.data(), S.randomPattern.size());
}

// makeImages of (color, B) (B NULL: identity) and makeHists on it; ag_out (optional) receives absSquaredGrad[0..2] one level after
// the other, ths_out (optional) thsSmoothed (w32*h32)
void oracle_pixsel_set_frame(void *sp, const float *color, const float *B, float minGradHistCut, float minGradHistAdd, float *ag_out,
                             float *ths_out) {
    Selector &s = *(Selector *) sp;
    make_images(s, color, B);
    make_hists(s, minGradHistCut, minGradHistAdd);
    if (ag_out)
        for (int l = 0; l < 3; l++) { memcpy(ag_out, s.ag[l].data(), sizeof(float) * s.ag[l].size()); ag_out += s.ag[l].size(); }
    if (ths_out) memcpy(ths_out, s.thsSmoothed.data(), sizeof(float) * s.thsSmoothed.size());
}

// thsSmoothed as select() reads it at pixel (xf, yf)
float oracle_pixsel_th(void *s, int xf, int yf) { return th_at(*(Selector *) s, xf, yf); }

// makeMaps on the frame set last; out4 = n2, n3, n4 of the final pass and the mixed cells of that pass
int oracle_pixsel_make_maps(void *sp, float density, int recursionsLeft, float thFactor, float gradDownweightPerLevel, int dirDist,
                            uint8_t *map_out, int out4[4]) {
    Selector &s = *(Selector *) sp;
    Params P{thFactor, gradDownweightPerLevel, dirDist};
    int c[3];
    const int r = make_maps(s, P, map_out, density, recursionsLeft, c);
    out4[0] = c[0]; out4[1] = c[1]; out4[2] = c[2]; out4[3] = s.mixed;
    return r;
}

}
