// ORACLE: LDSO's keyframe corner detection restated without dependencies — TEST INFRASTRUCTURE ONLY (built by corners.mk with
// -ffp-contract=off, like liboracle.so). FeatureDetector::DetectCorners (src/frontend/FeatureDetector.cc:34-130) with ShiTomasiScore
// and IC_Angle (include/frontend/FeatureDetector.h:50-114), ComputeDescriptor (FeatureDetector.cc:132-189) and the umax table of the
// detector's constructor (:10-28), working on level 0 of the pyramid FrameHessian::makeImages builds (I, dx, dy per pixel) and on
// absSquaredGrad[0] formed on the fly as makeImages forms it (FrameHessian.cc:91-97). Where the reference's result depends on
// library internals this restatement follows the rule the device follows (DESIGN.md §"Keyframe corners"):
//   - order within a cell: score descending; equal scores and NaN scores keep push order (x outer, y inner); NaNs after every number
//     (the reference's std::sort is not stable, and a NaN breaks its comparator);
//   - atan2f / cosf / sinf are evaluated in double and rounded to float.
// Configurations whose angle / descriptor footprints can leave the image are refused (the reference reads outside its buffer there).
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

const int HALF_PATCH_SIZE = 15;

struct Grid {
    int gs, gridX, gridY, skip, ncx, ncy, kcap;
    float nfeatInGrid;
};

// the grid of DetectCorners (FeatureDetector.cc:37-42); false for nFeatures <= 0, gridsize 0, or footprints that can leave the image
bool make_grid(int w, int h, int nFeatures, Grid &g) {
    if (w <= 0 || h <= 0 || nFeatures <= 0) return false;
    g.gs = int(sqrtf((float) (w * h / nFeatures)) + 0.5);
    if (g.gs <= 0) return false;
    g.gridX = w / g.gs + 1;
    g.gridY = h / g.gs + 1;
    g.nfeatInGrid = float(nFeatures) / (w * h) * (g.gs * g.gs);
    g.skip = HALF_PATCH_SIZE * 2 / g.gs + 1;
    g.ncx = std::max(0, g.gridX - 2 * g.skip);
    g.ncy = std::max(0, g.gridY - 2 * g.skip);
    int k = 0;                       // features taken per cell: the first k with k > nfeatInGrid
    while (!((float) k > g.nfeatInGrid)) k++;
    g.kcap = std::min(k, g.gs * g.gs);
    if (g.ncx > 0 && g.ncy > 0) {
        // every pixel of a cell may become a corner: IC_Angle reads +-HALF_PATCH_SIZE rows and columns around it, the descriptor's
        // rotated pattern at most 13 (|pattern| <= 13, and the angle is scaled by pi/180 before cos / sin)
        const int x0 = g.skip * g.gs, x1 = (g.gridX - g.skip) * g.gs - 1;
        const int y0 = g.skip * g.gs, y1 = (g.gridY - g.skip) * g.gs - 1;
        if (x0 - HALF_PATCH_SIZE < 0 || x1 + HALF_PATCH_SIZE > w - 1 || y0 - HALF_PATCH_SIZE < 0 || y1 + HALF_PATCH_SIZE > h - 1) return false;
    }
    return true;
}

// FeatureDetector's constructor: umax (cvFloor / cvCeil / cvRound of the same double expressions)
void make_umax(int umax[HALF_PATCH_SIZE + 1]) {
    int v, v0, vmax = (int) std::floor(HALF_PATCH_SIZE * std::sqrt(2.f) / 2 + 1);
    int vmin = (int) std::ceil(HALF_PATCH_SIZE * std::sqrt(2.f) / 2);
    const double hp2 = HALF_PATCH_SIZE * HALF_PATCH_SIZE;
    for (v = 0; v <= vmax; ++v) umax[v] = (int) std::lrint(std::sqrt(hp2 - v * v));
    for (v = HALF_PATCH_SIZE, v0 = 0; v >= vmin; --v) {
        while (umax[v0] == umax[v0 + 1]) ++v0;
        umax[v] = v0;
        ++v0;
    }
}

struct Img {
    const float *p;      // (I, dx, dy) per pixel
    int w, h;
    float I(int i) const { return p[3 * i]; }
    float dx(int i) const { return p[3 * i + 1]; }
    float dy(int i) const { return p[3 * i + 2]; }
};

// absSquaredGrad[0] as makeImages leaves it: dx*dx + dy*dy, times gw*gw when a response B is given
float abs_sq_grad(const Img &im, const float *B, int idx) {
    const float dx = im.dx(idx), dy = im.dy(idx);
    float g = dx * dx + dy * dy;
    if (B) {
        int c = im.I(idx) + 0.5f;                 // CalibHessian::getBGradOnly
        if (c < 5) c = 5;
        if (c > 250) c = 250;
        const float gw = B[c + 1] - B[c];
        g *= gw * gw;
    }
    return g;
}

float shi_tomasi(const Img &im, int u, int v) {
    const int halfbox = 4, box_size = 2 * halfbox, box_area = box_size * box_size;
    float dXX = 0.0, dYY = 0.0, dXY = 0.0;
    const int x_min = u - halfbox, x_max = u + halfbox, y_min = v - halfbox, y_max = v + halfbox;
    if (x_min < 1 || x_max >= im.w - 1 || y_min < 1 || y_max >= im.h - 1) return 0.0;
    for (int y = y_min; y < y_max; ++y)
        for (int x = x_min; x < x_max; ++x) {
            const float dx = im.dx(y * im.w + x), dy = im.dy(y * im.w + x);
            dXX += dx * dx;
            dYY += dy * dy;
            dXY += dx * dy;
        }
    dXX = dXX / (2.0 * box_area);
    dYY = dYY / (2.0 * box_area);
    dXY = dXY / (2.0 * box_area);
    const float t = dXX + dYY;
    const float disc = t * t - 4 * (dXX * dYY - dXY * dXY);
    float s = 0.5 * (t - sqrtf(disc));
    if (std::isnan(s)) {           // x86's default quiet NaN, which is what the reference stores for a negative discriminant
        const uint32_t q = 0xFFC00000u;
        std::memcpy(&s, &q, 4);
    }
    return s;
}

float ic_angle(const Img &im, const int umax[], int u0, int v0) {
    float m_01 = 0, m_10 = 0;
    const int c = v0 * im.w + u0;
    for (int u = -HALF_PATCH_SIZE; u <= HALF_PATCH_SIZE; ++u) m_10 += u * im.I(c + u);
    const int step = im.w;
    for (int v = 1; v <= HALF_PATCH_SIZE; ++v) {
        float v_sum = 0;
        const int d = umax[v];
        for (int u = -d; u <= d; ++u) {
            const float val_plus = im.I(c + u + v * step), val_minus = im.I(c + u - v * step);
            v_sum += (val_plus - val_minus);
            m_10 += u * (val_plus + val_minus);
        }
        m_01 += v * v_sum;
    }
    return (float) std::atan2((double) m_01, (double) m_10);
}

void descriptor(const Img &im, const int32_t *pattern_table, float angle_in, int u0, int v0, uint8_t desc[32]) {
    const float factorPI = (float) (3.1415926535897932384626433832795 / 180.f);
    const float angle = angle_in * factorPI;
    const float a = (float) std::cos((double) angle), b = (float) std::sin((double) angle);
    const int c = v0 * im.w + u0, step = im.w;
    const int32_t *pattern = pattern_table;
    for (int i = 0; i < 32; ++i, pattern += 32) {
        int val = 0;
        for (int j = 0; j < 8; j++) {
            const int32_t *p = pattern + 4 * j;
            const float y0 = p[0] * b + p[1] * a, x0 = p[0] * a - p[1] * b;
            const float y1 = p[2] * b + p[3] * a, x1 = p[2] * a - p[3] * b;
            const int t0 = (int) im.I(c + int(y0) * step + int(x0));
            const int t1 = (int) im.I(c + int(y1) * step + int(x1));
            val |= (t0 < t1) << j;
        }
        desc[i] = (uint8_t) val;
    }
}

// a before b in the order rule: score descending, NaN after every number, ties in push order
bool before(float sa, int pa, float sb, int pb) {
    const bool na = std::isnan(sa), nb = std::isnan(sb);
    if (na != nb) return nb;
    if (!na && sa != sb) return sa > sb;
    return pa < pb;
}

}  // namespace

extern "C" {

void oracle_corners_suppress(int n, const float *u, const float *v, const float *score, const uint8_t *initial, uint8_t *out);

// the number of features DetectCorners can return for (w, h, nFeatures): cells x features per cell; -1 for a refused configuration
long long oracle_corners_capacity(int w, int h, int nFeatures) {
    Grid g;
    if (!make_grid(w, h, nFeatures, g)) return -1;
    return (long long) g.ncx * g.ncy * g.kcap;
}

// grid parameters: gs, gridX, gridY, skip, ncx, ncy, kcap; returns 0, or -1 for a refused configuration
int oracle_corners_grid(int w, int h, int nFeatures, int out7[7], float *nfeatInGrid) {
    Grid g;
    if (!make_grid(w, h, nFeatures, g)) return -1;
    const int o[7] = {g.gs, g.gridX, g.gridY, g.skip, g.ncx, g.ncy, g.kcap};
    std::memcpy(out7, o, sizeof(o));
    if (nfeatInGrid) *nfeatInGrid = g.nfeatInGrid;
    return 0;
}

void oracle_corners_umax(int out16[16]) { make_umax(out16); }

// level 0 of FrameHessian::makeImages (FrameHessian.cc:44-92): (I, dx, dy) per pixel; dx, dy are 0 in the first and last row
void oracle_corners_level0(int w, int h, const float *color, float *img3) {
    for (int i = 0; i < w * h; i++) { img3[3 * i] = color[i]; img3[3 * i + 1] = 0; img3[3 * i + 2] = 0; }
    for (int idx = w; idx < w * (h - 1); idx++) {
        float dx = 0.5f * (color[idx + 1] - color[idx - 1]);
        float dy = 0.5f * (color[idx + w] - color[idx - w]);
        if (std::isnan(dx) || std::fabs(dx) > 255.0) dx = 0;
        if (std::isnan(dy) || std::fabs(dy) > 255.0) dy = 0;
        img3[3 * idx + 1] = dx;
        img3[3 * idx + 2] = dy;
    }
}

// The restatement of DetectCorners. Outputs in the reference's order, `capacity` entries each (oracle_corners_capacity); u, v, score,
// is_corner, angle, descriptor (32 bytes per feature); cell (optional): the feature's cell as (gx - skip) * ncy + (gy - skip).
// Returns the number of corners, or -1 for a refused configuration / too small a capacity. *n_out gets the number of features.
int oracle_detect_corners(int w, int h, const float *img3, const float *B, int nFeatures, const int32_t *pattern, int capacity,
                          float *u_out, float *v_out, float *score_out, uint8_t *is_corner_out, float *angle_out, uint8_t *desc_out,
                          int32_t *cell_out, int *n_out) {
    Grid g;
    if (!make_grid(w, h, nFeatures, g)) return -1;
    if ((long long) g.ncx * g.ncy * g.kcap > capacity) return -1;
    const Img im{img3, w, h};
    int umax[HALF_PATCH_SIZE + 1];
    make_umax(umax);
    const int gs = g.gs;
    float maxScore = 0;
    int n = 0;
    struct Cand { int idx; float s; int push; };
    for (int gx = g.skip; gx < g.gridX - g.skip; gx++) {
        for (int gy = g.skip; gy < g.gridY - g.skip; gy++) {
            const int base = gy * gs * w + gx * gs;
            float maxGrad = 0;
            for (int x = 0; x < gs; x++)
                for (int y = 0; y < gs; y++) {
                    const float gr = abs_sq_grad(im, B, base + y * w + x);
                    if (gr > maxGrad) maxGrad = gr;
                }
            const double gradTH = (0.5 * maxGrad) > 5 ? 0.5 * maxGrad : 5;
            std::vector<Cand> cand;
            for (int x = 0; x < gs; x++)
                for (int y = 0; y < gs; y++)
                    if (abs_sq_grad(im, B, base + y * w + x) > gradTH) {
                        const float s = shi_tomasi(im, gx * gs + x, gy * gs + y);
                        cand.push_back({y * gs + x, s, (int) cand.size()});
                        if (s > maxScore) maxScore = s;
                    }
            // the order rule (insertion into a sorted list keeps push order among equals)
            std::vector<Cand> sorted;
            for (const Cand &c : cand) {
                size_t at = sorted.size();
                while (at > 0 && before(c.s, c.push, sorted[at - 1].s, sorted[at - 1].push)) at--;
                sorted.insert(sorted.begin() + at, c);
            }
            int picked = 0;
            for (const Cand &c : sorted) {
                u_out[n] = (float) (gx * gs + c.idx % gs);
                v_out[n] = (float) (gy * gs + c.idx / gs);
                score_out[n] = c.s;
                if (cell_out) cell_out[n] = (gx - g.skip) * g.ncy + (gy - g.skip);
                n++;
                picked++;
                if (picked > g.nfeatInGrid) break;
            }
        }
    }
    const float scoreTH = 0.01 * maxScore;
    std::vector<uint8_t> initial(n);
    for (int i = 0; i < n; i++) initial[i] = score_out[i] > scoreTH;
    oracle_corners_suppress(n, u_out, v_out, score_out, initial.data(), is_corner_out);
    int nc = 0;
    for (int k = 0; k < n; k++) {
        const bool c = is_corner_out[k];
        std::memset(desc_out + 32 * k, 0, 32);
        angle_out[k] = 0;
        if (c) {
            const int u0 = (int) u_out[k], v0 = (int) v_out[k];
            angle_out[k] = ic_angle(im, umax, u0, v0);
            descriptor(im, pattern, angle_out[k], u0, v0, desc_out + 32 * k);
            nc++;
        }
    }
    *n_out = n;
    return nc;
}

// suppression (:107-118): corner k survives unless another initial corner p closer than 5 pixels has p < k && s_p > s_k or
// p > k && s_p >= s_k, which is the outcome of the reference's pairwise loop. initial = score > scoreTH; out gets the surviving flags
void oracle_corners_suppress(int n, const float *u, const float *v, const float *score, const uint8_t *initial, uint8_t *out) {
    for (int k = 0; k < n; k++) {
        bool c = initial[k];
        for (int p = 0; c && p < n; p++) {
            if (p == k || !initial[p]) continue;
            const float dx = u[p] - u[k], dy = v[p] - v[k];
            if (dx * dx + dy * dy >= 25) continue;
            if ((p < k && score[p] > score[k]) || (p > k && score[p] >= score[k])) c = false;
        }
        out[k] = c;
    }
}

}
