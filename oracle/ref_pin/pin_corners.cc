// PIN of the corner-detection restatement (../corners.cc) against the reference's own FeatureDetector.cc — TEST INFRASTRUCTURE ONLY,
// built by ../corners.mk where a reference checkout exists. The reference's src/frontend/FeatureDetector.cc, src/internal/FrameHessian.cc
// and src/Setting.cc are compiled unmodified, against ../ref_shim/ref_classes.h (the Frame stand-in) and ref_shim/corners/opencv2 (cvFloor,
// cvCeil, cvRound, CV_PI, no-op drawing). This file gives them a small C interface: the frame's pyramid comes from the reference's own
// FrameHessian::makeImages with a CalibHessian whose B is the caller's, and FeatureDetector::DetectCorners runs on it. The comparison
// with the restatement (which cells' picks differ, which angles / descriptors differ) is made by tests/corners_oracle.py, which loads
// this library and liboracle_corners.so side by side.
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstring>
#include <vector>

#include "frontend/FeatureDetector.h"
#include "Feature.h"

namespace ldso {
extern int bit_pattern_31_[256 * 4];
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
        std::vector<float> col(color, color + (size_t) w * h);          // makeImages takes a non-const image
        frame->frameHessian->makeImages(col.data(), HC);
    }
    ~RefFrame() {
        frame->features.clear();
        frame->frameHessian->frame.reset();      // the FrameHessian holds its Frame: break the cycle
        frame->frameHessian.reset();
    }
};
}  // namespace

extern "C" {

void cref_pattern(int32_t out[1024]) { std::memcpy(out, ldso::bit_pattern_31_, sizeof(int32_t) * 1024); }

// the reference's pyramid level 0 (I, dx, dy; w*h*3 floats) and absSquaredGrad[0] (w*h floats) for (color, B)
void cref_level0(int w, int h, const float *color, const float *B, float *img3, float *abs_grad) {
    RefFrame f(w, h, color, B);
    for (int i = 0; i < w * h; i++)
        for (int k = 0; k < 3; k++) img3[3 * i + k] = f.frame->frameHessian->dIp[0][i][k];
    std::memcpy(abs_grad, f.frame->frameHessian->absSquaredGrad[0], sizeof(float) * w * h);
}

// FeatureDetector::DetectCorners(nFeatures, frame) on the reference's makeImages of (color, B); B NULL keeps CalibHessian's identity.
// Fills up to `capacity` features in the reference's order; returns DetectCorners' value, or -1 when more than capacity came back.
int cref_detect(int w, int h, const float *color, const float *B, int nFeatures, int capacity, float *u, float *v, float *score,
                uint8_t *is_corner, float *angle, uint8_t *desc, int *n_out) {
    RefFrame f(w, h, color, B);
    ldso::FeatureDetector det;
    const int nc = det.DetectCorners(nFeatures, f.frame);
    const int n = (int) f.frame->features.size();
    *n_out = n;
    if (n > capacity) return -1;
    for (int i = 0; i < n; i++) {
        const ldso::Feature &ft = *f.frame->features[i];
        u[i] = ft.uv[0]; v[i] = ft.uv[1]; score[i] = ft.score; is_corner[i] = ft.isCorner; angle[i] = ft.angle;
        std::memcpy(desc + 32 * i, ft.descriptor, 32);
    }
    return nc;
}

// seconds per DetectCorners call on a frame whose pyramid is built (the feature list is cleared between calls, as each new keyframe
// starts with an empty one): the median of `runs` runs of `reps` calls each
double cref_time(int w, int h, const float *color, const float *B, int nFeatures, int reps, int runs) {
    RefFrame f(w, h, color, B);
    ldso::FeatureDetector det;
    std::vector<double> t;
    for (int k = 0; k < runs; k++) {
        const auto t0 = std::chrono::steady_clock::now();
        for (int i = 0; i < reps; i++) {
            f.frame->features.clear();
            f.frame->features.reserve(nFeatures);
            det.DetectCorners(nFeatures, f.frame);
        }
        t.push_back(std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() / reps);
    }
    std::sort(t.begin(), t.end());
    return t[t.size() / 2];
}

}
