// ORACLE: LDSO's per-frame undistortion restated without dependencies — TEST INFRASTRUCTURE ONLY (built by undistort.mk with
// -ffp-contract=off, like liboracle.so). PhotometricUndistorter::processFrame<T> (src/frontend/Undistort.cc:189-227) followed by
// Undistort::undistort<T>'s bilinear remap (Undistort.cc:357-457), working from the tables the reference builds (remapX / remapY,
// G, vignetteMapInv), with one defined difference: the photometric image is followed by wOrg + 1 zero pixels, so the two offsets the
// reference's range check lets through although their taps run past the end of the image (src_offset == (hOrg-1)*wOrg and
// (hOrg-1)*wOrg - 1) read 0 there. The benchmark noise settings (benchmark_varNoise, benchmark_varBlurNoise) are not restated.
#include <cstdint>
#include <cstring>
#include <vector>

namespace {

template<typename T>
void photometric(const T *raw, int n, const float *G, const float *vinv, int mode, float exposure, float factor, float *data) {
    if (G == nullptr || exposure <= 0 || mode == 0) {           // !valid || exposure_time <= 0 || setting_photometricCalibration == 0
        for (int i = 0; i < n; i++) data[i] = factor * raw[i];
    } else {
        for (int i = 0; i < n; i++) data[i] = G[raw[i]];
        if (mode == 2)
            for (int i = 0; i < n; i++) data[i] *= vinv[i];
    }
}

template<typename T>
void undistort(int wOrg, int hOrg, int w, int h, const float *remapX, const float *remapY, const float *G, const float *vinv, int mode,
               const T *raw, float exposure, float factor, float *out, unsigned char *past_end) {
    const int nOrg = wOrg * hOrg;
    std::vector<float> in(nOrg + wOrg + 1, 0.f);                // the zero padding of the edge rule
    photometric(raw, nOrg, G, vinv, mode, exposure, factor, in.data());
    if (remapX == nullptr) {                                    // passthrough (wOrg == w, hOrg == h)
        std::memcpy(out, in.data(), sizeof(float) * nOrg);
        if (past_end) std::memset(past_end, 0, nOrg);
        return;
    }
    for (int idx = w * h - 1; idx >= 0; idx--) {
        float xx = remapX[idx];
        float yy = remapY[idx];
        if (past_end) past_end[idx] = 0;
        if (xx < 0) {
            out[idx] = 0;
            continue;
        }
        const int xxi = xx;
        const int yyi = yy;
        xx -= xxi;
        yy -= yyi;
        const float xxyy = xx * yy;
        const int src_offset = xxi + yyi * wOrg;
        if (src_offset < 0 || src_offset > (hOrg - 1) * wOrg) {
            out[idx] = 0;
            continue;
        }
        const float *src = in.data() + src_offset;
        out[idx] = xxyy * src[1 + wOrg] + (yy - xxyy) * src[wOrg] + (xx - xxyy) * src[1] + (1 - xx - yy + xxyy) * src[0];
        if (past_end) past_end[idx] = src_offset + 1 + wOrg >= nOrg;
    }
}

}  // namespace

extern "C" {

// out: w*h floats (wOrg*hOrg in passthrough, remapX == NULL); past_end (optional): 1 where a tap lies at index >= wOrg*hOrg, i.e.
// where the reference reads past the end of its buffer. Returns the exposure time processFrame stores (1 when !use_exposure).
float oracle_undistort(int wOrg, int hOrg, int w, int h, const float *remapX, const float *remapY, const float *G, const float *vinv,
                       int mode, int use_exposure, const void *raw, int bytes_per_pixel, float exposure, float factor, float *out,
                       unsigned char *past_end) {
    if (bytes_per_pixel == 1)
        undistort(wOrg, hOrg, w, h, remapX, remapY, G, vinv, mode, (const uint8_t *) raw, exposure, factor, out, past_end);
    else
        undistort(wOrg, hOrg, w, h, remapX, remapY, G, vinv, mode, (const uint16_t *) raw, exposure, factor, out, past_end);
    return use_exposure ? exposure : 1.f;
}

}
