// STAND-IN for <opencv2/opencv.hpp> as src/frontend/FeatureDetector.cc uses it — TEST INFRASTRUCTURE ONLY (see ../../NumTypes.h).
// It adds to the back end's stand-in (../../opencv2/opencv.hpp, which stays as it is) what the detector names: cvFloor, cvCeil and
// cvRound for the umax table, CV_PI for the descriptor's angle, and DrawFeatures' drawing calls, which do nothing here.
#pragma once
#include "../../opencv2/opencv.hpp"
#include <cmath>
#include <string>
#define CV_PI 3.1415926535897932384626433832795
inline int cvFloor(double v) { return (int) std::floor(v); }
inline int cvCeil(double v) { return (int) std::ceil(v); }
inline int cvRound(double v) { return (int) std::lrint(v); }     // round half to even, as OpenCV's SSE2 conversion does
namespace cv {
struct Point2f { float x, y; Point2f(float x_, float y_) : x(x_), y(y_) {} };
struct Scalar { double v[4]; Scalar(double a, double b, double c, double d = 0) : v{a, b, c, d} {} };
inline void circle(Mat &, Point2f, int, const Scalar &, int = 1) {}
inline void imshow(const std::string &, const Mat &) {}
inline int waitKey(int = 0) { return -1; }
}
