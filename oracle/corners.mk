# ORACLE build of the keyframe corner detection — test infrastructure only (make -f corners.mk, from this directory).
#   liboracle_corners.so     the dependency-free restatement (corners.cc), -ffp-contract=off like liboracle.so
# and, where a reference checkout exists (REF, passed by __graft_entry__.build()), under _ref/ (git-ignored):
#   libref_corners_pin.so    the pin: the reference's FeatureDetector.cc, FrameHessian.cc and Setting.cc, compiled unmodified, behind
#                            ref_pin/pin_corners.cc's C interface (tests/corners_oracle.py compares it with the restatement)
#   libref_corners.so        ... with the reference's Release flags (-O3 -march=native): the CPU leg of tools/corners_time.py
# The reference's headers see ref_shim/NumTypes.h for Eigen, ref_shim/ref_classes.h for Frame, and ref_shim/corners/opencv2 (searched
# first) for the OpenCV names FeatureDetector.cc uses. The libraries keep their C++ runtime to themselves (see undistort.mk).
CXX ?= g++
REF ?= $(abspath ../../reference)

all: liboracle_corners.so

liboracle_corners.so: corners.cc
	$(CXX) -std=c++17 -O3 -march=native -fPIC -shared -Wall -ffp-contract=off corners.cc -o $@

ref_pin: _ref/libref_corners_pin.so _ref/libref_corners.so

CINC = -Iref_shim/corners -Iref_shim -I$(REF)/include -include ref_shim/ref_classes.h
CPIN = -std=c++17 -O2 -msse4.1 -fPIC -ffp-contract=off -pthread -w -Dprivate=public $(CINC)
CFAST = -std=c++17 -O3 -march=native -DNDEBUG -fPIC -pthread -w -Dprivate=public $(CINC)
CHDR = ref_shim/NumTypes.h ref_shim/ref_classes.h ref_shim/opencv2/opencv.hpp ref_shim/corners/opencv2/opencv.hpp
CREF = $(REF)/src/frontend/FeatureDetector.cc $(REF)/src/internal/FrameHessian.cc $(REF)/src/Setting.cc

_ref/libref_corners_pin.so: ref_pin/pin_corners.cc $(CREF) $(CHDR)
	mkdir -p _ref
	$(CXX) $(CPIN) -c $(REF)/src/frontend/FeatureDetector.cc -o _ref/FeatureDetector_cpin.o
	$(CXX) $(CPIN) -c $(REF)/src/internal/FrameHessian.cc -o _ref/FrameHessian_cpin.o
	$(CXX) $(CPIN) -c $(REF)/src/Setting.cc -o _ref/Setting_cpin.o
	$(CXX) $(CPIN) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL ref_pin/pin_corners.cc _ref/FeatureDetector_cpin.o \
	    _ref/FrameHessian_cpin.o _ref/Setting_cpin.o -o $@

_ref/libref_corners.so: ref_pin/pin_corners.cc $(CREF) $(CHDR)
	mkdir -p _ref
	$(CXX) $(CFAST) -c $(REF)/src/frontend/FeatureDetector.cc -o _ref/FeatureDetector_cfast.o
	$(CXX) $(CFAST) -c $(REF)/src/internal/FrameHessian.cc -o _ref/FrameHessian_cfast.o
	$(CXX) $(CFAST) -c $(REF)/src/Setting.cc -o _ref/Setting_cfast.o
	$(CXX) $(CFAST) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL ref_pin/pin_corners.cc _ref/FeatureDetector_cfast.o \
	    _ref/FrameHessian_cfast.o _ref/Setting_cfast.o -o $@

.PHONY: all ref_pin
