# ORACLE build of DSO's pixel selection — test infrastructure only (make -f pixsel.mk, from this directory).
#   liboracle_pixsel.so      the dependency-free restatement (pixsel.cc), -ffp-contract=off like liboracle.so
# and, where a reference checkout exists (REF, passed by __graft_entry__.build()), under _ref/ (git-ignored):
#   libref_pixsel_pin.so     the pin: the reference's PixelSelector2.cc, FrameHessian.cc and Setting.cc, compiled unmodified, behind
#                            ref_pin/pin_pixsel.cc's C interface (tests/pixsel_oracle.py compares it with the restatement)
#   libref_pixsel.so         ... with the reference's Release flags (-O3 -march=native): the CPU leg of tools/pixsel_time.py
# Same headers and flags as corners.mk.
CXX ?= g++
REF ?= $(abspath ../../reference)

all: liboracle_pixsel.so

liboracle_pixsel.so: pixsel.cc
	$(CXX) -std=c++17 -O3 -march=native -fPIC -shared -Wall -ffp-contract=off pixsel.cc -o $@

ref_pin: _ref/libref_pixsel_pin.so _ref/libref_pixsel.so

CINC = -Iref_shim/corners -Iref_shim -I$(REF)/include -include ref_shim/ref_classes.h
CPIN = -std=c++17 -O2 -msse4.1 -fPIC -ffp-contract=off -pthread -w -Dprivate=public $(CINC)
CFAST = -std=c++17 -O3 -march=native -DNDEBUG -fPIC -pthread -w -Dprivate=public $(CINC)
CHDR = ref_shim/NumTypes.h ref_shim/ref_classes.h ref_shim/opencv2/opencv.hpp ref_shim/corners/opencv2/opencv.hpp
PREF = $(REF)/src/frontend/PixelSelector2.cc $(REF)/src/internal/FrameHessian.cc $(REF)/src/Setting.cc

_ref/libref_pixsel_pin.so: ref_pin/pin_pixsel.cc $(PREF) $(CHDR)
	mkdir -p _ref
	$(CXX) $(CPIN) -c $(REF)/src/frontend/PixelSelector2.cc -o _ref/PixelSelector2_ppin.o
	$(CXX) $(CPIN) -c $(REF)/src/internal/FrameHessian.cc -o _ref/FrameHessian_ppin.o
	$(CXX) $(CPIN) -c $(REF)/src/Setting.cc -o _ref/Setting_ppin.o
	$(CXX) $(CPIN) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL ref_pin/pin_pixsel.cc _ref/PixelSelector2_ppin.o \
	    _ref/FrameHessian_ppin.o _ref/Setting_ppin.o -o $@

_ref/libref_pixsel.so: ref_pin/pin_pixsel.cc $(PREF) $(CHDR)
	mkdir -p _ref
	$(CXX) $(CFAST) -c $(REF)/src/frontend/PixelSelector2.cc -o _ref/PixelSelector2_pfast.o
	$(CXX) $(CFAST) -c $(REF)/src/internal/FrameHessian.cc -o _ref/FrameHessian_pfast.o
	$(CXX) $(CFAST) -c $(REF)/src/Setting.cc -o _ref/Setting_pfast.o
	$(CXX) $(CFAST) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL ref_pin/pin_pixsel.cc _ref/PixelSelector2_pfast.o \
	    _ref/FrameHessian_pfast.o _ref/Setting_pfast.o -o $@

.PHONY: all ref_pin
