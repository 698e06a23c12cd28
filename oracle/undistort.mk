# ORACLE build of the per-frame undistortion — test infrastructure only (make -f undistort.mk, from this directory).
#   liboracle_undistort.so   the dependency-free restatement (undistort.cc), -ffp-contract=off like liboracle.so
# and, where a reference checkout exists (REF, passed by __graft_entry__.build()), under _ref/ (git-ignored):
#   pin_undistort            the pin: the reference's Undistort.cc and Setting.cc, compiled unmodified, against the restatement
#   libref_undistort_pin.so  the same reference objects behind ref_pin/undistort_ref.cc's C interface, same flags
#   libref_undistort.so      ... with the reference's Release flags (-O3 -march=native): the CPU leg of tools/undistort_time.py
# The reference's headers see ref_shim/NumTypes.h for Eigen (ref_shim/undistort/Eigen/Core adds matrix printing). Undistort.cc is
# compiled without -Dprivate=public (its <sstream> does not survive it); undistort_ref.cc, which reads the private tables, with it.
# The two libraries keep the C++ runtime they were linked with to themselves (-Bsymbolic, --exclude-libs,ALL): loaded into a process
# that already exports a differently built copy of it (torch's libraries do), their iostreams would otherwise run half in each copy.
CXX ?= g++
REF ?= $(abspath ../../reference)

all: liboracle_undistort.so

liboracle_undistort.so: undistort.cc
	$(CXX) -std=c++17 -O3 -march=native -fPIC -shared -Wall -ffp-contract=off undistort.cc -o $@

ref_pin: _ref/pin_undistort _ref/libref_undistort_pin.so _ref/libref_undistort.so

UINC = -Iref_shim/undistort -Iref_shim -I$(REF)/include
UPIN = -std=c++17 -O2 -msse4.1 -fPIC -ffp-contract=off -pthread -w $(UINC)
UFAST = -std=c++17 -O3 -march=native -DNDEBUG -fPIC -pthread -w $(UINC)
UHDR = ref_shim/NumTypes.h ref_shim/undistort/Eigen/Core

_ref/Undistort_pin.o: $(REF)/src/frontend/Undistort.cc $(UHDR)
	mkdir -p _ref
	$(CXX) $(UPIN) -c $< -o $@
_ref/Setting_upin.o: $(REF)/src/Setting.cc $(UHDR)
	mkdir -p _ref
	$(CXX) $(UPIN) -c $< -o $@
_ref/undistort_ref_pin.o: ref_pin/undistort_ref.cc $(UHDR)
	mkdir -p _ref
	$(CXX) $(UPIN) -Dprivate=public -c $< -o $@
_ref/undistort_oracle_pin.o: undistort.cc
	mkdir -p _ref
	$(CXX) $(UPIN) -c $< -o $@
UPINOBJ = _ref/Undistort_pin.o _ref/Setting_upin.o _ref/undistort_ref_pin.o

_ref/pin_undistort: ref_pin/pin_undistort.cc $(UPINOBJ) _ref/undistort_oracle_pin.o
	$(CXX) $(UPIN) ref_pin/pin_undistort.cc $(UPINOBJ) _ref/undistort_oracle_pin.o -o $@

_ref/libref_undistort_pin.so: $(UPINOBJ)
	$(CXX) $(UPIN) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL $(UPINOBJ) -o $@

_ref/libref_undistort.so: ref_pin/undistort_ref.cc $(REF)/src/frontend/Undistort.cc $(REF)/src/Setting.cc $(UHDR)
	mkdir -p _ref
	$(CXX) $(UFAST) -c $(REF)/src/frontend/Undistort.cc -o _ref/Undistort_fast.o
	$(CXX) $(UFAST) -c $(REF)/src/Setting.cc -o _ref/Setting_ufast.o
	$(CXX) $(UFAST) -Dprivate=public -c ref_pin/undistort_ref.cc -o _ref/undistort_ref_fast.o
	$(CXX) $(UFAST) -shared -Wl,-Bsymbolic -Wl,--exclude-libs,ALL _ref/Undistort_fast.o _ref/Setting_ufast.o _ref/undistort_ref_fast.o -o $@

.PHONY: all ref_pin
