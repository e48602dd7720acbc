# ORACLE — test infrastructure only: the RigSimulator checker (ref_bridge_rigsim.cpp).  Run after the main Makefile's
# `ref` target and sweepview.mk, whose object Camera.o and generated Eigen header it uses:
#   make -C oracle -f rigsim.mk
# The app is compiled where it lies under $(REF) with main renamed, against the sweep-view stand-ins plus rigsimshim/,
# through a generated copy of refshim/opencv2 whose core.hpp gains Vec::cross (rigsim_vec_extra.h) and ends with
# rigsim_extra.h (norm(Vec), Vec / float, float INTER_AREA resize, vconcat, Eigen::Map); the stand-in's resize is
# renamed resizeShim there and its aborting vconcat dropped.  Vec's layout is unchanged, so the app links with the
# objects built against refshim/; the app's objects come first on the link line, so its resize and vconcat are the ones
# every object calls (the others' behaviour is unchanged: anything but float INTER_AREA goes on to resizeShim).
CXX ?= g++
REF ?= /root/reference
SOFLAGS := -shared -pthread -Wl,-Bsymbolic -Wl,--exclude-libs,ALL
INC := -I rigsimshim -I _ref/rigsiminc -I _ref/sweepinc -I sweepshim -I refshim -I $(REF)
FLAGS := -std=c++17 -O3 -funroll-loops -ffp-contract=off -fPIC -pthread -include opencv2/opencv.hpp $(INC)
SHIM := $(shell find rigsimshim sweepshim refshim -type f) ../include/derp_b200.h
GEN := _ref/rigsiminc/opencv2/core.hpp _ref/sweepinc/Eigen/Geometry
LINKED := _ref/Camera.o

all: $(if $(wildcard $(REF)/source/rig/RigSimulator.cpp),_ref/librigsim_ref.so)

_ref/rigsiminc/opencv2/core.hpp: refshim/opencv2/core.hpp $(wildcard refshim/opencv2/*.hpp refshim/opencv2/core/*.hpp)
	@mkdir -p $(dir $@)core
	cp refshim/opencv2/calib3d.hpp refshim/opencv2/highgui.hpp refshim/opencv2/imgproc.hpp $(dir $@)
	cp refshim/opencv2/core/types.hpp $(dir $@)core/
	{ echo '#include "rigsim_vec_extra.h"'; \
	  sed -e 's|^  static Vec all(T v) {|  REFSHIM_RIGSIM_VEC_EXTRA\n&|' \
	      -e 's|#include "../../cvprims.h"|#include "$(CURDIR)/cvprims.h"|' \
	      -e 's|^inline void resize(const Mat& src, Mat& dst,|inline void resizeShim(const Mat\& src, Mat\& dst,|' \
	      -e '/^inline void vconcat(/d' $<; \
	  echo '#include "rigsim_extra.h"'; } > $@

_ref/rigsim_app.o: $(GEN) $(SHIM)
	$(CXX) $(FLAGS) -w -Dmain=ref_rigsim_main -c $(REF)/source/rig/RigSimulator.cpp -o $@
_ref/rigsim_bridge.o: ref_bridge_rigsim.cpp $(GEN) $(SHIM)
	$(CXX) $(FLAGS) -Wall -c $< -o $@
_ref/librigsim_ref.so: _ref/rigsim_app.o _ref/rigsim_bridge.o $(LINKED)
	$(CXX) $(SOFLAGS) -o $@ $^

.PHONY: all
.SECONDARY:
