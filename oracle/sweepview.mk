# ORACLE — test infrastructure only: the two sweep-view checkers (ref_bridge_sweepview.cpp).  Run after the main
# Makefile's `ref` target, whose objects (Camera.o, CvUtil.o, ImageUtil.o) these libraries link:
#   make -C oracle -f sweepview.mk
# Each app is compiled where it lies under $(REF) with main renamed, against sweepshim/ (gflags DEFINE_*, the
# <opencv2/opencv.hpp> umbrella) and a generated copy of refshim/Eigen/Geometry that gains the vector members and the
# Transform / Quaternion types of sweepshim/ (layout unchanged, so it links with the objects built against refshim/).
CXX ?= g++
REF ?= /root/reference
SOFLAGS := -shared -pthread -Wl,-Bsymbolic -Wl,--exclude-libs,ALL
INC := -I _ref/sweepinc -I sweepshim -I refshim -I $(REF)
FLAGS := -std=c++17 -O3 -funroll-loops -ffp-contract=off -fPIC -pthread -include opencv2/opencv.hpp $(INC)
SHIM := $(shell find sweepshim refshim -type f) ../include/derp_sweepview.h ../include/derp_b200.h
LINKED := _ref/Camera.o _ref/CvUtil.o _ref/ImageUtil.o

all: $(if $(wildcard $(REF)/source/render/GenerateEquirect.cpp),_ref/libsweep_overlaps_ref.so _ref/libsweep_equirect_ref.so)

_ref/sweepinc/Eigen/Geometry: refshim/Eigen/Geometry sweepshim/vector_extra.h sweepshim/geometry_extra.h
	@mkdir -p $(dir $@)
	{ echo '#include "vector_extra.h"'; \
	  sed -e 's|^  static Matrix UnitX() {|  REFSHIM_SWEEP_VECTOR_EXTRA\n&|' \
	      -e 's|#include "DynamicMatrix.h"|#include "$(CURDIR)/refshim/Eigen/DynamicMatrix.h"|' $<; \
	  echo '#include "geometry_extra.h"'; } > $@

_ref/sweep_%_app.o: _ref/sweepinc/Eigen/Geometry $(SHIM)
	$(CXX) $(FLAGS) -w -Dmain=ref_sweep_$*_main -c $(REF)/source/render/$(APP_$*).cpp -o $@
APP_overlaps := GenerateCameraOverlaps
APP_equirect := GenerateEquirect

_ref/sweep_overlaps_bridge.o: ref_bridge_sweepview.cpp _ref/sweepinc/Eigen/Geometry $(SHIM)
	$(CXX) $(FLAGS) -Wall -DSWEEP_OVERLAPS -c $< -o $@
_ref/sweep_equirect_bridge.o: ref_bridge_sweepview.cpp _ref/sweepinc/Eigen/Geometry $(SHIM)
	$(CXX) $(FLAGS) -Wall -DSWEEP_EQUIRECT -c $< -o $@

_ref/libsweep_%_ref.so: _ref/sweep_%_app.o _ref/sweep_%_bridge.o $(LINKED)
	$(CXX) $(SOFLAGS) -o $@ $^

.PHONY: all
.SECONDARY:
