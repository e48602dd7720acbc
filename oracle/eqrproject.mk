# ORACLE — test infrastructure only: the ProjectEquirectsToCameras checker (ref_bridge_eqrproject.cpp).  Run after the
# main Makefile's `ref` target and sweepview.mk, whose objects (Camera.o, CvUtil.o, ImageUtil.o) and generated Eigen
# header it uses:
#   make -C oracle -f eqrproject.mk
# The app is compiled where it lies under $(REF) with main renamed, so that its rescaleCameras and flags are its own,
# against the sweep-view checkers' stand-ins (sweepshim/) plus eqrprojectshim/ (gflags::SetUsageMessage).
CXX ?= g++
REF ?= /root/reference
SOFLAGS := -shared -pthread -Wl,-Bsymbolic -Wl,--exclude-libs,ALL
INC := -I eqrprojectshim -I _ref/sweepinc -I sweepshim -I refshim -I $(REF)
FLAGS := -std=c++17 -O3 -funroll-loops -ffp-contract=off -fPIC -pthread -include opencv2/opencv.hpp $(INC)
SHIM := $(shell find eqrprojectshim sweepshim refshim -type f) ../include/derp_sweepview.h ../include/derp_b200.h
LINKED := _ref/Camera.o _ref/CvUtil.o _ref/ImageUtil.o

all: $(if $(wildcard $(REF)/source/conversion/ProjectEquirectsToCameras.cpp),_ref/libeqrproject_ref.so)

_ref/eqrproject_app.o: _ref/sweepinc/Eigen/Geometry $(SHIM)
	$(CXX) $(FLAGS) -w -Dmain=ref_eqrproject_main -c $(REF)/source/conversion/ProjectEquirectsToCameras.cpp -o $@
_ref/eqrproject_bridge.o: ref_bridge_eqrproject.cpp _ref/sweepinc/Eigen/Geometry $(SHIM)
	$(CXX) $(FLAGS) -Wall -c $< -o $@
_ref/libeqrproject_ref.so: _ref/eqrproject_app.o _ref/eqrproject_bridge.o $(LINKED)
	$(CXX) $(SOFLAGS) -o $@ $^

.PHONY: all
.SECONDARY:
