# ORACLE — test infrastructure only: the RigAnalyzer checker (ref_bridge_riganalyzer.cpp).  Run after the main
# Makefile's `ref` target and sweepview.mk, whose object Camera.o and generated Eigen header it uses:
#   make -C oracle -f riganalyzer.mk
# The app is compiled where it lies under $(REF) with main renamed, against the sweep-view stand-ins plus
# riganalyzershim/ (gflags::GetArgv) and a generated copy of _ref/sweepinc/Eigen/Geometry that gains the members of
# riganalyzershim/riganalyzer_extra.h (layouts unchanged, so it links with the objects built against refshim/).  The
# app uses fmt::format without including it (the real build reaches it through other headers): it is force-included.
CXX ?= g++
REF ?= /root/reference
SOFLAGS := -shared -pthread -Wl,-Bsymbolic -Wl,--exclude-libs,ALL
INC := -I riganalyzershim -I _ref/riganalyzerinc -I _ref/sweepinc -I sweepshim -I refshim -I $(REF)
FLAGS := -std=c++17 -O3 -funroll-loops -ffp-contract=off -fPIC -pthread -include opencv2/opencv.hpp $(INC)
SHIM := $(shell find riganalyzershim sweepshim refshim -type f)
GEN := _ref/riganalyzerinc/Eigen/Geometry
LINKED := _ref/Camera.o

all: $(if $(wildcard $(REF)/source/rig/RigAnalyzer.cpp),_ref/libriganalyzer_ref.so)

$(GEN): _ref/sweepinc/Eigen/Geometry riganalyzershim/riganalyzer_extra.h riganalyzershim/riganalyzer_types.h
	@mkdir -p $(dir $@)
	{ echo '#include "riganalyzer_extra.h"'; \
	  sed -e 's|^  static Matrix UnitX() {|  REFSHIM_RA_VECTOR_EXTRA\n&|' \
	      -e 's|^  explicit Matrix(Index n) : v((size_t)n) {}|&\n  REFSHIM_RA_DYNVEC_EXTRA|' \
	      -e 's|^    S\* p;  // first element, stride 3|&\n    REFSHIM_RA_COL_EXTRA|' $<; \
	  echo '#include "riganalyzer_types.h"'; } > $@

_ref/riganalyzer_app.o: $(GEN) $(SHIM)
	$(CXX) $(FLAGS) -include fmt/format.h -w -Dmain=ref_rig_analyzer_main -c $(REF)/source/rig/RigAnalyzer.cpp -o $@
_ref/riganalyzer_bridge.o: ref_bridge_riganalyzer.cpp $(GEN) $(SHIM)
	$(CXX) $(FLAGS) -Wall -c $< -o $@
_ref/libriganalyzer_ref.so: _ref/riganalyzer_app.o _ref/riganalyzer_bridge.o $(LINKED)
	$(CXX) $(SOFLAGS) -o $@ $^

.PHONY: all
.SECONDARY:
