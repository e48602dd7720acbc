# ORACLE — test infrastructure only: the two equirect-mesh checkers of include/derp_eqrmesh.h.
#   make -C oracle -f eqrmesh.mk
#   libeqrmesh_oracle.so        the CPU restatement (eqrmesh_oracle.cpp), built everywhere
#   _ref/libeqrmesh_ref.so      the reference's own MeshUtil.h / MeshSimplifier.cpp (ref_bridge_eqrmesh.cpp); built only
#                               where $(REF) exists, after the main Makefile's `ref` target, whose objects it links
# Flags as in the main Makefile (the reference build's -O3 -funroll-loops, no FMA contraction).
CXX ?= g++
REF ?= /root/reference
CXXFLAGS := -std=c++17 -O3 -funroll-loops -ffp-contract=off -fPIC -Wall -Wextra -Wno-unused-parameter -pthread
SOFLAGS := -shared -pthread -Wl,-Bsymbolic -Wl,--exclude-libs,ALL
REF_FLAGS := -std=c++17 -O3 -funroll-loops -ffp-contract=off -fPIC -pthread -I refshim -I $(REF)
HDRS := cvprims.h cvprims_linear.h ../include/derp_eqrmesh.h ../include/derp_b200.h
LINKED := _ref/MeshSimplifier.o _ref/Camera.o _ref/CvUtil.o _ref/ImageUtil.o

all: libeqrmesh_oracle.so $(if $(wildcard $(REF)/source/render/MeshUtil.h),_ref/libeqrmesh_ref.so)

libeqrmesh_oracle.so: eqrmesh_oracle.cpp $(HDRS)
	$(CXX) $(CXXFLAGS) $(SOFLAGS) -o $@ eqrmesh_oracle.cpp

_ref/eqrmesh_bridge.o: ref_bridge_eqrmesh.cpp $(HDRS) $(shell find refshim -type f)
	@mkdir -p _ref
	$(CXX) $(REF_FLAGS) -Wall -c $< -o $@

_ref/libeqrmesh_ref.so: _ref/eqrmesh_bridge.o $(LINKED)
	$(CXX) $(SOFLAGS) -o $@ $^

.PHONY: all
