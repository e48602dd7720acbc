// ORACLE — TEST INFRASTRUCTURE ONLY.  Vec::cross for the reference's RigSimulator.cpp (RaytracingPrimitives.h:47-69);
// rigsim.mk inserts the macro into a generated copy of ../refshim/opencv2/core.hpp (layout of Vec unchanged).
// matx.hpp's Vec<_Tp, 3>::cross: the three products and differences in the element type, in this order.
#pragma once
#define REFSHIM_RIGSIM_VEC_EXTRA                                                  \
  Vec cross(const Vec& b) const {                                                 \
    static_assert(N == 3, "cross");                                               \
    return Vec(T(val[1] * b.val[2] - val[2] * b.val[1]), T(val[2] * b.val[0] - val[0] * b.val[2]), \
               T(val[0] * b.val[1] - val[1] * b.val[0]));                         \
  }
