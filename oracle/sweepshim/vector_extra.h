// ORACLE — TEST INFRASTRUCTURE ONLY.  Members of the fixed-size Eigen vector stand-in that source/rig/RigTransform.h
// needs (see geometry_extra.h); sweepview.mk inserts the macro into the generated copy of ../refshim/Eigen/Geometry.
#pragma once
#define REFSHIM_SWEEP_VECTOR_EXTRA                       \
  static Matrix UnitY() {                                \
    Matrix r = Zero();                                   \
    r.v[1] = 1;                                          \
    return r;                                            \
  }                                                      \
  static Matrix UnitZ() {                                \
    Matrix r = Zero();                                   \
    r.v[2] = 1;                                          \
    return r;                                            \
  }                                                      \
  explicit Matrix(const S* p) {                          \
    for (int i = 0; i < N; ++i) v[i] = p[i];             \
  }
