// ORACLE — TEST INFRASTRUCTURE ONLY.  Members of the Eigen stand-in that source/rig/RigAnalyzer.cpp needs beyond the
// sweep-view checkers' (riganalyzer.mk inserts the macros into a generated copy of _ref/sweepinc/Eigen/Geometry; the
// layouts are unchanged, so the app links with the objects built against ../refshim):
//   - Vector3: operator*=(scalar) and normalize() (Eigen: v /= sqrt(squaredNorm()) when squaredNorm() > 0);
//   - VectorXd: minCoeff, maxCoeff, and array() == k / >= k with count();
//   - Matrix3::col(j): readable as a Vector3 and negatable (setRotation(xform.col(2), xform.col(1), -xform.col(0))).
#pragma once
#define REFSHIM_RA_VECTOR_EXTRA                  \
  Matrix& operator*=(S s) {                      \
    for (int i = 0; i < N; ++i) v[i] = v[i] * s; \
    return *this;                                \
  }                                              \
  void normalize() {                             \
    const S z = squaredNorm();                   \
    if (z > S(0)) {                              \
      const S n = std::sqrt(z);                  \
      for (int i = 0; i < N; ++i) v[i] = v[i] / n; \
    }                                            \
  }
#define REFSHIM_RA_DYNVEC_EXTRA                                                       \
  S minCoeff() const {                                                                \
    S m = v[0];                                                                       \
    for (size_t i = 1; i < v.size(); ++i) m = v[i] < m ? v[i] : m;                    \
    return m;                                                                         \
  }                                                                                   \
  S maxCoeff() const {                                                                \
    S m = v[0];                                                                       \
    for (size_t i = 1; i < v.size(); ++i) m = v[i] > m ? v[i] : m;                    \
    return m;                                                                         \
  }                                                                                   \
  struct CoeffCount {                                                                 \
    Index n;                                                                          \
    Index count() const { return n; }                                                 \
  };                                                                                  \
  struct ArrayView {                                                                  \
    const std::vector<S>* v;                                                          \
    CoeffCount operator==(S k) const {                                                \
      Index n = 0;                                                                    \
      for (const S& x : *v) n += x == k;                                              \
      return CoeffCount{n};                                                           \
    }                                                                                 \
    CoeffCount operator>=(S k) const {                                                \
      Index n = 0;                                                                    \
      for (const S& x : *v) n += x >= k;                                              \
      return CoeffCount{n};                                                           \
    }                                                                                 \
  };                                                                                  \
  ArrayView array() const { return ArrayView{&v}; }
#define REFSHIM_RA_COL_EXTRA                                       \
  operator V3() const { return V3(p[0], p[3], p[6]); }             \
  V3 operator-() const { return V3(-p[0], -p[3], -p[6]); }
