// ORACLE — TEST INFRASTRUCTURE ONLY.
// Appended to a copy of ../refshim/Eigen/Geometry that sweepview.mk generates under _ref/sweepinc/ for the two sweep-view
// checkers: the fixed-size vector gains UnitY(), UnitZ() and a constructor from a pointer (REFSHIM_SWEEP_VECTOR_EXTRA,
// inserted by sed; the layout is unchanged, so the objects built against ../refshim link with these), and this file adds
// what GenerateEquirect.cpp's centerRig and source/rig/RigTransform.h use:
// Quaternion, AngleAxis * AngleAxis, UniformScaling, Translation, Transform<double, 3, Affine> (Affine3d), and the
// inner product v1.transpose() * v2.  These are restatements, not pinned to a real Eigen build (DESIGN.md §2):
//   - AngleAxis -> Quaternion: (axis * sin(angle / 2), cos(angle / 2)) (Quaternion.h, operator=(AngleAxis));
//   - the quaternion product in Eigen's generic order (quat_product, not its SSE path), left to right;
//   - Quaternion::toRotationMatrix as Eigen writes it (tx = 2x, twx = tx * w, ..., 1 - (tyy + tzz));
//   - UniformScaling * Translation = [s I | s t]; Transform * Transform = [L1 L2 | L1 t2 + t1] and
//     Transform * v = L v + t, every 3-term sum left to right like ../../refshim/Eigen/Geometry.
#pragma once

namespace Eigen {

enum TransformTraits { Isometry = 1, Affine = 2, AffineCompact = 18, Projective = 3 };

inline double operator*(const Matrix<double, 3, 1>::Transposed& a, const Matrix<double, 3, 1>& b) {
  return a.m->dot(b);
}

template <class S>
class Quaternion {
 public:
  S x, y, z, w;
  Quaternion(S w_, S x_, S y_, S z_) : x(x_), y(y_), z(z_), w(w_) {}
  Quaternion(const AngleAxis<S>& aa) {
    const S ha = S(0.5) * aa.angle();
    const S s = std::sin(ha);
    x = aa.axis().x() * s;
    y = aa.axis().y() * s;
    z = aa.axis().z() * s;
    w = std::cos(ha);
  }
  Quaternion operator*(const Quaternion& b) const {
    const Quaternion& a = *this;
    return Quaternion(a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
                      a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x);
  }
  Quaternion operator*(const AngleAxis<S>& b) const { return *this * Quaternion(b); }
  Matrix<S, 3, 3> toRotationMatrix() const {
    Matrix<S, 3, 3> r;
    const S tx = S(2) * x, ty = S(2) * y, tz = S(2) * z;
    const S twx = tx * w, twy = ty * w, twz = tz * w;
    const S txx = tx * x, txy = ty * x, txz = tz * x;
    const S tyy = ty * y, tyz = tz * y, tzz = tz * z;
    r(0, 0) = S(1) - (tyy + tzz);
    r(0, 1) = txy - twz;
    r(0, 2) = txz + twy;
    r(1, 0) = txy + twz;
    r(1, 1) = S(1) - (txx + tzz);
    r(1, 2) = tyz - twx;
    r(2, 0) = txz - twy;
    r(2, 1) = tyz + twx;
    r(2, 2) = S(1) - (txx + tyy);
    return r;
  }
};
template <class S>
inline Quaternion<S> operator*(const AngleAxis<S>& a, const AngleAxis<S>& b) { return Quaternion<S>(a) * Quaternion<S>(b); }

template <class S>
class UniformScaling {
 public:
  explicit UniformScaling(const S& s) : s_(s) {}
  const S& factor() const { return s_; }

 private:
  S s_;
};

template <class S, int Dim>
class Translation {
 public:
  explicit Translation(const Matrix<S, 3, 1>& t) : t_(t) {}
  const Matrix<S, 3, 1>& vector() const { return t_; }

 private:
  Matrix<S, 3, 1> t_;
};
typedef Translation<double, 3> Translation3d;

template <class S, int Dim, int Mode>
class Transform {
 public:
  Matrix<S, 3, 3> L;
  Matrix<S, 3, 1> t;
  Transform() {}
  explicit Transform(const Quaternion<S>& q) : L(q.toRotationMatrix()), t(Matrix<S, 3, 1>::Zero()) {}
  Transform operator*(const Transform& o) const {
    Transform r;
    r.L = L * o.L;
    r.t = L * o.t + t;
    return r;
  }
  Matrix<S, 3, 1> operator*(const Matrix<S, 3, 1>& v) const { return L * v + t; }
};
typedef Transform<double, 3, Affine> Affine3d;

template <class S, int Dim>
inline Transform<S, Dim, Affine> operator*(const UniformScaling<S>& s, const Translation<S, Dim>& t) {
  Transform<S, Dim, Affine> r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r.L(i, j) = i == j ? s.factor() : S(0);
  r.t = t.vector() * s.factor();
  return r;
}
template <class S, int Dim>
inline Transform<S, Dim, Affine> operator*(const Transform<S, Dim, Affine>& x, const Translation<S, Dim>& t) {
  Transform<S, Dim, Affine> r;
  r.L = x.L;
  r.t = x.L * t.vector() + x.t;
  return r;
}
template <class S, int Dim>
inline Transform<S, Dim, Affine> operator*(const Transform<S, Dim, Affine>& x, const UniformScaling<S>& s) {
  Transform<S, Dim, Affine> r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r.L(i, j) = x.L(i, j) * s.factor();
  r.t = x.t;
  return r;
}

}  // namespace Eigen
