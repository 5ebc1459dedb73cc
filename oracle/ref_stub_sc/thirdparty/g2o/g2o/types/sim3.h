// Stand-in for g2o::Sim3 (cslam/thirdparty/g2o/g2o/types/sim3.h) as the Sim3 correction shim and its literal restatement use it
// (TEST INFRASTRUCTURE).  The reference's needs Eigen, which is not available here; this one carries the members the two loop bodies
// call, written from g2o's definitions in the same operation order (plain C++, compiled with -ffp-contract=off):
//   Sim3(r, t, s) keeps r as given (no normalisation, sim3.h:64-67); inverse() sim3.h:233-236; map() sim3.h:144-146 with Eigen's
//   Quaternion * Vector3 (_transformVector); Quaternion::toRotationMatrix as Eigen writes it.
#ifndef CCM_REF_STUB_SC_G2O_SIM3_H
#define CCM_REF_STUB_SC_G2O_SIM3_H

namespace g2o {

struct Vector3d {
  double v[3] = {0., 0., 0.};
  Vector3d() {}
  Vector3d(double a, double b, double c) { v[0] = a; v[1] = b; v[2] = c; }
  double& operator[](int i) { return v[i]; }
  double operator[](int i) const { return v[i]; }
  double operator()(int i) const { return v[i]; }
};

struct Quaterniond {
  double q[4] = {0., 0., 0., 1.};   // x y z w
  Quaterniond() {}
  Quaterniond(double w, double x, double y, double z) { q[0] = x; q[1] = y; q[2] = z; q[3] = w; }
  double x() const { return q[0]; }
  double y() const { return q[1]; }
  double z() const { return q[2]; }
  double w() const { return q[3]; }
  Quaterniond conjugate() const { return Quaterniond(w(), -x(), -y(), -z()); }
  Vector3d operator*(const Vector3d& v) const {   // _transformVector: uv = 2 (q.vec x v); v + w uv + q.vec x uv
    double u0 = y() * v[2] - z() * v[1], u1 = z() * v[0] - x() * v[2], u2 = x() * v[1] - y() * v[0];
    u0 += u0; u1 += u1; u2 += u2;
    return Vector3d(v[0] + w() * u0 + (y() * u2 - z() * u1), v[1] + w() * u1 + (z() * u0 - x() * u2), v[2] + w() * u2 + (x() * u1 - y() * u0));
  }
  void toRotationMatrix(double R[3][3]) const {
    const double tx = 2 * x(), ty = 2 * y(), tz = 2 * z();
    const double twx = tx * w(), twy = ty * w(), twz = tz * w();
    const double txx = tx * x(), txy = ty * x(), txz = tz * x();
    const double tyy = ty * y(), tyz = tz * y(), tzz = tz * z();
    R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz;       R[0][2] = txz + twy;
    R[1][0] = txy + twz;       R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
    R[2][0] = txz - twy;       R[2][1] = tyz + twx;       R[2][2] = 1 - (txx + tyy);
  }
};

class Sim3 {
 public:
  Sim3() {}
  Sim3(const Quaterniond& r_, const Vector3d& t_, double s_) : r(r_), t(t_), s(s_) {}
  Vector3d map(const Vector3d& xyz) const {
    const Vector3d rx = r * xyz;
    return Vector3d(s * rx[0] + t[0], s * rx[1] + t[1], s * rx[2] + t[2]);
  }
  Sim3 inverse() const {
    const double k = -1. / s;
    return Sim3(r.conjugate(), r.conjugate() * Vector3d(k * t[0], k * t[1], k * t[2]), 1. / s);
  }
  const Quaterniond& rotation() const { return r; }
  const Vector3d& translation() const { return t; }
  double scale() const { return s; }

 protected:
  Quaterniond r;
  Vector3d t;
  double s = 1.;
};

}  // namespace g2o
#endif
