// ba_oracle.cc -- CPU oracle: a dependency-free restatement of the reference's
// joint-optimisation (bundle adjustment) path in IEEE double.
//
// TEST INFRASTRUCTURE ONLY (see ba_oracle.h). Nothing under camera_calibration_b200/
// links, loads or calls this file.
//
// Paths below are relative to /root/reference;
//   APP = applications/camera_calibration/src/camera_calibration
//   LV  = libvis/src/libvis
//
// Every function cites the reference lines it restates. The restatement follows the
// reference's ALGORITHM (order of operations, constants, failure rules, float quirks);
// it does not reproduce generated code: the B-spline un-projection Jacobians, the
// pose/rig chain rule and the tangent-frame derivatives are re-derived in closed form
// (they agree with the generated expressions to rounding).
//
// Two Jacobian modes (b200ba_options::jacobian_mode):
//   NUMERIC  : what the reference does -- d pixel / d local_point by 3 forward
//              differences and d pixel / d intrinsics by re-projecting with each
//              of the 16 control points perturbed (APP/bundle_adjustment/
//              joint_optimization.cc:357-376, APP/models/central_grid.h:187-245,
//              APP/models/noncentral_generic.h:224-283).
//   ANALYTIC : implicit-function-theorem Jacobian at the converged projection
//              (SURVEY.md section 8a row J); this is what the GPU path computes.

#include "ba_oracle.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <vector>

#include "ba_dense_fast.h"

namespace {

// ------------------------------------------------------------------------------------
// small fixed-size algebra
// ------------------------------------------------------------------------------------
struct V3 {
  double x, y, z;
};
inline V3 mk(double x, double y, double z) { return V3{x, y, z}; }
inline V3 operator+(const V3& a, const V3& b) { return mk(a.x + b.x, a.y + b.y, a.z + b.z); }
inline V3 operator-(const V3& a, const V3& b) { return mk(a.x - b.x, a.y - b.y, a.z - b.z); }
inline V3 operator*(double s, const V3& a) { return mk(s * a.x, s * a.y, s * a.z); }
inline double dot(const V3& a, const V3& b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3 cross(const V3& a, const V3& b) {
  return mk(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
inline double norm(const V3& a) { return std::sqrt(dot(a, a)); }
// Eigen's normalized(): v / sqrt(squaredNorm) when squaredNorm > 0.
inline V3 normalized(const V3& a) {
  double z = dot(a, a);
  if (z > 0) {
    double n = std::sqrt(z);
    return mk(a.x / n, a.y / n, a.z / n);
  }
  return a;
}
inline double comp(const V3& a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }

struct Quat {
  double w, x, y, z;
};
struct Pose {
  Quat q;
  V3 t;
};

// Hamilton product (Eigen::Quaternion operator*).
inline Quat qmul(const Quat& a, const Quat& b) {
  Quat r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
// Eigen::Quaternion::toRotationMatrix (valid for unit quaternions).
inline void qrot(const Quat& q, double R[3][3]) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0][0] = 1 - (tyy + tzz);
  R[0][1] = txy - twz;
  R[0][2] = txz + twy;
  R[1][0] = txy + twz;
  R[1][1] = 1 - (txx + tzz);
  R[1][2] = tyz - twx;
  R[2][0] = txz - twy;
  R[2][1] = tyz + twx;
  R[2][2] = 1 - (txx + tyy);
}
inline V3 mat3_mul(const double R[3][3], const V3& p) {
  return mk(R[0][0] * p.x + R[0][1] * p.y + R[0][2] * p.z,
            R[1][0] * p.x + R[1][1] * p.y + R[1][2] * p.z,
            R[2][0] * p.x + R[2][1] * p.y + R[2][2] * p.z);
}
// Sophus SO3 constructor from a quaternion: full normalisation
// (libvis/third_party/sophus/sophus/so3.hpp:159-167, :535-541).
inline Quat qnormalized(const Quat& q) {
  double n = std::sqrt(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
  return Quat{q.w / n, q.x / n, q.y / n, q.z / n};
}
// Sophus SE3 product a * b: rotation product followed by the first-order
// renormalisation 2 / (1 + |q|^2) (so3.hpp:215-232); translation a.t + R(a) b.t.
inline Pose pose_mul(const Pose& a, const Pose& b) {
  Pose r;
  double R[3][3];
  qrot(a.q, R);
  r.t = a.t + mat3_mul(R, b.t);
  r.q = qmul(a.q, b.q);
  double sn = r.q.w * r.q.w + r.q.x * r.q.x + r.q.y * r.q.y + r.q.z * r.q.z;
  if (sn != 1.0) {
    double s = 2.0 / (1.0 + sn);
    r.q.w *= s;
    r.q.x *= s;
    r.q.y *= s;
    r.q.z *= s;
  }
  return r;
}

// ApplyLocalUpdateToQuaternion (APP/local_parametrizations/quaternion_parametrization.h:39-60).
// NOTE the float quirk: |update| and sin|u|/|u| are stored in float, and because libvis
// pulls in namespace std (LV/libvis.h:39) sin()/cos() resolve to the float overloads.
inline Quat apply_local_update_to_quaternion(const Quat& q, double u0, double u1, double u2) {
  const float norm_update = static_cast<float>(std::sqrt(u0 * u0 + u1 * u1 + u2 * u2));
  if (norm_update == 0) return q;
  const float sin_update_by_update = std::sin(norm_update) / norm_update;
  Quat uq;
  uq.w = std::cos(norm_update);
  uq.x = sin_update_by_update * u0;
  uq.y = sin_update_by_update * u1;
  uq.z = sin_update_by_update * u2;
  return qmul(uq, q);
}

// ------------------------------------------------------------------------------------
// tangent frames (APP/local_parametrizations/line_parametrization.h:54-60)
// ------------------------------------------------------------------------------------
struct Tangents {
  V3 t1, t2;
};
inline bool tangent_uses_ey(const V3& d) { return std::fabs(d.x) > static_cast<double>(0.9f); }
inline Tangents compute_tangents(const V3& d) {
  Tangents t;
  t.t1 = normalized(tangent_uses_ey(d) ? cross(d, mk(0, 1, 0)) : cross(d, mk(1, 0, 0)));
  t.t2 = cross(d, t.t1);
  return t;
}
// d t1 / d direction and d t2 / d direction (3x3 each), direction treated as a free
// 3-vector: the quantity TangentsJacobianWrtLineDirection provides
// (line_parametrization.h:62-105); re-derived from t1 = normalize(d x e), t2 = d x t1.
inline void tangents_wrt_direction(const V3& d, double T1[3][3], double T2[3][3]) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) T1[i][j] = T2[i][j] = 0;
  if (tangent_uses_ey(d)) {
    // t1 = (-dz, 0, dx)/n, t2 = (dx dy / n, -n, dy dz / n), n = sqrt(dx^2 + dz^2)
    const double n2 = d.x * d.x + d.z * d.z;
    const double in = 1.0 / std::sqrt(n2);
    const double in3 = in * in * in;
    T1[0][0] = d.x * d.z * in3;
    T1[0][2] = -d.x * d.x * in3;
    T1[2][0] = d.z * d.z * in3;
    T1[2][2] = -d.x * d.z * in3;
    T2[0][0] = d.y * d.z * d.z * in3;
    T2[0][1] = d.x * in;
    T2[0][2] = -d.x * d.y * d.z * in3;
    T2[1][0] = -d.x * in;
    T2[1][2] = -d.z * in;
    T2[2][0] = -d.x * d.y * d.z * in3;
    T2[2][1] = d.z * in;
    T2[2][2] = d.y * d.x * d.x * in3;
  } else {
    // t1 = (0, dz, -dy)/n, t2 = (-n, dx dy / n, dx dz / n), n = sqrt(dy^2 + dz^2)
    const double n2 = d.y * d.y + d.z * d.z;
    const double in = 1.0 / std::sqrt(n2);
    const double in3 = in * in * in;
    T1[1][1] = -d.y * d.z * in3;
    T1[1][2] = d.y * d.y * in3;
    T1[2][1] = -d.z * d.z * in3;
    T1[2][2] = d.y * d.z * in3;
    T2[0][1] = -d.y * in;
    T2[0][2] = -d.z * in;
    T2[1][0] = d.y * in;
    T2[1][1] = d.x * d.z * d.z * in3;
    T2[1][2] = -d.x * d.y * d.z * in3;
    T2[2][0] = d.z * in;
    T2[2][1] = -d.x * d.y * d.z * in3;
    T2[2][2] = d.x * d.y * d.y * in3;
  }
}
// ApplyLocalUpdateToDirection (direction_parametrization.h:45-55).
inline V3 apply_local_update_to_direction(const V3& d, const Tangents& t, double o1, double o2) {
  return normalized((d + o1 * t.t1) + o2 * t.t2);
}

// ------------------------------------------------------------------------------------
// uniform cubic B-spline (APP/b_spline.h:45-104), t in [3, 4)
// ------------------------------------------------------------------------------------
inline void bspline_weights(double t, double w[4]) {
  // b_spline.h:49-61 (a = index 0 ... d = index 3)
  const double t_for_d = t - 3;
  w[3] = 1. / 6. * t_for_d * t_for_d * t_for_d;
  w[2] = -1. / 2. * t * t * t + 5 * t * t - 16 * t + 50. / 3.;
  w[1] = 1. / 2. * t * t * t - 11. / 2. * t * t + (39. / 2.) * t - 131. / 6.;
  w[0] = -1. / 6. * (t - 4) * (t - 4) * (t - 4);
}
inline void bspline_dweights(double t, double dw[4]) {
  dw[3] = 0.5 * (t - 3) * (t - 3);
  dw[2] = -1.5 * t * t + 10 * t - 16;
  dw[1] = 1.5 * t * t - 11 * t + 19.5;
  dw[0] = -0.5 * (t - 4) * (t - 4);
}
inline V3 grid_at(const double* g, int gw, int x, int y) {
  const double* p = g + 3 * (x + static_cast<int64_t>(y) * gw);
  return mk(p[0], p[1], p[2]);
}
// EvalUniformCubicBSplineSurface (b_spline.h:65-104): x-pass per row, then y-pass.
inline V3 bspline_surface(const double* g, int gw, double x, double y) {
  x += 2;
  y += 2;
  const int ix = static_cast<int>(x);
  const int iy = static_cast<int>(y);
  double wx[4], wy[4];
  bspline_weights(x - (ix - 3), wx);
  V3 rows[4];
  for (int r = 0; r < 4; ++r) {
    const int ky = iy - 3 + r;
    rows[r] = ((wx[0] * grid_at(g, gw, ix - 3, ky) + wx[1] * grid_at(g, gw, ix - 2, ky)) +
               wx[2] * grid_at(g, gw, ix - 1, ky)) +
              wx[3] * grid_at(g, gw, ix - 0, ky);
  }
  bspline_weights(y - (iy - 3), wy);
  return ((wy[0] * rows[0] + wy[1] * rows[1]) + wy[2] * rows[2]) + wy[3] * rows[3];
}
// UniformBSplineBasisFunction (b_spline.h:35-43) and
// EvalUniformCubicBSplineSurfaceGenericSlow (b_spline.h:168-186).
double bspline_basis(int i, int order, double x) {
  if (order == 0) return (x >= i && x < i + 1) ? 1 : 0;
  return (x - i) / order * bspline_basis(i, order - 1, x) +
         (i + order + 1 - x) / order * bspline_basis(i + 1, order - 1, x);
}
inline V3 bspline_surface_slow(const double* g, int gw, double x, double y) {
  x += 2;
  y += 2;
  const int ix = static_cast<int>(x);
  const int iy = static_cast<int>(y);
  V3 r = mk(0, 0, 0);
  for (int ky = iy - 3; ky <= iy; ++ky)
    for (int kx = ix - 3; kx <= ix; ++kx)
      r = r + (bspline_basis(kx, 3, x) * bspline_basis(ky, 3, y)) * grid_at(g, gw, kx, ky);
  return r;
}

// ------------------------------------------------------------------------------------
// camera models
// ------------------------------------------------------------------------------------

// Number of doubles in a camera's flat intrinsics array (same rule as the C ABI documents).
inline int64_t intr_size(const b200ba_camera* c) {
  const int64_t G = int64_t(c->grid_width) * c->grid_height;
  switch (c->model_type) {
    case B200BA_MODEL_CENTRAL_GENERIC: return 3 * G;
    case B200BA_MODEL_NONCENTRAL_GENERIC: return 6 * G;
    default: return 12;
  }
}
struct Cam {
  b200ba_camera c;
  double* p;  // flat intrinsics; mutable because the numeric Jacobian perturbs control points

  bool central() const { return c.model_type != B200BA_MODEL_NONCENTRAL_GENERIC; }
  int G() const { return c.grid_width * c.grid_height; }
  double* dir_grid() const { return p; }               // central grid / noncentral direction grid
  double* point_grid() const { return p + 3 * G(); }   // noncentral only
  // IsInCalibratedArea (APP/models/camera_model.h:149-152)
  bool in_area(double x, double y) const {
    return x >= c.calibration_min_x && y >= c.calibration_min_y &&
           x < c.calibration_max_x + 1 && y < c.calibration_max_y + 1;
  }
  // CenterOfCalibratedArea (camera_model.h:154-157): 0.5f * int -> float arithmetic.
  double center_x() const {
    return 0.5f * static_cast<float>(c.calibration_min_x + c.calibration_max_x + 1);
  }
  double center_y() const {
    return 0.5f * static_cast<float>(c.calibration_min_y + c.calibration_max_y + 1);
  }
  // PixelCornerConvToGridPoint (APP/models/central_grid.h:150-154)
  void pixel_to_grid(double x, double y, double* gx, double* gy) const {
    *gx = 1.f + (c.grid_width - 3.f) * (x - c.calibration_min_x) /
                    (c.calibration_max_x + 1 - c.calibration_min_x);
    *gy = 1.f + (c.grid_height - 3.f) * (y - c.calibration_min_y) /
                    (c.calibration_max_y + 1 - c.calibration_min_y);
  }
  // PixelScaleToGridScaleX/Y (central_grid.h:156-161): the factor is a FLOAT division.
  double scale_x() const {
    return (c.grid_width - 3.f) / (c.calibration_max_x + 1 - c.calibration_min_x);
  }
  double scale_y() const {
    return (c.grid_height - 3.f) / (c.calibration_max_y + 1 - c.calibration_min_y);
  }
  int intrinsics_jacobian_size() const {
    switch (c.model_type) {
      case B200BA_MODEL_CENTRAL_GENERIC: return 32;
      case B200BA_MODEL_NONCENTRAL_GENERIC: return 80;
      default: return 12;
    }
  }
  int update_parameter_count() const {
    switch (c.model_type) {
      case B200BA_MODEL_CENTRAL_GENERIC: return 2 * G();
      case B200BA_MODEL_NONCENTRAL_GENERIC: return 5 * G();
      default: return 12;
    }
  }
};

// ---- central-generic -----------------------------------------------------------------

// CentralGenericModel::Unproject (APP/models/central_generic.h:97-105)
bool central_unproject(const Cam& m, double x, double y, V3* dir) {
  if (!m.in_area(x, y)) return false;
  double gx, gy;
  m.pixel_to_grid(x, y, &gx, &gy);
  *dir = normalized(bspline_surface(m.dir_grid(), m.c.grid_width, gx, gy));
  return true;
}

// Shared by both generic models: position of the 4x4 support and the weights.
struct Support {
  int x0, y0;  // top-left control point
  double wx[4], wy[4], dwx[4], dwy[4];
};
inline void make_support(const Cam& m, double x, double y, Support* s) {
  double gx, gy;
  m.pixel_to_grid(x, y, &gx, &gy);
  gx += 2;
  gy += 2;
  const int ix = static_cast<int>(std::floor(gx));
  const int iy = static_cast<int>(std::floor(gy));
  s->x0 = ix - 3;
  s->y0 = iy - 3;
  const double fx = gx - (ix - 3), fy = gy - (iy - 3);
  bspline_weights(fx, s->wx);
  bspline_weights(fy, s->wy);
  bspline_dweights(fx, s->dwx);
  bspline_dweights(fy, s->dwy);
}
// value, d/dgx, d/dgy of a 3-vector spline surface on the support
inline void spline_with_derivs(const double* g, int gw, const Support& s, V3* v, V3* vx, V3* vy) {
  *v = *vx = *vy = mk(0, 0, 0);
  for (int r = 0; r < 4; ++r) {
    V3 a = mk(0, 0, 0), ax = mk(0, 0, 0);
    for (int c = 0; c < 4; ++c) {
      V3 p = grid_at(g, gw, s.x0 + c, s.y0 + r);
      a = a + s.wx[c] * p;
      ax = ax + s.dwx[c] * p;
    }
    *v = *v + s.wy[r] * a;
    *vx = *vx + s.wy[r] * ax;
    *vy = *vy + s.dwy[r] * a;
  }
}

// CentralGenericModel::UnprojectWithJacobian (APP/models/central_generic.cc:521-549) with
// CentralGenericBSpline_Unproject_ComputeResidualAndJacobian
// (APP/models/central_generic_jacobians.cc:320-448) re-derived:
//   s = sum w_ij G_ij, u = s/|s|, du/dg = (ds/dg - u (u . ds/dg)) / |s|, then the
//   grid->pixel scale factors.
bool central_unproject_jac(const Cam& m, double x, double y, V3* dir, double J[3][2],
                           Support* sup_out = nullptr, double* inv_norm_out = nullptr) {
  if (!m.in_area(x, y)) return false;
  Support s;
  make_support(m, x, y, &s);
  V3 v, vx, vy;
  spline_with_derivs(m.dir_grid(), m.c.grid_width, s, &v, &vx, &vy);
  const double inv_n = 1.0 / std::sqrt(dot(v, v));
  const V3 u = inv_n * v;
  const V3 ux = inv_n * (vx - dot(u, vx) * u);
  const V3 uy = inv_n * (vy - dot(u, vy) * u);
  const double sx = m.scale_x(), sy = m.scale_y();
  *dir = u;
  J[0][0] = sx * ux.x;
  J[1][0] = sx * ux.y;
  J[2][0] = sx * ux.z;
  J[0][1] = sy * uy.x;
  J[1][1] = sy * uy.y;
  J[2][1] = sy * uy.z;
  if (sup_out) *sup_out = s;
  if (inv_norm_out) *inv_norm_out = inv_n;
  return true;
}

// The 2-parameter LM shared by both generic models' projection
// (central: APP/models/central_generic.cc:433-519, noncentral: noncentral_generic.cc:156-264):
// eps = 1e-12 on the squared residual, <= 100 outer iterations, lambda0 = 0.01 * 0.5 * tr(H)
// at the first iteration only, <= 10 attempts x2 / x0.5, trial clamped to
// [min, max + 0.999], returns true as soon as the cost measured BEFORE the step is < eps.
template <class EvalJ, class EvalCost>
bool projection_lm(const Cam& m, double* px, double* py, EvalJ eval_with_jacobian,
                   EvalCost eval_cost) {
  constexpr double kEpsilon = 1e-12;
  const int kMaxIterations = 100;
  double lambda = -1;
  for (int i = 0; i < kMaxIterations; ++i) {
    double cost, H00, H01, H11, b0, b1;
    if (!eval_with_jacobian(*px, *py, &cost, &H00, &H01, &H11, &b0, &b1)) {
      // The reference CHECK()-aborts here; callers guarantee an in-area start.
      return false;
    }
    if (lambda < 0) {
      constexpr double kInitialLambdaFactor = 0.01;
      lambda = kInitialLambdaFactor * 0.5 * (H00 + H11);
    }
    bool update_accepted = false;
    for (int lm_iteration = 0; lm_iteration < 10; ++lm_iteration) {
      const double H00_LM = H00 + lambda;
      const double H11_LM = H11 + lambda;
      const double x_1 = (b1 - H01 / H00_LM * b0) / (H11_LM - H01 * H01 / H00_LM);
      const double x_0 = (b0 - H01 * x_1) / H00_LM;
      const double tx = std::max<double>(m.c.calibration_min_x,
                                         std::min(m.c.calibration_max_x + 0.999, *px - x_0));
      const double ty = std::max<double>(m.c.calibration_min_y,
                                         std::min(m.c.calibration_max_y + 0.999, *py - x_1));
      double test_cost = std::numeric_limits<double>::infinity();
      eval_cost(tx, ty, &test_cost);
      if (test_cost < cost) {
        lambda *= 0.5;
        *px = tx;
        *py = ty;
        update_accepted = true;
        break;
      } else {
        lambda *= 2;
      }
    }
    if (!update_accepted) return cost < kEpsilon;
    if (cost < kEpsilon) return true;
  }
  return false;
}

// CentralGenericModel::ProjectDirectionWithInitialEstimate (central_generic.cc:433-519)
bool central_project_direction(const Cam& m, const V3& d, double* px, double* py) {
  auto evalJ = [&](double x, double y, double* cost, double* H00, double* H01, double* H11,
                   double* b0, double* b1) {
    V3 u;
    double J[3][2];
    if (!central_unproject_jac(m, x, y, &u, J)) return false;
    const double dx = u.x - d.x, dy = u.y - d.y, dz = u.z - d.z;
    *cost = dx * dx + dy * dy + dz * dz;
    *H00 = J[0][0] * J[0][0] + J[1][0] * J[1][0] + J[2][0] * J[2][0];
    *H01 = J[0][0] * J[0][1] + J[1][0] * J[1][1] + J[2][0] * J[2][1];
    *H11 = J[0][1] * J[0][1] + J[1][1] * J[1][1] + J[2][1] * J[2][1];
    *b0 = dx * J[0][0] + dy * J[1][0] + dz * J[2][0];
    *b1 = dx * J[0][1] + dy * J[1][1] + dz * J[2][1];
    return true;
  };
  auto evalC = [&](double x, double y, double* cost) {
    V3 u;
    if (central_unproject(m, x, y, &u)) {
      const double dx = u.x - d.x, dy = u.y - d.y, dz = u.z - d.z;
      *cost = dx * dx + dy * dy + dz * dz;
    }
  };
  return projection_lm(m, px, py, evalJ, evalC);
}

// ---- noncentral-generic ----------------------------------------------------------------

// NoncentralGenericModel::Unproject (APP/models/noncentral_generic.h:100-118): both grids are
// interpolated with the same weights (EvalTwoUniformCubicBSplineSurfaces, b_spline.h:106-166);
// the direction is normalised, the origin is not.
bool noncentral_unproject(const Cam& m, double x, double y, V3* origin, V3* dir) {
  if (!m.in_area(x, y)) return false;
  double gx, gy;
  m.pixel_to_grid(x, y, &gx, &gy);
  *dir = normalized(bspline_surface(m.dir_grid(), m.c.grid_width, gx, gy));
  *origin = bspline_surface(m.point_grid(), m.c.grid_width, gx, gy);
  return true;
}
// NoncentralGenericModel::UnprojectWithJacobian (noncentral_generic.cc:266-293; generated
// noncentral_generic_jacobians.cc:31-206 re-derived). J rows 0-2: direction, rows 3-5: origin.
bool noncentral_unproject_jac(const Cam& m, double x, double y, V3* origin, V3* dir,
                              double J[6][2], Support* sup_out = nullptr,
                              double* inv_norm_out = nullptr) {
  if (!m.in_area(x, y)) return false;
  Support s;
  make_support(m, x, y, &s);
  V3 v, vx, vy, o, ox, oy;
  spline_with_derivs(m.dir_grid(), m.c.grid_width, s, &v, &vx, &vy);
  spline_with_derivs(m.point_grid(), m.c.grid_width, s, &o, &ox, &oy);
  const double inv_n = 1.0 / std::sqrt(dot(v, v));
  const V3 u = inv_n * v;
  const V3 ux = inv_n * (vx - dot(u, vx) * u);
  const V3 uy = inv_n * (vy - dot(u, vy) * u);
  const double sx = m.scale_x(), sy = m.scale_y();
  *dir = u;
  *origin = o;
  for (int i = 0; i < 3; ++i) {
    J[i][0] = sx * comp(ux, i);
    J[i][1] = sy * comp(uy, i);
    J[3 + i][0] = sx * comp(ox, i);
    J[3 + i][1] = sy * comp(oy, i);
  }
  if (sup_out) *sup_out = s;
  if (inv_norm_out) *inv_norm_out = inv_n;
  return true;
}
// Residual of the noncentral projection and its 2x2 Jacobian wrt. the pixel
// (noncentral_generic.cc:166-193): r = (t1 . (o - p), t2 . (o - p)).
inline void noncentral_residual_jac(const V3& o, const V3& d, const double J[6][2], const V3& p,
                                    double r[2], double Rxy[2][2], Tangents* tan_out = nullptr) {
  Tangents t = compute_tangents(d);
  const V3 pto = o - p;
  r[0] = dot(t.t1, pto);
  r[1] = dot(t.t2, pto);
  double T1[3][3], T2[3][3];
  tangents_wrt_direction(d, T1, T2);
  for (int c = 0; c < 2; ++c) {
    const V3 dd = mk(J[0][c], J[1][c], J[2][c]);
    const V3 dor = mk(J[3][c], J[4][c], J[5][c]);
    const V3 dt1 = mk(T1[0][0] * dd.x + T1[0][1] * dd.y + T1[0][2] * dd.z,
                      T1[1][0] * dd.x + T1[1][1] * dd.y + T1[1][2] * dd.z,
                      T1[2][0] * dd.x + T1[2][1] * dd.y + T1[2][2] * dd.z);
    const V3 dt2 = mk(T2[0][0] * dd.x + T2[0][1] * dd.y + T2[0][2] * dd.z,
                      T2[1][0] * dd.x + T2[1][1] * dd.y + T2[1][2] * dd.z,
                      T2[2][0] * dd.x + T2[2][1] * dd.y + T2[2][2] * dd.z);
    Rxy[0][c] = dot(pto, dt1) + dot(t.t1, dor);
    Rxy[1][c] = dot(pto, dt2) + dot(t.t2, dor);
  }
  if (tan_out) *tan_out = t;
}
// NoncentralGenericModel::ProjectWithInitialEstimate (noncentral_generic.cc:156-264)
bool noncentral_project(const Cam& m, const V3& p, double* px, double* py) {
  auto evalJ = [&](double x, double y, double* cost, double* H00, double* H01, double* H11,
                   double* b0, double* b1) {
    V3 o, d;
    double J[6][2];
    if (!noncentral_unproject_jac(m, x, y, &o, &d, J)) return false;
    double r[2], R[2][2];
    noncentral_residual_jac(o, d, J, p, r, R);
    *cost = r[0] * r[0] + r[1] * r[1];
    *H00 = R[0][0] * R[0][0] + R[1][0] * R[1][0];
    *H01 = R[0][0] * R[0][1] + R[1][0] * R[1][1];
    *H11 = R[0][1] * R[0][1] + R[1][1] * R[1][1];
    *b0 = r[0] * R[0][0] + r[1] * R[1][0];
    *b1 = r[0] * R[0][1] + r[1] * R[1][1];
    return true;
  };
  auto evalC = [&](double x, double y, double* cost) {
    V3 o, d;
    if (noncentral_unproject(m, x, y, &o, &d)) {
      Tangents t = compute_tangents(d);
      const V3 pto = o - p;
      const double d1 = dot(t.t1, pto), d2 = dot(t.t2, pto);
      *cost = d1 * d1 + d2 * d2;
    }
  };
  return projection_lm(m, px, py, evalJ, evalC);
}

// ---- central OpenCV (12 parameters) -------------------------------------------------------

// CentralOpenCVModel::Project (APP/models/central_opencv.cc:59-99)
bool opencv_project(const Cam& m, const V3& lp, double* px, double* py) {
  if (lp.z <= 0) return false;
  const double nx = lp.x / lp.z, ny = lp.y / lp.z;
  const double x2 = nx * nx, xy = nx * ny, y2 = ny * ny;
  const double r2 = x2 + y2, r4 = r2 * r2, r6 = r4 * r2;
  const double* q = m.p;
  const double fx = q[0], fy = q[1], cx = q[2], cy = q[3];
  const double k1 = q[4], k2 = q[5], k3 = q[6], k4 = q[7], k5 = q[8], k6 = q[9], p1 = q[10],
               p2 = q[11];
  const double radial = (1 + k1 * r2 + k2 * r4 + k3 * r6) / (1 + k4 * r2 + k5 * r4 + k6 * r6);
  const double dx = 2.0 * p1 * xy + p2 * (r2 + 2.0 * x2);
  const double dy = 2.0 * p2 * xy + p1 * (r2 + 2.0 * y2);
  *px = fx * (nx * radial + dx) + cx;
  *py = fy * (ny * radial + dy) + cy;
  return *px >= 0 && *py >= 0 && *px < m.c.width && *py < m.c.height;
}
// CentralOpenCVModel::ProjectionJacobianWrtIntrinsics (central_opencv.h:98-176), restated
// from the projection formula: columns fx fy cx cy k1 k2 k3 k4 k5 k6 p1 p2.
void opencv_intrinsics_jacobian(const Cam& m, const V3& lp, double Jx[12], double Jy[12]) {
  const double nx = lp.x / lp.z, ny = lp.y / lp.z;
  const double x2 = nx * nx, xy = nx * ny, y2 = ny * ny;
  const double r2 = x2 + y2, r4 = r2 * r2, r6 = r4 * r2;
  const double* q = m.p;
  const double fx = q[0], fy = q[1];
  const double k1 = q[4], k2 = q[5], k3 = q[6], k4 = q[7], k5 = q[8], k6 = q[9], p1 = q[10],
               p2 = q[11];
  const double num = 1 + k1 * r2 + k2 * r4 + k3 * r6;
  const double den = 1 + k4 * r2 + k5 * r4 + k6 * r6;
  const double iden = 1.0 / den;
  const double radial = num * iden;
  Jx[0] = nx * radial + 2 * p1 * xy + p2 * (r2 + 2 * x2);
  Jx[1] = 0;
  Jx[2] = 1;
  Jx[3] = 0;
  Jx[4] = fx * nx * r2 * iden;
  Jx[5] = fx * nx * r4 * iden;
  Jx[6] = fx * nx * r6 * iden;
  Jx[7] = -fx * nx * num * iden * iden * r2;
  Jx[8] = -fx * nx * num * iden * iden * r4;
  Jx[9] = -fx * nx * num * iden * iden * r6;
  Jx[10] = fx * 2 * xy;
  Jx[11] = fx * (r2 + 2 * x2);
  Jy[0] = 0;
  Jy[1] = ny * radial + p1 * (r2 + 2 * y2) + 2 * p2 * xy;
  Jy[2] = 0;
  Jy[3] = 1;
  Jy[4] = fy * ny * r2 * iden;
  Jy[5] = fy * ny * r4 * iden;
  Jy[6] = fy * ny * r6 * iden;
  Jy[7] = -fy * ny * num * iden * iden * r2;
  Jy[8] = -fy * ny * num * iden * iden * r4;
  Jy[9] = -fy * ny * num * iden * iden * r6;
  Jy[10] = fy * (r2 + 2 * y2);
  Jy[11] = fy * 2 * xy;
}
// d pixel / d local_point in closed form (ANALYTIC mode only).
void opencv_point_jacobian(const Cam& m, const V3& lp, double P[2][3]) {
  const double iz = 1.0 / lp.z;
  const double nx = lp.x * iz, ny = lp.y * iz;
  const double x2 = nx * nx, xy = nx * ny, y2 = ny * ny;
  const double r2 = x2 + y2, r4 = r2 * r2, r6 = r4 * r2;
  const double* q = m.p;
  const double fx = q[0], fy = q[1];
  const double k1 = q[4], k2 = q[5], k3 = q[6], k4 = q[7], k5 = q[8], k6 = q[9], p1 = q[10],
               p2 = q[11];
  const double num = 1 + k1 * r2 + k2 * r4 + k3 * r6;
  const double den = 1 + k4 * r2 + k5 * r4 + k6 * r6;
  const double radial = num / den;
  const double dnum = k1 + 2 * k2 * r2 + 3 * k3 * r4;
  const double dden = k4 + 2 * k5 * r2 + 3 * k6 * r4;
  const double drad = (dnum * den - num * dden) / (den * den);  // d radial / d r2
  const double dxx = radial + 2 * x2 * drad + 2 * p1 * ny + 6 * p2 * nx;
  const double dxy = 2 * xy * drad + 2 * p1 * nx + 2 * p2 * ny;
  const double dyx = 2 * xy * drad + 2 * p2 * ny + 2 * p1 * nx;
  const double dyy = radial + 2 * y2 * drad + 2 * p2 * nx + 6 * p1 * ny;
  // d(nx, ny)/d(X, Y, Z) = [iz 0 -nx iz; 0 iz -ny iz]
  P[0][0] = fx * dxx * iz;
  P[0][1] = fx * dxy * iz;
  P[0][2] = fx * (-dxx * nx - dxy * ny) * iz;
  P[1][0] = fy * dyx * iz;
  P[1][1] = fy * dyy * iz;
  P[1][2] = fy * (-dyx * nx - dyy * ny) * iz;
}

// ---- model dispatch (IDENTIFY_CAMERA_MODEL, APP/models/all_models.h:46-81) ------------------
// CameraModel::ProjectWithInitialEstimate
bool project_with_initial_estimate(const Cam& m, const V3& lp, double* px, double* py) {
  switch (m.c.model_type) {
    case B200BA_MODEL_CENTRAL_GENERIC:
      return central_project_direction(m, normalized(lp), px, py);  // central_grid.h:86-88
    case B200BA_MODEL_NONCENTRAL_GENERIC:
      return noncentral_project(m, lp, px, py);
    case B200BA_MODEL_CENTRAL_OPENCV:
      return opencv_project(m, lp, px, py);  // central_opencv.h:61-67: estimate ignored
    default:
      return false;
  }
}

// ------------------------------------------------------------------------------------
// Huber loss (LV/loss_functions.h:94-133)
// ------------------------------------------------------------------------------------
inline double huber_cost_sq(double h, double sq) {
  if (sq < h * h) return 0.5 * sq;
  return h * (std::sqrt(sq) - 0.5 * h);
}
inline double huber_weight_sq(double h, double sq) { return (sq < h * h) ? 1 : (h / std::sqrt(sq)); }

// ------------------------------------------------------------------------------------
// problem / state views
// ------------------------------------------------------------------------------------
struct Layout {
  // JointOptimizationState offsets (APP/bundle_adjustment/joint_optimization.cc:97-170)
  int n_points, n_imagesets, n_cameras;
  bool localize_only, eliminate_points, rig_in_state;
  int first_rig_tr_global, first_camera_tr_rig, first_points, first_intrinsics;
  std::vector<int> intrinsics_offset;
  int dof;
  int block_size, num_blocks;  // Schur block structure (joint_optimization.cc:794-804)
  int block_dof() const { return block_size * num_blocks; }
  int dense_dof() const { return dof - block_dof(); }
};

Layout make_layout(const b200ba_problem& pb, const b200ba_options& opt) {
  Layout L;
  L.n_points = pb.n_points;
  L.n_imagesets = pb.n_imagesets;
  L.n_cameras = pb.n_cameras;
  L.localize_only = opt.localize_only != 0;
  L.eliminate_points = opt.eliminate_points != 0;
  L.rig_in_state = pb.n_cameras > 1;
  const int rig_dof = L.rig_in_state ? 6 * pb.n_cameras : 0;
  L.first_rig_tr_global = L.eliminate_points ? 3 * pb.n_points : 0;
  L.first_camera_tr_rig = L.first_rig_tr_global + 6 * pb.n_imagesets;
  L.first_points = L.eliminate_points ? 0 : (L.first_camera_tr_rig + rig_dof);
  L.first_intrinsics =
      L.eliminate_points ? (L.first_camera_tr_rig + rig_dof) : (L.first_points + 3 * pb.n_points);
  int off = L.first_intrinsics;
  int n_intr = 0;
  L.intrinsics_offset.resize(pb.n_cameras);
  for (int c = 0; c < pb.n_cameras; ++c) {
    L.intrinsics_offset[c] = off;
    Cam m{pb.cameras[c], nullptr};
    off += m.update_parameter_count();
    n_intr += m.update_parameter_count();
  }
  L.dof = rig_dof + 6 * pb.n_imagesets + (L.localize_only ? 0 : n_intr) + 3 * pb.n_points;
  if (L.eliminate_points) {
    L.block_size = 3;
    L.num_blocks = pb.n_points;
  } else {
    L.block_size = 6;
    L.num_blocks = pb.n_imagesets;
  }
  return L;
}

inline Pose load_pose(const double* p) { return Pose{Quat{p[0], p[1], p[2], p[3]}, mk(p[4], p[5], p[6])}; }
inline void store_pose(const Pose& P, double* p) {
  p[0] = P.q.w;
  p[1] = P.q.x;
  p[2] = P.q.y;
  p[3] = P.q.z;
  p[4] = P.t.x;
  p[5] = P.t.y;
  p[6] = P.t.z;
}

// A deep copy of the mutable state (the reference copies the whole state per LM attempt
// because it is not reversible, LV/lm_optimizer.h:917-919).
struct State {
  std::vector<double> points, rig_tr_global, camera_tr_rig;
  std::vector<std::vector<double>> intrinsics;
};
State load_state(const b200ba_problem& pb, const b200ba_state& s) {
  State S;
  S.points.assign(s.points, s.points + 3 * pb.n_points);
  S.rig_tr_global.assign(s.rig_tr_global, s.rig_tr_global + 7 * pb.n_imagesets);
  S.camera_tr_rig.assign(s.camera_tr_rig, s.camera_tr_rig + 7 * pb.n_cameras);
  S.intrinsics.resize(pb.n_cameras);
  for (int c = 0; c < pb.n_cameras; ++c) {
    int64_t n = intr_size(&pb.cameras[c]);
    S.intrinsics[c].assign(s.intrinsics[c], s.intrinsics[c] + n);
  }
  return S;
}
void store_state(const b200ba_problem& pb, const State& S, b200ba_state* s) {
  std::copy(S.points.begin(), S.points.end(), s->points);
  std::copy(S.rig_tr_global.begin(), S.rig_tr_global.end(), s->rig_tr_global);
  std::copy(S.camera_tr_rig.begin(), S.camera_tr_rig.end(), s->camera_tr_rig);
  for (int c = 0; c < pb.n_cameras; ++c)
    std::copy(S.intrinsics[c].begin(), S.intrinsics[c].end(), s->intrinsics[c]);
}

// JointOptimizationState::operator-= (joint_optimization.cc:172-214) with the models'
// SubtractDelta (central_grid.h:168-184, noncentral_generic.h:195-219, central_opencv.h:91-94).
void apply_update(const b200ba_problem& pb, const Layout& L, State* S, const double* delta) {
  int di = L.first_rig_tr_global;
  for (int i = 0; i < pb.n_imagesets; ++i, di += 6) {
    Pose P = load_pose(&S->rig_tr_global[7 * i]);
    // SE3d(quaternion, t) normalises the quaternion (sophus se3.hpp:546 -> so3.hpp:535-541).
    P.q = qnormalized(apply_local_update_to_quaternion(P.q, -delta[di], -delta[di + 1], -delta[di + 2]));
    P.t = P.t - mk(delta[di + 3], delta[di + 4], delta[di + 5]);
    store_pose(P, &S->rig_tr_global[7 * i]);
  }
  if (L.rig_in_state) {
    di = L.first_camera_tr_rig;
    for (int c = 0; c < pb.n_cameras; ++c, di += 6) {
      Pose P = load_pose(&S->camera_tr_rig[7 * c]);
      P.q = qnormalized(apply_local_update_to_quaternion(P.q, -delta[di], -delta[di + 1], -delta[di + 2]));
      P.t = P.t - mk(delta[di + 3], delta[di + 4], delta[di + 5]);
      store_pose(P, &S->camera_tr_rig[7 * c]);
    }
  }
  di = L.first_points;
  for (int i = 0; i < 3 * pb.n_points; ++i) S->points[i] -= delta[di + i];
  if (!L.localize_only) {
    for (int c = 0; c < pb.n_cameras; ++c) {
      Cam m{pb.cameras[c], S->intrinsics[c].data()};
      const double* d = delta + L.intrinsics_offset[c];
      const int G = m.G();
      if (m.c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
        for (int k = 0; k < G; ++k) {
          V3 dir = mk(m.p[3 * k], m.p[3 * k + 1], m.p[3 * k + 2]);
          Tangents t = compute_tangents(dir);
          dir = apply_local_update_to_direction(dir, t, -d[2 * k], -d[2 * k + 1]);
          m.p[3 * k] = dir.x;
          m.p[3 * k + 1] = dir.y;
          m.p[3 * k + 2] = dir.z;
        }
      } else if (m.c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
        double* dg = m.dir_grid();
        double* pg = m.point_grid();
        for (int k = 0; k < G; ++k) {
          V3 dir = mk(dg[3 * k], dg[3 * k + 1], dg[3 * k + 2]);
          V3 org = mk(pg[3 * k], pg[3 * k + 1], pg[3 * k + 2]);
          Tangents t = compute_tangents(dir);
          // ApplyLocalUpdateToLine (line_parametrization.h:107-120): the origin moves along
          // t1, t2 and the OLD direction; then the direction is updated.
          org = ((org + (-d[5 * k + 2]) * t.t1) + (-d[5 * k + 3]) * t.t2) + (-d[5 * k + 4]) * dir;
          dir = apply_local_update_to_direction(dir, t, -d[5 * k], -d[5 * k + 1]);
          dg[3 * k] = dir.x;
          dg[3 * k + 1] = dir.y;
          dg[3 * k + 2] = dir.z;
          pg[3 * k] = org.x;
          pg[3 * k + 1] = org.y;
          pg[3 * k + 2] = org.z;
        }
      } else {
        for (int k = 0; k < 12; ++k) m.p[k] -= d[k];
      }
    }
  }
}

// ------------------------------------------------------------------------------------
// H / b accumulation (LV/lm_optimizer_update_accumulator.h:108-555,
// LV/lm_optimizer_jtj_accumulator_base.h:175-412)
// ------------------------------------------------------------------------------------
struct Accumulator {
  // Storage split exactly like the reference (LV/lm_optimizer.h:657-685): block-diagonal
  // part, off-diagonal part (block rows x dense cols), dense part; only row <= col is written.
  int bs = 0, nb = 0, nd = 0;
  bool want_matrices = false;
  double* block_diag = nullptr;  // nb * bs * bs
  double* off_diag = nullptr;    // (nb*bs) * nd
  double* dense = nullptr;       // nd * nd
  std::vector<double> b_block, b_dense;
  std::vector<double>* cost_vector = nullptr;
  double cost = 0;
  double huber = 1.0;

  // optional per-observation outputs (oracle_evaluate)
  double* out_residuals = nullptr;
  double *out_jpoint = nullptr, *out_jpose = nullptr, *out_jrig = nullptr, *out_jintr = nullptr;
  int32_t* out_intr_index = nullptr;
  int32_t out_K = 0;
  int32_t* out_has_jacobian = nullptr;

  // record mode (threaded evaluation, compute_mt): the add_* calls of ONE observation are captured
  // instead of applied, and replayed later in the reference's sequential order
  struct Record {
    int kind = 0;  // 0 invalid, 1 residual only, 2 residual with Jacobian
    double rx = 0, ry = 0;
    int n = 0;
    int idx[3 + 6 + 6 + 80];
    double jx[3 + 6 + 6 + 80], jy[3 + 6 + 6 + 80];
  };
  Record* rec = nullptr;

  ~Accumulator() {
    free(block_diag);
    free(off_diag);
    free(dense);
  }
  void allocate(int block_size, int num_blocks, int n_dense) {
    bs = block_size;
    nb = num_blocks;
    nd = n_dense;
    want_matrices = true;
    // calloc: pages are committed on first touch only (matters for the bounded-sample timing).
    block_diag = static_cast<double*>(calloc(std::max<size_t>(1, size_t(nb) * bs * bs), sizeof(double)));
    off_diag = static_cast<double*>(calloc(std::max<size_t>(1, size_t(nb) * bs * nd), sizeof(double)));
    dense = static_cast<double*>(calloc(std::max<size_t>(1, size_t(nd) * nd), sizeof(double)));
    b_block.assign(size_t(nb) * bs, 0.0);
    b_dense.assign(nd, 0.0);
  }
  inline void addH(int i, int k, double v) {  // requires i <= k
    const int nbd = bs * nb;
    if (k < nbd) {
      const int blk = i / bs;
      block_diag[(size_t(blk) * bs + (i - blk * bs)) * bs + (k - blk * bs)] += v;
    } else if (i < nbd) {
      off_diag[size_t(i) * nd + (k - nbd)] += v;
    } else {
      dense[size_t(i - nbd) * nd + (k - nbd)] += v;
    }
  }
  inline void addB(int i, double v) {
    const int nbd = bs * nb;
    if (i < nbd)
      b_block[i] += v;
    else
      b_dense[i - nbd] += v;
  }
  void add_invalid() {
    if (rec) {
      rec->kind = 0;
      return;
    }
    if (cost_vector) cost_vector->push_back(-1);
  }
  void add_residual(double rx, double ry) {
    if (rec) {
      rec->kind = 1;
      rec->rx = rx;
      rec->ry = ry;
      return;
    }
    const double c = huber_cost_sq(huber, rx * rx + ry * ry);
    cost += c;
    if (cost_vector) cost_vector->push_back(c);
  }
  // AddResidualWithJacobian: cols sorted by ascending global index; H(i,k) += w (J_i . J_k),
  // b(i) += w (J_i . r).
  void add_residual_with_jacobian(double rx, double ry, int n, const int* idx, const double* jx,
                                  const double* jy) {
    if (rec) {
      rec->kind = 2;
      rec->rx = rx;
      rec->ry = ry;
      rec->n = n;
      std::copy(idx, idx + n, rec->idx);
      std::copy(jx, jx + n, rec->jx);
      std::copy(jy, jy + n, rec->jy);
      return;
    }
    add_residual(rx, ry);
    if (!want_matrices) return;
    const double w = huber_weight_sq(huber, rx * rx + ry * ry);
    for (int i = 0; i < n; ++i) {
      const double wjx = w * jx[i], wjy = w * jy[i];
      for (int k = i; k < n; ++k) addH(idx[i], idx[k], wjx * jx[k] + wjy * jy[k]);
      addB(idx[i], rx * wjx + ry * wjy);
    }
  }
  void replay(const Record& r) {
    if (r.kind == 0)
      add_invalid();
    else if (r.kind == 1)
      add_residual(r.rx, r.ry);
    else
      add_residual_with_jacobian(r.rx, r.ry, r.n, r.idx, r.jx, r.jy);
  }
};

// ------------------------------------------------------------------------------------
// the cost function (APP/bundle_adjustment/joint_optimization.cc:227-593)
// ------------------------------------------------------------------------------------
struct CostFunction {
  const b200ba_problem* pb;
  Layout L;
  double numerical_diff_delta;
  int jacobian_mode;
  double* last_projection;  // [2*n_obs], mutated like PointFeature::last_projection
  int64_t obs_begin = 0, obs_end = -1;  // restriction used by the bounded-sample timing

  // d pixel / d intrinsics by finite differences
  // central: central_grid.h:187-245; noncentral: noncentral_generic.h:224-283.
  bool numeric_intrinsics_jacobian(const Cam& m, const std::vector<Tangents>& tangents,
                                   const V3& lp, double px, double py, int* idx, double* jx,
                                   double* jy) const {
    double gx, gy;
    m.pixel_to_grid(px, py, &gx, &gy);
    const int ix = static_cast<int>(std::floor(gx));
    const int iy = static_cast<int>(std::floor(gy));
    const int gw = m.c.grid_width;
    const double delta = numerical_diff_delta;
    int li = 0;
    if (m.c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
      const V3 pd = normalized(lp);
      for (int y = 0; y < 4; ++y) {
        const int gyy = iy + y - 1;
        for (int x = 0; x < 4; ++x) {
          const int gxx = ix + x - 1;
          const int seq = gxx + gyy * gw;
          idx[li] = 2 * seq;
          idx[li + 1] = 2 * seq + 1;
          double* cp = m.dir_grid() + 3 * seq;
          const V3 orig = mk(cp[0], cp[1], cp[2]);
          for (int d = 0; d < 2; ++d) {
            V3 test = apply_local_update_to_direction(orig, tangents[seq], d == 0 ? delta : 0,
                                                      d == 1 ? delta : 0);
            cp[0] = test.x;
            cp[1] = test.y;
            cp[2] = test.z;
            double tx = px, ty = py;
            bool ok = central_project_direction(m, pd, &tx, &ty);
            cp[0] = orig.x;
            cp[1] = orig.y;
            cp[2] = orig.z;
            if (!ok) return false;
            jx[li + d] = (tx - px) / delta;
            jy[li + d] = (ty - py) / delta;
          }
          li += 2;
        }
      }
    } else {
      for (int y = 0; y < 4; ++y) {
        const int gyy = iy + y - 1;
        for (int x = 0; x < 4; ++x) {
          const int gxx = ix + x - 1;
          const int seq = gxx + gyy * gw;
          for (int i = 0; i < 5; ++i) idx[li + i] = 5 * seq + i;
          double* cd = m.dir_grid() + 3 * seq;
          double* co = m.point_grid() + 3 * seq;
          const V3 od = mk(cd[0], cd[1], cd[2]);
          const V3 oo = mk(co[0], co[1], co[2]);
          const Tangents& t = tangents[seq];
          for (int d = 0; d < 5; ++d) {
            double dl[5] = {0, 0, 0, 0, 0};
            dl[d] = delta;
            // ApplyLocalUpdateToLine (line_parametrization.h:107-120)
            V3 to = ((oo + dl[2] * t.t1) + dl[3] * t.t2) + dl[4] * od;
            V3 td = apply_local_update_to_direction(od, t, dl[0], dl[1]);
            co[0] = to.x; co[1] = to.y; co[2] = to.z;
            cd[0] = td.x; cd[1] = td.y; cd[2] = td.z;
            double tx = px, ty = py;
            bool ok = noncentral_project(m, lp, &tx, &ty);
            co[0] = oo.x; co[1] = oo.y; co[2] = oo.z;
            cd[0] = od.x; cd[1] = od.y; cd[2] = od.z;
            if (!ok) return false;
            jx[li + d] = (tx - px) / delta;
            jy[li + d] = (ty - py) / delta;
          }
          li += 5;
        }
      }
    }
    return true;
  }

  // ANALYTIC mode: d pixel / d local_point (2x3) and d pixel / d intrinsics by the implicit
  // function theorem at the converged projection (SURVEY.md 8a row J).
  bool analytic_jacobians(const Cam& m, const std::vector<Tangents>& tangents, const V3& lp,
                          double px, double py, double P[2][3], int* idx, double* jx,
                          double* jy, bool want_intrinsics) const {
    const int gw = m.c.grid_width;
    if (m.c.model_type == B200BA_MODEL_CENTRAL_GENERIC) {
      V3 u;
      double A[3][2];
      Support s;
      double inv_n;
      if (!central_unproject_jac(m, px, py, &u, A, &s, &inv_n)) return false;
      // M = (A^T A)^-1 A^T  (2x3)
      const double a00 = A[0][0] * A[0][0] + A[1][0] * A[1][0] + A[2][0] * A[2][0];
      const double a01 = A[0][0] * A[0][1] + A[1][0] * A[1][1] + A[2][0] * A[2][1];
      const double a11 = A[0][1] * A[0][1] + A[1][1] * A[1][1] + A[2][1] * A[2][1];
      const double idet = 1.0 / (a00 * a11 - a01 * a01);
      double M[2][3];
      for (int j = 0; j < 3; ++j) {
        M[0][j] = idet * (a11 * A[j][0] - a01 * A[j][1]);
        M[1][j] = idet * (-a01 * A[j][0] + a00 * A[j][1]);
      }
      // d dir / d p = (I - d d^T)/|p|, projected: P = M (I - d d^T) / |p|
      const double ilen = 1.0 / norm(lp);
      const V3 d = ilen * lp;
      for (int r = 0; r < 2; ++r) {
        const double md = M[r][0] * d.x + M[r][1] * d.y + M[r][2] * d.z;
        P[r][0] = (M[r][0] - md * d.x) * ilen;
        P[r][1] = (M[r][1] - md * d.y) * ilen;
        P[r][2] = (M[r][2] - md * d.z) * ilen;
      }
      if (want_intrinsics) {
        // d unproj / d G_k = w_k / |s| (I - u u^T); dx/dtheta_k = -M (that) [t1 t2]_k
        double Mu[2];
        for (int r = 0; r < 2; ++r) Mu[r] = M[r][0] * u.x + M[r][1] * u.y + M[r][2] * u.z;
        int li = 0;
        for (int y = 0; y < 4; ++y)
          for (int x = 0; x < 4; ++x) {
            const int seq = (s.x0 + x) + (s.y0 + y) * gw;
            const double wk = s.wx[x] * s.wy[y] * inv_n;
            idx[li] = 2 * seq;
            idx[li + 1] = 2 * seq + 1;
            const Tangents& t = tangents[seq];
            for (int dd = 0; dd < 2; ++dd) {
              const V3& tv = dd == 0 ? t.t1 : t.t2;
              const double ut = dot(u, tv);
              for (int r = 0; r < 2; ++r) {
                const double v = (M[r][0] * tv.x + M[r][1] * tv.y + M[r][2] * tv.z) - Mu[r] * ut;
                (r == 0 ? jx : jy)[li + dd] = -wk * v;
              }
            }
            li += 2;
          }
      }
      return true;
    } else if (m.c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
      V3 o, d;
      double J[6][2];
      Support s;
      double inv_n;
      if (!noncentral_unproject_jac(m, px, py, &o, &d, J, &s, &inv_n)) return false;
      double r[2], R[2][2];
      Tangents t;
      noncentral_residual_jac(o, d, J, lp, r, R, &t);
      const double idet = 1.0 / (R[0][0] * R[1][1] - R[0][1] * R[1][0]);
      const double Ri[2][2] = {{idet * R[1][1], -idet * R[0][1]}, {-idet * R[1][0], idet * R[0][0]}};
      // dr/dp = -[t1 t2]^T  =>  dx/dp = R^-1 [t1 t2]^T
      const V3 tt[2] = {t.t1, t.t2};
      for (int rr = 0; rr < 2; ++rr)
        for (int j = 0; j < 3; ++j)
          P[rr][j] = Ri[rr][0] * comp(tt[0], j) + Ri[rr][1] * comp(tt[1], j);
      if (want_intrinsics) {
        // dr/do = [t1 t2]^T ; dr/dd = [(o-p)^T dT1/dd ; (o-p)^T dT2/dd]
        double T1[3][3], T2[3][3];
        tangents_wrt_direction(d, T1, T2);
        const V3 pto = o - lp;
        double rd[2][3];
        for (int j = 0; j < 3; ++j) {
          rd[0][j] = pto.x * T1[0][j] + pto.y * T1[1][j] + pto.z * T1[2][j];
          rd[1][j] = pto.x * T2[0][j] + pto.y * T2[1][j] + pto.z * T2[2][j];
        }
        // through the normalisation of the interpolated direction: (I - d d^T)/|s|
        double rdn[2][3];
        for (int rr = 0; rr < 2; ++rr) {
          const double rdd = rd[rr][0] * d.x + rd[rr][1] * d.y + rd[rr][2] * d.z;
          rdn[rr][0] = (rd[rr][0] - rdd * d.x) * inv_n;
          rdn[rr][1] = (rd[rr][1] - rdd * d.y) * inv_n;
          rdn[rr][2] = (rd[rr][2] - rdd * d.z) * inv_n;
        }
        int li = 0;
        for (int y = 0; y < 4; ++y)
          for (int x = 0; x < 4; ++x) {
            const int seq = (s.x0 + x) + (s.y0 + y) * gw;
            const double wk = s.wx[x] * s.wy[y];
            const Tangents& tk = tangents[seq];
            const double* cd = m.dir_grid() + 3 * seq;
            const V3 dk = mk(cd[0], cd[1], cd[2]);
            // LineJacobianWrtLocalUpdate (line_parametrization.h:123-135)
            const V3 dirs[5] = {tk.t1, tk.t2, tk.t1, tk.t2, dk};
            for (int q = 0; q < 5; ++q) {
              idx[li + q] = 5 * seq + q;
              double dr[2];
              for (int rr = 0; rr < 2; ++rr) {
                if (q < 2)
                  dr[rr] = wk * (rdn[rr][0] * dirs[q].x + rdn[rr][1] * dirs[q].y + rdn[rr][2] * dirs[q].z);
                else
                  dr[rr] = wk * dot(tt[rr], dirs[q]);
              }
              jx[li + q] = -(Ri[0][0] * dr[0] + Ri[0][1] * dr[1]);
              jy[li + q] = -(Ri[1][0] * dr[0] + Ri[1][1] * dr[1]);
            }
            li += 5;
          }
      }
      return true;
    } else {
      opencv_point_jacobian(m, lp, P);
      if (want_intrinsics) {
        for (int i = 0; i < 12; ++i) idx[i] = i;
        opencv_intrinsics_jacobian(m, lp, jx, jy);
      }
      return true;
    }
  }

  // JointOptimizationCostFunction::Compute (joint_optimization.cc:240-306)
  void compute(bool compute_jacobians, State& S, Accumulator* acc) const {
    const b200ba_problem& P = *pb;
    // tangent images (joint_optimization.cc:254-270)
    std::vector<std::vector<Tangents>> tangents(P.n_cameras);
    if (compute_jacobians) {
      for (int c = 0; c < P.n_cameras; ++c) {
        Cam m{P.cameras[c], S.intrinsics[c].data()};
        if (m.c.model_type == B200BA_MODEL_CENTRAL_GENERIC ||
            m.c.model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
          const int G = m.G();
          tangents[c].resize(G);
          for (int k = 0; k < G; ++k)
            tangents[c][k] = compute_tangents(mk(m.p[3 * k], m.p[3 * k + 1], m.p[3 * k + 2]));
        }
      }
    }
    const int64_t o_begin = obs_begin;
    const int64_t o_end = obs_end < 0 ? P.n_obs : obs_end;
    if (oracle_fast::thread_count() > 1 && !acc->rec) {
      compute_mt(compute_jacobians, S, acc, tangents, o_begin, o_end);
      return;
    }
    int cur_imageset = -1, cur_camera = -1;
    Pose image_tr_global{};
    double R[3][3];
    for (int64_t o = o_begin; o < o_end; ++o) {
      const int iset = static_cast<int>(P.obs_imageset[o]);
      const int cam = static_cast<int>(P.obs_camera[o]);
      if (iset != cur_imageset || cam != cur_camera) {
        // image_tr_global = camera_tr_rig * rig_tr_global (joint_optimization.cc:277-280)
        image_tr_global = pose_mul(load_pose(&S.camera_tr_rig[7 * cam]), load_pose(&S.rig_tr_global[7 * iset]));
        qrot(image_tr_global.q, R);
        cur_imageset = iset;
        cur_camera = cam;
      }
      Cam m{P.cameras[cam], S.intrinsics[cam].data()};
      add_reprojection_residual(compute_jacobians, S, m, tangents[cam], o, iset, cam,
                                image_tr_global, R, acc);
    }
  }

  // Threaded evaluation for the full-size timing runs: the per-observation work (projection and
  // Jacobians -- in NUMERIC mode 3 + 32 / 80 re-projections with the control points perturbed IN
  // PLACE, hence one private copy of the state per thread) runs in parallel chunk by chunk; the
  // accumulation is then replayed sequentially in the reference's observation order, so H, b and
  // the cost vector are bitwise those of the single-threaded pass.
  void compute_mt(bool compute_jacobians, State& S, Accumulator* acc, const std::vector<std::vector<Tangents>>& tangents,
                  int64_t o_begin, int64_t o_end) const {
    const b200ba_problem& P = *pb;
    const int nt = oracle_fast::thread_count();
    const int64_t chunk = 32768;
    std::vector<Accumulator::Record> recs(static_cast<size_t>(std::min<int64_t>(chunk, std::max<int64_t>(0, o_end - o_begin))));
    std::vector<State> copies(nt, S);
    for (int64_t c0 = o_begin; c0 < o_end; c0 += chunk) {
      const int64_t c1 = std::min(o_end, c0 + chunk);
#pragma omp parallel num_threads(nt)
      {
#ifdef _OPENMP
        const int tid = omp_get_thread_num();
#else
        const int tid = 0;
#endif
        State& Sl = copies[tid];
        Accumulator ta;
        ta.huber = acc->huber;
        ta.out_residuals = acc->out_residuals;
        ta.out_jpoint = acc->out_jpoint;
        ta.out_jpose = acc->out_jpose;
        ta.out_jrig = acc->out_jrig;
        ta.out_jintr = acc->out_jintr;
        ta.out_intr_index = acc->out_intr_index;
        ta.out_K = acc->out_K;
        ta.out_has_jacobian = acc->out_has_jacobian;
#pragma omp for schedule(dynamic, 256)
        for (int64_t o = c0; o < c1; ++o) {
          const int iset = static_cast<int>(P.obs_imageset[o]);
          const int cam = static_cast<int>(P.obs_camera[o]);
          const Pose image_tr_global = pose_mul(load_pose(&Sl.camera_tr_rig[7 * cam]), load_pose(&Sl.rig_tr_global[7 * iset]));
          double R[3][3];
          qrot(image_tr_global.q, R);
          Cam m{P.cameras[cam], Sl.intrinsics[cam].data()};
          ta.rec = &recs[static_cast<size_t>(o - c0)];
          add_reprojection_residual(compute_jacobians, Sl, m, tangents[cam], o, iset, cam, image_tr_global, R, &ta);
        }
      }
      for (int64_t o = c0; o < c1; ++o) acc->replay(recs[static_cast<size_t>(o - c0)]);
    }
  }

  // AddReprojectionResidual (joint_optimization.cc:308-449)
  void add_reprojection_residual(bool compute_jacobians, State& S, const Cam& m,
                                 const std::vector<Tangents>& tangents, int64_t o, int iset,
                                 int cam, const Pose& image_tr_global, const double R[3][3],
                                 Accumulator* acc) const {
    const b200ba_problem& P = *pb;
    const int pidx = static_cast<int>(P.obs_point[o]);
    const V3 point = mk(S.points[3 * pidx], S.points[3 * pidx + 1], S.points[3 * pidx + 2]);
    const V3 lp = mat3_mul(R, point) + image_tr_global.t;
    const double mx = static_cast<double>(P.obs_xy[2 * o]);
    const double my = static_cast<double>(P.obs_xy[2 * o + 1]);

    double px = last_projection[2 * o], py = last_projection[2 * o + 1];
    if (!(px >= m.c.calibration_min_x && py >= m.c.calibration_min_y &&
          px < m.c.calibration_max_x + 1 && py < m.c.calibration_max_y + 1) ||
        std::isnan(px) || std::isnan(py)) {
      px = m.center_x();
      py = m.center_y();
    }
    if (!project_with_initial_estimate(m, lp, &px, &py)) {
      px = m.center_x();
      py = m.center_y();
      if (!project_with_initial_estimate(m, lp, &px, &py)) {
        acc->add_invalid();
        if (acc->out_residuals) {
          acc->out_residuals[2 * o] = std::numeric_limits<double>::quiet_NaN();
          acc->out_residuals[2 * o + 1] = std::numeric_limits<double>::quiet_NaN();
        }
        if (acc->out_has_jacobian) acc->out_has_jacobian[o] = 0;
        return;
      }
    }
    last_projection[2 * o] = px;
    last_projection[2 * o + 1] = py;
    const double rx = px - mx, ry = py - my;
    if (acc->out_residuals) {
      acc->out_residuals[2 * o] = rx;
      acc->out_residuals[2 * o + 1] = ry;
    }
    if (acc->out_has_jacobian) acc->out_has_jacobian[o] = 0;
    if (!compute_jacobians) {
      acc->add_residual(rx, ry);
      return;
    }

    const int K = m.intrinsics_jacobian_size();
    int intr_idx[80];
    double intr_jx[80], intr_jy[80];
    double Pm[2][3];  // d pixel / d local_point
    bool have_intr = false;
    if (jacobian_mode == B200BA_JACOBIAN_ANALYTIC) {
      if (!analytic_jacobians(m, tangents, lp, px, py, Pm, intr_idx, intr_jx, intr_jy,
                              !L.localize_only)) {
        acc->add_residual(rx, ry);
        return;
      }
      have_intr = true;
    } else {
      // numerical part (joint_optimization.cc:357-376): forward differences
      const double kDelta = numerical_diff_delta * (m.central() ? norm(lp) : 0.1);
      for (int dim = 0; dim < 3; ++dim) {
        V3 op = lp;
        if (dim == 0) op.x += kDelta;
        if (dim == 1) op.y += kDelta;
        if (dim == 2) op.z += kDelta;
        double ox = px, oy = py;
        if (!project_with_initial_estimate(m, op, &ox, &oy)) {
          acc->add_residual(rx, ry);
          return;
        }
        Pm[0][dim] = (ox - px) / kDelta;
        Pm[1][dim] = (oy - py) / kDelta;
      }
    }

    // analytical part (joint_optimization.cc:378-438). ComputeJacobian / ComputeRigJacobian
    // (joint_optimization_jacobians.h:39-118 / :120-343) re-derived: for the left update
    // q <- (1, delta) q, d(R(q) p)/d delta = -2 [R p]_x.
    double jpose[2][6], jrig[2][6], jpoint[2][3];
    auto times_neg2_skew = [](const double Pm_[2][3], const V3& v, double out[2][6]) {
      // Pm * (-2 [v]_x): column j of -2[v]_x is -2 (v x e_j)... (a x b = [a]_x b)
      // [v]_x = [0 -vz vy; vz 0 -vx; -vy vx 0]
      for (int r = 0; r < 2; ++r) {
        out[r][0] = -2 * (Pm_[r][1] * v.z - Pm_[r][2] * v.y);
        out[r][1] = -2 * (-Pm_[r][0] * v.z + Pm_[r][2] * v.x);
        out[r][2] = -2 * (Pm_[r][0] * v.y - Pm_[r][1] * v.x);
      }
    };
    if (L.rig_in_state) {
      const Pose ctr = load_pose(&S.camera_tr_rig[7 * cam]);
      const Pose rtg = load_pose(&S.rig_tr_global[7 * iset]);
      double Rc[3][3], Rr[3][3];
      qrot(ctr.q, Rc);
      qrot(rtg.q, Rr);
      const V3 rp = mat3_mul(Rr, point);       // R_r p
      const V3 rig_point = rp + rtg.t;         // R_r p + t_r
      const V3 crp = mat3_mul(Rc, rig_point);  // R_c (R_r p + t_r)
      // d local / d delta_r = R_c (-2 [R_r p]_x), d local / d t_r = R_c
      double PRc[2][3];
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 3; ++j)
          PRc[r][j] = Pm[r][0] * Rc[0][j] + Pm[r][1] * Rc[1][j] + Pm[r][2] * Rc[2][j];
      times_neg2_skew(PRc, rp, jpose);
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 3; ++j) jpose[r][3 + j] = PRc[r][j];
      // d local / d delta_c = -2 [R_c (R_r p + t_r)]_x, d local / d t_c = I
      times_neg2_skew(Pm, crp, jrig);
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 3; ++j) jrig[r][3 + j] = Pm[r][j];
      // d local / d p = R_c R_r
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 3; ++j)
          jpoint[r][j] = PRc[r][0] * Rr[0][j] + PRc[r][1] * Rr[1][j] + PRc[r][2] * Rr[2][j];
    } else {
      // Single camera: the reference differentiates with the COMPOSED image_q_global and an
      // identity translation block, and applies the result to rig_tr_global
      // (joint_optimization.cc:392-397,431-437) -- exact only when camera_tr_rig[0] = I
      // (SURVEY.md appendix B.5). Reproduced as is.
      const V3 rp = mat3_mul(R, point);
      times_neg2_skew(Pm, rp, jpose);
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 3; ++j) {
          jpose[r][3 + j] = Pm[r][j];
          jpoint[r][j] = Pm[r][0] * R[0][j] + Pm[r][1] * R[1][j] + Pm[r][2] * R[2][j];
          jrig[r][j] = jrig[r][3 + j] = 0;
        }
    }

    // model Jacobian (AccumulateModelJacobian, joint_optimization.cc:451-593)
    if (!L.localize_only && !have_intr) {
      if (m.c.model_type == B200BA_MODEL_CENTRAL_OPENCV) {
        for (int i = 0; i < 12; ++i) intr_idx[i] = i;
        opencv_intrinsics_jacobian(m, lp, intr_jx, intr_jy);
      } else if (!numeric_intrinsics_jacobian(m, tangents, lp, px, py, intr_idx, intr_jx, intr_jy)) {
        acc->add_residual(rx, ry);
        return;
      }
    }

    // assemble the column list in ascending global order (joint_optimization.cc:480-590)
    int idx[3 + 6 + 6 + 80];
    double jx[3 + 6 + 6 + 80], jy[3 + 6 + 6 + 80];
    int n = 0;
    auto push_point = [&]() {
      for (int j = 0; j < 3; ++j) {
        idx[n] = L.first_points + 3 * pidx + j;
        jx[n] = jpoint[0][j];
        jy[n] = jpoint[1][j];
        ++n;
      }
    };
    auto push_pose = [&]() {
      for (int j = 0; j < 6; ++j) {
        idx[n] = L.first_rig_tr_global + 6 * iset + j;
        jx[n] = jpose[0][j];
        jy[n] = jpose[1][j];
        ++n;
      }
    };
    auto push_rig = [&]() {
      if (!L.rig_in_state) return;
      for (int j = 0; j < 6; ++j) {
        idx[n] = L.first_camera_tr_rig + 6 * cam + j;
        jx[n] = jrig[0][j];
        jy[n] = jrig[1][j];
        ++n;
      }
    };
    if (L.eliminate_points) {
      push_point();
      push_pose();
      push_rig();
    } else {
      push_pose();
      push_rig();
      push_point();
    }
    if (!L.localize_only) {
      for (int j = 0; j < K; ++j) {
        idx[n] = L.intrinsics_offset[cam] + intr_idx[j];
        jx[n] = intr_jx[j];
        jy[n] = intr_jy[j];
        ++n;
      }
    }
    if (acc->out_has_jacobian) acc->out_has_jacobian[o] = 1;
    if (acc->out_jpoint)
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 3; ++j) acc->out_jpoint[(o * 2 + r) * 3 + j] = jpoint[r][j];
    if (acc->out_jpose)
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 6; ++j) acc->out_jpose[(o * 2 + r) * 6 + j] = jpose[r][j];
    if (acc->out_jrig)
      for (int r = 0; r < 2; ++r)
        for (int j = 0; j < 6; ++j) acc->out_jrig[(o * 2 + r) * 6 + j] = jrig[r][j];
    if (acc->out_jintr && !L.localize_only) {
      const int KK = acc->out_K;
      for (int j = 0; j < K && j < KK; ++j) {
        acc->out_jintr[(o * 2 + 0) * KK + j] = intr_jx[j];
        acc->out_jintr[(o * 2 + 1) * KK + j] = intr_jy[j];
        if (acc->out_intr_index) acc->out_intr_index[o * KK + j] = L.intrinsics_offset[cam] + intr_idx[j];
      }
    }
    acc->add_residual_with_jacobian(rx, ry, n, idx, jx, jy);
  }
};

// ------------------------------------------------------------------------------------
// dense solvers
// ------------------------------------------------------------------------------------
// Eigen::LDLT<MatrixXd, Lower>(H.selfadjointView<Upper>()).solve(b): symmetric-pivoting
// (largest |diagonal|) LDL^T, as used at LV/lm_optimizer.h:1022-1023, :1289 and :1361.
// A: n x n row-major; only the upper triangle is read. Unblocked (the oracle is run at
// small n); O(n^3 / 3).
bool ldlt_solve(int n, const double* A_upper, int lda, const double* b, int nrhs, int ldb,
                double* x, int ldx) {
  // lower-triangular working copy, row-major: L[i][j], j <= i
  std::vector<double> Lm(size_t(n) * n);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j <= i; ++j) Lm[size_t(i) * n + j] = A_upper[size_t(j) * lda + i];
  std::vector<int> transp(n);
  std::vector<double> col(n), odiag(n);
  auto at = [&](int i, int j) -> double& { return Lm[size_t(i) * n + j]; };
  // Eigen's unblocked LDLT is left-looking: when it searches the pivot of step k the
  // trailing diagonal entries still hold their ORIGINAL values (Eigen/src/Cholesky/LDLT.h,
  // ldlt_inplace<Lower>::unblocked). This right-looking restatement updates the trailing
  // block eagerly, so the original diagonal is tracked separately for the pivot search.
  for (int i = 0; i < n; ++i) odiag[i] = at(i, i);
  for (int k = 0; k < n; ++k) {
    int piv = k;
    double best = std::fabs(odiag[k]);
    for (int i = k + 1; i < n; ++i) {
      double v = std::fabs(odiag[i]);
      if (v > best) {
        best = v;
        piv = i;
      }
    }
    transp[k] = piv;
    if (piv != k) {
      std::swap(odiag[k], odiag[piv]);
      // symmetric row/column swap k <-> piv on the lower triangle
      for (int j = 0; j < k; ++j) std::swap(at(k, j), at(piv, j));
      for (int i = piv + 1; i < n; ++i) std::swap(at(i, k), at(i, piv));
      std::swap(at(k, k), at(piv, piv));
      for (int i = k + 1; i < piv; ++i) std::swap(at(i, k), at(piv, i));
    }
    // A[k][k] -= sum_j L[k][j]^2 D[j] and A[i][k] -= sum_j L[i][j] D[j] L[k][j] have been
    // applied eagerly (right-looking), so the current column is final.
    const double dk = at(k, k);
    const int rs = n - k - 1;
    if (rs > 0) {
      if (std::fabs(dk) > 0) {
        for (int i = k + 1; i < n; ++i) {
          col[i] = at(i, k);        // L[i][k] * d
          at(i, k) = col[i] / dk;   // L[i][k]
        }
        for (int i = k + 1; i < n; ++i) {
          const double lik = at(i, k);
          if (lik == 0) continue;
          double* row = &at(i, 0);
          for (int j = k + 1; j <= i; ++j) row[j] -= lik * col[j];
        }
      }
    }
  }
  // solve: x = P^T L^-T D^-1 L^-1 P b
  const double tolerance = 1.0 / std::numeric_limits<double>::max();
  std::vector<double> y(n);
  for (int r = 0; r < nrhs; ++r) {
    for (int i = 0; i < n; ++i) y[i] = b[size_t(i) * ldb + r];
    for (int k = 0; k < n; ++k) std::swap(y[k], y[transp[k]]);
    for (int i = 0; i < n; ++i) {
      double s = y[i];
      const double* row = &at(i, 0);
      for (int j = 0; j < i; ++j) s -= row[j] * y[j];
      y[i] = s;
    }
    for (int i = 0; i < n; ++i) {
      const double d = at(i, i);
      y[i] = (std::fabs(d) > tolerance) ? y[i] / d : 0.0;
    }
    for (int i = n - 1; i >= 0; --i) {
      const double yi = y[i];
      const double* row = &at(i, 0);
      for (int j = 0; j < i; ++j) y[j] -= row[j] * yi;
    }
    for (int k = n - 1; k >= 0; --k) std::swap(y[k], y[transp[k]]);
    for (int i = 0; i < n; ++i) x[size_t(i) * ldx + r] = y[i];
  }
  return true;
}

// SolveWithSchurComplementDenseOffDiag (LV/lm_optimizer.h:1246-1369), non-on-the-fly branch.
void schur_solve(int bs, int nb, int nd, const double* D, const double* B, const double* C,
                 const double* b1, const double* b2, double* x) {
  const int nbd = bs * nb;
  std::vector<double> DinvB(size_t(nbd) * nd), Dinvb(nbd);
  std::vector<double> I(size_t(bs) * bs, 0.0), Hb(size_t(bs) * bs);
  for (int i = 0; i < bs; ++i) I[size_t(i) * bs + i] = 1;
  for (int blk = 0; blk < nb; ++blk) {
    const int base = blk * bs;
    ldlt_solve(bs, D + size_t(blk) * bs * bs, bs, I.data(), bs, bs, Hb.data(), bs);  // :1289
    for (int row = 0; row < bs; ++row) {
      double r = 0;
      for (int k = 0; k < bs; ++k) r += Hb[size_t(row) * bs + k] * b1[base + k];
      Dinvb[base + row] = r;
      double* out = &DinvB[size_t(base + row) * nd];
      for (int col = 0; col < nd; ++col) {
        double rr = 0;
        for (int k = 0; k < bs; ++k) rr += Hb[size_t(row) * bs + k] * B[size_t(base + k) * nd + col];
        out[col] = rr;
      }
    }
  }
  // B^T D^-1 b (:1319) and the upper triangle of B^T D^-1 B (:1328); S = C - that (:1334-1335)
  std::vector<double> S(size_t(nd) * nd, 0.0), sb(nd);
  for (int i = 0; i < nd; ++i) {
    double r = 0;
    for (int k = 0; k < nbd; ++k) r += B[size_t(k) * nd + i] * Dinvb[k];
    sb[i] = b2[i] - r;
  }
  // rank-1 accumulation over the block rows keeps the loops contiguous
  for (int k = 0; k < nbd; ++k) {
    const double* brow = &B[size_t(k) * nd];
    const double* drow = &DinvB[size_t(k) * nd];
    for (int i = 0; i < nd; ++i) {
      const double bi = brow[i];
      if (bi == 0) continue;
      double* srow = &S[size_t(i) * nd];
      for (int j = i; j < nd; ++j) srow[j] += bi * drow[j];
    }
  }
  for (int i = 0; i < nd; ++i)
    for (int j = i; j < nd; ++j) S[size_t(i) * nd + j] = C[size_t(i) * nd + j] - S[size_t(i) * nd + j];
  std::vector<double> xd(nd);
  ldlt_solve(nd, S.data(), nd, sb.data(), 1, 1, xd.data(), 1);  // :1361
  for (int i = 0; i < nd; ++i) x[nbd + i] = xd[i];
  // back-substitution (:1366-1367)
  for (int k = 0; k < nbd; ++k) {
    double r = 0;
    const double* drow = &DinvB[size_t(k) * nd];
    for (int j = 0; j < nd; ++j) r += drow[j] * xd[j];
    x[k] = Dinvb[k] - r;
  }
}

// Full-size variants of ldlt_solve() / schur_solve() on the blocked, threaded kernels of
// ba_dense_fast.h (same quantities; summation order differs). Used above kFastDenseMinN.
double now_seconds();
constexpr int kFastDenseMinN = 768;
bool g_force_fast_dense = false;

// Lm: n x n row-major, lower triangle = the matrix; overwritten by the factor.
bool ldlt_solve_lower_fast(int n, double* Lm, const double* b, double* x) {
  std::vector<double> diag(n);
  for (int i = 0; i < n; ++i) diag[i] = Lm[size_t(i) * n + i];
  std::vector<int> transp;
  oracle_fast::ldlt_pivot_sequence(n, diag, &transp);
  bool any = false;
  for (int k = 0; k < n; ++k) any |= transp[k] != k;
  if (any) {
    // position -> original index after the whole transposition sequence; A'[i][j] = A[p[i]][p[j]]
    std::vector<int> p(n);
    for (int i = 0; i < n; ++i) p[i] = i;
    for (int k = 0; k < n; ++k) std::swap(p[k], p[transp[k]]);
    double* T = static_cast<double*>(malloc(size_t(n) * n * sizeof(double)));
#pragma omp parallel for schedule(dynamic, 16) num_threads(oracle_fast::thread_count())
    for (int i = 0; i < n; ++i)
      for (int j = 0; j <= i; ++j) {
        const int a = std::max(p[i], p[j]), c = std::min(p[i], p[j]);
        T[size_t(i) * n + j] = Lm[size_t(a) * n + c];
      }
#pragma omp parallel for schedule(dynamic, 16) num_threads(oracle_fast::thread_count())
    for (int i = 0; i < n; ++i) std::copy(T + size_t(i) * n, T + size_t(i) * n + i + 1, Lm + size_t(i) * n);
    free(T);
  }
  oracle_fast::ldlt_factor_blocked(n, Lm);
  const double tolerance = 1.0 / std::numeric_limits<double>::max();
  std::vector<double> y(b, b + n);
  for (int k = 0; k < n; ++k) std::swap(y[k], y[transp[k]]);
  for (int i = 0; i < n; ++i) {
    double s = y[i];
    const double* row = &Lm[size_t(i) * n];
    for (int j = 0; j < i; ++j) s -= row[j] * y[j];
    y[i] = s;
  }
  for (int i = 0; i < n; ++i) {
    const double d = Lm[size_t(i) * n + i];
    y[i] = (std::fabs(d) > tolerance) ? y[i] / d : 0.0;
  }
  for (int i = n - 1; i >= 0; --i) {
    const double yi = y[i];
    const double* row = &Lm[size_t(i) * n];
    for (int j = 0; j < i; ++j) y[j] -= row[j] * yi;
  }
  for (int k = n - 1; k >= 0; --k) std::swap(y[k], y[transp[k]]);
  std::copy(y.begin(), y.end(), x);
  return true;
}

void schur_solve_fast(int bs, int nb, int nd, const double* D, const double* B, const double* C,
                      const double* b1, const double* b2, double* x) {
  const int nbd = bs * nb;
  const int nt = oracle_fast::thread_count();
  // D^-1 b and (D^-1 B)^T, B^T: column i of B becomes row i (k contiguous). Tiled over the dense
  // columns so that both the row-major reads of B and the transposed writes stay cache-resident.
  const bool verbose = getenv("ORACLE_VERBOSE") != nullptr;
  double tp = now_seconds();
  std::vector<double> Dinvb(nbd), Hinv(size_t(nb) * bs * bs);
  double* Bt = static_cast<double*>(malloc(std::max<size_t>(1, size_t(nd) * nbd) * sizeof(double)));
  double* Xt = static_cast<double*>(malloc(std::max<size_t>(1, size_t(nd) * nbd) * sizeof(double)));
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int blk = 0; blk < nb; ++blk) {
    std::vector<double> I(size_t(bs) * bs, 0.0);
    for (int i = 0; i < bs; ++i) I[size_t(i) * bs + i] = 1;
    double* Hb = &Hinv[size_t(blk) * bs * bs];
    const int base = blk * bs;
    ldlt_solve(bs, D + size_t(blk) * bs * bs, bs, I.data(), bs, bs, Hb, bs);  // :1289
    for (int row = 0; row < bs; ++row) {
      double r = 0;
      for (int k = 0; k < bs; ++k) r += Hb[size_t(row) * bs + k] * b1[base + k];
      Dinvb[base + row] = r;
    }
  }
  constexpr int CT = 64;
  const int nct = (nd + CT - 1) / CT;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt)
  for (int ct = 0; ct < nct; ++ct) {
    const int c0 = ct * CT, c1 = std::min(nd, c0 + CT);
    for (int blk = 0; blk < nb; ++blk) {
      const int base = blk * bs;
      const double* Hb = &Hinv[size_t(blk) * bs * bs];
      for (int col = c0; col < c1; ++col) {
        for (int row = 0; row < bs; ++row) {
          double rr = 0;
          for (int k = 0; k < bs; ++k) rr += Hb[size_t(row) * bs + k] * B[size_t(base + k) * nd + col];
          Xt[size_t(col) * nbd + base + row] = rr;
          Bt[size_t(col) * nbd + base + row] = B[size_t(base + row) * nd + col];
        }
      }
    }
  }
  if (verbose) fprintf(stderr, "[oracle] schur: D^-1 B + transposes %.2f s\n", now_seconds() - tp), tp = now_seconds();
  std::vector<double> sb(nd);
#pragma omp parallel for schedule(static) num_threads(nt)
  for (int i = 0; i < nd; ++i) {
    double r = 0;
    const double* bt = Bt + size_t(i) * nbd;
    for (int k = 0; k < nbd; ++k) r += bt[k] * Dinvb[k];
    sb[i] = b2[i] - r;
  }
  // lower-triangular S: S[j][i] = C_upper[i][j] - sum_k Xt[j][k] Bt[i][k], i <= j   (:1328, :1334-1335)
  double* Sl = static_cast<double*>(malloc(std::max<size_t>(1, size_t(nd) * nd) * sizeof(double)));
  {
    constexpr int TT = 64;  // tiled transpose of the upper triangle of C
    const int ntt = (nd + TT - 1) / TT;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nt)
    for (int tj = 0; tj < ntt; ++tj)
      for (int ti = 0; ti <= tj; ++ti) {
        const int j1 = std::min(nd, (tj + 1) * TT), i1 = std::min(nd, (ti + 1) * TT);
        for (int i = ti * TT; i < i1; ++i)
          for (int j = std::max(i, tj * TT); j < j1; ++j) Sl[size_t(j) * nd + i] = C[size_t(i) * nd + j];
      }
  }
  if (verbose) fprintf(stderr, "[oracle] schur: S <- C^T %.2f s\n", now_seconds() - tp), tp = now_seconds();
  oracle_fast::gemm_nt_lower(nd, nd, nbd, -1.0, Xt, nbd, Bt, nbd, Sl, nd, 0);
  if (verbose) fprintf(stderr, "[oracle] schur: contraction %.2f s (%.1f GF/s)\n", now_seconds() - tp, double(nd) * nd * nbd / (now_seconds() - tp) / 1e9), tp = now_seconds();
  std::vector<double> xd(nd);
  ldlt_solve_lower_fast(nd, Sl, sb.data(), xd.data());  // :1361
  if (verbose) fprintf(stderr, "[oracle] schur: LDLT + solve %.2f s (%.1f GF/s)\n", now_seconds() - tp, double(nd) * nd * nd / 3 / (now_seconds() - tp) / 1e9), tp = now_seconds();
  free(Sl);
  free(Bt);
  for (int i = 0; i < nd; ++i) x[nbd + i] = xd[i];
  // back-substitution (:1366-1367): x_b = D^-1 b - (D^-1 B) x_d
  std::vector<double> t(nbd, 0.0);
  for (int j = 0; j < nd; ++j) {
    const double xj = xd[j];
    const double* xt = &Xt[size_t(j) * nbd];
    for (int k = 0; k < nbd; ++k) t[k] += xt[k] * xj;
  }
  for (int k = 0; k < nbd; ++k) x[k] = Dinvb[k] - t[k];
  free(Xt);
}

// CostIsSmallerThan (LV/lm_optimizer.h:993-1011)
bool cost_is_smaller_than(const std::vector<double>& left, const std::vector<double>& right) {
  double ls = 0, rs = 0;
  size_t count = 0;
  for (size_t i = 0; i < left.size(); ++i) {
    if (left[i] >= 0 && right[i] >= 0) {
      ls += left[i];
      rs += right[i];
      ++count;
    }
  }
  return count > 0 && ls < rs;
}

// outcome of each LM attempt of the last oracle_optimize (B200BA_LM_*; a NaN update is B200BA_LM_REFUSED_PIVOT)
std::vector<int32_t> g_lm_events;

double now_seconds() {
  using namespace std::chrono;
  return duration_cast<duration<double>>(steady_clock::now().time_since_epoch()).count();
}

bool check_options(const b200ba_problem* pb, const b200ba_options* opt) {
  if (!pb || !opt) return false;
  for (int c = 0; c < pb->n_cameras; ++c) {
    int t = pb->cameras[c].model_type;
    if (t != B200BA_MODEL_CENTRAL_GENERIC && t != B200BA_MODEL_NONCENTRAL_GENERIC &&
        t != B200BA_MODEL_CENTRAL_OPENCV)
      return false;
  }
  return true;
}

}  // namespace

// ------------------------------------------------------------------------------------
// C interface
// ------------------------------------------------------------------------------------
extern "C" {

int oracle_optimize(const b200ba_problem* pb, b200ba_state* state, const b200ba_options* opt,
                    b200ba_report* report) {
  if (!check_options(pb, opt) || !state || !report) return 1;
  memset(report, 0, sizeof(*report));
  g_lm_events.clear();
  const b200ba_problem& P = *pb;
  Layout L = make_layout(P, *opt);
  State S = load_state(P, *state);
  std::vector<double> last_proj(2 * P.n_obs, 0.0);
  if (state->last_projection) std::copy(state->last_projection, state->last_projection + 2 * P.n_obs, last_proj.begin());

  CostFunction cf;
  cf.pb = pb;
  cf.L = L;
  cf.numerical_diff_delta = opt->numerical_diff_delta;
  cf.jacobian_mode = opt->jacobian_mode;
  cf.last_projection = last_proj.data();

  const int nbd = L.block_dof(), nd = L.dense_dof(), dof = L.dof;
  std::vector<double> x(dof), orig_diag(dof);
  double lambda = 0;
  double init_lambda = opt->init_lambda;
  double final_cost = -1;
  std::vector<double> final_costs;

  // debug switches of OptimizeJointly (joint_optimization.cc:866-903)
  if (opt->debug_verify_cost) {
    double c[2];
    for (int r = 0; r < 2; ++r) {
      Accumulator a1, a2;
      a1.huber = a2.huber = opt->huber_parameter;
      cf.compute(false, S, &a1);
      Accumulator a2m;
      a2m.huber = opt->huber_parameter;
      a2m.allocate(L.block_size, L.num_blocks, nd);
      cf.compute(true, S, &a2m);
      if (std::fabs(a1.cost - a2m.cost) > 1e-3f)
        fprintf(stderr, "[oracle] Cost differs when computed with or without Jacobians: %.12g vs %.12g\n", a1.cost, a2m.cost);
      c[r] = a1.cost;
    }
    if (!(std::fabs(c[0] - c[1]) <= 1e-3f)) return 5;
  }
  std::vector<char> fixed;
  if (opt->debug_fix_points || opt->debug_fix_poses || opt->debug_fix_rig_poses || opt->debug_fix_intrinsics) {
    fixed.assign(dof, 0);
    if (opt->debug_fix_points)
      for (int i = 0; i < 3 * P.n_points; ++i) fixed[L.first_points + i] = 1;
    if (opt->debug_fix_poses)
      for (int i = 0; i < 6 * P.n_imagesets; ++i) fixed[L.first_rig_tr_global + i] = 1;
    if (opt->debug_fix_rig_poses && L.rig_in_state)
      for (int i = 0; i < 6 * P.n_cameras; ++i) fixed[L.first_camera_tr_rig + i] = 1;
    if (opt->debug_fix_intrinsics && !L.localize_only)
      for (int i = L.intrinsics_offset[0]; i < dof; ++i) fixed[i] = 1;
  }

  // OptimizeJointly's loop of single LM iterations (joint_optimization.cc:905-940); each
  // pass is LMOptimizer::OptimizeImpl with max_iteration_count = 1 (LV/lm_optimizer.h:628-991).
  for (int iteration = 0; iteration < opt->max_iteration_count; ++iteration) {
    int num_iterations_performed = 0;
    double last_cost;
    std::vector<double> residual_cost_vector;
    residual_cost_vector.reserve(P.n_obs);
    Accumulator acc;
    acc.allocate(L.block_size, L.num_blocks, nd);
    acc.cost_vector = &residual_cost_vector;
    acc.huber = opt->huber_parameter;
    double t0 = now_seconds();
    cf.compute(true, S, &acc);
    report->cost_and_jacobian_evaluation_time += now_seconds() - t0;
    last_cost = acc.cost;
    if (iteration == 0) report->initial_cost = last_cost;
    bool applied_update = false;
    if (acc.cost == 0) {
      final_cost = last_cost;
      final_costs = residual_cost_vector;
      break;  // "Cost is zero, stopping." -> num_iterations_performed == 0
    }
    // lambda (lm_optimizer.h:766-781)
    if (init_lambda >= 0) {
      lambda = init_lambda;
    } else {
      lambda = 0;
      for (int b = 0; b < L.num_blocks; ++b)
        for (int k = 0; k < L.block_size; ++k)
          lambda += acc.block_diag[(size_t(b) * L.block_size + k) * L.block_size + k];
      for (int i = 0; i < nd; ++i) lambda += acc.dense[size_t(i) * nd + i];
      lambda = opt->init_lambda_factor * lambda / dof;
    }
    // cache the diagonal (lm_optimizer.h:783-796)
    {
      int di = 0;
      for (int b = 0; b < L.num_blocks; ++b)
        for (int k = 0; k < L.block_size; ++k)
          orig_diag[di++] = acc.block_diag[(size_t(b) * L.block_size + k) * L.block_size + k];
      for (int i = 0; i < nd; ++i) orig_diag[di++] = acc.dense[size_t(i) * nd + i];
    }
    int attempts = 0;
    for (int lm_iteration = 0; lm_iteration < opt->max_lm_attempts; ++lm_iteration) {
      ++attempts;
      double ts = now_seconds();
      {
        int di = 0;
        for (int b = 0; b < L.num_blocks; ++b)
          for (int k = 0; k < L.block_size; ++k)
            acc.block_diag[(size_t(b) * L.block_size + k) * L.block_size + k] = orig_diag[di++] + lambda;
        for (int i = 0; i < nd; ++i) acc.dense[size_t(i) * nd + i] = orig_diag[di++] + lambda;
      }
      if (!fixed.empty()) {
        // SolveWithFixedVariables (LV/lm_optimizer.h:1069-1121): full H with the fixed rows / columns
        // removed, lambda on the thinned diagonal, dense LDLT, zero update for the fixed unknowns.
        // (the block / dense diagonals already carry + lambda from the loop above; the reference adds it
        // to the thinned copy of the un-damped H -- same matrix)
        std::vector<int> keep;
        for (int i = 0; i < dof; ++i)
          if (!fixed[i]) keep.push_back(i);
        const int m = static_cast<int>(keep.size());
        auto Hat = [&](int i, int k) -> double {  // i <= k, global indices
          if (k < nbd) {
            const int bi = i / L.block_size, bk = k / L.block_size;
            if (bi != bk) return 0.0;
            return acc.block_diag[(size_t(bi) * L.block_size + (i - bi * L.block_size)) * L.block_size + (k - bk * L.block_size)];
          }
          if (i < nbd) return acc.off_diag[size_t(i) * nd + (k - nbd)];
          return acc.dense[size_t(i - nbd) * nd + (k - nbd)];
        };
        std::vector<double> Ht(size_t(m) * m, 0.0), bt(m), xt(m);
        for (int a = 0; a < m; ++a) {
          for (int c = a; c < m; ++c) Ht[size_t(a) * m + c] = Hat(keep[a], keep[c]);
          bt[a] = keep[a] < nbd ? acc.b_block[keep[a]] : acc.b_dense[keep[a] - nbd];
        }
        ldlt_solve(m, Ht.data(), m, bt.data(), 1, 1, xt.data(), 1);
        std::fill(x.begin(), x.end(), 0.0);
        for (int a = 0; a < m; ++a) x[keep[a]] = xt[a];
      } else if (nbd > 0 && (nd >= kFastDenseMinN || g_force_fast_dense)) {
        schur_solve_fast(L.block_size, L.num_blocks, nd, acc.block_diag, acc.off_diag, acc.dense,
                         acc.b_block.data(), acc.b_dense.data(), x.data());
      } else if (nbd > 0) {
        schur_solve(L.block_size, L.num_blocks, nd, acc.block_diag, acc.off_diag, acc.dense,
                    acc.b_block.data(), acc.b_dense.data(), x.data());
      } else {
        ldlt_solve(nd, acc.dense, nd, acc.b_dense.data(), 1, 1, x.data(), 1);
      }
      report->solve_time += now_seconds() - ts;
      if (std::isnan(x[0])) {
        g_lm_events.push_back(B200BA_LM_REFUSED_PIVOT);
        lambda = 2.f * lambda;
        continue;
      }
      State updated = S;
      apply_update(P, L, &updated, x.data());
      std::vector<double> test_costs;
      test_costs.reserve(P.n_obs);
      Accumulator test;
      test.cost_vector = &test_costs;
      test.huber = opt->huber_parameter;
      double tc = now_seconds();
      cf.compute(false, updated, &test);
      report->cost_and_jacobian_evaluation_time += now_seconds() - tc;
      if (cost_is_smaller_than(test_costs, residual_cost_vector)) {
        g_lm_events.push_back(B200BA_LM_ACCEPTED);
        S = updated;
        lambda = 0.5f * lambda;
        applied_update = true;
        num_iterations_performed += 1;
        last_cost = test.cost;
        final_costs = test_costs;
        break;
      } else {
        g_lm_events.push_back(B200BA_LM_REJECTED_COST);
        lambda = 2.f * lambda;
      }
    }
    final_cost = last_cost;
    if (!applied_update) final_costs = residual_cost_vector;
    init_lambda = lambda;
    report->final_lambda = lambda;
    report->num_iterations_performed += num_iterations_performed;
    if (report->trace_len < B200BA_MAX_TRACE) {
      report->trace_cost[report->trace_len] = last_cost;
      report->trace_lambda[report->trace_len] = lambda;
      report->trace_attempts[report->trace_len] = attempts;
      report->trace_len++;
    }
    if (opt->print_progress)
      fprintf(stderr, "[oracle] iteration %d: cost %.12g lambda %.6g attempts %d%s\n", iteration,
              last_cost, lambda, attempts, applied_update ? "" : " (no update found)");
    if (num_iterations_performed == 0) break;
    report->performed_an_iteration = 1;
    if (last_cost == 0) break;
  }
  report->final_cost = final_cost;
  // final statistics: valid count and RMSE at the final state (residual-only pass from the
  // warm start, SURVEY.md 8d)
  {
    std::vector<double> res(2 * P.n_obs), costs;
    costs.reserve(P.n_obs);
    Accumulator a;
    a.cost_vector = &costs;
    a.huber = opt->huber_parameter;
    a.out_residuals = res.data();
    cf.compute(false, S, &a);
    double ss = 0;
    int64_t nv = 0;
    for (int64_t o = 0; o < P.n_obs; ++o)
      if (costs[o] >= 0) {
        ss += res[2 * o] * res[2 * o] + res[2 * o + 1] * res[2 * o + 1];
        ++nv;
      }
    report->n_valid = nv;
    report->n_invalid = P.n_obs - nv;
    report->rmse = nv > 0 ? std::sqrt(ss / nv) : 0;
  }
  store_state(P, S, state);
  if (state->last_projection) std::copy(last_proj.begin(), last_proj.end(), state->last_projection);
  return 0;
}

int32_t oracle_lm_events(int32_t* codes, int32_t cap) {
  const int32_t n = static_cast<int32_t>(g_lm_events.size());
  for (int32_t i = 0; i < n && i < cap && codes; ++i) codes[i] = g_lm_events[i];
  return n;
}

int oracle_evaluate(const b200ba_problem* pb, b200ba_state* state, const b200ba_options* opt,
                    int compute_jacobians, double* residuals, double* costs, double* total_cost,
                    double* j_point, double* j_pose, double* j_rig, double* j_intr,
                    int32_t* intr_index, int32_t K, int32_t* has_jacobian) {
  if (!check_options(pb, opt) || !state) return 1;
  const b200ba_problem& P = *pb;
  Layout L = make_layout(P, *opt);
  State S = load_state(P, *state);
  std::vector<double> last_proj(2 * P.n_obs, 0.0);
  if (state->last_projection) std::copy(state->last_projection, state->last_projection + 2 * P.n_obs, last_proj.begin());
  CostFunction cf;
  cf.pb = pb;
  cf.L = L;
  cf.numerical_diff_delta = opt->numerical_diff_delta;
  cf.jacobian_mode = opt->jacobian_mode;
  cf.last_projection = last_proj.data();
  std::vector<double> cv;
  cv.reserve(P.n_obs);
  Accumulator acc;
  acc.cost_vector = &cv;
  acc.huber = opt->huber_parameter;
  acc.out_residuals = residuals;
  acc.out_jpoint = j_point;
  acc.out_jpose = j_pose;
  acc.out_jrig = j_rig;
  acc.out_jintr = j_intr;
  acc.out_intr_index = intr_index;
  acc.out_K = K;
  acc.out_has_jacobian = has_jacobian;
  cf.compute(compute_jacobians != 0, S, &acc);
  if (costs) std::copy(cv.begin(), cv.end(), costs);
  if (total_cost) *total_cost = acc.cost;
  if (state->last_projection) std::copy(last_proj.begin(), last_proj.end(), state->last_projection);
  return 0;
}

int32_t oracle_degrees_of_freedom(const b200ba_problem* pb, const b200ba_options* opt) {
  if (!check_options(pb, opt)) return -1;
  return make_layout(*pb, *opt).dof;
}

int oracle_build_system(const b200ba_problem* pb, b200ba_state* state, const b200ba_options* opt,
                        int32_t n, double* H, double* b, double* cost) {
  if (!check_options(pb, opt) || !state) return 1;
  const b200ba_problem& P = *pb;
  Layout L = make_layout(P, *opt);
  if (n != L.dof) return 2;
  State S = load_state(P, *state);
  std::vector<double> last_proj(2 * P.n_obs, 0.0);
  if (state->last_projection) std::copy(state->last_projection, state->last_projection + 2 * P.n_obs, last_proj.begin());
  CostFunction cf;
  cf.pb = pb;
  cf.L = L;
  cf.numerical_diff_delta = opt->numerical_diff_delta;
  cf.jacobian_mode = opt->jacobian_mode;
  cf.last_projection = last_proj.data();
  Accumulator acc;
  const int nd = L.dense_dof(), nbd = L.block_dof(), bs = L.block_size;
  acc.allocate(bs, L.num_blocks, nd);
  acc.huber = opt->huber_parameter;
  cf.compute(true, S, &acc);
  std::fill(H, H + size_t(n) * n, 0.0);
  for (int blk = 0; blk < L.num_blocks; ++blk)
    for (int i = 0; i < bs; ++i)
      for (int k = i; k < bs; ++k)
        H[size_t(blk * bs + i) * n + (blk * bs + k)] = acc.block_diag[(size_t(blk) * bs + i) * bs + k];
  for (int i = 0; i < nbd; ++i)
    for (int k = 0; k < nd; ++k) H[size_t(i) * n + nbd + k] = acc.off_diag[size_t(i) * nd + k];
  for (int i = 0; i < nd; ++i)
    for (int k = i; k < nd; ++k) H[size_t(nbd + i) * n + nbd + k] = acc.dense[size_t(i) * nd + k];
  for (int i = 0; i < nbd; ++i) b[i] = acc.b_block[i];
  for (int i = 0; i < nd; ++i) b[nbd + i] = acc.b_dense[i];
  if (cost) *cost = acc.cost;
  if (state->last_projection) std::copy(last_proj.begin(), last_proj.end(), state->last_projection);
  return 0;
}

int oracle_schur_solve(int32_t bs, int32_t nb, int32_t nd, const double* D, const double* B,
                       const double* C, const double* b1, const double* b2, double* x) {
  schur_solve(bs, nb, nd, D, B, C, b1, b2, x);
  return 0;
}

int oracle_solve_dense(int32_t n, const double* H, const double* b, double* x) {
  return ldlt_solve(n, H, n, b, 1, 1, x, 1) ? 0 : 1;
}

int oracle_apply_update(const b200ba_problem* pb, b200ba_state* state, const b200ba_options* opt,
                        const double* delta) {
  if (!check_options(pb, opt) || !state) return 1;
  Layout L = make_layout(*pb, *opt);
  State S = load_state(*pb, *state);
  apply_update(*pb, L, &S, delta);
  store_state(*pb, S, state);
  return 0;
}

int oracle_project(const b200ba_camera* cam, const double* intrinsics, int64_t n,
                   const double* local_points, double* pixels, int32_t* ok) {
  std::vector<double> p(intrinsics, intrinsics + intr_size(cam));
  Cam m{*cam, p.data()};
  for (int64_t i = 0; i < n; ++i) {
    V3 lp = mk(local_points[3 * i], local_points[3 * i + 1], local_points[3 * i + 2]);
    double px = pixels[2 * i], py = pixels[2 * i + 1];
    bool r = project_with_initial_estimate(m, lp, &px, &py);
    pixels[2 * i] = px;
    pixels[2 * i + 1] = py;
    if (ok) ok[i] = r ? 1 : 0;
  }
  return 0;
}

// CentralGenericBSplineDirectionCostFunction::Compute (APP/models/central_generic.cc:152-228):
// Compute<true>  -> ComputeUnprojectedDirectionResidualAndJacobianWrtGridUpdates (:86-150): the
//                   normalised spline and d/d(control point) = w/|s| (I - u u^T) (generated code
//                   central_generic_jacobians.cc:31-317 re-derived), chained with [t1 t2] of the
//                   control point (DirectionJacobianWrtLocalUpdate, direction_parametrization.h:62-70);
// Compute<false> -> UnprojectFromGrid (b_spline.h fast evaluation, normalised).
// Quadratic loss: cost entry 1/2 r^2 per scalar residual.
static double dirfit_compute(bool jac, int gw, int gh, const std::vector<double>& grid, int64_t n,
                             const double* gp, const double* dirs, std::vector<double>* H,
                             std::vector<double>* b, std::vector<double>* costs) {
  const int dof = 2 * gw * gh;
  std::vector<Tangents> tan;
  if (jac) {
    tan.resize(size_t(gw) * gh);
    for (int i = 0; i < gw * gh; ++i) tan[i] = compute_tangents(grid_at(grid.data(), gw, i % gw, i / gw));
    std::fill(H->begin(), H->end(), 0.0);
    std::fill(b->begin(), b->end(), 0.0);
  }
  costs->clear();
  double cost = 0;
  for (int64_t i = 0; i < n; ++i) {
    const V3 m = mk(dirs[3 * i], dirs[3 * i + 1], dirs[3 * i + 2]);
    const double gx = gp[2 * i], gy = gp[2 * i + 1];
    V3 r;
    if (!jac) {
      r = normalized(bspline_surface(grid.data(), gw, gx, gy)) - m;
    } else {
      const int ix = static_cast<int>(std::floor(gx + 2)), iy = static_cast<int>(std::floor(gy + 2));
      const int x0 = ix - 3, y0 = iy - 3;
      double wx[4], wy[4];
      bspline_weights(gx + 2 - x0, wx);
      bspline_weights(gy + 2 - y0, wy);
      V3 sum = mk(0, 0, 0);
      for (int rr = 0; rr < 4; ++rr) {
        V3 a = mk(0, 0, 0);
        for (int c = 0; c < 4; ++c) a = a + wx[c] * grid_at(grid.data(), gw, x0 + c, y0 + rr);
        sum = sum + wy[rr] * a;
      }
      const double inv_n = 1.0 / std::sqrt(dot(sum, sum));
      const V3 u = inv_n * sum;
      r = u - m;
      double J[3][32];
      int idx[32];
      for (int rr = 0; rr < 4; ++rr)
        for (int c = 0; c < 4; ++c) {
          const int k = c + 4 * rr;
          const int seq = (x0 + c) + (y0 + rr) * gw;
          const double w = wx[c] * wy[rr] * inv_n;
          const Tangents& t = tan[seq];
          const V3 c1 = w * (t.t1 - dot(u, t.t1) * u);
          const V3 c2 = w * (t.t2 - dot(u, t.t2) * u);
          idx[2 * k] = 2 * seq;
          idx[2 * k + 1] = 2 * seq + 1;
          for (int q = 0; q < 3; ++q) {
            J[q][2 * k] = comp(c1, q);
            J[q][2 * k + 1] = comp(c2, q);
          }
        }
      // three scalar residuals, each AddResidualWithJacobian(residual, indices, row)
      for (int q = 0; q < 3; ++q) {
        const double rq = comp(r, q);
        for (int a = 0; a < 32; ++a) {
          (*b)[idx[a]] += J[q][a] * rq;
          for (int c = a; c < 32; ++c) (*H)[size_t(idx[a]) * dof + idx[c]] += J[q][a] * J[q][c];
        }
      }
    }
    for (int q = 0; q < 3; ++q) {
      const double c = 0.5 * comp(r, q) * comp(r, q);
      costs->push_back(c);
      cost += c;
    }
  }
  return cost;
}

// CentralGenericModel::FitToPixelDirectionsImpl (APP/models/central_generic.cc:551-568):
// LMOptimizer<double>::Optimize(state, cost, max_iteration_count, max_lm_attempts 10,
// init_lambda -1, init_lambda_factor 0.001f) with DirectionGridStateWithLocalUpdates (:40-83),
// no Schur structure -> SolveDensely (LV/lm_optimizer.h:1013-1024).
int oracle_fit_directions(int32_t gw, int32_t gh, double* grid_io, int64_t n, const double* grid_points,
                          const double* directions, int32_t max_iteration_count, b200ba_fit_report* report) {
  if (gw < 4 || gh < 4 || !grid_io || n < 0 || !report) return 1;
  memset(report, 0, sizeof(*report));
  const int dof = 2 * gw * gh;
  std::vector<double> grid(grid_io, grid_io + size_t(3) * gw * gh);
  std::vector<double> H(size_t(dof) * dof), b(dof), x(dof), orig_diag(dof), costs, test_costs;
  double lambda = 0, last_cost = 0;
  const double init_lambda_factor = static_cast<double>(0.001f);
  for (int iteration = 0; iteration < max_iteration_count; ++iteration) {
    last_cost = dirfit_compute(true, gw, gh, grid, n, grid_points, directions, &H, &b, &costs);
    if (iteration == 0) report->initial_cost = last_cost;
    if (last_cost == 0) break;
    if (iteration == 0) {
      lambda = 0;
      for (int i = 0; i < dof; ++i) lambda += H[size_t(i) * dof + i];
      lambda = init_lambda_factor * lambda / dof;
    }
    for (int i = 0; i < dof; ++i) orig_diag[i] = H[size_t(i) * dof + i];
    bool applied = false;
    for (int attempt = 0; attempt < 10; ++attempt) {
      report->lm_attempts++;
      for (int i = 0; i < dof; ++i) H[size_t(i) * dof + i] = orig_diag[i] + lambda;
      ldlt_solve(dof, H.data(), dof, b.data(), 1, 1, x.data(), 1);
      if (std::isnan(x[0])) {
        lambda = 2.f * lambda;
        continue;
      }
      // DirectionGridStateWithLocalUpdates::operator-= (central_generic.cc:65-80)
      std::vector<double> updated = grid;
      for (int i = 0; i < gw * gh; ++i) {
        const V3 d = grid_at(grid.data(), gw, i % gw, i / gw);
        const V3 nd = apply_local_update_to_direction(d, compute_tangents(d), -x[2 * i], -x[2 * i + 1]);
        updated[3 * i] = nd.x;
        updated[3 * i + 1] = nd.y;
        updated[3 * i + 2] = nd.z;
      }
      const double test_cost = dirfit_compute(false, gw, gh, updated, n, grid_points, directions, nullptr, nullptr, &test_costs);
      if (cost_is_smaller_than(test_costs, costs)) {
        grid = updated;
        lambda = 0.5f * lambda;
        applied = true;
        report->num_iterations_performed += 1;
        last_cost = test_cost;
        break;
      }
      lambda = 2.f * lambda;
    }
    if (!applied || last_cost == 0) break;
  }
  report->final_cost = last_cost;
  report->final_lambda = lambda;
  std::copy(grid.begin(), grid.end(), grid_io);
  return 0;
}

int oracle_unproject(const b200ba_camera* cam, const double* intrinsics, int64_t n,
                     const double* pixels, double* directions, double* origins, int32_t* ok) {
  std::vector<double> p(intrinsics, intrinsics + intr_size(cam));
  Cam m{*cam, p.data()};
  for (int64_t i = 0; i < n; ++i) {
    V3 d = mk(0, 0, 0), o = mk(0, 0, 0);
    bool r = false;
    if (cam->model_type == B200BA_MODEL_CENTRAL_GENERIC)
      r = central_unproject(m, pixels[2 * i], pixels[2 * i + 1], &d);
    else if (cam->model_type == B200BA_MODEL_NONCENTRAL_GENERIC)
      r = noncentral_unproject(m, pixels[2 * i], pixels[2 * i + 1], &o, &d);
    if (directions) {
      directions[3 * i] = d.x;
      directions[3 * i + 1] = d.y;
      directions[3 * i + 2] = d.z;
    }
    if (origins) {
      origins[3 * i] = o.x;
      origins[3 * i + 1] = o.y;
      origins[3 * i + 2] = o.z;
    }
    if (ok) ok[i] = r ? 1 : 0;
  }
  return 0;
}

int oracle_unproject_jacobian(const b200ba_camera* cam, const double* intrinsics, int64_t n,
                              const double* pixels, double* directions, double* origins,
                              double* jac, int32_t* ok) {
  std::vector<double> p(intrinsics, intrinsics + intr_size(cam));
  Cam m{*cam, p.data()};
  for (int64_t i = 0; i < n; ++i) {
    V3 d = mk(0, 0, 0), o = mk(0, 0, 0);
    bool r = false;
    if (cam->model_type == B200BA_MODEL_CENTRAL_GENERIC) {
      double J[3][2];
      r = central_unproject_jac(m, pixels[2 * i], pixels[2 * i + 1], &d, J);
      if (r && jac)
        for (int a = 0; a < 3; ++a)
          for (int b = 0; b < 2; ++b) jac[(i * 3 + a) * 2 + b] = J[a][b];
    } else if (cam->model_type == B200BA_MODEL_NONCENTRAL_GENERIC) {
      double J[6][2];
      r = noncentral_unproject_jac(m, pixels[2 * i], pixels[2 * i + 1], &o, &d, J);
      if (r && jac)
        for (int a = 0; a < 6; ++a)
          for (int b = 0; b < 2; ++b) jac[(i * 6 + a) * 2 + b] = J[a][b];
    }
    if (directions) {
      directions[3 * i] = d.x;
      directions[3 * i + 1] = d.y;
      directions[3 * i + 2] = d.z;
    }
    if (origins) {
      origins[3 * i] = o.x;
      origins[3 * i + 1] = o.y;
      origins[3 * i + 2] = o.z;
    }
    if (ok) ok[i] = r ? 1 : 0;
  }
  return 0;
}

int oracle_bspline_eval(int32_t gw, int32_t gh, const double* grid, double x, double y, int slow,
                        double out[3]) {
  (void)gh;
  V3 r = slow ? bspline_surface_slow(grid, gw, x, y) : bspline_surface(grid, gw, x, y);
  out[0] = r.x;
  out[1] = r.y;
  out[2] = r.z;
  return 0;
}

double oracle_huber_cost(double h, double r) {
  const double a = std::fabs(r);
  return a < h ? 0.5 * r * r : h * (a - 0.5 * h);
}
double oracle_huber_weight(double h, double r) {
  const double a = std::fabs(r);
  return a < h ? 1 : h / a;
}
double oracle_huber_cost_sq(double h, double sq) { return huber_cost_sq(h, sq); }
double oracle_huber_weight_sq(double h, double sq) { return huber_weight_sq(h, sq); }

double oracle_time_jacobian(const b200ba_problem* pb, b200ba_state* state,
                            const b200ba_options* opt, int32_t first_imageset, int32_t count,
                            int compute_jacobians) {
  if (!check_options(pb, opt) || !state) return -1;
  const b200ba_problem& P = *pb;
  Layout L = make_layout(P, *opt);
  State S = load_state(P, *state);
  std::vector<double> last_proj(2 * P.n_obs, 0.0);
  if (state->last_projection) std::copy(state->last_projection, state->last_projection + 2 * P.n_obs, last_proj.begin());
  CostFunction cf;
  cf.pb = pb;
  cf.L = L;
  cf.numerical_diff_delta = opt->numerical_diff_delta;
  cf.jacobian_mode = opt->jacobian_mode;
  cf.last_projection = last_proj.data();
  // observation range of the imagesets [first, first + count)
  int64_t ob = P.n_obs, oe = 0;
  for (int64_t o = 0; o < P.n_obs; ++o) {
    const int is = static_cast<int>(P.obs_imageset[o]);
    if (is >= first_imageset && is < first_imageset + count) {
      ob = std::min(ob, o);
      oe = std::max(oe, o + 1);
    }
  }
  if (oe <= ob) return -1;
  cf.obs_begin = ob;
  cf.obs_end = oe;
  std::vector<double> cv;
  cv.reserve(oe - ob);
  Accumulator acc;
  if (compute_jacobians) acc.allocate(L.block_size, L.num_blocks, L.dense_dof());
  acc.cost_vector = &cv;
  acc.huber = opt->huber_parameter;
  const double t0 = now_seconds();
  cf.compute(compute_jacobians != 0, S, &acc);
  const double t = now_seconds() - t0;
  if (state->last_projection) std::copy(last_proj.begin(), last_proj.end(), state->last_projection);
  return t;
}

double oracle_time_contraction(int32_t n_rows, int32_t n_cols) {
  // B^T D^-1 B on a dense random (n_rows x n_cols) B, upper triangle, plus the D^-1 B pass
  // of LV/lm_optimizer.h:1294-1311,1328 (3x3 blocks).
  const int bs = 3;
  if (n_rows % bs) return -1;
  std::vector<double> B(size_t(n_rows) * n_cols), DinvB(size_t(n_rows) * n_cols);
  uint64_t s = 88172645463325252ull;
  for (auto& v : B) {
    s ^= s << 13;
    s ^= s >> 7;
    s ^= s << 17;
    v = double(s % 2001) / 1000.0 - 1.0;
  }
  std::vector<double> S(size_t(n_cols) * n_cols, 0.0);
  const double t0 = now_seconds();
  for (int blk = 0; blk < n_rows / bs; ++blk) {
    const double Hb[3][3] = {{0.5, 0.1, 0.0}, {0.1, 0.4, 0.05}, {0.0, 0.05, 0.6}};
    for (int row = 0; row < bs; ++row)
      for (int col = 0; col < n_cols; ++col) {
        double r = 0;
        for (int k = 0; k < bs; ++k) r += Hb[row][k] * B[size_t(blk * bs + k) * n_cols + col];
        DinvB[size_t(blk * bs + row) * n_cols + col] = r;
      }
  }
  for (int k = 0; k < n_rows; ++k) {
    const double* brow = &B[size_t(k) * n_cols];
    const double* drow = &DinvB[size_t(k) * n_cols];
    for (int i = 0; i < n_cols; ++i) {
      const double bi = brow[i];
      double* srow = &S[size_t(i) * n_cols];
      for (int j = i; j < n_cols; ++j) srow[j] += bi * drow[j];
    }
  }
  const double t = now_seconds() - t0;
  volatile double sink = S[0] + S[S.size() - 1];
  (void)sink;
  return t;
}

double oracle_time_ldlt(int32_t n) {
  std::vector<double> A(size_t(n) * n, 0.0), b(n, 1.0), x(n);
  uint64_t s = 1234567ull;
  for (int i = 0; i < n; ++i)
    for (int j = i; j < n; ++j) {
      s ^= s << 13;
      s ^= s >> 7;
      s ^= s << 17;
      A[size_t(i) * n + j] = (double(s % 2001) / 1000.0 - 1.0) + (i == j ? n : 0);
    }
  const double t0 = now_seconds();
  ldlt_solve(n, A.data(), n, b.data(), 1, 1, x.data(), 1);
  return now_seconds() - t0;
}

// Host threads used by the full-size kernels (compute_mt, ba_dense_fast.h); 1 = the reference's
// single-threaded behaviour. Returns the value in effect.
int oracle_set_threads(int n) {
#ifdef _OPENMP
  if (n <= 0) n = omp_get_num_procs();
  oracle_fast::thread_count() = std::max(1, n);
#else
  (void)n;
  oracle_fast::thread_count() = 1;
#endif
  return oracle_fast::thread_count();
}
// Forces the blocked dense kernels also below kFastDenseMinN (agreement tests).
void oracle_force_fast_dense(int on) { g_force_fast_dense = on != 0; }
// Stand-alone blocked Schur solve (same interface as oracle_schur_solve).
int oracle_schur_solve_fast(int32_t bs, int32_t nb, int32_t nd, const double* D, const double* B,
                            const double* C, const double* b1, const double* b2, double* x) {
  schur_solve_fast(bs, nb, nd, D, B, C, b1, b2, x);
  return 0;
}

}  // extern "C"
