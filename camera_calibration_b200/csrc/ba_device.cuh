// ba_device.cuh -- device-side camera models for the residual / Jacobian kernel.
//
// What is computed follows the reference (paths relative to
// applications/camera_calibration/src/camera_calibration/):
//   models/central_generic.cc:433-549      iterative projection + un-projection Jacobian
//   models/noncentral_generic.cc:156-293   same for the non-central model
//   models/central_opencv.{h,cc}           closed-form 12-parameter model
//   b_spline.h:45-104                      uniform cubic B-spline surface
// How it is computed is written for the GPU: FP64 throughout, one thread per observation,
// basis weights in the numerically better u = t - 3 form, the 16 control points streamed
// row by row (never all 48 doubles live), and the trial evaluation of the projection LM
// also produces the Jacobian so that an accepted step needs no re-evaluation.
#pragma once

#include "ba_common.h"

namespace b200ba {

struct d3 {
  double x, y, z;
};
__device__ __forceinline__ d3 mk3(double x, double y, double z) { return d3{x, y, z}; }
__device__ __forceinline__ d3 operator+(d3 a, d3 b) { return mk3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ d3 operator-(d3 a, d3 b) { return mk3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ d3 operator*(double s, d3 a) { return mk3(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ double dot3(d3 a, d3 b) { return fma(a.x, b.x, fma(a.y, b.y, a.z * b.z)); }
__device__ __forceinline__ d3 cross3(d3 a, d3 b) {
  return mk3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}
__device__ __forceinline__ d3 fma3(double s, d3 a, d3 b) {
  return mk3(fma(s, a.x, b.x), fma(s, a.y, b.y), fma(s, a.z, b.z));
}
__device__ __forceinline__ d3 ld3(const double* __restrict__ p) { return mk3(__ldg(p), __ldg(p + 1), __ldg(p + 2)); }

// Uniform cubic B-spline basis and derivative, u in [0, 1) (b_spline.h:45-63 with t = u + 3).
__device__ __forceinline__ void bspline_basis(double u, double w[4], double dw[4]) {
  const double u2 = u * u, u3 = u2 * u;
  const double omu = 1.0 - u;
  constexpr double k6 = 1.0 / 6.0;
  w[0] = omu * omu * omu * k6;
  w[1] = (3.0 * u3 - 6.0 * u2 + 4.0) * k6;
  w[2] = (-3.0 * u3 + 3.0 * u2 + 3.0 * u + 1.0) * k6;
  w[3] = u3 * k6;
  dw[0] = -0.5 * omu * omu;
  dw[1] = 1.5 * u2 - 2.0 * u;
  dw[2] = -1.5 * u2 + u + 0.5;
  dw[3] = 0.5 * u2;
}

// Position of the 4x4 support of pixel (x, y): top-left control point and fractions, from the single-FMA map
// g = 1 + gmul (x - min). Used by every spline evaluation; the value is continuous across knots, so which of
// two neighbouring cells an ulp picks does not matter there (see locate_support for where it does).
__device__ __forceinline__ void locate(const CamDev& c, double x, double y, int& x0, int& y0, double& fu,
                                       double& fv) {
  const double gx = fma(c.gmul_x, x - c.min_x, 1.0);
  const double gy = fma(c.gmul_y, y - c.min_y, 1.0);
  const double flx = floor(gx), fly = floor(gy);
  x0 = static_cast<int>(flx) - 1;
  y0 = static_cast<int>(fly) - 1;
  fu = gx - flx;
  fv = gy - fly;
}

// One axis of locate_support(): pixel coordinate x of an axis with g control points over [mn, mx + 1) -> first
// control point i0 of the 4-wide support and the fraction u. The FMA map is within a few ulps of the reference's
// 1.f + (g - 3.f) (x - mn) / aw (central_grid.h:150-154), but next to a knot those ulps can move the floor to the
// neighbouring cell. There (|g - round(g)| < 1e-9, which no interior pixel meets by chance) the reference's own
// operations are redone without contraction, including the rounding of g + 2 before its (int)
// (b_spline.h:65-75). At x = max + 1 - ulp the reference's g + 2 can round up to the grid size itself and pick
// the cell g - 3, whose last column lies past the grid (weight 0); the support is kept at g - 4 with u = 1, the
// same value.
__device__ __forceinline__ void locate_axis(double gmul, double x, int mn, int mx, int g, int& i0, double& u) {
  const double d = x - mn;
  double gx = fma(gmul, d, 1.0);
  double fl = floor(gx);
  if (fabs(gx - rint(gx)) < 1e-9) {
    const double t = __dadd_rn(__dadd_rn(1.0, __ddiv_rn(__dmul_rn(static_cast<double>(g - 3), d),
                                                         static_cast<double>(mx + 1 - mn))), 2.0);
    fl = floor(t) - 2.0;  // exact, like t - 2.0 (t >= 3)
    gx = t - 2.0;
    if (fl > g - 3) {
      fl = g - 3;
      gx = fl + 1.0;
    }
  }
  i0 = static_cast<int>(fl) - 1;
  u = gx - fl;
}

// The support an observation's intrinsics Jacobian is attached to (its cell and the control points of its
// columns): the reference's, also at a knot.
__device__ __forceinline__ void locate_support(const CamDev& c, double x, double y, int& x0, int& y0, double& fu,
                                               double& fv) {
  locate_axis(c.gmul_x, x, c.min_x, c.max_x, c.gw, x0, fu);
  locate_axis(c.gmul_y, y, c.min_y, c.max_y, c.gh, y0, fv);
}

__device__ __forceinline__ bool in_area(const CamDev& c, double x, double y) {
  return x >= c.min_x && y >= c.min_y && x < c.max_x + 1 && y < c.max_y + 1;
}

// select element r of a 4-vector held in registers (no local-memory indexing)
__device__ __forceinline__ double sel4(const double w[4], int r) {
  return r == 0 ? w[0] : (r == 1 ? w[1] : (r == 2 ? w[2] : w[3]));
}

// value, d/dgx, d/dgy of a 3-vector spline surface. The 16 control points are streamed row by
// row; the row loop is deliberately NOT unrolled: 12 loads in flight per thread are enough at 16
// resident warps per SM, and hoisting all 48 loads costs ~100 registers (measured: 254 -> 128).
__device__ __forceinline__ void spline3(const double* __restrict__ g, int gw, int x0, int y0, const double wx[4],
                                        const double dwx[4], const double wy[4], const double dwy[4], d3& v,
                                        d3& vx, d3& vy) {
  v = vx = vy = mk3(0, 0, 0);
  const double* row = g + 3 * (static_cast<int64_t>(y0) * gw + x0);
#pragma unroll 1
  for (int r = 0; r < 4; ++r) {
    d3 a = mk3(0, 0, 0), ax = mk3(0, 0, 0);
#pragma unroll
    for (int cidx = 0; cidx < 4; ++cidx) {
      const d3 p = ld3(row + 3 * cidx);
      a = fma3(wx[cidx], p, a);
      ax = fma3(dwx[cidx], p, ax);
    }
    const double wyr = sel4(wy, r), dwyr = sel4(dwy, r);
    v = fma3(wyr, a, v);
    vx = fma3(wyr, ax, vx);
    vy = fma3(dwyr, a, vy);
    row += 3 * static_cast<int64_t>(gw);
  }
}

// ---- central-generic ----------------------------------------------------------------
struct CentralEval {
  d3 u, ux, uy;  // unit direction and its derivative wrt. the PIXEL (scale factors applied)
  double inv_n;  // 1 / |sum w G|
};
// CentralGenericModel::UnprojectWithJacobian (central_generic.cc:521-549)
__device__ __forceinline__ void central_eval(const CamDev& c, const double* __restrict__ grid, double x, double y,
                                             CentralEval& e) {
  int x0, y0;
  double fu, fv;
  locate(c, x, y, x0, y0, fu, fv);
  double wx[4], dwx[4], wy[4], dwy[4];
  bspline_basis(fu, wx, dwx);
  bspline_basis(fv, wy, dwy);
  d3 v, vx, vy;
  spline3(grid, c.gw, x0, y0, wx, dwx, wy, dwy, v, vx, vy);
  const double inv = rsqrt(dot3(v, v));  // <= 1 ulp in double (CUDA math API)
  e.inv_n = inv;
  e.u = inv * v;
  e.ux = (c.sx * inv) * (vx - dot3(e.u, vx) * e.u);
  e.uy = (c.sy * inv) * (vy - dot3(e.u, vy) * e.u);
}

// The 2-parameter LM of the projection (central_generic.cc:433-519): eps 1e-12 on the
// squared residual, <= 100 outer iterations, lambda0 = 0.01 * 0.5 * tr(H) once, <= 10
// attempts (x2 / x0.5), trial clamped to [min, max + 0.999], success as soon as the cost
// measured before a step is < eps. On return e is the evaluation at the final pixel.
//
// Written as ONE loop over spline evaluations (a single inlined call site): the reference
// evaluates "value + Jacobian at the current pixel" and "value at the trial pixel" separately;
// here every evaluation yields both, so the evaluation of an accepted trial IS the next
// iteration's current evaluation. Control flow and results are those of the reference.
// Return value: kProjFail / kProjOk as the reference's bool; kProjUnfinished when the evaluation
// budget max_evals ran out first (the caller then defers the observation to the straggler pass,
// which redoes it with an unlimited budget -- results are those of an uninterrupted run).
constexpr int kProjFail = 0, kProjOk = 1, kProjUnfinished = 2;
__device__ __forceinline__ int central_project(const CamDev& c, const double* __restrict__ grid, d3 dir,
                                               double& px, double& py, CentralEval& e, int& n_eval,
                                               int max_evals) {
  constexpr double kEpsilon = 1e-12;
  double tx = px, ty = py;
  double lambda = -1.0, cost = 0, H00 = 0, H01 = 0, H11 = 0, b0 = 0, b1 = 0;
  bool have_cur = false;
  int outer = 0, attempt = 0;
  const double lo_x = c.min_x, lo_y = c.min_y, hi_x = c.max_x + 0.999, hi_y = c.max_y + 0.999;
  while (true) {
    if (n_eval >= max_evals) return kProjUnfinished;
    CentralEval t;
    central_eval(c, grid, tx, ty, t);
    ++n_eval;
    const d3 r = t.u - dir;
    const double tcost = dot3(r, r);
    if (!have_cur || tcost < cost) {
      // first evaluation, or an accepted trial step
      px = tx;
      py = ty;
      e = t;
      if (have_cur) {
        lambda *= 0.5;
        if (cost < kEpsilon) return kProjOk;  // cost measured BEFORE the step
        if (outer >= 100) return kProjFail;
      }
      have_cur = true;
      ++outer;
      attempt = 0;
      cost = tcost;
      H00 = dot3(t.ux, t.ux);
      H01 = dot3(t.ux, t.uy);
      H11 = dot3(t.uy, t.uy);
      b0 = dot3(r, t.ux);
      b1 = dot3(r, t.uy);
      if (lambda < 0) lambda = 0.01 * 0.5 * (H00 + H11);
    } else {
      lambda *= 2.0;
      if (++attempt >= 10) return (cost < kEpsilon) ? kProjOk : kProjFail;
    }
    const double H00l = H00 + lambda, H11l = H11 + lambda;
    const double x1 = (b1 - H01 / H00l * b0) / (H11l - H01 * H01 / H00l);
    const double x0 = (b0 - H01 * x1) / H00l;
    tx = fmax(lo_x, fmin(hi_x, px - x0));
    ty = fmax(lo_y, fmin(hi_y, py - x1));
  }
}

// ---- tangent frames (local_parametrizations/line_parametrization.h:54-60) -----------------
__device__ __forceinline__ bool tangent_uses_ey(d3 d) { return fabs(d.x) > static_cast<double>(0.9f); }
__device__ __forceinline__ void compute_tangents(d3 d, d3& t1, d3& t2) {
  d3 c = tangent_uses_ey(d) ? mk3(-d.z, 0.0, d.x) : mk3(0.0, d.z, -d.y);
  const double n = sqrt(dot3(c, c));
  t1 = mk3(c.x / n, c.y / n, c.z / n);
  t2 = cross3(d, t1);
}
// (o - p)^T d t1 / d dir and (o - p)^T d t2 / d dir: rows of d r / d direction of the
// non-central projection residual (line_parametrization.h:62-105 contracted with o - p).
__device__ __forceinline__ void tangent_rows(d3 d, d3 q, d3& r1, d3& r2) {
  if (tangent_uses_ey(d)) {
    const double n2 = d.x * d.x + d.z * d.z;
    const double in = 1.0 / sqrt(n2);
    const double in3 = in * in * in;
    // T1 rows: [dx dz, 0, -dx^2] in3 ; 0 ; [dz^2, 0, -dx dz] in3
    r1 = mk3((q.x * d.x * d.z + q.z * d.z * d.z) * in3, 0.0, (-q.x * d.x * d.x - q.z * d.x * d.z) * in3);
    // T2 rows: [dy dz^2 in3, dx in, -dx dy dz in3] ; [-dx in, 0, -dz in] ; [-dx dy dz in3, dz in, dy dx^2 in3]
    r2 = mk3(q.x * d.y * d.z * d.z * in3 - q.y * d.x * in - q.z * d.x * d.y * d.z * in3,
             q.x * d.x * in + q.z * d.z * in,
             -q.x * d.x * d.y * d.z * in3 - q.y * d.z * in + q.z * d.y * d.x * d.x * in3);
  } else {
    const double n2 = d.y * d.y + d.z * d.z;
    const double in = 1.0 / sqrt(n2);
    const double in3 = in * in * in;
    // T1 rows: 0 ; [0, -dy dz, dy^2] in3 ; [0, -dz^2, dy dz] in3
    r1 = mk3(0.0, (-q.y * d.y * d.z - q.z * d.z * d.z) * in3, (q.y * d.y * d.y + q.z * d.y * d.z) * in3);
    // T2 rows: [0, -dy in, -dz in] ; [dy in, dx dz^2 in3, -dx dy dz in3] ; [dz in, -dx dy dz in3, dx dy^2 in3]
    r2 = mk3(q.y * d.y * in + q.z * d.z * in,
             -q.x * d.y * in + q.y * d.x * d.z * d.z * in3 - q.z * d.x * d.y * d.z * in3,
             -q.x * d.z * in - q.y * d.x * d.y * d.z * in3 + q.z * d.x * d.y * d.y * in3);
  }
}

// ---- noncentral-generic -------------------------------------------------------------------
struct NoncentralEval {
  d3 o, ox, oy;  // line origin and derivative wrt. pixel
  d3 u, ux, uy;  // unit line direction and derivative wrt. pixel
  double inv_n;
};
// NoncentralGenericModel::UnprojectWithJacobian (noncentral_generic.cc:266-293)
__device__ __forceinline__ void noncentral_eval(const CamDev& c, const double* __restrict__ dgrid,
                                                const double* __restrict__ pgrid, double x, double y,
                                                NoncentralEval& e) {
  int x0, y0;
  double fu, fv;
  locate(c, x, y, x0, y0, fu, fv);
  double wx[4], dwx[4], wy[4], dwy[4];
  bspline_basis(fu, wx, dwx);
  bspline_basis(fv, wy, dwy);
  d3 v, vx, vy;
  spline3(dgrid, c.gw, x0, y0, wx, dwx, wy, dwy, v, vx, vy);
  const double inv = rsqrt(dot3(v, v));
  e.inv_n = inv;
  e.u = inv * v;
  e.ux = (c.sx * inv) * (vx - dot3(e.u, vx) * e.u);
  e.uy = (c.sy * inv) * (vy - dot3(e.u, vy) * e.u);
  d3 o, ox, oy;
  spline3(pgrid, c.gw, x0, y0, wx, dwx, wy, dwy, o, ox, oy);
  e.o = o;
  e.ox = c.sx * ox;
  e.oy = c.sy * oy;
}
// Value-only B-spline weights and 3-vector surface value (the w / v parts of bspline_basis / spline3), for passes
// that need no pixel derivatives.
__device__ __forceinline__ void bspline_weights(double u, double w[4]) {
  const double u2 = u * u, u3 = u2 * u;
  const double omu = 1.0 - u;
  constexpr double k6 = 1.0 / 6.0;
  w[0] = omu * omu * omu * k6;
  w[1] = (3.0 * u3 - 6.0 * u2 + 4.0) * k6;
  w[2] = (-3.0 * u3 + 3.0 * u2 + 3.0 * u + 1.0) * k6;
  w[3] = u3 * k6;
}
__device__ __forceinline__ d3 spline3_value(const double* __restrict__ g, int gw, int x0, int y0, const double wx[4],
                                            const double wy[4]) {
  d3 v = mk3(0, 0, 0);
  const double* row = g + 3 * (static_cast<int64_t>(y0) * gw + x0);
#pragma unroll 1
  for (int r = 0; r < 4; ++r) {
    d3 a = mk3(0, 0, 0);
#pragma unroll
    for (int cidx = 0; cidx < 4; ++cidx) a = fma3(wx[cidx], ld3(row + 3 * cidx), a);
    v = fma3(sel4(wy, r), a, v);
    row += 3 * static_cast<int64_t>(gw);
  }
  return v;
}
// NoncentralGenericModel::UnprojectFromGrid (noncentral_generic.h:100-105) at pixel (x, y), value only: origin o and
// the direction normalised as Eigen's normalize() does, d = v / sqrt(|v|^2) (|v|^2 without FMA; v unchanged if 0).
__device__ __forceinline__ void noncentral_line(const CamDev& c, const double* __restrict__ dgrid,
                                                const double* __restrict__ pgrid, double x, double y, d3& o, d3& d) {
  int x0, y0;
  double fu, fv;
  locate(c, x, y, x0, y0, fu, fv);
  double wx[4], wy[4];
  bspline_weights(fu, wx);
  bspline_weights(fv, wy);
  const d3 v = spline3_value(dgrid, c.gw, x0, y0, wx, wy);
  o = spline3_value(pgrid, c.gw, x0, y0, wx, wy);
  const double n2 = __dadd_rn(__dadd_rn(__dmul_rn(v.x, v.x), __dmul_rn(v.y, v.y)), __dmul_rn(v.z, v.z));
  if (n2 > 0) {
    const double n = sqrt(n2);
    d = mk3(v.x / n, v.y / n, v.z / n);
  } else {
    d = v;
  }
}
// residual r = (t1 . (o - p), t2 . (o - p)) (noncentral_generic.cc:166-172)
__device__ __forceinline__ void noncentral_residual(const NoncentralEval& e, d3 p, double& r0, double& r1,
                                                    d3& t1, d3& t2) {
  compute_tangents(e.u, t1, t2);
  const d3 q = e.o - p;
  r0 = dot3(t1, q);
  r1 = dot3(t2, q);
}
// 2x2 Jacobian of the residual wrt. the pixel (noncentral_generic.cc:174-193)
__device__ __forceinline__ void noncentral_residual_jac(const NoncentralEval& e, d3 p, d3 t1, d3 t2,
                                                        double R[2][2]) {
  const d3 q = e.o - p;
  d3 rd1, rd2;
  tangent_rows(e.u, q, rd1, rd2);
  R[0][0] = dot3(rd1, e.ux) + dot3(t1, e.ox);
  R[0][1] = dot3(rd1, e.uy) + dot3(t1, e.oy);
  R[1][0] = dot3(rd2, e.ux) + dot3(t2, e.ox);
  R[1][1] = dot3(rd2, e.uy) + dot3(t2, e.oy);
}
// NoncentralGenericModel::ProjectWithInitialEstimate (noncentral_generic.cc:156-264); same
// single-evaluation-site formulation as central_project. On success R is the 2x2 residual
// Jacobian and (t1, t2) the tangent frame at the final pixel (inputs of the implicit-function step).
__device__ __forceinline__ int noncentral_project(const CamDev& c, const double* __restrict__ dgrid,
                                                  const double* __restrict__ pgrid, d3 p, double& px,
                                                  double& py, NoncentralEval& e, d3& t1, d3& t2,
                                                  double R[2][2], int& n_eval, int max_evals) {
  constexpr double kEpsilon = 1e-12;
  double tx = px, ty = py;
  double lambda = -1.0, cost = 0, H00 = 0, H01 = 0, H11 = 0, b0 = 0, b1 = 0;
  bool have_cur = false;
  int outer = 0, attempt = 0;
  const double lo_x = c.min_x, lo_y = c.min_y, hi_x = c.max_x + 0.999, hi_y = c.max_y + 0.999;
  while (true) {
    if (n_eval >= max_evals) return kProjUnfinished;
    NoncentralEval t;
    noncentral_eval(c, dgrid, pgrid, tx, ty, t);
    ++n_eval;
    double r0, r1;
    d3 tt1, tt2;
    noncentral_residual(t, p, r0, r1, tt1, tt2);
    const double tcost = r0 * r0 + r1 * r1;
    if (!have_cur || tcost < cost) {
      px = tx;
      py = ty;
      e = t;
      t1 = tt1;
      t2 = tt2;
      noncentral_residual_jac(t, p, tt1, tt2, R);
      if (have_cur) {
        lambda *= 0.5;
        if (cost < kEpsilon) return kProjOk;
        if (outer >= 100) return kProjFail;
      }
      have_cur = true;
      ++outer;
      attempt = 0;
      cost = tcost;
      H00 = R[0][0] * R[0][0] + R[1][0] * R[1][0];
      H01 = R[0][0] * R[0][1] + R[1][0] * R[1][1];
      H11 = R[0][1] * R[0][1] + R[1][1] * R[1][1];
      b0 = r0 * R[0][0] + r1 * R[1][0];
      b1 = r0 * R[0][1] + r1 * R[1][1];
      if (lambda < 0) lambda = 0.01 * 0.5 * (H00 + H11);
    } else {
      lambda *= 2.0;
      if (++attempt >= 10) return (cost < kEpsilon) ? kProjOk : kProjFail;
    }
    const double H00l = H00 + lambda, H11l = H11 + lambda;
    const double x1 = (b1 - H01 / H00l * b0) / (H11l - H01 * H01 / H00l);
    const double x0 = (b0 - H01 * x1) / H00l;
    tx = fmax(lo_x, fmin(hi_x, px - x0));
    ty = fmax(lo_y, fmin(hi_y, py - x1));
  }
}

// ---- central OpenCV ----------------------------------------------------------------------------
// CentralOpenCVModel::Project (central_opencv.cc:59-99). Every operation is rounded on its own in the
// reference's order (no fused multiply-add): the pixel decides validity at the image border, so it must be the
// reference's to the last bit.
__device__ __forceinline__ bool opencv_project(const CamDev& c, const double* __restrict__ q, d3 lp, double& px,
                                               double& py) {
  if (lp.z <= 0) return false;
  const double nx = __ddiv_rn(lp.x, lp.z), ny = __ddiv_rn(lp.y, lp.z);
  const double x2 = __dmul_rn(nx, nx), xy = __dmul_rn(nx, ny), y2 = __dmul_rn(ny, ny);
  const double r2 = __dadd_rn(x2, y2), r4 = __dmul_rn(r2, r2), r6 = __dmul_rn(r4, r2);
  const double num = __dadd_rn(__dadd_rn(__dadd_rn(1.0, __dmul_rn(q[4], r2)), __dmul_rn(q[5], r4)), __dmul_rn(q[6], r6));
  const double den = __dadd_rn(__dadd_rn(__dadd_rn(1.0, __dmul_rn(q[7], r2)), __dmul_rn(q[8], r4)), __dmul_rn(q[9], r6));
  const double radial = __ddiv_rn(num, den);
  const double dx = __dadd_rn(__dmul_rn(__dmul_rn(2.0, q[10]), xy), __dmul_rn(q[11], __dadd_rn(r2, __dmul_rn(2.0, x2))));
  const double dy = __dadd_rn(__dmul_rn(__dmul_rn(2.0, q[11]), xy), __dmul_rn(q[10], __dadd_rn(r2, __dmul_rn(2.0, y2))));
  px = __dadd_rn(__dmul_rn(q[0], __dadd_rn(__dmul_rn(nx, radial), dx)), q[2]);
  py = __dadd_rn(__dmul_rn(q[1], __dadd_rn(__dmul_rn(ny, radial), dy)), q[3]);
  return px >= 0 && py >= 0 && px < c.width && py < c.height;
}
// d pixel / d local_point (closed form) and d pixel / d (fx fy cx cy k1..k6 p1 p2)
// (central_opencv.h:98-176).
__device__ __forceinline__ void opencv_jacobians(const double* __restrict__ q, d3 lp, double P[2][3],
                                                 double Jx[12], double Jy[12]) {
  const double iz = 1.0 / lp.z;
  const double nx = lp.x * iz, ny = lp.y * iz;
  const double x2 = nx * nx, xy = nx * ny, y2 = ny * ny;
  const double r2 = x2 + y2, r4 = r2 * r2, r6 = r4 * r2;
  const double fx = q[0], fy = q[1];
  const double k1 = q[4], k2 = q[5], k3 = q[6], k4 = q[7], k5 = q[8], k6 = q[9], p1 = q[10], p2 = q[11];
  const double num = 1 + k1 * r2 + k2 * r4 + k3 * r6;
  const double den = 1 + k4 * r2 + k5 * r4 + k6 * r6;
  const double iden = 1.0 / den;
  const double radial = num * iden;
  const double dnum = k1 + 2 * k2 * r2 + 3 * k3 * r4;
  const double dden = k4 + 2 * k5 * r2 + 3 * k6 * r4;
  const double drad = (dnum * den - num * dden) * iden * iden;
  const double dxx = radial + 2 * x2 * drad + 2 * p1 * ny + 6 * p2 * nx;
  const double dxy = 2 * xy * drad + 2 * p1 * nx + 2 * p2 * ny;
  const double dyx = 2 * xy * drad + 2 * p2 * ny + 2 * p1 * nx;
  const double dyy = radial + 2 * y2 * drad + 2 * p2 * nx + 6 * p1 * ny;
  P[0][0] = fx * dxx * iz;
  P[0][1] = fx * dxy * iz;
  P[0][2] = fx * (-dxx * nx - dxy * ny) * iz;
  P[1][0] = fy * dyx * iz;
  P[1][1] = fy * dyy * iz;
  P[1][2] = fy * (-dyx * nx - dyy * ny) * iz;
  const double nni = num * iden * iden;
  Jx[0] = nx * radial + 2 * p1 * xy + p2 * (r2 + 2 * x2);
  Jx[1] = 0;
  Jx[2] = 1;
  Jx[3] = 0;
  Jx[4] = fx * nx * r2 * iden;
  Jx[5] = fx * nx * r4 * iden;
  Jx[6] = fx * nx * r6 * iden;
  Jx[7] = -fx * nx * nni * r2;
  Jx[8] = -fx * nx * nni * r4;
  Jx[9] = -fx * nx * nni * r6;
  Jx[10] = fx * 2 * xy;
  Jx[11] = fx * (r2 + 2 * x2);
  Jy[0] = 0;
  Jy[1] = ny * radial + p1 * (r2 + 2 * y2) + 2 * p2 * xy;
  Jy[2] = 0;
  Jy[3] = 1;
  Jy[4] = fy * ny * r2 * iden;
  Jy[5] = fy * ny * r4 * iden;
  Jy[6] = fy * ny * r6 * iden;
  Jy[7] = -fy * ny * nni * r2;
  Jy[8] = -fy * ny * nni * r4;
  Jy[9] = -fy * ny * nni * r6;
  Jy[10] = fy * (r2 + 2 * y2);
  Jy[11] = fy * 2 * xy;
}
// The distortion of normalised coordinates n -> (n radial + tangential) and its 2x2 derivative: the dxx, dxy, dyx,
// dyy of opencv_jacobians, i.e. CentralOpenCVModel::ProjectInnerPartWithJacobian (central_opencv.cc:101-148) with
// the derivative of the value it returns. (The reference's closed form of that Jacobian is not the derivative of its
// value; the un-projection below only uses it as a search direction, and its accept / stop rules are the reference's.)
__device__ __forceinline__ void opencv_distort(const double* __restrict__ q, double nx, double ny, double& ux,
                                               double& uy, double J[2][2]) {
  const double x2 = nx * nx, xy = nx * ny, y2 = ny * ny;
  const double r2 = x2 + y2, r4 = r2 * r2, r6 = r4 * r2;
  const double k1 = q[4], k2 = q[5], k3 = q[6], k4 = q[7], k5 = q[8], k6 = q[9], p1 = q[10], p2 = q[11];
  const double num = 1 + k1 * r2 + k2 * r4 + k3 * r6;
  const double den = 1 + k4 * r2 + k5 * r4 + k6 * r6;
  const double iden = 1.0 / den;
  const double radial = num * iden;
  const double dnum = k1 + 2 * k2 * r2 + 3 * k3 * r4;
  const double dden = k4 + 2 * k5 * r2 + 3 * k6 * r4;
  const double drad = (dnum * den - num * dden) * iden * iden;
  ux = nx * radial + (2.0 * p1 * xy + p2 * (r2 + 2.0 * x2));
  uy = ny * radial + (2.0 * p2 * xy + p1 * (r2 + 2.0 * y2));
  J[0][0] = radial + 2 * x2 * drad + 2 * p1 * ny + 6 * p2 * nx;
  J[0][1] = 2 * xy * drad + 2 * p1 * nx + 2 * p2 * ny;
  J[1][0] = 2 * xy * drad + 2 * p2 * ny + 2 * p1 * nx;
  J[1][1] = radial + 2 * y2 * drad + 2 * p2 * nx + 6 * p1 * ny;
}
// CentralOpenCVModel::Unproject (central_opencv.cc:150-156): UnprojectWithGaussNewton (parametric.h:60-148) from the
// normalised pixel, at most 100 iterations of up to 5 attempts (lambda_0 = 1.0 * 0.5 tr(H) at the first iteration,
// x0.1 on an accepted attempt, x10 on a rejected one), stopping after an iteration that ends with cost < 1e-10f or
// accepts nothing; then d = (x, y, 1) normalised. Returns false where the reference returns false.
__device__ __forceinline__ bool opencv_unproject(const double* __restrict__ q, double x, double y, d3& d) {
  const double dpx = (x - q[2]) / q[0], dpy = (y - q[3]) / q[1];
  double cx = dpx, cy = dpy;
  constexpr double kEpsilon = static_cast<double>(1e-10f);
  double lambda = -1;
  bool converged = false;
  for (int i = 0; i < 100; ++i) {
    double ux, uy, J[2][2];
    opencv_distort(q, cx, cy, ux, uy, J);
    double dx = ux - dpx, dy = uy - dpy;
    double cost = dx * dx + dy * dy;
    const double H00 = J[0][0] * J[0][0] + J[1][0] * J[1][0];
    const double H01 = J[0][0] * J[0][1] + J[1][0] * J[1][1];
    const double H11 = J[0][1] * J[0][1] + J[1][1] * J[1][1];
    const double b0 = dx * J[0][0] + dy * J[1][0];
    const double b1 = dx * J[0][1] + dy * J[1][1];
    if (lambda < 0) lambda = 1.0 * (0.5 * (H00 + H11));
    bool update_found = false;
    for (int attempt = 0; attempt < 5; ++attempt) {
      const double H00l = H00 + lambda, H11l = H11 + lambda;
      const double x1 = (b1 - H01 / H00l * b0) / (H11l - H01 * H01 / H00l);
      const double x0 = (b0 - H01 * x1) / H00l;
      const double tx = cx - x0, ty = cy - x1;
      double tux, tuy, TJ[2][2];
      opencv_distort(q, tx, ty, tux, tuy, TJ);
      dx = tux - dpx;
      dy = tuy - dpy;
      const double test_cost = dx * dx + dy * dy;
      if (test_cost < cost) {
        cost = test_cost;
        cx = tx;
        cy = ty;
        lambda *= 0.1;
        update_found = true;
        break;
      }
      lambda *= 10;
    }
    if (cost < kEpsilon) {
      converged = true;
      break;
    }
    if (!update_found) break;
  }
  if (!converged) return false;
  const double n = sqrt(cx * cx + cy * cy + 1.0);
  d = mk3(cx / n, cy / n, 1.0 / n);
  return true;
}

// ---- Huber (libvis loss_functions.h:94-133) ------------------------------------------------------
__device__ __forceinline__ double huber_cost_sq(double h, double sq) {
  return (sq < h * h) ? 0.5 * sq : h * (sqrt(sq) - 0.5 * h);
}
__device__ __forceinline__ double huber_weight_sq(double h, double sq) { return (sq < h * h) ? 1.0 : h / sqrt(sq); }

// ---- quaternions (w, x, y, z) --------------------------------------------------------------------
struct q4 {
  double w, x, y, z;
};
__device__ __forceinline__ q4 qmul(q4 a, q4 b) {
  q4 r;
  r.w = a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z;
  r.x = a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y;
  r.y = a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z;
  r.z = a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x;
  return r;
}
__device__ __forceinline__ void qrot(q4 q, double R[9]) {
  const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z;
  const double twx = tx * q.w, twy = ty * q.w, twz = tz * q.w;
  const double txx = tx * q.x, txy = ty * q.x, txz = tz * q.x;
  const double tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
  R[0] = 1 - (tyy + tzz);
  R[1] = txy - twz;
  R[2] = txz + twy;
  R[3] = txy + twz;
  R[4] = 1 - (txx + tzz);
  R[5] = tyz - twx;
  R[6] = txz - twy;
  R[7] = tyz + twx;
  R[8] = 1 - (txx + tyy);
}
__device__ __forceinline__ d3 rot_apply(const double R[9], d3 p) {
  return mk3(R[0] * p.x + R[1] * p.y + R[2] * p.z, R[3] * p.x + R[4] * p.y + R[5] * p.z,
             R[6] * p.x + R[7] * p.y + R[8] * p.z);
}

// ---- libvis RadtanCamera8d (libvis/camera.h: RadtanDistortion4 :500-591, PixelMapping4 :1011-1121) ---------------
// p = k1 k2 r1 r2 fx fy cx cy. UnprojectFromPixelCornerConv(x, y): n = (fx_inv x + cx_inv, fy_inv y + cy_inv) with
// fx_inv = 1 / fx, cx_inv = -cx / fx; then at most 5 Gauss-Newton steps from u = n: e = n - D(u),
// u += (J^T J)^-1 J^T e with Eigen's closed-form 2 x 2 inverse (1 / det times the adjugate) and the products taken left
// to right, stopping after the step whose e has |e|^2 < DBL_EPSILON. Returns (u.x, u.y), the direction being (u, 1).
// Every operation is rounded on its own (no fused multiply-add) in the reference's order, so that a restatement in
// double reproduces every bit; where the iteration diverges the values are whatever IEEE arithmetic gives (NaN, inf).
__device__ __forceinline__ void radtan8_unproject(const double* __restrict__ p, double x, double y, double& ux,
                                                  double& uy) {
  const double k1 = p[0], k2 = p[1], r1 = p[2], r2 = p[3];
  const double nx = __dadd_rn(__dmul_rn(__ddiv_rn(1.0, p[4]), x), __ddiv_rn(-p[6], p[4]));
  const double ny = __dadd_rn(__dmul_rn(__ddiv_rn(1.0, p[5]), y), __ddiv_rn(-p[7], p[5]));
  const double k1_2 = __dmul_rn(k1, 2.0), k2_4 = __dmul_rn(k2, 4.0);
  const double r1_2 = __dmul_rn(2.0, r1), r2_2 = __dmul_rn(2.0, r2), r1_6 = __dmul_rn(6.0, r1), r2_6 = __dmul_rn(6.0, r2);
  ux = nx;
  uy = ny;
  for (int i = 0; i < 5; ++i) {
    const double mx2 = __dmul_rn(ux, ux), my2 = __dmul_rn(uy, uy), mxy = __dmul_rn(ux, uy);
    const double rho2 = __dadd_rn(mx2, my2);
    const double k2rho2 = __dmul_rn(k2, rho2);
    const double rad = __dadd_rn(__dmul_rn(k1, rho2), __dmul_rn(k2rho2, rho2));
    const double one_rad = __dadd_rn(1.0, rad);
    const double k2rho2_4 = __dmul_rn(k2rho2, 4.0);
    const double j00 = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(one_rad, __dmul_rn(k1_2, mx2)), __dmul_rn(k2rho2_4, mx2)),
                                           __dmul_rn(r1_2, uy)),
                                 __dmul_rn(r2_6, ux));
    const double j10 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(k1_2, mxy), __dmul_rn(__dmul_rn(k2_4, rho2), mxy)),
                                           __dmul_rn(r1_2, ux)),
                                 __dmul_rn(r2_2, uy));
    const double j11 = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(one_rad, __dmul_rn(k1_2, my2)), __dmul_rn(k2rho2_4, my2)),
                                           __dmul_rn(r1_6, uy)),
                                 __dmul_rn(r2_2, ux));
    const double dx = __dadd_rn(__dadd_rn(__dadd_rn(ux, __dmul_rn(ux, rad)), __dmul_rn(r1_2, mxy)),
                                __dmul_rn(r2, __dadd_rn(rho2, __dmul_rn(2.0, mx2))));
    const double dy = __dadd_rn(__dadd_rn(__dadd_rn(uy, __dmul_rn(uy, rad)), __dmul_rn(r2_2, mxy)),
                                __dmul_rn(r1, __dadd_rn(rho2, __dmul_rn(2.0, my2))));
    const double ex = __dsub_rn(nx, dx), ey = __dsub_rn(ny, dy);
    // A = J^T J (J symmetric: J(0,1) = J(1,0) = j10)
    const double a00 = __dadd_rn(__dmul_rn(j00, j00), __dmul_rn(j10, j10));
    const double a01 = __dadd_rn(__dmul_rn(j00, j10), __dmul_rn(j10, j11));
    const double a10 = __dadd_rn(__dmul_rn(j10, j00), __dmul_rn(j11, j10));
    const double a11 = __dadd_rn(__dmul_rn(j10, j10), __dmul_rn(j11, j11));
    const double invdet = __ddiv_rn(1.0, __dsub_rn(__dmul_rn(a00, a11), __dmul_rn(a10, a01)));
    const double i00 = __dmul_rn(a11, invdet), i10 = __dmul_rn(-a10, invdet);
    const double i01 = __dmul_rn(-a01, invdet), i11 = __dmul_rn(a00, invdet);
    // M = A^-1 J^T, then M e
    const double m00 = __dadd_rn(__dmul_rn(i00, j00), __dmul_rn(i01, j10));
    const double m01 = __dadd_rn(__dmul_rn(i00, j10), __dmul_rn(i01, j11));
    const double m10 = __dadd_rn(__dmul_rn(i10, j00), __dmul_rn(i11, j10));
    const double m11 = __dadd_rn(__dmul_rn(i10, j10), __dmul_rn(i11, j11));
    ux = __dadd_rn(ux, __dadd_rn(__dmul_rn(m00, ex), __dmul_rn(m01, ey)));
    uy = __dadd_rn(uy, __dadd_rn(__dmul_rn(m10, ex), __dmul_rn(m11, ey)));
    if (__dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)) < 2.220446049250313080847e-16) break;
  }
}

}  // namespace b200ba
