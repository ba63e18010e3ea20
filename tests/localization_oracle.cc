// Sequential IEEE-double restatement of the pose fit of b200ba_localization_accuracy (include/b200ba.h): opengv's
// absolute_pose::optimize_nonlinear cost F = sum_i (1 - f_i' u_i)^2, u_i = normalize(R(c)' (p_i - t)), minimised by
// the same damped Newton iteration as the device (same H, gradient, lambda rules and stopping rules), with every sum
// taken point by point in order. Test infrastructure only: tests/test_localization_accuracy.py and
// scripts/localization_timing.py compile it with -ffp-contract=off and load it with ctypes.
#include <cmath>
#include <cstdint>

namespace {

struct V3 {
  double x, y, z;
};
V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
V3 operator*(double s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
double dot(V3 a, V3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
V3 unit(V3 v) {
  const double n = std::sqrt(dot(v, v));
  return {v.x / n, v.y / n, v.z / n};
}

constexpr int kSums = 28;  // F, grad F (6), H (21, lower triangle row by row)
int hidx(int i, int j) { return 7 + i * (i + 1) / 2 + j; }

// e = u - f and, with du != nullptr, du/d(t, c) (3 x 6, row-major)
void residual(const double* x, V3 p, V3 f, V3* e, double (*du)[6]) {
  const V3 v = {p.x - x[0], p.y - x[1], p.z - x[2]};
  const V3 c = {x[3], x[4], x[5]};
  const double cc = dot(c, c), cv = dot(c, v), inv_s = 1.0 / (1.0 + cc), one_m = 1.0 - cc;
  const V3 cxv = cross(c, v);
  const V3 q = inv_s * V3{one_m * v.x + 2.0 * cv * c.x - 2.0 * cxv.x, one_m * v.y + 2.0 * cv * c.y - 2.0 * cxv.y,
                          one_m * v.z + 2.0 * cv * c.z - 2.0 * cxv.z};
  const double nq = std::sqrt(dot(q, q));
  const V3 u = {q.x / nq, q.y / nq, q.z / nq};
  *e = u - f;
  if (!du) return;
  const double cs[3] = {c.x, c.y, c.z}, vs[3] = {v.x, v.y, v.z}, qs[3] = {q.x, q.y, q.z};
  const double inv_n = 1.0 / nq;
  for (int b = 0; b < 3; ++b) {
    // column b of R' (without 1 / s) and of (1 + c'c) dq/dc
    V3 rt = {2.0 * c.x * cs[b], 2.0 * c.y * cs[b], 2.0 * c.z * cs[b]};
    V3 m = {2.0 * (c.x * vs[b] - v.x * cs[b] - qs[0] * cs[b]), 2.0 * (c.y * vs[b] - v.y * cs[b] - qs[1] * cs[b]),
            2.0 * (c.z * vs[b] - v.z * cs[b] - qs[2] * cs[b])};
    if (b == 0) {
      rt = {rt.x + one_m, rt.y - 2.0 * c.z, rt.z + 2.0 * c.y};
      m = {m.x + 2.0 * cv, m.y + 2.0 * v.z, m.z - 2.0 * v.y};
    } else if (b == 1) {
      rt = {rt.x + 2.0 * c.z, rt.y + one_m, rt.z - 2.0 * c.x};
      m = {m.x - 2.0 * v.z, m.y + 2.0 * cv, m.z + 2.0 * v.x};
    } else {
      rt = {rt.x - 2.0 * c.y, rt.y + 2.0 * c.x, rt.z + one_m};
      m = {m.x + 2.0 * v.y, m.y - 2.0 * v.x, m.z + 2.0 * cv};
    }
    const V3 at = (-inv_s) * rt, ac = inv_s * m;
    const V3 jt = inv_n * (at - dot(u, at) * u), jc = inv_n * (ac - dot(u, ac) * u);
    du[0][b] = jt.x;
    du[1][b] = jt.y;
    du[2][b] = jt.z;
    du[0][3 + b] = jc.x;
    du[1][3 + b] = jc.y;
    du[2][3 + b] = jc.z;
  }
}

double cost_term(V3 e) {
  const double r = 0.5 * dot(e, e);
  return r * r;
}

V3 point(const double* a, int i) { return {a[3 * i], a[3 * i + 1], a[3 * i + 2]}; }

// the points in order 0 .. n-1, or n-1 .. 0 with `reverse`
double cost(int n, const double* p, const double* f, const double* x, bool reverse) {
  double F = 0;
  for (int k = 0; k < n; ++k) {
    const int i = reverse ? n - 1 - k : k;
    V3 e;
    residual(x, point(p, i), point(f, i), &e, nullptr);
    F += cost_term(e);
  }
  return F;
}

void system(int n, const double* p, const double* f, const double* x, bool reverse, double* sys) {
  for (int k = 0; k < kSums; ++k) sys[k] = 0;
  for (int k = 0; k < n; ++k) {
    const int pi = reverse ? n - 1 - k : k;
    V3 e;
    double du[3][6];
    residual(x, point(p, pi), point(f, pi), &e, du);
    sys[0] += cost_term(e);
    const double w = dot(e, e);
    double a[6];
    for (int j = 0; j < 6; ++j) {
      a[j] = (du[0][j] * e.x + du[1][j] * e.y) + du[2][j] * e.z;
      sys[1 + j] += w * a[j];
    }
    for (int i = 0; i < 6; ++i)
      for (int j = 0; j <= i; ++j)
        sys[hidx(i, j)] += w * ((du[0][i] * du[0][j] + du[1][i] * du[1][j]) + du[2][i] * du[2][j]) + 2.0 * a[i] * a[j];
  }
}

bool solve(const double* sys, double lambda, double* d) {
  double L[6][6] = {};
  bool ok = true;
  for (int i = 0; i < 6; ++i)
    for (int j = 0; j <= i; ++j) {
      double a = sys[hidx(i, j)] + (i == j ? lambda : 0.0);
      for (int k = 0; k < j; ++k) a -= L[i][k] * L[j][k];
      if (i == j) {
        ok = ok && a > 0;
        L[i][i] = std::sqrt(a);
      } else {
        L[i][j] = a / L[j][j];
      }
    }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double a = -sys[1 + i];
    for (int k = 0; k < i; ++k) a -= L[i][k] * y[k];
    y[i] = a / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double a = y[i];
    for (int k = i + 1; k < 6; ++k) a -= L[k][i] * d[k];
    d[i] = a / L[i][i];
  }
  return ok;
}

int fit(int n, const double* p, const double* f, bool reverse, double* x, double* cost_out, int32_t* iterations_out) {
  for (int k = 0; k < 6; ++k) x[k] = 0;
  double lambda = 0, F = 0;
  int iterations = 0;
  for (int it = 0; it < 100; ++it) {
    double sys[kSums];
    system(n, p, f, x, reverse, sys);
    F = sys[0];
    if (F == 0) break;
    if (it == 0) {
      double trace = 0;
      for (int i = 0; i < 6; ++i) trace += sys[hidx(i, i)];
      lambda = static_cast<double>(0.001f) * trace / 6;
    }
    bool applied = false;
    for (int attempt = 0; attempt < 10; ++attempt) {
      double d[6], xt[6];
      if (!solve(sys, lambda, d)) {
        lambda = 2.0 * lambda;
        continue;
      }
      for (int k = 0; k < 6; ++k) xt[k] = x[k] + d[k];
      const double test_cost = cost(n, p, f, xt, reverse);
      if (test_cost < F) {
        for (int k = 0; k < 6; ++k) x[k] = xt[k];
        lambda = 0.5 * lambda;
        applied = true;
        ++iterations;
        F = test_cost;
        break;
      }
      lambda = 2.0 * lambda;
    }
    if (!applied || F == 0) break;
  }
  if (cost_out) *cost_out = F;
  if (iterations_out) *iterations_out = iterations;
  return 0;
}

}  // namespace

extern "C" {

// One pose fit from x = 0: p, f [n][3]; x_out [6] (t, c); the final cost and the accepted steps.
int oracle_localization_fit(int n, const double* p, const double* f, double* x_out, double* cost_out,
                            int32_t* iterations_out) {
  return fit(n, p, f, false, x_out, cost_out, iterations_out);
}

// `trials` fits of 15 points each (p, f [trials][15][3]); the points summed in reverse order with `reverse`
// (to measure how much the result depends on the order of the sums).
int oracle_localization_fit_batch(int64_t trials, const double* p, const double* f, int reverse, double* x_out,
                                  double* cost_out, int32_t* iterations_out) {
  for (int64_t t = 0; t < trials; ++t)
    fit(15, p + 45 * t, f + 45 * t, reverse != 0, x_out + 6 * t, cost_out ? cost_out + t : nullptr,
        iterations_out ? iterations_out + t : nullptr);
  return 0;
}

// F at x, and {F, grad F, H} at x
double oracle_localization_cost(int n, const double* p, const double* f, const double* x) {
  return cost(n, p, f, x, false);
}
void oracle_localization_system(int n, const double* p, const double* f, const double* x, double* sys) {
  system(n, p, f, x, false, sys);
}

}  // extern "C"
