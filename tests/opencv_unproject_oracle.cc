// Sequential CPU restatement of the OpenCV un-projection of b200ba_compare_reconstructions, for
// tests/test_compare_reconstructions.py (which compiles it itself, with -ffp-contract=off): CentralOpenCVModel::
// Unproject (APP/models/central_opencv.cc:150-156) = UnprojectWithGaussNewton (APP/models/parametric.h:60-148) from
// the normalised pixel, then (x, y, 1) normalised. The iteration's 2 x 2 Jacobian is the derivative of the distortion
// value (include/b200ba.h explains why it is not the reference's closed form); the accept and stop rules are the
// reference's: lambda_0 = 1.0 * 0.5 (H00 + H11) at the first iteration, at most 5 attempts (x0.1 on an accepted step,
// x10 on a rejected one), at most 100 iterations, converged once an iteration ends with cost < 1e-10f, stop after an
// iteration that accepts nothing.
#include <cmath>
#include <cstdint>

namespace {

void distort(const double* q, double nx, double ny, double* ux, double* uy, double J[2][2]) {
  const double x2 = nx * nx, xy = nx * ny, y2 = ny * ny;
  const double r2 = x2 + y2, r4 = r2 * r2, r6 = r4 * r2;
  const double k1 = q[4], k2 = q[5], k3 = q[6], k4 = q[7], k5 = q[8], k6 = q[9], p1 = q[10], p2 = q[11];
  const double num = 1 + k1 * r2 + k2 * r4 + k3 * r6;
  const double den = 1 + k4 * r2 + k5 * r4 + k6 * r6;
  const double iden = 1.0 / den;
  const double radial = num * iden;
  const double drad = ((k1 + 2 * k2 * r2 + 3 * k3 * r4) * den - num * (k4 + 2 * k5 * r2 + 3 * k6 * r4)) * iden * iden;
  *ux = nx * radial + (2.0 * p1 * xy + p2 * (r2 + 2.0 * x2));
  *uy = ny * radial + (2.0 * p2 * xy + p1 * (r2 + 2.0 * y2));
  J[0][0] = radial + 2 * x2 * drad + 2 * p1 * ny + 6 * p2 * nx;
  J[0][1] = 2 * xy * drad + 2 * p1 * nx + 2 * p2 * ny;
  J[1][0] = 2 * xy * drad + 2 * p2 * ny + 2 * p1 * nx;
  J[1][1] = radial + 2 * y2 * drad + 2 * p2 * nx + 6 * p1 * ny;
}

bool unproject(const double* q, double x, double y, double d[3]) {
  const double px = (x - q[2]) / q[0], py = (y - q[3]) / q[1];
  double cx = px, cy = py;
  const double kEpsilon = 1e-10f;
  double lambda = -1;
  bool converged = false;
  for (int i = 0; i < 100; ++i) {
    double ux, uy, J[2][2];
    distort(q, cx, cy, &ux, &uy, J);
    double dx = ux - px, dy = uy - py;
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
      distort(q, tx, ty, &tux, &tuy, TJ);
      dx = tux - px;
      dy = tuy - py;
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
  const double n = std::sqrt(cx * cx + cy * cy + 1.0);
  d[0] = cx / n;
  d[1] = cy / n;
  d[2] = 1.0 / n;
  return true;
}

}  // namespace

// parameters [12] fx fy cx cy k1..k6 p1 p2; pixels [2 n]; directions [3 n] (0 where ok[i] == 0)
extern "C" void opencv_unproject_oracle(const double* parameters, int64_t n, const double* pixels, double* directions,
                                        int32_t* ok) {
  for (int64_t i = 0; i < n; ++i) {
    double* d = directions + 3 * i;
    d[0] = d[1] = d[2] = 0;
    ok[i] = unproject(parameters, pixels[2 * i], pixels[2 * i + 1], d) ? 1 : 0;
  }
}
