// A sequential restatement of feature refinement (b200ba_refine_features, include/b200ba.h): the pre-filter,
// matching against the rendered template, symmetry refinement and the final 0.75 px^2 test of the reference's
// RefineFeatureDetections with its CPU path. Gradient and gradient-magnitude images are computed up front, as the
// reference's CPU branch does, rather than on the fly as the kernel does. Compiled by tests/test_refine_features.py
// with -ffp-contract=off; the functions the kernel shares (atan2, PatternIntensityAt, 3 x 3 inverse, LDL^T) come
// from camera_calibration_b200/csrc/ba_common.h.
//
// Two summation modes: device order (lane l of 32 adds samples l, l + 32, ..., then xor butterflies 16, 8, 4, 2, 1),
// which the kernel must equal bit for bit, and reference order (one running float sum per accumulator), which
// measures what the parallel order changes.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

#include "../camera_calibration_b200/csrc/ba_common.h"

using b200ba::rf_inverse3;
using b200ba::rf_ldlt_solve;
using b200ba::rf_pattern_intensity;

namespace {

struct V2 {
  float x, y;
};

// per-accumulator sums over samples in either order
struct Sums {
  bool device;
  int n;
  std::vector<float> v;
  Sums(bool device_order, int count) : device(device_order), n(count), v((device_order ? 32 : 1) * count, 0.f) {}
  void add(int sample, int k, float x) {
    float& a = v[(device ? sample % 32 : 0) * n + k];
    a = a + x;
  }
  void finish(float* out) {
    if (device) {
      for (int o = 16; o; o >>= 1) {
        std::vector<float> w(v.size());
        for (int l = 0; l < 32; ++l)
          for (int k = 0; k < n; ++k) w[l * n + k] = v[l * n + k] + v[(l ^ o) * n + k];
        v.swap(w);
      }
    }
    for (int k = 0; k < n; ++k) out[k] = v[k];
  }
};

// one channel of an image: u8 or float pixels (row-major)
struct Channel {
  const uint8_t* u8 = nullptr;
  const float* f = nullptr;
  int stride = 1;  // floats between pixels
  int w = 0, h = 0;
  float at(int x, int y) const {
    const int64_t i = static_cast<int64_t>(y) * w + x;
    return u8 ? static_cast<float>(u8[i]) : f[i * stride];
  }
  bool inside(V2 p) const { return p.x >= 0 && p.y >= 0 && p.x < w - 1 && p.y < h - 1; }
  // Image::InterpolateBilinear
  float value(V2 p) const {
    const int ix = static_cast<int>(p.x), iy = static_cast<int>(p.y);
    const float fx = p.x - ix, fy = p.y - iy, fx_inv = 1.f - fx, fy_inv = 1.f - fy;
    return fx_inv * fy_inv * at(ix, iy) + fx * fy_inv * at(ix + 1, iy) + fx_inv * fy * at(ix, iy + 1) +
           fx * fy * at(ix + 1, iy + 1);
  }
  // Image::InterpolateBilinearWithJacobian; for u8 the differences are int subtractions
  float value_jac(V2 p, float* dx, float* dy) const {
    const int ix = static_cast<int>(p.x), iy = static_cast<int>(p.y);
    const float fx = p.x - ix, fy = p.y - iy, fx_inv = 1.f - fx, fy_inv = 1.f - fy;
    const float tl = at(ix, iy), tr = at(ix + 1, iy), bl = at(ix, iy + 1), br = at(ix + 1, iy + 1);
    const float top = fx_inv * tl + fx * tr;
    const float bottom = fx_inv * bl + fx * br;
    if (u8) {
      const int64_t i = static_cast<int64_t>(iy) * w + ix;
      const int dtl = u8[i], dtr = u8[i + 1], dbl = u8[i + w], dbr = u8[i + w + 1];
      *dx = fy * (dbr - dbl) + fy_inv * (dtr - dtl);
    } else {
      *dx = fy * (br - bl) + fy_inv * (tr - tl);
    }
    *dy = bottom - top;
    return fy_inv * top + fy * bottom;
  }
};

V2 hnorm(const float* m, float x, float y) {
  const float u = m[0] * x + m[1] * y + m[2] * 1.f;
  const float v = m[3] * x + m[4] * y + m[5] * 1.f;
  const float w = m[6] * x + m[7] * y + m[8] * 1.f;
  return {u / w, v / w};
}

bool valid_pattern_coord(const b200ba_pattern& p, float x, float y) {
  if (!(x >= -1.f && y >= -1.f && x <= p.squares_x - 1.f && y <= p.squares_y - 1.f)) return false;
  for (int k = 0; k < p.num_tags; ++k) {
    const b200ba_pattern_tag& t = p.tags[k];
    if (x >= t.x - 1 && y >= t.y - 1 && x <= t.x - 1 + t.width && y <= t.y - 1 + t.height) return false;
  }
  return true;
}

struct Context {
  const b200ba_pattern* pattern;
  const V2* samples;
  int n_samples, n_match, half, type;
  bool device;
  Channel u8, gradmag, gx, gy;
};

// ---- matching (cpu_refinement_by_matching.h) ----
bool match_cost(const Context& c, const std::vector<float>& q, V2 pos, float factor, float bias, float* cost) {
  Sums s(c.device, 1);
  for (int i = 0; i < c.n_match; ++i) {
    const V2 sp = {pos.x + c.half * c.samples[i].x, pos.y + c.half * c.samples[i].y};
    if (!c.u8.inside(sp)) return false;
    const float r = factor * c.u8.value(sp) + bias - q[i];
    s.add(i, 0, r * r);
  }
  s.finish(cost);
  return true;
}

int refine_by_matching(const Context& c, const float* M, V2 position, V2* out) {
  std::vector<float> q(c.n_match);
  for (int i = 0; i < c.n_match; ++i) {
    float sum = 0;
    for (int s = 0; s < 16; ++s) {
      const float ox = c.half * c.samples[i].x + static_cast<float>(-0.5 + 1 / 8.f + 1 / 4.f * (s % 4));
      const float oy = c.half * c.samples[i].y + static_cast<float>(-0.5 + 1 / 8.f + 1 / 4.f * (s / 4));
      const V2 po = hnorm(M, ox, oy);
      sum += rf_pattern_intensity(c.pattern->num_star_segments, po.x, po.y);
    }
    q[i] = sum;
  }
  float S[4];  // qp, p, q, pp
  {
    Sums s(c.device, 4);
    for (int i = 0; i < c.n_match; ++i) {
      const V2 sp = {position.x + c.half * c.samples[i].x, position.y + c.half * c.samples[i].y};
      if (!c.u8.inside(sp)) return B200BA_REFINE_MATCH_OUTSIDE;
      const float p = c.u8.value(sp);
      s.add(i, 0, q[i] * p);
      s.add(i, 1, p);
      s.add(i, 2, q[i]);
      s.add(i, 3, p * p);
    }
    s.finish(S);
  }
  const float denominator = S[3] - (S[1] * S[1] / c.n_match);
  float factor = std::fabs(denominator) > 1e-6f ? (S[0] - (S[1] / c.n_match) * S[2]) / denominator : 1.f;
  float bias = (1.f / c.n_match) * (S[2] - factor * S[1]);
  *out = position;
  float lambda = -1, last = std::numeric_limits<float>::infinity();
  bool converged = false;
  for (int iteration = 0; iteration < 50; ++iteration) {
    float A[15];  // H (10, packed upper), b (4), cost
    Sums s(c.device, 15);
    for (int i = 0; i < c.n_match; ++i) {
      const V2 sp = {out->x + c.half * c.samples[i].x, out->y + c.half * c.samples[i].y};
      if (!c.u8.inside(sp)) return B200BA_REFINE_MATCH_OUTSIDE;
      float dx, dy;
      const float v = c.u8.value_jac(sp, &dx, &dy);
      const float r = factor * v + bias - q[i];
      const float J[4] = {factor * dx, factor * dy, v, 1};
      for (int a = 0, k = 0; a < 4; ++a)
        for (int b = a; b < 4; ++b, ++k) s.add(i, k, J[a] * J[b]);
      for (int a = 0; a < 4; ++a) s.add(i, 10 + a, r * J[a]);
      s.add(i, 14, r * r);
    }
    s.finish(A);
    const float cost = A[14];
    if (lambda < 0) lambda = 0.001f * 0.5f * (A[0] + A[4] + A[7] + A[9]);
    bool applied = false;
    for (int attempt = 0; attempt < 10; ++attempt) {
      float x[4];
      rf_ldlt_solve<4>(A, lambda, A + 10, x);
      const V2 tp = {out->x - x[0], out->y - x[1]};
      const float tf = factor - x[2], tb = bias - x[3];
      float test_cost;
      if (!match_cost(c, q, tp, tf, tb, &test_cost)) return B200BA_REFINE_MATCH_OUTSIDE;
      if (test_cost < cost) {
        last = x[0] * x[0] + x[1] * x[1] + x[2] * x[2] + x[3] * x[3];
        *out = tp;
        factor = tf;
        bias = tb;
        lambda *= 0.5f;
        applied = true;
        break;
      }
      lambda *= 2.f;
    }
    if (!applied) {
      converged = true;
      break;
    }
    if (std::fabs(position.x - out->x) >= c.half || std::fabs(position.y - out->y) >= c.half)
      return B200BA_REFINE_MATCH_LEFT_WINDOW;
  }
  if (last < 1e-8) converged = true;
  if (!converged) return B200BA_REFINE_MATCH_NOT_CONVERGED;
  if (factor <= 0) return B200BA_REFINE_MATCH_BAD_FACTOR;
  return B200BA_REFINE_ACCEPTED;
}

// ---- symmetry (cpu_refinement_by_symmetry.h) ----
// d hnorm(P (t, 1)) / d(P00 .. P21): D[0..7] row 0, D[8..15] row 1
void position_wrt_homography(const float* P, float tx, float ty, float* D) {
  const float term0 = 1 / (P[6] * tx + P[7] * ty + 1);
  const float term1 = -1 * term0 * term0;
  const float term2 = (P[0] * tx + P[1] * ty + P[2]) * term1;
  const float term3 = (P[3] * tx + P[4] * ty + P[5]) * term1;
  const float row0[8] = {tx * term0, ty * term0, term0, 0, 0, 0, tx * term2, ty * term2};
  const float row1[8] = {0, 0, 0, tx * term0, ty * term0, term0, tx * term3, ty * term3};
  memcpy(D, row0, sizeof row0);
  memcpy(D + 8, row1, sizeof row1);
}

// the cost (and with H, the system: H 36 packed upper, b 8) at P
bool sym_eval(const Context& c, const std::vector<V2>& t, const float* P, float* H, float* b, float* cost) {
  const bool xy = c.type == B200BA_REFINE_GRADIENTS_XY;
  const Channel& ch = c.type == B200BA_REFINE_INTENSITIES ? c.u8 : (xy ? c.gx : c.gradmag);
  Sums s(c.device, H ? 45 : 1);
  for (int i = 0; i < c.n_samples; ++i) {
    const V2 pa = hnorm(P, t[i].x, t[i].y);
    if (!ch.inside(pa)) return false;
    const V2 pb = hnorm(P, -1 * t[i].x, -1 * t[i].y);
    if (!ch.inside(pb)) return false;
    const int n_rows = xy ? 2 : 1;
    float r[2], J[2][8];
    for (int row = 0; row < n_rows; ++row) {
      const Channel& cr = row == 0 ? ch : c.gy;
      if (!H) {
        r[row] = xy ? cr.value(pa) + cr.value(pb) : cr.value(pa) - cr.value(pb);
        continue;
      }
      float gax, gay, gbx, gby, Da[16], Db[16];
      const float va = cr.value_jac(pa, &gax, &gay);
      const float vb = cr.value_jac(pb, &gbx, &gby);
      position_wrt_homography(P, t[i].x, t[i].y, Da);
      position_wrt_homography(P, -1 * t[i].x, -1 * t[i].y, Db);
      r[row] = xy ? va + vb : va - vb;
      for (int k = 0; k < 8; ++k) {
        const float ja = gax * Da[k] + gay * Da[8 + k], jb = gbx * Db[k] + gby * Db[8 + k];
        J[row][k] = xy ? ja + jb : ja - jb;
      }
    }
    if (H) {
      for (int row = 0; row < n_rows; ++row) {
        for (int a = 0, k = 0; a < 8; ++a)
          for (int bb = a; bb < 8; ++bb, ++k) s.add(i, k, J[row][a] * J[row][bb]);
        for (int a = 0; a < 8; ++a) s.add(i, 36 + a, r[row] * J[row][a]);
      }
      s.add(i, 44, xy ? r[0] * r[0] + r[1] * r[1] : r[0] * r[0]);
    } else {
      s.add(i, 0, xy ? r[0] * r[0] + r[1] * r[1] : r[0] * r[0]);
    }
  }
  if (H) {
    float A[45];
    s.finish(A);
    memcpy(H, A, sizeof(float) * 36);
    memcpy(b, A + 36, sizeof(float) * 8);
    *cost = A[44];
  } else {
    s.finish(cost);
  }
  return true;
}

int refine_by_symmetry(const Context& c, const float* M, const float* L, V2 position, V2* out, float* final_cost) {
  *out = position;
  std::vector<V2> t(c.n_samples);
  for (int i = 0; i < c.n_samples; ++i) t[i] = hnorm(M, c.half * c.samples[i].x, c.half * c.samples[i].y);
  const float T[9] = {1, 0, position.x, 0, 1, position.y, 0, 0, 1};
  float P[9];
  for (int r = 0; r < 3; ++r)
    for (int col = 0; col < 3; ++col)
      P[r * 3 + col] = T[r * 3] * L[col] + T[r * 3 + 1] * L[3 + col] + T[r * 3 + 2] * L[6 + col];
  const float p22 = P[8];
  for (float& e : P) e /= p22;
  float lambda = -1, last = std::numeric_limits<float>::infinity();
  for (int iteration = 0; iteration < 30; ++iteration) {
    float H[36], b[8], cost;
    if (!sym_eval(c, t, P, H, b, &cost)) return B200BA_REFINE_SYM_OUTSIDE;
    *final_cost = cost;
    if (lambda < 0) {
      float d = 0;
      for (int k = 0, q = 0; k < 8; q += 8 - k, ++k) d = k == 0 ? H[0] : d + H[q];
      lambda = 0.001f * (1.f / 8) * d;
    }
    bool applied = false;
    for (int attempt = 0; attempt < 10; ++attempt) {
      float x[8], test[9];
      rf_ldlt_solve<8>(H, lambda, b, x);
      for (int k = 0; k < 8; ++k) test[k] = P[k] - x[k];
      test[8] = P[8];
      float test_cost;
      if (!sym_eval(c, t, test, nullptr, nullptr, &test_cost)) return B200BA_REFINE_SYM_OUTSIDE;
      if (test_cost < cost) {
        *final_cost = test_cost;
        last = x[2] * x[2] + x[5] * x[5];
        memcpy(P, test, sizeof P);
        lambda *= 0.5f;
        applied = true;
        break;
      }
      lambda *= 2.f;
    }
    if (!applied) return B200BA_REFINE_ACCEPTED;
    *out = {P[2], P[5]};
    if (std::fabs(position.x - out->x) >= c.half || std::fabs(position.y - out->y) >= c.half)
      return B200BA_REFINE_SYM_LEFT_WINDOW;
  }
  return last < 1e-4f ? B200BA_REFINE_ACCEPTED : B200BA_REFINE_SYM_NOT_CONVERGED;
}

}  // namespace

extern "C" {

// PatternData::PatternIntensityAt as the kernel computes it
float oracle_pattern_intensity(int num_star_segments, float x, float y) {
  return rf_pattern_intensity(num_star_segments, x, y);
}

float oracle_atan2(float y, float x) { return b200ba::rf_atan2(y, x); }

// bilinear value, then value, d/dx, d/dy of the Jacobian form, of a u8 image at (x, y)
void oracle_bilinear(const uint8_t* image, int w, int h, float x, float y, float* out) {
  Channel c;
  c.u8 = image, c.w = w, c.h = h;
  out[0] = c.value({x, y});
  out[1] = c.value_jac({x, y}, &out[2], &out[3]);
}

// The template's sub-samples (of the predictions that pass the pre-filter) whose segment changes when the C
// library's atan2f replaces rf_atan2; out[0] = changed, out[1] = total.
void oracle_atan2_template_changes(const b200ba_pattern* pattern, const float* samples, int half, int64_t n,
                                   const b200ba_feature_prediction* pred, int64_t* out) {
  const int n_match = (2 * half + 1) * (2 * half + 1);
  out[0] = out[1] = 0;
  for (int64_t f = 0; f < n; ++f) {
    float M[9];
    rf_inverse3(pred[f].local_pixel_tr_pattern, M);
    for (int i = 0; i < n_match; ++i)
      for (int s = 0; s < 16; ++s) {
        const float ox = half * samples[2 * i] + static_cast<float>(-0.5 + 1 / 8.f + 1 / 4.f * (s % 4));
        const float oy = half * samples[2 * i + 1] + static_cast<float>(-0.5 + 1 / 8.f + 1 / 4.f * (s / 4));
        const V2 p = hnorm(M, ox, oy);
        const float ours = rf_pattern_intensity(pattern->num_star_segments, p.x, p.y);
        // PatternIntensityAt with std::atan2 (float)
        V2 c;
        c.x = p.x - (p.x > 0 ? 1 : -1) * static_cast<int>(std::fabs(p.x) + 0.5f);
        c.y = p.y - (p.y > 0 ? 1 : -1) * static_cast<int>(std::fabs(p.y) + 0.5f);
        float theirs = 0.5f;
        if (!(c.x * c.x + c.y * c.y < 1e-8f)) {
          float angle = std::atan2(c.y, c.x) - 0.5f * M_PI;
          if (angle < 0) angle += 2 * M_PI;
          theirs = (static_cast<int>(pattern->num_star_segments * angle / (2 * M_PI)) % 2 == 0) ? 1.f : 0.f;
        }
        out[0] += ours != theirs;
        ++out[1];
      }
  }
}

// b200ba_refine_features restated; device_order selects the summation order
void oracle_refine(const b200ba_pattern* pattern, const uint8_t* images, int w, int h, const float* samples,
                   int n_samples, int half, int type, int64_t n, const b200ba_feature_prediction* pred,
                   int device_order, float* xy, float* final_cost, int32_t* status) {
  Context c;
  c.pattern = pattern;
  c.samples = reinterpret_cast<const V2*>(samples);
  c.n_samples = n_samples;
  c.n_match = static_cast<int>((1 / 8.) * n_samples);
  c.half = half;
  c.type = type;
  c.device = device_order != 0;
  const int64_t pixels = static_cast<int64_t>(w) * h;
  std::vector<float> grad, mag;
  int64_t cached = -1;
  for (int64_t f = 0; f < n; ++f) {
    const b200ba_feature_prediction& p = pred[f];
    const uint8_t* im = images + p.image * pixels;
    if (p.image != cached && type != B200BA_REFINE_INTENSITIES && type != B200BA_REFINE_NO_REFINEMENT) {
      // the gradient images of feature_detector_tagged_pattern.cc:269-287
      grad.assign(2 * pixels, 0.f);
      mag.assign(pixels, 0.f);
      for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
          const int mx = std::max(0, x - 1), px = std::min(w - 1, x + 1);
          const int my = std::max(0, y - 1), py = std::min(h - 1, y + 1);
          const float dx = (im[y * w + px] - static_cast<float>(im[y * w + mx])) / (px - mx);
          const float dy = (im[py * w + x] - static_cast<float>(im[my * w + x])) / (py - my);
          grad[2 * (y * w + x)] = dx;
          grad[2 * (y * w + x) + 1] = dy;
          mag[y * w + x] = std::sqrt(dx * dx + dy * dy);
        }
      cached = p.image;
    }
    c.u8 = Channel();
    c.u8.u8 = im, c.u8.w = w, c.u8.h = h;
    c.gradmag = Channel();
    c.gradmag.f = mag.data(), c.gradmag.w = w, c.gradmag.h = h;
    c.gx = Channel();
    c.gx.f = grad.data(), c.gx.stride = 2, c.gx.w = w, c.gx.h = h;
    c.gy = c.gx;
    c.gy.f = grad.data() + 1;
    int st = B200BA_REFINE_ACCEPTED;
    V2 pos = {p.position[0], p.position[1]}, m = pos;
    float cost = 0;
    float M[9];
    rf_inverse3(p.local_pixel_tr_pattern, M);
    if (!(pos.x - half >= 0 && pos.y - half >= 0 && pos.x + half < w - 1 && pos.y + half < h - 1)) {
      st = B200BA_REFINE_IMAGE_BORDER;
    } else {
      for (int corner = 0; corner < 4; ++corner) {
        const V2 o = hnorm(M, ((corner % 2 == 0) ? 1 : -1) * half, ((corner / 2 == 0) ? 1 : -1) * half);
        if (!valid_pattern_coord(*pattern, static_cast<float>(p.pattern_coordinate[0]) + o.x,
                                 static_cast<float>(p.pattern_coordinate[1]) + o.y)) {
          st = B200BA_REFINE_OUTSIDE_PATTERN;
          break;
        }
      }
    }
    if (st == B200BA_REFINE_ACCEPTED) st = refine_by_matching(c, M, pos, &m);
    pos = m;
    if (st == B200BA_REFINE_ACCEPTED && type != B200BA_REFINE_NO_REFINEMENT) {
      st = refine_by_symmetry(c, M, p.local_pixel_tr_pattern, m, &pos, &cost);
      const float dx = pos.x - m.x, dy = pos.y - m.y;
      if (st == B200BA_REFINE_ACCEPTED && dx * dx + dy * dy > 0.75f) st = B200BA_REFINE_INCONSISTENT;
    }
    const bool ok = st == B200BA_REFINE_ACCEPTED;
    const float nan = std::numeric_limits<float>::quiet_NaN();
    xy[2 * f] = ok ? pos.x : nan;
    xy[2 * f + 1] = ok ? pos.y : nan;
    final_cost[f] = ok ? cost : -1.f;
    status[f] = st;
  }
}

}  // extern "C"
