// A sequential restatement of --render_synthetic_dataset's rendering (render_synthetic_dataset.cc:79-291, libvis'
// geometry.h, PatternData::ComputePatternGeometry), written from the reference's description with the pinned rules
// of include/b200ba.h, for tests/test_render_synthetic.py. It loops over every polygon and every pixel of its
// bounding box as the reference does, clips with std::vectors and a float edge offset, and composes every pixel from
// its ray. Compiled with -ffp-contract=off so that no multiply-add is fused.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdint>
#include <vector>

#include "b200ba.h"

namespace {
struct V2f { float x, y; };
struct V2d { double x, y; };

bool valid_pattern_coord(const b200ba_pattern& p, float x, float y) {
  if (!(x >= -1.f && y >= -1.f && x <= p.squares_x - 1.f && y <= p.squares_y - 1.f)) return false;
  for (int k = 0; k < p.num_tags; ++k) {
    const b200ba_pattern_tag& t = p.tags[k];
    if (x >= t.x - 1 && y >= t.y - 1 && x <= t.x - 1 + t.width && y <= t.y - 1 + t.height) return false;
  }
  return true;
}

V2f star_coord(const b200ba_pattern& p, float i, float cx, float cy) {
  constexpr float square_length = 1;
  float angle = ((2 * M_PI) * i) / p.num_star_segments;
  float x = std::sin(angle);
  float y = std::cos(angle);
  float m = std::max(std::fabs(x), std::fabs(y));
  x /= m;
  y /= m;
  return {static_cast<float>(cx - 0.5 * square_length * x), static_cast<float>(cy - 0.5 * square_length * y)};
}

std::vector<std::vector<V2f>> pattern_geometry(const b200ba_pattern& p) {
  constexpr float square_length = 1;
  std::vector<std::vector<V2f>> out;  // generation order
  for (int y = -1; y < p.squares_y; ++y) {
    for (int x = -1; x < p.squares_x; ++x) {
      bool in_tag = false;
      for (int k = 0; k < p.num_tags; ++k) {
        const b200ba_pattern_tag& t = p.tags[k];
        if (x >= t.x && y >= t.y && x <= t.x - 2 + t.width && y <= t.y - 2 + t.height) {
          in_tag = true;
          break;
        }
      }
      if (in_tag) continue;
      for (int segment = 0; segment < p.num_star_segments; segment += 2) {
        V2f middle = star_coord(p, segment + 0.5f, x, y);
        if (!valid_pattern_coord(p, middle.x, middle.y)) continue;
        std::vector<V2f> poly;
        poly.push_back({static_cast<float>(x), static_cast<float>(y)});
        poly.push_back(star_coord(p, segment, x, y));
        float angle1 = (2 * M_PI) * (segment) / p.num_star_segments;
        float angle2 = (2 * M_PI) * (segment + 1) / p.num_star_segments;
        if (std::floor((angle1 - M_PI / 4) / (M_PI / 2)) != std::floor((angle2 - M_PI / 4) / (M_PI / 2))) {
          float corner_angle = (M_PI / 4) + (M_PI / 2) * std::floor((angle2 - M_PI / 4) / (M_PI / 2));
          float corner_x = std::sin(corner_angle);
          float corner_y = std::cos(corner_angle);
          float normalizer = std::fabs(corner_x);
          corner_x /= normalizer;
          corner_y /= normalizer;
          poly.push_back({static_cast<float>(x - 0.5 * square_length * corner_x),
                          static_cast<float>(y - 0.5 * square_length * corner_y)});
        }
        poly.push_back(star_coord(p, segment + 1, x, y));
        out.push_back(poly);
      }
    }
  }
  return out;
}

// static_cast<int>(double) / (float) as x86-64 executes it
int trunc86(double v) { return (v > -2147483649.0 && v < 2147483648.0) ? static_cast<int>(v) : INT_MIN; }
uint8_t u8_86(float v) {
  return static_cast<uint8_t>((v > -2147483649.f && v < 2147483648.f) ? static_cast<int>(v) : INT_MIN);
}

bool line_line_intersection(V2d a0, V2d a1, V2d b0, V2d b1, V2d* result) {
  double detL1 = a0.x * a1.y - a0.y * a1.x;
  double detL2 = b0.x * b1.y - b0.y * b1.x;
  double x1mx2 = a0.x - a1.x;
  double x3mx4 = b0.x - b1.x;
  double y1my2 = a0.y - a1.y;
  double y3my4 = b0.y - b1.y;
  double xnom = detL1 * x3mx4 - x1mx2 * detL2;
  double ynom = detL1 * y3my4 - y1my2 * detL2;
  double denom = x1mx2 * y3my4 - y1my2 * x3mx4;
  if (denom == 0) return false;
  result->x = xnom / denom;
  result->y = ynom / denom;
  return std::isfinite(result->x) && std::isfinite(result->y);
}

double dot(V2d a, V2d b) { return a.x * b.x + a.y * b.y; }

void convex_clip(const std::vector<V2d>& polygon, const std::vector<V2d>& clip, std::vector<V2d>* output) {
  const V2d &a = clip[0], &b = clip[1], &c = clip[2];
  float det = (b.x - a.x) * (c.y - a.y) - (c.x - a.x) * (b.y - a.y);
  int orientation = det > 0 ? 1 : -1;
  for (size_t e = 0; e < clip.size(); ++e) {
    size_t e1 = (e + 1) % clip.size();
    V2d edge{clip[e1].x - clip[e].x, clip[e1].y - clip[e].y};
    V2d right{edge.y, -edge.x};
    float edge_right = dot(right, clip[e1]);
    const std::vector<V2d>* input = e == 0 ? &polygon : output;
    std::vector<V2d> clipped;
    size_t n = input->size();
    for (size_t i = 0; i < n; ++i) {
      const V2d& cur = input->at(i);
      const V2d& prev = input->at((i + n - 1) % n);
      if (orientation * ((dot(right, cur) > edge_right) ? 1 : -1) < 0) {
        if (orientation * ((dot(right, prev) > edge_right) ? 1 : -1) > 0) {
          V2d r = prev;
          line_line_intersection(prev, cur, clip[e1], clip[e], &r);
          clipped.push_back(r);
        }
        clipped.push_back(cur);
      } else if (orientation * ((dot(right, prev) > edge_right) ? 1 : -1) < 0) {
        V2d r = prev;
        line_line_intersection(prev, cur, clip[e1], clip[e], &r);
        clipped.push_back(r);
      }
    }
    *output = clipped;
  }
}

double polygon_area(const std::vector<V2d>& p) {
  double result = 0;
  int prev = static_cast<int>(p.size()) - 1;
  for (int i = 0; i < static_cast<int>(p.size()); ++i) {
    result += (p[i].x - p[prev].x) * (p[i].y + p[prev].y);
    prev = i;
  }
  return std::fabs(0.5f * result);
}
}  // namespace

// images [n][h][w]; rendering (nullable) [n][h][w] float coverage images; sums (nullable) [n][2]: sum over pixels of
// (1 - rendering) in double, and sum over polygons of the area of the projected polygon clipped to [0, w] x [0, h]
extern "C" int oracle_render(const b200ba_pattern* pattern, const uint8_t* pattern_image, int32_t pw, int32_t ph,
                             int32_t w, int32_t h, const float* k, int64_t n, const double* poses, uint8_t* images,
                             float* rendering_out, double* sums) {
  const b200ba_pattern& p = *pattern;
  auto to_image = [&](V2f c) {
    float mx = p.pattern_start_x_mm + ((c.x + 1.f) / static_cast<float>(p.squares_x)) *
                                          (p.pattern_end_x_mm - p.pattern_start_x_mm);
    float my = p.pattern_start_y_mm + ((c.y + 1.f) / static_cast<float>(p.squares_y)) *
                                          (p.pattern_end_y_mm - p.pattern_start_y_mm);
    return V2f{(static_cast<float>(pw) / p.page_width_mm) * mx, (static_cast<float>(ph) / p.page_height_mm) * my};
  };
  std::vector<std::vector<V2f>> geometry = pattern_geometry(p);
  for (auto& poly : geometry)
    for (auto& v : poly) v = to_image(v);
  const float fx = k[0], fy = k[1], cx = k[2], cy = k[3];
  const float fx_inv = 1.f / fx, fy_inv = 1.f / fy, cx_inv = -cx / fx, cy_inv = -cy / fy;
  std::vector<float> rendering(static_cast<size_t>(w) * h);
  for (int64_t i = 0; i < n; ++i) {
    const double* R = poses + 12 * i;
    const double* t = R + 9;
    float Rf[9], tf[3], Rc[9], tc[3];
    for (int j = 0; j < 9; ++j) Rf[j] = static_cast<float>(R[j]);
    for (int j = 0; j < 3; ++j) tf[j] = static_cast<float>(t[j]);
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) Rc[r * 3 + c] = static_cast<float>(R[c * 3 + r]);
      tc[r] = static_cast<float>((R[r] * -t[0] + R[3 + r] * -t[1]) + R[6 + r] * -t[2]);
    }
    std::fill(rendering.begin(), rendering.end(), 1.f);
    double clipped_sum = 0;
    const std::vector<V2d> image_rect = {{0, 0}, {static_cast<double>(w), 0}, {static_cast<double>(w),
                                          static_cast<double>(h)}, {0, static_cast<double>(h)}};
    for (const auto& poly : geometry) {
      std::vector<V2d> projected(poly.size());
      bool nan = false;
      double min_x = 1.7976931348623157e308, min_y = min_x, max_x = -min_x, max_y = -min_x;
      for (size_t v = 0; v < poly.size(); ++v) {
        float q[3];
        for (int r = 0; r < 3; ++r)
          q[r] = (((Rf[r * 3] * poly[v].x) + (Rf[r * 3 + 1] * poly[v].y)) + (Rf[r * 3 + 2] * 0.f)) + tf[r];
        projected[v] = {static_cast<double>(fx * (q[0] / q[2]) + cx), static_cast<double>(fy * (q[1] / q[2]) + cy)};
        nan |= std::isnan(projected[v].x) || std::isnan(projected[v].y);
        min_x = std::min(min_x, projected[v].x);
        min_y = std::min(min_y, projected[v].y);
        max_x = std::max(max_x, projected[v].x);
        max_y = std::max(max_y, projected[v].y);
      }
      if (nan) continue;  // pinned: a NaN projected coordinate draws nothing
      if (sums) {
        std::vector<V2d> in_image;
        convex_clip(projected, image_rect, &in_image);
        clipped_sum += polygon_area(in_image);
      }
      int x0 = std::max<int>(0, trunc86(min_x)), x1 = std::min<int>(w - 1, trunc86(max_x));
      int y0 = std::max<int>(0, trunc86(min_y)), y1 = std::min<int>(h - 1, trunc86(max_y));
      for (int y = y0; y <= y1; ++y) {
        for (int x = x0; x <= x1; ++x) {
          std::vector<V2d> pixel = {{static_cast<double>(x), static_cast<double>(y)},
                                    {x + 1.0, static_cast<double>(y)},
                                    {x + 1.0, y + 1.0},
                                    {static_cast<double>(x), y + 1.0}};
          std::vector<V2d> inter;
          convex_clip(projected, pixel, &inter);
          float& r = rendering[static_cast<size_t>(y) * w + x];
          r = static_cast<float>(r - polygon_area(inter));
        }
      }
    }
    double coverage = 0;
    for (float r : rendering) coverage += 1.0 - r;
    if (sums) {
      sums[2 * i] = coverage;
      sums[2 * i + 1] = clipped_sum;
    }
    if (rendering_out)
      std::copy(rendering.begin(), rendering.end(), rendering_out + static_cast<size_t>(i) * w * h);
    uint8_t* img = images + static_cast<size_t>(i) * w * h;
    for (int y = 0; y < h; ++y) {
      for (int x = 0; x < w; ++x) {
        float px = x + 0.5f, py = y + 0.5f;
        float lx = fx_inv * px + cx_inv, ly = fy_inv * py + cy_inv;
        float d[3];
        for (int r = 0; r < 3; ++r) d[r] = ((Rc[r * 3] * lx) + (Rc[r * 3 + 1] * ly)) + (Rc[r * 3 + 2] * 1.f);
        float n2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
        if (n2 > 0.f) {
          float s = std::sqrt(n2);
          for (float& e : d) e = e / s;
        }
        const float offset = -0.f;
        float tt = -(offset + ((0.f * tc[0] + 0.f * tc[1]) + -1.f * tc[2])) / ((0.f * d[0] + 0.f * d[1]) + -1.f * d[2]);
        float X = tc[0] + d[0] * tt, Y = tc[1] + d[1] * tt;
        float lx2 = X - 0.f, ly2 = Y - -0.f;
        float ix = 1.f * lx2 + 0.f * ly2, iy = 0.f * lx2 + 1.f * ly2;
        float mx = (p.page_width_mm / static_cast<float>(pw)) * ix;
        float my = (p.page_height_mm / static_cast<float>(ph)) * iy;
        float ccx = ((mx - p.pattern_start_x_mm) / (p.pattern_end_x_mm - p.pattern_start_x_mm)) *
                        static_cast<float>(p.squares_x) - 1.f;
        float ccy = ((my - p.pattern_start_y_mm) / (p.pattern_end_y_mm - p.pattern_start_y_mm)) *
                        static_cast<float>(p.squares_y) - 1.f;
        uint8_t out = 0;
        if (valid_pattern_coord(p, ccx, ccy)) {
          out = u8_86(std::max<float>(0.f, 255.99f * rendering[static_cast<size_t>(y) * w + x]));
        } else {
          float qx = ix - 0.5f, qy = iy - 0.5f;
          if (qx >= 0 && qy >= 0 && qx < static_cast<float>(pw - 1) && qy < static_cast<float>(ph - 1)) {
            int jx = static_cast<int>(qx), jy = static_cast<int>(qy);
            float ffx = qx - jx, ffy = qy - jy, gx = 1.f - ffx, gy = 1.f - ffy;
            const uint8_t* row = pattern_image + static_cast<size_t>(jy) * pw + jx;
            out = u8_86(gx * gy * static_cast<float>(row[0]) + ffx * gy * static_cast<float>(row[1]) +
                        gx * ffy * static_cast<float>(row[pw]) + ffx * ffy * static_cast<float>(row[pw + 1]));
          }
        }
        img[static_cast<size_t>(y) * w + x] = out;
      }
    }
  }
  return 0;
}

// the pattern geometry in pattern-image pixels: verts [count][4][2] (unused vertices 0), nv [count]; returns count
extern "C" int64_t oracle_geometry(const b200ba_pattern* pattern, int32_t pw, int32_t ph, float* verts, int8_t* nv,
                                   int64_t capacity) {
  const b200ba_pattern& p = *pattern;
  std::vector<std::vector<V2f>> geometry = pattern_geometry(p);
  int64_t i = 0;
  for (const auto& poly : geometry) {
    if (i < capacity) {
      for (int v = 0; v < 4; ++v) {
        V2f c = v < static_cast<int>(poly.size()) ? poly[v] : V2f{-1.f, -1.f};
        float mx = p.pattern_start_x_mm + ((c.x + 1.f) / static_cast<float>(p.squares_x)) *
                                              (p.pattern_end_x_mm - p.pattern_start_x_mm);
        float my = p.pattern_start_y_mm + ((c.y + 1.f) / static_cast<float>(p.squares_y)) *
                                              (p.pattern_end_y_mm - p.pattern_start_y_mm);
        verts[8 * i + 2 * v] = v < static_cast<int>(poly.size()) ? (static_cast<float>(pw) / p.page_width_mm) * mx : 0.f;
        verts[8 * i + 2 * v + 1] = v < static_cast<int>(poly.size()) ? (static_cast<float>(ph) / p.page_height_mm) * my : 0.f;
      }
      nv[i] = static_cast<int8_t>(poly.size());
    }
    ++i;
  }
  return i;
}
