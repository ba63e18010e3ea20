// voronoi_oracle.cc -- sequential CPU restatement of the Voronoi error maps of the calibration report
// (APP/calibration_report.cc:354-545), the reference b200ba_render_voronoi is tested against. TEST INFRASTRUCTURE.
//
// A different algorithm from the library's per-pixel gather: every Voronoi cell is built explicitly and then
// rasterised the way the reference does it.
//   cell:   a box that contains the image and every site, clipped by the bisectors of the neighbours taken in order
//           of distance (a bucket grid yields them ring by ring); a neighbour farther than twice the farthest
//           vertex of the cell cannot cut it, so the walk stops there. A repeated position belongs to its lowest
//           index; later copies get no cell.
//   render: a triangle fan from the site over the cell's edges; each triangle is clipped against each pixel of its
//           bounding box and area * colour is accumulated in float; then + 0.5f, clamped to [0, 255.99f], truncated.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <queue>
#include <set>
#include <utility>
#include <vector>

namespace {

struct P2 {
  double x, y;
};

// keep the part of the convex polygon where a x + b y <= c
std::vector<P2> clip_half_plane(const std::vector<P2>& poly, double a, double b, double c) {
  std::vector<P2> out;
  const size_t n = poly.size();
  for (size_t k = 0; k < n; ++k) {
    const P2 p = poly[k], q = poly[(k + 1) % n];
    const double fp = a * p.x + b * p.y - c, fq = a * q.x + b * q.y - c;
    if (fp <= 0) out.push_back(p);
    if ((fp < 0 && fq > 0) || (fp > 0 && fq < 0)) {
      const double t = fp / (fp - fq);
      out.push_back(P2{p.x + t * (q.x - p.x), p.y + t * (q.y - p.y)});
    }
  }
  return out;
}

double polygon_area(const std::vector<P2>& poly) {
  double a = 0;
  for (size_t k = 0; k < poly.size(); ++k) {
    const P2 p = poly[k], q = poly[(k + 1) % poly.size()];
    a += p.x * q.y - q.x * p.y;
  }
  return std::fabs(0.5 * a);
}

}  // namespace

extern "C" {

// sites_q [2n] quarter-pixel integer sites, colors [3n]; image [h*w*3] u8 and value [h*w*3] (nullable): the float
// sum before + 0.5f. Returns the number of sites that own a cell.
int64_t oracle_render_voronoi(int32_t width, int32_t height, int64_t n, const int32_t* sites_q, const float* colors,
                              uint8_t* image, float* value) {
  const int64_t pixels = static_cast<int64_t>(width) * height;
  std::vector<float> acc(3 * pixels, 0.f);
  // the lowest index of every position
  std::vector<char> owner(n, 0);
  {
    std::set<std::pair<int32_t, int32_t>> seen;
    for (int64_t i = 0; i < n; ++i) owner[i] = seen.insert({sites_q[2 * i], sites_q[2 * i + 1]}).second ? 1 : 0;
  }
  std::vector<int64_t> live;
  for (int64_t i = 0; i < n; ++i)
    if (owner[i]) live.push_back(i);
  if (!live.empty()) {
    // the box (pixels): image and sites with a margin
    double bx0 = 0, by0 = 0, bx1 = width, by1 = height;
    for (int64_t i : live) {
      bx0 = std::min(bx0, 0.25 * sites_q[2 * i]);
      by0 = std::min(by0, 0.25 * sites_q[2 * i + 1]);
      bx1 = std::max(bx1, 0.25 * sites_q[2 * i]);
      by1 = std::max(by1, 0.25 * sites_q[2 * i + 1]);
    }
    bx0 -= 1; by0 -= 1; bx1 += 1; by1 += 1;
    // bucket grid of about 2 sites per bucket
    const double bs = std::max(1.0, std::sqrt((bx1 - bx0) * (by1 - by0) / (0.5 * live.size())));
    const int nx = static_cast<int>((bx1 - bx0) / bs) + 1, ny = static_cast<int>((by1 - by0) / bs) + 1;
    std::vector<std::vector<int64_t>> bucket(static_cast<size_t>(nx) * ny);
    auto bucket_of = [&](double x, double y, int* ix, int* iy) {
      *ix = std::min(nx - 1, std::max(0, static_cast<int>((x - bx0) / bs)));
      *iy = std::min(ny - 1, std::max(0, static_cast<int>((y - by0) / bs)));
    };
    for (int64_t i : live) {
      int ix, iy;
      bucket_of(0.25 * sites_q[2 * i], 0.25 * sites_q[2 * i + 1], &ix, &iy);
      bucket[static_cast<size_t>(iy) * nx + ix].push_back(i);
    }
    for (int64_t i : live) {
      const double sx = 0.25 * sites_q[2 * i], sy = 0.25 * sites_q[2 * i + 1];
      // the cell, relative to the site
      std::vector<P2> cell = {{bx0 - sx, by0 - sy}, {bx1 - sx, by0 - sy}, {bx1 - sx, by1 - sy}, {bx0 - sx, by1 - sy}};
      auto far2 = [&]() {
        double m = 0;
        for (const P2& p : cell) m = std::max(m, p.x * p.x + p.y * p.y);
        return m;
      };
      int cx, cy;
      bucket_of(sx, sy, &cx, &cy);
      using Item = std::pair<double, int64_t>;
      std::priority_queue<Item, std::vector<Item>, std::greater<Item>> near;
      for (int r = 0;; ++r) {
        bool any = false;
        for (int by = cy - r; by <= cy + r; ++by)
          for (int bx = cx - r; bx <= cx + r; ++bx) {
            if (std::max(std::abs(bx - cx), std::abs(by - cy)) != r || bx < 0 || by < 0 || bx >= nx || by >= ny) continue;
            any = true;
            for (int64_t j : bucket[static_cast<size_t>(by) * nx + bx]) {
              if (j == i) continue;
              const double dx = 0.25 * sites_q[2 * j] - sx, dy = 0.25 * sites_q[2 * j + 1] - sy;
              near.push({dx * dx + dy * dy, j});
            }
          }
        // every site not yet seen is at least r * bs away
        const double seen_bound = r * bs;
        while (!near.empty() && near.top().first <= seen_bound * seen_bound) {
          const Item it = near.top();
          near.pop();
          if (it.first > 4 * far2()) break;
          const double dx = 0.25 * sites_q[2 * it.second] - sx, dy = 0.25 * sites_q[2 * it.second + 1] - sy;
          // |q|^2 <= |q - d|^2  <=>  2 d . q <= |d|^2
          cell = clip_half_plane(cell, 2 * dx, 2 * dy, dx * dx + dy * dy);
        }
        const double f2 = far2();
        const double next = near.empty() ? seen_bound * seen_bound : std::min(near.top().first, seen_bound * seen_bound);
        if (next > 4 * f2 || (!any && near.empty())) break;
      }
      // triangle fan from the site, rasterised pixel by pixel
      const float* col = colors + 3 * i;
      for (size_t k = 0; k < cell.size(); ++k) {
        const P2 a{sx, sy}, b{cell[k].x + sx, cell[k].y + sy};
        const P2 c{cell[(k + 1) % cell.size()].x + sx, cell[(k + 1) % cell.size()].y + sy};
        const int x0 = std::max(0, static_cast<int>(std::floor(std::min({a.x, b.x, c.x}))));
        const int x1 = std::min(width - 1, static_cast<int>(std::floor(std::max({a.x, b.x, c.x}))));
        const int y0 = std::max(0, static_cast<int>(std::floor(std::min({a.y, b.y, c.y}))));
        const int y1 = std::min(height - 1, static_cast<int>(std::floor(std::max({a.y, b.y, c.y}))));
        for (int y = y0; y <= y1; ++y)
          for (int x = x0; x <= x1; ++x) {
            std::vector<P2> t = {a, b, c};
            t = clip_half_plane(t, -1, 0, -x);
            t = clip_half_plane(t, 1, 0, x + 1);
            t = clip_half_plane(t, 0, -1, -y);
            t = clip_half_plane(t, 0, 1, y + 1);
            if (t.size() < 3) continue;
            const float area = static_cast<float>(polygon_area(t));
            float* px = acc.data() + 3 * (static_cast<int64_t>(y) * width + x);
            for (int ch = 0; ch < 3; ++ch) px[ch] += area * col[ch];
          }
      }
    }
  }
  for (int64_t p = 0; p < 3 * pixels; ++p) {
    if (value) value[p] = acc[p];
    const float v = std::min(std::max(acc[p] + 0.5f, 0.f), 255.99f);
    image[p] = static_cast<uint8_t>(static_cast<int>(v));
  }
  return static_cast<int64_t>(live.size());
}

}  // extern "C"
