// b200ba_pipeline.hpp -- C++ host logic of the callers either side of the hot path (SURVEY.md 8f-3 / 8f-4):
// the outlier deletion between bundle-adjustment rounds (host-driven, and on the device), the metric rescaling, the pyramid resampling of the generic
// models, the calibration report's info files, the comparison of two calibrations, the localization accuracy test and
// the --bundle_adjustment / --compare_reconstructions tools, the calibration visualisation tools and the
// --render_synthetic_dataset tool, over the containers of
// b200ba_shim.hpp. (RunBundleAdjustment itself -- 8f-2 -- is in b200ba_shim.hpp and runs device-resident in the
// library.) The Python mirror is camera_calibration_b200/pipeline.py.
//
// Header-only. Every numerical step on observations (the re-projection of all features of a camera) runs in
// libb200ba.so through b200ba_project; there is no CPU fallback.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <filesystem>
#include <fstream>
#include <functional>
#include <iomanip>
#include <iostream>
#include <map>
#include <sstream>
#include <unordered_map>

#include "b200ba_io.hpp"
#include "b200ba_shim.hpp"

namespace b200ba_shim {

// (model, local points [3 n]) -> pixels [2 n], ok [n]. The default runs CameraModel::Project (start at the centre of
// the calibrated area, models/central_generic.cc:398-422) for all points in one b200ba_project call.
using ProjectMany = std::function<void(CameraModel&, const std::vector<double>&, std::vector<double>*, std::vector<int32_t>*)>;

inline void ProjectManyOnDevice(CameraModel& model, const std::vector<double>& local_points, std::vector<double>* pixels,
                                std::vector<int32_t>* ok) {
  const int64_t n = static_cast<int64_t>(local_points.size() / 3);
  b200ba_camera c{};
  c.model_type = static_cast<int32_t>(model.type());
  c.width = model.width();
  c.height = model.height();
  c.calibration_min_x = model.calibration_min_x();
  c.calibration_min_y = model.calibration_min_y();
  c.calibration_max_x = model.calibration_max_x();
  c.calibration_max_y = model.calibration_max_y();
  int rx = 0, ry = 0;
  if (model.GetGridResolution(&rx, &ry)) { c.grid_width = rx; c.grid_height = ry; }
  const Vec2d centre = model.CenterOfCalibratedArea();
  pixels->resize(2 * n);
  for (int64_t i = 0; i < n; ++i) { (*pixels)[2 * i] = centre.x; (*pixels)[2 * i + 1] = centre.y; }
  ok->assign(n, 0);
  if (n == 0) return;
  if (b200ba_project(-1, &c, model.flat_intrinsics().data(), n, local_points.data(), pixels->data(), ok->data()) != 0)
    throw std::runtime_error(std::string("b200ba_project: ") + b200ba_last_error(nullptr));
}

// calibration.cc:62-184 -- the quartile rule between BA rounds: re-project every feature of one camera, take the
// first and third quartile q1, q3 of the error magnitudes and erase the features that fail to project or whose
// error exceeds q3 + outlier_removal_factor (q3 - q1). Imagesets left with fewer than three features of this
// camera are marked unused. Returns the number of removed features.
inline int DeleteOutlierFeatures(int camera_index, Dataset* dataset, BAState* state, float outlier_removal_factor,
                                 const ProjectMany& project_many = ProjectManyOnDevice) {
  CameraModel& model = *state->intrinsics[camera_index];
  struct Span { int imageset; size_t first, last; };
  std::vector<Span> spans;
  std::vector<double> local_points;
  std::vector<float> observed;
  for (int i = 0; i < dataset->ImagesetCount(); ++i) {
    if (!state->image_used[i]) continue;
    const std::vector<PointFeature>& features = dataset->GetImageset(i)->FeaturesOfCamera(camera_index);
    const SE3d image_tr_global = state->image_tr_global(camera_index, i);
    const size_t first = observed.size() / 2;
    for (const PointFeature& f : features) {
      const Vec3d p = apply(image_tr_global, state->points[f.index]);
      local_points.insert(local_points.end(), {p.x, p.y, p.z});
      observed.push_back(f.xy.x);
      observed.push_back(f.xy.y);
    }
    spans.push_back(Span{i, first, observed.size() / 2});
  }
  const size_t n = observed.size() / 2;
  if (n == 0) return 0;
  std::vector<double> pixels;
  std::vector<int32_t> ok;
  project_many(model, local_points, &pixels, &ok);
  if (pixels.size() != 2 * n || ok.size() != n) throw std::runtime_error("DeleteOutlierFeatures: projector returned a wrong size");
  std::vector<double> error(n), sorted;
  for (size_t k = 0; k < n; ++k) {
    const double dx = pixels[2 * k] - static_cast<double>(observed[2 * k]), dy = pixels[2 * k + 1] - static_cast<double>(observed[2 * k + 1]);
    error[k] = std::sqrt(dx * dx + dy * dy);
    if (ok[k]) sorted.push_back(error[k]);
  }
  if (sorted.size() < 8) return 0;  // too few to detect outliers reliably (calibration.cc:97-100)
  std::sort(sorted.begin(), sorted.end());
  // quartile positions in float arithmetic, truncated (calibration.cc:103-104)
  const double first_quartile = sorted[static_cast<size_t>(0.25f * static_cast<float>(sorted.size()) + 0.5f)];
  const double third_quartile = sorted[static_cast<size_t>(0.75f * static_cast<float>(sorted.size()) + 0.5f)];
  const double threshold = third_quartile + static_cast<double>(outlier_removal_factor) * (third_quartile - first_quartile);
  int removed = 0;
  for (const Span& span : spans) {
    std::vector<PointFeature>& features = dataset->GetImageset(span.imageset)->FeaturesOfCamera(camera_index);
    size_t kept = 0;
    for (size_t k = span.first; k < span.last; ++k) {
      if (!ok[k] || error[k] > threshold) {
        ++removed;
        continue;
      }
      features[kept++] = features[k - span.first];
    }
    features.resize(kept);
    if (kept < 3) state->image_used[span.imageset] = false;
  }
  return removed;
}

namespace detail {
// b200ba_create on a flattening (problem arrays point into f)
inline b200ba_handle* create_handle(Flat& f, size_t n_points) {
  b200ba_problem pb{};
  pb.n_cameras = static_cast<int32_t>(f.cams.size());
  pb.cameras = f.cams.data();
  pb.n_imagesets = static_cast<int32_t>(f.used.size());
  pb.n_points = static_cast<int32_t>(n_points);
  pb.n_obs = static_cast<int64_t>(f.oi.size());
  pb.obs_imageset = f.oi.data();
  pb.obs_camera = f.oc.data();
  pb.obs_point = f.op.data();
  pb.obs_xy = f.oxy.data();
  b200ba_handle* h = nullptr;
  if (b200ba_create(&pb, -1, &h) != 0) throw std::runtime_error(std::string("b200ba_create: ") + b200ba_last_error(nullptr));
  return h;
}
// the state held in f (after b200ba_get_state) back into the containers: poses, points, last_projection; the intrinsics
// were written in place through flat_intrinsics()
inline void read_back(const Flat& f, Dataset* dataset, BAState* state) {
  for (size_t c = 0; c < state->camera_tr_rig.size(); ++c) state->camera_tr_rig[c] = pose_at(f.ctr, c);
  for (size_t s = 0; s < f.used.size(); ++s) state->rig_tr_global[f.used[s]] = pose_at(f.rtg, s);
  for (size_t p = 0; p < state->points.size(); ++p) state->points[p] = Vec3d{f.points[3 * p], f.points[3 * p + 1], f.points[3 * p + 2]};
  size_t o = 0;
  for (size_t seq = 0; seq < f.used.size(); ++seq)
    for (int c = 0; c < dataset->num_cameras(); ++c)
      for (PointFeature& ft : dataset->GetImageset(f.used[seq])->FeaturesOfCamera(c)) {
        ft.last_projection = Vec2d{f.lastp[2 * o], f.lastp[2 * o + 1]};
        ++o;
      }
}
// The outlier round of `cameras`, in order, on one handle with the state uploaded once: b200ba_delete_outliers per
// camera with imageset_used carried from one camera to the next, the reference's count line and image per camera that
// is not skipped, then the removals and the imageset rule applied to the containers.
inline std::vector<b200ba_outlier_report> outlier_round(const std::vector<int>& cameras, Dataset* dataset, BAState* state,
                                                        float outlier_removal_factor, const char* outlier_visualization_path) {
  Flat f;
  flatten(*dataset, state, &f);
  b200ba_handle* h = create_handle(f, state->points.size());
  b200ba_state st{f.points.data(), f.rtg.data(), f.ctr.data(), f.intr.data(), f.lastp.data()};
  std::vector<uint8_t> used(std::max<size_t>(f.used.size(), 1), 1), remove(std::max<size_t>(f.oi.size(), 1), 0),
      removed_any(f.oi.size(), 0);
  std::vector<b200ba_outlier_report> reports;
  int rc = b200ba_set_state(h, &st);
  for (size_t k = 0; rc == 0 && k < cameras.size(); ++k) {
    const int camera = cameras[k];
    const bool in_range = camera >= 0 && camera < static_cast<int>(state->intrinsics.size());
    const bool with_image = outlier_visualization_path != nullptr && in_range;
    const CameraModel* cam = in_range ? state->intrinsics[camera].get() : nullptr;
    std::vector<uint8_t> image(with_image ? 3 * static_cast<size_t>(cam->width()) * cam->height() : 0);
    b200ba_outlier_report report{};
    rc = b200ba_delete_outliers(h, camera, outlier_removal_factor, used.data(), remove.data(),
                                with_image ? image.data() : nullptr, &report, nullptr);
    if (rc) break;
    reports.push_back(report);
    if (report.skipped) continue;
    for (size_t o = 0; o < f.oi.size(); ++o) removed_any[o] |= remove[o];
    std::cerr << "Outlier detection removed " << report.removed << " outlier features." << std::endl;
    if (with_image) {
      const std::string path = std::string(outlier_visualization_path) + "_camera" + std::to_string(camera) + "_removed_outliers.png";
      const std::filesystem::path parent = std::filesystem::path(path).parent_path();
      if (!parent.empty()) std::filesystem::create_directories(parent);
      if (!WritePNG(path, cam->width(), cam->height(), 3, image.data())) std::cerr << "Cannot write file: " << path << std::endl;
    }
  }
  const std::string err = rc ? b200ba_last_error(h) : "";
  b200ba_destroy(h);
  if (rc) throw std::runtime_error("b200ba_delete_outliers: " + err);
  size_t o = 0;
  for (size_t seq = 0; seq < f.used.size(); ++seq)
    for (int c = 0; c < dataset->num_cameras(); ++c) {
      std::vector<PointFeature>& features = dataset->GetImageset(f.used[seq])->FeaturesOfCamera(c);
      size_t kept = 0;
      for (size_t j = 0; j < features.size(); ++j, ++o)
        if (!removed_any[o]) features[kept++] = features[j];
      features.resize(kept);
    }
  for (size_t seq = 0; seq < f.used.size(); ++seq) state->image_used[f.used[seq]] = used[seq] != 0;
  return reports;
}
}  // namespace detail

// DeleteOutlierFeatures (calibration.cc:62-184) for one camera with every step in the library: one handle on the
// flattening OptimizeJointly uses, one b200ba_delete_outliers (the report's error pass, the exact quartiles, the
// decisions). The removed features are erased (the survivors keep their order and last_projection), imagesets left with
// fewer than 3 features of the camera are marked unused and, with outlier_visualization_path and unless the camera was
// skipped (fewer than 8 successful projections), <path>_camera<i>_removed_outliers.png is written. Prints the
// reference's count line to stderr when the camera is not skipped. Returns the library's report; throws on a library
// error. The Python mirror is pipeline.DeleteOutlierFeaturesOnDevice.
inline b200ba_outlier_report DeleteOutlierFeaturesOnDevice(int camera_index, Dataset* dataset, BAState* state,
                                                           float outlier_removal_factor,
                                                           const char* outlier_visualization_path = nullptr) {
  return detail::outlier_round({camera_index}, dataset, state, outlier_removal_factor, outlier_visualization_path)[0];
}

// calibration.cc:307-370 -- geometric-mean ratio of the known pattern cell length to the optimised distance of
// neighbouring corners (right and down neighbours), applied with BAState::ScaleState. Returns the factor; throws
// when no neighbouring pair with known geometry exists (the reference divides by zero there).
inline double ScaleToMetric(const Dataset& dataset, BAState* state) {
  double log_sum = 0;
  long long count = 0;
  for (const KnownGeometry& geometry : dataset.known_geometries()) {
    std::map<std::pair<int, int>, int> position_to_index;
    for (const auto& item : geometry.feature_id_to_position) {
      auto it = state->feature_id_to_points_index.find(item.first);
      if (it != state->feature_id_to_points_index.end()) position_to_index[item.second] = it->second;
    }
    if (position_to_index.empty()) continue;
    for (const auto& item : geometry.feature_id_to_position) {
      auto self = position_to_index.find(item.second);
      if (self == position_to_index.end()) continue;
      const std::pair<int, int> neighbours[2] = {{item.second.first + 1, item.second.second}, {item.second.first, item.second.second + 1}};
      for (const auto& position : neighbours) {
        auto other = position_to_index.find(position);
        if (other == position_to_index.end()) continue;
        const Vec3d &a = state->points[self->second], &b = state->points[other->second];
        const double actual = std::sqrt((a.x - b.x) * (a.x - b.x) + (a.y - b.y) * (a.y - b.y) + (a.z - b.z) * (a.z - b.z));
        log_sum += std::log(static_cast<double>(geometry.cell_length_in_meters) / actual);
        ++count;
      }
    }
  }
  if (count == 0) throw std::runtime_error("ScaleToMetric: no neighbouring corners with known geometry");
  const double factor = std::exp(log_sum / static_cast<double>(count));
  state->ScaleState(factor);
  return factor;
}

// ---- pyramid resampling (SURVEY.md 8f-4) ------------------------------------------------------------------
// (model, pixels [2 n]) -> directions [3 n], ok [n]: CameraModel::Unproject for all pixels in one b200ba_unproject call
using UnprojectMany = std::function<void(CameraModel&, const std::vector<double>&, std::vector<double>*, std::vector<int32_t>*)>;
// (model, grid points [2 n], directions [3 n], max_iteration_count): CentralGenericModel::FitToPixelDirectionsImpl
using FitGridPoints = std::function<void(CentralGenericModel&, const std::vector<double>&, const std::vector<double>&, int)>;

inline void UnprojectManyOnDevice(CameraModel& model, const std::vector<double>& pixels, std::vector<double>* directions,
                                  std::vector<int32_t>* ok) {
  const int64_t n = static_cast<int64_t>(pixels.size() / 2);
  b200ba_camera c{};
  c.model_type = static_cast<int32_t>(model.type());
  c.width = model.width();
  c.height = model.height();
  c.calibration_min_x = model.calibration_min_x();
  c.calibration_min_y = model.calibration_min_y();
  c.calibration_max_x = model.calibration_max_x();
  c.calibration_max_y = model.calibration_max_y();
  int rx = 0, ry = 0;
  if (model.GetGridResolution(&rx, &ry)) { c.grid_width = rx; c.grid_height = ry; }
  directions->assign(3 * n, 0.0);
  ok->assign(n, 0);
  if (n == 0) return;
  std::vector<double> origins(3 * n, 0.0);
  if (b200ba_unproject(-1, &c, model.flat_intrinsics().data(), n, pixels.data(), directions->data(), origins.data(), ok->data()) != 0)
    throw std::runtime_error(std::string("b200ba_unproject: ") + b200ba_last_error(nullptr));
}
inline void FitGridPointsOnDevice(CentralGenericModel& model, const std::vector<double>& grid_points,
                                  const std::vector<double>& directions, int max_iteration_count) {
  b200ba_fit_report rep;
  if (b200ba_fit_directions(-1, model.gw, model.gh, model.grid.data(), static_cast<int64_t>(grid_points.size() / 2),
                            grid_points.data(), directions.data(), max_iteration_count, &rep) != 0)
    throw std::runtime_error(std::string("b200ba_fit_directions: ") + b200ba_last_error(nullptr));
}

// central_grid.h:138-148 -- FLOAT arithmetic, like the reference
inline Vec2d GridPointToPixelCornerConv(float x, float y, int min_x, int min_y, int max_x, int max_y, int grid_width, int grid_height) {
  const float px = static_cast<float>(min_x) + ((x - 1.f) / (static_cast<float>(grid_width) - 3.f)) * static_cast<float>(max_x + 1 - min_x);
  const float py = static_cast<float>(min_y) + ((y - 1.f) / (static_cast<float>(grid_height) - 3.f)) * static_cast<float>(max_y + 1 - min_y);
  return Vec2d{px, py};
}

// calibration.cc:531-540: integer division, + 0.5f, + the exterior cells, truncated
inline void ComputeGridResolution(int calibration_area_width, int calibration_area_height, int exterior_cells_per_side,
                                  int approx_pixels_per_cell, int* resolution_x, int* resolution_y) {
  *resolution_x = static_cast<int>(static_cast<float>(calibration_area_width / approx_pixels_per_cell) + 0.5f + static_cast<float>(2 * exterior_cells_per_side));
  *resolution_y = static_cast<int>(static_cast<float>(calibration_area_height / approx_pixels_per_cell) + 0.5f + static_cast<float>(2 * exterior_cells_per_side));
}
// calibration.cc:566-569
inline void CalcGridResolutionForLevel(int pyramid_level, int full_resolution_x, int full_resolution_y, int* resolution_x,
                                       int* resolution_y) {
  const double factor = std::pow(1.333, -pyramid_level);
  *resolution_x = static_cast<int>(full_resolution_x * factor + 0.5f);
  *resolution_y = static_cast<int>(full_resolution_y * factor + 0.5f);
}
// calibration.cc:615-641: bounding rectangle of the truncated feature positions of one camera (used imagesets)
inline void ComputeIntegerBoundingRectForFeatures(const Dataset& dataset, int camera_index, const std::vector<bool>& image_used,
                                                  int* min_x, int* min_y, int* max_x, int* max_y) {
  *min_x = *min_y = 2147483647;
  *max_x = *max_y = 0;
  for (int i = 0; i < dataset.ImagesetCount(); ++i) {
    if (!image_used[i]) continue;
    for (const PointFeature& f : dataset.GetImageset(i)->FeaturesOfCamera(camera_index)) {
      const int x = static_cast<int>(f.xy.x), y = static_cast<int>(f.xy.y);
      *min_x = std::min(*min_x, x);
      *min_y = std::min(*min_y, y);
      *max_x = std::max(*max_x, x);
      *max_y = std::max(*max_y, y);
    }
  }
}

namespace detail {
inline bool is_nan3(const double* v) { return v[0] != v[0] || v[1] != v[1] || v[2] != v[2]; }
// libvis Image::InterpolateBilinear for 3-vectors (libvis/image.h:152-176): truncation, FLOAT weights
inline void interpolate_bilinear3(const double* image, int width, double x, double y, double* out) {
  const int ix = static_cast<int>(x), iy = static_cast<int>(y);
  const float fx = static_cast<float>(x - ix), fy = static_cast<float>(y - iy);
  const float fx_inv = 1.f - fx, fy_inv = 1.f - fy;
  const double w00 = fx_inv * fy_inv, w10 = fx * fy_inv, w01 = fx_inv * fy, w11 = fx * fy;
  for (int k = 0; k < 3; ++k)
    out[k] = w00 * image[3 * (static_cast<size_t>(iy) * width + ix) + k] + w10 * image[3 * (static_cast<size_t>(iy) * width + ix + 1) + k] +
             w01 * image[3 * (static_cast<size_t>(iy + 1) * width + ix) + k] + w11 * image[3 * (static_cast<size_t>(iy + 1) * width + ix + 1) + k];
}
}  // namespace detail

// central_generic.cc:267-422 -- dense [dh * dw * 3]: one direction per pixel, NaN where the source model is undefined.
// Initialises every control point from the closest valid pixel (search radius < 5), extrapolates the rest linearly from
// their neighbours (in place: the sweep order matters, like the reference), then fits the grid to the sub-sampled
// dense directions (on the device unless `fit` is given).
inline bool FitToDenseModel(CentralGenericModel* model, const std::vector<double>& dense, int dw, int dh, int subsample_step,
                            int max_iteration_count, const FitGridPoints& fit = FitGridPointsOnDevice) {
  const int gw = model->gw, gh = model->gh;
  const double scale_x = dw / static_cast<double>(model->width()), scale_y = dh / static_cast<double>(model->height());
  auto valid = [&](int x, int y) { return dense[3 * (static_cast<size_t>(y) * dw + x)] == dense[3 * (static_cast<size_t>(y) * dw + x)]; };
  const double nan = std::nan("");
  std::vector<double> grid(3 * static_cast<size_t>(gw) * gh, nan);
  auto take = [&](int gx, int gy, int x, int y) {
    for (int k = 0; k < 3; ++k) grid[3 * (static_cast<size_t>(gy) * gw + gx) + k] = dense[3 * (static_cast<size_t>(y) * dw + x) + k];
  };
  bool have_nan = false;
  for (int gy = 0; gy < gh; ++gy)
    for (int gx = 0; gx < gw; ++gx) {
      const Vec2d p = GridPointToPixelCornerConv(static_cast<float>(gx), static_cast<float>(gy), model->calibration_min_x(), model->calibration_min_y(),
                                                 model->calibration_max_x(), model->calibration_max_y(), gw, gh);
      const int cx = static_cast<int>(scale_x * p.x), cy = static_cast<int>(scale_y * p.y);
      if (cx < 0 || cy < 0 || cx >= dw || cy >= dh) { have_nan = true; continue; }
      if (valid(cx, cy)) { take(gx, gy, cx, cy); continue; }
      bool found = false;
      for (int radius = 1; radius < 5 && !found; ++radius) {
        const int min_x = cx - radius, min_y = cy - radius, max_x = cx + radius, max_y = cy + radius;
        for (int x = std::max(0, min_x); x <= std::min(dw - 1, max_x) && !found; ++x) {  // top and bottom
          if (min_y >= 0 && valid(x, min_y)) { take(gx, gy, x, min_y); found = true; }
          else if (max_y < dh && valid(x, max_y)) { take(gx, gy, x, max_y); found = true; }
        }
        for (int y = std::max(0, min_y); y <= std::min(dh - 1, max_y) && !found; ++y) {  // left and right
          if (min_x >= 0 && valid(min_x, y)) { take(gx, gy, min_x, y); found = true; }
          else if (max_x < dw && valid(max_x, y)) { take(gx, gy, max_x, y); found = true; }
        }
      }
      if (!found) have_nan = true;
    }
  for (int iteration = 0; have_nan && iteration < dw + dh; ++iteration) {
    have_nan = false;
    for (int gy = 0; gy < gh; ++gy)
      for (int gx = 0; gx < gw; ++gx) {
        double* g = &grid[3 * (static_cast<size_t>(gy) * gw + gx)];
        if (!detail::is_nan3(g)) continue;
        double total[3] = {0, 0, 0};
        int count = 0;
        const int steps[4][2] = {{0, 1}, {0, -1}, {1, 0}, {-1, 0}};
        for (const auto& st : steps) {
          const int nx1 = gx + st[0], ny1 = gy + st[1], nx2 = gx + 2 * st[0], ny2 = gy + 2 * st[1];
          if (nx2 < 0 || ny2 < 0 || nx2 >= gw || ny2 >= gh) continue;
          const double* v1 = &grid[3 * (static_cast<size_t>(ny1) * gw + nx1)];
          const double* v2 = &grid[3 * (static_cast<size_t>(ny2) * gw + nx2)];
          if (detail::is_nan3(v1) || detail::is_nan3(v2)) continue;
          for (int k = 0; k < 3; ++k) total[k] += v1[k] + (v1[k] - v2[k]);
          ++count;
        }
        if (count > 0) {
          const double norm = std::sqrt(total[0] * total[0] + total[1] * total[1] + total[2] * total[2]);
          for (int k = 0; k < 3; ++k) g[k] = total[k] / norm;
        } else {
          have_nan = true;
        }
      }
  }
  if (have_nan) return false;
  model->grid = grid;
  // samples: every subsample_step-th pixel of the calibrated area with a valid direction
  const double model_to_camera_x = static_cast<double>(model->width()) / dw, model_to_camera_y = static_cast<double>(model->height()) / dh;
  std::vector<double> grid_points, directions;
  for (int y = model->calibration_min_y(); y <= model->calibration_max_y(); y += subsample_step)
    for (int x = model->calibration_min_x(); x <= model->calibration_max_x(); x += subsample_step) {
      const int dx = static_cast<int>(scale_x * x), dy = static_cast<int>(scale_y * y);
      if (!valid(dx, dy)) continue;
      const Vec2d gp = model->PixelCornerConvToGridPoint(model_to_camera_x * (dx + 0.5f), model_to_camera_y * (dy + 0.5f));
      grid_points.push_back(gp.x);
      grid_points.push_back(gp.y);
      for (int k = 0; k < 3; ++k) directions.push_back(dense[3 * (static_cast<size_t>(dy) * dw + dx) + k]);
    }
  fit(*model, grid_points, directions, max_iteration_count);
  return true;
}

// calibration.cc:373-522 for the generic target models (the parametric targets are outside this path). Returns the new
// model, or an empty pointer where the reference returns false. camera_tr_rig is untouched for these targets.
//   * NoncentralGeneric -> NoncentralGeneric: both grids re-sampled bilinearly (:386-424), host only;
//   * central source: a dense direction image of the old model (one Unproject per pixel centre, on the device) is fitted
//     by a CentralGenericModel of the target resolution (FitToDenseModel(dense, step, 3), at most 300 x 300 samples),
//     optionally wrapped into a NoncentralGenericModel with zero origins.
inline std::shared_ptr<CameraModel> ResampleModel(CameraModel& model_to_optimize, int calibration_min_x, int calibration_min_y,
                                                  int calibration_max_x, int calibration_max_y, CameraModel::Type model_type,
                                                  int target_resolution_x, int target_resolution_y,
                                                  const UnprojectMany& unproject_many = UnprojectManyOnDevice,
                                                  const FitGridPoints& fit = FitGridPointsOnDevice) {
  using T = CameraModel::Type;
  const int w = model_to_optimize.width(), h = model_to_optimize.height();
  if (model_to_optimize.type() == T::NoncentralGeneric && model_type == T::NoncentralGeneric) {
    auto& old = static_cast<NoncentralGenericModel&>(model_to_optimize);
    const size_t old_n = static_cast<size_t>(old.gw) * old.gh;
    std::shared_ptr<NoncentralGenericModel> fresh(new NoncentralGenericModel(target_resolution_x, target_resolution_y, calibration_min_x,
                                                                             calibration_min_y, calibration_max_x, calibration_max_y, w, h));
    const size_t new_n = static_cast<size_t>(target_resolution_x) * target_resolution_y;
    for (int y = 0; y < target_resolution_y; ++y)
      for (int x = 0; x < target_resolution_x; ++x) {
        const Vec2d pixel = GridPointToPixelCornerConv(static_cast<float>(x), static_cast<float>(y), calibration_min_x, calibration_min_y,
                                                       calibration_max_x, calibration_max_y, target_resolution_x, target_resolution_y);
        // noncentral_generic.h:167-171 (double arithmetic with the float constant (grid - 3.f))
        double gx = 1.0 + static_cast<double>(old.gw - 3.f) * (pixel.x - old.calibration_min_x()) / (old.calibration_max_x() + 1 - old.calibration_min_x());
        double gy = 1.0 + static_cast<double>(old.gh - 3.f) * (pixel.y - old.calibration_min_y()) / (old.calibration_max_y() + 1 - old.calibration_min_y());
        gx = std::min(std::max(gx, 0.0), old.gw - 1.001);
        gy = std::min(std::max(gy, 0.0), old.gh - 1.001);
        const size_t o = static_cast<size_t>(y) * target_resolution_x + x;
        detail::interpolate_bilinear3(old.grids.data(), old.gw, gx, gy, &fresh->grids[3 * o]);                      // directions
        detail::interpolate_bilinear3(old.grids.data() + 3 * old_n, old.gw, gx, gy, &fresh->grids[3 * (new_n + o)]);  // line origins
      }
    return fresh;
  }
  if (model_to_optimize.type() == T::NoncentralGeneric) return nullptr;  // not implemented in the reference either (:426-429)
  if (model_type != T::CentralGeneric && model_type != T::NoncentralGeneric) return nullptr;
  // dense direction model of the old camera
  std::vector<double> pixels(2 * static_cast<size_t>(w) * h), directions;
  std::vector<int32_t> ok;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      pixels[2 * (static_cast<size_t>(y) * w + x)] = x + 0.5;
      pixels[2 * (static_cast<size_t>(y) * w + x) + 1] = y + 0.5;
    }
  unproject_many(model_to_optimize, pixels, &directions, &ok);
  if (directions.size() != 3 * ok.size() || ok.size() != static_cast<size_t>(w) * h) throw std::runtime_error("ResampleModel: un-projector returned a wrong size");
  for (size_t i = 0; i < ok.size(); ++i)
    if (!ok[i]) directions[3 * i] = directions[3 * i + 1] = directions[3 * i + 2] = std::nan("");
  const int area_w = calibration_max_x - calibration_min_x + 1, area_h = calibration_max_y - calibration_min_y + 1;
  const int subsample_step = std::max(1, std::min(area_w / 300, area_h / 300));  // std::round(int / int): already integral
  std::shared_ptr<CentralGenericModel> central(new CentralGenericModel(target_resolution_x, target_resolution_y, calibration_min_x,
                                                                       calibration_min_y, calibration_max_x, calibration_max_y, w, h));
  if (!FitToDenseModel(central.get(), directions, w, h, subsample_step, 3, fit)) return nullptr;
  if (model_type == T::NoncentralGeneric) {
    // noncentral_generic.cc:136-146: same directions, all line origins at the optical centre
    std::shared_ptr<NoncentralGenericModel> fresh(new NoncentralGenericModel(target_resolution_x, target_resolution_y, calibration_min_x,
                                                                             calibration_min_y, calibration_max_x, calibration_max_y, w, h));
    std::copy(central->grid.begin(), central->grid.end(), fresh->grids.begin());
    return fresh;
  }
  return central;
}

// calibration.cc:572-612: re-sample every camera whose grid resolution differs from the one wanted on this pyramid level,
// or whose type differs. Returns the number of re-sampled models.
inline int ResampleModelsIfNecessary(const Dataset& dataset, BAState* state, CameraModel::Type model_type, int approx_pixels_per_cell,
                                     int pyramid_level, const UnprojectMany& unproject_many = UnprojectManyOnDevice,
                                     const FitGridPoints& fit = FitGridPointsOnDevice) {
  int count = 0;
  for (int c = 0; c < dataset.num_cameras(); ++c) {
    CameraModel& model = *state->intrinsics[c];
    int loaded_x = 0, loaded_y = 0;
    const bool has_grid = model.GetGridResolution(&loaded_x, &loaded_y);
    const int exterior = has_grid ? 1 : 0;  // central_generic.h / noncentral_generic.h: exterior_cells_per_side() == 1
    int full_x, full_y, want_x, want_y;
    ComputeGridResolution(model.calibration_max_x() - model.calibration_min_x() + 1, model.calibration_max_y() - model.calibration_min_y() + 1,
                          exterior, approx_pixels_per_cell, &full_x, &full_y);
    CalcGridResolutionForLevel(pyramid_level, full_x, full_y, &want_x, &want_y);
    if ((has_grid && (loaded_x != want_x || loaded_y != want_y)) || model.type() != model_type) {
      std::shared_ptr<CameraModel> fresh = ResampleModel(model, model.calibration_min_x(), model.calibration_min_y(), model.calibration_max_x(),
                                                         model.calibration_max_y(), model_type, want_x, want_y, unproject_many, fit);
      if (fresh) {
        state->intrinsics[c] = fresh;
        ++count;
      }
    }
  }
  return count;
}

// ---- calibration report --------------------------------------------------------------------------------------
namespace detail {
// std::ostream << double with setprecision(14), except that NaN is always written "nan" (glibc writes "-nan"
// when the sign bit is set, e.g. for 0.0 / 0), so that the Python writer (io.py) produces the same bytes
inline std::string report_number(double v) {
  if (v != v) return "nan";
  std::ostringstream s;
  s << std::setprecision(14) << v;
  return s.str();
}
}  // namespace detail

// calibration_report.cc:648-710 -- <base>_info.txt. The reference takes the error vector and sorts it for the
// median; here the median comes in (b200ba_calibration_report computes it) and its line is written when there is
// at least one error. The average is sum / count (NaN without errors). Returns false if the file cannot be opened.
inline bool WriteReportInfoFile(const std::string& path, const CameraModel& cam, double horizontal_fov, double vertical_fov,
                                int imageset_count, int num_localized_images, int64_t reprojection_error_count,
                                double reprojection_error_sum, double reprojection_error_max, double reprojection_error_median,
                                double biasedness, double histogram_extent_in_px = 0.2f, double max_error_in_px = 0.5) {
  std::ofstream stream(path, std::ios::out);
  if (!stream) return false;
  using detail::report_number;
  stream << "resolution : " << cam.width() << " x " << cam.height() << "\n";
  if (horizontal_fov >= 0) stream << "horizontal_fov : " << report_number(180.f / M_PI * horizontal_fov) << "\n";
  if (vertical_fov >= 0) stream << "vertical_fov : " << report_number(180.f / M_PI * vertical_fov) << "\n";
  stream << "\n";
  stream << "num_localized_imagesets : " << num_localized_images << "\n";
  stream << "num_total_imagesets : " << imageset_count << "\n";
  stream << "\n";
  stream << "reprojection_error_count : " << reprojection_error_count << "\n";
  if (reprojection_error_count > 0) stream << "reprojection_error_median : " << report_number(reprojection_error_median) << "\n";
  const double average = reprojection_error_count > 0 ? reprojection_error_sum / static_cast<double>(reprojection_error_count) : std::nan("");
  stream << "reprojection_error_average : " << report_number(average) << "\n";
  stream << "reprojection_error_maximum : " << report_number(reprojection_error_max) << "\n";
  stream << "median_kl_divergence : " << report_number(biasedness) << "\n";
  stream << "\n";
  stream << "reprojection_error_histogram_visualization_half_extent_in_pixels : " << report_number(histogram_extent_in_px) << "\n";
  stream << "maximum_error_visualization_maximum_error_in_pixels : " << report_number(max_error_in_px) << "\n";
  return static_cast<bool>(stream);
}

// _errors_histogram.png (calibration_report.cc:744-755): count * 255.99f / max, truncated; all zero for an empty
// histogram (where the reference divides 0 by 0)
inline std::vector<uint8_t> HistogramImage(const b200ba_camera_report& r) {
  constexpr int kBins = B200BA_REPORT_HIST * B200BA_REPORT_HIST;
  std::vector<uint8_t> img(kBins, 0);
  double max_entry = 0;
  for (int i = 0; i < kBins; ++i) max_entry = std::max(max_entry, static_cast<double>(r.histogram[i]));
  if (max_entry > 0)
    for (int i = 0; i < kBins; ++i) img[i] = static_cast<uint8_t>(static_cast<int>(static_cast<double>(r.histogram[i]) * 255.99f / max_entry));
  return img;
}

// _grid_point_locations.png (calibration_report.cc:820-838): white at every control point's pixel, truncated with
// static_cast<int> (so (-1, 0) counts as 0); RGB [height * width * 3]
inline std::vector<uint8_t> GridPointLocationsImage(const CentralGenericModel& model) {
  std::vector<uint8_t> img(3 * static_cast<size_t>(model.width()) * model.height(), 0);
  int gw = 0, gh = 0;
  model.GetGridResolution(&gw, &gh);
  for (int y = 0; y < gh; ++y)
    for (int x = 0; x < gw; ++x) {
      const Vec2d p = GridPointToPixelCornerConv(static_cast<float>(x), static_cast<float>(y), model.calibration_min_x(),
                                                 model.calibration_min_y(), model.calibration_max_x(), model.calibration_max_y(), gw, gh);
      const int px = static_cast<int>(p.x), py = static_cast<int>(p.y);
      if (px >= 0 && py >= 0 && px < model.width() && py < model.height())
        for (int k = 0; k < 3; ++k) img[3 * (static_cast<size_t>(py) * model.width() + px) + k] = 255;
    }
  return img;
}

// calibration_report.cc:932-981 -- the three .obj models of a non-central camera from the n_obj lines
// [n_obj][4][3] point_a, point_b, closest point, origin of b200ba_line_offsets: <base>_line_visualization.obj (a - b),
// <base>_line_visualization_cutoff.obj (a - closest point) and <base>_line_visualization_origins.obj (a, b, origin;
// the segment a - b), each with its "v" lines followed by its "l" lines, numbers with setprecision(14) (NaN written
// "nan" as in report_number). io.py's WriteLineVisualizationOBJ writes the same bytes. Returns false if a file cannot
// be opened.
inline bool WriteLineVisualizationOBJ(const std::string& base_path, const double* obj_lines, int64_t n_obj) {
  std::ofstream obj_stream(base_path + "_line_visualization.obj", std::ios::out);
  std::ofstream obj_stream_cutoff(base_path + "_line_visualization_cutoff.obj", std::ios::out);
  std::ofstream obj_stream_origins(base_path + "_line_visualization_origins.obj", std::ios::out);
  if (!obj_stream || !obj_stream_cutoff || !obj_stream_origins) return false;
  using detail::report_number;
  auto v = [](const double* p) {
    return "v " + report_number(p[0]) + " " + report_number(p[1]) + " " + report_number(p[2]) + "\n";
  };
  for (int64_t i = 0; i < n_obj; ++i) {
    const double* line = obj_lines + 12 * i;
    obj_stream << v(line) << v(line + 3);
    obj_stream_cutoff << v(line) << v(line + 6);
    obj_stream_origins << v(line) << v(line + 3) << v(line + 9);
  }
  int64_t vertex_index = 1;  // vertex indexing starts at 1 in .obj files
  for (int64_t i = 0; i < n_obj; ++i) {
    obj_stream << "l " << vertex_index << " " << (vertex_index + 1) << "\n";
    obj_stream_cutoff << "l " << vertex_index << " " << (vertex_index + 1) << "\n";
    obj_stream_origins << "l " << (3 * (vertex_index / 2) + 1) << " " << (3 * (vertex_index / 2) + 2) << "\n";
    vertex_index += 2;
  }
  return static_cast<bool>(obj_stream) && static_cast<bool>(obj_stream_cutoff) && static_cast<bool>(obj_stream_origins);
}

// calibration_report.cc:83-98: the numbers of CreateCalibrationReportForCamera (:713-817) for every camera, computed
// in the library (b200ba_calibration_report) on the flattening that OptimizeJointly uses, and written to
// <report_base_path>_camera<i>_info.txt. With visualizations, every camera also gets the reference's images
// (b200ba_report_images): _observation_directions.png (central- and non-central-generic cameras; OpenCV cameras have
// no device un-projection), _errors_histogram.png, _error_directions.png, _error_magnitudes.png and, for
// central-generic cameras, _grid_point_locations.png. With line_offsets, every non-central camera also gets the
// centre-point analysis of :839-982 (b200ba_line_offsets): _line_offsets.png and the three _line_visualization*.obj
// models. Neither argument is modified. Returns the per-camera numbers; throws on a library error.
inline std::vector<b200ba_camera_report> CreateCalibrationReport(const Dataset& dataset, const BAState& state,
                                                                 const std::string& report_base_path,
                                                                 bool visualizations = false, bool line_offsets = false) {
  detail::Flat f;
  // flatten() only reads; it takes mutable references because flat_intrinsics() hands out the model's storage
  detail::flatten(const_cast<Dataset&>(dataset), const_cast<BAState*>(&state), &f);
  b200ba_problem pb{};
  pb.n_cameras = static_cast<int32_t>(f.cams.size());
  pb.cameras = f.cams.data();
  pb.n_imagesets = static_cast<int32_t>(f.used.size());
  pb.n_points = static_cast<int32_t>(state.points.size());
  pb.n_obs = static_cast<int64_t>(f.oi.size());
  pb.obs_imageset = f.oi.data();
  pb.obs_camera = f.oc.data();
  pb.obs_point = f.op.data();
  pb.obs_xy = f.oxy.data();
  b200ba_handle* h = nullptr;
  if (b200ba_create(&pb, -1, &h) != 0) throw std::runtime_error(std::string("b200ba_create: ") + b200ba_last_error(nullptr));
  b200ba_state st{f.points.data(), f.rtg.data(), f.ctr.data(), f.intr.data(), nullptr};
  std::vector<b200ba_camera_report> reports(f.cams.size());
  int rc = b200ba_set_state(h, &st);
  if (rc == 0) rc = b200ba_calibration_report(h, reports.data(), nullptr, nullptr);
  const std::string err = rc ? b200ba_last_error(h) : "";
  if (rc) {
    b200ba_destroy(h);
    throw std::runtime_error("b200ba_calibration_report: " + err);
  }
  for (size_t c = 0; visualizations && c < reports.size(); ++c) {
    const CameraModel& cam = *state.intrinsics[c];
    const size_t n = 3 * static_cast<size_t>(cam.width()) * cam.height();
    const bool generic = cam.type() == CameraModel::Type::CentralGeneric || cam.type() == CameraModel::Type::NoncentralGeneric;
    std::vector<uint8_t> dirs(generic ? n : 0), err_dir(n), err_mag(n);
    if (b200ba_report_images(h, static_cast<int32_t>(c), generic ? dirs.data() : nullptr, err_dir.data(), err_mag.data(),
                             nullptr, nullptr) != 0) {
      const std::string e = b200ba_last_error(h);
      b200ba_destroy(h);
      throw std::runtime_error("b200ba_report_images: " + e);
    }
    const std::string base = report_base_path + "_camera" + std::to_string(c);
    const std::filesystem::path parent = std::filesystem::path(base).parent_path();
    if (!parent.empty()) std::filesystem::create_directories(parent);
    bool ok = true;
    if (generic) ok = ok && WritePNG(base + "_observation_directions.png", cam.width(), cam.height(), 3, dirs.data());
    ok = ok && WritePNG(base + "_errors_histogram.png", B200BA_REPORT_HIST, B200BA_REPORT_HIST, 1, HistogramImage(reports[c]).data());
    ok = ok && WritePNG(base + "_error_directions.png", cam.width(), cam.height(), 3, err_dir.data());
    ok = ok && WritePNG(base + "_error_magnitudes.png", cam.width(), cam.height(), 3, err_mag.data());
    if (cam.type() == CameraModel::Type::CentralGeneric)
      ok = ok && WritePNG(base + "_grid_point_locations.png", cam.width(), cam.height(), 3,
                          GridPointLocationsImage(static_cast<const CentralGenericModel&>(cam)).data());
    if (!ok) {
      b200ba_destroy(h);
      throw std::runtime_error("CreateCalibrationReport: cannot write the images of " + base);
    }
  }
  b200ba_destroy(h);
  int num_localized = 0;
  for (bool used : state.image_used) num_localized += used ? 1 : 0;
  for (size_t c = 0; c < reports.size(); ++c) {
    const b200ba_camera_report& r = reports[c];
    const std::string path = report_base_path + "_camera" + std::to_string(c) + "_info.txt";
    const std::filesystem::path parent = std::filesystem::path(path).parent_path();
    if (!parent.empty()) std::filesystem::create_directories(parent);  // the reference's mkpath (:720-721)
    if (!WriteReportInfoFile(path, *state.intrinsics[c], r.horizontal_fov, r.vertical_fov, dataset.ImagesetCount(), num_localized,
                             r.reprojection_error_count, r.reprojection_error_sum, r.reprojection_error_max,
                             r.reprojection_error_median, r.biasedness))
      throw std::runtime_error("CreateCalibrationReport: cannot write " + path);
  }
  for (size_t c = 0; line_offsets && c < reports.size(); ++c) {
    const CameraModel& cam = *state.intrinsics[c];
    if (cam.type() != CameraModel::Type::NoncentralGeneric) continue;
    constexpr int kStepForOBJ = 20;  // :933
    const int rw = cam.calibration_max_x() - cam.calibration_min_x() + 1, rh = cam.calibration_max_y() - cam.calibration_min_y() + 1;
    int64_t n_obj = (rw >= 1 && rh >= 1) ? static_cast<int64_t>((rw - 1) / kStepForOBJ + 1) * ((rh - 1) / kStepForOBJ + 1) : 0;
    std::vector<uint8_t> image(3 * static_cast<size_t>(cam.width()) * cam.height());
    std::vector<double> obj(12 * static_cast<size_t>(std::max<int64_t>(n_obj, 1)));
    b200ba_line_offsets_report rep{};
    if (b200ba_line_offsets(-1, &f.cams[c], f.intr[c], &rep, image.data(), nullptr, kStepForOBJ, obj.data(), &n_obj,
                            nullptr) != 0)
      throw std::runtime_error(std::string("b200ba_line_offsets: ") + b200ba_last_error(nullptr));
    const std::string base = report_base_path + "_camera" + std::to_string(c);
    if (!WritePNG(base + "_line_offsets.png", cam.width(), cam.height(), 3, image.data()) ||
        !WriteLineVisualizationOBJ(base, obj.data(), n_obj))
      throw std::runtime_error("CreateCalibrationReport: cannot write the line-offset files of " + base);
  }
  return reports;
}

// ---- calibration from a state ----------------------------------------------------------------------------------
// RunBundleAdjustment (calibration.cc:187-304) as Calibrate runs it: one handle, the device-resident loop of
// b200ba_run_bundle_adjustment, the reference's "[i] Cost:" line on stderr and, with state_output_path, the state
// directory written after every iteration (the reference's checkpoint). Returns the cost after each iteration.
inline std::vector<double> RunBundleAdjustmentWithCheckpoints(SchurMode schur_mode, int max_iteration_count,
                                                              double cost_reduction_threshold, Dataset* dataset, BAState* state,
                                                              double regularization_weight, const char* state_output_path) {
  detail::Flat f;
  detail::flatten(*dataset, state, &f);
  b200ba_handle* h = detail::create_handle(f, state->points.size());
  b200ba_state st{f.points.data(), f.rtg.data(), f.ctr.data(), f.intr.data(), f.lastp.data()};
  b200ba_options opt;
  b200ba_default_options(&opt);
  opt.max_iteration_count = 1;
  opt.init_lambda = -1;             // calibration.cc:203
  opt.numerical_diff_delta = 1e-4;  // calibration.cc:201
  opt.regularization_weight = regularization_weight;
  opt.localize_only = 0;
  opt.eliminate_points = 0;  // the product passes false (calibration.cc:232)
  opt.schur_mode = static_cast<int32_t>(schur_mode);
  opt.print_progress = 0;
  struct Ctx {
    b200ba_handle* h;
    b200ba_state* st;
    detail::Flat* f;
    Dataset* dataset;
    BAState* state;
    const char* path;
    std::vector<double> costs;
    bool failed;
  } ctx{h, &st, &f, dataset, state, state_output_path, {}, false};
  auto on_iteration = [](void* user, int32_t iteration, double cost) -> int {
    Ctx* c = static_cast<Ctx*>(user);
    c->costs.push_back(cost);
    if (c->path) {
      if (b200ba_get_state(c->h, c->st) != 0) {
        c->failed = true;
        return 1;
      }
      detail::read_back(*c->f, c->dataset, c->state);
      SaveBAState(c->path, *c->state);
    }
    std::fprintf(stderr, "[%d] Cost: %g\n", iteration + 1, cost);
    return 0;
  };
  b200ba_ba_report rep;
  int rc = b200ba_set_state(h, &st);
  if (rc == 0) rc = b200ba_run_bundle_adjustment(h, &opt, max_iteration_count, cost_reduction_threshold, &rep, on_iteration, &ctx);
  if (rc == 0 && ctx.failed) rc = 1;
  if (rc == 0) rc = b200ba_get_state(h, &st);
  const std::string err = rc ? b200ba_last_error(h) : "";
  b200ba_destroy(h);
  if (rc) throw std::runtime_error("b200ba_run_bundle_adjustment: " + err);
  detail::read_back(f, dataset, state);
  return ctx.costs;
}

// (dataset, state, max_iteration_count, cost_reduction_threshold, state_output_path): one RunBundleAdjustment of Calibrate
using CalibrateBundleAdjustment = std::function<void(Dataset*, BAState*, int, double, const char*)>;
// (dataset, state, outlier_removal_factor, outlier_visualization_path): the outlier round of every camera
using CalibrateOutlierRound = std::function<void(Dataset*, BAState*, float, const char*)>;

namespace detail {
inline const char* model_type_name(CameraModel::Type t) {
  switch (t) {
    case CameraModel::Type::CentralGeneric: return "CentralGeneric";
    case CameraModel::Type::NoncentralGeneric: return "NoncentralGeneric";
    case CameraModel::Type::CentralRadial: return "CentralRadial";
    case CameraModel::Type::CentralThinPrismFisheye: return "CentralThinPrismFisheye";
    case CameraModel::Type::CentralOpenCV: return "CentralOpenCV";
    default: return "InvalidType";
  }
}
inline std::string resolution_text(int x, int y) { return "(" + std::to_string(x) + ", " + std::to_string(y) + ")"; }
}  // namespace detail

// Calibrate() (calibration.cc:918-1143) from a loaded state, with use_cuda = false as CalibrateBatch passes: the same
// schedule, messages and refusals as pipeline.Calibrate (its docstring lists them). The defaults of the hooks run every
// numerical step in the library: BA through RunBundleAdjustmentWithCheckpoints, the outlier round of every camera on one
// handle (detail::outlier_round), the resampling through b200ba_unproject / b200ba_fit_directions.
inline bool Calibrate(Dataset* dataset, BAState* state, CameraModel::Type model_type, int num_pyramid_levels = 3,
                      int approx_pixels_per_cell = 25, double regularization_weight = 0, float outlier_removal_factor = 6,
                      bool localize_only = false, SchurMode schur_mode = SchurMode::Dense,
                      const char* outlier_visualization_path = nullptr, const char* dataset_output_path = nullptr,
                      const char* state_output_path = nullptr, CalibrateBundleAdjustment run_bundle_adjustment = nullptr,
                      CalibrateOutlierRound outlier_round = nullptr, const UnprojectMany& unproject_many = UnprojectManyOnDevice,
                      const FitGridPoints& fit = FitGridPointsOnDevice) {
  using T = CameraModel::Type;
  if (dataset->ImagesetCount() < 3) {
    std::cerr << "Calibration failed: too few input images given (" << dataset->ImagesetCount()
              << "), calibration requires at least 3. (In practice, many more should be used.)" << std::endl;
    return false;
  }
  if (localize_only) {
    std::cerr << "Calibrate: localize_only needs the dense initialization's localization, which is not built here." << std::endl;
    return false;
  }
  for (int c = 0; c < state->num_cameras(); ++c) {
    const T type = state->intrinsics[c]->type();
    if (type == T::CentralOpenCV && model_type != T::CentralOpenCV) {
      std::cerr << "Calibrate: camera " << c << " is an OpenCV model and would have to be resampled into a generic model, "
                   "which needs an OpenCV un-projection on the device (not built)." << std::endl;
      return false;
    }
    if (type != model_type && model_type != T::CentralGeneric && model_type != T::NoncentralGeneric) {
      std::cerr << "Calibrate: camera " << c << " would have to be fitted by a " << detail::model_type_name(model_type)
                << " model; only the generic models are resampling targets here." << std::endl;
      return false;
    }
  }
  if (!run_bundle_adjustment)
    run_bundle_adjustment = [&](Dataset* ds, BAState* st, int max_iteration_count, double threshold, const char* path) {
      RunBundleAdjustmentWithCheckpoints(schur_mode, max_iteration_count, threshold, ds, st, regularization_weight, path);
    };
  if (!outlier_round)
    outlier_round = [](Dataset* ds, BAState* st, float factor, const char* path) {
      std::vector<int> cameras(st->num_cameras());
      for (int c = 0; c < st->num_cameras(); ++c) cameras[c] = c;
      detail::outlier_round(cameras, ds, st, factor, path);
    };
  ResampleModelsIfNecessary(*dataset, state, model_type, approx_pixels_per_cell, num_pyramid_levels - 1, unproject_many, fit);
  state->ComputeFeatureIdToPointsIndex(dataset);
  const int nc = state->num_cameras();
  std::vector<int> full_x(nc, -1), full_y(nc, -1);
  for (int c = 0; c < nc; ++c) {
    const CameraModel& m = *state->intrinsics[c];
    int rx, ry;
    if (m.GetGridResolution(&rx, &ry))
      ComputeGridResolution(m.calibration_max_x() - m.calibration_min_x() + 1, m.calibration_max_y() - m.calibration_min_y() + 1, 1,
                            approx_pixels_per_cell, &full_x[c], &full_y[c]);
  }
  for (int level = num_pyramid_levels - 1; level > 0; --level) {
    std::cerr << "Bundle adjustment with pyramid level: " << level << std::endl;
    for (int c = 0; c < nc; ++c) {
      if (full_x[c] < 0) {
        std::cerr << "Calibrate: camera " << c << " has a model without a grid, which the pyramid scheme needs; set "
                     "num_pyramid_levels to 1." << std::endl;
        return false;
      }
      int want_x, want_y, rx = 0, ry = 0;
      CalcGridResolutionForLevel(level, full_x[c], full_y[c], &want_x, &want_y);
      state->intrinsics[c]->GetGridResolution(&rx, &ry);
      if (rx != want_x || ry != want_y) {
        std::cerr << "Calibrate: camera " << c << " has grid resolution " << detail::resolution_text(rx, ry) << " on pyramid level "
                  << level << ", not " << detail::resolution_text(want_x, want_y) << " (a resampling failed)." << std::endl;
        return false;
      }
      std::cerr << "Grid resolution on pyramid level " << level << " for camera " << c << ": " << want_x << " x " << want_y << std::endl;
    }
    run_bundle_adjustment(dataset, state, 10, 1e-4, state_output_path);
    run_bundle_adjustment(dataset, state, 50, 1.0, state_output_path);
    for (int c = 0; c < nc; ++c) {
      CameraModel& model = *state->intrinsics[c];
      int target_x, target_y;
      CalcGridResolutionForLevel(level - 1, full_x[c], full_y[c], &target_x, &target_y);
      std::shared_ptr<CameraModel> fresh = ResampleModel(model, model.calibration_min_x(), model.calibration_min_y(),
                                                         model.calibration_max_x(), model.calibration_max_y(), model_type,
                                                         target_x, target_y, unproject_many, fit);
      if (fresh) state->intrinsics[c] = fresh;
    }
  }
  for (int c = 0; c < nc; ++c) {
    if (full_x[c] < 0) continue;
    int rx = 0, ry = 0;
    state->intrinsics[c]->GetGridResolution(&rx, &ry);
    if (rx != full_x[c] || ry != full_y[c]) {
      std::cerr << "Calibrate: camera " << c << " has grid resolution " << detail::resolution_text(rx, ry) << ", not "
                << detail::resolution_text(full_x[c], full_y[c]) << " (a resampling failed)." << std::endl;
      return false;
    }
    std::cerr << "Bundle adjustment with final grid resolution for camera " << c << ": " << full_x[c] << " x " << full_y[c]
              << " ..." << std::endl;
  }
  if (outlier_removal_factor > 0) {
    run_bundle_adjustment(dataset, state, num_pyramid_levels == 1 ? 100 : 10, 1e-4, state_output_path);
    outlier_round(dataset, state, outlier_removal_factor, outlier_visualization_path);
    if (dataset_output_path) SaveDataset(dataset_output_path, *dataset);
  }
  run_bundle_adjustment(dataset, state, 100, 1e-4, state_output_path);
  try {
    ScaleToMetric(*dataset, state);
  } catch (const std::runtime_error&) {
    std::cerr << "Calibrate: ScaleToMetric: no neighbouring corners with known geometry (the reference divides by zero here)"
              << std::endl;
    return false;
  }
  return true;
}

// CalibrateBatch's dataset-file path (calibration.cc:1272-1334) from a state directory, like pipeline.CalibrateFromState
// (same messages, same files): load and merge dataset_files in order, load the state, Calibrate with the checkpoint in
// output_directory, then write output_directory's state, dataset.bin and the report (visualizations and line offsets;
// the outlier images share its base path). model_type in the reference's flag spelling: central_generic,
// noncentral_generic or central_opencv. Returns EXIT_SUCCESS / EXIT_FAILURE; on failure no final state is written.
inline int CalibrateFromState(const std::vector<std::string>& dataset_files, const std::string& state_directory,
                              const std::string& output_directory, const std::string& model_type = "central_generic",
                              int num_pyramid_levels = 3, int cell_length_in_pixels = 25, double regularization_weight = 0,
                              float outlier_removal_factor = 6, SchurMode schur_mode = SchurMode::Dense) {
  using T = CameraModel::Type;
  T type;
  if (model_type == "central_generic") type = T::CentralGeneric;
  else if (model_type == "noncentral_generic") type = T::NoncentralGeneric;
  else if (model_type == "central_opencv") type = T::CentralOpenCV;
  else {
    std::cerr << "Model type not handled: " << model_type << std::endl;
    return EXIT_FAILURE;
  }
  if (dataset_files.empty()) {
    std::cerr << "CalibrateFromState needs at least one dataset file" << std::endl;
    return EXIT_FAILURE;
  }
  std::shared_ptr<Dataset> dataset;
  for (size_t i = 0; i < dataset_files.size(); ++i) {
    std::cerr << "Dataset " << i << ": " << dataset_files[i] << std::endl;
    std::shared_ptr<Dataset> ds;
    if (!LoadDataset(dataset_files[i].c_str(), &ds)) {
      std::cerr << "Cannot read file: " << dataset_files[i] << std::endl;
      return EXIT_FAILURE;
    }
    if (!dataset) {
      dataset = ds;
    } else if (!dataset->Merge(*ds)) {
      std::cerr << "Cannot merge dataset " << dataset_files[i] << ": its camera count or image sizes differ" << std::endl;
      return EXIT_FAILURE;
    }
  }
  BAState state;
  if (!LoadBAState(state_directory.c_str(), &state, nullptr)) {
    std::cerr << "Cannot load state: " << state_directory << std::endl;
    return EXIT_FAILURE;
  }
  if (state.num_cameras() != dataset->num_cameras() || static_cast<int>(state.image_used.size()) != dataset->ImagesetCount()) {
    std::cerr << "The state in " << state_directory << " has " << state.num_cameras() << " cameras and " << state.image_used.size()
              << " imagesets, the dataset " << dataset->num_cameras() << " and " << dataset->ImagesetCount() << "." << std::endl;
    return EXIT_FAILURE;
  }
  const std::string report_base = (std::filesystem::path(output_directory) / "report").string();
  const std::string dataset_path = (std::filesystem::path(output_directory) / "dataset.bin").string();
  if (!Calibrate(dataset.get(), &state, type, num_pyramid_levels, cell_length_in_pixels, regularization_weight,
                 outlier_removal_factor, false, schur_mode, report_base.c_str(), dataset_path.c_str(), output_directory.c_str())) {
    std::cerr << "Calibration failed." << std::endl;
    return EXIT_FAILURE;
  }
  if (!SaveBAState(output_directory.c_str(), state)) {
    std::cerr << "Cannot write the state to: " << output_directory << std::endl;
    return EXIT_FAILURE;
  }
  SaveDataset(dataset_path.c_str(), *dataset);
  CreateCalibrationReport(*dataset, state, report_base, true, true);
  return EXIT_SUCCESS;
}

// ---- comparison of two calibrations ----------------------------------------------------------------------------
// fitting_report.h:186-200 -- <base>_fitting_info.txt. The reference sorts its error vector for the median; here the
// median comes in (b200ba_compare_models computes it) and its line is written when there is at least one error. The
// average is sum / count (NaN without errors). Returns false if the file cannot be opened.
inline bool WriteFittingInfoFile(const std::string& path, const b200ba_fitting_report& report) {
  std::ofstream stream(path, std::ios::out);
  if (!stream) return false;
  using detail::report_number;
  const int64_t count = report.reprojection_error_count;
  if (count > 0) stream << "median_reprojection_error : " << report_number(report.reprojection_error_median) << "\n";
  const double average = count > 0 ? report.reprojection_error_sum / static_cast<double>(count) : std::nan("");
  stream << "average_reprojection_error : " << report_number(average) << "\n";
  stream << "maximum_reprojection_error : " << report_number(report.reprojection_error_max) << "\n";
  stream << "error_magnitude_visualization_max_error_norm : " << report_number(report.max_error_norm) << "\n";
  stream << "error_direction_visualization_max_error_component : " << report_number(report.max_error_component) << "\n";
  return static_cast<bool>(stream);
}

// tools/compare_calibrations.cc:39-74: load both models, compare them in the library (b200ba_compare_models:
// CreateFittingErrorReport with base = A, fitted = B, rotation Identity) and write <report_base_path>_fitting_info.txt.
// With visualizations, the comparison is b200ba_fitting_images and its five images are written first, in the
// reference's order (fitting_report.h:180-184): _fitting_error_magnitudes.png, _fitting_error_direction_angles.png,
// _fitting_error_directions.png, _fitting_error_reprojection_magnitudes.png, _fitting_error_reprojections.png. The
// Python pipeline writes the same bytes. Returns EXIT_SUCCESS / EXIT_FAILURE with the reference's messages on stderr.
// Where the reference aborts on models of different image sizes (fitting_report.h:65-66), and where a file cannot be
// written, this returns EXIT_FAILURE. Throws on a library error.
inline int CompareCalibrations(const std::string& calibration_a, const std::string& calibration_b,
                               const std::string& report_base_path, bool visualizations = false) {
  if (calibration_a.empty() || calibration_b.empty() || report_base_path.empty()) {
    std::cerr << "For calibration comparison (--compare_calibrations), the input calibrations must be given with "
                 "--calibration_a and --calibration_b, and the output base path with --report_base_path.\n";
    return EXIT_FAILURE;
  }
  std::shared_ptr<CameraModel> model_a = LoadCameraModel(calibration_a.c_str());
  if (!model_a) {
    std::cerr << "Cannot load file: " << calibration_a << "\n";
    return EXIT_FAILURE;
  }
  std::shared_ptr<CameraModel> model_b = LoadCameraModel(calibration_b.c_str());
  if (!model_b) {
    std::cerr << "Cannot load file: " << calibration_b << "\n";
    return EXIT_FAILURE;
  }
  auto* a = dynamic_cast<CentralGenericModel*>(model_a.get());
  auto* b = dynamic_cast<CentralGenericModel*>(model_b.get());
  if (!a || !b) {
    std::cerr << "Calibration comparison is only implemented for CentralGenericModel at the moment.\n";
    return EXIT_FAILURE;
  }
  if (a->width() != b->width() || a->height() != b->height()) {
    std::cerr << "The calibrations differ in image size (" << a->width() << " x " << a->height() << " against "
              << b->width() << " x " << b->height() << ").\n";
    return EXIT_FAILURE;
  }
  const std::filesystem::path parent = std::filesystem::path(report_base_path).parent_path();
  if (!parent.empty()) std::filesystem::create_directories(parent);  // QFileInfo(base_path).dir().mkpath(".")
  auto camera = [](const CentralGenericModel& m) {
    b200ba_camera c{};
    c.model_type = B200BA_MODEL_CENTRAL_GENERIC;
    c.width = m.width();
    c.height = m.height();
    c.calibration_min_x = m.calibration_min_x();
    c.calibration_min_y = m.calibration_min_y();
    c.calibration_max_x = m.calibration_max_x();
    c.calibration_max_y = m.calibration_max_y();
    c.grid_width = m.gw;
    c.grid_height = m.gh;
    return c;
  };
  const b200ba_camera cam_a = camera(*a), cam_b = camera(*b);
  b200ba_fitting_report report{};
  if (visualizations) {
    const size_t n = static_cast<size_t>(a->width()) * a->height();
    std::vector<uint8_t> magnitudes(n), angles(3 * n), directions(3 * n), rep_magnitudes(n), reprojections(3 * n);
    if (b200ba_fitting_images(-1, &cam_a, a->grid.data(), &cam_b, b->grid.data(), &report, magnitudes.data(),
                              angles.data(), directions.data(), rep_magnitudes.data(), reprojections.data(),
                              nullptr) != 0)
      throw std::runtime_error(std::string("b200ba_fitting_images: ") + b200ba_last_error(nullptr));
    const std::pair<const char*, const std::vector<uint8_t>*> images[5] = {
        {"_fitting_error_magnitudes.png", &magnitudes},
        {"_fitting_error_direction_angles.png", &angles},
        {"_fitting_error_directions.png", &directions},
        {"_fitting_error_reprojection_magnitudes.png", &rep_magnitudes},
        {"_fitting_error_reprojections.png", &reprojections}};
    for (const auto& image : images) {
      const std::string png = report_base_path + image.first;
      if (!WritePNG(png, a->width(), a->height(), static_cast<int>(image.second->size() / n), image.second->data())) {
        std::cerr << "Cannot write file: " << png << "\n";
        return EXIT_FAILURE;
      }
    }
  } else if (b200ba_compare_models(-1, &cam_a, a->grid.data(), &cam_b, b->grid.data(), &report, nullptr, nullptr,
                                   nullptr) != 0) {
    throw std::runtime_error(std::string("b200ba_compare_models: ") + b200ba_last_error(nullptr));
  }
  const std::string path = report_base_path + "_fitting_info.txt";
  if (!WriteFittingInfoFile(path, report)) {
    std::cerr << "Cannot write file: " << path << "\n";
    return EXIT_FAILURE;
  }
  return EXIT_SUCCESS;
}

// ---- localization accuracy test ---------------------------------------------------------------------------------
// tools/localization_accuracy_test.cc:47-131: load both models, run b200ba_localization_accuracy (`trials` pose fits of
// one seeded random stream; the reference seeds with the time) and print "Average error [mm]" and "Median error [mm]"
// with std::ostream's default 6 significant digits, like the reference's LOG(INFO). Returns EXIT_SUCCESS /
// EXIT_FAILURE with the reference's messages on stderr; models that are not central-generic are refused with
// EXIT_FAILURE (the reference never ends for a non-central model). Throws on a library error.
inline int LocalizationAccuracyTest(const std::string& gt_model_yaml_path, const std::string& compared_model_yaml_path,
                                    int64_t trials = 10000, uint64_t seed = 0) {
  std::shared_ptr<CameraModel> gt_model = LoadCameraModel(gt_model_yaml_path.c_str());
  if (!gt_model) {
    std::cerr << "Cannot load ground truth camera model: " << gt_model_yaml_path << "\n";
    return EXIT_FAILURE;
  }
  std::shared_ptr<CameraModel> compared_model = LoadCameraModel(compared_model_yaml_path.c_str());
  if (!compared_model) {
    std::cerr << "Cannot load camera model to compare: " << compared_model_yaml_path << "\n";
    return EXIT_FAILURE;
  }
  if (gt_model->width() != compared_model->width() || gt_model->height() != compared_model->height()) {
    std::cerr << "The ground truth and compared camera models do not have the same image size.\n";
    return EXIT_FAILURE;
  }
  auto* gt = dynamic_cast<CentralGenericModel*>(gt_model.get());
  auto* compared = dynamic_cast<CentralGenericModel*>(compared_model.get());
  if (!gt || !compared) {
    std::cerr << "The localization accuracy test is only implemented for CentralGenericModel.\n";
    return EXIT_FAILURE;
  }
  auto camera = [](const CentralGenericModel& m) {
    b200ba_camera c{};
    c.model_type = B200BA_MODEL_CENTRAL_GENERIC;
    c.width = m.width();
    c.height = m.height();
    c.calibration_min_x = m.calibration_min_x();
    c.calibration_min_y = m.calibration_min_y();
    c.calibration_max_x = m.calibration_max_x();
    c.calibration_max_y = m.calibration_max_y();
    c.grid_width = m.gw;
    c.grid_height = m.gh;
    return c;
  };
  const b200ba_camera gt_cam = camera(*gt), cam = camera(*compared);
  b200ba_localization_report report{};
  if (b200ba_localization_accuracy(-1, &gt_cam, gt->grid.data(), &cam, compared->grid.data(), trials, seed, &report,
                                   nullptr, nullptr, nullptr, nullptr) != 0)
    throw std::runtime_error(std::string("b200ba_localization_accuracy: ") + b200ba_last_error(nullptr));
  std::cout << "Average error [mm]: " << (1000 * report.average_error) << "\n";
  std::cout << "Median error [mm]: " << (1000 * report.median_error) << "\n";
  std::cout.flush();
  return EXIT_SUCCESS;
}

// ---- --bundle_adjustment and --compare_reconstructions (tools/bundle_adjustment.cc) --------------------------------
// :50-220: load <state_directory>/intrinsics0.yaml and the COLMAP text model (LoadColmapProblem), run
// max_iteration_count single LM iterations (localize_only, eliminate_points, dense Schur mode) and write the state
// directory and cost.txt (14 significant digits) after every iteration. Returns EXIT_SUCCESS / EXIT_FAILURE; throws on
// a library error. pipeline.BundleAdjustment is the Python mirror.
inline int BundleAdjustment(const std::string& state_directory, const std::string& model_input_directory,
                            const std::string& model_output_directory, int max_iteration_count = 30) {
  std::shared_ptr<CameraModel> model = LoadCameraModel(io_detail::join(state_directory, "intrinsics0.yaml").c_str());
  if (!model) return EXIT_FAILURE;
  std::shared_ptr<Dataset> dataset;
  BAState state;
  if (!LoadColmapProblem(model, model_input_directory, &dataset, &state)) return EXIT_FAILURE;
  double lambda = -1;
  for (int iteration = 0; iteration < max_iteration_count; ++iteration) {
    const double cost = OptimizeJointly(*dataset, &state, 1, lambda, 1e-4, 0, true, true, SchurMode::Dense, &lambda,
                                        nullptr, false, false, false, false, false, /*print_progress*/ false);
    SaveBAState(model_output_directory.c_str(), state);
    io_detail::write_file(io_detail::join(model_output_directory, "cost.txt"), io_detail::num(cost) + "\n");
  }
  return EXIT_SUCCESS;
}

// The MeshLab project's paths (:327-372) on the bytes of the two path strings: the project's directory is their
// longest common prefix cut back to its last '/'; rest_k is path_k from the first differing byte on (empty when one
// path is a prefix of the other); a mesh file is absolute(path_k) + '/' + name, without a second '/' after a trailing
// one, absolute() prefixing the working directory + '/' to a relative path without normalising it.
struct MeshLabProjectPaths {
  std::string project, rest1, rest2;
  std::string files[4];  // points 1, poses 1, points 2, poses 2
};
inline MeshLabProjectPaths ReconstructionProjectPaths(const std::string& path1, const std::string& path2,
                                                      const std::string& cwd) {
  MeshLabProjectPaths r;
  size_t n = 0;
  while (n < std::min(path1.size(), path2.size()) && path1[n] == path2[n]) ++n;
  if (n < std::min(path1.size(), path2.size())) {
    r.rest1 = path1.substr(n);
    r.rest2 = path2.substr(n);
  }
  const size_t cut = path1.substr(0, n).rfind('/');
  r.project = (cut == std::string::npos ? std::string() : path1.substr(0, cut + 1)) + "reconstructions_aligned_at_start.mlp";
  const std::string* paths[2] = {&path1, &path2};
  for (int k = 0; k < 2; ++k) {
    const std::string absolute = (!paths[k]->empty() && (*paths[k])[0] == '/') ? *paths[k] : io_detail::join(cwd, *paths[k]);
    r.files[2 * k] = io_detail::join(absolute, "points.yaml.obj");
    r.files[2 * k + 1] = io_detail::join(absolute, "rig_tr_global.yaml.obj");
  }
  return r;
}

// :223-392: load both state directories, compare them on the device (b200ba_compare_reconstructions, every
// pixel_step-th pixel), print "intrinsics1_r_intrinsics2_4x4:", four rows of %.6g values separated by single spaces and
// "relative endpoint difference: <%.6g of 100 rel>%" to stdout, and write reconstructions_aligned_at_start.mlp.
// Returns EXIT_SUCCESS, also when the project cannot be written (a message on stderr, as in the reference), and
// EXIT_FAILURE with a message on stderr where a state does not load, the states differ in image count, camera count
// or image size (the reference aborts), or the library refuses them (return codes 2 and 4). pipeline.py's
// CompareReconstructions prints and writes the same bytes.
inline int CompareReconstructions(const std::string& reconstruction_path_1, const std::string& reconstruction_path_2,
                                  int pixel_step = 10) {
  BAState states[2];
  const std::string* paths[2] = {&reconstruction_path_1, &reconstruction_path_2};
  for (int k = 0; k < 2; ++k) {
    if (!LoadBAState(paths[k]->c_str(), &states[k], nullptr)) {
      std::cerr << "Cannot load reconstruction: " << *paths[k] << "\n";
      return EXIT_FAILURE;
    }
  }
  const BAState& s1 = states[0];
  const BAState& s2 = states[1];
  if (s1.rig_tr_global.size() != s2.rig_tr_global.size()) {
    std::cerr << "The reconstructions differ in image count (" << s1.rig_tr_global.size() << " against "
              << s2.rig_tr_global.size() << ").\n";
    return EXIT_FAILURE;
  }
  if (s1.intrinsics.size() != 1 || s2.intrinsics.size() != 1) {
    std::cerr << "Reconstruction comparison needs exactly one camera in each reconstruction.\n";
    return EXIT_FAILURE;
  }
  CameraModel& m1 = *s1.intrinsics[0];
  CameraModel& m2 = *s2.intrinsics[0];
  if (m1.width() != m2.width() || m1.height() != m2.height()) {
    std::cerr << "The cameras differ in image size (" << m1.width() << " x " << m1.height() << " against "
              << m2.width() << " x " << m2.height() << ").\n";
    return EXIT_FAILURE;
  }
  auto camera = [](CameraModel& m) {
    b200ba_camera c{};
    c.model_type = static_cast<int32_t>(m.type());
    c.width = m.width();
    c.height = m.height();
    c.calibration_min_x = m.calibration_min_x();
    c.calibration_min_y = m.calibration_min_y();
    c.calibration_max_x = m.calibration_max_x();
    c.calibration_max_y = m.calibration_max_y();
    int rx = 0, ry = 0;
    if (m.GetGridResolution(&rx, &ry)) {
      c.grid_width = rx;
      c.grid_height = ry;
    }
    return c;
  };
  auto flat = [](const std::vector<SE3d>& poses) {
    std::vector<double> v;
    for (const SE3d& T : poses) v.insert(v.end(), {T.qw, T.qx, T.qy, T.qz, T.tx, T.ty, T.tz});
    return v;
  };
  const b200ba_camera c1 = camera(m1), c2 = camera(m2);
  const std::vector<double> rtg1 = flat(s1.rig_tr_global), ctr1 = flat({s1.camera_tr_rig.at(0)});
  const std::vector<double> rtg2 = flat(s2.rig_tr_global), ctr2 = flat({s2.camera_tr_rig.at(0)});
  b200ba_reconstruction_comparison r{};
  const int rc = b200ba_compare_reconstructions(-1, &c1, m1.flat_intrinsics().data(), &c2, m2.flat_intrinsics().data(),
                                                static_cast<int32_t>(s1.rig_tr_global.size()), rtg1.data(), ctr1.data(),
                                                rtg2.data(), ctr2.data(), pixel_step, &r, nullptr);
  if (rc != 0) {
    std::cerr << "libb200ba error " << rc << ": " << b200ba_last_error(nullptr) << "\n";
    return EXIT_FAILURE;
  }
  std::string out = "intrinsics1_r_intrinsics2_4x4:\n";
  for (int row = 0; row < 4; ++row) {
    for (int col = 0; col < 4; ++col) {
      const double v = (row < 3 && col < 3) ? r.intrinsics1_r_intrinsics2[3 * row + col] : (row == col ? 1.0 : 0.0);
      char buf[64];
      std::snprintf(buf, sizeof(buf), col ? " %.6g" : "%.6g", v);
      out += buf;
    }
    out += "\n";
  }
  char buf[96];
  std::snprintf(buf, sizeof(buf), "relative endpoint difference: %.6g%%\n", 100 * r.relative_endpoint_difference);
  out += buf;
  std::cout << out;
  std::cout.flush();
  const MeshLabProjectPaths p = ReconstructionProjectPaths(reconstruction_path_1, reconstruction_path_2,
                                                           std::filesystem::current_path().string());
  std::vector<MeshLabMesh> meshes(4);
  const char* labels[4] = {"SfM cloud 1: ", "SfM camera poses 1: ", "SfM cloud 2: ", "SfM camera poses 2: "};
  for (int k = 0; k < 4; ++k) {
    meshes[k].label = labels[k] + (k < 2 ? p.rest1 : p.rest2);
    meshes[k].filename = p.files[k];
    for (int e = 0; e < 16; ++e)
      meshes[k].global_tr_mesh[e] = k < 2 ? (e == 15 ? 1.0 : (e % 5 == 0 ? r.scale : 0.0)) : r.firstimage1_tr_firstimage2[e];
  }
  if (!WriteMeshLabProject(p.project, meshes))
    std::cerr << "Failed to save MeshLab project to: " << p.project << "\n";
  return EXIT_SUCCESS;
}

// ---- --visualize_kalibr_calibration, --visualize_colmap_calibration and --create_legends -----------------------------
// VisualizeCameraModel(camera, path) (tools/visualize_calibration.cc:39-96): the image of b200ba_visualize_camera written
// as PNG. A camera the library refuses (return code 2: a size below 1, fx or fy 0, a parameter that is not finite) is
// skipped with a message; EXIT_FAILURE where the file cannot be written; throws on another library error.
inline int VisualizeCameraToFile(const std::string& name, int width, int height, const double params[8],
                                 const std::string& path) {
  std::vector<uint8_t> image(width > 0 && height > 0 ? 3 * static_cast<size_t>(width) * height : 0);
  const int rc = b200ba_visualize_camera(-1, width, height, params, image.data(), nullptr, nullptr, nullptr);
  if (rc == 2) {
    std::cerr << "Camera " << name << " skipped: " << b200ba_last_error(nullptr) << "\n";
    return EXIT_SUCCESS;
  }
  if (rc != 0) throw std::runtime_error(std::string("b200ba_visualize_camera: ") + b200ba_last_error(nullptr));
  if (!WritePNG(path, width, height, 3, image.data())) {
    std::cerr << "Cannot write file: " << path << "\n";
    return EXIT_FAILURE;
  }
  return EXIT_SUCCESS;
}

// tools/visualize_calibration.cc:98-165: for cam0, cam1, ... of the camchain up to the first missing key
// (ReadKalibrCamchain), the observation directions of every pinhole-radtan camera in their canonical orientation
// written to <camchain_path>.camN.png; other cameras are skipped with the reference's messages ("Camera model not
// handled: ...", "Distortion model not handled: ..."), and so are cameras without a resolution, 4 distortion
// coefficients and 4 intrinsics; messages go to stderr in file order. Kalibr's pixel-centre cu, cv are used as
// pixel-corner values, as the reference uses them. Returns EXIT_SUCCESS, or EXIT_FAILURE with "Cannot read file: ..."
// where the file cannot be read or parsed, or where a PNG cannot be written. pipeline.py's VisualizeKalibrCalibration
// prints and writes the same bytes.
inline int VisualizeKalibrCalibration(const std::string& camchain_path) {
  std::vector<KalibrCamera> cameras;
  if (!ReadKalibrCamchain(camchain_path, &cameras)) {
    std::cerr << "Cannot read file: " << camchain_path << "\n";
    return EXIT_FAILURE;
  }
  for (const KalibrCamera& cam : cameras) {
    if (cam.camera_model != "pinhole") {
      std::cerr << "Camera model not handled: " << cam.camera_model << "\n";
      continue;
    }
    if (cam.distortion_model != "radtan") {
      std::cerr << "Distortion model not handled: " << cam.distortion_model << "\n";
      continue;
    }
    int width = 0, height = 0;
    double params[8];
    if (!KalibrRadtanParameters(cam, &width, &height, params)) {
      std::cerr << "Camera " << cam.name << " skipped: it needs a resolution, 4 distortion coefficients and 4 intrinsics\n";
      continue;
    }
    if (VisualizeCameraToFile(cam.name, width, height, params, camchain_path + "." + cam.name + ".png") != EXIT_SUCCESS)
      return EXIT_FAILURE;
  }
  return EXIT_SUCCESS;
}

// tools/visualize_calibration.cc:167-207: for every camera of a COLMAP cameras.txt (ReadColmapCameras, file order), the
// observation directions of every OPENCV camera in their canonical orientation written to <cameras_path>.cam<id>.png;
// other models are skipped with "Camera model not handled: ...", and so are cameras with fewer than 8 parameters;
// messages go to stderr in file order. Returns EXIT_SUCCESS, or EXIT_FAILURE with "Cannot read file: ..." or where a
// PNG cannot be written. pipeline.py's VisualizeColmapCalibration prints and writes the same bytes.
inline int VisualizeColmapCalibration(const std::string& cameras_path) {
  std::vector<ColmapCamera> cameras;
  if (!ReadColmapCameras(cameras_path, &cameras)) {
    std::cerr << "Cannot read file: " << cameras_path << "\n";
    return EXIT_FAILURE;
  }
  for (const ColmapCamera& cam : cameras) {
    const std::string name = "cam" + std::to_string(cam.camera_id);
    if (cam.model_name != "OPENCV") {
      std::cerr << "Camera model not handled: " << cam.model_name << "\n";
      continue;
    }
    double params[8];
    if (!ColmapRadtanParameters(cam, params)) {
      std::cerr << "Camera " << name << " skipped: OPENCV needs 8 parameters, the file gives " << cam.parameters.size()
                << "\n";
      continue;
    }
    if (VisualizeCameraToFile(name, cam.width, cam.height, params, cameras_path + "." + name + ".png") != EXIT_SUCCESS)
      return EXIT_FAILURE;
  }
  return EXIT_SUCCESS;
}

// tools/create_legends.cc:35-54: <directory>/legend_error_directions.png (LegendErrorDirections). Returns EXIT_SUCCESS,
// or EXIT_FAILURE with "Cannot write file: ...". pipeline.py's CreateLegends writes the same bytes.
inline int CreateLegends(const std::string& directory = ".") {
  const std::string path = io_detail::join(directory, "legend_error_directions.png");
  if (!WritePNG(path, 200, 200, 3, LegendErrorDirections().data())) {
    std::cerr << "Cannot write file: " << path << "\n";
    return EXIT_FAILURE;
  }
  return EXIT_SUCCESS;
}

// ---- --intersect_datasets ------------------------------------------------------------------------------------------
// (n_datasets, list_offsets [n_lists * n_datasets + 1], xy [2 N], threshold) -> keep [N], report: the feature level of
// b200ba_intersect_features. The default runs it on the device.
using IntersectLists = std::function<void(int32_t, const std::vector<int64_t>&, const std::vector<float>&, double,
                                          std::vector<uint8_t>*, b200ba_intersection_report*)>;

inline void IntersectListsOnDevice(int32_t n_datasets, const std::vector<int64_t>& offsets, const std::vector<float>& xy,
                                   double threshold, std::vector<uint8_t>* keep, b200ba_intersection_report* report) {
  keep->assign(xy.size() / 2, 0);
  const int64_t n_lists = static_cast<int64_t>(offsets.size() - 1) / n_datasets;
  if (b200ba_intersect_features(-1, n_datasets, n_lists, offsets.data(), xy.data(), threshold, keep->data(), report,
                                nullptr) != 0)
    throw std::runtime_error(std::string("b200ba_intersect_features: ") + b200ba_last_error(nullptr));
}

inline int64_t IntersectFeatureCount(const Dataset& dataset) {
  int64_t count = 0;
  for (int k = 0; k < dataset.ImagesetCount(); ++k)
    for (int c = 0; c < dataset.num_cameras(); ++c) count += dataset.GetImageset(k)->FeaturesOfCamera(c).size();
  return count;
}

// tools/intersect_datasets.cc:41-261: of several dataset.bin files of one image sequence (e.g. one per feature
// detector), keep only the features that all of them detected, and write each to <path>.intersected.bin. Imagesets are
// matched by filename: dataset 0's imagesets are walked by index; a filename missing from another dataset is deleted
// from every dataset that has it (the first imageset of a repeated filename, as unordered_map::insert keeps it) and the
// walk steps back by one; a later duplicate in dataset 0 of a filename already deleted is itself deleted (the
// reference walks it forever); otherwise dataset 0's imageset and dataset i's first imageset of that filename form a
// task, and at the end every imageset of datasets 1.. whose filename dataset 0 no longer holds is deleted. The features
// of every (task, camera) are intersected by `intersect` (the rules are in b200ba.h); tasks that share an imageset run
// in separate calls in task order, so that a later task reads the features an earlier one thinned, as in the
// reference. Messages go to stderr; the two pinned counts are printed where they are not zero. Returns EXIT_SUCCESS, or
// EXIT_FAILURE for an empty path list or more than 32 paths (the device walk runs one warp per dataset in one CTA; the
// reference has no such limit), a file that cannot be read or written, or datasets with different camera counts.
// pipeline.py's IntersectDatasets prints and writes the same bytes.
inline int IntersectDatasets(const std::vector<std::string>& dataset_paths, double intersection_threshold = 3.0,
                             const IntersectLists& intersect = IntersectListsOnDevice) {
  if (dataset_paths.empty()) {
    std::cerr << "IntersectDatasets needs at least one dataset\n";
    return EXIT_FAILURE;
  }
  if (dataset_paths.size() > 32) {
    std::cerr << "IntersectDatasets takes at most 32 datasets, not " << dataset_paths.size() << "\n";
    return EXIT_FAILURE;
  }
  const int n = static_cast<int>(dataset_paths.size());
  std::vector<std::shared_ptr<Dataset>> datasets(n);
  for (int i = 0; i < n; ++i) {
    std::cerr << "Dataset " << i << ": " << dataset_paths[i] << "\n";
    if (!LoadDataset(dataset_paths[i].c_str(), &datasets[i])) {
      std::cerr << "Cannot read file: " << dataset_paths[i] << "\n";
      return EXIT_FAILURE;
    }
    if (i > 0 && datasets[i]->num_cameras() != datasets[0]->num_cameras()) {
      std::cerr << "Number of cameras in dataset " << dataset_paths[i]
                << " does not match the number of cameras in dataset " << dataset_paths[0] << "\n";
      return EXIT_FAILURE;
    }
  }
  for (int i = 0; i < n; ++i)
    std::cerr << "Input features in dataset " << i << ": " << IntersectFeatureCount(*datasets[i])
              << " (#imagesets: " << datasets[i]->ImagesetCount() << ")\n";

  std::vector<std::unordered_map<std::string, int>> maps(n);
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < datasets[i]->ImagesetCount(); ++k)
      maps[i].insert(std::make_pair(datasets[i]->GetImageset(k)->GetFilename(), k));
  std::vector<std::vector<std::shared_ptr<Imageset>>> tasks;
  for (int index = 0; index < datasets[0]->ImagesetCount();) {
    std::vector<std::shared_ptr<Imageset>> task{datasets[0]->GetImageset(index)};
    const std::string name = task[0]->GetFilename();
    for (int i = 1; i < n; ++i) {
      auto it = maps[i].find(name);
      if (it == maps[i].end()) break;
      task.push_back(datasets[i]->GetImageset(it->second));
    }
    if (static_cast<int>(task.size()) == n) {
      tasks.push_back(task);
      ++index;
      continue;
    }
    for (int i = 0; i < n; ++i) {
      auto it = maps[i].find(name);
      int doomed;
      if (it != maps[i].end()) {
        doomed = it->second;
        maps[i].erase(it);
      } else if (i == 0) {
        std::cerr << "Imageset " << name << " of dataset 0 deleted: its filename was deleted before\n";
        doomed = index;
      } else {
        continue;
      }
      datasets[i]->DeleteImageset(doomed);
      for (auto& item : maps[i])
        if (item.second > doomed) --item.second;
    }
  }

  // waves: a task runs after every earlier task that shares one of its imagesets
  std::vector<std::vector<size_t>> waves;
  std::unordered_map<const Imageset*, size_t> last_wave;
  for (size_t t = 0; t < tasks.size(); ++t) {
    size_t w = 0;
    for (const auto& s : tasks[t]) {
      auto it = last_wave.find(s.get());
      if (it != last_wave.end()) w = std::max(w, it->second + 1);
    }
    for (const auto& s : tasks[t]) last_wave[s.get()] = w;
    if (w == waves.size()) waves.emplace_back();
    waves[w].push_back(t);
  }
  const int ncam = datasets[0]->num_cameras();
  int64_t uncovered = 0, capped = 0;
  for (const std::vector<size_t>& wave : waves) {
    std::vector<int64_t> offsets{0};
    std::vector<float> xy;
    for (size_t t : wave)
      for (int c = 0; c < ncam; ++c)
        for (const auto& s : tasks[t]) {
          for (const PointFeature& f : s->FeaturesOfCamera(c)) {
            xy.push_back(f.xy.x);
            xy.push_back(f.xy.y);
          }
          offsets.push_back(static_cast<int64_t>(xy.size() / 2));
        }
    if (xy.empty()) continue;
    std::vector<uint8_t> keep;
    b200ba_intersection_report report{};
    intersect(n, offsets, xy, intersection_threshold, &keep, &report);
    uncovered += report.uncovered;
    capped += report.capped;
    size_t k = 0;
    for (size_t t : wave)
      for (int c = 0; c < ncam; ++c)
        for (const auto& s : tasks[t]) {
          std::vector<PointFeature>& features = s->FeaturesOfCamera(c);
          std::vector<PointFeature> kept;
          for (size_t j = 0; j < features.size(); ++j)
            if (keep[offsets[k] + j]) kept.push_back(features[j]);
          features.swap(kept);
          ++k;
        }
  }
  if (uncovered) std::cerr << "Features rejected with nothing covered, left in place: " << uncovered << "\n";
  if (capped) std::cerr << "Fixed-point loops stopped after 100 passes: " << capped << "\n";

  for (int i = 1; i < n; ++i)
    for (int k = 0; k < datasets[i]->ImagesetCount();) {
      if (maps[0].count(datasets[i]->GetImageset(k)->GetFilename()) == 0)
        datasets[i]->DeleteImageset(k);
      else
        ++k;
    }
  for (int i = 0; i < n; ++i) {
    const std::string out = dataset_paths[i] + ".intersected.bin";
    if (!SaveDataset(out.c_str(), *datasets[i])) {
      std::cerr << "Cannot write file: " << out << "\n";
      return EXIT_FAILURE;
    }
  }
  for (int i = 0; i < n; ++i)
    std::cerr << "Remaining features in dataset " << i << ": " << IntersectFeatureCount(*datasets[i]) << "\n";
  return EXIT_SUCCESS;
}

// ---- --render_synthetic_dataset -----------------------------------------------------------------------------------
// The b200ba_pattern of a pattern file; false when it has more than B200BA_PATTERN_MAX_TAGS tags.
inline bool PatternStruct(const PatternFile& file, b200ba_pattern* p) {
  if (file.tags.size() > B200BA_PATTERN_MAX_TAGS) return false;
  *p = b200ba_pattern{};
  p->squares_x = file.squares_x;
  p->squares_y = file.squares_y;
  p->num_star_segments = file.num_star_segments;
  p->num_tags = static_cast<int32_t>(file.tags.size());
  p->page_width_mm = file.page_width_mm;
  p->page_height_mm = file.page_height_mm;
  p->pattern_start_x_mm = file.pattern_start_x_mm;
  p->pattern_start_y_mm = file.pattern_start_y_mm;
  p->pattern_end_x_mm = file.pattern_end_x_mm;
  p->pattern_end_y_mm = file.pattern_end_y_mm;
  for (size_t k = 0; k < file.tags.size(); ++k)
    p->tags[k] = b200ba_pattern_tag{file.tags[k].x, file.tags[k].y, file.tags[k].width, file.tags[k].height,
                                    file.tags[k].index};
  return true;
}

// tools/render_synthetic_dataset.cc:43-298: a 640 x 480 pinhole camera (fx = fy = 480, cx = 320, cy = 240,
// pixel-corner convention) views the pattern of pattern_yaml / pattern_png from num_images random poses
// (b200ba_synthetic_poses, seeded; the reference seeds with the time and reads the pattern from beside its binary);
// the images are rendered on the device (b200ba_render_pattern_images). Writes <path>/dataset.yaml (the reference's
// text) and <path>/images0/000000.png ... (WritePNG), printing "Rendering image i ..." to stderr. Returns
// EXIT_SUCCESS / EXIT_FAILURE with the reference's messages. pipeline.py's RenderSyntheticDataset writes the same
// bytes.
inline int RenderSyntheticDataset(const std::string& path,
                                  const std::string& pattern_yaml = "pattern_resolution_17x24_segments_16_apriltag_0.yaml",
                                  const std::string& pattern_png = "pattern_resolution_17x24_segments_16_apriltag_0.png",
                                  int num_images = 500, uint64_t seed = 0, int device = -1) {
  const int width = 640, height = 480;
  const float fx = height, fy = height, cx = 0.5 * width, cy = 0.5 * height;
  const float k[4] = {fx, fy, cx, cy};
  PatternFile file;
  if (!LoadPatternYAML(pattern_yaml, &file)) {
    std::cerr << "Failed to load: " << pattern_yaml << "\n";
    return EXIT_FAILURE;
  }
  int pattern_w = 0, pattern_h = 0;
  std::vector<uint8_t> pattern_image;
  std::string error;
  if (!ReadPNG(pattern_png, &pattern_w, &pattern_h, &pattern_image, &error)) {
    if (error.rfind("DecodePNG", 0) == 0) std::cerr << error << "\n";
    std::cerr << "Cannot load the pattern image from: " << pattern_png << "\n";
    return EXIT_FAILURE;
  }
  b200ba_pattern pattern;
  if (!PatternStruct(file, &pattern)) {
    std::cerr << "The pattern has more than " << B200BA_PATTERN_MAX_TAGS << " AprilTags, which is not supported.\n";
    return EXIT_FAILURE;
  }
  std::error_code ec;
  std::filesystem::create_directories(path, ec);
  const std::string yaml_path = std::filesystem::absolute(std::filesystem::path(path) / "dataset.yaml").string();
  {
    std::ofstream yaml(yaml_path, std::ios::out | std::ios::binary);
    if (!yaml) {
      std::cerr << "Failed to write dataset YAML file at: " << yaml_path << "\n";
      return EXIT_FAILURE;
    }
    yaml << "- camera: \"Synthetic pinhole camera (fx: " << fx << ", fy: " << fy << ", cx: " << cx << ", cy: " << cy
         << ", 'pixel corner' coordinate origin convention)\"\n";
    yaml << "  path: \"images0\"\n";
  }
  const std::string images_dir = io_detail::join(path, "images0");
  std::filesystem::create_directories(images_dir, ec);
  if (num_images < 1) return EXIT_SUCCESS;
  std::vector<double> poses(12 * static_cast<size_t>(num_images));
  if (int rc = b200ba_synthetic_poses(&pattern, pattern_w, pattern_h, width, height, k, num_images, seed, poses.data(),
                                      nullptr)) {
    std::cerr << "b200ba_synthetic_poses failed (" << rc << "): " << b200ba_last_error(nullptr) << "\n";
    return EXIT_FAILURE;
  }
  std::vector<uint8_t> images(static_cast<size_t>(num_images) * width * height);
  if (int rc = b200ba_render_pattern_images(device, &pattern, pattern_image.data(), pattern_w, pattern_h, width, height,
                                            k, num_images, poses.data(), images.data(), nullptr)) {
    std::cerr << "b200ba_render_pattern_images failed (" << rc << "): " << b200ba_last_error(nullptr) << "\n";
    return EXIT_FAILURE;
  }
  for (int i = 0; i < num_images; ++i) {
    std::cerr << "Rendering image " << i << " ...\n";
    std::ostringstream name;
    name << std::setw(6) << std::setfill('0') << i << ".png";
    WritePNG(io_detail::join(images_dir, name.str()), width, height, 1,
             images.data() + static_cast<size_t>(i) * width * height);
  }
  return EXIT_SUCCESS;
}

// ---- feature refinement (FeatureDetectorTaggedPattern::RefineFeatureDetections) -----------------------------------
// The reference's sample offsets for window_half_extent (b200ba_feature_samples); empty for a bad extent.
inline std::vector<Vec2f> FeatureSamples(int window_half_extent) {
  const int n = static_cast<int>(8.0 * (2 * window_half_extent + 1) * (2 * window_half_extent + 1) + 0.5);
  std::vector<Vec2f> samples(std::max(n, 0));
  if (b200ba_feature_samples(window_half_extent, n, reinterpret_cast<float*>(samples.data())) != 0) samples.clear();
  return samples;
}

// The reference's FeatureDetection (feature_detector_tagged_pattern.h:291-317) plus the index of its image.
struct FeatureDetection {
  Vec2f position;            // pixel-centre convention
  Vec2i pattern_coordinate;  // integer feature coordinate in the pattern
  float final_cost = 0;      // negative for a rejected feature
  float local_pixel_tr_pattern[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};  // row-major
  int64_t image = 0;         // index into the images passed to RefineFeatureDetections
};

// RefineFeatureDetections (feature_detector_tagged_pattern.cc:1427-1648) for the features of any number of grey
// images of one size (images: n_images * width * height bytes), on the device (b200ba_refine_features, the
// arithmetic of the reference's CPU path for all four refinement types, B200BA_REFINE_*). output[i] is
// predicted_features[i] with the refined position and final_cost, or final_cost -1 and a NaN position when it is
// rejected; status (nullable) receives the reason codes. Returns the library's return code (0 on success).
inline int RefineFeatureDetections(const b200ba_pattern& pattern, const uint8_t* images, int width, int height,
                                   int64_t n_images, int window_half_extent, int refinement_type, int num_features,
                                   const FeatureDetection* predicted_features, FeatureDetection* output,
                                   std::vector<int32_t>* status = nullptr, int device = -1) {
  const std::vector<Vec2f> samples = FeatureSamples(window_half_extent);
  std::vector<b200ba_feature_prediction> pred(std::max(num_features, 0));
  for (int i = 0; i < num_features; ++i) {
    const FeatureDetection& f = predicted_features[i];
    pred[i].image = f.image;
    pred[i].position[0] = f.position.x, pred[i].position[1] = f.position.y;
    pred[i].pattern_coordinate[0] = f.pattern_coordinate.x, pred[i].pattern_coordinate[1] = f.pattern_coordinate.y;
    std::copy(f.local_pixel_tr_pattern, f.local_pixel_tr_pattern + 9, pred[i].local_pixel_tr_pattern);
  }
  std::vector<float> xy(2 * pred.size()), cost(pred.size());
  std::vector<int32_t> st(pred.size());
  const int rc = b200ba_refine_features(device, &pattern, images, width, height, n_images,
                                        reinterpret_cast<const float*>(samples.data()),
                                        static_cast<int32_t>(samples.size()), window_half_extent, refinement_type,
                                        num_features, pred.data(), xy.data(), cost.data(), st.data(), nullptr);
  if (rc != 0) return rc;
  for (int i = 0; i < num_features; ++i) {
    output[i] = predicted_features[i];
    output[i].position = Vec2f{xy[2 * i], xy[2 * i + 1]};
    output[i].final_cost = cost[i];
  }
  if (status) *status = st;
  return 0;
}

}  // namespace b200ba_shim
