// b200ba_shim.hpp -- C++ host side above the C ABI: OptimizeJointly() with the reference's own
// parameter list (applications/camera_calibration/src/camera_calibration/bundle_adjustment/
// joint_optimization.h:53-70) over containers shaped like the reference's Dataset / BAState /
// CameraModel (dataset.h:57-212, ba_state.h:46-97, models/camera_model.h:42-204).
//
// The reference builds against Eigen / Sophus, which this repository must not depend on, so the
// containers here are minimal look-alikes (same member names and meaning). In the reference tree
// the same 60 lines of flattening are written against the real classes -- INTEGRATION.md shows it.
//
// Header-only; link with -lb200ba. No CPU fallback: errors are returned, not hidden.
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "b200ba.h"

namespace b200ba_shim {

struct Vec2f { float x, y; };
struct Vec2i { int32_t x, y; };
struct Vec2d { double x, y; };
struct Vec3d { double x, y, z; };

// SE3d look-alike: unit quaternion (w, x, y, z) + translation. (Eigen::Quaterniond::coeffs() is
// ordered x, y, z, w -- convert when adapting the real class.)
struct SE3d {
  double qw = 1, qx = 0, qy = 0, qz = 0;
  double tx = 0, ty = 0, tz = 0;
};

// R(q) p + t and the group product (a * b)(p) = a(b(p)), as Sophus::SE3d::operator* does them
inline Vec3d apply(const SE3d& T, const Vec3d& p) {
  const double w = T.qw, x = T.qx, y = T.qy, z = T.qz;
  return Vec3d{(1 - 2 * (y * y + z * z)) * p.x + 2 * (x * y - w * z) * p.y + 2 * (x * z + w * y) * p.z + T.tx,
               2 * (x * y + w * z) * p.x + (1 - 2 * (x * x + z * z)) * p.y + 2 * (y * z - w * x) * p.z + T.ty,
               2 * (x * z - w * y) * p.x + 2 * (y * z + w * x) * p.y + (1 - 2 * (x * x + y * y)) * p.z + T.tz};
}
inline SE3d compose(const SE3d& a, const SE3d& b) {
  SE3d r;
  r.qw = a.qw * b.qw - a.qx * b.qx - a.qy * b.qy - a.qz * b.qz;
  r.qx = a.qw * b.qx + a.qx * b.qw + a.qy * b.qz - a.qz * b.qy;
  r.qy = a.qw * b.qy - a.qx * b.qz + a.qy * b.qw + a.qz * b.qx;
  r.qz = a.qw * b.qz + a.qx * b.qy - a.qy * b.qx + a.qz * b.qw;
  const double n = std::sqrt(r.qw * r.qw + r.qx * r.qx + r.qy * r.qy + r.qz * r.qz);
  r.qw /= n; r.qx /= n; r.qy /= n; r.qz /= n;
  SE3d rot = a;
  rot.tx = rot.ty = rot.tz = 0;
  const Vec3d t = apply(rot, Vec3d{b.tx, b.ty, b.tz});
  r.tx = a.tx + t.x; r.ty = a.ty + t.y; r.tz = a.tz + t.z;
  return r;
}

// models/camera_model.h:42-204 (only what the BA path touches)
class CameraModel {
 public:
  enum class Type { CentralGeneric = 0, NoncentralGeneric = 1, CentralRadial = 4, CentralThinPrismFisheye = 2,
                    CentralOpenCV = 3, InvalidType = 5 };
  CameraModel(int width, int height, int min_x, int min_y, int max_x, int max_y, Type type)
      : m_width(width), m_height(height), m_calibration_min_x(min_x), m_calibration_min_y(min_y),
        m_calibration_max_x(max_x), m_calibration_max_y(max_y), m_type(type) {}
  virtual ~CameraModel() {}
  virtual CameraModel* duplicate() = 0;
  virtual int update_parameter_count() const = 0;
  virtual bool GetGridResolution(int* rx, int* ry) const { (void)rx; (void)ry; return false; }
  // flat intrinsics in the layout include/b200ba.h documents
  virtual std::vector<double>& flat_intrinsics() = 0;
  // camera_model.h:127-129: only non-central models carry metric quantities
  virtual void Scale(double factor) { (void)factor; }
  // camera_model.h:182-185
  Vec2d CenterOfCalibratedArea() const {
    return Vec2d{0.5 * (m_calibration_min_x + m_calibration_max_x + 1), 0.5 * (m_calibration_min_y + m_calibration_max_y + 1)};
  }
  int width() const { return m_width; }
  int height() const { return m_height; }
  int calibration_min_x() const { return m_calibration_min_x; }
  int calibration_min_y() const { return m_calibration_min_y; }
  int calibration_max_x() const { return m_calibration_max_x; }
  int calibration_max_y() const { return m_calibration_max_y; }
  Type type() const { return m_type; }
 protected:
  int m_width, m_height, m_calibration_min_x, m_calibration_min_y, m_calibration_max_x, m_calibration_max_y;
  Type m_type;
};

// models/central_generic.h: grid of unit directions, row-major, xyz
class CentralGenericModel : public CameraModel {
 public:
  CentralGenericModel(int grid_resolution_x, int grid_resolution_y, int min_x, int min_y, int max_x, int max_y,
                      int width, int height)
      : CameraModel(width, height, min_x, min_y, max_x, max_y, Type::CentralGeneric), gw(grid_resolution_x),
        gh(grid_resolution_y), grid(3 * static_cast<size_t>(gw) * gh, 0.0) {}
  CameraModel* duplicate() override { return new CentralGenericModel(*this); }
  int update_parameter_count() const override { return 2 * gw * gh; }
  bool GetGridResolution(int* rx, int* ry) const override { *rx = gw; *ry = gh; return true; }
  std::vector<double>& flat_intrinsics() override { return grid; }
  static constexpr int IntrinsicsJacobianSize = 2 * 16;
  // central_grid.h:150-154 (double arithmetic with the float constant (grid - 3.f))
  Vec2d PixelCornerConvToGridPoint(double x, double y) const {
    return Vec2d{1.0 + static_cast<double>(gw - 3.f) * (x - m_calibration_min_x) / (m_calibration_max_x + 1 - m_calibration_min_x),
                 1.0 + static_cast<double>(gh - 3.f) * (y - m_calibration_min_y) / (m_calibration_max_y + 1 - m_calibration_min_y)};
  }
  // central_generic.cc:424-431 + :551-568: the LM over the direction grid runs in the library
  void FitToPixelDirections(const std::vector<Vec2d>& pixels, const std::vector<Vec3d>& directions,
                            int max_iteration_count) {
    std::vector<double> gp, d;
    gp.reserve(2 * pixels.size());
    d.reserve(3 * directions.size());
    for (const Vec2d& p : pixels) {
      const Vec2d g = PixelCornerConvToGridPoint(p.x, p.y);
      gp.push_back(g.x);
      gp.push_back(g.y);
    }
    for (const Vec3d& v : directions) {
      d.push_back(v.x);
      d.push_back(v.y);
      d.push_back(v.z);
    }
    b200ba_fit_report rep;
    if (b200ba_fit_directions(-1, gw, gh, grid.data(), static_cast<int64_t>(pixels.size()), gp.data(), d.data(),
                              max_iteration_count, &rep) != 0)
      throw std::runtime_error(std::string("b200ba_fit_directions: ") + b200ba_last_error(nullptr));
  }
  int gw, gh;
  std::vector<double> grid;
};

// models/noncentral_generic.h: direction grid followed by point grid
class NoncentralGenericModel : public CameraModel {
 public:
  NoncentralGenericModel(int grid_resolution_x, int grid_resolution_y, int min_x, int min_y, int max_x, int max_y,
                         int width, int height)
      : CameraModel(width, height, min_x, min_y, max_x, max_y, Type::NoncentralGeneric), gw(grid_resolution_x),
        gh(grid_resolution_y), grids(6 * static_cast<size_t>(gw) * gh, 0.0) {}
  CameraModel* duplicate() override { return new NoncentralGenericModel(*this); }
  int update_parameter_count() const override { return 5 * gw * gh; }
  bool GetGridResolution(int* rx, int* ry) const override { *rx = gw; *ry = gh; return true; }
  std::vector<double>& flat_intrinsics() override { return grids; }
  // noncentral_generic.cc:148-154: the line origins (second half of `grids`) are metric
  void Scale(double factor) override {
    for (size_t i = grids.size() / 2; i < grids.size(); ++i) grids[i] *= factor;
  }
  static constexpr int IntrinsicsJacobianSize = 5 * 16;
  int gw, gh;
  std::vector<double> grids;
};

// models/central_opencv.h: fx fy cx cy k1..k6 p1 p2
class CentralOpenCVModel : public CameraModel {
 public:
  CentralOpenCVModel(int width, int height)
      : CameraModel(width, height, 0, 0, width - 1, height - 1, Type::CentralOpenCV), parameters(12, 0.0) {}
  CameraModel* duplicate() override { return new CentralOpenCVModel(*this); }
  int update_parameter_count() const override { return 12; }
  std::vector<double>& flat_intrinsics() override { return parameters; }
  static constexpr int IntrinsicsJacobianSize = 12;
  std::vector<double> parameters;
};

// dataset.h:57-84
struct PointFeature {
  Vec2f xy{0, 0};
  int id = -1;
  int index = -1;
  Vec2d last_projection{0, 0};
};

// dataset.h:88-123
class Imageset {
 public:
  explicit Imageset(int num_cameras) : m_features(num_cameras) {}
  std::vector<PointFeature>& FeaturesOfCamera(int c) { return m_features[c]; }
  const std::vector<PointFeature>& FeaturesOfCamera(int c) const { return m_features[c]; }
  void SetFilename(const std::string& filename) { m_filename = filename; }
  const std::string& GetFilename() const { return m_filename; }
 private:
  std::string m_filename;
  std::vector<std::vector<PointFeature>> m_features;
};

// dataset.h:45-55: the known layout of one calibration pattern
struct KnownGeometry {
  float cell_length_in_meters = 0;
  // insertion-ordered (feature id, pattern x, pattern y); the reference keeps an unordered_map
  std::vector<std::pair<int, std::pair<int, int>>> feature_id_to_position;
};

// dataset.h:131-212
class Dataset {
 public:
  explicit Dataset(int num_cameras) : m_num_cameras(num_cameras), m_image_sizes(num_cameras, std::make_pair(0, 0)) {}
  void SetImageSize(int camera_index, int width, int height) { m_image_sizes[camera_index] = std::make_pair(width, height); }
  std::pair<int, int> GetImageSize(int camera_index) const { return m_image_sizes[camera_index]; }
  std::vector<KnownGeometry>& known_geometries() { return m_known_geometries; }
  const std::vector<KnownGeometry>& known_geometries() const { return m_known_geometries; }
  std::shared_ptr<Imageset> NewImageset() {
    m_imagesets.emplace_back(new Imageset(m_num_cameras));
    return m_imagesets.back();
  }
  void DeleteImageset(int i) { m_imagesets.erase(m_imagesets.begin() + i); }
  std::shared_ptr<Imageset> GetImageset(int i) { return m_imagesets[i]; }
  std::shared_ptr<const Imageset> GetImageset(int i) const { return m_imagesets[i]; }
  int ImagesetCount() const { return static_cast<int>(m_imagesets.size()); }
  int num_cameras() const { return m_num_cameras; }
  // dataset.cc:78-130: appends the imagesets and known geometries of `other`; false (nothing changed) where the camera
  // counts or image sizes differ. The feature ids of `other` and of its geometries are offset by 1 + the largest id of
  // this dataset's geometries (1 without any), so every geometry stays separate.
  bool Merge(const Dataset& other) {
    if (m_num_cameras != other.m_num_cameras || m_image_sizes != other.m_image_sizes) return false;
    int max_feature_id = 0;
    for (const KnownGeometry& g : m_known_geometries)
      for (const auto& entry : g.feature_id_to_position) max_feature_id = std::max(max_feature_id, entry.first);
    const int offset = max_feature_id + 1;
    for (const KnownGeometry& g : other.m_known_geometries) {
      KnownGeometry kg;
      kg.cell_length_in_meters = g.cell_length_in_meters;
      for (const auto& entry : g.feature_id_to_position) kg.feature_id_to_position.emplace_back(entry.first + offset, entry.second);
      m_known_geometries.push_back(kg);
    }
    first_imageset_indices_for_datasets.push_back(ImagesetCount());
    for (const std::shared_ptr<Imageset>& src : other.m_imagesets) {
      std::shared_ptr<Imageset> s = NewImageset();
      s->SetFilename(src->GetFilename());
      for (int c = 0; c < m_num_cameras; ++c) {
        s->FeaturesOfCamera(c) = src->FeaturesOfCamera(c);
        for (PointFeature& f : s->FeaturesOfCamera(c)) f.id += offset;
      }
    }
    return true;
  }
  std::vector<int> first_imageset_indices_for_datasets{0};
 private:
  int m_num_cameras;
  std::vector<std::pair<int, int>> m_image_sizes;
  std::vector<KnownGeometry> m_known_geometries;
  std::vector<std::shared_ptr<Imageset>> m_imagesets;
};

// ba_state.h:46-97
struct BAState {
  std::vector<bool> image_used;
  std::unordered_map<int, int> feature_id_to_points_index;
  std::vector<SE3d> camera_tr_rig;
  std::vector<SE3d> rig_tr_global;
  std::vector<std::shared_ptr<CameraModel>> intrinsics;
  std::vector<Vec3d> points;
  int num_cameras() const { return static_cast<int>(intrinsics.size()); }
  // ba_state.h:65-67: camera_tr_rig[camera] * rig_tr_global[imageset]
  SE3d image_tr_global(int camera_index, int imageset_index) const {
    return compose(camera_tr_rig[camera_index], rig_tr_global[imageset_index]);
  }
  // ba_state.cc:60-76: every translation, the points and the models' metric parts
  void ScaleState(double scaling_factor) {
    for (SE3d& T : camera_tr_rig) { T.tx *= scaling_factor; T.ty *= scaling_factor; T.tz *= scaling_factor; }
    for (SE3d& T : rig_tr_global) { T.tx *= scaling_factor; T.ty *= scaling_factor; T.tz *= scaling_factor; }
    for (Vec3d& p : points) { p.x *= scaling_factor; p.y *= scaling_factor; p.z *= scaling_factor; }
    for (auto& m : intrinsics) m->Scale(scaling_factor);
  }
  // ba_state.cc:78-91
  void ComputeFeatureIdToPointsIndex(Dataset* dataset) {
    for (int i = 0; i < dataset->ImagesetCount(); ++i)
      for (int c = 0; c < dataset->num_cameras(); ++c)
        for (PointFeature& f : dataset->GetImageset(i)->FeaturesOfCamera(c)) f.index = feature_id_to_points_index.at(f.id);
  }
};

// joint_optimization.h:38-47
enum class SchurMode { Dense = 0, DenseCUDA, DenseOnTheFly, Sparse, SparseOnTheFly };

// libvis lm_optimizer.h:55-77
struct OptimizationReport {
  double initial_cost = 0, final_cost = 0;
  int num_iterations_performed = 0;
  double cost_and_jacobian_evaluation_time = 0, solve_time = 0;
};

namespace detail {
struct Flat {
  std::vector<b200ba_camera> cams;
  std::vector<uint32_t> oi, oc, op;
  std::vector<float> oxy;
  std::vector<double> points, rtg, ctr, lastp;
  std::vector<double*> intr;
  std::vector<int> used;
};
inline void flatten(Dataset& dataset, BAState* state, Flat* f) {
  if (state->image_used.size() != state->rig_tr_global.size())
    throw std::runtime_error("image_used / rig_tr_global size mismatch");  // CHECK_EQ, joint_optimization.cc:72
  for (size_t i = 0; i < state->image_used.size(); ++i)
    if (state->image_used[i]) f->used.push_back(static_cast<int>(i));
  for (auto& m : state->intrinsics) {
    b200ba_camera c{};
    c.model_type = static_cast<int32_t>(m->type());
    c.width = m->width();
    c.height = m->height();
    c.calibration_min_x = m->calibration_min_x();
    c.calibration_min_y = m->calibration_min_y();
    c.calibration_max_x = m->calibration_max_x();
    c.calibration_max_y = m->calibration_max_y();
    int rx = 0, ry = 0;
    if (m->GetGridResolution(&rx, &ry)) { c.grid_width = rx; c.grid_height = ry; }
    f->cams.push_back(c);
    f->intr.push_back(m->flat_intrinsics().data());
  }
  // reference residual order: imageset, camera, feature (joint_optimization.cc:273-290)
  for (size_t seq = 0; seq < f->used.size(); ++seq)
    for (int c = 0; c < dataset.num_cameras(); ++c)
      for (const PointFeature& ft : dataset.GetImageset(f->used[seq])->FeaturesOfCamera(c)) {
        f->oi.push_back(static_cast<uint32_t>(seq));
        f->oc.push_back(static_cast<uint32_t>(c));
        f->op.push_back(static_cast<uint32_t>(ft.index));
        f->oxy.push_back(ft.xy.x);
        f->oxy.push_back(ft.xy.y);
        f->lastp.push_back(ft.last_projection.x);
        f->lastp.push_back(ft.last_projection.y);
      }
  for (const Vec3d& p : state->points) { f->points.push_back(p.x); f->points.push_back(p.y); f->points.push_back(p.z); }
  auto push_pose = [](std::vector<double>& v, const SE3d& T) {
    v.insert(v.end(), {T.qw, T.qx, T.qy, T.qz, T.tx, T.ty, T.tz});
  };
  for (int i : f->used) push_pose(f->rtg, state->rig_tr_global[i]);
  for (const SE3d& T : state->camera_tr_rig) push_pose(f->ctr, T);
}
inline SE3d pose_at(const std::vector<double>& v, size_t i) {
  SE3d T;
  T.qw = v[7 * i]; T.qx = v[7 * i + 1]; T.qy = v[7 * i + 2]; T.qz = v[7 * i + 3];
  T.tx = v[7 * i + 4]; T.ty = v[7 * i + 5]; T.tz = v[7 * i + 6];
  return T;
}
// Flattens (dataset, state), creates a handle, runs `body(handle, &flat_state)` and reads the result back.
template <class Body>
inline void run_with_handle(Dataset& dataset, BAState* state, const char* what, Body body) {
  Flat f;
  flatten(dataset, state, &f);
  b200ba_problem pb{};
  pb.n_cameras = static_cast<int32_t>(f.cams.size());
  pb.cameras = f.cams.data();
  pb.n_imagesets = static_cast<int32_t>(f.used.size());
  pb.n_points = static_cast<int32_t>(state->points.size());
  pb.n_obs = static_cast<int64_t>(f.oi.size());
  pb.obs_imageset = f.oi.data();
  pb.obs_camera = f.oc.data();
  pb.obs_point = f.op.data();
  pb.obs_xy = f.oxy.data();
  b200ba_handle* h = nullptr;
  if (b200ba_create(&pb, -1, &h) != 0) throw std::runtime_error(std::string("b200ba_create: ") + b200ba_last_error(nullptr));
  b200ba_state st{f.points.data(), f.rtg.data(), f.ctr.data(), f.intr.data(), f.lastp.data()};
  const int rc = body(h, &st);
  const std::string err = rc ? b200ba_last_error(h) : "";
  b200ba_destroy(h);
  if (rc) throw std::runtime_error(std::string(what) + ": " + err);
  // read back what the reference writes (joint_optimization.cc:942-950) + last_projection;
  // the intrinsics were updated in place through flat_intrinsics()
  for (size_t c = 0; c < state->camera_tr_rig.size(); ++c) state->camera_tr_rig[c] = pose_at(f.ctr, c);
  for (size_t s = 0; s < f.used.size(); ++s) state->rig_tr_global[f.used[s]] = pose_at(f.rtg, s);
  for (size_t p = 0; p < state->points.size(); ++p) state->points[p] = Vec3d{f.points[3 * p], f.points[3 * p + 1], f.points[3 * p + 2]};
  size_t o = 0;
  for (size_t seq = 0; seq < f.used.size(); ++seq)
    for (int c = 0; c < dataset.num_cameras(); ++c)
      for (PointFeature& ft : dataset.GetImageset(f.used[seq])->FeaturesOfCamera(c)) {
        ft.last_projection = Vec2d{f.lastp[2 * o], f.lastp[2 * o + 1]};
        ++o;
      }
}
inline void run(Dataset& dataset, BAState* state, const b200ba_options& opt, b200ba_report* rep) {
  run_with_handle(dataset, state, "b200ba_optimize_host",
                  [&](b200ba_handle* h, b200ba_state* st) { return b200ba_optimize_host(h, st, &opt, rep); });
}
}  // namespace detail

// joint_optimization.h:53-70 -- same parameters, same meaning. numerical_diff_delta is accepted
// for signature parity (the device path differentiates analytically); debug_* behave like the reference's.
inline double OptimizeJointly(Dataset& dataset, BAState* state, int max_iteration_count, double init_lambda,
                              double numerical_diff_delta, double regularization_weight, bool localize_only,
                              bool eliminate_points, SchurMode schur_mode, double* final_lambda,
                              bool* performed_an_iteration = nullptr, bool debug_verify_cost = false,
                              bool debug_fix_points = false, bool debug_fix_poses = false,
                              bool debug_fix_rig_poses = false, bool debug_fix_intrinsics = false,
                              bool print_progress = true) {
  if (performed_an_iteration) *performed_an_iteration = false;
  b200ba_options opt;
  b200ba_default_options(&opt);
  opt.max_iteration_count = max_iteration_count;
  opt.init_lambda = init_lambda;
  opt.numerical_diff_delta = numerical_diff_delta;
  opt.regularization_weight = regularization_weight;
  opt.localize_only = localize_only ? 1 : 0;
  opt.eliminate_points = eliminate_points ? 1 : 0;
  opt.schur_mode = static_cast<int32_t>(schur_mode);
  opt.print_progress = print_progress ? 1 : 0;
  opt.debug_verify_cost = debug_verify_cost ? 1 : 0;
  opt.debug_fix_points = debug_fix_points ? 1 : 0;
  opt.debug_fix_poses = debug_fix_poses ? 1 : 0;
  opt.debug_fix_rig_poses = debug_fix_rig_poses ? 1 : 0;
  opt.debug_fix_intrinsics = debug_fix_intrinsics ? 1 : 0;
  b200ba_report rep;
  detail::run(dataset, state, opt, &rep);
  if (final_lambda) *final_lambda = rep.final_lambda;
  if (performed_an_iteration) *performed_an_iteration = rep.performed_an_iteration != 0;
  return rep.final_cost;
}

// cuda_joint_optimization.h:45-59
inline OptimizationReport CudaOptimizeJointly(Dataset& dataset, BAState* state, int max_iteration_count,
                                              int /*max_inner_iterations*/, double init_lambda,
                                              double numerical_diff_delta, double regularization_weight,
                                              double* final_lambda, bool /*debug_verify_cost*/ = false,
                                              bool = false, bool = false, bool = false, bool = false,
                                              bool print_progress = true) {
  b200ba_options opt;
  b200ba_default_options(&opt);
  opt.max_iteration_count = max_iteration_count;
  opt.init_lambda = init_lambda;
  opt.numerical_diff_delta = numerical_diff_delta;
  opt.regularization_weight = regularization_weight;
  opt.print_progress = print_progress ? 1 : 0;
  b200ba_report rep;
  detail::run(dataset, state, opt, &rep);
  if (final_lambda) *final_lambda = rep.final_lambda;
  OptimizationReport r;
  r.initial_cost = rep.initial_cost;
  r.final_cost = rep.final_cost;
  r.num_iterations_performed = rep.num_iterations_performed;
  r.cost_and_jacobian_evaluation_time = rep.cost_and_jacobian_evaluation_time;
  r.solve_time = rep.solve_time;
  return r;
}


// RunBundleAdjustment (calibration.cc:187-304) for the CPU branch of the reference (`use_cuda == false`;
// the float32 PCG branch has no counterpart here): one upload, the whole loop -- single LM iterations,
// ChooseNiceCameraOrientation + camera_tr_rig update, stopping criterion -- device-resident inside
// b200ba_run_bundle_adjustment, one download. `on_iteration(iteration, cost)` (optional) returning true
// stops the loop like the reference's 'q' key; the calibration window / state_output_path hooks of the
// reference belong into it. Returns the cost after the last iteration.
inline double RunBundleAdjustment(SchurMode schur_mode, int max_iteration_count, double cost_reduction_threshold,
                                  Dataset* dataset, BAState* state, double regularization_weight, bool localize_only,
                                  bool eliminate_points = false, bool (*on_iteration)(int, double) = nullptr,
                                  b200ba_ba_report* report_out = nullptr) {
  b200ba_options opt;
  b200ba_default_options(&opt);
  opt.init_lambda = -1;             // calibration.cc:203
  opt.numerical_diff_delta = 1e-4;  // calibration.cc:201
  opt.regularization_weight = regularization_weight;
  opt.localize_only = localize_only ? 1 : 0;
  opt.eliminate_points = eliminate_points ? 1 : 0;  // the product passes false (calibration.cc:232)
  opt.schur_mode = static_cast<int32_t>(schur_mode);
  opt.print_progress = 0;
  b200ba_ba_report rep;
  struct Ctx {
    bool (*fn)(int, double);
  } ctx{on_iteration};
  auto tramp = [](void* user, int32_t it, double cost) -> int {
    Ctx* c = static_cast<Ctx*>(user);
    return (c->fn && c->fn(it, cost)) ? 1 : 0;
  };
  detail::run_with_handle(*dataset, state, "b200ba_run_bundle_adjustment", [&](b200ba_handle* h, b200ba_state* st) {
    if (int rc = b200ba_set_state(h, st)) return rc;
    if (int rc = b200ba_run_bundle_adjustment(h, &opt, max_iteration_count, cost_reduction_threshold, &rep,
                                              on_iteration ? static_cast<int (*)(void*, int32_t, double)>(tramp) : nullptr, &ctx))
      return rc;
    return b200ba_get_state(h, st);
  });
  if (report_out) *report_out = rep;
  return rep.final_cost;
}

}  // namespace b200ba_shim
