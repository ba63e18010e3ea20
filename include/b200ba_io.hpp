// b200ba_io.hpp -- C++ readers / writers of the reference's on-disk formats either side of the
// bundle-adjustment path (SURVEY.md 8f-1), over the containers of b200ba_shim.hpp: `dataset.bin` and the
// state directory (`intrinsicsN.yaml`, `rig_tr_global.yaml`, `camera_tr_rig.yaml`, `points.yaml`).
// The Python mirror is camera_calibration_b200/io.py; tests/test_cpp_io.py round-trips files between the two.
//
// Formats follow applications/camera_calibration/src/camera_calibration/io/calibration_io.cc (APP/io below):
//   * dataset.bin (SaveDataset :51-135, LoadDataset :137-246): magic "calib_data", u32 version 0, u32 camera
//     count, per camera u32 width, height; u32 imageset count, per imageset u32 filename length + bytes, per
//     camera u32 n + n x (f32 x, f32 y, i32 id); known geometries: u32 count, each f32 cell length, u32 n,
//     n x (i32 id, i32 x, i32 y). Integers are BIG-endian (htonl, io_util.h:56-64), floats raw host order
//     (io_util.h:66-69).
//   * camera model YAML (SaveCameraModel :526-647, LoadCameraModel :649-783): 14 significant digits, grids
//     flat row-major x, y, z; directions are re-normalised on load.
//   * poses YAML (SavePoses :785-839, LoadPoses :841-888): pose_count + list of index, tx ty tz, qx qy qz qw;
//     only used images are listed.
//   * points.yaml (:890-985): flat `points` + `feature_id_to_point_index` list.
// The reference parses YAML with yaml-cpp, which this repository must not depend on: the reader below
// understands the subset these files use (top-level `key : scalar`, `key : [flow, list]` possibly spanning
// lines, `key:` followed by a block list of flat maps, `#` comments).
//
// Header-only, host code only (no device work happens here). Every loader returns false on a malformed
// file, like the reference's.
#pragma once

#include <algorithm>
#include <cctype>
#include <cerrno>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iomanip>
#include <map>
#include <sstream>
#include <string>
#include <sys/stat.h>
#include <vector>

#include "b200ba_shim.hpp"

namespace b200ba_shim {
namespace io_detail {

inline uint32_t swap32(uint32_t v) {
  const uint16_t probe = 1;
  if (*reinterpret_cast<const uint8_t*>(&probe) == 0) return v;  // big-endian host
  return (v >> 24) | ((v >> 8) & 0xff00u) | ((v << 8) & 0xff0000u) | (v << 24);
}
inline void put_u32(std::string* out, uint32_t v) {
  v = swap32(v);
  out->append(reinterpret_cast<const char*>(&v), 4);
}
inline void put_f32(std::string* out, float v) { out->append(reinterpret_cast<const char*>(&v), 4); }

struct Reader {
  const std::string& d;
  size_t pos = 0;
  bool ok = true;
  explicit Reader(const std::string& data) : d(data) {}
  bool need(size_t n) {
    if (!ok || d.size() - pos < n) ok = false;
    return ok;
  }
  uint32_t u32() {
    if (!need(4)) return 0;
    uint32_t v;
    std::memcpy(&v, d.data() + pos, 4);
    pos += 4;
    return swap32(v);
  }
  float f32() {
    if (!need(4)) return 0;
    float v;
    std::memcpy(&v, d.data() + pos, 4);
    pos += 4;
    return v;
  }
};

inline bool read_file(const std::string& path, std::string* out) {
  std::ifstream f(path, std::ios::binary);
  if (!f) return false;
  std::ostringstream ss;
  ss << f.rdbuf();
  *out = ss.str();
  return true;
}
inline bool write_file(const std::string& path, const std::string& data) {
  std::ofstream f(path, std::ios::binary | std::ios::trunc);
  if (!f) return false;
  f.write(data.data(), static_cast<std::streamsize>(data.size()));
  return static_cast<bool>(f);
}
inline bool file_exists(const std::string& path) {
  struct stat st;
  return ::stat(path.c_str(), &st) == 0;
}
inline void make_directories(const std::string& path) {
  for (size_t i = 1; i <= path.size(); ++i)
    if (i == path.size() || path[i] == '/') {
      const std::string sub = path.substr(0, i);
      if (!sub.empty()) ::mkdir(sub.c_str(), 0777);
    }
}
inline std::string join(const std::string& dir, const std::string& name) {
  return (!dir.empty() && dir.back() == '/') ? dir + name : dir + "/" + name;
}

// std::ostream << double with setprecision(14)
inline std::string num(double v) {
  char buf[40];
  std::snprintf(buf, sizeof(buf), "%.14g", v);
  return buf;
}

// ---- the YAML subset -----------------------------------------------------------------------------------
struct Node {
  bool is_scalar = false, is_flow = false, is_block = false;
  std::string scalar;
  std::vector<double> flow;
  std::vector<std::map<std::string, std::string>> block;
};
using Document = std::map<std::string, Node>;

inline std::string trim(const std::string& s) {
  size_t a = 0, b = s.size();
  while (a < b && (s[a] == ' ' || s[a] == '\t' || s[a] == '\r')) ++a;
  while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\t' || s[b - 1] == '\r')) --b;
  return s.substr(a, b - a);
}
inline bool to_double(const std::string& s, double* v) {
  const std::string t = trim(s);
  if (t.empty()) return false;
  if (t == ".nan" || t == ".NaN") { *v = std::nan(""); return true; }
  if (t == ".inf") { *v = HUGE_VAL; return true; }
  if (t == "-.inf") { *v = -HUGE_VAL; return true; }
  char* end = nullptr;
  errno = 0;
  *v = std::strtod(t.c_str(), &end);
  return end && *end == '\0';
}
inline bool to_int(const std::string& s, long long* v) {
  const std::string t = trim(s);
  if (t.empty()) return false;
  char* end = nullptr;
  errno = 0;
  *v = std::strtoll(t.c_str(), &end, 10);
  return end && *end == '\0' && errno == 0;
}
// splits "key : value" at the first ':' that is followed by a blank or ends the line
inline bool split_key(const std::string& line, std::string* key, std::string* value) {
  for (size_t i = 0; i < line.size(); ++i)
    if (line[i] == ':' && (i + 1 == line.size() || line[i + 1] == ' ' || line[i + 1] == '\t')) {
      *key = trim(line.substr(0, i));
      *value = trim(line.substr(i + 1));
      return !key->empty();
    }
  return false;
}
inline bool parse_flow(const std::string& text, std::vector<double>* out) {
  // text starts behind '[' and ends before ']'
  size_t a = 0;
  const std::string t = trim(text);
  if (t.empty()) return true;
  while (a <= t.size()) {
    size_t b = t.find(',', a);
    if (b == std::string::npos) b = t.size();
    double v;
    if (!to_double(t.substr(a, b - a), &v)) return false;
    out->push_back(v);
    a = b + 1;
  }
  return true;
}
inline bool parse_document(const std::string& text, Document* doc) {
  std::vector<std::string> lines;
  {
    std::istringstream ss(text);
    std::string l;
    while (std::getline(ss, l)) {
      // comments: a '#' at the start of the line or after a blank
      for (size_t i = 0; i < l.size(); ++i)
        if (l[i] == '#' && (i == 0 || l[i - 1] == ' ' || l[i - 1] == '\t')) {
          l.resize(i);
          break;
        }
      lines.push_back(l);
    }
  }
  size_t i = 0;
  while (i < lines.size()) {
    const std::string& raw = lines[i];
    if (trim(raw).empty()) { ++i; continue; }
    if (raw[0] == ' ' || raw[0] == '\t' || raw[0] == '-') return false;  // not a top-level key
    std::string key, value;
    if (!split_key(raw, &key, &value)) return false;
    Node node;
    ++i;
    if (!value.empty() && value[0] == '[') {
      std::string body = value.substr(1);
      while (body.find(']') == std::string::npos) {
        if (i >= lines.size()) return false;
        body += " " + lines[i++];
      }
      body.resize(body.find(']'));
      node.is_flow = true;
      if (!parse_flow(body, &node.flow)) return false;
    } else if (!value.empty()) {
      node.is_scalar = true;
      node.scalar = value;
    } else {
      // block list of flat maps (or nothing: an empty list)
      node.is_block = true;
      while (i < lines.size()) {
        const std::string t = trim(lines[i]);
        if (t.empty()) { ++i; continue; }
        if (lines[i][0] != ' ' && lines[i][0] != '\t' && lines[i][0] != '-') break;  // next top-level key
        std::string entry = t;
        if (entry[0] == '-') {
          node.block.emplace_back();
          entry = trim(entry.substr(1));
          if (entry.empty()) { ++i; continue; }
        }
        if (node.block.empty()) return false;
        std::string k, v;
        if (!split_key(entry, &k, &v)) return false;
        node.block.back()[k] = v;
        ++i;
      }
    }
    (*doc)[key] = node;
  }
  return true;
}
inline bool get_int(const Document& doc, const char* key, int* out) {
  auto it = doc.find(key);
  long long v;
  if (it == doc.end() || !it->second.is_scalar || !to_int(it->second.scalar, &v)) return false;
  *out = static_cast<int>(v);
  return true;
}
inline bool get_flow(const Document& doc, const char* key, const std::vector<double>** out) {
  auto it = doc.find(key);
  if (it == doc.end() || !it->second.is_flow) return false;
  *out = &it->second.flow;
  return true;
}
inline void append_flow(std::string* out, const double* v, size_t n) {
  out->push_back('[');
  for (size_t i = 0; i < n; ++i) {
    if (i) out->append(", ");
    out->append(num(v[i]));
  }
  out->append("]\n");
}
inline std::string dir_of(const std::string& path) {
  const size_t p = path.find_last_of('/');
  return p == std::string::npos ? std::string() : path.substr(0, p);
}

}  // namespace io_detail

// ---- dataset.bin ----------------------------------------------------------------------------------------
// APP/io:51-135
inline bool SaveDataset(const char* path, const Dataset& dataset) {
  using namespace io_detail;
  std::string out = "calib_data";
  put_u32(&out, 0);
  put_u32(&out, static_cast<uint32_t>(dataset.num_cameras()));
  for (int c = 0; c < dataset.num_cameras(); ++c) {
    put_u32(&out, static_cast<uint32_t>(dataset.GetImageSize(c).first));
    put_u32(&out, static_cast<uint32_t>(dataset.GetImageSize(c).second));
  }
  put_u32(&out, static_cast<uint32_t>(dataset.ImagesetCount()));
  for (int i = 0; i < dataset.ImagesetCount(); ++i) {
    std::shared_ptr<const Imageset> s = dataset.GetImageset(i);
    put_u32(&out, static_cast<uint32_t>(s->GetFilename().size()));
    out.append(s->GetFilename());
    for (int c = 0; c < dataset.num_cameras(); ++c) {
      const std::vector<PointFeature>& features = s->FeaturesOfCamera(c);
      put_u32(&out, static_cast<uint32_t>(features.size()));
      for (const PointFeature& f : features) {
        put_f32(&out, f.xy.x);
        put_f32(&out, f.xy.y);
        put_u32(&out, static_cast<uint32_t>(f.id));
      }
    }
  }
  put_u32(&out, static_cast<uint32_t>(dataset.known_geometries().size()));
  for (const KnownGeometry& g : dataset.known_geometries()) {
    put_f32(&out, g.cell_length_in_meters);
    put_u32(&out, static_cast<uint32_t>(g.feature_id_to_position.size()));
    for (const auto& item : g.feature_id_to_position) {
      put_u32(&out, static_cast<uint32_t>(item.first));
      put_u32(&out, static_cast<uint32_t>(item.second.first));
      put_u32(&out, static_cast<uint32_t>(item.second.second));
    }
  }
  make_directories(dir_of(path));
  return write_file(path, out);
}

// APP/io:137-246. `dataset` is replaced; false on a missing, truncated or foreign file.
inline bool LoadDataset(const char* path, std::shared_ptr<Dataset>* dataset) {
  using namespace io_detail;
  std::string data;
  if (!read_file(path, &data)) return false;
  if (data.size() < 10 || data.compare(0, 10, "calib_data") != 0) return false;
  Reader r(data);
  r.pos = 10;
  if (r.u32() != 0 || !r.ok) return false;  // version
  const uint32_t num_cameras = r.u32();
  if (!r.ok || num_cameras > (1u << 16)) return false;
  std::shared_ptr<Dataset> ds(new Dataset(static_cast<int>(num_cameras)));
  for (uint32_t c = 0; c < num_cameras; ++c) {
    const uint32_t w = r.u32(), h = r.u32();
    ds->SetImageSize(static_cast<int>(c), static_cast<int>(w), static_cast<int>(h));
  }
  const uint32_t num_imagesets = r.u32();
  for (uint32_t i = 0; r.ok && i < num_imagesets; ++i) {
    const uint32_t len = r.u32();
    if (!r.need(len)) return false;
    std::shared_ptr<Imageset> s = ds->NewImageset();
    s->SetFilename(data.substr(r.pos, len));
    r.pos += len;
    for (uint32_t c = 0; c < num_cameras; ++c) {
      const uint32_t n = r.u32();
      if (!r.need(static_cast<size_t>(n) * 12)) return false;
      std::vector<PointFeature>& features = s->FeaturesOfCamera(static_cast<int>(c));
      features.resize(n);
      for (uint32_t k = 0; k < n; ++k) {
        features[k].xy.x = r.f32();
        features[k].xy.y = r.f32();
        features[k].id = static_cast<int>(r.u32());
      }
    }
  }
  const uint32_t num_geometries = r.u32();
  for (uint32_t g = 0; r.ok && g < num_geometries; ++g) {
    KnownGeometry geometry;
    geometry.cell_length_in_meters = r.f32();
    const uint32_t n = r.u32();
    if (!r.need(static_cast<size_t>(n) * 12)) return false;
    for (uint32_t k = 0; k < n; ++k) {
      const int id = static_cast<int>(r.u32()), x = static_cast<int>(r.u32()), y = static_cast<int>(r.u32());
      geometry.feature_id_to_position.emplace_back(id, std::make_pair(x, y));
    }
    ds->known_geometries().push_back(geometry);
  }
  if (!r.ok) return false;
  *dataset = ds;
  return true;
}

// ---- camera models --------------------------------------------------------------------------------------
// APP/io:526-647
inline bool SaveCameraModel(CameraModel& model, const char* path) {
  using namespace io_detail;
  std::string out;
  auto header = [&](const char* type, bool area) {
    out += std::string("type : ") + type + "\n";
    out += "width : " + std::to_string(model.width()) + "\nheight : " + std::to_string(model.height()) + "\n";
    if (area) {
      out += "calibration_min_x : " + std::to_string(model.calibration_min_x()) + "\ncalibration_min_y : " +
             std::to_string(model.calibration_min_y()) + "\n";
      out += "calibration_max_x : " + std::to_string(model.calibration_max_x()) + "\ncalibration_max_y : " +
             std::to_string(model.calibration_max_y()) + "\n";
      int gw = 0, gh = 0;
      model.GetGridResolution(&gw, &gh);
      out += "grid_width : " + std::to_string(gw) + "\ngrid_height : " + std::to_string(gh) + "\n";
    }
  };
  const std::vector<double>& flat = model.flat_intrinsics();
  switch (model.type()) {
    case CameraModel::Type::CentralGeneric:
      header("CentralGenericModel", true);
      out += "# The grid is stored in row-major order, top to bottom. Each row is stored left to right. "
             "Each grid point is stored as x, y, z.\n";
      out += "grid : ";
      append_flow(&out, flat.data(), flat.size());
      break;
    case CameraModel::Type::NoncentralGeneric:
      header("NoncentralGenericModel", true);
      out += "# The grids are stored in row-major order, top to bottom. Each row is stored left to right. "
             "Each grid point is stored as x, y, z.\n";
      out += "point_grid : ";
      append_flow(&out, flat.data() + flat.size() / 2, flat.size() / 2);
      out += "direction_grid : ";
      append_flow(&out, flat.data(), flat.size() / 2);
      break;
    case CameraModel::Type::CentralOpenCV:
      header("CentralOpenCVModel", false);
      out += "parameters : ";
      append_flow(&out, flat.data(), flat.size());
      break;
    default:
      return false;  // model type not on the accelerated path
  }
  make_directories(dir_of(path));
  return write_file(path, out);
}

// APP/io:649-783. Returns an empty pointer on a malformed file or a model type that is not on this path.
inline std::shared_ptr<CameraModel> LoadCameraModel(const char* path) {
  using namespace io_detail;
  std::string text;
  Document doc;
  if (!read_file(path, &text) || !parse_document(text, &doc)) return nullptr;
  int width = 0, height = 0;
  if (!get_int(doc, "width", &width) || !get_int(doc, "height", &height) || width < 1 || height < 1) return nullptr;
  auto type_it = doc.find("type");
  if (type_it == doc.end() || !type_it->second.is_scalar) return nullptr;
  const std::string type = type_it->second.scalar;
  auto normalise = [](double* v, size_t n_points) {  // APP/io:672-675
    for (size_t i = 0; i < n_points; ++i) {
      const double norm = std::sqrt(v[3 * i] * v[3 * i] + v[3 * i + 1] * v[3 * i + 1] + v[3 * i + 2] * v[3 * i + 2]);
      v[3 * i] /= norm;
      v[3 * i + 1] /= norm;
      v[3 * i + 2] /= norm;
    }
  };
  if (type == "CentralGenericModel" || type == "NoncentralGenericModel") {
    int gw, gh, min_x, min_y, max_x, max_y;
    if (!get_int(doc, "grid_width", &gw) || !get_int(doc, "grid_height", &gh) || !get_int(doc, "calibration_min_x", &min_x) ||
        !get_int(doc, "calibration_min_y", &min_y) || !get_int(doc, "calibration_max_x", &max_x) ||
        !get_int(doc, "calibration_max_y", &max_y) || gw < 1 || gh < 1)
      return nullptr;
    const size_t n = 3 * static_cast<size_t>(gw) * gh;
    if (type == "CentralGenericModel") {
      const std::vector<double>* grid;
      if (!get_flow(doc, "grid", &grid) || grid->size() != n) return nullptr;
      std::shared_ptr<CentralGenericModel> m(new CentralGenericModel(gw, gh, min_x, min_y, max_x, max_y, width, height));
      m->grid = *grid;
      normalise(m->grid.data(), n / 3);
      return m;
    }
    const std::vector<double>*point_grid, *direction_grid;
    if (!get_flow(doc, "point_grid", &point_grid) || !get_flow(doc, "direction_grid", &direction_grid) ||
        point_grid->size() != n || direction_grid->size() != n)
      return nullptr;
    std::shared_ptr<NoncentralGenericModel> m(new NoncentralGenericModel(gw, gh, min_x, min_y, max_x, max_y, width, height));
    std::copy(direction_grid->begin(), direction_grid->end(), m->grids.begin());
    std::copy(point_grid->begin(), point_grid->end(), m->grids.begin() + n);
    normalise(m->grids.data(), n / 3);
    return m;
  }
  if (type == "CentralOpenCVModel") {
    const std::vector<double>* parameters;
    if (!get_flow(doc, "parameters", &parameters) || parameters->size() != 12) return nullptr;
    std::shared_ptr<CentralOpenCVModel> m(new CentralOpenCVModel(width, height));
    m->parameters = *parameters;
    return m;
  }
  return nullptr;
}

// ---- poses ----------------------------------------------------------------------------------------------
// APP/io:785-839 (also writes <path>.obj with the camera centres, like the reference)
inline bool SavePoses(const std::vector<bool>& image_used, const std::vector<SE3d>& poses, const char* path) {
  using namespace io_detail;
  if (image_used.size() != poses.size()) throw std::runtime_error("image_used and poses differ in size");  // CHECK_EQ :791
  std::string out =
      "# Each pose gives the B_tr_A transformation (i.e., A to B with right-multiplication), where the spaces A and B "
      "are defined by the filename. Quaternions are written as used by the Eigen library.\n";
  out += "pose_count: " + std::to_string(image_used.size()) + "\nposes:\n";
  std::string obj;
  for (size_t i = 0; i < poses.size(); ++i) {
    if (!image_used[i]) continue;
    const SE3d& T = poses[i];
    out += "  - index: " + std::to_string(i) + "\n    tx: " + num(T.tx) + "\n    ty: " + num(T.ty) + "\n    tz: " + num(T.tz) +
           "\n    qx: " + num(T.qx) + "\n    qy: " + num(T.qy) + "\n    qz: " + num(T.qz) + "\n    qw: " + num(T.qw) + "\n";
    // camera centre -R^T t
    SE3d inverse_rotation = T;
    inverse_rotation.qx = -T.qx; inverse_rotation.qy = -T.qy; inverse_rotation.qz = -T.qz;
    inverse_rotation.tx = inverse_rotation.ty = inverse_rotation.tz = 0;
    const Vec3d c = apply(inverse_rotation, Vec3d{-T.tx, -T.ty, -T.tz});
    obj += "v " + num(c.x) + " " + num(c.y) + " " + num(c.z) + " 1 0 0\n";
  }
  make_directories(dir_of(path));
  return write_file(path, out) && write_file(std::string(path) + ".obj", obj);
}

// APP/io:841-888
inline bool LoadPoses(std::vector<bool>* image_used, std::vector<SE3d>* poses, const char* path) {
  using namespace io_detail;
  std::string text;
  Document doc;
  if (!read_file(path, &text) || !parse_document(text, &doc)) return false;
  int count = 0;
  if (!get_int(doc, "pose_count", &count) || count < 0) return false;
  image_used->assign(count, false);
  poses->assign(count, SE3d());
  auto it = doc.find("poses");
  if (it == doc.end()) return true;
  if (!it->second.is_block) return false;
  for (const auto& item : it->second.block) {
    long long index;
    double v[7];
    const char* keys[7] = {"qw", "qx", "qy", "qz", "tx", "ty", "tz"};
    auto idx = item.find("index");
    if (idx == item.end() || !to_int(idx->second, &index) || index < 0 || index >= count) return false;
    for (int k = 0; k < 7; ++k) {
      auto f = item.find(keys[k]);
      if (f == item.end() || !to_double(f->second, &v[k])) return false;
    }
    const double norm = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2] + v[3] * v[3]);  // SE3::setQuaternion normalises
    SE3d T;
    T.qw = v[0] / norm; T.qx = v[1] / norm; T.qy = v[2] / norm; T.qz = v[3] / norm;
    T.tx = v[4]; T.ty = v[5]; T.tz = v[6];
    (*image_used)[index] = true;
    (*poses)[index] = T;
  }
  return true;
}

// ---- points ---------------------------------------------------------------------------------------------
// APP/io:890-935. The mapping is written in ascending feature-id order (the reference iterates an
// unordered_map; the order carries no meaning).
inline bool SavePointsAndIndexMapping(const BAState& state, const char* path) {
  using namespace io_detail;
  std::string out = "# Each point is stored as x, y, z.\npoints : [";
  std::string obj;
  for (size_t i = 0; i < state.points.size(); ++i) {
    const Vec3d& p = state.points[i];
    if (i) out += ", ";
    out += num(p.x) + ", " + num(p.y) + ", " + num(p.z);
    obj += "v " + num(p.x) + " " + num(p.y) + " " + num(p.z) + " 0 0 1\n";
  }
  out += "]\nfeature_id_to_point_index:\n";
  std::map<int, int> ordered(state.feature_id_to_points_index.begin(), state.feature_id_to_points_index.end());
  for (const auto& item : ordered)
    out += "  - feature_id: " + std::to_string(item.first) + "\n    point_index: " + std::to_string(item.second) + "\n";
  make_directories(dir_of(path));
  return write_file(path, out) && write_file(std::string(path) + ".obj", obj);
}

// APP/io:937-985
inline bool LoadPointsAndIndexMapping(BAState* state, const char* path) {
  using namespace io_detail;
  std::string text;
  Document doc;
  if (!read_file(path, &text) || !parse_document(text, &doc)) return false;
  const std::vector<double>* flat;
  if (!get_flow(doc, "points", &flat) || flat->size() % 3 != 0) return false;
  std::vector<Vec3d> points(flat->size() / 3);
  for (size_t i = 0; i < points.size(); ++i) points[i] = Vec3d{(*flat)[3 * i], (*flat)[3 * i + 1], (*flat)[3 * i + 2]};
  std::unordered_map<int, int> mapping;
  auto it = doc.find("feature_id_to_point_index");
  if (it != doc.end()) {
    if (!it->second.is_block) return false;
    for (const auto& item : it->second.block) {
      long long id, index;
      auto a = item.find("feature_id"), b = item.find("point_index");
      if (a == item.end() || b == item.end() || !to_int(a->second, &id) || !to_int(b->second, &index)) return false;
      if (index < 0 || static_cast<size_t>(index) >= points.size()) return false;
      mapping[static_cast<int>(id)] = static_cast<int>(index);
    }
  }
  state->points.swap(points);
  state->feature_id_to_points_index.swap(mapping);
  return true;
}

// ---- the state directory --------------------------------------------------------------------------------
// APP/io:432-464
// ---- PNG (8-bit grey or RGB) ------------------------------------------------------------------------------------
// One IDAT chunk holding a zlib stream of stored (uncompressed) deflate blocks of at most 65535 bytes, filter type 0
// on every row: no compression library needed. io.py's EncodePNG writes the same bytes.
namespace io_detail {
inline uint32_t png_crc32(const std::string& data, size_t begin) {
  static uint32_t table[256];
  static bool init = false;
  if (!init) {
    for (uint32_t n = 0; n < 256; ++n) {
      uint32_t c = n;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xedb88320u ^ (c >> 1) : c >> 1;
      table[n] = c;
    }
    init = true;
  }
  uint32_t c = 0xffffffffu;
  for (size_t i = begin; i < data.size(); ++i) c = table[(c ^ static_cast<uint8_t>(data[i])) & 0xff] ^ (c >> 8);
  return c ^ 0xffffffffu;
}
inline uint32_t adler32(const std::string& data) {
  uint32_t a = 1, b = 0;
  for (char ch : data) {
    a = (a + static_cast<uint8_t>(ch)) % 65521u;
    b = (b + a) % 65521u;
  }
  return (b << 16) | a;
}
inline void put_be32(std::string* out, uint32_t v) {
  const char b[4] = {static_cast<char>(v >> 24), static_cast<char>(v >> 16), static_cast<char>(v >> 8), static_cast<char>(v)};
  out->append(b, 4);
}
inline void png_chunk(std::string* out, const char* kind, const std::string& data) {
  put_be32(out, static_cast<uint32_t>(data.size()));
  const size_t start = out->size();
  out->append(kind, 4);
  out->append(data);
  put_be32(out, png_crc32(*out, start));
}
}  // namespace io_detail

// channels: 1 (grey) or 3 (RGB); pixels [height * width * channels], row-major. Returns false if the file cannot be
// written or the arguments are invalid.
inline bool WritePNG(const std::string& path, int width, int height, int channels, const uint8_t* pixels) {
  if (width < 1 || height < 1 || (channels != 1 && channels != 3)) return false;
  const size_t row = static_cast<size_t>(width) * channels;
  std::string raw;
  raw.reserve((row + 1) * height);
  for (int y = 0; y < height; ++y) {
    raw.push_back(0);
    raw.append(reinterpret_cast<const char*>(pixels + y * row), row);
  }
  std::string z("\x78\x01", 2);
  size_t pos = 0;
  do {
    const size_t len = std::min<size_t>(65535, raw.size() - pos);
    const bool final = pos + len >= raw.size();
    z.push_back(final ? 1 : 0);
    const uint16_t l = static_cast<uint16_t>(len), nl = static_cast<uint16_t>(~l);
    const char hdr[4] = {static_cast<char>(l & 0xff), static_cast<char>(l >> 8), static_cast<char>(nl & 0xff), static_cast<char>(nl >> 8)};
    z.append(hdr, 4);
    z.append(raw, pos, len);
    pos += len;
  } while (pos < raw.size());
  io_detail::put_be32(&z, io_detail::adler32(raw));
  std::string ihdr;
  io_detail::put_be32(&ihdr, static_cast<uint32_t>(width));
  io_detail::put_be32(&ihdr, static_cast<uint32_t>(height));
  const char rest[5] = {8, static_cast<char>(channels == 1 ? 0 : 2), 0, 0, 0};
  ihdr.append(rest, 5);
  std::string out("\x89PNG\r\n\x1a\n", 8);
  io_detail::png_chunk(&out, "IHDR", ihdr);
  io_detail::png_chunk(&out, "IDAT", z);
  io_detail::png_chunk(&out, "IEND", std::string());
  return io_detail::write_file(path, out);
}

inline bool SaveBAState(const char* base_path, const BAState& state) {
  using namespace io_detail;
  make_directories(base_path);
  if (!SavePoses(state.image_used, state.rig_tr_global, join(base_path, "rig_tr_global.yaml").c_str())) return false;
  if (!SavePoses(std::vector<bool>(state.camera_tr_rig.size(), true), state.camera_tr_rig,
                 join(base_path, "camera_tr_rig.yaml").c_str()))
    return false;
  for (size_t c = 0; c < state.intrinsics.size(); ++c)
    if (!SaveCameraModel(*state.intrinsics[c], join(base_path, "intrinsics" + std::to_string(c) + ".yaml").c_str())) return false;
  return SavePointsAndIndexMapping(state, join(base_path, "points.yaml").c_str());
}

// APP/io:466-523. With a dataset, the features' point indices are refreshed from the loaded mapping.
inline bool LoadBAState(const char* base_path, BAState* state, Dataset* dataset) {
  using namespace io_detail;
  BAState loaded;
  if (!LoadPoses(&loaded.image_used, &loaded.rig_tr_global, join(base_path, "rig_tr_global.yaml").c_str())) return false;
  std::vector<bool> all_used;
  if (!LoadPoses(&all_used, &loaded.camera_tr_rig, join(base_path, "camera_tr_rig.yaml").c_str())) return false;
  for (int c = 0;; ++c) {
    const std::string path = join(base_path, "intrinsics" + std::to_string(c) + ".yaml");
    if (!file_exists(path)) {
      if (c == 0) return false;
      break;
    }
    std::shared_ptr<CameraModel> model = LoadCameraModel(path.c_str());
    if (!model) return false;
    loaded.intrinsics.push_back(model);
  }
  if (!LoadPointsAndIndexMapping(&loaded, join(base_path, "points.yaml").c_str())) return false;
  if (dataset) {
    // unknown feature ids make the reference's .at() throw: report a malformed pair instead
    for (int i = 0; i < dataset->ImagesetCount(); ++i)
      for (int c = 0; c < dataset->num_cameras(); ++c)
        for (const PointFeature& f : dataset->GetImageset(i)->FeaturesOfCamera(c))
          if (!loaded.feature_id_to_points_index.count(f.id)) return false;
    loaded.ComputeFeatureIdToPointsIndex(dataset);
  }
  *state = loaded;
  return true;
}

// ---- COLMAP text model (the --bundle_adjustment input) ---------------------------------------------------------
// libvis/src/libvis/external_io/colmap_model.cc:96-142: two lines per image, "IMAGE_ID QW QX QY QZ TX TY TZ CAMERA_ID
// NAME" then "X Y POINT3D_ID ..."; the pose is parsed into float like the reference's SE3f, the observations as double
// and then cast to float (io.py reads them the same way). Lines that are empty or start with '#' are skipped.
struct ColmapObservation {
  Vec2f xy;
  long long point3d_id;
};
struct ColmapImage {
  int image_id = 0;
  float q[4] = {1, 0, 0, 0};  // qw qx qy qz
  float t[3] = {0, 0, 0};
  int camera_id = 0;
  std::string file_path;
  std::vector<ColmapObservation> observations;
};
namespace io_detail {
inline std::vector<std::string> split_lines(const std::string& text) {
  std::vector<std::string> lines;
  size_t begin = 0;
  while (true) {
    const size_t end = text.find('\n', begin);
    lines.push_back(text.substr(begin, end == std::string::npos ? std::string::npos : end - begin));
    if (end == std::string::npos) break;
    begin = end + 1;
  }
  return lines;
}
inline std::vector<std::string> split_fields(const std::string& line) {
  std::istringstream in(line);
  std::vector<std::string> fields;
  std::string f;
  while (in >> f) fields.push_back(f);
  return fields;
}
}  // namespace io_detail

// Returns false if the file cannot be read or a line is malformed; `images` is keyed (and so ordered) by image id.
inline bool ReadColmapImages(const std::string& images_txt_path, bool read_observations,
                             std::map<int, ColmapImage>* images) {
  using namespace io_detail;
  std::string text;
  if (!read_file(images_txt_path, &text)) return false;
  const std::vector<std::string> lines = split_lines(text);
  images->clear();
  size_t i = 0;
  while (i < lines.size()) {
    const std::string& line = lines[i++];
    if (line.empty() || line[0] == '#') continue;
    const std::vector<std::string> f = split_fields(line);
    if (f.size() < 9) return false;
    ColmapImage image;
    char* end = nullptr;
    image.image_id = std::atoi(f[0].c_str());
    for (int k = 0; k < 4; ++k) image.q[k] = std::strtof(f[1 + k].c_str(), &end);
    for (int k = 0; k < 3; ++k) image.t[k] = std::strtof(f[5 + k].c_str(), &end);
    image.camera_id = std::atoi(f[8].c_str());
    if (f.size() > 9) image.file_path = f[9];
    const std::string obs_line = i < lines.size() ? lines[i] : std::string();
    ++i;
    if (read_observations) {
      const std::vector<std::string> v = split_fields(obs_line);
      for (size_t k = 0; k + 2 < v.size(); k += 3) {
        ColmapObservation o;
        o.xy = Vec2f{static_cast<float>(std::strtod(v[k].c_str(), &end)),
                     static_cast<float>(std::strtod(v[k + 1].c_str(), &end))};
        o.point3d_id = static_cast<long long>(std::strtod(v[k + 2].c_str(), &end));
        image.observations.push_back(o);
      }
    }
    (*images)[image.image_id] = image;
  }
  return true;
}

// colmap_model.cc:265-299: "ID X Y Z R G B ERROR track..." (positions as float; colours, error and tracks ignored)
inline bool ReadColmapPoints3D(const std::string& points3d_txt_path, std::map<int, Vec3d>* points) {
  using namespace io_detail;
  std::string text;
  if (!read_file(points3d_txt_path, &text)) return false;
  points->clear();
  for (const std::string& line : split_lines(text)) {
    if (line.empty() || line[0] == '#') continue;
    const std::vector<std::string> f = split_fields(line);
    if (f.size() < 4) return false;
    char* end = nullptr;
    (*points)[std::atoi(f[0].c_str())] = Vec3d{static_cast<double>(std::strtof(f[1].c_str(), &end)),
                                               static_cast<double>(std::strtof(f[2].c_str(), &end)),
                                               static_cast<double>(std::strtof(f[3].c_str(), &end))};
  }
  return true;
}

// tools/bundle_adjustment.cc:110-184: a COLMAP text model and the camera `model` -> (dataset, state). Images and
// points are ordered by increasing id, observations without a 3D point (id -1) are dropped, the single rig pose is the
// identity and every image is used; the float quaternion is normalised in double. Returns false if a file cannot be
// read; throws std::out_of_range for an observation of an unknown point.
inline bool LoadColmapProblem(const std::shared_ptr<CameraModel>& model, const std::string& model_input_directory,
                              std::shared_ptr<Dataset>* dataset, BAState* state) {
  using namespace io_detail;
  std::map<int, ColmapImage> images;
  std::map<int, Vec3d> points;
  if (!ReadColmapImages(join(model_input_directory, "images.txt"), true, &images) ||
      !ReadColmapPoints3D(join(model_input_directory, "points3D.txt"), &points))
    return false;
  auto ds = std::make_shared<Dataset>(1);
  ds->SetImageSize(0, model->width(), model->height());
  BAState st;
  st.intrinsics = {model};
  st.camera_tr_rig = {SE3d()};
  st.image_used.assign(images.size(), true);
  for (const auto& item : images) {
    const ColmapImage& image = item.second;
    const double q[4] = {image.q[0], image.q[1], image.q[2], image.q[3]};
    const double n = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    SE3d T;
    T.qw = q[0] / n; T.qx = q[1] / n; T.qy = q[2] / n; T.qz = q[3] / n;
    T.tx = image.t[0]; T.ty = image.t[1]; T.tz = image.t[2];
    st.rig_tr_global.push_back(T);
    std::shared_ptr<Imageset> set = ds->NewImageset();
    set->SetFilename(image.file_path);
    for (const ColmapObservation& o : image.observations) {
      if (o.point3d_id < 0) continue;
      PointFeature feature;
      feature.xy = o.xy;
      feature.id = static_cast<int>(o.point3d_id);
      set->FeaturesOfCamera(0).push_back(feature);
    }
  }
  for (const auto& item : points) {
    st.feature_id_to_points_index[item.first] = static_cast<int>(st.points.size());
    st.points.push_back(item.second);
  }
  st.ComputeFeatureIdToPointsIndex(ds.get());
  *dataset = ds;
  *state = st;
  return true;
}

// ---- MeshLab project (the --compare_reconstructions output) -------------------------------------------------------
// The bytes libvis' WriteMeshLabProject (external_io/meshlab_project.cc:81-111) saves through tinyxml2: one <MLMesh>
// per mesh, attributes escaped as tinyxml2 escapes them (& " ' < >), the matrix cast to float and printed as
// std::ostream prints a float (%g), each value followed by a space and each row by a newline. io.py's
// EncodeMeshLabProject writes the same bytes.
struct MeshLabMesh {
  std::string label, filename;
  double global_tr_mesh[16];  // row-major
};
namespace io_detail {
inline std::string xml_attribute(const std::string& s) {
  std::string out;
  for (char ch : s) {
    switch (ch) {
      case '&': out += "&amp;"; break;
      case '"': out += "&quot;"; break;
      case '\'': out += "&apos;"; break;
      case '<': out += "&lt;"; break;
      case '>': out += "&gt;"; break;
      default: out += ch;
    }
  }
  return out;
}
}  // namespace io_detail
inline std::string EncodeMeshLabProject(const std::vector<MeshLabMesh>& meshes) {
  using namespace io_detail;
  std::string out = "<MeshLabProject>\n    <MeshGroup>\n";
  for (const MeshLabMesh& mesh : meshes) {
    out += "        <MLMesh label=\"" + xml_attribute(mesh.label) + "\" filename=\"" + xml_attribute(mesh.filename) +
           "\">\n            <MLMatrix44>\n";
    for (int r = 0; r < 4; ++r) {
      for (int c = 0; c < 4; ++c) {
        char buf[64];
        std::snprintf(buf, sizeof(buf), "%g ", static_cast<double>(static_cast<float>(mesh.global_tr_mesh[4 * r + c])));
        out += buf;
      }
      out += "\n";
    }
    out += "</MLMatrix44>\n        </MLMesh>\n";
  }
  return out + "    </MeshGroup>\n</MeshLabProject>\n";
}
inline bool WriteMeshLabProject(const std::string& path, const std::vector<MeshLabMesh>& meshes) {
  return io_detail::write_file(path, EncodeMeshLabProject(meshes));
}

// ---- calibration visualisation inputs (the --visualize_kalibr_calibration / --visualize_colmap_calibration tools) ----
// Numbers are read from whole tokens as strtod / strtol read them, restricted to decimal texts (no hex, no '_'): io.py's
// ParseDecimal / ParseInt32 accept exactly the same texts.
namespace io_detail {
inline bool is_decimal_text(const std::string& t) {
  size_t i = 0;
  const size_t n = t.size();
  if (i < n && (t[i] == '+' || t[i] == '-')) ++i;
  std::string rest = t.substr(i);
  for (char& ch : rest) ch = static_cast<char>(std::tolower(static_cast<unsigned char>(ch)));
  if (rest == "inf" || rest == "infinity" || rest == "nan") return true;
  auto digit = [&](size_t k) { return k < n && t[k] >= '0' && t[k] <= '9'; };
  size_t digits = 0;
  while (digit(i)) ++i, ++digits;
  if (i < n && t[i] == '.') {
    ++i;
    while (digit(i)) ++i, ++digits;
  }
  if (digits == 0) return false;
  if (i < n && (t[i] == 'e' || t[i] == 'E')) {
    ++i;
    if (i < n && (t[i] == '+' || t[i] == '-')) ++i;
    size_t exponent_digits = 0;
    while (digit(i)) ++i, ++exponent_digits;
    if (exponent_digits == 0) return false;
  }
  return i == n;
}
}  // namespace io_detail
inline bool ParseDecimal(const std::string& text, double* v) {
  if (!io_detail::is_decimal_text(text)) return false;
  *v = std::strtod(text.c_str(), nullptr);
  return true;
}
inline bool ParseInt32(const std::string& text, int* v) {
  size_t i = (!text.empty() && (text[0] == '+' || text[0] == '-')) ? 1 : 0;
  if (i == text.size()) return false;
  for (size_t k = i; k < text.size(); ++k)
    if (text[k] < '0' || text[k] > '9') return false;
  errno = 0;
  const long long x = std::strtoll(text.c_str(), nullptr, 10);
  if (errno != 0 || x < -2147483648LL || x > 2147483647LL) return false;
  *v = static_cast<int>(x);
  return true;
}

// One camera of a Kalibr camchain: the texts of its fields (io.py's ReadKalibrCamchain returns the same). A model that is
// absent or not a scalar reads as ""; has_* is false for a number list that is absent or not a flat list.
struct KalibrCamera {
  std::string name, camera_model, distortion_model;
  bool has_resolution = false, has_distortion_coeffs = false, has_intrinsics = false;
  std::vector<std::string> resolution, distortion_coeffs, intrinsics;
};
namespace io_detail {
// a YAML value of the subset of Kalibr's camchain files: a scalar, a flat list of scalars (flow or block), or anything
// else (nested lists such as T_cn_cnm1, nested maps), which is skipped
struct KalibrValue {
  enum Kind { kScalar, kList, kOther } kind = kOther;
  std::string scalar;
  std::vector<std::string> items;
};
inline std::string unquote(const std::string& s) {
  if (s.size() >= 2 && (s[0] == '"' || s[0] == '\'') && s.back() == s[0]) return s.substr(1, s.size() - 2);
  return s;
}
inline size_t indent_of(const std::string& line) {
  size_t k = 0;
  while (k < line.size() && line[k] == ' ') ++k;
  return k;
}
// value text behind "key:"; a flow list may continue on the following lines (*i is advanced past them)
inline bool kalibr_value(const std::string& value, const std::vector<std::string>& lines, size_t* i, KalibrValue* out) {
  if (value.empty() || value[0] != '[') {
    out->kind = KalibrValue::kScalar;
    out->scalar = unquote(value);
    return true;
  }
  std::string body = value.substr(1);
  while (body.find(']') == std::string::npos) {
    if (*i >= lines.size()) return false;
    body += " " + lines[(*i)++];
  }
  if (!trim(body.substr(body.find(']') + 1)).empty()) return false;
  body.resize(body.find(']'));
  out->kind = KalibrValue::kList;
  if (body.find('[') != std::string::npos) out->kind = KalibrValue::kOther;
  const std::string t = trim(body);
  for (size_t a = 0; !t.empty() && a <= t.size();) {
    size_t b = t.find(',', a);
    if (b == std::string::npos) b = t.size();
    out->items.push_back(unquote(trim(t.substr(a, b - a))));
    a = b + 1;
  }
  return true;
}
}  // namespace io_detail

// The cameras of a Kalibr camchain YAML file as VisualizeKalibrCalibration reads them (APP/tools/visualize_calibration.cc
// :98-165): cam0, cam1, ... up to the first missing key, every field kept as text. The reference parses the file with
// yaml-cpp; the reader below understands what Kalibr writes: top-level `camN:` maps whose entries are `key: scalar`,
// `key: [flow, list]` (possibly spanning lines) or `key:` followed by a block list (`- 752`, or `- [...]` rows as in
// T_cn_cnm1, which are skipped), and `#` comments. Returns false if the file cannot be read or is not such a map.
inline bool ReadKalibrCamchain(const std::string& camchain_path, std::vector<KalibrCamera>* cameras) {
  using namespace io_detail;
  std::string text;
  if (!read_file(camchain_path, &text)) return false;
  std::vector<std::string> lines;
  for (std::string l : split_lines(text)) {
    for (size_t k = 0; k < l.size(); ++k)
      if (l[k] == '#' && (k == 0 || l[k - 1] == ' ' || l[k - 1] == '\t')) {
        l.resize(k);
        break;
      }
    while (!l.empty() && (l.back() == ' ' || l.back() == '\t' || l.back() == '\r')) l.pop_back();
    lines.push_back(l);
  }
  std::map<std::string, std::map<std::string, KalibrValue>> doc;
  size_t i = 0;
  while (i < lines.size()) {
    if (lines[i].empty()) { ++i; continue; }
    if (indent_of(lines[i]) != 0 || lines[i][0] == '-' || lines[i].find('\t') == 0) return false;
    std::string key, value;
    if (!split_key(lines[i++], &key, &value)) return false;
    std::map<std::string, KalibrValue>& node = doc[key];
    node.clear();
    if (!value.empty()) {  // a top-level scalar or list: not a camera map
      KalibrValue ignored;
      if (!kalibr_value(value, lines, &i, &ignored)) return false;
      continue;
    }
    size_t map_indent = 0;
    while (i < lines.size()) {
      const std::string& line = lines[i];
      if (line.empty()) { ++i; continue; }
      const size_t ind = indent_of(line);
      if (ind == 0 && line[0] != '-') break;  // the next top-level key
      if (map_indent == 0) {
        if (line[ind] == '-') {  // a top-level key holding a list: not a camera map
          while (i < lines.size() && (lines[i].empty() || indent_of(lines[i]) > 0 || lines[i][0] == '-')) ++i;
          break;
        }
        map_indent = ind;
      }
      if (ind != map_indent || line[ind] == '-') return false;
      std::string k, v;
      if (!split_key(line.substr(ind), &k, &v)) return false;
      ++i;
      KalibrValue& field = node[k];
      field = KalibrValue();
      if (!v.empty()) {
        if (!kalibr_value(v, lines, &i, &field)) return false;
        continue;
      }
      // a block below the key: list items at the key's indentation or deeper, or a nested map
      field.kind = KalibrValue::kList;
      while (i < lines.size()) {
        const std::string& item = lines[i];
        if (item.empty()) { ++i; continue; }
        const size_t item_ind = indent_of(item);
        if (item_ind < map_indent || (item_ind == map_indent && item[item_ind] != '-')) break;
        ++i;
        const std::string t = trim(item.substr(item_ind));
        if (t[0] != '-') {
          field.kind = KalibrValue::kOther;
          continue;
        }
        const std::string entry = trim(t.substr(1));
        std::string ek, ev;
        if (entry.empty() || entry[0] == '[' || entry[0] == '-' || split_key(entry, &ek, &ev)) {
          field.kind = KalibrValue::kOther;
          if (!entry.empty() && entry[0] == '[') {
            KalibrValue row;
            if (!kalibr_value(entry, lines, &i, &row)) return false;
          }
          continue;
        }
        field.items.push_back(unquote(entry));
      }
      if (field.kind != KalibrValue::kList) field.items.clear();
    }
  }
  if (doc.empty()) return false;  // no map at all
  cameras->clear();
  for (int c = 0;; ++c) {
    const std::string name = "cam" + std::to_string(c);
    auto it = doc.find(name);
    if (it == doc.end()) break;
    KalibrCamera cam;
    cam.name = name;
    const std::map<std::string, KalibrValue>& node = it->second;
    auto scalar = [&](const char* key) {
      auto f = node.find(key);
      return (f != node.end() && f->second.kind == KalibrValue::kScalar) ? f->second.scalar : std::string();
    };
    auto list = [&](const char* key, std::vector<std::string>* out) {
      auto f = node.find(key);
      if (f == node.end() || f->second.kind != KalibrValue::kList) return false;
      *out = f->second.items;
      return true;
    };
    cam.camera_model = scalar("camera_model");
    cam.distortion_model = scalar("distortion_model");
    cam.has_resolution = list("resolution", &cam.resolution);
    cam.has_distortion_coeffs = list("distortion_coeffs", &cam.distortion_coeffs);
    cam.has_intrinsics = list("intrinsics", &cam.intrinsics);
    cameras->push_back(cam);
  }
  return true;
}

// width, height and k1 k2 r1 r2 fx fy cx cy (distortion_coeffs followed by intrinsics, as the reference concatenates
// them) of a pinhole-radtan camera; false unless the resolution holds 2 ints and there are exactly 4 distortion
// coefficients and 4 intrinsics, all numbers (the reference reads out of bounds with fewer).
inline bool KalibrRadtanParameters(const KalibrCamera& camera, int* width, int* height, double params[8]) {
  if (!camera.has_resolution || !camera.has_distortion_coeffs || !camera.has_intrinsics || camera.resolution.size() != 2 ||
      camera.distortion_coeffs.size() != 4 || camera.intrinsics.size() != 4)
    return false;
  if (!ParseInt32(camera.resolution[0], width) || !ParseInt32(camera.resolution[1], height)) return false;
  for (int k = 0; k < 8; ++k)
    if (!ParseDecimal(k < 4 ? camera.distortion_coeffs[k] : camera.intrinsics[k - 4], &params[k])) return false;
  return true;
}

// libvis/src/libvis/external_io/colmap_model.cc:47-72: one camera per line, "CAMERA_ID MODEL WIDTH HEIGHT PARAMS[]";
// lines that are empty or start with '#' are skipped. The cameras come in file order; of an id that appears twice the
// first is kept (the reference's unordered_map::insert). The parameters are what libstdc++'s
// `while (!eof) { push_back(0); stream >> back(); }` reads: a line that ends in whitespace (a blank, a tab, a carriage
// return) gets one more parameter, 0. Where the reference never ends (a token that is not a number) the parameters stop
// before that token; a line whose first four fields are not an int, a name and two ints is skipped. Returns false if
// the file cannot be read. io.py's ReadColmapCameras returns the same.
struct ColmapCamera {
  int camera_id = 0;
  std::string model_name;
  int width = 0, height = 0;
  std::vector<double> parameters;
};
inline bool ReadColmapCameras(const std::string& cameras_txt_path, std::vector<ColmapCamera>* cameras) {
  using namespace io_detail;
  std::string text;
  if (!read_file(cameras_txt_path, &text)) return false;
  cameras->clear();
  std::vector<int> seen;
  auto space = [](char ch) { return ch == ' ' || ch == '\t' || ch == '\v' || ch == '\f' || ch == '\r'; };
  for (const std::string& line : split_lines(text)) {
    if (line.empty() || line[0] == '#') continue;
    std::vector<std::string> tokens;
    for (size_t a = 0; a < line.size();) {
      while (a < line.size() && space(line[a])) ++a;
      size_t b = a;
      while (b < line.size() && !space(line[b])) ++b;
      if (b > a) tokens.push_back(line.substr(a, b - a));
      a = b;
    }
    ColmapCamera cam;
    if (tokens.size() < 4 || !ParseInt32(tokens[0], &cam.camera_id) || !ParseInt32(tokens[2], &cam.width) ||
        !ParseInt32(tokens[3], &cam.height))
      continue;
    cam.model_name = tokens[1];
    bool stopped = false;
    for (size_t k = 4; k < tokens.size(); ++k) {
      double v;
      if (!ParseDecimal(tokens[k], &v)) {
        stopped = true;
        break;
      }
      cam.parameters.push_back(v);
    }
    if (!stopped && space(line.back())) cam.parameters.push_back(0.0);
    if (std::find(seen.begin(), seen.end(), cam.camera_id) != seen.end()) continue;
    seen.push_back(cam.camera_id);
    cameras->push_back(cam);
  }
  return true;
}

// k1 k2 r1 r2 fx fy cx cy of an OPENCV camera (COLMAP's fx fy cx cy k1 k2 p1 p2 with the halves swapped,
// visualize_calibration.cc:181-198); false with fewer than 8 parameters.
inline bool ColmapRadtanParameters(const ColmapCamera& camera, double params[8]) {
  if (camera.parameters.size() < 8) return false;
  for (int k = 0; k < 4; ++k) {
    params[k] = camera.parameters[4 + k];
    params[4 + k] = camera.parameters[k];
  }
  return true;
}

// legend_error_directions.png of CreateLegends (APP/tools/create_legends.cc:35-54): 200 x 200 RGB pixels, the offset
// e = (x + 0.5f, y + 0.5f) - (100, 100) in float, dir = (double)atan2f(e.y, e.x), colour (127 + 127 sin(dir) + 0.5,
// 127 + 127 cos(dir) + 0.5, 127) in double, truncated. io.py's LegendErrorDirectionsImage computes the same bytes with
// the same C library.
inline std::vector<uint8_t> LegendErrorDirections() {
  std::vector<uint8_t> image(200 * 200 * 3);
  for (int y = 0; y < 200; ++y)
    for (int x = 0; x < 200; ++x) {
      const float ex = (static_cast<float>(x) + 0.5f) - 100.f, ey = (static_cast<float>(y) + 0.5f) - 100.f;
      const double dir = static_cast<double>(atan2f(ey, ex));
      uint8_t* p = &image[3 * (200 * y + x)];
      p[0] = static_cast<uint8_t>(127 + 127 * std::sin(dir) + 0.5);
      p[1] = static_cast<uint8_t>(127 + 127 * std::cos(dir) + 0.5);
      p[2] = 127;
    }
  return image;
}

// ---- pattern YAML files (feature_detector_tagged_pattern.cc:175-196) ------------------------------------------------
// The subset the pattern files use: top-level `key: scalar`, the `page:` map of scalars and the `apriltags:` block list
// of flat maps (`- tag_x: 6` followed by the item's other keys, indented), `#` comments. Floats are read with strtof
// (what yaml-cpp's as<float>() reads), integers as decimal int32. io.py's LoadPatternYAML reads the same values.
struct PatternFile {
  int num_star_segments = 0, squares_x = 0, squares_y = 0;
  float page_width_mm = 0, page_height_mm = 0, pattern_start_x_mm = 0, pattern_start_y_mm = 0, pattern_end_x_mm = 0,
        pattern_end_y_mm = 0;
  struct Tag {
    int x, y, width, height, index;
  };
  std::vector<Tag> tags;
};

namespace io_detail {
inline std::string strip_comment(const std::string& line) {
  char quote = 0;
  for (size_t i = 0; i < line.size(); ++i) {
    const char c = line[i];
    if (quote) {
      if (c == quote) quote = 0;
    } else if (c == '"' || c == '\'') {
      quote = c;
    } else if (c == '#' && (i == 0 || line[i - 1] == ' ' || line[i - 1] == '\t')) {
      return line.substr(0, i);
    }
  }
  return line;
}
inline bool pattern_float(const std::map<std::string, std::string>& m, const char* key, float* out) {
  auto it = m.find(key);
  double unused;
  if (it == m.end() || !ParseDecimal(it->second, &unused)) return false;
  *out = std::strtof(it->second.c_str(), nullptr);
  return true;
}
inline bool pattern_int(const std::map<std::string, std::string>& m, const char* key, int* out) {
  auto it = m.find(key);
  return it != m.end() && ParseInt32(it->second, out);
}
}  // namespace io_detail

// Returns false when the file cannot be read or a field is missing or not a number.
inline bool LoadPatternYAML(const std::string& path, PatternFile* pattern) {
  std::string text;
  if (!io_detail::read_file(path, &text)) return false;
  std::map<std::string, std::string> top, page;
  std::vector<std::map<std::string, std::string>> tags;
  std::string section;  // "page" or "apriltags" while inside that block
  for (std::string line : io_detail::split_lines(text)) {
    if (!line.empty() && line.back() == '\r') line.pop_back();
    line = io_detail::strip_comment(line);
    if (io_detail::trim(line).empty()) continue;
    const size_t indent = line.find_first_not_of(" \t");
    std::string body = line.substr(indent);
    if (indent == 0) {
      section.clear();
      const size_t colon = body.find(':');
      if (colon == std::string::npos) return false;
      const std::string key = io_detail::trim(body.substr(0, colon));
      const std::string value = io_detail::trim(body.substr(colon + 1));
      if (value.empty() && (key == "page" || key == "apriltags")) {
        section = key;
      } else if (!(key == "apriltags" && value == "[]")) {  // "apriltags: []" is a pattern without tags
        top[key] = io_detail::unquote(value);
      }
      continue;
    }
    if (section.empty()) return false;
    std::map<std::string, std::string>* target = &page;
    if (section == "apriltags") {
      if (body[0] == '-') {
        tags.emplace_back();
        body = io_detail::trim(body.substr(1));
        if (body.empty()) continue;
      } else if (tags.empty()) {
        return false;
      }
      target = &tags.back();
    }
    const size_t colon = body.find(':');
    if (colon == std::string::npos) return false;
    (*target)[io_detail::trim(body.substr(0, colon))] = io_detail::unquote(io_detail::trim(body.substr(colon + 1)));
  }
  PatternFile p;
  if (!io_detail::pattern_int(top, "num_star_segments", &p.num_star_segments) ||
      !io_detail::pattern_int(top, "squares_x", &p.squares_x) || !io_detail::pattern_int(top, "squares_y", &p.squares_y) ||
      !io_detail::pattern_float(page, "width_mm", &p.page_width_mm) ||
      !io_detail::pattern_float(page, "height_mm", &p.page_height_mm) ||
      !io_detail::pattern_float(page, "pattern_start_x_mm", &p.pattern_start_x_mm) ||
      !io_detail::pattern_float(page, "pattern_start_y_mm", &p.pattern_start_y_mm) ||
      !io_detail::pattern_float(page, "pattern_end_x_mm", &p.pattern_end_x_mm) ||
      !io_detail::pattern_float(page, "pattern_end_y_mm", &p.pattern_end_y_mm))
    return false;
  for (const auto& t : tags) {
    PatternFile::Tag tag;
    if (!io_detail::pattern_int(t, "tag_x", &tag.x) || !io_detail::pattern_int(t, "tag_y", &tag.y) ||
        !io_detail::pattern_int(t, "width", &tag.width) || !io_detail::pattern_int(t, "height", &tag.height) ||
        !io_detail::pattern_int(t, "index", &tag.index))
      return false;
    p.tags.push_back(tag);
  }
  *pattern = p;
  return true;
}

// ---- PNG reading ----------------------------------------------------------------------------------------------------
// 8-bit, non-interlaced PNGs of colour type 0, 2, 4 or 6, any filter types, IDAT split over any number of chunks, as
// a grey image converted as libvis' libpng reader converts it (image_io_libpng.cc:219-226): alpha is dropped; a pixel
// with r == g == b is that value, any other RGB pixel is (6968 r + 23434 g + 2366 b) >> 15 (libpng's default
// rgb_to_gray weights, truncated; gAMA, sRGB and other ancillary chunks are ignored). The zlib stream is inflated
// here (stored, fixed- and dynamic-Huffman blocks), so no compression library is needed. io.py's DecodePNG decodes
// to the same pixels.
namespace io_detail {
struct Inflate {
  const uint8_t* in;
  size_t n, pos = 0;
  uint32_t bitbuf = 0;
  int bitcnt = 0;
  std::string* out;
  bool error = false;

  struct Huffman {
    short count[16];
    short symbol[288];
  };
  int bits(int need) {
    uint32_t val = bitbuf;
    while (bitcnt < need) {
      if (pos >= n) {
        error = true;
        return 0;
      }
      val |= static_cast<uint32_t>(in[pos++]) << bitcnt;
      bitcnt += 8;
    }
    bitbuf = val >> need;
    bitcnt -= need;
    return static_cast<int>(val & ((1u << need) - 1));
  }
  // canonical code from code lengths; false for an over-subscribed set
  static bool construct(Huffman* h, const short* length, int n) {
    for (int len = 0; len < 16; ++len) h->count[len] = 0;
    for (int s = 0; s < n; ++s) h->count[length[s]]++;
    int left = 1;
    for (int len = 1; len < 16; ++len) {
      left <<= 1;
      left -= h->count[len];
      if (left < 0) return false;
    }
    short offs[16];
    offs[1] = 0;
    for (int len = 1; len < 15; ++len) offs[len + 1] = offs[len] + h->count[len];
    for (int s = 0; s < n; ++s)
      if (length[s] != 0) h->symbol[offs[length[s]]++] = static_cast<short>(s);
    return true;
  }
  int decode(const Huffman& h) {
    int code = 0, first = 0, index = 0;
    for (int len = 1; len < 16; ++len) {
      code |= bits(1);
      if (error) return -1;
      const int count = h.count[len];
      if (code - count < first) return h.symbol[index + (code - first)];
      index += count;
      first += count;
      first <<= 1;
      code <<= 1;
    }
    error = true;
    return -1;
  }
  bool stored() {
    bitbuf = 0;
    bitcnt = 0;
    if (pos + 4 > n) return false;
    const unsigned len = in[pos] | (in[pos + 1] << 8);
    const unsigned nlen = in[pos + 2] | (in[pos + 3] << 8);
    pos += 4;
    if (len != (~nlen & 0xffffu) || pos + len > n) return false;
    out->append(reinterpret_cast<const char*>(in + pos), len);
    pos += len;
    return true;
  }
  bool codes(const Huffman& lencode, const Huffman& distcode) {
    static const short lbase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                    31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
    static const short lext[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
    static const short dbase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                    193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    static const short dext[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
    for (;;) {
      int symbol = decode(lencode);
      if (symbol < 0 || error) return false;
      if (symbol < 256) {
        out->push_back(static_cast<char>(symbol));
      } else if (symbol == 256) {
        return true;
      } else {
        symbol -= 257;
        if (symbol >= 29) return false;
        const int len = lbase[symbol] + bits(lext[symbol]);
        const int dsym = decode(distcode);
        if (dsym < 0 || dsym >= 30 || error) return false;
        const size_t dist = static_cast<size_t>(dbase[dsym] + bits(dext[dsym]));
        if (error || dist > out->size()) return false;
        for (int k = 0; k < len; ++k) out->push_back((*out)[out->size() - dist]);
      }
    }
  }
  bool fixed() {
    static Huffman lencode, distcode;
    static bool init = false;
    if (!init) {
      short lengths[288];
      int s = 0;
      for (; s < 144; ++s) lengths[s] = 8;
      for (; s < 256; ++s) lengths[s] = 9;
      for (; s < 280; ++s) lengths[s] = 7;
      for (; s < 288; ++s) lengths[s] = 8;
      construct(&lencode, lengths, 288);
      for (s = 0; s < 30; ++s) lengths[s] = 5;
      construct(&distcode, lengths, 30);
      init = true;
    }
    return codes(lencode, distcode);
  }
  bool dynamic() {
    static const short order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    const int nlen = bits(5) + 257, ndist = bits(5) + 1, ncode = bits(4) + 4;
    if (error || nlen > 286 || ndist > 30) return false;
    short lengths[320];
    int index = 0;
    for (; index < ncode; ++index) lengths[order[index]] = static_cast<short>(bits(3));
    for (; index < 19; ++index) lengths[order[index]] = 0;
    if (error) return false;
    Huffman lencode, distcode;
    if (!construct(&lencode, lengths, 19)) return false;
    index = 0;
    while (index < nlen + ndist) {
      int symbol = decode(lencode);
      if (symbol < 0 || error) return false;
      if (symbol < 16) {
        lengths[index++] = static_cast<short>(symbol);
      } else {
        short len = 0;
        int repeat;
        if (symbol == 16) {
          if (index == 0) return false;
          len = lengths[index - 1];
          repeat = 3 + bits(2);
        } else if (symbol == 17) {
          repeat = 3 + bits(3);
        } else {
          repeat = 11 + bits(7);
        }
        if (error || index + repeat > nlen + ndist) return false;
        while (repeat--) lengths[index++] = len;
      }
    }
    if (lengths[256] == 0) return false;
    if (!construct(&lencode, lengths, nlen) || !construct(&distcode, lengths + nlen, ndist)) return false;
    return codes(lencode, distcode);
  }
  // a zlib stream (RFC 1950) holding deflate blocks (RFC 1951); checks the header and the Adler-32
  bool zlib() {
    if (n < 6 || (in[0] & 0x0f) != 8 || ((in[0] << 8) | in[1]) % 31 != 0 || (in[1] & 0x20)) return false;
    pos = 2;
    int last;
    do {
      last = bits(1);
      const int type = bits(2);
      if (error) return false;
      const bool ok = type == 0 ? stored() : type == 1 ? fixed() : type == 2 ? dynamic() : false;
      if (!ok || error) return false;
    } while (!last);
    if (pos + 4 > n) return false;
    const uint32_t want = (static_cast<uint32_t>(in[pos]) << 24) | (in[pos + 1] << 16) | (in[pos + 2] << 8) | in[pos + 3];
    return want == adler32(*out);
  }
};
inline uint32_t be32(const std::string& s, size_t at) {
  return (static_cast<uint32_t>(static_cast<uint8_t>(s[at])) << 24) | (static_cast<uint8_t>(s[at + 1]) << 16) |
         (static_cast<uint8_t>(s[at + 2]) << 8) | static_cast<uint8_t>(s[at + 3]);
}
}  // namespace io_detail

// grey [height * width], row-major. Returns false with a message in *error for anything unsupported or broken.
inline bool DecodePNG(const std::string& data, int* width, int* height, std::vector<uint8_t>* grey, std::string* error) {
  auto fail = [&](const std::string& m) {
    if (error) *error = "DecodePNG: " + m;
    return false;
  };
  if (data.size() < 8 || data.compare(0, 8, std::string("\x89PNG\r\n\x1a\n", 8)) != 0) return fail("not a PNG file");
  size_t pos = 8;
  bool have_ihdr = false;
  uint32_t w = 0, h = 0;
  int depth = 0, color = 0, compression = 0, filter = 0, interlace = 0;
  std::string idat;
  while (pos + 8 <= data.size()) {
    const uint32_t length = io_detail::be32(data, pos);
    const std::string kind = data.substr(pos + 4, 4);
    if (pos + 12 + static_cast<size_t>(length) > data.size() + 4 || pos + 8 + static_cast<size_t>(length) > data.size())
      return fail("truncated chunk");
    if (kind == "IHDR" && length >= 13) {
      w = io_detail::be32(data, pos + 8);
      h = io_detail::be32(data, pos + 12);
      depth = static_cast<uint8_t>(data[pos + 16]);
      color = static_cast<uint8_t>(data[pos + 17]);
      compression = static_cast<uint8_t>(data[pos + 18]);
      filter = static_cast<uint8_t>(data[pos + 19]);
      interlace = static_cast<uint8_t>(data[pos + 20]);
      have_ihdr = true;
    } else if (kind == "IDAT") {
      idat.append(data, pos + 8, length);
    } else if (kind == "IEND") {
      break;
    }
    pos += 12 + static_cast<size_t>(length);
  }
  if (!have_ihdr) return fail("no IHDR chunk");
  if (depth != 8) return fail("bit depth " + std::to_string(depth) + " is not supported (only 8)");
  const int ch = color == 0 ? 1 : color == 2 ? 3 : color == 4 ? 2 : color == 6 ? 4 : 0;
  if (ch == 0) return fail("colour type " + std::to_string(color) + " is not supported (only 0, 2, 4 and 6)");
  if (interlace != 0) return fail("interlaced images are not supported");
  if (compression != 0 || filter != 0 || w < 1 || h < 1 || w > (1u << 24) || h > (1u << 24)) return fail("invalid IHDR");
  std::string raw;
  io_detail::Inflate inf{reinterpret_cast<const uint8_t*>(idat.data()), idat.size()};
  inf.out = &raw;
  if (!inf.zlib()) return fail("broken zlib stream");
  const size_t stride = static_cast<size_t>(w) * ch;
  if (raw.size() < (stride + 1) * h) return fail("image data too short");
  std::vector<uint8_t> prev(stride, 0), cur(stride);
  grey->assign(static_cast<size_t>(w) * h, 0);
  for (uint32_t y = 0; y < h; ++y) {
    const uint8_t* line = reinterpret_cast<const uint8_t*>(raw.data()) + y * (stride + 1);
    const int ft = line[0];
    if (ft > 4) return fail("unknown filter type " + std::to_string(ft));
    for (size_t x = 0; x < stride; ++x) {
      const int a = x >= static_cast<size_t>(ch) ? cur[x - ch] : 0, b = prev[x];
      const int c = x >= static_cast<size_t>(ch) ? prev[x - ch] : 0;
      int p = 0;
      if (ft == 1) {
        p = a;
      } else if (ft == 2) {
        p = b;
      } else if (ft == 3) {
        p = (a + b) >> 1;
      } else if (ft == 4) {
        const int pa = std::abs(b - c), pb = std::abs(a - c), pc = std::abs(a + b - 2 * c);
        p = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
      }
      cur[x] = static_cast<uint8_t>(line[1 + x] + p);
    }
    for (uint32_t x = 0; x < w; ++x) {
      const uint8_t* px = &cur[static_cast<size_t>(x) * ch];
      uint8_t g = px[0];
      if (ch >= 3 && !(px[0] == px[1] && px[0] == px[2]))
        g = static_cast<uint8_t>((6968u * px[0] + 23434u * px[1] + 2366u * px[2]) >> 15);
      (*grey)[static_cast<size_t>(y) * w + x] = g;
    }
    prev.swap(cur);
  }
  *width = static_cast<int>(w);
  *height = static_cast<int>(h);
  return true;
}

// DecodePNG of the file at path; false with "Cannot read file: ..." when it cannot be read.
inline bool ReadPNG(const std::string& path, int* width, int* height, std::vector<uint8_t>* grey, std::string* error) {
  std::string data;
  if (!io_detail::read_file(path, &data)) {
    if (error) *error = "Cannot read file: " + path;
    return false;
  }
  return DecodePNG(data, width, height, grey, error);
}

}  // namespace b200ba_shim
