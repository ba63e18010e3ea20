// Drives the C++ RefineFeatureDetections of include/b200ba_pipeline.hpp from the command line so that
// tests/test_refine_features.py can compare it with api.RefineFeatures:
//   samples <half> <out.raw>  FeatureSamples(half) as floats
//   refine <pattern.yaml> <images.raw> <width> <height> <n_images> <predictions.raw> <n> <half> <type> <out.raw>
// images.raw: the grey bytes; predictions.raw: n b200ba_feature_prediction records; out.raw: per feature x, y,
// final_cost (float) and status (int32). Exits with the library's return code.
#include <cstdint>
#include <cstdlib>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

static std::vector<char> read_all(const char* path) {
  std::ifstream f(path, std::ios::binary);
  return std::vector<char>(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv) {
  if (argc == 4 && std::string(argv[1]) == "samples") {
    const std::vector<Vec2f> s = FeatureSamples(std::atoi(argv[2]));
    std::ofstream o(argv[3], std::ios::binary);
    o.write(reinterpret_cast<const char*>(s.data()), sizeof(Vec2f) * s.size());
    return s.empty() ? 1 : 0;
  }
  if (argc != 12 || std::string(argv[1]) != "refine") return 2;
  PatternFile file;
  b200ba_pattern pattern;
  if (!LoadPatternYAML(argv[2], &file) || !PatternStruct(file, &pattern)) return 2;
  const std::vector<char> images = read_all(argv[3]);
  const int width = std::atoi(argv[4]), height = std::atoi(argv[5]);
  const int64_t n_images = std::atoll(argv[6]);
  const std::vector<char> raw = read_all(argv[7]);
  const int n = std::atoi(argv[8]);
  if (raw.size() != sizeof(b200ba_feature_prediction) * n) return 2;
  const auto* pred = reinterpret_cast<const b200ba_feature_prediction*>(raw.data());
  std::vector<FeatureDetection> in(n), out(n);
  for (int i = 0; i < n; ++i) {
    in[i].image = pred[i].image;
    in[i].position = Vec2f{pred[i].position[0], pred[i].position[1]};
    in[i].pattern_coordinate = Vec2i{pred[i].pattern_coordinate[0], pred[i].pattern_coordinate[1]};
    std::copy(pred[i].local_pixel_tr_pattern, pred[i].local_pixel_tr_pattern + 9, in[i].local_pixel_tr_pattern);
  }
  std::vector<int32_t> status;
  const int rc = RefineFeatureDetections(pattern, reinterpret_cast<const uint8_t*>(images.data()), width, height,
                                         n_images, std::atoi(argv[9]), std::atoi(argv[10]), n, in.data(), out.data(),
                                         &status);
  if (rc != 0) {
    std::cerr << "RefineFeatureDetections failed (" << rc << "): " << b200ba_last_error(nullptr) << "\n";
    return rc;
  }
  std::ofstream o(argv[11], std::ios::binary);
  for (int i = 0; i < n; ++i) {
    o.write(reinterpret_cast<const char*>(&out[i].position), 8);
    o.write(reinterpret_cast<const char*>(&out[i].final_cost), 4);
    o.write(reinterpret_cast<const char*>(&status[i]), 4);
  }
  return 0;
}
