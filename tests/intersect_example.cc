// Drives the C++ IntersectDatasets of include/b200ba_pipeline.hpp from the command line so that
// tests/test_intersect_datasets.py can compare it with the Python mirror (pipeline.py) and the restatement
// (tests/intersect_oracle.cc, linked in):
//   device <threshold> <dataset.bin>...  exit code of IntersectDatasets with the feature level on the device
//   oracle <threshold> <dataset.bin>...  the same with the restatement's feature level (no device)
#include <cstdlib>
#include <iostream>
#include <string>
#include <vector>

#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

extern "C" int oracle_intersect_lists(int32_t n_datasets, int64_t n_lists, const int64_t* off, const float* xy,
                                      double threshold, uint8_t* keep, int64_t* counts);

static void intersect_with_oracle(int32_t n_datasets, const std::vector<int64_t>& offsets, const std::vector<float>& xy,
                                  double threshold, std::vector<uint8_t>* keep, b200ba_intersection_report* report) {
  keep->assign(xy.size() / 2, 0);
  int64_t counts[5];
  oracle_intersect_lists(n_datasets, static_cast<int64_t>(offsets.size() - 1) / n_datasets, offsets.data(), xy.data(),
                         threshold, keep->data(), counts);
  report->intersections = counts[0];
  report->kept = counts[1];
  report->uncovered = counts[2];
  report->capped = counts[3];
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[1];
  const double threshold = std::strtod(argv[2], nullptr);
  const std::vector<std::string> paths(argv + 3, argv + argc);
  try {
    if (mode == "device") return IntersectDatasets(paths, threshold);
    if (mode == "oracle") return IntersectDatasets(paths, threshold, intersect_with_oracle);
  } catch (const std::exception& e) {
    std::cerr << "exception: " << e.what() << "\n";
    return 4;
  }
  return 2;
}
