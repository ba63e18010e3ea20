// Drives the C++ comparison of two calibrations of include/b200ba_pipeline.hpp from the command line so that
// tests/test_compare_calibrations.py can compare its files with the Python mirror (io.py, pipeline.py).
//   write <path> <count> <sum> <max> <median> <max_error_norm> <max_error_component>
//   compare <calibration_a> <calibration_b> <report base path>   (exit code of CompareCalibrations; a device is
//                                                                  needed once both files load as central-generic
//                                                                  models of one image size)
#include <cstdio>
#include <cstdlib>
#include <string>

#include "b200ba_io.hpp"
#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string mode = argv[1];
  try {
    if (mode == "write" && argc == 9) {
      auto d = [&](int i) { return std::strtod(argv[i], nullptr); };
      b200ba_fitting_report r{};
      r.reprojection_error_count = std::atoll(argv[3]);
      r.reprojection_error_sum = d(4);
      r.reprojection_error_max = d(5);
      r.reprojection_error_median = d(6);
      r.max_error_norm = d(7);
      r.max_error_component = d(8);
      return WriteFittingInfoFile(argv[2], r) ? 0 : 1;
    }
    if (mode == "compare" && argc == 5) return CompareCalibrations(argv[2], argv[3], argv[4]);
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
