// Drives the C++ comparison of two calibrations of include/b200ba_pipeline.hpp with its images from the command line,
// so that tests/test_fitting_images.py can compare its files with the Python mirror (pipeline.py).
//   compare <calibration_a> <calibration_b> <report base path> [visualize]   (exit code of CompareCalibrations)
#include <cstdio>
#include <string>

#include "b200ba_io.hpp"
#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

int main(int argc, char** argv) {
  if ((argc != 5 && argc != 6) || std::string(argv[1]) != "compare") return 2;
  const bool visualize = argc == 6 && std::string(argv[5]) == "visualize";
  if (argc == 6 && !visualize) return 2;
  try {
    return CompareCalibrations(argv[2], argv[3], argv[4], visualize);
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
}
