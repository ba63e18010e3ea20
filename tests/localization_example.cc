// Drives the C++ localization accuracy test of include/b200ba_pipeline.hpp from the command line so that
// tests/test_localization_accuracy.py can compare its output with the Python mirror (pipeline.py).
//   test <gt_model_yaml> <compared_model_yaml> [trials seed]   (exit code of LocalizationAccuracyTest; a device is
//                                                              needed once both files load as central-generic
//                                                              models of one image size)
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
    if (mode == "test" && argc == 4) return LocalizationAccuracyTest(argv[2], argv[3]);
    if (mode == "test" && argc == 6)
      return LocalizationAccuracyTest(argv[2], argv[3], std::atoll(argv[4]), std::strtoull(argv[5], nullptr, 10));
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
