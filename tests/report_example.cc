// Drives the C++ calibration report of include/b200ba_pipeline.hpp from the command line so that
// tests/test_calibration_report.py can compare its files with the Python mirror (io.py, pipeline.py).
//   write <path> <width> <height> <hfov> <vfov> <imagesets> <localized> <count> <sum> <max> <median> <biasedness>
//   report <dataset.bin> <state directory> <report base path>     (runs b200ba_calibration_report: needs a GPU)
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
    if (mode == "write" && argc == 14) {
      // the camera only supplies the resolution line
      CentralOpenCVModel cam(std::atoi(argv[3]), std::atoi(argv[4]));
      auto d = [&](int i) { return std::strtod(argv[i], nullptr); };
      return WriteReportInfoFile(argv[2], cam, d(5), d(6), std::atoi(argv[7]), std::atoi(argv[8]), std::atoll(argv[9]), d(10),
                                 d(11), d(12), d(13))
                 ? 0
                 : 1;
    }
    if (mode == "report" && argc == 5) {
      std::shared_ptr<Dataset> ds;
      BAState st;
      if (!LoadDataset(argv[2], &ds) || !LoadBAState(argv[3], &st, ds.get())) { std::printf("load failed\n"); return 1; }
      const std::vector<b200ba_camera_report> reports = CreateCalibrationReport(*ds, st, argv[4]);
      for (const b200ba_camera_report& r : reports)
        std::printf("count %lld cells %d\n", static_cast<long long>(r.reprojection_error_count), r.biasedness_cells);
      return 0;
    }
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
