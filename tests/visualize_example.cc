// Drives the C++ calibration visualisation code of include/b200ba_pipeline.hpp and include/b200ba_io.hpp from the
// command line so that tests/test_visualize_calibration.py can compare it with the Python mirror (pipeline.py, io.py).
//   kalibr <camchain.yaml>       exit code of VisualizeKalibrCalibration (a device is needed for a usable camera)
//   colmap <cameras.txt>         exit code of VisualizeColmapCalibration (likewise)
//   legends <directory>          exit code of CreateLegends (no device)
//   read_kalibr <camchain.yaml>  ReadKalibrCamchain + KalibrRadtanParameters, one line per camera (no device)
//   read_colmap <cameras.txt>    ReadColmapCameras + ColmapRadtanParameters, one line per camera (no device)
// The read_* modes print numbers with %.17g and exit with 1 where the file cannot be read.
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <string>

#include "b200ba_io.hpp"
#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

static void print_list(bool has, const std::vector<std::string>& items) {
  if (!has) {
    std::printf(" -");
    return;
  }
  std::printf(" [");
  for (size_t k = 0; k < items.size(); ++k) std::printf(k ? ",%s" : "%s", items[k].c_str());
  std::printf("]");
}

static void print_params(bool ok, const double p[8]) {
  if (!ok) {
    std::printf(" none\n");
    return;
  }
  for (int k = 0; k < 8; ++k) std::printf(" %.17g", p[k]);
  std::printf("\n");
}

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  const std::string mode = argv[1];
  try {
    if (mode == "kalibr") return VisualizeKalibrCalibration(argv[2]);
    if (mode == "colmap") return VisualizeColmapCalibration(argv[2]);
    if (mode == "legends") return CreateLegends(argv[2]);
    if (mode == "read_kalibr") {
      std::vector<KalibrCamera> cameras;
      if (!ReadKalibrCamchain(argv[2], &cameras)) return 1;
      for (const KalibrCamera& c : cameras) {
        std::printf("%s|%s|%s|", c.name.c_str(), c.camera_model.c_str(), c.distortion_model.c_str());
        print_list(c.has_resolution, c.resolution);
        print_list(c.has_distortion_coeffs, c.distortion_coeffs);
        print_list(c.has_intrinsics, c.intrinsics);
        int w = 0, h = 0;
        double p[8];
        const bool ok = KalibrRadtanParameters(c, &w, &h, p);
        if (ok) std::printf(" %d %d", w, h);
        print_params(ok, p);
      }
      return 0;
    }
    if (mode == "read_colmap") {
      std::vector<ColmapCamera> cameras;
      if (!ReadColmapCameras(argv[2], &cameras)) return 1;
      for (const ColmapCamera& c : cameras) {
        std::printf("%d|%s|%d|%d|", c.camera_id, c.model_name.c_str(), c.width, c.height);
        for (double v : c.parameters) std::printf(" %.17g", v);
        std::printf("|");
        double p[8];
        print_params(ColmapRadtanParameters(c, p), p);
      }
      return 0;
    }
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
