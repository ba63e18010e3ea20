// Drives the C++ report images of include/b200ba_io.hpp and include/b200ba_pipeline.hpp from the command line so
// that tests/test_report_images.py can compare their files with the Python mirror (io.py, pipeline.py).
//   png <raw file> <out.png> <width> <height> <channels>           WritePNG of the raw bytes
//   report <dataset.bin> <state directory> <report base path> <0|1>  CreateCalibrationReport (needs a GPU)
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
    if (mode == "png" && argc == 7) {
      std::string raw;
      if (!io_detail::read_file(argv[2], &raw)) return 1;
      const int w = std::atoi(argv[4]), h = std::atoi(argv[5]), ch = std::atoi(argv[6]);
      if (raw.size() != static_cast<size_t>(w) * h * ch) return 1;
      return WritePNG(argv[3], w, h, ch, reinterpret_cast<const uint8_t*>(raw.data())) ? 0 : 1;
    }
    if (mode == "report" && argc == 6) {
      std::shared_ptr<Dataset> ds;
      BAState st;
      if (!LoadDataset(argv[2], &ds) || !LoadBAState(argv[3], &st, ds.get())) { std::printf("load failed\n"); return 1; }
      CreateCalibrationReport(*ds, st, argv[4], std::atoi(argv[5]) != 0);
      return 0;
    }
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
