// Drives the C++ centre-point analysis of include/b200ba_pipeline.hpp from the command line so that
// tests/test_line_offsets.py can compare its files with the Python mirror (io.py, pipeline.py).
//   obj <lines file> <base path>                                              WriteLineVisualizationOBJ of the raw
//                                                                             [n][4][3] doubles
//   report <dataset.bin> <state directory> <report base path> <0|1> <0|1>     CreateCalibrationReport(visualizations,
//                                                                             line_offsets) (needs a GPU)
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
    if (mode == "obj" && argc == 4) {
      std::string raw;
      if (!io_detail::read_file(argv[2], &raw) || raw.size() % (12 * sizeof(double)) != 0) return 1;
      const int64_t n = static_cast<int64_t>(raw.size() / (12 * sizeof(double)));
      return WriteLineVisualizationOBJ(argv[3], reinterpret_cast<const double*>(raw.data()), n) ? 0 : 1;
    }
    if (mode == "report" && argc == 7) {
      std::shared_ptr<Dataset> ds;
      BAState st;
      if (!LoadDataset(argv[2], &ds) || !LoadBAState(argv[3], &st, ds.get())) { std::printf("load failed\n"); return 1; }
      CreateCalibrationReport(*ds, st, argv[4], std::atoi(argv[5]) != 0, std::atoi(argv[6]) != 0);
      return 0;
    }
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
