// Drives the C++ side of calibrating from a state (include/b200ba_shim.hpp, b200ba_io.hpp) from the command line so
// that tests/test_calibrate.py can compare its files with the Python mirror. Host logic only.
//   calibrate_example merge <out.bin> <a.bin> [<b.bin> ...]   load, Dataset::Merge in order, save; prints the
//                                                             first imageset index of every dataset
//   calibrate_example outliers <dataset.bin> <state dir> <factor> <out dir>
//                                                             DeleteOutlierFeaturesOnDevice for every camera in order
//                                                             (images under <out dir>/report), then <out dir>/dataset.bin
//                                                             and the state in <out dir>
//   calibrate_example calibrate <model> <levels> <cell> <factor> <state dir> <out dir> <a.bin> [<b.bin> ...]
//                                                             CalibrateFromState; exits with its return code
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>

#include "b200ba_io.hpp"
#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

int main(int argc, char** argv) {
  if (argc >= 4 && std::strcmp(argv[1], "merge") == 0) {
    std::shared_ptr<Dataset> merged;
    for (int i = 3; i < argc; ++i) {
      std::shared_ptr<Dataset> ds;
      if (!LoadDataset(argv[i], &ds)) {
        std::fprintf(stderr, "Cannot read file: %s\n", argv[i]);
        return 1;
      }
      if (!merged) {
        merged = ds;
      } else if (!merged->Merge(*ds)) {
        std::fprintf(stderr, "Cannot merge dataset %s: its camera count or image sizes differ\n", argv[i]);
        return 1;
      }
    }
    if (!SaveDataset(argv[2], *merged)) return 1;
    for (int first : merged->first_imageset_indices_for_datasets) std::printf("%d\n", first);
    return 0;
  }
  if (argc == 6 && std::strcmp(argv[1], "outliers") == 0) {
    std::shared_ptr<Dataset> ds;
    BAState state;
    if (!LoadDataset(argv[2], &ds) || !LoadBAState(argv[3], &state, ds.get())) return 1;
    const std::string out = argv[5];
    const std::string base = out + "/report";
    for (int c = 0; c < ds->num_cameras(); ++c) {
      const b200ba_outlier_report r =
          DeleteOutlierFeaturesOnDevice(c, ds.get(), &state, static_cast<float>(std::atof(argv[4])), base.c_str());
      std::printf("%d %lld %lld %d\n", c, static_cast<long long>(r.removed), static_cast<long long>(r.failed), r.skipped);
    }
    return (SaveDataset((out + "/dataset.bin").c_str(), *ds) && SaveBAState(out.c_str(), state)) ? 0 : 1;
  }
  if (argc >= 9 && std::strcmp(argv[1], "calibrate") == 0) {
    std::vector<std::string> files(argv + 8, argv + argc);
    return CalibrateFromState(files, argv[6], argv[7], argv[2], std::atoi(argv[3]), std::atoi(argv[4]), 0.0,
                              static_cast<float>(std::atof(argv[5])));
  }
  std::fprintf(stderr, "usage: calibrate_example merge <out.bin> <a.bin> [<b.bin> ...] | outliers <dataset.bin> "
                       "<state dir> <factor> <out dir>\n");
  return 2;
}
