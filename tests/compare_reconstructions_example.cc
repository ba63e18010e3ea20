// Drives the C++ --bundle_adjustment / --compare_reconstructions code of include/b200ba_pipeline.hpp and
// include/b200ba_io.hpp from the command line so that tests/test_compare_reconstructions.py can compare it with the
// Python mirror (pipeline.py, io.py).
//   compare <reconstruction_1> <reconstruction_2> [pixel_step]   exit code of CompareReconstructions (a device is
//                                                                 needed once both states load and agree)
//   ba <state_directory> <model_input_directory> <model_output_directory> [max_iteration_count]
//   colmap <intrinsics_yaml> <model_input_directory> <output_state_directory> <output_dataset_bin>
//                                                   LoadColmapProblem, then SaveBAState / SaveDataset (no device)
//   mlp <output.mlp>                                WriteMeshLabProject of the meshes on stdin: per mesh the label, the
//                                                   file name and 16 row-major values, one line each (no device)
//   paths <path_1> <path_2> <cwd>                   ReconstructionProjectPaths, one result per line (no device)
#include <cstdio>
#include <cstdlib>
#include <iostream>
#include <sstream>
#include <string>

#include "b200ba_io.hpp"
#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string mode = argv[1];
  try {
    if (mode == "compare" && (argc == 4 || argc == 5))
      return CompareReconstructions(argv[2], argv[3], argc == 5 ? std::atoi(argv[4]) : 10);
    if (mode == "ba" && (argc == 5 || argc == 6))
      return BundleAdjustment(argv[2], argv[3], argv[4], argc == 6 ? std::atoi(argv[5]) : 30);
    if (mode == "colmap" && argc == 6) {
      std::shared_ptr<CameraModel> model = LoadCameraModel(argv[2]);
      std::shared_ptr<Dataset> dataset;
      BAState state;
      if (!model || !LoadColmapProblem(model, argv[3], &dataset, &state)) return 1;
      return SaveBAState(argv[4], state) && SaveDataset(argv[5], *dataset) ? 0 : 3;
    }
    if (mode == "mlp" && argc == 3) {
      std::vector<MeshLabMesh> meshes;
      std::string label, filename, values;
      while (std::getline(std::cin, label) && std::getline(std::cin, filename) && std::getline(std::cin, values)) {
        MeshLabMesh mesh;
        mesh.label = label;
        mesh.filename = filename;
        std::istringstream in(values);
        for (double& v : mesh.global_tr_mesh) in >> v;
        if (!in) return 3;
        meshes.push_back(mesh);
      }
      return WriteMeshLabProject(argv[2], meshes) ? 0 : 1;
    }
    if (mode == "paths" && argc == 5) {
      const MeshLabProjectPaths p = ReconstructionProjectPaths(argv[2], argv[3], argv[4]);
      std::cout << p.project << "\n" << p.rest1 << "\n" << p.rest2 << "\n";
      for (const std::string& f : p.files) std::cout << f << "\n";
      return 0;
    }
  } catch (const std::exception& e) {
    std::printf("exception: %s\n", e.what());
    return 4;
  }
  return 2;
}
