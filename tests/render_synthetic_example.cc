// Drives the C++ side of --render_synthetic_dataset (include/b200ba_pipeline.hpp, include/b200ba_io.hpp) from the
// command line so that tests/test_render_synthetic.py can compare it with the Python mirror:
//   dataset <path> <pattern.yaml> <pattern.png> <num_images> <seed>  exit code of RenderSyntheticDataset
//   decode <file.png> <out.raw>  DecodePNG: writes "<w> <h>\n" and the grey pixels; exit 1 with the message
//   pattern <pattern.yaml>       LoadPatternYAML: prints every field (floats as their bits in hex); exit 1 on failure
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <string>

#include "b200ba_pipeline.hpp"

using namespace b200ba_shim;

static uint32_t bits(float v) {
  uint32_t b;
  std::memcpy(&b, &v, 4);
  return b;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[1];
  if (mode == "dataset" && argc == 7)
    return RenderSyntheticDataset(argv[2], argv[3], argv[4], std::atoi(argv[5]), std::strtoull(argv[6], nullptr, 10));
  if (mode == "decode" && argc == 4) {
    int w = 0, h = 0;
    std::vector<uint8_t> grey;
    std::string error;
    if (!ReadPNG(argv[2], &w, &h, &grey, &error)) {
      std::cout << error << "\n";
      return 1;
    }
    std::string out = std::to_string(w) + " " + std::to_string(h) + "\n";
    out.append(reinterpret_cast<const char*>(grey.data()), grey.size());
    return io_detail::write_file(argv[3], out) ? 0 : 3;
  }
  if (mode == "pattern") {
    PatternFile p;
    if (!LoadPatternYAML(argv[2], &p)) return 1;
    std::printf("%d %d %d\n", p.num_star_segments, p.squares_x, p.squares_y);
    for (float v : {p.page_width_mm, p.page_height_mm, p.pattern_start_x_mm, p.pattern_start_y_mm, p.pattern_end_x_mm,
                    p.pattern_end_y_mm})
      std::printf("%08x\n", bits(v));
    for (const PatternFile::Tag& t : p.tags) std::printf("%d %d %d %d %d\n", t.x, t.y, t.width, t.height, t.index);
    return 0;
  }
  return 2;
}
