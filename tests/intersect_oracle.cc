// A sequential restatement of --intersect_datasets (APP/tools/intersect_datasets.cc) for
// tests/test_intersect_datasets.py and scripts/intersect_timing.py, which compile it with -ffp-contract=off and load it
// with ctypes. It works as the reference does: on std::vectors of features, erasing elements and stepping the walk
// index back, with the rules pinned in include/b200ba.h where the reference never ends:
//   - a rejected walk that covered nothing in any dataset leaves the feature in place and moves on;
//   - a fixed-point loop stops after 100 passes with the 100th pass's result;
//   - a walked imageset of dataset 0 whose filename no map holds any more (a later duplicate of a filename already
//     deleted) is itself deleted from dataset 0.
//   oracle_intersect_lists     the feature level over the flat lists of b200ba_intersect_features
//   oracle_intersect_datasets  the whole tool: loads the datasets, writes <path><suffix> for each
#include <cstdint>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "b200ba_io.hpp"

using namespace b200ba_shim;

namespace {

struct Counts {
  int64_t intersections = 0, uncovered = 0, capped = 0, reruns = 0;
};

float squared_norm(float x, float y) { return x * x + y * y; }

// The features of one (task, camera), one vector per dataset.
void intersect_camera(const std::vector<std::vector<PointFeature>*>& features, double thr2, Counts* counts) {
  const int n = static_cast<int>(features.size());
  std::vector<Vec2f> centres;
  for (int f = 0; f < static_cast<int>(features[0]->size()); ++f) {
    Vec2f centre = features[0]->at(f).xy;
    std::vector<int> covered(n, -1);
    std::vector<int> previous;
    for (int pass = 1;; ++pass) {
      Vec2f sum{0.f, 0.f};
      int count = 0;
      for (int i = 0; i < n; ++i) {
        int closest = -1;
        double best = thr2;
        for (int o = 0; o < static_cast<int>(features[i]->size()); ++o) {
          const Vec2f p = features[i]->at(o).xy;
          const double d = squared_norm(p.x - centre.x, p.y - centre.y);
          if (d <= best) {
            best = d;
            closest = o;
          }
        }
        covered[i] = closest;
        if (closest >= 0) {
          sum.x += features[i]->at(closest).xy.x;
          sum.y += features[i]->at(closest).xy.y;
          ++count;
        }
      }
      centre.x = sum.x / static_cast<float>(count);
      centre.y = sum.y / static_cast<float>(count);
      if (covered == previous) break;
      previous = covered;
      if (pass == 100) {
        ++counts->capped;
        break;
      }
    }
    bool accept = true, any = false;
    for (int i = 0; i < n; ++i) {
      accept = accept && covered[i] >= 0;
      any = any || covered[i] >= 0;
    }
    if (accept) {
      centres.push_back(centre);
      ++counts->intersections;
    } else if (!any) {
      ++counts->uncovered;
    } else {
      for (int i = 0; i < n; ++i)
        if (covered[i] >= 0) features[i]->erase(features[i]->begin() + covered[i]);
      if (covered[0] == -1) ++counts->reruns;
      if (covered[0] <= f) --f;
    }
  }
  for (int i = 0; i < n; ++i) {
    for (int f = 0; f < static_cast<int>(features[i]->size()); ++f) {
      bool near = false;
      for (const Vec2f& c : centres) {
        const float d = squared_norm(c.x - features[i]->at(f).xy.x, c.y - features[i]->at(f).xy.y);
        if (d <= thr2) {
          near = true;
          break;
        }
      }
      if (!near) {
        features[i]->erase(features[i]->begin() + f);
        --f;
      }
    }
  }
}

}  // namespace

// counts [5]: intersections, kept, uncovered, capped, re-runs of one f (covered[0] == -1 with erasures). keep [N] as b200ba_intersect_features returns it.
extern "C" int oracle_intersect_lists(int32_t n_datasets, int64_t n_lists, const int64_t* off, const float* xy,
                                      double threshold, uint8_t* keep, int64_t* counts) {
  const double thr2 = threshold * threshold;
  Counts c;
  const int64_t total = off[n_lists * n_datasets];
  for (int64_t k = 0; k < total; ++k) keep[k] = 0;
  for (int64_t l = 0; l < n_lists; ++l) {
    std::vector<std::vector<PointFeature>> lists(n_datasets);
    std::vector<std::vector<PointFeature>*> features(n_datasets);
    for (int i = 0; i < n_datasets; ++i) {
      for (int64_t k = off[l * n_datasets + i]; k < off[l * n_datasets + i + 1]; ++k) {
        PointFeature p;
        p.xy = Vec2f{xy[2 * k], xy[2 * k + 1]};
        p.id = static_cast<int>(k - off[l * n_datasets]);
        lists[i].push_back(p);
      }
      features[i] = &lists[i];
    }
    intersect_camera(features, thr2, &c);
    for (int i = 0; i < n_datasets; ++i)
      for (const PointFeature& p : lists[i]) keep[off[l * n_datasets] + p.id] = 1;
  }
  int64_t kept = 0;
  for (int64_t k = 0; k < total; ++k) kept += keep[k];
  counts[0] = c.intersections;
  counts[1] = kept;
  counts[2] = c.uncovered;
  counts[3] = c.capped;
  counts[4] = c.reruns;
  return 0;
}

// Returns the tool's exit code. counts [3]: intersections, uncovered, capped.
extern "C" int oracle_intersect_datasets(int32_t n, const char* const* paths, double threshold, const char* suffix,
                                         int64_t* counts) {
  if (n < 1) return 1;
  const double thr2 = threshold * threshold;
  std::vector<std::shared_ptr<Dataset>> datasets(n);
  for (int i = 0; i < n; ++i) {
    if (!LoadDataset(paths[i], &datasets[i])) return 1;
    if (i > 0 && datasets[i]->num_cameras() != datasets[0]->num_cameras()) return 1;
  }
  std::vector<std::unordered_map<std::string, int>> maps(n);
  for (int i = 0; i < n; ++i)
    for (int k = 0; k < datasets[i]->ImagesetCount(); ++k)
      maps[i].insert(std::make_pair(datasets[i]->GetImageset(k)->GetFilename(), k));
  Counts c;
  for (int index = 0; index < datasets[0]->ImagesetCount(); ++index) {
    std::vector<std::shared_ptr<Imageset>> sets(n);
    sets[0] = datasets[0]->GetImageset(index);
    bool in_all = true;
    for (int i = 1; i < n; ++i) {
      auto it = maps[i].find(sets[0]->GetFilename());
      if (it == maps[i].end()) {
        in_all = false;
        break;
      }
      sets[i] = datasets[i]->GetImageset(it->second);
    }
    if (!in_all) {
      const std::string name = sets[0]->GetFilename();
      for (int i = 0; i < n; ++i) {
        auto it = maps[i].find(name);
        int doomed = -1;
        if (it != maps[i].end()) {
          doomed = it->second;
        } else if (i == 0) {
          doomed = index;  // pinned: the reference would walk this imageset forever
        } else {
          continue;
        }
        datasets[i]->DeleteImageset(doomed);
        for (auto& item : maps[i])
          if (item.second > doomed) --item.second;
        maps[i].erase(name);
      }
      --index;
      continue;
    }
    for (int camera = 0; camera < datasets[0]->num_cameras(); ++camera) {
      std::vector<std::vector<PointFeature>*> features(n);
      for (int i = 0; i < n; ++i) features[i] = &sets[i]->FeaturesOfCamera(camera);
      intersect_camera(features, thr2, &c);
    }
  }
  for (int i = 1; i < n; ++i)
    for (int k = 0; k < datasets[i]->ImagesetCount(); ++k)
      if (maps[0].count(datasets[i]->GetImageset(k)->GetFilename()) == 0) {
        datasets[i]->DeleteImageset(k);
        --k;
      }
  for (int i = 0; i < n; ++i)
    if (!SaveDataset((std::string(paths[i]) + suffix).c_str(), *datasets[i])) return 1;
  counts[0] = c.intersections;
  counts[1] = c.uncovered;
  counts[2] = c.capped;
  return 0;
}
