// Drives GroundRemoval through adapter/registrators_b200.h (GroundRemovalB200) with the stand-in headers of
// tests/stubs.  Reads <in>: int64 n, int32 min_point_num_in_voxel, float leaf_size, float height_threshold, float
// records[n * 5]; writes <out>: int64 m, int64 n_inliers, int64 n_outliers, then m 5-float records, the inliers and the
// outliers as int32.  tests/test_gpu_ground_removal_adapter.py builds and runs it.
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int64_t n = 0;
  int32_t min_points = 0;
  float leaf = 0.f, threshold = 0.f;
  in.read(reinterpret_cast<char*>(&n), 8);
  in.read(reinterpret_cast<char*>(&min_points), 4);
  in.read(reinterpret_cast<char*>(&leaf), 4);
  in.read(reinterpret_cast<char*>(&threshold), 4);
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  registrator::GroundRemovalB200 filter;
  filter.SetParam("min_point_num_in_voxel", 0, std::to_string(min_points));
  char text[64];
  snprintf(text, sizeof(text), "%.9g", leaf);
  filter.SetParam("leaf_size", 1, text);
  snprintf(text, sizeof(text), "%.9g", threshold);
  filter.SetParam("height_threshold", 1, text);
  data::InnerCloudType kept;
  std::vector<int> inliers, outliers;
  filter.Filter(cloud, &kept, &inliers, &outliers);

  std::ofstream out(argv[2], std::ios::binary);
  const int64_t counts[3] = {static_cast<int64_t>(kept.points.size()), static_cast<int64_t>(inliers.size()),
                             static_cast<int64_t>(outliers.size())};
  out.write(reinterpret_cast<const char*>(counts), sizeof(counts));
  out.write(reinterpret_cast<const char*>(kept.points.data()), counts[0] * sizeof(data::InnerPointType));
  for (const std::vector<int>* list : {&inliers, &outliers}) {
    std::vector<int32_t> index(list->begin(), list->end());
    out.write(reinterpret_cast<const char*>(index.data()), index.size() * sizeof(int32_t));
  }
  return 0;
}
