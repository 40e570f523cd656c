// Drives StatisticRemoval through adapter/registrators_b200.h (StatisticRemovalB200) with the stand-in headers of
// tests/stubs.  Reads <in>: int64 n, int32 point_num_meank, float std_mul, float records[n * 5]; writes <out>: int64 m,
// then m 5-float records, then m int32 inlier indices.  tests/test_gpu_statistic_removal_adapter.py builds and runs it.
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
  int32_t mean_k = 0;
  float std_mul = 0.f;
  in.read(reinterpret_cast<char*>(&n), 8);
  in.read(reinterpret_cast<char*>(&mean_k), 4);
  in.read(reinterpret_cast<char*>(&std_mul), 4);
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  registrator::StatisticRemovalB200 filter;
  filter.SetParam("point_num_meank", 0, std::to_string(mean_k));
  char text[64];
  snprintf(text, sizeof(text), "%.9g", std_mul);
  filter.SetParam("std_mul", 1, text);
  data::InnerCloudType kept;
  std::vector<int> inliers;
  filter.Filter(cloud, &kept, &inliers);

  std::ofstream out(argv[2], std::ios::binary);
  const int64_t m = static_cast<int64_t>(kept.points.size());
  out.write(reinterpret_cast<const char*>(&m), 8);
  out.write(reinterpret_cast<const char*>(kept.points.data()), m * sizeof(data::InnerPointType));
  std::vector<int32_t> index(inliers.begin(), inliers.end());
  out.write(reinterpret_cast<const char*>(index.data()), m * sizeof(int32_t));
  return 0;
}
