// Drives RandomSamplerWithPlaneDetect through adapter/registrators_b200.h (RandomSamplerWithPlaneDetectB200) with the
// stand-in headers of tests/stubs.  Reads <in>: int64 n, float sampling_rate, float leaf_size, uint64
// min_point_num_in_voxel, float records[n * 5]; writes <out>: int64 m, int64 n_inliers, int64 n_outliers, int64
// n_plane, then m 5-float records, the inliers, the outliers and the plane indices as int32.
// tests/test_gpu_plane_sampler_adapter.py builds and runs it.
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
  float rate = 0.f, leaf = 0.f;
  uint64_t min_points = 0;
  in.read(reinterpret_cast<char*>(&n), 8);
  in.read(reinterpret_cast<char*>(&rate), 4);
  in.read(reinterpret_cast<char*>(&leaf), 4);
  in.read(reinterpret_cast<char*>(&min_points), 8);
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  registrator::RandomSamplerWithPlaneDetectB200 sampler;
  sampler.SetSamplingRate(rate);
  sampler.SetLeafSize(leaf);
  sampler.SetMinPointNumInVoxel(min_points);
  data::InnerCloudType kept;
  sampler.Filter(cloud, &kept);
  const std::vector<int> lists[3] = {sampler.Inliers(), sampler.Outliers(), sampler.PlaneIndices()};

  std::ofstream out(argv[2], std::ios::binary);
  const int64_t counts[4] = {static_cast<int64_t>(kept.points.size()), static_cast<int64_t>(lists[0].size()),
                             static_cast<int64_t>(lists[1].size()), static_cast<int64_t>(lists[2].size())};
  out.write(reinterpret_cast<const char*>(counts), sizeof(counts));
  out.write(reinterpret_cast<const char*>(kept.points.data()), counts[0] * sizeof(data::InnerPointType));
  for (const std::vector<int>& list : lists) {
    std::vector<int32_t> index(list.begin(), list.end());
    out.write(reinterpret_cast<const char*>(index.data()), index.size() * sizeof(int32_t));
  }
  return 0;
}
