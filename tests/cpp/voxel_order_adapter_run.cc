// Drives VoxelGridFilterB200 and FilterChainB200::SetVoxelOrder (adapter/registrators_b200.h) with the stand-in
// headers of tests/stubs.  Reads <in>: int32 order, float voxel_size, uint32 seed, int64 n, float records[n * 5].
// Writes <out>: int64 m, m 5-float records of VoxelGridFilterB200(cloud, voxel_size, &out, 0, order); then the chain
// [VoxelGrid(voxel_size, order), RandomSampler(0.5, MT19937 at seed)]: int64 m, m records, m int32 inlier indices.
// tests/test_gpu_voxel_order.py builds and runs it.
#include <cstdint>
#include <fstream>
#include <string>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int32_t order = 0;
  float voxel_size = 0.f;
  uint32_t seed = 0;
  int64_t n = 0;
  in.read(reinterpret_cast<char*>(&order), sizeof(order));
  in.read(reinterpret_cast<char*>(&voxel_size), sizeof(voxel_size));
  in.read(reinterpret_cast<char*>(&seed), sizeof(seed));
  in.read(reinterpret_cast<char*>(&n), sizeof(n));
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  std::ofstream out(argv[2], std::ios::binary);
  data::InnerCloudType voxels;
  registrator::VoxelGridFilterB200(cloud, voxel_size, &voxels, 0, order);
  int64_t m = static_cast<int64_t>(voxels.points.size());
  out.write(reinterpret_cast<const char*>(&m), sizeof(m));
  out.write(reinterpret_cast<const char*>(voxels.points.data()), m * sizeof(data::InnerPointType));

  registrator::FilterChainB200 chain;
  chain.SetAllFilters(true);
  const int voxel = chain.Add("VoxelGrid");
  chain.SetParam(voxel, "voxel_size", 1, std::to_string(voxel_size));
  chain.SetVoxelOrder(voxel, order);
  const int sampler = chain.Add("RandomSampler");
  chain.SetParam(sampler, "sampling_rate", 1, "0.5");
  chain.SetRandomSampler(sampler, SM_FILTER_SAMPLER_MT19937, seed);
  data::InnerCloudType kept;
  std::vector<int> inliers;
  chain.Filter(cloud, &kept, &inliers);
  m = static_cast<int64_t>(kept.points.size());
  out.write(reinterpret_cast<const char*>(&m), sizeof(m));
  out.write(reinterpret_cast<const char*>(kept.points.data()), m * sizeof(data::InnerPointType));
  std::vector<int32_t> index(inliers.begin(), inliers.end());
  out.write(reinterpret_cast<const char*>(index.data()), index.size() * sizeof(int32_t));
  return out ? 0 : 4;
}
