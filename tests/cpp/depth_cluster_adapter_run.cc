// Drives RangeImage::DepthCluster through adapter/registrators_b200.h (FilterChainB200) with the stand-in headers of
// tests/stubs.  Reads <in>: int64 n, int32 V, int32 H, float top, float btm, float records[n * 5]; writes <out>:
// int64 m, then m {float x, y, z; uint32 label} records.  tests/test_gpu_depth_cluster.py builds and runs it.
#include <cstdint>
#include <cstdio>
#include <fstream>
#include <string>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

struct LabeledPoint { float x, y, z; uint32_t label; };   // pcl::PointXYZL's members

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int64_t n = 0;
  int32_t grid[2] = {0, 0};
  float angles[2] = {0, 0};
  in.read(reinterpret_cast<char*>(&n), 8);
  in.read(reinterpret_cast<char*>(grid), 8);
  in.read(reinterpret_cast<char*>(angles), 8);
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  registrator::FilterChainB200 chain;
  const int f = chain.Add("RangeImage");
  chain.SetParam(f, "vertical_line_num", 0, std::to_string(grid[0]));
  chain.SetParam(f, "horizontal_line_num", 0, std::to_string(grid[1]));
  char text[64];
  snprintf(text, sizeof(text), "%.9g", angles[0]);
  chain.SetParam(f, "top_angle", 1, text);
  snprintf(text, sizeof(text), "%.9g", angles[1]);
  chain.SetParam(f, "btm_angle", 1, text);
  std::vector<LabeledPoint> labeled;
  chain.DepthCluster(f, cloud, &labeled);

  std::ofstream out(argv[2], std::ios::binary);
  const int64_t m = static_cast<int64_t>(labeled.size());
  out.write(reinterpret_cast<const char*>(&m), 8);
  out.write(reinterpret_cast<const char*>(labeled.data()), m * sizeof(LabeledPoint));
  return 0;
}
