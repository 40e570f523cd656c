// Driver of MultiviewRegistratorLumPclB200 (adapter/registrators_b200.h) for tests/test_gpu_lum_adapter.py, built
// with the stand-ins of tests/stubs_multiview and tests/stubs.  Input: int64 frames, int64 calls, then per frame
// int64 n, 16 floats of the column-major pose and n records of 5 floats.  AlignAll runs `calls` times; the output is,
// per call, int64 m and m records.  TEST INFRASTRUCTURE.
#include <cstdint>
#include <cstdio>
#include <memory>
#include <vector>

#include "registrators_b200.h"

struct Point5 { float x, y, z, intensity, factor; };

int main(int argc, char** argv) {
  using Lum = static_map::registrator::MultiviewRegistratorLumPclB200<Point5>;
  if (argc != 3) return 2;
  FILE* in = fopen(argv[1], "rb");
  FILE* out = fopen(argv[2], "wb");
  if (!in || !out) return 2;
  int64_t frames = 0, calls = 0;
  if (fread(&frames, 8, 1, in) != 1 || fread(&calls, 8, 1, in) != 1) return 2;
  Lum lum;
  for (int64_t f = 0; f < frames; ++f) {
    int64_t n = 0;
    Eigen::Matrix4f pose;
    auto cloud = std::make_shared<pcl::PointCloud<Point5>>();
    if (fread(&n, 8, 1, in) != 1 || fread(pose.m, 4, 16, in) != 16) return 2;
    cloud->points.resize(n);
    if (n && fread(cloud->points.data(), sizeof(Point5), n, in) != static_cast<size_t>(n)) return 2;
    lum.AddNewCloud(cloud, pose);
  }
  for (int64_t c = 0; c < calls; ++c) {
    auto output = std::make_shared<pcl::PointCloud<Point5>>();
    lum.AlignAll(output);
    const int64_t m = static_cast<int64_t>(output->size());
    fwrite(&m, 8, 1, out);
    fwrite(output->points.data(), sizeof(Point5), m, out);
  }
  fclose(out);
  return lum.Size() == static_cast<size_t>(frames) ? 0 : 3;
}
