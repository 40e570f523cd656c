// Drives CalculateNormalsB200 (adapter/registrators_b200.h) with the stand-in headers of tests/stubs.  Reads <in>:
// int32 order, int64 n, double points[3 * n] (3xN column-major); runs CalculateNormalsB200(cloud, 0, order) on an
// EigenPointCloud and writes <out>: int64 m, double points[3 * m], double normals[3 * m].
// tests/test_gpu_normals_nth_element.py builds and runs it.
#include <cstdint>
#include <fstream>

#include "registrators_b200.h"

using namespace static_map;

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int32_t order = 0;
  int64_t n = 0;
  in.read(reinterpret_cast<char*>(&order), sizeof(order));
  in.read(reinterpret_cast<char*>(&n), sizeof(n));
  data::EigenPointCloud cloud;
  cloud.points = Eigen::MatrixXd(3, n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), 3 * n * sizeof(double));
  if (!in) return 3;
  registrator::CalculateNormalsB200(&cloud, 0, order);
  const int64_t m = cloud.points.cols();
  std::ofstream out(argv[2], std::ios::binary);
  out.write(reinterpret_cast<const char*>(&m), sizeof(m));
  out.write(reinterpret_cast<const char*>(cloud.points.data()), 3 * m * sizeof(double));
  out.write(reinterpret_cast<const char*>(cloud.normals.data()), 3 * m * sizeof(double));
  return out ? 0 : 4;
}
