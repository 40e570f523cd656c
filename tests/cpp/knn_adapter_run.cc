// Drives libnabo's k-NN through adapter/registrators_b200.h (KnnB200) with the stand-in headers of tests/stubs.  Reads
// <in>: int64 n_target, int64 n_query, int32 k, uint32 flags, double epsilon, double max_radius, int32 bucket, then the
// target and the query as 3xN column-major doubles; writes <out>: the k x n_query int32 indices, then the k x n_query
// double dists2.  tests/test_gpu_knn_adapter.py builds and runs it.
#include <cstdint>
#include <fstream>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

// libnabo's IndexMatrix (Eigen::MatrixXi) reduced to what KnnB200 touches
struct IndexMatrix {
  IndexMatrix(long r, long c) : rows_(r), cols_(c), v_((size_t)(r * c), 0) {}
  int32_t* data() { return v_.data(); }
  long rows() const { return rows_; }
  long cols() const { return cols_; }
  long rows_, cols_;
  std::vector<int32_t> v_;
};

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int64_t n[2] = {0, 0};
  int32_t k = 0, bucket = 8;
  uint32_t flags = 0;
  double eps = 0.0, radius = 0.0;
  in.read(reinterpret_cast<char*>(n), 16);
  in.read(reinterpret_cast<char*>(&k), 4);
  in.read(reinterpret_cast<char*>(&flags), 4);
  in.read(reinterpret_cast<char*>(&eps), 8);
  in.read(reinterpret_cast<char*>(&radius), 8);
  in.read(reinterpret_cast<char*>(&bucket), 4);
  Eigen::MatrixXd target(3, n[0]), query(3, n[1]);
  in.read(reinterpret_cast<char*>(target.data()), 3 * n[0] * sizeof(double));
  in.read(reinterpret_cast<char*>(query.data()), 3 * n[1] * sizeof(double));
  if (!in) return 3;

  registrator::KnnB200 nns(target, static_cast<unsigned>(bucket));
  IndexMatrix indices(k, n[1]);
  Eigen::MatrixXd dists2(k, n[1]);
  nns.knn(query, indices, dists2, k, eps, flags, radius);

  std::ofstream out(argv[2], std::ios::binary);
  out.write(reinterpret_cast<const char*>(indices.data()), (std::streamsize)(k * n[1] * sizeof(int32_t)));
  out.write(reinterpret_cast<const char*>(dists2.data()), (std::streamsize)(k * n[1] * sizeof(double)));
  return 0;
}
