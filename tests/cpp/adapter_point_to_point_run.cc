// Drives IcpFastB200 (adapter/registrators_b200.h) with SetErrorMinimizer through the stand-in headers of tests/stubs,
// with tests/stubs_inner_compensation's Interface in front of them.  Reads <in>: int64 ns, int64 nt, double
// src[ns*3], tgt[nt*3], normals[nt*3]; prints one "key v0 .. v15" line (the column-major result) per alignment and
// the return code of a bad minimizer value.  tests/test_gpu_icp_point_to_point.py builds it and compares every line
// with the oracles.
#include <cstdio>
#include <fstream>
#include <memory>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

static void Print(const char* key, const Eigen::Matrix4d& m) {
  std::printf("%s", key);
  for (int i = 0; i < 16; ++i) std::printf(" %.17g", m.data()[i]);
  std::printf("\n");
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int64_t n[2] = {0, 0};
  in.read(reinterpret_cast<char*>(n), 16);
  std::vector<double> src(3 * n[0]), tgt(3 * n[1]), nrm(3 * n[1]);
  in.read(reinterpret_cast<char*>(src.data()), src.size() * 8);
  in.read(reinterpret_cast<char*>(tgt.data()), tgt.size() * 8);
  in.read(reinterpret_cast<char*>(nrm.data()), nrm.size() * 8);
  if (!in) return 3;
  auto source = std::make_shared<data::InnerPointCloudData>();
  auto target = std::make_shared<data::InnerPointCloudData>();
  source->GetEigenCloud()->points = Eigen::MatrixXd(3, n[0]);
  target->GetEigenCloud()->points = Eigen::MatrixXd(3, n[1]);
  target->GetEigenCloud()->normals = Eigen::MatrixXd(3, n[1]);
  for (int64_t i = 0; i < n[0]; ++i)
    for (int d = 0; d < 3; ++d) source->GetEigenCloud()->points(d, i) = src[3 * i + d];
  for (int64_t i = 0; i < n[1]; ++i)
    for (int d = 0; d < 3; ++d) {
      target->GetEigenCloud()->points(d, i) = tgt[3 * i + d];
      target->GetEigenCloud()->normals(d, i) = nrm[3 * i + d];
    }

  registrator::IcpFastB200 matcher;
  matcher.InitWithOptions();
  matcher.SetInputSource(source);
  matcher.SetInputTarget(target);
  Eigen::Matrix4d result;
  matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("plane", result);
  matcher.SetErrorMinimizer(SM_ICP_POINT_TO_POINT);
  matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("p2p", result);
  matcher.SetErrorMinimizer(SM_ICP_POINT_TO_PLANE);
  matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("plane_again", result);

  // AlignBatch keeps each matcher's minimizer
  matcher.SetErrorMinimizer(SM_ICP_POINT_TO_POINT);
  std::vector<registrator::IcpFastB200*> ms = {&matcher};
  std::vector<Eigen::Matrix4d> guesses = {Eigen::Matrix4d::Identity()}, results;
  std::vector<bool> ok;
  registrator::AlignBatch(ms, guesses, &results, &ok);
  Print("batch_p2p", results[0]);
  // the setter CHECK-fails on a bad value; the C ABI underneath reports it
  std::printf("bad_value_rc %d\n", sm_set_icp_error_minimizer(matcher.handle(), 2));
  return 0;
}
