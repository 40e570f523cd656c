// Drives IcpUsingPointMatcherB200 (adapter/registrators_b200.h) with SetSurfaceNormals through the stand-in headers of
// tests/stubs.  Reads <in>: int64 ns, int64 nt, float src[ns*3], float tgt[nt*3]; prints one "key ok score v0 .. v15"
// line (the column-major result) per alignment, and the return code of a bad mode value.
// tests/test_gpu_pm_surface_normals.py builds it and compares every line with the oracle.
#include <cstdio>
#include <fstream>
#include <memory>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

static void Print(const char* key, bool ok, double score, const Eigen::Matrix4d& m) {
  std::printf("%s %d %.17g", key, ok ? 1 : 0, score);
  for (int i = 0; i < 16; ++i) std::printf(" %.17g", m.data()[i]);
  std::printf("\n");
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  std::ifstream in(argv[1], std::ios::binary);
  int64_t n[2] = {0, 0};
  in.read(reinterpret_cast<char*>(n), 16);
  std::vector<float> src(3 * n[0]), tgt(3 * n[1]);
  in.read(reinterpret_cast<char*>(src.data()), src.size() * 4);
  in.read(reinterpret_cast<char*>(tgt.data()), tgt.size() * 4);
  if (!in) return 3;
  auto make_cloud = [](const std::vector<float>& xyz, int64_t count) {
    auto c = std::make_shared<data::InnerPointCloudData>();
    c->GetInnerCloud()->points.resize(count);
    for (int64_t i = 0; i < count; ++i) {
      auto& p = c->GetInnerCloud()->points[i];
      p.x = xyz[3 * i]; p.y = xyz[3 * i + 1]; p.z = xyz[3 * i + 2];
    }
    return c;
  };
  auto source = make_cloud(src, n[0]), target = make_cloud(tgt, n[1]);

  registrator::IcpUsingPointMatcherB200 matcher;
  matcher.SetInputSource(source);
  matcher.SetInputTarget(target);
  Eigen::Matrix4d result;
  bool ok = matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("least_squares", ok, matcher.GetFitnessScore(), result);
  matcher.SetSurfaceNormals(SM_PM_NORMALS_EIGENVECTOR);
  ok = matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("eigenvector", ok, matcher.GetFitnessScore(), result);

  // AlignBatch keeps each matcher's mode
  registrator::IcpUsingPointMatcherB200 plane;
  plane.SetInputSource(source);
  plane.SetInputTarget(target);
  std::vector<registrator::IcpUsingPointMatcherB200*> ms = {&matcher, &plane};
  std::vector<Eigen::Matrix4d> guesses = {Eigen::Matrix4d::Identity(), Eigen::Matrix4d::Identity()}, results;
  std::vector<bool> oks;
  registrator::AlignBatch(ms, guesses, &results, &oks);
  Print("batch_eigenvector", oks[0], matcher.GetFitnessScore(), results[0]);
  Print("batch_least_squares", oks[1], plane.GetFitnessScore(), results[1]);
  // the setter CHECK-fails on a bad value; the C ABI underneath reports it
  std::printf("bad_value_rc %d\n", sm_set_pm_surface_normals(matcher.handle(), 2));
  return 0;
}
