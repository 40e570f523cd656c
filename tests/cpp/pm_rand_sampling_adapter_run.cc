// Drives IcpUsingPointMatcherB200 (adapter/registrators_b200.h) with SetReadingSampler, GetRandPosition and
// SetRandPosition through the stand-in headers of tests/stubs.  Reads <in>: int64 ns, int64 nt, float src[ns*3],
// float tgt[nt*3]; prints one "key ok score v0 .. v15" line (the column-major result) per alignment, the stream
// position around them, and the return codes of a bad mode and a bad position.
// tests/test_gpu_pm_rand_sampling.py builds it and compares every line with the oracle.
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

  registrator::IcpUsingPointMatcherB200 matcher;
  matcher.SetInputSource(make_cloud(src, n[0]));
  matcher.SetInputTarget(make_cloud(tgt, n[1]));
  matcher.SetReadingSampler(SM_PM_SAMPLING_GLIBC_RAND);
  std::vector<long long> positions = {static_cast<long long>(matcher.GetRandPosition())};
  Eigen::Matrix4d result;
  bool ok = matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("first", ok, matcher.GetFitnessScore(), result);
  positions.push_back(matcher.GetRandPosition());
  ok = matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("second", ok, matcher.GetFitnessScore(), result);
  positions.push_back(matcher.GetRandPosition());
  matcher.SetRandPosition(7);
  positions.push_back(matcher.GetRandPosition());
  ok = matcher.Align(Eigen::Matrix4d::Identity(), result);
  Print("at_7", ok, matcher.GetFitnessScore(), result);
  positions.push_back(matcher.GetRandPosition());
  std::printf("positions");
  for (long long p : positions) std::printf(" %lld", p);
  std::printf("\n");
  // the setters CHECK-fail on a bad value; the C ABI underneath reports it
  std::printf("bad_mode_rc %d\n", sm_set_pm_reading_sampler(matcher.handle(), 5));
  std::printf("bad_position_rc %d\n", sm_set_pm_rand_position(matcher.handle(), -1));
  return 0;
}
