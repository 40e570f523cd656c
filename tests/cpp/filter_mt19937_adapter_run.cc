// Drives the filter chain through adapter/registrators_b200.h (FilterChainB200) with the stand-in headers of
// tests/stubs, its RandomSamplers set by SetRandomSampler.  Reads <config>, one line per step: "filter <name>",
// "param <name> <type> <text>" or "sampler <mode> <seed>" (both of the last filter), and <in>: int64 n, float
// records[n * 5]; runs the chain <runs> times (default 1) and writes <out>: per run, int64 m, then m 5-float records
// and their m int32 inlier indices.  tests/test_gpu_filter_mt19937.py builds and runs it.
#include <cstdint>
#include <cstdlib>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const int runs = argc > 4 ? std::atoi(argv[4]) : 1;
  registrator::FilterChainB200 chain;
  std::ifstream config(argv[1]);
  std::string line;
  int filter = -1;
  while (std::getline(config, line)) {
    std::istringstream words(line);
    std::string step, name, text;
    int type = 0;
    words >> step;
    if (step == "filter") {
      words >> name;
      filter = chain.Add(name);
    } else if (step == "param") {
      words >> name >> type >> text;
      chain.SetParam(filter, name, type, text);
    } else if (step == "sampler") {
      int mode = 0;
      uint32_t seed = 0;
      words >> mode >> seed;
      chain.SetRandomSampler(filter, mode, seed);
    }
  }
  std::ifstream in(argv[2], std::ios::binary);
  int64_t n = 0;
  in.read(reinterpret_cast<char*>(&n), 8);
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  std::ofstream out(argv[3], std::ios::binary);
  for (int r = 0; r < runs; ++r) {
    data::InnerCloudType kept;
    std::vector<int> inliers;
    chain.Filter(cloud, &kept, &inliers);
    const int64_t m = static_cast<int64_t>(kept.points.size());
    out.write(reinterpret_cast<const char*>(&m), sizeof(m));
    out.write(reinterpret_cast<const char*>(kept.points.data()), m * sizeof(data::InnerPointType));
    std::vector<int32_t> index(inliers.begin(), inliers.end());
    out.write(reinterpret_cast<const char*>(index.data()), index.size() * sizeof(int32_t));
  }
  return 0;
}
