// Drives the filter chain with the option all_filters through adapter/registrators_b200.h (FilterChainB200) with the
// stand-in headers of tests/stubs.  Reads <config>, one line per step: "filter <name>" or "param <name> <type> <text>"
// (a param of the last filter), and <in>: int64 n, float records[n * 5]; writes <out>:
// int64 m, then m 5-float records and their m int32 inlier indices.  tests/test_gpu_filter_chain_all_adapter.py builds
// and runs it.
#include <cstdint>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "registrators_b200.h"

using namespace static_map;

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  registrator::FilterChainB200 chain;
  chain.SetAllFilters(true);
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
    }
  }
  std::ifstream in(argv[2], std::ios::binary);
  int64_t n = 0;
  in.read(reinterpret_cast<char*>(&n), 8);
  data::InnerCloudType cloud;
  cloud.points.resize(n);
  in.read(reinterpret_cast<char*>(cloud.points.data()), n * sizeof(data::InnerPointType));
  if (!in) return 3;

  data::InnerCloudType kept;
  std::vector<int> inliers;
  chain.Filter(cloud, &kept, &inliers);

  std::ofstream out(argv[3], std::ios::binary);
  const int64_t m = static_cast<int64_t>(kept.points.size());
  out.write(reinterpret_cast<const char*>(&m), sizeof(m));
  out.write(reinterpret_cast<const char*>(kept.points.data()), m * sizeof(data::InnerPointType));
  std::vector<int32_t> index(inliers.begin(), inliers.end());
  out.write(reinterpret_cast<const char*>(index.data()), index.size() * sizeof(int32_t));
  return 0;
}
