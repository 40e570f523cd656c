// CPU oracle of GroundRemoval (include/sm_b200.h): the reference's GroundRemoval::SetInputCloud and ::Filter
// (pre_processors/filter_ground_removal.cc:50-111) restated literally: a std::map keyed by the voxel index with the
// header's lexicographic comparison (.h:56-62), the same loops, initialisers and comparisons.  The one change is the
// float -> int conversion, undefined in C++ outside int's range: ToInt gives INT_MIN there, as the reference's x86
// build does.  Built into libsm_oracle.so by oracle/Makefile; tests/oracle_ground_removal.py binds it.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <map>
#include <tuple>
#include <vector>

namespace {

inline int ToInt(double q) { return (q > -2147483649.0 && q < 2147483648.0) ? static_cast<int>(q) : INT_MIN; }

struct Index {
  int v[3];
};

struct VectorCompare {
  bool operator()(const Index& a, const Index& b) const {
    return std::forward_as_tuple(a.v[0], a.v[1], a.v[2]) < std::forward_as_tuple(b.v[0], b.v[1], b.v[2]);
  }
};

}  // namespace

extern "C" {

// points: n records of stride_bytes, float x, y, z, intensity, factor first.  out (capacity n 5-float records) and
// index (capacity n): the emitted records and their input indices in emission order, *m their number; inliers /
// outliers (capacity n each): ascending, *n_inliers / *n_outliers.  Returns 0, or -1 for bad arguments.
int sm_oracle_ground_removal(const float* points, int64_t n, int64_t stride_bytes, int32_t min_point_num_in_voxel,
                             float leaf_size, float height_threshold, float* out, int64_t* m, int32_t* index,
                             int32_t* inliers, int64_t* n_inliers, int32_t* outliers, int64_t* n_outliers) {
  if (n < 0 || stride_bytes < 20 || stride_bytes % 4 || !m || !n_inliers || !n_outliers ||
      (n > 0 && (!points || !out || !index || !inliers || !outliers)))
    return -1;
  *m = *n_inliers = *n_outliers = 0;
  if (n == 0) return 0;                                 // SetInputCloud: "cloud empty, do nothing!"
  const int64_t step = stride_bytes / 4;
  auto point = [&](int64_t i) { return points + i * step; };

  std::map<Index, std::vector<int>, VectorCompare> voxels;
  for (int i = 0; i < n; ++i) {
    const float* p = point(i);
    const Index key = {{ToInt(p[0] / leaf_size), ToInt(p[1] / leaf_size), ToInt(p[2] / leaf_size)}};
    voxels[key].push_back(i);
  }

  std::vector<int> in, outl;
  int64_t emitted = 0;
  for (auto& index_vector : voxels) {
    auto& idx = index_vector.first;
    auto& vector = index_vector.second;
    if ((int32_t)vector.size() < min_point_num_in_voxel) continue;
    bool is_ground = false;
    if (idx.v[2] <= 0) {
      float max_z_in_voxel = -1.e9;
      float min_z_in_voxel = 1.e9;
      for (auto& i : vector) {
        const float z = point(i)[2];
        if (z > max_z_in_voxel) max_z_in_voxel = z;
        if (z < min_z_in_voxel) min_z_in_voxel = z;
      }
      auto delta = max_z_in_voxel - min_z_in_voxel;
      if (delta >= 0. && delta <= height_threshold) {
        is_ground = true;
        for (auto& i : vector) outl.push_back(i);
      }
    }
    if (!is_ground) {
      for (auto& i : vector) {
        in.push_back(i);
        std::copy(point(i), point(i) + 5, out + emitted * 5);
        index[emitted++] = i;
      }
    }
  }
  std::sort(in.begin(), in.end());
  std::sort(outl.begin(), outl.end());
  std::copy(in.begin(), in.end(), inliers);
  std::copy(outl.begin(), outl.end(), outliers);
  *m = emitted;
  *n_inliers = (int64_t)in.size();
  *n_outliers = (int64_t)outl.size();
  return 0;
}

}  // extern "C"
