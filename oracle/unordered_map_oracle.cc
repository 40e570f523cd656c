// ORACLE — TEST INFRASTRUCTURE ONLY (see sm_oracle.h).
//
// std::unordered_map<Eigen::Vector3i, ...> as pre_processers::filter::VoxelGrid::Filter fills it
// (pre_processors/filter_voxel_grid.cc:43-50), from this toolchain's libstdc++ itself: the voxel key
// (int(lround(x / s)), int(lround(y / s)), int(lround(z / s))) hashed by common/eigen_hash.h:31-43
// (boost's hash_combine over std::hash<int>), inserted by operator[] in input order.  Exports the
// literal iteration order (as the input index of each voxel's first member), bucket_count() after
// every distinct insert, and the hash itself, so the GPU's formulation of that order can be checked
// against the container rather than against a restatement of it.
#include <cmath>
#include <cstdint>
#include <unordered_map>

namespace {

struct Key3 {
  int v[3];
  bool operator==(const Key3& o) const { return v[0] == o.v[0] && v[1] == o.v[1] && v[2] == o.v[2]; }
};
struct Key3Hash {   // common/eigen_hash.h:34-42 with Scalar = int
  size_t operator()(const Key3& k) const {
    size_t seed = 0;
    for (int i = 0; i < 3; ++i) seed ^= std::hash<int>()(k.v[i]) + 0x9e3779b9 + (seed << 6) + (seed >> 2);
    return seed;
  }
};
struct First {   // the voxel's first member; operator[] value-initialises a new voxel
  int64_t index = -1;
};
using Grid = std::unordered_map<Key3, First, Key3Hash>;

// first-member indices in iteration order -> out; returns the number of voxels
int64_t emit(const Grid& grid, int64_t* out) {
  int64_t m = 0;
  for (const auto& g : grid) out[m++] = g.second.index;
  return m;
}

}  // namespace

extern "C" {

// points: n records of stride_floats floats, x, y, z first.  out: capacity n.  Every point is inserted,
// as in the reference (the caller passes finite points: lround of a NaN / inf quotient is unspecified).
int64_t sm_oracle_voxel_unordered_order(const float* points, int64_t n, int64_t stride_floats, float voxel_size,
                                        int64_t* out) {
  if (!(voxel_size > 1.e-6f)) return -1;
  Grid grid;
  for (int64_t i = 0; i < n; ++i) {
    const float* p = points + stride_floats * i;
    const Key3 k{{(int)std::lround(p[0] / voxel_size), (int)std::lround(p[1] / voxel_size),
                  (int)std::lround(p[2] / voxel_size)}};
    First& f = grid[k];
    if (f.index < 0) f.index = i;
  }
  return emit(grid, out);
}

// the same over given integer keys (keys_3n: n rows of x, y, z) -> the first index of every distinct key
int64_t sm_oracle_unordered_order_keys(const int32_t* keys_3n, int64_t n, int64_t* out) {
  Grid grid;
  for (int64_t i = 0; i < n; ++i) {
    First& f = grid[Key3{{keys_3n[3 * i], keys_3n[3 * i + 1], keys_3n[3 * i + 2]}}];
    if (f.index < 0) f.index = i;
  }
  return emit(grid, out);
}

// bucket_count() of a default-constructed map after each of m distinct inserts -> out[0 .. m - 1]
int sm_oracle_unordered_bucket_counts(int64_t m, uint64_t* out) {
  Grid grid;
  for (int64_t k = 0; k < m; ++k) {
    grid[Key3{{(int)k, (int)(k >> 31), 0}}];
    out[k] = grid.bucket_count();
  }
  return 0;
}

// Key3Hash of n keys -> out
int sm_oracle_key3_hash(const int32_t* keys_3n, int64_t n, uint64_t* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = Key3Hash()(Key3{{keys_3n[3 * i], keys_3n[3 * i + 1], keys_3n[3 * i + 2]}});
  return 0;
}

}  // extern "C"
