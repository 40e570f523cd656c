// CPU oracle of RandomSamplerWithPlaneDetect (include/sm_b200.h): the reference's sampler
// (pre_processors/random_sample_with_plane_detect.h:75-106) and PlaneDetector (plane_detector.h:71-153) restated
// literally, with the PCL 1.8.1 pieces they call written out: SACSegmentation<PointXYZI> with SACMODEL_PLANE,
// SAC_RANSAC, threshold 0.1, setOptimizeCoefficients(true) and the defaults (50 iterations, probability 0.99,
// random_ = false).  Every Eigen reduction is written in the order Eigen 3.3 gives it with SSE2: a 4-wide dot or norm
// as (a0 b0 + a2 b2) + (a1 b1 + a3 b3), a 3-wide norm as a0 + (a1 + a2).  Changes, each also in DESIGN §4l:
//   - the float -> int conversion gives INT_MIN where C++ leaves it undefined (ToInt), as the reference's x86 build;
//   - computeRoots' atan2, cos and sin are evaluated in double on the float arguments and rounded to float;
//   - plane_indices.front() on an empty vector reads as "no further plane point";
//   - every run starts from empty voxels (PlaneDetector::voxels_ is never cleared in the reference).
// Built into libsm_oracle.so by oracle/Makefile; tests/oracle_plane_sampler.py binds it.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <random>
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

// PointXYZI's data[4]: x, y, z, 1
struct P4 {
  float v[4];
};

inline float Dot4(const float* a, const float* b) { return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3]); }
inline float SquaredNorm3(const float* a) { return a[0] * a[0] + (a[1] * a[1] + a[2] * a[2]); }

// SampleConsensusModelPlane::isSampleGood / the collinearity test of computeModelCoefficients
bool SampleGood(const P4& p0, const P4& p1, const P4& p2) {
  float dy[4];
  for (int i = 0; i < 4; ++i) dy[i] = (p1.v[i] - p0.v[i]) / (p2.v[i] - p0.v[i]);
  return (dy[0] != dy[1]) || (dy[2] != dy[1]);
}

// SampleConsensusModelPlane::computeModelCoefficients after the collinearity test
void ModelCoefficients(const P4& p0, const P4& p1, const P4& p2, float* c) {
  float a[4], b[4];
  for (int i = 0; i < 4; ++i) { a[i] = p1.v[i] - p0.v[i]; b[i] = p2.v[i] - p0.v[i]; }
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
  c[3] = 0;
  const float z = Dot4(c, c);                     // Eigen normalize(): divide only when the squared norm is > 0
  if (z > 0.f) {
    const float s = std::sqrt(z);
    for (int i = 0; i < 4; ++i) c[i] /= s;
  }
  c[3] = -1 * Dot4(c, p0.v);
}

float Distance(const float* c, const P4& p) { return std::fabs(Dot4(c, p.v)); }

void ComputeRoots2(float b, float c, float* roots) {
  roots[0] = 0.f;
  float d = static_cast<float>(b * b - 4.0 * c);
  if (d < 0.0) d = 0.0;
  const float sd = std::sqrt(d);
  roots[2] = 0.5f * (b + sd);
  roots[1] = 0.5f * (b - sd);
}

void ComputeRoots(const float m[3][3], float* roots) {
  const float c0 = m[0][0] * m[1][1] * m[2][2] + 2.f * m[0][1] * m[0][2] * m[1][2] - m[0][0] * m[1][2] * m[1][2] -
                   m[1][1] * m[0][2] * m[0][2] - m[2][2] * m[0][1] * m[0][1];
  const float c1 = m[0][0] * m[1][1] - m[0][1] * m[0][1] + m[0][0] * m[2][2] - m[0][2] * m[0][2] +
                   m[1][1] * m[2][2] - m[1][2] * m[1][2];
  const float c2 = m[0][0] + m[1][1] + m[2][2];
  if (std::fabs(c0) < FLT_EPSILON) {
    ComputeRoots2(c2, c1, roots);
    return;
  }
  const float s_inv3 = static_cast<float>(1.0 / 3.0);
  const float s_sqrt3 = std::sqrt(3.f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.f) a_over_3 = 0.f;
  const float half_b = 0.5f * (c0 + c2_over_3 * (2.f * c2_over_3 * c2_over_3 - c1));
  float q = half_b * half_b + a_over_3 * a_over_3 * a_over_3;
  if (q > 0.f) q = 0.f;
  const float rho = std::sqrt(-a_over_3);
  const float theta = static_cast<float>(std::atan2(static_cast<double>(std::sqrt(-q)), static_cast<double>(half_b))) *
                      s_inv3;
  const float cos_theta = static_cast<float>(std::cos(static_cast<double>(theta)));
  const float sin_theta = static_cast<float>(std::sin(static_cast<double>(theta)));
  roots[0] = c2_over_3 + 2.f * rho * cos_theta;
  roots[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  roots[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
  if (roots[1] >= roots[2]) {
    std::swap(roots[1], roots[2]);
    if (roots[0] >= roots[1]) std::swap(roots[0], roots[1]);
  }
  if (roots[0] <= 0) ComputeRoots2(c2, c1, roots);
}

inline void Cross(const float* a, const float* b, float* r) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}

// pcl::eigen33(mat, eigenvalue, eigenvector): the eigenvector of the smallest eigenvalue
void Eigen33(const float mat[3][3], float* vec) {
  float scale = 0.f;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) scale = std::max(scale, std::fabs(mat[r][c]));
  if (scale <= FLT_MIN) scale = 1.f;
  float s[3][3];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) s[r][c] = mat[r][c] / scale;
  float roots[3];
  ComputeRoots(s, roots);
  for (int d = 0; d < 3; ++d) s[d][d] -= roots[0];
  float v[3][3];
  Cross(s[0], s[1], v[0]);
  Cross(s[0], s[2], v[1]);
  Cross(s[1], s[2], v[2]);
  const float len1 = SquaredNorm3(v[0]), len2 = SquaredNorm3(v[1]), len3 = SquaredNorm3(v[2]);
  int pick = 2;
  float len = len3;
  if (len1 >= len2 && len1 >= len3) { pick = 0; len = len1; }
  else if (len2 >= len1 && len2 >= len3) { pick = 1; len = len2; }
  const float root = std::sqrt(len);
  for (int d = 0; d < 3; ++d) vec[d] = v[pick][d] / root;
}

struct VoxelTrace {
  int32_t status, iterations, best, final_count;
  float coef[4];
};

// status of a voxel in the trace
enum { kSkipped = 0, kGroundPlane = 1, kGroundNot = 2, kSkippedRansac = 3, kRansacPlane = 4, kRansacNot = 5 };

const std::vector<uint32_t>& RawStream() {
  static const std::vector<uint32_t> words = [] {
    std::mt19937 engine(12345u);
    std::vector<uint32_t> w(3 * 1000 * 51);
    for (auto& x : w) x = engine();
    return w;
  }();
  return words;
}

// SACSegmentation::segment on one voxel's cloud: the refined inliers (positions in `cloud`) and the trace
std::vector<int> Segment(const std::vector<P4>& cloud, VoxelTrace* t) {
  const double threshold = 0.1;
  const int n = static_cast<int>(cloud.size());
  // SampleConsensusModel: rng_alg_.seed(12345u), rnd() = uniform_int<int>(0, INT_MAX) over it = engine() >> 1
  std::mt19937 engine(12345u);
  auto rnd = [&]() { return static_cast<int>(engine() >> 1); };
  std::vector<int> shuffled(n);
  for (int i = 0; i < n; ++i) shuffled[i] = i;
  auto count_within = [&](const float* c) {
    int nr = 0;
    for (int i = 0; i < n; ++i)
      if (Distance(c, cloud[i]) < threshold) nr++;
    return nr;
  };
  auto select_within = [&](const float* c) {
    std::vector<int> in;
    for (int i = 0; i < n; ++i)
      if (Distance(c, cloud[i]) < threshold) in.push_back(i);
    return in;
  };

  // RandomSampleConsensus::computeModel
  int iterations = 0;
  int n_best_inliers_count = -INT_MAX;
  double k = 1.0;
  std::vector<int> model;
  float model_coefficients[4] = {0, 0, 0, 0};
  const double log_probability = std::log(1.0 - 0.99);
  const double one_over_indices = 1.0 / static_cast<double>(n);
  unsigned skipped_count = 0;
  const unsigned max_skip = 50 * 10;
  while (iterations < k && skipped_count < max_skip) {
    // getSamples: up to max_sample_checks_ = 1000 draws
    std::vector<int> selection(3);
    bool good = false;
    for (unsigned iter = 0; iter < 1000; ++iter) {
      for (unsigned i = 0; i < 3; ++i)
        std::swap(shuffled[i], shuffled[i + (rnd() % (static_cast<size_t>(n) - i))]);
      std::copy(shuffled.begin(), shuffled.begin() + 3, selection.begin());
      if (SampleGood(cloud[selection[0]], cloud[selection[1]], cloud[selection[2]])) { good = true; break; }
    }
    if (!good) break;                               // selection.empty()
    if (!SampleGood(cloud[selection[0]], cloud[selection[1]], cloud[selection[2]])) { ++skipped_count; continue; }
    float c[4];
    ModelCoefficients(cloud[selection[0]], cloud[selection[1]], cloud[selection[2]], c);
    const int n_inliers_count = count_within(c);
    if (n_inliers_count > n_best_inliers_count) {
      n_best_inliers_count = n_inliers_count;
      model = selection;
      std::memcpy(model_coefficients, c, sizeof(c));
      const double w = static_cast<double>(n_best_inliers_count) * one_over_indices;
      double p_no_outliers = 1.0 - std::pow(w, static_cast<double>(selection.size()));
      p_no_outliers = std::max(std::numeric_limits<double>::epsilon(), p_no_outliers);
      p_no_outliers = std::min(1.0 - std::numeric_limits<double>::epsilon(), p_no_outliers);
      k = log_probability / std::log(p_no_outliers);
    }
    ++iterations;
    if (iterations > 50) break;
  }
  t->iterations = iterations;
  t->best = n_best_inliers_count;
  if (model.empty()) return {};                     // computeModel fails: segment clears the inliers

  std::vector<int> inliers = select_within(model_coefficients);
  // optimizeModelCoefficients
  float refined[4];
  std::memcpy(refined, model_coefficients, sizeof(refined));
  if (inliers.size() >= 4) {
    float accu[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};    // computeMeanAndCovarianceMatrix, the is_dense branch
    for (int i : inliers) {
      const float x = cloud[i].v[0], y = cloud[i].v[1], z = cloud[i].v[2];
      accu[0] += x * x; accu[1] += x * y; accu[2] += x * z;
      accu[3] += y * y; accu[4] += y * z; accu[5] += z * z;
      accu[6] += x; accu[7] += y; accu[8] += z;
    }
    for (float& a : accu) a /= static_cast<float>(inliers.size());
    const float centroid[4] = {accu[6], accu[7], accu[8], 1};
    float cov[3][3];
    cov[0][0] = accu[0] - accu[6] * accu[6];
    cov[0][1] = accu[1] - accu[6] * accu[7];
    cov[0][2] = accu[2] - accu[6] * accu[8];
    cov[1][1] = accu[3] - accu[7] * accu[7];
    cov[1][2] = accu[4] - accu[7] * accu[8];
    cov[2][2] = accu[5] - accu[8] * accu[8];
    cov[1][0] = cov[0][1];
    cov[2][0] = cov[0][2];
    cov[2][1] = cov[1][2];
    float v[3];
    Eigen33(cov, v);
    refined[0] = v[0]; refined[1] = v[1]; refined[2] = v[2]; refined[3] = 0;
    refined[3] = -1 * Dot4(refined, centroid);
  }
  std::memcpy(t->coef, refined, sizeof(refined));
  return select_within(refined);
}

// PlaneDetector::SetInputCloud on a fresh detector + Detect(plane_indices, 0.2)
std::vector<int> Detect(const float* points, int64_t n, int64_t step, float leaf_size, size_t min_point_num_in_voxel,
                        std::vector<VoxelTrace>* traces) {
  std::vector<int> ground_indices;
  const float distance_threshold = 0.2f;
  std::map<Index, std::vector<int>, VectorCompare> voxels;
  for (int i = 0; i < n; ++i) {
    const float* p = points + i * step;
    const Index key = {{ToInt(p[0] / leaf_size), ToInt(p[1] / leaf_size), ToInt(p[2] / leaf_size)}};
    voxels[key].push_back(i);
  }
  if (distance_threshold >= leaf_size) return ground_indices;   // "distance_threshold is too large."
  for (auto& index_vector : voxels) {
    const Index& index = index_vector.first;
    auto& indices = index_vector.second;
    VoxelTrace t = {kSkipped, 0, 0, 0, {0, 0, 0, 0}};
    if (indices.size() < min_point_num_in_voxel) {
      traces->push_back(t);
      continue;
    }
    if (index.v[2] <= 0) {
      float max_z_in_voxel = -1.e9;
      float min_z_in_voxel = 1.e9;
      for (auto& i : indices) {
        const float z = points[i * step + 2];
        if (z > max_z_in_voxel) max_z_in_voxel = z;
        if (z < min_z_in_voxel) min_z_in_voxel = z;
      }
      auto delta = max_z_in_voxel - min_z_in_voxel;
      t.status = kGroundNot;
      if (delta >= 0. && delta <= distance_threshold) {
        t.status = kGroundPlane;
        t.final_count = static_cast<int32_t>(indices.size());
        for (auto& i : indices) ground_indices.push_back(i);
      }
    } else {
      if (indices.size() < min_point_num_in_voxel * 2) {
        t.status = kSkippedRansac;
        traces->push_back(t);
        continue;
      }
      std::vector<P4> voxel_cloud;
      for (auto& i : indices) {
        const float* p = points + i * step;
        voxel_cloud.push_back({{p[0], p[1], p[2], 1.f}});
      }
      const std::vector<int> inliers = Segment(voxel_cloud, &t);
      t.final_count = static_cast<int32_t>(inliers.size());
      float inliers_rate = static_cast<float>(inliers.size()) / indices.size();
      t.status = kRansacNot;
      if (inliers_rate > 0.85) {
        t.status = kRansacPlane;
        for (auto index : inliers) ground_indices.push_back(indices[index]);
      }
    }
    traces->push_back(t);
  }
  return ground_indices;
}

}  // namespace

extern "C" {

// The raw stream of std::mt19937(12345): out[i] = word i, i < n <= 153000.
int sm_oracle_plane_sampler_raw_stream(uint32_t* out, int64_t n) {
  if (!out || n < 0 || n > static_cast<int64_t>(RawStream().size())) return -1;
  std::copy(RawStream().begin(), RawStream().begin() + n, out);
  return 0;
}

// The sampler's loop over k non-plane points (random_sample_with_plane_detect.h:96-104) at `rate`: keep[j] = 1 iff
// non-plane point j + 1 is kept, j < k.
int sm_oracle_plane_sampler_keep_loop(float rate, int64_t k, uint8_t* keep) {
  if (k < 0 || (k > 0 && !keep)) return -1;
  int other_sum = 0;
  int other_sapmled_sum = 0;
  for (int64_t j = 0; j < k; ++j) {
    other_sum++;
    keep[j] = 0;
    if (static_cast<float>(other_sapmled_sum) / static_cast<float>(other_sum) < rate) {
      keep[j] = 1;
      other_sapmled_sum++;
    }
  }
  return 0;
}

// One piece of a hypothesis.  op 0: isSampleGood over in = p0, p1, p2 (3 floats each): out[0] = 1 or 0.  op 1:
// computeModelCoefficients: out[0..3].  op 2: in = c[4], p[3]: out[0] = |c . (p, 1)|, out[1] = 1 iff it is < 0.1.
// op 3: pcl::eigen33 of the row-major 3x3 in: out[0..2] = the eigenvector.
int sm_oracle_plane_sampler_piece(int32_t op, const float* in, float* out) {
  if (!in || !out) return -1;
  auto p4 = [&](int k) { return P4{{in[3 * k], in[3 * k + 1], in[3 * k + 2], 1.f}}; };
  switch (op) {
    case 0: out[0] = SampleGood(p4(0), p4(1), p4(2)) ? 1.f : 0.f; return 0;
    case 1: ModelCoefficients(p4(0), p4(1), p4(2), out); return 0;
    case 2: {
      const P4 p = {{in[4], in[5], in[6], 1.f}};
      out[0] = Distance(in, p);
      out[1] = out[0] < 0.1 ? 1.f : 0.f;
      return 0;
    }
    case 3: {
      float m[3][3];
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) m[r][c] = in[3 * r + c];
      Eigen33(m, out);
      return 0;
    }
    default: return -1;
  }
}

// RandomSamplerWithPlaneDetect::SetInputCloud + Filter on a fresh sampler.  points: n records of stride_bytes, float
// x, y, z first.  rate, leaf_size and min_point_num_in_voxel as after the setters.  Writes keep (capacity n: 1 for
// the kept points), plane (capacity n: the sorted output of Detect, *n_plane) and, when traces is not null, one
// 8-word trace per voxel in map order (capacity n, *n_voxels; none when Detect does not run).  Returns 0, or -1 for
// bad arguments.
int sm_oracle_plane_sampler(const float* points, int64_t n, int64_t stride_bytes, float rate, float leaf_size,
                            uint64_t min_point_num_in_voxel, uint8_t* keep, int32_t* plane, int64_t* n_plane,
                            void* traces, int64_t* n_voxels) {
  if (n < 0 || stride_bytes < 12 || stride_bytes % 4 || !n_plane || !n_voxels ||
      (n > 0 && (!points || !keep || !plane)))
    return -1;
  *n_plane = *n_voxels = 0;
  if (n == 0) return 0;                              // SetInputCloud: "cloud is empty."; Filter returns
  if (rate > 0.999999) {
    std::fill(keep, keep + n, 1);
    return 0;
  }
  std::vector<VoxelTrace> tv;
  std::vector<int> plane_indices =
      Detect(points, n, stride_bytes / 4, leaf_size, static_cast<size_t>(min_point_num_in_voxel), &tv);
  std::sort(plane_indices.begin(), plane_indices.end());
  std::copy(plane_indices.begin(), plane_indices.end(), plane);
  *n_plane = static_cast<int64_t>(plane_indices.size());
  if (traces) std::memcpy(traces, tv.data(), tv.size() * sizeof(VoxelTrace));
  *n_voxels = static_cast<int64_t>(tv.size());

  int other_sum = 0;
  int other_sapmled_sum = 0;
  size_t next = 0;                                   // plane_indices.front() after the erased ones
  for (int i = 0; i < n; ++i) {
    keep[i] = 0;
    if (next < plane_indices.size() && i == plane_indices[next]) {
      keep[i] = 1;
      ++next;
    } else {
      other_sum++;
      if (static_cast<float>(other_sapmled_sum) / static_cast<float>(other_sum) < rate) {
        keep[i] = 1;
        other_sapmled_sum++;
      }
    }
  }
  return 0;
}

}  // extern "C"
