// ORACLE — TEST INFRASTRUCTURE ONLY (see sm_oracle.h).
//
// libpointmatcher 1.3.1 SamplingSurfaceNormalDataPointsFilter with knn 7 and samplingMethod 1, the reference filter
// of IcpUsingPointMatcher's default chain (icp_pointmatcher.cc:187-192), in PointMatcher<float>.  libpointmatcher is
// not in the reference tree; the filter is restated from its published source: the box recursion is the one the
// reference author ported as CalculateNormals (cloud_types.cc:105-144, restated in sm_oracle.cc NormalsBuilder), and
// each box of <= 7 points yields its float mean and the eigenvector of the smallest eigenvalue of its covariance.
//
// The leaf is a twin of the product's (staticmapping_b200/csrc/normals.cu leaf_eigen_normal) written from the same
// definition with this directory's linear algebra: the same operation order, no contraction (-ffp-contract=off),
// so the two agree bit for bit.  Upstream's summation order inside rowwise().sum(), its EigenSolver and its handling
// of dropped boxes cannot be checked here; the choices are the ones documented in DESIGN.md section 4e.
// Built into libsm_oracle.so by oracle/Makefile.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <limits>
#include <numeric>
#include <vector>

#include "linalg.h"
#include "sm_oracle.h"

namespace {

// The leaf.  members[count][3] in ascending original index.  Returns 1 kept, 0 dropped (mean and cov written).
int EigenLeaf(const float (*d)[3], int count, float* mean, float* cov, float* unit) {
  float s[3] = {d[0][0], d[0][1], d[0][2]};          // rowwise().sum(): from the first member, in member order
  for (int i = 1; i < count; ++i)
    for (int r = 0; r < 3; ++r) s[r] += d[i][r];
  for (int r = 0; r < 3; ++r) mean[r] = s[r] / (float)count;
  double C[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      float acc = (d[0][r] - mean[r]) * (d[0][c] - mean[c]);
      for (int i = 1; i < count; ++i) acc += (d[i][r] - mean[r]) * (d[i][c] - mean[c]);
      cov[r * 3 + c] = acc;
      C[r * 3 + c] = (double)acc;
    }
  // FullPivHouseholderQR<MatrixXf>::rank(): |R(i,i)| > |maxpivot| * (epsilon<float> * 3), on C widened to double
  sm_oracle::FullPivQR<3> qr;
  qr.Compute(C);
  const double thr = std::fabs(qr.maxpivot) * ((double)FLT_EPSILON * 3.0);
  int rank = 0;
  for (int i = 0; i < qr.nonzero_pivots; ++i) rank += (std::fabs(qr.R[i * 3 + i]) > thr) ? 1 : 0;
  if (rank + 1 < 3) return 0;
  double w[3], V[9];
  sm_oracle::JacobiEigenSym(C, 3, w, V);
  int k = 0;                                          // smallest eigenvalue, the first of equals
  for (int i = 1; i < 3; ++i)
    if (w[i] < w[k]) k = i;
  const double v[3] = {V[0 * 3 + k], V[1 * 3 + k], V[2 * 3 + k]};
  const double len = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  for (int r = 0; r < 3; ++r) unit[r] = (float)(v[r] / len);
  int big = 0;                                        // component of largest magnitude positive (M2DP's orient)
  for (int r = 1; r < 3; ++r)
    if (std::fabs(unit[r]) > std::fabs(unit[big])) big = r;
  if (unit[big] < 0.0f)
    for (int r = 0; r < 3; ++r) unit[r] = -unit[r];
  return 1;
}

struct Box { int64_t first_index; float mean[3], normal[3]; };

// The median-split recursion of CalculateNormals (cloud_types.cc:105-144) with the oracle's deterministic tie order
// (coordinate, then index), over the float cloud widened to double, as the product's k-d tree builder splits it.
struct Recursion {
  const float* pts;
  std::vector<double> p64;
  std::vector<int> idx;
  std::vector<Box> kept;

  void Leaf(int first, int last) {
    const int count = last - first;
    if (count <= 0) return;
    std::sort(idx.begin() + first, idx.begin() + last);
    float d[7][3];
    for (int i = 0; i < count; ++i)
      for (int r = 0; r < 3; ++r) d[i][r] = pts[3 * (size_t)idx[first + i] + r];
    Box b;
    float cov[9];
    if (!EigenLeaf(d, count, b.mean, cov, b.normal)) return;
    b.first_index = idx[first];
    kept.push_back(b);
  }

  void Build(int first, int last, const double* minv, const double* maxv) {
    const int count = last - first;
    if (count <= 7) { Leaf(first, last); return; }
    int cut_dim = 0;                                  // ArgMax (cloud_types.cc:41-56): first strictly greater, from 0
    double best = 0.0;
    for (int r = 0; r < 3; ++r)
      if (maxv[r] - minv[r] > best) { best = maxv[r] - minv[r]; cut_dim = r; }
    const int left_count = count - count / 2;
    const double* c = p64.data();
    std::nth_element(idx.begin() + first, idx.begin() + first + left_count, idx.begin() + last, [&](int a, int b) {
      const double ca = c[3 * (size_t)a + cut_dim], cb = c[3 * (size_t)b + cut_dim];
      return ca < cb || (ca == cb && a < b);
    });
    const double cut_val = c[3 * (size_t)idx[first + left_count] + cut_dim];
    double left_max[3] = {maxv[0], maxv[1], maxv[2]}, right_min[3] = {minv[0], minv[1], minv[2]};
    left_max[cut_dim] = cut_val;
    right_min[cut_dim] = cut_val;
    Build(first, first + left_count, minv, left_max);
    Build(first + left_count, last, right_min, maxv);
  }
};

}  // namespace

extern "C" {

int sm_oracle_pm_surface_normal_leaf(const float* members_3k, int count, float* mean3, float* cov9, float* normal3) {
  if (count < 1 || count > 7) return -1;
  float d[7][3];
  for (int i = 0; i < count; ++i)
    for (int r = 0; r < 3; ++r) d[i][r] = members_3k[3 * i + r];
  return EigenLeaf(d, count, mean3, cov9, normal3);
}

// The whole filter over n packed float points: the m kept boxes in ascending order of their smallest member index,
// means_3n / normals_3n (floats) and first_index_n; returns m.
int64_t sm_oracle_pm_surface_normals(const float* points_3n, int64_t n, float* means_3n, float* normals_3n,
                                     int64_t* first_index_n) {
  if (n <= 0) return 0;
  Recursion rc;
  rc.pts = points_3n;
  rc.p64.assign(points_3n, points_3n + 3 * (size_t)n);
  rc.idx.resize((size_t)n);
  std::iota(rc.idx.begin(), rc.idx.end(), 0);
  double minv[3], maxv[3];
  for (int r = 0; r < 3; ++r) { minv[r] = std::numeric_limits<double>::infinity(); maxv[r] = -minv[r]; }
  for (int64_t i = 0; i < n; ++i)
    for (int r = 0; r < 3; ++r) {
      minv[r] = std::min(minv[r], rc.p64[3 * (size_t)i + r]);
      maxv[r] = std::max(maxv[r], rc.p64[3 * (size_t)i + r]);
    }
  rc.Build(0, (int)n, minv, maxv);
  std::sort(rc.kept.begin(), rc.kept.end(), [](const Box& a, const Box& b) { return a.first_index < b.first_index; });
  for (size_t j = 0; j < rc.kept.size(); ++j) {
    for (int r = 0; r < 3; ++r) {
      means_3n[3 * j + r] = rc.kept[j].mean[r];
      normals_3n[3 * j + r] = rc.kept[j].normal[r];
    }
    first_index_n[j] = rc.kept[j].first_index;
  }
  return (int64_t)rc.kept.size();
}

}  // extern "C"
