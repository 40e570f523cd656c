// ORACLE — TEST INFRASTRUCTURE ONLY.  PARITY UNPINNED.  registrator::Ndt with each of pclomp's four neighbour
// searches (pclomp::NormalDistributionsTransform::setNeighborhoodSearchMethod, registrators/pclomp/ndt_omp.h:184;
// switch at ndt_omp_impl.hpp:233-246), restated on the CPU from the pieces libsm_oracle.so exports: the target
// grid (sm_oracle_ndt_voxels), the per-(point, voxel) term math (oracle/ndt_math.h) and the exact 1-NN of the
// fitness score.  tests/oracle_ndt_search.py builds it next to libsm_oracle.so and binds it.
//
// KDTREE is VoxelGridCovariance::radiusSearch as oracle/ndt_oracle.cc states it (centroids with float squared
// distance < resolution^2 in the 3x3x3 cells around the query, sorted by distance, ties by leaf index); with it,
// sm_oracle_ndt_align_search is sm_oracle_ndt_align operation for operation, and the tests require the two to agree
// bit for bit.
//
// DIRECT26 / DIRECT7 / DIRECT1 are VoxelGridCovariance::getNeighborhoodAtPoint / 7 / 1
// (voxel_grid_covariance_omp_impl.hpp:373-441).  Facts of that code kept on purpose:
//  * the query cell is static_cast<int>(floor(p / leaf_size_)) per axis (:379-381): a float DIVISION by the
//    resolution, where the grid build and the KDTREE probe multiply by inverse_leaf_size_; at resolutions that are
//    not powers of two the two disagree for points on or near a cell face;
//  * each offset d of the list is taken in list order when min_b <= ijk + d <= max_b on every axis (:385-390); its
//    leaf, (ijk + d - min_b) . divb_mul, is kept when it exists and has nr_points >= min_points_per_voxel_ = 6
//    (:394-395), so a leaf that failed the eigenvalue test or whose inverse covariance had an inf (nr_points = -1,
//    :337-341, :359-364) is NOT a neighbour, while KDTREE keeps it with icov = 0;
//  * no distance test and no sort: the per-point sums follow the offset order;
//  * DIRECT1 = {(0,0,0)} (:437-441); DIRECT7 = (0,0,0), (+1,0,0), (-1,0,0), (0,+1,0), (0,-1,0), (0,0,+1), (0,0,-1)
//    (:418-432); DIRECT26 = pcl::getAllNeighborCellIndices() (:413).  That function lives in stock PCL
//    (pcl/filters/voxel_grid.h), which is NOT vendored, so its list cannot be verified from the reference tree; it
//    is restated from upstream PCL: the 13 offsets (i, j, -1) for i = -1..1 and, inside that, j = -1..1, then
//    (i, -1, 0) for i = -1..1, then (-1, 0, 0), followed by their 13 negatives.  It holds no (0, 0, 0): DIRECT26
//    never visits the query's own cell.
// Decision where the reference is undefined: static_cast<int> of a non-finite or out-of-range floor value is
// undefined behaviour.  Here a point whose floor(p / leaf_size) is not finite or lies outside [min_b - 1, max_b + 1]
// on some axis has no neighbour; wherever the reference is defined that is its result.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <map>
#include <vector>

#include "ndt_math.h"
#include "sm_oracle.h"

namespace sm_oracle {
int ExactNn1Float(const float* target_xyz, int64_t nt, const float* query_xyz, int64_t nq, int32_t* ids_out);
}

using namespace sm_oracle;

namespace {

struct Leaf {
  int nr_points;
  bool searchable;
  double mean[3], icov[9];
  float centroid[3];
};

struct Grid {
  float leaf_size = 1.0f, inv_leaf = 1.0f;
  int min_b[3], max_b[3], mul[3];
  std::map<int, Leaf> leaves;

  bool Build(const float* pts, int64_t n, float resolution) {
    std::vector<int32_t> idx((size_t)n), npts((size_t)n), srch((size_t)n);
    std::vector<double> mean((size_t)(3 * n)), icov((size_t)(9 * n));
    std::vector<float> cen((size_t)(3 * n));
    const int64_t k = sm_oracle_ndt_voxels(pts, n, resolution, n, idx.data(), npts.data(), mean.data(), icov.data(),
                                           cen.data(), srch.data());
    if (k < 0) return false;
    leaf_size = resolution;
    inv_leaf = 1.0f / resolution;
    float mn[3] = {std::numeric_limits<float>::max(), std::numeric_limits<float>::max(), std::numeric_limits<float>::max()};
    float mx[3] = {-mn[0], -mn[1], -mn[2]};
    for (int64_t i = 0; i < n; ++i)
      for (int d = 0; d < 3; ++d) { mn[d] = std::min(mn[d], pts[3 * i + d]); mx[d] = std::max(mx[d], pts[3 * i + d]); }
    for (int d = 0; d < 3; ++d) {   // voxel_grid_covariance_omp_impl.hpp:88-97
      min_b[d] = (int)std::floor(mn[d] * inv_leaf);
      max_b[d] = (int)std::floor(mx[d] * inv_leaf);
    }
    mul[0] = 1; mul[1] = max_b[0] - min_b[0] + 1; mul[2] = mul[1] * (max_b[1] - min_b[1] + 1);
    for (int64_t i = 0; i < k; ++i) {
      Leaf l;
      l.nr_points = npts[(size_t)i];
      l.searchable = srch[(size_t)i] != 0;
      for (int d = 0; d < 3; ++d) { l.mean[d] = mean[(size_t)(3 * i + d)]; l.centroid[d] = cen[(size_t)(3 * i + d)]; }
      for (int q = 0; q < 9; ++q) l.icov[q] = icov[(size_t)(9 * i + q)];
      leaves[idx[(size_t)i]] = l;
    }
    return true;
  }

  // radiusSearch (voxel_grid_covariance_omp.h:471-499) as oracle/ndt_oracle.cc VoxelGrid::Neighbors states it
  int NeighborsKdtree(const float* q, int* keys) const {
    struct Cand { float d; int idx; };
    Cand cand[27];
    int nc = 0;
    int ijk[3];
    for (int d = 0; d < 3; ++d) ijk[d] = (int)(std::floor(q[d] * inv_leaf) - (float)min_b[d]);
    const float r2 = leaf_size * leaf_size;
    for (int dz = -1; dz <= 1; ++dz)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int a = ijk[0] + dx, b = ijk[1] + dy, c = ijk[2] + dz;
          if (a < 0 || b < 0 || c < 0 || a > max_b[0] - min_b[0] || b > max_b[1] - min_b[1] || c > max_b[2] - min_b[2])
            continue;
          const int idx = a * mul[0] + b * mul[1] + c * mul[2];
          auto it = leaves.find(idx);
          if (it == leaves.end() || !it->second.searchable) continue;
          const float dd = ndt_dist2f(q[0], q[1], q[2], it->second.centroid);
          if (dd < r2) cand[nc++] = Cand{dd, idx};
        }
    std::sort(cand, cand + nc, [](const Cand& a, const Cand& b) { return a.d < b.d || (a.d == b.d && a.idx < b.idx); });
    for (int i = 0; i < nc; ++i) keys[i] = cand[i].idx;
    return nc;
  }

  // getNeighborhoodAtPoint (voxel_grid_covariance_omp_impl.hpp:373-403) over the offset list rel (3 x m, column k
  // = offset k)
  int NeighborsDirect(const float* p, const int (*rel)[3], int m, int* keys) const {
    int ijk[3];
    for (int d = 0; d < 3; ++d) {
      const float f = std::floor(p[d] / leaf_size);   // :379-381, a division
      if (!(std::isfinite(f) && (double)f >= (double)min_b[d] - 1.0 && (double)f <= (double)max_b[d] + 1.0)) return 0;
      ijk[d] = static_cast<int>(f);
    }
    int k = 0;
    for (int ni = 0; ni < m; ++ni) {
      bool in_box = true;
      for (int d = 0; d < 3; ++d)   // (diff2min <= displacement).all() && (diff2max >= displacement).all()
        if (!(min_b[d] - ijk[d] <= rel[ni][d] && max_b[d] - ijk[d] >= rel[ni][d])) in_box = false;
      if (!in_box) continue;
      const int idx = (ijk[0] + rel[ni][0] - min_b[0]) * mul[0] + (ijk[1] + rel[ni][1] - min_b[1]) * mul[1] +
                      (ijk[2] + rel[ni][2] - min_b[2]) * mul[2];
      auto it = leaves.find(idx);
      if (it != leaves.end() && it->second.nr_points >= 6) keys[k++] = idx;
    }
    return k;
  }

  int Neighbors(int method, const float* p, int* keys) const {
    static const int kDirect1[1][3] = {{0, 0, 0}};
    static const int kDirect7[7][3] = {{0, 0, 0}, {1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
    static int kDirect26[26][3];
    static bool init = false;
    if (!init) {   // pcl::getHalfNeighborCellIndices, then getAllNeighborCellIndices (upstream PCL)
      int idx = 0;
      for (int i = -1; i < 2; i++)
        for (int j = -1; j < 2; j++) { kDirect26[idx][0] = i; kDirect26[idx][1] = j; kDirect26[idx][2] = -1; idx++; }
      for (int i = -1; i < 2; i++) { kDirect26[idx][0] = i; kDirect26[idx][1] = -1; kDirect26[idx][2] = 0; idx++; }
      kDirect26[idx][0] = -1; kDirect26[idx][1] = 0; kDirect26[idx][2] = 0;
      for (int c = 0; c < 13; ++c)
        for (int d = 0; d < 3; ++d) kDirect26[13 + c][d] = -kDirect26[c][d];
      init = true;
    }
    switch (method) {
      case 1: return NeighborsDirect(p, kDirect26, 26, keys);
      case 2: return NeighborsDirect(p, kDirect7, 7, keys);
      case 3: return NeighborsDirect(p, kDirect1, 1, keys);
      default: return NeighborsKdtree(p, keys);
    }
  }
};

// computeDerivatives (ndt_omp_impl.hpp:180-284), pclomp's float term math, serial, points in index order
void ComputeDerivatives(const Grid& grid, int method, const float* src, const float* trans, int64_t n, const double p[6],
                        const NdtGauss& g, double* score_out, double grad[6], double hess[36], double* mean_neighbors) {
  NdtAngular ang;
  ndt_angle_derivatives(p, &ang);
  double score = 0.0;
  for (int i = 0; i < 6; ++i) grad[i] = 0.0;
  for (int i = 0; i < 36; ++i) hess[i] = 0.0;
  int64_t total_nb = 0;
  for (int64_t i = 0; i < n; ++i) {
    int nb[27];
    const int k = grid.Neighbors(method, trans + 3 * i, nb);
    total_nb += k;
    double score_pt = 0.0, grad_pt[6] = {0, 0, 0, 0, 0, 0}, hess_pt[36];
    for (int q = 0; q < 36; ++q) hess_pt[q] = 0.0;
    for (int j = 0; j < k; ++j) {
      const Leaf& l = grid.leaves.at(nb[j]);
      score_pt += ndt_update_derivatives(&ang, &g, src + 3 * i, trans + 3 * i, l.mean, l.icov, grad_pt, hess_pt);
    }
    score += score_pt;
    for (int q = 0; q < 6; ++q) grad[q] += grad_pt[q];
    for (int q = 0; q < 36; ++q) hess[q] += hess_pt[q];
  }
  *score_out = score;
  if (mean_neighbors) *mean_neighbors = n > 0 ? (double)total_nb / (double)n : 0.0;
}

// Eigen::JacobiSVD(H).solve(b) as oracle/ndt_oracle.cc SvdSolve6 states it (ndt_omp_impl.hpp:127-129)
void SvdSolve6(const double* A, const double* b, double* x) {
  double U[36], V[36];
  for (int i = 0; i < 36; ++i) { U[i] = A[i]; V[i] = 0.0; }
  for (int i = 0; i < 6; ++i) V[i * 6 + i] = 1.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 6; ++p)
      for (int q = p + 1; q < 6; ++q) {
        double alpha = 0, beta = 0, gamma = 0;
        for (int k = 0; k < 6; ++k) { alpha += U[k * 6 + p] * U[k * 6 + p]; beta += U[k * 6 + q] * U[k * 6 + q]; gamma += U[k * 6 + p] * U[k * 6 + q]; }
        if (gamma == 0.0) continue;
        off = std::max(off, std::fabs(gamma) / std::sqrt(alpha * beta + std::numeric_limits<double>::min()));
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (std::fabs(zeta) + std::sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / std::sqrt(1.0 + t * t), s = c * t;
        for (int k = 0; k < 6; ++k) {
          const double up = U[k * 6 + p], uq = U[k * 6 + q];
          U[k * 6 + p] = c * up - s * uq; U[k * 6 + q] = s * up + c * uq;
          const double vp = V[k * 6 + p], vq = V[k * 6 + q];
          V[k * 6 + p] = c * vp - s * vq; V[k * 6 + q] = s * vp + c * vq;
        }
      }
    if (off < 1e-15) break;
  }
  double sv[6], svmax = 0.0;
  for (int j = 0; j < 6; ++j) {
    double s = 0.0;
    for (int k = 0; k < 6; ++k) s += U[k * 6 + j] * U[k * 6 + j];
    sv[j] = std::sqrt(s);
    svmax = std::max(svmax, sv[j]);
  }
  const double thr = std::max(svmax * 6.0 * std::numeric_limits<double>::epsilon(), std::numeric_limits<double>::min());
  for (int i = 0; i < 6; ++i) x[i] = 0.0;
  for (int j = 0; j < 6; ++j) {
    if (!(sv[j] > thr)) continue;
    double dot = 0.0;
    for (int k = 0; k < 6; ++k) dot += U[k * 6 + j] * b[k];
    dot /= (sv[j] * sv[j]);
    for (int i = 0; i < 6; ++i) x[i] += V[i * 6 + j] * dot;
  }
}

}  // namespace

extern "C" {

/* Neighbour leaf indices of each point (the points as the search sees them, i.e. already transformed) for method
 * 0 KDTREE, 1 DIRECT26, 2 DIRECT7, 3 DIRECT1: counts[i] entries keys_27n[27 i ..] in the order computeDerivatives
 * uses them.  -1: grid overflow (sm_oracle_ndt_voxels). */
int sm_oracle_ndt_search_neighbors(const float* target, int64_t nt, float resolution, int32_t method,
                                   const float* points, int64_t n, int32_t* counts, int32_t* keys_27n) {
  Grid grid;
  if (!grid.Build(target, nt, resolution)) return -1;
  for (int64_t i = 0; i < n; ++i) counts[i] = grid.Neighbors(method, points + 3 * i, keys_27n + 27 * i);
  return 0;
}

/* computeDerivatives at pose vector p with the method's neighbour search (pclomp's float term math). */
int sm_oracle_ndt_search_derivatives(const float* source, int64_t ns, const float* target, int64_t nt,
                                     const sm_oracle_ndt_options* opt, int32_t method, const double* p, double* score,
                                     double* grad6, double* hess36, double* mean_neighbors) {
  Grid grid;
  if (!grid.Build(target, nt, opt->resolution)) return -1;
  NdtGauss g;
  ndt_gauss_constants(opt->outlier_ratio, opt->resolution, &g);
  float T[16];
  ndt_transform_from_p(p, T);
  std::vector<float> trans((size_t)(3 * ns));
  for (int64_t i = 0; i < ns; ++i) ndt_transform_point(T, source + 3 * i, &trans[(size_t)(3 * i)]);
  ComputeDerivatives(grid, method, source, trans.data(), ns, p, g, score, grad6, hess36, mean_neighbors);
  return 0;
}

/* Ndt::Align (ndt.cc:38-64) with the method's neighbour search: sm_oracle_ndt_align plus the number of
 * computeDerivatives calls.  Returns 1 / 0 like the reference's bool, -1 on grid overflow. */
int sm_oracle_ndt_search_align(const float* source, int64_t ns, const float* target, int64_t nt, const double* guess,
                               const sm_oracle_ndt_options* opt, int32_t method, double* result, double* fitness,
                               int32_t* iterations, int32_t* evaluations, double* trans_probability,
                               double* mean_neighbors) {
  if (ns <= 0 || nt <= 0) return 0;
  Grid grid;
  if (!grid.Build(target, nt, opt->resolution)) return -1;
  NdtGauss g;
  ndt_gauss_constants(opt->outlier_ratio, opt->resolution, &g);
  float final_T[16], guess_f[16];
  bool guess_is_identity = true;
  for (int i = 0; i < 16; ++i) {
    guess_f[i] = (float)guess[i];
    final_T[i] = (i % 5 == 0) ? 1.0f : 0.0f;
    if (guess_f[i] != final_T[i]) guess_is_identity = false;
  }
  std::vector<float> trans(source, source + 3 * ns);
  if (!guess_is_identity) {                              // ndt_omp_impl.hpp:95-101
    std::memcpy(final_T, guess_f, sizeof(final_T));
    for (int64_t i = 0; i < ns; ++i) ndt_transform_point(guess_f, source + 3 * i, &trans[(size_t)(3 * i)]);
  }
  double p[6];
  ndt_p_from_transform(final_T, p);                      // :103-111
  double score = 0.0, grad[6], hess[36], nbm = 0.0, nb_sum = 0.0;
  int evals = 0;
  ComputeDerivatives(grid, method, source, trans.data(), ns, p, g, &score, grad, hess, &nbm);
  nb_sum += nbm; ++evals;
  int nr_iterations = 0;
  bool converged = false;
  while (!converged) {
    double neg_grad[6], delta[6];
    for (int i = 0; i < 6; ++i) neg_grad[i] = -grad[i];
    SvdSolve6(hess, neg_grad, delta);                    // :127-129
    double norm = 0.0;
    for (int i = 0; i < 6; ++i) norm += delta[i] * delta[i];
    norm = std::sqrt(norm);
    if (norm == 0.0 || norm != norm) break;              // :134-139
    for (int i = 0; i < 6; ++i) delta[i] /= norm;
    double d_phi_0 = 0.0;                                // computeStepLengthMT, loop never runs (:757-916)
    for (int i = 0; i < 6; ++i) d_phi_0 += grad[i] * delta[i];
    d_phi_0 = -d_phi_0;
    double a_t = 0.0;
    bool evaluate = true;
    if (d_phi_0 >= 0.0) {
      if (d_phi_0 == 0.0) evaluate = false;
      else for (int i = 0; i < 6; ++i) delta[i] = -delta[i];
    }
    if (evaluate) {
      a_t = std::max(std::min(norm, opt->step_size), opt->transformation_epsilon / 2.0);
      double x_t[6];
      for (int i = 0; i < 6; ++i) x_t[i] = p[i] + delta[i] * a_t;
      ndt_transform_from_p(x_t, final_T);                // :809-812
      for (int64_t i = 0; i < ns; ++i) ndt_transform_point(final_T, source + 3 * i, &trans[(size_t)(3 * i)]);
      ComputeDerivatives(grid, method, source, trans.data(), ns, x_t, g, &score, grad, hess, &nbm);
      nb_sum += nbm; ++evals;
    }
    for (int i = 0; i < 6; ++i) p[i] += delta[i] * a_t;  // :143,152
    if (nr_iterations > opt->max_iterations || (nr_iterations && std::fabs(a_t) < opt->transformation_epsilon))
      converged = true;                                   // :158-162
    ++nr_iterations;
  }
  *trans_probability = score / (double)ns;               // :170
  *iterations = nr_iterations;
  *evaluations = evals;
  *mean_neighbors = nb_sum / evals;
  std::vector<float> moved((size_t)(3 * ns));            // getFitnessScore (ndt.cc:60)
  for (int64_t i = 0; i < ns; ++i) ndt_transform_point(final_T, source + 3 * i, &moved[(size_t)(3 * i)]);
  std::vector<int32_t> ids((size_t)ns);
  ExactNn1Float(target, nt, moved.data(), ns, ids.data());
  double fit = 0.0;
  int64_t nr = 0;
  for (int64_t i = 0; i < ns; ++i) {
    if (ids[(size_t)i] < 0) continue;
    fit += (double)ndt_dist2f(moved[(size_t)(3 * i)], moved[(size_t)(3 * i + 1)], moved[(size_t)(3 * i + 2)],
                              target + 3 * (int64_t)ids[(size_t)i]);
    ++nr;
  }
  *fitness = nr > 0 ? fit / (double)nr : std::numeric_limits<double>::max();
  for (int i = 0; i < 16; ++i) result[i] = (double)final_T[i];
  return 1;
}

}  // extern "C"
