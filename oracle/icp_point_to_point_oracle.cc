// ORACLE — TEST INFRASTRUCTURE ONLY.  IcpFast::Align with the point-to-point minimizer: registrators/icp_fast.cc:455-529
// with ComputePointToPoint (:326-375) in place of ComputePointToPlane at :506-510, restated in double on the CPU
// from the pieces libsm_oracle.so exports: the libnabo k-d tree (sm_oracle_knn1), the trim index, the convergence
// test and common::InterpolateTransform.  Linked into libsm_oracle.so; tests/oracle_point_to_point.py binds
// it.
//
// ComputePointToPoint literally, all weights 1 after ErrorElements (:100-135): the means as Eigen's weighted row
// sums times 1 / w.sum(), the kept points centred in a second pass, M = target * source^T over the centred points,
// R = U V^T, the last row of V^T negated when det R < 0, t = qbar - R pbar.  No NaN guard (the reference has none).
// With inner compensation the step cloud is de-skewed as in icp_compensation_oracle.cc; the minimizer has no
// factor term.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

#include "linalg.h"
#include "sm_oracle.h"

// The written-out 3x3 SVD of the product (kabsch_rotation in staticmapping_b200/csrc/linalg_dev.cuh), compiled for
// the host: the SVD is not unique where M is degenerate, so product and oracle share the one whose choices are
// documented there.  The centring around it is restated here literally (two passes); numpy's SVD checks both.
#define __host__
#define __device__
#define __forceinline__ inline
#include "../staticmapping_b200/csrc/linalg_dev.cuh"
#undef __host__
#undef __device__
#undef __forceinline__

using namespace sm_oracle;

namespace {

constexpr double kInf = std::numeric_limits<double>::infinity();

// cloud_types.cc:288-296: 4xN homogeneous product, rows 0..2 kept
void ApplyTransform(const double* T, const double* in, double* out, int64_t n) {
  for (int64_t j = 0; j < n; ++j) {
    const double x = in[3 * j], y = in[3 * j + 1], z = in[3 * j + 2];
    for (int i = 0; i < 3; ++i) {
      double s = T[i + 0] * x;
      s = s + T[i + 4] * y;
      s = s + T[i + 8] * z;
      s = s + T[i + 12] * 1.0;
      out[3 * j + i] = s;
    }
  }
}

// cloud_types.cc:306-318 (with the parameter, see above): R_i * p + t_i
void ApplyMotionCompensation(const double* T, const double* in, double* out, int64_t n) {
  double ident[16], Ti[16];
  Identity4(ident);
  for (int64_t j = 0; j < n; ++j) {
    const double f = (double)j / (double)n;
    sm_oracle_interpolate_transform(ident, T, (float)f, Ti);
    const double x = in[3 * j], y = in[3 * j + 1], z = in[3 * j + 2];
    for (int i = 0; i < 3; ++i) out[3 * j + i] = ((Ti[i] * x + Ti[i + 4] * y) + Ti[i + 8] * z) + Ti[i + 12];
  }
}

}  // namespace

extern "C" {

typedef struct sm_oracle_p2p_trace {   // one record per iteration
  double T_iter[16];
  double limit;
  int64_t kept;
  double pbar[3], qbar[3];
  double M[9];                          // row-major, target x source^T of the centred kept points
  double R[9], t[3];                    // row-major
  int32_t path;                         // 3 Kabsch, 4 with the reflection fix
  int32_t pad;
} sm_oracle_p2p_trace;

// ComputePointToPoint (:326-375) over the n kept pairs p (reading) / q (reference), packed xyz
int sm_oracle_point_to_point(const double* p, const double* q, int64_t n, double* pbar, double* qbar, double* M,
                             double* R, double* t) {
  if (n <= 0) return -1;
  const double w_sum_inv = 1. / (double)n;   // w.sum() of n ones
  for (int r = 0; r < 3; ++r) {
    double sp = 0.0, sq = 0.0;
    for (int64_t j = 0; j < n; ++j) { sp += p[3 * j + r] * 1.0; sq += q[3 * j + r] * 1.0; }
    pbar[r] = sp * w_sum_inv; qbar[r] = sq * w_sum_inv;
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int64_t k = 0; k < n; ++k) s += ((q[3 * k + i] - qbar[i]) * 1.0) * (p[3 * k + j] - pbar[j]);
      M[i * 3 + j] = s;
    }
  const int fix = smb::la::kabsch_rotation(M, R);
  for (int i = 0; i < 3; ++i) t[i] = qbar[i] - ((R[i * 3] * pbar[0] + R[i * 3 + 1] * pbar[1]) + R[i * 3 + 2] * pbar[2]);
  return fix ? 4 : 3;
}

int sm_oracle_icp_fast_align_point_to_point(const double* source, int64_t n_source, const double* target,
                                            int64_t n_target, const double* guess, const sm_oracle_icp_options* opt,
                                            int32_t inner_compensation, double* result, double* final_score,
                                            int32_t* iterations, sm_oracle_p2p_trace* trace, int32_t trace_capacity) {
  if (n_source <= 0 || n_target <= 0) return -1;
  const int64_t ns = n_source, nt = n_target;
  double mean[3] = {0.0, 0.0, 0.0};   // :456-463
  for (int r = 0; r < 3; ++r) {
    double s = 0.0;
    for (int64_t j = 0; j < nt; ++j) s += target[3 * j + r];
    mean[r] = s / (double)(int)nt;
  }
  std::vector<double> Q((size_t)(3 * nt));
  for (int64_t j = 0; j < nt; ++j)
    for (int r = 0; r < 3; ++r) Q[(size_t)(3 * j + r)] = target[3 * j + r] - mean[r];
  double T_mean[16], T_mean_inv[16], G0[16];
  Identity4(T_mean); Identity4(T_mean_inv);
  for (int r = 0; r < 3; ++r) { T_mean[12 + r] = mean[r]; T_mean_inv[12 + r] = -mean[r]; }
  Mul4(T_mean_inv, guess, G0);
  std::vector<double> S0((size_t)(3 * ns)), P((size_t)(3 * ns));
  ApplyTransform(G0, source, S0.data(), ns);

  double T_iter[16];
  Identity4(T_iter);
  std::vector<double> history;
  std::vector<int32_t> ids((size_t)ns);
  std::vector<double> d2((size_t)ns), values, kp, kq;
  values.reserve((size_t)ns);
  int iterator = 0;
  while (true) {
    if (inner_compensation) ApplyMotionCompensation(T_iter, S0.data(), P.data(), ns);   // :487-488
    else ApplyTransform(T_iter, S0.data(), P.data(), ns);                               // :489-491
    sm_oracle_knn1(Q.data(), nt, P.data(), ns, opt->knn_epsilon, 8, opt->tie_mode, ids.data(), d2.data());
    values.clear();                                                                      // :65-90
    for (int64_t i = 0; i < ns; ++i)
      if (d2[(size_t)i] != kInf) values.push_back(d2[(size_t)i]);
    if (values.empty()) return -2;
    const double quantile = (double)opt->dist_outlier_ratio;
    double limit;
    if (quantile == 1.0) {
      limit = *std::max_element(values.begin(), values.end());
    } else {
      const int qi = sm_oracle_quantile_index((int64_t)values.size(), opt->dist_outlier_ratio);
      std::nth_element(values.begin(), values.begin() + qi, values.end());
      limit = values[(size_t)qi];
    }
    // :497-498 weights; :113-156 the kept points and their matched target points, in source order
    kp.clear(); kq.clear();
    double sum_sqrt = 0.0;
    for (int64_t i = 0; i < ns; ++i) {
      const double dist = d2[(size_t)i];
      if (dist == kInf || !(dist <= limit)) continue;
      for (int r = 0; r < 3; ++r) {
        kp.push_back(P[(size_t)(3 * i + r)]);
        kq.push_back(Q[(size_t)(3 * (int64_t)ids[(size_t)i] + r)]);
      }
      sum_sqrt += std::sqrt(dist);
    }
    const int64_t kept = (int64_t)(kp.size() / 3);
    if (kept == 0) return -3;
    double pbar[3], qbar[3], M[9], R[9], t[3];
    const int path = sm_oracle_point_to_point(kp.data(), kq.data(), kept, pbar, qbar, M, R, t);
    double dT[16];
    Identity4(dT);
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) dT[r + 4 * c] = R[r * 3 + c];
      dT[12 + r] = t[r];
    }
    Mul4(dT, T_iter, T_iter);                   // :506-510
    if (trace && iterator < trace_capacity) {
      sm_oracle_p2p_trace& tr = trace[iterator];
      std::memcpy(tr.T_iter, T_iter, sizeof(T_iter));
      tr.limit = limit; tr.kept = kept;
      std::memcpy(tr.pbar, pbar, sizeof(pbar)); std::memcpy(tr.qbar, qbar, sizeof(qbar));
      std::memcpy(tr.M, M, sizeof(M)); std::memcpy(tr.R, R, sizeof(R)); std::memcpy(tr.t, t, sizeof(t));
      tr.path = path; tr.pad = 0;
    }
    ++iterator;                                 // :513-515
    history.insert(history.end(), T_iter, T_iter + 16);
    int converged = 0;
    if (!opt->disable_convergence_check) sm_oracle_check_convergence_inputs(history.data(), iterator, &converged);
    if (converged || iterator >= opt->max_iteration) {   // :516-522
      *final_score = std::exp(-(sum_sqrt / (double)kept));
      break;
    }
  }
  double tmp[16];
  Mul4(T_mean, T_iter, tmp);                    // :527
  Mul4(tmp, G0, result);
  *iterations = iterator;
  return 1;
}

}  // extern "C"
