// ORACLE — TEST INFRASTRUCTURE ONLY.  IcpFast::Align with Interface::EnableInnerCompensation
// (registrators/icp_fast.cc:455-529 with :487-491, :506-510, :284-289), restated in double on the CPU from the
// pieces libsm_oracle.so exports: the libnabo k-d tree (sm_oracle_knn1), the trim index, the 6x6 solve, the
// convergence test and common::InterpolateTransform (oracle/motion_oracle.cc).  Linked into libsm_oracle.so;
// tests/oracle_compensation.py binds it.
//
// With the flag set, every iteration moves source point i (its column in SetInputSource, after G0) by
// InterpolateTransform(Identity, T_iter, f_i), f_i = (double)i / N (cloud_types.cc:340-344), passed as the
// function's float parameter, instead of by T_iter; the kept match's Jacobian column is scaled by the double
// f_i (wF and F, :284-289); the residual is not.  The reference's ApplyMotionCompensation (cloud_types.cc:306-318)
// interpolates towards a local that shadows its parameter and is read uninitialised (undefined behaviour); this
// restatement interpolates towards T_iter, which is what the code evidently intends.
//
// With the flag clear it is sm_oracle_icp_fast_align, operation for operation: the tests require the two to agree
// bit for bit.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

#include "linalg.h"
#include "sm_oracle.h"

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

int sm_oracle_icp_fast_align_compensated(const double* source, int64_t n_source, const double* target,
                                         const double* target_normals, int64_t n_target, const double* guess,
                                         const sm_oracle_icp_options* opt, int32_t inner_compensation,
                                         double* result, double* final_score, int32_t* iterations,
                                         sm_oracle_icp_trace* trace, int32_t trace_capacity) {
  if (n_source <= 0 || n_target <= 0) return -1;
  const int64_t ns = n_source, nt = n_target;
  // :456-463 target mean (a sequential loop per row), centre
  double mean[3] = {0.0, 0.0, 0.0};
  for (int r = 0; r < 3; ++r) {
    double s = 0.0;
    for (int64_t j = 0; j < nt; ++j) s += target[3 * j + r];
    mean[r] = s / (double)(int)nt;
  }
  std::vector<double> Q((size_t)(3 * nt));
  for (int64_t j = 0; j < nt; ++j)
    for (int r = 0; r < 3; ++r) Q[(size_t)(3 * j + r)] = target[3 * j + r] - mean[r];
  // :460-461,:469-471  T_mean, G0 = T_mean^-1 * guess, init_source = G0 (x) source
  double T_mean[16], T_mean_inv[16], G0[16];
  Identity4(T_mean); Identity4(T_mean_inv);
  for (int r = 0; r < 3; ++r) { T_mean[12 + r] = mean[r]; T_mean_inv[12 + r] = -mean[r]; }
  Mul4(T_mean_inv, guess, G0);
  std::vector<double> S0((size_t)(3 * ns)), P((size_t)(3 * ns));
  ApplyTransform(G0, source, S0.data(), ns);

  double T_iter[16];
  Identity4(T_iter);
  std::vector<double> history;   // T_iter of every iteration, for the convergence test (:377-405)
  std::vector<int32_t> ids((size_t)ns);
  std::vector<double> d2((size_t)ns), values;
  values.reserve((size_t)ns);
  int iterator = 0;
  while (true) {
    if (inner_compensation) ApplyMotionCompensation(T_iter, S0.data(), P.data(), ns);   // :487-488
    else ApplyTransform(T_iter, S0.data(), P.data(), ns);                               // :489-491
    // :493 (the tree over the centred target is the same on every iteration)
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
    // :497-498 weights; :113-156 compaction + gathers (factors travel with the kept points, :117,130,160);
    // :256-302 normal equations
    double A[36] = {0}, b[6] = {0};
    double sum_sqrt = 0.0;
    int64_t kept = 0;
    for (int64_t i = 0; i < ns; ++i) {
      const double dist = d2[(size_t)i];
      if (dist == kInf) continue;
      if (!(dist <= limit)) continue;
      const double* p = &P[(size_t)(3 * i)];
      const double* q = &Q[(size_t)(3 * (int64_t)ids[(size_t)i])];
      const double* nrm = target_normals + 3 * (int64_t)ids[(size_t)i];
      double F[6];
      F[0] = p[1] * nrm[2] - p[2] * nrm[1];   // :193-198
      F[1] = p[2] * nrm[0] - p[0] * nrm[2];
      F[2] = p[0] * nrm[1] - p[1] * nrm[0];
      F[3] = nrm[0]; F[4] = nrm[1]; F[5] = nrm[2];
      if (inner_compensation) {                // :284-289
        const double f = (double)i / (double)ns;
        for (int r = 0; r < 6; ++r) F[r] = F[r] * f;
      }
      double dot = 0.0;                        // :296-299
      dot += (p[0] - q[0]) * nrm[0];
      dot += (p[1] - q[1]) * nrm[1];
      dot += (p[2] - q[2]) * nrm[2];
      for (int r = 0; r < 6; ++r) {
        for (int c = 0; c < 6; ++c) A[r * 6 + c] += F[r] * F[c];   // :292 (w == 1)
        b[r] += F[r] * dot;
      }
      sum_sqrt += std::sqrt(dist);
      ++kept;
    }
    if (kept == 0) return -3;
    for (int r = 0; r < 6; ++r) b[r] = -b[r];  // :302
    double x[6];
    sm_oracle_solve6(A, b, x, nullptr);        // A is symmetric: its layout is moot
    // :307-321 parameters -> 4x4
    const double angle = std::sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    double axis[3] = {x[0], x[1], x[2]};
    const double sq = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
    if (sq > 0.0) for (int r = 0; r < 3; ++r) axis[r] = x[r] / std::sqrt(sq);
    double R[9];
    AngleAxisToRotation(angle, axis, R);
    bool has_nan = false;
    for (int i = 0; i < 9; ++i) has_nan |= std::isnan(R[i]);
    for (int i = 3; i < 6; ++i) has_nan |= std::isnan(x[i]);
    if (has_nan) { for (int i = 0; i < 9; ++i) R[i] = 0.0; R[0] = R[4] = R[8] = 1.0; }
    double dT[16];
    Identity4(dT);
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) dT[r + 4 * c] = R[r * 3 + c];
      dT[12 + r] = x[3 + r];
    }
    Mul4(dT, T_iter, T_iter);                   // :506-510
    if (trace && iterator < trace_capacity) {
      sm_oracle_icp_trace& t = trace[iterator];
      std::memcpy(t.T_iter, T_iter, sizeof(T_iter));
      t.limit = limit; t.kept = kept;
      std::memcpy(t.A, A, sizeof(A)); std::memcpy(t.b, b, sizeof(b));
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
  // :527  Eigen evaluates T_mean * T_iter * G0 left to right: (T_mean*T_iter)*G0
  Mul4(T_mean, T_iter, tmp);
  Mul4(tmp, G0, result);
  *iterations = iterator;
  return 1;
}

}  // extern "C"
