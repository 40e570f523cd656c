// Host side of registrator::Ndt: the scalar control flow of
// NormalDistributionsTransform::computeTransformation (ndt_omp_impl.hpp:81-171) and the small
// pieces it needs per iteration (Gauss constants :86-93, angular derivative tables :288-393,
// pose <-> 6-vector :103-111,146-149, 6x6 JacobiSVD solve :127-129).  The per-point work is in
// ndt.cu; one 44-double read-back per derivative evaluation is the only device -> host traffic.
#ifndef SM_B200_NDT_HOST_H_
#define SM_B200_NDT_HOST_H_

#include <math.h>
#include <string.h>

#include <algorithm>
#include <limits>

#include "kernels.h"

namespace smb {
namespace ndt {

struct Options {                 // defaults of the reference (ndt.cc:31, ndt_omp_impl.hpp:49-51,71-72)
  float resolution = 1.0f;
  double step_size = 0.1;
  double outlier_ratio = 0.55;
  double transformation_epsilon = 0.1;
  int max_iterations = 35;
  int search = kNdtKdtree;       // setNeighborhoodSearchMethod (ndt_omp.h:184); the reference sets KDTREE (ndt.cc:33)
};

inline void angle_tables(const double* p, NdtEvalParams* P) {
  double cx, cy, cz, sx, sy, sz;
  if (fabs(p[3]) < 10e-5) { cx = 1.0; sx = 0.0; } else { cx = cos(p[3]); sx = sin(p[3]); }
  if (fabs(p[4]) < 10e-5) { cy = 1.0; sy = 0.0; } else { cy = cos(p[4]); sy = sin(p[4]); }
  if (fabs(p[5]) < 10e-5) { cz = 1.0; sz = 0.0; } else { cz = cos(p[5]); sz = sin(p[5]); }
  const double J[8][3] = {
      {(-sx * sz + cx * sy * cz), (-sx * cz - cx * sy * sz), (-cx * cy)},
      {(cx * sz + sx * sy * cz), (cx * cz - sx * sy * sz), (-sx * cy)},
      {(-sy * cz), sy * sz, cy},
      {sx * cy * cz, (-sx * cy * sz), sx * sy},
      {(-cx * cy * cz), cx * cy * sz, (-cx * sy)},
      {(-cy * sz), (-cy * cz), 0},
      {(cx * cz - sx * sy * sz), (-cx * sz - sx * sy * cz), 0},
      {(sx * cz + cx * sy * sz), (cx * sy * cz - sx * sz), 0}};
  const double H[15][3] = {
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), sx * cy},
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), (-cx * cy)},
      {(cx * cy * cz), (-cx * cy * sz), (cx * sy)},
      {(sx * cy * cz), (-sx * cy * sz), (sx * sy)},
      {(-sx * cz - cx * sy * sz), (sx * sz - cx * sy * cz), 0},
      {(cx * cz - sx * sy * sz), (-sx * sy * cz - cx * sz), 0},
      {(-cy * cz), (cy * sz), (sy)},
      {(-sx * sy * cz), (sx * sy * sz), (sx * cy)},
      {(cx * sy * cz), (-cx * sy * sz), (-cx * cy)},
      {(sy * sz), (sy * cz), 0},
      {(-sx * cy * sz), (-sx * cy * cz), 0},
      {(cx * cy * sz), (cx * cy * cz), 0},
      {(-cy * cz), (cy * sz), 0},
      {(-cx * sz - sx * sy * cz), (-cx * cz + sx * sy * sz), 0},
      {(-sx * sz + cx * sy * cz), (-cx * sy * sz - sx * cz), 0}};
  for (int r = 0; r < 8; ++r) for (int c = 0; c < 3; ++c) { P->j_ang[r][c] = (float)J[r][c]; P->j_ang_d[r][c] = J[r][c]; }
  for (int r = 0; r < 15; ++r) for (int c = 0; c < 3; ++c) { P->h_ang[r][c] = (float)H[r][c]; P->h_ang_d[r][c] = H[r][c]; }
}

inline void axis_rotation(float angle, int axis, float* R) {   // AngleAxis<float>::toRotationMatrix
  const float s = sinf(angle), c = cosf(angle);
  float ax[3] = {0, 0, 0};
  ax[axis] = 1.0f;
  const float sa[3] = {s * ax[0], s * ax[1], s * ax[2]};
  const float ca[3] = {(1.0f - c) * ax[0], (1.0f - c) * ax[1], (1.0f - c) * ax[2]};
  float t;
  t = ca[0] * ax[1]; R[1] = t - sa[2]; R[3] = t + sa[2];
  t = ca[0] * ax[2]; R[2] = t + sa[1]; R[6] = t - sa[1];
  t = ca[1] * ax[2]; R[5] = t - sa[0]; R[7] = t + sa[0];
  R[0] = ca[0] * ax[0] + c; R[4] = ca[1] * ax[1] + c; R[8] = ca[2] * ax[2] + c;
}
inline void mul3(const float* A, const float* B, float* C) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) C[r * 3 + c] = (A[r * 3] * B[c] + A[r * 3 + 1] * B[3 + c]) + A[r * 3 + 2] * B[6 + c];
}
// Translation * AngleAxis(X) * AngleAxis(Y) * AngleAxis(Z), single precision, column-major out
inline void transform_from_p(const double* p, float* T) {
  float Rx[9], Ry[9], Rz[9], Rxy[9], R[9];
  axis_rotation((float)p[3], 0, Rx);
  axis_rotation((float)p[4], 1, Ry);
  axis_rotation((float)p[5], 2, Rz);
  mul3(Rx, Ry, Rxy);
  mul3(Rxy, Rz, R);
  for (int i = 0; i < 16; ++i) T[i] = 0.0f;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T[r + 4 * c] = R[r * 3 + c];
    T[12 + r] = (float)p[r];
  }
  T[15] = 1.0f;
}
// The parameters of computeDerivatives for o: Gauss constants (:86-93), radius, term math (f64_math: stock PCL's
// double form, else pclomp's float form); at pose vector p also its transform and angle tables, which newton_loop
// sets otherwise.
inline NdtEvalParams eval_params(const Options& o, bool f64_math, const double* p = nullptr) {
  NdtEvalParams P;
  memset(&P, 0, sizeof(P));
  const double c1 = 10.0 * (1 - o.outlier_ratio);
  const double c2 = o.outlier_ratio / pow((double)o.resolution, 3);
  const double d3 = -log(c2);
  P.gauss_d1 = -log(c1 + c2) - d3;
  P.gauss_d2 = -2 * log((-log(c1 * exp(-0.5) + c2) - d3) / P.gauss_d1);
  P.radius = o.resolution;
  P.f64_math = f64_math ? 1 : 0;
  if (p) {
    angle_tables(p, &P);
    transform_from_p(p, P.T);
  }
  return P;
}

// translation + rotation().eulerAngles(0,1,2), single precision (Eigen 3.3 EulerAngles.h)
inline void p_from_transform(const float* T, double* p) {
  const float pi = 3.14159265358979323846f;
  float r0 = atan2f(T[9], T[10]);
  const float c2 = sqrtf(T[0] * T[0] + T[4] * T[4]);
  float r1;
  if (r0 > 0.0f) { r0 -= pi; r1 = atan2f(-T[8], -c2); } else { r1 = atan2f(-T[8], c2); }
  const float s1 = sinf(r0), c1 = cosf(r0);
  const float r2 = atan2f(s1 * T[2] - c1 * T[1], c1 * T[5] - s1 * T[6]);
  p[0] = T[12]; p[1] = T[13]; p[2] = T[14];
  p[3] = -r0; p[4] = -r1; p[5] = -r2;
}

// JacobiSVD(H).solve(b) for a 6x6 (row-major) matrix: one-sided Jacobi
inline void svd_solve6(const double* A, const double* b, double* x) {
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
        off = std::max(off, fabs(gamma) / sqrt(alpha * beta + std::numeric_limits<double>::min()));
        const double zeta = (beta - alpha) / (2.0 * gamma);
        const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
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
    sv[j] = sqrt(s);
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

// NormalDistributionsTransform::computeTransformation (ndt_omp_impl.hpp:81-171) as the reference executes it, over
// an evaluation callback: eval(P, p, sums) runs computeDerivatives for the pose vector p (P.T and the angle tables
// of P are built from it) and fills
// sums[0] = score, sums[1..6] = gradient, sums[7..42] = Hessian (row-major), sums[43] = neighbour count over all
// points; it returns < 0 on error (propagated).  P comes in from eval_params without a pose.
// The device path passes a lambda around NdtStage::eval (ndt_run of the C ABI); the test hook sm_debug_ndt_newton
// passes a caller-supplied function, so this control flow is exercised on the host against an independent
// restatement.
struct NewtonOut {
  float final_T[16];           // final_transformation_, column-major
  int iterations = 0;          // nr_iterations_
  int evaluations = 0;         // computeDerivatives calls
  double score = 0.0;          // of the last evaluation
  double nb_sum = 0.0;         // sum over the evaluations of (neighbours per point)
};

template <class Eval>
inline int newton_loop(const Options& o, const double* guess, int ns, NdtEvalParams& P, Eval eval, NewtonOut* out) {
  float* final_T = out->final_T;
  bool guess_is_identity = true;
  for (int i = 0; i < 16; ++i) {
    final_T[i] = (i % 5 == 0) ? 1.0f : 0.0f;
    if ((float)guess[i] != final_T[i]) guess_is_identity = false;
  }
  if (!guess_is_identity) for (int i = 0; i < 16; ++i) final_T[i] = (float)guess[i];   // :95-101
  double p[6];
  p_from_transform(final_T, p);                                       // :103-111
  for (int i = 0; i < 16; ++i) P.T[i] = final_T[i];
  angle_tables(p, &P);
  double sums[44] = {0.0}, score = 0, grad[6], hess[36], nb_sum = 0.0;
  int evals = 0;
  auto read_sums = [&]() {
    score = sums[0];
    for (int i = 0; i < 6; ++i) grad[i] = sums[1 + i];
    for (int i = 0; i < 36; ++i) hess[i] = sums[7 + i];
    nb_sum += sums[43] / (double)ns;
    ++evals;
  };
  int rc = eval(P, p, sums);                                          // :119
  if (rc < 0) return rc;
  read_sums();
  int nr_iterations = 0;
  bool converged = false;
  while (!converged) {
    double neg_grad[6], delta[6];
    for (int i = 0; i < 6; ++i) neg_grad[i] = -grad[i];
    svd_solve6(hess, neg_grad, delta);                                // :127-129
    double norm = 0.0;
    for (int i = 0; i < 6; ++i) norm += delta[i] * delta[i];
    norm = sqrt(norm);
    if (norm == 0.0 || norm != norm) break;                           // :134-139
    for (int i = 0; i < 6; ++i) delta[i] /= norm;
    // computeStepLengthMT (:757-916); its More-Thuente loop never runs because
    // interval_converged starts as (step_max - step_min) > 0 == true (:802)
    double d_phi_0 = 0.0;
    for (int i = 0; i < 6; ++i) d_phi_0 += grad[i] * delta[i];
    d_phi_0 = -d_phi_0;
    double a_t = 0.0;
    bool evaluate = true;
    if (d_phi_0 >= 0.0) {
      if (d_phi_0 == 0.0) evaluate = false;
      else for (int i = 0; i < 6; ++i) delta[i] = -delta[i];
    }
    if (evaluate) {
      a_t = std::max(std::min(norm, o.step_size), o.transformation_epsilon / 2.0);
      double x_t[6];
      for (int i = 0; i < 6; ++i) x_t[i] = p[i] + delta[i] * a_t;
      transform_from_p(x_t, final_T);                                 // :809-812
      for (int i = 0; i < 16; ++i) P.T[i] = final_T[i];
      angle_tables(x_t, &P);
      rc = eval(P, x_t, sums);                                        // :818
      if (rc < 0) return rc;
      read_sums();
    }
    for (int i = 0; i < 6; ++i) p[i] += delta[i] * a_t;               // :143,152
    if (nr_iterations > o.max_iterations ||
        (nr_iterations && fabs(a_t) < o.transformation_epsilon))
      converged = true;                                                // :158-162
    ++nr_iterations;
  }
  out->iterations = nr_iterations;
  out->evaluations = evals;
  out->score = score;
  out->nb_sum = nb_sum;
  return 0;
}

}  // namespace ndt
}  // namespace smb

#endif  // SM_B200_NDT_HOST_H_
