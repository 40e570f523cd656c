// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked or imported by the product path.
//
// Small dense linear algebra (double) restating the Eigen routines the reference's
// registrators/ hot path calls.  Eigen is NOT vendored in the reference and is not
// installed in this image, so these are restatements of Eigen 3.3's published
// algorithms; the call sites that pin which routine is used are cited per function.
// All matrices here are row-major C arrays m[r*n+c] unless stated otherwise.
#ifndef ORACLE_LINALG_H_
#define ORACLE_LINALG_H_

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

namespace sm_oracle {

// 4x4 product C = A*B, column-major 4x4 (Eigen::Matrix4d layout), accumulation order
// k = 0..3 starting from the first product (Eigen lazy/gebp coefficient order).
// Used for icp_fast.cc:470, :506-510, :527.
inline void Mul4(const double* A, const double* B, double* C) {
  double out[16];
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i) {
      double s = A[i + 0 * 4] * B[0 + j * 4];
      s = s + A[i + 1 * 4] * B[1 + j * 4];
      s = s + A[i + 2 * 4] * B[2 + j * 4];
      s = s + A[i + 3 * 4] * B[3 + j * 4];
      out[i + j * 4] = s;
    }
  std::memcpy(C, out, sizeof(out));
}

inline void Identity4(double* T) {
  for (int i = 0; i < 16; ++i) T[i] = 0.0;
  T[0] = T[5] = T[10] = T[15] = 1.0;
}

// ---------------------------------------------------------------------------
// Eigen::FullPivHouseholderQR (Eigen/src/QR/FullPivHouseholderQR.h, computeInPlace,
// rank(), isInvertible()).  Call sites: icp_fast.cc:214 (6x6, isInvertible / rank /
// matrixQ / colsPermutation) and cloud_types.cc:89 (3x3 rank).
// On return:  Qt * A * P = R  (R upper-trapezoidal),  Qt is n x n orthogonal,
// perm[j] = source column of A that ended in column j (P(perm[j], j) = 1).
// ---------------------------------------------------------------------------
template <int N>
struct FullPivQR {
  double R[N * N];
  double Qt[N * N];
  int perm[N];
  int nonzero_pivots;
  double maxpivot;

  void Compute(const double* A) {
    const double eps = std::numeric_limits<double>::epsilon();
    const double precision = eps * double(N);
    std::memcpy(R, A, sizeof(double) * N * N);
    for (int i = 0; i < N * N; ++i) Qt[i] = 0.0;
    for (int i = 0; i < N; ++i) Qt[i * N + i] = 1.0;
    for (int i = 0; i < N; ++i) perm[i] = i;
    nonzero_pivots = N;
    maxpivot = 0.0;
    double biggest = 0.0;
    for (int k = 0; k < N; ++k) {
      // maxCoeff over the bottom-right corner, column-major visiting order, strict '>'.
      int rb = k, cb = k;
      double best = -1.0;
      for (int c = k; c < N; ++c)
        for (int r = k; r < N; ++r) {
          const double v = std::fabs(R[r * N + c]);
          if (v > best) { best = v; rb = r; cb = c; }
        }
      const double biggest_in_corner = best;
      if (k == 0) biggest = biggest_in_corner;
      // internal::isMuchSmallerThan(a, b, prec): |a| <= |b| * prec
      if (std::fabs(biggest_in_corner) <= std::fabs(biggest) * precision) {
        nonzero_pivots = k;
        break;
      }
      if (rb != k) {
        // Eigen swaps only the tail of the row in m_qr (the head holds Householder
        // vectors); R's head entries are zero in this explicit formulation, so a full
        // row swap is equivalent.  The same left operation is applied to Qt.
        for (int c = 0; c < N; ++c) std::swap(R[k * N + c], R[rb * N + c]);
        for (int c = 0; c < N; ++c) std::swap(Qt[k * N + c], Qt[rb * N + c]);
      }
      if (cb != k) {
        for (int r = 0; r < N; ++r) std::swap(R[r * N + k], R[r * N + cb]);
        std::swap(perm[k], perm[cb]);
      }
      // makeHouseholderInPlace on column k, rows k..N-1 (Eigen/src/Householder).
      double tail_sq = 0.0;
      for (int r = k + 1; r < N; ++r) tail_sq += R[r * N + k] * R[r * N + k];
      const double c0 = R[k * N + k];
      double beta, tau;
      double v[N];  // essential part, v[k] = 1 implicitly
      for (int r = 0; r < N; ++r) v[r] = 0.0;
      if (tail_sq <= std::numeric_limits<double>::min()) {
        tau = 0.0;
        beta = c0;
      } else {
        beta = std::sqrt(c0 * c0 + tail_sq);
        if (c0 >= 0.0) beta = -beta;
        for (int r = k + 1; r < N; ++r) v[r] = R[r * N + k] / (c0 - beta);
        tau = (beta - c0) / beta;
      }
      v[k] = 1.0;
      if (std::fabs(beta) > maxpivot) maxpivot = std::fabs(beta);
      // apply H = I - tau v v^T on the left of R (cols k+1..) and of Qt (all cols)
      R[k * N + k] = beta;
      for (int r = k + 1; r < N; ++r) R[r * N + k] = 0.0;
      if (tau != 0.0) {
        for (int c = k + 1; c < N; ++c) {
          double dot = 0.0;
          for (int r = k; r < N; ++r) dot += v[r] * R[r * N + c];
          for (int r = k; r < N; ++r) R[r * N + c] -= tau * v[r] * dot;
        }
        for (int c = 0; c < N; ++c) {
          double dot = 0.0;
          for (int r = k; r < N; ++r) dot += v[r] * Qt[r * N + c];
          for (int r = k; r < N; ++r) Qt[r * N + c] -= tau * v[r] * dot;
        }
      }
    }
  }

  // FullPivHouseholderQR::rank(): pivots with |R(i,i)| > |maxpivot| * eps * N.
  int Rank() const {
    const double thr =
        std::fabs(maxpivot) * (std::numeric_limits<double>::epsilon() * double(N));
    int rank = 0;
    for (int i = 0; i < nonzero_pivots; ++i)
      rank += (std::fabs(R[i * N + i]) > thr) ? 1 : 0;
    return rank;
  }
  bool IsInvertible() const { return Rank() == N; }
};

// Eigen::LLT (unblocked, lower) + solve.  icp_fast.cc:252 (6x6) and :231 (rank x rank).
// A is n x n row-major, symmetric.  Returns false if a pivot is <= 0 (Eigen reports
// NumericalIssue but still returns numbers; we return NaNs like a failed sqrt would).
inline bool LltSolve(const double* A, const double* b, double* x, int n) {
  double L[36];
  bool ok = true;
  for (int i = 0; i < n * n; ++i) L[i] = 0.0;
  for (int k = 0; k < n; ++k) {
    double d = A[k * n + k];
    for (int j = 0; j < k; ++j) d -= L[k * n + j] * L[k * n + j];
    if (d <= 0.0) ok = false;
    const double lkk = std::sqrt(d);
    L[k * n + k] = lkk;
    for (int i = k + 1; i < n; ++i) {
      double s = A[i * n + k];
      for (int j = 0; j < k; ++j) s -= L[i * n + j] * L[k * n + j];
      L[i * n + k] = s / lkk;
    }
  }
  double y[6];
  for (int i = 0; i < n; ++i) {
    double s = b[i];
    for (int j = 0; j < i; ++j) s -= L[i * n + j] * y[j];
    y[i] = s / L[i * n + i];
  }
  for (int i = n - 1; i >= 0; --i) {
    double s = y[i];
    for (int j = i + 1; j < n; ++j) s -= L[j * n + i] * x[j];
    x[i] = s / L[i * n + i];
  }
  return ok;
}

// Symmetric two-sided Jacobi eigen-decomposition A = V diag(w) V^T  (A n x n, n <= 6).
// Stands in for Eigen::JacobiSVD on the symmetric PSD normal matrix (icp_fast.cc:236)
// and for SelfAdjointEigenSolver (voxel_grid_covariance_omp_impl.hpp:333).  Eigenvalues
// are returned unsorted; V row-major with eigenvectors in columns.
inline void JacobiEigenSym(const double* Ain, int n, double* w, double* V) {
  double A[36];
  std::memcpy(A, Ain, sizeof(double) * n * n);
  for (int i = 0; i < n * n; ++i) V[i] = 0.0;
  for (int i = 0; i < n; ++i) V[i * n + i] = 1.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < n; ++p)
      for (int q = p + 1; q < n; ++q) off += A[p * n + q] * A[p * n + q];
    if (off == 0.0) break;
    for (int p = 0; p < n; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = A[p * n + q];
        if (apq == 0.0) continue;
        const double app = A[p * n + p], aqq = A[q * n + q];
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) /
                         (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = c * akp - s * akq;
          A[k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = c * apk - s * aqk;
          A[q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vkp = V[k * n + p], vkq = V[k * n + q];
          V[k * n + p] = c * vkp - s * vkq;
          V[k * n + q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < n; ++i) w[i] = A[i * n + i];
}

// JacobiSVD::solve for a symmetric matrix: pseudo-inverse with Eigen's default rank
// threshold  sv > max(sv_max * n * eps, DBL_MIN).
inline void SymSvdSolve(const double* A, const double* b, double* x, int n) {
  double w[6], V[36];
  JacobiEigenSym(A, n, w, V);
  double svmax = 0.0;
  for (int i = 0; i < n; ++i) svmax = std::max(svmax, std::fabs(w[i]));
  const double thr = std::max(svmax * double(n) * std::numeric_limits<double>::epsilon(),
                              std::numeric_limits<double>::min());
  for (int i = 0; i < n; ++i) x[i] = 0.0;
  for (int k = 0; k < n; ++k) {
    if (!(std::fabs(w[k]) > thr)) continue;
    double dot = 0.0;
    for (int i = 0; i < n; ++i) dot += V[i * n + k] * b[i];
    dot /= w[k];
    for (int i = 0; i < n; ++i) x[i] += V[i * n + k] * dot;
  }
}

// Dynamic-size MatrixXd::inverse() -> PartialPivLU::inverse()  (cloud_types.cc:93:
// `M_wave` is declared MatrixXd, so the fixed 3x3 cofactor path is NOT taken).
// Returns inv (row-major 3x3) of row-major 3x3 M.
inline void PartialPivLuInverse3(const double* M, double* inv) {
  double lu[9];
  int piv[3] = {0, 1, 2};
  std::memcpy(lu, M, sizeof(lu));
  for (int k = 0; k < 3; ++k) {
    int rb = k;
    double best = std::fabs(lu[k * 3 + k]);
    for (int r = k + 1; r < 3; ++r)
      if (std::fabs(lu[r * 3 + k]) > best) { best = std::fabs(lu[r * 3 + k]); rb = r; }
    if (rb != k) {
      for (int c = 0; c < 3; ++c) std::swap(lu[k * 3 + c], lu[rb * 3 + c]);
      std::swap(piv[k], piv[rb]);
    }
    for (int r = k + 1; r < 3; ++r) {
      lu[r * 3 + k] /= lu[k * 3 + k];
      for (int c = k + 1; c < 3; ++c) lu[r * 3 + c] -= lu[r * 3 + k] * lu[k * 3 + c];
    }
  }
  for (int col = 0; col < 3; ++col) {
    double y[3];
    for (int r = 0; r < 3; ++r) {
      double s = (piv[r] == col) ? 1.0 : 0.0;
      for (int j = 0; j < r; ++j) s -= lu[r * 3 + j] * y[j];
      y[r] = s;
    }
    double x[3];
    for (int r = 2; r >= 0; --r) {
      double s = y[r];
      for (int j = r + 1; j < 3; ++j) s -= lu[r * 3 + j] * x[j];
      x[r] = s / lu[r * 3 + r];
    }
    for (int r = 0; r < 3; ++r) inv[r * 3 + col] = x[r];
  }
}

// Eigen::AngleAxis::toRotationMatrix (Eigen/src/Geometry/AngleAxis.h); icp_fast.cc:310.
// R row-major 3x3.
inline void AngleAxisToRotation(double angle, const double axis[3], double* R) {
  const double s = std::sin(angle), c = std::cos(angle);
  const double sa[3] = {s * axis[0], s * axis[1], s * axis[2]};
  const double ca[3] = {(1.0 - c) * axis[0], (1.0 - c) * axis[1], (1.0 - c) * axis[2]};
  double tmp;
  tmp = ca[0] * axis[1]; R[0 * 3 + 1] = tmp - sa[2]; R[1 * 3 + 0] = tmp + sa[2];
  tmp = ca[0] * axis[2]; R[0 * 3 + 2] = tmp + sa[1]; R[2 * 3 + 0] = tmp - sa[1];
  tmp = ca[1] * axis[2]; R[1 * 3 + 2] = tmp - sa[0]; R[2 * 3 + 1] = tmp + sa[0];
  R[0] = ca[0] * axis[0] + c;
  R[4] = ca[1] * axis[1] + c;
  R[8] = ca[2] * axis[2] + c;
}

// Eigen::Quaternion(Matrix3) (Eigen/src/Geometry/Quaternion.h, quaternionbase_assign_impl);
// icp_fast.cc:514.  m row-major 3x3, q = (w, x, y, z).
inline void RotationToQuaternion(const double* m, double* q) {
  double t = m[0] + m[4] + m[8];
  if (t > 0.0) {
    t = std::sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (m[2 * 3 + 1] - m[1 * 3 + 2]) * t;
    q[2] = (m[0 * 3 + 2] - m[2 * 3 + 0]) * t;
    q[3] = (m[1 * 3 + 0] - m[0 * 3 + 1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[i * 3 + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = std::sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
    q[1 + i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t;
    q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
    q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
  }
}

// Eigen 3.3 QuaternionBase::angularDistance: d = a * conj(b); 2*atan2(|d.vec|, |d.w|).
// icp_fast.cc:391.
inline double QuaternionAngularDistance(const double* a, const double* b) {
  const double bw = b[0], bx = -b[1], by = -b[2], bz = -b[3];
  const double w = a[0] * bw - a[1] * bx - a[2] * by - a[3] * bz;
  const double x = a[0] * bx + a[1] * bw + a[2] * bz - a[3] * by;
  const double y = a[0] * by + a[2] * bw + a[3] * bx - a[1] * bz;
  const double z = a[0] * bz + a[3] * bw + a[1] * by - a[2] * bx;
  return 2.0 * std::atan2(std::sqrt(x * x + y * y + z * z), std::fabs(w));
}

}  // namespace sm_oracle

#endif  // ORACLE_LINALG_H_
