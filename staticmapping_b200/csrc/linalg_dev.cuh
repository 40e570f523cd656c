// Device-side 6x6 / 3x3 dense algebra used by the ICP finish step and by target prep.
// Follows the Eigen 3.3 routines the reference calls (FullPivHouseholderQR::rank /
// isInvertible, LLT::solve, JacobiSVD::solve on the symmetric normal matrix,
// PartialPivLU::inverse, AngleAxis::toRotationMatrix, Quaternion(Matrix3),
// angularDistance) — call sites: registrators/icp_fast.cc:204-254,307-321,377-405 and
// builder/data/cloud_types.cc:89-93.  Row-major m[r*N+c] unless noted.
#ifndef SM_B200_LINALG_DEV_CUH_
#define SM_B200_LINALG_DEV_CUH_

#include <float.h>

namespace smb {
namespace la {

constexpr double kEps = 2.220446049250313e-16;

template <int N>
struct PivQR {
  double R[N * N];
  double Qt[N * N];
  int perm[N];
  int nonzero_pivots;
  double maxpivot;

  __host__ __device__ void compute(const double* A) {
    const double precision = kEps * (double)N;
    for (int i = 0; i < N * N; ++i) { R[i] = A[i]; Qt[i] = 0.0; }
    for (int i = 0; i < N; ++i) { Qt[i * N + i] = 1.0; perm[i] = i; }
    nonzero_pivots = N;
    maxpivot = 0.0;
    double biggest = 0.0;
    for (int k = 0; k < N; ++k) {
      int rb = k, cb = k;
      double best = -1.0;
      for (int c = k; c < N; ++c)        // column-major visit, strict '>' (Eigen maxCoeff)
        for (int r = k; r < N; ++r) {
          const double v = fabs(R[r * N + c]);
          if (v > best) { best = v; rb = r; cb = c; }
        }
      if (k == 0) biggest = best;
      if (fabs(best) <= fabs(biggest) * precision) { nonzero_pivots = k; break; }
      if (rb != k)
        for (int c = 0; c < N; ++c) {
          double t = R[k * N + c]; R[k * N + c] = R[rb * N + c]; R[rb * N + c] = t;
          t = Qt[k * N + c]; Qt[k * N + c] = Qt[rb * N + c]; Qt[rb * N + c] = t;
        }
      if (cb != k) {
        for (int r = 0; r < N; ++r) {
          const double t = R[r * N + k]; R[r * N + k] = R[r * N + cb]; R[r * N + cb] = t;
        }
        const int t = perm[k]; perm[k] = perm[cb]; perm[cb] = t;
      }
      double tail_sq = 0.0;
      for (int r = k + 1; r < N; ++r) tail_sq += R[r * N + k] * R[r * N + k];
      const double c0 = R[k * N + k];
      double beta, tau, v[N];
      for (int r = 0; r < N; ++r) v[r] = 0.0;
      if (tail_sq <= DBL_MIN) { tau = 0.0; beta = c0; }
      else {
        beta = sqrt(c0 * c0 + tail_sq);
        if (c0 >= 0.0) beta = -beta;
        for (int r = k + 1; r < N; ++r) v[r] = R[r * N + k] / (c0 - beta);
        tau = (beta - c0) / beta;
      }
      v[k] = 1.0;
      if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
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
  __host__ __device__ int rank() const {
    const double thr = fabs(maxpivot) * (kEps * (double)N);
    int rk = 0;
    for (int i = 0; i < nonzero_pivots; ++i) rk += (fabs(R[i * N + i]) > thr) ? 1 : 0;
    return rk;
  }
};

// Cholesky solve, n <= 6
__host__ __device__ inline void llt_solve(const double* A, const double* b, double* x, int n) {
  double L[36];
  for (int i = 0; i < n * n; ++i) L[i] = 0.0;
  for (int k = 0; k < n; ++k) {
    double d = A[k * n + k];
    for (int j = 0; j < k; ++j) d -= L[k * n + j] * L[k * n + j];
    const double lkk = sqrt(d);
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
}

// symmetric Jacobi eigen-decomposition, n <= 6 (V columns = eigenvectors)
__host__ __device__ inline void jacobi_eig_sym(const double* Ain, int n, double* w, double* V) {
  double A[36];
  for (int i = 0; i < n * n; ++i) { A[i] = Ain[i]; V[i] = 0.0; }
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
        const double theta = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = A[k * n + p], akq = A[k * n + q];
          A[k * n + p] = c * akp - s * akq; A[k * n + q] = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = A[p * n + k], aqk = A[q * n + k];
          A[p * n + k] = c * apk - s * aqk; A[q * n + k] = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vkp = V[k * n + p], vkq = V[k * n + q];
          V[k * n + p] = c * vkp - s * vkq; V[k * n + q] = s * vkp + c * vkq;
        }
      }
  }
  for (int i = 0; i < n; ++i) w[i] = A[i * n + i];
}

__host__ __device__ inline void sym_svd_solve(const double* A, const double* b, double* x, int n) {
  double w[6], V[36];
  jacobi_eig_sym(A, n, w, V);
  double svmax = 0.0;
  for (int i = 0; i < n; ++i) svmax = fmax(svmax, fabs(w[i]));
  const double thr = fmax(svmax * (double)n * kEps, DBL_MIN);
  for (int i = 0; i < n; ++i) x[i] = 0.0;
  for (int k = 0; k < n; ++k) {
    if (!(fabs(w[k]) > thr)) continue;
    double dot = 0.0;
    for (int i = 0; i < n; ++i) dot += V[i * n + k] * b[i];
    dot /= w[k];
    for (int i = 0; i < n; ++i) x[i] += V[i * n + k] * dot;
  }
}

// icp_fast.cc:204-254.  path: 0 LLT, 1 rank-reduced min-norm, 2 SVD fallback.
__host__ __device__ inline int solve_possibly_underdetermined(const double* A, const double* b, double* x) {
  PivQR<6> qr;
  qr.compute(A);
  const int rank = qr.rank();
  if (rank == 6) { llt_solve(A, b, x, 6); return 0; }
  double QA[36], R1[36], Qb[6], G[36], y[6], xp[6];
  for (int r = 0; r < rank; ++r)
    for (int k = 0; k < 6; ++k) {
      double s = 0.0;
      for (int m = 0; m < 6; ++m) s += qr.Qt[r * 6 + m] * A[m * 6 + k];
      QA[r * 6 + k] = s;
    }
  for (int r = 0; r < rank; ++r) {
    for (int c = 0; c < 6; ++c) R1[r * 6 + c] = QA[r * 6 + qr.perm[c]];
    double s = 0.0;
    for (int m = 0; m < 6; ++m) s += qr.Qt[r * 6 + m] * b[m];
    Qb[r] = s;
  }
  for (int r = 0; r < rank; ++r)
    for (int c = 0; c < rank; ++c) {
      double s = 0.0;
      for (int k = 0; k < 6; ++k) s += R1[r * 6 + k] * R1[c * 6 + k];
      G[r * rank + c] = s;
    }
  for (int i = 0; i < 6; ++i) { y[i] = 0.0; xp[i] = 0.0; x[i] = 0.0; }
  if (rank > 0) llt_solve(G, Qb, y, rank);
  for (int c = 0; c < 6; ++c)
    for (int r = 0; r < rank; ++r)
      if (c >= r) xp[c] += R1[r * 6 + c] * y[r];
  for (int j = 0; j < 6; ++j) x[qr.perm[j]] = xp[j];
  double nb = 0.0, nax = 0.0, nd = 0.0;
  for (int r = 0; r < 6; ++r) {
    double ax = 0.0;
    for (int c = 0; c < 6; ++c) ax += A[r * 6 + c] * x[c];
    nb += b[r] * b[r]; nax += ax * ax; nd += (b[r] - ax) * (b[r] - ax);
  }
  if (!(nd <= 1e-10 * fmin(nb, nax))) { sym_svd_solve(A, b, x, 6); return 2; }
  return 1;
}

// 3x3 inverse via partial-pivot LU (dynamic MatrixXd::inverse path, cloud_types.cc:93)
__host__ __device__ inline void lu_inverse3(const double* M, double* inv) {
  double lu[9];
  int piv[3] = {0, 1, 2};
  for (int i = 0; i < 9; ++i) lu[i] = M[i];
  for (int k = 0; k < 3; ++k) {
    int rb = k;
    double best = fabs(lu[k * 3 + k]);
    for (int r = k + 1; r < 3; ++r)
      if (fabs(lu[r * 3 + k]) > best) { best = fabs(lu[r * 3 + k]); rb = r; }
    if (rb != k) {
      for (int c = 0; c < 3; ++c) { const double t = lu[k * 3 + c]; lu[k * 3 + c] = lu[rb * 3 + c]; lu[rb * 3 + c] = t; }
      const int t = piv[k]; piv[k] = piv[rb]; piv[rb] = t;
    }
    for (int r = k + 1; r < 3; ++r) {
      lu[r * 3 + k] /= lu[k * 3 + k];
      for (int c = k + 1; c < 3; ++c) lu[r * 3 + c] -= lu[r * 3 + k] * lu[k * 3 + c];
    }
  }
  for (int col = 0; col < 3; ++col) {
    double y[3], x[3];
    for (int r = 0; r < 3; ++r) {
      double s = (piv[r] == col) ? 1.0 : 0.0;
      for (int j = 0; j < r; ++j) s -= lu[r * 3 + j] * y[j];
      y[r] = s;
    }
    for (int r = 2; r >= 0; --r) {
      double s = y[r];
      for (int j = r + 1; j < 3; ++j) s -= lu[r * 3 + j] * x[j];
      x[r] = s / lu[r * 3 + r];
    }
    for (int r = 0; r < 3; ++r) inv[r * 3 + col] = x[r];
  }
}

__host__ __device__ inline void angle_axis_to_rotation(double angle, const double* axis, double* R) {
  double s, c;
  sincos(angle, &s, &c);
  const double sa0 = s * axis[0], sa1 = s * axis[1], sa2 = s * axis[2];
  const double ca0 = (1.0 - c) * axis[0], ca1 = (1.0 - c) * axis[1], ca2 = (1.0 - c) * axis[2];
  double t;
  t = ca0 * axis[1]; R[1] = t - sa2; R[3] = t + sa2;
  t = ca0 * axis[2]; R[2] = t + sa1; R[6] = t - sa1;
  t = ca1 * axis[2]; R[5] = t - sa0; R[7] = t + sa0;
  R[0] = ca0 * axis[0] + c; R[4] = ca1 * axis[1] + c; R[8] = ca2 * axis[2] + c;
}

__host__ __device__ inline void rotation_to_quaternion(const double* m, double* q) {
  double t = m[0] + m[4] + m[8];
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[0] = 0.5 * t; t = 0.5 / t;
    q[1] = (m[7] - m[5]) * t; q[2] = (m[2] - m[6]) * t; q[3] = (m[3] - m[1]) * t;
  } else {
    int i = 0;
    if (m[4] > m[0]) i = 1;
    if (m[8] > m[i * 3 + i]) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m[i * 3 + i] - m[j * 3 + j] - m[k * 3 + k] + 1.0);
    q[1 + i] = 0.5 * t; t = 0.5 / t;
    q[0] = (m[k * 3 + j] - m[j * 3 + k]) * t;
    q[1 + j] = (m[j * 3 + i] + m[i * 3 + j]) * t;
    q[1 + k] = (m[k * 3 + i] + m[i * 3 + k]) * t;
  }
}

__host__ __device__ inline double quaternion_angular_distance(const double* a, const double* b) {
  const double bw = b[0], bx = -b[1], by = -b[2], bz = -b[3];
  const double w = a[0] * bw - a[1] * bx - a[2] * by - a[3] * bz;
  const double x = a[0] * bx + a[1] * bw + a[2] * bz - a[3] * by;
  const double y = a[0] * by + a[2] * bw + a[3] * bx - a[1] * bz;
  const double z = a[0] * bz + a[3] * bw + a[1] * by - a[2] * bx;
  return 2.0 * atan2(sqrt(x * x + y * y + z * z), fabs(w));
}

// a * b, a + b and a - b rounded on their own: never contracted into an FMA, on the device or the host.  The point-to-
// point solve below is written with them only (division and sqrt are correctly rounded on both), so the device build
// inside icp_finish.o (which contracts elsewhere) and the host build give the same bits.
__host__ __device__ __forceinline__ double mul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double add_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ double sub_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dsub_rn(a, b);
#else
  return a - b;
#endif
}
// ((a0 b0 + a1 b1) + a2 b2), each operation rounded
__host__ __device__ __forceinline__ double dot3_rn(double a0, double a1, double a2, double b0, double b1, double b2) {
  return add_rn(add_rn(mul_rn(a0, b0), mul_rn(a1, b1)), mul_rn(a2, b2));
}
// a0 b0 - a1 b1, each operation rounded
__host__ __device__ __forceinline__ double cross_rn(double a0, double b0, double a1, double b1) {
  return sub_rn(mul_rn(a0, b0), mul_rn(a1, b1));
}

// The rotation of ComputePointToPoint (icp_fast.cc:353-367) for M = sum (q - qbar)(p - pbar)^T, row-major.
// M = U S V^T by one-sided Jacobi (Hestenes) on the columns of M, accumulated into V, singular values sorted
// descending (a stable sort: equal values keep their column order).  u_k = column k / s_k while
// s_k > 8 eps s_0; the other columns of U complete a right-handed orthonormal basis: u3 = u1 x u2, and at rank 1
// u2 = normalize(u1 x e_m) with e_m the axis u1 leans on least (the first of equals).  M = 0 gives U = V = I, so R = I.
// R = U V^T; if det R < 0 the column of V of the smallest singular value is negated (the last row of V^T) and
// R = U V^T again.  Returns 1 when that reflection fix ran.  Every array index is a constant once the loops are
// unrolled, so the device keeps it all in registers; every operation is rounded on its own (see mul_rn).
__host__ __device__ __forceinline__ int kabsch_rotation(const double* M, double* R) {
  double A[9], V[9], U[9], s[3];
#pragma unroll
  for (int i = 0; i < 9; ++i) { A[i] = M[i]; V[i] = (i % 4 == 0) ? 1.0 : 0.0; }
#pragma unroll 1
  for (int sweep = 0; sweep < 32; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;     // (0,1), (0,2), (1,2)
      const double alpha = dot3_rn(A[p], A[3 + p], A[6 + p], A[p], A[3 + p], A[6 + p]);
      const double beta = dot3_rn(A[q], A[3 + q], A[6 + q], A[q], A[3 + q], A[6 + q]);
      const double gamma = dot3_rn(A[p], A[3 + p], A[6 + p], A[q], A[3 + q], A[6 + q]);
      if (!(fabs(gamma) > mul_rn(mul_rn(kEps, sqrt(alpha)), sqrt(beta)))) continue;   // orthogonal to working precision
      rotated = true;
      const double zeta = sub_rn(beta, alpha) / mul_rn(2.0, gamma);
      const double t = (zeta >= 0.0 ? 1.0 : -1.0) / add_rn(fabs(zeta), sqrt(add_rn(1.0, mul_rn(zeta, zeta))));
      const double c = 1.0 / sqrt(add_rn(1.0, mul_rn(t, t))), sn = mul_rn(c, t);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double ap = A[k * 3 + p], aq = A[k * 3 + q];
        A[k * 3 + p] = cross_rn(c, ap, sn, aq); A[k * 3 + q] = add_rn(mul_rn(sn, ap), mul_rn(c, aq));
        const double vp = V[k * 3 + p], vq = V[k * 3 + q];
        V[k * 3 + p] = cross_rn(c, vp, sn, vq); V[k * 3 + q] = add_rn(mul_rn(sn, vp), mul_rn(c, vq));
      }
    }
    if (!rotated) break;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) s[k] = sqrt(dot3_rn(A[k], A[3 + k], A[6 + k], A[k], A[3 + k], A[6 + k]));
#pragma unroll
  for (int pq = 0; pq < 3; ++pq) {                        // bubble sort, descending: (0,1), (1,2), (0,1)
    const int p = pq == 1 ? 1 : 0, q = p + 1;
    if (s[p] < s[q]) {
      const double ts = s[p]; s[p] = s[q]; s[q] = ts;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        double x = A[k * 3 + p]; A[k * 3 + p] = A[k * 3 + q]; A[k * 3 + q] = x;
        x = V[k * 3 + p]; V[k * 3 + p] = V[k * 3 + q]; V[k * 3 + q] = x;
      }
    }
  }
  const double tol = mul_rn(8.0 * kEps, s[0]);
  const int rank = (s[0] > 0.0 ? 1 : 0) + (s[1] > tol ? 1 : 0) + (s[2] > tol ? 1 : 0);
#pragma unroll
  for (int i = 0; i < 9; ++i) U[i] = (i % 4 == 0) ? 1.0 : 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k)
    if (k < rank) {
#pragma unroll
      for (int r = 0; r < 3; ++r) U[r * 3 + k] = A[r * 3 + k] / s[k];
    }
  if (rank == 1) {
    const double a0 = fabs(U[0]), a1 = fabs(U[3]), a2 = fabs(U[6]);
    const int m = (a0 <= a1 && a0 <= a2) ? 0 : (a1 <= a2 ? 1 : 2);
    const double e0 = m == 0 ? 1.0 : 0.0, e1 = m == 1 ? 1.0 : 0.0, e2 = m == 2 ? 1.0 : 0.0;
    const double w0 = cross_rn(U[3], e2, U[6], e1), w1 = cross_rn(U[6], e0, U[0], e2),
                 w2 = cross_rn(U[0], e1, U[3], e0);   // u1 x e_m
    const double nw = sqrt(dot3_rn(w0, w1, w2, w0, w1, w2));
    U[1] = w0 / nw; U[4] = w1 / nw; U[7] = w2 / nw;
  }
  if (rank == 1 || rank == 2) {
    U[2] = cross_rn(U[3], U[7], U[6], U[4]);
    U[5] = cross_rn(U[6], U[1], U[0], U[7]);
    U[8] = cross_rn(U[0], U[4], U[3], U[1]);
  }
  int fix = 0;
#pragma unroll 1
  for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) R[r * 3 + c] = dot3_rn(U[r * 3], U[r * 3 + 1], U[r * 3 + 2], V[c * 3], V[c * 3 + 1], V[c * 3 + 2]);
    const double det = add_rn(sub_rn(mul_rn(R[0], cross_rn(R[4], R[8], R[5], R[7])),
                                      mul_rn(R[1], cross_rn(R[3], R[8], R[5], R[6]))),
                              mul_rn(R[2], cross_rn(R[3], R[7], R[4], R[6])));
    if (pass == 1 || !(det < 0.0)) break;
    fix = 1;
    V[2] = -V[2]; V[5] = -V[5]; V[8] = -V[8];
  }
  return fix;
}

// Number of sums of one point-to-point match record.  S[0..2] = sum p, S[3..5] = sum q, S[6 + 3i + j] =
// sum q_i p_j (all about the origin of the target-mean frame), S[27] = sum sqrt(d2), S[28] = count; the rest is 0.
// The centring (icp_fast.cc:337-350) as one sweep: pbar = S[0..2] / n, qbar = S[3..5] / n,
// M_ij = S[6+3i+j] - S[3+i] * pbar_j (one rounding each: one kept match gives M = 0 exactly), then
// R = kabsch_rotation(M) and t = qbar - R pbar.  Returns the solve path: 3 Kabsch, 4 Kabsch with the reflection fix.
// Every operation is rounded on its own, so the device and the host give the same bits.
__host__ __device__ __forceinline__ int kabsch_from_sums(const double* S, double* R, double* t) {
  const double inv_n = 1.0 / S[28];
  double pm[3], qm[3], M[9];
#pragma unroll
  for (int i = 0; i < 3; ++i) { pm[i] = mul_rn(S[i], inv_n); qm[i] = mul_rn(S[3 + i], inv_n); }
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) M[i * 3 + j] = sub_rn(S[6 + 3 * i + j], mul_rn(S[3 + i], pm[j]));
  const int fix = kabsch_rotation(M, R);
#pragma unroll
  for (int i = 0; i < 3; ++i) t[i] = sub_rn(qm[i], dot3_rn(R[i * 3], R[i * 3 + 1], R[i * 3 + 2], pm[0], pm[1], pm[2]));
  return fix ? 4 : 3;
}

// column-major 4x4 product, k-order accumulation
__host__ __device__ inline void mul4(const double* A, const double* B, double* C) {
  double out[16];
  for (int j = 0; j < 4; ++j)
    for (int i = 0; i < 4; ++i) {
      double s = A[i] * B[j * 4];
      s += A[i + 4] * B[1 + j * 4];
      s += A[i + 8] * B[2 + j * 4];
      s += A[i + 12] * B[3 + j * 4];
      out[i + j * 4] = s;
    }
  for (int i = 0; i < 16; ++i) C[i] = out[i];
}

}  // namespace la
}  // namespace smb

#endif  // SM_B200_LINALG_DEV_CUH_
