// The arithmetic of pcl::registration::LUM (PCL 1.8.1, lum.hpp) and of the two PCL helpers it calls, shared by the
// device build (lum.cu, -fmad=false) and the host steps of MultiviewRegistratorLumPcl, and by the oracle
// (oracle/lum_oracle.cc), which runs the host steps in float (PCL's Eigen::MatrixXf / Vector6f, literal mode) or as
// the product runs them (double).  PCL is not compiled here: everything below is restated from upstream PCL 1.8.1 and
// Eigen 3.3 and is to be re-verified if their source becomes available.
//
//   pose         Vector6f (x, y, z, roll, pitch, yaw); pcl::getTransformation gives the affine 3x4 in float:
//                A = cos yaw, B = sin yaw, C = cos pitch, D = sin pitch, E = cos roll, F = sin roll, DE = D*E, DF = D*F,
//                rows [A*C, A*DF - B*E, B*F + A*DE, x], [B*C, A*E + B*DF, B*DE - A*F, y], [-D, C*F, C*E, z].
//   transform    pcl::transformPointCloud's x' = ((m00*x + m01*y) + m02*z) + m03 in float, left to right; a point
//                with a non-finite coordinate is left as it is (the path PCL takes for a cloud that is not dense).
//   pair terms   computeEdge: s, t = the correspondence's points composed with their vertex poses, skipped unless all
//                six coordinates are finite; a = 0.5 * (s + t), d = s - t; the 15 float terms whose sums fill M'M and
//                M'Z (lum_pair_terms) and, once D is known, the float s^2 term (lum_ss_term).
//   edge solve   D = M'M^-1 M'Z (Eigen's 6x6 inverse: PartialPivLU), s^2 < 1e-13 or non-finite -> cinv = cinvd = 0,
//                else cinv = M'M * (1 / s^2), cinvd = M'Z * (1 / s^2) in float.
//   compute      G (6(n-1) square) and B from the forward edge (vi, vj) or else the backward one with B's sign
//                flipped, vertex 0 fixed; X = G.colPivHouseholderQr().solve(B); pose += -incidenceCorrection(pose)^-1
//                X_vi; converged when the sum of the pose changes' norms <= 0.001f * (n - 1) in float.
#ifndef SM_B200_LUM_HOST_H_
#define SM_B200_LUM_HOST_H_

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define LUM_HD __host__ __device__
#else
#define LUM_HD
#endif

#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

namespace smb {

constexpr int kLumRounds = 5;                  // max_iteration_num_ of the reference (rounds of AlignAll)
constexpr int kLumIterations = 5;              // lum_.setMaxIterations(5)
constexpr float kLumConvergence = 0.001f;       // lum_.setConvergenceThreshold(0.001), a float member
constexpr float kLumMaxDistance = 0.25f;       // determineCorrespondences(*corr, 0.25)
constexpr int kLumTerms = 15;                  // the float terms of one pair summed into M'M and M'Z
// The correspondence search of one AlignAll holds 16 bytes per (pair, query point): the per-query match and the
// compacted lists.  Its queries, the sum over pairs (j, i), j < i, of frame j's points, are capped at 2^28 (4.3 GB).
constexpr int64_t kLumMaxQueries = (int64_t)1 << 28;

// the queries of AlignAll over frames of counts[0..n)
inline int64_t lum_queries(const int64_t* counts, int n) {
  int64_t q = 0;
  for (int j = 0; j < n; ++j) q += counts[j] * (int64_t)(n - 1 - j);
  return q;
}

LUM_HD inline bool lum_finite3(const float* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }

// pcl::getTransformation(x, y, z, roll, pitch, yaw) as a row-major 3x4 (host only: cosf / sinf of the host libm)
inline void lum_pose_matrix(const float* pose, float* T) {
  const float A = cosf(pose[5]), B = sinf(pose[5]), C = cosf(pose[4]), D = sinf(pose[4]), E = cosf(pose[3]),
              F = sinf(pose[3]), DE = D * E, DF = D * F;
  T[0] = A * C; T[1] = A * DF - B * E; T[2] = B * F + A * DE; T[3] = pose[0];
  T[4] = B * C; T[5] = A * E + B * DF; T[6] = B * DE - A * F; T[7] = pose[1];
  T[8] = -D;    T[9] = C * F;          T[10] = C * E;         T[11] = pose[2];
}

// a column-major Matrix4f as the row-major 3x4 that transformPointCloud reads
inline void lum_matrix4_to_3x4(const float* M, float* T) {
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) T[r * 4 + c] = M[c * 4 + r];
}

// LUM::incidenceCorrection, row-major 6x6 in float
inline void lum_incidence(const float* pose, float* J) {
  for (int i = 0; i < 36; ++i) J[i] = (i % 7 == 0) ? 1.f : 0.f;
  const float cx = cosf(pose[3]), sx = sinf(pose[3]), cy = cosf(pose[4]), sy = sinf(pose[4]);
  J[0 * 6 + 4] = pose[1] * sx - pose[2] * cx;
  J[0 * 6 + 5] = pose[1] * cx * cy + pose[2] * sx * cy;
  J[1 * 6 + 3] = pose[2];
  J[1 * 6 + 4] = -pose[0] * sx;
  J[1 * 6 + 5] = -pose[0] * cx * cy + pose[2] * sy;
  J[2 * 6 + 3] = -pose[1];
  J[2 * 6 + 4] = pose[0] * cx;
  J[2 * 6 + 5] = -pose[0] * sx * cy - pose[1] * sy;
  J[3 * 6 + 5] = sy;
  J[4 * 6 + 4] = sx;
  J[4 * 6 + 5] = cx * cy;
  J[5 * 6 + 4] = cx;
  J[5 * 6 + 5] = -sx * cy;
}

// x' = T p, left to right in float; a point with a non-finite coordinate is copied
LUM_HD inline void lum_transform(const float* T, const float* p, float* out) {
  if (!lum_finite3(p)) { out[0] = p[0]; out[1] = p[1]; out[2] = p[2]; return; }
  for (int r = 0; r < 3; ++r) out[r] = ((T[r * 4] * p[0] + T[r * 4 + 1] * p[1]) + T[r * 4 + 2] * p[2]) + T[r * 4 + 3];
}

// Eigen's Affine3f * Vector3f (linear() * v + translation()), no finiteness test
LUM_HD inline void lum_compound(const float* T, const float* p, float* out) {
  for (int r = 0; r < 3; ++r) out[r] = ((T[r * 4] * p[0] + T[r * 4 + 1] * p[1]) + T[r * 4 + 2] * p[2]) + T[r * 4 + 3];
}

// the pair's average a and difference d; false when a compounded point is not finite (the pair is skipped)
LUM_HD inline bool lum_pair(const float* Ts, const float* Tt, const float* ps, const float* pt, float* a, float* d) {
  float s[3], t[3];
  lum_compound(Ts, ps, s);
  lum_compound(Tt, pt, t);
  if (!lum_finite3(s) || !lum_finite3(t)) return false;
  for (int k = 0; k < 3; ++k) { a[k] = 0.5f * (s[k] + t[k]); d[k] = s[k] - t[k]; }
  return true;
}

// the terms of computeEdge's M'M / M'Z loop: a0 a1 a2, a0a2 a0a1 a1a2, a1a1+a2a2 a0a0+a1a1 a0a0+a2a2, d0 d1 d2,
// a1d2-a2d1 a0d1-a1d0 a2d0-a0d2
LUM_HD inline void lum_pair_terms(const float* a, const float* d, float* t) {
  t[0] = a[0]; t[1] = a[1]; t[2] = a[2];
  t[3] = a[0] * a[2]; t[4] = a[0] * a[1]; t[5] = a[1] * a[2];
  t[6] = a[1] * a[1] + a[2] * a[2]; t[7] = a[0] * a[0] + a[1] * a[1]; t[8] = a[0] * a[0] + a[2] * a[2];
  t[9] = d[0]; t[10] = d[1]; t[11] = d[2];
  t[12] = a[1] * d[2] - a[2] * d[1]; t[13] = a[0] * d[1] - a[1] * d[0]; t[14] = a[2] * d[0] - a[0] * d[2];
}

// M'M (row-major) and M'Z from the 15 sums and the pair count
LUM_HD inline void lum_mm_mz(const float* S, int count, float* MM, float* MZ) {
  for (int i = 0; i < 36; ++i) MM[i] = 0.f;
  MM[0 * 6 + 4] = -S[1]; MM[0 * 6 + 5] = S[2]; MM[1 * 6 + 3] = -S[2]; MM[1 * 6 + 4] = S[0];
  MM[2 * 6 + 3] = S[1]; MM[2 * 6 + 5] = -S[0];
  MM[3 * 6 + 4] = -S[3]; MM[3 * 6 + 5] = -S[4]; MM[4 * 6 + 5] = -S[5];
  MM[3 * 6 + 3] = S[6]; MM[4 * 6 + 4] = S[7]; MM[5 * 6 + 5] = S[8];
  MM[0] = MM[7] = MM[14] = (float)count;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < r; ++c) MM[r * 6 + c] = MM[c * 6 + r];
  for (int k = 0; k < 6; ++k) MZ[k] = S[9 + k];
}

// computeEdge's s^2 term of one pair, in float: pow(x, 2.0f) as x * x
LUM_HD inline float lum_ss_term(const float* a, const float* d, const float* D) {
  const float r0 = d[0] - ((D[0] + a[2] * D[5]) - a[1] * D[4]);
  const float r1 = d[1] - ((D[1] + a[0] * D[4]) - a[2] * D[3]);
  const float r2 = d[2] - ((D[2] + a[1] * D[3]) - a[0] * D[5]);
  return (r0 * r0 + r1 * r1) + r2 * r2;
}

// Eigen's PartialPivLU inverse of an n x n (n <= 6) row-major matrix, restated serially: the first largest |pivot|,
// the column scaled by division, the rank-1 update, then the unit-lower and upper triangular solves of P I.
template <typename T>
LUM_HD inline void lum_lu_inverse(const T* A, int n, T* inv) {
  T lu[36];
  int perm[6];
  for (int i = 0; i < n * n; ++i) lu[i] = A[i];
  for (int i = 0; i < n; ++i) perm[i] = i;
  for (int k = 0; k < n; ++k) {
    int p = k;
    T big = fabs(lu[k * n + k]);
    for (int r = k + 1; r < n; ++r)
      if (fabs(lu[r * n + k]) > big) { big = fabs(lu[r * n + k]); p = r; }
    if (big != T(0)) {
      if (p != k) {
        for (int c = 0; c < n; ++c) { const T t = lu[k * n + c]; lu[k * n + c] = lu[p * n + c]; lu[p * n + c] = t; }
        const int t = perm[k]; perm[k] = perm[p]; perm[p] = t;
      }
      for (int r = k + 1; r < n; ++r) lu[r * n + k] = lu[r * n + k] / lu[k * n + k];
    }
    for (int r = k + 1; r < n; ++r)
      for (int c = k + 1; c < n; ++c) lu[r * n + c] = lu[r * n + c] - lu[r * n + k] * lu[k * n + c];
  }
  for (int e = 0; e < n; ++e) {
    T x[6];
    for (int r = 0; r < n; ++r) x[r] = perm[r] == e ? T(1) : T(0);
    for (int k = 0; k < n; ++k)
      for (int r = k + 1; r < n; ++r) x[r] = x[r] - x[k] * lu[r * n + k];
    for (int k = n - 1; k >= 0; --k) {
      x[k] = x[k] / lu[k * n + k];
      for (int r = 0; r < k; ++r) x[r] = x[r] - x[k] * lu[r * n + k];
    }
    for (int r = 0; r < n; ++r) inv[r * n + e] = x[r];
  }
}

// D = M'M^-1 M'Z with the inverse in T, rounded to float (Vector6f D)
template <typename T>
LUM_HD inline void lum_edge_d(const float* MM, const float* MZ, float* D) {
  T A[36], inv[36];
  for (int i = 0; i < 36; ++i) A[i] = (T)MM[i];
  lum_lu_inverse<T>(A, 6, inv);
  for (int r = 0; r < 6; ++r) {
    T s = T(0);
    for (int k = 0; k < 6; ++k) s = s + inv[r * 6 + k] * (T)MZ[k];
    D[r] = (float)s;
  }
}

// cinv / cinvd from M'M, M'Z and s^2; zero when s^2 < 1e-13 or not finite
LUM_HD inline void lum_edge_finish(const float* MM, const float* MZ, float ss, float* cinv, float* cinvd) {
  if ((double)ss < 0.0000000000001 || !isfinite(ss)) {
    for (int i = 0; i < 36; ++i) cinv[i] = 0.f;
    for (int i = 0; i < 6; ++i) cinvd[i] = 0.f;
    return;
  }
  const float s = 1.0f / ss;
  for (int i = 0; i < 36; ++i) cinv[i] = MM[i] * s;
  for (int i = 0; i < 6; ++i) cinvd[i] = MZ[i] * s;
}

// Eigen's ColPivHouseholderQR(A).solve(b) for a square m x m column-major A, restated with serial loops: column norms
// downdated and recomputed below sqrt(eps), the first largest norm as the pivot, m_nonzero_pivots set at the first
// squared norm below (max norm * eps)^2 / m * (m - k), Householder reflections as makeHouseholderInPlace, then
// Q^T b over the nonzero pivots, the upper triangular solve, zeros for the other components, and the permutation.
template <typename T>
void lum_colpiv_qr_solve(int m, std::vector<T> A, std::vector<T> b, std::vector<T>& x) {
  x.assign(m, T(0));
  if (m == 0) return;
  auto at = [&](int r, int c) -> T& { return A[(size_t)c * m + r]; };
  const T eps = std::numeric_limits<T>::epsilon();
  std::vector<T> upd(m), direct(m), hc(m);
  std::vector<int> perm(m);
  for (int c = 0; c < m; ++c) {
    T s = T(0);
    for (int r = 0; r < m; ++r) s = s + at(r, c) * at(r, c);
    upd[c] = direct[c] = std::sqrt(s);
    perm[c] = c;
  }
  T maxnorm = T(0);
  for (int c = 0; c < m; ++c) maxnorm = std::max(maxnorm, upd[c]);
  const T threshold_helper = (maxnorm * eps) * (maxnorm * eps) / (T)m;
  const T downdate_threshold = std::sqrt(eps);
  int nonzero = m;
  for (int k = 0; k < m; ++k) {
    int bc = k;
    for (int c = k + 1; c < m; ++c)
      if (upd[c] > upd[bc]) bc = c;
    const T big_sq = upd[bc] * upd[bc];
    if (nonzero == m && big_sq < threshold_helper * (T)(m - k)) nonzero = k;
    if (bc != k) {
      for (int r = 0; r < m; ++r) std::swap(at(r, k), at(r, bc));
      std::swap(upd[k], upd[bc]);
      std::swap(direct[k], direct[bc]);
      std::swap(perm[k], perm[bc]);
    }
    T tail = T(0);
    for (int r = k + 1; r < m; ++r) tail = tail + at(r, k) * at(r, k);
    const T c0 = at(k, k);
    T beta, tau;
    if (tail <= std::numeric_limits<T>::min()) {
      tau = T(0); beta = c0;
      for (int r = k + 1; r < m; ++r) at(r, k) = T(0);
    } else {
      beta = std::sqrt(c0 * c0 + tail);
      if (c0 >= T(0)) beta = -beta;
      for (int r = k + 1; r < m; ++r) at(r, k) = at(r, k) / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    hc[k] = tau;
    at(k, k) = beta;
    if (tau != T(0))
      for (int c = k + 1; c < m; ++c) {
        T dot = at(k, c);
        for (int r = k + 1; r < m; ++r) dot = dot + at(r, k) * at(r, c);
        at(k, c) = at(k, c) - tau * dot;
        for (int r = k + 1; r < m; ++r) at(r, c) = at(r, c) - (tau * at(r, k)) * dot;
      }
    for (int c = k + 1; c < m; ++c) {
      if (upd[c] == T(0)) continue;
      T t = std::fabs(at(k, c)) / upd[c];
      t = (T(1) + t) * (T(1) - t);
      if (t < T(0)) t = T(0);
      const T q = upd[c] / direct[c];
      const T t2 = t * (q * q);
      if (t2 <= downdate_threshold) {
        T s = T(0);
        for (int r = k + 1; r < m; ++r) s = s + at(r, c) * at(r, c);
        direct[c] = upd[c] = std::sqrt(s);
      } else {
        upd[c] = upd[c] * std::sqrt(t);
      }
    }
  }
  if (nonzero == 0) return;
  for (int k = 0; k < nonzero; ++k) {
    if (hc[k] == T(0)) continue;
    T dot = b[k];
    for (int r = k + 1; r < m; ++r) dot = dot + at(r, k) * b[r];
    b[k] = b[k] - hc[k] * dot;
    for (int r = k + 1; r < m; ++r) b[r] = b[r] - (hc[k] * at(r, k)) * dot;
  }
  for (int k = nonzero - 1; k >= 0; --k) {
    b[k] = b[k] / at(k, k);
    for (int r = 0; r < k; ++r) b[r] = b[r] - b[k] * at(r, k);
  }
  for (int i = 0; i < nonzero; ++i) x[perm[i]] = b[i];
}

struct LumEdge {
  int s, t;                 // source vertex j < target vertex i
  float cinv[36], cinvd[6];
};

// One LUM::compute iteration after computeEdge, over n >= 2 vertices: G and B in float as PCL fills them (vj ascending
// for each vi), then
//   T = float (literal): X over all 6(n-1) components in float; the update in float;
//   T = double (product): X over the vertices joined to vertex 0 by edges with a non-zero cinv, in double, zero for
//                         the others; the update in double, each pose rounded to float.
// poses: 6n floats, updated; X (optional): 6(n-1) values.  Returns the sum of the pose changes' norms.
template <typename T>
double lum_solve_update(int n, const std::vector<LumEdge>& edges, float* poses, std::vector<T>* X_out) {
  const bool literal = sizeof(T) == sizeof(float);
  struct Adj { int other, edge; bool forward; };
  std::vector<std::vector<Adj>> adj(n);
  for (size_t e = 0; e < edges.size(); ++e) {
    adj[edges[e].s].push_back({edges[e].t, (int)e, true});    // (vi = s, vj = t): the forward edge
    adj[edges[e].t].push_back({edges[e].s, (int)e, false});
  }
  for (auto& a : adj) std::sort(a.begin(), a.end(), [](const Adj& x, const Adj& y) { return x.other < y.other; });
  std::vector<int> slot(n, -1);   // the solved vertices' block index
  int k = 0;
  if (literal) {
    for (int v = 1; v < n; ++v) slot[v] = k++;
  } else {
    std::vector<char> joined(n, 0);
    std::vector<int> queue(1, 0);
    joined[0] = 1;
    for (size_t h = 0; h < queue.size(); ++h)
      for (const Adj& a : adj[queue[h]]) {
        bool live = false;
        for (int i = 0; i < 36 && !live; ++i) live = edges[a.edge].cinv[i] != 0.f;
        if (live && !joined[a.other]) { joined[a.other] = 1; queue.push_back(a.other); }
      }
    for (int v = 1; v < n; ++v)
      if (joined[v]) slot[v] = k++;
  }
  const int m = 6 * k;
  std::vector<float> G((size_t)m * m, 0.f), B(m, 0.f);   // G column-major
  for (int vi = 1; vi < n; ++vi) {
    if (slot[vi] < 0) continue;
    const int r0 = 6 * slot[vi];
    for (const Adj& a : adj[vi]) {
      const LumEdge& E = edges[a.edge];
      if (a.other > 0 && slot[a.other] >= 0)
        for (int r = 0; r < 6; ++r)
          for (int c = 0; c < 6; ++c) G[(size_t)(6 * slot[a.other] + c) * m + r0 + r] = -E.cinv[r * 6 + c];
      for (int r = 0; r < 6; ++r)
        for (int c = 0; c < 6; ++c) G[(size_t)(r0 + c) * m + r0 + r] += E.cinv[r * 6 + c];
      for (int r = 0; r < 6; ++r) B[r0 + r] += (a.forward ? 1.f : -1.f) * E.cinvd[r];
    }
  }
  std::vector<T> Xs, X((size_t)6 * (n - 1), T(0));
  lum_colpiv_qr_solve<T>(m, std::vector<T>(G.begin(), G.end()), std::vector<T>(B.begin(), B.end()), Xs);
  for (int v = 1; v < n; ++v)
    if (slot[v] >= 0)
      for (int c = 0; c < 6; ++c) X[6 * (v - 1) + c] = Xs[6 * slot[v] + c];
  T sum = T(0);
  for (int vi = 1; vi < n; ++vi) {
    float* pose = poses + 6 * vi;
    float Jf[36];
    lum_incidence(pose, Jf);
    T J[36], inv[36];
    for (int i = 0; i < 36; ++i) J[i] = (T)Jf[i];
    lum_lu_inverse<T>(J, 6, inv);
    T dp[6], sq = T(0);
    for (int r = 0; r < 6; ++r) {
      T s = T(0);
      for (int c = 0; c < 6; ++c) s = s + (-inv[r * 6 + c]) * X[6 * (vi - 1) + c];
      dp[r] = s;
      sq = sq + s * s;
    }
    sum = sum + std::sqrt(sq);
    for (int r = 0; r < 6; ++r) pose[r] = (float)((T)pose[r] + dp[r]);
  }
  if (X_out) *X_out = X;
  return (double)sum;
}

// the convergence test of LUM::compute, in float as PCL keeps it (convergence_threshold_ is a float, and so is the sum
// of the float mode; the double mode's sum is rounded to float first)
inline bool lum_converged(double sum, int n) { return (float)sum <= kLumConvergence * (float)(n - 1); }

}  // namespace smb

#endif  // SM_B200_LUM_HOST_H_
