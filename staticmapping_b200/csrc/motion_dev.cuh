// common::InterpolateTransform(Identity, T, factor) applied to one point (common/math.h:198-211), shared by
// the motion compensation either side of Align (motion.cu) and by IcpFast's in-loop compensation
// (icp_fast.cc:487-488, cloud_types.cc:306-318).  Host and device run the same code; its device users live in
// motion.cu, compiled with -fmad=false, so the operation order is the written one (the oracle's).
#ifndef SM_B200_MOTION_DEV_CUH_
#define SM_B200_MOTION_DEV_CUH_

#include <math.h>
#include <stdint.h>

namespace smb {

struct MotionParams {
  double qb[4];       // Quaternion(R_delta): w, x, y, z
  double t[3];        // translation of delta
  double d;           // dot(q_a, q_b) with q_a = identity
  double theta;       // acos(|d|)       (unused when lerp)
  double sin_theta;   // sin(theta)
  int lerp;           // |d| >= 1 - eps: Eigen falls back to linear weights
};

// Eigen::Quaternion(Matrix3) (quaternionbase_assign_impl); m column-major 4x4
__host__ __device__ __forceinline__ void rotation_to_quaternion(const double* T, double* q) {
  auto m = [&](int r, int c) { return T[r + 4 * c]; };
  double t = m(0, 0) + m(1, 1) + m(2, 2);
  if (t > 0.0) {
    t = sqrt(t + 1.0);
    q[0] = 0.5 * t;
    t = 0.5 / t;
    q[1] = (m(2, 1) - m(1, 2)) * t;
    q[2] = (m(0, 2) - m(2, 0)) * t;
    q[3] = (m(1, 0) - m(0, 1)) * t;
  } else {
    int i = 0;
    if (m(1, 1) > m(0, 0)) i = 1;
    if (m(2, 2) > m(i, i)) i = 2;
    const int j = (i + 1) % 3, k = (j + 1) % 3;
    t = sqrt(m(i, i) - m(j, j) - m(k, k) + 1.0);
    q[1 + i] = 0.5 * t;
    t = 0.5 / t;
    q[0] = (m(k, j) - m(j, k)) * t;
    q[1 + j] = (m(j, i) + m(i, j)) * t;
    q[1 + k] = (m(k, i) + m(i, k)) * t;
  }
}

// everything of the interpolation that does not depend on the point, computed exactly like Eigen 3.3's slerp
__host__ __device__ __forceinline__ MotionParams make_motion_params(const double* delta) {
  MotionParams P;
  rotation_to_quaternion(delta, P.qb);
  for (int k = 0; k < 3; ++k) P.t[k] = delta[12 + k];
  // q_a = Quaternion(Identity) = (1, 0, 0, 0); coeffs dot product in Eigen's (x, y, z, w) order
  P.d = ((0.0 * P.qb[1] + 0.0 * P.qb[2]) + 0.0 * P.qb[3]) + 1.0 * P.qb[0];
  const double one = 1.0 - 2.220446049250313e-16;
  const double abs_d = fabs(P.d);
  P.lerp = abs_d >= one ? 1 : 0;
  P.theta = P.lerp ? 0.0 : acos(abs_d);
  P.sin_theta = P.lerp ? 1.0 : sin(P.theta);
  return P;
}

// InterpolateTransform(Identity, delta, factor) applied to (x, y, z) (float or double), in double
template <typename Coord>
__host__ __device__ __forceinline__ void motion_point_d(const MotionParams& P, Coord x, Coord y, Coord z, float factor,
                                                        double* o) {
  const double t = (double)factor;
  double scale0, scale1;
  if (P.lerp) {
    scale0 = 1.0 - t; scale1 = t;
  } else {
    scale0 = sin((1.0 - t) * P.theta) / P.sin_theta;
    scale1 = sin(t * P.theta) / P.sin_theta;
  }
  if (P.d < 0.0) scale1 = -scale1;
  // coeffs = scale0 * q_a + scale1 * q_b with q_a = (1, 0, 0, 0)
  const double qw = scale0 * 1.0 + scale1 * P.qb[0];
  const double qx = scale0 * 0.0 + scale1 * P.qb[1];
  const double qy = scale0 * 0.0 + scale1 * P.qb[2];
  const double qz = scale0 * 0.0 + scale1 * P.qb[3];
  // QuaternionBase::toRotationMatrix (no normalisation, like Eigen)
  const double tx = 2.0 * qx, ty = 2.0 * qy, tz = 2.0 * qz;
  const double twx = tx * qw, twy = ty * qw, twz = tz * qw;
  const double txx = tx * qx, txy = ty * qx, txz = tz * qx;
  const double tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
  const double r00 = 1.0 - (tyy + tzz), r01 = txy - twz, r02 = txz + twy;
  const double r10 = txy + twz, r11 = 1.0 - (txx + tzz), r12 = tyz - twx;
  const double r20 = txz - twy, r21 = tyz + twx, r22 = 1.0 - (txx + tyy);
  const double px = (double)x, py = (double)y, pz = (double)z;
  o[0] = ((r00 * px + r01 * py) + r02 * pz) + P.t[0] * t;
  o[1] = ((r10 * px + r11 * py) + r12 * pz) + P.t[1] * t;
  o[2] = ((r20 * px + r21 * py) + r22 * pz) + P.t[2] * t;
}

// IcpFast's in-loop factor of the source point at caller column i (cloud_types.cc:340-344): i / N in double
__host__ __device__ __forceinline__ double source_factor(uint32_t i, int n) { return (double)i / (double)n; }

}  // namespace smb

#endif  // SM_B200_MOTION_DEV_CUH_
