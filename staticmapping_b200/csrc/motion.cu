// Motion compensation (de-skew) of a scan on the device: the per-point SE(3) interpolation the
// reference runs on the host either side of Align when
// front_end_options.motion_compensation_options.enable is set
// (builder/map_builder.cc:232-257 MotionCompensation, :320-352 the two call sites;
// common/math.h:198-211 InterpolateTransform).
//
// Per point the reference builds InterpolateTransform(Identity, delta, point.factor):
//   rotation    = Quaternion(Identity).slerp(factor, Quaternion(R_delta)).toRotationMatrix()
//   translation = 0 + (t_delta - 0) * factor
// and writes float(R * (x, y, z) + t), copying intensity and factor.  Everything that does not
// depend on the point (the two quaternions, their dot product, theta and sin(theta)) is computed
// once on the host exactly like Eigen 3.3's slerp does; the kernel evaluates the two sines, the
// blended quaternion, its rotation matrix and the point transform in double, one thread per
// point.  Compiled with -fmad=false so the operation order is the written one (the oracle's).
#include <math.h>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace smb {
namespace {

struct MotionParams {
  double qb[4];       // Quaternion(R_delta): w, x, y, z
  double t[3];        // translation of delta
  double d;           // dot(q_a, q_b) with q_a = identity
  double theta;       // acos(|d|)       (unused when lerp)
  double sin_theta;   // sin(theta)
  int lerp;           // |d| >= 1 - eps: Eigen falls back to linear weights
};

// one point: InterpolateTransform(Identity, delta, factor) applied to (x, y, z), written as float
__host__ __device__ __forceinline__ void motion_point(const MotionParams& P, float x, float y, float z, float factor,
                                                      float* o) {
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
  const double ox = ((r00 * px + r01 * py) + r02 * pz) + P.t[0] * t;
  const double oy = ((r10 * px + r11 * py) + r12 * pz) + P.t[1] * t;
  const double oz = ((r20 * px + r21 * py) + r22 * pz) + P.t[2] * t;
  o[0] = (float)ox; o[1] = (float)oy; o[2] = (float)oz;
}

__global__ void __launch_bounds__(256)
motion_compensation_kernel(const char* __restrict__ in, char* __restrict__ out, int64_t stride, int n,
                           MotionParams P, int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = reinterpret_cast<const float*>(in + (int64_t)i * stride);
  const float x = p[0], y = p[1], z = p[2], intensity = p[3], factor = p[4];
  // CHECK(factor >= 0. && factor <= 1.), common/math.h:201
  if (!(factor >= 0.f && factor <= 1.f)) atomicOr(bad, 1);
  float* o = reinterpret_cast<float*>(out + (int64_t)i * stride);
  motion_point(P, x, y, z, factor, o);
  o[3] = intensity; o[4] = factor;
}

// Eigen::Quaternion(Matrix3) (quaternionbase_assign_impl); m column-major 4x4
void rotation_to_quaternion_host(const double* T, double* q) {
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

MotionParams make_params(const double* delta) {
  MotionParams P;
  rotation_to_quaternion_host(delta, P.qb);
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

int run(const char* dev_in, char* dev_out, int64_t n, int64_t stride, const double* delta, int* dev_bad,
        cudaStream_t s) {
  const MotionParams P = make_params(delta);
  SMB_CUDA_OK(cudaMemsetAsync(dev_bad, 0, sizeof(int), s));
  motion_compensation_kernel<<<ceil_div(n, 256), 256, 0, s>>>(dev_in, dev_out, stride, (int)n, P, dev_bad);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace smb

using namespace smb;

extern "C" {

int sm_motion_compensation_device(int device, const float* dev_points, int64_t n, int64_t stride_bytes,
                                  const double* delta_4x4, float* dev_out, void* cuda_stream) {
  if (!dev_points || !dev_out || !delta_4x4 || n < 0 || n > (1 << 30) || stride_bytes < 20 || stride_bytes % 4)
    return SM_ERR_BAD_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  SMB_CUDA_OK(cudaSetDevice(device));
  if (n == 0) return SM_OK;
  cudaStream_t s = (cudaStream_t)cuda_stream;
  DevBuf bad;
  SMB_RC(bad.reserve(sizeof(int)));
  SMB_RC(run((const char*)dev_points, (char*)dev_out, n, stride_bytes, delta_4x4, (int*)bad.p, s));
  int host_bad = 0;
  SMB_CUDA_OK(cudaMemcpyAsync(&host_bad, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return host_bad ? SM_ERR_BAD_ARGUMENT : SM_OK;
}

// test hook (include/sm_b200_debug.h): make_params + motion_point on the host, packed 5-float records
int sm_debug_motion_host(const float* points, int64_t n, const double* delta_4x4, float* out) {
  if (!points || !out || !delta_4x4 || n < 0) return SM_ERR_BAD_ARGUMENT;
  const MotionParams P = make_params(delta_4x4);
  int bad = 0;
  for (int64_t i = 0; i < n; ++i) {
    const float* p = points + 5 * i;
    if (!(p[4] >= 0.f && p[4] <= 1.f)) bad = 1;
    motion_point(P, p[0], p[1], p[2], p[4], out + 5 * i);
    out[5 * i + 3] = p[3]; out[5 * i + 4] = p[4];
  }
  return bad ? SM_ERR_BAD_ARGUMENT : SM_OK;
}

int sm_motion_compensation(int device, const float* points, int64_t n, int64_t stride_bytes,
                           const double* delta_4x4, float* out) {
  if (!points || !out || !delta_4x4 || n < 0 || n > (1 << 30) || stride_bytes < 20 || stride_bytes % 4)
    return SM_ERR_BAD_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  SMB_CUDA_OK(cudaSetDevice(device));
  if (n == 0) return SM_OK;
  const size_t bytes = (size_t)n * (size_t)stride_bytes;
  DevBuf din, dout;
  SMB_RC(din.reserve(bytes));
  SMB_RC(dout.reserve(bytes));
  SMB_CUDA_OK(cudaMemcpy(din.p, points, bytes, cudaMemcpyHostToDevice));
  // bytes between the points (stride > 20) travel unchanged
  if (stride_bytes > 20) SMB_CUDA_OK(cudaMemcpy(dout.p, din.p, bytes, cudaMemcpyDeviceToDevice));
  const int rc = sm_motion_compensation_device(device, (const float*)din.p, n, stride_bytes, delta_4x4, (float*)dout.p, nullptr);
  if (rc != SM_OK && rc != SM_ERR_BAD_ARGUMENT) return rc;
  SMB_CUDA_OK(cudaMemcpy(out, dout.p, bytes, cudaMemcpyDeviceToHost));   // also for a bad time factor
  return rc;
}

}  // extern "C"
