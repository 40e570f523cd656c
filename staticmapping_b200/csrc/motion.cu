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
#include "icp_dev.cuh"
#include "motion_dev.cuh"

namespace smb {
namespace {

// one point: InterpolateTransform(Identity, delta, factor) applied to (x, y, z), written as float
__host__ __device__ __forceinline__ void motion_point(const MotionParams& P, float x, float y, float z, float factor,
                                                      float* o) {
  double d[3];
  motion_point_d(P, x, y, z, factor, d);
  o[0] = (float)d[0]; o[1] = (float)d[1]; o[2] = (float)d[2];
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

// IcpFast with inner compensation (icp_fast.cc:487-488): step_cloud.ApplyMotionCompensation(T_iter) instead of
// ApplyTransform(T_iter).  Every source point gets its own InterpolateTransform(Identity, T_iter, f_i), f_i = i / N
// of its caller column i; the result stays in double.  T_iter lives in device state, so the quaternion, theta and
// sin(theta) are formed per CTA from it; the output is read by both the k-NN search (phase A) and phase B.
__global__ void __launch_bounds__(256)
icp_deskew_kernel(IcpBuffers b, IcpParams p, double* __restrict__ out) {
  __shared__ MotionParams P;
  if (b.state->done) return;
  if (threadIdx.x == 0) P = make_motion_params(b.state->T_iter);
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.n_source) return;
  const float factor = (float)source_factor(b.src_sort.vals[0][i], p.n_source);   // InterpolateTransform's float
  double o[3];
  motion_point_d(P, b.src0[i], b.src0[b.sstride + i], b.src0[2 * b.sstride + i], factor, o);
  out[i] = o[0]; out[b.sstride + i] = o[1]; out[2 * b.sstride + i] = o[2];
}

int run(const char* dev_in, char* dev_out, int64_t n, int64_t stride, const double* delta, int* dev_bad,
        cudaStream_t s) {
  const MotionParams P = make_motion_params(delta);
  SMB_CUDA_OK(cudaMemsetAsync(dev_bad, 0, sizeof(int), s));
  motion_compensation_kernel<<<ceil_div(n, 256), 256, 0, s>>>(dev_in, dev_out, stride, (int)n, P, dev_bad);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace

void icp_deskew_launch(const IcpBuffers& b, const IcpParams& p, double* out, cudaStream_t stream) {
  icp_deskew_kernel<<<ceil_div(p.n_source, 256), 256, 0, stream>>>(b, p, out);
}

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

// test hook (include/sm_b200_debug.h): make_motion_params + motion_point on the host, packed 5-float records
int sm_debug_motion_host(const float* points, int64_t n, const double* delta_4x4, float* out) {
  if (!points || !out || !delta_4x4 || n < 0) return SM_ERR_BAD_ARGUMENT;
  const MotionParams P = make_motion_params(delta_4x4);
  int bad = 0;
  for (int64_t i = 0; i < n; ++i) {
    const float* p = points + 5 * i;
    if (!(p[4] >= 0.f && p[4] <= 1.f)) bad = 1;
    motion_point(P, p[0], p[1], p[2], p[4], out + 5 * i);
    out[5 * i + 3] = p[3]; out[5 * i + 4] = p[4];
  }
  return bad ? SM_ERR_BAD_ARGUMENT : SM_OK;
}

// test hook (include/sm_b200_debug.h): the arithmetic of icp_deskew_kernel and of phase B's compensated match
// terms on the host
int sm_debug_inner_compensation_host(const double* T_iter_4x4, const double* points_3n, const double* targets_3n,
                                     const double* normals_3n, int64_t n, double* out_points_3n, double* out_terms_7n) {
  if (!T_iter_4x4 || !points_3n || n <= 0 || n > (1 << 30) || !out_points_3n) return SM_ERR_BAD_ARGUMENT;
  const MotionParams P = make_motion_params(T_iter_4x4);
  for (int64_t i = 0; i < n; ++i) {
    const double f = source_factor((uint32_t)i, (int)n);
    double* o = out_points_3n + 3 * i;
    motion_point_d(P, points_3n[3 * i], points_3n[3 * i + 1], points_3n[3 * i + 2], (float)f, o);
    if (!targets_3n || !normals_3n || !out_terms_7n) continue;
    BucketPoint q; BucketNormal nr;
    q.x = targets_3n[3 * i]; q.y = targets_3n[3 * i + 1]; q.z = targets_3n[3 * i + 2]; q.id = 0;
    nr.x = normals_3n[3 * i]; nr.y = normals_3n[3 * i + 1]; nr.z = normals_3n[3 * i + 2]; nr.pad = 0.0;
    dev::compensated_match_terms(o[0], o[1], o[2], q, nr, f, out_terms_7n + 7 * i, out_terms_7n[7 * i + 6]);
  }
  return SM_OK;
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
