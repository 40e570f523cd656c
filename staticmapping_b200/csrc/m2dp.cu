// descriptor::M2dp on the device (descriptor/m2dp.cc:37-172): the loop-closure descriptor the
// reference computes from every finished submap (builder/submap.cc; back_end/loop_detector.cc
// compares them with matchTwoM2dpDescriptors before it spends an Align on a candidate pair).
//
//   preProcess (:45-70)        pcl::PCA in single precision: centroid, covariance / (n - 1),
//                              axes by descending eigenvalue, third = first x second,
//                              projection eigenvectors^T (x - mean), gate ||.|| <= max_distance
//   singleViewProcess (:72-127) p*q = 64 views; per view and point two float dot products, their
//                              ABSOLUTE values (`(p^T axis).norm()` of a 1x1 product), a float
//                              norm, a float atan2, bins l = floor(sqrt(len / r)), t = floor(angle /
//                              step) in double
//   setInputCloud (:129-153)   A (64 x 512 counts), first singular vectors -> [u1; v1]
//
// H100 formulation: the work is N x 64 (point, view) bin updates — integer scatter, no
// contraction.  One CTA owns a chunk of points and a GROUP of 8 views whose 8 x 512 histogram
// lives in shared memory (16 KB): the point is loaded and projected once per CTA-thread, the
// eight views hit shared-memory atomics only (the reference's |.| folds everything into the first
// quadrant, so a view touches ~128 distinct bins: global atomics would serialise in L2), and the
// non-empty bins are flushed to the global matrix with one atomic each at the end.  Sums for the
// PCA are double block reductions.  A A^T (64 x 64, exact in double: counts < 2^31) is formed on the
// device; the two tiny eigenproblems run on the host by power iteration (an algorithm deliberately
// different from the oracle's Jacobi sweeps).  Sign conventions: see oracle/m2dp_oracle.cc — they
// live inside Eigen in the reference and are fixed the same way on both sides here.
#include <math.h>

#include <vector>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "kernels.h"

namespace smb {
namespace {

constexpr int kViewsPerCta = 8;
constexpr int kHistThreads = 256;
constexpr int kPointsPerCta = 4096;

struct M2dpView { float xa[3], ya[3]; };
struct M2dpParams {
  float mean[3];
  float E[9];             // E[k * 3 + j]: component k of axis j
  double r, max_distance, angle_step;
  int l, t, cols, n_views;
};

__global__ void __launch_bounds__(256)
m2dp_mean_kernel(const char* __restrict__ pts, int64_t stride, int64_t n, double* __restrict__ sums) {
  __shared__ double sm[3][8];
  double s[3] = {0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* p = reinterpret_cast<const float*>(pts + i * stride);
    s[0] += (double)p[0]; s[1] += (double)p[1]; s[2] += (double)p[2];
  }
  for (int d = 0; d < 3; ++d) {
    double v = s[d];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[d][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    double v = 0.0;
    for (int w = 0; w < 8; ++w) v += sm[threadIdx.x][w];
    atomicAdd(&sums[threadIdx.x], v);
  }
}

// covariance sums of the float-demeaned cloud (pcl::demeanPointCloud works in float)
__global__ void __launch_bounds__(256)
m2dp_cov_kernel(const char* __restrict__ pts, int64_t stride, int64_t n, float cx, float cy, float cz,
                double* __restrict__ sums) {
  __shared__ double sm[6][8];
  double s[6] = {0, 0, 0, 0, 0, 0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* p = reinterpret_cast<const float*>(pts + i * stride);
    const float x = p[0] - cx, y = p[1] - cy, z = p[2] - cz;
    s[0] += (double)(x * x); s[1] += (double)(x * y); s[2] += (double)(x * z);
    s[3] += (double)(y * y); s[4] += (double)(y * z); s[5] += (double)(z * z);
  }
  for (int d = 0; d < 6; ++d) {
    double v = s[d];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sm[d][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    double v = 0.0;
    for (int w = 0; w < 8; ++w) v += sm[threadIdx.x][w];
    atomicAdd(&sums[threadIdx.x], v);
  }
}

// grid: (point chunks, view groups).  Dynamic shared memory: kViewsPerCta * cols ints.
__global__ void __launch_bounds__(kHistThreads)
m2dp_hist_kernel(const char* __restrict__ pts, int64_t stride, int64_t n, M2dpParams P,
                 const M2dpView* __restrict__ views, int* __restrict__ A) {
  extern __shared__ int hist[];
  __shared__ M2dpView sv[kViewsPerCta];
  const int v0 = blockIdx.y * kViewsPerCta;
  const int nv = min(kViewsPerCta, P.n_views - v0);
  for (int k = threadIdx.x; k < kViewsPerCta * P.cols; k += kHistThreads) hist[k] = 0;
  if (threadIdx.x < nv) sv[threadIdx.x] = views[v0 + threadIdx.x];
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kPointsPerCta;
  const int64_t end = min(base + (int64_t)kPointsPerCta, n);
  const double two_pi = M_PI * 2.;
  for (int64_t i = base + threadIdx.x; i < end; i += kHistThreads) {
    const float* p = reinterpret_cast<const float*>(pts + i * stride);
    const float x = p[0] - P.mean[0], y = p[1] - P.mean[1], z = p[2] - P.mean[2];
    const float px = P.E[0] * x + P.E[3] * y + P.E[6] * z, py = P.E[1] * x + P.E[4] * y + P.E[7] * z,
                pz = P.E[2] * x + P.E[5] * y + P.E[8] * z;
    const double d = (double)sqrtf(px * px + py * py + pz * pz);      // getLength<PointXYZ> (m2dp.cc:32-35)
    if (!(d <= P.max_distance)) continue;
    for (int k = 0; k < nv; ++k) {
      const M2dpView& vw = sv[k];
      const float u = fabsf(px * vw.xa[0] + py * vw.xa[1] + pz * vw.xa[2]);
      const float v = fabsf(px * vw.ya[0] + py * vw.ya[1] + pz * vw.ya[2]);
      const double length = (double)sqrtf(u * u + v * v);
      double angle = (double)atan2f(v, u);
      if (angle < 0.) angle += two_pi;
      int li = (int)floor(sqrt(length / P.r));
      if (li > P.l - 1) li = P.l - 1;                                   // "avoid over border" (:111-117)
      int ti = (int)floor(angle / P.angle_step);
      if (ti > P.t - 1) ti = P.t - 1;
      if (li >= 0 && ti >= 0) atomicAdd(&hist[k * P.cols + li * P.t + ti], 1);   // NaN input lands nowhere
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < nv * P.cols; k += kHistThreads) {
    const int c = hist[k];
    if (c != 0) atomicAdd(&A[(int64_t)(v0 + k / P.cols) * P.cols + (k % P.cols)], c);
  }
}

// G = A A^T (rows x rows) in double; one block per (a, b-tile)
__global__ void __launch_bounds__(256)
m2dp_gram_kernel(const int* __restrict__ A, int rows, int cols, double* __restrict__ G) {
  __shared__ double red[8];
  const int a = blockIdx.x, b = blockIdx.y;
  if (b < a) return;
  double s = 0.0;
  for (int k = threadIdx.x; k < cols; k += 256) s += (double)A[(int64_t)a * cols + k] * (double)A[(int64_t)b * cols + k];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];        // integer-valued partial sums < 2^53: exact in any order
    G[(int64_t)a * rows + b] = t; G[(int64_t)b * rows + a] = t;
  }
}

// dominant eigenpair of a symmetric PSD matrix by power iteration (host, double)
double power_iteration(const std::vector<double>& M, int n, std::vector<double>& v) {
  v.assign((size_t)n, 1.0 / sqrt((double)n));
  for (int k = 0; k < n; ++k) v[(size_t)k] *= 1.0 + 1e-3 * k;      // not orthogonal to anything by accident
  std::vector<double> w((size_t)n);
  double lambda = 0.0;
  for (int it = 0; it < 20000; ++it) {
    double norm = 0.0;
    for (int i = 0; i < n; ++i) {
      double s = 0.0;
      for (int j = 0; j < n; ++j) s += M[(size_t)i * n + j] * v[(size_t)j];
      w[(size_t)i] = s; norm += s * s;
    }
    norm = sqrt(norm);
    if (!(norm > 0.0)) return 0.0;
    double diff = 0.0;
    for (int i = 0; i < n; ++i) { const double nv = w[(size_t)i] / norm; diff += fabs(nv - v[(size_t)i]); v[(size_t)i] = nv; }
    lambda = norm;
    if (diff < 1e-15 * n) break;
  }
  return lambda;
}

void orient(double* v, int n) {    // component of largest magnitude positive
  int big = 0;
  for (int k = 1; k < n; ++k) if (fabs(v[k]) > fabs(v[big])) big = k;
  if (v[big] < 0) for (int k = 0; k < n; ++k) v[k] = -v[k];
}

}  // namespace
}  // namespace smb

using namespace smb;

extern "C" int64_t sm_m2dp_descriptor_length(double r, double max_distance, int32_t t, int32_t p, int32_t q) {
  if (r < 1.e-6 || !(max_distance > 0.0) || t <= 0 || p <= 0 || q <= 0) return SM_ERR_BAD_ARGUMENT;
  const double l = ceil(sqrt(max_distance / r));
  if (!(l >= 1.0) || l * t > 8192.0 || (double)p * q > 4096.0) return SM_ERR_BAD_ARGUMENT;
  return (int64_t)p * q + (int64_t)l * t;
}

extern "C" int sm_m2dp(int device, const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance,
                       int32_t t, int32_t p, int32_t q, float* descriptor, int64_t capacity, int32_t* A_out) {
  if (!points || !descriptor || n < 0 || n > (1ll << 30) || stride_bytes < 12 || stride_bytes % 4) return SM_ERR_BAD_ARGUMENT;
  const int64_t len = sm_m2dp_descriptor_length(r, max_distance, t, p, q);
  if (len < 0 || capacity < len) return SM_ERR_BAD_ARGUMENT;        // "r is too small" (m2dp.cc:64-67)
  if (n == 0) return 0;                                             // "source is empty": setInputCloud returns false
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  SMB_CUDA_OK(cudaSetDevice(device));
  const int rows = p * q, l = (int)ceil(sqrt(max_distance / r)), cols = l * t;
  const size_t in_bytes = (size_t)n * (size_t)stride_bytes;
  const size_t bytes = in_bytes + 256 + 16 * sizeof(double) + (size_t)rows * sizeof(M2dpView) + 256 +
                       (size_t)rows * cols * sizeof(int) + 256 + (size_t)rows * rows * sizeof(double) + 256;
  DevBuf buf;
  SMB_RC(buf.reserve(bytes));
  char* cur = (char*)buf.p;
  auto take = [&](size_t b) { char* ptr = cur; cur += (b + 255) & ~(size_t)255; return ptr; };
  char* d_in = take(in_bytes);
  double* d_sums = (double*)take(16 * sizeof(double));
  M2dpView* d_views = (M2dpView*)take((size_t)rows * sizeof(M2dpView));
  int* d_A = (int*)take((size_t)rows * cols * sizeof(int));
  double* d_G = (double*)take((size_t)rows * rows * sizeof(double));
  cudaStream_t s = nullptr;
  SMB_CUDA_OK(cudaMemcpyAsync(d_in, points, in_bytes, cudaMemcpyHostToDevice, s));
  SMB_CUDA_OK(cudaMemsetAsync(d_sums, 0, 16 * sizeof(double), s));
  SMB_CUDA_OK(cudaMemsetAsync(d_A, 0, (size_t)rows * cols * sizeof(int), s));
  const int red_blocks = (int)std::min<int64_t>(4 * kNumSMs, (n + 255) / 256);
  m2dp_mean_kernel<<<red_blocks, 256, 0, s>>>(d_in, stride_bytes, n, d_sums);
  double h[16];
  SMB_CUDA_OK(cudaMemcpyAsync(h, d_sums, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  M2dpParams P;
  for (int d = 0; d < 3; ++d) P.mean[d] = (float)(h[d] / (double)n);
  m2dp_cov_kernel<<<red_blocks, 256, 0, s>>>(d_in, stride_bytes, n, P.mean[0], P.mean[1], P.mean[2], d_sums + 8);
  SMB_CUDA_OK(cudaMemcpyAsync(h, d_sums + 8, 6 * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  {   // axes of the float covariance matrix, descending eigenvalue (pcl::PCA::initCompute)
    const double denom = (double)(float)(n - 1);
    const float c0 = (float)(h[0] / denom), c1 = (float)(h[1] / denom), c2 = (float)(h[2] / denom),
                c3 = (float)(h[3] / denom), c4 = (float)(h[4] / denom), c5 = (float)(h[5] / denom);
    std::vector<double> C = {c0, c1, c2, c1, c3, c4, c2, c4, c5};
    std::vector<double> e0, e1;
    const double l0 = power_iteration(C, 3, e0);
    std::vector<double> D = C;                                     // deflate the first axis
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) D[(size_t)i * 3 + j] -= l0 * e0[(size_t)i] * e0[(size_t)j];
    power_iteration(D, 3, e1);
    double dot = 0.0;                                              // re-orthogonalise against the first axis
    for (int i = 0; i < 3; ++i) dot += e0[(size_t)i] * e1[(size_t)i];
    double nrm = 0.0;
    for (int i = 0; i < 3; ++i) { e1[(size_t)i] -= dot * e0[(size_t)i]; nrm += e1[(size_t)i] * e1[(size_t)i]; }
    nrm = sqrt(nrm);
    if (nrm > 0) for (int i = 0; i < 3; ++i) e1[(size_t)i] /= nrm;
    orient(e0.data(), 3); orient(e1.data(), 3);
    for (int k = 0; k < 3; ++k) { P.E[k * 3 + 0] = (float)e0[(size_t)k]; P.E[k * 3 + 1] = (float)e1[(size_t)k]; }
    P.E[0 * 3 + 2] = P.E[1 * 3 + 0] * P.E[2 * 3 + 1] - P.E[2 * 3 + 0] * P.E[1 * 3 + 1];
    P.E[1 * 3 + 2] = P.E[2 * 3 + 0] * P.E[0 * 3 + 1] - P.E[0 * 3 + 0] * P.E[2 * 3 + 1];
    P.E[2 * 3 + 2] = P.E[0 * 3 + 0] * P.E[1 * 3 + 1] - P.E[1 * 3 + 0] * P.E[0 * 3 + 1];
  }
  P.r = r; P.max_distance = max_distance; P.angle_step = (M_PI * 2.) / t;
  P.l = l; P.t = t; P.cols = cols; P.n_views = rows;
  {   // view axes (m2dp.cc:73-83), float like the reference
    std::vector<M2dpView> hv((size_t)rows);
    const double theta_step = M_PI / p, phi_step = M_PI_2 / q;
    for (int pi = 0; pi < p; ++pi)
      for (int qi = 0; qi < q; ++qi) {
        const double theta = pi * theta_step, phi = qi * phi_step;
        const float mx = (float)(cos(theta) * cos(phi)), my = (float)(cos(theta) * sin(phi)), mz = (float)sin(theta);
        const float sgl = fabsf(mx);
        M2dpView& v = hv[(size_t)(pi * q + qi)];
        v.xa[0] = 1.f - sgl * mx; v.xa[1] = 0.f - sgl * my; v.xa[2] = 0.f - sgl * mz;
        v.ya[0] = my * v.xa[2] - mz * v.xa[1]; v.ya[1] = mz * v.xa[0] - mx * v.xa[2]; v.ya[2] = mx * v.xa[1] - my * v.xa[0];
      }
    SMB_CUDA_OK(cudaMemcpyAsync(d_views, hv.data(), (size_t)rows * sizeof(M2dpView), cudaMemcpyHostToDevice, s));
    SMB_CUDA_OK(cudaStreamSynchronize(s));          // hv goes out of scope
  }
  const dim3 grid((unsigned)((n + kPointsPerCta - 1) / kPointsPerCta), (unsigned)((rows + kViewsPerCta - 1) / kViewsPerCta));
  m2dp_hist_kernel<<<grid, kHistThreads, (size_t)kViewsPerCta * cols * sizeof(int), s>>>(d_in, stride_bytes, n, P, d_views, d_A);
  m2dp_gram_kernel<<<dim3((unsigned)rows, (unsigned)rows), 256, 0, s>>>(d_A, rows, cols, d_G);
  SMB_CUDA_OK(cudaGetLastError());
  std::vector<int> A((size_t)rows * cols);
  std::vector<double> G((size_t)rows * rows);
  SMB_CUDA_OK(cudaMemcpyAsync(A.data(), d_A, A.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaMemcpyAsync(G.data(), d_G, G.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  if (A_out) memcpy(A_out, A.data(), A.size() * sizeof(int));
  // first singular pair: u1 = dominant eigenvector of A A^T, sigma1^2 its eigenvalue, v1 = A^T u1 / sigma1
  std::vector<double> u;
  const double lambda = power_iteration(G, rows, u);
  orient(u.data(), rows);
  const double sigma = sqrt(lambda > 0 ? lambda : 0.0);
  for (int k = 0; k < rows; ++k) descriptor[k] = (float)u[(size_t)k];
  for (int c = 0; c < cols; ++c) {
    double sacc = 0.0;
    for (int a = 0; a < rows; ++a) sacc += (double)A[(size_t)a * cols + c] * u[(size_t)a];
    descriptor[rows + c] = sigma > 0 ? (float)(sacc / sigma) : 0.f;
  }
  return 1;
}

extern "C" double sm_m2dp_match(const float* P, const float* Q, int64_t n) {
  if (!P || !Q || n < 10) return -1.;                 // "The Descriptors do not match" (m2dp.cc:157-160)
  float pq = 0.f, pp = 0.f, qq = 0.f, sp = 0.f, sq = 0.f;
  for (int64_t i = 0; i < n; ++i) { pq += P[i] * Q[i]; pp += P[i] * P[i]; qq += Q[i] * Q[i]; sp += P[i]; sq += Q[i]; }
  const double N = (double)n;
  return fabs((N * pq - (double)(sp * sq)) / sqrt((N * pp - pow((double)sp, 2)) * (N * qq - pow((double)sq, 2))));
}
