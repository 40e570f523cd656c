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
// contraction.  One CTA owns a chunk of points and a GROUP of up to 8 views whose histograms
// live in shared memory (8 x 512 x 4 B = 16 KB by default; fewer views per CTA when a histogram
// is wider, so that a group always fits the 48 KB a block gets without opting in): the point is
// loaded and projected once per CTA-thread, the views hit shared-memory atomics only (the
// reference's |.| folds everything into the first quadrant, so a view touches ~128 distinct bins:
// global atomics would serialise in L2), and the non-empty bins are flushed to the global matrix
// with one atomic each at the end.  Sums for the PCA are double block reductions.  A A^T (64 x 64,
// exact in double: counts < 2^31) is formed on the device; the two small symmetric eigenproblems
// run on the host by cyclic Jacobi in double, whose error does not grow as the leading eigenvalues
// close in (a square patch has lambda1 ~ lambda2, and M2DP is meant to be invariant in that frame).
// Sign conventions: see oracle/m2dp_oracle.cc — they live inside Eigen in the reference and are
// fixed the same way on both sides here.
//
// The pieces: M2dpStage (device buffers and kernels, with the host steps between them),
// m2dp_axes (covariance -> axes) and m2dp_descriptor (A and A A^T -> [u1; v1]); sm_m2dp and the
// test hooks of csrc/sm_debug.cu call these.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace smb {
namespace {

constexpr int kViewsPerCta = 8;
constexpr int kHistThreads = 256;
constexpr int kPointsPerCta = 4096;

struct M2dpParams {
  float mean[3];
  float E[9];             // E[k * 3 + j]: component k of axis j
  double r, max_distance, angle_step;
  int l, t, cols, n_views;
  int views_per_cta;      // hist_views_per_cta(cols)
};

__global__ void __launch_bounds__(256)
m2dp_mean_kernel(const char* __restrict__ pts, int64_t stride, int64_t n, double* __restrict__ sums) {
  __shared__ double red[8][3];
  double s[3] = {0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* p = reinterpret_cast<const float*>(pts + i * stride);
    s[0] += (double)p[0]; s[1] += (double)p[1]; s[2] += (double)p[2];
  }
  const double v = block_sum<3, 256>(s, red);
  if (threadIdx.x < 3) atomicAdd(&sums[threadIdx.x], v);
}

// covariance sums of the float-demeaned cloud (pcl::demeanPointCloud works in float)
__global__ void __launch_bounds__(256)
m2dp_cov_kernel(const char* __restrict__ pts, int64_t stride, int64_t n, float cx, float cy, float cz,
                double* __restrict__ sums) {
  __shared__ double red[8][6];
  double s[6] = {0, 0, 0, 0, 0, 0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float* p = reinterpret_cast<const float*>(pts + i * stride);
    const float x = p[0] - cx, y = p[1] - cy, z = p[2] - cz;
    s[0] += (double)(x * x); s[1] += (double)(x * y); s[2] += (double)(x * z);
    s[3] += (double)(y * y); s[4] += (double)(y * z); s[5] += (double)(z * z);
  }
  const double v = block_sum<6, 256>(s, red);
  if (threadIdx.x < 6) atomicAdd(&sums[threadIdx.x], v);
}

// grid: (point chunks, view groups of P.views_per_cta).  Dynamic shared memory: views_per_cta * cols ints.
__global__ void __launch_bounds__(kHistThreads)
m2dp_hist_kernel(const char* __restrict__ pts, int64_t stride, int64_t n, M2dpParams P,
                 const M2dpView* __restrict__ views, int* __restrict__ A) {
  extern __shared__ int hist[];
  __shared__ M2dpView sv[kViewsPerCta];
  const int v0 = blockIdx.y * P.views_per_cta;
  const int nv = min(P.views_per_cta, P.n_views - v0);
  for (int k = threadIdx.x; k < nv * P.cols; k += kHistThreads) hist[k] = 0;
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

// views per histogram CTA: up to 8, as many histograms of cols counts as the kernel's dynamic shared memory holds
// without opting in (48 KB less its static part: 8 views up to cols = 1530, one view for the widest, 8192)
int hist_views_per_cta(int cols, int* vpc) {
  cudaFuncAttributes fa;
  SMB_CUDA_OK(cudaFuncGetAttributes(&fa, m2dp_hist_kernel));
  *vpc = std::max(1, std::min(kViewsPerCta, fa.maxDynamicSharedSizeBytes / (int)(cols * sizeof(int))));
  return 0;
}

// G = A A^T (rows x rows) in double; one block per (a, b-tile)
__global__ void __launch_bounds__(256)
m2dp_gram_kernel(const int* __restrict__ A, int rows, int cols, double* __restrict__ G) {
  __shared__ double red[8][1];
  const int a = blockIdx.x, b = blockIdx.y;
  if (b < a) return;
  double s = 0.0;
  for (int k = threadIdx.x; k < cols; k += 256) s += (double)A[(int64_t)a * cols + k] * (double)A[(int64_t)b * cols + k];
  const double t = block_sum<1, 256>(&s, red);   // integer-valued partial sums < 2^53: exact in any order
  if (threadIdx.x == 0) {
    G[(int64_t)a * rows + b] = t; G[(int64_t)b * rows + a] = t;
  }
}

// Eigen-decomposition of the symmetric n x n matrix a (row-major, double) by cyclic Jacobi rotations: on return
// a[j * n + j] is an eigenvalue and row j of vt its unit eigenvector.  A rotation is skipped once its off-diagonal
// entry is below the rounding of its two diagonal entries (|a_pq| <= eps sqrt(|a_pp a_qq|)), and the sweeps stop
// when one skips them all.  Each rotation is orthogonal, so the computed pairs belong to a matrix within a few
// roundings of a whatever the eigenvalue gaps; an eigenvector's error is then that over its gap, the conditioning
// of the problem itself, with no iteration count that depends on the gap as power iteration's does.
void jacobi_eigen(std::vector<double>& a, int n, std::vector<double>& vt) {
  vt.assign((size_t)n * n, 0.0);
  for (int i = 0; i < n; ++i) vt[(size_t)i * n + i] = 1.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        double* ap = &a[(size_t)p * n];
        double* aq = &a[(size_t)q * n];
        const double apq = ap[q], app = ap[p], aqq = aq[q];
        if (!(fabs(apq) > 2.2e-16 * sqrt(fabs(app) * fabs(aqq)))) continue;
        rotated = true;
        const double theta = (aqq - app) / (2.0 * apq);
        const double t = fabs(theta) > 1e150 ? 0.5 / theta
                                             : (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {               // rows p and q, mirrored into columns p and q
          if (k == p || k == q) continue;
          const double akp = ap[k], akq = aq[k];
          ap[k] = a[(size_t)k * n + p] = c * akp - s * akq;
          aq[k] = a[(size_t)k * n + q] = s * akp + c * akq;
        }
        ap[p] = app - t * apq; aq[q] = aqq + t * apq;
        ap[q] = aq[p] = 0.0;
        double* vp = &vt[(size_t)p * n];
        double* vq = &vt[(size_t)q * n];
        for (int k = 0; k < n; ++k) {
          const double x = vp[k], y = vq[k];
          vp[k] = c * x - s * y; vq[k] = s * x + c * y;
        }
      }
    if (!rotated) break;
  }
}

void orient(double* v, int n) {    // component of largest magnitude positive
  int big = 0;
  for (int k = 1; k < n; ++k) if (fabs(v[k]) > fabs(v[big])) big = k;
  if (v[big] < 0) for (int k = 0; k < n; ++k) v[k] = -v[k];
}

}  // namespace

// axes of the float covariance matrix, descending eigenvalue (pcl::PCA::initCompute), third = first x second in float
void m2dp_axes(const float* c, float* E) {
  double e[2][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}};   // no finite covariance (one point: 0 / 0): the input frame
  bool finite = true;
  for (int k = 0; k < 6; ++k) finite = finite && isfinite(c[k]);
  if (finite) {
    std::vector<double> a = {c[0], c[1], c[2], c[1], c[3], c[4], c[2], c[4], c[5]}, vt;
    jacobi_eigen(a, 3, vt);
    int order[3] = {0, 1, 2};
    std::stable_sort(order, order + 3, [&](int x, int y) { return a[(size_t)x * 4] > a[(size_t)y * 4]; });
    for (int j = 0; j < 2; ++j)
      for (int k = 0; k < 3; ++k) e[j][k] = vt[(size_t)order[j] * 3 + k];
  }
  orient(e[0], 3); orient(e[1], 3);
  for (int k = 0; k < 3; ++k) { E[k * 3 + 0] = (float)e[0][k]; E[k * 3 + 1] = (float)e[1][k]; }
  E[0 * 3 + 2] = E[1 * 3 + 0] * E[2 * 3 + 1] - E[2 * 3 + 0] * E[1 * 3 + 1];
  E[1 * 3 + 2] = E[2 * 3 + 0] * E[0 * 3 + 1] - E[0 * 3 + 0] * E[2 * 3 + 1];
  E[2 * 3 + 2] = E[0 * 3 + 0] * E[1 * 3 + 1] - E[1 * 3 + 0] * E[0 * 3 + 1];
}

// first singular pair of A (rows x cols) from G = A A^T: u1 = dominant eigenvector of G, sigma1^2 its eigenvalue,
// v1 = A^T u1 / sigma1; out = [u1; v1] in float, all zero when A is
void m2dp_descriptor(const int* A, const double* G, int rows, int cols, float* out) {
  std::vector<double> a(G, G + (size_t)rows * rows), vt;
  jacobi_eigen(a, rows, vt);
  int top = 0;
  for (int k = 1; k < rows; ++k) if (a[(size_t)k * rows + k] > a[(size_t)top * rows + top]) top = k;
  const double lambda = a[(size_t)top * rows + top];
  if (!(lambda > 0.0)) {
    for (int k = 0; k < rows + cols; ++k) out[k] = 0.f;
    return;
  }
  std::vector<double> u(vt.begin() + (size_t)top * rows, vt.begin() + (size_t)(top + 1) * rows);
  orient(u.data(), rows);
  const double sigma = sqrt(lambda);
  for (int k = 0; k < rows; ++k) out[k] = (float)u[(size_t)k];
  for (int c = 0; c < cols; ++c) {
    double sacc = 0.0;
    for (int a_ = 0; a_ < rows; ++a_) sacc += (double)A[(size_t)a_ * cols + c] * u[(size_t)a_];
    out[rows + c] = (float)(sacc / sigma);
  }
}

int M2dpStage::run(const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance, int t, int p,
                   int q, cudaStream_t s) {
  l = (int)ceil(sqrt(max_distance / r));
  rows = p * q; cols = l * t;
  const size_t in_bytes = (size_t)n * (size_t)stride_bytes;
  const size_t bytes = in_bytes + 256 + 16 * sizeof(double) + (size_t)rows * sizeof(M2dpView) + 256 +
                       (size_t)rows * cols * sizeof(int) + 256 + (size_t)rows * rows * sizeof(double) + 256;
  SMB_RC(buf.reserve(bytes));
  char* cur = (char*)buf.p;
  auto take = [&](size_t b) { char* ptr = cur; cur += (b + 255) & ~(size_t)255; return ptr; };
  char* d_in = take(in_bytes);
  double* d_sums = (double*)take(16 * sizeof(double));
  M2dpView* d_views = (M2dpView*)take((size_t)rows * sizeof(M2dpView));
  int* d_A = (int*)take((size_t)rows * cols * sizeof(int));
  double* d_G = (double*)take((size_t)rows * rows * sizeof(double));
  SMB_CUDA_OK(cudaMemcpyAsync(d_in, points, in_bytes, cudaMemcpyHostToDevice, s));
  SMB_CUDA_OK(cudaMemsetAsync(d_sums, 0, 16 * sizeof(double), s));
  SMB_CUDA_OK(cudaMemsetAsync(d_A, 0, (size_t)rows * cols * sizeof(int), s));
  const int red_blocks = (int)std::min<int64_t>(4 * kNumSMs, (n + 255) / 256);
  m2dp_mean_kernel<<<red_blocks, 256, 0, s>>>(d_in, stride_bytes, n, d_sums);
  double h[3];
  SMB_CUDA_OK(cudaMemcpyAsync(h, d_sums, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  M2dpParams P;
  for (int d = 0; d < 3; ++d) P.mean[d] = mean[d] = (float)(h[d] / (double)n);
  m2dp_cov_kernel<<<red_blocks, 256, 0, s>>>(d_in, stride_bytes, n, P.mean[0], P.mean[1], P.mean[2], d_sums + 8);
  SMB_CUDA_OK(cudaMemcpyAsync(cov_sums, d_sums + 8, 6 * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  const double denom = (double)(float)(n - 1);
  for (int k = 0; k < 6; ++k) cov[k] = (float)(cov_sums[k] / denom);
  m2dp_axes(cov, E);
  memcpy(P.E, E, sizeof(E));
  P.r = r; P.max_distance = max_distance; P.angle_step = (M_PI * 2.) / t;
  P.l = l; P.t = t; P.cols = cols; P.n_views = rows;
  SMB_RC(hist_views_per_cta(cols, &P.views_per_cta));
  views.resize((size_t)rows);               // view axes (m2dp.cc:73-83), float like the reference
  const double theta_step = M_PI / p, phi_step = M_PI_2 / q;
  for (int pi = 0; pi < p; ++pi)
    for (int qi = 0; qi < q; ++qi) {
      const double theta = pi * theta_step, phi = qi * phi_step;
      const float mx = (float)(cos(theta) * cos(phi)), my = (float)(cos(theta) * sin(phi)), mz = (float)sin(theta);
      const float sgl = fabsf(mx);
      M2dpView& v = views[(size_t)(pi * q + qi)];
      v.xa[0] = 1.f - sgl * mx; v.xa[1] = 0.f - sgl * my; v.xa[2] = 0.f - sgl * mz;
      v.ya[0] = my * v.xa[2] - mz * v.xa[1]; v.ya[1] = mz * v.xa[0] - mx * v.xa[2]; v.ya[2] = mx * v.xa[1] - my * v.xa[0];
    }
  SMB_CUDA_OK(cudaMemcpyAsync(d_views, views.data(), (size_t)rows * sizeof(M2dpView), cudaMemcpyHostToDevice, s));
  const dim3 grid((unsigned)((n + kPointsPerCta - 1) / kPointsPerCta),
                  (unsigned)((rows + P.views_per_cta - 1) / P.views_per_cta));
  m2dp_hist_kernel<<<grid, kHistThreads, (size_t)P.views_per_cta * cols * sizeof(int), s>>>(d_in, stride_bytes, n, P,
                                                                                           d_views, d_A);
  m2dp_gram_kernel<<<dim3((unsigned)rows, (unsigned)rows), 256, 0, s>>>(d_A, rows, cols, d_G);
  SMB_CUDA_OK(cudaGetLastError());
  A.resize((size_t)rows * cols);
  G.resize((size_t)rows * rows);
  SMB_CUDA_OK(cudaMemcpyAsync(A.data(), d_A, A.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaMemcpyAsync(G.data(), d_G, G.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace smb

using namespace smb;

// At most 8192 bins per view and 256 views: the eigenproblem of A A^T (p*q x p*q) is solved on the host by Jacobi,
// whose cost grows as (p*q)^3: about 2 ms at the default 64 views, 0.8 s at 256, 13 s at 512 (one CPU core).
extern "C" int64_t sm_m2dp_descriptor_length(double r, double max_distance, int32_t t, int32_t p, int32_t q) {
  if (r < 1.e-6 || !(max_distance > 0.0) || t <= 0 || p <= 0 || q <= 0) return SM_ERR_BAD_ARGUMENT;
  const double l = ceil(sqrt(max_distance / r));
  if (!(l >= 1.0) || l * t > 8192.0 || (double)p * q > 256.0) return SM_ERR_BAD_ARGUMENT;
  return (int64_t)p * q + (int64_t)l * t;
}

extern "C" int sm_m2dp(int device, const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance,
                       int32_t t, int32_t p, int32_t q, float* descriptor, int64_t capacity, int32_t* A_out) {
  if (!points || !descriptor || n < 0 || n > (1ll << 30) || stride_bytes < 12 || stride_bytes % 4) return SM_ERR_BAD_ARGUMENT;
  const int64_t len = sm_m2dp_descriptor_length(r, max_distance, t, p, q);
  if (len < 0 || capacity < len) return SM_ERR_BAD_ARGUMENT;        // "r is too small" (m2dp.cc:64-67)
  if (n == 0) return 0;                                             // "source is empty": setInputCloud returns false
  SMB_RC(select_device(device));
  M2dpStage st;
  SMB_RC(st.run(points, n, stride_bytes, r, max_distance, t, p, q, nullptr));
  if (A_out) memcpy(A_out, st.A.data(), st.A.size() * sizeof(int));
  m2dp_descriptor(st.A.data(), st.G.data(), st.rows, st.cols, descriptor);
  return 1;
}

extern "C" double sm_m2dp_match(const float* P, const float* Q, int64_t n) {
  if (!P || !Q || n < 10) return -1.;                 // "The Descriptors do not match" (m2dp.cc:157-160)
  float pq = 0.f, pp = 0.f, qq = 0.f, sp = 0.f, sq = 0.f;
  for (int64_t i = 0; i < n; ++i) { pq += P[i] * Q[i]; pp += P[i] * P[i]; qq += Q[i] * Q[i]; sp += P[i]; sq += Q[i]; }
  const double N = (double)n;
  return fabs((N * pq - (double)(sp * sq)) / sqrt((N * pp - pow((double)sp, 2)) * (N * qq - pow((double)sq, 2))));
}
