// Target preparation on the device: EigenPointCloud::CalculateNormals
// (builder/data/cloud_types.cc:347-368 with BuildNormals :105-144 and the leaf routine
// :73-103).  Callers in the reference: map_builder.cc:286,389 and submap.cc:161 — it runs
// right before every IcpFast::SetInputTarget, serially, on up to 500k points.
//
// The median-split recursion to leaves of <= 7 points is the SAME partition the k-d tree
// builder produces with bucket = 7, so this file only adds the per-leaf plane fit (one
// thread per leaf, ascending-original-index member order) and an order-preserving
// compaction of the surviving leaf representatives.  Compiled with -fmad=false: with
// the same operation order as the oracle the output is bit-identical to it.
//
// The same pipeline also runs libpointmatcher's SamplingSurfaceNormalDataPointsFilter (knn 7, samplingMethod 1),
// the reference filter of IcpUsingPointMatcher: the same boxes, with the box mean and the smallest eigenvector of
// the box covariance in float (leaf_eigen_normal).  run() takes which leaf routine to apply.
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"
#include "linalg_dev.cuh"

namespace smb {
namespace {

// The leaf routine (cloud_types.cc:73-103): M = sum d d^T and b = sum d over the members in the given order, mean,
// C = sum (d - mean)(d - mean)^T; dropped if rank(C) + 1 < 3 (:89-91); normal = normalize(M^-1 b) (:93-101).
// Returns false for a dropped leaf.  __host__ too: the test hook sm_debug_normals_leaf runs this very function.
__host__ __device__ __forceinline__ bool leaf_plane_fit(const double (*d)[3], int count, double* mean, double* unit) {
  double M[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < count; ++i)
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) M[r * 3 + c] += d[i][r] * d[i][c];
  double b[3] = {0, 0, 0};
  for (int r = 0; r < 3; ++r)
    for (int i = 0; i < count; ++i) b[r] += d[i][r];
  for (int r = 0; r < 3; ++r) mean[r] = b[r] / count;
  double C[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double s = 0.0;
      for (int i = 0; i < count; ++i) s += (d[i][r] - mean[r]) * (d[i][c] - mean[c]);
      C[r * 3 + c] = s;
    }
  la::PivQR<3> qr;
  qr.compute(C);
  if (qr.rank() + 1 < 3) return false;              // :89-91
  double Minv[9], nrm[3];
  la::lu_inverse3(M, Minv);                         // :93
  for (int r = 0; r < 3; ++r)
    nrm[r] = Minv[r * 3 + 0] * b[0] + Minv[r * 3 + 1] * b[1] + Minv[r * 3 + 2] * b[2];
  const double sq = nrm[0] * nrm[0] + nrm[1] * nrm[1] + nrm[2] * nrm[2];
  const double len = sqrt(sq);
  for (int r = 0; r < 3; ++r) unit[r] = (sq > 0.0) ? nrm[r] / len : nrm[r];
  return true;
}

// Heap slot h of the median-split recursion over n points: true if it is a leaf (<= 7 points), with its span
// [first, first + count) of the tree's leaf order.  Existence and the leaf test come from the shape arithmetic alone.
__device__ __forceinline__ bool leaf_span(int h, int n, int levels, int* first_out, int* count_out) {
  const int total = (1 << (levels + 1)) - 1;
  if (h >= total) return false;
  const int L = 31 - __clz(h + 1);
  int first = 0, count = n;
  {
    const int j = h + 1 - (1 << L);
    for (int l = L - 1; l >= 0; --l) {
      if (count <= 7) return false;                 // an ancestor was already a leaf
      const int right = count >> 1, left = count - right;
      if ((j >> l) & 1) { first += left; count = right; } else { count = left; }
    }
  }
  if (count > 7) return false;
  *first_out = first;
  *count_out = count;
  return true;
}

// rank(C) of Eigen's FullPivHouseholderQR (la::PivQR<3>, the same decomposition of the same double matrix, R only)
// with the threshold of a float matrix: the pivots above |max pivot| * 3 FLT_EPSILON.  Every index is a constant
// once the loops are unrolled: the pivot's row and column swaps are selects.
__host__ __device__ __forceinline__ int pm_rank3(const double* A) {
  double R[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) R[i] = A[i];
  const double precision = la::kEps * 3.0;
  int nonzero_pivots = 3;
  double maxpivot = 0.0, biggest = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    int rb = k, cb = k;
    double best = -1.0;
#pragma unroll
    for (int c = k; c < 3; ++c)                     // column-major visit, strict '>' (Eigen maxCoeff)
#pragma unroll
      for (int r = k; r < 3; ++r) {
        const double v = fabs(R[r * 3 + c]);
        if (v > best) { best = v; rb = r; cb = c; }
      }
    if (k == 0) biggest = best;
    if (fabs(best) <= fabs(biggest) * precision) { nonzero_pivots = k; break; }
#pragma unroll
    for (int r = k + 1; r < 3; ++r)
      if (r == rb)
#pragma unroll
        for (int c = 0; c < 3; ++c) { const double t = R[k * 3 + c]; R[k * 3 + c] = R[r * 3 + c]; R[r * 3 + c] = t; }
#pragma unroll
    for (int c = k + 1; c < 3; ++c)
      if (c == cb)
#pragma unroll
        for (int r = 0; r < 3; ++r) { const double t = R[r * 3 + k]; R[r * 3 + k] = R[r * 3 + c]; R[r * 3 + c] = t; }
    double tail_sq = 0.0;
#pragma unroll
    for (int r = k + 1; r < 3; ++r) tail_sq += R[r * 3 + k] * R[r * 3 + k];
    const double c0 = R[k * 3 + k];
    double beta, tau, v[3] = {0.0, 0.0, 0.0};
    if (tail_sq <= DBL_MIN) { tau = 0.0; beta = c0; }
    else {
      beta = sqrt(c0 * c0 + tail_sq);
      if (c0 >= 0.0) beta = -beta;
#pragma unroll
      for (int r = k + 1; r < 3; ++r) v[r] = R[r * 3 + k] / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    v[k] = 1.0;
    if (fabs(beta) > maxpivot) maxpivot = fabs(beta);
    R[k * 3 + k] = beta;
#pragma unroll
    for (int r = k + 1; r < 3; ++r) R[r * 3 + k] = 0.0;
    if (tau != 0.0)
#pragma unroll
      for (int c = k + 1; c < 3; ++c) {
        double dot = 0.0;
#pragma unroll
        for (int r = k; r < 3; ++r) dot += v[r] * R[r * 3 + c];
#pragma unroll
        for (int r = k; r < 3; ++r) R[r * 3 + c] -= tau * v[r] * dot;
      }
  }
  const double thr = fabs(maxpivot) * ((double)FLT_EPSILON * 3.0);
  int rk = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) rk += (i < nonzero_pivots && fabs(R[i * 3 + i]) > thr) ? 1 : 0;
  return rk;
}

// The leaf of SamplingSurfaceNormalDataPointsFilter (libpointmatcher 1.3.1, knn 7, samplingMethod 1) in
// PointMatcher<float>: the members d[0..count) in ascending original index;
//   mean = (d_0 + d_1 + ... + d_{count-1}) / float(count), summed in member order from d_0, in float;
//   C = sum (d_i - mean)(d_i - mean)^T in float, each entry summed in member order from i = 0;
//   dropped if rank(C) + 1 < 3 (pm_rank3, on C widened to double);
//   normal = the eigenvector of the smallest eigenvalue of C (the first of equals), by the double Jacobi of
//   la::jacobi_eig_sym, normalised in double, rounded to float, with its component of largest magnitude (the first
//   of equals) made positive, as M2DP orients its axes.
// Returns false for a dropped leaf.  __host__ too: the test hook sm_debug_pm_surface_normal_leaf_host runs this
// very function.  Loops run to 7 with a guard so that every index is a constant and d stays in registers.
__host__ __device__ __forceinline__ bool leaf_eigen_normal(const float (*d)[3], int count, float* mean, float* C,
                                                           float* unit) {
  float s[3] = {d[0][0], d[0][1], d[0][2]};
#pragma unroll
  for (int i = 1; i < 7; ++i)
    if (i < count)
#pragma unroll
      for (int r = 0; r < 3; ++r) s[r] += d[i][r];
  const float fc = (float)count;
#pragma unroll
  for (int r = 0; r < 3; ++r) mean[r] = s[r] / fc;
  float e[7][3];
#pragma unroll
  for (int i = 0; i < 7; ++i)
#pragma unroll
    for (int r = 0; r < 3; ++r) e[i][r] = i < count ? d[i][r] - mean[r] : 0.0f;
  double Cd[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float acc = e[0][r] * e[0][c];
#pragma unroll
      for (int i = 1; i < 7; ++i)
        if (i < count) acc += e[i][r] * e[i][c];
      C[r * 3 + c] = acc;
      Cd[r * 3 + c] = (double)acc;
    }
  if (pm_rank3(Cd) + 1 < 3) return false;
  double w[3], V[9];
  la::jacobi_eig_sym3(Cd, w, V);
  int k = 0;                                        // written with selects: no array is indexed by a variable
  double wk = w[0];
  if (w[1] < wk) { k = 1; wk = w[1]; }
  if (w[2] < wk) k = 2;
  const double v0 = k == 0 ? V[0] : (k == 1 ? V[1] : V[2]);
  const double v1 = k == 0 ? V[3] : (k == 1 ? V[4] : V[5]);
  const double v2 = k == 0 ? V[6] : (k == 1 ? V[7] : V[8]);
  const double len = sqrt(v0 * v0 + v1 * v1 + v2 * v2);
  unit[0] = (float)(v0 / len); unit[1] = (float)(v1 / len); unit[2] = (float)(v2 / len);
  float big = unit[0];
  if (fabsf(unit[1]) > fabsf(big)) big = unit[1];
  if (fabsf(unit[2]) > fabsf(big)) big = unit[2];
  if (big < 0.0f) { unit[0] = -unit[0]; unit[1] = -unit[1]; unit[2] = -unit[2]; }
  return true;
}

__global__ void normals_leaf_kernel(const double* __restrict__ coord, int64_t cstride,
                                    const KdNode* __restrict__ nodes,
                                    const uint32_t* __restrict__ leaf_order, int n, int levels,
                                    double* __restrict__ out_pts, double* __restrict__ out_nrm,
                                    uint32_t* __restrict__ keep) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  int first, count;
  if (!leaf_span(h, n, levels, &first, &count)) return;
  double d[7][3], mean[3], unit[3];
  for (int i = 0; i < count; ++i) {
    const uint32_t id = leaf_order[first + i];
    for (int r = 0; r < 3; ++r) d[i][r] = coord[r * cstride + id];
  }
  if (!leaf_plane_fit(d, count, mean, unit)) return;
  const uint32_t k = leaf_order[first];             // smallest original index of the leaf
  keep[k] = 1u;
  for (int r = 0; r < 3; ++r) {
    out_pts[3 * (int64_t)k + r] = mean[r];
    out_nrm[3 * (int64_t)k + r] = unit[r];
  }
}

// The eigenvector leaf over the same boxes: the float cloud as the pipeline's double input (exact widenings),
// rounded back to float per member.  Writes the float mean and normal, widened, to the box's smallest member index.
__global__ void pm_normals_leaf_kernel(const double* __restrict__ coord, int64_t cstride,
                                       const uint32_t* __restrict__ leaf_order, int n, int levels,
                                       double* __restrict__ out_pts, double* __restrict__ out_nrm,
                                       uint32_t* __restrict__ keep) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  int first, count;
  if (!leaf_span(h, n, levels, &first, &count)) return;
  float d[7][3];
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const uint32_t id = i < count ? leaf_order[first + i] : 0u;
#pragma unroll
    for (int r = 0; r < 3; ++r) d[i][r] = i < count ? (float)coord[r * cstride + id] : 0.0f;
  }
  float mean[3], C[9], unit[3];
  if (!leaf_eigen_normal(d, count, mean, C, unit)) return;
  const uint32_t k = leaf_order[first];             // smallest original index of the leaf
  keep[k] = 1u;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    out_pts[3 * (int64_t)k + r] = (double)mean[r];
    out_nrm[3 * (int64_t)k + r] = (double)unit[r];
  }
}

__global__ void __launch_bounds__(kCompactThreads)
compact_count_kernel(const uint32_t* __restrict__ keep, int n, uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += keep[base + r];
  tile_count_store(c, tile_cnt);
}

__global__ void __launch_bounds__(kCompactThreads)
compact_scatter_kernel(const uint32_t* __restrict__ keep, int n, const uint32_t* __restrict__ tile_off,
                       const double* __restrict__ pts, const double* __restrict__ nrm,
                       double* __restrict__ out_pts, double* __restrict__ out_nrm,
                       uint32_t* __restrict__ total_out) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n) ? keep[base + r] : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    if (f[r]) {
      const int64_t i = base + r;
      for (int k = 0; k < 3; ++k) {
        out_pts[3 * (int64_t)pos + k] = pts[3 * i + k];
        out_nrm[3 * (int64_t)pos + k] = nrm[3 * i + k];
      }
      ++pos;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *total_out = tile_off[gridDim.x];
}

}  // namespace

// host build of the leaf routine (test hook sm_debug_normals_leaf): members[count][3] in member order
int normals_debug_leaf_host(const double* members, int count, double* mean, double* unit) {
  if (count < 1 || count > 7) return -1;
  double d[7][3];
  for (int i = 0; i < count; ++i) for (int r = 0; r < 3; ++r) d[i][r] = members[3 * i + r];
  return leaf_plane_fit(d, count, mean, unit) ? 1 : 0;
}

// host build of the eigenvector leaf (test hook sm_debug_pm_surface_normal_leaf_host): members[count][3] in member
// order; mean[3], cov[9] (row-major) and unit[3] as the leaf computes them
int pm_normals_debug_leaf_host(const float* members, int count, float* mean, float* cov, float* unit) {
  if (count < 1 || count > 7) return -1;
  float d[7][3] = {};
  for (int i = 0; i < count; ++i) for (int r = 0; r < 3; ++r) d[i][r] = members[3 * i + r];
  return leaf_eigen_normal(d, count, mean, cov, unit) ? 1 : 0;
}

int NormalsPipeline::reserve(int n) {
  const int levels = kd_num_levels(n, 7);
  const size_t aos = (size_t)3 * (size_t)n * sizeof(double);
  stride = ((int64_t)n + 63) & ~(int64_t)63;
  SMB_RC(coord.reserve((size_t)3 * stride * sizeof(double)));
  SMB_RC(nodes.reserve((size_t)blocked_node_slots(levels) * sizeof(KdNode)));
  SMB_RC(order.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(tmp_pts.reserve(aos)); SMB_RC(tmp_nrm.reserve(aos));
  SMB_RC(keep.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(bsum.reserve(compact_count_bytes(n)));
  SMB_RC(out_pts.reserve(aos)); SMB_RC(out_nrm.reserve(aos));
  return count.reserve(sizeof(uint32_t));
}

int NormalsPipeline::run(int n, NormalsMode mode, cudaStream_t stream, uint32_t* m) {
  const int levels = kd_num_levels(n, 7);
  uint32_t* tile_cnt = (uint32_t*)bsum.p;
  KdWorkspace ws;
  SMB_RC(ws.carve(kdws, n, 7));
  SMB_RC(kd_build(input(), stride, n, 7, ws, (KdNode*)nodes.p, (uint32_t*)order.p, stream));
  SMB_CUDA_OK(cudaMemsetAsync(keep.p, 0, (size_t)n * sizeof(uint32_t), stream));
  const int total = (1 << (levels + 1)) - 1;
  if (mode == kNormalsEigenvector)
    pm_normals_leaf_kernel<<<ceil_div(total, 128), 128, 0, stream>>>(input(), stride, (const uint32_t*)order.p, n,
                                                                    levels, (double*)tmp_pts.p, (double*)tmp_nrm.p,
                                                                    (uint32_t*)keep.p);
  else
    normals_leaf_kernel<<<ceil_div(total, 128), 128, 0, stream>>>(input(), stride, (const KdNode*)nodes.p,
                                                                 (const uint32_t*)order.p, n, levels, (double*)tmp_pts.p,
                                                                 (double*)tmp_nrm.p, (uint32_t*)keep.p);
  const int tiles = compact_tiles(n);
  compact_count_kernel<<<tiles, kCompactThreads, 0, stream>>>((const uint32_t*)keep.p, n, tile_cnt);
  compact_scan(tile_cnt, tiles, stream);
  compact_scatter_kernel<<<tiles, kCompactThreads, 0, stream>>>(
      (const uint32_t*)keep.p, n, tile_cnt, (const double*)tmp_pts.p, (const double*)tmp_nrm.p, (double*)out_pts.p,
      (double*)out_nrm.p, (uint32_t*)count.p);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(m, count.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

}  // namespace smb
