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
#include "common.cuh"
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

__global__ void normals_leaf_kernel(const double* __restrict__ coord, int64_t cstride,
                                    const KdNode* __restrict__ nodes,
                                    const uint32_t* __restrict__ leaf_order, int n, int levels,
                                    double* __restrict__ out_pts, double* __restrict__ out_nrm,
                                    uint32_t* __restrict__ keep) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = (1 << (levels + 1)) - 1;
  if (h >= total) return;
  // existence / leaf test by the shape arithmetic (nodes[] of non-existent slots is garbage)
  const int L = 31 - __clz(h + 1);
  int first = 0, count = n;
  {
    const int j = h + 1 - (1 << L);
    for (int l = L - 1; l >= 0; --l) {
      if (count <= 7) return;                       // an ancestor was already a leaf
      const int right = count >> 1, left = count - right;
      if ((j >> l) & 1) { first += left; count = right; } else { count = left; }
    }
  }
  if (count > 7) return;
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

constexpr int kCT = 256, kCI = 8, kCTile = kCT * kCI;

__global__ void __launch_bounds__(kCT)
compact_count_kernel(const uint32_t* __restrict__ keep, int n, uint32_t* __restrict__ block_sum) {
  __shared__ uint32_t ws[kCT / 32];
  uint32_t c = 0;
  const int base = blockIdx.x * kCTile + threadIdx.x * kCI;
  for (int r = 0; r < kCI; ++r) if (base + r < n) c += keep[base + r];
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kCT / 32; ++w) t += ws[w];
    block_sum[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(kCT)
compact_scatter_kernel(const uint32_t* __restrict__ keep, int n, const uint32_t* __restrict__ block_off,
                       const double* __restrict__ pts, const double* __restrict__ nrm,
                       double* __restrict__ out_pts, double* __restrict__ out_nrm,
                       uint32_t* __restrict__ total_out, int nblk) {
  __shared__ uint32_t ws[kCT / 32];
  const int base = blockIdx.x * kCTile + threadIdx.x * kCI;
  uint32_t f[kCI], c = 0;
  for (int r = 0; r < kCI; ++r) { f[r] = (base + r < n) ? keep[base + r] : 0u; c += f[r]; }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t incl = c;
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) ws[w] = incl;
  __syncthreads();
  uint32_t wb = 0, tot = 0;
  for (int ww = 0; ww < kCT / 32; ++ww) { const uint32_t v = ws[ww]; if (ww < w) wb += v; tot += v; }
  uint32_t pos = block_off[blockIdx.x] + wb + incl - c;
  for (int r = 0; r < kCI; ++r) {
    if (f[r]) {
      const int64_t i = base + r;
      for (int k = 0; k < 3; ++k) {
        out_pts[3 * (int64_t)pos + k] = pts[3 * i + k];
        out_nrm[3 * (int64_t)pos + k] = nrm[3 * i + k];
      }
      ++pos;
    }
  }
  if (blockIdx.x == nblk - 1 && threadIdx.x == 0) *total_out = block_off[blockIdx.x] + tot;
}

}  // namespace

// host build of the leaf routine (test hook sm_debug_normals_leaf): members[count][3] in member order
int normals_debug_leaf_host(const double* members, int count, double* mean, double* unit) {
  if (count < 1 || count > 7) return -1;
  double d[7][3];
  for (int i = 0; i < count; ++i) for (int r = 0; r < 3; ++r) d[i][r] = members[3 * i + r];
  return leaf_plane_fit(d, count, mean, unit) ? 1 : 0;
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
  SMB_RC(bsum.reserve((size_t)(ceil_div(n, kCTile) + 1) * sizeof(uint32_t)));
  SMB_RC(out_pts.reserve(aos)); SMB_RC(out_nrm.reserve(aos));
  return count.reserve(sizeof(uint32_t));
}

int NormalsPipeline::run(int n, cudaStream_t stream, uint32_t* m) {
  const int levels = kd_num_levels(n, 7);
  uint32_t* block_sums = (uint32_t*)bsum.p;
  KdWorkspace ws;
  SMB_RC(ws.carve(kdws, n, 7));
  SMB_RC(kd_build(input(), stride, n, 7, ws, (KdNode*)nodes.p, (uint32_t*)order.p, stream));
  SMB_CUDA_OK(cudaMemsetAsync(keep.p, 0, (size_t)n * sizeof(uint32_t), stream));
  const int total = (1 << (levels + 1)) - 1;
  normals_leaf_kernel<<<ceil_div(total, 128), 128, 0, stream>>>(input(), stride, (const KdNode*)nodes.p,
                                                               (const uint32_t*)order.p, n, levels, (double*)tmp_pts.p,
                                                               (double*)tmp_nrm.p, (uint32_t*)keep.p);
  const int nblk = ceil_div(n, kCTile);
  compact_count_kernel<<<nblk, kCT, 0, stream>>>((const uint32_t*)keep.p, n, block_sums);
  radix_scan_kernel_launch(block_sums, nblk, 1, stream);
  compact_scatter_kernel<<<nblk, kCT, 0, stream>>>((const uint32_t*)keep.p, n, block_sums, (const double*)tmp_pts.p,
                                                   (const double*)tmp_nrm.p, (double*)out_pts.p, (double*)out_nrm.p,
                                                   (uint32_t*)count.p, nblk);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(m, count.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

}  // namespace smb
