// registrator::Ndt on the device (registrators/ndt.cc:28-64 -> vendored pclomp NDT,
// registrators/pclomp/ndt_omp_impl.hpp + voxel_grid_covariance_omp_impl.hpp).
//
//   target voxelisation   VoxelGridCovariance::applyFilter (_impl.hpp:49-370): the reference
//                         walks the points once, inserting into a std::map.  Here: voxel key per
//                         point -> stable radix sort -> one thread per voxel accumulates its
//                         points IN ORIGINAL ORDER (so sum x, sum x x^T and the float centroid
//                         round exactly like the serial loop), then mean / covariance / eigen
//                         inflation / inverse.  Searchable leaves (>= 6 points) go into an
//                         open-addressing hash table keyed by the voxel index.
//   neighbour search      radiusSearch over the centroid k-d tree with radius == leaf size
//                         (voxel_grid_covariance_omp.h:471-499) == probe the 3x3x3 voxels around
//                         the query and keep centroids with squared distance < r^2.
//   derivatives           computeDerivatives / updateDerivatives (ndt_omp_impl.hpp:180-284,
//                         483-535): per point and neighbour, single-precision math, double sums;
//                         block partials reduced in a fixed order.
//   fitness               pcl::Registration::getFitnessScore (ndt.cc:60): exact 1-NN in the full
//                         target through the same k-d tree as the ICP path (eps = 0).
// Compiled with -fmad=false: the per-leaf and per-(point, voxel) arithmetic is bit-identical
// to the oracle's written-out operation order.
#include <limits>

#include "common.cuh"
#include "compact.cuh"
#include "icp_dev.cuh"
#include "kernels.h"
#include "linalg_dev.cuh"
#include "reduce.cuh"

namespace smb {
using namespace dev;
namespace {

constexpr int kNdtThreads = 128;
constexpr int kNdtSums = 44;   // score, 6 gradient, 36 hessian, neighbour count

__host__ __device__ __forceinline__ int voxel_coord(float v, float inv_leaf, int min_b) {
  return (int)(floorf(v * inv_leaf) - (float)min_b);
}

// ---- grid parameters -------------------------------------------------------------------
// The size guard of VoxelGridCovariance::applyFilter (_impl.hpp:74-84): per axis int64 of the truncated float
// (max - min) * inv, plus 1; more than INT32_MAX voxels in the box and the int voxel index would wrap, two voxels
// could share a leaf.  The partial products are tested as they grow, so the test cannot overflow int64 either.
__host__ __device__ __forceinline__ int grid_too_large(const float* mn, const float* mx, float inv) {
  int64_t cells = 1;
  for (int d = 0; d < 3; ++d) {
    const float span = (mx[d] - mn[d]) * inv;
    if (!(span < 2147483648.0f)) return 1;
    cells *= (int64_t)span + 1;
    if (cells > 2147483647) return 1;
  }
  return 0;
}

__global__ void __launch_bounds__(256)
ndt_minmax_partial_kernel(const float* __restrict__ pts, int n, float* __restrict__ partial) {
  float mn[3] = {3.402823466e38f, 3.402823466e38f, 3.402823466e38f};
  float mx[3] = {-3.402823466e38f, -3.402823466e38f, -3.402823466e38f};
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256)
    for (int d = 0; d < 3; ++d) { const float v = pts[3 * (int64_t)i + d]; mn[d] = fminf(mn[d], v); mx[d] = fmaxf(mx[d], v); }
  const float2 r = block_minmax3<256>(mn, mx);
  if (threadIdx.x < 3) {
    partial[blockIdx.x * 6 + threadIdx.x] = r.x;
    partial[blockIdx.x * 6 + 3 + threadIdx.x] = r.y;
  }
}

__global__ void __launch_bounds__(256)
ndt_grid_params_kernel(const float* __restrict__ partial, int nparts, float resolution, NdtGrid* __restrict__ grid) {
  float mn[3] = {3.402823466e38f, 3.402823466e38f, 3.402823466e38f};
  float mx[3] = {-3.402823466e38f, -3.402823466e38f, -3.402823466e38f};
  for (int b = threadIdx.x; b < nparts; b += 256)
    for (int d = 0; d < 3; ++d) { mn[d] = fminf(mn[d], partial[b * 6 + d]); mx[d] = fmaxf(mx[d], partial[b * 6 + 3 + d]); }
  __shared__ float2 box[3];
  const float2 r = block_minmax3<256>(mn, mx);
  if (threadIdx.x < 3) box[threadIdx.x] = r;
  __syncthreads();
  if (threadIdx.x != 0) return;
  for (int d = 0; d < 3; ++d) { mn[d] = box[d].x; mx[d] = box[d].y; }
  const float inv = 1.0f / resolution;
  grid->inv_leaf = inv;
  grid->overflow = grid_too_large(mn, mx, inv);
  for (int d = 0; d < 3; ++d) {   // _impl.hpp:88-97
    grid->min_b[d] = (int)floorf(mn[d] * inv);
    const int max_b = (int)floorf(mx[d] * inv);
    grid->div_b[d] = max_b - grid->min_b[d] + 1;
  }
  grid->mul[0] = 1; grid->mul[1] = grid->div_b[0]; grid->mul[2] = grid->div_b[0] * grid->div_b[1];
}

__global__ void ndt_key_kernel(const float* __restrict__ pts, int n, const NdtGrid* __restrict__ grid,
                               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const NdtGrid g = *grid;
  const int i0 = voxel_coord(pts[3 * (int64_t)i], g.inv_leaf, g.min_b[0]);
  const int i1 = voxel_coord(pts[3 * (int64_t)i + 1], g.inv_leaf, g.min_b[1]);
  const int i2 = voxel_coord(pts[3 * (int64_t)i + 2], g.inv_leaf, g.min_b[2]);
  keys[i] = (uint64_t)(uint32_t)(i0 * g.mul[0] + i1 * g.mul[1] + i2 * g.mul[2]);
  vals[i] = (uint32_t)i;
}

// ---- voxel segments ------------------------------------------------------------------------
__device__ __forceinline__ uint32_t is_head(const uint64_t* keys, int i) {
  return (i == 0 || keys[i] != keys[i - 1]) ? 1u : 0u;
}

__global__ void __launch_bounds__(kCompactThreads)
ndt_heads_count_kernel(const uint64_t* __restrict__ keys, int n, uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += is_head(keys, base + r);
  tile_count_store(c, tile_cnt);
}

__global__ void __launch_bounds__(kCompactThreads)
ndt_heads_scatter_kernel(const uint64_t* __restrict__ keys, int n, const uint32_t* __restrict__ tile_off,
                         uint32_t* __restrict__ voxel_start, int* __restrict__ voxel_key,
                         NdtGrid* __restrict__ grid) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n) ? is_head(keys, base + r) : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r)
    if (f[r]) { voxel_start[pos] = (uint32_t)(base + r); voxel_key[pos] = (int)keys[base + r]; ++pos; }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint32_t v = tile_off[gridDim.x];
    grid->n_voxels = (int)v;
    voxel_start[v] = (uint32_t)n;   // sentinel
  }
}

// ---- per-voxel statistics (_impl.hpp:226-237, 283-366) --------------------------------------
__host__ __device__ __forceinline__ void inverse3_cofactor(const double* m, double* inv) {
  const double c00 = m[4] * m[8] - m[5] * m[7];
  const double c10 = m[5] * m[6] - m[3] * m[8];
  const double c20 = m[3] * m[7] - m[4] * m[6];
  const double det = (c00 * m[0] + c10 * m[1]) + c20 * m[2];
  const double invdet = 1.0 / det;
  inv[0] = c00 * invdet; inv[3] = c10 * invdet; inv[6] = c20 * invdet;
  inv[1] = (m[7] * m[2] - m[8] * m[1]) * invdet;
  inv[4] = (m[8] * m[0] - m[6] * m[2]) * invdet;
  inv[7] = (m[6] * m[1] - m[7] * m[0]) * invdet;
  inv[2] = (m[1] * m[5] - m[2] * m[4]) * invdet;
  inv[5] = (m[2] * m[3] - m[0] * m[5]) * invdet;
  inv[8] = (m[0] * m[4] - m[1] * m[3]) * invdet;
}

__global__ void ndt_gather_kernel(const float* __restrict__ pts, const uint32_t* __restrict__ order, int n,
                                  float* __restrict__ sorted) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t i = order[k];
  sorted[3 * (int64_t)k] = pts[3 * (int64_t)i];
  sorted[3 * (int64_t)k + 1] = pts[3 * (int64_t)i + 1];
  sorted[3 * (int64_t)k + 2] = pts[3 * (int64_t)i + 2];
}

// pts: the target points ALREADY in voxel order (ndt_gather_kernel), so a voxel is a contiguous run
// Second pass of applyFilter for one leaf (voxel_grid_covariance_omp_impl.hpp:283-366) from its running sums: sum x,
// cov = I + sum x x^T (Leaf() starts cov_ as identity), float centroid sum, point count.  __host__ too: the test hook
// sm_debug_ndt_leaf runs this very function.
__host__ __device__ __forceinline__ void finish_leaf(int n, const double* sum, const double* cov, const float* cen,
                                                     int min_points, double eig_mult, NdtLeaf* out_p) {
  NdtLeaf& out = *out_p;
  out.pad = 0;
  out.nr_points = n; out.searchable = 0;
  for (int k = 0; k < 9; ++k) out.icov[k] = 0.0;
  for (int d = 0; d < 3; ++d) { out.centroid[d] = cen[d] / (float)n; out.mean[d] = sum[d] / (double)n; }
  if (n >= min_points) {
    out.searchable = 1;
    double cv[9];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c)
        cv[r * 3 + c] = (cov[r * 3 + c] - 2 * (sum[r] * out.mean[c])) / (double)n + out.mean[r] * out.mean[c];
    const double scale = (n - 1.0) / n;
    for (int k = 0; k < 9; ++k) cv[k] *= scale;
    double w[3], V[9];
    la::jacobi_eig_sym(cv, 3, w, V);
    int ord[3] = {0, 1, 2};
    for (int a = 0; a < 3; ++a)
      for (int b = a + 1; b < 3; ++b)
        if (w[ord[b]] < w[ord[a]]) { const int t = ord[a]; ord[a] = ord[b]; ord[b] = t; }
    double ev[3], E[9];
    for (int a = 0; a < 3; ++a) {
      ev[a] = w[ord[a]];
      for (int r = 0; r < 3; ++r) E[r * 3 + a] = V[r * 3 + ord[a]];
    }
    if (ev[0] < 0 || ev[1] < 0 || ev[2] <= 0) {
      out.nr_points = -1;
    } else {
      const double min_ev = eig_mult * ev[2];
      if (ev[0] < min_ev) {
        ev[0] = min_ev;
        if (ev[1] < min_ev) ev[1] = min_ev;
        double Einv[9], ED[9];
        inverse3_cofactor(E, Einv);
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c) ED[r * 3 + c] = E[r * 3 + c] * ev[c];
        for (int r = 0; r < 3; ++r)
          for (int c = 0; c < 3; ++c)
            cv[r * 3 + c] = (ED[r * 3 + 0] * Einv[0 * 3 + c] + ED[r * 3 + 1] * Einv[1 * 3 + c]) + ED[r * 3 + 2] * Einv[2 * 3 + c];
      }
      inverse3_cofactor(cv, out.icov);
      const double inf = (double)INFINITY;
      double mx = -inf, mn = inf;
      for (int k = 0; k < 9; ++k) { mx = fmax(mx, out.icov[k]); mn = fmin(mn, out.icov[k]); }
      if (mx == inf || mn == -inf) out.nr_points = -1;
    }
  }
}

__global__ void ndt_leaf_kernel(const float* __restrict__ pts, const uint32_t* __restrict__ order,
                                const uint32_t* __restrict__ voxel_start, const NdtGrid* __restrict__ grid,
                                NdtLeaf* __restrict__ leaves, int min_points, double eig_mult) {
  // One WARP per voxel.  The 12 running sums of a leaf (sum x: 3, upper triangle of sum x x^T: 6,
  // float centroid: 3) are 12 independent serial chains that must add the voxel's points in
  // original order to round like the reference's serial loop.  Per batch of 32 points:
  //   phase 1 (all lanes, one point each): the 9 double addends (x*1 and the products are formed
  //            exactly like the serial code: (double)x_r * (double)x_c) go to shared memory,
  //            transposed to [chain][point];
  //   phase 2 (lane j owns chain j): 32 shared loads that do not depend on the chain, then the
  //            32 dependent adds — the serial cost per point is one DADD latency.
  // A dense voxel (tens of thousands of points next to the sensor) therefore costs ~10 cycles per
  // point instead of one thread's ~40 dependent FP64 operations.
  constexpr int kWarps = 8, kPad = 33;
  __shared__ double s_d[kWarps][9 * kPad];
  __shared__ float s_f[kWarps][3 * kPad];
  const int v = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  if (v >= grid->n_voxels) return;   // whole warps leave together
  const uint32_t s0 = voxel_start[v], s1 = voxel_start[v + 1];
  const int n = (int)(s1 - s0);
  double* sd = s_d[wib];
  float* sf = s_f[wib];
  // chain of the lane: 0..2 sum x_d, 3..8 sum x_r x_c for (r,c) = (0,0)(0,1)(0,2)(1,1)(1,2)(2,2);
  // lanes 9..11 carry the float centroid of x_{lane-9}; the clamps keep the other lanes on valid
  // (ignored) chains so the loop is branch-free
  const int dch = min(lane, 8), fch = (lane >= 9 && lane < 12) ? lane - 9 : 0;
  const double* my_d = sd + dch * kPad;
  const float* my_f = sf + fch * kPad;
  double accd = (lane == 3 || lane == 6 || lane == 8) ? 1.0 : 0.0;   // Leaf::cov_ starts as identity
  float accf = 0.0f;
  auto fetch = [&](uint32_t base, float& x, float& y, float& z) {
    const uint32_t i = min(base + (uint32_t)lane, s1 - 1);
    x = pts[3 * (int64_t)i]; y = pts[3 * (int64_t)i + 1]; z = pts[3 * (int64_t)i + 2];
  };
  float cx, cy, cz, nx = 0.f, ny = 0.f, nz = 0.f;
  fetch(s0, cx, cy, cz);
  for (uint32_t base = s0; base < s1; base += 32) {
    if (base + 32 < s1) fetch(base + 32, nx, ny, nz);
    const int cnt = (int)min(32u, s1 - base);
    {
      const double dx = (double)cx, dy = (double)cy, dz = (double)cz;
      sd[0 * kPad + lane] = dx; sd[1 * kPad + lane] = dy; sd[2 * kPad + lane] = dz;
      sd[3 * kPad + lane] = dx * dx; sd[4 * kPad + lane] = dx * dy; sd[5 * kPad + lane] = dx * dz;
      sd[6 * kPad + lane] = dy * dy; sd[7 * kPad + lane] = dy * dz; sd[8 * kPad + lane] = dz * dz;
      sf[0 * kPad + lane] = cx; sf[1 * kPad + lane] = cy; sf[2 * kPad + lane] = cz;
    }
    __syncwarp();
    if (cnt == 32) {
      double td[32]; float tf[32];
#pragma unroll
      for (int u = 0; u < 32; ++u) { td[u] = my_d[u]; tf[u] = my_f[u]; }
#pragma unroll
      for (int u = 0; u < 32; ++u) { accd += td[u]; accf += tf[u]; }
    } else {
      for (int u = 0; u < cnt; ++u) { accd += my_d[u]; accf += my_f[u]; }
    }
    __syncwarp();
    cx = nx; cy = ny; cz = nz;
  }
  double sum[3], cov[9];
  float cen[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) { sum[d] = __shfl_sync(0xffffffffu, accd, d); cen[d] = __shfl_sync(0xffffffffu, accf, 9 + d); }
#pragma unroll
  for (int j = 0; j < 6; ++j) {
    const double c = __shfl_sync(0xffffffffu, accd, 3 + j);
    const int r = j < 3 ? 0 : (j < 5 ? 1 : 2), cc = j < 3 ? j : (j < 5 ? j - 2 : 2);
    cov[r * 3 + cc] = c; cov[cc * 3 + r] = c;   // x_r * x_c == x_c * x_r bit for bit
  }
  if (lane != 0) return;
  NdtLeaf out;
  finish_leaf(n, sum, cov, cen, min_points, eig_mult, &out);
  leaves[v] = out;
}

// ---- hash table: voxel index -> leaf slot (searchable leaves only) --------------------------
__device__ __forceinline__ uint32_t hash_voxel(int key) {
  uint32_t h = (uint32_t)key * 2654435761u;
  return h ^ (h >> 15);
}

__global__ void ndt_hash_insert_kernel(const int* __restrict__ voxel_key, const NdtLeaf* __restrict__ leaves,
                                       const NdtGrid* __restrict__ grid, int* __restrict__ table_key,
                                       int* __restrict__ table_val, uint32_t table_mask) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= grid->n_voxels || !leaves[v].searchable) return;
  const int key = voxel_key[v];
  uint32_t h = hash_voxel(key) & table_mask;
  for (uint32_t probes = 0; probes <= table_mask; ++probes) {
    const int prev = atomicCAS(&table_key[h], -1, key);
    if (prev == -1 || prev == key) { table_val[h] = v; return; }
    h = (h + 1) & table_mask;
  }
}

__device__ __forceinline__ int hash_lookup(const int* __restrict__ table_key, const int* __restrict__ table_val,
                                           uint32_t mask, int key) {
  uint32_t h = hash_voxel(key) & mask;
  for (uint32_t probes = 0; probes <= mask; ++probes) {   // bounded: never spins on a bad table
    const int k = __ldg(table_key + h);
    if (k == key) return __ldg(table_val + h);
    if (k == -1) return -1;
    h = (h + 1) & mask;
  }
  return -1;
}

// ---- direct neighbour searches (pclomp DIRECT26 / DIRECT7 / DIRECT1) ------------------------
constexpr int kMinPointsPerVoxel = 6;   // min_points_per_voxel_ (voxel_grid_covariance_omp.h)

// Offset k of the method's list (voxel_grid_covariance_omp_impl.hpp:405-441).  DIRECT26 is
// pcl::getAllNeighborCellIndices() of stock PCL, which is not vendored; restated from upstream PCL: the 13 "half"
// offsets (i, j, -1) for i = -1..1, j = -1..1 (i outer), (i, -1, 0) for i = -1..1, (-1, 0, 0), then those 13
// negated.  It holds no (0, 0, 0): DIRECT26 never visits the query's own cell.
template <int kSearch>
__host__ __device__ __forceinline__ void direct_offset(int k, int* o) {
  if (kSearch == kNdtDirect26) {
    const int h = k < 13 ? k : k - 13, s = k < 13 ? 1 : -1;
    if (h < 9) { o[0] = h / 3 - 1; o[1] = h % 3 - 1; o[2] = -1; }
    else if (h < 12) { o[0] = h - 10; o[1] = -1; o[2] = 0; }
    else { o[0] = -1; o[1] = 0; o[2] = 0; }
    o[0] *= s; o[1] *= s; o[2] *= s;
  } else {   // DIRECT7: (0,0,0), (+1,0,0), (-1,0,0), (0,+1,0), (0,-1,0), (0,0,+1), (0,0,-1); DIRECT1: k = 0 only
    o[0] = o[1] = o[2] = 0;
    if (k > 0) o[(k - 1) / 2] = (k & 1) ? 1 : -1;
  }
}

// VoxelGridCovariance::getNeighborhoodAtPoint (voxel_grid_covariance_omp_impl.hpp:373-403) up to the leaf test:
// visit(key) for each offset cell of point x that lies in the grid's box, in list order, key = the cell's leaf
// index ((ijk + d - min_b) . divb_mul, the index build_grid gives it).  The caller keeps a cell whose leaf exists and
// has nr_points >= 6 (:394-395), so a leaf that failed the eigenvalue test (nr_points = -1) is never a neighbour
// here, while the KDTREE search keeps it with icov = 0.
// ijk = int(floor(x / leaf_size)), a float DIVISION (:379-381): the grid build multiplies by 1 / leaf_size, and the
// two disagree for points on or near a cell face when the resolution is not a power of two.
// Undefined input: the reference's static_cast<int> of a non-finite or out-of-range floor is undefined behaviour.
// Here a point has no neighbour when floor(x / leaf) is not finite or outside [min_b - 1, max_b + 1] on some axis.
// Wherever the reference is defined this is its result (no offset in {-1, 0, 1} reaches the box from there), and
// ijk + d cannot overflow.
template <int kSearch, class Visit>
__host__ __device__ __forceinline__ void for_each_direct_cell(const float* x, float leaf, const NdtGrid& g,
                                                              Visit visit) {
  int rel[3];
  for (int d = 0; d < 3; ++d) {
    const float f = floorf(x[d] / leaf);
    const double lo = (double)g.min_b[d] - 1.0, hi = (double)g.min_b[d] + (double)g.div_b[d];   // max_b + 1
    if (!((double)f >= lo && (double)f <= hi)) return;
    rel[d] = (int)f - g.min_b[d];
  }
  const int count = kSearch == kNdtDirect26 ? 26 : (kSearch == kNdtDirect7 ? 7 : 1);
#pragma unroll 1
  for (int k = 0; k < count; ++k) {
    int o[3];
    direct_offset<kSearch>(k, o);
    const int a = rel[0] + o[0], b = rel[1] + o[1], c = rel[2] + o[2];
    if (a < 0 || b < 0 || c < 0 || a >= g.div_b[0] || b >= g.div_b[1] || c >= g.div_b[2]) continue;
    visit(a * g.mul[0] + b * g.mul[1] + c * g.mul[2]);
  }
}

// ---- derivatives ----------------------------------------------------------------------------
__device__ __forceinline__ float dist2f(float qx, float qy, float qz, const float* c) {
  const float dx = qx - c[0], dy = qy - c[1], dz = qz - c[2];
  return (dx * dx + dy * dy) + dz * dz;
}

// one (point, voxel) term: computePointDerivatives (float overload, ndt_omp_impl.hpp:397-438)
// + updateDerivatives (:483-535); operation order as written out in oracle/ndt_math.h
__host__ __device__ __forceinline__ double update_derivatives(const NdtEvalParams& P, const float* x_orig,
                                                     const float* x_trans_f, const NdtLeaf& leaf,
                                                     double* grad_pt, double* hess_pt) {
  float xj[8], xh[15];
#pragma unroll
  for (int r = 0; r < 8; ++r) xj[r] = (P.j_ang[r][0] * x_orig[0] + P.j_ang[r][1] * x_orig[1]) + P.j_ang[r][2] * x_orig[2];
#pragma unroll
  for (int r = 0; r < 15; ++r) xh[r] = (P.h_ang[r][0] * x_orig[0] + P.h_ang[r][1] * x_orig[1]) + P.h_ang[r][2] * x_orig[2];
  const float pg[3][6] = {{1, 0, 0, 0, xj[2], xj[5]}, {0, 1, 0, xj[0], xj[3], xj[6]}, {0, 0, 1, xj[1], xj[4], xj[7]}};
  float xt[3], ci[3][3], xc[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) xt[d] = (float)((double)x_trans_f[d] - leaf.mean[d]);
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) ci[r][c] = (float)leaf.icov[r * 3 + c];
#pragma unroll
  for (int c = 0; c < 3; ++c) xc[c] = (xt[0] * ci[0][c] + xt[1] * ci[1][c]) + xt[2] * ci[2][c];
  const float q = (xt[0] * xc[0] + xt[1] * xc[1]) + xt[2] * xc[2];
  const float d2f = (float)P.gauss_d2;
  // expf of the reference (std::exp(float), glibc) and the double exp rounded to float differ by one
  // float ulp in about 7 of 10 000 terms of a lidar scene (tests/test_gpu_ndt_gicp_stages.py finds them)
  float e = (float)exp((double)(((-d2f) * q) * 0.5f));
  const float score_inc = (float)(-P.gauss_d1 * (double)e);
  e = d2f * e;
  if (e > 1 || e < 0 || e != e) return 0.0;
  e = (float)((double)e * P.gauss_d1);
  float cg[3][6], xg[6];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) cg[r][c] = (ci[r][0] * pg[0][c] + ci[r][1] * pg[1][c]) + ci[r][2] * pg[2][c];
#pragma unroll
  for (int c = 0; c < 6; ++c) xg[c] = (xt[0] * cg[0][c] + xt[1] * cg[1][c]) + xt[2] * cg[2][c];
#pragma unroll
  for (int c = 0; c < 6; ++c) grad_pt[c] += (double)(e * xg[c]);
#pragma unroll
  for (int i = 0; i < 6; ++i) {
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      float hrow = 0.0f;
      if (i >= 3 && j >= 3) {
        // point_hessian block (i, j): a..f of eq. 6.21, symmetric table {a,b,c; b,d,e; c,e,f}
        const int a = i - 3, b = j - 3;
        const int lo = a < b ? a : b, hi = a < b ? b : a;
        const int blk = lo == 0 ? hi : (lo == 1 ? 2 + hi : 5);        // 0:a 1:b 2:c 3:d 4:e 5:f
        float v0, v1, v2;
        if (blk < 3) { v0 = 0.0f; v1 = xh[2 * blk]; v2 = xh[2 * blk + 1]; }
        else { v0 = xh[6 + 3 * (blk - 3)]; v1 = xh[7 + 3 * (blk - 3)]; v2 = xh[8 + 3 * (blk - 3)]; }
        hrow = (xc[0] * v0 + xc[1] * v1) + xc[2] * v2;
      }
      const float gg = (pg[0][j] * cg[0][i] + pg[1][j] * cg[1][i]) + pg[2][j] * cg[2][i];
      hess_pt[i * 6 + j] += (double)(e * ((((-d2f) * xg[i]) * xg[j] + hrow) + gg));
    }
  }
  return (double)score_inc;
}

// the same term with double Eigen matrices: stock pcl::NormalDistributionsTransform
// (computePointDerivatives / updateDerivatives of PCL's ndt.hpp; the in-tree double overloads
// ndt_omp_impl.hpp:441-481 and updateHessian :596-629 are that code).  Used by NdtWithGicp.
__host__ __device__ __forceinline__ double update_derivatives_f64(const NdtEvalParams& P, const float* x_orig,
                                                         const float* x_trans_f, const NdtLeaf& leaf,
                                                         double* grad_pt, double* hess_pt) {
  const double x[3] = {(double)x_orig[0], (double)x_orig[1], (double)x_orig[2]};
  double xj[8], xh[15];
#pragma unroll
  for (int r = 0; r < 8; ++r) xj[r] = (x[0] * P.j_ang_d[r][0] + x[1] * P.j_ang_d[r][1]) + x[2] * P.j_ang_d[r][2];
#pragma unroll
  for (int r = 0; r < 15; ++r) xh[r] = (x[0] * P.h_ang_d[r][0] + x[1] * P.h_ang_d[r][1]) + x[2] * P.h_ang_d[r][2];
  const double pg[3][6] = {{1, 0, 0, 0, xj[2], xj[5]}, {0, 1, 0, xj[0], xj[3], xj[6]}, {0, 0, 1, xj[1], xj[4], xj[7]}};
  const double* ic = leaf.icov;
  double xt[3], cx[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) xt[d] = (double)x_trans_f[d] - leaf.mean[d];
#pragma unroll
  for (int r = 0; r < 3; ++r) cx[r] = (ic[r * 3] * xt[0] + ic[r * 3 + 1] * xt[1]) + ic[r * 3 + 2] * xt[2];
  double e = exp(-P.gauss_d2 * ((xt[0] * cx[0] + xt[1] * cx[1]) + xt[2] * cx[2]) / 2);
  const double score_inc = -P.gauss_d1 * e;
  e = P.gauss_d2 * e;
  if (e > 1 || e < 0 || e != e) return 0.0;
  e *= P.gauss_d1;
  double cdp[6][3], xdot[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
#pragma unroll
    for (int r = 0; r < 3; ++r) cdp[i][r] = (ic[r * 3] * pg[0][i] + ic[r * 3 + 1] * pg[1][i]) + ic[r * 3 + 2] * pg[2][i];
    xdot[i] = (xt[0] * cdp[i][0] + xt[1] * cdp[i][1]) + xt[2] * cdp[i][2];
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    grad_pt[i] += xdot[i] * e;
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      double hterm = 0.0;
      if (i >= 3 && j >= 3) {
        const int a = i - 3, b = j - 3;
        const int lo = a < b ? a : b, hi = a < b ? b : a;
        const int blk = lo == 0 ? hi : (lo == 1 ? 2 + hi : 5);
        double v0, v1, v2;
        if (blk < 3) { v0 = 0.0; v1 = xh[2 * blk]; v2 = xh[2 * blk + 1]; }
        else { v0 = xh[6 + 3 * (blk - 3)]; v1 = xh[7 + 3 * (blk - 3)]; v2 = xh[8 + 3 * (blk - 3)]; }
        double cv[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) cv[r] = (ic[r * 3] * v0 + ic[r * 3 + 1] * v1) + ic[r * 3 + 2] * v2;
        hterm = (xt[0] * cv[0] + xt[1] * cv[1]) + xt[2] * cv[2];
      }
      const double gdot = (pg[0][j] * cdp[i][0] + pg[1][j] * cdp[i][1]) + pg[2][j] * cdp[i][2];
      hess_pt[i * 6 + j] += e * ((-P.gauss_d2 * xdot[i] * xdot[j] + hterm) + gdot);
    }
  }
  return score_inc;
}

// kSearch: pclomp's neighbour search (ndt_omp_impl.hpp:233-246); KDTREE is the radius search the reference selects
template <int kSearch>
__global__ void __launch_bounds__(kNdtThreads)
ndt_derivatives_kernel(const float* __restrict__ src, int n, NdtEvalParams P,
                       const NdtGrid* __restrict__ grid, const NdtLeaf* __restrict__ leaves,
                       const int* __restrict__ table_key, const int* __restrict__ table_val,
                       uint32_t table_mask, double* __restrict__ partials) {
  __shared__ double red[kNdtThreads / 32][kNdtSums];
  double acc[kNdtSums];
#pragma unroll
  for (int k = 0; k < kNdtSums; ++k) acc[k] = 0.0;
  const int i = blockIdx.x * kNdtThreads + threadIdx.x;
  if (kSearch != kNdtKdtree && i < n) {
    const NdtGrid g = *grid;
    const float xo[3] = {src[3 * (int64_t)i], src[3 * (int64_t)i + 1], src[3 * (int64_t)i + 2]};
    float xt[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) xt[r] = ((P.T[r] * xo[0] + P.T[r + 4] * xo[1]) + P.T[r + 8] * xo[2]) + P.T[r + 12];
    double score_pt = 0.0, grad_pt[6], hess_pt[36];
#pragma unroll
    for (int q = 0; q < 6; ++q) grad_pt[q] = 0.0;
#pragma unroll
    for (int q = 0; q < 36; ++q) hess_pt[q] = 0.0;
    int nc = 0;
    // neighbours in offset order, no distance test and no sort (voxel_grid_covariance_omp_impl.hpp:383-400)
    for_each_direct_cell<kSearch>(xt, P.radius, g, [&](int key) {
      const int v = hash_lookup(table_key, table_val, table_mask, key);   // the table holds leaves of >= 6 points
      if (v < 0) return;
      const NdtLeaf leaf = leaves[v];
      if (leaf.nr_points < kMinPointsPerVoxel) return;                     // nr_points = -1: failed covariance
      ++nc;
      score_pt += P.f64_math ? update_derivatives_f64(P, xo, xt, leaf, grad_pt, hess_pt)
                             : update_derivatives(P, xo, xt, leaf, grad_pt, hess_pt);
    });
    acc[0] = score_pt;
#pragma unroll
    for (int q = 0; q < 6; ++q) acc[1 + q] = grad_pt[q];
#pragma unroll
    for (int q = 0; q < 36; ++q) acc[7 + q] = hess_pt[q];
    acc[43] = (double)nc;
  }
  if (kSearch == kNdtKdtree && i < n) {
    const NdtGrid g = *grid;
    const float xo[3] = {src[3 * (int64_t)i], src[3 * (int64_t)i + 1], src[3 * (int64_t)i + 2]};
    float xt[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) xt[r] = ((P.T[r] * xo[0] + P.T[r + 4] * xo[1]) + P.T[r + 8] * xo[2]) + P.T[r + 12];
    const int c0 = voxel_coord(xt[0], g.inv_leaf, g.min_b[0]);
    const int c1 = voxel_coord(xt[1], g.inv_leaf, g.min_b[1]);
    const int c2 = voxel_coord(xt[2], g.inv_leaf, g.min_b[2]);
    const float r2 = P.radius * P.radius;
    float cd[27];
    int cv[27], ck[27], nc = 0;
    for (int dz = -1; dz <= 1; ++dz)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dx = -1; dx <= 1; ++dx) {
          const int a = c0 + dx, b = c1 + dy, c = c2 + dz;
          if (a < 0 || b < 0 || c < 0 || a >= g.div_b[0] || b >= g.div_b[1] || c >= g.div_b[2]) continue;
          const int key = a * g.mul[0] + b * g.mul[1] + c * g.mul[2];
          const int v = hash_lookup(table_key, table_val, table_mask, key);
          if (v < 0) continue;
          const float d = dist2f(xt[0], xt[1], xt[2], leaves[v].centroid);
          if (d < r2) { cd[nc] = d; cv[nc] = v; ck[nc] = key; ++nc; }
        }
    // FLANN returns the neighbours sorted by distance; ties by voxel index
    for (int a = 1; a < nc; ++a) {
      const float d = cd[a]; const int v = cv[a], k = ck[a];
      int b = a - 1;
      while (b >= 0 && (cd[b] > d || (cd[b] == d && ck[b] > k))) { cd[b + 1] = cd[b]; cv[b + 1] = cv[b]; ck[b + 1] = ck[b]; --b; }
      cd[b + 1] = d; cv[b + 1] = v; ck[b + 1] = k;
    }
    double score_pt = 0.0, grad_pt[6], hess_pt[36];
#pragma unroll
    for (int q = 0; q < 6; ++q) grad_pt[q] = 0.0;
#pragma unroll
    for (int q = 0; q < 36; ++q) hess_pt[q] = 0.0;
    for (int j = 0; j < nc; ++j) {
      const NdtLeaf leaf = leaves[cv[j]];
      score_pt += P.f64_math ? update_derivatives_f64(P, xo, xt, leaf, grad_pt, hess_pt)
                             : update_derivatives(P, xo, xt, leaf, grad_pt, hess_pt);
    }
    acc[0] = score_pt;
#pragma unroll
    for (int q = 0; q < 6; ++q) acc[1 + q] = grad_pt[q];
#pragma unroll
    for (int q = 0; q < 36; ++q) acc[7 + q] = hess_pt[q];
    acc[43] = (double)nc;
  }
  const double v = block_sum<kNdtSums, kNdtThreads>(acc, red);
  if (threadIdx.x < kNdtSums) partials[(int64_t)blockIdx.x * kNdtSums + threadIdx.x] = v;
}

__global__ void __launch_bounds__(1024)
ndt_reduce_kernel(const double* __restrict__ partials, int nblocks, int width, double* __restrict__ out) {
  for (int k = threadIdx.x >> 5; k < width; k += 32) {
    const double v = warp_sum_rows(partials, nblocks, width, k);
    if ((threadIdx.x & 31) == 0) out[k] = v;
  }
}

// ---- fitness score ----------------------------------------------------------------------------
__global__ void ndt_float_to_soa_kernel(const float* __restrict__ pts, int n, double* __restrict__ soa,
                                        int64_t stride) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  soa[i] = (double)pts[3 * (int64_t)i];
  soa[stride + i] = (double)pts[3 * (int64_t)i + 1];
  soa[2 * stride + i] = (double)pts[3 * (int64_t)i + 2];
}

__global__ void __launch_bounds__(256)
ndt_fitness_kernel(const float* __restrict__ src, int n, NdtEvalParams P, const KdNode* __restrict__ nodes,
                   const BucketPoint* __restrict__ bpts, const float* __restrict__ tgt,
                   double* __restrict__ partials) {
  __shared__ double red[8][2];
  const int i = blockIdx.x * 256 + threadIdx.x;
  double sc[2] = {0.0, 0.0};   // squared distance, match count
  if (i < n) {
    const float xo[3] = {src[3 * (int64_t)i], src[3 * (int64_t)i + 1], src[3 * (int64_t)i + 2]};
    float xt[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) xt[r] = ((P.T[r] * xo[0] + P.T[r + 4] * xo[1]) + P.T[r + 8] * xo[2]) + P.T[r + 12];
    int slot; double d2;
    knn1(nodes, bpts, (double)xt[0], (double)xt[1], (double)xt[2], 1.0, slot, d2);
    if (slot >= 0) {
      const long long id = bpts[slot].id;
      sc[0] = (double)dist2f(xt[0], xt[1], xt[2], tgt + 3 * id);
      sc[1] = 1.0;
    }
  }
  const double v = block_sum<2, 256>(sc, red);
  if (threadIdx.x < 2) partials[(int64_t)blockIdx.x * 2 + threadIdx.x] = v;
}

}  // namespace

// host build of the per-axis voxel coordinate of the NDT grid (test hook sm_debug_voxel_index op 1)
int ndt_debug_voxel_coord_host(float v, float inv_leaf, int min_b) { return voxel_coord(v, inv_leaf, min_b); }

// host build of the direct searches' cell walk (test hook sm_debug_ndt_direct_neighbors)
int ndt_debug_direct_cells_host(int search, const float* x, float leaf, const NdtGrid& g, int* keys26) {
  int m = 0;
  auto keep = [&](int key) { keys26[m++] = key; };
  if (search == kNdtDirect26) for_each_direct_cell<kNdtDirect26>(x, leaf, g, keep);
  else if (search == kNdtDirect7) for_each_direct_cell<kNdtDirect7>(x, leaf, g, keep);
  else if (search == kNdtDirect1) for_each_direct_cell<kNdtDirect1>(x, leaf, g, keep);
  return m;
}
bool ndt_debug_direct_leaf_accepted_host(int nr_points) { return nr_points >= kMinPointsPerVoxel; }

// Host build of one leaf of the target grid (test hook sm_debug_ndt_leaf): the running sums are formed here in input
// order (the kernel forms them with one warp per voxel, in the same order), the rest is finish_leaf.
void ndt_debug_leaf_host(const float* pts, int n, int min_points, double eig_mult, double* mean3, double* icov9,
                         float* centroid3, int* nr_points, int* searchable) {
  double sum[3] = {0, 0, 0}, cov[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  float cen[3] = {0, 0, 0};
  for (int i = 0; i < n; ++i) {
    const double x[3] = {(double)pts[3 * i], (double)pts[3 * i + 1], (double)pts[3 * i + 2]};
    for (int r = 0; r < 3; ++r) {
      sum[r] += x[r];
      cen[r] += pts[3 * i + r];
      for (int c = 0; c < 3; ++c) cov[r * 3 + c] += x[r] * x[c];
    }
  }
  NdtLeaf leaf;
  finish_leaf(n, sum, cov, cen, min_points, eig_mult, &leaf);
  for (int d = 0; d < 3; ++d) { mean3[d] = leaf.mean[d]; centroid3[d] = leaf.centroid[d]; }
  for (int q = 0; q < 9; ++q) icov9[q] = leaf.icov[q];
  *nr_points = leaf.nr_points;
  *searchable = leaf.searchable;
}

// Host build of the per-(point, voxel) term (test hook sm_debug_ndt_term): out[0] = score increment,
// out[1..6] = gradient term, out[7..42] = Hessian term (row-major) of ONE neighbour voxel.
void ndt_debug_term_host(const NdtEvalParams& P, const float* x_orig, const float* x_trans, const double* mean,
                         const double* icov, double* out43) {
  NdtLeaf leaf;
  for (int d = 0; d < 3; ++d) { leaf.mean[d] = mean[d]; leaf.centroid[d] = (float)mean[d]; }
  for (int q = 0; q < 9; ++q) leaf.icov[q] = icov[q];
  leaf.nr_points = 6; leaf.searchable = 1; leaf.pad = 0;
  for (int q = 0; q < 43; ++q) out43[q] = 0.0;
  out43[0] = P.f64_math ? update_derivatives_f64(P, x_orig, x_trans, leaf, out43 + 1, out43 + 7)
                        : update_derivatives(P, x_orig, x_trans, leaf, out43 + 1, out43 + 7);
}

static int ndt_blocks(int n) { return ceil_div(n, kNdtThreads); }

static uint32_t ndt_table_size(int nt) {
  uint32_t s = 1024;
  while (s < 2u * (uint32_t)(nt > 0 ? nt : 1)) s <<= 1;   // voxels <= points; load factor <= 0.5
  return s;
}

static size_t workspace_bytes(int nt, int ns) {
  const int64_t st = (nt + 63) & ~63;
  size_t b = 0;
  b += 2 * st * sizeof(uint64_t) + 2 * st * sizeof(uint32_t);              // keys / order ping-pong
  b += radix_sort_scratch_bytes(nt, 1) + 4096;                              // scratch + block sums
  b += (st + 64) * sizeof(uint32_t) + st * sizeof(int);                     // voxel_start, voxel_key
  b += st * sizeof(NdtLeaf);                                                // leaves (<= nt voxels)
  b += 2 * (size_t)ndt_table_size(nt) * sizeof(int);                        // hash table
  b += (size_t)(ndt_blocks(ns) + 8) * kNdtSums * sizeof(double) + 64 * sizeof(double);
  b += 1024 * 6 * sizeof(float) + sizeof(NdtGrid) + 4096;
  b += 3 * st * sizeof(float) + 256;                                          // sorted_pts
  return b + 8192;
}

int NdtStage::reserve(int nt, int ns) {
  SMB_RC(buf.reserve(workspace_bytes(nt, ns)));
  const int64_t st = (nt + 63) & ~63;
  char* p = (char*)buf.p;
  auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) & ~(size_t)255; return r; };
  ws.stride = st;
  ws.keys[0] = (uint64_t*)take(st * sizeof(uint64_t)); ws.keys[1] = (uint64_t*)take(st * sizeof(uint64_t));
  ws.order[0] = (uint32_t*)take(st * sizeof(uint32_t)); ws.order[1] = (uint32_t*)take(st * sizeof(uint32_t));
  ws.scratch = (uint32_t*)take(radix_sort_scratch_bytes(nt, 1) + 4096);
  ws.voxel_start = (uint32_t*)take((st + 64) * sizeof(uint32_t));
  ws.voxel_key = (int*)take(st * sizeof(int));
  ws.leaves = (NdtLeaf*)take(st * sizeof(NdtLeaf));
  ws.table_size = ndt_table_size(nt);
  ws.table_key = (int*)take((size_t)ws.table_size * sizeof(int));
  ws.table_val = (int*)take((size_t)ws.table_size * sizeof(int));
  ws.partials = (double*)take((size_t)(ndt_blocks(ns) + 8) * kNdtSums * sizeof(double));
  ws.sums = (double*)take(64 * sizeof(double));
  ws.minmax = (float*)take(1024 * 6 * sizeof(float));
  ws.sorted_pts = (float*)take(3 * st * sizeof(float));
  ws.grid = (NdtGrid*)take(sizeof(NdtGrid));
  return 0;
}

// VoxelGridCovariance::filter(true) for the target (ndt_omp.h:117-122,271-278)
int NdtStage::build_grid(const float* tgt, int nt, float resolution, cudaStream_t stream) {
  const int nparts = nt < 256 * 512 ? ceil_div(nt, 256) : 512;
  ndt_minmax_partial_kernel<<<nparts, 256, 0, stream>>>(tgt, nt, ws.minmax);
  ndt_grid_params_kernel<<<1, 256, 0, stream>>>(ws.minmax, nparts, resolution, ws.grid);
  ndt_key_kernel<<<ceil_div(nt, 256), 256, 0, stream>>>(tgt, nt, ws.grid, ws.keys[0], ws.order[0]);
  int rc = radix_sort_pairs_u64(ws.keys[0], ws.order[0], ws.keys[1], ws.order[1], nt, 1, ws.stride,
                                ws.scratch, stream, 4);
  if (rc) return rc;
  const int tiles = compact_tiles(nt);
  ndt_heads_count_kernel<<<tiles, kCompactThreads, 0, stream>>>(ws.keys[0], nt, ws.scratch);
  compact_scan(ws.scratch, tiles, stream);
  ndt_heads_scatter_kernel<<<tiles, kCompactThreads, 0, stream>>>(ws.keys[0], nt, ws.scratch, ws.voxel_start,
                                                                 ws.voxel_key, ws.grid);
  // one warp per voxel; the voxel count is only known on the device, so launch for nt warps
  ndt_gather_kernel<<<ceil_div(nt, 256), 256, 0, stream>>>(tgt, ws.order[0], nt, ws.sorted_pts);
  ndt_leaf_kernel<<<ceil_div((int64_t)nt * 32, 256), 256, 0, stream>>>(ws.sorted_pts, ws.order[0], ws.voxel_start,
                                                                      ws.grid, ws.leaves, 6, 0.01);
  SMB_CUDA_OK(cudaMemsetAsync(ws.table_key, 0xff, (size_t)ws.table_size * sizeof(int), stream));
  ndt_hash_insert_kernel<<<ceil_div(nt, 256), 256, 0, stream>>>(ws.voxel_key, ws.leaves, ws.grid, ws.table_key,
                                                               ws.table_val, ws.table_size - 1);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

// computeDerivatives: out[44] = score, gradient, hessian (row-major), neighbour count
int NdtStage::eval(const float* src, int ns, const NdtEvalParams& P, int search, double* sums44,
                   cudaStream_t stream) {
  const int nb = ndt_blocks(ns);
  auto kernel = search == kNdtDirect26 ? ndt_derivatives_kernel<kNdtDirect26>
              : search == kNdtDirect7  ? ndt_derivatives_kernel<kNdtDirect7>
              : search == kNdtDirect1  ? ndt_derivatives_kernel<kNdtDirect1>
                                       : ndt_derivatives_kernel<kNdtKdtree>;
  kernel<<<nb, kNdtThreads, 0, stream>>>(src, ns, P, ws.grid, ws.leaves, ws.table_key, ws.table_val,
                                         ws.table_size - 1, ws.partials);
  ndt_reduce_kernel<<<1, 1024, 0, stream>>>(ws.partials, nb, kNdtSums, ws.sums);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(sums44, ws.sums, kNdtSums * sizeof(double), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

int ndt_float_to_soa(const float* pts, int n, double* soa, int64_t stride, cudaStream_t stream) {
  ndt_float_to_soa_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(pts, n, soa, stride);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

// getFitnessScore: the mean over the matched points of the squared NN distance (float each); sums2 stages the sum
// and the count
int NdtStage::fitness(const float* src, int ns, const float* tgt, const float* T, const FloatTree& t, double* sums2,
                      cudaStream_t stream, double* score) {
  NdtEvalParams P;
  memset(&P, 0, sizeof(P));
  for (int i = 0; i < 16; ++i) P.T[i] = T[i];
  const int nb = ceil_div(ns, 256);
  ndt_fitness_kernel<<<nb, 256, 0, stream>>>(src, ns, P, (const KdNode*)t.nodes.p, (const BucketPoint*)t.bpts.p, tgt,
                                            ws.partials);
  ndt_reduce_kernel<<<1, 1024, 0, stream>>>(ws.partials, nb, 2, ws.sums);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(sums2, ws.sums, 2 * sizeof(double), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  *score = sums2[1] > 0.0 ? sums2[0] / sums2[1] : std::numeric_limits<double>::max();
  return 0;
}
int NdtStage::fitness_launches(int nt) { return 24 + kd_num_levels(nt, 8) * 5 + 6; }

}  // namespace smb
