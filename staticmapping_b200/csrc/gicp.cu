// registrator::NdtWithGicp on the device (registrators/ndt_gicp.cc:28-112).  The arithmetic is
// stock PCL (external); the in-tree statement of the GICP math is the vendored
// registrators/pclomp/gicp_omp_impl.hpp, cited per kernel.
//
//   approx_*            pcl::ApproximateVoxelGrid::applyFilter (ndt_gicp.cc:59-70).  The reference
//                       algorithm is a single sequential pass over a 512-slot hash history; its
//                       slots are independent streams, so: stable sort by slot -> runs of equal
//                       voxel inside a slot -> one centroid per run (float sum in original order)
//                       -> runs ordered by the index of the point that evicts them (the order in
//                       which the sequential pass emits them), never-evicted runs last in slot order.
//   gicp_knn20_cov      computeCovariances (gicp_omp_impl.hpp:59-131): exact 20-NN in the cloud's
//                       own k-d tree, covariance, eigen-regularisation (1, 1, 1e-3).
//   gicp_correspond     the per-point part of computeTransformation (:430-461): exact 1-NN of the
//                       moved source point, distance gate, Mahalanobis matrix (R C1 R^T + C2)^-1.
//   gicp_cost           OptimizationFunctorWithIndices::fdf (:341-377): f, translation gradient and
//                       the 3x3 matrix R that computeRDerivative contracts; 13 double sums.
// Compiled with -fmad=false (same operation order as oracle/gicp_oracle.cc).
#include "common.cuh"
#include "compact.cuh"
#include "gicp_host.h"
#include "icp_dev.cuh"
#include "kernels.h"
#include "linalg_dev.cuh"
#include "reduce.cuh"

namespace smb {
using namespace dev;
namespace {

// ---- ApproximateVoxelGrid -------------------------------------------------------------------
constexpr int kHist = 512;

__host__ __device__ __forceinline__ void approx_cell(const float* p, float inv, int* ix, int* iy, int* iz, uint32_t* slot) {
  *ix = (int)floorf(p[0] * inv); *iy = (int)floorf(p[1] * inv); *iz = (int)floorf(p[2] * inv);
  *slot = (uint32_t)((*ix * 7171 + *iy * 3079 + *iz * 4231) & (kHist - 1));
}

__global__ void approx_key_kernel(const float* __restrict__ pts, int n, float inv, uint64_t* __restrict__ keys,
                                  uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int ix, iy, iz; uint32_t slot;
  approx_cell(pts + 3 * (int64_t)i, inv, &ix, &iy, &iz, &slot);
  keys[i] = slot;
  vals[i] = (uint32_t)i;
}

// position k of the slot-sorted order starts a run iff its slot or voxel differs from k-1
__device__ __forceinline__ uint32_t run_head(const float* pts, const uint32_t* order, const uint64_t* keys,
                                             float inv, int k) {
  if (k == 0 || keys[k] != keys[k - 1]) return 1u;
  int ax, ay, az, bx, by, bz; uint32_t s;
  approx_cell(pts + 3 * (int64_t)order[k], inv, &ax, &ay, &az, &s);
  approx_cell(pts + 3 * (int64_t)order[k - 1], inv, &bx, &by, &bz, &s);
  return (ax != bx || ay != by || az != bz) ? 1u : 0u;
}

__global__ void __launch_bounds__(kCompactThreads)
approx_heads_count_kernel(const float* __restrict__ pts, const uint32_t* __restrict__ order,
                          const uint64_t* __restrict__ keys, int n, float inv, uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += run_head(pts, order, keys, inv, base + r);
  tile_count_store(c, tile_cnt);
}

__global__ void __launch_bounds__(kCompactThreads)
approx_heads_scatter_kernel(const float* __restrict__ pts, const uint32_t* __restrict__ order,
                            const uint64_t* __restrict__ keys, int n, float inv,
                            const uint32_t* __restrict__ tile_off, uint32_t* __restrict__ run_start,
                            uint32_t* __restrict__ n_runs) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    f[r] = (base + r < n) ? run_head(pts, order, keys, inv, base + r) : 0u;
    c += f[r];
  }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) if (f[r]) run_start[pos++] = (uint32_t)(base + r);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const uint32_t v = tile_off[gridDim.x];
    *n_runs = v;
    run_start[v] = (uint32_t)n;
  }
}

// one thread per run: float centroid in original order + the emission key of the run
__global__ void approx_run_kernel(const float* __restrict__ pts, const uint32_t* __restrict__ order,
                                  const uint64_t* __restrict__ keys, const uint32_t* __restrict__ run_start,
                                  const uint32_t* __restrict__ n_runs, int n, float* __restrict__ centroid,
                                  uint64_t* __restrict__ emit_key, uint32_t* __restrict__ emit_val) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_runs) return;
  const uint32_t s0 = run_start[r], s1 = run_start[r + 1];
  float c[3] = {0.0f, 0.0f, 0.0f};
  for (uint32_t k = s0; k < s1; ++k) {
    const float* p = pts + 3 * (int64_t)order[k];
    c[0] += p[0]; c[1] += p[1]; c[2] += p[2];
  }
  const float cnt = (float)(s1 - s0);
  centroid[3 * (int64_t)r] = c[0] / cnt; centroid[3 * (int64_t)r + 1] = c[1] / cnt; centroid[3 * (int64_t)r + 2] = c[2] / cnt;
  // evicted by the first point of the next run of the same slot, else flushed at the end
  const bool evicted = (s1 < (uint32_t)n) && keys[s1] == keys[s0];
  emit_key[r] = evicted ? (uint64_t)order[s1] : (uint64_t)n + keys[s0];
  emit_val[r] = r;
}

__global__ void approx_emit_kernel(const float* __restrict__ centroid, const uint32_t* __restrict__ emit_val,
                                   const uint32_t* __restrict__ n_runs, float* __restrict__ out) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= *n_runs) return;
  const uint32_t s = emit_val[r];
  out[3 * (int64_t)r] = centroid[3 * (int64_t)s];
  out[3 * (int64_t)r + 1] = centroid[3 * (int64_t)s + 1];
  out[3 * (int64_t)r + 2] = centroid[3 * (int64_t)s + 2];
}

// ---- exact k-NN (k = 20) + covariances ---------------------------------------------------------
constexpr int kK = 20;

__device__ __forceinline__ bool cand_less(double d, int id, double wd, int wid) { return d < wd || (d == wd && id < wid); }

__device__ __forceinline__ void knn_k(const KdNode* __restrict__ nodes, const BucketPoint* __restrict__ bpts,
                                      double qx, double qy, double qz, double* bd, int* bi, int* cnt_out) {
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  int cnt = 0, wpos = 0, worst_id = 0x7fffffff;
  double worst = inf;                 // (worst, worst_id): the maximum of the held set once kK are held
  StackEntry stack[kMaxStack];
  int sp = 0, idx = 0;
  double rd = 0.0, ox = 0.0, oy = 0.0, oz = 0.0;
  for (int rounds = 0; rounds < (1 << 20); ++rounds) {
    KdNode nd = load_node(nodes, idx);
    int guard = 0;
    while (nd.dim != 3 && ++guard < 64) {
      const int cd = nd.dim;
      const double q = cd == 0 ? qx : (cd == 1 ? qy : qz);
      const double old_off = cd == 0 ? ox : (cd == 1 ? oy : oz);
      const double new_off = dsub(q, nd.cut);
      const int right = new_off > 0.0 ? 1 : 0;
      const double rd_new = dadd(rd, dadd(-dmul(old_off, old_off), dmul(new_off, new_off)));
      if ((cnt < kK || rd_new <= worst) && sp < kMaxStack) {
        StackEntry e;
        e.rd = rd_new;
        e.ox = cd == 0 ? new_off : ox; e.oy = cd == 1 ? new_off : oy; e.oz = cd == 2 ? new_off : oz;
        e.idx = child_idx(idx, 1 - right);
        stack[sp++] = e;
      }
      idx = child_idx(idx, right);
      nd = load_node(nodes, idx);
    }
    if (nd.dim == 3) {
      const long long packed = __double_as_longlong(nd.cut);
      const int first = (int)(packed & 0xffffffffll), count = (int)(packed >> 32);
      for (int k = 0; k < count; ++k) {
        const BucketPoint p = bpts[first + k];
        const double dx = dsub(qx, p.x), dy = dsub(qy, p.y), dz = dsub(qz, p.z);
        const double d = dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz));
        const int id = (int)p.id;
        // the held set is UNSORTED with its maximum tracked (worst, wpos): a candidate costs one compare,
        // an accepted one a 20-entry rescan — no shifting of a sorted list through local memory
        if (cnt < kK) {
          bd[cnt] = d; bi[cnt] = id; ++cnt;
          if (cnt == kK) {
            worst = bd[0]; worst_id = bi[0]; wpos = 0;
            for (int j = 1; j < kK; ++j) if (cand_less(worst, worst_id, bd[j], bi[j])) { worst = bd[j]; worst_id = bi[j]; wpos = j; }
          }
        } else if (cand_less(d, id, worst, worst_id)) {
          bd[wpos] = d; bi[wpos] = id;
          worst = bd[0]; worst_id = bi[0]; wpos = 0;
          for (int j = 1; j < kK; ++j) if (cand_less(worst, worst_id, bd[j], bi[j])) { worst = bd[j]; worst_id = bi[j]; wpos = j; }
        }
      }
    }
    bool found = false;
    while (sp > 0) {
      const StackEntry e = stack[--sp];
      if (cnt < kK || e.rd <= worst) { idx = e.idx; rd = e.rd; ox = e.ox; oy = e.oy; oz = e.oz; found = true; break; }
    }
    if (!found) break;
  }
  for (int a = 1; a < cnt; ++a) {     // ascending (d, id): the order the covariance sums are formed in
    const double d = bd[a]; const int id = bi[a];
    int b = a - 1;
    while (b >= 0 && cand_less(d, id, bd[b], bi[b])) { bd[b + 1] = bd[b]; bi[b + 1] = bi[b]; --b; }
    bd[b + 1] = d; bi[b + 1] = id;
  }
  *cnt_out = cnt;
}

__global__ void __launch_bounds__(64)
gicp_knn20_cov_kernel(const float* __restrict__ cloud, int n, const KdNode* __restrict__ nodes,
                      const BucketPoint* __restrict__ bpts, double eps, double* __restrict__ covs) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  // queries in the tree's own leaf order: the lanes of a warp are neighbours in space, walk the same
  // nodes and scan the same buckets (the cloud's input order is the voxel filter's eviction order)
  const int i = (int)bpts[t].id;
  double bd[kK]; int bi[kK]; int cnt;
  knn_k(nodes, bpts, (double)cloud[3 * (int64_t)i], (double)cloud[3 * (int64_t)i + 1], (double)cloud[3 * (int64_t)i + 2],
        bd, bi, &cnt);
  double mean[3] = {0, 0, 0}, cov[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < kK; ++j) {   // gicp_omp_impl.hpp:91-106 (float products, double sums)
    const float* pt = cloud + 3 * (int64_t)(j < cnt ? bi[j] : i);
    mean[0] += pt[0]; mean[1] += pt[1]; mean[2] += pt[2];
    cov[0] += pt[0] * pt[0];
    cov[3] += pt[1] * pt[0]; cov[4] += pt[1] * pt[1];
    cov[6] += pt[2] * pt[0]; cov[7] += pt[2] * pt[1]; cov[8] += pt[2] * pt[2];
  }
  for (int d = 0; d < 3; ++d) mean[d] /= (double)kK;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b <= a; ++b) {
      cov[a * 3 + b] /= (double)kK;
      cov[a * 3 + b] -= mean[a] * mean[b];
      cov[b * 3 + a] = cov[a * 3 + b];
    }
  double w[3], V[9];
  la::jacobi_eig_sym(cov, 3, w, V);
  int ord[3] = {0, 1, 2};
  for (int a = 0; a < 3; ++a)
    for (int b = a + 1; b < 3; ++b)
      if (fabs(w[ord[b]]) > fabs(w[ord[a]])) { const int t = ord[a]; ord[a] = ord[b]; ord[b] = t; }
  double out[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int kk = 0; kk < 3; ++kk) {   // :118-129: singular values -> (1, 1, gicp_epsilon)
    const double v = (kk == 2) ? eps : 1.0;
    const double col[3] = {V[0 * 3 + ord[kk]], V[1 * 3 + ord[kk]], V[2 * 3 + ord[kk]]};
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) out[r * 3 + c] += v * col[r] * col[c];
  }
  for (int q = 0; q < 9; ++q) covs[9 * (int64_t)i + q] = out[q];
}

// ---- correspondences + Mahalanobis ---------------------------------------------------------------
__host__ __device__ __forceinline__ void mulpt_f(const float* T, const float* p, float* out) {
#pragma unroll
  for (int r = 0; r < 3; ++r) out[r] = ((T[r] * p[0] + T[r + 4] * p[1]) + T[r + 8] * p[2]) + T[r + 12] * 1.0f;
}

__host__ __device__ __forceinline__ void inverse3(const double* m, double* inv) {
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

// M_i = (R C1 R^T + C2)^-1 (gicp_omp_impl.hpp:450-457); R row-major.  __host__ too (test hook sm_debug_gicp_point).
__host__ __device__ __forceinline__ void mahalanobis(const double* R, const double* C1, const double* C2, double* out) {
  double M[9], tmp[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      M[r * 3 + c] = (R[r * 3] * C1[c] + R[r * 3 + 1] * C1[3 + c]) + R[r * 3 + 2] * C1[6 + c];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c)
      tmp[r * 3 + c] = ((M[r * 3] * R[c * 3] + M[r * 3 + 1] * R[c * 3 + 1]) + M[r * 3 + 2] * R[c * 3 + 2]) + C2[r * 3 + c];
  inverse3(tmp, out);
}

__global__ void __launch_bounds__(128)
gicp_correspond_kernel(const float* __restrict__ src, int ns, const float* __restrict__ tgt, GicpIterParams P,
                       const KdNode* __restrict__ nodes, const BucketPoint* __restrict__ bpts,
                       const double* __restrict__ cov_s, const double* __restrict__ cov_t,
                       int32_t* __restrict__ match, double* __restrict__ maha, uint32_t* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (i < ns) {
    float q1[3], q[3];
    mulpt_f(P.guess, src + 3 * (int64_t)i, q1);          // gicp_omp_impl.hpp:437-439
    mulpt_f(P.transformation, q1, q);
    int slot; double d2;
    knn1(nodes, bpts, (double)q[0], (double)q[1], (double)q[2], 1.0, slot, d2);
    int j = -1;
    if (slot >= 0) {
      j = (int)bpts[slot].id;
      const float* t = tgt + 3 * (int64_t)j;
      const float dx = q[0] - t[0], dy = q[1] - t[1], dz = q[2] - t[2];
      const float d = (dx * dx + dy * dy) + dz * dz;
      if ((double)d < P.dist_threshold) {                // :448
        mahalanobis(P.R, cov_s + 9 * (int64_t)i, cov_t + 9 * (int64_t)j, maha + 9 * (int64_t)i);
        valid = true;
      }
    }
    match[i] = valid ? j : -1;
  }
  const uint32_t m = __ballot_sync(0xffffffffu, valid);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(count, (uint32_t)__popc(m));
}

// ---- cost / gradient ------------------------------------------------------------------------------
constexpr int kCostSums = 13;

// one correspondence of OptimizationFunctorWithIndices (gicp_omp_impl.hpp:341-377): acc[0] = res^T M res,
// acc[1..3] = M res, acc[4..12] = (base p)(M res)^T row-major.  __host__ too (test hook sm_debug_gicp_point).
__host__ __device__ __forceinline__ void cost_terms(const float* T, const float* base, const float* ps, const float* pt,
                                                    const double* M, double* acc) {
  float pp[3], pb[3];
  mulpt_f(T, ps, pp);
  const double res[3] = {(double)(pp[0] - pt[0]), (double)(pp[1] - pt[1]), (double)(pp[2] - pt[2])};
  double temp[3];
  for (int r = 0; r < 3; ++r) temp[r] = (M[r * 3] * res[0] + M[r * 3 + 1] * res[1]) + M[r * 3 + 2] * res[2];
  acc[0] = (res[0] * temp[0] + res[1] * temp[1]) + res[2] * temp[2];
  for (int r = 0; r < 3; ++r) acc[1 + r] = temp[r];
  mulpt_f(base, ps, pb);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) acc[4 + r * 3 + c] = (double)pb[r] * temp[c];
}

__global__ void __launch_bounds__(256)
gicp_cost_kernel(const float* __restrict__ src, int ns, const float* __restrict__ tgt, GicpCostParams P,
                 const int32_t* __restrict__ match, const double* __restrict__ maha, double* __restrict__ partials,
                 double* __restrict__ sums, uint32_t* __restrict__ ticket, double* __restrict__ host_sums,
                 volatile long long* __restrict__ host_flag, long long seq) {
  __shared__ double red[8][kCostSums];
  __shared__ bool is_last;
  double acc[kCostSums];
#pragma unroll
  for (int k = 0; k < kCostSums; ++k) acc[k] = 0.0;
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i < ns) {
    const int j = match[i];
    if (j >= 0) {
      cost_terms(P.T, P.base, src + 3 * (int64_t)i, tgt + 3 * (int64_t)j, maha + 9 * (int64_t)i, acc);
    }
  }
  const double v = block_sum<kCostSums, 256>(acc, red);
  if (threadIdx.x < kCostSums) partials[(int64_t)blockIdx.x * kCostSums + threadIdx.x] = v;
  // The block that finishes last reduces the partial sums (fixed order: the same tree whichever block
  // it is) and hands the 13 results to the host through mapped pinned memory: one launch and no copy per
  // BFGS evaluation (31 per alignment) instead of two launches, a copy and a stream synchronisation.
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  for (int k = threadIdx.x >> 5; k < kCostSums; k += 8) {
    const double v = warp_sum_rows(reinterpret_cast<volatile const double*>(partials), (int)gridDim.x, kCostSums, k);
    if ((threadIdx.x & 31) == 0) { sums[k] = v; if (host_sums) host_sums[k] = v; }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *ticket = 0;                                   // ready for the next evaluation
    if (host_flag) { __threadfence_system(); *host_flag = seq; }
  }
}

// test hook sm_debug_float_tree_knn: the two searches over a FloatTree that have no kernel of their own, one query
// per thread.  k = 1: knn1 with eps = 0 (ndt_fitness_kernel, gicp_correspond_kernel); k = kK: knn_k
// (gicp_knn20_cov_kernel).  Row i of ids / d2 holds k entries; knn_k's unused ones are -1 / +inf.
__global__ void debug_float_tree_knn_kernel(const KdNode* __restrict__ nodes, const BucketPoint* __restrict__ bpts,
                                            const double* __restrict__ q, int nq, int k, int32_t* __restrict__ ids,
                                            double* __restrict__ d2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nq) return;
  const double qx = q[3 * (int64_t)i], qy = q[3 * (int64_t)i + 1], qz = q[3 * (int64_t)i + 2];
  if (k == 1) {
    int slot; double d;
    knn1(nodes, bpts, qx, qy, qz, 1.0, slot, d);
    ids[i] = slot >= 0 ? (int32_t)bpts[slot].id : -1;
    d2[i] = d;
    return;
  }
  double bd[kK]; int bi[kK]; int cnt;
  knn_k(nodes, bpts, qx, qy, qz, bd, bi, &cnt);
  for (int j = 0; j < kK; ++j) {
    ids[(int64_t)i * kK + j] = j < cnt ? bi[j] : -1;
    d2[(int64_t)i * kK + j] = j < cnt ? bd[j] : __longlong_as_double(0x7ff0000000000000ll);
  }
}

}  // namespace

int float_tree_debug_knn(const FloatTree& t, const double* q, int nq, int k, int32_t* ids, double* d2,
                         cudaStream_t stream) {
  if (k != 1 && k != kK) return -1;
  if (nq <= 0) return 0;
  debug_float_tree_knn_kernel<<<ceil_div(nq, 64), 64, 0, stream>>>((const KdNode*)t.nodes.p,
                                                                  (const BucketPoint*)t.bpts.p, q, nq, k, ids, d2);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

// host build of ApproximateVoxelGrid's cell and hash slot of one point (test hook sm_debug_voxel_index op 2)
void gicp_debug_approx_cell_host(const float* p, float inv, int* ixyz, uint32_t* slot) {
  approx_cell(p, inv, &ixyz[0], &ixyz[1], &ixyz[2], slot);
}

// host builds of the per-point GICP arithmetic (test hook sm_debug_gicp_point)
void gicp_debug_mahalanobis_host(const double* R, const double* C1, const double* C2, double* out9) {
  mahalanobis(R, C1, C2, out9);
}
void gicp_debug_cost_terms_host(const float* T, const float* base, const float* ps, const float* pt, const double* M,
                                double* acc13) {
  cost_terms(T, base, ps, pt, M, acc13);
}

// pcl::ApproximateVoxelGrid::filter: keys, runs and centroids, then (with the run count on the host to size the
// sort) the runs in emission order
int ApproxVoxelGrid::filter(const float* pts, int n, float leaf, DevBuf& out, int* m_out, cudaStream_t stream) {
  const int64_t st = (n + 63) & ~63;
  SMB_RC(ws.reserve((size_t)(4 * st * sizeof(uint64_t) + 4 * st * sizeof(uint32_t) + (st + 64) * sizeof(uint32_t) +
                             3 * st * sizeof(float) + radix_sort_scratch_bytes(n, 1) + 8192)));
  SMB_RC(out.reserve((size_t)n * 12 + 64));
  SMB_RC(counter.reserve(64));
  uint32_t* n_out_dev = (uint32_t*)counter.p;
  char* p = (char*)ws.p;
  auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) & ~(size_t)255; return r; };
  uint64_t* keys0 = (uint64_t*)take(st * 8); uint64_t* keys1 = (uint64_t*)take(st * 8);
  uint64_t* ekey0 = (uint64_t*)take(st * 8); uint64_t* ekey1 = (uint64_t*)take(st * 8);
  uint32_t* ord0 = (uint32_t*)take(st * 4); uint32_t* ord1 = (uint32_t*)take(st * 4);
  uint32_t* eval0 = (uint32_t*)take(st * 4); uint32_t* eval1 = (uint32_t*)take(st * 4);
  uint32_t* run_start = (uint32_t*)take((st + 64) * 4);
  float* centroid = (float*)take(3 * st * 4);
  uint32_t* scratch = (uint32_t*)take(radix_sort_scratch_bytes(n, 1) + 4096);
  const float inv = 1.0f / leaf;
  approx_key_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(pts, n, inv, keys0, ord0);
  SMB_RC(radix_sort_pairs_u64(keys0, ord0, keys1, ord1, n, 1, st, scratch, stream, 2));
  const int tiles = compact_tiles(n);
  approx_heads_count_kernel<<<tiles, kCompactThreads, 0, stream>>>(pts, ord0, keys0, n, inv, scratch);
  compact_scan(scratch, tiles, stream);
  approx_heads_scatter_kernel<<<tiles, kCompactThreads, 0, stream>>>(pts, ord0, keys0, n, inv, scratch, run_start, n_out_dev);
  approx_run_kernel<<<ceil_div(n, 128), 128, 0, stream>>>(pts, ord0, keys0, run_start, n_out_dev, n, centroid, ekey0, eval0);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t m = 0;
  SMB_CUDA_OK(cudaMemcpyAsync(&m, n_out_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  *m_out = (int)m;
  if (m == 0) return 0;
  SMB_RC(radix_sort_pairs_u64(ekey0, eval0, ekey1, eval1, (int)m, 1, st, scratch, stream, 4));
  approx_emit_kernel<<<ceil_div(m, 256), 256, 0, stream>>>(centroid, eval0, n_out_dev, (float*)out.p);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

static int cost_blocks(int ns) { return ceil_div(ns, 256); }

int gicp::Stage::reserve(int ns, int nt, cudaStream_t stream) {
  SMB_RC(cov_s.reserve((size_t)ns * 9 * sizeof(double)));
  SMB_RC(cov_t.reserve((size_t)nt * 9 * sizeof(double)));
  SMB_RC(maha.reserve((size_t)ns * 9 * sizeof(double)));
  SMB_RC(match.reserve((size_t)ns * sizeof(int32_t)));
  SMB_RC(partials.reserve((size_t)(cost_blocks(ns) + 1) * kCostSums * sizeof(double) + 256));
  SMB_RC(counter.reserve(64));
  sums = (double*)partials.p + (size_t)cost_blocks(ns) * kCostSums;
  ticket = (uint32_t*)counter.p + 8;
  SMB_CUDA_OK(cudaMemsetAsync(ticket, 0, sizeof(uint32_t), stream));
  seq = 0;
  return 0;
}

int gicp::Stage::covariances(const gicp::Options& o, const float* cloud, int n, const FloatTree& t, const DevBuf& out,
                             cudaStream_t stream) const {
  if (o.k_correspondences > n) {   // gicp_omp_impl.hpp:61-65: PCL_ERROR and the covariances stay unset
    SMB_CUDA_OK(cudaMemsetAsync(out.p, 0, (size_t)n * 9 * sizeof(double), stream));
    return 0;
  }
  gicp_knn20_cov_kernel<<<ceil_div(n, 64), 64, 0, stream>>>(cloud, n, (const KdNode*)t.nodes.p,
                                                           (const BucketPoint*)t.bpts.p, o.gicp_epsilon,
                                                           (double*)out.p);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

int gicp::Stage::correspond(const gicp::Options& o, const float* src, int ns, const float* tgt, const FloatTree& tt,
                            const float* guess, const float* transformation, const double* R, cudaStream_t stream,
                            int* m) {
  GicpIterParams P;
  for (int i = 0; i < 16; ++i) { P.guess[i] = guess[i]; P.transformation[i] = transformation[i]; }
  for (int q = 0; q < 9; ++q) P.R[q] = R[q];
  P.dist_threshold = o.corr_dist_threshold * o.corr_dist_threshold;
  uint32_t* count = (uint32_t*)counter.p;
  SMB_CUDA_OK(cudaMemsetAsync(count, 0, sizeof(uint32_t), stream));
  gicp_correspond_kernel<<<ceil_div(ns, 128), 128, 0, stream>>>(src, ns, tgt, P, (const KdNode*)tt.nodes.p,
                                                               (const BucketPoint*)tt.bpts.p, (const double*)cov_s.p,
                                                               (const double*)cov_t.p, (int32_t*)match.p,
                                                               (double*)maha.p, count);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t mu = 0;
  SMB_CUDA_OK(cudaMemcpyAsync(&mu, count, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  *m = (int)mu;
  return 0;
}

int gicp::Stage::cost(const float* src, int ns, const float* tgt, const float* T, const float* base, double* host_sums,
                      long long* host_seq, cudaStream_t stream) {
  GicpCostParams P;
  for (int i = 0; i < 16; ++i) { P.T[i] = T[i]; P.base[i] = base[i]; }
  gicp_cost_kernel<<<cost_blocks(ns), 256, 0, stream>>>(src, ns, tgt, P, (const int32_t*)match.p, (const double*)maha.p,
                                                       (double*)partials.p, sums, ticket, host_sums, host_seq,
                                                       host_seq ? ++seq : 0);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace smb
