// RandomSamplerWithPlaneDetect (pre_processors/random_sample_with_plane_detect.h) with its PlaneDetector
// (pre_processors/plane_detector.h) on the device, behind its own handle (sm_plane_sampler_*), built on the
// record-filter core of record_filter.h.  The contract is the header comment of sm_plane_sampler_* in
// include/sm_b200.h; DESIGN §4l has the derivations.
//
// Reference: Filter copies the cloud when rate > 0.999999 (:80-83).  Otherwise Detect files the points under
// GroundRemoval's voxel keys, in the std::map order, and for every voxel of at least min points: iz <= 0 -> the z-range
// rule with threshold 0.2 (all its points are plane points or none); iz > 0 and at least 2 min points -> PCL's RANSAC
// plane fit with refinement, and the refined inliers are plane points iff their share is > 0.85.  The sampler then
// keeps every plane point and the non-plane point k (1-based) iff (float)s / (float)k < rate, s = those kept before.
// Here:
//   voxels   voxel_sort (ground_removal.cu): bounds, keys, stable radix sort, voxel starts
//   detect   one warp per voxel, grid-strided (ps_detect_warp_kernel): the size tests, the z-range rule and, up to
//            kPsWarpMax points, the RANSAC with the shuffled indices in shared memory.  Bigger RANSAC voxels go on a
//            list that ps_detect_cta_kernel works through one CTA per voxel, the shuffled indices in the voxel's slice
//            of a global scratch indexed by sorted position.  Either writes the plane flag of its points.
//   ratio    the non-plane points counted per tile and scanned (compact.cuh) give each one its rank k; ps_keep_kernel
//            evaluates the literal float test with s(k - 1) in closed form (ps_kept_before) and stores the keep counts
//   emit     filter_compact_records; the inliers, outliers and plane indices are three flag_list compactions
// One read-back, at the end.  Compiled with -fmad=false.
//
// RANSAC (SACSegmentation::segment on the voxel's points in input order): every voxel gets a new model seeded 12345u,
// so all of them read the same raw stream, std::mt19937(12345) >> 1, computed once per handle.  The draws, the
// shuffle and the sample test are serial (rank 0 of the group); the inlier counts of each hypothesis are shared by the
// group and added as integers; the float mean and covariance of the refinement are nine serial chains in inlier order,
// one per lane, over addends the group stages through shared memory (ndt_leaf_kernel's layout).
#include <float.h>
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <random>
#include <utility>
#include <vector>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"
#include "record_filter.h"
#include "reduce.cuh"

namespace smb {

// ---- one hypothesis, host and device (test hook sm_debug_plane_sampler_piece_host) ---------------------------------
// Eigen 3.3's SSE2 reduction of a 4-wide dot product or squared norm
__host__ __device__ __forceinline__ float ps_dot4(const float* a, float b0, float b1, float b2, float b3) {
  return (a[0] * b0 + a[2] * b2) + (a[1] * b1 + a[3] * b3);
}

// isSampleGood, and the same test in computeModelCoefficients: p1 - p0 over p2 - p0 per component
__host__ __device__ __forceinline__ bool ps_sample_good(const float* p0, const float* p1, const float* p2) {
  const float d0 = (p1[0] - p0[0]) / (p2[0] - p0[0]);
  const float d1 = (p1[1] - p0[1]) / (p2[1] - p0[1]);
  const float d2 = (p1[2] - p0[2]) / (p2[2] - p0[2]);
  return d0 != d1 || d2 != d1;
}

// computeModelCoefficients: the normalised cross product (a zero normal stays zero), then d = -n . p0
__host__ __device__ __forceinline__ void ps_model(const float* p0, const float* p1, const float* p2, float* c) {
  const float ax = p1[0] - p0[0], ay = p1[1] - p0[1], az = p1[2] - p0[2];
  const float bx = p2[0] - p0[0], by = p2[1] - p0[1], bz = p2[2] - p0[2];
  c[0] = ay * bz - az * by;
  c[1] = az * bx - ax * bz;
  c[2] = ax * by - ay * bx;
  c[3] = 0.f;
  const float z = ps_dot4(c, c[0], c[1], c[2], c[3]);
  if (z > 0.f) {
    const float s = sqrtf(z);
    c[0] /= s; c[1] /= s; c[2] /= s; c[3] /= s;
  }
  c[3] = -ps_dot4(c, p0[0], p0[1], p0[2], 1.f);
}

__host__ __device__ __forceinline__ float ps_distance(const float* c, const float* p) {
  return fabsf(ps_dot4(c, p[0], p[1], p[2], 1.f));
}

// countWithinDistance / selectWithinDistance: the float distance against the double threshold 0.1
__host__ __device__ __forceinline__ bool ps_inlier(const float* c, const float* p) {
  return (double)ps_distance(c, p) < 0.1;
}

__host__ __device__ __forceinline__ void ps_roots2(float b, float c, float* r) {
  r[0] = 0.f;
  float d = (float)((double)(b * b) - 4.0 * (double)c);
  if (d < 0.f) d = 0.f;
  const float sd = sqrtf(d);
  r[2] = 0.5f * (b + sd);
  r[1] = 0.5f * (b - sd);
}

// pcl::computeRoots; atan2, cos and sin in double on the float arguments, rounded to float (DESIGN §4l)
__host__ __device__ __forceinline__ void ps_roots(const float (&m)[3][3], float* r) {
  const float c0 = (((m[0][0] * m[1][1]) * m[2][2] + ((2.f * m[0][1]) * m[0][2]) * m[1][2]) -
                    (m[0][0] * m[1][2]) * m[1][2]) - (m[1][1] * m[0][2]) * m[0][2] - (m[2][2] * m[0][1]) * m[0][1];
  const float c1 = ((((m[0][0] * m[1][1] - m[0][1] * m[0][1]) + m[0][0] * m[2][2]) - m[0][2] * m[0][2]) +
                    m[1][1] * m[2][2]) - m[1][2] * m[1][2];
  const float c2 = (m[0][0] + m[1][1]) + m[2][2];
  if (fabsf(c0) < FLT_EPSILON) {
    ps_roots2(c2, c1, r);
    return;
  }
  const float s_inv3 = (float)(1.0 / 3.0);
  const float s_sqrt3 = sqrtf(3.f);
  const float c2_over_3 = c2 * s_inv3;
  float a_over_3 = (c1 - c2 * c2_over_3) * s_inv3;
  if (a_over_3 > 0.f) a_over_3 = 0.f;
  const float half_b = 0.5f * (c0 + c2_over_3 * ((2.f * c2_over_3) * c2_over_3 - c1));
  float q = half_b * half_b + (a_over_3 * a_over_3) * a_over_3;
  if (q > 0.f) q = 0.f;
  const float rho = sqrtf(-a_over_3);
  const float theta = (float)atan2((double)sqrtf(-q), (double)half_b) * s_inv3;
#ifdef __CUDA_ARCH__
  // theta is in [0, pi / 3]: cospi / sinpi of theta / pi need no Payne-Hanek reduction, whose array would live in
  // local memory; the quotient's rounding moves the result by less than a double ulp
  const float cos_theta = (float)cospi((double)theta / M_PI);
  const float sin_theta = (float)sinpi((double)theta / M_PI);
#else
  const float cos_theta = (float)cos((double)theta);
  const float sin_theta = (float)sin((double)theta);
#endif
  r[0] = c2_over_3 + (2.f * rho) * cos_theta;
  r[1] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  r[2] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  float t;
  if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  if (r[1] >= r[2]) {
    t = r[1]; r[1] = r[2]; r[2] = t;
    if (r[0] >= r[1]) { t = r[0]; r[0] = r[1]; r[1] = t; }
  }
  if (r[0] <= 0.f) ps_roots2(c2, c1, r);
}

__host__ __device__ __forceinline__ void ps_cross(const float* a, const float* b, float* r) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}

// pcl::eigen33: the eigenvector of the smallest eigenvalue of the symmetric m, from the longest row cross product
__host__ __device__ __forceinline__ void ps_eigen33(const float (&mat)[3][3], float* vec) {
  float scale = 0.f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) scale = fmaxf(scale, fabsf(mat[i][j]));
  if (scale <= FLT_MIN) scale = 1.f;
  float s[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) s[i][j] = mat[i][j] / scale;
  float roots[3];
  ps_roots(s, roots);
  for (int d = 0; d < 3; ++d) s[d][d] -= roots[0];
  float v[3][3], len[3];
  ps_cross(s[0], s[1], v[0]);
  ps_cross(s[0], s[2], v[1]);
  ps_cross(s[1], s[2], v[2]);
  for (int k = 0; k < 3; ++k) len[k] = v[k][0] * v[k][0] + (v[k][1] * v[k][1] + v[k][2] * v[k][2]);
  // the pick by selects, not by a run-time index, so that v stays in registers
  const bool p0 = len[0] >= len[1] && len[0] >= len[2], p1 = !p0 && len[1] >= len[0] && len[1] >= len[2];
  const float root = sqrtf(p0 ? len[0] : p1 ? len[1] : len[2]);
  for (int d = 0; d < 3; ++d) vec[d] = (p0 ? v[0][d] : p1 ? v[1][d] : v[2][d]) / root;
}

// optimizeModelCoefficients from computeMeanAndCovarianceMatrix's nine sums, already divided by the inlier count
__host__ __device__ __forceinline__ void ps_refine(const float* a, float* c) {
  float cov[3][3];
  cov[0][0] = a[0] - a[6] * a[6];
  cov[0][1] = a[1] - a[6] * a[7];
  cov[0][2] = a[2] - a[6] * a[8];
  cov[1][1] = a[3] - a[7] * a[7];
  cov[1][2] = a[4] - a[7] * a[8];
  cov[2][2] = a[5] - a[8] * a[8];
  cov[1][0] = cov[0][1];
  cov[2][0] = cov[0][2];
  cov[2][1] = cov[1][2];
  ps_eigen33(cov, c);
  c[3] = 0.f;
  c[3] = -ps_dot4(c, a[6], a[7], a[8], 1.f);
}

// RandomSampleConsensus::computeModel's k after a new best count (probability 0.99, a sample of 3)
__host__ __device__ __forceinline__ double ps_k(int best, int count) {
  const double w = (double)best * (1.0 / (double)count);
  double p = 1.0 - pow(w, 3.0);
  p = fmax(DBL_EPSILON, p);
  p = fmin(1.0 - DBL_EPSILON, p);
  return log(1.0 - 0.99) / log(p);
}

// ---- the ratio rule ----------------------------------------------------------------------------------------------
// The float test (float)s / (float)k < rate, for 0 <= s <= k <= 2^24 (exact in float), holds iff s / k < mid, or
// s / k == mid when pred is even, where pred = nextafterf(rate, 0) and mid = (pred + rate) / 2: the reals that round to
// a float below rate.  So the loop keeps point k iff s(k - 1) < mid k (<= with the tie), and by induction (DESIGN §4l)
//   s(k) = ceil(mid k), or floor(mid k) + 1 with the tie,   k >= 1.
// mid has 25 significant bits and k at most 25, so mid k is exact in double.  A NaN rate keeps nothing.
struct PsRatio {
  double mid;
  bool tie_le;
};

__host__ __device__ __forceinline__ PsRatio ps_ratio(float rate) {
  const float pred = nextafterf(rate, 0.f);
  uint32_t bits;
  memcpy(&bits, &pred, 4);
  return {((double)pred + (double)rate) * 0.5, (bits & 1u) == 0u};
}

// s(k): the number kept among the first k non-plane points
__host__ __device__ __forceinline__ uint32_t ps_kept_before(const PsRatio& r, uint32_t k) {
  if (k == 0) return 0u;
  const double t = r.mid * (double)k;
  if (!(t >= 0.0)) return 0u;
  return r.tie_le ? (uint32_t)floor(t) + 1u : (uint32_t)ceil(t);
}

// the reference's test for non-plane point k >= 1
__host__ __device__ __forceinline__ bool ps_keep(float rate, const PsRatio& r, uint32_t k) {
  return (float)ps_kept_before(r, k - 1) / (float)k < rate;
}

namespace {

constexpr int kPsWarpMax = 512;                 // voxels up to this size: one warp; bigger RANSAC voxels: one CTA
constexpr int kPsCtaThreads = 256;
constexpr int kPsWarpsPerBlock = 8;
constexpr int kPsDraws = 1000, kPsMaxIterations = 50, kPsMaxSkip = 500;
constexpr int kPsRndWords = 3 * kPsDraws * (kPsMaxIterations + 1);
constexpr float kPsGroundThreshold = 0.2f;
// meta[0..5]: voxel_sort's bounds; [8] records out, [9] inliers, [10] outliers, [11] plane points, [12] CTA voxels,
// [13] voxels
constexpr int kPsMeta = 14;

__device__ __forceinline__ const float* ps_point(const char* pts, int64_t stride, uint32_t i) {
  return reinterpret_cast<const float*>(pts + (int64_t)i * stride);
}

// the per-group shared state: the drawn sample and the covariance chains' staged addends
template <int NT>
struct PsShared {
  int sample[3];
  int ok;
  int red[NT / 32];
  float add[9][NT];
  uint8_t in[NT];
  float accu[9];
};

struct WarpGroup {
  static constexpr int kThreads = 32;
  __device__ int rank() const { return threadIdx.x & 31; }
  __device__ void sync() const { __syncwarp(); }
  template <int NT>
  __device__ int sum(int v, PsShared<NT>&) const { return (int)__reduce_add_sync(0xffffffffu, (unsigned)v); }
};

struct CtaGroup {
  static constexpr int kThreads = kPsCtaThreads;
  __device__ int rank() const { return threadIdx.x; }
  __device__ void sync() const { __syncthreads(); }
  template <int NT>
  __device__ int sum(int v, PsShared<NT>& sm) const {
    v = (int)__reduce_add_sync(0xffffffffu, (unsigned)v);
    if ((threadIdx.x & 31) == 0) sm.red[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
    for (int w = 0; w < NT / 32; ++w) t += sm.red[w];
    __syncthreads();
    return t;
  }
};

// the inliers of c among the voxel's points, counted by the group
template <class G, int NT>
__device__ __forceinline__ int ps_count(const G& g, PsShared<NT>& sm, const char* pts, int64_t stride,
                                        const uint32_t* ord, int count, const float* c) {
  int n = 0;
  for (int j = g.rank(); j < count; j += NT) n += ps_inlier(c, ps_point(pts, stride, ord[j])) ? 1 : 0;
  return g.sum(n, sm);
}

// SACSegmentation::segment with setOptimizeCoefficients(true) on the count points ord[0..count) (input order), by a
// group of NT threads; sh: count shuffled indices.  Writes the plane flags and the trace.
template <class G, typename Idx>
__device__ void ps_ransac(const G& g, PsShared<G::kThreads>& sm, Idx* sh, const char* pts, int64_t stride,
                          const uint32_t* ord, int count, const uint32_t* __restrict__ rnd, uint8_t* plane,
                          PsTrace* trace) {
  constexpr int NT = G::kThreads;
  const int r = g.rank();
  for (int j = r; j < count; j += NT) sh[j] = (Idx)j;
  g.sync();
  auto P = [&](int j) { return ps_point(pts, stride, ord[j]); };
  int it = 0, skipped = 0, best = -INT_MAX, cursor = 0;
  double k = 1.0;
  float bc[4] = {0.f, 0.f, 0.f, 0.f};
  while (it < k && skipped < kPsMaxSkip) {
    if (r == 0) {                                       // getSamples: up to 1000 draws of drawIndexSample
      int ok = 0;
      for (int d = 0; d < kPsDraws && !ok; ++d) {
        for (int i = 0; i < 3; ++i) {
          const int j = i + (int)(rnd[cursor++] % (uint32_t)(count - i));
          const Idx t = sh[i];
          sh[i] = sh[j];
          sh[j] = t;
        }
        ok = ps_sample_good(P(sh[0]), P(sh[1]), P(sh[2]));
      }
      sm.ok = ok;
      for (int i = 0; i < 3; ++i) sm.sample[i] = sh[i];
    }
    g.sync();
    const int ok = sm.ok, s0 = sm.sample[0], s1 = sm.sample[1], s2 = sm.sample[2];
    g.sync();
    if (!ok) break;                                     // an empty selection
    // computeModelCoefficients repeats the sample test, which passed: skipped stays 0
    float c[4];
    ps_model(P(s0), P(s1), P(s2), c);
    const int n_in = ps_count(g, sm, pts, stride, ord, count, c);
    if (n_in > best) {
      best = n_in;
      for (int i = 0; i < 4; ++i) bc[i] = c[i];
      k = ps_k(best, count);
    }
    ++it;
    if (it > kPsMaxIterations) break;
  }
  float rc[4] = {0.f, 0.f, 0.f, 0.f};
  int n_final = 0;
  if (best != -INT_MAX) {                               // a model was found
    for (int i = 0; i < 4; ++i) rc[i] = bc[i];
    const int n1 = ps_count(g, sm, pts, stride, ord, count, bc);
    if (n1 >= 4) {
      // computeMeanAndCovarianceMatrix: lane a < 9 adds the addends of sum a in inlier order
      float acc = 0.f;
      for (int base = 0; base < count; base += NT) {
        const int j = base + r;
        if (j < count) {
          const float* p = P(j);
          const float x = p[0], y = p[1], z = p[2];
          sm.in[r] = ps_inlier(bc, p) ? 1 : 0;
          sm.add[0][r] = x * x; sm.add[1][r] = x * y; sm.add[2][r] = x * z;
          sm.add[3][r] = y * y; sm.add[4][r] = y * z; sm.add[5][r] = z * z;
          sm.add[6][r] = x; sm.add[7][r] = y; sm.add[8][r] = z;
        }
        g.sync();
        if (r < 9) {
          const int m = min(NT, count - base);
          for (int t = 0; t < m; ++t)
            if (sm.in[t]) acc += sm.add[r][t];
        }
        g.sync();
      }
      if (r < 9) sm.accu[r] = acc / (float)n1;
      g.sync();
      float a[9];
      for (int i = 0; i < 9; ++i) a[i] = sm.accu[i];
      ps_refine(a, rc);
    }
    n_final = ps_count(g, sm, pts, stride, ord, count, rc);
  }
  const bool is_plane = (double)((float)n_final / (float)count) > 0.85;
  if (is_plane)
    for (int j = r; j < count; j += NT)
      if (ps_inlier(rc, P(j))) plane[ord[j]] = 1;
  if (trace && r == 0) {
    trace->status = is_plane ? kPsRansacPlane : kPsRansacNot;
    trace->iterations = it;
    trace->best = best;
    trace->final_count = n_final;
    for (int i = 0; i < 4; ++i) trace->coef[i] = rc[i];
  }
}

// one warp per voxel, grid-strided over the *n_voxels voxels; a RANSAC voxel of more than kPsWarpMax points goes on
// the CTA list
__global__ void __launch_bounds__(32 * kPsWarpsPerBlock)
ps_detect_warp_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ order,
                      const uint32_t* __restrict__ voxel_start, const uint32_t* __restrict__ n_voxels, float leaf,
                      uint64_t min_points, const uint32_t* __restrict__ rnd, uint8_t* __restrict__ plane,
                      uint32_t* __restrict__ cta_list, uint32_t* __restrict__ cta_count, PsTrace* __restrict__ trace) {
  __shared__ PsShared<32> shared[kPsWarpsPerBlock];
  __shared__ uint16_t shuffled[kPsWarpsPerBlock][kPsWarpMax];
  const WarpGroup g;
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * kPsWarpsPerBlock;
  const int64_t nv = *n_voxels;
  for (int64_t v = (int64_t)blockIdx.x * kPsWarpsPerBlock + w; v < nv; v += warps) {
    const uint32_t s0 = voxel_start[v], s1 = voxel_start[v + 1];
    const uint64_t count = s1 - s0;
    PsTrace* t = trace ? trace + v : nullptr;
    int ixyz[3];
    gr_index(ps_point(pts, stride, order[s0]), leaf, ixyz);
    int status = kPsSkipped;
    if (count < min_points) {
      status = kPsSkipped;
    } else if (ixyz[2] <= 0) {                          // the z-range rule (plane_detector.h:106-124)
      float max_z = -1.e9f, min_z = 1.e9f;
      for (uint32_t k = s0 + lane; k < s1; k += 32) {
        const float z = ps_point(pts, stride, order[k])[2];
        gr_z_update(z, z, &max_z, &min_z);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        gr_z_update(__shfl_xor_sync(0xffffffffu, max_z, o), __shfl_xor_sync(0xffffffffu, min_z, o), &max_z, &min_z);
      status = gr_voxel_status((int32_t)count, ixyz[2], max_z, min_z, 0, kPsGroundThreshold) == kGrGround
                   ? kPsGroundPlane : kPsGroundNot;
      if (status == kPsGroundPlane)
        for (uint32_t k = s0 + lane; k < s1; k += 32) plane[order[k]] = 1;
    } else if (count < min_points * 2) {
      status = kPsSkippedRansac;
    } else if (count > kPsWarpMax) {
      if (lane == 0) cta_list[atomicAdd(cta_count, 1u)] = (uint32_t)v;
      continue;
    } else {
      ps_ransac(g, shared[w], shuffled[w], pts, stride, order + s0, (int)count, rnd, plane, t);
      continue;
    }
    if (t && lane == 0) *t = PsTrace{status, 0, 0, status == kPsGroundPlane ? (int32_t)count : 0, {0.f, 0.f, 0.f, 0.f}};
  }
}

// one CTA per voxel of the list, grid-strided; scratch: the shuffled indices, the voxel's slice at its sorted positions
__global__ void __launch_bounds__(kPsCtaThreads, 4)
ps_detect_cta_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ order,
                     const uint32_t* __restrict__ voxel_start, const uint32_t* __restrict__ cta_list,
                     const uint32_t* __restrict__ cta_count, const uint32_t* __restrict__ rnd,
                     uint8_t* __restrict__ plane, uint32_t* __restrict__ scratch, PsTrace* __restrict__ trace) {
  __shared__ PsShared<kPsCtaThreads> shared;
  const CtaGroup g;
  const uint32_t nb = *cta_count;
  for (uint32_t b = blockIdx.x; b < nb; b += gridDim.x) {
    const uint32_t v = cta_list[b];
    const uint32_t s0 = voxel_start[v], s1 = voxel_start[v + 1];
    ps_ransac(g, shared, scratch + s0, pts, stride, order + s0, (int)(s1 - s0), rnd, plane,
              trace ? trace + v : nullptr);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kCompactThreads)
ps_other_count_kernel(const uint8_t* __restrict__ plane, int n, uint32_t* __restrict__ tile_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n && !plane[base + r]) ++c;
  tile_count_store(c, tile_cnt);
}

// keep[i] for every point (all of them on the copy path) and the keep counts of the ordered compaction; other_off:
// the scanned non-plane counts (unused on the copy path)
__global__ void __launch_bounds__(kCompactThreads)
ps_keep_kernel(const uint8_t* __restrict__ plane, int n, int copy, const uint32_t* __restrict__ other_off, float rate,
               PsRatio ratio, uint8_t* __restrict__ keep, uint32_t* __restrict__ keep_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint8_t f[kCompactItems];
  uint32_t others = 0, c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    f[r] = (base + r < n) ? plane[base + r] : 1;
    others += f[r] ? 0u : 1u;
  }
  uint32_t k = copy ? 0u : tile_exclusive(others, other_off);   // non-plane points before this thread's first
  for (int r = 0; r < kCompactItems; ++r) {
    if (base + r >= n) break;
    uint8_t kp = 1;
    if (!copy && !f[r]) kp = ps_keep(rate, ratio, ++k) ? 1 : 0;
    keep[base + r] = kp;
    c += kp;
  }
  tile_count_store(c, keep_cnt);
}

const std::vector<uint32_t>& ps_raw_stream() {
  static const std::vector<uint32_t> words = [] {
    std::mt19937 engine(12345u);                        // boost::mt19937 seeded 12345u
    std::vector<uint32_t> w(kPsRndWords);
    for (auto& x : w) x = engine() >> 1;                // boost::uniform_int<int>(0, INT_MAX): engine() / 2
    return w;
  }();
  return words;
}

}  // namespace

// host builds (test hooks sm_debug_plane_sampler_*_host)
int ps_debug_piece_host(int op, const float* in, float* out) {
  switch (op) {
    case 0: out[0] = ps_sample_good(in, in + 3, in + 6) ? 1.f : 0.f; return 0;
    case 1: ps_model(in, in + 3, in + 6, out); return 0;
    case 2: out[0] = ps_distance(in, in + 4); out[1] = ps_inlier(in, in + 4) ? 1.f : 0.f; return 0;
    case 3: {
      float m[3][3];
      for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) m[i][j] = in[3 * i + j];
      ps_eigen33(m, out);
      return 0;
    }
    default: return -1;
  }
}

void ps_debug_keep_host(float rate, int64_t k0, int64_t k1, uint8_t* out) {
  const PsRatio r = ps_ratio(rate);
  for (int64_t k = k0; k < k1; ++k) out[k - k0] = ps_keep(rate, r, (uint32_t)k) ? 1 : 0;
}

int PlaneSampler::reserve(int64_t n) {
  SMB_RC(sort.reserve(RadixPairs::bytes(voxel_sort_stride(n), (int)n)));
  SMB_RC(tile_cnt.reserve(5 * compact_count_bytes(n)));
  SMB_RC(voxel_start.reserve(((size_t)n + 1) * sizeof(uint32_t)));
  SMB_RC(scratch.reserve((size_t)n * sizeof(uint32_t)));        // the CTA voxels' shuffled indices
  SMB_RC(cta_list.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(plane.reserve((size_t)n));
  SMB_RC(keep.reserve((size_t)n));
  SMB_RC(meta.reserve(kPsMeta * sizeof(uint32_t)));
  if (trace_on) SMB_RC(trace.reserve((size_t)n * sizeof(PsTrace)));
  for (DevBuf& b : lists_next) SMB_RC(b.reserve((size_t)n * sizeof(int32_t)));
  if (!rnd.p) {
    SMB_RC(rnd.reserve(kPsRndWords * sizeof(uint32_t)));
    SMB_CUDA_OK(cudaMemcpy(rnd.p, ps_raw_stream().data(), kPsRndWords * sizeof(uint32_t), cudaMemcpyHostToDevice));
  }
  return SM_OK;
}

int PlaneSampler::run(const char* pts, int64_t n, int64_t stride, float* out, uint32_t* out_index, int64_t* m,
                      cudaStream_t s) {
  const int ni = (int)n;
  const int tiles = compact_tiles(n);
  const bool copy = (double)rate > 0.999999;
  const bool detect = !copy && !(kPsGroundThreshold >= leaf_size);   // plane_detector.h:98-101
  SMB_RC(reserve(n));
  uint32_t* mt = (uint32_t*)meta.p;
  uint32_t* tc[5];
  for (int j = 0; j < 5; ++j) tc[j] = (uint32_t*)tile_cnt.p + (size_t)j * (tiles + 1);
  uint8_t* pl = (uint8_t*)plane.p;
  uint8_t* kp = (uint8_t*)keep.p;
  PsTrace* tr = trace_on ? (PsTrace*)trace.p : nullptr;
  SMB_CUDA_OK(cudaMemsetAsync(mt, 0, kPsMeta * sizeof(uint32_t), s));
  SMB_CUDA_OK(cudaMemsetAsync(pl, 0, (size_t)n, s));
  if (detect) {
    RadixPairs rp;
    rp.carve(sort.p, voxel_sort_stride(n));
    uint32_t* vs = (uint32_t*)voxel_start.p;
    SMB_RC(voxel_sort(pts, ni, stride, leaf_size, rp, mt, tc[0], vs, s));
    const uint32_t* order = rp.vals[0];
    const int warp_blocks = (int)std::min<int64_t>(ceil_div(n, 8 * kPsWarpsPerBlock), 16 * kNumSMs);
    ps_detect_warp_kernel<<<warp_blocks, 32 * kPsWarpsPerBlock, 0, s>>>(
        pts, stride, order, vs, tc[0] + tiles, leaf_size, min_points, (const uint32_t*)rnd.p, pl,
        (uint32_t*)cta_list.p, mt + 12, tr);
    ps_detect_cta_kernel<<<4 * kNumSMs, kPsCtaThreads, 0, s>>>(pts, stride, order, vs, (const uint32_t*)cta_list.p,
                                                              mt + 12, (const uint32_t*)rnd.p, pl,
                                                              (uint32_t*)scratch.p, tr);
    SMB_CUDA_OK(cudaMemcpyAsync(mt + 13, tc[0] + tiles, sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
  }
  if (!copy) {
    ps_other_count_kernel<<<tiles, kCompactThreads, 0, s>>>(pl, ni, tc[1]);
    compact_scan(tc[1], tiles, s);
  }
  ps_keep_kernel<<<tiles, kCompactThreads, 0, s>>>(pl, ni, copy ? 1 : 0, tc[1], rate, ps_ratio(rate), kp, tc[2]);
  filter_compact_records(pts, stride, nullptr, ni, kp, tc[2], out, out_index, mt + 8, s);
  flag_list(kp, ni, 1, tc[3], (int32_t*)lists_next[0].p, mt + 9, s);
  flag_list(kp, ni, 0, tc[4], (int32_t*)lists_next[1].p, mt + 10, s);
  flag_list(pl, ni, 1, tc[1], (int32_t*)lists_next[2].p, mt + 11, s);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t host[kPsMeta];
  SMB_CUDA_OK(cudaMemcpyAsync(host, mt, sizeof(host), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  if (detect && !voxel_span_ok(host)) return SM_ERR_BAD_ARGUMENT;
  for (int j = 0; j < 3; ++j) {
    std::swap(lists[j], lists_next[j]);
    n_lists[j] = host[9 + j];
  }
  n_voxels = trace_on ? host[13] : 0;
  *m = (int64_t)host[8];
  return SM_OK;
}

}  // namespace smb

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace smb;

struct sm_plane_sampler : RecordFilter {
  PlaneSampler f;
  explicit sm_plane_sampler(int device) : RecordFilter(device, "RandomSamplerWithPlaneDetect") {}
};

namespace smb {
PlaneSampler* plane_sampler_of(::sm_plane_sampler* h) { return h ? &h->f : nullptr; }
}  // namespace smb

extern "C" {

int sm_plane_sampler_create(int device, sm_plane_sampler** out) { return create_record_filter(device, out); }

int sm_plane_sampler_destroy(sm_plane_sampler* h) { return destroy_record_filter(h); }

int sm_plane_sampler_set_sampling_rate(sm_plane_sampler* h, float rate) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  h->error[0] = 0;
  if (rate > 1.) {
    h->fail(SM_OK, "rate should not be large than 1.");
    rate = 1.;
  } else if (rate < 1.e-6) {
    h->fail(SM_OK, "rate should not be less than 1.e-6");
    rate = 1.e-6;
  }
  h->f.rate = rate;
  return SM_OK;
}

int sm_plane_sampler_set_leaf_size(sm_plane_sampler* h, float leaf_size) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  h->error[0] = 0;
  h->f.leaf_size = leaf_size;
  return SM_OK;
}

int sm_plane_sampler_set_min_point_num_in_voxel(sm_plane_sampler* h, uint64_t num) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  h->error[0] = 0;
  if (num < 5) h->fail(SM_OK, "setting num is too small, reset to default minimum : 5");
  h->f.min_points = num < 5 ? 5 : num;
  return SM_OK;
}

int sm_plane_sampler_run_device(sm_plane_sampler* h, const float* dev_points, int64_t n, int64_t stride_bytes,
                                float* dev_out, int64_t* m_out, int32_t* dev_index, void* cuda_stream) {
  if (!h || !records_ok(dev_points, n, stride_bytes, dev_out, m_out)) return SM_ERR_BAD_ARGUMENT;
  if (n > (1 << 24))
    return h->fail(SM_ERR_BAD_ARGUMENT, "more than 2^24 points: the reference's float ratio is not exact past that");
  SMB_RC(h->use_device());
  if (n == 0) {
    *m_out = 0;
    for (int64_t& c : h->f.n_lists) c = 0;
    h->f.n_voxels = 0;
    return SM_OK;
  }
  uint32_t* idx = (uint32_t*)dev_index;
  if (!idx) {
    SMB_RC(h->cuda_fail(h->host_idx.reserve((size_t)n * sizeof(int32_t))));
    idx = (uint32_t*)h->host_idx.p;
  }
  const int rc = h->f.run((const char*)dev_points, n, stride_bytes, dev_out, idx, m_out, (cudaStream_t)cuda_stream);
  if (rc == SM_ERR_BAD_ARGUMENT)
    return h->fail(rc, "the voxel indices of an axis span more than 2^21 - 1 voxels (the 63-bit voxel key)");
  return h->cuda_fail(rc);
}

int sm_plane_sampler_run(sm_plane_sampler* h, const float* points, int64_t n, int64_t stride_bytes, float* out,
                         int64_t* m_out, int32_t* index) {
  if (!h || !records_ok(points, n, stride_bytes, out, m_out)) return SM_ERR_BAD_ARGUMENT;
  if (n > (1 << 24))
    return h->fail(SM_ERR_BAD_ARGUMENT, "more than 2^24 points: the reference's float ratio is not exact past that");
  SMB_RC(h->use_device());
  return run_record_filter(h, sm_plane_sampler_run_device, points, n, stride_bytes, out, m_out, index);
}

int sm_plane_sampler_indices(const sm_plane_sampler* h, int32_t* inliers, int64_t* n_inliers, int32_t* outliers,
                             int64_t* n_outliers) {
  if (!h || !n_inliers || !n_outliers) return SM_ERR_BAD_ARGUMENT;
  *n_inliers = h->f.n_lists[0];
  *n_outliers = h->f.n_lists[1];
  const bool copy_in = inliers && h->f.n_lists[0] > 0, copy_out = outliers && h->f.n_lists[1] > 0;
  if (!copy_in && !copy_out) return SM_OK;
  SMB_RC(select_device(h->device));
  if (copy_in)
    SMB_CUDA_OK(cudaMemcpy(inliers, h->f.lists[0].p, (size_t)h->f.n_lists[0] * sizeof(int32_t),
                           cudaMemcpyDeviceToHost));
  if (copy_out)
    SMB_CUDA_OK(cudaMemcpy(outliers, h->f.lists[1].p, (size_t)h->f.n_lists[1] * sizeof(int32_t),
                           cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_plane_sampler_plane_indices(const sm_plane_sampler* h, int32_t* plane, int64_t* n_plane) {
  if (!h || !n_plane) return SM_ERR_BAD_ARGUMENT;
  *n_plane = h->f.n_lists[2];
  if (!plane || h->f.n_lists[2] == 0) return SM_OK;
  SMB_RC(select_device(h->device));
  SMB_CUDA_OK(cudaMemcpy(plane, h->f.lists[2].p, (size_t)h->f.n_lists[2] * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return SM_OK;
}

const char* sm_plane_sampler_last_error(const sm_plane_sampler* h) { return h ? h->error : ""; }

}  // extern "C"
