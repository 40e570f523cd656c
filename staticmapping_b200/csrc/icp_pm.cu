// PmStage: the device work of the IcpUsingPointMatcher stand-in (type 1) that is not IcpFast's or CalculateNormals'
// -- the reading filter and the score pass.  The module chain they belong to is described above pm_align (sm_api.cu).
#include "common.cuh"
#include "compact.cuh"
#include "icp_dev.cuh"
#include "kernels.h"

namespace smb {
namespace {

// ---- reading filter: RandomSampling (icp_pointmatcher.cc:173) with a counter hash for std::rand ----------------
__device__ __forceinline__ bool pm_keep(uint32_t i, uint32_t seed, uint32_t thresh, bool all) {
  uint32_t x = i * 0x9E3779B9u + seed;
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return all || x < thresh;
}

__global__ void __launch_bounds__(kCompactThreads)
pm_sample_count_kernel(int n, uint32_t seed, uint32_t thresh, int all, uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r)
    if (base + r < n) c += pm_keep((uint32_t)(base + r), seed, thresh, all != 0) ? 1u : 0u;
  tile_count_store(c, tile_cnt);
}

// kept points, original order, as 3xN column-major doubles (EigenPointCloud::FromPointCloud)
__global__ void __launch_bounds__(kCompactThreads)
pm_sample_scatter_kernel(const float* __restrict__ pts, int n, uint32_t seed, uint32_t thresh, int all,
                         const uint32_t* __restrict__ tile_off, double* __restrict__ out) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    f[r] = (base + r < n && pm_keep((uint32_t)(base + r), seed, thresh, all != 0)) ? 1u : 0u;
    c += f[r];
  }
  int64_t d = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    if (!f[r]) continue;
    const int64_t i = base + r;
    out[3 * d] = (double)pts[3 * i];
    out[3 * d + 1] = (double)pts[3 * i + 1];
    out[3 * d + 2] = (double)pts[3 * i + 2];
    ++d;
  }
}

// ---- score of the IcpUsingPointMatcher stand-in (icp_pointmatcher.cc:131-148): the UNFILTERED
// reading cloud moved by the result is matched against the UNFILTERED reference (same k-d tree
// matcher, eps 3.16), trimmed at the 0.7 quantile, and the mean kept distance goes into exp(-x)
__global__ void __launch_bounds__(256)
pm_score_knn_kernel(const float* __restrict__ src, int n, const double* __restrict__ T, const KdNode* __restrict__ nodes,
                    const BucketPoint* __restrict__ bpts, double max_error2, uint64_t* __restrict__ keys,
                    uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = (double)src[3 * (int64_t)i], y = (double)src[3 * (int64_t)i + 1], z = (double)src[3 * (int64_t)i + 2];
  double px, py, pz;
  dev::transform_point(T, x, y, z, px, py, pz);
  int slot; double d2;
  dev::knn1(nodes, bpts, px, py, pz, max_error2, slot, d2);
  keys[i] = (uint64_t)__double_as_longlong(d2);     // non-negative doubles sort like their bit patterns; +inf = no match
  vals[i] = (uint32_t)i;
}

// keys sorted ascending; out[0] = mean of sqrt(d2) over the kept matches, out[1] = kept, out[2] = valid
__global__ void __launch_bounds__(1024)
pm_score_reduce_kernel(const uint64_t* __restrict__ keys, int n, float ratio, double* __restrict__ out) {
  __shared__ double red[32];
  __shared__ int s_kept, s_valid;
  const uint64_t inf_bits = 0x7ff0000000000000ull;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n;                                // first index with key >= +inf
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] < inf_bits) lo = mid + 1; else hi = mid; }
    const int valid = lo;
    int kept = 0;
    if (valid > 0) {
      const double q = (double)ratio;                  // GetDistsQuantile, as icp_fast.cc:82-89
      int qi = (q == 1.0) ? valid - 1 : (int)((double)valid * q);
      if (qi > valid - 1) qi = valid - 1;
      const uint64_t limit = keys[qi];
      lo = qi; hi = valid;                             // first index with key > limit
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] <= limit) lo = mid + 1; else hi = mid; }
      kept = lo;
    }
    s_kept = kept; s_valid = valid;
  }
  __syncthreads();
  const int kept = s_kept;
  double v = 0.0;
  for (int i = threadIdx.x; i < kept; i += 1024) v += sqrt(__longlong_as_double((long long)keys[i]));
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 32; ++w) t += red[w];
    out[0] = kept > 0 ? t / (double)kept : 0.0;
    out[1] = (double)kept;
    out[2] = (double)s_valid;
  }
}

constexpr size_t kScoreHead = 256;   // bytes before the sort: 16 doubles of pose, then 3 of output

}  // namespace

int PmStage::reserve(int n_source) {
  SMB_RC(cnt.reserve(compact_count_bytes(n_source)));
  SMB_RC(sampled.reserve((size_t)3 * (size_t)n_source * sizeof(double)));
  return score.reserve(kScoreHead + RadixPairs::bytes(((int64_t)n_source + 63) & ~(int64_t)63, n_source));
}

int PmStage::sample(const float* src, int n, float prob_f, uint32_t seed, cudaStream_t s, uint32_t* kept) {
  const double prob = (double)prob_f;
  const int all = prob >= 1.0 ? 1 : 0;
  const uint32_t thresh = prob <= 0.0 ? 0u : (all ? 0xffffffffu : (uint32_t)(prob * 4294967296.0));
  uint32_t* tile_cnt = (uint32_t*)cnt.p;
  const int tiles = compact_tiles(n);
  pm_sample_count_kernel<<<tiles, kCompactThreads, 0, s>>>(n, seed, thresh, all, tile_cnt);
  compact_scan(tile_cnt, tiles, s);
  pm_sample_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(src, n, seed, thresh, all, tile_cnt, (double*)sampled.p);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(kept, tile_cnt + tiles, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

int PmStage::score_pass(const float* src, int n, const double* T_host_pinned, const FloatTree& target,
                        double max_error2, float ratio, double* out3_host, cudaStream_t s) {
  const int64_t st = ((int64_t)n + 63) & ~(int64_t)63;
  double* Tdev = (double*)score.p;
  double* outdev = Tdev + 16;
  RadixPairs sp;
  sp.carve((char*)score.p + kScoreHead, st);
  SMB_CUDA_OK(cudaMemcpyAsync(Tdev, T_host_pinned, 16 * sizeof(double), cudaMemcpyHostToDevice, s));
  pm_score_knn_kernel<<<ceil_div(n, 256), 256, 0, s>>>(src, n, Tdev, (const KdNode*)target.nodes.p,
                                                       (const BucketPoint*)target.bpts.p, max_error2, sp.keys[0],
                                                       sp.vals[0]);
  SMB_RC(radix_sort_pairs_u64(sp.keys[0], sp.vals[0], sp.keys[1], sp.vals[1], n, 1, st, sp.scratch, s, 8));
  pm_score_reduce_kernel<<<1, 1024, 0, s>>>(sp.keys[0], n, ratio, outdev);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(out3_host, outdev, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return 0;
}

}  // namespace smb
