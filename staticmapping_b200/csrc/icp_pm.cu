// PmStage: the device work of the IcpUsingPointMatcher stand-in (type 1) that is not IcpFast's or CalculateNormals'
// -- the reading filter and the score pass.  The module chain they belong to is described above pm_align (sm_api.cu).
#include "common.cuh"
#include "compact.cuh"
#include "icp_dev.cuh"
#include "kernels.h"

namespace smb {
namespace {

// ---- reading filter: RandomSampling (icp_pointmatcher.cc:173) with a counter hash for std::rand ----------------
// With rand_bits (the rand sampler's flags) the flag of point i is its bit there instead.
__device__ __forceinline__ bool pm_keep(uint32_t i, uint32_t seed, uint32_t thresh, bool all,
                                        const uint32_t* __restrict__ rand_bits) {
  if (rand_bits) return (rand_bits[i >> 5] >> (i & 31)) & 1u;
  uint32_t x = i * 0x9E3779B9u + seed;
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return all || x < thresh;
}

__global__ void __launch_bounds__(kCompactThreads)
pm_sample_count_kernel(int n, uint32_t seed, uint32_t thresh, int all, const uint32_t* __restrict__ rand_bits,
                       uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r)
    if (base + r < n) c += pm_keep((uint32_t)(base + r), seed, thresh, all != 0, rand_bits) ? 1u : 0u;
  tile_count_store(c, tile_cnt);
}

// kept points, original order, as 3xN column-major doubles (EigenPointCloud::FromPointCloud)
__global__ void __launch_bounds__(kCompactThreads)
pm_sample_scatter_kernel(const float* __restrict__ pts, int n, uint32_t seed, uint32_t thresh, int all,
                         const uint32_t* __restrict__ rand_bits, const uint32_t* __restrict__ tile_off,
                         double* __restrict__ out) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    f[r] = (base + r < n && pm_keep((uint32_t)(base + r), seed, thresh, all != 0, rand_bits)) ? 1u : 0u;
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

// ---- reading filter: RandomSampling with glibc's rand() stream (sm_set_pm_reading_sampler GLIBC_RAND) -----------
// glibc's TYPE_3 rand(): r[0] = seed (0 -> 1), r[1..30] = 16807 r mod (2^31 - 1), r[31..33] = r[0..2], then
// r[k] = r[k-3] + r[k-31] (mod 2^32); 310 outputs are discarded and draw p is r[344 + p] >> 1.  With s_k = r[3 + k]
// the recurrence is s_k = s_{k-3} + s_{k-31} for every k >= 31, linear over Z/2^32 with characteristic polynomial
// P = x^31 - x^28 - 1, so s_{k+m} = sum_j c_j s_{k+j} with c = x^m mod P whatever k: a window of 31 consecutive s
// moves by m in O(log m) polynomial squarings.  The window at position p is s_{310+p} .. s_{340+p}: the next draw
// is (w[0] + w[28]) >> 1.

// a <- a^2 mod P
__host__ __device__ __forceinline__ void rand_poly_square(uint32_t* a) {
  uint32_t t[2 * kPmRandDeg - 1];
#pragma unroll
  for (int k = 0; k < 2 * kPmRandDeg - 1; ++k) t[k] = 0u;
#pragma unroll
  for (int i = 0; i < kPmRandDeg; ++i) {
    t[2 * i] += a[i] * a[i];
#pragma unroll
    for (int j = i + 1; j < kPmRandDeg; ++j) t[i + j] += 2u * a[i] * a[j];
  }
#pragma unroll
  for (int k = 2 * kPmRandDeg - 2; k >= kPmRandDeg; --k) {   // x^k = x^(k-3) + x^(k-31), highest first
    t[k - 3] += t[k];
    t[k - kPmRandDeg] += t[k];
  }
#pragma unroll
  for (int i = 0; i < kPmRandDeg; ++i) a[i] = t[i];
}

// a <- a x mod P
__host__ __device__ __forceinline__ void rand_poly_shift(uint32_t* a) {
  const uint32_t top = a[kPmRandDeg - 1];
#pragma unroll
  for (int i = kPmRandDeg - 1; i > 0; --i) a[i] = a[i - 1];
  a[0] = top;
  a[kPmRandDeg - 3] += top;
}

// w <- the window m steps further on
__host__ __device__ __forceinline__ void rand_window_advance(uint32_t* w, uint64_t m) {
  uint32_t c[kPmRandDeg];
#pragma unroll
  for (int i = 0; i < kPmRandDeg; ++i) c[i] = i == 0 ? 1u : 0u;
  for (int b = 63; b >= 0; --b) {             // c = x^m mod P, square-and-multiply from the top bit of m
    if ((m >> b) == 0) continue;
    rand_poly_square(c);
    if ((m >> b) & 1) rand_poly_shift(c);
  }
  uint32_t out[kPmRandDeg];
#pragma unroll
  for (int i = 0; i < kPmRandDeg; ++i) {      // s_{k+m+i} = (x^(m+i) mod P) . w
    uint32_t v = 0;
#pragma unroll
    for (int j = 0; j < kPmRandDeg; ++j) v += c[j] * w[j];
    out[i] = v;
    rand_poly_shift(c);
  }
#pragma unroll
  for (int i = 0; i < kPmRandDeg; ++i) w[i] = out[i];
}

// (float)rand() / (float)RAND_MAX < prob, as x86 evaluates it: (float)RAND_MAX is 2^31, so the division is exact
__host__ __device__ __forceinline__ bool rand_keep(uint32_t r, float prob) {
  return (float)(r >> 1) / 2147483648.0f < prob;
}

// One thread per slice of kPmRandSlice draws: it moves the window at the stream position to its slice's start, runs
// the recurrence forward and writes the keep flags of its draws as bits (bit i % 32 of word i / 32).
constexpr int kPmRandSlice = 32 * kPmRandDeg;   // 31 bodies of 31 draws fill 31 flag words
constexpr int kPmRandThreads = 128;

__global__ void __launch_bounds__(kPmRandThreads)
pm_rand_flags_kernel(int n, PmRandWindow at, float prob, uint32_t* __restrict__ bits) {
  const int t = blockIdx.x * kPmRandThreads + threadIdx.x;
  const int first = t * kPmRandSlice;
  if (first >= n) return;
  uint32_t w[kPmRandDeg];
#pragma unroll
  for (int i = 0; i < kPmRandDeg; ++i) w[i] = at.w[i];
  rand_window_advance(w, (uint64_t)first);
  const int words = min(kPmRandDeg, (n - first + 31) / 32);
  uint32_t* out = bits + (int64_t)t * kPmRandDeg;
  uint64_t acc = 0;
  int fill = 0, wi = 0;
  for (int body = 0; body < 32 && wi < words; ++body) {
    uint32_t f = 0;
#pragma unroll
    for (int k = 0; k < kPmRandDeg; ++k) {      // w[k] holds s_{j-31}, w[(k+28) % 31] s_{j-3}
      const uint32_t s = w[k] + w[(k + kPmRandDeg - 3) % kPmRandDeg];
      w[k] = s;
      f |= (rand_keep(s, prob) ? 1u : 0u) << k;
    }
    acc |= (uint64_t)f << fill;
    fill += kPmRandDeg;
    if (fill >= 32) {
      out[wi++] = (uint32_t)acc;
      acc >>= 32;
      fill -= 32;
    }
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
  __shared__ double red[32][1];
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
  const double t = block_sum<1, 1024>(&v, red);
  if (threadIdx.x == 0) {
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

PmRandWindow pm_rand_window(uint32_t seed, uint64_t position) {
  // srandom_r: the seed is held in an int32_t, so a seed >= 2^31 is negative and the Schrage step below uses C's
  // truncating / and %, as glibc does
  int32_t r[kPmRandDeg];
  int32_t word = (int32_t)(seed == 0 ? 1u : seed);
  r[0] = word;
  for (int i = 1; i < kPmRandDeg; ++i) {
    const int64_t hi = word / 127773, lo = word % 127773;
    word = (int32_t)(16807 * lo - 2836 * hi);
    if (word < 0) word += 2147483647;
    r[i] = word;
  }
  PmRandWindow at;   // s_0 .. s_30 = r[3 .. 30], then the copies r[31 .. 33] = r[0 .. 2]
  for (int j = 0; j < kPmRandDeg; ++j) at.w[j] = (uint32_t)r[(j + 3) % kPmRandDeg];
  rand_window_advance(at.w, 310u + position);
  return at;
}

void pm_rand_debug_advance_host(PmRandWindow& at, uint64_t m) { rand_window_advance(at.w, m); }

void pm_rand_debug_draws_host(PmRandWindow at, int64_t count, int32_t* out) {
  uint32_t* w = at.w;
  for (int64_t i = 0; i < count; ++i) {
    const uint32_t s = w[0] + w[kPmRandDeg - 3];
    for (int j = 0; j < kPmRandDeg - 1; ++j) w[j] = w[j + 1];
    w[kPmRandDeg - 1] = s;
    out[i] = (int32_t)(s >> 1);
  }
}

int PmStage::sample(const float* src, int n, float prob_f, uint32_t seed, cudaStream_t s, uint32_t* kept,
                    const PmRandWindow* rand) {
  const double prob = (double)prob_f;
  const int all = prob >= 1.0 ? 1 : 0;
  const uint32_t thresh = prob <= 0.0 ? 0u : (all ? 0xffffffffu : (uint32_t)(prob * 4294967296.0));
  uint32_t* tile_cnt = (uint32_t*)cnt.p;
  const int tiles = compact_tiles(n);
  const uint32_t* bits = nullptr;
  if (rand) {
    SMB_RC(rand_flags.reserve((size_t)ceil_div(n, 32) * sizeof(uint32_t)));
    const int slices = ceil_div(n, kPmRandSlice);
    pm_rand_flags_kernel<<<ceil_div(slices, kPmRandThreads), kPmRandThreads, 0, s>>>(n, *rand, prob_f,
                                                                                       (uint32_t*)rand_flags.p);
    bits = rand_bits();
  }
  pm_sample_count_kernel<<<tiles, kCompactThreads, 0, s>>>(n, seed, thresh, all, bits, tile_cnt);
  compact_scan(tile_cnt, tiles, s);
  pm_sample_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(src, n, seed, thresh, all, bits, tile_cnt,
                                                             (double*)sampled.p);
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

// an even number of passes leaves the sort's result in keys[0], the first array carved behind the head
const uint64_t* PmStage::sorted_keys() const { return (const uint64_t*)((const char*)score.p + kScoreHead); }

}  // namespace smb
