// Block-level sums, min/max and scans in one fixed order.  The float sums of the library are compared with the
// oracle bit for bit or to a few ulps, which holds because every block adds its values the same way:
//   1. each warp sums with an xor butterfly (offsets 16, 8, 4, 2, 1), so every lane holds the warp total;
//   2. lane 0 of each warp stores the warp total in shared memory;
//   3. one thread per sum adds the warp totals in warp order, starting from 0.
// Min/max follow the same shape, starting from warp 0's value.  Integer scans give the same values in any order.
// Everything here is inline, so each translation unit compiles it with its own flags (-fmad=false or not).
#ifndef SM_B200_REDUCE_CUH_
#define SM_B200_REDUCE_CUH_

#include <cstdint>

namespace smb {

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__device__ __forceinline__ T warp_min(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

template <typename T>
__device__ __forceinline__ T warp_max(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// K sums over a block of NT threads: thread k < K returns sum k of acc[k], every other thread 0.  Every thread must
// call it.  red: [NT / 32][K] in shared memory.
template <int K, int NT, typename T>
__device__ __forceinline__ T block_sum(const T* acc, T (*red)[K]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const T v = warp_sum(acc[k]);
    if (lane == 0) red[w][k] = v;
  }
  __syncthreads();
  T v = 0;
  if (threadIdx.x < K)
    for (int ww = 0; ww < NT / 32; ++ww) v += red[ww][threadIdx.x];
  return v;
}

// The cross-block step: one warp adds entry k of the [nrows][width] rows, lane-strided over the rows, then
// butterflies.  Every lane returns the total.  R is the row pointer's type, so a caller can keep volatile loads.
template <typename R>
__device__ __forceinline__ double warp_sum_rows(R rows, int nrows, int width, int k) {
  double v = 0.0;
  for (int b = threadIdx.x & 31; b < nrows; b += 32) v += rows[(int64_t)b * width + k];
  return warp_sum(v);
}

// Per-axis min and max of three floats over a block of NT threads: thread d < 3 returns {min, max} of axis d,
// every other thread {0, 0}.  Every thread must call it.
template <int NT>
__device__ __forceinline__ float2 block_minmax3(const float (&mn)[3], const float (&mx)[3]) {
  __shared__ float smn[3][NT / 32], smx[3][NT / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int d = 0; d < 3; ++d) {
    const float a = warp_min(mn[d]), b = warp_max(mx[d]);
    if (lane == 0) { smn[d][w] = a; smx[d][w] = b; }
  }
  __syncthreads();
  float2 r = {0.0f, 0.0f};
  if (threadIdx.x < 3) {
    r = {smn[threadIdx.x][0], smx[threadIdx.x][0]};
    for (int ww = 1; ww < NT / 32; ++ww) { r.x = fminf(r.x, smn[threadIdx.x][ww]); r.y = fmaxf(r.y, smx[threadIdx.x][ww]); }
  }
  return r;
}

__device__ __forceinline__ uint32_t warp_inclusive_scan(uint32_t v) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += u;
  }
  return v;
}

// Exclusive scan of one value per thread over the first NW warps of the block; later warps must pass 0.  Returns
// the values of the lower threads added up, and the block total in *total if given.  Every thread must call it.
// warp_tot: one entry per warp of the block in shared memory; if threads may still be reading it from an earlier
// call, the caller syncs first.  Up to 8 warps, each thread adds the warp totals serially (without a total only the
// lower warps', which keeps the compaction scatter kernels at their register count); more warps scan them with one
// shuffle ladder.
template <int NW>
__device__ __forceinline__ uint32_t block_scan_excl(uint32_t v, uint32_t* warp_tot, uint32_t* total = nullptr) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const uint32_t incl = warp_inclusive_scan(v);
  if (lane == 31) warp_tot[w] = incl;
  __syncthreads();
  if constexpr (NW <= 8) {
    uint32_t base = 0;
    if (total) {   // one pass over all the warp totals gives both
      uint32_t tot = 0;
#pragma unroll
      for (int ww = 0; ww < NW; ++ww) { const uint32_t x = warp_tot[ww]; if (ww < w) base += x; tot += x; }
      *total = tot;
    } else {
      for (int ww = 0; ww < w; ++ww) base += warp_tot[ww];
    }
    return base + incl - v;
  } else {
    const uint32_t x = lane < NW ? warp_tot[lane] : 0u;
    const uint32_t xi = warp_inclusive_scan(x);
    if (total) *total = __shfl_sync(0xffffffffu, xi, 31);
    return __shfl_sync(0xffffffffu, xi - x, w) + incl - v;
  }
}

}  // namespace smb

#endif  // SM_B200_REDUCE_CUH_
