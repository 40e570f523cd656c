// Block-level sums, min/max and scans in one fixed order.  The float sums of the library are compared with the
// oracle bit for bit or to a few ulps, which holds because every block adds its values the same way:
//   1. each warp sums with an xor butterfly (offsets 16, 8, 4, 2, 1), so every lane holds the warp total;
//   2. lane 0 of each warp stores the warp total in shared memory;
//   3. one thread per sum adds the warp totals in warp order, starting from 0.
// Min/max follow the same shape, starting from warp 0's value.  Integer scans give the same values in any order.
// Everything here is inline, so each translation unit compiles it with its own flags (-fmad=false or not).
#ifndef SM_B200_REDUCE_CUH_
#define SM_B200_REDUCE_CUH_

#include <math.h>
#include <string.h>

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

// ---- exact float sums --------------------------------------------------------------------------------------------
// A float is m * 2^(b - 150) with an integer mantissa m < 2^24 and a biased exponent b = 1..254 (subnormals: b = 0,
// taken as b = 1 without the hidden bit), so a sum of floats is sum_b (sum of the m of bin b) * 2^(b - 150).  Each
// bin's sum is an integer of magnitude below 2^24 * 2^31 < 2^63 for up to 2^31 terms: int64 bins added in any order
// give the same bins, and a finish turns them into the value nearest the exact sum (ties to even), whatever the launch
// shape.  StatisticRemoval sums non-negative terms (exact_finish, to double); LUM sums signed ones (exact_finish_float,
// to float).
constexpr int kExactBins = 255;       // biased float exponents 1..254; bin 0 counts +inf terms
constexpr int kExactLimbs = 10;

// bin and mantissa of a non-negative float or +inf (bin 0, mantissa 1: counted apart)
__host__ __device__ __forceinline__ void exact_bin(float v, int* bin, uint32_t* mant) {
  uint32_t u;
#ifdef __CUDA_ARCH__
  u = __float_as_uint(v);
#else
  memcpy(&u, &v, 4);
#endif
  const uint32_t e = (u >> 23) & 0xffu, f = u & 0x7fffffu;
  if (e == 0xffu) { *bin = 0; *mant = 1u; return; }
  *bin = e == 0u ? 1 : (int)e;
  *mant = e == 0u ? f : (f | 0x800000u);
}

// limb = the integer N = sum_b sign * bins[b] * 2^(b - 1) (b = 1..254) over the bins of that sign (sign * bins[b] > 0),
// in units of 2^-149: N < 2^308, ten 32-bit limbs, carried once.
__host__ __device__ inline void exact_limbs(const int64_t* bins, int sign, uint64_t* limb) {
  for (int j = 0; j < kExactLimbs; ++j) limb[j] = 0u;
  for (int b = 1; b < kExactBins; ++b) {
    const int64_t sv = sign > 0 ? bins[b] : -bins[b];
    if (sv <= 0) continue;
    const uint64_t v = (uint64_t)sv;
    const int shift = b - 1, w = shift >> 5, s = shift & 31;
    // v < 2^63 shifted by s < 32 spans three limbs; each limb gets < 2^32 per bin, 254 bins: no overflow of 64 bits
    const uint64_t lo = (v << s) & 0xffffffffu;
    const uint64_t mid = s ? ((v >> (32 - s)) & 0xffffffffu) : ((v >> 32) & 0xffffffffu);
    const uint64_t hi = s ? (v >> (64 - s)) : 0u;
    limb[w] += lo;
    if (w + 1 < kExactLimbs) limb[w + 1] += mid;
    if (w + 2 < kExactLimbs) limb[w + 2] += hi;
  }
  for (int j = 0; j + 1 < kExactLimbs; ++j) { limb[j + 1] += limb[j] >> 32; limb[j] &= 0xffffffffu; }
}

// N * 2^-149 (N in carried limbs) rounded to `bits` significant bits, ties to even, as a double (exact for bits <= 53)
__host__ __device__ inline double exact_round(const uint64_t* limb, int bits) {
  int top = kExactLimbs - 1;
  while (top >= 0 && limb[top] == 0u) --top;
  if (top < 0) return 0.0;
  int msb = 31;
  while (!((limb[top] >> msb) & 1u)) --msb;
  const int nbits = top * 32 + msb + 1;              // N has nbits bits
  if (nbits <= bits) {                                // exact
    uint64_t m = 0u;
    for (int j = top; j >= 0; --j) m = (m << 32) | limb[j];
    return ldexp((double)m, -149);
  }
  // the top `bits` bits, the next (round) bit and whether any bit below it is set (sticky)
  auto bit = [&](int p) -> uint64_t { return (limb[p >> 5] >> (p & 31)) & 1u; };
  const int low = nbits - bits;                       // position of the least significant kept bit
  uint64_t m = 0u;
  for (int p = nbits - 1; p >= low; --p) m = (m << 1) | bit(p);
  const uint64_t round = bit(low - 1);
  bool sticky = false;
  for (int p = low - 2; p >= 0 && !sticky; --p) sticky = bit(p) != 0u;
  if (round && (sticky || (m & 1u))) ++m;            // m may become 2^bits: still exact in a double
  return ldexp((double)m, low - 149);
}

// The double nearest sum_b bins[b] * 2^(b - 150) (b = 1..254, bins >= 0), +inf if bins[0] (the +inf terms) is not
// zero.  limb: kExactLimbs words of scratch (shared memory on the device, where a dynamically indexed array would be
// local)
__host__ __device__ inline double exact_finish(const int64_t* bins, uint64_t* limb) {
  if (bins[0] != 0) return __builtin_huge_val();
  exact_limbs(bins, 1, limb);
  return exact_round(limb, 53);
}

// Signed float terms: bins[1..254] hold signed mantissa sums (exact_bin of |v|, added with v's sign); bins[0], bins[255]
// and bins[256] count the +inf, -inf and NaN terms.  kExactSignedBins int64 per sum.
constexpr int kExactSignedBins = kExactBins + 2;

__host__ __device__ __forceinline__ void exact_bin_signed(float v, int* bin, int64_t* mant) {
  if (v != v) { *bin = kExactBins + 1; *mant = 1; return; }
  uint32_t m;
  exact_bin(fabsf(v), bin, &m);
  if (*bin == 0) { *bin = v > 0.f ? 0 : kExactBins; *mant = 1; return; }
  *mant = v < 0.f ? -(int64_t)m : (int64_t)m;
}

// The float nearest the exact sum (ties to even): NaN for a NaN term or for +inf and -inf terms together, else +-inf
// for an infinite term, else the finite sum (+inf / -inf when it rounds past FLT_MAX; +0 when it is zero).
// pos, neg: kExactLimbs words of scratch each.
__host__ __device__ inline float exact_finish_float(const int64_t* bins, uint64_t* pos, uint64_t* neg) {
  const bool pinf = bins[0] != 0, ninf = bins[kExactBins] != 0;
  if (bins[kExactBins + 1] != 0 || (pinf && ninf)) return __builtin_nanf("");
  if (pinf) return __builtin_huge_valf();
  if (ninf) return -__builtin_huge_valf();
  exact_limbs(bins, 1, pos);
  exact_limbs(bins, -1, neg);
  int cmp = 0;
  for (int j = kExactLimbs - 1; j >= 0 && cmp == 0; --j) cmp = pos[j] > neg[j] ? 1 : (pos[j] < neg[j] ? -1 : 0);
  if (cmp == 0) return 0.f;
  uint64_t* a = cmp > 0 ? pos : neg;                 // a -= b, |a| > |b|
  const uint64_t* b = cmp > 0 ? neg : pos;
  uint64_t borrow = 0u;
  for (int j = 0; j < kExactLimbs; ++j) {
    const uint64_t sub = b[j] + borrow;
    borrow = a[j] < sub ? 1u : 0u;
    a[j] = (a[j] + (borrow << 32)) - sub;
  }
  const float r = (float)exact_round(a, 24);          // 24 bits and at least 2^-149: exactly a float (or past FLT_MAX)
  return cmp > 0 ? r : -r;
}

}  // namespace smb

#endif  // SM_B200_REDUCE_CUH_
