// The arithmetic of PCL's StatisticalOutlierRemoval::applyFilterIndices that the device and the host test hooks share
// (statistic_removal.cu, knn.cu, include/sm_b200_debug.h): the per-point mean distance and the correctly rounded sum
// of the per-point terms.
//
// Per point (FLANN's L2_Simple<float> distance, then PCL's loop over the neighbours 1..K):
//   dx = qx - px in float, d2 = ((0 + dx*dx) + dy*dy) + dz*dz in float, dist_sum += sqrt((double)d2) in list order,
//   distance = (float)(dist_sum / K).
// Every operation is spelled with a round-to-nearest intrinsic on the device, so no contraction can change it.
//
// Exact sum of n non-negative floats (and +inf): a float is m * 2^(b - 150) with an integer mantissa m < 2^24 and a
// biased exponent b = 1..254 (subnormals: b = 0, taken as b = 1 without the hidden bit), so the sum is
// sum_b (sum of the m of bin b) * 2^(b - 150).  Each bin's sum is an integer below 2^24 * 2^30 < 2^63 for up to 2^30
// terms: int64 bins added in any order give the same bins.  sr_exact_finish turns them into the one double nearest the
// exact sum (ties to even).
#ifndef SM_B200_STATISTIC_REMOVAL_CUH_
#define SM_B200_STATISTIC_REMOVAL_CUH_

#include <math.h>
#include <stdint.h>
#include <string.h>

namespace smb {

constexpr int kSrBins = 255;          // biased float exponents 1..254; bin 0 counts +inf terms
constexpr int kSrMaxMeanK = 63;       // K + 1 neighbours must stay within the search's 64

__host__ __device__ __forceinline__ float sr_fsub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  return a - b;
#endif
}
__host__ __device__ __forceinline__ float sr_fadd(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
__host__ __device__ __forceinline__ float sr_fmul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}

// one neighbour's term of dist_sum: sqrt((double)d2) of L2_Simple<float>'s d2
__host__ __device__ __forceinline__ double sr_neighbour_term(float qx, float qy, float qz, float px, float py, float pz) {
  const float dx = sr_fsub(qx, px), dy = sr_fsub(qy, py), dz = sr_fsub(qz, pz);
  const float d2 = sr_fadd(sr_fadd(sr_fadd(0.f, sr_fmul(dx, dx)), sr_fmul(dy, dy)), sr_fmul(dz, dz));
#ifdef __CUDA_ARCH__
  return __dsqrt_rn((double)d2);
#else
  return sqrt((double)d2);
#endif
}

__host__ __device__ __forceinline__ double sr_dadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

__host__ __device__ __forceinline__ float sr_mean_distance(double dist_sum, int K) {
#ifdef __CUDA_ARCH__
  return __double2float_rn(__ddiv_rn(dist_sum, (double)K));
#else
  return (float)(dist_sum / (double)K);
#endif
}

// bin and mantissa of a non-negative float or +inf (bin 0, mantissa 1: counted apart)
__host__ __device__ __forceinline__ void sr_exact_bin(float v, int* bin, uint32_t* mant) {
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

// The double nearest sum_b bins[b] * 2^(b - 150) (b = 1..254), +inf if bins[0] (the +inf terms) is not zero.
// The exact sum is an integer N in units of 2^-149 below 2^308: ten 32-bit limbs, carried once, then rounded to 53 bits.
// limb: kSrLimbs words of scratch (shared memory on the device, where a dynamically indexed array would be local)
constexpr int kSrLimbs = 10;
__host__ __device__ inline double sr_exact_finish(const int64_t* bins, uint64_t* limb) {
  if (bins[0] != 0) return __builtin_huge_val();
  constexpr int kLimbs = kSrLimbs;
  for (int j = 0; j < kLimbs; ++j) limb[j] = 0u;
  for (int b = 1; b < kSrBins; ++b) {
    const uint64_t v = (uint64_t)bins[b];
    if (v == 0u) continue;
    const int shift = b - 1, w = shift >> 5, s = shift & 31;
    // v < 2^63 shifted by s < 32 spans three limbs; each limb gets < 2^32 per bin, 254 bins: no overflow of 64 bits
    const uint64_t lo = (v << s) & 0xffffffffu;
    const uint64_t mid = s ? ((v >> (32 - s)) & 0xffffffffu) : ((v >> 32) & 0xffffffffu);
    const uint64_t hi = s ? (v >> (64 - s)) : 0u;
    limb[w] += lo;
    if (w + 1 < kLimbs) limb[w + 1] += mid;
    if (w + 2 < kLimbs) limb[w + 2] += hi;
  }
  for (int j = 0; j + 1 < kLimbs; ++j) { limb[j + 1] += limb[j] >> 32; limb[j] &= 0xffffffffu; }
  int top = kLimbs - 1;
  while (top >= 0 && limb[top] == 0u) --top;
  if (top < 0) return 0.0;
  int msb = 31;
  while (!((limb[top] >> msb) & 1u)) --msb;
  const int nbits = top * 32 + msb + 1;              // N has nbits bits
  if (nbits <= 53) {                                  // exact
    uint64_t m = 0u;
    for (int j = top; j >= 0; --j) m = (m << 32) | limb[j];
    return ldexp((double)m, -149);
  }
  // the top 53 bits, the next (round) bit and whether any bit below it is set (sticky)
  auto bit = [&](int p) -> uint64_t { return (limb[p >> 5] >> (p & 31)) & 1u; };
  const int low = nbits - 53;                         // position of the least significant kept bit
  uint64_t m = 0u;
  for (int p = nbits - 1; p >= low; --p) m = (m << 1) | bit(p);
  const uint64_t round = bit(low - 1);
  bool sticky = false;
  for (int p = low - 2; p >= 0 && !sticky; --p) sticky = bit(p) != 0u;
  if (round && (sticky || (m & 1u))) ++m;            // m may become 2^53: still exact in a double
  return ldexp((double)m, low - 149);
}

}  // namespace smb

#endif  // SM_B200_STATISTIC_REMOVAL_CUH_
