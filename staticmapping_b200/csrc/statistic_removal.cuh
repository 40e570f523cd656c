// The arithmetic of PCL's StatisticalOutlierRemoval::applyFilterIndices that the device and the host test hooks share
// (statistic_removal.cu, knn.cu, include/sm_b200_debug.h): the per-point mean distance and the correctly rounded sum
// of the per-point terms.
//
// Per point (FLANN's L2_Simple<float> distance, then PCL's loop over the neighbours 1..K):
//   dx = qx - px in float, d2 = ((0 + dx*dx) + dy*dy) + dz*dz in float, dist_sum += sqrt((double)d2) in list order,
//   distance = (float)(dist_sum / K).
// Every operation is spelled with a round-to-nearest intrinsic on the device, so no contraction can change it.
//
// The sum of the per-point terms and of their squares is exact and rounded once (exact_bin / exact_finish, reduce.cuh).
#ifndef SM_B200_STATISTIC_REMOVAL_CUH_
#define SM_B200_STATISTIC_REMOVAL_CUH_

#include <math.h>
#include <stdint.h>
#include <string.h>

#include "reduce.cuh"

namespace smb {

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

}  // namespace smb

#endif  // SM_B200_STATISTIC_REMOVAL_CUH_
