// Shared device/host helpers for libsm_b200 (sm_90a only).
#ifndef SM_B200_COMMON_CUH_
#define SM_B200_COMMON_CUH_

#include <cuda_runtime.h>
#include <limits.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/sm_b200.h"

namespace smb {

// ---- error plumbing: every CUDA call inside the library goes through this ----------
#define SMB_CUDA_OK(expr)                                                        \
  do {                                                                           \
    cudaError_t _e = (expr);                                                     \
    if (_e != cudaSuccess) {                                                     \
      ::smb::set_cuda_error(_e, #expr, __FILE__, __LINE__);                      \
      return -100;                                                               \
    }                                                                            \
  } while (0)
// propagate the negative return code of an internal call (SMB_CUDA_OK's -100 == SM_ERR_CUDA)
#define SMB_RC(expr)                                                             \
  do {                                                                           \
    const int _rc = (expr);                                                      \
    if (_rc < 0) return _rc;                                                     \
  } while (0)

void set_cuda_error(cudaError_t e, const char* expr, const char* file, int line);
const char* last_cuda_error();

// the preamble of every entry point given a device ordinal: SM_ERR_NO_DEVICE without a CUDA device,
// SM_ERR_BAD_ARGUMENT for an ordinal out of range, else cudaSetDevice
inline int select_device(int device) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  if (device < 0 || device >= ndev) return SM_ERR_BAD_ARGUMENT;
  SMB_CUDA_OK(cudaSetDevice(device));
  return SM_OK;
}

// A float / double -> int conversion outside int's range is undefined in C++; the reference's x86 build yields INT_MIN
// there (also for NaN), which its clamps and range tests then read as "below 0".  Restated so on every side.
__host__ __device__ __forceinline__ int to_int(double q) {
  return (q > -2147483649.0 && q < 2147483648.0) ? (int)q : INT_MIN;
}

constexpr int kNumSMs = 132;  // H100 SXM; grids are sized in multiples

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// ---- exact (non-contracted) double arithmetic --------------------------------------
// The oracle is compiled with -ffp-contract=off; wherever the k-NN index set or a
// comparison depends on rounding we use the _rn intrinsics so nvcc cannot fuse a*b+c.
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }

// double -> radix-sortable u64 (total order incl. -0 < +0; NaNs sort last/first).
__host__ __device__ __forceinline__ uint64_t sortable_key(double v) {
  uint64_t u;
#ifdef __CUDA_ARCH__
  u = (uint64_t)__double_as_longlong(v);
#else
  memcpy(&u, &v, 8);
#endif
  return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}

// ---- k-d tree node (heap layout, 16 B, one LDG.128 per visit) ----------------------
// inner: {cut (f64), dim 0..2, -}; leaf: {first,count packed in the f64 slot, dim = 3}.
struct __align__(16) KdNode {
  double cut;   // leaf: low 32 bits = first bucket slot, high 32 bits = count
  int dim;
  int pad;
};

// Node storage order: the implicit heap (children of h are 2h+1 / 2h+2) is cut into blocks of
// 3 levels = 7 nodes that share one 128-byte line (8 slots of 16 B, slot 7 unused); the blocks
// themselves form an 8-ary heap.  A root-to-leaf descent of L levels touches ceil((L+1)/3)
// lines instead of L+1.  heap index h -> slot index (block * 8 + local).
__host__ __device__ __forceinline__ int blocked_index(int h) {
  int l = 0;
  while (((h + 1) >> (l + 1)) != 0) ++l;      // floor(log2(h+1))
  const int j = h + 1 - (1 << l);
  const int bl = l / 3, sl = l % 3;
  const int base = ((1 << (3 * bl)) - 1) / 7;
  const int B = base + (j >> sl);
  const int p = (1 << sl) - 1 + (j & ((1 << sl) - 1));
  return B * 8 + p;
}
// number of 16-byte node slots needed for a tree whose deepest level index is `levels`
__host__ __device__ __forceinline__ int64_t blocked_node_slots(int levels) {
  const int nbl = levels / 3 + 1;
  return ((((int64_t)1 << (3 * nbl)) - 1) / 7) * 8;
}

// bucket entry: target point in leaf order (two LDG.128)
struct __align__(32) BucketPoint {
  double x, y, z;
  long long id;  // original column index in the caller's cloud
};
struct __align__(32) BucketNormal {
  double x, y, z, pad;
};
// padded bucket entry of a normals tree as ICP phase B reads it: the point and its normal in one 64-byte line
// (three LDG.128 from two sectors), pad = 0
struct __align__(64) BucketMatch {
  double x, y, z, nx, ny, nz, pad[2];
};

}  // namespace smb

#endif  // SM_B200_COMMON_CUH_
