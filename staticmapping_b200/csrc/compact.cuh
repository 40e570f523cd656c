// Ordered compaction: a stage flags some of its n items and writes the flagged ones (or their positions) in input
// order, in three launches: its count kernel (tile_count_store), compact_scan, its scatter kernel (tile_exclusive).
// After compact_scan, cnt[b] = flagged items before tile b and cnt[tiles] = the number of flagged items.
// Both kernels run compact_tiles(n) blocks of kCompactThreads threads; thread t of tile b owns the items
// b * kCompactTile + t * kCompactItems .. + kCompactItems - 1.
#ifndef SM_B200_COMPACT_CUH_
#define SM_B200_COMPACT_CUH_

#include "kernels.h"

namespace smb {

constexpr int kCompactThreads = 256, kCompactItems = 8, kCompactTile = kCompactThreads * kCompactItems;

inline int compact_tiles(int64_t n) { return ceil_div(n, kCompactTile); }
inline size_t compact_count_bytes(int64_t n) { return ((size_t)compact_tiles(n) + 1) * sizeof(uint32_t); }

// count kernel: c = the thread's number of flagged items.  Stores the tile's count, and clears the slot behind the
// last tile that the scan turns into the total.
__device__ __forceinline__ void tile_count_store(uint32_t c, uint32_t* __restrict__ cnt) {
  __shared__ uint32_t ws[kCompactThreads / 32];
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) ws[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int w = 0; w < kCompactThreads / 32; ++w) t += ws[w];
    cnt[blockIdx.x] = t;
    if (blockIdx.x == 0) cnt[gridDim.x] = 0;
  }
}

// tile counts -> tile offsets and the total, in place
inline void compact_scan(uint32_t* cnt, int tiles, cudaStream_t stream) {
  radix_scan_kernel_launch(cnt, tiles + 1, 1, stream);
}

// scatter kernel: c as above -> the output position of the thread's first flagged item
__device__ __forceinline__ uint32_t tile_exclusive(uint32_t c, const uint32_t* __restrict__ tile_off) {
  __shared__ uint32_t ws[kCompactThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t incl = c;
  for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) ws[w] = incl;
  __syncthreads();
  uint32_t pos = tile_off[blockIdx.x] + incl - c;
  for (int ww = 0; ww < w; ++ww) pos += ws[ww];
  return pos;
}

}  // namespace smb

#endif  // SM_B200_COMPACT_CUH_
