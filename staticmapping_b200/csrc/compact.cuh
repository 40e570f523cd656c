// Ordered compaction: a stage flags some of its n items and writes the flagged ones (or their positions) in input
// order, in three launches: its count kernel (tile_count_store), compact_scan, its scatter kernel (tile_exclusive).
// After compact_scan, cnt[b] = flagged items before tile b and cnt[tiles] = the number of flagged items.
// Both kernels run compact_tiles(n) blocks of kCompactThreads threads; thread t of tile b owns the items
// b * kCompactTile + t * kCompactItems .. + kCompactItems - 1.
#ifndef SM_B200_COMPACT_CUH_
#define SM_B200_COMPACT_CUH_

#include "kernels.h"
#include "reduce.cuh"

namespace smb {

constexpr int kCompactThreads = 256, kCompactItems = 8, kCompactTile = kCompactThreads * kCompactItems;

inline int compact_tiles(int64_t n) { return ceil_div(n, kCompactTile); }
inline size_t compact_count_bytes(int64_t n) { return ((size_t)compact_tiles(n) + 1) * sizeof(uint32_t); }

// count kernel: c = the thread's number of flagged items.  Stores the tile's count, and clears the slot behind the
// last tile that the scan turns into the total.
__device__ __forceinline__ void tile_count_store(uint32_t c, uint32_t* __restrict__ cnt) {
  __shared__ uint32_t ws[kCompactThreads / 32][1];
  const uint32_t t = block_sum<1, kCompactThreads>(&c, ws);
  if (threadIdx.x == 0) {
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
  return tile_off[blockIdx.x] + block_scan_excl<kCompactThreads / 32>(c, ws);
}

}  // namespace smb

#endif  // SM_B200_COMPACT_CUH_
