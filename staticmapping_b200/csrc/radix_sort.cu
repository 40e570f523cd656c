// Stable LSD radix sort of (u64 key, u32 value) pairs, `batch` independent sorts per
// launch (grid.y).  Used once per Align for the three per-axis orderings of the
// k-d tree builder (replaces the O(N log N) std::nth_element recursion inside
// NNS::create, registrators/icp_fast.cc:466-467).  Hand-written: no CUB/thrust.
//
// Pass = 3 launches: per-tile digit histogram -> one-block exclusive scan (digit-major)
// -> stable scatter.  Tile = 256 threads x 8 keys; warp w owns 256 contiguous keys so
// that (tile, warp, row, lane) order == input order, which is what makes it stable.
#include "common.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace smb {
namespace {

constexpr int kThreads = 256;
constexpr int kItems = 8;
constexpr int kTile = kThreads * kItems;  // 2048
constexpr int kWarps = kThreads / 32;
constexpr int kFusedScanMaxTiles = 128;   // <= 262 144 keys: the scatter kernel scans the histograms itself

__global__ void __launch_bounds__(kThreads)
radix_hist_kernel(const uint64_t* __restrict__ keys, int n, int64_t stride, int shift,
                  uint32_t* __restrict__ block_hist, int nblk) {
  __shared__ uint32_t hist[256];
  const int b = blockIdx.y;
  keys += (int64_t)b * stride;
  hist[threadIdx.x] = 0;
  __syncthreads();
  const int base = blockIdx.x * kTile;
#pragma unroll
  for (int r = 0; r < kItems; ++r) {
    const int i = base + r * kThreads + threadIdx.x;
    if (i < n) atomicAdd(&hist[(keys[i] >> shift) & 255u], 1u);
  }
  __syncthreads();
  block_hist[((int64_t)b * 256 + threadIdx.x) * nblk + blockIdx.x] = hist[threadIdx.x];
}

// exclusive scan over `count` u32 entries per batch, one 1024-thread block per batch.
__global__ void __launch_bounds__(1024)
radix_scan_kernel(uint32_t* __restrict__ data, int count) {
  __shared__ uint32_t warp_sums[32];
  uint32_t* d = data + (int64_t)blockIdx.x * count;
  const int per = (count + 1023) / 1024;
  const int lo = min(count, (int)threadIdx.x * per), hi = min(count, lo + per);
  uint32_t s = 0;
  for (int i = lo; i < hi; ++i) s += d[i];
  uint32_t run = block_scan_excl<32>(s, warp_sums);
  for (int i = lo; i < hi; ++i) {
    const uint32_t v = d[i];
    d[i] = run;
    run += v;
  }
}

// Large sorts (more than kFusedScanMaxTiles tiles): the 256 x nblk counters of a batch are scanned
// by many blocks instead of one.  Each block scans one chunk of kScanChunk counters in place
// (exclusive, relative to the chunk) and publishes the chunk total; the block that finishes last
// (ticket counter) turns the chunk totals of every batch into exclusive chunk offsets.  The
// scatter kernel adds chunk_off[entry / kScanChunk] to the counter it reads.
constexpr int kScanChunk = 4096;   // counters per scan block: 1024 threads x 4

__global__ void __launch_bounds__(1024)
radix_scan_chunks_kernel(uint32_t* __restrict__ data, int count, int nchunks, uint32_t* __restrict__ chunk_tot,
                         uint32_t* __restrict__ ticket) {
  __shared__ uint32_t warp_sums[32];
  __shared__ bool is_last;
  const int b = blockIdx.y, c = blockIdx.x;
  uint32_t* d = data + (int64_t)b * count;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int i0 = c * kScanChunk + threadIdx.x * 4;
  uint32_t v[4], s = 0;
#pragma unroll
  for (int r = 0; r < 4; ++r) { v[r] = (i0 + r < count) ? d[i0 + r] : 0u; s += v[r]; }
  uint32_t total;
  uint32_t run = block_scan_excl<32>(s, warp_sums, &total);
  if (threadIdx.x == 0) chunk_tot[b * nchunks + c] = total;
#pragma unroll
  for (int r = 0; r < 4; ++r) { if (i0 + r < count) d[i0 + r] = run; run += v[r]; }
  // ---- last block: chunk totals -> exclusive chunk offsets, per batch --------------------------
  __threadfence();
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x == 0) *ticket = 0;                 // ready for the next pass
  // one warp per batch, 32 chunk totals per pass with the running carry; one chunk per 16 tiles of 2048 keys, so
  // 2^20 keys make 32 chunks and larger sorts take more than one pass
  for (int bb = w; bb < (int)gridDim.y; bb += 32) {
    uint32_t carry = 0;
    for (int base = 0; base < nchunks; base += 32) {
      const int k = base + lane;
      const uint32_t x = k < nchunks ? *reinterpret_cast<volatile uint32_t*>(chunk_tot + bb * nchunks + k) : 0u;
      const uint32_t xi = warp_inclusive_scan(x);
      if (k < nchunks) chunk_tot[bb * nchunks + k] = carry + xi - x;
      carry += __shfl_sync(0xffffffffu, xi, 31);
    }
  }
}

// FUSED_SCAN: block_offs holds the RAW per-tile histograms [batch][digit][tile]; every block derives
// its own offsets (row prefix up to its tile + totals of the lower digits), which saves the
// separate one-block scan launch.  Worth it only while a histogram row is short (each block reads
// 256 x nblk counters), i.e. for the ~100 k-point sorts of the ICP prologue.
template <int SCAN_MODE>   // 0: offsets fully scanned, 1: raw histograms (fused scan), 2: chunk-relative + chunk_off
__global__ void __launch_bounds__(kThreads)
radix_scatter_kernel(const uint64_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in,
                     uint64_t* __restrict__ keys_out, uint32_t* __restrict__ vals_out, int n,
                     int64_t stride, int shift, const uint32_t* __restrict__ block_offs,
                     int nblk, const uint32_t* __restrict__ chunk_off, int nchunks) {
  __shared__ uint32_t warp_hist[kWarps][256];
  const int b = blockIdx.y;
  keys_in += (int64_t)b * stride; vals_in += (int64_t)b * stride;
  keys_out += (int64_t)b * stride; vals_out += (int64_t)b * stride;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < kWarps * 256; i += kThreads) (&warp_hist[0][0])[i] = 0;
  __syncthreads();
  const int base = blockIdx.x * kTile + w * (32 * kItems);
  uint64_t key[kItems];
  uint32_t val[kItems], rank[kItems];
#pragma unroll
  for (int r = 0; r < kItems; ++r) {
    const int i = base + r * 32 + lane;
    const bool ok = i < n;
    key[r] = ok ? keys_in[i] : 0;
    val[r] = ok ? vals_in[i] : 0;
    const uint32_t d = ok ? (uint32_t)((key[r] >> shift) & 255u) : 0xffffu;
    const uint32_t peers = __match_any_sync(0xffffffffu, d);
    const uint32_t before = ok ? warp_hist[w][d] : 0;
    rank[r] = before + __popc(peers & ((1u << lane) - 1u));
    __syncwarp();
    if (ok && (peers & ((1u << lane) - 1u)) == 0) warp_hist[w][d] = before + __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  __shared__ uint32_t digit_base[kWarps];
  {  // exclusive scan across warps for digit = threadIdx.x, plus the global offset
    const int d = threadIdx.x;
    uint32_t run;
    if (SCAN_MODE == 1) {
      const uint32_t* row = block_offs + ((int64_t)b * 256 + d) * nblk;
      uint32_t before = 0, total = 0;
      for (int t = 0; t < nblk; ++t) { const uint32_t c = row[t]; if (t < (int)blockIdx.x) before += c; total += c; }
      run = block_scan_excl<kWarps>(total, digit_base) + before;   // exclusive scan of the digit totals
    } else {
      const int64_t e = (int64_t)d * nblk + blockIdx.x;          // entry inside this batch
      run = block_offs[(int64_t)b * 256 * nblk + e];
      if (SCAN_MODE == 2) run += chunk_off[b * nchunks + (int)(e / kScanChunk)];
    }
#pragma unroll
    for (int ww = 0; ww < kWarps; ++ww) {
      const uint32_t c = warp_hist[ww][d];
      warp_hist[ww][d] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kItems; ++r) {
    const int i = base + r * 32 + lane;
    if (i < n) {
      const uint32_t d = (uint32_t)((key[r] >> shift) & 255u);
      const uint32_t pos = warp_hist[w][d] + rank[r];
      keys_out[pos] = key[r];
      vals_out[pos] = val[r];
    }
  }
}

}  // namespace

void radix_scan_kernel_launch(uint32_t* data, int count, int batch, cudaStream_t stream) {
  radix_scan_kernel<<<batch, 1024, 0, stream>>>(data, count);
}

size_t radix_sort_scratch_bytes(int n, int batch) {
  const int nblk = ceil_div(n, kTile);
  const size_t count = (size_t)256 * (size_t)nblk;
  return ((size_t)batch * count + (size_t)batch * ((count + kScanChunk - 1) / kScanChunk) + 8) * sizeof(uint32_t);
}

size_t RadixPairs::bytes(int64_t stride, int n) {
  return (size_t)stride * (2 * sizeof(uint64_t) + 2 * sizeof(uint32_t)) + radix_sort_scratch_bytes(n, 1);
}

void RadixPairs::carve(void* base, int64_t stride) {
  keys[0] = (uint64_t*)base;
  keys[1] = keys[0] + stride;
  vals[0] = (uint32_t*)(keys[1] + stride);
  vals[1] = vals[0] + stride;
  scratch = vals[1] + stride;
}

// Sorts keys_a/vals_a (layout [batch][stride]); keys_b/vals_b are ping-pong buffers.
// `passes` 8-bit digits are sorted starting from bit 0 (8 = full 64-bit keys); for an even
// number of passes the sorted data ends in the *_a buffers, otherwise in *_b.
int radix_sort_pairs_u64(uint64_t* keys_a, uint32_t* vals_a, uint64_t* keys_b, uint32_t* vals_b,
                         int n, int batch, int64_t stride, uint32_t* scratch,
                         cudaStream_t stream, int passes) {
  if (n <= 0) return 0;
  const int nblk = ceil_div(n, kTile);
  const dim3 grid(nblk, batch);
  uint64_t* kin = keys_a; uint32_t* vin = vals_a;
  uint64_t* kout = keys_b; uint32_t* vout = vals_b;
  for (int pass = 0; pass < passes; ++pass) {
    const int shift = pass * 8;
    radix_hist_kernel<<<grid, kThreads, 0, stream>>>(kin, n, stride, shift, scratch, nblk);
    if (nblk <= kFusedScanMaxTiles) {
      radix_scatter_kernel<1><<<grid, kThreads, 0, stream>>>(kin, vin, kout, vout, n, stride, shift, scratch, nblk,
                                                             nullptr, 0);
    } else {
      const int count = 256 * nblk, nchunks = ceil_div(count, kScanChunk);
      uint32_t* chunk_tot = scratch + (int64_t)batch * count;     // [batch][nchunks], then the ticket
      uint32_t* ticket = chunk_tot + (int64_t)batch * nchunks;
      if (pass == 0) cudaMemsetAsync(ticket, 0, sizeof(uint32_t), stream);
      radix_scan_chunks_kernel<<<dim3(nchunks, batch), 1024, 0, stream>>>(scratch, count, nchunks, chunk_tot, ticket);
      radix_scatter_kernel<2><<<grid, kThreads, 0, stream>>>(kin, vin, kout, vout, n, stride, shift, scratch, nblk,
                                                             chunk_tot, nchunks);
    }
    uint64_t* tk = kin; kin = kout; kout = tk;
    uint32_t* tv = vin; vin = vout; vout = tv;
  }
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace smb
