// pre_processers::filter::VoxelGrid::Filter on the device
// (pre_processors/filter_voxel_grid.cc:37-78; used by Submap::InsertFrame's down-sampling,
// builder/submap.cc:144-158, the step that produces the ICP / NDT targets).
//
// Reference: every point goes into std::unordered_map<Vector3i, vector<point>> under the key
// (lround(x / s), lround(y / s), lround(z / s)); each voxel emits the mean of x, y, z, intensity,
// accumulated in double in insertion order (== input order), cast to float; factor = 0.
// Here: 63-bit voxel key per point -> stable radix sort (points of a voxel stay in input order)
// -> segment heads -> points gathered into voxel order -> one warp per voxel adds the four double
// chains in order (addends staged through shared memory, like ndt_leaf_kernel) -> one output
// point per voxel; in the filter chain, also the scan index of each voxel's first member.  Every output value is bit-identical to the reference's; the ORDER of the
// output points is ascending (ix, iy, iz), whereas the reference's is the iteration order of a
// libstdc++ unordered_map (an accident of its rehash history; nothing downstream depends on it
// beyond summation order).  Compiled with -fmad=false.
#include <limits.h>
#include <math.h>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace smb {
namespace {

constexpr long long kSpan = 1ll << 21;   // voxel indices of one axis must span < 2^21 (3 x 21-bit key)

// meta[0..2]: per-axis minimum voxel index over the finite points; meta[3]: dropped (non-finite) points;
// meta[4]: 1 if an axis spans 2^21 voxels or more
__host__ __device__ __forceinline__ bool vf_index(const float* p, float voxel, long long* ix, long long* iy, long long* iz) {
  const float qx = p[0] / voxel, qy = p[1] / voxel, qz = p[2] / voxel;
  // std::lround of a NaN / inf quotient is unspecified in the reference: such points are dropped here
  if (!(fabsf(qx) < 9.0e18f && fabsf(qy) < 9.0e18f && fabsf(qz) < 9.0e18f)) return false;
  *ix = llroundf(qx); *iy = llroundf(qy); *iz = llroundf(qz);
  return true;
}

__global__ void __launch_bounds__(256)
vf_min_kernel(const char* __restrict__ pts, int64_t stride, int n, float voxel, long long* __restrict__ meta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  long long ix = LLONG_MAX, iy = LLONG_MAX, iz = LLONG_MAX;
  if (i < n) {
    long long a, b, c;
    if (vf_index(reinterpret_cast<const float*>(pts + (int64_t)i * stride), voxel, &a, &b, &c)) { ix = a; iy = b; iz = c; }
  }
  ix = warp_min(ix); iy = warp_min(iy); iz = warp_min(iz);
  if ((threadIdx.x & 31) == 0) { atomicMin(&meta[0], ix); atomicMin(&meta[1], iy); atomicMin(&meta[2], iz); }
}

__global__ void __launch_bounds__(256)
vf_key_kernel(const char* __restrict__ pts, int64_t stride, int n, float voxel, uint64_t* __restrict__ keys,
              uint32_t* __restrict__ vals, long long* __restrict__ meta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long ix, iy, iz;
  uint64_t key = ~0ull;                      // dropped points sort behind every voxel
  if (vf_index(reinterpret_cast<const float*>(pts + (int64_t)i * stride), voxel, &ix, &iy, &iz)) {
    // offsets from the cloud's own minimum: the key order stays ascending (ix, iy, iz)
    const unsigned long long ox = (unsigned long long)(ix - meta[0]), oy = (unsigned long long)(iy - meta[1]),
                             oz = (unsigned long long)(iz - meta[2]);
    if (ox < (unsigned long long)kSpan && oy < (unsigned long long)kSpan && oz < (unsigned long long)kSpan)
      key = (ox << 42) | (oy << 21) | oz;
    else
      atomicExch((unsigned long long*)&meta[4], 1ull);
  } else {
    atomicAdd((unsigned long long*)&meta[3], 1ull);
  }
  keys[i] = key;
  vals[i] = (uint32_t)i;
}

__device__ __forceinline__ uint32_t vf_is_head(const uint64_t* keys, int i) {
  return (keys[i] != ~0ull && (i == 0 || keys[i] != keys[i - 1])) ? 1u : 0u;
}

__global__ void __launch_bounds__(kCompactThreads)
vf_heads_count_kernel(const uint64_t* __restrict__ keys, int n, uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += vf_is_head(keys, base + r);
  tile_count_store(c, tile_cnt);
}

// voxel_start[v] = first sorted position of voxel v; voxel_start[n_voxels] = n
__global__ void __launch_bounds__(kCompactThreads)
vf_heads_scatter_kernel(const uint64_t* __restrict__ keys, int n, const uint32_t* __restrict__ tile_off,
                        uint32_t* __restrict__ voxel_start, const long long* __restrict__ meta) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n) ? vf_is_head(keys, base + r) : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) if (f[r]) voxel_start[pos++] = (uint32_t)(base + r);
  if (blockIdx.x == 0 && threadIdx.x == 0) voxel_start[tile_off[gridDim.x]] = (uint32_t)(n - (int)meta[3]);   // sentinel: first dropped point
}

__global__ void __launch_bounds__(256)
vf_gather_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ order, int n,
                 float4* __restrict__ sorted) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float* p = reinterpret_cast<const float*>(pts + (int64_t)order[k] * stride);
  sorted[k] = make_float4(p[0], p[1], p[2], p[3]);
}

// one warp per voxel; lanes 0..3 own the running sums of x, y, z, intensity
__global__ void __launch_bounds__(256)
vf_mean_kernel(const float4* __restrict__ sorted, const uint32_t* __restrict__ voxel_start,
               const uint32_t* __restrict__ n_voxels_dev, float* __restrict__ out) {
  constexpr int kPad = 33;
  __shared__ double s_d[8][4 * kPad];
  const int64_t v = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;    // n may exceed 2^27: 64-bit
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  if (v >= (int64_t)*n_voxels_dev) return;
  const uint32_t s0 = voxel_start[v], s1 = voxel_start[v + 1];
  double* sd = s_d[wib];
  const double* mine = sd + min(lane, 3) * kPad;
  double acc = 0.0;
  for (uint32_t base = s0; base < s1; base += 32) {
    const uint32_t i = min(base + (uint32_t)lane, s1 - 1);
    const float4 p = sorted[i];
    sd[0 * kPad + lane] = (double)p.x; sd[1 * kPad + lane] = (double)p.y;
    sd[2 * kPad + lane] = (double)p.z; sd[3 * kPad + lane] = (double)p.w;
    __syncwarp();
    const int cnt = (int)min(32u, s1 - base);
    if (cnt == 32) {
      double t[32];
#pragma unroll
      for (int u = 0; u < 32; ++u) t[u] = mine[u];
#pragma unroll
      for (int u = 0; u < 32; ++u) acc += t[u];
    } else {
      for (int u = 0; u < cnt; ++u) acc += mine[u];
    }
    __syncwarp();
  }
  if (lane < 4) out[5 * v + lane] = (float)(acc / (double)(int)(s1 - s0));   // sum / size, size is an int
  if (lane == 4) out[5 * v + 4] = 0.0f;                                      // factor keeps its default
}

// out_index[v] = the scan index of voxel v's first member in input order (the sort is stable: its first sorted position)
__global__ void __launch_bounds__(256)
vf_first_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ voxel_start,
                const uint32_t* __restrict__ n_voxels_dev, const uint32_t* __restrict__ index_in,
                uint32_t* __restrict__ out_index) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (int64_t)*n_voxels_dev) return;
  const uint32_t i = order[voxel_start[v]];
  out_index[v] = index_in ? index_in[i] : i;
}

}  // namespace

// host build of the voxel index of one point (test hook sm_debug_voxel_index op 0)
bool vf_debug_index_host(const float* p, float voxel, long long* ixyz) { return vf_index(p, voxel, &ixyz[0], &ixyz[1], &ixyz[2]); }

int VoxelGrid::reserve(int64_t n) {
  const int64_t st = (n + 63) & ~(int64_t)63;
  SMB_RC(sort.reserve(RadixPairs::bytes(st, (int)n)));
  SMB_RC(tile_cnt.reserve(compact_count_bytes(n)));
  SMB_RC(voxel_start.reserve(((size_t)n + 8) * sizeof(uint32_t)));
  SMB_RC(sorted.reserve((size_t)n * sizeof(float4)));
  return meta.reserve(8 * sizeof(long long));
}

int VoxelGrid::run(const char* pts, int64_t n, int64_t stride, float voxel, const uint32_t* index_in, float* out,
                   uint32_t* out_index, int64_t* m, cudaStream_t s) {
  const int ni = (int)n;
  const int tiles = compact_tiles(n);
  const int64_t st = (n + 63) & ~(int64_t)63;
  SMB_RC(reserve(n));
  RadixPairs rp;
  rp.carve(sort.p, st);
  uint32_t* tc = (uint32_t*)tile_cnt.p;
  uint32_t* vs = (uint32_t*)voxel_start.p;
  float4* sd = (float4*)sorted.p;
  long long* mt = (long long*)meta.p;
  const long long meta_init[8] = {LLONG_MAX, LLONG_MAX, LLONG_MAX, 0, 0, 0, 0, 0};
  SMB_CUDA_OK(cudaMemcpyAsync(mt, meta_init, sizeof(meta_init), cudaMemcpyHostToDevice, s));
  vf_min_kernel<<<ceil_div(n, 256), 256, 0, s>>>(pts, stride, ni, voxel, mt);
  vf_key_kernel<<<ceil_div(n, 256), 256, 0, s>>>(pts, stride, ni, voxel, rp.keys[0], rp.vals[0], mt);
  SMB_RC(radix_sort_pairs_u64(rp.keys[0], rp.vals[0], rp.keys[1], rp.vals[1], ni, 1, st, rp.scratch, s, 8));
  // 8 passes: the sorted pairs are back in the first buffers
  vf_heads_count_kernel<<<tiles, kCompactThreads, 0, s>>>(rp.keys[0], ni, tc);
  compact_scan(tc, tiles, s);                                                   // tc[tiles] = number of voxels
  vf_heads_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(rp.keys[0], ni, tc, vs, mt);
  vf_gather_kernel<<<ceil_div(n, 256), 256, 0, s>>>(pts, stride, rp.vals[0], ni, sd);
  vf_mean_kernel<<<ceil_div((int64_t)n * 32, 256), 256, 0, s>>>(sd, vs, tc + tiles, out);
  if (out_index) vf_first_kernel<<<ceil_div(n, 256), 256, 0, s>>>(rp.vals[0], vs, tc + tiles, index_in, out_index);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t voxels = 0;
  long long host_meta[8] = {0};
  SMB_CUDA_OK(cudaMemcpyAsync(&voxels, tc + tiles, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaMemcpyAsync(host_meta, mt, sizeof(host_meta), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  if (host_meta[4]) return SM_ERR_BAD_ARGUMENT;   // the finite points span 2^21 voxels or more along an axis
  *m = (int64_t)voxels;
  return SM_OK;
}

}  // namespace smb

using namespace smb;

extern "C" int sm_voxel_grid_filter(int device, const float* points, int64_t n, int64_t stride_bytes,
                                    float voxel_size, float* out, int64_t* m_out) {
  if (!points || !out || !m_out || n < 0 || n > (1 << 30) || stride_bytes < 16 || stride_bytes % 4 ||
      !(voxel_size > 1.e-6f))       // ConfigsValid(), filter_voxel_grid.cc:35
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  *m_out = 0;
  if (n == 0) return SM_OK;
  const size_t in_bytes = (size_t)n * (size_t)stride_bytes;
  DevBuf d_in, d_out;
  VoxelGrid vg;
  SMB_RC(d_in.reserve(in_bytes));
  SMB_RC(d_out.reserve((size_t)n * 20));
  cudaStream_t s = nullptr;
  SMB_CUDA_OK(cudaMemcpyAsync(d_in.p, points, in_bytes, cudaMemcpyHostToDevice, s));
  int64_t m = 0;
  SMB_RC(vg.run((const char*)d_in.p, n, stride_bytes, voxel_size, nullptr, (float*)d_out.p, nullptr, &m, s));
  if (m > 0) SMB_CUDA_OK(cudaMemcpy(out, d_out.p, (size_t)m * 5 * sizeof(float), cudaMemcpyDeviceToHost));
  *m_out = m;
  return SM_OK;
}
