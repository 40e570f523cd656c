// pre_processers::filter::GroundRemoval (v1, pre_processors/filter_ground_removal.{h,cc}) on the device, behind its
// own handle (sm_ground_removal_*), built on the record-filter core of record_filter.h.
//
// Reference: SetInputCloud files every point under the key ((int)(x / leaf_size), (int)(y / leaf_size),
// (int)(z / leaf_size)) of a std::map compared lexicographically on signed ints (.h:56-62).  Filter walks the map in
// key order (.cc:74-108): a voxel of fewer than min_point_num_in_voxel points is skipped (in neither list); a voxel with
// iz <= 0 whose z range max_z - min_z (from -1e9 / 1e9, strict > / <) lies in [0, height_threshold] is ground and its
// points are outliers; every other voxel emits its records in input order and its points are inliers.  Both lists are
// sorted.  Here (bounds to voxels: voxel_sort, which plane_sampler.cu shares; lists: flag_list, which it shares too):
//   bounds   per-point voxel index (gr_index), per-axis min / max of the indices other than INT_MIN (grid-strided,
//            warp and block reductions, then one atomic per block on an order-preserving unsigned encoding)
//   key      63-bit key, 21 bits per axis: 0 for INT_MIN, else index - min + 1, so the keys ascend in the map's order
//   sort     radix_sort_pairs_u64 with the input index as payload; stable, so a voxel's points stay in input order
//   voxels   segment heads, ordered compaction (compact.cuh) -> voxel_start
//   decide   one warp per voxel, grid-strided: size test, z range (gr_z_update, then a warp reduction with the same
//            strict comparisons), gr_voxel_status; writes the emit flag of every sorted position and the status of
//            every input point
//   emit     emitted records gathered into sorted order with the flag counts, then filter_compact_records with the
//            sorted input indices as index_in (in the chain's stage, their scan indices: gr_scan_index_kernel)
//   lists    inliers and outliers: two ordered compactions of the status over the input (the own handle only)
// One read-back, at the end: the per-axis bounds (the span check), the number emitted and the two list lengths.
// Compiled with -fmad=false.
#include <limits.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <utility>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"
#include "record_filter.h"
#include "reduce.cuh"

namespace smb {
namespace {

constexpr int kGrSlotBits = 21;
constexpr uint32_t kGrSlots = 1u << kGrSlotBits;   // slot 0: INT_MIN; slots 1 .. 2^21 - 1: index - min + 1
constexpr uint32_t kGrSign = 0x80000000u;           // int -> order-preserving unsigned
// meta[0..2]: ~enc(min index) per axis, meta[3..5]: enc(max index), both over the indices other than INT_MIN (0: none)
// (voxel_sort); meta[8]: records emitted, meta[9]: inliers, meta[10]: outliers
constexpr int kGrMeta = 12;

// grid-strided, a few blocks per SM: one atomic per block and bound, so that the atomics do not serialise on meta
__global__ void __launch_bounds__(256)
gr_bounds_kernel(const char* __restrict__ pts, int64_t stride, int n, float leaf, uint32_t* __restrict__ meta) {
  __shared__ uint32_t block[6];
  if (threadIdx.x < 6) block[threadIdx.x] = 0u;
  __syncthreads();
  uint32_t b[6] = {0u, 0u, 0u, 0u, 0u, 0u};          // ~enc(min), then enc(max) per axis
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int ixyz[3];
    gr_index(gr_point(pts, stride, i), leaf, ixyz);
    for (int d = 0; d < 3; ++d)
      if (ixyz[d] != INT_MIN) {
        const uint32_t u = (uint32_t)ixyz[d] ^ kGrSign;
        b[d] = max(b[d], ~u);
        b[3 + d] = max(b[3 + d], u);
      }
  }
  for (int j = 0; j < 6; ++j) b[j] = warp_max(b[j]);
  if ((threadIdx.x & 31) == 0)
    for (int j = 0; j < 6; ++j) if (b[j]) atomicMax(&block[j], b[j]);
  __syncthreads();
  if (threadIdx.x < 6 && block[threadIdx.x]) atomicMax(&meta[threadIdx.x], block[threadIdx.x]);
}

__global__ void __launch_bounds__(256)
gr_key_kernel(const char* __restrict__ pts, int64_t stride, int n, float leaf, const uint32_t* __restrict__ meta,
              uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int ixyz[3];
  gr_index(gr_point(pts, stride, i), leaf, ixyz);
  uint64_t key = 0;
  for (int d = 0; d < 3; ++d) {
    uint64_t slot = 0;
    if (ixyz[d] != INT_MIN) {
      const int lo = (int)(~meta[d] ^ kGrSign);
      slot = (uint64_t)((int64_t)ixyz[d] - lo + 1) & (kGrSlots - 1);   // the host refuses a span that does not fit
    }
    key = (key << kGrSlotBits) | slot;
  }
  keys[i] = key;
  vals[i] = (uint32_t)i;
}

__device__ __forceinline__ uint32_t gr_is_head(const uint64_t* keys, int k) {
  return (k == 0 || keys[k] != keys[k - 1]) ? 1u : 0u;
}

__global__ void __launch_bounds__(kCompactThreads)
gr_heads_count_kernel(const uint64_t* __restrict__ keys, int n, uint32_t* __restrict__ tile_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += gr_is_head(keys, base + r);
  tile_count_store(c, tile_cnt);
}

// voxel_start[v] = first sorted position of voxel v; voxel_start[n_voxels] = n
__global__ void __launch_bounds__(kCompactThreads)
gr_heads_scatter_kernel(const uint64_t* __restrict__ keys, int n, const uint32_t* __restrict__ tile_off,
                        uint32_t* __restrict__ voxel_start) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n) ? gr_is_head(keys, base + r) : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) if (f[r]) voxel_start[pos++] = (uint32_t)(base + r);
  if (blockIdx.x == 0 && threadIdx.x == 0) voxel_start[tile_off[gridDim.x]] = (uint32_t)n;
}

// one warp per voxel, grid-strided over the *n_voxels voxels: emit[k] for every sorted position k of the voxel,
// status[i] for every input point i
__global__ void __launch_bounds__(256)
gr_decide_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ order,
                 const uint32_t* __restrict__ voxel_start, const uint32_t* __restrict__ n_voxels, float leaf,
                 int32_t min_points, float height_threshold, uint8_t* __restrict__ emit, uint8_t* __restrict__ status) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t nv = *n_voxels;
  for (int64_t v = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; v < nv; v += warps) {
    const uint32_t s0 = voxel_start[v], s1 = voxel_start[v + 1];
    int ixyz[3];
    gr_index(gr_point(pts, stride, order[s0]), leaf, ixyz);
    float max_z = -1.e9f, min_z = 1.e9f;
    if ((int32_t)(s1 - s0) >= min_points && ixyz[2] <= 0) {   // warp-uniform
      for (uint32_t k = s0 + lane; k < s1; k += 32) {
        const float z = gr_point(pts, stride, order[k])[2];
        gr_z_update(z, z, &max_z, &min_z);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1)
        gr_z_update(__shfl_xor_sync(0xffffffffu, max_z, o), __shfl_xor_sync(0xffffffffu, min_z, o), &max_z, &min_z);
    }
    // lanes may hold zeros of different signs here; either gives the same decision
    const int st = gr_voxel_status((int32_t)(s1 - s0), ixyz[2], max_z, min_z, min_points, height_threshold);
    for (uint32_t k = s0 + lane; k < s1; k += 32) {
      emit[k] = st == kGrKept ? 1 : 0;
      status[order[k]] = (uint8_t)st;
    }
  }
}

// the emitted records in sorted order (the others are not written) and the emit counts of the ordered compaction
__global__ void __launch_bounds__(kCompactThreads)
gr_gather_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ order, int n,
                 const uint8_t* __restrict__ emit, float* __restrict__ sorted, uint32_t* __restrict__ tile_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    const int k = base + r;
    if (k >= n) break;
    if (!emit[k]) continue;
    const float* p = gr_point(pts, stride, order[k]);
    float* q = sorted + (int64_t)k * 5;
    q[0] = p[0]; q[1] = p[1]; q[2] = p[2]; q[3] = p[3]; q[4] = p[4];
    ++c;
  }
  tile_count_store(c, tile_cnt);
}

__global__ void __launch_bounds__(kCompactThreads)
gr_list_count_kernel(const uint8_t* __restrict__ status, int n, int want, uint32_t* __restrict__ tile_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n && status[base + r] == want) ++c;
  tile_count_store(c, tile_cnt);
}

// list: the input indices whose status is `want`, ascending; *m = their number
__global__ void __launch_bounds__(kCompactThreads)
gr_list_scatter_kernel(const uint8_t* __restrict__ status, int n, int want, const uint32_t* __restrict__ tile_off,
                       int32_t* __restrict__ list, uint32_t* __restrict__ m) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n && status[base + r] == want) ? 1u : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) if (f[r]) list[pos++] = base + r;
  if (blockIdx.x == 0 && threadIdx.x == 0) *m = tile_off[gridDim.x];
}

// scan[k] = index_in[order[k]]: the scan index of the point at sorted position k, when the input is a chain stage's
__global__ void __launch_bounds__(256)
gr_scan_index_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ index_in, int n,
                     uint32_t* __restrict__ scan) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) scan[k] = index_in[order[k]];
}

}  // namespace

int voxel_sort(const char* pts, int n, int64_t stride, float leaf, const RadixPairs& rp, uint32_t* meta,
               uint32_t* tile_cnt, uint32_t* voxel_start, cudaStream_t s) {
  const int tiles = compact_tiles(n);
  const int blocks = ceil_div(n, 256);
  gr_bounds_kernel<<<std::min(blocks, 4 * kNumSMs), 256, 0, s>>>(pts, stride, n, leaf, meta);
  gr_key_kernel<<<blocks, 256, 0, s>>>(pts, stride, n, leaf, meta, rp.keys[0], rp.vals[0]);
  SMB_RC(radix_sort_pairs_u64(rp.keys[0], rp.vals[0], rp.keys[1], rp.vals[1], n, 1, voxel_sort_stride(n), rp.scratch,
                              s, 8));
  // 8 passes: the sorted pairs are back in the first buffers
  gr_heads_count_kernel<<<tiles, kCompactThreads, 0, s>>>(rp.keys[0], n, tile_cnt);
  compact_scan(tile_cnt, tiles, s);                     // tile_cnt[tiles] = the number of voxels
  gr_heads_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(rp.keys[0], n, tile_cnt, voxel_start);
  return SM_OK;
}

bool voxel_span_ok(const uint32_t* host_meta) {
  for (int d = 0; d < 3; ++d) {
    if (!host_meta[3 + d]) continue;                    // no index but INT_MIN on this axis
    const int64_t lo = (int)(~host_meta[d] ^ kGrSign), hi = (int)(host_meta[3 + d] ^ kGrSign);
    if (hi - lo + 1 > (int64_t)kGrSlots - 1) return false;
  }
  return true;
}

void flag_list(const uint8_t* flag, int n, int want, uint32_t* tile_cnt, int32_t* list, uint32_t* m, cudaStream_t s) {
  const int tiles = compact_tiles(n);
  gr_list_count_kernel<<<tiles, kCompactThreads, 0, s>>>(flag, n, want, tile_cnt);
  compact_scan(tile_cnt, tiles, s);
  gr_list_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(flag, n, want, tile_cnt, list, m);
}

// host builds of the per-point index and the per-voxel decision (test hooks sm_debug_ground_removal_*_host)
void gr_debug_index_host(const float* p, float leaf, int* ixyz) { gr_index(p, leaf, ixyz); }
int gr_debug_voxel_host(const float* z, int64_t count, int iz, int32_t min_points, float height_threshold,
                        float* max_min) {
  float max_z = -1.e9f, min_z = 1.e9f;
  if (count >= min_points && iz <= 0)
    for (int64_t k = 0; k < count; ++k) gr_z_update(z[k], z[k], &max_z, &min_z);
  max_min[0] = max_z;
  max_min[1] = min_z;
  return gr_voxel_status((int32_t)count, iz, max_z, min_z, min_points, height_threshold);
}

int GroundRemoval::reserve(int64_t n) {
  SMB_RC(sort.reserve(RadixPairs::bytes(voxel_sort_stride(n), (int)n)));
  SMB_RC(tile_cnt.reserve(4 * compact_count_bytes(n)));
  SMB_RC(voxel_start.reserve(((size_t)n + 1) * sizeof(uint32_t)));
  SMB_RC(emit.reserve((size_t)n));
  SMB_RC(status.reserve((size_t)n));
  SMB_RC(sorted.reserve((size_t)n * 20));
  SMB_RC(meta.reserve(kGrMeta * sizeof(uint32_t)));
  SMB_RC(inliers_next.reserve((size_t)n * sizeof(int32_t)));
  return outliers_next.reserve((size_t)n * sizeof(int32_t));
}

int GroundRemoval::run(const char* pts, int64_t n, int64_t stride, const uint32_t* index_in, float* out,
                       uint32_t* out_index, int64_t* m, cudaStream_t s, bool lists) {
  const float leaf = params.leaf_size;
  const int ni = (int)n;
  const int tiles = compact_tiles(n);
  SMB_RC(reserve(n));
  RadixPairs rp;
  rp.carve(sort.p, voxel_sort_stride(n));
  uint32_t* mt = (uint32_t*)meta.p;
  uint32_t* tc[4];
  for (int j = 0; j < 4; ++j) tc[j] = (uint32_t*)tile_cnt.p + (size_t)j * (tiles + 1);
  SMB_CUDA_OK(cudaMemsetAsync(mt, 0, kGrMeta * sizeof(uint32_t), s));
  SMB_RC(voxel_sort(pts, ni, stride, leaf, rp, mt, tc[0], (uint32_t*)voxel_start.p, s));
  const uint32_t* order = rp.vals[0];
  const int decide_blocks = (int)std::min<int64_t>(ceil_div(n, 8), 32 * kNumSMs);
  gr_decide_kernel<<<decide_blocks, 256, 0, s>>>(pts, stride, order, (const uint32_t*)voxel_start.p, tc[0] + tiles,
                                                 leaf, params.min_point_num_in_voxel, params.height_threshold,
                                                 (uint8_t*)emit.p, (uint8_t*)status.p);
  gr_gather_kernel<<<tiles, kCompactThreads, 0, s>>>(pts, stride, order, ni, (const uint8_t*)emit.p,
                                                     (float*)sorted.p, tc[1]);
  // the scan index of every sorted position, in the sort's free ping-pong buffer, for the scatter to carry
  const uint32_t* scan = order;
  if (index_in) {
    gr_scan_index_kernel<<<ceil_div(n, 256), 256, 0, s>>>(order, index_in, ni, rp.vals[1]);
    scan = rp.vals[1];
  }
  filter_compact_records((const char*)sorted.p, 20, scan, ni, (const uint8_t*)emit.p, tc[1], out, out_index, mt + 8,
                         s);
  const std::pair<int, DevBuf*> list_of[2] = {{kGrKept, &inliers_next}, {kGrGround, &outliers_next}};
  if (lists)
    for (int j = 0; j < 2; ++j)
      flag_list((const uint8_t*)status.p, ni, list_of[j].first, tc[2 + j], (int32_t*)list_of[j].second->p, mt + 9 + j,
                s);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t host[11];
  SMB_CUDA_OK(cudaMemcpyAsync(host, mt, sizeof(host), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  if (!voxel_span_ok(host)) return SM_ERR_BAD_ARGUMENT;
  if (lists) {
    std::swap(inliers, inliers_next);
    std::swap(outliers, outliers_next);
    n_inliers = host[9];
    n_outliers = host[10];
  }
  *m = (int64_t)host[8];
  return SM_OK;
}

}  // namespace smb

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace smb;

struct sm_ground_removal : RecordFilter {
  GroundRemoval f;
  explicit sm_ground_removal(int device) : RecordFilter(device, "GroundRemoval") {}
};

extern "C" {

int sm_ground_removal_create(int device, sm_ground_removal** out) { return create_record_filter(device, out); }

int sm_ground_removal_destroy(sm_ground_removal* h) { return destroy_record_filter(h); }

int sm_ground_removal_set_param(sm_ground_removal* h, const char* name, int type, const char* text) {
  if (!h || !name || !text) return SM_ERR_BAD_ARGUMENT;
  return h->set_param(h->f.params, name, type, text);
}

int sm_ground_removal_run_device(sm_ground_removal* h, const float* dev_points, int64_t n, int64_t stride_bytes,
                                 float* dev_out, int64_t* m_out, int32_t* dev_index, void* cuda_stream) {
  if (!h || !records_ok(dev_points, n, stride_bytes, dev_out, m_out)) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(h->use_device());
  if (n == 0) {
    *m_out = 0;
    h->f.n_inliers = h->f.n_outliers = 0;
    return SM_OK;
  }
  uint32_t* idx = (uint32_t*)dev_index;
  if (!idx) {
    SMB_RC(h->cuda_fail(h->host_idx.reserve((size_t)n * sizeof(int32_t))));
    idx = (uint32_t*)h->host_idx.p;
  }
  const int rc = h->f.run((const char*)dev_points, n, stride_bytes, nullptr, dev_out, idx, m_out,
                          (cudaStream_t)cuda_stream, true);
  if (rc == SM_ERR_BAD_ARGUMENT)
    return h->fail(rc, "the voxel indices of an axis span more than 2^21 - 1 voxels (the 63-bit voxel key)");
  return h->cuda_fail(rc);
}

int sm_ground_removal_run(sm_ground_removal* h, const float* points, int64_t n, int64_t stride_bytes, float* out,
                          int64_t* m_out, int32_t* index) {
  if (!h || !records_ok(points, n, stride_bytes, out, m_out)) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(h->use_device());
  return run_record_filter(h, sm_ground_removal_run_device, points, n, stride_bytes, out, m_out, index);
}

int sm_ground_removal_indices(const sm_ground_removal* h, int32_t* inliers, int64_t* n_inliers, int32_t* outliers,
                              int64_t* n_outliers) {
  if (!h || !n_inliers || !n_outliers) return SM_ERR_BAD_ARGUMENT;
  *n_inliers = h->f.n_inliers;
  *n_outliers = h->f.n_outliers;
  const bool copy_in = inliers && h->f.n_inliers > 0, copy_out = outliers && h->f.n_outliers > 0;
  if (!copy_in && !copy_out) return SM_OK;
  SMB_RC(select_device(h->device));
  if (copy_in)
    SMB_CUDA_OK(cudaMemcpy(inliers, h->f.inliers.p, (size_t)h->f.n_inliers * sizeof(int32_t), cudaMemcpyDeviceToHost));
  if (copy_out)
    SMB_CUDA_OK(cudaMemcpy(outliers, h->f.outliers.p, (size_t)h->f.n_outliers * sizeof(int32_t),
                           cudaMemcpyDeviceToHost));
  return SM_OK;
}

const char* sm_ground_removal_last_error(const sm_ground_removal* h) { return h ? h->error : ""; }

}  // extern "C"
