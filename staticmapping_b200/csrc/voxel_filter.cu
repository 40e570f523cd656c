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
// output points is ascending (ix, iy, iz) by default (SM_VOXEL_ORDER_ASCENDING), whereas the reference's is
// the iteration order of a libstdc++ unordered_map.  That order matters downstream: CalculateNormals in
// std::nth_element's order permutes the one index array it is given, so its leaves, their summation order
// and representatives, and its column order all follow the voxel order.  SM_VOXEL_ORDER_UNORDERED_MAP
// reproduces the container's order (DESIGN §4f):
//   libstdc++ keeps all nodes in one singly linked list in which every bucket is one contiguous run.  An insert
//   into a non-empty bucket goes to the head of its run, one into an empty bucket to the front of the list; a
//   rehash to B buckets walks the old list front to back and moves each node to the front of the new list if its
//   new bucket is still empty, else to the head of that bucket's run.  Between two rehashes (an epoch e, from
//   c_e distinct keys on, B_e buckets, n_e keys at its end) the list is therefore sorted by (run key, within-run
//   key).  With t the insertion rank, r the position before the epoch's rehash and v = r for a voxel present
//   before it (t < c_e), v = t for one of the epoch's own: run key = n_e - 1 - (min v over the bucket), within-run
//   key = n_e - 1 - v.  Every old r is below every new t, so both keys put new runs before old ones and, inside a
//   run, new voxels (latest first) before old ones (last position first).
//   Each epoch is one bucket-min pass (atomicMin over B_e entries) and one radix sort of the n_e voxels
//   present on a key of 2 * ceil(log2 n_e) bits: about 2 m sorted keys over about log2 m epochs.
// Compiled with -fmad=false.
#include <limits.h>
#include <math.h>

#include <mutex>
#include <unordered_map>
#include <utility>
#include <vector>

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

// common/eigen_hash.h:31-43 with Scalar = int: boost's hash_combine on a 64-bit size_t over std::hash<int>, which
// sign-extends
__host__ __device__ __forceinline__ uint64_t vf_hash(const int32_t* k) {
  uint64_t seed = 0;
  for (int i = 0; i < 3; ++i) seed ^= (uint64_t)(int64_t)k[i] + 0x9e3779b9ull + (seed << 6) + (seed >> 2);
  return seed;
}

// mark[first member of voxel v] = v (ascending voxel index); mark is ~0u elsewhere
__global__ void __launch_bounds__(256)
vf_mark_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ voxel_start,
               const uint32_t* __restrict__ n_voxels_dev, uint32_t* __restrict__ mark) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= (int64_t)*n_voxels_dev) return;
  mark[order[voxel_start[v]]] = (uint32_t)v;
}

__global__ void __launch_bounds__(kCompactThreads)
vf_rank_count_kernel(const uint32_t* __restrict__ mark, int n, uint32_t* __restrict__ tile_cnt) {
  uint32_t c = 0;
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += mark[base + r] != ~0u;
  tile_count_store(c, tile_cnt);
}

// the first members in input order: voxel of insertion rank t -> its ascending index, first member and hash.  The key
// is int(lround(.)) as the reference forms it: a long past int's range wraps, as on GCC (no two voxels within the
// key's 2^21 span can meet so).
__global__ void __launch_bounds__(kCompactThreads)
vf_rank_scatter_kernel(const char* __restrict__ pts, int64_t stride, float voxel, const uint32_t* __restrict__ mark,
                       int n, const uint32_t* __restrict__ tile_off, uint64_t* __restrict__ hash,
                       uint32_t* __restrict__ asc, uint32_t* __restrict__ first) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) if (base + r < n) c += mark[base + r] != ~0u;
  uint32_t t = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n || mark[i] == ~0u) continue;
    long long ix, iy, iz;
    vf_index(reinterpret_cast<const float*>(pts + (int64_t)i * stride), voxel, &ix, &iy, &iz);   // finite: a member
    const int32_t k[3] = {(int32_t)ix, (int32_t)iy, (int32_t)iz};
    hash[t] = vf_hash(k);
    asc[t] = mark[i];
    first[t] = (uint32_t)i;
    ++t;
  }
}

// epoch [c, ne) with `buckets` buckets: table[b] = min v over the voxels present in bucket b (v = pos for t < c,
// t for the epoch's own inserts)
__global__ void __launch_bounds__(256)
vf_bucket_min_kernel(const uint64_t* __restrict__ hash, const uint32_t* __restrict__ pos, int ne, int c,
                     uint64_t buckets, uint32_t* __restrict__ bucket, uint32_t* __restrict__ table) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ne) return;
  const uint32_t b = (uint32_t)(hash[t] % buckets);   // _Mod_range_hashing
  bucket[t] = b;
  atomicMin(&table[b], t < c ? pos[t] : (uint32_t)t);
}

// the list position of every voxel after the epoch's rehash and inserts, as one sort key: run key, within-run key
__global__ void __launch_bounds__(256)
vf_epoch_key_kernel(const uint32_t* __restrict__ pos, const uint32_t* __restrict__ bucket,
                    const uint32_t* __restrict__ table, int ne, int c, int bits, uint64_t* __restrict__ keys,
                    uint32_t* __restrict__ vals) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= ne) return;
  const uint32_t top = (uint32_t)(ne - 1), v = t < c ? pos[t] : (uint32_t)t;
  keys[t] = ((uint64_t)(top - table[bucket[t]]) << bits) | (uint64_t)(top - v);
  vals[t] = (uint32_t)t;
}

__global__ void __launch_bounds__(256)
vf_epoch_pos_kernel(const uint32_t* __restrict__ sorted_vals, int ne, uint32_t* __restrict__ pos) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p < ne) pos[sorted_vals[p]] = (uint32_t)p;
}

// voxel of rank t -> its list position: its mean record and the scan index of its first member
__global__ void __launch_bounds__(256)
vf_emit_kernel(const float* __restrict__ staged, const uint32_t* __restrict__ asc, const uint32_t* __restrict__ first,
               const uint32_t* __restrict__ pos, int m, const uint32_t* __restrict__ index_in, float* __restrict__ out,
               uint32_t* __restrict__ out_index) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const int64_t p = pos[t], a = asc[t];
#pragma unroll
  for (int k = 0; k < 5; ++k) out[5 * p + k] = staged[5 * a + k];
  if (out_index) out_index[p] = index_in ? index_in[first[t]] : first[t];
}

// The schedule of a default-constructed std::unordered_map, from the policy object the container itself consults
// before every insert (_Hashtable::_M_insert_unique_node): _M_need_rehash(bucket count, element count, 1).
struct RehashSchedule {
  std::mutex mu;
  std::__detail::_Prime_rehash_policy policy;
  uint64_t buckets = 1;                                // the single bucket of an empty map
  int64_t done = 0;                                    // element counts 0 .. done - 1 have been asked about
  std::vector<std::pair<int64_t, uint64_t>> epochs;
};

}  // namespace

std::vector<std::pair<int64_t, uint64_t>> unordered_map_epochs(int64_t m) {
  static RehashSchedule sch;
  std::lock_guard<std::mutex> lock(sch.mu);
  for (; sch.done < m; ++sch.done) {
    const std::pair<bool, size_t> r = sch.policy._M_need_rehash(sch.buckets, (size_t)sch.done, 1);
    if (r.first) sch.buckets = r.second;
    if (r.first || sch.done == 0) sch.epochs.emplace_back(sch.done, sch.buckets);
  }
  std::vector<std::pair<int64_t, uint64_t>> out;
  for (const auto& e : sch.epochs) if (e.first < m) out.push_back(e);
  return out;
}

uint64_t vf_debug_hash_host(const int32_t* k3) { return vf_hash(k3); }

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

// SM_VOXEL_ORDER_UNORDERED_MAP, after vf_mean_kernel has written the ascending records into `staged`: the insertion
// ranks, then one pass per rehash epoch, then every record to its list position
int VoxelGrid::unordered_emit(const char* pts, int n, int64_t stride, float voxel, const uint32_t* index_in,
                              float* out, uint32_t* out_index, int64_t* m, cudaStream_t s) {
  const int tiles = compact_tiles(n);
  const int64_t st = (n + 63) & ~(int64_t)63;
  RadixPairs rp;
  rp.carve(sort.p, st);
  uint32_t* tc = (uint32_t*)tile_cnt.p;
  uint32_t* mk = (uint32_t*)mark.p;
  uint32_t* rc = (uint32_t*)rank_cnt.p;
  rank_stride = n;
  SMB_CUDA_OK(cudaMemsetAsync(mk, 0xff, (size_t)n * sizeof(uint32_t), s));
  vf_mark_kernel<<<ceil_div(n, 256), 256, 0, s>>>(rp.vals[0], (const uint32_t*)voxel_start.p, tc + tiles, mk);
  vf_rank_count_kernel<<<tiles, kCompactThreads, 0, s>>>(mk, n, rc);
  compact_scan(rc, tiles, s);
  vf_rank_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(pts, stride, voxel, mk, n, rc, hash(), asc(), first());
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t voxels = 0;
  long long host_meta[8] = {0};
  SMB_CUDA_OK(cudaMemcpyAsync(&voxels, tc + tiles, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaMemcpyAsync(host_meta, meta.p, sizeof(host_meta), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  if (host_meta[4]) return SM_ERR_BAD_ARGUMENT;
  const int mv = (int)voxels;
  *m = mv;
  if (mv == 0) return SM_OK;
  const std::vector<std::pair<int64_t, uint64_t>> epochs = unordered_map_epochs(mv);
  SMB_RC(table.reserve((size_t)epochs.back().second * sizeof(uint32_t)));
  uint32_t* tb = (uint32_t*)table.p;
  uint32_t* ps = pos();
  uint32_t* bk = bucket();
  if (epoch_trace) epoch_trace->clear();
  for (size_t e = 0; e < epochs.size(); ++e) {
    const int c = (int)epochs[e].first;
    const int ne = e + 1 < epochs.size() ? (int)epochs[e + 1].first : mv;
    const uint64_t buckets = epochs[e].second;
    const int bits = ne > 1 ? 64 - __builtin_clzll((unsigned long long)(ne - 1)) : 1;
    const int passes = (2 * bits + 7) / 8;
    SMB_CUDA_OK(cudaMemsetAsync(tb, 0xff, (size_t)buckets * sizeof(uint32_t), s));
    vf_bucket_min_kernel<<<ceil_div(ne, 256), 256, 0, s>>>(hash(), ps, ne, c, buckets, bk, tb);
    vf_epoch_key_kernel<<<ceil_div(ne, 256), 256, 0, s>>>(ps, bk, tb, ne, c, bits, rp.keys[0], rp.vals[0]);
    SMB_RC(radix_sort_pairs_u64(rp.keys[0], rp.vals[0], rp.keys[1], rp.vals[1], ne, 1, st, rp.scratch, s, passes));
    vf_epoch_pos_kernel<<<ceil_div(ne, 256), 256, 0, s>>>(rp.vals[passes & 1], ne, ps);
    SMB_CUDA_OK(cudaGetLastError());
    if (epoch_trace) {
      epoch_trace->emplace_back((size_t)ne);
      SMB_CUDA_OK(cudaMemcpyAsync(epoch_trace->back().data(), ps, (size_t)ne * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost, s));
      SMB_CUDA_OK(cudaStreamSynchronize(s));
    }
  }
  vf_emit_kernel<<<ceil_div(mv, 256), 256, 0, s>>>((const float*)staged.p, asc(), first(), ps, mv, index_in, out,
                                                   out_index);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return SM_OK;
}

int VoxelGrid::run(const char* pts, int64_t n, int64_t stride, float voxel, int32_t order, const uint32_t* index_in,
                   float* out, uint32_t* out_index, int64_t* m, cudaStream_t s) {
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
  if (order == SM_VOXEL_ORDER_UNORDERED_MAP) {
    SMB_RC(mark.reserve((size_t)n * sizeof(uint32_t)));
    SMB_RC(rank_cnt.reserve(compact_count_bytes(n)));
    SMB_RC(by_rank.reserve((size_t)n * (sizeof(uint64_t) + 4 * sizeof(uint32_t))));
    SMB_RC(staged.reserve((size_t)n * 5 * sizeof(float)));
    vf_mean_kernel<<<ceil_div((int64_t)n * 32, 256), 256, 0, s>>>(sd, vs, tc + tiles, (float*)staged.p);
    return unordered_emit(pts, ni, stride, voxel, index_in, out, out_index, m, s);
  }
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
  return sm_voxel_grid_filter_ordered(device, points, n, stride_bytes, voxel_size, SM_VOXEL_ORDER_ASCENDING, out,
                                      m_out);
}

extern "C" int sm_voxel_grid_filter_ordered(int device, const float* points, int64_t n, int64_t stride_bytes,
                                            float voxel_size, int32_t order, float* out, int64_t* m_out) {
  if (!points || !out || !m_out || n < 0 || n > (1 << 30) || stride_bytes < 16 || stride_bytes % 4 ||
      !(voxel_size > 1.e-6f) ||     // ConfigsValid(), filter_voxel_grid.cc:35
      (order != SM_VOXEL_ORDER_ASCENDING && order != SM_VOXEL_ORDER_UNORDERED_MAP))
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
  SMB_RC(vg.run((const char*)d_in.p, n, stride_bytes, voxel_size, order, nullptr, (float*)d_out.p, nullptr, &m, s));
  if (m > 0) SMB_CUDA_OK(cudaMemcpy(out, d_out.p, (size_t)m * 5 * sizeof(float), cudaMemcpyDeviceToHost));
  *m_out = m;
  return SM_OK;
}
