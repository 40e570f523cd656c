// RangeImage::DepthCluster on the device (pre_processors/filter_range_image.cc:143-173, :245-309): the range image of
// Filter (:82-141) segmented by the angle criterion of Bogoslavskyi and Stachniss, with the reference's labels and
// the reference's visiting order.
//
//   image      the pixel owners of the RangeImage stage (range_image_owner, filters.cu: the first input point per
//              pixel), then one pass for the owner's range sqrtf(x^2 + y^2 + z^2) of the offset point.
//   edges      one pass: a 6-bit mask per pixel over the neighbour steps (0,1) (0,-1) (0,2) (0,-2) (1,0) (-1,0)
//              (:38-43), bit k set iff the neighbour is in the image and occupied and depth_edge holds.  The
//              predicate is symmetric in the pair, so the mask is too: both ends evaluate the same expression.
//   components union-find over the forward edges (0,1) (0,2) (1,0), hooking the larger root under the smaller with
//              atomicCAS (ECL-CC); every tree's root is its smallest row-major pixel, the seed the reference's scan
//              (:146-158) reaches first.  Labels are 1 + the rank of the root among all roots (ordered compaction,
//              compact.cuh), so dropped components take a label too, as in the reference.  Sizes per label.
//   order      the components of >= 20 pixels are compacted in label order with their output offsets (two scans
//              of per-tile counts, however many components there are); then one CTA per kept component, on a grid
//              of at most kBfsCtas CTAs that stride over them, runs LabelOneComponent's FIFO level by level, the
//              queue being the cluster's own slice of the output.  The pop order of std::queue is BFS order in which a pixel of
//              level L + 1 sits at (queue position r of its first-popped parent with an edge, step k): every
//              frontier entry r claims each edge neighbour with atomicMin(r * 6 + k), then the winners are
//              compacted in (r, k) order by a block scan.  Keys grow with r, so a pixel claimed on an earlier level
//              never wins again.  One launch for all levels of all components.
//   emit       clusters in ascending label (std::map, :159-172), each in its queue order: x, y, z of the un-offset
//              input point, the label and the input index.
// Compiled with -fmad=false like filters.cu.  sinf / cosf of the two angular resolutions are taken on the host (the
// reference's own libm calls); atan2f is CUDA's, so an edge whose beta lies within a few ulps of the threshold can
// differ from the reference (DESIGN.md section 4h).
#include <math.h>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"

namespace smb {
namespace {

constexpr int kBfsThreads = 256;
constexpr int kBfsCtas = 1024;          // the BFS grid: each CTA takes every 1024th kept component
constexpr uint32_t kMinCluster = 20;    // a cluster needs at least 20 points (:306)
constexpr uint32_t kNone = 0xffffffffu;

constexpr float kDepthThreshold = (float)(10 / 180. * M_PI);   // segmentation_rad_threshold_ (filter_range_image.h:101)

__host__ __device__ inline bool depth_occupied(float r) { return !((double)r < 1.e-6); }   // matrix_image_ < 1.e-6

// :288-301 for two occupied pixels of ranges a, b, s / c = sinf / cosf of the step's resolution; symmetric in a, b
__host__ __device__ inline bool depth_edge(float a, float b, float s, float c, float* beta_out = nullptr) {
  const float d1 = a < b ? b : a, d2 = b < a ? b : a;     // std::max, std::min
  const float beta = atan2f(d2 * s, d1 - d2 * c);
  if (beta_out) *beta_out = beta;
  return beta > kDepthThreshold;
}

// neighbour pixel of (row, col) by step k, -1 outside the rows (:273-281: columns wrap once)
__host__ __device__ inline int depth_neighbor(int row, int col, int k, int V, int H) {
  const int dr = k == 4 ? 1 : (k == 5 ? -1 : 0);
  const int dc = k >= 4 ? 0 : ((k & 1) ? -(1 + (k >> 1)) : 1 + (k >> 1));
  const int r = row + dr;
  if (r < 0 || r >= V) return -1;
  int c = col + dc;
  if (c < 0) c += H; else if (c >= H) c -= H;
  return r * H + c;
}

// ---- union-find (ECL-CC): parent[x] <= x always, the root of a tree is its smallest pixel ------------------------
__device__ __forceinline__ uint32_t uf_find(uint32_t* parent, uint32_t x) {
  uint32_t cur = __ldcg(&parent[x]);
  if (cur != x) {                    // path halving; every store writes an ancestor, so lost updates are harmless
    uint32_t prev = x, next;
    while (cur > (next = __ldcg(&parent[cur]))) { parent[prev] = next; prev = cur; cur = next; }
  }
  return cur;
}

__device__ __forceinline__ void uf_unite(uint32_t* parent, uint32_t a, uint32_t b) {
  a = uf_find(parent, a); b = uf_find(parent, b);
  while (a != b) {
    if (a > b) { const uint32_t t = a; a = b; b = t; }
    const uint32_t old = atomicCAS(&parent[b], b, a);   // hooks b only while it is still a root
    if (old == b) break;
    b = old;
  }
}

// owner's range, and the per-call state of every pixel
__global__ void __launch_bounds__(256)
dc_image_kernel(const char* __restrict__ pts, int64_t stride, const FilterParams f, int P,
                const uint32_t* __restrict__ owner, float* __restrict__ image, uint32_t* __restrict__ parent,
                uint32_t* __restrict__ claim, int32_t* __restrict__ level) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  const uint32_t o = owner[p];
  float r = 0.f;
  if (o != kNone) {                  // :103-105, :129-130
    const float* q = reinterpret_cast<const float*>(pts + (int64_t)o * stride);
    const float x = q[0] + f.offset_x, y = q[1] + f.offset_y, z = q[2] + f.offset_z;
    r = sqrtf(x * x + y * y + z * z);
  }
  image[p] = r;
  parent[p] = (uint32_t)p;
  claim[p] = kNone;
  level[p] = -1;
}

__global__ void __launch_bounds__(256)
dc_edge_kernel(int V, int H, const DepthConsts c, const float* __restrict__ image, uint8_t* __restrict__ mask) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= V * H) return;
  const float a = image[p];
  uint32_t m = 0;
  if (depth_occupied(a)) {
    const int row = p / H, col = p - row * H;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const int q = depth_neighbor(row, col, k, V, H);
      if (q < 0) continue;
      const float b = image[q];
      if (depth_occupied(b) && depth_edge(a, b, k < 4 ? c.sin_h : c.sin_v, k < 4 ? c.cos_h : c.cos_v)) m |= 1u << k;
    }
  }
  mask[p] = (uint8_t)m;
}

__global__ void __launch_bounds__(256)
dc_union_kernel(int V, int H, const uint8_t* __restrict__ mask, uint32_t* __restrict__ parent) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= V * H) return;
  const uint32_t m = mask[p];
  if (!(m & 0x15u)) return;
  const int row = p / H, col = p - row * H;
  for (int k = 0; k < 6; k += 2)     // the forward steps (0,1) (0,2) (1,0); the mask is symmetric
    if (m >> k & 1u) uf_unite(parent, (uint32_t)p, (uint32_t)depth_neighbor(row, col, k, V, H));
}

__device__ __forceinline__ bool is_root(const float* image, const uint32_t* parent, int p) {
  return depth_occupied(image[p]) && parent[p] == (uint32_t)p;
}

__global__ void __launch_bounds__(kCompactThreads)
dc_root_count_kernel(int P, const float* __restrict__ image, const uint32_t* __restrict__ parent,
                     uint32_t* __restrict__ block_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems && base + r < P; ++r) c += is_root(image, parent, base + r) ? 1u : 0u;
  tile_count_store(c, block_cnt);
}

// label[root] = 1 + the root's rank, roots[rank] = the root; *n_roots = the number of components
__global__ void __launch_bounds__(kCompactThreads)
dc_root_scatter_kernel(int P, const float* __restrict__ image, const uint32_t* __restrict__ parent,
                       const uint32_t* __restrict__ tile_off, uint32_t* __restrict__ label, uint32_t* __restrict__ roots,
                       uint32_t* __restrict__ n_roots) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f = 0, c = 0;
  for (int r = 0; r < kCompactItems; ++r)
    if (base + r < P && is_root(image, parent, base + r)) { f |= 1u << r; ++c; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    if (!(f >> r & 1u)) continue;
    label[base + r] = pos + 1;
    roots[pos] = (uint32_t)(base + r);
    ++pos;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_roots = tile_off[gridDim.x];
}

// every pixel's label (0 = empty) and the pixel count per label, one atomic per label and warp
__global__ void __launch_bounds__(256)
dc_label_kernel(int P, const float* __restrict__ image, uint32_t* __restrict__ parent, uint32_t* __restrict__ label,
                uint32_t* __restrict__ size) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  uint32_t l = 0;
  if (p < P && depth_occupied(image[p])) {
    const uint32_t root = uf_find(parent, (uint32_t)p);
    l = root == (uint32_t)p ? label[p] : __ldcg(&label[root]);
    if (root != (uint32_t)p) label[p] = l;
  } else if (p < P) {
    label[p] = 0;
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, l);
  if (l && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&size[l - 1], (uint32_t)__popc(peers));
}

// per tile of components: the kept ones (>= kMinCluster pixels, :306-308) and their pixels, row 0 and row 1 of
// cnt ([2][stride]); the slot behind the last tile is cleared for the scan's totals
__global__ void __launch_bounds__(kCompactThreads)
dc_keep_count_kernel(int n, const uint32_t* __restrict__ size, uint32_t* __restrict__ cnt, int stride) {
  __shared__ uint32_t red[kCompactThreads / 32][2];
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t acc[2] = {0, 0};
  for (int r = 0; r < kCompactItems && base + r < n; ++r) {
    const uint32_t sz = size[base + r];
    if (sz >= kMinCluster) { acc[0] += 1; acc[1] += sz; }
  }
  const uint32_t t = block_sum<2, kCompactThreads>(acc, red);
  if (threadIdx.x < 2) {
    cnt[threadIdx.x * stride + blockIdx.x] = t;
    if (blockIdx.x == 0) cnt[threadIdx.x * stride + gridDim.x] = 0;
  }
}

// kept[j] = the j-th kept component in label order, kept_off[j] = where its queue starts in the output;
// totals = {kept components, clustered pixels}
__global__ void __launch_bounds__(kCompactThreads)
dc_keep_scatter_kernel(int n, const uint32_t* __restrict__ size, const uint32_t* __restrict__ cnt, int stride,
                       uint32_t* __restrict__ kept, uint32_t* __restrict__ kept_off, uint32_t* __restrict__ totals) {
  __shared__ uint32_t ws[2][kCompactThreads / 32];
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f = 0, c = 0, px = 0;
  for (int r = 0; r < kCompactItems && base + r < n; ++r) {
    const uint32_t sz = size[base + r];
    if (sz >= kMinCluster) { f |= 1u << r; ++c; px += sz; }
  }
  uint32_t pos = cnt[blockIdx.x] + block_scan_excl<kCompactThreads / 32>(c, ws[0]);
  uint32_t at = cnt[stride + blockIdx.x] + block_scan_excl<kCompactThreads / 32>(px, ws[1]);
  for (int r = 0; r < kCompactItems; ++r) {
    if (!(f >> r & 1u)) continue;
    kept[pos] = (uint32_t)(base + r); kept_off[pos] = at;
    ++pos; at += size[base + r];
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) { totals[0] = cnt[gridDim.x]; totals[1] = cnt[stride + gridDim.x]; }
}

// LabelOneComponent's FIFO (:245-305) for the kept components blockIdx.x, blockIdx.x + gridDim.x, ...;
// order[kept_off[j] ..] is the queue of first pops of kept component j
__global__ void __launch_bounds__(kBfsThreads)
dc_bfs_kernel(int V, int H, const uint8_t* __restrict__ mask, const uint32_t* __restrict__ roots,
              const uint32_t* __restrict__ kept, const uint32_t* __restrict__ kept_off,
              const uint32_t* __restrict__ totals, uint32_t* __restrict__ claim, int32_t* __restrict__ level,
              uint32_t* __restrict__ seq, uint32_t* __restrict__ order) {
  __shared__ uint32_t warp_tot[kBfsThreads / 32];
  for (uint32_t j = blockIdx.x; j < totals[0]; j += gridDim.x) {
    uint32_t* q = order + kept_off[j];
    if (threadIdx.x == 0) {
      const uint32_t root = roots[kept[j]];
      q[0] = root; level[root] = 0; seq[root] = 0;
    }
    __syncthreads();
    uint32_t head = 0, tail = 1;
    for (int lvl = 1; head < tail; ++lvl) {
      for (uint32_t r = head + threadIdx.x; r < tail; r += kBfsThreads) {
        const uint32_t p = q[r], m = mask[p];
        const int row = (int)(p / (uint32_t)H), col = (int)(p - (uint32_t)row * (uint32_t)H);
        for (int k = 0; k < 6; ++k) {
          if (!(m >> k & 1u)) continue;
          const int nb = depth_neighbor(row, col, k, V, H);
          if (__ldcg(&level[nb]) < 0) atomicMin(&claim[nb], r * 6u + (uint32_t)k);
        }
      }
      __syncthreads();
      uint32_t next = tail;
      for (uint32_t r0 = head; r0 < tail; r0 += kBfsThreads) {
        const uint32_t r = r0 + threadIdx.x;
        uint32_t won = 0, p = 0;
        if (r < tail) {
          p = q[r];
          const uint32_t m = mask[p];
          const int row = (int)(p / (uint32_t)H), col = (int)(p - (uint32_t)row * (uint32_t)H);
          for (int k = 0; k < 6; ++k)
            if ((m >> k & 1u) && __ldcg(&claim[depth_neighbor(row, col, k, V, H)]) == r * 6u + (uint32_t)k)
              won |= 1u << k;
        }
        uint32_t total;
        uint32_t pos = next + block_scan_excl<kBfsThreads / 32>((uint32_t)__popc(won), warp_tot, &total);
        if (won) {
          const int row = (int)(p / (uint32_t)H), col = (int)(p - (uint32_t)row * (uint32_t)H);
          for (int k = 0; k < 6; ++k) {
            if (!(won >> k & 1u)) continue;
            const int nb = depth_neighbor(row, col, k, V, H);
            q[pos] = (uint32_t)nb; level[nb] = lvl; seq[nb] = pos;
            ++pos;
          }
        }
        next += total;
        __syncthreads();               // warp_tot is read again by the next chunk's scan; q by the next level
      }
      head = tail; tail = next;
    }
  }
}

// output j: the pixel order[j] (clusters in ascending label, each in queue order) as its owner's record
__global__ void __launch_bounds__(256)
dc_emit_kernel(const char* __restrict__ pts, int64_t stride, int bound, const uint32_t* __restrict__ m,
               const uint32_t* __restrict__ order, const uint32_t* __restrict__ owner, const uint32_t* __restrict__ label,
               float* __restrict__ out_xyz, uint32_t* __restrict__ out_label, int32_t* __restrict__ out_index) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= bound || (uint32_t)j >= *m) return;
  const uint32_t px = order[j], i = owner[px];
  const float* p = reinterpret_cast<const float*>(pts + (int64_t)i * stride);
  out_xyz[3 * (int64_t)j] = p[0]; out_xyz[3 * (int64_t)j + 1] = p[1]; out_xyz[3 * (int64_t)j + 2] = p[2];
  out_label[j] = label[px];
  out_index[j] = (int32_t)i;
}

__global__ void __launch_bounds__(256)
dc_point_label_kernel(int n, const uint32_t* __restrict__ pixel, const uint32_t* __restrict__ owner,
                      const uint32_t* __restrict__ label, uint32_t* __restrict__ point_label) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t px = pixel[i];
  point_label[i] = (px != kNone && owner[px] == (uint32_t)i) ? label[px] : 0u;
}

}  // namespace

DepthConsts depth_consts(const FilterParams& f) {
  // :255-259: the vertical resolution divides by the double 180. where Filter divides by 180.f
  const float hres = (float)(M_PI * 2 / (double)(float)f.horizontal_line_num);
  const float vres = (float)((double)((f.top_angle - f.btm_angle) / (float)f.vertical_line_num) / 180. * M_PI);
  DepthConsts c;
  c.sin_h = sinf(hres); c.cos_h = cosf(hres);
  c.sin_v = sinf(vres); c.cos_v = cosf(vres);
  return c;
}

bool depth_debug_edge_host(const DepthConsts& c, float a, float b, int k, float* beta) {
  return depth_edge(a, b, k < 4 ? c.sin_h : c.sin_v, k < 4 ? c.cos_h : c.cos_v, beta);
}

int DepthCluster::reserve(int64_t n, int64_t P) {
  SMB_RC(pixel.reserve((size_t)n * sizeof(uint32_t)));
  for (DevBuf* b : {&owner, &image, &parent, &label, &claim, &level, &seq, &order, &roots})
    SMB_RC(b->reserve((size_t)P * 4));
  SMB_RC(mask.reserve((size_t)P));
  SMB_RC(size.reserve(((size_t)P + 1) * 4));
  SMB_RC(kept.reserve((size_t)P / kMinCluster * 4 + 4));
  SMB_RC(kept_off.reserve((size_t)P / kMinCluster * 4 + 4));
  SMB_RC(block_cnt.reserve(2 * compact_count_bytes(P)));   // the root compaction's tile counts, then [2] per component tile
  SMB_RC(count.reserve(4 * sizeof(uint32_t)));
  return 0;
}

int DepthCluster::run(const FilterParams& f, const char* pts, int n, int64_t stride, float* out_xyz,
                      uint32_t* out_label, int32_t* out_index, uint32_t* point_label, int64_t* m, cudaStream_t s) {
  *m = 0;
  const int V = f.vertical_line_num, H = f.horizontal_line_num, P = V * H;
  SMB_RC(reserve(n, P));
  uint32_t* d_owner = (uint32_t*)owner.p; uint32_t* d_parent = (uint32_t*)parent.p;
  uint32_t* d_label = (uint32_t*)label.p; uint32_t* d_count = (uint32_t*)count.p;
  float* d_image = (float*)image.p;
  SMB_RC(range_image_owner(f, pts, n, stride, (uint32_t*)pixel.p, d_owner, s));
  dc_image_kernel<<<ceil_div(P, 256), 256, 0, s>>>(pts, stride, f, P, d_owner, d_image, d_parent, (uint32_t*)claim.p,
                                                   (int32_t*)level.p);
  dc_edge_kernel<<<ceil_div(P, 256), 256, 0, s>>>(V, H, depth_consts(f), d_image, (uint8_t*)mask.p);
  dc_union_kernel<<<ceil_div(P, 256), 256, 0, s>>>(V, H, (const uint8_t*)mask.p, d_parent);
  const int tiles = compact_tiles(P);
  dc_root_count_kernel<<<tiles, kCompactThreads, 0, s>>>(P, d_image, d_parent, (uint32_t*)block_cnt.p);
  compact_scan((uint32_t*)block_cnt.p, tiles, s);
  dc_root_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(P, d_image, d_parent, (const uint32_t*)block_cnt.p, d_label,
                                                           (uint32_t*)roots.p, d_count);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t n_comp = 0;                 // sizes the label pass and the BFS grid
  SMB_CUDA_OK(cudaMemcpyAsync(&n_comp, d_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  components = (int)n_comp;
  uint32_t* d_totals = d_count + 2;   // kept components, clustered pixels
  SMB_CUDA_OK(cudaMemsetAsync(d_totals, 0, 2 * sizeof(uint32_t), s));
  SMB_CUDA_OK(cudaMemsetAsync(size.p, 0, ((size_t)n_comp + 1) * sizeof(uint32_t), s));
  dc_label_kernel<<<ceil_div(P, 256), 256, 0, s>>>(P, d_image, d_parent, d_label, (uint32_t*)size.p);
  if (n_comp > 0) {
    const int ktiles = compact_tiles(n_comp);
    uint32_t* d_cnt = (uint32_t*)block_cnt.p;
    dc_keep_count_kernel<<<ktiles, kCompactThreads, 0, s>>>((int)n_comp, (const uint32_t*)size.p, d_cnt, ktiles + 1);
    radix_scan_kernel_launch(d_cnt, ktiles + 1, 2, s);
    dc_keep_scatter_kernel<<<ktiles, kCompactThreads, 0, s>>>((int)n_comp, (const uint32_t*)size.p, d_cnt, ktiles + 1,
                                                              (uint32_t*)kept.p, (uint32_t*)kept_off.p, d_totals);
    dc_bfs_kernel<<<n_comp < (uint32_t)kBfsCtas ? n_comp : kBfsCtas, kBfsThreads, 0, s>>>(
        V, H, (const uint8_t*)mask.p, (const uint32_t*)roots.p, (const uint32_t*)kept.p, (const uint32_t*)kept_off.p,
        d_totals, (uint32_t*)claim.p, (int32_t*)level.p, (uint32_t*)seq.p, (uint32_t*)order.p);
  }
  const int bound = n < P ? n : P;     // at most one output per occupied pixel
  if (out_xyz)
    dc_emit_kernel<<<ceil_div(bound, 256), 256, 0, s>>>(pts, stride, bound, d_totals + 1, (const uint32_t*)order.p,
                                                        d_owner, d_label, out_xyz, out_label, out_index);
  if (point_label)
    dc_point_label_kernel<<<ceil_div(n, 256), 256, 0, s>>>(n, (const uint32_t*)pixel.p, d_owner, d_label, point_label);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t total = 0;
  SMB_CUDA_OK(cudaMemcpyAsync(&total, d_totals + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  *m = total;
  return 0;
}

}  // namespace smb
