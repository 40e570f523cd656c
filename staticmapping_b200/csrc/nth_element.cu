// CalculateNormals' median split in the order libstdc++'s std::nth_element leaves (SM_NORMALS_ORDER_NTH_ELEMENT).
// The reference (builder/data/cloud_types.cc:105-144) calls nth_element(first, first + leftCount, last) with a plain
// '<' on the cut-axis coordinate, on ONE index array that the whole recursion permutes in place; each leaf is then
// summed in the member order left behind and represented by its first member.  This file reproduces that array.
//
// std::nth_element is introselect, restated here from the algorithm:
//   while last - first > 3:
//     after 2 * floor(log2 n) rounds: heap select of [first, nth + 1) over [first, last), swap first and nth, stop;
//     move the median of (first + 1, mid, last - 1) to first, in the library's comparison order;
//     Hoare's unguarded partition of [first + 1, last) around the key at first -> cut; keep the side holding nth;
//   insertion sort of the <= 3 elements left.
// A round's partition runs in parallel from counts.  Let a left stopper be an x with !(x < p), met scanning up, and
// a right stopper an x with !(p < x), met scanning down.  The a-th left stopper L_a swaps with the a-th right stopper
// R_a exactly while L_a < R_a, i.e. iff at least a right stoppers lie above L_a (a swap only ever places a stopper in
// the other scan's path, where that scan had to stop anyway).  With K such pairs the scan stops at
// min(L_{K+1}, R_K), R_0 = last.  tests/nth_element_model.py checks this rule round for round against the sequential
// restatement, and that against std::nth_element itself.
//
// Launch structure (NormalsPipeline::run_nth_element): level by level, one CTA per node takes the widest axis of the
// node's implicit bounds, gathers the node's keys on it and runs the rounds, with one thread finishing once the live
// range is small, then writes its children's bounds around the key left at nth; from the level whose nodes hold
// <= kThreadMax points, one thread finishes each whole subtree.  Keys and indices stay in global memory (a 500k-point
// cloud's 6 MB of them stay in L2).  The bounds are carried here, not taken from the k-d build: with tied
// coordinates the two orders send different tied points left, so below such a split the cuts can differ.
#include "common.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace smb {
namespace {

constexpr int kThreads = 512;
constexpr int kItems = 4;
constexpr int kTile = kThreads * kItems;
constexpr int kSerialMax = 256;      // a CTA's live range at or below this finishes on one thread
constexpr int kThreadMax = 64;       // nodes at or below this size run their whole subtree on one thread

__device__ __forceinline__ int floor_log2(int n) { return 31 - __clz(n); }

__device__ __forceinline__ void swap_at(double* k, uint32_t* p, int a, int b) {
  const double tk = k[a]; k[a] = k[b]; k[b] = tk;
  const uint32_t tp = p[a]; p[a] = p[b]; p[b] = tp;
}

// the median of (a, b, c) moves to `first`, with the comparisons of libstdc++'s __move_median_to_first
__device__ void median_to_first(double* k, uint32_t* p, int first, int a, int b, int c) {
  int m;
  if (k[a] < k[b]) m = (k[b] < k[c]) ? b : ((k[a] < k[c]) ? c : a);
  else if (k[a] < k[c]) m = a;
  else if (k[b] < k[c]) m = c;
  else m = b;
  swap_at(k, p, first, m);
}

// sift the hole at `hole` of the heap [base, base + len) down to a leaf, then the value back up (__adjust_heap)
__device__ void adjust_heap(double* k, uint32_t* p, int base, int hole, int len, double vk, uint32_t vp) {
  const int top = hole;
  int child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (k[base + child] < k[base + child - 1]) --child;
    k[base + hole] = k[base + child]; p[base + hole] = p[base + child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    k[base + hole] = k[base + child - 1]; p[base + hole] = p[base + child - 1];
    hole = child - 1;
  }
  int parent = (hole - 1) / 2;
  while (hole > top && k[base + parent] < vk) {
    k[base + hole] = k[base + parent]; p[base + hole] = p[base + parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  k[base + hole] = vk; p[base + hole] = vp;
}

// the depth-limit fallback: a max-heap of [first, middle), every later element below its top replaces the top
// (__heap_select).  Serial, for correctness: adversarial inputs only.
__device__ void heap_select(double* k, uint32_t* p, int first, int middle, int last) {
  const int len = middle - first;
  if (len >= 2)
    for (int parent = (len - 2) / 2;; --parent) {
      adjust_heap(k, p, first, parent, len, k[first + parent], p[first + parent]);
      if (parent == 0) break;
    }
  for (int i = middle; i < last; ++i)
    if (k[i] < k[first]) {
      const double vk = k[i]; const uint32_t vp = p[i];
      k[i] = k[first]; p[i] = p[first];
      adjust_heap(k, p, first, 0, len, vk, vp);
    }
}

__device__ void insertion_sort(double* k, uint32_t* p, int first, int last) {
  for (int i = first + 1; i < last; ++i) {
    const double vk = k[i]; const uint32_t vp = p[i];
    int j = i;
    if (vk < k[first]) {
      for (; j > first; --j) { k[j] = k[j - 1]; p[j] = p[j - 1]; }
    } else {
      for (; vk < k[j - 1]; --j) { k[j] = k[j - 1]; p[j] = p[j - 1]; }
    }
    k[j] = vk; p[j] = vp;
  }
}

// introselect on one thread from a given state (first, last, rounds left)
__device__ void introselect_serial(double* k, uint32_t* p, int first, int nth, int last, int depth) {
  while (last - first > 3) {
    if (depth == 0) {
      heap_select(k, p, first, nth + 1, last);
      swap_at(k, p, first, nth);
      return;
    }
    --depth;
    median_to_first(k, p, first, first + 1, first + (last - first) / 2, last - 1);
    const double pk = k[first];
    int lo = first + 1, hi = last;
    for (;;) {
      while (k[lo] < pk) ++lo;
      --hi;
      while (pk < k[hi]) --hi;
      if (!(lo < hi)) break;
      swap_at(k, p, lo, hi);
      ++lo;
    }
    if (lo <= nth) first = lo; else last = lo;
  }
  insertion_sort(k, p, first, last);
}

// One partition round of [first + 1, last) around k[first] by the whole CTA, from stopper counts.  lpos / rpos:
// scratch with room for last - first entries from `first`.  Returns the cut.  Every thread must call it.
__device__ int block_partition(double* k, uint32_t* p, uint32_t* lpos, uint32_t* rpos, int first, int last) {
  __shared__ uint32_t s_wl[kThreads / 32], s_wr[kThreads / 32], s_red[kThreads / 32][1];
  __shared__ uint32_t s_nr, s_k;
  __shared__ int s_min_l;
  const double pk = k[first];
  // right stoppers in all
  uint32_t nr = 0;
  for (int i = first + 1 + threadIdx.x; i < last; i += kThreads) nr += !(pk < k[i]);
  const uint32_t acc[1] = {nr};
  const uint32_t tot = block_sum<1, kThreads>(acc, s_red);
  if (threadIdx.x == 0) { s_nr = tot; s_k = 0; s_min_l = last; }
  __syncthreads();
  const uint32_t n_r = s_nr;
  uint32_t below_l = 0, below_r = 0;          // stoppers below the current tile
  for (int t0 = first + 1; t0 < last; t0 += kTile) {
    const int base = t0 + threadIdx.x * kItems;
    uint32_t fl = 0, fr = 0;                  // bit r: item r is a left / right stopper
#pragma unroll
    for (int r = 0; r < kItems; ++r) {
      if (base + r < last) {
        const double x = k[base + r];
        fl |= (uint32_t)!(x < pk) << r;
        fr |= (uint32_t)!(pk < x) << r;
      }
    }
    uint32_t tl, tr;
    uint32_t cl = below_l + block_scan_excl<kThreads / 32>(__popc(fl), s_wl, &tl);
    uint32_t cr = below_r + block_scan_excl<kThreads / 32>(__popc(fr), s_wr, &tr);
    uint32_t swaps = 0;
    int min_l = last;
#pragma unroll
    for (int r = 0; r < kItems; ++r) {
      const int i = base + r;
      const bool il = (fl >> r) & 1u, ir = (fr >> r) & 1u;
      if (il) {
        const uint32_t a = cl + 1;                     // rank from the bottom, from 1
        const uint32_t above_r = n_r - cr - (ir ? 1u : 0u);
        if (above_r >= a) { lpos[first + a - 1] = (uint32_t)i; ++swaps; }
        else min_l = min(min_l, i);
      }
      if (ir) {
        const uint32_t b = n_r - cr;                   // rank from the top, from 1
        if (cl >= b) rpos[first + b - 1] = (uint32_t)i;
      }
      cl += il; cr += ir;
    }
    if (swaps) atomicAdd(&s_k, swaps);
    if (min_l < last) atomicMin(&s_min_l, min_l);
    below_l += tl; below_r += tr;
    __syncthreads();                                   // the warp totals are read again by the next tile's scans
  }
  const int K = (int)s_k;
  for (int a = threadIdx.x; a < K; a += kThreads) swap_at(k, p, (int)lpos[first + a], (int)rpos[first + a]);
  const int cut = min(s_min_l, K ? (int)rpos[first + K - 1] : last);
  __syncthreads();
  return cut;
}

// std::nth_element(first, nth, last) by one CTA on the keys k and indices p.  Every thread must call it.
__device__ void block_introselect(double* k, uint32_t* p, uint32_t* lpos, uint32_t* rpos, int first, int nth,
                                  int last) {
  if (first == last || nth == last) return;
  int depth = 2 * floor_log2(last - first);
  while (last - first > kSerialMax && depth > 0) {
    if (threadIdx.x == 0) median_to_first(k, p, first, first + 1, first + (last - first) / 2, last - 1);
    __syncthreads();
    const int cut = block_partition(k, p, lpos, rpos, first, last);
    --depth;
    if (cut <= nth) first = cut; else last = cut;
  }
  if (threadIdx.x == 0) introselect_serial(k, p, first, nth, last, depth);
  __syncthreads();
}

// node j of level L of the split over n points -> its span; false if an ancestor was already a leaf
__device__ __forceinline__ bool node_span(int j, int L, int n, int* first_out, int* count_out) {
  int first = 0, count = n;
  for (int l = L - 1; l >= 0; --l) {
    if (count <= 7) return false;
    const int right = count >> 1, left = count - right;
    if ((j >> l) & 1) { first += left; count = right; } else { count = left; }
  }
  *first_out = first;
  *count_out = count;
  return true;
}

// cloud_types.cc:41-56: the first strictly greater extent wins, from 0
__device__ __forceinline__ int widest_axis(const double* b) {
  double mv = 0.0;
  int mi = 0;
  for (int d = 0; d < 3; ++d) {
    const double e = b[3 + d] - b[d];
    if (e > mv) { mv = e; mi = d; }
  }
  return mi;
}

// one CTA per node of level L: the cut axis from the node's implicit bounds (bounds_in[j]: min[3], max[3]), the keys
// on it gathered, nth_element(first + leftCount), then the children's bounds around the key that lands at nth.  The
// bounds are this order's own: with tied coordinates the children's point sets, and so their cuts, depend on which
// tied points nth_element sends left.
__global__ void __launch_bounds__(kThreads)
nth_level_kernel(const double* __restrict__ coord, int64_t cstride, int n, int L, const double* __restrict__ bounds_in,
                 double* __restrict__ bounds_out, uint32_t* __restrict__ perm, double* __restrict__ key,
                 uint32_t* __restrict__ lpos, uint32_t* __restrict__ rpos) {
  const int j = blockIdx.x;
  int first, count;
  if (!node_span(j, L, n, &first, &count) || count <= 7) return;
  double b[6];
  for (int d = 0; d < 6; ++d) b[d] = bounds_in[(int64_t)j * 6 + d];
  const int dim = widest_axis(b);
  for (int i = first + threadIdx.x; i < first + count; i += kThreads) key[i] = coord[dim * cstride + perm[i]];
  __syncthreads();
  const int nth = first + count - (count >> 1);
  block_introselect(key, perm, lpos, rpos, first, nth, first + count);
  if (threadIdx.x < 6) {
    const int d = threadIdx.x;
    const double cut = key[nth];
    bounds_out[(int64_t)(2 * j) * 6 + d] = (d == 3 + dim) ? cut : b[d];
    bounds_out[(int64_t)(2 * j + 1) * 6 + d] = (d == dim) ? cut : b[d];
  }
}

// one thread per node of level L finishes its whole subtree (nodes of <= kThreadMax points, so at most 4 levels)
__global__ void nth_subtree_kernel(const double* __restrict__ coord, int64_t cstride, int n, int L,
                                   const double* __restrict__ bounds_in, uint32_t* __restrict__ perm,
                                   double* __restrict__ key) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (1 << L)) return;
  int first0, count0;
  if (!node_span(j, L, n, &first0, &count0) || count0 <= 7) return;
  struct Node { int first, count; double b[6]; };
  Node stack[8];
  int top = 0;
  stack[0].first = first0; stack[0].count = count0;
  for (int d = 0; d < 6; ++d) stack[0].b[d] = bounds_in[(int64_t)j * 6 + d];
  ++top;
  while (top > 0) {
    const Node nd = stack[--top];
    if (nd.count <= 7) continue;
    const int dim = widest_axis(nd.b);
    for (int i = nd.first; i < nd.first + nd.count; ++i) key[i] = coord[dim * cstride + perm[i]];
    const int left = nd.count - (nd.count >> 1);
    introselect_serial(key, perm, nd.first, nd.first + left, nd.first + nd.count, 2 * floor_log2(nd.count));
    const double cut = key[nd.first + left];
    Node& l = stack[top++];
    l.first = nd.first; l.count = left;
    for (int d = 0; d < 6; ++d) l.b[d] = nd.b[d];
    l.b[3 + dim] = cut;
    Node& r = stack[top++];
    r.first = nd.first + left; r.count = nd.count - left;
    for (int d = 0; d < 6; ++d) r.b[d] = nd.b[d];
    r.b[dim] = cut;
  }
}

// per-axis min and max of the first n points -> bounds[0..6) (min[3], max[3]), one CTA
__global__ void __launch_bounds__(kThreads)
nth_root_bounds_kernel(const double* __restrict__ coord, int64_t cstride, int n, double* __restrict__ bounds) {
  __shared__ double s[6][kThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int d = 0; d < 3; ++d) {
    double mn = coord[d * cstride], mx = mn;
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const double v = coord[d * cstride + i];
      mn = fmin(mn, v); mx = fmax(mx, v);
    }
    mn = warp_min(mn); mx = warp_max(mx);
    if (lane == 0) { s[d][w] = mn; s[3 + d][w] = mx; }
  }
  __syncthreads();
  if (threadIdx.x < 6) {
    double v = s[threadIdx.x][0];
    for (int ww = 1; ww < kThreads / 32; ++ww) v = threadIdx.x < 3 ? fmin(v, s[threadIdx.x][ww]) : fmax(v, s[threadIdx.x][ww]);
    bounds[threadIdx.x] = v;
  }
}

__global__ void iota_kernel(uint32_t* __restrict__ perm, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) perm[i] = (uint32_t)i;
}

__global__ void nonfinite_kernel(const double* __restrict__ coord, int64_t cstride, int n, uint32_t* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!isfinite(coord[i]) || !isfinite(coord[cstride + i]) || !isfinite(coord[2 * cstride + i])) *bad = 1u;
}

// the single-array test hook: keys[i] at perm[i] = i, then one CTA's nth_element
__global__ void __launch_bounds__(kThreads)
nth_single_kernel(const double* __restrict__ keys_in, int n, int nth, uint32_t* __restrict__ perm,
                  double* __restrict__ key, uint32_t* __restrict__ lpos, uint32_t* __restrict__ rpos) {
  for (int i = threadIdx.x; i < n; i += kThreads) { key[i] = keys_in[i]; perm[i] = (uint32_t)i; }
  __syncthreads();
  block_introselect(key, perm, lpos, rpos, 0, nth, n);
}

}  // namespace

// BuildNormals' index array over the first n points of coord (SoA [3][cstride]) in std::nth_element's order.
// perm, key, lpos, rpos: n entries each; bounds: 2 * 6 * 2^kd_num_levels(n, 7) doubles.
int nth_element_recursion(const double* coord, int64_t cstride, int n, uint32_t* perm, double* key, uint32_t* lpos,
                          uint32_t* rpos, double* bounds, cudaStream_t stream) {
  const int levels = kd_num_levels(n, 7);
  double* bnd[2] = {bounds, bounds + ((size_t)6 << levels)};
  iota_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(perm, n);
  nth_root_bounds_kernel<<<1, kThreads, 0, stream>>>(coord, cstride, n, bnd[0]);
  int L = 0;
  for (int64_t c = n; L < levels && c > kThreadMax; c = (c + 1) / 2, ++L)
    nth_level_kernel<<<1 << L, kThreads, 0, stream>>>(coord, cstride, n, L, bnd[L & 1], bnd[(L + 1) & 1], perm, key,
                                                      lpos, rpos);
  if (L < levels)
    nth_subtree_kernel<<<ceil_div(1 << L, 128), 128, 0, stream>>>(coord, cstride, n, L, bnd[L & 1], perm, key);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

size_t nth_element_bounds_bytes(int n) { return ((size_t)12 << kd_num_levels(n, 7)) * sizeof(double); }

// 1 if any of the first n points of coord has a non-finite coordinate (waits for the answer)
int any_nonfinite(const double* coord, int64_t cstride, int n, uint32_t* flag_dev, cudaStream_t stream, bool* bad) {
  uint32_t h = 0;
  SMB_CUDA_OK(cudaMemsetAsync(flag_dev, 0, sizeof(uint32_t), stream));
  nonfinite_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(coord, cstride, n, flag_dev);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(&h, flag_dev, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  *bad = h != 0;
  return 0;
}

// test hook sm_debug_nth_element: one CTA's std::nth_element(nth) over n device keys -> perm (device, n entries)
int nth_element_single(const double* keys, int n, int nth, uint32_t* perm, double* key, uint32_t* lpos,
                       uint32_t* rpos, cudaStream_t stream) {
  nth_single_kernel<<<1, kThreads, 0, stream>>>(keys, n, nth, perm, key, lpos, rpos);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace smb
