// GPU builder for the libnabo-compatible k-d tree (KDTREE_LINEAR_HEAP semantics:
// implicit-bounds widest-axis median split, leftCount = n - n/2, bucket size 8;
// call site registrators/icp_fast.cc:466-467) and, with bucket 7, for the leaf
// partition of EigenPointCloud::CalculateNormals (builder/data/cloud_types.cc:105-144).
//
// GPU formulation instead of the reference's recursive std::nth_element:
//   * the tree SHAPE depends only on (N, bucket): every node's [first, first+count) is
//     pure integer arithmetic, so nodes live in an implicit heap layout (children of h
//     are 2h+1 / 2h+2) and nothing about the shape is stored or communicated;
//   * the three per-axis orderings are radix-sorted once; each level then needs only the
//     median (an array lookup) and a stable partition of the three lists, done for ALL
//     nodes of the level at once with a flag + prefix-scan + scatter;
//   * ties are broken by the total order (coordinate, original index).
#include "common.cuh"
#include "kernels.h"
#include "reduce.cuh"

namespace smb {
namespace {

struct Seg {
  int first, count;
  bool exists;
};

// node j of level L -> its segment; exists == false when an ancestor was already a leaf.
__device__ __forceinline__ Seg locate_node(int j, int L, int n, int bucket) {
  int first = 0, count = n;
  for (int l = L - 1; l >= 0; --l) {
    if (count <= bucket) return Seg{first, count, false};
    const int right = count >> 1, left = count - right;
    if ((j >> l) & 1) { first += left; count = right; } else { count = left; }
  }
  return Seg{first, count, true};
}

// position i -> the level-L node containing it (or the shallower leaf that does).
// Returns true when the node is an INNER node of level L (i.e. it will be split now).
__device__ __forceinline__ bool locate_pos(int i, int L, int n, int bucket, int* j_out,
                                           int* first_out, int* count_out) {
  int first = 0, count = n, j = 0;
  for (int l = 0; l < L; ++l) {
    if (count <= bucket) { *j_out = j; *first_out = first; *count_out = count; return false; }
    const int right = count >> 1, left = count - right;
    if (i < first + left) { j = 2 * j; count = left; }
    else { j = 2 * j + 1; first += left; count = right; }
  }
  *j_out = j; *first_out = first; *count_out = count;
  return count > bucket;
}

__device__ __forceinline__ int argmax3(double ex, double ey, double ez) {
  // cloud_types.cc:41-56 / libnabo argMax: first strictly-greater-than wins, from 0.
  double mv = 0.0; int mi = 0;
  if (ex > mv) { mv = ex; mi = 0; }
  if (ey > mv) { mv = ey; mi = 1; }
  if (ez > mv) { mv = ez; mi = 2; }
  return mi;
}

// {cut, dim} of one node as the search kernel loads it (KdCompact::node)
__device__ __forceinline__ double2 packed_node(double cut, int dim) {
  return make_double2(cut, __longlong_as_double((long long)dim));
}

// ---- per level: node kernel -----------------------------------------------------------
__global__ void kd_node_kernel(const double* __restrict__ coord, int64_t cstride,
                               const uint32_t* __restrict__ lists, int64_t lstride, int n,
                               int bucket, int L, const double* __restrict__ bounds_in,
                               double* __restrict__ bounds_out, int* __restrict__ level_dim,
                               KdNode* __restrict__ nodes, double* __restrict__ ccut,
                               uint8_t* __restrict__ cdim, double2* __restrict__ cnode) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= (1 << L)) return;
  const Seg s = locate_node(j, L, n, bucket);
  if (!s.exists) return;
  const int h = (1 << L) - 1 + j;
  if (s.count <= bucket) {
    KdNode leaf;
    leaf.cut = __longlong_as_double(((long long)s.count << 32) | (long long)(unsigned)s.first);
    leaf.dim = 3; leaf.pad = 0;
    nodes[blocked_index(h)] = leaf;
    level_dim[j] = 3;
    if (cdim) cdim[h] = 3;
    if (cnode) cnode[h + 1] = packed_node(0.0, 3);
    return;
  }
  double mn[3], mx[3];
  if (L == 0) {
    for (int d = 0; d < 3; ++d) {
      mn[d] = coord[d * cstride + lists[d * lstride + 0]];
      mx[d] = coord[d * cstride + lists[d * lstride + (n - 1)]];
    }
  } else {
    for (int d = 0; d < 3; ++d) {
      mn[d] = bounds_in[(int64_t)j * 6 + d];
      mx[d] = bounds_in[(int64_t)j * 6 + 3 + d];
    }
  }
  const int dim = argmax3(dsub(mx[0], mn[0]), dsub(mx[1], mn[1]), dsub(mx[2], mn[2]));
  const int left = s.count - (s.count >> 1);
  const uint32_t pid = lists[dim * lstride + s.first + left];
  const double cut = coord[dim * cstride + pid];
  KdNode nd; nd.cut = cut; nd.dim = dim; nd.pad = 0;
  nodes[blocked_index(h)] = nd;
  level_dim[j] = dim;
  if (ccut) { ccut[h] = cut; cdim[h] = (uint8_t)dim; }
  if (cnode) cnode[h + 1] = packed_node(cut, dim);
  double* bl = bounds_out + (int64_t)(2 * j) * 6;
  double* br = bounds_out + (int64_t)(2 * j + 1) * 6;
  for (int d = 0; d < 3; ++d) {
    bl[d] = mn[d]; bl[3 + d] = (d == dim) ? cut : mx[d];
    br[d] = (d == dim) ? cut : mn[d]; br[3 + d] = mx[d];
  }
}

// ---- per level: side flag per point ----------------------------------------------------
__global__ void kd_flag_kernel(const uint32_t* __restrict__ lists, int64_t lstride, int n,
                               int bucket, int L, const int* __restrict__ level_dim,
                               uint8_t* __restrict__ flag) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int j, first, count;
  if (!locate_pos(i, L, n, bucket, &j, &first, &count)) return;
  const int dim = level_dim[j];
  const int left = count - (count >> 1);
  const uint32_t pid = lists[dim * lstride + i];
  flag[pid] = (i - first >= left) ? 1 : 0;
}

// ---- per level: stable partition of the three lists -------------------------------------
constexpr int kPartThreads = 256;
constexpr int kPartItems = 8;
constexpr int kPartTile = kPartThreads * kPartItems;

__global__ void __launch_bounds__(kPartThreads)
kd_part_count_kernel(const uint32_t* __restrict__ lists, int64_t lstride, int n, int bucket,
                     int L, const uint8_t* __restrict__ flag, uint32_t* __restrict__ gloc,
                     uint32_t* __restrict__ block_sum, int nblk) {
  __shared__ uint32_t warp_sums[kPartThreads / 32];
  const int d = blockIdx.y;
  const uint32_t* list = lists + d * lstride;
  const int base = blockIdx.x * kPartTile + threadIdx.x * kPartItems;
  uint32_t isleft[kPartItems];
  uint32_t cnt = 0;
#pragma unroll
  for (int r = 0; r < kPartItems; ++r) {
    const int i = base + r;
    uint32_t f = 0;
    if (i < n) {
      int j, first, count;
      const bool inner = locate_pos(i, L, n, bucket, &j, &first, &count);
      f = inner ? (flag[list[i]] == 0) : 1u;
    }
    isleft[r] = f;
    cnt += f;
  }
  uint32_t total;
  uint32_t run = block_scan_excl<kPartThreads / 32>(cnt, warp_sums, &total);
#pragma unroll
  for (int r = 0; r < kPartItems; ++r) {
    const int i = base + r;
    if (i < n) gloc[d * lstride + i] = run;
    run += isleft[r];
  }
  if (threadIdx.x == 0) block_sum[d * nblk + blockIdx.x] = total;
}

// FUSED_SCAN: block_off holds the RAW per-tile counts of kd_part_count_kernel and every block scans
// them itself (at most 256 tiles = 524 288 points), which saves one launch per tree level.
template <bool FUSED_SCAN>
__global__ void __launch_bounds__(kPartThreads)
kd_part_scatter_kernel(const uint32_t* __restrict__ lists, uint32_t* __restrict__ lists_out,
                       int64_t lstride, int n, int bucket, int L,
                       const uint8_t* __restrict__ flag, const uint32_t* __restrict__ gloc,
                       const uint32_t* __restrict__ block_off, int nblk) {
  __shared__ uint32_t s_off[kPartThreads];
  __shared__ uint32_t s_warp[kPartThreads / 32];
  const int d = blockIdx.y;
  if (FUSED_SCAN) {
    const int t = threadIdx.x;
    s_off[t] = block_scan_excl<kPartThreads / 32>(t < nblk ? block_off[d * nblk + t] : 0u, s_warp);
    __syncthreads();
  }
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* list = lists + d * lstride;
  const uint32_t pid = list[i];
  int j, first, count;
  const bool inner = locate_pos(i, L, n, bucket, &j, &first, &count);
  int pos = i;
  if (inner) {
    const uint32_t oi = FUSED_SCAN ? s_off[i / kPartTile] : block_off[d * nblk + i / kPartTile];
    const uint32_t of = FUSED_SCAN ? s_off[first / kPartTile] : block_off[d * nblk + first / kPartTile];
    const uint32_t gi = gloc[d * lstride + i] + oi;
    const uint32_t gs = gloc[d * lstride + first] + of;
    const int rank_left = (int)(gi - gs);
    const int left = count - (count >> 1);
    pos = (flag[pid] == 0) ? first + rank_left : first + left + ((i - first) - rank_left);
  }
  lists_out[d * lstride + pos] = pid;
}

// ---- the bottom of the tree inside one CTA ------------------------------------------------------
// Once a node's segment fits a CTA's shared memory (<= kSubMax points) its whole subtree is finished by
// ONE CTA: the same four steps per level (nodes, side flags, stable partition of the three lists), with
// __syncthreads between them instead of four launches per level.  For a 106 784-point target the global
// passes stop at level 6 (segments of <= 1 669 points) and 64 CTAs do levels 6..13: 56 launches become 25.
// The tree is the same one (same medians, same tie rule, same implicit bounds).  tests/test_gpu_kdtree_stages.py
// compares every array each tree owner fills with a numpy model of the build (tests/kd_tree_model.py), node for
// node, at n = capacity and capacity + 1 for every bucket size and past the unfused partition scan.
constexpr int kSubThreads = 512;
constexpr int kSubItems = 4;
constexpr int kSubMax = kSubThreads * kSubItems;     // 2048 points
constexpr int kSubNodes = 256;                       // a level with an inner node has <= count / bucket nodes

__host__ __device__ __forceinline__ int kd_sub_capacity(int bucket) { return min(kSubMax, kSubNodes * bucket); }

struct SubSeg { int jl, first, count; bool at_level; };
// local position i of a subtree segment of `count0` points -> the node of local level k containing it
__device__ __forceinline__ SubSeg sub_locate(int i, int k, int count0, int bucket) {
  int first = 0, count = count0, jl = 0;
  for (int l = 0; l < k; ++l) {
    if (count <= bucket) return SubSeg{jl, first, count, false};
    const int right = count >> 1, left = count - right;
    if (i < first + left) { jl = 2 * jl; count = left; }
    else { jl = 2 * jl + 1; first += left; count = right; }
  }
  return SubSeg{jl, first, count, true};
}

__global__ void __launch_bounds__(kSubThreads)
kd_subtree_kernel(const double* __restrict__ coord, int64_t cstride, uint32_t* __restrict__ lists, int64_t lstride,
                  int n, int bucket, int Lg, int levels, const double* __restrict__ bounds_in,
                  uint8_t* __restrict__ flag, KdNode* __restrict__ nodes, double* __restrict__ ccut,
                  uint8_t* __restrict__ cdim, double2* __restrict__ cnode) {
  __shared__ uint32_t s_list[3][kSubMax];
  __shared__ uint32_t s_scan[kSubMax + 1];
  __shared__ double s_bounds[kSubNodes][6];
  __shared__ int s_ndim[kSubNodes];
  __shared__ uint32_t s_warp[kSubThreads / 32];
  __shared__ int s_any_inner;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const int j0 = blockIdx.x;
  const Seg seg0 = locate_node(j0, Lg, n, bucket);
  if (!seg0.exists || seg0.count <= bucket) {                // a leaf (or nothing) at level Lg: kd_leaf_kernel's job
    if (seg0.exists && cdim && Lg < levels && threadIdx.x == 0) {
      cdim[(1 << Lg) - 1 + j0] = 3;
      if (cnode) cnode[(1 << Lg) + j0] = packed_node(0.0, 3);
    }
    return;
  }
  const int count0 = seg0.count;
  for (int d = 0; d < 3; ++d)
    for (int i = t; i < count0; i += kSubThreads) s_list[d][i] = lists[d * lstride + seg0.first + i];
  if (t < 6) {
    if (Lg == 0) {     // root bounds: per-axis min / max of the data (the sorted lists' ends)
      const int d = t % 3;
      const uint32_t pid = lists[d * lstride + (t < 3 ? 0 : n - 1)];
      s_bounds[0][t] = coord[d * cstride + pid];
    } else {
      s_bounds[0][t] = bounds_in[(int64_t)j0 * 6 + t];
    }
  }
  __syncthreads();
  for (int k = 0; Lg + k < levels; ++k) {
    const int L = Lg + k, nnodes = 1 << k;
    if (t == 0) s_any_inner = 0;
    __syncthreads();
    // ---- nodes of this level (children bounds are formed in registers and stored after the barrier) ----
    double bl[6], br[6];
    bool has_children = false;
    for (int jl = t; jl < nnodes; jl += kSubThreads) {        // > kSubThreads nodes only on all-leaf levels
      int first = 0, count = count0;
      bool exists = true;
      for (int l = k - 1; l >= 0; --l) {
        if (count <= bucket) { exists = false; break; }
        const int right = count >> 1, left = count - right;
        if ((jl >> l) & 1) { first += left; count = right; } else { count = left; }
      }
      if (jl < kSubNodes) s_ndim[jl] = 3;
      if (!exists) continue;
      const int h = (1 << L) - 1 + ((j0 << k) | jl);
      if (count <= bucket) {
        KdNode leaf;
        leaf.cut = __longlong_as_double(((long long)count << 32) | (long long)(unsigned)(seg0.first + first));
        leaf.dim = 3; leaf.pad = 0;
        nodes[blocked_index(h)] = leaf;
        if (cdim) cdim[h] = 3;
        if (cnode) cnode[h + 1] = packed_node(0.0, 3);
        continue;
      }
      double mn[3], mx[3];
      for (int d = 0; d < 3; ++d) { mn[d] = s_bounds[jl][d]; mx[d] = s_bounds[jl][3 + d]; }
      const int dim = argmax3(dsub(mx[0], mn[0]), dsub(mx[1], mn[1]), dsub(mx[2], mn[2]));
      const int left = count - (count >> 1);
      const uint32_t pid = s_list[dim][first + left];
      const double cut = coord[dim * cstride + pid];
      KdNode nd; nd.cut = cut; nd.dim = dim; nd.pad = 0;
      nodes[blocked_index(h)] = nd;
      if (ccut) { ccut[h] = cut; cdim[h] = (uint8_t)dim; }
      if (cnode) cnode[h + 1] = packed_node(cut, dim);
      s_ndim[jl] = dim;
      s_any_inner = 1;
      for (int d = 0; d < 3; ++d) {
        bl[d] = mn[d]; bl[3 + d] = (d == dim) ? cut : mx[d];
        br[d] = (d == dim) ? cut : mn[d]; br[3 + d] = mx[d];
      }
      has_children = true;                                     // inner nodes only exist while nnodes <= kSubNodes
    }
    __syncthreads();
    if (!s_any_inner) break;
    if (has_children && 2 * t + 1 < kSubNodes) {
      for (int d = 0; d < 6; ++d) { s_bounds[2 * t][d] = bl[d]; s_bounds[2 * t + 1][d] = br[d]; }
    }
    // NOTE: with nnodes <= kSubNodes / 2 every inner node is handled by thread jl == t (one node per thread)
    // ---- side flags + per-item node data ---------------------------------------------------------------
    int it_first[kSubItems], it_left[kSubItems];
    bool it_inner[kSubItems];
#pragma unroll
    for (int r = 0; r < kSubItems; ++r) {
      const int i = t * kSubItems + r;
      it_inner[r] = false; it_first[r] = 0; it_left[r] = 0;
      if (i < count0) {
        const SubSeg sg = sub_locate(i, k, count0, bucket);
        if (sg.at_level && sg.count > bucket) {
          const int dim = s_ndim[sg.jl];
          it_inner[r] = true; it_first[r] = sg.first; it_left[r] = sg.count - (sg.count >> 1);
          flag[s_list[dim][i]] = (i - sg.first >= it_left[r]) ? 1 : 0;
        }
      }
    }
    __syncthreads();
    // ---- stable partition of the three lists (block scan of the left flags, in place) ------------------------
    for (int d = 0; d < 3; ++d) {
      uint32_t pid[kSubItems], isleft[kSubItems], cnt = 0;
#pragma unroll
      for (int r = 0; r < kSubItems; ++r) {
        const int i = t * kSubItems + r;
        pid[r] = i < count0 ? s_list[d][i] : 0u;
        isleft[r] = (i < count0 && it_inner[r]) ? (flag[pid[r]] == 0 ? 1u : 0u) : 1u;
        cnt += isleft[r];
      }
      const uint32_t incl = warp_inclusive_scan(cnt);
      if (lane == 31) s_warp[w] = incl;
      __syncthreads();
      uint32_t wb = 0;
      for (int ww = 0; ww < w; ++ww) wb += s_warp[ww];
      uint32_t run = wb + incl - cnt;
#pragma unroll
      for (int r = 0; r < kSubItems; ++r) { s_scan[t * kSubItems + r] = run; run += isleft[r]; }
      __syncthreads();
#pragma unroll
      for (int r = 0; r < kSubItems; ++r) {
        const int i = t * kSubItems + r;
        if (i >= count0) continue;
        int pos = i;
        if (it_inner[r]) {
          const int rank_left = (int)(s_scan[i] - s_scan[it_first[r]]);
          pos = isleft[r] ? it_first[r] + rank_left : it_first[r] + it_left[r] + ((i - it_first[r]) - rank_left);
        }
        s_list[d][pos] = pid[r];      // every position is read (into registers) before the barrier above
      }
      __syncthreads();
    }
  }
  // the x-ordered list, partitioned down to the leaves, goes back for kd_leaf_kernel
  for (int i = t; i < count0; i += kSubThreads) lists[seg0.first + i] = s_list[0][i];
}

// ---- leaves: canonical (ascending original index) order ---------------------------------
__global__ void kd_leaf_kernel(const uint32_t* __restrict__ list0, int n, int bucket, int levels,
                               KdNode* __restrict__ nodes, uint32_t* __restrict__ leaf_order) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = (1 << (levels + 1)) - 1;
  if (h >= total) return;
  const int L = 31 - __clz(h + 1);
  const int j = h + 1 - (1 << L);
  const Seg s = locate_node(j, L, n, bucket);
  if (!s.exists || s.count > bucket) return;
  KdNode leaf;
  leaf.cut = __longlong_as_double(((long long)s.count << 32) | (long long)(unsigned)s.first);
  leaf.dim = 3; leaf.pad = 0;
  nodes[blocked_index(h)] = leaf;
  uint32_t ids[16];
  for (int k = 0; k < s.count; ++k) ids[k] = list0[s.first + k];
  for (int a = 1; a < s.count; ++a) {  // insertion sort, count <= bucket <= 16
    const uint32_t v = ids[a];
    int b = a - 1;
    while (b >= 0 && ids[b] > v) { ids[b + 1] = ids[b]; --b; }
    ids[b + 1] = v;
  }
  for (int k = 0; k < s.count; ++k) leaf_order[s.first + k] = ids[k];
}

// ---- compact search layout (KdCompact, kernels.h): padded buckets ------------------------
// Entry e = bucket * 8 + k of the padded bucket space; bucket = in-level index of a leaf at
// level `levels`, or (index << 1) of a leaf one level higher (its odd twin stays empty).
// Coordinates are stored per bucket as x[8] y[8] z[8]; empty entries hold +inf, so their
// squared distance is +inf (or NaN) and the strict '<' of the search never takes them.
// pm (normals trees): the same point beside its normal, one 64-byte record per entry (zero normal when empty).
__global__ void kd_compact_buckets_kernel(const double* __restrict__ coord, int64_t cstride,
                                          const double* __restrict__ nrm, int64_t nstride,
                                          const uint32_t* __restrict__ leaf_order, int n, int bucket,
                                          int levels, double* __restrict__ pb,
                                          BucketMatch* __restrict__ pm, int32_t* __restrict__ pid) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= ((int64_t)8 << levels)) return;
  const int jL = (int)(e >> 3), k = (int)(e & 7);
  int first = 0, count = n, l = 0;
  while (l < levels && count > bucket) {
    const int right = count >> 1, left = count - right;
    if ((jL >> (levels - 1 - l)) & 1) { first += left; count = right; } else { count = left; }
    ++l;
  }
  const bool owner = (jL & ((1 << (levels - l)) - 1)) == 0;   // left-most descendant slot of the leaf
  const bool valid = owner && k < count;
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  double x = inf, y = inf, z = inf;
  double nx = 0.0, ny = 0.0, nz = 0.0;
  int32_t id = -1;
  if (valid) {
    id = (int32_t)leaf_order[first + k];
    x = coord[id]; y = coord[cstride + id]; z = coord[2 * cstride + id];
    if (nrm) { nx = nrm[id]; ny = nrm[nstride + id]; nz = nrm[2 * nstride + id]; }
  }
  double* o = pb + (int64_t)jL * 24 + k;
  o[0] = x; o[8] = y; o[16] = z;
  if (pm) {
    double2* r = reinterpret_cast<double2*>(pm + e);
    r[0] = make_double2(x, y); r[1] = make_double2(z, nx);
    r[2] = make_double2(ny, nz); r[3] = make_double2(0.0, 0.0);
  }
  if (pid) pid[e] = id;
}

// bucket slot s of the blocked tree (FloatTree): the point of leaf_order[s]
__global__ void fill_buckets_kernel(const double* __restrict__ coord, int64_t cstride,
                                    const uint32_t* __restrict__ leaf_order, int n, BucketPoint* __restrict__ bpts) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const uint32_t id = leaf_order[s];
  BucketPoint p;
  p.x = coord[id]; p.y = coord[cstride + id]; p.z = coord[2 * cstride + id]; p.id = id;
  bpts[s] = p;
}

// keys32: the coordinates are exactly representable as float (clouds that entered as float): the float
// bit pattern orders them like the double one and the sort needs 4 byte passes instead of 8
__global__ void kd_keys_kernel(const double* __restrict__ coord, int64_t cstride, int n,
                               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals,
                               int64_t lstride, int keys32) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    // + 0.0 turns -0.0 into +0.0 (every other value is unchanged): the reference's comparator, and the oracle's
    // total order (coordinate, index), treat the two zeros as EQUAL coordinates, the bit-pattern key would not
    const double v = dadd(coord[d * cstride + i], 0.0);
    uint64_t key;
    if (keys32) {
      const uint32_t u = __float_as_uint((float)v);
      key = (u >> 31) ? (uint32_t)~u : (u | 0x80000000u);
    } else {
      key = sortable_key(v);
    }
    keys[d * lstride + i] = key;
    vals[d * lstride + i] = (uint32_t)i;
  }
}

}  // namespace

int kd_num_levels(int n, int bucket) {
  int L = 0;
  int64_t c = n;
  while (c > bucket) { c = (c + 1) / 2; ++L; }  // ceil halving: largest node of the level
  return L;  // all nodes of level L are leaves; heap has 2^(L+1)-1 slots
}

static size_t kd_workspace_bytes(int n, int bucket) {
  const int levels = kd_num_levels(n, bucket);
  const int64_t ls = (n + 63) & ~63;
  size_t b = 0;
  b += 2 * 3 * ls * sizeof(uint64_t);                // keys ping-pong
  b += 2 * 3 * ls * sizeof(uint32_t);                // lists ping-pong
  b += 3 * ls * sizeof(uint32_t);                    // gloc
  b += ls;                                           // flag
  b += radix_sort_scratch_bytes(n, 3) + 256;         // sort scratch / block sums
  b += 2 * ((size_t)1 << levels) * 6 * sizeof(double);  // bounds ping-pong
  b += ((size_t)1 << levels) * sizeof(int);          // level dims
  return b + 4096;
}

int KdWorkspace::carve(DevBuf& buf, int n, int bucket) {
  SMB_RC(buf.reserve(kd_workspace_bytes(n, bucket)));
  const int levels = kd_num_levels(n, bucket);
  lstride = (n + 63) & ~63;
  char* p = (char*)buf.p;
  auto take = [&](size_t bytes) { char* r = p; p += (bytes + 255) & ~(size_t)255; return r; };
  keys[0] = (uint64_t*)take(3 * lstride * sizeof(uint64_t));
  keys[1] = (uint64_t*)take(3 * lstride * sizeof(uint64_t));
  lists[0] = (uint32_t*)take(3 * lstride * sizeof(uint32_t));
  lists[1] = (uint32_t*)take(3 * lstride * sizeof(uint32_t));
  gloc = (uint32_t*)take(3 * lstride * sizeof(uint32_t));
  flag = (uint8_t*)take(lstride);
  scratch = (uint32_t*)take(radix_sort_scratch_bytes(n, 3) + 256);
  bounds[0] = (double*)take(((size_t)1 << levels) * 6 * sizeof(double));
  bounds[1] = (double*)take(((size_t)1 << levels) * 6 * sizeof(double));
  level_dim = (int*)take(((size_t)1 << levels) * sizeof(int));
  return 0;
}

// entries of the compact layout's cut[] / dim[]: 2^levels - 1 inner-capable nodes, rounded up to a multiple of
// 16 because bulk copies move multiples of 16 bytes
static size_t kd_compact_node_slots(int levels) {
  const size_t n = (size_t)1 << levels;
  return n < 16 ? 16 : n;
}

// node[] of the compact layout, behind cut[] in the same allocation
static double2* compact_node_array(const KdCompactTree& t) {
  return reinterpret_cast<double2*>((double*)t.cut.p + kd_compact_node_slots(t.levels));
}

// coord: SoA [3][cstride] doubles (already centred).  Writes nodes (heap layout,
// 2^(levels+1)-1 entries) and leaf_order[n] (point ids in bucket order).
int kd_build(const double* coord, int64_t cstride, int n, int bucket, KdWorkspace& ws,
             KdNode* nodes, uint32_t* leaf_order, cudaStream_t stream, const KdCompactTree* compact,
             bool coords_are_float) {
  if (n <= 0) return -1;
  double* ccut = compact ? (double*)compact->cut.p : nullptr;
  uint8_t* cdim = compact ? (uint8_t*)compact->dim.p : nullptr;
  double2* cnode = compact ? compact_node_array(*compact) : nullptr;
  const int levels = kd_num_levels(n, bucket);
  const int64_t ls = ws.lstride;
  kd_keys_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(coord, cstride, n, ws.keys[0],
                                                       ws.lists[0], ls, coords_are_float ? 1 : 0);
  int rc = radix_sort_pairs_u64(ws.keys[0], ws.lists[0], ws.keys[1], ws.lists[1], n, 3, ls,
                                ws.scratch, stream, coords_are_float ? 4 : 8);
  if (rc) return rc;
  int cur = 0;
  const int nblk = ceil_div(n, kPartTile);
  // global passes down to the level whose segments fit one CTA, the rest of every subtree in shared memory
  int Lg = 0;
  {
    const int cap = kd_sub_capacity(bucket);
    int64_t c = n;
    while (Lg < levels && c > cap) { c = (c + 1) / 2; ++Lg; }
  }
  for (int L = 0; L < Lg; ++L) {
    const int nodes_l = 1 << L;
    kd_node_kernel<<<ceil_div(nodes_l, 128), 128, 0, stream>>>(
        coord, cstride, ws.lists[cur], ls, n, bucket, L, ws.bounds[L & 1], ws.bounds[(L + 1) & 1],
        ws.level_dim, nodes, ccut, cdim, cnode);
    kd_flag_kernel<<<ceil_div(n, 256), 256, 0, stream>>>(ws.lists[cur], ls, n, bucket, L,
                                                        ws.level_dim, ws.flag);
    kd_part_count_kernel<<<dim3(nblk, 3), kPartThreads, 0, stream>>>(
        ws.lists[cur], ls, n, bucket, L, ws.flag, ws.gloc, ws.scratch, nblk);
    if (nblk <= kPartThreads) {
      kd_part_scatter_kernel<true><<<dim3(ceil_div(n, kPartThreads), 3), kPartThreads, 0, stream>>>(
          ws.lists[cur], ws.lists[cur ^ 1], ls, n, bucket, L, ws.flag, ws.gloc, ws.scratch, nblk);
    } else {
      radix_scan_kernel_launch(ws.scratch, nblk, 3, stream);
      kd_part_scatter_kernel<false><<<dim3(ceil_div(n, kPartThreads), 3), kPartThreads, 0, stream>>>(
          ws.lists[cur], ws.lists[cur ^ 1], ls, n, bucket, L, ws.flag, ws.gloc, ws.scratch, nblk);
    }
    cur ^= 1;
  }
  if (Lg < levels)
    kd_subtree_kernel<<<1 << Lg, kSubThreads, 0, stream>>>(coord, cstride, ws.lists[cur], ls, n, bucket, Lg, levels,
                                                          ws.bounds[Lg & 1], ws.flag, nodes, ccut, cdim, cnode);
  const int total = (1 << (levels + 1)) - 1;
  kd_leaf_kernel<<<ceil_div(total, 128), 128, 0, stream>>>(ws.lists[cur], n, bucket, levels,
                                                          nodes, leaf_order);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

int KdCompactTree::reserve(int n, int bucket, Payload payload) {
  levels = kd_num_levels(n, bucket);
  const size_t slots = kd_compact_node_slots(levels), entries = (size_t)8 << levels;
  SMB_RC(nodes.reserve((size_t)blocked_node_slots(levels) * sizeof(KdNode)));
  SMB_RC(leaf_order.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(cut.reserve(slots * (sizeof(double) + sizeof(double2))));
  SMB_RC(dim.reserve(slots));
  SMB_RC(pb.reserve(entries * 3 * sizeof(double)));
  return payload == kNormals ? pm.reserve(entries * sizeof(BucketMatch)) : pid.reserve(entries * sizeof(int32_t));
}

int KdCompactTree::build(const double* coord, const double* nrm, int64_t cstride, int n, int bucket,
                         KdWorkspace& ws, cudaStream_t stream) const {
  if (bucket > 8) return -1;
  SMB_RC(kd_build(coord, cstride, n, bucket, ws, (KdNode*)nodes.p, (uint32_t*)leaf_order.p, stream, this));
  const int64_t total = (int64_t)8 << levels;
  kd_compact_buckets_kernel<<<ceil_div(total, 256), 256, 0, stream>>>(
      coord, cstride, nrm, cstride, (const uint32_t*)leaf_order.p, n, bucket, levels, (double*)pb.p,
      (BucketMatch*)pm.p, (int32_t*)pid.p);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

KdCompact KdCompactTree::view() const {
  return {(const double*)cut.p, (const uint8_t*)dim.p, compact_node_array(*this), (const double*)pb.p,
          (const BucketMatch*)pm.p, (const int32_t*)pid.p, levels, 0};
}

int FloatTree::build(const float* pts, int n, DevBuf& kdws, cudaStream_t stream) {
  const int levels = kd_num_levels(n, 8);
  const int64_t stride = ((int64_t)n + 63) & ~(int64_t)63;
  SMB_RC(soa.reserve((size_t)(3 * stride) * sizeof(double)));
  SMB_RC(nodes.reserve((size_t)blocked_node_slots(levels) * sizeof(KdNode)));
  SMB_RC(order.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(bpts.reserve((size_t)(n + 8) * sizeof(BucketPoint)));
  KdWorkspace ws;
  SMB_RC(ws.carve(kdws, n, 8));
  SMB_RC(ndt_float_to_soa(pts, n, (double*)soa.p, stride, stream));
  SMB_RC(kd_build((const double*)soa.p, stride, n, 8, ws, (KdNode*)nodes.p, (uint32_t*)order.p, stream, nullptr,
                  true));       // the cloud entered as float: 32-bit sort keys
  fill_buckets_kernel<<<ceil_div(n, 256), 256, 0, stream>>>((const double*)soa.p, stride, (const uint32_t*)order.p, n,
                                                            (BucketPoint*)bpts.p);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace smb
