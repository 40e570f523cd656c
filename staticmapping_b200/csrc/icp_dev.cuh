// Device-side building blocks of the ICP iteration shared by icp.cu (phases A, B) and
// icp_finish.cu (phase C).  See icp.cu for the phase structure.
#ifndef SM_B200_ICP_DEV_CUH_
#define SM_B200_ICP_DEV_CUH_

#include "common.cuh"
#include "kernels.h"

namespace smb {
namespace dev {

#ifndef SMB_KNN_THREADS
#define SMB_KNN_THREADS 256
#endif
constexpr int kKnnThreads = SMB_KNN_THREADS;
constexpr int kAccThreads = 256;
constexpr int kAccItems = 2;
constexpr int kAccTile = kAccThreads * kAccItems;  // points per accumulate block
constexpr int kNumSums = 29;                        // 21 (A upper) + 6 (b) + sum sqrt + count
constexpr int kFinThreads = 1024;
constexpr int kMaxStack = 32;

// monotone bin of a non-negative finite double: 1/32-octave resolution over 2^-40..2^24
__device__ __forceinline__ int dist_bin(double d2) {
  const long long bits = __double_as_longlong(d2);
  const int key = (int)(bits >> 47) - ((1023 - 40) << 5);
  return min(max(key, 0), kHistBins - 1);
}

// second-level bin inside one first-level bin: the next 11 bits (valid when the first-level
// bin is not one of the two clamp bins, i.e. all its members share bits 63..47)
__device__ __forceinline__ int sub_bin(double d2) {
  return (int)((__double_as_longlong(d2) >> 36) & 2047ll);
}
__device__ __forceinline__ bool clamp_bin(int bin) { return bin <= 0 || bin >= kHistBins - 1; }

__device__ __forceinline__ bool finite_d2(double d) { return d < __longlong_as_double(0x7ff0000000000000ll); }

// p = T (x) s with the reference's accumulation order (cloud_types.cc:288-296)
__device__ __forceinline__ void transform_point(const double* __restrict__ T, double x, double y,
                                                double z, double& px, double& py, double& pz) {
  px = dadd(dadd(dadd(dmul(T[0], x), dmul(T[4], y)), dmul(T[8], z)), T[12]);
  py = dadd(dadd(dadd(dmul(T[1], x), dmul(T[5], y)), dmul(T[9], z)), T[13]);
  pz = dadd(dadd(dadd(dmul(T[2], x), dmul(T[6], y)), dmul(T[10], z)), T[14]);
}

__device__ __forceinline__ KdNode load_node(const KdNode* __restrict__ nodes, int h) {
  const int4 v = __ldg(reinterpret_cast<const int4*>(nodes + h));
  KdNode n;
  n.cut = __hiloint2double(v.y, v.x);
  n.dim = v.z; n.pad = v.w;
  return n;
}

// 16-byte / 8-byte read-only loads as volatile asm: issued in program order, so the 16 loads
// of a bucket go out back to back (one L2 round trip per bucket instead of eight).
__device__ __forceinline__ double2 ldg_f64x2(const void* p) {
  double2 v;
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}
__device__ __forceinline__ double ldg_f64(const void* p) {
  double v;
  asm volatile("ld.global.nc.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

// Scan one bucket.  All 8 entries are fetched up front (the bucket array is padded by 8
// entries, so reading past `count` is safe); entries >= count are ignored.
// libnabo walks the bucket in order and replaces the head on a strict '<', i.e. it ends with the
// FIRST entry that attains the bucket minimum, provided that minimum is below the head.  The 8
// squared distances are formed with the reference's exact operation order; the selection then
// runs on their bit patterns (non-negative doubles order like unsigned integers; a NaN sorts
// above +inf and is never taken, like a false '<') as a 3-level tournament in which the lower
// index wins ties.  FP64 compares sit on the 23-cycle double pipe (profiles/microbench), so a
// serial compare/select chain over 8 entries was the longest dependency of a bucket visit.
__device__ __forceinline__ void scan_leaf(const BucketPoint* __restrict__ bpts, const KdNode& leaf,
                                          double qx, double qy, double qz, double& head,
                                          int& best) {
  const long long packed = __double_as_longlong(leaf.cut);
  const int first = (int)(packed & 0xffffffffll), count = (int)(packed >> 32);
  double2 xy[8];
  double z[8];
  const char* base = reinterpret_cast<const char*>(bpts + first);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    xy[k] = ldg_f64x2(base + 32 * k);
    z[k] = ldg_f64(base + 32 * k + 16);
  }
  unsigned long long key[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double dx = dsub(qx, xy[k].x), dy = dsub(qy, xy[k].y), dz = dsub(qz, z[k]);
    const double dist = dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz));
    key[k] = k < count ? (unsigned long long)__double_as_longlong(dist) : ~0ull;
  }
  int arg[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) arg[k] = k;
#pragma unroll
  for (int step = 1; step < 8; step <<= 1) {
#pragma unroll
    for (int k = 0; k < 8; k += 2 * step) {
      const bool take = key[k + step] < key[k];      // strict: the lower index keeps a tie
      key[k] = take ? key[k + step] : key[k];
      arg[k] = take ? arg[k + step] : arg[k];
    }
  }
  if (key[0] < (unsigned long long)__double_as_longlong(head)) {
    head = __longlong_as_double((long long)key[0]);
    best = first + arg[0];
  }
}

struct StackEntry {
  double rd, ox, oy, oz;
  int idx;
};

// child of the node at blocked index `idx` (see blocked_index in common.cuh): inside a
// 7-node block the local heap rule applies; leaving a block jumps to one of its 8 child blocks.
__device__ __forceinline__ int child_idx(int idx, int right) {
  const int p = idx & 7, B = idx >> 3;
  return (p < 3) ? ((B << 3) | (2 * p + 1 + right))
                 : ((8 * B + 1 + (((p - 3) << 1) | right)) << 3);
}

// Visit the subtree rooted at `idx` exactly like libnabo's recurseKnn would (near child
// first, far child if rd*(1+eps)^2 < head at that moment).  Far subtrees are pushed only if
// they pass the test against the head known at push time (the head only shrinks, so nothing
// the recursion would visit is dropped) and re-tested when popped, which is when the
// recursion tests them.
// The side of the cut is decided by `q > cut` (== `q - cut > 0` for IEEE doubles) and the near
// child's node is requested at once; the far-side bookkeeping (new_off, rd, the push test: six
// dependent FP64 operations) then runs in the shadow of that load instead of in front of it.
// The pending subtrees live in (L1-cached) local memory: a shared-memory stack was measured
// slower, it takes its bytes from the L1 that caches the tree lines.
__device__ __forceinline__ int visit_subtree(const KdNode* __restrict__ nodes,
                                              const BucketPoint* __restrict__ bpts, double qx,
                                              double qy, double qz, double max_error2, int idx,
                                              double rd, double ox, double oy, double oz,
                                              double& head, int& best, int max_rounds = 1 << 20,
                                              bool first_bucket_scanned = false) {
  StackEntry stack[kMaxStack];
  int sp = 0, rounds = 0;
  while (max_rounds-- > 0) {
    ++rounds;
    KdNode nd = load_node(nodes, idx);
    int guard = 0;
    while (nd.dim != 3 && ++guard < 64) {   // a valid tree is at most 25 levels deep
      const int cd = nd.dim;
      const double q = cd == 0 ? qx : (cd == 1 ? qy : qz);
      const double old_off = cd == 0 ? ox : (cd == 1 ? oy : oz);
      const int right = q > nd.cut ? 1 : 0;
      const int next = child_idx(idx, right);
      const KdNode nd_next = load_node(nodes, next);
      const double new_off = dsub(q, nd.cut);
      // rd += - old_off*old_off + new_off*new_off
      const double rd_new = dadd(rd, dadd(-dmul(old_off, old_off), dmul(new_off, new_off)));
      if (dmul(rd_new, max_error2) < head && sp < kMaxStack) {
        StackEntry e;
        e.rd = rd_new;
        e.ox = cd == 0 ? new_off : ox;
        e.oy = cd == 1 ? new_off : oy;
        e.oz = cd == 2 ? new_off : oz;
        e.idx = child_idx(idx, 1 - right);
        stack[sp++] = e;
      }
      idx = next;
      nd = nd_next;
    }
    if (nd.dim == 3 && !(first_bucket_scanned && rounds == 1)) scan_leaf(bpts, nd, qx, qy, qz, head, best);
    bool found = false;
    while (sp > 0) {
      const StackEntry e = stack[--sp];
      if (dmul(e.rd, max_error2) < head) {
        idx = e.idx; rd = e.rd; ox = e.ox; oy = e.oy; oz = e.oz;
        found = true;
        break;
      }
    }
    if (!found) break;
  }
  return rounds;
}

// libnabo knn, k = 1, allowSelfMatch, maxRadius = inf (icp_fast.cc:177-178), one query per
// thread.  A read-only first descent seeds the head; along it rd_new == new_off^2 exactly
// (rd = 0, all offsets 0), so if min(new_off^2)*(1+eps)^2 >= head no far subtree can ever
// qualify and the query is done after one bucket.  Otherwise the recursion is replayed from
// the root by visit_subtree (ONE loop for all far visits: the k-th bucket visit of every lane
// of a warp happens in the same round, so a warp costs max-over-lanes rounds).
__device__ __forceinline__ void knn1(const KdNode* __restrict__ nodes,
                                     const BucketPoint* __restrict__ bpts, double qx, double qy,
                                     double qz, double max_error2, int& best_slot, double& best_d2,
                                     int max_rounds = 1 << 30, int* rounds_out = nullptr) {
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  double head = inf;
  int best = -1;
  int idx = 0;
  double min_off2 = inf;
  KdNode nd = load_node(nodes, 0);
  int guard = 0;
  while (nd.dim != 3 && ++guard < 64) {
    const double q = nd.dim == 0 ? qx : (nd.dim == 1 ? qy : qz);
    idx = child_idx(idx, (q > nd.cut) ? 1 : 0);
    const KdNode nd_next = load_node(nodes, idx);
    const double off = dsub(q, nd.cut);
    min_off2 = fmin(min_off2, dmul(off, off));
    nd = nd_next;
  }
  if (nd.dim == 3) scan_leaf(bpts, nd, qx, qy, qz, head, best);
  // re-scanning the first bucket during the replay is harmless (strict '<' keeps the winner)
  int rounds = 0;
  if (dmul(min_off2, max_error2) < head)
    rounds = visit_subtree(nodes, bpts, qx, qy, qz, max_error2, 0, 0.0, 0.0, 0.0, 0.0, head, best, max_rounds, true);
  if (rounds_out) *rounds_out = rounds;
  best_slot = best;
  best_d2 = head;
}

struct BinSel { int bin; int below; int qi; int nvalid; };

// every block locates the quantile bin from the global histogram (2048 bins, 8 per thread
// on the first 256 threads; all threads of the block must call this)
__device__ __forceinline__ BinSel select_bin(const uint32_t* __restrict__ ghist, float ratio,
                                             uint32_t* warp_tot /*[8]*/, BinSel* out_sm) {
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  const bool active = t < 256;
  uint32_t c[8], s = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) { c[k] = active ? ghist[t * 8 + k] : 0u; s += c[k]; }
  uint32_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (active && lane == 31) warp_tot[w] = incl;
  if (t == 0) { out_sm->bin = -1; out_sm->below = 0; out_sm->qi = 0; out_sm->nvalid = 0; }   // never left unset
  __syncthreads();
  uint32_t base = 0, total = 0;
#pragma unroll
  for (int ww = 0; ww < 8; ++ww) { const uint32_t v = warp_tot[ww]; if (ww < w) base += v; total += v; }
  const uint32_t excl = base + incl - s;
  // icp_fast.cc:82-89: quantile == 1.0 -> max element, else index int(size * quantile)
  const double q = (double)ratio;
  int qi = (q == 1.0) ? (int)total - 1 : (int)((double)total * q);
  if (qi > (int)total - 1) qi = (int)total - 1;
  if (active && total > 0 && (uint32_t)qi >= excl && (uint32_t)qi < excl + s) {
    uint32_t run = excl;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      if ((uint32_t)qi >= run && (uint32_t)qi < run + c[k]) {
        out_sm->bin = t * 8 + k; out_sm->below = (int)run;
      }
      run += c[k];
    }
    out_sm->qi = qi; out_sm->nvalid = (int)total;
  }
  __syncthreads();
  return *out_sm;
}

// contribution of one match to the normal equations (icp_fast.cc:268-302), in two halves so
// that phase B can park the terms of a quantile-bin member for phase C
__host__ __device__ __forceinline__ void match_terms(double px, double py, double pz, const BucketPoint& q,
                                            const BucketNormal& n, double* F, double& dot) {
  F[0] = py * n.z - pz * n.y;
  F[1] = pz * n.x - px * n.z;
  F[2] = px * n.y - py * n.x;
  F[3] = n.x; F[4] = n.y; F[5] = n.z;
  dot = (px - q.x) * n.x + (py - q.y) * n.y + (pz - q.z) * n.z;
}
// IcpFast with inner compensation (icp_fast.cc:284-289): the Jacobian column of the match scaled by the point's
// factor f (wF and F both, so A sums (f F)(f F)^T and b sums (f F) * dot); the residual is not scaled
__host__ __device__ __forceinline__ void compensated_match_terms(double px, double py, double pz, const BucketPoint& q,
                                                                 const BucketNormal& n, double f, double* F,
                                                                 double& dot) {
  match_terms(px, py, pz, q, n, F, dot);
#pragma unroll
  for (int r = 0; r < 6; ++r) F[r] = F[r] * f;
}
__host__ __device__ __forceinline__ void add_terms(double* acc, const double* F, double dot, double d2) {
  int k = 0;
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int c = r; c < 6; ++c) acc[k++] += F[r] * F[c];
#pragma unroll
  for (int r = 0; r < 6; ++r) acc[21 + r] += F[r] * dot;
  acc[27] += sqrt(d2);
  acc[28] += 1.0;
}
// acc += pred ? terms : 0 (adding +0.0 leaves a sum unchanged, so no branch is needed and the
// loads feeding several matches can be in flight together); sq = sqrt(d2)
__device__ __forceinline__ void add_terms_if(double* acc, const double* Fin, double dot_in, double sq,
                                             bool pred) {
  double F[6];
#pragma unroll
  for (int r = 0; r < 6; ++r) F[r] = pred ? Fin[r] : 0.0;
  const double dot = pred ? dot_in : 0.0;
  int k = 0;
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int c = r; c < 6; ++c) acc[k++] += F[r] * F[c];
#pragma unroll
  for (int r = 0; r < 6; ++r) acc[21 + r] += F[r] * dot;
  acc[27] += pred ? sq : 0.0;
  acc[28] += pred ? 1.0 : 0.0;
}

// Sum 32 per-lane values across the warp: on return lane L holds the warp total of v[L].
// 31 exchanges instead of the 160 of 32 separate butterflies; the pairing is the butterfly's
// (offsets 16, 8, 4, 2, 1), so each total is bit-identical to the xor-shuffle reduction.
__device__ __forceinline__ double warp_transpose_reduce32(double (&v)[32], int lane) {
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) {
    const bool up = (lane & h) != 0;
#pragma unroll
    for (int i = 0; i < h; ++i) {
      const double send = up ? v[i] : v[i + h];
      const double keep = up ? v[i + h] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, h);
    }
  }
  return v[0];
}

// deterministic block reduction of kNumSums doubles (fixed shuffle tree, fixed warp order)
template <int NT>
__device__ __forceinline__ void block_reduce_sums(double* acc, double (*sm)[kNumSums], double* out) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double v32[32];
#pragma unroll
  for (int k = 0; k < 32; ++k) v32[k] = k < kNumSums ? acc[k] : 0.0;
  const double tot = warp_transpose_reduce32(v32, lane);
  if (lane < kNumSums) sm[w][lane] = tot;
  __syncthreads();
  if (threadIdx.x < kNumSums) {
    double v = 0.0;
    for (int ww = 0; ww < NT / 32; ++ww) v += sm[ww][threadIdx.x];
    out[threadIdx.x] = v;
  }
}

}  // namespace dev
}  // namespace smb

#endif  // SM_B200_ICP_DEV_CUH_
