// libnabo-compatible 1-NN (KDTREE_LINEAR_HEAP, k = 1, allowSelfMatch, maxRadius = inf;
// call site registrators/icp_fast.cc:177-178) over the compact tree layout (KdCompact), with
// the node arrays resident in SHARED MEMORY.
//
// H100 formulation
//   * nodes are {cut f64}[h] + {dim u8}[h] in heap order.  Every CTA stages the TOP levels
//     (kKnnSmemLevels = 11: 2047 nodes, 18 KB — the part of the tree every query walks) into
//     shared memory with bulk async copies (cp.async.bulk.shared::cluster.global + mbarrier
//     complete_tx; SASS UBLKCP / SYNCS) while its threads fetch and transform their queries;
//     the deeper levels are read through the read-only path (L1).  Staging all 14 inner levels
//     of a ~107 k-point target (144 KB) would fit the 227 KB a block may use, but leaves one
//     CTA per SM and no room for the kernels of other alignments in flight;
//   * leaves carry no payload: a leaf's bucket is (in-level index << (levels - level)) in the
//     padded bucket array, one bucket = x[8] y[8] z[8] = 12 aligned 16-byte loads;
//   * no stack, and no local memory for the search state: the heap index of the reached leaf encodes the whole path, and
//     the pending far sides of a query are siblings of that path's nodes, at most one per level, so
//     the search state is the leaf plus a `pending` and a `turns` bit per level, in registers.  The
//     rd / off[] of a popped far child are replayed exactly over the turns above it (knn_pop).
// The visit ORDER and every comparison are those of libnabo's recurseKnn, so index sets and
// squared distances are bit-identical to the oracle for any epsilon (tests/test_gpu_icp.py).
#ifndef SM_B200_KNN_SMEM_CUH_
#define SM_B200_KNN_SMEM_CUH_

#include "common.cuh"
#include "kernels.h"

namespace smb {
namespace dev {

#ifndef SMB_KNN_THREADS
#define SMB_KNN_THREADS 256
#endif
#ifndef SMB_KNN_SMEM_LEVELS
#define SMB_KNN_SMEM_LEVELS 11
#endif
#ifndef SMB_KNN_HALF_SCAN
#define SMB_KNN_HALF_SCAN 1
#endif
#ifndef SMB_KNN_Q_FROM_SMEM
#define SMB_KNN_Q_FROM_SMEM 0
#endif
#if SMB_KNN_Q_FROM_SMEM      // the query of a bucket scan re-read from its shared-memory column (frees six registers)
#define SMB_KNN_Q(t, reg, d) ((t).sq[(d) * kKnnCtaThreads])
#else
#define SMB_KNN_Q(t, reg, d) (reg)
#endif
constexpr int kKnnCtaThreads = SMB_KNN_THREADS;        // threads (= traversal slots) per CTA
constexpr int kKnnSmemLevels = SMB_KNN_SMEM_LEVELS;    // tree levels staged in shared memory: 2^11 * 9 B = 18 KB
constexpr int kKnnCtasPerSm = 1024 / kKnnCtaThreads;   // 64 registers per thread -> 1024 threads per SM

struct SmemTree {
  const double* s_cut;      // shared memory
  const uint8_t* s_dim;     // shared memory
  int n_smem;               // heap indices < n_smem are resident in shared memory
  const double* g_cut;      // global (all nodes)
  const uint8_t* g_dim;
  const double2* g_node;    // global, packed {cut, dim} of heap node h at slot h + 1 (one 16-byte load per node)
  const double* pb;         // padded buckets
  int levels;
  double* sq;               // this thread's query: sq[d * kKnnCtaThreads] (shared memory, d = 0..2), and
                            // its off[] of the recursion right behind it: sq[(3 + d) * kKnnCtaThreads]
};

// ---- mbarrier + bulk async copy (TMA engine, non-tensor form) --------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst_smem)), "l"(__cvta_generic_to_global(src_gmem)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
  } while (!ok);
}

// shared-memory footprint of the staged tree: cut[slots] + dim[slots] + barrier + 16 doubles
__host__ __device__ __forceinline__ int knn_smem_slots(int levels) {
  const int ls = levels < kKnnSmemLevels ? levels : kKnnSmemLevels;
  const int n = 1 << ls;
  return n < 16 ? 16 : n;
}
__host__ __device__ __forceinline__ size_t knn_smem_bytes(int levels) {
  // nodes, barrier (+pad), 16 doubles, per-thread query / offset columns
  return (size_t)knn_smem_slots(levels) * 9 + 16 + 16 * sizeof(double) + 6 * (size_t)kKnnCtaThreads * sizeof(double);
}

// Called by ALL threads of the CTA (contains __syncthreads).  Thread 0 arms the barrier and
// issues the copies; everyone may then do independent work and must call mbar_wait(bar, 0)
// before the first tree access.
__device__ __forceinline__ SmemTree stage_tree(const KdCompact& t, unsigned char* smem, uint64_t** bar_out,
                                               double** extra_out) {
  const int slots = knn_smem_slots(t.levels);
  double* s_cut = reinterpret_cast<double*>(smem);
  uint8_t* s_dim = smem + (size_t)slots * 8;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + (size_t)slots * 9);
  *extra_out = reinterpret_cast<double*>(bar + 2);
  if (threadIdx.x == 0) { mbar_init(bar, 1); fence_proxy_async_smem(); }
  __syncthreads();
  if (threadIdx.x == 0) {
    const uint32_t cut_bytes = (uint32_t)slots * 8u, dim_bytes = (uint32_t)slots;
    mbar_arrive_expect_tx(bar, cut_bytes + dim_bytes);
    constexpr uint32_t kChunk = 32768u;
    for (uint32_t off = 0; off < cut_bytes; off += kChunk)
      bulk_copy_g2s(smem + off, reinterpret_cast<const unsigned char*>(t.cut) + off,
                    cut_bytes - off < kChunk ? cut_bytes - off : kChunk, bar);
    bulk_copy_g2s(s_dim, t.dim, dim_bytes, bar);
  }
  *bar_out = bar;
  SmemTree st;
  st.s_cut = s_cut; st.s_dim = s_dim; st.n_smem = slots;
  st.g_cut = t.cut; st.g_dim = t.dim; st.g_node = t.node; st.pb = t.pb; st.levels = t.levels;
  st.sq = *extra_out + 16 + threadIdx.x;
  return st;
}

template <bool kAllSmem>
__device__ __forceinline__ void tree_node(const SmemTree& t, int h, double& cut, int& dim) {
  if (kAllSmem || h < t.n_smem) { cut = t.s_cut[h]; dim = t.s_dim[h]; }
  else { cut = __ldg(t.g_cut + h); dim = __ldg(t.g_dim + h); }
}

__device__ __forceinline__ double2 ldg_nc_f64x2(const void* p) {
  double2 v;
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "l"(p));
  return v;
}

// A node of the levels below the staged ones: cut and dimension in ONE 16-byte load (two dependent
// loads of two arrays before).
__device__ __forceinline__ void ldg_node(const double2* __restrict__ g_node, int h, double& cut, int& dim) {
  const double2 v = ldg_nc_f64x2(g_node + h + 1);
  cut = v.x;
  dim = (int)__double_as_longlong(v.y);
}

// 32 bytes as two 16-byte loads (sm_90 has no 256-bit load), issued back to back
struct Double4 { double a, b, c, d; };
__device__ __forceinline__ Double4 ldg_nc_f64x4(const void* p) {
  const double2 lo = ldg_nc_f64x2(p), hi = ldg_nc_f64x2(reinterpret_cast<const char*>(p) + 16);
  return {lo.x, lo.y, hi.x, hi.y};
}

// One padded bucket: 12 16-byte loads, 8 squared distances in the reference's operation order, then
// a tournament on the bit patterns in which the lower index wins ties (libnabo walks the bucket in
// order and replaces the head on a strict '<').  Padding entries are +inf: their distance is +inf
// or NaN, never below the head.  SMB_KNN_HALF_SCAN: four points at a time (half the registers).
__device__ __forceinline__ unsigned long long dist_key(double qx, double qy, double qz, double x, double y, double z) {
  const double dx = dsub(qx, x), dy = dsub(qy, y), dz = dsub(qz, z);
  return (unsigned long long)__double_as_longlong(dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz)));
}

__device__ __forceinline__ void scan_bucket(const double* __restrict__ pb, int bucket, double qx, double qy,
                                            double qz, double& head, int& best) {
  const char* base = reinterpret_cast<const char*>(pb + (int64_t)bucket * 24);
#if SMB_KNN_HALF_SCAN
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const Double4 vx = ldg_nc_f64x4(base + 32 * half), vy = ldg_nc_f64x4(base + 64 + 32 * half),
                  vz = ldg_nc_f64x4(base + 128 + 32 * half);
    unsigned long long k0 = dist_key(qx, qy, qz, vx.a, vy.a, vz.a), k1 = dist_key(qx, qy, qz, vx.b, vy.b, vz.b);
    unsigned long long k2 = dist_key(qx, qy, qz, vx.c, vy.c, vz.c), k3 = dist_key(qx, qy, qz, vx.d, vy.d, vz.d);
    int a0 = 0, a2 = 2;
    if (k1 < k0) { k0 = k1; a0 = 1; }
    if (k3 < k2) { k2 = k3; a2 = 3; }
    if (k2 < k0) { k0 = k2; a0 = a2; }
    if (k0 < (unsigned long long)__double_as_longlong(head)) {
      head = __longlong_as_double((long long)k0);
      best = bucket * 8 + 4 * half + a0;
    }
  }
#else
  unsigned long long key[8];
  double2 v[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) v[k] = ldg_nc_f64x2(base + 16 * k);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const double x = (k & 1) ? v[k >> 1].y : v[k >> 1].x;
    const double y = (k & 1) ? v[4 + (k >> 1)].y : v[4 + (k >> 1)].x;
    const double z = (k & 1) ? v[8 + (k >> 1)].y : v[8 + (k >> 1)].x;
    key[k] = dist_key(qx, qy, qz, x, y, z);
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
    best = bucket * 8 + arg[0];
  }
#endif
}

// Far-side state of a query, with no stack.  Pushes during a descent come in increasing level order and a
// pop takes the deepest pending entry, so everything still pending after a pop at level j lies above j and
// the next descent pushes only below it: at most one pending far child per level, the sibling of the current
// path's node one level down.  The whole state is therefore the current leaf (hp1 = heap index + 1, ll = its
// level: hp1 >> (ll - a) is the path node of level a, plus one), a `pending` bit per level and a `turns` bit
// per level (the path went to the FAR child there).  rd and off[] change only at turns, so those of a popped
// far child are replayed exactly over the turns above it (knn_pop).  Bit a of a mask = path level a.
constexpr int kKnnMaxLevels = 24;        // sm_api rejects deeper trees (the masks have one bit per level)

// A path node: from the staged levels in shared memory when it is one of them, else one packed record (L1).
__device__ __forceinline__ void path_node(const SmemTree& t, int n, double& cut, int& dim) {
  if (n < t.n_smem) { cut = t.s_cut[n]; dim = t.s_dim[n]; }
  else ldg_node(t.g_node, n, cut, dim);
}

// The coordinate of the query / the recursion's off[] along a node's cut dimension are read from
// per-thread shared-memory columns indexed by that dimension (one LDS instead of a three-way select
// on register pairs: the descent loop of a far visit shrank from 69 to ~30 SASS instructions a level).
//
// Pop: the deepest pending level j, and the rd / off[] the recursion had for its far child, replayed from
// rd = 0, off = 0 over the turn levels above j and then j itself with the recursion's own operations
// (rd += -old_off^2 + new_off^2, off[cd] = new_off), so rd is bit-identical to what the recursion computed
// when it pushed that child; re-tested with the head of this moment, which is when the recursion tests it.
// On success h is the far child, rd its rd, its off[] in t.sq, and the path turns at j.  false: nothing left.
__device__ __forceinline__ bool knn_pop(const SmemTree& t, double me2, double head, int hp1, int ll,
                                        uint32_t& pending, uint32_t& turns, int& h, double& rd) {
  while (pending != 0u) {
    const int j = 31 - __clz(pending);
    pending &= ~(1u << j);
    const uint32_t upto = (turns & ((1u << j) - 1u)) | (1u << j);
    t.sq[3 * kKnnCtaThreads] = 0.0; t.sq[4 * kKnnCtaThreads] = 0.0; t.sq[5 * kKnnCtaThreads] = 0.0;
    double r = 0.0;
    uint32_t steps = upto;
    do {
      const int a = __ffs(steps) - 1;
      steps &= steps - 1u;
      double cut; int cd;
      path_node(t, (hp1 >> (ll - a)) - 1, cut, cd);
      const double old_off = t.sq[(3 + cd) * kKnnCtaThreads];
      const double new_off = dsub(t.sq[cd * kKnnCtaThreads], cut);
      r = dadd(r, dadd(-dmul(old_off, old_off), dmul(new_off, new_off)));
      t.sq[(3 + cd) * kKnnCtaThreads] = new_off;
    } while (steps != 0u);
    if (dmul(r, me2) < head) {
      h = ((hp1 >> (ll - j - 1)) ^ 1) - 1;             // sibling of the path node of level j + 1
      rd = r;
      turns = upto;
      return true;
    }
  }
  return false;
}

// recurseKnn's descent from heap node h (rd at entry, off[] in its t.sq column): near child first down to a leaf; a far
// child that passes rd_new*(1+eps)^2 < head now (the head only shrinks) sets the pending bit of its parent's
// level.  Far subtrees start deep in the tree: nodes come through the read-only path (L1).  Leaves the new
// path in hp1 / ll and returns the leaf's bucket.
__device__ __forceinline__ int knn_descend(const SmemTree& t, double me2, double head, int h, double rd,
                                           uint32_t& pending, int& hp1, int& ll) {
  int l = 31 - __clz(h + 1);
  while (l < t.levels) {
    double cut; int cd;
    ldg_node(t.g_node, h, cut, cd);
    if (cd == 3) break;
    const double q = t.sq[cd * kKnnCtaThreads];
    const double old_off = t.sq[(3 + cd) * kKnnCtaThreads];
    const double new_off = dsub(q, cut);
    const double rd_new = dadd(rd, dadd(-dmul(old_off, old_off), dmul(new_off, new_off)));
    const int right = q > cut ? 1 : 0;              // == (q - cut > 0) for IEEE doubles
    if (dmul(rd_new, me2) < head) pending |= 1u << l;
    h = 2 * h + 1 + right;
    ++l;
  }
  hp1 = h + 1; ll = l;
  return (h + 1 - (1 << l)) << (t.levels - l);
}

// The descent of a query from the root to its leaf (heap index h, level l): the staged levels from shared
// memory, the rest one packed record per level.  Leaves the query in its t.sq column.
template <bool kAllSmem>
__device__ __forceinline__ void knn_root_descent(const SmemTree& t, double qx, double qy, double qz, int& h_out,
                                                 int& l_out) {
  t.sq[0] = qx; t.sq[kKnnCtaThreads] = qy; t.sq[2 * kKnnCtaThreads] = qz;
  const int lsm = kAllSmem ? t.levels : min(t.levels, kKnnSmemLevels);    // levels staged in shared memory
  int h = 0, l = 0;
  bool leaf = false;
  while (l < lsm) {
    const int cd = t.s_dim[h];
    if (cd == 3) { leaf = true; break; }
    h = 2 * h + 1 + (t.sq[cd * kKnnCtaThreads] > t.s_cut[h] ? 1 : 0);
    ++l;
  }
  if (!kAllSmem && !leaf) {
    while (l < t.levels) {
      double cut; int cd;
      ldg_node(t.g_node, h, cut, cd);
      if (cd == 3) break;
      h = 2 * h + 1 + (t.sq[cd * kKnnCtaThreads] > cut ? 1 : 0);
      ++l;
    }
  }
  h_out = h; l_out = l;
}

// First visit of a query: the root descent, the first bucket, and the mask of the path levels whose far
// side passes with the head that bucket left, each tested exactly (node re-read: shared memory or L1).
// rd = 0 and off = 0 along the whole root path, so rd_new(a) = 0 + (-(0*0) + off^2) = off^2 exactly, and
// the pop re-tests every level of the mask with the head of its moment.
template <bool kAllSmem>
__device__ __forceinline__ void knn_root_visit(const SmemTree& t, double qx, double qy, double qz, double me2,
                                               double& head, int& best, int& hp1_out, int& ll_out, uint32_t& mask_out) {
  head = __longlong_as_double(0x7ff0000000000000ll);
  best = -1;
  int h, l;
  knn_root_descent<kAllSmem>(t, qx, qy, qz, h, l);
  scan_bucket(t.pb, (h + 1 - (1 << l)) << (t.levels - l), qx, qy, qz, head, best);
  const int hp1 = h + 1, ll = l;
  uint32_t mask = 0u;
  for (int a = 0; a < ll; ++a) {
    double cut; int cd;
    path_node(t, (hp1 >> (ll - a)) - 1, cut, cd);
    const double off = dsub(t.sq[cd * kKnnCtaThreads], cut);
    if (dmul(dmul(off, off), me2) < head) mask |= 1u << a;
  }
  hp1_out = hp1; ll_out = ll; mask_out = mask;
}

// best: padded entry index (bucket * 8 + k) or -1; d2: squared distance (+inf if none)
template <bool kAllSmem>
__device__ __forceinline__ void knn1_smem(const SmemTree& t, double qx, double qy, double qz, double me2,
                                          int& best_out, double& d2_out) {
  double head, rd; int best, hp1, ll, h; uint32_t pending, turns = 0u;
  knn_root_visit<kAllSmem>(t, qx, qy, qz, me2, head, best, hp1, ll, pending);
  while (knn_pop(t, me2, head, hp1, ll, pending, turns, h, rd)) {
    const int bucket = knn_descend(t, me2, head, h, rd, pending, hp1, ll);
    scan_bucket(t.pb, bucket, SMB_KNN_Q(t, qx, 0), SMB_KNN_Q(t, qy, 1), SMB_KNN_Q(t, qz, 2), head, best);
  }
  best_out = best;
  d2_out = head;
}

// One CTA's range [begin, end), one query per thread (consecutive threads = consecutive queries).  The first
// query is loaded while the tree top is being staged, each next one right after the previous result is stored.
// load_q(i, x, y, z), store(i, best, d2).
template <bool kAllSmem, typename LoadQ, typename Store>
__device__ __forceinline__ void knn1_cta(const SmemTree& tree, uint64_t* bar, int begin, int end, double me2,
                                         LoadQ load_q, Store store) {
  int i = begin + threadIdx.x;
  double3 q = make_double3(0.0, 0.0, 0.0);
  if (i < end) load_q(i, q.x, q.y, q.z);
  mbar_wait(bar, 0);      // every thread waits: the CTA must not retire while the copy engine writes its smem
  while (i < end) {
    int slot; double d2;
    knn1_smem<kAllSmem>(tree, q.x, q.y, q.z, me2, slot, d2);
    store(i, slot, d2);
    i += kKnnCtaThreads;
    if (i < end) load_q(i, q.x, q.y, q.z);
  }
}

// ---- far visits of a batch of queries, one WARP working through a list ---------------------------
// A query whose root visit left far-side candidates (knn_root_visit's mask != 0) is parked as a
// KnnItem (its leaf and mask; a parked query has no turns); the lanes of the warp then pull items from
// the list.  Every pass of the loop below is ONE bucket visit per busy lane — the next subtree of the
// lane's query (knn_pop, as knn1_smem pops it), the descent into it, the bucket — and a lane whose query
// is finished takes the next item in the same pass.  The per-query visit order is the recursion's; only
// WHICH lane runs a query and when is different, so results are bit-identical.  Static one-query-per-lane
// scheduling leaves 13 of 32 lanes busy (the visit count per query is 1..29, mean 2.9); here the bucket
// scans and descents of a pass run with most lanes busy.
struct KnnItem { int i, hp1, ll; uint32_t mask; };      // 16 bytes

template <typename LoadQuery, typename StoreResult>
__device__ __forceinline__ void knn_far_phase(const SmemTree& t, double me2, const int4* __restrict__ items,
                                              int n_items, LoadQuery load_query, StoreResult store_result) {
  const unsigned lt = (1u << (threadIdx.x & 31)) - 1u;
  int next = 0;
  int qi = -1, hp1 = 1, ll = 0, best = -1;            // qi < 0: the lane has no query
  uint32_t pending = 0u, turns = 0u;
  double head = 0.0;
  while (true) {
    const unsigned need = __ballot_sync(0xffffffffu, qi < 0);
    if (qi < 0) {
      const int idx = next + __popc(need & lt);
      if (idx < n_items) {
        const int4 it = __ldcg(items + idx);
        qi = it.x; hp1 = it.y; ll = it.z; pending = (uint32_t)it.w; turns = 0u;
        double qx, qy, qz;
        load_query(qi, qx, qy, qz, head, best);
        t.sq[0] = qx; t.sq[kKnnCtaThreads] = qy; t.sq[2 * kKnnCtaThreads] = qz;
      }
    }
    next += __popc(need);
    if (!__any_sync(0xffffffffu, qi >= 0)) break;
    bool go = false;
    int h = 0;
    double rd = 0.0;
    if (qi >= 0) {
      go = knn_pop(t, me2, head, hp1, ll, pending, turns, h, rd);
      if (!go) { store_result(qi, best, head); qi = -1; }
    }
    if (go) {
      const int bucket = knn_descend(t, me2, head, h, rd, pending, hp1, ll);
      // the query from its shared-memory column: six registers fewer across the loop, no spills
      scan_bucket(t.pb, bucket, t.sq[0], t.sq[kKnnCtaThreads], t.sq[2 * kKnnCtaThreads], head, best);
    }
  }
}

// One CTA's range [begin, end) in batches of 256 * qpt queries (per_cta is a multiple of the CTA size):
//   (1) every thread loads its queries (one per pass, consecutive threads = consecutive queries) and does
//       their root visits in lockstep with its warp.  A query without far-side candidates is final here;
//   (2) the others are parked (park: head and best of the moment; a 16-byte item in the warp's slice of
//       items_all, which lies inside the batch's own index range) and the warp works through its list
//       (knn_far_phase).
// load_q(i, x, y, z), park(i, best, head), unpark(i, head&, best&), finish(i, best, head).
constexpr int kKnnMaxQpt = 4;
template <bool kAllSmem, typename LoadQ, typename Park, typename Unpark, typename Finish>
__device__ __forceinline__ void knn_batch_cta(const SmemTree& tree, int begin, int end, int per_cta, double me2,
                                              int4* __restrict__ items_all, LoadQ load_q, Park park,
                                              Unpark unpark, Finish finish) {
  const int warp = threadIdx.x >> 5;
  const unsigned lt = (1u << (threadIdx.x & 31)) - 1u;
  // qb: the batch's queries per thread, min(qpt, what is left of the range) with qpt = min(kKnnMaxQpt,
  // per_cta / 256); what is left never exceeds per_cta / 256, so qpt itself need not be held across the far phase
  for (int base = begin, qb; base < end; base += kKnnCtaThreads * qb) {
    qb = min(kKnnMaxQpt, (begin + per_cta - base) / kKnnCtaThreads);
    int4* items = items_all + base + warp * 32 * qb;
    int count = 0;
    for (int j = 0; j < qb; ++j) {
      const int i = base + j * kKnnCtaThreads + threadIdx.x;
      bool far = false;
      int4 item = make_int4(0, 0, 0, 0);
      if (i < end) {
        double px, py, pz, head;
        int best, hp1, ll;
        uint32_t mask;
        load_q(i, px, py, pz);
        knn_root_visit<kAllSmem>(tree, px, py, pz, me2, head, best, hp1, ll, mask);
        if (mask == 0u) {
          finish(i, best, head);
        } else {
          park(i, best, head);
          far = true;
          item = make_int4(i, hp1, ll, (int)mask);
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, far);
      if (far) items[count + __popc(m & lt)] = item;
      count += __popc(m);
    }
    __syncwarp();
    knn_far_phase(tree, me2, items, count,
                  [&](int i, double& qx, double& qy, double& qz, double& head, int& best) {
                    load_q(i, qx, qy, qz);
                    unpark(i, head, best);
                  },
                  finish);
    __syncwarp();
  }
}

}  // namespace dev
}  // namespace smb

#endif  // SM_B200_KNN_SMEM_CUH_
