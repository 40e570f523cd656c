// libnabo's k-nearest-neighbour search on the device: NNS::knn(query, indices, dists2, k, epsilon, optionFlags,
// maxRadius) of KDTREE_LINEAR_HEAP for k = 1..64, over the tree sm_knn1 builds (KdCompactTree with the ids payload).
//
// The search is the 1-NN kernel's (knn_smem.cuh): the root descent through the staged tree top, the path levels whose
// far side may still hold a neighbour kept as a `pending` bit per level, and knn_pop / knn_descend for the far visits,
// all unchanged.  What k > 1, the radius and self-match exclusion change:
//   * the head is the k-th entry of a sorted list of k (id, d2) pairs, initialised to (-1, +inf).  A point of a
//     bucket enters iff d2 <= maxRadius^2, d2 < head and (ALLOW_SELF_MATCH or d2 > DBL_EPSILON); it goes after every
//     entry of equal distance and the k-th entry drops out (libnabo's IndexHeapBruteForceVector::replaceHead).  The
//     bucket is walked in its order, so among equal distances the earlier-visited point comes first;
//   * a far side is visited iff rd <= maxRadius^2 and rd * (1 + eps)^2 < head, tested when libnabo tests it: after
//     the near side has finished.  knn_descend marks a far side pending only if rd * (1 + eps)^2 < head holds when it
//     is passed (the head only shrinks, so one that fails then fails later too) and knn_pop re-tests it with the head
//     of the moment; the radius test does not depend on the head, so it is made on the popped rd, and a far side that
//     fails it is dropped before its descent.  The root path's mask applies both tests to rd = off^2.
// The list lives in registers for k <= 8 (K = 4 or 8: fully unrolled insertion, no dynamic index, so no local memory)
// and in shared memory for 9 <= k <= 64 (K = 0: one column of k doubles and k ints per thread, [entry][thread], so a
// warp's accesses fall in distinct banks whatever entry each lane touches).
#include "common.cuh"
#include "kernels.h"
#include "knn_smem.cuh"
#include "statistic_removal.cuh"

namespace smb {
using namespace dev;
namespace {

constexpr double kInfD = __builtin_huge_val();
constexpr double kDblEpsilon = 2.220446049250313080847e-16;   // std::numeric_limits<double>::epsilon()
constexpr int kKnnMaxK = 64;

// sorted (d2, padded entry) list of k <= K entries in registers.  The list is d[K - k .. K - 1]; the K - k entries in
// front of it hold -inf, which no insertion moves (every accepted distance is >= 0), so the head is d[K - 1] and every
// index is a compile-time constant
template <int K>
struct RegList {
  double d[K];
  int e[K];
  __device__ __forceinline__ void init(int k) {
#pragma unroll
    for (int j = 0; j < K; ++j) { d[j] = j < K - k ? -kInfD : kInfD; e[j] = -1; }
  }
  // v < d[K - 1]: v goes after the entries <= v, the ones after it move down one, d[K - 1] drops out; returns the head
  __device__ __forceinline__ double insert(double v, int entry, int) {
#pragma unroll
    for (int j = K - 1; j >= 0; --j) {
      const double prev = d[j > 0 ? j - 1 : 0];
      if (!(d[j] <= v)) {
        const bool here = j == 0 || prev <= v;
        e[j] = here ? entry : e[j > 0 ? j - 1 : 0];
        d[j] = here ? v : prev;
      }
    }
    return d[K - 1];
  }
  __device__ __forceinline__ void store(const int32_t* __restrict__ pid, int k, int32_t* ids, double* d2) const {
#pragma unroll
    for (int j = 0; j < K; ++j)
      if (j >= K - k) { ids[j - (K - k)] = e[j] >= 0 ? pid[e[j]] : -1; d2[j - (K - k)] = d[j]; }
  }
  // f(j, entry) for the list's entries j = 0 .. k - 1 in order
  template <class F>
  __device__ __forceinline__ void for_each(int k, F f) const {
#pragma unroll
    for (int j = 0; j < K; ++j)
      if (j >= K - k) f(j - (K - k), e[j]);
  }
};

// the same list in this thread's shared-memory columns: entry j at d[j * kKnnCtaThreads]
struct SmemList {
  double* d;
  int* e;
  __device__ __forceinline__ void init(int k) {
    for (int j = 0; j < k; ++j) { d[j * kKnnCtaThreads] = kInfD; e[j * kKnnCtaThreads] = -1; }
  }
  __device__ __forceinline__ double insert(double v, int entry, int k) {
    int j = k - 1;
    while (j > 0) {
      const double prev = d[(j - 1) * kKnnCtaThreads];
      if (prev <= v) break;
      d[j * kKnnCtaThreads] = prev;
      e[j * kKnnCtaThreads] = e[(j - 1) * kKnnCtaThreads];
      --j;
    }
    d[j * kKnnCtaThreads] = v;
    e[j * kKnnCtaThreads] = entry;
    return d[(k - 1) * kKnnCtaThreads];
  }
  __device__ __forceinline__ void store(const int32_t* __restrict__ pid, int k, int32_t* ids, double* d2) const {
    for (int j = 0; j < k; ++j) {
      const int en = e[j * kKnnCtaThreads];
      ids[j] = en >= 0 ? pid[en] : -1;
      d2[j] = d[j * kKnnCtaThreads];
    }
  }
  template <class F>
  __device__ __forceinline__ void for_each(int k, F f) const {
    for (int j = 0; j < k; ++j) f(j, e[j * kKnnCtaThreads]);
  }
};

struct KnnKParams {
  int k;
  int allow_self;
  double me2;     // (1 + eps)^2
  double r2;      // maxRadius^2
};

// One padded bucket in its order: 12 16-byte loads, the squared distance of each entry in the reference's operation
// order, then libnabo's acceptance test against the head of that moment.  Padding entries are +inf: their distance is
// +inf or NaN and never passes d2 < head.
template <class List>
__device__ __forceinline__ void scan_bucket_k(const double* __restrict__ pb, int bucket, double qx, double qy,
                                              double qz, const KnnKParams& p, List& list, double& head) {
  const char* base = reinterpret_cast<const char*>(pb + (int64_t)bucket * 24);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const Double4 vx = ldg_nc_f64x4(base + 32 * half), vy = ldg_nc_f64x4(base + 64 + 32 * half),
                  vz = ldg_nc_f64x4(base + 128 + 32 * half);
    const double x[4] = {vx.a, vx.b, vx.c, vx.d}, y[4] = {vy.a, vy.b, vy.c, vy.d}, z[4] = {vz.a, vz.b, vz.c, vz.d};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const double dx = dsub(qx, x[c]), dy = dsub(qy, y[c]), dz = dsub(qz, z[c]);
      const double dist = dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz));
      if (dist <= p.r2 && dist < head && (p.allow_self || dist > kDblEpsilon))
        head = list.insert(dist, bucket * 8 + 4 * half + c, p.k);
    }
  }
}

// recurseKnn for one query: the root visit (knn_root_visit's, with the k-entry list and both far-side tests), then the
// far visits deepest pending level first
template <bool kAllSmem, class List>
__device__ __forceinline__ void knn_k_search(const SmemTree& t, double qx, double qy, double qz, const KnnKParams& p,
                                             List& list) {
  double head = kInfD;
  int h, l;
  knn_root_descent<kAllSmem>(t, qx, qy, qz, h, l);
  scan_bucket_k(t.pb, (h + 1 - (1 << l)) << (t.levels - l), qx, qy, qz, p, list, head);
  int hp1 = h + 1, ll = l;
  uint32_t pending = 0u, turns = 0u;
  for (int a = 0; a < ll; ++a) {
    double cut; int cd;
    path_node(t, (hp1 >> (ll - a)) - 1, cut, cd);
    const double off = dsub(t.sq[cd * kKnnCtaThreads], cut);
    const double rd = dmul(off, off);
    if (rd <= p.r2 && dmul(rd, p.me2) < head) pending |= 1u << a;
  }
  double rd;
  while (knn_pop(t, p.me2, head, hp1, ll, pending, turns, h, rd)) {
    // a far side outside the radius is dropped: every level still pending lies above the popped one, so their pops
    // replay only the turns above them and the turn just recorded is never used
    if (!(rd <= p.r2)) continue;
    const int bucket = knn_descend(t, p.me2, head, h, rd, pending, hp1, ll);
    scan_bucket_k(t.pb, bucket, qx, qy, qz, p, list, head);
  }
}

// What a query keeps of its finished list.  at(kc, p, i, qx, qy, qz) is called before the search and returns the
// function the finished list is handed to.  KnnRows forms the row's address there, ahead of the search: formed after
// it, ptxas schedules the shared-memory list's search differently.  The returned functions capture copies, not `this`:
// capturing `this` costs the register-list mean-distance kernels 20 to 22 registers.
// KnnRows: the query's k-row, original ids (-1: no entry) and squared distances.
struct KnnRows {
  static constexpr int kMinCtasPerSm = 0;      // no minimum
  int32_t* ids;
  double* d2;
  __device__ __forceinline__ auto at(const KdCompact& kc, const KnnKParams& p, int i, double, double, double) const {
    int32_t* out_ids = ids + (int64_t)i * p.k;
    double* out_d2 = d2 + (int64_t)i * p.k;
    return [&kc, &p, out_ids, out_d2](const auto& list) { list.store(kc.pid, p.k, out_ids, out_d2); };
  }
};

// KnnMeanDistance: StatisticalOutlierRemoval's per-point mean distance (statistic_removal.cuh), for k = K + 1 (eps = 0,
// self-match allowed, no radius): instead of the k-row it reads each list entry's point back from the padded bucket the
// entry names and writes one float per query, at dist[qindex[i]].  Entry 0 (d2 = 0: the query or a duplicate of it) is
// dropped.  The minimum of one CTA per SM leaves ptxas room for the shared-memory list variant's epilogue without a
// spill (it holds two CTAs per SM at K = 30 by its shared memory anyway).
struct KnnMeanDistance {
  static constexpr int kMinCtasPerSm = 1;
  const uint32_t* qindex;
  float* dist;
  __device__ __forceinline__ auto at(const KdCompact& kc, const KnnKParams& p, int i, double qx, double qy,
                                     double qz) const {
    return [&kc, &p, i, qx, qy, qz, qindex = qindex, dist = dist](const auto& list) {
      const float fx = (float)qx, fy = (float)qy, fz = (float)qz;   // exact: the coordinates are widened floats
      double sum = 0.0;
      list.for_each(p.k, [&](int j, int en) {
        if (j == 0 || en < 0) return;            // en < 0 is not reached: the tree holds more than K points
        const double* b = kc.pb + (int64_t)(en >> 3) * 24 + (en & 7);
        sum = sr_dadd(sum, sr_neighbour_term(fx, fy, fz, (float)__ldg(b), (float)__ldg(b + 8), (float)__ldg(b + 16)));
      });
      dist[qindex[i]] = sr_mean_distance(sum, p.k - 1);
    };
  }
};

// one query per thread; K = 4 / 8: the list in registers (k <= K), K = 0: in shared memory behind the staged tree
template <int K, bool kAllSmem, class Epilogue>
__global__ void __launch_bounds__(kKnnCtaThreads, Epilogue::kMinCtasPerSm)
knn_k_kernel(KdCompact kc, const double* __restrict__ query, int64_t qstride, int nq, KnnKParams p,
             Epilogue epilogue) {
  extern __shared__ __align__(128) unsigned char knn_smem[];
  uint64_t* bar; double* extra;
  const SmemTree tree = stage_tree(kc, knn_smem, &bar, &extra);
  const int i = blockIdx.x * kKnnCtaThreads + threadIdx.x;
  const double qx = i < nq ? query[i] : 0.0, qy = i < nq ? query[qstride + i] : 0.0,
               qz = i < nq ? query[2 * qstride + i] : 0.0;
  mbar_wait(bar, 0);
  if (i >= nq) return;
  const auto finish = epilogue.at(kc, p, i, qx, qy, qz);
  const auto search = [&](auto& list) {
    list.init(p.k);
    knn_k_search<kAllSmem>(tree, qx, qy, qz, p, list);
    finish(list);
  };
  if constexpr (K > 0) {
    RegList<K> list;
    search(list);
  } else {
    const size_t at = (knn_smem_bytes(kc.levels) + 15) & ~(size_t)15;
    SmemList list{reinterpret_cast<double*>(knn_smem + at) + threadIdx.x,
                  reinterpret_cast<int*>(knn_smem + at + (size_t)p.k * kKnnCtaThreads * sizeof(double)) + threadIdx.x};
    search(list);
  }
}

size_t knn_k_smem_bytes(int levels, int k) {
  const size_t tree = (knn_smem_bytes(levels) + 15) & ~(size_t)15;
  return k <= 8 ? knn_smem_bytes(levels) : tree + (size_t)k * kKnnCtaThreads * (sizeof(double) + sizeof(int));
}

// the kernel for p.k (list in registers up to k = 8) and the tree's depth (all inner levels staged or not)
template <class Epilogue>
int launch_k(const KdCompact& kc, const double* query, int64_t qstride, int nq, const KnnKParams& p,
             const Epilogue& epilogue, cudaStream_t s) {
  const size_t smem = knn_k_smem_bytes(kc.levels, p.k);
  const auto launch = [&](auto kernel) {
    if (smem > 48 * 1024)
      SMB_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<ceil_div(nq, kKnnCtaThreads), kKnnCtaThreads, smem, s>>>(kc, query, qstride, nq, p, epilogue);
    SMB_CUDA_OK(cudaGetLastError());
    return 0;
  };
  const bool all = kc.levels <= kKnnSmemLevels;
  if (p.k <= 4) return all ? launch(knn_k_kernel<4, true, Epilogue>) : launch(knn_k_kernel<4, false, Epilogue>);
  if (p.k <= 8) return all ? launch(knn_k_kernel<8, true, Epilogue>) : launch(knn_k_kernel<8, false, Epilogue>);
  return all ? launch(knn_k_kernel<0, true, Epilogue>) : launch(knn_k_kernel<0, false, Epilogue>);
}

}  // namespace

int knn_k_query(const KdCompact& kc, const double* query, int64_t qstride, int nq, int k, double max_error2,
                double max_radius2, bool allow_self_match, int32_t* ids, double* d2, cudaStream_t stream) {
  if (nq <= 0) return 0;
  if (k < 1 || k > kKnnMaxK) return -1;
  return launch_k(kc, query, qstride, nq, KnnKParams{k, allow_self_match ? 1 : 0, max_error2, max_radius2},
                  KnnRows{ids, d2}, stream);
}

int knn_mean_distance_query(const KdCompact& kc, const double* query, int64_t qstride, int nq, int mean_k,
                            const uint32_t* qindex, float* dist, cudaStream_t stream) {
  if (nq <= 0) return 0;
  if (mean_k < 1 || mean_k >= kKnnMaxK) return -1;
  return launch_k(kc, query, qstride, nq, KnnKParams{mean_k + 1, 1, 1.0, kInfD}, KnnMeanDistance{qindex, dist}, stream);
}

}  // namespace smb
