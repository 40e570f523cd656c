// ORACLE — TEST INFRASTRUCTURE ONLY.  libnabo 1.0.7 NearestNeighbourSearch<double>::knn with KDTREE_LINEAR_HEAP
// (KDTreeUnbalancedPtInLeavesImplicitBoundsStackOpt with IndexHeapBruteForceVector) for general k, epsilon, maxRadius
// and option flags, on the tree oracle/sm_oracle.cc's Knn1 builds (tie_mode 0), with the same bucket order.  The
// reference calls it with k = 1 (registrators/icp_fast.cc:177-178); libpointmatcher's
// SamplingSurfaceNormalDataPointsFilter asks for knn 7 and KDTreeMatcher for a maxDist
// (registrators/icp_pointmatcher.cc:178,186-189).
//
// The rules below are upstream knowledge: libnabo is not part of the reference tree and is not compiled here, so they
// are restated from its published 1.0.7 sources and cannot be checked against a build of it (as for SURVEY.md
// Appendix C):
//   * heap: a sorted array of k (index, value) entries initialised to (-1, +inf); the head is the k-th entry.  A
//     candidate is accepted iff dist <= maxRadius^2, dist < head (strict) and (ALLOW_SELF_MATCH or
//     dist > numeric_limits<double>::epsilon());
//   * placement (replaceHead): an accepted entry goes after every entry of equal value; the earlier-visited entry comes
//     first among ties and a tie with the k-th entry is rejected;
//   * recursion: near child first, then the far side iff rd <= maxRadius^2 and rd * (1 + eps)^2 < head, with
//     rd += -old_off^2 + new_off^2 and off[cd] = new_off around the far visit;
//   * output: the heap is already sorted ascending, so SORT_RESULTS changes nothing; k x nQ column-major.  Entries never
//     filled stay (-1, +inf).  libnabo's own behaviour for k > n_target is not verified here.
#include <stdint.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

namespace {

constexpr double kInf = std::numeric_limits<double>::infinity();

struct Node {
  int dim;          // 0..2 inner, 3 = leaf
  double cut_val;   // inner
  int right_child;  // inner (left child is pos + 1)
  int bucket_first; // leaf
  int bucket_count; // leaf
};

struct Tree {
  const double* cloud = nullptr;  // 3xN column-major
  int bucket_size = 8;
  std::vector<Node> nodes;
  std::vector<int> buckets;

  // libnabo argMax: first strictly greater, from maxVal = 0
  static int ArgMax3(const double v[3]) {
    double m = 0.0;
    int a = 0;
    for (int i = 0; i < 3; ++i)
      if (v[i] > m) { m = v[i]; a = i; }
    return a;
  }

  int Build(std::vector<int>& idx, int first, int last, const double mn[3], const double mx[3]) {
    const int count = last - first;
    const int pos = (int)nodes.size();
    if (count <= bucket_size) {
      std::sort(idx.begin() + first, idx.begin() + last);          // canonical bucket order: ascending index
      nodes.push_back(Node{3, 0.0, -1, (int)buckets.size(), count});
      for (int i = first; i < last; ++i) buckets.push_back(idx[i]);
      return pos;
    }
    const double ext[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};
    const int cd = ArgMax3(ext);
    const int left_count = count - count / 2;
    const double* c = cloud;
    // nth_element with the total order (coordinate, index): the partition is a unique set
    std::nth_element(idx.begin() + first, idx.begin() + first + left_count, idx.begin() + last, [c, cd](int a, int b) {
      const double ca = c[3 * (size_t)a + cd], cb = c[3 * (size_t)b + cd];
      return ca < cb || (ca == cb && a < b);
    });
    const double cut = cloud[3 * (size_t)idx[first + left_count] + cd];
    nodes.push_back(Node{cd, cut, -1, -1, 0});
    double lmx[3] = {mx[0], mx[1], mx[2]}, rmn[3] = {mn[0], mn[1], mn[2]};
    lmx[cd] = cut;
    rmn[cd] = cut;
    Build(idx, first, first + left_count, mn, lmx);
    const int right = Build(idx, first + left_count, last, rmn, mx);
    nodes[(size_t)pos].right_child = right;
    return pos;
  }

  void Build(const double* pts, int64_t n, int bucket) {
    cloud = pts;
    bucket_size = bucket;
    double mn[3] = {kInf, kInf, kInf}, mx[3] = {-kInf, -kInf, -kInf};
    std::vector<int> idx((size_t)n);
    for (int64_t i = 0; i < n; ++i) {
      idx[(size_t)i] = (int)i;
      for (int r = 0; r < 3; ++r) {
        mn[r] = std::min(mn[r], pts[3 * i + r]);
        mx[r] = std::max(mx[r], pts[3 * i + r]);
      }
    }
    if (n > 0) Build(idx, 0, (int)n, mn, mx);
  }
};

// IndexHeapBruteForceVector: sorted ascending, head = last entry
struct LinearHeap {
  std::vector<int> idx;
  std::vector<double> val;
  explicit LinearHeap(int k) : idx((size_t)k, -1), val((size_t)k, kInf) {}
  double head() const { return val.back(); }
  void replace_head(int index, double value) {
    size_t i = val.size() - 1;
    for (; i > 0; --i) {
      if (val[i - 1] > value) { val[i] = val[i - 1]; idx[i] = idx[i - 1]; }
      else break;
    }
    val[i] = value;
    idx[i] = index;
  }
};

struct Search {
  const Tree& t;
  double max_error2, max_radius2;
  bool allow_self;
  void Recurse(const double* q, int n, double rd, double off[3], LinearHeap& heap) const {
    const Node& node = t.nodes[(size_t)n];
    if (node.dim == 3) {
      for (int i = 0; i < node.bucket_count; ++i) {
        const int index = t.buckets[(size_t)(node.bucket_first + i)];
        const double* p = t.cloud + 3 * (size_t)index;
        double dist = 0.0;
        for (int r = 0; r < 3; ++r) {
          const double diff = q[r] - p[r];
          dist += diff * diff;
        }
        if (dist <= max_radius2 && dist < heap.head() &&
            (allow_self || dist > std::numeric_limits<double>::epsilon()))
          heap.replace_head(index, dist);
      }
      return;
    }
    const int cd = node.dim;
    const double old_off = off[cd];
    const double new_off = q[cd] - node.cut_val;
    const int near = new_off > 0.0 ? node.right_child : n + 1;
    const int far = new_off > 0.0 ? n + 1 : node.right_child;
    Recurse(q, near, rd, off, heap);
    rd += -old_off * old_off + new_off * new_off;
    if (rd <= max_radius2 && rd * max_error2 < heap.head()) {
      off[cd] = new_off;
      Recurse(q, far, rd, off, heap);
      off[cd] = old_off;
    }
  }
};

}  // namespace

extern "C" {

// flags: 1 ALLOW_SELF_MATCH, 2 SORT_RESULTS.  ids / dists2: k x n_query column-major.  Returns 0, or -1 for arguments
// the product rejects too (k outside 1..64, eps < 0 or NaN, radius < 0 or NaN, bucket outside 2..8, unknown flags).
int sm_oracle_knn(const double* target, int64_t n_target, const double* query, int64_t n_query, int32_t k,
                  double epsilon, double max_radius, uint32_t flags, int bucket_size, int32_t* ids, double* dists2) {
  if (n_target < 1 || n_query < 0 || k < 1 || k > 64 || !(epsilon >= 0.0) || !(max_radius >= 0.0) ||
      bucket_size < 2 || bucket_size > 8 || (flags & ~3u) != 0u)
    return -1;
  Tree tree;
  tree.Build(target, n_target, bucket_size);
  const Search s{tree, (1.0 + epsilon) * (1.0 + epsilon), max_radius * max_radius, (flags & 1u) != 0u};
#pragma omp parallel for schedule(guided, 32)
  for (int64_t i = 0; i < n_query; ++i) {
    LinearHeap heap(k);
    double off[3] = {0.0, 0.0, 0.0};
    s.Recurse(query + 3 * i, 0, 0.0, off, heap);
    for (int j = 0; j < k; ++j) {
      ids[i * k + j] = heap.idx[(size_t)j];
      dists2[i * k + j] = heap.val[(size_t)j];
    }
  }
  return 0;
}

}  // extern "C"
