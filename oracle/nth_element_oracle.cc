// CalculateNormals in the order std::nth_element leaves (sm_calculate_normals_ordered with
// SM_NORMALS_ORDER_NTH_ELEMENT), taken from the standard library's own std::nth_element.  TEST INFRASTRUCTURE.
//
//   sm_oracle_nth_element_perm      std::nth_element(idx, idx + nth, idx + n) over iota with a < b on keys[a] < keys[b]
//   sm_oracle_normals_nth_perm      the index array BuildNormals (builder/data/cloud_types.cc:105-144) leaves behind,
//                                   every node split by std::nth_element with CompareDim's comparator (plain '<' on
//                                   the cut-axis coordinate) on the one array the whole recursion permutes
//   sm_oracle_nth_element_adversary keys that drive std::nth_element into its depth limit, found by running it
//                                   against an adversarial comparator in the style of McIlroy's "A Killer Adversary
//                                   for Quicksort" (Software: Practice and Experience 29(4), 1999)
// Nothing here restates the library: every permutation is the one the library call leaves.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <numeric>
#include <vector>

namespace {

struct KeyLess {
  const double* keys;
  bool operator()(int32_t a, int32_t b) const { return keys[a] < keys[b]; }
};

struct AxisLess {           // CompareDim: the cut-axis coordinate, nothing else
  const double* pts;        // 3xN column-major
  int dim;
  bool operator()(int32_t a, int32_t b) const { return pts[3 * (size_t)a + dim] < pts[3 * (size_t)b + dim]; }
};

// cloud_types.cc:41-56: first strictly greater extent wins, from 0
int arg_max3(const double v[3]) {
  double mv = 0.0;
  int mi = 0;
  for (int i = 0; i < 3; ++i)
    if (v[i] > mv) { mv = v[i]; mi = i; }
  return mi;
}

// cloud_types.cc:105-144 without the leaf routine (which reads the permutation, never changes it)
void build(const double* pts, std::vector<int32_t>& idx, int first, int last, const double* mn, const double* mx) {
  const int count = last - first;
  if (count <= 7) return;
  const double ext[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};
  const int dim = arg_max3(ext);
  const int left = count - count / 2;
  std::nth_element(idx.begin() + first, idx.begin() + first + left, idx.begin() + last, AxisLess{pts, dim});
  const double cut = pts[3 * (size_t)idx[first + left] + dim];
  double lmx[3] = {mx[0], mx[1], mx[2]}, rmn[3] = {mn[0], mn[1], mn[2]};
  lmx[dim] = cut;
  rmn[dim] = cut;
  build(pts, idx, first, first + left, mn, lmx);
  build(pts, idx, first + left, last, rmn, mx);
}

// McIlroy's adversary: every item starts as "gas" (unknown, above every solid value); when two gas items meet, one is
// frozen to the next solid value; the item most recently seen as gas is the pivot candidate and is frozen first.
// The answers stay consistent with the final values, so the library makes the same comparisons on the output keys.
struct Adversary {
  std::vector<int64_t>* val;
  int64_t* nsolid;
  int32_t* candidate;
  int64_t gas;
  bool operator()(int32_t x, int32_t y) const {
    std::vector<int64_t>& v = *val;
    if (v[x] == gas && v[y] == gas) {
      if (x == *candidate) v[x] = (*nsolid)++;
      else v[y] = (*nsolid)++;
    }
    if (v[x] == gas) *candidate = x;
    else if (v[y] == gas) *candidate = y;
    return v[x] < v[y];
  }
};

}  // namespace

extern "C" {

// perm_out[0 .. n): the index array std::nth_element(nth) leaves, from iota, comparing keys[a] < keys[b]
int sm_oracle_nth_element_perm(const double* keys, int64_t n, int64_t nth, int32_t* perm_out) {
  if (n < 0 || n > (1 << 30) || nth < 0 || nth > n || (n > 0 && (!keys || !perm_out))) return -1;
  std::vector<int32_t> idx((size_t)n);
  std::iota(idx.begin(), idx.end(), 0);
  std::nth_element(idx.begin(), idx.begin() + nth, idx.end(), KeyLess{keys});
  std::copy(idx.begin(), idx.end(), perm_out);
  return 0;
}

// perm_out[0 .. n): BuildNormals' index array after the whole recursion (points 3xN column-major, finite)
int sm_oracle_normals_nth_perm(const double* points, int64_t n, int32_t* perm_out) {
  if (n <= 0 || n > (1 << 30) || !points || !perm_out) return -1;
  std::vector<int32_t> idx((size_t)n);
  std::iota(idx.begin(), idx.end(), 0);
  const double inf = std::numeric_limits<double>::infinity();
  double mn[3] = {inf, inf, inf}, mx[3] = {-inf, -inf, -inf};
  for (int64_t i = 0; i < n; ++i)
    for (int r = 0; r < 3; ++r) {
      mn[r] = std::min(mn[r], points[3 * i + r]);
      mx[r] = std::max(mx[r], points[3 * i + r]);
    }
  build(points, idx, 0, (int)n, mn, mx);
  std::copy(idx.begin(), idx.end(), perm_out);
  return 0;
}

// keys_out[0 .. n): values 0 .. s-1 for the items the adversary froze, in freezing order, and s for the rest
int sm_oracle_nth_element_adversary(int64_t n, int64_t nth, double* keys_out) {
  if (n < 0 || n > (1 << 30) || nth < 0 || nth > n || (n > 0 && !keys_out)) return -1;
  std::vector<int64_t> val((size_t)n, n);
  std::vector<int32_t> idx((size_t)n);
  std::iota(idx.begin(), idx.end(), 0);
  int64_t nsolid = 0;
  int32_t candidate = 0;
  std::nth_element(idx.begin(), idx.begin() + nth, idx.end(), Adversary{&val, &nsolid, &candidate, n});
  for (int64_t i = 0; i < n; ++i) keys_out[i] = (double)(val[(size_t)i] == n ? nsolid : val[(size_t)i]);
  return 0;
}

}  // extern "C"
