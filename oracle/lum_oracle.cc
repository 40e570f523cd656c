// CPU oracle of MultiviewRegistratorLumPcl (include/sm_b200.h, sm_lum_*): AlignAll's five rounds of addPointCloud /
// CorrespondenceEstimation / setCorrespondences / compute over a persistent pcl::registration::LUM graph.  PCL is not
// compiled here: LUM, CorrespondenceEstimation::determineCorrespondences, transformPointCloud and getTransformation
// are restated from upstream PCL 1.8.1 (to be re-verified if its source becomes available).  The per-point float
// arithmetic and the host algebra are the product's own (staticmapping_b200/csrc/lum_host.h, written with the
// expressions PCL evaluates).  Built into libsm_oracle.so by oracle/Makefile; tests/oracle_lum.py binds it.  Modes:
//   product (0)  what the GPU computes: 1-NN in double over the float coordinates, ((dx^2 + dy^2) + dz^2), the smallest
//                index among equal distances, kept iff d2 <= 0.25^2; each per-edge sum exact and rounded once to float
//                (written here with Shewchuk's partials, independently of the product's per-exponent bins); D with a
//                double inverse; X with a double column-pivoted QR over the vertices joined to vertex 0; the pose
//                update in double.
//   literal (1)  PCL's float arithmetic: 1-NN by FLANN's float metric ((dx^2 + dy^2) + dz^2) (ties to the smallest
//                index: FLANN's own order is its visit order), serial float sums in correspondence order, D with a
//                float inverse, X with a float column-pivoted QR over all 6(n - 1) components, the update in float.
// Non-finite points are never a query or a match in either mode.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <numeric>
#include <vector>

#include "../staticmapping_b200/csrc/lum_host.h"

using namespace smb;

namespace {

// ---- exact float sums: Shewchuk's partials, then the float nearest their exact sum ------------------------------
void Grow(std::vector<double>& partials, double x) {
  size_t i = 0;
  for (double y : partials) {
    if (std::fabs(x) < std::fabs(y)) std::swap(x, y);
    const double hi = x + y;
    const double lo = y - (hi - x);
    if (lo != 0.0) partials[i++] = lo;
    x = hi;
  }
  partials.resize(i);
  partials.push_back(x);
}

// sign of (sum of partials) - v, exactly
int SignMinus(std::vector<double> partials, double v) {
  Grow(partials, -v);
  for (size_t k = partials.size(); k-- > 0;)
    if (partials[k] != 0.0) return partials[k] > 0.0 ? 1 : -1;
  return 0;
}

float ExactFloatSum(const std::vector<float>& terms) {
  bool pinf = false, ninf = false, nan = false;
  std::vector<double> partials;
  for (float t : terms) {
    if (std::isnan(t)) nan = true;
    else if (std::isinf(t)) (t > 0 ? pinf : ninf) = true;
    else Grow(partials, (double)t);
  }
  if (nan || (pinf && ninf)) return std::numeric_limits<float>::quiet_NaN();
  if (pinf) return std::numeric_limits<float>::infinity();
  if (ninf) return -std::numeric_limits<float>::infinity();
  double approx = 0.0;
  for (double p : partials) approx += p;
  float f = (float)approx;
  if (std::isinf(f)) {   // past FLT_MAX: infinity iff the exact sum reaches FLT_MAX + half an ulp
    const double edge = std::ldexp(2.0 - std::ldexp(1.0, -24), 127) * (f > 0 ? 1 : -1);
    const int s = SignMinus(partials, edge);
    if (f > 0 ? s < 0 : s > 0) f = f > 0 ? std::numeric_limits<float>::max() : -std::numeric_limits<float>::max();
    else return f;
  }
  // step to the nearest float: the exact sum lies within a few double ulps of approx, so at most one float away
  for (int it = 0; it < 4; ++it) {
    const float up = std::nextafter(f, std::numeric_limits<float>::infinity());
    const float dn = std::nextafter(f, -std::numeric_limits<float>::infinity());
    const double mid_up = ((double)f + (double)up) / 2, mid_dn = ((double)f + (double)dn) / 2;
    const int su = std::isinf(up) ? -1 : SignMinus(partials, mid_up);
    const int sd = std::isinf(dn) ? 1 : SignMinus(partials, mid_dn);
    uint32_t bits;
    std::memcpy(&bits, &f, 4);
    const bool even = (bits & 1u) == 0u;
    if (su > 0 || (su == 0 && !even)) { f = up; continue; }
    if (sd < 0 || (sd == 0 && !even)) { f = dn; continue; }
    break;
  }
  if (f == 0.f) f = 0.f;   // +0 for a zero sum
  return f;
}

// ---- exact 1-NN with the smallest index among ties, in the mode's metric -----------------------------------------
struct Tree {
  const float* pts;   // packed xyz of the frame
  std::vector<int> idx;
  struct Node { int lo, hi, dim, left, right; float cut; };
  std::vector<Node> nodes;
  int Build(int lo, int hi) {
    Node nd{lo, hi, -1, -1, -1, 0.f};
    if (hi - lo > 8) {
      float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
      for (int k = lo; k < hi; ++k)
        for (int d = 0; d < 3; ++d) { mn[d] = std::min(mn[d], pts[3 * idx[k] + d]); mx[d] = std::max(mx[d], pts[3 * idx[k] + d]); }
      int dim = 0;
      for (int d = 1; d < 3; ++d) if (mx[d] - mn[d] > mx[dim] - mn[dim]) dim = d;
      const int mid = (lo + hi) / 2;
      std::nth_element(idx.begin() + lo, idx.begin() + mid, idx.begin() + hi,
                       [&](int a, int b) { return pts[3 * a + dim] < pts[3 * b + dim]; });
      nd.dim = dim;
      nd.cut = pts[3 * idx[mid] + dim];
    }
    const int me = (int)nodes.size();
    nodes.push_back(nd);
    if (nd.dim >= 0) {
      const int mid = (lo + hi) / 2;
      const int l = Build(lo, mid), r = Build(mid, hi);
      nodes[me].left = l;
      nodes[me].right = r;
    }
    return me;
  }
};

double Metric(bool literal, const float* q, const float* p) {
  if (literal) {
    const float dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
    return (double)((dx * dx + dy * dy) + dz * dz);
  }
  const double dx = (double)q[0] - (double)p[0], dy = (double)q[1] - (double)p[1], dz = (double)q[2] - (double)p[2];
  return (dx * dx + dy * dy) + dz * dz;
}

void Search(const Tree& t, int node, bool literal, const float* q, double& best, int& best_id) {
  const Tree::Node& nd = t.nodes[node];
  if (nd.dim < 0) {
    for (int k = nd.lo; k < nd.hi; ++k) {
      const int id = t.idx[k];
      const double d = Metric(literal, q, t.pts + 3 * id);
      if (d < best || (d == best && id < best_id)) { best = d; best_id = id; }
    }
    return;
  }
  // the cut is a point coordinate and a side holds points on both sides' boundary: both sides may hold ties
  const double off = (double)q[nd.dim] - (double)nd.cut;
  const int near = off > 0 ? nd.right : nd.left, far = off > 0 ? nd.left : nd.right;
  Search(t, near, literal, q, best, best_id);
  if (off * off <= best * (1.0 + 1e-6) + 1e-300) Search(t, far, literal, q, best, best_id);
}

struct Oracle {
  bool literal;
  int64_t stride = 0;
  std::vector<std::vector<char>> frames;
  std::vector<float> frame_pose;
  std::vector<int> vertex_frame;
  std::vector<float> poses;
  std::vector<std::vector<int32_t>> corr;   // per pair (j, i) in loop order: query, match pairs
  bool trace_on = false;
  struct Iter { int n; std::vector<float> edges; std::vector<double> X; std::vector<float> poses; double sum; };
  std::vector<Iter> trace;
};

constexpr int kTraceEdge = 67;

int64_t Count(const Oracle& o, int f) { return (int64_t)(o.frames[f].size() / o.stride); }

void ComputeEdge(const Oracle& o, int s, int t, const std::vector<int32_t>& c, const std::vector<std::vector<float>>& xyz,
                 float* rec) {
  float Ts[12], Tt[12];
  lum_pose_matrix(&o.poses[6 * s], Ts);
  lum_pose_matrix(&o.poses[6 * t], Tt);
  const int fs = o.vertex_frame[s], ft = o.vertex_frame[t];
  std::vector<std::vector<float>> terms(kLumTerms);
  std::vector<float> av, df;
  for (size_t k = 0; k < c.size() / 2; ++k) {
    float a[3], d[3], tm[kLumTerms];
    if (!lum_pair(Ts, Tt, &xyz[fs][3 * (size_t)c[2 * k]], &xyz[ft][3 * (size_t)c[2 * k + 1]], a, d)) continue;
    lum_pair_terms(a, d, tm);
    for (int r = 0; r < kLumTerms; ++r) terms[r].push_back(tm[r]);
    av.insert(av.end(), a, a + 3);
    df.insert(df.end(), d, d + 3);
  }
  const int pairs = (int)av.size() / 3;
  float S[kLumTerms], MM[36], MZ[6], D[6] = {0, 0, 0, 0, 0, 0}, ss = 0.f, cinv[36], cinvd[6];
  for (int r = 0; r < kLumTerms; ++r) {
    if (o.literal) {
      float acc = 0.f;
      for (float v : terms[r]) acc += v;
      S[r] = acc;
    } else {
      S[r] = ExactFloatSum(terms[r]);
    }
  }
  lum_mm_mz(S, pairs, MM, MZ);
  if (pairs >= 3) {
    if (o.literal) lum_edge_d<float>(MM, MZ, D);
    else lum_edge_d<double>(MM, MZ, D);
    std::vector<float> st;
    for (int k = 0; k < pairs; ++k) st.push_back(lum_ss_term(&av[3 * k], &df[3 * k], D));
    if (o.literal) { for (float v : st) ss += v; }
    else ss = ExactFloatSum(st);
    lum_edge_finish(MM, MZ, ss, cinv, cinvd);
  } else {
    std::fill(cinv, cinv + 36, 0.f);
    std::fill(cinvd, cinvd + 6, 0.f);
  }
  rec[0] = (float)s; rec[1] = (float)t; rec[2] = (float)pairs;
  std::memcpy(rec + 3, S, sizeof(S));
  std::memcpy(rec + 18, D, sizeof(D));
  rec[24] = ss;
  std::memcpy(rec + 25, cinv, sizeof(cinv));
  std::memcpy(rec + 61, cinvd, sizeof(cinvd));
}

void Compute(Oracle& o, const std::vector<std::pair<int, int>>& edges, const std::vector<const std::vector<int32_t>*>& ec,
             const std::vector<std::vector<float>>& xyz) {
  const int n = (int)o.vertex_frame.size();
  if (n < 2) return;
  for (int it = 0; it < kLumIterations; ++it) {
    std::vector<float> rec(edges.size() * kTraceEdge);
    std::vector<LumEdge> le(edges.size());
    for (size_t e = 0; e < edges.size(); ++e) {
      float* r = &rec[e * kTraceEdge];
      ComputeEdge(o, edges[e].first, edges[e].second, *ec[e], xyz, r);
      le[e].s = edges[e].first;
      le[e].t = edges[e].second;
      std::memcpy(le[e].cinv, r + 25, sizeof(le[e].cinv));
      std::memcpy(le[e].cinvd, r + 61, sizeof(le[e].cinvd));
    }
    double sum;
    std::vector<double> X;
    if (o.literal) {
      std::vector<float> Xf;
      sum = lum_solve_update<float>(n, le, o.poses.data(), &Xf);
      X.assign(Xf.begin(), Xf.end());
    } else {
      sum = lum_solve_update<double>(n, le, o.poses.data(), &X);
    }
    if (o.trace_on) o.trace.push_back({n, rec, X, o.poses, sum});
    if (lum_converged(sum, n)) return;
  }
}

}  // namespace

extern "C" {

void* sm_oracle_lum_create(int32_t mode) {
  Oracle* o = new Oracle();
  o->literal = mode == 1;
  return o;
}

void sm_oracle_lum_destroy(void* h) { delete static_cast<Oracle*>(h); }

int sm_oracle_lum_add_cloud(void* h, const float* points, int64_t n, int64_t stride, const float* pose16) {
  Oracle& o = *static_cast<Oracle*>(h);
  if (!pose16 || n < 0 || (n > 0 && !points) || stride < 12 || stride % 4 || (o.stride && stride != o.stride))
    return -1;
  o.stride = stride;
  const char* p = reinterpret_cast<const char*>(points);
  o.frames.emplace_back(p, p + n * stride);
  o.frame_pose.insert(o.frame_pose.end(), pose16, pose16 + 16);
  return 0;
}

int sm_oracle_lum_align_all(void* h, float* out, int64_t capacity, int64_t* m_out) {
  Oracle& o = *static_cast<Oracle*>(h);
  const int N = (int)o.frames.size();
  *m_out = 0;
  if (N == 0) return 0;
  const int V0 = (int)o.vertex_frame.size();
  std::vector<int> vf(N);
  int64_t need = 0;
  for (int v = 0; v < N; ++v) { vf[v] = v < V0 ? o.vertex_frame[v] : v - V0; need += Count(o, vf[v]); }
  std::vector<int64_t> counts(N);
  for (int f = 0; f < N; ++f) counts[f] = Count(o, f);
  if (lum_queries(counts.data(), N) > kLumMaxQueries) return -1;
  if (out && capacity < need) { *m_out = need; return -1; }
  // transformPointCloud of every frame by its pose
  std::vector<std::vector<float>> xyz(N);
  for (int f = 0; f < N; ++f) {
    float T[12];
    lum_matrix4_to_3x4(&o.frame_pose[16 * f], T);
    const int64_t c = Count(o, f);
    xyz[f].resize(3 * c);
    for (int64_t q = 0; q < c; ++q)
      lum_transform(T, reinterpret_cast<const float*>(o.frames[f].data() + q * o.stride), &xyz[f][3 * q]);
  }
  // determineCorrespondences(source j, target i) for j < i
  o.corr.clear();
  std::vector<std::pair<int, int>> edges;
  std::vector<const std::vector<int32_t>*> ec;
  std::vector<Tree> trees(N);
  for (int i = 1; i < N; ++i) {
    trees[i].pts = xyz[i].data();
    for (int64_t q = 0; q < Count(o, i); ++q)
      if (lum_finite3(&xyz[i][3 * q])) trees[i].idx.push_back((int)q);
    if (!trees[i].idx.empty()) trees[i].Build(0, (int)trees[i].idx.size());
  }
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < i; ++j) {
      std::vector<int32_t> c;
      if (!trees[i].idx.empty())
        for (int64_t q = 0; q < Count(o, j); ++q) {
          const float* p = &xyz[j][3 * q];
          if (!lum_finite3(p)) continue;
          double best = INFINITY;
          int id = -1;
          Search(trees[i], 0, o.literal, p, best, id);
          if (id >= 0 && !(best > (double)kLumMaxDistance * (double)kLumMaxDistance)) {
            c.push_back((int32_t)q);
            c.push_back(id);
          }
        }
      o.corr.push_back(c);
    }
  for (int i = 0, p = 0; i < N; ++i)
    for (int j = 0; j < i; ++j, ++p)
      if (o.corr[p].size() / 2 > 2) {
        if (Count(o, vf[j]) < Count(o, j) || Count(o, vf[i]) < Count(o, i)) return -1;
        edges.push_back({j, i});
        ec.push_back(&o.corr[p]);
      }
  // the vertices' clouds are the transformed frames: vertex v reads xyz[vertex_frame[v]]
  for (int r = 0; r < kLumRounds; ++r) {
    for (int f = 0; f < N; ++f) {
      o.vertex_frame.push_back(f);
      for (int k = 0; k < 6; ++k) o.poses.push_back(0.f);
    }
    Compute(o, edges, ec, xyz);
  }
  *m_out = need;
  if (!out) return 0;
  char* w = reinterpret_cast<char*>(out);
  for (int v = 0; v < N; ++v) {
    float T[12];
    lum_pose_matrix(&o.poses[6 * v], T);
    const int f = vf[v];
    for (int64_t q = 0; q < Count(o, f); ++q) {
      std::memcpy(w, o.frames[f].data() + q * o.stride, o.stride);
      lum_transform(T, &xyz[f][3 * q], reinterpret_cast<float*>(w));
      w += o.stride;
    }
  }
  return 0;
}

int sm_oracle_lum_poses(void* h, float* out, int64_t capacity, int64_t* n) {
  Oracle& o = *static_cast<Oracle*>(h);
  *n = (int64_t)o.vertex_frame.size();
  if (!out) return 0;
  if (capacity < *n) return -1;
  std::copy(o.poses.begin(), o.poses.end(), out);
  return 0;
}

int sm_oracle_lum_correspondences(void* h, int32_t j, int32_t i, int32_t* pairs, int64_t capacity, int64_t* n) {
  Oracle& o = *static_cast<Oracle*>(h);
  const int64_t p = (int64_t)i * (i - 1) / 2 + j;
  if (j < 0 || i <= j || p >= (int64_t)o.corr.size()) return -1;
  *n = (int64_t)o.corr[p].size() / 2;
  if (!pairs) return 0;
  if (capacity < *n) return -1;
  std::copy(o.corr[p].begin(), o.corr[p].end(), pairs);
  return 0;
}

int sm_oracle_lum_trace(void* h, int32_t enable) {
  Oracle& o = *static_cast<Oracle*>(h);
  o.trace_on = enable != 0;
  o.trace.clear();
  return 0;
}

int sm_oracle_lum_trace_get(void* h, int64_t it, int32_t* nv, int32_t* ne, float* edges, double* X, float* poses,
                            double* sum) {
  Oracle& o = *static_cast<Oracle*>(h);
  if (it < 0) { *nv = 0; *ne = (int32_t)o.trace.size(); *sum = 0; return 0; }
  if (it >= (int64_t)o.trace.size()) return -1;
  const Oracle::Iter& t = o.trace[it];
  *nv = t.n;
  *ne = (int32_t)(t.edges.size() / kTraceEdge);
  *sum = t.sum;
  if (edges) std::copy(t.edges.begin(), t.edges.end(), edges);
  if (X) std::copy(t.X.begin(), t.X.end(), X);
  if (poses) std::copy(t.poses.begin(), t.poses.end(), poses);
  return 0;
}

}  // extern "C"
