// CPU oracle of StatisticRemoval (include/sm_b200.h): PCL's StatisticalOutlierRemoval::applyFilterIndices with
// setMeanK(K) and setStddevMulThresh(std_mul), the call filter_statistic_removal.cc:44-59 of the reference leaves
// commented out.  PCL is not compiled here: the rules are restated from PCL 1.8 / 1.10 and FLANN's L2_Simple<float>.
// Built into libsm_oracle.so by oracle/Makefile; tests/oracle_statistic_removal.py binds it.  Two modes:
//   product (0)  what the GPU computes: the K + 1 neighbours from the k-NN oracle (sm_oracle_knn: libnabo's rules over
//                the coordinates widened to double, eps = 0, self-match allowed), and the two sums over all points
//                summed exactly and rounded once (Shewchuk's partials, finished as Python's math.fsum does) — written
//                here independently of the product's per-exponent bins;
//   literal (1)  PCL as it runs: neighbours ranked by FLANN's float d2, and the two sums serial in double in index
//                order.
// Steps 1 and 3-5 are the same in both: non-finite points get distance 0 and are not valid; entry 0 of the list is
// dropped; dist_sum += sqrt((double)d2) over entries 1..K in list order with the float d2 of L2_Simple<float>;
// distance = (float)(dist_sum / K); mean, variance, stddev and threshold in double; kept iff !(distance > threshold).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

extern "C" int sm_oracle_knn(const double* target, int64_t n_target, const double* query, int64_t n_query, int32_t k,
                             double epsilon, double max_radius, uint32_t flags, int bucket_size, int32_t* ids,
                             double* dists2);

namespace {

// FLANN's L2_Simple<float>: float differences, the squares accumulated in float from 0
float FloatD2(const float* q, const float* p) {
  float r = 0.f;
  for (int d = 0; d < 3; ++d) {
    const float diff = q[d] - p[d];
    r = r + diff * diff;
  }
  return r;
}

// Shewchuk's exact partials and the correctly rounded finish of CPython's math.fsum, for finite or +inf terms >= 0
double ExactSum(const std::vector<double>& terms) {
  std::vector<double> partials;
  for (double x : terms) {
    if (std::isinf(x)) return x;
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
  double hi = 0.0;
  size_t n = partials.size();
  if (n > 0) {
    hi = partials[--n];
    double lo = 0.0;
    while (n > 0) {
      const double x = hi, y = partials[--n];
      hi = x + y;
      const double yr = hi - x;
      lo = y - yr;
      if (lo != 0.0) break;
    }
    if (n > 0 && ((lo < 0.0 && partials[n - 1] < 0.0) || (lo > 0.0 && partials[n - 1] > 0.0))) {
      const double y = lo * 2.0;
      const double x = hi + y;
      const double yr = x - hi;
      if (y == yr) hi = x;
    }
  }
  return hi;
}

}  // namespace

extern "C" {

// points: n records of stride_bytes (x, y, z, intensity, factor first).  out: capacity n 5-float records, inliers:
// capacity n, distances: n floats, stats4: mean, stddev, threshold, valid.  Returns 0, -1 for K outside 1..63 or a bad
// stride / mode, -5 for 1..K finite points (nothing written).
int sm_oracle_statistic_removal(const float* points, int64_t n, int64_t stride_bytes, int32_t K, float std_mul,
                                int32_t mode, float* out, int64_t* m, int32_t* inliers, float* distances,
                                double* stats4) {
  if (K < 1 || K > 63 || stride_bytes < 20 || stride_bytes % 4 || n < 0 || (mode != 0 && mode != 1)) return -1;
  auto rec = [&](int64_t i) { return reinterpret_cast<const float*>(reinterpret_cast<const char*>(points) + i * stride_bytes); };
  std::vector<int64_t> finite;
  for (int64_t i = 0; i < n; ++i) {
    const float* p = rec(i);
    if (std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2])) finite.push_back(i);
  }
  const int64_t nf = (int64_t)finite.size();
  if (nf >= 1 && nf <= K) return -5;
  std::vector<float> dist((size_t)n, 0.f);
  if (nf > 0) {
    std::vector<double> xyz(3 * (size_t)nf);
    std::vector<float> fxyz(3 * (size_t)nf);
    for (int64_t j = 0; j < nf; ++j)
      for (int d = 0; d < 3; ++d) { fxyz[3 * j + d] = rec(finite[j])[d]; xyz[3 * j + d] = (double)fxyz[3 * j + d]; }
    // product: exactly the K + 1 of libnabo; literal: up to 64 candidates of libnabo, re-ranked by float d2
    const int kc = mode == 0 ? K + 1 : (int)std::min<int64_t>(64, nf);
    std::vector<int32_t> ids((size_t)nf * kc);
    std::vector<double> d2((size_t)nf * kc);
    sm_oracle_knn(xyz.data(), nf, xyz.data(), nf, kc, 0.0, INFINITY, 1u, 8, ids.data(), d2.data());
#pragma omp parallel for schedule(guided, 64)
    for (int64_t j = 0; j < nf; ++j) {
      const float* q = &fxyz[3 * j];
      std::vector<int32_t> list(ids.begin() + j * kc, ids.begin() + (j + 1) * kc);
      if (mode == 1) {
        std::vector<std::pair<float, int32_t>> cand;
        for (int32_t id : list) cand.push_back({FloatD2(q, &fxyz[3 * (size_t)id]), id});
        std::stable_sort(cand.begin(), cand.end(),
                         [](const std::pair<float, int32_t>& a, const std::pair<float, int32_t>& b) { return a.first < b.first; });
        // every point outside the candidates has double d2 >= the last candidate's; its float d2 is within 1e-6 of that
        const float sel = cand[(size_t)K].first;
        const double last = d2[(size_t)j * kc + kc - 1];
        if (kc < nf && !(sel == 0.f || (double)sel <= last * (1.0 - 1e-6))) {
          cand.clear();                               // margin too small: rank every finite point
          for (int64_t t = 0; t < nf; ++t) cand.push_back({FloatD2(q, &fxyz[3 * t]), (int32_t)t});
          std::stable_sort(cand.begin(), cand.end(), [](const std::pair<float, int32_t>& a,
                                                        const std::pair<float, int32_t>& b) { return a.first < b.first; });
        }
        for (int t = 0; t <= K; ++t) list[(size_t)t] = cand[(size_t)t].second;
      }
      double dist_sum = 0.0;
      for (int t = 1; t <= K; ++t) dist_sum += std::sqrt((double)FloatD2(q, &fxyz[3 * (size_t)list[(size_t)t]]));
      dist[(size_t)finite[j]] = (float)(dist_sum / K);
    }
  }
  double sum = 0.0, sq_sum = 0.0;
  if (mode == 0) {
    std::vector<double> a((size_t)n), b((size_t)n);
    for (int64_t i = 0; i < n; ++i) { a[i] = (double)dist[i]; b[i] = (double)(dist[i] * dist[i]); }
    sum = ExactSum(a);
    sq_sum = ExactSum(b);
  } else {
    for (int64_t i = 0; i < n; ++i) { sum += dist[i]; sq_sum += dist[i] * dist[i]; }
  }
  const double valid = (double)nf;
  const double mean = sum / valid;
  const double variance = (sq_sum - sum * sum / valid) / (valid - 1);
  const double stddev = std::sqrt(variance);
  const double threshold = mean + (double)std_mul * stddev;
  int64_t k = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (dist[i] > threshold) continue;
    std::memcpy(out + 5 * k, rec(i), 5 * sizeof(float));
    inliers[k++] = (int32_t)i;
  }
  *m = k;
  std::memcpy(distances, dist.data(), (size_t)n * sizeof(float));
  stats4[0] = mean; stats4[1] = stddev; stats4[2] = threshold; stats4[3] = valid;
  return 0;
}

}  // extern "C"
