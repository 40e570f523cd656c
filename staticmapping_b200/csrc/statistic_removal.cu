// pre_processers::filter::StatisticRemoval on the device: PCL's StatisticalOutlierRemoval::applyFilterIndices with
// setMeanK(point_num_meank) and setStddevMulThresh(std_mul), the call the reference's filter_statistic_removal.cc:44-59
// leaves commented out under a TODO (its Filter does nothing).  PCL is not compiled here: the rules are restated from
// PCL 1.8 / 1.10 (the libpcl-dev of the reference's Dockerfiles), see DESIGN.md section 4j.
//
//   pack    flag the finite points (x, y, z all finite) and compact them in input order into a double SoA with their
//           input indices (compact.cuh); a non-finite point gets distance 0.  Read back: the finite count nf.
//   tree    KdCompactTree over the nf finite points, ids payload, bucket 8 (the tree of sm_knn).
//   search  knn_mean_distance_query: the K + 1 nearest finite points of each finite point (eps = 0, self-match allowed,
//           no radius, libnabo's tie rules), entry 0 dropped, the mean of sqrt(float d2) over entries 1..K, one float
//           per point (statistic_removal.cuh).
//   stats   sum and sum of squares of the n distances, each the exact sum rounded once to double (per-exponent int64
//           bins, shared then global integer atomics, one thread to finish); mean, stddev and threshold stay on the
//           device.
//   select  keep iff !(distance > threshold), then the chain's ordered scatter of whole records, which carries the scan
//           indices of a chain stage's input.  Read back: m.
// Compiled with -fmad=false.
#include <math.h>
#include <string.h>

#include <algorithm>

#include "../../include/sm_b200.h"
#include "../../include/sm_b200_debug.h"
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"
#include "record_filter.h"
#include "statistic_removal.cuh"

namespace smb {
namespace {

constexpr int kSrBinThreads = 256;

inline int64_t sr_pad64(int64_t n) { return (n + 63) & ~(int64_t)63; }

__device__ __forceinline__ bool sr_finite(const float* p) { return isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]); }

__global__ void __launch_bounds__(kCompactThreads)
sr_finite_count_kernel(const char* __restrict__ pts, int64_t stride, int n, uint8_t* __restrict__ flag,
                       uint32_t* __restrict__ tile_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n) break;
    const bool keep = sr_finite(reinterpret_cast<const float*>(pts + (int64_t)i * stride));
    flag[i] = keep ? 1 : 0;
    c += keep ? 1u : 0u;
  }
  tile_count_store(c, tile_cnt);
}

// coord: [3][cstride] doubles of the finite points in input order, index: their input indices, *nf: their number;
// dist = 0 for the other points
__global__ void __launch_bounds__(kCompactThreads)
sr_pack_kernel(const char* __restrict__ pts, int64_t stride, int n, const uint8_t* __restrict__ flag,
               const uint32_t* __restrict__ tile_off, double* __restrict__ coord, int64_t cstride,
               uint32_t* __restrict__ index, float* __restrict__ dist, uint32_t* __restrict__ nf) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n) ? flag[base + r] : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n) break;
    if (!f[r]) { dist[i] = 0.f; continue; }
    const float* p = reinterpret_cast<const float*>(pts + (int64_t)i * stride);
    coord[pos] = (double)p[0]; coord[cstride + pos] = (double)p[1]; coord[2 * cstride + pos] = (double)p[2];
    index[pos] = (uint32_t)i;
    ++pos;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *nf = tile_off[gridDim.x];
}

// bins[0 .. kExactBins): the distances, bins[kExactBins ..): their float squares (zeroed before)
__global__ void __launch_bounds__(kSrBinThreads)
sr_bins_kernel(const float* __restrict__ dist, int n, unsigned long long* __restrict__ bins) {
  __shared__ unsigned long long s[2 * kExactBins];
  for (int b = threadIdx.x; b < 2 * kExactBins; b += blockDim.x) s[b] = 0ull;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const float v = dist[i];
    int b; uint32_t m;
    exact_bin(v, &b, &m);
    if (m) atomicAdd(&s[b], (unsigned long long)m);
    exact_bin(__fmul_rn(v, v), &b, &m);
    if (m) atomicAdd(&s[kExactBins + b], (unsigned long long)m);
  }
  __syncthreads();
  for (int b = threadIdx.x; b < 2 * kExactBins; b += blockDim.x)
    if (s[b]) atomicAdd(&bins[b], s[b]);
}

// stats[0..3] = mean, stddev, threshold, valid (PCL's expressions in double, literally)
__global__ void __launch_bounds__(32)
sr_finish_kernel(const unsigned long long* __restrict__ bins, const uint32_t* __restrict__ nf, float std_mul,
                 double* __restrict__ stats) {
  __shared__ uint64_t limb[kExactLimbs];
  if (threadIdx.x != 0) return;
  const double sum = exact_finish(reinterpret_cast<const int64_t*>(bins), limb);
  const double sq_sum = exact_finish(reinterpret_cast<const int64_t*>(bins) + kExactBins, limb);
  const double valid = (double)*nf;
  const double mean = __ddiv_rn(sum, valid);
  const double variance = __ddiv_rn(__dsub_rn(sq_sum, __ddiv_rn(__dmul_rn(sum, sum), valid)), __dsub_rn(valid, 1.0));
  const double stddev = __dsqrt_rn(variance);
  stats[0] = mean;
  stats[1] = stddev;
  stats[2] = __dadd_rn(mean, __dmul_rn((double)std_mul, stddev));
  stats[3] = valid;
}

__global__ void __launch_bounds__(kCompactThreads)
sr_select_kernel(const float* __restrict__ dist, int n, const double* __restrict__ stats, uint8_t* __restrict__ flag,
                 uint32_t* __restrict__ tile_cnt) {
  const double threshold = stats[2];
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n) break;
    const bool keep = !((double)dist[i] > threshold);
    flag[i] = keep ? 1 : 0;
    c += keep ? 1u : 0u;
  }
  tile_count_store(c, tile_cnt);
}

}  // namespace

bool StatisticRemoval::k_ok() const { return params.point_num_meank >= 1 && params.point_num_meank <= kSrMaxMeanK; }

int StatisticRemoval::reserve(int64_t n) {
  SMB_RC(flag.reserve((size_t)n));
  SMB_RC(tile_cnt.reserve(compact_count_bytes(n)));
  SMB_RC(coord.reserve((size_t)3 * sr_pad64(n) * sizeof(double)));
  SMB_RC(index.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(dist.reserve((size_t)n * sizeof(float)));
  SMB_RC(bins.reserve(2 * kExactBins * sizeof(unsigned long long)));
  SMB_RC(stats.reserve(4 * sizeof(double)));
  return count.reserve(2 * sizeof(uint32_t));
}

int StatisticRemoval::run(const char* pts, int64_t n, int64_t stride, const uint32_t* index_in, float* out,
                          uint32_t* out_index, int64_t* m, cudaStream_t s) {
  const int K = params.point_num_meank;
  const int ni = (int)n;
  const int tiles = compact_tiles(n);
  const int64_t cs = sr_pad64(n);
  SMB_RC(reserve(n));
  last_n = 0;
  uint32_t* cnt = (uint32_t*)count.p;
  uint32_t* tc = (uint32_t*)tile_cnt.p;
  SMB_CUDA_OK(cudaMemsetAsync(bins.p, 0, 2 * kExactBins * sizeof(unsigned long long), s));
  sr_finite_count_kernel<<<tiles, kCompactThreads, 0, s>>>(pts, stride, ni, (uint8_t*)flag.p, tc);
  compact_scan(tc, tiles, s);
  sr_pack_kernel<<<tiles, kCompactThreads, 0, s>>>(pts, stride, ni, (const uint8_t*)flag.p, tc, (double*)coord.p, cs,
                                                   (uint32_t*)index.p, (float*)dist.p, cnt);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t nf = 0;                                   // sizes the tree
  SMB_CUDA_OK(cudaMemcpyAsync(&nf, cnt, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  if (nf >= 1 && nf <= (uint32_t)K) return SM_ERR_CHECK_FAILED;   // PCL reads past its k-list there
  if (nf > 0) {
    if (kd_num_levels((int)nf, 8) > 24) return SM_ERR_BAD_ARGUMENT;
    SMB_RC(tree.reserve((int)nf, 8, KdCompactTree::kIds));
    KdWorkspace ws;
    SMB_RC(ws.carve(kdws, (int)nf, 8));
    SMB_RC(tree.build((const double*)coord.p, nullptr, cs, (int)nf, 8, ws, s));
    SMB_RC(knn_mean_distance_query(tree.view(), (const double*)coord.p, cs, (int)nf, K, (const uint32_t*)index.p,
                                   (float*)dist.p, s));
  }
  const int bin_blocks = (int)std::min<int64_t>(ceil_div(n, kSrBinThreads), 4 * kNumSMs);
  sr_bins_kernel<<<bin_blocks, kSrBinThreads, 0, s>>>((const float*)dist.p, ni, (unsigned long long*)bins.p);
  sr_finish_kernel<<<1, 32, 0, s>>>((const unsigned long long*)bins.p, cnt, params.std_mul, (double*)stats.p);
  sr_select_kernel<<<tiles, kCompactThreads, 0, s>>>((const float*)dist.p, ni, (const double*)stats.p,
                                                     (uint8_t*)flag.p, tc);
  filter_compact_records(pts, stride, index_in, ni, (const uint8_t*)flag.p, tc, out, out_index, cnt + 1, s);
  SMB_CUDA_OK(cudaGetLastError());
  uint32_t kept = 0;
  SMB_CUDA_OK(cudaMemcpyAsync(&kept, cnt + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaMemcpyAsync(host_stats, stats.p, 4 * sizeof(double), cudaMemcpyDeviceToHost, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  last_n = n;
  *m = (int64_t)kept;
  return SM_OK;
}

}  // namespace smb

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace smb;

struct sm_statistic_removal : RecordFilter {
  StatisticRemoval f;
  explicit sm_statistic_removal(int device) : RecordFilter(device, "StatisticRemoval") {}
};

namespace {
// the checks both run entry points make before a device is selected
int sr_check(sm_statistic_removal* h, const void* points, int64_t n, int64_t stride_bytes, const void* out,
             const int64_t* m_out) {
  if (!h || !records_ok(points, n, stride_bytes, out, m_out)) return SM_ERR_BAD_ARGUMENT;
  if (!h->f.k_ok())
    return h->fail(SM_ERR_BAD_ARGUMENT, "point_num_meank %d is outside 1..%d", h->f.params.point_num_meank,
                   kSrMaxMeanK);
  return SM_OK;
}
}  // namespace

extern "C" {

int sm_statistic_removal_create(int device, sm_statistic_removal** out) { return create_record_filter(device, out); }

int sm_statistic_removal_destroy(sm_statistic_removal* h) { return destroy_record_filter(h); }

int sm_statistic_removal_set_param(sm_statistic_removal* h, const char* name, int type, const char* text) {
  if (!h || !name || !text) return SM_ERR_BAD_ARGUMENT;
  return h->set_param(h->f.params, name, type, text);
}

int sm_statistic_removal_run_device(sm_statistic_removal* h, const float* dev_points, int64_t n, int64_t stride_bytes,
                                    float* dev_out, int64_t* m_out, int32_t* dev_inlier_index, void* cuda_stream) {
  SMB_RC(sr_check(h, dev_points, n, stride_bytes, dev_out, m_out));
  SMB_RC(h->use_device());
  if (n == 0) {
    *m_out = 0;
    h->f.last_n = 0;
    h->f.host_stats[0] = h->f.host_stats[1] = h->f.host_stats[2] = NAN;   // no finite point: 0 / 0
    h->f.host_stats[3] = 0.0;
    return SM_OK;
  }
  uint32_t* idx = (uint32_t*)dev_inlier_index;
  if (!idx) {
    SMB_RC(h->cuda_fail(h->host_idx.reserve((size_t)n * sizeof(int32_t))));
    idx = (uint32_t*)h->host_idx.p;
  }
  const int rc = h->f.run((const char*)dev_points, n, stride_bytes, nullptr, dev_out, idx, m_out,
                          (cudaStream_t)cuda_stream);
  if (rc == SM_ERR_CHECK_FAILED)
    return h->fail(rc, "Check failed: between 1 and point_num_meank finite points (PCL reads past its k-list)");
  if (rc == SM_ERR_BAD_ARGUMENT) return h->fail(rc, "more finite points than the 24-level k-d tree holds");
  return h->cuda_fail(rc);
}

int sm_statistic_removal_run(sm_statistic_removal* h, const float* points, int64_t n, int64_t stride_bytes, float* out,
                             int64_t* m_out, int32_t* inlier_index) {
  SMB_RC(sr_check(h, points, n, stride_bytes, out, m_out));
  SMB_RC(h->use_device());
  return run_record_filter(h, sm_statistic_removal_run_device, points, n, stride_bytes, out, m_out, inlier_index);
}

int sm_statistic_removal_stats(const sm_statistic_removal* h, double* out4) {
  if (!h || !out4) return SM_ERR_BAD_ARGUMENT;
  memcpy(out4, h->f.host_stats, 4 * sizeof(double));
  return SM_OK;
}

const char* sm_statistic_removal_last_error(const sm_statistic_removal* h) { return h ? h->error : ""; }

// ---- test hooks (include/sm_b200_debug.h) -------------------------------------------------------------------------
int sm_debug_statistic_removal_exact_sum_host(const float* terms, int64_t n, double* sum) {
  if ((n > 0 && !terms) || n < 0 || n > (1 << 30) || !sum) return SM_ERR_BAD_ARGUMENT;
  int64_t bins[kExactBins] = {0};
  for (int64_t i = 0; i < n; ++i) {
    if (!(terms[i] >= 0.f)) return SM_ERR_BAD_ARGUMENT;     // the sum is defined for non-negative terms and +inf
    int b; uint32_t m;
    exact_bin(terms[i], &b, &m);
    bins[b] += m;
  }
  uint64_t limb[kExactLimbs];
  *sum = exact_finish(bins, limb);
  return SM_OK;
}

int sm_debug_statistic_removal_distance_host(const float* query_3, const float* neighbours_3k, int32_t K,
                                             float* distance) {
  if (!query_3 || !neighbours_3k || !distance || K < 1 || K > kSrMaxMeanK) return SM_ERR_BAD_ARGUMENT;
  double sum = 0.0;
  for (int j = 0; j < K; ++j)
    sum = sr_dadd(sum, sr_neighbour_term(query_3[0], query_3[1], query_3[2], neighbours_3k[3 * j],
                                         neighbours_3k[3 * j + 1], neighbours_3k[3 * j + 2]));
  *distance = sr_mean_distance(sum, K);
  return SM_OK;
}

int sm_debug_statistic_removal_distances(const sm_statistic_removal* h, float* out, int64_t capacity, int64_t* n) {
  if (!h || !n || capacity < 0 || (capacity > 0 && !out)) return SM_ERR_BAD_ARGUMENT;
  *n = h->f.last_n;
  if (h->f.last_n == 0) return SM_OK;
  if (capacity < h->f.last_n) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(h->device));
  SMB_CUDA_OK(cudaMemcpy(out, h->f.dist.p, (size_t)h->f.last_n * sizeof(float), cudaMemcpyDeviceToHost));
  return SM_OK;
}

}  // extern "C"
