// pre_processers::filter::Factory::Filter on the device (pre_processors/filter_factory.cc:83-106): the chain every
// scan goes through before it is matched (builder/data/data_collector.cc:137-141), over Range, AxisRange,
// BoundingBoxRemoval, RandomSampler, RangeImage and GroundRemoval2.
//
// Every filter emits its inliers in ascending input index, whole records (x, y, z, intensity, factor) copied.
//   Range / AxisRange / BoundingBoxRemoval / RandomSampler are per-point predicates: consecutive ones run as ONE
//     flag kernel, then an ordered compaction (compact.cuh).  RandomSampler is a deterministic stand-in, see filter_keep.
//   RangeImage (filter_range_image.cc:82-141): the first point in input order to reach an empty pixel is the inlier.
//     atomicMin of the point index on a pixel-owner image gives exactly that, whatever the thread order.
//   GroundRemoval2 (filter_ground_removal2.cc:127-414): polar cell per point -> stable radix sort by cell (members of
//     a cell stay in input order) -> one thread per cell walks its points in order (running minimum and membership
//     are order dependent, :195-209) -> one thread per segment runs FitLines' sequential scan (:240-316) -> one
//     thread per point for ClusterGround (:337-396) -> ordered compaction of the non-ground points.
// Compiled with -fmad=false: the float expressions are the reference's, operation by operation.  sqrtf and the
// divisions are correctly rounded on both sides; atan2f is CUDA's here and glibc's there, so a point within a few
// ulps of a row / column / segment border can land next door (DESIGN.md section 4h).
#include <float.h>
#include <limits.h>
#include <math.h>
#include <string.h>

#include "../../include/sm_b200.h"
#include "common.cuh"
#include "compact.cuh"
#include "kernels.h"

namespace smb {
namespace {

constexpr int kMaxRun = 8;              // predicates of one flag kernel; a longer run is split
constexpr int kMaxCells = 1 << 24;      // RangeImage pixels / GroundRemoval2 cells

struct PredicateRun { int count; uint32_t seed; FilterParams f[kMaxRun]; };

// A float / double -> int conversion outside int's range is undefined in C++; the reference's x86 build yields INT_MIN
// there (also for NaN), which its clamps and range tests then read as "below 0".  Restated so on every side.
__host__ __device__ __forceinline__ int to_int(double q) {
  return (q > -2147483649.0 && q < 2147483648.0) ? (int)q : INT_MIN;
}

__host__ __device__ __forceinline__ uint32_t fmix32(uint32_t x) {   // MurmurHash3's 32-bit finaliser
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return x;
}

// inlier test of the four predicate filters; `index` is the point's index in the scan handed to the chain
__host__ __device__ inline bool filter_keep(const FilterParams& f, const float* p, uint32_t index, uint32_t seed) {
  switch (f.kind) {
    case kFilterRange: {            // filter_range.cc:59-68
      const float range = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
      return range >= f.min_range && range <= f.max_range;
    }
    case kFilterAxisRange: {        // filter_axis_range.cc:50-90: a NaN coordinate is neither < min nor > max and stays
      if (f.min == -FLT_MAX && f.max == FLT_MAX) return true;
      if (f.axis_index < 0 || f.axis_index > 2) return true;   // the switch's default branch
      const float v = p[f.axis_index];
      return !(v < f.min || v > f.max);
    }
    case kFilterBoundingBoxRemoval:  // filter_bounding_box.cc:69-78, common/bounding_box.cc:117-121: inside = removed
      return !((p[0] >= f.min_x && p[0] <= f.max_x) && (p[1] >= f.min_y && p[1] <= f.max_y) &&
               (p[2] >= f.min_z && p[2] <= f.max_z));
    case kFilterRandomSampler:      // filter_random_sample.cc:44-72
      if ((double)f.sampling_rate > 0.999) return true;
      // The reference draws from mt19937(random_device()): its result is not a function of its inputs.  Stand-in:
      // a counter hash of the scan index, so the filter stays a pure per-point predicate.
      return (double)fmix32(index * 0x9E3779B9u + seed) <= (double)f.sampling_rate * 4294967296.0;
    default: return true;
  }
}

// filter_range_image.cc:102-126: the pixel of a point, false for the outlier branches
__host__ __device__ inline bool range_image_pixel(const FilterParams& f, const RangeImageConsts& c, const float* p,
                                                  int* row, int* col) {
  const float x = p[0] + f.offset_x, y = p[1] + f.offset_y, z = p[2] + f.offset_z;
  const float dxy = sqrtf(x * x + y * y);
  if (dxy < 0.01f) return false;
  const float v = atan2f(z, dxy);
  const int r = to_int(((double)v - c.btm) / (double)c.vres);     // double expression (M_PI), truncated toward zero
  if (r < 0 || r >= f.vertical_line_num) return false;
  float h = atan2f(y, x);
  if (h < 0.f) h = (float)((double)h + M_PI * 2);
  long cc = lroundf(h / c.hres);
  if (cc >= f.horizontal_line_num) cc -= f.horizontal_line_num;
  if (cc < 0 || cc >= f.horizontal_line_num) return false;
  *row = r; *col = (int)cc;
  return true;
}

// filter_ground_removal2.cc:163-191: every point is binned (the range test at :165 is never true), indices clamped
__host__ __device__ inline void gr2_cell(const FilterParams& f, const Gr2Consts& c, const float* p, float* range,
                                         int* s, int* b) {
  const float r = sqrtf(p[0] * p[0] + p[1] * p[1]);
  float rad = atan2f(p[1], p[0]);
  if (rad < 0.f) rad += c.two_pi;
  int si = to_int(rad / c.delta_alpha), bi = to_int((r - f.r_min) / c.delta_bin);
  if (bi >= f.bin_num) bi = f.bin_num - 1; else if (bi < 0) bi = 0;
  if (si >= f.segment_num) si = f.segment_num - 1; else if (si < 0) si = 0;
  *range = r; *s = si; *b = bi;
}

// FitLocalLine (filter_ground_removal2.cc:29-44): [d 1] (m b)^T = z by Eigen's ColPivHouseholderQR in double, the result
// cast to float.  A written-out QR (column norms, pivoting with norm down-dating, two Householder reflections, the
// reflections applied to z, back substitution) with every sum taken in index order; a0, a1, c: n doubles each,
// `ws` apart.  n >= 2.
__host__ __device__ inline void gr2_fit_line(const float* d, const float* z, int64_t ps, int n, double* a0, double* a1,
                                             double* c, int64_t ws, float* m_out, float* b_out) {
  for (int i = 0; i < n; ++i) { a0[i * ws] = (double)d[i * ps]; a1[i * ws] = 1.0; c[i * ws] = (double)z[i * ps]; }
  double* col[2] = {a0, a1};
  double upd[2], dir[2], tau[2];
  for (int j = 0; j < 2; ++j) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += col[j][i * ws] * col[j][i * ws];
    upd[j] = dir[j] = sqrt(s);
  }
  const double eps = DBL_EPSILON;
  const double maxn = upd[1] > upd[0] ? upd[1] : upd[0];
  const double thr_helper = (maxn * eps) * (maxn * eps) / (double)n;
  const double downdate = sqrt(eps);
  int nzp = 2;
  bool swapped = false;
  for (int k = 0; k < 2; ++k) {
    int big = k;
    for (int j = k + 1; j < 2; ++j) if (upd[j] > upd[big]) big = j;
    if (nzp == 2 && upd[big] * upd[big] < thr_helper * (double)(n - k)) nzp = k;
    if (big != k) {
      double* t = col[k]; col[k] = col[big]; col[big] = t;
      double u = upd[k]; upd[k] = upd[big]; upd[big] = u;
      u = dir[k]; dir[k] = dir[big]; dir[big] = u;
      swapped = !swapped;
    }
    double* x = col[k];
    // makeHouseholderInPlace on rows k..n-1
    double tail = 0.0;
    for (int i = k + 1; i < n; ++i) tail += x[i * ws] * x[i * ws];
    const double c0 = x[k * ws];
    double beta;
    if (tail <= DBL_MIN) {
      tau[k] = 0.0; beta = c0;
      for (int i = k + 1; i < n; ++i) x[i * ws] = 0.0;
    } else {
      beta = sqrt(c0 * c0 + tail);
      if (c0 >= 0.0) beta = -beta;
      for (int i = k + 1; i < n; ++i) x[i * ws] = x[i * ws] / (c0 - beta);
      tau[k] = (beta - c0) / beta;
    }
    x[k * ws] = beta;
    for (int j = k + 1; j < 2; ++j) {
      double* y = col[j];
      if (n - k == 1) {
        y[k * ws] *= 1.0 - tau[k];
      } else if (tau[k] != 0.0) {
        double t = 0.0;
        for (int i = k + 1; i < n; ++i) t += x[i * ws] * y[i * ws];
        t += y[k * ws];
        y[k * ws] -= tau[k] * t;
        for (int i = k + 1; i < n; ++i) y[i * ws] -= t * (tau[k] * x[i * ws]);
      }
      if (upd[j] != 0.0) {          // norm down-date
        double t = fabs(y[k * ws]) / upd[j];
        t = (1.0 + t) * (1.0 - t);
        t = t < 0.0 ? 0.0 : t;
        const double q = upd[j] / dir[j];
        const double t2 = t * (q * q);
        if (t2 <= downdate) {
          double s = 0.0;
          for (int i = k + 1; i < n; ++i) s += y[i * ws] * y[i * ws];
          dir[j] = upd[j] = sqrt(s);
        } else {
          upd[j] *= sqrt(t);
        }
      }
    }
  }
  // c = Q^T z over the first nzp reflections
  for (int k = 0; k < nzp; ++k) {
    const double* x = col[k];
    if (n - k == 1) {
      c[k * ws] *= 1.0 - tau[k];
    } else if (tau[k] != 0.0) {
      double t = 0.0;
      for (int i = k + 1; i < n; ++i) t += x[i * ws] * c[i * ws];
      t += c[k * ws];
      c[k * ws] -= tau[k] * t;
      for (int i = k + 1; i < n; ++i) c[i * ws] -= t * (tau[k] * x[i * ws]);
    }
  }
  double r[2] = {0.0, 0.0};
  if (nzp == 2) {
    r[1] = c[1 * ws] / col[1][1 * ws];
    r[0] = (c[0] - r[1] * col[1][0]) / col[0][0];
  } else if (nzp == 1) {
    r[0] = c[0] / col[0][0];
  }
  // column permutation: r[i] belongs to the source column that ended in column i
  *m_out = (float)(swapped ? r[1] : r[0]);
  *b_out = (float)(swapped ? r[0] : r[1]);
}

// VerticalDistanceToSegment (filter_ground_removal2.cc:398-414): no break, the last line whose interval holds the point
// wins; *bad is set where the reference CHECK-fails (:403)
__host__ __device__ inline float gr2_vertical_distance(const Gr2Line* lines, int n_lines, float d, float z, int* bad) {
  const float margin = 0.1f;
  float distance = -1.f;
  for (int l = 0; l < n_lines; ++l) {
    const Gr2Line line = lines[l];
    if (!(line.d0 < line.d1)) { *bad = 1; continue; }
    if (line.d0 - margin < d && line.d1 + margin > d) {
      const float delta_z = line.z1 - line.z0, delta_d = line.d1 - line.d0;
      const float expected_z = (d - line.d0) / delta_d * delta_z + line.z0;
      distance = fabsf(z - expected_z);
    }
  }
  return distance;
}

// ---- predicates and the scatter every stage ends in ---------------------------------------------------------------
__global__ void __launch_bounds__(kCompactThreads)
filter_predicate_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ index_in, int n,
                        const __grid_constant__ PredicateRun run, uint8_t* __restrict__ flag,
                        uint32_t* __restrict__ block_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n) break;
    const float* p = reinterpret_cast<const float*>(pts + (int64_t)i * stride);
    const uint32_t index = index_in ? index_in[i] : (uint32_t)i;
    bool keep = true;
    for (int k = 0; k < run.count && keep; ++k) keep = filter_keep(run.f[k], p, index, run.seed);
    flag[i] = keep ? 1 : 0;
    c += keep ? 1u : 0u;
  }
  tile_count_store(c, block_cnt);
}

// out / index_out: the flagged records in input order; *m = their number.  tile_off: records kept before each tile
__global__ void __launch_bounds__(kCompactThreads)
filter_scatter_kernel(const char* __restrict__ pts, int64_t stride, const uint32_t* __restrict__ index_in, int n,
                      const uint8_t* __restrict__ flag, const uint32_t* __restrict__ tile_off,
                      float* __restrict__ out, uint32_t* __restrict__ index_out, uint32_t* __restrict__ m) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t f[kCompactItems], c = 0;
  for (int r = 0; r < kCompactItems; ++r) { f[r] = (base + r < n) ? flag[base + r] : 0u; c += f[r]; }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    if (!f[r]) continue;
    const int i = base + r;
    const float* p = reinterpret_cast<const float*>(pts + (int64_t)i * stride);
    float* q = out + (int64_t)pos * 5;
    q[0] = p[0]; q[1] = p[1]; q[2] = p[2]; q[3] = p[3]; q[4] = p[4];
    index_out[pos] = index_in ? index_in[i] : (uint32_t)i;
    ++pos;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *m = tile_off[gridDim.x];
}

// ---- RangeImage -----------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
range_image_owner_kernel(const char* __restrict__ pts, int64_t stride, int n, const FilterParams f,
                         const RangeImageConsts c, uint32_t* __restrict__ pixel, uint32_t* __restrict__ owner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int row, col;
  uint32_t px = 0xffffffffu;
  if (range_image_pixel(f, c, reinterpret_cast<const float*>(pts + (int64_t)i * stride), &row, &col)) {
    px = (uint32_t)row * (uint32_t)f.horizontal_line_num + (uint32_t)col;
    atomicMin(&owner[px], (uint32_t)i);
  }
  pixel[i] = px;
}

__global__ void __launch_bounds__(kCompactThreads)
range_image_flag_kernel(const uint32_t* __restrict__ pixel, const uint32_t* __restrict__ owner, int n,
                        uint8_t* __restrict__ flag, uint32_t* __restrict__ block_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n) break;
    const uint32_t px = pixel[i];
    const bool keep = px != 0xffffffffu && owner[px] == (uint32_t)i;
    flag[i] = keep ? 1 : 0;
    c += keep ? 1u : 0u;
  }
  tile_count_store(c, block_cnt);
}

// ---- GroundRemoval2 -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gr2_key_kernel(const char* __restrict__ pts, int64_t stride, int n, const FilterParams f, const Gr2Consts c,
               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ cell_of,
               float2* __restrict__ pt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = reinterpret_cast<const float*>(pts + (int64_t)i * stride);
  float range; int s, b;
  gr2_cell(f, c, p, &range, &s, &b);
  const uint32_t cell = (uint32_t)s * (uint32_t)f.bin_num + (uint32_t)b;
  keys[i] = cell; vals[i] = (uint32_t)i; cell_of[i] = cell;
  pt[i] = make_float2(range, p[2]);
}

// cell_range[2 * cell], [2 * cell + 1]: first and one past the last sorted position of the cell (zeroed before)
__global__ void __launch_bounds__(256)
gr2_bounds_kernel(const uint64_t* __restrict__ keys, int n, uint32_t* __restrict__ cell_range) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = keys[i];
  if (i == 0 || keys[i - 1] != k) cell_range[2 * k] = (uint32_t)i;
  if (i == n - 1 || keys[i + 1] != k) cell_range[2 * k + 1] = (uint32_t)(i + 1);
}

// filter_ground_removal2.cc:195-209, one thread per cell over its points in input order: min_z_point is replaced on a
// strict < or while the cell has no member; a point joins iff z <= the running minimum + 0.5 at that moment
__global__ void __launch_bounds__(128)
gr2_cell_kernel(const uint32_t* __restrict__ order, const uint32_t* __restrict__ cell_range, int n_cells,
                const float2* __restrict__ pt, uint8_t* __restrict__ member, uint32_t* __restrict__ cell_cnt,
                float2* __restrict__ cell_min) {
  const int cell = blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= n_cells) return;
  float2 mn = make_float2(1.e6f, 1.e6f);
  uint32_t cnt = 0;
  for (uint32_t j = cell_range[2 * cell], e = cell_range[2 * cell + 1]; j < e; ++j) {
    const uint32_t i = order[j];
    const float2 p = pt[i];
    if (cnt == 0 || p.y < mn.y) mn = p;
    const bool joins = (double)p.y <= (double)mn.y + 0.5;
    member[i] = joins ? 1 : 0;
    cnt += joins ? 1u : 0u;
  }
  cell_cnt[cell] = cnt;
  cell_min[cell] = mn;
}

// FitLines (filter_ground_removal2.cc:240-316), one thread per segment.  current_line_points is always a window
// [lo, hi] of the segment's occupied bins in bin order (a push appends the next occupied bin, the erase keeps the
// last one), so the points are compacted once into occ and the --i retry re-reads entry hi + 1.
// occ: [2][bin_num][segment_num] floats (d, z); work: [3][bin_num][segment_num] doubles; lines: [segment][max_lines]
__global__ void __launch_bounds__(64)
gr2_fit_kernel(const FilterParams f, const uint32_t* __restrict__ cell_cnt, const float2* __restrict__ cell_min,
               float* __restrict__ occ, double* __restrict__ work, Gr2Line* __restrict__ lines, int max_lines,
               int* __restrict__ n_lines, int* __restrict__ status) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  const int S = f.segment_num, B = f.bin_num;
  if (s >= S) return;
  const int64_t plane = (int64_t)B * S;
  float* od = occ + s; float* oz = occ + plane + s;
  double* a0 = work + s; double* a1 = work + plane + s; double* cc = work + 2 * plane + s;
  int cnt = 0, first = -1;
  for (int b = 0; b < B; ++b) {
    if (cell_cnt[s * B + b] == 0) continue;
    if (first < 0) first = b;
    const float2 p = cell_min[s * B + b];
    od[(int64_t)cnt * S] = p.x; oz[(int64_t)cnt * S] = p.y;
    ++cnt;
  }
  int nl = 0;
  Gr2Line* out = lines + (int64_t)s * max_lines;
  if (first >= 0 && first < B - 1) {
    int lo = 0, hi = 0;
    float cm = 0.f, cb = 0.f;
    bool long_line = false;
    float ground_height = f.start_ground_height;
    auto emit = [&](int l, int h) {
      float m, b;
      gr2_fit_line(od + (int64_t)l * S, oz + (int64_t)l * S, S, h - l + 1, a0, a1, cc, S, &m, &b);
      Gr2Line line;
      line.d0 = od[(int64_t)l * S]; line.z0 = m * line.d0 + b;
      line.d1 = od[(int64_t)h * S]; line.z1 = m * line.d1 + b;
      if (!(line.d0 < line.d1)) *status = 1;
      if (nl < max_lines) out[nl] = line;
      ++nl;
      return m * line.d1 + b;
    };
    for (int e = 1; e < cnt; ++e) {
      const float de = od[(int64_t)e * S], ze = oz[(int64_t)e * S];
      if (de - od[(int64_t)hi * S] >= f.long_line_threshold) long_line = true;
      float expected_z = FLT_MAX;
      const int size = hi - lo + 1;
      if (long_line && size > 2) expected_z = cm * de + cb;
      if (size >= 2) {
        hi = e;
        gr2_fit_line(od + (int64_t)lo * S, oz + (int64_t)lo * S, S, hi - lo + 1, a0, a1, cc, S, &cm, &cb);
        float err = 0.f;
        for (int k = lo; k <= hi; ++k) {
          const float er = fabsf(cm * od[(int64_t)k * S] + cb - oz[(int64_t)k * S]);
          if (er > err) err = er;
        }
        if (err > f.max_error || fabsf(cm) > f.max_slope ||
            (long_line && fabsf(expected_z - ze) > f.max_long_line_height)) {
          hi = e - 1;
          if (hi - lo + 1 >= 3) ground_height = emit(lo, hi);
          long_line = false;
          lo = hi;
          --e;
        }
      } else {
        if (!long_line && fabsf(oz[(int64_t)hi * S] - ground_height) < f.max_start_height) hi = e;
        else lo = hi = e;
      }
    }
    if (hi - lo + 1 > 2) emit(lo, hi);
  }
  n_lines[s] = nl;
}

// ClusterGround (filter_ground_removal2.cc:337-396) per member point: own segment first; on a distance < 0 the
// neighbours +k, -k, ..., +1, -1, breaking on a distance > 0; ground iff 0 < distance <= max_dist_to_line.
// flag = 1 for the points that stay (not ground).
__global__ void __launch_bounds__(kCompactThreads)
gr2_ground_kernel(const FilterParams f, const Gr2Consts c, int n, const uint32_t* __restrict__ cell_of,
                  const float2* __restrict__ pt, const uint8_t* __restrict__ member,
                  const Gr2Line* __restrict__ lines, int max_lines, const int* __restrict__ n_lines,
                  uint8_t* __restrict__ flag, uint32_t* __restrict__ block_cnt, int* __restrict__ status) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t cnt = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    const int i = base + r;
    if (i >= n) break;
    bool ground = false;
    if (member[i]) {
      const int s = (int)(cell_of[i] / (uint32_t)f.bin_num);
      const float2 p = pt[i];
      int bad = 0;
      float distance = gr2_vertical_distance(lines + (int64_t)s * max_lines, n_lines[s], p.x, p.y, &bad);
      if (distance < 0.f) {
        for (int k = c.search_steps; k > 0; --k) {
          for (int sign = 1; sign >= -1; sign -= 2) {
            int t = s + sign * k;
            if (t < 0) t += f.segment_num; else if (t >= f.segment_num) t -= f.segment_num;
            distance = gr2_vertical_distance(lines + (int64_t)t * max_lines, n_lines[t], p.x, p.y, &bad);
            if (distance > 0.f) break;
          }
          if (distance > 0.f) break;
        }
      }
      ground = distance > 0.f && distance <= f.max_dist_to_line;
      if (bad) *status = 1;
    }
    flag[i] = ground ? 0 : 1;
    cnt += ground ? 0u : 1u;
  }
  tile_count_store(cnt, block_cnt);
}

int sort_passes(int n_cells) { return n_cells <= (1 << 16) ? 2 : 4; }   // even: the sorted pairs end in the first buffers

}  // namespace

// ---- parameters -------------------------------------------------------------------------------------------------
FilterParams filter_defaults(int kind) {
  FilterParams f;
  memset(&f, 0, sizeof(f));
  f.kind = kind;
  f.min_range = 0.f; f.max_range = FLT_MAX;
  f.min = -FLT_MAX; f.max = FLT_MAX; f.axis_index = 2;
  f.min_x = f.min_y = f.min_z = -FLT_MAX; f.max_x = f.max_y = f.max_z = FLT_MAX;
  f.sampling_rate = 1.f;
  f.top_angle = 30.f; f.btm_angle = -15.f; f.vertical_line_num = 40; f.horizontal_line_num = 1800;
  f.r_max = 100.f; f.r_min = 1.f; f.bin_num = 200; f.segment_num = 180;
  f.start_ground_height = -0.25f; f.long_line_threshold = 1.0f; f.max_long_line_height = 0.1f;
  f.max_start_height = 0.2f; f.max_error = 0.05f; f.max_slope = (float)tan(M_PI / 12.); f.max_b = 0.1f;
  f.max_dist_to_line = 0.05f; f.search_angle = 10.f; f.thread_num = 4;
  return f;
}

bool filter_param(FilterParams& f, const char* name, void** target, int* type) {
  struct Entry { int kind; const char* name; int type; void* p; };
  const Entry table[] = {
      {kFilterRange, "min_range", 1, &f.min_range}, {kFilterRange, "max_range", 1, &f.max_range},
      {kFilterAxisRange, "min", 1, &f.min}, {kFilterAxisRange, "max", 1, &f.max},
      {kFilterAxisRange, "axis_index", 0, &f.axis_index},
      {kFilterBoundingBoxRemoval, "min_x", 1, &f.min_x}, {kFilterBoundingBoxRemoval, "min_y", 1, &f.min_y},
      {kFilterBoundingBoxRemoval, "min_z", 1, &f.min_z}, {kFilterBoundingBoxRemoval, "max_x", 1, &f.max_x},
      {kFilterBoundingBoxRemoval, "max_y", 1, &f.max_y}, {kFilterBoundingBoxRemoval, "max_z", 1, &f.max_z},
      {kFilterRandomSampler, "sampling_rate", 1, &f.sampling_rate},
      {kFilterRangeImage, "top_angle", 1, &f.top_angle}, {kFilterRangeImage, "btm_angle", 1, &f.btm_angle},
      {kFilterRangeImage, "offset_x", 1, &f.offset_x}, {kFilterRangeImage, "offset_y", 1, &f.offset_y},
      {kFilterRangeImage, "offset_z", 1, &f.offset_z},
      {kFilterRangeImage, "vertical_line_num", 0, &f.vertical_line_num},
      {kFilterRangeImage, "horizontal_line_num", 0, &f.horizontal_line_num},
      {kFilterGroundRemoval2, "r_max", 1, &f.r_max}, {kFilterGroundRemoval2, "r_min", 1, &f.r_min},
      {kFilterGroundRemoval2, "start_ground_height", 1, &f.start_ground_height},
      {kFilterGroundRemoval2, "long_line_threshold", 1, &f.long_line_threshold},
      {kFilterGroundRemoval2, "max_long_line_height", 1, &f.max_long_line_height},
      {kFilterGroundRemoval2, "max_start_height", 1, &f.max_start_height},
      {kFilterGroundRemoval2, "max_error", 1, &f.max_error}, {kFilterGroundRemoval2, "max_slope", 1, &f.max_slope},
      {kFilterGroundRemoval2, "max_b", 1, &f.max_b},
      {kFilterGroundRemoval2, "max_dist_to_line", 1, &f.max_dist_to_line},
      {kFilterGroundRemoval2, "search_angle", 1, &f.search_angle},
      {kFilterGroundRemoval2, "bin_num", 0, &f.bin_num}, {kFilterGroundRemoval2, "segment_num", 0, &f.segment_num},
      {kFilterGroundRemoval2, "thread_num", 0, &f.thread_num},
  };
  for (const Entry& e : table)
    if (e.kind == f.kind && strcmp(e.name, name) == 0) { *target = e.p; *type = e.type; return true; }
  return false;
}

bool filter_configs_valid(const FilterParams& f) {
  switch (f.kind) {
    case kFilterAxisRange: return f.max > f.min && f.axis_index >= 0 && f.axis_index <= 2;   // filter_axis_range.cc:41-43
    case kFilterBoundingBoxRemoval: return f.min_x < f.max_x && f.min_y < f.max_y && f.min_z < f.max_z;   // filter_bounding_box.cc:49-51
    case kFilterRandomSampler: return f.sampling_rate >= 0.f && f.sampling_rate <= 1.f;       // filter_random_sample.cc:35-37
    default: return true;                                                                    // Interface::ConfigsValid
  }
}

RangeImageConsts range_image_consts(const FilterParams& f) {
  RangeImageConsts c;
  c.hres = (float)(M_PI * 2 / (double)(float)f.horizontal_line_num);
  c.vres = (float)((double)((f.top_angle - f.btm_angle) / (float)f.vertical_line_num / 180.f) * M_PI);
  c.btm = (double)(f.btm_angle / 180.f) * M_PI;
  return c;
}

Gr2Consts gr2_consts(const FilterParams& f) {
  Gr2Consts c;
  c.two_pi = (float)(M_PI * 2);
  c.delta_alpha = c.two_pi / (float)f.segment_num;
  c.delta_bin = (f.r_max - f.r_min) / (float)f.bin_num;
  const float cluster_delta_alpha = (float)(M_PI * 2 / (double)f.segment_num);   // :340 derives it again, in double
  c.search_steps = to_int((double)f.search_angle / 180. * M_PI / (double)cluster_delta_alpha);
  return c;
}

bool filter_debug_keep_host(const FilterParams& f, const float* rec, uint32_t index, uint32_t seed) {
  return filter_keep(f, rec, index, seed);
}
bool filter_debug_pixel_host(const FilterParams& f, const float* rec, int* row, int* col) {
  return range_image_pixel(f, range_image_consts(f), rec, row, col);
}
void filter_debug_cell_host(const FilterParams& f, const float* rec, float* range, int* s, int* b) {
  gr2_cell(f, gr2_consts(f), rec, range, s, b);
}
void filter_debug_fit_host(const float* d, const float* z, int n, float* m, float* b) {
  std::vector<double> w(3 * (size_t)n);
  gr2_fit_line(d, z, 1, n, w.data(), w.data() + n, w.data() + 2 * (size_t)n, 1, m, b);
}
float filter_debug_distance_host(const Gr2Line* lines, int n_lines, float d, float z, int* bad) {
  return gr2_vertical_distance(lines, n_lines, d, z, bad);
}

// ---- FilterChain ------------------------------------------------------------------------------------------------
int FilterChain::stage_end(int first) const {
  if (filters[first].kind > kFilterRandomSampler) return first + 1;
  int e = first;
  while (e < (int)filters.size() && e - first < kMaxRun && filters[e].kind <= kFilterRandomSampler) ++e;
  return e;
}

int FilterChain::reserve(int64_t n) {
  for (int k = 0; k < 2; ++k) {
    SMB_RC(rec[k].reserve((size_t)n * 20));
    SMB_RC(idx[k].reserve((size_t)n * sizeof(uint32_t)));
  }
  SMB_RC(flag.reserve((size_t)n));
  SMB_RC(block_cnt.reserve(compact_count_bytes(n)));
  SMB_RC(count.reserve(2 * sizeof(uint32_t)));
  for (const FilterParams& f : filters) {
    if (f.kind == kFilterRangeImage) {
      SMB_RC(pixel.reserve((size_t)n * sizeof(uint32_t)));
      SMB_RC(owner.reserve((size_t)f.vertical_line_num * (size_t)f.horizontal_line_num * sizeof(uint32_t)));
    } else if (f.kind == kFilterGroundRemoval2) {
      const size_t n_cells = (size_t)f.bin_num * (size_t)f.segment_num;
      const int64_t st = (n + 63) & ~(int64_t)63;
      SMB_RC(sort.reserve(RadixPairs::bytes(st, (int)n) + 256));
      SMB_RC(cell_of.reserve((size_t)n * sizeof(uint32_t)));
      SMB_RC(pt.reserve((size_t)n * sizeof(float2)));
      SMB_RC(member.reserve((size_t)n));
      SMB_RC(cells.reserve(n_cells * (2 * sizeof(uint32_t) + sizeof(uint32_t) + sizeof(float2))));
      SMB_RC(occ.reserve(2 * n_cells * sizeof(float)));
      SMB_RC(work.reserve(3 * n_cells * sizeof(double)));
      const size_t max_lines = (size_t)f.bin_num / 2 + 1;
      SMB_RC(lines.reserve((size_t)f.segment_num * (max_lines * sizeof(Gr2Line) + sizeof(int)) + 256));
    }
  }
  return 0;
}

int FilterChain::predicate_stage(int first, int cnt, const char* in, const uint32_t* index_in, int n, int64_t stride,
                                 float* out, uint32_t* index_out, cudaStream_t s) {
  PredicateRun run;
  run.count = cnt; run.seed = sample_seed;
  for (int k = 0; k < cnt; ++k) run.f[k] = filters[first + k];
  const int tiles = compact_tiles(n);
  filter_predicate_kernel<<<tiles, kCompactThreads, 0, s>>>(in, stride, index_in, n, run, (uint8_t*)flag.p,
                                                            (uint32_t*)block_cnt.p);
  compact_scan((uint32_t*)block_cnt.p, tiles, s);
  filter_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(in, stride, index_in, n, (const uint8_t*)flag.p,
                                                          (const uint32_t*)block_cnt.p, out, index_out,
                                                          (uint32_t*)count.p);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

int FilterChain::range_image_stage(const FilterParams& f, const char* in, const uint32_t* index_in, int n,
                                   int64_t stride, float* out, uint32_t* index_out, cudaStream_t s) {
  const RangeImageConsts c = range_image_consts(f);
  const size_t pixels = (size_t)f.vertical_line_num * (size_t)f.horizontal_line_num;
  const int tiles = compact_tiles(n);
  SMB_CUDA_OK(cudaMemsetAsync(owner.p, 0xff, pixels * sizeof(uint32_t), s));
  range_image_owner_kernel<<<ceil_div(n, 256), 256, 0, s>>>(in, stride, n, f, c, (uint32_t*)pixel.p, (uint32_t*)owner.p);
  range_image_flag_kernel<<<tiles, kCompactThreads, 0, s>>>((const uint32_t*)pixel.p, (const uint32_t*)owner.p, n,
                                                            (uint8_t*)flag.p, (uint32_t*)block_cnt.p);
  compact_scan((uint32_t*)block_cnt.p, tiles, s);
  filter_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(in, stride, index_in, n, (const uint8_t*)flag.p,
                                                          (const uint32_t*)block_cnt.p, out, index_out,
                                                          (uint32_t*)count.p);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

int FilterChain::ground_removal2_stage(const FilterParams& f, const char* in, const uint32_t* index_in, int n,
                                       int64_t stride, float* out, uint32_t* index_out, cudaStream_t s) {
  const Gr2Consts c = gr2_consts(f);
  const int n_cells = f.bin_num * f.segment_num;
  const int tiles = compact_tiles(n);
  const int64_t st = ((int64_t)n + 63) & ~(int64_t)63;
  RadixPairs rp;
  rp.carve(sort.p, st);
  uint32_t* cell_range = (uint32_t*)cells.p;
  uint32_t* cell_cnt = cell_range + 2 * (size_t)n_cells;
  float2* cell_min = (float2*)(cell_cnt + n_cells);
  const int max_lines = f.bin_num / 2 + 1;
  Gr2Line* ln = (Gr2Line*)lines.p;
  int* n_lines = (int*)(ln + (size_t)f.segment_num * max_lines);
  int* status = (int*)((uint32_t*)count.p + 1);
  SMB_CUDA_OK(cudaMemsetAsync(status, 0, sizeof(int), s));
  SMB_CUDA_OK(cudaMemsetAsync(cell_range, 0, 2 * (size_t)n_cells * sizeof(uint32_t), s));
  gr2_key_kernel<<<ceil_div(n, 256), 256, 0, s>>>(in, stride, n, f, c, rp.keys[0], rp.vals[0], (uint32_t*)cell_of.p,
                                                  (float2*)pt.p);
  SMB_RC(radix_sort_pairs_u64(rp.keys[0], rp.vals[0], rp.keys[1], rp.vals[1], n, 1, st, rp.scratch, s,
                              sort_passes(n_cells)));
  gr2_bounds_kernel<<<ceil_div(n, 256), 256, 0, s>>>(rp.keys[0], n, cell_range);
  gr2_cell_kernel<<<ceil_div(n_cells, 128), 128, 0, s>>>(rp.vals[0], cell_range, n_cells, (const float2*)pt.p,
                                                         (uint8_t*)member.p, cell_cnt, cell_min);
  gr2_fit_kernel<<<ceil_div(f.segment_num, 64), 64, 0, s>>>(f, cell_cnt, cell_min, (float*)occ.p, (double*)work.p, ln,
                                                            max_lines, n_lines, status);
  gr2_ground_kernel<<<tiles, kCompactThreads, 0, s>>>(f, c, n, (const uint32_t*)cell_of.p, (const float2*)pt.p,
                                                      (const uint8_t*)member.p, ln, max_lines, n_lines,
                                                      (uint8_t*)flag.p, (uint32_t*)block_cnt.p, status);
  compact_scan((uint32_t*)block_cnt.p, tiles, s);
  filter_scatter_kernel<<<tiles, kCompactThreads, 0, s>>>(in, stride, index_in, n, (const uint8_t*)flag.p,
                                                          (const uint32_t*)block_cnt.p, out, index_out,
                                                          (uint32_t*)count.p);
  SMB_CUDA_OK(cudaGetLastError());
  gr2 = {(const uint32_t*)cell_of.p, (const uint8_t*)member.p, cell_cnt, cell_min, ln, n_lines, (const uint8_t*)flag.p,
         max_lines, 0};
  return 0;
}

int FilterChain::run(const char* in, int64_t n, int64_t stride, float* out, int32_t* out_index, int64_t* m,
                     cudaStream_t s) {
  *m = 0;
  for (const FilterParams& f : filters) {
    // RangeImage::SetInputCloud keeps its previous cloud for such a size (filter_range_image.cc:72-74); the box of an
    // invalid BoundingBoxRemoval CHECK-fails in its constructor (common/bounding_box.cc:114)
    if (f.kind == kFilterRangeImage && (f.vertical_line_num <= 0 || f.horizontal_line_num <= 0 ||
                                        (int64_t)f.vertical_line_num * f.horizontal_line_num > kMaxCells))
      return SM_ERR_BAD_ARGUMENT;
    if (f.kind == kFilterGroundRemoval2 &&
        (f.bin_num <= 0 || f.segment_num <= 0 || (int64_t)f.bin_num * f.segment_num > kMaxCells ||
         gr2_consts(f).search_steps < 0 || gr2_consts(f).search_steps >= f.segment_num))
      return SM_ERR_BAD_ARGUMENT;
    if (f.kind == kFilterBoundingBoxRemoval && !filter_configs_valid(f)) return SM_ERR_CHECK_FAILED;
  }
  if (n == 0) return 0;
  SMB_RC(reserve(n));
  const char* cur = in;
  const uint32_t* cur_idx = nullptr;
  int64_t cur_stride = stride;
  uint32_t cur_n = (uint32_t)n;
  const int n_filters = (int)filters.size();
  int stage = 0, first = 0;
  do {   // an empty chain is one stage without a predicate: a copy
    const int end = n_filters ? stage_end(first) : 0;
    const bool last = end >= n_filters;
    float* dst = last ? out : (float*)rec[stage & 1].p;
    uint32_t* dst_idx = (last && out_index) ? (uint32_t*)out_index : (uint32_t*)idx[stage & 1].p;
    int gr2_status = 0;
    if (!n_filters || filters[first].kind <= kFilterRandomSampler) {
      SMB_RC(predicate_stage(first, end - first, cur, cur_idx, (int)cur_n, cur_stride, dst, dst_idx, s));
    } else if (filters[first].kind == kFilterRangeImage) {
      SMB_RC(range_image_stage(filters[first], cur, cur_idx, (int)cur_n, cur_stride, dst, dst_idx, s));
    } else {
      SMB_RC(ground_removal2_stage(filters[first], cur, cur_idx, (int)cur_n, cur_stride, dst, dst_idx, s));
      gr2_status = 1;
    }
    uint32_t host[2] = {0, 0};    // the stage's count sizes the next stage's grids
    SMB_CUDA_OK(cudaMemcpyAsync(host, count.p, sizeof(host), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaStreamSynchronize(s));
    if (gr2_status && host[1]) { gr2.status = 1; return SM_ERR_CHECK_FAILED; }   // CHECK(line.start[0] < line.end[0])
    cur = (const char*)dst; cur_idx = dst_idx; cur_stride = 20; cur_n = host[0];
    first = end; ++stage;
  } while (first < n_filters && cur_n > 0);   // a filter handed an empty cloud does nothing (its SetInputCloud)
  *m = (int64_t)cur_n;
  return 0;
}

}  // namespace smb

// ---- C ABI ------------------------------------------------------------------------------------------------------
using namespace smb;

struct sm_filter_chain {
  int device = 0;
  FilterChain chain;
  cudaStream_t stream = nullptr;
  DevBuf host_in, host_out, host_idx;
  char error[256] = {0};
};

namespace smb {
const FilterChain* filter_chain_of(const ::sm_filter_chain* c) { return c ? &c->chain : nullptr; }
}  // namespace smb

namespace {
int chain_fail(sm_filter_chain* c, int rc, const char* fmt, const char* arg) {
  snprintf(c->error, sizeof(c->error), fmt, arg);
  return rc;
}
int chain_device(sm_filter_chain* c) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
    return chain_fail(c, SM_ERR_NO_DEVICE, "no CUDA device: the filter chain has no CPU fallback%s", "");
  SMB_CUDA_OK(cudaSetDevice(c->device));
  return 0;
}
}  // namespace

extern "C" {

int sm_filter_chain_create(int device, sm_filter_chain** out) {
  if (!out || device < 0) return SM_ERR_BAD_ARGUMENT;
  *out = new sm_filter_chain;
  (*out)->device = device;
  return SM_OK;
}

int sm_filter_chain_destroy(sm_filter_chain* c) {
  if (!c) return SM_ERR_BAD_ARGUMENT;
  if (c->stream) { cudaSetDevice(c->device); cudaStreamDestroy(c->stream); }
  delete c;
  return SM_OK;
}

int sm_filter_chain_add(sm_filter_chain* c, const char* filter_name) {
  if (!c || !filter_name) return SM_ERR_BAD_ARGUMENT;
  static const char* const built[] = {"Range", "AxisRange", "BoundingBoxRemoval", "RandomSampler", "RangeImage",
                                      "GroundRemoval2"};
  for (int k = 0; k < 6; ++k)
    if (strcmp(filter_name, built[k]) == 0) {
      c->chain.filters.push_back(filter_defaults(k));
      return (int)c->chain.filters.size() - 1;
    }
  for (const char* name : {"GroundRemoval", "StatisticRemoval", "VoxelGrid"})
    if (strcmp(filter_name, name) == 0)
      return chain_fail(c, SM_ERR_UNSUPPORTED_TYPE, "filter %s is not built into the chain", filter_name);
  return chain_fail(c, SM_ERR_UNKNOWN_OPTION, "%s not supported yet.", filter_name);
}

int sm_filter_chain_set_param(sm_filter_chain* c, int filter, const char* name, int type, const char* text) {
  if (!c || !name || !text || filter < 0 || filter >= (int)c->chain.filters.size()) return SM_ERR_BAD_ARGUMENT;
  void* target = nullptr;
  int declared = 0;
  if (!filter_param(c->chain.filters[filter], name, &target, &declared))
    return chain_fail(c, SM_ERR_UNKNOWN_OPTION, "Check failed: all_right (unknown param %s)", name);
  if (type != 0 && type != 1)
    return chain_fail(c, SM_ERR_BAD_ARGUMENT, "Check failed: all_right (param %s without a type of 0 or 1)", name);
  // pugixml's as_int / as_float by the XML type, then XmlInterface::SetValue's cast to the declared type
  const double v = type == 0 ? (double)(int32_t)strtol(text, nullptr, 10) : (double)(float)strtod(text, nullptr);
  if (declared == 0) *(int32_t*)target = type == 0 ? (int32_t)v : (int32_t)to_int(v);
  else *(float*)target = (float)v;
  return SM_OK;
}

int sm_filter_chain_validate(sm_filter_chain* c, int filter) {
  if (!c || filter < 0 || filter >= (int)c->chain.filters.size()) return SM_ERR_BAD_ARGUMENT;
  return filter_configs_valid(c->chain.filters[filter]) ? 1 : 0;
}

int sm_filter_chain_set_option(sm_filter_chain* c, const char* name, const char* text) {
  if (!c || !name || !text) return SM_ERR_BAD_ARGUMENT;
  if (strcmp(name, "sample_seed") != 0) return chain_fail(c, SM_ERR_UNKNOWN_OPTION, "unknown chain option %s", name);
  c->chain.sample_seed = (uint32_t)strtoul(text, nullptr, 10);
  return SM_OK;
}

int sm_filter_chain_run_device(sm_filter_chain* c, const float* dev_points, int64_t n, int64_t stride_bytes,
                               float* dev_out, int64_t* m_out, int32_t* dev_inlier_index, void* cuda_stream) {
  if (!c || !m_out || n < 0 || n > (1 << 30) || stride_bytes < 20 || stride_bytes % 4 ||
      (n > 0 && (!dev_points || !dev_out)))
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(chain_device(c));
  const int rc = c->chain.run((const char*)dev_points, n, stride_bytes, dev_out, dev_inlier_index, m_out,
                              (cudaStream_t)cuda_stream);
  if (rc == SM_ERR_CHECK_FAILED)
    chain_fail(c, rc, "Check failed: %s", "an inverted BoundingBoxRemoval box or line.start[0] < line.end[0]");
  else if (rc == SM_ERR_BAD_ARGUMENT)
    chain_fail(c, rc, "%s", "a RangeImage or GroundRemoval2 grid size the chain cannot run");
  else if (rc == SM_ERR_CUDA)
    chain_fail(c, rc, "%s", last_cuda_error());
  return rc;
}

int sm_filter_chain_run(sm_filter_chain* c, const float* points, int64_t n, int64_t stride_bytes, float* out,
                        int64_t* m_out, int32_t* inlier_index) {
  if (!c || !m_out || n < 0 || n > (1 << 30) || stride_bytes < 20 || stride_bytes % 4 || (n > 0 && (!points || !out)))
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(chain_device(c));
  *m_out = 0;
  if (n == 0) return sm_filter_chain_run_device(c, nullptr, 0, stride_bytes, nullptr, m_out, nullptr, nullptr);
  if (!c->stream) SMB_CUDA_OK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  const size_t in_bytes = (size_t)n * (size_t)stride_bytes;
  SMB_RC(c->host_in.reserve(in_bytes));
  SMB_RC(c->host_out.reserve((size_t)n * 20));
  SMB_RC(c->host_idx.reserve((size_t)n * sizeof(int32_t)));
  SMB_CUDA_OK(cudaMemcpyAsync(c->host_in.p, points, in_bytes, cudaMemcpyHostToDevice, c->stream));
  SMB_RC(sm_filter_chain_run_device(c, (const float*)c->host_in.p, n, stride_bytes, (float*)c->host_out.p, m_out,
                                    (int32_t*)c->host_idx.p, c->stream));
  if (*m_out > 0) {
    SMB_CUDA_OK(cudaMemcpyAsync(out, c->host_out.p, (size_t)*m_out * 20, cudaMemcpyDeviceToHost, c->stream));
    if (inlier_index)
      SMB_CUDA_OK(cudaMemcpyAsync(inlier_index, c->host_idx.p, (size_t)*m_out * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                  c->stream));
    SMB_CUDA_OK(cudaStreamSynchronize(c->stream));
  }
  return SM_OK;
}

const char* sm_filter_chain_last_error(const sm_filter_chain* c) { return c ? c->error : ""; }

}  // extern "C"
