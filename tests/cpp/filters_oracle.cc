// CPU restatement of the reference's scan pre-processing filters (pre_processors/filter_*.cc), sequential and in the
// reference's order.  TEST INFRASTRUCTURE: the GPU filter chain (csrc/filters.cu) is compared against this, and this
// against the independent numpy restatement tests/pyref_filters.py.  Compiled with -ffp-contract=off.
//
//   Range               filter_range.cc:45-88
//   AxisRange           filter_axis_range.cc:41-102
//   BoundingBoxRemoval  filter_bounding_box.cc:49-83, common/bounding_box.cc:112-121
//   RandomSampler       filter_random_sample.cc:35-77 with the engine's deterministic stand-in for the mt19937 draw:
//                       keep iff fmix32(scan_index * 0x9E3779B9 + seed) <= rate * 2^32
//   RangeImage          filter_range_image.cc:82-141
//   GroundRemoval2      filter_ground_removal2.cc:127-414; FitLocalLine's colPivHouseholderQr().solve() is written out
//                       after Eigen/src/QR/ColPivHouseholderQR.h (computeInPlace, _solve_impl) with plain loops, as
//                       oracle/linalg.h does for FullPivHouseholderQR
// A float -> int conversion outside int's range is undefined; x86 gives INT_MIN there, which is what ToInt returns.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>
#include <utility>
#include <vector>

namespace {

enum Kind { kRange = 0, kAxisRange, kBoundingBoxRemoval, kRandomSampler, kRangeImage, kGroundRemoval2 };

struct Point { float x, y, z, intensity, factor; };

inline int ToInt(double q) { return (q > -2147483649.0 && q < 2147483648.0) ? static_cast<int>(q) : INT_MIN; }

inline uint32_t Fmix32(uint32_t h) {
  h ^= h >> 16; h *= 0x85EBCA6Bu; h ^= h >> 13; h *= 0xC2B2AE35u; h ^= h >> 16;
  return h;
}

// ---- ColPivHouseholderQR of an n x 2 matrix, column-major in qr, and the least-squares solve ---------------------------
void SolveColPivQr(std::vector<double> qr, std::vector<double> rhs, int rows, double* result2) {
  const int cols = 2;
  auto at = [&](int r, int c) -> double& { return qr[static_cast<size_t>(c) * rows + r]; };
  double norms_updated[2], norms_direct[2], h_coeffs[2];
  int transpositions[2];
  for (int k = 0; k < cols; ++k) {
    double sq = 0.0;
    for (int r = 0; r < rows; ++r) sq += at(r, k) * at(r, k);
    norms_direct[k] = std::sqrt(sq);
    norms_updated[k] = norms_direct[k];
  }
  const double epsilon = DBL_EPSILON;
  double max_norm = norms_updated[0];
  if (norms_updated[1] > max_norm) max_norm = norms_updated[1];
  const double threshold_helper = (max_norm * epsilon) * (max_norm * epsilon) / static_cast<double>(rows);
  const double norm_downdate_threshold = std::sqrt(epsilon);
  const int size = rows < cols ? rows : cols;
  int nonzero_pivots = size;
  for (int k = 0; k < size; ++k) {
    int biggest_col_index = k;
    for (int j = k + 1; j < cols; ++j)
      if (norms_updated[j] > norms_updated[biggest_col_index]) biggest_col_index = j;
    const double biggest_col_sq_norm = norms_updated[biggest_col_index] * norms_updated[biggest_col_index];
    if (nonzero_pivots == size && biggest_col_sq_norm < threshold_helper * static_cast<double>(rows - k))
      nonzero_pivots = k;
    transpositions[k] = biggest_col_index;
    if (k != biggest_col_index) {
      for (int r = 0; r < rows; ++r) std::swap(at(r, k), at(r, biggest_col_index));
      std::swap(norms_updated[k], norms_updated[biggest_col_index]);
      std::swap(norms_direct[k], norms_direct[biggest_col_index]);
    }
    // makeHouseholderInPlace on the tail of column k
    double tail_sq_norm = 0.0;
    for (int r = k + 1; r < rows; ++r) tail_sq_norm += at(r, k) * at(r, k);
    const double c0 = at(k, k);
    double beta, tau;
    if (tail_sq_norm <= DBL_MIN) {
      tau = 0.0;
      beta = c0;
      for (int r = k + 1; r < rows; ++r) at(r, k) = 0.0;
    } else {
      beta = std::sqrt(c0 * c0 + tail_sq_norm);
      if (c0 >= 0.0) beta = -beta;
      for (int r = k + 1; r < rows; ++r) at(r, k) = at(r, k) / (c0 - beta);
      tau = (beta - c0) / beta;
    }
    at(k, k) = beta;
    h_coeffs[k] = tau;
    // applyHouseholderOnTheLeft to the remaining columns
    for (int j = k + 1; j < cols; ++j) {
      if (rows - k == 1) {
        at(k, j) *= 1.0 - tau;
      } else if (tau != 0.0) {
        double tmp = 0.0;
        for (int r = k + 1; r < rows; ++r) tmp += at(r, k) * at(r, j);
        tmp += at(k, j);
        at(k, j) -= tau * tmp;
        for (int r = k + 1; r < rows; ++r) at(r, j) -= tmp * (tau * at(r, k));
      }
    }
    // update the norms of the remaining columns
    for (int j = k + 1; j < cols; ++j) {
      if (norms_updated[j] != 0.0) {
        double temp = std::fabs(at(k, j)) / norms_updated[j];
        temp = (1.0 + temp) * (1.0 - temp);
        temp = temp < 0.0 ? 0.0 : temp;
        const double ratio = norms_updated[j] / norms_direct[j];
        const double temp2 = temp * (ratio * ratio);
        if (temp2 <= norm_downdate_threshold) {
          double sq = 0.0;
          for (int r = k + 1; r < rows; ++r) sq += at(r, j) * at(r, j);
          norms_direct[j] = std::sqrt(sq);
          norms_updated[j] = norms_direct[j];
        } else {
          norms_updated[j] *= std::sqrt(temp);
        }
      }
    }
  }
  // _solve_impl: c = Q^T rhs, back substitution on the leading block, un-permute
  result2[0] = result2[1] = 0.0;
  if (nonzero_pivots == 0) return;
  for (int k = 0; k < nonzero_pivots; ++k) {
    if (rows - k == 1) {
      rhs[k] *= 1.0 - h_coeffs[k];
    } else if (h_coeffs[k] != 0.0) {
      double tmp = 0.0;
      for (int r = k + 1; r < rows; ++r) tmp += at(r, k) * rhs[r];
      tmp += rhs[k];
      rhs[k] -= h_coeffs[k] * tmp;
      for (int r = k + 1; r < rows; ++r) rhs[r] -= tmp * (h_coeffs[k] * at(r, k));
    }
  }
  for (int i = nonzero_pivots - 1; i >= 0; --i) {
    for (int j = i + 1; j < nonzero_pivots; ++j) rhs[i] -= rhs[j] * at(i, j);
    rhs[i] = rhs[i] / at(i, i);
  }
  int permutation[2] = {0, 1};
  for (int k = 0; k < size; ++k) std::swap(permutation[k], permutation[transpositions[k]]);
  for (int i = 0; i < nonzero_pivots; ++i) result2[permutation[i]] = rhs[i];
}

// ---- GroundRemoval2 (filter_ground_removal2.cc:127-414) ----------------------------------------------------------------
// Laid out as flat tables rather than the reference's per-cell containers: a cell id per point, one record per polar
// cell, and per sector the list of spans found.  The span search keeps a window [head, tail] over the sector's
// occupied cells in outward order: that is what the reference's growing and trimmed point list always is.
struct Gr2Params {
  float r_max, r_min, start_ground_height, long_line_threshold, max_long_line_height, max_start_height, max_error,
      max_slope, max_b, max_dist_to_line, search_angle;
  int bin_num, segment_num;
};
struct Span { float d_from, z_from, d_to, z_to; };       // one fitted ground line of a sector, inner end to outer end
struct Slope { float m, b; };
struct CellRecord { float low_d = 1.e6f, low_z = 1.e6f; uint32_t joined = 0; };

Gr2Params MakeGr2(const float* fp, const int* ip) {
  Gr2Params p;
  p.r_max = fp[0]; p.r_min = fp[1]; p.start_ground_height = fp[2]; p.long_line_threshold = fp[3];
  p.max_long_line_height = fp[4]; p.max_start_height = fp[5]; p.max_error = fp[6]; p.max_slope = fp[7]; p.max_b = fp[8];
  p.max_dist_to_line = fp[9]; p.search_angle = fp[10];
  p.bin_num = ip[0]; p.segment_num = ip[1];
  return p;
}

// sectors looked at on either side of a point's own (:340-341): the sector width is taken in double here, cast to float
int NeighbourReach(const Gr2Params& p) {
  const float width = static_cast<float>(M_PI * 2 / p.segment_num);
  return ToInt(p.search_angle / 180. * M_PI / width);
}

bool Gr2Usable(const Gr2Params& p) {
  if (p.bin_num <= 0 || p.segment_num <= 0) return false;
  const int reach = NeighbourReach(p);
  return reach >= 0 && reach < p.segment_num;
}

// :144-146, :164-186: planar range, sector and ring of one point, both indices clamped into the grid
void PolarCell(const Gr2Params& p, const Point& q, float* planar, int* sector, int* ring) {
  const float turn = static_cast<float>(M_PI * 2);
  const float sector_width = turn / static_cast<float>(p.segment_num);
  const float ring_width = (p.r_max - p.r_min) / static_cast<float>(p.bin_num);
  *planar = std::sqrt(q.x * q.x + q.y * q.y);
  float azimuth = std::atan2(q.y, q.x);
  if (azimuth < 0.f) azimuth += turn;
  const int s = ToInt(azimuth / sector_width), r = ToInt((*planar - p.r_min) / ring_width);
  *sector = s < 0 ? 0 : (s >= p.segment_num ? p.segment_num - 1 : s);
  *ring = r < 0 ? 0 : (r >= p.bin_num ? p.bin_num - 1 : r);
}

Slope FitSlope(const float* d, const float* z, int count) {   // :29-44
  std::vector<double> A(2 * static_cast<size_t>(count)), y(count);
  for (int i = 0; i < count; ++i) { A[i] = d[i]; A[count + i] = 1.0; y[i] = z[i]; }
  double mb[2];
  SolveColPivQr(A, y, count, mb);
  return Slope{static_cast<float>(mb[0]), static_cast<float>(mb[1])};
}

struct GroundModel {
  Gr2Params p;
  std::vector<int> cell_of;               // per point: sector * bin_num + ring
  std::vector<float> planar;              // per point
  std::vector<uint8_t> joined;            // per point: it entered its cell's member list (:204-208)
  std::vector<CellRecord> cells;
  std::vector<std::vector<Span>> spans;   // per sector
  bool inverted_span = false;             // the reference's CHECK at :403 would have fired

  // :195-209, points in input order: the cell's lowest point is replaced on a strictly lower z or while nothing has
  // joined; a point joins when it is at most 0.5 above the lowest point AS IT STANDS THEN
  void Bin(const Point* pts, int n) {
    cells.assign(static_cast<size_t>(p.bin_num) * p.segment_num, CellRecord());
    cell_of.resize(n); planar.resize(n); joined.assign(n, 0);
    for (int i = 0; i < n; ++i) {
      int sector, ring;
      PolarCell(p, pts[i], &planar[i], &sector, &ring);
      cell_of[i] = sector * p.bin_num + ring;
    }
    for (int i = 0; i < n; ++i) {
      CellRecord& c = cells[cell_of[i]];
      const float z = pts[i].z;
      if (c.joined == 0 || z < c.low_z) { c.low_d = planar[i]; c.low_z = z; }
      if (static_cast<double>(z) <= static_cast<double>(c.low_z) + 0.5) { joined[i] = 1; ++c.joined; }
    }
  }

  // :240-316 for one sector
  void SearchSpans(int sector) {
    std::vector<Span>& found = spans[sector];
    found.clear();
    std::vector<float> d, z;              // lowest points of the occupied cells, outward
    int first_ring = -1;
    for (int ring = 0; ring < p.bin_num; ++ring) {
      const CellRecord& c = cells[static_cast<size_t>(sector) * p.bin_num + ring];
      if (c.joined == 0) continue;
      if (first_ring < 0) first_ring = ring;
      d.push_back(c.low_d); z.push_back(c.low_z);
    }
    if (first_ring < 0 || first_ring >= p.bin_num - 1) return;   // :250: nothing beyond the first occupied ring
    const int total = static_cast<int>(d.size());
    int head = 0, tail = 0;               // the window under construction, inclusive
    Slope running{0.f, 0.f};              // the last fit made, accepted or not (:279)
    bool stretched = false;               // a gap of long_line_threshold or more was seen since the last break
    float floor_z = p.start_ground_height;
    auto close_window = [&]() {           // :287-292, :311-313: fit the window, record its span, return z at its outer end
      const Slope s = FitSlope(&d[head], &z[head], tail - head + 1);
      found.push_back(Span{d[head], s.m * d[head] + s.b, d[tail], s.m * d[tail] + s.b});
      return s.m * d[tail] + s.b;
    };
    int next = 1;
    while (next < total) {
      if (d[next] - d[tail] >= p.long_line_threshold) stretched = true;
      const int held = tail - head + 1;
      float predicted = FLT_MAX;
      if (stretched && held > 2) predicted = running.m * d[next] + running.b;
      if (held < 2) {                     // :300-309: a second point is taken only near the current floor
        if (!stretched && std::fabs(z[tail] - floor_z) < p.max_start_height) tail = next;
        else head = tail = next;
        ++next;
        continue;
      }
      running = FitSlope(&d[head], &z[head], next - head + 1);
      float worst = 0.f;
      for (int k = head; k <= next; ++k) {
        const float miss = std::fabs(running.m * d[k] + running.b - z[k]);
        if (miss > worst) worst = miss;
      }
      const bool rejected = worst > p.max_error || std::fabs(running.m) > p.max_slope ||
                            (stretched && std::fabs(predicted - z[next]) > p.max_long_line_height);
      if (!rejected) { tail = next++; continue; }
      if (held >= 3) floor_z = close_window();
      stretched = false;
      head = tail;                        // the outer point starts the next window; `next` is looked at again (:296-298)
    }
    if (tail - head + 1 > 2) close_window();
  }

  // :398-414: height gap of (d, z) to the LAST span whose range, widened by 0.1, holds d; -1 when none does
  float HeightGap(const std::vector<Span>& sector_spans, float d, float z) {
    const float slack = 0.1f;
    float gap = -1.f;
    for (const Span& s : sector_spans) {
      if (!(s.d_from < s.d_to)) { inverted_span = true; continue; }
      if (s.d_from - slack < d && s.d_to + slack > d) {
        const float rise = s.z_to - s.z_from, run = s.d_to - s.d_from;
        gap = std::fabs(z - ((d - s.d_from) / run * rise + s.z_from));
      }
    }
    return gap;
  }

  // :350-386 for one joined point: its own sector, then on "no span" the sectors +reach, -reach, ..., +1, -1 until one
  // answers with a positive gap; ground when 0 < gap <= max_dist_to_line
  bool IsGround(int i, float z, int reach) {
    const int own = cell_of[i] / p.bin_num;
    float gap = HeightGap(spans[own], planar[i], z);
    for (int step = reach; gap < 0.f && step > 0; --step) {
      for (int side = 0; side < 2; ++side) {
        int other = side == 0 ? own + step : own - step;
        if (other < 0) other += p.segment_num; else if (other >= p.segment_num) other -= p.segment_num;
        gap = HeightGap(spans[other], planar[i], z);
        if (gap > 0.f) break;
      }
      if (gap > 0.f) break;
    }
    return gap > 0.f && gap <= p.max_dist_to_line;
  }

  void Run(const Point* pts, int n, uint8_t* keep) {
    Bin(pts, n);
    spans.assign(p.segment_num, {});
    for (int s = 0; s < p.segment_num; ++s) SearchSpans(s);
    const int reach = NeighbourReach(p);
    for (int i = 0; i < n; ++i) keep[i] = (joined[i] && IsGround(i, pts[i].z, reach)) ? 0 : 1;
  }
};

// ---- RangeImage (filter_range_image.cc:89-126): the pixel of one point, false for its outlier branches ------------------
bool PixelOf(const float* fp, const int* ip, const Point& q, int* row, int* col) {
  const int rows = ip[0], cols = ip[1];
  const float az_step = static_cast<float>(M_PI * 2 / static_cast<float>(cols));
  const float el_step = static_cast<float>((fp[0] - fp[1]) / static_cast<float>(rows) / 180.f * M_PI);
  const double el_floor = fp[1] / 180.f * M_PI;
  const float x = q.x + fp[2], y = q.y + fp[3], z = q.z + fp[4];
  const float planar = std::sqrt(x * x + y * y);
  if (planar < 0.01f) return false;
  const float elevation = std::atan2(z, planar);
  const int r = ToInt((elevation - el_floor) / el_step);          // double arithmetic, truncated toward zero
  if (r < 0 || r >= rows) return false;
  float azimuth = std::atan2(y, x);
  if (azimuth < 0.f) azimuth = static_cast<float>(azimuth + M_PI * 2);
  long c = std::lround(azimuth / az_step);
  if (c >= cols) c -= cols;
  if (c < 0 || c >= cols) return false;
  *row = r; *col = static_cast<int>(c);
  return true;
}

}  // namespace

extern "C" {

// One filter over n packed records.  fp / ip: the filter's float / int parameters in the order of
// tests/oracle_filters.py PARAMS.  scan_index (RandomSampler; null = identity): each record's index in the scan handed
// to the chain.  keep: n flags.  Returns 0, -1 for a configuration the filter cannot run, -5 for a failed CHECK.
int sm_oracle_filter(int kind, const float* fp, const int* ip, uint32_t seed, const float* records, int64_t n,
                     const int32_t* scan_index, uint8_t* keep) {
  const Point* pts = reinterpret_cast<const Point*>(records);
  const int count = static_cast<int>(n);
  switch (kind) {
    case kRange:                  // filter_range.cc:59-68
      for (int i = 0; i < count; ++i) {
        const float r = std::sqrt(pts[i].x * pts[i].x + pts[i].y * pts[i].y + pts[i].z * pts[i].z);
        keep[i] = r >= fp[0] && r <= fp[1];
      }
      return 0;
    case kAxisRange: {            // filter_axis_range.cc:50-90; an axis outside 0..2 removes nothing
      const bool open = (fp[0] == -FLT_MAX && fp[1] == FLT_MAX) || ip[0] < 0 || ip[0] > 2;
      for (int i = 0; i < count; ++i) {
        const float v = open ? 0.f : (&pts[i].x)[ip[0]];
        keep[i] = open || !(v < fp[0] || v > fp[1]);
      }
      return 0;
    }
    case kBoundingBoxRemoval: {   // filter_bounding_box.cc:60-78, common/bounding_box.cc:112-121, compared in double
      const double lo[3] = {fp[0], fp[1], fp[2]}, hi[3] = {fp[3], fp[4], fp[5]};
      if (!(lo[0] < hi[0] && lo[1] < hi[1] && lo[2] < hi[2])) return -5;
      for (int i = 0; i < count; ++i) {
        bool inside = true;
        for (int a = 0; a < 3; ++a) {
          const double v = (&pts[i].x)[a];
          inside = inside && v >= lo[a] && v <= hi[a];
        }
        keep[i] = !inside;
      }
      return 0;
    }
    case kRandomSampler:          // filter_random_sample.cc:44-72 with the stand-in draw
      for (int i = 0; i < count; ++i) {
        const uint32_t index = scan_index ? static_cast<uint32_t>(scan_index[i]) : static_cast<uint32_t>(i);
        keep[i] = fp[0] > 0.999 || static_cast<double>(Fmix32(index * 0x9E3779B9u + seed)) <= fp[0] * 4294967296.0;
      }
      return 0;
    case kRangeImage: {           // filter_range_image.cc:72-74, :128-136: the first point to reach a pixel owns it
      if (ip[0] <= 0 || ip[1] <= 0) return -1;
      std::vector<uint8_t> taken(static_cast<size_t>(ip[0]) * ip[1], 0);
      for (int i = 0; i < count; ++i) {
        int row, col;
        keep[i] = 0;
        if (!PixelOf(fp, ip, pts[i], &row, &col)) continue;
        uint8_t& t = taken[static_cast<size_t>(row) * ip[1] + col];
        keep[i] = !t;
        t = 1;
      }
      return 0;
    }
    case kGroundRemoval2: {
      GroundModel g;
      g.p = MakeGr2(fp, ip);
      if (!Gr2Usable(g.p)) return -1;
      g.Run(pts, count, keep);
      return g.inverted_span ? -5 : 0;
    }
    default: return -1;
  }
}

// GroundRemoval2's intermediates, laid out as sm_debug_filter_ground_removal2 returns them
int sm_oracle_gr2_stages(const float* fp, const int* ip, const float* records, int64_t n, int32_t max_lines,
                         uint32_t* cell, uint8_t* member, uint32_t* cell_members, float* cell_min_2c, float* lines_4,
                         int32_t* n_lines, uint8_t* keep) {
  GroundModel g;
  g.p = MakeGr2(fp, ip);
  if (!Gr2Usable(g.p)) return -1;
  const int count = static_cast<int>(n);
  g.Run(reinterpret_cast<const Point*>(records), count, keep);
  for (int i = 0; i < count; ++i) { cell[i] = static_cast<uint32_t>(g.cell_of[i]); member[i] = g.joined[i]; }
  for (size_t c = 0; c < g.cells.size(); ++c) {
    cell_members[c] = g.cells[c].joined;
    cell_min_2c[2 * c] = g.cells[c].low_d;
    cell_min_2c[2 * c + 1] = g.cells[c].low_z;
  }
  for (int s = 0; s < g.p.segment_num; ++s) {
    n_lines[s] = static_cast<int32_t>(g.spans[s].size());
    for (int l = 0; l < n_lines[s] && l < max_lines; ++l) {
      const Span& sp = g.spans[s][l];
      float* out = lines_4 + 4 * (static_cast<size_t>(s) * max_lines + l);
      out[0] = sp.d_from; out[1] = sp.z_from; out[2] = sp.d_to; out[3] = sp.z_to;
    }
  }
  return g.inverted_span ? -5 : 0;
}

void sm_oracle_fit_line(const float* d, const float* z, int32_t n, float* m_b) {
  const Slope s = FitSlope(d, z, n);
  m_b[0] = s.m; m_b[1] = s.b;
}

// per record: RangeImage's (row, col) or (-1, -1)
void sm_oracle_pixels(const float* fp, const int* ip, const float* records, int64_t n, int32_t* row_col) {
  const Point* pts = reinterpret_cast<const Point*>(records);
  for (int64_t i = 0; i < n; ++i)
    if (!PixelOf(fp, ip, pts[i], &row_col[2 * i], &row_col[2 * i + 1])) row_col[2 * i] = row_col[2 * i + 1] = -1;
}

// per record: GroundRemoval2's (segment, bin) and range
void sm_oracle_cells(const float* fp, const int* ip, const float* records, int64_t n, int32_t* s_b, float* range) {
  const Point* pts = reinterpret_cast<const Point*>(records);
  const Gr2Params p = MakeGr2(fp, ip);
  for (int64_t i = 0; i < n; ++i) PolarCell(p, pts[i], &range[i], &s_b[2 * i], &s_b[2 * i + 1]);
}

float sm_oracle_vertical_distance(const float* lines_4l, int32_t n_lines, float d, float z) {
  GroundModel g;
  std::vector<Span> spans(n_lines);
  for (int l = 0; l < n_lines; ++l)
    spans[l] = Span{lines_4l[4 * l], lines_4l[4 * l + 1], lines_4l[4 * l + 2], lines_4l[4 * l + 3]};
  return g.HeightGap(spans, d, z);
}

}  // extern "C"
