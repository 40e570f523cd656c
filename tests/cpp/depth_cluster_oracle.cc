// Sequential CPU model of RangeImage::DepthCluster (pre_processors/filter_range_image.cc: the projection of Filter,
// :82-141, then DepthCluster, :143-173, with LabelOneComponent, :245-309).  TEST INFRASTRUCTURE: the device path
// (csrc/depth_cluster.cu) is compared against this, and this against the independent numpy model
// tests/pyref_depth_cluster.py.  Compiled with -ffp-contract=off.
//
// What it keeps from the reference, because the order of the output depends on it: a FIFO (std::queue) per component,
// a cell taken when it is popped for the first time, a neighbour pushed whenever a popped cell finds it free and
// joined to it (so a cell can sit in the queue more than once), components numbered in row-major order of their first
// cell, and the reference's mix of float and double in the pitches and the angle test.
// Parameters as tests/oracle_filters.py packs a RangeImage: fp = top_angle, btm_angle, offset_x/y/z; ip = rows, cols.
#include <climits>
#include <cmath>
#include <cstdint>
#include <map>
#include <queue>
#include <utility>
#include <vector>

namespace {

struct Record { float x, y, z, intensity, factor; };

inline int ToInt(double q) { return (q > -2147483649.0 && q < 2147483648.0) ? static_cast<int>(q) : INT_MIN; }

// the neighbour steps (row, column) in the order the reference visits them (:38-43)
constexpr int kStepRow[6] = {0, 0, 0, 0, 1, -1};
constexpr int kStepCol[6] = {1, -1, 2, -2, 0, 0};
constexpr uint32_t kMinPoints = 20;                      // smallest cluster that is reported (:306)
const float kJoinAngle = 10 / 180. * M_PI;               // the 10 degree criterion, as a float (filter_range_image.h:101)

struct Params {
  int rows, cols;
  float top, bottom, shift[3];
};

Params Unpack(const float* fp, const int* ip) { return Params{ip[0], ip[1], fp[0], fp[1], {fp[2], fp[3], fp[4]}}; }

// angular pitch between neighbouring columns (float of a double quotient) and, for the segmentation only, between
// neighbouring rows: (top - bottom) / rows in float, then the double 180. and pi (:255-259)
float ColumnPitch(const Params& p) { return static_cast<float>(M_PI * 2 / static_cast<float>(p.cols)); }
float RowPitchOfSegmentation(const Params& p) {
  const float degrees = (p.top - p.bottom) / static_cast<float>(p.rows);
  return static_cast<float>(degrees / 180. * M_PI);
}

// Bogoslavskyi-Stachniss: the angle at the nearer point between the laser ray and the line to the farther point
bool Joined(float u, float v, float pitch) {
  const float farther = u < v ? v : u;    // std::max(u, v)
  const float nearer = v < u ? v : u;     // std::min(u, v)
  const float angle = std::atan2(nearer * std::sin(pitch), farther - nearer * std::cos(pitch));
  return angle > kJoinAngle;
}

struct Sheet {
  Params p;
  std::vector<float> depth;           // range of the cell's point, 0 = empty
  std::vector<int32_t> source;        // input index of the cell's point, -1 = empty
  std::vector<uint32_t> tag;          // component number, 0 = not taken yet
  std::vector<int32_t> ring;          // queue generation at which the cell was taken (for the stage tests)
  std::map<uint32_t, std::vector<int>> reported;   // component number -> input indices in pop order
  const uint8_t* given_edges = nullptr;            // when set, bit k of a cell replaces Joined along step k

  explicit Sheet(const Params& params)
      : p(params), depth(static_cast<size_t>(p.rows) * p.cols, 0.f), source(depth.size(), -1), tag(depth.size(), 0),
        ring(depth.size(), -1) {}

  bool Empty(int cell) const { return depth[cell] < 1.e-6; }

  // the projection of Filter: the first record in input order that reaches a cell owns it
  void Project(const Record* cloud, int64_t n) {
    const float az_step = ColumnPitch(p);
    const float el_step = static_cast<float>((p.top - p.bottom) / static_cast<float>(p.rows) / 180.f * M_PI);
    const double el_floor = p.bottom / 180.f * M_PI;
    for (int64_t i = 0; i < n; ++i) {
      const float x = cloud[i].x + p.shift[0], y = cloud[i].y + p.shift[1], z = cloud[i].z + p.shift[2];
      const float planar = std::sqrt(x * x + y * y);
      if (planar < 0.01f) continue;
      const float elevation = std::atan2(z, planar);
      const int row = ToInt((elevation - el_floor) / el_step);
      if (row < 0 || row >= p.rows) continue;
      float azimuth = std::atan2(y, x);
      if (azimuth < 0.f) azimuth = static_cast<float>(azimuth + M_PI * 2);
      long col = std::lround(azimuth / az_step);
      if (col >= p.cols) col -= p.cols;
      if (col < 0 || col >= p.cols) continue;
      const int cell = row * p.cols + static_cast<int>(col);
      if (!Empty(cell)) continue;
      depth[cell] = std::sqrt(x * x + y * y + z * z);
      source[cell] = static_cast<int32_t>(i);
    }
  }

  // the cell one step k away, -1 past the first or last row; columns wrap around once
  int Across(int cell, int k) const {
    const int row = cell / p.cols + kStepRow[k];
    if (row < 0 || row >= p.rows) return -1;
    int col = cell % p.cols + kStepCol[k];
    if (col < 0) col += p.cols;
    else if (col >= p.cols) col -= p.cols;
    return row * p.cols + col;
  }

  bool Linked(int cell, int k, int other) const {
    if (given_edges) return (given_edges[cell] >> k) & 1;
    return Joined(depth[cell], depth[other], kStepRow[k] == 0 ? ColumnPitch(p) : RowPitchOfSegmentation(p));
  }

  void Grow(uint32_t number, int seed) {
    std::queue<std::pair<int, int32_t>> fifo;        // (cell, generation)
    std::vector<int> members;
    fifo.emplace(seed, 0);
    while (!fifo.empty()) {
      const int cell = fifo.front().first;
      const int32_t generation = fifo.front().second;
      fifo.pop();
      if (Empty(cell) || tag[cell] != 0) continue;   // queued twice and already taken
      tag[cell] = number;
      ring[cell] = generation;
      members.push_back(source[cell]);
      for (int k = 0; k < 6; ++k) {
        const int other = Across(cell, k);
        if (other < 0 || Empty(other) || tag[other] != 0) continue;
        if (Linked(cell, k, other)) fifo.emplace(other, generation + 1);
      }
    }
    if (members.size() >= kMinPoints) reported[number] = std::move(members);
  }

  void Segment() {
    uint32_t next = 1;
    for (int cell = 0; cell < static_cast<int>(depth.size()); ++cell)
      if (!Empty(cell) && tag[cell] == 0) Grow(next++, cell);
  }

  // the labelled cloud in ascending component number, then the per-cell state; returns the number of components
  int64_t Write(const Record* cloud, float* xyz, uint32_t* label, int32_t* index, int64_t* m, float* depth_out,
                int32_t* source_out, uint32_t* tag_out, int32_t* ring_out) const {
    int64_t j = 0;
    for (const auto& entry : reported)
      for (int i : entry.second) {
        xyz[3 * j] = cloud[i].x; xyz[3 * j + 1] = cloud[i].y; xyz[3 * j + 2] = cloud[i].z;
        label[j] = entry.first;
        index[j] = i;
        ++j;
      }
    *m = j;
    uint32_t highest = 0;
    for (size_t c = 0; c < depth.size(); ++c) {
      if (depth_out) depth_out[c] = depth[c];
      if (source_out) source_out[c] = source[c];
      tag_out[c] = tag[c];
      ring_out[c] = ring[c];
      if (tag[c] > highest) highest = tag[c];
    }
    return highest;
  }
};

}  // namespace

extern "C" {

// Filter's projection + DepthCluster.  Outputs: the labelled cloud (capacity n), then per cell the range, the owning
// input index (-1 empty), the label (0 empty) and the queue generation (of every component, dropped ones too).
// Returns the number of components, -1 for a grid the reference cannot run (rows <= 0, cols < 2), -5 for an empty
// cloud (the reference's CHECK that it has an input cloud).
int64_t sm_oracle_depth_cluster(const float* fp, const int* ip, const float* records, int64_t n, float* out_xyz,
                                uint32_t* out_label, int32_t* out_index, int64_t* m, float* image, int32_t* owner,
                                uint32_t* pixel_label, int32_t* level) {
  if (n == 0) return -5;
  if (ip[0] <= 0 || ip[1] < 2) return -1;
  const Record* cloud = reinterpret_cast<const Record*>(records);
  Sheet sheet(Unpack(fp, ip));
  sheet.Project(cloud, n);
  sheet.Segment();
  return sheet.Write(cloud, out_xyz, out_label, out_index, m, image, owner, pixel_label, level);
}

// DepthCluster over a given image (ranges, owners) and edge mask (bit k: an edge along step k), as the device
// computed them: the labelling and the visiting order alone.
int64_t sm_oracle_depth_cluster_from(int V, int H, const float* image, const int32_t* owner, const uint8_t* mask,
                                     const float* records, float* out_xyz, uint32_t* out_label, int32_t* out_index,
                                     int64_t* m, uint32_t* pixel_label, int32_t* level) {
  Sheet sheet(Params{V, H, 0.f, 0.f, {0.f, 0.f, 0.f}});
  sheet.depth.assign(image, image + sheet.depth.size());
  sheet.source.assign(owner, owner + sheet.depth.size());
  sheet.given_edges = mask;
  sheet.Segment();
  return sheet.Write(reinterpret_cast<const Record*>(records), out_xyz, out_label, out_index, m, nullptr, nullptr,
                     pixel_label, level);
}

// the angle test for pairs of ranges a[i], b[i] along step k[i]
void sm_oracle_depth_edge(const float* fp, const int* ip, const float* a, const float* b, const int32_t* k, int64_t n,
                          uint8_t* edge) {
  const Params p = Unpack(fp, ip);
  const float column = ColumnPitch(p), row = RowPitchOfSegmentation(p);
  for (int64_t i = 0; i < n; ++i) edge[i] = Joined(a[i], b[i], kStepRow[k[i]] == 0 ? column : row) ? 1 : 0;
}

}  // extern "C"
