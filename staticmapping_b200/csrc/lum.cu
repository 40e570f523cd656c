// registrator::MultiviewRegistratorLumPcl on the device: PCL's Lu-Milios multi-view alignment (pcl::registration::LUM,
// PCL 1.8.1, restated from upstream: lum_host.h) over the frames of a MultiviewInterface, with AlignAll's five rounds
// of addPointCloud / setCorrespondences / compute.  See DESIGN.md section 4m.
//
//   transform  one launch: every frame's records by its Matrix4f pose (lum_transform), packed xyz.
//   trees      per target frame i >= 1: its finite points compacted in input order (compact.cuh), a FloatTree.
//   search     one launch over every pair (j, i), j < i: for each finite point of frame j, knn1 (eps = 0) on frame i's
//              tree, then the smallest index among the points at exactly that distance (lum_nearest_min_id); kept iff
//              d2 <= 0.25^2.  Then one ordered compaction of all pairs: each pair's list ascending in query index, the
//              pairs in the reference's loop order.  Read back: the per-pair counts; a pair with more than 2 is an edge.
//   compute    per LUM iteration, over all edges' correspondences: the 15 terms of M'M / M'Z (and the pair count) into
//              per-edge signed exact bins, one block per edge to finish them (rounded once to float) and to solve D in
//              double; the s^2 terms likewise; cinv / cinvd read back.  The host assembles G and B, solves the
//              vertices joined to vertex 0 with a double column-pivoted QR, updates the poses and tests convergence.
//   output     one launch: each vertex i < N's cloud (frame f(i) transformed) moved by getTransformation(pose_i),
//              whole records in vertex order.
// Compiled with -fmad=false.
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/sm_b200.h"
#include "../../include/sm_b200_debug.h"
#include "common.cuh"
#include "compact.cuh"
#include "icp_dev.cuh"
#include "kernels.h"
#include "lum_host.h"
#include "reduce.cuh"

namespace smb {
namespace {

constexpr int kLumMaxFrames = 64;
constexpr int64_t kLumMaxPoints = (int64_t)1 << 20;
constexpr int kLumThreads = 256;
constexpr int kLumChunk = kLumThreads * 8;             // correspondences per block of the edge passes
constexpr int kLumEdgeSums = kLumTerms * kExactSignedBins;

struct LumTree {
  const KdNode* nodes;
  const BucketPoint* bpts;
  const uint32_t* map;     // packed position -> index in the frame
  int nf;
  int pad;
};

// per edge: the vertices and frames of its two ends and its correspondence list
struct LumEdgeDev {
  int s, t, fs, ft;
  int64_t first;
  int count;
  int pad;
};

// per edge and iteration (trace layout of sm_debug_lum_trace_get, after s, t)
struct LumEdgeOut {
  float pairs;             // finite pairs
  float S[kLumTerms];
  float D[6];
  float ss;
  float cinv[36];
  float cinvd[6];
  float MM[36];
  float MZ[6];
};
constexpr int kLumTraceEdge = 2 + 1 + kLumTerms + 6 + 1 + 36 + 6;   // s, t, then LumEdgeOut up to cinvd

__global__ void __launch_bounds__(kLumThreads)
lum_transform_kernel(const char* __restrict__ rec, int64_t stride, const int64_t* __restrict__ off,
                     const int64_t* __restrict__ cnt, const float* __restrict__ T12, float* __restrict__ xyz) {
  const int f = blockIdx.y;
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= cnt[f]) return;
  const int64_t g = off[f] + q;
  lum_transform(T12 + 12 * f, reinterpret_cast<const float*>(rec + g * stride), xyz + 3 * g);
}

__global__ void __launch_bounds__(kCompactThreads)
lum_finite_count_kernel(const float* __restrict__ xyz, int n, uint32_t* __restrict__ tile_cnt) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r)
    if (base + r < n && lum_finite3(xyz + 3 * (int64_t)(base + r))) ++c;
  tile_count_store(c, tile_cnt);
}

__global__ void __launch_bounds__(kCompactThreads)
lum_finite_pack_kernel(const float* __restrict__ xyz, int n, const uint32_t* __restrict__ tile_off,
                       float* __restrict__ packed, uint32_t* __restrict__ map) {
  const int base = blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  bool f[kCompactItems];
  for (int r = 0; r < kCompactItems; ++r) {
    f[r] = base + r < n && lum_finite3(xyz + 3 * (int64_t)(base + r));
    c += f[r] ? 1u : 0u;
  }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r) {
    if (!f[r]) continue;
    const float* p = xyz + 3 * (int64_t)(base + r);
    packed[3 * (int64_t)pos] = p[0]; packed[3 * (int64_t)pos + 1] = p[1]; packed[3 * (int64_t)pos + 2] = p[2];
    map[pos] = (uint32_t)(base + r);
    ++pos;
  }
}

// The smallest bucket id among the tree's points at exactly d2 = head from q (knn1's squared distance, formed as
// scan_leaf forms it).  Every subtree whose cut lies within sqrt(head) of q is visited: a point across a cut is at
// least |q - cut| away, and rounding is monotone, so no point at d2 = head is skipped.
__device__ int lum_nearest_min_id(const KdNode* __restrict__ nodes, const BucketPoint* __restrict__ bpts, double qx,
                                  double qy, double qz, double head, int best_id) {
  int stack[dev::kMaxStack];
  int sp = 0;
  stack[sp++] = 0;
  while (sp > 0) {
    int idx = stack[--sp];
    KdNode nd = dev::load_node(nodes, idx);
    int guard = 0;
    while (nd.dim != 3 && ++guard < 64) {
      const double q = nd.dim == 0 ? qx : (nd.dim == 1 ? qy : qz);
      const int right = q > nd.cut ? 1 : 0;
      const double off = dsub(q, nd.cut);
      if (dmul(off, off) <= head && sp < dev::kMaxStack) stack[sp++] = dev::child_idx(idx, 1 - right);
      idx = dev::child_idx(idx, right);
      nd = dev::load_node(nodes, idx);
    }
    if (nd.dim != 3) continue;
    const long long packed = __double_as_longlong(nd.cut);
    const int first = (int)(packed & 0xffffffffll), count = (int)(packed >> 32);
    for (int k = 0; k < count; ++k) {
      const BucketPoint p = bpts[first + k];
      const double dx = dsub(qx, p.x), dy = dsub(qy, p.y), dz = dsub(qz, p.z);
      const double d = dadd(dadd(dmul(dx, dx), dmul(dy, dy)), dmul(dz, dz));
      if (d == head && (int)p.id < best_id) best_id = (int)p.id;
    }
  }
  return best_id;
}

// qm[pair_off[p] + q] = {q, match in frame i or -1} for the points q of frame j of pair p = (j, i)
__global__ void __launch_bounds__(kLumThreads)
lum_search_kernel(const float* __restrict__ xyz, const int64_t* __restrict__ off, const int64_t* __restrict__ cnt,
                  const LumTree* __restrict__ trees, const int2* __restrict__ pairs,
                  const int64_t* __restrict__ pair_off, int2* __restrict__ qm, uint32_t* __restrict__ pair_cnt) {
  const int p = blockIdx.y;
  const int j = pairs[p].x, i = pairs[p].y;
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int m = -1;
  const bool live = q < cnt[j];
  if (live) {
    const float* pq = xyz + 3 * (off[j] + q);
    const LumTree t = trees[i];
    if (t.nf > 0 && lum_finite3(pq)) {
      const double qx = pq[0], qy = pq[1], qz = pq[2];
      int slot; double d2;
      dev::knn1(t.nodes, t.bpts, qx, qy, qz, 1.0, slot, d2);
      if (slot >= 0 && d2 <= (double)kLumMaxDistance * (double)kLumMaxDistance) {
        const int id = lum_nearest_min_id(t.nodes, t.bpts, qx, qy, qz, d2, (int)t.bpts[slot].id);
        m = (int)t.map[id];
      }
    }
    qm[pair_off[p] + q] = make_int2((int)q, m);
  }
  const uint32_t b = __ballot_sync(0xffffffffu, m >= 0);
  if ((threadIdx.x & 31) == 0 && b) atomicAdd(&pair_cnt[p], (uint32_t)__popc(b));
}

__global__ void __launch_bounds__(kCompactThreads)
lum_match_count_kernel(const int2* __restrict__ qm, int64_t n, uint32_t* __restrict__ tile_cnt) {
  const int64_t base = (int64_t)blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r)
    if (base + r < n && qm[base + r].y >= 0) ++c;
  tile_count_store(c, tile_cnt);
}

__global__ void __launch_bounds__(kCompactThreads)
lum_match_scatter_kernel(const int2* __restrict__ qm, int64_t n, const uint32_t* __restrict__ tile_off,
                         int2* __restrict__ list) {
  const int64_t base = (int64_t)blockIdx.x * kCompactTile + threadIdx.x * kCompactItems;
  int2 v[kCompactItems];
  uint32_t c = 0;
  for (int r = 0; r < kCompactItems; ++r) {
    v[r] = base + r < n ? qm[base + r] : make_int2(0, -1);
    c += v[r].y >= 0 ? 1u : 0u;
  }
  uint32_t pos = tile_exclusive(c, tile_off);
  for (int r = 0; r < kCompactItems; ++r)
    if (v[r].y >= 0) list[pos++] = v[r];
}

// the pair (a, d) of correspondence k of edge E under the vertex matrices vT; false when it is skipped
__device__ __forceinline__ bool lum_edge_pair(const LumEdgeDev& E, const int2* __restrict__ list,
                                              const float* __restrict__ xyz, const int64_t* __restrict__ off,
                                              const float* __restrict__ vT, int64_t k, float* a, float* d) {
  const int2 c = list[E.first + k];
  float Ts[12], Tt[12], ps[3], pt[3];
  for (int r = 0; r < 12; ++r) { Ts[r] = vT[12 * E.s + r]; Tt[r] = vT[12 * E.t + r]; }
  for (int r = 0; r < 3; ++r) {
    ps[r] = xyz[3 * (off[E.fs] + c.x) + r];
    pt[r] = xyz[3 * (off[E.ft] + c.y) + r];
  }
  return lum_pair(Ts, Tt, ps, pt, a, d);
}

// pass 1: the 15 terms of every finite pair into bins[edge][term][kExactSignedBins], the pairs into pairs[edge]
__global__ void __launch_bounds__(kLumThreads)
lum_sums_kernel(const int2* __restrict__ chunks, const LumEdgeDev* __restrict__ edges, const int2* __restrict__ list,
                const float* __restrict__ xyz, const int64_t* __restrict__ off, const float* __restrict__ vT,
                unsigned long long* __restrict__ bins, uint32_t* __restrict__ pairs) {
  __shared__ unsigned long long s[kLumEdgeSums];
  __shared__ uint32_t ws[kLumThreads / 32][1];
  for (int b = threadIdx.x; b < kLumEdgeSums; b += blockDim.x) s[b] = 0ull;
  __syncthreads();
  const int e = chunks[blockIdx.x].x;
  const LumEdgeDev E = edges[e];
  const int64_t begin = chunks[blockIdx.x].y, end = min((int64_t)E.count, begin + kLumChunk);
  uint32_t c = 0;
  for (int64_t k = begin + threadIdx.x; k < end; k += blockDim.x) {
    float a[3], d[3], t[kLumTerms];
    if (!lum_edge_pair(E, list, xyz, off, vT, k, a, d)) continue;
    ++c;
    lum_pair_terms(a, d, t);
    for (int r = 0; r < kLumTerms; ++r) {
      int bin; int64_t m;
      exact_bin_signed(t[r], &bin, &m);
      if (m) atomicAdd(&s[r * kExactSignedBins + bin], (unsigned long long)m);
    }
  }
  const uint32_t tot = block_sum<1, kLumThreads>(&c, ws);
  if (threadIdx.x == 0 && tot) atomicAdd(&pairs[e], tot);
  __syncthreads();
  for (int b = threadIdx.x; b < kLumEdgeSums; b += blockDim.x)
    if (s[b]) atomicAdd(&bins[(int64_t)e * kLumEdgeSums + b], s[b]);
}

// one block per edge: the 15 sums rounded once to float, M'M, M'Z and D (double inverse)
__global__ void __launch_bounds__(32)
lum_sums_finish_kernel(const unsigned long long* __restrict__ bins, const uint32_t* __restrict__ pairs,
                       LumEdgeOut* __restrict__ out) {
  __shared__ uint64_t limb[kLumTerms][2][kExactLimbs];
  __shared__ float S[kLumTerms];
  const int e = blockIdx.x;
  const int r = threadIdx.x;
  if (r < kLumTerms)
    S[r] = exact_finish_float(reinterpret_cast<const int64_t*>(bins) + (int64_t)e * kLumEdgeSums + r * kExactSignedBins,
                              limb[r][0], limb[r][1]);
  __syncthreads();
  if (r != 0) return;
  LumEdgeOut& o = out[e];
  const int count = (int)pairs[e];
  o.pairs = (float)count;
  for (int k = 0; k < kLumTerms; ++k) o.S[k] = S[k];
  lum_mm_mz(S, count, o.MM, o.MZ);
  if (count < 3) { for (int k = 0; k < 6; ++k) o.D[k] = 0.f; return; }
  lum_edge_d<double>(o.MM, o.MZ, o.D);
}

// pass 2: the s^2 term of every finite pair of the edges with 3 or more into bins[edge][kExactSignedBins]
__global__ void __launch_bounds__(kLumThreads)
lum_ss_kernel(const int2* __restrict__ chunks, const LumEdgeDev* __restrict__ edges, const int2* __restrict__ list,
              const float* __restrict__ xyz, const int64_t* __restrict__ off, const float* __restrict__ vT,
              const LumEdgeOut* __restrict__ eo, unsigned long long* __restrict__ bins) {
  __shared__ unsigned long long s[kExactSignedBins];
  for (int b = threadIdx.x; b < kExactSignedBins; b += blockDim.x) s[b] = 0ull;
  __syncthreads();
  const int e = chunks[blockIdx.x].x;
  const LumEdgeDev E = edges[e];
  const int64_t begin = chunks[blockIdx.x].y, end = min((int64_t)E.count, begin + kLumChunk);
  if (eo[e].pairs >= 3.f) {
    float D[6];
    for (int k = 0; k < 6; ++k) D[k] = eo[e].D[k];
    for (int64_t k = begin + threadIdx.x; k < end; k += blockDim.x) {
      float a[3], d[3];
      if (!lum_edge_pair(E, list, xyz, off, vT, k, a, d)) continue;
      int bin; int64_t m;
      exact_bin_signed(lum_ss_term(a, d, D), &bin, &m);
      if (m) atomicAdd(&s[bin], (unsigned long long)m);
    }
  }
  __syncthreads();
  for (int b = threadIdx.x; b < kExactSignedBins; b += blockDim.x)
    if (s[b]) atomicAdd(&bins[(int64_t)e * kExactSignedBins + b], s[b]);
}

__global__ void __launch_bounds__(32)
lum_ss_finish_kernel(const unsigned long long* __restrict__ bins, LumEdgeOut* __restrict__ out) {
  __shared__ uint64_t limb[2][kExactLimbs];
  if (threadIdx.x != 0) return;
  LumEdgeOut& o = out[blockIdx.x];
  if (o.pairs < 3.f) {
    o.ss = 0.f;
    for (int k = 0; k < 36; ++k) o.cinv[k] = 0.f;
    for (int k = 0; k < 6; ++k) o.cinvd[k] = 0.f;
    return;
  }
  o.ss = exact_finish_float(reinterpret_cast<const int64_t*>(bins) + (int64_t)blockIdx.x * kExactSignedBins, limb[0],
                            limb[1]);
  lum_edge_finish(o.MM, o.MZ, o.ss, o.cinv, o.cinvd);
}

// vertex v < N of the output: frame vf[v]'s records, xyz = vertex matrix v applied to the frame's transformed xyz
__global__ void __launch_bounds__(kLumThreads)
lum_output_kernel(const char* __restrict__ rec, int64_t stride, const int64_t* __restrict__ off,
                  const int64_t* __restrict__ cnt, const int* __restrict__ vf, const int64_t* __restrict__ out_off,
                  const float* __restrict__ vT, const float* __restrict__ xyz, char* __restrict__ out) {
  const int v = blockIdx.y, f = vf[v];
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= cnt[f]) return;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(rec + (off[f] + q) * stride);
  uint32_t* dst = reinterpret_cast<uint32_t*>(out + (out_off[v] + q) * stride);
  for (int64_t w = 3; w < stride / 4; ++w) dst[w] = src[w];
  float p[3];
  lum_transform(vT + 12 * v, xyz + 3 * (off[f] + q), p);
  float* d = reinterpret_cast<float*>(dst);
  d[0] = p[0]; d[1] = p[1]; d[2] = p[2];
}

}  // namespace
}  // namespace smb

// ---- C handle -----------------------------------------------------------------------------------------------------
using namespace smb;

struct sm_lum {
  int device;
  cudaStream_t stream = nullptr;
  char error[256] = {0};
  int64_t stride = 0;                         // fixed by the first cloud
  std::vector<std::vector<char>> frames;      // the records of each frame, as added
  std::vector<float> frame_pose;              // 16 floats per frame, column-major
  std::vector<int> vertex_frame;              // the frame whose transformed cloud vertex k holds
  std::vector<float> poses;                   // 6 per vertex
  // the pairs of the last AlignAll: (j, i) in loop order, their counts and list offsets
  std::vector<int2> pairs;
  std::vector<uint32_t> pair_cnt;
  std::vector<int64_t> pair_first;
  DevBuf rec, off, cnt, T12, xyz, packed, map, tile_cnt, trees_d, pairs_d, pair_off_d, pair_cnt_d, qm, list, kdws,
      edges_d, chunks_d, vT, bins, ebins, epairs, eout, vf_d, out_off_d, out;
  std::vector<FloatTree> trees;
  bool trace_on = false;
  struct Iter {
    int n;
    std::vector<float> edges;     // kLumTraceEdge floats per edge
    std::vector<double> X;
    std::vector<float> poses;
    double sum;
  };
  std::vector<Iter> trace;

  explicit sm_lum(int d) : device(d) {}
  ~sm_lum() { if (stream) cudaStreamDestroy(stream); }
  __attribute__((format(printf, 3, 4))) int fail(int rc, const char* fmt, ...) {
    va_list args;
    va_start(args, fmt);
    vsnprintf(error, sizeof(error), fmt, args);
    va_end(args);
    return rc;
  }
  int cuda_fail(int rc) { return rc == SM_ERR_CUDA ? fail(rc, "%s", last_cuda_error()) : rc; }
  int align(float* out_host, int64_t capacity, int64_t* m_out);
  int compute(int N, const std::vector<LumEdgeDev>& edges, int64_t T);
};

namespace {

int lum_use_device(sm_lum* h) {
  const int rc = select_device(h->device);
  if (rc == SM_ERR_NO_DEVICE) return h->fail(rc, "no CUDA device: MultiviewRegistratorLumPcl has no CPU fallback");
  if (rc == SM_ERR_BAD_ARGUMENT) return h->fail(rc, "device %d is out of range", h->device);
  return h->cuda_fail(rc);
}

template <typename V>
int upload(DevBuf& b, const std::vector<V>& v, cudaStream_t s) {
  SMB_RC(b.reserve(std::max<size_t>(v.size() * sizeof(V), 16)));
  if (!v.empty()) SMB_CUDA_OK(cudaMemcpyAsync(b.p, v.data(), v.size() * sizeof(V), cudaMemcpyHostToDevice, s));
  return 0;
}

}  // namespace

// LUM::compute over the current graph: up to kLumIterations of the edge passes and the host solve
int sm_lum::compute(int N, const std::vector<LumEdgeDev>& edges, int64_t T) {
  const int n = (int)vertex_frame.size();
  if (n < 2) return SM_OK;
  const int E = (int)edges.size();
  std::vector<int2> chunks;
  for (int e = 0; e < E; ++e)
    for (int64_t b = 0; b < edges[e].count; b += kLumChunk) chunks.push_back(make_int2(e, (int)b));
  SMB_RC(upload(chunks_d, chunks, stream));
  SMB_RC(bins.reserve((size_t)std::max(E, 1) * kLumEdgeSums * sizeof(uint64_t)));
  SMB_RC(ebins.reserve((size_t)std::max(E, 1) * kExactSignedBins * sizeof(uint64_t)));
  SMB_RC(epairs.reserve((size_t)std::max(E, 1) * sizeof(uint32_t)));
  SMB_RC(eout.reserve((size_t)std::max(E, 1) * sizeof(LumEdgeOut)));
  std::vector<LumEdgeOut> eo(E);
  std::vector<float> mats((size_t)12 * N);
  for (int it = 0; it < kLumIterations; ++it) {
    if (E > 0) {
      for (int v = 0; v < N; ++v) lum_pose_matrix(&poses[6 * v], &mats[12 * v]);
      SMB_RC(upload(vT, mats, stream));
      SMB_CUDA_OK(cudaMemsetAsync(bins.p, 0, (size_t)E * kLumEdgeSums * sizeof(uint64_t), stream));
      SMB_CUDA_OK(cudaMemsetAsync(ebins.p, 0, (size_t)E * kExactSignedBins * sizeof(uint64_t), stream));
      SMB_CUDA_OK(cudaMemsetAsync(epairs.p, 0, (size_t)E * sizeof(uint32_t), stream));
      if (!chunks.empty())
        lum_sums_kernel<<<(unsigned)chunks.size(), kLumThreads, 0, stream>>>(
            (const int2*)chunks_d.p, (const LumEdgeDev*)edges_d.p, (const int2*)list.p, (const float*)xyz.p,
            (const int64_t*)off.p, (const float*)vT.p, (unsigned long long*)bins.p, (uint32_t*)epairs.p);
      lum_sums_finish_kernel<<<E, 32, 0, stream>>>((const unsigned long long*)bins.p, (const uint32_t*)epairs.p,
                                                   (LumEdgeOut*)eout.p);
      if (!chunks.empty())
        lum_ss_kernel<<<(unsigned)chunks.size(), kLumThreads, 0, stream>>>(
            (const int2*)chunks_d.p, (const LumEdgeDev*)edges_d.p, (const int2*)list.p, (const float*)xyz.p,
            (const int64_t*)off.p, (const float*)vT.p, (const LumEdgeOut*)eout.p, (unsigned long long*)ebins.p);
      lum_ss_finish_kernel<<<E, 32, 0, stream>>>((const unsigned long long*)ebins.p, (LumEdgeOut*)eout.p);
      SMB_CUDA_OK(cudaGetLastError());
      SMB_CUDA_OK(cudaMemcpyAsync(eo.data(), eout.p, (size_t)E * sizeof(LumEdgeOut), cudaMemcpyDeviceToHost, stream));
      SMB_CUDA_OK(cudaStreamSynchronize(stream));
    }
    std::vector<LumEdge> le(E);
    for (int e = 0; e < E; ++e) {
      le[e].s = edges[e].s;
      le[e].t = edges[e].t;
      memcpy(le[e].cinv, eo[e].cinv, sizeof(le[e].cinv));
      memcpy(le[e].cinvd, eo[e].cinvd, sizeof(le[e].cinvd));
    }
    std::vector<double> X;
    const double sum = lum_solve_update<double>(n, le, poses.data(), trace_on ? &X : nullptr);
    if (trace_on) {
      Iter rec_it{n, std::vector<float>((size_t)E * kLumTraceEdge), X, poses, sum};
      for (int e = 0; e < E; ++e) {
        float* r = &rec_it.edges[(size_t)e * kLumTraceEdge];
        r[0] = (float)edges[e].s;
        r[1] = (float)edges[e].t;
        memcpy(r + 2, &eo[e], (kLumTraceEdge - 2) * sizeof(float));
      }
      trace.push_back(std::move(rec_it));
    }
    if (lum_converged(sum, n)) break;
  }
  return SM_OK;
}

int sm_lum::align(float* out_host, int64_t capacity, int64_t* m_out) {
  const int N = (int)frames.size();
  *m_out = 0;
  if (N == 0) return SM_OK;
  const int V0 = (int)vertex_frame.size();
  auto frame_of = [&](int v) { return v < V0 ? vertex_frame[v] : v - V0; };   // vertex v < N after round 0
  std::vector<int64_t> fcnt(N), foff(N + 1, 0);
  for (int f = 0; f < N; ++f) {
    fcnt[f] = (int64_t)(frames[f].size() / stride);
    foff[f + 1] = foff[f] + fcnt[f];
  }
  std::vector<int> vf(N);
  std::vector<int64_t> out_off(N + 1, 0);
  for (int v = 0; v < N; ++v) {
    vf[v] = frame_of(v);
    out_off[v + 1] = out_off[v] + fcnt[vf[v]];
  }
  const int64_t need = out_off[N];
  if (lum_queries(fcnt.data(), N) > kLumMaxQueries)
    return fail(SM_ERR_BAD_ARGUMENT, "%lld correspondence queries over all pairs: at most %lld",
                (long long)lum_queries(fcnt.data(), N), (long long)kLumMaxQueries);
  if (out_host && capacity < need) {
    *m_out = need;
    return fail(SM_ERR_BAD_ARGUMENT, "the output holds %lld records, AlignAll writes %lld", (long long)capacity,
                (long long)need);
  }
  SMB_RC(lum_use_device(this));
  if (!stream) SMB_CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
  const int64_t total = foff[N];
  int64_t maxn = 1;
  for (int f = 0; f < N; ++f) maxn = std::max(maxn, fcnt[f]);
  // transform
  SMB_RC(rec.reserve((size_t)std::max<int64_t>(total, 1) * stride));
  for (int f = 0; f < N; ++f)
    if (fcnt[f])
      SMB_CUDA_OK(cudaMemcpyAsync((char*)rec.p + foff[f] * stride, frames[f].data(), frames[f].size(),
                                  cudaMemcpyHostToDevice, stream));
  std::vector<float> fT((size_t)12 * N);
  for (int f = 0; f < N; ++f) lum_matrix4_to_3x4(&frame_pose[16 * f], &fT[12 * f]);
  SMB_RC(upload(off, foff, stream));
  SMB_RC(upload(cnt, fcnt, stream));
  SMB_RC(upload(T12, fT, stream));
  SMB_RC(xyz.reserve((size_t)std::max<int64_t>(total, 1) * 3 * sizeof(float)));
  lum_transform_kernel<<<dim3(ceil_div(maxn, kLumThreads), N), kLumThreads, 0, stream>>>(
      (const char*)rec.p, stride, (const int64_t*)off.p, (const int64_t*)cnt.p, (const float*)T12.p, (float*)xyz.p);
  SMB_CUDA_OK(cudaGetLastError());
  // trees over the finite points of frames 1..N-1
  trees.resize(N);
  std::vector<LumTree> th(N, LumTree{nullptr, nullptr, nullptr, 0, 0});
  SMB_RC(packed.reserve((size_t)std::max<int64_t>(total, 1) * 3 * sizeof(float)));
  SMB_RC(map.reserve((size_t)std::max<int64_t>(total, 1) * sizeof(uint32_t)));
  SMB_RC(tile_cnt.reserve(compact_count_bytes(maxn)));
  for (int f = 1; f < N; ++f) {
    const int n = (int)fcnt[f];
    if (n == 0) continue;
    const float* fx = (const float*)xyz.p + 3 * foff[f];
    float* pk = (float*)packed.p + 3 * foff[f];
    uint32_t* mp = (uint32_t*)map.p + foff[f];
    uint32_t* tc = (uint32_t*)tile_cnt.p;
    const int tiles = compact_tiles(n);
    lum_finite_count_kernel<<<tiles, kCompactThreads, 0, stream>>>(fx, n, tc);
    compact_scan(tc, tiles, stream);
    lum_finite_pack_kernel<<<tiles, kCompactThreads, 0, stream>>>(fx, n, tc, pk, mp);
    SMB_CUDA_OK(cudaGetLastError());
    uint32_t nf = 0;
    SMB_CUDA_OK(cudaMemcpyAsync(&nf, tc + tiles, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
    SMB_CUDA_OK(cudaStreamSynchronize(stream));
    if (nf == 0) continue;
    SMB_RC(trees[f].build(pk, (int)nf, kdws, stream));
    th[f] = LumTree{(const KdNode*)trees[f].nodes.p, (const BucketPoint*)trees[f].bpts.p, mp, (int)nf, 0};
  }
  SMB_RC(upload(trees_d, th, stream));
  // all pairs (j, i), j < i, in the reference's loop order
  pairs.clear();
  std::vector<int64_t> pair_off(1, 0);
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < i; ++j) {
      pairs.push_back(make_int2(j, i));
      pair_off.push_back(pair_off.back() + fcnt[j]);
    }
  const int P = (int)pairs.size();
  const int64_t T = pair_off.back();
  pair_cnt.assign(P, 0u);
  pair_first.assign(P + 1, 0);
  if (P > 0 && T > 0) {
    SMB_RC(upload(pairs_d, pairs, stream));
    SMB_RC(upload(pair_off_d, pair_off, stream));
    SMB_RC(pair_cnt_d.reserve((size_t)P * sizeof(uint32_t)));
    SMB_CUDA_OK(cudaMemsetAsync(pair_cnt_d.p, 0, (size_t)P * sizeof(uint32_t), stream));
    SMB_RC(qm.reserve((size_t)T * sizeof(int2)));
    SMB_RC(list.reserve((size_t)T * sizeof(int2)));
    SMB_RC(tile_cnt.reserve(compact_count_bytes(T)));
    lum_search_kernel<<<dim3(ceil_div(maxn, kLumThreads), P), kLumThreads, 0, stream>>>(
        (const float*)xyz.p, (const int64_t*)off.p, (const int64_t*)cnt.p, (const LumTree*)trees_d.p,
        (const int2*)pairs_d.p, (const int64_t*)pair_off_d.p, (int2*)qm.p, (uint32_t*)pair_cnt_d.p);
    const int tiles = compact_tiles(T);
    lum_match_count_kernel<<<tiles, kCompactThreads, 0, stream>>>((const int2*)qm.p, T, (uint32_t*)tile_cnt.p);
    compact_scan((uint32_t*)tile_cnt.p, tiles, stream);
    lum_match_scatter_kernel<<<tiles, kCompactThreads, 0, stream>>>((const int2*)qm.p, T, (const uint32_t*)tile_cnt.p,
                                                                     (int2*)list.p);
    SMB_CUDA_OK(cudaGetLastError());
    SMB_CUDA_OK(cudaMemcpyAsync(pair_cnt.data(), pair_cnt_d.p, (size_t)P * sizeof(uint32_t), cudaMemcpyDeviceToHost,
                                stream));
    SMB_CUDA_OK(cudaStreamSynchronize(stream));
  }
  for (int p = 0; p < P; ++p) pair_first[p + 1] = pair_first[p] + pair_cnt[p];
  // the edges: pairs of more than 2 correspondences.  Vertex k's cloud is frame vf[k]'s, which the indices of frame k
  // must fit (a second AlignAll after AddNewCloud can pair an old round's vertex with a new frame)
  std::vector<LumEdgeDev> edges;
  for (int p = 0; p < P; ++p) {
    if (pair_cnt[p] <= 2) continue;
    const int j = pairs[p].x, i = pairs[p].y;
    if (fcnt[vf[j]] < fcnt[j] || fcnt[vf[i]] < fcnt[i])
      return fail(SM_ERR_BAD_ARGUMENT,
                  "vertex %d holds a cloud of %lld points and vertex %d one of %lld, fewer than frames %d and %d whose "
                  "correspondences index them (PCL reads past the cloud)",
                  j, (long long)fcnt[vf[j]], i, (long long)fcnt[vf[i]], j, i);
    edges.push_back(LumEdgeDev{j, i, vf[j], vf[i], pair_first[p], (int)pair_cnt[p], 0});
  }
  SMB_RC(upload(edges_d, edges, stream));
  // the rounds: N vertices with zero poses each, then compute
  for (int r = 0; r < kLumRounds; ++r) {
    for (int f = 0; f < N; ++f) {
      vertex_frame.push_back(f);
      for (int k = 0; k < 6; ++k) poses.push_back(0.f);
    }
    SMB_RC(cuda_fail(compute(N, edges, T)));
  }
  *m_out = need;
  if (!out_host || need == 0) return SM_OK;
  std::vector<float> mats((size_t)12 * N);
  for (int v = 0; v < N; ++v) lum_pose_matrix(&poses[6 * v], &mats[12 * v]);
  SMB_RC(upload(vT, mats, stream));
  SMB_RC(upload(vf_d, vf, stream));
  SMB_RC(upload(out_off_d, out_off, stream));
  SMB_RC(out.reserve((size_t)need * stride));
  lum_output_kernel<<<dim3(ceil_div(maxn, kLumThreads), N), kLumThreads, 0, stream>>>(
      (const char*)rec.p, stride, (const int64_t*)off.p, (const int64_t*)cnt.p, (const int*)vf_d.p,
      (const int64_t*)out_off_d.p, (const float*)vT.p, (const float*)xyz.p, (char*)out.p);
  SMB_CUDA_OK(cudaGetLastError());
  SMB_CUDA_OK(cudaMemcpyAsync(out_host, out.p, (size_t)need * stride, cudaMemcpyDeviceToHost, stream));
  SMB_CUDA_OK(cudaStreamSynchronize(stream));
  return SM_OK;
}

extern "C" {

int sm_lum_create(int device, sm_lum** out) {
  if (!out) return SM_ERR_BAD_ARGUMENT;
  *out = nullptr;
  const int rc = select_device(device);
  if (rc < 0) return rc;
  *out = new sm_lum(device);
  return SM_OK;
}

int sm_lum_destroy(sm_lum* h) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (select_device(h->device) == SM_OK) cudaDeviceSynchronize();
  delete h;
  return SM_OK;
}

int sm_lum_add_cloud(sm_lum* h, const float* points, int64_t n, int64_t stride_bytes, const float* pose_4x4) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (!pose_4x4 || n < 0 || (n > 0 && !points) || stride_bytes < 12 || stride_bytes % 4 != 0)
    return h->fail(SM_ERR_BAD_ARGUMENT, "a cloud needs a pose, n >= 0 records and a stride of 12 bytes or more, a "
                                        "multiple of 4");
  if (h->stride != 0 && stride_bytes != h->stride)
    return h->fail(SM_ERR_BAD_ARGUMENT, "stride %lld differs from the %lld of the first cloud", (long long)stride_bytes,
                   (long long)h->stride);
  if ((int)h->frames.size() >= kLumMaxFrames)
    return h->fail(SM_ERR_BAD_ARGUMENT, "more than %d frames", kLumMaxFrames);
  if (n > kLumMaxPoints)
    return h->fail(SM_ERR_BAD_ARGUMENT, "a frame of %lld points: at most %lld", (long long)n, (long long)kLumMaxPoints);
  h->stride = stride_bytes;
  const char* p = reinterpret_cast<const char*>(points);
  h->frames.emplace_back(p, p + n * stride_bytes);
  h->frame_pose.insert(h->frame_pose.end(), pose_4x4, pose_4x4 + 16);
  return SM_OK;
}

int64_t sm_lum_size(const sm_lum* h) { return h ? (int64_t)h->frames.size() : SM_ERR_BAD_ARGUMENT; }

int sm_lum_align_all(sm_lum* h, float* out, int64_t capacity, int64_t* m_out) {
  if (!h || !m_out || capacity < 0) return SM_ERR_BAD_ARGUMENT;
  return h->align(out, capacity, m_out);
}

int sm_lum_poses(const sm_lum* h, float* out_or_null, int64_t capacity, int64_t* n_vertices) {
  if (!h || !n_vertices) return SM_ERR_BAD_ARGUMENT;
  const int64_t n = (int64_t)h->vertex_frame.size();
  *n_vertices = n;
  if (!out_or_null) return SM_OK;
  if (capacity < n) return SM_ERR_BAD_ARGUMENT;
  if (n) memcpy(out_or_null, h->poses.data(), (size_t)n * 6 * sizeof(float));
  return SM_OK;
}

const char* sm_lum_last_error(const sm_lum* h) { return h ? h->error : ""; }

// ---- test hooks (include/sm_b200_debug.h) -------------------------------------------------------------------------
int sm_debug_lum_correspondences(const sm_lum* h, int32_t j, int32_t i, int32_t* pairs_or_null, int64_t capacity,
                                 int64_t* n) {
  if (!h || !n || j < 0 || i <= j || i >= (int)h->frames.size()) return SM_ERR_BAD_ARGUMENT;
  const int64_t p = (int64_t)i * (i - 1) / 2 + j;
  if (p >= (int64_t)h->pair_cnt.size()) return SM_ERR_BAD_ARGUMENT;   // no AlignAll over these frames yet
  *n = h->pair_cnt[p];
  if (!pairs_or_null || *n == 0) return SM_OK;
  if (capacity < *n) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(h->device));
  SMB_CUDA_OK(cudaMemcpy(pairs_or_null, (const int2*)h->list.p + h->pair_first[p], (size_t)*n * sizeof(int2),
                         cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_lum_trace(sm_lum* h, int32_t enable) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  h->trace_on = enable != 0;
  h->trace.clear();
  return SM_OK;
}

int sm_debug_lum_trace_get(const sm_lum* h, int64_t iteration, int32_t* n_vertices, int32_t* n_edges,
                           float* edges_or_null, double* x_or_null, float* poses_or_null, double* sum) {
  if (!h || !n_vertices || !n_edges || !sum) return SM_ERR_BAD_ARGUMENT;
  if (iteration < 0) { *n_vertices = 0; *n_edges = (int32_t)h->trace.size(); *sum = 0; return SM_OK; }
  if (iteration >= (int64_t)h->trace.size()) return SM_ERR_BAD_ARGUMENT;
  const sm_lum::Iter& t = h->trace[iteration];
  *n_vertices = t.n;
  *n_edges = (int32_t)(t.edges.size() / kLumTraceEdge);
  *sum = t.sum;
  if (edges_or_null && !t.edges.empty()) memcpy(edges_or_null, t.edges.data(), t.edges.size() * sizeof(float));
  if (x_or_null && !t.X.empty()) memcpy(x_or_null, t.X.data(), t.X.size() * sizeof(double));
  if (poses_or_null) memcpy(poses_or_null, t.poses.data(), t.poses.size() * sizeof(float));
  return SM_OK;
}

}  // extern "C"
