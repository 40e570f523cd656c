// IcpFast::Align on the device (registrators/icp_fast.cc:455-529), double precision.
//
// One ICP iteration = three phases, each a kernel here (the same __device__ phase bodies
// are meant to be driven by a persistent cooperative kernel as well):
//   A  transform + epsilon-approximate 1-NN in the libnabo-compatible tree (icp_fast.cc:
//      486-493, 169-180) + a 2048-bin histogram of the squared distances;
//   B  locate the histogram bin that holds the floor(N*0.7f)-th order statistic
//      (icp_fast.cc:65-90); every match strictly below that bin is accumulated into the
//      point-to-plane normal equations right away (icp_fast.cc:256-302), matches inside
//      the bin are compacted (deterministically, ascending index) as candidates;
//   C  one CTA: exact radix-select of the limit among the candidates, add the candidates
//      <= limit, fixed-order reduction of the per-block partial sums, 6x6 solve, pose
//      update, convergence test and score (icp_fast.cc:204-254, 307-321, 377-405, 513-527).
// Nothing returns to the host between iterations; kernels early-out on state->done.
#include "common.cuh"
#include "kernels.h"
#include "icp_dev.cuh"
#include "knn_smem.cuh"
#include "linalg_dev.cuh"
#include "motion_dev.cuh"

#include <nvtx3/nvToolsExt.h>

namespace smb {
using namespace dev;
namespace {

// ------------------------------------------------------------------------------ prologue
constexpr int kMeanChunk = 1024;   // target points per mean_partial_kernel block (4 per thread), 4 doubles out each

__global__ void __launch_bounds__(256)
mean_partial_kernel(const double* __restrict__ raw, int64_t stride, int n,
                    double* __restrict__ partials) {
  __shared__ double red[8][3];
  double s[3] = {0.0, 0.0, 0.0};
  const int base = blockIdx.x * kMeanChunk;
  for (int r = 0; r < 4; ++r) {
    const int i = base + r * 256 + threadIdx.x;
    if (i < n) { s[0] += raw[i]; s[1] += raw[stride + i]; s[2] += raw[2 * stride + i]; }
  }
  const double v = block_sum<3, 256>(s, red);
  if (threadIdx.x < 3) partials[blockIdx.x * 4 + threadIdx.x] = v;
}

__global__ void __launch_bounds__(256)
center_kernel(const double* __restrict__ raw, double* __restrict__ out, int64_t stride, int n,
              const double* __restrict__ partials, int nparts, IcpState* __restrict__ st) {
  __shared__ double mean[3];
  if (threadIdx.x < 3) {
    double v = 0.0;
    for (int b = 0; b < nparts; ++b) v += partials[b * 4 + threadIdx.x];
    v = v / (double)n;
    mean[threadIdx.x] = v;
    if (blockIdx.x == 0) st->mean[threadIdx.x] = v;
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    out[i] = dsub(raw[i], mean[0]);
    out[stride + i] = dsub(raw[stride + i], mean[1]);
    out[2 * stride + i] = dsub(raw[2 * stride + i], mean[2]);
  }
}

// one block: G0 = T_mean^-1 * guess, state reset, histogram clear (icp_fast.cc:460-480)
__global__ void icp_init_kernel(IcpState* __restrict__ st, const double* __restrict__ guess,
                                uint32_t* __restrict__ hist) {
  for (int i = threadIdx.x; i < 2 * kHistBins; i += blockDim.x) hist[i] = 0;  // hist + hist2
  if (threadIdx.x != 0) return;
  double Tm[16], Tmi[16];
  for (int i = 0; i < 16; ++i) { Tm[i] = (i % 5 == 0) ? 1.0 : 0.0; Tmi[i] = Tm[i]; }
  for (int r = 0; r < 3; ++r) { Tm[12 + r] = st->mean[r]; Tmi[12 + r] = -st->mean[r]; }
  double g[16];
  for (int i = 0; i < 16; ++i) g[i] = guess[i];
  double G0[16];
  la::mul4(Tmi, g, G0);
  for (int i = 0; i < 16; ++i) {
    st->T_mean[i] = Tm[i]; st->G0[i] = G0[i];
    st->T_iter[i] = (i % 5 == 0) ? 1.0 : 0.0;
    st->result[i] = 0.0;
  }
  st->quat_hist[0][0] = 1.0; st->quat_hist[0][1] = 0.0; st->quat_hist[0][2] = 0.0; st->quat_hist[0][3] = 0.0;
  st->trans_hist[0][0] = 0.0; st->trans_hist[0][1] = 0.0; st->trans_hist[0][2] = 0.0;
  st->hist_len = 1; st->iteration = 0; st->done = 0; st->status = 0; st->solve_path = 0;
  st->final_score = 0.0; st->limit = 0.0; st->kept = 0;
}

// 30-bit Morton key on a 0.25 m lattice (coordinates wrap every 256 m, harmless for a key
// that only has to make neighbouring threads spatially close)
__device__ __forceinline__ uint32_t spread10(uint32_t v) {
  v &= 1023u;
  v = (v | (v << 16)) & 0x030000ffu;
  v = (v | (v << 8)) & 0x0300f00fu;
  v = (v | (v << 4)) & 0x030c30c3u;
  v = (v | (v << 2)) & 0x09249249u;
  return v;
}

// init_source = G0 (x) source (icp_fast.cc:469-471) + the spatial sort key of each point
__global__ void apply_g0_kernel(const double* __restrict__ in, double* __restrict__ out,
                                int64_t stride, int n, const IcpState* __restrict__ st,
                                uint64_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double px, py, pz;
  transform_point(st->G0, in[i], in[stride + i], in[2 * stride + i], px, py, pz);
  out[i] = px; out[stride + i] = py; out[2 * stride + i] = pz;
  const uint32_t ix = (uint32_t)(int)floor(px * 4.0), iy = (uint32_t)(int)floor(py * 4.0),
                 iz = (uint32_t)(int)floor(pz * 4.0);
  keys[i] = (uint64_t)(spread10(ix) | (spread10(iy) << 1) | (spread10(iz) << 2));
  vals[i] = (uint32_t)i;
}

// queries in Morton order: neighbouring threads walk the same tree lines and hit the same
// buckets.  Only sums are formed over the source, so its order is free.
__global__ void gather_source_kernel(const double* __restrict__ in, double* __restrict__ out,
                                     int64_t stride, int n, const uint32_t* __restrict__ perm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t s = perm[i];
  out[i] = in[s]; out[stride + i] = in[stride + s]; out[2 * stride + i] = in[2 * stride + s];
}

// -------------------------------------------------------------------------------- phase A
// ApplyTransform + FindClosests (icp_fast.cc:486-493, 169-180) + the 2048-bin histogram of the
// squared distances.  One query per thread over a contiguous, Morton-ordered range per CTA
// (neighbouring threads walk the same nodes and buckets); every CTA stages the top levels of the
// tree into shared memory with bulk async copies while its threads load and transform their
// queries (knn_smem.cuh).
#ifndef SMB_KNN_MIN_CTAS
#define SMB_KNN_MIN_CTAS 4
#endif
// Phase A, one query per thread (a single alignment in flight: 469 CTAs, all resident at once, the
// kernel lasts as long as its longest search).
// the query of source point i: T_iter (x) src0_i, or with inner compensation the de-skewed point of the iteration
template <bool kComp>
__device__ __forceinline__ void load_query(const IcpBuffers& b, const double* T, const double* __restrict__ deskewed,
                                           int i, double& x, double& y, double& z) {
  if constexpr (kComp) {
    x = deskewed[i]; y = deskewed[b.sstride + i]; z = deskewed[2 * b.sstride + i];
  } else {
    transform_point(T, b.src0[i], b.src0[b.sstride + i], b.src0[2 * b.sstride + i], x, y, z);
  }
}

// the match of source point i for phase B, and its d2 counted in the 2048-bin global histogram (a fire-and-forget
// reduction, L2-resident)
__device__ __forceinline__ void store_match(const IcpBuffers& b, int i, int slot, double d2) {
  b.slot[i] = slot;
  b.d2[i] = d2;
  if (finite_d2(d2)) atomicAdd(&b.hist[dist_bin(d2)], 1u);
}

template <bool kAllSmem, bool kComp>
__global__ void __launch_bounds__(kKnnCtaThreads, SMB_KNN_MIN_CTAS)
icp_knn_kernel(IcpBuffers b, IcpParams p, int per_cta, const double* __restrict__ deskewed) {
  extern __shared__ __align__(128) unsigned char knn_smem[];
  if (b.state->done) return;
  uint64_t* bar; double* T;
  const SmemTree tree = stage_tree(b.kc, knn_smem, &bar, &T);
  if (threadIdx.x < 16) T[threadIdx.x] = b.state->T_iter[threadIdx.x];
  __syncthreads();
  const int begin = blockIdx.x * per_cta, end = min(begin + per_cta, p.n_source);
  knn1_cta<kAllSmem>(
      tree, bar, begin, end, p.max_error2,
      [&](int i, double& x, double& y, double& z) { load_query<kComp>(b, T, deskewed, i, x, y, z); },
      [&](int i, int slot, double d2) { store_match(b, i, slot, d2); });
}

// Phase A with several queries per thread (many alignments in flight: queries_per_cta > 256): lockstep root
// visits, then the lanes of every warp pull the parked searches of their batch (knn_batch_cta, knn_smem.cuh).
// The one-query-per-thread form spends its time in passes in which a few lanes finish long searches
// (11.7 of 32 lanes busy on average, 18.0 here).
template <bool kAllSmem, bool kComp>
__global__ void __launch_bounds__(kKnnCtaThreads, SMB_KNN_MIN_CTAS)
icp_knn_batch_kernel(IcpBuffers b, IcpParams p, int per_cta, const double* __restrict__ deskewed) {
  extern __shared__ __align__(128) unsigned char knn_smem[];
  if (b.state->done) return;
  uint64_t* bar; double* T;
  const SmemTree tree = stage_tree(b.kc, knn_smem, &bar, &T);
  if (threadIdx.x < 16) T[threadIdx.x] = b.state->T_iter[threadIdx.x];
  __syncthreads();
  const int begin = blockIdx.x * per_cta, end = min(begin + per_cta, p.n_source);
  mbar_wait(bar, 0);      // every thread waits: the CTA must not retire while the copy engine writes its smem
  knn_batch_cta<kAllSmem>(
      tree, begin, end, per_cta, p.max_error2, b.knn_items,
      [&](int i, double& x, double& y, double& z) { load_query<kComp>(b, T, deskewed, i, x, y, z); },
      [&](int i, int best, double head) { b.slot[i] = best; b.d2[i] = head; },
      [&](int i, double& head, int& best) { head = __ldcg(b.d2 + i); best = __ldcg(b.slot + i); },
      [&](int i, int slot, double d2) { store_match(b, i, slot, d2); });
}

// -------------------------------------------------------------------------------- phase B
// kComp: inner compensation (icp_fast.cc:284-289): the points are the iteration's de-skewed ones and every
// match's Jacobian column is scaled by the point's factor, both for the sums and for the parked candidates
// kP2P: the point-to-point minimizer (icp_fast.cc:326-375): a match contributes the raw moments of add_p2p_terms_if
// (no normal is read, and with kComp the factor is not used); a parked candidate is {p, q, 0, sqrt(d2)}
// SMB_ACC_SECTIONS (diagnostic builds, profiles/accum_sections.py): every block adds the clock64 cycles thread 0
// spent in each section below to state->stamps[0..5] and 1 to stamps[6], over all iterations and alignments
#ifdef SMB_ACC_SECTIONS
constexpr bool kAccSections = true;
#else
constexpr bool kAccSections = false;
#endif
enum AccSection { kSecLoads, kSecSelectBin, kSecGather, kSecTerms, kSecCompaction, kSecReduction, kAccSectionCount };

template <bool kComp, bool kP2P>
__global__ void __launch_bounds__(kAccThreads)
icp_accum_kernel(IcpBuffers b, IcpParams p, const double* __restrict__ deskewed) {
  __shared__ uint32_t warp_tot[8];
  __shared__ BinSel sel_sm;
  __shared__ double T[16];
  __shared__ double red[kAccThreads / 32][kNumSums];
  __shared__ uint32_t cand_warp[kAccItems][kAccThreads / 32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int tile0 = blockIdx.x * kAccTile;
  [[maybe_unused]] long long sec[kAccSectionCount] = {}, sec_t = 0;
  const auto mark = [&](int s) {
    if constexpr (kAccSections) { const long long now = clock64(); sec[s] += now - sec_t; sec_t = now; }
  };
  if constexpr (kAccSections) sec_t = clock64();
  // Item r of a thread is point tile0 + r * kAccThreads + threadIdx.x; the items run in passes of kAccPass,
  // so the registers held per thread do not grow with the tile.
  // (1) everything that does not depend on the quantile bin is requested up front, for all the
  //     points of the pass at once (the first pass's reads overlap the histogram read of select_bin)
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  const double* src = kComp ? deskewed : b.src0;
  double d2[kAccPass], sx[kAccPass], sy[kAccPass], sz[kAccPass];
  [[maybe_unused]] double fac[kAccPass];
  int slot[kAccPass];
  const auto load_pass = [&](int r0) {
#pragma unroll
    for (int r = 0; r < kAccPass; ++r) {
      const int i = tile0 + (r0 + r) * kAccThreads + threadIdx.x;
      const bool in = i < p.n_source;
      d2[r] = in ? b.d2[i] : inf;
      slot[r] = in ? b.slot[i] : -1;
      sx[r] = in ? src[i] : 0.0;
      sy[r] = in ? src[b.sstride + i] : 0.0;
      sz[r] = in ? src[2 * b.sstride + i] : 0.0;
      if constexpr (kComp && !kP2P) fac[r] = in ? source_factor(b.src_sort.vals[0][i], p.n_source) : 0.0;
    }
  };
  load_pass(0);
  if (b.state->done) return;
  if (threadIdx.x < 16) T[threadIdx.x] = b.state->T_iter[threadIdx.x];
  mark(kSecLoads);
  const BinSel sel = select_bin(b.hist, p.dist_outlier_ratio, warp_tot, &sel_sm);
  mark(kSecSelectBin);
  double acc[kNumSums];
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) acc[k] = 0.0;
  uint32_t base = 0;
#pragma unroll 1
  for (int r0 = 0; r0 < kAccItems; r0 += kAccPass) {
    if (r0 > 0) { load_pass(r0); mark(kSecLoads); }
    // (2) the matched target point and normal of every point at or below the quantile bin: one 64-byte
    //     record, three 16-byte loads; the other lanes read entry 0 and are masked out, so the gathers of
    //     all items of the pass go out together
    bool use[kAccPass], is_cand[kAccPass];
    int bin[kAccPass];
    double2 r01[kAccPass], r23[kAccPass], r45[kAccPass];    // {x, y}, {z, nx}, {ny, nz}
#pragma unroll
    for (int r = 0; r < kAccPass; ++r) {
      bin[r] = finite_d2(d2[r]) ? dist_bin(d2[r]) : kHistBins;
      use[r] = sel.bin >= 0 && slot[r] >= 0 && bin[r] <= sel.bin;
      const double2* rec = reinterpret_cast<const double2*>(b.kc.pm + (use[r] ? slot[r] : 0));
      r01[r] = __ldg(rec); r23[r] = __ldg(rec + 1);
      if constexpr (!kP2P) r45[r] = __ldg(rec + 2);
    }
    mark(kSecGather);
    double F[kAccPass][6], dot[kAccPass], sq[kAccPass];   // kP2P: F = {p, q}, dot = 0
#pragma unroll
    for (int r = 0; r < kAccPass; ++r) {
      BucketPoint q; BucketNormal n;
      q.x = r01[r].x; q.y = r01[r].y; q.z = r23[r].x;
      if constexpr (kP2P) {
        if constexpr (kComp) { F[r][0] = sx[r]; F[r][1] = sy[r]; F[r][2] = sz[r]; }
        else transform_point(T, sx[r], sy[r], sz[r], F[r][0], F[r][1], F[r][2]);
        F[r][3] = q.x; F[r][4] = q.y; F[r][5] = q.z;
        dot[r] = 0.0;
        sq[r] = sqrt(use[r] ? d2[r] : 0.0);
        add_p2p_terms_if(acc, F[r], F[r] + 3, sq[r], use[r] && bin[r] < sel.bin);
        is_cand[r] = use[r] && bin[r] == sel.bin;
        if (is_cand[r]) atomicAdd(&b.hist2[sub_bin(d2[r])], 1u);
        continue;
      }
      n.x = r23[r].y; n.y = r45[r].x; n.z = r45[r].y;
      if constexpr (kComp) {
        compensated_match_terms(sx[r], sy[r], sz[r], q, n, fac[r], F[r], dot[r]);
      } else {
        double px, py, pz;
        transform_point(T, sx[r], sy[r], sz[r], px, py, pz);
        match_terms(px, py, pz, q, n, F[r], dot[r]);
      }
      sq[r] = sqrt(use[r] ? d2[r] : 0.0);
      add_terms_if(acc, F[r], dot[r], sq[r], use[r] && bin[r] < sel.bin);
      is_cand[r] = use[r] && bin[r] == sel.bin;
      if (is_cand[r]) atomicAdd(&b.hist2[sub_bin(d2[r])], 1u);
    }
    mark(kSecTerms);
    // (3) ordered compaction of the quantile-bin members: (item, warp, lane) == ascending point index; the
    //     passes append in item order behind `base`
    uint32_t m[kAccPass];
#pragma unroll
    for (int r = 0; r < kAccPass; ++r) {
      m[r] = __ballot_sync(0xffffffffu, is_cand[r]);
      if (lane == 0) cand_warp[r0 + r][w] = __popc(m[r]);
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < kAccPass; ++r) {
      uint32_t off = base, tot = 0;
#pragma unroll
      for (int ww = 0; ww < kAccThreads / 32; ++ww) {
        const uint32_t c = cand_warp[r0 + r][ww];
        if (ww < w) off += c;
        tot += c;
      }
      if (is_cand[r]) {
        const int64_t dst = tile0 + off + __popc(m[r] & ((1u << lane) - 1u));
        b.cand_key[dst] = (unsigned long long)__double_as_longlong(d2[r]);
        double2* o = reinterpret_cast<double2*>(b.cand_terms + 8 * dst);
        o[0] = make_double2(F[r][0], F[r][1]); o[1] = make_double2(F[r][2], F[r][3]);
        o[2] = make_double2(F[r][4], F[r][5]); o[3] = make_double2(dot[r], sq[r]);
      }
      base += tot;
    }
    mark(kSecCompaction);
  }
  if (threadIdx.x == 0) b.cand_cnt[blockIdx.x] = base;
  block_reduce_sums<kAccThreads>(acc, red, b.partials + (int64_t)blockIdx.x * 32);
  if constexpr (kAccSections) {
    mark(kSecReduction);
    if (threadIdx.x == 0) {
      unsigned long long* st = reinterpret_cast<unsigned long long*>(b.state->stamps);
      for (int s = 0; s < kAccSectionCount; ++s) atomicAdd(st + s, (unsigned long long)sec[s]);
      atomicAdd(st + kAccSectionCount, 1ull);
    }
  }
}

template <bool kAllSmem>
__global__ void __launch_bounds__(kKnnCtaThreads)
knn_query_kernel(KdCompact kc, const double* __restrict__ query, int64_t qstride, int nq,
                 double max_error2, int per_cta, int32_t* __restrict__ ids, double* __restrict__ d2) {
  extern __shared__ __align__(128) unsigned char knn_smem[];
  uint64_t* bar; double* extra;
  const SmemTree tree = stage_tree(kc, knn_smem, &bar, &extra);
  const int begin = blockIdx.x * per_cta, end = min(begin + per_cta, nq);
  knn1_cta<kAllSmem>(
      tree, bar, begin, end, max_error2,
      [&](int i, double& x, double& y, double& z) { x = query[i]; y = query[qstride + i]; z = query[2 * qstride + i]; },
      [&](int i, int slot, double d) { ids[i] = slot >= 0 ? kc.pid[slot] : -1; d2[i] = d; });
}


// the same search with the batch scheduling of icp_knn_batch_kernel (sm_debug_knn1_batched: parity tests of
// the warp-pulled far visits against the oracle's index sets); ids[] / d2[] double as the parking arrays
template <bool kAllSmem>
__global__ void __launch_bounds__(kKnnCtaThreads, SMB_KNN_MIN_CTAS)
knn_query_batch_kernel(KdCompact kc, const double* __restrict__ query, int64_t qstride, int nq,
                       double max_error2, int per_cta, int32_t* __restrict__ ids, double* __restrict__ d2,
                       int4* __restrict__ items) {
  extern __shared__ __align__(128) unsigned char knn_smem[];
  uint64_t* bar; double* extra;
  const SmemTree tree = stage_tree(kc, knn_smem, &bar, &extra);
  const int begin = blockIdx.x * per_cta, end = min(begin + per_cta, nq);
  mbar_wait(bar, 0);
  knn_batch_cta<kAllSmem>(
      tree, begin, end, per_cta, max_error2, items,
      [&](int i, double& x, double& y, double& z) { x = query[i]; y = query[qstride + i]; z = query[2 * qstride + i]; },
      [&](int i, int best, double head) { ids[i] = best; d2[i] = head; },
      [&](int i, double& head, int& best) { head = __ldcg(d2 + i); best = __ldcg(ids + i); },
      [&](int i, int slot, double d) { ids[i] = slot >= 0 ? kc.pid[slot] : -1; d2[i] = d; });
}

}  // namespace

int icp_accum_blocks(int n_source) { return ceil_div(n_source, kAccTile); }

// a warp's item list may extend past the last query of the last batch
size_t knn_items_bytes(int nq) { return ((size_t)nq + 4096) * sizeof(int4); }

constexpr int kSumWords = 32;    // one record of normal-equation sums: kNumSums padded to 32 doubles
constexpr int kCandWords = 8;    // one quantile-bin candidate: 6 Jacobian terms, the residual, sqrt(d2)
// hist: the two histograms, 64 words of padding, then the iteration's sums record
constexpr size_t kHistSumsOffset = (2 * kHistBins + 64) * sizeof(uint32_t);
// slot: the per-point match slots, padded to 256 bytes, then the parked-search items
static size_t slot_bytes(int ns) { return (((size_t)ns * sizeof(int32_t) + 64 + 255) / 256) * 256; }

int IcpFastBuffers::reserve(int ns, int nt, int64_t sstride, int64_t tstride, bool inner_compensation) {
  this->ns = ns; this->sstride = sstride; this->tstride = tstride;
  const int nb = icp_accum_blocks(ns);
  SMB_RC(tgt.reserve((size_t)(3 * tstride) * sizeof(double)));
  SMB_RC(src0.reserve((size_t)(3 * sstride) * sizeof(double)));
  SMB_RC(src_g0.reserve((size_t)(3 * sstride) * sizeof(double)));
  SMB_RC(src_sort.reserve(RadixPairs::bytes(sstride, ns)));
  SMB_RC(tree.reserve(nt, 8, KdCompactTree::kNormals));
  SMB_RC(slot.reserve(slot_bytes(ns) + knn_items_bytes(ns)));
  SMB_RC(d2.reserve((size_t)ns * sizeof(double)));
  SMB_RC(hist.reserve(kHistSumsOffset + kSumWords * sizeof(double)));
  SMB_RC(cand_terms.reserve((size_t)nb * kAccTile * kCandWords * sizeof(double)));
  SMB_RC(cand_key.reserve((size_t)nb * kAccTile * sizeof(unsigned long long)));
  SMB_RC(cand_cnt.reserve((size_t)nb * sizeof(uint32_t)));
  SMB_RC(partials.reserve((size_t)nb * kSumWords * sizeof(double)));
  SMB_RC(mean_partials.reserve((size_t)ceil_div(nt, kMeanChunk) * 4 * sizeof(double)));
  SMB_RC(state.reserve(sizeof(IcpState)));
  SMB_RC(guess.reserve(16 * sizeof(double)));
  if (inner_compensation) SMB_RC(deskewed.reserve((size_t)(3 * sstride) * sizeof(double)));
  return 0;
}

void IcpFastBuffers::fill(IcpBuffers& b, const double* tgt_raw, const double* nrm, const double* src_raw) const {
  b.tgt = (double*)tgt.p; b.tgt_raw = (double*)tgt_raw; b.nrm = (double*)nrm;
  b.tstride = tstride;
  b.nodes = (KdNode*)tree.nodes.p; b.leaf_order = (uint32_t*)tree.leaf_order.p;
  b.kc = tree.view();
  b.src_raw = (double*)src_raw; b.src0 = (double*)src0.p; b.sstride = sstride;
  b.src_g0 = (double*)src_g0.p;
  b.src_sort.carve(src_sort.p, sstride);
  b.slot = (int32_t*)slot.p;
  b.knn_items = reinterpret_cast<int4*>((char*)slot.p + slot_bytes(ns));
  b.d2 = (double*)d2.p; b.hist = (uint32_t*)hist.p;
  b.hist2 = b.hist + kHistBins;
  b.sums = (double*)((char*)hist.p + kHistSumsOffset);
  b.cand_terms = (double*)cand_terms.p;
  b.cand_key = (unsigned long long*)cand_key.p; b.cand_cnt = (uint32_t*)cand_cnt.p;
  b.partials = (double*)partials.p; b.mean_partials = (double*)mean_partials.p;
  b.state = (IcpState*)state.p;
}

// Launch geometry of the search kernels: `per_cta` consecutive queries per 256-thread CTA.
// queries_per_cta == 0: one query per thread (120 000 queries = 469 CTAs, ~3 per SM, all
// resident at once); a larger value makes a CTA loop over its range, which amortises the staging
// of the tree top over more queries.
static void knn_geometry(int nq, int queries_per_cta, int* grid, int* per_cta) {
  int per = queries_per_cta > 0 ? queries_per_cta : kKnnCtaThreads;
  per = ((per + kKnnCtaThreads - 1) / kKnnCtaThreads) * kKnnCtaThreads;
  *per_cta = per;
  *grid = ceil_div(nq, per);
}

int knn_query(const KdCompact& kc, const double* query, int64_t qstride, int nq, double max_error2,
              int32_t* ids, double* d2, cudaStream_t stream, int queries_per_cta, int4* items) {
  if (nq <= 0) return 0;
  int grid, per;
  knn_geometry(nq, queries_per_cta, &grid, &per);
  const size_t smem = knn_smem_bytes(kc.levels);
  const bool all = kc.levels <= kKnnSmemLevels;
  if (per > kKnnCtaThreads) {
    if (!items) return -1;
    if (all) knn_query_batch_kernel<true><<<grid, kKnnCtaThreads, smem, stream>>>(kc, query, qstride, nq, max_error2, per, ids, d2, items);
    else knn_query_batch_kernel<false><<<grid, kKnnCtaThreads, smem, stream>>>(kc, query, qstride, nq, max_error2, per, ids, d2, items);
  } else if (all) {
    knn_query_kernel<true><<<grid, kKnnCtaThreads, smem, stream>>>(kc, query, qstride, nq, max_error2, per, ids, d2);
  } else {
    knn_query_kernel<false><<<grid, kKnnCtaThreads, smem, stream>>>(kc, query, qstride, nq, max_error2, per, ids, d2);
  }
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

// icp_fast.cc:456-480: centre the target, rebuild the tree, G0, initial source transform.
int icp_prologue(const IcpBuffers& b, const IcpParams& p, const double* guess_dev,
                 KdWorkspace& ws, const KdCompactTree& tree, cudaStream_t stream) {
  const int nt = p.n_target, ns = p.n_source;
  const int nparts = ceil_div(nt, kMeanChunk);
  mean_partial_kernel<<<nparts, 256, 0, stream>>>(b.tgt_raw, b.tstride, nt, b.mean_partials);
  center_kernel<<<ceil_div(nt, 256), 256, 0, stream>>>(b.tgt_raw, b.tgt, b.tstride, nt,
                                                      b.mean_partials, nparts, b.state);
  nvtxRangePushA("BuildKdTree");                 // icp_fast.cc:465
  int rc = tree.build(b.tgt, b.nrm, b.tstride, nt, 8, ws, stream);
  nvtxRangePop();
  if (rc) return rc;
  const RadixPairs& sp = b.src_sort;
  icp_init_kernel<<<1, 256, 0, stream>>>(b.state, guess_dev, b.hist);
  apply_g0_kernel<<<ceil_div(ns, 256), 256, 0, stream>>>(b.src_raw, b.src_g0, b.sstride, ns, b.state,
                                                        sp.keys[0], sp.vals[0]);
  rc = radix_sort_pairs_u64(sp.keys[0], sp.vals[0], sp.keys[1], sp.vals[1], ns, 1, b.sstride, sp.scratch, stream, 4);
  if (rc) return rc;
  gather_source_kernel<<<ceil_div(ns, 256), 256, 0, stream>>>(b.src_g0, b.src0, b.sstride, ns, sp.vals[0]);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

// kernel launches of icp_prologue with a target tree of `levels` levels: centring 2, tree build 27 + 5 per level,
// init and G0 2, Morton sort and gather 13
int icp_prologue_launches(int levels) { return 2 + 1 + 24 + levels * 5 + 1 + 1 + 2 + 13; }

// Iterations start_iteration .. start_iteration+count-1 of one Align: three launches each, four with inner
// compensation (the de-skew of the source goes first).
int icp_iteration_launches(bool inner_compensation) { return inner_compensation ? 4 : 3; }

template <bool kComp>
void icp_enqueue_search(const IcpBuffers& b, const IcpParams& p, int grid, int per, size_t smem, cudaStream_t stream,
                        const double* deskewed) {
  if (per > kKnnCtaThreads) {
    if (p.tree_levels <= kKnnSmemLevels)
      icp_knn_batch_kernel<true, kComp><<<grid, kKnnCtaThreads, smem, stream>>>(b, p, per, deskewed);
    else
      icp_knn_batch_kernel<false, kComp><<<grid, kKnnCtaThreads, smem, stream>>>(b, p, per, deskewed);
  } else if (p.tree_levels <= kKnnSmemLevels) {
    icp_knn_kernel<true, kComp><<<grid, kKnnCtaThreads, smem, stream>>>(b, p, per, deskewed);
  } else {
    icp_knn_kernel<false, kComp><<<grid, kKnnCtaThreads, smem, stream>>>(b, p, per, deskewed);
  }
}

void icp_search_launch(const IcpBuffers& b, const IcpParams& p, const double* deskewed, cudaStream_t stream) {
  int grid, per;
  knn_geometry(p.n_source, p.knn_queries_per_cta, &grid, &per);
  const size_t smem = knn_smem_bytes(p.tree_levels);
  if (p.inner_compensation) icp_enqueue_search<true>(b, p, grid, per, smem, stream, deskewed);
  else icp_enqueue_search<false>(b, p, grid, per, smem, stream, nullptr);
}

void icp_accum_launch(const IcpBuffers& b, const IcpParams& p, const double* deskewed, cudaStream_t stream) {
  const int nb = icp_accum_blocks(p.n_source);
  if (p.error_minimizer == kIcpPointToPoint) {
    if (p.inner_compensation) icp_accum_kernel<true, true><<<nb, kAccThreads, 0, stream>>>(b, p, deskewed);
    else icp_accum_kernel<false, true><<<nb, kAccThreads, 0, stream>>>(b, p, nullptr);
  } else if (p.inner_compensation) {
    icp_accum_kernel<true, false><<<nb, kAccThreads, 0, stream>>>(b, p, deskewed);
  } else {
    icp_accum_kernel<false, false><<<nb, kAccThreads, 0, stream>>>(b, p, nullptr);
  }
}

int icp_enqueue_iterations(const IcpBuffers& b, const IcpParams& p, int start_iteration, int count,
                           cudaStream_t stream, cudaEvent_t* events, double* deskewed) {
  const bool comp = p.inner_compensation != 0;
  if (comp && !deskewed) return -1;
  const int nb = icp_accum_blocks(p.n_source);
  for (int it = 0; it < count; ++it) {
    nvtxRangePushA("Iteration");                 // REGISTER_BLOCK("Iteration"), icp_fast.cc:484
    if (events) cudaEventRecord(events[4 * it + 0], stream);
    if (comp) {
      nvtxRangePushA("ApplyMotionCompensation");   // icp_fast.cc:487-488
      icp_deskew_launch(b, p, deskewed, stream);
      nvtxRangePop();
    }
    nvtxRangePushA("FindClosests");              // icp_fast.cc:169-180
    icp_search_launch(b, p, deskewed, stream);
    nvtxRangePop();
    if (events) cudaEventRecord(events[4 * it + 1], stream);
    nvtxRangePushA("ErrorElements");             // icp_fast.cc:92-167 (+ the sums of ComputePointToPlane)
    icp_accum_launch(b, p, deskewed, stream);
    nvtxRangePop();
    if (events) cudaEventRecord(events[4 * it + 2], stream);
    nvtxRangePushA(p.error_minimizer == kIcpPointToPoint ? "ComputePointToPoint"    // icp_fast.cc:326-375
                                                         : "ComputePointToPlane");  // icp_fast.cc:256-323
    icp_finish_launch(b, p, nb, stream);
    nvtxRangePop();
    if (events) cudaEventRecord(events[4 * it + 3], stream);
    nvtxRangePop();
  }
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace smb
