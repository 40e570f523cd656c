// Phase C of the ICP iteration (see icp.cu), one CTA:
//   * exact floor(N*0.7f)-th order statistic of the squared match distances
//     (icp_fast.cc:65-90).  Phase A left a 2048-bin histogram, phase B a second-level
//     2048-bin histogram of the members of the quantile bin, so only the handful of keys in
//     ONE second-level bin are ranked exactly;
//   * members of the quantile bin with d2 <= limit join the normal equations.  Phase B parked
//     their Jacobian terms (cand_terms), so a member costs one memory round trip here: members
//     of a lower second-level bin are below the limit by construction and are added while the
//     candidate lists are walked; only the keys of the quantile's own second-level bin wait for
//     the exact limit;
//   * all partial sums are reduced in a fixed order (deterministic result);
//   * warp 0: 6x6 solve, pose update, convergence test, score (icp_fast.cc:204-254,
//     307-321, 377-405, 513-527); with the point-to-point minimizer (kP2P) lane 0 centres the
//     moments and runs the 3x3 SVD of la::kabsch_from_sums instead of the solve (:326-375).  The code is deliberately compact (rolled loops, shared
//     memory): a single warp fetching kilobytes of straight-line code cold costs far more
//     than the arithmetic.
// The per-block candidate lists are never flattened: thread t handles the global candidate
// ranks t, t + 512, ... and finds (block, position) by a binary search over the block offsets
// held in shared memory.
#include "icp_dev.cuh"
#include "linalg_dev.cuh"

namespace smb {
using namespace dev;
namespace {

constexpr int kSelThreads = 512;    // 128 registers per thread: the 29 running sums stay in registers
constexpr int kSelWarps = kSelThreads / 32;
constexpr int kMaxExactKeys = 1024;
constexpr int kStateWords = (int)(sizeof(IcpState) / 8);

struct SolveSmem {
  double S[32];       // reduced sums
  double A[36];       // normal matrix (row-major, symmetric)
  double Z[6][8];     // columns 0..5: L^-1 (certificate), column 6: L^-1 rhs
  double rhs[6], x[6];
  double dT[16], Tn[16], tmp[16];
};

__device__ __noinline__ int solve_exact_path(const double* A, const double* rhs, double* x) {
  return la::solve_possibly_underdetermined(A, rhs, x);
}

// icp_fast.cc:204-254 with a fast path.  The reference asks Eigen's fullPivHouseholderQr
// whether A is invertible (rank 6 at threshold 6*eps*maxpivot) and then solves with LLT.
// For the SPD normal matrix we first factor A = L L^T and bound its condition number by
// trace(A) * ||L^-1||_F^2 >= lambda_max / lambda_min.  Full-pivoting QR keeps every
// |r_kk| >= sigma_k / (6 * 2^5), so a bound below 1e9 certifies rank 6 with five orders
// of magnitude to spare and the pivoted QR is skipped; otherwise the exact restatement
// (QR rank, min-norm branch, SVD fallback) runs.  Returns the path: 0 LLT, 1 min-norm, 2 SVD.
__device__ __forceinline__ int tri(int i, int j) { return (i * (i + 1)) / 2 + j; }

// The 21 entries of the lower triangle live one per lane (lane = tri(i, j)); pivots and
// multipliers travel by shuffle, so a factorisation step is sqrt -> divide -> multiply-subtract
// with no shared-memory round trip in the dependent chain.
__device__ __forceinline__ int solve_warp(SolveSmem& sm, int lane) {
  const int l20 = min(lane, 20);      // lanes 21..31 shadow lane 20 (results ignored)
  int li = 0;
#pragma unroll
  for (int r = 1; r < 6; ++r) li += (l20 >= tri(r, 0)) ? 1 : 0;
  const int lj = l20 - tri(li, 0);
  // S holds the upper triangle row-major: A(i,j) with i >= j is entry (j, i)
  double a = sm.S[lj * 6 - (lj * (lj - 1)) / 2 + (li - lj)];
  const double trace = warp_sum((li == lj && lane < 21) ? a : 0.0);
  // The dependent chain of the whole solve is its square roots and divisions (a double-precision
  // sqrt or divide is a ~20-instruction dependent sequence), so each pivot costs ONE such
  // sequence: r = 1/sqrt(d) gives l_kk = d*r and every later division by l_kk is a multiplication
  // by r.  (Eigen's LLT divides; the two differ by rounding only, ~cond(A)*1e-16 relative with
  // cond(A) < 1e9 certified below, against a parity bar of 1e-4.)
  bool ok = true;
  double rinv = 0.0;                  // lane tri(k, k): 1 / l_kk
#pragma unroll 1
  for (int k = 0; k < 6; ++k) {
    const double dkk = __shfl_sync(0xffffffffu, a, tri(k, k));
    ok = ok && (dkk > 0.0);
    const double r = rsqrt(dkk);
    if (lj == k) {
      if (li == k) { a = dkk * r; rinv = r; } else { a = a * r; }
    }
    const double lik = __shfl_sync(0xffffffffu, a, tri(li, k));
    const double ljk = __shfl_sync(0xffffffffu, a, tri(lj, k));   // meaningful for k < lj only
    if (lj > k) a -= lik * ljk;
  }
  // forward substitution on 7 right-hand sides at once, one lane per column: the six unit
  // vectors (columns of L^-1, the certificate) and rhs = -b (first half of LLT::solve,
  // icp_fast.cc:252); lanes 7..31 carry a zero column so that every lane joins the shuffles
  const int c = min(lane, 7);
  double fro2 = 0.0;
#pragma unroll 1
  for (int i = 0; i < 6; ++i) {
    double v = (c < 6) ? ((i == c) ? 1.0 : 0.0) : ((c == 6) ? -sm.S[21 + i] : 0.0);
#pragma unroll 1
    for (int j = 0; j < i; ++j) v -= __shfl_sync(0xffffffffu, a, tri(i, j)) * sm.Z[j][c];
    v *= __shfl_sync(0xffffffffu, rinv, tri(i, i));
    sm.Z[i][c] = v;
    if (c < 6) fro2 += v * v;
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) fro2 += __shfl_xor_sync(0xffffffffu, fro2, o);
  fro2 = __shfl_sync(0xffffffffu, fro2, 0);
  const double cond_bound = trace * fro2;
  const bool certified = ok && (cond_bound < 1e9);   // false for NaN/inf as well
  int path = 0;
  __syncwarp();
  if (certified) {
    // backward substitution L^T x = y, column oriented: lane j carries row j's running value
    double s = (lane < 6) ? sm.Z[lane][6] : 0.0;
#pragma unroll 1
    for (int i = 5; i >= 0; --i) {
      const double ri = __shfl_sync(0xffffffffu, rinv, tri(i, i));
      const double xi = __shfl_sync(0xffffffffu, s * ri, i);
      const double lil = __shfl_sync(0xffffffffu, a, tri(i, min(lane, i)));   // L(i, lane)
      if (lane == i) sm.x[i] = xi;
      if (lane < i) s -= lil * xi;
    }
  } else {
#pragma unroll 1
    for (int idx = lane; idx < 36; idx += 32) {
      const int r = idx / 6, cc = idx % 6;
      const int lo = min(r, cc), hi = max(r, cc);
      sm.A[idx] = sm.S[lo * 6 - (lo * (lo - 1)) / 2 + (hi - lo)];
    }
    if (lane < 6) sm.rhs[lane] = -sm.S[21 + lane];
    __syncwarp();
    if (lane == 0) path = solve_exact_path(sm.A, sm.rhs, sm.x);
  }
  __syncwarp();
  return __shfl_sync(0xffffffffu, path, 0);
}

// C = A * B for column-major 4x4 in shared memory, lanes 0..15 one element each (k-order
// accumulation like la::mul4); C must not alias A or B
__device__ __forceinline__ void mul4_warp(const double* A, const double* B, double* C, int lane) {
  if (lane < 16) {
    const int i = lane & 3, j = lane >> 2;
    double s = A[i] * B[j * 4];
    s += A[i + 4] * B[1 + j * 4];
    s += A[i + 8] * B[2 + j * 4];
    s += A[i + 12] * B[3 + j * 4];
    C[lane] = s;
  }
  __syncwarp();
}

// pose update + convergence + score on warp 0 (icp_fast.cc:307-321,377-405,513-527); `st` is
// the shared-memory copy of the state.  kP2P: dT = [R t; 0 1] of la::kabsch_from_sums over the reduced moments
// (icp_fast.cc:326-375, no NaN guard there), and its return value is the solve path.
template <bool kP2P>
__device__ __forceinline__ void update_pose(IcpState* st, const IcpParams& p, SolveSmem& sm, int path,
                                            int lane) {
  if (kP2P && lane == 0) {
    double R[9], t[3];
    st->solve_path = la::kabsch_from_sums(sm.S, R, t);
#pragma unroll 1
    for (int i = 0; i < 16; ++i) sm.dT[i] = (i % 5 == 0) ? 1.0 : 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) sm.dT[r + 4 * c] = R[r * 3 + c];
      sm.dT[12 + r] = t[r];
    }
  }
  if (!kP2P && lane == 0) {
    const double* x = sm.x;
    st->solve_path = path;
    const double sq = x[0] * x[0] + x[1] * x[1] + x[2] * x[2];
    const double angle = sqrt(sq);
    double axis[3] = {x[0], x[1], x[2]};
    if (sq > 0.0) { axis[0] = x[0] / angle; axis[1] = x[1] / angle; axis[2] = x[2] / angle; }
    double R[9];
    la::angle_axis_to_rotation(angle, axis, R);
    bool has_nan = false;
#pragma unroll 1
    for (int i = 0; i < 9; ++i) has_nan |= isnan(R[i]);
#pragma unroll 1
    for (int i = 3; i < 6; ++i) has_nan |= isnan(x[i]);
    if (has_nan) {
#pragma unroll 1
      for (int i = 0; i < 9; ++i) R[i] = (i % 4 == 0) ? 1.0 : 0.0;
    }
#pragma unroll 1
    for (int i = 0; i < 16; ++i) sm.dT[i] = (i % 5 == 0) ? 1.0 : 0.0;
#pragma unroll 1
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) sm.dT[r + 4 * c] = R[r * 3 + c];
      sm.dT[12 + r] = x[3 + r];
    }
  }
  __syncwarp();
  mul4_warp(sm.dT, st->T_iter, sm.Tn, lane);
  if (lane < 16) st->T_iter[lane] = sm.Tn[lane];
  __syncwarp();
  const double* Tn = sm.Tn;
  int finish = 0;
  if (lane == 0) {
    const int iteration = st->iteration + 1;
    st->iteration = iteration;
    bool conv = false;
    if (!p.disable_convergence) {
      double Rm[9], qn[4];
#pragma unroll 1
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) Rm[r * 3 + c] = Tn[r + 4 * c];
      la::rotation_to_quaternion(Rm, qn);
      const int len = st->hist_len;
      for (int k = 0; k < 4; ++k) st->quat_hist[len % 5][k] = qn[k];
      for (int k = 0; k < 3; ++k) st->trans_hist[len % 5][k] = Tn[12 + k];
      st->hist_len = len + 1;
      if (len + 1 > 4) {
        double rot = 0.0, tr = 0.0;
#pragma unroll 1
        for (int i = len; i >= len + 1 - 4; --i) {
          rot += fabs(la::quaternion_angular_distance(st->quat_hist[i % 5], st->quat_hist[(i - 1) % 5]));
          const double dx = st->trans_hist[i % 5][0] - st->trans_hist[(i - 1) % 5][0];
          const double dy = st->trans_hist[i % 5][1] - st->trans_hist[(i - 1) % 5][1];
          const double dz = st->trans_hist[i % 5][2] - st->trans_hist[(i - 1) % 5][2];
          tr += fabs(sqrt(dx * dx + dy * dy + dz * dz));
        }
        rot /= 4.0; tr /= 4.0;
        conv = rot < 0.001 && tr < 0.01;
      }
    }
    if (conv || iteration >= p.max_iteration) {
      finish = 1;
      st->final_score = exp(-(sm.S[27] / sm.S[28]));
      st->done = 1;
    }
  }
  finish = __shfl_sync(0xffffffffu, finish, 0);
  if (finish) {
    mul4_warp(st->T_mean, Tn, sm.tmp, lane);           // (T_mean * T_iter) * G0, icp_fast.cc:527
    mul4_warp(sm.tmp, st->G0, st->result, lane);
  }
}

// exclusive scan of the candidate counts of blocks [base, base + kSelThreads) into
// blk_off[0..kSelThreads] (the last entry = number of candidates in the chunk)
__device__ __forceinline__ void scan_chunk(const uint32_t* __restrict__ cand_cnt, int base, int nblocks,
                                           uint32_t* blk_off, uint32_t* warp_tot, uint32_t cnt0 = 0u,
                                           bool have_cnt0 = false) {
  const int t = threadIdx.x;
  const int blk = base + t;
  const uint32_t c = (have_cnt0 && base == 0) ? cnt0 : (blk < nblocks ? cand_cnt[blk] : 0);
  uint32_t tot;
  __syncthreads();              // previous users of warp_tot are done
  blk_off[t] = block_scan_excl<kSelWarps>(c, warp_tot, &tot);
  if (t == 0) blk_off[kSelThreads] = tot;
  __syncthreads();
}

__device__ __forceinline__ uint32_t locate_candidate(const uint32_t* blk_off, int base, uint32_t k) {
  int lo = 0, hi = kSelThreads;       // blk_off[lo] <= k < blk_off[hi]
#pragma unroll 1
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (blk_off[mid] <= k) lo = mid; else hi = mid;
  }
  return (uint32_t)((base + lo) * kAccTile) + (k - blk_off[lo]);
}

// f(slot) for every candidate of every phase-B block, slot = index into cand_key / cand_terms.
// The assignment candidate -> thread is fixed (global rank modulo the block size), which keeps the sums
// built on top of it deterministic.  All threads of the block must call this.
template <typename F>
__device__ __forceinline__ void for_each_candidate(const IcpBuffers& b, int nblocks_b, uint32_t* blk_off,
                                                   uint32_t* warp_tot, bool& have_scan, F f) {
  const int t = threadIdx.x;
#pragma unroll 1
  for (int base = 0; base < nblocks_b; base += kSelThreads) {
    if (!have_scan) scan_chunk(b.cand_cnt, base, nblocks_b, blk_off, warp_tot);
    const uint32_t tot = blk_off[kSelThreads];
#pragma unroll 1
    for (uint32_t k = t; k < tot; k += kSelThreads) {
      f(locate_candidate(blk_off, base, k));
    }
  }
  have_scan = nblocks_b <= kSelThreads;   // a single chunk stays valid for the next walk
}

// terms of one candidate as parked by phase B: F[0..5], residual, sqrt(d2)
struct CandTerms { double2 a0, a1, a2, a3; };
__device__ __forceinline__ CandTerms load_candidate(const IcpBuffers& b, uint32_t slot) {
  const double2* o = reinterpret_cast<const double2*>(b.cand_terms + 8 * (int64_t)slot);
  return CandTerms{o[0], o[1], o[2], o[3]};
}
template <bool kP2P>
__device__ __forceinline__ void add_candidate(double* acc, const CandTerms& c, bool member) {
  const double F[6] = {c.a0.x, c.a0.y, c.a1.x, c.a1.y, c.a2.x, c.a2.y};
  if constexpr (kP2P) add_p2p_terms_if(acc, F, F + 3, c.a3.y, member);   // {p, q, 0, sqrt(d2)}
  else add_terms_if(acc, F, c.a3.x, c.a3.y, member);
}

template <bool kP2P>
__global__ void __launch_bounds__(kSelThreads)
icp_finish_kernel(IcpBuffers b, IcpParams p, int nblocks_b) {
  __shared__ IcpState sst;
  __shared__ uint32_t warp_tot[32];
  __shared__ BinSel sel_sm;
  __shared__ int sub_sel[3];                 // second-level bin, count below it, its count
  __shared__ unsigned long long keys[kMaxExactKeys], skeys[kMaxExactKeys];
  __shared__ uint32_t kslot[kMaxExactKeys], sslot[kMaxExactKeys];
  __shared__ uint32_t nkeys;
  __shared__ unsigned long long limit_bits;
  __shared__ uint32_t sh_hist[256];
  __shared__ int sh_rank;
  __shared__ uint32_t blk_off[kSelThreads + 1];
  __shared__ double red[kSelWarps][kNumSums];
  __shared__ SolveSmem solve;
  const int t = threadIdx.x, lane = t & 31, w = t >> 5;
  unsigned long long* gstate = reinterpret_cast<unsigned long long*>(b.state);
  unsigned long long* sstate = reinterpret_cast<unsigned long long*>(&sst);
  static_assert(kStateWords <= kSelThreads, "one state word per thread");
  if (t < kStateWords) sstate[t] = gstate[t];
  if (t == 0) { nkeys = 0; sub_sel[0] = -1; sub_sel[1] = 0; sub_sel[2] = 0; limit_bits = 0ull; }
  __syncthreads();
  if (sst.done) return;
  if (t == 0) sst.stamps[0] = clock64();
  // independent global reads issued together with select_bin's histogram read
  const uint32_t cnt0 = t < nblocks_b ? b.cand_cnt[t] : 0u;
  const uint4 cq = *reinterpret_cast<const uint4*>(b.hist2 + 4 * t);
  const BinSel sel = select_bin(b.hist, p.dist_outlier_ratio, warp_tot, &sel_sm);
  if (sel.nvalid == 0) {
    if (t == 0) { b.state->status = -2; b.state->done = 1; }  // CHECK(!values.empty()), icp_fast.cc:81
    return;
  }
  const int r = sel.qi - sel.below;          // rank inside the quantile bin
  if (t == 0) sst.stamps[1] = clock64();
  bool fallback = clamp_bin(sel.bin);
  if (!fallback) {
    // ---- second-level histogram: 4 bins per thread, block exclusive scan ------------------
    static_assert(kSelThreads * 4 == kHistBins, "4 second-level bins per thread");
    const uint32_t c[4] = {cq.x, cq.y, cq.z, cq.w};
    const uint32_t s = c[0] + c[1] + c[2] + c[3];
    __syncthreads();            // previous users of warp_tot are done
    uint32_t run = block_scan_excl<kSelWarps>(s, warp_tot);
    if ((uint32_t)r >= run && (uint32_t)r < run + s) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if ((uint32_t)r >= run && (uint32_t)r < run + c[q]) { sub_sel[0] = 4 * t + q; sub_sel[1] = (int)run; sub_sel[2] = (int)c[q]; }
        run += c[q];
      }
    }
    __syncthreads();
    if (sub_sel[0] < 0 || sub_sel[2] > kMaxExactKeys) fallback = true;   // block-uniform
  }
  if (t == 0) sst.stamps[2] = clock64();
  double acc[kNumSums];
#pragma unroll
  for (int k = 0; k < kNumSums; ++k) acc[k] = 0.0;
  bool have_scan = false;
  double limit;
  if (!fallback) {
    // ---- one walk over the candidates: lower second-level bins are members outright, the
    //      quantile's own second-level bin is collected for the exact ranking -----------------
    const int sb = sub_sel[0], r2 = r - sub_sel[1];
    constexpr int R = 3;                  // candidates per thread whose loads are in flight together
#pragma unroll 1
    for (int base = 0; base < nblocks_b; base += kSelThreads) {
      if (!have_scan) scan_chunk(b.cand_cnt, base, nblocks_b, blk_off, warp_tot, cnt0, true);
      const uint32_t tot = blk_off[kSelThreads];
#pragma unroll 1
      for (uint32_t k0 = 0; k0 < tot; k0 += kSelThreads * R) {
        uint32_t slot[R]; bool valid[R];
        unsigned long long key[R]; CandTerms ct[R];
#pragma unroll
        for (int q = 0; q < R; ++q) {
          const uint32_t k = k0 + q * kSelThreads + t;
          valid[q] = k < tot;
          slot[q] = valid[q] ? locate_candidate(blk_off, base, k) : 0u;   // slot 0 is always readable
        }
#pragma unroll
        for (int q = 0; q < R; ++q) { key[q] = b.cand_key[slot[q]]; ct[q] = load_candidate(b, slot[q]); }
#pragma unroll
        for (int q = 0; q < R; ++q) {
          const int sub = (int)((key[q] >> 36) & 2047ull);
          add_candidate<kP2P>(acc, ct[q], valid[q] && sub < sb);
          if (valid[q] && sub == sb) {
            const uint32_t j = atomicAdd(&nkeys, 1u);
            if (j < (uint32_t)kMaxExactKeys) { keys[j] = key[q]; kslot[j] = slot[q]; }
          }
        }
      }
    }
    have_scan = nblocks_b <= kSelThreads;
    __syncthreads();
    if (t == 0) sst.stamps[3] = clock64();
    // rank by counting; ties broken by slot so that every key gets a unique, run-independent
    // position (the order the atomics filled keys[] in does not matter)
    const int nk = min((int)nkeys, kMaxExactKeys);
#pragma unroll 1
    for (int i = t; i < nk; i += kSelThreads) {
      const unsigned long long my = keys[i];
      const uint32_t myslot = kslot[i];
      int pos = 0;
#pragma unroll 1
      for (int j = 0; j < nk; ++j) {
        const unsigned long long o = keys[j];
        pos += (o < my) || (o == my && kslot[j] < myslot);
      }
      skeys[pos] = my; sslot[pos] = myslot;
    }
    __syncthreads();
    if (t == 0) limit_bits = (r2 >= 0 && r2 < nk) ? skeys[r2] : 0ull;
    __syncthreads();
    limit = __longlong_as_double((long long)limit_bits);
#pragma unroll 1
    for (int i = t; i < nk; i += kSelThreads)   // non-negative doubles order like their bit patterns
      if (skeys[i] <= limit_bits) add_candidate<kP2P>(acc, load_candidate(b, sslot[i]), true);
  } else {
    // ---- general path (clamp bins, e.g. identical clouds: all d2 == 0): MSB radix select ---
    if (t == 0) { sh_rank = r; limit_bits = 0ull; }
    __syncthreads();
#pragma unroll 1
    for (int pass = 7; pass >= 0; --pass) {
      const int shift = pass * 8;
      if (t < 256) sh_hist[t] = 0;
      __syncthreads();
      const unsigned long long prefix = limit_bits;
      const unsigned long long mask = (pass == 7) ? 0ull : (~0ull << (shift + 8));
      for_each_candidate(b, nblocks_b, blk_off, warp_tot, have_scan, [&](uint32_t slot) {
        const unsigned long long key = b.cand_key[slot];
        if ((key & mask) == prefix) atomicAdd(&sh_hist[(key >> shift) & 255ull], 1u);
      });
      __syncthreads();
      if (w == 0) {   // parallel digit search: 8 bins per lane
        uint32_t c[8], s = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) { c[k] = sh_hist[lane * 8 + k]; s += c[k]; }
        const uint32_t excl = warp_inclusive_scan(s) - s;
        const uint32_t rk = (uint32_t)sh_rank;
        __syncwarp();
        if (rk >= excl && rk < excl + s) {
          uint32_t run = excl;
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            if (rk >= run && rk < run + c[k]) {
              sh_rank = (int)(rk - run);
              limit_bits = prefix | ((unsigned long long)(lane * 8 + k) << shift);
            }
            run += c[k];
          }
        }
      }
      __syncthreads();
    }
    limit = __longlong_as_double((long long)limit_bits);
    // ---- members of the quantile bin with d2 <= limit (icp_fast.cc:497-498) ---------------
    for_each_candidate(b, nblocks_b, blk_off, warp_tot, have_scan, [&](uint32_t slot) {
      const double d2 = __longlong_as_double((long long)b.cand_key[slot]);
      if (d2 <= limit) add_candidate<kP2P>(acc, load_candidate(b, slot), true);
    });
  }
  if (t == 0) sst.stamps[4] = clock64();
  // ---- fixed-order reduction: candidates of this kernel + phase-B partials ---------------------
  // after the transposed warp reduction lane k holds the warp's total of sum k; the same lane
  // adds the k-th entry of the phase-B partials of blocks w, w + 32, ... (coalesced rows)
  {
    double v32[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) v32[k] = k < kNumSums ? acc[k] : 0.0;
    double v = warp_transpose_reduce32(v32, lane);
#pragma unroll 1
    for (int blk0 = w; blk0 < nblocks_b; blk0 += kSelWarps * 8) {
      double pv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {       // the 8 loads go out together
        const int blk = blk0 + kSelWarps * i;
        pv[i] = (blk < nblocks_b && lane < kNumSums) ? b.partials[(int64_t)blk * 32 + lane] : 0.0;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) v += pv[i];
    }
    if (lane < kNumSums) red[w][lane] = v;
  }
#pragma unroll 1
  for (int k = t; k < 2 * kHistBins; k += kSelThreads) b.hist[k] = 0;   // hist, hist2
  __syncthreads();
  if (t == 0) sst.stamps[5] = clock64();
#pragma unroll 1
  for (int k = w; k < kNumSums; k += kSelWarps) {
    double v = lane < kSelWarps ? red[lane][k] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) { solve.S[k] = v; b.sums[k] = v; }
  }
  __syncthreads();
  if (w != 0) return;
  // ---- warp 0: solve + pose update -----------------------------------------------------------
  if (lane == 0) sst.stamps[6] = clock64();
  const double kept = solve.S[28];
  if (lane == 0) { sst.limit = limit; sst.kept = (long long)kept; }
  if (!(kept > 0.0)) {
    if (lane == 0) {   // "no point to minimize", icp_fast.cc:114
      b.state->limit = limit; b.state->kept = (long long)kept; b.state->status = -3; b.state->done = 1;
    }
    return;
  }
  const int path = kP2P ? 0 : solve_warp(solve, lane);
  if (lane == 0) sst.stamps[7] = clock64();
  update_pose<kP2P>(&sst, p, solve, path, lane);
  if (lane == 0) sst.stamps[8] = clock64();
#ifdef SMB_FINISH_EXPERIMENT
  {   // how long does the same solve take with its code already fetched?
    const int path2 = solve_warp(solve, lane);
    if (lane == 0) { sst.stamps[9] = clock64(); sst.stamps[10] = path2; }
  }
#endif
  __syncwarp();
#ifdef SMB_ACC_SECTIONS
  // the stamps hold phase B's section sums in this build (icp.cu) and stay as phase B left them
  constexpr int kCopyWords = (int)(offsetof(IcpState, stamps) / 8);
#else
  constexpr int kCopyWords = kStateWords;
#endif
#pragma unroll 1
  for (int i = lane; i < kCopyWords; i += 32) gstate[i] = sstate[i];
}

}  // namespace

void icp_finish_launch(const IcpBuffers& b, const IcpParams& p, int nblocks_b, cudaStream_t stream) {
  if (p.error_minimizer == kIcpPointToPoint) icp_finish_kernel<true><<<1, kSelThreads, 0, stream>>>(b, p, nblocks_b);
  else icp_finish_kernel<false><<<1, kSelThreads, 0, stream>>>(b, p, nblocks_b);
}

}  // namespace smb
