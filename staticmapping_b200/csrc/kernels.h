// Internal host-side launch API shared by the .cu translation units of libsm_b200.
#ifndef SM_B200_KERNELS_H_
#define SM_B200_KERNELS_H_

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <utility>
#include <vector>

#include "common.cuh"

struct sm_filter_chain;
struct sm_plane_sampler;

namespace smb {

// One device allocation, freed with its owner.  reserve() only grows, with 1/8 + 4 KB slack so
// that clouds of slightly varying size keep their buffers: the IcpFast graph keys hash buffer
// pointers, and a reallocation means a new capture.
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }   // move-only
  DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~DevBuf() { if (p) cudaFree(p); }
  int reserve(size_t bytes) {
    if (bytes <= cap) return 0;
    if (p) { SMB_CUDA_OK(cudaFree(p)); p = nullptr; cap = 0; }
    const size_t want = bytes + bytes / 8 + 4096;
    SMB_CUDA_OK(cudaMalloc(&p, want));
    cap = want;
    return 0;
  }
};

// ---- radix_sort.cu ---------------------------------------------------------------------
size_t radix_sort_scratch_bytes(int n, int batch);
// One sort of up to `stride` (key, value) pairs: the ping-pong buffers and the scratch, carved from one
// allocation of bytes(stride, n) bytes.
struct RadixPairs {
  uint64_t* keys[2];
  uint32_t* vals[2];
  uint32_t* scratch;
  static size_t bytes(int64_t stride, int n);
  void carve(void* base, int64_t stride);
};
int radix_sort_pairs_u64(uint64_t* keys_a, uint32_t* vals_a, uint64_t* keys_b, uint32_t* vals_b,
                         int n, int batch, int64_t stride, uint32_t* scratch,
                         cudaStream_t stream, int passes = 8);
// exclusive scan of `count` u32 per batch (in place), one block per batch
void radix_scan_kernel_launch(uint32_t* data, int count, int batch, cudaStream_t stream);

// ---- kdtree.cu -------------------------------------------------------------------------
int kd_num_levels(int n, int bucket);
struct KdWorkspace {
  uint64_t* keys[2];
  uint32_t* lists[2];
  uint32_t* gloc;
  uint8_t* flag;
  uint32_t* scratch;
  double* bounds[2];
  int* level_dim;
  int64_t lstride;
  int carve(DevBuf& buf, int n, int bucket);   // grows buf to what (n, bucket) needs, then carves it
};
// Compact search layout of a tree built by kd_build, shaped for a shared-memory resident traversal:
//   cut[h], dim[h]  heap order (children of h: 2h+1, 2h+2) for the levels above the deepest
//                   leaf level; dim 3 = leaf.  8 + 1 bytes per node: the 14 inner levels of a
//                   ~107 k-point target are 144 KB and are staged into shared memory with bulk
//                   async copies (cp.async.bulk + mbarrier) once per CTA;
//   pb              padded buckets, x[8] y[8] z[8] doubles per leaf slot of the deepest level
//                   (+inf padding), so a leaf's bucket address is pure index arithmetic and a
//                   bucket scan is 12 aligned 16-byte loads;
//   pm, pid         per padded entry (entry = bucket * 8 + k): the point and its normal in one 64-byte record
//                   (what ICP phase B gathers per match; the search reads pb only) / the original id.
struct KdCompact {
  const double* cut;
  const uint8_t* dim;
  const double2* node;    // {cut, dim as a 64-bit integer} of heap node h at slot h + 1, 2^levels slots: the
                          // search reads the levels below the shared-memory ones with one 16-byte load per node
  const double* pb;
  const BucketMatch* pm;
  const int32_t* pid;
  int levels;
  int pad;                // set too: IcpBuffers embeds this struct, and its bytes are a graph key
};
// The device buffers of one tree in the compact layout, with its blocked node array and leaf order.  reserve()
// sizes them for (n, bucket) with one payload per padded entry, the point + normal records (pm) or the original
// ids (pid); they only grow, so a tree of the same size keeps its pointers.  build() fills them.
struct KdCompactTree {
  enum Payload { kNormals, kIds };
  DevBuf nodes, leaf_order, cut, dim, pb, pm, pid;   // cut: cut[] then node[]
  int levels = 0;
  int reserve(int n, int bucket, Payload payload);
  // coord / nrm: SoA [3][cstride]; nrm only with the kNormals payload
  int build(const double* coord, const double* nrm, int64_t cstride, int n, int bucket, KdWorkspace& ws,
            cudaStream_t stream) const;
  KdCompact view() const;
};
// compact (optional): also write its node arrays
// coords_are_float: every coordinate is exactly a float (clouds uploaded as float): 32-bit sort keys
int kd_build(const double* coord, int64_t cstride, int n, int bucket, KdWorkspace& ws, KdNode* nodes,
             uint32_t* leaf_order, cudaStream_t stream, const KdCompactTree* compact = nullptr,
             bool coords_are_float = false);

// k-d tree over a packed float cloud (fitness scores, GICP correspondences, the type-1 score): the cloud as
// SoA doubles, the blocked node array, the leaf order and the buckets; kdws is the build workspace.
struct FloatTree {
  DevBuf soa, nodes, order, bpts;
  int build(const float* pts, int n, DevBuf& kdws, cudaStream_t stream);
};

// ---- icp.cu ----------------------------------------------------------------------------
constexpr int kHistBins = 2048;

// Device-resident state of one IcpFast::Align call (one per handle).
struct IcpState {
  double T_iter[16];      // column-major, accumulated iteration transform
  double G0[16];          // T_mean^-1 * guess
  double T_mean[16];
  double result[16];
  double mean[3];
  double final_score;
  double quat_hist[5][4]; // ring of the last 5 rotations (w,x,y,z)
  double trans_hist[5][3];
  double limit;           // last quantile limit (debug / parity)
  long long kept;         // last K
  int hist_len;           // number of entries pushed (incl. the initial identity)
  int iteration;
  int done;               // 1 once converged or max_iteration reached
  int status;             // 0 ok, <0 error (-2 no finite distance, -3 nothing kept)
  int solve_path;         // 0 LLT, 1 min-norm, 2 SVD; point-to-point: 3 Kabsch, 4 with the reflection fix (last iteration)
  int pad;
  long long stamps[12];   // clock64 at the section boundaries of the last finish kernel (diagnostics)
};
static_assert(sizeof(IcpState) % 8 == 0, "IcpState is copied as 8-byte words");

struct IcpParams {
  int n_source, n_target;
  int max_iteration;
  float dist_outlier_ratio;
  double max_error2;       // (1+eps)^2
  int disable_convergence;
  int tree_levels;         // kd_num_levels(n_target, 8): depth of the root-to-leaf path
  int knn_queries_per_cta; // phase A: 0 = one query per thread, else queries per 256-thread CTA
  // host-side selectors (no kernel reads them; they pick the instantiations and are part of the graph keys).  Both
  // are 16 bits so that they share the 4 bytes inner_compensation had as an int: the struct stays 40 bytes with no
  // padding, and no kernel argument moves.
  int16_t inner_compensation;  // 1: IcpFast::EnableInnerCompensation, the source is de-skewed in every iteration
  int16_t error_minimizer;     // kIcpPointToPlane or kIcpPointToPoint (phases B and C)
};
static_assert(sizeof(IcpParams) == 40, "the two 16-bit selectors share inner_compensation's former 4 bytes: kernel argument offsets stay put");
constexpr int kIcpPointToPlane = 0, kIcpPointToPoint = 1;   // sm_icp_error_minimizer

struct IcpBuffers {
  // target (caller order, SoA, centred in place by the prologue)
  double* tgt;            // [3][tstride]
  double* tgt_raw;        // [3][tstride] as uploaded (un-centred)
  double* nrm;            // [3][tstride]
  int64_t tstride;
  // tree: build-time node array (blocked layout), leaf order, and the compact search layout
  KdNode* nodes;
  uint32_t* leaf_order;
  KdCompact kc;
  // source
  double* src_raw;        // [3][sstride] as uploaded
  double* src_g0;         // [3][sstride] after G0, caller order
  double* src0;           // [3][sstride] after G0, Morton order (what the iterations read)
  RadixPairs src_sort;    // Morton keys and the permutation
  int64_t sstride;
  // per-iteration
  int32_t* slot;          // [n_source] padded bucket entry of the match (kc.pb / kc.pm index)
  int4* knn_items;        // [knn_items_bytes(n_source)] parked searches of the k-NN kernel's second phase (16 B each)
  double* d2;             // [n_source]
  uint32_t* hist;         // [kHistBins] first-level histogram of dist^2 (phase A)
  uint32_t* hist2;        // [kHistBins] second-level histogram inside the quantile bin (phase B)
  double* sums;           // [32] the iteration's 29 reduced normal-equation sums, written by phase C before it tests
                          // the kept count (a record for tests; nothing reads it back)
  double* cand_terms;     // [blocks*tile][8] per-block compacted candidates (members of the quantile bin):
                          // the 6 Jacobian terms, the residual and sqrt(d2) of the match (phase B -> C)
  unsigned long long* cand_key;  // [blocks*tile] bit pattern of the candidate's dist^2
  uint32_t* cand_cnt;     // [accum blocks]
  double* partials;       // [accum blocks][32]
  double* mean_partials;  // [blocks][4]
  IcpState* state;
};

size_t knn_items_bytes(int nq);   // the parked searches of the batched k-NN kernels for nq queries

// The device buffers of IcpFast's iterations and its target tree.  reserve() sizes them for ns source / nt target
// points in SoA clouds of strides sstride / tstride (deskewed with inner compensation only); they only grow, so
// clouds of the same size keep their pointers and the captured graphs.  fill() lays them out as IcpBuffers.
struct IcpFastBuffers {
  DevBuf tgt, src0, src_g0, src_sort, slot, d2, hist, cand_terms, cand_key, cand_cnt, partials, mean_partials, state,
      guess, deskewed;
  KdCompactTree tree;
  int ns = 0;
  int64_t sstride = 0, tstride = 0;
  int reserve(int ns, int nt, int64_t sstride, int64_t tstride, bool inner_compensation);
  void fill(IcpBuffers& b, const double* tgt_raw, const double* nrm, const double* src_raw) const;
};

// builds the target tree into `tree`, whose view is b.kc
int icp_prologue(const IcpBuffers& b, const IcpParams& p, const double* guess_dev,
                 KdWorkspace& ws, const KdCompactTree& tree, cudaStream_t stream);
int icp_prologue_launches(int tree_levels);
// events (optional): 4 per iteration — before A, after A, after B, after C
// deskewed: [3][sstride] doubles, the de-skewed source of the iteration; needed when p.inner_compensation
int icp_enqueue_iterations(const IcpBuffers& b, const IcpParams& p, int start_iteration, int count,
                           cudaStream_t stream, cudaEvent_t* events, double* deskewed = nullptr);
int icp_iteration_launches(bool inner_compensation);
// The phases of one iteration, in the order icp_enqueue_iterations runs them (the stage test hook runs them one at a
// time): icp_deskew_launch with inner compensation, then A, B and C.  nblocks_b = icp_accum_blocks(p.n_source).
void icp_search_launch(const IcpBuffers& b, const IcpParams& p, const double* deskewed, cudaStream_t stream);
void icp_accum_launch(const IcpBuffers& b, const IcpParams& p, const double* deskewed, cudaStream_t stream);
void icp_finish_launch(const IcpBuffers& b, const IcpParams& p, int nblocks_b, cudaStream_t stream);
int icp_accum_blocks(int n_source);
// stand-alone k-NN over an already built tree (compact layout incl. pid): ids = original indices
int knn_query(const KdCompact& kc, const double* query, int64_t qstride, int nq, double max_error2,
              int32_t* ids, double* d2, cudaStream_t stream, int queries_per_cta = 0, int4* items = nullptr);

// ---- knn.cu ------------------------------------------------------------------------------
// libnabo's k-NN (KDTREE_LINEAR_HEAP) over an already built tree (compact layout incl. pid), k = 1..64: ids / d2 are
// nq x k row-major, each row ascending, (-1, +inf) where fewer than k points qualify.  max_radius2 = maxRadius^2.
int knn_k_query(const KdCompact& kc, const double* query, int64_t qstride, int nq, int k, double max_error2,
                double max_radius2, bool allow_self_match, int32_t* ids, double* d2, cudaStream_t stream);
// StatisticalOutlierRemoval's mean distance over the same search: for each query i, its mean_k + 1 (<= 64) nearest
// points (eps = 0, self-match allowed, no radius), entry 0 dropped, mean_k terms of statistic_removal.cuh; the float
// lands at dist[qindex[i]].  The tree must hold more than mean_k points.
int knn_mean_distance_query(const KdCompact& kc, const double* query, int64_t qstride, int nq, int mean_k,
                            const uint32_t* qindex, float* dist, cudaStream_t stream);

// ---- motion.cu ---------------------------------------------------------------------------
// one iteration's de-skewed source of IcpFast with inner compensation: out = Interp(T_iter, f_i) (x) src0_i
void icp_deskew_launch(const IcpBuffers& b, const IcpParams& p, double* out, cudaStream_t stream);

// ---- ndt.cu ------------------------------------------------------------------------------
struct NdtGrid {            // VoxelGridCovariance bookkeeping (_impl.hpp:88-103)
  float inv_leaf;
  int min_b[3], div_b[3], mul[3];
  int n_voxels;
  int overflow;             // 1: the box holds more than INT32_MAX voxels (_impl.hpp:74-84), the grid is unusable
};
struct NdtLeaf {            // VoxelGridCovariance::Leaf (voxel_grid_covariance_omp.h:92-186)
  double mean[3];
  double icov[9];           // zero for leaves that failed the eigenvalue test
  float centroid[3];
  int nr_points;            // -1: invalid covariance (still searchable, like the reference)
  int searchable;           // >= min_points_per_voxel: centroid is in the search cloud
  int pad;
};
struct NdtEvalParams {      // everything one computeDerivatives call needs, by value
  float T[16];              // final_transformation_, column-major
  float j_ang[8][3];        // computeAngleDerivatives (ndt_omp_impl.hpp:288-393)
  float h_ang[15][3];
  double gauss_d1, gauss_d2;
  float radius;             // resolution_
  int f64_math;             // 1: stock pcl::NormalDistributionsTransform term math (double), the
                            //    class NdtWithGicp uses; 0: pclomp's single-precision math
  double j_ang_d[8][3];     // the same tables in double (stock PCL keeps them as Vector3d)
  double h_ang_d[15][3];
};
// pclomp's NeighborSearchMethod (ndt_omp.h:52-57), same values as sm_ndt_search_method
enum NdtSearch : int { kNdtKdtree = 0, kNdtDirect26 = 1, kNdtDirect7 = 2, kNdtDirect1 = 3 };
// host build of the direct neighbour searches of ndt.cu (test hook sm_debug_ndt_direct_neighbors): the keys of the
// in-box offset cells of point x in offset order, at most 26; returns their number
int ndt_debug_direct_cells_host(int search, const float* x, float leaf, const NdtGrid& g, int* keys26);
// the leaf test the kernel applies to those cells: nr_points >= min_points_per_voxel_
bool ndt_debug_direct_leaf_accepted_host(int nr_points);
// host build of the leaf plane fit of normals.cu (test hook sm_debug_normals_leaf): 1 kept, 0 dropped, < 0 bad count
int normals_debug_leaf_host(const double* members, int count, double* mean, double* unit);
// host build of the eigenvector leaf of normals.cu (test hook sm_debug_pm_surface_normal_leaf_host), float members;
// mean, row-major covariance and normal as the leaf computes them: 1 kept, 0 dropped, < 0 bad count
int pm_normals_debug_leaf_host(const float* members, int count, float* mean, float* cov, float* unit);
// host build of one target-grid leaf of ndt.cu (test hook sm_debug_ndt_leaf)
void ndt_debug_leaf_host(const float* pts, int n, int min_points, double eig_mult, double* mean3, double* icov9,
                         float* centroid3, int* nr_points, int* searchable);
// host build of the per-(point, voxel) derivative term of ndt.cu (test hook sm_debug_ndt_term)
void ndt_debug_term_host(const NdtEvalParams& P, const float* x_orig, const float* x_trans, const double* mean,
                         const double* icov, double* out43);
struct NdtWorkspace {
  uint64_t* keys[2];
  uint32_t* order[2];
  uint32_t* scratch;
  uint32_t* voxel_start;
  int* voxel_key;
  NdtLeaf* leaves;
  int* table_key;
  int* table_val;
  uint32_t table_size;
  double* partials;
  double* sums;             // [64] reduced outputs
  float* minmax;
  float* sorted_pts;        // target points gathered into voxel order (packed xyz)
  NdtGrid* grid;
  int64_t stride;
};
// The NDT target grid and the evaluation sums of one Align, carved from one allocation sized by reserve() for nt
// target / ns source points.  eval reads computeDerivatives' 44 sums (score, gradient, Hessian row-major, neighbour
// count) back into host memory, fitness getFitnessScore's 2 (squared-distance sum, count) through sums2.
struct NdtStage {
  DevBuf buf;
  NdtWorkspace ws;
  int reserve(int nt, int ns);
  int build_grid(const float* tgt, int nt, float resolution, cudaStream_t stream);   // setInputTarget -> init()
  static constexpr int kGridLaunches = 12 + 12;
  int eval(const float* src, int ns, const NdtEvalParams& P, int search, double* sums44, cudaStream_t stream);
  static constexpr int kEvalLaunches = 2;
  int fitness(const float* src, int ns, const float* tgt, const float* T, const FloatTree& t, double* sums2,
              cudaStream_t stream, double* score);
  static int fitness_launches(int nt);   // with the build of the target's float tree
};
int ndt_float_to_soa(const float* pts, int n, double* soa, int64_t stride, cudaStream_t stream);

// ---- gicp.cu -----------------------------------------------------------------------------
struct GicpIterParams {     // one outer GICP iteration (gicp_omp_impl.hpp:414-461)
  float guess[16];          // base transformation (NDT result), column-major
  float transformation[16]; // transformation_ of this iteration
  double R[9];              // rotation of transformation_ * guess, row-major, double
  double dist_threshold;    // corr_dist_threshold_^2
};
struct GicpCostParams {     // one BFGS function evaluation (:255-377)
  float T[16];              // base with applyState(x)
  float base[16];
};
// host builds of the three voxel-index functions (test hook sm_debug_voxel_index)
bool vf_debug_index_host(const float* p, float voxel, long long* ixyz);
int ndt_debug_voxel_coord_host(float v, float inv_leaf, int min_b);
void gicp_debug_approx_cell_host(const float* p, float inv, int* ixyz, uint32_t* slot);
// host builds of gicp.cu's per-point arithmetic (test hook sm_debug_gicp_point)
void gicp_debug_mahalanobis_host(const double* R, const double* C1, const double* C2, double* out9);
void gicp_debug_cost_terms_host(const float* T, const float* base, const float* ps, const float* pt, const double* M,
                                double* acc13);
// pcl::ApproximateVoxelGrid::filter of packed float clouds into out (grown to room for n points): the workspace and
// the output count m, which filter() reads back between its two halves.
struct ApproxVoxelGrid {
  DevBuf ws, counter;
  int filter(const float* pts, int n, float leaf, DevBuf& out, int* m, cudaStream_t stream);
};
// test hook sm_debug_float_tree_knn: knn1 (eps = 0, k = 1) or knn_k (k = 20) over t for nq AoS double queries
int float_tree_debug_knn(const FloatTree& t, const double* q, int nq, int k, int32_t* ids, double* d2,
                         cudaStream_t stream);

// ---- normals.cu ------------------------------------------------------------------------
// The leaf routine of the normals pipeline, same values as sm_pm_surface_normals: CalculateNormals' least-squares
// plane (double) or libpointmatcher SamplingSurfaceNormal's smallest eigenvector of the box covariance (float)
enum NormalsMode : int { kNormalsLeastSquares = 0, kNormalsEigenvector = 1 };
// The device buffers of CalculateNormals over n points, sized by reserve(n): the input cloud, the bucket-7 tree
// with its workspace, the per-leaf scratch, and the AoS 3xM outputs with their count M.
struct NormalsPipeline {
  DevBuf coord, nodes, order, kdws, tmp_pts, tmp_nrm, keep, bsum, out_pts, out_nrm, count;
  DevBuf perm, nth_key, lpos, rpos, nth_bounds;   // std::nth_element's order only, sized by run_nth_element
  int64_t stride = 0;
  int reserve(int n);
  double* input() const { return (double*)coord.p; }   // SoA [3][stride], filled by the caller
  // runs the pipeline with the given leaf routine on the first n points of input() and waits for M; keep then holds
  // 1 at the smallest member index of every kept box (the outputs' source positions, in order)
  int run(int n, NormalsMode mode, cudaStream_t stream, uint32_t* m);
  // CalculateNormals in the order std::nth_element leaves (SM_NORMALS_ORDER_NTH_ELEMENT): the least-squares leaf over
  // the members in that order, keep set at each leaf's first member; perm then holds the recursion's index array.
  // SM_ERR_BAD_ARGUMENT, with nothing written, if a coordinate is not finite.
  int run_nth_element(int n, cudaStream_t stream, uint32_t* m);
  int fit_leaves(int n, NormalsMode mode, const uint32_t* leaf_order, cudaStream_t stream, uint32_t* m);
  const double* points() const { return (const double*)out_pts.p; }
  const double* normals() const { return (const double*)out_nrm.p; }
};

// ---- nth_element.cu --------------------------------------------------------------------
// BuildNormals' index array over the first n points of coord (SoA [3][cstride]) as std::nth_element leaves it;
// perm, key, lpos, rpos: n entries each; bounds: nth_element_bounds_bytes(n) of scratch
int nth_element_recursion(const double* coord, int64_t cstride, int n, uint32_t* perm, double* key, uint32_t* lpos,
                          uint32_t* rpos, double* bounds, cudaStream_t stream);
size_t nth_element_bounds_bytes(int n);
// *bad = some coordinate of the first n points is not finite; flag_dev: one device word of scratch.  Waits.
int any_nonfinite(const double* coord, int64_t cstride, int n, uint32_t* flag_dev, cudaStream_t stream, bool* bad);
// test hook: one CTA's std::nth_element(nth) over n device keys -> perm; key, lpos, rpos: n entries of scratch
int nth_element_single(const double* keys, int n, int nth, uint32_t* perm, double* key, uint32_t* lpos,
                       uint32_t* rpos, cudaStream_t stream);

// ---- icp_pm.cu -------------------------------------------------------------------------
// glibc's rand() stream (TYPE_3, degree 31) as 31 consecutive words of its additive recurrence: the window at
// position p (p draws taken since srand) is the one whose next draw is draw p.
constexpr int kPmRandDeg = 31;
struct PmRandWindow { uint32_t w[kPmRandDeg]; };
// the window at `position` after srand(seed), in O(log position) (icp_pm.cu)
PmRandWindow pm_rand_window(uint32_t seed, uint64_t position);
// host builds of the generator (test hooks sm_debug_pm_rand_*_host): the window m draws further on, and count draws
void pm_rand_debug_advance_host(PmRandWindow& at, uint64_t m);
void pm_rand_debug_draws_host(PmRandWindow at, int64_t count, int32_t* out);

// The reading filter and the score pass of the IcpUsingPointMatcher stand-in (icp_pointmatcher.cc:131-148, :173),
// with their buffers, sized by reserve() for a reading cloud of n_source points.
struct PmStage {
  DevBuf cnt, sampled, score;   // tile counts; the kept reading points; pose, output and sort of the score pass
  DevBuf rand_flags;            // the rand sampler's keep flags, one bit per point
  int reserve(int n_source);
  // subsample of the packed float cloud src into points(); waits for and returns the number kept.  With rand null,
  // point i is kept by the counter hash of (i, seed); with rand, by (float)rand() / (float)RAND_MAX < prob where
  // point i takes the i-th draw from the window *rand (libpointmatcher's RandomSamplingDataPointsFilter).
  int sample(const float* src, int n, float prob, uint32_t seed, cudaStream_t s, uint32_t* kept,
             const PmRandWindow* rand = nullptr);
  const uint32_t* rand_bits() const { return (const uint32_t*)rand_flags.p; }   // after a rand sample: n flag bits
  const double* points() const { return (const double*)sampled.p; }   // AoS 3xM doubles
  // the unfiltered reading moved by T (16 doubles, pinned host memory) against the target's float tree, trimmed at
  // `ratio`; waits for out3_host = mean kept distance, kept, valid
  int score_pass(const float* src, int n, const double* T_host_pinned, const FloatTree& target, double max_error2,
                 float ratio, double* out3_host, cudaStream_t s);
  // the last score pass's n squared distances in ascending order, as sorted bit patterns (+inf = no match)
  const uint64_t* sorted_keys() const;
};

// ---- m2dp.cu -----------------------------------------------------------------------------
struct M2dpView { float xa[3], ya[3]; };   // x_axis, y_axis of one view (m2dp.cc:73-83), not normalised
static_assert(sizeof(M2dpView) == 6 * sizeof(float), "the test hook copies views as 6 floats each");
// The device work of M2dp::setInputCloud over n >= 1 records of stride_bytes (float xyz first): the buffers, carved
// from one allocation, and the mean, covariance, histogram and Gram kernels with the host steps between them.  run()
// leaves every intermediate in host memory: the float mean, the six double covariance sums (xx xy xz yy yz zz) and
// the float covariance entries sum / float(n - 1), the axes E = m2dp_axes(cov), the view axes, A (rows x cols counts,
// row-major) and G = A A^T.
struct M2dpStage {
  DevBuf buf;
  int rows = 0, cols = 0, l = 0;
  float mean[3];
  double cov_sums[6];
  float cov[6];
  float E[9];                // E[k * 3 + j]: component k of axis j
  std::vector<M2dpView> views;
  std::vector<int> A;
  std::vector<double> G;
  int run(const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance, int t, int p, int q,
          cudaStream_t stream);
};
// the PCA axes from the six float covariance entries: descending eigenvalue, largest-magnitude component positive,
// third = first x second in float; the identity when an entry is not finite
void m2dp_axes(const float* cov6, float* E9);
// [u1; v1] (rows + cols floats) from A and G = A A^T; zero when A is
void m2dp_descriptor(const int* A, const double* G, int rows, int cols, float* out);

// ---- filters.cu --------------------------------------------------------------------------
// pre_processers::filter::Factory (pre_processors/filter_factory.cc:63-106) over the six filters built here, and
// with the chain option all_filters over the reference's other three: kFilterStatisticRemoval, kFilterGroundRemoval
// and kFilterVoxelGrid, whose stages (StatisticRemoval, GroundRemoval, VoxelGrid below) also run behind their own
// entry points, sm_statistic_removal (statistic_removal.cu), sm_ground_removal (ground_removal.cu) and
// sm_voxel_grid_filter (voxel_filter.cu).
enum FilterKind : int {
  kFilterRange = 0, kFilterAxisRange, kFilterBoundingBoxRemoval, kFilterRandomSampler, kFilterRangeImage,
  kFilterGroundRemoval2, kFilterStatisticRemoval, kFilterGroundRemoval, kFilterVoxelGrid
};
// One filter of the chain: the members of the reference class of its kind under their XML names, at the
// constructors' defaults (filter_range.cc:31-38, filter_axis_range.h:56-57, filter_bounding_box.h,
// filter_random_sample.cc:29, filter_range_image.cc:29-37, filter_ground_removal2.cc:74-89,
// filter_statistic_removal.h, filter_ground_removal.cc:29-39, filter_voxel_grid.h:55).  Passed to the kernels by
// value.  StatisticRemoval's two members, VoxelGrid's one and RandomSampler's generator share Range's storage and
// GroundRemoval's three AxisRange's: a FilterParams holds the parameters of one kind, and its size and layout are what
// the chain's kernels take.
struct FilterParams {
  int kind;
  union {
    struct { float min_range, max_range; };                         // Range
    struct { int32_t point_num_meank; float std_mul; };             // StatisticRemoval
    struct { float voxel_size; int32_t voxel_order; };              // VoxelGrid (sm_filter_chain_set_voxel_order)
    struct { int32_t sampler_mode; uint32_t sampler_seed; };        // RandomSampler (sm_filter_chain_set_random_sampler)
  };
  union {
    struct { float min, max; int axis_index; };                     // AxisRange
    struct { int32_t min_point_num_in_voxel; float leaf_size, height_threshold; };   // GroundRemoval
  };
  float min_x, min_y, min_z, max_x, max_y, max_z;                   // BoundingBoxRemoval
  float sampling_rate;                                              // RandomSampler
  float top_angle, btm_angle, offset_x, offset_y, offset_z;         // RangeImage
  int vertical_line_num, horizontal_line_num;
  float r_max, r_min, start_ground_height, long_line_threshold,     // GroundRemoval2
      max_long_line_height, max_start_height, max_error, max_slope, max_b, max_dist_to_line, search_angle;
  int bin_num, segment_num, thread_num;
};
static_assert(sizeof(FilterParams) == 136, "the chain's kernels take FilterParams by value: its layout stays put");
FilterParams filter_defaults(int kind);
// the reference's name for `kind`'s parameter -> its address and type (0 int32, 1 float), or false
bool filter_param(FilterParams& f, const char* name, void** target, int* type);
// One <param type=... name=...>text</param> of Interface::InitFromXmlNode on `f`: pugixml's as_int / as_float by the
// XML type, then XmlInterface::SetValue's cast to the declared type.  SM_OK, SM_ERR_UNKNOWN_OPTION for a name the kind
// does not register, SM_ERR_BAD_ARGUMENT for a type other than 0 / 1; `f` is unchanged on an error.
int filter_set_param(FilterParams& f, const char* name, int type, const char* text);
bool filter_configs_valid(const FilterParams& f);                   // ConfigsValid of the kind
// constants the reference derives per Filter call, in its mix of float and double
struct RangeImageConsts { float hres, vres; double btm; };         // filter_range_image.cc:89-93, :112
struct Gr2Consts { float two_pi, delta_alpha, delta_bin; int search_steps; };   // filter_ground_removal2.cc:144-146, :340-341
RangeImageConsts range_image_consts(const FilterParams& f);
Gr2Consts gr2_consts(const FilterParams& f);
struct Gr2Line { float d0, z0, d1, z1; };                           // GroundRemoval2::Line: start (d, z), end (d, z)
// host builds of the per-point functions of filters.cu (test hook sm_debug_filter_host)
bool filter_debug_keep_host(const FilterParams& f, const float* rec, uint32_t index, uint32_t seed);
bool filter_debug_pixel_host(const FilterParams& f, const float* rec, int* row, int* col);
void filter_debug_cell_host(const FilterParams& f, const float* rec, float* range, int* s, int* b);
void filter_debug_fit_host(const float* d, const float* z, int n, float* m, float* b);
float filter_debug_distance_host(const Gr2Line* lines, int n_lines, float d, float z, int* bad);
// raw words 0 .. count - 1 of std::mt19937(seed), by the recurrence mt19937_sampler_kernel runs (test hook)
void mt19937_debug_words_host(uint32_t seed, int64_t count, uint32_t* out);
// A RandomSampler in SM_FILTER_SAMPLER_MT19937 mode over n points: flag[j] = 1 iff draw j of std::mt19937(sampler_seed)
// through uniform_real_distribution<double>(0, 1) is <= sampling_rate, every flag 1 without a draw at a rate
// > 0.999; the tile counts (compact_count_bytes(n)) are left for filter_compact_records.
int mt19937_sampler_flags(const FilterParams& f, int n, uint8_t* flag, uint32_t* tile_cnt, cudaStream_t s);
// the RangeImage stage's pixel of every point (0xffffffff: outlier) and the first point per pixel (0xffffffff: empty)
int range_image_owner(const FilterParams& f, const char* pts, int n, int64_t stride, uint32_t* pixel, uint32_t* owner,
                      cudaStream_t s);
struct FilterChain;
const FilterChain* filter_chain_of(const ::sm_filter_chain* c);   // the chain behind the C handle, null for null
// The end of every filter stage: after a flag kernel has stored its tile counts (compact.cuh), copies the flagged
// records of `pts` (5 floats each) to out in input order with their scan indices (index_in, null = identity) and
// leaves their number in *m (device memory).  tile_cnt: compact_count_bytes(n), turned into offsets in place.
void filter_compact_records(const char* pts, int64_t stride, const uint32_t* index_in, int n, const uint8_t* flag,
                            uint32_t* tile_cnt, float* out, uint32_t* index_out, uint32_t* m, cudaStream_t s);

// ---- ground_removal.cu -------------------------------------------------------------------------
// the fate of a GroundRemoval voxel (filter_ground_removal.cc:74-108): skipped (in neither list), ground (its points
// are outliers) or kept (its records are emitted, its points are inliers)
enum GrStatus : int { kGrSkipped = 0, kGrGround = 1, kGrKept = 2 };

// (int)(coordinate / leaf_size) per axis: a float division, truncated toward zero, INT_MIN for a NaN quotient or one
// outside int's range (to_int).  GroundRemoval and PlaneDetector (plane_detector.h:80-83) key their voxels so.
__host__ __device__ __forceinline__ void gr_index(const float* p, float leaf, int* ixyz) {
  ixyz[0] = to_int(p[0] / leaf);
  ixyz[1] = to_int(p[1] / leaf);
  ixyz[2] = to_int(p[2] / leaf);
}

// one step of the reference's z loop (.cc:81-89, plane_detector.h:109-118): a NaN z updates neither
__host__ __device__ __forceinline__ void gr_z_update(float z_max, float z_min, float* max_z, float* min_z) {
  if (z_max > *max_z) *max_z = z_max;
  if (z_min < *min_z) *min_z = z_min;
}

// the voxel's fate (.cc:77-107); max_z / min_z are read only when the size test passes and iz <= 0
__host__ __device__ __forceinline__ int gr_voxel_status(int32_t count, int iz, float max_z, float min_z,
                                                        int32_t min_points, float height_threshold) {
  if (count < min_points) return kGrSkipped;
  if (iz > 0) return kGrKept;
  const float delta = max_z - min_z;
  return (delta >= 0.f && delta <= height_threshold) ? kGrGround : kGrKept;
}

__device__ __forceinline__ const float* gr_point(const char* pts, int64_t stride, uint32_t i) {
  return reinterpret_cast<const float*>(pts + (int64_t)i * stride);
}

// The voxels of GroundRemoval and PlaneDetector (plane_sampler.cu) in the reference's std::map order, lexicographic
// on signed (ix, iy, iz).  For n >= 1 records, after the caller has zeroed meta[0..5]: meta[0..5] = the
// per-axis index bounds (voxel_span_ok reads them), the sorted 63-bit keys in rp.keys[0] with the input indices in
// rp.vals[0] (stable: a voxel keeps its points in input order), voxel_start[v] = the first sorted position of voxel
// v, voxel_start[voxels] = n, and tile_cnt[compact_tiles(n)] = the number of voxels.  rp: carved with
// voxel_sort_stride(n); tile_cnt: compact_count_bytes(n).
inline int64_t voxel_sort_stride(int64_t n) { return (n + 63) & ~(int64_t)63; }
int voxel_sort(const char* pts, int n, int64_t stride, float leaf, const RadixPairs& rp, uint32_t* meta,
               uint32_t* tile_cnt, uint32_t* voxel_start, cudaStream_t s);
// false when the indices other than INT_MIN of an axis span more than 2^21 - 1 voxels (the key cannot hold them);
// host_meta: meta[0..5] read back after voxel_sort
bool voxel_span_ok(const uint32_t* host_meta);
// list = the i < n with flag[i] == want, ascending, and *m their number (device memory); tile_cnt:
// compact_count_bytes(n)
void flag_list(const uint8_t* flag, int n, int want, uint32_t* tile_cnt, int32_t* list, uint32_t* m, cudaStream_t s);
// host builds of the per-point voxel index and of the per-voxel decision over the voxel's z in input order (test hooks
// sm_debug_ground_removal_index_host / _voxel_host); max_min: the z loop's max_z, min_z
void gr_debug_index_host(const float* p, float leaf, int* ixyz);
int gr_debug_voxel_host(const float* z, int64_t count, int iz, int32_t min_points, float height_threshold,
                        float* max_min);
// The device buffers and parameters of one GroundRemoval, shared by sm_ground_removal_* and the chain's stage.
// reserve() sizes the buffers for n records; they only grow.  run(): n >= 1 records of `stride` bytes in device memory
// (index_in: their scan indices, null = identity) -> out (capacity n records) and out_index (capacity n) in the map's
// order, each index the scan index of the record's input point, *m; returns after the stream has finished.  With
// `lists`, the run's inlier and outlier lists (input indices, ascending) are written into the *_next buffers and
// swapped in when it succeeds, so that inliers / outliers always hold the last successful run's.
// SM_ERR_BAD_ARGUMENT: an axis whose indices other than INT_MIN span more than 2^21 - 1 voxels (the 63-bit key cannot
// hold them); out and out_index have been written then.
struct GroundRemoval {
  FilterParams params = filter_defaults(kFilterGroundRemoval);
  DevBuf sort, tile_cnt, voxel_start, emit, status, sorted, meta, inliers, outliers, inliers_next, outliers_next;
  int64_t n_inliers = 0, n_outliers = 0;
  int reserve(int64_t n);
  int run(const char* pts, int64_t n, int64_t stride, const uint32_t* index_in, float* out, uint32_t* out_index,
          int64_t* m, cudaStream_t s, bool lists);
};

// ---- statistic_removal.cu ----------------------------------------------------------------------
// The device buffers and parameters of one StatisticRemoval, shared by sm_statistic_removal_* and the chain's stage.
// reserve() sizes them for n records; they only grow.  run(): n >= 1 records of `stride` bytes in device memory
// (index_in: their scan indices, null = identity) -> the kept records in input order in out (capacity n records),
// their scan indices in out_index (capacity n), *m; returns after the stream has finished.  The caller checks k_ok()
// first.  SM_ERR_CHECK_FAILED: 1..K finite points; SM_ERR_BAD_ARGUMENT: more finite points than a 24-level tree holds;
// out and out_index are untouched then.
struct StatisticRemoval {
  FilterParams params = filter_defaults(kFilterStatisticRemoval);
  DevBuf flag, tile_cnt, coord, index, dist, bins, stats, count, kdws;
  KdCompactTree tree;
  int64_t last_n = 0;                                  // points of the last run (its distances are in dist)
  double host_stats[4] = {NAN, NAN, NAN, 0.0};
  bool k_ok() const;                                   // point_num_meank in 1..63: K + 1 neighbours within 64
  int reserve(int64_t n);
  int run(const char* pts, int64_t n, int64_t stride, const uint32_t* index_in, float* out, uint32_t* out_index,
          int64_t* m, cudaStream_t s);
};

// ---- voxel_filter.cu ---------------------------------------------------------------------------
// The device buffers of one VoxelGrid::Filter (filter_voxel_grid.cc:37-78), shared by sm_voxel_grid_filter and the
// chain's stage.  reserve() sizes them for n records; they only grow.  run(): n >= 1 records of `stride` (>= 16)
// bytes in device memory, x, y, z, intensity first -> one record per voxel in out (capacity n records), in the
// sm_voxel_order `order` (the caller checks it), the voxel's mean with factor 0, *m; returns after the stream has
// finished.  out_index (optional, capacity n): the scan index (index_in, null = identity) of each voxel's first member
// in input order.  Points with a NaN / inf quotient are dropped.  voxel > 1e-6 (the caller checks).
// SM_ERR_BAD_ARGUMENT: the finite points span 2^21 voxels or more along an axis; out and out_index may have been
// written then.
// SM_VOXEL_ORDER_UNORDERED_MAP keeps, per voxel in insertion rank t (the order of first members): its hash, its
// ascending index, its first member and its list position; epoch_trace (test hook), when set, receives the positions
// of the voxels present after every rehash epoch.
struct VoxelGrid {
  DevBuf sort, tile_cnt, voxel_start, sorted, meta;
  DevBuf mark, rank_cnt, by_rank, table, staged;   // SM_VOXEL_ORDER_UNORDERED_MAP only
  std::vector<std::vector<uint32_t>>* epoch_trace = nullptr;
  int reserve(int64_t n);
  int run(const char* pts, int64_t n, int64_t stride, float voxel, int32_t order, const uint32_t* index_in,
          float* out, uint32_t* out_index, int64_t* m, cudaStream_t s);
  int64_t rank_stride = 0;                         // by_rank holds five arrays of this many entries
  uint64_t* hash() const { return (uint64_t*)by_rank.p; }
  uint32_t* asc() const { return (uint32_t*)(hash() + rank_stride); }
  uint32_t* first() const { return asc() + rank_stride; }
  uint32_t* pos() const { return asc() + 2 * rank_stride; }
  uint32_t* bucket() const { return asc() + 3 * rank_stride; }

 private:
  int unordered_emit(const char* pts, int n, int64_t stride, float voxel, const uint32_t* index_in, float* out,
                     uint32_t* out_index, int64_t* m, cudaStream_t s);
};
// std::unordered_map's rehash epochs for m distinct inserts, from the libstdc++ this library is built with: pairs
// (c_e, B_e), the insert of key c_e rehashes to B_e buckets; the first pair is (0, B_0).  Cached up to the largest m.
std::vector<std::pair<int64_t, uint64_t>> unordered_map_epochs(int64_t m);
// common/eigen_hash.h:31-43 on an int key (test hook sm_debug_voxel_hash_host)
uint64_t vf_debug_hash_host(const int32_t* k3);

// ---- plane_sampler.cu --------------------------------------------------------------------------
// what Detect did with a voxel (plane_detector.h:103-152): skipped (fewer than min points), the z-range rule (iz <= 0)
// with or without plane points, skipped before RANSAC (iz > 0, fewer than 2 min points), RANSAC with or without
enum PsStatus : int32_t {
  kPsSkipped = 0, kPsGroundPlane = 1, kPsGroundNot = 2, kPsSkippedRansac = 3, kPsRansacPlane = 4, kPsRansacNot = 5
};
// one voxel of the last run, in map order (test hook sm_debug_plane_sampler_voxels): its status; for a RANSAC voxel
// the loop's iterations, the best count (-INT_MAX when no sample was found), the refined coefficients (the best
// model's when there were 3 inliers or fewer); the plane points it gave
struct PsTrace {
  int32_t status, iterations, best, final_count;
  float coef[4];
};
// host builds (test hooks sm_debug_plane_sampler_piece_host / _keep_host)
int ps_debug_piece_host(int op, const float* in, float* out);
void ps_debug_keep_host(float rate, int64_t k0, int64_t k1, uint8_t* out);
// The device buffers and parameters of one RandomSamplerWithPlaneDetect; the buffers only grow.  run(): n in
// 1..2^24 records of `stride` bytes in device memory -> out (capacity n records) and out_index (capacity n), the
// kept records in input order, *m; returns after the stream has finished.  SM_ERR_BAD_ARGUMENT: a voxel span past
// voxel_sort's key.  The lists (inliers, outliers, plane indices) of a run are written into lists_next and swapped in
// when it succeeds.
struct PlaneSampler {
  float rate = 1.f, leaf_size = 0.8f;
  uint64_t min_points = 10;
  bool trace_on = false;                 // sm_debug_plane_sampler_trace: keep the per-voxel trace of every run
  DevBuf sort, tile_cnt, voxel_start, scratch, cta_list, plane, keep, meta, rnd, trace, lists[3], lists_next[3];
  int64_t n_lists[3] = {0, 0, 0};
  int64_t n_voxels = 0;                  // traced voxels of the last run
  int reserve(int64_t n);
  int run(const char* pts, int64_t n, int64_t stride, float* out, uint32_t* out_index, int64_t* m, cudaStream_t s);
};
PlaneSampler* plane_sampler_of(::sm_plane_sampler* h);   // the state behind the C handle, null for null

// ---- depth_cluster.cu --------------------------------------------------------------------------
// sinf / cosf of RangeImage::LabelOneComponent's horizontal and vertical resolution (filter_range_image.cc:255-259)
struct DepthConsts { float sin_h, cos_h, sin_v, cos_v; };
bool depth_cluster_grid_ok(const FilterParams& f);   // a RangeImage grid DepthCluster can run (filters.cu)
DepthConsts depth_consts(const FilterParams& f);
// the edge predicate compiled for the host (test hook sm_debug_depth_edge_host): step k of the neighbour list
bool depth_debug_edge_host(const DepthConsts& c, float a, float b, int k, float* beta);
// RangeImage::DepthCluster (filter_range_image.cc:143-173) over n records in device memory, for a RangeImage `f`
// with vertical_line_num >= 1, horizontal_line_num >= 2 and at most 2^24 pixels.  Writes the clustered points
// (capacity: the occupied pixels, at most n) and, if point_label is not null, the label of every input point that
// owns its pixel (0 elsewhere); returns after the stream has finished, with the count in *m.  The per-pixel arrays
// stay valid until the next run (test hook sm_debug_depth_cluster).
struct DepthCluster {
  DevBuf pixel, owner, image, mask, parent, label, size, kept, kept_off, claim, level, seq, order, roots, block_cnt,
      count;
  int components = 0;                // of the last run, dropped ones included
  int reserve(int64_t n, int64_t pixels);
  int run(const FilterParams& f, const char* pts, int n, int64_t stride, float* out_xyz, uint32_t* out_label,
          int32_t* out_index, uint32_t* point_label, int64_t* m, cudaStream_t s);
};

// The device buffers and the stages of one filter chain.  reserve() sizes the buffers for n records and the chain's
// RangeImage / GroundRemoval2 grids; they only grow, and so do those of the GroundRemoval, StatisticRemoval and
// VoxelGrid stages.  run() applies the filters in order to n records of `stride` bytes in device memory and leaves
// the records of the last stage, packed, in `out` (capacity n records) with their indices in the input scan in
// `out_index` (optional), in emission order; it returns after the stream has finished, with the count in *m.  On
// SM_ERR_BAD_ARGUMENT / SM_ERR_CHECK_FAILED, `fault` says why.
struct FilterChain {
  std::vector<FilterParams> filters;
  uint32_t sample_seed = 1;
  uint32_t all_filters = 0;          // chain option: sm_filter_chain_add accepts the three kinds above
  const char* fault = "";
  DevBuf rec[2], idx[2], flag, block_cnt, count, pixel, owner, sort, cell_of, pt, member, cells, occ, work, lines;
  GroundRemoval ground;
  StatisticRemoval statistic;
  VoxelGrid voxel;
  // the intermediates of the last GroundRemoval2 stage (test hook sm_debug_filter_ground_removal2)
  struct Gr2View {
    const uint32_t* cell_of; const uint8_t* member; const uint32_t* cell_cnt; const float2* cell_min;
    const Gr2Line* lines; const int* n_lines; const uint8_t* keep; int max_lines; int status;
  } gr2 = {};
  int reserve(int64_t n);
  int run(const char* in, int64_t n, int64_t stride, float* out, int32_t* out_index, int64_t* m, cudaStream_t stream);

 private:
  // each stage reads n records (index_in: their scan indices, null = identity) and compacts the inliers
  int predicate_stage(int first, int count, const char* in, const uint32_t* index_in, int n, int64_t stride,
                      float* out, uint32_t* index_out, cudaStream_t s);
  int mt19937_sampler_stage(const FilterParams& f, const char* in, const uint32_t* index_in, int n, int64_t stride,
                            float* out, uint32_t* index_out, cudaStream_t s);
  int range_image_stage(const FilterParams& f, const char* in, const uint32_t* index_in, int n, int64_t stride,
                        float* out, uint32_t* index_out, cudaStream_t s);
  int ground_removal2_stage(const FilterParams& f, const char* in, const uint32_t* index_in, int n, int64_t stride,
                            float* out, uint32_t* index_out, cudaStream_t s);
  // GroundRemoval, StatisticRemoval and VoxelGrid; *m = the stage's count
  int record_stage(const FilterParams& f, const char* in, const uint32_t* index_in, int n, int64_t stride, float* out,
                   uint32_t* index_out, int64_t* m, cudaStream_t s);
  int stage_end(int first) const;   // one past the last filter of the stage that starts at `first`
  int bad_grid() { fault = "a RangeImage or GroundRemoval2 grid size the chain cannot run"; return SM_ERR_BAD_ARGUMENT; }
  int check_failed() {
    fault = "Check failed: an inverted BoundingBoxRemoval box or line.start[0] < line.end[0]";
    return SM_ERR_CHECK_FAILED;
  }
};

}  // namespace smb

#endif  // SM_B200_KERNELS_H_
