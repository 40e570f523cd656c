/* sm_b200.h — C ABI of libsm_b200.so, the H100-native scan-matching engine that stands in
 * for StaticMapping's registrators/ hot path.
 *
 * Drop-in boundary: the reference has no FFI of its own (it is one C++ process); the
 * interface a maintainer binds is registrator::Interface
 * (registrators/interface.h:67-119 of the reference).  Each entry point below names the
 * reference member it replaces.  INTEGRATION.md shows the C++ adapter
 * (adapter/registrators_b200.h) that maps these 1:1 onto that class.
 *
 * Conventions
 *   - plain pointers and sizes only; no C++/torch types; never throws across the ABI;
 *   - 4x4 transforms are 16 doubles, COLUMN-major (Eigen::Matrix4d storage);
 *   - clouds are 3xN column-major doubles (x0,y0,z0,x1,...) == Eigen::MatrixXd of
 *     data::EigenPointCloud::points / ::normals (builder/data/cloud_types.h:143-146);
 *   - return value: >= 0 success, < 0 error (sm_last_error gives the text).  Where the
 *     reference would glog-CHECK-abort the C++ adapter turns the negative code into the
 *     same CHECK failure (SURVEY.md section 5 "failure detection");
 *   - one handle is used by one thread at a time; different handles may run concurrently
 *     from different threads (map_builder.cc:655,706-708; loop_detector.cc:224-228).  Each
 *     handle owns its CUDA stream and workspace.
 */
#ifndef SM_B200_H_
#define SM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sm_handle sm_handle;

/* registrator::Type (interface.h:41-50); values match the XML `type="N"` attribute. */
enum sm_matcher_type {
  SM_TYPE_ICP_PM = 1,
  SM_TYPE_NDT_WITH_GICP = 3,
  SM_TYPE_NDT = 5,
  SM_TYPE_FAST_ICP = 6
};

enum sm_error {
  SM_OK = 0,
  SM_ERR_BAD_ARGUMENT = -1,
  SM_ERR_NO_FINITE_MATCH = -2,   /* CHECK(!values.empty())            icp_fast.cc:81  */
  SM_ERR_NOTHING_TO_MINIMIZE = -3, /* CHECK_GT(points_count, 0)        icp_fast.cc:114 */
  SM_ERR_MISSING_INPUT = -4,     /* CHECK(cloud) / missing normals    icp_fast.cc:422-430 */
  SM_ERR_CHECK_FAILED = -5,      /* a CHECK of the filter chain: bounding_box.cc:114, filter_ground_removal2.cc:403 */
  SM_ERR_UNKNOWN_OPTION = -10,   /* "Init an unknown option"          interface.cc:66-67 */
  SM_ERR_UNSUPPORTED_TYPE = -11, /* CreateMatcher default branch      interface.cc:158-160 */
  SM_ERR_NO_DEVICE = -20,        /* no CUDA device: the engine has no CPU fallback */
  SM_ERR_CUDA = -100
};

/* CreateMatcher(options) (interface.cc:139-173) + the concrete constructors
 * (IcpFast::IcpFast icp_fast.cc:407-419).  `device` is the CUDA ordinal. */
int sm_create(int type, int device, sm_handle** out);
int sm_destroy(sm_handle* h);

/* Interface::InitWithXml (interface.cc:62-90): one <param name=...>text</param> entry.
 * `text` is parsed like pugixml's as_int / as_float / as_bool for the registered type.
 * Registered names, IcpFast (icp_fast.cc:411-418): knn_normal_estimate (int, unused),
 * max_iteration (int, 100), dist_outlier_ratio (float, 0.7).  Added by this engine:
 * knn_epsilon (float, 3.16 = icp_fast.cc:174), knn_queries_per_cta (int, 0 = one query per
 * thread; 1024 suits many alignments in flight), disable_convergence_check (bool, false;
 * fixed-iteration throughput runs), profile_kernels (bool, false; CUDA events around
 * every phase kernel, reported by sm_get_align_info), use_graphs (bool, true; replay the
 * launch sequence of an Align as CUDA graphs).  Unknown name -> SM_ERR_UNKNOWN_OPTION.
 * registrator::Ndt registers NO option (ndt.cc:28-34) — the reference-facing mirrors reject
 * every <param> for type 5; the engine itself accepts the pclomp setters hard-coded by the
 * reference: resolution (1.0), step_size (0.1), outlier_ratio (0.55),
 * transformation_epsilon (0.1), max_iterations (35).
 * SM_TYPE_ICP_PM is NOT a bit-level parity implementation of registrator::IcpUsingPointMatcher: libpointmatcher
 * 1.3.1 is an external float library whose RandomSampling filter draws from the process-global std::rand stream
 * (two Align calls on the same clouds give poses ~0.5 mm apart: the reference's result is not a function of its
 * inputs) and whose surface-normal filter uses eigenvector normals.  Type 1 is a deterministic matcher with the
 * same module chain (DESIGN.md section 4e): bit-checked against a composition of this repository's oracle
 * pieces, and shown to lie within the literal chain's own call-to-call variation by a restatement of
 * libpointmatcher's filters (tests/pyref.py icp_pm_literal, tests/test_oracle_vs_python_restatement.py).
 * sm_set_pm_surface_normals switches its reference filter to libpointmatcher's own eigenvector normals, and
 * sm_set_pm_reading_sampler its reading filter to glibc's rand() stream at a given seed and stream position.
 * SM_TYPE_ICP_PM (stand-in for IcpUsingPointMatcher's default libpointmatcher chain,
 * icp_pointmatcher.cc:166-247; float clouds through the _f32 setters) registers no option in the
 * reference either; the engine accepts the IcpFast names (max_iteration defaults to 150, :214)
 * plus reading_sample_prob (0.9, :173), accept_min_score (0.6, :145) and sample_seed (1). */
int sm_set_option(sm_handle* h, const char* name, const char* text);
/* Interface::PrintOptions (interface.cc:115-137): writes one "name -> value\n" line per option
 * sm_set_option accepts for the handle's type. */
int sm_print_options(sm_handle* h, char* buf, int64_t buf_len);
/* Interface::EnableInnerCompensation / DisableInnerCompensation (interface.h:89-91, interface.cc:34-36):
 * enable != 0 switches IcpFast::Align to its in-loop motion compensation from the next Align on (sm_align,
 * sm_align_async, sm_align_batch and sm_align_pairs alike).  Every handle type accepts it; only SM_TYPE_FAST_ICP
 * reads it, as in the reference.  In every iteration source point i (f_i = i / N, its column in
 * sm_set_input_source) is moved by InterpolateTransform(Identity, T_iter, f_i) (icp_fast.cc:487-488) instead of
 * T_iter, and its match's Jacobian column is scaled by f_i (:284-289).  Deviation: the reference's
 * EigenPointCloud::ApplyMotionCompensation (cloud_types.cc:306-318) declares a local `transform` that shadows the
 * parameter and interpolates towards that uninitialised local (undefined behaviour); the engine interpolates
 * towards T_iter, which is what the code evidently intends.  Not an XML option: sm_print_options does not list
 * it. */
int sm_set_inner_compensation(sm_handle* h, int32_t enable);
/* pclomp::NormalDistributionsTransform::setNeighborhoodSearchMethod (registrators/pclomp/ndt_omp.h:184), the
 * neighbour search of the per-point derivative evaluation (switch at ndt_omp_impl.hpp:233-246).  Values are
 * pclomp's NeighborSearchMethod (ndt_omp.h:52-57).  The reference's Ndt sets KDTREE (ndt.cc:33), the default here;
 * pclomp's own default is DIRECT7 (ndt_omp_impl.hpp:74).
 *   KDTREE    radius search over the voxel centroids (radius = resolution), sorted by distance; a voxel whose
 *             covariance failed the eigenvalue test stays searchable with a zero inverse covariance.
 *   DIRECT26 / DIRECT7 / DIRECT1  VoxelGridCovariance::getNeighborhoodAtPoint / 7 / 1
 *             (voxel_grid_covariance_omp_impl.hpp:373-441): the query cell is int(floor(x / resolution)) per axis, a
 *             float division (the grid itself is built with a multiplication by 1 / resolution), and the voxels at
 *             fixed offsets from it are taken in list order, without a distance test or a sort, when they lie in the
 *             target's voxel box and hold >= 6 points with a valid covariance.  DIRECT1: the query cell;
 *             DIRECT7: it and its 6 face neighbours; DIRECT26: the 26 surrounding cells WITHOUT the query cell
 *             (pcl::getAllNeighborCellIndices of stock PCL, restated from upstream PCL).  A point whose
 *             floor(x / resolution) is not finite or lies more than one cell outside the box on some axis has no
 *             neighbour (the reference's int conversion is undefined there).
 * Applies from the next Align on (sm_align and sm_align_batch alike).  SM_TYPE_NDT only: every other type returns
 * SM_ERR_UNSUPPORTED_TYPE (the NDT stage of NdtWithGicp is stock pcl::NormalDistributionsTransform, which has no
 * such setter); a method outside 0..3 returns SM_ERR_BAD_ARGUMENT and leaves the setting unchanged.  Not an XML
 * option (the reference's Ndt registers none): sm_print_options does not list it. */
enum sm_ndt_search_method {
  SM_NDT_KDTREE = 0,
  SM_NDT_DIRECT26 = 1,
  SM_NDT_DIRECT7 = 2,
  SM_NDT_DIRECT1 = 3
};
int sm_set_ndt_search_method(sm_handle* h, int32_t method);
/* The error minimizer of the ICP iteration.  POINT_TO_PLANE (the default) is what IcpFast::Align calls
 * (registrators/icp_fast.cc:506-510).  POINT_TO_POINT is the reference's ComputePointToPoint (:326-375), a copy of
 * libpointmatcher's PointToPointErrorMinimizer: over the matches the trim keeps, p the step cloud's point and q its
 * matched target point (target-mean frame), M = sum (q - qbar)(p - pbar)^T = U S V^T, R = U V^T with the last row
 * of V^T negated when det R < 0, t = qbar - R pbar, T_iter <- [R t; 0 1] T_iter.  Everything else (tree, search,
 * trim, convergence test, score) is unchanged, and there is no NaN guard, as in the reference.
 *   - Normals are still required: SetInputTarget CHECKs them whatever the minimizer (:430); they are not read.
 *   - With inner compensation the step cloud is de-skewed as before (:487-491); the minimizer has no factor term,
 *     so f_i is not used.
 *   - Degenerate M: the 3x3 SVD is written out (csrc/linalg_dev.cuh kabsch_rotation, one-sided Jacobi).  One kept
 *     match gives M = 0 and R = I.  Where R is not unique (rank-1 M, e.g. collinear matches) the result is the
 *     rotation that completes U to a right-handed basis as documented there; it attains the optimal objective.
 *     Every operation of the solve is rounded on its own (no FMA), so the device gives the same bits as the host
 *     build of the same code.
 *   - The sums are raw moments about the origin of the target-mean frame, centred in one sweep (DESIGN §4); the
 *     reference centres the points in a second pass.  The two differ by rounding.
 * sm_align_info.solve_path reports 3 (Kabsch) or 4 (Kabsch with the reflection fix).
 * Applies from the next Align on (sm_align, sm_align_async / wait, sm_align_batch and sm_align_pairs alike).
 * SM_TYPE_FAST_ICP sets it on the handle, SM_TYPE_ICP_PM on the IcpFast chain it composes; every other type returns
 * SM_ERR_UNSUPPORTED_TYPE.  A value outside 0..1 returns SM_ERR_BAD_ARGUMENT and leaves the setting unchanged.
 * Not an XML option: sm_print_options does not list it. */
enum sm_icp_error_minimizer {
  SM_ICP_POINT_TO_PLANE = 0,
  SM_ICP_POINT_TO_POINT = 1
};
int sm_set_icp_error_minimizer(sm_handle* h, int32_t minimizer);
/* The reference filter of SM_TYPE_ICP_PM, libpointmatcher's SamplingSurfaceNormalDataPointsFilter (knn 7,
 * samplingMethod 1, icp_pointmatcher.cc:187-192).  Both modes split the reference cloud into the same boxes of at
 * most 7 points (the median-split recursion of CalculateNormals, cloud_types.cc:105-144) and keep one point and
 * one normal per box, in ascending order of the box's smallest point index.
 *   LEAST_SQUARES (the default)  CalculateNormals' leaf (cloud_types.cc:73-103), the reference author's own port of
 *             the filter: in double, the box mean and normalize(M^-1 b), M = sum d d^T, b = sum d.
 *   EIGENVECTOR  the filter's own leaf in PointMatcher<float>: the float box mean (members summed in ascending
 *             index order, divided by float(count)), C = sum (d - mean)(d - mean)^T in float, the box dropped if
 *             rank(C) + 1 < 3 (FullPivHouseholderQR's rank with a float matrix's threshold, on C widened to
 *             double), and the eigenvector of the smallest eigenvalue of C (symmetric Jacobi in double, normalised,
 *             rounded to float) with its component of largest magnitude positive.  The kept point is the float mean.
 *             The point-to-plane terms do not depend on the normal's sign; the sign only makes the output
 *             deterministic.  libpointmatcher's own eigensolver is not reproduced (DESIGN.md section 4e).
 * Applies from the next Align on (sm_align and sm_align_batch alike); a change of mode filters the reference cloud
 * anew, setting the mode it already has does not.  SM_TYPE_ICP_PM only: every other type returns
 * SM_ERR_UNSUPPORTED_TYPE and is left unchanged.  A mode outside 0..1 returns SM_ERR_BAD_ARGUMENT and leaves the
 * setting unchanged.  Not an XML option: sm_print_options does not list it. */
enum sm_pm_surface_normals {
  SM_PM_NORMALS_LEAST_SQUARES = 0,
  SM_PM_NORMALS_EIGENVECTOR = 1
};
int sm_set_pm_surface_normals(sm_handle* h, int32_t mode);
/* The reading filter of SM_TYPE_ICP_PM, libpointmatcher 1.3.1's RandomSamplingDataPointsFilter (prob =
 * reading_sample_prob, icp_pointmatcher.cc:173), which keeps column i iff (float)rand() / (float)RAND_MAX < prob,
 * drawing once per column on every ICP::compute.
 *   HASH (the default)  a counter hash instead of rand(): point i is kept iff murmur3_fmix32(i * 0x9E3779B9 +
 *             sample_seed) < prob * 2^32.  The filtered reading cloud is kept across Aligns until the source cloud,
 *             reading_sample_prob or sample_seed changes.
 *   GLIBC_RAND  glibc's rand() itself: the TYPE_3 additive-feedback generator after srand((unsigned)sample_seed)
 *             (the default sample_seed 1 is glibc's default seed), read from the handle's stream position (below).
 *             Every Align filters the reading cloud anew: point i takes draw position + i, non-finite points
 *             included, and the position then advances by the number of reading points.  Draw p is reached in
 *             O(log p) (DESIGN.md section 4e), and the keep test is exact: the draw rounded to float and divided by
 *             2^31, as x86 evaluates it.  With the eigenvector reference filter (sm_set_pm_surface_normals) type 1
 *             then runs libpointmatcher's default chain's data filters themselves, given the seed and the position.
 * Applies from the next Align on (sm_align and sm_align_batch alike).  SM_TYPE_ICP_PM only: every other type returns
 * SM_ERR_UNSUPPORTED_TYPE and is left unchanged.  A mode outside 0..1 returns SM_ERR_BAD_ARGUMENT and leaves the
 * setting unchanged.  Not an XML option: sm_print_options does not list it. */
enum sm_pm_reading_sampler {
  SM_PM_SAMPLING_HASH = 0,
  SM_PM_SAMPLING_GLIBC_RAND = 1
};
int sm_set_pm_reading_sampler(sm_handle* h, int32_t mode);
/* The GLIBC_RAND sampler's stream position: the number of rand() draws taken since srand(sample_seed).  It starts at
 * 0, setting sample_seed resets it to 0 (as srand does), and every type-1 Align in GLIBC_RAND mode advances it by
 * the number of reading points once the filter has run; HASH mode leaves it alone.  A negative position returns
 * SM_ERR_BAD_ARGUMENT; an Align that would advance it past 2^63 - 1 returns SM_ERR_BAD_ARGUMENT before any work.
 * A process running the reference draws every Align's points from ONE global stream, in the order its Aligns run.
 * To reproduce that, give each handle the position the reference process had reached when that Align started: the
 * previous Align's position plus its reading size, across handles.  sm_align_batch runs type-1 handles on worker
 * threads, each from its own position, so set every handle's position before the batch.  SM_TYPE_ICP_PM only:
 * every other type returns SM_ERR_UNSUPPORTED_TYPE and is left unchanged. */
int sm_get_pm_rand_position(sm_handle* h, int64_t* position);
int sm_set_pm_rand_position(sm_handle* h, int64_t position);
/* Interface::GetType (interface.h:106). */
int sm_get_type(const sm_handle* h);

/* IcpFast::SetInputSource / SetInputTarget (icp_fast.cc:421-431): deep copy into the
 * engine (host pointers are not retained).  The target must carry unit normals
 * (CHECK(HasNormals()), icp_fast.cc:430) — the caller computed them with
 * EigenPointCloud::CalculateNormals (map_builder.cc:286,389) or sm_calculate_normals.
 * SM_TYPE_FAST_ICP only: every other type returns SM_ERR_UNSUPPORTED_TYPE and keeps its clouds. */
int sm_set_input_source(sm_handle* h, const double* points_3xn, int64_t n);
int sm_set_input_target(sm_handle* h, const double* points_3xn, const double* normals_3xn,
                        int64_t n);
/* Ndt / NdtWithGicp keep the caller's float cloud (Interface::SetInputSource/Target,
 * interface.cc:38-60, converted by ToPclPointCloud at Align, ndt.cc:48-51).  `xyz` points at
 * the first x; consecutive points are `stride_bytes` apart (sizeof(InnerPointType) == 20 for
 * the reference's std::vector<InnerPointType>, 12 for packed xyz).  Ndt, NdtWithGicp and SM_TYPE_ICP_PM only: an
 * IcpFast handle returns SM_ERR_UNSUPPORTED_TYPE and keeps its clouds. */
int sm_set_input_source_f32(sm_handle* h, const float* xyz, int64_t n, int64_t stride_bytes);
int sm_set_input_target_f32(sm_handle* h, const float* xyz, int64_t n, int64_t stride_bytes);
int sm_set_input_source_f32_device(sm_handle* h, const float* dev_xyz, int64_t n, int64_t stride_bytes);
int sm_set_input_target_f32_device(sm_handle* h, const float* dev_xyz, int64_t n, int64_t stride_bytes);

/* Same, for clouds already resident in this device's memory (same layout); SM_TYPE_FAST_ICP only, like the host
 * variants. */
int sm_set_input_source_device(sm_handle* h, const double* dev_points_3xn, int64_t n);
int sm_set_input_target_device(sm_handle* h, const double* dev_points_3xn,
                               const double* dev_normals_3xn, int64_t n);

/* Interface::Align(const Matrix4d& guess, Matrix4d& result) (interface.h:103-104;
 * IcpFast::Align icp_fast.cc:455-529).  Returns 1 (true) / 0 (false) like the
 * reference's bool, or a negative sm_error. */
int sm_align(sm_handle* h, const double* guess_4x4, double* result_4x4);
/* The same Align in two halves, so ONE host thread can keep several matcher instances in
 * flight (the reference gets its concurrency from a thread pool / TBB tasks calling Align on
 * distinct instances: map_builder.cc:655,706-708; loop_detector.cc:224-228):
 * sm_align_async enqueues everything and returns; sm_align_wait blocks for the result (and,
 * with the convergence test enabled, keeps enqueuing 8-iteration chunks until it fires).
 * IcpFast only: on any other type both return SM_ERR_UNSUPPORTED_TYPE.  sm_align == async + wait. */
int sm_align_async(sm_handle* h, const double* guess_4x4);
int sm_align_wait(sm_handle* h, double* result_4x4);
/* Batched Align.  The reference fans independent Align calls out to a thread pool / TBB tasks
 * (back_end/loop_detector.cc:216-228 one task per loop-closure candidate; builder/map_builder.cc:
 * 655,706-708 submap pairs); here ONE host thread keeps many alignments in flight on the GPU.
 *
 * sm_align_batch: `n` matcher instances whose SetInputSource / SetInputTarget have been called.
 * IcpFast instances are all enqueued before the first result is awaited; the other matcher types
 * (host-driven Newton / BFGS loops) run on up to 16 internal worker threads.  guesses / results:
 * n x 16 doubles; rc_n[i] = what sm_align would have returned for instance i.  Returns SM_OK or the
 * most negative rc.
 *
 * sm_align_pairs: `n_pairs` independent IcpFast alignments pipelined over `n_handles` instances
 * (pair k runs on instance k % n_handles; an instance's previous result is collected right before
 * it is given its next pair).  Host clouds are uploaded asynchronously on the instance's stream —
 * unlike sm_set_input_*, the arrays of a pair must stay valid until sm_align_pairs returns (pinned
 * host memory makes the copies overlap the other pipelines' kernels).  scores_n (optional) receives
 * GetFitnessScore per pair.  rc_n[k] = what sm_set_input_target, sm_set_input_source and sm_align
 * would have returned for pair k; returns SM_OK or the most negative rc.
 * A failed pair (rc_n[k] < 0) gets scores_n[k] = 0.0 wherever it failed, and its results_16n slot
 * is left as the caller passed it.  Nothing of a pair outlives the call: a pair the counts, pointers
 * or the instance's options refuse is refused before any of it is enqueued, and when a pair fails
 * after its uploads were enqueued, its instance's stream is synchronized before the next pair. */
typedef struct sm_pair {
  const double* source_3xn;          /* SetInputSource */
  int64_t n_source;
  const double* target_3xn;          /* SetInputTarget (points + unit normals) */
  const double* target_normals_3xn;
  int64_t n_target;
  const double* guess_4x4;           /* NULL = identity */
  int32_t on_device;                 /* 1: the three cloud pointers are device pointers */
  int32_t reserved;
} sm_pair;
int sm_align_batch(sm_handle* const* handles, int32_t n, const double* guesses_16n, double* results_16n,
                   int32_t* rc_n);
int sm_align_pairs(sm_handle* const* handles, int32_t n_handles, const sm_pair* pairs, int32_t n_pairs,
                   double* results_16n, double* scores_n, int32_t* rc_n);
/* Interface::GetFitnessScore (interface.h:100). */
double sm_get_fitness_score(const sm_handle* h);

typedef struct sm_align_info {
  int32_t iterations;      /* ICP iterations executed */
  int32_t status;          /* 0 or sm_error */
  int32_t solve_path;      /* last 6x6 solve: 0 Cholesky, 1 rank-reduced, 2 SVD; point-to-point: 3 Kabsch,
                              4 Kabsch with the reflection fix */
  int32_t reserved;
  int64_t kept;            /* matches kept by the 70 % trim in the last iteration */
  double limit;            /* its squared-distance limit */
  float ms_upload;         /* device time of the last SetInput* copies */
  float ms_prologue;       /* centre + tree build + G0 (icp_fast.cc:456-480) */
  float ms_iterations;     /* all ICP iterations */
  int32_t kernel_launches; /* kernels launched by the last sm_align */
  /* filled only when option profile_kernels=1: summed device time of each phase kernel */
  float ms_knn;            /* transform + k-NN + histogram        (icp_fast.cc:486-493) */
  float ms_accum;          /* quantile bin + normal equations      (icp_fast.cc:496-503) */
  float ms_finish;         /* exact limit, solve, pose update      (icp_fast.cc:506-523) */
  int32_t profiled_iterations;
  /* NDT only */
  int32_t evaluations;        /* computeDerivatives calls (ndt_omp_impl.hpp:180) */
  double trans_probability;   /* score / N_source (ndt_omp_impl.hpp:170) */
  double mean_neighbors;      /* mean number of neighbour voxels per source point */
  /* IcpUsingPointMatcher stand-in (type 1): [0] IcpFast's own score of the last iteration,
   * [1] matches kept by the trim in the final score pass, [2] reading / [3] reference points after
   * the data filters.
   * NdtWithGicp only: [0] NDT fitness (the <= 1.0 gate, ndt_gicp.cc:92), [1] GICP fitness,
   * [2] source points after ApproximateVoxelGrid, [3] target points after it;
   * iterations = GICP outer iterations, profiled_iterations = BFGS cost evaluations */
  double aux[4];
} sm_align_info;
int sm_get_align_info(const sm_handle* h, sm_align_info* out);

/* Run this handle's work on the caller's CUDA stream (a cudaStream_t passed as void*;
 * NULL restores the handle's own stream).  Lets a host that already owns a stream —
 * e.g. the bench's torch stream — order and time the engine's kernels with its own
 * events.  No reference counterpart (the reference is CPU-only). */
int sm_set_stream(sm_handle* h, void* cuda_stream);

const char* sm_last_error(const sm_handle* h);

/* ---- building blocks exposed for parity tests and for callers that hold clouds ------- */

/* libnabo-compatible tree build + 1-NN (NNS::create + knn, icp_fast.cc:466-467,177-178).
 * ids: original target column, -1 if none; dists2: squared distances.  bucket_size 2..8
 * (libnabo's default is 8; one padded bucket of the search layout holds 8 points). */
int sm_knn1(int device, const double* target_3xn, int64_t n_target, const double* query_3xn,
            int64_t n_query, double epsilon, int bucket_size, int32_t* ids, double* dists2);

/* libnabo's k-nearest-neighbour search: NNS::create(target, 3, KDTREE_LINEAR_HEAP, 0, {bucketSize}) +
 * knn(query, indices, dists2, k, epsilon, optionFlags, maxRadius), on the tree sm_knn1 builds.  It is what the
 * reference's k > 1 and radius searches call (libpointmatcher's SamplingSurfaceNormalDataPointsFilter knn 7,
 * KDTreeMatcher's maxDist, icp_pointmatcher.cc:178,186-189).  Rules (libnabo 1.0.7, restated in
 * oracle/knn_oracle.cc): a point enters the sorted k-list iff d2 <= max_radius^2, d2 < the k-th entry and, without
 * SM_KNN_ALLOW_SELF_MATCH, d2 > DBL_EPSILON; it goes after every entry of equal distance (the earlier-visited one
 * first).  A far side is visited iff rd <= max_radius^2 and rd * (1 + epsilon)^2 < the k-th entry.
 * ids / dists2: k x n_query column-major (libnabo's MatrixXi(k, nQ)), i.e. row i of an n_query x k row-major array
 * holds query i's neighbours, ascending.  SORT_RESULTS is accepted and changes nothing: the list is always sorted.
 * When fewer than k points qualify (k > n_target, the radius, self-match exclusion) the rest of the row is
 * -1 / +inf.  Whether libnabo itself accepts k > n_target, and how it fills such a row, is not verified here.
 * SM_ERR_BAD_ARGUMENT: k outside 1..64, epsilon < 0 or NaN, max_radius < 0 or NaN, bucket_size outside 2..8, a flag
 * bit other than the two below, n_target < 1.  The _device form takes device pointers (3xN clouds and the outputs),
 * runs on `cuda_stream` (a cudaStream_t, NULL = default stream) and returns after that stream has finished. */
#define SM_KNN_ALLOW_SELF_MATCH 1u   /* NNS::ALLOW_SELF_MATCH */
#define SM_KNN_SORT_RESULTS 2u       /* NNS::SORT_RESULTS */
int sm_knn(int device, const double* target_3xn, int64_t n_target, const double* query_3xn, int64_t n_query,
           int32_t k, double epsilon, double max_radius, uint32_t flags, int bucket_size, int32_t* ids,
           double* dists2);
int sm_knn_device(int device, const double* target_3xn, int64_t n_target, const double* query_3xn, int64_t n_query,
                  int32_t k, double epsilon, double max_radius, uint32_t flags, int bucket_size, int32_t* ids,
                  double* dists2, void* cuda_stream);

/* EigenPointCloud::CalculateNormals (builder/data/cloud_types.cc:347-368): median-split
 * the cloud into leaves of <= 7 points, fit n.p = 1 per leaf, keep one point (the leaf
 * mean) + unit normal per valid leaf, survivors in ascending order of the smallest
 * original index of their leaf.  out_points / out_normals: capacity 3*n doubles;
 * *m_out receives the number of survivors.  Called by the reference right before
 * IcpFast::SetInputTarget (map_builder.cc:286,389; submap.cc:161).
 * DEVIATION from the reference (cloud_types.cc:79-100): there a leaf is represented by
 * indices[first] and summed in the member order std::nth_element happens to leave, both of which
 * depend on the standard library's partition internals; here (SM_NORMALS_ORDER_INDEX) the split
 * breaks coordinate ties by index, the representative is the member with the smallest original
 * index and members are summed in ascending index.  With distinct coordinates the SET of leaves is
 * the reference's; with tied coordinates (float lidar clouds have many) the leaves themselves can
 * differ, and so can the column order and the last bits of a mean / normal.
 * sm_calculate_normals_ordered with SM_NORMALS_ORDER_NTH_ELEMENT gives the reference's own order. */
int sm_calculate_normals(int device, const double* points_3xn, int64_t n, double* out_points,
                         double* out_normals, int64_t* m_out);

/* The order CalculateNormals splits, sums and represents its leaves in.
 *   SM_NORMALS_ORDER_INDEX        sm_calculate_normals' order: ties broken by index, members summed
 *                                 in ascending index, representative = smallest index
 *   SM_NORMALS_ORDER_NTH_ELEMENT  the reference's: every node split by libstdc++'s std::nth_element
 *                                 with '<' on the cut-axis coordinate over the one index array the
 *                                 recursion permutes; members summed in the order it leaves,
 *                                 representative = first member; columns in ascending
 *                                 representative index.  Bit-identical to that recursion run on the
 *                                 CPU, so a build that switches to the GPU gets its own targets back.
 *                                 A non-finite coordinate is refused with SM_ERR_BAD_ARGUMENT (the
 *                                 library's unguarded scans are undefined on NaN); nothing is written. */
enum sm_normals_order {
  SM_NORMALS_ORDER_INDEX = 0,
  SM_NORMALS_ORDER_NTH_ELEMENT = 1,
};
/* sm_calculate_normals in the given order (sm_normals_order); an unknown order is SM_ERR_BAD_ARGUMENT. */
int sm_calculate_normals_ordered(int device, const double* points_3xn, int64_t n, int32_t order,
                                 double* out_points, double* out_normals, int64_t* m_out);

/* MotionCompensation (builder/map_builder.cc:232-257; called either side of Align at :320-352
 * when motion_compensation_options.enable is set): every point is moved by
 * common::InterpolateTransform(Identity, delta, point.factor) (common/math.h:198-211 — slerp of
 * the rotation, linear translation).  `points` / `out` are arrays of the reference's
 * data::InnerPointType {float x, y, z, intensity, factor} (builder/data/cloud_types.h:46-52),
 * consecutive points `stride_bytes` (>= 20) apart; intensity and factor are copied.  `delta` is
 * 16 doubles, column-major.  Returns SM_ERR_BAD_ARGUMENT where the reference CHECK-fails
 * (a factor outside [0, 1], common/math.h:201); `out` is still written in that case.
 * The _device form takes device pointers (in and out may not overlap) and runs on
 * `cuda_stream` (a cudaStream_t, NULL = default stream); it returns after the stream has
 * finished. */
int sm_motion_compensation(int device, const float* points, int64_t n, int64_t stride_bytes,
                           const double* delta_4x4, float* out);
int sm_motion_compensation_device(int device, const float* dev_points, int64_t n,
                                  int64_t stride_bytes, const double* delta_4x4, float* dev_out,
                                  void* cuda_stream);

/* pre_processers::filter::VoxelGrid::Filter (pre_processors/filter_voxel_grid.cc:37-78), the
 * down-sampling Submap::InsertFrame applies before CalculateNormals (builder/submap.cc:144-161):
 * one output point per occupied voxel, voxel index = lround(coordinate / voxel_size) per axis
 * (:47-49), x / y / z / intensity = mean of the voxel's points accumulated in double in input
 * order (:58-70), factor = 0.  `points`: data::InnerPointType records (x, y, z, intensity, ...)
 * `stride_bytes` (>= 16) apart; `out`: capacity n records of 5 packed floats; *m_out = number of
 * voxels.  Every value is bit-identical to the reference's; the ORDER of the output points is
 * ascending (ix, iy, iz), where the reference emits them in std::unordered_map iteration order
 * (sm_voxel_grid_filter_ordered with SM_VOXEL_ORDER_UNORDERED_MAP gives that order).
 * Points with a NaN / inf coordinate are dropped (std::lround of such a value is unspecified in the
 * reference; one bad lidar return must not stop the mapper).  SM_ERR_BAD_ARGUMENT: voxel_size <= 1e-6
 * (ConfigsValid, :35), or finite points that span 2^21 voxels or more along one axis (209 km at the
 * reference's 0.1 m voxels). */
int sm_voxel_grid_filter(int device, const float* points, int64_t n, int64_t stride_bytes,
                         float voxel_size, float* out, int64_t* m_out);

/* The order VoxelGrid emits its voxels in.
 *   SM_VOXEL_ORDER_ASCENDING      sm_voxel_grid_filter's: ascending (ix, iy, iz)
 *   SM_VOXEL_ORDER_UNORDERED_MAP  the reference's: the iteration order of its std::unordered_map<Eigen::Vector3i, ...>
 *                                 (hash common/eigen_hash.h:31-43, boost's hash_combine over the int keys) as the
 *                                 libstdc++ this library is built with leaves it after inserting the voxels in the
 *                                 order of their first member, its rehash schedule included.  Non-finite points are
 *                                 dropped before insertion, so the order is the container's when fed the finite
 *                                 points in input order (the reference's lround of such a point is unspecified).
 *                                 Fed to CalculateNormals in SM_NORMALS_ORDER_NTH_ELEMENT, this gives the
 *                                 reference's submap targets (Submap::InsertFrame, builder/submap.cc:144-161). */
enum sm_voxel_order {
  SM_VOXEL_ORDER_ASCENDING = 0,
  SM_VOXEL_ORDER_UNORDERED_MAP = 1
};
/* sm_voxel_grid_filter in the given order (sm_voxel_order): the same records, permuted.  An unknown order is
 * SM_ERR_BAD_ARGUMENT, with nothing written. */
int sm_voxel_grid_filter_ordered(int device, const float* points, int64_t n, int64_t stride_bytes,
                                 float voxel_size, int32_t order, float* out, int64_t* m_out);

/* descriptor::M2dp (descriptor/m2dp.cc:37-172; parameters of the constructor, m2dp.h:50-51: r = 0.1,
 * max_distance = 100, t = 16, p = 4, q = 16), the loop-closure descriptor of a submap:
 * M2dp::setInputCloud + getFinalDescriptor.  `points`: float x, y, z records `stride_bytes` (>= 12) apart
 * (data::InnerPointType = 20).  descriptor: p*q + l*t floats, l = ceil(sqrt(max_distance / r)) — [u1; v1],
 * the first left / right singular vectors of the p*q x l*t signature matrix (:148-152); A_out (optional):
 * that matrix as counts, row-major.  Returns 1 (true), 0 for an empty cloud (setInputCloud returns false,
 * :130-133), SM_ERR_BAD_ARGUMENT for r < 1e-6 (:64-67), l*t > 8192, p*q > 256 (the first singular pair is
 * solved on the host in time cubic in p*q) or a too small `capacity`.  A is zero when the max_distance gate
 * drops every point, and so is the descriptor.
 * Two orientations are Eigen-internal in the reference and fixed here: each of the first two PCA axes has
 * its component of largest magnitude positive, and so has u1 (v1 follows).  sm_m2dp_match does not depend
 * on the second; the first decides which points the reference's |.| projections fold together.
 * sm_m2dp_match: matchTwoM2dpDescriptors (:155-170) = |Pearson correlation|, -1 for n < 10. */
int64_t sm_m2dp_descriptor_length(double r, double max_distance, int32_t t, int32_t p, int32_t q);
int sm_m2dp(int device, const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance,
            int32_t t, int32_t p, int32_t q, float* descriptor, int64_t capacity, int32_t* A_out);
double sm_m2dp_match(const float* P, const float* Q, int64_t n);

/* ---- pre_processers::filter::Factory: the scan pre-processing chain --------------------------------------------
 * Every scan the reference matches has gone through filter::Factory::Filter (builder/data/data_collector.cc:137-141;
 * the chain is built from the <filters> node, pre_processors/filter_factory.cc:63-106).  A chain applies its filters
 * in the order they were added; every filter emits its inliers in ascending input index, whole
 * data::InnerPointType records (x, y, z, intensity, factor) copied.  One chain is used by one thread at a time.
 * Built here, under the reference's names and parameter names (type 0 int, 1 float):
 *   Range               filter_range.cc:45-88        min_range (0), max_range (FLT_MAX): sqrtf(x^2+y^2+z^2) in [min, max]
 *   AxisRange           filter_axis_range.cc:41-102  min, max (-/+FLT_MAX), axis_index (2).  A NaN coordinate is kept,
 *                                                    as in the reference (it is neither < min nor > max).
 *   BoundingBoxRemoval  filter_bounding_box.cc:49-83 min_x .. max_z (-/+FLT_MAX): REMOVES the points inside the closed
 *                                                    box; the default box removes every finite point.
 *   RandomSampler       filter_random_sample.cc:35-77 sampling_rate (1); a rate > 0.999 passes everything.  The
 *                       reference builds std::mt19937 eng(rand_dev()) on every Filter call and keeps point j of its
 *                       own input iff uniform_real_distribution<double>(0, 1)(eng) <= sampling_rate: its result is not
 *                       a function of its inputs, only of them and the seed rand_dev() returned.  Two modes, set per
 *                       filter by sm_filter_chain_set_random_sampler:
 *                       HASH (the default), a deterministic stand-in: point i is kept iff
 *                       murmur3_fmix32(i * 0x9E3779B9 + sample_seed) <= sampling_rate * 2^32, i = the point's index in
 *                       the scan handed to the chain (not in the filter's own input), sample_seed a chain option.
 *                       MT19937, the reference's draw at a given seed: every run builds std::mt19937(seed) anew and
 *                       point j of the filter's own input (the previous filter's output, in its emission order) takes
 *                       draw j, two 32-bit engine words w0, w1 -> (double(w0) + double(w1) * 2^32) * 2^-64 as
 *                       libstdc++'s generate_canonical<double, 53> forms it; the float rate is promoted to double.
 *                       Such a filter is a stage of its own, and a run with the same seed gives the same points.
 *   RangeImage          filter_range_image.cc:66-141 (Filter only) top_angle (30), btm_angle (-15), offset_x/y/z (0),
 *                       vertical_line_num (40), horizontal_line_num (1800): the first point in input order per pixel.
 *   GroundRemoval2      filter_ground_removal2.cc:127-414  r_max (100), r_min (1), bin_num (200), segment_num (180),
 *                       start_ground_height (-0.25), long_line_threshold (1), max_long_line_height (0.1),
 *                       max_start_height (0.2), max_error (0.05), max_slope (tan 15 deg), max_b (0.1, unused),
 *                       max_dist_to_line (0.05), search_angle (10), thread_num (4, unused).
 * atan2f is CUDA's here and glibc's in the reference: a point within a few float ulps of a RangeImage row / column
 * border or a GroundRemoval2 segment border can land in the neighbouring pixel / segment.  A float -> int conversion
 * outside int's range (undefined in C++) gives INT_MIN, as the reference's x86 build does.
 * With the chain option all_filters, the reference's other three filters are built too, as the GPU filters of their
 * own entry points.  None of them gives the reference Factory's result by default, which is why the option is off:
 * the reference's StatisticRemoval::Filter is an empty body (filter_statistic_removal.cc:44-59), its VoxelGrid emits
 * in std::unordered_map order unless sm_filter_chain_set_voxel_order selects that order, and its GroundRemoval breaks
 * the ascending order above.  With the option on, each
 * stage reads the previous stage's records in their order, and a run's inlier_index holds the scan index of every
 * emitted record in emission order; the six kinds above emit in ascending order, so their chains are unchanged.
 *   GroundRemoval       min_point_num_in_voxel (10), leaf_size (0.8), height_threshold (0.15): sm_ground_removal_*
 *                       steps 1-3 on the stage's input, records in map order, each index the scan index of the
 *                       record's input point.  A voxel span past 2^21 - 1: SM_ERR_BAD_ARGUMENT.
 *   StatisticRemoval    point_num_meank (30), std_mul (1): sm_statistic_removal_* on the stage's input, kept records in
 *                       input order.  point_num_meank outside 1..63: SM_ERR_BAD_ARGUMENT before any work; 1..K finite
 *                       points: SM_ERR_CHECK_FAILED.
 *   VoxelGrid           voxel_size (0.1): sm_voxel_grid_filter on the stage's input, the same voxel means bit for bit
 *                       (factor 0) in ascending (ix, iy, iz), or in the order sm_filter_chain_set_voxel_order sets,
 *                       non-finite points dropped; each record's index is the scan index of its voxel's first member
 *                       in the stage's input order, which a later HASH RandomSampler keys on (an MT19937 one draws in
 *                       emission order).  voxel_size <= 1e-6 (ConfigsValid, where the reference would run with
 *                       an undefined lround): SM_ERR_BAD_ARGUMENT before any work; finite points spanning 2^21 voxels
 *                       or more along an axis: SM_ERR_BAD_ARGUMENT. */
typedef struct sm_filter_chain sm_filter_chain;
/* filter::Factory::Factory (filter_factory.h).  Needs no device; the first run binds CUDA ordinal `device`. */
int sm_filter_chain_create(int device, sm_filter_chain** out);
int sm_filter_chain_destroy(sm_filter_chain* chain);
/* One <filter name=...> of Factory::InitFromXmlNode (filter_factory.cc:64-80): appends the filter at its constructor's
 * defaults and returns its index.  GroundRemoval (see sm_ground_removal_*), StatisticRemoval (an empty body in the
 * reference, filter_statistic_removal.cc:44-59; PCL's filter is sm_statistic_removal_*) and VoxelGrid (see
 * sm_voxel_grid_filter) are added only while the option all_filters is on, else SM_ERR_UNSUPPORTED_TYPE.  A name the
 * reference does not register either (it skips it, :68-71): SM_ERR_UNKNOWN_OPTION; the chain is unchanged. */
int sm_filter_chain_add(sm_filter_chain* chain, const char* filter_name);
/* One <param type=... name=...>text</param> of Interface::InitFromXmlNode (filter_interface.cc:38-58): `text` is read
 * as pugixml's as_int (type 0) or as_float (type 1), then cast to the parameter's declared type
 * (XmlInterface::SetValue, xml_interface.h:55-75).  Where the reference CHECK-fails (:57): SM_ERR_UNKNOWN_OPTION for a
 * name the filter does not register, SM_ERR_BAD_ARGUMENT for a type other than 0 / 1 (a <param> without `type`). */
int sm_filter_chain_set_param(sm_filter_chain* chain, int filter, const char* name, int type, const char* text);
/* Interface::ConfigsValid of the filter (filter_interface.cc:59; AxisRange filter_axis_range.cc:41-43,
 * BoundingBoxRemoval filter_bounding_box.cc:49-51, RandomSampler filter_random_sample.cc:35-37, VoxelGrid
 * filter_voxel_grid.cc:35): 1 / 0.  As in the reference's Factory (filter_factory.cc:77), an invalid filter still
 * runs, except a VoxelGrid (see above). */
int sm_filter_chain_validate(sm_filter_chain* chain, int filter);
/* Chain options, no reference counterpart: sample_seed (unsigned, 1), the seed of RandomSampler's stand-in;
 * all_filters (unsigned, 0): non-zero makes sm_filter_chain_add accept GroundRemoval, StatisticRemoval and VoxelGrid,
 * 0 restores their refusal.  all_filters affects sm_filter_chain_add only: filters already added stay. */
int sm_filter_chain_set_option(sm_filter_chain* chain, const char* name, const char* text);
/* The generator of the chain's RandomSampler `filter` (see above), no reference counterpart: the reference registers
 * only sampling_rate, so this is not a <param>, and it builds one engine per filter, so it is not a chain option.
 * HASH ignores `seed` (the chain's sample_seed applies); MT19937 draws from std::mt19937(seed), where `seed` is the
 * value the reference's rand_dev() returned for that filter.  SM_ERR_BAD_ARGUMENT, with the chain unchanged, for a
 * `filter` out of range or not a RandomSampler, or an unknown mode.  Applies from the next run on; the _device form
 * runs the generator on its stream. */
enum sm_filter_sampler {
  SM_FILTER_SAMPLER_HASH = 0,
  SM_FILTER_SAMPLER_MT19937 = 1
};
int sm_filter_chain_set_random_sampler(sm_filter_chain* chain, int filter, int32_t mode, uint32_t seed);
/* The emission order of the chain's VoxelGrid `filter` (sm_voxel_order, default SM_VOXEL_ORDER_ASCENDING), no
 * reference counterpart: the reference registers only voxel_size, so this is not a <param>.  Only the order of the
 * stage's records changes; each keeps the scan index of its voxel's first member.  SM_ERR_BAD_ARGUMENT, with the
 * chain unchanged, for a `filter` out of range or not a VoxelGrid, or an unknown order.  Applies from the next run on,
 * in both run forms. */
int sm_filter_chain_set_voxel_order(sm_filter_chain* chain, int filter, int32_t order);
/* Factory::SetInputCloud + Factory::Filter (filter_factory.cc:83-106).  `points`: n records `stride_bytes` (>= 20)
 * apart; `out`: capacity n packed 5-float records; *m_out = the number of inliers; inlier_index (optional, capacity
 * n): their indices in `points`, in emission order (ascending without GroundRemoval and VoxelGrid).  An empty chain
 * copies the input (:90-93); an empty intermediate cloud ends the chain.  `out` and inlier_index are written on
 * success only, except by a failing GroundRemoval2 stage of the _device form.
 * SM_ERR_BAD_ARGUMENT: the errors of the three stages above, a
 * RangeImage with vertical_line_num <= 0 or horizontal_line_num <= 0 (its SetInputCloud keeps the previous cloud,
 * filter_range_image.cc:72-74) or a grid of more than 2^24 pixels / cells.  SM_ERR_CHECK_FAILED: an inverted
 * BoundingBoxRemoval box (CHECK in common/bounding_box.cc:114) or a fitted ground line that does not run outward
 * (CHECK(line.start[0] < line.end[0]), filter_ground_removal2.cc:403).
 * The _device form takes device pointers (in and out may not overlap), runs on `cuda_stream` (a cudaStream_t, NULL =
 * default stream) and returns after the stream has finished; its output feeds sm_motion_compensation_device and
 * sm_set_input_source_f32_device (stride 20) without a host copy. */
int sm_filter_chain_run(sm_filter_chain* chain, const float* points, int64_t n, int64_t stride_bytes, float* out,
                        int64_t* m_out, int32_t* inlier_index_or_null);
int sm_filter_chain_run_device(sm_filter_chain* chain, const float* dev_points, int64_t n, int64_t stride_bytes,
                               float* dev_out, int64_t* m_out, int32_t* dev_inlier_index_or_null, void* cuda_stream);
/* RangeImage::DepthCluster (filter_range_image.cc:143-173, :245-309) after SetInputCloud + Filter of `points` by the
 * chain's filter `filter`, which must be a RangeImage (its parameters are used; the rest of the chain is not run).
 * The range image is Filter's: the first point in input order per pixel, its range sqrtf(x^2+y^2+z^2) of the offset
 * point.  Components of the image under the steps (0,+-1), (0,+-2) (columns wrap) and (+-1,0), an edge where
 * beta = atan2f(d2 sinf(alpha), d1 - d2 cosf(alpha)) > float(10 deg) (d1 / d2 the larger / smaller range, alpha the
 * horizontal resolution for the column steps and the vertical one for the row steps).  Labels 1, 2, ... in row-major
 * order of each component's first pixel, every component counted; the components of >= 20 pixels are emitted in
 * ascending label, each in the reference's breadth-first (std::queue) order.
 * Outputs, capacity n each: out_xyz (3 floats per point: the un-offset input point), out_label, out_index (the
 * point's index in `points`); *m_out = their number.  point_label_or_null (capacity n): the label of every input point
 * that owns its pixel, components under 20 points included, 0 for every other point.
 * SM_ERR_BAD_ARGUMENT: `filter` is not a RangeImage, vertical_line_num <= 0, horizontal_line_num < 2 (the reference
 * steps outside its image there) or more than 2^24 pixels.  SM_ERR_CHECK_FAILED: n == 0 (CHECK(inner_cloud_ !=
 * nullptr), :144).
 * sinf and cosf are taken on the host; atan2f is CUDA's here and glibc's in the reference, so besides the pixel
 * borders above, an edge whose beta lies within a few float ulps of the threshold can differ. */
int sm_filter_chain_depth_cluster(sm_filter_chain* chain, int filter, const float* points, int64_t n,
                                  int64_t stride_bytes, float* out_xyz, uint32_t* out_label, int32_t* out_index,
                                  int64_t* m_out, uint32_t* point_label_or_null);
const char* sm_filter_chain_last_error(const sm_filter_chain* chain);

/* ---- pre_processers::filter::StatisticRemoval: PCL's statistical outlier removal ---------------------------------
 * The reference registers StatisticRemoval (filter_factory.cc:44-52) with point_num_meank (int32, 30) and std_mul
 * (float, 1.0), but its Filter body is a commented-out pcl::StatisticalOutlierRemoval call (setMeanK(point_num_meank),
 * setStddevMulThresh(std_mul)) under a TODO (filter_statistic_removal.cc:44-59): there the filter does nothing.  This
 * is that PCL filter (StatisticalOutlierRemoval::applyFilterIndices of PCL 1.8 / 1.10), restated from upstream PCL and
 * FLANN; no PCL is compiled to check it.  It is a chain stage only with the chain option all_filters; it has its own
 * handle, used by one thread at a time.  Its device buffers belong to the handle and only grow.
 *   1. A point is finite when x, y and z are; only finite points are searched.  A non-finite point gets distance 0.
 *   2. The K + 1 nearest finite points of each finite point, K = point_num_meank: exact search, self-match allowed, over
 *      the coordinates widened to double, with libnabo's tie rules (sm_knn).  Entry 0 (d2 = 0) is dropped.
 *   3. For entries 1..K, in list order: dx = qx - px in float, d2 = ((0 + dx*dx) + dy*dy) + dz*dz in float (FLANN's
 *      L2_Simple<float>), dist_sum += sqrt((double)d2); distance = (float)(dist_sum / K).
 *   4. valid = the number of finite points; sum = sum of distance and sq_sum = sum of (distance * distance, a float
 *      product) over all points; mean = sum / valid, variance = (sq_sum - sum * sum / valid) / (valid - 1),
 *      stddev = sqrt(variance), threshold = mean + (double)std_mul * stddev, all in double.
 *   5. A point is kept iff !(distance > threshold): whole records (x, y, z, intensity, factor) in input order.
 * DIFFERENCE from PCL: sum and sq_sum are the exact sums of their float terms rounded once to double, not PCL's serial
 * double sums in index order, so mean, stddev and threshold depend on the set of inputs alone and are the same on
 * every launch shape.  A point whose distance lies within the few ulps the two sums differ by of the threshold can be
 * kept where PCL removes it, or the reverse (DESIGN.md section 4j).  A slightly negative variance gives a NaN threshold
 * and keeps every point, as in PCL; with no finite point every point is kept.  PCL's setNegative and keep_organized are
 * not used by the reference and are not built. */
typedef struct sm_statistic_removal sm_statistic_removal;
/* Needs no device; the first run binds CUDA ordinal `device`. */
int sm_statistic_removal_create(int device, sm_statistic_removal** out);
int sm_statistic_removal_destroy(sm_statistic_removal* filter);
/* One <param type=... name=...>text</param> of the filter's XML node, parsed exactly as sm_filter_chain_set_param parses
 * it: SM_ERR_UNKNOWN_OPTION for a name other than point_num_meank / std_mul, SM_ERR_BAD_ARGUMENT for a type other than
 * 0 / 1.  Any value is stored; run refuses a point_num_meank outside 1..63. */
int sm_statistic_removal_set_param(sm_statistic_removal* filter, const char* name, int type, const char* text);
/* SetInputCloud + Filter.  `points`: n records `stride_bytes` (>= 20, a multiple of 4) apart, float x, y, z,
 * intensity, factor first; `out`: capacity n packed 5-float records; *m_out = the number kept; inlier_index (optional,
 * capacity n): their indices in `points`, ascending.  n = 0: *m_out = 0.  SM_ERR_BAD_ARGUMENT: point_num_meank outside
 * 1..63 (K + 1 must stay within sm_knn's 64), a bad stride, null pointers with n > 0, more than 2^30 points or more
 * finite points than a 24-level tree of 8-point buckets holds.  SM_ERR_CHECK_FAILED, outputs untouched: between 1 and
 * point_num_meank finite points (PCL reads past its k-list there).
 * The _device form takes device pointers (in and out may not overlap), runs on `cuda_stream` (a cudaStream_t, NULL =
 * default stream) and returns after the stream has finished; it reads the stream's results back twice (the finite
 * count, which sizes the tree, and the number kept).  Its output feeds sm_set_input_source_f32_device (stride 20). */
int sm_statistic_removal_run(sm_statistic_removal* filter, const float* points, int64_t n, int64_t stride_bytes,
                             float* out, int64_t* m_out, int32_t* inlier_index_or_null);
int sm_statistic_removal_run_device(sm_statistic_removal* filter, const float* dev_points, int64_t n,
                                    int64_t stride_bytes, float* dev_out, int64_t* m_out,
                                    int32_t* dev_inlier_index_or_null, void* cuda_stream);
/* The last successful run's mean, stddev, threshold and valid (step 4), as four doubles. */
int sm_statistic_removal_stats(const sm_statistic_removal* filter, double* out4);
const char* sm_statistic_removal_last_error(const sm_statistic_removal* filter);

/* ---- pre_processers::filter::GroundRemoval: the voxel height-range ground filter ---------------------------------
 * GroundRemoval (v1, filter_ground_removal.{h,cc}) with min_point_num_in_voxel (int32, 10), leaf_size (float, 0.8) and
 * height_threshold (float, 0.15).  It is a chain stage only with the chain option all_filters; it has its own handle,
 * used by one thread at a time.  Its device buffers belong to the handle and only grow.
 *   1. Voxel index per axis: (int)(coordinate / leaf_size), a float division truncated toward zero; a NaN quotient or
 *      one outside int's range gives INT_MIN (the reference's x86 build).  Such points are kept in that voxel, so
 *      leaf_size = 0 puts every point into (INT_MIN, INT_MIN, INT_MIN).
 *   2. Voxels in the order of the reference's std::map: lexicographic on signed (ix, iy, iz); a voxel holds its points
 *      in input order.
 *   3. Per voxel: fewer than min_point_num_in_voxel points -> skipped (neither inlier nor outlier).  Else, if iz <= 0:
 *      max_z / min_z from -1e9 / 1e9 with strict > / < (a NaN z updates neither), delta = max_z - min_z in float, and
 *      the voxel is ground iff delta >= 0 && delta <= height_threshold: its points are outliers.  Every other voxel
 *      emits its whole records (x, y, z, intensity, factor) in input order and its points are inliers.
 * LIMIT: the voxel key has 21 bits per axis.  Per axis, the indices other than INT_MIN must span at most 2^21 - 1
 * voxels (about 1 677 km at leaf_size 0.8); past that the run returns SM_ERR_BAD_ARGUMENT where the reference runs. */
typedef struct sm_ground_removal sm_ground_removal;
/* Needs no device; the first run binds CUDA ordinal `device`. */
int sm_ground_removal_create(int device, sm_ground_removal** out);
int sm_ground_removal_destroy(sm_ground_removal* filter);
/* One <param type=... name=...>text</param> of the filter's XML node, parsed exactly as sm_filter_chain_set_param parses
 * it: SM_ERR_UNKNOWN_OPTION for a name other than min_point_num_in_voxel / leaf_size / height_threshold,
 * SM_ERR_BAD_ARGUMENT for a type other than 0 / 1.  Every value is accepted, as in the reference (no ConfigsValid). */
int sm_ground_removal_set_param(sm_ground_removal* filter, const char* name, int type, const char* text);
/* SetInputCloud + Filter.  `points`: n records `stride_bytes` (>= 20, a multiple of 4) apart, float x, y, z,
 * intensity, factor first; `out`: capacity n packed 5-float records, the emitted ones in voxel order; *m_out = their
 * number; index (optional, capacity n): the input index of each emitted record, in emission order, so NOT ascending
 * (Inliers() is sm_ground_removal_indices).  n = 0: *m_out = 0 and empty index lists.  SM_ERR_BAD_ARGUMENT: a bad
 * stride, null pointers with n > 0, more than 2^30 points, or a span past the key limit above.
 * The _device form takes device pointers (in and out may not overlap), runs on `cuda_stream` (a cudaStream_t, NULL =
 * default stream) and returns after the stream has finished; it reads the stream's results back once (the counts and
 * the per-axis index bounds).  Its output feeds sm_set_input_source_f32_device (stride 20). */
int sm_ground_removal_run(sm_ground_removal* filter, const float* points, int64_t n, int64_t stride_bytes, float* out,
                          int64_t* m_out, int32_t* index_or_null);
int sm_ground_removal_run_device(sm_ground_removal* filter, const float* dev_points, int64_t n, int64_t stride_bytes,
                                 float* dev_out, int64_t* m_out, int32_t* dev_index_or_null, void* cuda_stream);
/* Inliers() / Outliers() of the last successful run, ascending input indices: the points of the emitted voxels and of
 * the ground voxels.  *n_inliers / *n_outliers = their numbers; null arrays return the counts only. */
int sm_ground_removal_indices(const sm_ground_removal* filter, int32_t* inliers_or_null, int64_t* n_inliers,
                              int32_t* outliers_or_null, int64_t* n_outliers);
const char* sm_ground_removal_last_error(const sm_ground_removal* filter);

/* ---- RandomSamplerWithPlaneDetect: keep the plane points, sample the rest ------------------------------------------
 * The submap sampler RandomSamplerWithPlaneDetect (random_sample_with_plane_detect.h) with its PlaneDetector
 * (plane_detector.h).  Parameters are the class's setters (no XML node): sampling_rate (float, 1), leaf_size (float,
 * 0.8: the sampler's constructor overrides the detector's 0.5) and min_point_num_in_voxel (size_t, 10).  The ground
 * height threshold is fixed at 0.2 and the RANSAC distance threshold at 0.1.  It is not part of the chain
 * (sm_filter_chain_add refuses the name, as filter::Factory does not register it); it has its own handle, used by one
 * thread at a time, whose device buffers only grow.  A run, in order:
 *   1. n = 0: nothing is emitted.
 *   2. rate > 0.999999 (in double): every record is copied and no detection runs; no plane indices.
 *   3. Voxels: GroundRemoval's keys and order (sm_ground_removal_* steps 1-2), INT_MIN for a NaN or out-of-range
 *      quotient included.
 *   4. Detect: if 0.2 >= leaf_size there are no plane points.  Otherwise, per voxel in map order: fewer than min points
 *      -> skipped; iz <= 0 -> GroundRemoval's z-range rule with threshold 0.2: all its points are plane points, or
 *      none are; iz > 0 with fewer than 2 min points -> skipped; else PCL's SACSegmentation (SACMODEL_PLANE, SAC_RANSAC,
 *      threshold 0.1, optimised coefficients, 50 iterations, probability 0.99, generator seeded 12345u) on its points
 *      in input order, and the refined inliers are plane points iff (float)inliers / (float)count > 0.85 (in double).
 *      DESIGN §4l restates the RANSAC step by step.
 *   5. Sampler, over the input in index order: a plane point is kept; any other point increments other_sum and is kept
 *      iff (float)sampled / (float)other_sum < rate, which then increments sampled.
 * Output: the kept records in input order; Inliers() = the kept indices, Outliers() = the rest, PlaneIndices() = the
 * sorted output of Detect, all ascending.
 * Where the reference is undefined or leaks state, this settles it:
 *   - plane_indices.front() on an empty vector (after the last plane point, or with none) means "no further plane
 *     point";
 *   - PlaneDetector::voxels_ is never cleared, so a reused reference sampler mixes in the voxels of earlier clouds;
 *     every run here starts fresh, as the reference's first call on a new object does;
 *   - PlaneDetector's min_z_ / max_z_ are computed and never read: they do not exist here.
 * LIMITS: the float other_sum is exact up to 2^24, so a run of more than 2^24 points returns SM_ERR_BAD_ARGUMENT; the
 * voxel key's span limit of sm_ground_removal_* applies (SM_ERR_BAD_ARGUMENT) whenever Detect runs.
 * Difference: computeRoots' atan2, cos and sin are evaluated in double and rounded to float (DESIGN §4l). */
typedef struct sm_plane_sampler sm_plane_sampler;
/* Needs no device; the first run binds CUDA ordinal `device`. */
int sm_plane_sampler_create(int device, sm_plane_sampler** out);
int sm_plane_sampler_destroy(sm_plane_sampler* sampler);
/* SetSamplingRate: above 1 -> 1, below 1e-6 (in double) -> (float)1e-6, with the reference's warning as the last
 * error; SM_OK either way. */
int sm_plane_sampler_set_sampling_rate(sm_plane_sampler* sampler, float rate);
int sm_plane_sampler_set_leaf_size(sm_plane_sampler* sampler, float leaf_size);
/* SetMinPointNumInVoxel (size_t): below 5 -> 5, with the reference's warning as the last error. */
int sm_plane_sampler_set_min_point_num_in_voxel(sm_plane_sampler* sampler, uint64_t num);
/* SetInputCloud + Filter.  `points`: n records `stride_bytes` (>= 20, a multiple of 4) apart, float x, y, z,
 * intensity, factor first; `out`: capacity n packed 5-float records, the kept ones in input order; *m_out = their
 * number; index (optional, capacity n): their input indices (= Inliers()).  SM_ERR_BAD_ARGUMENT: a bad stride, null
 * pointers with n > 0, more than 2^24 points, or the span limit.  The _device form takes device pointers (in and out
 * may not overlap), runs on `cuda_stream` (NULL = default stream) and returns after the stream has finished, with one
 * read-back of the counts.  Its output feeds sm_calculate_normals and sm_set_input_target_f32_device (stride 20). */
int sm_plane_sampler_run(sm_plane_sampler* sampler, const float* points, int64_t n, int64_t stride_bytes, float* out,
                         int64_t* m_out, int32_t* index_or_null);
int sm_plane_sampler_run_device(sm_plane_sampler* sampler, const float* dev_points, int64_t n, int64_t stride_bytes,
                                float* dev_out, int64_t* m_out, int32_t* dev_index_or_null, void* cuda_stream);
/* Inliers() / Outliers() of the last successful run, ascending; null arrays return the counts only. */
int sm_plane_sampler_indices(const sm_plane_sampler* sampler, int32_t* inliers_or_null, int64_t* n_inliers,
                             int32_t* outliers_or_null, int64_t* n_outliers);
/* The sorted plane indices of the last successful run (empty on the copy path); a null array returns the count. */
int sm_plane_sampler_plane_indices(const sm_plane_sampler* sampler, int32_t* plane_or_null, int64_t* n_plane);
const char* sm_plane_sampler_last_error(const sm_plane_sampler* sampler);

/* ---- registrator::MultiviewRegistratorLumPcl (registrators/multiview_registrator_lum_pcl.h) ----------------------
 * PCL's Lu-Milios globally consistent alignment (pcl::registration::LUM, PCL 1.8.1) over the frames given to
 * sm_lum_add_cloud, with the reference's fixed settings: 5 rounds of AlignAll, 5 LUM iterations, convergence threshold
 * 0.001, correspondences within 0.25 m.  Each AlignAll adds every frame again as a new graph vertex in each of its 5
 * rounds, so after k calls on N frames the graph has 5kN vertices; vertex v is the v-th cloud ever added and keeps
 * the pose LUM reached.  Records are stride_bytes apart with float x, y, z at offset 0; the rest of each record is
 * copied to the output, so any PCL point type works.  All clouds of a handle share one stride.
 *   sm_lum_add_cloud   MultiviewInterface::AddNewCloud: a copy of n records (n may be 0) and the frame's pose, a
 *                      column-major Matrix4f.  SM_ERR_BAD_ARGUMENT: a null pose, a stride below 12 or not a multiple
 *                      of 4 or unlike the first cloud's, more than 64 frames, more than 2^20 points in a frame.
 *   sm_lum_size        the number of frames.
 *   sm_lum_align_all   AlignAll(output): the output is getTransformedCloud(v) for v < N concatenated; *m_out = its
 *                      record count.  A null out runs the alignment and writes nothing.  SM_ERR_BAD_ARGUMENT, before
 *                      any work: more than 2^28 correspondence queries (the points of frame j summed over all pairs
 *                      j < i; the search holds 16 bytes per query), capacity (records) below *m_out; after the search and before the graph changes: a
 *                      vertex whose cloud has fewer points than the frame whose correspondence indices it is given
 *                      (PCL reads past the cloud there).
 *   sm_lum_poses       the graph's vertex poses, 6 floats (x, y, z, roll, pitch, yaw) per vertex; a null array
 *                      returns the vertex count. */
typedef struct sm_lum sm_lum;
int sm_lum_create(int device, sm_lum** out);
int sm_lum_destroy(sm_lum* h);
int sm_lum_add_cloud(sm_lum* h, const float* points, int64_t n, int64_t stride_bytes, const float* pose_4x4);
int64_t sm_lum_size(const sm_lum* h);
int sm_lum_align_all(sm_lum* h, float* out, int64_t capacity, int64_t* m_out);
int sm_lum_poses(const sm_lum* h, float* out_or_null, int64_t capacity, int64_t* n_vertices);
const char* sm_lum_last_error(const sm_lum* h);

int sm_device_count(void);
const char* sm_version(void);

#ifdef __cplusplus
}
#endif
#endif /* SM_B200_H_ */
