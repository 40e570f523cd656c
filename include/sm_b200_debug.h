/* sm_b200_debug.h — TEST HOOKS of libsm_b200.so.  Not part of the drop-in boundary (include/sm_b200.h):
 * nothing in the reference binds these.  They let tests/ drive pieces of PRODUCT code that have no entry point of
 * their own against INDEPENDENT implementations (numpy / scipy / tests/pyref.py), so that a transcription error
 * shared by the product and the oracle cannot pass unnoticed — most of them without a GPU (DESIGN.md section 2a):
 *   host code of the product, over caller-supplied evaluations
 *     sm_debug_bfgs_minimize   the BFGS minimiser of the GICP stage (csrc/gicp_host.h: PCL's port of GSL
 *                              vector_bfgs2 with the Fletcher line search, gicp_omp_impl.hpp:218-224)
 *     sm_debug_ndt_newton      the NDT Newton loop (csrc/ndt_host.h newton_loop, ndt_omp_impl.hpp:81-171)
 *     sm_debug_gicp_outer      the GICP outer loop (csrc/gicp_host.h outer_loop, gicp_omp_impl.hpp:381-514, :187-246)
 *     sm_debug_ndt_host        6x6 Jacobi-SVD solve, pose <-> 6-vector with Eigen's eulerAngles(0,1,2), Gauss constants
 *     sm_debug_gicp_host       applyState, computeRDerivative
 *     sm_debug_m2dp_host       M2DP's two eigenproblems: PCA axes from the float covariance, [u1; v1] from A and A A^T
 *   device math of the product compiled for the host (the same __host__ __device__ source the kernels call)
 *     sm_debug_solve6_host     SolvePossiblyUnderdeterminedLinearSystem (csrc/linalg_dev.cuh, icp_fast.cc:204-254)
 *     sm_debug_kabsch_host     the point-to-point minimizer: centring, 3x3 SVD, reflection fix (csrc/linalg_dev.cuh,
 *                              icp_fast.cc:326-375)
 *     sm_debug_icp_host        per-match normal-equation terms, AngleAxis / quaternion / angularDistance helpers
 *     sm_debug_ndt_leaf        one leaf of the NDT target grid: covariance, eigenvalue inflation, inverse
 *     sm_debug_ndt_term        one (point, voxel) term of computeDerivatives, pclomp float and stock-PCL double forms
 *     sm_debug_gicp_point      Mahalanobis matrix of a correspondence, one correspondence's cost / gradient terms
 *     sm_debug_voxel_index     the voxel index of a point in the submap filter, the NDT grid and ApproximateVoxelGrid
 *     sm_debug_motion_host     InterpolateTransform(Identity, delta, factor) applied to a point
 *     sm_debug_normals_leaf    the leaf plane fit of CalculateNormals (cloud_types.cc:73-103)
 *     sm_debug_pm_surface_normal_leaf_host  the eigenvector leaf of libpointmatcher's SamplingSurfaceNormal filter
 *     sm_debug_ndt_direct_neighbors  the NDT derivative kernel's DIRECT26 / DIRECT7 / DIRECT1 neighbour searches
 *     sm_debug_filter_host     the filter chain's per-point functions: predicate, RangeImage pixel, GroundRemoval2 cell
 *     sm_debug_filter_fit_host, sm_debug_filter_distance_host  GroundRemoval2's line fit and VerticalDistanceToSegment
 *     sm_debug_depth_edge_host RangeImage::DepthCluster's edge predicate
 *     sm_debug_statistic_removal_exact_sum_host  StatisticRemoval's correctly rounded sum of non-negative floats
 *     sm_debug_statistic_removal_distance_host   StatisticRemoval's per-point mean distance over a neighbour list
 *     sm_debug_ground_removal_index_host, sm_debug_ground_removal_voxel_host  GroundRemoval's voxel index of a point
 *                              and its decision for one voxel
 *     sm_debug_pm_rand_window_host, sm_debug_pm_rand_advance_host, sm_debug_pm_rand_draws_host  the rand reading
 *                              sampler's jump-ahead on glibc's rand() stream and the draws it reaches
 *   on the device
 *     sm_debug_solve6          the 6x6 solver exactly as icp_finish_kernel calls it
 *     sm_debug_knn1_batched    sm_knn1 with the scheduling the ICP iteration uses when many alignments are in flight
 *                              (queries_per_cta > 256: lockstep root visits, then the lanes of a warp pull parked
 *                              searches), so that path's index sets and squared distances meet the oracle's directly
 *     sm_debug_ndt_grid        the NDT target grid as NdtStage::build_grid leaves it: voxel keys, leaves, size guard
 *     sm_debug_ndt_derivatives the 44 sums of NdtStage::eval (computeDerivatives) at given pose vectors, both forms
 *     sm_debug_ndt_derivatives_search  the same with each of pclomp's four neighbour searches
 *     sm_debug_float_tree_knn  the float tree's exact searches: knn1 (eps = 0) and the 20-NN of the covariances
 *     sm_debug_icp_iteration_minimizer  the same with the point-to-point minimizer's phases B and C
 *     sm_debug_icp_iteration   one IcpFast iteration phase by phase: the prologue's mean, G0 and Morton order; phase A's
 *                              matches, distances and histogram; phase B's candidates and per-block partial sums;
 *                              phase C's 29 reduced sums, limit, kept count and pose update
 *     sm_debug_pm_stages       the IcpUsingPointMatcher stand-in's reading filter and score pass: kept points, sorted
 *                              squared distances of the approximate search, trim counts and mean
 *     sm_debug_pm_surface_normals  the stand-in's reference filter (NormalsPipeline) in either leaf mode: kept means,
 *                              normals and box indices, after an optional earlier build into the same owner
 *     sm_debug_pm_rand_sample  the stand-in's reading filter with the rand sampler: keep flags and kept points
 *     sm_debug_approx_voxel_grid  ApproximateVoxelGrid's output cloud, in emission order
 *     sm_debug_gicp_covariances   the GICP covariances of a cloud
 *     sm_debug_gicp_step       correspondences, Mahalanobis matrices and cost sums of one GICP outer iteration
 *     sm_debug_m2dp_stages     every intermediate of M2dpStage: mean, covariance, axes, view axes, A, A A^T, descriptor
 *     sm_debug_radix_sort      radix_sort_pairs_u64 as the tree build, the voxel filters and the NDT grid call it
 *     sm_debug_kd_tree         every array a k-d tree owner (KdCompactTree, NormalsPipeline, FloatTree) fills, after
 *                              an optional earlier build into the same owner
 *     sm_debug_filter_ground_removal2  every intermediate of FilterChain's GroundRemoval2 stage
 *     sm_debug_depth_cluster   DepthCluster's range image, edge mask, labels and BFS level / position per pixel
 *     sm_debug_statistic_removal_distances  the per-point distances of a StatisticRemoval handle's last run
 *   so each device stage of Ndt / NdtWithGicp meets the oracle bit for bit, not only through the final pose, and
 *   each stage of M2DP and of IcpFast's iteration meets a float64 model fed with the device's previous stage */
#ifndef SM_B200_DEBUG_H_
#define SM_B200_DEBUG_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* A: row-major 6x6 (symmetric in the ICP use), b: 6.  path: 0 LLT, 1 rank-reduced min-norm, 2 SVD. */
int sm_debug_solve6(int device, const double* A_36, const double* b_6, double* x_6, int32_t* path);

/* the same routine compiled for the host (no GPU needed): the source both builds share is csrc/linalg_dev.cuh */
int sm_debug_solve6_host(const double* A_36, const double* b_6, double* x_6, int32_t* path);

/* The point-to-point minimizer's solve (la::kabsch_from_sums, as icp_finish_kernel<true> runs it) on the host.
 * sums_32 in the layout phase B/C reduce: [0..2] sum p, [3..5] sum q, [6 + 3i + j] sum q_i p_j, [27] sum sqrt(d2),
 * [28] count (> 0).  R_9 row-major, t_3; path: 3 Kabsch, 4 Kabsch with the reflection fix. */
int sm_debug_kabsch_host(const double* sums_32, double* R_9, double* t_3, int32_t* path);

/* f and/or g may be NULL (value-only / gradient-only evaluations of the line search); return < 0 to abort. */
typedef int (*sm_debug_fdf)(const double* x_6, double* f, double* g_6, void* user);
/* Runs the GICP inner loop (gicp_omp_impl.hpp:225-240): set, then iterate + test_gradient(grad_tol) until
 * it reports success / no progress or max_iterations.  status: 0 success, 1 still running (iteration cap),
 * 2 no progress, -1 error. */
int sm_debug_bfgs_minimize(sm_debug_fdf fn, void* user, double* x_6_inout, double grad_tol,
                           int32_t max_iterations, int32_t* iterations, int32_t* evaluations, int32_t* status);

/* sm_knn1 (include/sm_b200.h) with `queries_per_cta` queries per 256-thread CTA (rounded up to a multiple of
 * 256; 0 = sm_knn1's own one query per thread). */
int sm_debug_knn1_batched(int device, const double* target_3xn, int64_t n_target, const double* query_3xn,
                          int64_t n_query, double epsilon, int bucket_size, int32_t queries_per_cta,
                          int32_t* ids, double* dists2);

/* The host-side scalar pieces of registrator::Ndt's Newton loop (csrc/ndt_host.h), runnable without a GPU, so that
 * product code is compared with numpy directly (tests/test_independent_checks.py):
 *   op 0: JacobiSVD(H).solve(b), ndt_omp_impl.hpp:127-129     in = H[36] row-major, b[6]       out = x[6]
 *   op 1: Translation * AngleAxis(X) * AngleAxis(Y) * AngleAxis(Z) in float, :146-149 / :797-800
 *                                                              in = p[6]                        out = T[16] col-major
 *   op 2: translation + rotation().eulerAngles(0, 1, 2) in float, :103-111
 *                                                              in = T[16] col-major             out = p[6]
 *   op 3: Gauss constants d1, d2, :86-93                       in = {outlier_ratio, resolution} out = {d1, d2}
 * Returns 0, or SM_ERR_BAD_ARGUMENT for an unknown op / null pointer. */
int sm_debug_ndt_host(int32_t op, const double* in, double* out);

/* The ICP iteration's per-match arithmetic and pose-update helpers compiled for the host (csrc/icp_dev.cuh,
 * csrc/linalg_dev.cuh; ErrorElements + ComputePointToPlane, icp_fast.cc:268-313, CheckConvergence :377-405):
 *   op 0: in = n records {p[3], q[3], normal[3], d2}  out = 29 sums: upper triangle of A = sum F F^T (21, row by row),
 *         sum F (n . (p - q)) (6), sum sqrt(d2), count;  F = [p x normal; normal]
 *   op 1: in = {angle, axis[3]}        out = R[9] row-major   (Eigen::AngleAxis::toRotationMatrix)
 *   op 2: in = R[9] row-major          out = {w, x, y, z}     (Eigen::Quaterniond(Matrix3d))
 *   op 3: in = two quaternions {w,x,y,z}  out[0] = angularDistance
 *   op 4: in = two column-major 4x4    out = their product */
int sm_debug_icp_host(int32_t op, const double* in, int64_t n, double* out);

/* The Newton loop of registrator::Ndt (NormalDistributionsTransform::computeTransformation, ndt_omp_impl.hpp:81-171,
 * with the step-length routine whose More-Thuente loop never runs, :757-916) as the product runs it: csrc/ndt_host.h
 * newton_loop, the function that drives the device evaluations in sm_align.  Here the evaluation is the caller's:
 * fn(T, p, sums, user) receives final_transformation_ (column-major 4x4, float-valued) and the pose vector p[6] it
 * was built from (the angle-derivative tables belong to p) and fills sums[0] = score, [1..6] = gradient, [7..42] = Hessian row-major, [43] = neighbour count
 * summed over the points; it returns < 0 to abort. */
typedef int (*sm_debug_ndt_eval)(const double* T_4x4, const double* p_6, double* sums_44, void* user);
int sm_debug_ndt_newton(sm_debug_ndt_eval fn, void* user, const double* guess_4x4, int32_t n_source, float resolution,
                        double step_size, double outlier_ratio, double transformation_epsilon, int32_t max_iterations,
                        double* final_4x4, int32_t* iterations, int32_t* evaluations, double* score);

/* The outer loop of the GICP stage as the product runs it (csrc/gicp_host.h outer_loop =
 * GeneralizedIterativeClosestPoint::computeTransformation + estimateRigidTransformationBFGS, gicp_omp_impl.hpp:381-514,
 * :187-246, with the options of ndt_gicp.cc:50-51), over the caller's per-point work:
 *   correspond(transformation_4x4, R_9, &m, user): correspondences and Mahalanobis matrices for transformation_ (column-
 *       major, float-valued) with R = rot(transformation_ * guess) row-major in double; m = number of correspondences
 *   cost(T_4x4, S_13, user): S[0] = sum res^T M res, S[1..3] = sum M res, S[4..12] = sum (guess p)(M res)^T row-major
 *       for T = guess with applyState(x) (column-major, float-valued)
 * both return < 0 to abort. */
typedef int (*sm_debug_gicp_correspond)(const double* transformation_4x4, const double* R_9, int32_t* m, void* user);
typedef int (*sm_debug_gicp_cost)(const double* T_4x4, double* S_13, void* user);
int sm_debug_gicp_outer(sm_debug_gicp_correspond correspond, sm_debug_gicp_cost cost, void* user,
                        const double* guess_4x4, double* final_4x4, int32_t* iterations, int32_t* bfgs_evaluations);

/* The voxel index of one point {x, y, z} as the three voxelisations compute it (device functions compiled for the host):
 *   op 0: submap filter, lround(x / voxel) (filter_voxel_grid.cc:50-52), param = voxel size; out[3] = 0: point dropped
 *   op 1: NDT grid, int(floor(x * inv) - float(min_b)) per axis (voxel_grid_covariance_omp_impl.hpp:218-220), param = inv
 *   op 2: ApproximateVoxelGrid, floor(x * inv) per axis, out[3] = hash slot (ix * 7171 + iy * 3079 + iz * 4231) & 511 */
int sm_debug_voxel_index(int32_t op, const float* p_3, float param, int32_t min_b, int64_t* out_4);

/* The per-point arithmetic of the GICP kernels compiled for the host (csrc/gicp.cu mahalanobis / cost_terms):
 *   op 0: M = (R C1 R^T + C2)^-1, gicp_omp_impl.hpp:450-457    in = R[9], C1[9], C2[9] row-major     out = M[9]
 *   op 1: one correspondence of the functor, :341-377          in = T[16], base[16] col-major, p_src[3], p_tgt[3], M[9]
 *         out = {res^T M res, (M res)[3], ((base p_src)(M res)^T)[9] row-major} */
int sm_debug_gicp_point(int32_t op, const double* in, double* out);

/* Host pieces of the GICP stage besides the minimiser (csrc/gicp_host.h):
 *   op 0: applyState, gicp_omp_impl.hpp:516-527   in = T[16] col-major, x[6]      out = T'[16] (float arithmetic)
 *   op 1: computeRDerivative, :133-183            in = x[6], R[9] row-major       out = {g[3], g[4], g[5]} */
int sm_debug_gicp_host(int32_t op, const double* in, double* out);

/* The leaf routine of EigenPointCloud::CalculateNormals (cloud_types.cc:73-103; csrc/normals.cu leaf_plane_fit compiled
 * for the host): count (1..7) members {x, y, z} in member order -> mean, unit normal of the plane n . p = 1, kept = 0
 * when rank(covariance) + 1 < 3. */
int sm_debug_normals_leaf(const double* members_3k, int32_t count, double* mean_3, double* normal_3, int32_t* kept);

/* The leaf of libpointmatcher's SamplingSurfaceNormalDataPointsFilter as sm_set_pm_surface_normals(EIGENVECTOR) runs it
 * (csrc/normals.cu leaf_eigen_normal compiled for the host): count (1..7) float members {x, y, z} in member order ->
 * the float mean, the float covariance sum (row-major 3x3) and the unit normal; kept = 0 when rank(C) + 1 < 3 (mean and
 * covariance are still written, the normal is not). */
int sm_debug_pm_surface_normal_leaf_host(const float* members_3k, int32_t count, float* mean_3, float* cov_9,
                                         float* normal_3, int32_t* kept);

/* sm_motion_compensation's arithmetic on the host (csrc/motion_dev.cuh make_motion_params + motion_point): packed
 * {x, y, z, intensity, factor} float records in and out; SM_ERR_BAD_ARGUMENT if a factor is outside [0, 1]. */
int sm_debug_motion_host(const float* points_5n, int64_t n, const double* delta_4x4, float* out_5n);

/* IcpFast's inner compensation on the host (csrc/motion.cu icp_deskew_kernel and icp.cu's compensated phase B, the
 * same __host__ __device__ code): the n points (3xN, the source after G0, caller order, f_i = i / n) de-skewed with
 * InterpolateTransform(Identity, T_iter, f_i) into out_points_3n; if targets_3n, normals_3n and out_terms_7n are
 * given, each point's match against (target i, normal i) as {f_i F[6], residual} (icp_fast.cc:268-302, :284-289). */
int sm_debug_inner_compensation_host(const double* T_iter_4x4, const double* points_3n, const double* targets_3n,
                                     const double* normals_3n, int64_t n, double* out_points_3n, double* out_terms_7n);

/* One leaf of VoxelGridCovariance::applyFilter (voxel_grid_covariance_omp_impl.hpp:209-366; csrc/ndt.cu finish_leaf
 * compiled for the host): the n points of a voxel in input order -> mean, inverse covariance (zero when the leaf has
 * fewer than min_points points or fails the eigenvalue test), float centroid, nr_points (-1 = invalid covariance),
 * searchable. */
int sm_debug_ndt_leaf(const float* points_3n, int32_t n, int32_t min_points, double eig_mult, double* mean_3,
                      double* icov_9, float* centroid_3, int32_t* nr_points, int32_t* searchable);

/* One (point, voxel) term of computeDerivatives (ndt_omp_impl.hpp:397-438 + :483-535; f64_math = 1: the stock PCL
 * double form NdtWithGicp uses): csrc/ndt.cu's update_derivatives compiled for the host, evaluation tables built by
 * csrc/ndt_host.h for the pose vector p.  out43 = {score increment, gradient term[6], Hessian term[36] row-major}. */
int sm_debug_ndt_term(const double* p_6, double outlier_ratio, float resolution, int32_t f64_math,
                      const float* x_orig_3, const float* x_trans_3, const double* voxel_mean_3,
                      const double* voxel_icov_9, double* out43);

/* ---- the device stages of Ndt and NdtWithGicp, each run by the owner sm_align runs it with (NdtStage in
 * csrc/ndt.cu, ApproxVoxelGrid and gicp::Stage in csrc/gicp.cu, FloatTree in csrc/kdtree.cu) on buffers of the
 * hook's own.  Clouds are packed float xyz; 4x4 matrices are column-major; every output array is sized by the
 * caller for the worst case stated. */

/* NdtStage::build_grid (VoxelGridCovariance::filter(true)): the voxels in the device's order (ascending voxel index as
 * a 32-bit unsigned key), each array holding up to n entries.  overflow = 1: the target's box holds more than
 * INT32_MAX voxels (voxel_grid_covariance_omp_impl.hpp:74-84) and the grid is unusable. */
int sm_debug_ndt_grid(int device, const float* target_3n, int64_t n, float resolution, int32_t* n_voxels,
                      int32_t* overflow, int32_t* key, int32_t* nr_points, int32_t* searchable, double* mean_3,
                      double* icov_9, float* centroid_3);

/* NdtStage::build_grid, then NdtStage::eval (computeDerivatives) at each of the n_poses pose vectors p, with the
 * evaluation parameters sm_debug_ndt_term builds; f64_math = 1: the stock-PCL double term math.  sums_44k[44 k ..]: score,
 * gradient[6], Hessian[36] row-major, neighbour count. */
int sm_debug_ndt_derivatives(int device, const float* target_3n, int64_t nt, const float* source_3n, int64_t ns,
                      float resolution, double outlier_ratio, int32_t f64_math, const double* p_6k, int32_t n_poses,
                      double* sums_44k);

/* sm_debug_ndt_derivatives (pclomp's float term math) with the neighbour search of sm_set_ndt_search_method:
 * search_method 0 KDTREE, 1 DIRECT26, 2 DIRECT7, 3 DIRECT1. */
int sm_debug_ndt_derivatives_search(int device, const float* target_3n, int64_t nt, const float* source_3n,
                                    int64_t ns, float resolution, double outlier_ratio, int32_t search_method,
                                    const double* p_6k, int32_t n_poses, double* sums_44k);

/* The direct neighbour searches of the derivative kernel (csrc/ndt.cu for_each_direct_cell and its leaf test,
 * voxel_grid_covariance_omp_impl.hpp:373-441) compiled for the host, no GPU needed: for each point {x, y, z} (the
 * transformed source point), search_method 1 DIRECT26 / 2 DIRECT7 / 3 DIRECT1, cells of `resolution` in the box
 * min_b_3 .. min_b_3 + div_b_3 - 1, and the grid's leaves (leaf_key: leaf index, leaf_nr_points: nr_points, -1 for
 * a failed covariance), counts_n[i] neighbours whose leaf indices are keys_26n[26 i ..], in the order the kernel
 * visits them. */
int sm_debug_ndt_direct_neighbors(int32_t search_method, const float* points_3n, int64_t n, float resolution,
                                  const int32_t* min_b_3, const int32_t* div_b_3, const int32_t* leaf_key,
                                  const int32_t* leaf_nr_points, int64_t n_leaves, int32_t* counts_n,
                                  int32_t* keys_26n);

/* FloatTree::build over the cloud, then for each double query {x, y, z}: k = 1, knn1 with eps = 0 (the fitness
 * score and the GICP correspondences); k = 20, knn_k (the GICP covariances), ascending (d2, id), unused entries
 * -1 / +inf.  ids / d2 hold nq * k entries; ids are indices into the cloud. */
int sm_debug_float_tree_knn(int device, const float* cloud_3n, int64_t n, const double* query_3m, int64_t nq,
                            int32_t k, int32_t* ids, double* d2);

/* The IcpUsingPointMatcher stand-in's device stages (csrc/icp_pm.cu PmStage) as pm_align runs them, on packed float
 * clouds: PmStage::sample of the n reading points with prob and seed -> *kept and sampled_3n (3 * kept doubles in input
 * order; capacity 3 * n); FloatTree::build of the nt target points, then PmStage::score_pass of the UNFILTERED reading
 * moved by T_4x4 (column-major) with the bound (1 + knn_epsilon)^2 and the trim ratio -> keys_n (the n squared
 * distances in ascending order, +inf where no match was found) and out_3 = {mean kept distance, kept, valid}. */
int sm_debug_pm_stages(int device, const float* reading_3n, int64_t n, const float* target_3n, int64_t nt, float prob,
                       uint32_t seed, const double* T_4x4, float knn_epsilon, float ratio, int64_t* kept,
                       double* sampled_3n, double* keys_n, double* out_3);

/* The generator of the rand reading sampler (sm_set_pm_reading_sampler GLIBC_RAND; csrc/icp_pm.cu, the same
 * __host__ __device__ jump-ahead the device runs) compiled for the host, no GPU needed.  A window is 31 consecutive
 * words of glibc's TYPE_3 additive recurrence; the window at position p is the one whose next draw is draw p.
 *   sm_debug_pm_rand_window_host   the window at `position` after srand(seed)
 *   sm_debug_pm_rand_advance_host  the window `steps` draws after window_31
 *   sm_debug_pm_rand_draws_host    draws position .. position + count - 1 (rand() values), from the window at
 *                                  `position` and then the recurrence one step at a time. */
int sm_debug_pm_rand_window_host(uint32_t seed, int64_t position, uint32_t* window_31);
int sm_debug_pm_rand_advance_host(const uint32_t* window_31, uint64_t steps, uint32_t* out_31);
int sm_debug_pm_rand_draws_host(uint32_t seed, int64_t position, int64_t count, int32_t* out);

/* PmStage::sample with the rand sampler as pm_align runs it: the n packed float reading points (n <= 2^24), draw i
 * taken from position + i of srand(seed)'s stream, kept iff (float)rand() / (float)RAND_MAX < prob -> *kept,
 * sampled_3n (3 * kept doubles in input order; capacity 3 * n) and keep_n (the device's flag of each point, 0 / 1). */
int sm_debug_pm_rand_sample(int device, const float* reading_3n, int64_t n, float prob, uint32_t seed,
                            int64_t position, int64_t* kept, double* sampled_3n, uint8_t* keep_n);

/* The IcpUsingPointMatcher stand-in's reference filter as pm_align runs it: the packed float cloud widened into a
 * NormalsPipeline and run with `mode` (sm_pm_surface_normals).  With n_first > 0 the first cloud is run first, with
 * the same mode, into the SAME owner.  Writes the m kept boxes in output order: points_3m and normals_3m (doubles,
 * capacity 3 * n each), the smallest member index of each box index_m (capacity n), and *m. */
int sm_debug_pm_surface_normals(int device, int32_t mode, const float* first_3n, int64_t n_first, const float* cloud_3n,
                                int64_t n, double* points_3m, double* normals_3m, int64_t* index_m, int64_t* m);

/* One IcpFast iteration as sm_align runs it (IcpFastBuffers, KdWorkspace, no graphs; csrc/icp.cu): icp_prologue and
 * iterations 1 .. iteration-1, then iteration `iteration` one phase at a time with a synchronise and a copy after
 * each.  Double clouds are n x 3 in caller order; guess_4x4 is column-major; max_iteration = iteration and the
 * convergence test is off, so the iteration computes the final score.  geometry_2 = {nb, tile}: the phase-B blocks
 * for ns and the Morton positions per block; with source_3n NULL only geometry_2 is written.  Every other output
 * may be NULL and is sized by the caller:
 *   prologue_35   target mean[3], G0[16], T_iter entering the iteration[16]       perm_n  Morton position -> caller index
 *   phase A (per source point, caller order)   match_n  target index (caller order) or -1, d2_n, pm_6n the {point,
 *                 normal} record phase B gathers (zero without a match); hist_2048
 *   phase B       hist2_2048, cand_cnt[nb], cand_key[nb * tile] and cand_terms_8[nb * tile * 8] (block j's candidates
 *                 start at j * tile: the d2 bits; F[6], residual, sqrt(d2)), partials_29[nb * 29]
 *   phase C       sums_29 (all-ones bit patterns unless phase C reached its reduction), final_18 = {limit, final_score,
 *                 T_iter[16]}, final_5 = {kept, status, solve_path, iteration, done}, hist_after_4096 (hist, hist2). */
int sm_debug_icp_iteration(int device, const double* source_3n, int64_t ns, const double* target_3n,
                           const double* normals_3n, int64_t nt, const double* guess_4x4, float dist_outlier_ratio,
                           float knn_epsilon, int32_t knn_queries_per_cta, int32_t inner_compensation, int32_t iteration,
                           int32_t* geometry_2, double* prologue_35, uint32_t* perm_n, int32_t* match_n, double* d2_n,
                           double* pm_6n, uint32_t* hist_2048, uint32_t* hist2_2048, uint32_t* cand_cnt, uint64_t* cand_key,
                           double* cand_terms_8, double* partials_29, double* sums_29, double* final_18, int64_t* final_5,
                           uint32_t* hist_after_4096);

/* sm_debug_icp_iteration with the error minimizer of sm_set_icp_error_minimizer (SM_ICP_POINT_TO_PLANE gives
 * sm_debug_icp_iteration itself; another value returns SM_ERR_BAD_ARGUMENT).  With SM_ICP_POINT_TO_POINT every
 * iteration runs the point-to-point phases B and C: cand_terms_8 holds {p[3], q[3], 0, sqrt(d2)} per candidate,
 * partials_29 and sums_29 the moments of la::kabsch_from_sums ([0..2] sum p, [3..5] sum q, [6 + 3i + j] sum q_i p_j,
 * [27] sum sqrt(d2), [28] count, the rest 0), final_5[2] the solve path 3 / 4. */
int sm_debug_icp_iteration_minimizer(int device, const double* source_3n, int64_t ns, const double* target_3n,
                                     const double* normals_3n, int64_t nt, const double* guess_4x4,
                                     float dist_outlier_ratio, float knn_epsilon, int32_t knn_queries_per_cta,
                                     int32_t inner_compensation, int32_t error_minimizer, int32_t iteration,
                                     int32_t* geometry_2, double* prologue_35, uint32_t* perm_n, int32_t* match_n,
                                     double* d2_n, double* pm_6n, uint32_t* hist_2048, uint32_t* hist2_2048,
                                     uint32_t* cand_cnt, uint64_t* cand_key, double* cand_terms_8, double* partials_29,
                                     double* sums_29, double* final_18, int64_t* final_5, uint32_t* hist_after_4096);

/* ApproxVoxelGrid::filter (pcl::ApproximateVoxelGrid): *m_out points into out_3n (capacity n). */
int sm_debug_approx_voxel_grid(int device, const float* points_3n, int64_t n, float leaf, float* out_3n,
                               int64_t* m_out);

/* the cloud's own float tree + gicp::Stage::covariances (computeCovariances, k = 20, epsilon 1e-3): n row-major 3x3;
 * zeros for fewer than 20 points, as the GICP stage leaves them. */
int sm_debug_gicp_covariances(int device, const float* cloud_3n, int64_t n, double* covs_9n);

/* One GICP outer iteration's device work (gicp::Stage): the covariances of both clouds, the correspondences for
 * transformation_ with R = rot(transformation_ * guess) from gicp::outer_rotation, then the cost at each of the
 * n_states states x (T = guess with applyState(x)), in sequence on one last-block ticket.  match[ns]: target index or -1;
 * maha_9n: the Mahalanobis matrix of each matched source point (row-major); *count: matches;
 * sums_13k[13 k ..]: sum res^T M res, sum M res[3], sum (guess p)(M res)^T[9] row-major. */
int sm_debug_gicp_step(int device, const float* source_3n, int64_t ns, const float* target_3n, int64_t nt,
                       const double* guess_4x4, const double* transformation_4x4, const double* x_6k, int32_t n_states,
                       int32_t* match, double* maha_9n, int32_t* count, double* sums_13k);

/* The host routines of M2dp::setInputCloud (csrc/m2dp.cu), no GPU needed:
 *   op 0: m2dp_axes       in = cov_6 (float xx xy xz yy yz zz)    out = E[9] (E[k * 3 + j]: component k of axis j)
 *         axes by descending eigenvalue, each of the first two with its largest-magnitude component positive,
 *         third = first x second in float; the identity when an entry is not finite
 *   op 1: m2dp_descriptor in = A (rows x cols int32, row-major), gram = A A^T (rows x rows)
 *                                                                  out = [u1; v1] (rows + cols floats), zero if A is */
int sm_debug_m2dp_host(int32_t op, const float* cov_6, const int32_t* A, const double* gram, int32_t rows, int32_t cols,
                       float* out);

/* M2dpStage::run as sm_m2dp runs it (arguments as for sm_m2dp, n >= 1), then m2dp_descriptor: the float mean, the six
 * double covariance sums and the six float entries sum / float(n - 1), E[9], the view axes {xa[3], ya[3]} of each of
 * the rows = p * q views (6 * rows floats), A (rows x cols counts), A A^T (rows x rows) and the descriptor
 * (rows + cols floats), with cols = ceil(sqrt(max_distance / r)) * t. */
int sm_debug_m2dp_stages(int device, const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance,
                         int32_t t, int32_t p, int32_t q, float* mean_3, double* cov_sums_6, float* cov_6, float* E_9,
                         float* views_6r, int32_t* A, double* gram, float* descriptor);

/* ---- the two device stages every matcher builds on, run through the functions and owners the matchers call */

/* radix_sort_pairs_u64 (csrc/radix_sort.cu) over `batch` independent arrays [batch][stride] of n (key, value) pairs,
 * the low 8 * passes bits of the keys ordered (stable), with scratch sized by radix_sort_scratch_bytes(n, batch).
 * Both ping-pong buffers start as copies of the caller's arrays, entries n..stride-1 of each batch included, and
 * keys_out / vals_out ([batch][stride]) receive the buffer holding the result, so a write past n shows. */
int sm_debug_radix_sort(int device, const uint64_t* keys, const uint32_t* vals, int64_t n, int32_t batch, int64_t stride,
                        int32_t passes, uint64_t* keys_out, uint32_t* vals_out);

/* One k-d tree owner, built as the matchers build it: with n_first > 0 first over the first cloud, then over the cloud,
 * into the SAME owner, workspace and input buffers (a reused handle).  variant:
 *   0  KdCompactTree with the normals payload (IcpFast's target): double clouds, normals_3n required, bucket 2..8
 *   1  KdCompactTree with the ids payload (sm_knn1): double clouds, bucket 2..8
 *   2  NormalsPipeline (CalculateNormals): double clouds, bucket 7
 *   3  FloatTree (Ndt fitness, GICP, type-1 score): packed float clouds, bucket 8
 * levels must equal kd_num_levels(n, bucket), L below; the arrays the owner fills are copied out, unwritten slots as
 * the device holds them:
 *   nodes    blocked_node_slots(L) 16-byte KdNode records          order  n leaf-order ids
 *   variants 0 / 1:  cut, dim  2^L - 1 entries (heap order)          node_2l  2^L {cut, dim as int64} records
 *                    pb  (8 << L) * 3 doubles                        pn  (8 << L) * 4 doubles (0) / pid  8 << L (1)
 *   variant 3:       bpts  n 32-byte {x, y, z, id} records
 * Arrays of other variants may be NULL. */
int sm_debug_kd_tree(int device, int32_t variant, int32_t bucket, const void* first_3n, const double* first_normals_3n,
                     int64_t n_first, const void* cloud_3n, const double* normals_3n, int64_t n, int32_t levels,
                     void* nodes, uint32_t* order, double* cut, uint8_t* dim, double* node_2l, double* pb, double* pn,
                     int32_t* pid, void* bpts);

/* The per-point functions of the filter chain (csrc/filters.cu) compiled for the host, for filter `filter` of `chain`
 * over n packed 5-float records (record i is given scan index i):
 *   op 0  the predicate of Range / AxisRange / BoundingBoxRemoval / RandomSampler: iout[i] = 1 kept, 0 removed
 *   op 1  RangeImage's pixel (filter_range_image.cc:102-126): iout[2i] = row, iout[2i+1] = col, -1 -1 for an outlier
 *   op 2  GroundRemoval2's cell (filter_ground_removal2.cc:163-191): iout[2i] = segment, iout[2i+1] = bin, fout[i] = range */
struct sm_filter_chain;
int sm_debug_filter_host(const struct sm_filter_chain* chain, int32_t filter, int32_t op, const float* records, int64_t n,
                         int32_t* iout, float* fout);
/* FitLocalLine (filter_ground_removal2.cc:29-44) over n >= 2 points (d, z): m_b = {m, b}. */
int sm_debug_filter_fit_host(const float* d, const float* z, int32_t n, float* m_b);
/* VerticalDistanceToSegment (filter_ground_removal2.cc:398-414) of point (d, z) to a segment's lines, each
 * {start d, start z, end d, end z}; SM_ERR_CHECK_FAILED where the reference's CHECK(line.start[0] < line.end[0]) fails. */
int sm_debug_filter_distance_host(const float* lines_4l, int32_t n_lines, float d, float z, float* distance);
/* FilterChain's GroundRemoval2 stage with the parameters of filter `filter` of `chain`, over n host records:
 *   cell[n]            segment * bin_num + bin of each point       member[n]  1 if the point joined its cell (:204-209)
 *   cell_members[c]    members per cell                            cell_min_2c  min_z_point (d, z) per cell (valid
 *                                                                               where the cell has a member)
 *   lines_4, n_lines   [segment_num][max_lines] lines {d0, z0, d1, z1} and their number per segment;
 *                      max_lines must be bin_num / 2 + 1
 *   keep[n]            1 for the points that are not ground
 * Returns SM_OK, or SM_ERR_CHECK_FAILED with the arrays filled when a line does not run outward. */
int sm_debug_filter_ground_removal2(int device, const struct sm_filter_chain* chain, int32_t filter, const float* points,
                                    int64_t n, int64_t stride_bytes, int32_t max_lines, uint32_t* cell, uint8_t* member,
                                    uint32_t* cell_members, float* cell_min_2c, float* lines_4, int32_t* n_lines,
                                    uint8_t* keep);
/* RangeImage::DepthCluster's edge predicate (csrc/depth_cluster.cu, filter_range_image.cc:288-301) compiled for the
 * host, with the resolutions of filter `filter` (a RangeImage) of `chain`: for pair i of ranges a[i], b[i] and
 * neighbour step step[i] (0..3 the column steps, 4..5 the row steps) edge[i] = 1 / 0 and beta[i].
 * sin_cos4 (optional): sinf / cosf of the horizontal, then of the vertical resolution. */
int sm_debug_depth_edge_host(const struct sm_filter_chain* chain, int32_t filter, const float* a, const float* b,
                             const int32_t* step, int64_t n, uint8_t* edge, float* beta, float* sin_cos4);
/* sm_filter_chain_depth_cluster's device stages for filter `filter` of `chain` over n host records, per pixel
 * (row-major, vertical_line_num x horizontal_line_num): image (the owner's range, 0 when empty), owner (input index,
 * -1), mask (bit k: an edge along neighbour step k), label (0 when empty), level (BFS level in its cluster, -1 outside
 * the kept clusters) and seq (position in its cluster's output order, -1 likewise); *components = every component,
 * dropped ones included.  Return codes as sm_filter_chain_depth_cluster. */
int sm_debug_depth_cluster(int device, const struct sm_filter_chain* chain, int32_t filter, const float* points,
                           int64_t n, int64_t stride_bytes, float* image, int32_t* owner, uint8_t* mask, uint32_t* label,
                           int32_t* level, int32_t* seq, int32_t* components);

/* StatisticRemoval's correctly rounded sum (csrc/statistic_removal.cuh) compiled for the host: the double nearest the
 * exact sum of n non-negative floats, +inf if one term is +inf.  SM_ERR_BAD_ARGUMENT for a negative or NaN term. */
int sm_debug_statistic_removal_exact_sum_host(const float* terms, int64_t n, double* sum);
/* StatisticRemoval's step 3 (csrc/statistic_removal.cuh) compiled for the host: the distance of query (x, y, z) over
 * its neighbours 1..K, given as K (x, y, z) triples in list order (entry 0 excluded), K = 1..63. */
int sm_debug_statistic_removal_distance_host(const float* query_3, const float* neighbours_3k, int32_t K,
                                             float* distance);
/* The per-point distances of `filter`'s last successful run, in input order (0 for a non-finite point): *n = that
 * run's point count (0 before any run); SM_ERR_BAD_ARGUMENT when capacity < *n. */
int sm_debug_statistic_removal_distances(const struct sm_statistic_removal* filter, float* out, int64_t capacity,
                                         int64_t* n);

/* GroundRemoval's voxel index (csrc/ground_removal.cu gr_index) compiled for the host: ixyz[3i + d] = the index along
 * axis d of record i of n records `stride_bytes` apart, (int)(coordinate / leaf_size) or INT_MIN. */
int sm_debug_ground_removal_index_host(const float* points, int64_t n, int64_t stride_bytes, float leaf_size,
                                       int32_t* ixyz);
/* GroundRemoval's decision for one voxel (gr_z_update, gr_voxel_status) compiled for the host, over the z of its
 * `count` points in input order and its z index iz: *status 0 skipped, 1 ground (outliers), 2 kept (inliers);
 * max_min_2 = max_z, min_z as the reference's loop leaves them (-1e9, 1e9 when the loop does not run). */
int sm_debug_ground_removal_voxel_host(const float* z, int64_t count, int32_t iz, int32_t min_point_num_in_voxel,
                                       float height_threshold, int32_t* status, float* max_min_2);

/* RandomSamplerWithPlaneDetect's single-hypothesis pieces (csrc/plane_sampler.cu) compiled for the host.  op 0:
 * isSampleGood over in = p0, p1, p2 (x, y, z each): out[0] = 1 or 0.  op 1: computeModelCoefficients over the same:
 * out[0..3].  op 2: in = c[4], p[3]: out[0] = |c . (p, 1)|, out[1] = 1 iff it is an inlier (< 0.1 in double).
 * op 3: pcl::eigen33 of the row-major symmetric 3x3 in: out[0..2] = the eigenvector of the smallest eigenvalue. */
int sm_debug_plane_sampler_piece_host(int32_t op, const float* in, float* out);
/* The ratio rule in closed form compiled for the host: out[k - k0] = 1 iff non-plane point k (1-based) is kept at
 * `rate`, for k0 <= k < k1, 1 <= k0, k1 <= 2^24 + 1. */
int sm_debug_plane_sampler_keep_host(float rate, int64_t k0, int64_t k1, uint8_t* out);
/* Keep (on = 1) or stop keeping the per-voxel trace of the sampler's runs. */
int sm_debug_plane_sampler_trace(struct sm_plane_sampler* sampler, int32_t on);
/* The trace of the last successful run with the trace on: one record of 8 words per voxel in map order (int32
 * status, iterations, best count, final count; float refined coefficients[4]); status 0 skipped, 1 / 2 z-range rule
 * with / without plane points, 3 skipped before RANSAC, 4 / 5 RANSAC with / without.  *n = the voxels (0 when Detect
 * did not run); SM_ERR_BAD_ARGUMENT when capacity < *n. */
int sm_debug_plane_sampler_voxels(struct sm_plane_sampler* sampler, void* out, int64_t capacity, int64_t* n);

#ifdef __cplusplus
}
#endif
#endif /* SM_B200_DEBUG_H_ */
