// Test hooks of include/sm_b200_debug.h: the product's host code driven by a caller's callbacks, its device math
// compiled for the host, and its Ndt / NdtWithGicp / M2DP device stages run on buffers of their own.
#include "../../include/sm_b200.h"
#include "../../include/sm_b200_debug.h"

#include <string.h>

#include <map>
#include <vector>

#include "common.cuh"
#include "compact.cuh"
#include "icp_dev.cuh"
#include "kernels.h"
#include "linalg_dev.cuh"
#include "gicp_host.h"
#include "ndt_host.h"

namespace smb {
namespace {

__global__ void debug_solve6_kernel(const double* __restrict__ A, const double* __restrict__ b, double* __restrict__ x,
                                    int* __restrict__ path) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *path = la::solve_possibly_underdetermined(A, b, x);
}

}  // namespace
}  // namespace smb

using namespace smb;

extern "C" {

int sm_debug_solve6(int device, const double* A, const double* b, double* x, int32_t* path) {
  if (!A || !b || !x || !path) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf buf;
  SMB_RC(buf.reserve(64 * sizeof(double)));
  double* d = (double*)buf.p;
  SMB_CUDA_OK(cudaMemcpy(d, A, 36 * sizeof(double), cudaMemcpyHostToDevice));
  SMB_CUDA_OK(cudaMemcpy(d + 36, b, 6 * sizeof(double), cudaMemcpyHostToDevice));
  debug_solve6_kernel<<<1, 32>>>(d, d + 36, d + 42, reinterpret_cast<int*>(d + 48));
  int p = 0;
  SMB_CUDA_OK(cudaMemcpy(x, d + 42, 6 * sizeof(double), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(&p, d + 48, sizeof(int), cudaMemcpyDeviceToHost));
  *path = p;
  return SM_OK;
}

// test hook: csrc/linalg_dev.cuh's solver (the code icp_finish_kernel runs when its Cholesky certificate is not
// conclusive) compiled for the HOST, so the product's transcription is checked against numpy without a GPU
int sm_debug_solve6_host(const double* A, const double* b, double* x, int32_t* path) {
  if (!A || !b || !x || !path) return SM_ERR_BAD_ARGUMENT;
  *path = la::solve_possibly_underdetermined(A, b, x);
  return SM_OK;
}

// test hook: the point-to-point minimizer's centring, 3x3 SVD and reflection fix (csrc/linalg_dev.cuh
// kabsch_from_sums, the code icp_finish_kernel<true> runs on lane 0) compiled for the HOST
int sm_debug_kabsch_host(const double* sums, double* R, double* t, int32_t* path) {
  if (!sums || !R || !t || !path) return SM_ERR_BAD_ARGUMENT;
  *path = la::kabsch_from_sums(sums, R, t);
  return SM_OK;
}

// test hook: the NDT Newton loop of the product (ndt_host.h newton_loop, the function ndt_run drives the device
// with) over a caller-supplied evaluation — no GPU involved
int sm_debug_ndt_newton(sm_debug_ndt_eval fn, void* user, const double* guess_4x4, int32_t n_source, float resolution,
                        double step_size, double outlier_ratio, double transformation_epsilon, int32_t max_iterations,
                        double* final_4x4, int32_t* iterations, int32_t* evaluations, double* score) {
  if (!fn || !guess_4x4 || !final_4x4 || !iterations || !evaluations || !score || n_source <= 0)
    return SM_ERR_BAD_ARGUMENT;
  ndt::Options o;
  o.resolution = resolution; o.step_size = step_size; o.outlier_ratio = outlier_ratio;
  o.transformation_epsilon = transformation_epsilon; o.max_iterations = max_iterations;
  NdtEvalParams P = ndt::eval_params(o, false);
  ndt::NewtonOut nw;
  const int rc = ndt::newton_loop(o, guess_4x4, n_source, P, [&](const NdtEvalParams& Pe, const double* p6, double* sums) -> int {
    double T[16];
    for (int i = 0; i < 16; ++i) T[i] = (double)Pe.T[i];
    return fn(T, p6, sums, user);
  }, &nw);
  if (rc < 0) return rc;
  for (int i = 0; i < 16; ++i) final_4x4[i] = (double)nw.final_T[i];
  *iterations = nw.iterations; *evaluations = nw.evaluations; *score = nw.score;
  return SM_OK;
}

// test hook: the GICP outer loop of the product (gicp_host.h outer_loop: start vector, f / g from the 13 sums, BFGS
// driver, convergence test, final composition — the function gicp_run drives the device with) over a caller's
// correspondence and cost functions; no GPU involved
int sm_debug_gicp_outer(sm_debug_gicp_correspond correspond, sm_debug_gicp_cost cost, void* user, const double* guess_4x4,
                        double* final_4x4, int32_t* iterations, int32_t* bfgs_evaluations) {
  if (!correspond || !cost || !guess_4x4 || !final_4x4 || !iterations || !bfgs_evaluations) return SM_ERR_BAD_ARGUMENT;
  float guess[16];
  for (int i = 0; i < 16; ++i) guess[i] = (float)guess_4x4[i];
  gicp::OuterOut go;
  const int rc = gicp::outer_loop(
      gicp::Options(), guess,
      [&](const float* transformation, const double* R, int* m) -> int {
        double T[16];
        for (int i = 0; i < 16; ++i) T[i] = (double)transformation[i];
        int32_t mm = 0;
        const int r = correspond(T, R, &mm, user);
        *m = (int)mm;
        return r;
      },
      [&](const float* Tf, double* S) -> int {
        double T[16];
        for (int i = 0; i < 16; ++i) T[i] = (double)Tf[i];
        return cost(T, S, user);
      },
      &go);
  if (rc < 0) return SM_ERR_CUDA;
  for (int i = 0; i < 16; ++i) final_4x4[i] = (double)go.final_T[i];
  *iterations = go.iterations;
  *bfgs_evaluations = go.bfgs_evals;
  return SM_OK;
}

// test hook: the leaf routine of CalculateNormals (normals.cu leaf_plane_fit) compiled for the host
int sm_debug_normals_leaf(const double* members_3k, int32_t count, double* mean3, double* normal3, int32_t* kept) {
  if (!members_3k || !mean3 || !normal3 || !kept) return SM_ERR_BAD_ARGUMENT;
  const int r = normals_debug_leaf_host(members_3k, count, mean3, normal3);
  if (r < 0) return SM_ERR_BAD_ARGUMENT;
  *kept = r;
  return SM_OK;
}

// test hook: the eigenvector leaf of SamplingSurfaceNormal (normals.cu leaf_eigen_normal) compiled for the host
int sm_debug_pm_surface_normal_leaf_host(const float* members_3k, int32_t count, float* mean_3, float* cov_9,
                                         float* normal_3, int32_t* kept) {
  if (!members_3k || !mean_3 || !cov_9 || !normal_3 || !kept) return SM_ERR_BAD_ARGUMENT;
  const int r = pm_normals_debug_leaf_host(members_3k, count, mean_3, cov_9, normal_3);
  if (r < 0) return SM_ERR_BAD_ARGUMENT;
  *kept = r;
  return SM_OK;
}

// test hook: the voxel index of a point as the three voxelisations compute it, compiled for the host
int sm_debug_ground_removal_index_host(const float* points, int64_t n, int64_t stride_bytes, float leaf_size,
                                       int32_t* ixyz) {
  if ((n > 0 && (!points || !ixyz)) || n < 0 || stride_bytes < 12 || stride_bytes % 4) return SM_ERR_BAD_ARGUMENT;
  for (int64_t i = 0; i < n; ++i)
    gr_debug_index_host(points + i * (stride_bytes / 4), leaf_size, ixyz + 3 * i);
  return SM_OK;
}

int sm_debug_ground_removal_voxel_host(const float* z, int64_t count, int32_t iz, int32_t min_point_num_in_voxel,
                                       float height_threshold, int32_t* status, float* max_min_2) {
  if ((count > 0 && !z) || count < 0 || count > INT32_MAX || !status || !max_min_2) return SM_ERR_BAD_ARGUMENT;
  *status = gr_debug_voxel_host(z, count, iz, min_point_num_in_voxel, height_threshold, max_min_2);
  return SM_OK;
}

// test hooks: RandomSamplerWithPlaneDetect's pieces and closed-form ratio rule compiled for the host, its trace
int sm_debug_plane_sampler_piece_host(int32_t op, const float* in, float* out) {
  if (!in || !out) return SM_ERR_BAD_ARGUMENT;
  return ps_debug_piece_host(op, in, out) == 0 ? SM_OK : SM_ERR_BAD_ARGUMENT;
}

int sm_debug_plane_sampler_keep_host(float rate, int64_t k0, int64_t k1, uint8_t* out) {
  if (k0 < 1 || k1 < k0 || k1 > (1 << 24) + 1 || (k1 > k0 && !out)) return SM_ERR_BAD_ARGUMENT;
  ps_debug_keep_host(rate, k0, k1, out);
  return SM_OK;
}

int sm_debug_plane_sampler_trace(sm_plane_sampler* sampler, int32_t on) {
  PlaneSampler* f = plane_sampler_of(sampler);
  if (!f) return SM_ERR_BAD_ARGUMENT;
  f->trace_on = on != 0;
  return SM_OK;
}

int sm_debug_plane_sampler_voxels(sm_plane_sampler* sampler, void* out, int64_t capacity, int64_t* n) {
  PlaneSampler* f = plane_sampler_of(sampler);
  if (!f || !n) return SM_ERR_BAD_ARGUMENT;
  *n = f->n_voxels;
  if (f->n_voxels == 0) return SM_OK;
  if (!out || capacity < f->n_voxels) return SM_ERR_BAD_ARGUMENT;
  SMB_CUDA_OK(cudaMemcpy(out, f->trace.p, (size_t)f->n_voxels * sizeof(PsTrace), cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_voxel_index(int32_t op, const float* p3, float param, int32_t min_b, int64_t* out4) {
  if (!p3 || !out4) return SM_ERR_BAD_ARGUMENT;
  switch (op) {
    case 0: {   // submap filter (filter_voxel_grid.cc:50-52): lround(x / voxel); out[3] = 0 when the point is dropped
      long long ix[3] = {0, 0, 0};
      const bool ok = vf_debug_index_host(p3, param, ix);
      out4[0] = ix[0]; out4[1] = ix[1]; out4[2] = ix[2]; out4[3] = ok ? 1 : 0;
      return SM_OK;
    }
    case 1:     // NDT grid (voxel_grid_covariance_omp_impl.hpp:218-220): int(floor(x * inv) - float(min_b)), per axis
      for (int d = 0; d < 3; ++d) out4[d] = ndt_debug_voxel_coord_host(p3[d], param, min_b);
      out4[3] = 1;
      return SM_OK;
    case 2: {   // ApproximateVoxelGrid: floor(x * inv) per axis and the 512-slot hash
      int ix[3]; uint32_t slot = 0;
      gicp_debug_approx_cell_host(p3, param, ix, &slot);
      out4[0] = ix[0]; out4[1] = ix[1]; out4[2] = ix[2]; out4[3] = (int64_t)slot;
      return SM_OK;
    }
    default: return SM_ERR_BAD_ARGUMENT;
  }
}

// test hook: the per-point arithmetic of the GICP kernels (gicp.cu mahalanobis / cost_terms) compiled for the host
int sm_debug_gicp_point(int32_t op, const double* in, double* out) {
  if (!in || !out) return SM_ERR_BAD_ARGUMENT;
  switch (op) {
    case 0: gicp_debug_mahalanobis_host(in, in + 9, in + 18, out); return SM_OK;   // in = R[9], C1[9], C2[9] row-major
    case 1: {   // in = T[16], base[16] (col-major, cast to float), p_src[3], p_tgt[3] (cast to float), M[9]
      float T[16], base[16], ps[3], pt[3];
      for (int i = 0; i < 16; ++i) { T[i] = (float)in[i]; base[i] = (float)in[16 + i]; }
      for (int i = 0; i < 3; ++i) { ps[i] = (float)in[32 + i]; pt[i] = (float)in[35 + i]; }
      gicp_debug_cost_terms_host(T, base, ps, pt, in + 38, out);
      return SM_OK;
    }
    default: return SM_ERR_BAD_ARGUMENT;
  }
}

// test hook: the host pieces of the GICP stage other than the minimiser (csrc/gicp_host.h), no GPU involved
int sm_debug_gicp_host(int32_t op, const double* in, double* out) {
  if (!in || !out) return SM_ERR_BAD_ARGUMENT;
  switch (op) {
    case 0: {   // applyState (gicp_omp_impl.hpp:516-527): in = T[16] col-major (cast to float), x[6]; out = T'[16]
      float T[16];
      for (int i = 0; i < 16; ++i) T[i] = (float)in[i];
      gicp::apply_state(T, in + 16);
      for (int i = 0; i < 16; ++i) out[i] = (double)T[i];
      return SM_OK;
    }
    case 1:     // computeRDerivative (:133-183): in = x[6], R[9] row-major; out[0..2] = g[3..5]
      { double g[6] = {0, 0, 0, 0, 0, 0}; gicp::r_derivative(in, in + 6, g); out[0] = g[3]; out[1] = g[4]; out[2] = g[5]; }
      return SM_OK;
    default: return SM_ERR_BAD_ARGUMENT;
  }
}

// test hook: the per-match contribution to the point-to-plane normal equations (icp_dev.cuh match_terms /
// add_terms, the functions icp_accum_kernel and icp_finish_kernel call) and the pose-update helpers of
// linalg_dev.cuh, compiled for the HOST
int sm_debug_icp_host(int32_t op, const double* in, int64_t n, double* out) {
  if (!in || !out || n < 0) return SM_ERR_BAD_ARGUMENT;
  switch (op) {
    case 0: {   // in = n records {p[3], q[3], normal[3], d2}; out = the 29 sums, matches added in order
      for (int k = 0; k < dev::kNumSums; ++k) out[k] = 0.0;
      for (int64_t i = 0; i < n; ++i) {
        const double* r = in + 10 * i;
        BucketPoint q; q.x = r[3]; q.y = r[4]; q.z = r[5];
        BucketNormal nn; nn.x = r[6]; nn.y = r[7]; nn.z = r[8];
        double F[6], dot;
        dev::match_terms(r[0], r[1], r[2], q, nn, F, dot);
        dev::add_terms(out, F, dot, r[9]);
      }
      return SM_OK;
    }
    case 1: la::angle_axis_to_rotation(in[0], in + 1, out); return SM_OK;          // out = R[9] row-major
    case 2: la::rotation_to_quaternion(in, out); return SM_OK;                     // in = R[9], out = {w, x, y, z}
    case 3: out[0] = la::quaternion_angular_distance(in, in + 4); return SM_OK;    // in = two quaternions
    case 4: la::mul4(in, in + 16, out); return SM_OK;                              // column-major 4x4 product
    default: return SM_ERR_BAD_ARGUMENT;
  }
}

// test hook: one leaf of the NDT target grid (ndt.cu finish_leaf: covariance, eigen-inflation, inverse) on the host
int sm_debug_ndt_leaf(const float* points_3n, int32_t n, int32_t min_points, double eig_mult, double* mean3,
                      double* icov9, float* centroid3, int32_t* nr_points, int32_t* searchable) {
  if (!points_3n || n <= 0 || !mean3 || !icov9 || !centroid3 || !nr_points || !searchable) return SM_ERR_BAD_ARGUMENT;
  int np = 0, se = 0;
  ndt_debug_leaf_host(points_3n, n, min_points, eig_mult, mean3, icov9, centroid3, &np, &se);
  *nr_points = np; *searchable = se;
  return SM_OK;
}

// test hook: the per-(point, voxel) derivative term of ndt.cu (update_derivatives / update_derivatives_f64, the
// functions ndt_derivatives_kernel calls) compiled for the HOST, with the evaluation parameters built by the
// product's own host code (ndt_host.h) for pose vector p — no GPU involved
int sm_debug_ndt_term(const double* p6, double outlier_ratio, float resolution, int32_t f64_math, const float* x_orig,
                      const float* x_trans, const double* mean3, const double* icov9, double* out43) {
  if (!p6 || !x_orig || !x_trans || !mean3 || !icov9 || !out43) return SM_ERR_BAD_ARGUMENT;
  ndt::Options o;
  o.outlier_ratio = outlier_ratio;
  o.resolution = resolution;
  ndt_debug_term_host(ndt::eval_params(o, f64_math != 0, p6), x_orig, x_trans, mean3, icov9, out43);
  return SM_OK;
}

// test hook (include/sm_b200_debug.h): the scalar host pieces of the NDT Newton loop, no GPU involved
int sm_debug_ndt_host(int32_t op, const double* in, double* out) {
  if (!in || !out) return SM_ERR_BAD_ARGUMENT;
  switch (op) {
    case 0: ndt::svd_solve6(in, in + 36, out); return SM_OK;
    case 1: {
      float T[16];
      ndt::transform_from_p(in, T);
      for (int i = 0; i < 16; ++i) out[i] = (double)T[i];
      return SM_OK;
    }
    case 2: {
      float T[16];
      for (int i = 0; i < 16; ++i) T[i] = (float)in[i];
      ndt::p_from_transform(T, out);
      return SM_OK;
    }
    case 3: {
      ndt::Options o;
      o.outlier_ratio = in[0];
      o.resolution = (float)in[1];
      const NdtEvalParams P = ndt::eval_params(o, false);
      out[0] = P.gauss_d1; out[1] = P.gauss_d2;
      return SM_OK;
    }
    default: return SM_ERR_BAD_ARGUMENT;
  }
}

int sm_debug_bfgs_minimize(sm_debug_fdf fn, void* user, double* x, double grad_tol, int32_t max_iterations,
                           int32_t* iterations, int32_t* evaluations, int32_t* status) {
  if (!fn || !x || !iterations || !evaluations || !status) return SM_ERR_BAD_ARGUMENT;
  int evals = 0;
  gicp::Minimizer mz;
  mz.fdf = [&](const double* xx, double* f, double* g) -> int { ++evals; return fn(xx, f, g, user); };
  mz.init(x);
  int result = gicp::kRunning, inner = 0;
  do {                                   // gicp_omp_impl.hpp:225-240
    ++inner;
    result = mz.one_step(x);
    if (result) break;
    result = mz.test_gradient(grad_tol);
  } while (result == gicp::kRunning && inner < max_iterations);
  *iterations = inner; *evaluations = evals; *status = mz.failed ? gicp::kError : result;
  return SM_OK;
}

// ---- test hooks of the Ndt / NdtWithGicp device stages (include/sm_b200_debug.h) ------------------------------------
// Each runs the product's own launch functions on buffers of its own, on the default stream, with no handle.

// a packed float xyz cloud of n points copied into buf
static int debug_upload_f32(const float* pts, int64_t n, DevBuf& buf) {
  SMB_RC(buf.reserve((size_t)n * 12 + 64));
  SMB_CUDA_OK(cudaMemcpy(buf.p, pts, (size_t)n * 12, cudaMemcpyHostToDevice));
  return SM_OK;
}

static bool debug_cloud_ok(const float* pts, int64_t n) { return pts && n > 0 && n <= (1 << 24); }

// the NDT grid of the target, in a stage sized for ns source points
static int debug_ndt_build(const float* target, int64_t nt, int64_t ns, float resolution, DevBuf& tgt, NdtStage& st,
                           NdtGrid* grid) {
  SMB_RC(debug_upload_f32(target, nt, tgt));
  SMB_RC(st.reserve((int)nt, (int)ns));
  SMB_RC(st.build_grid((const float*)tgt.p, (int)nt, resolution, nullptr));
  SMB_CUDA_OK(cudaMemcpy(grid, st.ws.grid, sizeof(NdtGrid), cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_ndt_grid(int device, const float* target_3n, int64_t n, float resolution, int32_t* n_voxels,
                      int32_t* overflow, int32_t* key, int32_t* nr_points, int32_t* searchable, double* mean_3,
                      double* icov_9, float* centroid_3) {
  if (!debug_cloud_ok(target_3n, n) || !(resolution > 0.0f) || !n_voxels || !overflow || !key || !nr_points ||
      !searchable || !mean_3 || !icov_9 || !centroid_3)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf tgt;
  NdtStage st;
  NdtGrid g;
  SMB_RC(debug_ndt_build(target_3n, n, 1, resolution, tgt, st, &g));
  const int nv = g.n_voxels;
  std::vector<int> keys((size_t)nv);
  std::vector<NdtLeaf> leaves((size_t)nv);
  SMB_CUDA_OK(cudaMemcpy(keys.data(), st.ws.voxel_key, (size_t)nv * sizeof(int), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(leaves.data(), st.ws.leaves, (size_t)nv * sizeof(NdtLeaf), cudaMemcpyDeviceToHost));
  *n_voxels = nv;
  *overflow = g.overflow;
  for (int v = 0; v < nv; ++v) {
    const NdtLeaf& l = leaves[(size_t)v];
    key[v] = keys[(size_t)v]; nr_points[v] = l.nr_points; searchable[v] = l.searchable;
    for (int d = 0; d < 3; ++d) { mean_3[3 * v + d] = l.mean[d]; centroid_3[3 * v + d] = l.centroid[d]; }
    for (int q = 0; q < 9; ++q) icov_9[9 * v + q] = l.icov[q];
  }
  return SM_OK;
}

int sm_debug_ndt_derivatives(int device, const float* target_3n, int64_t nt, const float* source_3n, int64_t ns,
                      float resolution, double outlier_ratio, int32_t f64_math, const double* p_6k, int32_t n_poses,
                      double* sums_44k) {
  if (!debug_cloud_ok(target_3n, nt) || !debug_cloud_ok(source_3n, ns) || !(resolution > 0.0f) || !p_6k ||
      n_poses <= 0 || !sums_44k)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf tgt, src;
  NdtStage st;
  NdtGrid g;
  SMB_RC(debug_ndt_build(target_3n, nt, ns, resolution, tgt, st, &g));
  SMB_RC(debug_upload_f32(source_3n, ns, src));
  ndt::Options o;                      // the evaluation parameters as sm_debug_ndt_term builds them
  o.outlier_ratio = outlier_ratio;
  o.resolution = resolution;
  for (int k = 0; k < n_poses; ++k) {
    SMB_RC(st.eval((const float*)src.p, (int)ns, ndt::eval_params(o, f64_math != 0, p_6k + 6 * k), kNdtKdtree,
                   sums_44k + 44 * (int64_t)k, nullptr));
  }
  return SM_OK;
}

int sm_debug_ndt_derivatives_search(int device, const float* target_3n, int64_t nt, const float* source_3n,
                                    int64_t ns, float resolution, double outlier_ratio, int32_t search_method,
                                    const double* p_6k, int32_t n_poses, double* sums_44k) {
  if (!debug_cloud_ok(target_3n, nt) || !debug_cloud_ok(source_3n, ns) || !(resolution > 0.0f) || !p_6k ||
      n_poses <= 0 || !sums_44k || search_method < SM_NDT_KDTREE || search_method > SM_NDT_DIRECT1)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf tgt, src;
  NdtStage st;
  NdtGrid g;
  SMB_RC(debug_ndt_build(target_3n, nt, ns, resolution, tgt, st, &g));
  SMB_RC(debug_upload_f32(source_3n, ns, src));
  ndt::Options o;
  o.outlier_ratio = outlier_ratio;
  o.resolution = resolution;
  for (int k = 0; k < n_poses; ++k)
    SMB_RC(st.eval((const float*)src.p, (int)ns, ndt::eval_params(o, false, p_6k + 6 * k), search_method,
                   sums_44k + 44 * (int64_t)k, nullptr));
  return SM_OK;
}

// test hook: the direct searches' cell walk and leaf test (ndt.cu for_each_direct_cell, the code the derivative
// kernel runs) compiled for the host, over a caller's grid box and leaves — no GPU involved
int sm_debug_ndt_direct_neighbors(int32_t search_method, const float* points_3n, int64_t n, float resolution,
                                  const int32_t* min_b_3, const int32_t* div_b_3, const int32_t* leaf_key,
                                  const int32_t* leaf_nr_points, int64_t n_leaves, int32_t* counts_n,
                                  int32_t* keys_26n) {
  if (search_method < SM_NDT_DIRECT26 || search_method > SM_NDT_DIRECT1 || !points_3n || n < 0 || !min_b_3 ||
      !div_b_3 || n_leaves < 0 || (n_leaves > 0 && (!leaf_key || !leaf_nr_points)) || !counts_n || !keys_26n)
    return SM_ERR_BAD_ARGUMENT;
  NdtGrid g;
  memset(&g, 0, sizeof(g));
  for (int d = 0; d < 3; ++d) { g.min_b[d] = min_b_3[d]; g.div_b[d] = div_b_3[d]; }
  g.mul[0] = 1; g.mul[1] = g.div_b[0]; g.mul[2] = g.div_b[0] * g.div_b[1];
  std::map<int, int> nr;   // leaf index -> nr_points
  for (int64_t l = 0; l < n_leaves; ++l) nr[leaf_key[l]] = leaf_nr_points[l];
  for (int64_t i = 0; i < n; ++i) {
    int cells[26];
    const int m = ndt_debug_direct_cells_host(search_method, points_3n + 3 * i, resolution, g, cells);
    int k = 0;
    for (int j = 0; j < m; ++j) {
      const auto it = nr.find(cells[j]);
      if (it != nr.end() && ndt_debug_direct_leaf_accepted_host(it->second)) keys_26n[26 * i + k++] = cells[j];
    }
    counts_n[i] = k;
  }
  return SM_OK;
}

int sm_debug_float_tree_knn(int device, const float* cloud_3n, int64_t n, const double* query_3m, int64_t nq,
                            int32_t k, int32_t* ids, double* d2) {
  if (!debug_cloud_ok(cloud_3n, n) || !query_3m || nq <= 0 || nq > (1 << 24) || (k != 1 && k != 20) || !ids || !d2 ||
      kd_num_levels((int)n, 8) > 24)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf cloud, kdws, q, ids_d, d2_d;
  FloatTree t;
  SMB_RC(debug_upload_f32(cloud_3n, n, cloud));
  SMB_RC(t.build((const float*)cloud.p, (int)n, kdws, nullptr));
  SMB_RC(q.reserve((size_t)nq * 3 * sizeof(double)));
  SMB_RC(ids_d.reserve((size_t)nq * k * sizeof(int32_t)));
  SMB_RC(d2_d.reserve((size_t)nq * k * sizeof(double)));
  SMB_CUDA_OK(cudaMemcpy(q.p, query_3m, (size_t)nq * 3 * sizeof(double), cudaMemcpyHostToDevice));
  SMB_RC(float_tree_debug_knn(t, (const double*)q.p, (int)nq, k, (int32_t*)ids_d.p, (double*)d2_d.p, nullptr));
  SMB_CUDA_OK(cudaMemcpy(ids, ids_d.p, (size_t)nq * k * sizeof(int32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(d2, d2_d.p, (size_t)nq * k * sizeof(double), cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_pm_stages(int device, const float* reading_3n, int64_t n, const float* target_3n, int64_t nt, float prob,
                       uint32_t seed, const double* T_4x4, float knn_epsilon, float ratio, int64_t* kept,
                       double* sampled_3n, double* keys_n, double* out_3) {
  if (!debug_cloud_ok(reading_3n, n) || !debug_cloud_ok(target_3n, nt) || !T_4x4 || !kept || !sampled_3n || !keys_n ||
      !out_3 || kd_num_levels((int)nt, 8) > 24)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf src, tgt, kdws;
  PmStage st;
  FloatTree tree;
  SMB_RC(debug_upload_f32(reading_3n, n, src));
  SMB_RC(debug_upload_f32(target_3n, nt, tgt));
  SMB_RC(st.reserve((int)n));
  uint32_t m = 0;
  SMB_RC(st.sample((const float*)src.p, (int)n, prob, seed, nullptr, &m));
  SMB_CUDA_OK(cudaMemcpy(sampled_3n, st.points(), (size_t)m * 3 * sizeof(double), cudaMemcpyDeviceToHost));
  *kept = (int64_t)m;
  SMB_RC(tree.build((const float*)tgt.p, (int)nt, kdws, nullptr));
  double* pinned = nullptr;   // the pose, as score_pass expects it, and the three outputs
  SMB_CUDA_OK(cudaMallocHost((void**)&pinned, 19 * sizeof(double)));
  memcpy(pinned, T_4x4, 16 * sizeof(double));
  const double eps = (double)knn_epsilon;   // as pm_align derives the search's bound from the option
  const int rc = st.score_pass((const float*)src.p, (int)n, pinned, tree, (1.0 + eps) * (1.0 + eps), ratio,
                               pinned + 16, nullptr);
  if (rc == 0) memcpy(out_3, pinned + 16, 3 * sizeof(double));
  cudaFreeHost(pinned);
  SMB_RC(rc);
  SMB_CUDA_OK(cudaMemcpy(keys_n, st.sorted_keys(), (size_t)n * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  return SM_OK;
}

// test hooks: the rand reading sampler's generator (icp_pm.cu) compiled for the host, and its device stage
int sm_debug_pm_rand_window_host(uint32_t seed, int64_t position, uint32_t* window_31) {
  if (position < 0 || !window_31) return SM_ERR_BAD_ARGUMENT;
  const PmRandWindow at = pm_rand_window(seed, (uint64_t)position);
  memcpy(window_31, at.w, sizeof(at.w));
  return SM_OK;
}

int sm_debug_pm_rand_advance_host(const uint32_t* window_31, uint64_t steps, uint32_t* out_31) {
  if (!window_31 || !out_31) return SM_ERR_BAD_ARGUMENT;
  PmRandWindow at;
  memcpy(at.w, window_31, sizeof(at.w));
  pm_rand_debug_advance_host(at, steps);
  memcpy(out_31, at.w, sizeof(at.w));
  return SM_OK;
}

int sm_debug_pm_rand_draws_host(uint32_t seed, int64_t position, int64_t count, int32_t* out) {
  if (position < 0 || count < 0 || (count > 0 && !out)) return SM_ERR_BAD_ARGUMENT;
  pm_rand_debug_draws_host(pm_rand_window(seed, (uint64_t)position), count, out);
  return SM_OK;
}

int sm_debug_pm_rand_sample(int device, const float* reading_3n, int64_t n, float prob, uint32_t seed,
                            int64_t position, int64_t* kept, double* sampled_3n, uint8_t* keep_n) {
  if (!debug_cloud_ok(reading_3n, n) || position < 0 || !kept || !sampled_3n || !keep_n) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf src;
  PmStage st;
  SMB_RC(debug_upload_f32(reading_3n, n, src));
  SMB_RC(st.reserve((int)n));
  const PmRandWindow at = pm_rand_window(seed, (uint64_t)position);
  uint32_t m = 0;
  SMB_RC(st.sample((const float*)src.p, (int)n, prob, seed, nullptr, &m, &at));
  SMB_CUDA_OK(cudaMemcpy(sampled_3n, st.points(), (size_t)m * 3 * sizeof(double), cudaMemcpyDeviceToHost));
  std::vector<uint32_t> bits((size_t)(n + 31) / 32);
  SMB_CUDA_OK(cudaMemcpy(bits.data(), st.rand_bits(), bits.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  for (int64_t i = 0; i < n; ++i) keep_n[i] = (uint8_t)((bits[(size_t)(i >> 5)] >> (i & 31)) & 1u);
  *kept = (int64_t)m;
  return SM_OK;
}

int sm_debug_pm_surface_normals(int device, int32_t mode, const float* first_3n, int64_t n_first, const float* cloud_3n,
                                int64_t n, double* points_3m, double* normals_3m, int64_t* index_m, int64_t* m) {
  if ((mode != kNormalsLeastSquares && mode != kNormalsEigenvector) || !debug_cloud_ok(cloud_3n, n) || n_first < 0 ||
      (n_first > 0 && !debug_cloud_ok(first_3n, n_first)) || !points_3m || !normals_3m || !index_m || !m)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  NormalsPipeline np;
  DevBuf in;
  uint32_t kept = 0;
  for (int pass = n_first > 0 ? 0 : 1; pass < 2; ++pass) {   // as pm_align: widen the float cloud, then run
    const float* c = pass == 0 ? first_3n : cloud_3n;
    const int64_t k = pass == 0 ? n_first : n;
    SMB_RC(np.reserve((int)k));
    SMB_RC(debug_upload_f32(c, k, in));
    SMB_RC(ndt_float_to_soa((const float*)in.p, (int)k, np.input(), np.stride, nullptr));
    SMB_RC(np.run((int)k, (NormalsMode)mode, nullptr, &kept));
  }
  SMB_CUDA_OK(cudaMemcpy(points_3m, np.points(), (size_t)kept * 3 * sizeof(double), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(normals_3m, np.normals(), (size_t)kept * 3 * sizeof(double), cudaMemcpyDeviceToHost));
  std::vector<uint32_t> keep((size_t)n);
  SMB_CUDA_OK(cudaMemcpy(keep.data(), np.keep.p, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  int64_t j = 0;
  for (int64_t i = 0; i < n; ++i)
    if (keep[(size_t)i]) { if (j < (int64_t)kept) index_m[j] = i; ++j; }
  if (j != (int64_t)kept) return SM_ERR_CUDA;   // the compaction's count disagrees with its flags
  *m = (int64_t)kept;
  return SM_OK;
}

int sm_debug_approx_voxel_grid(int device, const float* points_3n, int64_t n, float leaf, float* out_3n,
                               int64_t* m_out) {
  if (!debug_cloud_ok(points_3n, n) || !(leaf > 0.0f) || !out_3n || !m_out) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf pts, out;
  ApproxVoxelGrid filter;
  SMB_RC(debug_upload_f32(points_3n, n, pts));
  int m = 0;
  SMB_RC(filter.filter((const float*)pts.p, (int)n, leaf, out, &m, nullptr));
  SMB_CUDA_OK(cudaMemcpy(out_3n, out.p, (size_t)m * 12, cudaMemcpyDeviceToHost));
  *m_out = (int64_t)m;
  return SM_OK;
}

int sm_debug_gicp_covariances(int device, const float* cloud_3n, int64_t n, double* covs_9n) {
  if (!debug_cloud_ok(cloud_3n, n) || !covs_9n || kd_num_levels((int)n, 8) > 24) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf cloud, kdws;
  gicp::Stage g;                       // the cloud as the stage's source
  SMB_RC(debug_upload_f32(cloud_3n, n, cloud));
  SMB_RC(g.source_tree.build((const float*)cloud.p, (int)n, kdws, nullptr));
  SMB_RC(g.reserve((int)n, (int)n, nullptr));
  SMB_RC(g.covariances(gicp::Options(), (const float*)cloud.p, (int)n, g.source_tree, g.cov_s, nullptr));
  SMB_CUDA_OK(cudaMemcpy(covs_9n, g.cov_s.p, (size_t)n * 9 * sizeof(double), cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_gicp_step(int device, const float* source_3n, int64_t ns, const float* target_3n, int64_t nt,
                       const double* guess_4x4, const double* transformation_4x4, const double* x_6k, int32_t n_states,
                       int32_t* match, double* maha_9n, int32_t* count, double* sums_13k) {
  if (!debug_cloud_ok(source_3n, ns) || !debug_cloud_ok(target_3n, nt) || !guess_4x4 || !transformation_4x4 ||
      !x_6k || n_states <= 0 || !match || !maha_9n || !count || !sums_13k || kd_num_levels((int)ns, 8) > 24 ||
      kd_num_levels((int)nt, 8) > 24)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  const gicp::Options o;
  DevBuf src, tgt, kdws;
  FloatTree tt;
  gicp::Stage g;
  SMB_RC(debug_upload_f32(source_3n, ns, src));
  SMB_RC(debug_upload_f32(target_3n, nt, tgt));
  SMB_RC(tt.build((const float*)tgt.p, (int)nt, kdws, nullptr));
  SMB_RC(g.source_tree.build((const float*)src.p, (int)ns, kdws, nullptr));
  SMB_RC(g.reserve((int)ns, (int)nt, nullptr));
  SMB_RC(g.covariances(o, (const float*)tgt.p, (int)nt, tt, g.cov_t, nullptr));
  SMB_RC(g.covariances(o, (const float*)src.p, (int)ns, g.source_tree, g.cov_s, nullptr));
  float guess[16], transformation[16];
  for (int i = 0; i < 16; ++i) { guess[i] = (float)guess_4x4[i]; transformation[i] = (float)transformation_4x4[i]; }
  double R[9];
  gicp::outer_rotation(transformation, guess, R);
  int m = 0;
  SMB_RC(g.correspond(o, (const float*)src.p, (int)ns, (const float*)tgt.p, tt, guess, transformation, R, nullptr, &m));
  SMB_CUDA_OK(cudaMemcpy(match, g.match.p, (size_t)ns * sizeof(int32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(maha_9n, g.maha.p, (size_t)ns * 9 * sizeof(double), cudaMemcpyDeviceToHost));
  *count = (int32_t)m;
  // the evaluations share one ticket, as the BFGS evaluations of an outer iteration do: each relies on the
  // previous one's last block having reset it
  for (int k = 0; k < n_states; ++k) {
    float T[16];
    for (int i = 0; i < 16; ++i) T[i] = guess[i];
    gicp::apply_state(T, x_6k + 6 * k);
    SMB_RC(g.cost((const float*)src.p, (int)ns, (const float*)tgt.p, T, guess, nullptr, nullptr, nullptr));
    SMB_CUDA_OK(cudaMemcpy(sums_13k + 13 * (int64_t)k, g.sums, 13 * sizeof(double), cudaMemcpyDeviceToHost));
  }
  return SM_OK;
}

// test hook: the host routines of M2DP (m2dp.cu m2dp_axes / m2dp_descriptor), no GPU involved
int sm_debug_m2dp_host(int32_t op, const float* cov_6, const int32_t* A, const double* gram, int32_t rows, int32_t cols,
                       float* out) {
  if (!out) return SM_ERR_BAD_ARGUMENT;
  switch (op) {
    case 0:
      if (!cov_6) return SM_ERR_BAD_ARGUMENT;
      m2dp_axes(cov_6, out);
      return SM_OK;
    case 1:
      if (!A || !gram || rows <= 0 || cols <= 0) return SM_ERR_BAD_ARGUMENT;
      m2dp_descriptor(A, gram, rows, cols, out);
      return SM_OK;
    default: return SM_ERR_BAD_ARGUMENT;
  }
}

// test hook: M2dpStage exactly as sm_m2dp runs it, every intermediate copied out, then m2dp_descriptor
int sm_debug_m2dp_stages(int device, const float* points, int64_t n, int64_t stride_bytes, double r, double max_distance,
                         int32_t t, int32_t p, int32_t q, float* mean_3, double* cov_sums_6, float* cov_6, float* E_9,
                         float* views_6r, int32_t* A, double* gram, float* descriptor) {
  if (!points || n <= 0 || n > (1ll << 30) || stride_bytes < 12 || stride_bytes % 4 || !mean_3 || !cov_sums_6 ||
      !cov_6 || !E_9 || !views_6r || !A || !gram || !descriptor || sm_m2dp_descriptor_length(r, max_distance, t, p, q) < 0)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  M2dpStage st;
  SMB_RC(st.run(points, n, stride_bytes, r, max_distance, t, p, q, nullptr));
  memcpy(mean_3, st.mean, sizeof(st.mean));
  memcpy(cov_sums_6, st.cov_sums, sizeof(st.cov_sums));
  memcpy(cov_6, st.cov, sizeof(st.cov));
  memcpy(E_9, st.E, sizeof(st.E));
  memcpy(views_6r, st.views.data(), st.views.size() * sizeof(M2dpView));
  memcpy(A, st.A.data(), st.A.size() * sizeof(int));
  memcpy(gram, st.G.data(), st.G.size() * sizeof(double));
  m2dp_descriptor(st.A.data(), st.G.data(), st.rows, st.cols, descriptor);
  return SM_OK;
}

// ---- test hooks of the shared build stages: the radix sort and the k-d tree owners ----------------------------------
int sm_debug_radix_sort(int device, const uint64_t* keys, const uint32_t* vals, int64_t n, int32_t batch, int64_t stride,
                        int32_t passes, uint64_t* keys_out, uint32_t* vals_out) {
  if (!keys || !vals || !keys_out || !vals_out || n <= 0 || n > (1 << 30) || batch < 1 || batch > 16 || stride < n ||
      stride > (1 << 30) || passes < 1 || passes > 8)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  const size_t words = (size_t)batch * (size_t)stride;
  DevBuf k, v, scratch;
  SMB_RC(k.reserve(2 * words * sizeof(uint64_t)));
  SMB_RC(v.reserve(2 * words * sizeof(uint32_t)));
  SMB_RC(scratch.reserve(radix_sort_scratch_bytes((int)n, batch)));
  uint64_t* ka = (uint64_t*)k.p;
  uint32_t* va = (uint32_t*)v.p;
  for (int h = 0; h < 2; ++h) {   // both ping-pong halves start as the caller's arrays, the padding past n included
    SMB_CUDA_OK(cudaMemcpy(ka + h * words, keys, words * sizeof(uint64_t), cudaMemcpyHostToDevice));
    SMB_CUDA_OK(cudaMemcpy(va + h * words, vals, words * sizeof(uint32_t), cudaMemcpyHostToDevice));
  }
  SMB_RC(radix_sort_pairs_u64(ka, va, ka + words, va + words, (int)n, batch, stride, (uint32_t*)scratch.p, nullptr,
                              passes));
  const size_t res = passes % 2 == 0 ? 0 : words;   // an odd number of passes ends in the second half
  SMB_CUDA_OK(cudaMemcpy(keys_out, ka + res, words * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(vals_out, va + res, words * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  return SM_OK;
}

// n AoS double points -> SoA [3][stride] doubles at dev
static int debug_soa(const double* aos, int64_t n, int64_t stride, double* dev) {
  std::vector<double> soa((size_t)(3 * stride), 0.0);
  for (int64_t i = 0; i < n; ++i)
    for (int d = 0; d < 3; ++d) soa[(size_t)(d * stride + i)] = aos[3 * i + d];
  SMB_CUDA_OK(cudaMemcpy(dev, soa.data(), soa.size() * sizeof(double), cudaMemcpyHostToDevice));
  return SM_OK;
}

namespace {
// the owners of the four tree variants, and the buffers that outlive one build in a handle
struct DebugKdOwners {
  KdCompactTree tree;
  NormalsPipeline np;
  FloatTree ft;
  DevBuf coord, nrm, kdws;
};
}  // namespace

// one build of `cloud` into the owner of `variant`, as sm_align / sm_knn1 / sm_calculate_normals run it
static int debug_kd_build(DebugKdOwners& o, int variant, int bucket, const void* cloud, const double* normals,
                          int64_t n) {
  const int64_t stride = (n + 63) & ~(int64_t)63;
  if (variant <= 1) {
    SMB_RC(o.coord.reserve((size_t)(3 * stride) * sizeof(double)));
    SMB_RC(debug_soa((const double*)cloud, n, stride, (double*)o.coord.p));
    if (variant == 0) {
      SMB_RC(o.nrm.reserve((size_t)(3 * stride) * sizeof(double)));
      SMB_RC(debug_soa(normals, n, stride, (double*)o.nrm.p));
    }
    SMB_RC(o.tree.reserve((int)n, bucket, variant == 0 ? KdCompactTree::kNormals : KdCompactTree::kIds));
    KdWorkspace ws;
    SMB_RC(ws.carve(o.kdws, (int)n, bucket));
    SMB_RC(o.tree.build((const double*)o.coord.p, variant == 0 ? (const double*)o.nrm.p : nullptr, stride, (int)n,
                        bucket, ws, nullptr));
  } else if (variant == 2) {
    SMB_RC(o.np.reserve((int)n));
    SMB_RC(debug_soa((const double*)cloud, n, o.np.stride, o.np.input()));
    uint32_t m = 0;
    SMB_RC(o.np.run((int)n, kNormalsLeastSquares, nullptr, &m));
  } else {
    SMB_RC(debug_upload_f32((const float*)cloud, n, o.coord));
    SMB_RC(o.ft.build((const float*)o.coord.p, (int)n, o.kdws, nullptr));
  }
  SMB_CUDA_OK(cudaDeviceSynchronize());
  return SM_OK;
}

int sm_debug_kd_tree(int device, int32_t variant, int32_t bucket, const void* first_3n, const double* first_normals_3n,
                     int64_t n_first, const void* cloud_3n, const double* normals_3n, int64_t n, int32_t levels,
                     void* nodes, uint32_t* order, double* cut, uint8_t* dim, double* node_2l, double* pb, double* pn,
                     int32_t* pid, void* bpts) {
  if (variant < 0 || variant > 3 || !cloud_3n || n <= 0 || n > (1 << 30) || n_first < 0 || n_first > (1 << 30) ||
      (n_first > 0 && !first_3n) || !nodes || !order)
    return SM_ERR_BAD_ARGUMENT;
  if (variant <= 1 && (bucket < 2 || bucket > 8 || !cut || !dim || !node_2l || !pb)) return SM_ERR_BAD_ARGUMENT;
  if (variant == 0 && (!normals_3n || !pn || (n_first > 0 && !first_normals_3n))) return SM_ERR_BAD_ARGUMENT;
  if (variant == 1 && !pid) return SM_ERR_BAD_ARGUMENT;
  if ((variant == 2 && bucket != 7) || (variant == 3 && (bucket != 8 || !bpts))) return SM_ERR_BAD_ARGUMENT;
  const int lv = kd_num_levels((int)n, bucket);
  if (lv != levels || lv > 24 || (n_first > 0 && kd_num_levels((int)n_first, bucket) > 24)) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DebugKdOwners o;
  if (n_first > 0) SMB_RC(debug_kd_build(o, variant, bucket, first_3n, first_normals_3n, n_first));
  SMB_RC(debug_kd_build(o, variant, bucket, cloud_3n, normals_3n, n));
  const DevBuf& nd = variant <= 1 ? o.tree.nodes : variant == 2 ? o.np.nodes : o.ft.nodes;
  const DevBuf& od = variant <= 1 ? o.tree.leaf_order : variant == 2 ? o.np.order : o.ft.order;
  SMB_CUDA_OK(cudaMemcpy(nodes, nd.p, (size_t)blocked_node_slots(lv) * sizeof(KdNode), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(order, od.p, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (variant <= 1) {
    const KdCompact kc = o.tree.view();
    const size_t inner = ((size_t)1 << lv) - 1, entries = (size_t)8 << lv;
    if (kc.levels != lv) return SM_ERR_BAD_ARGUMENT;
    SMB_CUDA_OK(cudaMemcpy(cut, kc.cut, inner * sizeof(double), cudaMemcpyDeviceToHost));
    SMB_CUDA_OK(cudaMemcpy(dim, kc.dim, inner, cudaMemcpyDeviceToHost));
    SMB_CUDA_OK(cudaMemcpy(node_2l, kc.node, (inner + 1) * sizeof(double2), cudaMemcpyDeviceToHost));
    SMB_CUDA_OK(cudaMemcpy(pb, kc.pb, entries * 3 * sizeof(double), cudaMemcpyDeviceToHost));
    // pn[e] = {nx, ny, nz, 0}: the normal half of the 64-byte record, pad included
    if (variant == 0)
      SMB_CUDA_OK(cudaMemcpy2D(pn, sizeof(BucketNormal), (const char*)kc.pm + offsetof(BucketMatch, nx),
                               sizeof(BucketMatch), sizeof(BucketNormal), entries, cudaMemcpyDeviceToHost));
    else SMB_CUDA_OK(cudaMemcpy(pid, kc.pid, entries * sizeof(int32_t), cudaMemcpyDeviceToHost));
  } else if (variant == 3) {
    SMB_CUDA_OK(cudaMemcpy(bpts, o.ft.bpts.p, (size_t)n * sizeof(BucketPoint), cudaMemcpyDeviceToHost));
  }
  return SM_OK;
}

// ---- test hook of IcpFast's iteration (icp.cu, icp_finish.cu) -------------------------------------------------------
// caller index of the target point in padded bucket entry e of a bucket-8 normals tree (kd_compact_buckets_kernel's
// walk from the root to the leaf that owns the entry)
static int32_t debug_entry_target(const std::vector<uint32_t>& leaf_order, int n, int levels, int64_t e) {
  const int jL = (int)(e >> 3), k = (int)(e & 7);
  int first = 0, count = n, l = 0;
  while (l < levels && count > 8) {
    const int right = count >> 1, left = count - right;
    if ((jL >> (levels - 1 - l)) & 1) { first += left; count = right; } else { count = left; }
    ++l;
  }
  return k < count ? (int32_t)leaf_order[first + k] : -1;
}

static int debug_copy_out(void* dst, const void* src, size_t bytes) {
  if (dst) SMB_CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_icp_iteration_minimizer(int device, const double* source_3n, int64_t ns, const double* target_3n,
                                     const double* normals_3n, int64_t nt, const double* guess_4x4,
                                     float dist_outlier_ratio, float knn_epsilon, int32_t knn_queries_per_cta,
                                     int32_t inner_compensation, int32_t error_minimizer, int32_t iteration,
                                     int32_t* geometry_2, double* prologue_35, uint32_t* perm_n, int32_t* match_n,
                                     double* d2_n, double* pm_6n, uint32_t* hist_2048, uint32_t* hist2_2048,
                                     uint32_t* cand_cnt, uint64_t* cand_key, double* cand_terms_8, double* partials_29,
                                     double* sums_29, double* final_18, int64_t* final_5, uint32_t* hist_after_4096) {
  if (!geometry_2 || ns <= 0 || ns > (1 << 30)) return SM_ERR_BAD_ARGUMENT;
  if (error_minimizer < SM_ICP_POINT_TO_PLANE || error_minimizer > SM_ICP_POINT_TO_POINT) return SM_ERR_BAD_ARGUMENT;
  const int nb = icp_accum_blocks((int)ns);
  geometry_2[0] = nb; geometry_2[1] = dev::kAccTile;
  if (!source_3n) return SM_OK;
  if (!target_3n || !normals_3n || nt <= 0 || nt > (1 << 30) || kd_num_levels((int)nt, 8) > 24 || !guess_4x4 ||
      iteration < 1 || !(dist_outlier_ratio >= 0.0f && dist_outlier_ratio <= 1.0f) || !(knn_epsilon >= 0.0f) ||
      knn_queries_per_cta < 0)
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  // the owners and the parameters of icp_begin, without graphs
  const int64_t sstride = (ns + 63) & ~(int64_t)63, tstride = (nt + 63) & ~(int64_t)63;
  const bool comp = inner_compensation != 0;
  IcpFastBuffers f;
  DevBuf src_raw, tgt_raw, nrm, kdws;
  SMB_RC(f.reserve((int)ns, (int)nt, sstride, tstride, comp));
  SMB_RC(src_raw.reserve((size_t)(3 * sstride) * sizeof(double)));
  SMB_RC(tgt_raw.reserve((size_t)(3 * tstride) * sizeof(double)));
  SMB_RC(nrm.reserve((size_t)(3 * tstride) * sizeof(double)));
  SMB_RC(debug_soa(source_3n, ns, sstride, (double*)src_raw.p));
  SMB_RC(debug_soa(target_3n, nt, tstride, (double*)tgt_raw.p));
  SMB_RC(debug_soa(normals_3n, nt, tstride, (double*)nrm.p));
  KdWorkspace ws;
  SMB_RC(ws.carve(kdws, (int)nt, 8));
  IcpBuffers b;
  f.fill(b, (const double*)tgt_raw.p, (const double*)nrm.p, (const double*)src_raw.p);
  IcpParams p = {};
  p.n_source = (int)ns; p.n_target = (int)nt;
  p.max_iteration = iteration;
  p.dist_outlier_ratio = dist_outlier_ratio;
  p.max_error2 = (1.0 + (double)knn_epsilon) * (1.0 + (double)knn_epsilon);
  p.disable_convergence = 1;
  p.knn_queries_per_cta = knn_queries_per_cta;
  p.tree_levels = kd_num_levels((int)nt, 8);
  p.inner_compensation = comp ? 1 : 0;
  p.error_minimizer = (int16_t)error_minimizer;
  double* deskewed = comp ? (double*)f.deskewed.p : nullptr;
  SMB_CUDA_OK(cudaMemcpy(f.guess.p, guess_4x4, 16 * sizeof(double), cudaMemcpyHostToDevice));
  SMB_CUDA_OK(cudaMemset(b.sums, 0xff, dev::kNumSums * sizeof(double)));   // all-ones until phase C writes it
  SMB_RC(icp_prologue(b, p, (const double*)f.guess.p, ws, f.tree, nullptr));
  if (iteration > 1) SMB_RC(icp_enqueue_iterations(b, p, 0, iteration - 1, nullptr, nullptr, deskewed));
  SMB_CUDA_OK(cudaDeviceSynchronize());
  IcpState st;
  SMB_CUDA_OK(cudaMemcpy(&st, b.state, sizeof(IcpState), cudaMemcpyDeviceToHost));
  std::vector<uint32_t> perm((size_t)ns);
  SMB_CUDA_OK(cudaMemcpy(perm.data(), b.src_sort.vals[0], (size_t)ns * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  if (prologue_35) {
    memcpy(prologue_35, st.mean, 3 * sizeof(double));
    memcpy(prologue_35 + 3, st.G0, 16 * sizeof(double));
    memcpy(prologue_35 + 19, st.T_iter, 16 * sizeof(double));
  }
  if (perm_n) memcpy(perm_n, perm.data(), (size_t)ns * sizeof(uint32_t));
  // phase A, per source point in caller order
  if (comp) icp_deskew_launch(b, p, deskewed, nullptr);
  icp_search_launch(b, p, deskewed, nullptr);
  SMB_CUDA_OK(cudaDeviceSynchronize());
  {
    std::vector<int32_t> slot((size_t)ns);
    std::vector<double> d2((size_t)ns);
    std::vector<uint32_t> leaf_order((size_t)nt);
    const int64_t entries = (int64_t)8 << f.tree.levels;
    std::vector<BucketMatch> pm((size_t)entries);
    SMB_CUDA_OK(cudaMemcpy(slot.data(), b.slot, (size_t)ns * sizeof(int32_t), cudaMemcpyDeviceToHost));
    SMB_CUDA_OK(cudaMemcpy(d2.data(), b.d2, (size_t)ns * sizeof(double), cudaMemcpyDeviceToHost));
    SMB_CUDA_OK(cudaMemcpy(leaf_order.data(), f.tree.leaf_order.p, (size_t)nt * sizeof(uint32_t), cudaMemcpyDeviceToHost));
    SMB_CUDA_OK(cudaMemcpy(pm.data(), b.kc.pm, (size_t)entries * sizeof(BucketMatch), cudaMemcpyDeviceToHost));
    for (int64_t i = 0; i < ns; ++i) {
      const uint32_t c = perm[(size_t)i];
      const int32_t s = slot[(size_t)i];
      const bool ok = s >= 0 && s < entries;
      if (match_n) match_n[c] = ok ? debug_entry_target(leaf_order, (int)nt, f.tree.levels, s) : -1;
      if (d2_n) d2_n[c] = d2[(size_t)i];
      if (pm_6n) {
        const BucketMatch r = ok ? pm[(size_t)s] : BucketMatch{};
        const double v[6] = {r.x, r.y, r.z, r.nx, r.ny, r.nz};
        memcpy(pm_6n + 6 * c, v, sizeof(v));
      }
    }
  }
  SMB_RC(debug_copy_out(hist_2048, b.hist, kHistBins * sizeof(uint32_t)));
  // phase B, per block of Morton positions
  icp_accum_launch(b, p, deskewed, nullptr);
  SMB_CUDA_OK(cudaDeviceSynchronize());
  SMB_RC(debug_copy_out(hist2_2048, b.hist2, kHistBins * sizeof(uint32_t)));
  SMB_RC(debug_copy_out(cand_cnt, b.cand_cnt, (size_t)nb * sizeof(uint32_t)));
  SMB_RC(debug_copy_out(cand_key, b.cand_key, (size_t)nb * dev::kAccTile * sizeof(uint64_t)));
  SMB_RC(debug_copy_out(cand_terms_8, b.cand_terms, (size_t)nb * dev::kAccTile * 8 * sizeof(double)));
  if (partials_29)
    SMB_CUDA_OK(cudaMemcpy2D(partials_29, dev::kNumSums * sizeof(double), b.partials, 32 * sizeof(double),
                             dev::kNumSums * sizeof(double), nb, cudaMemcpyDeviceToHost));
  // phase C
  icp_finish_launch(b, p, nb, nullptr);
  SMB_CUDA_OK(cudaDeviceSynchronize());
  SMB_RC(debug_copy_out(sums_29, b.sums, dev::kNumSums * sizeof(double)));
  SMB_RC(debug_copy_out(hist_after_4096, b.hist, 2 * kHistBins * sizeof(uint32_t)));
  SMB_CUDA_OK(cudaMemcpy(&st, b.state, sizeof(IcpState), cudaMemcpyDeviceToHost));
  if (final_18) {
    final_18[0] = st.limit; final_18[1] = st.final_score;
    memcpy(final_18 + 2, st.T_iter, 16 * sizeof(double));
  }
  if (final_5) {
    final_5[0] = st.kept; final_5[1] = st.status; final_5[2] = st.solve_path; final_5[3] = st.iteration;
    final_5[4] = st.done;
  }
  return SM_OK;
}

int sm_debug_icp_iteration(int device, const double* source_3n, int64_t ns, const double* target_3n,
                           const double* normals_3n, int64_t nt, const double* guess_4x4, float dist_outlier_ratio,
                           float knn_epsilon, int32_t knn_queries_per_cta, int32_t inner_compensation, int32_t iteration,
                           int32_t* geometry_2, double* prologue_35, uint32_t* perm_n, int32_t* match_n, double* d2_n,
                           double* pm_6n, uint32_t* hist_2048, uint32_t* hist2_2048, uint32_t* cand_cnt, uint64_t* cand_key,
                           double* cand_terms_8, double* partials_29, double* sums_29, double* final_18, int64_t* final_5,
                           uint32_t* hist_after_4096) {
  return sm_debug_icp_iteration_minimizer(device, source_3n, ns, target_3n, normals_3n, nt, guess_4x4,
                                          dist_outlier_ratio, knn_epsilon, knn_queries_per_cta, inner_compensation,
                                          SM_ICP_POINT_TO_PLANE, iteration, geometry_2, prologue_35, perm_n, match_n,
                                          d2_n, pm_6n, hist_2048, hist2_2048, cand_cnt, cand_key, cand_terms_8,
                                          partials_29, sums_29, final_18, final_5, hist_after_4096);
}

// ---- test hooks of the filter chain (filters.cu) ---------------------------------------------------------------------
int sm_debug_filter_host(const sm_filter_chain* chain, int32_t filter, int32_t op, const float* records, int64_t n,
                         int32_t* iout, float* fout) {
  const FilterChain* fc = filter_chain_of(chain);
  if (!fc || filter < 0 || filter >= (int)fc->filters.size() || !records || !iout || n < 0) return SM_ERR_BAD_ARGUMENT;
  const FilterParams& f = fc->filters[filter];
  for (int64_t i = 0; i < n; ++i) {
    const float* p = records + 5 * i;
    switch (op) {
      case 0: iout[i] = filter_debug_keep_host(f, p, (uint32_t)i, fc->sample_seed) ? 1 : 0; break;
      case 1: if (!filter_debug_pixel_host(f, p, &iout[2 * i], &iout[2 * i + 1])) iout[2 * i] = iout[2 * i + 1] = -1; break;
      case 2:
        if (!fout) return SM_ERR_BAD_ARGUMENT;
        filter_debug_cell_host(f, p, &fout[i], &iout[2 * i], &iout[2 * i + 1]);
        break;
      default: return SM_ERR_BAD_ARGUMENT;
    }
  }
  return SM_OK;
}

int sm_debug_filter_fit_host(const float* d, const float* z, int32_t n, float* m_b) {
  if (!d || !z || !m_b || n < 2) return SM_ERR_BAD_ARGUMENT;
  filter_debug_fit_host(d, z, n, &m_b[0], &m_b[1]);
  return SM_OK;
}

int sm_debug_filter_distance_host(const float* lines_4l, int32_t n_lines, float d, float z, float* distance) {
  if ((n_lines > 0 && !lines_4l) || n_lines < 0 || !distance) return SM_ERR_BAD_ARGUMENT;
  int bad = 0;
  *distance = filter_debug_distance_host((const Gr2Line*)lines_4l, n_lines, d, z, &bad);
  return bad ? SM_ERR_CHECK_FAILED : SM_OK;
}

int sm_debug_mt19937_words_host(uint32_t seed, int64_t count, uint32_t* out) {
  if (count < 0 || (count > 0 && !out)) return SM_ERR_BAD_ARGUMENT;
  mt19937_debug_words_host(seed, count, out);
  return SM_OK;
}

int sm_debug_filter_mt19937_flags(int device, int64_t n, float rate, uint32_t seed, uint8_t* keep_n, int64_t* kept) {
  if (n < 0 || n > (1 << 30) || (n > 0 && !keep_n) || !kept) return SM_ERR_BAD_ARGUMENT;
  *kept = 0;
  if (n == 0) return SM_OK;
  SMB_RC(select_device(device));
  FilterParams f = filter_defaults(kFilterRandomSampler);
  f.sampling_rate = rate;
  f.sampler_mode = SM_FILTER_SAMPLER_MT19937;
  f.sampler_seed = seed;
  DevBuf flag, tile_cnt;
  SMB_RC(flag.reserve((size_t)n));
  SMB_RC(tile_cnt.reserve(compact_count_bytes(n)));
  SMB_RC(mt19937_sampler_flags(f, (int)n, (uint8_t*)flag.p, (uint32_t*)tile_cnt.p, nullptr));
  std::vector<uint32_t> cnt(compact_count_bytes(n) / sizeof(uint32_t));
  SMB_CUDA_OK(cudaMemcpy(keep_n, flag.p, (size_t)n, cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(cnt.data(), tile_cnt.p, cnt.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  for (uint32_t c : cnt) *kept += c;      // the tile counts the compaction reads, the last slot 0
  return SM_OK;
}

int sm_debug_filter_ground_removal2(int device, const sm_filter_chain* chain, int32_t filter, const float* points,
                                    int64_t n, int64_t stride_bytes, int32_t max_lines, uint32_t* cell, uint8_t* member,
                                    uint32_t* cell_members, float* cell_min_2c, float* lines_4, int32_t* n_lines,
                                    uint8_t* keep) {
  const FilterChain* fc = filter_chain_of(chain);
  if (!fc || filter < 0 || filter >= (int)fc->filters.size() || fc->filters[filter].kind != kFilterGroundRemoval2 ||
      !points || n <= 0 || n > (1 << 30) || stride_bytes < 20 || stride_bytes % 4 || !cell || !member ||
      !cell_members || !cell_min_2c || !lines_4 || !n_lines || !keep)
    return SM_ERR_BAD_ARGUMENT;
  const FilterParams& f = fc->filters[filter];
  if (f.bin_num <= 0 || max_lines != f.bin_num / 2 + 1) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  FilterChain one;
  one.filters.push_back(f);
  DevBuf in, out;
  SMB_RC(in.reserve((size_t)n * (size_t)stride_bytes));
  SMB_RC(out.reserve((size_t)n * 20));
  SMB_CUDA_OK(cudaMemcpy(in.p, points, (size_t)n * (size_t)stride_bytes, cudaMemcpyHostToDevice));
  int64_t m = 0;
  const int rc = one.run((const char*)in.p, n, stride_bytes, (float*)out.p, nullptr, &m, nullptr);
  if (rc < 0 && rc != SM_ERR_CHECK_FAILED) return rc;
  const size_t cells = (size_t)f.bin_num * (size_t)f.segment_num;
  SMB_CUDA_OK(cudaMemcpy(cell, one.gr2.cell_of, (size_t)n * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(member, one.gr2.member, (size_t)n, cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(cell_members, one.gr2.cell_cnt, cells * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(cell_min_2c, one.gr2.cell_min, cells * sizeof(float2), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(lines_4, one.gr2.lines, (size_t)f.segment_num * max_lines * sizeof(Gr2Line), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(n_lines, one.gr2.n_lines, (size_t)f.segment_num * sizeof(int), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(keep, one.gr2.keep, (size_t)n, cudaMemcpyDeviceToHost));
  return rc;
}

// ---- test hooks of DepthCluster (depth_cluster.cu) -------------------------------------------------------------------
int sm_debug_depth_edge_host(const sm_filter_chain* chain, int32_t filter, const float* a, const float* b,
                             const int32_t* step, int64_t n, uint8_t* edge, float* beta, float* sin_cos4) {
  const FilterChain* fc = filter_chain_of(chain);
  if (!fc || filter < 0 || filter >= (int)fc->filters.size() || fc->filters[filter].kind != kFilterRangeImage ||
      n < 0 || (n > 0 && (!a || !b || !step || !edge || !beta)))
    return SM_ERR_BAD_ARGUMENT;
  const DepthConsts c = depth_consts(fc->filters[filter]);
  for (int64_t i = 0; i < n; ++i) {
    if (step[i] < 0 || step[i] > 5) return SM_ERR_BAD_ARGUMENT;
    edge[i] = depth_debug_edge_host(c, a[i], b[i], step[i], &beta[i]) ? 1 : 0;
  }
  if (sin_cos4) { sin_cos4[0] = c.sin_h; sin_cos4[1] = c.cos_h; sin_cos4[2] = c.sin_v; sin_cos4[3] = c.cos_v; }
  return SM_OK;
}

int sm_debug_depth_cluster(int device, const sm_filter_chain* chain, int32_t filter, const float* points, int64_t n,
                           int64_t stride_bytes, float* image, int32_t* owner, uint8_t* mask, uint32_t* label,
                           int32_t* level, int32_t* seq, int32_t* components) {
  const FilterChain* fc = filter_chain_of(chain);
  if (!fc || filter < 0 || filter >= (int)fc->filters.size() || fc->filters[filter].kind != kFilterRangeImage ||
      n < 0 || n > (1 << 30) || stride_bytes < 20 || stride_bytes % 4 || !image || !owner || !mask || !label ||
      !level || !seq || !components)
    return SM_ERR_BAD_ARGUMENT;
  if (n == 0) return SM_ERR_CHECK_FAILED;   // before the points: an empty cloud may come without them
  if (!points) return SM_ERR_BAD_ARGUMENT;
  const FilterParams& f = fc->filters[filter];
  if (!depth_cluster_grid_ok(f)) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DepthCluster dc;
  DevBuf in;
  SMB_RC(in.reserve((size_t)n * (size_t)stride_bytes));
  SMB_CUDA_OK(cudaMemcpy(in.p, points, (size_t)n * (size_t)stride_bytes, cudaMemcpyHostToDevice));
  int64_t m = 0;
  SMB_RC(dc.run(f, (const char*)in.p, (int)n, stride_bytes, nullptr, nullptr, nullptr, nullptr, &m, nullptr));
  const size_t P = (size_t)f.vertical_line_num * (size_t)f.horizontal_line_num;
  SMB_CUDA_OK(cudaMemcpy(image, dc.image.p, P * sizeof(float), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(owner, dc.owner.p, P * sizeof(int32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(mask, dc.mask.p, P, cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(label, dc.label.p, P * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(level, dc.level.p, P * sizeof(int32_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(seq, dc.seq.p, P * sizeof(int32_t), cudaMemcpyDeviceToHost));
  for (size_t p = 0; p < P; ++p) if (level[p] < 0) seq[p] = -1;   // seq is written for the visited pixels only
  *components = dc.components;
  return SM_OK;
}

// test hook: one CTA's std::nth_element on one key array (nth_element.cu block_introselect)
int sm_debug_nth_element(int device, const double* keys_n, int64_t n, int64_t nth, int32_t* perm_n) {
  if (!keys_n || !perm_n || n <= 0 || n > (1 << 24) || nth < 0 || nth > n) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf keys, perm, key, lpos, rpos;
  SMB_RC(keys.reserve((size_t)n * sizeof(double)));
  SMB_RC(key.reserve((size_t)n * sizeof(double)));
  SMB_RC(perm.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(lpos.reserve((size_t)n * sizeof(uint32_t)));
  SMB_RC(rpos.reserve((size_t)n * sizeof(uint32_t)));
  SMB_CUDA_OK(cudaMemcpy(keys.p, keys_n, (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
  SMB_RC(nth_element_single((const double*)keys.p, (int)n, (int)nth, (uint32_t*)perm.p, (double*)key.p,
                            (uint32_t*)lpos.p, (uint32_t*)rpos.p, nullptr));
  SMB_CUDA_OK(cudaMemcpy(perm_n, perm.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return SM_OK;
}

// test hook: the recursion's index array of sm_calculate_normals_ordered(SM_NORMALS_ORDER_NTH_ELEMENT)
int sm_debug_normals_nth_perm(int device, const double* points_3n, int64_t n, int32_t* perm_n) {
  if (!points_3n || !perm_n || n <= 0 || n > (1 << 30)) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  NormalsPipeline np;
  SMB_RC(np.reserve((int)n));
  std::vector<double> soa((size_t)n);
  for (int d = 0; d < 3; ++d) {
    for (int64_t i = 0; i < n; ++i) soa[(size_t)i] = points_3n[3 * i + d];
    SMB_CUDA_OK(cudaMemcpy(np.input() + d * np.stride, soa.data(), (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
  }
  uint32_t m = 0;
  SMB_RC(np.run_nth_element((int)n, nullptr, &m));
  SMB_CUDA_OK(cudaMemcpy(perm_n, np.perm.p, (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return SM_OK;
}

int sm_debug_voxel_bucket_counts_host(int64_t m, uint64_t* out_m) {
  if (m < 0 || m > (1 << 30) || (m > 0 && !out_m)) return SM_ERR_BAD_ARGUMENT;
  const std::vector<std::pair<int64_t, uint64_t>> epochs = unordered_map_epochs(m);
  for (size_t e = 0; e < epochs.size(); ++e) {
    const int64_t end = e + 1 < epochs.size() ? epochs[e + 1].first : m;
    for (int64_t k = epochs[e].first; k < end; ++k) out_m[k] = epochs[e].second;
  }
  return SM_OK;
}

int sm_debug_voxel_hash_host(const int32_t* keys_3n, int64_t n, uint64_t* out_n) {
  if (n < 0 || (n > 0 && (!keys_3n || !out_n))) return SM_ERR_BAD_ARGUMENT;
  for (int64_t i = 0; i < n; ++i) out_n[i] = vf_debug_hash_host(keys_3n + 3 * i);
  return SM_OK;
}

// test hook: VoxelGrid::run in SM_VOXEL_ORDER_UNORDERED_MAP with its per-epoch positions
int sm_debug_voxel_unordered_epochs(int device, const float* points, int64_t n, int64_t stride_bytes,
                                    float voxel_size, uint64_t* hash_m, int32_t* rank_m, int32_t* pos,
                                    int64_t capacity, int64_t* m_out, int32_t* n_epochs) {
  if (!points || !hash_m || !rank_m || !m_out || !n_epochs || n <= 0 || n > (1 << 30) || stride_bytes < 16 ||
      stride_bytes % 4 || !(voxel_size > 1.e-6f) || capacity < 0 || (capacity > 0 && !pos))
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf d_in, d_out;
  SMB_RC(d_in.reserve((size_t)n * (size_t)stride_bytes));
  SMB_RC(d_out.reserve((size_t)n * 20));
  SMB_CUDA_OK(cudaMemcpy(d_in.p, points, (size_t)n * (size_t)stride_bytes, cudaMemcpyHostToDevice));
  VoxelGrid vg;
  std::vector<std::vector<uint32_t>> trace;
  vg.epoch_trace = &trace;
  int64_t m = 0;
  SMB_RC(vg.run((const char*)d_in.p, n, stride_bytes, voxel_size, SM_VOXEL_ORDER_UNORDERED_MAP, nullptr,
                (float*)d_out.p, nullptr, &m, nullptr));
  *m_out = m;
  *n_epochs = (int32_t)trace.size();
  if (m == 0) return SM_OK;
  std::vector<uint64_t> hash((size_t)m);
  std::vector<uint32_t> asc((size_t)m);
  SMB_CUDA_OK(cudaMemcpy(hash.data(), vg.hash(), (size_t)m * sizeof(uint64_t), cudaMemcpyDeviceToHost));
  SMB_CUDA_OK(cudaMemcpy(asc.data(), vg.asc(), (size_t)m * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  for (int64_t t = 0; t < m; ++t) { hash_m[asc[t]] = hash[t]; rank_m[asc[t]] = (int32_t)t; }
  if (capacity < m * (int64_t)trace.size()) return SM_ERR_BAD_ARGUMENT;
  for (size_t e = 0; e < trace.size(); ++e)
    for (int64_t t = 0; t < m; ++t) pos[e * m + t] = t < (int64_t)trace[e].size() ? (int32_t)trace[e][t] : -1;
  return SM_OK;
}

}  // extern "C"
