// Host side of registrator::NdtWithGicp's GICP stage: the BFGS minimiser PCL uses
// (pcl/registration/bfgs.h, a port of GSL's vector_bfgs2 + the Fletcher line search of
// multimin/linear_minimize.c; parameters set at gicp_omp_impl.hpp:218-224), applyState
// (:516-527), computeRDerivative (:133-183).  The cost / gradient sums come from gicp.cu.
#ifndef SM_B200_GICP_HOST_H_
#define SM_B200_GICP_HOST_H_

#include <math.h>

#include <algorithm>
#include <functional>
#include <limits>

#include "ndt_host.h"

namespace smb {
namespace gicp {

struct Options {                       // gicp_omp.h:108-118 with the overrides of ndt_gicp.cc:50-51
  int k_correspondences = 20;
  double gicp_epsilon = 0.001;
  double rotation_epsilon = 1e-3;
  double transformation_epsilon = 5e-4;
  double corr_dist_threshold = 5.0;
  int max_iterations = 35;
  int max_inner_iterations = 20;
};

inline void apply_state(float* t, const double* x) {   // t: column-major 4x4
  float Rx[9], Ry[9], Rz[9], Rzy[9], R[9], old[9], neu[9];
  ndt::axis_rotation((float)x[3], 0, Rx);
  ndt::axis_rotation((float)x[4], 1, Ry);
  ndt::axis_rotation((float)x[5], 2, Rz);
  ndt::mul3(Rz, Ry, Rzy);
  ndt::mul3(Rzy, Rx, R);
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) old[r * 3 + c] = t[r + 4 * c];
  ndt::mul3(R, old, neu);
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) t[r + 4 * c] = neu[r * 3 + c];
  t[12] += (float)x[0]; t[13] += (float)x[1]; t[14] += (float)x[2];
}

inline void r_derivative(const double* x, const double* R, double* g) {   // R row-major
  const double phi = x[3], theta = x[4], psi = x[5];
  const double cphi = cos(phi), sphi = sin(phi), ctheta = cos(theta), stheta = sin(theta);
  const double cpsi = cos(psi), spsi = sin(psi);
  const double dPhi[9] = {0, sphi * spsi + cphi * cpsi * stheta, cphi * spsi - cpsi * sphi * stheta,
                          0, -cpsi * sphi + cphi * spsi * stheta, -cphi * cpsi - sphi * spsi * stheta,
                          0, cphi * ctheta, -ctheta * sphi};
  const double dTheta[9] = {-cpsi * stheta, cpsi * ctheta * sphi, cphi * cpsi * ctheta,
                            -spsi * stheta, ctheta * sphi * spsi, cphi * ctheta * spsi,
                            -ctheta, -sphi * stheta, -cphi * stheta};
  const double dPsi[9] = {-ctheta * spsi, -cphi * cpsi - sphi * spsi * stheta, cpsi * sphi - cphi * spsi * stheta,
                          cpsi * ctheta, -cphi * spsi + cpsi * sphi * stheta, sphi * spsi + cphi * cpsi * stheta,
                          0, 0, 0};
  auto inner = [&](const double* a) {   // matricesInnerProd (gicp_omp.h:318-327)
    double r = 0.0;
    for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) r += a[j * 3 + i] * R[i * 3 + j];
    return r;
  };
  g[3] = inner(dPhi); g[4] = inner(dTheta); g[5] = inner(dPsi);
}

enum Status { kSuccess = 0, kRunning = 1, kNoProgress = 2, kError = -1 };
struct Params { double rho = 0.01, sigma = 0.01, tau1 = 9, tau2 = 0.05, tau3 = 0.5, step_size = 0.01; int order = 3; };
typedef std::function<int(const double* x, double* f, double* g)> Fdf;   // returns < 0 on device error

inline int solve_quadratic(double a, double b, double c, double* x0, double* x1) {
  const double disc = b * b - 4 * a * c;
  if (a == 0) { if (b == 0) return 0; *x0 = -c / b; return 1; }
  if (disc > 0) {
    if (b == 0) { const double r = fabs(0.5 * sqrt(disc) / a); *x0 = -r; *x1 = r; }
    else {
      const double sgnb = (b > 0 ? 1 : -1);
      const double temp = -0.5 * (b + sgnb * sqrt(disc));
      const double r1 = temp / a, r2 = c / temp;
      if (r1 < r2) { *x0 = r1; *x1 = r2; } else { *x0 = r2; *x1 = r1; }
    }
    return 2;
  }
  if (disc == 0) { *x0 = -0.5 * b / a; *x1 = -0.5 * b / a; return 2; }
  return 0;
}
inline double cubic(double c0, double c1, double c2, double c3, double z) { return c0 + z * (c1 + z * (c2 + z * c3)); }
inline void check_extremum(double c0, double c1, double c2, double c3, double z, double* zmin, double* fmin) {
  const double y = cubic(c0, c1, c2, c3, z);
  if (y < *fmin) { *zmin = z; *fmin = y; }
}
inline double interp_quad(double f0, double fp0, double f1, double zl, double zh) {
  const double fl = f0 + zl * (fp0 + zl * (f1 - f0 - fp0));
  const double fh = f0 + zh * (fp0 + zh * (f1 - f0 - fp0));
  const double c = 2 * (f1 - f0 - fp0);
  double zmin = zl, fmin = fl;
  if (fh < fmin) { zmin = zh; fmin = fh; }
  if (c > 0) {
    const double z = -fp0 / c;
    if (z > zl && z < zh) {
      const double f = f0 + z * (fp0 + z * (f1 - f0 - fp0));
      if (f < fmin) { zmin = z; fmin = f; }
    }
  }
  return zmin;
}
inline double interp_cubic(double f0, double fp0, double f1, double fp1, double zl, double zh) {
  const double eta = 3 * (f1 - f0) - 2 * fp0 - fp1;
  const double xi = fp0 + fp1 - 2 * (f1 - f0);
  const double c0 = f0, c1 = fp0, c2 = eta, c3 = xi;
  double zmin = zl, fmin = cubic(c0, c1, c2, c3, zl), z0 = 0, z1 = 0;
  check_extremum(c0, c1, c2, c3, zh, &zmin, &fmin);
  const int n = solve_quadratic(3 * c3, 2 * c2, c1, &z0, &z1);
  if (n == 2) {
    if (z0 > zl && z0 < zh) check_extremum(c0, c1, c2, c3, z0, &zmin, &fmin);
    if (z1 > zl && z1 < zh) check_extremum(c0, c1, c2, c3, z1, &zmin, &fmin);
  } else if (n == 1) {
    if (z0 > zl && z0 < zh) check_extremum(c0, c1, c2, c3, z0, &zmin, &fmin);
  }
  return zmin;
}
inline double interpolate(double a, double fa, double fpa, double b, double fb, double fpb, double xmin,
                          double xmax, int order) {
  double ymin = (xmin - a) / (b - a), ymax = (xmax - a) / (b - a);
  if (ymin > ymax) std::swap(ymin, ymax);
  double z;
  if (order > 2 && !(fpb != fpb)) z = interp_cubic(fa, fpa * (b - a), fb, fpb * (b - a), ymin, ymax);
  else z = interp_quad(fa, fpa * (b - a), fb, ymin, ymax);
  return a + z * (b - a);
}

struct Minimizer {
  static const int N = 6;
  Fdf fdf;
  Params par;
  double x0[N], g0[N], p[N], gradient[N], x_alpha[N], g_alpha[N];
  double f = 0, g0norm = 0, pnorm = 0, fp0 = 0, delta_f = 0;
  double f_alpha = 0, df_alpha = 0, f_key = 0, df_key = 0, x_key = 0, g_key = 0;
  bool failed = false;

  static double dot(const double* a, const double* b) { double s = 0; for (int i = 0; i < N; ++i) s += a[i] * b[i]; return s; }
  static double norm(const double* a) { return sqrt(dot(a, a)); }
  void call(const double* x, double* fo, double* g) { if (fdf(x, fo, g) < 0) failed = true; }
  void move_to(double alpha) {
    if (alpha == x_key) return;
    for (int i = 0; i < N; ++i) x_alpha[i] = x0[i] + alpha * p[i];
    x_key = alpha;
  }
  double slope() const { return dot(g_alpha, p); }
  double eval_f(double alpha) {
    if (alpha == f_key) return f_alpha;
    move_to(alpha);
    call(x_alpha, &f_alpha, nullptr);
    f_key = alpha;
    return f_alpha;
  }
  double eval_df(double alpha) {
    if (alpha == df_key) return df_alpha;
    move_to(alpha);
    if (alpha != g_key) { call(x_alpha, nullptr, g_alpha); g_key = alpha; }
    df_alpha = slope();
    df_key = alpha;
    return df_alpha;
  }
  void eval_fdf(double alpha, double* fo, double* dfo) {
    if (alpha == f_key && alpha == df_key) { *fo = f_alpha; *dfo = df_alpha; return; }
    if (alpha == f_key || alpha == df_key) { *fo = eval_f(alpha); *dfo = eval_df(alpha); return; }
    move_to(alpha);
    call(x_alpha, &f_alpha, g_alpha);
    f_key = alpha; g_key = alpha;
    df_alpha = slope(); df_key = alpha;
    *fo = f_alpha; *dfo = df_alpha;
  }
  void update_position(double alpha, double* x, double* fo, double* g) {
    double f_a, df_a;
    eval_fdf(alpha, &f_a, &df_a);
    *fo = f_a;
    for (int i = 0; i < N; ++i) { x[i] = x_alpha[i]; g[i] = g_alpha[i]; }
  }
  void change_direction() {
    for (int i = 0; i < N; ++i) { x_alpha[i] = x0[i]; g_alpha[i] = g0[i]; }
    x_key = 0; f_key = 0; g_key = 0;
    f_alpha = f; df_alpha = slope(); df_key = 0;
  }
  void init(double* x) {
    delta_f = 0;
    call(x, &f, gradient);
    for (int i = 0; i < N; ++i) { x0[i] = x[i]; g0[i] = gradient[i]; }
    g0norm = norm(g0);
    for (int i = 0; i < N; ++i) p[i] = gradient[i] * (-1 / g0norm);
    pnorm = norm(p);
    fp0 = -g0norm;
    change_direction();
  }
  int line_search(double alpha1, double* alpha_new) {
    double f0v, fp0v, falpha, falpha_prev, fpalpha = 0, fpalpha_prev, delta, alpha_next;
    double alpha = alpha1, alpha_prev = 0.0;
    double a = 0.0, b = alpha, fa, fb = 0.0, fpa, fpb = 0.0;
    int i = 0;
    eval_fdf(0.0, &f0v, &fp0v);
    falpha_prev = f0v; fpalpha_prev = fp0v;
    fa = f0v; fpa = fp0v;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    while (i++ < 100) {
      falpha = eval_f(alpha);
      if (falpha > f0v + alpha * par.rho * fp0v || falpha >= falpha_prev) {
        a = alpha_prev; fa = falpha_prev; fpa = fpalpha_prev;
        b = alpha; fb = falpha; fpb = nan;
        break;
      }
      fpalpha = eval_df(alpha);
      if (fabs(fpalpha) <= -par.sigma * fp0v) { *alpha_new = alpha; return kSuccess; }
      if (fpalpha >= 0) {
        a = alpha; fa = falpha; fpa = fpalpha;
        b = alpha_prev; fb = falpha_prev; fpb = fpalpha_prev;
        break;
      }
      delta = alpha - alpha_prev;
      alpha_next = interpolate(alpha_prev, falpha_prev, fpalpha_prev, alpha, falpha, fpalpha, alpha + delta,
                               alpha + par.tau1 * delta, par.order);
      alpha_prev = alpha; falpha_prev = falpha; fpalpha_prev = fpalpha;
      alpha = alpha_next;
    }
    while (i++ < 100) {
      delta = b - a;
      alpha = interpolate(a, fa, fpa, b, fb, fpb, a + par.tau2 * delta, b - par.tau3 * delta, par.order);
      falpha = eval_f(alpha);
      if ((a - alpha) * fpa <= std::numeric_limits<double>::epsilon()) return kNoProgress;
      if (falpha > f0v + par.rho * alpha * fp0v || falpha >= fa) {
        b = alpha; fb = falpha; fpb = nan;
      } else {
        fpalpha = eval_df(alpha);
        if (fabs(fpalpha) <= -par.sigma * fp0v) { *alpha_new = alpha; return kSuccess; }
        if (((b - a) >= 0 && fpalpha >= 0) || ((b - a) <= 0 && fpalpha <= 0)) {
          b = a; fb = fa; fpb = fpa;
          a = alpha; fa = falpha; fpa = fpalpha;
        } else {
          a = alpha; fa = falpha; fpa = fpalpha;
        }
      }
    }
    return kSuccess;
  }
  int one_step(double* x) {
    double alpha = 0.0, alpha1;
    const double f0v = f;
    if (pnorm == 0.0 || g0norm == 0.0 || fp0 == 0) return kNoProgress;
    if (delta_f < 0) {
      const double del = std::max(-delta_f, 10 * std::numeric_limits<double>::epsilon() * fabs(f0v));
      alpha1 = std::min(1.0, 2.0 * del / (-fp0));
    } else {
      alpha1 = fabs(par.step_size);
    }
    const int status = line_search(alpha1, &alpha);
    if (status != kSuccess) return status;
    update_position(alpha, x, &f, gradient);
    delta_f = f - f0v;
    double dx0[N], dg0[N];
    for (int i = 0; i < N; ++i) { dx0[i] = x[i] - x0[i]; dg0[i] = gradient[i] - g0[i]; }
    const double dxg = dot(dx0, gradient), dgg = dot(dg0, gradient), dxdg = dot(dx0, dg0), dgnorm = norm(dg0);
    double A = 0, B = 0;
    if (dxdg != 0) { B = dxg / dxdg; A = -(1.0 + dgnorm * dgnorm / dxdg) * B + dgg / dxdg; }
    for (int i = 0; i < N; ++i) p[i] = gradient[i] - A * dx0[i] - B * dg0[i];
    for (int i = 0; i < N; ++i) { g0[i] = gradient[i]; x0[i] = x[i]; }
    g0norm = norm(g0);
    pnorm = norm(p);
    const double dir = (dot(p, gradient) > 0) ? -1.0 : 1.0;
    for (int i = 0; i < N; ++i) p[i] *= dir / pnorm;
    pnorm = norm(p);
    fp0 = dot(p, g0);
    change_direction();
    return kSuccess;
  }
  int test_gradient(double epsabs) const { return norm(gradient) < epsabs ? kSuccess : kRunning; }
};

// GeneralizedIterativeClosestPoint::computeTransformation (gicp_omp_impl.hpp:381-514) with
// estimateRigidTransformationBFGS (:187-246) as the reference executes them, over two callbacks:
//   correspond(transformation, R, &m): the per-point part of one outer iteration (:419-463) for transformation_
//       (column-major float 4x4) and R = rot(transformation_ * guess) in double, row-major; m = correspondences
//   cost(T, S): the sums of one functor evaluation (:255-377) for T = base with applyState(x):
//       S[0] = sum res^T M res, S[1..3] = sum M res, S[4..12] = sum (base p)(M res)^T row-major
// both return < 0 on error (propagated as -1).  The device path passes lambdas around Stage's correspond and
// cost (gicp_run of the C ABI); the test hook sm_debug_gicp_outer passes a caller's functions, so this control flow —
// start vector, f / g assembly, BFGS driver, convergence test, final composition — is exercised on the host.
// transform_R = transformation_ * guess in double (:423-429): its rotation, row-major, for the correspondences
inline void outer_rotation(const float* transformation, const float* guess, double* R) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      double s = 0.0;
      for (int k = 0; k < 4; ++k) s += (double)transformation[i + 4 * k] * (double)guess[k + 4 * j];
      R[i * 3 + j] = s;
    }
}

struct OuterOut {
  float final_T[16];
  int iterations = 0;
  int bfgs_evals = 0;
};

template <class Correspond, class Cost>
inline int outer_loop(const Options& o, const float* guess, Correspond correspond, Cost cost, OuterOut* out) {
  float transformation[16], previous[16];
  for (int i = 0; i < 16; ++i) transformation[i] = previous[i] = (i % 5 == 0) ? 1.0f : 0.0f;
  int nr_iterations = 0, evals = 0;
  bool converged = false, callback_error = false;
  while (!converged) {
    double R[9];
    outer_rotation(transformation, guess, R);
    int m = 0;
    if (correspond(transformation, R, &m) < 0) return -1;
    for (int i = 0; i < 16; ++i) previous[i] = transformation[i];
    if (m < 4) break;                    // NotEnoughPointsException, caught at :489-492
    double x[6] = {(double)transformation[12], (double)transformation[13], (double)transformation[14],
                   atan2((double)transformation[2 + 4 * 1], (double)transformation[2 + 4 * 2]),
                   asin(-(double)transformation[2 + 4 * 0]),
                   atan2((double)transformation[1 + 4 * 0], (double)transformation[0 + 4 * 0])};
    Minimizer mz;
    mz.fdf = [&](const double* xx, double* f, double* g) -> int {
      ++evals;
      float T[16];
      for (int i = 0; i < 16; ++i) T[i] = guess[i];
      apply_state(T, xx);
      double S[13];
      if (cost(T, S) < 0) return -1;
      if (f) *f = S[0] / (double)m;
      if (g) {
        double Rm[9];
        for (int r = 0; r < 3; ++r) g[r] = S[1 + r] * (2.0 / m);
        for (int q = 0; q < 9; ++q) Rm[q] = S[4 + q] * (2.0 / m);
        r_derivative(xx, Rm, g);
      }
      return 0;
    };
    mz.init(x);
    int result = kRunning, inner = 0;
    do {
      ++inner;
      result = mz.one_step(x);
      if (result) break;
      result = mz.test_gradient(1e-2);
    } while (result == kRunning && inner < o.max_inner_iterations);
    if (mz.failed) { callback_error = true; break; }
    if (result == kNoProgress || result == kSuccess || inner == o.max_inner_iterations) {
      for (int i = 0; i < 16; ++i) transformation[i] = (i % 5 == 0) ? 1.0f : 0.0f;
      apply_state(transformation, x);
    } else {
      break;
    }
    double delta = 0.0;
    for (int k = 0; k < 4; ++k)
      for (int l = 0; l < 4; ++l) {
        const double ratio = (k < 3 && l < 3) ? 1.0 / o.rotation_epsilon : 1.0 / o.transformation_epsilon;
        const double c_delta = ratio * fabs((double)previous[k + 4 * l] - (double)transformation[k + 4 * l]);
        if (c_delta > delta) delta = c_delta;
      }
    ++nr_iterations;
    if (nr_iterations >= o.max_iterations || delta < 1) {
      converged = true;
      for (int i = 0; i < 16; ++i) previous[i] = transformation[i];
    }
  }
  if (callback_error) return -1;
  float Rp[9], Rg[9], Rf[9];            // :505-508
  for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { Rp[r * 3 + c] = previous[r + 4 * c]; Rg[r * 3 + c] = guess[r + 4 * c]; }
  ndt::mul3(Rp, Rg, Rf);
  float* final_T = out->final_T;
  for (int i = 0; i < 16; ++i) final_T[i] = (i % 5 == 0) ? 1.0f : 0.0f;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) final_T[r + 4 * c] = Rf[r * 3 + c];
    final_T[12 + r] = previous[12 + r] + guess[12 + r];
  }
  out->iterations = nr_iterations;
  out->bfgs_evals = evals;
  return 0;
}

// The device side of the GICP stage (gicp.cu): the source's float tree, both clouds' covariances, the matches with
// their Mahalanobis matrices, and the cost kernel's partial sums, ticket and sequence number.  reserve() sizes the
// buffers for ns source / nt target points, zeroes the ticket (each cost evaluation's last block resets it) and
// restarts the sequence.
struct Stage {
  FloatTree source_tree;
  DevBuf cov_s, cov_t, maha, match, partials, counter;   // counter: the match count, then the ticket
  double* sums = nullptr;      // device: the 13 sums of the last cost evaluation
  uint32_t* ticket = nullptr;
  long long seq = 0;
  int reserve(int ns, int nt, cudaStream_t stream);
  // computeCovariances (:59-131) over the cloud's own tree t into out; zeros below k_correspondences points, where
  // the reference logs an error and leaves them unset
  int covariances(const Options& o, const float* cloud, int n, const FloatTree& t, const DevBuf& out,
                  cudaStream_t stream) const;
  // the per-point part of one outer iteration (:430-461) over the target's tree tt; waits for the match count m
  int correspond(const Options& o, const float* src, int ns, const float* tgt, const FloatTree& tt, const float* guess,
                 const float* transformation, const double* R, cudaStream_t stream, int* m);
  // one functor evaluation (:255-377) at T; with host_sums / host_seq (device views of mapped pinned memory) the
  // kernel also writes the 13 sums there, then the sequence number ++seq
  int cost(const float* src, int ns, const float* tgt, const float* T, const float* base, double* host_sums,
           long long* host_seq, cudaStream_t stream);
};

}  // namespace gicp
}  // namespace smb

#endif  // SM_B200_GICP_HOST_H_
