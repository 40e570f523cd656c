// C ABI of libsm_b200.so (include/sm_b200.h): handles, option registry, uploads, Align.
#include "../../include/sm_b200.h"
#include "../../include/sm_b200_debug.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <iterator>
#include <mutex>
#include <string>
#include <thread>
#include <variant>
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "common.cuh"
#include "kernels.h"
#include "gicp_host.h"
#include "ndt_host.h"

namespace smb {

// NVTX ranges named like the reference's timer blocks (common/performance/simple_prof.h:
// REGISTER_FUNC in FindClosests / ErrorElements / ComputePointToPlane, REGISTER_BLOCK("Iteration"),
// "BuildKdTree", icp_fast.cc:103,171,261,465,484), visible in nsys / ncu timelines.
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

static thread_local std::string g_cuda_error;
void set_cuda_error(cudaError_t e, const char* expr, const char* file, int line) {
  char buf[512];
  snprintf(buf, sizeof(buf), "CUDA error %d (%s) at %s:%d: %s", (int)e, cudaGetErrorString(e),
           file, line, expr);
  g_cuda_error = buf;
}
const char* last_cuda_error() { return g_cuda_error.c_str(); }

namespace {

__global__ void deinterleave3_kernel(const double* __restrict__ aos, double* __restrict__ soa,
                                     int64_t stride, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  soa[i] = aos[3 * (int64_t)i];
  soa[stride + i] = aos[3 * (int64_t)i + 1];
  soa[2 * stride + i] = aos[3 * (int64_t)i + 2];
}

// a 3xN AoS cloud (host memory, staged through `stage`, or device memory) de-interleaved into
// SoA [3][stride], in stream order
int upload_soa(const double* pts, int64_t n, bool on_device, DevBuf& stage, double* soa, int64_t stride,
               cudaStream_t s) {
  const double* aos = pts;
  if (!on_device) {
    SMB_RC(stage.reserve((size_t)(3 * n) * sizeof(double)));
    SMB_CUDA_OK(cudaMemcpyAsync(stage.p, pts, (size_t)(3 * n) * sizeof(double), cudaMemcpyHostToDevice, s));
    aos = (const double*)stage.p;
  }
  deinterleave3_kernel<<<ceil_div(n, 256), 256, 0, s>>>(aos, soa, stride, (int)n);
  SMB_CUDA_OK(cudaGetLastError());
  return 0;
}

enum OptKind { kOptInt, kOptFloat, kOptDouble, kOptBool };
struct OptionDef { const char* name; OptKind kind; size_t offset; };

struct IcpOptions {
  int32_t knn_for_normal_estimate = 7;   // icp_fast.h:57
  int32_t max_iteration = 100;           // icp_fast.h:58
  float dist_outlier_ratio = 0.7f;       // icp_fast.h:59
  float knn_epsilon = 3.16f;             // icp_fast.cc:174 (engine option; same default)
  bool disable_convergence_check = false;
  bool profile_kernels = false;
  bool use_graphs = true;
  int32_t knn_queries_per_cta = 0; // phase A geometry: 0 = one query per thread, else queries per 256-thread CTA
  // type 1 (IcpUsingPointMatcher stand-in) only, icp_pointmatcher.cc:166-247
  float reading_sample_prob = 0.9f;      // RandomSamplingDataPointsFilter prob (:173)
  float accept_min_score = 0.6f;         // Align returns false below it (:145)
  int32_t sample_seed = 1;
};

struct NdtGicpOptions {                  // ndt_gicp.h:71-75
  float voxel_resolution = 0.2f;
  bool using_voxel_filter = true;
  bool use_ndt = true;
};

// The handle's mapped pinned block: what the device hands back to the host.  The GICP cost kernel writes its sums
// and then the sequence word straight into it; the other fields arrive with a read-back and a synchronisation.
struct HostBlock {
  double ndt_sums[44];     // one NDT evaluation (score, gradient, Hessian row-major, neighbours) or the fitness pass
  int ndt_overflow;        // the NDT grid's size guard, read back with the first evaluation
  double gicp_sums[13];    // one GICP cost evaluation
  long long gicp_seq;      // its sequence number, written after the sums
  double pm_score[3];      // the type-1 score pass: mean kept distance, kept, valid
  double spare[2];
};
static_assert(sizeof(HostBlock) == 64 * sizeof(double), "the mapped pinned block is 64 doubles");

// A captured launch sequence, replayed while the key (all pointers and sizes baked into the
// kernel arguments) is unchanged: one cudaGraphLaunch instead of ~100 kernel launches.
struct GraphCache {
  cudaGraphExec_t exec = nullptr;
  std::string key;
  ~GraphCache() { reset(); }
  void reset() { if (exec) cudaGraphExecDestroy(exec); exec = nullptr; key.clear(); }
};

// One state object per matcher type; a handle holds the one of its type.  A cloud count of 0 means "not set".
// IcpFast, and the ICP chain type 1 runs on its filtered clouds: the uploaded SoA double clouds, the iteration
// buffers, the tree's build workspace and the in-flight Align (sm_align_async .. sm_align_wait)
struct IcpFastMatcher {
  IcpOptions opt;
  bool inner_compensation = false;  // Interface::EnableInnerCompensation; set on IcpFast handles only
  int error_minimizer = kIcpPointToPlane;   // sm_set_icp_error_minimizer
  DevBuf kdws;                      // k-d build workspace of the target tree (and of type 1's score tree)
  DevBuf stage, stage_src, stage_tgt, stage_nrm, tgt_raw, nrm, src_raw;
  IcpFastBuffers bufs;
  int64_t n_source = 0, n_target = 0, sstride = 0, tstride = 0;
  bool up_src = false, up_tgt = false;
  IcpState* host_state = nullptr;  // pinned, allocated by sm_create
  GraphCache g_prologue, g_iterations;
  struct {
    IcpBuffers b; IcpParams p; KdWorkspace ws; std::string key;
    double* deskewed = nullptr;
    bool graphs = false, active = false;
    int enqueued = 0, launches = 0, max_it = 0;
  } run;
  ~IcpFastMatcher() { if (host_state) cudaFreeHost(host_state); }
};

// the packed float clouds (12 bytes per point) of the _f32 setters
struct F32Clouds { DevBuf src, tgt; int64_t n_src = 0, n_tgt = 0; };

// Ndt and NdtWithGicp: the float clouds, the NDT stage, the target's tree (fitness score, GICP correspondences) and
// the build workspace of their trees
struct NdtBase { F32Clouds in; NdtStage ndt; FloatTree target_tree; DevBuf kdws; };
struct NdtMatcher : NdtBase { ndt::Options opt; };
struct NdtGicpMatcher : NdtBase {
  NdtGicpOptions opt;
  DevBuf src_filt, tgt_filt;
  ApproxVoxelGrid approx;
  gicp::Stage gicp;
};

// IcpUsingPointMatcher stand-in (type 1): raw float clouds -> filtered double clouds -> the IcpFast chain it
// composes.  The normals pipeline has its own k-d workspace: icp.kdws.p is part of the IcpFast graph keys.
struct PmMatcher {
  IcpFastMatcher icp;
  F32Clouds in;
  bool src_dirty = false, tgt_dirty = false, score_tree_dirty = true;
  int surface_normals = SM_PM_NORMALS_LEAST_SQUARES;   // sm_set_pm_surface_normals
  int reading_sampler = SM_PM_SAMPLING_HASH;           // sm_set_pm_reading_sampler
  int64_t rand_position = 0;                           // rand() draws since srand(sample_seed)
  NormalsPipeline normals;
  PmStage stage;
  FloatTree score_tree;
  PmMatcher() { icp.opt.max_iteration = 150; }   // CounterTransformationChecker, icp_pointmatcher.cc:214
};

}  // namespace
}  // namespace smb

using namespace smb;

// What every matcher type uses, and the state object of the handle's type (created by sm_create).  Everything a
// handle owns is released by its destructor.
struct sm_handle {
  int type = 0;
  int device = 0;
  cudaStream_t stream = nullptr;      // stream in use
  cudaStream_t own_stream = nullptr;  // created by sm_create
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev_up[4] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<cudaEvent_t> prof_events;
  double* host_guess = nullptr;    // pinned, 16 doubles
  HostBlock* host = nullptr;       // pinned + mapped
  HostBlock* host_dev = nullptr;   // its device view
  std::string error;
  double final_score = 0.0;
  sm_align_info info = {};
  std::variant<std::monostate, IcpFastMatcher, NdtMatcher, NdtGicpMatcher, PmMatcher> m;

  template <class T> T* as() { return std::get_if<T>(&m); }   // the state object if it is a T, else null
  // the ICP chain: IcpFast's own, or the one type 1 composes
  IcpFastMatcher* icp_chain() { return as<PmMatcher>() ? &as<PmMatcher>()->icp : as<IcpFastMatcher>(); }

  ~sm_handle() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_up) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : prof_events) cudaEventDestroy(e);
    if (host) cudaFreeHost(host);
    if (host_guess) cudaFreeHost(host_guess);
    if (own_stream) cudaStreamDestroy(own_stream);
  }
};

namespace {

const OptionDef kIcpOptions[] = {
    {"knn_normal_estimate", kOptInt, offsetof(IcpOptions, knn_for_normal_estimate)},
    {"max_iteration", kOptInt, offsetof(IcpOptions, max_iteration)},
    {"dist_outlier_ratio", kOptFloat, offsetof(IcpOptions, dist_outlier_ratio)},
    {"knn_epsilon", kOptFloat, offsetof(IcpOptions, knn_epsilon)},
    {"disable_convergence_check", kOptBool, offsetof(IcpOptions, disable_convergence_check)},
    {"profile_kernels", kOptBool, offsetof(IcpOptions, profile_kernels)},
    {"use_graphs", kOptBool, offsetof(IcpOptions, use_graphs)},
    {"knn_queries_per_cta", kOptInt, offsetof(IcpOptions, knn_queries_per_cta)},
    {"reading_sample_prob", kOptFloat, offsetof(IcpOptions, reading_sample_prob)},
    {"accept_min_score", kOptFloat, offsetof(IcpOptions, accept_min_score)},
    {"sample_seed", kOptInt, offsetof(IcpOptions, sample_seed)},
};

const OptionDef kNdtOptions[] = {
    {"max_iterations", kOptInt, offsetof(ndt::Options, max_iterations)},
    {"resolution", kOptFloat, offsetof(ndt::Options, resolution)},
    {"step_size", kOptDouble, offsetof(ndt::Options, step_size)},
    {"outlier_ratio", kOptDouble, offsetof(ndt::Options, outlier_ratio)},
    {"transformation_epsilon", kOptDouble, offsetof(ndt::Options, transformation_epsilon)},
};

const OptionDef kNdtGicpOptions[] = {   // ndt_gicp.cc:31-36
    {"use_ndt", kOptBool, offsetof(NdtGicpOptions, use_ndt)},
    {"using_voxel_filter", kOptBool, offsetof(NdtGicpOptions, using_voxel_filter)},
    {"voxel_resolution", kOptFloat, offsetof(NdtGicpOptions, voxel_resolution)},
};

// the option table of the handle's type and the struct its offsets point into
struct OptionTable { const OptionDef* begin; const OptionDef* end; char* base; };
OptionTable options_of(sm_handle* h) {
  if (NdtMatcher* m = h->as<NdtMatcher>())
    return {std::begin(kNdtOptions), std::end(kNdtOptions), reinterpret_cast<char*>(&m->opt)};
  if (NdtGicpMatcher* m = h->as<NdtGicpMatcher>())
    return {std::begin(kNdtGicpOptions), std::end(kNdtGicpOptions), reinterpret_cast<char*>(&m->opt)};
  return {std::begin(kIcpOptions), std::end(kIcpOptions), reinterpret_cast<char*>(&h->icp_chain()->opt)};  // and type 1
}

// pugixml as_bool: first non-blank character in "1tTyY" -> true
bool as_bool(const char* text) {
  while (*text == ' ' || *text == '\t' || *text == '\n') ++text;
  return *text == '1' || *text == 't' || *text == 'T' || *text == 'y' || *text == 'Y';
}

int fail(sm_handle* h, int code, const std::string& msg) {
  if (h) h->error = msg;
  return code;
}
int cuda_fail(sm_handle* h) { return fail(h, SM_ERR_CUDA, last_cuda_error()); }

#define H_CUDA(expr)                                                   \
  do {                                                                 \
    cudaError_t _e = (expr);                                           \
    if (_e != cudaSuccess) {                                           \
      set_cuda_error(_e, #expr, __FILE__, __LINE__);                   \
      return cuda_fail(h);                                             \
    }                                                                  \
  } while (0)
#define H_RC(expr)                                                     \
  do {                                                                 \
    int _rc = (expr);                                                  \
    if (_rc == -100) return cuda_fail(h);                              \
    if (_rc < 0) return fail(h, _rc, #expr " failed");                 \
  } while (0)

int64_t pad64(int64_t n) { return (n + 63) & ~(int64_t)63; }

template <typename F>
int run_graphed(sm_handle* h, GraphCache& gc, const std::string& key, F enqueue) {
  if (gc.exec == nullptr || gc.key != key) {
    gc.reset();
    H_CUDA(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
    const int rc = enqueue();
    cudaGraph_t graph = nullptr;
    const cudaError_t e = cudaStreamEndCapture(h->stream, &graph);
    if (rc < 0 || e != cudaSuccess || graph == nullptr) {
      if (graph) cudaGraphDestroy(graph);
      if (e != cudaSuccess) set_cuda_error(e, "cudaStreamEndCapture", __FILE__, __LINE__);
      return rc < 0 ? rc : cuda_fail(h);
    }
    const cudaError_t e2 = cudaGraphInstantiate(&gc.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e2 != cudaSuccess) { gc.exec = nullptr; set_cuda_error(e2, "cudaGraphInstantiate", __FILE__, __LINE__); return cuda_fail(h); }
    gc.key = key;
  }
  H_CUDA(cudaGraphLaunch(gc.exec, h->stream));
  return 0;
}

template <typename T>
void key_append(std::string& k, const T& v) { k.append(reinterpret_cast<const char*>(&v), sizeof(T)); }

// upload (or adopt) an AoS 3xN cloud and de-interleave it into SoA [3][stride]
// own_stage: a staging buffer used by this cloud only.  Then nothing is reused before the stream
// has consumed it (stream order), the copy stays asynchronous and the caller's host array must
// stay valid until the stream reaches it (sm_align_pairs); with the shared staging buffer the call
// returns after the copy, which is the deep-copy contract of SetInputSource / SetInputTarget.
int load_cloud(sm_handle* h, const double* pts, int64_t n, bool on_device, DevBuf& soa, int64_t stride,
               DevBuf& stage, bool own_stage) {
  H_RC(soa.reserve((size_t)(3 * stride) * sizeof(double)));
  H_RC(upload_soa(pts, n, on_device, stage, (double*)soa.p, stride, h->stream));
  if (!on_device && !own_stage) H_CUDA(cudaStreamSynchronize(h->stream));  // the shared stage buffer is reused
  return 0;
}

// What can refuse a cloud or an alignment, checked before anything is enqueued: each returns 0 or the rc.
int icp_check_source(sm_handle* h, const double* pts, int64_t n) {
  if (!pts || n <= 0) return fail(h, SM_ERR_MISSING_INPUT, "SetInputSource: empty cloud");
  if (n > (1 << 30)) return fail(h, SM_ERR_BAD_ARGUMENT, "SetInputSource: too many points");
  return 0;
}

int icp_check_target(sm_handle* h, const double* pts, const double* nrm, int64_t n) {
  if (!pts || n <= 0) return fail(h, SM_ERR_MISSING_INPUT, "SetInputTarget: empty cloud");
  if (!nrm) return fail(h, SM_ERR_MISSING_INPUT, "SetInputTarget: IcpFast target needs normals");
  if (n > (1 << 30)) return fail(h, SM_ERR_BAD_ARGUMENT, "SetInputTarget: too many points");
  return 0;
}

// an alignment of ns -> nt points under the handle's options (icp_begin)
int icp_check_align(sm_handle* h, const IcpFastMatcher& f, int64_t ns, int64_t nt) {
  if (ns <= 0 || nt <= 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: source/target not set");
  const float q = f.opt.dist_outlier_ratio;   // CHECK(quantile >= 0 && quantile <= 1), icp_fast.cc:68
  if (!(q >= 0.0f && q <= 1.0f)) return fail(h, SM_ERR_BAD_ARGUMENT, "Align: dist_outlier_ratio outside [0, 1] (icp_fast.cc:68)");
  if (!(f.opt.knn_epsilon >= 0.0f)) return fail(h, SM_ERR_BAD_ARGUMENT, "Align: knn_epsilon must be >= 0");
  if (kd_num_levels((int)nt, 8) > 24) return fail(h, SM_ERR_BAD_ARGUMENT, "target too large (tree deeper than 24 levels)");
  return 0;
}

// a pair of sm_align_pairs, in the order sm_set_input_target, sm_set_input_source and sm_align check it: the rc is
// the one those calls would return
int icp_check_pair(sm_handle* h, const IcpFastMatcher& f, const sm_pair& pr) {
  int rc = icp_check_target(h, pr.target_3xn, pr.target_normals_3xn, pr.n_target);
  if (rc == 0) rc = icp_check_source(h, pr.source_3xn, pr.n_source);
  if (rc == 0) rc = icp_check_align(h, f, pr.n_source, pr.n_target);
  return rc;
}

int icp_set_source(sm_handle* h, IcpFastMatcher& f, const double* pts, int64_t n, bool on_device, bool async = false) {
  if (int rc = icp_check_source(h, pts, n)) return rc;
  H_CUDA(cudaEventRecord(h->ev_up[0], h->stream));
  f.sstride = pad64(n);
  H_RC(load_cloud(h, pts, n, on_device, f.src_raw, f.sstride, async ? f.stage_src : f.stage, async));
  H_CUDA(cudaEventRecord(h->ev_up[1], h->stream));
  f.up_src = true;
  f.n_source = n;
  return 0;
}

int icp_set_target(sm_handle* h, IcpFastMatcher& f, const double* pts, const double* nrm, int64_t n, bool on_device,
                   bool async = false) {
  if (int rc = icp_check_target(h, pts, nrm, n)) return rc;
  H_CUDA(cudaEventRecord(h->ev_up[2], h->stream));
  f.tstride = pad64(n);
  H_RC(load_cloud(h, pts, n, on_device, f.tgt_raw, f.tstride, async ? f.stage_tgt : f.stage, async));
  H_RC(load_cloud(h, nrm, n, on_device, f.nrm, f.tstride, async ? f.stage_nrm : f.stage, async));
  H_CUDA(cudaEventRecord(h->ev_up[3], h->stream));
  f.up_tgt = true;
  f.n_target = n;
  return 0;
}

int build_tree_f32(sm_handle* h, DevBuf& kdws, const float* pts, int n, FloatTree& t) {
  if (kd_num_levels(n, 8) > 24) return fail(h, SM_ERR_BAD_ARGUMENT, "cloud too large");
  H_RC(t.build(pts, n, kdws, h->stream));
  return 0;
}

// one chunk of iterations + the asynchronous read-back of the state record
int icp_enqueue_chunk(sm_handle* h, IcpFastMatcher& f) {
  auto& r = f.run;
  const IcpParams& p = r.p;
  const int chunk = p.disable_convergence ? (r.max_it - r.enqueued)
                                          : ((r.max_it - r.enqueued) < 8 ? (r.max_it - r.enqueued) : 8);
  cudaEvent_t* evs = nullptr;
  if (f.opt.profile_kernels) {
    while ((int)h->prof_events.size() < 4 * (r.enqueued + chunk)) {
      cudaEvent_t e; H_CUDA(cudaEventCreate(&e)); h->prof_events.push_back(e);
    }
    evs = h->prof_events.data() + 4 * r.enqueued;
  }
  if (r.graphs) {
    std::string ikey = r.key;
    const int first_chunk = r.enqueued == 0 ? 1 : 0;
    key_append(ikey, chunk); key_append(ikey, first_chunk);
    H_RC(run_graphed(h, f.g_iterations, ikey, [&]() {
      return icp_enqueue_iterations(r.b, p, r.enqueued, chunk, h->stream, nullptr, r.deskewed);
    }));
  } else {
    H_RC(icp_enqueue_iterations(r.b, p, r.enqueued, chunk, h->stream, evs, r.deskewed));
  }
  r.enqueued += chunk;
  r.launches += icp_iteration_launches(p.inner_compensation != 0) * chunk;
  H_CUDA(cudaMemcpyAsync(f.host_state, f.bufs.state.p, sizeof(IcpState), cudaMemcpyDeviceToHost, h->stream));
  return 0;
}

// IcpFast::Align, first half: everything is enqueued, nothing is waited for
int icp_begin(sm_handle* h, IcpFastMatcher& f, const double* guess) {
  auto& r = f.run;
  r.active = false;
  if (int rc = icp_check_align(h, f, f.n_source, f.n_target)) return rc;
  NvtxRange nvtx_align("IcpFast::Align");
  const int ns = (int)f.n_source, nt = (int)f.n_target;
  const int levels = kd_num_levels(nt, 8);
  // EnableInnerCompensation: IcpFast::Align reads it (icp_fast.cc:487, :509); type 1 runs the IcpFast chain but,
  // like IcpUsingPointMatcher, ignores it: its flag stays false
  H_RC(f.bufs.reserve(ns, nt, f.sstride, f.tstride, f.inner_compensation));
  KdWorkspace& ws = r.ws;
  H_RC(ws.carve(f.kdws, nt, 8));

  IcpBuffers& b = r.b;
  f.bufs.fill(b, (const double*)f.tgt_raw.p, (const double*)f.nrm.p, (const double*)f.src_raw.p);
  IcpParams& p = r.p;
  p.n_source = ns; p.n_target = nt;
  p.max_iteration = f.opt.max_iteration;
  p.dist_outlier_ratio = f.opt.dist_outlier_ratio;
  const double eps = (double)f.opt.knn_epsilon;
  p.max_error2 = (1.0 + eps) * (1.0 + eps);
  p.disable_convergence = f.opt.disable_convergence_check ? 1 : 0;
  p.knn_queries_per_cta = f.opt.knn_queries_per_cta;
  p.tree_levels = levels;
  p.inner_compensation = f.inner_compensation ? 1 : 0;
  p.error_minimizer = (int16_t)f.error_minimizer;
  r.deskewed = f.inner_compensation ? (double*)f.bufs.deskewed.p : nullptr;

  memcpy(h->host_guess, guess, 16 * sizeof(double));   // pinned: the caller's array may go away
  H_CUDA(cudaMemcpyAsync(f.bufs.guess.p, h->host_guess, 16 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  H_CUDA(cudaEventRecord(h->ev[0], h->stream));
  r.graphs = f.opt.use_graphs && !f.opt.profile_kernels;
  r.key.clear();
  key_append(r.key, b); key_append(r.key, p); key_append(r.key, f.bufs.guess.p); key_append(r.key, f.kdws.p);
  key_append(r.key, r.deskewed);   // p.inner_compensation and p.error_minimizer are part of p
  if (r.graphs) {
    H_RC(run_graphed(h, f.g_prologue, r.key, [&]() {
      return icp_prologue(b, p, (const double*)f.bufs.guess.p, ws, f.bufs.tree, h->stream);
    }));
  } else {
    H_RC(icp_prologue(b, p, (const double*)f.bufs.guess.p, ws, f.bufs.tree, h->stream));
  }
  H_CUDA(cudaEventRecord(h->ev[1], h->stream));
  r.launches = icp_prologue_launches(levels);
  r.enqueued = 0;
  r.max_it = p.max_iteration > 0 ? p.max_iteration : 1;
  H_RC(icp_enqueue_chunk(h, f));
  r.active = true;
  return 0;
}

// second half: wait, continue in chunks while the convergence test has not fired, report
int icp_end(sm_handle* h, IcpFastMatcher& f, double* result) {
  auto& r = f.run;
  if (!r.active) return fail(h, SM_ERR_BAD_ARGUMENT, "sm_align_wait without sm_align_async");
  r.active = false;
  while (true) {
    H_CUDA(cudaStreamSynchronize(h->stream));
    if (f.host_state->done || r.enqueued >= r.max_it) break;
    H_RC(icp_enqueue_chunk(h, f));
  }
  H_CUDA(cudaEventRecord(h->ev[2], h->stream));
  H_CUDA(cudaEventSynchronize(h->ev[2]));
  const IcpState& st = *f.host_state;
  h->info.iterations = st.iteration;
  h->info.status = st.status;
  h->info.solve_path = st.solve_path;
  h->info.kept = st.kept;
  h->info.limit = st.limit;
  h->info.ms_upload = 0.f;
  float ms = 0.f;
  if (f.up_src && cudaEventElapsedTime(&ms, h->ev_up[0], h->ev_up[1]) == cudaSuccess) h->info.ms_upload += ms;
  if (f.up_tgt && cudaEventElapsedTime(&ms, h->ev_up[2], h->ev_up[3]) == cudaSuccess) h->info.ms_upload += ms;
  f.up_src = f.up_tgt = false;
  cudaEventElapsedTime(&h->info.ms_prologue, h->ev[0], h->ev[1]);
  cudaEventElapsedTime(&h->info.ms_iterations, h->ev[1], h->ev[2]);
  h->info.kernel_launches = r.launches;
  h->info.ms_knn = h->info.ms_accum = h->info.ms_finish = 0.f;
  h->info.profiled_iterations = 0;
  if (f.opt.profile_kernels) {
    for (int it = 0; it < st.iteration && 4 * it + 3 < (int)h->prof_events.size(); ++it) {
      float a = 0.f, bb = 0.f, c = 0.f;
      cudaEventElapsedTime(&a, h->prof_events[4 * it], h->prof_events[4 * it + 1]);
      cudaEventElapsedTime(&bb, h->prof_events[4 * it + 1], h->prof_events[4 * it + 2]);
      cudaEventElapsedTime(&c, h->prof_events[4 * it + 2], h->prof_events[4 * it + 3]);
      h->info.ms_knn += a; h->info.ms_accum += bb; h->info.ms_finish += c;
      h->info.profiled_iterations++;
    }
  }
  if (st.status < 0)
    return fail(h, st.status, st.status == -2 ? "Align: no finite match distance (icp_fast.cc:81)"
                                              : "Align: no point to minimize (icp_fast.cc:114)");
  memcpy(result, st.result, 16 * sizeof(double));
  h->final_score = st.final_score;
  return 1;  // IcpFast::Align always returns true (icp_fast.cc:528)
}

int icp_align(sm_handle* h, IcpFastMatcher& f, const double* guess, double* result) {
  H_RC(icp_begin(h, f, guess));
  return icp_end(h, f, result);
}

// ---- IcpUsingPointMatcher stand-in (type 1) ------------------------------------------------
// registrators/icp_pointmatcher.cc:125-247 drives libpointmatcher 1.3.1 (external, float) with
//   reading filter    RandomSampling prob 0.9                      -> PmStage::sample: by default a
//                     counter hash instead of std::rand, so the kept set is reproducible; with
//                     sm_set_pm_reading_sampler(GLIBC_RAND) glibc's rand() stream itself, drawn from
//                     the handle's stream position (icp_pm.cu pm_rand_flags_kernel)
//   reference filter  SamplingSurfaceNormal knn 7, one point per box -> NormalsPipeline: by default
//                     CalculateNormals, the reference author's own restatement of that filter
//                     (cloud_types.cc:73-144); with sm_set_pm_surface_normals(EIGENVECTOR) the filter's
//                     own float box mean and smallest-eigenvector normal (normals.cu leaf_eigen_normal)
//   matcher / outlier filter / minimiser / checkers                 -> the IcpFast chain, which
//                     icp_fast.cc ported from exactly these modules (k-d tree eps 3.16, trim 0.7,
//                     point-to-plane, 4-sample differential checker 0.001 rad / 0.01 m), here in
//                     double, capped at 150 iterations
//   score (:131-148)  unfiltered reading moved by the result vs unfiltered reference, same matcher,
//                     trim 0.7, exp(-mean kept distance); Align() false below 0.6 (:145)
// It is a deterministic equivalent, not a bit-level restatement: libpointmatcher's float ICP
// arithmetic is not reproduced, and its rand() stream only in GLIBC_RAND mode, given seed and position.
int pm_align(sm_handle* h, PmMatcher& pm, const double* guess, double* result) {
  if (pm.in.n_src <= 0 || pm.in.n_tgt <= 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: source/target not set");
  cudaStream_t s = h->stream;
  if (pm.tgt_dirty) {
    const int n = (int)pm.in.n_tgt;
    NormalsPipeline& np = pm.normals;
    H_RC(np.reserve(n));
    H_RC(ndt_float_to_soa((const float*)pm.in.tgt.p, n, np.input(), np.stride, s));
    uint32_t m = 0;
    H_RC(np.run(n, (NormalsMode)pm.surface_normals, s, &m));
    if (m == 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: no target point survived the surface-normal filter");
    H_RC(icp_set_target(h, pm.icp, np.points(), np.normals(), (int64_t)m, true));
    pm.tgt_dirty = false;
  }
  PmStage& st = pm.stage;
  H_RC(st.reserve((int)pm.in.n_src));
  // the rand sampler draws anew on every Align, as the filter does inside ICP::compute
  const bool rand = pm.reading_sampler == SM_PM_SAMPLING_GLIBC_RAND;
  if (rand && pm.rand_position > INT64_MAX - pm.in.n_src)
    return fail(h, SM_ERR_BAD_ARGUMENT, "Align: the rand() stream position would pass 2^63 - 1");
  if (pm.src_dirty || rand) {
    uint32_t kept = 0;
    PmRandWindow at;
    if (rand) at = pm_rand_window((uint32_t)pm.icp.opt.sample_seed, (uint64_t)pm.rand_position);
    H_RC(st.sample((const float*)pm.in.src.p, (int)pm.in.n_src, pm.icp.opt.reading_sample_prob,
                   (uint32_t)pm.icp.opt.sample_seed, s, &kept, rand ? &at : nullptr));
    if (rand) pm.rand_position += pm.in.n_src;   // one draw per reading point
    if (kept == 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: the reading filter kept no point");
    H_RC(icp_set_source(h, pm.icp, st.points(), (int64_t)kept, true));
    pm.src_dirty = rand;   // the next Align filters anew, whichever sampler it runs
  }
  const int rc = icp_align(h, pm.icp, guess, result);
  h->info.aux[2] = (double)pm.icp.n_source;   // reading points after the filter
  h->info.aux[3] = (double)pm.icp.n_target;   // reference points after the filter
  if (rc < 0) return rc;
  h->info.aux[0] = h->final_score;        // IcpFast's own score (last iteration, filtered clouds)
  // ---- "compute the final score" (icp_pointmatcher.cc:131-148) -------------------------------
  {
    const int ns = (int)pm.in.n_src, nt = (int)pm.in.n_tgt;
    if (pm.score_tree_dirty) {
      H_RC(build_tree_f32(h, pm.icp.kdws, (const float*)pm.in.tgt.p, nt, pm.score_tree));
      pm.score_tree_dirty = false;
    }
    for (int i = 0; i < 16; ++i) h->host_guess[i] = result[i];      // pinned staging
    const double eps = (double)pm.icp.opt.knn_epsilon;
    H_RC(st.score_pass((const float*)pm.in.src.p, ns, h->host_guess, pm.score_tree, (1.0 + eps) * (1.0 + eps),
                       pm.icp.opt.dist_outlier_ratio, h->host->pm_score, s));
    if (!(h->host->pm_score[1] > 0.0)) return fail(h, SM_ERR_NOTHING_TO_MINIMIZE, "Align: no matched point for the score");
    h->final_score = exp(-h->host->pm_score[0]);
    h->info.aux[1] = h->host->pm_score[1];     // matches kept by the trim in the score pass
  }
  return h->final_score < (double)pm.icp.opt.accept_min_score ? 0 : 1;
}

// ---- Ndt ---------------------------------------------------------------------------------
// the packed float source or target cloud of Ndt, NdtWithGicp and type 1
int set_input_f32(sm_handle* h, const float* xyz, int64_t n, int64_t stride, bool target, bool on_device) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  NdtMatcher* nm = h->as<NdtMatcher>();
  NdtGicpMatcher* gm = h->as<NdtGicpMatcher>();
  PmMatcher* pm = h->as<PmMatcher>();
  F32Clouds* in = nm ? &nm->in : gm ? &gm->in : pm ? &pm->in : nullptr;
  if (!in) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "SetInput (float): IcpFast takes sm_set_input_source / _target");
  if (!xyz || n <= 0) return fail(h, SM_ERR_MISSING_INPUT, "SetInput: empty cloud");
  if (stride < 12 || n > (1 << 30)) return fail(h, SM_ERR_BAD_ARGUMENT, "SetInput: bad stride / size");
  H_CUDA(cudaSetDevice(h->device));
  DevBuf& dst = target ? in->tgt : in->src;
  H_RC(dst.reserve((size_t)n * 12 + 64));
  H_CUDA(cudaMemcpy2DAsync(dst.p, 12, xyz, (size_t)stride, 12, (size_t)n,
                           on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
  if (!on_device) H_CUDA(cudaStreamSynchronize(h->stream));
  (target ? in->n_tgt : in->n_src) = n;
  if (pm && target) pm->tgt_dirty = pm->score_tree_dirty = true;
  if (pm && !target) pm->src_dirty = true;
  return 0;
}

struct NdtRunOut {
  float final_T[16];
  double fitness = 0, trans_probability = 0, mean_neighbors = 0;
  int iterations = 0, evaluations = 0, launches = 0;
  float ms_grid = 0, ms_iter = 0, ms_fit = 0;
};

// pcl::Registration::align -> NormalDistributionsTransform::computeTransformation
// (ndt_omp_impl.hpp:81-171) -> getFitnessScore, on device clouds src/tgt (packed float xyz).
int ndt_run(sm_handle* h, NdtBase& m, const float* src, int ns, const float* tgt, int nt, const ndt::Options& o,
            bool f64_math, const double* guess, NdtRunOut* out) {
  NdtStage& st = m.ndt;
  H_RC(st.reserve(nt, ns));
  H_CUDA(cudaEventRecord(h->ev[0], h->stream));
  H_RC(st.build_grid(tgt, nt, o.resolution, h->stream));        // setInputTarget -> init()
  // the grid's size guard arrives with the first evaluation's sums
  volatile int* overflow = &h->host->ndt_overflow;
  *overflow = 0;
  H_CUDA(cudaMemcpyAsync((void*)overflow, &st.ws.grid->overflow, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  H_CUDA(cudaEventRecord(h->ev[1], h->stream));
  NdtEvalParams P = ndt::eval_params(o, f64_math);
  // the Newton loop itself is host code shared with the test hook sm_debug_ndt_newton (ndt_host.h newton_loop);
  // one evaluation = computeDerivatives on the device, 44 sums handed back through mapped pinned memory
  ndt::NewtonOut nw;
  int launches = NdtStage::kGridLaunches;
  const int nrc = ndt::newton_loop(o, guess, ns, P, [&](const NdtEvalParams& Pe, const double*, double* sums) -> int {
    H_RC(st.eval(src, ns, Pe, o.search, h->host->ndt_sums, h->stream));
    if (*overflow) return SM_ERR_BAD_ARGUMENT;
    for (int i = 0; i < 44; ++i) sums[i] = h->host->ndt_sums[i];
    launches += NdtStage::kEvalLaunches;
    return 0;
  }, &nw);
  // the reference clears the grid and goes on to search a tree that was never given a cloud (undefined behaviour)
  if (*overflow)
    return fail(h, SM_ERR_BAD_ARGUMENT, "Align: the NDT target's bounding box holds more than INT32_MAX voxels at "
                                        "this resolution (voxel indices would overflow)");
  H_RC(nrc);
  float* final_T = out->final_T;
  for (int i = 0; i < 16; ++i) final_T[i] = nw.final_T[i];
  H_CUDA(cudaEventRecord(h->ev[2], h->stream));
  // getFitnessScore (ndt.cc:60): exact 1-NN over the full target (PCL builds this search
  // tree in setInputTarget; the reference calls that on every Align)
  H_RC(build_tree_f32(h, m.kdws, tgt, nt, m.target_tree));
  H_RC(st.fitness(src, ns, tgt, final_T, m.target_tree, h->host->ndt_sums, h->stream, &out->fitness));
  H_CUDA(cudaEventRecord(h->ev[3], h->stream));
  H_CUDA(cudaEventSynchronize(h->ev[3]));
  out->iterations = nw.iterations;
  out->evaluations = nw.evaluations;
  out->trans_probability = nw.score / (double)ns;
  out->mean_neighbors = nw.evaluations ? nw.nb_sum / nw.evaluations : 0.0;
  out->launches = launches + NdtStage::fitness_launches(nt);
  cudaEventElapsedTime(&out->ms_grid, h->ev[0], h->ev[1]);
  cudaEventElapsedTime(&out->ms_iter, h->ev[1], h->ev[2]);
  cudaEventElapsedTime(&out->ms_fit, h->ev[2], h->ev[3]);
  return 0;
}

// Ndt::Align (ndt.cc:38-64)
int ndt_align(sm_handle* h, NdtMatcher& m, const double* guess, double* result) {
  if (m.in.n_src <= 0 || m.in.n_tgt <= 0) {    // ndt.cc:40-42: return false
    for (int i = 0; i < 16; ++i) result[i] = guess[i];
    return 0;
  }
  NdtRunOut r;
  const int rc = ndt_run(h, m, (const float*)m.in.src.p, (int)m.in.n_src, (const float*)m.in.tgt.p, (int)m.in.n_tgt,
                         m.opt, false, guess, &r);
  if (rc < 0) return rc;                        // with ndt_run's own message
  h->final_score = r.fitness;
  for (int i = 0; i < 16; ++i) result[i] = (double)r.final_T[i];     // .cast<double>() (ndt.cc:61)
  memset(&h->info, 0, sizeof(h->info));
  h->info.iterations = r.iterations;
  h->info.evaluations = r.evaluations;
  h->info.trans_probability = r.trans_probability;
  h->info.mean_neighbors = r.mean_neighbors;
  h->info.kernel_launches = r.launches;
  h->info.ms_prologue = r.ms_grid; h->info.ms_iterations = r.ms_iter; h->info.ms_finish = r.ms_fit;
  return 1;
}

// ---- NdtWithGicp ---------------------------------------------------------------------------
// GeneralizedIterativeClosestPoint::computeTransformation (gicp_omp_impl.hpp:381-514) with the
// BFGS inner solver on the host; the target tree must be built in m.target_tree.
int gicp_run(sm_handle* h, NdtGicpMatcher& m, const float* src, int ns, const float* tgt, int nt, const float* guess,
             const gicp::Options& o, float* final_T, int* iterations, int* bfgs_evals) {
  gicp::Stage& g = m.gicp;
  const FloatTree& tt = m.target_tree;
  H_RC(build_tree_f32(h, m.kdws, src, ns, g.source_tree));
  H_RC(g.reserve(ns, nt, h->stream));
  volatile long long* seq_word = &h->host->gicp_seq;
  *seq_word = 0;
  H_RC(g.covariances(o, tgt, nt, tt, g.cov_t, h->stream));
  H_RC(g.covariances(o, src, ns, g.source_tree, g.cov_s, h->stream));
  // the outer loop, the BFGS driver and the assembly of f / g from the 13 sums are host code shared with the test
  // hook sm_debug_gicp_outer (gicp_host.h outer_loop); the two callbacks are the device work
  gicp::OuterOut go;
  bool cuda_error = false;
  const int grc = gicp::outer_loop(
      o, guess,
      [&](const float* transformation, const double* R, int* m) -> int {
        if (g.correspond(o, src, ns, tgt, tt, guess, transformation, R, h->stream, m) != 0) { cuda_error = true; return -1; }
        return 0;
      },
      [&](const float* T, double* S) -> int {
        // the kernel's last block writes the 13 sums and then the sequence word into mapped pinned memory
        if (g.cost(src, ns, tgt, T, guess, h->host_dev->gicp_sums, &h->host_dev->gicp_seq, h->stream) != 0) {
          cuda_error = true;
          return -1;
        }
        for (long spins = 0; *seq_word != g.seq; ++spins) {
          if ((spins & 0xfff) == 0xfff && cudaStreamQuery(h->stream) != cudaErrorNotReady) {
            if (*seq_word == g.seq) break;
            if (cudaStreamSynchronize(h->stream) != cudaSuccess || *seq_word != g.seq) { cuda_error = true; return -1; }   // the kernel failed
          }
        }
        std::atomic_thread_fence(std::memory_order_acquire);
        for (int q = 0; q < 13; ++q) S[q] = h->host->gicp_sums[q];
        return 0;
      },
      &go);
  if (grc < 0 || cuda_error) return cuda_fail(h);
  for (int i = 0; i < 16; ++i) final_T[i] = go.final_T[i];
  *iterations = go.iterations;
  *bfgs_evals = go.bfgs_evals;
  return 0;
}

// NdtWithGicp::Align (ndt_gicp.cc:55-112)
int ndt_gicp_align(sm_handle* h, NdtGicpMatcher& m, const double* guess, double* result) {
  if (m.in.n_src <= 0 || m.in.n_tgt <= 0)
    return fail(h, SM_ERR_MISSING_INPUT, "Align: source/target not set");   // null deref in the reference
  const float* src = (const float*)m.in.src.p;
  const float* tgt = (const float*)m.in.tgt.p;
  int ns = (int)m.in.n_src, nt = (int)m.in.n_tgt;
  if (m.opt.using_voxel_filter) {           // pcl::ApproximateVoxelGrid::filter (ndt_gicp.cc:59-70)
    H_RC(m.approx.filter(src, ns, m.opt.voxel_resolution, m.src_filt, &ns, h->stream));
    H_RC(m.approx.filter(tgt, nt, m.opt.voxel_resolution, m.tgt_filt, &nt, h->stream));
    src = (const float*)m.src_filt.p;
    tgt = (const float*)m.tgt_filt.p;
  }
  memset(&h->info, 0, sizeof(h->info));
  h->info.aux[2] = ns; h->info.aux[3] = nt;
  if (ns <= 0 || nt <= 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: empty cloud after the voxel filter");
  float ndt_guess[16];
  for (int i = 0; i < 16; ++i) ndt_guess[i] = (float)guess[i];
  double ndt_score = 0.9;
  if (m.opt.use_ndt) {                    // ndt_gicp.cc:82-88, configuration :44-47
    ndt::Options no;                      // stock pcl::NormalDistributionsTransform: KDTREE only
    no.transformation_epsilon = 0.01; no.step_size = 0.1; no.resolution = 1.0f; no.max_iterations = 35;
    NdtRunOut r;
    const int rc = ndt_run(h, m, src, ns, tgt, nt, no, true, guess, &r);
    if (rc < 0) return rc;                      // with ndt_run's own message
    ndt_score = r.fitness;
    for (int i = 0; i < 16; ++i) ndt_guess[i] = r.final_T[i];
    h->info.evaluations = r.evaluations;
    h->info.ms_prologue = r.ms_grid + r.ms_iter + r.ms_fit;
  } else {
    H_RC(build_tree_f32(h, m.kdws, tgt, nt, m.target_tree));
  }
  h->info.aux[0] = ndt_score;
  double icp_score = 10.0;
  if (ndt_score <= 1.0) {                 // :92-103
    float final_T[16];
    int it = 0, evals = 0;
    H_CUDA(cudaEventRecord(h->ev[0], h->stream));
    H_RC(gicp_run(h, m, src, ns, tgt, nt, ndt_guess, gicp::Options(), final_T, &it, &evals));
    H_RC(m.ndt.reserve(nt, ns));
    H_RC(m.ndt.fitness(src, ns, tgt, final_T, m.target_tree, h->host->ndt_sums, h->stream, &icp_score));
    H_CUDA(cudaEventRecord(h->ev[1], h->stream));
    H_CUDA(cudaEventSynchronize(h->ev[1]));
    cudaEventElapsedTime(&h->info.ms_iterations, h->ev[0], h->ev[1]);
    h->final_score = exp(-icp_score);
    for (int i = 0; i < 16; ++i) result[i] = (double)final_T[i];
    h->info.iterations = it;
    h->info.profiled_iterations = evals;   // BFGS cost evaluations
    h->info.aux[1] = icp_score;
    return 1;
  }
  for (int i = 0; i < 16; ++i) result[i] = guess[i];   // :104-108
  h->final_score = exp(-icp_score);
  return 0;
}

// the double source or target cloud: IcpFast's setters; the other types take float clouds through the _f32 setters
int set_f64(sm_handle* h, bool target, bool on_device, const double* pts, int64_t n, const double* nrm = nullptr) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  IcpFastMatcher* f = h->as<IcpFastMatcher>();
  if (!f) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "sm_set_input_source / _target (double clouds): IcpFast only");
  H_CUDA(cudaSetDevice(h->device));
  return target ? icp_set_target(h, *f, pts, nrm, n, on_device) : icp_set_source(h, *f, pts, n, on_device);
}

// The set-up the stand-alone searches share: the target uploaded AoS -> SoA and its kIds tree built, then, for nq > 0,
// the queries uploaded and search(tree, queries, query stride) run, all on stream s, which is synchronised after the
// target's upload and again before returning.  Host clouds go through one staging buffer; device clouds are read in
// place.
template <class Search>
int knn_on_target(const double* target, int64_t nt, const double* query, int64_t nq, int bucket, bool on_device,
                  cudaStream_t s, Search search) {
  const int64_t ts = pad64(nt), qs = pad64(nq > 0 ? nq : 1);
  DevBuf stage, tgt, qry, kdws;
  KdCompactTree tree;
  if (!on_device) SMB_RC(stage.reserve((size_t)3 * (size_t)(nt > nq ? nt : nq) * sizeof(double)));   // both uploads
  SMB_RC(tgt.reserve((size_t)3 * ts * sizeof(double)));
  SMB_RC(qry.reserve((size_t)3 * qs * sizeof(double)));
  SMB_RC(tree.reserve((int)nt, bucket, KdCompactTree::kIds));
  KdWorkspace ws;
  SMB_RC(ws.carve(kdws, (int)nt, bucket));
  SMB_RC(upload_soa(target, nt, on_device, stage, (double*)tgt.p, ts, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  SMB_RC(tree.build((const double*)tgt.p, nullptr, ts, (int)nt, bucket, ws, s));
  if (nq > 0) {
    SMB_RC(upload_soa(query, nq, on_device, stage, (double*)qry.p, qs, s));
    SMB_RC(search(tree.view(), (const double*)qry.p, qs));
  }
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return SM_OK;
}

}  // namespace

extern "C" {

int sm_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}

const char* sm_version(void) { return "sm_b200 0.1 (sm_90a)"; }

int sm_create(int type, int device, sm_handle** out) {
  if (!out) return SM_ERR_BAD_ARGUMENT;
  *out = nullptr;
  sm_handle* h = new sm_handle();   // its state objects allocate nothing until they are used
  if (type == SM_TYPE_FAST_ICP) h->m.emplace<IcpFastMatcher>();
  else if (type == SM_TYPE_NDT) h->m.emplace<NdtMatcher>();
  else if (type == SM_TYPE_NDT_WITH_GICP) h->m.emplace<NdtGicpMatcher>();
  else if (type == SM_TYPE_ICP_PM) h->m.emplace<PmMatcher>();
  const int rc = h->m.index() == 0 ? SM_ERR_UNSUPPORTED_TYPE : select_device(device);
  if (rc < 0) { delete h; return rc; }
  h->type = type;
  h->device = device;
  IcpFastMatcher* f = h->icp_chain();
  if (cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
      (f && cudaMallocHost((void**)&f->host_state, sizeof(IcpState)) != cudaSuccess) ||
      cudaHostAlloc((void**)&h->host, sizeof(HostBlock), cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&h->host_dev, h->host, 0) != cudaSuccess ||
      cudaMallocHost((void**)&h->host_guess, 16 * sizeof(double)) != cudaSuccess) {
    delete h;
    return SM_ERR_CUDA;
  }
  h->stream = h->own_stream;
  for (int i = 0; i < 4; ++i) { cudaEventCreate(&h->ev[i]); cudaEventCreate(&h->ev_up[i]); }
  *out = h;
  return SM_OK;
}

int sm_destroy(sm_handle* h) {
  if (!h) return SM_OK;
  cudaSetDevice(h->device);
  if (h->stream) cudaStreamSynchronize(h->stream);
  delete h;
  return SM_OK;
}

int sm_get_type(const sm_handle* h) { return h ? h->type : 0; }

int sm_set_stream(sm_handle* h, void* cuda_stream) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  h->stream = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
  return SM_OK;
}

int sm_set_option(sm_handle* h, const char* name, const char* text) {
  if (!h || !name || !text) return SM_ERR_BAD_ARGUMENT;
  const OptionTable t = options_of(h);
  for (const OptionDef* d = t.begin; d != t.end; ++d) {
    if (strcmp(d->name, name) != 0) continue;
    char* v = t.base + d->offset;
    switch (d->kind) {
      case kOptInt: *reinterpret_cast<int32_t*>(v) = (int32_t)strtol(text, nullptr, 10); break;
      case kOptFloat: *reinterpret_cast<float*>(v) = strtof(text, nullptr); break;
      case kOptDouble: *reinterpret_cast<double*>(v) = strtod(text, nullptr); break;
      case kOptBool: *reinterpret_cast<bool*>(v) = as_bool(text); break;
    }
    // type 1 keeps the filtered reading cloud until the source changes; a new filter option must filter it anew
    PmMatcher* pm = h->as<PmMatcher>();
    if (pm && (strcmp(name, "reading_sample_prob") == 0 || strcmp(name, "sample_seed") == 0)) pm->src_dirty = true;
    if (pm && strcmp(name, "sample_seed") == 0) pm->rand_position = 0;   // srand restarts the rand() stream
    return SM_OK;
  }
  return fail(h, SM_ERR_UNKNOWN_OPTION, std::string("Init an unknown option of this matcher! ") + name);
}

int sm_set_inner_compensation(sm_handle* h, int32_t enable) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (IcpFastMatcher* f = h->as<IcpFastMatcher>()) f->inner_compensation = enable != 0;   // the other types ignore it
  return SM_OK;
}

int sm_set_icp_error_minimizer(sm_handle* h, int32_t minimizer) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  IcpFastMatcher* f = h->icp_chain();
  if (!f) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "SetErrorMinimizer: IcpFast (type 6) and IcpUsingPointMatcher (type 1) only");
  if (minimizer < SM_ICP_POINT_TO_PLANE || minimizer > SM_ICP_POINT_TO_POINT)
    return fail(h, SM_ERR_BAD_ARGUMENT, "SetErrorMinimizer: minimizer must be 0..1");
  f->error_minimizer = minimizer;
  return SM_OK;
}

int sm_set_pm_surface_normals(sm_handle* h, int32_t mode) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  PmMatcher* pm = h->as<PmMatcher>();
  if (!pm) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "SetSurfaceNormals: IcpUsingPointMatcher (type 1) only");
  if (mode < SM_PM_NORMALS_LEAST_SQUARES || mode > SM_PM_NORMALS_EIGENVECTOR)
    return fail(h, SM_ERR_BAD_ARGUMENT, "SetSurfaceNormals: mode must be 0..1");
  if (mode != pm->surface_normals) pm->tgt_dirty = true;   // the filtered reference cloud is built anew
  pm->surface_normals = mode;
  return SM_OK;
}

int sm_set_pm_reading_sampler(sm_handle* h, int32_t mode) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  PmMatcher* pm = h->as<PmMatcher>();
  if (!pm) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "SetReadingSampler: IcpUsingPointMatcher (type 1) only");
  if (mode < SM_PM_SAMPLING_HASH || mode > SM_PM_SAMPLING_GLIBC_RAND)
    return fail(h, SM_ERR_BAD_ARGUMENT, "SetReadingSampler: mode must be 0..1");
  if (mode != pm->reading_sampler) pm->src_dirty = true;   // the filtered reading cloud is built anew
  pm->reading_sampler = mode;
  return SM_OK;
}

int sm_get_pm_rand_position(sm_handle* h, int64_t* position) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  PmMatcher* pm = h->as<PmMatcher>();
  if (!pm) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "GetRandPosition: IcpUsingPointMatcher (type 1) only");
  if (!position) return fail(h, SM_ERR_BAD_ARGUMENT, "GetRandPosition: null output");
  *position = pm->rand_position;
  return SM_OK;
}

int sm_set_pm_rand_position(sm_handle* h, int64_t position) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  PmMatcher* pm = h->as<PmMatcher>();
  if (!pm) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "SetRandPosition: IcpUsingPointMatcher (type 1) only");
  if (position < 0) return fail(h, SM_ERR_BAD_ARGUMENT, "SetRandPosition: the position must be >= 0");
  pm->rand_position = position;
  return SM_OK;
}

int sm_set_ndt_search_method(sm_handle* h, int32_t method) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  NdtMatcher* m = h->as<NdtMatcher>();
  if (!m) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "SetNeighborhoodSearchMethod: registrator::Ndt (type 5) only");
  if (method < SM_NDT_KDTREE || method > SM_NDT_DIRECT1)
    return fail(h, SM_ERR_BAD_ARGUMENT, "SetNeighborhoodSearchMethod: method must be 0..3");
  m->opt.search = method;
  return SM_OK;
}

int sm_print_options(sm_handle* h, char* buf, int64_t buf_len) {
  if (!h || !buf || buf_len <= 0) return SM_ERR_BAD_ARGUMENT;
  std::string out;
  char line[128];
  const OptionTable t = options_of(h);
  for (const OptionDef* d = t.begin; d != t.end; ++d) {
    const char* v = t.base + d->offset;
    switch (d->kind) {
      case kOptInt: snprintf(line, sizeof(line), "%25s -> %d\n", d->name, *reinterpret_cast<const int32_t*>(v)); break;
      case kOptFloat: snprintf(line, sizeof(line), "%25s -> %.6g\n", d->name, *reinterpret_cast<const float*>(v)); break;
      case kOptDouble: snprintf(line, sizeof(line), "%25s -> %.15g\n", d->name, *reinterpret_cast<const double*>(v)); break;
      case kOptBool: snprintf(line, sizeof(line), "%25s -> %s\n", d->name, *reinterpret_cast<const bool*>(v) ? "true" : "false"); break;
    }
    out += line;
  }
  strncpy(buf, out.c_str(), (size_t)buf_len - 1);
  buf[buf_len - 1] = 0;
  return (int)out.size();
}

int sm_set_input_source(sm_handle* h, const double* p, int64_t n) { return set_f64(h, false, false, p, n); }
int sm_set_input_source_device(sm_handle* h, const double* p, int64_t n) { return set_f64(h, false, true, p, n); }
int sm_set_input_target(sm_handle* h, const double* p, const double* nrm, int64_t n) {
  return set_f64(h, true, false, p, n, nrm);
}
int sm_set_input_target_device(sm_handle* h, const double* p, const double* nrm, int64_t n) {
  return set_f64(h, true, true, p, n, nrm);
}

int sm_set_input_source_f32(sm_handle* h, const float* xyz, int64_t n, int64_t stride) {
  return set_input_f32(h, xyz, n, stride, false, false);
}
int sm_set_input_target_f32(sm_handle* h, const float* xyz, int64_t n, int64_t stride) {
  return set_input_f32(h, xyz, n, stride, true, false);
}
int sm_set_input_source_f32_device(sm_handle* h, const float* xyz, int64_t n, int64_t stride) {
  return set_input_f32(h, xyz, n, stride, false, true);
}
int sm_set_input_target_f32_device(sm_handle* h, const float* xyz, int64_t n, int64_t stride) {
  return set_input_f32(h, xyz, n, stride, true, true);
}

int sm_align(sm_handle* h, const double* guess, double* result) {
  if (!h || !guess || !result) return SM_ERR_BAD_ARGUMENT;
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(h, SM_ERR_CUDA, "cudaSetDevice failed");
  if (IcpFastMatcher* m = h->as<IcpFastMatcher>()) return icp_align(h, *m, guess, result);
  if (NdtMatcher* m = h->as<NdtMatcher>()) return ndt_align(h, *m, guess, result);
  if (NdtGicpMatcher* m = h->as<NdtGicpMatcher>()) return ndt_gicp_align(h, *m, guess, result);
  if (PmMatcher* m = h->as<PmMatcher>()) return pm_align(h, *m, guess, result);
  return fail(h, SM_ERR_UNSUPPORTED_TYPE, "matcher type not supported");
}

int sm_align_async(sm_handle* h, const double* guess) {
  if (!h || !guess) return SM_ERR_BAD_ARGUMENT;
  IcpFastMatcher* f = h->as<IcpFastMatcher>();
  if (!f) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "sm_align_async: IcpFast only");
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(h, SM_ERR_CUDA, "cudaSetDevice failed");
  return icp_begin(h, *f, guess);
}

int sm_align_wait(sm_handle* h, double* result) {
  if (!h || !result) return SM_ERR_BAD_ARGUMENT;
  IcpFastMatcher* f = h->as<IcpFastMatcher>();
  if (!f) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "sm_align_wait: IcpFast only");
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(h, SM_ERR_CUDA, "cudaSetDevice failed");
  return icp_end(h, *f, result);
}

int sm_align_batch(sm_handle* const* handles, int32_t n, const double* guesses_16n, double* results_16n,
                   int32_t* rc_n) {
  if (!handles || n < 0 || !guesses_16n || !results_16n || !rc_n) return SM_ERR_BAD_ARGUMENT;
  for (int i = 0; i < n; ++i) if (!handles[i]) return SM_ERR_BAD_ARGUMENT;
  NvtxRange nvtx("sm_align_batch");
  // IcpFast instances: everything is enqueued from this thread before the first result is awaited
  std::vector<int> other;
  for (int i = 0; i < n; ++i) {
    sm_handle* h = handles[i];
    rc_n[i] = 0;
    IcpFastMatcher* f = h->as<IcpFastMatcher>();
    if (!f) { other.push_back(i); continue; }
    if (cudaSetDevice(h->device) != cudaSuccess) { rc_n[i] = fail(h, SM_ERR_CUDA, "cudaSetDevice failed"); continue; }
    rc_n[i] = icp_begin(h, *f, guesses_16n + 16 * (size_t)i);
  }
  // the other matchers drive their optimiser from the host (Newton / BFGS steps with a read-back
  // each): one worker thread per instance, at most 16 at a time, like the reference's thread pool
  std::vector<std::thread> workers;
  std::atomic<int> next(0);
  const int nworkers = (int)other.size() < 16 ? (int)other.size() : 16;
  for (int w = 0; w < nworkers; ++w)
    workers.emplace_back([&]() {
      for (;;) {
        const int k = next.fetch_add(1);
        if (k >= (int)other.size()) break;
        const int i = other[(size_t)k];
        rc_n[i] = sm_align(handles[i], guesses_16n + 16 * (size_t)i, results_16n + 16 * (size_t)i);
      }
    });
  for (int i = 0; i < n; ++i) {
    sm_handle* h = handles[i];
    IcpFastMatcher* f = h->as<IcpFastMatcher>();
    if (!f || rc_n[i] < 0) continue;
    if (cudaSetDevice(h->device) != cudaSuccess) { rc_n[i] = SM_ERR_CUDA; continue; }
    rc_n[i] = icp_end(h, *f, results_16n + 16 * (size_t)i);
  }
  for (std::thread& t : workers) t.join();
  int worst = 0;
  for (int i = 0; i < n; ++i) if (rc_n[i] < worst) worst = rc_n[i];
  return worst < 0 ? worst : SM_OK;
}

int sm_align_pairs(sm_handle* const* handles, int32_t n_handles, const sm_pair* pairs, int32_t n_pairs,
                   double* results_16n, double* scores_n, int32_t* rc_n) {
  if (!handles || n_handles <= 0 || !pairs || n_pairs < 0 || !results_16n || !rc_n) return SM_ERR_BAD_ARGUMENT;
  for (int i = 0; i < n_handles; ++i)   // fail() leaves a null handle alone
    if (!handles[i] || !handles[i]->as<IcpFastMatcher>())
      return fail(handles[i], SM_ERR_UNSUPPORTED_TYPE, "sm_align_pairs: IcpFast only");
  NvtxRange nvtx("sm_align_pairs");
  static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  std::vector<int> in_flight((size_t)n_handles, -1);     // pair index a pipeline is working on
  auto collect = [&](int hi) {
    const int k = in_flight[(size_t)hi];
    if (k < 0) return;
    sm_handle* h = handles[hi];
    cudaSetDevice(h->device);
    rc_n[k] = icp_end(h, *h->as<IcpFastMatcher>(), results_16n + 16 * (size_t)k);
    if (rc_n[k] < 0) cudaStreamSynchronize(h->stream);   // a chunk enqueued before the failure runs out here
    if (scores_n) scores_n[k] = rc_n[k] < 0 ? 0.0 : h->final_score;   // final_score is another pair's
    in_flight[(size_t)hi] = -1;
  };
  for (int k = 0; k < n_pairs; ++k) {
    const int hi = k % n_handles;
    sm_handle* h = handles[hi];
    IcpFastMatcher& f = *h->as<IcpFastMatcher>();
    collect(hi);                                          // the pipeline's previous pair
    const sm_pair& pr = pairs[k];
    rc_n[k] = 0;
    if (scores_n) scores_n[k] = 0.0;
    if (cudaSetDevice(h->device) != cudaSuccess) { rc_n[k] = fail(h, SM_ERR_CUDA, "cudaSetDevice failed"); continue; }
    int rc = icp_check_pair(h, f, pr);                    // a refused pair enqueues nothing
    if (rc < 0) { rc_n[k] = rc; continue; }
    const bool dev = pr.on_device != 0;
    rc = icp_set_target(h, f, pr.target_3xn, pr.target_normals_3xn, pr.n_target, dev, !dev);
    if (rc >= 0) rc = icp_set_source(h, f, pr.source_3xn, pr.n_source, dev, !dev);
    if (rc >= 0) rc = icp_begin(h, f, pr.guess_4x4 ? pr.guess_4x4 : kIdentity);
    if (rc < 0) {                                         // the uploads may still read the caller's arrays
      cudaStreamSynchronize(h->stream);
      rc_n[k] = rc;
      continue;
    }
    in_flight[(size_t)hi] = k;
  }
  for (int hi = 0; hi < n_handles; ++hi) collect(hi);
  int worst = 0;
  for (int k = 0; k < n_pairs; ++k) if (rc_n[k] < worst) worst = rc_n[k];
  return worst < 0 ? worst : SM_OK;
}

double sm_get_fitness_score(const sm_handle* h) { return h ? h->final_score : 0.0; }

int sm_get_align_info(const sm_handle* h, sm_align_info* out) {
  if (!h || !out) return SM_ERR_BAD_ARGUMENT;
  *out = h->info;
  return SM_OK;
}

const char* sm_last_error(const sm_handle* h) { return h ? h->error.c_str() : "null handle"; }


// Diagnostics, not part of include/sm_b200.h: clock64 stamps of the sections of the last
// icp_finish_kernel of the last IcpFast Align (profiles/finish_sections.py).
int sm_debug_icp_stamps(const sm_handle* h, long long* out12) {
  const IcpFastMatcher* f = h ? const_cast<sm_handle*>(h)->icp_chain() : nullptr;
  if (!f || !out12 || !f->host_state) return SM_ERR_BAD_ARGUMENT;
  for (int i = 0; i < 12; ++i) out12[i] = f->host_state->stamps[i];
  return SM_OK;
}

int sm_calculate_normals(int device, const double* points, int64_t n, double* out_points,
                         double* out_normals, int64_t* m_out) {
  return sm_calculate_normals_ordered(device, points, n, SM_NORMALS_ORDER_INDEX, out_points, out_normals, m_out);
}

int sm_calculate_normals_ordered(int device, const double* points, int64_t n, int32_t order, double* out_points,
                                 double* out_normals, int64_t* m_out) {
  if (!points || !out_points || !out_normals || !m_out || n <= 0 || n > (1 << 30) ||
      (order != SM_NORMALS_ORDER_INDEX && order != SM_NORMALS_ORDER_NTH_ELEMENT))
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  cudaStream_t s = nullptr;
  NormalsPipeline np;
  DevBuf stage;
  SMB_RC(np.reserve((int)n));
  SMB_RC(upload_soa(points, n, false, stage, np.input(), np.stride, s));
  uint32_t m = 0;
  if (order == SM_NORMALS_ORDER_NTH_ELEMENT) SMB_RC(np.run_nth_element((int)n, s, &m));
  else SMB_RC(np.run((int)n, kNormalsLeastSquares, s, &m));
  if (m > 0) {
    SMB_CUDA_OK(cudaMemcpyAsync(out_points, np.points(), (size_t)3 * m * sizeof(double), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaMemcpyAsync(out_normals, np.normals(), (size_t)3 * m * sizeof(double), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaStreamSynchronize(s));
  }
  *m_out = (int64_t)m;
  return SM_OK;
}

// sm_knn1 / sm_debug_knn1_batched: host clouds, the default stream, synchronised before returning
static int knn1_impl(int device, const double* target, int64_t nt, const double* query, int64_t nq,
                     double epsilon, int bucket, int queries_per_cta, int32_t* ids, double* d2) {
  // buckets hold at most 8 points (one padded bucket = x[8] y[8] z[8]); libnabo's default is 8
  if (!target || !query || nt <= 0 || nt > (1 << 30) || nq < 0 || nq > (1 << 30) || bucket < 2 || bucket > 8 ||
      !(epsilon >= 0.0))
    return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  if (kd_num_levels((int)nt, bucket) > 24) return SM_ERR_BAD_ARGUMENT;
  cudaStream_t s = nullptr;
  DevBuf ids_d, d2_d, items;
  SMB_RC(ids_d.reserve((size_t)(nq > 0 ? nq : 1) * sizeof(int32_t)));
  SMB_RC(d2_d.reserve((size_t)(nq > 0 ? nq : 1) * sizeof(double)));
  SMB_RC(items.reserve(knn_items_bytes((int)nq)));
  const auto search = [&](const KdCompact& kc, const double* q, int64_t qs) -> int {
    SMB_RC(knn_query(kc, q, qs, (int)nq, (1.0 + epsilon) * (1.0 + epsilon), (int32_t*)ids_d.p, (double*)d2_d.p, s,
                     queries_per_cta, (int4*)items.p));
    SMB_CUDA_OK(cudaMemcpyAsync(ids, ids_d.p, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaMemcpyAsync(d2, d2_d.p, (size_t)nq * sizeof(double), cudaMemcpyDeviceToHost, s));
    return SM_OK;
  };
  return knn_on_target(target, nt, query, nq, bucket, false, s, search);
}

int sm_knn1(int device, const double* target, int64_t nt, const double* query, int64_t nq,
            double epsilon, int bucket, int32_t* ids, double* d2) {
  return knn1_impl(device, target, nt, query, nq, epsilon, bucket, 0, ids, d2);
}

// test hook (include/sm_b200_debug.h): the same search with the launch shape and warp-level scheduling the
// ICP iteration uses with many alignments in flight
int sm_debug_knn1_batched(int device, const double* target, int64_t nt, const double* query, int64_t nq,
                          double epsilon, int bucket, int32_t queries_per_cta, int32_t* ids, double* d2) {
  if (queries_per_cta < 0 || queries_per_cta > (1 << 20)) return SM_ERR_BAD_ARGUMENT;
  return knn1_impl(device, target, nt, query, nq, epsilon, bucket, queries_per_cta, ids, d2);
}

// sm_knn / sm_knn_device: the tree of sm_knn1, then knn_k_query.  Host clouds go through a staging buffer on the
// default stream; device clouds are read in place and the results written to the caller's buffers on its stream.
// Either way the stream is synchronised before returning.
static int knn_impl(int device, const double* target, int64_t nt, const double* query, int64_t nq, int32_t k,
                    double epsilon, double max_radius, uint32_t flags, int bucket, int32_t* ids, double* d2,
                    bool on_device, cudaStream_t s) {
  if (!target || !query || !ids || !d2 || nt <= 0 || nt > (1 << 30) || nq < 0 || nq > (1 << 30) || k < 1 ||
      k > 64 || !(epsilon >= 0.0) || !(max_radius >= 0.0) || bucket < 2 || bucket > 8 ||
      (flags & ~(uint32_t)(SM_KNN_ALLOW_SELF_MATCH | SM_KNN_SORT_RESULTS)) != 0u)
    return SM_ERR_BAD_ARGUMENT;
  if (kd_num_levels((int)nt, bucket) > 24) return SM_ERR_BAD_ARGUMENT;
  SMB_RC(select_device(device));
  DevBuf ids_d, d2_d;
  if (!on_device) {
    const size_t n_out = (size_t)(nq > 0 ? nq : 1) * (size_t)k;
    SMB_RC(ids_d.reserve(n_out * sizeof(int32_t)));
    SMB_RC(d2_d.reserve(n_out * sizeof(double)));
  }
  const auto search = [&](const KdCompact& kc, const double* q, int64_t qs) -> int {
    int32_t* ids_out = on_device ? ids : (int32_t*)ids_d.p;
    double* d2_out = on_device ? d2 : (double*)d2_d.p;
    SMB_RC(knn_k_query(kc, q, qs, (int)nq, k, (1.0 + epsilon) * (1.0 + epsilon), max_radius * max_radius,
                       (flags & SM_KNN_ALLOW_SELF_MATCH) != 0u, ids_out, d2_out, s));
    if (!on_device) {
      SMB_CUDA_OK(cudaMemcpyAsync(ids, ids_d.p, (size_t)nq * k * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
      SMB_CUDA_OK(cudaMemcpyAsync(d2, d2_d.p, (size_t)nq * k * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    return SM_OK;
  };
  return knn_on_target(target, nt, query, nq, bucket, on_device, s, search);
}

int sm_knn(int device, const double* target_3xn, int64_t n_target, const double* query_3xn, int64_t n_query,
           int32_t k, double epsilon, double max_radius, uint32_t flags, int bucket_size, int32_t* ids,
           double* dists2) {
  return knn_impl(device, target_3xn, n_target, query_3xn, n_query, k, epsilon, max_radius, flags, bucket_size, ids,
                  dists2, false, nullptr);
}

int sm_knn_device(int device, const double* target_3xn, int64_t n_target, const double* query_3xn, int64_t n_query,
                  int32_t k, double epsilon, double max_radius, uint32_t flags, int bucket_size, int32_t* ids,
                  double* dists2, void* cuda_stream) {
  return knn_impl(device, target_3xn, n_target, query_3xn, n_query, k, epsilon, max_radius, flags, bucket_size, ids,
                  dists2, true, (cudaStream_t)cuda_stream);
}

}  // extern "C"
