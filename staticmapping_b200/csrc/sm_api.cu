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
#include <vector>

#include <nvtx3/nvToolsExt.h>

#include "common.cuh"
#include "icp_dev.cuh"
#include "kernels.h"
#include "linalg_dev.cuh"
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

// ---- reading filter of the IcpUsingPointMatcher stand-in (see pm_align) ----------------------
__device__ __forceinline__ bool pm_keep(uint32_t i, uint32_t seed, uint32_t thresh, bool all) {
  uint32_t x = i * 0x9E3779B9u + seed;
  x ^= x >> 16; x *= 0x85EBCA6Bu; x ^= x >> 13; x *= 0xC2B2AE35u; x ^= x >> 16;
  return all || x < thresh;
}

__global__ void __launch_bounds__(256)
pm_sample_count_kernel(int n, uint32_t seed, uint32_t thresh, int all, uint32_t* __restrict__ block_cnt) {
  __shared__ uint32_t wc[8];
  const int i = blockIdx.x * 256 + threadIdx.x;
  const bool k = i < n && pm_keep((uint32_t)i, seed, thresh, all != 0);
  const uint32_t m = __ballot_sync(0xffffffffu, k);
  if ((threadIdx.x & 31) == 0) wc[threadIdx.x >> 5] = __popc(m);
  __syncthreads();
  if (threadIdx.x == 0) { uint32_t t = 0; for (int w = 0; w < 8; ++w) t += wc[w]; block_cnt[blockIdx.x] = t; }
}

// kept points, original order, as 3xN column-major doubles (EigenPointCloud::FromPointCloud)
__global__ void __launch_bounds__(256)
pm_sample_scatter_kernel(const float* __restrict__ pts, int n, uint32_t seed, uint32_t thresh, int all,
                         const uint32_t* __restrict__ block_off, double* __restrict__ out) {
  __shared__ uint32_t wc[8];
  const int i = blockIdx.x * 256 + threadIdx.x;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const bool k = i < n && pm_keep((uint32_t)i, seed, thresh, all != 0);
  const uint32_t m = __ballot_sync(0xffffffffu, k);
  if (lane == 0) wc[w] = __popc(m);
  __syncthreads();
  uint32_t off = block_off[blockIdx.x];
  for (int ww = 0; ww < w; ++ww) off += wc[ww];
  if (k) {
    const int64_t d = off + __popc(m & ((1u << lane) - 1u));
    out[3 * d] = (double)pts[3 * (int64_t)i];
    out[3 * d + 1] = (double)pts[3 * (int64_t)i + 1];
    out[3 * d + 2] = (double)pts[3 * (int64_t)i + 2];
  }
}

// ---- score of the IcpUsingPointMatcher stand-in (icp_pointmatcher.cc:131-148): the UNFILTERED
// reading cloud moved by the result is matched against the UNFILTERED reference (same k-d tree
// matcher, eps 3.16), trimmed at the 0.7 quantile, and the mean kept distance goes into exp(-x)
__global__ void __launch_bounds__(256)
pm_score_knn_kernel(const float* __restrict__ src, int n, const double* __restrict__ T, const KdNode* __restrict__ nodes,
                    const BucketPoint* __restrict__ bpts, double max_error2, uint64_t* __restrict__ keys,
                    uint32_t* __restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = (double)src[3 * (int64_t)i], y = (double)src[3 * (int64_t)i + 1], z = (double)src[3 * (int64_t)i + 2];
  double px, py, pz;
  dev::transform_point(T, x, y, z, px, py, pz);
  int slot; double d2;
  dev::knn1(nodes, bpts, px, py, pz, max_error2, slot, d2);
  keys[i] = (uint64_t)__double_as_longlong(d2);     // non-negative doubles sort like their bit patterns; +inf = no match
  vals[i] = (uint32_t)i;
}

// keys sorted ascending; out[0] = mean of sqrt(d2) over the kept matches, out[1] = kept, out[2] = valid
__global__ void __launch_bounds__(1024)
pm_score_reduce_kernel(const uint64_t* __restrict__ keys, int n, float ratio, double* __restrict__ out) {
  __shared__ double red[32];
  __shared__ int s_kept, s_valid;
  const uint64_t inf_bits = 0x7ff0000000000000ull;
  if (threadIdx.x == 0) {
    int lo = 0, hi = n;                                // first index with key >= +inf
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] < inf_bits) lo = mid + 1; else hi = mid; }
    const int valid = lo;
    int kept = 0;
    if (valid > 0) {
      const double q = (double)ratio;                  // GetDistsQuantile, as icp_fast.cc:82-89
      int qi = (q == 1.0) ? valid - 1 : (int)((double)valid * q);
      if (qi > valid - 1) qi = valid - 1;
      const uint64_t limit = keys[qi];
      lo = qi; hi = valid;                             // first index with key > limit
      while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] <= limit) lo = mid + 1; else hi = mid; }
      kept = lo;
    }
    s_kept = kept; s_valid = valid;
  }
  __syncthreads();
  const int kept = s_kept;
  double v = 0.0;
  for (int i = threadIdx.x; i < kept; i += 1024) v += sqrt(__longlong_as_double((long long)keys[i]));
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < 32; ++w) t += red[w];
    out[0] = kept > 0 ? t / (double)kept : 0.0;
    out[1] = (double)kept;
    out[2] = (double)s_valid;
  }
}

__global__ void debug_solve6_kernel(const double* __restrict__ A, const double* __restrict__ b, double* __restrict__ x,
                                    int* __restrict__ path) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *path = la::solve_possibly_underdetermined(A, b, x);
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

// A captured launch sequence, replayed while the key (all pointers and sizes baked into the
// kernel arguments) is unchanged: one cudaGraphLaunch instead of ~100 kernel launches.
struct GraphCache {
  cudaGraphExec_t exec = nullptr;
  std::string key;
  ~GraphCache() { reset(); }
  void reset() { if (exec) cudaGraphExecDestroy(exec); exec = nullptr; key.clear(); }
};

}  // namespace
}  // namespace smb

using namespace smb;

// Everything a handle owns is released by its destructor; each group of device buffers is used
// by one matcher type only, so a handle allocates one group (plus the shared kdws).
struct sm_handle {
  int type = 0;
  int device = 0;
  cudaStream_t stream = nullptr;      // stream in use
  cudaStream_t own_stream = nullptr;  // created by sm_create
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t ev_up[4] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<cudaEvent_t> prof_events;
  double* host_guess = nullptr;    // pinned, 16 doubles
  double* host_sums = nullptr;     // pinned + mapped, 64 doubles; word 60 doubles as the GICP evaluation flag
  double* host_sums_dev = nullptr; // its device view
  std::string error;
  double final_score = 0.0;
  sm_align_info info;
  int64_t n_source = 0, n_target = 0;
  bool has_source = false, has_target = false;
  IcpOptions icp;
  bool inner_compensation = false;  // Interface::EnableInnerCompensation; only IcpFast reads it
  ndt::Options ndt;
  NdtGicpOptions ng;
  DevBuf kdws;                     // k-d tree build workspace of every tree below

  // IcpFast, and the ICP chain of type 1: SoA double clouds, the tree, the iteration buffers
  struct {
    DevBuf stage, stage_src, stage_tgt, stage_nrm, tgt_raw, tgt, nrm, src_raw, src0, src_g0, src_sort, slot, d2,
        hist, cand_terms, cand_key, cand_cnt, partials, mean_partials, state, guess;
    DevBuf deskewed;                 // [3][sstride]: the source of the iteration, with inner compensation only
    KdCompactTree tree;
    int64_t sstride = 0, tstride = 0;
    bool up_src = false, up_tgt = false;
    IcpState* host_state = nullptr;  // pinned
    GraphCache g_prologue, g_iterations;
    // in-flight Align (sm_align_async .. sm_align_wait)
    struct {
      IcpBuffers b; IcpParams p; KdWorkspace ws; std::string key;
      double* deskewed = nullptr;
      bool graphs = false, active = false;
      int enqueued = 0, launches = 0, max_it = 0;
    } run;
  } fast;

  // Ndt, NdtWithGicp and type 1: packed float clouds (12 bytes per point), the NDT workspace and the
  // target's tree (fitness scores, GICP correspondences, the type-1 score)
  struct {
    DevBuf src, tgt, ndt_ws;
    FloatTree target_tree;
  } f32;

  // NdtWithGicp
  struct {
    DevBuf src_filt, tgt_filt, approx_ws, cov_s, cov_t, maha, match, partials, counter;
    FloatTree source_tree;
    long long seq = 0;
  } ndt_gicp;

  // IcpUsingPointMatcher stand-in (type 1): raw float clouds -> filtered double clouds.  The normals
  // pipeline has its own k-d workspace: h->kdws.p is part of the IcpFast graph keys.
  struct {
    int64_t n_src = 0, n_tgt = 0;
    bool src_dirty = false, tgt_dirty = false, score_tree_dirty = true;
    NormalsPipeline normals;
    DevBuf cnt, src, score_buf;       // sampling counts, the sampled source, the score's sort and I/O
  } pm;

  ~sm_handle() {
    for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : ev_up) if (e) cudaEventDestroy(e);
    for (cudaEvent_t e : prof_events) cudaEventDestroy(e);
    if (fast.host_state) cudaFreeHost(fast.host_state);
    if (host_sums) cudaFreeHost(host_sums);
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
  switch (h->type) {
    case SM_TYPE_NDT: return {std::begin(kNdtOptions), std::end(kNdtOptions), reinterpret_cast<char*>(&h->ndt)};
    case SM_TYPE_NDT_WITH_GICP:
      return {std::begin(kNdtGicpOptions), std::end(kNdtGicpOptions), reinterpret_cast<char*>(&h->ng)};
    default: return {std::begin(kIcpOptions), std::end(kIcpOptions), reinterpret_cast<char*>(&h->icp)};  // IcpFast, type 1
  }
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
int load_cloud(sm_handle* h, const double* pts, int64_t n, bool on_device, DevBuf& soa,
               int64_t stride, DevBuf* own_stage = nullptr) {
  H_RC(soa.reserve((size_t)(3 * stride) * sizeof(double)));
  H_RC(upload_soa(pts, n, on_device, own_stage ? *own_stage : h->fast.stage, (double*)soa.p, stride, h->stream));
  if (!on_device && !own_stage) H_CUDA(cudaStreamSynchronize(h->stream));  // the shared stage buffer is reused
  return 0;
}

int set_source(sm_handle* h, const double* pts, int64_t n, bool on_device, bool async = false) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (!pts || n <= 0) return fail(h, SM_ERR_MISSING_INPUT, "SetInputSource: empty cloud");
  if (n > (1 << 30)) return fail(h, SM_ERR_BAD_ARGUMENT, "SetInputSource: too many points");
  H_CUDA(cudaSetDevice(h->device));
  H_CUDA(cudaEventRecord(h->ev_up[0], h->stream));
  auto& f = h->fast;
  f.sstride = pad64(n);
  H_RC(load_cloud(h, pts, n, on_device, f.src_raw, f.sstride, async ? &f.stage_src : nullptr));
  H_CUDA(cudaEventRecord(h->ev_up[1], h->stream));
  f.up_src = true;
  h->n_source = n;
  h->has_source = true;
  return 0;
}

int set_target(sm_handle* h, const double* pts, const double* nrm, int64_t n, bool on_device, bool async = false) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (!pts || n <= 0) return fail(h, SM_ERR_MISSING_INPUT, "SetInputTarget: empty cloud");
  if (h->type == SM_TYPE_FAST_ICP && !nrm)
    return fail(h, SM_ERR_MISSING_INPUT, "SetInputTarget: IcpFast target needs normals");
  if (n > (1 << 30)) return fail(h, SM_ERR_BAD_ARGUMENT, "SetInputTarget: too many points");
  H_CUDA(cudaSetDevice(h->device));
  H_CUDA(cudaEventRecord(h->ev_up[2], h->stream));
  auto& f = h->fast;
  f.tstride = pad64(n);
  H_RC(load_cloud(h, pts, n, on_device, f.tgt_raw, f.tstride, async ? &f.stage_tgt : nullptr));
  if (nrm) H_RC(load_cloud(h, nrm, n, on_device, f.nrm, f.tstride, async ? &f.stage_nrm : nullptr));
  H_CUDA(cudaEventRecord(h->ev_up[3], h->stream));
  f.up_tgt = true;
  h->n_target = n;
  h->has_target = true;
  return 0;
}

int ndt_align(sm_handle* h, const double* guess, double* result);
int ndt_gicp_align(sm_handle* h, const double* guess, double* result);
int pm_align(sm_handle* h, const double* guess, double* result);
int build_tree_f32(sm_handle* h, const float* pts, int n, FloatTree& t) {
  if (kd_num_levels(n, 8) > 24) return fail(h, SM_ERR_BAD_ARGUMENT, "cloud too large");
  H_RC(t.build(pts, n, h->kdws, h->stream));
  return 0;
}

// one chunk of iterations + the asynchronous read-back of the state record
int icp_enqueue_chunk(sm_handle* h) {
  auto& f = h->fast;
  auto& r = f.run;
  const IcpParams& p = r.p;
  const int chunk = p.disable_convergence ? (r.max_it - r.enqueued)
                                          : ((r.max_it - r.enqueued) < 8 ? (r.max_it - r.enqueued) : 8);
  cudaEvent_t* evs = nullptr;
  if (h->icp.profile_kernels) {
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
  r.launches += (p.inner_compensation ? 4 : 3) * chunk;
  H_CUDA(cudaMemcpyAsync(f.host_state, f.state.p, sizeof(IcpState), cudaMemcpyDeviceToHost, h->stream));
  return 0;
}

// IcpFast::Align, first half: everything is enqueued, nothing is waited for
int icp_begin(sm_handle* h, const double* guess) {
  auto& f = h->fast;
  auto& r = f.run;
  r.active = false;
  if (!h->has_source || !h->has_target)
    return fail(h, SM_ERR_MISSING_INPUT, "Align: source/target not set");
  {   // CHECK(quantile >= 0 && quantile <= 1), icp_fast.cc:68
    const float q = h->icp.dist_outlier_ratio;
    if (!(q >= 0.0f && q <= 1.0f)) return fail(h, SM_ERR_BAD_ARGUMENT, "Align: dist_outlier_ratio outside [0, 1] (icp_fast.cc:68)");
    if (!(h->icp.knn_epsilon >= 0.0f)) return fail(h, SM_ERR_BAD_ARGUMENT, "Align: knn_epsilon must be >= 0");
  }
  NvtxRange nvtx_align("IcpFast::Align");
  const int ns = (int)h->n_source, nt = (int)h->n_target;
  const int levels = kd_num_levels(nt, 8);
  const int nb = icp_accum_blocks(ns);
  H_RC(f.tgt.reserve((size_t)(3 * f.tstride) * sizeof(double)));
  H_RC(f.src0.reserve((size_t)(3 * f.sstride) * sizeof(double)));
  H_RC(f.src_g0.reserve((size_t)(3 * f.sstride) * sizeof(double)));
  H_RC(f.src_sort.reserve(RadixPairs::bytes(f.sstride, ns)));
  H_RC(f.tree.reserve(nt, 8, KdCompactTree::kNormals));
  const size_t slot_bytes = (((size_t)ns * sizeof(int32_t) + 64 + 255) / 256) * 256;
  H_RC(f.slot.reserve(slot_bytes + ((size_t)ns + kKnnItemSlack) * sizeof(int4)));
  H_RC(f.d2.reserve((size_t)ns * sizeof(double)));
  H_RC(f.hist.reserve((2 * kHistBins + 64) * sizeof(uint32_t) + 32 * sizeof(double)));
  H_RC(f.cand_terms.reserve((size_t)nb * 512 * 8 * sizeof(double)));
  H_RC(f.cand_key.reserve((size_t)nb * 512 * sizeof(unsigned long long)));
  H_RC(f.cand_cnt.reserve((size_t)nb * sizeof(uint32_t)));
  H_RC(f.partials.reserve((size_t)nb * 32 * sizeof(double)));
  H_RC(f.mean_partials.reserve((size_t)ceil_div(nt, 1024) * 4 * sizeof(double)));
  H_RC(f.state.reserve(sizeof(IcpState)));
  H_RC(f.guess.reserve(16 * sizeof(double)));
  KdWorkspace& ws = r.ws;
  H_RC(ws.carve(h->kdws, nt, 8));

  IcpBuffers& b = r.b;
  b.tgt = (double*)f.tgt.p; b.tgt_raw = (double*)f.tgt_raw.p; b.nrm = (double*)f.nrm.p;
  b.tstride = f.tstride;
  b.nodes = (KdNode*)f.tree.nodes.p; b.leaf_order = (uint32_t*)f.tree.leaf_order.p;
  b.kc = f.tree.view();
  b.src_raw = (double*)f.src_raw.p; b.src0 = (double*)f.src0.p; b.sstride = f.sstride;
  b.src_g0 = (double*)f.src_g0.p;
  b.src_sort.carve(f.src_sort.p, f.sstride);
  b.slot = (int32_t*)f.slot.p;
  b.knn_items = reinterpret_cast<int4*>((char*)f.slot.p + slot_bytes);
  b.d2 = (double*)f.d2.p; b.hist = (uint32_t*)f.hist.p;
  b.hist2 = b.hist + kHistBins;
  b.sums = (double*)(b.hist + 2 * kHistBins + 64);
  b.cand_terms = (double*)f.cand_terms.p;
  b.cand_key = (unsigned long long*)f.cand_key.p; b.cand_cnt = (uint32_t*)f.cand_cnt.p;
  b.partials = (double*)f.partials.p; b.mean_partials = (double*)f.mean_partials.p;
  b.state = (IcpState*)f.state.p;
  IcpParams& p = r.p;
  p.n_source = ns; p.n_target = nt;
  p.max_iteration = h->icp.max_iteration;
  p.dist_outlier_ratio = h->icp.dist_outlier_ratio;
  const double eps = (double)h->icp.knn_epsilon;
  p.max_error2 = (1.0 + eps) * (1.0 + eps);
  p.disable_convergence = h->icp.disable_convergence_check ? 1 : 0;
  p.knn_queries_per_cta = h->icp.knn_queries_per_cta;
  p.tree_levels = levels;
  // EnableInnerCompensation: IcpFast::Align reads it (icp_fast.cc:487, :509); type 1 runs the IcpFast chain but,
  // like IcpUsingPointMatcher, ignores it
  p.inner_compensation = (h->type == SM_TYPE_FAST_ICP && h->inner_compensation) ? 1 : 0;
  r.deskewed = nullptr;
  if (p.inner_compensation) {
    H_RC(f.deskewed.reserve((size_t)(3 * f.sstride) * sizeof(double)));
    r.deskewed = (double*)f.deskewed.p;
  }
  if (levels > 24) return fail(h, SM_ERR_BAD_ARGUMENT, "target too large (tree deeper than 24 levels)");

  memcpy(h->host_guess, guess, 16 * sizeof(double));   // pinned: the caller's array may go away
  H_CUDA(cudaMemcpyAsync(f.guess.p, h->host_guess, 16 * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  H_CUDA(cudaEventRecord(h->ev[0], h->stream));
  r.graphs = h->icp.use_graphs && !h->icp.profile_kernels;
  r.key.clear();
  key_append(r.key, b); key_append(r.key, p); key_append(r.key, f.guess.p); key_append(r.key, h->kdws.p);
  key_append(r.key, r.deskewed);   // p.inner_compensation is part of p
  if (r.graphs) {
    H_RC(run_graphed(h, f.g_prologue, r.key, [&]() {
      return icp_prologue(b, p, (const double*)f.guess.p, ws, f.tree, h->stream);
    }));
  } else {
    H_RC(icp_prologue(b, p, (const double*)f.guess.p, ws, f.tree, h->stream));
  }
  H_CUDA(cudaEventRecord(h->ev[1], h->stream));
  r.launches = 2 + 1 + 24 + levels * 5 + 1 + 1 + 2 + 13;
  r.enqueued = 0;
  r.max_it = p.max_iteration > 0 ? p.max_iteration : 1;
  H_RC(icp_enqueue_chunk(h));
  r.active = true;
  return 0;
}

// second half: wait, continue in chunks while the convergence test has not fired, report
int icp_end(sm_handle* h, double* result) {
  auto& f = h->fast;
  auto& r = f.run;
  if (!r.active) return fail(h, SM_ERR_BAD_ARGUMENT, "sm_align_wait without sm_align_async");
  r.active = false;
  while (true) {
    H_CUDA(cudaStreamSynchronize(h->stream));
    if (f.host_state->done || r.enqueued >= r.max_it) break;
    H_RC(icp_enqueue_chunk(h));
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
  if (h->icp.profile_kernels) {
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

int icp_align(sm_handle* h, const double* guess, double* result) {
  H_RC(icp_begin(h, guess));
  return icp_end(h, result);
}

// ---- IcpUsingPointMatcher stand-in (type 1) ------------------------------------------------
// registrators/icp_pointmatcher.cc:125-247 drives libpointmatcher 1.3.1 (external, float) with
//   reading filter    RandomSampling prob 0.9                      -> pm_sample_* below (a counter
//                     hash instead of std::rand, so the kept set is reproducible)
//   reference filter  SamplingSurfaceNormal knn 7, one point per box -> CalculateNormals, the
//                     reference author's own restatement of that filter (cloud_types.cc:73-144)
//   matcher / outlier filter / minimiser / checkers                 -> the IcpFast chain, which
//                     icp_fast.cc ported from exactly these modules (k-d tree eps 3.16, trim 0.7,
//                     point-to-plane, 4-sample differential checker 0.001 rad / 0.01 m), here in
//                     double, capped at 150 iterations
//   score (:131-148)  unfiltered reading moved by the result vs unfiltered reference, same matcher,
//                     trim 0.7, exp(-mean kept distance); Align() false below 0.6 (:145)
// It is a deterministic equivalent, not a bit-level restatement: libpointmatcher's float
// arithmetic and its rand() stream cannot be pinned from this tree.
int pm_align(sm_handle* h, const double* guess, double* result) {
  if (!h->has_source || !h->has_target || h->pm.n_src <= 0 || h->pm.n_tgt <= 0)
    return fail(h, SM_ERR_MISSING_INPUT, "Align: source/target not set");
  cudaStream_t s = h->stream;
  if (h->pm.tgt_dirty) {
    const int n = (int)h->pm.n_tgt;
    NormalsPipeline& np = h->pm.normals;
    H_RC(np.reserve(n));
    H_RC(ndt_float_to_soa((const float*)h->f32.tgt.p, n, np.input(), np.stride, s));
    uint32_t m = 0;
    H_RC(np.run(n, s, &m));
    if (m == 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: no target point survived the surface-normal filter");
    H_RC(set_target(h, np.points(), np.normals(), (int64_t)m, true));
    h->pm.tgt_dirty = false;
  }
  if (h->pm.src_dirty) {
    const int64_t n = h->pm.n_src;
    const int nb = ceil_div(n, 256);
    H_RC(h->pm.cnt.reserve(((size_t)nb + 8) * sizeof(uint32_t)));
    H_RC(h->pm.src.reserve((size_t)3 * (size_t)n * sizeof(double)));
    const double prob = (double)h->icp.reading_sample_prob;
    const int all = prob >= 1.0 ? 1 : 0;
    const uint32_t thresh = prob <= 0.0 ? 0u : (all ? 0xffffffffu : (uint32_t)(prob * 4294967296.0));
    uint32_t* cnt = (uint32_t*)h->pm.cnt.p;
    H_CUDA(cudaMemsetAsync(cnt + nb, 0, sizeof(uint32_t), s));
    pm_sample_count_kernel<<<nb, 256, 0, s>>>((int)n, (uint32_t)h->icp.sample_seed, thresh, all, cnt);
    radix_scan_kernel_launch(cnt, nb + 1, 1, s);            // exclusive: cnt[nb] = number kept
    pm_sample_scatter_kernel<<<nb, 256, 0, s>>>((const float*)h->f32.src.p, (int)n, (uint32_t)h->icp.sample_seed, thresh,
                                              all, cnt, (double*)h->pm.src.p);
    H_CUDA(cudaGetLastError());
    uint32_t kept = 0;
    H_CUDA(cudaMemcpyAsync(&kept, cnt + nb, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    H_CUDA(cudaStreamSynchronize(s));
    if (kept == 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: the reading filter kept no point");
    H_RC(set_source(h, (const double*)h->pm.src.p, (int64_t)kept, true));
    h->pm.src_dirty = false;
  }
  const int rc = icp_align(h, guess, result);
  h->info.aux[2] = (double)h->n_source;   // reading points after the filter
  h->info.aux[3] = (double)h->n_target;   // reference points after the filter
  if (rc < 0) return rc;
  h->info.aux[0] = h->final_score;        // IcpFast's own score (last iteration, filtered clouds)
  // ---- "compute the final score" (icp_pointmatcher.cc:131-148) -------------------------------
  {
    const int ns = (int)h->pm.n_src, nt = (int)h->pm.n_tgt;
    if (h->pm.score_tree_dirty) {
      H_RC(build_tree_f32(h, (const float*)h->f32.tgt.p, nt, h->f32.target_tree));
      h->pm.score_tree_dirty = false;
    }
    const int64_t st = pad64(ns);
    H_RC(h->pm.score_buf.reserve(256 + RadixPairs::bytes(st, ns)));
    double* Tdev = (double*)h->pm.score_buf.p;      // 16 doubles of pose, 8 of output, then the sort
    double* outdev = Tdev + 16;
    RadixPairs sp;
    sp.carve((char*)h->pm.score_buf.p + 256, st);
    for (int i = 0; i < 16; ++i) h->host_guess[i] = result[i];      // pinned staging
    H_CUDA(cudaMemcpyAsync(Tdev, h->host_guess, 16 * sizeof(double), cudaMemcpyHostToDevice, s));
    const double eps = (double)h->icp.knn_epsilon;
    pm_score_knn_kernel<<<ceil_div(ns, 256), 256, 0, s>>>((const float*)h->f32.src.p, ns, Tdev, (const KdNode*)h->f32.target_tree.nodes.p,
                                                       (const BucketPoint*)h->f32.target_tree.bpts.p, (1.0 + eps) * (1.0 + eps),
                                                       sp.keys[0], sp.vals[0]);
    H_RC(radix_sort_pairs_u64(sp.keys[0], sp.vals[0], sp.keys[1], sp.vals[1], ns, 1, st, sp.scratch, s, 8));
    pm_score_reduce_kernel<<<1, 1024, 0, s>>>(sp.keys[0], ns, h->icp.dist_outlier_ratio, outdev);
    H_CUDA(cudaGetLastError());
    H_CUDA(cudaMemcpyAsync(h->host_sums, outdev, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
    H_CUDA(cudaStreamSynchronize(s));
    if (!(h->host_sums[1] > 0.0)) return fail(h, SM_ERR_NOTHING_TO_MINIMIZE, "Align: no matched point for the score");
    h->final_score = exp(-h->host_sums[0]);
    h->info.aux[1] = h->host_sums[1];     // matches kept by the trim in the score pass
  }
  return h->final_score < (double)h->icp.accept_min_score ? 0 : 1;
}

// ---- Ndt ---------------------------------------------------------------------------------
// the packed float source or target cloud (Ndt, NdtWithGicp, type 1)
int set_input_f32(sm_handle* h, const float* xyz, int64_t n, int64_t stride, bool target, bool on_device) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (!xyz || n <= 0) return fail(h, SM_ERR_MISSING_INPUT, "SetInput: empty cloud");
  if (stride < 12 || n > (1 << 30)) return fail(h, SM_ERR_BAD_ARGUMENT, "SetInput: bad stride / size");
  H_CUDA(cudaSetDevice(h->device));
  DevBuf& dst = target ? h->f32.tgt : h->f32.src;
  H_RC(dst.reserve((size_t)n * 12 + 64));
  H_CUDA(cudaMemcpy2DAsync(dst.p, 12, xyz, (size_t)stride, 12, (size_t)n,
                           on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, h->stream));
  if (!on_device) H_CUDA(cudaStreamSynchronize(h->stream));
  if (target) {
    h->n_target = n; h->has_target = true; h->pm.n_tgt = n; h->pm.tgt_dirty = true; h->pm.score_tree_dirty = true;
  } else {
    h->n_source = n; h->has_source = true; h->pm.n_src = n; h->pm.src_dirty = true;
  }
  return 0;
}

int ndt_eval_sync(sm_handle* h, const float* src, int ns, const NdtEvalParams& P, NdtWorkspace& ws) {
  H_RC(ndt_eval(src, ns, P, ws, h->stream));
  H_CUDA(cudaMemcpyAsync(h->host_sums, ws.sums, 44 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  H_CUDA(cudaStreamSynchronize(h->stream));
  return 0;
}

struct NdtRunOut {
  float final_T[16];
  double fitness = 0, trans_probability = 0, mean_neighbors = 0;
  int iterations = 0, evaluations = 0, launches = 0;
  float ms_grid = 0, ms_iter = 0, ms_fit = 0;
};

// pcl::Registration::getFitnessScore over h->f32.target_tree
int fitness_score(sm_handle* h, const float* src, int ns, const float* tgt, const float* T, NdtWorkspace& ws,
                  double* out) {
  NdtEvalParams P;
  memset(&P, 0, sizeof(P));
  for (int i = 0; i < 16; ++i) P.T[i] = T[i];
  const FloatTree& t = h->f32.target_tree;
  H_RC(ndt_fitness(src, ns, P, (const KdNode*)t.nodes.p, (const BucketPoint*)t.bpts.p, tgt, ws, h->stream));
  H_CUDA(cudaMemcpyAsync(h->host_sums, ws.sums, 2 * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  H_CUDA(cudaStreamSynchronize(h->stream));
  *out = h->host_sums[1] > 0.0 ? h->host_sums[0] / h->host_sums[1] : std::numeric_limits<double>::max();
  return 0;
}

// pcl::Registration::align -> NormalDistributionsTransform::computeTransformation
// (ndt_omp_impl.hpp:81-171) -> getFitnessScore, on device clouds src/tgt (packed float xyz).
int ndt_run(sm_handle* h, const float* src, int ns, const float* tgt, int nt, const ndt::Options& o,
            bool f64_math, const double* guess, NdtRunOut* out) {
  H_RC(h->f32.ndt_ws.reserve(NdtWorkspace::bytes_needed(nt, ns)));
  NdtWorkspace ws;
  ws.carve(h->f32.ndt_ws.p, nt, ns);
  H_CUDA(cudaEventRecord(h->ev[0], h->stream));
  H_RC(ndt_build_grid(tgt, nt, o.resolution, ws, h->stream));        // setInputTarget -> init()
  H_CUDA(cudaEventRecord(h->ev[1], h->stream));
  NdtEvalParams P;
  memset(&P, 0, sizeof(P));
  ndt::gauss_constants(o, &P.gauss_d1, &P.gauss_d2);
  P.radius = o.resolution;
  P.f64_math = f64_math ? 1 : 0;
  // the Newton loop itself is host code shared with the test hook sm_debug_ndt_newton (ndt_host.h newton_loop);
  // one evaluation = computeDerivatives on the device, 44 sums handed back through mapped pinned memory
  ndt::NewtonOut nw;
  int launches = 12 + 12;
  const int nrc = ndt::newton_loop(o, guess, ns, P, [&](const NdtEvalParams& Pe, const double*, double* sums) -> int {
    const int rc = ndt_eval_sync(h, src, ns, Pe, ws);
    if (rc < 0) return rc;
    for (int i = 0; i < 44; ++i) sums[i] = h->host_sums[i];
    launches += 2;
    return 0;
  }, &nw);
  H_RC(nrc);
  float* final_T = out->final_T;
  for (int i = 0; i < 16; ++i) final_T[i] = nw.final_T[i];
  const int nr_iterations = nw.iterations, evals = nw.evaluations;
  const double score = nw.score, nb_sum = nw.nb_sum;
  H_CUDA(cudaEventRecord(h->ev[2], h->stream));
  // getFitnessScore (ndt.cc:60): exact 1-NN over the full target (PCL builds this search
  // tree in setInputTarget; the reference calls that on every Align)
  H_RC(build_tree_f32(h, tgt, nt, h->f32.target_tree));
  H_RC(fitness_score(h, src, ns, tgt, final_T, ws, &out->fitness));
  H_CUDA(cudaEventRecord(h->ev[3], h->stream));
  H_CUDA(cudaEventSynchronize(h->ev[3]));
  out->iterations = nr_iterations;
  out->evaluations = evals;
  out->trans_probability = score / (double)ns;
  out->mean_neighbors = evals ? nb_sum / evals : 0.0;
  out->launches = launches + 24 + kd_num_levels(nt, 8) * 5 + 6;
  cudaEventElapsedTime(&out->ms_grid, h->ev[0], h->ev[1]);
  cudaEventElapsedTime(&out->ms_iter, h->ev[1], h->ev[2]);
  cudaEventElapsedTime(&out->ms_fit, h->ev[2], h->ev[3]);
  return 0;
}

// Ndt::Align (ndt.cc:38-64)
int ndt_align(sm_handle* h, const double* guess, double* result) {
  if (!h->has_source || !h->has_target) {       // ndt.cc:40-42: return false
    for (int i = 0; i < 16; ++i) result[i] = guess[i];
    return 0;
  }
  NdtRunOut r;
  H_RC(ndt_run(h, (const float*)h->f32.src.p, (int)h->n_source, (const float*)h->f32.tgt.p, (int)h->n_target,
               h->ndt, false, guess, &r));
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
// pcl::ApproximateVoxelGrid::filter (ndt_gicp.cc:59-70)
int approx_filter(sm_handle* h, const float* pts, int n, float leaf, DevBuf& out, int* m_out) {
  auto& g = h->ndt_gicp;
  H_RC(g.approx_ws.reserve(approx_ws_bytes(n)));
  H_RC(out.reserve((size_t)n * 12 + 64));
  H_RC(g.counter.reserve(64));
  uint32_t* cnt = (uint32_t*)g.counter.p;
  H_RC(approx_voxel_grid(pts, n, leaf, g.approx_ws.p, (float*)out.p, cnt, h->stream));
  uint32_t m = 0;
  H_CUDA(cudaMemcpyAsync(&m, cnt, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream));
  H_CUDA(cudaStreamSynchronize(h->stream));
  H_RC(approx_voxel_grid_emit(n, (int)m, g.approx_ws.p, (float*)out.p, cnt, h->stream));
  *m_out = (int)m;
  return 0;
}

// GeneralizedIterativeClosestPoint::computeTransformation (gicp_omp_impl.hpp:381-514) with the
// BFGS inner solver on the host; the target tree must be built in h->f32.target_tree.
int gicp_run(sm_handle* h, const float* src, int ns, const float* tgt, int nt, const float* guess,
             const gicp::Options& o, float* final_T, int* iterations, int* bfgs_evals) {
  auto& g = h->ndt_gicp;
  const FloatTree& tt = h->f32.target_tree;
  H_RC(build_tree_f32(h, src, ns, g.source_tree));
  H_RC(g.cov_s.reserve((size_t)ns * 9 * sizeof(double)));
  H_RC(g.cov_t.reserve((size_t)nt * 9 * sizeof(double)));
  H_RC(g.maha.reserve((size_t)ns * 9 * sizeof(double)));
  H_RC(g.match.reserve((size_t)ns * sizeof(int32_t)));
  H_RC(g.partials.reserve((size_t)(gicp_cost_blocks(ns) + 1) * 13 * sizeof(double) + 256));
  H_RC(g.counter.reserve(64));
  double* sums_dev = (double*)g.partials.p + (size_t)gicp_cost_blocks(ns) * 13;
  uint32_t* ticket_dev = (uint32_t*)g.counter.p + 8;
  H_CUDA(cudaMemsetAsync(ticket_dev, 0, sizeof(uint32_t), h->stream));
  *reinterpret_cast<volatile long long*>(h->host_sums + 60) = 0;
  g.seq = 0;
  if (o.k_correspondences <= nt)   // :61-65: otherwise PCL_ERROR and the covariances stay unset
    H_RC(gicp_covariances(tgt, nt, (const KdNode*)tt.nodes.p, (const BucketPoint*)tt.bpts.p, o.gicp_epsilon,
                          (double*)g.cov_t.p, h->stream));
  else H_CUDA(cudaMemsetAsync(g.cov_t.p, 0, (size_t)nt * 9 * sizeof(double), h->stream));
  if (o.k_correspondences <= ns)
    H_RC(gicp_covariances(src, ns, (const KdNode*)g.source_tree.nodes.p,
                          (const BucketPoint*)g.source_tree.bpts.p, o.gicp_epsilon,
                          (double*)g.cov_s.p, h->stream));
  else H_CUDA(cudaMemsetAsync(g.cov_s.p, 0, (size_t)ns * 9 * sizeof(double), h->stream));
  // the outer loop, the BFGS driver and the assembly of f / g from the 13 sums are host code shared with the test
  // hook sm_debug_gicp_outer (gicp_host.h outer_loop); the two callbacks are the device work
  gicp::OuterOut go;
  bool cuda_error = false;
  const int grc = gicp::outer_loop(
      o, guess,
      [&](const float* transformation, const double* R, int* m_out) -> int {
        GicpIterParams IP;
        for (int i = 0; i < 16; ++i) { IP.guess[i] = guess[i]; IP.transformation[i] = transformation[i]; }
        for (int q = 0; q < 9; ++q) IP.R[q] = R[q];
        IP.dist_threshold = o.corr_dist_threshold * o.corr_dist_threshold;
        if (gicp_correspond(src, ns, tgt, IP, (const KdNode*)tt.nodes.p, (const BucketPoint*)tt.bpts.p,
                            (const double*)g.cov_s.p, (const double*)g.cov_t.p, (int32_t*)g.match.p,
                            (double*)g.maha.p, (uint32_t*)g.counter.p, h->stream) != 0) { cuda_error = true; return -1; }
        uint32_t m_u = 0;
        if (cudaMemcpyAsync(&m_u, g.counter.p, sizeof(uint32_t), cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
            cudaStreamSynchronize(h->stream) != cudaSuccess) { cuda_error = true; return -1; }
        *m_out = (int)m_u;
        return 0;
      },
      [&](const float* T, double* S) -> int {
        GicpCostParams CP;
        for (int i = 0; i < 16; ++i) { CP.T[i] = T[i]; CP.base[i] = guess[i]; }
        // the kernel's last block writes the 13 sums and then the sequence word into mapped pinned memory
        volatile long long* flag = reinterpret_cast<volatile long long*>(h->host_sums + 60);
        const long long seq = ++g.seq;
        if (gicp_cost(src, ns, tgt, CP, (const int32_t*)g.match.p, (const double*)g.maha.p,
                      (double*)g.partials.p, sums_dev, ticket_dev, h->host_sums_dev,
                      reinterpret_cast<long long*>(h->host_sums_dev + 60), seq, h->stream) != 0) { cuda_error = true; return -1; }
        for (long spins = 0; *flag != seq; ++spins) {
          if ((spins & 0xfff) == 0xfff && cudaStreamQuery(h->stream) != cudaErrorNotReady) {
            if (*flag == seq) break;
            if (cudaStreamSynchronize(h->stream) != cudaSuccess || *flag != seq) { cuda_error = true; return -1; }   // the kernel failed
          }
        }
        std::atomic_thread_fence(std::memory_order_acquire);
        for (int q = 0; q < 13; ++q) S[q] = h->host_sums[q];
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
int ndt_gicp_align(sm_handle* h, const double* guess, double* result) {
  if (!h->has_source || !h->has_target)
    return fail(h, SM_ERR_MISSING_INPUT, "Align: source/target not set");   // null deref in the reference
  const float* src = (const float*)h->f32.src.p;
  const float* tgt = (const float*)h->f32.tgt.p;
  int ns = (int)h->n_source, nt = (int)h->n_target;
  if (h->ng.using_voxel_filter) {
    auto& g = h->ndt_gicp;
    H_RC(approx_filter(h, src, ns, h->ng.voxel_resolution, g.src_filt, &ns));
    H_RC(approx_filter(h, tgt, nt, h->ng.voxel_resolution, g.tgt_filt, &nt));
    src = (const float*)g.src_filt.p;
    tgt = (const float*)g.tgt_filt.p;
  }
  memset(&h->info, 0, sizeof(h->info));
  h->info.aux[2] = ns; h->info.aux[3] = nt;
  if (ns <= 0 || nt <= 0) return fail(h, SM_ERR_MISSING_INPUT, "Align: empty cloud after the voxel filter");
  float ndt_guess[16];
  for (int i = 0; i < 16; ++i) ndt_guess[i] = (float)guess[i];
  double ndt_score = 0.9;
  if (h->ng.use_ndt) {                    // ndt_gicp.cc:82-88, configuration :44-47
    ndt::Options no;
    no.transformation_epsilon = 0.01; no.step_size = 0.1; no.resolution = 1.0f; no.max_iterations = 35;
    NdtRunOut r;
    H_RC(ndt_run(h, src, ns, tgt, nt, no, true, guess, &r));
    ndt_score = r.fitness;
    for (int i = 0; i < 16; ++i) ndt_guess[i] = r.final_T[i];
    h->info.evaluations = r.evaluations;
    h->info.ms_prologue = r.ms_grid + r.ms_iter + r.ms_fit;
  } else {
    H_RC(build_tree_f32(h, tgt, nt, h->f32.target_tree));
  }
  h->info.aux[0] = ndt_score;
  double icp_score = 10.0;
  if (ndt_score <= 1.0) {                 // :92-103
    float final_T[16];
    int it = 0, evals = 0;
    H_CUDA(cudaEventRecord(h->ev[0], h->stream));
    H_RC(gicp_run(h, src, ns, tgt, nt, ndt_guess, gicp::Options(), final_T, &it, &evals));
    H_RC(h->f32.ndt_ws.reserve(NdtWorkspace::bytes_needed(nt, ns)));
    NdtWorkspace ws;
    ws.carve(h->f32.ndt_ws.p, nt, ns);
    H_RC(fitness_score(h, src, ns, tgt, final_T, ws, &icp_score));
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
  if (type != SM_TYPE_FAST_ICP && type != SM_TYPE_NDT && type != SM_TYPE_NDT_WITH_GICP && type != SM_TYPE_ICP_PM)
    return SM_ERR_UNSUPPORTED_TYPE;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  if (device < 0 || device >= ndev) return SM_ERR_BAD_ARGUMENT;
  sm_handle* h = new sm_handle();
  h->type = type;
  h->device = device;
  if (type == SM_TYPE_ICP_PM) h->icp.max_iteration = 150;   // CounterTransformationChecker, icp_pointmatcher.cc:214
  memset(&h->info, 0, sizeof(h->info));
  if (cudaSetDevice(device) != cudaSuccess ||
      cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMallocHost((void**)&h->fast.host_state, sizeof(IcpState)) != cudaSuccess ||
      cudaHostAlloc((void**)&h->host_sums, 64 * sizeof(double), cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&h->host_sums_dev, h->host_sums, 0) != cudaSuccess ||
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
    return SM_OK;
  }
  return fail(h, SM_ERR_UNKNOWN_OPTION, std::string("Init an unknown option of this matcher! ") + name);
}

int sm_set_inner_compensation(sm_handle* h, int32_t enable) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  h->inner_compensation = enable != 0;
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

int sm_set_input_source(sm_handle* h, const double* p, int64_t n) { return set_source(h, p, n, false); }
int sm_set_input_source_device(sm_handle* h, const double* p, int64_t n) { return set_source(h, p, n, true); }
int sm_set_input_target(sm_handle* h, const double* p, const double* nrm, int64_t n) {
  return set_target(h, p, nrm, n, false);
}
int sm_set_input_target_device(sm_handle* h, const double* p, const double* nrm, int64_t n) {
  return set_target(h, p, nrm, n, true);
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
  if (h->type == SM_TYPE_FAST_ICP) return icp_align(h, guess, result);
  if (h->type == SM_TYPE_NDT) return ndt_align(h, guess, result);
  if (h->type == SM_TYPE_NDT_WITH_GICP) return ndt_gicp_align(h, guess, result);
  if (h->type == SM_TYPE_ICP_PM) return pm_align(h, guess, result);
  return fail(h, SM_ERR_UNSUPPORTED_TYPE, "matcher type not supported");
}

int sm_align_async(sm_handle* h, const double* guess) {
  if (!h || !guess) return SM_ERR_BAD_ARGUMENT;
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(h, SM_ERR_CUDA, "cudaSetDevice failed");
  if (h->type != SM_TYPE_FAST_ICP) return fail(h, SM_ERR_UNSUPPORTED_TYPE, "sm_align_async: IcpFast only");
  return icp_begin(h, guess);
}

int sm_align_wait(sm_handle* h, double* result) {
  if (!h || !result) return SM_ERR_BAD_ARGUMENT;
  if (cudaSetDevice(h->device) != cudaSuccess) return fail(h, SM_ERR_CUDA, "cudaSetDevice failed");
  return icp_end(h, result);
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
    if (h->type != SM_TYPE_FAST_ICP) { other.push_back(i); continue; }
    if (cudaSetDevice(h->device) != cudaSuccess) { rc_n[i] = fail(h, SM_ERR_CUDA, "cudaSetDevice failed"); continue; }
    rc_n[i] = icp_begin(h, guesses_16n + 16 * (size_t)i);
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
    if (h->type != SM_TYPE_FAST_ICP || rc_n[i] < 0) continue;
    if (cudaSetDevice(h->device) != cudaSuccess) { rc_n[i] = SM_ERR_CUDA; continue; }
    rc_n[i] = icp_end(h, results_16n + 16 * (size_t)i);
  }
  for (std::thread& t : workers) t.join();
  int worst = 0;
  for (int i = 0; i < n; ++i) if (rc_n[i] < worst) worst = rc_n[i];
  return worst < 0 ? worst : SM_OK;
}

int sm_align_pairs(sm_handle* const* handles, int32_t n_handles, const sm_pair* pairs, int32_t n_pairs,
                   double* results_16n, double* scores_n, int32_t* rc_n) {
  if (!handles || n_handles <= 0 || !pairs || n_pairs < 0 || !results_16n || !rc_n) return SM_ERR_BAD_ARGUMENT;
  for (int i = 0; i < n_handles; ++i)
    if (!handles[i] || handles[i]->type != SM_TYPE_FAST_ICP) return SM_ERR_UNSUPPORTED_TYPE;
  NvtxRange nvtx("sm_align_pairs");
  static const double kIdentity[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
  std::vector<int> in_flight((size_t)n_handles, -1);     // pair index a pipeline is working on
  auto collect = [&](int hi) {
    const int k = in_flight[(size_t)hi];
    if (k < 0) return;
    sm_handle* h = handles[hi];
    cudaSetDevice(h->device);
    rc_n[k] = icp_end(h, results_16n + 16 * (size_t)k);
    if (scores_n) scores_n[k] = h->final_score;
    in_flight[(size_t)hi] = -1;
  };
  for (int k = 0; k < n_pairs; ++k) {
    const int hi = k % n_handles;
    sm_handle* h = handles[hi];
    collect(hi);                                          // the pipeline's previous pair
    const sm_pair& pr = pairs[k];
    rc_n[k] = 0;
    if (scores_n) scores_n[k] = 0.0;
    if (cudaSetDevice(h->device) != cudaSuccess) { rc_n[k] = fail(h, SM_ERR_CUDA, "cudaSetDevice failed"); continue; }
    const bool dev = pr.on_device != 0;
    int rc = set_target(h, pr.target_3xn, pr.target_normals_3xn, pr.n_target, dev, !dev);
    if (rc >= 0) rc = set_source(h, pr.source_3xn, pr.n_source, dev, !dev);
    if (rc >= 0) rc = icp_begin(h, pr.guess_4x4 ? pr.guess_4x4 : kIdentity);
    if (rc < 0) { rc_n[k] = rc; continue; }
    in_flight[(size_t)hi] = k;
  }
  for (int hi = 0; hi < n_handles; ++hi) collect(hi);
  int worst = 0;
  for (int k = 0; k < n_pairs; ++k) if (rc_n[k] < worst) worst = rc_n[k];
  return worst < 0 ? worst : SM_OK;
}

int sm_debug_solve6(int device, const double* A, const double* b, double* x, int32_t* path) {
  if (!A || !b || !x || !path) return SM_ERR_BAD_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  SMB_CUDA_OK(cudaSetDevice(device));
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
  NdtEvalParams P;
  memset(&P, 0, sizeof(P));
  ndt::gauss_constants(o, &P.gauss_d1, &P.gauss_d2);
  P.radius = o.resolution;
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

// test hook: the voxel index of a point as the three voxelisations compute it, compiled for the host
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
  NdtEvalParams P;
  memset(&P, 0, sizeof(P));
  ndt::gauss_constants(o, &P.gauss_d1, &P.gauss_d2);
  ndt::angle_tables(p6, &P);
  ndt::transform_from_p(p6, P.T);
  P.radius = resolution;
  P.f64_math = f64_math ? 1 : 0;
  ndt_debug_term_host(P, x_orig, x_trans, mean3, icov9, out43);
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
      ndt::gauss_constants(o, &out[0], &out[1]);
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
  if (!h || !out12 || !h->fast.host_state) return SM_ERR_BAD_ARGUMENT;
  for (int i = 0; i < 12; ++i) out12[i] = h->fast.host_state->stamps[i];
  return SM_OK;
}

int sm_calculate_normals(int device, const double* points, int64_t n, double* out_points,
                         double* out_normals, int64_t* m_out) {
  if (!points || !out_points || !out_normals || !m_out || n <= 0 || n > (1 << 30))
    return SM_ERR_BAD_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  SMB_CUDA_OK(cudaSetDevice(device));
  cudaStream_t s = nullptr;
  NormalsPipeline np;
  DevBuf stage;
  SMB_RC(np.reserve((int)n));
  SMB_RC(upload_soa(points, n, false, stage, np.input(), np.stride, s));
  uint32_t m = 0;
  SMB_RC(np.run((int)n, s, &m));
  if (m > 0) {
    SMB_CUDA_OK(cudaMemcpyAsync(out_points, np.points(), (size_t)3 * m * sizeof(double), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaMemcpyAsync(out_normals, np.normals(), (size_t)3 * m * sizeof(double), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaStreamSynchronize(s));
  }
  *m_out = (int64_t)m;
  return SM_OK;
}

static int knn1_impl(int device, const double* target, int64_t nt, const double* query, int64_t nq,
                     double epsilon, int bucket, int queries_per_cta, int32_t* ids, double* d2);

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

static int knn1_impl(int device, const double* target, int64_t nt, const double* query, int64_t nq,
                     double epsilon, int bucket, int queries_per_cta, int32_t* ids, double* d2) {
  // buckets hold at most 8 points (one padded bucket = x[8] y[8] z[8]); libnabo's default is 8
  if (!target || !query || nt <= 0 || nt > (1 << 30) || nq < 0 || nq > (1 << 30) || bucket < 2 || bucket > 8 ||
      !(epsilon >= 0.0))
    return SM_ERR_BAD_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) return SM_ERR_NO_DEVICE;
  SMB_CUDA_OK(cudaSetDevice(device));
  cudaStream_t s = nullptr;
  const int64_t ts = pad64(nt), qs = pad64(nq > 0 ? nq : 1);
  const int levels = kd_num_levels((int)nt, bucket);
  if (levels > 24) return SM_ERR_BAD_ARGUMENT;
  DevBuf stage, tgt, qry, kdws, ids_d, d2_d, items;
  KdCompactTree tree;
  SMB_RC(stage.reserve((size_t)3 * (size_t)(nt > nq ? nt : nq) * sizeof(double)));   // shared by both uploads
  SMB_RC(tgt.reserve((size_t)3 * ts * sizeof(double)));
  SMB_RC(qry.reserve((size_t)3 * qs * sizeof(double)));
  SMB_RC(tree.reserve((int)nt, bucket, KdCompactTree::kIds));
  KdWorkspace ws;
  SMB_RC(ws.carve(kdws, (int)nt, bucket));
  SMB_RC(ids_d.reserve((size_t)(nq > 0 ? nq : 1) * sizeof(int32_t)));
  SMB_RC(d2_d.reserve((size_t)(nq > 0 ? nq : 1) * sizeof(double)));
  SMB_RC(items.reserve(((size_t)nq + kKnnItemSlack) * sizeof(int4)));
  SMB_RC(upload_soa(target, nt, false, stage, (double*)tgt.p, ts, s));
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  SMB_RC(tree.build((const double*)tgt.p, nullptr, ts, (int)nt, bucket, ws, s));
  if (nq > 0) {
    SMB_RC(upload_soa(query, nq, false, stage, (double*)qry.p, qs, s));
    SMB_RC(knn_query(tree.view(), (const double*)qry.p, qs, (int)nq, (1.0 + epsilon) * (1.0 + epsilon), (int32_t*)ids_d.p,
                     (double*)d2_d.p, s, queries_per_cta, (int4*)items.p));
    SMB_CUDA_OK(cudaMemcpyAsync(ids, ids_d.p, (size_t)nq * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    SMB_CUDA_OK(cudaMemcpyAsync(d2, d2_d.p, (size_t)nq * sizeof(double), cudaMemcpyDeviceToHost, s));
  }
  SMB_CUDA_OK(cudaStreamSynchronize(s));
  return SM_OK;
}

}  // extern "C"
