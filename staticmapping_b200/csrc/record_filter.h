// The C handle core of the filters over records (sm_filter_chain in filters.cu, sm_statistic_removal in
// statistic_removal.cu, sm_ground_removal in ground_removal.cu): each handle derives from RecordFilter and adds its
// filter's state.
#ifndef SM_B200_RECORD_FILTER_H_
#define SM_B200_RECORD_FILTER_H_

#include <stdarg.h>
#include <stdio.h>

#include "kernels.h"

namespace smb {

// the argument check of the run entry points: n in 0..2^30 records of a stride of at least 20 bytes, a multiple of 4,
// and the pointers given when n > 0
inline bool records_ok(const void* points, int64_t n, int64_t stride, const void* out, const int64_t* m_out) {
  return m_out && n >= 0 && n <= (1 << 30) && stride >= 20 && stride % 4 == 0 && (n == 0 || (points && out));
}

struct RecordFilter {
  int device;
  const char* name;                    // the filter in the device messages
  cudaStream_t stream = nullptr;       // of the host entry points, created on first use
  DevBuf host_in, host_out, host_idx;  // their records in, records out and indices out; they only grow
  char error[256] = {0};

  RecordFilter(int device, const char* name) : device(device), name(name) {}

  __attribute__((format(printf, 3, 4))) int fail(int rc, const char* fmt, ...) {
    va_list args;
    va_start(args, fmt);
    vsnprintf(error, sizeof(error), fmt, args);
    va_end(args);
    return rc;
  }
  // an SM_ERR_CUDA gets the CUDA error as its message; other codes pass through
  int cuda_fail(int rc) { return rc == SM_ERR_CUDA ? fail(rc, "%s", last_cuda_error()) : rc; }

  int use_device() {
    const int rc = select_device(device);
    if (rc == SM_ERR_NO_DEVICE) return fail(rc, "no CUDA device: %s has no CPU fallback", name);
    if (rc == SM_ERR_BAD_ARGUMENT) return fail(rc, "device %d is out of range: %s has no CPU fallback", device, name);
    return cuda_fail(rc);
  }

  // one <param> of the filter's XML node (filter_set_param)
  int set_param(FilterParams& f, const char* param, int type, const char* text) {
    const int rc = filter_set_param(f, param, type, text);
    if (rc == SM_ERR_UNKNOWN_OPTION) return fail(rc, "Check failed: all_right (unknown param %s)", param);
    if (rc == SM_ERR_BAD_ARGUMENT)
      return fail(rc, "Check failed: all_right (param %s without a type of 0 or 1)", param);
    return rc;
  }

  // n >= 1 records of `stride` bytes in host memory -> host_in, enqueued on the stream; host_out grows to out_bytes.
  // An SM_ERR_CUDA comes back without a message: the caller reports it with cuda_fail.
  int stage(const void* points, int64_t n, int64_t stride, size_t out_bytes) {
    if (!stream) SMB_CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    const size_t in_bytes = (size_t)n * (size_t)stride;
    SMB_RC(host_in.reserve(in_bytes));
    SMB_RC(host_out.reserve(out_bytes));
    SMB_CUDA_OK(cudaMemcpyAsync(host_in.p, points, in_bytes, cudaMemcpyHostToDevice, stream));
    return SM_OK;
  }
};

template <class Handle>
int create_record_filter(int device, Handle** out) {
  if (!out || device < 0) return SM_ERR_BAD_ARGUMENT;
  *out = new Handle(device);
  return SM_OK;
}

template <class Handle>
int destroy_record_filter(Handle* h) {
  if (!h) return SM_ERR_BAD_ARGUMENT;
  if (h->stream) { cudaSetDevice(h->device); cudaStreamDestroy(h->stream); }
  delete h;
  return SM_OK;
}

// The host entry of a record filter, after its own checks: the n records of `stride` bytes at `points` are staged, the
// device form run_device (the handle's sm_*_run_device) writes the kept ones and their indices into host_out / host_idx
// on the handle's stream, and the m kept records and indices (optional) are copied back before one synchronise.  n = 0
// runs the device form alone.  Past n = 0, *m_out is written on success only.
template <class Handle, class RunDevice>
int run_record_filter(Handle* h, RunDevice run_device, const float* points, int64_t n, int64_t stride, float* out,
                      int64_t* m_out, int32_t* index) {
  if (n == 0) return run_device(h, nullptr, 0, stride, nullptr, m_out, nullptr, nullptr);
  int64_t m = 0;
  const int rc = h->cuda_fail([&]() -> int {
    SMB_RC(h->stage(points, n, stride, (size_t)n * 20));
    SMB_RC(h->host_idx.reserve((size_t)n * sizeof(int32_t)));
    SMB_RC(run_device(h, (const float*)h->host_in.p, n, stride, (float*)h->host_out.p, &m, (int32_t*)h->host_idx.p,
                      h->stream));
    if (m == 0) return SM_OK;
    SMB_CUDA_OK(cudaMemcpyAsync(out, h->host_out.p, (size_t)m * 20, cudaMemcpyDeviceToHost, h->stream));
    if (index)
      SMB_CUDA_OK(cudaMemcpyAsync(index, h->host_idx.p, (size_t)m * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                  h->stream));
    SMB_CUDA_OK(cudaStreamSynchronize(h->stream));
    return SM_OK;
  }());
  if (rc == SM_OK) *m_out = m;
  return rc;
}

}  // namespace smb

#endif  // SM_B200_RECORD_FILTER_H_
