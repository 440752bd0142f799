// obca_devstage.h -- host glue of the C-ABI's CUDA translation units (obca_lib.cu, obca_plan.cu, obca_plan3d.cu): error reporting,
// the device check, the layout of the typed arrays carved from one device buffer, typed copies, a per-horizon scatter and owners of
// per-call device resources.  Host code only, and not included by obca_host.h: the development emulation builds without CUDA headers.
#pragma once
#include <cuda_runtime.h>
#include <string.h>

#include <memory>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/obca.h"

void obca_set_last_error(const std::string& s);      // obca_lib.cu: the text of obca_last_error()

// A failed CUDA call records "<call>: <CUDA error>" for obca_last_error() and returns OBCA_ERR_CUDA from the enclosing function.
#define CK(call)                                                                                   \
  do {                                                                                               \
    cudaError_t e_ = (call);                                                                         \
    if (e_ != cudaSuccess) {                                                                         \
      obca_set_last_error(std::string(#call) + ": " + cudaGetErrorString(e_));                       \
      return OBCA_ERR_CUDA;                                                                          \
    }                                                                                                \
  } while (0)

namespace obca {

// A CUDA device must be visible and dev one of them; argument errors are reported before this check.
inline int check_device(int dev) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { obca_set_last_error("no CUDA device visible"); return OBCA_ERR_NO_DEVICE; }
  if (dev < 0 || dev >= n) { obca_set_last_error("bad device ordinal"); return OBCA_ERR_ARG; }
  return 0;
}

// Typed arrays in one device buffer, each at a 256-byte boundary, and their host counterparts.  Recording an array grows `bytes`, so the
// size of a buffer is the sum of what is carved from it; place(base) then points every recorded pointer into a buffer of that size.
//   add(d, n)       device only
//   in(d, h, n)     copied from h to the device by copy_in()
//   out(d, h, n)    copied from the device to h by copy_out()
//   inout(d, h, n)  both
// copy_in() and copy_out() issue their copies in the order the arrays were recorded, with n * sizeof(T) bytes each; a null host pointer
// (an optional input or output the caller did not pass) skips that copy.
class DevLayout {
 public:
  size_t bytes = 0;
  template <class T>
  void add(T*& d, size_t n) { record(d, n, nullptr, nullptr); }
  template <class T>
  void in(T*& d, const std::remove_const_t<T>* h, size_t n) { record(d, n, h, nullptr); }      // d may be a pointer to const
  template <class T>
  void out(T*& d, T* h, size_t n) { record(d, n, nullptr, h); }
  template <class T>
  void inout(T*& d, T* h, size_t n) { record(d, n, h, h); }
  static size_t padded(size_t b) { return (b + 255) / 256 * 256; }
  void place(void* base) {
    base_ = (char*)base;
    for (const Part& q : parts_) q.set(q.slot, base_ + q.off);
  }
  cudaError_t copy_in(cudaStream_t st) const {
    for (const Part& q : parts_)
      if (q.src && q.n) {
        const cudaError_t e = cudaMemcpyAsync(base_ + q.off, q.src, q.n, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return e;
      }
    return cudaSuccess;
  }
  cudaError_t copy_out(cudaStream_t st) const {
    for (const Part& q : parts_)
      if (q.dst && q.n) {
        const cudaError_t e = cudaMemcpyAsync(q.dst, base_ + q.off, q.n, cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) return e;
      }
    return cudaSuccess;
  }
  // the address of the recorded array d in a host copy of the placed buffer
  template <class T>
  const T* in_copy(const T* d, const void* copy) const { return (const T*)((const char*)copy + ((const char*)d - base_)); }

 private:
  struct Part {
    void* slot;
    void (*set)(void*, char*);
    size_t off, n;      // bytes
    const void* src;
    void* dst;
  };
  template <class T>
  static void set(void* slot, char* at) { *(T**)slot = (T*)at; }
  template <class T>
  void record(T*& d, size_t n, const void* src, void* dst) {
    parts_.push_back({&d, &set<T>, bytes, n * sizeof(T), src, dst});
    bytes += padded(n * sizeof(T));
  }
  std::vector<Part> parts_;
  char* base_ = nullptr;
};

// n elements from the device to h on the stream st
template <class T>
cudaError_t to_host(T* h, const T* d, size_t n, cudaStream_t st) {
  return cudaMemcpyAsync(h, d, n * sizeof(T), cudaMemcpyDeviceToHost, st);
}

// Problem q of a per-problem array with the stride `per` (laid out for the batch's longest horizon) keeps rows * (Nb[q] + ext)
// entries: only those go from the host scratch src to dst, so the padding past each problem's horizon is never written.  dst null:
// an optional output the caller did not pass.
inline void scatter_horizons(double* dst, const double* src, int B, const int* Nb, size_t per, size_t rows, int ext) {
  if (!dst) return;
  for (int q = 0; q < B; ++q) memcpy(dst + per * q, src + per * q, rows * (size_t)(Nb[q] + ext) * sizeof(double));
}

// Owner of a per-call CUDA handle, released on every return path.
template <class H, cudaError_t (*Release)(H)>
struct Owned {
  H h = nullptr;
  Owned() = default;
  Owned(const Owned&) = delete;
  Owned& operator=(const Owned&) = delete;
  ~Owned() {
    if (h) Release(h);
  }
};
using DevBuf = Owned<void*, cudaFree>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;

// a device buffer of the layout's size, with the layout's pointers placed in it
inline cudaError_t alloc_layout(DevBuf& buf, DevLayout& lay) {
  const cudaError_t e = cudaMalloc(&buf.h, lay.bytes);
  if (e == cudaSuccess) lay.place(buf.h);
  return e;
}

}  // namespace obca

// The GPU Hybrid A* of obca_plan.cu, for the entries that plan there and for obca_parking_plan_solve_goals (obca_lib.cu), which keeps
// the plans on the device.
// plan_check_args: the planner's argument checks, in the entries' order and with their messages (args: no required array is null).
int plan_check_args(int B, bool args, int n_ob, double Ts, int sampleN);
// Device outputs of the planner, in the layout of obca_plan_parking_warmstart_goals with the stride cap.
struct PlanDevOut {
  double *rx, *ry, *ryaw, *xWS, *uWS;
  int *N, *status, *expansions;
};
// Plans B >= 1 start poses x0 (host, 3 per pose: x, y, yaw) towards their goals xF (host, 3 per pose) into `out` on the stream st of the
// current device dev (k_plan_hmap, then k_plan), with arguments that passed plan_check_args and cap >= 2.  Returns once the stream is
// synchronised, after the planner's device scratch is freed; plan_ms (may be null): device time of k_plan.
int plan_warmstart_dev(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                       int sampleN, int max_expansions, int max_nodes, int cap, int dev, cudaStream_t st, const PlanDevOut& out,
                       float* plan_ms);

// The GPU 3-D A* of obca_plan3d.cu, for obca_plan_quadcopter_warmstart_batch and for obca_quadcopter_plan_solve (obca_lib.cu), which keeps
// the plans on the device.  The host set-up (obstacle bitmap, grid geometry, the pairs' cells) stays behind Plan3dSetup, so that only
// obca_plan3d.cu, built without FMA contraction, compiles it.
struct Plan3dSetup;
struct Plan3dSetupFree {
  void operator()(Plan3dSetup* s) const;
};
using Plan3dSetupPtr = std::unique_ptr<Plan3dSetup, Plan3dSetupFree>;
// The planner's argument checks, in the entry's order and with its messages (args: no required array is null), then its host set-up
// of B pairs (x0, xF: host, 3 per pair, in planner units) for paths of at most cap points.  Returns 0 or OBCA_ERR_ARG; touches no device.
int plan3d_prepare(Plan3dSetupPtr& S, int B, bool args, const double* x0, const double* xF, const double* ox, const double* oy,
                   const double* oz, int n_ob, const double* lo, const double* hi, double reso, int max_nodes, int cap);
// Device outputs of the planner, in the layout of obca_plan_quadcopter_warmstart_batch with the stride cap; expansions may be null.
struct Plan3dDevOut {
  double *rx, *ry, *rz;
  int *N, *status, *expansions;
};
// Plans the B >= 1 pairs of S into `out` on the stream st of the current device dev (k_plan3d).  Returns once the stream is
// synchronised, after the planner's device scratch is freed; plan_ms (may be null): device time of k_plan3d.
int plan3d_dev(const Plan3dSetup& S, int B, int dev, cudaStream_t st, const Plan3dDevOut& out, float* plan_ms);
