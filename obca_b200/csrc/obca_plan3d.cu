// obca_plan3d.cu -- the GPU 3-D A* warm-start producer of the quadcopter flow (obca_plan_quadcopter_warmstart_batch of include/obca.h):
// k_plan3d and its entry.  Built as its own translation unit WITHOUT FMA contraction (-fmad=false), because the host planner it reproduces
// is built with -ffp-contract=off; linked into libobca.so next to obca_lib.cu (see __graft_entry__.build()).
//
// k_plan3d: persistent CTAs of P3_WARPS warps; every warp takes pairs from an atomic counter (the longest config-4 search expands 10x
// the cells of the shortest) and runs astar3d_one (obca_astar3d_core.h) with its 32 lanes: lanes 0..25 test one neighbour each, a ballot
// and a prefix count give the new nodes and the insertion ticks in motion order, and the lanes compare the 32 children of a queue entry in
// one reduction.  Each warp owns its scratch in global memory (cell -> node table, node pool, queue), reused pair after pair.
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "../../include/obca.h"
#include "../../include/obca_planner.h"
#include "../planner/csrc/obca_astar3d_core.h"
#include "obca_devstage.h"

static_assert(obca_astar3d::A3_POOL_FULL == OBCA_PLAN_POOL_FULL, "status code of a full node pool or queue");
static_assert(obca_astar3d::A3_CAPACITY == OBCA_PLAN_CAPACITY && obca_astar3d::A3_NO_PATH == OBCA_PLAN_NO_PATH, "status codes");

using namespace obca;
using namespace obca_astar3d;

namespace {

constexpr int P3_WARPS = 4;                    // warps per CTA, one CTA per SM: 528 searches in flight on a 132-SM H100
constexpr int P3_DEFAULT_NODES = 1 << 18;      // the most nodes a config-4 search of quadcopter_batch(2048, seed=2) uses is 229043
constexpr unsigned FULL = 0xffffffffu;

// The 32 lanes of a warp: lane m < 26 holds the values of move m.
struct WarpLanes {
  template <class T> using PerMove = T;
  __device__ int lane() const { return threadIdx.x & 31; }
  __device__ int width() const { return 32; }
  __device__ void sync() const { __syncwarp(); }
  template <class T> __device__ T& at(T& v, int) const { return v; }
  template <class T> __device__ T take(const T& v, int m) const { return __shfl_sync(FULL, v, m); }
  __device__ unsigned mask(bool v) const { return __ballot_sync(FULL, lane() < N_MOVES && v); }
  // the smallest (f, tick) over the lanes; bj < 0: this lane holds no child
  __device__ void qmin(A3Item& best, int& bj) const {
    for (int o = 16; o > 0; o >>= 1) {
      const double f = __shfl_xor_sync(FULL, best.f, o);
      const unsigned t = __shfl_xor_sync(FULL, best.tick, o);
      const int nd = __shfl_xor_sync(FULL, best.node, o), j = __shfl_xor_sync(FULL, bj, o);
      const A3Item x{f, t, nd};
      if (j >= 0 && (bj < 0 || a3_less(x, best))) { best = x; bj = j; }
    }
  }
};

__global__ void __launch_bounds__(P3_WARPS * 32) k_plan3d(int B, A3Const C, A3IO io, A3Scratch W0, size_t table_stride, int* counter) {
  const size_t w = (size_t)blockIdx.x * P3_WARPS + threadIdx.x / 32;
  const A3Scratch W{W0.table + w * table_stride, W0.pool + w * C.max_nodes, W0.queue + w * C.max_queue};
  const WarpLanes ln{};
  for (;;) {
    int p = 0;
    if (ln.lane() == 0) p = atomicAdd(counter, 1);
    p = __shfl_sync(FULL, p, 0);
    if (p >= B) break;
    astar3d_one(ln, C, W, io, p);
  }
}

}  // namespace

struct Plan3dSetup : A3Setup {};
void Plan3dSetupFree::operator()(Plan3dSetup* s) const { delete s; }

int plan3d_prepare(Plan3dSetupPtr& S, int B, bool args, const double* x0, const double* xF, const double* ox, const double* oy,
                   const double* oz, int n_ob, const double* lo, const double* hi, double reso, int max_nodes, int cap) {
  if (!args) { obca_set_last_error("null argument"); return OBCA_ERR_ARG; }
  if (max_nodes > A3_MAX_NODES) { obca_set_last_error("max_nodes > 2^28"); return OBCA_ERR_ARG; }
  S.reset(new Plan3dSetup);
  std::string why;
  if (astar3d_setup(*S, why, B, x0, xF, ox, oy, oz, n_ob, lo, hi, reso, cap)) { obca_set_last_error(why); return OBCA_ERR_ARG; }
  if (max_nodes <= 0) max_nodes = P3_DEFAULT_NODES;
  S->C.max_nodes = max_nodes;
  S->C.max_queue = max_nodes / 4 > 64 ? max_nodes / 4 : 64;
  return 0;
}

int plan3d_dev(const Plan3dSetup& S, int B, int dev, cudaStream_t st, const Plan3dDevOut& out, float* plan_ms) {
  A3Const C = S.C;
  int sms = 0;
  Event e0, e1;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CK(cudaEventCreate(&e0.h));
  CK(cudaEventCreate(&e1.h));
  const int grid = (B + P3_WARPS - 1) / P3_WARPS < sms ? (B + P3_WARPS - 1) / P3_WARPS : sms;
  const size_t nw = (size_t)grid * P3_WARPS, nmap = S.map.size(), Bs = (size_t)B;
  // batch constants: the obstacle bitmap, the pairs' cells, the counter
  uint32_t* dmap;
  long long *ds, *dg;
  int* dcounter;
  DevLayout cl;
  cl.in(dmap, S.map.data(), nmap);
  cl.in(ds, S.s.data(), 3 * Bs);
  cl.in(dg, S.g.data(), 3 * Bs);
  cl.add(dcounter, 1);
  DevBuf dconst;
  CK(alloc_layout(dconst, cl));
  CK(cl.copy_in(st));
  CK(cudaMemsetAsync(dcounter, 0, sizeof(int), st));
  C.map = dmap;
  // per warp: cell table, node pool, queue
  const size_t table_stride = DevLayout::padded((size_t)(S.cells > 0 ? S.cells : 1) * sizeof(int)) / sizeof(int);
  A3Scratch W0;
  DevLayout wl;
  wl.add(W0.table, table_stride * nw);
  wl.add(W0.pool, (size_t)C.max_nodes * nw);
  wl.add(W0.queue, (size_t)C.max_queue * nw);
  DevBuf dscr;
  CK(alloc_layout(dscr, wl));
  CK(cudaMemsetAsync(W0.table, 0xff, table_stride * nw * sizeof(int), st));      // -1: no node
  const A3IO io{ds, dg, out.rx, out.ry, out.rz, out.N, out.status, out.expansions, nullptr, nullptr};
  CK(cudaEventRecord(e0.h, st));
  k_plan3d<<<grid, P3_WARPS * 32, 0, st>>>(B, C, io, W0, table_stride, dcounter);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e1.h, st));
  CK(cudaStreamSynchronize(st));      // the scratch is freed on return
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0.h, e1.h));
  if (plan_ms) *plan_ms = ms;
  return 0;
}

// The outputs are copied to the device first, so that the kernel leaves every entry it does not write as the caller had it.
extern "C" int obca_plan_quadcopter_warmstart_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy,
                                                    const double* oz, int n_ob, const double* lo, const double* hi, double reso,
                                                    int max_nodes, int cap, const obca_opts* opts, double* rx, double* ry, double* rz,
                                                    int* N, int* status, int* expansions, double* plan_seconds) {
  Plan3dSetupPtr S;
  int rc = plan3d_prepare(S, B, rx && ry && rz && N && status, x0, xF, ox, oy, oz, n_ob, lo, hi, reso, max_nodes, cap);
  if (rc) return rc;
  const int dev = opts ? opts->device : 0;
  rc = check_device(dev);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = 0.0;
  if (B == 0) return 0;
  Stream st;
  CK(cudaSetDevice(dev));
  CK(cudaStreamCreateWithFlags(&st.h, cudaStreamNonBlocking));
  const size_t Bs = (size_t)B, cb = Bs * cap;
  Plan3dDevOut o;
  DevLayout il;
  il.inout(o.rx, rx, cb);
  il.inout(o.ry, ry, cb);
  il.inout(o.rz, rz, cb);
  il.inout(o.N, N, Bs);
  il.out(o.status, status, Bs);
  il.inout(o.expansions, expansions, Bs);
  DevBuf dio;
  CK(alloc_layout(dio, il));
  CK(il.copy_in(st.h));
  if (!expansions) o.expansions = nullptr;
  float ms = 0.f;
  rc = plan3d_dev(*S, B, dev, st.h, o, &ms);
  if (rc) return rc;
  CK(il.copy_out(st.h));
  CK(cudaStreamSynchronize(st.h));
  if (plan_seconds) *plan_seconds = ms * 1e-3;
  return 0;
}
