// obca_plan.cu -- the GPU Hybrid A* warm-start producer (obca_plan_parking_warmstart_batch of include/obca.h): k_plan and its entry.
// Built as its own translation unit WITHOUT FMA contraction (-fmad=false), because the host planner it reproduces is built with
// -ffp-contract=off; linked into libobca.so next to obca_lib.cu (see __graft_entry__.build()).
//
// k_plan: persistent CTAs of PLAN_THREADS threads take start poses from an atomic counter, so that the short plans (the median plan is
// about 100 times shorter than the longest) do not wait for the long ones.  Each resident CTA owns its scratch in global memory (cell ->
// node table, node pool, heap, course and path buffers), reused pose after pose.
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "../../include/obca.h"
#include "../../include/obca_planner.h"
#include "obca_devstage.h"
#include "obca_plan.cuh"

static_assert(obca_plan::PLAN_NODE_POOL == OBCA_PLAN_POOL_FULL, "status code of a full node pool");

using namespace obca;
using namespace obca_plan;

namespace {

constexpr int PLAN_THREADS = 128;
constexpr int PLAN_CTAS_PER_SM = 4;
constexpr int PLAN_DEFAULT_NODES = 32768;      // 7x the most nodes a plan of the demo sweeps inserts (4493)

struct CtaDev {
  __device__ int tid() const { return threadIdx.x; }
  __device__ int nth() const { return blockDim.x; }
  __device__ void sync() const { __syncthreads(); }
};

__global__ void __launch_bounds__(PLAN_THREADS) k_plan(int B, PlanConst C, PlanIO io, PlanScratch W0, int* counter) {
  __shared__ PlanSmem sm;
  __shared__ int prob;
  const size_t b = blockIdx.x, P = plan_path_max(C.cap, C.sampleN);
  PlanScratch W{W0.table + b * C.table_size, W0.pool + b * C.max_nodes, W0.heap + b * C.max_nodes,
                W0.rsx + b * RS_MAX_PTS, W0.rsy + b * RS_MAX_PTS, W0.rsyaw + b * RS_MAX_PTS, W0.rspar + b * RS_MAX_PTS,
                W0.rsseg + b * RS_MAX_PTS, W0.px + b * P, W0.py + b * P, W0.pyaw + b * P, W0.work + b * 9 * (P + 40)};
  for (;;) {
    if (threadIdx.x == 0) prob = atomicAdd(counter, 1);
    __syncthreads();
    const int p = prob;
    __syncthreads();
    if (p >= B) break;
    plan_one(CtaDev(), C, W, sm, io, p);
  }
}

}  // namespace

extern "C" int obca_plan_parking_warmstart_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob,
                                                 double Ts, double L, int sampleN, int max_expansions, int max_nodes, int cap,
                                                 const obca_opts* opts, double* rx, double* ry, double* ryaw, double* xWS, double* uWS,
                                                 int* N, int* status, int* expansions, double* plan_seconds) {
  if (B < 0) { obca_set_last_error("B < 0"); return OBCA_ERR_ARG; }
  if (!x0 || !xF || !ox || !oy || !rx || !ry || !ryaw || !xWS || !uWS || !N || !status) {
    obca_set_last_error("null argument"); return OBCA_ERR_ARG;
  }
  if (n_ob <= 0) { obca_set_last_error("n_ob <= 0: the planner needs obstacle points"); return OBCA_ERR_ARG; }
  if (!(Ts > 0)) { obca_set_last_error("Ts <= 0"); return OBCA_ERR_ARG; }
  if (sampleN < 1) { obca_set_last_error("sampleN < 1"); return OBCA_ERR_ARG; }
  if (cap < 2) { obca_set_last_error("cap < 2"); return OBCA_ERR_ARG; }
  if (motion_nlist() != PLAN_NLIST) { obca_set_last_error("motion primitive length differs from the kernel's"); return OBCA_ERR_UNSUPPORTED; }
  const int dev = opts ? opts->device : 0;
  const int rc = check_device(dev);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = 0.0;
  if (B == 0) return 0;
  if (max_nodes <= 0) max_nodes = PLAN_DEFAULT_NODES;

  PlanSetup S;
  plan_setup(S, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap);
  int sms = 0;
  Stream st;
  Event e0, e1;
  CK(cudaSetDevice(dev));
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CK(cudaStreamCreateWithFlags(&st.h, cudaStreamNonBlocking));
  CK(cudaEventCreate(&e0.h));
  CK(cudaEventCreate(&e1.h));
  const int grid = B < sms * PLAN_CTAS_PER_SM ? B : sms * PLAN_CTAS_PER_SM;
  const size_t P = plan_path_max(cap, sampleN), nc = (size_t)S.ob.start.size(), ni = S.ob.ids.size(), nh = S.H.pmap.size();
  // batch constants: obstacle points, cell grid (CSR), heuristic map, counter
  double *dox, *doy, *dpmap;
  int *dstart, *dids, *dcounter;
  DevLayout cl;
  cl.in(dox, S.ob.ox.data(), n_ob);
  cl.in(doy, S.ob.oy.data(), n_ob);
  cl.in(dstart, S.ob.start.data(), nc);
  cl.in(dids, ni > 0 ? S.ob.ids.data() : nullptr, ni > 0 ? ni : 1);
  cl.in(dpmap, nh > 0 ? S.H.pmap.data() : nullptr, nh > 0 ? nh : 1);
  cl.add(dcounter, 1);
  DevBuf dconst;
  CK(alloc_layout(dconst, cl));
  CK(cl.copy_in(st.h));
  CK(cudaMemsetAsync(dcounter, 0, sizeof(int), st.h));
  PlanConst C = S.C;
  C.grid.start = dstart; C.grid.ids = dids; C.grid.ox = dox; C.grid.oy = doy; C.pmap = dpmap;
  // per resident CTA: cell table, node pool, heap, course and path buffers
  PlanScratch W0;
  DevLayout wl;
  wl.add(W0.table, C.table_size * grid);
  wl.add(W0.pool, (size_t)max_nodes * grid);
  wl.add(W0.heap, (size_t)max_nodes * grid);
  wl.add(W0.rsx, (size_t)RS_MAX_PTS * grid);
  wl.add(W0.rsy, (size_t)RS_MAX_PTS * grid);
  wl.add(W0.rsyaw, (size_t)RS_MAX_PTS * grid);
  wl.add(W0.rspar, (size_t)RS_MAX_PTS * grid);
  wl.add(W0.rsseg, (size_t)RS_MAX_PTS * grid);
  wl.add(W0.px, P * grid);
  wl.add(W0.py, P * grid);
  wl.add(W0.pyaw, P * grid);
  wl.add(W0.work, 9 * (P + 40) * grid);
  DevBuf dscr;
  CK(alloc_layout(dscr, wl));
  CK(cudaMemsetAsync(W0.table, 0xff, C.table_size * grid * sizeof(int), st.h));      // -1: no node
  // inputs / outputs: outputs are copied in first, so that the kernel leaves every entry it does not write as the caller had it
  const size_t cb = (size_t)B * cap;
  double *dx0, *drx, *dry, *dryaw, *dxWS, *duWS;
  int *dN, *dst, *dex;
  DevLayout il;
  il.in(dx0, x0, 3 * (size_t)B);
  il.inout(drx, rx, cb);
  il.inout(dry, ry, cb);
  il.inout(dryaw, ryaw, cb);
  il.inout(dxWS, xWS, 4 * cb);
  il.inout(duWS, uWS, 2 * cb);
  il.inout(dN, N, B);
  il.out(dst, status, B);
  il.out(dex, expansions, B);
  DevBuf dio;
  CK(alloc_layout(dio, il));
  CK(il.copy_in(st.h));
  PlanIO io{dx0, drx, dry, dryaw, dxWS, duWS, dN, dst, dex};
  CK(cudaEventRecord(e0.h, st.h));
  k_plan<<<grid, PLAN_THREADS, 0, st.h>>>(B, C, io, W0, dcounter);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e1.h, st.h));
  CK(il.copy_out(st.h));
  CK(cudaStreamSynchronize(st.h));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0.h, e1.h));
  if (plan_seconds) *plan_seconds = ms * 1e-3;
  return 0;
}
