// obca_plan.cu -- the GPU Hybrid A* warm-start producer (obca_plan_parking_warmstart_goals / _batch of include/obca.h): k_plan_hmap,
// k_plan and their entries.  Built as its own translation unit WITHOUT FMA contraction (-fmad=false), because the host planner it
// reproduces is built with -ffp-contract=off; linked into libobca.so next to obca_lib.cu (see __graft_entry__.build()).
//
// k_plan_hmap: one CTA per distinct goal cell of the call relaxes that cell's heuristic map (hmap_one) in shared memory when it fits,
// else in place in global memory, and leaves it in global memory for k_plan.
// k_plan: persistent CTAs of PLAN_THREADS threads take start poses from an atomic counter, so that the short plans (the median plan is
// about 100 times shorter than the longest) do not wait for the long ones.  Each resident CTA owns its scratch in global memory (cell ->
// node table, node pool, heap, course and path buffers), reused pose after pose; each pose reads the map of its own goal cell.
#include <cuda_runtime.h>

#include <cmath>
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
constexpr int HMAP_THREADS = 512;

struct CtaDev {
  __device__ int tid() const { return threadIdx.x; }
  __device__ int nth() const { return blockDim.x; }
  __device__ void sync() const { __syncthreads(); }
  __device__ int sync_or(int v) const { return __syncthreads_or(v); }
};

// The heuristic maps: map g from the goal cell (gcell[2g], gcell[2g+1]) into maps + g * xw * yw.  smem: relax in dynamic shared memory
// (xw * yw doubles) and copy the result out, else relax in place.
__global__ void __launch_bounds__(HMAP_THREADS) k_plan_hmap(const char* obmap, long minx, long miny, int xw, int yw, const long* gcell,
                                                            double sqrt2, bool smem, double* maps) {
  extern __shared__ double hs[];
  const size_t cells = (size_t)xw * yw;
  double* out = maps + blockIdx.x * cells;
  double* d = smem ? hs : out;
  hmap_one(CtaDev(), obmap, xw, yw, gcell[2 * blockIdx.x] - minx, gcell[2 * blockIdx.x + 1] - miny, sqrt2, d);
  if (smem)
    for (size_t k = threadIdx.x; k < cells; k += blockDim.x) out[k] = d[k];
}

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

// The maps of the goal cells gcell (2 per map) into dmaps on the stream st, with the obstacle map H copied to the device first (into
// dbuf, which the caller keeps until the stream is done).  ev0 / ev1 (may be null): recorded around the kernel.
int launch_hmaps(const HeurGrid& H, const std::vector<long>& gcell, double* dmaps, int dev, cudaStream_t st, DevBuf& dbuf, cudaEvent_t ev0,
                 cudaEvent_t ev1) {
  const size_t cells = (size_t)H.xw * H.yw, G = gcell.size() / 2;
  if (G == 0 || cells == 0) return 0;
  char* dob;
  long* dg;
  DevLayout l;
  l.in(dob, H.obmap.data(), cells);
  l.in(dg, gcell.data(), gcell.size());
  CK(alloc_layout(dbuf, l));
  CK(l.copy_in(st));
  int optin = 0;
  CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const size_t bytes = cells * sizeof(double);
  const bool smem = bytes <= (size_t)optin;
  if (smem) CK(cudaFuncSetAttribute(k_plan_hmap, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  if (ev0) CK(cudaEventRecord(ev0, st));
  k_plan_hmap<<<(unsigned)G, HMAP_THREADS, smem ? bytes : 0, st>>>(dob, H.minx, H.miny, H.xw, H.yw, dg, std::sqrt(2.0), smem, dmaps);
  CK(cudaGetLastError());
  if (ev1) CK(cudaEventRecord(ev1, st));
  return 0;
}

}  // namespace

int plan_check_args(int B, bool args, int n_ob, double Ts, int sampleN) {
  if (B < 0) { obca_set_last_error("B < 0"); return OBCA_ERR_ARG; }
  if (!args) { obca_set_last_error("null argument"); return OBCA_ERR_ARG; }
  if (n_ob <= 0) { obca_set_last_error("n_ob <= 0: the planner needs obstacle points"); return OBCA_ERR_ARG; }
  if (!(Ts > 0)) { obca_set_last_error("Ts <= 0"); return OBCA_ERR_ARG; }
  if (sampleN < 1) { obca_set_last_error("sampleN < 1"); return OBCA_ERR_ARG; }
  if (motion_nlist() != PLAN_NLIST) { obca_set_last_error("motion primitive length differs from the kernel's"); return OBCA_ERR_UNSUPPORTED; }
  return 0;
}

int plan_warmstart_dev(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                       int sampleN, int max_expansions, int max_nodes, int cap, int dev, cudaStream_t st, const PlanDevOut& out,
                       float* plan_ms) {
  if (max_nodes <= 0) max_nodes = PLAN_DEFAULT_NODES;
  PlanSetup S;
  plan_setup(S, B, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap);
  int sms = 0;
  Event e0, e1;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  CK(cudaEventCreate(&e0.h));
  CK(cudaEventCreate(&e1.h));
  const int grid = B < sms * PLAN_CTAS_PER_SM ? B : sms * PLAN_CTAS_PER_SM;
  const size_t P = plan_path_max(cap, sampleN), nc = (size_t)S.ob.start.size(), ni = S.ob.ids.size();
  const size_t nh = S.C.hcells * (S.gcell.size() / 2);
  // batch constants: obstacle points, cell grid (CSR), one heuristic map per distinct goal cell, counter; the poses and goals
  double *dox, *doy, *dpmap, *dx0, *dxF;
  int *dstart, *dids, *dcounter, *dhidx;
  DevLayout cl;
  cl.in(dox, S.ob.ox.data(), n_ob);
  cl.in(doy, S.ob.oy.data(), n_ob);
  cl.in(dstart, S.ob.start.data(), nc);
  cl.in(dids, ni > 0 ? S.ob.ids.data() : nullptr, ni > 0 ? ni : 1);
  cl.add(dpmap, nh > 0 ? nh : 1);
  cl.add(dcounter, 1);
  cl.in(dx0, x0, 3 * (size_t)B);
  cl.in(dxF, xF, 3 * (size_t)B);
  cl.in(dhidx, S.hidx.data(), B);
  DevBuf dconst, dhmap;
  CK(alloc_layout(dconst, cl));
  CK(cl.copy_in(st));
  CK(cudaMemsetAsync(dcounter, 0, sizeof(int), st));
  const int hrc = launch_hmaps(S.H, S.gcell, dpmap, dev, st, dhmap, nullptr, nullptr);
  if (hrc) return hrc;
  PlanConst C = S.C;
  C.grid.start = dstart; C.grid.ids = dids; C.grid.ox = dox; C.grid.oy = doy; C.pmap = dpmap; C.goals = dxF; C.hidx = dhidx;
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
  CK(cudaMemsetAsync(W0.table, 0xff, C.table_size * grid * sizeof(int), st));      // -1: no node
  PlanIO io{dx0, out.rx, out.ry, out.ryaw, out.xWS, out.uWS, out.N, out.status, out.expansions};
  CK(cudaEventRecord(e0.h, st));
  k_plan<<<grid, PLAN_THREADS, 0, st>>>(B, C, io, W0, dcounter);
  CK(cudaGetLastError());
  CK(cudaEventRecord(e1.h, st));
  CK(cudaStreamSynchronize(st));      // the scratch is freed on return
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0.h, e1.h));
  if (plan_ms) *plan_ms = ms;
  return 0;
}

// Both warm-start entries: B start poses, goal p at xF + goal_stride * p (3: a goal per pose, 0: one goal for the batch).  The outputs
// are copied to the device first, so that the kernel leaves every entry it does not write as the caller had it.
static int plan_warmstart(int B, const double* x0, const double* xF, size_t goal_stride, const double* ox, const double* oy, int n_ob,
                          double Ts, double L, int sampleN, int max_expansions, int max_nodes, int cap, const obca_opts* opts, double* rx,
                          double* ry, double* ryaw, double* xWS, double* uWS, int* N, int* status, int* expansions, double* plan_seconds) {
  int rc = plan_check_args(B, x0 && xF && ox && oy && rx && ry && ryaw && xWS && uWS && N && status, n_ob, Ts, sampleN);
  if (rc) return rc;
  if (cap < 2) { obca_set_last_error("cap < 2"); return OBCA_ERR_ARG; }
  const int dev = opts ? opts->device : 0;
  rc = check_device(dev);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = 0.0;
  if (B == 0) return 0;

  std::vector<double> xFs(3 * (size_t)B);
  for (int p = 0; p < B; ++p)
    for (int r = 0; r < 3; ++r) xFs[3 * (size_t)p + r] = xF[goal_stride * p + r];
  Stream st;
  CK(cudaSetDevice(dev));
  CK(cudaStreamCreateWithFlags(&st.h, cudaStreamNonBlocking));
  const size_t cb = (size_t)B * cap;
  PlanDevOut o;
  DevLayout il;
  il.inout(o.rx, rx, cb);
  il.inout(o.ry, ry, cb);
  il.inout(o.ryaw, ryaw, cb);
  il.inout(o.xWS, xWS, 4 * cb);
  il.inout(o.uWS, uWS, 2 * cb);
  il.inout(o.N, N, B);
  il.out(o.status, status, B);
  il.out(o.expansions, expansions, B);
  DevBuf dio;
  CK(alloc_layout(dio, il));
  CK(il.copy_in(st.h));
  float ms = 0.f;
  rc = plan_warmstart_dev(B, x0, xFs.data(), ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap, dev, st.h, o, &ms);
  if (rc) return rc;
  CK(il.copy_out(st.h));
  CK(cudaStreamSynchronize(st.h));
  if (plan_seconds) *plan_seconds = ms * 1e-3;
  return 0;
}

extern "C" int obca_plan_parking_warmstart_goals(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob,
                                                 double Ts, double L, int sampleN, int max_expansions, int max_nodes, int cap,
                                                 const obca_opts* opts, double* rx, double* ry, double* ryaw, double* xWS, double* uWS,
                                                 int* N, int* status, int* expansions, double* plan_seconds) {
  return plan_warmstart(B, x0, xF, 3, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap, opts, rx, ry, ryaw, xWS, uWS, N, status,
                        expansions, plan_seconds);
}

extern "C" int obca_plan_parking_warmstart_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob,
                                                 double Ts, double L, int sampleN, int max_expansions, int max_nodes, int cap,
                                                 const obca_opts* opts, double* rx, double* ry, double* ryaw, double* xWS, double* uWS,
                                                 int* N, int* status, int* expansions, double* plan_seconds) {
  return plan_warmstart(B, x0, xF, 0, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap, opts, rx, ry, ryaw, xWS, uWS, N, status,
                        expansions, plan_seconds);
}

extern "C" int obca_plan_parking_heuristic_maps(int G, const double* goals, const double* ox, const double* oy, int n_ob, const obca_opts* opts,
                                                long long* mn, int* w, double* maps, long long cap, double* map_seconds) {
  if (G < 0) { obca_set_last_error("G < 0"); return OBCA_ERR_ARG; }
  if (!goals || !ox || !oy || !mn || !w) { obca_set_last_error("null argument"); return OBCA_ERR_ARG; }
  if (n_ob <= 0) { obca_set_last_error("n_ob <= 0: the planner needs obstacle points"); return OBCA_ERR_ARG; }
  const std::vector<double> vx(ox, ox + n_ob), vy(oy, oy + n_ob);
  const HeurGrid H = calc_heur_grid(vx, vy, XY_GRID_RESOLUTION, VEHICLE_RADIUS);
  mn[0] = H.minx; mn[1] = H.miny; w[0] = H.xw; w[1] = H.yw;
  const size_t cells = (size_t)H.xw * H.yw;
  if (!maps || (long long)(cells * G) > cap) { obca_set_last_error("maps: fewer than G x xw x yw entries"); return OBCA_ERR_ARG; }
  const int dev = opts ? opts->device : 0;
  const int rc = check_device(dev);
  if (rc) return rc;
  if (map_seconds) *map_seconds = 0.0;
  if (G == 0 || cells == 0) return 0;
  std::vector<long> gcell(2 * (size_t)G);
  for (int g = 0; g < G; ++g) heur_goal_cell(goals[2 * (size_t)g], goals[2 * (size_t)g + 1], XY_GRID_RESOLUTION, gcell[2 * g], gcell[2 * g + 1]);
  Stream st;
  Event e0, e1;
  CK(cudaSetDevice(dev));
  CK(cudaStreamCreateWithFlags(&st.h, cudaStreamNonBlocking));
  CK(cudaEventCreate(&e0.h));
  CK(cudaEventCreate(&e1.h));
  double* dmaps;
  DevLayout l;
  l.out(dmaps, maps, cells * G);
  DevBuf dbuf, dhmap;
  CK(alloc_layout(dbuf, l));
  const int hrc = launch_hmaps(H, gcell, dmaps, dev, st.h, dhmap, e0.h, e1.h);
  if (hrc) return hrc;
  CK(l.copy_out(st.h));
  CK(cudaStreamSynchronize(st.h));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0.h, e1.h));
  if (map_seconds) *map_seconds = ms * 1e-3;
  return 0;
}
