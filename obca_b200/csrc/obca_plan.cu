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
#include "obca_plan.cuh"

void obca_set_last_error(const std::string& s);      // obca_lib.cu
static_assert(obca_plan::PLAN_NODE_POOL == OBCA_PLAN_POOL_FULL, "status code of a full node pool");

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

#define PCK(call)                                                                    \
  do {                                                                               \
    cudaError_t e_ = (call);                                                         \
    if (e_ != cudaSuccess) {                                                         \
      obca_set_last_error(std::string(#call) + ": " + cudaGetErrorString(e_));       \
      rc = OBCA_ERR_CUDA;                                                            \
      goto done;                                                                     \
    }                                                                                \
  } while (0)

template <class T>
T* carve(char*& p, size_t n) {
  T* r = (T*)p;
  p += (n * sizeof(T) + 255) / 256 * 256;
  return r;
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
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { obca_set_last_error("no CUDA device visible"); return OBCA_ERR_NO_DEVICE; }
  const int dev = opts ? opts->device : 0;
  if (dev < 0 || dev >= ndev) { obca_set_last_error("bad device ordinal"); return OBCA_ERR_ARG; }
  if (plan_seconds) *plan_seconds = 0.0;
  if (B == 0) return 0;
  if (max_nodes <= 0) max_nodes = PLAN_DEFAULT_NODES;

  PlanSetup S;
  plan_setup(S, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap);
  int rc = 0, sms = 0;
  cudaStream_t st = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  char *dconst = nullptr, *dscr = nullptr, *dio = nullptr;
  {
    PCK(cudaSetDevice(dev));
    PCK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    PCK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    PCK(cudaEventCreate(&e0)); PCK(cudaEventCreate(&e1));
    const int grid = B < sms * PLAN_CTAS_PER_SM ? B : sms * PLAN_CTAS_PER_SM;
    const size_t P = plan_path_max(cap, sampleN), nc = (size_t)S.ob.start.size(), ni = S.ob.ids.size(), nh = S.H.pmap.size();
    // batch constants: obstacle points, cell grid (CSR), heuristic map, counter
    const size_t const_bytes = 2 * ((n_ob * 8 + 255) / 256 * 256) + (nc * 4 + 255) / 256 * 256 + (ni * 4 + 255) / 256 * 256 +
                               (nh * 8 + 255) / 256 * 256 + 4 * 256;
    PCK(cudaMalloc(&dconst, const_bytes));
    char* q = dconst;
    double* dox = carve<double>(q, n_ob); double* doy = carve<double>(q, n_ob);
    int* dstart = carve<int>(q, nc); int* dids = carve<int>(q, ni > 0 ? ni : 1);
    double* dpmap = carve<double>(q, nh > 0 ? nh : 1); int* dcounter = carve<int>(q, 1);
    PCK(cudaMemcpyAsync(dox, S.ob.ox.data(), n_ob * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(doy, S.ob.oy.data(), n_ob * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(dstart, S.ob.start.data(), nc * 4, cudaMemcpyHostToDevice, st));
    if (ni) PCK(cudaMemcpyAsync(dids, S.ob.ids.data(), ni * 4, cudaMemcpyHostToDevice, st));
    if (nh) PCK(cudaMemcpyAsync(dpmap, S.H.pmap.data(), nh * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemsetAsync(dcounter, 0, sizeof(int), st));
    PlanConst C = S.C;
    C.grid.start = dstart; C.grid.ids = dids; C.grid.ox = dox; C.grid.oy = doy; C.pmap = dpmap;
    // per resident CTA: cell table, node pool, heap, course and path buffers
    const size_t per_cta = (C.table_size * 4 + 255) / 256 * 256 + ((size_t)max_nodes * sizeof(PNode) + 255) / 256 * 256 +
                           ((size_t)max_nodes * sizeof(HeapItem) + 255) / 256 * 256 + 5 * ((RS_MAX_PTS * 8 + 255) / 256 * 256) +
                           3 * ((P * 8 + 255) / 256 * 256) + (9 * (P + 40) * 8 + 255) / 256 * 256;
    PCK(cudaMalloc(&dscr, per_cta * grid + 12 * 256));
    q = dscr;
    PlanScratch W0;
    W0.table = carve<int>(q, C.table_size * grid); W0.pool = carve<PNode>(q, (size_t)max_nodes * grid);
    W0.heap = carve<HeapItem>(q, (size_t)max_nodes * grid);
    W0.rsx = carve<double>(q, (size_t)RS_MAX_PTS * grid); W0.rsy = carve<double>(q, (size_t)RS_MAX_PTS * grid);
    W0.rsyaw = carve<double>(q, (size_t)RS_MAX_PTS * grid); W0.rspar = carve<double>(q, (size_t)RS_MAX_PTS * grid);
    W0.rsseg = carve<int>(q, (size_t)RS_MAX_PTS * grid);
    W0.px = carve<double>(q, P * grid); W0.py = carve<double>(q, P * grid); W0.pyaw = carve<double>(q, P * grid);
    W0.work = carve<double>(q, 9 * (P + 40) * grid);
    PCK(cudaMemsetAsync(W0.table, 0xff, C.table_size * grid * 4, st));      // -1: no node
    // inputs / outputs: outputs are copied in first, so that the kernel leaves every entry it does not write as the caller had it
    const size_t cb = (size_t)B * cap;
    const size_t io_bytes = ((3 * B * 8 + 255) / 256 + (3 * cb * 8 + 255) / 256 + (4 * cb * 8 + 255) / 256 + (2 * cb * 8 + 255) / 256 +
                             3 * ((B * 4 + 255) / 256)) * 256 + 8 * 256;
    PCK(cudaMalloc(&dio, io_bytes));
    q = dio;
    double* dx0 = carve<double>(q, 3 * (size_t)B);
    double* drx = carve<double>(q, 3 * cb); double* dxWS = carve<double>(q, 4 * cb); double* duWS = carve<double>(q, 2 * cb);
    int* dN = carve<int>(q, B); int* dst = carve<int>(q, B); int* dex = carve<int>(q, B);
    PCK(cudaMemcpyAsync(dx0, x0, 3 * (size_t)B * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(drx, rx, cb * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(drx + cb, ry, cb * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(drx + 2 * cb, ryaw, cb * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(dxWS, xWS, 4 * cb * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(duWS, uWS, 2 * cb * 8, cudaMemcpyHostToDevice, st));
    PCK(cudaMemcpyAsync(dN, N, B * 4, cudaMemcpyHostToDevice, st));
    PlanIO io{dx0, drx, drx + cb, drx + 2 * cb, dxWS, duWS, dN, dst, dex};
    PCK(cudaEventRecord(e0, st));
    k_plan<<<grid, PLAN_THREADS, 0, st>>>(B, C, io, W0, dcounter);
    PCK(cudaGetLastError());
    PCK(cudaEventRecord(e1, st));
    PCK(cudaMemcpyAsync(rx, drx, cb * 8, cudaMemcpyDeviceToHost, st));
    PCK(cudaMemcpyAsync(ry, drx + cb, cb * 8, cudaMemcpyDeviceToHost, st));
    PCK(cudaMemcpyAsync(ryaw, drx + 2 * cb, cb * 8, cudaMemcpyDeviceToHost, st));
    PCK(cudaMemcpyAsync(xWS, dxWS, 4 * cb * 8, cudaMemcpyDeviceToHost, st));
    PCK(cudaMemcpyAsync(uWS, duWS, 2 * cb * 8, cudaMemcpyDeviceToHost, st));
    PCK(cudaMemcpyAsync(N, dN, B * 4, cudaMemcpyDeviceToHost, st));
    PCK(cudaMemcpyAsync(status, dst, B * 4, cudaMemcpyDeviceToHost, st));
    if (expansions) PCK(cudaMemcpyAsync(expansions, dex, B * 4, cudaMemcpyDeviceToHost, st));
    PCK(cudaStreamSynchronize(st));
    float ms = 0.f;
    PCK(cudaEventElapsedTime(&ms, e0, e1));
    if (plan_seconds) *plan_seconds = ms * 1e-3;
  }
done:
  if (dio) cudaFree(dio);
  if (dscr) cudaFree(dscr);
  if (dconst) cudaFree(dconst);
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  if (st) cudaStreamDestroy(st);
  return rc;
}
