// obca_lib.cu -- sm_90a kernels + the C-ABI of include/obca.h.
//
// Kernels
//   obca_phased.cuh          the parking solver: phase-split rounds (k_pk_eval, k_pk_sweep, k_pk_step) over all active
//                            problems + the persistent tail kernel k_pk_tail
//   k_quad_solve<SDV>        quadcopter model (config 4): persistent CTA per problem, block-cooperative KKT sweep on FP64 tensor cores (DMMA)
//   k_dualws<VM>             K2: one thread per (problem, stage, obstacle) micro interior-point solve.
//   k_check                  K5: ParkingConstraints twin + strict audit, one CTA per problem.
//   k_flow_list, k_flow_gather, k_flow_scatter   the index maps of obca_parking_plan_solve_goals (obca_flow.h): plans -> solve -> poses
//   k_qflow_gather, k_qflow_scatter              the same for obca_quadcopter_plan_solve (obca_qflow.h), with k_flow_list
//   k_check_batch_args       the device-pointer mixed entries' check of the per-problem horizons and sampling times in device memory
// There is NO CPU fallback: every compute entry point returns OBCA_ERR_NO_DEVICE without a CUDA device.
// Each solve and check family (parking solve, DualMultWS, parking check, quadcopter solve, quadcopter check) passes its arguments as one
// struct to one entry function, shared by its host-pointer entries and their device-pointer twins: the refusals in one order, the device
// context and lock once, the host staging or the wait on the caller's stream, then the family's device core, which the
// plan -> solve -> check flows call directly.  Host-pointer entries stage their arrays through one device buffer per device
// (DevCtx::stage), laid out, copied and scattered back with the helpers of obca_devstage.h, which the GPU planners (obca_plan.cu,
// obca_plan3d.cu) use for their per-call buffers too.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/obca.h"
#include "../../include/obca_planner.h"
#include "obca_check.cuh"
#include "obca_devstage.h"
#include "obca_dualws.cuh"
#include "obca_eval.cuh"
#include "obca_flow.h"
#include "obca_host.h"
#include "obca_phased.cuh"
#include "obca_qflow.h"

using namespace obca;

// ---------------------------------------------------------------------------------------------------------
// device-side batch description
// ---------------------------------------------------------------------------------------------------------
// Arrays laid out for the horizon P.N; Nb (optional): per-problem horizons, stages past Nb[b] are left alone.
template <int VM>
__global__ void k_dualws(const __grid_constant__ ParkProblem P, int B, const int* __restrict__ Nb, const double* __restrict__ rx,
                         const double* __restrict__ ry, const double* __restrict__ ryaw, double tol, int max_iter,
                         double* __restrict__ lp, double* __restrict__ np, double* __restrict__ dd) {
  const int NS = P.N + 1, nOb = P.nOb, V = P.V;
  const size_t total = (size_t)B * nOb * NS;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(idx % NS);
    const int j = (int)((idx / NS) % nOb);
    const size_t b = idx / ((size_t)NS * nOb);
    if (Nb && k > Nb[b]) continue;
    ObsRows<VM> R;
    R.v = P.vOb[j];
#pragma unroll
    for (int i = 0; i < VM; ++i) {
      const bool on = i < R.v;
      const int r = P.voff[j] + (on ? i : 0);
      R.a1[i] = on ? P.A[r][0] : 0.0; R.a2[i] = on ? P.A[r][1] : 0.0; R.bb[i] = on ? P.b[r] : 0.0;
    }
    double lam[VM], mu[4], d;
    const size_t o = (size_t)NS * b + k;
    dualws_solve<VM>(P, R, rx[o], ry[o], ryaw[o], tol, max_iter, lam, mu, &d);
#pragma unroll
    for (int i = 0; i < VM; ++i)
      if (i < R.v) lp[(size_t)V * NS * b + (size_t)(P.voff[j] + i) * NS + k] = lam[i];
#pragma unroll
    for (int m = 0; m < 4; ++m) np[(size_t)4 * nOb * NS * b + (size_t)(4 * j + m) * NS + k] = mu[m];
    if (dd) dd[(size_t)nOb * NS * b + (size_t)j * NS + k] = d;
  }
}

// K1 stand-alone (obca_eval.cuh): one thread per (problem, stage); consecutive threads = consecutive stages, so every
// warp streams contiguous slices of the stacked (x, u, l, n, sl, y) arrays.
template <int VM, bool SDV>
__global__ void __launch_bounds__(128)
k_parking_eval(const __grid_constant__ ParkProblem P, int B, EvalIn in, EvalOut out) {
  const int N = P.N, NS = N + 1, nOb = P.nOb, V = P.V;
  const size_t m = eval_m(P), n = eval_n(P);
  const size_t total = (size_t)B * NS;
  for (size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (size_t)gridDim.x * blockDim.x) {
    const size_t b = idx / NS;
    const int k = (int)(idx - b * NS);
    EvalIn ib;
    ib.x0 = in.x0 + 4 * b; ib.xF = in.xF + 4 * b; ib.rx = in.rx + NS * b; ib.ry = in.ry + NS * b; ib.ryaw = in.ryaw + NS * b;
    ib.xp = in.xp + (size_t)4 * NS * b; ib.up = in.up + (size_t)2 * N * b; ib.ts = in.ts ? in.ts + NS * b : nullptr;
    ib.lp = in.lp + (size_t)V * NS * b; ib.np = in.np + (size_t)4 * nOb * NS * b;
    ib.sl = in.sl ? in.sl + (size_t)nOb * NS * b : nullptr;
    ib.y = in.y ? in.y + m * b : nullptr;
    EvalOut ob;
    ob.c = out.c + m * b; ob.gradL = out.gradL + n * b; ob.fk = out.fk + NS * b;
    eval_stage<VM, SDV>(P, k, ib, ob);
  }
}

// Arrays laid out for the horizon P.N; Nb (optional): per-problem horizons, problem b is audited on its stages 0..Nb[b].
__global__ void k_check(const __grid_constant__ ParkProblem P, int B, const int* __restrict__ Nb, const double* __restrict__ x0,
                        const double* __restrict__ xF, const double* __restrict__ x, const double* __restrict__ u,
                        const double* __restrict__ l, const double* __restrict__ n, const double* __restrict__ ts,
                        const double* __restrict__ sl, int sd, int* __restrict__ feasible, int* __restrict__ e_out,
                        int* __restrict__ strict_out) {
  __shared__ ChkPart s_c[2][4];
  const int N = P.N, NS = N + 1, V = P.V, nOb = P.nOb;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const int Nprob = Nb ? Nb[b] : N;
    const double* xb = x + (size_t)4 * NS * b; const double* ub = u + (size_t)2 * N * b;
    const double* lb = l + (size_t)V * NS * b; const double* nb = n + (size_t)4 * nOb * NS * b;
    const double* tb = ts + (size_t)NS * b; const double* sb = sl ? sl + (size_t)nOb * NS * b : nullptr;
    ChkPart c[2];
    chk_init(c[0]); chk_init(c[1]);
    for (int k = threadIdx.x; k <= Nprob; k += blockDim.x) {
      for (int st = 0; st < 2; ++st) {
        ChkPart ck;
        check_stage(P, Nprob, k, x0 + 4 * (size_t)b, xF + 4 * (size_t)b, xb, ub, lb, nb, tb, sb, sd, st, ck);
        chk_merge(c[st], ck);
      }
    }
    for (int st = 0; st < 2; ++st) {
      for (int off = 16; off > 0; off >>= 1) {
        ChkPart o;
#pragma unroll
        for (int i = 0; i < 5; ++i) o.c0[i] = __shfl_down_sync(0xffffffffu, c[st].c0[i], off);
        o.c1 = __shfl_down_sync(0xffffffffu, c[st].c1, off); o.c2 = __shfl_down_sync(0xffffffffu, c[st].c2, off);
        o.c3 = __shfl_down_sync(0xffffffffu, c[st].c3, off); o.c4 = __shfl_down_sync(0xffffffffu, c[st].c4, off);
        o.c5 = __shfl_down_sync(0xffffffffu, c[st].c5, off); o.c6 = __shfl_down_sync(0xffffffffu, c[st].c6, off);
        o.sbox = __shfl_down_sync(0xffffffffu, c[st].sbox, off);
        chk_merge(c[st], o);
      }
      if ((threadIdx.x & 31) == 0) s_c[st][threadIdx.x >> 5] = c[st];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int st = 0; st < 2; ++st) {
        ChkPart m = s_c[st][0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) chk_merge(m, s_c[st][w]);
        int e[7];
        const int f = check_finish(P, m, tb, st, 5e-5, e);
        if (st == 0) {
          feasible[b] = f;
          if (e_out) for (int i = 0; i < 7; ++i) e_out[7 * (size_t)b + i] = e[i];
        } else if (strict_out) strict_out[b] = f;
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------
// plan -> solve -> check without leaving the device (obca_parking_plan_solve_goals): copies along the index maps of obca_flow.h
// ---------------------------------------------------------------------------------------------------------
// One CTA lists the poses obca_flow::listed takes, in pose order: list[q] = p, Nb[q] = its horizon; cnt[0] = the count, cnt[1] = the
// largest listed horizon.  A pose planned OK to a horizon the solver does not take gets OBCA_PLAN_CAPACITY.
constexpr int FLOW_LIST_THREADS = 1024;
__global__ void __launch_bounds__(FLOW_LIST_THREADS) k_flow_list(int B, int Ncap, int* __restrict__ status, const int* __restrict__ N,
                                                                 int* __restrict__ list, int* __restrict__ Nb, int* __restrict__ cnt) {
  __shared__ int s_warp[FLOW_LIST_THREADS / 32];
  __shared__ int s_base, s_max;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (threadIdx.x == 0) { s_base = 0; s_max = 0; }
  __syncthreads();
  for (int p0 = 0; p0 < B; p0 += blockDim.x) {
    const int p = p0 + threadIdx.x;
    bool on = false;
    if (p < B) {
      const int st = status[p], n = N[p];
      on = obca_flow::listed(st, n, Ncap);
      if (st == OBCA_PLAN_OK && !on) status[p] = OBCA_PLAN_CAPACITY;
      if (on) atomicMax(&s_max, n);
    }
    const unsigned m = __ballot_sync(0xffffffffu, on);
    if (lane == 0) s_warp[warp] = __popc(m);
    __syncthreads();
    int off = s_base + __popc(m & ((1u << lane) - 1));
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    if (on) { list[off] = p; Nb[off] = N[p]; }
    __syncthreads();
    if (threadIdx.x == 0)
      for (int w = 0; w < nw; ++w) s_base += s_warp[w];
    __syncthreads();
  }
  if (threadIdx.x == 0) { cnt[0] = s_base; cnt[1] = s_max; }
}

// One thread per (slot q < Bs, stage k <= M): the planner's outputs and x0 / xF of pose list[q] to the solve's inputs at the horizon M.
__global__ void k_flow_gather(int Bs, int M, int cap, const int* __restrict__ list, const int* __restrict__ Nb, const obca_flow::Gather g) {
  const size_t total = (size_t)Bs * (M + 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i / (M + 1)), k = (int)(i % (M + 1));
    obca_flow::gather_stage(g, q, list[q], Nb[q], k, M, cap);
  }
}

// One thread per (slot q < Bs, stage k <= M): the outputs of slot q (at the horizon M) to pose list[q] (at Ncap), its own horizon only.
__global__ void k_flow_scatter(int Bs, int M, int Ncap, int V, int nOb, const int* __restrict__ list, const int* __restrict__ Nb,
                               const obca_flow::Outs src, const obca_flow::Outs dst) {
  const size_t total = (size_t)Bs * (M + 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i / (M + 1)), k = (int)(i % (M + 1));
    obca_flow::scatter_stage(src, dst, V, nOb, q, list[q], Nb[q], k, M, Ncap);
  }
}

// The same two copies for obca_quadcopter_plan_solve (obca_qflow.h); k_flow_list lists its pairs.  One thread per (slot q < Bs, stage
// k <= M): pair list[q]'s path, x0 and xF to the warm start and inputs of the mixed solve at the horizon M, and its sampling time.
__global__ void k_qflow_gather(int Bs, int M, int cap, const int* __restrict__ list, const int* __restrict__ Nb, const obca_qflow::Gather g) {
  const size_t total = (size_t)Bs * (M + 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i / (M + 1)), k = (int)(i % (M + 1));
    obca_qflow::gather_stage(g, q, list[q], Nb[q], k, M, cap);
  }
}

__global__ void k_qflow_scatter(int Bs, int M, int Ncap, const int* __restrict__ list, const int* __restrict__ Nb,
                                const obca_qflow::Outs src, const obca_qflow::Outs dst) {
  const size_t total = (size_t)Bs * (M + 1);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int q = (int)(i / (M + 1)), k = (int)(i % (M + 1));
    obca_qflow::scatter_stage(src, dst, q, list[q], Nb[q], k, M, Ncap);
  }
}

// ---------------------------------------------------------------------------------------------------------
// quadcopter (obca_quad.cuh): persistent solver kernel + constrSatisfaction twin
// ---------------------------------------------------------------------------------------------------------
// Arrays laid out for the horizon c_qP.N.  Nb, Tsb (optional, together): per-problem horizons <= c_qP.N and sampling times;
// when null, every problem has the horizon c_qP.N and the sampling time c_qP.Ts.
struct QBatchPtrs {
  const double *x0, *xF, *xWS;
  const int* Nb;
  const double* Tsb;
  double timeWS;
  double *xp, *up, *ts, *lp, *slack;
  int *exitflag, *iters;
  double* kkt_err;
  int B;
  unsigned long long* prof;   // 8 per-phase cycle counters summed over the batch (see obca_last_profile)
};

#ifndef OBCA_MINB_Q
#define OBCA_MINB_Q 2
#endif
template <bool SDV>
__global__ void __launch_bounds__(QUAD_CTA, OBCA_MINB_Q)
k_quad_solve(const __grid_constant__ QuadProblem P, const __grid_constant__ IpmOpts O, const QLay L, const QBatchPtrs bp,
             double* __restrict__ Wall, int* __restrict__ counter) {
  extern __shared__ double s_kkt[];      // QuadSolver::smem_doubles(N): block-cooperative KKT sweep
  __shared__ ProbState S;
  __shared__ double s_red[(QUAD_CTA / 32) * 12];      // one partial per warp (launched with at most QUAD_CTA threads)
  __shared__ int s_b;
  __shared__ double s_sum[QUAD_CTA / 32];
  const int N = P.N, NS = N + 1;      // the layout: strides of the per-problem arrays
  double* W = Wall + (size_t)blockIdx.x * L.total * L.NSP;
  for (;;) {
    if (threadIdx.x == 0) s_b = atomicAdd(counter, 1);
    __syncthreads();
    const int b = s_b;
    if (b >= bp.B) break;
    QCtx C;
    C.P = &P; C.O = &O; C.L = L; C.W = W; C.red_scratch = s_red; C.tile = s_kkt; C.S = &S;
    C.N = bp.Nb ? bp.Nb[b] : c_qP.N; C.Ts = bp.Tsb ? bp.Tsb[b] : c_qP.Ts;      // this problem's horizon and sampling time
    C.in.x0 = bp.x0 + 12 * (size_t)b; C.in.xF = bp.xF + 12 * (size_t)b; C.in.xWS = bp.xWS + (size_t)12 * NS * b;
    C.in.timeWS = bp.timeWS;
    QOutputs out;
    out.xp = bp.xp + (size_t)12 * NS * b; out.up = bp.up + (size_t)4 * N * b; out.ts = bp.ts + (size_t)NS * b;
    out.lp = bp.lp + (size_t)30 * NS * b; out.slack = bp.slack ? bp.slack + (size_t)5 * NS * b : nullptr;
    IpmDriver<QuadSolver<SDV> >::solve(C);      // flag = 1 in the reference: a single attempt (QuadcopterSignedDist.jl:227-235)
    __syncthreads();
    double ssum = 0.0;
    const int Np = C.N;
    for (int k = threadIdx.x; k <= Np; k += blockDim.x) {
      QuadSolver<SDV>::store_stage(C, k, out);
      if (SDV) for (int j = 0; j < QNOB; ++j) ssum += W[(size_t)(L.SLK + j) * L.NSP + k];
    }
    for (int off = 16; off > 0; off >>= 1) ssum += __shfl_down_sync(0xffffffffu, ssum, off);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = ssum;
    __syncthreads();
    if (threadIdx.x == 0) {
      double tot = 0.0;
      for (int w = 0; w < QuadSolver<SDV>::own_warps(C); ++w) tot += s_sum[w];      // the problem's own warps (see reduce)
      int ef = S.status == 1 ? 1 : 0;
      if (SDV && ef == 1 && tot > 1e-3) ef = 2;      // sum-slack gate, QuadcopterSignedDist.jl:283-288
      bp.exitflag[b] = ef; bp.iters[b] = S.iters; bp.kkt_err[b] = S.e0;
      if (bp.prof)
        for (int i = 0; i < 8; ++i) atomicAdd(bp.prof + i, (unsigned long long)S.prof[i]);
    }
    __syncthreads();
  }
}

// Arrays laid out for the horizon P.N; Nb, Tsb (optional, together): problem b is checked on its stages 0..Nb[b] with the
// sampling time Tsb[b].
__global__ void k_quad_check(const __grid_constant__ QuadProblem P, int B, const int* __restrict__ Nb, const double* __restrict__ Tsb,
                             const double* __restrict__ x0, const double* __restrict__ xF, const double* __restrict__ x,
                             const double* __restrict__ u, const double* __restrict__ ts, const double* __restrict__ lam,
                             int* __restrict__ feasible, double* __restrict__ worst_out) {
  __shared__ double s_w[4], s_l[4];
  const int N = P.N, NS = N + 1;
  for (int b = blockIdx.x; b < B; b += gridDim.x) {
    const int Np = Nb ? Nb[b] : N;
    const double Tsp = Tsb ? Tsb[b] : P.Ts;
    double w = 0.0, wl = -1e300;      // the stages' groups; the lambda group, max(-lambda) over all columns (NaN if one is NaN)
    for (int k = threadIdx.x; k <= Np; k += blockDim.x) {
      double lk;
      w = fmax(w, quad_check_stage(P, Np, Tsp, k, x0 + 12 * (size_t)b, xF + 12 * (size_t)b, x + (size_t)12 * NS * b, u + (size_t)4 * N * b,
                                   ts + (size_t)NS * b, lam + (size_t)30 * NS * b, &lk));
      wl = dmax_nan(wl, lk);
    }
    for (int off = 16; off > 0; off >>= 1) {
      w = fmax(w, __shfl_down_sync(0xffffffffu, w, off));
      wl = dmax_nan(wl, __shfl_down_sync(0xffffffffu, wl, off));
    }
    if ((threadIdx.x & 31) == 0) { s_w[threadIdx.x >> 5] = w; s_l[threadIdx.x >> 5] = wl; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < (int)(blockDim.x >> 5); ++i) { w = fmax(w, s_w[i]); wl = dmax_nan(wl, s_l[i]); }
      if (wl == wl) w = fmax(w, wl);      // a NaN anywhere in lambda turns the lambda group off (:162), not the others
      feasible[b] = w <= 1e-3 ? 1 : 0;
      if (worst_out) worst_out[b] = w;
    }
    __syncthreads();
  }
}

// The device-pointer entries' check of a device-resident batch (obca_*_mixed_dev): the first problem i whose horizon Nb[i] lies
// outside [2, Nmax], or (Tsb not null) whose sampling time Tsb[i] is not a finite number > 0, as the key (order << 32) | Nb[i] in
// *first_bad, which starts at ~0.  order = i for a bad horizon and B + i for a bad sampling time: a bad horizon anywhere in the batch
// comes first, as the host-pointer entries check all horizons before any sampling time.
__global__ void k_check_batch_args(int B, const int* __restrict__ Nb, int Nmax, const double* __restrict__ Tsb,
                                   unsigned long long* __restrict__ first_bad) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)B; i += (size_t)gridDim.x * blockDim.x) {
    const int n = Nb[i];
    if (n < 2 || n > Nmax) atomicMin(first_bad, (unsigned long long)i << 32 | (unsigned)n);
    if (Tsb && !(isfinite(Tsb[i]) && Tsb[i] > 0.0)) atomicMin(first_bad, (unsigned long long)(B + i) << 32);
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static void set_err(const std::string& s) { g_err = s; }
// the GPU planner's translation unit (obca_plan.cu, built without FMA contraction) reports through obca_last_error() as well
void obca_set_last_error(const std::string& s) { g_err = s; }
struct DevCtx {
  bool init = false;
  cudaStream_t st = nullptr;
  cudaEvent_t ev0 = nullptr, evm = nullptr, ev1 = nullptr;
  cudaEvent_t evs = nullptr;                        // device-pointer entries: recorded on the caller's stream, waited for on st
  unsigned long long* bad = nullptr;                // k_check_batch_args: the first bad problem of a device-resident batch
  int sms = 0;
  double* W = nullptr; size_t Wbytes = 0;
  int* counter = nullptr;
  unsigned long long* prof = nullptr;
  unsigned long long prof_host[8] = {0};
  char* stage = nullptr; size_t stage_bytes = 0;   // device staging for the host-pointer API
  double* wsd = nullptr; size_t wsd_bytes = 0;     // warm-start duals of DualMultWS when the caller passes lWS = nWS = NULL
  // phase-split driver (obca_phased.cuh)
  double* slots = nullptr; size_t slots_bytes = 0;  // stage slots of every problem, B x (N+1) x RSTRIDE
  char* pstate = nullptr; size_t pstate_bytes = 0;  // ProbState per problem
  int* act = nullptr; size_t act_bytes = 0;         // two active lists
  int* ncnt = nullptr;                              // device: three rotating active counts, [3] tail work counter,
                                                    // [4] / [5] work queues of k_pk_eval / k_pk_step
  int* h_n = nullptr;                               // pinned ring of active counts read back per round
  cudaEvent_t evr[16] = {nullptr};
  std::vector<cudaEvent_t> tev;                     // OBCA_PHASE_TIMING=1: pool of timing events
  int last_rounds = 0, last_tail = 0;
  double phase_ms[5] = {0, 0, 0, 0, 0};             // OBCA_PHASE_TIMING=1: summed event times of eval, sweep, step, tail; [4] DualMultWS
  double last_dualws_s = 0.0, last_solve_s = 0.0;
  std::recursive_mutex mu;
};
constexpr int MAX_DEVICES = 64;
static DevCtx g_dev[MAX_DEVICES];
static std::mutex g_init_mu;

static int get_ctx(int dev, DevCtx** out) {
  const int rc = check_device(dev);
  if (rc) return rc;
  if (dev >= MAX_DEVICES) { set_err("bad device ordinal"); return OBCA_ERR_ARG; }
  DevCtx& c = g_dev[dev];
  CK(cudaSetDevice(dev));
  std::lock_guard<std::mutex> lk(g_init_mu);
  if (!c.init) {
    CK(cudaStreamCreateWithFlags(&c.st, cudaStreamNonBlocking));
    CK(cudaEventCreate(&c.ev0)); CK(cudaEventCreate(&c.evm)); CK(cudaEventCreate(&c.ev1));
    cudaDeviceProp pr;
    CK(cudaGetDeviceProperties(&pr, dev));
    c.sms = pr.multiProcessorCount;
    CK(cudaEventCreateWithFlags(&c.evs, cudaEventDisableTiming));
    CK(cudaMalloc(&c.bad, sizeof(unsigned long long)));
    CK(cudaMalloc(&c.counter, sizeof(int)));
    CK(cudaMalloc(&c.prof, 8 * sizeof(unsigned long long)));
    CK(cudaMalloc(&c.ncnt, 6 * sizeof(int)));
    CK(cudaMallocHost(&c.h_n, 16 * sizeof(int)));
    for (int i = 0; i < 16; ++i) CK(cudaEventCreateWithFlags(&c.evr[i], cudaEventDisableTiming));
    c.init = true;
  }
  *out = &c;
  return 0;
}
// the context of a device that has run a call (obca_last_*), or null
static const DevCtx* used_ctx(int dev) { return dev >= 0 && dev < MAX_DEVICES && g_dev[dev].init ? &g_dev[dev] : nullptr; }
static int ensure(void** p, size_t* have, size_t need) {
  if (*have >= need) return 0;
  if (*p) cudaFree(*p);
  *p = nullptr; *have = 0;
  CK(cudaMalloc(p, need));
  *have = need;
  return 0;
}

static IpmOpts to_ipm(const obca_opts* o) {
  IpmOpts r = default_opts();
  if (!o) return r;
  r.tol = o->tol; r.max_iter = o->max_iter; r.mu_init = o->mu_init; r.mu_min = o->mu_min;
  r.kappa_eps = o->kappa_eps; r.kappa_mu = o->kappa_mu; r.theta_mu = o->theta_mu; r.tau_min = o->tau_min;
  r.kappa1 = o->kappa1; r.kappa2 = o->kappa2; r.kappa_sigma = o->kappa_sigma; r.s_max = o->s_max;
  r.dual_inf_tol = o->dual_inf_tol; r.constr_viol_tol = o->constr_viol_tol; r.compl_inf_tol = o->compl_inf_tol;
  r.dw_min = o->dw_min; r.dw_first = o->dw_first; r.dw_max = o->dw_max; r.kw_minus = o->kw_minus;
  r.kw_plus = o->kw_plus; r.kw_plus_first = o->kw_plus_first;
  r.gamma_theta = o->gamma_theta; r.gamma_phi = o->gamma_phi; r.delta = o->delta; r.s_theta = o->s_theta;
  r.s_phi = o->s_phi; r.eta_phi = o->eta_phi; r.gamma_alpha = o->gamma_alpha; r.max_backtrack = o->max_backtrack;
  r.dc = o->dc; r.max_kick = o->max_kick; r.quad_dual_ws = o->quad_dual_ws;
  return r;
}

static int run_dualws(DevCtx& c, const ParkProblem& P, int B, const int* Nb, const double* rx, const double* ry,
                      const double* ryaw, double* lp, double* np, double* dd) {
  const size_t total = (size_t)B * P.nOb * (P.N + 1);
  const int threads = 128;
  const int blocks = (int)((total + threads - 1) / threads);
  with_variant(P, [&](auto vm, auto) {      // the multipliers do not depend on the formulation
    k_dualws<decltype(vm)::value><<<blocks, threads, 0, c.st>>>(P, B, Nb, rx, ry, ryaw, 1e-5, 100, lp, np, dd);
    return 0;
  });
  CK(cudaGetLastError());
  return 0;
}

// ---------------------------------------------------------------------------------------------------------
// phase-split driver (obca_phased.cuh): rounds of [K_A, K_B, K_C] over the active problems, then the tail kernel
// ---------------------------------------------------------------------------------------------------------
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}

// Where k_pk_step keeps the step rows dLAM .. dRS (V + 10 nOb + 5 rows of NSP doubles): in shared memory while the kernel
// still has OBCA_STEP_SMEM_MIN_CTAS resident CTAs per SM with them there, else in the workspace (no dynamic shared memory).
// The default is the kernel's launch bound (the reference's scenes at N = 80 need 40-51 rows and stay in shared memory);
// profiles/lot_h100.md has the measurement behind the rule.
#ifndef OBCA_STEP_SMEM_MIN_CTAS
#define OBCA_STEP_SMEM_MIN_CTAS OBCA_MINB_C
#endif
template <class K>
static cudaError_t step_rows_in_smem(K kernel, const PkLay& L, int* in_smem, size_t* smem) {
  const size_t need = (size_t)(L.dRS + 1 - L.dLAM) * L.NSP * sizeof(double);
  int dev = 0, optin = 0, occ = 0;
  cudaFuncAttributes fa;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, kernel);
  *in_smem = 0; *smem = 0;
  // a CTA's dynamic and static shared memory together may not exceed the opt-in limit
  if (e != cudaSuccess || need + fa.sharedSizeBytes > (size_t)optin) return e;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)need);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, PK_THREADS, need);
  if (e == cudaSuccess && occ >= OBCA_STEP_SMEM_MIN_CTAS) { *in_smem = 1; *smem = need; }
  return e;
}

template <int VM, bool SDV>
static int launch_phased(DevCtx& c, const ParkProblem& P, const IpmOpts& O, const BatchPtrs& bp, int mode) {
  PkLay L = make_layout(P, LocalDims<VM, SDV>::NFAC);
  const int B = bp.B, NS = P.N + 1;
  const size_t smem_slots = (size_t)NS * RSTRIDE * sizeof(double);
  {   // the entries check N <= OBCA_PK_NMAX, which is sized for the H100: a device with less shared memory per CTA refuses here
    int dev = 0, optin = 0;
    cudaFuncAttributes fe, ft;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    CK(cudaFuncGetAttributes(&fe, k_pk_eval<VM, SDV>));
    CK(cudaFuncGetAttributes(&ft, k_pk_tail<VM, SDV>));
    const size_t st = fe.sharedSizeBytes > ft.sharedSizeBytes ? fe.sharedSizeBytes : ft.sharedSizeBytes;
    if (smem_slots + st > (size_t)optin) {
      set_err("horizon too long for this device: N + 1 = " + std::to_string(NS) + " stage slots need " + std::to_string(smem_slots + st) +
              " bytes of shared memory per CTA, the device allows " + std::to_string(optin));
      return OBCA_ERR_UNSUPPORTED;
    }
  }
  CK(cudaFuncSetAttribute(k_pk_eval<VM, SDV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_slots));
  CK(cudaFuncSetAttribute(k_pk_tail<VM, SDV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_slots));
  const size_t smem_sweep = (size_t)SWEEP_WARPS * SWEEP_WARP_DOUBLES * sizeof(double);
  CK(cudaFuncSetAttribute(k_pk_sweep<VM, SDV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sweep));
  size_t smem_step = 0;
  int step_smem = 0;
  CK(step_rows_in_smem(k_pk_step<VM, SDV>, L, &step_smem, &smem_step));
  int occ_t = 0, occ_e = 0, occ_s = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_t, k_pk_tail<VM, SDV>, PK_THREADS, smem_slots));
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_e, k_pk_eval<VM, SDV>, PK_THREADS, smem_slots));
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_s, k_pk_step<VM, SDV>, PK_THREADS, smem_step));
  if (occ_t < 1) occ_t = 1;
  if (occ_e < 1) occ_e = 1;
  if (occ_s < 1) occ_s = 1;
  {   // development: fewer resident CTAs per SM than the occupancy allows (how much do co-resident CTAs slow each other down?)
    const int oe = env_int("OBCA_EVAL_OCC", occ_e), os = env_int("OBCA_STEP_OCC", occ_s);
    if (oe >= 1 && oe < occ_e) occ_e = oe;
    if (os >= 1 && os < occ_s) occ_s = os;
  }
  const int tail_cap = c.sms * occ_t, eval_cap = c.sms * occ_e, step_cap = c.sms * occ_s;
  int rc = ensure((void**)&c.W, &c.Wbytes, (size_t)B * L.total * L.NSP * sizeof(double));
  if (rc) return rc;
  rc = ensure((void**)&c.pstate, &c.pstate_bytes, (size_t)B * sizeof(ProbState));
  if (rc) return rc;
  ProbState* Sg = (ProbState*)c.pstate;
  cudaStream_t st = c.st;
  // mode 1: tail kernel only; mode 2: rounds only (until the active set is empty, or OBCA_TAIL_THRESH if set); auto: rounds for
  // large batches until the active set has shrunk to the hand-over point, then the tail kernel.  Hand-over point: measured on
  // an H100 SXM (700 W, config 2, B = 4096) the solve time is flat (135.7-138.0 ms) between 1536 and 3072 remaining problems
  // and higher below (142.0 ms at 1024, 146.6 ms at 512): lock-step rounds do more evaluations per second while all SMs are
  // busy, the persistent kernel finishes the stragglers without a launch-bound round per iteration.
  const int thresh = env_int("OBCA_TAIL_THRESH", mode == 2 ? 0 : (B / 2 > tail_cap ? B / 2 : tail_cap));
  const bool rounds = mode == 2 || (mode == 0 && B > 2 * tail_cap);
  c.last_rounds = 0; c.last_tail = B;
  int h_init[6] = {B, 0, 0, 0, 0, 0};
  CK(cudaMemcpyAsync(c.ncnt, h_init, 6 * sizeof(int), cudaMemcpyHostToDevice, st));
  if (!rounds) {
    const int grid = B < tail_cap ? B : tail_cap;
    k_pk_tail<VM, SDV><<<grid, PK_THREADS, smem_slots, st>>>(P, O, L, bp, c.W, Sg, nullptr, c.ncnt, c.ncnt + 3, 1);
    CK(cudaGetLastError());
    return 0;
  }
  rc = ensure((void**)&c.slots, &c.slots_bytes, (size_t)B * NS * RSTRIDE * sizeof(double));
  if (rc) return rc;
  rc = ensure((void**)&c.act, &c.act_bytes, 2 * (size_t)B * sizeof(int));
  if (rc) return rc;
  int* act[2] = {c.act, c.act + B};
  int n_bound = B, done_r = 0, r = 0;
  const int max_rounds = 8 * (O.max_iter + 8);
  const bool timing = env_int("OBCA_PHASE_TIMING", 0) != 0;      // development / bench: per-kernel event times, summed per solve
  size_t n_ev = 0;
  auto mark = [&]() {
    if (!timing) return;
    if (n_ev == c.tev.size()) { cudaEvent_t e; cudaEventCreate(&e); c.tev.push_back(e); }
    cudaEventRecord(c.tev[n_ev++], st);
  };
  auto cap = [](int n, int m) { return n < m ? (n > 0 ? n : 1) : m; };
  // one round = three launches + the read-back of the active count; grids from an upper bound nb of the active count.  Work
  // queues: k_pk_eval takes from ncnt[4] and zeroes ncnt[5] for the k_pk_step of its round, which zeroes ncnt[4] in turn.
  // The two launches must stay paired and alternate: a schedule that launches one without the other (a k_pk_step alone before
  // the hand-over, say) has to zero the counter it takes from itself, or the launch finds it spent and skips every problem.
  auto launch_round = [&](int rr, int nb, bool readback) -> int {
    const int* a_in = act[rr & 1]; int* a_out = act[(rr + 1) & 1];
    int* n_in = c.ncnt + (rr % 3); int* n_out = c.ncnt + ((rr + 1) % 3); int* n_zero = c.ncnt + ((rr + 2) % 3);
    int* q_eval = c.ncnt + 4; int* q_step = c.ncnt + 5;
    mark();
    k_pk_eval<VM, SDV><<<cap(nb, eval_cap), PK_THREADS, smem_slots, st>>>(P, O, L, bp, c.W, c.slots, Sg, a_in, n_in, a_out, n_out, rr == 0 ? 1 : 0,
                                                                          q_eval, q_step);
    mark();
    k_pk_sweep<VM, SDV><<<(nb + SWEEP_WARPS - 1) / SWEEP_WARPS, 32 * SWEEP_WARPS, smem_sweep, st>>>(P, O, L, c.W, c.slots, Sg, a_out, n_out, n_zero);
    mark();
    k_pk_step<VM, SDV><<<cap(nb, step_cap), PK_THREADS, smem_step, st>>>(P, O, L, bp, c.W, c.slots, Sg, a_out, n_out, q_step, q_eval,
                                                                          step_smem);
    mark();
    CK(cudaGetLastError());
    if (readback) CK(cudaMemcpyAsync(c.h_n + (rr & 15), n_out, sizeof(int), cudaMemcpyDeviceToHost, st));
    return 0;
  };
  // Rounds as a CUDA graph: the buffer pattern of a round (active lists: period 2, counters: period 3) repeats every 6 rounds, so
  // rounds 1..6 are captured once per call and the graph is replayed -- about 14 driver calls per solve instead of ~420
  // (3 launches + copy + event per round), which is what paces the host when 8 ranks share one box.  The grids inside the graph
  // are those of the count at capture time (an upper bound later on: surplus CTAs / warps exit at once); the host looks at the
  // active count once per replay, one replay behind, so the hand-over point is overshot by up to 12 rounds (the solve time is
  // flat there, see above).  OBCA_GRAPH=0 or OBCA_PHASE_TIMING=1: plain launches, count read back every round.
  const bool use_graph = !timing && env_int("OBCA_GRAPH", 1) != 0;
  if (use_graph) {
    rc = launch_round(0, B, true);
    if (rc) return rc;
    r = 1;
    cudaGraph_t graph = nullptr; cudaGraphExec_t gexec = nullptr;
    CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
    for (int q = 0; q < 6 && rc == 0; ++q) rc = launch_round(1 + q, B, q == 5);
    cudaError_t ce = cudaStreamEndCapture(st, &graph);
    if (rc) { if (graph) cudaGraphDestroy(graph); return rc; }
    CK(ce);
    CK(cudaGraphInstantiate(&gexec, graph, 0));
    int g = 0;
    for (; r < max_rounds; ++g) {
      CK(cudaGraphLaunch(gexec, st));
      CK(cudaEventRecord(c.evr[g & 1], st));
      r += 6;
      if (g >= 1) {
        CK(cudaEventSynchronize(c.evr[(g - 1) & 1]));
        n_bound = c.h_n[(1 + 5) & 15];      // count after the last round of a replay (the replay in flight may refresh it: still a bound)
        if (n_bound <= thresh) break;
      }
    }
    CK(cudaStreamSynchronize(st));
    n_bound = c.h_n[(1 + 5) & 15];
    cudaGraphExecDestroy(gexec); cudaGraphDestroy(graph);
  } else {
    for (; r < max_rounds; ++r) {
      rc = launch_round(r, n_bound, true);
      if (rc) return rc;
      CK(cudaEventRecord(c.evr[r & 15], st));
      // the active set only shrinks: the count of any completed round bounds every later round
      if (r - done_r >= 8) CK(cudaEventSynchronize(c.evr[done_r & 15]));
      while (done_r <= r && cudaEventQuery(c.evr[done_r & 15]) == cudaSuccess) { n_bound = c.h_n[done_r & 15]; ++done_r; }
      if (n_bound <= thresh) {
        CK(cudaStreamSynchronize(st));
        n_bound = c.h_n[r & 15];
        ++r;
        break;
      }
    }
  }
  c.last_rounds = r; c.last_tail = n_bound;
  if (timing) {
    CK(cudaStreamSynchronize(st));
    double t[3] = {0, 0, 0};      // four marks per round: | eval | sweep | step |
    for (size_t i = 0; i + 3 < n_ev; i += 4)
      for (int j = 0; j < 3; ++j) { float ms = 0.f; cudaEventElapsedTime(&ms, c.tev[i + j], c.tev[i + j + 1]); t[j] += ms; }
    for (int j = 0; j < 3; ++j) c.phase_ms[j] += t[j];
  }
  if (n_bound > 0) {
    // after r rounds the active list is act[r & 1] with count ncnt[r % 3]
    const int grid = n_bound < tail_cap ? n_bound : tail_cap;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (timing) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, st); }
    k_pk_tail<VM, SDV><<<grid, PK_THREADS, smem_slots, st>>>(P, O, L, bp, c.W, Sg, act[r & 1], c.ncnt + (r % 3), c.ncnt + 3, 0);
    CK(cudaGetLastError());
    if (timing) {
      cudaEventRecord(e1, st); cudaEventSynchronize(e1);
      float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1); c.phase_ms[3] += ms;
      cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
  }
  return 0;
}

// Elements per problem of a batch's per-problem arrays laid out for the horizon N, for the host code (staging, chunks, scratch, the
// flows' layouts): ns = N + 1 (stages: time scales, reference path), then states, inputs, multipliers and slacks.
struct ParkSizes { size_t ns, x, u, l, n, sl; };      // N + 1, 4 (N + 1), 2N, V (N + 1), 4 nOb (N + 1), nOb (N + 1)
static ParkSizes park_sizes(int N, int V, int nOb) {
  const size_t ns = (size_t)N + 1;
  return {ns, 4 * ns, 2 * (size_t)N, V * ns, 4 * (size_t)nOb * ns, nOb * ns};
}
struct QuadSizes { size_t ns, x, u, l, s; };          // N + 1, 12 (N + 1), 4N, 30 (N + 1), 5 (N + 1)
static QuadSizes quad_sizes(int N) {
  const size_t ns = (size_t)N + 1;
  return {ns, 12 * ns, 4 * (size_t)N, 30 * ns, 5 * ns};
}

static int solve_dev_impl(DevCtx& c, const ParkProblem& P, const IpmOpts& O, BatchPtrs bp, double* seconds) {
  // problem, options and workspace layout -> __constant__ memory (stream-ordered with the kernels below)
  const PkLay Lc = make_layout(P, nfac_for(P));
  CK(cudaMemcpyToSymbolAsync(c_pkP, &P, sizeof(P), 0, cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyToSymbolAsync(c_pkO, &O, sizeof(O), 0, cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyToSymbolAsync(c_pkL, &Lc, sizeof(Lc), 0, cudaMemcpyHostToDevice, c.st));
  CK(cudaMemsetAsync(c.prof, 0, 8 * sizeof(unsigned long long), c.st));
  bp.prof = c.prof;
  for (int i = 0; i < 4; ++i) c.phase_ms[i] = 0.0;
  int rc;
  const int mode = env_int("OBCA_MODE", 0);
  // large batches are solved in chunks so that the per-problem workspace (0.19 MB for config 2, 0.6 MB at 11 obstacles, N = 80;
  // INTEGRATION.md section 3a) stays within a few GB.  Past NSP = 128 doubles per row the chunk shrinks with the row length, so
  // that no shape needs more memory per chunk than it does at N = 127.
  const int chunk = env_int("OBCA_CHUNK", Lc.NSP > 128 ? 16384 * 128 / Lc.NSP : 16384);
  const ParkSizes z = park_sizes(P.N, P.V, P.nOb);
  rc = 0;
  for (int b0 = 0; b0 < bp.B && rc == 0; b0 += chunk) {
    BatchPtrs q = bp;
    q.B = bp.B - b0 < chunk ? bp.B - b0 : chunk;
    const size_t o = (size_t)b0;
    q.x0 += 4 * o; q.xF += 4 * o; q.rx += z.ns * o; q.ry += z.ns * o; q.ryaw += z.ns * o; q.xWS += z.x * o; q.uWS += z.u * o;
    q.lWS += z.l * o; q.nWS += z.n * o;
    q.xp += z.x * o; q.up += z.u * o; q.ts += z.ns * o; q.lp += z.l * o; q.np += z.n * o;
    if (q.sl) q.sl += z.sl * o;
    if (q.duals) q.duals += ((size_t)4 * P.N + z.n) * o;
    if (q.Nb) q.Nb += o;
    q.exitflag += o; q.iters += o; q.kkt_err += o;
#ifdef OBCA_FAST_BUILD   // development builds: only the config-2 instantiation
    if (!(P.signed_dist && max_vob(P) <= 2)) { set_err("fast build: only <2,true>"); return OBCA_ERR_UNSUPPORTED; }
    rc = launch_phased<2, true>(c, P, O, q, mode);
#else
    // OBCA_MODE: 0 auto (phase-split rounds for large batches + tail kernel for the stragglers, tail kernel alone for small
    // batches), 1 tail kernel only, 2 rounds only
    rc = with_variant(P, [&](auto vm, auto sdv) { return launch_phased<decltype(vm)::value, decltype(sdv)::value>(c, P, O, q, mode); });
#endif
  }
  if (rc) return rc;
  CK(cudaEventRecord(c.ev1, c.st));
  CK(cudaMemcpyAsync(c.prof_host, c.prof, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c.st));
  CK(cudaStreamSynchronize(c.st));
  // the reference's `time` is the wall time of solve(m) alone (ParkingSignedDist.jl:239-241,297): DualMultWS (:219) and
  // the model build are outside it.  ev0 .. evm = DualMultWS (when the library runs it), evm .. ev1 = the solve.
  float ms = 0.f, ms_ws = 0.f;
  CK(cudaEventElapsedTime(&ms, c.evm, c.ev1));
  CK(cudaEventElapsedTime(&ms_ws, c.ev0, c.evm));
  c.last_solve_s = ms * 1e-3; c.last_dualws_s = ms_ws * 1e-3; c.phase_ms[4] = ms_ws;
  if (seconds) *seconds = ms * 1e-3;
  return 0;
}

template <bool SDV>
static int launch_quad(DevCtx& c, const QuadProblem& P, const IpmOpts& O, const QBatchPtrs& bp) {
  QLay L = make_qlayout(P);
  // the workspace rows keep the stride NSP = round32(N+1); past QUAD_CTA stages a thread handles several of them
  const int threads = L.NSP < QUAD_CTA ? L.NSP : QUAD_CTA;
  const size_t smem = (size_t)QuadSolver<SDV>::smem_doubles(P.N) * sizeof(double);
  if (smem > 200 * 1024) { set_err("horizon too long for the quadcopter kernel's shared memory"); return OBCA_ERR_UNSUPPORTED; }
  CK(cudaFuncSetAttribute(k_quad_solve<SDV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int occ = 0;
  CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_quad_solve<SDV>, threads, smem));
  if (occ < 1) occ = 1;
  int grid = c.sms * occ;
  if (grid > bp.B) grid = bp.B;
  const size_t need = (size_t)grid * L.total * L.NSP * sizeof(double);
  int rc = ensure((void**)&c.W, &c.Wbytes, need);
  if (rc) return rc;
  CK(cudaMemcpyToSymbolAsync(c_pkO, &O, sizeof(O), 0, cudaMemcpyHostToDevice, c.st));   // IpmDriver reads the options here
  CK(cudaMemcpyToSymbolAsync(c_qP, &P, sizeof(P), 0, cudaMemcpyHostToDevice, c.st));
  CK(cudaMemcpyToSymbolAsync(c_qL, &L, sizeof(L), 0, cudaMemcpyHostToDevice, c.st));
  CK(cudaMemsetAsync(c.counter, 0, sizeof(int), c.st));
  k_quad_solve<SDV><<<grid, threads, smem, c.st>>>(P, O, L, bp, c.W, c.counter);
  CK(cudaGetLastError());
  return 0;
}

// The parking solver's horizon bound, checked by every solve entry before any device work: a refused call launches nothing and
// writes no output.
static int check_park_horizon(int N) {
  if (N <= OBCA_PK_NMAX) return 0;
  set_err("horizon too long for the parking solver: N = " + std::to_string(N) + " > " + std::to_string(OBCA_PK_NMAX) +
          " (N + 1 <= " + std::to_string(OBCA_PK_NMAX + 1) + " stages)");
  return OBCA_ERR_UNSUPPORTED;
}

// The quadcopter solver's horizon bound, checked before any device work: a refused call launches nothing and writes no output.
static int check_quad_horizon(int N) {
  if (N <= QUAD_NMAX) return 0;
  set_err("horizon too long for the quadcopter solver: N = " + std::to_string(N) + " > " + std::to_string(QUAD_NMAX) +
          " (N + 1 <= " + std::to_string(QUAD_NMAX + 1) + " stages)");
  return OBCA_ERR_UNSUPPORTED;
}

// The refusal of problem q's horizon n outside [2, Nmax] and of its sampling time t (not finite and > 0), for host- and device-resident
// batches alike.
static int bad_horizon(int q, int n, int Nmax) {
  set_err("Nb[" + std::to_string(q) + "] = " + std::to_string(n) + " outside [2, Nmax = " + std::to_string(Nmax) + "]");
  return OBCA_ERR_ARG;
}
static int bad_sampling_time(int q, double t) {
  set_err("Tsb[" + std::to_string(q) + "] = " + std::to_string(t) + " is not a finite sampling time > 0");
  return OBCA_ERR_ARG;
}

// per-problem horizons: Nb present and, in host memory, every Nb[q] in [2, Nmax] (in device memory: check_batch_args_dev)
static int check_horizons(int B, const int* Nb, int Nmax, bool on_host) {
  if (!Nb) { set_err("null argument: Nb"); return OBCA_ERR_ARG; }
  for (int q = 0; on_host && q < B; ++q)
    if (Nb[q] < 2 || Nb[q] > Nmax) return bad_horizon(q, Nb[q], Nmax);
  return 0;
}

// per-problem sampling times: Tsb present and, in host memory, every Tsb[q] finite and > 0 (in device memory: check_batch_args_dev)
static int check_sampling_times(int B, const double* Tsb, bool on_host) {
  if (!Tsb) { set_err("null argument: Tsb"); return OBCA_ERR_ARG; }
  for (int q = 0; on_host && q < B; ++q)
    if (!(std::isfinite(Tsb[q]) && Tsb[q] > 0.0)) return bad_sampling_time(q, Tsb[q]);
  return 0;
}

// check_horizons and (Tsb not null) check_sampling_times for device-resident Nb and Tsb, with their messages: k_check_batch_args on the
// library's stream, then one 8-byte readback decides (a refused sampling time reads its value back for the message).  Runs before any
// output is written.
static int check_batch_args_dev(DevCtx& c, int B, const int* Nb, int Nmax, const double* Tsb) {
  CK(cudaMemsetAsync(c.bad, 0xff, sizeof(unsigned long long), c.st));
  const int threads = 256, need = (int)(((size_t)B + threads - 1) / threads), blocks = need < 4 * c.sms ? need : 4 * c.sms;
  k_check_batch_args<<<blocks, threads, 0, c.st>>>(B, Nb, Nmax, Tsb, c.bad);
  CK(cudaGetLastError());
  unsigned long long bad = 0;
  CK(to_host(&bad, c.bad, 1, c.st));
  CK(cudaStreamSynchronize(c.st));
  if (bad == ~0ull) return 0;
  const long long order = (long long)(bad >> 32);
  if (order < B) return bad_horizon((int)order, (int)(unsigned)bad, Nmax);
  const int q = (int)(order - B);
  double t = 0.0;
  CK(to_host(&t, Tsb + q, 1, c.st));
  CK(cudaStreamSynchronize(c.st));
  return bad_sampling_time(q, t);
}

// Where the arrays of an entry live.  HOST: host memory, staged through the device's staging buffer.  DEV: device memory, read on the
// library's stream without waiting for any other (obca_parking_solve_batch_dev).  STREAM: device memory, read after the work the caller
// enqueued on its stream (the *_dev entries with a stream argument).
enum class Arrays { HOST, DEV, STREAM };

// The start of a host-pointer entry: its layout placed in the device's staging buffer, which only grows (the whole call runs under the
// device lock), and its inputs copied in.
static int stage_in(DevCtx& c, DevLayout& lay) {
  const int rc = ensure((void**)&c.stage, &c.stage_bytes, lay.bytes);
  if (rc) return rc;
  lay.place(c.stage);
  CK(lay.copy_in(c.st));
  return 0;
}

// The start of a device-pointer entry, before any output is written.  STREAM: the library's stream waits for what the caller enqueued on
// `stream` (a cudaStream_t of the context's device; null: its default stream), so that nothing the library enqueues after this reads an
// input before the caller's producers have finished.  Then a mixed batch's device-resident horizons Nb and (not null) sampling times Tsb
// are checked.
static int dev_start(DevCtx& c, Arrays at, void* stream, int B, const int* Nb, int Nmax, const double* Tsb) {
  if (at == Arrays::STREAM) {
    CK(cudaEventRecord(c.evs, (cudaStream_t)stream));
    CK(cudaStreamWaitEvent(c.st, c.evs, 0));
  }
  return Nb ? check_batch_args_dev(c, B, Nb, Nmax, Tsb) : 0;
}

// ---- the solve and check families: one argument struct, one device core and one entry function each ------------------------------------
// Each struct holds its entries' arguments by name, in their order.  A device core takes the struct with every per-problem array in
// device memory (the scene is in the problem it is given), checks nothing and takes no lock.  An entry function runs a whole call, with
// the arrays where `at` says: the refusals in the entries' order (the values of host-resident Nb / Tsb directly after their presence),
// get_ctx and the device lock, stage_in or dev_start, the core, and for host arrays the copy back.

// obca_parking_solve_batch[_dev] and obca_parking_solve_mixed[_dev].  Every per-problem array is laid out for the horizon N; Nb:
// per-problem horizons <= N (mixed entries; problem b uses the first Nb[b] + 1 stages of its arrays), else null.
struct ParkSolve {
  int B, N;
  const int* Nb;
  int nOb;
  const int* vOb;
  const double *A, *b, *x0, *xF;
  double Ts, L;
  const double *ego, *XYbounds, *rx, *ry, *ryaw, *xWS, *uWS, *lWS, *nWS;
  int fixTime, signed_dist;
  const obca_opts* opts;
  double *xp, *up, *ts, *lp, *np, *sl;
  int *exitflag, *iters;
  double *kkt_err, *solve_seconds;
};

// The parking solve of P: DualMultWS into the library's scratch when lWS / nWS are null, then the solve.  Returns once the device's
// stream is synchronised.
static int parking_solve_dev(DevCtx& c, const ParkProblem& P, const ParkSolve& a) {
  const obca_opts* opts = a.opts;
  BatchPtrs bp;
  bp.x0 = a.x0; bp.xF = a.xF; bp.rx = a.rx; bp.ry = a.ry; bp.ryaw = a.ryaw; bp.xWS = a.xWS; bp.uWS = a.uWS; bp.Nb = a.Nb;
  bp.xp = a.xp; bp.up = a.up; bp.ts = a.ts; bp.lp = a.lp; bp.np = a.np; bp.sl = a.sl; bp.duals = nullptr;
  bp.exitflag = a.exitflag; bp.iters = a.iters; bp.kkt_err = a.kkt_err; bp.B = a.B; bp.retry = opts ? opts->retry : 1;
  bp.q4 = opts ? opts->q4 : 0;
  CK(cudaEventRecord(c.ev0, c.st));
  if (a.lWS && a.nWS) { bp.lWS = a.lWS; bp.nWS = a.nWS; }
  else {
    // the reference runs DualMultWS inside the NLP driver (ParkingSignedDist.jl:219); its result goes to a scratch of
    // the library (never to the caller's output arrays, which stay untouched until a problem has finished)
    const ParkSizes z = park_sizes(P.N, P.V, P.nOb);
    const size_t nl = z.l * a.B, nn = z.n * a.B;
    int rc = ensure((void**)&c.wsd, &c.wsd_bytes, (nl + nn) * sizeof(double));
    if (rc) return rc;
    rc = run_dualws(c, P, a.B, a.Nb, a.rx, a.ry, a.ryaw, c.wsd, c.wsd + nl, nullptr);
    if (rc) return rc;
    bp.lWS = c.wsd; bp.nWS = c.wsd + nl;
  }
  CK(cudaEventRecord(c.evm, c.st));      // `time` = the solve alone, as in the reference (:239-241); see obca_last_times
  return solve_dev_impl(c, P, to_ipm(opts), bp, a.solve_seconds);
}

// mixed: Nb holds per-problem horizons in [2, N].
static int parking_solve(const ParkSolve& a, Arrays at, bool mixed, void* stream) {
  const bool host = at == Arrays::HOST;
  if (a.B <= 0 || !a.vOb || !a.A || !a.b || !a.ego || !a.XYbounds || !a.x0 || !a.xF || !a.rx || !a.ry || !a.ryaw || !a.xWS || !a.uWS ||
      !a.xp || !a.up || !a.ts || !a.lp || !a.np || !a.exitflag || !a.iters || !a.kkt_err) { set_err("null argument"); return OBCA_ERR_ARG; }
  int rc = mixed ? check_horizons(a.B, a.Nb, a.N, host) : 0;
  if (rc) return rc;
  // the shape decides the staging sizes below: checked before anything is sized, copied or written
  ParkProblem P;
  if (const int e_ = fill_problem(P, a.N, a.nOb, a.vOb, a.A, a.b, a.Ts, a.L, a.ego, a.XYbounds, a.fixTime, a.signed_dist)) {
    set_err(shape_error(e_)); return OBCA_ERR_ARG;
  }
  rc = check_park_horizon(a.N);
  if (rc) return rc;
  DevCtx* c;
  rc = get_ctx(a.opts ? a.opts->device : 0, &c);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  const size_t Bs = a.B;
  const ParkSizes z = park_sizes(a.N, P.V, a.nOb);
  ParkSolve d = a;      // the call on the staged arrays (host arrays)
  char* dout = nullptr;
  DevLayout outs;       // host arrays: the per-problem outputs, copied back in one piece when the horizons differ
  DevLayout lay;        // host arrays: all of their staging
  if (host) {
    const bool have_ws = a.lWS && a.nWS;
    outs.out(d.xp, a.xp, z.x * Bs);
    outs.out(d.up, a.up, z.u * Bs);
    outs.out(d.ts, a.ts, z.ns * Bs);
    outs.out(d.lp, a.lp, z.l * Bs);
    outs.out(d.np, a.np, z.n * Bs);
    outs.out(d.sl, a.sl, z.sl * Bs);
    outs.out(d.kkt_err, a.kkt_err, Bs);
    lay.in(d.x0, a.x0, 4 * Bs);
    lay.in(d.xF, a.xF, 4 * Bs);
    lay.in(d.rx, a.rx, z.ns * Bs);
    lay.in(d.ry, a.ry, z.ns * Bs);
    lay.in(d.ryaw, a.ryaw, z.ns * Bs);
    lay.in(d.xWS, a.xWS, z.x * Bs);
    lay.in(d.uWS, a.uWS, z.u * Bs);
    lay.in(d.lWS, have_ws ? a.lWS : nullptr, z.l * Bs);
    lay.in(d.nWS, have_ws ? a.nWS : nullptr, z.n * Bs);
    lay.in(d.Nb, a.Nb, Bs);
    lay.add(dout, outs.bytes);
    lay.out(d.exitflag, a.exitflag, Bs);
    lay.out(d.iters, a.iters, Bs);
    rc = stage_in(*c, lay);
    outs.place(dout);
    if (!have_ws) d.lWS = d.nWS = nullptr;
    if (!a.Nb) d.Nb = nullptr;
  } else {
    rc = dev_start(*c, at, stream, a.B, a.Nb, a.N, nullptr);
  }
  if (!rc) rc = parking_solve_dev(*c, P, d);
  // device arrays: the kernels write each problem's outputs over its own horizon only, so the caller's arrays need no scatter
  if (rc || !host) return rc;
  cudaStream_t st = c->st;
  CK(lay.copy_out(st));
  if (!mixed) {
    CK(outs.copy_out(st));
    CK(cudaStreamSynchronize(st));
    return 0;
  }
  // per-problem horizons: the outputs come back through a host scratch, and only the entries of each problem's own
  // horizon are copied into the caller's arrays (the padding past it is never written)
  std::vector<double> h(outs.bytes / sizeof(double));
  CK(to_host((char*)h.data(), dout, outs.bytes, st));
  CK(cudaStreamSynchronize(st));
  scatter_horizons(a.xp, outs.in_copy(d.xp, h.data()), a.B, a.Nb, z.x, 4, 1);
  scatter_horizons(a.up, outs.in_copy(d.up, h.data()), a.B, a.Nb, z.u, 2, 0);
  scatter_horizons(a.ts, outs.in_copy(d.ts, h.data()), a.B, a.Nb, z.ns, 1, 1);
  scatter_horizons(a.lp, outs.in_copy(d.lp, h.data()), a.B, a.Nb, z.l, P.V, 1);
  scatter_horizons(a.np, outs.in_copy(d.np, h.data()), a.B, a.Nb, z.n, 4 * (size_t)a.nOb, 1);
  scatter_horizons(a.sl, outs.in_copy(d.sl, h.data()), a.B, a.Nb, z.sl, a.nOb, 1);
  memcpy(a.kkt_err, outs.in_copy(d.kkt_err, h.data()), Bs * sizeof(double));
  return 0;
}

// obca_dualmultws_batch[_dev]: laid out for the horizon N.
struct DualWs {
  int B, N, nOb;
  const int* vOb;
  const double *A, *b, *ego, *rx, *ry, *ryaw;
  const obca_opts* opts;
  double *lp, *np, *dd;
};

static int dualmultws(const DualWs& a, Arrays at, void* stream) {
  if (a.B <= 0 || !a.vOb || !a.A || !a.b || !a.ego || !a.rx || !a.ry || !a.ryaw || !a.lp || !a.np) {
    set_err("null argument"); return OBCA_ERR_ARG;
  }
  ParkProblem P;
  const double xy[4] = {0, 1, 0, 1};
  if (const int e_ = fill_problem(P, a.N, a.nOb, a.vOb, a.A, a.b, 1.0, 1.0, a.ego, xy, 0, 1)) { set_err(shape_error(e_)); return OBCA_ERR_ARG; }
  DevCtx* c;
  int rc = get_ctx(a.opts ? a.opts->device : 0, &c);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  DualWs d = a;      // the call on the staged arrays (host arrays)
  DevLayout lay;     // host arrays: their staging
  if (at == Arrays::HOST) {
    const size_t Bs = a.B;
    const ParkSizes z = park_sizes(a.N, P.V, a.nOb);
    lay.in(d.rx, a.rx, z.ns * Bs);
    lay.in(d.ry, a.ry, z.ns * Bs);
    lay.in(d.ryaw, a.ryaw, z.ns * Bs);
    lay.out(d.lp, a.lp, z.l * Bs);
    lay.out(d.np, a.np, z.n * Bs);
    lay.out(d.dd, a.dd, z.sl * Bs);
    rc = stage_in(*c, lay);
  } else {
    rc = dev_start(*c, at, stream, a.B, nullptr, a.N, nullptr);
  }
  if (!rc) rc = run_dualws(*c, P, a.B, nullptr, d.rx, d.ry, d.ryaw, d.lp, d.np, d.dd);
  if (rc) return rc;
  CK(lay.copy_out(c->st));
  CK(cudaStreamSynchronize(c->st));
  return 0;
}

// obca_check_parking[_dev] and obca_check_parking_mixed[_dev].  Every per-problem array is laid out for the horizon N; Nb: per-problem
// horizons <= N (mixed entries), else null.
struct ParkCheck {
  int B, N;
  const int* Nb;
  int nOb;
  const int* vOb;
  const double *A, *b, *x0, *xF;
  double Ts, L;
  const double *ego, *XYbounds, *x, *u, *l, *n, *timeScale, *sl;
  int fixTime, sd;
  const obca_opts* opts;
  int *feasible, *e, *strict;
};

// ParkingConstraints over the batch on the device's stream (Nb, sl, e, strict may be null).
static int check_parking_dev(DevCtx& c, const ParkProblem& P, const ParkCheck& a) {
  const int grid = a.B < 4 * c.sms ? a.B : 4 * c.sms;
  k_check<<<grid, 128, 0, c.st>>>(P, a.B, a.Nb, a.x0, a.xF, a.x, a.u, a.l, a.n, a.timeScale, a.sl, a.sd, a.feasible, a.e, a.strict);
  CK(cudaGetLastError());
  return 0;
}

static int check_parking(const ParkCheck& a, Arrays at, bool mixed, void* stream) {
  const bool host = at == Arrays::HOST;
  int rc = mixed ? check_horizons(a.B, a.Nb, a.N, host) : 0;
  if (rc) return rc;
  if (a.B <= 0 || !a.vOb || !a.A || !a.b || !a.x0 || !a.xF || !a.ego || !a.XYbounds || !a.x || !a.u || !a.l || !a.n || !a.timeScale ||
      !a.feasible) { set_err("null argument"); return OBCA_ERR_ARG; }
  ParkProblem P;
  if (const int e_ = fill_problem(P, a.N, a.nOb, a.vOb, a.A, a.b, a.Ts, a.L, a.ego, a.XYbounds, a.fixTime, a.sd)) {
    set_err(shape_error(e_)); return OBCA_ERR_ARG;
  }
  DevCtx* c;
  rc = get_ctx(a.opts ? a.opts->device : 0, &c);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  ParkCheck d = a;      // the call on the staged arrays (host arrays)
  DevLayout lay;        // host arrays: their staging
  if (host) {
    const size_t Bs = a.B;
    const ParkSizes z = park_sizes(a.N, P.V, a.nOb);
    lay.in(d.x0, a.x0, 4 * Bs);
    lay.in(d.xF, a.xF, 4 * Bs);
    lay.in(d.x, a.x, z.x * Bs);
    lay.in(d.u, a.u, z.u * Bs);
    lay.in(d.l, a.l, z.l * Bs);
    lay.in(d.n, a.n, z.n * Bs);
    lay.in(d.timeScale, a.timeScale, z.ns * Bs);
    lay.in(d.sl, a.sl, z.sl * Bs);
    lay.in(d.Nb, a.Nb, Bs);
    lay.out(d.feasible, a.feasible, Bs);
    lay.out(d.e, a.e, 7 * Bs);
    lay.out(d.strict, a.strict, Bs);
    rc = stage_in(*c, lay);
    if (!a.sl) d.sl = nullptr;
    if (!a.Nb) d.Nb = nullptr;
  } else {
    rc = dev_start(*c, at, stream, a.B, a.Nb, a.N, nullptr);
  }
  if (!rc) rc = check_parking_dev(*c, P, d);
  if (rc) return rc;
  CK(lay.copy_out(c->st));
  CK(cudaStreamSynchronize(c->st));
  return 0;
}

// obca_quadcopter_solve_batch[_dev] and obca_quadcopter_solve_mixed[_dev].  Every per-problem array is laid out for the horizon N; Nb, Tsb
// (mixed entries): per-problem horizons <= N and sampling times, problem b uses the first Nb[b] + 1 stages of its arrays and nothing past
// them is written; otherwise both null.
struct QuadSolve {
  int B, N;
  const int* Nb;
  const double *Tsb, *x0, *xF;
  double Ts, R;
  const double *ob, *xWS;
  double timeWS;
  int signed_dist;
  const obca_opts* opts;
  double *xp, *up, *ts, *lp, *slack;
  int *exitflag, *iters;
  double *kkt_err, *solve_seconds;
};

// The quadcopter solve of P on the device's stream between the context's events ev0 and ev1, then the phase counters back to prof_host
// (obca_last_profile).  quad_solve_seconds reads its time once the stream is synchronised.
static int quad_solve_dev(DevCtx& c, const QuadProblem& P, const QuadSolve& a) {
  IpmOpts O = to_ipm(a.opts);
  if (!a.opts) O.max_iter = 3000;                        // the reference sets no max_iter here (Ipopt default)
  QBatchPtrs bp;
  bp.x0 = a.x0; bp.xF = a.xF; bp.xWS = a.xWS; bp.Nb = a.Nb; bp.Tsb = a.Tsb;
  bp.timeWS = a.timeWS; bp.xp = a.xp; bp.up = a.up; bp.ts = a.ts; bp.lp = a.lp;
  bp.slack = P.signed_dist ? a.slack : nullptr;          // the Dist formulation has no slacks
  bp.exitflag = a.exitflag; bp.iters = a.iters; bp.kkt_err = a.kkt_err; bp.B = a.B;
  bp.prof = c.prof;
  CK(cudaMemsetAsync(c.prof, 0, 8 * sizeof(unsigned long long), c.st));
  CK(cudaEventRecord(c.ev0, c.st));
  const int rc = P.signed_dist ? launch_quad<true>(c, P, O, bp) : launch_quad<false>(c, P, O, bp);
  if (rc) return rc;
  CK(cudaEventRecord(c.ev1, c.st));
  CK(to_host(c.prof_host, c.prof, 8, c.st));
  return 0;
}
static int quad_solve_seconds(DevCtx& c, double* seconds) {
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, c.ev0, c.ev1));
  if (seconds) *seconds = ms * 1e-3;
  return 0;
}

// mixed: Nb, Tsb hold per-problem horizons in [2, N] and sampling times.
static int quad_solve(const QuadSolve& a, Arrays at, bool mixed, void* stream) {
  const bool host = at == Arrays::HOST;
  if (a.B <= 0 || !a.x0 || !a.xF || !a.ob || !a.xWS || !a.xp || !a.up || !a.ts || !a.lp || !a.exitflag || !a.iters || !a.kkt_err) {
    set_err("null argument"); return OBCA_ERR_ARG;
  }
  int rc = mixed ? check_horizons(a.B, a.Nb, a.N, host) : 0;
  if (!rc && mixed) rc = check_sampling_times(a.B, a.Tsb, host);
  if (rc) return rc;
  QuadProblem P;
  if (fill_quad_problem(P, a.N, a.Ts, a.R, a.ob, a.signed_dist)) { set_err("unsupported problem shape"); return OBCA_ERR_ARG; }
  rc = check_quad_horizon(a.N);
  if (rc) return rc;
  DevCtx* c;
  rc = get_ctx(a.opts ? a.opts->device : 0, &c);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  const size_t Bs = a.B;
  const QuadSizes z = quad_sizes(a.N);
  const bool scatter = host && mixed;      // host arrays of a mixed batch come back through a host scratch, each problem's horizon only
  QuadSolve d = a;      // the call on the staged arrays (host arrays)
  char* dout = nullptr;
  DevLayout outs;       // host arrays: the per-problem outputs, copied back in one piece when the horizons differ
  DevLayout lay;        // host arrays: all of their staging
  if (host) {
    outs.out(d.xp, a.xp, z.x * Bs);
    outs.out(d.up, a.up, z.u * Bs);
    outs.out(d.ts, a.ts, z.ns * Bs);
    outs.out(d.lp, a.lp, z.l * Bs);
    outs.out(d.slack, a.signed_dist ? a.slack : nullptr, z.s * Bs);
    outs.out(d.kkt_err, a.kkt_err, Bs);
    lay.in(d.x0, a.x0, 12 * Bs);
    lay.in(d.xF, a.xF, 12 * Bs);
    lay.in(d.xWS, a.xWS, z.x * Bs);
    lay.in(d.Nb, a.Nb, Bs);
    lay.in(d.Tsb, a.Tsb, Bs);
    lay.add(dout, outs.bytes);
    lay.out(d.exitflag, a.exitflag, Bs);
    lay.out(d.iters, a.iters, Bs);
    rc = stage_in(*c, lay);
    outs.place(dout);
    if (!mixed) { d.Nb = nullptr; d.Tsb = nullptr; }
  } else {
    rc = dev_start(*c, at, stream, a.B, a.Nb, a.N, a.Tsb);
  }
  if (!rc) rc = quad_solve_dev(*c, P, d);
  if (rc) return rc;
  cudaStream_t st = c->st;
  if (!scatter) CK(outs.copy_out(st));
  CK(lay.copy_out(st));
  std::vector<double> h;
  if (scatter) {
    h.resize(outs.bytes / sizeof(double));
    CK(to_host((char*)h.data(), dout, outs.bytes, st));
  }
  CK(cudaStreamSynchronize(st));
  rc = quad_solve_seconds(*c, a.solve_seconds);
  if (rc || !scatter) return rc;
  scatter_horizons(a.xp, outs.in_copy(d.xp, h.data()), a.B, a.Nb, z.x, 12, 1);
  scatter_horizons(a.up, outs.in_copy(d.up, h.data()), a.B, a.Nb, z.u, 4, 0);
  scatter_horizons(a.ts, outs.in_copy(d.ts, h.data()), a.B, a.Nb, z.ns, 1, 1);
  scatter_horizons(a.lp, outs.in_copy(d.lp, h.data()), a.B, a.Nb, z.l, 30, 1);
  scatter_horizons(a.signed_dist ? a.slack : nullptr, outs.in_copy(d.slack, h.data()), a.B, a.Nb, z.s, 5, 1);
  memcpy(a.kkt_err, outs.in_copy(d.kkt_err, h.data()), Bs * sizeof(double));
  return 0;
}

// obca_check_quadcopter[_dev] and obca_check_quadcopter_mixed[_dev].  Every per-problem array is laid out for the horizon N; Nb, Tsb
// (mixed entries): per-problem horizons <= N and sampling times, otherwise both null.
struct QuadCheck {
  int B, N;
  const int* Nb;
  const double *Tsb, *x, *u, *timeScale, *x0, *xF;
  double Ts;
  const double *lambda, *ob;
  double R;
  const obca_opts* opts;
  int* feasible;
  double* worst;
};

// constrSatisfaction over the batch on the device's stream (Nb and Tsb together, and worst, may be null).
static int quad_check_dev(DevCtx& c, const QuadProblem& P, const QuadCheck& a) {
  const int grid = a.B < 4 * c.sms ? a.B : 4 * c.sms;
  k_quad_check<<<grid, 128, 0, c.st>>>(P, a.B, a.Nb, a.Tsb, a.x0, a.xF, a.x, a.u, a.timeScale, a.lambda, a.feasible, a.worst);
  CK(cudaGetLastError());
  return 0;
}

static int quad_check(const QuadCheck& a, Arrays at, bool mixed, void* stream) {
  const bool host = at == Arrays::HOST;
  int rc = mixed ? check_horizons(a.B, a.Nb, a.N, host) : 0;
  if (!rc && mixed) rc = check_sampling_times(a.B, a.Tsb, host);
  if (rc) return rc;
  if (a.B <= 0 || !a.x || !a.u || !a.timeScale || !a.x0 || !a.xF || !a.lambda || !a.ob || !a.feasible) {
    set_err("null argument"); return OBCA_ERR_ARG;
  }
  QuadProblem P;
  if (fill_quad_problem(P, a.N, a.Ts, a.R, a.ob, 0)) { set_err("unsupported problem shape"); return OBCA_ERR_ARG; }
  DevCtx* c;
  rc = get_ctx(a.opts ? a.opts->device : 0, &c);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  QuadCheck d = a;      // the call on the staged arrays (host arrays)
  DevLayout lay;        // host arrays: their staging
  if (host) {
    const size_t Bs = a.B;
    const QuadSizes z = quad_sizes(a.N);
    lay.in(d.x0, a.x0, 12 * Bs);
    lay.in(d.xF, a.xF, 12 * Bs);
    lay.in(d.x, a.x, z.x * Bs);
    lay.in(d.u, a.u, z.u * Bs);
    lay.in(d.timeScale, a.timeScale, z.ns * Bs);
    lay.in(d.lambda, a.lambda, z.l * Bs);
    lay.in(d.Nb, a.Nb, Bs);
    lay.in(d.Tsb, a.Tsb, Bs);
    lay.out(d.feasible, a.feasible, Bs);
    lay.out(d.worst, a.worst, Bs);
    rc = stage_in(*c, lay);
    if (!mixed) { d.Nb = nullptr; d.Tsb = nullptr; }
  } else {
    rc = dev_start(*c, at, stream, a.B, a.Nb, a.N, a.Tsb);
  }
  if (!rc) rc = quad_check_dev(*c, P, d);
  if (rc) return rc;
  CK(lay.copy_out(c->st));
  CK(cudaStreamSynchronize(c->st));
  return 0;
}

// ---- plan -> solve -> check without leaving the device, for one formulation or for both on one plan ------------------------------------

// The first null required field of a flow output set (its name), or null when every required field is there.
static const char* missing_field(const obca_parking_flow_out& o) {
  return !o.xp ? "xp" : !o.up ? "up" : !o.ts ? "ts" : !o.lp ? "lp" : !o.np ? "np" : !o.exitflag ? "exitflag" : !o.iters ? "iters"
       : !o.kkt_err ? "kkt_err" : !o.feasible ? "feasible" : nullptr;
}
static const char* missing_field(const obca_quadcopter_flow_out& o) {
  return !o.xp ? "xp" : !o.up ? "up" : !o.ts ? "ts" : !o.lp ? "lp" : !o.exitflag ? "exitflag" : !o.iters ? "iters"
       : !o.kkt_err ? "kkt_err" : !o.feasible ? "feasible" : nullptr;
}

// The null checks of the *_both entries on their two output sets, with the set and the field named in the message.
template <class Out>
static int check_both_sets(const Out* dist, const Out* sd) {
  const Out* sets[2] = {dist, sd};
  const char* names[2] = {"dist", "sd"};
  for (int f = 0; f < 2; ++f) {
    if (!sets[f]) { set_err(std::string("null argument: ") + names[f]); return OBCA_ERR_ARG; }
    if (const char* m = missing_field(*sets[f])) { set_err(std::string("null argument: ") + names[f] + "." + m); return OBCA_ERR_ARG; }
  }
  return 0;
}

// One formulation of a flow call: its signed_dist and the caller's arrays it writes.
template <class Out>
struct FlowSet {
  int signed_dist;
  const Out* out;
};

template <class Out>
static bool sets_complete(int nf, const FlowSet<Out>* sets) {
  for (int f = 0; f < nf; ++f)
    if (missing_field(*sets[f].out)) return false;
  return true;
}

// obca_parking_plan_solve_goals (nf = 1) and obca_parking_plan_solve_both (nf = 2, Dist then SD): the stages the formulations share
// (checks, plan, list, gather) run once, then each formulation is solved, checked and scattered into its own set in turn.
static int parking_plan_solve(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                              int sampleN, int max_expansions, int max_nodes, int nOb, const int* vOb, const double* A, const double* b,
                              const double* ego, const double* XYbounds, int fixTime, const obca_opts* opts, int Ncap, int* N, int* status,
                              int* expansions, double* plan_seconds, int nf, const FlowSet<obca_parking_flow_out>* sets) {
  // the planner's checks, then the solver's, with the messages of the entries this one composes; nothing is written before they pass
  int rc = plan_check_args(B, x0 && xF && ox && oy && vOb && A && b && ego && XYbounds && N && status && sets_complete(nf, sets), n_ob, Ts,
                           sampleN);
  if (rc) return rc;
  if (Ncap < 2) { set_err("Ncap < 2"); return OBCA_ERR_ARG; }
  ParkProblem P;
  for (int f = 0; f < nf; ++f)
    if (const int e_ = fill_problem(P, Ncap, nOb, vOb, A, b, Ts, L, ego, XYbounds, fixTime, sets[f].signed_dist)) {
      set_err(shape_error(e_)); return OBCA_ERR_ARG;
    }
  rc = check_park_horizon(Ncap);
  if (rc) return rc;
  DevCtx* c;
  const int dev = opts ? opts->device : 0;
  rc = get_ctx(dev, &c);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = 0.0;
  for (int f = 0; f < nf; ++f)
    if (sets[f].out->solve_seconds) *sets[f].out->solve_seconds = 0.0;
  if (B == 0) return 0;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  cudaStream_t st = c->st;
  const int V = P.V, cap = Ncap + 1;      // the planner's stride: stages 0..Ncap, so a longer plan comes back as OBCA_PLAN_CAPACITY
  const size_t Bs = B;
  // stage 1: plan into device buffers (N is copied in first: the planner leaves it alone where it finds no path)
  std::vector<double> x03(3 * Bs), xF3(3 * Bs);
  for (size_t p = 0; p < Bs; ++p)
    for (int r = 0; r < 3; ++r) { x03[3 * p + r] = x0[4 * p + r]; xF3[3 * p + r] = xF[4 * p + r]; }
  PlanDevOut po;
  double *d0, *dF;
  int *dlist, *dNb, *dcnt;
  DevLayout pl;
  pl.add(po.rx, cap * Bs);
  pl.add(po.ry, cap * Bs);
  pl.add(po.ryaw, cap * Bs);
  pl.add(po.xWS, 4 * cap * Bs);
  pl.add(po.uWS, 2 * cap * Bs);
  pl.inout(po.N, N, Bs);
  pl.out(po.status, status, Bs);
  pl.out(po.expansions, expansions, Bs);
  pl.in(d0, x0, 4 * Bs);
  pl.in(dF, xF, 4 * Bs);
  pl.add(dlist, Bs);
  pl.add(dNb, Bs);
  pl.add(dcnt, 2);
  DevBuf dplan;
  CK(alloc_layout(dplan, pl));
  CK(pl.copy_in(st));
  float plan_ms = 0.f;
  rc = plan_warmstart_dev(B, x03.data(), xF3.data(), ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap, dev, st, po, &plan_ms);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = plan_ms * 1e-3;
  // stage 2: list the poses to solve; their count and longest horizon size the solve (its occupancy follows the layout's horizon)
  k_flow_list<<<1, FLOW_LIST_THREADS, 0, st>>>(B, Ncap, po.status, po.N, dlist, dNb, dcnt);
  CK(cudaGetLastError());
  int cnt[2] = {0, 0};
  CK(to_host(cnt, dcnt, 2, st));
  CK(cudaStreamSynchronize(st));
  const int Bq = cnt[0], M = cnt[1];
  if (Bq == 0) {
    CK(pl.copy_out(st));
    CK(cudaStreamSynchronize(st));
    return 0;
  }
  // stage 3: gather the listed poses into the inputs of the mixed solve at the horizon M, once for every formulation
  const size_t Qs = Bq;
  const ParkSizes zm = park_sizes(M, V, nOb), zc = park_sizes(Ncap, V, nOb);      // the solve's layout, the caller's
  obca_flow::Gather g;
  g.rx = po.rx; g.ry = po.ry; g.ryaw = po.ryaw; g.xWS = po.xWS; g.uWS = po.uWS; g.x0 = d0; g.xF = dF;
  obca_flow::Outs so;
  char* dout;
  DevLayout outs;
  outs.add(so.xp, zm.x * Qs);
  outs.add(so.up, zm.u * Qs);
  outs.add(so.ts, zm.ns * Qs);
  outs.add(so.lp, zm.l * Qs);
  outs.add(so.np, zm.n * Qs);
  outs.add(so.sl, zm.sl * Qs);
  outs.add(so.kkt_err, Qs);
  outs.add(so.exitflag, Qs);
  outs.add(so.iters, Qs);
  outs.add(so.feasible, Qs);
  outs.add(so.strict, Qs);
  DevLayout sl_;
  sl_.add(g.mrx, zm.ns * Qs);
  sl_.add(g.mry, zm.ns * Qs);
  sl_.add(g.mryaw, zm.ns * Qs);
  sl_.add(g.mxWS, zm.x * Qs);
  sl_.add(g.muWS, zm.u * Qs);
  sl_.add(g.mx0, 4 * Qs);
  sl_.add(g.mxF, 4 * Qs);
  sl_.add(dout, outs.bytes);
  DevBuf dsolve;
  CK(alloc_layout(dsolve, sl_));
  outs.place(dout);
  const size_t items = Qs * zm.ns;
  const int threads = 256, blocks = (int)((items + threads - 1) / threads);
  k_flow_gather<<<blocks, threads, 0, st>>>(Bq, M, cap, dlist, dNb, g);
  CK(cudaGetLastError());
  for (int f = 0; f < nf; ++f) {
    const int sd = sets[f].signed_dist;
    const obca_parking_flow_out& u = *sets[f].out;
    ParkProblem PM;
    fill_problem(PM, M, nOb, vOb, A, b, Ts, L, ego, XYbounds, fixTime, sd);      // the shape passed above, with 2 <= M <= Ncap
    // stage 4: the mixed solve (DualMultWS inside) into outputs that start as zeros; stage 5: ParkingConstraints on its outputs
    CK(cudaMemsetAsync(dout, 0, outs.bytes, st));
    rc = parking_solve_dev(*c, PM, {Bq, M, dNb, nOb, vOb, A, b, g.mx0, g.mxF, Ts, L, ego, XYbounds, g.mrx, g.mry, g.mryaw, g.mxWS, g.muWS,
                                    nullptr, nullptr, fixTime, sd, opts, so.xp, so.up, so.ts, so.lp, so.np, so.sl, so.exitflag, so.iters,
                                    so.kkt_err, u.solve_seconds});
    if (rc) return rc;
    rc = check_parking_dev(*c, PM, {Bq, M, dNb, nOb, vOb, A, b, g.mx0, g.mxF, Ts, L, ego, XYbounds, so.xp, so.up, so.lp, so.np, so.ts,
                                    so.sl, fixTime, sd, opts, so.feasible, nullptr, so.strict});
    if (rc) return rc;
    // stage 6: the solved poses' outputs into the caller's arrays (copied to the device first, so that every entry the call does not
    // write keeps the caller's value), then back in one pass; this staging is freed before the next formulation runs
    obca_flow::Outs d;
    DevLayout ol;
    ol.inout(d.xp, u.xp, zc.x * Bs);
    ol.inout(d.up, u.up, zc.u * Bs);
    ol.inout(d.ts, u.ts, zc.ns * Bs);
    ol.inout(d.lp, u.lp, zc.l * Bs);
    ol.inout(d.np, u.np, zc.n * Bs);
    ol.inout(d.sl, u.sl, zc.sl * Bs);
    ol.inout(d.kkt_err, u.kkt_err, Bs);
    ol.inout(d.exitflag, u.exitflag, Bs);
    ol.inout(d.iters, u.iters, Bs);
    ol.inout(d.feasible, u.feasible, Bs);
    ol.inout(d.strict, u.strict, Bs);
    DevBuf dcaller;
    CK(alloc_layout(dcaller, ol));
    if (!u.sl) d.sl = nullptr;
    if (!u.strict) d.strict = nullptr;
    CK(ol.copy_in(st));
    k_flow_scatter<<<blocks, threads, 0, st>>>(Bq, M, Ncap, V, nOb, dlist, dNb, so, d);
    CK(cudaGetLastError());
    CK(ol.copy_out(st));
    CK(cudaStreamSynchronize(st));
  }
  CK(pl.copy_out(st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

// obca_quadcopter_plan_solve (nf = 1) and obca_quadcopter_plan_solve_both (nf = 2, Dist then SD): the stages the formulations share
// (checks, plan, list, warm starts) run once, then each formulation is solved, checked and scattered into its own set in turn.
static int quad_plan_solve(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz, int n_ob,
                           const double* lo, const double* hi, double reso, int max_nodes, double Ts, double R, const double* ob,
                           double timeWS, const obca_opts* opts, int Ncap, int* N, double* Tsb, int* status, int* expansions,
                           double* plan_seconds, int nf, const FlowSet<obca_quadcopter_flow_out>* sets) {
  // the planner's checks and set-up (start and goal on its grid, scaled here as mainQuadcopter.jl:114-119 does), then the solve's;
  // nothing is written before they pass
  // the planner's stride: stages 0..Ncap, so a longer path comes back as OBCA_PLAN_CAPACITY (an Ncap out of range is refused below)
  const int cap = Ncap >= 2 && Ncap <= QUAD_NMAX ? Ncap + 1 : 3;
  std::vector<double> s3(3 * (size_t)(B > 0 ? B : 1)), g3(s3.size());
  if (x0 && xF)
    for (int p = 0; p < B; ++p)
      for (int r = 0; r < 3; ++r) {
        s3[3 * (size_t)p + r] = OBCA_QUAD_GRID_SCALE * x0[12 * (size_t)p + r];
        g3[3 * (size_t)p + r] = OBCA_QUAD_GRID_SCALE * xF[12 * (size_t)p + r];
      }
  Plan3dSetupPtr S;
  int rc = plan3d_prepare(S, B, x0 && xF && ob && N && Tsb && status && sets_complete(nf, sets), s3.data(), g3.data(), ox, oy, oz, n_ob,
                          lo, hi, reso, max_nodes, cap);
  if (rc) return rc;
  if (Ncap < 2) { set_err("Ncap < 2"); return OBCA_ERR_ARG; }
  rc = check_quad_horizon(Ncap);
  if (rc) return rc;
  if (!(std::isfinite(Ts) && Ts > 0)) { set_err("Ts must be a finite number > 0"); return OBCA_ERR_ARG; }
  if (obca_qflow::ts_hundredths(Ts, Ncap) < 1) {
    set_err("Ts = " + std::to_string(Ts) + " gives a pair planned to N = Ncap = " + std::to_string(Ncap) + " the sampling time 0");
    return OBCA_ERR_ARG;
  }
  QuadProblem P;
  for (int f = 0; f < nf; ++f)
    if (fill_quad_problem(P, Ncap, std::nan(""), R, ob, sets[f].signed_dist)) { set_err("unsupported problem shape"); return OBCA_ERR_ARG; }
  DevCtx* c;
  const int dev = opts ? opts->device : 0;
  rc = get_ctx(dev, &c);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = 0.0;
  for (int f = 0; f < nf; ++f)
    if (sets[f].out->solve_seconds) *sets[f].out->solve_seconds = 0.0;
  if (B == 0) return 0;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  cudaStream_t st = c->st;
  const size_t Bs = B;
  // stage 1: plan into device buffers (N and expansions are copied in first: the planner leaves them alone where it does not write them)
  Plan3dDevOut po;
  double *d0, *dF;
  int *dlist, *dNb, *dcnt;
  DevLayout pl;
  pl.add(po.rx, cap * Bs);
  pl.add(po.ry, cap * Bs);
  pl.add(po.rz, cap * Bs);
  pl.inout(po.N, N, Bs);
  pl.out(po.status, status, Bs);
  pl.inout(po.expansions, expansions, Bs);
  pl.in(d0, x0, 12 * Bs);
  pl.in(dF, xF, 12 * Bs);
  pl.add(dlist, Bs);
  pl.add(dNb, Bs);
  pl.add(dcnt, 2);
  DevBuf dplan;
  CK(alloc_layout(dplan, pl));
  CK(pl.copy_in(st));
  if (!expansions) po.expansions = nullptr;
  float plan_ms = 0.f;
  rc = plan3d_dev(*S, B, dev, st, po, &plan_ms);
  if (rc) return rc;
  if (plan_seconds) *plan_seconds = plan_ms * 1e-3;
  // stage 2: list the pairs to solve; their count and longest horizon size the solve (its occupancy follows the layout's horizon)
  k_flow_list<<<1, FLOW_LIST_THREADS, 0, st>>>(B, Ncap, po.status, po.N, dlist, dNb, dcnt);
  CK(cudaGetLastError());
  int cnt[2] = {0, 0};
  CK(to_host(cnt, dcnt, 2, st));
  CK(cudaStreamSynchronize(st));
  const int Bq = cnt[0], M = cnt[1];
  if (Bq == 0) {
    CK(pl.copy_out(st));
    CK(cudaStreamSynchronize(st));
    return 0;
  }
  // stage 3: the listed pairs' warm starts, x0, xF and sampling times as the inputs of the mixed solve at the horizon M, once for every
  // formulation.  The check takes the Dist bounds whatever the formulation, as obca_check_quadcopter_mixed does.
  QuadProblem PC;
  fill_quad_problem(PC, M, std::nan(""), R, ob, 0);      // the shape passed above, with 2 <= M <= Ncap
  const size_t Qs = Bq;
  const QuadSizes zm = quad_sizes(M), zc = quad_sizes(Ncap);      // the solve's layout, the caller's
  obca_qflow::Gather g;
  g.rx = po.rx; g.ry = po.ry; g.rz = po.rz; g.x0 = d0; g.xF = dF; g.Ts = Ts;
  obca_qflow::Outs so;
  char* dout;
  DevLayout outs;
  outs.add(so.xp, zm.x * Qs);
  outs.add(so.up, zm.u * Qs);
  outs.add(so.ts, zm.ns * Qs);
  outs.add(so.lp, zm.l * Qs);
  outs.add(so.slack, zm.s * Qs);
  outs.add(so.kkt_err, Qs);
  outs.add(so.worst, Qs);
  outs.add(so.exitflag, Qs);
  outs.add(so.iters, Qs);
  outs.add(so.feasible, Qs);
  DevLayout sl_;
  sl_.add(g.mxWS, zm.x * Qs);
  sl_.add(g.mx0, 12 * Qs);
  sl_.add(g.mxF, 12 * Qs);
  sl_.add(g.mTsb, Qs);
  sl_.add(dout, outs.bytes);
  DevBuf dsolve;
  CK(alloc_layout(dsolve, sl_));
  outs.place(dout);
  so.Tsb = g.mTsb;
  const size_t items = Qs * zm.ns;
  const int threads = 256, blocks = (int)((items + threads - 1) / threads);
  k_qflow_gather<<<blocks, threads, 0, st>>>(Bq, M, cap, dlist, dNb, g);
  CK(cudaGetLastError());
  for (int f = 0; f < nf; ++f) {
    const int sd = sets[f].signed_dist;
    const obca_quadcopter_flow_out& u = *sets[f].out;
    QuadProblem PM;
    fill_quad_problem(PM, M, std::nan(""), R, ob, sd);
    // stage 4: the mixed solve into outputs that start as zeros; stage 5: constrSatisfaction on its outputs
    CK(cudaMemsetAsync(dout, 0, outs.bytes, st));
    rc = quad_solve_dev(*c, PM, {Bq, M, dNb, g.mTsb, g.mx0, g.mxF, std::nan(""), R, ob, g.mxWS, timeWS, sd, opts, so.xp, so.up, so.ts,
                                 so.lp, so.slack, so.exitflag, so.iters, so.kkt_err, u.solve_seconds});
    if (rc) return rc;
    rc = quad_check_dev(*c, PC, {Bq, M, dNb, g.mTsb, so.xp, so.up, so.ts, g.mx0, g.mxF, std::nan(""), so.lp, ob, R, opts, so.feasible,
                                 so.worst});
    if (rc) return rc;
    // stage 6: the solved pairs' outputs into the caller's arrays (copied to the device first, so that every entry the call does not
    // write keeps the caller's value), then back in one pass; this staging is freed before the next formulation runs
    double* slack_out = sd ? u.slack : nullptr;      // the Dist formulation has no slacks
    obca_qflow::Outs d;
    DevLayout ol;
    ol.inout(d.xp, u.xp, zc.x * Bs);
    ol.inout(d.up, u.up, zc.u * Bs);
    ol.inout(d.ts, u.ts, zc.ns * Bs);
    ol.inout(d.lp, u.lp, zc.l * Bs);
    ol.inout(d.slack, slack_out, slack_out ? zc.s * Bs : 0);
    ol.inout(d.kkt_err, u.kkt_err, Bs);
    ol.inout(d.Tsb, Tsb, Bs);
    ol.inout(d.worst, u.worst, u.worst ? Bs : 0);
    ol.inout(d.exitflag, u.exitflag, Bs);
    ol.inout(d.iters, u.iters, Bs);
    ol.inout(d.feasible, u.feasible, Bs);
    DevBuf dcaller;
    CK(alloc_layout(dcaller, ol));
    if (!slack_out) d.slack = nullptr;
    if (!u.worst) d.worst = nullptr;
    CK(ol.copy_in(st));
    k_qflow_scatter<<<blocks, threads, 0, st>>>(Bq, M, Ncap, dlist, dNb, so, d);
    CK(cudaGetLastError());
    CK(ol.copy_out(st));
    CK(cudaStreamSynchronize(st));
    rc = quad_solve_seconds(*c, u.solve_seconds);
    if (rc) return rc;
  }
  CK(pl.copy_out(st));
  CK(cudaStreamSynchronize(st));
  return 0;
}

extern "C" {

#ifdef OBCA_QPROF   // development builds only: cycles of the quadcopter sweep's phases, summed over CTAs; resets the counters
int obca_debug_qprof(unsigned long long* out8) {
  unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (cudaMemcpyFromSymbol(out8, g_qprof, sizeof(z)) != cudaSuccess) return -1;
  return cudaMemcpyToSymbol(g_qprof, z, sizeof(z)) == cudaSuccess ? 0 : -1;
}
#endif

int obca_version(void) { return OBCA_VERSION; }
int obca_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
  return n;
}
const char* obca_last_error(void) { return g_err.c_str(); }
void obca_default_opts(obca_opts* o) {
  IpmOpts d = default_opts();
  o->tol = d.tol; o->max_iter = d.max_iter; o->mu_init = d.mu_init; o->mu_min = d.mu_min;
  o->kappa_eps = d.kappa_eps; o->kappa_mu = d.kappa_mu; o->theta_mu = d.theta_mu; o->tau_min = d.tau_min;
  o->kappa1 = d.kappa1; o->kappa2 = d.kappa2; o->kappa_sigma = d.kappa_sigma; o->s_max = d.s_max;
  o->dual_inf_tol = d.dual_inf_tol; o->constr_viol_tol = d.constr_viol_tol; o->compl_inf_tol = d.compl_inf_tol;
  o->dw_min = d.dw_min; o->dw_first = d.dw_first; o->dw_max = d.dw_max; o->kw_minus = d.kw_minus;
  o->kw_plus = d.kw_plus; o->kw_plus_first = d.kw_plus_first;
  o->gamma_theta = d.gamma_theta; o->gamma_phi = d.gamma_phi; o->delta = d.delta; o->s_theta = d.s_theta;
  o->s_phi = d.s_phi; o->eta_phi = d.eta_phi; o->gamma_alpha = d.gamma_alpha; o->max_backtrack = d.max_backtrack;
  o->dc = d.dc; o->max_kick = d.max_kick; o->quad_dual_ws = d.quad_dual_ws;
  o->device = 0; o->retry = 1; o->q4 = 0;
}

int obca_parking_solve_batch_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b,
                                 const double* x0, const double* xF, double Ts, double L, const double* ego,
                                 const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                                 const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                                 int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up,
                                 double* ts, double* lp, double* np, double* sl, int* exitflag, int* iters,
                                 double* kkt_err, double* solve_seconds) {
  return parking_solve({B, N, nullptr, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, rx, ry, ryaw, xWS, uWS, lWS, nWS, fixTime, signed_dist,
                        opts, xp, up, ts, lp, np, sl, exitflag, iters, kkt_err, solve_seconds}, Arrays::DEV, false, nullptr);
}

int obca_parking_solve_batch(int B, int N, int nOb, const int* vOb, const double* A, const double* b,
                             const double* x0, const double* xF, double Ts, double L, const double* ego,
                             const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                             const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                             int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up, double* ts,
                             double* lp, double* np, double* sl, int* exitflag, int* iters, double* kkt_err,
                             double* solve_seconds) {
  return parking_solve({B, N, nullptr, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, rx, ry, ryaw, xWS, uWS, lWS, nWS, fixTime, signed_dist,
                        opts, xp, up, ts, lp, np, sl, exitflag, iters, kkt_err, solve_seconds}, Arrays::HOST, false, nullptr);
}

int obca_parking_solve_mixed(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                             const double* x0, const double* xF, double Ts, double L, const double* ego,
                             const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                             const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                             int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up, double* ts,
                             double* lp, double* np, double* sl, int* exitflag, int* iters, double* kkt_err,
                             double* solve_seconds) {
  return parking_solve({B, Nmax, Nb, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, rx, ry, ryaw, xWS, uWS, lWS, nWS, fixTime, signed_dist,
                        opts, xp, up, ts, lp, np, sl, exitflag, iters, kkt_err, solve_seconds}, Arrays::HOST, true, nullptr);
}

int obca_dualmultws_batch(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* ego,
                          const double* rx, const double* ry, const double* ryaw, const obca_opts* opts, double* lp,
                          double* np, double* dd) {
  return dualmultws({B, N, nOb, vOb, A, b, ego, rx, ry, ryaw, opts, lp, np, dd}, Arrays::HOST, nullptr);
}

int obca_check_parking(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* x0,
                       const double* xF, double Ts, double L, const double* ego, const double* XYbounds,
                       const double* x, const double* u, const double* l, const double* n, const double* timeScale,
                       const double* sl, int fixTime, int sd, const obca_opts* opts, int* feasible, int* e,
                       int* strict) {
  return check_parking({B, N, nullptr, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, x, u, l, n, timeScale, sl, fixTime, sd, opts, feasible,
                        e, strict}, Arrays::HOST, false, nullptr);
}

int obca_check_parking_mixed(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                             const double* x0, const double* xF, double Ts, double L, const double* ego,
                             const double* XYbounds, const double* x, const double* u, const double* l, const double* n,
                             const double* timeScale, const double* sl, int fixTime, int sd, const obca_opts* opts,
                             int* feasible, int* e, int* strict) {
  return check_parking({B, Nmax, Nb, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, x, u, l, n, timeScale, sl, fixTime, sd, opts, feasible,
                        e, strict}, Arrays::HOST, true, nullptr);
}

int obca_quadcopter_solve_batch(int B, int N, const double* x0, const double* xF, double Ts, double R, const double* ob,
                                const double* xWS, double timeWS, int signed_dist, const obca_opts* opts, double* xp,
                                double* up, double* ts, double* lp, double* slack, int* exitflag, int* iters,
                                double* kkt_err, double* solve_seconds) {
  return quad_solve({B, N, nullptr, nullptr, x0, xF, Ts, R, ob, xWS, timeWS, signed_dist, opts, xp, up, ts, lp, slack, exitflag, iters,
                     kkt_err, solve_seconds}, Arrays::HOST, false, nullptr);
}

// The mixed quadcopter entries' batch has no sampling time of its own: Ts is NaN, so that a read of it instead of Tsb[b] could not go
// unnoticed.
int obca_quadcopter_solve_mixed(int B, const int* Nb, int Nmax, const double* x0, const double* xF, const double* Tsb,
                                double R, const double* ob, const double* xWS, double timeWS, int signed_dist,
                                const obca_opts* opts, double* xp, double* up, double* ts, double* lp, double* slack,
                                int* exitflag, int* iters, double* kkt_err, double* solve_seconds) {
  return quad_solve({B, Nmax, Nb, Tsb, x0, xF, std::nan(""), R, ob, xWS, timeWS, signed_dist, opts, xp, up, ts, lp, slack, exitflag, iters,
                     kkt_err, solve_seconds}, Arrays::HOST, true, nullptr);
}

int obca_check_quadcopter(int B, int N, const double* x, const double* u, const double* timeScale, const double* x0,
                          const double* xF, double Ts, const double* lambda, const double* ob, double R,
                          const obca_opts* opts, int* feasible, double* worst) {
  return quad_check({B, N, nullptr, nullptr, x, u, timeScale, x0, xF, Ts, lambda, ob, R, opts, feasible, worst}, Arrays::HOST, false,
                    nullptr);
}

int obca_check_quadcopter_mixed(int B, const int* Nb, int Nmax, const double* x, const double* u, const double* timeScale,
                                const double* x0, const double* xF, const double* Tsb, const double* lambda,
                                const double* ob, double R, const obca_opts* opts, int* feasible, double* worst) {
  return quad_check({B, Nmax, Nb, Tsb, x, u, timeScale, x0, xF, std::nan(""), lambda, ob, R, opts, feasible, worst}, Arrays::HOST, true,
                    nullptr);
}

int obca_parking_solve_mixed_dev(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                                 const double* x0, const double* xF, double Ts, double L, const double* ego,
                                 const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                                 const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                                 int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up, double* ts,
                                 double* lp, double* np, double* sl, int* exitflag, int* iters, double* kkt_err,
                                 double* solve_seconds, void* stream) {
  return parking_solve({B, Nmax, Nb, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, rx, ry, ryaw, xWS, uWS, lWS, nWS, fixTime, signed_dist,
                        opts, xp, up, ts, lp, np, sl, exitflag, iters, kkt_err, solve_seconds}, Arrays::STREAM, true, stream);
}

int obca_dualmultws_batch_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* ego,
                              const double* rx, const double* ry, const double* ryaw, const obca_opts* opts, double* lp,
                              double* np, double* dd, void* stream) {
  return dualmultws({B, N, nOb, vOb, A, b, ego, rx, ry, ryaw, opts, lp, np, dd}, Arrays::STREAM, stream);
}

int obca_check_parking_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* x0,
                           const double* xF, double Ts, double L, const double* ego, const double* XYbounds,
                           const double* x, const double* u, const double* l, const double* n, const double* timeScale,
                           const double* sl, int fixTime, int sd, const obca_opts* opts, int* feasible, int* e,
                           int* strict, void* stream) {
  return check_parking({B, N, nullptr, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, x, u, l, n, timeScale, sl, fixTime, sd, opts, feasible,
                        e, strict}, Arrays::STREAM, false, stream);
}

int obca_check_parking_mixed_dev(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                                 const double* x0, const double* xF, double Ts, double L, const double* ego,
                                 const double* XYbounds, const double* x, const double* u, const double* l, const double* n,
                                 const double* timeScale, const double* sl, int fixTime, int sd, const obca_opts* opts,
                                 int* feasible, int* e, int* strict, void* stream) {
  return check_parking({B, Nmax, Nb, nOb, vOb, A, b, x0, xF, Ts, L, ego, XYbounds, x, u, l, n, timeScale, sl, fixTime, sd, opts, feasible,
                        e, strict}, Arrays::STREAM, true, stream);
}

int obca_quadcopter_solve_batch_dev(int B, int N, const double* x0, const double* xF, double Ts, double R, const double* ob,
                                    const double* xWS, double timeWS, int signed_dist, const obca_opts* opts, double* xp,
                                    double* up, double* ts, double* lp, double* slack, int* exitflag, int* iters,
                                    double* kkt_err, double* solve_seconds, void* stream) {
  return quad_solve({B, N, nullptr, nullptr, x0, xF, Ts, R, ob, xWS, timeWS, signed_dist, opts, xp, up, ts, lp, slack, exitflag, iters,
                     kkt_err, solve_seconds}, Arrays::STREAM, false, stream);
}

int obca_quadcopter_solve_mixed_dev(int B, const int* Nb, int Nmax, const double* x0, const double* xF, const double* Tsb,
                                    double R, const double* ob, const double* xWS, double timeWS, int signed_dist,
                                    const obca_opts* opts, double* xp, double* up, double* ts, double* lp, double* slack,
                                    int* exitflag, int* iters, double* kkt_err, double* solve_seconds, void* stream) {
  return quad_solve({B, Nmax, Nb, Tsb, x0, xF, std::nan(""), R, ob, xWS, timeWS, signed_dist, opts, xp, up, ts, lp, slack, exitflag, iters,
                     kkt_err, solve_seconds}, Arrays::STREAM, true, stream);
}

int obca_check_quadcopter_dev(int B, int N, const double* x, const double* u, const double* timeScale, const double* x0,
                              const double* xF, double Ts, const double* lambda, const double* ob, double R,
                              const obca_opts* opts, int* feasible, double* worst, void* stream) {
  return quad_check({B, N, nullptr, nullptr, x, u, timeScale, x0, xF, Ts, lambda, ob, R, opts, feasible, worst}, Arrays::STREAM, false,
                    stream);
}

int obca_check_quadcopter_mixed_dev(int B, const int* Nb, int Nmax, const double* x, const double* u, const double* timeScale,
                                    const double* x0, const double* xF, const double* Tsb, const double* lambda,
                                    const double* ob, double R, const obca_opts* opts, int* feasible, double* worst, void* stream) {
  return quad_check({B, Nmax, Nb, Tsb, x, u, timeScale, x0, xF, std::nan(""), lambda, ob, R, opts, feasible, worst}, Arrays::STREAM, true,
                    stream);
}

int obca_parking_plan_solve_goals(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts,
                                  double L, int sampleN, int max_expansions, int max_nodes, int nOb, const int* vOb, const double* A,
                                  const double* b, const double* ego, const double* XYbounds, int fixTime, int signed_dist,
                                  const obca_opts* opts, int Ncap, double* xp, double* up, double* ts, double* lp, double* np, double* sl,
                                  int* N, int* status, int* expansions, int* exitflag, int* iters, double* kkt_err, int* feasible,
                                  int* strict, double* plan_seconds, double* solve_seconds) {
  const obca_parking_flow_out out = {xp, up, ts, lp, np, sl, exitflag, iters, kkt_err, feasible, strict, solve_seconds};
  const FlowSet<obca_parking_flow_out> set = {signed_dist, &out};
  return parking_plan_solve(B, x0, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, nOb, vOb, A, b, ego, XYbounds, fixTime,
                            opts, Ncap, N, status, expansions, plan_seconds, 1, &set);
}

int obca_parking_plan_solve_both(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts,
                                 double L, int sampleN, int max_expansions, int max_nodes, int nOb, const int* vOb, const double* A,
                                 const double* b, const double* ego, const double* XYbounds, int fixTime, const obca_opts* opts,
                                 int Ncap, int* N, int* status, int* expansions, double* plan_seconds, const obca_parking_flow_out* dist,
                                 const obca_parking_flow_out* sd) {
  const int rc = check_both_sets(dist, sd);
  if (rc) return rc;
  const FlowSet<obca_parking_flow_out> sets[2] = {{0, dist}, {1, sd}};      // main.jl:258, then :269
  return parking_plan_solve(B, x0, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, nOb, vOb, A, b, ego, XYbounds, fixTime,
                            opts, Ncap, N, status, expansions, plan_seconds, 2, sets);
}

int obca_quadcopter_plan_solve(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz, int n_ob,
                               const double* lo, const double* hi, double reso, int max_nodes, double Ts, double R, const double* ob,
                               double timeWS, int signed_dist, const obca_opts* opts, int Ncap, double* xp, double* up, double* ts,
                               double* lp, double* slack, int* N, double* Tsb, int* status, int* expansions, int* exitflag, int* iters,
                               double* kkt_err, int* feasible, double* worst, double* plan_seconds, double* solve_seconds) {
  const obca_quadcopter_flow_out out = {xp, up, ts, lp, slack, exitflag, iters, kkt_err, feasible, worst, solve_seconds};
  const FlowSet<obca_quadcopter_flow_out> set = {signed_dist, &out};
  return quad_plan_solve(B, x0, xF, ox, oy, oz, n_ob, lo, hi, reso, max_nodes, Ts, R, ob, timeWS, opts, Ncap, N, Tsb, status, expansions,
                         plan_seconds, 1, &set);
}

int obca_quadcopter_plan_solve_both(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz,
                                    int n_ob, const double* lo, const double* hi, double reso, int max_nodes, double Ts, double R,
                                    const double* ob, double timeWS, const obca_opts* opts, int Ncap, int* N, double* Tsb, int* status,
                                    int* expansions, double* plan_seconds, const obca_quadcopter_flow_out* dist,
                                    const obca_quadcopter_flow_out* sd) {
  const int rc = check_both_sets(dist, sd);
  if (rc) return rc;
  const FlowSet<obca_quadcopter_flow_out> sets[2] = {{0, dist}, {1, sd}};      // mainQuadcopter.jl:145-147, then :152-154
  return quad_plan_solve(B, x0, xF, ox, oy, oz, n_ob, lo, hi, reso, max_nodes, Ts, R, ob, timeWS, opts, Ncap, N, Tsb, status, expansions,
                         plan_seconds, 2, sets);
}

int obca_last_profile(int device, unsigned long long* out8) {
  const DevCtx* c = used_ctx(device);
  if (!c || !out8) { set_err("no profile"); return OBCA_ERR_ARG; }
  for (int i = 0; i < 8; ++i) out8[i] = c->prof_host[i];
  return 0;
}

int obca_last_schedule(int device, int* rounds, int* handed_over, double* kernel_ms5) {
  const DevCtx* c = used_ctx(device);
  if (!c) { set_err("no schedule"); return OBCA_ERR_ARG; }
  if (rounds) *rounds = c->last_rounds;
  if (handed_over) *handed_over = c->last_tail;
  if (kernel_ms5) for (int i = 0; i < 5; ++i) kernel_ms5[i] = c->phase_ms[i];
  return 0;
}

int obca_last_times(int device, double* dualws_seconds, double* solve_seconds) {
  const DevCtx* c = used_ctx(device);
  if (!c) { set_err("no solve yet"); return OBCA_ERR_ARG; }
  if (dualws_seconds) *dualws_seconds = c->last_dualws_s;
  if (solve_seconds) *solve_seconds = c->last_solve_s;
  return 0;
}

int obca_parking_eval_sizes(int N, int nOb, const int* vOb, int signed_dist, long long* n_out, long long* m_out) {
  ParkProblem P;
  double A[2 * OBCA_MAX_ROWS] = {0}, b[OBCA_MAX_ROWS] = {0}, ego[4] = {1, 1, 1, 1}, xy[4] = {0, 1, 0, 1};
  if (const int e_ = fill_problem(P, N, nOb, vOb, A, b, 1.0, 1.0, ego, xy, 0, signed_dist)) { set_err(shape_error(e_)); return OBCA_ERR_ARG; }
  if (n_out) *n_out = (long long)eval_n(P);
  if (m_out) *m_out = (long long)eval_m(P);
  return 0;
}

int obca_parking_eval_batch_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b,
                                const double* x0, const double* xF, double Ts, double L, const double* ego,
                                const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                                const double* xp, const double* up, const double* ts, const double* lp,
                                const double* np, const double* sl, const double* y, int fixTime, int signed_dist,
                                const obca_opts* opts, double* c_out, double* gradL_out, double* fk_out, int reps,
                                double* kernel_ms) {
  if (B <= 0 || !vOb || !A || !b || !x0 || !xF || !ego || !XYbounds || !rx || !ry || !ryaw || !xp || !up || !lp || !np ||
      !c_out || !gradL_out || !fk_out || (signed_dist && !sl) || (!fixTime && !ts)) { set_err("null argument"); return OBCA_ERR_ARG; }
  ParkProblem P;
  if (const int e_ = fill_problem(P, N, nOb, vOb, A, b, Ts, L, ego, XYbounds, fixTime, signed_dist)) { set_err(shape_error(e_)); return OBCA_ERR_ARG; }
  DevCtx* c;
  int rc = get_ctx(opts ? opts->device : 0, &c);
  if (rc) return rc;
  std::lock_guard<std::recursive_mutex> lk(c->mu);
  EvalIn in; in.x0 = x0; in.xF = xF; in.rx = rx; in.ry = ry; in.ryaw = ryaw; in.xp = xp; in.up = up; in.ts = ts; in.lp = lp;
  in.np = np; in.sl = sl; in.y = y;
  EvalOut out; out.c = c_out; out.gradL = gradL_out; out.fk = fk_out;
  if (reps < 1) reps = 1;
  const size_t total = (size_t)B * (P.N + 1);
  const int threads = 128;
  const int blocks = (int)((total + threads - 1) / threads);
  CK(cudaEventRecord(c->ev0, c->st));
  with_variant(P, [&](auto vm, auto sdv) {
    for (int r = 0; r < reps; ++r) k_parking_eval<decltype(vm)::value, decltype(sdv)::value><<<blocks, threads, 0, c->st>>>(P, B, in, out);
    return 0;
  });
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaStreamSynchronize(c->st));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
  if (kernel_ms) *kernel_ms = ms / reps;
  return 0;
}
}
