// obca_phased.cuh -- phase-split ("lock-step") schedule of the batched parking solve.
//
// The phase functions of IpmDriver<M> (obca_solver.cuh: phase_A, phase_B_serial, phase_C), run from separate kernels over
// ALL active problems of the batch, so that the parallel phases and the serial-in-time KKT sweep of an iteration each get
// the launch shape that suits them.  One round = three launches:
//     k_pk_eval    persistent CTAs, one problem at a time: K1 -- item pass (one thread per (obstacle, stage) block:
//                  evaluation, KKT-error partials, condensation onto the stage pose; hand-over of the 12 doubles per block
//                  the assembly needs IN THE STAGE SLOT, shared memory, for the first six obstacles, in workspace rows for
//                  the others), stage pass (dynamics, objective, bounds, assembly
//                  of the stage models), reductions, convergence test, barrier update -- and, when the barrier parameter
//                  was reduced, the re-evaluation, in the same launch.  The finished stage models leave shared memory in
//                  ONE bulk copy (cp.async.bulk.global.shared::cta, 53 KB per problem).  Also: initial point, end of
//                  attempt (status / retry / checker), compaction of the active list.
//     k_pk_sweep   one WARP per problem: K3 stage-banded KKT sweep; the 656-byte stage slots are streamed from HBM through
//                  an 8-deep ring of cp.async (LDGSTS) copies, gains and costate rows written back in place;
//                  inertia-correction bookkeeping (phase_B_serial).
//     k_pk_step    persistent CTAs, one problem at a time: K4 -- item pass (steps of the block unknowns from the stored
//                  local maps) + stage pass (costates, bounds), fraction-to-the-boundary, filter line search (merit
//                  function: item + stage pass), iterate update.  The step of the block unknowns lives in shared memory
//                  while the kernel keeps its resident CTAs with it there, else in the workspace.
// The persistent CTAs of k_pk_eval and k_pk_step take their problems from an atomic work queue (pk_queue_next).
// The iterate, the local maps and the stage slots of every problem live in HBM (layout: problem-major, then [array][stage],
// so each warp streams contiguous slices); between kernels a problem is described by its ProbState record (phase,
// iteration, barrier parameter, filter, ...).  When the active set has shrunk far enough the remaining problems are handed to
//     k_pk_tail    persistent CTA per problem: the phase functions in a loop (the loop of IpmDriver::solve plus the end of
//                  attempt), stage slots in shared memory
// which is also the whole solver for small batches.
//
// Every floating-point operation of a phase lives in ONE out-of-line device function per template instance
// (IpmDriver::phase_A / phase_C and the per-item / per-stage functions of ParkSolver) that all kernels call: the
// schedules produce bit-identical iterates by construction (tests/test_gpu_parking.py::test_phased_equals_persistent).
#pragma once
#include "obca_check.cuh"
#include "obca_solver.cuh"

namespace obca {

struct BatchPtrs {
  const double *x0, *xF, *rx, *ry, *ryaw, *xWS, *uWS, *lWS, *nWS;
  const int* Nb;              // per-problem horizons (<= P.N), or null: every problem has the horizon P.N
  double *xp, *up, *ts, *lp, *np, *sl, *duals;
  int *exitflag, *iters;
  double* kkt_err;
  int B;
  int retry;
  int q4;                     // 1: reproduce the inverted test of ParkingDist.jl:278-282 after a second failure (SURVEY Q4)
  unsigned long long* prof;   // optional: 8 counters summed over the batch (device pointer)
};

#if defined(__CUDACC__)

// ------------------------------------------------------------------------------------------------------------
// Bulk copy (sm_90) of the finished stage slots from shared to global memory (k_pk_eval)
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
// shared -> global bulk copy (bulk async-group completion)
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;\n" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
// writes of the generic proxy (st.shared) become visible to the async proxy (the bulk copy engine)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }

// ------------------------------------------------------------------------------------------------------------
// helpers
// ------------------------------------------------------------------------------------------------------------
// ProbState <-> global memory, cooperatively, as 8-byte words
static_assert(sizeof(ProbState) % 8 == 0, "ProbState must be a whole number of 8-byte words");
__device__ __forceinline__ void state_load(ProbState& S, const ProbState* g) {
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(g);
  unsigned long long* dst = reinterpret_cast<unsigned long long*>(&S);
  for (int i = threadIdx.x; i < (int)(sizeof(ProbState) / 8); i += blockDim.x) dst[i] = src[i];
}
__device__ __forceinline__ void state_store(ProbState* g, const ProbState& S) {
  const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&S);
  unsigned long long* dst = reinterpret_cast<unsigned long long*>(g);
  for (int i = threadIdx.x; i < (int)(sizeof(ProbState) / 8); i += blockDim.x) dst[i] = src[i];
}

__device__ __forceinline__ int pk_horizon(const BatchPtrs& bp, const ParkProblem& P, int b) { return bp.Nb ? bp.Nb[b] : P.N; }

// Every per-problem array of the batch is laid out for the batch's horizon P.N (strides); problem b uses its own first
// Nb[b] + 1 stages of them (extents, C.N).
template <int VM, bool SDV>
__device__ __forceinline__ void pk_make_ctx(PkCtx& C, PkOutputs& out, const ParkProblem& P, const IpmOpts& O, const PkLay& L,
                                            const BatchPtrs& bp, int b, double* W) {
  const int N = P.N, NS = N + 1, V = P.V, nOb = P.nOb;
  C.P = &P; C.N = pk_horizon(bp, P, b); C.O = &O; C.L = L; C.W = W; C.Wd = W + (size_t)L.dLAM * L.NSP;
  C.in.x0 = bp.x0 + 4 * (size_t)b; C.in.xF = bp.xF + 4 * (size_t)b;
  C.in.rx = bp.rx + (size_t)NS * b; C.in.ry = bp.ry + (size_t)NS * b; C.in.ryaw = bp.ryaw + (size_t)NS * b;
  C.in.xWS = bp.xWS + (size_t)4 * NS * b; C.in.ldx = NS;
  C.in.uWS = bp.uWS + (size_t)2 * N * b; C.in.ldu = N;
  C.in.lWS = bp.lWS + (size_t)V * NS * b; C.in.nWS = bp.nWS + (size_t)4 * nOb * NS * b;
  out.xp = bp.xp + (size_t)4 * NS * b; out.up = bp.up + (size_t)2 * N * b; out.ts = bp.ts + (size_t)NS * b;
  out.lp = bp.lp + (size_t)V * NS * b; out.np = bp.np + (size_t)4 * nOb * NS * b;
  out.sl = bp.sl ? bp.sl + (size_t)nOb * NS * b : nullptr;
  out.duals = bp.duals ? bp.duals + ((size_t)4 * N + (size_t)4 * nOb * NS) * b : nullptr;
}

struct PkFinalScratch {
  ChkPart chk[8];
  int feas;
};

// End of an attempt (phase PH_END): the reference's status / retry logic around solve(m).
//   ParkingSignedDist.jl:256-283: status Optimal -> exitflag 1; Error / UserLimit -> one more solve from the last iterate;
//     after a second failure ParkingConstraints decides (exitflag = Feasible).
//   ParkingDist.jl:245-289: the first failure is followed by ParkingConstraints; only an INFEASIBLE point is solved again
//     (a feasible one is accepted: exitflag 1, :259-262); after a second failure the reference's test is inverted
//     (:278-282, Feasible == 0 -> exitflag 1: SURVEY Q4) -- reproduced with opts.q4 = 1, fixed (exitflag = Feasible) otherwise.
// Leaves PH_INIT (second attempt) or PH_DONE (outputs written).
template <int VM, bool SDV>
__device__ __noinline__ void pk_end_of_attempt(const PkCtx& C, const PkOutputs& out, const BatchPtrs& bp, int b, PkFinalScratch& F) {
  ProbState& S = *C.S;
  const ParkProblem& P = CTX_P(C);
  const int NS = C.N + 1;
  const int status = S.status;
  const int attempt = S.attempt;
  __syncthreads();      // everybody has read the state before thread 0 changes it
  const bool failed = status != 1 && bp.retry;
  if (failed && attempt == 0 && SDV) {      // SignedDist: always solve again
    if (threadIdx.x == 0) { S.iters_total += S.iters; S.attempt = 1; S.phase = PH_INIT; }
    __syncthreads();
    return;
  }
  for (int k = threadIdx.x; k < NS; k += blockDim.x) ParkSolver<VM, SDV>::store_stage(C, k, out);
  __syncthreads();
  int exitflag = status == 1 ? 1 : 0;
  if (failed) {
    ChkPart c;
    chk_init(c);
    for (int k = threadIdx.x; k < NS; k += blockDim.x) {
      ChkPart ck;
      check_stage(P, C.N, k, C.in.x0, C.in.xF, out.xp, out.up, out.lp, out.np, out.ts, out.sl, SDV ? 1 : 0, 0, ck);
      chk_merge(c, ck);
    }
    for (int off = 16; off > 0; off >>= 1) {
      ChkPart o;
#pragma unroll
      for (int i = 0; i < 5; ++i) o.c0[i] = __shfl_down_sync(0xffffffffu, c.c0[i], off);
      o.c1 = __shfl_down_sync(0xffffffffu, c.c1, off); o.c2 = __shfl_down_sync(0xffffffffu, c.c2, off);
      o.c3 = __shfl_down_sync(0xffffffffu, c.c3, off); o.c4 = __shfl_down_sync(0xffffffffu, c.c4, off);
      o.c5 = __shfl_down_sync(0xffffffffu, c.c5, off); o.c6 = __shfl_down_sync(0xffffffffu, c.c6, off);
      o.sbox = __shfl_down_sync(0xffffffffu, c.sbox, off);
      chk_merge(c, o);
    }
    if ((threadIdx.x & 31) == 0) F.chk[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < (int)(blockDim.x >> 5); ++w) chk_merge(c, F.chk[w]);
      int e[7];
      F.feas = check_finish(P, c, out.ts, 0, 5e-5, e);
    }
    __syncthreads();
    const int feas = F.feas;
    if (!SDV && attempt == 0) {
      // ParkingDist.jl:256-263: only an infeasible point is solved again
      if (!feas) {
        if (threadIdx.x == 0) { S.iters_total += S.iters; S.attempt = 1; S.phase = PH_INIT; }
        __syncthreads();
        return;
      }
      exitflag = 1;
    } else if (!SDV && bp.q4) {
      exitflag = feas ? 0 : 1;          // ParkingDist.jl:278-282 as written (inverted)
    } else {
      exitflag = feas ? 1 : 0;          // ParkingSignedDist.jl:278-283
    }
  }
  if (threadIdx.x == 0) {
    bp.exitflag[b] = exitflag;
    bp.iters[b] = S.iters_total + S.iters;
    bp.kkt_err[b] = S.e0;
    S.phase = PH_DONE;
  }
  __syncthreads();
}

// phase A of one problem including the attempt bookkeeping; returns with phase in {PH_KKT, PH_DONE}
template <int VM, bool SDV>
__device__ __forceinline__ void pk_step_A(const PkCtx& C, const PkOutputs& out, const BatchPtrs& bp, int b, PkFinalScratch& F) {
  ProbState& S = *C.S;
  for (;;) {
    if (S.phase == PH_END) pk_end_of_attempt<VM, SDV>(C, out, bp, b, F);
    if (S.phase == PH_DONE) return;
    IpmDriver<ParkSolver<VM, SDV> >::phase_A(C);
    if (S.phase != PH_END) return;
  }
}

#ifndef OBCA_PK_THREADS
#define OBCA_PK_THREADS 128
#endif
// CTA size of the per-problem kernels (item passes: nOb (N+1) work items, stage passes: N+1).  The same for all of them: the
// per-thread partial sums of a reduction depend on it, and the schedules must round identically.
constexpr int PK_THREADS = OBCA_PK_THREADS;

// Work queues of K_eval and K_step: a CTA takes the next problem of the active list from an atomic counter when it has
// finished the last one, instead of every gridDim.x-th problem.  The cost of a problem varies several-fold (re-evaluation
// after a barrier update, end of an attempt, backtracking in the line search), and with a fixed stride a launch lasted as
// long as the CTA whose share held the most of it.  Each of the two kernels has its own counter and zeroes the other's
// (the two alternate on the stream, with the sweep between them), so no host memset is needed between the launches of a
// CUDA graph.
__device__ __forceinline__ int pk_queue_next(int* queue, int* s_i) {
  if (threadIdx.x == 0) *s_i = atomicAdd(queue, 1);
  __syncthreads();
  return *s_i;
}

// ------------------------------------------------------------------------------------------------------------
// K_eval: persistent CTAs, one problem at a time (see the file header).  fresh: first launch of a solve -- every problem
// of the batch starts from its warm start (no active list yet).
// ------------------------------------------------------------------------------------------------------------
#ifndef OBCA_MINB_A
#define OBCA_MINB_A 3
#endif
template <int VM, bool SDV>
__global__ void __launch_bounds__(PK_THREADS, OBCA_MINB_A)
k_pk_eval(const __grid_constant__ ParkProblem P, const __grid_constant__ IpmOpts O, const PkLay L, const BatchPtrs bp,
          double* __restrict__ Wall, double* __restrict__ slots, ProbState* __restrict__ Sg,
          const int* __restrict__ act_in, const int* __restrict__ n_in, int* __restrict__ act_out, int* __restrict__ n_out,
          int fresh, int* __restrict__ queue, int* __restrict__ queue_next) {
  extern __shared__ __align__(16) double s_ric[];     // (N+1) x RSTRIDE stage slots: hand-over area of the item pass, then
                                                     // the assembled stage models, bulk-copied out for the sweep kernel
  __shared__ ProbState S;
  __shared__ double s_red[4 * 12];
  __shared__ PkFinalScratch s_fin;
  __shared__ int s_i;
  __shared__ PkCtx C; __shared__ PkOutputs out;
  const int NSL = P.N + 1;      // stage slots per problem in `slots`
  const int n = fresh ? bp.B : *n_in;
  if (blockIdx.x == 0 && threadIdx.x == 0) *queue_next = 0;
  unsigned long long n_eval = 0, n_eval2 = 0;
  for (;;) {
    const int a = pk_queue_next(queue, &s_i);
    if (a >= n) break;
    const int b = fresh ? a : act_in[a];
    if (fresh) state_fresh(S, pk_horizon(bp, P, b)); else state_load(S, Sg + b);
    if (threadIdx.x == 0) {
      bulk_wait_read0();      // the bulk copy of the previous problem has finished reading the slots
      pk_make_ctx<VM, SDV>(C, out, P, O, L, bp, b, Wall + (size_t)b * L.total * L.NSP);
      C.ric = s_ric; C.pp = s_ric; C.red_scratch = s_red; C.tile = nullptr; C.S = &S;
    }
    __syncthreads();
    if (threadIdx.x == 0) { S.prof[7] = 0; S.prof[5] = 0; }
    __syncthreads();
    pk_step_A<VM, SDV>(C, out, bp, b, s_fin);
    if (S.phase == PH_KKT) {
      fence_proxy_async();
      __syncthreads();
      if (threadIdx.x == 0) {
        bulk_s2g(slots + (size_t)b * NSL * RSTRIDE, s_ric, (unsigned)((C.N + 1) * RSTRIDE * sizeof(double)));
        bulk_commit();
      }
    }
    state_store(Sg + b, S);
    if (threadIdx.x == 0) {
      n_eval += (unsigned long long)S.prof[7]; n_eval2 += (unsigned long long)S.prof[5];
      if (S.phase != PH_DONE) act_out[atomicAdd(n_out, 1)] = b;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    bulk_wait_read0();
    if (bp.prof) { atomicAdd(bp.prof + 7, n_eval); atomicAdd(bp.prof + 5, n_eval2); }
  }
}

// ------------------------------------------------------------------------------------------------------------
// K_sweep: one WARP per problem (wide lane program of ParkSolver: <= 2 scalar tasks per lane and step).  Backward Riccati
// sweep + forward roll-out with the stage slots streamed from global memory (each slot = 656 contiguous bytes) through a
// ring of asynchronous copies, SWEEP_DEPTH - 1 stages ahead: the recursion is a serial chain, so the look-ahead has to
// cover the memory latency at a fraction of a microsecond per stage.  Gains and the P_k rows needed by the multiplier
// recovery are written back in place (consumed Q/q space of the slots).
// The ring uses LDGSTS (cp.async, 41 x 16 bytes per slot spread over the lanes), not bulk copies: with cp.async.bulk + an
// mbarrier per slot (one elected lane) the issue sequence of a bulk copy (expect-tx, uniform-register moves, try-wait) sits
// on the latency-bound chain of every stage, the LDGSTS of a lane does not.
// ------------------------------------------------------------------------------------------------------------
#ifndef OBCA_SWEEP_DEPTH
#define OBCA_SWEEP_DEPTH 8
#endif
constexpr int SWEEP_DEPTH = OBCA_SWEEP_DEPTH;      // ring slots per warp (power of two)
constexpr int SWEEP_WARP_DOUBLES = SWEEP_DEPTH * RSTRIDE + 256;   // ring + tile (ParkSolver::WIDE_TILE)
static_assert((RSTRIDE * 8) % 16 == 0 && (SWEEP_WARP_DOUBLES % 2) == 0, "16-byte alignment of the ring slots");

__device__ __forceinline__ void sweep_prefetch(double* ring, const double* gslots, int k, int lane, int n) {
  if (k >= 0 && k < n) {
    double* dst = ring + (k & (SWEEP_DEPTH - 1)) * RSTRIDE;
    const double* src = gslots + (size_t)k * RSTRIDE;
    cp_async16(dst + 2 * lane, src + 2 * lane);                          // 41 x 16 bytes: 32 + 9
    if (lane < RSTRIDE / 2 - 32) cp_async16(dst + 64 + 2 * lane, src + 64 + 2 * lane);
  }
  cp_async_commit();
}

// one warp, one problem of horizon N.  Returns 1 if the sweep found inertia (n, m, 0).
template <int VM, bool SDV>
__device__ int pk_sweep_warp(const ParkProblem& Pp, const IpmOpts& O, const PkLay& Lay, int N, double* W, double* gslots,
                             ProbState* Sgl, double* ring, double* tile) {
  typedef ParkSolver<VM, SDV> PS;
  const int lane = threadIdx.x & 31;
  PkCtx C;
  C.P = &Pp; C.N = N; C.O = &O; C.L = Lay; C.W = W; C.Wd = W; C.ric = ring; C.pp = gslots;   // ric: any shared address (OBCA_LOCALS)
  typename PS::WideLane L;
#pragma unroll
  for (int a = 1; a < SWEEP_DEPTH; ++a) sweep_prefetch(ring, gslots, N - a, lane, N);
  PS::wl_init(L, lane);
  PS::wl_zero(lane, tile, gslots + (size_t)N * RSTRIDE);
  __syncwarp();
  PS::wl_terminal(lane, tile, gslots + (size_t)N * RSTRIDE, C);
  __syncwarp();
  for (int k = N - 1; k >= 0; --k) {
    sweep_prefetch(ring, gslots, k - (SWEEP_DEPTH - 1), lane, N);
    cp_async_wait<SWEEP_DEPTH - 1>();
    __syncwarp();
    const double* slot = ring + (k & (SWEEP_DEPTH - 1)) * RSTRIDE;
    PS::wl_step1(L, slot, tile);
    __syncwarp();
    PS::wl_step2(L, slot, tile);
    __syncwarp();
    PS::wl_step3(L, gslots + (size_t)k * RSTRIDE, tile);
    __syncwarp();
    if (!L.ok) break;
  }
  cp_async_wait<0>();
  if (!L.ok) return 0;
  __threadfence();      // the gains written above are read back through the ring below
  __syncwarp();
#pragma unroll
  for (int a = 0; a < SWEEP_DEPTH - 1; ++a) sweep_prefetch(ring, gslots, a, lane, N);
  const int ok = PS::kkt_forward_warp(C, tile, Sgl, true, [&](int k) {
    sweep_prefetch(ring, gslots, k + (SWEEP_DEPTH - 1), lane, N);
    cp_async_wait<SWEEP_DEPTH - 1>();
    __syncwarp();
    return (const double*)(ring + (k & (SWEEP_DEPTH - 1)) * RSTRIDE);
  });
  cp_async_wait<0>();
  return ok;
}

constexpr int SWEEP_WARPS = 4;
template <int VM, bool SDV>
__global__ void __launch_bounds__(32 * SWEEP_WARPS)
k_pk_sweep(const __grid_constant__ ParkProblem P, const __grid_constant__ IpmOpts O, const PkLay L,
           double* __restrict__ Wall, double* __restrict__ slots, ProbState* __restrict__ Sg,
           const int* __restrict__ act, const int* __restrict__ n_act, int* __restrict__ n_zero) {
  extern __shared__ __align__(16) double s_w[];      // SWEEP_WARPS x SWEEP_WARP_DOUBLES
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (blockIdx.x == 0 && threadIdx.x == 0 && n_zero) *n_zero = 0;      // the active count that the next round's K_eval fills
  const int n = *n_act;
  const int idx = blockIdx.x * SWEEP_WARPS + warp;
  if (idx >= n) return;
  const int b = act[idx];
  ProbState* S = Sg + b;
  if (S->phase != PH_KKT) return;
  const int NSL = P.N + 1;      // stage slots per problem in `slots`
  double* hw = s_w + (size_t)warp * SWEEP_WARP_DOUBLES;
  int ok = 0;
  if (S->ok != 0)
    ok = pk_sweep_warp<VM, SDV>(P, O, L, S->N, Wall + (size_t)b * L.total * L.NSP, slots + (size_t)b * NSL * RSTRIDE, S, hw,
                                hw + SWEEP_DEPTH * RSTRIDE);
  __syncwarp();
  if (lane == 0) IpmDriver<ParkSolver<VM, SDV> >::phase_B_serial(*S, O, ok);
}

// ------------------------------------------------------------------------------------------------------------
// K_step: persistent CTAs, one problem at a time.  The rows of the step that the sweep does not produce (block unknowns,
// new multipliers, slack steps: V + 10 nOb + 5 rows, 40 of 46 for config 2) stay in shared memory when they fit there
// (step_smem = 1; the host's rule, step_rows_in_smem); otherwise they are the workspace rows dLAM .. dRS, as in k_pk_tail.
// ------------------------------------------------------------------------------------------------------------
#ifndef OBCA_MINB_C
#define OBCA_MINB_C 5
#endif
template <int VM, bool SDV>
__global__ void __launch_bounds__(PK_THREADS, OBCA_MINB_C)
k_pk_step(const __grid_constant__ ParkProblem P, const __grid_constant__ IpmOpts O, const PkLay L, const BatchPtrs bp,
          double* __restrict__ Wall, double* __restrict__ slots, ProbState* __restrict__ Sg,
          const int* __restrict__ act, const int* __restrict__ n_act, int* __restrict__ queue, int* __restrict__ queue_next,
          int step_smem) {
  extern __shared__ __align__(16) double s_step[];      // step_smem: (dRS + 1 - dLAM) x NSP, else empty
  __shared__ ProbState S;
  __shared__ double s_red[4 * 12];
  __shared__ int s_i;
  __shared__ PkCtx C; __shared__ PkOutputs out;
  const int NSL = P.N + 1;      // stage slots per problem in `slots`
  const int n = *n_act;
  if (blockIdx.x == 0 && threadIdx.x == 0) *queue_next = 0;
  unsigned long long n_merit = 0;
  for (;;) {
    const int a = pk_queue_next(queue, &s_i);
    if (a >= n) break;
    const int b = act[a];
    if (Sg[b].phase != PH_RECOVER) {      // (uniform: every thread reads the same word)
      __syncthreads();                    // every thread has read s_i before thread 0 takes the next problem
      continue;
    }
    state_load(S, Sg + b);
    if (threadIdx.x == 0) {
      pk_make_ctx<VM, SDV>(C, out, P, O, L, bp, b, Wall + (size_t)b * L.total * L.NSP);
      if (step_smem) C.Wd = s_step;
      C.ric = s_step /* unused here; a shared address as OBCA_LOCALS assumes */; C.pp = slots + (size_t)b * NSL * RSTRIDE; C.red_scratch = s_red; C.tile = nullptr; C.S = &S;
    }
    __syncthreads();
    if (threadIdx.x == 0) S.prof[6] = 0;
    __syncthreads();
    IpmDriver<ParkSolver<VM, SDV> >::phase_C(C);
    state_store(Sg + b, S);
    if (threadIdx.x == 0) n_merit += (unsigned long long)S.prof[6];
    __syncthreads();
  }
  if (threadIdx.x == 0 && bp.prof) atomicAdd(bp.prof + 6, n_merit);
}

// ------------------------------------------------------------------------------------------------------------
// tail / small-batch kernel: persistent CTAs pull problems (fresh, or handed over by the round kernels at a round
// boundary) and run the phases in a loop with the stage slots in shared memory.
// ------------------------------------------------------------------------------------------------------------
#ifndef OBCA_MIN_BLOCKS
#define OBCA_MIN_BLOCKS 3
#endif
template <int VM, bool SDV>
__global__ void __launch_bounds__(PK_THREADS, OBCA_MIN_BLOCKS)
k_pk_tail(const __grid_constant__ ParkProblem P, const __grid_constant__ IpmOpts O, const PkLay L, const BatchPtrs bp,
          double* __restrict__ Wall, ProbState* __restrict__ Sg, const int* __restrict__ act, const int* __restrict__ n_act,
          int* __restrict__ counter, int fresh) {
  extern __shared__ __align__(16) double s_ric[];
  __shared__ ProbState S;
  __shared__ double s_tile[ParkSolver<VM, SDV>::WIDE_TILE];
  __shared__ double s_red[4 * 12];
  __shared__ PkFinalScratch s_fin;
  __shared__ int s_i;
  __shared__ PkCtx C; __shared__ PkOutputs out;
  typedef ParkSolver<VM, SDV> PS;
  const int n = fresh ? bp.B : *n_act;
  unsigned long long n_eval = 0, n_merit = 0;
  for (;;) {
    if (threadIdx.x == 0) s_i = atomicAdd(counter, 1);
    __syncthreads();
    const int i = s_i;
    if (i >= n) break;
    const int b = fresh ? i : act[i];
    if (fresh) state_fresh(S, pk_horizon(bp, P, b)); else state_load(S, Sg + b);
    if (threadIdx.x == 0) {
      pk_make_ctx<VM, SDV>(C, out, P, O, L, bp, b, Wall + (size_t)b * L.total * L.NSP);
      C.ric = s_ric; C.pp = s_ric; C.red_scratch = s_red; C.tile = s_tile; C.S = &S;
    }
    __syncthreads();
    if (threadIdx.x == 0) { S.prof[7] = 0; S.prof[6] = 0; }
    __syncthreads();
    for (;;) {
      pk_step_A<VM, SDV>(C, out, bp, b, s_fin);
      const int ph = S.phase;
      __syncthreads();      // every thread has read the phase before thread 0 moves it on (phase_B_serial)
      if (ph == PH_DONE) break;
      const int ok = PS::factor(C);
      if (threadIdx.x == 0) IpmDriver<PS>::phase_B_serial(S, O, ok);
      __syncthreads();
      if (S.phase == PH_RECOVER) IpmDriver<PS>::phase_C(C);
    }
    if (threadIdx.x == 0) { n_eval += (unsigned long long)S.prof[7]; n_merit += (unsigned long long)S.prof[6]; }
    __syncthreads();
  }
  if (threadIdx.x == 0 && bp.prof) { atomicAdd(bp.prof + 4, n_eval); atomicAdd(bp.prof + 3, n_merit); }
}

#endif  // __CUDACC__

}  // namespace obca
