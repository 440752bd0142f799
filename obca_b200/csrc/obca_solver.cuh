// obca_solver.cuh -- one OBCA parking NLP solved by one CTA (thread k <-> stage k).
//
// Replaces, for the batched path, what the reference does with JuMP + Ipopt + MUMPS inside
// ParkingSignedDist.jl:41-43,213-240 / ParkingDist.jl:41-43,215-241:
//   K1  stage_eval     fused evaluation of objective, constraints, Jacobian/Hessian blocks and KKT-error pieces,
//                      with in-register condensation of every OBCA block onto the stage pose
//   K3  kkt_solve      stage-banded KKT solve (Riccati sweep = block LDL' in time order) + inertia test
//   K4  recover / merit / update   step recovery, fraction-to-the-boundary, filter line search, iterate update
// The algorithm is the published Ipopt algorithm (Waechter & Biegler 2006): monotone barrier update, inertia
// correction by delta_w escalation, filter line search (oracle/ipm_ref.py is the independent restatement).
//
// Execution model: OBCA_FOR_STAGES bodies run once per stage (device: thread k of the CTA; host emulation: a loop),
// OBCA_SERIAL bodies run once per problem (device: thread 0).  Everything that lives across phases is in the
// per-CTA workspace W (global memory, L2 resident) or in the ProbState struct (shared memory).
#pragma once
#include "obca_common.cuh"
#include "obca_local.cuh"
#include "obca_stage.cuh"

#if defined(__CUDA_ARCH__)
#define OBCA_FOR_STAGES(k, ns) for (int k = threadIdx.x; k < (ns); k += blockDim.x)
#define OBCA_FOR_ITEMS(i, n) for (int i = threadIdx.x; i < (n); i += blockDim.x)
#define OBCA_SYNC() __syncthreads()
#define OBCA_SERIAL if (threadIdx.x == 0)
// phase profiling of the models with M::PROF_CYCLES: thread 0 charges the cycles since the last mark to counter i (call right
// after a barrier); OBCA_PROF_START() sets the first mark
#define OBCA_PROF_START() do { if (M::PROF_CYCLES && threadIdx.x == 0) S.tmark = clock64(); } while (0)
#define OBCA_PROF(i) do { if (M::PROF_CYCLES && threadIdx.x == 0) { long long t_ = clock64(); S.prof[i] += t_ - S.tmark; S.tmark = t_; } } while (0)
#else
#define OBCA_PROF_START()
#define OBCA_PROF(i)
#define OBCA_FOR_STAGES(k, ns) for (int k = 0; k < (ns); ++k)
#define OBCA_FOR_ITEMS(i, n) for (int i = 0; i < (n); ++i)
#define OBCA_SYNC()
#define OBCA_SERIAL
#endif

namespace obca {

// Problem description, options and workspace layout as seen by the per-stage functions.  On the device they live in
// __constant__ memory (set by the host before every launch, stream-ordered): every workspace access WA(name, k) then
// takes its array offset as an immediate constant-bank operand instead of a load from the context struct in local
// memory followed by a dependent address computation.  The host emulation reads them through the context.
#if defined(__CUDA_ARCH__)
#define CTX_P(C) c_pkP
#define CTX_O(C) c_pkO
#define CTX_L(C) c_pkL
#else
#define CTX_P(C) (*(C).P)
#define CTX_O(C) (*(C).O)
#define CTX_L(C) ((C).L)
#endif

// ---- per-stage partial results that are reduced over the stages of one problem ----
struct EvalPart {   // KKT-error / merit pieces
  double e_dual, e_pr, cmax, cmin, sy, sz, th, phi, rt, f;
  int ok;
};
struct StepPart { double apr, adu, dphi; };
struct MeritPart { double th, phi; };
OBCA_HD void part_init(EvalPart& p) { p.e_dual = 0; p.e_pr = 0; p.cmax = 0; p.cmin = 1e300; p.sy = 0; p.sz = 0; p.th = 0; p.phi = 0; p.rt = 0; p.f = 0; p.ok = 1; }
OBCA_HD void part_init(StepPart& p) { p.apr = 1.0; p.adu = 1.0; p.dphi = 0.0; }
OBCA_HD void part_init(MeritPart& p) { p.th = 0.0; p.phi = 0.0; }
OBCA_HD void part_merge(EvalPart& a, const EvalPart& b) {
  a.e_dual = dmax(a.e_dual, b.e_dual); a.e_pr = dmax(a.e_pr, b.e_pr); a.cmax = dmax(a.cmax, b.cmax); a.cmin = dmin_(a.cmin, b.cmin);
  a.sy += b.sy; a.sz += b.sz; a.th += b.th; a.phi += b.phi; a.rt += b.rt; a.f += b.f; a.ok &= b.ok;
}
OBCA_HD void part_merge(StepPart& a, const StepPart& b) { a.apr = dmin_(a.apr, b.apr); a.adu = dmin_(a.adu, b.adu); a.dphi += b.dphi; }
OBCA_HD void part_merge(MeritPart& a, const MeritPart& b) { a.th += b.th; a.phi += b.phi; }
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ EvalPart part_shfl(const EvalPart& p, int off) {
  EvalPart o;
  o.e_dual = __shfl_down_sync(0xffffffffu, p.e_dual, off); o.e_pr = __shfl_down_sync(0xffffffffu, p.e_pr, off);
  o.cmax = __shfl_down_sync(0xffffffffu, p.cmax, off); o.cmin = __shfl_down_sync(0xffffffffu, p.cmin, off);
  o.sy = __shfl_down_sync(0xffffffffu, p.sy, off); o.sz = __shfl_down_sync(0xffffffffu, p.sz, off);
  o.th = __shfl_down_sync(0xffffffffu, p.th, off); o.phi = __shfl_down_sync(0xffffffffu, p.phi, off);
  o.rt = __shfl_down_sync(0xffffffffu, p.rt, off); o.f = __shfl_down_sync(0xffffffffu, p.f, off);
  o.ok = __shfl_down_sync(0xffffffffu, p.ok, off);
  return o;
}
__device__ __forceinline__ StepPart part_shfl(const StepPart& p, int off) {
  StepPart o;
  o.apr = __shfl_down_sync(0xffffffffu, p.apr, off); o.adu = __shfl_down_sync(0xffffffffu, p.adu, off);
  o.dphi = __shfl_down_sync(0xffffffffu, p.dphi, off);
  return o;
}
__device__ __forceinline__ MeritPart part_shfl(const MeritPart& p, int off) {
  MeritPart o;
  o.th = __shfl_down_sync(0xffffffffu, p.th, off); o.phi = __shfl_down_sync(0xffffffffu, p.phi, off);
  return o;
}
// deterministic block reduction (fixed shuffle tree, then warp 0..3 in order); result valid in thread 0.
// Contains one __syncthreads().  `scratch`: shared memory, >= 4 * sizeof(EvalPart) bytes.
template <typename T>
__device__ __forceinline__ void block_reduce(T& v, void* scratch) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { T o = part_shfl(v, off); part_merge(v, o); }
  T* sc = reinterpret_cast<T*>(scratch);
  if ((threadIdx.x & 31) == 0) sc[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < (int)((blockDim.x + 31) >> 5); ++w) part_merge(v, sc[w]);
}
// the same, merging only the first nw warps of the block: a problem that needs fewer warps than its CTA has merges only its
// own (the surplus warps hold identities, but -0.0 + 0.0 = +0.0, so merging them could change the sign of a zero sum)
template <typename T>
__device__ __forceinline__ void block_reduce_warps(T& v, void* scratch, int nw) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) { T o = part_shfl(v, off); part_merge(v, o); }
  T* sc = reinterpret_cast<T*>(scratch);
  if ((threadIdx.x & 31) == 0) sc[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    for (int w = 1; w < nw; ++w) part_merge(v, sc[w]);
}
#define OBCA_REDUCE(v) M::reduce(v, C)      // IpmDriver<M>: the model's own block reduction
#else
#define OBCA_REDUCE(v)
#endif

// ---- what one (stage, obstacle) OBCA block contributes to its stage (K1).  The blocks are evaluated by the "item" pass of
//      an evaluation (one thread per (obstacle, stage) pair); the 12 doubles the stage assembly needs (Schur complement,
//      gradient, Lagrangian-gradient rows of the pose) are handed over through the stage's own slot in shared memory for
//      the first HO_SLOT_OB obstacles and through the workspace rows HO for the others, the KKT-error / merit partials are
//      merged into the thread's running EvalPart ----
struct BlockOut {
  double Sxx[6], rx3[3];   // Schur complement and gradient on the pose (X, Y, psi)      (assembly)
  double gx[3];            // the block's rows of the Lagrangian gradient on the pose    (errors)
  double e_dual, e_pr, cmax, cmin, sum_y, sum_z, th, lsum, fobj;   // KKT-error / merit partials; lsum = sum of log(gap)
  int ok;                  // 1: every local pivot had the sign required for inertia (n, m, 0)
};
constexpr int HO_N = 12;   // doubles per block handed over: Sxx 6 | rx3 3 | gx 3 (slot offset HO_N * j, or rows HO + HO_N * (j - HO_SLOT_OB))
constexpr int HO_SLOT_OB = 6;   // obstacles whose hand-over fits in a stage slot: HO_N * HO_SLOT_OB = 72 <= RSTRIDE = 82

// ---- workspace layout: every entry is an array of NSP doubles indexed by stage ----
struct PkLay {
  int NSP;
  // iterate
  int X, Y, PS, VL, DE, AC, LAM, MU, SL;
  int ZXL, ZXU, ZYL, ZYU, ZVL, ZVU, ZDL, ZDU, ZAL, ZAU, ZLAM, ZMU;
  int PI, YN, YR;
  int SD, VD, SN, VN, RS, RVL, RVU;
  // step
  int dX, dY, dPS, dVL, dDE, dAC, dLAM, dMU, dSL;
  int PIn, YNn, YRn, dSD, dSN, dRS;
  // KKT workspace
  int LF;
  int nfac;
  int HO;      // hand-over of the item pass for obstacles j >= HO_SLOT_OB: HO_N rows each (none with nOb <= HO_SLOT_OB)
  int total;
};

#if defined(__CUDACC__)
__constant__ ParkProblem c_pkP;
__constant__ IpmOpts c_pkO;
__constant__ PkLay c_pkL;
#endif

inline PkLay make_layout(const ParkProblem& P, int nfac) {
  PkLay L;
  const int NS = P.N + 1;      // the batch's horizon (the largest of a mixed batch): shorter problems leave rows unused
  L.NSP = (NS + 1) & ~1;      // row stride: even, so that every row starts on a 16-byte boundary (bulk copies)
  int c = 0;
  auto take = [&](int n) { int o = c; c += n; return o; };
  L.X = take(1); L.Y = take(1); L.PS = take(1); L.VL = take(1); L.DE = take(1); L.AC = take(1);
  L.LAM = take(P.V); L.MU = take(4 * P.nOb); L.SL = take(P.nOb);
  L.ZXL = take(1); L.ZXU = take(1); L.ZYL = take(1); L.ZYU = take(1); L.ZVL = take(1); L.ZVU = take(1);
  L.ZDL = take(1); L.ZDU = take(1); L.ZAL = take(1); L.ZAU = take(1);
  L.ZLAM = take(P.V); L.ZMU = take(4 * P.nOb);
  L.PI = take(4); L.YN = take(P.nOb); L.YR = take(2 * P.nOb);
  L.SD = take(P.nOb); L.VD = take(P.nOb); L.SN = take(P.nOb); L.VN = take(P.nOb);
  L.RS = take(1); L.RVL = take(1); L.RVU = take(1);
  L.dX = take(1); L.dY = take(1); L.dPS = take(1); L.dVL = take(1); L.dDE = take(1); L.dAC = take(1);
  L.dLAM = take(P.V); L.dMU = take(4 * P.nOb); L.dSL = take(P.nOb);
  L.PIn = take(4); L.YNn = take(P.nOb); L.YRn = take(2 * P.nOb);
  L.dSD = take(P.nOb); L.dSN = take(P.nOb); L.dRS = take(1);
  L.nfac = nfac;
  L.LF = take(P.nOb * nfac);
  L.HO = take(HO_N * (P.nOb > HO_SLOT_OB ? P.nOb - HO_SLOT_OB : 0));
  L.total = c;
  return L;
}

// ---- per-stage slot of the KKT solve (shared memory on the device): RSTRIDE doubles per stage ----
//   after stage_eval(k):   [RQ..] Q (45, packed 9x9) | [Rq..] q (9) | [RDYN..] dynamics Jacobian (20) | [RR4..] residual (4)
//   after the backward sweep passed stage k:  [RK..] gain K (2x7) + feed-forward (2)  and, in slot k+1,
//                                             [RPP..] rows 0..3 of P_{k+1} (4x7) + p_{k+1}[0..3]  (consumed Q/q space)
// 82 doubles = 656 bytes: a multiple of 16, so that the whole slot array of a problem leaves shared memory in ONE bulk
// copy (cp.async.bulk) and the sweep kernel streams single slots back with bulk copies; 82 = 2 mod 4 costs a 2-way bank
// conflict on the thread-per-stage accesses (an odd stride would be conflict-free but misaligns every second slot).
constexpr int RSTRIDE = 82;
static_assert(HO_N * HO_SLOT_OB <= RSTRIDE, "the hand-over of the first HO_SLOT_OB obstacles must fit in a stage slot");
constexpr int RQ = 0, Rq = 45, RDYN = 54, RR4 = 74;
constexpr int RK = 0, RPP = 16, Rpp = 44;   // RPP: rows 0..3 of P_{k+1}, row-major 4x7;  Rpp: p_{k+1}[0..3]

// where the solve of a problem stands between the phase functions of IpmDriver (ProbState::phase)
enum { PH_INIT = 0, PH_EVAL = 1, PH_EVAL2 = 2, PH_REASM = 3, PH_KKT = 4, PH_RECOVER = 5, PH_END = 6, PH_DONE = 7 };

// per-problem scalar state (shared memory on the device)
struct ProbState {
  double t, zTL, zTU, dt;           // time scale, its bound multipliers, its step
  double eN[4];                     // predicted end-point error of the step (stage N is pinned to xF)
  double eNq[12];                   // same, quadcopter model
  double mu, tau;
  double dw, dw_last;
  double theta_max, theta_min;
  double th_k, ph_k, dphi, f_k;
  double e0, e_dual, e_pr, e_cmax, e_cmin, sum_y, sum_z, rz_t;
  double a_pr, a_du, alpha, a_min;
  double th_t, ph_t;
  int nfilt;
  double filt_th[64], filt_ph[64];
  int status;     // 1 converged, 0 running / max_iter, -1 line-search failure, -2 inertia failure
  int iters;
  int flag;       // generic broadcast flag
  int ok;
  int n_fact;     // factorisations
  int n_kick;     // barrier kicks after line-search failures
  long long prof[8];   // device cycle counters per phase: eval, kkt, recover, merit, update, serial, n_merit, n_eval
  long long tmark;
  // state machine of IpmDriver's phase functions (between kernels in the parking rounds, obca_phased.cuh)
  int phase;        // PH_* above
  int it;           // iteration counter of the current attempt
  int attempt;      // 0: from the warm start, 1: the reference's second solve(m) from the last iterate
  int first;        // theta_max / theta_min not yet initialised for this attempt
  int iters_total;  // iterations of the finished attempts
  int N;            // horizon of this problem (set when the problem is picked up fresh; read by the sweep kernel)
};

// a problem picked up fresh: first attempt from the warm start, profile counters zeroed
OBCA_HD void state_fresh(ProbState& S, int N) {
  OBCA_SERIAL {
    S.N = N;
    S.phase = PH_INIT; S.attempt = 0; S.iters_total = 0; S.it = 0; S.first = 1; S.status = 0; S.iters = 0;
    S.t = 1.0; S.e0 = 0.0; S.ok = 0; S.flag = 0;
    for (int i = 0; i < 8; ++i) S.prof[i] = 0;
  }
}

struct PkInputs {
  const double* x0;    // 4
  const double* xF;    // 4
  const double* rx;    // NS
  const double* ry;
  const double* ryaw;
  const double* xWS;   // (N+1) x 4 column-major  (ParkingSignedDist.jl:216: setvalue(x, xWS'))
  int ldx;             // leading dimension (rows) of xWS
  const double* uWS;   // rows x 2 column-major, rows >= N (:217)
  int ldu;
  const double* lWS;   // (N+1) x V column-major (:221), leading dimension ldx (laid out like xWS)
  const double* nWS;   // (N+1) x 4nOb column-major (:222), leading dimension ldx
};

// outputs of one problem, in the reference's return shapes (ParkingSignedDist.jl:302-313), column-major
struct PkOutputs {
  double* xp;      // 4 x (N+1)
  double* up;      // 2 x N
  double* ts;      // N+1   (timeScalep; ones if fixTime, :304-308)
  double* lp;      // V x (N+1)
  double* np;      // 4nOb x (N+1)
  double* sl;      // nOb x (N+1)  (SD only; may be null)
  double* duals;   // optional (may be null): pi 4 x N, then y_rot 2nOb x (N+1), y_norm nOb x (N+1), vd nOb x (N+1)
};

struct PkCtx {
  const ParkProblem* P;   // P->N: the horizon the batch's arrays are laid out for (the largest of the batch)
  int N;                  // horizon of this problem (<= P->N): every loop over stages, items or the sweep runs to it
  const IpmOpts* O;
  PkLay L;
  double* W;
  double* Wd;      // rows dLAM .. dRS of the step (those the sweep does not write): W + dLAM * NSP, or shared memory
  double* ric;     // (N+1) x RSTRIDE slots
  const double* pp;  // where recover_stage finds rows 0..3 of P_{k+1} / p_{k+1}: the stage slots (shared memory in the
                     // persistent kernel and the emulation; the global slot array written by the sweep kernel in the rounds)
  void* red_scratch;   // device: shared-memory scratch of block_reduce
  double* tile;        // device: 7*9+7 doubles of shared memory for the warp-cooperative KKT sweep
  ProbState* S;
  PkInputs in;
#if !defined(__CUDACC__)
  PkCtx() : N(0) {}       // host (development emulation): a context built without a horizon solves at the layout's, P->N
#endif
};

// horizon of the problem of context C.  The device kernels always set C.N; on the host C.N = 0 stands for the layout's horizon.
#if defined(__CUDA_ARCH__)
#define CTX_N(C) ((C).N)
#else
#define CTX_N(C) ((C).N > 0 ? (C).N : (C).P->N)
#endif

// The context lives in shared memory and is passed by reference: after every store through a double* the compiler has to
// assume that C.W / C.ric / ... changed and reloads them.  Functions that use the accessors below therefore start with
// OBCA_LOCALS(C), which copies the base pointers into locals (registers) once.
#if defined(__CUDA_ARCH__)
// the workspace is global memory and the stage slots are shared memory in every kernel: with the address space known the
// compiler emits LDG / STG / LDS / STS (32-bit shared addresses) instead of generic accesses.  Wd and pp are shared in some
// kernels and global in others and stay generic.
#define OBCA_ASSUME_SPACES() __builtin_assume(__isGlobal(W_)); __builtin_assume(__isShared(ric_))
#else
#define OBCA_ASSUME_SPACES() (void)0
#endif
#define OBCA_LOCALS(C)                                                                                              \
  double* const W_ = (C).W; double* const Wd_ = (C).Wd; double* const ric_ = (C).ric; const double* const pp_ = (C).pp; \
  OBCA_ASSUME_SPACES();                                                                                             \
  (void)W_; (void)Wd_; (void)ric_; (void)pp_
#define WA(name, k) (W_[(size_t)(CTX_L(C).name) * CTX_L(C).NSP + (k)])
#define WV(name, i, k) (W_[(size_t)(CTX_L(C).name + (i)) * CTX_L(C).NSP + (k)])
// step rows that live in the step buffer (dLAM, dMU, dSL, PIn, YNn, YRn, dSD, dSN, dRS: contiguous in the layout)
#define WD(name, k) (Wd_[(size_t)(CTX_L(C).name - CTX_L(C).dLAM) * CTX_L(C).NSP + (k)])
#define WDV(name, i, k) (Wd_[(size_t)(CTX_L(C).name - CTX_L(C).dLAM + (i)) * CTX_L(C).NSP + (k)])
#define RIC(off, k) (ric_[(k) * RSTRIDE + (off)])
#define PPV(off, k) (pp_[(size_t)(k) * RSTRIDE + (off)])

OBCA_HD double push_lo(double x, double lo, double hi, double k1, double k2) {
  const double pl = dmin_(k1 * dmax(1.0, dabs(lo)), k2 * (hi - lo));
  const double pu = dmin_(k1 * dmax(1.0, dabs(hi)), k2 * (hi - lo));
  x = dmax(x, lo + pl);
  x = dmin_(x, hi - pu);
  return x;
}


template <int VM, bool SDV>
struct ParkSolver {
  typedef LocalDims<VM, SDV> LD;

  // ---------------------------------------------------------------------------------------------------
  // load rows / variables of block (k, j), optionally at the trial point  z + alpha dz
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD static void load_rows(const PkCtx& C, int j, ObsRows<VM>& R) {
    const ParkProblem& P = CTX_P(C);
    R.v = P.vOb[j];
#pragma unroll
    for (int i = 0; i < VM; ++i) {
      const bool on = i < R.v;
      const int r = P.voff[j] + (on ? i : 0);
      R.a1[i] = on ? P.A[r][0] : 0.0;
      R.a2[i] = on ? P.A[r][1] : 0.0;
      R.bb[i] = on ? P.b[r] : 0.0;
    }
  }
  OBCA_HD static void load_vars(const PkCtx& C, int k, int j, const ObsRows<VM>& R, ObsVars<VM>& Q) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
#pragma unroll
    for (int i = 0; i < VM; ++i) {
      const bool on = i < R.v;
      Q.lam[i] = on ? WV(LAM, P.voff[j] + i, k) : 1.0;
      Q.zlam[i] = on ? WV(ZLAM, P.voff[j] + i, k) : 0.0;
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) { Q.mu[m] = WV(MU, 4 * j + m, k); Q.zmu[m] = WV(ZMU, 4 * j + m, k); }
    Q.sl = SDV ? WV(SL, j, k) : 0.0;
    Q.yn = SDV ? WV(YN, j, k) : 0.0;
    Q.yr1 = WV(YR, 2 * j, k); Q.yr2 = WV(YR, 2 * j + 1, k);
    Q.sd = WV(SD, j, k); Q.vd = WV(VD, j, k);
    Q.sn = SDV ? 0.0 : WV(SN, j, k);
    Q.vn = SDV ? 0.0 : WV(VN, j, k);
  }

  // ---------------------------------------------------------------------------------------------------
  // P0: initial point (ParkingSignedDist.jl:213-222) + Ipopt's projection into the bounds, slacks, multipliers
  // ---------------------------------------------------------------------------------------------------
  // restart != 0: re-initialise from the current iterate (the reference's second solve(m) restarts Ipopt from
  // JuMP's stored primal values, ParkingSignedDist.jl:256-263) instead of from the warm-start inputs.
  OBCA_HD_NI static void init_stage(const PkCtx& C, int k, int restart) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const IpmOpts& O = CTX_O(C);
    const int N = CTX_N(C);
    const bool pose_free = (k >= 1 && k <= N - 1);
    double X, Y, ps, v;
    if (restart) { X = WA(X, k); Y = WA(Y, k); ps = WA(PS, k); v = WA(VL, k); }
    else {
      X = C.in.xWS[0 * C.in.ldx + k]; Y = C.in.xWS[1 * C.in.ldx + k];
      ps = C.in.xWS[2 * C.in.ldx + k]; v = C.in.xWS[3 * C.in.ldx + k];
    }
    if (k == 0) { X = C.in.x0[0]; Y = C.in.x0[1]; ps = C.in.x0[2]; v = C.in.x0[3]; }
    if (k == N) { X = C.in.xF[0]; Y = C.in.xF[1]; ps = C.in.xF[2]; v = C.in.xF[3]; }
    if (pose_free) {
      X = push_lo(X, P.xyb[0], P.xyb[1], O.kappa1, O.kappa2);
      Y = push_lo(Y, P.xyb[2], P.xyb[3], O.kappa1, O.kappa2);
      v = push_lo(v, -1.0, 2.0, O.kappa1, O.kappa2);
    }
    WA(X, k) = X; WA(Y, k) = Y; WA(PS, k) = ps; WA(VL, k) = v;
    WA(ZXL, k) = 1.0; WA(ZXU, k) = 1.0; WA(ZYL, k) = 1.0; WA(ZYU, k) = 1.0; WA(ZVL, k) = 1.0; WA(ZVU, k) = 1.0;
    double de = 0.0, ac = 0.0;
    if (k < N) {
      de = push_lo(restart ? WA(DE, k) : C.in.uWS[0 * C.in.ldu + k], -0.6, 0.6, O.kappa1, O.kappa2);
      ac = push_lo(restart ? WA(AC, k) : C.in.uWS[1 * C.in.ldu + k], -0.4, 0.4, O.kappa1, O.kappa2);
    }
    WA(DE, k) = de; WA(AC, k) = ac;
    WA(ZDL, k) = 1.0; WA(ZDU, k) = 1.0; WA(ZAL, k) = 1.0; WA(ZAU, k) = 1.0;
#pragma unroll
    for (int i = 0; i < 4; ++i) WV(PI, i, k) = 0.0;
    const double lpush = O.kappa1;   // lower bound 0: kappa1 * max(1, |0|)
    for (int r = 0; r < P.V; ++r) {
      WV(LAM, r, k) = dmax(restart ? WV(LAM, r, k) : C.in.lWS[(size_t)r * C.in.ldx + k], lpush);
      WV(ZLAM, r, k) = 1.0;
    }
    for (int r = 0; r < 4 * P.nOb; ++r) {
      WV(MU, r, k) = dmax(restart ? WV(MU, r, k) : C.in.nWS[(size_t)r * C.in.ldx + k], lpush);
      WV(ZMU, r, k) = 1.0;
    }
    for (int j = 0; j < P.nOb; ++j) {
      if (SDV) { if (!restart) WV(SL, j, k) = 0.0; WV(YN, j, k) = 0.0; }
      WV(YR, 2 * j, k) = 0.0; WV(YR, 2 * j + 1, k) = 0.0;
    }
  }
  // slacks need the pushed primal point of the neighbours -> separate phase
  OBCA_HD_NI static void init_slacks(const PkCtx& C, int k) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const IpmOpts& O = CTX_O(C);
    const int N = CTX_N(C);
    const double X = WA(X, k), Y = WA(Y, k), ps = WA(PS, k);
    double s, c;
    sincos(ps, &s, &c);
    for (int j = 0; j < P.nOb; ++j) {
      ObsRows<VM> R; ObsVars<VM> Q; ObsGeom<VM> G;
      load_rows(C, j, R);
      load_vars(C, k, j, R, Q);
      Q.sd = 0.0; Q.sn = 0.0;
      obs_geom<VM, SDV>(P, X, Y, c, s, R, Q, G);
      WV(SD, j, k) = dmax(G.gd, P.dmin + O.kappa1 * dmax(1.0, dabs(P.dmin)));
      WV(VD, j, k) = 1.0;
      if (!SDV) { WV(SN, j, k) = dmin_(G.pp, 1.0 - O.kappa1); WV(VN, j, k) = 1.0; }
    }
    if (k < N) {
      const double h = (P.fix_time ? 1.0 : C.S->t) * P.Ts;
      const double wd = k > 0 ? WA(DE, k - 1) : 0.0;
      const double gr = (wd - WA(DE, k)) / h;
      WA(RS, k) = push_lo(gr, -0.6, 0.6, O.kappa1, O.kappa2);
      WA(RVL, k) = 1.0; WA(RVU, k) = 1.0;
    }
  }

  // ---------------------------------------------------------------------------------------------------
  // K1, one (stage k, obstacle j) block: residuals / KKT-error partials (do_err) and the condensation of the block onto
  // the stage pose with the local factor stored in the workspace (do_asm).  (X, Y, cs_, sn_) = pose of the stage.
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD static void block_eval(const PkCtx& C, int k, int j, double X, double Y, double cs_, double sn_, double mu_b,
                                 double dw, bool do_err, bool do_asm, BlockOut& B) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    double e_dual = 0.0, e_pr = 0.0, cmax = 0.0, cmin = 1e300, sum_y = 0.0, sum_z = 0.0, th = 0.0, fobj = 0.0;
    LogAcc lacc;
    B.gx[0] = B.gx[1] = B.gx[2] = 0.0;
    B.ok = 1;
#pragma unroll
    for (int i = 0; i < 6; ++i) B.Sxx[i] = 0.0;
    B.rx3[0] = B.rx3[1] = B.rx3[2] = 0.0;
    {
      ObsRows<VM> R; ObsVars<VM> Qv; ObsGeom<VM> G;
      load_rows(C, j, R);
      load_vars(C, k, j, R, Qv);
      obs_geom<VM, SDV>(P, X, Y, cs_, sn_, R, Qv, G);
      if (do_err) {
        double rl[VM], rm[4], rs_, gx[3];
        obs_lagr_grad<VM, SDV>(P, R, Qv, G, rl, rm, rs_, gx);
        B.gx[0] = gx[0]; B.gx[1] = gx[1]; B.gx[2] = gx[2];
#pragma unroll
        for (int i = 0; i < VM; ++i) {
          if (i < R.v) {
            e_dual = dmax(e_dual, dabs(rl[i]));
            const double cp = Qv.lam[i] * Qv.zlam[i];
            cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
            sum_z += Qv.zlam[i];
            lacc.add(Qv.lam[i]);
          }
        }
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          e_dual = dmax(e_dual, dabs(rm[m]));
          const double cp = Qv.mu[m] * Qv.zmu[m];
          cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
          sum_z += Qv.zmu[m];
          lacc.add(Qv.mu[m]);
        }
        if (SDV) { e_dual = dmax(e_dual, dabs(rs_)); fobj += 1e2 * Qv.sl + 1e4 * Qv.sl * Qv.sl; }
        e_pr = dmax(e_pr, dmax(dmax(dabs(G.cn), dabs(G.cd)), dmax(dabs(G.cr1), dabs(G.cr2))));
        th += dabs(G.cn) + dabs(G.cd) + dabs(G.cr1) + dabs(G.cr2);
        sum_y += dabs(Qv.yr1) + dabs(Qv.yr2) + Qv.vd + (SDV ? dabs(Qv.yn) : Qv.vn);
        sum_z += Qv.vd + (SDV ? 0.0 : Qv.vn);
        {
          const double cp = (Qv.sd - P.dmin) * Qv.vd;
          cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
          lacc.add(Qv.sd - P.dmin);
        }
        if (!SDV) {
          const double cp = (1.0 - Qv.sn) * Qv.vn;
          cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
          lacc.add(1.0 - Qv.sn);
        }
      } else if (SDV) {
        fobj += 1e2 * Qv.sl + 1e4 * Qv.sl * Qv.sl;
      }
      if (do_asm) {
        const int piv = choose_pivot<VM, SDV>(R, G);
        if (piv != 0) {
          swap_rows(R, Qv, piv);
          obs_geom<VM, SDV>(P, X, Y, cs_, sn_, R, Qv, G);
        }
        B.ok = obs_condense<VM, SDV>(P, R, Qv, G, mu_b, dw, CTX_O(C).dc, B.Sxx, B.rx3, &WV(LF, j * CTX_L(C).nfac, k), CTX_L(C).NSP);
      }
    }
    B.e_dual = e_dual; B.e_pr = e_pr; B.cmax = cmax; B.cmin = cmin; B.sum_y = sum_y; B.sum_z = sum_z; B.th = th;
    B.lsum = do_err ? lacc.total() : 0.0; B.fobj = fobj;
  }
  // ---------------------------------------------------------------------------------------------------
  // K1, item pass: item i = (obstacle j, stage k), i = j * (N+1) + k, so that consecutive threads work on consecutive
  // stages (contiguous slices of every stacked array).  Evaluates the block (block_eval), hands the 12 doubles the stage
  // assembly needs over in the stage's own slot (offset HO_N * j; the stage pass reads them before it zeroes its Q / q
  // area) or, for j >= HO_SLOT_OB, in the workspace rows HO, and merges the block's KKT-error / merit partials into the
  // thread's running EvalPart.
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD_NI static void block_item_eval(const PkCtx& C, int i, bool do_err, EvalPart& acc) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int NS = CTX_N(C) + 1;
    const int j = i / NS, k = i - j * NS;
    const double mu_b = S.mu;
    const double X = WA(X, k), Y = WA(Y, k), ps = WA(PS, k);
    double sn_, cs_;
    sincos(ps, &sn_, &cs_);
    BlockOut B;
    block_eval(C, k, j, X, Y, cs_, sn_, mu_b, S.dw, do_err, true, B);
    if (j < HO_SLOT_OB) {
      double* const h = &RIC(HO_N * j, k);
#pragma unroll
      for (int e = 0; e < 6; ++e) h[e] = B.Sxx[e];
#pragma unroll
      for (int e = 0; e < 3; ++e) { h[6 + e] = B.rx3[e]; h[9 + e] = B.gx[e]; }
    } else {
      const int r = HO_N * (j - HO_SLOT_OB);
#pragma unroll
      for (int e = 0; e < 6; ++e) WV(HO, r + e, k) = B.Sxx[e];
#pragma unroll
      for (int e = 0; e < 3; ++e) { WV(HO, r + 6 + e, k) = B.rx3[e]; WV(HO, r + 9 + e, k) = B.gx[e]; }
    }
    acc.ok &= B.ok;
    acc.f += B.fobj;
    if (do_err) {
      acc.e_dual = dmax(acc.e_dual, B.e_dual); acc.e_pr = dmax(acc.e_pr, B.e_pr);
      acc.cmax = dmax(acc.cmax, B.cmax); acc.cmin = dmin_(acc.cmin, B.cmin);
      acc.sy += B.sum_y; acc.sz += B.sum_z; acc.th += B.th;
      acc.phi += B.fobj - mu_b * B.lsum;
    }
  }

  // ---------------------------------------------------------------------------------------------------
  // K1 with more than HO_SLOT_OB obstacles, between the item and the stage pass: sums the hand-overs of stage k over all
  // obstacles in index order (slot offsets of obstacles 0..5, then the workspace rows HO), stores the sum in obstacle 0's place
  // of the slot and zeroes the places of obstacles 1..5.  stage_eval's sum over the slot then gives the same bits (the sum
  // starts from +0.0, so it is never -0.0, and adding +0.0 leaves it unchanged), and stage_eval itself stays as small as
  // for up to six obstacles.
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD_NI static void fold_far_handover(const PkCtx& C, int k) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    double hs[HO_N];
#pragma unroll
    for (int e = 0; e < HO_N; ++e) hs[e] = 0.0;
    for (int j = 0; j < HO_SLOT_OB; ++j) {
#pragma unroll
      for (int e = 0; e < HO_N; ++e) hs[e] += RIC(HO_N * j + e, k);
    }
    for (int j = HO_SLOT_OB; j < P.nOb; ++j) {
#pragma unroll
      for (int e = 0; e < HO_N; ++e) hs[e] += WV(HO, HO_N * (j - HO_SLOT_OB) + e, k);
    }
#pragma unroll
    for (int e = 0; e < HO_N; ++e) RIC(e, k) = hs[e];
    for (int i = HO_N; i < HO_N * HO_SLOT_OB; ++i) RIC(i, k) = 0.0;
  }

  // ---------------------------------------------------------------------------------------------------
  // P1 (K1): fused evaluation at the current iterate.
  //   do_err: KKT-error / merit partials into RED;   do_asm: stage model Q, q, dynamics, local factors.
  // ---------------------------------------------------------------------------------------------------
  // stage pass of an evaluation: everything of stage k that is not an obstacle block (state objective and bounds, controls,
  // input-rate terms, steering-rate row, dynamics with second derivatives, time scale) + the sums of the block hand-overs
  OBCA_HD_NI static void stage_eval(const PkCtx& C, int k, bool do_err, bool do_asm, EvalPart& out) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int N = CTX_N(C);
    const bool fix = P.fix_time != 0;
    const double mu_b = S.mu, dw = S.dw;
    const bool pose_free = (k >= 1 && k <= N - 1);
    const bool has_u = k < N;
    const double t = fix ? 1.0 : S.t;
    const double X = WA(X, k), Y = WA(Y, k), ps = WA(PS, k), v = WA(VL, k);

    // hand-overs of the item pass (sum over the obstacles in index order), read before the slot is reused for Q / q
    double hs[HO_N];
#pragma unroll
    for (int e = 0; e < HO_N; ++e) hs[e] = 0.0;
    const int n_slot = P.nOb < HO_SLOT_OB ? P.nOb : HO_SLOT_OB;      // more obstacles: folded into slot 0 (fold_far_handover)
    for (int j = 0; j < n_slot; ++j) {
#pragma unroll
      for (int e = 0; e < HO_N; ++e) hs[e] += RIC(HO_N * j + e, k);
    }
    // the stage model (packed 9x9 Q, q) is accumulated directly in the stage slot (shared memory on the device)
#pragma unroll
    for (int i = 0; i < NQ + NYV; ++i) RIC(RQ + i, k) = 0.0;
#pragma unroll
    for (int i = RR4 + 4; i < RSTRIDE; ++i) RIC(i, k) = 0.0;      // padding of the slot (it is copied out as a whole)
    double e_dual = 0.0, e_pr = 0.0, cmax = 0.0, cmin = 1e300, sum_y = 0.0, sum_z = 0.0, th = 0.0, phi = 0.0, fobj = 0.0;
    double rz_t = 0.0;
    int ok = 1;
    LogAcc lacc;   // barrier terms: phi -= mu * sum(log gap)

    // ---- (C) obstacle blocks: Schur complements / gradients on the pose, Lagrangian-gradient rows ----
    double rzX = hs[9], rzY = hs[10], rzP = hs[11], rzV = 0.0;
    if (do_asm && pose_free) {
      RIC(RQ + sym_idx<NYV>(IX, IX), k) = hs[0]; RIC(RQ + sym_idx<NYV>(IX, IY), k) = hs[1]; RIC(RQ + sym_idx<NYV>(IX, IP), k) = hs[2];
      RIC(RQ + sym_idx<NYV>(IY, IY), k) = hs[3]; RIC(RQ + sym_idx<NYV>(IY, IP), k) = hs[4]; RIC(RQ + sym_idx<NYV>(IP, IP), k) = hs[5];
      RIC(Rq + IX, k) = hs[6]; RIC(Rq + IY, k) = hs[7]; RIC(Rq + IP, k) = hs[8];
    }
    // ---- (A) state objective + bounds ----
    {
      const double ex = X - C.in.rx[k], ey = Y - C.in.ry[k], ep = ps - C.in.ryaw[k];
      fobj += 1e-4 * v * v + 1e-3 * ex * ex + 1e-3 * ey * ey + P.w_yaw * ep * ep;
      if (pose_free) {
        const double gX = 2e-3 * ex, gY = 2e-3 * ey, gP = 2.0 * P.w_yaw * ep, gV = 2e-4 * v;
        const double aXl = X - P.xyb[0], aXu = P.xyb[1] - X, aYl = Y - P.xyb[2], aYu = P.xyb[3] - Y;
        const double aVl = v + 1.0, aVu = 2.0 - v;
        const double zXl = WA(ZXL, k), zXu = WA(ZXU, k), zYl = WA(ZYL, k), zYu = WA(ZYU, k), zVl = WA(ZVL, k), zVu = WA(ZVU, k);
        RIC(RQ + sym_idx<NYV>(IX, IX), k) += 2e-3 + zXl * rcp(aXl) + zXu * rcp(aXu) + dw;
        RIC(RQ + sym_idx<NYV>(IY, IY), k) += 2e-3 + zYl * rcp(aYl) + zYu * rcp(aYu) + dw;
        RIC(RQ + sym_idx<NYV>(IP, IP), k) += 2.0 * P.w_yaw + dw;
        RIC(RQ + sym_idx<NYV>(IV, IV), k) += 2e-4 + zVl * rcp(aVl) + zVu * rcp(aVu) + dw;
        RIC(Rq + IX, k) += gX - mu_b * rcp(aXl) + mu_b * rcp(aXu);
        RIC(Rq + IY, k) += gY - mu_b * rcp(aYl) + mu_b * rcp(aYu);
        RIC(Rq + IP, k) += gP;
        RIC(Rq + IV, k) += gV - mu_b * rcp(aVl) + mu_b * rcp(aVu);
        rzX += gX - zXl + zXu; rzY += gY - zYl + zYu; rzP += gP; rzV += gV - zVl + zVu;
        // multiplier of the dynamics row that produced x_k
        rzX += WV(PI, 0, k - 1); rzY += WV(PI, 1, k - 1); rzP += WV(PI, 2, k - 1); rzV += WV(PI, 3, k - 1);
        if (do_err) {
          const double c6[6] = {aXl * zXl, aXu * zXu, aYl * zYl, aYu * zYu, aVl * zVl, aVu * zVu};
#pragma unroll
          for (int i = 0; i < 6; ++i) { cmax = dmax(cmax, c6[i]); cmin = dmin_(cmin, c6[i]); }
          sum_z += zXl + zXu + zYl + zYu + zVl + zVu;
          lacc.add(aXl); lacc.add(aXu); lacc.add(aYl); lacc.add(aYu); lacc.add(aVl); lacc.add(aVu);
        }
      }
    }
    // ---- (B) controls, input-rate terms, steering-rate row, dynamics ----
    if (has_u) {
      DynOut dyn;
      double r4[4];
      const double de = WA(DE, k), ac = WA(AC, k);
      const double wd = k > 0 ? WA(DE, k - 1) : 0.0, wa = k > 0 ? WA(AC, k - 1) : 0.0;
      const double h = t * P.Ts, ih = rcp(h), ih2 = ih * ih, it = rcp(t);
      const double ed = de - wd, ea = ac - wa;
      const double T = 0.1 * (ed * ed + ea * ea) * ih2;
      fobj += 0.01 * de * de + P.w_a * ac * ac + T;
      const double gD = 0.02 * de + 0.2 * ed * ih2, gA = 2.0 * P.w_a * ac + 0.2 * ea * ih2;
      const double gWd = -0.2 * ed * ih2, gWa = -0.2 * ea * ih2;
      const double gT = fix ? 0.0 : -2.0 * T * it;
      const double aDl = de + 0.6, aDu = 0.6 - de, aAl = ac + 0.4, aAu = 0.4 - ac;
      const double zDl = WA(ZDL, k), zDu = WA(ZDU, k), zAl = WA(ZAL, k), zAu = WA(ZAU, k);
      RIC(RQ + sym_idx<NYV>(IDE, IDE), k) += 0.02 + 0.2 * ih2 + zDl * rcp(aDl) + zDu * rcp(aDu) + dw;
      RIC(RQ + sym_idx<NYV>(IAC, IAC), k) += 2.0 * P.w_a + 0.2 * ih2 + zAl * rcp(aAl) + zAu * rcp(aAu) + dw;
      RIC(RQ + sym_idx<NYV>(IWD, IWD), k) += 0.2 * ih2;
      RIC(RQ + sym_idx<NYV>(IWA, IWA), k) += 0.2 * ih2;
      RIC(RQ + sym_idx<NYV>(IWD, IDE), k) += -0.2 * ih2;
      RIC(RQ + sym_idx<NYV>(IWA, IAC), k) += -0.2 * ih2;
      if (!fix) {
        RIC(RQ + sym_idx<NYV>(IT, IDE), k) += -0.4 * ed * ih2 * it;
        RIC(RQ + sym_idx<NYV>(IT, IAC), k) += -0.4 * ea * ih2 * it;
        RIC(RQ + sym_idx<NYV>(IWD, IT), k) += 0.4 * ed * ih2 * it;
        RIC(RQ + sym_idx<NYV>(IWA, IT), k) += 0.4 * ea * ih2 * it;
        RIC(RQ + sym_idx<NYV>(IT, IT), k) += 6.0 * T * it * it;
      }
      // steering-rate row (ParkingSignedDist.jl:167-173):  -0.6 <= (wd - de)/(t Ts) <= 0.6
      const double gr = (wd - de) * ih;
      const double rs = WA(RS, k), rvl = WA(RVL, k), rvu = WA(RVU, k);
      const double yIr = rvu - rvl;
      const double gl = rs + 0.6, gu = 0.6 - rs;
      const double Sr = rvl * rcp(gl) + rvu * rcp(gu);
      const double cIr = gr - rs;
      const double yr0 = -mu_b * rcp(gl) + mu_b * rcp(gu) + Sr * cIr;
      const double jw = ih, jd = -ih, jt = fix ? 0.0 : -gr * it;
      RIC(RQ + sym_idx<NYV>(IWD, IWD), k) += Sr * jw * jw;
      RIC(RQ + sym_idx<NYV>(IWD, IDE), k) += Sr * jw * jd;
      RIC(RQ + sym_idx<NYV>(IDE, IDE), k) += Sr * jd * jd;
      if (!fix) {
        RIC(RQ + sym_idx<NYV>(IWD, IT), k) += Sr * jw * jt - yIr * ih * it;
        RIC(RQ + sym_idx<NYV>(IT, IDE), k) += Sr * jt * jd + yIr * ih * it;
        RIC(RQ + sym_idx<NYV>(IT, IT), k) += Sr * jt * jt + yIr * 2.0 * gr * it * it;
      }
      RIC(Rq + IWD, k) += gWd + jw * yr0;
      RIC(Rq + IWA, k) += gWa;
      RIC(Rq + IDE, k) += gD + jd * yr0 - mu_b * rcp(aDl) + mu_b * rcp(aDu);
      RIC(Rq + IAC, k) += gA - mu_b * rcp(aAl) + mu_b * rcp(aAu);
      RIC(Rq + IT, k) += gT + jt * yr0;
      // dynamics
      double pi[4], H5[15];
#pragma unroll
      for (int i = 0; i < 4; ++i) pi[i] = WV(PI, i, k);
      dyn_eval(P, X, Y, ps, v, de, ac, t, dyn, pi, H5);
      {
        int e = 0;
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
          for (int j = i; j < 5; ++j) RIC(RQ + sym_idx_any<NYV>(q5_to_y(i), q5_to_y(j)), k) += H5[e++];
      }
      double xn[4];
      if (k + 1 == N) { xn[0] = C.in.xF[0]; xn[1] = C.in.xF[1]; xn[2] = C.in.xF[2]; xn[3] = C.in.xF[3]; }
      else { xn[0] = WA(X, k + 1); xn[1] = WA(Y, k + 1); xn[2] = WA(PS, k + 1); xn[3] = WA(VL, k + 1); }
#pragma unroll
      for (int i = 0; i < 4; ++i) r4[i] = dyn.f[i] - xn[i];
      if (do_asm) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          RIC(RDYN + 5 * i + 0, k) = dyn.fx[i][0]; RIC(RDYN + 5 * i + 1, k) = dyn.fx[i][1]; RIC(RDYN + 5 * i + 2, k) = dyn.ft[i];
          RIC(RDYN + 5 * i + 3, k) = dyn.fu[i][0]; RIC(RDYN + 5 * i + 4, k) = dyn.fu[i][1];
          RIC(RR4 + i, k) = r4[i];
        }
      }
      // Lagrangian gradient: -A' pi on the pose rows
      if (pose_free) {
        rzX -= pi[0]; rzY -= pi[1];
        rzP -= pi[0] * dyn.fx[0][0] + pi[1] * dyn.fx[1][0] + pi[2] * dyn.fx[2][0] + pi[3] * dyn.fx[3][0];
        rzV -= pi[0] * dyn.fx[0][1] + pi[1] * dyn.fx[1][1] + pi[2] * dyn.fx[2][1] + pi[3] * dyn.fx[3][1];
      }
      if (do_err) {
        // rows of (de_k, a_k): own terms + the "previous control" role in stage k+1
        double rzD = gD + jd * yIr - zDl + zDu, rzA = gA - zAl + zAu;
#pragma unroll
        for (int i = 0; i < 4; ++i) { rzD -= pi[i] * dyn.fu[i][0]; rzA -= pi[i] * dyn.fu[i][1]; }
        if (k + 1 < N) {
          const double ed2 = WA(DE, k + 1) - de, ea2 = WA(AC, k + 1) - ac;
          rzD += -0.2 * ed2 * ih2 + (WA(RVU, k + 1) - WA(RVL, k + 1)) * ih;
          rzA += -0.2 * ea2 * ih2;
        }
        e_dual = dmax(e_dual, dmax(dabs(rzD), dabs(rzA)));
        if (!fix) {
          rz_t += gT + jt * yIr;
#pragma unroll
          for (int i = 0; i < 4; ++i) rz_t -= pi[i] * dyn.ft[i];
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) { e_pr = dmax(e_pr, dabs(r4[i])); th += dabs(r4[i]); sum_y += dabs(pi[i]); }
        e_pr = dmax(e_pr, dabs(cIr)); th += dabs(cIr);
        sum_y += dabs(yIr); sum_z += rvl + rvu + zDl + zDu + zAl + zAu;
        const double c6[6] = {aDl * zDl, aDu * zDu, aAl * zAl, aAu * zAu, gl * rvl, gu * rvu};
#pragma unroll
        for (int i = 0; i < 6; ++i) { cmax = dmax(cmax, c6[i]); cmin = dmin_(cmin, c6[i]); }
        lacc.add(aDl); lacc.add(aDu); lacc.add(aAl); lacc.add(aAu); lacc.add(gl); lacc.add(gu);
      }
    }
    // ---- (D) time-scale variable: objective (N+1)(0.5 t + t^2) (:89) and its (N+1) bound pairs ----
    if (k == 0 && !fix) {
      const double m = (double)(N + 1);
      const double gl = t - 0.8, gu = 1.2 - t;
      fobj += m * (0.5 * t + t * t);
      RIC(RQ + sym_idx<NYV>(IT, IT), k) += 2.0 * m + m * (S.zTL * rcp(gl) + S.zTU * rcp(gu)) + m * dw;   // N+1 copies of timeScale, each regularised
      RIC(Rq + IT, k) += m * (0.5 + 2.0 * t) + m * (-mu_b * rcp(gl) + mu_b * rcp(gu));
      if (do_err) {
        rz_t += m * (0.5 + 2.0 * t) - m * (S.zTL - S.zTU);
        cmax = dmax(cmax, dmax(gl * S.zTL, gu * S.zTU));
        cmin = dmin_(cmin, dmin_(gl * S.zTL, gu * S.zTU));
        sum_z += m * (S.zTL + S.zTU);
        phi -= m * mu_b * (log(gl) + log(gu));
      }
    }
    if (do_err) phi -= mu_b * lacc.total();
    if (do_err && pose_free) e_dual = dmax(e_dual, dmax(dmax(dabs(rzX), dabs(rzY)), dmax(dabs(rzP), dabs(rzV))));
    out.e_dual = e_dual; out.e_pr = e_pr; out.cmax = cmax; out.cmin = cmin; out.sy = sum_y; out.sz = sum_z;
    out.th = th; out.phi = phi + fobj; out.rt = rz_t; out.f = fobj; out.ok = ok;
  }

  // ---------------------------------------------------------------------------------------------------
  // K3: stage-banded KKT solve.  Backward Riccati sweep, root (dt), forward roll-out.  Serial per problem.
  //     returns 1 if every pivot is positive (KKT inertia (n, m, 0)).
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD static int kkt_solve(const PkCtx& C) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    ProbState& S = *C.S;
    const int N = CTX_N(C);
    const bool fix = P.fix_time != 0;
    constexpr int NP = NSV * (NSV + 1) / 2;
    double Pn[NP], pn[NSV];
#pragma unroll
    for (int i = 0; i < NP; ++i) Pn[i] = 0.0;
#pragma unroll
    for (int i = 0; i < NSV; ++i) pn[i] = 0.0;
    // terminal value: regularised end-point rows  x_N == xF  (ParkingSignedDist.jl:128-131)
    const double rho = 1.0 / CTX_O(C).dc;
#pragma unroll
    for (int i = 0; i < 4; ++i) { Pn[sym_idx<NSV>(i, i)] = rho; pn[i] = -WV(PI, i, N - 1); }
    int ok = 1;
    for (int k = N - 1; k >= 0; --k) {
      // P_{k+1}, p_{k+1} are needed by the forward sweep (multipliers)
#pragma unroll
      for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int l = 0; l < NSV; ++l) RIC(RPP + i * NSV + l, k + 1) = Pn[sym_idx_any<NSV>(i, l)];
        RIC(Rpp + i, k + 1) = pn[i];
      }
      DynOut d;
      double r4[4], Q[NQ], q[NYV];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        d.fx[i][0] = RIC(RDYN + 5 * i + 0, k); d.fx[i][1] = RIC(RDYN + 5 * i + 1, k); d.ft[i] = RIC(RDYN + 5 * i + 2, k);
        d.fu[i][0] = RIC(RDYN + 5 * i + 3, k); d.fu[i][1] = RIC(RDYN + 5 * i + 4, k);
        r4[i] = RIC(RR4 + i, k);
      }
#pragma unroll
      for (int e = 0; e < NQ; ++e) Q[e] = RIC(RQ + e, k);
#pragma unroll
      for (int e = 0; e < NYV; ++e) q[e] = RIC(Rq + e, k);
      double Pk[NP], pk[NSV];
      RicStage G;
      ok &= riccati_step(d, r4, Q, q, Pn, pn, Pk, pk, G);
#pragma unroll
      for (int j = 0; j < NSV; ++j) { RIC(RK + j, k) = G.K[0][j]; RIC(RK + NSV + j, k) = G.K[1][j]; }
      RIC(RK + 14, k) = G.kf[0]; RIC(RK + 15, k) = G.kf[1];
#pragma unroll
      for (int e = 0; e < NP; ++e) Pn[e] = Pk[e];
#pragma unroll
      for (int e = 0; e < NSV; ++e) pn[e] = pk[e];
    }
    return ok & kkt_root_forward(C, Pn[sym_idx<NSV>(IT, IT)], pn[IT]);
  }

  // root of the recursion (x_0, w_0 fixed; dt free if variable time) + forward roll-out of the primal step.
  // Light and strictly sequential: run by one thread.  The new multipliers of the dynamics rows are computed
  // afterwards, stage-parallel, in recover_stage().
  OBCA_HD static int kkt_root_forward(const PkCtx& C, double ptt, double pt) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    ProbState& S = *C.S;
    const int N = CTX_N(C);
    int ok = 1;
    double dt = 0.0;
    if (!P.fix_time) {
      if (!(ptt > 0.0)) { ok = 0; ptt = 1e300; }
      dt = -pt / ptt;
    }
    S.dt = dt;
    double s[NSV] = {0, 0, 0, 0, 0, 0, dt};
    for (int k = 0; k < N; ++k) {
      double u0 = RIC(RK + 14, k), u1 = RIC(RK + 15, k);
#pragma unroll
      for (int j = 0; j < NSV; ++j) { u0 += RIC(RK + j, k) * s[j]; u1 += RIC(RK + NSV + j, k) * s[j]; }
      WA(dDE, k) = u0; WA(dAC, k) = u1;
      double sn[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        sn[i] = RIC(RR4 + i, k) + RIC(RDYN + 5 * i + 0, k) * s[IP] + RIC(RDYN + 5 * i + 1, k) * s[IV] +
                RIC(RDYN + 5 * i + 2, k) * s[IT] + RIC(RDYN + 5 * i + 3, k) * u0 + RIC(RDYN + 5 * i + 4, k) * u1;
      }
      sn[0] += s[IX]; sn[1] += s[IY];
      if (k + 1 < N) { WA(dX, k + 1) = sn[0]; WA(dY, k + 1) = sn[1]; WA(dPS, k + 1) = sn[2]; WA(dVL, k + 1) = sn[3]; }
      else { S.eN[0] = sn[0]; S.eN[1] = sn[1]; S.eN[2] = sn[2]; S.eN[3] = sn[3]; }
      s[0] = sn[0]; s[1] = sn[1]; s[2] = sn[2]; s[3] = sn[3]; s[IWD] = u0; s[IWA] = u1;
    }
    WA(dX, 0) = 0.0; WA(dY, 0) = 0.0; WA(dPS, 0) = 0.0; WA(dVL, 0) = 0.0;
    WA(dX, N) = 0.0; WA(dY, N) = 0.0; WA(dPS, N) = 0.0; WA(dVL, N) = 0.0;
    WA(dDE, N) = 0.0; WA(dAC, N) = 0.0;
    return ok;
  }

  // a0 b0 + a1 b1 + a2 b2 + a3 b3 as two fused chains
  OBCA_HD static double dot4(double a0, double b0, double a1, double b1, double a2, double b2, double a3, double b3) {
    return fma(a1, b1, a0 * b0) + fma(a3, b3, a2 * b2);
  }
  // forward roll-out of the step: control row `kr` of the gain, state row `dr` of the dynamics Jacobian
  OBCA_HD static double roll_u(double kf, const double* kr, double s0, double s1, double s2, double s3, double s4, double s5,
                               double dt) {
    return (fma(kr[1], s1, kr[0] * s0) + fma(kr[3], s3, kr[2] * s2)) + (fma(kr[5], s5, kr[4] * s4) + fma(kr[6], dt, kf));
  }
  OBCA_HD static double roll_x(double r, double selx, double sely, const double* dr, double s0, double s1, double s2, double s3,
                               double dt, double u0, double u1) {
    return (fma(sely, s1, selx * s0) + fma(dr[1], s3, dr[0] * s2)) + (fma(dr[4], u1, dr[3] * u0) + fma(dr[2], dt, r));
  }
  // -------------------------------------------------------------------------------------------------
  // Wide (full-warp) KKT sweep: the device path of the sweep kernel and of the persistent kernel.
  // The stage recursion is a serial chain of 2 N steps per problem and nothing else of an iteration is, so its latency --
  // not its operation count -- bounds the solve time of the slowest problems of a batch.  Each of the three matrix steps
  // of a stage is cut into scalar TASKS (one entry of T, H or P each: a 4-term inner product or a rank-2 update), at most
  // two per lane, described by offsets that a lane computes once per sweep; the steps exchange through a 2 KB tile:
  //   step 1 (42 tasks): T = P Phi (the 5 dense columns) and g = p + P r~                         reads P, slot   writes T
  //   step 2 (54 tasks): H = Q + Phi' T (45 entries, both triangles stored), hv = q + Phi' g      reads T, slot   writes H
  //   step 3 (35 tasks): 2x2 pivot on (de, a) (every lane: one reciprocal), gain column, new P entry / p entry
  //                                                                                               reads H         writes P, T(:, X|Y)
  // Tile (doubles): P 7x7 full [0,49) | p [49,56) | T 7x10 (columns of the stage vector + g) [56,126) |
  //                 H 9x10 (column 9 = hv) [126,216) | zeros [216,224) | dump [224,256): one cell per lane for the stores of
  //                 its idle tasks (a lane only ever races with itself there)
  // Gains go to the stage's slot (RK..), rows 0..3 of P_k / p_k too (RPP.., Rpp..: consumed Q/q space) for recover_stage.
  // -------------------------------------------------------------------------------------------------
  static constexpr int WP = 0, Wp = 49, WT = 56, WH = 126, WZ = 216, WDUMP = 224, WIDE_TILE = 256;
  struct WideLane {
    int s1_p[2], s1_j[2], s1_js[2], s1_x[2], s1_o[2];
    int s2_q[2], s2_j[2], s2_js[2], s2_t[2], s2_x[2], s2_o1[2], s2_o2[2];
    int s3_h[2], s3_hid[2], s3_hia[2], s3_hdj[2], s3_haj[2], s3_o1[2], s3_o2[2], s3_t1[2], s3_t2[2], s3_g1[2], s3_g2[2], s3_k[2], s3_ks[2];
    int dump;
    int ok;
  };
  OBCA_HD static constexpr int col5(int c) { return c == 0 ? IP : c == 1 ? IV : c == 2 ? IT : c == 3 ? IDE : IAC; }
  OBCA_HD static constexpr int idx5(int y) { return y == IP ? 0 : y == IV ? 1 : y == IT ? 2 : y == IDE ? 3 : y == IAC ? 4 : -1; }
  // packed pair index -> (i, j), i <= j < n
  OBCA_HD static void unpack_pair(int t, int n, int& i, int& j) {
    i = 0;
    while (t >= n - i) { t -= n - i; ++i; }
    j = i + t;
  }
  OBCA_HD static void wl_init(WideLane& L, int lane) {
    const int dump = WDUMP + lane;
    L.dump = dump;
    for (int u = 0; u < 2; ++u) {
      const int t = lane + 32 * u;
      // ---- step 1: task t = 6 a + c6 ----
      if (t < 42) {
        const int a = t / 6, c6 = t - 6 * a;
        L.s1_p[u] = WP + 7 * a;
        L.s1_j[u] = c6 < 5 ? RDYN + c6 : RR4;
        L.s1_js[u] = c6 < 5 ? 5 : 1;
        L.s1_x[u] = c6 == 2 ? WP + 7 * a + 6 : c6 == 3 ? WP + 7 * a + 4 : c6 == 4 ? WP + 7 * a + 5 : c6 == 5 ? Wp + a : WZ;
        L.s1_o[u] = WT + 10 * a + (c6 < 5 ? col5(c6) : 9);
      } else {
        L.s1_p[u] = WP; L.s1_j[u] = RDYN; L.s1_js[u] = 5; L.s1_x[u] = WZ; L.s1_o[u] = dump;
      }
      // ---- step 2: t < 45: H(i, j), i <= j;  45 <= t < 54: hv(i) ----
      if (t < 54) {
        int i, j;
        if (t < 45) unpack_pair(t, NYV, i, j); else { i = t - 45; j = 9; }
        // representation with the row index in the dense set {psi, v, t, de, a} when there is one
        int r = i, c = j;
        if (idx5(i) < 0 && j < 9 && idx5(j) >= 0) { r = j; c = i; }
        const int r5 = idx5(r);
        L.s2_q[u] = j < 9 ? RQ + sym_idx<NYV>(i, j) : Rq + i;
        L.s2_j[u] = r5 >= 0 ? RDYN + r5 : -1;
        L.s2_js[u] = r5 >= 0 ? 5 : 1;
        L.s2_t[u] = WT + c;
        L.s2_x[u] = r == IT ? WT + 60 + c : r == IDE ? WT + 40 + c : r == IAC ? WT + 50 + c : r == IX ? WT + c : r == IY ? WT + 10 + c : WZ;
        L.s2_o1[u] = WH + 10 * i + j;
        L.s2_o2[u] = (j < 9 && i != j) ? WH + 10 * j + i : dump;
      } else {
        L.s2_q[u] = RQ; L.s2_j[u] = -1; L.s2_js[u] = 1; L.s2_t[u] = WT; L.s2_x[u] = WZ; L.s2_o1[u] = dump; L.s2_o2[u] = dump;
      }
      // ---- step 3: t < 28: P(i, j), i <= j < 7;  28 <= t < 35: p(i) ----
      if (t < 35) {
        int i, j;
        if (t < 28) unpack_pair(t, NSV, i, j); else { i = t - 28; j = 9; }
        L.s3_h[u] = WH + 10 * i + j; L.s3_hid[u] = WH + 10 * i + IDE; L.s3_hia[u] = WH + 10 * i + IAC;
        L.s3_hdj[u] = WH + 10 * IDE + j; L.s3_haj[u] = WH + 10 * IAC + j;
        if (j < 7) {
          L.s3_o1[u] = WP + 7 * i + j; L.s3_o2[u] = WP + 7 * j + i;
          L.s3_t1[u] = j < 2 ? WT + 10 * i + j : dump;              // T(:, X | Y) = P(:, 0 | 1)
          L.s3_t2[u] = (i < 2 && i != j) ? WT + 10 * j + i : dump;
          L.s3_g1[u] = i < 4 ? RPP + NSV * i + j : -1;
          L.s3_g2[u] = (j < 4 && i != j) ? RPP + NSV * j + i : -1;
          L.s3_k[u] = i == 0 ? RK + j : -1; L.s3_ks[u] = NSV;
        } else {
          L.s3_o1[u] = Wp + i; L.s3_o2[u] = dump; L.s3_t1[u] = dump; L.s3_t2[u] = dump;
          L.s3_g1[u] = i < 4 ? Rpp + i : -1; L.s3_g2[u] = -1;
          L.s3_k[u] = i == 0 ? RK + 14 : -1; L.s3_ks[u] = 1;
        }
      } else {
        L.s3_h[u] = WZ; L.s3_hid[u] = WZ; L.s3_hia[u] = WZ; L.s3_hdj[u] = WZ; L.s3_haj[u] = WZ;
        L.s3_o1[u] = dump; L.s3_o2[u] = dump; L.s3_t1[u] = dump; L.s3_t2[u] = dump;
        L.s3_g1[u] = -1; L.s3_g2[u] = -1; L.s3_k[u] = -1; L.s3_ks[u] = 1;
      }
    }
    L.ok = 1;
  }
  // terminal value (regularised end-point rows x_N == xF, multiplier estimate pi_{N-1}) into the tile; its rows 0..3 into
  // slot N.  Two lane passes (zero, then set) with a warp barrier in between.
  OBCA_HD static void wl_zero(int lane, double* tile, double* slotN) {
    for (int e = lane; e < WIDE_TILE; e += 32) tile[e] = 0.0;
    if (lane < 28) slotN[RPP + lane] = 0.0;
  }
  OBCA_HD static void wl_terminal(int lane, double* tile, double* slotN, const PkCtx& C) {
    OBCA_LOCALS(C);
    const int N = CTX_N(C);
    if (lane < 4) {
      const double rho = 1.0 / CTX_O(C).dc, pl = -WV(PI, lane, N - 1);
      tile[WP + 8 * lane] = rho; tile[Wp + lane] = pl;
      if (lane < 2) tile[WT + 10 * lane + lane] = rho;
      slotN[RPP + NSV * lane + lane] = rho; slotN[Rpp + lane] = pl;
    }
  }
  OBCA_HD static void wl_step1(const WideLane& L, const double* slot, double* tile) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const double* const pr = tile + L.s1_p[u];
      const double* const jc = slot + L.s1_j[u];
      const int js = L.s1_js[u];
      const double acc = dot4(pr[0], jc[0], pr[1], jc[js], pr[2], jc[2 * js], pr[3], jc[3 * js]);
      tile[L.s1_o[u]] = tile[L.s1_x[u]] + acc;
    }
  }
  OBCA_HD static void wl_step2(const WideLane& L, const double* slot, double* tile) {
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const double* const jc = L.s2_j[u] >= 0 ? slot + L.s2_j[u] : tile + WZ;
      const double* const tc = tile + L.s2_t[u];
      const int js = L.s2_js[u];
      const double acc = dot4(jc[0], tc[0], jc[js], tc[10], jc[2 * js], tc[20], jc[3 * js], tc[30]);
      const double v = (slot[L.s2_q[u]] + tile[L.s2_x[u]]) + acc;
      tile[L.s2_o1[u]] = v; tile[L.s2_o2[u]] = v;
    }
  }
  // `out`: the stage's slot (gains, rows 0..3 of P_k / p_k)
  OBCA_HD static void wl_step3(WideLane& L, double* out, double* tile) {
    const double h77 = tile[WH + 10 * IDE + IDE], h78 = tile[WH + 10 * IDE + IAC], h88 = tile[WH + 10 * IAC + IAC];
    double det = fma(h77, h88, -(h78 * h78));
    if (!(h77 > 0.0) || !(det > 0.0)) { L.ok = 0; det = 1e300; }
    const double idet = rcp(det);
    const double n00 = h88 * idet, n01 = -h78 * idet, n11 = h77 * idet;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const double hdj = tile[L.s3_hdj[u]], haj = tile[L.s3_haj[u]];
      const double K0 = -fma(n00, hdj, n01 * haj), K1 = -fma(n01, hdj, n11 * haj);
      const double v = fma(tile[L.s3_hia[u]], K1, fma(tile[L.s3_hid[u]], K0, tile[L.s3_h[u]]));
      double* const g1 = L.s3_g1[u] >= 0 ? out + L.s3_g1[u] : tile + L.dump;
      double* const g2 = L.s3_g2[u] >= 0 ? out + L.s3_g2[u] : tile + L.dump;
      double* const kp = L.s3_k[u] >= 0 ? out + L.s3_k[u] : tile + L.dump;
      const int ks = L.s3_k[u] >= 0 ? L.s3_ks[u] : 0;
      *g1 = v; *g2 = v;
      kp[0] = K0; kp[ks] = K1;
      tile[L.s3_o1[u]] = v; tile[L.s3_o2[u]] = v; tile[L.s3_t1[u]] = v; tile[L.s3_t2[u]] = v;
    }
  }

#if defined(__CUDA_ARCH__)
  // root (x_0, w_0 fixed; dt free) + forward roll-out of the primal step, lane-parallel: lanes 0,1 -> controls, lanes 0..3 ->
  // next state rows.  SRC(k): pointer to the slot of stage k (gains, dynamics Jacobian, residual).
  template <class SlotOf>
  __device__ static __forceinline__ int kkt_forward_warp(const PkCtx& C, const double* tile, ProbState* Sout, bool write, SlotOf slot_of) {
    const ParkProblem& Pp = CTX_P(C);
    const int N = CTX_N(C);
    const int lane = threadIdx.x & 31;
    int ok = 1;
    double dt = 0.0;
    if (!Pp.fix_time) {
      double ptt = tile[WP + 7 * IT + IT];
      if (!(ptt > 0.0)) { ok = 0; ptt = 1e300; }
      dt = -tile[Wp + IT] / ptt;
    }
    if (lane == 0 && write) Sout->dt = dt;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0, s4 = 0.0, s5 = 0.0;
    const int ur = lane & 1, xr = lane & 3;
    const unsigned FULL = 0xffffffffu;
    const double selx = (xr == 0) ? 1.0 : 0.0, sely = (xr == 1) ? 1.0 : 0.0;
    double* const dxw = C.W + (size_t)(CTX_L(C).dX + xr) * CTX_L(C).NSP;      // dX, dY, dPS, dVL are consecutive arrays
    double* const duw = C.W + (size_t)(CTX_L(C).dDE + ur) * CTX_L(C).NSP;     // dDE, dAC are consecutive arrays
    for (int k = 0; k < N; ++k) {
      const double* const slot = slot_of(k);
      const double* const kr = slot + RK + ur * NSV;
      const double u = roll_u(slot[RK + 14 + ur], kr, s0, s1, s2, s3, s4, s5, dt);
      const double u0 = __shfl_sync(FULL, u, 0), u1 = __shfl_sync(FULL, u, 1);
      const double* const dr = slot + RDYN + 5 * xr;
      const double sn = roll_x(slot[RR4 + xr], selx, sely, dr, s0, s1, s2, s3, dt, u0, u1);
      if (lane < 2 && write) duw[k] = u;
      s0 = __shfl_sync(FULL, sn, 0); s1 = __shfl_sync(FULL, sn, 1); s2 = __shfl_sync(FULL, sn, 2); s3 = __shfl_sync(FULL, sn, 3);
      s4 = u0; s5 = u1;
      if (lane < 4 && write) {
        if (k + 1 < N) dxw[k + 1] = sn;
        else Sout->eN[xr] = sn;
      }
      __syncwarp();      // every lane is done with slot k before the ring slot is refilled (sweep kernel)
    }
    if (write) {
      if (lane < 4) { dxw[0] = 0.0; dxw[N] = 0.0; }
      if (lane < 2) duw[N] = 0.0;
    }
    return ok;
  }
  // the whole sweep with the stage slots in shared memory (persistent kernel): one warp
  __device__ static int kkt_solve_warp(const PkCtx& C, double* tile) {
    const int N = CTX_N(C);
    const int lane = threadIdx.x & 31;
    WideLane L;
    wl_init(L, lane);
    wl_zero(lane, tile, C.ric + N * RSTRIDE);
    __syncwarp();
    wl_terminal(lane, tile, C.ric + N * RSTRIDE, C);
    __syncwarp();
    for (int k = N - 1; k >= 0; --k) {
      double* const slot = C.ric + k * RSTRIDE;
      wl_step1(L, slot, tile);
      __syncwarp();
      wl_step2(L, slot, tile);
      __syncwarp();
      wl_step3(L, slot, tile);
      __syncwarp();
      if (!L.ok) return 0;      // wrong inertia: the sweep result is discarded anyway (all lanes see the same pivot)
    }
    double* const ric = C.ric;
    return kkt_forward_warp(C, tile, C.S, true, [ric](int k) { return (const double*)(ric + k * RSTRIDE); });
  }
#else
  // host emulation of the warp: the 32 lanes run each step one after the other (a step only reads what earlier
  // steps wrote, exactly what __syncwarp() guarantees on the device)
  static int kkt_solve_warp_emul(const PkCtx& C, double* tile) {
    const int N = CTX_N(C);
    WideLane L[32];
    double* const slotN = C.ric + N * RSTRIDE;
    for (int l = 0; l < 32; ++l) wl_init(L[l], l);
    for (int l = 0; l < 32; ++l) wl_zero(l, tile, slotN);
    for (int l = 0; l < 32; ++l) wl_terminal(l, tile, slotN, C);
    for (int k = N - 1; k >= 0; --k) {
      double* const slot = C.ric + k * RSTRIDE;
      for (int l = 0; l < 32; ++l) wl_step1(L[l], slot, tile);
      for (int l = 0; l < 32; ++l) wl_step2(L[l], slot, tile);
      for (int l = 0; l < 32; ++l) wl_step3(L[l], slot, tile);
      if (!L[0].ok) return 0;
    }
    return kkt_root_forward(C, tile[WP + 7 * IT + IT], tile[Wp + IT]);
  }
#endif

  // fraction-to-the-boundary helpers.  The largest step keeping every gap at (1 - tau) of its value is
  // tau * min_i gap_i / (-dgap_i) over the shrinking gaps; the minimum is tracked as a fraction g/d and compared by
  // cross-multiplication (all gaps and -dgap are positive), so that ONE division per stage replaces one per bound.
  struct Ftb {
    double g, d;
    OBCA_HD Ftb() : g(1.0), d(0.0) {}
    OBCA_HD double alpha(double tau) const { return d > 0.0 ? dmin_(1.0, tau * g / d) : 1.0; }
  };
  OBCA_HD static void ftb(double gap, double dgap, double, Ftb& a) {
    if (dgap < 0.0 && gap * a.d < a.g * -dgap) { a.g = gap; a.d = -dgap; }
  }
  // dual step of a bound multiplier z with primal gap `gap` whose gap moves by dgap
  OBCA_HD static double dzb(double z, double gap, double dgap, double mu_b) { return (mu_b - z * dgap) * rcp(gap) - z; }

  // ---------------------------------------------------------------------------------------------------
  // K4a: recover local steps, slack steps; step-length partials; directional derivative of the barrier objective
  // ---------------------------------------------------------------------------------------------------
  // ---------------------------------------------------------------------------------------------------
  // K4a, one (stage k, obstacle j) block: step of the local unknowns from the factor stored by block_eval and the pose step
  // (dX, dY, dP); fraction-to-the-boundary and barrier-derivative partials of the block.
  // ---------------------------------------------------------------------------------------------------
  struct RBlockOut { double apr_g, apr_d, adu_g, adu_d, dphi; };
  OBCA_HD static void block_recover(const PkCtx& C, int k, int j, double X, double Y, double cs_, double sn_, double dX, double dY,
                                    double dP, double mu_b, double dw, RBlockOut& rbo) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const double tau = 0.0;      // (unused by ftb: the fractions are scaled by tau when the stage is finished)
    Ftb apr, adu;
    double dphi = 0.0;
    {
      ObsRows<VM> R; ObsVars<VM> Qv; ObsGeom<VM> G;
      load_rows(C, j, R);
      load_vars(C, k, j, R, Qv);
      obs_geom<VM, SDV>(P, X, Y, cs_, sn_, R, Qv, G);
      const int piv = choose_pivot<VM, SDV>(R, G);
      if (piv != 0) {
        swap_rows(R, Qv, piv);
        obs_geom<VM, SDV>(P, X, Y, cs_, sn_, R, Qv, G);
      }
      ObsStep<VM> St;
      obs_recover<VM, SDV>(P, R, Qv, G, mu_b, dw, &WV(LF, j * CTX_L(C).nfac, k), CTX_L(C).NSP, dX, dY, dP, St);
      // un-permute lambda
      if (piv != 0) {
#pragma unroll
        for (int i = 1; i < VM; ++i)
          if (i == piv) {
            double tmp = St.dlam[0]; St.dlam[0] = St.dlam[i]; St.dlam[i] = tmp;
            tmp = Qv.lam[0]; Qv.lam[0] = Qv.lam[i]; Qv.lam[i] = tmp;
            tmp = Qv.zlam[0]; Qv.zlam[0] = Qv.zlam[i]; Qv.zlam[i] = tmp;
          }
      }
#pragma unroll
      for (int i = 0; i < VM; ++i) {
        if (i < R.v) {
          WDV(dLAM, P.voff[j] + i, k) = St.dlam[i];
          ftb(Qv.lam[i], St.dlam[i], tau, apr);
          ftb(Qv.zlam[i], dzb(Qv.zlam[i], Qv.lam[i], St.dlam[i], mu_b), tau, adu);
          dphi += -mu_b * rcp(Qv.lam[i]) * St.dlam[i];
        }
      }
#pragma unroll
      for (int m = 0; m < 4; ++m) {
        WDV(dMU, 4 * j + m, k) = St.dmu[m];
        ftb(Qv.mu[m], St.dmu[m], tau, apr);
        ftb(Qv.zmu[m], dzb(Qv.zmu[m], Qv.mu[m], St.dmu[m], mu_b), tau, adu);
        dphi += -mu_b * rcp(Qv.mu[m]) * St.dmu[m];
      }
      if (SDV) {
        WDV(dSL, j, k) = St.dsl; WDV(YNn, j, k) = St.yn_new;
        dphi += (1e2 + 2e4 * Qv.sl) * St.dsl;
      }
      WDV(YRn, 2 * j, k) = St.yr1_new; WDV(YRn, 2 * j + 1, k) = St.yr2_new;
      WDV(dSD, j, k) = St.dsd;
      {
        const double gap = Qv.sd - P.dmin;
        ftb(gap, St.dsd, tau, apr);
        ftb(Qv.vd, dzb(Qv.vd, gap, St.dsd, mu_b), tau, adu);
        dphi += -mu_b * rcp(gap) * St.dsd;
      }
      if (!SDV) {
        WDV(dSN, j, k) = St.dsn;
        const double gap = 1.0 - Qv.sn;
        ftb(gap, -St.dsn, tau, apr);
        ftb(Qv.vn, dzb(Qv.vn, gap, -St.dsn, mu_b), tau, adu);
        dphi += mu_b * rcp(gap) * St.dsn;
      }
    }
    rbo.apr_g = apr.g; rbo.apr_d = apr.d; rbo.adu_g = adu.g; rbo.adu_d = adu.d; rbo.dphi = dphi;
  }
  // K4a, item pass: step of the unknowns of block i = (obstacle j, stage k); its tightest fractions to the boundary and its
  // part of the barrier directional derivative go straight into the thread's running StepPart (min / min / sum)
  OBCA_HD_NI static void block_item_recover(const PkCtx& C, int i, StepPart& acc) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int NS = CTX_N(C) + 1;
    const int j = i / NS, k = i - j * NS;
    const double X = WA(X, k), Y = WA(Y, k), ps = WA(PS, k);
    const double dX = WA(dX, k), dY = WA(dY, k), dP = WA(dPS, k);
    double sn_, cs_;
    sincos(ps, &sn_, &cs_);
    RBlockOut rb;
    block_recover(C, k, j, X, Y, cs_, sn_, dX, dY, dP, S.mu, S.dw, rb);
    Ftb apr, adu;
    apr.g = rb.apr_g; apr.d = rb.apr_d; adu.g = rb.adu_g; adu.d = rb.adu_d;
    acc.apr = dmin_(acc.apr, apr.alpha(S.tau)); acc.adu = dmin_(acc.adu, adu.alpha(S.tau));
    acc.dphi += rb.dphi;
  }

  // K4a, stage pass (everything of stage k that is not an obstacle block)
  OBCA_HD_NI static void recover_stage(const PkCtx& C, int k, StepPart& out) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int N = CTX_N(C);
    const bool fix = P.fix_time != 0;
    const double mu_b = S.mu, dw = S.dw, tau = S.tau;
    const bool pose_free = (k >= 1 && k <= N - 1);
    const double t = fix ? 1.0 : S.t;
    const double X = WA(X, k), Y = WA(Y, k), ps = WA(PS, k), v = WA(VL, k);
    const double dX = WA(dX, k), dY = WA(dY, k), dP = WA(dPS, k), dV = WA(dVL, k);
    Ftb apr, adu;
    double dphi = 0.0;
    if (k < N) {
      // new multiplier of the dynamics row k:  pi+ = -(P_{k+1} s_{k+1} + p_{k+1})_x   (costate of the Riccati sweep)
      double sn[NSV];
      if (k + 1 < N) { sn[0] = WA(dX, k + 1); sn[1] = WA(dY, k + 1); sn[2] = WA(dPS, k + 1); sn[3] = WA(dVL, k + 1); }
      else { sn[0] = S.eN[0]; sn[1] = S.eN[1]; sn[2] = S.eN[2]; sn[3] = S.eN[3]; }
      sn[IWD] = WA(dDE, k); sn[IWA] = WA(dAC, k); sn[IT] = S.dt;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        double acc = PPV(Rpp + i, k + 1);
#pragma unroll
        for (int l = 0; l < NSV; ++l) acc += PPV(RPP + i * NSV + l, k + 1) * sn[l];
        WDV(PIn, i, k) = -acc;
      }
    }
    if (pose_free) {
      const double ex = X - C.in.rx[k], ey = Y - C.in.ry[k], ep = ps - C.in.ryaw[k];
      const double aXl = X - P.xyb[0], aXu = P.xyb[1] - X, aYl = Y - P.xyb[2], aYu = P.xyb[3] - Y, aVl = v + 1.0, aVu = 2.0 - v;
      ftb(aXl, dX, tau, apr); ftb(aXu, -dX, tau, apr); ftb(aYl, dY, tau, apr); ftb(aYu, -dY, tau, apr);
      ftb(aVl, dV, tau, apr); ftb(aVu, -dV, tau, apr);
      double z;
      z = WA(ZXL, k); ftb(z, dzb(z, aXl, dX, mu_b), tau, adu);
      z = WA(ZXU, k); ftb(z, dzb(z, aXu, -dX, mu_b), tau, adu);
      z = WA(ZYL, k); ftb(z, dzb(z, aYl, dY, mu_b), tau, adu);
      z = WA(ZYU, k); ftb(z, dzb(z, aYu, -dY, mu_b), tau, adu);
      z = WA(ZVL, k); ftb(z, dzb(z, aVl, dV, mu_b), tau, adu);
      z = WA(ZVU, k); ftb(z, dzb(z, aVu, -dV, mu_b), tau, adu);
      dphi += (2e-3 * ex - mu_b * rcp(aXl) + mu_b * rcp(aXu)) * dX + (2e-3 * ey - mu_b * rcp(aYl) + mu_b * rcp(aYu)) * dY +
              2.0 * P.w_yaw * ep * dP + (2e-4 * v - mu_b * rcp(aVl) + mu_b * rcp(aVu)) * dV;
    }
    if (k < N) {
      const double de = WA(DE, k), ac = WA(AC, k), dD = WA(dDE, k), dA = WA(dAC, k);
      const double wd = k > 0 ? WA(DE, k - 1) : 0.0, wa = k > 0 ? WA(AC, k - 1) : 0.0;
      const double dwd = k > 0 ? WA(dDE, k - 1) : 0.0, dwa = k > 0 ? WA(dAC, k - 1) : 0.0;
      const double h = t * P.Ts, ih = rcp(h), ih2 = ih * ih, it = rcp(t);
      const double ed = de - wd, ea = ac - wa;
      const double T = 0.1 * (ed * ed + ea * ea) * ih2;
      const double aDl = de + 0.6, aDu = 0.6 - de, aAl = ac + 0.4, aAu = 0.4 - ac;
      ftb(aDl, dD, tau, apr); ftb(aDu, -dD, tau, apr); ftb(aAl, dA, tau, apr); ftb(aAu, -dA, tau, apr);
      double z;
      z = WA(ZDL, k); ftb(z, dzb(z, aDl, dD, mu_b), tau, adu);
      z = WA(ZDU, k); ftb(z, dzb(z, aDu, -dD, mu_b), tau, adu);
      z = WA(ZAL, k); ftb(z, dzb(z, aAl, dA, mu_b), tau, adu);
      z = WA(ZAU, k); ftb(z, dzb(z, aAu, -dA, mu_b), tau, adu);
      // rate slack
      const double gr = (wd - de) * ih;
      const double rs = WA(RS, k);
      const double gl = rs + 0.6, gu = 0.6 - rs;
      const double drs = (dwd - dD) * ih - (fix ? 0.0 : gr * it * S.dt) + (gr - rs);
      WD(dRS, k) = drs;
      ftb(gl, drs, tau, apr); ftb(gu, -drs, tau, apr);
      z = WA(RVL, k); ftb(z, dzb(z, gl, drs, mu_b), tau, adu);
      z = WA(RVU, k); ftb(z, dzb(z, gu, -drs, mu_b), tau, adu);
      dphi += (0.02 * de + 0.2 * ed * ih2 - mu_b * rcp(aDl) + mu_b * rcp(aDu)) * dD + (2.0 * P.w_a * ac + 0.2 * ea * ih2 - mu_b * rcp(aAl) + mu_b * rcp(aAu)) * dA +
              (-0.2 * ed * ih2) * dwd + (-0.2 * ea * ih2) * dwa + (fix ? 0.0 : -2.0 * T * it * S.dt) +
              (-mu_b * rcp(gl) + mu_b * rcp(gu)) * drs;
    }
    if (k == 0 && !fix) {
      const double m = (double)(N + 1);
      const double gl = t - 0.8, gu = 1.2 - t;
      ftb(gl, S.dt, tau, apr); ftb(gu, -S.dt, tau, apr);
      ftb(S.zTL, dzb(S.zTL, gl, S.dt, mu_b), tau, adu);
      ftb(S.zTU, dzb(S.zTU, gu, -S.dt, mu_b), tau, adu);
      dphi += m * (0.5 + 2.0 * t - mu_b * rcp(gl) + mu_b * rcp(gu)) * S.dt;
    }
    out.apr = apr.alpha(tau); out.adu = adu.alpha(tau); out.dphi = dphi;
  }

  // ---------------------------------------------------------------------------------------------------
  // K4b: merit-function partials at the trial point z + alpha dz  (theta = ||c||_1, phi = barrier objective)
  // ---------------------------------------------------------------------------------------------------
  // item pass: block i = (obstacle j, stage k) at the trial point
  OBCA_HD_NI static void block_item_merit(const PkCtx& C, int i, double alpha, MeritPart& acc) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int NS = CTX_N(C) + 1;
    const int j = i / NS, k = i - j * NS;
    const double mu_b = S.mu;
    const double X = WA(X, k) + alpha * WA(dX, k), Y = WA(Y, k) + alpha * WA(dY, k);
    const double ps = WA(PS, k) + alpha * WA(dPS, k);
    double sn_, cs_;
    sincos(ps, &sn_, &cs_);
    double th = 0.0, phi = 0.0;
    bool bad = false;
    LogAcc lacc;
    ObsRows<VM> R; ObsVars<VM> Qv; ObsGeom<VM> G;
    load_rows(C, j, R);
#pragma unroll
    for (int r = 0; r < VM; ++r) {
      const bool on = r < R.v;
      Qv.lam[r] = on ? WV(LAM, P.voff[j] + r, k) + alpha * WDV(dLAM, P.voff[j] + r, k) : 1.0;
      Qv.zlam[r] = 0.0;
      if (on) { bad |= !(Qv.lam[r] > 0.0); lacc.add(Qv.lam[r]); }
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      Qv.mu[m] = WV(MU, 4 * j + m, k) + alpha * WDV(dMU, 4 * j + m, k);
      Qv.zmu[m] = 0.0;
      bad |= !(Qv.mu[m] > 0.0); lacc.add(Qv.mu[m]);
    }
    Qv.sl = SDV ? WV(SL, j, k) + alpha * WDV(dSL, j, k) : 0.0;
    Qv.sd = WV(SD, j, k) + alpha * WDV(dSD, j, k);
    Qv.sn = SDV ? 0.0 : WV(SN, j, k) + alpha * WDV(dSN, j, k);
    Qv.yn = Qv.yr1 = Qv.yr2 = Qv.vd = Qv.vn = 0.0;
    obs_geom<VM, SDV>(P, X, Y, cs_, sn_, R, Qv, G);
    th += dabs(G.cn) + dabs(G.cd) + dabs(G.cr1) + dabs(G.cr2);
    if (SDV) phi += 1e2 * Qv.sl + 1e4 * Qv.sl * Qv.sl;
    { const double gap = Qv.sd - P.dmin; bad |= !(gap > 0.0); lacc.add(gap); }
    if (!SDV) { const double gap = 1.0 - Qv.sn; bad |= !(gap > 0.0); lacc.add(gap); }
    phi -= mu_b * lacc.total();
    acc.th += th;
    acc.phi += bad ? 1e300 : phi;
  }

  // stage pass: everything of stage k that is not an obstacle block
  OBCA_HD_NI static void merit_stage(const PkCtx& C, int k, double alpha, MeritPart& out) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int N = CTX_N(C);
    const bool fix = P.fix_time != 0;
    const double mu_b = S.mu;
    const bool pose_free = (k >= 1 && k <= N - 1);
    const double t = fix ? 1.0 : S.t + alpha * S.dt;
    const double X = WA(X, k) + alpha * WA(dX, k), Y = WA(Y, k) + alpha * WA(dY, k);
    const double ps = WA(PS, k) + alpha * WA(dPS, k), v = WA(VL, k) + alpha * WA(dVL, k);
    double th = 0.0, phi = 0.0;
    bool bad = false;
    LogAcc lacc;
    {
      const double ex = X - C.in.rx[k], ey = Y - C.in.ry[k], ep = ps - C.in.ryaw[k];
      phi += 1e-4 * v * v + 1e-3 * ex * ex + 1e-3 * ey * ey + P.w_yaw * ep * ep;
      if (pose_free) {
        const double g6[6] = {X - P.xyb[0], P.xyb[1] - X, Y - P.xyb[2], P.xyb[3] - Y, v + 1.0, 2.0 - v};
#pragma unroll
        for (int i = 0; i < 6; ++i) { bad |= !(g6[i] > 0.0); lacc.add(g6[i]); }
      }
    }
    if (k < N) {
      const double de = WA(DE, k) + alpha * WA(dDE, k), ac = WA(AC, k) + alpha * WA(dAC, k);
      const double wd = k > 0 ? WA(DE, k - 1) + alpha * WA(dDE, k - 1) : 0.0;
      const double wa = k > 0 ? WA(AC, k - 1) + alpha * WA(dAC, k - 1) : 0.0;
      const double h = t * P.Ts, ih = 1.0 / h;
      const double ed = de - wd, ea = ac - wa;
      phi += 0.01 * de * de + P.w_a * ac * ac + 0.1 * (ed * ed + ea * ea) * ih * ih;
      const double rs = WA(RS, k) + alpha * WD(dRS, k);
      const double g6[6] = {de + 0.6, 0.6 - de, ac + 0.4, 0.4 - ac, rs + 0.6, 0.6 - rs};
#pragma unroll
      for (int i = 0; i < 6; ++i) { bad |= !(g6[i] > 0.0); lacc.add(g6[i]); }
      th += dabs((wd - de) * ih - rs);
      DynOut dyn;
      dyn_eval(P, X, Y, ps, v, de, ac, t, dyn, nullptr, nullptr);
      double xn[4];
      if (k + 1 == N) { xn[0] = C.in.xF[0]; xn[1] = C.in.xF[1]; xn[2] = C.in.xF[2]; xn[3] = C.in.xF[3]; }
      else {
        xn[0] = WA(X, k + 1) + alpha * WA(dX, k + 1); xn[1] = WA(Y, k + 1) + alpha * WA(dY, k + 1);
        xn[2] = WA(PS, k + 1) + alpha * WA(dPS, k + 1); xn[3] = WA(VL, k + 1) + alpha * WA(dVL, k + 1);
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) th += dabs(dyn.f[i] - xn[i]);
    }
    if (k == 0 && !fix) {
      const double m = (double)(N + 1);
      const double gl = t - 0.8, gu = 1.2 - t;
      bad |= !(gl > 0.0) || !(gu > 0.0);
      phi += m * (0.5 * t + t * t) - m * mu_b * (log(gl) + log(gu));
    }
    phi -= mu_b * lacc.total();
    out.th = th;
    out.phi = bad ? 1e300 : phi;
  }

  // ---------------------------------------------------------------------------------------------------
  // K4c: accept the step (primal alpha, dual a_du, equality multipliers a_y) + Ipopt's multiplier safeguard
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD static double clipz(double z, double gap, double mu_b, double ks) {
    const double mg = mu_b * rcp(gap);
    return dmax(dmin_(z, ks * mg), mg * rcp(ks));
  }
  OBCA_HD static void upd_pair(double& q, double dq, double& zl, double& zu, double lo, double hi, double alpha,
                               double adu, double mu_b, double ks) {
    const double gl = q - lo, gu = hi - q;
    const double dzl = dzb(zl, gl, dq, mu_b), dzu = dzb(zu, gu, -dq, mu_b);
    q += alpha * dq; zl += adu * dzl; zu += adu * dzu;
    zl = clipz(zl, q - lo, mu_b, ks); zu = clipz(zu, hi - q, mu_b, ks);
  }
  // item pass: the variables of block i = (obstacle j, stage k)
  OBCA_HD_NI static void block_item_update(const PkCtx& C, int i) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int NS = CTX_N(C) + 1;
    const int j = i / NS, k = i - j * NS;
    const double mu_b = S.mu, ks = CTX_O(C).kappa_sigma;
    const double alpha = S.alpha, adu = S.a_du, ay = dmin_(S.alpha, S.a_du);   // alpha_for_y = min (:41)
    for (int r = P.voff[j]; r < P.voff[j + 1]; ++r) {
      double q = WV(LAM, r, k), z = WV(ZLAM, r, k);
      const double dq = WDV(dLAM, r, k);
      const double dz = dzb(z, q, dq, mu_b);
      q += alpha * dq; z += adu * dz;
      WV(LAM, r, k) = q; WV(ZLAM, r, k) = clipz(z, q, mu_b, ks);
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int r = 4 * j + m;
      double q = WV(MU, r, k), z = WV(ZMU, r, k);
      const double dq = WDV(dMU, r, k);
      const double dz = dzb(z, q, dq, mu_b);
      q += alpha * dq; z += adu * dz;
      WV(MU, r, k) = q; WV(ZMU, r, k) = clipz(z, q, mu_b, ks);
    }
    if (SDV) {
      WV(SL, j, k) += alpha * WDV(dSL, j, k);
      WV(YN, j, k) += ay * (WDV(YNn, j, k) - WV(YN, j, k));
    }
    WV(YR, 2 * j, k) += ay * (WDV(YRn, 2 * j, k) - WV(YR, 2 * j, k));
    WV(YR, 2 * j + 1, k) += ay * (WDV(YRn, 2 * j + 1, k) - WV(YR, 2 * j + 1, k));
    {
      double s = WV(SD, j, k), z = WV(VD, j, k);
      const double ds = WDV(dSD, j, k);
      const double dz = dzb(z, s - P.dmin, ds, mu_b);
      s += alpha * ds; z += adu * dz;
      WV(SD, j, k) = s; WV(VD, j, k) = clipz(z, s - P.dmin, mu_b, ks);
    }
    if (!SDV) {
      double s = WV(SN, j, k), z = WV(VN, j, k);
      const double ds = WDV(dSN, j, k);
      const double dz = dzb(z, 1.0 - s, -ds, mu_b);
      s += alpha * ds; z += adu * dz;
      WV(SN, j, k) = s; WV(VN, j, k) = clipz(z, 1.0 - s, mu_b, ks);
    }
  }

  // stage pass: pose, speed, controls, rate slack, multipliers of the dynamics rows
  OBCA_HD_NI static void update_stage(const PkCtx& C, int k) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const ProbState& S = *C.S;
    const int N = CTX_N(C);
    const double mu_b = S.mu, ks = CTX_O(C).kappa_sigma;
    const double alpha = S.alpha, adu = S.a_du, ay = dmin_(S.alpha, S.a_du);   // alpha_for_y = min (:41)
    const bool pose_free = (k >= 1 && k <= N - 1);
    if (pose_free) {
      double q, zl, zu;
      q = WA(X, k); zl = WA(ZXL, k); zu = WA(ZXU, k);
      upd_pair(q, WA(dX, k), zl, zu, P.xyb[0], P.xyb[1], alpha, adu, mu_b, ks);
      WA(X, k) = q; WA(ZXL, k) = zl; WA(ZXU, k) = zu;
      q = WA(Y, k); zl = WA(ZYL, k); zu = WA(ZYU, k);
      upd_pair(q, WA(dY, k), zl, zu, P.xyb[2], P.xyb[3], alpha, adu, mu_b, ks);
      WA(Y, k) = q; WA(ZYL, k) = zl; WA(ZYU, k) = zu;
      q = WA(VL, k); zl = WA(ZVL, k); zu = WA(ZVU, k);
      upd_pair(q, WA(dVL, k), zl, zu, -1.0, 2.0, alpha, adu, mu_b, ks);
      WA(VL, k) = q; WA(ZVL, k) = zl; WA(ZVU, k) = zu;
      WA(PS, k) += alpha * WA(dPS, k);
    }
    if (k < N) {
      double q, zl, zu;
      q = WA(DE, k); zl = WA(ZDL, k); zu = WA(ZDU, k);
      upd_pair(q, WA(dDE, k), zl, zu, -0.6, 0.6, alpha, adu, mu_b, ks);
      WA(DE, k) = q; WA(ZDL, k) = zl; WA(ZDU, k) = zu;
      q = WA(AC, k); zl = WA(ZAL, k); zu = WA(ZAU, k);
      upd_pair(q, WA(dAC, k), zl, zu, -0.4, 0.4, alpha, adu, mu_b, ks);
      WA(AC, k) = q; WA(ZAL, k) = zl; WA(ZAU, k) = zu;
      q = WA(RS, k); zl = WA(RVL, k); zu = WA(RVU, k);
      upd_pair(q, WD(dRS, k), zl, zu, -0.6, 0.6, alpha, adu, mu_b, ks);
      WA(RS, k) = q; WA(RVL, k) = zl; WA(RVU, k) = zu;
#pragma unroll
      for (int i = 0; i < 4; ++i) WV(PI, i, k) += ay * (WDV(PIn, i, k) - WV(PI, i, k));
    }
  }

  // ---------------------------------------------------------------------------------------------------
  // The four stage-parallel phases of an iteration as the driver sees them: an item pass over the (obstacle, stage) blocks
  // and a stage pass.  Only the evaluation needs a barrier between the two (the hand-over in the stage slots); the partial
  // results of both passes accumulate in the same per-thread record, which the caller reduces over the CTA.
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD static void eval_phase(const PkCtx& C, bool do_err, EvalPart& ep) {
    const int NS = CTX_N(C) + 1, NI = CTX_P(C).nOb * NS;
    OBCA_FOR_ITEMS(i, NI) block_item_eval(C, i, do_err, ep);
    OBCA_SYNC();
    // (the same thread handles stage k in both stage loops: no barrier between them)
    if (CTX_P(C).nOb > HO_SLOT_OB) OBCA_FOR_STAGES(k, NS) fold_far_handover(C, k);
    OBCA_FOR_STAGES(k, NS) { EvalPart e1; stage_eval(C, k, do_err, true, e1); part_merge(ep, e1); }
  }
  OBCA_HD static void recover_phase(const PkCtx& C, StepPart& sp) {
    const int NS = CTX_N(C) + 1, NI = CTX_P(C).nOb * NS;
    OBCA_FOR_ITEMS(i, NI) block_item_recover(C, i, sp);
    OBCA_FOR_STAGES(k, NS) { StepPart s1; recover_stage(C, k, s1); part_merge(sp, s1); }
  }
  OBCA_HD static void merit_phase(const PkCtx& C, double alpha, MeritPart& mp) {
    const int NS = CTX_N(C) + 1, NI = CTX_P(C).nOb * NS;
    OBCA_FOR_ITEMS(i, NI) block_item_merit(C, i, alpha, mp);
    OBCA_FOR_STAGES(k, NS) { MeritPart m1; merit_stage(C, k, alpha, m1); part_merge(mp, m1); }
  }
  OBCA_HD static void update_phase(const PkCtx& C) {
    const int NS = CTX_N(C) + 1, NI = CTX_P(C).nOb * NS;
    OBCA_FOR_ITEMS(i, NI) block_item_update(C, i);
    OBCA_FOR_STAGES(k, NS) update_stage(C, k);
  }

  // write the solution of stage k in the reference's output layout
  OBCA_HD static void store_stage(const PkCtx& C, int k, const PkOutputs& o) {
    OBCA_LOCALS(C);
    const ParkProblem& P = CTX_P(C);
    const int N = CTX_N(C);                   // extent: the problem's own horizon
    const int NL = P.N, NSL = NL + 1;         // strides of the optional duals: the batch layout
    o.xp[4 * k + 0] = WA(X, k); o.xp[4 * k + 1] = WA(Y, k); o.xp[4 * k + 2] = WA(PS, k); o.xp[4 * k + 3] = WA(VL, k);
    if (k < N) { o.up[2 * k + 0] = WA(DE, k); o.up[2 * k + 1] = WA(AC, k); }
    o.ts[k] = P.fix_time ? 1.0 : C.S->t;
    for (int r = 0; r < P.V; ++r) o.lp[(size_t)P.V * k + r] = WV(LAM, r, k);
    for (int r = 0; r < 4 * P.nOb; ++r) o.np[(size_t)4 * P.nOb * k + r] = WV(MU, r, k);
    if (SDV && o.sl) for (int j = 0; j < P.nOb; ++j) o.sl[(size_t)P.nOb * k + j] = WV(SL, j, k);
    if (o.duals) {
      double* d = o.duals;
      if (k < N) for (int i = 0; i < 4; ++i) d[4 * k + i] = WV(PI, i, k);
      d += 4 * NL;
      for (int r = 0; r < 2 * P.nOb; ++r) d[(size_t)2 * P.nOb * k + r] = WV(YR, r, k);
      d += (size_t)2 * P.nOb * NSL;
      for (int j = 0; j < P.nOb; ++j) d[(size_t)P.nOb * k + j] = SDV ? WV(YN, j, k) : WV(VN, j, k);
      d += (size_t)P.nOb * NSL;
      for (int j = 0; j < P.nOb; ++j) d[(size_t)P.nOb * k + j] = WV(VD, j, k);
    }
  }

  // ---------------------------------------------------------------------------------------------------
  // serial helpers (thread 0)
  // ---------------------------------------------------------------------------------------------------
  // number of multipliers (for Ipopt's s_d, s_c scaling)
  OBCA_HD static void mult_counts(const ParkProblem& P, int N, double& n_mult, double& n_bmult) {
    const int NS = N + 1;
    double nb = 6.0 * (N - 1) + 4.0 * N + (P.V + 4.0 * P.nOb) * NS + (P.fix_time ? 0.0 : 2.0 * NS);   // variable bounds
    nb += 2.0 * N + (double)P.nOb * NS + (P.signed_dist ? 0.0 : (double)P.nOb * NS);                   // slack bounds
    const double mE = 4.0 * N + 2.0 * P.nOb * NS + (P.signed_dist ? (double)P.nOb * NS : 0.0);
    const double mI = N + (double)P.nOb * NS + (P.signed_dist ? 0.0 : (double)P.nOb * NS);
    n_bmult = nb; n_mult = nb + mE + mI;
  }
  // ---- adapters used by the generic interior-point driver (IpmDriver below) ----
  typedef PkCtx Ctx;
  static constexpr bool PROF_CYCLES = false;   // prof[5] counts the re-evaluations after a barrier update
#if defined(__CUDA_ARCH__)
  template <typename T>
  __device__ static void reduce(T& v, const PkCtx& C) { block_reduce(v, C.red_scratch); }   // every warp of the CTA
#endif
  OBCA_HD static int n_stages(const PkCtx& C) { return CTX_N(C) + 1; }
  OBCA_HD static bool fixed_time(const PkCtx& C) { return CTX_P(C).fix_time != 0; }
  OBCA_HD static void mult_counts(const PkCtx& C, double& n_mult, double& n_bmult) { mult_counts(*C.P, CTX_N(C), n_mult, n_bmult); }
  OBCA_HD static void init_scalars(const PkCtx& C, int restart) {
    ProbState& S = *C.S;
    const IpmOpts& O = CTX_O(C);
    S.t = CTX_P(C).fix_time ? 1.0 : push_lo(restart ? S.t : 1.0, 0.8, 1.2, O.kappa1, O.kappa2);   // setvalue(timeScale, 1) (:214)
    S.zTL = 1.0; S.zTU = 1.0; S.dt = 0.0;
  }
  OBCA_HD static void update_scalars(const PkCtx& C) {
    ProbState& S = *C.S;
    if (!CTX_P(C).fix_time) {
      double q = S.t, zl = S.zTL, zu = S.zTU;
      upd_pair(q, S.dt, zl, zu, 0.8, 1.2, S.alpha, S.a_du, S.mu, CTX_O(C).kappa_sigma);
      S.t = q; S.zTL = zl; S.zTU = zu;
    }
  }
  // the KKT solve of an iteration, skipped (0) when the local blocks already failed the inertia test.  All threads call it;
  // the result is valid in thread 0, which may write S as soon as it returns.  Device: warp 0 runs the sweep over the stage
  // slots in shared memory (only warp 0 reads S.ok, and its __syncwarp orders those reads before thread 0's writes); host: the
  // emulation of that warp, or the serial sweep when the context has no tile.
  OBCA_HD static int factor(const PkCtx& C) {
#if defined(__CUDA_ARCH__)
    int ok = 0;
    if (threadIdx.x < 32) {
      ok = C.S->ok;
      if (ok) ok = kkt_solve_warp(C, C.tile);
      __syncwarp();
    }
    return ok;
#else
    if (!C.S->ok) return 0;
    return C.tile ? kkt_solve_warp_emul(C, C.tile) : kkt_solve(C);
#endif
  }
};

// ------------------------------------------------------------------------------------------------------------
// Generic interior-point driver (Ipopt's algorithm: monotone barrier update, inertia correction, filter line
// search).  M is the model policy (ParkSolver<VM,SDV>, QuadSolver<SDV>): per-stage phase functions, the block reduction
// (reduce), the KKT solve (factor) and what prof[5] holds (PROF_CYCLES).
// ------------------------------------------------------------------------------------------------------------
template <class M>
struct IpmDriver {
  typedef typename M::Ctx Ctx;
  OBCA_HD static void apply_errors(const Ctx& C, const EvalPart& e) {
    ProbState& S = *C.S;
    S.e_dual = M::fixed_time(C) ? e.e_dual : dmax(e.e_dual, dabs(e.rt));
    S.e_pr = e.e_pr; S.e_cmax = e.cmax; S.e_cmin = e.cmin; S.sum_y = e.sy; S.sum_z = e.sz;
    S.th_k = e.th; S.ph_k = e.phi; S.rz_t = e.rt; S.f_k = e.f;
  }
  OBCA_HD static double err_mu(const Ctx& C, double mu_t) {
    const ProbState& S = *C.S;
    const IpmOpts& O = CTX_O(C);
    double n_mult, n_bmult;
    M::mult_counts(C, n_mult, n_bmult);
    const double sd = dmax(O.s_max, (S.sum_y + S.sum_z) / n_mult) / O.s_max;
    const double sc = dmax(O.s_max, S.sum_z / n_bmult) / O.s_max;
    const double comp = dmax(S.e_cmax - mu_t, mu_t - S.e_cmin);
    return dmax(dmax(S.e_dual / sd, S.e_pr), comp / sc);
  }

  // ---------------------------------------------------------------------------------------------------
  // The iteration as phase functions: all threads of the CTA call them with the same context; S.phase says where the solve
  // stands between them.  solve() runs them in one loop, the parking rounds run them from separate kernels (obca_phased.cuh).
  // On the device phase_A / phase_C are out of line: one copy of their floating-point operations per template instance,
  // whichever kernel calls them, so that every schedule rounds the same way.
  // ---------------------------------------------------------------------------------------------------
  // B (serial part, one thread, after the KKT solve): Ipopt's inertia-correction bookkeeping.  `ok`: 1 if every pivot of
  // the sweep had the required sign, 0 otherwise (also when the local blocks already failed and the sweep was skipped).
  OBCA_HD static void phase_B_serial(ProbState& S, const IpmOpts& O, int ok) {
    S.n_fact++;
    if (!ok) {
      if (S.dw == 0.0) S.dw = (S.dw_last == 0.0) ? O.dw_first : dmax(O.dw_min, O.kw_minus * S.dw_last);
      else S.dw *= (S.dw_last == 0.0) ? O.kw_plus_first : O.kw_plus;
      if (S.dw > O.dw_max) { S.status = -2; ok = -1; }
    } else if (S.dw > 0.0) {
      S.dw_last = S.dw;
    }
    S.ok = ok;
    S.phase = ok > 0 ? PH_RECOVER : (ok == 0 ? PH_REASM : PH_END);
  }

  // A: [init] -> evaluate at the current iterate, convergence test, barrier update (+ re-evaluation), or re-assembly
  //    with a larger delta_w.  Leaves phase = PH_KKT (stage models ready) or PH_END (attempt over).
  OBCA_HD_NI static void phase_A(const Ctx& C) {
    const IpmOpts& O = CTX_O(C);
    ProbState& S = *C.S;
    const int NS = M::n_stages(C);
    const int ph = S.phase;
    EvalPart ep;
    if (ph == PH_REASM) {
      reassemble(C);
      return;
    }
    if (ph == PH_INIT) {
      const int restart = S.attempt;
      OBCA_SERIAL {
        M::init_scalars(C, restart);
        S.mu = O.mu_init; S.tau = dmax(O.tau_min, 1.0 - O.mu_init);
        S.dw = 0.0; S.dw_last = 0.0; S.nfilt = 0; S.status = 0; S.iters = 0; S.n_fact = 0; S.n_kick = 0;
        S.it = 0; S.first = 1;
      }
      OBCA_PROF_START();
      OBCA_SYNC();
      OBCA_FOR_STAGES(k, NS) M::init_stage(C, k, restart);
      OBCA_SYNC();
      OBCA_FOR_STAGES(k, NS) M::init_slacks(C, k);
      // (S.phase may only change behind a barrier: every thread read it on entry)
      OBCA_SERIAL { S.phase = PH_EVAL; }
      OBCA_SYNC();
    }
    // (PH_EVAL: new iterate -- or a barrier kick: new direction from the same iterate)
    OBCA_SERIAL { S.dw = 0.0; }
    OBCA_SYNC();
    part_init(ep);
    M::eval_phase(C, true, ep);
    OBCA_REDUCE(ep);
    OBCA_PROF(0);
    OBCA_SERIAL {
      S.prof[7]++;
      apply_errors(C, ep);
      S.ok = ep.ok;
      if (S.first) {
        S.theta_max = 1e4 * dmax(1.0, S.th_k);
        S.theta_min = 1e-4 * dmax(1.0, S.th_k);
        S.first = 0;
      }
      S.e0 = err_mu(C, 0.0);
      S.iters = S.it;
      S.flag = 0;
      if (S.e0 <= O.tol && S.e_dual <= O.dual_inf_tol && S.e_pr <= O.constr_viol_tol && S.e_cmax <= O.compl_inf_tol) {
        S.status = 1; S.flag = 1;
      } else if (S.it >= O.max_iter) {
        S.status = 0; S.flag = 1;
      } else {
        // monotone barrier update
        bool changed = false;
        while (S.mu > O.mu_min && err_mu(C, S.mu) <= O.kappa_eps * S.mu) {
          S.mu = dmax(O.mu_min, dmin_(O.kappa_mu * S.mu, pow(S.mu, O.theta_mu)));
          S.tau = dmax(O.tau_min, 1.0 - S.mu);
          changed = true;
        }
        if (changed) { S.nfilt = 0; S.flag = 2; }
      }
      S.phase = (S.flag == 1) ? PH_END : PH_KKT;
    }
    OBCA_SYNC();
    OBCA_PROF(5);
    if (S.flag == 2) {
      // mu changed: the barrier terms of the stage models (and phi) are stale
      part_init(ep);
      M::eval_phase(C, true, ep);
      OBCA_REDUCE(ep);
      OBCA_PROF(0);
      OBCA_SERIAL { apply_errors(C, ep); S.ok = ep.ok; S.prof[7]++; if (!M::PROF_CYCLES) S.prof[5]++; }
      OBCA_SYNC();
      OBCA_PROF(5);
    }
  }
  // Re-assembly with the current delta_w (inertia correction).  (Inertia failures are found by the sweep: a wrong sign among
  // the local pivots of the blocks alone is rare -- handling it inside this launch did not change the number of rounds.)
  OBCA_HD static void reassemble(const Ctx& C) {
    ProbState& S = *C.S;
    EvalPart ep;
    part_init(ep);
    M::eval_phase(C, false, ep);
    OBCA_REDUCE(ep);
    OBCA_SERIAL { S.ok = ep.ok; S.phase = PH_KKT; S.prof[7]++; }
    OBCA_SYNC();
    OBCA_PROF(0);
  }

  // C: recover the full step, step lengths, filter line search, and -- when a step is accepted -- the iterate update.
  //    Leaves PH_EVAL (new iterate, or barrier kick: same iterate, new barrier parameter) or PH_END (line-search failure).
  OBCA_HD_NI static void phase_C(const Ctx& C) {
    const IpmOpts& O = CTX_O(C);
    ProbState& S = *C.S;
    StepPart sp;
    part_init(sp);
    M::recover_phase(C, sp);
    OBCA_REDUCE(sp);
    OBCA_PROF(2);
    OBCA_SERIAL {
      const double apr = sp.apr, adu = sp.adu, dphi = sp.dphi;
      S.a_pr = apr; S.a_du = adu; S.dphi = dphi;
      const double th = S.th_k;
      if (dphi < 0.0 && th <= S.theta_min)
        S.a_min = O.gamma_alpha * dmin_(O.gamma_theta, dmin_(O.gamma_phi * th / (-dphi), O.delta * pow(th, O.s_theta) / pow(-dphi, O.s_phi)));
      else if (dphi < 0.0)
        S.a_min = O.gamma_alpha * dmin_(O.gamma_theta, O.gamma_phi * th / (-dphi));
      else
        S.a_min = O.gamma_alpha * O.gamma_theta;
      S.alpha = apr;
      S.flag = 0;
    }
    OBCA_SYNC();
    for (int nbt = 0;; ++nbt) {
      const double alpha = S.alpha;
      MeritPart mp;
      part_init(mp);
      M::merit_phase(C, alpha, mp);
      OBCA_REDUCE(mp);
      OBCA_PROF(3);
      OBCA_SERIAL {
        S.prof[6]++;
        const double th = mp.th, ph = mp.phi;
        S.th_t = th; S.ph_t = ph;
        bool in_filter = th >= S.theta_max || !(ph < 1e299);
        for (int i = 0; i < S.nfilt && !in_filter; ++i) in_filter = (th >= S.filt_th[i] && ph >= S.filt_ph[i]);
        bool accepted = false, ftype = false;
        if (!in_filter) {
          const bool sw = S.dphi < 0.0 && alpha * pow(-S.dphi, O.s_phi) > O.delta * pow(S.th_k, O.s_theta);
          if (S.th_k <= S.theta_min && sw) {
            if (ph <= S.ph_k + O.eta_phi * alpha * S.dphi + 10.0 * 2.220446049250313e-16 * dabs(S.ph_k)) { accepted = true; ftype = true; }
          } else {
            if (th <= (1.0 - O.gamma_theta) * S.th_k || ph <= S.ph_k - O.gamma_phi * S.th_k) accepted = true;
          }
        }
        if (accepted) {
          S.flag = 1;
          if (!ftype && S.nfilt < 64) {
            S.filt_th[S.nfilt] = (1.0 - O.gamma_theta) * S.th_k;
            S.filt_ph[S.nfilt] = S.ph_k - O.gamma_phi * S.th_k;
            S.nfilt++;
          }
        } else {
          S.alpha = 0.5 * alpha;
          if (S.alpha < S.a_min || nbt + 1 >= O.max_backtrack) {
            // Ipopt would enter its restoration phase here.  Substitute ("barrier kick"): forget the filter,
            // raise the barrier parameter one decade and recompute the direction from the same iterate; after
            // max_kick kicks the attempt ends with a line-search failure (the caller's retry logic takes over).
            if (S.n_kick < O.max_kick) {
              S.n_kick++;
              S.nfilt = 0;
              S.mu = dmin_(O.mu_init, 10.0 * S.mu);
              S.tau = dmax(O.tau_min, 1.0 - S.mu);
              S.flag = -2;
            } else {
              S.flag = -1; S.status = -1;
            }
          }
        }
        if (S.flag == 1) S.phase = PH_EVAL;
        else if (S.flag == -2) { S.it++; S.phase = PH_EVAL; }
        else if (S.flag == -1) S.phase = PH_END;
      }
      OBCA_SYNC();
      OBCA_PROF(5);
      if (S.flag != 0) break;
    }
    if (S.flag == 1) {      // accept
      M::update_phase(C);
      OBCA_SERIAL { M::update_scalars(C); S.it++; }
      OBCA_SYNC();
      OBCA_PROF(4);
    }
  }

  // ---------------------------------------------------------------------------------------------------
  // the solve of one problem from its warm start: all threads of the CTA call this with the same context
  // ---------------------------------------------------------------------------------------------------
  OBCA_HD static void solve(const Ctx& C) {
    ProbState& S = *C.S;
    state_fresh(S, M::n_stages(C) - 1);
    OBCA_SYNC();
    for (;;) {
      phase_A(C);
      const int ph = S.phase;
      OBCA_SYNC();      // every thread has read the phase before thread 0 moves it on (phase_B_serial)
      if (ph == PH_END) break;
      const int ok = M::factor(C);
      OBCA_SERIAL { phase_B_serial(S, CTX_O(C), ok); }
      OBCA_SYNC();
      OBCA_PROF(1);
      if (S.phase == PH_RECOVER) phase_C(C);
      if (S.phase == PH_END) break;
    }
  }
};

}  // namespace obca
