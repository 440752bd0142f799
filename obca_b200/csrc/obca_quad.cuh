// obca_quad.cuh -- model policy of the quadcopter NLPs for the generic interior-point driver (obca_solver.cuh).
//
// Replaces the JuMP + Ipopt solve inside QuadcopterNavigation/QuadcopterSignedDist.jl:25-300 (SDV = true) and
// QuadcopterDist.jl:25-282 (SDV = false): 12-state quadrotor, 4 rotor speeds, ball ego, five box obstacles, time scaling.
// Same exact reformulations as the parking model (pinned end states are parameters, one time-scale variable with
// multiplicity N+1, bounds are bounds) plus quirk Q5 (SURVEY.md A.4): the body-rate products of :153-155 are the
// stage-1 values x0[9..11] (constants).
//
// Stage vector of the KKT sweep:  y = [ x (12) | w = previous control (4) | t | u (4) ],  17 states + 4 controls.
// The stage models live in the per-CTA global workspace ([array][stage]); the Riccati sweep is block-cooperative: the three
// matrix products of a stage run on the FP64 tensor cores (DMMA) over dense zero-padded tiles in shared memory
// (kkt_solve_block); kkt_dense is the same elimination as a plain one-thread recursion (host emulation, tests).
#pragma once
#include "obca_quad_dyn_gen.cuh"
#include "obca_quad_local.cuh"
#include "obca_solver.cuh"

namespace obca {

constexpr int QNX = 12, QNU = 4, QNSV = 17, QNYV = 21;
constexpr int QIW = 12, QIT = 16, QIU = 17;
constexpr int QNQ = QNYV * (QNYV + 1) / 2;     // 231
constexpr int QNP = QNSV * (QNSV + 1) / 2;     // 153
constexpr double QUAD_REG3 = 1e-4;              // :55
constexpr double QUAD_WH = 4.479906037125444;   // sqrt(mass*g/(4 k_F)) = sqrt(0.5*9.81/(0.0611*4)), :62
constexpr int QNOB = 5;
// The solver kernel runs a problem in a CTA of min(round32(N+1), QUAD_CTA) threads; thread t handles the stages t, t + QUAD_CTA,
// ...  The horizon is bounded so that a thread handles at most four stages (N + 1 <= 512).
constexpr int QUAD_CTA = 128;
constexpr int QUAD_NMAX = 4 * QUAD_CTA - 1;

struct QuadProblem {
  int N;          // the horizon the batch's arrays and the workspace are laid out for (the largest of a mixed batch)
  double Ts, R;   // Ts: the batch's sampling time when it has one; each problem's own horizon and Ts are in QCtx
  double obs[QNOB][6];
  double xlo[QNX], xhi[QNX];   // :78-93 (x10 bounds differ between the variants, QuadcopterDist.jl:88)
  int signed_dist;
};

struct QLay {
  int NSP;
  int X, U, LAM, SLK;
  int ZXL, ZXU, ZUL, ZUU, ZLAM, ZSLK;
  int PI, YN, SD, VD;
  int dX, dU, dLAM, dSLK, PIn, YNn, dSD;
  int LF, nfac;
  int QS, qs, JV, R12, RK, RP;
  int total;
};

inline QLay make_qlayout(const QuadProblem& P) {
  QLay L;
  const int NS = P.N + 1;
  L.NSP = ((NS + 31) / 32) * 32;
  int c = 0;
  auto take = [&](int n) { int o = c; c += n; return o; };
  L.X = take(QNX); L.U = take(QNU); L.LAM = take(6 * QNOB); L.SLK = take(QNOB);
  L.ZXL = take(QNX); L.ZXU = take(QNX); L.ZUL = take(QNU); L.ZUU = take(QNU); L.ZLAM = take(6 * QNOB); L.ZSLK = take(QNOB);
  L.PI = take(QNX); L.YN = take(QNOB); L.SD = take(QNOB); L.VD = take(QNOB);
  L.dX = take(QNX); L.dU = take(QNU); L.dLAM = take(6 * QNOB); L.dSLK = take(QNOB); L.PIn = take(QNX); L.YNn = take(QNOB);
  L.dSD = take(QNOB);
  L.nfac = P.signed_dist ? QLocalDims<true>::NFAC : QLocalDims<false>::NFAC;
  L.LF = take(QNOB * L.nfac);
  L.QS = take(QNQ); L.qs = take(QNYV); L.JV = take(QD_NJ); L.R12 = take(QNX);
  L.RK = take(4 * 24); L.RP = take(QNX * QNSV + QNX);
  L.total = c;
  return L;
}

struct QInputs {
  const double* x0;    // 12
  const double* xF;    // 12
  const double* xWS;   // 12 x (N+1) column-major (QuadcopterSignedDist.jl:201: setvalue(x, xWS))
  double timeWS;       // :199
};
struct QOutputs {
  double *xp, *up, *ts, *lp, *slack;   // 12x(N+1), 4xN, (N+1), 30x(N+1), 5x(N+1) (:277-298)
};

struct QCtx {
  const QuadProblem* P;   // P->N, P->Ts: the horizon the batch's arrays are laid out for and the batch's sampling time
  int N;                  // horizon of this problem (<= P->N): every stage loop, the KKT sweep and the reductions run to it
  double Ts;              // sampling time of this problem
  const IpmOpts* O;
  QLay L;
  double* W;
  void* red_scratch;
  double* tile;
  ProbState* S;
  QInputs in;
#if !defined(__CUDACC__)
  QCtx() : N(0), Ts(0.0) {}   // host (development emulation): a context built without a horizon solves at P->N, P->Ts
#endif
};

// Problem, options and layout: __constant__ memory on the device (as for the parking model, obca_solver.cuh), the context on the host.
#if defined(__CUDACC__)
__constant__ QuadProblem c_qP;
__constant__ QLay c_qL;
#endif
#if defined(__CUDA_ARCH__)
#define QCTX_P(C) c_qP
#define QCTX_O(C) c_pkO
#define QCTX_L(C) c_qL
// the workspace is global memory: lets the compiler emit LDG / STG instead of generic accesses
#define QLOCALS(C) double* const W_ = (C).W; __builtin_assume(__isGlobal(W_)); (void)W_
#else
#define QCTX_P(C) (*(C).P)
#define QCTX_O(C) (*(C).O)
#define QCTX_L(C) ((C).L)
#define QLOCALS(C) double* const W_ = (C).W; (void)W_
#endif
// horizon and sampling time of the problem of context C.  The device kernel always sets both; on the host C.N = 0 stands for
// the layout's horizon and the batch's sampling time.
#if defined(__CUDA_ARCH__)
#define QCTX_N(C) ((C).N)
#define QCTX_TS(C) ((C).Ts)
#else
#define QCTX_N(C) ((C).N > 0 ? (C).N : (C).P->N)
#define QCTX_TS(C) ((C).N > 0 ? (C).Ts : (C).P->Ts)
#endif
#define QA(name, i, k) (W_[(size_t)(QCTX_L(C).name + (i)) * QCTX_L(C).NSP + (k)])

OBCA_HD void quad_jac_tables(const int*& jr, const int*& jc, const int*& hi, const int*& hj) {
  static constexpr int JR[QD_NJ] = OBCA_QD_J_ROW;
  static constexpr int JC[QD_NJ] = OBCA_QD_J_COL;
  static constexpr int HI[QD_NH] = OBCA_QD_H_I;
  static constexpr int HJ[QD_NH] = OBCA_QD_H_J;
  jr = JR; jc = JC; hi = HI; hj = HJ;
}

#ifdef OBCA_QPROF
__device__ unsigned long long g_qprof[8];   // development: cycles of the sweep's phases (thread 0 of every CTA)
#endif
template <bool SDV>
struct QuadSolver {
  typedef QCtx Ctx;
  typedef QLocalDims<SDV> LD;

  OBCA_HD static int n_stages(const QCtx& C) { return QCTX_N(C) + 1; }
#if defined(__CUDA_ARCH__)
  // warps that hold stages of the problem: ceil((N+1)/32), at most the CTA's (past QUAD_CTA stages every warp has some)
  __device__ static int own_warps(const QCtx& C) { return min((QCTX_N(C) + 32) >> 5, (int)(blockDim.x >> 5)); }
  // block reductions over the problem's own warps, so that a problem gives the same bits in a CTA sized for a longer horizon
  // of its batch as in one sized for its own
  template <typename T>
  __device__ static void reduce(T& v, const QCtx& C) { block_reduce_warps(v, C.red_scratch, own_warps(C)); }
#endif
  OBCA_HD static bool fixed_time(const QCtx&) { return false; }
  OBCA_HD static void mult_counts(const QCtx& C, double& n_mult, double& n_bmult) {
    const double N = QCTX_N(C), NS = N + 1;
    double nb = 24.0 * (N - 1) + 8.0 * N + 30.0 * NS + 2.0 * NS + (SDV ? 5.0 * NS : 0.0);   // variable bounds
    nb += 5.0 * NS;                                                                          // dist slack bounds
    n_bmult = nb; n_mult = nb + 12.0 * N + 5.0 * NS + 5.0 * NS;
  }
  OBCA_HD static void init_scalars(const QCtx& C, int restart) {
    ProbState& S = *C.S;
    S.t = push_lo(restart ? S.t : C.in.timeWS, 0.5, 2.0, QCTX_O(C).kappa1, QCTX_O(C).kappa2);   // :96, :199
    S.zTL = 1.0; S.zTU = 1.0; S.dt = 0.0;
  }
  OBCA_HD static void update_scalars(const QCtx& C) {
    ProbState& S = *C.S;
    double q = S.t, zl = S.zTL, zu = S.zTU;
    upd_pair(q, S.dt, zl, zu, 0.5, 2.0, S.alpha, S.a_du, S.mu, QCTX_O(C).kappa_sigma);
    S.t = q; S.zTL = zl; S.zTU = zu;
  }
  OBCA_HD static void ftb(double gap, double dgap, double tau, double& amax) {
    if (dgap < 0.0) amax = dmin_(amax, -tau * gap * rcp(dgap));
  }
  OBCA_HD static double dzb(double z, double gap, double dgap, double mu_b) { return (mu_b - z * dgap) * rcp(gap) - z; }
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

  OBCA_HD static void load_obs(const QCtx& C, int k, int o, QObsVars& Q, double alpha) {
    QLOCALS(C);
    qobs_load_const(Q, QCTX_P(C).obs[o]);
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      Q.lam[i] = QA(LAM, 6 * o + i, k) + (alpha != 0.0 ? alpha * QA(dLAM, 6 * o + i, k) : 0.0);
      Q.zlam[i] = QA(ZLAM, 6 * o + i, k);
    }
    Q.sl = SDV ? QA(SLK, o, k) + (alpha != 0.0 ? alpha * QA(dSLK, o, k) : 0.0) : 0.0;
    Q.zsl = SDV ? QA(ZSLK, o, k) : 0.0;
    Q.yn = QA(YN, o, k);
    Q.sd = QA(SD, o, k) + (alpha != 0.0 ? alpha * QA(dSD, o, k) : 0.0);
    Q.vd = QA(VD, o, k);
  }

  // ---- P0 ----
  OBCA_HD_NI static void init_stage(const QCtx& C, int k, int restart) {
    QLOCALS(C);
    const QuadProblem& P = QCTX_P(C);
    const IpmOpts& O = QCTX_O(C);
    const int N = QCTX_N(C);
    const bool free_x = (k >= 1 && k <= N - 1);
    for (int i = 0; i < QNX; ++i) {
      double v = restart ? QA(X, i, k) : C.in.xWS[(size_t)QNX * k + i];
      if (k == 0) v = C.in.x0[i];
      if (k == N) v = C.in.xF[i];
      if (free_x) v = push_lo(v, P.xlo[i], P.xhi[i], O.kappa1, O.kappa2);
      QA(X, i, k) = v; QA(ZXL, i, k) = 1.0; QA(ZXU, i, k) = 1.0; QA(PI, i, k) = 0.0;
    }
    for (int j = 0; j < QNU; ++j) {
      double v = restart ? QA(U, j, k) : QUAD_WH;                          // setvalue(u, w_H) (:202)
      QA(U, j, k) = k < N ? push_lo(v, 1.2, 7.8, O.kappa1, O.kappa2) : 0.0;
      QA(ZUL, j, k) = 1.0; QA(ZUU, j, k) = 1.0;
    }
    for (int o = 0; o < QNOB; ++o) {
      double lw[6];
      if (!restart) {
        if (QCTX_O(C).quad_dual_ws) {
          const double pos[3] = {QA(X, 0, k), QA(X, 1, k), QA(X, 2, k)};
          quad_dual_ws(pos, P.obs[o], lw);                                  // closed-form dual warm start
        } else {
          for (int r = 0; r < 6; ++r) lw[r] = 0.05;                         // setvalue(l, 0.05) (:204-208)
        }
      }
      for (int r = 0; r < 6; ++r) {
        QA(LAM, 6 * o + r, k) = dmax(restart ? QA(LAM, 6 * o + r, k) : lw[r], O.kappa1);
        QA(ZLAM, 6 * o + r, k) = 1.0;
      }
    }
    for (int o = 0; o < QNOB; ++o) {
      if (SDV) { QA(SLK, o, k) = dmax(restart ? QA(SLK, o, k) : 1.0, O.kappa1); QA(ZSLK, o, k) = 1.0; }   // slack = 1 (:210)
      QA(YN, o, k) = 0.0;
    }
  }
  OBCA_HD_NI static void init_slacks(const QCtx& C, int k) {
    QLOCALS(C);
    const QuadProblem& P = QCTX_P(C);
    double pos[3] = {QA(X, 0, k), QA(X, 1, k), QA(X, 2, k)};
    for (int o = 0; o < QNOB; ++o) {
      QObsVars Q; QObsGeom G;
      load_obs(C, k, o, Q, 0.0);
      Q.sd = 0.0;
      qobs_geom<SDV>(pos, Q, G);
      QA(SD, o, k) = dmax(G.gd, P.R + QCTX_O(C).kappa1 * dmax(1.0, dabs(P.R)));
      QA(VD, o, k) = 1.0;
    }
  }

  // ---- K1 ----
  OBCA_HD_NI static void stage_eval(const QCtx& C, int k, bool do_err, bool do_asm, EvalPart& out) {
    QLOCALS(C);
    const QuadProblem& P = QCTX_P(C);
    const ProbState& S = *C.S;
    const int N = QCTX_N(C);
    const double mu_b = S.mu, dw = S.dw, t = S.t;
    const bool free_x = (k >= 1 && k <= N - 1);
    const bool has_u = k < N;
    double e_dual = 0.0, e_pr = 0.0, cmax = 0.0, cmin = 1e300, sum_y = 0.0, sum_z = 0.0, th = 0.0, phi = 0.0, fobj = 0.0, rz_t = 0.0;
    int ok = 1;
    LogAcc lacc;
    double x[QNX], rzx[QNX];
    for (int i = 0; i < QNX; ++i) { x[i] = QA(X, i, k); rzx[i] = 0.0; }
    if (do_asm && has_u) {
      for (int e = 0; e < QNQ; ++e) QA(QS, e, k) = 0.0;
      for (int e = 0; e < QNYV; ++e) QA(qs, e, k) = 0.0;
    }
#define QQ(i, j) QA(QS, sym_idx_any<QNYV>((i), (j)), k)
#define Qq(i) QA(qs, (i), k)
    // ---- state objective + bounds ----
    fobj += QUAD_REG3 * (x[9] * x[9] + x[10] * x[10] + x[11] * x[11]);
    if (free_x) {
      for (int i = 0; i < QNX; ++i) {
        const double g = i >= 9 ? 2.0 * QUAD_REG3 * x[i] : 0.0;
        const double al = x[i] - P.xlo[i], au = P.xhi[i] - x[i];
        const double ial = rcp(al), iau = rcp(au);
        const double zl = QA(ZXL, i, k), zu = QA(ZXU, i, k);
        if (do_asm) {
          QQ(i, i) += (i >= 9 ? 2.0 * QUAD_REG3 : 0.0) + zl * ial + zu * iau + dw;
          Qq(i) += g - mu_b * ial + mu_b * iau;
        }
        rzx[i] += g - zl + zu + QA(PI, i, k - 1);
        if (do_err) {
          cmax = dmax(cmax, dmax(al * zl, au * zu)); cmin = dmin_(cmin, dmin_(al * zl, au * zu));
          sum_z += zl + zu;
          lacc.add(al); lacc.add(au);
        }
      }
    }
    // ---- controls + dynamics ----
    if (has_u) {
      double u[QNU], pi[QNX], c0[3] = {C.in.x0[9], C.in.x0[10], C.in.x0[11]};
      for (int i = 0; i < QNX; ++i) pi[i] = QA(PI, i, k);
      double rzu[QNU];
      for (int j = 0; j < QNU; ++j) {
        u[j] = QA(U, j, k);
        const double w = k > 0 ? QA(U, j, k - 1) : 0.0;
        const double eh = QUAD_WH - u[j], ed = k > 0 ? (w - u[j]) : 0.0;
        fobj += 1e-3 * eh * eh + 1e-2 * ed * ed;
        const double gu = -2e-3 * eh - 2e-2 * ed, gw = 2e-2 * ed;
        const double al = u[j] - 1.2, au = 7.8 - u[j], ial = rcp(al), iau = rcp(au);
        const double zl = QA(ZUL, j, k), zu = QA(ZUU, j, k);
        if (do_asm) {
          QQ(QIU + j, QIU + j) += 2e-3 + (k > 0 ? 2e-2 : 0.0) + zl * ial + zu * iau + dw;
          if (k > 0) { QQ(QIW + j, QIW + j) += 2e-2; QQ(QIW + j, QIU + j) += -2e-2; }
          Qq(QIU + j) += gu - mu_b * ial + mu_b * iau;
          Qq(QIW + j) += gw;
        }
        rzu[j] = gu - zl + zu;
        if (k + 1 < N) rzu[j] += 2e-2 * (u[j] - QA(U, j, k + 1));      // role as "previous control" of stage k+1
        if (do_err) {
          cmax = dmax(cmax, dmax(al * zl, au * zu)); cmin = dmin_(cmin, dmin_(al * zl, au * zu));
          sum_z += zl + zu;
          lacc.add(al); lacc.add(au);
        }
      }
      double f[QNX], Jv[QD_NJ], Hv[QD_NH];
      quad_dyn_full(x, u, t, QCTX_TS(C), c0, pi, f, Jv, Hv);
      const int *jr, *jc, *hi, *hj;
      quad_jac_tables(jr, jc, hi, hj);
      if (do_asm) {
        for (int e = 0; e < QD_NH; ++e) QQ(hi[e], hj[e]) += Hv[e];
        for (int e = 0; e < QD_NJ; ++e) QA(JV, e, k) = Jv[e];
      }
      for (int i = 0; i < QNX; ++i) {
        const double xn = (k + 1 == N) ? C.in.xF[i] : QA(X, i, k + 1);
        const double r = f[i] - xn;
        if (do_asm) QA(R12, i, k) = r;
        if (do_err) { e_pr = dmax(e_pr, dabs(r)); th += dabs(r); sum_y += dabs(pi[i]); }
      }
      // Lagrangian gradient: - J' pi
      for (int e = 0; e < QD_NJ; ++e) {
        const double v = pi[jr[e]] * Jv[e];
        const int c = jc[e];
        if (c < QNX) rzx[c] -= v;
        else if (c == QIT) rz_t -= v;
        else rzu[c - QIU] -= v;
      }
      if (do_err)
        for (int j = 0; j < QNU; ++j) e_dual = dmax(e_dual, dabs(rzu[j]));
    }
    // ---- obstacle blocks ----
    double pos[3] = {x[0], x[1], x[2]};
    for (int o = 0; o < QNOB; ++o) {
      QObsVars Q; QObsGeom G;
      load_obs(C, k, o, Q, 0.0);
      qobs_geom<SDV>(pos, Q, G);
      if (do_err) {
        double rl[6], rs, gx[3];
        qobs_lagr_grad<SDV>(Q, G, rl, rs, gx);
        rzx[0] += gx[0]; rzx[1] += gx[1]; rzx[2] += gx[2];
        for (int i = 0; i < 6; ++i) {
          e_dual = dmax(e_dual, dabs(rl[i]));
          const double cp = Q.lam[i] * Q.zlam[i];
          cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
          sum_z += Q.zlam[i];
          lacc.add(Q.lam[i]);
          fobj += QUAD_REG2 * Q.lam[i] * Q.lam[i];
        }
        if (SDV) {
          e_dual = dmax(e_dual, dabs(rs));
          const double cp = Q.sl * Q.zsl;
          cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
          sum_z += Q.zsl;
          lacc.add(Q.sl);
          fobj += 1e2 * Q.sl + 1e3 * Q.sl * Q.sl;
        }
        e_pr = dmax(e_pr, dmax(dabs(G.cn), dabs(G.cd)));
        th += dabs(G.cn) + dabs(G.cd);
        sum_y += dabs(Q.yn) + Q.vd; sum_z += Q.vd;
        const double cp = (Q.sd - P.R) * Q.vd;
        cmax = dmax(cmax, cp); cmin = dmin_(cmin, cp);
        lacc.add(Q.sd - P.R);
      }
      if (do_asm) {
        const int piv = qobs_choose_pivot(G);
        if (piv != 0) { qobs_swap(Q, piv); qobs_geom<SDV>(pos, Q, G); }
        double Sxx[6], rx3[3];
        ok &= qobs_condense<SDV>(P.R, Q, G, mu_b, dw, QCTX_O(C).dc, Sxx, rx3, &QA(LF, o * QCTX_L(C).nfac, k), QCTX_L(C).NSP);
        if (free_x && has_u) {
          QQ(0, 0) += Sxx[0]; QQ(0, 1) += Sxx[1]; QQ(0, 2) += Sxx[2]; QQ(1, 1) += Sxx[3]; QQ(1, 2) += Sxx[4]; QQ(2, 2) += Sxx[5];
          Qq(0) += rx3[0]; Qq(1) += rx3[1]; Qq(2) += rx3[2];
        }
      }
    }
    // ---- time scale: objective (N+1)(0.25 t + 5 t^2) (:68) and its N+1 bound pairs ----
    if (k == 0) {
      const double m = (double)(N + 1);
      const double gl = t - 0.5, gu = 2.0 - t, igl = rcp(gl), igu = rcp(gu);
      fobj += m * (0.25 * t + 5.0 * t * t);
      if (do_asm) {
        QQ(QIT, QIT) += 10.0 * m + m * (S.zTL * igl + S.zTU * igu) + m * dw;   // N+1 copies of timeScale, each regularised
        Qq(QIT) += m * (0.25 + 10.0 * t) + m * (-mu_b * igl + mu_b * igu);
      }
      if (do_err) {
        rz_t += m * (0.25 + 10.0 * t) - m * (S.zTL - S.zTU);
        cmax = dmax(cmax, dmax(gl * S.zTL, gu * S.zTU)); cmin = dmin_(cmin, dmin_(gl * S.zTL, gu * S.zTU));
        sum_z += m * (S.zTL + S.zTU);
        phi -= m * mu_b * (log(gl) + log(gu));
      }
    }
    if (do_err) phi -= mu_b * lacc.total();
    if (do_err && free_x)
      for (int i = 0; i < QNX; ++i) e_dual = dmax(e_dual, dabs(rzx[i]));
    out.e_dual = e_dual; out.e_pr = e_pr; out.cmax = cmax; out.cmin = cmin; out.sy = sum_y; out.sz = sum_z;
    out.th = th; out.phi = phi + fobj; out.rt = rz_t; out.f = fobj; out.ok = ok;
#undef QQ
#undef Qq
  }

  // ---- K3: dense Riccati sweep over [x | w | t] (17) with 4 controls, run by one thread ----
  OBCA_HD static int kkt_dense(const QCtx& C) {
    QLOCALS(C);
    ProbState& S = *C.S;
    const int N = QCTX_N(C);
    const int *jr, *jc, *hi, *hj;
    quad_jac_tables(jr, jc, hi, hj);
    double P[QNSV][QNSV], p[QNSV];
    for (int a = 0; a < QNSV; ++a) { p[a] = 0.0; for (int b = 0; b < QNSV; ++b) P[a][b] = 0.0; }
    const double rho = 1.0 / QCTX_O(C).dc;
    for (int i = 0; i < QNX; ++i) { P[i][i] = rho; p[i] = -QA(PI, i, N - 1); }
    int ok = 1;
    for (int k = N - 1; k >= 0 && ok; --k) {
      // rows 0..11 of P_{k+1}, p_{k+1} for the multiplier recovery
      for (int i = 0; i < QNX; ++i) {
        for (int l = 0; l < QNSV; ++l) QA(RP, i * QNSV + l, k + 1) = P[i][l];
        QA(RP, QNX * QNSV + i, k + 1) = p[i];
      }
      double Jv[QD_NJ], r12[QNX];
      for (int e = 0; e < QD_NJ; ++e) Jv[e] = QA(JV, e, k);
      for (int i = 0; i < QNX; ++i) r12[i] = QA(R12, i, k);
      // g = p + P r~ ;  T = P Phi
      double g[QNSV], T[QNSV][QNYV];
      for (int a = 0; a < QNSV; ++a) {
        double acc = p[a];
        for (int l = 0; l < QNX; ++l) acc += P[a][l] * r12[l];
        g[a] = acc;
        for (int c = 0; c < QNYV; ++c) T[a][c] = 0.0;
        for (int e = 0; e < QD_NJ; ++e) T[a][jc[e]] += P[a][jr[e]] * Jv[e];
        for (int j = 0; j < QNU; ++j) T[a][QIU + j] += P[a][QIW + j];
        T[a][QIT] += P[a][QIT];
      }
      // H = Q + Phi' T (full), hv = q + Phi' g
      double H[QNYV][QNYV], hv[QNYV];
      for (int a = 0; a < QNYV; ++a) {
        hv[a] = QA(qs, a, k);
        for (int b = 0; b < QNYV; ++b) H[a][b] = QA(QS, sym_idx_any<QNYV>(a, b), k);
      }
      for (int e = 0; e < QD_NJ; ++e) {
        const int c = jc[e], r = jr[e];
        const double v = Jv[e];
        hv[c] += v * g[r];
        for (int b = 0; b < QNYV; ++b) H[c][b] += v * T[r][b];
      }
      for (int j = 0; j < QNU; ++j) {
        hv[QIU + j] += g[QIW + j];
        for (int b = 0; b < QNYV; ++b) H[QIU + j][b] += T[QIW + j][b];
      }
      hv[QIT] += g[QIT];
      for (int b = 0; b < QNYV; ++b) H[QIT][b] += T[QIT][b];
      // Cholesky of Huu (4x4), must be positive definite
      double Lc[QNU][QNU];
      for (int a = 0; a < QNU; ++a) {
        for (int b = 0; b <= a; ++b) {
          double acc = H[QIU + a][QIU + b];
          for (int l = 0; l < b; ++l) acc -= Lc[a][l] * Lc[b][l];
          if (a == b) {
            if (!(acc > 0.0)) { ok = 0; acc = 1e300; }
            Lc[a][a] = sqrt(acc);
          } else {
            Lc[a][b] = acc / Lc[b][b];
          }
        }
      }
      if (!ok) break;
      // K = -Huu^{-1} Hus (4x17), kf = -Huu^{-1} hu
      double K[QNU][QNSV + 1];
      for (int c = 0; c <= QNSV; ++c) {
        double y4[QNU];
        for (int a = 0; a < QNU; ++a) {
          double acc = c < QNSV ? H[QIU + a][c] : hv[QIU + a];
          for (int l = 0; l < a; ++l) acc -= Lc[a][l] * y4[l];
          y4[a] = acc / Lc[a][a];
        }
        for (int a = QNU - 1; a >= 0; --a) {
          double acc = y4[a];
          for (int l = a + 1; l < QNU; ++l) acc -= Lc[l][a] * K[l][c];
          K[a][c] = acc / Lc[a][a];
        }
        for (int a = 0; a < QNU; ++a) K[a][c] = -K[a][c];
      }
      for (int a = 0; a < QNU; ++a) {
        for (int c = 0; c < QNSV; ++c) QA(RK, a * QNSV + c, k) = K[a][c];
        QA(RK, QNU * QNSV + a, k) = K[a][QNSV];
      }
      for (int a = 0; a < QNSV; ++a) {
        double acc = hv[a];
        for (int l = 0; l < QNU; ++l) acc += H[a][QIU + l] * K[l][QNSV];
        p[a] = acc;
        for (int b = a; b < QNSV; ++b) {
          double v = H[a][b];
          for (int l = 0; l < QNU; ++l) v += H[a][QIU + l] * K[l][b];
          P[a][b] = v; P[b][a] = v;
        }
      }
    }
    if (!ok) return 0;
    double ptt = P[QIT][QIT];
    if (!(ptt > 0.0)) return 0;
    const double dt = -p[QIT] / ptt;
    S.dt = dt;
    // forward roll-out
    double s[QNSV];
    for (int a = 0; a < QNSV; ++a) s[a] = 0.0;
    s[QIT] = dt;
    for (int k = 0; k < N; ++k) {
      double u[QNU];
      for (int a = 0; a < QNU; ++a) {
        double acc = QA(RK, QNU * QNSV + a, k);
        for (int c = 0; c < QNSV; ++c) acc += QA(RK, a * QNSV + c, k) * s[c];
        u[a] = acc;
        QA(dU, a, k) = acc;
      }
      double sn[QNX];
      for (int i = 0; i < QNX; ++i) sn[i] = QA(R12, i, k);
      for (int e = 0; e < QD_NJ; ++e) {
        const int c = jc[e];
        const double yv = c < QNSV ? s[c] : u[c - QIU];
        sn[jr[e]] += QA(JV, e, k) * yv;
      }
      for (int i = 0; i < QNX; ++i) {
        if (k + 1 < N) QA(dX, i, k + 1) = sn[i];
        else S.eNq[i] = sn[i];
        s[i] = sn[i];
      }
      for (int a = 0; a < QNU; ++a) s[QIW + a] = u[a];
    }
    for (int i = 0; i < QNX; ++i) { QA(dX, i, 0) = 0.0; QA(dX, i, N) = 0.0; }
    for (int a = 0; a < QNU; ++a) QA(dU, a, N) = 0.0;
    return 1;
  }
  // the KKT solve of an iteration, skipped (0) when the local blocks already failed the inertia test.  All threads call it;
  // the result is valid in thread 0, which may write S as soon as it returns.  Device: the block-cooperative sweep
  // (kkt_solve_block); host: kkt_dense.
  OBCA_HD static int factor(const QCtx& C) {
#if defined(__CUDA_ARCH__)
    const int ok = C.S->ok;      // uniform: S.ok was published before the last barrier
    __syncthreads();             // every thread has read it before thread 0 updates it (phase_B_serial)
    return ok ? kkt_solve_block(C) : 0;
#else
    return C.S->ok ? kkt_dense(C) : 0;
#endif
  }
  // prof[0..5]: clock64 cycles of the driver's phases (eval, kkt, recover, merit, update, serial)
  static constexpr bool PROF_CYCLES = true;
  static constexpr int STG_N = QNQ + QNYV + QD_NJ + QNX;     // per-stage data of the sweep: Q 231 | q 21 | Jv 66 | r 12
  // shared-memory layout of the tensor-core sweep (kkt_solve_block below)
  static constexpr int V2_LDP = 20, V2_LDF = 24, V2_LDT = 24, V2_LDQ = 24, V2_LDH = 28, V2_LDK = 24;
  static constexpr int V2_FSZ = 20 * V2_LDF, V2_QSZ = 24 * V2_LDQ;
  static constexpr int V2_P = 0, V2_p = V2_P + 24 * V2_LDP, V2_F = V2_p + 24, V2_Q = V2_F + 2 * V2_FSZ, V2_T = V2_Q + 2 * V2_QSZ,
                       V2_H = V2_T + 20 * V2_LDT, V2_K = V2_H + 24 * V2_LDH, V2_y = V2_K + 4 * V2_LDK, V2_flag = V2_y + 24,
                       V2_TOTAL = V2_flag + 2;
  static constexpr int V2_KG = 4 * V2_LDK;          // gains of one stage in global memory (dense 4 x 24)
  static constexpr int V2_FD = 4, V2_SLOT = V2_KG + QD_NJ + QNX + 2;     // forward ring: [K 96 | Jv 66 | r 12 | pad]
  static_assert(V2_FD * V2_SLOT <= 2 * V2_QSZ, "forward ring must fit into the Q buffers");
  static_assert((V2_F % 2) == 0 && (V2_Q % 2) == 0 && (V2_T % 2) == 0 && (V2_H % 2) == 0 && (V2_K % 2) == 0, "16-byte alignment");

  OBCA_HD static int smem_doubles(int) { return V2_TOTAL; }

#if defined(__CUDA_ARCH__)
#ifdef OBCA_QPROF
#define QPROF(i) do { if (threadIdx.x == 0) { long long t_ = clock64(); qacc[i] += t_ - qt; qt = t_; } } while (0)
#else
#define QPROF(i) do { } while (0)
#endif
  // -------------------------------------------------------------------------------------------------
  // Device version: the whole CTA cooperates on every stage of the backward sweep; the three matrix steps of a stage run on the
  // FP64 tensor cores (mma.sync m8n8k4, SASS DMMA).
  // All operands are dense, zero-padded tiles in shared memory:
  //   P    24 x 20   value function of stage k+1 (rows / columns >= 17 are zero)
  //   F    20 x 24   [ Phi | r~ ]: the dynamics Jacobian scattered to its dense positions, the identity rows of w+ = u and t+ = t,
  //                  and the dynamics residual as column 21                       (double buffered, filled by cp.async)
  //   Q    24 x 24   stage Hessian (upper triangle) with the stage gradient as column 21   (double buffered, cp.async)
  //   T  = P F  (+ p on column 21)           9 tiles x 5 k-steps
  //   H  = Q + F' T                           6 upper tiles x 5 k-steps;   column 21 of H is the gradient hv = q + Phi'(p + P r~)
  //   K  = -Huu^{-1} [Hus | hu]               18 threads, LDL' of the 4x4 pivot block (inertia test); feed-forward as column 21
  //   P' = Hss + Hsu K                        6 upper tiles x 1 k-step, mirrored;   column 21 is the new p
  // so the gradient recursion rides along as one more column of the same products.  Same elimination as kkt_dense().
  // Four barriers per stage.  The gains go to global memory ([stage][4 x 24], contiguous) and come back through a four-deep cp.async
  // ring in the forward roll-out (warp 0), together with the Jacobian values and residuals of the stage.
  // -------------------------------------------------------------------------------------------------
  __device__ static __forceinline__ void dmma(double& d0, double& d1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n" : "+d"(d0), "+d"(d1) : "d"(a), "d"(b));
  }
  // shared-memory destination of element e of the per-stage record [Q 231 | q 21 | Jv 66 | r 12]: offset inside buffer 0 and
  // the distance to the same element in buffer 1
  __device__ static __forceinline__ void v2_dst(int e, int& off, int& bstride) {
    const int *jr, *jc, *hi, *hj;
    quad_jac_tables(jr, jc, hi, hj);
    if (e < QNQ) {
      int i = 0, r = e;
      while (r >= QNYV - i) { r -= QNYV - i; ++i; }
      off = V2_Q + i * V2_LDQ + (i + r); bstride = V2_QSZ;
    } else if (e < QNQ + QNYV) {
      off = V2_Q + (e - QNQ) * V2_LDQ + 21; bstride = V2_QSZ;
    } else if (e < QNQ + QNYV + QD_NJ) {
      const int q = e - QNQ - QNYV;
      off = V2_F + jr[q] * V2_LDF + jc[q]; bstride = V2_FSZ;
    } else {
      off = V2_F + (e - QNQ - QNYV - QD_NJ) * V2_LDF + 21; bstride = V2_FSZ;
    }
  }
  static constexpr int QPROF_N = 7;
  __device__ __noinline__ static int kkt_solve_block(const QCtx& C) {
    QLOCALS(C);
    extern __shared__ __align__(16) double obca_dyn_smem[];      // == C.tile; named here so that the accesses are LDS / STS
#ifdef OBCA_QPROF
    long long qacc[8] = {0, 0, 0, 0, 0, 0, 0, 0}, qt = clock64();
#endif
    ProbState& S = *C.S;
    const int N = QCTX_N(C);
    const int tid = threadIdx.x, nt = blockDim.x;
    const int lane = tid & 31, warp = tid >> 5, nwarp = nt >> 5;
    const int gid = lane >> 2, tig = lane & 3;
    double* const sm = obca_dyn_smem;
    double *const Pm = sm + V2_P, *const pv = sm + V2_p, *const Tm = sm + V2_T, *const Hm = sm + V2_H, *const Km = sm + V2_K, *const yv = sm + V2_y;
    static constexpr int JC[QD_NJ] = OBCA_QD_J_COL;
    static constexpr int RPT[QNX + 1] = OBCA_QD_ROW_PTR;
    const double rho = 1.0 / QCTX_O(C).dc;
    const size_t nsp = (size_t)QCTX_L(C).NSP;
    const double* const gQ = W_ + (size_t)QCTX_L(C).QS * nsp;     // QS, qs, JV, R12 are consecutive arrays of the workspace
    double* const gK = W_ + (size_t)QCTX_L(C).RK * nsp;           // gains, [stage][4 x 24]
    double* const gRP = W_ + (size_t)QCTX_L(C).RP * nsp;
    // ---- per-thread constants of the stage prefetch: issued by the upper half of the warps (they have one tile of the
    //      value-function update, the lower half two); six elements per thread when the CTA has four warps ----
    constexpr int PFN = 6;
    const int pf_w0 = nwarp >= 2 ? nwarp / 2 : 0;                  // first prefetching warp
    const int pf_nt = nt - pf_w0 * 32, pf_tid = tid - pf_w0 * 32;  // prefetching threads, this thread's index among them
    const bool pf_fast = (pf_nt * PFN >= STG_N);
    const double* pf_src[PFN];
    int pf_off[PFN], pf_bs[PFN];
#pragma unroll
    for (int i = 0; i < PFN; ++i) {
      const int e = pf_tid + i * pf_nt;
      const bool on = pf_tid >= 0 && e < STG_N;
      pf_src[i] = gQ + (size_t)(on ? e : 0) * nsp;
      pf_off[i] = -1; pf_bs[i] = 0;
      if (on) v2_dst(e, pf_off[i], pf_bs[i]);
    }
    auto prefetch = [&](int k) {      // stage k -> buffer k & 1
      if (k >= 0 && pf_tid >= 0) {
        const int buf = k & 1;
        if (pf_fast) {
#pragma unroll
          for (int i = 0; i < PFN; ++i)
            if (pf_off[i] >= 0) cp_async8(sm + pf_off[i] + buf * pf_bs[i], pf_src[i] + k);
        } else {
          for (int e = pf_tid; e < STG_N; e += pf_nt) {
            int off, bs;
            v2_dst(e, off, bs);
            cp_async8(sm + off + buf * bs, gQ + (size_t)e * nsp + k);
          }
        }
      }
      cp_async_commit();
    };
    // rows 0..11 of P_{k+1} and p_{k+1} go to global memory for the multiplier recovery: stored during the gain phase by the
    // warps that have no gain column (all of them but warp 0 when there are several)
    const int rp_t0 = nwarp >= 2 ? 32 : 0, rp_nt = nt - rp_t0;
    constexpr int RPN = 3;                                          // 216 values / 96 threads
    const bool rp_fast = (rp_nt * RPN >= QNX * QNSV + QNX);
    double* rp_dst[RPN];
    int rp_src[RPN];
#pragma unroll
    for (int i = 0; i < RPN; ++i) {
      const int e = (tid - rp_t0) + i * rp_nt;
      const bool on = tid >= rp_t0 && e < QNX * QNSV + QNX;
      rp_dst[i] = gRP + (size_t)(on ? e : 0) * nsp;
      rp_src[i] = !on ? -1 : (e < QNX * QNSV ? V2_P + (e / QNSV) * V2_LDP + (e % QNSV) : V2_p + (e - QNX * QNSV));
    }
    // ---- initial contents: zeros, the constant entries of F, the terminal value function ----
    for (int e = tid; e < V2_TOTAL; e += nt) sm[e] = 0.0;
    __syncthreads();
    if (tid < 2 * (QNU + 1)) {
      const int buf = tid / (QNU + 1), j = tid % (QNU + 1);
      double* F = sm + V2_F + buf * V2_FSZ;
      if (j < QNU) F[(QIW + j) * V2_LDF + QIU + j] = 1.0;      // w+ = u
      else F[QIT * V2_LDF + QIT] = 1.0;                        // t+ = t
    }
    for (int i = tid; i < QNX; i += nt) { Pm[i * V2_LDP + i] = rho; pv[i] = -QA(PI, i, N - 1); }
    if (tid == 0) sm[V2_flag] = 1.0;
    prefetch(N - 1);
    for (int k = N - 1; k >= 0; --k) {
      const double* const Fb = sm + V2_F + (k & 1) * V2_FSZ;
      const double* const Qb = sm + V2_Q + (k & 1) * V2_QSZ;
      prefetch(k - 1);
      QPROF(0);
      cp_async_wait<1>();
      __syncthreads();                     // stage data landed; P, p of stage k+1 final
      QPROF(1);
      // ---- T = P F (+ p on column 21): tiles idx = warp, warp + nwarp, ... of the 3 x 3 grid ----
      for (int idx = warp; idx < 9; idx += nwarp) {
        const int m = idx / 3, n = idx % 3;
        double c0 = 0.0, c1 = 0.0;
        const double* const ap = Pm + (m * 8 + gid) * V2_LDP + tig;
        const double* const bp = Fb + tig * V2_LDF + n * 8 + gid;
#pragma unroll
        for (int ks = 0; ks < 5; ++ks) dmma(c0, c1, ap[ks * 4], bp[ks * 4 * V2_LDF]);
        const int row = m * 8 + gid;
        if (row < 20) {
          if (n == 2 && tig == 2) c1 += pv[row];
          *reinterpret_cast<double2*>(Tm + row * V2_LDT + n * 8 + tig * 2) = make_double2(c0, c1);
        }
      }
      __syncthreads();
      QPROF(2);
      // ---- H = Q + F' T: the six upper tiles ----
      for (int idx = warp; idx < 6; idx += nwarp) {
        const int m = idx < 3 ? 0 : (idx < 5 ? 1 : 2), n = idx < 3 ? idx : (idx < 5 ? idx - 2 : 2);
        const double2 q2 = *reinterpret_cast<const double2*>(Qb + (m * 8 + gid) * V2_LDQ + n * 8 + tig * 2);
        double c0 = q2.x, c1 = q2.y;
        const double* const ap = Fb + tig * V2_LDF + m * 8 + gid;
        const double* const bp = Tm + tig * V2_LDT + n * 8 + gid;
#pragma unroll
        for (int ks = 0; ks < 5; ++ks) dmma(c0, c1, ap[ks * 4 * V2_LDF], bp[ks * 4 * V2_LDT]);
        *reinterpret_cast<double2*>(Hm + (m * 8 + gid) * V2_LDH + n * 8 + tig * 2) = make_double2(c0, c1);
      }
      __syncthreads();
      QPROF(3);
      // ---- K = -Huu^{-1} [Hus | hu]: column c = 0..17 (17: the feed-forward, stored as column 21), one thread per column, each with its
      //      own LDL' of the 4x4 pivot block (inertia test: all pivots positive) -- 18 short dependent chains side by side instead of one
      //      factorisation followed by a hand-over.  Meanwhile the other warps store rows 0..11 of P_{k+1} for the multiplier recovery. ----
      if (tid <= QNSV) {
        const int c = tid;
        double Lm[QNU][QNU], dd[QNU], di[QNU];      // unit lower factor, pivots d and 1/d
        int ok = 1;
#pragma unroll
        for (int a = 0; a < QNU; ++a) {
#pragma unroll
          for (int b = 0; b < a; ++b) {
            double acc = Hm[(QIU + b) * V2_LDH + QIU + a];
#pragma unroll
            for (int l = 0; l < b; ++l) acc -= Lm[a][l] * Lm[b][l] * dd[l];
            Lm[a][b] = acc * di[b];
          }
          double d = Hm[(QIU + a) * V2_LDH + QIU + a];
#pragma unroll
          for (int l = 0; l < a; ++l) d -= Lm[a][l] * Lm[a][l] * dd[l];
          if (!(d > 0.0)) { ok = 0; d = 1e300; }
          dd[a] = d; di[a] = __drcp_rn(d);
        }
        if (!ok && tid == 0) sm[V2_flag] = 0.0;
        double y4[QNU], k4[QNU];
#pragma unroll
        for (int a = 0; a < QNU; ++a) {
          double acc = c < QNSV ? Hm[c * V2_LDH + QIU + a] : Hm[(QIU + a) * V2_LDH + 21];
#pragma unroll
          for (int l = 0; l < a; ++l) acc -= Lm[a][l] * y4[l];
          y4[a] = acc;
        }
#pragma unroll
        for (int a = QNU - 1; a >= 0; --a) {
          double acc = y4[a] * di[a];
#pragma unroll
          for (int l = a + 1; l < QNU; ++l) acc -= Lm[l][a] * k4[l];
          k4[a] = acc;
        }
        const int col = c < QNSV ? c : 21;
        double* const kg = gK + (size_t)k * V2_KG + col;
#pragma unroll
        for (int a = 0; a < QNU; ++a) { Km[a * V2_LDK + col] = -k4[a]; kg[a * V2_LDK] = -k4[a]; }
      }
      if (tid >= rp_t0) {      // P, p of stage k+1 (unchanged since the top of the stage) for the multiplier recovery
        if (rp_fast) {
#pragma unroll
          for (int i = 0; i < RPN; ++i)
            if (rp_src[i] >= 0) rp_dst[i][k + 1] = sm[rp_src[i]];
        } else {
          for (int e = tid - rp_t0; e < QNX * QNSV + QNX; e += rp_nt)
            gRP[(size_t)e * nsp + k + 1] = e < QNX * QNSV ? Pm[(e / QNSV) * V2_LDP + (e % QNSV)] : pv[e - QNX * QNSV];
        }
      }
      __syncthreads();
      QPROF(4);
      if (sm[V2_flag] == 0.0) { cp_async_wait<0>(); return 0; }
      // ---- value function of stage k: P = Hss + Hsu K on the six upper tiles (one DMMA each), mirrored; column 21 is p ----
      for (int idx = warp; idx < 6; idx += nwarp) {
        const int m = idx < 3 ? 0 : (idx < 5 ? 1 : 2), n = idx < 3 ? idx : (idx < 5 ? idx - 2 : 2);
        const double* const hrow = Hm + (m * 8 + gid) * V2_LDH;
        const double2 h2 = *reinterpret_cast<const double2*>(hrow + n * 8 + tig * 2);
        double c0 = h2.x, c1 = h2.y;
        dmma(c0, c1, hrow[QIU + tig], Km[tig * V2_LDK + n * 8 + gid]);
        const int a = m * 8 + gid, b = n * 8 + tig * 2;
        if (a < QNSV) {
          if (b < QNSV && a <= b) { Pm[a * V2_LDP + b] = c0; Pm[b * V2_LDP + a] = c0; }
          if (b + 1 < QNSV && a <= b + 1) { Pm[a * V2_LDP + b + 1] = c1; Pm[(b + 1) * V2_LDP + a] = c1; }
          if (b + 1 == 21) pv[a] = c1;
        }
      }
    }
    cp_async_wait<0>();
    __syncthreads();
    QPROF(5);
    // root
    if (tid == 0) {
      const double ptt = Pm[QIT * V2_LDP + QIT];
      if (!(ptt > 0.0)) sm[V2_flag] = 0.0;
      else S.dt = -pv[QIT] / ptt;
    }
    __syncthreads();
    if (sm[V2_flag] == 0.0) return 0;
    // ---- forward roll-out: warp 0 alone; gains, Jacobian values and residuals of the next stages arrive through a ring ----
    if (tid < 32) {
      double* const ring = sm + V2_Q;
      const double* const gJ = gQ + (size_t)(QNQ + QNYV) * nsp;       // Jv | r
      auto pf = [&](int k) {
        if (k < N) {
          double* const slot = ring + (k % V2_FD) * V2_SLOT;
          for (int i = lane; i < V2_KG / 2; i += 32) cp_async16(slot + 2 * i, gK + (size_t)k * V2_KG + 2 * i);
          for (int e = lane; e < QD_NJ + QNX; e += 32) cp_async8(slot + V2_KG + e, gJ + (size_t)e * nsp + k);
        }
        cp_async_commit();
      };
      if (lane < 24) yv[lane] = (lane == QIT) ? S.dt : 0.0;
#pragma unroll
      for (int a = 0; a < V2_FD - 1; ++a) pf(a);
      __syncwarp();
      const int ua = lane >> 3, uj = lane & 7;
      // row `lane` of the dynamics Jacobian (CSR): first entry, number of entries (at most 9), columns -- in registers
      constexpr int RMAX = 9;
      const int rq0 = lane < QNX ? RPT[lane] : 0, rnq = lane < QNX ? RPT[lane + 1] - RPT[lane] : 0;
      int rcol[RMAX];
#pragma unroll
      for (int i = 0; i < RMAX; ++i) rcol[i] = i < rnq ? JC[rq0 + i] : 0;
      for (int k = 0; k < N; ++k) {
        pf(k + V2_FD - 1);
        cp_async_wait<V2_FD - 1>();
        __syncwarp();
        const double* const slot = ring + (k % V2_FD) * V2_SLOT;
        const double* const kr = slot + ua * V2_LDK;
        // u = kf + K s: eight lanes per control, three terms each, butterfly sum
        double part = kr[uj] * yv[uj] + kr[uj + 8] * yv[uj + 8];
        if (uj == 0) part += kr[16] * yv[16];
        part += __shfl_xor_sync(0xffffffffu, part, 1);
        part += __shfl_xor_sync(0xffffffffu, part, 2);
        part += __shfl_xor_sync(0xffffffffu, part, 4);
        const double uval = part + kr[21];
        if (uj == 0) { yv[QIU + ua] = uval; QA(dU, ua, k) = uval; }
        __syncwarp();
        const double* const Jv = slot + V2_KG;
        const double* const r12 = Jv + QD_NJ;
        double snv = 0.0;
        if (lane < QNX) {
          snv = r12[lane];
#pragma unroll
          for (int i = 0; i < RMAX; ++i)
            if (i < rnq) snv += Jv[rq0 + i] * yv[rcol[i]];
          if (k + 1 < N) QA(dX, lane, k + 1) = snv; else S.eNq[lane] = snv;
        }
        __syncwarp();
        if (lane < QNX) yv[lane] = snv;
        else if (lane < QNX + QNU) yv[lane] = yv[QIU + (lane - QNX)];      // w+ = u
        __syncwarp();
      }
      cp_async_wait<0>();
      for (int i = lane; i < QNX; i += 32) { QA(dX, i, 0) = 0.0; QA(dX, i, N) = 0.0; }
      if (lane < QNU) QA(dU, lane, N) = 0.0;
    }
    __syncthreads();
#ifdef OBCA_QPROF
    QPROF(6);
    if (threadIdx.x == 0) { for (int i = 0; i < QPROF_N; ++i) atomicAdd(&g_qprof[i], (unsigned long long)qacc[i]); atomicAdd(&g_qprof[7], 1ull); }
#endif
    return 1;
  }
#endif

  // ---- K4a ----
  OBCA_HD_NI static void recover_stage(const QCtx& C, int k, StepPart& out) {
    QLOCALS(C);
    const QuadProblem& P = QCTX_P(C);
    const ProbState& S = *C.S;
    const int N = QCTX_N(C);
    const double mu_b = S.mu, tau = S.tau;
    const bool free_x = (k >= 1 && k <= N - 1);
    double apr = 1.0, adu = 1.0, dphi = 0.0;
    if (k < N) {
      double sn[QNSV];
      for (int i = 0; i < QNX; ++i) sn[i] = (k + 1 < N) ? QA(dX, i, k + 1) : S.eNq[i];
      for (int a = 0; a < QNU; ++a) sn[QIW + a] = QA(dU, a, k);
      sn[QIT] = S.dt;
      for (int i = 0; i < QNX; ++i) {
        double acc = QA(RP, QNX * QNSV + i, k + 1);
        for (int l = 0; l < QNSV; ++l) acc += QA(RP, i * QNSV + l, k + 1) * sn[l];
        QA(PIn, i, k) = -acc;
      }
      for (int j = 0; j < QNU; ++j) {
        const double u = QA(U, j, k), du = QA(dU, j, k);
        const double w = k > 0 ? QA(U, j, k - 1) : 0.0, dwv = k > 0 ? QA(dU, j, k - 1) : 0.0;
        const double al = u - 1.2, au = 7.8 - u;
        ftb(al, du, tau, apr); ftb(au, -du, tau, apr);
        double z = QA(ZUL, j, k); ftb(z, dzb(z, al, du, mu_b), tau, adu);
        z = QA(ZUU, j, k); ftb(z, dzb(z, au, -du, mu_b), tau, adu);
        const double eh = QUAD_WH - u, ed = k > 0 ? (w - u) : 0.0;
        dphi += (-2e-3 * eh - 2e-2 * ed - mu_b * rcp(al) + mu_b * rcp(au)) * du + 2e-2 * ed * dwv;
      }
    }
    double x[QNX], dx[QNX];
    for (int i = 0; i < QNX; ++i) { x[i] = QA(X, i, k); dx[i] = QA(dX, i, k); }
    if (free_x) {
      for (int i = 0; i < QNX; ++i) {
        const double al = x[i] - P.xlo[i], au = P.xhi[i] - x[i];
        ftb(al, dx[i], tau, apr); ftb(au, -dx[i], tau, apr);
        double z = QA(ZXL, i, k); ftb(z, dzb(z, al, dx[i], mu_b), tau, adu);
        z = QA(ZXU, i, k); ftb(z, dzb(z, au, -dx[i], mu_b), tau, adu);
        dphi += ((i >= 9 ? 2.0 * QUAD_REG3 * x[i] : 0.0) - mu_b * rcp(al) + mu_b * rcp(au)) * dx[i];
      }
    }
    double pos[3] = {x[0], x[1], x[2]}, dpos[3] = {dx[0], dx[1], dx[2]};
    for (int o = 0; o < QNOB; ++o) {
      QObsVars Q; QObsGeom G;
      load_obs(C, k, o, Q, 0.0);
      qobs_geom<SDV>(pos, Q, G);
      const int piv = qobs_choose_pivot(G);
      if (piv != 0) { qobs_swap(Q, piv); qobs_geom<SDV>(pos, Q, G); }
      QObsStep St;
      qobs_recover<SDV>(P.R, Q, G, mu_b, &QA(LF, o * QCTX_L(C).nfac, k), QCTX_L(C).NSP, dpos, St);
      if (piv != 0) {
        for (int i = 1; i < 6; ++i)
          if (i == piv) {
            double tmp = St.dlam[0]; St.dlam[0] = St.dlam[i]; St.dlam[i] = tmp;
            tmp = Q.lam[0]; Q.lam[0] = Q.lam[i]; Q.lam[i] = tmp;
            tmp = Q.zlam[0]; Q.zlam[0] = Q.zlam[i]; Q.zlam[i] = tmp;
          }
      }
      for (int i = 0; i < 6; ++i) {
        QA(dLAM, 6 * o + i, k) = St.dlam[i];
        ftb(Q.lam[i], St.dlam[i], tau, apr);
        ftb(Q.zlam[i], dzb(Q.zlam[i], Q.lam[i], St.dlam[i], mu_b), tau, adu);
        dphi += (2.0 * QUAD_REG2 * Q.lam[i] - mu_b * rcp(Q.lam[i])) * St.dlam[i];
      }
      if (SDV) {
        QA(dSLK, o, k) = St.dsl;
        ftb(Q.sl, St.dsl, tau, apr);
        ftb(Q.zsl, dzb(Q.zsl, Q.sl, St.dsl, mu_b), tau, adu);
        dphi += (1e2 + 2e3 * Q.sl - mu_b * rcp(Q.sl)) * St.dsl;
      }
      QA(YNn, o, k) = St.yn_new;
      QA(dSD, o, k) = St.dsd;
      const double gap = Q.sd - P.R;
      ftb(gap, St.dsd, tau, apr);
      ftb(Q.vd, dzb(Q.vd, gap, St.dsd, mu_b), tau, adu);
      dphi += -mu_b * rcp(gap) * St.dsd;
    }
    if (k == 0) {
      const double m = (double)(N + 1), t = S.t;
      const double gl = t - 0.5, gu = 2.0 - t;
      ftb(gl, S.dt, tau, apr); ftb(gu, -S.dt, tau, apr);
      ftb(S.zTL, dzb(S.zTL, gl, S.dt, mu_b), tau, adu);
      ftb(S.zTU, dzb(S.zTU, gu, -S.dt, mu_b), tau, adu);
      dphi += m * (0.25 + 10.0 * t - mu_b * rcp(gl) + mu_b * rcp(gu)) * S.dt;
    }
    out.apr = apr; out.adu = adu; out.dphi = dphi;
  }

  // ---- K4b ----
  OBCA_HD_NI static void merit_stage(const QCtx& C, int k, double alpha, MeritPart& out) {
    QLOCALS(C);
    const QuadProblem& P = QCTX_P(C);
    const ProbState& S = *C.S;
    const int N = QCTX_N(C);
    const double mu_b = S.mu;
    const bool free_x = (k >= 1 && k <= N - 1);
    const double t = S.t + alpha * S.dt;
    double th = 0.0, phi = 0.0;
    bool bad = false;
    LogAcc lacc;
    double x[QNX];
    for (int i = 0; i < QNX; ++i) x[i] = QA(X, i, k) + alpha * QA(dX, i, k);
    phi += QUAD_REG3 * (x[9] * x[9] + x[10] * x[10] + x[11] * x[11]);
    if (free_x)
      for (int i = 0; i < QNX; ++i) {
        const double al = x[i] - P.xlo[i], au = P.xhi[i] - x[i];
        bad |= !(al > 0.0) || !(au > 0.0);
        lacc.add(al); lacc.add(au);
      }
    if (k < N) {
      double u[QNU], c0[3] = {C.in.x0[9], C.in.x0[10], C.in.x0[11]};
      for (int j = 0; j < QNU; ++j) {
        u[j] = QA(U, j, k) + alpha * QA(dU, j, k);
        const double w = k > 0 ? QA(U, j, k - 1) + alpha * QA(dU, j, k - 1) : 0.0;
        const double eh = QUAD_WH - u[j], ed = k > 0 ? (w - u[j]) : 0.0;
        phi += 1e-3 * eh * eh + 1e-2 * ed * ed;
        const double al = u[j] - 1.2, au = 7.8 - u[j];
        bad |= !(al > 0.0) || !(au > 0.0);
        lacc.add(al); lacc.add(au);
      }
      double f[QNX];
      quad_dyn_f(x, u, t, QCTX_TS(C), c0, f);
      for (int i = 0; i < QNX; ++i) {
        const double xn = (k + 1 == N) ? C.in.xF[i] : QA(X, i, k + 1) + alpha * QA(dX, i, k + 1);
        th += dabs(f[i] - xn);
      }
    }
    double pos[3] = {x[0], x[1], x[2]};
    for (int o = 0; o < QNOB; ++o) {
      QObsVars Q; QObsGeom G;
      load_obs(C, k, o, Q, alpha);
      qobs_geom<SDV>(pos, Q, G);
      th += dabs(G.cn) + dabs(G.cd);
      for (int i = 0; i < 6; ++i) {
        bad |= !(Q.lam[i] > 0.0);
        phi += QUAD_REG2 * Q.lam[i] * Q.lam[i]; lacc.add(Q.lam[i]);
      }
      if (SDV) { bad |= !(Q.sl > 0.0); phi += 1e2 * Q.sl + 1e3 * Q.sl * Q.sl; lacc.add(Q.sl); }
      const double gap = Q.sd - P.R;
      bad |= !(gap > 0.0);
      lacc.add(gap);
    }
    if (k == 0) {
      const double m = (double)(N + 1);
      const double gl = t - 0.5, gu = 2.0 - t;
      bad |= !(gl > 0.0) || !(gu > 0.0);
      phi += m * (0.25 * t + 5.0 * t * t) - m * mu_b * (log(gl) + log(gu));
    }
    phi -= mu_b * lacc.total();
    out.th = th;
    out.phi = bad ? 1e300 : phi;
  }

  // ---- K4c ----
  OBCA_HD_NI static void update_stage(const QCtx& C, int k) {
    QLOCALS(C);
    const QuadProblem& P = QCTX_P(C);
    const ProbState& S = *C.S;
    const int N = QCTX_N(C);
    const double mu_b = S.mu, ks = QCTX_O(C).kappa_sigma;
    const double alpha = S.alpha, adu = S.a_du, ay = dmin_(S.alpha, S.a_du);
    const bool free_x = (k >= 1 && k <= N - 1);
    if (free_x)
      for (int i = 0; i < QNX; ++i) {
        double q = QA(X, i, k), zl = QA(ZXL, i, k), zu = QA(ZXU, i, k);
        upd_pair(q, QA(dX, i, k), zl, zu, P.xlo[i], P.xhi[i], alpha, adu, mu_b, ks);
        QA(X, i, k) = q; QA(ZXL, i, k) = zl; QA(ZXU, i, k) = zu;
      }
    if (k < N) {
      for (int j = 0; j < QNU; ++j) {
        double q = QA(U, j, k), zl = QA(ZUL, j, k), zu = QA(ZUU, j, k);
        upd_pair(q, QA(dU, j, k), zl, zu, 1.2, 7.8, alpha, adu, mu_b, ks);
        QA(U, j, k) = q; QA(ZUL, j, k) = zl; QA(ZUU, j, k) = zu;
      }
      for (int i = 0; i < QNX; ++i) QA(PI, i, k) += ay * (QA(PIn, i, k) - QA(PI, i, k));
    }
    for (int r = 0; r < 6 * QNOB; ++r) {
      double q = QA(LAM, r, k), z = QA(ZLAM, r, k);
      const double dq = QA(dLAM, r, k);
      const double dz = dzb(z, q, dq, mu_b);
      q += alpha * dq; z += adu * dz;
      QA(LAM, r, k) = q; QA(ZLAM, r, k) = clipz(z, q, mu_b, ks);
    }
    for (int o = 0; o < QNOB; ++o) {
      if (SDV) {
        double q = QA(SLK, o, k), z = QA(ZSLK, o, k);
        const double dq = QA(dSLK, o, k);
        const double dz = dzb(z, q, dq, mu_b);
        q += alpha * dq; z += adu * dz;
        QA(SLK, o, k) = q; QA(ZSLK, o, k) = clipz(z, q, mu_b, ks);
      }
      QA(YN, o, k) += ay * (QA(YNn, o, k) - QA(YN, o, k));
      double s = QA(SD, o, k), z = QA(VD, o, k);
      const double ds = QA(dSD, o, k);
      const double dz = dzb(z, s - P.R, ds, mu_b);
      s += alpha * ds; z += adu * dz;
      QA(SD, o, k) = s; QA(VD, o, k) = clipz(z, s - P.R, mu_b, ks);
    }
  }

  // phase wrappers of the generic driver (the quadcopter model has no separate item pass: its 5 box blocks are evaluated
  // inside the stage functions)
  OBCA_HD static void eval_phase(const QCtx& C, bool do_err, EvalPart& ep) {
    const int NS = QCTX_N(C) + 1;
    OBCA_FOR_STAGES(k, NS) { EvalPart e1; stage_eval(C, k, do_err, true, e1); part_merge(ep, e1); }
  }
  OBCA_HD static void recover_phase(const QCtx& C, StepPart& sp) {
    const int NS = QCTX_N(C) + 1;
    OBCA_FOR_STAGES(k, NS) { StepPart s1; recover_stage(C, k, s1); part_merge(sp, s1); }
  }
  OBCA_HD static void merit_phase(const QCtx& C, double alpha, MeritPart& mp) {
    const int NS = QCTX_N(C) + 1;
    OBCA_FOR_STAGES(k, NS) { MeritPart m1; merit_stage(C, k, alpha, m1); part_merge(mp, m1); }
  }
  OBCA_HD static void update_phase(const QCtx& C) {
    const int NS = QCTX_N(C) + 1;
    OBCA_FOR_STAGES(k, NS) update_stage(C, k);
  }

  OBCA_HD static void store_stage(const QCtx& C, int k, const QOutputs& o) {
    QLOCALS(C);
    const int N = QCTX_N(C);
    for (int i = 0; i < QNX; ++i) o.xp[(size_t)QNX * k + i] = QA(X, i, k);
    if (k < N) for (int j = 0; j < QNU; ++j) o.up[(size_t)QNU * k + j] = QA(U, j, k);
    o.ts[k] = C.S->t;
    for (int r = 0; r < 6 * QNOB; ++r) o.lp[(size_t)6 * QNOB * k + r] = QA(LAM, r, k);      // lp = [l1; ...; l5] (:296)
    if (SDV && o.slack) for (int j = 0; j < QNOB; ++j) o.slack[(size_t)QNOB * k + j] = QA(SLK, j, k);
  }
};


// ------------------------------------------------------------------------------------------------------------
// K5 (quadcopter): twin of QuadcopterNavigation/constrSatisfaction.jl:25-204, restated verbatim: tolerance 1e-3,
// rows checked for i = 1..N only (:80), state box of the Dist variant ([-1.5, 3] on x10, :107,:119) for both
// variants, norm row one-sided (<= 0, :166-176), quirk Q5 in the body-rate rows (:151-153).
// x 12x(N+1), u 4xN, ts (N+1), lambda 30x(N+1) column-major.  N, Ts: the problem's own horizon and sampling time (P.N is the
// layout's horizon of a batch, P.Ts its shared sampling time).
// The reference tests groups: maximum(group) > tol, minimum(group) < -tol, norm(group, Inf) > tol.  A group that holds a NaN has a
// NaN maximum and never fails, but the other groups still decide.  So each group is reduced with dmax_nan and a NaN group
// contributes nothing.  Returns the largest contribution of stage k's groups: the start (k = 0) or end (k = N) state, and for
// k < N the four box groups (1.0 when violated: they fail at any violation), the 13 dynamics rows with the timeScale difference,
// the 5 norm rows and the 5 distance rows.  The lambda group (:162) spans every column of lambda; *lam gets column k's part of
// it, max(-lambda[:, k]) with NaN propagated, and the caller adds max(-lambda) over all columns unless it is NaN.
// (<= 1e-3 everywhere  <=>  the reference returns true.)
// ------------------------------------------------------------------------------------------------------------
OBCA_HD double quad_check_stage(const QuadProblem& P, int N, double Ts, int k, const double* x0, const double* xF, const double* x,
                                const double* u, const double* ts, const double* lam, double* lamk) {
  double worst = 0.0;
  const double* lk = lam + (size_t)30 * k;
  double ln = -lk[0];
  for (int r = 1; r < 30; ++r) ln = dmax_nan(ln, -lk[r]);
  *lamk = ln;
  const double* xk = x + (size_t)QNX * k;
  if (k == 0) {
    double g = dabs(xk[0] - x0[0]);
    for (int i = 1; i < QNX; ++i) g = dmax_nan(g, dabs(xk[i] - x0[i]));                          // :56-61
    if (g == g) worst = dmax(worst, g);
  }
  if (k == N) {
    double g = dabs(xk[0] - xF[0]);
    for (int i = 1; i < QNX; ++i) g = dmax_nan(g, dabs(xk[i] - xF[i]));                          // :63-68
    if (g == g) worst = dmax(worst, g);
    return worst;
  }
  const double* uk = u + (size_t)QNU * k;
  const double lo[QNX] = {0, 0, 0, -3, -0.2, -0.2, -1, -1, -1, -1.5, -1, -1};                       // :107
  const double hi[QNX] = {10, 10, 5, 3, 0.2, 0.2, 1, 1, 1, 3, 1, 1};                                // :119
  // the box groups are hard (> 0 fails, :83,:95,:108,:120): a violated one contributes 1.0, above the tolerance
  double gl = 1.2 - uk[0], gh = uk[0] - 7.8;
  for (int j = 1; j < QNU; ++j) { gl = dmax_nan(gl, 1.2 - uk[j]); gh = dmax_nan(gh, uk[j] - 7.8); }
  if (gl > 0.0 || gh > 0.0) worst = dmax(worst, 1.0);
  gl = lo[0] - xk[0]; gh = xk[0] - hi[0];
  for (int i = 1; i < QNX; ++i) { gl = dmax_nan(gl, lo[i] - xk[i]); gh = dmax_nan(gh, xk[i] - hi[i]); }
  if (gl > 0.0 || gh > 0.0) worst = dmax(worst, 1.0);
  double f[QNX];
  const double c0[3] = {x[9], x[10], x[11]};                                                         // linear indexing, :151-153
  quad_dyn_f(xk, uk, ts[k], Ts, c0, f);
  double g = dabs(x[(size_t)QNX * (k + 1)] - f[0]);
  for (int i = 1; i < QNX; ++i) g = dmax_nan(g, dabs(x[(size_t)QNX * (k + 1) + i] - f[i]));         // :127-153
  g = dmax_nan(g, dabs(ts[k] - ts[k + 1]));                                                          // :154
  if (g == g) worst = dmax(worst, g);
  double gn = -1e300, gd = -1e300;
  for (int o = 0; o < QNOB; ++o) {
    const double* l = lk + 6 * o;
    double bl = 0.0;
    for (int r = 0; r < 6; ++r) bl += P.obs[o][r] * l[r];
    const double p0 = l[0] - l[3], p1 = l[1] - l[4], p2 = l[2] - l[5];
    gn = dmax_nan(gn, p0 * p0 + p1 * p1 + p2 * p2 - 1.0);                                           // :171-182 (one-sided)
    // the distance row sums A[j, c] * l[j] over all six j (A = [I; -I]) like :185-194: equal to p on finite multipliers, NaN where an
    // infinite multiplier meets a zero of A
    double a[3];
    for (int c = 0; c < 3; ++c) {
      a[c] = 0.0;
      for (int r = 0; r < 6; ++r) a[c] += (r == c ? 1.0 : r == c + 3 ? -1.0 : 0.0) * l[r];
    }
    gd = dmax_nan(gd, -(-bl + xk[0] * a[0] + xk[1] * a[1] + xk[2] * a[2] - P.R));                   // :185-199
  }
  if (gn == gn) worst = dmax(worst, gn);
  if (gd == gd) worst = dmax(worst, gd);
  return worst;
}

}  // namespace obca
