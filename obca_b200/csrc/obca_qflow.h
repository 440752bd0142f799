// obca_qflow.h -- index maps and warm start of obca_quadcopter_plan_solve (include/obca.h), which plans, solves and checks a batch of
// quadcopter start / goal pairs without leaving the device.  The layouts are those of obca_flow.h with the quadcopter's rows:
//   planner  the outputs of the GPU 3-D A* (obca_plan3d.cu) with the stride cap per pair: rx / ry / rz [p*cap + k], on the 10x grid;
//   mixed    the per-problem arrays of obca_quadcopter_solve_mixed laid out for the horizon M: x0 / xF 12 per problem, xWS and the
//            outputs rows x (M+ext) column-major (obca_flow::out_entry);
//   caller   the outputs of the entry in pair order: the mixed layout with M = Ncap.
// The warm start is a_star_3d.plan_quadcopter_warm_start's (native.quadcopter_warm_start, mainQuadcopter.jl:130-137): xWS = the path
// / 10 in rows 0-2 and zeros in rows 3-11, Ts_as = jround(Ts * 80 / N * 100) / 100.  obca_lib.cu is built with FMA contraction, so the
// device side of that rounding uses the _rn intrinsics, which never contract; the host side (the argument check of the entry and a CPU
// test, tests/test_quad_plan_solve.py) is plain arithmetic.
#pragma once
#include <math.h>

#include "../../include/obca.h"
#include "obca_flow.h"

namespace obca_qflow {

using obca_flow::out_entry;
using obca_flow::plan_stage;

// jround(Ts * 80 / n * 100): the pair's sampling time in hundredths, Julia's round (ties away from zero), as a double.
OBCA_FHD double ts_hundredths(double Ts, int n) {
#ifdef __CUDA_ARCH__
  const double v = __dmul_rn(__ddiv_rn(__dmul_rn(Ts, 80.0), (double)n), 100.0);
  const double r = floor(__dadd_rn(fabs(v), 0.5));
#else
  const double v = Ts * 80.0 / (double)n * 100.0;
  const double r = floor(fabs(v) + 0.5);
#endif
  return v >= 0 ? r : -r;
}

// Ts_as of a pair planned to the horizon n
OBCA_FHD double warm_start_ts(double Ts, int n) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(ts_hundredths(Ts, n), 100.0);
#else
  return ts_hundredths(Ts, n) / 100.0;
#endif
}

OBCA_FHD double from_grid(double v) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(v, OBCA_QUAD_GRID_SCALE);
#else
  return v / OBCA_QUAD_GRID_SCALE;
#endif
}

// Gather: slot q of the solve, pair p, horizon n, stage k <= M of the mixed layout.  Stages past n are zero.  The stage-0 call also
// copies the pair's x0 and xF (12 values each: M can be 2, so fewer than twelve stages may exist) and writes the slot's Ts_as.
struct Gather {
  const double *rx, *ry, *rz;      // planner layout, stride cap
  const double *x0, *xF;           // 12 per pair
  double Ts;                       // the nominal sampling time
  double *mxWS, *mx0, *mxF, *mTsb;  // mixed layout at M: xWS 12 x (M+1), 12 and 1 per slot
};
OBCA_FHD void gather_stage(const Gather& g, int q, int p, int n, int k, int M, int cap) {
  const bool on = k <= n;
  const double* path[3] = {g.rx, g.ry, g.rz};
  for (int r = 0; r < 3; ++r) g.mxWS[out_entry(q, r, k, 12, M, 1)] = on ? from_grid(path[r][plan_stage(p, k, cap)]) : 0.0;
  for (int r = 3; r < 12; ++r) g.mxWS[out_entry(q, r, k, 12, M, 1)] = 0.0;
  if (k == 0) {
    for (int r = 0; r < 12; ++r) { g.mx0[12 * (size_t)q + r] = g.x0[12 * (size_t)p + r]; g.mxF[12 * (size_t)q + r] = g.xF[12 * (size_t)p + r]; }
    g.mTsb[q] = warm_start_ts(g.Ts, n);
  }
}

// The outputs of the entry: xp 12 x (M+1), up 4 x M, ts M+1, lp 30 x (M+1), slack 5 x (M+1) per problem, and one value per problem of
// the rest.  slack and worst may be null.
struct Outs {
  double *xp, *up, *ts, *lp, *slack, *kkt_err, *Tsb, *worst;
  int *exitflag, *iters, *feasible;
};
// Scatter: the outputs of slot q (mixed layout at M) to pair p (mixed layout at Ncap), stage k of the slot's horizon n.
OBCA_FHD void scatter_stage(const Outs& s, const Outs& d, int q, int p, int n, int k, int M, int Ncap) {
  obca_flow::scatter_rows(s.xp, d.xp, 12, 1, q, p, n, k, M, Ncap);
  obca_flow::scatter_rows(s.up, d.up, 4, 0, q, p, n, k, M, Ncap);
  obca_flow::scatter_rows(s.ts, d.ts, 1, 1, q, p, n, k, M, Ncap);
  obca_flow::scatter_rows(s.lp, d.lp, 30, 1, q, p, n, k, M, Ncap);
  obca_flow::scatter_rows(s.slack, d.slack, 5, 1, q, p, n, k, M, Ncap);
  if (k == 0) {
    d.exitflag[p] = s.exitflag[q]; d.iters[p] = s.iters[q]; d.kkt_err[p] = s.kkt_err[q]; d.feasible[p] = s.feasible[q];
    d.Tsb[p] = s.Tsb[q];
    if (d.worst) d.worst[p] = s.worst[q];
  }
}

}  // namespace obca_qflow
