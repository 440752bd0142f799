// obca_flow.h -- index maps of obca_parking_plan_solve_goals (include/obca.h), which plans, solves and checks a batch of start poses
// without leaving the device.  Three layouts meet there:
//   planner  the outputs of the GPU Hybrid A* (obca_plan.cu) with the stride cap per pose: rx / ry / ryaw [p*cap + k], xWS (n+1) x 4 at
//            [p*4*cap ..] and uWS n x 2 at [p*2*cap ..], column-major with the column strides n+1 and n (n: the pose's own horizon);
//   mixed    the per-problem arrays of obca_parking_solve_mixed laid out for the horizon M: rx [q*(M+1) + k], xWS (M+1) x 4 and uWS M x 2
//            column-major with the column strides M+1 and M; outputs rows x (M+ext) column-major, so problem q's own horizon n is the
//            prefix of rows * (n+ext) entries of its slice;
//   caller   the outputs of the entry in pose order: the mixed layout with M = Ncap.
// Host and device code: the kernels of obca_lib.cu and a CPU test (tests/test_plan_solve.py) run the same arithmetic.
#pragma once
#include <stddef.h>

#ifdef __CUDACC__
#define OBCA_FHD __host__ __device__ __forceinline__
#else
#define OBCA_FHD inline
#endif

namespace obca_flow {

// A pose is solved when it planned (status 0, OBCA_PLAN_OK) to a horizon the solver takes: 2 <= n <= Ncap.
OBCA_FHD bool listed(int status, int n, int Ncap) { return status == 0 && n >= 2 && n <= Ncap; }

// planner layout
OBCA_FHD size_t plan_stage(int p, int k, int cap) { return (size_t)p * cap + k; }
OBCA_FHD size_t plan_xws(int p, int c, int k, int n, int cap) { return (size_t)p * 4 * cap + (size_t)c * (n + 1) + k; }
OBCA_FHD size_t plan_uws(int p, int c, int k, int n, int cap) { return (size_t)p * 2 * cap + (size_t)c * n + k; }

// mixed layout at the horizon M
OBCA_FHD size_t mixed_stage(int q, int k, int M) { return (size_t)q * (M + 1) + k; }
OBCA_FHD size_t mixed_xws(int q, int c, int k, int M) { return (size_t)q * 4 * (M + 1) + (size_t)c * (M + 1) + k; }
OBCA_FHD size_t mixed_uws(int q, int c, int k, int M) { return (size_t)q * 2 * M + (size_t)c * M + k; }

// Entry (r, k) of problem q of an output with `rows` rows and M + ext columns (ext = 1 for stage arrays, 0 for the controls).
OBCA_FHD size_t out_entry(int q, int r, int k, int rows, int M, int ext) { return (size_t)q * rows * (M + ext) + (size_t)k * rows + r; }

// Gather: slot q of the solve, pose p, horizon n, stage k <= M of the mixed layout.  Stages past n are zero in the solve's inputs.  The
// stage-0 call also copies the pose's x0 and xF (4 values each): M can be 2, so fewer than four stages may exist.
struct Gather {
  const double *rx, *ry, *ryaw, *xWS, *uWS;      // planner layout, stride cap
  const double *x0, *xF;                         // 4 per pose
  double *mrx, *mry, *mryaw, *mxWS, *muWS;       // mixed layout at M
  double *mx0, *mxF;                             // 4 per slot
};
OBCA_FHD void gather_stage(const Gather& g, int q, int p, int n, int k, int M, int cap) {
  const bool on = k <= n;
  g.mrx[mixed_stage(q, k, M)] = on ? g.rx[plan_stage(p, k, cap)] : 0.0;
  g.mry[mixed_stage(q, k, M)] = on ? g.ry[plan_stage(p, k, cap)] : 0.0;
  g.mryaw[mixed_stage(q, k, M)] = on ? g.ryaw[plan_stage(p, k, cap)] : 0.0;
  for (int c = 0; c < 4; ++c) g.mxWS[mixed_xws(q, c, k, M)] = on ? g.xWS[plan_xws(p, c, k, n, cap)] : 0.0;
  if (k < M)
    for (int c = 0; c < 2; ++c) g.muWS[mixed_uws(q, c, k, M)] = k < n ? g.uWS[plan_uws(p, c, k, n, cap)] : 0.0;
  if (k == 0)
    for (int r = 0; r < 4; ++r) { g.mx0[4 * (size_t)q + r] = g.x0[4 * (size_t)p + r]; g.mxF[4 * (size_t)q + r] = g.xF[4 * (size_t)p + r]; }
}

// Scatter: the outputs of slot q (mixed layout at M) to pose p (mixed layout at Ncap), stage k of the slot's horizon n.  Only the
// entries of stages 0..n (controls 0..n-1) are written; src / dst null: an output the caller did not ask for.
OBCA_FHD void scatter_rows(const double* src, double* dst, int rows, int ext, int q, int p, int n, int k, int M, int Ncap) {
  if (!dst || k >= n + ext) return;
  for (int r = 0; r < rows; ++r) dst[out_entry(p, r, k, rows, Ncap, ext)] = src[out_entry(q, r, k, rows, M, ext)];
}

// The outputs of the entry: xp 4 x (M+1), up 2 x M, ts M+1, lp V x (M+1), np 4nOb x (M+1), sl nOb x (M+1) per problem, and one value
// per problem of the rest.  sl and strict may be null.
struct Outs {
  double *xp, *up, *ts, *lp, *np, *sl, *kkt_err;
  int *exitflag, *iters, *feasible, *strict;
};
OBCA_FHD void scatter_stage(const Outs& s, const Outs& d, int V, int nOb, int q, int p, int n, int k, int M, int Ncap) {
  scatter_rows(s.xp, d.xp, 4, 1, q, p, n, k, M, Ncap);
  scatter_rows(s.up, d.up, 2, 0, q, p, n, k, M, Ncap);
  scatter_rows(s.ts, d.ts, 1, 1, q, p, n, k, M, Ncap);
  scatter_rows(s.lp, d.lp, V, 1, q, p, n, k, M, Ncap);
  scatter_rows(s.np, d.np, 4 * nOb, 1, q, p, n, k, M, Ncap);
  scatter_rows(s.sl, d.sl, nOb, 1, q, p, n, k, M, Ncap);
  if (k == 0) {
    d.exitflag[p] = s.exitflag[q]; d.iters[p] = s.iters[q]; d.kkt_err[p] = s.kkt_err[q]; d.feasible[p] = s.feasible[q];
    if (d.strict) d.strict[p] = s.strict[q];
  }
}

}  // namespace obca_flow
