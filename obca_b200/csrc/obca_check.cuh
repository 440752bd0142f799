// obca_check.cuh -- K5: constraint-satisfaction audit.
//
// check_stage_ref(): per-stage partial results of AutonomousParking/ParkingConstraints.jl:29-149, restated verbatim
// INCLUDING its quirks (SURVEY.md A.4-Q3):
//   * variable-time branch overwrites c3[1,i] four times, so only the v-row of the dynamics is checked (:76-79)
//   * c6[.,i] is overwritten per obstacle, so only the LAST obstacle is checked (:117-128)
//   * c5 divides by timeScale[1] only (:92);  X/Y/v box bounds are never checked
//   * in sd=1 mode the distance row ignores the slack sl (:127-128) and the norm row is abs(pp) - 1 (:117)
// check_stage_strict(): the same audit without the quirks (all dynamics rows, all obstacles, box bounds,
// |pp - 1| for the signed-distance variant, slack-aware distance row).
// Arrays are in the reference's shapes: x 4x(N+1), u 2xN, l Vx(N+1), n 4nOb x(N+1), ts (N+1), column-major.
// Every max is dmax_nan: a NaN fails its group, as it does through the reference's maximum().
#pragma once
#include "obca_common.cuh"

namespace obca {

struct ChkPart {
  double c0[5];   // max|u1|, max|u2|, max|ts-1|, -min l, -min n   (before subtracting the limits)
  double c1, c2;  // start / end
  double c3;      // max |dynamics rows checked|
  double c4;      // max |diff ts|
  double c5;      // max |diff [0 u1]|
  double c6;      // max over obstacle rows
  double sbox;    // strict only: worst box-bound violation
};

OBCA_HD void chk_init(ChkPart& c) {
  c.c0[0] = c.c0[1] = c.c0[2] = 0.0; c.c0[3] = c.c0[4] = -1e300;
  c.c1 = c.c2 = c.c3 = c.c4 = c.c5 = 0.0; c.c6 = -1e300; c.sbox = -1e300;
}
OBCA_HD void chk_merge(ChkPart& a, const ChkPart& b) {
#pragma unroll
  for (int i = 0; i < 5; ++i) a.c0[i] = dmax_nan(a.c0[i], b.c0[i]);
  a.c1 = dmax_nan(a.c1, b.c1); a.c2 = dmax_nan(a.c2, b.c2); a.c3 = dmax_nan(a.c3, b.c3); a.c4 = dmax_nan(a.c4, b.c4);
  a.c5 = dmax_nan(a.c5, b.c5); a.c6 = dmax_nan(a.c6, b.c6); a.sbox = dmax_nan(a.sbox, b.sbox);
}

OBCA_HD void chk_dyn(const ParkProblem& P, const double* xk, const double* uk, double tsk, double* f) {
  const double h = P.fix_time ? P.Ts : tsk * P.Ts;
  const double tl = tan(uk[0]) / P.L;
  const double vm = xk[3] + 0.5 * h * uk[1];
  const double th = xk[2] + 0.5 * h * xk[3] * tl;
  f[0] = xk[0] + h * vm * cos(th);
  f[1] = xk[1] + h * vm * sin(th);
  f[2] = xk[2] + h * vm * tl;
  f[3] = xk[3] + h * uk[1];
}

// strict != 0 -> quirk-free audit
// N: the horizon of this problem (stages 0..N of the arrays are read)
OBCA_HD void check_stage(const ParkProblem& P, int N, int k, const double* x0, const double* xF, const double* x,
                         const double* u, const double* l, const double* n, const double* ts, const double* sl,
                         int sd, int strict, ChkPart& c) {
  chk_init(c);
  const double* xk = x + 4 * k;
  if (k < N) {
    const double* uk = u + 2 * k;
    c.c0[0] = dabs(uk[0]); c.c0[1] = dabs(uk[1]);
    double f[4];
    chk_dyn(P, xk, uk, ts[k], f);
    const double* xn = x + 4 * (k + 1);
    if (P.fix_time || strict) {
      c.c3 = dmax_nan(dmax_nan(dabs(xn[0] - f[0]), dabs(xn[1] - f[1])), dmax_nan(dabs(xn[2] - f[2]), dabs(xn[3] - f[3])));
    } else {
      c.c3 = dabs(xn[3] - f[3]);                       // ParkingConstraints.jl:76-79 (last assignment wins)
    }
    if (!P.fix_time) c.c4 = dabs(ts[k + 1] - ts[k]);   // :91
    const double up1 = k > 0 ? u[2 * (k - 1)] : 0.0;
    c.c5 = dabs(uk[0] - up1);                          // :88/:92, scaled by the caller
    if (strict) c.c5 /= (P.fix_time ? P.Ts : ts[k] * P.Ts);
  }
  c.c0[2] = P.fix_time && strict ? 0.0 : dabs(ts[k] - 1.0);   // :47 checks timeScale with fixed time too; the strict audit does not
  for (int r = 0; r < P.V; ++r) c.c0[3] = dmax_nan(c.c0[3], -l[(size_t)P.V * k + r]);
  for (int r = 0; r < 4 * P.nOb; ++r) c.c0[4] = dmax_nan(c.c0[4], -n[(size_t)4 * P.nOb * k + r]);
  if (k == 0) c.c1 = dmax_nan(dmax_nan(dabs(xk[0] - x0[0]), dabs(xk[1] - x0[1])), dmax_nan(dabs(xk[2] - x0[2]), dabs(xk[3] - x0[3])));
  if (k == N) c.c2 = dmax_nan(dmax_nan(dabs(xk[0] - xF[0]), dabs(xk[1] - xF[1])), dmax_nan(dabs(xk[2] - xF[2]), dabs(xk[3] - xF[3])));
  double sn_, cs_;
  sincos(xk[2], &sn_, &cs_);
  const int j0 = strict ? 0 : P.nOb - 1;
  for (int j = j0; j < P.nOb; ++j) {
    double p1 = 0.0, p2 = 0.0, bl = 0.0;
    for (int r = P.voff[j]; r < P.voff[j + 1]; ++r) {
      const double lr = l[(size_t)P.V * k + r];
      p1 += P.A[r][0] * lr; p2 += P.A[r][1] * lr; bl += P.b[r] * lr;
    }
    const double* nj = n + (size_t)4 * P.nOb * k + 4 * j;
    const double pp = p1 * p1 + p2 * p2;
    double c61 = strict && sd ? dabs(pp - 1.0) : pp - 1.0;                               // :116-120
    const double c62 = dabs((nj[0] - nj[2]) + cs_ * p1 + sn_ * p2);                      // :123
    const double c63 = dabs((nj[1] - nj[3]) - sn_ * p1 + cs_ * p2);                      // :124
    double dist = -(P.g[0] * nj[0] + P.g[1] * nj[1] + P.g[2] * nj[2] + P.g[3] * nj[3]) + (xk[0] + cs_ * P.off) * p1 +
                  (xk[1] + sn_ * P.off) * p2 - bl;
    if (strict && sd && sl) dist += sl[(size_t)P.nOb * k + j];
    const double c64 = -dist + P.dmin;                                                    // :127-128
    c.c6 = dmax_nan(c.c6, dmax_nan(dmax_nan(c61, c62), dmax_nan(c63, c64)));
  }
  if (strict && k >= 1 && k <= N - 1) {
    c.sbox = dmax_nan(dmax_nan(P.xyb[0] - xk[0], xk[0] - P.xyb[1]), dmax_nan(P.xyb[2] - xk[1], xk[1] - P.xyb[3]));
    c.sbox = dmax_nan(c.sbox, dmax_nan(-1.0 - xk[3], xk[3] - 2.0));
  }
}

// final flags from the merged partials.  e[0..6] = ParkingConstraints.jl:133-139.  returns sum(e) == 7.
OBCA_HD int check_finish(const ParkProblem& P, const ChkPart& c, const double* ts, int strict, double tol, int* e) {
  const double c0 = dmax_nan(dmax_nan(c.c0[0] - 0.6, c.c0[1] - 0.4), dmax_nan(dmax_nan(c.c0[2] - 0.2, c.c0[3]), c.c0[4]));
  double c5;
  if (strict) c5 = c.c5 - 0.6;
  else c5 = c.c5 / (P.fix_time ? P.Ts : ts[0] * P.Ts) - 0.6;
  e[0] = c0 <= tol; e[1] = c.c1 <= tol; e[2] = c.c2 <= tol; e[3] = c.c3 <= tol;
  e[4] = (P.fix_time ? 0.0 : c.c4) <= tol; e[5] = c5 <= tol; e[6] = c.c6 <= tol;
  int s = e[0] + e[1] + e[2] + e[3] + e[4] + e[5] + e[6];
  if (strict) return s == 7 && c.sbox <= tol;
  return s == 7;
}

}  // namespace obca
