// tests/emul/emul_quad_mixed.cpp -- DEVELOPMENT / TEST TOOL ONLY.
//
// The development emulation of one quadcopter solver CTA (see emul.cpp) for a batch whose problems have different horizons and
// sampling times: every per-problem array is laid out for the batch's horizon Nmax (the layout of obca_quadcopter_solve_mixed)
// and problem b is solved at its own horizon Nb[b] and sampling time Tsb[b] -- the per-problem path of the OBCA_HD solver
// sources, run on the host.  Not linked into libobca.so, not a fallback of the product path.
#include <stdio.h>
#include <stdlib.h>

#include <cmath>
#include <vector>

#include "../../obca_b200/csrc/obca_host.h"

using namespace obca;

// quadcopter: problem b solved at its own horizon Nb[b] and sampling time Tsb[b], every per-problem array laid out for Nmax
// (the layout of obca_quadcopter_solve_mixed).  The batch's shared sampling time is NaN: a read of it instead of the
// problem's own would show in every output.
extern "C" int emul_quadcopter_solve_mixed(int B, const int* Nb, int Nmax, const double* x0, const double* xF, const double* Tsb,
                                           double R, const double* obs, const double* xWS, double timeWS, int signed_dist,
                                           const IpmOpts* opts, double* xp, double* up, double* ts, double* lp, double* slack,
                                           int* status, int* iters, double* kkt_err) {
  QuadProblem P;
  if (fill_quad_problem(P, Nmax, std::nan(""), R, obs, signed_dist)) return -1;
  for (int i = 0; i < B; ++i)
    if (Nb[i] < 2 || Nb[i] > Nmax) return -4;
  IpmOpts O = opts ? *opts : default_opts();
  QLay Lay = make_qlayout(P);
  const size_t NS = Nmax + 1;
#pragma omp parallel for schedule(dynamic)
  for (int i = 0; i < B; ++i) {
    std::vector<double> W((size_t)Lay.total * Lay.NSP, 0.0);
    QCtx C;
    ProbState S;
    C.P = &P; C.N = Nb[i]; C.Ts = Tsb[i]; C.O = &O; C.L = Lay; C.W = W.data(); C.red_scratch = nullptr; C.tile = nullptr; C.S = &S;
    C.in.x0 = x0 + 12 * (size_t)i; C.in.xF = xF + 12 * (size_t)i; C.in.xWS = xWS + 12 * NS * i; C.in.timeWS = timeWS;
    QOutputs out;
    out.xp = xp + 12 * NS * i; out.up = up + (size_t)4 * Nmax * i; out.ts = ts + NS * i; out.lp = lp + 30 * NS * i;
    out.slack = slack ? slack + 5 * NS * i : nullptr;
    if (signed_dist) {
      IpmDriver<QuadSolver<true> >::solve(C);
      for (int k = 0; k <= Nb[i]; ++k) QuadSolver<true>::store_stage(C, k, out);
    } else {
      IpmDriver<QuadSolver<false> >::solve(C);
      for (int k = 0; k <= Nb[i]; ++k) QuadSolver<false>::store_stage(C, k, out);
    }
    status[i] = S.status; iters[i] = S.iters; kkt_err[i] = S.e0;
  }
  return 0;
}
