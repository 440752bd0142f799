// tests/emul/emul_check.cpp -- DEVELOPMENT / TEST TOOL ONLY.
//
// The constraint checkers of libobca.so (k_check: check_stage / chk_merge / check_finish, and k_quad_check: quad_check_stage) on
// the host, with the kernels' reduction: 128 lanes, lane t takes the stages t, t + 128, ..., then a shuffle-down tree in each warp
// of 32 and lane 0 merging warps 1..3.  order_seed != 0 merges the stages' partials in a seeded random order instead, so a test can
// require that the verdicts do not depend on the order.  Not linked into libobca.so, not a fallback of the product path.
#include <stdint.h>

#include <algorithm>
#include <random>
#include <vector>

#include "../../obca_b200/csrc/obca_host.h"
#include "../../obca_b200/csrc/obca_check.cuh"

using namespace obca;

namespace {

constexpr int LANES = 128, WARP = 32;

// The kernels' reduction of one partial per lane: __shfl_down_sync(v, off) reads lane + off, or its own value past the warp.
template <class T, class M>
T reduce_lanes(std::vector<T> v, M merge) {
  for (int w = 0; w < LANES / WARP; ++w)
    for (int off = 16; off > 0; off >>= 1) {
      std::vector<T> nw(WARP);
      for (int i = 0; i < WARP; ++i) {
        nw[i] = v[WARP * w + i];
        merge(nw[i], v[WARP * w + (i + off < WARP ? i + off : i)]);
      }
      std::copy(nw.begin(), nw.end(), v.begin() + WARP * w);
    }
  T m = v[0];
  for (int w = 1; w < LANES / WARP; ++w) merge(m, v[WARP * w]);
  return m;
}

// The stages' partials (stage k at index k) merged in the kernels' order, or in a random order when seed != 0.
template <class T, class M>
T reduce_stages(const std::vector<T>& st, const T& init, uint64_t seed, M merge) {
  if (seed) {
    std::vector<int> ord(st.size());
    for (size_t i = 0; i < ord.size(); ++i) ord[i] = (int)i;
    std::mt19937_64 g(seed);
    std::shuffle(ord.begin(), ord.end(), g);
    T m = init;
    for (int i : ord) merge(m, st[i]);
    return m;
  }
  std::vector<T> lane(LANES, init);
  for (size_t k = 0; k < st.size(); ++k) merge(lane[k % LANES], st[k]);
  return reduce_lanes(lane, merge);
}

}  // namespace

// One parking problem in the C-ABI's arguments (obca_check_parking with B = 1): feasible, e[7] and strict as k_check computes them.
extern "C" int emul_check_parking(int N, int nOb, const int* vOb, const double* A, const double* b, const double* x0, const double* xF,
                                  double Ts, double L, const double* ego, const double* XYbounds, const double* x, const double* u,
                                  const double* l, const double* n, const double* ts, const double* sl, int fixTime, int sd,
                                  uint64_t order_seed, int* feasible, int* e, int* strict) {
  ParkProblem P;
  if (fill_problem(P, N, nOb, vOb, A, b, Ts, L, ego, XYbounds, fixTime, sd)) return -1;
  for (int st = 0; st < 2; ++st) {
    std::vector<ChkPart> part(N + 1);
    for (int k = 0; k <= N; ++k) check_stage(P, N, k, x0, xF, x, u, l, n, ts, sl, sd, st, part[k]);
    ChkPart init;
    chk_init(init);
    const ChkPart m = reduce_stages(part, init, order_seed, [](ChkPart& a, const ChkPart& c) { chk_merge(a, c); });
    int ee[7];
    const int f = check_finish(P, m, ts, st, 5e-5, ee);
    if (st == 0) {
      *feasible = f;
      for (int i = 0; i < 7; ++i) e[i] = ee[i];
    } else {
      *strict = f;
    }
  }
  return 0;
}

// One quadcopter problem in the C-ABI's arguments (obca_check_quadcopter with B = 1): feasible and worst as k_quad_check computes them.
extern "C" int emul_check_quadcopter(int N, const double* x, const double* u, const double* ts, const double* x0, const double* xF,
                                     double Ts, const double* lam, const double* ob, double R, uint64_t order_seed, int* feasible,
                                     double* worst) {
  QuadProblem P;
  if (fill_quad_problem(P, N, Ts, R, ob, 0)) return -1;
  struct Part { double w, l; };
  std::vector<Part> part(N + 1);
  for (int k = 0; k <= N; ++k) part[k].w = quad_check_stage(P, N, Ts, k, x0, xF, x, u, ts, lam, &part[k].l);
  const Part m = reduce_stages(part, Part{0.0, -1e300}, order_seed, [](Part& a, const Part& c) {
    a.w = fmax(a.w, c.w);
    a.l = dmax_nan(a.l, c.l);
  });
  const double w = m.l == m.l ? fmax(m.w, m.l) : m.w;
  *feasible = w <= 1e-3 ? 1 : 0;
  *worst = w;
  return 0;
}
