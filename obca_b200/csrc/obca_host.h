// obca_host.h -- host-side helpers shared by the C-ABI (obca_lib.cu) and the development emulation (tests/emul/): building the
// POD problem description from the reference's argument list and choosing a parking problem's template variant.
#pragma once
#include <string.h>

#include <type_traits>

#include "obca_solver.cuh"
#include "obca_quad.cuh"

namespace obca {

// the bounds on nOb and vOb[j] bound sum(vOb): no shape that passes them overflows the problem's half-space arrays
static_assert(OBCA_MAX_OB * OBCA_VMAX <= OBCA_MAX_ROWS, "sum(vOb) is bounded through nOb and vOb[j]");

// Arguments as in ParkingSignedDist.jl:29: vOb = half-space counts per obstacle, A = sum(vOb) x 2 column-major,
// b = sum(vOb), ego = [x_up, y_up, -x_lo, -y_lo] (main.jl:72-73), XYbounds = [xL, xU, yL, yU] (main.jl:209-210).
inline int fill_problem(ParkProblem& P, int N, int nOb, const int* vOb, const double* A, const double* b, double Ts,
                        double L, const double* ego, const double* XYbounds, int fixTime, int signed_dist) {
  memset(&P, 0, sizeof(P));
  if (N < 2 || nOb < 1 || nOb > OBCA_MAX_OB) return -1;
  P.N = N; P.nOb = nOb;
  int V = 0;
  for (int j = 0; j < nOb; ++j) {
    if (vOb[j] < 1 || vOb[j] > OBCA_VMAX) return -2;
    P.vOb[j] = vOb[j]; P.voff[j] = V; V += vOb[j];
  }
  P.voff[nOb] = V;
  P.V = V;      // <= OBCA_MAX_OB * OBCA_VMAX <= OBCA_MAX_ROWS (static_assert above)
  for (int r = 0; r < V; ++r) { P.A[r][0] = A[r]; P.A[r][1] = A[V + r]; P.b[r] = b[r]; }
  P.Ts = Ts; P.L = L;
  const double W_ev = ego[1] + ego[3], L_ev = ego[0] + ego[2];           // ParkingSignedDist.jl:182-183
  P.g[0] = L_ev / 2; P.g[1] = W_ev / 2; P.g[2] = L_ev / 2; P.g[3] = W_ev / 2;   // :185
  P.off = (ego[0] + ego[2]) / 2 - ego[2];                                 // :188
  for (int i = 0; i < 4; ++i) P.xyb[i] = XYbounds[i];
  P.dmin = 0.05;                                                          // :33
  P.fix_time = fixTime ? 1 : 0;
  P.signed_dist = signed_dist ? 1 : 0;
  P.w_a = (fixTime || !signed_dist) ? 0.5 : 0.1;                          // :79,:86 ; ParkingDist.jl:79,87
  P.w_yaw = fixTime ? 0.01 : 0.0001;                                      // :82,:91
  return 0;
}

#define OBCA_STR_(x) #x
#define OBCA_STR(x) OBCA_STR_(x)
// the message for a nonzero return of fill_problem: the bound the problem breaks
inline const char* shape_error(int rc) {
  switch (rc) {
    case -1: return "unsupported problem shape: need N >= 2 and 1 <= nOb <= " OBCA_STR(OBCA_MAX_OB) " obstacles";
    case -2: return "unsupported problem shape: need 1 <= vOb[j] <= " OBCA_STR(OBCA_VMAX) " half-spaces per obstacle";
    default: return "unsupported problem shape";
  }
}

// Arguments of QuadcopterSignedDist.jl:25: obs = ob1..ob5 as 6 x 5 column-major; bounds of :78-93 (QuadcopterDist.jl:88).
inline int fill_quad_problem(QuadProblem& P, int N, double Ts, double R, const double* obs, int signed_dist) {
  memset(&P, 0, sizeof(P));
  if (N < 2) return -1;
  P.N = N; P.Ts = Ts; P.R = R; P.signed_dist = signed_dist ? 1 : 0;
  for (int o = 0; o < QNOB; ++o)
    for (int r = 0; r < 6; ++r) P.obs[o][r] = obs[6 * o + r];
  const double lo[12] = {0, 0, 0, -3, -0.2, -0.2, -1, -1, -1, signed_dist ? -1.0 : -1.5, -1, -1};
  const double hi[12] = {10, 10, 5, 3, 0.2, 0.2, 1, 1, 1, signed_dist ? 1.0 : 3.0, 1, 1};
  for (int i = 0; i < 12; ++i) { P.xlo[i] = lo[i]; P.xhi[i] = hi[i]; }
  return 0;
}

inline int max_vob(const ParkProblem& P) {
  int m = 0;
  for (int j = 0; j < P.nOb; ++j) m = P.vOb[j] > m ? P.vOb[j] : m;
  return m;
}

// The template variant of a parking problem: f(vm, sdv) with vm = std::integral_constant<int, VM> (VM = 2 when no obstacle has more
// than two half-spaces, else 4) and sdv = std::integral_constant<bool, SDV> (the signed-distance formulation).
template <class F>
inline auto with_variant(const ParkProblem& P, F&& f) {
  using V2 = std::integral_constant<int, 2>;
  using V4 = std::integral_constant<int, 4>;
  if (P.signed_dist) return max_vob(P) <= 2 ? f(V2(), std::true_type()) : f(V4(), std::true_type());
  return max_vob(P) <= 2 ? f(V2(), std::false_type()) : f(V4(), std::false_type());
}

inline int nfac_for(const ParkProblem& P) {
  return with_variant(P, [](auto vm, auto sdv) { return LocalDims<decltype(vm)::value, decltype(sdv)::value>::NFAC; });
}

}  // namespace obca
