// obca_common.cuh -- shared definitions for the sm_90a OBCA kernels.
//
// All arithmetic on this path is IEEE float64 (SURVEY.md section 8: Julia Float64 / Ipopt Number=double).
// The per-stage math lives in OBCA_HD functions so that the very same source is (a) compiled by nvcc into the
// persistent solver kernel and (b) compiled by g++ into tests/emul/ (a development-only emulation of one CTA,
// never part of libobca.so and never a fallback).
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define OBCA_HD __host__ __device__ __forceinline__
#define OBCA_D __device__ __forceinline__
// big per-stage phase functions: ONE copy in the kernel (the solver kernel is instruction-cache bound otherwise)
#define OBCA_HD_NI __host__ __device__ __noinline__
#else
#define OBCA_HD inline
#define OBCA_D inline
#define OBCA_HD_NI inline
#endif

#define OBCA_MAX_OB 16     // obstacles per problem
#define OBCA_MAX_ROWS 64   // total half-spaces (sum vOb)
#define OBCA_VMAX 4        // half-spaces per obstacle supported by the kernels (templates instantiate 2 and 4)
// parking horizon: k_pk_eval and k_pk_tail hold the N + 1 stage slots of a problem (656 bytes each) in dynamic shared memory;
// 320 of them (210 KB) leave room for the kernels' static shared memory under the H100's 227 KB per CTA
#define OBCA_PK_NMAX 319

namespace obca {

// ----------------------------------------------------------------------------------------------------------
// Problem description shared by every problem of a batch (obstacles, car, horizon).  POD, copied to the device.
// Mirrors the scalar arguments of ParkingSignedDist.jl:29 / ParkingDist.jl:29.
// ----------------------------------------------------------------------------------------------------------
struct ParkProblem {
  int N;            // horizon (number of control intervals)
  int nOb;          // obstacles
  int V;            // sum(vOb)
  int vOb[OBCA_MAX_OB];
  int voff[OBCA_MAX_OB + 1];
  double A[OBCA_MAX_ROWS][2];
  double b[OBCA_MAX_ROWS];
  double Ts, L;
  double g[4];      // ego half-extents  [L_ev/2, W_ev/2, L_ev/2, W_ev/2]   (ParkingSignedDist.jl:182-185)
  double off;       // rear-axle -> ego-centre offset                         (ParkingSignedDist.jl:188)
  double xyb[4];    // XYbounds
  double dmin;      // 0.05 (ParkingSignedDist.jl:33)
  int fix_time;     // fixTime
  int signed_dist;  // 1: ParkingSignedDist (norm == 1, slack), 0: ParkingDist (norm <= 1, no slack)
  double w_a;       // accel weight: 0.1 (SD var-time) / 0.5 otherwise        (ParkingSignedDist.jl:79,86; ParkingDist.jl:79,87)
  double w_yaw;     // yaw tracking weight: 1e-4 var-time / 1e-2 fixed-time   (:82,:91)
};

// Interior-point options (the Ipopt options that matter, ParkingSignedDist.jl:41-43; rest = Ipopt defaults).
struct IpmOpts {
  double tol;            // 1e-5
  int max_iter;          // 200
  double mu_init;        // 0.1
  double mu_min;         // tol/10
  double kappa_eps, kappa_mu, theta_mu, tau_min;
  double kappa1, kappa2, kappa_sigma, s_max;
  double dual_inf_tol, constr_viol_tol, compl_inf_tol;
  double dw_min, dw_first, dw_max, kw_minus, kw_plus, kw_plus_first;
  double gamma_theta, gamma_phi, delta, s_theta, s_phi, eta_phi, gamma_alpha;
  int max_backtrack;
  double dc;             // always-on dual regularisation on norm rows and the terminal dynamics rows (1e-9)
  int max_kick;          // barrier kicks (restoration substitute) per attempt; 0 = fail at the first line-search failure
  int quad_dual_ws;      // quadcopter: 1 = closed-form dual warm start, 0 = the reference's l = 0.05
};

OBCA_HD IpmOpts default_opts() {
  IpmOpts o;
  o.tol = 1e-5; o.max_iter = 200; o.mu_init = 0.1; o.mu_min = 1e-6;
  o.kappa_eps = 10.0; o.kappa_mu = 0.2; o.theta_mu = 1.5; o.tau_min = 0.99;
  o.kappa1 = 1e-2; o.kappa2 = 1e-2; o.kappa_sigma = 1e10; o.s_max = 100.0;
  o.dual_inf_tol = 1.0; o.constr_viol_tol = 1e-4; o.compl_inf_tol = 1e-4;
  o.dw_min = 1e-12; o.dw_first = 1e-4; o.dw_max = 1e20; o.kw_minus = 1.0 / 3.0; o.kw_plus = 8.0; o.kw_plus_first = 100.0;
  o.gamma_theta = 1e-5; o.gamma_phi = 1e-8; o.delta = 1.0; o.s_theta = 1.1; o.s_phi = 2.3; o.eta_phi = 1e-8;
  o.gamma_alpha = 0.05; o.max_backtrack = 40; o.dc = 1e-9; o.max_kick = 3; o.quad_dual_ws = 1;
  return o;
}

// Reciprocal used on the Newton-step path: computed once per gap / pivot and reused for every quotient with that
// denominator.  Device: rcp.rn.f64 (correctly rounded, so bit-identical to the host's 1.0 / x) -- about half the
// instructions of the IEEE division subroutine, and it sits on the latency-bound chain of the KKT sweep.
#if defined(__CUDA_ARCH__)
OBCA_HD double rcp(double x) { return __drcp_rn(x); }
#else
OBCA_HD double rcp(double x) { return 1.0 / x; }
#endif

OBCA_HD double dmax(double a, double b) { return a > b ? a : b; }
// The checkers' max: NaN wins, like Julia's maximum() in the references they restate (dmax drops a NaN in its first argument).
// Equal to dmax whenever neither argument is NaN; commutative and associative (up to the sign of a zero), so a
// reduction's result does not depend on its order.
OBCA_HD double dmax_nan(double a, double b) { return a > b || a != a ? a : b; }
OBCA_HD double dmin_(double a, double b) { return a < b ? a : b; }
OBCA_HD double dabs(double a) { return a < 0 ? -a : a; }

// sum of log(gap) over many gaps with few log() calls: products of up to 6 gaps (gaps lie in ~[1e-12, 1e2], so a product
// stays far inside the double range); FP64 log is ~50 instructions and the solver kernel is issue bound.
struct LogAcc {
  double prod, sum;
  int n;
  OBCA_HD LogAcc() : prod(1.0), sum(0.0), n(0) {}
  OBCA_HD void add(double g) {
    prod *= g;
    if (++n == 6) { sum += log(prod); prod = 1.0; n = 0; }
  }
  OBCA_HD double total() { if (n) { sum += log(prod); prod = 1.0; n = 0; } return sum; }
};

#if defined(__CUDACC__)
// Ampere-style asynchronous global -> shared copies (LDGSTS): the sweeps stream their per-stage data through small
// shared-memory rings so that the HBM / L2 latency of stage k-1 hides behind the arithmetic of stage k.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }
#endif

// packed upper-triangular index for an n x n symmetric matrix, i <= j
template <int N>
OBCA_HD constexpr int sym_idx(int i, int j) { return i * N - (i * (i - 1)) / 2 + (j - i); }
template <int N>
OBCA_HD constexpr int sym_idx_any(int i, int j) { return i <= j ? sym_idx<N>(i, j) : sym_idx<N>(j, i); }

}  // namespace obca
