/* obca.h -- C-ABI of libobca.so, the H100-native replacement for the JuMP + Ipopt solve inside the OBCA
 * reference's NLP drivers.  Plain C, plain pointers and sizes; no allocation escapes the library.
 *
 * The reference (XiaojingGeorgeZhang/OBCA) has no FFI of its own: its boundary is the set of Julia functions that
 * AutonomousParking/main.jl calls positionally.  Each entry point below is what the Julia shim of the same name
 * (julia/*.jl, see INTEGRATION.md) `ccall`s in place of the reference's `Model(solver=IpoptSolver(...))` ...
 * `solve(m)` ... `getvalue(...)` sequence:
 *
 *   obca_parking_solve_batch  <- ParkingSignedDist.jl:29-314  (signed_dist=1)  and  ParkingDist.jl:29-315 (=0)
 *                                 called from main.jl:269 / main.jl:258
 *   obca_dualmultws_batch     <- DualMultWS.jl:29-86           called from ParkingSignedDist.jl:219, ParkingDist.jl:221
 *   obca_check_parking        <- ParkingConstraints.jl:29-149  called from ParkingSignedDist.jl:253,278, ParkingDist.jl:259,277
 *   obca_parking_solve_mixed / obca_check_parking_mixed: the same two for a batch whose problems have different horizons
 *                                 (the Hybrid A* warm starts of main.jl:215-248 each come with their own N)
 *   obca_parking_plan_solve_goals: main.jl:215-269 (plan -> solve -> accept) for a batch of start poses in one call
 *   obca_quadcopter_solve_batch / obca_check_quadcopter  <- QuadcopterSignedDist.jl / QuadcopterDist.jl / constrSatisfaction.jl
 *   obca_quadcopter_solve_mixed / obca_check_quadcopter_mixed: the same two for a batch whose problems have different
 *                                 horizons and sampling times (the 3-D A* warm starts of mainQuadcopter.jl:122-137 each
 *                                 come with their own N and Ts = round(Ts*80/N, 2))
 *   obca_quadcopter_plan_solve: mainQuadcopter.jl:114-154 (plan -> warm start -> solve -> check) for a batch of start / goal
 *                                 pairs in one call
 *   obca_parking_plan_solve_both / obca_quadcopter_plan_solve_both: the same two flows planned once and solved with both
 *                                 formulations, Distance then Signed Distance, as main.jl and mainQuadcopter.jl run them
 *
 * Conventions
 *   - every array is float64, COLUMN-MAJOR exactly as the Julia caller holds it; a batch of B problems is the B
 *     per-problem arrays stored one after the other (problem index slowest).  B = 1 reproduces the reference call.
 *   - vOb[nOb] are HALF-SPACE counts (main.jl:101 passes vObMPC = vOb-1); A is sum(vOb) x 2, b is sum(vOb)
 *     (obstHrep.jl:39-40), shared by the whole batch.
 *   - return value: 0 = executed (per-problem success is in exitflag[]), < 0 = usage / CUDA error (see
 *     obca_last_error()).  The library never throws and never falls back to a CPU path: without a CUDA device
 *     every compute entry point returns OBCA_ERR_NO_DEVICE.
 *   - `*_dev` variants take DEVICE pointers (cudaMalloc'ed by the caller on opts->device) and enqueue on the
 *     library's stream of that device; they return after the stream has been synchronised.
 *
 * Device-pointer entries on the caller's stream
 *   obca_parking_solve_mixed_dev, obca_dualmultws_batch_dev, obca_check_parking_dev, obca_check_parking_mixed_dev,
 *   obca_quadcopter_solve_batch_dev, obca_quadcopter_solve_mixed_dev, obca_check_quadcopter_dev, obca_check_quadcopter_mixed_dev
 *   take the arguments of their host-pointer twin (the name without _dev), in its order and with its shapes, layout and nullability,
 *   and one more, `stream`.  Every per-problem array (inputs and outputs, Nb and Tsb included) is a device pointer on opts->device;
 *   the scene data (vOb, A, b, ego, XYbounds, ob), opts and solve_seconds stay host pointers.
 *   - stream: a cudaStream_t of opts->device; NULL is that device's default stream.  On entry the library records an event on
 *     `stream` and its own stream waits for it, so work enqueued on `stream` before the call has finished before any input is read.
 *     The entry returns once the library's stream has finished: the outputs are then ready for any stream.  No entry synchronises
 *     the device or waits for work on any other stream.  (obca_parking_solve_batch_dev predates this and takes no stream: it runs
 *     on the library's stream only.)
 *   - Each writes bit for bit what its twin writes for the same inputs and options: every output over each problem's own horizon,
 *     exitflag (the quadcopter's 2 included), iters, kkt_err, feasible, e, strict, worst, DualMultWS's lp, np and d; and
 *     obca_last_times / obca_last_profile / obca_last_schedule report the call as they report the twin's.
 *   - The mixed entries write nothing past a problem's own horizon in the caller's arrays.
 *   - Refusals: the twin's checks with its messages and codes -- a null argument, a shape error, a horizon bound (OBCA_ERR_UNSUPPORTED)
 *     -- on the host, before any device work.  Nb and Tsb are in device memory: they are checked on the device (one small kernel and
 *     an 8-byte readback) after the wait and before anything is written; a bad entry returns OBCA_ERR_ARG with the twin's message
 *     (e.g. "Nb[37] = 1 outside [2, Nmax = 80]") and no output touched.  Without a CUDA device: OBCA_ERR_NO_DEVICE.
 */
#ifndef OBCA_H
#define OBCA_H

#ifdef __cplusplus
extern "C" {
#endif

#define OBCA_VERSION 200
#define OBCA_ERR_ARG (-1)
#define OBCA_ERR_NO_DEVICE (-2)
#define OBCA_ERR_CUDA (-3)
#define OBCA_ERR_UNSUPPORTED (-4)

/* Interior-point options: the Ipopt options set at ParkingSignedDist.jl:41-43 (tol, max_iter,
 * min_hessian_perturbation -> dw_min, jacobian_regularization_value is replaced by the always-on dc) and the Ipopt
 * defaults the reference leaves untouched.  obca_default_opts() fills in exactly those values. */
typedef struct obca_opts {
  double tol;
  int max_iter;
  double mu_init, mu_min;
  double kappa_eps, kappa_mu, theta_mu, tau_min;
  double kappa1, kappa2, kappa_sigma, s_max;
  double dual_inf_tol, constr_viol_tol, compl_inf_tol;
  double dw_min, dw_first, dw_max, kw_minus, kw_plus, kw_plus_first;
  double gamma_theta, gamma_phi, delta, s_theta, s_phi, eta_phi, gamma_alpha;
  int max_backtrack;
  double dc;
  int max_kick;      /* restoration substitute: barrier kicks per attempt after a failed line search (default 3) */
  int quad_dual_ws;  /* quadcopter: 1 (default) closed-form dual warm start; 0 the reference's l = 0.05 start */
  /* execution */
  int device;        /* CUDA device ordinal used by this call */
  int retry;         /* 1: the reference's status / retry logic: ParkingSignedDist.jl:256-290 (a failed first attempt is always
                        followed by one more solve from the last iterate, then ParkingConstraints decides) and
                        ParkingDist.jl:245-289 (after a failed first attempt ParkingConstraints decides whether the point is
                        accepted or solved again); 0: single attempt, exitflag = converged */
  int q4;            /* ParkingDist only: 1 reproduces the reference's inverted test after a SECOND failure
                        (ParkingDist.jl:278-282: Feasible == 0 -> exitflag 1, SURVEY.md A.4-Q4); 0 (default): exitflag = Feasible */
} obca_opts;

int obca_version(void);
int obca_device_count(void);                 /* number of visible CUDA devices (0 if none) */
const char* obca_last_error(void);
void obca_default_opts(obca_opts* o);

/* Batched ParkingSignedDist / ParkingDist.
 * inputs (per problem):  x0[4], xF[4], rx/ry/ryaw[N+1], xWS (N+1)x4, uWS Nx2 (first N rows of the reference's uWS,
 *                        ParkingSignedDist.jl:217), lWS (N+1)xV and nWS (N+1)x4nOb as returned by DualMultWS
 *                        (pass lWS = nWS = NULL to have the library run DualMultWS itself, as the reference does
 *                        at ParkingSignedDist.jl:219)
 * outputs (per problem): xp 4x(N+1), up 2xN, ts (N+1) [ones if fixTime], lp Vx(N+1), np 4nOb x(N+1)
 *                        (ParkingSignedDist.jl:302-313), sl nOb x(N+1) (may be NULL),
 *                        exitflag (1 = converged, 0 = not), iters, kkt_err (Ipopt's scaled NLP error E_0),
 *                        solve_seconds[1] = device time of the solve alone -- the reference's `time` (:239-241, :297) is
 *                        the wall time of solve(m), which excludes DualMultWS (:219); obca_last_times() gives both.
 * shape bounds: 1 <= nOb <= 16 obstacles, 1 <= vOb[j] <= 4 half-spaces per obstacle, sum(vOb) <= 64, 2 <= N <= 319
 *                        (N + 1 <= 320 stages); another shape returns OBCA_ERR_ARG (OBCA_ERR_UNSUPPORTED for a longer horizon)
 *                        with the bound in obca_last_error(), before any device work, and writes no output.  */
int obca_parking_solve_batch(int B, int N, int nOb, const int* vOb, const double* A, const double* b,
                             const double* x0, const double* xF, double Ts, double L, const double* ego,
                             const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                             const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                             int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up, double* ts,
                             double* lp, double* np, double* sl, int* exitflag, int* iters, double* kkt_err,
                             double* solve_seconds);

/* Same, all batch arrays (x0 ... nWS, xp ... kkt_err) are device pointers on opts->device; vOb, A, b, ego,
 * XYbounds, opts and solve_seconds stay host pointers. */
int obca_parking_solve_batch_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b,
                                 const double* x0, const double* xF, double Ts, double L, const double* ego,
                                 const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                                 const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                                 int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up,
                                 double* ts, double* lp, double* np, double* sl, int* exitflag, int* iters,
                                 double* kkt_err, double* solve_seconds);

/* Batched ParkingSignedDist / ParkingDist over problems with different horizons, in ONE solve.  Problem b has horizon
 * Nb[b], 2 <= Nb[b] <= Nmax.  Every per-problem array has the shape it has in obca_parking_solve_batch with N = Nmax
 * (inputs rx/ry/ryaw Nmax+1, xWS (Nmax+1)x4, uWS Nmax x2, lWS (Nmax+1)xV, nWS (Nmax+1)x4nOb; outputs xp 4x(Nmax+1),
 * up 2xNmax, ts Nmax+1, lp Vx(Nmax+1), np 4nOb x(Nmax+1), sl nOb x(Nmax+1)); problem b uses the first Nb[b]+1 stages and
 * the first Nb[b] control rows of them.  The solver never reads input entries past that point and never writes output
 * entries past it.  Problem b's results (outputs over its own horizon, exitflag, iters, kkt_err) are bit-identical to
 * solving it with obca_parking_solve_batch at N = Nb[b] and the same options.  Nb = NULL or an Nb[b] outside [2, Nmax]:
 * OBCA_ERR_ARG.  Shape bounds as for obca_parking_solve_batch (nOb <= 16, vOb[j] <= 4, sum(vOb) <= 64); Nmax > 319 returns
 * OBCA_ERR_UNSUPPORTED whatever the problems' own horizons, before any device work and with no output written.
 * obca_last_times / obca_last_schedule / obca_last_profile report this call like any other. */
int obca_parking_solve_mixed(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                             const double* x0, const double* xF, double Ts, double L, const double* ego,
                             const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                             const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                             int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up, double* ts,
                             double* lp, double* np, double* sl, int* exitflag, int* iters, double* kkt_err,
                             double* solve_seconds);

/* obca_parking_solve_mixed on device pointers (Nb included), on the caller's stream: see "Device-pointer entries" above. */
int obca_parking_solve_mixed_dev(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                                 const double* x0, const double* xF, double Ts, double L, const double* ego,
                                 const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                                 const double* xWS, const double* uWS, const double* lWS, const double* nWS,
                                 int fixTime, int signed_dist, const obca_opts* opts, double* xp, double* up, double* ts,
                                 double* lp, double* np, double* sl, int* exitflag, int* iters, double* kkt_err,
                                 double* solve_seconds, void* stream);

/* Batched DualMultWS (DualMultWS.jl:29; `ego` is a global there, :39).  lp (N+1)xV, np (N+1)x4nOb per problem
 * (already transposed like :81-84); d (N+1)xnOb optional (optimal objective = ego/obstacle distance). */
int obca_dualmultws_batch(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* ego,
                          const double* rx, const double* ry, const double* ryaw, const obca_opts* opts, double* lp,
                          double* np, double* d);

/* obca_dualmultws_batch on device pointers (rx, ry, ryaw, lp, np, d), on the caller's stream. */
int obca_dualmultws_batch_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* ego,
                              const double* rx, const double* ry, const double* ryaw, const obca_opts* opts, double* lp,
                              double* np, double* d, void* stream);

/* Batched ParkingConstraints (ParkingConstraints.jl:29-149), restated verbatim including its quirks
 * (SURVEY.md A.4-Q3).  x 4x(N+1), u 2xN, l Vx(N+1), n 4nOb x(N+1), timeScale (N+1).
 * feasible[B] = the reference's return value (0/1); e[7*B] = its seven pass flags; strict[B] (optional) = a
 * checker without the quirks: every dynamics row, every obstacle, box bounds, slack-aware distance row.  e[0] checks
 * |timeScale - 1| with fixTime = 1 too, as the reference does (:47); strict exempts fixed time from it.
 * Non-finite inputs: the reference's maximum() propagates NaN, so a group (e flag) that reads a NaN fails, and strict is 0
 * whenever an entry it reads is NaN.  An infinite entry fails its group, directly or through the NaN it produces. */
int obca_check_parking(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* x0,
                       const double* xF, double Ts, double L, const double* ego, const double* XYbounds,
                       const double* x, const double* u, const double* l, const double* n, const double* timeScale,
                       const double* sl, int fixTime, int sd, const obca_opts* opts, int* feasible, int* e,
                       int* strict);

/* obca_check_parking over problems with different horizons: Nb[b] in [2, Nmax], arrays laid out for Nmax as in
 * obca_parking_solve_mixed; problem b is audited on its first Nb[b]+1 stages. */
int obca_check_parking_mixed(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                             const double* x0, const double* xF, double Ts, double L, const double* ego,
                             const double* XYbounds, const double* x, const double* u, const double* l, const double* n,
                             const double* timeScale, const double* sl, int fixTime, int sd, const obca_opts* opts,
                             int* feasible, int* e, int* strict);

/* obca_check_parking and obca_check_parking_mixed on device pointers (Nb, x0 ... sl, feasible, e, strict), on the caller's stream. */
int obca_check_parking_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b, const double* x0,
                           const double* xF, double Ts, double L, const double* ego, const double* XYbounds,
                           const double* x, const double* u, const double* l, const double* n, const double* timeScale,
                           const double* sl, int fixTime, int sd, const obca_opts* opts, int* feasible, int* e,
                           int* strict, void* stream);
int obca_check_parking_mixed_dev(int B, const int* Nb, int Nmax, int nOb, const int* vOb, const double* A, const double* b,
                                 const double* x0, const double* xF, double Ts, double L, const double* ego,
                                 const double* XYbounds, const double* x, const double* u, const double* l, const double* n,
                                 const double* timeScale, const double* sl, int fixTime, int sd, const obca_opts* opts,
                                 int* feasible, int* e, int* strict, void* stream);

/* Batched QuadcopterSignedDist (signed_dist=1, QuadcopterNavigation/QuadcopterSignedDist.jl:25-300, called from
 * mainQuadcopter.jl:152) / QuadcopterDist (signed_dist=0, QuadcopterDist.jl:25-282, mainQuadcopter.jl:145).
 * inputs:  x0, xF 12 per problem; ob = ob1..ob5 as a 6 x 5 column-major block shared by the batch; xWS 12x(N+1) per
 *          problem; timeWS scalar.  (uWS is ignored by the reference, QuadcopterSignedDist.jl:202.)
 * outputs: xp 12x(N+1), up 4xN, ts (N+1), lp 30x(N+1) (= [l1;l2;l3;l4;l5], :296), slack 5x(N+1) (SD only, may be
 *          NULL), exitflag 1 / 0 / 2 (2 = converged but sum(slack) > 1e-3, :283-288), iters, kkt_err, solve_seconds.
 * A single solve attempt, like the reference (flag = 1, :227-235).  opts == NULL: defaults with max_iter = 3000
 * (the reference leaves Ipopt's default).  Horizons 2 <= N <= 511 (N + 1 <= 512 stages); N > 511: OBCA_ERR_UNSUPPORTED
 * (the bound is in obca_last_error()), returned before any device work, no output touched. */
int obca_quadcopter_solve_batch(int B, int N, const double* x0, const double* xF, double Ts, double R, const double* ob,
                                const double* xWS, double timeWS, int signed_dist, const obca_opts* opts, double* xp,
                                double* up, double* ts, double* lp, double* slack, int* exitflag, int* iters,
                                double* kkt_err, double* solve_seconds);

/* Batched constrSatisfaction (QuadcopterNavigation/constrSatisfaction.jl:25-204, called from mainQuadcopter.jl:147,154),
 * restated verbatim (tolerance 1e-3, rows for i = 1..N, Dist-variant box on x10, one-sided norm row, quirk Q5).
 * feasible[B] = the reference's Bool; worst[B] (optional) = the largest contribution of the reference's groups: the start and
 * end state (max |.|), per stage the u and x box groups (1.0 when violated), the 13 dynamics rows with the timeScale difference
 * (max |.|), the 5 norm rows (max), the 5 distance rows (-min), and lambda (-min over the whole matrix); a zero (possibly -0.0) when none is positive.
 * feasible = worst <= 1e-3.  Non-finite inputs: a test of the reference whose group holds a NaN never fails, so such a group
 * contributes nothing (a NaN anywhere in lambda turns the lambda group off), while the other groups still decide. */
int obca_check_quadcopter(int B, int N, const double* x, const double* u, const double* timeScale, const double* x0,
                          const double* xF, double Ts, const double* lambda, const double* ob, double R,
                          const obca_opts* opts, int* feasible, double* worst);

/* Batched QuadcopterSignedDist / QuadcopterDist over problems with different horizons and sampling times, in ONE solve.
 * Problem b has horizon Nb[b], 2 <= Nb[b] <= Nmax, and sampling time Tsb[b] (finite, > 0).  Obstacles, R, the state
 * bounds and timeWS are shared by the batch.  Every per-problem array has the shape it has in
 * obca_quadcopter_solve_batch with N = Nmax (inputs xWS 12x(Nmax+1); outputs xp 12x(Nmax+1), up 4xNmax, ts Nmax+1,
 * lp 30x(Nmax+1), slack 5x(Nmax+1)); problem b uses the first Nb[b]+1 stages and the first Nb[b] control columns of them.
 * The solver never reads input entries past that point and never writes output entries past it.  Problem b's results
 * (outputs over its own horizon, exitflag including the slack gate value 2, iters, kkt_err) are bit-identical to solving
 * it with obca_quadcopter_solve_batch at N = Nb[b], Ts = Tsb[b] and the same options.  Nb or Tsb NULL, an Nb[b] outside
 * [2, Nmax] or a Tsb[b] that is not a finite number > 0: OBCA_ERR_ARG (the index is in obca_last_error()), no output
 * touched.  Nmax <= 511 (N + 1 <= 512 stages), as for obca_quadcopter_solve_batch; Nmax > 511: OBCA_ERR_UNSUPPORTED
 * (the bound is in obca_last_error()), whatever the problems' own horizons, no output touched. */
int obca_quadcopter_solve_mixed(int B, const int* Nb, int Nmax, const double* x0, const double* xF, const double* Tsb,
                                double R, const double* ob, const double* xWS, double timeWS, int signed_dist,
                                const obca_opts* opts, double* xp, double* up, double* ts, double* lp, double* slack,
                                int* exitflag, int* iters, double* kkt_err, double* solve_seconds);

/* obca_check_quadcopter over problems with different horizons and sampling times: Nb[b] in [2, Nmax], Tsb[b] finite > 0,
 * arrays laid out for Nmax as in obca_quadcopter_solve_mixed; problem b is checked on its first Nb[b]+1 stages with Tsb[b]. */
int obca_check_quadcopter_mixed(int B, const int* Nb, int Nmax, const double* x, const double* u, const double* timeScale,
                                const double* x0, const double* xF, const double* Tsb, const double* lambda,
                                const double* ob, double R, const obca_opts* opts, int* feasible, double* worst);

/* The quadcopter solves and checkers on device pointers (Nb, Tsb, x0, xF, xWS and every output but solve_seconds; the checkers' x ... lambda,
 * feasible and worst), on the caller's stream. */
int obca_quadcopter_solve_batch_dev(int B, int N, const double* x0, const double* xF, double Ts, double R, const double* ob,
                                    const double* xWS, double timeWS, int signed_dist, const obca_opts* opts, double* xp,
                                    double* up, double* ts, double* lp, double* slack, int* exitflag, int* iters,
                                    double* kkt_err, double* solve_seconds, void* stream);
int obca_quadcopter_solve_mixed_dev(int B, const int* Nb, int Nmax, const double* x0, const double* xF, const double* Tsb,
                                    double R, const double* ob, const double* xWS, double timeWS, int signed_dist,
                                    const obca_opts* opts, double* xp, double* up, double* ts, double* lp, double* slack,
                                    int* exitflag, int* iters, double* kkt_err, double* solve_seconds, void* stream);
int obca_check_quadcopter_dev(int B, int N, const double* x, const double* u, const double* timeScale, const double* x0,
                              const double* xF, double Ts, const double* lambda, const double* ob, double R,
                              const obca_opts* opts, int* feasible, double* worst, void* stream);
int obca_check_quadcopter_mixed_dev(int B, const int* Nb, int Nmax, const double* x, const double* u, const double* timeScale,
                                    const double* x0, const double* xF, const double* Tsb, const double* lambda,
                                    const double* ob, double R, const obca_opts* opts, int* feasible, double* worst, void* stream);

/* Hybrid A* warm starts on the GPU: B start poses x0 and a goal per pose xF (both 3 x B column-major: x, y, yaw) among the obstacle
 * points (ox[i], oy[i]), i < n_ob, in ONE call -- main.jl:215-248 for each pose, as obca_plan_warmstart_cloud_batch of
 * include/obca_planner.h does on host threads, with the same search decisions (the same heuristic maps, priorities, insertion order and
 * expansion budget) and the same outputs up to the last bits of sin / cos / atan2 / acos / tan / atan.  The heuristic map depends on the
 * goal only through its grid cell (round(gx / 0.3), round(gy / 0.3)): one CTA per distinct goal cell builds that cell's map on the device
 * (k_plan_hmap), bit for bit the host's Dijkstra, then one CTA plans one pose at a time (k_plan) against its goal's map.
 *   Ts: the sampling time (> 0) of the warm start; L: wheelbase of the steering extraction; sampleN: down-sampling of the 0.1 m path.
 *   max_expansions <= 0: 200000 (obca_plan_warmstart's budget).
 *   max_nodes: node pool per resident CTA; <= 0 selects 32768 (the demo sweeps insert at most ~4500 nodes per plan).  Device scratch per
 *     resident CTA (4 per SM): max_nodes x 176 bytes + a 4-byte cell table over the search grid (~1 MB for the demo clouds)
 *     + ~0.2 MB of course buffers + 96 x cap x sampleN bytes; about 7.1 MB at the defaults, cap = 512, sampleN = 3.
 *     Device memory of one call: min(B, 4 x SMs) x that scratch -- about 3.7 GB on a 132-SM H100 for B >= 528 at the defaults --,
 *     the heuristic maps, distinct goal cells x hxw x hyw x 8 bytes (hxw x hyw: the cloud's extent in 0.3 m cells; 3520 cells, 28 KB per
 *     goal cell, for the demo "backwards" cloud, 3384 / 27 KB for the 10-car lot), plus the batch's goals and outputs,
 *     72 x B x cap + 64 x B bytes (151 MB at B = 4096, cap = 512), which are copied to the device first (so that the entries the planner
 *     does not write keep the caller's values) and back after the kernel.  All of it is freed before the call returns.
 * Outputs, with the stride cap, in the layout of obca_plan_warmstart_batch: rx / ry / ryaw [i*cap ..] (N[i]+1 values), xWS [i*4*cap ..]
 * as (N[i]+1) x 4, uWS [i*2*cap ..] as N[i] x 2 column-major.  Nothing past a problem's own N[i]+1 stages is written.
 * status[i]: OBCA_PLAN_OK (0), OBCA_PLAN_NO_PATH (1), OBCA_PLAN_CAPACITY (2; N[i] holds the horizon, nothing else written), or
 * OBCA_PLAN_POOL_FULL (4): the search outgrew its device scratch and was stopped: it needed more than max_nodes nodes, or -- only for
 * a start pose hundreds of metres from the goal -- an analytic expansion longer than the kernel's 4096-point course buffer (409.6 m).
 * That pose is NOT planned (nothing else written, never a partial path); the host planner can plan it
 * (obca_b200.planner.device.plan_goals_batch does so).
 * expansions[i] (may be NULL): nodes expanded.  plan_seconds (may be NULL): device time of the search kernel k_plan.
 * Return: 0, OBCA_ERR_ARG (B < 0, a null array, n_ob <= 0, Ts <= 0, sampleN < 1, cap < 2; reason in obca_last_error()),
 * OBCA_ERR_NO_DEVICE, OBCA_ERR_CUDA. */
#define OBCA_PLAN_POOL_FULL 4
int obca_plan_parking_warmstart_goals(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob,
                                      double Ts, double L, int sampleN, int max_expansions, int max_nodes, int cap,
                                      const obca_opts* opts, double* rx, double* ry, double* ryaw, double* xWS, double* uWS,
                                      int* N, int* status, int* expansions, double* plan_seconds);

/* The same with ONE goal xF (x, y, yaw) for the whole batch -- the randomised sweeps of main.jl:165-168, as obca_plan_warmstart_batch of
 * include/obca_planner.h plans them on host threads: obca_plan_parking_warmstart_goals with xF repeated for every pose (one heuristic
 * map), same outputs, status codes and device memory. */
int obca_plan_parking_warmstart_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob,
                                      double Ts, double L, int sampleN, int max_expansions, int max_nodes, int cap,
                                      const obca_opts* opts, double* rx, double* ry, double* ryaw, double* xWS, double* uWS,
                                      int* N, int* status, int* expansions, double* plan_seconds);

/* The heuristic maps the two entries above build on the device (k_plan_hmap), read back; used by tests and tools/bench_plan_goals.py.
 * For the cloud (ox, oy, n_ob > 0): mn[2] = (minx, miny), w[2] = (xw, yw) (the map's cell (i, j), 1 <= i <= xw, 1 <= j <= yw, is the grid cell
 * (i + minx, j + miny)); then, one map per goal g < G (goals: 2 x G column-major, gx, gy), maps[(g * xw + i-1) * yw + j-1] = the 8-connected
 * distance of that cell from the goal's cell, INF where unreachable -- calc_dist_policy of obca_b200/planner/csrc/obca_plan_core.h, bit
 * for bit.  map_seconds (may be NULL): device time of k_plan_hmap.  Return: 0, OBCA_ERR_ARG (G < 0, a null array, n_ob <= 0, or fewer
 * than G x xw x yw entries in cap -- mn and w are written first, so a call with maps = NULL reads the size), OBCA_ERR_NO_DEVICE,
 * OBCA_ERR_CUDA. */
int obca_plan_parking_heuristic_maps(int G, const double* goals, const double* ox, const double* oy, int n_ob, const obca_opts* opts,
                                     long long* mn, int* w, double* maps, long long cap, double* map_seconds);

/* main.jl:215-269 for a batch: plan every start pose towards its goal (obca_plan_parking_warmstart_goals), solve every pose that planned
 * (obca_parking_solve_mixed, DualMultWS inside) and run ParkingConstraints on the results (obca_check_parking_mixed) in ONE call, with
 * nothing leaving the device between the stages.  All on the library's stream of opts->device:
 *   1. plan (k_plan_hmap, k_plan) with the stride Ncap + 1 into device buffers, then free the planner's scratch;
 *   2. list the poses planned OK to a horizon 2 <= N[i] <= Ncap, in pose order; their count and longest horizon Nmax are the only values
 *      read back before the solve, which is laid out for that Nmax, not for Ncap;
 *   3. gather those poses' warm starts, x0 and xF into the inputs of the mixed solve;  4. solve;  5. check;
 *   6. scatter the results to the caller's pose order and copy them back once.
 * Inputs: the planner's (x0 4 x B: x, y, yaw, v -- the planner reads x, y, yaw and the solve starts from all four --; xF 4 x B, the
 * planner reads x, y, yaw; the cloud ox, oy, n_ob; Ts, L, sampleN, max_expansions, max_nodes as for obca_plan_parking_warmstart_goals)
 * and the solve's (nOb, vOb, A, b, ego, XYbounds, fixTime, signed_dist, opts; Ts and L are the solve's too).
 * Ncap: 2 <= Ncap <= 319, the horizon the caller's arrays hold.  Outputs, in the caller's pose order, in the layout of
 * obca_parking_solve_mixed with Nmax = Ncap: xp, up, ts, lp, np, sl (may be NULL); kkt_err, exitflag, iters and feasible (the return
 * value of ParkingConstraints), strict (may be NULL) one per pose; N[i], status[i] and expansions[i] (may be NULL) as the planner writes
 * them.  status[i]:
 *   OBCA_PLAN_OK (0)         planned and solved: every output of pose i over its own horizon N[i] is written, nothing past it;
 *   OBCA_PLAN_NO_PATH (1)    no path: only status and N (as the planner leaves it) are written;
 *   OBCA_PLAN_POOL_FULL (4)  the search outgrew its device scratch: the same (no host fallback here; obca_b200.planner.device plans such
 *                            poses on the host);
 *   OBCA_PLAN_CAPACITY (2)   the planned horizon N[i] is greater than Ncap (or below the solver's 2): N[i] holds it, nothing else.
 * A pose that is not solved leaves every other output entry as the caller had it.  Pose i's solve, check and outputs are bit-identical
 * to obca_parking_solve_mixed followed by obca_check_parking_mixed (with sl) on the planner's output for it.  plan_seconds (may be NULL):
 * device time of k_plan; solve_seconds (may be NULL): as for obca_parking_solve_mixed; obca_last_times / obca_last_schedule report the
 * solve.  Device memory, freed before the call returns apart from the solve's workspace, which stays with the library as after any
 * solve: the planner's buffers, 72 x B x (Ncap + 1) + 84 x B bytes; while planning, the planner's scratch on top (about 3.7 GB on a
 * 132-SM H100 for B >= 528, see obca_plan_parking_warmstart_goals), freed before the solve allocates; then the solve's inputs and outputs
 * for the Bs poses it takes, about 8 x Bs x (Nmax + 1) x (16 + V + 5 nOb) bytes, its workspace (as obca_parking_solve_mixed at Nmax), and at
 * the end the caller's outputs, about 8 x B x (Ncap + 1) x (7 + V + 5 nOb) bytes, which are copied to the device first.
 * Return: 0, OBCA_ERR_ARG (the planner's: B < 0, a null required array, n_ob <= 0, Ts <= 0, sampleN < 1; Ncap < 2; the solver's shape
 * errors), OBCA_ERR_UNSUPPORTED (Ncap > 319, the bound in obca_last_error()), all before any device work and with nothing written;
 * OBCA_ERR_NO_DEVICE, OBCA_ERR_CUDA.  B = 0, or a batch in which no pose is solved, returns 0 without launching the solve. */
int obca_parking_plan_solve_goals(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts,
                                  double L, int sampleN, int max_expansions, int max_nodes, int nOb, const int* vOb, const double* A,
                                  const double* b, const double* ego, const double* XYbounds, int fixTime, int signed_dist,
                                  const obca_opts* opts, int Ncap, double* xp, double* up, double* ts, double* lp, double* np, double* sl,
                                  int* N, int* status, int* expansions, int* exitflag, int* iters, double* kkt_err, int* feasible,
                                  int* strict, double* plan_seconds, double* solve_seconds);

/* 3-D A* warm starts of the quadcopter flow on the GPU: B start / goal pairs (x0, xF: 3 x B column-major positions, each pair its own)
 * among one obstacle point cloud (ox, oy, oz, n_ob >= 0 points; lo, hi: the bound corners in raw units; reso > 0: the cell size) in ONE
 * call -- the inputs and outputs of obca_astar3d_batch of include/obca_planner.h, with the same search decisions bit for bit (the search
 * compiles from the same source, obca_b200/planner/csrc/obca_astar3d_core.h): the same status, N, path and expansion count.  One warp
 * plans one pair at a time (k_plan3d); the obstacle bitmap is built on the host, once per call.
 *   max_nodes: node pool per warp; <= 0 selects 262144 (2^18; the largest config-4 search of 2048 pairs uses 229043 nodes); at most 2^28.
 *     The queue holds max_nodes / 4 entries (at least 64).  Device scratch per warp: a 4-byte cell table over the map (2.4 MB for the
 *     105 x 105 x 55 demo grid) + max_nodes x 16 bytes + the queue's 4 x max_nodes bytes; about 7.7 MB at the defaults.
 *     Device memory of one call: min(B rounded up to 4, 4 x SMs) warps x that scratch -- about 4.0 GB on a 132-SM H100 for B >= 528 at
 *     the defaults --, plus the bitmap (w0 x w1 x w2 / 8 bytes, 76 KB for the demo grid), 48 x B bytes of cells and the outputs,
 *     24 x B x cap + 12 x B bytes, which are copied to the device first (so that the entries the planner does not write keep the
 *     caller's values) and back after the kernel.  All of it is freed before the call returns.
 * Outputs, with the stride cap: rx / ry / rz [i*cap ..]: the path, start first, as cell * reso (N[i]+1 points).
 * status[i]: OBCA_PLAN_OK (0), OBCA_PLAN_NO_PATH (1), OBCA_PLAN_CAPACITY (2: more than cap points; N[i] holds the horizon, nothing else
 * written), or OBCA_PLAN_POOL_FULL (4): the search needed more than max_nodes nodes or max_nodes / 4 queue entries and was stopped; that
 * pair is NOT planned (nothing else written); the host library can plan it (obca_b200.planner.device.plan_quadcopter_batch does so).
 * expansions[i] (may be NULL): cells closed, the goal included.  plan_seconds (may be NULL): device time of the search kernel.
 * Return: 0, OBCA_ERR_ARG (B < 0, a null array, n_ob < 0, reso <= 0, cap < 1, max_nodes > 2^28, a non-finite coordinate, a map of
 * more than 2^27 cells or a start / goal more than 2^30 cells from it; reason in obca_last_error(), nothing written), OBCA_ERR_NO_DEVICE,
 * OBCA_ERR_CUDA. */
int obca_plan_quadcopter_warmstart_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz,
                                         int n_ob, const double* lo, const double* hi, double reso, int max_nodes, int cap,
                                         const obca_opts* opts, double* rx, double* ry, double* rz, int* N, int* status, int* expansions,
                                         double* plan_seconds);

/* The grid scale of the quadcopter flow: the 3-D A* plans on a grid 10x finer than the solve's units (mainQuadcopter.jl:114-119 scales
 * the start and goal up, a_star_3d.plan_quadcopter_warm_start divides the path back down). */
#define OBCA_QUAD_GRID_SCALE 10.0

/* mainQuadcopter.jl:114-154 for a batch: plan every start / goal pair with the 3-D A* (obca_plan_quadcopter_warmstart_batch), build the
 * warm start of every pair that planned (a_star_3d.plan_quadcopter_warm_start), solve those pairs (obca_quadcopter_solve_mixed) and run
 * constrSatisfaction on the results (obca_check_quadcopter_mixed) in ONE call, with nothing leaving the device between the stages.  All
 * on the library's stream of opts->device:
 *   1. plan (k_plan3d) with the stride Ncap + 1 into device buffers, then free the planner's scratch;
 *   2. list the pairs planned OK to a horizon 2 <= N[i] <= Ncap, in pair order; their count and longest horizon Nmax are the only values
 *      read back before the solve, which is laid out for that Nmax, not for Ncap;
 *   3. build those pairs' warm starts: xWS = the path / OBCA_QUAD_GRID_SCALE in rows 1-3 and zeros in rows 4-12, the sampling time
 *      Tsb[i] = jround(Ts * 80 / N[i] * 100) / 100 (jround: round half away from zero) computed in IEEE double without fused
 *      operations, and x0 / xF gathered into the inputs of the mixed solve;  4. solve;  5. check;
 *   6. scatter the results to the caller's pair order and copy them back once.
 * Inputs: x0, xF 12 x B in the solve's units, as for obca_quadcopter_solve_mixed; the planner's start and goal are OBCA_QUAD_GRID_SCALE
 * times their rows 1-3, multiplied on the host.  The cloud ox, oy, oz (n_ob points), the bound corners lo, hi, the cell size reso and
 * max_nodes are the planner's, in its units, as for obca_plan_quadcopter_warmstart_batch.  Ts: the nominal sampling time (0.25 in
 * mainQuadcopter.jl).  R, ob, timeWS, signed_dist, opts: the solve's, as for obca_quadcopter_solve_mixed; opts == NULL: defaults with
 * max_iter = 3000.  Ncap: 2 <= Ncap <= 511, the horizon the caller's arrays hold.
 * Outputs, in the caller's pair order, in the layout of obca_quadcopter_solve_mixed with Nmax = Ncap: xp 12x(Ncap+1), up 4xNcap,
 * ts Ncap+1, lp 30x(Ncap+1), slack 5x(Ncap+1) (may be NULL; written for signed_dist = 1 only); one value per pair: N (the planned
 * horizon), Tsb (the pair's sampling time), status, expansions (may be NULL) as the planner writes them, exitflag, iters, kkt_err,
 * feasible (the value constrSatisfaction returns) and worst (may be NULL; the largest violation it found).  status[i]:
 *   OBCA_PLAN_OK (0)         planned and solved: every output of pair i over its own horizon N[i] is written, nothing past it;
 *   OBCA_PLAN_NO_PATH (1)    no path: only status and N (as the planner leaves it) are written;
 *   OBCA_PLAN_POOL_FULL (4)  the search outgrew its device scratch: the same (no host fallback here; obca_b200.planner.device plans such
 *                            pairs on the host);
 *   OBCA_PLAN_CAPACITY (2)   the path has more than Ncap + 1 points, or fewer than 3 (N[i] < 2): N[i] holds the horizon, nothing else.
 * A pair that is not solved leaves every other output entry as the caller had it.  Pair i's warm start, solve, check and outputs are
 * bit-identical to obca_quadcopter_solve_mixed followed by obca_check_quadcopter_mixed on the warm start
 * a_star_3d.plan_quadcopter_warm_start builds from obca_plan_quadcopter_warmstart_batch's path.  plan_seconds (may be NULL): device time
 * of k_plan3d; solve_seconds (may be NULL): as for obca_quadcopter_solve_mixed.  Device memory, freed before the call returns apart from
 * the solve's workspace, which stays with the library as after any solve: the planner's buffers and the pairs' states,
 * 24 x B x (Ncap + 1) + 212 x B bytes; while planning, the planner's scratch on top (about 4.0 GB on a 132-SM H100 for B >= 528, see
 * obca_plan_quadcopter_warmstart_batch), freed before the solve allocates; then the solve's inputs and outputs for the Bs pairs it
 * takes, about 8 x Bs x (Nmax + 1) x 64 bytes, its workspace (as obca_quadcopter_solve_mixed at Nmax), and at the end the caller's
 * outputs, about 8 x B x (Ncap + 1) x 52 bytes, which are copied to the device first.
 * One call solves one formulation: mainQuadcopter.jl solves QuadcopterDist and QuadcopterSignedDist on the same plan, which
 * obca_quadcopter_plan_solve_both does from one plan.
 * Return: 0, OBCA_ERR_ARG (the planner's: a null required array, max_nodes > 2^28, B < 0, n_ob < 0, reso <= 0, a non-finite coordinate,
 * a map of more than 2^27 cells or a start / goal more than 2^30 cells from it; Ncap < 2; Ts not a finite number > 0, or so small that
 * jround(Ts * 80 / Ncap * 100) < 1, which would give a pair a sampling time of 0), OBCA_ERR_UNSUPPORTED (Ncap > 511, the bound in
 * obca_last_error()), all before any device work and with nothing written; OBCA_ERR_NO_DEVICE, OBCA_ERR_CUDA.  B = 0, or a batch in
 * which no pair is solved, returns 0 without launching the solve (solve_seconds = 0). */
int obca_quadcopter_plan_solve(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz, int n_ob,
                               const double* lo, const double* hi, double reso, int max_nodes, double Ts, double R, const double* ob,
                               double timeWS, int signed_dist, const obca_opts* opts, int Ncap, double* xp, double* up, double* ts,
                               double* lp, double* slack, int* N, double* Tsb, int* status, int* expansions, int* exitflag, int* iters,
                               double* kkt_err, int* feasible, double* worst, double* plan_seconds, double* solve_seconds);

/* The outputs of one formulation of a flow call that solves both (obca_parking_plan_solve_both, obca_quadcopter_plan_solve_both):
 * the arrays obca_parking_plan_solve_goals / obca_quadcopter_plan_solve take for their solve and check, with the same shapes, layout
 * and nullability.  Parking: sl, strict and solve_seconds may be NULL, every other field is required.  Quadcopter: slack, worst and
 * solve_seconds may be NULL, every other field is required; slack is written for the Signed Distance set only. */
typedef struct obca_parking_flow_out {
  double *xp, *up, *ts, *lp, *np, *sl;
  int *exitflag, *iters;
  double* kkt_err;
  int *feasible, *strict;
  double* solve_seconds;
} obca_parking_flow_out;

typedef struct obca_quadcopter_flow_out {
  double *xp, *up, *ts, *lp, *slack;
  int *exitflag, *iters;
  double* kkt_err;
  int* feasible;
  double* worst;
  double* solve_seconds;
} obca_quadcopter_flow_out;

/* main.jl:215-269 as the reference runs it: plan every start pose ONCE, then solve and check the poses that planned with ParkingDist
 * (main.jl:258) and then with ParkingSignedDist (main.jl:269), in one call.  Inputs and shared outputs (N, status, expansions,
 * plan_seconds) are those of obca_parking_plan_solve_goals without signed_dist, written once as it writes them.  dist and sd (both
 * required) receive the outputs of the Distance and the Signed Distance formulation: each set is bit for bit what
 * obca_parking_plan_solve_goals with signed_dist = 0 / 1 writes for the same inputs, including the entries it leaves as the caller had
 * them (poses not solved, entries past a pose's own horizon).  Both solves take the same listed poses at the same layout horizon Nmax,
 * and DualMultWS runs inside each, as in the reference.  The Distance solve runs first: after the call obca_last_times,
 * obca_last_schedule and obca_last_profile report the Signed Distance solve.
 * Device memory: the peak of obca_parking_plan_solve_goals at the same B, Ncap and shape.  The planner's buffers and the gathered
 * solve inputs and outputs stay allocated across both solves; for each formulation the outputs are zeroed, solved, checked, scattered
 * to the caller's layout (about 8 x B x (Ncap + 1) x (7 + V + 5 nOb) bytes, copied to the device first) and copied back, and that
 * caller-layout staging is freed before the next formulation runs.
 * Return: the refusals of obca_parking_plan_solve_goals, and OBCA_ERR_ARG for a null dist or sd, or a null required field of either
 * (obca_last_error() names it, e.g. "null argument: sd.xp"), all before any device work and with nothing written; OBCA_ERR_NO_DEVICE;
 * OBCA_ERR_CUDA, after which the dist set may already have been written.  B = 0, or a batch in which no pose is solved, returns 0
 * without a solve, with both solve_seconds 0. */
int obca_parking_plan_solve_both(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts,
                                 double L, int sampleN, int max_expansions, int max_nodes, int nOb, const int* vOb, const double* A,
                                 const double* b, const double* ego, const double* XYbounds, int fixTime, const obca_opts* opts,
                                 int Ncap, int* N, int* status, int* expansions, double* plan_seconds, const obca_parking_flow_out* dist,
                                 const obca_parking_flow_out* sd);

/* mainQuadcopter.jl:114-154 as the reference runs it: plan every start / goal pair ONCE and build its warm start, then solve and check
 * the pairs that planned with QuadcopterDist and constrSatisfaction (:145-147) and then with QuadcopterSignedDist and constrSatisfaction
 * (:152-154), in one call.  Inputs and shared outputs (N, Tsb, status, expansions, plan_seconds) are those of obca_quadcopter_plan_solve
 * without signed_dist, written once as it writes them.  dist and sd (both required) receive the outputs of the Distance and the Signed
 * Distance formulation: each set is bit for bit what obca_quadcopter_plan_solve with signed_dist = 0 / 1 writes for the same inputs,
 * including the entries it leaves as the caller had them (dist->slack is never written).  The Distance solve runs first: after the call
 * obca_last_profile reports the Signed Distance solve.
 * Device memory: the peak of obca_quadcopter_plan_solve at the same B and Ncap.  The planner's buffers, the pairs' states and the
 * gathered solve inputs and outputs stay allocated across both solves; for each formulation the outputs are zeroed, solved, checked,
 * scattered to the caller's layout (about 8 x B x (Ncap + 1) x 52 bytes, copied to the device first) and copied back, and that
 * caller-layout staging is freed before the next formulation runs.
 * Return: the refusals of obca_quadcopter_plan_solve, and OBCA_ERR_ARG for a null dist or sd, or a null required field of either
 * (obca_last_error() names it, e.g. "null argument: dist.feasible"), all before any device work and with nothing written;
 * OBCA_ERR_NO_DEVICE; OBCA_ERR_CUDA, after which the dist set may already have been written.  B = 0, or a batch in which no pair is
 * solved, returns 0 without a solve, with both solve_seconds 0. */
int obca_quadcopter_plan_solve_both(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz,
                                    int n_ob, const double* lo, const double* hi, double reso, int max_nodes, double Ts, double R,
                                    const double* ob, double timeWS, const obca_opts* opts, int Ncap, int* N, double* Tsb, int* status,
                                    int* expansions, double* plan_seconds, const obca_quadcopter_flow_out* dist,
                                    const obca_quadcopter_flow_out* sd);

/* Device times of the last obca_parking_solve_batch[_dev] / obca_parking_solve_mixed on `device`: DualMultWS (0 when the caller passed lWS / nWS) and the
 * solve alone (= what solve_seconds reports; the reference's `time`, ParkingSignedDist.jl:297). */
int obca_last_times(int device, double* dualws_seconds, double* solve_seconds);

/* Counters of the last solve on `device`, summed over the batch.  Parking (phase-split schedule): out8[7] = K1 evaluations in
 * the round kernel k_pk_eval (of which out8[5] are re-evaluations after a barrier update), out8[6] = merit-function
 * evaluations in k_pk_step, out8[4] / out8[3] = K1 / merit evaluations inside the tail kernel.  Quadcopter kernel: per-phase
 * device cycle counters {eval, kkt, recover, merit, update, serial, #merit evaluations, #K1 evaluations} (thread 0 of every
 * CTA, clock64).  Diagnostic only. */
int obca_last_profile(int device, unsigned long long* out8);

/* How the last obca_parking_solve_batch[_dev] on `device` was scheduled (last chunk of the batch): number of phase-split
 * rounds ([k_pk_eval, k_pk_sweep, k_pk_step] kernel triples over all active problems) and the number of problems handed to
 * the persistent tail kernel afterwards (= the batch size when no rounds were run).  Environment overrides for experiments:
 * OBCA_MODE (0 auto, 1 tail kernel only, 2 rounds only), OBCA_TAIL_THRESH (hand-over point), OBCA_CHUNK (problems per
 * chunk).  kernel_ms5 (may be NULL): with OBCA_PHASE_TIMING=1 in the environment the solve records CUDA events around
 * every kernel and reports the summed times of {k_pk_eval (K1 + decisions), k_pk_sweep (K3), k_pk_step (K4), tail kernel,
 * DualMultWS} in milliseconds.  Diagnostic only. */
int obca_last_schedule(int device, int* rounds, int* handed_over, double* kernel_ms5);

/* K1 stand-alone: fused evaluation of the parking NLP in the REFERENCE's formulation at B given points (no solve);
 * what JuMP's eval_g / eval_grad_f / eval_jac_g' * y do for Ipopt (ParkingSignedDist.jl:240), one thread per
 * (problem, stage).  Per problem it reads z = (xp, ts, up, lp, np[, sl]) (n values), the row multipliers y (m values,
 * may be NULL = zeros) and rx, ry, ryaw, and writes c (m rows; inequality rows = their bodies),
 * gradL = grad_z [f + y'c] (n values) and fk (objective per stage, N+1 values).
 *   rows of c / y:  start 4 | end 4 | dyn 4xN | chain N | rate N | norm nOb x(N+1) | rot 2nOb x(N+1) | dist nOb x(N+1)
 *   entries of gradL: x 4x(N+1) | timeScale (N+1) | u 2xN | l Vx(N+1) | n 4nOb x(N+1) | sl nOb x(N+1) (SD only)
 * Algorithmic HBM bytes per problem per call: 8 * (2n + 2m + 3(N+1))  (SURVEY.md 8(d), fused variant).
 * All batch arrays are DEVICE pointers.  `reps` launches are timed together; kernel_ms = mean per launch. */
int obca_parking_eval_sizes(int N, int nOb, const int* vOb, int signed_dist, long long* n_out, long long* m_out);
int obca_parking_eval_batch_dev(int B, int N, int nOb, const int* vOb, const double* A, const double* b,
                                const double* x0, const double* xF, double Ts, double L, const double* ego,
                                const double* XYbounds, const double* rx, const double* ry, const double* ryaw,
                                const double* xp, const double* up, const double* ts, const double* lp,
                                const double* np, const double* sl, const double* y, int fixTime, int signed_dist,
                                const obca_opts* opts, double* c_out, double* gradL_out, double* fk_out, int reps,
                                double* kernel_ms);

#ifdef __cplusplus
}
#endif
#endif
