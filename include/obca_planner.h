/* obca_planner.h -- C-ABI of the host-side warm-start producer (libobca_planner.so, plain C++, no CUDA).
 *
 * Replaces, for a caller that has no Julia-0.6 environment, the part of AutonomousParking/main.jl that runs BEFORE the NLP:
 *   hybrid_a_star.calc_hybrid_astar_path   hybrid_a_star.jl:104-190   (with reeds_shepp.jl, collision_check.jl, a_star.jl:47-128)
 *   veloSmooth                              veloSmooth.jl:29-109
 *   the warm-start extraction               main.jl:215-248
 * Same algorithms as the Python restatement obca_b200/planner/ (which documents the reference line by line); the two are tested to
 * produce the same paths (tests/test_planner_native.py).  The reference's planner is host code as well and runs once per problem.
 * GPU twins: obca_plan_parking_warmstart_goals / _batch in include/obca.h (libobca.so) plan a batch of start poses in one call with the same
 * search decisions; both libraries compile the algorithm from one source, obca_b200/planner/csrc/obca_plan_core.h.
 *
 * All arrays are Float64, owned by the caller, column-major where two-dimensional (Julia layout).
 */
#ifndef OBCA_PLANNER_H
#define OBCA_PLANNER_H
#ifdef __cplusplus
extern "C" {
#endif

#define OBCA_PLAN_OK 0
#define OBCA_PLAN_NO_PATH 1        /* the search exhausted its open list / expansion budget (the reference prints an error and returns nothing) */
#define OBCA_PLAN_CAPACITY 2       /* the caller's arrays are too short; *n_out holds the required length */
#define OBCA_PLAN_BAD_ARG 3

int obca_planner_version(void);

/* Hybrid A* (hybrid_a_star.jl:104): start (sx, sy, syaw) -> goal (gx, gy, gyaw) among the obstacle points (ox[i], oy[i]), i < n_ob.
 * xyreso / yawreso: grid resolutions (main.jl passes XY_GRID_RESOLUTION = 0.3 and YAW_GRID_RESOLUTION = 5 deg; <= 0 selects them).
 * Output: the path sampled every MOTION_RESOLUTION = 0.1 m, *n_out points written to rx, ry, ryaw (capacity cap). */
int obca_hybrid_astar(double sx, double sy, double syaw, double gx, double gy, double gyaw, const double* ox, const double* oy, int n_ob,
                      double xyreso, double yawreso, int max_expansions, int cap, double* rx, double* ry, double* ryaw, int* n_out);

/* The obstacle point cloud of the reference's two demo scenarios (main.jl:111-142 "backwards" = 0, :170-205 "parallel" = 1). */
int obca_scenario_obstacle_points(int scenario, int cap, double* ox, double* oy, int* n_out);

/* main.jl:215-248 in one call: Hybrid A* from x0 = (x, y, yaw) to xF, speed profile, veloSmooth, steering, down-sampling by sampleN.
 * Ts <= 0 selects the scenario's variable-time sampling time (main.jl:43-58).  On success *N_out = N and
 *   rx, ry, ryaw   N+1 values each (the down-sampled path, main.jl:237-239)
 *   xWS            (N+1) x 4 column-major: x, y, yaw, v        (main.jl:247)
 *   uWS            N x 2 column-major: steering, acceleration  (main.jl:248)
 * cap = capacity of the arrays in stages (N+1 <= cap). */
int obca_plan_warmstart(const double* x0, const double* xF, int scenario, double Ts, double L, int sampleN, int cap, double* rx, double* ry,
                        double* ryaw, double* xWS, double* uWS, int* N_out);

/* The same for B start poses (x0: 3 x B column-major) towards one goal -- the randomised sweeps of main.jl:165-168 --, on nthreads host
 * threads (<= 0: hardware concurrency).  Problem i writes N[i], status[i] (OBCA_PLAN_OK / NO_PATH / CAPACITY) and, with the stride cap,
 * rx / ry / ryaw [i*cap ..], xWS [i*4*cap ..] as (N[i]+1) x 4 column-major, uWS [i*2*cap ..] as N[i] x 2 column-major. */
int obca_plan_warmstart_batch(int B, const double* x0, const double* xF, int scenario, double Ts, double L, int sampleN, int cap, int nthreads,
                              double* rx, double* ry, double* ryaw, double* xWS, double* uWS, int* N, int* status);

/* The per-pose body of obca_plan_warmstart among any obstacle point cloud (ox[i], oy[i]), i < n_ob, for B start poses x0 and a goal per
 * pose xF (both 3 x B column-major: x, y, yaw), on nthreads host threads (<= 0: hardware concurrency).  Ts > 0 is the sampling time of the
 * warm start and L the wheelbase of the steering extraction, both used as given.  Outputs as obca_plan_warmstart_batch, plus
 * expansions[i] (may be NULL): the nodes pose i's search expanded.  The heuristic's obstacle map is built once per call; its distances
 * once per pose.  Return OBCA_PLAN_BAD_ARG (nothing written) for B < 0, a null array, n_ob <= 0, Ts <= 0, sampleN < 1 or cap < 2, else
 * OBCA_PLAN_OK.  With one goal repeated and a demo cloud it writes what obca_plan_warmstart_batch writes, byte for byte.
 * GPU twin: obca_plan_parking_warmstart_goals in include/obca.h, with the same search decisions and expansion counts. */
int obca_plan_warmstart_cloud_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                                    int sampleN, int cap, int nthreads, double* rx, double* ry, double* ryaw, double* xWS, double* uWS, int* N,
                                    int* status, int* expansions);

/* 3-D grid A* of the quadcopter flow (a_star_3D.jl:49-154, mainQuadcopter.jl:122-135) for B start / goal pairs among one obstacle point
 * cloud, on nthreads host threads (<= 0: hardware concurrency).  The decisions are those of the Python restatement
 * obca_b200/planner/a_star_3d.py (calc_astar_path), bit for bit.
 *   x0, xF: 3 x B column-major start / goal positions (each pair its own); ox, oy, oz: n_ob >= 0 obstacle points; lo, hi: the two bound
 *   corners (x, y, z) of the map, in raw units -- not divided by reso, as in calc_obstacle_map; reso > 0: the cell size.
 * Pair i writes status[i] (OBCA_PLAN_OK / NO_PATH / CAPACITY), expansions[i] (may be NULL: cells closed, the goal included) and, on OK,
 * N[i] = points - 1 and the path, start first, as cell * reso into rx / ry / rz [i*cap ..]; on CAPACITY (more than cap points) only N[i].
 * Return OBCA_PLAN_BAD_ARG (no output written) for B < 0, a null array, n_ob < 0, reso <= 0, cap < 1, a non-finite coordinate, a map of
 * more than 2^27 cells or a start / goal more than 2^30 cells away from it; else OBCA_PLAN_OK.
 * GPU twin: obca_plan_quadcopter_warmstart_batch in include/obca.h; both compile the search from obca_b200/planner/csrc/obca_astar3d_core.h. */
int obca_astar3d_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz, int n_ob,
                       const double* lo, const double* hi, double reso, int cap, int nthreads, double* rx, double* ry, double* rz, int* N,
                       int* status, int* expansions);

/* The obstacle map both 3-D A* entries build (calc_obstacle_map of a_star_3d.py for the points divided by reso): mn[3] (the cell of map
 * index 0), w[3] (the map's extent), and, when w0 * w1 * w2 <= cap, blocked[(ix * w1 + iy) * w2 + iz] = 1 for a blocked cell, else 0
 * (OBCA_PLAN_CAPACITY otherwise).  Used by tests. */
int obca_astar3d_obstacle_map(const double* ox, const double* oy, const double* oz, int n_ob, const double* lo, const double* hi, double reso,
                              long long* mn, int* w, unsigned char* blocked, long long cap);

/* Reeds-Shepp shortest path length between two poses for maximum curvature maxc (reeds_shepp.jl:79-96); used by tests. */
double obca_reeds_shepp_length(double sx, double sy, double syaw, double gx, double gy, double gyaw, double maxc);

#ifdef __cplusplus
}
#endif
#endif
