// emul_plan_goals.cpp -- DEVELOPMENT emulation of the GPU Hybrid A* planner with a goal per start pose (obca_b200/csrc/obca_plan.cuh:
// k_plan_hmap's relaxation and k_plan's search) on one host thread, with the GPU entry's host set-up, so that tests/test_plan_goals.py
// can compare them with libobca_planner.so and calc_dist_policy bit for bit.  (tests/emul/emul_plan.cpp emulates the one-goal entry.)
// Test tool only.
// Build: g++ -O2 -std=c++17 -ffp-contract=off (the host planner's flags).
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/obca_planner.h"
#include "../../obca_b200/csrc/obca_plan.cuh"

using namespace obca_plan;

namespace {
struct CtaSeq {
  int tid() const { return 0; }
  int nth() const { return 1; }
  void sync() const {}
  int sync_or(int v) const { return v; }
};

// obca_plan_parking_warmstart_goals's arguments and outputs (max_nodes > 0 here): the maps are relaxed as k_plan_hmap does, then the
// poses are planned one after the other.
int plan_goals(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
               int sampleN, int max_expansions, int max_nodes, int cap, double* rx, double* ry, double* ryaw, double* xWS, double* uWS, int* N,
               int* status, int* expansions) {
  if (B < 0 || !x0 || !xF || !ox || !oy || n_ob <= 0 || !(Ts > 0) || sampleN < 1 || cap < 2 || max_nodes < 1 || motion_nlist() != PLAN_NLIST)
    return OBCA_PLAN_BAD_ARG;
  PlanSetup S;
  plan_setup(S, B, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap);
  const size_t G = S.gcell.size() / 2;
  std::vector<double> maps(S.C.hcells * G + 1);
  for (size_t g = 0; g < G; ++g)
    hmap_one(CtaSeq(), S.H.obmap.data(), S.H.xw, S.H.yw, S.gcell[2 * g] - S.H.minx, S.gcell[2 * g + 1] - S.H.miny, std::sqrt(2.0),
             maps.data() + g * S.C.hcells);
  S.C.pmap = maps.data();
  const size_t P = plan_path_max(cap, sampleN);
  std::vector<int> table(S.C.table_size, -1), rsseg(RS_MAX_PTS);
  std::vector<PNode> pool(max_nodes);
  std::vector<HeapItem> heap(max_nodes);
  std::vector<double> rsx(RS_MAX_PTS), rsy(RS_MAX_PTS), rsyaw(RS_MAX_PTS), rspar(RS_MAX_PTS), px(P), py(P), pyaw(P), work(9 * (P + 40));
  PlanScratch W{table.data(), pool.data(), heap.data(), rsx.data(), rsy.data(), rsyaw.data(), rspar.data(), rsseg.data(),
                px.data(), py.data(), pyaw.data(), work.data()};
  PlanIO io{x0, rx, ry, ryaw, xWS, uWS, N, status, expansions};
  std::vector<PlanSmem> sm(1);
  for (int p = 0; p < B; ++p) plan_one(CtaSeq(), S.C, W, sm[0], io, p);
  return OBCA_PLAN_OK;
}
}  // namespace

// obca_plan_parking_warmstart_goals's arguments and outputs (xF: 3 x B, max_nodes > 0 here), planned one pose after the other.
extern "C" int emul_plan_goals(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                               int sampleN, int max_expansions, int max_nodes, int cap, double* rx, double* ry, double* ryaw, double* xWS,
                               double* uWS, int* N, int* status, int* expansions) {
  return plan_goals(B, x0, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap, rx, ry, ryaw, xWS, uWS, N, status, expansions);
}

// The heuristic maps of G goals (2 x G: gx, gy) among the cloud (ox, oy), each three ways, into maps (3 x G x xw x yw when it holds cap
// entries; mn[2] / w[2] are written first): which = 0 calc_dist_policy, 1 its two parts (calc_heur_grid, then dist_from_goal), 2 the
// relaxation of k_plan_hmap on one thread.
extern "C" int emul_plan_hmaps(int G, const double* goals, const double* ox, const double* oy, int n_ob, long long* mn, int* w, double* maps,
                               long long cap) {
  if (G < 0 || !goals || !ox || !oy || n_ob <= 0 || !mn || !w) return OBCA_PLAN_BAD_ARG;
  const std::vector<double> vx(ox, ox + n_ob), vy(oy, oy + n_ob);
  const HeurGrid H = calc_heur_grid(vx, vy, XY_GRID_RESOLUTION, VEHICLE_RADIUS);
  mn[0] = H.minx; mn[1] = H.miny; w[0] = H.xw; w[1] = H.yw;
  const size_t cells = (size_t)H.xw * H.yw;
  if (!maps || (long long)(3 * cells * G) > cap) return OBCA_PLAN_CAPACITY;
  for (int g = 0; g < G; ++g) {
    const double gx = goals[2 * g], gy = goals[2 * g + 1];
    long g0, g1;
    heur_goal_cell(gx, gy, XY_GRID_RESOLUTION, g0, g1);
    const DistPolicy a = calc_dist_policy(gx, gy, vx, vy, XY_GRID_RESOLUTION, VEHICLE_RADIUS), b = dist_from_goal(H, g0, g1);
    std::memcpy(maps + g * cells, a.pmap.data(), cells * sizeof(double));
    std::memcpy(maps + (G + g) * cells, b.pmap.data(), cells * sizeof(double));
    hmap_one(CtaSeq(), H.obmap.data(), H.xw, H.yw, g0 - H.minx, g1 - H.miny, std::sqrt(2.0), maps + (2 * (size_t)G + g) * cells);
  }
  return OBCA_PLAN_OK;
}
