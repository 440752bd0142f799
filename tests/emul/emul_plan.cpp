// emul_plan.cpp -- DEVELOPMENT emulation of the GPU Hybrid A* planner (obca_b200/csrc/obca_plan.cuh) on one host thread.
// Compiles the search the kernel runs, with its heap, cell table and node pool, and the GPU entry's host set-up, so that
// tests/test_plan_device.py can compare it with libobca_planner.so bit for bit.  Test tool only.
// Build: g++ -O2 -std=c++17 -ffp-contract=off (the host planner's flags).
#include <vector>

#include "../../include/obca_planner.h"
#include "../../obca_b200/csrc/obca_plan.cuh"

using namespace obca_plan;

namespace {
struct CtaSeq {
  int tid() const { return 0; }
  int nth() const { return 1; }
  void sync() const {}
};
}  // namespace

// obca_plan_parking_warmstart_batch's arguments and outputs (max_nodes > 0 here), planned one pose after the other.
extern "C" int emul_plan_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                               int sampleN, int max_expansions, int max_nodes, int cap, double* rx, double* ry, double* ryaw, double* xWS,
                               double* uWS, int* N, int* status, int* expansions) {
  if (B < 0 || !x0 || !xF || !ox || !oy || n_ob <= 0 || !(Ts > 0) || sampleN < 1 || cap < 2 || max_nodes < 1 || motion_nlist() != PLAN_NLIST)
    return OBCA_PLAN_BAD_ARG;
  PlanSetup S;
  plan_setup(S, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap);
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
