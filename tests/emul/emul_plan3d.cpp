// emul_plan3d.cpp -- DEVELOPMENT emulation of the GPU 3-D A* planner (k_plan3d of obca_b200/csrc/obca_plan3d.cu) on one host thread.
// Runs the search source the kernel runs (obca_astar3d_core.h) with the kernel's fixed scratch -- one cell table, node pool and queue of
// max_nodes / max_queue entries, reused pair after pair -- so that tests/test_plan_quad_native.py can check its POOL_FULL outcomes and
// its table reset against libobca_planner.so.  Also reports the nodes and the longest queue of every search.  Test tool only.
// Build: g++ -O2 -std=c++17 -ffp-contract=off (the host planner's flags).
#include <string>
#include <vector>

#include "../../include/obca_planner.h"
#include "../../obca_b200/planner/csrc/obca_astar3d_core.h"

using namespace obca_astar3d;

extern "C" int emul_plan3d_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz, int n_ob,
                                 const double* lo, const double* hi, double reso, int max_nodes, int max_queue, int cap, double* rx,
                                 double* ry, double* rz, int* N, int* status, int* expansions, int* nodes, int* queue_max) {
  A3Setup S;
  std::string why;
  if (!rx || !ry || !rz || !N || !status || max_nodes < 1 || max_queue < 1) return OBCA_PLAN_BAD_ARG;
  if (astar3d_setup(S, why, B, x0, xF, ox, oy, oz, n_ob, lo, hi, reso, cap)) return OBCA_PLAN_BAD_ARG;
  S.C.max_nodes = max_nodes;
  S.C.max_queue = max_queue;
  std::vector<int> table(S.cells > 0 ? S.cells : 1, -1);
  std::vector<A3Node> pool(max_nodes);
  std::vector<A3Item> queue(max_queue);
  const A3IO io{S.s.data(), S.g.data(), rx, ry, rz, N, status, expansions, nodes, queue_max};
  for (int p = 0; p < B; ++p) astar3d_one(SeqLanes(), S.C, A3Scratch{table.data(), pool.data(), queue.data()}, io, p);
  for (long long c = 0; c < S.cells; ++c)
    if (table[c] != -1) return -1;      // the table must be empty after every search
  return OBCA_PLAN_OK;
}
