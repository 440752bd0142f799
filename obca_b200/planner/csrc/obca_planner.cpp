// obca_planner.cpp -- host-side warm-start producer behind include/obca_planner.h (plain C++17, no CUDA): Hybrid A* with the
// Reeds-Shepp analytic expansion, the vehicle / obstacle-point collision test, the grid heuristic, veloSmooth and the warm-start
// extraction of main.jl:215-248.  The algorithm's pieces live in obca_plan_core.h, which the GPU planner of libobca.so
// (obca_b200/csrc/obca_plan.cu) compiles as well; this file holds the host search (hash maps and a priority queue) and the C entries.
// Same algorithms, in the same order of floating-point operations, as the Python restatement obca_b200/planner/*.py (which cites the
// reference line by line and documents its quirks); tests/test_planner_native.py compares the two.
// Build: g++ -O2 -std=c++17 -ffp-contract=off -shared -fPIC (see __graft_entry__.build()).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <queue>
#include <thread>
#include <tuple>
#include <unordered_map>
#include <vector>

#include "../../../include/obca_planner.h"
#include "obca_astar3d_core.h"
#include "obca_plan_core.h"

namespace {

using std::vector;
using namespace obca_plan;
const double INF = std::numeric_limits<double>::infinity();

// =====================================================================================================================
// Reeds-Shepp (obca_b200/planner/reeds_shepp.py)
// =====================================================================================================================
RsSet generate_path(const double q0[3], const double q1[3], double maxc) {
  double x, y, phi, xb, yb;
  rs_frame(q0, q1, maxc, x, y, phi, xb, yb);
  RsSet s;
  s.n = 0;
  for (int j = 0; j < RS_NCAND; ++j) {
    RsCand c;
    if (rs_candidate(j, x, y, phi, xb, yb, c)) set_path(s, c);
  }
  return s;
}
// calc_shortest_path (reeds_shepp.jl:59-76): the shortest candidate's course in global coordinates, its lengths scaled by 1/maxc.
// Only the shortest candidate is interpolated: the pick depends on the lengths alone.
bool calc_shortest_path(double sx, double sy, double syaw, double gx, double gy, double gyaw, double maxc, double step_size, RsCand& best,
                        vector<double>& px, vector<double>& py, vector<double>& pyaw) {
  const double q0[3] = {sx, sy, syaw}, q1[3] = {gx, gy, gyaw};
  const RsSet s = generate_path(q0, q1, maxc);
  const int bi = rs_shortest(s, maxc);
  if (bi < 0) return false;
  best = s.p[bi];
  const double step = step_size * maxc;
  const int npoint = rs_npoint(s.L[bi], best.n, step);
  vector<int> seg(npoint);
  vector<double> par(npoint);
  int n = rs_course_plan(best, step, npoint, seg.data(), par.data());
  double org[RS_MAX_SEG][3];
  rs_origins(best, maxc, org);
  vector<double> lx(n), ly(n), lyaw(n);
  for (int i = 0; i < n; ++i) rs_point(best, maxc, org, seg[i], par[i], lx[i], ly[i], lyaw[i]);
  while (n > 0 && lx[n - 1] == 0.0) --n;
  const double cq = std::cos(-q0[2]), sq = std::sin(-q0[2]);
  px.resize(n); py.resize(n); pyaw.resize(n);
  for (int i = 0; i < n; ++i) rs_to_global(q0, cq, sq, lx[i], ly[i], lyaw[i], px[i], py[i], pyaw[i]);
  for (int i = 0; i < best.n; ++i) best.len[i] = best.len[i] / maxc;
  return true;
}

bool check_collision(const vector<double>& x, const vector<double>& y, const vector<double>& yaw, const ObGridView& g) {      // true = free
  for (size_t k = 0; k < x.size(); ++k)
    if (pose_collides(g, x[k], y[k], yaw[k])) return false;
  return true;
}

// =====================================================================================================================
// Hybrid A* (obca_b200/planner/hybrid_a_star.py)
// =====================================================================================================================
struct Node {
  long xind, yind, yawind;
  bool direction;
  vector<double> x, y, yaw;
  double steer, cost;
  long pind;
};
// HG: the heuristic's obstacle map of (ox, oy) at xyreso (calc_heur_grid), which does not depend on the goal; expansions: the nodes
// expanded, on every outcome.
int hybrid_astar(double sx, double sy, double syaw, double gx, double gy, double gyaw, const vector<double>& ox, const vector<double>& oy,
                 const HeurGrid& HG, double xyreso, double yawreso, long max_expansions, vector<double>& rx, vector<double>& ry,
                 vector<double>& ryaw, long& expansions) {
  syaw = pi_2_pi(syaw); gyaw = pi_2_pi(gyaw);
  const Config c = calc_config(ox, oy, xyreso, yawreso);
  Obstacles ob; ob.ox = ox; ob.oy = oy; ob.build();
  const ObGridView grid = ob.view();
  Node nstart{jround(sx / xyreso), jround(sy / xyreso), jround(syaw / yawreso), true, {sx}, {sy}, {syaw}, 0.0, 0.0, -1};
  Node ngoal{jround(gx / xyreso), jround(gy / xyreso), jround(gyaw / yawreso), true, {gx}, {gy}, {gyaw}, 0.0, 0.0, -1};
  long g0, g1;
  heur_goal_cell(gx, gy, xyreso, g0, g1);
  const DistPolicy H = dist_from_goal(HG, g0, g1);
  auto cost_of = [&](const Node& n) { return n.cost + H_COST * heuristic(H.pmap.data(), H.minx, H.miny, H.xw, H.yw, n.xind, n.yind); };
  std::unordered_map<long, Node> open_, closed;
  const long sid = calc_index(nstart.xind, nstart.yind, nstart.yawind, c);
  open_[sid] = nstart;
  typedef std::tuple<double, long, long> Item;      // (priority, insertion tick, node id): heapq order of the Python restatement
  std::priority_queue<Item, vector<Item>, std::greater<Item> > pq;
  long tick = 0;
  pq.push(Item(cost_of(nstart), tick, sid));
  vector<double> us, ds, tanu;
  motion_inputs(us, ds, tanu);
  const int nlist = motion_nlist();
  const double maxc = max_curvature();
  Node final_node;
  expansions = 0;
  for (;;) {
    if (open_.empty() || pq.empty() || expansions > max_expansions) return OBCA_PLAN_NO_PATH;
    const long c_id = std::get<2>(pq.top());
    pq.pop();
    auto it = open_.find(c_id);
    if (it == open_.end()) continue;
    Node cur = it->second;
    ++expansions;
    RsCand ap;
    vector<double> apx, apy, apyaw;
    const bool have = calc_shortest_path(cur.x.back(), cur.y.back(), cur.yaw.back(), ngoal.x.back(), ngoal.y.back(), ngoal.yaw.back(), maxc,
                                         MOTION_RESOLUTION, ap, apx, apy, apyaw);
    if (have && check_collision(apx, apy, apyaw, grid)) {
      if (apx.size() >= 2) {
        cur.x.insert(cur.x.end(), apx.begin() + 1, apx.end() - 1);
        cur.y.insert(cur.y.end(), apy.begin() + 1, apy.end() - 1);
        cur.yaw.insert(cur.yaw.end(), apyaw.begin() + 1, apyaw.end() - 1);
      }
      cur.cost += calc_rs_path_cost(ap.len, ap.ty, ap.n);
      final_node = cur;
      break;
    }
    open_.erase(it);
    closed[c_id] = cur;
    for (size_t m = 0; m < us.size(); ++m) {
      Node node;
      node.x.assign(nlist, 0.0); node.y.assign(nlist, 0.0); node.yaw.assign(nlist, 0.0);
      next_poses(cur.x.back(), cur.y.back(), cur.yaw.back(), ds[m], tanu[m], nlist, node.x.data(), node.y.data(), node.yaw.data());
      node.xind = jround(node.x.back() / c.xyreso); node.yind = jround(node.y.back() / c.xyreso); node.yawind = jround(node.yaw.back() / c.yawreso);
      node.direction = ds[m] > 0; node.steer = us[m]; node.cost = cur.cost + step_cost(cur.direction, cur.steer, us[m], ds[m]); node.pind = c_id;
      if (!(0 < node.xind - c.minx && node.xind - c.minx < c.xw) || !(0 < node.yind - c.miny && node.yind - c.miny < c.yw)) continue;
      if (!check_collision(node.x, node.y, node.yaw, grid)) continue;
      const long nid = calc_index(node.xind, node.yind, node.yawind, c);
      if (closed.count(nid) || open_.count(nid)) continue;
      const double pr = cost_of(node);
      open_[nid] = std::move(node);
      ++tick;
      pq.push(Item(pr, tick, nid));
    }
  }
  // get_final_path (hybrid_a_star.jl:506-534): goal point, then the node chain back to the start cell
  vector<double> bx = ngoal.x, by = ngoal.y, byaw = ngoal.yaw;
  Node n = final_node;
  for (;;) {
    bx.insert(bx.end(), n.x.rbegin(), n.x.rend());
    by.insert(by.end(), n.y.rbegin(), n.y.rend());
    byaw.insert(byaw.end(), n.yaw.rbegin(), n.yaw.rend());
    if (n.xind == nstart.xind && n.yind == nstart.yind && n.yawind == nstart.yawind) break;
    auto f = closed.find(n.pind);
    if (f == closed.end()) return OBCA_PLAN_NO_PATH;
    n = f->second;
  }
  rx.assign(bx.rbegin(), bx.rend()); ry.assign(by.rbegin(), by.rend()); ryaw.assign(byaw.rbegin(), byaw.rend());
  return OBCA_PLAN_OK;
}

vector<double> frange(double a, double b, double step) {
  const int n = (int)std::floor((b - a) / step + 1e-9);
  vector<double> r;
  for (int i = 0; i <= n; ++i) r.push_back(a + i * step);
  return r;
}
int obstacle_points(int scenario, vector<double>& ox, vector<double>& oy) {
  ox.clear(); oy.clear();
  if (scenario == 0) {
    for (double v : frange(-12.0, -1.3, 0.1)) { ox.push_back(v); oy.push_back(5.0); }
    for (int i = -2; i < 6; ++i) { ox.push_back(-1.3); oy.push_back((double)i); }
    for (int i = -2; i < 6; ++i) { ox.push_back(1.3); oy.push_back((double)i); }
    for (double v : frange(1.3, 12.0, 0.1)) { ox.push_back(v); oy.push_back(5.0); }
    for (int i = -12; i < 13; ++i) { ox.push_back((double)i); oy.push_back(11.0); }
  } else if (scenario == 1) {
    for (double v : frange(-12.0, -3.0, 0.1)) { ox.push_back(v); oy.push_back(5.0); }
    for (int i = -2; i < 6; ++i) { ox.push_back(-3.0); oy.push_back((double)i); }
    for (int i = -3; i < 4; ++i) { ox.push_back((double)i); oy.push_back(2.5); }
    for (int i = -2; i < 6; ++i) { ox.push_back(3.0); oy.push_back((double)i); }
    for (double v : frange(3.0, 12.0, 0.1)) { ox.push_back(v); oy.push_back(5.0); }
    for (int i = -12; i < 13; ++i) { ox.push_back((double)i); oy.push_back(11.5); }
  } else {
    return OBCA_PLAN_BAD_ARG;
  }
  return OBCA_PLAN_OK;
}

// main.jl:215-248 for one start pose x0 and goal xF among the points (ox, oy) whose heuristic obstacle map is HG: Hybrid A*, speed profile,
// veloSmooth, steering, down-sampling by sampleN.  *expanded (may be null): the nodes expanded.
int plan_warmstart_one(const double* x0, const double* xF, const vector<double>& ox, const vector<double>& oy, const HeurGrid& HG, double Ts,
                       double L, int sampleN, int cap, double* rx, double* ry, double* ryaw, double* xWS, double* uWS, int* N_out, int* expanded) {
  vector<double> px, py, pyaw;
  long nexp = 0;
  const int rc = hybrid_astar(x0[0], x0[1], x0[2], xF[0], xF[1], xF[2], ox, oy, HG, XY_GRID_RESOLUTION, YAW_GRID_RESOLUTION, 200000, px, py, pyaw,
                              nexp);
  if (expanded) *expanded = (int)nexp;
  if (rc) return rc;
  // main.jl:222-248
  const int n = (int)px.size();
  const double dt = Ts / sampleN;
  vector<double> rv(n, 0.0), v(n), a(n > 0 ? n - 1 : 0), work(5 * (size_t)(n + 40));
  for (int i = 0; i + 1 < n; ++i) rv[i] = ws_speed(px.data(), py.data(), pyaw.data(), i, dt);
  velo_smooth(rv.data(), n, WS_AMAX, dt, work.data(), v.data(), a.data());
  vector<double> delta(n > 0 ? n - 1 : 0);
  for (int i = 0; i + 1 < n; ++i) delta[i] = ws_steer(pyaw.data(), v.data(), i, L);
  const int ns = (n + sampleN - 1) / sampleN;      // len(rx[::sampleN])
  *N_out = ns - 1;
  if (ns > cap || !rx || !ry || !ryaw || !xWS || !uWS) return OBCA_PLAN_CAPACITY;
  ws_store(px.data(), py.data(), pyaw.data(), v.data(), a.data(), delta.data(), n, sampleN, rx, ry, ryaw, xWS, uWS);
  return OBCA_PLAN_OK;
}

// plan_warmstart_one for B poses on nthreads host threads (<= 0: hardware concurrency); pose i's goal is xF + goal_stride * i.  The
// heuristic's obstacle map is built once for the batch.
void plan_warmstart_many(int B, const double* x0, const double* xF, size_t goal_stride, const vector<double>& ox, const vector<double>& oy,
                         double Ts, double L, int sampleN, int cap, int nthreads, double* rx, double* ry, double* ryaw, double* xWS, double* uWS,
                         int* N, int* status, int* expansions) {
  const HeurGrid HG = calc_heur_grid(ox, oy, XY_GRID_RESOLUTION, VEHICLE_RADIUS);
  if (nthreads <= 0) nthreads = (int)std::thread::hardware_concurrency();
  if (nthreads < 1) nthreads = 1;
  if (nthreads > B) nthreads = B > 0 ? B : 1;
  std::atomic<int> next(0);
  auto work = [&]() {
    for (;;) {
      const int i = next.fetch_add(1);
      if (i >= B) break;
      status[i] = plan_warmstart_one(x0 + 3 * (size_t)i, xF + goal_stride * i, ox, oy, HG, Ts, L, sampleN, cap, rx + (size_t)i * cap,
                                     ry + (size_t)i * cap, ryaw + (size_t)i * cap, xWS + (size_t)i * 4 * cap, uWS + (size_t)i * 2 * cap, N + i,
                                     expansions ? expansions + i : nullptr);
    }
  };
  vector<std::thread> pool;
  for (int t = 1; t < nthreads; ++t) pool.emplace_back(work);
  work();
  for (auto& t : pool) t.join();
}

}  // namespace

extern "C" {

int obca_planner_version(void) { return 100; }

int obca_hybrid_astar(double sx, double sy, double syaw, double gx, double gy, double gyaw, const double* ox, const double* oy, int n_ob,
                      double xyreso, double yawreso, int max_expansions, int cap, double* rx, double* ry, double* ryaw, int* n_out) {
  if (!ox || !oy || n_ob <= 0 || !n_out) return OBCA_PLAN_BAD_ARG;
  vector<double> vx(ox, ox + n_ob), vy(oy, oy + n_ob), px, py, pyaw;
  const double xy = xyreso > 0 ? xyreso : XY_GRID_RESOLUTION;
  long nexp;
  const int rc = hybrid_astar(sx, sy, syaw, gx, gy, gyaw, vx, vy, calc_heur_grid(vx, vy, xy, VEHICLE_RADIUS), xy,
                              yawreso > 0 ? yawreso : YAW_GRID_RESOLUTION, max_expansions > 0 ? max_expansions : 200000, px, py, pyaw, nexp);
  if (rc) return rc;
  *n_out = (int)px.size();
  if ((int)px.size() > cap || !rx || !ry || !ryaw) return OBCA_PLAN_CAPACITY;
  std::memcpy(rx, px.data(), px.size() * sizeof(double)); std::memcpy(ry, py.data(), py.size() * sizeof(double));
  std::memcpy(ryaw, pyaw.data(), pyaw.size() * sizeof(double));
  return OBCA_PLAN_OK;
}

int obca_scenario_obstacle_points(int scenario, int cap, double* ox, double* oy, int* n_out) {
  vector<double> vx, vy;
  const int rc = obstacle_points(scenario, vx, vy);
  if (rc) return rc;
  if (n_out) *n_out = (int)vx.size();
  if ((int)vx.size() > cap || !ox || !oy) return OBCA_PLAN_CAPACITY;
  std::memcpy(ox, vx.data(), vx.size() * sizeof(double)); std::memcpy(oy, vy.data(), vy.size() * sizeof(double));
  return OBCA_PLAN_OK;
}

int obca_plan_warmstart(const double* x0, const double* xF, int scenario, double Ts, double L, int sampleN, int cap, double* rx, double* ry,
                        double* ryaw, double* xWS, double* uWS, int* N_out) {
  if (!x0 || !xF || !N_out || sampleN < 1) return OBCA_PLAN_BAD_ARG;
  if (Ts <= 0) Ts = (scenario == 0 ? 0.6 : 0.9) / 3 * sampleN;
  if (L <= 0) L = 2.7;
  vector<double> ox, oy;
  const int rc = obstacle_points(scenario, ox, oy);
  if (rc) return rc;
  return plan_warmstart_one(x0, xF, ox, oy, calc_heur_grid(ox, oy, XY_GRID_RESOLUTION, VEHICLE_RADIUS), Ts, L, sampleN, cap, rx, ry, ryaw, xWS,
                            uWS, N_out, nullptr);
}

int obca_plan_warmstart_batch(int B, const double* x0, const double* xF, int scenario, double Ts, double L, int sampleN, int cap, int nthreads,
                              double* rx, double* ry, double* ryaw, double* xWS, double* uWS, int* N, int* status) {
  if (B < 0 || !x0 || !xF || !rx || !ry || !ryaw || !xWS || !uWS || !N || !status || cap < 2) return OBCA_PLAN_BAD_ARG;
  vector<double> ox, oy;
  const int rc = sampleN < 1 ? OBCA_PLAN_BAD_ARG : obstacle_points(scenario, ox, oy);
  if (rc) {      // what obca_plan_warmstart reports for every pose
    for (int i = 0; i < B; ++i) status[i] = rc;
    return OBCA_PLAN_OK;
  }
  if (Ts <= 0) Ts = (scenario == 0 ? 0.6 : 0.9) / 3 * sampleN;
  if (L <= 0) L = 2.7;
  plan_warmstart_many(B, x0, xF, 0, ox, oy, Ts, L, sampleN, cap, nthreads, rx, ry, ryaw, xWS, uWS, N, status, nullptr);
  return OBCA_PLAN_OK;
}

int obca_plan_warmstart_cloud_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L,
                                    int sampleN, int cap, int nthreads, double* rx, double* ry, double* ryaw, double* xWS, double* uWS, int* N,
                                    int* status, int* expansions) {
  if (B < 0 || !x0 || !xF || !ox || !oy || n_ob <= 0 || !(Ts > 0) || sampleN < 1 || cap < 2 || !rx || !ry || !ryaw || !xWS || !uWS || !N ||
      !status)
    return OBCA_PLAN_BAD_ARG;
  plan_warmstart_many(B, x0, xF, 3, vector<double>(ox, ox + n_ob), vector<double>(oy, oy + n_ob), Ts, L, sampleN, cap, nthreads, rx, ry, ryaw,
                      xWS, uWS, N, status, expansions);
  return OBCA_PLAN_OK;
}

int obca_astar3d_batch(int B, const double* x0, const double* xF, const double* ox, const double* oy, const double* oz, int n_ob,
                       const double* lo, const double* hi, double reso, int cap, int nthreads, double* rx, double* ry, double* rz, int* N,
                       int* status, int* expansions) {
  namespace a3 = obca_astar3d;
  if (!rx || !ry || !rz || !N || !status) return OBCA_PLAN_BAD_ARG;
  a3::A3Setup S;
  std::string why;
  if (a3::astar3d_setup(S, why, B, x0, xF, ox, oy, oz, n_ob, lo, hi, reso, cap)) return OBCA_PLAN_BAD_ARG;
  if (nthreads <= 0) nthreads = (int)std::thread::hardware_concurrency();
  if (nthreads < 1) nthreads = 1;
  if (nthreads > B) nthreads = B > 0 ? B : 1;
  const a3::A3IO io{S.s.data(), S.g.data(), rx, ry, rz, N, status, expansions, nullptr, nullptr};
  const long long most_nodes = S.cells + 1;      // every map cell and a start outside the map
  std::atomic<int> next(0);
  auto work = [&]() {
    // one scratch per thread, reused pair after pair; a search that outgrows it is repeated with twice the room (same decisions)
    a3::A3Const C = S.C;
    C.max_nodes = (int)std::min<long long>(most_nodes, 1 << 16);
    C.max_queue = 1 << 14;
    vector<int> table(S.cells > 0 ? S.cells : 1, -1);
    vector<a3::A3Node> pool(C.max_nodes);
    vector<a3::A3Item> queue(C.max_queue);
    for (;;) {
      const int i = next.fetch_add(1);
      if (i >= B) break;
      for (;;) {
        a3::astar3d_one(a3::SeqLanes(), C, a3::A3Scratch{table.data(), pool.data(), queue.data()}, io, i);
        if (status[i] != a3::A3_POOL_FULL) break;
        C.max_nodes = (int)std::min<long long>(most_nodes, 2LL * C.max_nodes);
        C.max_queue *= 2;
        pool.resize(C.max_nodes);
        queue.resize(C.max_queue);
      }
    }
  };
  vector<std::thread> threads;
  for (int t = 1; t < nthreads; ++t) threads.emplace_back(work);
  work();
  for (auto& t : threads) t.join();
  return OBCA_PLAN_OK;
}

int obca_astar3d_obstacle_map(const double* ox, const double* oy, const double* oz, int n_ob, const double* lo, const double* hi, double reso,
                              long long* mn, int* w, unsigned char* blocked, long long cap) {
  namespace a3 = obca_astar3d;
  if (!mn || !w) return OBCA_PLAN_BAD_ARG;
  a3::A3Setup S;
  std::string why;
  const double zero[3] = {0.0, 0.0, 0.0};
  if (a3::astar3d_setup(S, why, 0, zero, zero, ox, oy, oz, n_ob, lo, hi, reso, 1)) return OBCA_PLAN_BAD_ARG;
  for (int a = 0; a < 3; ++a) { mn[a] = S.C.mn[a]; w[a] = S.C.w[a]; }
  if (S.cells > cap || !blocked) return OBCA_PLAN_CAPACITY;
  for (long long c = 0; c < S.cells; ++c) blocked[c] = (S.map[c >> 5] >> (c & 31)) & 1u;
  return OBCA_PLAN_OK;
}

double obca_reeds_shepp_length(double sx, double sy, double syaw, double gx, double gy, double gyaw, double maxc) {
  const double q0[3] = {sx, sy, syaw}, q1[3] = {gx, gy, gyaw};
  const RsSet s = generate_path(q0, q1, maxc);
  double best = INF;
  for (int i = 0; i < s.n; ++i) best = std::min(best, s.L[i] / maxc);
  return best;
}

}  // extern "C"
