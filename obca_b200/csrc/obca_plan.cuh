// obca_plan.cuh -- the GPU Hybrid A* search: one CTA plans one start pose at a time (obca_plan.cu), reproducing the host planner's
// decisions (obca_b200/planner/csrc/obca_planner.cpp) with a binary heap, a cell -> node table and a node pool instead of its hash maps.
// Written once for a CTA policy `Cta` (tid / nth / sync / sync_or): the kernel runs it with the threads of a CTA, the development emulation
// (tests/emul/emul_plan.cpp for one goal, tests/emul/emul_plan_goals.cpp for a goal per pose and the heuristic-map relaxation) with one
// host thread, so the emulation checks this very source against the host planner bit for bit.
//
// One expansion:
//   1. thread 0 pops the heap (priority cost + H_COST * h, then insertion tick; no trig, so the pops are those of std::priority_queue);
//   2. the 46 Reeds-Shepp candidate words in parallel; thread 0 dedups them in order (set_path) and picks the shortest (the last of
//      equally short ones), then runs the serial arc-parameter accumulation of generate_local_course;
//   3. the course points in parallel, then their collision tests ("any hit");
//   4. the 22 motion primitives' poses in parallel, then the collision tests of their 22 x 4 poses;
//   5. thread 0 inserts the free successors in the order m = 0..21 (an id only when it is neither open nor closed).
// Everything that sets a priority or an index is host arithmetic reproduced exactly; only sin / cos / atan2 / acos / tan / atan of the
// device's libm differ from the host's in their last bits.
#pragma once

#include "../planner/csrc/obca_plan_core.h"

namespace obca_plan {

constexpr int PLAN_NLIST = 4;          // poses per motion primitive (arc 0.3 m in steps of 0.1 m); the entry checks motion_nlist()
constexpr int RS_MAX_PTS = 4096;       // course points of one analytic expansion (a path of up to ~400 m)
constexpr int PLAN_NODE_POOL = 4;      // status: the node pool reached max_nodes (OBCA_PLAN_POOL_FULL in include/obca.h)

enum : int { NODE_OPEN = 1, NODE_CLOSED = 2 };

struct PNode {
  double x[PLAN_NLIST], y[PLAN_NLIST], yaw[PLAN_NLIST];
  double cost, steer;
  long id;
  int parent, np, xind, yind, yawind, dir;
  int state;
};
struct HeapItem {
  double pr;
  long tick;
  int node;
};
OBCA_PHD bool heap_less(const HeapItem& a, const HeapItem& b) { return a.pr < b.pr || (a.pr == b.pr && a.tick < b.tick); }

// Constants of one call, shared by every problem of the batch (pointers: device memory in the kernel, host memory in the emulation).
struct PlanConst {
  Config cfg;
  ObGridView grid;
  const double* pmap;              // the heuristic maps of the call's distinct goal cells, hcells entries each
  long hminx, hminy;
  int hxw, hyw;
  size_t hcells;                   // hxw * hyw
  const double* goals;             // the goals (x, y, yaw): pose p's at goals + 3 * per_pose * p
  const int* hidx;                 // hidx[per_pose * p]: the heuristic map of pose p's goal cell
  int per_pose;                    // 1: a goal per pose; 0: goals[0..2] and map 0 for every pose
  double maxc;
  double us[N_MOTION], ds[N_MOTION], tanu[N_MOTION];
  long max_expansions;
  int max_nodes;
  long table_size;                 // cells of the cell -> node table
  double dt, L;                    // Ts / sampleN, wheelbase of the steering extraction
  int sampleN, cap;
};
// Inputs / outputs of the batch: x0 3 x B, the outputs in the layout of obca_plan_warmstart_batch (stride cap).
struct PlanIO {
  const double* x0;
  double *rx, *ry, *ryaw, *xWS, *uWS;
  int *N, *status, *expansions;
};
// Scratch of one CTA (global memory), reused problem after problem.
struct PlanScratch {
  int* table;                      // table_size entries, -1 = no node; reset after every problem
  PNode* pool;                     // max_nodes
  HeapItem* heap;                  // max_nodes
  double *rsx, *rsy, *rsyaw, *rspar;
  int* rsseg;                      // RS_MAX_PTS each
  double *px, *py, *pyaw;          // the path: cap * sampleN each
  double* work;                    // 9 * (cap * sampleN + 40): veloSmooth (5 rows) + speed, smoothed speed, acceleration, steering
};
OBCA_PHD size_t plan_path_max(int cap, int sampleN) { return (size_t)cap * sampleN; }

// Host set-up of one call, shared by the batch: obstacle cell grid, the heuristic's obstacle map, the distinct goal cells, primitives.
// S.C points into S (host memory).  plan_setup(S, B, xF, ...): a goal per pose (xF 3 x B); S.C.pmap is left to the caller, who builds
// one map per goal cell (hmap_one) in goal-cell order.  plan_setup(S, xF, ...): one goal for every pose, its map built here by the host's
// Dijkstra (dist_from_goal).
struct PlanSetup {
  Obstacles ob;
  HeurGrid H;
  std::vector<double> goals;       // 3 per goal
  std::vector<long> gcell;         // (g0, g1) of each distinct goal cell, in order of first appearance
  std::vector<int> hidx;           // the goal cell of each goal
  std::vector<double> map;         // the one-goal set-up's heuristic map
  PlanConst C;
};
inline void plan_setup(PlanSetup& S, int B, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L, int sampleN,
                       int max_expansions, int max_nodes, int cap) {
  S.ob.ox.assign(ox, ox + n_ob); S.ob.oy.assign(oy, oy + n_ob); S.ob.build();
  PlanConst& C = S.C;
  C.cfg = calc_config(S.ob.ox, S.ob.oy, XY_GRID_RESOLUTION, YAW_GRID_RESOLUTION);
  C.grid = S.ob.view();
  S.H = calc_heur_grid(S.ob.ox, S.ob.oy, XY_GRID_RESOLUTION, VEHICLE_RADIUS);
  S.goals.assign(xF, xF + 3 * (size_t)B);
  S.gcell.clear(); S.hidx.assign(B, 0);
  std::unordered_map<uint64_t, int> seen;
  for (int p = 0; p < B; ++p) {
    long g0, g1;
    heur_goal_cell(xF[3 * (size_t)p], xF[3 * (size_t)p + 1], XY_GRID_RESOLUTION, g0, g1);
    const uint64_t key = ((uint64_t)(uint32_t)(int32_t)g0 << 32) | (uint32_t)(int32_t)g1;
    auto f = seen.find(key);
    if (f == seen.end()) { f = seen.emplace(key, (int)(S.gcell.size() / 2)).first; S.gcell.push_back(g0); S.gcell.push_back(g1); }
    S.hidx[p] = f->second;
  }
  C.pmap = nullptr; C.hminx = S.H.minx; C.hminy = S.H.miny; C.hxw = S.H.xw; C.hyw = S.H.yw; C.hcells = (size_t)S.H.xw * S.H.yw;
  C.goals = S.goals.data(); C.hidx = S.hidx.data(); C.per_pose = 1;
  C.maxc = max_curvature();
  std::vector<double> us, ds, tanu;
  motion_inputs(us, ds, tanu);
  for (int m = 0; m < N_MOTION; ++m) { C.us[m] = us[m]; C.ds[m] = ds[m]; C.tanu[m] = tanu[m]; }
  C.max_expansions = max_expansions > 0 ? max_expansions : 200000;      // obca_plan_warmstart's budget
  C.max_nodes = max_nodes;
  C.table_size = (C.cfg.yaww + 1) * C.cfg.xw * C.cfg.yw;
  C.dt = Ts / sampleN; C.L = L; C.sampleN = sampleN; C.cap = cap;
}
inline void plan_setup(PlanSetup& S, const double* xF, const double* ox, const double* oy, int n_ob, double Ts, double L, int sampleN,
                       int max_expansions, int max_nodes, int cap) {
  plan_setup(S, 1, xF, ox, oy, n_ob, Ts, L, sampleN, max_expansions, max_nodes, cap);
  S.map = dist_from_goal(S.H, S.gcell[0], S.gcell[1]).pmap;
  S.C.pmap = S.map.data(); S.C.per_pose = 0;
}

// The heuristic map of one goal cell into d (xw * yw entries, the layout of DistPolicy::pmap); (gi, gj) = the goal cell - (minx, miny),
// its map coordinates.  d is the fixed point of d(v) = min(d(v), d(u) + c) over the 8 neighbours u of every target v, c = 1 or sqrt2 (the
// host libm's sqrt(2.0)), relaxed sweep after sweep until a sweep changes nothing.  Round-to-nearest addition is monotone and c >= 1, so
// the fixed point is unique -- every cell gets the smallest left-to-right sum over its paths from the goal -- and it is what
// dist_from_goal's Dijkstra computes, bit for bit, whatever the order of the updates.  The goal is a source even when it is blocked or
// outside the map; targets are the free cells of the strict interior (dist_from_goal's ok()); every other entry stays INF, the goal's
// own entry 0 when it lies in the map.  Every thread calls it.
template <class Cta>
OBCA_PHD void hmap_one(const Cta& cta, const char* obmap, int xw, int yw, long gi, long gj, double sqrt2, double* d) {
  const int t = cta.tid(), nt = cta.nth(), cells = xw * yw;
  for (int k = t; k < cells; k += nt) d[k] = (k / yw + 1 == gi && k % yw + 1 == gj) ? 0.0 : pinf();
  cta.sync();
  const int MX[8] = {1, 0, -1, 0, -1, -1, 1, 1}, MY[8] = {0, 1, 0, -1, -1, 1, -1, 1};
  for (;;) {
    int changed = 0;
    for (int k = t; k < cells; k += nt) {
      const int i = k / yw + 1, j = k % yw + 1;
      if (!(i < xw && j < yw) || obmap[k]) continue;
      double best = d[k];
      for (int m = 0; m < 8; ++m) {
        const int ni = i + MX[m], nj = j + MY[m];
        const double du = (ni == gi && nj == gj) ? 0.0 : ((1 <= ni && ni <= xw && 1 <= nj && nj <= yw) ? d[(ni - 1) * yw + (nj - 1)] : pinf());
        const double nc = du + (m < 4 ? 1.0 : sqrt2);
        if (nc < best) best = nc;
      }
      if (best < d[k]) { d[k] = best; changed = 1; }
    }
    if (!cta.sync_or(changed)) break;
  }
}

// CTA-shared state of one problem.
struct PlanSmem {
  int status;                      // -1 while searching, else OBCA_PLAN_* / PLAN_NODE_POOL
  int cur, heap_n, n_nodes, rs_n, rs_hit, have_rs, len;
  long tick, expansions, sid;
  double q[3], goal[3];             // goal: (gx, gy, pi_2_pi(gyaw)) of this pose
  const double* hmap;              // its heuristic map
  RsCand cand[RS_NCAND];
  bool cand_ok[RS_NCAND];
  RsSet set;
  RsCand best;
  double org[RS_MAX_SEG][3];
  double nx[N_MOTION][PLAN_NLIST], ny[N_MOTION][PLAN_NLIST], nyaw[N_MOTION][PLAN_NLIST];
  int nok[N_MOTION], hit[N_MOTION];
};

OBCA_PHD void heap_push(HeapItem* h, int& n, const HeapItem& it) {
  int i = n++;
  while (i > 0) {
    const int p = (i - 1) >> 1;
    if (!heap_less(it, h[p])) break;
    h[i] = h[p]; i = p;
  }
  h[i] = it;
}
OBCA_PHD HeapItem heap_pop(HeapItem* h, int& n) {
  const HeapItem top = h[0], last = h[--n];
  int i = 0;
  for (;;) {
    int c = 2 * i + 1;
    if (c >= n) break;
    if (c + 1 < n && heap_less(h[c + 1], h[c])) ++c;
    if (!heap_less(h[c], last)) break;
    h[i] = h[c]; i = c;
  }
  if (n > 0) h[i] = last;
  return top;
}

OBCA_PHD double node_priority(const PlanConst& C, const double* hmap, const PNode& n) {
  return n.cost + H_COST * heuristic(hmap, C.hminx, C.hminy, C.hxw, C.hyw, n.xind, n.yind);
}

// Plan problem p: main.jl:215-248 for start pose x0[:, p] and its goal.  Every thread of the CTA calls it; it ends with a sync.
template <class Cta>
OBCA_PHD void plan_one(const Cta& cta, const PlanConst& C, const PlanScratch& W, PlanSmem& sm, const PlanIO& io, int p) {
  const int t = cta.tid(), nt = cta.nth();
  const Config& c = C.cfg;
  if (t == 0) {
    const double *x0 = io.x0 + 3 * (size_t)p, *xF = C.goals + 3 * (size_t)C.per_pose * p;
    sm.goal[0] = xF[0]; sm.goal[1] = xF[1]; sm.goal[2] = pi_2_pi(xF[2]);
    sm.hmap = C.pmap + (size_t)C.hidx[(size_t)C.per_pose * p] * C.hcells;
    PNode& n = W.pool[0];
    const double syaw = pi_2_pi(x0[2]);
    n.np = 1; n.x[0] = x0[0]; n.y[0] = x0[1]; n.yaw[0] = syaw;
    n.xind = (int)jround(x0[0] / c.xyreso); n.yind = (int)jround(x0[1] / c.xyreso); n.yawind = (int)jround(syaw / c.yawreso);
    n.dir = 1; n.steer = 0.0; n.cost = 0.0; n.parent = -1; n.state = NODE_OPEN;
    n.id = calc_index(n.xind, n.yind, n.yawind, c);
    sm.sid = n.id;
    if (n.id >= 0 && n.id < C.table_size) W.table[n.id] = 0;
    sm.n_nodes = 1; sm.heap_n = 0; sm.tick = 0; sm.expansions = 0; sm.status = -1;
    heap_push(W.heap, sm.heap_n, HeapItem{node_priority(C, sm.hmap, n), 0, 0});
  }
  for (;;) {
    // Every thread has read sm.status / sm.cur of the previous step (and thread 0's set-up) before thread 0 writes them again: without
    // this barrier a warp that reads sm.status late would see the NO_PATH of the next pop, leave the search one barrier early and pair
    // every later barrier of the CTA with the wrong one.
    cta.sync();
    // ---- 1. pop ----
    if (t == 0) {
      sm.cur = -1;
      if (sm.heap_n == 0 || sm.expansions > C.max_expansions) {
        sm.status = OBCA_PLAN_NO_PATH;
      } else {
        const HeapItem it = heap_pop(W.heap, sm.heap_n);
        if (W.pool[it.node].state == NODE_OPEN) {
          sm.cur = it.node;
          ++sm.expansions;
          const PNode& n = W.pool[it.node];
          sm.q[0] = n.x[n.np - 1]; sm.q[1] = n.y[n.np - 1]; sm.q[2] = n.yaw[n.np - 1];
        }
      }
    }
    cta.sync();
    if (sm.status >= 0) break;
    if (sm.cur < 0) continue;
    // ---- 2. analytic expansion: candidate words ----
    {
      double x, y, phi, xb, yb;
      rs_frame(sm.q, sm.goal, C.maxc, x, y, phi, xb, yb);
      for (int j = t; j < RS_NCAND; j += nt) sm.cand_ok[j] = rs_candidate(j, x, y, phi, xb, yb, sm.cand[j]);
    }
    cta.sync();
    if (t == 0) {
      sm.set.n = 0;
      for (int j = 0; j < RS_NCAND; ++j)
        if (sm.cand_ok[j]) set_path(sm.set, sm.cand[j]);
      const int bi = rs_shortest(sm.set, C.maxc);
      sm.have_rs = bi >= 0;
      sm.rs_n = 0; sm.rs_hit = 0;
      if (bi >= 0) {
        sm.best = sm.set.p[bi];
        const double step = MOTION_RESOLUTION * C.maxc;
        const int npoint = rs_npoint(sm.set.L[bi], sm.best.n, step);
        if (npoint > RS_MAX_PTS) {
          sm.status = PLAN_NODE_POOL;
        } else {
          sm.rs_n = rs_course_plan(sm.best, step, npoint, W.rsseg, W.rspar);
          rs_origins(sm.best, C.maxc, sm.org);
        }
      }
    }
    cta.sync();
    if (sm.status >= 0) break;
    // ---- 3. course points, then their collision tests ----
    if (sm.have_rs) {
      for (int i = t; i < sm.rs_n; i += nt) rs_point(sm.best, C.maxc, sm.org, W.rsseg[i], W.rspar[i], W.rsx[i], W.rsy[i], W.rsyaw[i]);
      cta.sync();
      if (t == 0) {
        int n = sm.rs_n;
        while (n > 0 && W.rsx[n - 1] == 0.0) --n;
        sm.rs_n = n;
      }
      cta.sync();
      {
        const double cq = cos(-sm.q[2]), sq = sin(-sm.q[2]);
        for (int i = t; i < sm.rs_n; i += nt) {
          double gx, gy, gyaw;
          rs_to_global(sm.q, cq, sq, W.rsx[i], W.rsy[i], W.rsyaw[i], gx, gy, gyaw);
          W.rsx[i] = gx; W.rsy[i] = gy; W.rsyaw[i] = gyaw;
          if (!*(volatile int*)&sm.rs_hit && pose_collides(C.grid, gx, gy, gyaw)) sm.rs_hit = 1;
        }
      }
      cta.sync();
      if (!sm.rs_hit) {
        if (t == 0) sm.status = OBCA_PLAN_OK;      // final node: cur + the course points 1 .. rs_n-2
        break;
      }
    }
    // ---- 4. close cur; the successors' poses, then their collision tests ----
    const PNode& cur = W.pool[sm.cur];
    for (int m = t; m < N_MOTION; m += nt) {
      next_poses(sm.q[0], sm.q[1], sm.q[2], C.ds[m], C.tanu[m], PLAN_NLIST, sm.nx[m], sm.ny[m], sm.nyaw[m]);
      const long xind = jround(sm.nx[m][PLAN_NLIST - 1] / c.xyreso), yind = jround(sm.ny[m][PLAN_NLIST - 1] / c.xyreso);
      sm.nok[m] = (0 < xind - c.minx && xind - c.minx < c.xw) && (0 < yind - c.miny && yind - c.miny < c.yw);
      sm.hit[m] = 0;
    }
    cta.sync();
    for (int i = t; i < N_MOTION * PLAN_NLIST; i += nt) {
      const int m = i / PLAN_NLIST, k = i % PLAN_NLIST;
      if (sm.nok[m] && !*(volatile int*)&sm.hit[m] && pose_collides(C.grid, sm.nx[m][k], sm.ny[m][k], sm.nyaw[m][k])) sm.hit[m] = 1;
    }
    cta.sync();
    // ---- 5. insert in the order m = 0..21 ----
    if (t == 0) {
      W.pool[sm.cur].state = NODE_CLOSED;
      for (int m = 0; m < N_MOTION; ++m) {
        if (!sm.nok[m] || sm.hit[m]) continue;
        const long xind = jround(sm.nx[m][PLAN_NLIST - 1] / c.xyreso), yind = jround(sm.ny[m][PLAN_NLIST - 1] / c.xyreso);
        const long yawind = jround(sm.nyaw[m][PLAN_NLIST - 1] / c.yawreso);
        const long nid = calc_index(xind, yind, yawind, c);
        if (nid == sm.sid) continue;
        if (nid >= 0 && nid < C.table_size && W.table[nid] >= 0) continue;
        if (sm.n_nodes >= C.max_nodes) { sm.status = PLAN_NODE_POOL; break; }
        const int k = sm.n_nodes++;
        PNode& n = W.pool[k];
        for (int i = 0; i < PLAN_NLIST; ++i) { n.x[i] = sm.nx[m][i]; n.y[i] = sm.ny[m][i]; n.yaw[i] = sm.nyaw[m][i]; }
        n.np = PLAN_NLIST; n.xind = (int)xind; n.yind = (int)yind; n.yawind = (int)yawind;
        n.dir = C.ds[m] > 0; n.steer = C.us[m]; n.cost = cur.cost + step_cost(cur.dir != 0, cur.steer, C.us[m], C.ds[m]);
        n.parent = sm.cur; n.id = nid; n.state = NODE_OPEN;
        if (nid >= 0 && nid < C.table_size) W.table[nid] = k;
        ++sm.tick;
        heap_push(W.heap, sm.heap_n, HeapItem{node_priority(C, sm.hmap, n), sm.tick, k});
      }
    }
    cta.sync();
    if (sm.status >= 0) break;
  }
  cta.sync();      // every thread has left the search before thread 0 updates sm.status below
  // ---- the path (get_final_path, hybrid_a_star.jl:506-534) and the warm start (main.jl:222-248) ----
  const int cap = C.cap, sampleN = C.sampleN;
  if (t == 0 && sm.status == OBCA_PLAN_OK) {
    const PNode& s = W.pool[0];
    const int nrs = sm.rs_n >= 2 ? sm.rs_n - 2 : 0;
    int len = 1 + nrs, k = sm.cur;
    for (;;) {
      const PNode& n = W.pool[k];
      len += n.np;
      if (n.xind == s.xind && n.yind == s.yind && n.yawind == s.yawind) break;
      k = n.parent;
      if (k < 0) { sm.status = OBCA_PLAN_NO_PATH; break; }
    }
    const int ns = (len + sampleN - 1) / sampleN;
    sm.len = len;
    if (sm.status == OBCA_PLAN_OK) {
      io.N[p] = ns - 1;
      if (ns > cap) sm.status = OBCA_PLAN_CAPACITY;
    }
    if (sm.status == OBCA_PLAN_OK) {
      int e = len - 1;
      W.px[e] = sm.goal[0]; W.py[e] = sm.goal[1]; W.pyaw[e] = sm.goal[2];
      for (int i = nrs; i >= 1; --i) { --e; W.px[e] = W.rsx[i]; W.py[e] = W.rsy[i]; W.pyaw[e] = W.rsyaw[i]; }
      for (k = sm.cur;; k = W.pool[k].parent) {
        const PNode& n = W.pool[k];
        for (int i = n.np - 1; i >= 0; --i) { --e; W.px[e] = n.x[i]; W.py[e] = n.y[i]; W.pyaw[e] = n.yaw[i]; }
        if (n.xind == s.xind && n.yind == s.yind && n.yawind == s.yawind) break;
      }
    }
  }
  cta.sync();
  if (sm.status == OBCA_PLAN_OK) {
    const int n = sm.len;
    const size_t M = plan_path_max(cap, sampleN) + 40;
    double *rv = W.work + 5 * M, *v = rv + M, *a = v + M, *delta = a + M;
    for (int i = t; i < n; i += nt) rv[i] = i + 1 < n ? ws_speed(W.px, W.py, W.pyaw, i, C.dt) : 0.0;
    cta.sync();
    if (t == 0) velo_smooth(rv, n, WS_AMAX, C.dt, W.work, v, a);
    cta.sync();
    for (int i = t; i + 1 < n; i += nt) delta[i] = ws_steer(W.pyaw, v, i, C.L);
    cta.sync();
    if (t == 0)
      ws_store(W.px, W.py, W.pyaw, v, a, delta, n, sampleN, io.rx + (size_t)p * cap, io.ry + (size_t)p * cap, io.ryaw + (size_t)p * cap,
               io.xWS + (size_t)p * 4 * cap, io.uWS + (size_t)p * 2 * cap);
  }
  if (t == 0) {
    io.status[p] = sm.status;
    if (io.expansions) io.expansions[p] = (int)sm.expansions;
  }
  // leave the cell table empty for the next problem
  for (int i = t; i < sm.n_nodes; i += nt) {
    const long id = W.pool[i].id;
    if (id >= 0 && id < C.table_size) W.table[id] = -1;
  }
  cta.sync();
}

}  // namespace obca_plan
