// obca_astar3d_core.h -- the 3-D grid A* of the quadcopter flow (obca_b200/planner/a_star_3d.py, calc_astar_path), ONE source for both
// of its implementations:
//   libobca_planner.so (obca_planner.cpp, g++ -ffp-contract=off): obca_astar3d_batch, one pair per host thread;
//   libobca.so (obca_b200/csrc/obca_plan3d.cu, nvcc -fmad=false): obca_plan_quadcopter_warmstart_batch, one warp per pair.
// The search (astar3d_one) is written once over a lane policy `L`: the kernel runs it with the 32 lanes of a warp (one neighbour per lane,
// a ballot for the insertion ticks, a warp-wide reduction over the children of a 32-ary heap), SeqLanes runs it on one host thread.
// The host set-up (the obstacle bitmap, the grid geometry, the motion constants, the start / goal cells) is host code both entries run.
//
// The decisions are those of the Python planner, bit for bit:
//   - cells s = jround(sx / reso), g = jround(gx / reso); the 26 moves in itertools.product((-1, 0, 1), repeat=3) order, cost sqrt(dx²+dy²+dz²);
//   - heuristic h = sqrt(double(integer sum of squares)); key f = nc + 1.1 * h (a product, then an add: no FMA); the start's key 1.1 * h(s);
//   - the queue is ordered by (f, tick), tick counting the improvements; every key is unique, so any exact min-queue pops the cells of heapq;
//   - lazy deletion: a popped cell that is already closed is skipped; the goal test happens at pop;
//   - a neighbour is rejected outside 0 < i < w (strict at both ends), in the map or closed; it improves when strictly nc < cost;
//   - the start cell is never bounds- or map-checked.
// Scratch of one search: a cell -> node table (-1 = no node; A3_CLOSED marks a closed cell), a node pool (cost, cell, parent) and the
// queue; the table is reset through the touched nodes at the end of every search, so that it can be reused pair after pair.
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define OBCA_A3 __host__ __device__ __forceinline__
#else
#define OBCA_A3 inline
#endif

#include <cmath>
#include <string>
#include <vector>

namespace obca_astar3d {

constexpr double VEHICLE_RADIUS = 2.5;      // a_star_3d.VEHICLE_RADIUS (a_star_3D.jl:30)
constexpr double H_WEIGHT = 1.1;            // a_star_3d.H_WEIGHT
constexpr int N_MOVES = 26;
constexpr int HEAP_ARITY = 32;              // children of a queue entry: one per lane of a warp
constexpr long long MAX_CELLS = 1LL << 27;  // map cells (16 MB of bitmap); keeps cell indices and insertion ticks in 32 bits
constexpr long long MAX_OFFSET = 1LL << 30; // start / goal cells at most this far from the map's corner
constexpr int A3_CLOSED = 1 << 30;          // table entry flag: the cell is closed
constexpr int A3_MAX_NODES = 1 << 28;
// status codes: OBCA_PLAN_OK, _NO_PATH, _CAPACITY of include/obca_planner.h and OBCA_PLAN_POOL_FULL of include/obca.h
enum : int { A3_OK = 0, A3_NO_PATH = 1, A3_CAPACITY = 2, A3_BAD_ARG = 3, A3_POOL_FULL = 4 };

OBCA_A3 long long a3_jround(double v) { return (long long)floor(fabs(v) + 0.5) * (v >= 0 ? 1 : -1); }      // Julia round(Int64, x)
OBCA_A3 double a3_h(long long dx, long long dy, long long dz) { return sqrt((double)(dx * dx + dy * dy + dz * dz)); }
OBCA_A3 int a3_popc(unsigned v) {
#ifdef __CUDA_ARCH__
  return __popc(v);
#else
  return __builtin_popcount(v);
#endif
}
OBCA_A3 int a3_lowest(unsigned v) {      // index of the lowest set bit of v != 0
#ifdef __CUDA_ARCH__
  return __ffs(v) - 1;
#else
  return __builtin_ctz(v);
#endif
}

struct A3Node {
  double cost;
  int cell;       // linear map index ((ix * w1 + iy) * w2 + iz); -1 for a start outside the map
  int parent;     // node index, -1 for the start
};
struct A3Item {
  double f;
  unsigned tick;
  int node;
};
OBCA_A3 bool a3_less(const A3Item& a, const A3Item& b) { return a.f < b.f || (a.f == b.f && a.tick < b.tick); }

// Constants of one call, shared by every pair (map: device memory in the kernel, host memory otherwise).
struct A3Const {
  const uint32_t* map;             // bit (ix * w1 + iy) * w2 + iz: cell (ix + mn0, iy + mn1, iz + mn2) is blocked
  long long mn[3];
  int w[3];
  int mv[N_MOVES][3];
  double dc[N_MOVES];
  double reso;
  int max_nodes, max_queue, cap;
};
// Inputs / outputs of a batch: s, g are the start / goal cells relative to mn (3 x B); outputs with the stride cap.
struct A3IO {
  const long long *s, *g;
  double *rx, *ry, *rz;
  int *N, *status, *expansions;
  int *nodes, *queue_max;          // optional (may be NULL): nodes used and the longest queue, for sizing the device scratch
};
struct A3Scratch {
  int* table;                      // one entry per map cell, -1 everywhere between searches
  A3Node* pool;                    // max_nodes
  A3Item* queue;                   // max_queue
};

// One host thread plays every lane: per-move values are arrays.
struct SeqLanes {
  template <class T> using PerMove = T[N_MOVES];
  int lane() const { return 0; }
  int width() const { return 1; }
  void sync() const {}
  template <class T> T& at(T (&v)[N_MOVES], int m) const { return v[m]; }
  template <class T> T take(const T (&v)[N_MOVES], int m) const { return v[m]; }
  unsigned mask(const bool (&v)[N_MOVES]) const {
    unsigned r = 0;
    for (int m = 0; m < N_MOVES; ++m) r |= (unsigned)v[m] << m;
    return r;
  }
  void qmin(A3Item&, int&) const {}
};

// Remove the queue's top (which the caller has read): the children of an entry are compared across the lanes, then lane 0 moves the
// smallest one up.  Every lane keeps the same n.
template <class L>
OBCA_A3 void a3_pop(const L& ln, A3Item* h, int& n) {
  const A3Item last = h[n - 1];
  ln.sync();      // every lane has read the top and the last entry before lane 0 overwrites them
  --n;
  int i = 0;
  for (;;) {
    const int c0 = HEAP_ARITY * i + 1;
    if (c0 >= n) break;
    A3Item best{0.0, 0xffffffffu, -1};
    int bj = -1;
    for (int j = ln.lane(); j < HEAP_ARITY; j += ln.width()) {
      const int c = c0 + j;
      if (c < n) {
        const A3Item x = h[c];
        if (bj < 0 || a3_less(x, best)) { best = x; bj = c; }
      }
    }
    ln.qmin(best, bj);
    if (!a3_less(best, last)) break;
    if (ln.lane() == 0) h[i] = best;
    i = bj;
  }
  if (ln.lane() == 0 && n > 0) h[i] = last;
  ln.sync();
}
OBCA_A3 void a3_push(A3Item* h, int n, const A3Item& it) {      // n entries before the push
  int i = n;
  while (i > 0) {
    const int pa = (i - 1) / HEAP_ARITY;
    if (!a3_less(it, h[pa])) break;
    h[i] = h[pa];
    i = pa;
  }
  h[i] = it;
}

// Plan pair p: calc_astar_path from cell s[:, p] to cell g[:, p].  Every lane calls it; it ends with the table reset and a sync.
// Writes status[p] and expansions[p] (closed cells, the goal included); on OBCA_PLAN_OK the path, start first, as cell * reso into
// rx / ry / rz [p * cap ..] and N[p] = points - 1; on CAPACITY only N[p]; on NO_PATH and POOL_FULL nothing else.
template <class L>
OBCA_A3 void astar3d_one(const L& ln, const A3Const& C, const A3Scratch& W, const A3IO& io, int p) {
  const int lane = ln.lane();
  const long long* sp = io.s + 3 * (size_t)p;
  const long long* gp = io.g + 3 * (size_t)p;
  const long long sx = sp[0], sy = sp[1], sz = sp[2], gx = gp[0], gy = gp[1], gz = gp[2];
  const long long W0 = C.w[0], W1 = C.w[1], W2 = C.w[2];
  const bool s_in = 0 <= sx && sx < W0 && 0 <= sy && sy < W1 && 0 <= sz && sz < W2;
  const bool g_in = 0 <= gx && gx < W0 && 0 <= gy && gy < W1 && 0 <= gz && gz < W2;
  const int s_lin = s_in ? (int)((sx * W1 + sy) * W2 + sz) : -1;
  const int g_lin = g_in ? (int)((gx * W1 + gy) * W2 + gz) : -2;      // never a node's cell
  const bool s_is_g = sx == gx && sy == gy && sz == gz;
  if (lane == 0) {
    W.pool[0] = A3Node{0.0, s_lin, -1};
    if (s_in) W.table[s_lin] = 0;
    W.queue[0] = A3Item{H_WEIGHT * a3_h(sx - gx, sy - gy, sz - gz), 0u, 0};
  }
  ln.sync();
  int n_nodes = 1, qn = 1, qmax = 1, goal = -1, status = -1, expansions = 0;
  unsigned tick = 0;
  for (;;) {
    if (qn == 0) { status = A3_NO_PATH; break; }
    const A3Item top = W.queue[0];
    a3_pop(ln, W.queue, qn);
    const int k = top.node;
    const A3Node cur = W.pool[k];
    const bool closed = cur.cell >= 0 && (W.table[cur.cell] & A3_CLOSED);
    ln.sync();      // every lane has read the table entry before lane 0 marks it
    if (closed) continue;
    if (lane == 0 && cur.cell >= 0) W.table[cur.cell] = k | A3_CLOSED;
    ++expansions;
    if (k == 0 ? s_is_g : cur.cell == g_lin) { status = A3_OK; goal = k; break; }
    long long cx = sx, cy = sy, cz = sz;
    if (k != 0) { cx = cur.cell / (W1 * W2); cy = cur.cell / W2 % W1; cz = cur.cell % W2; }
    // ---- the 26 neighbours: bounds, map, closed, cost ----
    typename L::template PerMove<bool> imp, fresh;
    typename L::template PerMove<int> node, lin;
    typename L::template PerMove<double> f, nc;
    for (int m = lane; m < N_MOVES; m += ln.width()) {
      const long long nx = cx + C.mv[m][0], ny = cy + C.mv[m][1], nz = cz + C.mv[m][2];
      bool ok = 0 < nx && nx < W0 && 0 < ny && ny < W1 && 0 < nz && nz < W2;
      int li = 0, t = -1;
      if (ok) {
        li = (int)((nx * W1 + ny) * W2 + nz);
        ok = !((C.map[li >> 5] >> (li & 31)) & 1u);
      }
      if (ok) {
        t = W.table[li];
        ok = t < 0 || !(t & A3_CLOSED);
      }
      const double c = cur.cost + C.dc[m];
      const bool better = ok && (t < 0 || c < W.pool[t].cost);
      ln.at(imp, m) = better;
      ln.at(fresh, m) = better && t < 0;
      ln.at(node, m) = t;
      ln.at(lin, m) = li;
      ln.at(nc, m) = c;
      ln.at(f, m) = better ? c + H_WEIGHT * a3_h(nx - gx, ny - gy, nz - gz) : 0.0;
    }
    const unsigned mi = ln.mask(imp), mf = ln.mask(fresh);
    const int nnew = a3_popc(mf), nimp = a3_popc(mi);
    if (n_nodes + nnew > C.max_nodes || qn + nimp > C.max_queue) { status = A3_POOL_FULL; break; }
    // ---- new nodes in motion order, improved costs, then the pushes with ticks in motion order ----
    for (int m = lane; m < N_MOVES; m += ln.width()) {
      if (!ln.at(imp, m)) continue;
      int& t = ln.at(node, m);
      if (t < 0) {
        t = n_nodes + a3_popc(mf & ((1u << m) - 1u));
        W.table[ln.at(lin, m)] = t;
      }
      W.pool[t] = A3Node{ln.at(nc, m), ln.at(lin, m), k};
    }
    for (unsigned b = mi; b; b &= b - 1) {
      const int m = a3_lowest(b);
      const double fm = ln.take(f, m);
      const int tm = ln.take(node, m);
      ++tick;
      if (lane == 0) a3_push(W.queue, qn, A3Item{fm, tick, tm});
      ++qn;
    }
    qmax = qn > qmax ? qn : qmax;
    n_nodes += nnew;
    ln.sync();
  }
  // ---- the path, start first ----
  if (lane == 0) {
    if (status == A3_OK) {
      int len = 1;
      for (int k = goal; W.pool[k].parent >= 0; k = W.pool[k].parent) ++len;
      io.N[p] = len - 1;
      if (len > C.cap) {
        status = A3_CAPACITY;
      } else {
        const size_t o = (size_t)p * C.cap;
        int k = goal;
        for (int e = len - 1; e >= 0; --e) {
          const int cell = W.pool[k].cell;
          long long x = sx, y = sy, z = sz;
          if (k != 0) { x = cell / (W1 * W2); y = cell / W2 % W1; z = cell % W2; }
          io.rx[o + e] = (double)(x + C.mn[0]) * C.reso;
          io.ry[o + e] = (double)(y + C.mn[1]) * C.reso;
          io.rz[o + e] = (double)(z + C.mn[2]) * C.reso;
          k = W.pool[k].parent;
        }
      }
    }
    io.status[p] = status;
    if (io.expansions) io.expansions[p] = expansions;
    if (io.nodes) io.nodes[p] = n_nodes;
    if (io.queue_max) io.queue_max[p] = qmax;
  }
  // leave the table empty for the next pair
  for (int i = lane; i < n_nodes; i += ln.width()) {
    const int c = W.pool[i].cell;
    if (c >= 0) W.table[c] = -1;
  }
  ln.sync();
}

// =====================================================================================================================
// Host set-up, shared by both libraries
// =====================================================================================================================
struct A3Setup {
  std::vector<uint32_t> map;
  std::vector<long long> s, g;     // 3 x B, relative to mn
  long long cells;
  A3Const C;
};

// calc_obstacle_map (a_star_3d.py): the points divided by reso, the two bound corners appended in raw units, min / max through jround;
// a cell is blocked iff sqrt((dx² + dy²) + dz²) <= VEHICLE_RADIUS / reso for some point (the distance cKDTree reports).  Each point marks
// the cells of the cube around it.  Then the motion constants and the pairs' cells.  Returns OBCA_PLAN_OK, or BAD_ARG with the reason.
inline int astar3d_setup(A3Setup& S, std::string& why, int B, const double* x0, const double* xF, const double* ox, const double* oy,
                         const double* oz, int n_ob, const double* lo, const double* hi, double reso, int cap) {
  if (B < 0) { why = "B < 0"; return A3_BAD_ARG; }
  if (!x0 || !xF || !lo || !hi || (n_ob > 0 && (!ox || !oy || !oz))) { why = "null argument"; return A3_BAD_ARG; }
  if (n_ob < 0) { why = "n_ob < 0"; return A3_BAD_ARG; }
  if (!(reso > 0) || !std::isfinite(reso)) { why = "reso must be a finite number > 0"; return A3_BAD_ARG; }
  if (cap < 1) { why = "cap < 1"; return A3_BAD_ARG; }
  const size_t n = (size_t)n_ob + 2;
  std::vector<double> P[3];
  for (int a = 0; a < 3; ++a) {
    const double* src = a == 0 ? ox : a == 1 ? oy : oz;
    P[a].resize(n);
    for (int i = 0; i < n_ob; ++i) P[a][i] = src[i] / reso;
    P[a][n - 2] = lo[a];
    P[a][n - 1] = hi[a];
    for (size_t i = 0; i < n; ++i)
      if (!std::isfinite(P[a][i]) || fabs(P[a][i]) > 1e15) { why = "obstacle points and bounds must be finite"; return A3_BAD_ARG; }
  }
  A3Const& C = S.C;
  long long w[3];
  S.cells = 1;
  for (int a = 0; a < 3; ++a) {
    double mn = P[a][0], mx = P[a][0];
    for (size_t i = 1; i < n; ++i) { mn = P[a][i] < mn ? P[a][i] : mn; mx = P[a][i] > mx ? P[a][i] : mx; }
    C.mn[a] = a3_jround(mn);
    w[a] = a3_jround(mx) - C.mn[a];
    if (w[a] > MAX_CELLS) { why = "map larger than 2^27 cells"; return A3_BAD_ARG; }
    S.cells *= w[a];
    if (S.cells > MAX_CELLS) { why = "map larger than 2^27 cells"; return A3_BAD_ARG; }
    C.w[a] = (int)w[a];
  }
  S.map.assign((size_t)(S.cells + 31) / 32 + 1, 0u);
  const double r = VEHICLE_RADIUS / reso;
  for (size_t i = 0; i < n; ++i) {
    long long b0[3], b1[3];
    bool any = true;
    for (int a = 0; a < 3; ++a) {      // cells ix + mn within r of the point along this axis, one cell of margin, clipped to the map
      b0[a] = (long long)ceil(P[a][i] - r) - 1 - C.mn[a];
      b1[a] = (long long)floor(P[a][i] + r) + 1 - C.mn[a];
      if (b0[a] < 0) b0[a] = 0;
      if (b1[a] > w[a] - 1) b1[a] = w[a] - 1;
      any = any && b0[a] <= b1[a];
    }
    if (!any) continue;
    for (long long ix = b0[0]; ix <= b1[0]; ++ix) {
      const double dx = (double)(ix + C.mn[0]) - P[0][i];
      for (long long iy = b0[1]; iy <= b1[1]; ++iy) {
        const double dy = (double)(iy + C.mn[1]) - P[1][i];
        const double dxy = dx * dx + dy * dy;
        for (long long iz = b0[2]; iz <= b1[2]; ++iz) {
          const double dz = (double)(iz + C.mn[2]) - P[2][i];
          if (sqrt(dxy + dz * dz) <= r) {
            const long long li = (ix * w[1] + iy) * w[2] + iz;
            S.map[li >> 5] |= 1u << (li & 31);
          }
        }
      }
    }
  }
  C.map = S.map.data();
  int m = 0;
  for (int dx = -1; dx <= 1; ++dx)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dz = -1; dz <= 1; ++dz) {
        if (dx == 0 && dy == 0 && dz == 0) continue;
        C.mv[m][0] = dx; C.mv[m][1] = dy; C.mv[m][2] = dz;
        C.dc[m] = sqrt((double)(dx * dx + dy * dy + dz * dz));
        ++m;
      }
  C.reso = reso;
  C.cap = cap;
  C.max_nodes = C.max_queue = 0;
  S.s.resize(3 * (size_t)B);
  S.g.resize(3 * (size_t)B);
  for (int p = 0; p < B; ++p)
    for (int a = 0; a < 3; ++a) {
      const double vs = x0[3 * (size_t)p + a] / reso, vg = xF[3 * (size_t)p + a] / reso;
      if (!std::isfinite(vs) || !std::isfinite(vg)) { why = "start / goal coordinates must be finite"; return A3_BAD_ARG; }
      const long long cs = a3_jround(vs) - C.mn[a], cg = a3_jround(vg) - C.mn[a];
      if (fabs(vs) > 1e15 || fabs(vg) > 1e15 || cs > MAX_OFFSET || cs < -MAX_OFFSET || cg > MAX_OFFSET || cg < -MAX_OFFSET) {
        why = "start / goal cell more than 2^30 cells from the map"; return A3_BAD_ARG;
      }
      S.s[3 * (size_t)p + a] = cs;
      S.g[3 * (size_t)p + a] = cg;
    }
  return A3_OK;
}

}  // namespace obca_astar3d
