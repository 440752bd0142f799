// obca_plan_core.h -- the algorithm of the Hybrid A* warm-start producer, ONE source for both of its implementations:
//   libobca_planner.so (obca_planner.cpp, g++ -ffp-contract=off): the host planner, one pose per host thread;
//   libobca.so (obca_b200/csrc/obca_plan.cu, nvcc -fmad=false): the GPU planner, a batch of poses in one call.
// Everything marked OBCA_PHD is __host__ __device__ under nvcc and plain inline under g++; the rest (the obstacle cell grid, the
// configuration and the Dijkstra heuristic map) is host-only set-up that both entries run with this very code, so that the heuristic's
// sums of 1 and sqrt(2) -- and with them the search priorities -- carry the same bits.  Same algorithms, in the same order of
// floating-point operations, as the Python restatement obca_b200/planner/*.py (which cites the reference line by line).
#pragma once

#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define OBCA_PHD __host__ __device__ __forceinline__
#else
#define OBCA_PHD inline
#endif

#include <algorithm>
#include <functional>
#include <limits>
#include <queue>
#include <tuple>
#include <unordered_map>
#include <unordered_set>
#include <vector>

namespace obca_plan {

// ---- constants of the reference (hybrid_a_star.jl:42-67, collision_check.jl:31-35, reeds_shepp.jl:35) ----
constexpr double PI = 3.141592653589793;
constexpr double VEHICLE_RADIUS = 1.0, YAW_GRID_RESOLUTION = 5.0 * PI / 180.0, N_STEER = 5.0, XY_GRID_RESOLUTION = 0.3, MOTION_RESOLUTION = 0.1;
constexpr double SB_COST = 10.0, BACK_COST = 0.0, STEER_CHANGE_COST = 10.0, STEER_COST = 0.0, H_COST = 1.0, WB = 2.7, MAX_STEER = 0.6;
constexpr double CAR_B = 1.0, CAR_C = 3.7, CAR_I = 2.0;
constexpr double WBUBBLE_DIST = (CAR_B + CAR_C) / 2.0 - CAR_B, WBUBBLE_R = (CAR_B + CAR_C) / 2.0;
constexpr double RS_STEP_SIZE = 0.1;
constexpr double HP = 0.5 * PI;
constexpr int RS_MAX_SEG = 5;       // segments of the longest Reeds-Shepp word (CCSCC)
constexpr int RS_NCAND = 46;        // candidate words per query: SLS, SRS and 11 families x 4 symmetries (reeds_shepp.jl:99-121)
constexpr int N_MOTION = 22;        // motion primitives per expansion: (2 * N_STEER + 1) steering values x 2 directions

OBCA_PHD double pinf() { return __builtin_huge_val(); }

OBCA_PHD long jround(double v) { return (long)floor(fabs(v) + 0.5) * (v >= 0 ? 1 : -1); }      // Julia round(Int64, x)
OBCA_PHD double pi_2_pi(double a) {
  while (a > PI) a -= 2.0 * PI;
  while (a < -PI) a += 2.0 * PI;
  return a;
}
OBCA_PHD double pymod(double x, double m) {      // Python float %: result has the sign of the divisor
  double v = fmod(x, m);
  if (v != 0.0 && ((v < 0.0) != (m < 0.0))) v += m;
  return v;
}
OBCA_PHD double mod2pi(double x) {
  double v = pymod(x, 2.0 * PI);
  if (v < -PI) v += 2.0 * PI;
  else if (v > PI) v -= 2.0 * PI;
  return v;
}
OBCA_PHD void polar(double x, double y, double& r, double& th) { r = sqrt(x * x + y * y); th = atan2(y, x); }

// =====================================================================================================================
// Reeds-Shepp words (obca_b200/planner/reeds_shepp.py)
// =====================================================================================================================
struct Word { bool ok; double t, u, v; };

OBCA_PHD Word LSL(double x, double y, double phi) {
  double u, t; polar(x - sin(phi), y - 1.0 + cos(phi), u, t);
  if (t >= 0.0) { double v = mod2pi(phi - t); if (v >= 0.0) return {true, t, u, v}; }
  return {false, 0, 0, 0};
}
OBCA_PHD Word LSR(double x, double y, double phi) {
  double u1, t1; polar(x + sin(phi), y - 1.0 - cos(phi), u1, t1);
  u1 = u1 * u1;
  if (u1 >= 4.0) {
    double u = sqrt(u1 - 4.0), theta = atan2(2.0, u), t = mod2pi(t1 + theta), v = mod2pi(t - phi);
    if (t >= 0.0 && v >= 0.0) return {true, t, u, v};
  }
  return {false, 0, 0, 0};
}
OBCA_PHD Word LRL(double x, double y, double phi) {
  double u1, t1; polar(x - sin(phi), y - 1.0 + cos(phi), u1, t1);
  if (u1 <= 4.0) {
    double u = -2.0 * asin(0.25 * u1), t = mod2pi(t1 + 0.5 * u + PI), v = mod2pi(phi - t + u);
    if (t >= 0.0 && u <= 0.0) return {true, t, u, v};
  }
  return {false, 0, 0, 0};
}
OBCA_PHD Word SLS(double x, double y, double phi) {
  phi = mod2pi(phi);
  if (phi > 0.0 && phi < PI * 0.99 && y != 0.0) {
    double xd = -y / tan(phi) + x, t = xd - tan(phi / 2.0), u = phi;
    double r = sqrt((x - xd) * (x - xd) + y * y), v = (y > 0.0 ? r : -r) - tan(phi / 2.0);
    return {true, t, u, v};
  }
  return {false, 0, 0, 0};
}
OBCA_PHD void tau_omega(double u, double v, double xi, double eta, double phi, double& tau, double& omega) {
  double delta = mod2pi(u - v), A = sin(u) - sin(delta), B = cos(u) - cos(delta) - 1.0;
  double t1 = atan2(eta * A - xi * B, xi * A + eta * B);
  double t2 = 2.0 * (cos(delta) - cos(v) - cos(u)) + 3.0;
  tau = t2 < 0 ? mod2pi(t1 + PI) : mod2pi(t1);
  omega = mod2pi(tau - u + v - phi);
}
OBCA_PHD Word LRLRn(double x, double y, double phi) {
  double xi = x + sin(phi), eta = y - 1.0 - cos(phi), rho = 0.25 * (2.0 + sqrt(xi * xi + eta * eta));
  if (rho <= 1.0) {
    double u = acos(rho), t, v; tau_omega(u, -u, xi, eta, phi, t, v);
    if (t >= 0.0 && v <= 0.0) return {true, t, u, v};
  }
  return {false, 0, 0, 0};
}
OBCA_PHD Word LRLRp(double x, double y, double phi) {
  double xi = x + sin(phi), eta = y - 1.0 - cos(phi), rho = (20.0 - xi * xi - eta * eta) / 16.0;
  if (0.0 <= rho && rho <= 1.0) {
    double u = -acos(rho);
    if (u >= -0.5 * PI) { double t, v; tau_omega(u, u, xi, eta, phi, t, v); if (t >= 0.0 && v >= 0.0) return {true, t, u, v}; }
  }
  return {false, 0, 0, 0};
}
OBCA_PHD Word LRSR(double x, double y, double phi) {
  double xi = x + sin(phi), eta = y - 1.0 - cos(phi), rho, theta; polar(-eta, xi, rho, theta);
  if (rho >= 2.0) {
    double t = theta, u = 2.0 - rho, v = mod2pi(t + 0.5 * PI - phi);
    if (t >= 0.0 && u <= 0.0 && v <= 0.0) return {true, t, u, v};
  }
  return {false, 0, 0, 0};
}
OBCA_PHD Word LRSL(double x, double y, double phi) {
  double xi = x - sin(phi), eta = y - 1.0 + cos(phi), rho, theta; polar(xi, eta, rho, theta);
  if (rho >= 2.0) {
    double r = sqrt(rho * rho - 4.0), u = 2.0 - r, t = mod2pi(theta + atan2(r, -2.0)), v = mod2pi(phi - 0.5 * PI - t);
    if (t >= 0.0 && u <= 0.0 && v <= 0.0) return {true, t, u, v};
  }
  return {false, 0, 0, 0};
}
OBCA_PHD Word LRSLR(double x, double y, double phi) {
  double xi = x + sin(phi), eta = y - 1.0 - cos(phi), rho, th; polar(xi, eta, rho, th);
  if (rho >= 2.0) {
    double u = 4.0 - sqrt(rho * rho - 4.0);
    if (u <= 0.0) {
      double t = mod2pi(atan2((4.0 - u) * xi - 2.0 * eta, -2.0 * xi + (u - 4.0) * eta)), v = mod2pi(t - phi);
      if (t >= 0.0 && v >= 0.0) return {true, t, u, v};
    }
  }
  return {false, 0, 0, 0};
}

// One candidate word: segment lengths (unscaled) and types 'L' / 'S' / 'R'.
struct RsCand {
  int n;
  double len[RS_MAX_SEG];
  char ty[RS_MAX_SEG];
};
OBCA_PHD char swap_lr(char c) { return c == 'L' ? 'R' : (c == 'R' ? 'L' : 'S'); }

// Candidate j of reeds_shepp.jl:99-121 (generate_path), j = 0..RS_NCAND-1, in the reference's order: SLS, SRS, then the families below
// with their four symmetries (timeflip / reflect).  (x, y, phi): goal in the start frame scaled by maxc; (xb, yb): its backwards form.
// Returns false when the word does not exist.
OBCA_PHD bool rs_candidate(int j, double x, double y, double phi, double xb, double yb, RsCand& c) {
  if (j < 2) {
    const Word w = j == 0 ? SLS(x, y, phi) : SLS(x, -y, -phi);
    if (!w.ok) return false;
    c.n = 3; c.len[0] = w.t; c.len[1] = w.u; c.len[2] = w.v;
    c.ty[0] = 'S'; c.ty[1] = j == 0 ? 'L' : 'R'; c.ty[2] = 'S';
    return true;
  }
  const int f = (j - 2) >> 2, k = (j - 2) & 3;
  // families: 0 LSL, 1 LSR, 2 LRL, 3 LRL backwards, 4 LRLR (n), 5 LRLR (p), 6 LRSL, 7 LRSR, 8 LRSL backwards, 9 LRSR backwards, 10 LRSLR
  const bool back = f == 3 || f == 8 || f == 9;
  const double bx = back ? xb : x, by = back ? yb : y;
  const double fx = (k & 1) ? -bx : bx, fy = (k & 2) ? -by : by, fp = (k == 1 || k == 2) ? -phi : phi;
  Word w;
  const char* word;
  switch (f) {
    case 0: w = LSL(fx, fy, fp); word = "LSL"; break;
    case 1: w = LSR(fx, fy, fp); word = "LSR"; break;
    case 2: case 3: w = LRL(fx, fy, fp); word = "LRL"; break;
    case 4: w = LRLRn(fx, fy, fp); word = "LRLR"; break;
    case 5: w = LRLRp(fx, fy, fp); word = "LRLR"; break;
    case 6: case 8: w = LRSL(fx, fy, fp); word = "LRSL"; break;
    case 7: case 9: w = LRSR(fx, fy, fp); word = "LRSR"; break;
    default: w = LRSLR(fx, fy, fp); word = "LRSLR"; break;
  }
  if (!w.ok) return false;
  double l[RS_MAX_SEG];
  int n;
  if (f <= 3) { n = 3; l[0] = w.t; l[1] = w.u; l[2] = w.v; }                                   // tuv
  else if (f == 4) { n = 4; l[0] = w.t; l[1] = w.u; l[2] = -w.u; l[3] = w.v; }                 // ccccn
  else if (f == 5) { n = 4; l[0] = w.t; l[1] = w.u; l[2] = w.u; l[3] = w.v; }                  // ccccp
  else if (f <= 9) { n = 4; l[0] = w.t; l[1] = -HP; l[2] = w.u; l[3] = w.v; }                  // ccsc
  else { n = 5; l[0] = w.t; l[1] = -HP; l[2] = w.u; l[3] = -HP; l[4] = w.v; }                  // ccscc
  c.n = n;
  for (int i = 0; i < n; ++i) {
    const int s = back ? n - 1 - i : i;
    c.len[i] = (k & 1) ? -l[s] : l[s];
    c.ty[i] = (k & 2) ? swap_lr(word[s]) : word[s];
  }
  return true;
}

// Python's built-in sum() of floats (CPython >= 3.12: Neumaier's compensated summation) -- the Python restatement uses it for the two
// sums of set_path, and the order of candidate words depends on their last bits
struct PySum {
  double f = 0.0, c = 0.0;
  OBCA_PHD void add(double x) {
    const double t = f + x;
    if (fabs(f) >= fabs(x)) c += (f - t) + x;
    else c += (x - t) + f;
    f = t;
  }
  OBCA_PHD double value() const { return (c != 0.0 && isfinite(c)) ? f + c : f; }
};

// The distinct candidate paths of one query, in insertion order, with their total (unscaled) lengths.
struct RsSet {
  int n;
  RsCand p[RS_NCAND];
  double L[RS_NCAND];
};
OBCA_PHD void set_path(RsSet& s, const RsCand& c) {      // reeds_shepp.jl:207-230, quirk kept
  for (int q = 0; q < s.n; ++q) {
    const RsCand& tp = s.p[q];
    bool same = tp.n == c.n;
    for (int i = 0; same && i < c.n; ++i) same = tp.ty[i] == c.ty[i];
    if (!same) continue;
    PySum d;
    for (int i = 0; i < c.n; ++i) d.add(tp.len[i] - c.len[i]);
    if (d.value() <= 0.01) return;
  }
  PySum Ls;
  for (int i = 0; i < c.n; ++i) Ls.add(fabs(c.len[i]));
  const double L = Ls.value();
  if (L < 0.01) return;
  s.p[s.n] = c; s.L[s.n] = L; ++s.n;
}
// The query frame of generate_path (reeds_shepp.jl:99-104): the goal q1 relative to q0, scaled by maxc.
OBCA_PHD void rs_frame(const double q0[3], const double q1[3], double maxc, double& x, double& y, double& phi, double& xb, double& yb) {
  const double dx = q1[0] - q0[0], dy = q1[1] - q0[1], dth = q1[2] - q0[2];
  const double c = cos(q0[2]), s = sin(q0[2]);
  x = (c * dx + s * dy) * maxc; y = (-s * dx + c * dy) * maxc; phi = dth;
  xb = x * cos(phi) + y * sin(phi); yb = x * sin(phi) - y * cos(phi);
}
// Index of the shortest path of the set (the last of equally short candidates wins, reeds_shepp.jl:67-72), -1 if the set is empty.
OBCA_PHD int rs_shortest(const RsSet& s, double maxc) {
  double minL = pinf();
  int bi = -1;
  for (int i = 0; i < s.n; ++i)
    if (s.L[i] / maxc <= minL) { minL = s.L[i] / maxc; bi = i; }
  return bi;
}

// ---- generate_local_course (reeds_shepp.jl:233-282) ----
// Number of course points allocated for a path of total length L (normalised) sampled every step (normalised).
OBCA_PHD int rs_npoint(double L, int nseg, double step) { return (int)(L / step) + 2 * nseg + 8; }
// The serial part of generate_local_course: which segment and which arc parameter the LAST write to each course index uses.  seg[i] = -1
// for an index nothing is written to (its point stays 0).  Returns the number of indices written to (<= npoint).
OBCA_PHD int rs_course_plan(const RsCand& c, double step, int npoint, int* seg, double* par) {
  for (int i = 0; i < npoint; ++i) { seg[i] = -1; par[i] = 0.0; }
  int ind = 1, hi = 0;
  double d = c.len[0] > 0.0 ? step : -step, pd = d, ll = 0.0;
  for (int i = 0; i < c.n; ++i) {
    const double l = c.len[i];
    d = l > 0.0 ? step : -step;
    ind -= 1;
    if (i >= 1 && c.len[i - 1] * c.len[i] > 0) pd = -d - ll;
    else pd = d - ll;
    while (fabs(pd) <= fabs(l)) {
      ind += 1;
      seg[ind] = i; par[ind] = pd;
      pd += d;
    }
    ll = l - pd - d;
    ind += 1;
    seg[ind] = i; par[ind] = l;
    if (ind + 1 > hi) hi = ind + 1;
  }
  return hi;
}
OBCA_PHD void interpolate(double l, char m, double maxc, double ox, double oy, double oyaw, double& px, double& py, double& pyaw) {
  if (m == 'S') {
    px = ox + l / maxc * cos(oyaw);
    py = oy + l / maxc * sin(oyaw);
    pyaw = oyaw;
  } else {
    double ldx = sin(l) / maxc, ldy = (1.0 - cos(l)) / (m == 'L' ? maxc : -maxc);
    double gdx = cos(-oyaw) * ldx + sin(-oyaw) * ldy, gdy = -sin(-oyaw) * ldx + cos(-oyaw) * ldy;
    px = ox + gdx;
    py = oy + gdy;
    pyaw = m == 'L' ? oyaw + l : oyaw - l;
  }
}
// Segment origins of the local course: the first segment starts at (0, 0, 0), segment i+1 at the end point of segment i.
OBCA_PHD void rs_origins(const RsCand& c, double maxc, double org[RS_MAX_SEG][3]) {
  org[0][0] = org[0][1] = org[0][2] = 0.0;
  for (int i = 0; i + 1 < c.n; ++i)
    interpolate(c.len[i], c.ty[i], maxc, org[i][0], org[i][1], org[i][2], org[i + 1][0], org[i + 1][1], org[i + 1][2]);
}
// Course point of index i (local frame, seg < 0: the unwritten 0), then its global pose (calc_paths, reeds_shepp.jl:36-49);
// cq / sq = cos / sin(-q0[2]).
OBCA_PHD void rs_point(const RsCand& c, double maxc, const double org[RS_MAX_SEG][3], int seg, double par, double& x, double& y, double& yaw) {
  if (seg < 0) { x = y = yaw = 0.0; return; }
  interpolate(par, c.ty[seg], maxc, org[seg][0], org[seg][1], org[seg][2], x, y, yaw);
}
OBCA_PHD void rs_to_global(const double q0[3], double cq, double sq, double x, double y, double yaw, double& gx, double& gy, double& gyaw) {
  gx = cq * x + sq * y + q0[0];
  gy = -sq * x + cq * y + q0[1];
  gyaw = pi_2_pi(yaw + q0[2]);
}
// calc_rs_path_cost (hybrid_a_star.jl:448-483) on the lengths scaled by 1/maxc.
OBCA_PHD double calc_rs_path_cost(const double* len, const char* ty, int n) {
  double cost = 0.0;
  for (int i = 0; i < n; ++i) cost += len[i] >= 0 ? len[i] : fabs(len[i]) * BACK_COST;
  for (int i = 0; i + 1 < n; ++i)
    if (len[i] * len[i + 1] < 0.0) cost += SB_COST;
  for (int i = 0; i < n; ++i)
    if (ty[i] != 'S') cost += STEER_COST * fabs(MAX_STEER);
  for (int i = 0; i + 1 < n; ++i) {
    const double u0 = ty[i] == 'R' ? -MAX_STEER : (ty[i] == 'L' ? MAX_STEER : 0.0);
    const double u1 = ty[i + 1] == 'R' ? -MAX_STEER : (ty[i + 1] == 'L' ? MAX_STEER : 0.0);
    cost += STEER_CHANGE_COST * fabs(u1 - u0);
  }
  return cost;
}

// =====================================================================================================================
// collision test (obca_b200/planner/collision.py)
// =====================================================================================================================
// collision_check.jl:58-98 for one point, with c = cos(-iyaw), s = sin(-iyaw)
OBCA_PHD bool point_in_car_cs(double c, double s, double ix, double iy, double px, double py) {
  const double VRX[5] = {CAR_C, CAR_C, -CAR_B, -CAR_B, CAR_C};
  const double VRY[5] = {-CAR_I / 2.0, CAR_I / 2.0, CAR_I / 2.0, -CAR_I / 2.0, -CAR_I / 2.0};
  const double tx = px - ix, ty = py - iy;
  const double lx = c * tx - s * ty, ly = s * tx + c * ty;
  double sumangle = 0.0;
  for (int e = 0; e < 4; ++e) {
    const double x1 = VRX[e] - lx, y1 = VRY[e] - ly, x2 = VRX[e + 1] - lx, y2 = VRY[e + 1] - ly;
    const double d1 = sqrt(x1 * x1 + y1 * y1), d2 = sqrt(x2 * x2 + y2 * y2);
    const double th1 = atan2(y1, x1);
    const double tty = -sin(th1) * x2 + cos(th1) * y2;
    double tmp = (x1 * x2 + y1 * y2) / (d1 * d2);
    if (!(tmp <= 1.0) && tmp == tmp) tmp = 1.0;      // min(tmp, 1) that keeps NaN
    const double ang = acos(tmp);
    sumangle += tty >= 0.0 ? ang : -ang;
  }
  return sumangle >= PI;
}
OBCA_PHD bool point_in_car(double ix, double iy, double iyaw, double px, double py) {
  return point_in_car_cs(cos(-iyaw), sin(-iyaw), ix, iy, px, py);
}
// Uniform grid over the obstacle points (cell = bubble radius), stored as CSR: the points of cell (i, j) are ids[start[j*nx+i] ..
// start[j*nx+i+1]) in increasing order.  A plain view, so that the same test runs on host vectors and on device copies.
struct ObGridView {
  double x0, y0, cell;
  int nx, ny;
  const int* start;
  const int* ids;
  const double* ox;
  const double* oy;
};
// Does any obstacle point inside the bubble of pose (x, y, yaw) lie in the car?  (The host returns at the first hit; "any hit" does
// not depend on the order of the tests.)
OBCA_PHD bool pose_collides(const ObGridView& g, double x, double y, double yaw) {
  if (g.nx == 0) return false;
  const double cx = x + WBUBBLE_DIST * cos(yaw), cy = y + WBUBBLE_DIST * sin(yaw);
  const int ci = (int)floor((cx - g.x0) / g.cell), cj = (int)floor((cy - g.y0) / g.cell);
  double c = 0.0, s = 0.0;
  bool have_cs = false;
  for (int j = cj - 1; j <= cj + 1; ++j) {
    if (j < 0 || j >= g.ny) continue;
    for (int i = ci - 1; i <= ci + 1; ++i) {
      if (i < 0 || i >= g.nx) continue;
      for (int q = g.start[j * g.nx + i]; q < g.start[j * g.nx + i + 1]; ++q) {
        const int id = g.ids[q];
        const double dx = g.ox[id] - cx, dy = g.oy[id] - cy;
        if (sqrt(dx * dx + dy * dy) <= WBUBBLE_R) {
          if (!have_cs) { c = cos(-yaw); s = sin(-yaw); have_cs = true; }
          if (point_in_car_cs(c, s, x, y, g.ox[id], g.oy[id])) return true;
        }
      }
    }
  }
  return false;
}

// =====================================================================================================================
// Hybrid A* pieces (obca_b200/planner/hybrid_a_star.py)
// =====================================================================================================================
struct Config { long minx, miny, minyaw, maxx, maxy, maxyaw, xw, yw, yaww; double xyreso, yawreso; };
OBCA_PHD long calc_index(long xind, long yind, long yawind, const Config& c) {
  return (yawind - c.minyaw) * c.xw * c.yw + (yind - c.miny) * c.xw + (xind - c.minx);
}
// The poses of calc_next_node (hybrid_a_star.jl:369-400) from the parent's last pose; tanu = tan(u), computed by the host's libm.
OBCA_PHD void next_poses(double x, double y, double yaw, double d, double tanu, int nlist, double* nx, double* ny, double* nyaw) {
  nx[0] = x + d * MOTION_RESOLUTION * cos(yaw);
  ny[0] = y + d * MOTION_RESOLUTION * sin(yaw);
  nyaw[0] = pi_2_pi(yaw + d * MOTION_RESOLUTION / WB * tanu);
  for (int i = 0; i < nlist - 1; ++i) {
    nx[i + 1] = nx[i] + d * MOTION_RESOLUTION * cos(nyaw[i]);
    ny[i + 1] = ny[i] + d * MOTION_RESOLUTION * sin(nyaw[i]);
    nyaw[i + 1] = pi_2_pi(nyaw[i] + d * MOTION_RESOLUTION / WB * tanu);
  }
}
// The cost calc_next_node adds for primitive (u, d) after a node driven in direction cur_dir with steering cur_steer.
OBCA_PHD double step_cost(bool cur_dir, double cur_steer, double u, double d) {
  const double arc_l = XY_GRID_RESOLUTION;
  const bool direction = d > 0;
  double added = direction ? fabs(arc_l) : fabs(arc_l) * BACK_COST;
  if (direction != cur_dir) added += SB_COST;
  added += STEER_COST * fabs(u);
  added += STEER_CHANGE_COST * fabs(cur_steer - u);
  return added;
}
// Heuristic of a cell: the Dijkstra map (h = INF outside it).
OBCA_PHD double heuristic(const double* pmap, long minx, long miny, int xw, int yw, long xind, long yind) {
  const long i = xind - minx, j = yind - miny;
  return (1 <= i && i <= xw && 1 <= j && j <= yw) ? pmap[(size_t)(i - 1) * yw + (j - 1)] : pinf();
}

// =====================================================================================================================
// veloSmooth (obca_b200/planner/velo_smooth.py) and the warm-start extraction (warmstart.py, main.jl:222-248)
// =====================================================================================================================
OBCA_PHD double sgn(double v) { return v > 0 ? 1.0 : (v < 0 ? -1.0 : 0.0); }
OBCA_PHD double linspace_at(double a, double b, int num, int i) {      // linspace(a, b, num)[i]
  if (num == 1) return a;
  if (i == num - 1) return b;
  const double step = (b - a) / (num - 1);
  return step != 0.0 ? (double)i * step + a : a;
}
// veloSmooth.jl:29-109.  v[n] -> v_mm[n], a[n-1].  work: 5 * (n + 40) doubles.
OBCA_PHD void velo_smooth(const double* v, int n, double amax, double Ts, double* work, double* v_mm, double* a) {
  const int PAD = 19, M = n + 40;
  double* v_ex = work;
  double* v_bar = work + M;      // 4 rows of M
  for (int i = 0; i < 5 * M; ++i) work[i] = 0.0;
  for (int i = 0; i < n; ++i) { v_ex[PAD + i] = v[i]; for (int r = 0; r < 4; ++r) v_bar[r * M + PAD + i] = v[i]; }
  const double v0 = fabs(v[0]), cut1 = 0.25 * v0, cut2 = 1.25 * v0;
  const int acc = (int)jround(v0 / amax / Ts);
  // v_bar[row, lo:hi] = linspace(A, B, hi - lo + 1), 1-based inclusive
  auto put = [&](int row, int lo, int hi, double A, double B) {
    if (hi < lo) return;
    for (int k = lo; k <= hi; ++k)
      if (k >= 1 && k <= M) v_bar[row * M + k - 1] = linspace_at(A, B, hi - lo + 1, k - lo);
  };
  auto ex = [&](int i) { return v_ex[i - 1]; };
  // the four index lists of the reference (1-based indices into diff(v_ex)) in increasing order; each fills its own row, so the rows
  // are filled one after the other, each list in its order.  The first entry of idx1 / idx3 is moved from 19 to 20 (reference quirk).
  for (int cat = 0; cat < 4; ++cat) {
    bool first = true;
    for (int i0 = 0; i0 + 1 < M; ++i0) {
      const double dv = v_ex[i0 + 1] - v_ex[i0];
      const bool in = cat == 0 ? (dv > cut1 && dv < cut2) : cat == 1 ? (dv < -cut1 && dv > -cut2) : cat == 2 ? (dv > cut2) : (dv < -cut2);
      if (!in) continue;
      int i = i0 + 1;
      if (first && cat < 2 && i == 19) i += 1;
      first = false;
      if (cat == 0) {
        if (ex(i) > cut1 || ex(i + 1) > cut1) put(0, i, i + acc, 0.0, v0);
        else if (ex(i) < -cut1 || ex(i + 1) < -cut1) put(0, i - acc + 1, i + 1, -v0, 0.0);
      } else if (cat == 1) {
        if (ex(i) > cut1 || ex(i + 1) > cut1) put(1, i - acc + 1, i + 1, v0, 0.0);
        else if (ex(i) < -cut1 || ex(i + 1) < -cut1) put(1, i, i + acc, 0.0, -v0);
      } else if (cat == 2) {
        put(2, i - acc, i + acc, -v0, v0);
      } else {
        put(3, i - acc, i + acc, v0, -v0);
      }
    }
  }
  for (int j = 0; j < n; ++j) {
    const double ve = v_ex[PAD + j];
    double mn = pinf(), mx = -pinf();
    for (int r = 0; r < 4; ++r) {
      const double vb = v_bar[r * M + PAD + j];
      const double w = vb == 0.0 ? vb : (sgn(ve) != sgn(vb) ? ve : vb);
      mn = w < mn ? w : mn;
      mx = w > mx ? w : mx;
    }
    v_mm[j] = ve > 0 ? mn : mx;
  }
  for (int j = 0; j + 1 < n; ++j) a[j] = (v_mm[j + 1] - v_mm[j]) / Ts;
}
// The speed of path point i (main.jl:222-226) and the steering of step i (main.jl:229-233).
OBCA_PHD double ws_speed(const double* px, const double* py, const double* pyaw, int i, double dt) {
  return (px[i + 1] - px[i]) / dt * cos(pyaw[i]) + (py[i + 1] - py[i]) / dt * sin(pyaw[i]);
}
OBCA_PHD double ws_steer(const double* pyaw, const double* v, int i, double L) {
  return atan((pyaw[i + 1] - pyaw[i]) * L / MOTION_RESOLUTION * sgn(v[i]));
}
// Down-sampling by sampleN (main.jl:237-248) into the caller's arrays: rx, ry, ryaw [ns], xWS ns x 4, uWS N x 2 (column-major, N = ns-1).
OBCA_PHD void ws_store(const double* px, const double* py, const double* pyaw, const double* v, const double* a, const double* delta, int n,
                       int sampleN, double* rx, double* ry, double* ryaw, double* xWS, double* uWS) {
  const int ns = (n + sampleN - 1) / sampleN, N = ns - 1;
  for (int k = 0; k < ns; ++k) {
    const int i = k * sampleN;
    rx[k] = px[i]; ry[k] = py[i]; ryaw[k] = pyaw[i];
    xWS[k] = px[i]; xWS[ns + k] = py[i]; xWS[2 * ns + k] = pyaw[i]; xWS[3 * ns + k] = v[i];
  }
  for (int k = 0; k < N; ++k) {
    const int i = k * sampleN;
    uWS[k] = delta[i]; uWS[N + k] = a[i];
  }
}
constexpr double WS_AMAX = 0.3;      // main.jl:226

// =====================================================================================================================
// host-only set-up, shared by the host planner and the GPU planner's entry
// =====================================================================================================================
struct Obstacles {
  std::vector<double> ox, oy;
  double x0 = 0, y0 = 0, cell = WBUBBLE_R;
  int nx = 0, ny = 0;
  std::vector<int> start, ids;
  int cell_of(double v, double v0, int n) const { int c = (int)std::floor((v - v0) / cell); return c < 0 ? 0 : (c >= n ? n - 1 : c); }
  void build() {
    if (ox.empty()) return;
    x0 = *std::min_element(ox.begin(), ox.end()); y0 = *std::min_element(oy.begin(), oy.end());
    const double x1 = *std::max_element(ox.begin(), ox.end()), y1 = *std::max_element(oy.begin(), oy.end());
    nx = (int)std::floor((x1 - x0) / cell) + 1; ny = (int)std::floor((y1 - y0) / cell) + 1;
    std::vector<std::vector<int> > cells((size_t)nx * ny);
    for (size_t i = 0; i < ox.size(); ++i) cells[(size_t)cell_of(oy[i], y0, ny) * nx + cell_of(ox[i], x0, nx)].push_back((int)i);
    start.assign((size_t)nx * ny + 1, 0); ids.clear();
    for (size_t c = 0; c < cells.size(); ++c) {
      std::sort(cells[c].begin(), cells[c].end());
      ids.insert(ids.end(), cells[c].begin(), cells[c].end());
      start[c + 1] = (int)ids.size();
    }
  }
  ObGridView view() const { return ObGridView{x0, y0, cell, nx, ny, start.data(), ids.data(), ox.data(), oy.data()}; }
};

inline Config calc_config(const std::vector<double>& ox, const std::vector<double>& oy, double xyreso, double yawreso) {
  Config c;
  c.minx = jround(*std::min_element(ox.begin(), ox.end()) / xyreso); c.miny = jround(*std::min_element(oy.begin(), oy.end()) / xyreso);
  c.maxx = jround(*std::max_element(ox.begin(), ox.end()) / xyreso); c.maxy = jround(*std::max_element(oy.begin(), oy.end()) / xyreso);
  c.minyaw = jround(-PI / yawreso) - 1; c.maxyaw = jround(PI / yawreso);
  c.xw = c.maxx - c.minx; c.yw = c.maxy - c.miny; c.yaww = c.maxyaw - c.minyaw; c.xyreso = xyreso; c.yawreso = yawreso;
  return c;
}

// grid heuristic (obca_b200/planner/grid_policy.py): exact 8-connected shortest distances from the goal.  Two parts: the obstacle map,
// which does not depend on the goal (HeurGrid, built once per cloud), and the distances from one goal cell (dist_from_goal);
// calc_dist_policy is their composition.  The distances depend on the goal only through its cell heur_goal_cell(gx, gy, reso).
struct HeurGrid {
  std::vector<char> obmap;       // [xw][yw], 1 = blocked; entry (i-1, j-1) <-> cell (i + minx, j + miny)
  long minx = 0, miny = 0;
  int xw = 0, yw = 0;
};
struct DistPolicy {
  std::vector<double> pmap;      // [xw][yw], INF where unreachable; entry (i-1, j-1) <-> cell (i + minx, j + miny)
  long minx = 0, miny = 0;
  int xw = 0, yw = 0;
};
OBCA_PHD void heur_goal_cell(double gx, double gy, double reso, long& g0, long& g1) { g0 = jround(gx / reso); g1 = jround(gy / reso); }
inline HeurGrid calc_heur_grid(const std::vector<double>& ox, const std::vector<double>& oy, double reso, double vr) {
  using std::vector;
  HeurGrid G;
  vector<double> oxs(ox.size()), oys(oy.size());
  for (size_t i = 0; i < ox.size(); ++i) { oxs[i] = ox[i] / reso; oys[i] = oy[i] / reso; }
  const long minx = jround(*std::min_element(oxs.begin(), oxs.end())), miny = jround(*std::min_element(oys.begin(), oys.end()));
  const long maxx = jround(*std::max_element(oxs.begin(), oxs.end())), maxy = jround(*std::max_element(oys.begin(), oys.end()));
  const int xw = (int)(maxx - minx), yw = (int)(maxy - miny);
  G.minx = minx; G.miny = miny; G.xw = xw; G.yw = yw;
  G.obmap.assign((size_t)xw * yw, 0);
  const double lim = vr / reso;
  for (int ix = 1; ix <= xw; ++ix)
    for (int iy = 1; iy <= yw; ++iy) {
      const double cx = (double)(ix + minx), cy = (double)(iy + miny);
      double best = pinf();
      for (size_t k = 0; k < oxs.size(); ++k) {
        const double dx = oxs[k] - cx, dy = oys[k] - cy, d2 = dx * dx + dy * dy;
        if (d2 < best) best = d2;
      }
      G.obmap[(size_t)(ix - 1) * yw + (iy - 1)] = std::sqrt(best) <= lim;
    }
  return G;
}
// Dijkstra from the goal cell (g0, g1).  The goal is a source even when it is blocked or outside the map; a target must lie in the strict
// interior 0 < ix < xw, 0 < iy < yw and be free; pmap is written only inside 1..xw x 1..yw.
inline DistPolicy dist_from_goal(const HeurGrid& G, long g0, long g1) {
  using std::vector;
  DistPolicy P;
  const long minx = G.minx, miny = G.miny;
  const int xw = G.xw, yw = G.yw;
  const vector<char>& obmap = G.obmap;
  P.minx = minx; P.miny = miny; P.xw = xw; P.yw = yw;
  P.pmap.assign((size_t)xw * yw, pinf());
  auto ok = [&](long x, long y) {
    const long ix = x - minx, iy = y - miny;
    return 0 < ix && ix < xw && 0 < iy && iy < yw && !obmap[(size_t)(ix - 1) * yw + (iy - 1)];
  };
  typedef std::tuple<double, long, long> Item;
  std::priority_queue<Item, vector<Item>, std::greater<Item> > heap;
  auto key = [](long x, long y) { return ((uint64_t)(uint32_t)(int32_t)x << 32) | (uint32_t)(int32_t)y; };
  std::unordered_map<uint64_t, double> best;
  std::unordered_set<uint64_t> done;
  heap.push(Item(0.0, g0, g1));
  best[key(g0, g1)] = 0.0;
  const int MX[8] = {1, 0, -1, 0, -1, -1, 1, 1}, MY[8] = {0, 1, 0, -1, -1, 1, -1, 1};
  const double s2 = std::sqrt(2.0);
  const double MC[8] = {1.0, 1.0, 1.0, 1.0, s2, s2, s2, s2};
  while (!heap.empty()) {
    const Item it = heap.top(); heap.pop();
    const double c = std::get<0>(it);
    const long x = std::get<1>(it), y = std::get<2>(it);
    if (done.count(key(x, y))) continue;
    done.insert(key(x, y));
    const long ix = x - minx, iy = y - miny;
    if (1 <= ix && ix <= xw && 1 <= iy && iy <= yw) P.pmap[(size_t)(ix - 1) * yw + (iy - 1)] = c;
    for (int m = 0; m < 8; ++m) {
      const long nx = x + MX[m], ny = y + MY[m];
      if (done.count(key(nx, ny)) || !ok(nx, ny)) continue;
      const double nc = c + MC[m];
      auto f = best.find(key(nx, ny));
      if (f == best.end() || nc < f->second) { best[key(nx, ny)] = nc; heap.push(Item(nc, nx, ny)); }
    }
  }
  return P;
}
inline DistPolicy calc_dist_policy(double gx, double gy, const std::vector<double>& ox, const std::vector<double>& oy, double reso, double vr) {
  long g0, g1;
  heur_goal_cell(gx, gy, reso, g0, g1);
  return dist_from_goal(calc_heur_grid(ox, oy, reso, vr), g0, g1);
}

// The motion primitives (u, d) of hybrid_a_star.jl:402-414 in the order successors are generated, and tan(u) of each.
inline void motion_inputs(std::vector<double>& us, std::vector<double>& ds, std::vector<double>& tanu) {
  const double step = MAX_STEER / N_STEER;
  std::vector<double> up;
  for (int i = 0; i < (int)jround(N_STEER); ++i) up.push_back(step * (i + 1));
  std::vector<double> u{0.0};
  for (double v : up) u.push_back(v);
  for (double v : up) u.push_back(-v);
  us = u; us.insert(us.end(), u.begin(), u.end());
  ds.assign(u.size(), 1.0); ds.insert(ds.end(), u.size(), -1.0);
  tanu.resize(us.size());
  for (size_t m = 0; m < us.size(); ++m) tanu[m] = std::tan(us[m]);
}
inline int motion_nlist() { return (int)jround(XY_GRID_RESOLUTION / MOTION_RESOLUTION) + 1; }
inline double max_curvature() { return std::tan(MAX_STEER) / WB; }

}  // namespace obca_plan
