// cell_solver.cuh — one (obstacle, stage) cell of the LamMuZ problem and its multiplier update.
//
// Replaces, per cell, the reference's per-obstacle cvxpy/ECOS solve and the numpy update loops:
//   problem      rda_solver.py:389-421 (LamMuZ_cost_cons), :874-909 (Hm_LamMu, Im_LamMu),
//                cones :1034-1050; separable over the horizon (max of norms <= 1, :408-416)
//   updates      update_xi :668-690, update_zeta :639-666, lam'A / lam'b :529-542
//
// Method (DESIGN.md §3).  With v = A'lam, g = G'mu and support functions sigma_O, sigma_Rob the
// cell is the 4-variable convex problem
//     min_{|v|<=1, g}  1/2 neg(stuff)^2 + ro2/2 |g + R'v + xi|^2,
//     stuff = v.p - sigma_O(v) - sigma_Rob(g) - d + zeta,
// solved in coordinates relative to the robot reference point p:
//   fast path : xi == 0 and obstacle/robot disjoint  -> closest pair of points (exact);
//               robot-vertex contact candidates accepted by their KKT conditions (exact);
//   slow path : small dense primal-dual interior point method in float64.
// Tie-break where the reference argmin is not unique: max margin, LP-vertex multipliers,
// z = theta * max(stuff, 0).
#pragma once
#include "rda_hd.h"

namespace rda {

// tangential residual of g accepted at the closed-form stationary point of a robot-edge x obstacle-edge contact (rounding only)
constexpr double CELL_EE_TANG = 1e-4;

enum { CELL_FAST_INACTIVE = 0, CELL_FAST_VERTEX = 1, CELL_SLOW_A = 2, CELL_SLOW_B = 3,
       CELL_OVERLAP_FREE = 4, CELL_FAILED = 5, CELL_NEEDS_SLOW = 6 };

template <typename Real>
struct CellOut {
  Real lam[RDA_MAX_EDGE];
  Real mu[RDA_MAX_ROBOT_EDGE];
  Real z, zeta_new, xi0_new, xi1_new;   // multiplier state after the update
  Real ax, ay, c0, gx, gy;              // su-QP hinge inputs (lam'A, offset, mu'G + xi)
  Real hm0, hm1;                        // Hm of this cell (primal residual, :682)
  int path;
};

// value, gradient (on x0, x1 and x_tv) and Hessian of the one nonlinear constraint
struct ConeEval { double f, g0, g1, gt, h00, h11, h0t, h1t, htt; };
RDA_HD ConeEval cone_eval(const double* x, int tv) {
  ConeEval c;
  if (tv < 0) {
    c.f = x[0] * x[0] + x[1] * x[1] - 1.0;
    c.g0 = 2 * x[0]; c.g1 = 2 * x[1]; c.gt = 0;
    c.h00 = 2; c.h11 = 2; c.h0t = 0; c.h1t = 0; c.htt = 0;
  } else {
    double t = x[tv], n2 = x[0] * x[0] + x[1] * x[1];
    c.f = n2 / t - t;
    c.g0 = 2 * x[0] / t; c.g1 = 2 * x[1] / t; c.gt = -n2 / (t * t) - 1.0;
    c.h00 = 2 / t; c.h11 = 2 / t; c.h0t = -2 * x[0] / (t * t); c.h1t = -2 * x[1] / (t * t);
    c.htt = 2 * n2 / (t * t * t);
  }
  return c;
}

// ---------------------------------------------------------------------------------------------
// Geometry of one cell, relative to the robot reference point.
// ---------------------------------------------------------------------------------------------
template <typename Real>
struct CellGeom {
  int kind, ne;
  Real vx[RDA_MAX_EDGE], vy[RDA_MAX_EDGE];     // polygon vertices (vertex i joins rows i-1, i)
  Real nx[RDA_MAX_EDGE], ny[RDA_MAX_EDGE];     // unit outward normals of rows
  Real inv_norm[RDA_MAX_EDGE];                 // 1/|A_i|
  Real cx, cy, rad;                            // disc
  Real yx[RDA_MAX_ROBOT_EDGE], yy[RDA_MAX_ROBOT_EDGE];  // robot vertices rotated into the world frame
  Real mx[RDA_MAX_ROBOT_EDGE], my[RDA_MAX_ROBOT_EDGE];  // robot edge normals in the world frame
};

template <typename Real>
RDA_HD Real support_obs(const CellGeom<Real>& g, Real vx, Real vy, int* arg) {
  if (g.kind == RDA_OBS_CIRCLE) {
    *arg = 0;
    return vx * g.cx + vy * g.cy + g.rad * sqrt_(vx * vx + vy * vy);
  }
  Real best = -1e30f;
  int bi = 0;
  for (int i = 0; i < g.ne; ++i) {
    Real s = vx * g.vx[i] + vy * g.vy[i];
    if (s > best) { best = s; bi = i; }
  }
  *arg = bi;
  return best;
}

template <typename Real>
RDA_HD Real support_rob(const RobotGeom& rb, Real gx, Real gy, int* arg) {
  Real best = -1e30f;
  int bj = 0;
  for (int j = 0; j < rb.R; ++j) {
    Real s = gx * (Real)rb.yx[j] + gy * (Real)rb.yy[j];
    if (s > best) { best = s; bj = j; }
  }
  *arg = bj;
  return best;
}

// LP-vertex multipliers of the obstacle for the direction v = A'lam: v = al n_{a} + be n_{b} at the vertex joining rows a and b.
// The two ends of a short edge have supports within |edge| of each other, and the vertex between two nearly parallel rows is
// computed to a float32 error of eps |b| / det; so the support can go to the wrong end of a short edge.  v then lies outside
// that vertex's normal cone: one coefficient is negative, and between nearly parallel rows the other is huge (|A'lam| = 26 on
// a hull with a 1.2e-4 m edge).  A clearly negative coefficient therefore moves the vertex towards its row until v lies in
// the cone.  At a correct support vertex nothing moves, so results there are unchanged.
// Between rows delta apart the coefficients also carry a rounding error of eps / delta (the 2x2 determinant is delta), so
// |al n_a + be n_b| can exceed |v| <= 1 by that much: cone_rescale (rda_hd.h) scales such a pair back to the length of v.
template <typename Real>
RDA_HD void obs_vertex_lam(const CellGeom<Real>& g, int io, Real v0, Real v1, Real* lam) {
  const int ne = g.ne;
  const Real tol = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
  int a = (io + ne - 1) % ne, bb = io;
  Real det = g.nx[a] * g.ny[bb] - g.ny[a] * g.nx[bb];
  Real al = (v0 * g.ny[bb] - v1 * g.nx[bb]) / det;
  Real be = (g.nx[a] * v1 - g.ny[a] * v0) / det;
  if (rmin(al, be) < -tol) {
    const bool back = be < al;            // v lies before row a: previous vertex; past row bb: next vertex
    for (int s = 1; s < ne; ++s) {
      if (back) { bb = a; a = (a + ne - 1) % ne; }
      else { a = bb; bb = (bb + 1) % ne; }
      det = g.nx[a] * g.ny[bb] - g.ny[a] * g.nx[bb];
      al = (v0 * g.ny[bb] - v1 * g.nx[bb]) / det;
      be = (g.nx[a] * v1 - g.ny[a] * v0) / det;
      if ((back ? be : al) >= -tol) break;
    }
  }
  al = rmax(al, (Real)0); be = rmax(be, (Real)0);
  cone_rescale<Real>(g.nx[a], g.ny[a], g.nx[bb], g.ny[bb], v0, v1, al, be);
  lam[a] = al * g.inv_norm[a];
  lam[bb] = be * g.inv_norm[bb];
}

// g (body frame) inside the normal cone of body vertex j?
template <typename Real>
RDA_HD bool in_cone_rob(const RobotGeom& rb, int j, Real gx, Real gy, Real tol) {
  const int R = rb.R;
  int jp = (j + R - 1) % R, jn = (j + 1) % R;
  Real epx = (Real)rb.yx[j] - (Real)rb.yx[jp], epy = (Real)rb.yy[j] - (Real)rb.yy[jp];
  Real enx = (Real)rb.yx[jn] - (Real)rb.yx[j], eny = (Real)rb.yy[jn] - (Real)rb.yy[j];
  Real gn = sqrt_(gx * gx + gy * gy);
  Real a = gx * epx + gy * epy, b = gx * enx + gy * eny;
  return a >= -tol * gn * sqrt_(epx * epx + epy * epy) && b <= tol * gn * sqrt_(enx * enx + eny * eny);
}

// Everything one cell carries between its three stages (front: geometry + closed forms,
// slow: interior point, back: multipliers and updates).
template <typename Real>
struct CellWork {
  CellGeom<Real> g;
  Real k0, cphi, sphi, xi0, xi1, ro2;
  bool sep, xi_zero, circ;
  Real best, byx, byy;
  Real rob_in[RDA_MAX_ROBOT_EDGE], obs_in[RDA_MAX_EDGE];
  Real v0, v1, g0, g1;
  bool exact_zero_q, have;
  int path;
};

// ---- stage 1: geometry relative to the robot reference point and the closed-form cases ----------
// EXTRA: also try the candidates that only the (rare) cells of the last pass need: robot edge against obstacle edge.
// The searched pass leaves them out (every one of its cells would pay for the extra candidates, r02 measurement).
template <typename Real, bool EXTRA = false>
RDA_HD void cell_front(const RobotGeom& rb, int kind, int E, const float* A, const float* b, Real px, Real py,
                       Real cphi, Real sphi, Real dbar, Real zeta, Real xi0, Real xi1, Real ro2,
                       CellWork<Real>& w) {
  const int R = rb.R;
  const Real k0 = dbar - zeta;
  const Real eps = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
  CellGeom<Real>& g = w.g;
  w.k0 = k0; w.cphi = cphi; w.sphi = sphi; w.xi0 = xi0; w.xi1 = xi1; w.ro2 = ro2;
  w.circ = (kind == RDA_OBS_CIRCLE);
  g.kind = kind;
  for (int j = 0; j < R; ++j) {
    Real yx = rb.yx[j], yy = rb.yy[j];
    g.yx[j] = cphi * yx - sphi * yy;
    g.yy[j] = sphi * yx + cphi * yy;
    Real nx = rb.nx[j], ny = rb.ny[j];
    g.mx[j] = cphi * nx - sphi * ny;
    g.my[j] = sphi * nx + cphi * ny;
  }
  int ne = 0;
  Real brel[RDA_MAX_EDGE];
  if (kind == RDA_OBS_CIRCLE) {
    g.cx = (Real)b[0] - px;
    g.cy = (Real)b[1] - py;
    g.rad = -(Real)b[2];
    g.ne = 0;
  } else {
    for (int i = 0; i < E; ++i) {
      Real ax = A[2 * i], ay = A[2 * i + 1];
      Real n2 = ax * ax + ay * ay;
      if (!(n2 > 0)) break;
      Real inv = rsqrt_(n2);
      g.nx[i] = ax * inv;
      g.ny[i] = ay * inv;
      g.inv_norm[i] = inv;
      brel[i] = ((Real)b[i] - ax * px - ay * py) * inv;
      ne = i + 1;
    }
    g.ne = ne;
    for (int i = 0; i < ne; ++i) {
      int a = (i + ne - 1) % ne;
      Real det = g.nx[a] * g.ny[i] - g.ny[a] * g.nx[i];
      Real inv = (Real)1 / det;
      g.vx[i] = (brel[a] * g.ny[i] - brel[i] * g.ny[a]) * inv;
      g.vy[i] = (g.nx[a] * brel[i] - g.nx[i] * brel[a]) * inv;
    }
  }
  // ---- closest pair / separation ----
  bool sep = false;
  Real best = 1e30f, bdx = 0, bdy = 0;
  Real byx = 0, byy = 0;            // robot-side point of the closest pair, body frame
  int ce_i = -1, ce_j = -1;         // closest pair = (obstacle vertex i / disc, interior of robot edge j)
  int ei_of[RDA_MAX_ROBOT_EDGE];    // per robot edge: nearest obstacle vertex
  for (int j = 0; j < R; ++j) ei_of[j] = 0;
  Real dj2[RDA_MAX_ROBOT_EDGE], djx[RDA_MAX_ROBOT_EDGE], djy[RDA_MAX_ROBOT_EDGE];
  for (int j = 0; j < R; ++j) { dj2[j] = 1e30f; w.rob_in[j] = -1e30f; }
  if (kind == RDA_OBS_CIRCLE) {
    bool inside = true;
    for (int j = 0; j < R; ++j) {
      int jn = (j + 1) % R;
      Real fx = g.yx[jn] - g.yx[j], fy = g.yy[jn] - g.yy[j];
      Real rx = g.cx - g.yx[j], ry = g.cy - g.yy[j];
      if (g.mx[j] * rx + g.my[j] * ry > 0) inside = false;
      Real t = rclamp((rx * fx + ry * fy) / (fx * fx + fy * fy), (Real)0, (Real)1);
      Real dx = -(rx - t * fx), dy = -(ry - t * fy);       // robot point minus centre
      Real d2 = dx * dx + dy * dy;
      if (d2 < best) {
        best = d2; bdx = dx; bdy = dy;
        byx = (Real)rb.yx[j] + t * ((Real)rb.yx[jn] - (Real)rb.yx[j]);
        byy = (Real)rb.yy[j] + t * ((Real)rb.yy[jn] - (Real)rb.yy[j]);
        ce_i = 0; ce_j = (t > (Real)0 && t < (Real)1) ? j : -1;
      }
      Real vx_ = g.yx[j] - g.cx, vy_ = g.yy[j] - g.cy;     // robot vertex minus centre
      Real dv = sqrt_(vx_ * vx_ + vy_ * vy_);
      Real dd = dv - g.rad;
      if (dv > eps && dd > 0) {
        dj2[j] = dd * dd;
        djx[j] = vx_ / dv * dd;
        djy[j] = vy_ / dv * dd;
      } else {
        dj2[j] = 0; djx[j] = 0; djy[j] = 0;
      }
    }
    Real dc = sqrt_(best);
    sep = (!inside) && (dc > g.rad + eps);
    if (sep) {
      Real dd = dc - g.rad;
      bdx = bdx / dc * dd;
      bdy = bdy / dc * dd;
      best = dd * dd;
    }
  } else {
    for (int i = 0; i < ne; ++i) {
      int in = (i + 1) % ne;
      Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
      Real ie2 = (Real)1 / (ex * ex + ey * ey);
      Real mins = 1e30f;
      for (int j = 0; j < R; ++j) {
        Real rx = g.yx[j] - g.vx[i], ry = g.yy[j] - g.vy[i];
        Real sd = g.nx[i] * rx + g.ny[i] * ry;
        mins = rmin(mins, sd);
        w.rob_in[j] = rmax(w.rob_in[j], sd);        // <= 0 for every edge: robot vertex j inside O
        Real t = rclamp((rx * ex + ry * ey) * ie2, (Real)0, (Real)1);
        Real dx = rx - t * ex, dy = ry - t * ey;
        Real d2 = dx * dx + dy * dy;
        if (d2 < dj2[j]) { dj2[j] = d2; djx[j] = dx; djy[j] = dy; }
      }
      if (mins > eps) sep = true;
    }
    for (int j = 0; j < R; ++j)
      if (dj2[j] < best) { best = dj2[j]; bdx = djx[j]; bdy = djy[j]; byx = rb.yx[j]; byy = rb.yy[j]; ce_j = -1; }
    for (int j = 0; j < R; ++j) {
      int jn = (j + 1) % R;
      Real fx = g.yx[jn] - g.yx[j], fy = g.yy[jn] - g.yy[j];
      Real if2 = (Real)1 / (fx * fx + fy * fy);
      Real mins = 1e30f, ebest = 1e30f;
      for (int i = 0; i < ne; ++i) {
        Real rx = g.vx[i] - g.yx[j], ry = g.vy[i] - g.yy[j];
        Real sd = g.mx[j] * rx + g.my[j] * ry;
        mins = rmin(mins, sd);
        w.obs_in[i] = (j == 0) ? sd : rmax(w.obs_in[i], sd);   // <= 0: obstacle vertex i inside the robot
        Real t = rclamp((rx * fx + ry * fy) * if2, (Real)0, (Real)1);
        Real dx = -(rx - t * fx), dy = -(ry - t * fy);
        Real d2 = dx * dx + dy * dy;
        if (d2 < ebest && sd > 0) { ebest = d2; ei_of[j] = i; }
        if (d2 < best) {
          best = d2; bdx = dx; bdy = dy;
          byx = (Real)rb.yx[j] + t * ((Real)rb.yx[jn] - (Real)rb.yx[j]);
          byy = (Real)rb.yy[j] + t * ((Real)rb.yy[jn] - (Real)rb.yy[j]);
          ce_i = i; ce_j = (t > (Real)0 && t < (Real)1) ? j : -1;
        }
      }
      if (mins > eps) sep = true;
    }
  }
  w.sep = sep; w.best = best; w.byx = byx; w.byy = byy;
  // ---- closed-form candidates ----
  Real v0 = 0, v1 = 0, g0 = 0, g1 = 0;
  bool exact_zero_q = false, have = false;
  int path = CELL_FAILED;
  const bool xi_zero = (xi0 == (Real)0) && (xi1 == (Real)0);
  w.xi_zero = xi_zero;
  if (sep && xi_zero) {
    Real dist = sqrt_(best);
    if (dist - k0 >= 0) {
      v0 = bdx / dist; v1 = bdy / dist;
      g0 = -(cphi * v0 + sphi * v1);
      g1 = -(-sphi * v0 + cphi * v1);
      exact_zero_q = true; have = true; path = CELL_FAST_INACTIVE;
    }
  }
  if (!have && !sep && xi_zero && k0 <= 0) {
    // overlapping sets, no tilt: max margin is 0 at v = 0 (stuff = -k0 >= 0)
    exact_zero_q = true; have = true; path = CELL_OVERLAP_FREE;
  }
  if (!have && sep) {
    const Real tolc = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
    for (int j = 0; j < R && !have; ++j) {
      Real dj = sqrt_(dj2[j]);
      if (!(dj > eps)) continue;
      Real vjx = djx[j] / dj, vjy = djy[j] / dj;
      Real yx = rb.yx[j], yy = rb.yy[j];
      Real Dj = dj + xi0 * yx + xi1 * yy - k0;
      Real rvx = cphi * vjx + sphi * vjy, rvy = -sphi * vjx + cphi * vjy;   // R'v
      if (Dj >= 0) {
        Real cgx = -rvx - xi0, cgy = -rvy - xi1;
        if (in_cone_rob<Real>(rb, j, cgx, cgy, tolc)) {
          v0 = vjx; v1 = vjy; g0 = cgx; g1 = cgy;
          exact_zero_q = true; have = true; path = CELL_FAST_VERTEX;
        }
      } else {
        Real tau = -Dj / ((Real)1 + (yx * yx + yy * yy) / ro2);
        Real qx = -tau * yx / ro2, qy = -tau * yy / ro2;
        Real cgx = qx - rvx - xi0, cgy = qy - rvy - xi1;
        if (in_cone_rob<Real>(rb, j, cgx, cgy, tolc)) {
          v0 = vjx; v1 = vjy; g0 = cgx; g1 = cgy;
          have = true; path = CELL_FAST_VERTEX;
        }
      }
    }
  }
  for (int ecand = 0; ecand <= R && !have; ++ecand) {
    // candidate edges: the closest pair's edge (disjoint sets); for overlapping sets every robot edge
    // with the nearest obstacle vertex in front of it
    if (ecand == 0) { if (!sep || ce_j < 0) continue; }
    else { if (kind == RDA_OBS_CIRCLE) break; ce_j = ecand - 1; ce_i = ei_of[ce_j]; }
    // Robot-EDGE contact: the optimal body point lies in the interior of edge j, the obstacle point is
    // the vertex (or disc centre) ce_i.  One-dimensional problem along the edge,
    //    maximise  N(s)/W(s),  N = k0 - xi.y - rho(s),  W^2 = 1 + |y|^2/ro2   (W = 1: max-margin stage)
    // solved by safeguarded Newton on h(s) = N' W^2 - N (y.f)/ro2, then accepted by the KKT conditions
    // of the (convex) cell problem: multiplier of the edge >= 0 and v in the obstacle's normal cone.
    const int j = ce_j, jn = (j + 1) % R;
    const Real yjx = rb.yx[j], yjy = rb.yy[j];
    const Real fx = (Real)rb.yx[jn] - yjx, fy = (Real)rb.yy[jn] - yjy;           // body frame
    const Real wfx = cphi * fx - sphi * fy, wfy = sphi * fx + cphi * fy;         // R f
    const Real ox = (kind == RDA_OBS_CIRCLE) ? g.cx : g.vx[ce_i], oy = (kind == RDA_OBS_CIRCLE) ? g.cy : g.vy[ce_i];
    const Real rad = (kind == RDA_OBS_CIRCLE) ? g.rad : (Real)0;
    const Real xf = xi0 * fx + xi1 * fy;
    Real sA = -1;                    // maximiser of the unweighted margin N along the edge (stage A)
    for (int stage = 0; stage < 2 && !have; ++stage) {
      const bool weighted = stage == 1;
      Real hv = 0, Nv = 0, W2 = 1, vx_ = 0, vy_ = 0, yx = 0, yy = 0;
      // h(s) = d/ds of N/W (times W^3): N' W^2 - N (y.f)/ro2;  unweighted: N'
      auto eval = [&](Real sc) {
        yx = yjx + sc * fx; yy = yjy + sc * fy;
        const Real rx = (cphi * yx - sphi * yy) - ox, ry = (sphi * yx + cphi * yy) - oy;
        const Real rn = sqrt_(rx * rx + ry * ry);
        vx_ = rx / rn; vy_ = ry / rn;
        Nv = k0 - (xi0 * yx + xi1 * yy) - (rn - rad);
        const Real Np = -xf - (vx_ * wfx + vy_ * wfy);
        W2 = weighted ? (Real)1 + (yx * yx + yy * yy) / ro2 : (Real)1;
        hv = weighted ? Np * W2 - Nv * (yx * fx + yy * fy) / ro2 : Np;
      };
      Real lo = 0, hi = 1;
      int dir = 0;                   // weighted stage: which side of sA the maximiser lies on
      bool bracket = true;
      // h at the bracket ends (flo > 0 at lo, fhi < 0 at hi) where it was evaluated inside the region N > 0
      Real flo = 0, fhi = 0;
      bool vlo = false, vhi = false;
      if (!weighted) {
        eval((Real)0); const Real h0 = hv;
        eval((Real)1); const Real h1 = hv;
        if (!(h0 > 0 && h1 < 0)) {                     // N has no interior maximum on this edge:
          bracket = false;                             // concave N, so it is largest at the end it increases towards
          // the WEIGHTED margin may still peak inside the edge; rare (0.02 % of the cells), so only the last pass looks
          // for it: the searched pass would pay a root search per candidate edge
          sA = !EXTRA ? (Real)-1 : h1 >= 0 ? (Real)1 : (Real)0;
        }
        flo = h0; fhi = h1; vlo = vhi = true;
      } else {
        // sA: maximiser of the unweighted margin N on the edge (an end point when N is monotone there).  The WEIGHTED margin
        // N/W is quasi-concave where N > 0, an interval that contains sA: its maximiser lies on the side of sA that h points to.
        if (!(sA >= 0)) bracket = false;
        else {
          eval(sA);
          if (!(Nv > 0)) bracket = false;              // hinge cannot be active with contact on this edge
          else if (hv > 0) {
            dir = 1; lo = sA; hi = 1; flo = hv; vlo = true;
            eval((Real)1);
            if (Nv > 0 && hv > 0) bracket = false;
            fhi = hv; vhi = Nv > 0;
          } else {
            dir = -1; lo = 0; hi = sA; fhi = hv; vhi = true;
            eval((Real)0);
            if (Nv > 0 && hv < 0) bracket = false;
            flo = hv; vlo = Nv > 0;
          }
        }
      }
      if (bracket) {
        // Root of h on [lo, hi]: regula falsi with the Illinois modification where both end values are valid,
        // plain bisection otherwise (outside the region N > 0 the ratio N/W is not quasi-concave: steer back
        // towards sA).  Superlinear: ~6-8 evaluations instead of the 26 of pure bisection (ncu r02: the
        // bisection was half of k_cells_mid's instructions).
        const Real tol = sizeof(Real) == 4 ? (Real)2e-7 : (Real)1e-13;
        Real sc = (Real)0.5 * (lo + hi), sprev = -1;
        int side = 0;
        for (int itn = 0; itn < 40; ++itn) {
          const Real w = hi - lo;
          if (vlo && vhi && flo > 0 && fhi < 0) {
            sc = lo + w * (flo / (flo - fhi));
            sc = rclamp(sc, lo + (Real)0.02 * w, hi - (Real)0.02 * w);
          } else {
            sc = (Real)0.5 * (lo + hi);
          }
          eval(sc);
          const bool valid = !weighted || Nv > 0;
          const bool pos = valid ? hv > 0 : dir < 0;
          if (pos) { lo = sc; flo = hv; vlo = valid; if (side > 0 && vhi) fhi *= (Real)0.5; side = 1; }
          else { hi = sc; fhi = hv; vhi = valid; if (side < 0 && vlo) flo *= (Real)0.5; side = -1; }
          if (hi - lo < tol || abs_(sc - sprev) < tol || (valid && hv == (Real)0)) break;
          sprev = sc;
        }
        if (!weighted) sA = sc;
      }
      if (!bracket) continue;
      // KKT of the cell problem at this point
      const Real rvx = cphi * vx_ + sphi * vy_, rvy = -sphi * vx_ + cphi * vy_;   // R'v
      const Real tolc = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
      // tangential residual of g on the edge: h is the tangential component of the gradient scaled by W^2 |f| (steep: a
      // slope of 1e4..1e5 per unit s with the metric's ro), so ONE float32 ulp of s leaves a residual of 1e-4; such a root
      // fails this test and its cell goes on to the interior point iteration (DESIGN.md §3.1)
      const Real tole = sizeof(Real) == 4 ? (Real)3e-5 : (Real)1e-9;
      bool cone_ok = true;
      if (kind != RDA_OBS_CIRCLE) {
        const int ip = (ce_i + ne - 1) % ne, inx = (ce_i + 1) % ne;
        const Real epx = g.vx[ce_i] - g.vx[ip], epy = g.vy[ce_i] - g.vy[ip];
        const Real enx = g.vx[inx] - g.vx[ce_i], eny = g.vy[inx] - g.vy[ce_i];
        cone_ok = (vx_ * epx + vy_ * epy >= -tolc * sqrt_(epx * epx + epy * epy)) &&
                  (vx_ * enx + vy_ * eny <= tolc * sqrt_(enx * enx + eny * eny));
      }
      if (!cone_ok) continue;
      if (!weighted) {
        if (Nv <= 0) {   // max margin -N >= 0 with Hm + xi = 0: inactive
          const Real cgx = -rvx - xi0, cgy = -rvy - xi1;
          // g must be a non-negative multiple of the edge normal: no tangential component left
          const Real tang = abs_(cgx * fx + cgy * fy) * rsqrt_(fx * fx + fy * fy);
          if (cgx * (Real)rb.nx[j] + cgy * (Real)rb.ny[j] >= -tolc && tang <= tole) {
            v0 = vx_; v1 = vy_; g0 = cgx; g1 = cgy;
            exact_zero_q = true; have = true; path = CELL_FAST_VERTEX;
          }
        }
      } else if (Nv > 0) {
        const Real tau = Nv / W2;
        const Real cgx = -tau * yx / ro2 - rvx - xi0, cgy = -tau * yy / ro2 - rvy - xi1;
        const Real tang = abs_(cgx * fx + cgy * fy) * rsqrt_(fx * fx + fy * fy);
        if (cgx * (Real)rb.nx[j] + cgy * (Real)rb.ny[j] >= -tolc && tang <= tole) {
          v0 = vx_; v1 = vy_; g0 = cgx; g1 = cgy;
          have = true; path = CELL_FAST_VERTEX;
        }
      }
    }
  }
  if (EXTRA && !have && sep && kind != RDA_OBS_CIRCLE) {
    // Robot-EDGE against obstacle-EDGE contact (disjoint sets, active hinge): the optimal body point lies in the
    // interior of body edge j and its nearest obstacle point in the interior of obstacle edge i, so v = n_i and the
    // distance n_i.(R y - V_i) is LINEAR along the body edge: the weighted margin N/W has the closed-form stationary
    // point s* = -(beta a + alpha b)/(beta b + alpha c) (as in the overlap cases below), accepted through the KKT
    // conditions.  (With the unweighted margin N is linear in s: no interior maximum, those are vertex contacts.)
    const Real tolc = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
    for (int j = 0; j < R && !have; ++j) {
      const int jn = (j + 1) % R;
      const Real yjx = rb.yx[j], yjy = rb.yy[j];
      const Real fx = (Real)rb.yx[jn] - yjx, fy = (Real)rb.yy[jn] - yjy;            // body frame
      const Real wfx = cphi * fx - sphi * fy, wfy = sphi * fx + cphi * fy;          // R f
      const Real a_ = (Real)1 + (yjx * yjx + yjy * yjy) / ro2, b_ = (yjx * fx + yjy * fy) / ro2;
      const Real c_ = (fx * fx + fy * fy) / ro2;
      for (int i = 0; i < ne && !have; ++i) {
        const Real nix = g.nx[i], niy = g.ny[i];
        const Real nf = nix * wfx + niy * wfy;                                         // n_i . R f
        const Real rho0 = nix * (g.yx[j] - g.vx[i]) + niy * (g.yy[j] - g.vy[i]);       // distance of R y_j to the edge line
        const Real al = k0 - (xi0 * yjx + xi1 * yjy) - rho0, be = (xi0 * fx + xi1 * fy) + nf;
        const Real den = be * b_ + al * c_;
        if (!(abs_(den) > (Real)1e-20)) continue;
        const Real sst = -(be * a_ + al * b_) / den;
        if (!(sst > tolc && sst < (Real)1 - tolc)) continue;
        const Real yx = yjx + sst * fx, yy = yjy + sst * fy;
        const Real rho = rho0 + sst * nf;
        const Real Nv = al - be * sst;
        if (!(rho > eps && Nv > 0)) continue;
        // foot of the body point on obstacle edge i must lie strictly inside the edge
        const int in = (i + 1) % ne;
        const Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
        const Real wx = (cphi * yx - sphi * yy) - rho * nix - g.vx[i], wy = (sphi * yx + cphi * yy) - rho * niy - g.vy[i];
        const Real so_ = (wx * ex + wy * ey) / (ex * ex + ey * ey);
        if (!(so_ > tolc && so_ < (Real)1 - tolc)) continue;
        const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
        const Real rvx = cphi * nix + sphi * niy, rvy = -sphi * nix + cphi * niy;      // R'v
        const Real cgx = -tau * yx / ro2 - rvx - xi0, cgy = -tau * yy / ro2 - rvy - xi1;
        // s* is a stationary point in closed form: the tangential component of g is rounding only (bounded loosely)
        const Real tang = abs_(cgx * fx + cgy * fy) * rsqrt_(fx * fx + fy * fy);
        if (!(cgx * (Real)rb.nx[j] + cgy * (Real)rb.ny[j] >= -tolc && tang <= (Real)CELL_EE_TANG)) continue;
        v0 = nix; v1 = niy; g0 = cgx; g1 = cgy;
        have = true; path = CELL_FAST_VERTEX;
      }
    }
  }
  if (!have && !sep && k0 > 0) {
    // Deep overlap: the optimal contact point y = -ro2 xi / k0 lies inside the robot AND inside the
    // obstacle; then v = 0, g = 0 (lam = mu = 0), tau = k0 and q = xi satisfy the KKT conditions.
    const Real yx = -ro2 * xi0 / k0, yy = -ro2 * xi1 / k0;
    bool inside = true;
    for (int j = 0; j < R; ++j) {
      const Real sd = (Real)rb.nx[j] * (yx - (Real)rb.yx[j]) + (Real)rb.ny[j] * (yy - (Real)rb.yy[j]);
      if (sd > -eps) inside = false;
    }
    const Real wx = cphi * yx - sphi * yy, wy = sphi * yx + cphi * yy;
    if (kind == RDA_OBS_CIRCLE) {
      const Real dx = wx - g.cx, dy = wy - g.cy;
      if (dx * dx + dy * dy > (g.rad - eps) * (g.rad - eps) || g.rad <= eps) inside = false;
    } else {
      for (int i = 0; i < ne; ++i) {
        const Real sd = g.nx[i] * (wx - g.vx[i]) + g.ny[i] * (wy - g.vy[i]);
        if (sd > -eps) inside = false;
      }
    }
    if (inside) {
      v0 = 0; v1 = 0; g0 = 0; g1 = 0;
      exact_zero_q = false; have = true; path = CELL_OVERLAP_FREE;
    }
  }
  if (!have && !sep) {
    // Overlapping sets, contact point with zero distance.  Along a line y = p + s d (body frame) the
    // weighted margin (k0 - xi.y)/sqrt(1 + |y|^2/ro2) has the closed-form stationary point
    //    s* = -(beta a + alpha b)/(beta b + alpha c),  alpha = k0 - xi.p, beta = xi.d,
    //    a = 1 + |p|^2/ro2, b = p.d/ro2, c = |d|^2/ro2.
    const Real tolc = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
    // (ii) y on robot edge j, P(y) strictly inside the obstacle: v = 0, g = gamma m_j
    for (int j = 0; j < R && !have; ++j) {
      const int jn = (j + 1) % R;
      const Real px_ = rb.yx[j], py_ = rb.yy[j];
      const Real dx_ = (Real)rb.yx[jn] - px_, dy_ = (Real)rb.yy[jn] - py_;
      const Real al = k0 - (xi0 * px_ + xi1 * py_), be = xi0 * dx_ + xi1 * dy_;
      const Real a_ = (Real)1 + (px_ * px_ + py_ * py_) / ro2, b_ = (px_ * dx_ + py_ * dy_) / ro2;
      const Real c_ = (dx_ * dx_ + dy_ * dy_) / ro2;
      const Real den = be * b_ + al * c_;
      if (!(abs_(den) > (Real)1e-20)) continue;
      const Real sst = -(be * a_ + al * b_) / den;
      if (!(sst > tolc && sst < (Real)1 - tolc)) continue;
      const Real yx = px_ + sst * dx_, yy = py_ + sst * dy_;
      const Real Nv = k0 - (xi0 * yx + xi1 * yy);
      if (!(Nv > 0)) continue;
      const Real wx = cphi * yx - sphi * yy, wy = sphi * yx + cphi * yy;
      bool inside = true;
      if (kind == RDA_OBS_CIRCLE) {
        const Real ex = wx - g.cx, ey = wy - g.cy;
        inside = g.rad > eps && ex * ex + ey * ey < (g.rad - eps) * (g.rad - eps);
      } else {
        for (int i = 0; i < ne; ++i)
          if (g.nx[i] * (wx - g.vx[i]) + g.ny[i] * (wy - g.vy[i]) > -eps) inside = false;
      }
      if (!inside) continue;
      const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
      const Real cgx = -tau * yx / ro2 - xi0, cgy = -tau * yy / ro2 - xi1;
      if (cgx * (Real)rb.nx[j] + cgy * (Real)rb.ny[j] < -tolc) continue;
      v0 = 0; v1 = 0; g0 = cgx; g1 = cgy;
      have = true; path = CELL_OVERLAP_FREE;
    }
    // (iii) P(y) on obstacle edge i, y strictly inside the robot: g = 0, v = alpha n_i, 0 <= alpha <= 1
    if (kind != RDA_OBS_CIRCLE) {
      for (int i = 0; i < ne && !have; ++i) {
        const int in = (i + 1) % ne;
        const Real px_ = cphi * g.vx[i] + sphi * g.vy[i], py_ = -sphi * g.vx[i] + cphi * g.vy[i];   // R'V_i
        const Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
        const Real dx_ = cphi * ex + sphi * ey, dy_ = -sphi * ex + cphi * ey;
        const Real al = k0 - (xi0 * px_ + xi1 * py_), be = xi0 * dx_ + xi1 * dy_;
        const Real a_ = (Real)1 + (px_ * px_ + py_ * py_) / ro2, b_ = (px_ * dx_ + py_ * dy_) / ro2;
        const Real c_ = (dx_ * dx_ + dy_ * dy_) / ro2;
        const Real den = be * b_ + al * c_;
        if (!(abs_(den) > (Real)1e-20)) continue;
        const Real sst = -(be * a_ + al * b_) / den;
        if (!(sst > tolc && sst < (Real)1 - tolc)) continue;
        const Real yx = px_ + sst * dx_, yy = py_ + sst * dy_;
        const Real Nv = k0 - (xi0 * yx + xi1 * yy);
        if (!(Nv > 0)) continue;
        bool inside = true;
        for (int j = 0; j < R; ++j)
          if ((Real)rb.nx[j] * (yx - (Real)rb.yx[j]) + (Real)rb.ny[j] * (yy - (Real)rb.yy[j]) > -eps) inside = false;
        if (!inside) continue;
        const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
        const Real rx = -tau * yx / ro2 - xi0, ry = -tau * yy / ro2 - xi1;      // must equal R'v
        const Real nbx = cphi * g.nx[i] + sphi * g.ny[i], nby = -sphi * g.nx[i] + cphi * g.ny[i];
        const Real alpha = rx * nbx + ry * nby;
        if (!(alpha >= -tolc && alpha <= (Real)1 + tolc)) continue;
        const Real ac = rclamp(alpha, (Real)0, (Real)1);
        v0 = ac * g.nx[i]; v1 = ac * g.ny[i]; g0 = 0; g1 = 0;
        have = true; path = CELL_OVERLAP_FREE;
      }
      // (iv) obstacle vertex i strictly inside the robot: y = R'V_i, g = 0, v = R(-tau y/ro2 - xi) must lie
      //      in the normal cone of the vertex with |v| <= 1
      for (int i = 0; i < ne && !have; ++i) {
        if (!(w.obs_in[i] < -eps)) continue;
        const Real yx = cphi * g.vx[i] + sphi * g.vy[i], yy = -sphi * g.vx[i] + cphi * g.vy[i];
        const Real Nv = k0 - (xi0 * yx + xi1 * yy);
        if (!(Nv > 0)) continue;
        const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
        const Real rx = -tau * yx / ro2 - xi0, ry = -tau * yy / ro2 - xi1;
        const Real vx_ = cphi * rx - sphi * ry, vy_ = sphi * rx + cphi * ry;          // v = R r
        if (vx_ * vx_ + vy_ * vy_ > (Real)1 + tolc) continue;
        const int ip = (i + ne - 1) % ne, in = (i + 1) % ne;
        const Real epx = g.vx[i] - g.vx[ip], epy = g.vy[i] - g.vy[ip];
        const Real enx = g.vx[in] - g.vx[i], eny = g.vy[in] - g.vy[i];
        if (vx_ * epx + vy_ * epy < -tolc * sqrt_(epx * epx + epy * epy)) continue;
        if (vx_ * enx + vy_ * eny > tolc * sqrt_(enx * enx + eny * eny)) continue;
        v0 = vx_; v1 = vy_; g0 = 0; g1 = 0;
        have = true; path = CELL_OVERLAP_FREE;
      }
      // (v) crossing of robot edge j and obstacle edge i: y fixed, g = gamma m_j, v = alpha n_i with
      //     gamma m_j + alpha R'n_i = -tau y/ro2 - xi  (2 x 2 linear system), gamma >= 0, 0 <= alpha <= 1
      for (int j = 0; j < R && !have; ++j) {
        const int jn = (j + 1) % R;
        const Real ax_ = g.yx[j], ay_ = g.yy[j];
        const Real fx_ = g.yx[jn] - ax_, fy_ = g.yy[jn] - ay_;                        // world frame
        for (int i = 0; i < ne && !have; ++i) {
          const int in = (i + 1) % ne;
          const Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
          const Real det = fx_ * ey - fy_ * ex;
          if (!(abs_(det) > (Real)1e-12)) continue;
          const Real wx_ = g.vx[i] - ax_, wy_ = g.vy[i] - ay_;
          const Real sr = (wx_ * ey - wy_ * ex) / det;          // along the robot edge
          const Real so_ = (wx_ * fy_ - wy_ * fx_) / det;       // along the obstacle edge
          if (!(sr > tolc && sr < (Real)1 - tolc && so_ > tolc && so_ < (Real)1 - tolc)) continue;
          const Real yx = (Real)rb.yx[j] + sr * ((Real)rb.yx[jn] - (Real)rb.yx[j]);
          const Real yy = (Real)rb.yy[j] + sr * ((Real)rb.yy[jn] - (Real)rb.yy[j]);
          const Real Nv = k0 - (xi0 * yx + xi1 * yy);
          if (!(Nv > 0)) continue;
          const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
          const Real rx = -tau * yx / ro2 - xi0, ry = -tau * yy / ro2 - xi1;
          const Real mjx = rb.nx[j], mjy = rb.ny[j];
          const Real nbx = cphi * g.nx[i] + sphi * g.ny[i], nby = -sphi * g.nx[i] + cphi * g.ny[i];
          const Real d2 = mjx * nby - mjy * nbx;
          if (!(abs_(d2) > (Real)1e-9)) continue;
          const Real gam = (rx * nby - ry * nbx) / d2;
          const Real alp = (mjx * ry - mjy * rx) / d2;
          if (!(gam >= -tolc && alp >= -tolc && alp <= (Real)1 + tolc)) continue;
          const Real ac = rclamp(alp, (Real)0, (Real)1), gc = rmax(gam, (Real)0);
          v0 = ac * g.nx[i]; v1 = ac * g.ny[i]; g0 = gc * mjx; g1 = gc * mjy;
          have = true; path = CELL_OVERLAP_FREE;
        }
      }
    }
  }
  w.v0 = v0; w.v1 = v1; w.g0 = g0; w.g1 = g1;
  w.exact_zero_q = exact_zero_q; w.have = have; w.path = path;
}

}  // namespace rda
#include "coop_ipm.cuh"
namespace rda {

// ---- stage 2: interior point (float64) for the cells the closed forms do not cover -------------
// Polygon obstacle: sigma_O(v) = max_i v.x_i, |v| <= 1 (ball).  Disc: sigma_O(v) = v.c + rad*tv with
// |v| <= tv <= 1 (cone constraint, extra variable tv), exact also when the robot overlaps the disc.
constexpr int CELL_NVA = 5, CELL_MCA = 2 * RDA_MAX_EDGE + 2;
constexpr int CELL_NVB = 8, CELL_MCB = 2 * RDA_MAX_EDGE + 3;
struct CellSlowStore {
  union U {
    CoopQP<CELL_NVA, CELL_MCA> a;
    CoopQP<CELL_NVB, CELL_MCB> b;
    RDA_HD U() {}
  } u;
  int need_a, ok, inactive, circ;
};

template <typename Real, typename Ctx>
RDA_HD void cell_slow(const RobotGeom& rb, CellWork<Real>& w, CellSlowStore& S, Ctx& ctx) {
  // Lane 0 owns `w` (the other lanes' copies are never read); all lanes run the solver loops.
  const int lane = ctx.lane();
  const int R = rb.R;
  if (lane == 0) {
    const CellGeom<Real>& g = w.g;
    const double x0 = w.xi0, x1 = w.xi1, k0d = (double)w.k0, c_ = w.cphi, s_ = w.sphi;
    // The max margin c* = min_{x in O, y in Rob} |P(y) - x| + xi.y - k0 is bounded above by its value
    // at any feasible pair: if that is negative the hinge is active for sure and stage A is skipped.
    bool need_a = true;
    if (w.sep) {
      double ub = sqrt((double)w.best) + x0 * (double)w.byx + x1 * (double)w.byy - k0d;
      if (ub < -1e-9) need_a = false;
    } else if (!w.circ) {
      double ub = 1e300;
      for (int j = 0; j < R; ++j)
        if (w.rob_in[j] <= 0) ub = rmin(ub, x0 * (double)rb.yx[j] + x1 * (double)rb.yy[j]);
      for (int i = 0; i < g.ne; ++i)
        if (w.obs_in[i] <= 0) {
          double wx = g.vx[i], wy = g.vy[i];
          ub = rmin(ub, x0 * (c_ * wx + s_ * wy) + x1 * (-s_ * wx + c_ * wy));
        }
      if (ub - k0d < -1e-9) need_a = false;
    }
    S.need_a = need_a ? 1 : 0;
    S.ok = 1; S.inactive = 0; S.circ = w.circ ? 1 : 0;
    if (need_a) {   // stage A: max margin with Hm + xi = 0; x = (v0, v1, so, sr, tv)
      CoopQP<CELL_NVA, CELL_MCA>& P = S.u.a;
      P.clear();
      P.c[2] = 1; P.c[3] = 1;
      const double radd = w.circ ? (double)g.rad : 0.0;
      const int nv_o = w.circ ? 1 : g.ne;
      for (int i = 0; i < nv_o; ++i) {
        double ox = w.circ ? (double)g.cx : (double)g.vx[i], oy = w.circ ? (double)g.cy : (double)g.vy[i];
        P.row(0, ox, 1, oy, 2, -1.0, 4, radd, 0.0);                      // v.x_i + rad tv <= so
      }
      double hmax = 0;
      for (int j = 0; j < R; ++j) {
        // g.y_j <= sr with g = -R'v - xi :  -(R y_j).v - sr <= xi.y_j
        double yx = rb.yx[j], yy = rb.yy[j];
        P.row(0, -(c_ * yx - s_ * yy), 1, -(s_ * yx + c_ * yy), 3, -1.0, 3, 0.0, x0 * yx + x1 * yy);
        hmax = rmax(hmax, fabs(x0 * yx + x1 * yy));
      }
      P.row(4, 1.0, 4, 0.0, 4, 0.0, 4, 0.0, 1.0);          // tv <= 1
      P.row(4, -1.0, 4, 0.0, 4, 0.0, 4, 0.0, 0.0);         // tv >= 0
      P.tv = w.circ ? 4 : -1;
      P.x[0] = 0; P.x[1] = 0; P.x[2] = 1.0 + radd; P.x[3] = 1.0 + hmax; P.x[4] = 0.5;
      for (int k = 0; k < CELL_NVA; ++k) P.x0[k] = P.x[k];
    }
  }
  ctx.sync();
  if (S.need_a) {
    CoopQP<CELL_NVA, CELL_MCA>& P = S.u.a;
    bool ok = !(S.circ != 0) && coop_ipm<CELL_NVA, CELL_MCA, Ctx>(P, ctx);
    if (!ok) {   // discs, and the rare polygon cell on which the primal-dual iteration cycles
      ctx.sync();
      if (lane == 0) for (int k = 0; k < CELL_NVA; ++k) P.x[k] = P.x0[k];
      ctx.sync();
      ok = coop_barrier<CELL_NVA, CELL_MCA, Ctx>(P, ctx);
    }
    ctx.sync();
    if (lane == 0) {
      S.ok = ok ? 1 : 0;
      double cst = -P.x[2] - P.x[3] - (double)w.k0;
      if (ok && cst >= 0) {
        S.inactive = 1;
        double va = P.x[0], vb = P.x[1];
        w.v0 = (Real)va; w.v1 = (Real)vb;
        w.g0 = (Real)(-((double)w.cphi * va + (double)w.sphi * vb) - (double)w.xi0);
        w.g1 = (Real)(-(-(double)w.sphi * va + (double)w.cphi * vb) - (double)w.xi1);
        w.exact_zero_q = true; w.have = true; w.path = CELL_SLOW_A;
      }
    }
    ctx.sync();
  }
  if (S.ok && !S.inactive) {   // stage B: x = (v0, v1, g0, g1, so, sr, w, tv)
    CoopQP<CELL_NVB, CELL_MCB>& P = S.u.b;
    if (lane == 0) {
      const CellGeom<Real>& g = w.g;
      const double x0 = w.xi0, x1 = w.xi1, k0d = (double)w.k0, c_ = w.cphi, s_ = w.sphi, r2 = w.ro2;
      P.clear();
      // ro2/2 |g + R'v + xi|^2 : with u = (v, g), q = M u + xi, M = [R' I]
      const double Mx[4] = {c_, s_, 1, 0}, My[4] = {-s_, c_, 0, 1};
      for (int k = 0; k < 4; ++k)
        for (int j = 0; j < 4; ++j) P.Q[k][j] = r2 * (Mx[k] * Mx[j] + My[k] * My[j]);
      for (int k = 0; k < 4; ++k) P.c[k] = r2 * (Mx[k] * x0 + My[k] * x1);
      P.Q[6][6] = 1.0;   // 1/2 w^2  (ro1 == 1 inside LamMuZ, rda_solver.py:257)
      const double radd = w.circ ? (double)g.rad : 0.0;
      const int nv_o = w.circ ? 1 : g.ne;
      for (int i = 0; i < nv_o; ++i) {
        double ox = w.circ ? (double)g.cx : (double)g.vx[i], oy = w.circ ? (double)g.cy : (double)g.vy[i];
        P.row(0, ox, 1, oy, 4, -1.0, 7, radd, 0.0);
      }
      for (int j = 0; j < R; ++j) P.row(2, (double)rb.yx[j], 3, (double)rb.yy[j], 5, -1.0, 5, 0.0, 0.0);
      P.row(4, 1.0, 5, 1.0, 6, -1.0, 6, 0.0, -k0d);        // so + sr + k0 <= w
      P.row(7, 1.0, 7, 0.0, 7, 0.0, 7, 0.0, 1.0);          // tv <= 1
      P.row(7, -1.0, 7, 0.0, 7, 0.0, 7, 0.0, 0.0);         // tv >= 0
      P.tv = w.circ ? 7 : -1;
      const double so0 = 1.0 + radd;
      const double xs[CELL_NVB] = {0, 0, 0, 0, so0, 1.0, rmax(so0 + 2.0 + k0d, 1.0), 0.5};
      for (int k = 0; k < CELL_NVB; ++k) { P.x[k] = xs[k]; P.x0[k] = xs[k]; }
    }
    ctx.sync();
    bool ok = !(S.circ != 0) && coop_ipm<CELL_NVB, CELL_MCB, Ctx>(P, ctx);
    if (!ok) {
      ctx.sync();
      if (lane == 0) for (int k = 0; k < CELL_NVB; ++k) P.x[k] = P.x0[k];
      ctx.sync();
      ok = coop_barrier<CELL_NVB, CELL_MCB, Ctx>(P, ctx);
    }
    ctx.sync();
    if (lane == 0) {
      S.ok = ok ? 1 : 0;
      if (ok) {
        w.v0 = (Real)P.x[0]; w.v1 = (Real)P.x[1]; w.g0 = (Real)P.x[2]; w.g1 = (Real)P.x[3];
        w.exact_zero_q = false; w.have = true; w.path = CELL_SLOW_B;
      }
    }
    ctx.sync();
  }
  if (lane == 0 && !S.ok) { w.have = false; w.path = CELL_FAILED; }
}

// ---- stage 3: multipliers, updates, su-QP inputs ----------------------------------------------
template <typename Real>
RDA_HD void cell_back(const RobotGeom& rb, const CellWork<Real>& w, Real zeta, Real theta, CellOut<Real>& out) {
  const CellGeom<Real>& g = w.g;
  const int R = rb.R, kind = g.kind;
  const Real v0 = w.v0, v1 = w.v1, g0 = w.g0, g1 = w.g1, cphi = w.cphi, sphi = w.sphi;
  const Real xi0 = w.xi0, xi1 = w.xi1, k0 = w.k0;
  for (int i = 0; i < RDA_MAX_EDGE; ++i) out.lam[i] = 0;
  for (int j = 0; j < RDA_MAX_ROBOT_EDGE; ++j) out.mu[j] = 0;
  out.path = w.path;
  if (!w.have) {
    // keep-previous-iterate rule (rda_solver.py:791-793) is applied by the caller
    out.z = 0; out.zeta_new = zeta; out.xi0_new = xi0; out.xi1_new = xi1;
    out.ax = out.ay = out.c0 = out.gx = out.gy = out.hm0 = out.hm1 = 0;
    return;
  }
  int io = 0, jr = 0;
  Real sO = support_obs<Real>(g, v0, v1, &io);
  Real sR = support_rob<Real>(rb, g0, g1, &jr);
  Real vn = sqrt_(v0 * v0 + v1 * v1);
  if (kind == RDA_OBS_CIRCLE) {
    out.lam[0] = v0; out.lam[1] = v1; out.lam[2] = -vn;          // (v, -|v|), mpc.py:440-458
  } else if (vn > 0) {
    obs_vertex_lam<Real>(g, io, v0, v1, out.lam);
  }
  Real gn = sqrt_(g0 * g0 + g1 * g1);
  if (gn > 0) {
    int a = (jr + R - 1) % R, bb = jr;
    Real nax = rb.nx[a], nay = rb.ny[a], nbx = rb.nx[bb], nby = rb.ny[bb];
    Real det = nax * nby - nay * nbx;
    Real al = (g0 * nby - g1 * nbx) / det;
    Real be = (nax * g1 - nay * g0) / det;
    out.mu[a] = rmax(al, (Real)0) / (Real)rb.gnorm[a];
    out.mu[bb] = rmax(be, (Real)0) / (Real)rb.gnorm[bb];
  }
  Real marg = -sO - sR;                 // lam'(A p - b) - mu'h
  Real stuff = marg - k0;
  Real z = theta * rmax(stuff, (Real)0);
  Real q0, q1;
  if (w.exact_zero_q) { q0 = 0; q1 = 0; }
  else {
    q0 = g0 + (cphi * v0 + sphi * v1) + xi0;
    q1 = g1 + (-sphi * v0 + cphi * v1) + xi1;
  }
  out.z = z;
  out.zeta_new = stuff - z;             // zeta + Im - d - z  (:666)
  out.xi0_new = q0;                     // xi + Hm            (:683)
  out.xi1_new = q1;
  out.hm0 = q0 - xi0;
  out.hm1 = q1 - xi1;
  out.ax = v0;
  out.ay = v1;
  out.c0 = marg - z + out.zeta_new;     // a.p - lam'b - mu'h - z + zeta   (Im_su without -d, :846-851)
  out.gx = g0 + q0;                     // mu'G + xi                       (:868)
  out.gy = g1 + q1;
}

// One cell, one thread (CPU port, tests): front -> slow (single lane) -> back.
template <typename Real>
RDA_HD void cell_solve(const RobotGeom& rb, int kind, int E, const float* A, const float* b,
                       Real px, Real py, Real cphi, Real sphi, Real dbar, Real zeta, Real xi0,
                       Real xi1, Real ro2, Real theta, CellOut<Real>& out) {
  CellWork<Real> w;
  cell_front<Real, true>(rb, kind, E, A, b, px, py, cphi, sphi, dbar, zeta, xi0, xi1, ro2, w);
  if (!w.have) {
    CellSlowStore S;
    SeqCtx ctx;
    cell_slow<Real, SeqCtx>(rb, w, S, ctx);
  }
  cell_back<Real>(rb, w, zeta, theta, out);
}

}  // namespace rda
