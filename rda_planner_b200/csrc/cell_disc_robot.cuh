// cell_disc_robot.cuh — the (obstacle, stage) cell of the LamMuZ problem for a DISC robot.
//
// Reference: car_tuple.cone_type == 'norm2' — cone_cp_array(-indep_mu, 'norm2'), rda_solver.py:1034-1039, used by
// LamMuZ_cost_cons :419 — with the ir-sim description of a circular body, G = [[1,0],[0,1],[0,0]], h = (cx, cy, -r):
// mu has three rows, -mu in the second-order cone means |mu[0:2]| <= -mu[2], G'mu = mu[0:2] =: g and
// mu'h = g.c - r mu[2] >= g.c + r|g|, so the body enters the cell problem of cell_solver.cuh through its support
// function sigma_Rob(g) = g.c + r|g| only:
//     min_{|v|<=1, g}  1/2 neg(stuff)^2 + ro2/2 |g + R'v + xi|^2,   stuff = v.p - sigma_O(v) - sigma_Rob(g) - d + zeta.
// Closed forms (one thread per cell, Real): the two cases that cover the inactive hinges (xi = 0 and a non-negative
// margin: closest point of the obstacle to the disc centre; overlap without tilt).  Everything else — active hinges,
// tilted cells — is a small second-order cone programme with TWO cones (|v| <= 1 or the obstacle disc's cone, and the
// body's |g| <= t_g), solved in float64 by the feasible log-barrier Newton method below.  Same tie-break as the polygon
// body (DESIGN.md §3): max margin, mu[2] = -|g| (the LP-vertex analogue: smallest mu'h), z = theta * max(stuff, 0).
#pragma once
#include "cell_solver.cuh"      // includes coop_ipm.cuh: coop_chol, tri_solve, the cooperative context interface

namespace rda {

// min 1/2 x'Qx + c'x  s.t.  a_i'x <= b_i (i < m)  and  |(x[ia_k] + sa_k, x[ib_k] + sb_k)| <= (it_k >= 0 ? x[it_k] : 1), k < nc
// Problem data and the work space of the barrier method in one block: shared memory when a warp solves the problem
// cooperatively (one lane per row / vector component / Newton-matrix entry, as coop_ipm.cuh), local memory when one
// thread does (SeqCtx: CPU port, tests).
template <int NV, int MC>
struct SocQP {
  double Q[NV][NV], c[NV], ad[MC][NV], b[MC];
  int m, nc;
  int ia[2], ib[2], it[2];
  double sa[2], sb[2];
  double x[NV];
  double H[NV][NV], L[NV][NV], gr[NV], dx[NV], xn[NV], w[MC];
  int flag;
  int newton;                  // Newton steps of the last soc_barrier call (statistics)
  RDA_HD void clear() {
    for (int k = 0; k < NV; ++k) { c[k] = 0; for (int j = 0; j < NV; ++j) Q[k][j] = 0; }
    m = 0; nc = 0;
  }
  RDA_HD int new_row(double rhs) {
    for (int k = 0; k < NV; ++k) ad[m][k] = 0;
    b[m] = rhs;
    return m++;
  }
  RDA_HD void cone(int a, int b_, int t, double sha, double shb) { ia[nc] = a; ib[nc] = b_; it[nc] = t; sa[nc] = sha; sb[nc] = shb; ++nc; }
};

// value of t*f0 + barrier at y (1e300 outside the domain); cooperative, the result is uniform over the lanes
template <int NV, int MC, typename Ctx>
RDA_HD double soc_value(const SocQP<NV, MC>& P, const double* y, double t, Ctx& ctx) {
  const int lane = ctx.lane(), nl = ctx.nlanes();
  double f = 0;
  int bad = 0;
  for (int k = lane; k < NV; k += nl) {
    double qx = 0;
    for (int j = 0; j < NV; ++j) qx += P.Q[k][j] * y[j];
    f += t * y[k] * (0.5 * qx + P.c[k]);
  }
  for (int i = lane; i < P.m; i += nl) {
    double sl = P.b[i];
    for (int k = 0; k < NV; ++k) sl -= P.ad[i][k] * y[k];
    if (!(sl > 0)) bad = 1; else f -= log(sl);
  }
  for (int k = lane; k < P.nc; k += nl) {
    const double u = y[P.ia[k]] + P.sa[k], w = y[P.ib[k]] + P.sb[k];
    const double tq = P.it[k] >= 0 ? y[P.it[k]] : 1.0;
    const double psi = tq * tq - u * u - w * w;
    if (!(psi > 0) || !(tq > 0)) bad = 1; else f -= log(psi);
  }
  f = ctx.sum(f);
  return ctx.max((double)bad) > 0 ? 1e300 : f;
}

// component r of grad(psi_k) / Hessian diagonal sign of cone k (0 when r is not one of its variables)
template <int NV, int MC>
RDA_HD double soc_cone_grad(const SocQP<NV, MC>& P, int k, int r, double u, double wv, double tq) {
  return r == P.ia[k] ? -2 * u : (r == P.ib[k] ? -2 * wv : (r == P.it[k] ? 2 * tq : 0.0));
}

// Feasible-start path following: damped Newton with backtracking on t*f0 + barrier, t = 1, MU, MU^2, ... up to TMAX
// (duality gap (m + 2 nc)/t ~ 3e-11 at the end); intermediate centres only to a Newton decrement of BARRIER_CENTER (the
// path is followed, not traced), the last one to 1e-9 — the path of coop_barrier (coop_ipm.cuh).  x must hold a strictly
// feasible point.  Measured on the committed disc-body cases (CPU): MU 8 / centre 1e-9 -> 85 Newton steps per solve,
// MU 50 / 1e-2 -> 53, identical results.
template <int NV, int MC, typename Ctx>
RDA_HD bool soc_barrier(SocQP<NV, MC>& P, Ctx& ctx) {
  const int lane = ctx.lane(), nl = ctx.nlanes();
  const int m = P.m;
  double t = 1.0;
  int newton = 0;
  for (int outer = 0; outer < 64; ++outer) {
    const bool last = t >= BARRIER_TMAX;
    for (int itn = 0; itn < 30; ++itn) {
      ++newton;
      for (int i = lane; i < m; i += nl) {
        double sl = P.b[i];
        for (int k = 0; k < NV; ++k) sl -= P.ad[i][k] * P.x[k];
        P.w[i] = 1.0 / sl;
      }
      ctx.sync();
      // the cones at the current point (every lane: two cones at most)
      double cu[2] = {0, 0}, cw[2] = {0, 0}, ct[2] = {1, 1}, cip[2] = {0, 0};
      for (int k = 0; k < P.nc; ++k) {
        cu[k] = P.x[P.ia[k]] + P.sa[k]; cw[k] = P.x[P.ib[k]] + P.sb[k];
        ct[k] = P.it[k] >= 0 ? P.x[P.it[k]] : 1.0;
        cip[k] = 1.0 / (ct[k] * ct[k] - cu[k] * cu[k] - cw[k] * cw[k]);
      }
      for (int k = lane; k < NV; k += nl) {
        double v = P.c[k];
        for (int j = 0; j < NV; ++j) v += P.Q[k][j] * P.x[j];
        v *= t;
        for (int i = 0; i < m; ++i) v += P.ad[i][k] * P.w[i];
        for (int q = 0; q < P.nc; ++q) v -= soc_cone_grad<NV, MC>(P, q, k, cu[q], cw[q], ct[q]) * cip[q];     // -grad(psi)/psi
        P.gr[k] = v;
        P.dx[k] = -v;
      }
      for (int e = lane; e < NV * (NV + 1) / 2; e += nl) {
        int r = 0, rem = e;
        while (rem > r) { rem -= r + 1; ++r; }
        const int cidx = rem;               // r >= cidx
        double h = t * P.Q[r][cidx];
        for (int i = 0; i < m; ++i) h += P.w[i] * P.w[i] * P.ad[i][r] * P.ad[i][cidx];
        for (int q = 0; q < P.nc; ++q) {
          // -log psi: Hessian grad grad'/psi^2 - hess(psi)/psi, hess(psi) = diag(-2, -2, +2) on (ia, ib, it)
          const double gr_ = soc_cone_grad<NV, MC>(P, q, r, cu[q], cw[q], ct[q]);
          const double gc_ = soc_cone_grad<NV, MC>(P, q, cidx, cu[q], cw[q], ct[q]);
          h += gr_ * gc_ * cip[q] * cip[q];
          if (r == cidx) {
            if (r == P.ia[q] || r == P.ib[q]) h += 2 * cip[q];
            else if (r == P.it[q]) h -= 2 * cip[q];
          }
        }
        if (r == cidx) h += 1e-13 * (1.0 + h);
        P.H[r][cidx] = h;
      }
      ctx.sync();
      if (!coop_chol<NV, Ctx>(P.H, P.L, &P.flag, ctx)) return false;
      if (lane == 0) tri_solve<NV>(P.L, P.dx);
      ctx.sync();
      double lam2 = 0;
      for (int k = lane; k < NV; k += nl) lam2 -= P.gr[k] * P.dx[k];
      lam2 = ctx.sum(lam2);
      if (!(lam2 == lam2)) return false;
      if (lam2 < (last ? 1e-9 : BARRIER_CENTER)) break;
      const double f0 = soc_value<NV, MC, Ctx>(P, P.x, t, ctx);
      double step = 1.0;
      bool moved = false;
      for (int bt = 0; bt < 50; ++bt, step *= 0.5) {
        for (int k = lane; k < NV; k += nl) P.xn[k] = P.x[k] + step * P.dx[k];
        ctx.sync();
        const double f1 = soc_value<NV, MC, Ctx>(P, P.xn, t, ctx);
        if (f1 <= f0 - 0.1 * step * lam2) { moved = true; break; }
        ctx.sync();
      }
      if (!moved) break;
      ctx.sync();
      for (int k = lane; k < NV; k += nl) P.x[k] = P.xn[k];
      ctx.sync();
    }
    if (last) break;
    t = rmin(t * BARRIER_MU, BARRIER_TMAX);
  }
  if (lane == 0) P.newton = newton;
  return true;
}

// ---- POINT contact of the disc body (float64): the obstacle point nearest to the optimal body point is a fixed point w --------
// (a polygon vertex, or the centre of a disc obstacle of radius rho_o).  World frame relative to the robot reference point:
// body disc of centre (cx, cy) and radius r, tilt xi' = R xi, numerator N(y) = k0 + rho_o - xi'.y - |y - w|, weight
// W^2 = 1 + |y|^2/ro2.  Stage 0 maximises N over the disc (concave, optimum on the rim), stage 1 maximises N/W where N > 0
// (quasi-concave: rim, or a stationary point inside the disc).  One-dimensional root search on the rim angle (Illinois) and
// a two-dimensional Newton iteration inside, all in float64 — the contact direction turns by r/|y - w| per radian, so float32
// cannot resolve the stationarity conditions of close contacts (the lesson of the polygon body's edge contacts, DESIGN §3.1).
// The caller accepts the point through the KKT conditions of the convex cell problem (direction inside the vertex' normal cone).
struct DiscContactD { double yx, yy, ux, uy, N, gam, tau; int rim; };
RDA_HD_NOINLINE bool disc_point_contact(int weighted, double cx, double cy, double r, double wx, double wy, double rho_o,
                                        double xix, double xiy, double k0, double ro2, DiscContactD& o) {
  double h = 0;
  auto eval = [&](double th) {
    const double ux_ = cos(th), uy_ = sin(th);
    o.yx = cx + r * ux_; o.yy = cy + r * uy_;
    const double dx = o.yx - wx, dy = o.yy - wy, L = sqrt(dx * dx + dy * dy);
    o.ux = dx / L; o.uy = dy / L;
    o.N = k0 + rho_o - (xix * o.yx + xiy * o.yy) - L;
    o.tau = weighted ? o.N / (1.0 + (o.yx * o.yx + o.yy * o.yy) / ro2) : 0.0;
    const double gx = -xix - o.ux - o.tau * o.yx / ro2, gy = -xiy - o.uy - o.tau * o.yy / ro2;
    h = -gx * uy_ + gy * ux_;            // tangential component of the gradient
    o.gam = gx * ux_ + gy * uy_;         // outward component: multiplier of the rim
  };
  const double th0 = atan2(wy - cy, wx - cx);
  double lo = th0 - 1.5, hi = th0 + 1.5;
  eval(lo); double flo = h; if (!(flo > 0) || (weighted && !(o.N > 0))) {
    // the region N > 0 may be a short arc around th0: shrink the bracket towards it
    bool found = false;
    for (int k = 0; k < 12 && !found; ++k) { lo = 0.5 * (lo + th0); eval(lo); flo = h; found = flo > 0 && (!weighted || o.N > 0); }
    if (!found) return false;
  }
  eval(hi); double fhi = h; if (!(fhi < 0) || (weighted && !(o.N > 0))) {
    bool found = false;
    for (int k = 0; k < 12 && !found; ++k) { hi = 0.5 * (hi + th0); eval(hi); fhi = h; found = fhi < 0 && (!weighted || o.N > 0); }
    if (!found) return false;
  }
  if (!(lo < hi)) return false;
  int side = 0;
  for (int itn = 0; itn < 80; ++itn) {
    const double wdt = hi - lo;
    double th = lo + wdt * (flo / (flo - fhi));
    th = rclamp(th, lo + 0.02 * wdt, hi - 0.02 * wdt);
    eval(th);
    if (weighted && !(o.N > 0)) return false;
    if (h > 0) { lo = th; flo = h; if (side > 0) fhi *= 0.5; side = 1; }
    else { hi = th; fhi = h; if (side < 0) flo *= 0.5; side = -1; }
    if (hi - lo < 1e-14 || h == 0) break;
  }
  o.rim = 1;
  if (o.gam >= -1e-10) return true;
  if (!weighted) return false;
  // the rim is not where N/W peaks: stationary point inside the disc, xi' + u + tau y/ro2 = 0 (2 x 2 Newton, damped)
  double yx = o.yx - 0.05 * r * cos(0.5 * (lo + hi)), yy = o.yy - 0.05 * r * sin(0.5 * (lo + hi));
  for (int itn = 0; itn < 50; ++itn) {
    const double dx = yx - wx, dy = yy - wy, L = sqrt(dx * dx + dy * dy);
    if (!(L > 1e-12)) return false;
    const double ux_ = dx / L, uy_ = dy / L;
    const double W2 = 1.0 + (yx * yx + yy * yy) / ro2;
    const double N = k0 + rho_o - (xix * yx + xiy * yy) - L;
    if (!(N > 0)) return false;
    const double tau = N / W2;
    const double G0 = xix + ux_ + tau * yx / ro2, G1 = xiy + uy_ + tau * yy / ro2;
    // grad tau = grad N / W2 - 2 N y / (ro2 W2^2)
    const double tx = (-xix - ux_) / W2 - 2.0 * N * yx / (ro2 * W2 * W2), ty = (-xiy - uy_) / W2 - 2.0 * N * yy / (ro2 * W2 * W2);
    const double J00 = (1.0 - ux_ * ux_) / L + tau / ro2 + yx * tx / ro2, J01 = -ux_ * uy_ / L + yx * ty / ro2;
    const double J10 = -ux_ * uy_ / L + yy * tx / ro2, J11 = (1.0 - uy_ * uy_) / L + tau / ro2 + yy * ty / ro2;
    const double det = J00 * J11 - J01 * J10;
    if (!(fabs(det) > 1e-300)) return false;
    double sx = -(J11 * G0 - J01 * G1) / det, sy = -(-J10 * G0 + J00 * G1) / det;
    // damping: stay inside the disc and move at most half way to the point w
    double a = 1.0;
    for (int bt = 0; bt < 30; ++bt, a *= 0.5) {
      const double nx_ = yx + a * sx, ny_ = yy + a * sy;
      if ((nx_ - cx) * (nx_ - cx) + (ny_ - cy) * (ny_ - cy) < r * r && (nx_ - wx) * (nx_ - wx) + (ny_ - wy) * (ny_ - wy) > 0.25 * L * L) break;
    }
    yx += a * sx; yy += a * sy;
    o.yx = yx; o.yy = yy; o.ux = ux_; o.uy = uy_; o.N = N; o.tau = tau; o.gam = 0; o.rim = 0;
    if (sqrt(G0 * G0 + G1 * G1) < 1e-12 && a == 1.0) {
      // re-evaluate at the final point
      const double ex = yx - wx, ey = yy - wy, L2 = sqrt(ex * ex + ey * ey);
      o.ux = ex / L2; o.uy = ey / L2;
      o.N = k0 + rho_o - (xix * yx + xiy * yy) - L2;
      o.tau = o.N / (1.0 + (yx * yx + yy * yy) / ro2);
      return o.N > 0;
    }
  }
  return false;
}

constexpr int DR_NVA = 5, DR_NVB = 8, DR_MC = RDA_MAX_EDGE + 3;
struct DiscSlowStore {
  union U {
    SocQP<DR_NVA, DR_MC> a;
    SocQP<DR_NVB, DR_MC> b;
    RDA_HD U() {}
  } u;
  int need_a, ok, inactive, bad;      // control flow shared by the lanes of a cooperative solve
};

// ---- stage 1: geometry relative to the robot reference point and the closed forms of the inactive hinge ----------
// Fills w.g (obstacle part), w.k0 ..., w.best (squared distance from the DISC CENTRE to the obstacle, 0 inside),
// w.byx / w.byy (unit direction obstacle -> centre, world frame) and, when a closed form applies, the solution.
template <typename Real>
RDA_HD void cell_front_dr(const RobotGeom& rb, int kind, int E, const float* A, const float* b, Real px, Real py,
                          Real cphi, Real sphi, Real dbar, Real zeta, Real xi0, Real xi1, Real ro2, CellWork<Real>& w,
                          bool searched_forms = true) {
  const Real k0 = dbar - zeta;
  const Real eps = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
  CellGeom<Real>& g = w.g;
  w.k0 = k0; w.cphi = cphi; w.sphi = sphi; w.xi0 = xi0; w.xi1 = xi1; w.ro2 = ro2;
  w.circ = (kind == RDA_OBS_CIRCLE);
  g.kind = kind;
  const Real rr = rb.rad;
  const Real cwx = cphi * (Real)rb.cx - sphi * (Real)rb.cy, cwy = sphi * (Real)rb.cx + cphi * (Real)rb.cy;   // R c
  Real dc = 0, dirx = 0, diry = 0;     // distance of the disc centre to the obstacle (0 inside), direction obstacle -> centre
  bool sep;
  if (kind == RDA_OBS_CIRCLE) {
    g.cx = (Real)b[0] - px; g.cy = (Real)b[1] - py; g.rad = -(Real)b[2]; g.ne = 0;
    const Real dx = cwx - g.cx, dy = cwy - g.cy;
    const Real dn = sqrt_(dx * dx + dy * dy);
    dc = rmax(dn - g.rad, (Real)0);
    if (dn > eps) { dirx = dx / dn; diry = dy / dn; }
    sep = dn > g.rad + rr + eps;
  } else {
    int ne = 0;
    Real brel[RDA_MAX_EDGE];
    for (int i = 0; i < E; ++i) {
      const Real ax = A[2 * i], ay = A[2 * i + 1];
      const Real n2 = ax * ax + ay * ay;
      if (!(n2 > 0)) break;
      const Real inv = rsqrt_(n2);
      g.nx[i] = ax * inv; g.ny[i] = ay * inv; g.inv_norm[i] = inv;
      brel[i] = ((Real)b[i] - ax * px - ay * py) * inv;
      ne = i + 1;
    }
    g.ne = ne;
    for (int i = 0; i < ne; ++i) {
      const int a = (i + ne - 1) % ne;
      const Real det = g.nx[a] * g.ny[i] - g.ny[a] * g.nx[i];
      const Real inv = (Real)1 / det;
      g.vx[i] = (brel[a] * g.ny[i] - brel[i] * g.ny[a]) * inv;
      g.vy[i] = (g.nx[a] * brel[i] - g.nx[i] * brel[a]) * inv;
    }
    bool inside = true;
    Real best = 1e30f, bdx = 0, bdy = 0;
    for (int i = 0; i < ne; ++i) {
      const int in = (i + 1) % ne;
      const Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
      const Real rx = cwx - g.vx[i], ry = cwy - g.vy[i];
      if (g.nx[i] * rx + g.ny[i] * ry > 0) inside = false;
      const Real t = rclamp((rx * ex + ry * ey) / (ex * ex + ey * ey), (Real)0, (Real)1);
      const Real dx = rx - t * ex, dy = ry - t * ey;
      const Real d2 = dx * dx + dy * dy;
      if (d2 < best) { best = d2; bdx = dx; bdy = dy; }
    }
    if (ne == 0) { inside = false; best = 1e30f; }
    const Real dn = sqrt_(best);
    dc = inside ? (Real)0 : dn;
    if (!inside && dn > eps) { dirx = bdx / dn; diry = bdy / dn; }
    sep = !inside && dn > rr + eps;
  }
  w.sep = sep; w.best = dc * dc; w.byx = dirx; w.byy = diry;
  Real v0 = 0, v1 = 0, g0 = 0, g1 = 0;
  bool exact_zero_q = false, have = false;
  int path = CELL_FAILED;
  const bool xi_zero = (xi0 == (Real)0) && (xi1 == (Real)0);
  w.xi_zero = xi_zero;
  if (sep && xi_zero && dc - rr - k0 >= 0) {
    // disjoint, no tilt, non-negative margin: unit normal of the closest pair (it lies on the line through the centre)
    v0 = dirx; v1 = diry;
    g0 = -(cphi * v0 + sphi * v1);
    g1 = -(-sphi * v0 + cphi * v1);
    exact_zero_q = true; have = true; path = CELL_FAST_INACTIVE;
  } else if (!sep && xi_zero && k0 <= 0) {
    // overlapping sets, no tilt: max margin 0 at v = 0 (stuff = -k0 >= 0)
    exact_zero_q = true; have = true; path = CELL_OVERLAP_FREE;
  }
  if (searched_forms && !have && sep && kind != RDA_OBS_CIRCLE) {
    // EDGE contact: the obstacle point nearest to the optimal body point y lies in the interior of obstacle edge i.  There the
    // distance is the signed distance to the edge line, e_i(y) = n_i.(R y) - brel_i, LINEAR in y, so the numerator of the
    // (weighted) margin is N_i(y) = alpha - beta.y with alpha = k0 + brel_i, beta = xi + R'n_i (body frame).  Since
    // dist(P(y), O) >= e_i(y) everywhere, N_true <= N_i pointwise with equality where the feature holds: a maximiser of the
    // edge problem whose foot lies inside the edge is the maximiser of the cell problem (tilted cells included).
    //   max margin (stage A): max of N_i over the disc at y = c - r beta/|beta|; -N >= 0 there => inactive, v = n_i, g = -beta;
    //   active hinge (N > 0), body centred on the reference point (c = 0): N_i/W with W^2 = 1 + |y|^2/ro2 peaks at
    //   y = -t beta/|beta|, t = min(r, ro2 |beta|/alpha) (t = r when alpha <= 0): inside the disc g = 0, on its rim g = -(|beta| - tau r/ro2) beta/|beta|.
    const Real tolc = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
    const Real bcx = rb.cx, bcy = rb.cy;
    const bool centred = bcx == (Real)0 && bcy == (Real)0;
    const int ne = g.ne;
    for (int i = 0; i < ne && !have; ++i) {
      const int in = (i + 1) % ne;
      const Real nix = g.nx[i], niy = g.ny[i];
      const Real bx_ = xi0 + (cphi * nix + sphi * niy), by_ = xi1 + (-sphi * nix + cphi * niy);      // beta = xi + R'n_i
      const Real bn = sqrt_(bx_ * bx_ + by_ * by_);
      if (!(bn > tolc)) continue;
      const Real alpha = k0 - (nix * (-g.vx[i]) + niy * (-g.vy[i]));      // k0 + brel_i, brel_i = n_i.V_i (relative to p)
      const Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
      const Real ie2 = (Real)1 / (ex * ex + ey * ey);
      for (int stage = 0; stage < 2 && !have; ++stage) {
        Real yx, yy;
        if (stage == 0) { yx = bcx - rr * bx_ / bn; yy = bcy - rr * by_ / bn; }
        else {
          if (!centred) break;
          // f(t) = (alpha + t |beta|)/sqrt(1 + t^2/ro2) along y = -t beta/|beta|: increasing for every t when alpha <= 0
          const Real t = alpha > 0 ? rmin(rr, ro2 * bn / alpha) : rr;
          yx = -t * bx_ / bn; yy = -t * by_ / bn;
        }
        const Real wx = cphi * yx - sphi * yy, wy = sphi * yx + cphi * yy;          // R y
        const Real ed = nix * (wx - g.vx[i]) + niy * (wy - g.vy[i]);                  // distance of P(y) to the edge line
        const Real so_ = ((wx - g.vx[i]) * ex + (wy - g.vy[i]) * ey) * ie2;          // foot along the edge
        if (!(ed > eps && so_ > tolc && so_ < (Real)1 - tolc)) continue;
        const Real Nv = alpha - (bx_ * yx + by_ * yy);
        if (stage == 0) {
          if (Nv <= 0) {
            v0 = nix; v1 = niy; g0 = -bx_; g1 = -by_;
            exact_zero_q = true; have = true; path = CELL_FAST_VERTEX;
          }
        } else if (Nv > 0) {
          const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
          v0 = nix; v1 = niy;
          g0 = -tau * yx / ro2 - bx_; g1 = -tau * yy / ro2 - by_;
          // interior of the disc: g vanishes up to rounding (stationary point); make it exact
          if (alpha > 0 && ro2 * bn / alpha < rr) { g0 = 0; g1 = 0; }
          have = true; path = CELL_FAST_VERTEX;
        }
      }
    }
  }
  if (searched_forms && !have && sep) {
    // POINT contacts (float64, disc_point_contact): each obstacle vertex whose normal cone can hold the contact direction,
    // or the centre of a disc obstacle
    const double c_ = cphi, s_ = sphi;
    const double cwxd = c_ * (double)rb.cx - s_ * (double)rb.cy, cwyd = s_ * (double)rb.cx + c_ * (double)rb.cy;
    const double xwx = c_ * (double)xi0 - s_ * (double)xi1, xwy = s_ * (double)xi0 + c_ * (double)xi1;      // R xi
    const int npt = kind == RDA_OBS_CIRCLE ? 1 : g.ne;
    for (int stage = 0; stage < 2 && !have; ++stage) {
      for (int i = 0; i < npt && !have; ++i) {
        const double wxd = kind == RDA_OBS_CIRCLE ? (double)g.cx : (double)g.vx[i], wyd = kind == RDA_OBS_CIRCLE ? (double)g.cy : (double)g.vy[i];
        const double rho_o = kind == RDA_OBS_CIRCLE ? (double)g.rad : 0.0;
        DiscContactD o;
        if (!disc_point_contact(stage, cwxd, cwyd, (double)rr, wxd, wyd, rho_o, xwx, xwy, (double)k0, (double)ro2, o)) continue;
        if (kind != RDA_OBS_CIRCLE) {
          // the nearest obstacle point is vertex i only while the direction lies strictly inside its normal cone
          const int ne = g.ne, ip = (i + ne - 1) % ne, inx = (i + 1) % ne;
          const double epx = (double)g.vx[i] - (double)g.vx[ip], epy = (double)g.vy[i] - (double)g.vy[ip];
          const double enx = (double)g.vx[inx] - (double)g.vx[i], eny = (double)g.vy[inx] - (double)g.vy[i];
          if (!(o.ux * epx + o.uy * epy >= 1e-7 * sqrt(epx * epx + epy * epy) && o.ux * enx + o.uy * eny <= -1e-7 * sqrt(enx * enx + eny * eny)))
            continue;
        }
        if (stage == 0) {
          if (o.N <= 0) {      // max margin -N >= 0: inactive, Hm + xi = 0
            v0 = (Real)o.ux; v1 = (Real)o.uy;
            g0 = (Real)(-(c_ * o.ux + s_ * o.uy) - (double)xi0);
            g1 = (Real)(-(-s_ * o.ux + c_ * o.uy) - (double)xi1);
            exact_zero_q = true; have = true; path = CELL_FAST_VERTEX;
          }
        } else if (o.N > 0) {
          v0 = (Real)o.ux; v1 = (Real)o.uy;
          if (o.rim) {
            // g = gamma * (outward unit normal of the rim at y), body frame
            const double nxw = (o.yx - cwxd) / (double)rr, nyw = (o.yy - cwyd) / (double)rr;
            g0 = (Real)(o.gam * (c_ * nxw + s_ * nyw)); g1 = (Real)(o.gam * (-s_ * nxw + c_ * nyw));
          } else { g0 = 0; g1 = 0; }
          exact_zero_q = false; have = true; path = CELL_FAST_VERTEX;
        }
      }
    }
  }
  if (searched_forms && !have && !sep) {
    // OVERLAPPING sets: the contact distance is zero, the numerator of the weighted margin is k0 - xi.y and the optimum sits
    // (ii) at a body point whose image lies strictly inside the obstacle (v = 0), (iii) on an obstacle edge strictly inside the
    // body (g = 0), (iv) at an obstacle vertex strictly inside the body, or (v) where the body's rim crosses an obstacle edge —
    // the disc body's versions of cell_front's overlap cases, each accepted through the KKT conditions of the cell problem.
    const Real tolc = sizeof(Real) == 4 ? (Real)1e-5 : (Real)1e-11;
    const Real bcx = rb.cx, bcy = rb.cy;
    const bool centred = bcx == (Real)0 && bcy == (Real)0;
    const int ne = g.ne;
    auto inside_obstacle = [&](Real wx, Real wy) {
      if (kind == RDA_OBS_CIRCLE) {
        const Real ex = wx - g.cx, ey = wy - g.cy;
        return g.rad > eps && ex * ex + ey * ey < (g.rad - eps) * (g.rad - eps);
      }
      for (int i = 0; i < ne; ++i)
        if (g.nx[i] * (wx - g.vx[i]) + g.ny[i] * (wy - g.vy[i]) > -eps) return false;
      return ne >= 3;
    };
    // (ii) v = 0: maximise (k0 - xi.y)/W over the disc
    {
      const Real xn = sqrt_(xi0 * xi0 + xi1 * xi1);
      Real yx = 0, yy = 0;
      bool cand = false, interior = true;
      if (centred) {
        const Real t = xn > 0 ? (k0 > 0 ? rmin(rr, ro2 * xn / k0) : rr) : (Real)0;
        if (xn > 0) { yx = -t * xi0 / xn; yy = -t * xi1 / xn; }
        interior = !(xn > 0) || (k0 > 0 && ro2 * xn / k0 < rr);
        cand = true;
      } else if (k0 > 0) {
        yx = -ro2 * xi0 / k0; yy = -ro2 * xi1 / k0;      // stationary point; only valid strictly inside the disc
        cand = (yx - bcx) * (yx - bcx) + (yy - bcy) * (yy - bcy) < (rr - eps) * (rr - eps);
      }
      if (cand) {
        const Real Nv = k0 - (xi0 * yx + xi1 * yy);
        if (Nv > 0 && inside_obstacle(cphi * yx - sphi * yy, sphi * yx + cphi * yy)) {
          const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
          v0 = 0; v1 = 0;
          if (interior) { g0 = 0; g1 = 0; } else { g0 = -tau * yx / ro2 - xi0; g1 = -tau * yy / ro2 - xi1; }
          exact_zero_q = false; have = true; path = CELL_OVERLAP_FREE;
        }
      }
    }
    if (kind != RDA_OBS_CIRCLE) {
      // (iii) P(y) on obstacle edge i, y strictly inside the body: g = 0, v = a n_i, 0 <= a <= 1 (closed-form stationary point
      //       of (k0 - xi.y)/W on the edge line, as cell_front's case iii)
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
        if (!((yx - bcx) * (yx - bcx) + (yy - bcy) * (yy - bcy) < (rr - eps) * (rr - eps))) continue;
        const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
        const Real rx = -tau * yx / ro2 - xi0, ry = -tau * yy / ro2 - xi1;      // must equal R'v
        const Real nbx = cphi * g.nx[i] + sphi * g.ny[i], nby = -sphi * g.nx[i] + cphi * g.ny[i];
        const Real alpha = rx * nbx + ry * nby;
        if (!(alpha >= -tolc && alpha <= (Real)1 + tolc)) continue;
        const Real ac = rclamp(alpha, (Real)0, (Real)1);
        v0 = ac * g.nx[i]; v1 = ac * g.ny[i]; g0 = 0; g1 = 0;
        exact_zero_q = false; have = true; path = CELL_OVERLAP_FREE;
      }
      // (iv) obstacle vertex i strictly inside the body: y = R'V_i, g = 0, v = R(-tau y/ro2 - xi) in the vertex' normal cone, |v| <= 1
      for (int i = 0; i < ne && !have; ++i) {
        const Real yx = cphi * g.vx[i] + sphi * g.vy[i], yy = -sphi * g.vx[i] + cphi * g.vy[i];
        if (!((yx - bcx) * (yx - bcx) + (yy - bcy) * (yy - bcy) < (rr - eps) * (rr - eps))) continue;
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
        exact_zero_q = false; have = true; path = CELL_OVERLAP_FREE;
      }
      // (v) the body's rim crosses obstacle edge i: y fixed, g = gamma u (u: outward unit normal of the rim at y, body frame),
      //     v = a n_i with gamma u + a R'n_i = -tau y/ro2 - xi (2 x 2), gamma >= 0, 0 <= a <= 1
      const Real cwx_ = cphi * bcx - sphi * bcy, cwy_ = sphi * bcx + cphi * bcy;      // R c
      for (int i = 0; i < ne && !have; ++i) {
        const int in = (i + 1) % ne;
        const Real ex = g.vx[in] - g.vx[i], ey = g.vy[in] - g.vy[i];
        const Real fx = g.vx[i] - cwx_, fy = g.vy[i] - cwy_;
        const Real qa = ex * ex + ey * ey, qb = (Real)2 * (fx * ex + fy * ey), qc = fx * fx + fy * fy - rr * rr;
        const Real disc = qb * qb - (Real)4 * qa * qc;
        if (!(disc > 0)) continue;
        const Real sq = sqrt_(disc);
        for (int root = 0; root < 2 && !have; ++root) {
          const Real so_ = (-qb + (root ? sq : -sq)) / ((Real)2 * qa);
          if (!(so_ > tolc && so_ < (Real)1 - tolc)) continue;
          const Real wx = g.vx[i] + so_ * ex, wy = g.vy[i] + so_ * ey;               // crossing point, world
          const Real yx = cphi * wx + sphi * wy, yy = -sphi * wx + cphi * wy;
          const Real Nv = k0 - (xi0 * yx + xi1 * yy);
          if (!(Nv > 0)) continue;
          const Real tau = Nv / ((Real)1 + (yx * yx + yy * yy) / ro2);
          const Real rx = -tau * yx / ro2 - xi0, ry = -tau * yy / ro2 - xi1;
          const Real ux_ = (yx - bcx) / rr, uy_ = (yy - bcy) / rr;
          const Real nbx = cphi * g.nx[i] + sphi * g.ny[i], nby = -sphi * g.nx[i] + cphi * g.ny[i];
          const Real d2 = ux_ * nby - uy_ * nbx;
          if (!(abs_(d2) > (Real)1e-9)) continue;
          const Real gam = (rx * nby - ry * nbx) / d2;
          const Real alp = (ux_ * ry - uy_ * rx) / d2;
          if (!(gam >= -tolc && alp >= -tolc && alp <= (Real)1 + tolc)) continue;
          const Real ac = rclamp(alp, (Real)0, (Real)1), gc = rmax(gam, (Real)0);
          v0 = ac * g.nx[i]; v1 = ac * g.ny[i]; g0 = gc * ux_; g1 = gc * uy_;
          exact_zero_q = false; have = true; path = CELL_OVERLAP_FREE;
        }
      }
    }
  }
  w.v0 = v0; w.v1 = v1; w.g0 = g0; w.g1 = g1;
  w.exact_zero_q = exact_zero_q; w.have = have; w.path = path;
}

// ---- stage 2: the two-cone programmes (float64) ---------------------------------------------------------------------
// Lane 0 owns `w` and sets the problems up; all lanes of the context run the barrier iterations (cell_slow's pattern).
template <typename Real, typename Ctx>
RDA_HD void cell_slow_dr(const RobotGeom& rb, CellWork<Real>& w, DiscSlowStore& S, Ctx& ctx) {
  const int lane = ctx.lane();
  const double rr = rb.rad, bcx = rb.cx, bcy = rb.cy;
  if (lane == 0) {
    const CellGeom<Real>& g = w.g;
    const double x0 = w.xi0, x1 = w.xi1, k0d = (double)w.k0, c_ = w.cphi, s_ = w.sphi;
    const double cwx = c_ * bcx - s_ * bcy, cwy = s_ * bcx + c_ * bcy;          // R c
    const double ax_ = c_ * x0 - s_ * x1, ay_ = s_ * x0 + c_ * x1;                // R xi
    const bool circ = w.circ;
    const double radd = circ ? (double)g.rad : 0.0;
    const int nv_o = circ ? 1 : g.ne;
    S.bad = (!circ && g.ne < 3) ? 1 : 0;
    // upper bound of the max margin from the closest pair: negative => the hinge is active for sure, stage A skipped
    bool need_a = true;
    if (w.sep) {
      const double dirx = w.byx, diry = w.byy;
      // body point of the closest pair, body frame: c - r R'dir
      const double ybx = bcx - rr * (c_ * dirx + s_ * diry), yby = bcy - rr * (-s_ * dirx + c_ * diry);
      const double ub = (sqrt((double)w.best) - rr) + x0 * ybx + x1 * yby - k0d;
      if (ub < -1e-9) need_a = false;
    }
    S.need_a = need_a ? 1 : 0; S.ok = 1; S.inactive = 0;
    if (need_a && !S.bad) {   // stage A: max margin with Hm + xi = 0 (g = -R'v - xi);  x = (v0, v1, so, tg, tv)
      SocQP<DR_NVA, DR_MC>& P = S.u.a;
      P.clear();
      P.c[0] = -cwx; P.c[1] = -cwy; P.c[2] = 1; P.c[3] = rr;     // so + sigma_Rob(g) + xi.c = so + r tg - v.(R c)
      for (int i = 0; i < nv_o; ++i) {
        const int r = P.new_row(0.0);                            // v.x_i + rad tv <= so
        P.ad[r][0] = circ ? (double)g.cx : (double)g.vx[i];
        P.ad[r][1] = circ ? (double)g.cy : (double)g.vy[i];
        P.ad[r][2] = -1.0; P.ad[r][4] = radd;
      }
      { const int r = P.new_row(1.0); P.ad[r][4] = 1.0; }        // tv <= 1
      { const int r = P.new_row(0.0); P.ad[r][4] = -1.0; }       // tv >= 0
      P.cone(0, 1, circ ? 4 : -1, 0.0, 0.0);                     // |v| <= 1  /  |v| <= tv
      P.cone(0, 1, 3, ax_, ay_);                                 // |g| = |v + R xi| <= tg
      P.x[0] = 0; P.x[1] = 0; P.x[2] = 1.0 + radd; P.x[3] = sqrt(ax_ * ax_ + ay_ * ay_) + 1.0; P.x[4] = 0.5;
    }
  }
  ctx.sync();
  if (S.bad) { if (lane == 0) { w.have = false; w.path = CELL_FAILED; } return; }
  if (S.need_a) {
    const bool ok = soc_barrier<DR_NVA, DR_MC, Ctx>(S.u.a, ctx);
    ctx.sync();
    if (lane == 0) {
      S.ok = ok ? 1 : 0;
      if (ok) {
        const CellGeom<Real>& g = w.g;
        const SocQP<DR_NVA, DR_MC>& P = S.u.a;
        const double x0 = w.xi0, x1 = w.xi1, c_ = w.cphi, s_ = w.sphi;
        const double cwx = c_ * bcx - s_ * bcy, cwy = s_ * bcx + c_ * bcy, ax_ = c_ * x0 - s_ * x1, ay_ = s_ * x0 + c_ * x1;
        const double va = P.x[0], vb = P.x[1];
        const double gn = sqrt((va + ax_) * (va + ax_) + (vb + ay_) * (vb + ay_));
        // margin at the barrier's v with the supports evaluated exactly (so, tg carry the barrier's 1/t slack)
        double so = w.circ ? va * (double)g.cx + vb * (double)g.cy + (double)g.rad * sqrt(va * va + vb * vb) : -1e300;
        if (!w.circ) for (int i = 0; i < g.ne; ++i) so = rmax(so, va * (double)g.vx[i] + vb * (double)g.vy[i]);
        const double cst = -(so + rr * gn - (va * cwx + vb * cwy) - (x0 * bcx + x1 * bcy)) - (double)w.k0;
        if (cst >= 0) {
          S.inactive = 1;
          w.v0 = (Real)va; w.v1 = (Real)vb;
          w.g0 = (Real)(-(c_ * va + s_ * vb) - x0);
          w.g1 = (Real)(-(-s_ * va + c_ * vb) - x1);
          w.exact_zero_q = true; w.have = true; w.path = CELL_SLOW_A;
        }
      }
    }
    ctx.sync();
  }
  if (S.ok && !S.inactive) {   // stage B: active hinge;  x = (v0, v1, g0, g1, so, tg, w, tv)
    SocQP<DR_NVB, DR_MC>& P = S.u.b;
    if (lane == 0) {
      const CellGeom<Real>& g = w.g;
      const double x0 = w.xi0, x1 = w.xi1, k0d = (double)w.k0, c_ = w.cphi, s_ = w.sphi, r2 = w.ro2;
      const bool circ = w.circ;
      const double radd = circ ? (double)g.rad : 0.0;
      const int nv_o = circ ? 1 : g.ne;
      P.clear();
      const double Mx[4] = {c_, s_, 1, 0}, My[4] = {-s_, c_, 0, 1};      // q = M (v, g) + xi, M = [R' I]
      for (int k = 0; k < 4; ++k)
        for (int j = 0; j < 4; ++j) P.Q[k][j] = r2 * (Mx[k] * Mx[j] + My[k] * My[j]);
      for (int k = 0; k < 4; ++k) P.c[k] = r2 * (Mx[k] * x0 + My[k] * x1);
      P.Q[6][6] = 1.0;                                                    // 1/2 w^2 (ro1 == 1 inside LamMuZ, rda_solver.py:257)
      for (int i = 0; i < nv_o; ++i) {
        const int r = P.new_row(0.0);
        P.ad[r][0] = circ ? (double)g.cx : (double)g.vx[i];
        P.ad[r][1] = circ ? (double)g.cy : (double)g.vy[i];
        P.ad[r][4] = -1.0; P.ad[r][7] = radd;
      }
      { const int r = P.new_row(-k0d); P.ad[r][4] = 1.0; P.ad[r][2] = bcx; P.ad[r][3] = bcy; P.ad[r][5] = rr; P.ad[r][6] = -1.0; }   // so + sigma_Rob + k0 <= w
      { const int r = P.new_row(1.0); P.ad[r][7] = 1.0; }
      { const int r = P.new_row(0.0); P.ad[r][7] = -1.0; }
      P.cone(0, 1, circ ? 7 : -1, 0.0, 0.0);
      P.cone(2, 3, 5, 0.0, 0.0);                                          // |g| <= tg
      const double so0 = 1.0 + radd;
      const double xs[DR_NVB] = {0, 0, 0, 0, so0, 1.0, rmax(so0 + rr + k0d + 2.0, 1.0), 0.5};
      for (int k = 0; k < DR_NVB; ++k) P.x[k] = xs[k];
    }
    ctx.sync();
    const bool ok = soc_barrier<DR_NVB, DR_MC, Ctx>(P, ctx);
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

// ---- stage 3: multipliers, updates, su-QP inputs (cell_back with the disc body's mu and support function) --------
template <typename Real>
RDA_HD void cell_back_dr(const RobotGeom& rb, const CellWork<Real>& w, Real zeta, Real theta, CellOut<Real>& out) {
  const CellGeom<Real>& g = w.g;
  const int ne = g.ne, kind = g.kind;
  const Real v0 = w.v0, v1 = w.v1, g0 = w.g0, g1 = w.g1, cphi = w.cphi, sphi = w.sphi;
  const Real xi0 = w.xi0, xi1 = w.xi1, k0 = w.k0;
  for (int i = 0; i < RDA_MAX_EDGE; ++i) out.lam[i] = 0;
  for (int j = 0; j < RDA_MAX_ROBOT_EDGE; ++j) out.mu[j] = 0;
  out.path = w.path;
  if (!w.have) {
    out.z = 0; out.zeta_new = zeta; out.xi0_new = xi0; out.xi1_new = xi1;
    out.ax = out.ay = out.c0 = out.gx = out.gy = out.hm0 = out.hm1 = 0;
    return;
  }
  int io = 0;
  const Real sO = support_obs<Real>(g, v0, v1, &io);
  const Real vn = sqrt_(v0 * v0 + v1 * v1);
  if (kind == RDA_OBS_CIRCLE) {
    out.lam[0] = v0; out.lam[1] = v1; out.lam[2] = -vn;
  } else if (vn > 0) {
    const int a = (io + ne - 1) % ne, bb = io;
    const Real det = g.nx[a] * g.ny[bb] - g.ny[a] * g.nx[bb];
    const Real al = (v0 * g.ny[bb] - v1 * g.nx[bb]) / det;
    const Real be = (g.nx[a] * v1 - g.ny[a] * v0) / det;
    out.lam[a] = rmax(al, (Real)0) * g.inv_norm[a];
    out.lam[bb] = rmax(be, (Real)0) * g.inv_norm[bb];
  }
  const Real gn = sqrt_(g0 * g0 + g1 * g1);
  out.mu[0] = g0; out.mu[1] = g1; out.mu[2] = -gn;                       // (g, -|g|): smallest mu'h in the cone
  const Real sR = g0 * (Real)rb.cx + g1 * (Real)rb.cy + (Real)rb.rad * gn;
  const Real marg = -sO - sR;
  const Real stuff = marg - k0;
  const Real z = theta * rmax(stuff, (Real)0);
  Real q0, q1;
  if (w.exact_zero_q) { q0 = 0; q1 = 0; }
  else {
    q0 = g0 + (cphi * v0 + sphi * v1) + xi0;
    q1 = g1 + (-sphi * v0 + cphi * v1) + xi1;
  }
  out.z = z;
  out.zeta_new = stuff - z;
  out.xi0_new = q0; out.xi1_new = q1;
  out.hm0 = q0 - xi0; out.hm1 = q1 - xi1;
  out.ax = v0; out.ay = v1;
  out.c0 = marg - z + out.zeta_new;
  out.gx = g0 + q0; out.gy = g1 + q1;
}

// One cell, one thread (CPU port, tests).
template <typename Real>
RDA_HD void cell_solve_dr(const RobotGeom& rb, int kind, int E, const float* A, const float* b, Real px, Real py,
                          Real cphi, Real sphi, Real dbar, Real zeta, Real xi0, Real xi1, Real ro2, Real theta,
                          CellOut<Real>& out, bool searched_forms = true) {
  CellWork<Real> w;
  cell_front_dr<Real>(rb, kind, E, A, b, px, py, cphi, sphi, dbar, zeta, xi0, xi1, ro2, w, searched_forms);
  if (!w.have) {
    DiscSlowStore S;
    SeqCtx ctx;
    cell_slow_dr<Real, SeqCtx>(rb, w, S, ctx);
  }
  cell_back_dr<Real>(rb, w, zeta, theta, out);
}

}  // namespace rda
