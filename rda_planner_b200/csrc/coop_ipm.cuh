// coop_ipm.cuh — warp-cooperative version of the small interior point solvers of cell_solver.cuh.
//
// One warp solves ONE small problem
//     min 1/2 x'Qx + c'x   s.t.  a_i'x <= b_i (i < m),  and the ball |x01| <= 1 (tv < 0) or the
//                               second-order cone |x01| <= x_tv (tv >= 0)
// with all data in shared memory: lane i owns row i (slack, multiplier, step), lane k owns
// component k of the vectors and lane e owns entry e of the Newton matrix.  The code is written
// against the same cooperative context as su_solver.cuh (lane(), nlanes(), sync(), sum/min/max),
// so that the g++ build (one lane) runs the identical arithmetic for the CPU tests.
#pragma once
#include "rda_hd.h"

namespace rda {

template <int NV, int MC>
struct CoopQP {
  double Q[NV][NV];
  double c[NV];
  double ad[MC][NV];          // dense rows
  double b[MC];
  int m, tv;
  double x[NV], x0[NV], s[MC + 1], l[MC + 1];
  // work space
  double rd[NV], ra[NV], rc[NV], rp[MC + 1], w[MC + 1], t1[MC + 1];
  double dsa[MC + 1], dla[MC + 1], ds[MC + 1], dl[MC + 1], rcs[MC + 1];
  double H[NV][NV], L[NV][NV];
  int flag;

  RDA_HD void clear() {
    for (int k = 0; k < NV; ++k) { c[k] = 0; for (int j = 0; j < NV; ++j) Q[k][j] = 0; }
    m = 0; tv = -1;
  }
  RDA_HD void row(int i0, double v0, int i1, double v1, int i2, double v2, int i3, double v3, double rhs) {
    for (int k = 0; k < NV; ++k) ad[m][k] = 0;
    ad[m][i0] += v0; ad[m][i1] += v1; ad[m][i2] += v2; ad[m][i3] += v3;
    b[m] = rhs; ++m;
  }
};

// Cholesky H = L L' (lower), cooperative; returns false (uniformly) on a non-positive pivot.
template <int NV, typename Ctx>
RDA_HD bool coop_chol(double H[NV][NV], double L[NV][NV], int* flag, Ctx& ctx) {
  const int lane = ctx.lane(), nl = ctx.nlanes();
  if (lane == 0) *flag = 1;
  ctx.sync();
  for (int j = 0; j < NV; ++j) {
    if (lane == 0) {
      double d = H[j][j];
      for (int k = 0; k < j; ++k) d -= L[j][k] * L[j][k];
      if (!(d > 0)) { *flag = 0; d = 1; }
      L[j][j] = sqrt(d);
    }
    ctx.sync();
    const double inv = 1.0 / L[j][j];
    for (int r = j + 1 + lane; r < NV; r += nl) {
      double sacc = H[r][j];
      for (int k = 0; k < j; ++k) sacc -= L[r][k] * L[j][k];
      L[r][j] = sacc * inv;
    }
    ctx.sync();
  }
  return *flag != 0;
}

// in-place solve L L' y = r by one lane
template <int NV>
RDA_HD void tri_solve(const double L[NV][NV], double* r) {
  for (int i = 0; i < NV; ++i) {
    double sacc = r[i];
    for (int k = 0; k < i; ++k) sacc -= L[i][k] * r[k];
    r[i] = sacc / L[i][i];
  }
  for (int i = NV - 1; i >= 0; --i) {
    double sacc = r[i];
    for (int k = i + 1; k < NV; ++k) sacc -= L[k][i] * r[k];
    r[i] = sacc / L[i][i];
  }
}

// Mehrotra predictor-corrector (same algorithm as tiny_ipm).  x must hold a strictly feasible
// start.  Returns true when converged (or acceptable at the rounding floor).
template <int NV, int MC, typename Ctx>
RDA_HD bool coop_ipm(CoopQP<NV, MC>& P, Ctx& ctx) {
  const int lane = ctx.lane(), nl = ctx.nlanes();
  const int m = P.m, M = m + 1, tv = P.tv;
  for (int i = lane; i < m; i += nl) {
    double ax = 0;
    for (int k = 0; k < NV; ++k) ax += P.ad[i][k] * P.x[k];
    double sv = rmax(P.b[i] - ax, 1e-3);
    P.s[i] = sv; P.l[i] = 1.0 / sv;
  }
  if (lane == 0) {
    double sv = rmax(-cone_eval(P.x, tv).f, 1e-3);
    P.s[m] = sv; P.l[m] = 1.0 / sv;
  }
  double scale = 1.0;
  for (int i = lane; i < m; i += nl) {
    scale = rmax(scale, fabs(P.b[i]));
    for (int k = 0; k < NV; ++k) scale = rmax(scale, fabs(P.ad[i][k]));
  }
  for (int k = lane; k < NV; k += nl) scale = rmax(scale, fabs(P.c[k]));
  scale = ctx.max(scale);
  ctx.sync();
  bool acceptable = false;
  for (int it = 0; it < 40; ++it) {
    const ConeEval ce = cone_eval(P.x, tv);
    const double lm = P.l[m], sm = P.s[m];
    // ---- residuals ----
    double rdn = 0, rpn = 0, mus = 0;
    for (int k = lane; k < NV; k += nl) {
      double v = P.c[k];
      for (int j = 0; j < NV; ++j) v += P.Q[k][j] * P.x[j];
      for (int i = 0; i < m; ++i) v += P.ad[i][k] * P.l[i];
      if (k == 0) v += ce.g0 * lm;
      if (k == 1) v += ce.g1 * lm;
      if (k == tv) v += ce.gt * lm;
      P.rd[k] = v;
      rdn = rmax(rdn, fabs(v));
    }
    for (int i = lane; i < M; i += nl) {
      double r;
      if (i < m) {
        double ax = 0;
        for (int k = 0; k < NV; ++k) ax += P.ad[i][k] * P.x[k];
        r = ax + P.s[i] - P.b[i];
      } else {
        r = ce.f + sm;
      }
      P.rp[i] = r;
      rpn = rmax(rpn, fabs(r));
      mus += P.s[i] * P.l[i];
      P.w[i] = P.l[i] / P.s[i];
      P.t1[i] = (P.l[i] * r - P.s[i] * P.l[i]) / P.s[i];       // affine: rc_i = s_i l_i
    }
    rdn = ctx.max(rdn); rpn = ctx.max(rpn);
    const double mu = ctx.sum(mus) / M;
    if (!(rdn == rdn) || !(mu == mu)) return false;
    acceptable = rdn < 1e-6 * scale && rpn < 1e-6 * scale && mu < 1e-7;
    if (rdn < 1e-9 * scale && rpn < 1e-9 * scale && mu < 1e-10) return true;
    if (mu < 1e-14) return acceptable;
    ctx.sync();
    // ---- Newton matrix (lower triangle) and affine right-hand side ----
    const double wm = P.w[m];
    for (int e = lane; e < NV * (NV + 1) / 2; e += nl) {
      int r = 0, rem = e;
      while (rem > r) { rem -= r + 1; ++r; }
      const int cidx = rem;               // r >= cidx
      double h = P.Q[r][cidx];
      for (int i = 0; i < m; ++i) h += P.w[i] * P.ad[i][r] * P.ad[i][cidx];
      const double gr = (r == 0 ? ce.g0 : r == 1 ? ce.g1 : r == tv ? ce.gt : 0.0);
      const double gc = (cidx == 0 ? ce.g0 : cidx == 1 ? ce.g1 : cidx == tv ? ce.gt : 0.0);
      h += wm * gr * gc;
      if (r == 0 && cidx == 0) h += lm * ce.h00;
      if (r == 1 && cidx == 1) h += lm * ce.h11;
      if (tv >= 0 && r == tv) {
        if (cidx == 0) h += lm * ce.h0t;
        if (cidx == 1) h += lm * ce.h1t;
        if (cidx == tv) h += lm * ce.htt;
      }
      if (r == cidx) h += 1e-12;
      P.H[r][cidx] = h;
    }
    for (int k = lane; k < NV; k += nl) {
      double v = -P.rd[k];
      for (int i = 0; i < m; ++i) v -= P.ad[i][k] * P.t1[i];
      const double gk = (k == 0 ? ce.g0 : k == 1 ? ce.g1 : k == tv ? ce.gt : 0.0);
      v -= gk * P.t1[m];
      P.ra[k] = v;
    }
    ctx.sync();
    if (!coop_chol<NV, Ctx>(P.H, P.L, &P.flag, ctx)) return acceptable;
    if (lane == 0) tri_solve<NV>(P.L, P.ra);
    ctx.sync();
    // ---- affine step: lengths and centring parameter ----
    double ratio = 0, sa0 = 0, sa1 = 0, sa2 = 0;
    for (int i = lane; i < M; i += nl) {
      double gd = 0;
      if (i < m) { for (int k = 0; k < NV; ++k) gd += P.ad[i][k] * P.ra[k]; }
      else gd = ce.g0 * P.ra[0] + ce.g1 * P.ra[1] + (tv >= 0 ? ce.gt * P.ra[tv] : 0.0);
      const double sv = P.s[i], lv = P.l[i];
      const double dsv = -P.rp[i] - gd;
      const double dlv = -(sv * lv + lv * dsv) / sv;
      P.dsa[i] = dsv; P.dla[i] = dlv;
      ratio = rmax(ratio, rmax(-dsv / sv, -dlv / lv));
      sa0 += sv * lv; sa1 += sv * dlv + lv * dsv; sa2 += dsv * dlv;
    }
    ratio = ctx.max(ratio);
    const double aaff = ratio > 1.0 ? 1.0 / ratio : 1.0;
    const double mua = (ctx.sum(sa0) + aaff * ctx.sum(sa1) + aaff * aaff * ctx.sum(sa2)) / M;
    double sig = mua / mu;
    sig = sig * sig * sig;
    ctx.sync();
    // ---- corrector ----
    for (int i = lane; i < M; i += nl) {
      const double rcv = P.s[i] * P.l[i] + P.dsa[i] * P.dla[i] - sig * mu;
      P.rcs[i] = rcv;
      P.t1[i] = (P.l[i] * P.rp[i] - rcv) / P.s[i];
    }
    ctx.sync();
    for (int k = lane; k < NV; k += nl) {
      double v = -P.rd[k];
      for (int i = 0; i < m; ++i) v -= P.ad[i][k] * P.t1[i];
      const double gk = (k == 0 ? ce.g0 : k == 1 ? ce.g1 : k == tv ? ce.gt : 0.0);
      v -= gk * P.t1[m];
      P.rc[k] = v;
    }
    ctx.sync();
    if (lane == 0) tri_solve<NV>(P.L, P.rc);
    ctx.sync();
    double ratio2 = 0;
    for (int i = lane; i < M; i += nl) {
      double gd = 0;
      if (i < m) { for (int k = 0; k < NV; ++k) gd += P.ad[i][k] * P.rc[k]; }
      else gd = ce.g0 * P.rc[0] + ce.g1 * P.rc[1] + (tv >= 0 ? ce.gt * P.rc[tv] : 0.0);
      const double sv = P.s[i], lv = P.l[i];
      const double dsv = -P.rp[i] - gd;
      const double dlv = -(P.rcs[i] + lv * dsv) / sv;
      P.ds[i] = dsv; P.dl[i] = dlv;
      ratio2 = rmax(ratio2, rmax(-dsv / sv, -dlv / lv));
    }
    ratio2 = ctx.max(ratio2);
    const double alpha = ratio2 > 0.995 ? 0.995 / ratio2 : 1.0;
    ctx.sync();
    for (int k = lane; k < NV; k += nl) P.x[k] += alpha * P.rc[k];
    for (int i = lane; i < M; i += nl) { P.s[i] += alpha * P.ds[i]; P.l[i] += alpha * P.dl[i]; }
    ctx.sync();
  }
  return acceptable;
}

// Feasible log-barrier method (same algorithm as tiny_barrier): damped Newton with backtracking.
template <int NV, int MC, typename Ctx>
RDA_HD double coop_barrier_value(const CoopQP<NV, MC>& P, const double* x, double t, Ctx& ctx) {
  const int lane = ctx.lane(), nl = ctx.nlanes();
  double f = 0;
  int bad = 0;
  for (int k = lane; k < NV; k += nl) {
    double qx = 0;
    for (int j = 0; j < NV; ++j) qx += P.Q[k][j] * x[j];
    f += t * x[k] * (0.5 * qx + P.c[k]);
  }
  for (int i = lane; i < P.m; i += nl) {
    double sl = P.b[i];
    for (int k = 0; k < NV; ++k) sl -= P.ad[i][k] * x[k];
    if (!(sl > 0)) bad = 1; else f -= log(sl);
  }
  if (lane == 0) {
    double tq = P.tv >= 0 ? x[P.tv] : 1.0;
    double psi = tq * tq - x[0] * x[0] - x[1] * x[1];
    if (!(psi > 0) || !(tq > 0)) bad = 1; else f -= log(psi);
  }
  f = ctx.sum(f);
  return ctx.max((double)bad) > 0 ? 1e300 : f;
}

// The barrier path t = 1, BARRIER_MU, BARRIER_MU^2, ... BARRIER_TMAX is followed, not traced: intermediate centres only to a
// Newton decrement of BARRIER_CENTER, the last one to 1e-9 (r02: MU 8 with every centre to 1e-9 needed 85 Newton steps per
// solve, MU 50 with 1e-2 needs 53, same results to the last digit of the float32 outputs).
constexpr double BARRIER_MU = 50.0, BARRIER_TMAX = 5.0e11, BARRIER_CENTER = 1e-2;

template <int NV, int MC, typename Ctx>
RDA_HD bool coop_barrier(CoopQP<NV, MC>& P, Ctx& ctx) {
  const int lane = ctx.lane(), nl = ctx.nlanes();
  const int m = P.m, tv = P.tv;
  double t = 1.0;
  for (int outer = 0; outer < 64; ++outer) {
    const bool last = t >= BARRIER_TMAX;
    for (int it = 0; it < 30; ++it) {
      // slack reciprocals
      for (int i = lane; i < m; i += nl) {
        double sl = P.b[i];
        for (int k = 0; k < NV; ++k) sl -= P.ad[i][k] * P.x[k];
        P.w[i] = 1.0 / sl;
      }
      ctx.sync();
      const double tq = tv >= 0 ? P.x[tv] : 1.0;
      const double psi = tq * tq - P.x[0] * P.x[0] - P.x[1] * P.x[1];
      const double ip = 1.0 / psi;
      const double gp0 = -2 * P.x[0], gp1 = -2 * P.x[1], gpt = 2 * tq;
      for (int k = lane; k < NV; k += nl) {
        double v = P.c[k];
        for (int j = 0; j < NV; ++j) v += P.Q[k][j] * P.x[j];
        v *= t;
        for (int i = 0; i < m; ++i) v += P.ad[i][k] * P.w[i];
        const double gk = (k == 0 ? gp0 : k == 1 ? gp1 : k == tv ? gpt : 0.0);
        v -= gk * ip;
        P.rd[k] = v;            // gradient
        P.ra[k] = -v;
      }
      for (int e = lane; e < NV * (NV + 1) / 2; e += nl) {
        int r = 0, rem = e;
        while (rem > r) { rem -= r + 1; ++r; }
        const int cidx = rem;
        double h = t * P.Q[r][cidx];
        for (int i = 0; i < m; ++i) h += P.w[i] * P.w[i] * P.ad[i][r] * P.ad[i][cidx];
        const double gr = (r == 0 ? gp0 : r == 1 ? gp1 : r == tv ? gpt : 0.0);
        const double gc = (cidx == 0 ? gp0 : cidx == 1 ? gp1 : cidx == tv ? gpt : 0.0);
        h += gr * gc * ip * ip;
        if (r == cidx) {
          if (r == 0 || r == 1) h += 2 * ip;
          if (tv >= 0 && r == tv) h -= 2 * ip;
          h += 1e-13 * (1.0 + h);
        }
        P.H[r][cidx] = h;
      }
      ctx.sync();
      if (!coop_chol<NV, Ctx>(P.H, P.L, &P.flag, ctx)) return false;
      if (lane == 0) tri_solve<NV>(P.L, P.ra);
      ctx.sync();
      double lam2 = 0;
      for (int k = lane; k < NV; k += nl) lam2 -= P.rd[k] * P.ra[k];
      lam2 = ctx.sum(lam2);
      if (!(lam2 == lam2)) return false;
      if (lam2 < (last ? 1e-9 : BARRIER_CENTER)) break;
      const double f0 = coop_barrier_value<NV, MC, Ctx>(P, P.x, t, ctx);
      double step = 1.0;
      bool moved = false;
      for (int bt = 0; bt < 50; ++bt, step *= 0.5) {
        for (int k = lane; k < NV; k += nl) P.rc[k] = P.x[k] + step * P.ra[k];
        ctx.sync();
        const double f1 = coop_barrier_value<NV, MC, Ctx>(P, P.rc, t, ctx);
        if (f1 <= f0 - 0.1 * step * lam2) { moved = true; break; }
        ctx.sync();
      }
      if (!moved) break;
      ctx.sync();
      for (int k = lane; k < NV; k += nl) P.x[k] = P.rc[k];
      ctx.sync();
    }
    if (last) break;
    t = rmin(t * BARRIER_MU, BARRIER_TMAX);
  }
  return true;
}

}  // namespace rda
