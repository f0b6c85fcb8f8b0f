// su_solver.cuh — the state/control "su" QP of one planning instance.
//
// Replaces rda_solver.py: su_prob_solve :692-700 (cvxpy -> ECOS) for the problem defined by
// construct_su_prob :216-231, nav_cost_cons :313-328, update_su_cost_cons :330-387,
// Im_su :831-851, Hm_su :853-872, dynamics_constraint :911-928, bound_su_constraints :930-938,
// bound_dis_constraints :940-947, C0_cost :1011-1029, C1_cost :1031-1032, and the
// re-linearisation assign_state_parameter :436-460 / linear_*_model :949-994.
//
// Method (DESIGN.md §4): Mehrotra predictor-corrector primal-dual interior point method.
//  * decision variables (u_t, d_t); states follow the linearised dynamics exactly, so every Newton
//    step is an equality-constrained LQ problem solved by a Riccati recursion over the horizon
//    with state (s_t, u_{t-1}) in R^5 and control (u_t, d_t) in R^3 (the banded KKT system);
//  * inequality constraints: |u| <= max_speed, |u_t - u_{t-1}| <= max_acce*dt, min_sd <= d <= max_sd;
//  * every hinge term ro1/2 neg(Im)^2 is the exact partial minimum over a slack w of
//    ro1/2 w^2 s.t. Im + w >= 0; w is eliminated analytically (w = nu/ro1), leaving one
//    (slack, multiplier) pair per hinge and a rank-one term in the stage Hessian.
// The code is written against a "cooperative group" context Ctx (lane(), nlanes(), sync(),
// min/sum reductions): one warp per instance on the GPU (lanes = horizon stages), one lane on the
// host (tests/host_shim).
#pragma once
#include "rda_hd.h"

namespace rda {

#ifndef RDA_SU_CH
#define RDA_SU_CH 2      // hinges per chunk of the su-QP hinge loops (loads grouped ahead of the arithmetic)
#endif

struct SuParams {
  int T, N, dynamics, accelerated;
  float dt, L, umax[2], ab[2], ws, wu;
  float slack_gain, dmin, dmax, ro1, ro2;
  int max_iter;
  float mu0;      // initial complementarity of the interior point iteration
  float prune;    // > 0: hinges whose value at the nominal point exceeds it even for d = max_sd are left out of
                  // the interior point iteration and verified afterwards (accelerated mode only); 0: keep all
};

// Per-instance workspace.  All arrays indexed by stage t (0..T-1) unless noted; hinge arrays indexed
// [o*T + t].  Real: arithmetic, iterate and slack / multiplier type.
template <typename Real>
struct SuWork {
  Real *s, *u, *d;            // iterate: 3(T+1), 2T, T
  float *ref;                 // 3(T+1)   (inputs stay in the float32 they arrive in)
  float *lins, *linu;         // linearisation point 3(T+1), 2T; linu is dead after the setup (shares dv)
  Real *Aj, *Bj, *Cj;         // 2T (A02, A12), 6T, 3T; Cj is dead after the initial rollout (shares K)
  Real *Skk, *Sgk;            // aggregated rotation-consensus terms
  float *pref;                // 2T positions the hinge offsets refer to
  float *hx, *hy, *hc;        // hinge rows: lam'A (2) and offset
  Real *hs, *hnu;             // hinge slack / multiplier
  unsigned *hmask;            // T x ceil(N/32) words: hinges of stage t that take part in the interior point iteration
  Real *bs, *bnu;             // 10T box/rate slack / multiplier, entry (t, c) at 10 * t + c
  Real *Wm;                   // 3T hinge Hessian of the position block after the elimination of d_t (xx, xy, yy)
  Real *Ed;                   // 3T elimination of d_t: (M_xd / Q_dd, M_yd / Q_dd, 1 / Q_dd)
  Real *g5q;                  // T   reduced-out gradient of d_t: g_d / Q_dd (d step = -(g5q + Ed . dp))
  Real *gw;                   // 8T gradient in stage coordinates: right-hand side of a backward sweep
  Real *wb;                   // 5T barrier weights (u0, u1, d, rate0, rate1)
  Real *K, *Lc, *kf;          // 10T, 3T, 2T Riccati gains / L D L' of Hvv / feed-forward (controls u_t; d_t eliminated)
  Real *dz, *dv;              // 5(T+1), 3T Newton step.  Shares the storage of gw: the corrector's forward
                              // sweep writes it after the backward sweep has consumed gw, and it is dead
                              // (iterate updated) before the next predictor assembles gw.
  Real *dza, *dva;            // affine (predictor) step.  Shares the storage of (Wm, wb): those are
                              // consumed by the factorising backward sweep of the predictor, the affine
                              // step is produced by the forward sweep that follows it and is dead before
                              // the next predictor assembles (Wm, wb) again.
  Real vref;
  int restarts;               // out: 1 when the pruned solve failed its verification and was repeated with all hinges
};

// Workspace placement.  `base` is the fast memory of the instance (shared memory on the GPU), `gbase` an
// optional per-instance slab of global memory (L2).  Everything lives in `base`, except that with
// hinge_arrays = false the per-hinge arrays (hx, hy, hc: caller; hs, hnu: `gbase`) are left out of it (each
// entry is touched only by the lane that owns its stage).  Returns the bytes of `base` used; *gbytes the
// bytes of `gbase`.
template <typename Real>
RDA_HD size_t su_work_layout(int T, int N, SuWork<Real>* w, char* base, bool hinge_arrays = true,
                             char* gbase = nullptr, size_t* gbytes = nullptr) {
  size_t offs = 0, offg = 0;
  auto takes = [&](size_t n, size_t elt) {
    offs = (offs + 15) & ~(size_t)15;
    char* p = base ? base + offs : nullptr;
    offs += n * elt;
    return p;
  };
  auto takeg = [&](size_t n, size_t elt) {
    offg = (offg + 15) & ~(size_t)15;
    char* p = gbase ? gbase + offg : nullptr;
    offg += n * elt;
    return p;
  };
#define RDA_TAKE_S(field, n, type) { char* p_ = takes((size_t)(n), sizeof(type)); if (w) w->field = (type*)p_; }
#define RDA_TAKE_G(field, n, type) { char* p_ = takeg((size_t)(n), sizeof(type)); if (w) w->field = (type*)p_; }
  RDA_TAKE_S(s, 3 * (T + 1), Real) RDA_TAKE_S(u, 2 * T, Real) RDA_TAKE_S(d, T, Real)
  RDA_TAKE_S(ref, 3 * (T + 1), float) RDA_TAKE_S(lins, 3 * (T + 1), float)
  RDA_TAKE_S(Aj, 2 * T, Real) RDA_TAKE_S(Bj, 6 * T, Real)
  RDA_TAKE_S(Skk, T, Real) RDA_TAKE_S(Sgk, T, Real) RDA_TAKE_S(pref, 2 * T, float)
  RDA_TAKE_S(hmask, T * ((N + 31) / 32 > 0 ? (N + 31) / 32 : 1), unsigned)
  if (hinge_arrays) {
    RDA_TAKE_S(hx, N * T, float) RDA_TAKE_S(hy, N * T, float) RDA_TAKE_S(hc, N * T, float)
    RDA_TAKE_S(hs, N * T, Real) RDA_TAKE_S(hnu, N * T, Real)
  } else {
    RDA_TAKE_G(hs, N * T, Real) RDA_TAKE_G(hnu, N * T, Real)
  }
  RDA_TAKE_S(bs, 10 * T, Real) RDA_TAKE_S(bnu, 10 * T, Real)
  RDA_TAKE_S(Wm, 8 * T + 5, Real)                                     // (Wm, wb) | (dza, dva)
  if (w) { w->wb = w->Wm + 3 * T; w->dza = w->Wm; w->dva = w->Wm + 5 * (T + 1); }
  RDA_TAKE_S(Ed, 3 * T, Real) RDA_TAKE_S(g5q, T, Real)
  RDA_TAKE_S(gw, 8 * T + 5, Real)                                     // gw | (dz, dv)
  if (w) { w->dz = w->gw; w->dv = w->gw + 5 * (T + 1); }
  RDA_TAKE_S(K, 10 * T, Real) RDA_TAKE_S(Lc, 3 * T, Real) RDA_TAKE_S(kf, 2 * T, Real)
  if (w) { w->Cj = w->K; w->linu = (float*)w->dv; }
#undef RDA_TAKE_S
#undef RDA_TAKE_G
  if (gbytes) *gbytes = (offg + 15) & ~(size_t)15;
  return (offs + 15) & ~(size_t)15;
}

// size-only query of su_work_layout
template <typename Real>
RDA_HD size_t su_work_bytes(int T, int N, bool hinge_arrays = true, size_t* gbytes = nullptr) {
  return su_work_layout<Real>(T, N, (SuWork<Real>*)nullptr, nullptr, hinge_arrays, nullptr, gbytes);
}

// Jacobians of the discrete model about (s, u): linear_ackermann_model :949-963,
// linear_diff_model :966-979, linear_omni_model :982-994.
template <typename Real>
RDA_HD void su_linearise(const SuParams& P, const Real* st, const Real* ut, Real* Aj, Real* Bj, Real* Cj) {
  const Real dt = P.dt;
  if (P.dynamics == RDA_DYN_OMNI) {
    Real phi = ut[1], v = ut[0];
    Real c = cos(phi), s = sin(phi);
    Aj[0] = 0; Aj[1] = 0;
    Bj[0] = c * dt; Bj[1] = -v * s * dt; Bj[2] = s * dt; Bj[3] = v * c * dt; Bj[4] = 0; Bj[5] = 0;
    Cj[0] = phi * v * s * dt; Cj[1] = -phi * v * c * dt; Cj[2] = 0;
    return;
  }
  Real phi = st[2], v = ut[0];
  Real c = cos(phi), s = sin(phi);
  Aj[0] = -v * dt * s; Aj[1] = v * dt * c;
  Bj[0] = c * dt; Bj[1] = 0; Bj[2] = s * dt; Bj[3] = 0;
  Cj[0] = phi * v * s * dt; Cj[1] = -phi * v * c * dt;
  if (P.dynamics == RDA_DYN_ACKER) {
    Real psi = ut[1];
    Real cp = cos(psi);
    Real k = v * dt / ((Real)P.L * cp * cp);
    Bj[4] = tan(psi) * dt / (Real)P.L; Bj[5] = k;
    Cj[2] = -psi * k;
  } else {
    Bj[4] = 0; Bj[5] = dt;
    Cj[2] = 0;
  }
}

// One inequality row of stage t.  c in 0..9: (u0 hi, u0 lo, u1 hi, u1 lo, d hi, d lo,
// rate0 hi, rate0 lo, rate1 hi, rate1 lo).  value g >= 0, gradient = sgn on component `comp`
// (3: u0, 4: u1, 5: d) and -sgn on the previous control for rate rows.
template <typename Real>
struct Row { Real g; Real sgn; int comp; bool rate; bool live; };

template <typename Real>
RDA_HD Row<Real> su_row(const SuParams& P, const SuWork<Real>& W, int t, int c) {
  Row<Real> r;
  r.rate = c >= 6;
  r.live = true;
  const bool hi = (c & 1) == 0;
  r.sgn = hi ? (Real)-1 : (Real)1;
  if (c < 4) {
    int k = c >> 1;
    r.comp = 3 + k;
    Real uv = W.u[2 * t + k], m = P.umax[k];
    r.g = hi ? m - uv : uv + m;
  } else if (c < 6) {
    r.comp = 5;
    Real dv = W.d[t];
    Real lo = P.dmin > 0 ? P.dmin : 0;
    r.g = hi ? (Real)P.dmax - dv : dv - lo;
    r.live = P.N > 0;
  } else {
    int k = (c - 6) >> 1;
    r.comp = 3 + k;
    r.live = t >= 1;
    Real du = r.live ? W.u[2 * t + k] - W.u[2 * (t - 1) + k] : (Real)0;
    r.g = hi ? (Real)P.ab[k] - du : (Real)P.ab[k] + du;
  }
  return r;
}

// directional derivative of row (t, c) along the Newton step held in (dz, dv)
template <typename Real>
RDA_HD Real su_row_dir(const Row<Real>& r, const Real* dz_t, const Real* dv_t) {
  Real x = dv_t[r.comp - 3];
  if (r.rate) x -= dz_t[3 + (r.comp - 3)];
  return r.sgn * x;
}

template <typename Real, typename Ctx>
RDA_HD void su_riccati(const SuParams& P, SuWork<Real>& W, Ctx& ctx, bool factor, Real* dz, Real* dv) {
  // Riccati recursion of the Newton step (banded KKT system).  Stage t: state z = (s_t, u_{t-1}),
  // control v = u_t.  The safety distance d_t appears in stage t only (hinges and its own bounds), so
  // it has been eliminated from the stage cost by the assembly (Schur complement on Q_dd: W.Wm holds
  // the reduced position block, W.gw[0..1] the reduced gradient) and is recovered after the forward
  // sweep from W.Ed / W.g5q.  The stage cost is quadratic in q = (s_{t+1}, u_t) = J [z; v] with
  // J = [[A 0 B], [0 0 I]] plus the rate-limit coupling between u_t and u_{t-1}; the sparsity of J is
  // written out by hand.  Every lane runs the same recursion (no broadcast needed); lane 0 stores the
  // gains.
  const int T = P.T;
  const Real reg = (Real)1e-9;
  const Real tw = 2 * (Real)P.ws, tw3 = (P.dynamics == RDA_DYN_OMNI ? (Real)0 : tw);
  Real Pm[5][5], pv[5];
  for (int a = 0; a < 5; ++a) { pv[a] = 0; for (int b = 0; b < 5; ++b) Pm[a][b] = 0; }
  const bool writer = ctx.lane() == 0;
  for (int t = T - 1; t >= 0; --t) {
    const Real a02 = W.Aj[2 * t], a12 = W.Aj[2 * t + 1];
    const Real* Bt = W.Bj + 6 * t;
    const Real b00 = Bt[0], b01 = Bt[1], b10 = Bt[2], b11 = Bt[3], b20 = Bt[4], b21 = Bt[5];
    // gradient in q-space (+ cost-to-go), pulled back through J
    const Real* gw = W.gw + 8 * t;
    const Real q0 = gw[0] + pv[0], q1 = gw[1] + pv[1], q2 = gw[2] + pv[2], q3 = gw[3] + pv[3], q4 = gw[4] + pv[4];
    const Real gz0 = q0, gz1 = q1, gz2 = a02 * q0 + a12 * q1 + q2, gz3 = gw[6], gz4 = gw[7];
    const Real gv0 = b00 * q0 + b10 * q1 + b20 * q2 + q3;
    const Real gv1 = b01 * q0 + b11 * q1 + b21 * q2 + q4;
    Real i00, L10, i11;   // L D L' of Hvv: unit-lower entry and reciprocal pivots
    Real Kt[2][5];
    if (factor) {
      const Real* wb = W.wb + 5 * t;
      const Real wr0 = wb[3], wr1 = wb[4];
      Real Q[5][5];
      for (int a = 0; a < 5; ++a) for (int b = 0; b < 5; ++b) Q[a][b] = Pm[a][b];
      const Real* M = W.Wm + 3 * t;
      Q[0][0] += tw + M[0]; Q[0][1] += M[1]; Q[1][0] += M[1]; Q[1][1] += tw + M[2];
      Q[2][2] += tw3 + (Real)P.ro2 * W.Skk[t];
      Q[3][3] += 2 * (Real)P.wu + reg + wb[0] + wr0;
      Q[4][4] += reg + wb[1] + wr1;
      // T1 = Q J for the columns of J that are not unit vectors
      Real t2[5], t5[5], t6[5];
      for (int r = 0; r < 5; ++r) {
        t2[r] = a02 * Q[r][0] + a12 * Q[r][1] + Q[r][2];
        t5[r] = b00 * Q[r][0] + b10 * Q[r][1] + b20 * Q[r][2] + Q[r][3];
        t6[r] = b01 * Q[r][0] + b11 * Q[r][1] + b21 * Q[r][2] + Q[r][4];
      }
#define RDA_J2(x) (a02 * (x)[0] + a12 * (x)[1] + (x)[2])
#define RDA_J5(x) (b00 * (x)[0] + b10 * (x)[1] + b20 * (x)[2] + (x)[3])
#define RDA_J6(x) (b01 * (x)[0] + b11 * (x)[1] + b21 * (x)[2] + (x)[4])
      // Hzz (rows/cols 0..2 dense, 3..4 only the rate terms)
      Real Hzz[5][5];
      for (int a = 0; a < 5; ++a) for (int b = 0; b < 5; ++b) Hzz[a][b] = 0;
      Hzz[0][0] = Q[0][0]; Hzz[0][1] = Q[0][1]; Hzz[1][1] = Q[1][1];
      Hzz[0][2] = t2[0]; Hzz[1][2] = t2[1]; Hzz[2][2] = RDA_J2(t2);
      Hzz[1][0] = Hzz[0][1]; Hzz[2][0] = Hzz[0][2]; Hzz[2][1] = Hzz[1][2];
      Hzz[3][3] = wr0; Hzz[4][4] = wr1;
      // Hvz (2 x 5)
      Real Hvz[2][5];
      Hvz[0][0] = t5[0]; Hvz[0][1] = t5[1]; Hvz[0][2] = RDA_J2(t5); Hvz[0][3] = -wr0; Hvz[0][4] = 0;
      Hvz[1][0] = t6[0]; Hvz[1][1] = t6[1]; Hvz[1][2] = RDA_J2(t6); Hvz[1][3] = 0; Hvz[1][4] = -wr1;
      // Hvv (2 x 2)
      const Real h00 = RDA_J5(t5), h10 = RDA_J6(t5), h11 = RDA_J6(t6);
#undef RDA_J2
#undef RDA_J5
#undef RDA_J6
      // Hvv = L D L' (unit lower L: L10; reciprocal pivots i00, i11) — no square roots
      i00 = rcp_(h00);
      L10 = h10 * i00;
      i11 = rcp_(h11 - L10 * h10);
      for (int b = 0; b < 5; ++b) {
        Real y0 = -Hvz[0][b];
        Real y1 = -Hvz[1][b] - L10 * y0;
        Real x1 = y1 * i11;
        Real x0 = y0 * i00 - L10 * x1;
        Kt[0][b] = x0; Kt[1][b] = x1;
      }
      for (int a = 0; a < 5; ++a)
        for (int b = a; b < 5; ++b) {
          Real v = Hzz[a][b] + Hvz[0][a] * Kt[0][b] + Hvz[1][a] * Kt[1][b];
          Pm[a][b] = v; Pm[b][a] = v;
        }
      if (writer) {
        Real* Ls = W.Lc + 3 * t;
        Ls[0] = i00; Ls[1] = L10; Ls[2] = i11;
        for (int k = 0; k < 2; ++k) for (int b = 0; b < 5; ++b) W.K[10 * t + 5 * k + b] = Kt[k][b];
      }
    } else {
      const Real* Ls = W.Lc + 3 * t;
      i00 = Ls[0]; L10 = Ls[1]; i11 = Ls[2];
      for (int k = 0; k < 2; ++k) for (int b = 0; b < 5; ++b) Kt[k][b] = W.K[10 * t + 5 * k + b];
    }
    {
      Real y0 = -gv0;
      Real y1 = -gv1 - L10 * y0;
      Real x1 = y1 * i11;
      Real x0 = y0 * i00 - L10 * x1;
      if (writer) { W.kf[2 * t] = x0; W.kf[2 * t + 1] = x1; }
      pv[0] = gz0 + Kt[0][0] * gv0 + Kt[1][0] * gv1;
      pv[1] = gz1 + Kt[0][1] * gv0 + Kt[1][1] * gv1;
      pv[2] = gz2 + Kt[0][2] * gv0 + Kt[1][2] * gv1;
      pv[3] = gz3 + Kt[0][3] * gv0 + Kt[1][3] * gv1;
      pv[4] = gz4 + Kt[0][4] * gv0 + Kt[1][4] * gv1;
    }
  }
  ctx.sync();
  // forward sweep
  Real z[5] = {0, 0, 0, 0, 0};
  for (int t = 0; t < T; ++t) {
    Real v[2];
    for (int k = 0; k < 2; ++k) {
      Real sacc = W.kf[2 * t + k];
      for (int b = 0; b < 5; ++b) sacc += W.K[10 * t + 5 * k + b] * z[b];
      v[k] = sacc;
    }
    if (writer) {
      for (int a = 0; a < 5; ++a) dz[5 * t + a] = z[a];
      dv[3 * t] = v[0]; dv[3 * t + 1] = v[1];
    }
    Real n0 = z[0] + W.Aj[2 * t] * z[2] + W.Bj[6 * t] * v[0] + W.Bj[6 * t + 1] * v[1];
    Real n1 = z[1] + W.Aj[2 * t + 1] * z[2] + W.Bj[6 * t + 2] * v[0] + W.Bj[6 * t + 3] * v[1];
    Real n2 = z[2] + W.Bj[6 * t + 4] * v[0] + W.Bj[6 * t + 5] * v[1];
    z[0] = n0; z[1] = n1; z[2] = n2; z[3] = v[0]; z[4] = v[1];
  }
  if (writer) for (int a = 0; a < 5; ++a) dz[5 * T + a] = z[a];
  ctx.sync();
  // recover the step of the eliminated safety distances (each lane its own stages)
  for (int t = ctx.lane(); t < T; t += ctx.nlanes())
    dv[3 * t + 2] = P.N > 0 ? -(W.g5q[t] + W.Ed[3 * t] * dz[5 * t + 5] + W.Ed[3 * t + 1] * dz[5 * t + 6]) : (Real)0;
}

// Solve the su-QP.  Inputs already staged in W: lins, linu, ref, vref, hx/hy/hc, pref, Skk/Sgk
// are computed here from (gx, gy) planes passed as pointers (global or shared memory, [o*T+t]).
// On entry W.d holds para_dis (initial guess of d).  Returns 0 (converged), 1 (iteration cap),
// 2 (non-finite).  On return W.s, W.u, W.d hold the solution.
template <typename Real, typename Ctx>
RDA_HD int su_solve(const SuParams& P, SuWork<Real>& W, Ctx& ctx, const float* gx, const float* gy,
                    int* iters_out) {
  const int T = P.T, N = P.N;
  const int lane = ctx.lane(), nl = ctx.nlanes();
  const Real ro1 = P.ro1, ro2 = P.ro2;
  const Real iro1 = (Real)1 / ro1;
  const bool acc = P.accelerated != 0;
  // ---- linearisation and aggregated rotation terms (lane-parallel over stages) ----
  for (int t = lane; t < T; t += nl) {
    const Real st[3] = {(Real)W.lins[3 * t], (Real)W.lins[3 * t + 1], (Real)W.lins[3 * t + 2]};
    const Real ut[2] = {(Real)W.linu[2 * t], (Real)W.linu[2 * t + 1]};
    su_linearise<Real>(P, st, ut, W.Aj + 2 * t, W.Bj + 6 * t, W.Cj + 3 * t);
    Real phib = st[2];
    Real c = cos(phib), s = sin(phib);
    Real skk = 0, sgk = 0;
    for (int o = 0; o < N; ++o) {
      Real ax = W.hx[o * T + t], ay = W.hy[o * T + t];
      Real k0 = -ax * s + ay * c, k1 = -ax * c - ay * s;          // a R'
      Real g0 = (Real)gx[o * T + t] + ax * c + ay * s;            // mu'G + xi + a R
      Real g1 = (Real)gy[o * T + t] - ax * s + ay * c;
      skk += k0 * k0 + k1 * k1;
      sgk += g0 * k0 + g1 * k1;
    }
    W.Skk[t] = skk; W.Sgk[t] = sgk;
    W.u[2 * t] = ut[0]; W.u[2 * t + 1] = ut[1];
  }
  ctx.sync();
  // Hinge pruning (accelerated mode).  A hinge 1/2 ro1 neg(l)^2 that is inactive at the minimiser changes neither the
  // cost nor its gradient there, so the minimiser of the problem WITHOUT such hinges is the minimiser of the full
  // problem provided every left-out hinge ends with l >= 0 — which is verified after convergence; a violation
  // repeats the interior point iteration with all hinges, started from the (dynamically feasible) point reached.  Left out: hinges with l > prune at the nominal point even for d = max_sd
  // (obstacles the robot is far from: ~3/4 of the hinges of the bench workload), so the per-hinge passes — about
  // two thirds of this kernel's time (profiles/ncu_r02_ksu_lines_before.md) — run over the rest only.
  const int NW = (N + 31) / 32 > 0 ? (N + 31) / 32 : 1;
  const bool can_prune = acc && N > 0 && P.prune > 0;
  int status = 1, it = 0, it_total = 0;
  W.restarts = 0;
  for (int attempt = 0; attempt < 2; ++attempt) {
  const bool full = !can_prune || attempt == 1;
  W.restarts = attempt;
  // ---- initial iterate: roll the linearised model out from s_0 (second attempt: continue from the point reached) ----
  if (lane == 0 && attempt == 0) {
    W.s[0] = W.lins[0]; W.s[1] = W.lins[1]; W.s[2] = W.lins[2];
    for (int t = 0; t < T; ++t) {
      const Real* s0 = W.s + 3 * t;
      Real u0 = W.u[2 * t], u1 = W.u[2 * t + 1];
      W.s[3 * t + 3] = s0[0] + W.Aj[2 * t] * s0[2] + W.Bj[6 * t] * u0 + W.Bj[6 * t + 1] * u1 + W.Cj[3 * t];
      W.s[3 * t + 4] = s0[1] + W.Aj[2 * t + 1] * s0[2] + W.Bj[6 * t + 2] * u0 + W.Bj[6 * t + 3] * u1 + W.Cj[3 * t + 1];
      W.s[3 * t + 5] = s0[2] + W.Bj[6 * t + 4] * u0 + W.Bj[6 * t + 5] * u1 + W.Cj[3 * t + 2];
    }
  }
  ctx.sync();
  const Real mu0 = P.mu0 > 0 ? (Real)P.mu0 : (Real)1;
  int nrows = 0;
  for (int t = lane; t < T; t += nl) {
    _Pragma("unroll 1") for (int c = 0; c < 10; ++c) {
      Row<Real> r = su_row<Real>(P, W, t, c);
      Real sv = r.live ? rmax(r.g, (Real)1e-2) : (Real)1;
      W.bs[10 * t + c] = sv;
      W.bnu[10 * t + c] = r.live ? mu0 / sv : (Real)0;
      if (r.live) ++nrows;
    }
    if (acc) {
      Real dx = W.s[3 * t + 3] - W.pref[2 * t], dy = W.s[3 * t + 4] - W.pref[2 * t + 1];
      for (int w = 0; w < NW; ++w) W.hmask[t * NW + w] = 0u;
      // the two hinges nearest to activity always take part: they keep d_t's direction curved (a stage without any
      // hinge leaves d_t to its bounds alone, on which Mehrotra's single step length was seen to cycle)
      Real lmin1 = (Real)1e30, lmin2 = (Real)1e30;
      if (!full)
        for (int o = 0; o < N; ++o) {
          const Real lp = (Real)W.hx[o * T + t] * dx + (Real)W.hy[o * T + t] * dy + (Real)W.hc[o * T + t];
          if (lp < lmin1) { lmin2 = lmin1; lmin1 = lp; } else if (lp < lmin2) lmin2 = lp;
        }
      for (int o = 0; o < N; ++o) {
        const Real lp = (Real)W.hx[o * T + t] * dx + (Real)W.hy[o * T + t] * dy + (Real)W.hc[o * T + t];
        if (!full && lp - (Real)P.dmax > (Real)P.prune && lp > lmin2) continue;        // left out, verified after convergence
        W.hmask[t * NW + (o >> 5)] |= 1u << (o & 31);
        Real l = lp - W.d[t];
        Real sv = (l + sqrt_(l * l + 4 * mu0 / ro1)) / 2;
        W.hs[o * T + t] = sv;
        W.hnu[o * T + t] = mu0 / sv;
        ++nrows;
      }
    } else {
      for (int w = 0; w < NW; ++w) W.hmask[t * NW + w] = (N - 32 * w >= 32) ? 0xffffffffu : ((N - 32 * w > 0) ? ((1u << (N - 32 * w)) - 1u) : 0u);
    }
  }
  const Real Mrows = ctx.sum((Real)nrows);
  ctx.sync();
  // RDA_SU_TOL: complementarity / residual tolerance of the float64 iteration (default 1e-9; ECOS stops at 1e-8)
#ifndef RDA_SU_TOL
#define RDA_SU_TOL 1e-9
#endif
  const Real tol_mu = sizeof(Real) == 4 ? (Real)1e-6 : (Real)RDA_SU_TOL;
  const Real tol_r = sizeof(Real) == 4 ? (Real)1e-5 : (Real)RDA_SU_TOL;
  const Real reg = (Real)1e-9;
#ifndef RDA_SU_TOL_STEP
#define RDA_SU_TOL_STEP 1e-6
#endif
  const Real tol_step = sizeof(Real) == 4 ? (Real)2e-4 : (Real)RDA_SU_TOL_STEP;
  const Real tol_floor = sizeof(Real) == 4 ? (Real)1e-7 : (Real)1e-13;
  Real last_step = 1e30f;       // size of the previous Newton update (stationarity proxy)
  status = 1;
  const int it_cap = full ? P.max_iter : (P.max_iter < 24 ? P.max_iter : 24);     // pruned attempt: give up earlier
  for (it = 0; it < it_cap; ++it) {
    Real sigma_mu = 0;
    Real mu = 0;
    for (int phase = 0; phase < 2; ++phase) {
      // ---- assemble stage gradients (and, in phase 0, Hessian weights) ----
      Real acc_mu = 0, acc_r = 0;
      for (int t = lane; t < T; t += nl) {
        Real* gw = W.gw + 8 * t;
        const Real* sn = W.s + 3 * t + 3;
        const Real tw = 2 * (Real)P.ws;
        gw[0] = tw * (sn[0] - W.ref[3 * t + 3]);
        gw[1] = tw * (sn[1] - W.ref[3 * t + 4]);
        gw[2] = (P.dynamics == RDA_DYN_OMNI ? (Real)0 : tw * (sn[2] - W.ref[3 * t + 5]))
                + ro2 * (W.Skk[t] * (sn[2] - W.lins[3 * t + 2]) + W.Sgk[t]);
        gw[3] = 2 * (Real)P.wu * (W.u[2 * t] - W.vref) + reg * W.u[2 * t];
        gw[4] = reg * W.u[2 * t + 1];
        gw[5] = N > 0 ? -(Real)P.slack_gain + reg * W.d[t] : (Real)0;
        gw[6] = 0; gw[7] = 0;
        Real wb[5] = {0, 0, 0, 0, 0};
        _Pragma("unroll 1") for (int c = 0; c < 10; ++c) {
          Row<Real> r = su_row<Real>(P, W, t, c);
          if (!r.live) continue;
          Real sv = W.bs[10 * t + c], nu = W.bnu[10 * t + c];
          Real res = r.g - sv;
          const Real isv = rcp_(sv);
          Real om = nu * isv;
          Real term;
          if (phase == 0) {
            term = -om * res;
            acc_mu += sv * nu;
            acc_r = rmax(acc_r, abs_(res));
          } else {
            Real dir = su_row_dir<Real>(r, W.dza + 5 * t, W.dva + 3 * t);
            Real dsa = dir + res;
            Real dna = -nu - om * dsa;
            term = (sigma_mu - dsa * dna) * isv - om * res;
          }
          // g -= grad * term
          gw[r.comp] -= r.sgn * term;
          if (r.rate) gw[r.comp + 3] += r.sgn * term;
          if (phase == 0) wb[(r.rate ? 3 : 0) + (r.comp - 3)] += om;
        }
        if (phase == 0) for (int k = 0; k < 5; ++k) W.wb[5 * t + k] = wb[k];
        Real m0 = 0, m1 = 0, m2 = 0, m3 = 0, m4 = 0, m5 = 0;
        Real dx = sn[0] - W.pref[2 * t], dy = sn[1] - W.pref[2 * t + 1];
        Real dd = W.d[t];
        Real g0 = gw[0], g1 = gw[1], g5 = gw[5];     // accumulated in registers: no store inside the hinge loop
        // hinges in chunks of RDA_SU_CH: all (global-memory) loads of a chunk are issued before its arithmetic
        const Real adx = phase == 1 ? W.dza[5 * t + 5] : (Real)0, ady = phase == 1 ? W.dza[5 * t + 6] : (Real)0;
        const Real add = phase == 1 ? W.dva[3 * t + 2] : (Real)0;
        for (int w_ = 0; w_ < NW; ++w_) {
          unsigned m_ = W.hmask[t * NW + w_];
          while (m_) {
          int oi[RDA_SU_CH], cnt_ = 0;
          Real axv[RDA_SU_CH], ayv[RDA_SU_CH], hcv[RDA_SU_CH], svv[RDA_SU_CH], nuv[RDA_SU_CH];
#pragma unroll
          for (int k = 0; k < RDA_SU_CH; ++k) {
            if (m_) { oi[k] = (32 * w_ + ctz_(m_)) * T + t; m_ &= m_ - 1u; cnt_ = k + 1; } else oi[k] = oi[0];
            const int i = oi[k];
            axv[k] = W.hx[i]; ayv[k] = W.hy[i]; hcv[k] = W.hc[i];
            svv[k] = acc ? (Real)W.hs[i] : (Real)1; nuv[k] = acc ? (Real)W.hnu[i] : (Real)1;
          }
#pragma unroll
          for (int k = 0; k < RDA_SU_CH; ++k) {
            if (k >= cnt_) break;
            const Real ax = axv[k], ay = ayv[k];
            const Real l = ax * dx + ay * dy + hcv[k] - dd;
            Real tk, om;
            if (acc) {
              const Real sv = svv[k], nu = nuv[k];
              const Real nr = nu * iro1;
              const Real res = l + nr - sv;
              const Real iden = rcp_(sv + nr);
              om = nu * iden;
              if (phase == 0) {
                tk = om * (nr - res);
                acc_mu += sv * nu;
                acc_r = rmax(acc_r, abs_(res));
              } else {
                const Real dir = ax * adx + ay * ady - add;
                const Real dna = -om * (sv + res + dir);
                const Real dsa = dir + dna * iro1 + res;
                const Real cc = sv * nu - sigma_mu + dsa * dna;
                tk = nu - (cc + nu * res) * iden;
              }
            } else {
              om = ro1;               // plain quadratic 1/2 ro1 Im^2  (rda_solver.py:378-379)
              tk = -ro1 * l;
            }
            g0 -= ax * tk; g1 -= ay * tk; g5 += tk;
            if (phase == 0) {
              m0 += om * ax * ax; m1 += om * ax * ay; m2 -= om * ax;
              m3 += om * ay * ay; m4 -= om * ay; m5 += om;
            }
          }
          }
        }
        // eliminate d_t (it enters stage t only): Schur complement on Q_dd = reg + barrier weights + sum om
        if (phase == 0) {
          const Real iq = N > 0 ? rcp_(reg + wb[2] + m5) : (Real)1;
          const Real e0 = m2 * iq, e1 = m4 * iq;
          Real* M = W.Wm + 3 * t;
          M[0] = m0 - m2 * e0; M[1] = m1 - m2 * e1; M[2] = m3 - m4 * e1;
          W.Ed[3 * t] = e0; W.Ed[3 * t + 1] = e1; W.Ed[3 * t + 2] = iq;
        }
        W.g5q[t] = g5 * W.Ed[3 * t + 2];
        gw[0] = g0 - W.Ed[3 * t] * g5; gw[1] = g1 - W.Ed[3 * t + 1] * g5; gw[5] = g5;
      }
      if (phase == 0) {
        mu = ctx.sum(acc_mu) / Mrows;
        Real rmx = ctx.max(acc_r);
#ifdef RDA_SU_DEBUG
        printf("it %d mu %.3e rmx %.3e last_step %.3e\n", it, (double)mu, (double)rmx, (double)last_step);
#endif
        if (!finite_(mu)) { status = 2; break; }
        // converged: complementarity and residuals small, and the last Newton update small
        // (degenerate problems approach the solution like sqrt(mu): stop at the rounding floor)
        if (mu < tol_mu && rmx < tol_r && (last_step < tol_step || mu < tol_floor)) { status = 0; break; }
      }
      ctx.sync();
      su_riccati<Real, Ctx>(P, W, ctx, phase == 0, phase == 0 ? W.dza : W.dz, phase == 0 ? W.dva : W.dv);
      // ---- step lengths ----
      const Real* dz = phase == 0 ? W.dza : W.dz;
      const Real* dv = phase == 0 ? W.dva : W.dv;
      Real rmaxr = 0, s0 = 0, s1 = 0, s2 = 0;   // rmaxr = max over rows of (-delta / value): 1 / max step
      for (int t = lane; t < T; t += nl) {
        _Pragma("unroll 1") for (int c = 0; c < 10; ++c) {
          Row<Real> r = su_row<Real>(P, W, t, c);
          if (!r.live) continue;
          Real sv = W.bs[10 * t + c], nu = W.bnu[10 * t + c];
          Real res = r.g - sv;
          Real dir = su_row_dir<Real>(r, dz + 5 * t, dv + 3 * t);
          Real ds = dir + res, dn;
          const Real ip = rcp_(sv * nu);
          const Real isv = nu * ip, inu = sv * ip, om = nu * isv;
          if (phase == 0) dn = -nu - om * ds;
          else {
            Real dira = su_row_dir<Real>(r, W.dza + 5 * t, W.dva + 3 * t);
            Real dsa = dira + res;
            Real dna = -nu - om * dsa;
            dn = (sigma_mu - dsa * dna) * isv - nu - om * ds;
          }
          rmaxr = rmax(rmaxr, rmax(-ds * isv, -dn * inu));
          s0 += sv * nu; s1 += sv * dn + nu * ds; s2 += ds * dn;
        }
        if (acc) {
          const Real dx = W.s[3 * t + 3] - W.pref[2 * t], dy = W.s[3 * t + 4] - W.pref[2 * t + 1], dd = W.d[t];
          const Real zdx = dz[5 * t + 5], zdy = dz[5 * t + 6], zdd = dv[3 * t + 2];
          const Real adx = W.dza[5 * t + 5], ady = W.dza[5 * t + 6], add = W.dva[3 * t + 2];
          for (int w_ = 0; w_ < NW; ++w_) {
            unsigned m_ = W.hmask[t * NW + w_];
            while (m_) {
            int oi[RDA_SU_CH], cnt_ = 0;
            Real axv[RDA_SU_CH], ayv[RDA_SU_CH], hcv[RDA_SU_CH], svv[RDA_SU_CH], nuv[RDA_SU_CH];
#pragma unroll
            for (int k = 0; k < RDA_SU_CH; ++k) {
              if (m_) { oi[k] = (32 * w_ + ctz_(m_)) * T + t; m_ &= m_ - 1u; cnt_ = k + 1; } else oi[k] = oi[0];
              const int i = oi[k];
              axv[k] = W.hx[i]; ayv[k] = W.hy[i]; hcv[k] = W.hc[i]; svv[k] = W.hs[i]; nuv[k] = W.hnu[i];
            }
#pragma unroll
            for (int k = 0; k < RDA_SU_CH; ++k) {
              if (k >= cnt_) break;
              const Real ax = axv[k], ay = ayv[k], sv = svv[k], nu = nuv[k];
              const Real l = ax * dx + ay * dy + hcv[k] - dd;
              const Real nr = nu * iro1;
              const Real res = l + nr - sv;
              const Real iden = rcp_(sv + nr);
              const Real om = nu * iden;
              const Real dir = ax * zdx + ay * zdy - zdd;
              Real cc = sv * nu;
              if (phase == 1) {
                const Real dira = ax * adx + ay * ady - add;
                const Real dna = -om * (sv + res + dira);
                const Real dsa = dira + dna * iro1 + res;
                cc = sv * nu - sigma_mu + dsa * dna;
              }
              const Real dn = -(cc + nu * res + nu * dir) * iden;
              const Real ds = dir + dn * iro1 + res;
              const Real ip = rcp_(sv * nu);
              rmaxr = rmax(rmaxr, rmax(-ds * nu * ip, -dn * sv * ip));
              s0 += sv * nu; s1 += sv * dn + nu * ds; s2 += ds * dn;
            }
            }
          }
        }
      }
      rmaxr = ctx.max(rmaxr);
      const Real amax = rmaxr > (Real)1e-30 ? (Real)1 / rmaxr : (Real)1e30;
      if (phase == 0) {
        Real a = rmin((Real)1, amax);
        Real mua = (ctx.sum(s0) + a * ctx.sum(s1) + a * a * ctx.sum(s2)) / Mrows;
        Real sg = mua / mu;
        sg = sg * sg * sg;
        sigma_mu = rmin(sg, (Real)1) * mu;
      } else {
        // fixed fraction to the boundary: an adaptive one saved iterations but cycled on a box-only problem (DESIGN.md §4)
        Real a = rmin((Real)1, (Real)0.995 * amax);
#ifdef RDA_SU_DEBUG
        printf("   alpha %.3e sigma_mu %.3e\n", (double)a, (double)sigma_mu);
#endif
        // ---- update (needs the corrector quantities once more) ----
        for (int t = lane; t < T; t += nl) {
          // rows first: they read the OLD iterate through su_row
          Real gsave[10];
          _Pragma("unroll 1") for (int c = 0; c < 10; ++c) { Row<Real> r = su_row<Real>(P, W, t, c); gsave[c] = r.g; }
          _Pragma("unroll 1") for (int c = 0; c < 10; ++c) {
            Row<Real> r = su_row<Real>(P, W, t, c);
            if (!r.live) continue;
            Real sv = W.bs[10 * t + c], nu = W.bnu[10 * t + c];
            Real res = gsave[c] - sv;
            Real dir = su_row_dir<Real>(r, W.dz + 5 * t, W.dv + 3 * t);
            Real ds = dir + res;
            Real dira = su_row_dir<Real>(r, W.dza + 5 * t, W.dva + 3 * t);
            Real dsa = dira + res;
            const Real isv = rcp_(sv), om = nu * isv;
            Real dna = -nu - om * dsa;
            Real dn = (sigma_mu - dsa * dna) * isv - nu - om * ds;
            W.bs[10 * t + c] = sv + a * ds;
            W.bnu[10 * t + c] = nu + a * dn;
          }
          if (acc) {
            const Real dx = W.s[3 * t + 3] - W.pref[2 * t], dy = W.s[3 * t + 4] - W.pref[2 * t + 1], dd = W.d[t];
            const Real zdx = W.dz[5 * t + 5], zdy = W.dz[5 * t + 6], zdd = W.dv[3 * t + 2];
            const Real adx = W.dza[5 * t + 5], ady = W.dza[5 * t + 6], add = W.dva[3 * t + 2];
            for (int w_ = 0; w_ < NW; ++w_) {
              unsigned m_ = W.hmask[t * NW + w_];
              while (m_) {
              int oi[RDA_SU_CH], cnt_ = 0;
              Real axv[RDA_SU_CH], ayv[RDA_SU_CH], hcv[RDA_SU_CH], svv[RDA_SU_CH], nuv[RDA_SU_CH];
#pragma unroll
              for (int k = 0; k < RDA_SU_CH; ++k) {
                if (m_) { oi[k] = (32 * w_ + ctz_(m_)) * T + t; m_ &= m_ - 1u; cnt_ = k + 1; } else oi[k] = oi[0];
                const int i = oi[k];
                axv[k] = W.hx[i]; ayv[k] = W.hy[i]; hcv[k] = W.hc[i]; svv[k] = W.hs[i]; nuv[k] = W.hnu[i];
              }
#pragma unroll
              for (int k = 0; k < RDA_SU_CH; ++k) {
                if (k >= cnt_) break;
                const Real ax = axv[k], ay = ayv[k], sv = svv[k], nu = nuv[k];
                const Real l = ax * dx + ay * dy + hcv[k] - dd;
                const Real nr = nu * iro1;
                const Real res = l + nr - sv;
                const Real iden = rcp_(sv + nr);
                const Real om = nu * iden;
                const Real dir = ax * zdx + ay * zdy - zdd;
                const Real dira = ax * adx + ay * ady - add;
                const Real dna = -om * (sv + res + dira);
                const Real dsa = dira + dna * iro1 + res;
                const Real cc = sv * nu - sigma_mu + dsa * dna;
                const Real dn = -(cc + nu * res + nu * dir) * iden;
                const Real ds = dir + dn * iro1 + res;
                W.hs[oi[k]] = sv + a * ds;
                W.hnu[oi[k]] = nu + a * dn;
              }
              }
            }
          }
        }
        ctx.sync();   // every lane has finished reading the old (s, u, d) of its neighbours
        Real stepmax = 0;
        for (int t = lane; t < T; t += nl) {
          stepmax = rmax(stepmax, rmax(abs_(W.dv[3 * t]), rmax(abs_(W.dv[3 * t + 1]), abs_(W.dv[3 * t + 2]))));
          W.u[2 * t] += a * W.dv[3 * t]; W.u[2 * t + 1] += a * W.dv[3 * t + 1];
          if (N > 0) W.d[t] += a * W.dv[3 * t + 2];
          W.s[3 * t + 3] += a * W.dz[5 * t + 5];
          W.s[3 * t + 4] += a * W.dz[5 * t + 6];
          W.s[3 * t + 5] += a * W.dz[5 * t + 7];
        }
        last_step = a * ctx.max(stepmax);
        ctx.sync();
      }
    }
    if (status != 1) break;
  }
  it_total += it;
  if (full || status == 2) break;
  if (status == 1) continue;          // the pruned problem did not converge (iteration cap): repeat with all hinges
  // verification of the left-out hinges at the solution: any l < 0 means the pruned problem was not equivalent
  {
    int viol = 0;
    for (int t = lane; t < T; t += nl) {
      const Real dx = W.s[3 * t + 3] - W.pref[2 * t], dy = W.s[3 * t + 4] - W.pref[2 * t + 1], dd = W.d[t];
      for (int o = 0; o < N; ++o) {
        if (W.hmask[t * NW + (o >> 5)] & (1u << (o & 31))) continue;
        const Real l = (Real)W.hx[o * T + t] * dx + (Real)W.hy[o * T + t] * dy + (Real)W.hc[o * T + t] - dd;
        if (l < (Real)0) viol = 1;
      }
    }
    viol = ctx.max(viol);
    if (!viol) break;
  }
  ctx.sync();
  }   // attempt
  if (iters_out) *iters_out = it_total;
  return status;
}

}  // namespace rda
