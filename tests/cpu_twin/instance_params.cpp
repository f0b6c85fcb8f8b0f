// CPU twin of the per-instance parameter table (rda_set_instance_params) — test infrastructure only.
// The g++ build of the kernels' cores (oracle/cpu_port) solves with one rda_config / rda_tunables per call; this twin
// gives instance b its own pair, selected from row b of the table with the helpers the kernels use: su_params_row for
// the su-QP parameters (su_instance, k_admm_small) and inst_ro2 for the cells' ro2 (the listed cell passes).  Each
// instance is then solved on its own: instances of a batch never interact.  Layouts as port_solve_batch; inst may be
// NULL (the handle's values for every instance, port_solve_batch itself).
#include "../../oracle/cpu_port/rda_cpu_port.cpp"

extern "C" int twin_solve_batch_inst(const rda_config* cfg, const rda_tunables* tun, int B, const float* nom_s,
                                     const float* nom_u, const float* ref_s, const float* ref_speed, const float* obs_A,
                                     const float* obs_b, const int* obs_kind, const int* obs_count, int tv, int iter_num,
                                     float thr, float* u_opt, float* s_opt, float* resi_pri, float* resi_dual,
                                     int* iters_out, int* fails_out, int nthreads, const float* inst) {
  if (!inst)
    return port_solve_batch(cfg, tun, B, nom_s, nom_u, ref_s, ref_speed, obs_A, obs_b, obs_kind, obs_count, tv, iter_num,
                            thr, u_opt, s_opt, resi_pri, resi_dual, iters_out, fails_out, nthreads);
  const size_t T = cfg->receding, N = cfg->max_obs_num, E = cfg->max_edge_num, Tc = tv ? T + 1 : 1;
  for (int b = 0; b < B; ++b) {
    // the handle's values, then row b over them, as su_instance does
    SuParams P;
    P.umax[0] = cfg->max_speed[0]; P.umax[1] = cfg->max_speed[1];
    P.ab[0] = cfg->acce_bound[0]; P.ab[1] = cfg->acce_bound[1];
    P.ws = cfg->ws; P.wu = cfg->wu;
    P.slack_gain = tun->slack_gain; P.dmax = tun->max_sd; P.dmin = tun->min_sd; P.ro1 = tun->ro1; P.ro2 = tun->ro2;
    su_params_row(P, inst + (size_t)b * RDA_INST_PARAMS);
    rda_config c = *cfg;
    rda_tunables t = *tun;
    c.batch = 1;
    c.max_speed[0] = P.umax[0]; c.max_speed[1] = P.umax[1];
    c.acce_bound[0] = P.ab[0]; c.acce_bound[1] = P.ab[1];
    c.ws = P.ws; c.wu = P.wu;
    t.slack_gain = P.slack_gain; t.max_sd = P.dmax; t.min_sd = P.dmin; t.ro1 = P.ro1;
    t.ro2 = inst_ro2(inst, b, tun->ro2);                     // the cells' ro2, as the cell passes select it
    const int rc = port_solve_batch(
        &c, &t, 1, nom_s + b * 3 * (T + 1), nom_u + b * 2 * T, ref_s + b * 3 * (T + 1), ref_speed + b,
        obs_A ? obs_A + b * N * Tc * E * 2 : nullptr, obs_b ? obs_b + b * N * Tc * E : nullptr,
        obs_kind ? obs_kind + b * N : nullptr, obs_count ? obs_count + b : nullptr, tv, iter_num, thr,
        u_opt + b * 2 * T, s_opt + b * 3 * (T + 1), resi_pri + b, resi_dual + b, iters_out ? iters_out + b : nullptr,
        fails_out ? fails_out + 4 * b : nullptr, nthreads);
    if (rc) return rc;
  }
  return 0;
}
