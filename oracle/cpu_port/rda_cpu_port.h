// TEST / BASELINE INFRASTRUCTURE (oracle/): the whole-batch entry point of the CPU port (rda_cpu_port.cpp), for the
// CPU twins of tests/cpu_twin that are linked with it into one library and call it instance by instance.
#pragma once
#include "../../include/rda_b200.h"

// The ADMM loop of rda_kernels.cu over B instances (OpenMP over instances; nthreads <= 0: the OpenMP default).
// Layouts as in include/rda_b200.h; every instance starts cold.  iters_out and fails_out [B][4] may be NULL.
extern "C" int port_solve_batch(const rda_config* cfg, const rda_tunables* tun, int B, const float* nom_s,
                                const float* nom_u, const float* ref_s, const float* ref_speed, const float* obs_A,
                                const float* obs_b, const int* obs_kind, const int* obs_count, int tv, int iter_num,
                                float thr, float* u_opt, float* s_opt, float* resi_pri, float* resi_dual, int* iters_out,
                                int* fails_out, int nthreads);
