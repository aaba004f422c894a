// b2k_rne_gen.h -- interface of the robot-specialised RNE code generator (b2k_rne_gen.cpp).
#pragma once

#include <string>
#include <vector>

#include "b2k_common.cuh"

struct b2k_gen_opts {
    int mode = B2K_GEN_RNE; // B2K_GEN_RNE..B2K_GEN_RNE_WRENCH (b2k_common.cuh)
    int grav_mask = 7;  // bit k: base acceleration component k may be non-zero
    int has_fext = 0;   // a tip wrench is given
};

struct b2k_gen_out {
    std::string source;         // one __device__ function `rne_row(C, grav, fext, st, ct, in1, in2, out)` in terms of `real`
    std::vector<double> consts; // the constant bank C the function reads
    int n_mul = 0, n_fma = 0, n_add = 0;
    std::string error;
};

// A rigid-body tree in the form Robot.rne walks it (reference Robot.py:1704-1903): n joint groups in link order, group j
// hangs off group parent[j] (-1: the base) through the constant transform C[j] (3x4 row-major; the static links of the
// group and the constant part of the joint link folded) followed by ONE joint of kind axis[j] (B2K_RX..B2K_TZ, flip[j])
// reading q[jindex[j]]; I6[j] is the 6x6 spatial inertia of the group in the joint link's frame, [linear; angular] order.
#define B2K_TREE_MAX 16
struct b2k_tree_s {
    int n;
    int parent[B2K_TREE_MAX], axis[B2K_TREE_MAX], flip[B2K_TREE_MAX], jindex[B2K_TREE_MAX];
    double C[B2K_TREE_MAX][12];
    double I6[B2K_TREE_MAX][36];
    void *spec;
};
int b2k_tree_generate(const b2k_tree_s *t, const b2k_gen_opts &o, b2k_gen_out &out);

// outputs of the generated function: RNE / GRAVLOAD / ITORQUE n values; INERTIA / CORIOLIS n*n; ACCEL n*n + n
// (rows of M followed by torque - rne(q, qd, 0), the wrapper solves the system); RNE_WRENCH n + 6 (tau, then the wrench
// [f; m] the base exerts on link 1, in frame 0, moment about its origin).  Trees (b2k_tree_generate) reject RNE_WRENCH.
// Trees only: RNE_DERIV generates `rne_deriv_row(C, grav, fext, st, ct, qq, qd, qdd, dq, dqd)`, dq / dqd the n x n blocks
// d tau_i / d q_k and d tau_i / d qd_k (i group order, k q order); ACCEL_DERIV generates the ACCEL `rne_row` followed by
// that `rne_deriv_row` over one constant bank.  TREE_REGRESSOR (trees only) generates
// `rne_regressor_row(C, grav, fext, st, ct, qq, qd, qdd, i, y)`: joint row i of the regressor, y[10k + c] = d tau_i / d pi_c
// of group k (10 n reals, group order, exact 0 unless group k is i or hangs below it).
int b2k_rne_generate(const b2k_rne_s *r, const b2k_gen_opts &o, b2k_gen_out &out);
