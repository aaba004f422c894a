// fp64 instantiations of the IK kernels with the quadratic-programming step (b2k_ikine_qp)
#include "b2k_ik.cuh"
int b2k_ik_qp_launch_f64(const b2k_chain_s *c, const void *Tep, long long nprob, const void *q0, int ilimit, int slimit,
                         double tol, int reject_jl, const double *we, unsigned long long seed, int rng_per_row,
                         void *q_out, int *success, int *iterations, int *searches, void *residual, const IkQpArgs &qp,
                         cudaStream_t st)
{
    return ik_qp_launch<double>(c, Tep, nprob, q0, ilimit, slimit, tol, reject_jl, we, seed, rng_per_row, q_out, success,
                                iterations, searches, residual, qp, st);
}
