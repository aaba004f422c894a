// fp64 instantiations of the IK kernels with the null-space term (b2k_ikine_null)
#include "b2k_ik.cuh"
int b2k_ik_ns_launch_f64(const b2k_chain_s *c, const void *Tep, long long nprob, const void *q0, int ilimit, int slimit,
                         double tol, int reject_jl, const double *we, double lambda, int method, unsigned long long seed,
                         int rng_per_row, void *q_out, int *success, int *iterations, int *searches, void *residual,
                         const IkNullArgs &ns, cudaStream_t st)
{
    return ik_ns_launch<double>(c, Tep, nprob, q0, ilimit, slimit, tol, reject_jl, we, lambda, method, seed, rng_per_row,
                                q_out, success, iterations, searches, residual, ns, st);
}
