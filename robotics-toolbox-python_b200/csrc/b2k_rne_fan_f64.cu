// fp64 instantiations of the dynamics fan-out kernels (inertia, gravload, itorque, coriolis, accel)
#include "b2k_rne.cuh"
int b2k_rne_generic_fan_f64(const b2k_rne_s *r, int op, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    return rne_generic_launch<double, B2K_GEN_INERTIA, B2K_GEN_GRAVLOAD, B2K_GEN_ITORQUE, B2K_GEN_CORIOLIS, B2K_GEN_ACCEL>(r, op, a, st);
}
