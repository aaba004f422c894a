// fp32 instantiations of the analytical derivatives of the recursion (rne_derivatives, accel_derivatives)
#include "b2k_rne.cuh"
int b2k_rne_generic_deriv_f32(const b2k_rne_s *r, int op, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    return rne_generic_launch<float, B2K_GEN_RNE_DERIV, B2K_GEN_ACCEL_DERIV>(r, op, a, st);
}
