// instantiations of the RNE kernel that also writes the base wrench, for both dtypes (a unit of its own, so that
// b2k_rne.o and its k_rne instantiations are untouched by them)
#include "b2k_rne.cuh"
int b2k_rne_generic_wrench(const b2k_rne_s *r, int op, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    return dtype == B2K_F64 ? rne_generic_launch<double, B2K_GEN_RNE_WRENCH>(r, op, a, st)
                            : rne_generic_launch<float, B2K_GEN_RNE_WRENCH>(r, op, a, st);
}
