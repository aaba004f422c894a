// instantiations of the RNE kernel for both dtypes
#include "b2k_rne.cuh"
int b2k_rne_generic_rne(const b2k_rne_s *r, int op, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    return dtype == B2K_F64 ? rne_generic_launch<double, B2K_GEN_RNE>(r, op, a, st) : rne_generic_launch<float, B2K_GEN_RNE>(r, op, a, st);
}
