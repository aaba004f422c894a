// fp32 instantiations of the dynamics regressor and its normal equations (rne_regressor, regressor_gram)
#include "b2k_rne.cuh"
int b2k_rne_generic_regressor_f32(const b2k_rne_s *r, int op, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    return rne_generic_launch<float, B2K_GEN_RNE_REGRESSOR>(r, op, a, st);
}
int b2k_rne_regressor_gram_f32(const b2k_rne_s *r, const b2k_rne_args &a, const void *tau, const double *w, double *G, double *b,
                              double *s, cudaStream_t st)
{
    return rne_regressor_gram<float>(r, a, tau, w, G, b, s, st);
}
