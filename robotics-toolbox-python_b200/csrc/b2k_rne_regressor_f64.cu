// fp64 instantiations of the dynamics regressor and its normal equations (rne_regressor, regressor_gram; the tree
// regressor's normal equations)
#include "b2k_rne.cuh"
int b2k_rne_generic_regressor_f64(const b2k_rne_s *r, int op, int dtype, const b2k_rne_args &a, cudaStream_t st)
{
    return rne_generic_launch<double, B2K_GEN_RNE_REGRESSOR>(r, op, a, st);
}
int b2k_rne_regressor_gram_f64(const b2k_rne_s *r, const b2k_rne_args &a, const void *tau, const double *w, double *G, double *b,
                              double *s, cudaStream_t st)
{
    return rne_regressor_gram<double>(r, a, tau, w, G, b, s, st);
}
// the tree regressor's normal equations (b2k_tree_regressor_gram): the same chunks over the generated kernel, p = 10 n
int b2k_tree_regressor_gram_f64(b2k_tree_t t, int n, const b2k_rne_args &a, const void *tau, const double *w, double *G,
                                double *b, double *s, cudaStream_t st)
{
    return regressor_gram<double>(n, 10 * n, a, tau, w, G, b, s, st,
                                [&](const b2k_rne_args &ca) { return b2k_tree_regressor_rows(t, B2K_F64, ca, st); });
}
