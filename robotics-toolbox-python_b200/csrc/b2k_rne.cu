// instantiations of the RNE kernel for both dtypes
#include "b2k_rne.cuh"
int b2k_rne_launch(const b2k_rne_s *r, int dtype, const void *q, const void *qd, const void *qdd, long long nrows,
                   const double *grav, const double *fext, void *tau, cudaStream_t st)
{
    if (dtype == B2K_F64) return rne_launch<double, false>(r, q, qd, qdd, nrows, grav, fext, tau, nullptr, st);
    return rne_launch<float, false>(r, q, qd, qdd, nrows, grav, fext, tau, nullptr, st);
}
