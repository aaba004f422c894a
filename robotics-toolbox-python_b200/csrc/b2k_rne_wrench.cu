// instantiations of the RNE kernel that also writes the base wrench, for both dtypes (a unit of its own, so that
// b2k_rne.o and its k_rne instantiations are untouched by them)
#include "b2k_rne.cuh"
int b2k_rne_wrench_launch(const b2k_rne_s *r, int dtype, const void *q, const void *qd, const void *qdd, long long nrows,
                          const double *grav, const double *fext, void *tau, void *wbase, cudaStream_t st)
{
    if (dtype == B2K_F64) return rne_launch<double, true>(r, q, qd, qdd, nrows, grav, fext, tau, wbase, st);
    return rne_launch<float, true>(r, q, qd, qdd, nrows, grav, fext, tau, wbase, st);
}
