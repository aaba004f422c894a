// fp32 instantiations of the analytical derivatives of the recursion (rne_derivatives, accel_derivatives)
#include "b2k_rne.cuh"
int b2k_rne_deriv_launch_f32(const b2k_rne_s *r, int mode, const void *in0, const void *in1, const void *in2, long long nrows,
                             const double *grav, const double *fext, void *out0, void *out1, void *out2, cudaStream_t st)
{
    return rne_deriv_launch<float>(r, mode, in0, in1, in2, nrows, grav, fext, out0, out1, out2, st);
}
