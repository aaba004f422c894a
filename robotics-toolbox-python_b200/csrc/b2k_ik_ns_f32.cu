// fp32 instantiations of the IK kernels with the null-space term (b2k_ikine_null)
#include "b2k_ik.cuh"
int b2k_ik_ns_launch_f32(const b2k_chain_s *c, const IkArgs &a, cudaStream_t st)
{
    const bool pinv = a.method == B2K_IK_NR || a.method == B2K_IK_GN;
    return pinv ? ik_launch<float, 1, true>(c, a, st) : ik_launch<float, 0, true>(c, a, st);
}
