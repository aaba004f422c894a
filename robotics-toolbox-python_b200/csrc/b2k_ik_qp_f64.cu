// fp64 instantiations of the IK kernels with the quadratic-programming step (b2k_ikine_qp)
#include "b2k_ik.cuh"
int b2k_ik_qp_launch_f64(const b2k_chain_s *c, const IkArgs &a, cudaStream_t st) { return ik_launch<double, 2>(c, a, st); }
