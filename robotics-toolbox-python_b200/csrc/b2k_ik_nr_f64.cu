// f64 instantiations of the IK kernels with the pseudo-inverse step (Newton-Raphson / Gauss-Newton)
#include "b2k_ik.cuh"
int b2k_ik_nr_launch_f64(const b2k_chain_s *c, const IkArgs &a, cudaStream_t st) { return ik_launch<double, 1>(c, a, st); }
