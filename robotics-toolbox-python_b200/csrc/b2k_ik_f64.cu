// fp64 instantiations of the fused LM IK kernel
#include "b2k_ik.cuh"
int b2k_ik_launch_f64(const b2k_chain_s *c, const IkArgs &a, cudaStream_t st) { return ik_launch<double, 0>(c, a, st); }
