// The row-mode sweep instantiations of rollout_pendulum_kernel (des_rollout_eval_solutions_sweep, des_envs.cu), in a
// translation unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

template int rollout_kernels<true, SweepArgs>(const SweepArgs &, int, unsigned, size_t, cudaStream_t);

}  // namespace des
