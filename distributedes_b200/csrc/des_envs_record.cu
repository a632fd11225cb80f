// The recording instantiations of rollout_pendulum_kernel (des_rollout_record[_solutions], des_envs.cu), in a translation
// unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

// The kernels first, both modes at each width: cicc's code for rollout_pendulum_kernel<8, true, RecordArgs> depends on
// the order in which the unit instantiates them.  This order keeps the schedule the recording kernels were measured
// with; one mode after the other, as the two launchers alone would instantiate them, hoists an address computation.
template __global__ void rollout_pendulum_kernel<1, true, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<1, false, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<2, true, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<2, false, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<4, true, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<4, false, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<6, true, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<6, false, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<8, true, RecordArgs>(RecordArgs);
template __global__ void rollout_pendulum_kernel<8, false, RecordArgs>(RecordArgs);
template int rollout_kernels<false, RecordArgs>(const RecordArgs &, int, unsigned, size_t, cudaStream_t);
template int rollout_kernels<true, RecordArgs>(const RecordArgs &, int, unsigned, size_t, cudaStream_t);

}  // namespace des
