// The row-mode sweep instantiations of rollout_pendulum_kernel (des_rollout_eval_solutions_sweep, des_envs.cu), in a
// translation unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

int rollout_rows_sweep_launch(const SweepArgs &a, int H, unsigned blocks, size_t smem, cudaStream_t st) {
    void (*kernel)(SweepArgs);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rollout_pendulum_kernel<1, true, SweepArgs>; break;
        case 2: kernel = rollout_pendulum_kernel<2, true, SweepArgs>; break;
        case 4: kernel = rollout_pendulum_kernel<4, true, SweepArgs>; break;
        case 6: kernel = rollout_pendulum_kernel<6, true, SweepArgs>; break;
        default: kernel = rollout_pendulum_kernel<8, true, SweepArgs>; break;
    }
    return launch_smem("rollout_pendulum_kernel", kernel, blocks, 32, smem, st, a);
}

}  // namespace des
