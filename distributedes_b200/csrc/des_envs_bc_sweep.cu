// The behaviour-writing sweep instantiations of rollout_pendulum_kernel (des_rollout_eval_bc_sweep, des_envs.cu), in a
// translation unit of their own: see des_envs.cuh.
#include "des_envs.cuh"

namespace des {

int rollout_bc_sweep_launch(const BcSweepArgs &a, int H, unsigned blocks, size_t smem, cudaStream_t st) {
    void (*kernel)(BcSweepArgs);
    switch (H / 16) {                    // R = H/16 hidden units per lane
        case 1: kernel = rollout_pendulum_kernel<1, false, BcSweepArgs>; break;
        case 2: kernel = rollout_pendulum_kernel<2, false, BcSweepArgs>; break;
        case 4: kernel = rollout_pendulum_kernel<4, false, BcSweepArgs>; break;
        case 6: kernel = rollout_pendulum_kernel<6, false, BcSweepArgs>; break;
        default: kernel = rollout_pendulum_kernel<8, false, BcSweepArgs>; break;
    }
    return launch_smem("rollout_pendulum_kernel", kernel, blocks, 32, smem, st, a);
}

}  // namespace des
